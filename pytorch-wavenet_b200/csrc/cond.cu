// cond.cu -- global conditioning (WaveNet paper section 2.5): the condition table the forward kernels and the sampler read,
// and the per-sequence frame sums behind the gradient of the conditioning weights.
//
// For one sequence b the condition h_b only adds Vf h_b / Vg h_b to the filter / gate biases, so the block kernels take a
// table [layer][item][2D] of each item's biases bf + Vf h_b | bg + Vg h_b and read it instead of bf / bg: the epilogues do the
// same work as unconditioned ones.  The backward's data gradients do not change (they read the saved tanh / sigmoid).
#include "common.cuh"
#include <cuda_bf16.h>

namespace wn {
namespace cond {

// out[l][i][c] = sum_g V_l[c][g] * h[i][g] + b_l[c], V_l = Vf / b_l = bf (c < D) or Vg / bg (c >= D); V (D, G, 1) contiguous,
// biases may be null; blockIdx.y = layer.  A sequential sum over g in one thread: a one-hot h gives exactly one column of V
// (and V = 0 gives exactly the bias).
__global__ void table_kernel(const float* const* __restrict__ ptrs, int D, int G, const float* __restrict__ h, int n_items,
                             float* __restrict__ out) {
    const int l = blockIdx.y;
    const float* vf = ptrs[4 * l];
    const float* vg = ptrs[4 * l + 1];
    const float* bf = ptrs[4 * l + 2];
    const float* bg = ptrs[4 * l + 3];
    const int n = n_items * 2 * D;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int item = i / (2 * D), c = i % (2 * D);
        const float* v = c < D ? vf + (size_t)c * G : vg + (size_t)(c - D) * G;
        const float* x = h + (size_t)item * G;
        float acc = 0.f;
        for (int g = 0; g < G; ++g) acc = fmaf(__ldg(v + g), __ldg(x + g), acc);
        const float* bias = c < D ? bf : bg;
        out[(size_t)l * n + i] = acc + (bias ? __ldg(bias + (c < D ? c : c - D)) : 0.f);
    }
}

// out[b][c] = sum_{gz <= t < L} dfg[b][t][c], deterministic (fixed summation order, no atomics).  Block (32, FS):
//   frames layout (B, L, C) fp32: lane x owns channel 32 * blockIdx.x + x (a warp reads 128 contiguous bytes of a frame), row y
//     sums the frames gz + y, gz + y + FS, ...
//   chunked pair (B, 2, C/8, L, 8) bf16, value = hi + lo: the block owns chunk blockIdx.x; lane x = 8 * q + e reads channel e
//     of frame gz + 4 * y + q, stepping 4 * FS frames (a warp reads 64 contiguous bytes of each plane).
// The partial sums are then added in a fixed order.
constexpr int FS = 16;
template <bool PAIR>
__global__ void __launch_bounds__(32 * FS) frame_sums_kernel(const void* __restrict__ src, int L, int C, int gz,
                                                             float* __restrict__ out) {
    __shared__ float part[FS][33];
    const int x = threadIdx.x, y = threadIdx.y, b = blockIdx.y;
    float acc = 0.f;
    if constexpr (PAIR) {
        const int e = x & 7, q = x >> 3, ck = blockIdx.x;
        const __nv_bfloat16* hi = reinterpret_cast<const __nv_bfloat16*>(src) + ((size_t)b * 2 * (C / 8) + ck) * L * 8 + e;
        const __nv_bfloat16* lo = hi + (size_t)(C / 8) * L * 8;
        for (int t = gz + 4 * y + q; t < L; t += 4 * FS) acc += __bfloat162float(hi[(size_t)t * 8]) + __bfloat162float(lo[(size_t)t * 8]);
        part[y][x] = acc;
        __syncthreads();
        if (y == 0 && x < 8) {
            float s = 0.f;
            for (int k = 0; k < FS; ++k)
#pragma unroll
                for (int qq = 0; qq < 4; ++qq) s += part[k][8 * qq + x];
            out[(size_t)b * C + ck * 8 + x] = s;
        }
    } else {
        const int c = blockIdx.x * 32 + x;
        if (c < C) {
            const float* f = reinterpret_cast<const float*>(src) + (size_t)b * L * C + c;
            for (int t = gz + y; t < L; t += FS) acc += __ldg(f + (size_t)t * C);
        }
        part[y][x] = acc;
        __syncthreads();
        if (y == 0 && c < C) {
            float s = part[0][x];
#pragma unroll
            for (int k = 1; k < FS; ++k) s += part[k][x];
            out[(size_t)b * C + c] = s;
        }
    }
}

}  // namespace cond
}  // namespace wn

using namespace wn;

extern "C" int wn_cond_table(const float* const* d_ptrs, int n_layers, int D, int G, const float* d_h, int n_items, float* d_out,
                             void* stream) {
    WN_REQUIRE(d_ptrs && d_h && d_out, WN_E_BADARG, "wn_cond_table: null pointer");
    WN_REQUIRE(n_layers > 0 && D > 0 && G > 0 && n_items > 0, WN_E_BADARG, "wn_cond_table: bad sizes");
    const int n = n_items * 2 * D;
    const int gx = (n + 255) / 256 > 256 ? 256 : (n + 255) / 256;
    cond::table_kernel<<<dim3(gx, n_layers), 256, 0, (cudaStream_t)stream>>>(d_ptrs, D, G, d_h, n_items, d_out);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_cond_frame_sums(const void* d_dfg, int pair, int B, int L, int C, int gz, float* d_out, void* stream) {
    WN_REQUIRE(d_dfg && d_out, WN_E_BADARG, "wn_cond_frame_sums: null pointer");
    WN_REQUIRE(B > 0 && L > 0 && C > 0 && gz >= 0 && (!pair || C % 8 == 0), WN_E_BADARG, "wn_cond_frame_sums: bad sizes");
    const dim3 block(32, cond::FS);
    cudaStream_t st = (cudaStream_t)stream;
    if (pair) cond::frame_sums_kernel<true><<<dim3(C / 8, B), block, 0, st>>>(d_dfg, L, C, gz, d_out);
    else cond::frame_sums_kernel<false><<<dim3((C + 31) / 32, B), block, 0, st>>>(d_dfg, L, C, gz, d_out);
    WN_CUDA(cudaGetLastError());
    return 0;
}
