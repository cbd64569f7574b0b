// cond.cu -- global conditioning (WaveNet paper section 2.5): the condition table the forward kernels and the sampler read,
// and the per-sequence frame sums behind the gradient of the conditioning weights.
//
// For one sequence b the condition h_b only adds Vf h_b / Vg h_b to the filter / gate biases, so the block kernels take a
// table [layer][item][2D] of each item's biases bf + Vf h_b | bg + Vg h_b and read it instead of bf / bg: the epilogues do the
// same work as unconditioned ones.  The backward's data gradients do not change (they read the saved tanh / sigmoid).
//
// Local conditioning adds Uf y_f / Ug y_f for a frame-rate series y (repeat upsampling: frame f covers positions
// [f * hop, (f + 1) * hop)), so the table gains a frame axis, [layer][item][frame][2D]; the global table is its n_frames = 1
// case.  The U term is a GEMM per layer (M = items * frames, K = C, N = 2D) on the register-tiled fp32 SGEMM core.
#include "sgemm_core.cuh"
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

// A row m = frame t0 + m of one item of y (C, ld) fp32 (frames contiguous per channel), zero past n_frames / C.
struct FrameLoader {
    const float* y;
    int C, ld, t0, nf;
    static constexpr bool vec = false;
    __device__ __forceinline__ float load1(int m, int kidx) const {
        const int t = t0 + m;
        return (kidx < C && t < nf) ? __ldg(y + (size_t)kidx * ld + t) : 0.f;
    }
    __device__ __forceinline__ float4 load4(int, int) const { return make_float4(0.f, 0.f, 0.f, 0.f); }
};

// out[l][i][f][c] = base[l][i][c] + (sum_k U_l[c][k] * y[i][k][f]).  base is the global table (wn_cond_table: sum_g V h + b),
// computed once per item; without one (no global term) base[l][i][c] = b_l[c].  CTA = TMF frames of one item of one layer
// (blockIdx.x, .y, .z); the U term is mainloop() over the layer's packed U [C][n1p(D)] (wn_pack_gate_weights, k = 1: 128-column
// chunks of 64 filter | 64 gate channels), a sequential fp32 sum over k from 0 -- the same sum table_kernel forms over g.  So
// U = 0 gives exactly the global table (base + 0) and U = V = 0 exactly the biases.
constexpr int TMF = 64;
__global__ void __launch_bounds__(NT) table_frames_kernel(const float* const* __restrict__ ptrs, const float* __restrict__ upk,
                                                          int D, const float* __restrict__ base, int C,
                                                          const float* __restrict__ y, int y_ld, int n_items, int n_frames,
                                                          float* __restrict__ out) {
    using T = Tile<TMF>;
    __shared__ __align__(16) float As[2 * KS * TMF];
    __shared__ __align__(16) float Bs[2 * KS * NC];
    const int l = blockIdx.z, item = blockIdx.y, f0 = blockIdx.x * TMF;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    const int n1p = n1p_of(D);
    const float* bf = ptrs[4 * l + 2];
    const float* bg = ptrs[4 * l + 3];
    const float* bi = base ? base + ((size_t)l * n_items + item) * 2 * D : nullptr;      // this item's global row
    FrameLoader al;
    al.y = y + (size_t)item * C * y_ld; al.C = C; al.ld = y_ld; al.t0 = f0; al.nf = n_frames;
    float* o = out + ((size_t)l * n_items + item) * n_frames * 2 * D;
    for (int ch = 0; ch < n1p / NC; ++ch) {
        float acc[T::MI][8];
#pragma unroll
        for (int i = 0; i < T::MI; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        mainloop<TMF, false>(acc, al, nullptr, upk + (size_t)l * C * n1p, n1p, ch * NC, C, As, Bs);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int c = ch * 64 + tx * 4 + q;
            if (c >= D) continue;
            const float b_f = bi ? __ldg(bi + c) : (bf ? __ldg(bf + c) : 0.f);
            const float b_g = bi ? __ldg(bi + D + c) : (bg ? __ldg(bg + c) : 0.f);
#pragma unroll
            for (int i = 0; i < T::MI; ++i) {
                const int f = f0 + T::row(ty, i);
                if (f >= n_frames) continue;
                o[(size_t)f * 2 * D + c] = acc[i][q] + b_f;
                o[(size_t)f * 2 * D + D + c] = acc[i][4 + q] + b_g;
            }
        }
    }
}

// out[b][f][c] = sum over t in [max(gz, f * hop), min(L, (f + 1) * hop)) of dfg[b][t][c]: frame_sums_kernel's block and
// summation order over each frame's segment (blockIdx.y strides over the frames, blockIdx.z = b).  Empty segments give 0.
template <bool PAIR>
__global__ void __launch_bounds__(32 * FS) segment_sums_kernel(const void* __restrict__ src, int L, int C, int gz, int hop,
                                                               int n_frames, float* __restrict__ out) {
    __shared__ float part[FS][33];
    const int x = threadIdx.x, y = threadIdx.y, b = blockIdx.z;
    for (int f = blockIdx.y; f < n_frames; f += gridDim.y) {
        const long long s0 = (long long)f * hop, s1 = s0 + hop;
        const int lo = (int)(s0 < gz ? gz : (s0 > L ? L : s0)), hi = (int)(s1 > L ? L : s1);
        float* o = out + ((size_t)b * n_frames + f) * C;
        float acc = 0.f;
        if constexpr (PAIR) {
            const int e = x & 7, q = x >> 3, ck = blockIdx.x;
            const __nv_bfloat16* hp = reinterpret_cast<const __nv_bfloat16*>(src) + ((size_t)b * 2 * (C / 8) + ck) * L * 8 + e;
            const __nv_bfloat16* lp = hp + (size_t)(C / 8) * L * 8;
            for (int t = lo + 4 * y + q; t < hi; t += 4 * FS) acc += __bfloat162float(hp[(size_t)t * 8]) + __bfloat162float(lp[(size_t)t * 8]);
            part[y][x] = acc;
            __syncthreads();
            if (y == 0 && x < 8) {
                float s = 0.f;
                for (int k = 0; k < FS; ++k)
#pragma unroll
                    for (int qq = 0; qq < 4; ++qq) s += part[k][8 * qq + x];
                o[ck * 8 + x] = s;
            }
        } else {
            const int c = blockIdx.x * 32 + x;
            if (c < C) {
                const float* p = reinterpret_cast<const float*>(src) + (size_t)b * L * C + c;
                for (int t = lo + y; t < hi; t += FS) acc += __ldg(p + (size_t)t * C);
            }
            part[y][x] = acc;
            __syncthreads();
            if (y == 0 && c < C) {
                float s = part[0][x];
#pragma unroll
                for (int k = 1; k < FS; ++k) s += part[k][x];
                o[c] = s;
            }
        }
        __syncthreads();                                   // part[] is reused by the next frame
    }
}


// ---------------------------------------------------------------------------------------------- audio-rate local conditioning
// With a learned upsampler every position has its own condition features c[t] (C channels), and the gradients of U and c are
// contractions with the pre-activation gradient dfg (the backward's chunked pair tensor [b][plane][N/8][t][8], N = 2D, value
// hi + lo) over the positions t >= gz:
//     dU[n][k]     = sum_b sum_t dfg[b][t][n] * c[b][k][t]    (local_du_kernel: partial sums per frame split, then a fixed-order
//                                                              reduction over the splits)
//     dc[b][k][t] += sum_n U[n][k] * dfg[b][t][n]              (local_dc_kernel: every element has one owner thread)
// Both read dfg where it is, as exact fp32 hi + lo, and accumulate with fp32 FMAs; neither uses atomics, so both are
// deterministic.  c and dc are fp32 (B, C, L), U fp32 [N][C].
constexpr int LT = 64, LS = 32, LMAX_SPLITS = 64;

__device__ __forceinline__ void pair8(const uint4* __restrict__ dfg, size_t hi_idx, size_t plane, float (&v)[8]) {
    const uint4 h = dfg[hi_idx], l = dfg[hi_idx + plane];
    const unsigned hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        v[2 * e] = __uint_as_float(hw[e] << 16) + __uint_as_float(lw[e] << 16);
        v[2 * e + 1] = __uint_as_float(hw[e] & 0xffff0000u) + __uint_as_float(lw[e] & 0xffff0000u);
    }
}

__global__ void __launch_bounds__(256) local_du_kernel(const uint4* __restrict__ dfg, const float* __restrict__ c, int L, int N,
                                                       int C, int gz, int tiles_per_seq, int total_tiles, int tiles_per_split,
                                                       float* __restrict__ part) {
    __shared__ __align__(16) float As[LS][LT + 4];     // [frame][n]
    __shared__ __align__(16) float Bs[LS][LT + 4];     // [frame][k]
    const int n0 = blockIdx.x * LT, k0 = blockIdx.y * LT, split = blockIdx.z;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int chunks = N / 8;
    const size_t plane = (size_t)chunks * L;
    float acc[4][4] = {};
    const int first = split * tiles_per_split, last = min(total_tiles, first + tiles_per_split);
    for (int tile = first; tile < last; ++tile) {
        const int b = tile / tiles_per_seq, t0 = gz + (tile % tiles_per_seq) * LS;
        {
            const int tt = tid % LS, ck = tid / LS, t = t0 + tt, chunk = n0 / 8 + ck;
            float v[8] = {};
            if (t < L && chunk < chunks) pair8(dfg, ((size_t)b * 2 * chunks + chunk) * L + t, plane, v);
#pragma unroll
            for (int e = 0; e < 8; ++e) As[tt][ck * 8 + e] = v[e];
        }
        for (int i = tid; i < LT * LS; i += 256) {
            const int tt = i % LS, kk = i / LS, t = t0 + tt, k = k0 + kk;
            Bs[tt][kk] = (t < L && k < C) ? c[((size_t)b * C + k) * L + t] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int tt = 0; tt < LS; ++tt) {
            const float4 a = *reinterpret_cast<const float4*>(&As[tt][ty * 4]);
            const float4 w = *reinterpret_cast<const float4*>(&Bs[tt][tx * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + ty * 4 + i, k = k0 + tx * 4 + j;
            if (n < N && k < C) part[((size_t)split * N + n) * C + k] = acc[i][j];
        }
}

__global__ void local_du_reduce_kernel(const float* __restrict__ part, int splits, int NC, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= NC) return;
    float s = 0.f;
    for (int j = 0; j < splits; ++j) s += part[(size_t)j * NC + i];
    out[i] = s;
}

__global__ void __launch_bounds__(256) local_dc_kernel(const uint4* __restrict__ dfg, const float* __restrict__ u, int L, int N,
                                                       int C, int gz, float* __restrict__ dc) {
    __shared__ __align__(16) float As[LS][LT + 4];     // [n][frame]
    __shared__ __align__(16) float Bs[LS][LT + 4];     // [n][k]
    const int t0 = gz + blockIdx.x * LT, k0 = blockIdx.y * LT, b = blockIdx.z;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int chunks = N / 8;
    const size_t plane = (size_t)chunks * L;
    float acc[4][4] = {};                              // [k][frame]
    for (int nb = 0; nb < N; nb += LS) {
        {
            const int tt = tid % LT, ck = tid / LT, t = t0 + tt, chunk = nb / 8 + ck;
            float v[8] = {};
            if (t < L) pair8(dfg, ((size_t)b * 2 * chunks + chunk) * L + t, plane, v);
#pragma unroll
            for (int e = 0; e < 8; ++e) As[ck * 8 + e][tt] = v[e];
        }
        for (int i = tid; i < LS * LT; i += 256) {
            const int kk = i % LT, nn = i / LT, k = k0 + kk;
            Bs[nn][kk] = k < C ? u[(size_t)(nb + nn) * C + k] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int nn = 0; nn < LS; ++nn) {
            const float4 a = *reinterpret_cast<const float4*>(&As[nn][tx * 4]);
            const float4 w = *reinterpret_cast<const float4*>(&Bs[nn][ty * 4]);
            const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(wv[i], av[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int k = k0 + ty * 4 + i;
        if (k >= C) continue;
        float* row = dc + ((size_t)b * C + k) * L;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int t = t0 + tx * 4 + j;
            if (t < L) row[t] += acc[i][j];
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

extern "C" int wn_cond_table_frames(const float* const* d_ptrs, const float* d_u_packed, int n_layers, int D,
                                    const float* d_base, int C, const float* d_y, int y_ld, int n_items, int n_frames, float* d_out,
                                    void* stream) {
    WN_REQUIRE(d_ptrs && d_u_packed && d_y && d_out, WN_E_BADARG, "wn_cond_table_frames: null pointer");
    // U is read as float4 (its rows are wn_n1p(D) floats, a multiple of 4); y, base and out are read / written per float
    WN_REQUIRE((uintptr_t)d_u_packed % 16 == 0 && ((uintptr_t)d_y | (uintptr_t)d_base | (uintptr_t)d_out) % 4 == 0, WN_E_BADARG,
               "wn_cond_table_frames: U must be 16-byte aligned, y, the base table and the output 4-byte aligned");
    WN_REQUIRE(n_layers > 0 && D > 0 && C > 0 && n_items > 0 && n_frames > 0 && y_ld >= n_frames && n_items <= 65535 &&
                   n_layers <= 65535, WN_E_BADARG, "wn_cond_table_frames: bad sizes");
    const dim3 grid((unsigned)ceil_div(n_frames, cond::TMF), (unsigned)n_items, (unsigned)n_layers);
    cond::table_frames_kernel<<<grid, NT, 0, (cudaStream_t)stream>>>(d_ptrs, d_u_packed, D, d_base, C, d_y, y_ld, n_items,
                                                                    n_frames, d_out);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_cond_segment_sums(const void* d_dfg, int pair, int B, int L, int C, int gz, int hop, int n_frames, float* d_out,
                                    void* stream) {
    WN_REQUIRE(d_dfg && d_out, WN_E_BADARG, "wn_cond_segment_sums: null pointer");
    WN_REQUIRE(B > 0 && B <= 65535 && L > 0 && C > 0 && gz >= 0 && hop >= 1 && n_frames > 0 && (!pair || C % 8 == 0), WN_E_BADARG,
               "wn_cond_segment_sums: bad sizes");
    const dim3 block(32, cond::FS);
    const unsigned gy = (unsigned)(n_frames < 65535 ? n_frames : 65535);
    cudaStream_t st = (cudaStream_t)stream;
    if (pair) cond::segment_sums_kernel<true><<<dim3(C / 8, gy, B), block, 0, st>>>(d_dfg, L, C, gz, hop, n_frames, d_out);
    else cond::segment_sums_kernel<false><<<dim3((C + 31) / 32, gy, B), block, 0, st>>>(d_dfg, L, C, gz, hop, n_frames, d_out);
    WN_CUDA(cudaGetLastError());
    return 0;
}

// frame splits of the dU partial sums: a function of the shape only, so the reduction order (and the result) is fixed
static int local_splits(int B, int L, int N, int C, int gz, int* tiles_per_seq, int* total, int* per_split) {
    *tiles_per_seq = ceil_div(L - gz, cond::LS);
    *total = B * *tiles_per_seq;
    const int blocks_xy = ceil_div(N, cond::LT) * ceil_div(C, cond::LT);
    int s = ceil_div(512, blocks_xy);
    s = s > cond::LMAX_SPLITS ? cond::LMAX_SPLITS : s;
    s = s > *total ? *total : s;
    *per_split = ceil_div(*total, s);
    return ceil_div(*total, *per_split);
}

extern "C" size_t wn_local_weight_grad_workspace_bytes(int N, int C) {
    return N > 0 && C > 0 ? (size_t)cond::LMAX_SPLITS * N * C * sizeof(float) : 0;
}

extern "C" int wn_local_weight_grad(const void* d_dfg, int B, int L, int N, int gz, const float* d_c, int C, float* d_work,
                                    float* d_du, void* stream) {
    WN_REQUIRE(d_dfg && d_c && d_work && d_du, WN_E_BADARG, "wn_local_weight_grad: null pointer");
    WN_REQUIRE(B > 0 && L > 0 && N > 0 && N % 8 == 0 && C > 0 && gz >= 0 && (uintptr_t)d_dfg % 16 == 0, WN_E_BADARG,
               "wn_local_weight_grad: bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    if (gz >= L) {
        WN_CUDA(cudaMemsetAsync(d_du, 0, sizeof(float) * (size_t)N * C, st));
        return 0;
    }
    int tps, total, per;
    const int splits = local_splits(B, L, N, C, gz, &tps, &total, &per);
    const dim3 grid((unsigned)ceil_div(N, cond::LT), (unsigned)ceil_div(C, cond::LT), (unsigned)splits);
    cond::local_du_kernel<<<grid, 256, 0, st>>>((const uint4*)d_dfg, d_c, L, N, C, gz, tps, total, per, d_work);
    WN_CUDA(cudaGetLastError());
    cond::local_du_reduce_kernel<<<ceil_div(N * C, 256), 256, 0, st>>>(d_work, splits, N * C, d_du);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_local_data_grad_add(const void* d_dfg, int B, int L, int N, int gz, const float* d_u, int C, float* d_dc,
                                      void* stream) {
    WN_REQUIRE(d_dfg && d_u && d_dc, WN_E_BADARG, "wn_local_data_grad_add: null pointer");
    WN_REQUIRE(B > 0 && B <= 65535 && L > 0 && N > 0 && N % cond::LS == 0 && C > 0 && gz >= 0 && (uintptr_t)d_dfg % 16 == 0,
               WN_E_BADARG, "wn_local_data_grad_add: bad sizes");
    if (gz >= L) return 0;
    const dim3 grid((unsigned)ceil_div(L - gz, cond::LT), (unsigned)ceil_div(C, cond::LT), (unsigned)B);
    cond::local_dc_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((const uint4*)d_dfg, d_u, L, N, C, gz, d_dc);
    WN_CUDA(cudaGetLastError());
    return 0;
}
