// train_misc.cu -- the pieces of a training step around the stack (SURVEY.md section 8, row f1): what WavenetTrainer.train does
// between model(x) and optimizer.step() (reference wavenet_training.py:64-76).
//   wn_ce_fwd_bwd    F.cross_entropy(output, target) (wavenet_training.py:69) and its gradient in ONE pass over the logits:
//                    loss = mean_i (logsumexp(x_i) - x_i[target_i]),  dlogits = (softmax(x_i) - onehot(target_i)) / N.
//                    The eager path reads / writes the (B*output_length, classes) logits five times (log_softmax, nll, their
//                    backward kernels); this reads them once and writes the gradient once.  Deterministic: per-block partial
//                    sums added in fixed order.
//   wn_adam_step     torch.optim.Adam's update (the reference's default optimizer, wavenet_training.py:24) for ALL parameter
//                    tensors in one launch, from a device table of segments.
//   wn_scatter_rows  the start_conv gradient for index input: table[idx[b][t]][:] += dh0[b][t][:]  (what autograd's conv
//                    backward computes on the one-hot input, as a scatter-add of frames).
//   wn_colsum        bias gradients: column sums of a (rows, C) frames tensor, deterministic two-stage reduction.
#include "common.cuh"
#include <cstdint>
#include <cmath>

namespace wn {
namespace misc {

constexpr int CE_WARPS = 8;

// one warp per row; C <= 32 * CE_MAXV
constexpr int CE_MAXV = 32;
__global__ void __launch_bounds__(CE_WARPS * 32)
ce_fwd_bwd_kernel(const float* __restrict__ logits, const long long* __restrict__ target, float* __restrict__ dlogits,
                  float* __restrict__ loss_part, int* __restrict__ err, int N, int C, float inv_n) {
    __shared__ float wsum[CE_WARPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float my_loss = 0.f;
    for (int row = blockIdx.x * CE_WARPS + warp; row < N; row += gridDim.x * CE_WARPS) {
        const float* x = logits + (size_t)row * C;
        float v[CE_MAXV];
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < CE_MAXV; ++i) {
            const int c = lane + 32 * i;
            v[i] = c < C ? x[c] : -INFINITY;
            mx = fmaxf(mx, v[i]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < CE_MAXV; ++i) {
            const int c = lane + 32 * i;
            v[i] = c < C ? expf(v[i] - mx) : 0.f;
            s += v[i];
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        long long tg = target[row];
        if (tg < 0 || tg >= C) { if (lane == 0 && err) atomicExch(err, 1); tg = tg < 0 ? 0 : C - 1; }
        const float inv = 1.f / s;
        float* d = dlogits + (size_t)row * C;
#pragma unroll
        for (int i = 0; i < CE_MAXV; ++i) {
            const int c = lane + 32 * i;
            if (c < C) d[c] = (v[i] * inv - (c == (int)tg ? 1.f : 0.f)) * inv_n;
        }
        // mx - x[tg] first: it is exact for logits of one sign within a factor of two of each other, where logf(s) + mx
        // would round at the ulp of the largest logit (5e-4 at logits near 1e4)
        if (lane == 0) my_loss += logf(s) + (mx - x[tg]);
    }
    if (lane == 0) wsum[warp] = my_loss;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int i = 0; i < CE_WARPS; ++i) t += wsum[i];
        loss_part[blockIdx.x] = t;
    }
}
__global__ void ce_finish_kernel(const float* __restrict__ part, int n, float inv_n, float* __restrict__ loss) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < n; ++i) t += (double)part[i];
        *loss = (float)(t * (double)inv_n);
    }
}

// ---------------------------------------------------------------------------------------------- Adam
struct AdamSeg { float* p; const float* g; float* m; float* v; long long n; };
constexpr int ADAM_CHUNK = 4096;
__global__ void __launch_bounds__(256)
adam_kernel(const AdamSeg* __restrict__ segs, const int2* __restrict__ chunks, int n_chunks, float step_size, float omb1, float b2,
            float omb2, float eps, float wd, float bc2_sqrt) {
    // coefficients come rounded once from double: omb1 = 1 - beta1, omb2 = 1 - beta2, step_size = lr / (1 - beta1^step)
    const int ci = blockIdx.x;
    if (ci >= n_chunks) return;
    const int2 ck = chunks[ci];                         // (segment, first element / ADAM_CHUNK)
    const AdamSeg s = segs[ck.x];
    const long long base = (long long)ck.y * ADAM_CHUNK;
    for (int i = threadIdx.x; i < ADAM_CHUNK; i += 256) {
        const long long e = base + i;
        if (e >= s.n) break;
        float g = s.g[e];
        const float p = s.p[e];
        if (wd != 0.f) g = fmaf(wd, p, g);
        const float m = fmaf(omb1, g - s.m[e], s.m[e]);                     // m + (1 - b1)(g - m) == lerp, as torch does
        const float v = fmaf(omb2, g * g, b2 * s.v[e]);
        s.m[e] = m;
        s.v[e] = v;
        const float denom = sqrtf(v) / bc2_sqrt + eps;
        s.p[e] = p - step_size * (m / denom);
    }
}

// ---------------------------------------------------------------------------------------------- start-conv gradient
// table[(cls)*R + r] += dh[b][t][r] for t in [t_begin, L): one warp per frame, atomics on a (classes x R) table
template <typename IDX>
__global__ void scatter_rows_kernel(const IDX* __restrict__ idx, const float* __restrict__ dh, float* __restrict__ table, int B, int L,
                                    int R, int classes, int t_begin) {
    const int warps = (blockDim.x >> 5) * gridDim.x, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const long long frames = (long long)B * (L - t_begin);
    for (long long f = w; f < frames; f += warps) {
        const int b = (int)(f / (L - t_begin)), t = t_begin + (int)(f % (L - t_begin));
        long long cls = (long long)idx[(size_t)b * L + t];
        cls = cls < 0 ? 0 : (cls >= classes ? classes - 1 : cls);
        const float* src = dh + ((size_t)b * L + t) * R;
        float* dst = table + (size_t)cls * R;
        for (int r = lane; r < R; r += 32) atomicAdd(dst + r, src[r]);
    }
}

__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols) {      // out[c][r] = in[r][c]
    __shared__ float tile[32][33];
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int r = r0 + j, c = c0 + threadIdx.x;
        tile[j][threadIdx.x] = (r < rows && c < cols) ? in[(size_t)r * cols + c] : 0.f;
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += blockDim.y) {
        const int c = c0 + j, r = r0 + threadIdx.x;
        if (r < rows && c < cols) out[(size_t)c * rows + r] = tile[threadIdx.x][j];
    }
}

// column sums of rows [0, rows) of x (rows, ld) -> out[C]; stage 1: per block partials, stage 2: fixed-order sum
constexpr int CS_ROWS = 256;
__global__ void colsum_part_kernel(const float* __restrict__ x, float* __restrict__ part, long long rows, int C, int ld) {
    const long long r0 = (long long)blockIdx.x * CS_ROWS, r1 = r0 + CS_ROWS < rows ? r0 + CS_ROWS : rows;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s = 0.f;
        for (long long r = r0; r < r1; ++r) s += x[(size_t)r * ld + c];
        part[(size_t)blockIdx.x * C + c] = s;
    }
}
__global__ void colsum_finish_kernel(const float* __restrict__ part, float* __restrict__ out, int n_part, int C) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float s = 0.f;
    for (int i = 0; i < n_part; ++i) s += part[(size_t)i * C + c];
    out[c] = s;
}
__global__ void relu_copy_kernel(const float4* __restrict__ x, float4* __restrict__ y, long long n4) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = x[i];
        y[i] = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
    }
}

// x *= *scale (a device scalar: the gradient autograd hands to the loss node), skipped entirely when the scalar is 1
__global__ void scale_by_kernel(float4* __restrict__ x, long long n4, const float* __restrict__ scale) {
    const float s = *scale;
    if (s == 1.f) return;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 v = x[i];
        v.x *= s; v.y *= s; v.z *= s; v.w *= s;
        x[i] = v;
    }
}

}  // namespace misc
}  // namespace wn

using namespace wn;

extern "C" size_t wn_ce_workspace_bytes(void) { return 1184 * sizeof(float); }

extern "C" int wn_ce_fwd_bwd(const float* d_logits, const int64_t* d_target, float* d_dlogits, float* d_loss, float* d_work, int* d_err,
                             int N, int C, void* stream) {
    WN_REQUIRE(d_logits && d_target && d_dlogits && d_loss && d_work, WN_E_BADARG, "wn_ce_fwd_bwd: null pointer");
    WN_REQUIRE(N > 0 && C > 0 && C <= 32 * misc::CE_MAXV, WN_E_UNSUPP, "wn_ce_fwd_bwd: needs 0 < classes <= %d (got %d)", 32 * misc::CE_MAXV, C);
    cudaStream_t st = (cudaStream_t)stream;
    int blocks = (N + misc::CE_WARPS - 1) / misc::CE_WARPS;
    if (blocks > 1184) blocks = 1184;
    const float inv_n = 1.f / (float)N;
    misc::ce_fwd_bwd_kernel<<<blocks, misc::CE_WARPS * 32, 0, st>>>(d_logits, (const long long*)d_target, d_dlogits, d_work, d_err, N, C, inv_n);
    misc::ce_finish_kernel<<<1, 32, 0, st>>>(d_work, blocks, inv_n, d_loss);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_adam_step_f64(const wn_adam_seg* d_segs, const int* d_chunks, int n_chunks, double lr, double beta1, double beta2,
                                double eps, double weight_decay, int step, void* stream) {
    WN_REQUIRE(d_segs && d_chunks && n_chunks > 0 && step >= 1, WN_E_BADARG, "wn_adam_step: bad arguments");
    // torch.optim.Adam forms these in double (Python floats); 1 - beta2 from a float beta2 = 0.999f would be 1.3e-5 off
    const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
    misc::adam_kernel<<<n_chunks, 256, 0, (cudaStream_t)stream>>>((const misc::AdamSeg*)d_segs, (const int2*)d_chunks, n_chunks,
                                                                   (float)(lr / bc1), (float)(1.0 - beta1), (float)beta2,
                                                                   (float)(1.0 - beta2), (float)eps, (float)weight_decay,
                                                                   (float)sqrt(bc2));
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_adam_step(const wn_adam_seg* d_segs, const int* d_chunks, int n_chunks, float lr, float beta1, float beta2, float eps,
                            float weight_decay, int step, void* stream) {
    return wn_adam_step_f64(d_segs, d_chunks, n_chunks, lr, beta1, beta2, eps, weight_decay, step, stream);
}

extern "C" int wn_scatter_rows(const void* d_idx, int idx_is_u8, const float* d_dh, float* d_table, float* d_out_t, int B, int L, int R,
                               int classes, int t_begin, void* stream) {
    WN_REQUIRE(d_idx && d_dh && d_table && B > 0 && L > 0 && R > 0 && classes > 0 && t_begin >= 0 && t_begin <= L, WN_E_BADARG,
               "wn_scatter_rows: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    WN_CUDA(cudaMemsetAsync(d_table, 0, sizeof(float) * (size_t)classes * R, st));
    if (t_begin < L) {
        if (idx_is_u8) misc::scatter_rows_kernel<uint8_t><<<592, 256, 0, st>>>((const uint8_t*)d_idx, d_dh, d_table, B, L, R, classes, t_begin);
        else misc::scatter_rows_kernel<long long><<<592, 256, 0, st>>>((const long long*)d_idx, d_dh, d_table, B, L, R, classes, t_begin);
    }
    if (d_out_t)      // (R, classes): the layout of start_conv.weight
        misc::transpose_kernel<<<dim3((R + 31) / 32, (classes + 31) / 32), dim3(32, 8), 0, st>>>(d_table, d_out_t, classes, R);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" size_t wn_colsum_workspace_bytes(long long rows, int C) { return (size_t)((rows + misc::CS_ROWS - 1) / misc::CS_ROWS) * C * sizeof(float); }

extern "C" int wn_colsum(const float* d_x, float* d_out, float* d_work, long long rows, int C, int ld, void* stream) {
    WN_REQUIRE(d_x && d_out && d_work && rows >= 0 && C > 0 && ld >= C, WN_E_BADARG, "wn_colsum: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    if (rows == 0) { WN_CUDA(cudaMemsetAsync(d_out, 0, sizeof(float) * C, st)); return 0; }
    const int n_part = (int)((rows + misc::CS_ROWS - 1) / misc::CS_ROWS);
    misc::colsum_part_kernel<<<n_part, 256, 0, st>>>(d_x, d_work, rows, C, ld);
    misc::colsum_finish_kernel<<<(C + 255) / 256, 256, 0, st>>>(d_work, d_out, n_part, C);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_relu_copy(const float* d_x, float* d_y, long long n, void* stream) {
    WN_REQUIRE(d_x && d_y && n >= 0 && n % 4 == 0, WN_E_BADARG, "wn_relu_copy: bad arguments (n must be a multiple of 4)");
    if (n == 0) return 0;
    misc::relu_copy_kernel<<<1184, 256, 0, (cudaStream_t)stream>>>((const float4*)d_x, (float4*)d_y, n / 4);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_scale_by(float* d_x, long long n, const float* d_scale, void* stream) {
    WN_REQUIRE(d_x && d_scale && n >= 0 && n % 4 == 0, WN_E_BADARG, "wn_scale_by: bad arguments (n must be a multiple of 4)");
    if (n == 0) return 0;
    misc::scale_by_kernel<<<1184, 256, 0, (cudaStream_t)stream>>>((float4*)d_x, n / 4, d_scale);
    WN_CUDA(cudaGetLastError());
    return 0;
}
