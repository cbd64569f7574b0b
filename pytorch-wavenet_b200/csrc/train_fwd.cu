// train_fwd.cu -- training-time forward of the dilated causal convolution stack, exact-fp32 (FFMA) kernels.
//
// Replaces (reference file:line): start_conv wavenet_model.py:127; the residual block loop body :142-165
// together with dilate() wavenet_modules.py:10-39 and the constant pad :80-127; the head :167-169 and
// forward()'s slice/transpose :191-196.
//
// Data layout ("frames"): activations (B, L, C) fp32 with C contiguous, absolute time axis, zero history left
// of a layer's valid start.  One CTA owns TM consecutive frames of one sequence and ALL channels, so the gated
// activation z never leaves shared memory between the dilated conv and the two 1x1 convs:
//
//   phase 1   FG[TM x 2D] = A[TM x kR] * Wfg_t        A row t = [h(t-(k-1)d) | ... | h(t)], zero left of in_start
//             z = tanh(F + bf) * sigmoid(G + bg)  ->  Zs[D][TM] (shared memory, K-outer for phase 2)
//   phase 2   OS[TM x (R+S)] = Zs^T * Wrs_t           cols < R: h_out = . + br + h(t);  cols >= R: skip (+)= . + bs
//
// Both phases are register-tiled SGEMMs (16x16 threads, (TM/16) x 8 accumulators per thread, K slabs of 16,
// one __syncthreads per slab with register prefetch of the next slab).  The head kernel is the same two-phase
// machine with relu epilogues.  Weights come pre-packed K-outer (see wn_pack_* in wavenet_b200.h).
#include "sgemm_core.cuh"

namespace wn {

// ------------------------------------------------------------------------------------------------ packing
__global__ void pack_gate_kernel(const float* __restrict__ wf, const float* __restrict__ wg,
                                 const float* __restrict__ bf, const float* __restrict__ bg,
                                 int R, int D, int k, int N1p, float* __restrict__ wfg_t, float* __restrict__ bfg) {
    const long long total = (long long)k * R * N1p;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int row = (int)(i / N1p), col = (int)(i % N1p);
        const int chunk = col >> 7, within = col & 127, ch = chunk * 64 + (within & 63);
        const int j = row / R, r = row % R;
        float v = 0.f;
        if (ch < D) v = (within >= 64 ? wg : wf)[((size_t)ch * R + r) * k + j];
        wfg_t[i] = v;
        if (row == 0) {
            const float* b = within >= 64 ? bg : bf;
            bfg[col] = (ch < D && b != nullptr) ? b[ch] : 0.f;
        }
    }
}

// generic (N,K) row-major -> [K][Np] with zero padding; used for residual|skip (two sources) and the 1x1 head convs
__global__ void pack_rows_kernel(const float* __restrict__ w0, const float* __restrict__ b0, int N0,
                                 const float* __restrict__ w1, const float* __restrict__ b1, int N1,
                                 int K, int Np, float* __restrict__ w_t, float* __restrict__ b_p) {
    const long long total = (long long)K * Np;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int kk = (int)(i / Np), n = (int)(i % Np);
        float v = 0.f, bv = 0.f;
        if (n < N0) {
            v = w0[(size_t)n * K + kk];
            bv = b0 ? b0[n] : 0.f;
        } else if (n < N0 + N1) {
            v = w1[(size_t)(n - N0) * K + kk];
            bv = b1 ? b1[n - N0] : 0.f;
        }
        w_t[i] = v;
        if (kk == 0) b_p[n] = bv;
    }
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ------------------------------------------------------------------------------------------------ block kernel
struct BlockParams {
    const float* h_in; float* h_out; float* skip;
    const float* wfg_t; const float* bfg; const float* wrs_t; const float* brs;
    int B, L, R, D, S, ktaps, dil;
    int in_start, out_start, skip_start, skip_init;
    int N1p, N2p, Kz;       // Kz = z channels incl. padding = N1p/2
    float* fg_save;         // optional (B,L,2D): tanh / sigmoid outputs for the backward
    const float* cond;      // optional (B,2D): per-sequence filter / gate biases [bf + Vf h | bg + Vg h], used instead of bfg
    int cond_frames, cond_hop;   // cond_hop > 0: cond is (B, cond_frames, 2D), frame t / cond_hop holds frame t's biases
};

template <int TM>
__global__ void __launch_bounds__(NT, 1) block_fwd_kernel(const BlockParams p) {
    using T = Tile<TM>;
    constexpr int MI = T::MI;
    extern __shared__ __align__(16) float smem[];
    float* As = smem;                        // [2][KS][TM]
    float* Bs = As + 2 * KS * TM;            // [2][KS][NC]
    float* Zs = Bs + 2 * KS * NC;            // [Kz][TM+ZPAD]

    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int b = blockIdx.y;
    const int t0 = p.out_start + blockIdx.x * TM;
    const int Tsk = p.L - p.skip_start;

    TapLoader al;
    al.h = p.h_in + (size_t)b * p.L * p.R;
    al.R = p.R; al.ktaps = p.ktaps; al.dil = p.dil; al.t0 = t0; al.L = p.L; al.in_start = p.in_start;
    al.K = p.ktaps * p.R;
    al.vec = (p.R % KS == 0);

    // ---------------- phase 1: dilated conv + gate -> Zs
    const int n1_chunks = p.N1p / NC;
    for (int ch = 0; ch < n1_chunks; ++ch) {
        float acc[MI][8];
#pragma unroll
        for (int i = 0; i < MI; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        mainloop<TM, false>(acc, al, nullptr, p.wfg_t, p.N1p, ch * NC, al.K, As, Bs);
        const float4 bf4 = __ldg(reinterpret_cast<const float4*>(p.bfg + ch * NC + tx * 4));
        const float4 bg4 = __ldg(reinterpret_cast<const float4*>(p.bfg + ch * NC + 64 + tx * 4));
        float bfv[4] = {bf4.x, bf4.y, bf4.z, bf4.w}, bgv[4] = {bg4.x, bg4.y, bg4.z, bg4.w};
        if (p.cond != nullptr && p.cond_hop > 0) {                 // locally conditioned: every frame's own biases
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                float* zrow = Zs + (size_t)(ch * 64 + tx * 4 + q) * (TM + ZPAD);
                const int c = ch * 64 + tx * 4 + q;
#pragma unroll
                for (int i = 0; i < MI; ++i) {
                    const int t = t0 + T::row(ty, i), tc = t < p.L ? t : p.L - 1;     // rows past L read the last frame
                    const float* cb = p.cond + ((size_t)b * p.cond_frames + tc / p.cond_hop) * 2 * p.D;
                    const float f = tanhf(acc[i][q] + (c < p.D ? __ldg(cb + c) : 0.f));
                    const float g = sigmoidf_(acc[i][4 + q] + (c < p.D ? __ldg(cb + p.D + c) : 0.f));
                    zrow[T::row(ty, i)] = f * g;
                    if (p.fg_save != nullptr && t < p.L && c < p.D) {
                        float* dst = p.fg_save + ((size_t)b * p.L + t) * (2 * p.D);
                        dst[c] = f;
                        dst[p.D + c] = g;
                    }
                }
            }
            continue;
        }
        if (p.cond != nullptr) {                                   // conditioned: this sequence's own biases
            const float* cb = p.cond + (size_t)b * 2 * p.D;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int c = ch * 64 + tx * 4 + q;
                bfv[q] = c < p.D ? __ldg(cb + c) : 0.f;
                bgv[q] = c < p.D ? __ldg(cb + p.D + c) : 0.f;
            }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            float* zrow = Zs + (size_t)(ch * 64 + tx * 4 + q) * (TM + ZPAD);
            const int c = ch * 64 + tx * 4 + q;
#pragma unroll
            for (int i = 0; i < MI; ++i) {
                const float f = tanhf(acc[i][q] + bfv[q]), g = sigmoidf_(acc[i][4 + q] + bgv[q]);
                zrow[T::row(ty, i)] = f * g;
                if (p.fg_save != nullptr) {
                    const int t = t0 + T::row(ty, i);
                    if (t < p.L && c < p.D) {
                        float* dst = p.fg_save + ((size_t)b * p.L + t) * (2 * p.D);
                        dst[c] = f;
                        dst[p.D + c] = g;
                    }
                }
            }
        }
    }
    __syncthreads();

    // ---------------- phase 2: residual 1x1 (+ identity) and skip 1x1 (+ running skip)
    const float* hin_b = p.h_in + (size_t)b * p.L * p.R;
    float* hout_b = p.h_out + (size_t)b * p.L * p.R;
    float* skip_b = p.skip + (size_t)b * Tsk * p.S;
    const bool vecR = (p.R % 4 == 0), vecS = (p.S % 4 == 0) && vecR;
    const int n2_chunks = p.N2p / NC;
    const bool tile_has_skip = (t0 + TM > p.skip_start);
    for (int ch = 0; ch < n2_chunks; ++ch) {
        if (ch * NC >= p.R && !tile_has_skip) break;          // skip columns, tile left of the surviving skip range
        float acc[MI][8];
#pragma unroll
        for (int i = 0; i < MI; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        mainloop<TM, true>(acc, al, Zs, p.wrs_t, p.N2p, ch * NC, p.D, As, Bs);
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            const int n0 = ch * NC + g * 64 + tx * 4;
            if (n0 >= p.R + p.S) continue;
            const float4 bb = __ldg(reinterpret_cast<const float4*>(p.brs + n0));
            const float bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
            for (int i = 0; i < MI; ++i) {
                const int t = t0 + T::row(ty, i);
                if (t >= p.L) continue;
                float o[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) o[q] = acc[i][g * 4 + q] + bv[q];
                if (vecR && n0 + 3 < p.R) {                                   // 4 residual outputs
                    float* dst = hout_b + (size_t)t * p.R + n0;
                    if (t >= p.in_start) {
                        const float4 x = __ldg(reinterpret_cast<const float4*>(hin_b + (size_t)t * p.R + n0));
                        o[0] += x.x; o[1] += x.y; o[2] += x.z; o[3] += x.w;
                    }
                    *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
                } else if (vecS && n0 >= p.R && n0 + 3 < p.R + p.S) {          // 4 skip outputs
                    if (t >= p.skip_start) {
                        float* dst = skip_b + (size_t)(t - p.skip_start) * p.S + (n0 - p.R);
                        if (!p.skip_init) {
                            const float4 x = *reinterpret_cast<const float4*>(dst);
                            o[0] += x.x; o[1] += x.y; o[2] += x.z; o[3] += x.w;
                        }
                        *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
                    }
                } else {                                                       // ragged channel counts
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int n = n0 + q;
                        if (n < p.R) {
                            float v = o[q];
                            if (t >= p.in_start) v += __ldg(hin_b + (size_t)t * p.R + n);
                            hout_b[(size_t)t * p.R + n] = v;
                        } else if (n < p.R + p.S && t >= p.skip_start) {
                            float* dst = skip_b + (size_t)(t - p.skip_start) * p.S + (n - p.R);
                            *dst = p.skip_init ? o[q] : (o[q] + *dst);
                        }
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ head kernel
struct HeadParams {
    const float* skip; float* logits;
    const float* w1_t; const float* b1; const float* w2_t; const float* b2;
    int B, L, S, E, classes, skip_start, out_len;
    int N1p, N2p, Kz;       // N1p = n2p(E) = Kz; N2p = n2p(classes)
};

template <int TM>
__global__ void __launch_bounds__(NT, 1) head_fwd_kernel(const HeadParams p) {
    using T = Tile<TM>;
    constexpr int MI = T::MI;
    extern __shared__ __align__(16) float smem[];
    float* As = smem;
    float* Bs = As + 2 * KS * TM;
    float* Zs = Bs + 2 * KS * NC;

    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int b = blockIdx.y;
    const int t_first = p.L - p.out_len;
    const int t0 = t_first + blockIdx.x * TM;
    const int Tsk = p.L - p.skip_start;

    ReluRowLoader al;
    al.s = p.skip + (size_t)b * Tsk * p.S;
    al.S = p.S; al.t0 = t0; al.L = p.L; al.skip_start = p.skip_start;
    al.vec = (p.S % KS == 0);

    for (int ch = 0; ch < p.N1p / NC; ++ch) {
        float acc[MI][8];
#pragma unroll
        for (int i = 0; i < MI; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        mainloop<TM, false>(acc, al, nullptr, p.w1_t, p.N1p, ch * NC, p.S, As, Bs);
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            const float4 bb = __ldg(reinterpret_cast<const float4*>(p.b1 + ch * NC + g * 64 + tx * 4));
            const float bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                float* zrow = Zs + (size_t)(ch * NC + g * 64 + tx * 4 + q) * (TM + ZPAD);
#pragma unroll
                for (int i = 0; i < MI; ++i) zrow[T::row(ty, i)] = fmaxf(acc[i][g * 4 + q] + bv[q], 0.f);
            }
        }
    }
    __syncthreads();

    float* out_b = p.logits + (size_t)b * p.out_len * p.classes;
    const bool vecC = (p.classes % 4 == 0);
    for (int ch = 0; ch < p.N2p / NC; ++ch) {
        float acc[MI][8];
#pragma unroll
        for (int i = 0; i < MI; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        mainloop<TM, true>(acc, al, Zs, p.w2_t, p.N2p, ch * NC, p.E, As, Bs);
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            const int n0 = ch * NC + g * 64 + tx * 4;
            if (n0 >= p.classes) continue;
            const float4 bb = __ldg(reinterpret_cast<const float4*>(p.b2 + n0));
            const float bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
            for (int i = 0; i < MI; ++i) {
                const int t = t0 + T::row(ty, i);
                if (t >= p.L) continue;
                float* dst = out_b + (size_t)(t - t_first) * p.classes + n0;
                if (vecC) {
                    *reinterpret_cast<float4*>(dst) = make_float4(acc[i][g * 4 + 0] + bv[0], acc[i][g * 4 + 1] + bv[1],
                                                                  acc[i][g * 4 + 2] + bv[2], acc[i][g * 4 + 3] + bv[3]);
                } else {
#pragma unroll
                    for (int q = 0; q < 4; ++q)
                        if (n0 + q < p.classes) dst[q] = acc[i][g * 4 + q] + bv[q];
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ start conv
struct StartParams {
    const float* x; const float* w_t; const float* b_p; float* h;
    int B, classes, L, R, Np;
};

template <int TM>
__global__ void __launch_bounds__(NT, 2) start_dense_kernel(const StartParams p) {
    using T = Tile<TM>;
    constexpr int MI = T::MI;
    extern __shared__ __align__(16) float smem[];
    float* As = smem;
    float* Bs = As + 2 * KS * TM;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int b = blockIdx.y, t0 = blockIdx.x * TM;
    ColumnLoader al;
    al.x = p.x + (size_t)b * p.classes * p.L;
    al.classes = p.classes; al.t0 = t0; al.L = p.L;
    float* h_b = p.h + (size_t)b * p.L * p.R;
    for (int ch = 0; ch < p.Np / NC; ++ch) {
        float acc[MI][8];
#pragma unroll
        for (int i = 0; i < MI; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        mainloop<TM, false>(acc, al, nullptr, p.w_t, p.Np, ch * NC, p.classes, As, Bs);
#pragma unroll
        for (int g = 0; g < 2; ++g) {
            const int n0 = ch * NC + g * 64 + tx * 4;
#pragma unroll
            for (int i = 0; i < MI; ++i) {
                const int t = t0 + T::row(ty, i);
                if (t >= p.L) continue;
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (n0 + q < p.R) h_b[(size_t)t * p.R + n0 + q] = acc[i][g * 4 + q] + __ldg(p.b_p + n0 + q);
            }
        }
    }
}

// index form: h[b,t,:] = w_t[idx[b,t]][:] + bias  -- a row gather of the packed (classes, Np) table
template <typename IdxT>
__global__ void start_index_kernel(const IdxT* __restrict__ idx, const float* __restrict__ w_t,
                                   const float* __restrict__ b_p, float* __restrict__ h,
                                   long long frames, int classes, int R, int Np) {
    const long long total = frames * R;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long f = i / R;
        const int r = (int)(i - f * R);
        long long c = (long long)idx[f];
        c = c < 0 ? 0 : (c >= classes ? classes - 1 : c);
        h[i] = __ldg(w_t + (size_t)c * Np + r) + __ldg(b_p + r);
    }
}

// ------------------------------------------------------------------------------------------------ launch helpers
static size_t two_phase_smem(int TM, int Kz) {
    return sizeof(float) * ((size_t)2 * KS * TM + (size_t)2 * KS * NC + (size_t)Kz * (TM + ZPAD));
}
static int pick_tm(int Kz, int smem_limit) {
    const int cands[4] = {128, 64, 32, 16};
    for (int i = 0; i < 4; ++i)
        if (two_phase_smem(cands[i], Kz) <= (size_t)smem_limit) return cands[i];
    return 0;
}
static int smem_limit_bytes() {
    int dev = 0, v = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) return 0;
    return v;
}

template <int TM>
static int launch_block(const BlockParams& p, size_t smem, cudaStream_t st) {
    WN_CUDA(cudaFuncSetAttribute(block_fwd_kernel<TM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int tiles = ceil_div(p.L - p.out_start, TM);
    block_fwd_kernel<TM><<<dim3(tiles, p.B), NT, smem, st>>>(p);
    WN_CUDA(cudaGetLastError());
    return 0;
}
template <int TM>
static int launch_head(const HeadParams& p, size_t smem, cudaStream_t st) {
    WN_CUDA(cudaFuncSetAttribute(head_fwd_kernel<TM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int tiles = ceil_div(p.out_len, TM);
    head_fwd_kernel<TM><<<dim3(tiles, p.B), NT, smem, st>>>(p);
    WN_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace wn

using namespace wn;

// ================================================================================================ C ABI
extern "C" int wn_n1p(int D) { return n1p_of(D); }
extern "C" int wn_n2p(int N) { return n2p_of(N); }

extern "C" int wn_pack_gate_weights(const float* d_wf, const float* d_wg, const float* d_bf, const float* d_bg,
                                    int R, int D, int k, float* d_wfg_t, float* d_bfg, void* stream) {
    WN_REQUIRE(d_wf && d_wg && d_wfg_t && d_bfg, WN_E_BADARG, "wn_pack_gate_weights: null pointer");
    WN_REQUIRE(R > 0 && D > 0 && k >= 1, WN_E_BADARG, "wn_pack_gate_weights: bad shape R=%d D=%d k=%d", R, D, k);
    const int N1p = n1p_of(D);
    const long long total = (long long)k * R * N1p;
    const int grid = (int)((total + 255) / 256 > 4096 ? 4096 : (total + 255) / 256);
    pack_gate_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(d_wf, d_wg, d_bf, d_bg, R, D, k, N1p, d_wfg_t, d_bfg);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_pack_res_skip_weights(const float* d_wr, const float* d_ws, const float* d_br, const float* d_bs,
                                        int R, int D, int S, float* d_wrs_t, float* d_brs, void* stream) {
    WN_REQUIRE(d_wr && d_ws && d_wrs_t && d_brs, WN_E_BADARG, "wn_pack_res_skip_weights: null pointer");
    WN_REQUIRE(R > 0 && D > 0 && S > 0, WN_E_BADARG, "wn_pack_res_skip_weights: bad shape");
    const int Np = n2p_of(R + S);
    const long long total = (long long)D * Np;
    const int grid = (int)((total + 255) / 256 > 4096 ? 4096 : (total + 255) / 256);
    pack_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(d_wr, d_br, R, d_ws, d_bs, S, D, Np, d_wrs_t, d_brs);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_pack_1x1_weights(const float* d_w, const float* d_b, int N, int K, float* d_w_t, float* d_b_p,
                                   void* stream) {
    WN_REQUIRE(d_w && d_w_t && d_b_p, WN_E_BADARG, "wn_pack_1x1_weights: null pointer");
    WN_REQUIRE(N > 0 && K > 0, WN_E_BADARG, "wn_pack_1x1_weights: bad shape");
    const int Np = n2p_of(N);
    const long long total = (long long)K * Np;
    const int grid = (int)((total + 255) / 256 > 4096 ? 4096 : (total + 255) / 256);
    pack_rows_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(d_w, d_b, N, nullptr, nullptr, 0, K, Np, d_w_t, d_b_p);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_start_fwd_dense(const float* d_x, const float* d_w_t, const float* d_b_p, float* d_h,
                                  int B, int classes, int L, int R, void* stream) {
    WN_REQUIRE(d_x && d_w_t && d_b_p && d_h, WN_E_BADARG, "wn_start_fwd_dense: null pointer");
    WN_REQUIRE(B > 0 && classes > 0 && L > 0 && R > 0, WN_E_BADARG, "wn_start_fwd_dense: bad shape");
    StartParams p{d_x, d_w_t, d_b_p, d_h, B, classes, L, R, n2p_of(R)};
    constexpr int TM = 64;
    const size_t smem = sizeof(float) * (2 * KS * TM + 2 * KS * NC);
    start_dense_kernel<TM><<<dim3(ceil_div(L, TM), B), NT, smem, (cudaStream_t)stream>>>(p);
    WN_CUDA(cudaGetLastError());
    return 0;
}

template <typename IdxT>
static int start_index_impl(const IdxT* d_idx, const float* d_w_t, const float* d_b_p, float* d_h, int B, int classes,
                            int L, int R, void* stream) {
    WN_REQUIRE(d_idx && d_w_t && d_b_p && d_h, WN_E_BADARG, "wn_start_fwd_index: null pointer");
    WN_REQUIRE(B > 0 && classes > 0 && L > 0 && R > 0, WN_E_BADARG, "wn_start_fwd_index: bad shape");
    const long long frames = (long long)B * L, total = frames * R;
    const int grid = (int)((total + 255) / 256 > 148 * 16 ? 148 * 16 : (total + 255) / 256);
    start_index_kernel<IdxT><<<grid, 256, 0, (cudaStream_t)stream>>>(d_idx, d_w_t, d_b_p, d_h, frames, classes, R,
                                                                    n2p_of(R));
    WN_CUDA(cudaGetLastError());
    return 0;
}
extern "C" int wn_start_fwd_index_u8(const uint8_t* d_idx, const float* d_w_t, const float* d_b_p, float* d_h, int B,
                                     int classes, int L, int R, void* stream) {
    return start_index_impl<uint8_t>(d_idx, d_w_t, d_b_p, d_h, B, classes, L, R, stream);
}
extern "C" int wn_start_fwd_index_i64(const int64_t* d_idx, const float* d_w_t, const float* d_b_p, float* d_h, int B,
                                      int classes, int L, int R, void* stream) {
    return start_index_impl<int64_t>(d_idx, d_w_t, d_b_p, d_h, B, classes, L, R, stream);
}

extern "C" int wn_block_fwd(const wn_block_args* a, void* stream) { return wn_block_fwd_cond(a, nullptr, stream); }

static int block_fwd_impl(const wn_block_args* a, const float* d_cond, int n_frames, int hop, void* stream);

extern "C" int wn_block_fwd_cond(const wn_block_args* a, const float* d_cond, void* stream) {
    return block_fwd_impl(a, d_cond, 0, 0, stream);
}

extern "C" int wn_block_fwd_cond_frames(const wn_block_args* a, const float* d_cond, int n_frames, int hop, void* stream) {
    WN_REQUIRE(a && d_cond, WN_E_BADARG, "wn_block_fwd_cond_frames: null pointer");
    WN_REQUIRE(hop >= 1 && a->L > 0 && n_frames >= ceil_div(a->L, hop), WN_E_BADARG,
               "wn_block_fwd_cond_frames: %d frames of hop %d do not cover %d positions", n_frames, hop, a->L);
    WN_REQUIRE((uintptr_t)d_cond % 4 == 0, WN_E_BADARG, "wn_block_fwd_cond_frames: the condition table must be 4-byte aligned");
    return block_fwd_impl(a, d_cond, n_frames, hop, stream);
}

static int block_fwd_impl(const wn_block_args* a, const float* d_cond, int n_frames, int hop, void* stream) {
    WN_REQUIRE(a, WN_E_BADARG, "wn_block_fwd: null args");
    WN_REQUIRE(a->d_h_in && a->d_h_out && a->d_skip && a->d_wfg_t && a->d_bfg && a->d_wrs_t && a->d_brs, WN_E_BADARG,
               "wn_block_fwd: null pointer");
    WN_REQUIRE(a->B > 0 && a->L > 0 && a->R > 0 && a->D > 0 && a->S > 0 && a->k >= 1 && a->dilation >= 1, WN_E_BADARG,
               "wn_block_fwd: bad shape");
    WN_REQUIRE(a->in_start >= 0 && a->out_start >= a->in_start && a->out_start < a->L && a->skip_start >= a->out_start &&
                   a->skip_start < a->L,
               WN_E_BADARG, "wn_block_fwd: bad frame ranges in=%d out=%d skip=%d L=%d", a->in_start, a->out_start,
               a->skip_start, a->L);
    WN_REQUIRE(a->d_h_in != a->d_h_out, WN_E_BADARG, "wn_block_fwd: in-place update is not supported (taps read h_in)");
    WN_REQUIRE(a->mode == 0, WN_E_UNSUPP, "wn_block_fwd: mode %d not available in this build", a->mode);
    BlockParams p;
    p.h_in = a->d_h_in; p.h_out = a->d_h_out; p.skip = a->d_skip;
    p.wfg_t = a->d_wfg_t; p.bfg = a->d_bfg; p.wrs_t = a->d_wrs_t; p.brs = a->d_brs;
    p.B = a->B; p.L = a->L; p.R = a->R; p.D = a->D; p.S = a->S; p.ktaps = a->k; p.dil = a->dilation;
    p.in_start = a->in_start; p.out_start = a->out_start; p.skip_start = a->skip_start; p.skip_init = a->skip_init;
    p.N1p = n1p_of(a->D); p.N2p = n2p_of(a->R + a->S); p.Kz = p.N1p / 2;
    p.fg_save = a->d_fg_save;
    p.cond = d_cond;
    p.cond_frames = n_frames; p.cond_hop = hop;
    const int tm = pick_tm(p.Kz, smem_limit_bytes());
    WN_REQUIRE(tm > 0, WN_E_UNSUPP, "wn_block_fwd: dilation_channels=%d does not fit shared memory", a->D);
    const size_t smem = two_phase_smem(tm, p.Kz);
    cudaStream_t st = (cudaStream_t)stream;
    switch (tm) {
        case 128: return launch_block<128>(p, smem, st);
        case 64: return launch_block<64>(p, smem, st);
        case 32: return launch_block<32>(p, smem, st);
        default: return launch_block<16>(p, smem, st);
    }
}

extern "C" int wn_head_fwd(const wn_head_args* a, void* stream) {
    WN_REQUIRE(a, WN_E_BADARG, "wn_head_fwd: null args");
    WN_REQUIRE(a->d_skip && a->d_logits && a->d_w1_t && a->d_b1 && a->d_w2_t && a->d_b2, WN_E_BADARG,
               "wn_head_fwd: null pointer");
    WN_REQUIRE(a->B > 0 && a->L > 0 && a->S > 0 && a->E > 0 && a->classes > 0, WN_E_BADARG, "wn_head_fwd: bad shape");
    WN_REQUIRE(a->out_len > 0 && a->out_len <= a->L - a->skip_start, WN_E_BADARG,
               "wn_head_fwd: output_length %d exceeds the %d frames the stack produces", a->out_len,
               a->L - a->skip_start);
    WN_REQUIRE(a->mode == 0, WN_E_UNSUPP, "wn_head_fwd: mode %d not available in this build", a->mode);
    HeadParams p;
    p.skip = a->d_skip; p.logits = a->d_logits; p.w1_t = a->d_w1_t; p.b1 = a->d_b1; p.w2_t = a->d_w2_t; p.b2 = a->d_b2;
    p.B = a->B; p.L = a->L; p.S = a->S; p.E = a->E; p.classes = a->classes; p.skip_start = a->skip_start;
    p.out_len = a->out_len;
    p.N1p = n2p_of(a->E); p.N2p = n2p_of(a->classes); p.Kz = p.N1p;
    const int tm = pick_tm(p.Kz, smem_limit_bytes());
    WN_REQUIRE(tm > 0, WN_E_UNSUPP, "wn_head_fwd: end_channels=%d does not fit shared memory", a->E);
    const size_t smem = two_phase_smem(tm, p.Kz);
    cudaStream_t st = (cudaStream_t)stream;
    switch (tm) {
        case 128: return launch_head<128>(p, smem, st);
        case 64: return launch_head<64>(p, smem, st);
        case 32: return launch_head<32>(p, smem, st);
        default: return launch_head<16>(p, smem, st);
    }
}
