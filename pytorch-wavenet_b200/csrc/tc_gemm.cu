// tc_gemm.cu -- tensor-core (wgmma / TMA) form of the training block: fp32-class numerics through bf16 (hi, lo) operand
// pairs (hi = bf16(x), lo = bf16(x - hi); hi*hi + lo*hi + hi*lo per k-step, fp32 accumulation in registers): 16 mantissa
// bits per operand, ~3e-6 on the logits after 50 layers (inside the 1e-4 bar).
//
// Same mathematics and frames layout as train_fwd.cu (reference wavenet_model.py:142-165), split in two launches
// per block because the gated activation cannot stay on chip in split form (128 frames x 256 ch x {hi,lo} = 256 KB):
//   pass A   FG[128 frames x 256] per tile = A[128 x kR] * Wa^T      A rows = taps of h_in (TMA boxes shifted by
//            the dilation; frames left of in_start come back as zeros from the TMA out-of-bounds fill)
//            epilogue: z = tanh(F+bf) * sigmoid(G+bg)  -> z (B,L,D)  [+ optional f,g for the backward]
//   pass B   [O|S][128 x 256] per tile = z[128 x D] * Wb^T ;  h_out = O + br + h_in,  skip (+)= S + bs
// Kernel anatomy (one CTA per SM, persistent over (sequence, 128-frame tile) items, 288 threads):
//   warp 8        TMA producer: per K slab (16 fp32 = one 64-byte swizzle row) loads A raw, W_hi, W_lo (6-stage ring)
//   warps 0-7     two consumer warpgroups, each owning 64 of the 128 frames: split the warpgroup's rows of the landed A
//                 slab into bf16 hi / lo tiles, issue wgmma m64n128k16 bf16 (hi*hi + lo*hi + hi*lo) into two 128-column
//                 register accumulators, then apply gate / residual / skip from the fragments
// mbarriers: full (TMA landed), empty (every consumer thread is done with the stage).
#include "common.cuh"
#include "tc_ptx.cuh"
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstdlib>
#include <cstring>

namespace wn {
namespace tc {
using namespace px;

constexpr int BM = 128;            // frames per tile (UMMA M)
constexpr int BN = 256;            // output columns per tile (UMMA N)
constexpr int BK = 16;             // fp32 per K slab = 64 bytes = one 64B-swizzle row (one bf16 k-step)
// the operand tiles are bf16 (hi, lo) pairs with 32-byte rows; the raw fp32 A slab keeps its own buffer, so a stage is
// A_raw 8K | A_hi 4K | A_lo 4K | W_hi 8K | W_lo 8K = 32 KB and six stages fit
constexpr int STAGES = 6;
constexpr int A_BYTES = BM * BK * 4;          // 8 KB
constexpr int ABF_BYTES = BM * BK * 2;        // 4 KB
constexpr int WBF_BYTES = BN * BK * 2;        // 8 KB
constexpr int STAGE_BYTES = A_BYTES + 2 * ABF_BYTES + 2 * WBF_BYTES;     // 32 KB
constexpr int NTHREADS = 288;             // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int CONSUMERS = 256;

// swizzled K-major descriptor (layout 3 = 32B swizzle): sbo = bytes between 8-row atoms
__device__ __forceinline__ unsigned long long desc32(unsigned saddr) { return wg_desc(saddr, 16, 8 * 32, 3); }

// ---------------------------------------------------------------------------------------------- kernel
enum { EPI_GATE = 0, EPI_RES_SKIP = 1, EPI_GATE_BWD = 2, EPI_ADD = 3 };

struct TcParams {
    int B, L, t_begin;            // frames [t_begin, L) of every sequence are produced
    int taps, dil, C;             // A row = taps x C channels; tap j reads frame t - (taps-1-j)*dil  (dil < 0: future frames)
    int a_origin;                 // frame that coordinate 0 of the A tensor map corresponds to
    // optional second A source appended along K (backward dz: A row = [dh_out(t) | dskip(t)]): C2 channels read through
    // mapA2 at frame t - a2_origin; when C2 > 0 and C == 0 the first source is absent (last layer: no dh_out)
    int C2, a2_origin;
    int n_tiles, n_total;         // output columns = n_tiles * BN; the W map holds hi rows [0,n_total) then lo rows
    // epilogue
    const float* bias;            // [n_total] in tile column order
    float* out0;                  // GATE: z (B,L,D)            RES_SKIP: h_out (B,L,R)
    float* out1;                  // GATE: fg_save (B,L,2D)|0   RES_SKIP: skip (B,L-skip_start,S)
    const float* res;             // RES_SKIP: h_in (B,L,R)     GATE_BWD: fg (B,L,2D)      ADD: dh_out (B,L,R) or null
    float* out2;                  // GATE_BWD: z (B,L,D)
    int id_start;                 // ADD: frames >= id_start carry `res` straight through
    int D, R, S, in_start, skip_start, skip_init;
    long long* dbg;               // optional trace buffer (WN_TC_TRACE): CTA 0 stamps clock64 per stage, see tools/tc_trace.py
};

__device__ __forceinline__ float sigmoid_tc(float x) { return 1.f / (1.f + expf(-x)); }

template <int EPI>
__global__ void __launch_bounds__(NTHREADS, 1)
frames_gemm_tc(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapA2,
               const __grid_constant__ CUtensorMap mapW, const TcParams p) {
    constexpr int ST = STAGES, SB = STAGE_BYTES;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned char* stage_mem = base;                                           // ST * SB
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(base + ST * SB);
    unsigned long long* full = bars;                 // [ST]
    unsigned long long* empty = bars + ST;           // [ST]
    float* bias_s = reinterpret_cast<float*>(base + ST * SB + 512);                                // [n_total]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m_tiles = (p.L - p.t_begin + BM - 1) / BM;
    const int items = p.B * m_tiles;                            // item = (sequence b, 128-frame tile), dealt round-robin to the CTAs
    const int slabs_per_tap = p.C / BK;
    const int slabs1 = p.taps * slabs_per_tap;                  // K slabs of the first A source
    const int slabs = slabs1 + p.C2 / BK;

    if (tid == 0) {
        for (int i = 0; i < ST; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, CONSUMERS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapW) : "memory");
    }
    for (int i = tid; i < p.n_total; i += NTHREADS) bias_s[i] = p.bias ? p.bias[i] : 0.f;
    __syncthreads();

    if (warp == 8) {
        // ================================================================= TMA producer
        if (lane == 0) {
            unsigned it = 0;
            for (int item = blockIdx.x; item < items; item += gridDim.x) {
                const int b = item / m_tiles, t0 = p.t_begin + (item % m_tiles) * BM;
                for (int nt = 0; nt < p.n_tiles; ++nt)
                    for (int sl = 0; sl < slabs; ++sl, ++it) {
                        const int st = it % ST;
                        const unsigned ph = (it / ST) & 1;
                        if (p.dbg && blockIdx.x == 0 && it < 512) p.dbg[it * 8 + 0] = clock64();
                        mbar_wait(empty + st, ph ^ 1);
                        if (p.dbg && blockIdx.x == 0 && it < 512) p.dbg[it * 8 + 1] = clock64();
                        unsigned char* sm = stage_mem + st * SB;
                        mbar_expect_tx(full + st, A_BYTES + 2 * WBF_BYTES);
                        if (sl < slabs1) {
                            const int j = sl / slabs_per_tap, c0 = (sl % slabs_per_tap) * BK;
                            tma_load_3d(sm, &mapA, c0, t0 - (p.taps - 1 - j) * p.dil - p.a_origin, b, full + st);
                        } else {
                            tma_load_3d(sm, &mapA2, (sl - slabs1) * BK, t0 - p.a2_origin, b, full + st);
                        }
                        constexpr int W0 = A_BYTES + 2 * ABF_BYTES;         // offset of W_hi in the stage
                        for (int h = 0; h < 2; ++h) {                       // the map's box is 128 rows: two per tile
                            tma_load_2d(sm + W0 + h * (WBF_BYTES / 2), &mapW, sl * BK, nt * BN + h * 128, full + st);
                            tma_load_2d(sm + W0 + WBF_BYTES + h * (WBF_BYTES / 2), &mapW, sl * BK, p.n_total + nt * BN + h * 128,
                                        full + st);
                        }
                    }
            }
        }
    } else {
        // ================================================================= consumers: warpgroup g = warps 4g..4g+3, frames 64g..64g+63
        const int g = warp >> 2, gtid = tid & 127;
        const int r0 = 64 * g + 16 * (warp & 3) + (lane >> 2);        // fragment rows r0, r0 + 8
        const int q2 = 2 * (lane & 3);                                 // fragment columns q2, q2 + 1 of every 8-column group
        float acc[2][64];
        unsigned it = 0;
        for (int item = blockIdx.x; item < items; item += gridDim.x) {
            const int b = item / m_tiles, t0 = p.t_begin + (item % m_tiles) * BM;
            for (int nt = 0; nt < p.n_tiles; ++nt) {
                for (int sl = 0; sl < slabs; ++sl, ++it) {
                    const int st = it % ST;
                    const unsigned ph = (it / ST) & 1;
                    if (p.dbg && blockIdx.x == 0 && it < 512 && tid == 0) p.dbg[it * 8 + 2] = clock64();
                    mbar_wait(full + st, ph);
                    if (p.dbg && blockIdx.x == 0 && it < 512 && tid == 0) p.dbg[it * 8 + 3] = clock64();
                    unsigned char* sm = stage_mem + st * SB;
                    // ---- split this warpgroup's 64 rows of the raw A slab (rows are 64 bytes = 4 float4)
                    // raw slab: 128 rows x 64 bytes, 64B-swizzled by the TMA (16-byte chunk c of row r sits at c ^ ((r>>1)&3));
                    // operand tiles: 128 rows x 32 bytes of bf16, 32B swizzle (chunk c of row r sits at c ^ ((r>>2)&1))
                    const float4* raw = reinterpret_cast<const float4*>(sm);
                    unsigned char* ahi = sm + A_BYTES;
                    unsigned char* alo = ahi + ABF_BYTES;
#pragma unroll
                    for (int i = g * 256 + gtid; i < g * 256 + 256; i += 128) {
                        const float4 x = raw[i];
                        const int row = i >> 2, lch = (i & 3) ^ ((row >> 1) & 3);      // logical chunk: fp32 k = 4*lch .. 4*lch+3
                        const __nv_bfloat162 h01 = __floats2bfloat162_rn(x.x, x.y), h23 = __floats2bfloat162_rn(x.z, x.w);
                        const float2 f01 = __bfloat1622float2(h01), f23 = __bfloat1622float2(h23);
                        const __nv_bfloat162 l01 = __floats2bfloat162_rn(x.x - f01.x, x.y - f01.y);
                        const __nv_bfloat162 l23 = __floats2bfloat162_rn(x.z - f23.x, x.w - f23.y);
                        const unsigned off = (unsigned)row * 32u + ((unsigned)((lch >> 1) ^ ((row >> 2) & 1)) << 4) + (unsigned)(lch & 1) * 8u;
                        uint2 hv, lv;
                        hv.x = *reinterpret_cast<const unsigned*>(&h01); hv.y = *reinterpret_cast<const unsigned*>(&h23);
                        lv.x = *reinterpret_cast<const unsigned*>(&l01); lv.y = *reinterpret_cast<const unsigned*>(&l23);
                        *reinterpret_cast<uint2*>(ahi + off) = hv;
                        *reinterpret_cast<uint2*>(alo + off) = lv;
                    }
                    fence_async_smem();                       // generic writes -> visible to the MMA
                    wg_bar(1 + g, 128);
                    if (p.dbg && blockIdx.x == 0 && it < 512 && tid == 0) p.dbg[it * 8 + 4] = clock64();
                    // ---- MMAs of this warpgroup's 64 rows against both 128-row halves of the weight tile
                    const unsigned sa = s32(sm);
                    wgmma_fence();
                    const unsigned a_hi = sa + A_BYTES + g * 64 * 32, a_lo = a_hi + ABF_BYTES;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const unsigned w_hi = sa + A_BYTES + 2 * ABF_BYTES + h * (WBF_BYTES / 2), w_lo = w_hi + WBF_BYTES;
                        wgmma_bf16_t00(acc[h], desc32(a_hi), desc32(w_hi), sl != 0);
                        wgmma_bf16_t00(acc[h], desc32(a_lo), desc32(w_hi), 1u);
                        wgmma_bf16_t00(acc[h], desc32(a_hi), desc32(w_lo), 1u);
                    }
                    wgmma_commit();
                    wgmma_wait0();
                    wgmma_keep(acc[0]);
                    wgmma_keep(acc[1]);
                    mbar_arrive(empty + st);                     // stage reusable once every consumer thread got here
                    if (p.dbg && blockIdx.x == 0 && it < 512 && tid == 0) p.dbg[it * 8 + 5] = clock64();
                }
                // ================================================================= epilogue from the fragments
                const int n0 = nt * BN;
                const int Tsk = p.L - p.skip_start;
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int nb = 0; nb < 16; ++nb)
#pragma unroll
                        for (int r = 0; r < 2; ++r) {
                            const int fr = t0 + r0 + 8 * r;
                            if (fr >= p.L) continue;
                            const float v0 = acc[h][4 * nb + 2 * r], v1 = acc[h][4 * nb + 2 * r + 1];
                            const int c = 8 * nb + q2;                       // column inside the 128-column half
                            if (EPI == EPI_GATE) {
                                // tile columns: half 0 = F of channels 128*nt.., half 1 = G of the same channels
                                if (h == 1) continue;
                                const float* bt = bias_s + n0;
                                const float gv0 = acc[1][4 * nb + 2 * r], gv1 = acc[1][4 * nb + 2 * r + 1];
                                const float f0 = tanhf(v0 + bt[c]), f1 = tanhf(v1 + bt[c + 1]);
                                const float g0 = sigmoid_tc(gv0 + bt[128 + c]), g1 = sigmoid_tc(gv1 + bt[128 + c + 1]);
                                const int ch = nt * 128 + c;
                                *reinterpret_cast<float2*>(p.out0 + ((size_t)b * p.L + fr) * p.D + ch) = make_float2(f0 * g0, f1 * g1);
                                if (p.out1) {
                                    float* fs = p.out1 + ((size_t)b * p.L + fr) * (2 * p.D) + ch;
                                    *reinterpret_cast<float2*>(fs) = make_float2(f0, f1);
                                    *reinterpret_cast<float2*>(fs + p.D) = make_float2(g0, g1);
                                }
                            } else if (EPI == EPI_GATE_BWD) {
                                // dz (columns = dilation channels n): dF = dz*g*(1-f^2), dG = dz*f*g*(1-g), z = f*g
                                const int n = n0 + 128 * h + c;
                                const float* fgp = p.res + ((size_t)b * p.L + fr) * (2 * p.D) + n;
                                const float2 f = __ldg(reinterpret_cast<const float2*>(fgp));
                                const float2 gg = __ldg(reinterpret_cast<const float2*>(fgp + p.D));
                                float* dfg = p.out0 + ((size_t)b * p.L + fr) * (2 * p.D) + n;
                                *reinterpret_cast<float2*>(dfg) = make_float2(v0 * gg.x * (1.f - f.x * f.x), v1 * gg.y * (1.f - f.y * f.y));
                                *reinterpret_cast<float2*>(dfg + p.D) = make_float2(v0 * f.x * gg.x * (1.f - gg.x), v1 * f.y * gg.y * (1.f - gg.y));
                                *reinterpret_cast<float2*>(p.out2 + ((size_t)b * p.L + fr) * p.D + n) = make_float2(f.x * gg.x, f.y * gg.y);
                            } else if (EPI == EPI_ADD) {
                                // dh_in (columns = residual channels n) = acc + dh_out(t) for t >= id_start
                                const int n = n0 + 128 * h + c;
                                float2 x = make_float2(0.f, 0.f);
                                if (p.res != nullptr && fr >= p.id_start) x = __ldg(reinterpret_cast<const float2*>(p.res + ((size_t)b * p.L + fr) * p.R + n));
                                *reinterpret_cast<float2*>(p.out0 + ((size_t)b * p.L + fr) * p.R + n) = make_float2(v0 + x.x, v1 + x.y);
                            } else {
                                // global output column n: n < R residual, else skip channel n - R
                                const int n = n0 + 128 * h + c;
                                const float o0 = v0 + bias_s[n], o1 = v1 + bias_s[n + 1];
                                if (n0 < p.R) {
                                    float2 x = make_float2(0.f, 0.f);
                                    if (fr >= p.in_start) x = __ldg(reinterpret_cast<const float2*>(p.res + ((size_t)b * p.L + fr) * p.R + n));
                                    *reinterpret_cast<float2*>(p.out0 + ((size_t)b * p.L + fr) * p.R + n) = make_float2(o0 + x.x, o1 + x.y);
                                } else if (fr >= p.skip_start) {
                                    float* sk = p.out1 + ((size_t)b * Tsk + (fr - p.skip_start)) * p.S + (n - p.R);
                                    float2 x = make_float2(0.f, 0.f);
                                    if (!p.skip_init) x = *reinterpret_cast<const float2*>(sk);
                                    *reinterpret_cast<float2*>(sk) = make_float2(o0 + x.x, o1 + x.y);
                                }
                            }
                        }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- weight packing
// Every packed weight array is [2][rows][K] bf16: element i of a [rows][K] image as hi = bf16(x) at i, lo = bf16(x - hi) at
// total + i.
__device__ __forceinline__ void put_pair(__nv_bfloat16* __restrict__ w, long long total, long long i, float v) {
    const __nv_bfloat16 hi = __float2bfloat16_rn(v);
    w[i] = hi;
    w[total + i] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// pass A: rows in tile order (tile p: F channels 128p.., then G channels 128p..), columns kk = j*R + r
__global__ void pack_a_kernel(const float* __restrict__ wf, const float* __restrict__ wg, const float* __restrict__ bf,
                              const float* __restrict__ bg, int R, int D, int k, __nv_bfloat16* __restrict__ wa,
                              float* __restrict__ ba) {
    const int K = k * R, N = 2 * D;
    const long long total = (long long)N * K;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i / K), kk = (int)(i % K);
        const int tile = n / 256, w = n % 256, ch = tile * 128 + (w & 127);
        const bool is_g = w >= 128;
        const int j = kk / R, r = kk % R;
        put_pair(wa, total, i, (is_g ? wg : wf)[((size_t)ch * R + r) * k + j]);
        if (kk == 0) {
            const float* bsrc = is_g ? bg : bf;
            ba[n] = bsrc ? bsrc[ch] : 0.f;
        }
    }
}
// pass B: rows = residual outputs then skip outputs, columns = dilation channel
__global__ void pack_b_kernel(const float* __restrict__ wr, const float* __restrict__ ws, const float* __restrict__ br,
                              const float* __restrict__ bs, int R, int D, int S, __nv_bfloat16* __restrict__ wb,
                              float* __restrict__ bb) {
    const int N = R + S;
    const long long total = (long long)N * D;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int n = (int)(i / D), c = (int)(i % D);
        put_pair(wb, total, i, n < R ? wr[(size_t)n * D + c] : ws[(size_t)(n - R) * D + c]);
        if (c == 0) bb[n] = n < R ? (br ? br[n] : 0.f) : (bs ? bs[n - R] : 0.f);
    }
}

// backward dz: rows = dilation channels c, columns k: [0,R) = residual_conv.weight[k][c], [R,R+S) = skip_conv.weight[k-R][c]
__global__ void pack_dz_kernel(const float* __restrict__ wr, const float* __restrict__ ws, int R, int D, int S,
                               __nv_bfloat16* __restrict__ w) {
    const int K = R + S;
    const long long total = (long long)D * K;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i / K), kk = (int)(i % K);
        put_pair(w, total, i, kk < R ? wr[(size_t)kk * D + c] : ws[(size_t)(kk - R) * D + c]);
    }
}
// backward dh_in: rows = residual channels r, columns j*2D + n: [filter;gate].weight[n][r][j]
__global__ void pack_dh_kernel(const float* __restrict__ wf, const float* __restrict__ wg, int R, int D, int k,
                               __nv_bfloat16* __restrict__ w) {
    const int K = k * 2 * D;
    const long long total = (long long)R * K;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i / K), kk = (int)(i % K);
        const int j = kk / (2 * D), n = kk % (2 * D);
        put_pair(w, total, i, n < D ? wf[((size_t)n * R + r) * k + j] : wg[((size_t)(n - D) * R + r) * k + j]);
    }
}

// ---------------------------------------------------------------------------------------------- host: tensor maps
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && p)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}
// activations (B, L, C) fp32: dims {C, L - origin, B}, box {32, 128, 1}; frames left of `origin` are out of bounds -> zeros
static int make_act_map(CUtensorMap* m, const float* base, int B, int L, int C, int origin) {
    EncodeTiledFn fn = encode_fn();
    WN_REQUIRE(fn, WN_E_UNSUPP, "cuTensorMapEncodeTiled is not available from this driver");
    WN_REQUIRE(L - origin >= 1, WN_E_BADARG, "empty activation range");
    cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)(L - origin), (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)C * 4, (cuuint64_t)L * C * 4};
    cuuint32_t box[3] = {BK, BM, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)(base + (size_t)origin * C), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, (BK * 4 == 128) ? CU_TENSOR_MAP_SWIZZLE_128B : (BK * 4 == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B), CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    WN_REQUIRE(r == CUDA_SUCCESS, WN_E_UNSUPP, "cuTensorMapEncodeTiled(activations) failed with %d", (int)r);
    return 0;
}
// weights (rows, K) bf16 K-major, one plane of a [2][rows][K] pair array: dims {K, rows}, box {BK, 128} (32-byte slab rows)
// `col0`: first K column (element offset into every row)
static int make_w_map(CUtensorMap* m, const void* base, int rows, int K, int col0 = 0) {
    EncodeTiledFn fn = encode_fn();
    WN_REQUIRE(fn, WN_E_UNSUPP, "cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    cuuint32_t box[2] = {BK, BN / 2};           // half a tile: 128 rows
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, (void*)((const unsigned char*)base + (size_t)col0 * 2), dims, strides,
                    box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_32B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    WN_REQUIRE(r == CUDA_SUCCESS, WN_E_UNSUPP, "cuTensorMapEncodeTiled(weights) failed with %d", (int)r);
    return 0;
}

static size_t tc_smem_bytes(int n_total) {
    return 1024 + (size_t)STAGES * STAGE_BYTES + 512 + sizeof(float) * ((n_total + 3) & ~3);
}

template <int EPI>
static int launch_tc(const CUtensorMap& mA, const CUtensorMap& mA2, const CUtensorMap& mW, const TcParams& p, cudaStream_t st) {
    int dev = 0, sms = 0;
    WN_CUDA(cudaGetDevice(&dev));
    WN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const size_t smem = tc_smem_bytes(p.n_total);
    WN_CUDA(cudaFuncSetAttribute(frames_gemm_tc<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int items = p.B * ((p.L - p.t_begin + BM - 1) / BM);
    const int grid = items < sms ? items : sms;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(NTHREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    WN_CUDA(cudaLaunchKernelEx(&cfg, frames_gemm_tc<EPI>, mA, mA2, mW, p));
    WN_CUDA(cudaGetLastError());
    return 0;
}


// ============================================================================================== weight gradients
// dW[n][c] = sum over sequences b and frames t of g[b][t][n] * x[b][t][c]  (what wn_wgrad computes on the FMA pipe,
// wgrad.cu) on the tensor cores.  The contraction runs over frames, the SLOW axis of both row-major operands, so the
// tiles arrive "MN-major"; the consumers -- which have to rewrite every element as a bf16 (hi, lo) pair anyway -- write
// the operand tiles TRANSPOSED, i.e. in the same K-major, 32-byte-swizzled form the block kernels use.  One CTA = one
// 128-row tile of n (M) x all C = 256 columns (N) x one range of K slabs (16 frames each); its fp32 partial goes to the
// split-frames workspace and wgrad_tc_reduce_kernel adds the partials.
//   warp 8      TMA producer: raw fp32 tiles g[16 frames][128 ch] and x[16 frames][256 ch] (no swizzle), 4-stage ring
//   warps 0-7   split (thread = (channel, 8 frames): 8 conflict-free LDS.32 down a column, bf16 hi/lo split, one 16-byte
//               store per operand tile row chunk), then warpgroup g issues wgmma for rows 64g..64g+63: hi*hi + lo*hi + hi*lo;
//               after the last slab: registers -> workspace
constexpr int WG_THREADS = 288;
constexpr int WG_SPLIT_THREADS = 256;
constexpr int WG_STAGES = 4;
constexpr int WG_RAW_A = BK * BM * 4;            // 8 KB   [16 frames][128 ch] fp32
constexpr int WG_RAW_B = BK * BN * 4;            // 16 KB  [16 frames][256 ch] fp32
constexpr int WG_STAGE_BYTES = WG_RAW_A + WG_RAW_B + 2 * ABF_BYTES + 2 * WBF_BYTES;      // 48 KB

struct WgTcParams {
    int slabs_per_seq, total_slabs, slabs_per_split, m_tiles;
    int N, C;
    float* work;                  // [splits][N][C]
};

__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad_tc_kernel(const __grid_constant__ CUtensorMap mapG, const __grid_constant__ CUtensorMap mapX, const WgTcParams p) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(base + WG_STAGES * WG_STAGE_BYTES);
    unsigned long long* full = bars;                       // [WG_STAGES] TMA landed
    unsigned long long* empty = bars + WG_STAGES;          // [WG_STAGES] every consumer thread is done with the stage

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int m_tile = blockIdx.x % p.m_tiles, sp = blockIdx.x / p.m_tiles;
    const int s_beg = sp * p.slabs_per_split;
    const int s_end = (s_beg + p.slabs_per_split < p.total_slabs) ? s_beg + p.slabs_per_split : p.total_slabs;
    const int n_slabs = s_end > s_beg ? s_end - s_beg : 0;

    if (tid == 0) {
        for (int i = 0; i < WG_STAGES; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, WG_SPLIT_THREADS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapG) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapX) : "memory");
    }
    __syncthreads();

    if (warp == 8) {
        if (lane == 0) {
            for (int i = 0; i < n_slabs; ++i) {
                const int st = i % WG_STAGES;
                const unsigned ph = (i / WG_STAGES) & 1;
                mbar_wait(empty + st, ph ^ 1);
                unsigned char* sm = base + st * WG_STAGE_BYTES;
                const int s = s_beg + i, b = s / p.slabs_per_seq, t0 = (s % p.slabs_per_seq) * BK;
                mbar_expect_tx(full + st, WG_RAW_A + WG_RAW_B);
                tma_load_3d(sm, &mapG, m_tile * BM, t0, b, full + st);           // frames past the sequence end: zero fill
                tma_load_3d(sm + WG_RAW_A, &mapX, 0, t0, b, full + st);
            }
        }
    } else {
        // ---------------------------------------------------------------- split (256 threads), MMA, then epilogue
        const int g = warp >> 2;
        float acc[2][64];
        for (int i = 0; i < n_slabs; ++i) {
            const int st = i % WG_STAGES;
            const unsigned ph = (i / WG_STAGES) & 1;
            mbar_wait(full + st, ph);
            unsigned char* sm = base + st * WG_STAGE_BYTES;
            const float* rawA = reinterpret_cast<const float*>(sm);
            const float* rawB = reinterpret_cast<const float*>(sm + WG_RAW_A);
            unsigned char* tiles = sm + WG_RAW_A + WG_RAW_B;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                // groups 0..255: A (128 channels x 2 halves of 8 frames); groups 256..767: B (256 channels x 2 halves)
                const int gr = tid + WG_SPLIT_THREADS * j;
                const bool isA = gr < 2 * BM;
                const int gg = isA ? gr : gr - 2 * BM;
                const int nch = isA ? BM : BN;
                const int ch = gg % nch, half = gg / nch;
                const float* src = (isA ? rawA : rawB) + (half * 8) * nch + ch;
                float x[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) x[k] = src[k * nch];
                unsigned hv[4], lv[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) split2(x[2 * k], x[2 * k + 1], hv[k], lv[k]);
                // K-major tile, 32-byte rows (16 bf16), 32B swizzle: 16-byte chunk `half` of row `ch` sits at half ^ ((ch>>2)&1)
                const unsigned off = (unsigned)ch * 32u + ((unsigned)(half ^ ((ch >> 2) & 1)) << 4);
                unsigned char* hi_t = tiles + (isA ? 0 : 2 * ABF_BYTES);
                unsigned char* lo_t = hi_t + (isA ? ABF_BYTES : WBF_BYTES);
                *reinterpret_cast<uint4*>(hi_t + off) = make_uint4(hv[0], hv[1], hv[2], hv[3]);
                *reinterpret_cast<uint4*>(lo_t + off) = make_uint4(lv[0], lv[1], lv[2], lv[3]);
            }
            fence_async_smem();
            wg_bar(1, WG_SPLIT_THREADS);                  // both warpgroups read the whole B tile
            const unsigned sa = s32(tiles);
            const unsigned a_hi = sa + g * 64 * 32, a_lo = a_hi + ABF_BYTES;
            wgmma_fence();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const unsigned b_hi = sa + 2 * ABF_BYTES + h * (WBF_BYTES / 2), b_lo = b_hi + WBF_BYTES;
                wgmma_bf16_t00(acc[h], desc32(a_hi), desc32(b_hi), i != 0);
                wgmma_bf16_t00(acc[h], desc32(a_lo), desc32(b_hi), 1u);
                wgmma_bf16_t00(acc[h], desc32(a_hi), desc32(b_lo), 1u);
            }
            wgmma_commit();
            wgmma_wait0();
            wgmma_keep(acc[0]);
            wgmma_keep(acc[1]);
            mbar_arrive(empty + st);
        }
        // epilogue: fragment rows of the n tile, all 256 columns
        const int r0 = 64 * g + 16 * (warp & 3) + (lane >> 2), q2 = 2 * (lane & 3);
        float* out = p.work + ((size_t)sp * p.N + m_tile * BM) * p.C;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int nb = 0; nb < 16; ++nb)
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const float2 v = n_slabs > 0 ? make_float2(acc[h][4 * nb + 2 * r], acc[h][4 * nb + 2 * r + 1]) : make_float2(0.f, 0.f);
                    *reinterpret_cast<float2*>(out + (size_t)(r0 + 8 * r) * p.C + 128 * h + 8 * nb + q2) = v;
                }
    }
}

__global__ void wgrad_tc_reduce_kernel(const float* __restrict__ work, float* __restrict__ dw, int N, int C, int splits,
                                       long long n_stride, long long c_stride) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= N * C) return;
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += work[(size_t)k * N * C + idx];
    const int n = idx / C, c = idx - n * C;
    dw[n * n_stride + c * c_stride] = s;
}

// raw (B, rows, ld) fp32 rows as a 3D map {channels, rows, B}, box {box_ch, 16, 1}, no swizzle, zero fill past `rows`
static int make_rows_map(CUtensorMap* m, const float* base, int channels, int rows, int B, int ld, long long seq, int box_ch) {
    EncodeTiledFn fn = encode_fn();
    WN_REQUIRE(fn, WN_E_UNSUPP, "cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[3] = {(cuuint64_t)channels, (cuuint64_t)rows, (cuuint64_t)B};
    cuuint64_t strides[2] = {(cuuint64_t)ld * 4, (cuuint64_t)seq * 4};
    cuuint32_t box[3] = {(cuuint32_t)box_ch, BK, 1};
    cuuint32_t estr[3] = {1, 1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    WN_REQUIRE(r == CUDA_SUCCESS, WN_E_UNSUPP, "cuTensorMapEncodeTiled(wgrad rows) failed with %d", (int)r);
    return 0;
}

}  // namespace tc
}  // namespace wn

using namespace wn;

static long long* g_tc_dbg = nullptr;
extern "C" int wn_tc_read_trace(long long* host_out, int n) {
    WN_REQUIRE(g_tc_dbg && host_out && n > 0 && n <= 512 * 8, WN_E_STATE, "wn_tc_read_trace: tracing is off (WN_TC_TRACE=1) or bad n");
    WN_CUDA(cudaDeviceSynchronize());
    WN_CUDA(cudaMemcpy(host_out, g_tc_dbg, sizeof(long long) * n, cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int wn_tc_supported(int R, int D, int S, int k) {
    return (R % 256 == 0) && (S % 256 == 0) && (D % 128 == 0) && k >= 1 && (R + S) <= 2048 && 2 * D <= 2048;
}

extern "C" int wn_tc_pack_block_weights(const float* d_wf, const float* d_wg, const float* d_bf, const float* d_bg,
                                        const float* d_wr, const float* d_ws, const float* d_br, const float* d_bs, int R,
                                        int D, int S, int k, void* d_wa, float* d_ba, void* d_wb, float* d_bb, void* stream) {
    WN_REQUIRE(d_wf && d_wg && d_wr && d_ws && d_wa && d_ba && d_wb && d_bb, WN_E_BADARG, "wn_tc_pack_block_weights: null pointer");
    WN_REQUIRE(wn_tc_supported(R, D, S, k), WN_E_UNSUPP, "wn_tc_pack_block_weights: shape R=%d D=%d S=%d not supported", R, D, S);
    cudaStream_t st = (cudaStream_t)stream;
    tc::pack_a_kernel<<<1024, 256, 0, st>>>(d_wf, d_wg, d_bf, d_bg, R, D, k, (__nv_bfloat16*)d_wa, d_ba);
    tc::pack_b_kernel<<<512, 256, 0, st>>>(d_wr, d_ws, d_br, d_bs, R, D, S, (__nv_bfloat16*)d_wb, d_bb);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_tc_block_fwd(const wn_tc_block_args* a, void* stream) {
    WN_REQUIRE(a, WN_E_BADARG, "wn_tc_block_fwd: null args");
    WN_REQUIRE(a->d_h_in && a->d_h_out && a->d_skip && a->d_z && a->d_wa && a->d_ba && a->d_wb && a->d_bb, WN_E_BADARG,
               "wn_tc_block_fwd: null pointer");
    WN_REQUIRE(wn_tc_supported(a->R, a->D, a->S, a->k), WN_E_UNSUPP, "wn_tc_block_fwd: shape not supported by the tensor-core path");
    WN_REQUIRE(a->B > 0 && a->L > 0 && a->dilation >= 1 && a->in_start >= 0 && a->out_start >= a->in_start &&
                   a->out_start < a->L && a->skip_start >= a->out_start && a->skip_start < a->L,
               WN_E_BADARG, "wn_tc_block_fwd: bad frame ranges");
    cudaStream_t st = (cudaStream_t)stream;
    CUtensorMap mA, mWa, mZ, mWb;
    if (int rc = tc::make_act_map(&mA, a->d_h_in, a->B, a->L, a->R, a->in_start)) return rc;
    if (int rc = tc::make_w_map(&mWa, a->d_wa, 2 * 2 * a->D, a->k * a->R)) return rc;
    if (int rc = tc::make_act_map(&mZ, a->d_z, a->B, a->L, a->D, a->out_start)) return rc;
    if (int rc = tc::make_w_map(&mWb, a->d_wb, 2 * (a->R + a->S), a->D)) return rc;
    tc::TcParams p;
    memset(&p, 0, sizeof(p));
    if (getenv("WN_TC_TRACE")) {
        if (!g_tc_dbg) WN_CUDA(cudaMalloc(&g_tc_dbg, sizeof(long long) * 512 * 8));
        p.dbg = g_tc_dbg;
    }
    p.B = a->B; p.L = a->L; p.t_begin = a->out_start;
    p.D = a->D; p.R = a->R; p.S = a->S; p.in_start = a->in_start; p.skip_start = a->skip_start; p.skip_init = a->skip_init;
    // pass A: conv taps + gate
    p.taps = a->k; p.dil = a->dilation; p.C = a->R; p.a_origin = a->in_start;
    p.n_total = 2 * a->D; p.n_tiles = p.n_total / tc::BN;
    p.bias = a->d_ba; p.out0 = a->d_z; p.out1 = a->d_fg_save; p.res = nullptr;
    if (int rc = tc::launch_tc<tc::EPI_GATE>(mA, mA, mWa, p, st)) return rc;
    // pass B: residual + skip 1x1
    if (const char* which = getenv("WN_TC_TRACE_PASS")) { if (which[0] == 'A') p.dbg = nullptr; }     // keep pass A's stamps
    p.taps = 1; p.dil = 0; p.C = a->D; p.a_origin = a->out_start;
    p.n_total = a->R + a->S; p.n_tiles = p.n_total / tc::BN;
    p.bias = a->d_bb; p.out0 = a->d_h_out; p.out1 = a->d_skip; p.res = a->d_h_in;
    return tc::launch_tc<tc::EPI_RES_SKIP>(mZ, mZ, mWb, p, st);
}

extern "C" int wn_tc_bwd_supported(int R, int D, int S, int k) {
    return (R % 256 == 0) && (S % 256 == 0) && (D % 256 == 0) && k >= 1 && (R + S) <= 2048 && k * 2 * D <= 4096;
}

extern "C" int wn_tc_pack_block_bwd_weights(const float* d_wf, const float* d_wg, const float* d_wr, const float* d_ws, int R,
                                            int D, int S, int k, void* d_wdz, void* d_wdh, void* stream) {
    WN_REQUIRE(d_wf && d_wg && d_wr && d_ws && d_wdz && d_wdh, WN_E_BADARG, "wn_tc_pack_block_bwd_weights: null pointer");
    WN_REQUIRE(wn_tc_bwd_supported(R, D, S, k), WN_E_UNSUPP, "wn_tc_pack_block_bwd_weights: shape not supported");
    cudaStream_t st = (cudaStream_t)stream;
    tc::pack_dz_kernel<<<512, 256, 0, st>>>(d_wr, d_ws, R, D, S, (__nv_bfloat16*)d_wdz);
    tc::pack_dh_kernel<<<1024, 256, 0, st>>>(d_wf, d_wg, R, D, k, (__nv_bfloat16*)d_wdh);
    WN_CUDA(cudaGetLastError());
    return 0;
}

// Tensor-core form of wn_block_bwd_data (same arguments; d_wrs_rows / d_wfg_bwd are replaced by the packed bf16 pairs
// d_wdz [2][D][R+S] and d_wdh [2][R][k*2D] of wn_tc_pack_block_bwd_weights).
extern "C" int wn_tc_block_bwd_data(const wn_block_bwd_args* a, const void* d_wdz, const void* d_wdh, void* stream) {
    WN_REQUIRE(a && d_wdz && d_wdh, WN_E_BADARG, "wn_tc_block_bwd_data: null args");
    WN_REQUIRE(a->d_dskip && a->d_fg && a->d_dfg && a->d_z && a->d_dh_in, WN_E_BADARG, "wn_tc_block_bwd_data: null pointer");
    WN_REQUIRE(wn_tc_bwd_supported(a->R, a->D, a->S, a->k), WN_E_UNSUPP, "wn_tc_block_bwd_data: shape not supported");
    WN_REQUIRE(a->gz >= a->out_start && a->gz < a->L && a->gs_in >= a->in_start && a->gs_in <= a->gz && a->ds_start >= a->out_start &&
                   a->ds_start < a->L,
               WN_E_BADARG, "wn_tc_block_bwd_data: bad gradient frame ranges");
    cudaStream_t st = (cudaStream_t)stream;
    const int R = a->R, D = a->D, S = a->S, L = a->L, B = a->B;
    const bool have_dh = a->d_dh_out != nullptr && a->gs_out < L;
    CUtensorMap mDh, mDs, mW1, mDfg, mW2;
    if (int rc = tc::make_act_map(&mDs, a->d_dskip, B, L - a->ds_start, S, 0)) return rc;          // (B, L-ds_start, S): own frame axis
    if (have_dh) { if (int rc = tc::make_act_map(&mDh, a->d_dh_out, B, L, R, a->gs_out)) return rc; }
    else mDh = mDs;
    if (int rc = tc::make_w_map(&mW1, d_wdz, 2 * D, R + S, have_dh ? 0 : R)) return rc;       // without dh_out: start at column R
    tc::TcParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.L = L; p.D = D; p.R = R; p.S = S;
    // ---- dz + gate backward for frames [gz, L)
    p.t_begin = a->gz;
    p.taps = have_dh ? 1 : 0; p.dil = 0; p.C = have_dh ? R : 0; p.a_origin = a->gs_out;
    p.C2 = S; p.a2_origin = a->ds_start;
    p.n_total = D; p.n_tiles = D / tc::BN;
    p.bias = nullptr; p.out0 = a->d_dfg; p.out2 = a->d_z; p.res = a->d_fg;
    if (int rc = tc::launch_tc<tc::EPI_GATE_BWD>(mDh, mDs, mW1, p, st)) return rc;
    // ---- dh_in = dh_out (identity) + anti-causal taps of dfg, for frames [gs_in, L)
    if (int rc = tc::make_act_map(&mDfg, a->d_dfg, B, L, 2 * D, a->gz)) return rc;
    if (int rc = tc::make_w_map(&mW2, d_wdh, 2 * R, a->k * 2 * D)) return rc;
    p.t_begin = a->gs_in;
    p.taps = a->k; p.dil = -a->dilation; p.C = 2 * D; p.a_origin = a->gz;
    p.C2 = 0; p.a2_origin = 0;
    p.n_total = R; p.n_tiles = R / tc::BN;
    p.out0 = a->d_dh_in; p.out2 = nullptr; p.res = a->d_dh_out;
    p.id_start = a->gs_out > a->out_start ? a->gs_out : a->out_start;
    return tc::launch_tc<tc::EPI_ADD>(mDfg, mDfg, mW2, p, st);
}

// Tensor-core form of wn_wgrad (same argument block and workspace): C must be 256 and N a multiple of 128, pitches and
// strides multiples of 4 floats, pointers 16-byte aligned; bf16-pair split, fp32 accumulation.
extern "C" int wn_tc_wgrad_supported(int N, int C) { return C == tc::BN && N > 0 && N % tc::BM == 0; }

extern "C" int wn_tc_wgrad(const wn_wgrad_args* a, void* stream) {
    WN_REQUIRE(a != nullptr, WN_E_BADARG, "wn_tc_wgrad: null argument block");
    WN_REQUIRE(wn_tc_wgrad_supported(a->N, a->C), WN_E_UNSUPP, "wn_tc_wgrad: needs C == 256 and N %% 128 == 0 (got N=%d C=%d)", a->N, a->C);
    WN_REQUIRE(a->B > 0 && a->rows >= 1, WN_E_BADARG, "wn_tc_wgrad: bad sizes B=%d rows=%d", a->B, a->rows);
    WN_REQUIRE(a->d_g && a->d_x && a->d_dw && a->d_work, WN_E_BADARG, "wn_tc_wgrad: null device pointer");
    WN_REQUIRE(a->ldg >= a->N && a->ldx >= a->C && a->ldg % 4 == 0 && a->ldx % 4 == 0 && a->g_seq_stride % 4 == 0 &&
                   a->x_seq_stride % 4 == 0 && (uintptr_t)a->d_g % 16 == 0 && (uintptr_t)a->d_x % 16 == 0,
               WN_E_BADARG, "wn_tc_wgrad: pitches / strides must be multiples of 4 floats and pointers 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    int dev = 0, sms = 0;
    WN_CUDA(cudaGetDevice(&dev));
    WN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    tc::WgTcParams p;
    p.N = a->N; p.C = a->C; p.work = a->d_work;
    p.m_tiles = a->N / tc::BM;
    p.slabs_per_seq = (a->rows + tc::BK - 1) / tc::BK;
    const long long total = (long long)a->B * p.slabs_per_seq;
    WN_REQUIRE(total < (1ll << 30), WN_E_UNSUPP, "wn_tc_wgrad: too many frames");
    p.total_slabs = (int)total;
    // the workspace holds wn_wgrad_workspace_bytes(N, C) = ceil(296 / (N/128 * C/128)) partials of N x C
    const int max_splits = (296 + 2 * p.m_tiles - 1) / (2 * p.m_tiles);
    int splits = sms / p.m_tiles;
    if (splits > max_splits) splits = max_splits;
    if (splits > p.total_slabs / 4) splits = p.total_slabs / 4;
    if (splits < 1) splits = 1;
    p.slabs_per_split = (p.total_slabs + splits - 1) / splits;
    splits = (p.total_slabs + p.slabs_per_split - 1) / p.slabs_per_split;
    CUtensorMap mG, mX;
    if (int rc = tc::make_rows_map(&mG, a->d_g, a->N, a->rows, a->B, a->ldg, a->g_seq_stride, tc::BM)) return rc;
    if (int rc = tc::make_rows_map(&mX, a->d_x, a->C, a->rows, a->B, a->ldx, a->x_seq_stride, tc::BN)) return rc;
    const size_t smem = 1024 + (size_t)tc::WG_STAGES * tc::WG_STAGE_BYTES + 256;
    WN_CUDA(cudaFuncSetAttribute(tc::wgrad_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    tc::wgrad_tc_kernel<<<p.m_tiles * splits, tc::WG_THREADS, smem, st>>>(mG, mX, p);
    WN_CUDA(cudaGetLastError());
    const int total_out = a->N * a->C;
    tc::wgrad_tc_reduce_kernel<<<(total_out + 255) / 256, 256, 0, st>>>(a->d_work, a->d_dw, a->N, a->C, splits, a->dw_n_stride,
                                                                         a->dw_c_stride);
    WN_CUDA(cudaGetLastError());
    return 0;
}
