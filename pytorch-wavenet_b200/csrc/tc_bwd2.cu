// tc_bwd2.cu -- backward of the residual block (what autograd computes through reference wavenet_model.py:142-165 after
// loss.backward(), wavenet_training.py:71) on the chunked bf16-pair layout of tc_block.cu, wgmma throughout.
//
// Data gradients, two launches per block (the second needs dF|dG of OTHER frames, t and t + d, so it cannot be fused):
//   pair_gemm<EPI_DZ>  dz[t] = Wr^T dh_out[t] + Ws^T dskip[t]           (K = 512, N = 256 dilation channels)
//                      epilogue: dF = dz g (1 - f^2), dG = dz f g (1 - g), z = f g  ->  dFG pair (512 ch), z pair
//   pair_gemm<EPI_DH>  dh_in[t] = dh_out[t] + sum_tap [Wf;Wg]_tap^T dFG[t + (1-tap) d]      (K = 1024, N = 256 residual ch.)
// Same machinery as the forward's pass A: 256-frame items over a CTA pair (128 frames per CTA), a ring of 48 KB stages
// (activation slot + both weight halves per 32-channel k-slab), two consumer warpgroups with register accumulators of
// 64 frames x 256 columns each, the TMA producer running ahead while they compute the epilogue.  Frames outside a tensor's valid range come back as zeros from the TMA bounds check, which
// is exactly the structure of the gradients (zero left of gs_out / ds_start / gz, nothing right of L).
//
// Weight gradients: dW[n][c] = sum_b sum_t g[b][t][n] x[b][t][c] contracts over FRAMES.  In the chunked layout a tile
// [8-channel chunk][frame][8] is the SWIZZLE_NONE *MN-major* operand image (LBO = 128 between 8-frame groups, SBO =
// frames*16 between chunks), so the TMA boxes feed wgmma directly as transposed operands -- no transposing splitter.  One
// launch per block covers all six 256x256 jobs (skip, residual, filter/gate x 2 taps); a job is split over frame ranges
// across CTA pairs (each CTA of a pair takes 128 of the 256 rows), partial sums go to a workspace and a second kernel adds them in fixed order (deterministic).
#include "common.cuh"
#include "tc_ptx.cuh"
#include <cstdlib>
#include <cstring>

namespace wn {
namespace tb {
int make_pair_map(CUtensorMap* m, const void* base, int B, int L, int C, int origin, int box_frames, int box_chunks, int box_planes);
int make_wrows_map(CUtensorMap* m, const void* base, long long rows);
}
namespace tb2 {
using namespace px;

constexpr int BM = 128, PM = 256;
constexpr int SLOT = 16384, STAGE = 3 * SLOT;
constexpr int NTHREADS = 288, EPI_WARPS = 8, CONSUMERS = 256;     // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int NST = (227 * 1024 - 384) / STAGE;
constexpr unsigned LBO = BM * 16, SBO = 128;
enum { EPI_DZ = 0, EPI_DH = 1 };

// channels and operand precision, as tb::Cfg (tc_block.cu): PAIR = bf16 (hi, lo) operand pairs, three MMAs per product;
// !PAIR = single-pass bf16 operands (hi planes only).  Gradient tensors are always STORED as pairs.
template <int CH_, bool PAIR_>
struct Cfg {
    static constexpr int CH = CH_;
    static constexpr bool PAIR = PAIR_;
    static constexpr int PLANES = PAIR ? 2 : 1;
    static constexpr int KC = PAIR ? 4 : 8;                  // 8-channel chunks per k-slab slot
    static constexpr int KS = KC * 8;
    static constexpr int NT = CH / 256;                      // 256-column n-tiles of dz (dilation channels) / dh_in (residual channels)
    static constexpr int SLABS_DZ = 2 * CH / KS;             // K of dz: [dh_out CH | dskip CH]
    static constexpr int SLABS_DH = 4 * CH / KS;             // K of dh: 2 taps x (dF CH | dG CH)
    static constexpr int WROWS_DZ = NT * SLABS_DZ * 2 * 8;   // 2 KB rows
    static constexpr int WROWS_BWD_LAYER = WROWS_DZ + NT * SLABS_DH * 2 * 8;
    static constexpr size_t WB_LAYER_BYTES = (size_t)WROWS_BWD_LAYER * 2048;
};
constexpr size_t SMEM_PG = 128 + (size_t)NST * STAGE + 256;

struct KSeg { int shift, origin, slabs, pad; };    // A rows of frame t: the segment's tensor at frame t + shift - origin
struct PgParams {
    int B, L, t_begin, tiles_per_seq, n_items;
    int n_seg; KSeg seg[2];
    int w_row0, w_slabs_per_tile, w_slab_off;      // weight half h of (n-tile j, k-slab s): rows w_row0 + ((j*w_slabs_per_tile + w_slab_off + s)*2 + h)*8
    const float4* fg;        // DZ: chunked (B, 2CH/4, L, 4) tanh | sigmoid outputs
    uint4* out0;             // DZ: dFG pair (B, 2, 2CH/8, L, 8)      DH: dh_in pair (B, 2, CH/8, L, 8)
    uint4* out1;             // DZ: z pair (B, 2, CH/8, L, 8)
    const uint4* res;        // DH: dh_out pair or null
    int id_start;            // DH: frames >= id_start carry dh_out straight through
};

template <typename C, int EPI>
__global__ void __launch_bounds__(NTHREADS, 1)
pair_gemm_kernel(const __grid_constant__ CUtensorMap mapA0, const __grid_constant__ CUtensorMap mapA1,
                 const __grid_constant__ CUtensorMap mapW, const PgParams p) {
    constexpr int CH = C::CH;
    extern __shared__ unsigned char smem_raw[];
    unsigned char* ring = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(ring + NST * STAGE);
    unsigned long long* full = bars;                   // [NST]
    unsigned long long* empty = bars + NST;            // [NST]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rank = (int)(blockIdx.x & 1);
    const int n_pairs = gridDim.x >> 1, pair_id = blockIdx.x >> 1;
    if (tid == 0) {
        for (int i = 0; i < NST; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, CONSUMERS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA0) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA1) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapW) : "memory");
    }
    __syncthreads();
    const int slabs = p.seg[0].slabs + (p.n_seg > 1 ? p.seg[1].slabs : 0);

    if (warp == EPI_WARPS) {
        if (lane == 0) {
            unsigned it = 0;
            for (int item = pair_id; item < p.n_items; item += n_pairs) {
                const int b = item / p.tiles_per_seq, t0 = p.t_begin + (item % p.tiles_per_seq) * PM + rank * BM;
                for (int j = 0; j < C::NT; ++j) {
                    int gsl = 0;
                    for (int sg = 0; sg < p.n_seg; ++sg) {
                        const KSeg s = p.seg[sg];
                        const CUtensorMap* map = sg == 0 ? &mapA0 : &mapA1;
                        for (int sl = 0; sl < s.slabs; ++sl, ++gsl, ++it) {
                            const unsigned st = it % NST, ph = (it / NST) & 1;
                            mbar_wait(empty + st, ph ^ 1);
                            mbar_expect_tx(full + st, STAGE);
                            unsigned char* dst = ring + st * STAGE;
                            tma_load_4d(dst, map, 2 * (t0 + s.shift - s.origin), sl * C::KC, 0, b, full + st);
                            for (int h = 0; h < 2; ++h)
                                tma_load_2d(dst + (1 + h) * SLOT, &mapW, 0,
                                            p.w_row0 + ((j * p.w_slabs_per_tile + p.w_slab_off + gsl) * 2 + h) * 8, full + st);
                        }
                    }
                }
            }
        }
    } else {
        const int g = warp >> 2;
        const int r0 = 64 * g + 16 * (warp & 3) + (lane >> 2);        // fragment rows r0, r0 + 8
        const int q2 = 2 * (lane & 3);                                 // fragment columns q2, q2 + 1 of every 8-column group
        const unsigned a_off = (unsigned)(64 * g * 16);
        const size_t L = (size_t)p.L;
        unsigned it = 0;
        float acc[2][64];
        for (int item = pair_id; item < p.n_items; item += n_pairs)
          for (int j = 0; j < C::NT; ++j) {
            const int b = item / p.tiles_per_seq;
            const int tf = p.t_begin + (item % p.tiles_per_seq) * PM + rank * BM;
            const int n0 = j * 256;                                     // first output channel of this n-tile
            for (int sl = 0; sl < slabs; ++sl, ++it) {
                const unsigned s = it % NST, ph = (it / NST) & 1;
                mbar_wait(full + s, ph);
                const unsigned st = s32(ring + s * STAGE);
                wgmma_fence();
#pragma unroll
                for (int ks = 0; ks < C::KS / 16; ++ks)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const unsigned a = st + a_off + ks * 2 * LBO, w = st + (1 + h) * SLOT + ks * 2 * LBO;
                        const unsigned long long ah = wg_desc(a, LBO, SBO), bh = wg_desc(w, LBO, SBO);
                        wgmma_bf16_t00(acc[h], ah, bh, (sl == 0 && ks == 0) ? 0u : 1u);
                        if constexpr (C::PAIR) {
                            wgmma_bf16_t00(acc[h], wg_desc(a + SLOT / 2, LBO, SBO), bh, 1u);
                            wgmma_bf16_t00(acc[h], ah, wg_desc(w + SLOT / 2, LBO, SBO), 1u);
                        }
                    }
                wgmma_commit();
                wgmma_wait0();
                wgmma_keep(acc[0]);
                wgmma_keep(acc[1]);
                mbar_arrive(empty + s);
            }
            if (EPI == EPI_DZ) {
                const float* fg = reinterpret_cast<const float*>(p.fg) + (size_t)b * (2 * CH / 4) * L * 4;
                unsigned* dfg = reinterpret_cast<unsigned*>(p.out0 + (size_t)b * 2 * (2 * CH / 8) * L);   // planes of 2CH/8 chunks
                unsigned* zo = reinterpret_cast<unsigned*>(p.out1 + (size_t)b * 2 * (CH / 8) * L);          // planes of CH/8 chunks
                const size_t pl_fg = (size_t)(2 * CH / 8) * L * 4, pl_z = (size_t)(CH / 8) * L * 4;       // 32-bit words per plane
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int nb = 0; nb < 16; ++nb) {
                        const int n = n0 + 128 * h + 8 * nb + q2;          // first of this thread's two dilation channels
#pragma unroll
                        for (int r = 0; r < 2; ++r) {
                            const int t = tf + r0 + 8 * r;
                            if (t >= p.L) continue;
                            const float2 f = __ldg(reinterpret_cast<const float2*>(fg + ((size_t)(n / 4) * L + t) * 4 + (n & 3)));
                            const float2 gg = __ldg(reinterpret_cast<const float2*>(fg + ((size_t)(CH / 4 + n / 4) * L + t) * 4 + (n & 3)));
                            const float v0 = acc[h][4 * nb + 2 * r], v1 = acc[h][4 * nb + 2 * r + 1];
                            unsigned fh, fl, gh, gl, zh, zl;
                            split2(v0 * gg.x * (1.f - f.x * f.x), v1 * gg.y * (1.f - f.y * f.y), fh, fl);
                            split2(v0 * f.x * gg.x * (1.f - gg.x), v1 * f.y * gg.y * (1.f - gg.y), gh, gl);
                            split2(f.x * gg.x, f.y * gg.y, zh, zl);
                            const size_t wf = ((size_t)(n / 8) * L + t) * 4 + (q2 >> 1);
                            const size_t wg = wf + (size_t)(CH / 8) * L * 4;
                            dfg[wf] = fh; dfg[wf + pl_fg] = fl;
                            dfg[wg] = gh; dfg[wg + pl_fg] = gl;
                            zo[wf] = zh; zo[wf + pl_z] = zl;
                        }
                    }
            } else {
                const size_t pl = (size_t)(CH / 8) * L * 4;                // 32-bit words per plane
                const unsigned* rs = p.res ? reinterpret_cast<const unsigned*>(p.res + (size_t)b * 2 * (CH / 8) * L) : nullptr;
                unsigned* o0 = reinterpret_cast<unsigned*>(p.out0 + (size_t)b * 2 * (CH / 8) * L);
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int nb = 0; nb < 16; ++nb) {
                        const int n = n0 + 128 * h + 8 * nb + q2;          // first of this thread's two residual channels
#pragma unroll
                        for (int r = 0; r < 2; ++r) {
                            const int t = tf + r0 + 8 * r;
                            if (t >= p.L) continue;
                            const size_t w = ((size_t)(n / 8) * L + t) * 4 + (q2 >> 1);
                            float2 x = make_float2(0.f, 0.f);
                            if (rs != nullptr && t >= p.id_start) {
                                const float2 xh = unpack_bf16x2(__ldg(rs + w)), xl = unpack_bf16x2(__ldg(rs + w + pl));
                                x = make_float2(xh.x + xl.x, xh.y + xl.y);
                            }
                            unsigned hi, lo;
                            split2(acc[h][4 * nb + 2 * r] + x.x, acc[h][4 * nb + 2 * r + 1] + x.y, hi, lo);
                            o0[w] = hi;
                            o0[w + pl] = lo;
                        }
                    }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- weight packing (backward)
// dz blocks [n-tile j][k-slab][half r]: N row n = 256j + r*128 + row = dilation channel; K index kk = sl*KS + ck*8 + e: kk < CH ->
// residual_conv.weight[kk][n], else skip_conv.weight[kk-CH][n].  dh blocks [n-tile j][k-slab][r]: N row = residual channel;
// kk = tap*2CH + m (tap 0 pairs with dFG(t + d), tap 1 with dFG(t)), m < CH -> filter.weight[m][n][tap], else gate.
// All layers in one launch: ptrs[layer] = {wf, wg, bf, bg, wr, ws, br, bs} (the table of wn_tb_pack_all_weights).
template <typename C>
__global__ void pack_bwd_all_kernel(const float* const* __restrict__ ptrs, __nv_bfloat16* __restrict__ out_all) {
    constexpr int CH = C::CH;
    const float* const* q = ptrs + (size_t)blockIdx.y * 8;
    const float* wf = q[0]; const float* wg = q[1]; const float* wr = q[4]; const float* ws = q[5];
    __nv_bfloat16* out = out_all + (size_t)blockIdx.y * (C::WB_LAYER_BYTES / 2);
    constexpr int n_dz = C::NT * C::SLABS_DZ * 2, n_blocks = n_dz + C::NT * C::SLABS_DH * 2;
    constexpr int per_plane = SLOT / 2 / C::PLANES;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)n_blocks * per_plane;
         i += (long long)gridDim.x * blockDim.x) {
        const int blk = (int)(i / per_plane), w = (int)(i % per_plane);
        const int ck = w / (BM * 8), row = (w / 8) % BM, e = w % 8;
        float v;
        if (blk < n_dz) {
            const int j = blk / (C::SLABS_DZ * 2), sl = (blk / 2) % C::SLABS_DZ, r = blk % 2;
            const int n = j * 256 + r * 128 + row, kk = sl * C::KS + ck * 8 + e;
            v = kk < CH ? wr[(size_t)kk * CH + n] : ws[(size_t)(kk - CH) * CH + n];
        } else {
            const int bb = blk - n_dz, j = bb / (C::SLABS_DH * 2), sl = (bb / 2) % C::SLABS_DH, r = bb % 2;
            const int n = j * 256 + r * 128 + row, kk = sl * C::KS + ck * 8 + e;
            const int tap = kk / (2 * CH), m = kk % (2 * CH);
            v = m < CH ? wf[((size_t)m * CH + n) * 2 + tap] : wg[((size_t)(m - CH) * CH + n) * 2 + tap];
        }
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        __nv_bfloat16* o = out + (size_t)blk * (SLOT / 2) + w;
        o[0] = h;
        if constexpr (C::PAIR) o[per_plane] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
}

// ============================================================================================== weight gradients
constexpr int WG_KF = 32;                         // frames per k-slab: slot image [plane][chunk 16][frame 32][16 B]
constexpr int WG_STAGE = 3 * SLOT;                // g box (this CTA's 128 channels) + two x boxes (all 256 channels)
constexpr int WG_NST = (227 * 1024 - 384) / WG_STAGE;
constexpr int WG_THREADS = 288;                   // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr size_t SMEM_WG = 128 + (size_t)WG_NST * WG_STAGE + 256;
constexpr int WG_MAX_JOBS = 24;

struct WgJob {
    int g_map, g_chunk0, g_origin;                // g operand: tensor map index, first chunk of the 256-channel M tile, map origin frame
    int x_map, x_origin, x_shift, x_chunk0;       // x operand: frames t + x_shift, first chunk of the 256-channel N tile
    int t_lo, slabs_per_seq, total_slabs;         // frames [t_lo, L) of every sequence, in slabs of 32
    int split0, n_splits, slabs_per_split;        // CTA pairs [split0, split0 + n_splits) work on this job
    int work_slot0;                               // partial (256 x 256 fp32) index of split 0 in the workspace
};
struct WgParams {
    int n_jobs, B;
    WgJob job[WG_MAX_JOBS];
    float* work;
};

// CTA r of a pair computes rows 128r..128r+127 (g channels) x all 256 columns (x channels) of its split's partial
template <bool PAIR>
__global__ void __launch_bounds__(WG_THREADS, 1)
wgrad2_kernel(const __grid_constant__ CUtensorMap m0, const __grid_constant__ CUtensorMap m1, const __grid_constant__ CUtensorMap m2,
              const __grid_constant__ CUtensorMap m3, const __grid_constant__ CUtensorMap m4, const WgParams p) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char* ring = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(ring + WG_NST * WG_STAGE);
    unsigned long long* full = bars;                   // [WG_NST]
    unsigned long long* empty = bars + WG_NST;         // [WG_NST]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rank = (int)(blockIdx.x & 1);
    const int pair_id = blockIdx.x >> 1;
    // which job / split is this pair's
    int ji = -1;
    for (int j = 0; j < p.n_jobs; ++j)
        if (pair_id >= p.job[j].split0 && pair_id < p.job[j].split0 + p.job[j].n_splits) ji = j;
    const WgJob jb = p.job[ji < 0 ? 0 : ji];
    const int sp = pair_id - jb.split0;
    const int s_beg = ji < 0 ? 0 : sp * jb.slabs_per_split;
    const int s_end = ji < 0 ? 0 : (s_beg + jb.slabs_per_split < jb.total_slabs ? s_beg + jb.slabs_per_split : jb.total_slabs);
    const int n_slabs = s_end > s_beg ? s_end - s_beg : 0;
    if (tid == 0) {
        for (int i = 0; i < WG_NST; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, CONSUMERS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto map_of = [&](int i) -> const CUtensorMap* { return i == 0 ? &m0 : (i == 1 ? &m1 : (i == 2 ? &m2 : (i == 3 ? &m3 : &m4))); };
    constexpr int BOX = PAIR ? SLOT : SLOT / 2;        // bytes of one {32 frames, 16 chunks, planes} box

    if (warp == EPI_WARPS) {
        if (lane == 0) {
            const CUtensorMap* gm = map_of(jb.g_map);
            const CUtensorMap* xm = map_of(jb.x_map);
            for (int i = 0; i < n_slabs; ++i) {
                const int s = s_beg + i, b = s / jb.slabs_per_seq, t0 = jb.t_lo + (s % jb.slabs_per_seq) * WG_KF;
                const unsigned st = i % WG_NST, ph = (i / WG_NST) & 1;
                mbar_wait(empty + st, ph ^ 1);
                mbar_expect_tx(full + st, 3 * BOX);
                unsigned char* dst = ring + st * WG_STAGE;
                tma_load_4d(dst, gm, 2 * (t0 - jb.g_origin), jb.g_chunk0 + 16 * rank, 0, b, full + st);
                for (int h = 0; h < 2; ++h)
                    tma_load_4d(dst + (1 + h) * SLOT, xm, 2 * (t0 + jb.x_shift - jb.x_origin), jb.x_chunk0 + 16 * h, 0, b, full + st);
            }
        }
    } else if (ji >= 0) {
        // consumer warpgroup g: rows 64g..64g+63 of this CTA's 128 (= chunks 8g..8g+7 of the g box), both operands MN-major
        constexpr unsigned KLBO = 128, KSBO = WG_KF * 16;               // 8-frame groups / 8-channel chunks
        const int g = warp >> 2;
        float acc[2][64];
        for (int i = 0; i < n_slabs; ++i) {
            const unsigned s = i % WG_NST, ph = (i / WG_NST) & 1;
            mbar_wait(full + s, ph);
            const unsigned st = s32(ring + s * WG_STAGE);
            const unsigned ga = st + (unsigned)g * 8 * KSBO;
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < WG_KF / 16; ++ks)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const unsigned xa = st + (1 + h) * SLOT;
                    const unsigned long long gh = wg_desc(ga + ks * 2 * KLBO, KLBO, KSBO), xh = wg_desc(xa + ks * 2 * KLBO, KLBO, KSBO);
                    wgmma_bf16_t11(acc[h], gh, xh, (i == 0 && ks == 0) ? 0u : 1u);
                    if constexpr (PAIR) {
                        wgmma_bf16_t11(acc[h], wg_desc(ga + BOX / 2 + ks * 2 * KLBO, KLBO, KSBO), xh, 1u);
                        wgmma_bf16_t11(acc[h], gh, wg_desc(xa + BOX / 2 + ks * 2 * KLBO, KLBO, KSBO), 1u);
                    }
                }
            wgmma_commit();
            wgmma_wait0();
            wgmma_keep(acc[0]);
            wgmma_keep(acc[1]);
            mbar_arrive(empty + s);
        }
        // partial[row n = rank*128 + r][256 columns] -> workspace
        const int r0 = 64 * g + 16 * (warp & 3) + (lane >> 2), q2 = 2 * (lane & 3);
        float* out = p.work + ((size_t)(jb.work_slot0 + sp) * 256 + rank * 128) * 256;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int nb = 0; nb < 16; ++nb)
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const float2 v = n_slabs > 0 ? make_float2(acc[h][4 * nb + 2 * r], acc[h][4 * nb + 2 * r + 1]) : make_float2(0.f, 0.f);
                    *reinterpret_cast<float2*>(out + (size_t)(r0 + 8 * r) * 256 + 128 * h + 8 * nb + q2) = v;
                }
    }
}

struct WgOut { float* dst; long long n_stride, c_stride; int work_slot0, n_splits; };
struct WgReduceParams { int n_jobs; WgOut o[WG_MAX_JOBS]; const float* work; };
// dst[n * n_stride + c * c_stride] = sum over the job's splits, in split order (deterministic)
__global__ void wgrad2_reduce_kernel(const WgReduceParams p) {
    const int j = blockIdx.y;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= p.n_jobs || idx >= 256 * 256) return;
    const WgOut o = p.o[j];
    float s = 0.f;
    for (int k = 0; k < o.n_splits; ++k) s += p.work[(size_t)(o.work_slot0 + k) * 65536 + idx];
    o.dst[(idx >> 8) * o.n_stride + (idx & 255) * o.c_stride] = s;
}

}  // namespace tb2
}  // namespace wn

using namespace wn;

// dispatch over (channels, precision): f.template operator()<Cfg>()
template <typename F>
static int with_cfg(int channels, int precision, F&& f) {
    if (precision == WN_PREC_BF16_PAIRS) return f.template operator()<tb2::Cfg<256, true>>();
    if (channels == 256) return f.template operator()<tb2::Cfg<256, false>>();
    return f.template operator()<tb2::Cfg<512, false>>();
}

extern "C" size_t wn_tb_bwd_weight_bytes_per_layer(int channels, int precision) {
    if (!wn_tb_precision_supported(channels, precision)) return 0;
    size_t r = 0;
    with_cfg(channels, precision, [&]<typename C>() { r = C::WB_LAYER_BYTES; return 0; });
    return r;
}

extern "C" int wn_tb_pack_all_bwd_weights(const float* const* d_ptrs, int n_layers, int channels, int precision, void* d_wb_all,
                                          void* stream) {
    WN_REQUIRE(d_ptrs && d_wb_all && n_layers > 0, WN_E_BADARG, "wn_tb_pack_all_bwd_weights: bad arguments");
    WN_REQUIRE(wn_tb_precision_supported(channels, precision), WN_E_UNSUPP, "wn_tb_pack_all_bwd_weights: %d channels with precision %d is not supported",
               channels, precision);
    cudaStream_t st = (cudaStream_t)stream;
    with_cfg(channels, precision, [&]<typename C>() {
        tb2::pack_bwd_all_kernel<C><<<dim3(74, n_layers), 256, 0, st>>>(d_ptrs, (__nv_bfloat16*)d_wb_all);
        return 0;
    });
    WN_CUDA(cudaGetLastError());
    return 0;
}

template <typename C, int EPI>
static int launch_pg(const CUtensorMap& a0, const CUtensorMap& a1, const CUtensorMap& w, const tb2::PgParams& p, cudaStream_t st) {
    int dev = 0, sms = 0;
    WN_CUDA(cudaGetDevice(&dev));
    WN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    WN_CUDA(cudaFuncSetAttribute(tb2::pair_gemm_kernel<C, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tb2::SMEM_PG));
    int grid = 2 * p.n_items;
    const int max_grid = (sms / 2) * 2;
    if (grid > max_grid) grid = max_grid;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(tb2::NTHREADS);
    cfg.dynamicSmemBytes = tb2::SMEM_PG;
    cfg.stream = st;
    WN_CUDA(cudaLaunchKernelEx(&cfg, tb2::pair_gemm_kernel<C, EPI>, a0, a1, w, p));
    WN_CUDA(cudaGetLastError());
    return 0;
}

template <typename C>
static int bwd_data(const wn_tb_bwd_args* a, cudaStream_t st) {
    const int B = a->B, L = a->L, CH = C::CH;
    const bool have_dh = a->d_dh_out != nullptr && a->gs_out < L;
    CUtensorMap mDh, mDs, mW, mDfg;
    if (int rc = tb::make_pair_map(&mDs, a->d_dskip, B, L - a->ds_start, CH, 0, tb2::BM, C::KC, C::PLANES)) return rc;
    if (have_dh) { if (int rc = tb::make_pair_map(&mDh, a->d_dh_out, B, L, CH, a->gs_out, tb2::BM, C::KC, C::PLANES)) return rc; }
    else mDh = mDs;
    if (int rc = tb::make_wrows_map(&mW, a->d_wb_all, (long long)a->n_layers * C::WROWS_BWD_LAYER)) return rc;
    tb2::PgParams p;
    memset(&p, 0, sizeof(p));
    p.B = B; p.L = L;
    // ---- dz + gate backward, frames [gz, L)
    p.t_begin = a->gz;
    p.tiles_per_seq = (L - a->gz + tb2::PM - 1) / tb2::PM;
    p.n_items = B * p.tiles_per_seq;
    const int row0 = a->layer * C::WROWS_BWD_LAYER;
    p.w_row0 = row0; p.w_slabs_per_tile = C::SLABS_DZ;
    if (have_dh) {
        p.n_seg = 2;
        p.seg[0].shift = 0; p.seg[0].origin = a->gs_out; p.seg[0].slabs = CH / C::KS;
        p.seg[1].shift = 0; p.seg[1].origin = a->ds_start; p.seg[1].slabs = CH / C::KS;
        p.w_slab_off = 0;
    } else {
        p.n_seg = 1;
        p.seg[0].shift = 0; p.seg[0].origin = a->ds_start; p.seg[0].slabs = CH / C::KS;
        p.w_slab_off = CH / C::KS;                               // the skip part of the packed dz weights only
    }
    p.fg = (const float4*)a->d_fg; p.out0 = (uint4*)a->d_dfg; p.out1 = (uint4*)a->d_z;
    if (int rc = launch_pg<C, tb2::EPI_DZ>(have_dh ? mDh : mDs, mDs, mW, p, st)) return rc;
    // ---- dh_in = dh_out + anti-causal taps of dFG, frames [gs_in, L)
    if (int rc = tb::make_pair_map(&mDfg, a->d_dfg, B, L, 2 * CH, a->gz, tb2::BM, C::KC, C::PLANES)) return rc;
    p.t_begin = a->gs_in;
    p.tiles_per_seq = (L - a->gs_in + tb2::PM - 1) / tb2::PM;
    p.n_items = B * p.tiles_per_seq;
    p.n_seg = 2;
    p.seg[0].shift = a->dilation; p.seg[0].origin = a->gz; p.seg[0].slabs = 2 * CH / C::KS;
    p.seg[1].shift = 0; p.seg[1].origin = a->gz; p.seg[1].slabs = 2 * CH / C::KS;
    p.w_row0 = row0 + C::WROWS_DZ; p.w_slabs_per_tile = C::SLABS_DH; p.w_slab_off = 0;
    p.fg = nullptr; p.out0 = (uint4*)a->d_dh_in; p.out1 = nullptr;
    p.res = have_dh ? (const uint4*)a->d_dh_out : nullptr;
    p.id_start = a->gs_out > a->out_start ? a->gs_out : a->out_start;
    return launch_pg<C, tb2::EPI_DH>(mDfg, mDfg, mW, p, st);
}

extern "C" int wn_tb_block_bwd_data(const wn_tb_bwd_args* a, void* stream) {
    WN_REQUIRE(a, WN_E_BADARG, "wn_tb_block_bwd_data: null args");
    WN_REQUIRE(a->d_dskip && a->d_fg && a->d_dfg && a->d_z && a->d_dh_in && a->d_wb_all, WN_E_BADARG, "wn_tb_block_bwd_data: null pointer");
    WN_REQUIRE(wn_tb_precision_supported(a->channels, a->precision), WN_E_UNSUPP, "wn_tb_block_bwd_data: %d channels with precision %d is not supported",
               a->channels, a->precision);
    WN_REQUIRE(a->B > 0 && a->L > 0 && a->dilation >= 1 && a->layer >= 0 && a->layer < a->n_layers, WN_E_BADARG, "wn_tb_block_bwd_data: bad sizes");
    WN_REQUIRE(a->gz >= a->out_start && a->gz < a->L && a->gs_in >= a->in_start && a->gs_in <= a->gz && a->ds_start >= a->out_start &&
                   a->ds_start < a->L,
               WN_E_BADARG, "wn_tb_block_bwd_data: bad gradient frame ranges");
    cudaStream_t st = (cudaStream_t)stream;
    return with_cfg(a->channels, a->precision, [&]<typename C>() { return bwd_data<C>(a, st); });
}

extern "C" size_t wn_tb_wgrad_workspace_bytes(void) { return (size_t)160 * 65536 * 4; }

extern "C" int wn_tb_wgrad(const wn_tb_wgrad_args* a, void* stream) {
    WN_REQUIRE(a, WN_E_BADARG, "wn_tb_wgrad: null args");
    WN_REQUIRE(a->d_dskip && a->d_dfg && a->d_z && a->d_h_in && a->d_gws && a->d_gwr && a->d_gwf && a->d_gwg && a->d_work, WN_E_BADARG,
               "wn_tb_wgrad: null pointer");
    WN_REQUIRE(wn_tb_precision_supported(a->channels, a->precision), WN_E_UNSUPP, "wn_tb_wgrad: %d channels with precision %d is not supported",
               a->channels, a->precision);
    WN_REQUIRE(a->B > 0 && a->L > 0 && a->dilation >= 1, WN_E_BADARG, "wn_tb_wgrad: bad sizes");
    cudaStream_t st = (cudaStream_t)stream;
    int dev = 0, sms = 0;
    WN_CUDA(cudaGetDevice(&dev));
    WN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int B = a->B, L = a->L, d = a->dilation, CH = a->channels;
    const bool pair = a->precision == WN_PREC_BF16_PAIRS;
    const int planes = pair ? 2 : 1;
    const bool have_dh = a->d_dh_out != nullptr && a->id_start < L;
    // tensor maps with the MN-major box {32 frames, 16 chunks, planes}: 0 dskip, 1 dh_out, 2 dFG, 3 z, 4 h_in
    CUtensorMap m[5];
    if (int rc = tb::make_pair_map(&m[0], a->d_dskip, B, L - a->ds_start, CH, 0, tb2::WG_KF, 16, planes)) return rc;
    if (have_dh) { if (int rc = tb::make_pair_map(&m[1], a->d_dh_out, B, L, CH, a->id_start, tb2::WG_KF, 16, planes)) return rc; }
    else m[1] = m[0];
    if (int rc = tb::make_pair_map(&m[2], a->d_dfg, B, L, 2 * CH, a->gz, tb2::WG_KF, 16, planes)) return rc;
    if (int rc = tb::make_pair_map(&m[3], a->d_z, B, L, CH, a->gz, tb2::WG_KF, 16, planes)) return rc;
    if (int rc = tb::make_pair_map(&m[4], a->d_h_in, B, L, CH, a->in_start, tb2::WG_KF, 16, planes)) return rc;
    tb2::WgParams p;
    tb2::WgReduceParams rp;
    memset(&p, 0, sizeof(p));
    memset(&rp, 0, sizeof(rp));
    p.B = B; p.work = a->d_work; rp.work = a->d_work;
    int nj = 0;
    const int T = CH / 256;                                   // 256-channel tiles per side
    // out[(n0 + n) * ns + (c0 + c) * cs]: one job per (256 g-channels, 256 x-channels) tile
    auto add = [&](int g_map, int g_chunk_base, int g_origin, int x_map, int x_origin, int x_shift, int t_lo, float* dst, long long ns, long long cs) {
        for (int mt = 0; mt < T; ++mt)
            for (int nt = 0; nt < T; ++nt) {
                tb2::WgJob& j = p.job[nj];
                j.g_map = g_map; j.g_chunk0 = g_chunk_base + 32 * mt; j.g_origin = g_origin;
                j.x_map = x_map; j.x_origin = x_origin; j.x_shift = x_shift; j.x_chunk0 = 32 * nt;
                j.t_lo = t_lo < L ? t_lo : L;
                j.slabs_per_seq = (L - j.t_lo + tb2::WG_KF - 1) / tb2::WG_KF;
                j.total_slabs = B * j.slabs_per_seq;
                rp.o[nj].dst = dst + (size_t)(256 * mt) * ns + (size_t)(256 * nt) * cs; rp.o[nj].n_stride = ns; rp.o[nj].c_stride = cs;
                ++nj;
            }
    };
    const long long CC = CH;
    add(0, 0, a->ds_start, 3, a->gz, 0, a->ds_start, a->d_gws, CC, 1);                                   // skip_conv.weight (S, D, 1)
    if (have_dh) add(1, 0, a->id_start, 3, a->gz, 0, a->id_start, a->d_gwr, CC, 1);                      // residual_conv.weight (R, D, 1)
    for (int tap = 0; tap < 2; ++tap) {
        const int sh = (1 - tap) * d;
        const int lo = a->gz > a->in_start + sh ? a->gz : a->in_start + sh;      // frames whose tap lands on real input
        add(2, 0, a->gz, 4, a->in_start, -sh, lo, a->d_gwf + tap, 2 * CC, 2);          // filter.weight (D, R, 2)[:, :, tap]
        add(2, CH / 8, a->gz, 4, a->in_start, -sh, lo, a->d_gwg + tap, 2 * CC, 2);     // gate.weight
    }
    p.n_jobs = rp.n_jobs = nj;
    // CTA pairs per job proportional to its slabs (at least 1), one wave of sms/2 pairs
    const int n_clusters = sms / 2;
    long long total = 0;
    for (int j = 0; j < nj; ++j) total += p.job[j].total_slabs > 0 ? p.job[j].total_slabs : 1;
    int used = 0, slot = 0;
    for (int j = 0; j < nj; ++j) {
        tb2::WgJob& jb = p.job[j];
        const long long sl = jb.total_slabs > 0 ? jb.total_slabs : 1;
        int n = (int)((sl * (n_clusters - nj)) / total) + 1;
        if (n > jb.total_slabs) n = jb.total_slabs > 0 ? jb.total_slabs : 1;
        jb.slabs_per_split = jb.total_slabs > 0 ? (jb.total_slabs + n - 1) / n : 0;
        if (jb.total_slabs > 0) n = (jb.total_slabs + jb.slabs_per_split - 1) / jb.slabs_per_split;
        jb.n_splits = n; jb.split0 = used; jb.work_slot0 = slot;
        rp.o[j].work_slot0 = slot; rp.o[j].n_splits = n;
        used += n; slot += n;
    }
    WN_REQUIRE((size_t)slot * 65536 * 4 <= wn_tb_wgrad_workspace_bytes(), WN_E_UNSUPP, "wn_tb_wgrad: workspace too small for %d partials", slot);
    if (!have_dh) WN_CUDA(cudaMemsetAsync(a->d_gwr, 0, sizeof(float) * CC * CC, st));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(2 * used));
    cfg.blockDim = dim3(tb2::WG_THREADS);
    cfg.dynamicSmemBytes = tb2::SMEM_WG;
    cfg.stream = st;
    if (pair) {
        WN_CUDA(cudaFuncSetAttribute(tb2::wgrad2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tb2::SMEM_WG));
        WN_CUDA(cudaLaunchKernelEx(&cfg, tb2::wgrad2_kernel<true>, m[0], m[1], m[2], m[3], m[4], p));
    } else {
        WN_CUDA(cudaFuncSetAttribute(tb2::wgrad2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tb2::SMEM_WG));
        WN_CUDA(cudaLaunchKernelEx(&cfg, tb2::wgrad2_kernel<false>, m[0], m[1], m[2], m[3], m[4], p));
    }
    WN_CUDA(cudaGetLastError());
    tb2::wgrad2_reduce_kernel<<<dim3(256, nj), 256, 0, st>>>(rp);
    WN_CUDA(cudaGetLastError());
    return 0;
}
