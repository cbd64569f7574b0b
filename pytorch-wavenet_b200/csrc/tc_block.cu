// tc_block.cu -- the training-time residual block (reference wavenet_model.py:142-165) as ONE tensor-core kernel per layer.
//
//   z[t]     = tanh(Wf0 h[t-d] + Wf1 h[t] + bf) * sigmoid(Wg0 h[t-d] + Wg1 h[t] + bg)          (h[t] = 0 left of in_start)
//   h_out[t] = Wr z[t] + br + h[t]                                                             t in [out_start, L)
//   skip[t]  (+)= Ws z[t] + bs                                                                 t in [skip_start, L)
//
// Numerics: fp32-class through bf16 PAIRS -- every operand x is carried as hi = bf16(x), lo = bf16(x - hi) and a product is
// hi*hi + lo*hi + hi*lo on wgmma (bf16 operands, fp32 accumulation in registers; 16 mantissa bits per operand, see
// tools/split_sim.py; the parity bar is 1e-4).
//
// Data layout ("chunked pair layout", DESIGN.md section 2): an activation tensor of C channels over L frames is stored as
//   [sequence b][plane: hi, lo][channel chunk c/8][frame t][8 channels] bf16            (same bytes as fp32 (B,L,C))
// so that  (1) a TMA box {128 frames, 4 chunks, 2 planes} lands in shared memory exactly as the SWIZZLE_NONE K-major
// core-matrix image wgmma consumes ([k-chunk][row][16 B], LBO = 2048, SBO = 128): no splitter, no swizzle, no conflicts;
//          (2) the four lanes of a quad hold the 8 channels of one frame of an accumulator fragment, so an epilogue store
// instruction of a warp writes 8 consecutive frames of one chunk = 128 contiguous bytes, with no shared-memory transpose;
//          (3) the same image is the MN-major operand of the weight-gradient GEMM (contraction over frames).
// skip is [b][channel chunk c/4][frame][4 channels] fp32 for the same reason.  Weights are pre-split and pre-tiled into the
// shared-memory image of every (n-tile, k-slab, 128-row half), so a weight slab half is one contiguous 16 KB TMA box.
//
// Kernel: an item is 256 frames; CTA r = blockIdx.x & 1 of a pair owns frames t0+128r..+127 (the two CTAs do not talk).
//   warp 8      TMA producer: ring of 48 KB stages = one activation slot (32 channels of one tap, hi+lo) + the two 16 KB
//               halves of a weight slab; pass B stages carry weights only (its A operand z is resident)
//   warps 0-7   two consumer warpgroups; warpgroup g owns frames 64g..64g+63 of the CTA: wgmma m64n128k16 into two
//               128-column register accumulators, then the epilogue straight from the fragments
// Per item a warpgroup runs pass A, n-tile j: acc0 = filter, acc1 = gate pre-activations of channels 128j..128j+127 (K = 2 taps
// x CH), and writes z as a bf16 pair image into shared memory (the A operand of pass B never leaves the SM; each warpgroup
// reads back only its own rows); pass B: residual tiles, then skip tiles (skipped for items left of skip_start).
#include "common.cuh"
#include "tc_ptx.cuh"
#include <cstdlib>
#include <cstring>
#include <vector>

namespace wn {
namespace tb {
using namespace px;

constexpr int BM = 128;                   // frames per CTA
constexpr int PM = 256;                   // frames per item (CTA pair)
constexpr int SLOT = 16384;               // one activation slot / one weight half
constexpr int STAGE = 3 * SLOT;           // activation slot + both weight halves
constexpr int NTHREADS = 288;
constexpr int EPI_WARPS = 8;              // consumer warps (two warpgroups)
constexpr int CONSUMERS = 32 * EPI_WARPS;
constexpr unsigned LBO = BM * 16, SBO = 128;
constexpr int SMEM_MAX = 227 * 1024;

// Shapes and operand precision.  PAIR: every MMA operand is a bf16 (hi, lo) pair and a product costs three MMAs
// (fp32-class: the parity path).  !PAIR: single-pass bf16 operands (the hi planes only) with fp32 accumulation -- the
// "bf16 training" mode of BASELINE.json configs[4]; the residual stream h and skip stay fp32-class (h is still stored and
// updated as a pair, skip as fp32), only the matrix products see bf16.
template <int CH_, bool PAIR_>
struct Cfg {
    static constexpr int CH = CH_;
    static constexpr bool PAIR = PAIR_;
    static constexpr int PLANES = PAIR ? 2 : 1;              // planes of an MMA operand image
    static constexpr int KC = PAIR ? 4 : 8;                  // 8-channel chunks per k-slab slot: [plane][chunk][row 128][16 B] = 16 KB
    static constexpr int KS = KC * 8;                        // channels per k-slab
    static constexpr int SLABS_A = 2 * CH / KS;              // k-slabs per pass-A n-tile (2 taps)
    static constexpr int SLABS_B = CH / KS;
    static constexpr int NT_A = 2 * CH / 256;                // pass-A n-tiles: [tanh | sigmoid] pre-activations of 128 channels each
    static constexpr int NT_R = CH / 256;                    // pass-B n-tiles: residual, then as many skip tiles
    static constexpr int NT_B = 2 * CH / 256;
    static constexpr int ZPLANE = (CH / 8) * BM * 16;        // one plane of the resident z image
    static constexpr int ZBYTES = PLANES * ZPLANE;
    static constexpr int WROWS_A = NT_A * SLABS_A * 2 * 8;   // 2 KB rows of one layer's packed pass-A weights
    static constexpr int WROWS_LAYER = WROWS_A + NT_B * SLABS_B * 2 * 8;
    static constexpr size_t W_LAYER_BYTES = (size_t)WROWS_LAYER * 2048;
    static constexpr int NST = (SMEM_MAX - 384 - ZBYTES) / STAGE;     // ring depth that fits beside z
    static constexpr size_t SMEM_BYTES = 128 + ZBYTES + (size_t)NST * STAGE + 256;
    static_assert(NST >= 2, "the ring needs two stages beside the z image");
};

// One layer of a launch.  A single-layer launch carries it as a kernel parameter; the whole-stack launch reads an array of
// them from global memory (the tensor map must then be 64-byte aligned there).
struct alignas(128) LayerDesc {
    CUtensorMap mapH;              // this layer's input pair tensor, origin = in_start
    int t_begin, in_start, dil, skip_init;
    int tiles_per_seq, n_items, item_base, w_row0;     // items of this layer are global items [item_base, item_base + n_items)
    const float* bias;             // [bf CH | bg CH | br CH | bs CH]
    const uint4* h_in;             // chunked pair (B, 2, CH/8, L, 8) bf16, viewed as 16-byte pieces
    uint4* h_out;
    float4* fg_save;               // optional chunked (B, 2CH/4, L, 4) fp32: tanh outputs in chunks [0,CH/4), sigmoid after
    int war_layer;                 // >= 0: every item of that earlier layer must be complete before this layer writes h_out
    const float* cond;             // conditioned launches: [B][2CH] per-sequence filter / gate biases [bf + Vf h | bg + Vg h]
    int cond_frames, cond_hop;     // locally conditioned launches: cond is [B][cond_frames][2CH], position t reads frame t / cond_hop
};
static_assert(sizeof(LayerDesc) % 128 == 0, "LayerDesc array elements must keep the tensor map aligned");

struct BlockParams {
    int B, L, skip_start;
    int n_layers, total_items;
    float4* skip;                  // chunked (B, CH/4, L - skip_start, 4) fp32
    const LayerDesc* layers;       // whole-stack launch: [n_layers] in global memory
    unsigned* item_done;           // whole-stack launch: [total_items] arrival counters (2 CTAs x 8 consumer warps = 16 when complete)
    unsigned* layer_done;          //                     [n_layers] completed items per layer
};

__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void wait_counter(const unsigned* p, unsigned target) {
    unsigned spins = 0;
    while (ld_acquire_gpu(p) < target) {
        __nanosleep(64);
        if (++spins > (1u << 24)) asm volatile("trap;");          // a dependency that never completes must not hang the GPU
    }
}

// One k-slab of a warpgroup: acc[h] (+)= A[64 rows x KS] * W_h[KS x 128] for the two weight halves h.  a: this warpgroup's
// rows of the activation image (hi plane), a_lo: bytes to its lo plane, w: the first weight half (the second follows at
// +SLOT, each half's lo plane at +SLOT/2).  first: the slab starts the accumulation.
template <typename C>
__device__ __forceinline__ void slab_mma(float (&acc)[2][64], unsigned a, unsigned a_lo, unsigned w, bool first) {
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < C::KS / 16; ++ks)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const unsigned long long ah = wg_desc(a + ks * 2 * LBO, LBO, SBO), bh = wg_desc(w + h * SLOT + ks * 2 * LBO, LBO, SBO);
            wgmma_bf16_t00(acc[h], ah, bh, (first && ks == 0) ? 0u : 1u);
            if constexpr (C::PAIR) {
                wgmma_bf16_t00(acc[h], wg_desc(a + a_lo + ks * 2 * LBO, LBO, SBO), bh, 1u);
                wgmma_bf16_t00(acc[h], ah, wg_desc(w + h * SLOT + SLOT / 2 + ks * 2 * LBO, LBO, SBO), 1u);
            }
        }
    wgmma_commit();
    wgmma_wait0();
    wgmma_keep(acc[0]);
    wgmma_keep(acc[1]);
}

// Audio-rate local conditioning features (learned upsampling) as extra K-slabs of pass A: Uf c[t] | Ug c[t] is more contraction
// of the filter / gate pre-activations, K = Cpad more rows after the 2 * CH of the two taps.
struct KslabParams {
    CUtensorMap mapC;              // c as a chunked pair tensor (B, 2, Cpad/8, L, 8), origin 0; shared by all layers
    CUtensorMap mapU;              // every layer's packed [Uf; Ug] image (wn_tb_pack_local_weights), 2 KB rows
    int n_slabs;                   // Cpad / KS k-slabs per pass-A n-tile
};

// MULTI = false: one layer (`single`), items are independent.  MULTI = true: ALL layers of a forward in one persistent launch:
// the global item list is layer-major and dealt round-robin to the CTA pairs, an item waits (in its producer) for the items of
// the previous layer that wrote the frames it reads, and announces itself when its epilogues have stored -- no launch gaps and
// no idle tail between layers.  COND: every sequence has its own filter / gate biases, read from the condition table instead of
// bf / bg (a separate instantiation, so the unconditioned kernels carry no trace of it).  FRAMES (with COND): the table has a frame
// axis (local conditioning), and each of a thread's two rows reads its own frame's row of it.  KS (empty, or one KslabParams):
// after each pass-A n-tile's activation slabs the producer streams KslabParams::n_slabs more stages (the c slab at the CTA's
// absolute frames and the two U halves) and the consumers accumulate them with the same slab_mma.  KSLAB runs as its own kernel
// (block_fused_local_kernel), so the other kernels keep their parameter list.
template <typename C, bool MULTI, bool COND, bool FRAMES, bool KSLAB>
__device__ __forceinline__ void block_fused_body(const LayerDesc& single, const CUtensorMap& mapW, const BlockParams p,
                                                 const KslabParams* kslab) {
    constexpr int CH = C::CH, NST = C::NST;
    auto LD = [&](int l) -> const LayerDesc& { return MULTI ? p.layers[l] : single; };
    extern __shared__ unsigned char smem_raw[];
    unsigned char* base = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~(uintptr_t)127);
    unsigned char* zbuf = base;
    unsigned char* ring = base + C::ZBYTES;
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(ring + NST * STAGE);
    unsigned long long* full = bars;                   // [NST]  the stage's bytes have landed
    unsigned long long* empty = bars + NST;            // [NST]  every consumer thread is done with the stage

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int rank = (int)(blockIdx.x & 1);
    const int n_pairs = gridDim.x >> 1, pair_id = blockIdx.x >> 1;

    if (tid == 0) {
        for (int i = 0; i < NST; ++i) { mbar_init(full + i, 1); mbar_init(empty + i, CONSUMERS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapW) : "memory");
    }
    __syncthreads();

    if (warp == EPI_WARPS) {
        // ===================================================================== TMA producer (one lane)
        if (lane == 0) {
            unsigned it = 0;
            auto acquire = [&](unsigned long long*& bar, unsigned bytes) -> unsigned char* {
                const unsigned s = it % NST, ph = (it / NST) & 1;
                mbar_wait(empty + s, ph ^ 1);
                bar = full + s;
                mbar_expect_tx(bar, bytes);
                ++it;
                return ring + s * STAGE;
            };
            int l = 0;
            for (int n = pair_id; n < p.total_items; n += n_pairs) {
                while (n >= LD(l).item_base + LD(l).n_items) ++l;
                const LayerDesc& Ld = LD(l);
                const int item = n - Ld.item_base, dil = Ld.dil, w_row0 = Ld.w_row0;
                const int b = item / Ld.tiles_per_seq, t0 = Ld.t_begin + (item % Ld.tiles_per_seq) * PM;
                const bool need_skip = t0 + PM > p.skip_start;
                const int tc = t0 + rank * BM - Ld.in_start;               // this CTA's first frame, relative to the map origin
                const CUtensorMap* mapH = &Ld.mapH;
                if (MULTI && l > 0) {
                    // the previous layer's items that produced frames [t0 - d, t0 - d + 255] and [t0, t0 + 255] of this sequence
                    // (they also performed the previous accumulation into the skip frames this item updates)
                    const LayerDesc& Lp = LD(l - 1);
                    const int pt = Lp.t_begin, ptiles = Lp.tiles_per_seq;
                    const unsigned* flags = p.item_done + Lp.item_base + b * ptiles;
                    for (int rg = 0; rg < 2; ++rg) {
                        int lo = t0 - (rg == 0 ? dil : 0), hi = lo + PM - 1;
                        lo = lo < pt ? pt : lo;
                        hi = hi >= p.L ? p.L - 1 : hi;
                        if (lo > hi) continue;
                        for (int tl = (lo - pt) / PM; tl <= (hi - pt) / PM; ++tl) wait_counter(flags + tl, 2 * EPI_WARPS);
                    }
                    if (Ld.war_layer >= 0) wait_counter(p.layer_done + Ld.war_layer, (unsigned)LD(Ld.war_layer).n_items);
                    asm volatile("fence.proxy.async;" ::: "memory");      // generic-proxy writes of other SMs -> this thread's TMA reads
                }
                for (int j = 0; j < C::NT_A; ++j) {
                    for (int sl = 0; sl < C::SLABS_A; ++sl) {
                        unsigned long long* bar;
                        unsigned char* dst = acquire(bar, 3 * SLOT);
                        const int tap = sl / (C::SLABS_A / 2);              // tap 0 reads h[t - d], tap 1 reads h[t]
                        tma_load_4d(dst, mapH, 2 * (tc - (1 - tap) * dil), (sl % (C::SLABS_A / 2)) * C::KC, 0, b, bar);
                        for (int h = 0; h < 2; ++h)
                            tma_load_2d(dst + (1 + h) * SLOT, &mapW, 0, w_row0 + ((j * C::SLABS_A + sl) * 2 + h) * 8, bar);
                    }
                    if constexpr (KSLAB) {
                        const KslabParams& kp = *kslab;
                        const int u_row0 = (w_row0 / C::WROWS_LAYER) * C::NT_A * kp.n_slabs * 16;
                        for (int sl = 0; sl < kp.n_slabs; ++sl) {
                            unsigned long long* bar;
                            unsigned char* dst = acquire(bar, 3 * SLOT);
                            tma_load_4d(dst, &kp.mapC, 2 * (t0 + rank * BM), sl * C::KC, 0, b, bar);
                            for (int h = 0; h < 2; ++h)
                                tma_load_2d(dst + (1 + h) * SLOT, &kp.mapU, 0, u_row0 + ((j * kp.n_slabs + sl) * 2 + h) * 8, bar);
                        }
                    }
                }
                for (int j = 0; j < (need_skip ? C::NT_B : C::NT_R); ++j)
                    for (int s8 = 0; s8 < C::SLABS_B; ++s8) {
                        unsigned long long* bar;
                        unsigned char* dst = acquire(bar, 2 * SLOT);
                        for (int h = 0; h < 2; ++h)
                            tma_load_2d(dst + (1 + h) * SLOT, &mapW, 0, w_row0 + C::WROWS_A + ((j * C::SLABS_B + s8) * 2 + h) * 8, bar);
                    }
            }
        }
    } else {
        // ===================================================================== consumers: warpgroup g = warps 4g..4g+3
        const int g = warp >> 2;
        const int r0 = 64 * g + 16 * (warp & 3) + (lane >> 2);        // this thread's fragment rows: r0 and r0 + 8
        const int q2 = 2 * (lane & 3);                                 // its columns in every 8-column group: q2, q2 + 1
        const unsigned a_off = (unsigned)(64 * g * 16);               // the warpgroup's rows inside an operand image
        const size_t plane_stride = (size_t)(CH / 8) * p.L;            // 16-byte pieces per plane of a pair tensor
        const int Tsk = p.L - p.skip_start;
        unsigned it = 0;
        float acc[2][64];
        auto wait_stage = [&]() -> unsigned {
            const unsigned s = it % NST, ph = (it / NST) & 1;
            ++it;
            mbar_wait(full + s, ph);
            return s;
        };
        int l = 0;
        for (int n = pair_id; n < p.total_items; n += n_pairs) {
            while (n >= LD(l).item_base + LD(l).n_items) ++l;
            const LayerDesc& Ld = LD(l);
            const int item = n - Ld.item_base;
            const int b = item / Ld.tiles_per_seq, t0 = Ld.t_begin + (item % Ld.tiles_per_seq) * PM;
            const bool need_skip = t0 + PM > p.skip_start;
            const int tf = t0 + rank * BM;                             // first frame of this CTA
            // pass A reads the filter / gate biases: this item's row of the condition table under COND.  Pass B re-reads the
            // layer's residual / skip biases from the descriptor, so only one bias pointer is live across the MMAs.
            const float* bias = COND ? Ld.cond : Ld.bias;
            const int q2b = (COND && !FRAMES) ? q2 + b * 2 * CH : q2;   // this thread's column, in this item's row under COND
            float* fg_save = reinterpret_cast<float*>(Ld.fg_save);
            const int skip_init = Ld.skip_init;
            // ---------------- pass A + gate: z = tanh(F + bf) * sigmoid(G + bg) -> shared-memory operand image (+ optional saves)
            for (int j = 0; j < C::NT_A; ++j) {
                for (int sl = 0; sl < C::SLABS_A; ++sl) {
                    const unsigned s = wait_stage();
                    const unsigned st = s32(ring + s * STAGE);
                    slab_mma<C>(acc, st + a_off, SLOT / 2, st + SLOT, sl == 0);
                    mbar_arrive(empty + s);
                }
                if constexpr (KSLAB) {
                    for (int sl = 0; sl < kslab->n_slabs; ++sl) {
                        const unsigned s = wait_stage();
                        const unsigned st = s32(ring + s * STAGE);
                        slab_mma<C>(acc, st + a_off, SLOT / 2, st + SLOT, false);
                        mbar_arrive(empty + s);
                    }
                }
                // FRAMES: the table rows of this thread's two rows' frames, derived after the n-tile's MMAs so that nothing new is
                // live across them; rows past L (last tile) read the last frame's row
                const float* fr[2] = {nullptr, nullptr};
                if constexpr (FRAMES) {
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const int t = tf + r0 + 8 * r, tc = t < p.L ? t : p.L - 1;
                        fr[r] = bias + ((size_t)b * Ld.cond_frames + tc / Ld.cond_hop) * 2 * CH + j * 128 + q2;
                    }
                }
#pragma unroll
                for (int nb = 0; nb < 16; ++nb) {
                    const int ch = j * 128 + 8 * nb + q2;                      // first of this thread's two dilation channels
                    const float* bq = COND ? bias + j * 128 + 8 * nb + q2b : bias + ch;
                    float2 bf, bg;
                    if constexpr (!FRAMES) {
                        bf = __ldg(reinterpret_cast<const float2*>(bq));
                        bg = __ldg(reinterpret_cast<const float2*>(bq + CH));
                    }
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        const int row = r0 + 8 * r, t = tf + row;
                        if constexpr (FRAMES) {
                            bf = __ldg(reinterpret_cast<const float2*>(fr[r] + 8 * nb));
                            bg = __ldg(reinterpret_cast<const float2*>(fr[r] + 8 * nb + CH));
                        }
                        const float f0 = tanh_fast(acc[0][4 * nb + 2 * r] + bf.x), f1 = tanh_fast(acc[0][4 * nb + 2 * r + 1] + bf.y);
                        const float g0 = sigmoid_fast(acc[1][4 * nb + 2 * r] + bg.x), g1 = sigmoid_fast(acc[1][4 * nb + 2 * r + 1] + bg.y);
                        if (fg_save != nullptr && t < p.L) {
                            float* fs = fg_save + (((size_t)b * (2 * CH / 4) + ch / 4) * p.L + t) * 4 + (ch & 3);
                            *reinterpret_cast<float2*>(fs) = make_float2(f0, f1);
                            *reinterpret_cast<float2*>(fs + (size_t)(CH / 4) * p.L * 4) = make_float2(g0, g1);
                        }
                        unsigned hi, lo;
                        split2(f0 * g0, f1 * g1, hi, lo);
                        unsigned char* zr = zbuf + (ch / 8) * (BM * 16) + row * 16 + q2 * 2;
                        *reinterpret_cast<unsigned*>(zr) = hi;
                        if constexpr (C::PAIR) *reinterpret_cast<unsigned*>(zr + C::ZPLANE) = lo;
                    }
                }
            }
            // the warpgroup's rows of z are complete: make the generic-proxy stores visible to its wgmma reads
            fence_async_smem();
            wg_bar(1 + g, 128);
            // ---------------- pass B tiles: residual h_out = acc + br + h_in -> pair; then skip (+)= acc + bs
            if constexpr (COND) bias = Ld.bias;
            for (int j = 0; j < (need_skip ? C::NT_B : C::NT_R); ++j) {
                for (int s8 = 0; s8 < C::SLABS_B; ++s8) {
                    const unsigned s = wait_stage();
                    slab_mma<C>(acc, s32(zbuf) + a_off + (unsigned)s8 * C::KC * LBO, C::ZPLANE, s32(ring + s * STAGE) + SLOT, s8 == 0);
                    mbar_arrive(empty + s);
                }
                if (j < C::NT_R) {
                    const unsigned* hin = reinterpret_cast<const unsigned*>(Ld.h_in + (size_t)b * 2 * plane_stride);
                    unsigned* hout = reinterpret_cast<unsigned*>(Ld.h_out + (size_t)b * 2 * plane_stride);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int nb = 0; nb < 16; ++nb) {
                            const int ch = j * 256 + 128 * h + 8 * nb + q2;        // first of this thread's two residual channels
                            const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + 2 * CH + ch));
#pragma unroll
                            for (int r = 0; r < 2; ++r) {
                                const int t = tf + r0 + 8 * r;
                                if (t >= p.L) continue;
                                const size_t w = ((size_t)(ch / 8) * p.L + t) * 4 + (q2 >> 1);    // 32-bit word of the hi plane
                                // plain (coherent) loads: in the whole-stack launch h_in was written by other CTAs of this kernel
                                const float2 xh = unpack_bf16x2(hin[w]), xl = unpack_bf16x2(hin[w + plane_stride * 4]);
                                unsigned hi, lo;
                                split2(acc[h][4 * nb + 2 * r] + bb.x + (xh.x + xl.x), acc[h][4 * nb + 2 * r + 1] + bb.y + (xh.y + xl.y), hi, lo);
                                hout[w] = hi;
                                hout[w + plane_stride * 4] = lo;
                            }
                        }
                } else {
#pragma unroll
                    for (int h = 0; h < 2; ++h)
#pragma unroll
                        for (int nb = 0; nb < 16; ++nb) {
                            const int ch = (j - C::NT_R) * 256 + 128 * h + 8 * nb + q2;   // first of this thread's two skip channels
                            const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + 3 * CH + ch));
#pragma unroll
                            for (int r = 0; r < 2; ++r) {
                                const int t = tf + r0 + 8 * r;
                                if (t >= p.L || t < p.skip_start) continue;
                                float* sk = reinterpret_cast<float*>(p.skip) + (((size_t)b * (CH / 4) + ch / 4) * Tsk + (t - p.skip_start)) * 4 + (ch & 3);
                                float2 x = make_float2(0.f, 0.f);
                                if (!skip_init) x = *reinterpret_cast<const float2*>(sk);
                                *reinterpret_cast<float2*>(sk) = make_float2(acc[h][4 * nb + 2 * r] + bb.x + x.x, acc[h][4 * nb + 2 * r + 1] + bb.y + x.y);
                            }
                        }
                }
            }
            if (MULTI) {
                // this warp's stores of h_out / skip are done: publish (release at gpu scope); the 16th arrival completes the item
                __threadfence();
                __syncwarp();
                if (lane == 0) {
                    const unsigned old = atomicAdd(p.item_done + n, 1u);
                    if (old == 2 * EPI_WARPS - 1) { __threadfence(); atomicAdd(p.layer_done + l, 1u); }
                }
            }
        }
    }
}

template <typename C, bool MULTI, bool COND, bool FRAMES>
__global__ void __launch_bounds__(NTHREADS, 1)
block_fused_kernel(const __grid_constant__ LayerDesc single, const __grid_constant__ CUtensorMap mapW, const BlockParams p) {
    block_fused_body<C, MULTI, COND, FRAMES, false>(single, mapW, p, nullptr);
}
template <typename C, bool MULTI, bool COND>
__global__ void __launch_bounds__(NTHREADS, 1)
block_fused_local_kernel(const __grid_constant__ LayerDesc single, const __grid_constant__ CUtensorMap mapW, const BlockParams p,
                         const __grid_constant__ KslabParams kslab) {
    block_fused_body<C, MULTI, COND, false, true>(single, mapW, p, &kslab);
}

// ---------------------------------------------------------------------------------------------- weight packing
// Packed image of one layer (bf16): pass A blocks [n-tile j][k-slab sl][half r], pass B blocks [j][s][r]; a block is the 16 KB
// slot image [plane][chunk KC][row 128][8].  Pass A: N row n = r*128 + row is filter (r = 0) or gate (r = 1) channel 128j + row;
// K index sl*KS + ck*8 + e = tap*CH + input channel (tap 0 = weight[:, :, 0], the older frame).  Pass B: tiles j < NT_R are
// residual rows, the rest skip rows, output channel 256*(j mod NT_R) + r*128 + row; K = dilation channel.
// All layers in one launch: ptrs[layer] = {wf, wg, bf, bg, wr, ws, br, bs} (biases may be null); blockIdx.y = layer.
template <typename C>
__global__ void pack_block_all_kernel(const float* const* __restrict__ ptrs, __nv_bfloat16* __restrict__ out_all, float* __restrict__ bias_all) {
    constexpr int CH = C::CH;
    const float* const* q = ptrs + (size_t)blockIdx.y * 8;
    const float* wf = q[0]; const float* wg = q[1]; const float* wr = q[4]; const float* ws = q[5];
    __nv_bfloat16* out = out_all + (size_t)blockIdx.y * (C::W_LAYER_BYTES / 2);
    constexpr int n_a = C::NT_A * C::SLABS_A * 2, n_blocks = n_a + C::NT_B * C::SLABS_B * 2;
    constexpr int per_plane = SLOT / 2 / C::PLANES;                        // bf16 elements of one plane of a slot image
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)n_blocks * per_plane;
         i += (long long)gridDim.x * blockDim.x) {
        const int blk = (int)(i / per_plane), w = (int)(i % per_plane);   // w: element index inside one plane of the block
        const int ck = w / (BM * 8), row = (w / 8) % BM, e = w % 8;
        float v;
        if (blk < n_a) {
            const int j = blk / (C::SLABS_A * 2), sl = (blk / 2) % C::SLABS_A, r = blk % 2;
            const int kk = sl * C::KS + ck * 8 + e, tap = kk / CH, cin = kk % CH, cout = j * 128 + row;
            v = (r == 0 ? wf : wg)[((size_t)cout * CH + cin) * 2 + tap];
        } else {
            const int bb = blk - n_a, j = bb / (C::SLABS_B * 2), s8 = (bb / 2) % C::SLABS_B, r = bb % 2;
            const int cin = s8 * C::KS + ck * 8 + e, cout = (j % C::NT_R) * 256 + r * 128 + row;
            v = (j < C::NT_R ? wr : ws)[(size_t)cout * CH + cin];
        }
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        __nv_bfloat16* o = out + (size_t)blk * (SLOT / 2) + w;
        o[0] = h;
        if constexpr (C::PAIR) o[per_plane] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
    if (blockIdx.x == 0)
        for (int i = threadIdx.x; i < 4 * CH; i += blockDim.x) {
            const float* src = i < CH ? q[2] : (i < 2 * CH ? q[3] : (i < 3 * CH ? q[6] : q[7]));
            bias_all[(size_t)blockIdx.y * 4 * CH + i] = src ? src[i % CH] : 0.f;
        }
}

// Packed [Uf; Ug] image of the audio-rate local conditioning (KslabParams::mapU), same tiling as the pass-A blocks above: blocks
// [n-tile j][k-slab sl < Cpad / KS][half r], N row r*128 + row = filter (r = 0) / gate (r = 1) channel 128j + row, K index
// sl*KS + ck*8 + e = condition channel (zero from C up to Cpad).  ptrs[layer] = {Uf, Ug}, each (CH, C, 1); blockIdx.y = layer.
template <typename C>
__global__ void pack_local_all_kernel(const float* const* __restrict__ ptrs, int Cc, int n_slabs, __nv_bfloat16* __restrict__ out_all) {
    const float* uf = ptrs[(size_t)blockIdx.y * 2];
    const float* ug = ptrs[(size_t)blockIdx.y * 2 + 1];
    const int n_blocks = C::NT_A * n_slabs * 2;
    __nv_bfloat16* out = out_all + (size_t)blockIdx.y * n_blocks * (SLOT / 2);
    constexpr int per_plane = SLOT / 2 / C::PLANES;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (long long)n_blocks * per_plane;
         i += (long long)gridDim.x * blockDim.x) {
        const int blk = (int)(i / per_plane), w = (int)(i % per_plane);
        const int ck = w / (BM * 8), row = (w / 8) % BM, e = w % 8;
        const int j = blk / (n_slabs * 2), sl = (blk / 2) % n_slabs, r = blk % 2;
        const int k = sl * C::KS + ck * 8 + e, cout = j * 128 + row;
        const float v = k < Cc ? (r == 0 ? uf : ug)[(size_t)cout * Cc + k] : 0.f;
        const __nv_bfloat16 h = __float2bfloat16_rn(v);
        __nv_bfloat16* o = out + (size_t)blk * (SLOT / 2) + w;
        o[0] = h;
        if constexpr (C::PAIR) o[per_plane] = __float2bfloat16_rn(v - __bfloat162float(h));
    }
}

// ---------------------------------------------------------------------------------------------- layout converters
// channel-major fp32 (B, C, L) -> chunked pair (B, 2, Cpad/8, L, 8), channels [C, Cpad) zero
__global__ void pair_from_channels_kernel(const float* __restrict__ x, uint4* __restrict__ out, int B, int C, int L, int c_pad) {
    const int chunks = c_pad / 8;
    const long long total = (long long)B * chunks * L;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % L), ck = (int)((i / L) % chunks), b = (int)(i / ((long long)L * chunks));
        float v[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int c = ck * 8 + e;
            v[e] = c < C ? x[((size_t)b * C + c) * L + t] : 0.f;
        }
        unsigned hi[4], lo[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) split2(v[2 * k], v[2 * k + 1], hi[k], lo[k]);
        uint4* o = out + ((size_t)b * 2 * chunks + ck) * L + t;
        o[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        o[(size_t)chunks * L] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
}
// fp32 frames (B, L, C) -> chunked pair (B, 2, C/8, L, 8) for frames [t_begin, L)
__global__ void pair_from_frames_kernel(const float* __restrict__ x, uint4* __restrict__ out, int B, int L, int C, int t_begin) {
    const int chunks = C / 8;
    const long long total = (long long)B * chunks * (L - t_begin);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int t = t_begin + (int)(i % (L - t_begin)), ck = (int)((i / (L - t_begin)) % chunks), b = (int)(i / ((long long)(L - t_begin) * chunks));
        const float4* s = reinterpret_cast<const float4*>(x + ((size_t)b * L + t) * C + ck * 8);
        const float4 a = s[0], c = s[1];
        unsigned hi[4], lo[4];
        split2(a.x, a.y, hi[0], lo[0]); split2(a.z, a.w, hi[1], lo[1]); split2(c.x, c.y, hi[2], lo[2]); split2(c.z, c.w, hi[3], lo[3]);
        uint4* o = out + ((size_t)b * 2 * chunks + ck) * L + t;
        o[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        o[(size_t)chunks * L] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
    }
}
// chunked pair -> fp32 frames (hi + lo) for frames [t_begin, L)
__global__ void frames_from_pair_kernel(const uint4* __restrict__ in, float* __restrict__ x, int B, int L, int C, int t_begin) {
    const int chunks = C / 8;
    const long long total = (long long)B * chunks * (L - t_begin);
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ck = (int)(i % chunks), t = t_begin + (int)((i / chunks) % (L - t_begin)), b = (int)(i / ((long long)(L - t_begin) * chunks));
        const uint4* s = in + ((size_t)b * 2 * chunks + ck) * L + t;
        const uint4 h = s[0], l = s[(size_t)chunks * L];
        const unsigned hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
        float o[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 a = unpack_bf16x2(hw[k]), c = unpack_bf16x2(lw[k]);
            o[2 * k] = a.x + c.x; o[2 * k + 1] = a.y + c.y;
        }
        float4* d = reinterpret_cast<float4*>(x + ((size_t)b * L + t) * C + ck * 8);
        d[0] = make_float4(o[0], o[1], o[2], o[3]);
        d[1] = make_float4(o[4], o[5], o[6], o[7]);
    }
}
// chunked fp32 (B, C/4, T, 4) <-> frames (B, T, C) for frames [t_first, t_first + n) of the chunked tensor
__global__ void frames_from_chunks4_kernel(const float4* __restrict__ in, float* __restrict__ x, int B, int T, int C, int t_first, int n) {
    const int chunks = C / 4;
    const long long total = (long long)B * chunks * n;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int ck = (int)(i % chunks), tt = (int)((i / chunks) % n), b = (int)(i / ((long long)n * chunks));
        reinterpret_cast<float4*>(x + ((size_t)b * n + tt) * C)[ck] = in[((size_t)b * chunks + ck) * T + t_first + tt];
    }
}
// start conv on class indices (reference wavenet_model.py:65-68,127 on one-hot input == a gather of one weight column):
// h0 pair <- table[idx[b][t]] where table (classes, ldt) holds start_conv.weight^T (+ bias) as packed by wn_pack_1x1_weights
template <typename IDX>
__global__ void start_pair_kernel(const IDX* __restrict__ idx, const float* __restrict__ table, const float* __restrict__ bias,
                                  uint4* __restrict__ out, int B, int L, int classes, int ldt, int R, int* __restrict__ err) {
    const int chunks = R / 8;
    const long long total = (long long)B * chunks * L;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i % L), ck = (int)((i / L) % chunks), b = (int)(i / ((long long)L * chunks));
        long long cls = (long long)idx[(size_t)b * L + t];
        if (cls < 0 || cls >= classes) { if (err) atomicExch(err, 1); cls = cls < 0 ? 0 : classes - 1; }
        const float4* s = reinterpret_cast<const float4*>(table + (size_t)cls * ldt + ck * 8);
        const float4* bb = reinterpret_cast<const float4*>(bias + ck * 8);
        const float4 a = __ldg(s), c = __ldg(s + 1), ba = __ldg(bb), bc = __ldg(bb + 1);
        unsigned hi[4], lo[4];
        split2(a.x + ba.x, a.y + ba.y, hi[0], lo[0]); split2(a.z + ba.z, a.w + ba.w, hi[1], lo[1]);
        split2(c.x + bc.x, c.y + bc.y, hi[2], lo[2]); split2(c.z + bc.z, c.w + bc.w, hi[3], lo[3]);
        uint4* o = out + ((size_t)b * 2 * chunks + ck) * L + t;
        o[0] = make_uint4(hi[0], hi[1], hi[2], hi[3]);
        o[(size_t)chunks * L] = make_uint4(lo[0], lo[1], lo[2], lo[3]);
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
// chunked pair tensor (B, 2, C/8, L, 8) bf16 as 8-byte elements: dims {2(L - origin), C/8, 2, B}; box {2 box_frames, box_chunks,
// box_planes, 1} (box_planes = 1: the hi plane only, for single-pass bf16 operands).  Frames left of `origin` (and right of L)
// are out of bounds -> zeros.
int make_pair_map(CUtensorMap* m, const void* base, int B, int L, int C, int origin, int box_frames, int box_chunks, int box_planes) {
    EncodeTiledFn fn = encode_fn();
    WN_REQUIRE(fn, WN_E_UNSUPP, "cuTensorMapEncodeTiled is not available from this driver");
    WN_REQUIRE(L - origin >= 1, WN_E_BADARG, "empty activation range");
    const cuuint64_t chunks = (cuuint64_t)(C / 8);
    cuuint64_t dims[4] = {(cuuint64_t)2 * (L - origin), chunks, 2, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)L * 16, chunks * L * 16, 2 * chunks * L * 16};
    cuuint32_t box[4] = {(cuuint32_t)(2 * box_frames), (cuuint32_t)box_chunks, (cuuint32_t)box_planes, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 4, (void*)((const unsigned char*)base + (size_t)origin * 16), dims, strides, box,
                    estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    WN_REQUIRE(r == CUDA_SUCCESS, WN_E_UNSUPP, "cuTensorMapEncodeTiled(pair activations) failed with %d", (int)r);
    return 0;
}
// packed weights: rows of 2 KB (256 8-byte elements); box = 8 rows = one 16 KB slot image
int make_wrows_map(CUtensorMap* m, const void* base, long long rows) {
    EncodeTiledFn fn = encode_fn();
    WN_REQUIRE(fn, WN_E_UNSUPP, "cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[2] = {256, (cuuint64_t)rows};
    cuuint64_t strides[1] = {2048};
    cuuint32_t box[2] = {256, 8};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, (void*)base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                    CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    WN_REQUIRE(r == CUDA_SUCCESS, WN_E_UNSUPP, "cuTensorMapEncodeTiled(packed weights) failed with %d", (int)r);
    return 0;
}

}  // namespace tb
}  // namespace wn

using namespace wn;

extern "C" int wn_tb_supported(int R, int D, int S, int k) { return R == D && D == S && (R == 256 || R == 512) && k == 2; }
// precision: WN_PREC_BF16_PAIRS (fp32-class, channels == 256 only: the z image of 512 channels does not fit as a pair) or
// WN_PREC_BF16 (single-pass bf16 operands, 256 or 512 channels)
extern "C" int wn_tb_precision_supported(int channels, int precision) {
    return (precision == WN_PREC_BF16_PAIRS && channels == 256) || (precision == WN_PREC_BF16 && (channels == 256 || channels == 512));
}
extern "C" size_t wn_tb_weight_bytes_per_layer(int channels, int precision) {
    if (!wn_tb_precision_supported(channels, precision)) return 0;
    if (precision == WN_PREC_BF16_PAIRS) return tb::Cfg<256, true>::W_LAYER_BYTES;
    return channels == 256 ? tb::Cfg<256, false>::W_LAYER_BYTES : tb::Cfg<512, false>::W_LAYER_BYTES;
}

extern "C" int wn_tb_pack_all_weights(const float* const* d_ptrs, int n_layers, int channels, int precision, void* d_w_all,
                                      float* d_bias_all, void* stream) {
    WN_REQUIRE(d_ptrs && d_w_all && d_bias_all && n_layers > 0, WN_E_BADARG, "wn_tb_pack_all_weights: bad arguments");
    WN_REQUIRE(wn_tb_precision_supported(channels, precision), WN_E_UNSUPP, "wn_tb_pack_all_weights: %d channels with precision %d is not supported",
               channels, precision);
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid(74, n_layers);
    if (precision == WN_PREC_BF16_PAIRS) tb::pack_block_all_kernel<tb::Cfg<256, true>><<<grid, 256, 0, st>>>(d_ptrs, (__nv_bfloat16*)d_w_all, d_bias_all);
    else if (channels == 256) tb::pack_block_all_kernel<tb::Cfg<256, false>><<<grid, 256, 0, st>>>(d_ptrs, (__nv_bfloat16*)d_w_all, d_bias_all);
    else tb::pack_block_all_kernel<tb::Cfg<512, false>><<<grid, 256, 0, st>>>(d_ptrs, (__nv_bfloat16*)d_w_all, d_bias_all);
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_pair_from_frames(const float* d_frames, void* d_pair, int B, int L, int C, int t_begin, void* stream) {
    WN_REQUIRE(d_frames && d_pair && B > 0 && L > 0 && C > 0 && C % 8 == 0 && t_begin >= 0 && t_begin < L, WN_E_BADARG,
               "wn_pair_from_frames: bad arguments");
    tb::pair_from_frames_kernel<<<1184, 256, 0, (cudaStream_t)stream>>>(d_frames, (uint4*)d_pair, B, L, C, t_begin);
    WN_CUDA(cudaGetLastError());
    return 0;
}
extern "C" int wn_frames_from_pair(const void* d_pair, float* d_frames, int B, int L, int C, int t_begin, void* stream) {
    WN_REQUIRE(d_frames && d_pair && B > 0 && L > 0 && C > 0 && C % 8 == 0 && t_begin >= 0 && t_begin < L, WN_E_BADARG,
               "wn_frames_from_pair: bad arguments");
    tb::frames_from_pair_kernel<<<1184, 256, 0, (cudaStream_t)stream>>>((const uint4*)d_pair, d_frames, B, L, C, t_begin);
    WN_CUDA(cudaGetLastError());
    return 0;
}
extern "C" int wn_frames_from_chunks4(const float* d_chunked, float* d_frames, int B, int T, int C, int t_first, int n, void* stream) {
    WN_REQUIRE(d_chunked && d_frames && B > 0 && T > 0 && C > 0 && C % 4 == 0 && t_first >= 0 && n >= 1 && t_first + n <= T, WN_E_BADARG,
               "wn_frames_from_chunks4: bad arguments");
    tb::frames_from_chunks4_kernel<<<1184, 256, 0, (cudaStream_t)stream>>>((const float4*)d_chunked, d_frames, B, T, C, t_first, n);
    WN_CUDA(cudaGetLastError());
    return 0;
}

static int start_pair(const void* d_idx, bool u8, const float* d_w_t, const float* d_b_p, void* d_h_pair, int B, int classes, int L,
                      int R, int* d_err, void* stream) {
    WN_REQUIRE(d_idx && d_w_t && d_b_p && d_h_pair && B > 0 && L > 0 && classes > 0, WN_E_BADARG, "wn_tb_start_index: bad arguments");
    WN_REQUIRE(R > 0 && R % 8 == 0, WN_E_UNSUPP, "wn_tb_start_index: R must be a multiple of 8");
    const int ldt = wn_n2p(R);
    cudaStream_t st = (cudaStream_t)stream;
    if (u8) tb::start_pair_kernel<uint8_t><<<1184, 256, 0, st>>>((const uint8_t*)d_idx, d_w_t, d_b_p, (uint4*)d_h_pair, B, L, classes, ldt, R, d_err);
    else tb::start_pair_kernel<long long><<<1184, 256, 0, st>>>((const long long*)d_idx, d_w_t, d_b_p, (uint4*)d_h_pair, B, L, classes, ldt, R, d_err);
    WN_CUDA(cudaGetLastError());
    return 0;
}
extern "C" int wn_tb_start_index_u8(const uint8_t* d_idx, const float* d_w_t, const float* d_b_p, void* d_h_pair, int B, int classes,
                                    int L, int R, int* d_err, void* stream) {
    return start_pair(d_idx, true, d_w_t, d_b_p, d_h_pair, B, classes, L, R, d_err, stream);
}
extern "C" int wn_tb_start_index_i64(const int64_t* d_idx, const float* d_w_t, const float* d_b_p, void* d_h_pair, int B, int classes,
                                     int L, int R, int* d_err, void* stream) {
    return start_pair(d_idx, false, d_w_t, d_b_p, d_h_pair, B, classes, L, R, d_err, stream);
}

static int launch_cfg(cudaLaunchConfig_t& cfg, int grid, size_t smem, cudaStream_t st) {
    cfg = cudaLaunchConfig_t{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(tb::NTHREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    return 0;
}

// the fused block kernel of an instantiation; a KslabParams argument selects the K-slab (audio-rate local conditioning) kernel
template <typename C, bool MULTI, bool COND, bool FRAMES, typename... KS>
static auto kernel_of() {
    if constexpr (sizeof...(KS) > 0) return tb::block_fused_local_kernel<C, MULTI, COND>;
    else return tb::block_fused_kernel<C, MULTI, COND, FRAMES>;
}

template <typename C>
static int fill_layer(tb::LayerDesc& d, const void* h_in, void* h_out, const float* bias4, float* fg_save, int layer, int B, int L,
                      int dilation, int in_start, int out_start, int skip_init, int item_base, const float* cond,
                      int cond_frames = 0, int cond_hop = 0) {
    memset(&d, 0, sizeof(d));
    if (int rc = tb::make_pair_map(&d.mapH, h_in, B, L, C::CH, in_start, tb::BM, C::KC, C::PLANES)) return rc;
    d.t_begin = out_start; d.in_start = in_start; d.dil = dilation; d.skip_init = skip_init;
    d.tiles_per_seq = (L - out_start + tb::PM - 1) / tb::PM;
    d.n_items = B * d.tiles_per_seq;
    d.item_base = item_base;
    d.w_row0 = layer * C::WROWS_LAYER;
    d.bias = bias4; d.h_in = (const uint4*)h_in; d.h_out = (uint4*)h_out; d.fg_save = (float4*)fg_save;
    d.war_layer = -1;
    d.cond = cond;
    d.cond_frames = cond_frames; d.cond_hop = cond_hop;
    return 0;
}

template <typename C, bool COND, bool FRAMES, typename... KS>
static int launch_block(const wn_tb_block_args* a, const float* cond, int n_frames, int hop, cudaStream_t st, const KS&... ks) {
    int dev = 0, sms = 0;
    WN_CUDA(cudaGetDevice(&dev));
    WN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    tb::LayerDesc d;
    CUtensorMap mW;
    if (int rc = fill_layer<C>(d, a->d_h_in, a->d_h_out, a->d_bias4, a->d_fg_save, a->layer, a->B, a->L, a->dilation, a->in_start,
                               a->out_start, a->skip_init, 0, cond, n_frames, hop)) return rc;
    if (int rc = tb::make_wrows_map(&mW, a->d_w_all, (long long)a->n_layers * C::WROWS_LAYER)) return rc;
    tb::BlockParams p;
    memset(&p, 0, sizeof(p));
    p.B = a->B; p.L = a->L; p.skip_start = a->skip_start; p.n_layers = 1; p.total_items = d.n_items;
    p.skip = (float4*)a->d_skip;
    const auto kern = kernel_of<C, false, COND, FRAMES, KS...>();
    WN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    int grid = 2 * p.total_items;
    const int max_grid = (sms / 2) * 2;
    if (grid > max_grid) grid = max_grid;
    cudaLaunchConfig_t cfg;
    launch_cfg(cfg, grid, C::SMEM_BYTES, st);
    WN_CUDA(cudaLaunchKernelEx(&cfg, kern, d, mW, p, ks...));
    WN_CUDA(cudaGetLastError());
    return 0;
}

template <typename C>
static int launch_block_c(const wn_tb_block_args* a, const float* cond, int n_frames, int hop, cudaStream_t st) {
    if (cond && hop > 0) return launch_block<C, true, true>(a, cond, n_frames, hop, st);
    return cond ? launch_block<C, true, false>(a, cond, 0, 0, st) : launch_block<C, false, false>(a, nullptr, 0, 0, st);
}

extern "C" int wn_tb_block_fwd(const wn_tb_block_args* a, void* stream) { return wn_tb_block_fwd_cond(a, nullptr, stream); }

static int tb_block_fwd_impl(const wn_tb_block_args* a, const float* d_cond, int n_frames, int hop, void* stream);

extern "C" int wn_tb_block_fwd_cond(const wn_tb_block_args* a, const float* d_cond, void* stream) {
    return tb_block_fwd_impl(a, d_cond, 0, 0, stream);
}

extern "C" int wn_tb_block_fwd_cond_frames(const wn_tb_block_args* a, const float* d_cond, int n_frames, int hop, void* stream) {
    WN_REQUIRE(a && d_cond, WN_E_BADARG, "wn_tb_block_fwd_cond_frames: null pointer");
    WN_REQUIRE(hop >= 1 && a->L > 0 && n_frames >= ceil_div(a->L, hop), WN_E_BADARG,
               "wn_tb_block_fwd_cond_frames: %d frames of hop %d do not cover %d positions", n_frames, hop, a->L);
    return tb_block_fwd_impl(a, d_cond, n_frames, hop, stream);
}

static int tb_block_fwd_impl(const wn_tb_block_args* a, const float* d_cond, int n_frames, int hop, void* stream) {
    WN_REQUIRE(a, WN_E_BADARG, "wn_tb_block_fwd: null args");
    WN_REQUIRE(a->d_h_in && a->d_h_out && a->d_skip && a->d_w_all && a->d_bias4, WN_E_BADARG, "wn_tb_block_fwd: null pointer");
    WN_REQUIRE(wn_tb_precision_supported(a->channels, a->precision), WN_E_UNSUPP, "wn_tb_block_fwd: %d channels with precision %d is not supported",
               a->channels, a->precision);
    WN_REQUIRE(a->B > 0 && a->L > 0 && a->dilation >= 1 && a->in_start >= 0 && a->out_start >= a->in_start && a->out_start < a->L &&
                   a->skip_start >= a->out_start && a->skip_start < a->L && a->layer >= 0 && a->layer < a->n_layers,
               WN_E_BADARG, "wn_tb_block_fwd: bad frame ranges or layer index");
    WN_REQUIRE(((uintptr_t)a->d_h_in | (uintptr_t)a->d_h_out | (uintptr_t)a->d_skip | (uintptr_t)a->d_w_all | (uintptr_t)d_cond) % 16 == 0,
               WN_E_BADARG, "wn_tb_block_fwd: buffers must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    if (a->precision == WN_PREC_BF16_PAIRS) return launch_block_c<tb::Cfg<256, true>>(a, d_cond, n_frames, hop, st);
    if (a->channels == 256) return launch_block_c<tb::Cfg<256, false>>(a, d_cond, n_frames, hop, st);
    return launch_block_c<tb::Cfg<512, false>>(a, d_cond, n_frames, hop, st);
}

// ---------------------------------------------------------------------------------------------- the whole stack in one launch
extern "C" size_t wn_tb_stack_desc_bytes(void) { return sizeof(tb::LayerDesc); }
extern "C" long long wn_tb_stack_items(int n_layers, int B, int L, const int* out_start) {
    long long n = 0;
    for (int i = 0; i < n_layers; ++i) n += (long long)B * ((L - out_start[i] + tb::PM - 1) / tb::PM);
    return n;
}

template <typename C, bool COND, bool FRAMES, typename... KS>
static int launch_stack(const wn_tb_stack_args* a, const float* cond, int n_frames, int hop, cudaStream_t st, const KS&... ks) {
    int dev = 0, sms = 0;
    WN_CUDA(cudaGetDevice(&dev));
    WN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int nl = a->n_layers;
    std::vector<tb::LayerDesc> desc((size_t)nl);
    int base = 0;
    for (int i = 0; i < nl; ++i) {
        float* fg = a->d_fg_all ? a->d_fg_all + (size_t)i * a->B * (2 * C::CH) * a->L : nullptr;
        if (int rc = fill_layer<C>(desc[i], a->h_ptrs[i], const_cast<void*>(a->h_ptrs[i + 1]), a->d_bias_all + (size_t)i * 4 * C::CH, fg, i, a->B, a->L,
                                   a->dilations[i], a->in_start[i], a->out_start[i], i == 0, base,
                                   COND ? cond + (size_t)i * a->B * (FRAMES ? n_frames : 1) * 2 * C::CH : nullptr,
                                   n_frames, hop)) return rc;
        WN_REQUIRE(a->in_start[i] >= 0 && a->out_start[i] >= a->in_start[i] && a->out_start[i] < a->L && a->skip_start >= a->out_start[i],
                   WN_E_BADARG, "wn_tb_stack_fwd: bad frame ranges of layer %d", i);
        WN_REQUIRE(a->h_ptrs[i] && a->h_ptrs[i + 1] && a->h_ptrs[i] != a->h_ptrs[i + 1] && (uintptr_t)a->h_ptrs[i + 1] % 16 == 0,
                   WN_E_BADARG, "wn_tb_stack_fwd: layer %d needs distinct 16-byte aligned input and output buffers", i);
        WN_REQUIRE(i == 0 || a->h_ptrs[i + 1] != a->h_ptrs[i - 1], WN_E_BADARG,
                   "wn_tb_stack_fwd: layer %d may not write the buffer layer %d is reading (rotate three buffers)", i, i - 1);
        // write-after-read: the latest earlier layer that READS the buffer this layer writes must be complete first
        for (int j = i - 2; j >= 0; --j)
            if (a->h_ptrs[j] == a->h_ptrs[i + 1]) { desc[i].war_layer = j; break; }
        base += desc[i].n_items;
    }
    CUtensorMap mW;
    if (int rc = tb::make_wrows_map(&mW, a->d_w_all, (long long)nl * C::WROWS_LAYER)) return rc;
    WN_CUDA(cudaMemcpyAsync(a->d_desc, desc.data(), sizeof(tb::LayerDesc) * nl, cudaMemcpyHostToDevice, st));
    WN_CUDA(cudaMemsetAsync(a->d_flags, 0, sizeof(unsigned) * ((size_t)base + nl), st));
    tb::BlockParams p;
    memset(&p, 0, sizeof(p));
    p.B = a->B; p.L = a->L; p.skip_start = a->skip_start; p.n_layers = nl; p.total_items = base;
    p.skip = (float4*)a->d_skip;
    p.layers = (const tb::LayerDesc*)a->d_desc;
    p.item_done = a->d_flags; p.layer_done = a->d_flags + base;
    const auto kern = kernel_of<C, true, COND, FRAMES, KS...>();
    WN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    // every CTA must be resident (items wait for items of other CTAs): one CTA per SM, at most sms/2 pairs
    int grid = 2 * base;
    const int max_grid = (sms / 2) * 2;
    if (grid > max_grid) grid = max_grid;
    cudaLaunchConfig_t cfg;
    launch_cfg(cfg, grid, C::SMEM_BYTES, st);
    WN_CUDA(cudaLaunchKernelEx(&cfg, kern, desc[0], mW, p, ks...));
    WN_CUDA(cudaGetLastError());
    return 0;
}

template <typename C>
static int launch_stack_c(const wn_tb_stack_args* a, const float* cond, int n_frames, int hop, cudaStream_t st) {
    if (cond && hop > 0) return launch_stack<C, true, true>(a, cond, n_frames, hop, st);
    return cond ? launch_stack<C, true, false>(a, cond, 0, 0, st) : launch_stack<C, false, false>(a, nullptr, 0, 0, st);
}

extern "C" int wn_tb_stack_fwd(const wn_tb_stack_args* a, void* stream) { return wn_tb_stack_fwd_cond(a, nullptr, stream); }

static int tb_stack_fwd_impl(const wn_tb_stack_args* a, const float* d_cond, int n_frames, int hop, void* stream);

extern "C" int wn_tb_stack_fwd_cond(const wn_tb_stack_args* a, const float* d_cond, void* stream) {
    return tb_stack_fwd_impl(a, d_cond, 0, 0, stream);
}

extern "C" int wn_tb_stack_fwd_cond_frames(const wn_tb_stack_args* a, const float* d_cond, int n_frames, int hop, void* stream) {
    WN_REQUIRE(a && d_cond, WN_E_BADARG, "wn_tb_stack_fwd_cond_frames: null pointer");
    WN_REQUIRE(hop >= 1 && a->L > 0 && n_frames >= ceil_div(a->L, hop), WN_E_BADARG,
               "wn_tb_stack_fwd_cond_frames: %d frames of hop %d do not cover %d positions", n_frames, hop, a->L);
    return tb_stack_fwd_impl(a, d_cond, n_frames, hop, stream);
}

static int tb_stack_fwd_impl(const wn_tb_stack_args* a, const float* d_cond, int n_frames, int hop, void* stream) {
    WN_REQUIRE(a, WN_E_BADARG, "wn_tb_stack_fwd: null args");
    WN_REQUIRE(a->h_ptrs && a->d_skip && a->d_w_all && a->d_bias_all && a->d_desc && a->d_flags && a->dilations && a->in_start && a->out_start,
               WN_E_BADARG, "wn_tb_stack_fwd: null pointer");
    WN_REQUIRE(wn_tb_precision_supported(a->channels, a->precision), WN_E_UNSUPP, "wn_tb_stack_fwd: %d channels with precision %d is not supported",
               a->channels, a->precision);
    WN_REQUIRE(a->B > 0 && a->L > 0 && a->n_layers > 0 && a->skip_start >= 0 && a->skip_start < a->L && (uintptr_t)a->d_desc % 128 == 0,
               WN_E_BADARG, "wn_tb_stack_fwd: bad sizes (d_desc must be 128-byte aligned)");
    WN_REQUIRE((uintptr_t)d_cond % 16 == 0, WN_E_BADARG, "wn_tb_stack_fwd: the condition table must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    if (a->precision == WN_PREC_BF16_PAIRS) return launch_stack_c<tb::Cfg<256, true>>(a, d_cond, n_frames, hop, st);
    if (a->channels == 256) return launch_stack_c<tb::Cfg<256, false>>(a, d_cond, n_frames, hop, st);
    return launch_stack_c<tb::Cfg<512, false>>(a, d_cond, n_frames, hop, st);
}

// ---------------------------------------------------------------------------------------------- audio-rate local conditioning
// The learned upsampler's output c (B, C, L) enters pass A as K-slabs (block_fused_kernel with a KslabParams): c is converted
// once per forward to a chunked pair tensor of Cpad channels, and every layer's [Uf; Ug] is packed into its own slab image.
template <typename C>
static int local_slabs(int Cc) { return ceil_div(Cc, C::KS); }
static int local_slab_width(int precision) { return precision == WN_PREC_BF16_PAIRS ? tb::Cfg<256, true>::KS : tb::Cfg<256, false>::KS; }

extern "C" int wn_tb_local_padded_channels(int C, int precision) {
    if (C < 1 || (precision != WN_PREC_BF16_PAIRS && precision != WN_PREC_BF16)) return 0;
    return ceil_div(C, local_slab_width(precision)) * local_slab_width(precision);
}
extern "C" size_t wn_tb_local_weight_bytes_per_layer(int C, int channels, int precision) {
    if (!wn_tb_precision_supported(channels, precision) || C < 1) return 0;
    return (size_t)(2 * channels / 256) * (wn_tb_local_padded_channels(C, precision) / local_slab_width(precision)) * 2 * tb::SLOT;
}

extern "C" int wn_tb_pack_local_weights(const float* const* d_ptrs, int n_layers, int C, int channels, int precision, void* d_u_all,
                                        void* stream) {
    WN_REQUIRE(d_ptrs && d_u_all && n_layers > 0 && C > 0, WN_E_BADARG, "wn_tb_pack_local_weights: bad arguments");
    WN_REQUIRE(wn_tb_precision_supported(channels, precision), WN_E_UNSUPP,
               "wn_tb_pack_local_weights: %d channels with precision %d is not supported", channels, precision);
    cudaStream_t st = (cudaStream_t)stream;
    const dim3 grid(74, n_layers);
    __nv_bfloat16* out = (__nv_bfloat16*)d_u_all;
    if (precision == WN_PREC_BF16_PAIRS) {
        using Cf = tb::Cfg<256, true>;
        tb::pack_local_all_kernel<Cf><<<grid, 256, 0, st>>>(d_ptrs, C, local_slabs<Cf>(C), out);
    } else if (channels == 256) {
        using Cf = tb::Cfg<256, false>;
        tb::pack_local_all_kernel<Cf><<<grid, 256, 0, st>>>(d_ptrs, C, local_slabs<Cf>(C), out);
    } else {
        using Cf = tb::Cfg<512, false>;
        tb::pack_local_all_kernel<Cf><<<grid, 256, 0, st>>>(d_ptrs, C, local_slabs<Cf>(C), out);
    }
    WN_CUDA(cudaGetLastError());
    return 0;
}

extern "C" int wn_tb_local_from_channels(const float* d_c, void* d_c_pair, int B, int C, int L, int precision, void* stream) {
    const int c_pad = wn_tb_local_padded_channels(C, precision);
    WN_REQUIRE(d_c && d_c_pair && B > 0 && C > 0 && L > 0 && c_pad > 0, WN_E_BADARG, "wn_tb_local_from_channels: bad arguments");
    tb::pair_from_channels_kernel<<<1184, 256, 0, (cudaStream_t)stream>>>(d_c, (uint4*)d_c_pair, B, C, L, c_pad);
    WN_CUDA(cudaGetLastError());
    return 0;
}

template <typename C>
static int make_kslab(tb::KslabParams& k, const void* d_c_pair, const void* d_u_all, int B, int L, int Cc, int n_layers) {
    memset(&k, 0, sizeof(k));
    k.n_slabs = local_slabs<C>(Cc);
    if (int rc = tb::make_pair_map(&k.mapC, d_c_pair, B, L, k.n_slabs * C::KS, 0, tb::BM, C::KC, C::PLANES)) return rc;
    return tb::make_wrows_map(&k.mapU, d_u_all, (long long)n_layers * C::NT_A * k.n_slabs * 16);
}

static int check_local(const void* d_c_pair, int C, const void* d_u_all, const char* who) {
    WN_REQUIRE(d_c_pair && d_u_all && C > 0, WN_E_BADARG, "%s: null pointer or no condition channels", who);
    WN_REQUIRE(((uintptr_t)d_c_pair | (uintptr_t)d_u_all) % 16 == 0, WN_E_BADARG, "%s: c and U must be 16-byte aligned", who);
    return 0;
}

template <typename C>
static int launch_block_local(const wn_tb_block_args* a, const float* cond, const void* d_c_pair, int Cc, const void* d_u_all,
                              cudaStream_t st) {
    tb::KslabParams k;
    if (int rc = make_kslab<C>(k, d_c_pair, d_u_all, a->B, a->L, Cc, a->n_layers)) return rc;
    return cond ? launch_block<C, true, false>(a, cond, 0, 0, st, k) : launch_block<C, false, false>(a, nullptr, 0, 0, st, k);
}

extern "C" int wn_tb_block_fwd_local(const wn_tb_block_args* a, const float* d_cond, const void* d_c_pair, int C, const void* d_u_all,
                                     void* stream) {
    if (int rc = check_local(d_c_pair, C, d_u_all, "wn_tb_block_fwd_local")) return rc;
    WN_REQUIRE(a, WN_E_BADARG, "wn_tb_block_fwd: null args");
    WN_REQUIRE(a->d_h_in && a->d_h_out && a->d_skip && a->d_w_all && a->d_bias4, WN_E_BADARG, "wn_tb_block_fwd: null pointer");
    WN_REQUIRE(wn_tb_precision_supported(a->channels, a->precision), WN_E_UNSUPP, "wn_tb_block_fwd: %d channels with precision %d is not supported",
               a->channels, a->precision);
    WN_REQUIRE(a->B > 0 && a->L > 0 && a->dilation >= 1 && a->in_start >= 0 && a->out_start >= a->in_start && a->out_start < a->L &&
                   a->skip_start >= a->out_start && a->skip_start < a->L && a->layer >= 0 && a->layer < a->n_layers,
               WN_E_BADARG, "wn_tb_block_fwd: bad frame ranges or layer index");
    WN_REQUIRE(((uintptr_t)a->d_h_in | (uintptr_t)a->d_h_out | (uintptr_t)a->d_skip | (uintptr_t)a->d_w_all | (uintptr_t)d_cond) % 16 == 0,
               WN_E_BADARG, "wn_tb_block_fwd: buffers must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    if (a->precision == WN_PREC_BF16_PAIRS) return launch_block_local<tb::Cfg<256, true>>(a, d_cond, d_c_pair, C, d_u_all, st);
    if (a->channels == 256) return launch_block_local<tb::Cfg<256, false>>(a, d_cond, d_c_pair, C, d_u_all, st);
    return launch_block_local<tb::Cfg<512, false>>(a, d_cond, d_c_pair, C, d_u_all, st);
}

template <typename C>
static int launch_stack_local(const wn_tb_stack_args* a, const float* cond, const void* d_c_pair, int Cc, const void* d_u_all,
                              cudaStream_t st) {
    tb::KslabParams k;
    if (int rc = make_kslab<C>(k, d_c_pair, d_u_all, a->B, a->L, Cc, a->n_layers)) return rc;
    return cond ? launch_stack<C, true, false>(a, cond, 0, 0, st, k) : launch_stack<C, false, false>(a, nullptr, 0, 0, st, k);
}

extern "C" int wn_tb_stack_fwd_local(const wn_tb_stack_args* a, const float* d_cond, const void* d_c_pair, int C, const void* d_u_all,
                                     void* stream) {
    if (int rc = check_local(d_c_pair, C, d_u_all, "wn_tb_stack_fwd_local")) return rc;
    WN_REQUIRE(a, WN_E_BADARG, "wn_tb_stack_fwd: null args");
    WN_REQUIRE(a->h_ptrs && a->d_skip && a->d_w_all && a->d_bias_all && a->d_desc && a->d_flags && a->dilations && a->in_start && a->out_start,
               WN_E_BADARG, "wn_tb_stack_fwd: null pointer");
    WN_REQUIRE(wn_tb_precision_supported(a->channels, a->precision), WN_E_UNSUPP, "wn_tb_stack_fwd: %d channels with precision %d is not supported",
               a->channels, a->precision);
    WN_REQUIRE(a->B > 0 && a->L > 0 && a->n_layers > 0 && a->skip_start >= 0 && a->skip_start < a->L && (uintptr_t)a->d_desc % 128 == 0,
               WN_E_BADARG, "wn_tb_stack_fwd: bad sizes (d_desc must be 128-byte aligned)");
    WN_REQUIRE((uintptr_t)d_cond % 16 == 0, WN_E_BADARG, "wn_tb_stack_fwd: the condition table must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    if (a->precision == WN_PREC_BF16_PAIRS) return launch_stack_local<tb::Cfg<256, true>>(a, d_cond, d_c_pair, C, d_u_all, st);
    if (a->channels == 256) return launch_stack_local<tb::Cfg<256, false>>(a, d_cond, d_c_pair, C, d_u_all, st);
    return launch_stack_local<tb::Cfg<512, false>>(a, d_cond, d_c_pair, C, d_u_all, st);
}
