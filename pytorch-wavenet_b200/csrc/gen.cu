// gen.cu -- Fast-WaveNet sampling as ONE persistent cooperative kernel.
//
// Replaces (reference file:line): WaveNetModel.generate_fast's warm-up and sampling loops wavenet_model.py:260-302,
// queue_dilate :177-184, the layer loop :131-165 and head :167-169 evaluated on single columns, and
// DilatedQueue.enqueue/dequeue/reset wavenet_modules.py:55-77.
//
// Work decomposition.  One network evaluation is a chain of matrix-vector products with a full dependency
// between stages, so the whole GPU works on every stage and stages are separated by a grid barrier:
//   per layer   stage 1: rows (f_c, g_c) of the k-tap conv for the CTA's dilation channels c -> z_c (exchange buffer)
//               stage 2: rows of residual_conv (-> next layer's ring slot for time t) and of skip_conv
//                        (-> running skip sum, kept in shared memory of the owning CTA across all layers)
//   head        end_conv_1 rows -> end_conv_2 rows -> every CTA redundantly picks the next sample
// Row r of a stage belongs to CTA (r mod G); one warp computes one row for all streams (lanes split K, butterfly
// reduction), so a stream's arithmetic does not depend on how many streams run beside it.
// The rings ("dilated queues") are the exchange medium between layers: ring l has (k-1)*d_l+1 slots of
// [n_streams][R]; slot (t mod len) holds the layer's input at time t, unwritten slots are zero (reset).
// Exchanged vectors are read with ld.global.cg (L2) because L1 is not coherent across SMs.
#include "common.cuh"
#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

namespace wn {

constexpr int GEN_NT = 256;
constexpr int GEN_WARPS = GEN_NT / 32;

struct GenLayer {
    const float *wf, *wg, *wr, *ws, *bf, *bg, *br, *bs;
    long long ring_off;     // in floats, from rings base
    int dil, ring_len;
};

// One stream's sampling settings: the library's device copy of a wn_gen_stream_params record; trunc = 1 when the truncation
// rule applies to the stream (temperature > 0 and a bound that drops classes).  origin / sample0 / first0: its
// wn_gen_stream_pos record (all 0 without positions): evaluation t is position t - origin of the stream, its prompt row
// starts at position first0 and its output / uniform / forced columns at sample sample0.
struct GenStream {
    int n_given, top_k, trunc;
    int origin, sample0, first0;
    float temperature, regularize;
    double top_p;
};

struct GenParams {
    const GenLayer* layers;
    int n_layers, k, R, D, S, E, C, NS;
    const float *start_w, *start_b, *e1w, *e1b, *e2w, *e2b;
    float* rings;
    float *zbuf, *skipbuf, *y1buf, *logitbuf;
    int* cur_idx;
    unsigned* bar;
    // run
    const int* first; int n_given;
    const int* forced; const double* uniforms;
    int* out_idx; float* out_logits;
    int n_samples, t0, n_evals;
    float temperature, regularize;
    // smem carve (floats)
    int regA, regB, pre_n, skacc_n;
    // ---- flag-in-data ("LL") exchange kernel
    uint2* ringLL;          // same geometry as rings, 8-byte {value, tag} elements
    uint2 *zLL, *skipLL, *y1LL, *logitLL;      // [2 parities][...] exchange vectors
    int* err;               // set to 1 by a CTA that timed out waiting for a tag
    int part_n;             // partial-sum scratch (floats)
    int wslot_floats, n_wslots;                // weight prefetch ring in shared memory (0 slots: read weights via L2)
    long long* trace;       // optional: clock64 stamps of CTA 0 / thread 0 during the last evaluation (wn_gen_read_trace)
    const unsigned char* cl8_img;              // batched cluster kernel: fragment-ordered bf16 hi/lo weight images (cl8_pack_kernel)
    const float* cond;      // optional condition table [n_layers][NS][2D]: each stream's filter / gate biases (bf + Vf h | bg + Vg h)
    // local conditioning (cond_hop > 0): cond is a window [n_layers][NS][cond_frames][2D] of frames [cond_frame0, +cond_frames);
    // evaluation t reads row t / cond_hop - cond_frame0 (per-stream windows: see cond_row).  cond_sstride = floats per
    // stream (2D for a global table).
    int cond_hop, cond_frame0, cond_frames, cond_sstride;
    // top-k / nucleus truncation (wn_gen_set_truncation): trunc = 1 when the rule applies to this launch (temperature > 0
    // and a bound that drops classes); the kernels branch to choose_truncated on it and run their own selection otherwise
    int top_k, trunc;
    double top_p;
    // per-stream settings (wn_gen_set_stream_params; null: every stream uses the scalars above).  The head runs at every
    // evaluation t >= head_from (min over streams of n_given - 1, n_given - 1 on the scalar path); n_given is then the
    // pitch of `first`, and trunc is set when any stream truncates (it only sizes kernel 1's scratch)
    const GenStream* ps;
    int head_from;
    // with ps: each stream's local-conditioning window {cond_origin, cond_frame0} (cond_row; {0, 0} under one shared window).
    // Kept apart from GenStream so that the kernels which never read it keep their record layout.
    const int2* pcw;
};

// Every role of every multi-stream kernel (workers, weight producers, pusher) decides whether evaluation t runs the head
// with this one predicate, so that they all schedule the same stages.
__device__ __forceinline__ bool head_at(const GenParams& p, int t) { return t >= p.head_from; }

// Stream s's settings: its record under per-stream parameters, the launch's scalars otherwise.  Read where the stream is
// known (input select, regularizer, selection), never held across the per-layer loops.  PS: PS_ANY tests p.ps; a kernel
// with an instantiation per path passes PS_OFF (p.ps is null: it then carries no trace of the records) or PS_ON (set).
enum { PS_OFF = 0, PS_ON = 1, PS_ANY = 2 };
template <int PS = PS_ANY>
__device__ __forceinline__ bool has_records(const GenParams& p) { return PS == PS_ANY ? p.ps != nullptr : PS == PS_ON; }
template <int PS = PS_ANY>
__device__ __forceinline__ GenStream stream_set(const GenParams& p, int s) {
    if (has_records<PS>(p)) return p.ps[s];
    GenStream g;
    g.n_given = p.n_given; g.top_k = p.top_k; g.trunc = p.trunc;
    g.origin = g.sample0 = g.first0 = 0;
    g.temperature = p.temperature; g.regularize = p.regularize; g.top_p = p.top_p;
    return g;
}

// The given input of evaluation t of stream s at its position q = t - origin: its prompt sample (first has pitch
// p.n_given; the row starts at position first0), else its forced sample when teacher forcing (the row starts at sample
// sample0).  false: the stream feeds back its own last choice.
template <int PS = PS_ANY>
__device__ __forceinline__ bool given_input(const GenParams& p, int s, int t, int& v) {
    int ng = p.n_given, q = t, f0 = 0, s0 = 0;
    if (has_records<PS>(p)) {
        const GenStream& g = p.ps[s];
        ng = g.n_given; q = t - g.origin; f0 = g.first0; s0 = g.sample0;
    }
    if (q < ng) { v = p.first[(size_t)s * p.n_given + (q - f0)]; return true; }
    if (p.forced != nullptr) { v = p.forced[(size_t)s * p.n_samples + (q - ng - s0)]; return true; }
    return false;
}

// The output / uniform column of the sample stream s chooses at evaluation t: sample q - (n_given - 1) minus sample0
// (negative while the stream is still inside its prompt: no selection then; wn_gen_run keeps it so).
template <int PS = PS_ANY>
__device__ __forceinline__ int sample_of(const GenParams& p, int s, int t) {
    if (has_records<PS>(p)) {
        const GenStream& g = p.ps[s];
        return t - g.origin - (g.n_given - 1) - g.sample0;
    }
    return t - (p.n_given - 1);
}

// This evaluation's condition table: the window row of t's frame under local conditioning (once per evaluation).
__device__ __forceinline__ const float* cond_at(const GenParams& p, int t, int D) {
    return p.cond_hop ? p.cond + (size_t)(t / p.cond_hop - p.cond_frame0) * 2 * D : p.cond;
}

// Stream s's condition row at evaluation t, in floats from the stream's first row: under local conditioning window row
// (t - cond_origin) / cond_hop - cond_frame0 - p.cond_frame0 with the stream's p.pcw[s] = {cond_origin, cond_frame0}
// (wn_gen_set_condition_stream_frames: the stream's origin and first frame, p.cond_frame0 = 0; a shared window: 0 and 0),
// t / cond_hop - p.cond_frame0 without records; 0 for a global table.  Formed once per evaluation and stream.
template <int PS = PS_ANY>
__device__ __forceinline__ int cond_row(const GenParams& p, int s, int t, int D) {
    if (!p.cond_hop) return 0;
    int q = t, f0 = p.cond_frame0;
    if (has_records<PS>(p)) {
        const int2 w = p.pcw[s];
        q = t - w.x; f0 += w.y;
    }
    return (q / p.cond_hop - f0) * 2 * D;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Row ownership: CTA c owns the contiguous rows [c*per, min(N, (c+1)*per)), per = ceil(N/G).  Contiguous (not
// interleaved) so that what a CTA publishes per stage is one run of {value,tag} pairs: with >= 4 rows per CTA the
// stores of one warp instruction fill whole 32-byte sectors rather than 16-byte partial-sector writes from twice as many
// CTAs (tools/lat_probe.cu compares the two).
__device__ __forceinline__ int own_per(int N, int G) { return (N + G - 1) / G; }
__device__ __forceinline__ int own_cnt(int N, int G, int cta) {
    const int per = own_per(N, G), n = N - cta * per;
    return n < 0 ? 0 : (n < per ? n : per);
}

__device__ __forceinline__ void grid_barrier(unsigned* ctr, unsigned& target, unsigned G) {
    __syncthreads();
    if (threadIdx.x == 0) {
        target += G;
        __threadfence();
        atomicAdd(ctr, 1u);
        unsigned v;
        do {
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
        } while ((int)(v - target) < 0);
    }
    __syncthreads();
}

// dot products of one weight row (K floats, global) with the vectors xs[s][0..K) (shared) for streams s0..s0+SB
template <int SB>
__device__ __forceinline__ void row_dot(const float* __restrict__ w, const float* __restrict__ xs, int K, int NS,
                                        int s0, int lane, float (&acc)[SB]) {
#pragma unroll
    for (int j = 0; j < SB; ++j) acc[j] = 0.f;
    if ((K & 3) == 0) {
        const float4* w4p = reinterpret_cast<const float4*>(w);
        for (int i4 = lane; i4 < (K >> 2); i4 += 32) {
            const float4 w4 = __ldg(w4p + i4);
#pragma unroll
            for (int j = 0; j < SB; ++j) {
                if (s0 + j < NS) {
                    const float4 x4 = *reinterpret_cast<const float4*>(xs + (size_t)(s0 + j) * K + 4 * i4);
                    float a = acc[j];
                    a = fmaf(w4.x, x4.x, a); a = fmaf(w4.y, x4.y, a); a = fmaf(w4.z, x4.z, a); a = fmaf(w4.w, x4.w, a);
                    acc[j] = a;
                }
            }
        }
    } else {
        for (int i = lane; i < K; i += 32) {
            const float wv = __ldg(w + i);
#pragma unroll
            for (int j = 0; j < SB; ++j)
                if (s0 + j < NS) acc[j] = fmaf(wv, xs[(size_t)(s0 + j) * K + i], acc[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < SB; ++j) acc[j] = warp_sum(acc[j]);
}

// Activations of the sampler kernels (all three kernels use these, so they stay bit-identical to each other):
// ex2-based exp and fast division, absolute error ~2e-7 -- the same order as the difference between expf and the
// reference's CPU math, at a fraction of the instructions on the latency-critical path.
__device__ __forceinline__ float sigmoid_(float x) { return __fdividef(1.f, 1.f + __expf(-x)); }
__device__ __forceinline__ float tanh_(float x) { return 2.f * sigmoid_(2.f * x) - 1.f; }

// The argmax of every kernel: one warp over the C logits lg (shared memory), the lowest index wins ties.
__device__ __forceinline__ int warp_argmax(const float* lg, int C, int lane) {
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < C; c += 32) {
        const float x = lg[c];
        if (x > best || (x == best && c < bi)) { best = x; bi = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
    }
    return bi == 0x7fffffff ? 0 : bi;
}

// argmax (first index wins ties) or numpy.random.choice's inverse-CDF draw, by one warp over C logits in shared memory.
// Kept out of line so that its fp64 code does not sit in the instruction stream of the per-layer loop.
__device__ __noinline__ int choose_sample(float* logit_s, double* cdf, int C, int lane, float temperature, const double* u_ptr) {
    int choice;
    if (temperature > 0.f) {
        float m = -INFINITY;
        for (int c = lane; c < C; c += 32) {
            const float x = logit_s[c] / temperature;
            logit_s[c] = x;
            m = fmaxf(m, x);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        float sum = 0.f;
        for (int c = lane; c < C; c += 32) {
            const float e = expf(logit_s[c] - m);
            logit_s[c] = e;
            sum += e;
        }
        sum = warp_sum(sum);
        __syncwarp();
        // numpy.random.choice: float64 cumulative sum of the float32 probabilities, normalised by its last element,
        // searchsorted(side='right').  The running sum is taken per lane over a contiguous chunk plus a warp scan
        // (equal to the sequential sum up to float64 rounding, i.e. ~1e-16 relative on the CDF).
        const int per = (C + 31) / 32;
        const int c_lo = lane * per, c_hi = min(C, c_lo + per);
        double run = 0.0;
        for (int c = c_lo; c < c_hi; ++c) { run += (double)(logit_s[c] / sum); cdf[c] = run; }
        double incl = run;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const double up = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += up;
        }
        double excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 0.0;
        const double total = __shfl_sync(0xffffffffu, incl, 31);
        const double u = *u_ptr;
        const double ut = u * total;
        int cnt = 0;
        for (int c = c_lo; c < c_hi; ++c) {
            const double v = cdf[c] + excl;
            bool le = v <= ut;
            if (fabs(v - ut) <= 1e-9 * total) le = (v / total) <= u;       // exact rule only where it can matter
            cnt += le ? 1 : 0;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        choice = cnt < C ? cnt : C - 1;
    } else {
        choice = warp_argmax(logit_s, C, lane);
    }
    return choice;
}

// ---- top-k / nucleus (top-p) selection, shared by all five kernels (wn_gen_set_truncation states the rule)
// Order-preserving key of a logit: a larger float gets a larger key; -0 is folded onto +0 so that the two tie, as numbers.
__device__ __forceinline__ unsigned logit_key(float v) {
    const unsigned b = __float_as_uint(v + 0.f);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
// Rank key: the logit key above the class index reversed, so that of equal logits the lower index ranks higher.  All
// rank keys of a row are distinct, and none equals ~0 (that would need a NaN logit).
__device__ __forceinline__ unsigned long long rank_key(const unsigned* key_s, int c, int C) {
    return ((unsigned long long)key_s[c] << 32) | (unsigned)(C - 1 - c);
}
__device__ __forceinline__ double warp_sum_d(double v) {   // xor butterfly: every lane ends with the same bits
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// One warp draws from the C logits lg (shared memory) with only the top_k highest-ranked classes (0: all) and, of those,
// the shortest rank-ordered prefix holding top_p of their probability mass.  key_s and p_s are C-entry scratch of the
// warp; key_s may be lg itself (each lane reads lg[c] before it writes key_s[c]), p_s must not overlap either.
//   1. p_c: the kernels' fp32 softmax of lg / temperature, bit for bit (same divisions, expf, and summation order).
//   2. K1 = the top_k largest rank keys: bisection for the largest bound with at least top_k keys at or above it, which
//      stops as soon as exactly top_k are (the keys are distinct, so it always gets there).
//   3. K = the largest bound >= K1's whose keys carry >= top_p * (float64 mass of K1), bisected until one key separates
//      the bounds that pass and fail: K is then exactly the shortest prefix that reaches the threshold.
//   4. The kernels' inverse CDF over the classes of K in index order (per-lane chunks + a warp scan in float64), edges
//      <= u counted over K only, the count mapped to the kept class of that rank and clamped to the last kept class.
// Out of line, as choose_sample is, so that none of it enters the register allocation of the per-layer loops.
__device__ __noinline__ int choose_truncated(const float* lg, unsigned* key_s, float* p_s, int C, int lane,
                                             float temperature, int top_k, double top_p, const double* u_ptr) {
    float m = -INFINITY;
    for (int c = lane; c < C; c += 32) {
        const float l = lg[c];
        const float x = l / temperature;
        key_s[c] = logit_key(l);
        p_s[c] = x;
        m = fmaxf(m, x);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) {
        const float e = expf(p_s[c] - m);
        p_s[c] = e;
        sum += e;
    }
    sum = warp_sum(sum);
    for (int c = lane; c < C; c += 32) p_s[c] = p_s[c] / sum;
    __syncwarp();

    unsigned long long lo = 0ull;                           // kept: rank key >= lo
    if (top_k > 0 && top_k < C) {
        unsigned long long hi = ~0ull;                      // fewer than top_k keys >= hi
        int n_lo = C;
        while (n_lo != top_k) {
            const unsigned long long mid = lo + ((hi - lo) >> 1);
            int n = 0;
            for (int c = lane; c < C; c += 32) n += rank_key(key_s, c, C) >= mid ? 1 : 0;
            n = __reduce_add_sync(0xffffffffu, n);
            if (n >= top_k) { lo = mid; n_lo = n; } else hi = mid;
        }
    }
    if (top_p < 1.0) {
        int n_lo = 0;
        double s_lo = 0.0;
        for (int c = lane; c < C; c += 32)
            if (rank_key(key_s, c, C) >= lo) { ++n_lo; s_lo += (double)p_s[c]; }
        n_lo = __reduce_add_sync(0xffffffffu, n_lo);
        const double thr = top_p * warp_sum_d(s_lo);
        unsigned long long hi = ~0ull;                      // the keys >= hi carry less than thr
        int n_hi = 0;
        while (n_lo - n_hi > 1) {
            const unsigned long long mid = lo + ((hi - lo) >> 1);
            int n = 0;
            double s = 0.0;
            for (int c = lane; c < C; c += 32)
                if (rank_key(key_s, c, C) >= mid) { ++n; s += (double)p_s[c]; }
            n = __reduce_add_sync(0xffffffffu, n);
            if (warp_sum_d(s) >= thr) { lo = mid; n_lo = n; } else { hi = mid; n_hi = n; }
        }
    }

    const int per = (C + 31) / 32;
    const int c_lo = lane * per, c_hi = min(C, c_lo + per);
    double run = 0.0;
    int nk = 0;
    for (int c = c_lo; c < c_hi; ++c)
        if (rank_key(key_s, c, C) >= lo) { run += (double)p_s[c]; ++nk; }
    double incl = run;
    int kincl = nk;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double up = __shfl_up_sync(0xffffffffu, incl, o);
        const int kup = __shfl_up_sync(0xffffffffu, kincl, o);
        if (lane >= o) { incl += up; kincl += kup; }
    }
    double excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 0.0;
    const int kexcl = kincl - nk;
    const double total = __shfl_sync(0xffffffffu, incl, 31);
    const int n_kept = __shfl_sync(0xffffffffu, kincl, 31);
    const double u = *u_ptr;
    const double ut = u * total;
    int cnt = 0;
    run = 0.0;
    for (int c = c_lo; c < c_hi; ++c) {
        if (rank_key(key_s, c, C) < lo) continue;
        run += (double)p_s[c];
        const double v = run + excl;
        bool le = v <= ut;
        if (fabs(v - ut) <= 1e-9 * total) le = (v / total) <= u;           // exact rule only where it can matter
        cnt += le ? 1 : 0;
    }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    const int r = cnt < n_kept ? cnt : n_kept - 1;                          // rank among the kept classes, ascending index
    int choice = -1;
    if (r >= kexcl && r < kexcl + nk) {
        int seen = kexcl;
        for (int c = c_lo; c < c_hi; ++c)
            if (rank_key(key_s, c, C) >= lo && seen++ == r) { choice = c; break; }
    }
    return __reduce_max_sync(0xffffffffu, choice);
}

template <int SB>
__global__ void __launch_bounds__(GEN_NT, 1) gen_kernel(const GenParams p) {
    extern __shared__ __align__(16) float sm[];
    float* regA = sm;                          // stage-1 inputs [NS][k*R] / head input [NS][S]
    float* regB = regA + p.regA;               // z [NS][D] / y1 [NS][E]
    float* pre = regB + p.regB;                // per-item results [items][NS]
    float* skacc = pre + p.pre_n;              // running skip sums of the rows this CTA owns [rows][NS]
    int* idx_s = reinterpret_cast<int*>(skacc + p.skacc_n);     // current input index per stream [NS]
    int* crow_s = idx_s + p.NS;                                 // this evaluation's condition row per stream [NS] (cond_row)
    float* prob = reinterpret_cast<float*>(crow_s + p.NS);      // [GEN_WARPS][C] softmax scratch

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cta = blockIdx.x, G = gridDim.x;
    const int NS = p.NS, R = p.R, D = p.D, S = p.S, E = p.E, C = p.C, k = p.k;
    const int K1 = k * R;
    unsigned bar_target = 0;

    // owned rows per stage: row r belongs to CTA (r mod G); local index r / G
    const int nD = own_cnt(D, G, cta), oD = cta * own_per(D, G);
    const int nR = own_cnt(R, G, cta), oR = cta * own_per(R, G);
    const int nS = own_cnt(S, G, cta), oS = cta * own_per(S, G);
    const int nE = own_cnt(E, G, cta), oE = cta * own_per(E, G);
    const int nC = own_cnt(C, G, cta), oC = cta * own_per(C, G);

    // the index chosen by the evaluation before t0 (continuation of a previous launch)
    for (int s = tid; s < NS; s += GEN_NT) idx_s[s] = p.cur_idx[s];
    __syncthreads();

    for (int ev = 0; ev < p.n_evals; ++ev) {
        const int t = p.t0 + ev;                           // absolute evaluation counter == time
        const bool want_head = head_at(p, t);
        // ---- input index and condition row of this evaluation
        for (int s = tid; s < NS; s += GEN_NT) {
            int v;
            if (given_input(p, s, t, v)) idx_s[s] = v;
            if (p.cond) crow_s[s] = cond_row(p, s, t, D);
        }
        for (int i = tid; i < nS * NS; i += GEN_NT) skacc[i] = 0.f;
        __syncthreads();

        for (int l = 0; l < p.n_layers; ++l) {
            const GenLayer L = p.layers[l];
            float* ring = p.rings + L.ring_off;
            const int slot_t = t % L.ring_len;
            // ---- gather stage-1 inputs, interleaved like a conv weight row: regA[s][r*k + j] = tap j of channel r
            for (int i = tid; i < NS * K1; i += GEN_NT) {
                const int s = i / K1, rem = i - s * K1, r = rem / k, j = rem - r * k;
                float v;
                if (j == k - 1 && l == 0) {                 // current input of layer 0 = start conv column
                    int c = idx_s[s];
                    c = c < 0 ? 0 : (c >= C ? C - 1 : c);
                    v = __ldg(p.start_w + (size_t)r * C + c) + (p.start_b ? __ldg(p.start_b + r) : 0.f);
                    if (r >= oR && r < oR + nR) ring[((size_t)slot_t * NS + s) * R + r] = v;       // enqueue (owner writes)
                } else {
                    int tt = t - (k - 1 - j) * L.dil;        // time of tap j
                    int slot = tt % L.ring_len;
                    if (slot < 0) slot += L.ring_len;        // never-written slot: zero history
                    v = __ldcg(ring + ((size_t)slot * NS + s) * R + r);
                }
                regA[i] = v;
            }
            __syncthreads();
            // ---- stage 1: filter / gate rows of the owned dilation channels
            for (int it = warp; it < 2 * nD; it += GEN_WARPS) {
                const int c = oD + (it >> 1);
                const float* w = ((it & 1) ? L.wg : L.wf) + (size_t)c * K1;
                const float* bp = (it & 1) ? L.bg : L.bf;
                const float bias = bp ? __ldg(bp + c) : 0.f;
                const float* cb = p.cond ? p.cond + (size_t)l * NS * p.cond_sstride + ((it & 1) ? D : 0) + c : nullptr;
                for (int s0 = 0; s0 < NS; s0 += SB) {
                    float acc[SB];
                    row_dot<SB>(w, regA, K1, NS, s0, lane, acc);
                    if (lane == 0) {
#pragma unroll
                        for (int j = 0; j < SB; ++j)
                            if (s0 + j < NS)
                                pre[it * NS + s0 + j] = acc[j] + (cb ? __ldg(cb + (size_t)(s0 + j) * p.cond_sstride + crow_s[s0 + j]) : bias);
                    }
                }
            }
            __syncthreads();
            for (int i = tid; i < nD * NS; i += GEN_NT) {
                const int ci = i / NS, s = i - ci * NS;
                const float z = tanh_(pre[(2 * ci) * NS + s]) * sigmoid_(pre[(2 * ci + 1) * NS + s]);
                p.zbuf[(size_t)s * D + oD + ci] = z;
            }
            grid_barrier(p.bar, bar_target, G);
            // ---- stage 2: residual rows (not needed after the last layer) and skip rows (not needed in warm-up)
            for (int i = tid; i < NS * D; i += GEN_NT) regB[i] = __ldcg(p.zbuf + i);
            __syncthreads();
            const int nres = (l + 1 < p.n_layers) ? nR : 0;
            const int nskp = want_head ? nS : 0;
            for (int it = warp; it < nres + nskp; it += GEN_WARPS) {
                const bool is_res = it < nres;
                const int li = is_res ? it : it - nres;
                const int row = (is_res ? oR : oS) + li;
                const float* w = (is_res ? L.wr : L.ws) + (size_t)row * D;
                const float* bp = is_res ? L.br : L.bs;
                const float bias = bp ? __ldg(bp + row) : 0.f;
                for (int s0 = 0; s0 < NS; s0 += SB) {
                    float acc[SB];
                    row_dot<SB>(w, regB, D, NS, s0, lane, acc);
                    if (lane == 0) {
#pragma unroll
                        for (int j = 0; j < SB; ++j) {
                            const int s = s0 + j;
                            if (s >= NS) break;
                            const float v = acc[j] + bias;
                            if (is_res) {
                                const GenLayer& Ln = p.layers[l + 1];
                                const float cur = regA[(size_t)s * K1 + row * k + (k - 1)];
                                p.rings[Ln.ring_off + ((size_t)(t % Ln.ring_len) * NS + s) * R + row] = v + cur;
                            } else {
                                skacc[li * NS + s] = v + skacc[li * NS + s];
                            }
                        }
                    }
                }
            }
            if (l + 1 == p.n_layers && want_head) {
                __syncthreads();
                for (int i = tid; i < nS * NS; i += GEN_NT) {
                    const int li = i / NS, s = i - li * NS;
                    p.skipbuf[(size_t)s * S + oS + li] = skacc[i];
                }
            }
            grid_barrier(p.bar, bar_target, G);
        }
        if (!want_head) continue;

        // ---- head A: y1 = relu(W1 relu(skip) + b1)
        for (int i = tid; i < NS * S; i += GEN_NT) regA[i] = fmaxf(__ldcg(p.skipbuf + i), 0.f);
        __syncthreads();
        for (int it = warp; it < nE; it += GEN_WARPS) {
            const int row = oE + it;
            const float bias = __ldg(p.e1b + row);
            for (int s0 = 0; s0 < NS; s0 += SB) {
                float acc[SB];
                row_dot<SB>(p.e1w + (size_t)row * S, regA, S, NS, s0, lane, acc);
                if (lane == 0) {
#pragma unroll
                    for (int j = 0; j < SB; ++j)
                        if (s0 + j < NS) p.y1buf[(size_t)(s0 + j) * E + row] = fmaxf(acc[j] + bias, 0.f);
                }
            }
        }
        grid_barrier(p.bar, bar_target, G);
        // ---- head B: logits = W2 y1 + b2, minus the regularizer (wavenet_model.py:273-274,280)
        for (int i = tid; i < NS * E; i += GEN_NT) regB[i] = __ldcg(p.y1buf + i);
        __syncthreads();
        for (int it = warp; it < nC; it += GEN_WARPS) {
            const int row = oC + it;
            const float bias = __ldg(p.e2b + row);
            const float dc = (float)row - (float)C / 2.f;
            const float reg = (dc * dc) * p.regularize;
            for (int s0 = 0; s0 < NS; s0 += SB) {
                float acc[SB];
                row_dot<SB>(p.e2w + (size_t)row * E, regB, E, NS, s0, lane, acc);
                if (lane == 0) {
#pragma unroll
                    for (int j = 0; j < SB; ++j) {
                        const int s = s0 + j;
                        if (s >= NS) break;
                        const float v = (acc[j] + bias) - (p.ps ? __fmul_rn(dc * dc, p.ps[s].regularize) : reg);
                        p.logitbuf[(size_t)s * C + row] = v;
                        const int samp = sample_of(p, s, t);
                        if (p.out_logits && samp >= 0) p.out_logits[((size_t)s * p.n_samples + samp) * C + row] = v;
                    }
                }
            }
        }
        grid_barrier(p.bar, bar_target, G);
        // ---- choose (every CTA redundantly, so no broadcast barrier is needed): warp per stream
        float* pw = prob + warp * C;
        for (int s = warp; s < NS; s += GEN_WARPS) {
            const GenStream ss = stream_set(p, s);
            const int samp = sample_of(p, s, t);           // output column of the sample this evaluation chooses
            if (samp < 0) continue;                        // still inside its prompt
            // the logits (written by other CTAs: through the L2) into the warp's scratch
            const float* lg = p.logitbuf + (size_t)s * C;
            for (int c = lane; c < C; c += 32) pw[c] = __ldcg(lg + c);
            __syncwarp();
            int choice;
            if (ss.trunc) {
                // the logits become the rank keys; probabilities in the truncation scratch that the host adds past prob
                // only for such launches
                choice = choose_truncated(pw, reinterpret_cast<unsigned*>(pw), prob + (GEN_WARPS + warp) * C, C, lane,
                                          ss.temperature, ss.top_k, ss.top_p, p.uniforms + (size_t)s * p.n_samples + samp);
            } else if (ss.temperature > 0.f) {
                float m = -INFINITY;
                for (int c = lane; c < C; c += 32) {
                    const float x = pw[c] / ss.temperature;
                    pw[c] = x;
                    m = fmaxf(m, x);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                float sum = 0.f;
                for (int c = lane; c < C; c += 32) {
                    const float e = expf(pw[c] - m);
                    pw[c] = e;
                    sum += e;
                }
                sum = warp_sum(sum);
                __syncwarp();
                choice = 0;
                if (lane == 0) {
                    // numpy.random.choice: float64 cumulative sum, normalised by its last element, searchsorted 'right'
                    double total = 0.0;
                    for (int c = 0; c < C; ++c) total += (double)(pw[c] / sum);
                    const double u = p.uniforms[(size_t)s * p.n_samples + samp];
                    double run = 0.0;
                    int cnt = 0;
                    for (int c = 0; c < C; ++c) {
                        run += (double)(pw[c] / sum);
                        cnt += ((run / total) <= u) ? 1 : 0;
                    }
                    choice = cnt < C ? cnt : C - 1;
                }
                choice = __shfl_sync(0xffffffffu, choice, 0);
            } else {
                choice = warp_argmax(pw, C, lane);
            }
            if (lane == 0) {
                idx_s[s] = choice;
                if (cta == 0) p.out_idx[(size_t)s * p.n_samples + samp] = choice;
            }
        }
        __syncthreads();
    }
    if (cta == 0)
        for (int s = tid; s < NS; s += GEN_NT) p.cur_idx[s] = idx_s[s];
}

// ================================================================================================ LL kernel
// Same decomposition as gen_kernel, but no grid barriers: every exchanged float travels as an 8-byte {value, tag}
// pair written with one volatile store; consumers spin on the pair itself until the tag they expect appears
// (the NCCL "LL" idea).  Tags: ring slot of time tau carries tau+1; per-evaluation vectors carry t+1 and are
// double-buffered by the parity of t.  A location is rewritten two evaluations (or one full ring period) after it
// was last read, and a writer can only get there once every CTA has finished the evaluation in between -- each CTA
// owns at least one dilation channel (G <= D) whose z every residual row needs -- so no reader is ever overtaken.
// The weight rows a CTA needs for the next stages are prefetched into shared memory with cp.async.bulk (TMA) while
// it waits for data; they are the same rows every evaluation, in the parameters' own (state_dict) layout.
constexpr long long GEN_TIMEOUT_CYCLES = 6000000000LL;     // ~3 s: a missing tag aborts the launch instead of hanging

// one naturally aligned 64-bit word = single-copy atomic; gpu scope keeps the traffic at the L2
__device__ __forceinline__ uint2 ld_pair(const uint2* p) {
    unsigned long long w;
    asm volatile("ld.relaxed.gpu.global.b64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
    return make_uint2((unsigned)(w & 0xffffffffull), (unsigned)(w >> 32));
}
__device__ __forceinline__ void st_pair(uint2* p, float val, unsigned tag) {
    const unsigned long long w = ((unsigned long long)tag << 32) | (unsigned long long)__float_as_uint(val);
    asm volatile("st.relaxed.gpu.global.b64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}
__device__ __forceinline__ float poll_pair(const uint2* p, unsigned tag, int* err, int* abort_s) {
    uint2 v = ld_pair(p);
    if (v.y != tag) {
        const long long t0 = clock64();
        do {
            __nanosleep(40);                      // keep the polling storm off the L2 slice the producer writes to
            v = ld_pair(p);
            if (clock64() - t0 > GEN_TIMEOUT_CYCLES || *reinterpret_cast<volatile int*>(err) != 0) {
                *reinterpret_cast<volatile int*>(err) = 1;
                *reinterpret_cast<volatile int*>(abort_s) = 1;
                break;
            }
        } while (v.y != tag);
    }
    return __uint_as_float(v.x);
}

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst)),
                 "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    unsigned done;
    do {
        asm volatile(
            "{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
            : "=r"(done)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!done);
}

// partial dot products over K-range [k0, k1) (multiples of 4 when K%4==0) -- weights from shared or global memory
template <int SB, bool W_SMEM>
__device__ __forceinline__ void row_dot_part(const float* __restrict__ w, const float* __restrict__ xs, int K, int k0,
                                             int k1, int NS, int s0, int lane, float (&acc)[SB]) {
#pragma unroll
    for (int j = 0; j < SB; ++j) acc[j] = 0.f;
    if ((K & 3) == 0) {
        const float4* w4p = reinterpret_cast<const float4*>(w);
        for (int i4 = (k0 >> 2) + lane; i4 < (k1 >> 2); i4 += 32) {
            float4 w4;
            if constexpr (W_SMEM) w4 = w4p[i4];
            else w4 = __ldg(w4p + i4);
#pragma unroll
            for (int j = 0; j < SB; ++j) {
                if (s0 + j < NS) {
                    const float4 x4 = *reinterpret_cast<const float4*>(xs + (size_t)(s0 + j) * K + 4 * i4);
                    float a = acc[j];
                    a = fmaf(w4.x, x4.x, a); a = fmaf(w4.y, x4.y, a); a = fmaf(w4.z, x4.z, a); a = fmaf(w4.w, x4.w, a);
                    acc[j] = a;
                }
            }
        }
    } else {
        for (int i = k0 + lane; i < k1; i += 32) {
            float wv;
            if constexpr (W_SMEM) wv = w[i];
            else wv = __ldg(w + i);
#pragma unroll
            for (int j = 0; j < SB; ++j)
                if (s0 + j < NS) acc[j] = fmaf(wv, xs[(size_t)(s0 + j) * K + i], acc[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < SB; ++j) acc[j] = warp_sum(acc[j]);
}

// Rows of one stage for one CTA.  Stage numbering inside an evaluation: 2l = conv rows of layer l, 2l+1 = 1x1 rows
// of layer l, 2NL = end_conv_1 rows, 2NL+1 = end_conv_2 rows.
struct StageDesc {
    int n, K;                 // rows, row length
    int n_first;              // stage 2: residual rows come first (n_first of them), then skip rows
    int n_nom;                // nominal row count of the stage (fixes the K split, whatever rows are active)
};
__device__ __forceinline__ StageDesc stage_desc(const GenParams& p, int st, bool want_head, int nD, int nR, int nS,
                                                int nE, int nC) {
    StageDesc d;
    const int NL = p.n_layers;
    if (st < 2 * NL) {
        const int l = st >> 1;
        if ((st & 1) == 0) { d.n = 2 * nD; d.K = p.k * p.R; d.n_first = d.n; d.n_nom = d.n; }
        else { d.n_first = (l + 1 < NL) ? nR : 0; d.n = d.n_first + (want_head ? nS : 0); d.K = p.D; d.n_nom = nR + nS; }
    } else if (st == 2 * NL) { d.n = nE; d.K = p.S; d.n_first = d.n; d.n_nom = d.n; }
    else { d.n = nC; d.K = p.E; d.n_first = d.n; d.n_nom = d.n; }
    return d;
}
__device__ __forceinline__ const float* stage_row(const GenParams& p, const GenLayer* layers, int st, const StageDesc& d,
                                                  int i, int cta, int G) {
    const int NL = p.n_layers;
    if (st < 2 * NL) {
        const GenLayer& L = layers[st >> 1];
        if ((st & 1) == 0) return ((i & 1) ? L.wg : L.wf) + (size_t)(cta * own_per(p.D, G) + (i >> 1)) * d.K;
        if (i < d.n_first) return L.wr + (size_t)(cta * own_per(p.R, G) + i) * d.K;
        return L.ws + (size_t)(cta * own_per(p.S, G) + (i - d.n_first)) * d.K;
    }
    if (st == 2 * NL) return p.e1w + (size_t)(cta * own_per(p.E, G) + i) * d.K;
    return p.e2w + (size_t)(cta * own_per(p.C, G) + i) * d.K;
}

template <int SB, bool PREFETCH>
__global__ void __launch_bounds__(GEN_NT, 1) gen_kernel_ll(const GenParams p) {
    extern __shared__ __align__(16) float sm[];
    float* regA = sm;                          // stage-1 inputs [NS][k*R] / head input [NS][S] / logits [NS][C]
    float* regB = regA + p.regA;               // z [NS][D] / y1 [NS][E]
    float* part = regB + p.regB;               // partial sums [item][kpart][NS]
    float* skacc = part + p.part_n;            // running skip sums of the rows this CTA owns [rows][NS]
    float* prob = skacc + p.skacc_n;           // [GEN_WARPS][C] softmax scratch
    double* cdf = reinterpret_cast<double*>(prob + GEN_WARPS * p.C);   // [GEN_WARPS][C]
    float* wbuf = reinterpret_cast<float*>(cdf + GEN_WARPS * p.C);     // [n_wslots][wslot_floats]
    unsigned long long* fullb = reinterpret_cast<unsigned long long*>(wbuf + (size_t)p.n_wslots * p.wslot_floats);
    GenLayer* lay_s = reinterpret_cast<GenLayer*>(fullb + 8);           // per-layer table, copied from global once
    int* idx_s = reinterpret_cast<int*>(lay_s + p.n_layers);            // current input index per stream [NS]
    int* abort_s = idx_s + p.NS;
    int* crow_s = abort_s + 1;                                          // this evaluation's condition row per stream [NS]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cta = blockIdx.x, G = gridDim.x;
    const int NS = p.NS, R = p.R, D = p.D, S = p.S, E = p.E, C = p.C, k = p.k, NL = p.n_layers;
    const int K1 = k * R;
    const int nD = own_cnt(D, G, cta), oD = cta * own_per(D, G);
    const int nR = own_cnt(R, G, cta), oR = cta * own_per(R, G);
    const int nS = own_cnt(S, G, cta), oS = cta * own_per(S, G);
    const int nE = own_cnt(E, G, cta), oE = cta * own_per(E, G);
    const int nC = own_cnt(C, G, cta), oC = cta * own_per(C, G);
    const int NSLOT = p.n_wslots;

    for (int s = tid; s < NS; s += GEN_NT) idx_s[s] = p.cur_idx[s];
    {
        const int* src = reinterpret_cast<const int*>(p.layers);
        int* dst = reinterpret_cast<int*>(lay_s);
        for (int i = tid; i < NL * (int)(sizeof(GenLayer) / sizeof(int)); i += GEN_NT) dst[i] = src[i];
    }
    if (tid == 0) {
        *abort_s = 0;
        if (PREFETCH)
            for (int i = 0; i < NSLOT; ++i) mbar_init(fullb + i, 1);
    }
    if (PREFETCH) asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();

    // ---- weight prefetch pipeline (thread 0 produces): stage q of the launch lives in slot q % NSLOT
    int pf_ev = 0, pf_st = 0;                 // producer cursor
    long long pf_q = 0, cons_q = 0;
    auto stages_in_eval = [&](int ev) { return head_at(p, p.t0 + ev) ? 2 * NL + 2 : 2 * NL; };
    auto produce_one = [&]() {                // the last thread only (it has no epilogue work)
        if (pf_ev >= p.n_evals) return;
        const bool wh = head_at(p, p.t0 + pf_ev);
        const StageDesc d = stage_desc(p, pf_st, wh, nD, nR, nS, nE, nC);
        const int slot = (int)(pf_q % NSLOT);
        mbar_expect_tx(fullb + slot, (unsigned)(d.n * d.K * 4));
        float* dst = wbuf + (size_t)slot * p.wslot_floats;
        for (int i = 0; i < d.n; ++i) bulk_g2s(dst + (size_t)i * d.K, stage_row(p, lay_s, pf_st, d, i, cta, G), d.K * 4, fullb + slot);
        ++pf_q;
        if (++pf_st >= stages_in_eval(pf_ev)) { pf_st = 0; ++pf_ev; }
    };
    if (PREFETCH && tid == GEN_NT - 1)
        for (int i = 0; i < NSLOT; ++i) produce_one();

    // One dot-product stage: rows of `st` times the vectors xs[s][0..K) -> part[item][kpart][s]; all 8 warps work,
    // rows are split over nw = 8/items warps along K when there are fewer rows than warps.
    auto run_stage = [&](int st, const StageDesc& d, const float* xs, int& nw_out) {
        int nw = 1;
        while (nw * 2 * d.n_nom <= GEN_WARPS && (d.K / (nw * 2)) % 4 == 0 && d.K / (nw * 2) >= 32) nw *= 2;
        if (d.n_nom == 0) nw = 1;
        nw_out = nw;
        const float* wslot = nullptr;
        if (PREFETCH) {
            const int slot = (int)(cons_q % NSLOT);
            mbar_wait(fullb + slot, (unsigned)((cons_q / NSLOT) & 1));
            wslot = wbuf + (size_t)slot * p.wslot_floats;
        }
        const int kchunk = d.K / nw;
        for (int wi = warp; wi < d.n * nw; wi += GEN_WARPS) {
            const int it = wi / nw, kp = wi - it * nw;
            const int k0 = kp * kchunk, k1 = (kp == nw - 1) ? d.K : k0 + kchunk;
            for (int s0 = 0; s0 < NS; s0 += SB) {
                float acc[SB];
                if (PREFETCH) row_dot_part<SB, true>(wslot + (size_t)it * d.K, xs, d.K, k0, k1, NS, s0, lane, acc);
                else row_dot_part<SB, false>(stage_row(p, lay_s, st, d, it, cta, G), xs, d.K, k0, k1, NS, s0, lane, acc);
                if (lane == 0) {
#pragma unroll
                    for (int j = 0; j < SB; ++j)
                        if (s0 + j < NS) part[(size_t)(it * nw + kp) * NS + s0 + j] = acc[j];
                }
            }
        }
        ++cons_q;
    };
    auto sum_parts = [&](int it, int nw, int s) {
        float v = part[(size_t)(it * nw) * NS + s];
        for (int kp = 1; kp < nw; ++kp) v += part[(size_t)(it * nw + kp) * NS + s];
        return v;
    };

    for (int ev = 0; ev < p.n_evals; ++ev) {
        const int t = p.t0 + ev;
        const unsigned tag = (unsigned)t + 1u;
        const int par = t & 1;
        const bool want_head = head_at(p, t);
        for (int s = tid; s < NS; s += GEN_NT) {
            int v;
            if (given_input(p, s, t, v)) idx_s[s] = v;
            if (p.cond) crow_s[s] = cond_row(p, s, t, D);
        }
        for (int i = tid; i < nS * NS; i += GEN_NT) skacc[i] = 0.f;
        __syncthreads();
        if (*abort_s) return;

        for (int l = 0; l < NL; ++l) {
            const GenLayer& L = lay_s[l];
            uint2* ring = p.ringLL + L.ring_off;
            const int slot_t = t % L.ring_len;
            // ---- stage-1 inputs: regA[s][r*k + j] = tap j of channel r (tap k-1 = the value just enqueued)
            for (int i = tid; i < NS * K1; i += GEN_NT) {
                const int s = i / K1, rem = i - s * K1, r = rem / k, j = rem - r * k;
                float v;
                if (j == k - 1 && l == 0) {
                    int c = idx_s[s];
                    c = c < 0 ? 0 : (c >= C ? C - 1 : c);
                    v = __ldg(p.start_w + (size_t)r * C + c) + (p.start_b ? __ldg(p.start_b + r) : 0.f);
                    if (r >= oR && r < oR + nR) st_pair(ring + ((size_t)slot_t * NS + s) * R + r, v, tag);       // enqueue
                } else {
                    const int tt = t - (k - 1 - j) * L.dil;
                    if (tt < 0) v = 0.f;                                                             // zero history
                    else v = poll_pair(ring + ((size_t)(tt % L.ring_len) * NS + s) * R + r, (unsigned)tt + 1u, p.err, abort_s);
                }
                regA[i] = v;
            }
            __syncthreads();
            if (*abort_s) return;
            // ---- stage 1: filter / gate rows -> z
            int nw;
            StageDesc d1 = stage_desc(p, 2 * l, want_head, nD, nR, nS, nE, nC);
            run_stage(2 * l, d1, regA, nw);
            __syncthreads();
            if (PREFETCH && tid == GEN_NT - 1) produce_one();
            uint2* zl = p.zLL + ((size_t)(par * NL + l) * NS) * D;
            for (int i = tid; i < nD * NS; i += GEN_NT) {
                const int ci = i / NS, s = i - ci * NS, c = oD + ci;
                const float* cb = p.cond ? p.cond + ((size_t)l * NS + s) * p.cond_sstride + crow_s[s] : nullptr;   // this stream's biases
                const float f = sum_parts(2 * ci, nw, s) + (cb ? __ldg(cb + c) : (L.bf ? __ldg(L.bf + c) : 0.f));
                const float g = sum_parts(2 * ci + 1, nw, s) + (cb ? __ldg(cb + D + c) : (L.bg ? __ldg(L.bg + c) : 0.f));
                st_pair(zl + (size_t)s * D + c, tanh_(f) * sigmoid_(g), tag);
            }
            // ---- stage 2: residual rows (-> next layer's ring slot t) and skip rows (-> running sums)
            StageDesc d2 = stage_desc(p, 2 * l + 1, want_head, nD, nR, nS, nE, nC);
            if (d2.n > 0) {
                for (int i = tid; i < NS * D; i += GEN_NT) regB[i] = poll_pair(zl + i, tag, p.err, abort_s);
            }
            __syncthreads();                       // also protects `part` (read above) against the next run_stage
            if (*abort_s) return;
            run_stage(2 * l + 1, d2, regB, nw);
            __syncthreads();
            if (PREFETCH && tid == GEN_NT - 1) produce_one();
            for (int i = tid; i < d2.n * NS; i += GEN_NT) {
                const int it = i / NS, s = i - it * NS;
                if (it < d2.n_first) {
                    const int row = oR + it;
                    const GenLayer& Ln = lay_s[l + 1];
                    const float v = sum_parts(it, nw, s) + (L.br ? __ldg(L.br + row) : 0.f);
                    const float cur = regA[(size_t)s * K1 + row * k + (k - 1)];
                    st_pair(p.ringLL + Ln.ring_off + ((size_t)(t % Ln.ring_len) * NS + s) * R + row, v + cur, tag);
                } else {
                    const int li = it - d2.n_first, row = oS + li;
                    const float v = sum_parts(it, nw, s) + (L.bs ? __ldg(L.bs + row) : 0.f);
                    skacc[li * NS + s] = v + skacc[li * NS + s];
                }
            }
            __syncthreads();                       // the epilogue read regA (cur) and part: done before the next gather
        }
        if (!want_head) continue;

        // ---- head: skip -> end_conv_1 -> end_conv_2 -> choose
        __syncthreads();
        uint2* skl = p.skipLL + (size_t)par * NS * S;
        for (int i = tid; i < nS * NS; i += GEN_NT) {
            const int li = i / NS, s = i - li * NS;
            st_pair(skl + (size_t)s * S + oS + li, skacc[i], tag);
        }
        int nw;
        StageDesc dA = stage_desc(p, 2 * NL, true, nD, nR, nS, nE, nC);
        if (dA.n > 0)
            for (int i = tid; i < NS * S; i += GEN_NT) regA[i] = fmaxf(poll_pair(skl + i, tag, p.err, abort_s), 0.f);
        __syncthreads();
        if (*abort_s) return;
        run_stage(2 * NL, dA, regA, nw);
        __syncthreads();
        if (PREFETCH && tid == GEN_NT - 1) produce_one();
        uint2* yl = p.y1LL + (size_t)par * NS * E;
        for (int i = tid; i < nE * NS; i += GEN_NT) {
            const int it = i / NS, s = i - it * NS, row = oE + it;
            st_pair(yl + (size_t)s * E + row, fmaxf(sum_parts(it, nw, s) + __ldg(p.e1b + row), 0.f), tag);
        }
        StageDesc dB = stage_desc(p, 2 * NL + 1, true, nD, nR, nS, nE, nC);
        if (dB.n > 0)
            for (int i = tid; i < NS * E; i += GEN_NT) regB[i] = poll_pair(yl + i, tag, p.err, abort_s);
        __syncthreads();
        if (*abort_s) return;
        run_stage(2 * NL + 1, dB, regB, nw);
        __syncthreads();
        if (PREFETCH && tid == GEN_NT - 1) produce_one();
        uint2* lgl = p.logitLL + (size_t)par * NS * C;
        for (int i = tid; i < nC * NS; i += GEN_NT) {
            const int it = i / NS, s = i - it * NS, row = oC + it;
            const float dc = (float)row - (float)C / 2.f;
            const float v = (sum_parts(it, nw, s) + __ldg(p.e2b + row)) - (dc * dc) * (p.ps ? p.ps[s].regularize : p.regularize);
            st_pair(lgl + (size_t)s * C + row, v, tag);
            const int samp = sample_of(p, s, t);
            if (p.out_logits && samp >= 0) p.out_logits[((size_t)s * p.n_samples + samp) * C + row] = v;
        }
        // ---- every CTA collects all logits and picks the next sample itself (no broadcast needed)
        for (int i = tid; i < NS * C; i += GEN_NT) regA[i] = poll_pair(lgl + i, tag, p.err, abort_s);
        __syncthreads();
        if (*abort_s) return;
        float* pw = prob + warp * C;
        double* cw = cdf + warp * C;
        for (int s = warp; s < NS; s += GEN_WARPS) {
            const GenStream ss = stream_set(p, s);
            const int samp = sample_of(p, s, t);
            if (samp < 0) continue;                        // still inside its prompt
            const float* lg = regA + (size_t)s * C;
            int choice;
            if (ss.trunc) {
                choice = choose_truncated(lg, reinterpret_cast<unsigned*>(pw), reinterpret_cast<float*>(cw), C, lane,
                                          ss.temperature, ss.top_k, ss.top_p, p.uniforms + (size_t)s * p.n_samples + samp);
            } else {
                for (int c = lane; c < C; c += 32) pw[c] = lg[c];      // choose_sample overwrites its input
                __syncwarp();
                choice = choose_sample(pw, cw, C, lane, ss.temperature,
                                       p.uniforms ? p.uniforms + (size_t)s * p.n_samples + samp : nullptr);
            }
            if (lane == 0) {
                idx_s[s] = choice;
                if (cta == 0) p.out_idx[(size_t)s * p.n_samples + samp] = choice;
            }
        }
        __syncthreads();
    }
    if (cta == 0)
        for (int s = tid; s < NS; s += GEN_NT) p.cur_idx[s] = idx_s[s];
}

// ================================================================================================ fast kernel
// Single stream, k = 2, power-of-two grid, every stage's rows a divisor of 8: the latency-critical special case
// (cfg 2).  Same exchange protocol, same tags, same summation order as gen_kernel_ll, but the per-stage critical
// path is stripped down: every warp owns one (row, K-part) pair for the whole launch, polls exactly the {value,tag}
// pairs it multiplies straight into registers (no staging, no index arithmetic with divisions), and there is ONE
// __syncthreads per stage (partial sums are double buffered).  Ring positions advance incrementally.
struct Pair2 { uint2 a, b; };
__device__ __forceinline__ Pair2 ld_pair2(const uint2* p) {
    unsigned long long w0, w1;
    asm volatile("ld.relaxed.gpu.global.v2.b64 {%0,%1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(p) : "memory");
    Pair2 r;
    r.a = make_uint2((unsigned)(w0 & 0xffffffffull), (unsigned)(w0 >> 32));
    r.b = make_uint2((unsigned)(w1 & 0xffffffffull), (unsigned)(w1 >> 32));
    return r;
}
// two consecutive pairs carrying `tag`; spins (bounded) until both are there
// slow path of poll2, out of line: spinning code (with its timeout) must not bloat the per-layer instruction stream
__device__ __noinline__ Pair2 poll2_spin(const uint2* p, unsigned tag, int* err, int* abort_s) {
    Pair2 q;
    const long long t0 = clock64();
    unsigned spins = 0;
    do {
        q = ld_pair2(p);
        if ((++spins & 255u) == 0 &&
            (clock64() - t0 > GEN_TIMEOUT_CYCLES || *reinterpret_cast<volatile int*>(err) != 0)) {
            *reinterpret_cast<volatile int*>(err) = 1;
            *reinterpret_cast<volatile int*>(abort_s) = 1;
            break;
        }
    } while (q.a.y != tag || q.b.y != tag);
    return q;
}
__device__ __forceinline__ void poll2(const uint2* p, unsigned tag, float& v0, float& v1, int* err, int* abort_s) {
    Pair2 q = ld_pair2(p);
    if (q.a.y != tag || q.b.y != tag) q = poll2_spin(p, tag, err, abort_s);
    v0 = __uint_as_float(q.a.x);
    v1 = __uint_as_float(q.b.x);
}

constexpr int FAST_MAXI = 4;      // float4 iterations per lane per row part (K part <= 512)

// All the pairs one lane multiplies in a stage, fetched with every load in flight at once (one L2 round trip when the
// data is already there) and re-fetched as a batch until all tags match.  Iteration `it` covers pairs
// [first + it*128, +4) of `base` (4 consecutive values = one float4 of the weight row).
__device__ __forceinline__ void poll_quads(const uint2* base, int first, int n_iter, unsigned tag, float (&v)[FAST_MAXI][4],
                                           int* err, int* abort_s) {
    Pair2 a[FAST_MAXI], b[FAST_MAXI];
    const long long t0 = clock64();
    unsigned spins = 0;
    for (;;) {
#pragma unroll
        for (int it = 0; it < FAST_MAXI; ++it)
            if (it < n_iter) {
                a[it] = ld_pair2(base + first + it * 128);
                b[it] = ld_pair2(base + first + it * 128 + 2);
            }
        bool ok = true;
#pragma unroll
        for (int it = 0; it < FAST_MAXI; ++it)
            if (it < n_iter) ok = ok && a[it].a.y == tag && a[it].b.y == tag && b[it].a.y == tag && b[it].b.y == tag;
        if (ok) break;
        if ((++spins & 255u) == 0 &&
            (clock64() - t0 > GEN_TIMEOUT_CYCLES || *reinterpret_cast<volatile int*>(err) != 0)) {
            *reinterpret_cast<volatile int*>(err) = 1;
            *reinterpret_cast<volatile int*>(abort_s) = 1;
            break;
        }
    }
#pragma unroll
    for (int it = 0; it < FAST_MAXI; ++it)
        if (it < n_iter) {
            v[it][0] = __uint_as_float(a[it].a.x); v[it][1] = __uint_as_float(a[it].b.x);
            v[it][2] = __uint_as_float(b[it].a.x); v[it][3] = __uint_as_float(b[it].b.x);
        }
}
// Same for the 2-tap conv input: iteration `it` needs channels (r0, r0+1), r0 = first_r + it*64, from two ring slots
// (time t-d with tag_old unless the history is still empty, time t with tag_cur unless `cur` comes from elsewhere).
__device__ __forceinline__ void poll_taps(const uint2* old_slot, unsigned tag_old, bool have_old, const uint2* cur_slot,
                                          unsigned tag_cur, bool have_cur, int first_r, int n_iter,
                                          float (&o)[FAST_MAXI][2], float (&c)[FAST_MAXI][2], int* err, int* abort_s) {
    Pair2 a[FAST_MAXI], b[FAST_MAXI];
    const long long t0 = clock64();
    for (;;) {
#pragma unroll
        for (int it = 0; it < FAST_MAXI; ++it)
            if (it < n_iter) {
                if (have_old) a[it] = ld_pair2(old_slot + first_r + it * 64);
                if (have_cur) b[it] = ld_pair2(cur_slot + first_r + it * 64);
            }
        bool ok = true;
#pragma unroll
        for (int it = 0; it < FAST_MAXI; ++it)
            if (it < n_iter) {
                if (have_old) ok = ok && a[it].a.y == tag_old && a[it].b.y == tag_old;
                if (have_cur) ok = ok && b[it].a.y == tag_cur && b[it].b.y == tag_cur;
            }
        if (ok) break;
        if (clock64() - t0 > GEN_TIMEOUT_CYCLES || *reinterpret_cast<volatile int*>(err) != 0) {
            *reinterpret_cast<volatile int*>(err) = 1;
            *reinterpret_cast<volatile int*>(abort_s) = 1;
            break;
        }
    }
#pragma unroll
    for (int it = 0; it < FAST_MAXI; ++it)
        if (it < n_iter) {
            o[it][0] = have_old ? __uint_as_float(a[it].a.x) : 0.f;
            o[it][1] = have_old ? __uint_as_float(a[it].b.x) : 0.f;
            if (have_cur) { c[it][0] = __uint_as_float(b[it].a.x); c[it][1] = __uint_as_float(b[it].b.x); }
        }
}

#define WORKER_SYNC() asm volatile("bar.sync 1, 256;" ::: "memory")
__device__ __forceinline__ void mbar_arrive_(unsigned long long* b) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}

template <bool PREFETCH, bool TRACE>
__global__ void __launch_bounds__(GEN_NT + 32, 1) gen_kernel_fast(const GenParams p) {
    extern __shared__ __align__(16) float sm[];
    float* part = sm;                                   // [2][GEN_WARPS] partial sums, double buffered by stage parity
    float* skacc = part + 2 * GEN_WARPS;                // [nS]
    float* cur_own = skacc + ((p.S / (int)gridDim.x + 3) & ~3);      // [2][nR] layer input at the residual rows this CTA owns
    float* xin = cur_own + 2 * ((p.R / (int)gridDim.x + 3) & ~3);    // [2][XN] the polled input vector of a stage
    const int XN = p.regA;                              // max(R, D, S, E, C) rounded to 4 (set by the host)
    double* cdf = reinterpret_cast<double*>(xin + 2 * XN);                     // [C]
    float* wbuf = reinterpret_cast<float*>(cdf + p.C);                         // [n_wslots][wslot_floats]
    unsigned long long* fullb = reinterpret_cast<unsigned long long*>(wbuf + (size_t)p.n_wslots * p.wslot_floats);
    unsigned long long* emptyb = fullb + 4;             // consumers -> producer: slot may be refilled (8 warps arrive)
    GenLayer* lay_s = reinterpret_cast<GenLayer*>(fullb + 8);
    uint2* old_s = reinterpret_cast<uint2*>(lay_s + p.n_layers);               // [2][R] prefetched old taps (see below)
    int* slot_s = reinterpret_cast<int*>(old_s + 2 * p.R);                     // [NL] ring slot of time t per layer
    int* misc = slot_s + p.n_layers;                                           // [0] current index, [1] abort

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int cta = blockIdx.x, G = gridDim.x;
    const int R = p.R, D = p.D, S = p.S, E = p.E, C = p.C, NL = p.n_layers;
    const int K1 = 2 * R;
    const int nD = D / G, nR = R / G, nS = S / G, nE = E / G, nC = C / G;
    const int oD = cta * nD, oR = cta * nR, oS = cta * nS, oE = cta * nE, oC = cta * nC;
    const int NSLOT = p.n_wslots;
    // fixed warp -> (row, K-part) assignment per stage kind, and this lane's float4 range inside the part
    const int HS1 = GEN_WARPS / (2 * nD), HS2 = GEN_WARPS / (nR + nS), HSA = GEN_WARPS / nE, HSB = GEN_WARPS / nC;
    const int row1 = warp / HS1, g1 = ((warp - row1 * HS1) * (K1 / HS1) >> 2) + lane, n1 = (((K1 / HS1) >> 2) - lane + 31) / 32;
    const int row2 = warp / HS2, g2 = ((warp - row2 * HS2) * (D / HS2) >> 2) + lane, n2 = (((D / HS2) >> 2) - lane + 31) / 32;
    const int rowA = warp / HSA, gA = ((warp - rowA * HSA) * (S / HSA) >> 2) + lane, nA = (((S / HSA) >> 2) - lane + 31) / 32;
    const int rowB = warp / HSB, gB = ((warp - rowB * HSB) * (E / HSB) >> 2) + lane, nB = (((E / HSB) >> 2) - lane + 31) / 32;

    {
        const int* src = reinterpret_cast<const int*>(p.layers);
        int* dst = reinterpret_cast<int*>(lay_s);
        for (int i = tid; i < NL * (int)(sizeof(GenLayer) / sizeof(int)); i += GEN_NT + 32) dst[i] = src[i];
    }
    if (tid == 0) {
        misc[0] = p.cur_idx[0];
        misc[1] = 0;
        if (PREFETCH)
            for (int i = 0; i < NSLOT; ++i) { mbar_init(fullb + i, 1); mbar_init(emptyb + i, GEN_WARPS); }
    }
    if (PREFETCH) asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    for (int l = tid; l < NL; l += GEN_NT) {          // slot of time t0-1, advanced at the top of every evaluation
        const int len = lay_s[l].ring_len;
        slot_s[l] = (p.t0 + len - 1) % len;
    }
    // ---- weight prefetch: a dedicated producer warp (warp 8) runs ahead of the 8 worker warps through the same stage
    // sequence as gen_kernel_ll (all rows of a stage are always fetched); full[slot] = bytes landed, empty[slot] = all
    // worker warps are done with the slot.  Keeping the producer off the worker warps matters: every stage needs every
    // worker warp's row, so anything a worker lane does besides its row is on the critical path of the whole GPU.
    int* abort_s = misc + 1;
    const unsigned smask = (unsigned)NSLOT - 1u, sshift = (NSLOT == 4) ? 2u : 1u;
    if (warp == GEN_WARPS) {
        if (PREFETCH && lane == 0) {
            unsigned q = 0;
            for (int ev = 0; ev < p.n_evals; ++ev) {
                const bool wh = (p.t0 + ev >= p.n_given - 1);
                const int n_st = wh ? 2 * NL + 2 : 2 * NL;
                for (int st = 0; st < n_st; ++st, ++q) {
                    StageDesc d = stage_desc(p, st, true, nD, nR, nS, nE, nC);
                    if (st < 2 * NL && (st & 1)) { d.n_first = nR; d.n = nR + nS; }
                    const int slot = (int)(q & smask);
                    if (q >= (unsigned)NSLOT) {                       // wait until the workers released this slot
                        const unsigned par = ((q >> sshift) & 1u) ^ 1u;
                        unsigned done = 0, spins = 0;
                        while (!done) {
                            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                                         : "=r"(done) : "r"(smem_u32(emptyb + slot)), "r"(par) : "memory");
                            if (!done && (++spins & 1023u) == 0 && *reinterpret_cast<volatile int*>(abort_s)) return;
                        }
                    }
                    mbar_expect_tx(fullb + slot, (unsigned)(d.n * d.K * 4));
                    float* dst = wbuf + (size_t)slot * p.wslot_floats;
                    for (int i = 0; i < d.n; ++i)
                        bulk_g2s(dst + (size_t)i * d.K, stage_row(p, lay_s, st, d, i, cta, G), d.K * 4, fullb + slot);
                }
            }
        }
        return;
    }
    unsigned cons_q = 0;
    // weights of (stage, row): shared-memory slot when prefetching, else the parameter tensor itself
    auto stage_weights = [&](int st, int row, int K) -> const float* {
        if (PREFETCH) {
            const int slot = (int)(cons_q & smask);
            mbar_wait(fullb + slot, (cons_q >> sshift) & 1u);
            return wbuf + (size_t)slot * p.wslot_floats + (size_t)row * K;
        }
        StageDesc d = stage_desc(p, st, true, nD, nR, nS, nE, nC);
        if (st < 2 * NL && (st & 1)) { d.n_first = nR; d.n = nR + nS; }
        return stage_row(p, lay_s, st, d, row, cta, G);
    };
    auto ldw = [&](const float* w, int i4) -> float4 {
        if (PREFETCH) return reinterpret_cast<const float4*>(w)[i4];
        return __ldg(reinterpret_cast<const float4*>(w) + i4);
    };
    auto release_slot = [&]() {                       // this warp is done reading the weight slot of the current stage
        if (PREFETCH) { __syncwarp(); if (lane == 0) mbar_arrive_(emptyb + (cons_q & smask)); }
        ++cons_q;
    };
    // One CTA-wide poll of a published vector: warps 4..7 (which never have epilogue work, so they are free the moment
    // the dot barrier opens) fetch N {value,tag} pairs ONCE per CTA -- 8x fewer L2 requests on the hot lines than every
    // warp polling its own operands, which measured as the dominant cost -- and leave the values in shared memory.
    auto poll_vector = [&](const uint2* src, int N, unsigned tg, float* dst, bool relu) {
        if (warp >= 4) {
            for (int j = tid - 128; 2 * j < N; j += 128) {
                float a, b;
                poll2(src + 2 * j, tg, a, b, p.err, abort_s);
                if (relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
                *reinterpret_cast<float2*>(dst + 2 * j) = make_float2(a, b);
            }
        }
    };
    unsigned stage_par = 0;
    WORKER_SYNC();
    // Old taps (the ring slot of time t-d) were written >= 1 evaluation ago; they are fetched one stage ahead with
    // cp.async into shared memory: during stage 2 of layer l for layer l+1 (or for layer 0 of the next evaluation).
    auto prefetch_old = [&](int ln, int te, int slot_te) {        // slot_te = ring slot of time te in layer ln
        const GenLayer& Lp = lay_s[ln];
        if (te >= Lp.dil && tid < R / 2) {
            const int so = (slot_te + 1 == Lp.ring_len) ? 0 : slot_te + 1;
            const uint2* src = p.ringLL + Lp.ring_off + (size_t)so * R + 2 * tid;
            const unsigned dst = (unsigned)__cvta_generic_to_shared(old_s + (ln & 1) * R + 2 * tid);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    {
        const int len0 = lay_s[0].ring_len;
        prefetch_old(0, p.t0, p.t0 % len0);
        asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    WORKER_SYNC();

    for (int ev = 0; ev < p.n_evals; ++ev) {
        const int t = p.t0 + ev;
        const unsigned tag = (unsigned)t + 1u;
        const int par = t & 1;
        const float* ct = p.cond ? cond_at(p, t, D) : nullptr;
        const bool want_head = (t >= p.n_given - 1);
        const int samp = t - (p.n_given - 1);
        if (tid == 0) {
            if (t < p.n_given) misc[0] = p.first[t];
            else if (p.forced != nullptr) misc[0] = p.forced[t - p.n_given];
        }
        for (int l = tid; l < NL; l += GEN_NT) {
            const int s1 = slot_s[l] + 1;
            slot_s[l] = (s1 == lay_s[l].ring_len) ? 0 : s1;
        }
        for (int i = tid; i < nS; i += GEN_NT) skacc[i] = 0.f;
        WORKER_SYNC();
        if (*abort_s) return;
        int idx = misc[0];
        idx = idx < 0 ? 0 : (idx >= C ? C - 1 : idx);
        const bool tr_on = TRACE && p.trace != nullptr && cta == 0 && tid == 0 && ev == p.n_evals - 1;
        int tr_n = 0;
#define TR() do { if (TRACE) { if (tr_on && tr_n < 2040) p.trace[tr_n++] = clock64(); } } while (0)
        TR();

        for (int l = 0; l < NL; ++l) {
            const GenLayer& L = lay_s[l];
            uint2* ring = p.ringLL + L.ring_off;
            const int slot_t = slot_s[l];
            const int slot_old = (slot_t + 1 == L.ring_len) ? 0 : slot_t + 1;          // time t-d with len = d+1
            const bool have_old = (t >= L.dil);
            const unsigned tag_old = (unsigned)(t - L.dil) + 1u;
            float* cur_l = cur_own + (l & 1) * ((nR + 3) & ~3);
            float* xc = xin + stage_par * XN;
            // ================= stage 1 inputs: the layer's current input vector (R values) -> xc
            if (warp >= 4) {
                for (int j = tid - 128; 2 * j < R; j += 128) {
                    const int r0 = 2 * j;
                    float c0, c1;
                    if (l == 0) {                                  // start conv column of the current sample index
                        c0 = __ldg(p.start_w + (size_t)r0 * C + idx) + (p.start_b ? __ldg(p.start_b + r0) : 0.f);
                        c1 = __ldg(p.start_w + (size_t)(r0 + 1) * C + idx) + (p.start_b ? __ldg(p.start_b + r0 + 1) : 0.f);
                        if (r0 >= oR && r0 < oR + nR) st_pair(ring + (size_t)slot_t * R + r0, c0, tag);          // enqueue
                        if (r0 + 1 >= oR && r0 + 1 < oR + nR) st_pair(ring + (size_t)slot_t * R + r0 + 1, c1, tag);
                    } else {
                        poll2(ring + (size_t)slot_t * R + r0, tag, c0, c1, p.err, abort_s);
                    }
                    if (r0 >= oR && r0 < oR + nR) cur_l[r0 - oR] = c0;
                    if (r0 + 1 >= oR && r0 + 1 < oR + nR) cur_l[r0 + 1 - oR] = c1;
                    *reinterpret_cast<float2*>(xc + r0) = make_float2(c0, c1);
                }
            }
            const float* w1 = stage_weights(2 * l, row1, K1);
            TR();          // 1: own share of the inputs polled (pollers) / weights ready
            WORKER_SYNC();
            // ================= stage 1: filter/gate rows, K = 2R interleaved (old, cur) per channel
            {
                const uint2* os = old_s + (l & 1) * R;
                float acc = 0.f;
                bool old_ok = true;
#pragma unroll
                for (int it = 0; it < FAST_MAXI; ++it)
                    if (it < n1) {
                        const int g4 = g1 + it * 32, r0 = 2 * g4;
                        float o0 = 0.f, o1 = 0.f;
                        if (have_old) {
                            const uint4 q = *reinterpret_cast<const uint4*>(os + r0);
                            old_ok = old_ok && q.y == tag_old && q.w == tag_old;
                            o0 = __uint_as_float(q.x);
                            o1 = __uint_as_float(q.z);
                        }
                        const float2 c = *reinterpret_cast<const float2*>(xc + r0);
                        const float4 w4 = ldw(w1, g4);
                        acc = fmaf(w4.x, o0, acc); acc = fmaf(w4.y, c.x, acc); acc = fmaf(w4.z, o1, acc); acc = fmaf(w4.w, c.y, acc);
                    }
                if (!__all_sync(0xffffffffu, old_ok)) {            // prefetched copy not there yet (rare): poll the ring itself
                    acc = 0.f;
                    for (int it = 0; it < n1; ++it) {
                        const int g4 = g1 + it * 32, r0 = 2 * g4;
                        float o0, o1;
                        poll2(ring + (size_t)slot_old * R + r0, tag_old, o0, o1, p.err, abort_s);
                        const float2 c = *reinterpret_cast<const float2*>(xc + r0);
                        const float4 w4 = ldw(w1, g4);
                        acc = fmaf(w4.x, o0, acc); acc = fmaf(w4.y, c.x, acc); acc = fmaf(w4.z, o1, acc); acc = fmaf(w4.w, c.y, acc);
                    }
                }
                acc = warp_sum(acc);
                if (lane == 0) part[stage_par * GEN_WARPS + warp] = acc;
                release_slot();
            }
            TR();          // 2: stage-1 dot done
            WORKER_SYNC();
            TR();          // 3: barrier passed
            if (*abort_s) return;
            uint2* zl = p.zLL + (size_t)(par * NL + l) * D;
            if (tid < nD) {
                const int c = oD + tid;
                const float* pf = part + stage_par * GEN_WARPS + (2 * tid) * HS1;
                float f = pf[0], g = pf[HS1];
                for (int q = 1; q < HS1; ++q) { f += pf[q]; g += pf[HS1 + q]; }
                if (ct) {                                          // one stream: the table is [n_layers][1][(frames)][2D]
                    f += __ldg(ct + (size_t)l * p.cond_sstride + c);
                    g += __ldg(ct + (size_t)l * p.cond_sstride + D + c);
                } else {
                    f += L.bf ? __ldg(L.bf + c) : 0.f;
                    g += L.bg ? __ldg(L.bg + c) : 0.f;
                }
                st_pair(zl + c, tanh_(f) * sigmoid_(g), tag);
            }
            TR();          // 4: z published
            stage_par ^= 1;
            // ================= stage 2 inputs: z of all CTAs -> xz; old taps of the next stage 1 start flying now
            float* xz = xin + stage_par * XN;
            const bool active2 = (row2 < nR) ? (l + 1 < NL) : want_head;
            if (l + 1 < NL) prefetch_old(l + 1, t, slot_s[l + 1]);
            else if (ev + 1 < p.n_evals) prefetch_old(0, t + 1, (slot_s[0] + 1 == lay_s[0].ring_len) ? 0 : slot_s[0] + 1);
            poll_vector(zl, D, tag, xz, false);
            const float* w2 = stage_weights(2 * l + 1, row2, D);
            TR();          // 5: own share of z polled
            WORKER_SYNC();
            // ================= stage 2: residual rows (first nR) and skip rows (next nS), K = D
            {
                float acc = 0.f;
                if (active2) {
#pragma unroll
                    for (int it = 0; it < FAST_MAXI; ++it)
                        if (it < n2) {
                            const float4 z4 = *reinterpret_cast<const float4*>(xz + 4 * (g2 + it * 32));
                            const float4 w4 = ldw(w2, g2 + it * 32);
                            acc = fmaf(w4.x, z4.x, acc); acc = fmaf(w4.y, z4.y, acc); acc = fmaf(w4.z, z4.z, acc); acc = fmaf(w4.w, z4.w, acc);
                        }
                    acc = warp_sum(acc);
                }
                if (lane == 0) part[stage_par * GEN_WARPS + warp] = acc;
                release_slot();
                asm volatile("cp.async.wait_group 0;" ::: "memory");      // the old taps for the next stage 1 have landed
            }
            TR();          // 6: stage-2 dot done
            WORKER_SYNC();
            TR();          // 7: barrier passed
            if (*abort_s) return;
            if (tid < nR + nS) {
                const float* ps = part + stage_par * GEN_WARPS + tid * HS2;
                float v = ps[0];
                for (int q = 1; q < HS2; ++q) v += ps[q];
                if (tid < nR) {
                    if (l + 1 < NL) {
                        const int row = oR + tid;
                        const GenLayer& Ln = lay_s[l + 1];
                        v += L.br ? __ldg(L.br + row) : 0.f;
                        st_pair(p.ringLL + Ln.ring_off + (size_t)slot_s[l + 1] * R + row, v + cur_l[tid], tag);
                    }
                } else if (want_head) {
                    const int li = tid - nR, row = oS + li;
                    v += L.bs ? __ldg(L.bs + row) : 0.f;
                    skacc[li] = v + skacc[li];
                }
            }
            TR();          // 8: h' published
            stage_par ^= 1;
            // no barrier here: part, xin and cur_own are double buffered, and their next writers sit behind a barrier
            // that this epilogue's threads must reach first
        }
        if (!want_head) continue;

        // ================= head
        uint2* skl = p.skipLL + (size_t)par * S;
        if (tid >= nR && tid < nR + nS) st_pair(skl + oS + (tid - nR), skacc[tid - nR], tag);   // same thread that summed it
        uint2* yl = p.y1LL + (size_t)par * E;
        {
            float* xs = xin + stage_par * XN;
            poll_vector(skl, S, tag, xs, true);
            const float* w = stage_weights(2 * NL, rowA, S);
            WORKER_SYNC();
            float acc = 0.f;
#pragma unroll
            for (int it = 0; it < FAST_MAXI; ++it)
                if (it < nA) {
                    const float4 z4 = *reinterpret_cast<const float4*>(xs + 4 * (gA + it * 32));
                    const float4 w4 = ldw(w, gA + it * 32);
                    acc = fmaf(w4.x, z4.x, acc); acc = fmaf(w4.y, z4.y, acc); acc = fmaf(w4.z, z4.z, acc); acc = fmaf(w4.w, z4.w, acc);
                }
            acc = warp_sum(acc);
            if (lane == 0) part[stage_par * GEN_WARPS + warp] = acc;
            release_slot();
        }
        WORKER_SYNC();
        if (*abort_s) return;
        if (tid < nE) {
            const int row = oE + tid;
            const float* ps = part + stage_par * GEN_WARPS + tid * HSA;
            float v = ps[0];
            for (int q = 1; q < HSA; ++q) v += ps[q];
            st_pair(yl + row, fmaxf(v + __ldg(p.e1b + row), 0.f), tag);
        }
        stage_par ^= 1;
        uint2* lgl = p.logitLL + (size_t)par * C;
        {
            float* xs = xin + stage_par * XN;
            poll_vector(yl, E, tag, xs, false);
            const float* w = stage_weights(2 * NL + 1, rowB, E);
            WORKER_SYNC();
            float acc = 0.f;
#pragma unroll
            for (int it = 0; it < FAST_MAXI; ++it)
                if (it < nB) {
                    const float4 z4 = *reinterpret_cast<const float4*>(xs + 4 * (gB + it * 32));
                    const float4 w4 = ldw(w, gB + it * 32);
                    acc = fmaf(w4.x, z4.x, acc); acc = fmaf(w4.y, z4.y, acc); acc = fmaf(w4.z, z4.z, acc); acc = fmaf(w4.w, z4.w, acc);
                }
            acc = warp_sum(acc);
            if (lane == 0) part[stage_par * GEN_WARPS + warp] = acc;
            release_slot();
        }
        WORKER_SYNC();
        if (*abort_s) return;
        if (tid < nC) {
            const int row = oC + tid;
            const float* ps = part + stage_par * GEN_WARPS + tid * HSB;
            float v = ps[0];
            for (int q = 1; q < HSB; ++q) v += ps[q];
            const float dc = (float)row - (float)C / 2.f;
            v = (v + __ldg(p.e2b + row)) - (dc * dc) * p.regularize;
            st_pair(lgl + row, v, tag);
            if (p.out_logits) p.out_logits[(size_t)samp * C + row] = v;
        }
        stage_par ^= 1;
        // ---- all logits -> shared memory (cooperative poll), then warp 0 chooses
        float* logit_s = xin + stage_par * XN;
        poll_vector(lgl, C, tag, logit_s, false);
        WORKER_SYNC();
        if (*abort_s) return;
        if (warp == 0) {
            const int choice = p.trunc ? choose_truncated(logit_s, reinterpret_cast<unsigned*>(cdf),
                                                          reinterpret_cast<float*>(cdf) + C, C, lane, p.temperature,
                                                          p.top_k, p.top_p, p.uniforms + samp)
                                       : choose_sample(logit_s, cdf, C, lane, p.temperature, p.uniforms ? p.uniforms + samp : nullptr);
            if (lane == 0) {
                misc[0] = choice;
                if (cta == 0) p.out_idx[samp] = choice;
            }
        }
        stage_par ^= 1;
        // the top-of-evaluation barrier publishes misc[0]
    }
    WORKER_SYNC();
    if (cta == 0 && tid == 0) p.cur_idx[0] = misc[0];
}

// ================================================================================================ cluster kernel
// One thread-block cluster (16 CTAs) per stream.  The stage-to-stage exchange no longer goes through the L2: a CTA
// that has computed a value stores the {value, tag} pair straight into the shared memory of all 16 CTAs of its
// cluster (distributed shared memory), and consumers spin on their OWN shared memory, which is closer than an L2
// all-to-all (tools/lat_probe.cu measures both).
//   stage 1 (conv rows)   warp-local: local poll of the layer input -> 4 rows per warp over the full K -> warp reduce ->
//                         every lane recomputes z of the warp's 2 channels and stores it to one of the 16 CTAs
//   stage 2 (1x1 rows)    warps 0-3 residual rows, warps 4-7 skip rows; one CTA barrier per layer before h' is
//                         published keeps slow warps from being overtaken (buffers are double buffered by layer parity)
//   head                  skip -> end_conv_1 -> end_conv_2 -> every CTA holds all logits; rank 0 records the choice
// Clusters do not talk to each other, so a launch may hold any number of streams (they run in waves of co-resident
// clusters) and needs no cooperative launch.  History (ring slots of time t-d) still lives in global memory and is
// fetched one stage ahead with cp.async, as in gen_kernel_fast; weights stream through a TMA ring fed by warp 8.
constexpr int CL = 16;                      // CTAs per cluster
constexpr int CL_ROWS = 4;                  // max rows per warp per stage

__device__ __forceinline__ unsigned cluster_rank() {
    unsigned r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// {value, tag} into the same shared-memory offset of CTA `dst` of this cluster
__device__ __forceinline__ void st_remote_pair(const void* local_ptr, unsigned dst, float v, unsigned tag) {
    unsigned laddr = smem_u32(local_ptr), raddr;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(laddr), "r"(dst));
    const unsigned long long w = ((unsigned long long)tag << 32) | (unsigned long long)__float_as_uint(v);
    asm volatile("st.shared::cluster.b64 [%0], %1;" ::"r"(raddr), "l"(w) : "memory");
}
// local spin on a shared-memory {value, tag} pair (volatile: the writer is another SM)
__device__ __forceinline__ float wait_local(const uint2* p, unsigned tag, int* abort_s) {
    const volatile unsigned long long* vp = reinterpret_cast<const volatile unsigned long long*>(p);
    unsigned long long w = *vp;
    if ((unsigned)(w >> 32) != tag) {
        const long long t0 = clock64();
        unsigned spins = 0;
        do {
            w = *vp;
            if ((++spins & 1023u) == 0 && clock64() - t0 > GEN_TIMEOUT_CYCLES) asm volatile("trap;");   // never hang the GPU
        } while ((unsigned)(w >> 32) != tag);
    }
    return __uint_as_float((unsigned)w);
}

__global__ void __launch_bounds__(GEN_NT + 32, 1) gen_kernel_cluster(const GenParams p) {
    extern __shared__ __align__(16) float sm[];
    // exchange buffers first: they must sit at the same offset in every CTA (mapa keeps the offset)
    uint2* xcur = reinterpret_cast<uint2*>(sm);                  // [2][R]  layer input (h), by layer parity
    uint2* xz = xcur + 2 * p.R;                                  // [2][D]  gated activation z, by layer parity
    uint2* xhead = xz + 2 * p.D;                                 // [S + E + C] skip, y1, logits of the current evaluation
    uint2* old_s = xhead + (p.S + p.E + p.C);                    // [2][R] prefetched old taps
    float* skacc = reinterpret_cast<float*>(old_s + 2 * p.R);    // [S/CL]
    float* cur_own = skacc + ((p.S / CL + 3) & ~3);              // [2][R/CL]
    float* part = cur_own + 2 * ((p.R / CL + 3) & ~3);           // [E/CL + C/CL + 32] row sums of the head stages
    float* logit_s = part + (((p.E + p.C) / CL + 32 + 3) & ~3);  // [C]
    double* cdf = reinterpret_cast<double*>(logit_s + ((p.C + 3) & ~3));      // [C]
    float* wbuf = reinterpret_cast<float*>(cdf + p.C);                        // [n_wslots][wslot_floats]
    unsigned long long* fullb = reinterpret_cast<unsigned long long*>(wbuf + (size_t)p.n_wslots * p.wslot_floats);
    unsigned long long* emptyb = fullb + 4;
    GenLayer* lay_s = reinterpret_cast<GenLayer*>(fullb + 8);
    int* slot_s = reinterpret_cast<int*>(lay_s + p.n_layers);
    int* misc = slot_s + p.n_layers;                             // [0] current index, [1] abort

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rank = (int)cluster_rank();
    const int stream = blockIdx.x / CL, NS = p.NS;
    const int R = p.R, D = p.D, S = p.S, E = p.E, C = p.C, NL = p.n_layers;
    const int K1 = 2 * R;
    const int nD = D / CL, nR = R / CL, nS = S / CL, nE = E / CL, nC = C / CL;
    const int oD = rank * nD, oR = rank * nR, oS = rank * nS, oE = rank * nE, oC = rank * nC;
    const int NSLOT = p.n_wslots;
    const int rw1 = 2 * nD / GEN_WARPS, rw2 = (nR + nS) / GEN_WARPS;       // rows per warp in stage 1 / stage 2 (<= CL_ROWS)

    {   // zero the exchange buffers (tag 0 = nothing yet), copy the layer table
        unsigned long long* z0 = reinterpret_cast<unsigned long long*>(xcur);
        const int n0 = 2 * R + 2 * D + S + E + C + 2 * R;
        for (int i = tid; i < n0; i += GEN_NT + 32) z0[i] = 0ull;
        const int* src = reinterpret_cast<const int*>(p.layers);
        int* dst = reinterpret_cast<int*>(lay_s);
        for (int i = tid; i < NL * (int)(sizeof(GenLayer) / sizeof(int)); i += GEN_NT + 32) dst[i] = src[i];
    }
    if (tid == 0) {
        misc[0] = p.cur_idx[stream];
        misc[1] = 0;
        for (int i = 0; i < NSLOT; ++i) { mbar_init(fullb + i, 1); mbar_init(emptyb + i, GEN_WARPS); }
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    for (int l = tid; l < NL; l += GEN_NT) {
        const int len = lay_s[l].ring_len;
        slot_s[l] = (p.t0 + len - 1) % len;
    }
    cluster_sync_all();                                          // nobody may store into a peer before it is zeroed
    int* abort_s = misc + 1;
    const unsigned smask = (unsigned)NSLOT - 1u, sshift = (NSLOT == 4) ? 2u : 1u;

    // ---- producer warp: weight rows of this CTA for every stage, in order, through the TMA ring
    if (warp == GEN_WARPS) {
        if (lane == 0) {
            unsigned q = 0;
            for (int ev = 0; ev < p.n_evals; ++ev) {
                const bool wh = head_at(p, p.t0 + ev);
                const int n_st = wh ? 2 * NL + 2 : 2 * NL;
                for (int st = 0; st < n_st; ++st, ++q) {
                    StageDesc d = stage_desc(p, st, true, nD, nR, nS, nE, nC);
                    if (st < 2 * NL && (st & 1)) { d.n_first = nR; d.n = nR + nS; }
                    const int slot = (int)(q & smask);
                    if (q >= (unsigned)NSLOT) {
                        const unsigned par = ((q >> sshift) & 1u) ^ 1u;
                        unsigned done = 0, spins = 0;
                        while (!done) {
                            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                                         : "=r"(done) : "r"(smem_u32(emptyb + slot)), "r"(par) : "memory");
                            if (!done && ++spins > (1u << 30)) asm volatile("trap;");
                        }
                    }
                    mbar_expect_tx(fullb + slot, (unsigned)(d.n * d.K * 4));
                    float* dst = wbuf + (size_t)slot * p.wslot_floats;
                    for (int i = 0; i < d.n; ++i)
                        bulk_g2s(dst + (size_t)i * d.K, stage_row(p, lay_s, st, d, i, rank, CL), d.K * 4, fullb + slot);
                }
            }
        }
        cluster_sync_all();                                      // matches the workers' final cluster barrier
        return;
    }
    unsigned cons_q = 0;
    auto stage_weights = [&](int row, int K) -> const float* {
        const int slot = (int)(cons_q & smask);
        mbar_wait(fullb + slot, (cons_q >> sshift) & 1u);
        return wbuf + (size_t)slot * p.wslot_floats + (size_t)row * K;
    };
    auto release_slot = [&]() {
        __syncwarp();
        if (lane == 0) mbar_arrive_(emptyb + (cons_q & smask));
        ++cons_q;
    };
    const size_t ring_stream = (size_t)stream * R;               // ring element (slot, stream, r): (slot*NS + stream)*R + r
    auto prefetch_old = [&](int ln, int te, int slot_te) {
        const GenLayer& Lp = lay_s[ln];
        if (te >= Lp.dil && tid < R / 2) {
            const int so = (slot_te + 1 == Lp.ring_len) ? 0 : slot_te + 1;
            const uint2* src = p.ringLL + Lp.ring_off + (size_t)so * NS * R + ring_stream + 2 * tid;
            const unsigned dst = (unsigned)__cvta_generic_to_shared(old_s + (ln & 1) * R + 2 * tid);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    prefetch_old(0, p.t0, p.t0 % lay_s[0].ring_len);
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    WORKER_SYNC();
    unsigned seq = (unsigned)p.t0 * (unsigned)(2 * NL + 4);      // exchange tag counter, unique per (evaluation, stage)

    for (int ev = 0; ev < p.n_evals; ++ev) {
        const int t = p.t0 + ev;
        const unsigned rtag = (unsigned)t + 1u;                  // ring tag of time t
        const float* ct = p.cond ? p.cond + cond_row(p, stream, t, D) : nullptr;     // this stream's row of evaluation t
        const bool want_head = head_at(p, t);
        if (tid == 0) {
            int v;
            if (given_input(p, stream, t, v)) misc[0] = v;
        }
        for (int l = tid; l < NL; l += GEN_NT) {
            const int s1 = slot_s[l] + 1;
            slot_s[l] = (s1 == lay_s[l].ring_len) ? 0 : s1;
        }
        for (int i = tid; i < nS; i += GEN_NT) skacc[i] = 0.f;
        asm volatile("cp.async.wait_group 0;" ::: "memory");    // layer 0's history, requested at the end of the last evaluation
        WORKER_SYNC();
        int idx = misc[0];
        idx = idx < 0 ? 0 : (idx >= C ? C - 1 : idx);
        const unsigned etag = seq + 1u;                          // tags of this evaluation: etag + 2l (cur), etag + 2l + 1 (z)
        seq += (unsigned)(2 * NL + 4);

        // layer 0's input: the start-conv column, computed locally by every CTA; owners also enqueue it
        {
            const GenLayer& L0 = lay_s[0];
            for (int r = tid; r < R; r += GEN_NT) {
                const float v = __ldg(p.start_w + (size_t)r * C + idx) + (p.start_b ? __ldg(p.start_b + r) : 0.f);
                reinterpret_cast<unsigned long long*>(xcur)[r] =
                    ((unsigned long long)etag << 32) | (unsigned long long)__float_as_uint(v);
                if (r >= oR && r < oR + nR)
                    st_pair(p.ringLL + L0.ring_off + ((size_t)slot_s[0] * NS) * R + ring_stream + r, v, rtag);
            }
        }
        WORKER_SYNC();

        for (int l = 0; l < NL; ++l) {
            const GenLayer& L = lay_s[l];
            const bool have_old = (t >= L.dil);
            const unsigned tag_old = (unsigned)(t - L.dil) + 1u, tag_cur = etag + 2u * (unsigned)l, tag_z = tag_cur + 1u;
            const uint2* xc = xcur + (l & 1) * R;
            const uint2* os = old_s + (l & 1) * R;
            uint2* zbuf = xz + (l & 1) * D;
            float* cur_l = cur_own + (l & 1) * ((nR + 3) & ~3);
            // ================= stage 1: rows [warp*rw1, +rw1) of this CTA's 2*nD conv rows, full K, warp-local
            {
                const float* w = stage_weights(warp * rw1, K1);
                float acc[CL_ROWS];
#pragma unroll
                for (int j = 0; j < CL_ROWS; ++j) acc[j] = 0.f;
                for (int g4 = lane; g4 < (K1 >> 2); g4 += 32) {
                    const int r0 = 2 * g4;
                    float o0 = 0.f, o1 = 0.f;
                    if (have_old) {
                        uint4 q = *reinterpret_cast<const uint4*>(os + r0);
                        if (q.y != tag_old || q.w != tag_old) {          // prefetched copy not there yet (rare): go to the ring
                            const int so = (slot_s[l] + 1 == L.ring_len) ? 0 : slot_s[l] + 1;
                            poll2(p.ringLL + L.ring_off + (size_t)so * NS * R + ring_stream + r0, tag_old, o0, o1, p.err, abort_s);
                        } else {
                            o0 = __uint_as_float(q.x);
                            o1 = __uint_as_float(q.z);
                        }
                    }
                    const float c0 = wait_local(xc + r0, tag_cur, abort_s), c1 = wait_local(xc + r0 + 1, tag_cur, abort_s);
                    if (r0 >= oR && r0 < oR + nR) cur_l[r0 - oR] = c0;           // every warp writes the same values
                    if (r0 + 1 >= oR && r0 + 1 < oR + nR) cur_l[r0 + 1 - oR] = c1;
#pragma unroll
                    for (int j = 0; j < CL_ROWS; ++j)
                        if (j < rw1) {
                            const float4 w4 = reinterpret_cast<const float4*>(w + (size_t)j * K1)[g4];
                            float a = acc[j];
                            a = fmaf(w4.x, o0, a); a = fmaf(w4.y, c0, a); a = fmaf(w4.z, o1, a); a = fmaf(w4.w, c1, a);
                            acc[j] = a;
                        }
                }
#pragma unroll
                for (int j = 0; j < CL_ROWS; ++j)
                    if (j < rw1) acc[j] = warp_sum(acc[j]);
                release_slot();
                // rows come in (filter, gate) pairs: channel ci = (warp*rw1 + 2*jj)/2; every lane recomputes z and
                // lane -> (channel jj = lane / 16, destination CTA = lane % 16)
                const int dst = lane & 15;
#pragma unroll
                for (int jj = 0; jj < CL_ROWS / 2; ++jj)
                    if (2 * jj < rw1 && ((lane >> 4) == (jj & 1))) {
                        const int ci = (warp * rw1 >> 1) + jj, c = oD + ci;
                        const float* cb = ct ? ct + ((size_t)l * NS + stream) * p.cond_sstride : nullptr;
                        const float f = acc[2 * jj] + (cb ? __ldg(cb + c) : (L.bf ? __ldg(L.bf + c) : 0.f));
                        const float g = acc[2 * jj + 1] + (cb ? __ldg(cb + D + c) : (L.bg ? __ldg(L.bg + c) : 0.f));
                        st_remote_pair(zbuf + c, (unsigned)dst, tanh_(f) * sigmoid_(g), tag_z);
                    }
            }
            // ================= stage 2: warps [0, nR/rw2) residual rows, the rest skip rows; K = D
            {
                if (l + 1 < NL) prefetch_old(l + 1, t, slot_s[l + 1]);
                const int row0 = warp * rw2;
                const bool is_res = row0 < nR;
                const bool active = is_res ? (l + 1 < NL) : want_head;
                const float* w = stage_weights(row0, D);
                float acc[CL_ROWS];
#pragma unroll
                for (int j = 0; j < CL_ROWS; ++j) acc[j] = 0.f;
                if (active) {
                    for (int g4 = lane; g4 < (D >> 2); g4 += 32) {
                        const float z0 = wait_local(zbuf + 4 * g4, tag_z, abort_s), z1 = wait_local(zbuf + 4 * g4 + 1, tag_z, abort_s);
                        const float z2 = wait_local(zbuf + 4 * g4 + 2, tag_z, abort_s), z3 = wait_local(zbuf + 4 * g4 + 3, tag_z, abort_s);
#pragma unroll
                        for (int j = 0; j < CL_ROWS; ++j)
                            if (j < rw2) {
                                const float4 w4 = reinterpret_cast<const float4*>(w + (size_t)j * D)[g4];
                                float a = acc[j];
                                a = fmaf(w4.x, z0, a); a = fmaf(w4.y, z1, a); a = fmaf(w4.z, z2, a); a = fmaf(w4.w, z3, a);
                                acc[j] = a;
                            }
                    }
#pragma unroll
                    for (int j = 0; j < CL_ROWS; ++j)
                        if (j < rw2) acc[j] = warp_sum(acc[j]);
                }
                release_slot();
                asm volatile("cp.async.wait_group 0;" ::: "memory");
                // all warps of this CTA are past their reads of z(l) and h(l) before h'(l) leaves (see header comment)
                WORKER_SYNC();
                if (l + 1 == NL && ev + 1 < p.n_evals)       // history of the next evaluation's layer 0 (buffer 0 is free now)
                    prefetch_old(0, t + 1, (slot_s[0] + 1 == lay_s[0].ring_len) ? 0 : slot_s[0] + 1);
                        if (is_res) {
                    if (l + 1 < NL) {
                        const GenLayer& Ln = lay_s[l + 1];
                        uint2* xn = xcur + ((l + 1) & 1) * R;
                        const unsigned tag_n = tag_cur + 2u;
                        // lane -> (row j = lane / 16 + 2*pass, destination CTA = lane % 16)
#pragma unroll
                        for (int ps = 0; ps < CL_ROWS / 2; ++ps) {
                            const int j = (lane >> 4) + 2 * ps;
                            if (j < rw2) {
                                const int li = row0 + j, row = oR + li;
                                float v = (j == 0) ? acc[0] : (j == 1) ? acc[1] : (j == 2) ? acc[2] : acc[3];
                                v += L.br ? __ldg(L.br + row) : 0.f;
                                v += cur_l[li];
                                st_remote_pair(xn + row, (unsigned)(lane & 15), v, tag_n);
                                if ((lane & 15) == 0)                      // history for the taps d steps from now
                                    st_pair(p.ringLL + Ln.ring_off + ((size_t)slot_s[l + 1] * NS) * R + ring_stream + row, v, rtag);
                            }
                        }
                    }
                } else if (want_head && lane == 0) {
#pragma unroll
                    for (int j = 0; j < CL_ROWS; ++j)
                        if (j < rw2) {
                            const int li = row0 + j - nR, row = oS + li;
                            const float v = acc[j] + (L.bs ? __ldg(L.bs + row) : 0.f);
                            skacc[li] = v + skacc[li];
                        }
                }
            }
        }
        if (!want_head) continue;

        // ================= head (3 exchanges per evaluation; rows spread one per warp-iteration)
        const unsigned tag_s = etag + 2u * (unsigned)NL + 1u, tag_y = tag_s + 1u, tag_l = tag_s + 2u;
        uint2* xs = xhead, *xy = xhead + S, *xl = xhead + S + E;
        WORKER_SYNC();                                           // skacc complete (written by the skip warps' lane 0)
        for (int i = tid; i < nS * CL; i += GEN_NT) st_remote_pair(xs + oS + (i >> 4), (unsigned)(i & 15), skacc[i >> 4], tag_s);
        {
            const float* w = stage_weights(0, S);
            for (int it = warp; it < nE; it += GEN_WARPS) {
                float acc = 0.f;
                for (int g4 = lane; g4 < (S >> 2); g4 += 32) {
                    const float4 w4 = reinterpret_cast<const float4*>(w + (size_t)it * S)[g4];
                    acc = fmaf(w4.x, fmaxf(wait_local(xs + 4 * g4, tag_s, abort_s), 0.f), acc);
                    acc = fmaf(w4.y, fmaxf(wait_local(xs + 4 * g4 + 1, tag_s, abort_s), 0.f), acc);
                    acc = fmaf(w4.z, fmaxf(wait_local(xs + 4 * g4 + 2, tag_s, abort_s), 0.f), acc);
                    acc = fmaf(w4.w, fmaxf(wait_local(xs + 4 * g4 + 3, tag_s, abort_s), 0.f), acc);
                }
                acc = warp_sum(acc);
                const int row = oE + it;
                if (lane < CL) st_remote_pair(xy + row, (unsigned)lane, fmaxf(acc + __ldg(p.e1b + row), 0.f), tag_y);
            }
            release_slot();
        }
        {
            const float* w = stage_weights(0, E);
            for (int it = warp; it < nC; it += GEN_WARPS) {
                float acc = 0.f;
                for (int g4 = lane; g4 < (E >> 2); g4 += 32) {
                    const float4 w4 = reinterpret_cast<const float4*>(w + (size_t)it * E)[g4];
                    acc = fmaf(w4.x, wait_local(xy + 4 * g4, tag_y, abort_s), acc);
                    acc = fmaf(w4.y, wait_local(xy + 4 * g4 + 1, tag_y, abort_s), acc);
                    acc = fmaf(w4.z, wait_local(xy + 4 * g4 + 2, tag_y, abort_s), acc);
                    acc = fmaf(w4.w, wait_local(xy + 4 * g4 + 3, tag_y, abort_s), acc);
                }
                acc = warp_sum(acc);
                const int row = oC + it;
                const float dc = (float)row - (float)C / 2.f;
                const float v = (acc + __ldg(p.e2b + row)) - (dc * dc) * (p.ps ? p.ps[stream].regularize : p.regularize);
                if (lane < CL) st_remote_pair(xl + row, (unsigned)lane, v, tag_l);
                const int samp = sample_of(p, stream, t);
                if (lane == 0 && p.out_logits && samp >= 0) p.out_logits[((size_t)stream * p.n_samples + samp) * C + row] = v;
            }
            release_slot();
        }
        for (int c = tid; c < C; c += GEN_NT) logit_s[c] = wait_local(xl + c, tag_l, abort_s);
        WORKER_SYNC();
        if (warp == 0) {
            const GenStream ss = stream_set(p, stream);
            const int samp = sample_of(p, stream, t);
            if (samp >= 0) {                                     // no selection while the stream is inside its prompt
                const int choice = ss.trunc ? choose_truncated(logit_s, reinterpret_cast<unsigned*>(cdf),
                                                               reinterpret_cast<float*>(cdf) + C, C, lane, ss.temperature,
                                                               ss.top_k, ss.top_p, p.uniforms + (size_t)stream * p.n_samples + samp)
                                            : choose_sample(logit_s, cdf, C, lane, ss.temperature,
                                                            p.uniforms ? p.uniforms + (size_t)stream * p.n_samples + samp : nullptr);
                if (lane == 0) {
                    misc[0] = choice;
                    if (rank == 0) p.out_idx[(size_t)stream * p.n_samples + samp] = choice;
                }
            }
        }
    }
    WORKER_SYNC();
    if (rank == 0 && tid == 0) p.cur_idx[stream] = misc[0];
    cluster_sync_all();                                          // peers may still be storing into this CTA's shared memory
}

// ================================================================================================ batched cluster kernel
// Tensor-core sampler for nets of width W = 256 or 512 (R = D = S = E = W, classes = 256, k = 2), one stream or many: a
// thread-block cluster advances up to CL8_SB = 8 independent streams together, so the weights of a stage enter shared
// memory ONCE per 8 streams and step (gen_kernel_cluster streams all 79 MB per stream and step; only 7 of its clusters are
// co-resident, so 64 streams ran as waves).  Every exchanged vector is W / 16 blocks ("virtual ranks") of 16 channels x 8
// streams; a CTA owns one block (W = 256, clusters of 16) or two (W = 256, clusters of 8; W = 512, clusters of 16) and
// computes those rows of every stage for all 8 streams:
//   * the dot products are mma.sync m16n8k16 (M = 16 rows of the stage, N = the 8 streams, K = 16 input channels = one
//     block) with bf16 hi/lo operand pairs -- x = hi + lo up to 2^-17 relative, three MMAs per product (lo.hi, hi.lo, hi.hi
//     on independent accumulators), fp32 accumulation: the scheme of the training kernels (tc_block.cu).  Weights are
//     pre-split ONCE per session into fragment-ordered images (cl8_pack_kernel): a warp's A fragments are two conflict-free
//     LDS.128, a stage's image is one bulk copy.  Activations are exchanged already split, in B-fragment order: a k-step's
//     B operands are one LDS.128.  8 warps = 2 m-tiles x 4 K quarters; the partials meet in shared memory and 128-256
//     finishing threads apply bias / tanh.sigmoid / the residual add and stage the CTA's block(s);
//   * exchange: a pusher warp reads a staged 512-byte block back and issues ONE st.async.v4 per destination CTA, crediting
//     the bytes to an mbarrier there; consumers sleep on their own mbarrier; tools/dsmem_probe.cu compares this (H) with a bulk
//     copy per destination (F) and per-lane stores (E);
//   * weights: producer warp(s) keep a ring of images full (bulk copies; cp.async for the second half of a CTA's image when
//     it owns two blocks): 128 KB of whole stages at W = 256; at W = 512 a stage's image doubles with K and the vectors
//     double too, so the ring is 2 x 32 KB and carries every stage in K-chunks (CL8 chunk constants below);
//   * history: the {value, tag} fp32 ring of the other kernels (same layout: sessions, queue export and kernel switches keep
//     working), written by the owning CTA, fetched one stage ahead into registers, validated by tag, split on arrival.
// Streams never mix (N is the stream index of the MMA) and both cluster sizes add in the same order: a stream's indices and
// logits do not depend on how many streams run beside it, bit for bit.
constexpr int CL8_SB = 8;               // streams per cluster
constexpr int CL8_C = 256;              // classes of every net this kernel serves
constexpr int CL8_BLK = 512;            // bytes of one (source CTA) block of an exchanged vector: 8 streams x 16 channels x (hi, lo)
constexpr int CL8_IMGH = 16 * 1024;     // one virtual rank's chunk of an end_conv_1 image: 16 k-steps of one m-tile
// k-steps of one ring chunk of a layer stage (both m-tiles of a virtual rank): the whole K = 256 at W = 256, a quarter of
// K = 512 at W = 512 (so that a CTA's chunk, 2 x 16 KB, fits a 32 KB slot)
__host__ __device__ constexpr int cl8_ksc(int W) { return W == 256 ? 16 : 8; }
// byte offset of the (hi pair | lo pair) unit of channels (c & ~1, c | 1) of stream s inside a block: per stream 64 bytes =
// 4 x [unit t | unit t+4], the order in which lane (g = stream, t) of an m16n8k16 B fragment consumes them
__device__ __forceinline__ int cl8_unit_off(int s, int c) {
    const int u = c >> 1;
    return s * 64 + (u & 3) * 16 + (u >> 2) * 8;
}
__device__ __forceinline__ void cl8_split(float x, unsigned short& hi, unsigned short& lo) {
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
    hi = __bfloat16_as_ushort(h);
    lo = __bfloat16_as_ushort(l);
}
// one value of a block, written as two 16-bit stores (the pair partner is written by another thread)
__device__ __forceinline__ void cl8_put(unsigned char* blk, int s, int c, float x) {
    unsigned short hi, lo;
    cl8_split(x, hi, lo);
    unsigned short* q = reinterpret_cast<unsigned short*>(blk + cl8_unit_off(s, c)) + (c & 1);
    q[0] = hi;
    q[2] = lo;
}
__device__ __forceinline__ void mma_bf16_16816(float (&d)[4], const uint4& a, unsigned b0, unsigned b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a.x), "r"(a.y), "r"(a.z), "r"(a.w), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void mbar_wait_bounded(unsigned long long* bar, unsigned parity) {
    unsigned done = 0, spins = 0;
    const unsigned a = smem_u32(bar);
    while (true) {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(a), "r"(parity) : "memory");
        if (done) break;
        if (++spins > (1u << 26)) asm volatile("trap;");        // never hang the GPU
    }
}
__device__ __forceinline__ unsigned mapa_u32(unsigned laddr, unsigned dst) {
    unsigned r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(laddr), "r"(dst));
    return r;
}

// Weight images.  One (m-tile, k-step) = 1 KB: [hi: 32 lanes x 16 B][lo: 32 lanes x 16 B], lane's 16 bytes = the A fragment
// registers a0..a3 of m16n8k16: a_j covers row g + 8*(j&1), k pair 2t + 8*(j>>1) (g = lane>>2, t = lane&3).
//   layout [layer][kind][chunk][virtual rank 0..W/16-1][image = [m-tile][k-step 0..KSC-1][hi | lo]], kind 0 = stage 1, tap
//   0 (old; m-tile 0 = filter rows, 1 = gate rows; k-step = channel block), 1 = stage 1, tap 1 (current), 2 = stage 2
//   (m-tile 0 = residual rows, 1 = skip rows; k-step = z block); chunk c holds k-steps c*KSC .. c*KSC+KSC-1 (KSC =
//   cl8_ksc(W): one 32 KB chunk per virtual rank at W = 256, four of 16 KB at W = 512).  Then end_conv_1 as
//   [chunk of 16 k-steps][virtual rank][16 KB: one m-tile] and end_conv_2 as [virtual rank 0-15][one m-tile, all W/16
//   k-steps] (at W = 256 both are [virtual rank][16 KB]).  The images of consecutive virtual ranks are adjacent, so a CTA
//   that owns VR of them fetches a chunk with ONE copy.
template <int W>
__global__ void cl8_pack_kernel(const GenLayer* layers, int n_layers, const float* e1w, const float* e2w, unsigned* img) {
    constexpr int NVR = W / 16, KSC = cl8_ksc(W), NCH = NVR / KSC;
    constexpr size_t IW = 2 * KSC * 256, HW = CL8_IMGH / 4;         // words per layer chunk image / end_conv_1 chunk image
    const size_t per_layer = 3 * NCH * NVR * IW, total = per_layer * n_layers + (size_t)(NVR + CL8_C / 16) * NVR * 256;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const float* src;      // row-major weight matrix the word comes from
        int row, col, ld, stride = 1;
        size_t w = i;
        if (w < per_layer * n_layers) {
            const int l = (int)(w / per_layer);
            w -= (size_t)l * per_layer;
            const int kind = (int)(w / (NCH * NVR * IW));   // 0: stage 1, tap 0 (old)   1: stage 1, tap 1 (current)   2: stage 2
            w -= (size_t)kind * NCH * NVR * IW;
            int c = 0;
            if constexpr (NCH > 1) {
                c = (int)(w / (NVR * IW));
                w -= (size_t)c * NVR * IW;
            }
            const int vrank = (int)(w / IW);
            w -= (size_t)vrank * IW;
            const GenLayer& L = layers[l];
            const int j = (int)(w & 3), lane = (int)((w >> 2) & 31), ks = c * KSC + (int)((w >> 8) & (KSC - 1)),
                      mt = (int)(w / (KSC * 256));
            const int g = lane >> 2, t = lane & 3;
            row = vrank * 16 + g + 8 * (j & 1);
            const int kk = 2 * t + 8 * (j >> 1);
            if (kind < 2) { src = mt ? L.wg : L.wf; col = (ks * 16 + kk) * 2 + kind; ld = 2 * W; stride = 2; }
            else { src = mt ? L.ws : L.wr; col = ks * 16 + kk; ld = W; }
        } else if (W == 256) {
            w -= per_layer * n_layers;
            const int which = (int)(w / (CL * HW));         // 0: end_conv_1   1: end_conv_2
            w -= (size_t)which * CL * HW;
            const int vrank = (int)(w / HW);
            w -= (size_t)vrank * HW;
            const int j = (int)(w & 3), lane = (int)((w >> 2) & 31), ks = (int)(w >> 8);
            const int g = lane >> 2, t = lane & 3;
            row = vrank * 16 + g + 8 * (j & 1);
            col = ks * 16 + 2 * t + 8 * (j >> 1);
            ld = W;
            src = which ? e2w : e1w;
        } else {
            w -= per_layer * n_layers;
            const bool e2 = w >= (size_t)NVR * NVR * 256;   // end_conv_1: NVR chunks of NVR x 16 KB; end_conv_2: 16 x NVR KB
            int vrank, ks;
            if (!e2) {
                const int c = (int)(w / (NVR * HW));
                w -= (size_t)c * NVR * HW;
                vrank = (int)(w / HW);
                w -= (size_t)vrank * HW;
                ks = c * 16 + (int)(w >> 8);
            } else {
                w -= (size_t)NVR * NVR * 256;
                vrank = (int)(w / (NVR * 256));
                w -= (size_t)vrank * NVR * 256;
                ks = (int)(w >> 8);
            }
            const int j = (int)(w & 3), lane = (int)((w >> 2) & 31);
            const int g = lane >> 2, t = lane & 3;
            row = vrank * 16 + g + 8 * (j & 1);
            col = ks * 16 + 2 * t + 8 * (j >> 1);
            ld = W;
            src = e2 ? e2w : e1w;
        }
        const int half = (int)((i >> 7) & 1);                // every image is a multiple of 256 words: bit 7 of i is the hi/lo plane
        const float x0 = src[(size_t)row * ld + col], x1 = src[(size_t)row * ld + col + stride];
        unsigned short h0, l0, h1, l1;
        cl8_split(x0, h0, l0);
        cl8_split(x1, h1, l1);
        img[i] = half ? ((unsigned)l1 << 16 | l0) : ((unsigned)h1 << 16 | h0);
    }
}

// W = the net's width (256 or 512).  CS = CTAs per cluster (16 or 8 at W = 256, 16 at W = 512).  The exchanged vectors
// consist of NVR = W / 16 blocks ("virtual ranks" of 16 channels); a CTA of a CS-cluster owns VR = NVR / CS consecutive
// virtual ranks and walks them one after the other in every stage.  Only few clusters of 16 CTAs are co-resident
// (tools/cluster_occ.cu) but about twice as many clusters of 8: CS = 8 runs 64 streams (8 clusters) in one wave on 64 SMs,
// at twice the per-CTA work -- the step is bound by the exchange latency, not by it.  At W = 512 VR = 2 with clusters of
// 16 already; clusters of 8 (VR = 4) would need twice the accumulators and staging, and do not fit.  The logit vector has
// 256 rows at both widths: NVRH = 16 virtual ranks, VRH = 16 / CS per CTA (1 at W = 512: the rows of CTA rank r are
// classes 16r .. 16r+15).
// COND: the filter / gate biases come from the condition table (a separate instantiation: the per-layer branch costs the
// unconditioned single-stream kernel ~6 % of its time per sample).  FRAMES (with COND): the table is a local-conditioning
// window, and each evaluation reads its frame's rows (a third instantiation, so the other two carry no trace of it).
// PS: per-stream settings (p.ps set); the scalar path runs the PS = false instantiations, which read only the scalars.
template <int W, int CS, bool COND, bool FRAMES, bool PS>
__global__ void __launch_bounds__(GEN_NT + 64 + (W / 16 / CS == 2 ? 32 : 0), 1) gen_kernel_cl8(const GenParams p) {
    extern __shared__ __align__(128) unsigned char smb[];
    constexpr int C = CL8_C, SB = CL8_SB, NV = 16, BLK = CL8_BLK, NVR = W / NV, VEC = NVR * BLK, VR = NVR / CS, NVC = NV * VR;
    constexpr int VRH = C / NV / CS;                    // virtual ranks of the logit vector per CTA
    static_assert((W == 256 || W == 512) && VR * CS == NVR && (VR == 1 || VR == 2), "gen_kernel_cl8: unsupported geometry");
    // ring chunks: a layer stage is NCH chunks of KSC k-steps (KQ per warp), end_conv_1 NCH1 chunks of 16 k-steps, and
    // end_conv_2 one chunk of VRH virtual ranks x NVR k-steps
    constexpr int KSC = cl8_ksc(W), NCH = NVR / KSC, KQ = KSC / 4, IMGC = 2 * KSC * 1024, NCH1 = NVR / 16;
    // exchanged vectors first: same offsets in every CTA (mapa keeps the offset).  Each is NVR blocks of 512 bytes.
    unsigned char* Xcur = smb;                          // [2] layer input h (hi/lo split), by layer parity
    unsigned char* Xz = Xcur + 2 * VEC;                 // [2] gated activation z, by layer parity; Xz[1] doubles as sampling scratch
    unsigned char* Xs = Xz + 2 * VEC;                   // relu(skip sum)           \  Xz[1], Xs, Xy are contiguous: 3 vectors that no
    unsigned char* Xy = Xs + VEC;                       // end_conv_1 output        /  peer writes while this CTA samples
    unsigned char* Xl = Xy + VEC;                       // logits, fp32: [virtual rank 0-15][stream][16]
    unsigned char* Xold = Xl + VEC;                     // history taps of the coming stage 1 (local)
    unsigned char* stg = Xold + VEC;                    // [2][VR][BLK] this CTA's contribution of a stage, staged for the pusher
    float* part = reinterpret_cast<float*>(stg + 2 * VR * BLK);               // [2][VR][8 warps][32 lanes][4] partial C fragments
    float* hown = part + 2 * VR * 8 * 128;              // [2][VR][16][SB] fp32 layer input at the channels this CTA owns
    // weight ring: 4 x 32 KB (W = 256, VR = 1), 2 x 64 KB (W = 256, VR = 2) or 2 x 32 KB (W = 512)
    constexpr int SLOTB = VR * IMGC, NSLOT = W == 256 ? 4 / VR : 2;
    constexpr int NTHR = GEN_NT + 64 + (VR == 2 ? 32 : 0);      // workers + producer + pusher (+ second producer for VR = 2)
    unsigned char* wbuf = reinterpret_cast<unsigned char*>(hown + 2 * NVC * SB);         // [NSLOT][SLOTB] weight image ring
    unsigned long long* fullb = reinterpret_cast<unsigned long long*>(wbuf + (size_t)NSLOT * SLOTB);
    unsigned long long* emptyb = fullb + 4;
    unsigned long long* xbar = emptyb + 4;              // [0,1] h by layer parity, [2,3] z by layer parity, [4] skip, [5] y1, [6] logits
    GenLayer* lay_s = reinterpret_cast<GenLayer*>(xbar + 8);
    int* slot_s = reinterpret_cast<int*>(lay_s + p.n_layers);
    int* idx_s = slot_s + p.n_layers;                   // [SB] current class index per stream, [SB] abort flag
    float* logit_s = reinterpret_cast<float*>(Xz + VEC);                      // [SB][C] sampling scratch (aliases Xz[1])
    double* cdf = reinterpret_cast<double*>(Xs);                              // [SB][C]  (aliases Xs; Xy too at W = 256)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int rank = (int)cluster_rank(), cl = blockIdx.x / CS, NS = p.NS, NL = p.n_layers;
    const int v0 = rank * VR;                           // first virtual rank of this CTA
    // live streams of this cluster: slots 0 .. n_live-1.  A stream's bytes in every exchanged block are contiguous (64 at
    // s * 64: cl8_unit_off, and the [stream][16] fp32 logits), so only the first 64 * n_live bytes of each block travel.
    const int n_live = min(SB, NS - cl * SB);
    const unsigned XVEC = 64u * (unsigned)n_live * NVR; // bytes of one exchange round that land in each CTA
    const unsigned XVECL = 64u * (unsigned)n_live * (C / NV);     // ... of the logit round (= XVEC at W = 256)
    const int o0 = v0 * NV;                             // first channel this CTA owns in every stage vector

    {
        unsigned* z0 = reinterpret_cast<unsigned*>(smb);
        const int n0 = (int)((reinterpret_cast<unsigned char*>(wbuf) - smb) / 4);
        for (int i = tid; i < n0; i += NTHR) z0[i] = 0u;
        const int* src = reinterpret_cast<const int*>(p.layers);
        int* dst = reinterpret_cast<int*>(lay_s);
        for (int i = tid; i < NL * (int)(sizeof(GenLayer) / sizeof(int)); i += NTHR) dst[i] = src[i];
    }
    if (tid < 2 * SB) idx_s[tid] = (tid < SB && cl * SB + tid < NS) ? p.cur_idx[cl * SB + tid] : 0;
    if (tid == 0) {
        for (int i = 0; i < NSLOT; ++i) { mbar_init(fullb + i, VR == 2 ? 33 : 1); mbar_init(emptyb + i, GEN_WARPS); }
        for (int i = 0; i < 7; ++i) mbar_init(xbar + i, 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncthreads();
    // Every exchange barrier expects the live bytes only.  The columns of empty stream slots are then never written by
    // peers and may hold stale values or sampling scratch: harmless, since MMA columns (= streams) are independent, and
    // every reduction and store works per (row, stream) and is guarded by fs_on / hs_g < NS.
    if (tid == 0)
        for (int i = 0; i < 7; ++i) mbar_expect_tx(xbar + i, (W != 256 && i == 6) ? XVECL : XVEC);     // arm phase 0 of every exchange barrier
    for (int l = tid; l < NL; l += GEN_NT) {
        const int len = lay_s[l].ring_len;
        slot_s[l] = (p.t0 + len - 1) % len;
    }
    cluster_sync_all();                                  // nobody may store into a peer before its barriers exist
    constexpr unsigned smask = (unsigned)NSLOT - 1u, sshift = (NSLOT == 4) ? 2u : 1u;
    const size_t img_kind = (size_t)NVR * IMGC;          // bytes of one (layer, kind, chunk): all virtual ranks
    const unsigned char* img_mine = p.cl8_img + (size_t)v0 * IMGC;
    const unsigned char* img_head = p.cl8_img + 3 * NCH * img_kind * NL + (size_t)v0 * CL8_IMGH;
    // end_conv_2 (W = 512; at W = 256 it is end_conv_1's second chunk): this CTA's VRH virtual ranks x NVR k-steps
    const unsigned char* img_e2 = p.cl8_img + 3 * NCH * img_kind * NL + (size_t)NVR * NVR * 1024 + (size_t)rank * VRH * NVR * 1024;
    // the source and size of ring chunk st of an evaluation: the layer stages' chunks, then the head's
    auto chunk_src = [&](int st, unsigned& bytes) {
        const unsigned char* src;
        if (st < 3 * NCH * NL) {
            src = img_mine + (size_t)st * img_kind;
            bytes = VR * IMGC;
        } else if (W == 256 || st - 3 * NCH * NL < NCH1) {
            src = img_head + (size_t)(st - 3 * NCH * NL) * NVR * CL8_IMGH;
            bytes = VR * CL8_IMGH;
        } else {
            src = img_e2;
            bytes = VRH * NVR * 1024;
        }
        return src;
    };

    // push the staged blocks `sb` into blocks v0 .. v0+VR-1 of vector `vec` of every CTA of the cluster: the pusher warp
    // (warp 9) reads the live part of each 512-byte block back (16 bytes per lane, lanes 0 .. 4*n_live-1) and issues ONE
    // st.async.v4 per destination and lane -- a whole block per instruction when all 8 streams are live, its bytes
    // credited to the destination's mbarrier.  With one live stream a round moves 64 bytes per (source, destination)
    // instead of 512 (tools/dsmem_probe.cu: I against H).  The alternatives tools/dsmem_probe.cu
    // compares are one cp.async.bulk per destination (which also occupies the SM's bulk-copy engine and needs a proxy
    // fence after staging), per-lane 8-byte stores from the worker warps, and a multicast copy from a global staging slot
    // (which needs a fence after the global stores).  The workers only signal "staged" (bar.arrive on barrier 2) and
    // move on to the next stage.
    const unsigned sm_base = smem_u32(smb);
    unsigned rdelta[CS];                                 // shared::cluster address of CTA d minus the local address (pusher warp)
#pragma unroll
    for (int d = 0; d < CS; ++d) rdelta[d] = (warp == GEN_WARPS + 1) ? mapa_u32(sm_base, (unsigned)d) - sm_base : 0u;
    auto push = [&](int sb, unsigned char* vec, int bar_i) {
        if (lane >= 4 * n_live) return;
        const bool lg = W != 256 && bar_i == 6;          // the logit vector: VRH blocks from rank * VRH
#pragma unroll
        for (int vr = 0; vr < VR; ++vr) {
            if (lg && vr >= VRH) break;
            const uint4 v = *reinterpret_cast<const uint4*>(stg + (sb * VR + vr) * BLK + lane * 16);
            const unsigned la = smem_u32(vec + ((lg ? rank * VRH : v0) + vr) * BLK + lane * 16), lb = smem_u32(xbar + bar_i);
#pragma unroll
            for (int d = 0; d < CS; ++d)
                asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];" ::"r"(
                                 la + rdelta[d]),
                             "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(lb + rdelta[d])
                             : "memory");
        }
    };
#define CL8_STAGED_SYNC() asm volatile("bar.sync 2, 288;" ::: "memory")
#define CL8_STAGED_ARRIVE() asm volatile("bar.arrive 2, 288;" ::: "memory")
    if (warp == GEN_WARPS + 1) {
        int sb = 0;
        for (int ev = 0; ev < p.n_evals; ++ev) {
            const bool wh = head_at(p, p.t0 + ev);
            for (int l = 0; l < NL; ++l) {
                CL8_STAGED_SYNC();
                push(sb, Xz + (l & 1) * VEC, 2 + (l & 1));
                sb ^= 1;
                if (l + 1 < NL) {
                    CL8_STAGED_SYNC();
                    push(sb, Xcur + ((l + 1) & 1) * VEC, (l + 1) & 1);
                    sb ^= 1;
                }
            }
            if (wh) {
                CL8_STAGED_SYNC(); push(sb, Xs, 4); sb ^= 1;
                CL8_STAGED_SYNC(); push(sb, Xy, 5); sb ^= 1;
                CL8_STAGED_SYNC(); push(sb, Xl, 6); sb ^= 1;
            }
        }
        cluster_sync_all();
        return;
    }
    // ---- producer warp: the weight images of this CTA for every stage, in order: ONE bulk copy per stage kind (the images
    // of the CTA's VR virtual ranks are adjacent).  One lane issues; the issuing thread is held per
    // instruction, so whole images it is: fewer, larger copies with two in flight give an SM the most bytes per cycle
    // (tools/bulk_bw_probe.cu).  The exchange does not use the bulk-copy engine (st.async), which would throttle these copies.
    if (warp == GEN_WARPS) {
        if (lane == 0) {
            unsigned q = 0;
            for (int ev = 0; ev < p.n_evals; ++ev) {
                const bool wh = head_at(p, p.t0 + ev);
                // per layer: old taps, current input, stage 2 (NCH chunks each); then the head stages' chunks
                const int n_st = wh ? 3 * NCH * NL + NCH1 + 1 : 3 * NCH * NL;
                for (int st = 0; st < n_st; ++st, ++q) {
                    unsigned bytes;
                    const unsigned char* src = chunk_src(st, bytes);
                    const int slot = (int)(q & smask);
                    if (q >= (unsigned)NSLOT) {
                        const unsigned par = ((q >> sshift) & 1u) ^ 1u;
                        unsigned done = 0, spins = 0;
                        while (!done) {
                            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                                         : "=r"(done) : "r"(smem_u32(emptyb + slot)), "r"(par) : "memory");
                            if (!done && ++spins > (1u << 30)) asm volatile("trap;");
                        }
                    }
                    // VR = 2: the bulk copy brings the first virtual rank's image, warp 10 the second one (below)
                    mbar_expect_tx(fullb + slot, bytes / VR);
                    bulk_g2s(wbuf + (size_t)slot * SLOTB, src, bytes / VR, fullb + slot);
                }
            }
        }
        cluster_sync_all();                              // matches the workers' final cluster barrier
        return;
    }
    // ---- second producer (VR = 2 only): one bulk copy at a time streams ~31 bytes/cycle into the 2-slot ring, which made
    // the 192 KB of a layer the bottleneck; this warp fetches the second half of every chunk (the second virtual rank's
    // image; end_conv_2 at W = 512: the second half of its k-steps) as 16-byte cp.async copies (load/store path, ~27
    // bytes/cycle for one warp) in parallel with the bulk copy of the first.
    if (VR == 2 && warp == GEN_WARPS + 2) {
        unsigned q = 0;
        for (int ev = 0; ev < p.n_evals; ++ev) {
            const bool wh = head_at(p, p.t0 + ev);
            const int n_st = wh ? 3 * NCH * NL + NCH1 + 1 : 3 * NCH * NL;
            for (int st = 0; st < n_st; ++st, ++q) {
                unsigned half;
                const unsigned char* src = chunk_src(st, half);
                half /= 2;
                src += half;
                const int slot = (int)(q & smask);
                if (q >= (unsigned)NSLOT) {
                    const unsigned par = ((q >> sshift) & 1u) ^ 1u;
                    unsigned done = 0, spins = 0;
                    while (!done) {
                        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                                     : "=r"(done) : "r"(smem_u32(emptyb + slot)), "r"(par) : "memory");
                        if (!done && ++spins > (1u << 30)) asm volatile("trap;");
                    }
                }
                const unsigned dst = smem_u32(wbuf + (size_t)slot * SLOTB + half) + lane * 16;
                const unsigned char* sp = src + lane * 16;
#pragma unroll 8
                for (unsigned o = 0; o < half; o += 512)
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + o), "l"(sp + o) : "memory");
                // this lane's arrival on the slot's "full" barrier fires when its copies above have landed
                asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(fullb + slot)) : "memory");
            }
        }
        cluster_sync_all();
        return;
    }
    unsigned cons_q = 0;
    auto stage_weights = [&]() -> const unsigned char* {
        const int slot = (int)(cons_q & smask);
        mbar_wait(fullb + slot, (cons_q >> sshift) & 1u);
        return wbuf + (size_t)slot * SLOTB;
    };
    auto release_slot = [&]() {
        __syncwarp();
        if (lane == 0) mbar_arrive_(emptyb + (cons_q & smask));
        ++cons_q;
    };
    // exchange barrier i: wait for the phase all threads are at, then thread 0 arms the next phase (it has seen this one end)
    unsigned xpar = 0;                                   // bit i = parity of the phase of xbar[i] to wait for next
    auto xwait = [&](int i) {
        mbar_wait_bounded(xbar + i, (xpar >> i) & 1u);
        xpar ^= 1u << i;
        if constexpr (W == 256) {
            if (tid == 0) mbar_expect_tx(xbar + i, XVEC);
        } else {
            if (tid == 0) mbar_expect_tx(xbar + i, i == 6 ? XVECL : XVEC);
        }
    };
    // one k-step of this warp's m-tile: A fragments (hi, lo) from the stage image, B fragments of the 8 streams from a block
    const int mt = warp & 1, kq = warp >> 1;
    // three independent accumulation chains (lo.hi, hi.lo, hi.hi) so that consecutive MMAs do not wait for each other; they
    // are added in a fixed order when the partial is stored
    struct Acc3 { float lh[4], hl[4], hh[4]; };
    auto acc_zero = [](Acc3& d) {
#pragma unroll
        for (int i = 0; i < 4; ++i) d.lh[i] = d.hl[i] = d.hh[i] = 0.f;
    };
    auto acc_store = [&](const Acc3& d, float* dst) {
        *reinterpret_cast<float4*>(dst) = make_float4((d.lh[0] + d.hl[0]) + d.hh[0], (d.lh[1] + d.hl[1]) + d.hh[1],
                                                      (d.lh[2] + d.hl[2]) + d.hh[2], (d.lh[3] + d.hl[3]) + d.hh[3]);
    };
    auto mma_step = [&](const unsigned char* a, const unsigned char* xblk, Acc3& d) {      // a: this lane's hi fragment; lo at +512
        const uint4 ah = *reinterpret_cast<const uint4*>(a), al = *reinterpret_cast<const uint4*>(a + 512);
        const uint4 b = *reinterpret_cast<const uint4*>(xblk + (lane >> 2) * 64 + (lane & 3) * 16);
        mma_bf16_16816(d.lh, al, b.x, b.z);
        mma_bf16_16816(d.hl, ah, b.y, b.w);
        mma_bf16_16816(d.hh, ah, b.x, b.z);
    };
    // this warp's KQ k-steps (KQ*kq .. KQ*kq+KQ-1) of its m-tile of ring chunk c of every virtual rank (images VR apart by
    // IMGC) against blocks c*KSC + KQ*kq.. of vector x.  The virtual ranks' chains are interleaved k-step by k-step: they are
    // independent, share the B fragments, and hide each other's MMA latency (nothing is stored until all are issued).
    auto mma_quarter = [&](const unsigned char* wimg, const unsigned char* x, int c, Acc3 (&d)[VR]) {
#pragma unroll
        for (int i = 0; i < KQ; ++i)
#pragma unroll
            for (int vr = 0; vr < VR; ++vr)
                mma_step(wimg + vr * IMGC + ((size_t)(mt * KSC + KQ * kq + i) * 2) * 512 + lane * 16,
                         x + (c * KSC + KQ * kq + i) * BLK, d[vr]);
    };
    // sum over the 4 K quarters of output (m-tile m, row r of the tile, stream s): fragment element (lane', j) of each partial
    auto part_sum = [&](const float* pb, int m, int r, int s) {
        const float* q = pb + ((m * 32 + (r & 7) * 4 + (s >> 1)) << 2) + ((r >> 3) << 1) + (s & 1);
        return ((q[0] + q[256]) + q[512]) + q[768];
    };
    // history taps: thread -> (stream = warp, channels 2*lane + 64*j + {0,1}), fetched into registers one stage ahead
    const int hs_g = cl * SB + warp;                     // global stream whose taps this thread fetches (and which it samples)
    constexpr int NHQ = W / 64;
    Pair2 hq[NHQ];
    const uint2* hsrc = nullptr;
    unsigned htag = 0;
    auto issue_old = [&](int ln, int te, int slot_te) {  // slot_te = ring slot of time te in layer ln
        const GenLayer& Lp = lay_s[ln];
        hsrc = nullptr;
        if (te >= Lp.dil && hs_g < NS) {
            const int so = (slot_te + 1 == Lp.ring_len) ? 0 : slot_te + 1;
            hsrc = p.ringLL + Lp.ring_off + ((size_t)so * NS + hs_g) * W + 2 * lane;
            htag = (unsigned)(te - Lp.dil) + 1u;
#pragma unroll
            for (int j = 0; j < NHQ; ++j) hq[j] = ld_pair2(hsrc + 64 * j);
        }
    };
    auto commit_old = [&]() {
#pragma unroll
        for (int j = 0; j < NHQ; ++j) {
            float a = 0.f, b = 0.f;
            if (hsrc != nullptr) {
                if (hq[j].a.y != htag || hq[j].b.y != htag) hq[j] = poll2_spin(hsrc + 64 * j, htag, p.err, idx_s + SB);
                a = __uint_as_float(hq[j].a.x);
                b = __uint_as_float(hq[j].b.x);
            }
            const int c0 = 2 * lane + 64 * j;             // channels c0, c0 + 1: one (hi pair | lo pair) unit
            unsigned short h0, l0, h1, l1;
            cl8_split(a, h0, l0);
            cl8_split(b, h1, l1);
            *reinterpret_cast<uint2*>(Xold + (c0 >> 4) * BLK + cl8_unit_off(warp, c0 & 15)) =
                make_uint2((unsigned)h1 << 16 | h0, (unsigned)l1 << 16 | l0);
        }
    };
    issue_old(0, p.t0, p.t0 % lay_s[0].ring_len);
    commit_old();
    WORKER_SYNC();
    // finishing threads: output (virtual rank fvr of this CTA, channel fc of its 16, stream fs).  VR = 2: every thread finishes
    // one conv / residual output AND one skip output; VR = 1: threads 0-127 the conv / residual ones, 128-255 the skip ones.
    const int fvr = (VR == 2) ? (tid >> 7) : 0, fc = (tid >> 3) & 15, fs = tid & 7;
    const bool fin_a = (VR == 2) || tid < NV * SB, fin_s = (VR == 2) || tid >= NV * SB;
    const int fch = o0 + fvr * NV + fc;                   // the channel (= row of the stage's weight matrix) this thread finishes
    // the logit this thread finishes (end_conv_2 row): fch where the logit vector splits like the others (VRH = VR), else
    // class rank*16 + fc in threads 0-127
    const bool fin_l = (VRH == VR) ? fin_a : tid < NV * SB;
    const int fcl = (VRH == VR) ? fch : rank * NV + fc, fvl = (VRH == VR) ? fvr : 0;
    const int fsg = cl * SB + fs;
    const bool fs_on = fsg < NS;
    unsigned pb_i = 0, sb_i = 0;                          // partial-sum / staging double-buffer indices
    auto part_of = [&](unsigned pb, int vr) { return part + (pb * VR + vr) * 8 * 128; };
    auto stg_of = [&](unsigned sb, int vr) { return stg + (sb * VR + vr) * BLK; };

    for (int ev = 0; ev < p.n_evals; ++ev) {
        const int t = p.t0 + ev;
        const unsigned rtag = (unsigned)t + 1u;          // ring tag of time t
        const bool want_head = head_at(p, t);
        const bool tr_on = p.trace != nullptr && blockIdx.x == 0 && tid == 0 && ev == p.n_evals - 1;
        // FRAMES: this stream's rows of evaluation t's frame; layer l's row is l * NS * cond_sstride further
        // (PS: the row of the finishing stream's own window)
        const float* cs_t = nullptr;
        if constexpr (FRAMES && PS) cs_t = p.cond + (size_t)fsg * p.cond_sstride + (fs_on ? cond_row<PS_ON>(p, fsg, t, W) : 0);
        else if constexpr (FRAMES) cs_t = cond_at(p, t, W) + (size_t)fsg * p.cond_sstride;
        int tr_n = 0;
#define TR8() do { if (tr_on && tr_n < 2040) p.trace[tr_n++] = clock64(); } while (0)
        if (tr_on) p.trace[2040] = clock64();             // whole-evaluation stamps live at [2040..2047]
        if (tid < SB && cl * SB + tid < NS) {
            int v;
            if (given_input<PS ? PS_ON : PS_OFF>(p, cl * SB + tid, t, v)) idx_s[tid] = v;
        }
        for (int l = tid; l < NL; l += GEN_NT) {
            const int s1 = slot_s[l] + 1;
            slot_s[l] = (s1 == lay_s[l].ring_len) ? 0 : s1;
        }
        WORKER_SYNC();
        // layer 0's input: the start-conv column of every stream (warp = stream), computed locally by every CTA; the
        // owners of a channel also enqueue it in the ring and keep the fp32 value for the residual add
        {
            int idx = idx_s[warp];
            idx = idx < 0 ? 0 : (idx >= C ? C - 1 : idx);
            const GenLayer& L0 = lay_s[0];
            uint2* ring0 = p.ringLL + L0.ring_off + ((size_t)slot_s[0] * NS + hs_g) * W;
#pragma unroll
            for (int j = 0; j < W / 32; ++j) {
                const int r = lane + 32 * j;
                const float v = __ldg(p.start_w + (size_t)r * C + idx) + (p.start_b ? __ldg(p.start_b + r) : 0.f);
                cl8_put(Xcur + (r >> 4) * BLK, warp, r & 15, v);
                if (r >= o0 && r < o0 + NVC) {
                    hown[(r - o0) * SB + warp] = v;
                    if (hs_g < NS) st_pair(ring0 + r, v, rtag);
                }
            }
        }
        WORKER_SYNC();
        float skr = 0.f;                                  // skip sum of (channel fch, stream fs) in the fin_s threads
        TR8();             // layer stamps start here (index 0)

        for (int l = 0; l < NL; ++l) {
            const GenLayer& L = lay_s[l];
            const bool more = (l + 1 < NL);
            unsigned char* xc = Xcur + (l & 1) * VEC;
            unsigned char* zb = Xz + (l & 1) * VEC;
            // biases of this thread's outputs: requested now, used one or two stages later
            // conditioned: the stream's own filter / gate biases, from the condition table
            const float* cb = FRAMES ? cs_t + (size_t)l * NS * p.cond_sstride : (COND ? p.cond + ((size_t)l * NS + fsg) * 2 * W : nullptr);
            const float b_f = COND ? ((fin_a && fs_on) ? __ldg(cb + fch) : 0.f) : ((fin_a && L.bf) ? __ldg(L.bf + fch) : 0.f);
            const float b_g = COND ? ((fin_a && fs_on) ? __ldg(cb + W + fch) : 0.f) : ((fin_a && L.bg) ? __ldg(L.bg + fch) : 0.f);
            const float b_r = (fin_a && L.br) ? __ldg(L.br + fch) : 0.f, b_s = (fin_s && L.bs) ? __ldg(L.bs + fch) : 0.f;
            // ================= stage 1: m-tile 0 = filter rows, 1 = gate rows; k-steps 4*kq+i of the old taps, then of h
            {
                // history taps of the NEXT stage 1 start their trip through the L2 now; they are used a whole stage later
                if (more) issue_old(l + 1, t, slot_s[l + 1]);
                else if (ev + 1 < p.n_evals) issue_old(0, t + 1, (slot_s[0] + 1 == lay_s[0].ring_len) ? 0 : slot_s[0] + 1);
                else hsrc = nullptr;
                Acc3 d[VR];
#pragma unroll
                for (int c = 0; c < NCH; ++c) {
                    const unsigned char* wimg = stage_weights();
                    if (c == 0) {
                        TR8();         // 1: stage-1 weights (old tap) landed
#pragma unroll
                        for (int vr = 0; vr < VR; ++vr) acc_zero(d[vr]);
                    }
                    mma_quarter(wimg, Xold, c, d);
                    release_slot();
                }
#pragma unroll
                for (int c = 0; c < NCH; ++c) {
                    const unsigned char* wimg = stage_weights();
                    if (c == 0) {
                        if (l > 0) xwait(l & 1);
                        TR8();         // 2: old-tap MMAs done, h arrived
                    }
                    mma_quarter(wimg, xc, c, d);
                    release_slot();
                }
#pragma unroll
                for (int vr = 0; vr < VR; ++vr) acc_store(d[vr], part_of(pb_i, vr) + ((kq * 2 + mt) * 32 + lane) * 4);
                TR8();         // 3: MMAs done, partials stored
                WORKER_SYNC();
                TR8();         // 4: barrier
                if (fin_a) {
                    const float* pb = part_of(pb_i, fvr);
                    const float f = part_sum(pb, 0, fc, fs) + b_f;
                    const float g = part_sum(pb, 1, fc, fs) + b_g;
                    cl8_put(stg_of(sb_i, fvr), fs, fc, tanh_(f) * sigmoid_(g));
                }
                pb_i ^= 1;
                TR8();         // 5: z computed and staged
                CL8_STAGED_ARRIVE();
                sb_i ^= 1;
            }
            // ================= stage 2: m-tile 0 = residual rows, 1 = skip rows; k-steps 4*kq+i of z
            {
                // every warp is past its stage-1 reads of Xold (two barriers ago): refill it while z is in flight
                commit_old();
                TR8();         // 6: next history taps in place
                const bool active = (mt == 0) ? more : want_head;
                Acc3 d[VR];
#pragma unroll
                for (int c = 0; c < NCH; ++c) {
                    const unsigned char* wimg = stage_weights();
                    if (c == 0) {
                        TR8();         // 7: stage-2 weights landed
                        xwait(2 + (l & 1));
                        TR8();         // 8: z arrived
#pragma unroll
                        for (int vr = 0; vr < VR; ++vr) acc_zero(d[vr]);
                    }
                    if (active) mma_quarter(wimg, zb, c, d);
                    release_slot();
                }
#pragma unroll
                for (int vr = 0; vr < VR; ++vr) acc_store(d[vr], part_of(pb_i, vr) + ((kq * 2 + mt) * 32 + lane) * 4);
                TR8();         // 9: MMAs done, partials stored
                WORKER_SYNC();
                TR8();         // 10: barrier
                const float* pb = part_of(pb_i, fvr);
                if (fin_a && more) {
                    const GenLayer& Ln = lay_s[l + 1];
                    float v = part_sum(pb, 0, fc, fs) + b_r;
                    v += hown[(l & 1) * NVC * SB + (fvr * NV + fc) * SB + fs];
                    hown[((l + 1) & 1) * NVC * SB + (fvr * NV + fc) * SB + fs] = v;
                    if (fs_on) st_pair(p.ringLL + Ln.ring_off + ((size_t)slot_s[l + 1] * NS + fsg) * W + fch, v, rtag);
                    cl8_put(stg_of(sb_i, fvr), fs, fc, v);
                }
                if (fin_s && want_head) {
                    const float v = part_sum(pb, 1, fc, fs) + b_s;
                    skr = v + skr;
                }
                pb_i ^= 1;
                TR8();         // 11: h' computed and staged
                if (more) {
                    CL8_STAGED_ARRIVE();
                    sb_i ^= 1;
                }
            }
        }
        if (tr_on) p.trace[2041] = clock64();             // layers done
        if (!want_head) continue;

        // ================= head: relu(skip) -> end_conv_1 -> relu -> end_conv_2; one m-tile per virtual rank, the k-steps
        // of each chunk spread over the 8 warps (end_conv_1: 2 of 16 each; end_conv_2: NVR / 8 of NVR)
        if (fin_s) cl8_put(stg_of(sb_i, fvr), fs, fc, fmaxf(skr, 0.f));
        CL8_STAGED_ARRIVE();
        sb_i ^= 1;
        // this warp's k-steps of each of the stage's nvr virtual ranks' m-tiles over its nch chunks of kpc k-steps -> part
        auto head_stage = [&](const unsigned char* x, int nch, int nvr, int kpc) {
            Acc3 d[VR];
#pragma unroll
            for (int c = 0; c < NCH1; ++c) {
                if (c >= nch) break;
                const unsigned char* wimg = stage_weights();
                if (c == 0) {
#pragma unroll
                    for (int vr = 0; vr < VR; ++vr) acc_zero(d[vr]);
                }
#pragma unroll
                for (int i = 0; i < NVR / 8; ++i) {
                    if (i >= kpc / 8) break;
#pragma unroll
                    for (int vr = 0; vr < VR; ++vr) {
                        if (vr >= nvr) break;
                        const int ks = (kpc / 8) * warp + i;
                        mma_step(wimg + vr * kpc * 1024 + ((size_t)ks * 2) * 512 + lane * 16, x + (c * kpc + ks) * BLK, d[vr]);
                    }
                }
                release_slot();
            }
#pragma unroll
            for (int vr = 0; vr < VR; ++vr)
                if (vr < nvr) acc_store(d[vr], part_of(pb_i, vr) + (warp * 32 + lane) * 4);
        };
        auto head_sum = [&](const float* pb, int r, int s) {  // 8 partials, one per warp
            const float* q = pb + (((r & 7) * 4 + (s >> 1)) << 2) + ((r >> 3) << 1) + (s & 1);
            float v = q[0];
#pragma unroll
            for (int i = 1; i < 8; ++i) v += q[i * 128];
            return v;
        };
        xwait(4);
        head_stage(Xs, NCH1, VR, 16);
        WORKER_SYNC();
        if (fin_a) {
            const float y = fmaxf(head_sum(part_of(pb_i, fvr), fc, fs) + __ldg(p.e1b + fch), 0.f);
            cl8_put(stg_of(sb_i, fvr), fs, fc, y);
        }
        pb_i ^= 1;
        CL8_STAGED_ARRIVE();
        sb_i ^= 1;
        xwait(5);
        head_stage(Xy, 1, VRH, NVR);
        WORKER_SYNC();
        if (fin_l) {
            const float dc = (float)fcl - (float)C / 2.f;
            const float v = (head_sum(part_of(pb_i, fvl), fc, fs) + __ldg(p.e2b + fcl)) -
                            (dc * dc) * ((PS && fs_on) ? p.ps[fsg].regularize : p.regularize);
            if (fs_on && p.out_logits) {
                const int samp = sample_of<PS ? PS_ON : PS_OFF>(p, fsg, t);
                if (samp >= 0) p.out_logits[((size_t)fsg * p.n_samples + samp) * C + fcl] = v;
            }
            reinterpret_cast<float*>(stg_of(sb_i, fvl))[fs * NV + fc] = v;               // logits travel as fp32: [stream][16]
        }
        pb_i ^= 1;
        CL8_STAGED_ARRIVE();
        sb_i ^= 1;
        xwait(6);
        if (tr_on) p.trace[2042] = clock64();             // head done, logits everywhere
        // every CTA holds all logits of its 8 streams: warp = stream draws the next index (all CTAs agree)
        if (hs_g < NS) {
            const GenStream ss = stream_set<PS ? PS_ON : PS_OFF>(p, hs_g);
            const int samp = sample_of<PS ? PS_ON : PS_OFF>(p, hs_g, t);
            if (samp >= 0) {                              // no selection while the stream is inside its prompt
                float* lg = logit_s + warp * C;
                const float* xl = reinterpret_cast<const float*>(Xl);
                for (int c = lane; c < C; c += 32) lg[c] = xl[(c >> 4) * (BLK / 4) + warp * NV + (c & 15)];
                __syncwarp();
                const int choice = ss.trunc ? choose_truncated(lg, reinterpret_cast<unsigned*>(cdf + warp * C),
                                                               reinterpret_cast<float*>(cdf + warp * C) + C, C, lane,
                                                               ss.temperature, ss.top_k, ss.top_p,
                                                               p.uniforms + (size_t)hs_g * p.n_samples + samp)
                                            : choose_sample(lg, cdf + warp * C, C, lane, ss.temperature,
                                                            p.uniforms ? p.uniforms + (size_t)hs_g * p.n_samples + samp : nullptr);
                if (lane == 0) {
                    // with forced samples the next evaluation's input is given, and the top of the loop stores it from
                    // another thread that no barrier separates from this one: store the choice only where it is used
                    if (p.forced == nullptr || ev + 1 == p.n_evals) idx_s[warp] = choice;
                    if (rank == 0) p.out_idx[(size_t)hs_g * p.n_samples + samp] = choice;
                }
            }
        }
        if (tr_on) p.trace[2043] = clock64();             // sampled
        // the top-of-evaluation barrier publishes idx_s
    }
    WORKER_SYNC();
    if (rank == 0 && tid < SB && cl * SB + tid < NS) p.cur_idx[cl * SB + tid] = idx_s[tid];
    cluster_sync_all();                                  // peers may still be storing into this CTA's shared memory
}

// ------------------------------------------------------------------------------------------------ ring prefill / seating
// One layer's input at times [t_lo, t_end), computed by a forward pass, into the ring slots t % ring_len: frame
// f_end - (t_end - t) of sequence j of src, fp32 frames (B, L, R) or chunked bf16 pairs (B, 2, R/8, L, 8) (value hi + lo).
// plain: kernel 1's ring of floats; otherwise the {value, tag = t + 1} pairs the flag-exchange kernels poll for.
// seats.n == 0 (wn_gen_prefill_layer): sequence j is stream j, for every stream.  seats.n > 0 (wn_gen_seat_layer): sequence
// j is stream seats.slot[j], whose position at t_end is seats.q_end[j]; times of negative positions, and every time when
// src is null, get 0 (times t < 0 go to slot t mod ring_len, the slot kernel 1 reads for them).
constexpr int GEN_SEAT_MAX = 128;
struct GenSeatList { int n; int slot[GEN_SEAT_MAX]; int q_end[GEN_SEAT_MAX]; };

__global__ void gen_prefill_kernel(const void* __restrict__ src, int pairs, int L, int f_end, int t_lo, int t_end, int NS,
                                   int R, int ring_len, float* __restrict__ rings, long long ring_off, int plain,
                                   const GenSeatList seats) {
    const int rows = seats.n ? seats.n : NS;
    const long long n = (long long)(t_end - t_lo) * rows * R;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(i % R);
        const long long q = i / R;
        const int j = (int)(q % rows), t = t_lo + (int)(q / rows);
        const int s = seats.n ? seats.slot[j] : j;
        const bool live = src != nullptr && (seats.n == 0 || seats.q_end[j] - (t_end - t) >= 0);
        const long long f = f_end - (t_end - t);
        float v = 0.f;
        if (live && pairs) {
            const __nv_bfloat16* b = reinterpret_cast<const __nv_bfloat16*>(src);
            const size_t hi = ((((size_t)j * 2) * (R / 8) + r / 8) * L + f) * 8 + (r & 7);
            v = __bfloat162float(b[hi]) + __bfloat162float(b[hi + (size_t)(R / 8) * L * 8]);
        } else if (live) {
            v = reinterpret_cast<const float*>(src)[((size_t)j * L + f) * R + r];
        }
        int slot = t % ring_len;
        if (slot < 0) slot += ring_len;
        const size_t e = ((size_t)slot * NS + s) * R + r;
        if (plain) rings[ring_off + e] = v;                          // ring_off counts elements of either kind
        else reinterpret_cast<uint2*>(rings)[ring_off + e] = make_uint2(__float_as_uint(v), (unsigned)t + 1u);
    }
}

// ------------------------------------------------------------------------------------------------ host side
struct ScratchLayout {
    size_t bar, cur_idx, layers, zbuf, skipbuf, y1buf, logitbuf, err, zLL, skipLL, y1LL, logitLL, ll_end, trace, cl8_img, cl8_bytes, total;
};
// the batched cluster kernel's shape: a k = 2 net of 256 classes whose other four widths are all 256 or all 512 (any
// number of streams)
static bool cl8_shape_ok(const wn_gen_shape& s) {
    return s.n_streams >= 1 && s.k == 2 && s.n_layers >= 2 && (s.R == 256 || s.R == 512) && s.D == s.R && s.S == s.R &&
           s.E == s.R && s.classes == CL8_C;
}
// bytes of its weight images (cl8_pack_kernel): per layer 3 kinds x W/16 virtual ranks x 2 m-tiles x W/16 k-steps of 1 KB,
// then end_conv_1 (W/16 x W/16 KB) and end_conv_2 (16 x W/16 KB): 1.5 MB per layer at W = 256, 6 MB at W = 512
static size_t cl8_image_bytes(const wn_gen_shape& s) {
    const size_t nvr = (size_t)s.R / 16;
    return 1024 * (6 * nvr * nvr * (size_t)s.n_layers + nvr * nvr + 16 * nvr);
}
static size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static ScratchLayout scratch_layout(const wn_gen_shape& s) {
    ScratchLayout o;
    size_t off = 0;
    o.bar = off; off += 256;
    o.cur_idx = off; off = align_up(off + sizeof(int) * s.n_streams, 256);
    o.layers = off; off = align_up(off + sizeof(GenLayer) * s.n_layers, 256);
    o.zbuf = off; off = align_up(off + sizeof(float) * (size_t)s.n_streams * s.D, 256);
    o.skipbuf = off; off = align_up(off + sizeof(float) * (size_t)s.n_streams * s.S, 256);
    o.y1buf = off; off = align_up(off + sizeof(float) * (size_t)s.n_streams * s.E, 256);
    o.logitbuf = off; off = align_up(off + sizeof(float) * (size_t)s.n_streams * s.classes, 256);
    o.err = off; off += 256;
    o.zLL = off; off = align_up(off + sizeof(uint2) * 2 * (size_t)s.n_layers * s.n_streams * s.D, 256);
    o.skipLL = off; off = align_up(off + sizeof(uint2) * 2 * (size_t)s.n_streams * s.S, 256);
    o.y1LL = off; off = align_up(off + sizeof(uint2) * 2 * (size_t)s.n_streams * s.E, 256);
    o.logitLL = off; off = align_up(off + sizeof(uint2) * 2 * (size_t)s.n_streams * s.classes, 256);
    o.ll_end = off;
    o.trace = off; off += 8 * 2048;
    o.cl8_img = off;
    o.cl8_bytes = cl8_shape_ok(s) ? cl8_image_bytes(s) : 0;
    off = align_up(off + o.cl8_bytes, 256);
    o.total = off;
    return o;
}
static size_t ring_floats(const wn_gen_shape& s, std::vector<long long>* offs) {
    size_t total = 0;
    for (int l = 0; l < s.n_layers; ++l) {
        if (offs) offs->push_back((long long)total);
        total += (size_t)((s.k - 1) * s.dilations[l] + 1) * s.n_streams * s.R;
    }
    return total;
}

}  // namespace wn

using namespace wn;

struct wn_gen_handle {
    wn_gen_shape shape;
    std::vector<int> dil;
    std::vector<GenLayer> layers;
    GenParams base;
    ScratchLayout lay;
    char* scratch;
    size_t ring_bytes;
    int grid, sm_count;
    size_t smem;
    bool tables_uploaded;
    int cur_t;
    int mode;               // what wn_gen_set_mode stored (0 = best kernel for the shape, the default); pick_kernel decides
    size_t smem_ll;
    bool fast_ok;           // single stream, k=2, power-of-two grid, rows per stage divide 8: gen_kernel_fast applies
    size_t smem_fast;
    int n_wslots_fast;
    int xn_fast;
    bool cluster_ok;        // k=2, 256-class nets whose rows split over 16 CTAs x 8 warps: gen_kernel_cluster applies
    size_t smem_cluster;
    int n_wslots_cluster, wslot_cluster;
    bool cl8_ok, cl8_packed;   // gen_kernel_cl8 applies (cl8_shape_ok and the shared memory fits); its weight images are built
    bool generic_ok, ll_ok;    // the grid-barrier / the generic flag-exchange kernel fit in shared memory for this stream count
    bool cl8_8_ok;             // ... and so does its 8-CTA-cluster instantiation
    int cl8_cs;                // its cluster size, 16 or 8 (wn_gen_create)
    int cl8_w;                 // its width instantiation, 256 or 512 (the net's R)
    size_t smem_cl8, smem_cl8_8;
    int top_k;              // wn_gen_set_truncation (0, 1.0: off)
    double top_p;
    // wn_gen_set_stream_params: the host records (empty: the scalar path), their device copy (allocated at the first call,
    // outside the workspace; GenStream [NS] then the windows of GenParams::pcw, int2 [NS]), whether it still has to be
    // uploaded, and what wn_gen_run checks and derives from them
    std::vector<wn_gen_stream_params> sp;
    GenStream* d_sp;
    bool sp_dirty, sp_any_trunc, sp_any_temp;
    int sp_max_given, sp_head_from;
    // wn_gen_prefill_*: the t_end each layer's ring was filled for (-1: not filled since wn_gen_reset), and the ring layout
    // the fill wrote (-1: none; 1: plain floats of kernel 1, 0: {value, tag} pairs of every other kernel)
    std::vector<int> pf_t_end;
    int pf_plain;
    // wn_gen_set_stream_positions: one record per stream (empty: cleared).  run_origin: each stream's origin at the last
    // wn_gen_run (0 after wn_gen_reset, INT_MIN after wn_gen_set_time: every stream must then be seated); seat_t /
    // seat_origin [layer * n_streams + stream]: the t a stream's ring was last seated at (wn_gen_seat_layer) and the origin
    // that seat implied; seat_plain: the ring layout the seats wrote (as pf_plain)
    std::vector<wn_gen_stream_pos> pos;
    std::vector<int> run_origin, seat_t, seat_origin;
    int seat_plain;
    // wn_gen_set_condition_stream_frames: each stream's first window frame (empty: one window shared by all streams)
    std::vector<int> cond_f0;
};

static int validate_shape(const wn_gen_shape* s) {
    WN_REQUIRE(s && s->dilations, WN_E_BADARG, "wn_gen: null shape");
    WN_REQUIRE(s->n_layers > 0 && s->k >= 1 && s->R > 0 && s->D > 0 && s->S > 0 && s->E > 0 && s->classes > 0 &&
                   s->n_streams > 0,
               WN_E_BADARG, "wn_gen: bad shape");
    for (int l = 0; l < s->n_layers; ++l) WN_REQUIRE(s->dilations[l] >= 1, WN_E_BADARG, "wn_gen: bad dilation");
    return 0;
}

extern "C" int wn_gen_workspace_bytes(const wn_gen_shape* s, size_t* ring_bytes, size_t* scratch_bytes) {
    if (int rc = validate_shape(s)) return rc;
    if (ring_bytes) *ring_bytes = sizeof(uint2) * ring_floats(*s, nullptr);   // {value, tag} pairs
    if (scratch_bytes) *scratch_bytes = scratch_layout(*s).total;
    return 0;
}

// The batched cluster kernel's launch at cluster size cs; attr holds the cluster dimension that cfg points to.
static cudaLaunchConfig_t cl8_config(const wn_gen_handle* h, int cs, cudaStream_t st, cudaLaunchAttribute* attr) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)((h->shape.n_streams + CL8_SB - 1) / CL8_SB * cs));
    // 8 worker warps, the weight producer warp(s) (two where a CTA owns two virtual ranks), the pusher warp
    cfg.blockDim = dim3(GEN_NT + 64 + (h->cl8_w / 16 / cs == 2 ? 32 : 0));
    cfg.dynamicSmemBytes = cs == 16 ? h->smem_cl8 : h->smem_cl8_8;
    cfg.stream = st;
    attr->id = cudaLaunchAttributeClusterDimension;
    attr->val.clusterDim.x = cs;
    attr->val.clusterDim.y = 1;
    attr->val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cfg;
}

// Cluster size of the batched cluster kernel: 16 CTAs (least work per CTA) while all clusters are co-resident, else 8
// (15 clusters fit instead of 7).  WN_GEN_CL8_CS=16|8 forces one (8 only where it fits).  512-wide nets run clusters of 16.
static int choose_cl8_cs(wn_gen_handle* h) {
    if (h->cl8_w == 512) {
        h->cl8_cs = 16;
        return 0;
    }
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = cl8_config(h, 16, nullptr, &attr);
    WN_CUDA(cudaFuncSetAttribute(gen_kernel_cl8<256, 16, false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)cfg.dynamicSmemBytes));
    WN_CUDA(cudaFuncSetAttribute(gen_kernel_cl8<256, 16, false, false, false>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    int fit16 = 0;
    WN_CUDA(cudaOccupancyMaxActiveClusters(&fit16, gen_kernel_cl8<256, 16, false, false, false>, &cfg));
    const int need = (h->shape.n_streams + CL8_SB - 1) / CL8_SB;
    h->cl8_cs = (need <= fit16 || !h->cl8_8_ok) ? 16 : 8;
    if (const char* e = getenv("WN_GEN_CL8_CS")) {
        const int v = atoi(e);
        if (v == 16 || (v == 8 && h->cl8_8_ok)) h->cl8_cs = v;
    }
    return 0;
}

// The kernel wn_gen_run launches in the handle's mode (the mode number of wn_gen_set_mode), 0 when none fits.
static int pick_kernel(const wn_gen_handle* h) {
    const int m = h->mode;
    if (m == 3 || m == 4 || m == 6) return m;               // wn_gen_set_mode accepts these only where they apply
    if (m == 0) {
        if (h->cl8_ok) return 6;                            // any number of streams of a 256- or 512-wide net
        if (h->cluster_ok && (h->shape.n_streams > 1 || !h->fast_ok)) return 4;
        // kernel 3 only where kernel 2 or 4 fits too: a net too deep for kernel 2's shared memory (on an H100 from ~2 240
        // layers of 256 channels with 512 end channels and classes) keeps kernel 1, which auto has always run there
        // kernel 3 reads no per-stream records: with positions set one stream runs kernel 2 (same sums) or 4
        if (h->fast_ok && (h->ll_ok || h->cluster_ok)) return h->pos.empty() ? 3 : (h->ll_ok ? 2 : 4);
    }
    if (m != 1 && h->ll_ok) return 2;                       // modes 0 and 2
    return h->generic_ok ? 1 : 0;
}

extern "C" int wn_gen_create(const wn_gen_shape* s, const wn_gen_weights* w, float* d_rings, void* d_scratch,
                             wn_gen_handle** out) {
    if (int rc = validate_shape(s)) return rc;
    WN_REQUIRE(w && d_rings && d_scratch && out, WN_E_BADARG, "wn_gen_create: null pointer");
    WN_REQUIRE(w->d_start_w && w->d_wf && w->d_wg && w->d_wr && w->d_ws && w->d_end1_w && w->d_end1_b && w->d_end2_w &&
                   w->d_end2_b,
               WN_E_BADARG, "wn_gen_create: null weight pointer");
    int dev = 0, sms = 0, smem_optin = 0;
    WN_CUDA(cudaGetDevice(&dev));
    WN_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    WN_CUDA(cudaDeviceGetAttribute(&smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));

    wn_gen_handle* h = new (std::nothrow) wn_gen_handle();
    WN_REQUIRE(h, WN_E_BADARG, "wn_gen_create: out of host memory");
    h->shape = *s;
    h->mode = 0;
    h->top_k = 0;
    h->top_p = 1.0;
    h->d_sp = nullptr;
    h->sp_dirty = false;
    h->dil.assign(s->dilations, s->dilations + s->n_layers);
    h->shape.dilations = h->dil.data();
    h->lay = scratch_layout(h->shape);
    h->scratch = (char*)d_scratch;
    std::vector<long long> offs;
    h->ring_bytes = sizeof(uint2) * ring_floats(h->shape, &offs);
    h->layers.resize(s->n_layers);
    for (int l = 0; l < s->n_layers; ++l) {
        GenLayer& L = h->layers[l];
        L.wf = w->d_wf[l]; L.wg = w->d_wg[l]; L.wr = w->d_wr[l]; L.ws = w->d_ws[l];
        L.bf = w->d_bf ? w->d_bf[l] : nullptr; L.bg = w->d_bg ? w->d_bg[l] : nullptr;
        L.br = w->d_br ? w->d_br[l] : nullptr; L.bs = w->d_bs ? w->d_bs[l] : nullptr;
        if (!(L.wf && L.wg && L.wr && L.ws)) {
            delete h;
            return set_err(WN_E_BADARG, "wn_gen_create: null weight pointer in layer %d", l);
        }
        L.ring_off = offs[l];
        L.dil = s->dilations[l];
        L.ring_len = (s->k - 1) * s->dilations[l] + 1;
    }
    GenParams& p = h->base;
    p.layers = reinterpret_cast<const GenLayer*>(h->scratch + h->lay.layers);
    p.n_layers = s->n_layers; p.k = s->k; p.R = s->R; p.D = s->D; p.S = s->S; p.E = s->E; p.C = s->classes;
    p.NS = s->n_streams;
    p.start_w = w->d_start_w; p.start_b = w->d_start_b;
    p.e1w = w->d_end1_w; p.e1b = w->d_end1_b; p.e2w = w->d_end2_w; p.e2b = w->d_end2_b;
    p.rings = d_rings;
    p.zbuf = reinterpret_cast<float*>(h->scratch + h->lay.zbuf);
    p.skipbuf = reinterpret_cast<float*>(h->scratch + h->lay.skipbuf);
    p.y1buf = reinterpret_cast<float*>(h->scratch + h->lay.y1buf);
    p.logitbuf = reinterpret_cast<float*>(h->scratch + h->lay.logitbuf);
    p.cur_idx = reinterpret_cast<int*>(h->scratch + h->lay.cur_idx);
    p.bar = reinterpret_cast<unsigned*>(h->scratch + h->lay.bar);

    // grid: as many CTAs as keep the per-stage row count per CTA minimal, at most one per SM
    // grid: a power of two, at most one CTA per SM, and -- when the net is wide enough -- at least 4 rows of every
    // exchanged vector per CTA so that a CTA's published pairs fill whole 32-byte sectors (see own_per above)
    int mind = s->D;
    if (s->R < mind) mind = s->R;
    if (s->E < mind) mind = s->E;
    if (s->classes < mind) mind = s->classes;
    int G = 1;
    while (G * 2 <= sms && G * 2 * 4 <= mind) G *= 2;
    if (G == 1)
        while (G * 2 <= sms && G * 2 <= s->D) G *= 2;
    if (const char* e = getenv("WN_GEN_GRID")) {            // tuning knob: fewer, fatter CTAs
        const int v = atoi(e);
        if (v >= 1 && v <= G) G = v;
    }
    if (G < 1) G = 1;
    h->grid = G;
    h->sm_count = sms;
    const int NS = s->n_streams;
    auto cdiv = [](int a, int b) { return (a + b - 1) / b; };
    const int mx1 = (s->k * s->R > s->S) ? s->k * s->R : s->S;
    const int mx2 = (s->D > s->E) ? s->D : s->E;
    p.regA = NS * mx1;
    p.regB = NS * mx2;
    int items = 2 * cdiv(s->D, G);
    p.pre_n = items * NS;
    p.skacc_n = cdiv(s->S, G) * NS;
    if (p.skacc_n < 4) p.skacc_n = 4;
    p.regA = (p.regA + 3) / 4 * 4; p.regB = (p.regB + 3) / 4 * 4; p.pre_n = (p.pre_n + 3) / 4 * 4;
    p.skacc_n = (p.skacc_n + 3) / 4 * 4;
    h->smem = sizeof(float) * ((size_t)p.regA + p.regB + p.pre_n + p.skacc_n + 2 * NS + (size_t)GEN_WARPS * s->classes);
    // the grid-barrier / generic kernels stage all streams' vectors in every CTA; the cluster kernels do not
    const bool cluster_shape = s->k == 2 && s->n_layers >= 2 && s->D % CL == 0 && s->R % CL == 0 && s->S % CL == 0 &&
                               s->E % CL == 0 && s->classes % CL == 0;
    if (h->smem > (size_t)smem_optin && !cluster_shape) {
        const size_t need = h->smem;
        delete h;
        return set_err(WN_E_UNSUPP, "wn_gen_create: %zu bytes of shared memory needed for %d streams, %d available", need,
                       NS, smem_optin);
    }
    // ---- LL kernel: exchange regions, shared-memory carve, weight prefetch ring
    p.ringLL = reinterpret_cast<uint2*>(d_rings);
    p.zLL = reinterpret_cast<uint2*>(h->scratch + h->lay.zLL);
    p.skipLL = reinterpret_cast<uint2*>(h->scratch + h->lay.skipLL);
    p.y1LL = reinterpret_cast<uint2*>(h->scratch + h->lay.y1LL);
    p.logitLL = reinterpret_cast<uint2*>(h->scratch + h->lay.logitLL);
    p.err = reinterpret_cast<int*>(h->scratch + h->lay.err);
    p.trace = getenv("WN_GEN_TRACE") ? reinterpret_cast<long long*>(h->scratch + h->lay.trace) : nullptr;
    {
        const int nDm = cdiv(s->D, G), nRm = cdiv(s->R, G), nSm = cdiv(s->S, G), nEm = cdiv(s->E, G), nCm = cdiv(s->classes, G);
        int mxA = mx1 > s->classes ? mx1 : s->classes;
        const int regA_ll = (NS * mxA + 3) / 4 * 4;
        int items_max = 2 * nDm;
        if (nRm + nSm > items_max) items_max = nRm + nSm;
        if (nEm > items_max) items_max = nEm;
        if (nCm > items_max) items_max = nCm;
        p.part_n = ((items_max > GEN_WARPS ? items_max : GEN_WARPS) * NS + 3) / 4 * 4;
        long long slot = (long long)2 * nDm * s->k * s->R;
        if ((long long)(nRm + nSm) * s->D > slot) slot = (long long)(nRm + nSm) * s->D;
        if ((long long)nEm * s->S > slot) slot = (long long)nEm * s->S;
        if ((long long)nCm * s->E > slot) slot = (long long)nCm * s->E;
        slot = (slot + 3) / 4 * 4;
        const size_t base = sizeof(float) * ((size_t)regA_ll + p.regB + p.part_n + p.skacc_n + (size_t)GEN_WARPS * s->classes) +
                            sizeof(double) * (size_t)GEN_WARPS * s->classes + 64 + sizeof(GenLayer) * (size_t)s->n_layers +
                            sizeof(int) * (size_t)(2 * NS + 4);
        const bool k_ok = ((s->k * s->R) % 4 == 0) && (s->D % 4 == 0) && (s->S % 4 == 0) && (s->E % 4 == 0);
        int nslots = 0;
        if (k_ok && base < (size_t)smem_optin) {
            long long fit = ((long long)smem_optin - (long long)base) / (slot * 4);
            nslots = fit >= 4 ? 4 : (fit >= 2 ? (int)fit : 0);
        }
        if (getenv("WN_GEN_NOPREFETCH")) nslots = 0;        // tuning knob: read weights through L2 instead
        p.wslot_floats = (int)slot;
        p.n_wslots = nslots;
        h->smem_ll = base + (size_t)nslots * slot * 4;
        // regA of the LL kernel also stages the logits; keep one GenParams for both kernels
        if (regA_ll > p.regA) {
            p.regA = regA_ll;
            h->smem = sizeof(float) * ((size_t)p.regA + p.regB + p.pre_n + p.skacc_n + 2 * NS + (size_t)GEN_WARPS * s->classes);
        }
        // ---- fast kernel eligibility (same K split as the generic kernel so both sum in the same order)
        auto pow2 = [](int v) { return v > 0 && (v & (v - 1)) == 0; };
        auto split_ok = [&](int rows, int K) {
            if (!(rows == 1 || rows == 2 || rows == 4 || rows == 8)) return false;
            const int hs = GEN_WARPS / rows;
            return K % hs == 0 && (K / hs) % 4 == 0 && (K / hs) >= 32 && (K / hs) <= FAST_MAXI * 128;
        };
        bool ok = NS == 1 && s->k == 2 && pow2(G) && G >= 2 && s->n_layers >= 2 && s->D % G == 0 && s->R % G == 0 &&
                  s->S % G == 0 && s->E % G == 0 && s->classes % G == 0;
        if (ok)
            ok = split_ok(2 * (s->D / G), 2 * s->R) && split_ok((s->R + s->S) / G, s->D) && split_ok(s->E / G, s->S) &&
                 split_ok(s->classes / G, s->E);
        h->fast_ok = false;
        if (ok) {
            int xn = s->R;
            if (s->D > xn) xn = s->D;
            if (s->S > xn) xn = s->S;
            if (s->E > xn) xn = s->E;
            if (s->classes > xn) xn = s->classes;
            xn = (xn + 3) & ~3;
            h->xn_fast = xn;
            const size_t fbase = sizeof(float) * (2 * GEN_WARPS + ((s->S / G + 3) & ~3) + 2 * ((s->R / G + 3) & ~3) + 2 * xn) +
                                 sizeof(double) * s->classes + 64 + sizeof(GenLayer) * (size_t)s->n_layers +
                                 sizeof(uint2) * 2 * (size_t)s->R + sizeof(int) * (size_t)(s->n_layers + 4);
            int fs = 0;
            if (fbase < (size_t)smem_optin) {
                long long fit = ((long long)smem_optin - (long long)fbase) / (slot * 4);
                fs = fit >= 4 ? 4 : (fit >= 2 ? 2 : 0);
            }
            if (getenv("WN_GEN_NOPREFETCH")) fs = 0;
            h->n_wslots_fast = fs;
            h->smem_fast = fbase + (size_t)fs * slot * 4;
            h->fast_ok = h->smem_fast <= (size_t)smem_optin;
        }
    }
    // ---- cluster kernel eligibility: rows of every stage split evenly over 16 CTAs x 8 warps, <= 4 rows per warp
    {
        auto div_ok = [&](int N) { return N % CL == 0; };
        bool ok = s->k == 2 && s->n_layers >= 2 && div_ok(s->D) && div_ok(s->R) && div_ok(s->S) && div_ok(s->E) &&
                  div_ok(s->classes) && (s->R % 4 == 0) && (s->D % 4 == 0) && (s->S % 4 == 0) && (s->E % 4 == 0);
        if (ok) {
            const int nD = s->D / CL, nR = s->R / CL, nS = s->S / CL;
            const int rw1 = 2 * nD / GEN_WARPS, rw2 = (nR + nS) / GEN_WARPS;
            ok = (2 * nD) % GEN_WARPS == 0 && (nR + nS) % GEN_WARPS == 0 && (rw1 == 2 || rw1 == 4) && rw2 >= 1 && rw2 <= CL_ROWS &&
                 nR % rw2 == 0 && (rw2 == 2 || rw2 == 4 || rw2 == 1);
        }
        h->cluster_ok = false;
        if (ok && !getenv("WN_GEN_NOCLUSTER")) {
            long long slot = (long long)2 * (s->D / CL) * 2 * s->R;
            if ((long long)(s->R / CL + s->S / CL) * s->D > slot) slot = (long long)(s->R / CL + s->S / CL) * s->D;
            if ((long long)(s->E / CL) * s->S > slot) slot = (long long)(s->E / CL) * s->S;
            if ((long long)(s->classes / CL) * s->E > slot) slot = (long long)(s->classes / CL) * s->E;
            slot = (slot + 3) / 4 * 4;
            const size_t cbase = sizeof(uint2) * (size_t)(2 * s->R + 2 * s->D + s->S + s->E + s->classes + 2 * s->R) +
                                 sizeof(float) * (size_t)(((s->S / CL + 3) & ~3) + 2 * ((s->R / CL + 3) & ~3) +
                                                          (((s->E + s->classes) / CL + 32 + 3) & ~3) + ((s->classes + 3) & ~3)) +
                                 sizeof(double) * s->classes + 64 + sizeof(GenLayer) * (size_t)s->n_layers +
                                 sizeof(int) * (size_t)(s->n_layers + 4);
            int cs = 0;
            if (cbase < (size_t)smem_optin) {
                long long fit = ((long long)smem_optin - (long long)cbase) / (slot * 4);
                cs = fit >= 4 ? 4 : (fit >= 2 ? 2 : 0);
            }
            h->n_wslots_cluster = cs;
            h->wslot_cluster = (int)slot;
            h->smem_cluster = cbase + (size_t)cs * slot * 4;
            h->cluster_ok = cs >= 2 && h->smem_cluster <= (size_t)smem_optin;
        }
    }
    // ---- batched cluster kernel (8 streams per cluster, tensor cores)
    {
        // gen_kernel_cl8's carve: 8 exchanged vectors of W/16 blocks, staging, partials, fp32 inputs, barriers, layer
        // table, then the weight ring (4 x 32 KB at W = 256; 2 x 32 KB at W = 512, where the vectors take 128 KB)
        const int W = s->R;
        auto smem_for = [&](int vr) {
            const size_t fixed = (size_t)8 * (W / 16) * CL8_BLK + (size_t)2 * vr * CL8_BLK +
                                 sizeof(float) * (size_t)(2 * vr * 8 * 128 + 2 * 16 * vr * CL8_SB) + 16 * 8 +
                                 sizeof(GenLayer) * (size_t)s->n_layers + sizeof(int) * (size_t)(s->n_layers + 2 * CL8_SB);
            return align_up(fixed, 16) + (W == 256 ? 4 : 2) * (size_t)32 * 1024;
        };
        h->cl8_w = W;
        h->smem_cl8 = smem_for(W / 16 / 16);
        h->smem_cl8_8 = smem_for(2);
        h->cl8_ok = cl8_shape_ok(*s) && h->smem_cl8 <= (size_t)smem_optin && !getenv("WN_GEN_NOCL8");
        h->cl8_8_ok = h->cl8_ok && W == 256 && h->smem_cl8_8 <= (size_t)smem_optin;
        h->cl8_packed = false;
        p.cl8_img = reinterpret_cast<const unsigned char*>(h->scratch + h->lay.cl8_img);
    }
    h->generic_ok = h->smem <= (size_t)smem_optin;
    h->ll_ok = h->smem_ll <= (size_t)smem_optin && s->n_layers >= 2;
    if (!h->generic_ok && !h->cl8_ok && !h->cluster_ok) {
        const size_t need = h->smem > h->smem_ll ? h->smem : h->smem_ll;
        delete h;
        return set_err(WN_E_UNSUPP, "wn_gen_create: %zu bytes of shared memory needed for %d streams, %d available", need,
                       s->n_streams, smem_optin);
    }
    if (int rc = h->cl8_ok ? choose_cl8_cs(h) : 0) {
        delete h;
        return rc;
    }
    h->tables_uploaded = false;
    h->cur_t = 0;
    h->pf_t_end.assign(s->n_layers, -1);
    h->pf_plain = -1;
    h->run_origin.assign(NS, 0);
    h->seat_t.assign((size_t)s->n_layers * NS, -1);
    h->seat_origin.assign((size_t)s->n_layers * NS, 0);
    h->seat_plain = -1;
    *out = h;
    return 0;
}

extern "C" int wn_gen_reset(wn_gen_handle* h, void* stream) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_reset: null handle");
    cudaStream_t st = (cudaStream_t)stream;
    WN_CUDA(cudaMemsetAsync(h->base.rings, 0, h->ring_bytes, st));
    WN_CUDA(cudaMemsetAsync(h->scratch + h->lay.cur_idx, 0, sizeof(int) * h->shape.n_streams, st));
    WN_CUDA(cudaMemsetAsync(h->scratch + h->lay.err, 0, h->lay.ll_end - h->lay.err, st));
    if (!h->tables_uploaded) {
        WN_CUDA(cudaMemcpyAsync(h->scratch + h->lay.layers, h->layers.data(), sizeof(GenLayer) * h->layers.size(),
                                cudaMemcpyHostToDevice, st));
        WN_CUDA(cudaStreamSynchronize(st));       // h->layers is pageable host memory owned by the handle
        h->tables_uploaded = true;
    }
    if (h->cl8_ok && !h->cl8_packed) {               // weights are constant for the life of a handle: split them once
        unsigned* img = reinterpret_cast<unsigned*>(h->scratch + h->lay.cl8_img);
        if (h->cl8_w == 512)
            cl8_pack_kernel<512><<<1184, 256, 0, st>>>(h->base.layers, h->shape.n_layers, h->base.e1w, h->base.e2w, img);
        else
            cl8_pack_kernel<256><<<1184, 256, 0, st>>>(h->base.layers, h->shape.n_layers, h->base.e1w, h->base.e2w, img);
        WN_CUDA(cudaGetLastError());
        h->cl8_packed = true;
    }
    h->cur_t = 0;
    h->pf_t_end.assign(h->shape.n_layers, -1);
    h->pf_plain = -1;
    h->run_origin.assign(h->shape.n_streams, 0);
    h->seat_t.assign(h->seat_t.size(), -1);
    h->seat_plain = -1;
    return 0;
}

// Nothing but the rings carries state into a launch at t0 > 0 when evaluation t0 reads a given sample: cur_idx is read only
// when it does not, and every exchange tag is either in shared memory (kernels 4, 6: zeroed at launch; kernel 4's `seq`
// starts from t0) or tagged t + 1 in the scratch wn_gen_reset zeroes (kernels 2, 3), and kernel 1's barrier counter is
// cleared before every launch.  So rings written here continue exactly like rings written by evaluations [0, t_end).
extern "C" int wn_gen_prefill_layer(wn_gen_handle* h, int layer, const void* d_src, int layout, int L, int frame_of_t_end,
                                    int t_end, void* stream) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_prefill_layer: null handle");
    WN_REQUIRE(h->tables_uploaded && h->cur_t == 0, WN_E_STATE,
               "wn_gen_prefill_layer: prefill only right after wn_gen_reset (the handle is at t = %d)", h->cur_t);
    WN_REQUIRE(layer >= 0 && layer < h->shape.n_layers && d_src && (layout == WN_GEN_SRC_FRAMES || layout == WN_GEN_SRC_PAIRS) &&
                   t_end >= 1 && L >= 1 && frame_of_t_end <= L,
               WN_E_BADARG, "wn_gen_prefill_layer: bad arguments (layer %d, layout %d, L %d, frame %d, t_end %d)", layer, layout,
               L, frame_of_t_end, t_end);
    const int R = h->shape.R, NS = h->shape.n_streams;
    WN_REQUIRE(layout == WN_GEN_SRC_FRAMES || R % 8 == 0, WN_E_BADARG, "wn_gen_prefill_layer: chunked pairs need R %% 8 == 0");
    const GenLayer& Lr = h->layers[layer];
    const int n_t = std::min(t_end, Lr.ring_len);
    WN_REQUIRE(frame_of_t_end - n_t >= 0, WN_E_BADARG,
               "wn_gen_prefill_layer: layer %d needs frames [%d, %d), the buffer starts at 0", layer, frame_of_t_end - n_t,
               frame_of_t_end);
    const int kid = pick_kernel(h);
    WN_REQUIRE(kid != 0, WN_E_UNSUPP, "wn_gen_prefill_layer: no sampler kernel fits this net in mode %d", h->mode);
    const int plain = kid == 1;
    WN_REQUIRE(h->pf_plain < 0 || h->pf_plain == plain, WN_E_STATE,
               "wn_gen_prefill_layer: the sampler kernel changed between layers (ring layout differs)");
    const long long n = (long long)n_t * NS * R;
    const int grid = (int)std::min<long long>((n + 255) / 256, 4LL * h->sm_count);
    GenSeatList all;
    all.n = 0;
    gen_prefill_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(d_src, layout == WN_GEN_SRC_PAIRS, L, frame_of_t_end, t_end - n_t,
                                                               t_end, NS, R, Lr.ring_len, h->base.rings, Lr.ring_off, plain, all);
    WN_CUDA(cudaGetLastError());
    h->pf_plain = plain;
    h->pf_t_end[layer] = t_end;
    return 0;
}

extern "C" int wn_gen_prefill_commit(wn_gen_handle* h, int t_end) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_prefill_commit: null handle");
    WN_REQUIRE(h->cur_t == 0, WN_E_STATE, "wn_gen_prefill_commit: the handle is at t = %d, not right after wn_gen_reset",
               h->cur_t);
    for (int l = 0; l < h->shape.n_layers; ++l)
        WN_REQUIRE(h->pf_t_end[l] == t_end, WN_E_STATE, "wn_gen_prefill_commit: layer %d was filled for t_end %d, not %d", l,
                   h->pf_t_end[l], t_end);
    h->cur_t = t_end;
    return 0;
}

extern "C" int wn_gen_set_time(wn_gen_handle* h, int t) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_set_time: null handle");
    WN_REQUIRE(h->tables_uploaded && h->cur_t == 0 && h->pf_plain < 0 && h->seat_plain < 0, WN_E_STATE,
               "wn_gen_set_time: only right after wn_gen_reset (the handle is at t = %d)", h->cur_t);
    WN_REQUIRE(t >= 0, WN_E_BADARG, "wn_gen_set_time: t must be >= 0, got %d", t);
    h->cur_t = t;
    h->run_origin.assign(h->shape.n_streams, INT_MIN);       // no stream's rings hold anything for these times
    return 0;
}

extern "C" int wn_gen_seat_layer(wn_gen_handle* h, int layer, int n, const int* slots, const int* q_end, const void* d_src,
                                 int layout, int L, int frame_of_end, void* stream) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_seat_layer: null handle");
    WN_REQUIRE(h->tables_uploaded, WN_E_STATE, "wn_gen_seat_layer: call wn_gen_reset first");
    const int NS = h->shape.n_streams, R = h->shape.R, t = h->cur_t;
    WN_REQUIRE(layer >= 0 && layer < h->shape.n_layers && n >= 1 && slots && q_end, WN_E_BADARG,
               "wn_gen_seat_layer: bad arguments (layer %d, %d slots)", layer, n);
    const GenLayer& Lr = h->layers[layer];
    if (d_src) {
        WN_REQUIRE((layout == WN_GEN_SRC_FRAMES || (layout == WN_GEN_SRC_PAIRS && R % 8 == 0)) && L >= 1 && frame_of_end <= L,
                   WN_E_BADARG, "wn_gen_seat_layer: bad source (layout %d, L %d, frame %d)", layout, L, frame_of_end);
    }
    std::vector<char> seen(NS, 0);
    for (int j = 0; j < n; ++j) {
        WN_REQUIRE(slots[j] >= 0 && slots[j] < NS && !seen[slots[j]], WN_E_BADARG,
                   "wn_gen_seat_layer: slot %d is out of range or listed twice", slots[j]);
        seen[slots[j]] = 1;
        WN_REQUIRE(q_end[j] >= 0 && (long long)t - q_end[j] >= INT_MIN / 2, WN_E_BADARG,
                   "wn_gen_seat_layer: slot %d: bad prompt end position %d", slots[j], q_end[j]);
        const int need = std::min(q_end[j], Lr.ring_len);    // positions [q_end - need, q_end) come from the source
        if (d_src && need > 0) {
            WN_REQUIRE(frame_of_end - need >= 0, WN_E_BADARG,
                       "wn_gen_seat_layer: layer %d needs frames [%d, %d), the buffer starts at 0", layer, frame_of_end - need,
                       frame_of_end);
            // every kernel reads times < 0 as zero history without looking at the ring
            WN_REQUIRE(t - need >= 0, WN_E_BADARG,
                       "wn_gen_seat_layer: slot %d: positions [%d, %d) would lie at times [%d, %d), and times < 0 read as "
                       "zero (start the handle later with wn_gen_set_time)", slots[j], q_end[j] - need, q_end[j], t - need, t);
        }
    }
    const int kid = pick_kernel(h);
    WN_REQUIRE(kid != 0, WN_E_UNSUPP, "wn_gen_seat_layer: no sampler kernel fits this net in mode %d", h->mode);
    const int plain = kid == 1;
    WN_REQUIRE(h->seat_plain < 0 || h->seat_plain == plain, WN_E_STATE,
               "wn_gen_seat_layer: the sampler kernel changed between seats (ring layout differs)");
    for (int j0 = 0; j0 < n; j0 += GEN_SEAT_MAX) {
        GenSeatList list;
        list.n = std::min(GEN_SEAT_MAX, n - j0);
        for (int j = 0; j < list.n; ++j) { list.slot[j] = slots[j0 + j]; list.q_end[j] = q_end[j0 + j]; }
        // sequence j of the source is listed slot j: offset the source to this chunk's first sequence
        const void* src = d_src;
        if (d_src)
            src = static_cast<const char*>(d_src) + (size_t)j0 * L * R * (layout == WN_GEN_SRC_PAIRS ? 2 * sizeof(__nv_bfloat16)
                                                                                                      : sizeof(float));
        const long long cnt = (long long)Lr.ring_len * list.n * R;
        const int grid = (int)std::min<long long>((cnt + 255) / 256, 4LL * h->sm_count);
        gen_prefill_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, layout == WN_GEN_SRC_PAIRS, L, frame_of_end,
                                                                   t - Lr.ring_len, t, NS, R, Lr.ring_len, h->base.rings,
                                                                   Lr.ring_off, plain, list);
        WN_CUDA(cudaGetLastError());
    }
    h->seat_plain = plain;
    for (int j = 0; j < n; ++j) {
        h->seat_t[(size_t)layer * NS + slots[j]] = t;
        h->seat_origin[(size_t)layer * NS + slots[j]] = t - q_end[j];
    }
    return 0;
}

template <int SB>
static int launch_gen(wn_gen_handle* h, GenParams& p, cudaStream_t st) {
    // a truncated draw needs a second C-float scratch per warp (the other kernels have a float64 one already)
    const size_t smem = h->smem + (p.trunc ? sizeof(float) * GEN_WARPS * (size_t)p.C : 0);
    if (p.trunc) {
        int optin = 0, dev = 0;
        WN_CUDA(cudaGetDevice(&dev));
        WN_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        WN_REQUIRE(smem <= (size_t)optin, WN_E_UNSUPP,
                   "wn_gen_run: kernel 1 needs %zu bytes of shared memory with truncation, %d available", smem, optin);
    }
    WN_CUDA(cudaFuncSetAttribute(gen_kernel<SB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    WN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gen_kernel<SB>, GEN_NT, smem));
    WN_REQUIRE(per_sm * h->sm_count >= h->grid, WN_E_UNSUPP, "wn_gen_run: %d CTAs cannot be co-resident", h->grid);
    void* args[] = {(void*)&p};
    WN_CUDA(cudaLaunchCooperativeKernel((const void*)gen_kernel<SB>, dim3(h->grid), dim3(GEN_NT), args, smem, st));
    return 0;
}

template <int SB, bool PF>
static int launch_gen_ll(wn_gen_handle* h, GenParams& p, cudaStream_t st) {
    WN_CUDA(cudaFuncSetAttribute(gen_kernel_ll<SB, PF>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_ll));
    int per_sm = 0;
    WN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gen_kernel_ll<SB, PF>, GEN_NT, h->smem_ll));
    WN_REQUIRE(per_sm * h->sm_count >= h->grid, WN_E_UNSUPP, "wn_gen_run: %d CTAs cannot be co-resident", h->grid);
    void* args[] = {(void*)&p};
    WN_CUDA(cudaLaunchCooperativeKernel((const void*)gen_kernel_ll<SB, PF>, dim3(h->grid), dim3(GEN_NT), args, h->smem_ll, st));
    return 0;
}

static int launch_gen_cluster(wn_gen_handle* h, GenParams& p, cudaStream_t st) {
    WN_CUDA(cudaFuncSetAttribute(gen_kernel_cluster, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_cluster));
    WN_CUDA(cudaFuncSetAttribute(gen_kernel_cluster, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(h->shape.n_streams * CL));
    cfg.blockDim = dim3(GEN_NT + 32);
    cfg.dynamicSmemBytes = h->smem_cluster;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CL;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int max_clusters = 0;
    WN_CUDA(cudaOccupancyMaxActiveClusters(&max_clusters, gen_kernel_cluster, &cfg));
    WN_REQUIRE(max_clusters >= 1, WN_E_UNSUPP, "wn_gen_run: a %d-CTA cluster cannot be scheduled on this device", CL);
    WN_CUDA(cudaLaunchKernelEx(&cfg, gen_kernel_cluster, p));
    return 0;
}

template <int W, int CS, bool COND, bool FRAMES, bool PS>
static int launch_gen_cl8_cs(wn_gen_handle* h, GenParams& p, cudaStream_t st) {
    cudaLaunchAttribute attr;
    const cudaLaunchConfig_t cfg = cl8_config(h, CS, st, &attr);
    WN_CUDA(cudaFuncSetAttribute(gen_kernel_cl8<W, CS, COND, FRAMES, PS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)cfg.dynamicSmemBytes));
    WN_CUDA(cudaFuncSetAttribute(gen_kernel_cl8<W, CS, COND, FRAMES, PS>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
    int max_clusters = 0;
    WN_CUDA(cudaOccupancyMaxActiveClusters(&max_clusters, gen_kernel_cl8<W, CS, COND, FRAMES, PS>, &cfg));
    WN_REQUIRE(max_clusters >= 1, WN_E_UNSUPP, "wn_gen_run: a %d-CTA cluster cannot be scheduled on this device", CS);
    WN_CUDA(cudaLaunchKernelEx(&cfg, gen_kernel_cl8<W, CS, COND, FRAMES, PS>, p));   // clusters are independent: more than fit run in waves
    return 0;
}
template <bool COND, bool FRAMES, bool PS>
static int launch_gen_cl8_w(wn_gen_handle* h, GenParams& p, cudaStream_t st) {
    if (h->cl8_w == 512) return launch_gen_cl8_cs<512, 16, COND, FRAMES, PS>(h, p, st);
    return h->cl8_cs == 16 ? launch_gen_cl8_cs<256, 16, COND, FRAMES, PS>(h, p, st) : launch_gen_cl8_cs<256, 8, COND, FRAMES, PS>(h, p, st);
}
template <bool PS>
static int launch_gen_cl8_cond(wn_gen_handle* h, GenParams& p, cudaStream_t st) {
    if (p.cond && p.cond_hop) return launch_gen_cl8_w<true, true, PS>(h, p, st);
    if (p.cond) return launch_gen_cl8_w<true, false, PS>(h, p, st);
    return launch_gen_cl8_w<false, false, PS>(h, p, st);
}
static int launch_gen_cl8(wn_gen_handle* h, GenParams& p, cudaStream_t st) {
    return p.ps ? launch_gen_cl8_cond<true>(h, p, st) : launch_gen_cl8_cond<false>(h, p, st);
}

template <bool PF, bool TRACE>
static int launch_gen_fast_t(wn_gen_handle* h, GenParams& p, cudaStream_t st) {
    WN_CUDA(cudaFuncSetAttribute(gen_kernel_fast<PF, TRACE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->smem_fast));
    int per_sm = 0;
    WN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gen_kernel_fast<PF, TRACE>, GEN_NT + 32, h->smem_fast));
    WN_REQUIRE(per_sm * h->sm_count >= h->grid, WN_E_UNSUPP, "wn_gen_run: %d CTAs cannot be co-resident", h->grid);
    void* args[] = {(void*)&p};
    WN_CUDA(cudaLaunchCooperativeKernel((const void*)gen_kernel_fast<PF, TRACE>, dim3(h->grid), dim3(GEN_NT + 32), args,
                                        h->smem_fast, st));
    return 0;
}
template <bool PF>
static int launch_gen_fast(wn_gen_handle* h, GenParams& p, cudaStream_t st) {
    // the stamping variant is a separate instantiation so that the production kernel's hot loop carries no trace code
    return p.trace ? launch_gen_fast_t<PF, true>(h, p, st) : launch_gen_fast_t<PF, false>(h, p, st);
}

extern "C" int wn_gen_set_mode(wn_gen_handle* h, int mode) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_set_mode: null handle");
    WN_REQUIRE(mode >= 0 && mode <= 6 && mode != 5, WN_E_BADARG,
               "wn_gen_set_mode: mode must be 0 (auto), 1 (grid barrier), 2 (generic flag exchange), 3 (single-stream L2 kernel), "
               "4 (cluster / DSMEM kernel) or 6 (batched tensor-core cluster kernel), got %d", mode);
    if (mode == 3) WN_REQUIRE(h->fast_ok, WN_E_UNSUPP, "wn_gen_set_mode: the single-stream L2 kernel does not apply to this shape");
    if (mode == 4) WN_REQUIRE(h->cluster_ok, WN_E_UNSUPP, "wn_gen_set_mode: the cluster kernel does not apply to this shape");
    if (mode == 6) WN_REQUIRE(h->cl8_ok, WN_E_UNSUPP, "wn_gen_set_mode: the batched cluster kernel does not apply to this shape");
    WN_REQUIRE(h->cur_t == 0, WN_E_STATE, "wn_gen_set_mode: switch kernels only right after wn_gen_reset");
    if (mode != 1) WN_REQUIRE(h->shape.n_layers >= 2, WN_E_UNSUPP, "wn_gen_set_mode: flag exchange needs >= 2 layers");
    h->mode = mode;
    return 0;
}

extern "C" int wn_gen_weights_changed(wn_gen_handle* h) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_weights_changed: null handle");
    h->cl8_packed = false;          // the next wn_gen_reset splits the weights again
    return 0;
}

// Leaves per-stream windows: the records' cond_origin / cond_frame0 go back to 0 at the next upload.
static void clear_stream_frames(wn_gen_handle* h) {
    if (h->cond_f0.empty()) return;
    h->cond_f0.clear();
    h->sp_dirty = true;
}

extern "C" int wn_gen_set_condition(wn_gen_handle* h, const float* d_cond) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_set_condition: null handle");
    clear_stream_frames(h);
    h->base.cond = d_cond;
    h->base.cond_hop = h->base.cond_frame0 = 0;
    h->base.cond_frames = 1;
    h->base.cond_sstride = 2 * h->shape.D;
    return 0;
}

extern "C" int wn_gen_set_condition_frames(wn_gen_handle* h, const float* d_cond, int frame0, int n_frames, int hop) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_set_condition_frames: null handle");
    if (d_cond == nullptr) return wn_gen_set_condition(h, nullptr);
    WN_REQUIRE(frame0 >= 0 && n_frames >= 1 && hop >= 1, WN_E_BADARG,
               "wn_gen_set_condition_frames: bad window (frame0 %d, %d frames, hop %d)", frame0, n_frames, hop);
    clear_stream_frames(h);
    h->base.cond = d_cond;
    h->base.cond_hop = hop; h->base.cond_frame0 = frame0; h->base.cond_frames = n_frames;
    h->base.cond_sstride = n_frames * 2 * h->shape.D;
    return 0;
}

extern "C" int wn_gen_set_condition_stream_frames(wn_gen_handle* h, const float* d_cond, const int* frame0, int n_frames,
                                                  int hop) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_set_condition_stream_frames: null handle");
    if (d_cond == nullptr) return wn_gen_set_condition(h, nullptr);
    WN_REQUIRE(frame0 && n_frames >= 1 && hop >= 1, WN_E_BADARG,
               "wn_gen_set_condition_stream_frames: bad window (%d frames, hop %d, frame0 %s)", n_frames, hop,
               frame0 ? "set" : "null");
    const int NS = h->shape.n_streams;
    for (int s = 0; s < NS; ++s)
        WN_REQUIRE(frame0[s] >= 0, WN_E_BADARG, "wn_gen_set_condition_stream_frames: stream %d: frame0 %d must be >= 0", s,
                   frame0[s]);
    h->base.cond = d_cond;
    h->base.cond_hop = hop; h->base.cond_frame0 = 0; h->base.cond_frames = n_frames;   // the records carry the windows
    h->base.cond_sstride = n_frames * 2 * h->shape.D;
    h->cond_f0.assign(frame0, frame0 + NS);
    h->sp_dirty = true;
    return 0;
}

extern "C" int wn_gen_set_truncation(wn_gen_handle* h, int top_k, double top_p) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_set_truncation: null handle");
    WN_REQUIRE(top_k >= 0, WN_E_BADARG, "wn_gen_set_truncation: top_k must be >= 0 (0: off), got %d", top_k);
    WN_REQUIRE(top_p > 0.0 && top_p <= 1.0, WN_E_BADARG, "wn_gen_set_truncation: top_p must lie in (0, 1] (1: off), got %g",
               top_p);                                      // NaN fails both comparisons
    h->top_k = top_k;
    h->top_p = top_p;
    return 0;
}

static bool stream_truncates(const wn_gen_stream_params& q, int classes) {
    return q.temperature > 0.f && ((q.top_k > 0 && q.top_k < classes) || q.top_p < 1.0);
}

extern "C" int wn_gen_set_stream_params(wn_gen_handle* h, const wn_gen_stream_params* params) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_set_stream_params: null handle");
    if (params == nullptr) {
        h->sp.clear();
        return 0;
    }
    const int NS = h->shape.n_streams;
    for (int s = 0; s < NS; ++s) {                          // all records are checked before any is taken
        const wn_gen_stream_params& q = params[s];
        WN_REQUIRE(q.n_given >= 1, WN_E_BADARG, "wn_gen_set_stream_params: stream %d: n_given must be >= 1, got %d", s, q.n_given);
        WN_REQUIRE(q.top_k >= 0, WN_E_BADARG, "wn_gen_set_stream_params: stream %d: top_k must be >= 0 (0: off), got %d", s, q.top_k);
        WN_REQUIRE(q.top_p > 0.0 && q.top_p <= 1.0, WN_E_BADARG,
                   "wn_gen_set_stream_params: stream %d: top_p must lie in (0, 1] (1: off), got %g", s, q.top_p);
        WN_REQUIRE(std::isfinite(q.temperature) && std::isfinite(q.regularize), WN_E_BADARG,
                   "wn_gen_set_stream_params: stream %d: temperature %g and regularize %g must be finite", s,
                   (double)q.temperature, (double)q.regularize);
    }
    h->sp.assign(params, params + NS);
    h->sp_max_given = 0;
    h->sp_head_from = 0x7fffffff;
    h->sp_any_trunc = h->sp_any_temp = false;
    for (const wn_gen_stream_params& q : h->sp) {
        h->sp_max_given = std::max(h->sp_max_given, q.n_given);
        h->sp_head_from = std::min(h->sp_head_from, q.n_given - 1);
        h->sp_any_trunc = h->sp_any_trunc || stream_truncates(q, h->shape.classes);
        h->sp_any_temp = h->sp_any_temp || q.temperature > 0.f;
    }
    if (NS > 1) {                                           // one stream: wn_gen_run folds the record into the scalars
        if (h->d_sp == nullptr) WN_CUDA(cudaMalloc(&h->d_sp, (sizeof(GenStream) + sizeof(int2)) * (size_t)NS));
    }
    h->sp_dirty = true;
    return 0;
}

extern "C" int wn_gen_set_stream_positions(wn_gen_handle* h, const wn_gen_stream_pos* pos) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_set_stream_positions: null handle");
    if (pos == nullptr) {
        h->pos.clear();
        h->sp_dirty = true;
        return 0;
    }
    WN_REQUIRE(!h->sp.empty(), WN_E_STATE, "wn_gen_set_stream_positions: positions need per-stream records "
                                           "(wn_gen_set_stream_params) first");
    const int NS = h->shape.n_streams;
    for (int s = 0; s < NS; ++s)
        WN_REQUIRE(pos[s].sample0 >= 0 && pos[s].first0 >= 0, WN_E_BADARG,
                   "wn_gen_set_stream_positions: stream %d: sample0 %d and first0 %d must be >= 0", s, pos[s].sample0,
                   pos[s].first0);
    if (h->d_sp == nullptr) WN_CUDA(cudaMalloc(&h->d_sp, (sizeof(GenStream) + sizeof(int2)) * (size_t)NS));
    h->pos.assign(pos, pos + NS);
    h->sp_dirty = true;
    return 0;
}

extern "C" int wn_gen_check(wn_gen_handle* h, void* stream) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_check: null handle");
    int flag = 0;
    WN_CUDA(cudaMemcpyAsync(&flag, h->scratch + h->lay.err, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    WN_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    WN_REQUIRE(flag == 0, WN_E_STATE, "wn_gen_check: the sampler timed out waiting for an exchange tag (launch aborted)");
    return 0;
}

extern "C" int wn_gen_run(wn_gen_handle* h, const wn_gen_run_args* a, void* stream) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_run: null handle");
    WN_REQUIRE(h->tables_uploaded, WN_E_STATE, "wn_gen_run: call wn_gen_reset first");
    WN_REQUIRE(a && a->d_first && a->d_out_idx, WN_E_BADARG, "wn_gen_run: null pointer");
    WN_REQUIRE(a->n_given >= 1 && a->n_samples >= 0 && a->n_evals >= 0 && a->t0 >= 0, WN_E_BADARG, "wn_gen_run: bad counts");
    WN_REQUIRE(a->t0 == h->cur_t, WN_E_STATE, "wn_gen_run: t0=%d does not continue the previous call (expected %d)", a->t0,
               h->cur_t);
    const bool per_stream = !h->sp.empty(), positions = !h->pos.empty();
    WN_REQUIRE(!positions || per_stream, WN_E_STATE, "wn_gen_run: stream positions need per-stream records");
    if (per_stream) {
        WN_REQUIRE(positions || a->n_given == h->sp_max_given, WN_E_BADARG,
                   "wn_gen_run: with per-stream parameters n_given is the pitch of d_first and must equal the longest prompt "
                   "(%d), got %d", h->sp_max_given, a->n_given);
        WN_REQUIRE(a->temperature == 0.f && a->regularize == 0.f && h->top_k == 0 && h->top_p == 1.0, WN_E_BADARG,
                   "wn_gen_run: with per-stream parameters the scalar temperature and regularize must be 0 and the "
                   "handle's truncation off (the records hold them)");
        WN_REQUIRE(!h->sp_any_temp || a->d_uniforms, WN_E_BADARG, "wn_gen_run: a stream with temperature > 0 needs d_uniforms");
    }
    int head_from = per_stream ? h->sp_head_from : a->n_given - 1;
    const int NS = h->shape.n_streams;
    if (positions) {
        // per stream: positions [q0, q1] of the launch; every read of first / forced and every written column in its row
        head_from = INT_MAX;
        for (int s = 0; s < NS; ++s) {
            const wn_gen_stream_pos& o = h->pos[s];
            const int ng = h->sp[s].n_given;
            WN_REQUIRE(o.origin <= a->t0, WN_E_BADARG, "wn_gen_run: stream %d starts at t = %d, after t0 = %d", s, o.origin,
                       a->t0);
            const long long q0 = (long long)a->t0 - o.origin, q1 = q0 + a->n_evals - 1;
            head_from = (int)std::min<long long>(head_from, (long long)o.origin + ng - 1);
            if (a->n_evals == 0) continue;
            if (q0 < ng)
                WN_REQUIRE(q0 - o.first0 >= 0 && std::min<long long>(q1, ng - 1) - o.first0 < a->n_given, WN_E_BADARG,
                           "wn_gen_run: stream %d reads prompt positions [%lld, %lld], its row holds [%d, %d)", s, q0,
                           std::min<long long>(q1, ng - 1), o.first0, o.first0 + a->n_given);
            if (a->d_forced && q1 >= ng)
                WN_REQUIRE(std::max<long long>(q0, ng) - ng - o.sample0 >= 0 && q1 - ng - o.sample0 < a->n_samples,
                           WN_E_BADARG, "wn_gen_run: stream %d reads forced samples outside its row", s);
            const long long i0 = std::max<long long>(q0 - (ng - 1), 0), i1 = q1 - (ng - 1);
            if (i1 >= i0)
                WN_REQUIRE(i0 - o.sample0 >= 0 && i1 - o.sample0 < a->n_samples, WN_E_BADARG,
                           "wn_gen_run: stream %d selects samples [%lld, %lld] into columns [%lld, %lld], outside [0, %d)", s,
                           i0, i1, i0 - o.sample0, i1 - o.sample0, a->n_samples);
        }
    } else {
        WN_REQUIRE(a->t0 + a->n_evals <= head_from + a->n_samples, WN_E_BADARG,
                   "wn_gen_run: evaluations [%d,%d) exceed the schedule of %d samples from evaluation %d", a->t0,
                   a->t0 + a->n_evals, a->n_samples, head_from);
    }
    // a stream that starts at another origin than it ran with: its rings must have been seated for it at this t, and its
    // first evaluation must read a prompt sample (cur_idx holds the previous job's last choice)
    for (int s = 0; s < NS; ++s) {
        const int origin = positions ? h->pos[s].origin : 0;
        if (origin == h->run_origin[s]) continue;
        for (int l = 0; l < h->shape.n_layers; ++l) {
            const size_t e = (size_t)l * NS + s;
            WN_REQUIRE(h->seat_t[e] == h->cur_t && h->seat_origin[e] == origin, WN_E_STATE,
                       "wn_gen_run: stream %d starts at t = %d but layer %d was not seated for it at t = %d", s, origin, l,
                       h->cur_t);
        }
        WN_REQUIRE(!positions || (long long)a->t0 - origin < h->sp[s].n_given || a->n_evals == 0, WN_E_BADARG,
                   "wn_gen_run: the first evaluation of newly seated stream %d must read a prompt sample", s);
    }
    WN_REQUIRE(!(a->temperature > 0.f) || a->d_uniforms, WN_E_BADARG, "wn_gen_run: temperature > 0 needs d_uniforms");
    const bool stream_frames = !h->cond_f0.empty();
    WN_REQUIRE(!stream_frames || per_stream, WN_E_STATE,
               "wn_gen_run: per-stream condition windows need per-stream records (wn_gen_set_stream_params)");
    if (a->n_evals == 0) return 0;
    if (stream_frames) {
        // per stream: the frames of positions [q0, q0 + n_evals) inside its own window
        const int hop = h->base.cond_hop, nf = h->base.cond_frames;
        for (int s = 0; s < NS; ++s) {
            const int origin = positions ? h->pos[s].origin : 0;
            const long long q0 = (long long)a->t0 - origin, q1 = q0 + a->n_evals - 1;
            const long long f_lo = q0 / hop, f_hi = q1 / hop;
            WN_REQUIRE(f_lo >= h->cond_f0[s] && f_hi < (long long)h->cond_f0[s] + nf, WN_E_BADARG,
                       "wn_gen_run: stream %d at positions [%lld, %lld) reads frames %lld..%lld, its window holds [%d, %d)", s,
                       q0, q1 + 1, f_lo, f_hi, h->cond_f0[s], h->cond_f0[s] + nf);
        }
    } else if (h->base.cond && h->base.cond_hop) {
        const int f_lo = a->t0 / h->base.cond_hop, f_hi = (a->t0 + a->n_evals - 1) / h->base.cond_hop;
        WN_REQUIRE(f_lo >= h->base.cond_frame0 && f_hi < h->base.cond_frame0 + h->base.cond_frames, WN_E_BADARG,
                   "wn_gen_run: evaluations [%d,%d) read frames [%d,%d], outside the condition window [%d,%d)", a->t0,
                   a->t0 + a->n_evals, f_lo, f_hi, h->base.cond_frame0, h->base.cond_frame0 + h->base.cond_frames);
    }
    const int kid = pick_kernel(h);
    WN_REQUIRE(kid != 0, WN_E_UNSUPP,
               "wn_gen_run: %d streams need a cluster kernel (modes 4, 6) for this net; mode %d does not fit in shared memory",
               h->shape.n_streams, h->mode);
    WN_REQUIRE(!(positions && kid == 3), WN_E_UNSUPP, "wn_gen_run: kernel 3 reads no stream positions (mode 2 sums alike)");
    WN_REQUIRE(h->seat_plain < 0 || h->seat_plain == (kid == 1), WN_E_STATE,
               "wn_gen_run: the rings were seated for another kernel's ring layout than kernel %d keeps", kid);
    if (h->pf_plain >= 0) {
        WN_REQUIRE(h->cur_t > 0, WN_E_STATE, "wn_gen_run: rings were prefilled but not committed (wn_gen_prefill_commit)");
        WN_REQUIRE(h->pf_plain == (kid == 1), WN_E_STATE,
                   "wn_gen_run: the rings were prefilled for kernel %s, kernel %d keeps another ring layout",
                   h->pf_plain ? "1" : "2, 3, 4 or 6", kid);
        // the first evaluation after the prefill must read a given sample: no evaluation chose the one before it
        WN_REQUIRE(a->t0 != h->pf_t_end[0] || a->t0 <= head_from, WN_E_BADARG,
                   "wn_gen_run: evaluation %d after a prefill must read a prompt sample (prompts of %d samples)", a->t0,
                   head_from + 1);
    }
    cudaStream_t st = (cudaStream_t)stream;
    // one stream without positions folds its record into the scalars (kernel 3 reads only those)
    const bool records = per_stream && (h->shape.n_streams > 1 || positions);
    if (records && h->sp_dirty) {
        // in stream order, so that a launch still reading the previous records finishes first
        const size_t NSr = h->sp.size();
        std::vector<GenStream> recs(NSr + (NSr * sizeof(int2) + sizeof(GenStream) - 1) / sizeof(GenStream));
        int2* wins = reinterpret_cast<int2*>(recs.data() + NSr);
        for (size_t s = 0; s < NSr; ++s) {
            const wn_gen_stream_params& q = h->sp[s];
            recs[s].n_given = q.n_given; recs[s].top_k = q.top_k; recs[s].trunc = stream_truncates(q, h->shape.classes);
            recs[s].temperature = q.temperature; recs[s].regularize = q.regularize; recs[s].top_p = q.top_p;
            recs[s].origin = positions ? h->pos[s].origin : 0;
            recs[s].sample0 = positions ? h->pos[s].sample0 : 0;
            recs[s].first0 = positions ? h->pos[s].first0 : 0;
            wins[s] = make_int2(stream_frames && positions ? h->pos[s].origin : 0, stream_frames ? h->cond_f0[s] : 0);
        }
        WN_CUDA(cudaMemcpyAsync(h->d_sp, recs.data(), (sizeof(GenStream) + sizeof(int2)) * NSr, cudaMemcpyHostToDevice, st));
        WN_CUDA(cudaStreamSynchronize(st));                   // recs is pageable host memory that dies with this scope
        h->sp_dirty = false;
    }
    const int bars_per_eval = 2 * h->shape.n_layers + 2;
    int done = 0;
    while (done < a->n_evals) {
        // keep the barrier counter below 2^31: chunk very long runs
        long long max_evals = (long long)0x7fffffff / ((long long)bars_per_eval * h->grid);
        int n = a->n_evals - done;
        if ((long long)n > max_evals) n = (int)max_evals;
        GenParams p = h->base;
        p.first = a->d_first; p.n_given = a->n_given; p.forced = a->d_forced; p.uniforms = a->d_uniforms;
        p.out_idx = a->d_out_idx; p.out_logits = a->d_out_logits; p.n_samples = a->n_samples;
        p.t0 = a->t0 + done; p.n_evals = n; p.temperature = a->temperature; p.regularize = a->regularize;
        p.top_k = h->top_k; p.top_p = h->top_p;
        p.trunc = a->temperature > 0.f && ((h->top_k > 0 && h->top_k < h->shape.classes) || h->top_p < 1.0);
        p.ps = nullptr; p.pcw = nullptr;
        p.head_from = head_from;
        if (per_stream && !records) {                          // the single record becomes the scalars (kernel 3 reads only those)
            const wn_gen_stream_params& q = h->sp[0];
            p.temperature = q.temperature; p.regularize = q.regularize; p.top_k = q.top_k; p.top_p = q.top_p;
            p.trunc = stream_truncates(q, h->shape.classes);
            if (stream_frames) p.cond_frame0 = h->cond_f0[0];  // and its window the shared one (origin 0 without positions)
        } else if (records) {
            p.ps = h->d_sp;
            p.pcw = reinterpret_cast<const int2*>(h->d_sp + h->shape.n_streams);
            p.trunc = h->sp_any_trunc;                          // sizes kernel 1's truncation scratch; the records decide
        }
        WN_CUDA(cudaMemsetAsync(p.bar, 0, sizeof(unsigned), st));
        int rc;
        switch (kid) {
        case 6:                                              // 256- or 512-wide nets: 8 streams per cluster
            rc = launch_gen_cl8(h, p, st);
            break;
        case 4:
            p.n_wslots = h->n_wslots_cluster;
            p.wslot_floats = h->wslot_cluster;
            rc = launch_gen_cluster(h, p, st);
            break;
        case 3:
            p.n_wslots = h->n_wslots_fast;
            p.regA = h->xn_fast;                    // the fast kernel reads its input-vector pitch from regA
            rc = p.n_wslots ? launch_gen_fast<true>(h, p, st) : launch_gen_fast<false>(h, p, st);
            break;
        case 2:
            if (h->shape.n_streams == 1)
                rc = p.n_wslots ? launch_gen_ll<1, true>(h, p, st) : launch_gen_ll<1, false>(h, p, st);
            else
                rc = p.n_wslots ? launch_gen_ll<8, true>(h, p, st) : launch_gen_ll<8, false>(h, p, st);
            break;
        default:
            rc = (h->shape.n_streams == 1) ? launch_gen<1>(h, p, st) : launch_gen<8>(h, p, st);
        }
        if (rc) return rc;
        done += n;
    }
    h->cur_t = a->t0 + a->n_evals;
    for (int s = 0; s < NS; ++s) h->run_origin[s] = positions ? h->pos[s].origin : 0;
    return 0;
}

extern "C" int wn_gen_read_trace(wn_gen_handle* h, long long* host_out, int n, void* stream) {
    WN_REQUIRE(h && host_out && n > 0 && n <= 2048, WN_E_BADARG, "wn_gen_read_trace: bad arguments");
    WN_REQUIRE(h->base.trace, WN_E_STATE, "wn_gen_read_trace: tracing is off (set WN_GEN_TRACE=1 before wn_gen_create)");
    WN_CUDA(cudaMemcpyAsync(host_out, h->base.trace, sizeof(long long) * n, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    WN_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return 0;
}

extern "C" int wn_gen_destroy(wn_gen_handle* h) {
    if (h && h->d_sp) cudaFree(h->d_sp);
    delete h;
    return 0;
}

/* the kernel wn_gen_run picks in the handle's current mode: the mode number (1-4, 6) of wn_gen_set_mode, 0 when none fits */
extern "C" int wn_gen_kernel_id(const wn_gen_handle* h) { return h ? pick_kernel(h) : 0; }

extern "C" int wn_gen_launch_info(const wn_gen_handle* h, int* grid, int* block, int* barriers_per_eval) {
    WN_REQUIRE(h, WN_E_STATE, "wn_gen_launch_info: null handle");
    const int kid = pick_kernel(h);
    WN_REQUIRE(kid != 0, WN_E_UNSUPP, "wn_gen_launch_info: no sampler kernel fits this net in mode %d", h->mode);
    int g = kid == 4 ? h->shape.n_streams * CL : h->grid;
    int b = (kid == 4 || kid == 3) ? GEN_NT + 32 : GEN_NT;                      // + the helper warp
    if (kid == 6) {
        cudaLaunchAttribute attr;
        const cudaLaunchConfig_t cfg = cl8_config(h, h->cl8_cs, nullptr, &attr);
        g = (int)cfg.gridDim.x;
        b = (int)cfg.blockDim.x;
    }
    if (grid) *grid = g;
    if (block) *block = b;
    if (barriers_per_eval) *barriers_per_eval = 2 * h->shape.n_layers + 2;      // exchange stages per evaluation
    return 0;
}
