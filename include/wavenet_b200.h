/* wavenet_b200.h -- C ABI of libwavenet_b200.so (sm_90a, H100).
 *
 * Drop-in boundary for the two hot paths of vincentherrmann/pytorch-wavenet:
 *   (T) the training-time dilated causal convolution stack  WaveNetModel.forward / .wavenet
 *       (reference wavenet_model.py:125-196, wavenet_modules.py:10-39,80-127), and
 *   (G) the Fast-WaveNet cached-queue sampling loop         WaveNetModel.generate_fast
 *       (reference wavenet_model.py:237-315, wavenet_modules.py:42-77).
 * The reference is pure Python on torch and has no FFI of its own; these entry points are what a binding
 * for those Python methods calls (see INTEGRATION.md for the ctypes stub a maintainer would add).
 *
 * Conventions
 *   - every function returns 0 on success, a positive cudaError_t value, or a negative WN_E_* argument error;
 *     nothing throws; wn_last_error_string() describes the last failure on the calling thread.
 *   - all pointers named d_* are DEVICE pointers owned by the caller; no function allocates persistent device
 *     memory behind the caller's back (the sampler handle owns only host-side bookkeeping).
 *   - every launch is asynchronous on the cudaStream_t passed as `void* stream` (NULL = legacy default stream).
 *   - "frames layout": activations are (B, L, C) fp32, C contiguous, frame t of sequence b at ((b*L+t)*C);
 *     time is ABSOLUTE (frame L-1 is the newest sample); a layer's valid frames are [start, L) and history
 *     left of `start` reads as zero -- this restates the reference's left zero-pad + time->batch fold
 *     (wavenet_modules.py:24-37) without moving data.
 */
#ifndef WAVENET_B200_H
#define WAVENET_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WN_ABI_VERSION 3

/* operand precision of the tensor-core training kernels (wn_tb_*): what the MATRIX PRODUCTS see; the residual stream and
 * skip stay fp32-class and accumulation is fp32 in both */
#define WN_PREC_BF16       1   /* single-pass bf16 operands (BASELINE.json configs[4], "bf16 training")             */
#define WN_PREC_BF16_PAIRS 2   /* bf16 (hi, lo) pairs, three MMAs per product: fp32-class, the 1e-4 parity path       */

#define WN_E_BADARG   (-1)   /* null pointer / non-positive size / inconsistent shapes        */
#define WN_E_UNSUPP   (-2)   /* shape outside what the kernels cover (message says which)     */
#define WN_E_NODEVICE (-3)   /* no sm_90 device visible                                       */
#define WN_E_STATE    (-4)   /* sampler handle used before wn_gen_bind / after destroy        */

/* ---------------------------------------------------------------- library / device */
int         wn_version(void);
const char* wn_last_error_string(void);
/* sm_count, compute capability, max opt-in shared memory per block, L2 bytes of the CURRENT device */
int         wn_device_info(int* sm_count, int* cc_major, int* cc_minor, int* smem_optin, int* l2_bytes);

/* ---------------------------------------------------------------- (T) weight packing
 * The training kernels read weights K-outer ("transposed") so a K-slab is a contiguous copy into shared
 * memory.  Packing is device->device, asynchronous, and must be redone after the parameters change.
 *
 *   filter/gate  (D,R,k) x2 + biases -> wfg_t [k*R][N1p],  bfg [N1p],  N1p = wn_n1p(D)
 *        column chunk c (128 wide): cols [0,64) = filter channels 64c.., cols [64,128) = gate channels 64c..
 *        row j*R + r holds tap j (j = 0 is the OLDEST tap, as in nn.Conv1d weight[:,:,0]) of input channel r
 *   residual (R,D,1) + skip (S,D,1) + biases -> wrs_t [D][N2p], brs [N2p], N2p = wn_n2p(R+S)
 *        cols [0,R) residual outputs, [R,R+S) skip outputs
 *   plain 1x1 (N,K,1) + bias -> w_t [K][Np], b [Np], Np = wn_n2p(N)          (end_conv_1 / end_conv_2)
 * Bias pointers may be NULL (bias=False in the reference ctor, wavenet_model.py:39): packed bias is zero. */
int wn_n1p(int D);
int wn_n2p(int N);
int wn_pack_gate_weights(const float* d_wf, const float* d_wg, const float* d_bf, const float* d_bg,
                         int R, int D, int k, float* d_wfg_t, float* d_bfg, void* stream);
int wn_pack_res_skip_weights(const float* d_wr, const float* d_ws, const float* d_br, const float* d_bs,
                             int R, int D, int S, float* d_wrs_t, float* d_brs, void* stream);
int wn_pack_1x1_weights(const float* d_w, const float* d_b, int N, int K, float* d_w_t, float* d_b_p, void* stream);

/* ---------------------------------------------------------------- (T) start conv
 * replaces: start_conv applied to the (B,classes,L) input, wavenet_model.py:65-68,127.
 * dense : d_x (B,classes,L) fp32 (any values; one-hot in the reference data path, audio_data.py:119-121)
 * index : d_idx (B,L) class indices (uint8 / int64) -- equals the dense form on one-hot input bit for bit.
 * d_w_t / d_b_p: start_conv.weight (R,classes,1) and bias packed by wn_pack_1x1_weights (N=R, K=classes), i.e.
 * a (classes, wn_n2p(R)) table whose row c is the embedding of class c.  Output d_h (B,L,R) frames layout. */
int wn_start_fwd_dense(const float* d_x, const float* d_w_t, const float* d_b_p, float* d_h,
                       int B, int classes, int L, int R, void* stream);
int wn_start_fwd_index_u8(const uint8_t* d_idx, const float* d_w_t, const float* d_b_p, float* d_h,
                          int B, int classes, int L, int R, void* stream);
int wn_start_fwd_index_i64(const int64_t* d_idx, const float* d_w_t, const float* d_b_p, float* d_h,
                           int B, int classes, int L, int R, void* stream);

/* ---------------------------------------------------------------- (T) one residual block, one launch
 * replaces the loop body of WaveNetModel.wavenet, wavenet_model.py:142-165, including both dilate() calls
 * (wavenet_modules.py:10-39) and the constant pad (:80-127):
 *     z[t]     = tanh(sum_j Wf[:,:,j] hp[t-(k-1-j)d] + bf) * sigmoid(sum_j Wg[:,:,j] hp[t-(k-1-j)d] + bg)
 *     h_out[t] = Wr z[t] + br + hp[t]                     for t in [out_start, L)
 *     skip[t]  = Ws z[t] + bs (+ skip[t] unless skip_init) for t in [skip_start, L)
 * with hp[t] = h_in[t] for t >= in_start, else 0.  d_skip is (B, L-skip_start, S) frames layout.
 * mode: 0 = exact fp32 FFMA (any shape); other values are reserved for the tensor-core variants. */
typedef struct wn_block_args {
    const float* d_h_in;  float* d_h_out;  float* d_skip;
    const float* d_wfg_t; const float* d_bfg; const float* d_wrs_t; const float* d_brs;
    int B, L, R, D, S, k, dilation;
    int in_start, out_start, skip_start, skip_init;
    int mode;
    float* d_fg_save;   /* optional (B,L,2D): tanh(F) in [0,D), sigmoid(G) in [D,2D) per frame, kept for the backward */
} wn_block_args;
int wn_block_fwd(const wn_block_args* a, void* stream);

/* ---------------------------------------------------------------- (T) the same block on the tensor cores
 * wgmma bf16 with bf16 (hi, lo) operand pairs (hi = bf16(x), lo = bf16(x - hi); hi*hi + lo*hi + hi*lo, fp32 accumulation
 * in registers): fp32-class accuracy (~3e-6 relative on the logits after 50 layers) at tensor-core rate.  Two launches
 * per block (conv+gate -> z, then the 1x1s); d_z is a caller-provided (B,L,D) workspace.  Shapes: R % 256 == 0,
 * S % 256 == 0, D % 128 == 0 (wn_tc_supported).
 * Weights are packed K-major as bf16 pair arrays [2][rows][K] ([0] = hi, [1] = lo): d_wa [2][2D][k*R] (rows in 256-wide
 * tiles: 128 filter channels then the same 128 gate channels; column j*R+r = tap j of input channel r), d_ba [2D] fp32 in
 * the same row order, d_wb [2][R+S][D] (residual rows then skip rows), d_bb [R+S] fp32. */
int wn_tc_supported(int R, int D, int S, int k);
int wn_tc_pack_block_weights(const float* d_wf, const float* d_wg, const float* d_bf, const float* d_bg,
                             const float* d_wr, const float* d_ws, const float* d_br, const float* d_bs,
                             int R, int D, int S, int k, void* d_wa, float* d_ba, void* d_wb, float* d_bb, void* stream);
typedef struct wn_tc_block_args {
    const float* d_h_in; float* d_h_out; float* d_skip; float* d_z;
    const void* d_wa; const float* d_ba; const void* d_wb; const float* d_bb;
    int B, L, R, D, S, k, dilation;
    int in_start, out_start, skip_start, skip_init;
    float* d_fg_save;
} wn_tc_block_args;
int wn_tc_block_fwd(const wn_tc_block_args* a, void* stream);
/* Debug aid (WN_TC_TRACE=1): per-stage clock64 stamps of CTA 0 of the most recent tensor-core launch, 8 per stage:
 * producer before/after the empty wait, MMA warp before/after the operand wait and after issue, splitter start/end
 * (first splitter warp), end of the last splitter warp. */
int wn_tc_read_trace(long long* host_out, int n);

/* ---------------------------------------------------------------- (T) the block as ONE tensor-core launch (round 2 default)
 * Same mathematics as wn_block_fwd (reference wavenet_model.py:142-165) for R = D = S = 256, k = 2 (wn_tb_supported), with
 * fp32-class accuracy from bf16 (hi, lo) operand pairs on wgmma (fp32 accumulation in registers); the
 * gated activation z never leaves the SM.  Activations use the CHUNKED PAIR LAYOUT: a (B, L, C) activation is stored as
 *     bf16 [b][plane: 0 = hi, 1 = lo][c / 8][t][c % 8]         x = hi + lo, hi = bf16(x), lo = bf16(x - hi)
 * (the same number of bytes as fp32 frames), and skip as fp32 [b][c / 4][t - skip_start][c % 4].  wn_pair_from_frames /
 * wn_frames_from_pair / wn_frames_from_chunks4 convert to and from the frames layout of the other entry points.
 * Weights: wn_tb_pack_all_weights writes every layer's pre-split, pre-tiled image (wn_tb_weight_bytes_per_layer(channels,
 * precision) bytes each) into ONE array d_w_all [n_layers][bytes_per_layer] and the bias vectors [bf | bg | br | bs].
 * wn_tb_start_index_* is start_conv on class indices (wavenet_model.py:65-68,127) writing that layout; *d_err (optional) is
 * set to 1 when an index is outside [0, classes) -- the reference's one-hot scatter would raise there. */
int    wn_tb_supported(int R, int D, int S, int k);                  /* R = D = S in {256, 512}, k = 2                        */
int    wn_tb_precision_supported(int channels, int precision);       /* pairs: 256 channels; single-pass bf16: 256 or 512   */
size_t wn_tb_weight_bytes_per_layer(int channels, int precision);
/* all layers in one launch: d_ptrs is a DEVICE table [n_layers][8] of {wf, wg, bf, bg, wr, ws, br, bs} (biases may be 0);
 * d_bias_all receives [n_layers][4 * channels] = [bf | bg | br | bs] */
int    wn_tb_pack_all_weights(const float* const* d_ptrs, int n_layers, int channels, int precision, void* d_w_all,
                              float* d_bias_all, void* stream);
int    wn_tb_start_index_u8(const uint8_t* d_idx, const float* d_w_t, const float* d_b_p, void* d_h_pair,
                            int B, int classes, int L, int R, int* d_err, void* stream);
int    wn_tb_start_index_i64(const int64_t* d_idx, const float* d_w_t, const float* d_b_p, void* d_h_pair,
                             int B, int classes, int L, int R, int* d_err, void* stream);
int    wn_pair_from_frames(const float* d_frames, void* d_pair, int B, int L, int C, int t_begin, void* stream);
int    wn_frames_from_pair(const void* d_pair, float* d_frames, int B, int L, int C, int t_begin, void* stream);
/* frames [t_first, t_first + n) of a chunked fp32 tensor (B, C/4, T, 4) -> (B, n, C) */
int    wn_frames_from_chunks4(const float* d_chunked, float* d_frames, int B, int T, int C, int t_first, int n, void* stream);
typedef struct wn_tb_block_args {
    const void* d_h_in; void* d_h_out;     /* chunked pairs (B, 2, channels/8, L, 8) bf16                           */
    float* d_skip;                         /* chunked (B, channels/4, L - skip_start, 4) fp32                       */
    const void* d_w_all; const float* d_bias4;   /* all layers' packed weights; THIS layer's biases [4 * channels] */
    int layer, n_layers;
    int channels, precision;               /* 256 / 512; WN_PREC_*                                                  */
    int B, L, dilation;
    int in_start, out_start, skip_start, skip_init;
    float* d_fg_save;                      /* optional chunked (B, 2*channels/4, L, 4) fp32: tanh | sigmoid outputs (for the backward) */
} wn_tb_block_args;
int    wn_tb_block_fwd(const wn_tb_block_args* a, void* stream);

/* ALL residual blocks of a forward in ONE persistent launch: the (layer, 256-frame item) list is dealt round-robin to the CTA
 * pairs, an item waits for the previous layer's items that wrote the frames it reads (device-side flags), so there is no launch
 * gap and no idle tail between layers.  h_ptrs: HOST array [n_layers + 1] of device pair tensors, layer i reads h_ptrs[i] and
 * writes h_ptrs[i+1]; buffers may repeat with period >= 3 (never h_ptrs[i+1] == h_ptrs[i] or h_ptrs[i-1]).  d_bias_all:
 * [n_layers][4*channels]; d_fg_all: optional (n_layers, B, 2*channels/4, L, 4); d_desc: n_layers * wn_tb_stack_desc_bytes()
 * bytes of 128-byte aligned device scratch; d_flags: (wn_tb_stack_items(...) + n_layers) uint32 of device scratch.
 * dilations / in_start / out_start: HOST arrays [n_layers]. */
size_t    wn_tb_stack_desc_bytes(void);
long long wn_tb_stack_items(int n_layers, int B, int L, const int* out_start);
typedef struct wn_tb_stack_args {
    const void* const* h_ptrs;
    float* d_skip; const void* d_w_all; const float* d_bias_all; float* d_fg_all;
    void* d_desc; unsigned* d_flags;
    int n_layers, channels, precision, B, L, skip_start;
    const int* dilations; const int* in_start; const int* out_start;
} wn_tb_stack_args;
int       wn_tb_stack_fwd(const wn_tb_stack_args* a, void* stream);

/* Backward of the same block on the same layout (wgmma, bf16 pairs), replacing autograd's backward through
 * wavenet_model.py:142-165.  Frame-range arguments are those of wn_block_bwd_args.  Buffers: d_dh_out (B,2,32,L,8) pair or
 * NULL (last layer), d_dskip (B,2,32,L-ds_start,8) pair on its own frame axis, d_fg the forward's d_fg_save, outputs d_dfg
 * (B,2,64,L,8) pair [dF chunks 0..31 | dG chunks 32..63], d_z (B,2,32,L,8) pair (recomputed tanh*sigmoid), d_dh_in pair.
 * d_wb_all: [n_layers][wn_tb_bwd_weight_bytes_per_layer(channels, precision)] images written by wn_tb_pack_all_bwd_weights. */
size_t wn_tb_bwd_weight_bytes_per_layer(int channels, int precision);
int    wn_tb_pack_all_bwd_weights(const float* const* d_ptrs, int n_layers, int channels, int precision, void* d_wb_all,
                                  void* stream);
typedef struct wn_tb_bwd_args {
    const void* d_dh_out; const void* d_dskip; const float* d_fg;
    void* d_dfg; void* d_z; void* d_dh_in;
    const void* d_wb_all;
    int layer, n_layers;
    int channels, precision;
    int B, L, dilation;
    int in_start, out_start;
    int gs_out, ds_start, gz, gs_in;
} wn_tb_bwd_args;
int    wn_tb_block_bwd_data(const wn_tb_bwd_args* a, void* stream);
/* All weight gradients of one block in one launch (+ a deterministic reduction): the contraction over frames reads the
 * chunked tiles as MN-major wgmma operands.  Outputs are the parameter-shaped tensors: d_gws (S,D,1), d_gwr (R,D,1),
 * d_gwf / d_gwg (D,R,2).  id_start: first frame where dh_out flows straight into dh_in (= max(out_start, gs_out)).
 * d_work: wn_tb_wgrad_workspace_bytes() bytes. */
size_t wn_tb_wgrad_workspace_bytes(void);
typedef struct wn_tb_wgrad_args {
    const void* d_dskip; const void* d_dh_out; const void* d_dfg; const void* d_z; const void* d_h_in;
    float* d_gws; float* d_gwr; float* d_gwf; float* d_gwg; float* d_work;
    int channels, precision;
    int B, L, dilation;
    int in_start, ds_start, id_start, gz;
} wn_tb_wgrad_args;
int    wn_tb_wgrad(const wn_tb_wgrad_args* a, void* stream);

/* ---------------------------------------------------------------- (T) global conditioning
 * One condition vector h (G,) per sequence (WaveNet paper section 2.5) shifts every layer's pre-activations:
 *     z[t] = tanh(Wf * x + bf + Vf h) * sigmoid(Wg * x + bg + Vg h)
 * For one sequence, bf + Vf h and bg + Vg h are just that sequence's filter / gate biases.  The kernels read them from a
 * CONDITION TABLE instead of bf / bg, so a conditioned epilogue does the same work as an unconditioned one:
 *     d_cond [n_layers][n_items][2D] fp32: bf + Vf h in [0, D), bg + Vg h in [D, 2D)   (items = sequences or sampler streams)
 * wn_cond_table builds it for all layers in one launch: d_ptrs is a DEVICE table [n_layers][4] of {Vf, Vg, bf, bg} (Vf / Vg
 * are the (D, G, 1) weights of the 1x1 conditioning convolutions; biases may be 0), d_h (n_items, G) fp32.  Each entry is a
 * sequential fp32 sum over g plus the bias, so one-hot rows (class labels) give exactly bias + one column of V, and V = 0
 * gives exactly the bias.
 * The *_cond entry points are the plain ones plus the table; a NULL table is the plain entry point.  wn_block_fwd_cond and
 * wn_tb_block_fwd_cond take ONE layer's slice [B][2D] (2 * channels), wn_tb_stack_fwd_cond the whole table [n_layers][B][2D].
 * wn_cond_frame_sums is the reduction behind the gradient of V:  dV[n][g] = sum_b h[b][g] * d_out[b][n] with
 *     d_out[b][n] = sum_{gz <= t < L} dfg[b][t][n]                            (n < C = 2D; deterministic; no atomics)
 * over the filter/gate pre-activation gradient of the backward: pair = 0 for the frames layout (B, L, C) fp32 of
 * wn_block_bwd_data, pair = 1 for the chunked pair layout (B, 2, C/8, L, 8) bf16 of wn_tb_block_bwd_data (hi + lo). */
int wn_cond_table(const float* const* d_ptrs, int n_layers, int D, int G, const float* d_h, int n_items, float* d_out,
                  void* stream);
int wn_block_fwd_cond(const wn_block_args* a, const float* d_cond, void* stream);
int wn_tb_block_fwd_cond(const wn_tb_block_args* a, const float* d_cond, void* stream);
int wn_tb_stack_fwd_cond(const wn_tb_stack_args* a, const float* d_cond, void* stream);
int wn_cond_frame_sums(const void* d_dfg, int pair, int B, int L, int C, int gz, float* d_out, void* stream);

/* ---------------------------------------------------------------- (T) local conditioning
 * A frame-rate condition series y (C channels, one frame per `hop` positions: repeat upsampling, WaveNet paper section 2.5)
 * shifts the pre-activations of position t by Uf y[t / hop] / Ug y[t / hop]:
 *     z[t] = tanh(Wf * x + bf + Vf h + Uf y[t / hop]) * sigmoid(Wg * x + bg + Vg h + Ug y[t / hop])
 * so for one sequence it is a filter / gate bias that changes every hop positions.  The condition table gains a frame axis:
 *     d_cond [n_layers][n_items][n_frames][2D] fp32        (the global table is the case n_frames = 1)
 * wn_cond_table_frames builds it for all layers in one launch:
 *     out[l][i][f][c] = base[l][i][c] + (sum_k U_l[c][k] * y[i][k][f])
 * d_base is the global table [n_layers][n_items][2D] of wn_cond_table (sum_g V h + b) for a model with both kinds of
 * conditioning, or NULL: base[l][i][c] = b_l[c] from d_ptrs (laid out as for wn_cond_table; only the bias slots are read).
 * d_u_packed [n_layers][C][wn_n1p(D)] (16-byte aligned) holds each layer's Uf / Ug (the (D, C, 1) weights of the local 1x1
 * convolutions) packed by wn_pack_gate_weights with R = C, k = 1 and no biases; d_y (n_items, C, y_ld) fp32 with frames
 * contiguous: frames [0, n_frames) of each item are read.  The U term is a sequential fp32 sum from k = 0 (register-tiled SGEMM
 * core, no TF32), the same sum wn_cond_table forms over g: U = 0 gives exactly the global table, U = V = 0 exactly the biases.
 * The *_cond_frames entry points take ONE layer's slice [B][n_frames][2D] (wn_block_fwd_cond_frames, wn_tb_block_fwd_cond_frames)
 * or the whole table (wn_tb_stack_fwd_cond_frames); position t of a sequence reads frame t / hop.  They require hop >= 1 and
 * n_frames >= ceil(L / hop); the tensor-core entry points read float2 pairs and need a 16-byte aligned table, the FFMA one
 * reads single floats.
 * wn_cond_segment_sums is the reduction behind the gradient of U:  dU[n][k] = sum_b sum_f y[b][k][f] * d_out[b][f][n] with
 *     d_out[b][f][n] = sum over t in [max(gz, f * hop), min(L, (f + 1) * hop)) of dfg[b][t][n]      (n < C = 2D)
 * on both dfg layouts (pair as for wn_cond_frame_sums); deterministic (no atomics); a frame with no position >= gz gives 0. */
int wn_cond_table_frames(const float* const* d_ptrs, const float* d_u_packed, int n_layers, int D, const float* d_base, int C,
                         const float* d_y, int y_ld, int n_items, int n_frames, float* d_out, void* stream);
int wn_block_fwd_cond_frames(const wn_block_args* a, const float* d_cond, int n_frames, int hop, void* stream);
int wn_tb_block_fwd_cond_frames(const wn_tb_block_args* a, const float* d_cond, int n_frames, int hop, void* stream);
int wn_tb_stack_fwd_cond_frames(const wn_tb_stack_args* a, const float* d_cond, int n_frames, int hop, void* stream);
int wn_cond_segment_sums(const void* d_dfg, int pair, int B, int L, int C, int gz, int hop, int n_frames, float* d_out,
                         void* stream);

/* ---------------------------------------------------------------- (T) audio-rate local conditioning (learned upsampling)
 * A learned upsampler brings the frame-rate series to one feature vector c[t] (C channels) per position, and every layer adds
 *     Uf c[t] / Ug c[t]   to its filter / gate pre-activations.
 * On the fused tensor-core blocks that is more contraction of pass A, not a table: c enters as K = Cpad more rows after the two
 * taps, Cpad = C rounded up to the k-slab width (wn_tb_local_padded_channels: 32 with bf16 pairs, 64 single-pass; channels
 * [C, Cpad) are zero in both c and U, so they add exact zeros).
 * wn_tb_local_from_channels converts c (B, C, L) fp32, frames contiguous, to the chunked pair layout (B, 2, Cpad/8, L, 8) bf16
 * with Cpad = wn_tb_local_padded_channels(C, precision), the channel count the forward entry points' tensor map reads.
 * wn_tb_pack_local_weights packs every layer's [Uf; Ug] (the (channels, C, 1) weights of the local 1x1 convolutions) into ONE
 * image d_u_all [n_layers][wn_tb_local_weight_bytes_per_layer(C, channels, precision)] with the tiling of the pass-A blocks of
 * wn_tb_pack_all_weights; d_ptrs is a DEVICE table [n_layers][2] of {Uf, Ug}.
 * wn_tb_block_fwd_local / wn_tb_stack_fwd_local are wn_tb_block_fwd / wn_tb_stack_fwd plus those K-slabs: d_c_pair is the
 * converted c of the batch (frames [0, L), shared by all layers), d_u_all the packed image.  The pass-A biases are the layer's
 * bf | bg, or, with d_cond non-NULL, the global condition table (one layer's slice [B][2 * channels] for the block entry point,
 * the whole table [n_layers][B][2 * channels] for the stack one; see wn_cond_table).  Rows past L read zeros. */
int    wn_tb_local_padded_channels(int C, int precision);
size_t wn_tb_local_weight_bytes_per_layer(int C, int channels, int precision);
int    wn_tb_local_from_channels(const float* d_c, void* d_c_pair, int B, int C, int L, int precision, void* stream);
int    wn_tb_pack_local_weights(const float* const* d_ptrs, int n_layers, int C, int channels, int precision, void* d_u_all,
                                void* stream);
int    wn_tb_block_fwd_local(const wn_tb_block_args* a, const float* d_cond, const void* d_c_pair, int C, const void* d_u_all,
                             void* stream);
int    wn_tb_stack_fwd_local(const wn_tb_stack_args* a, const float* d_cond, const void* d_c_pair, int C, const void* d_u_all,
                             void* stream);
/* The backward of the same term, on the pre-activation gradient dfg of wn_tb_block_bwd_data (chunked pairs (B, 2, N/8, L, 8),
 * N = 2 * channels; read in place as exact fp32 hi + lo) over the positions t >= gz, with c fp32 (B, C, L):
 *     wn_local_weight_grad:    d_du[n][k] = sum_b sum_{t >= gz} dfg[b][t][n] * c[b][k][t]          ([N][C] = [dUf; dUg])
 *     wn_local_data_grad_add:  d_dc[b][k][t] += sum_n d_u[n][k] * dfg[b][t][n]   for t >= gz   (d_u [N][C] fp32 = [Uf; Ug];
 *                              d_dc (B, C, L) fp32; the layers add in turn)
 * fp32 FMA with fixed summation orders and no atomics: both are deterministic.  d_work: wn_local_weight_grad_workspace_bytes
 * (N, C) bytes. */
size_t wn_local_weight_grad_workspace_bytes(int N, int C);
int    wn_local_weight_grad(const void* d_dfg, int B, int L, int N, int gz, const float* d_c, int C, float* d_work, float* d_du,
                            void* stream);
int    wn_local_data_grad_add(const void* d_dfg, int B, int L, int N, int gz, const float* d_u, int C, float* d_dc, void* stream);

/* ---------------------------------------------------------------- (T) head
 * replaces relu -> end_conv_1 -> relu -> end_conv_2 (wavenet_model.py:167-169) and forward()'s
 * slice/transpose/view (:191-196): logits (B*out_len, classes) for the LAST out_len frames only.
 * d_skip is (B, L-skip_start, S); requires out_len <= L-skip_start (the reference raises on view otherwise). */
typedef struct wn_head_args {
    const float* d_skip; float* d_logits;
    const float* d_w1_t; const float* d_b1; const float* d_w2_t; const float* d_b2;
    int B, L, S, E, classes, skip_start, out_len;
    int mode;
} wn_head_args;
int wn_head_fwd(const wn_head_args* a, void* stream);

/* ---------------------------------------------------------------- (T) backward, data gradients
 * replace autograd's backward through the layer loop (the reference calls loss.backward(), wavenet_training.py:71).
 * Gradient buffers use the frames layout; each carries a first valid frame, left of which it is structurally zero
 * and is neither read nor written:
 *   gs_out   first frame where d_dh_out may be non-zero (L if the block output is unused, as for the last layer)
 *   ds_start first frame of d_dskip, which is (B, L-ds_start, S)       (= L - output_length)
 *   gz       first frame for which dz / d_dfg / d_z are produced       (>= out_start)
 *   gs_in    first frame for which d_dh_in is produced                 (>= in_start)
 * d_wrs_rows: [(R+S)][wn_n2p(D)] rows of residual_conv.weight then skip_conv.weight (zero padded columns);
 * d_wfg_bwd : [k*2D][wn_n2p(R)], row j*2D+n holds [filter;gate].weight[n, :, j].
 * Weight gradients are plain GEMMs over the produced buffers (dWr = dh_out^T z, dWs = dskip^T z,
 * dW{f,g}[:,:,j] = d{F,G}^T h_in(t-(k-1-j)d), biases = column sums) and are left to the caller. */
typedef struct wn_block_bwd_args {
    const float* d_dh_out; const float* d_dskip; const float* d_fg;
    float* d_dfg; float* d_z; float* d_dh_in;
    const float* d_wrs_rows; const float* d_wfg_bwd;
    int B, L, R, D, S, k, dilation;
    int in_start, out_start;
    int gs_out, ds_start, gz, gs_in;
} wn_block_bwd_args;
int wn_block_bwd_data(const wn_block_bwd_args* a, void* stream);

/* The same two data-gradient GEMMs on the tensor cores (wgmma, bf16 (hi, lo) operand pairs as in wn_tc_block_fwd), for
 * R % 256 == 0, S % 256 == 0, D % 256 == 0: weights packed K-major by wn_tc_pack_block_bwd_weights into the bf16 pair arrays
 * d_wdz [2][D][R+S] (row c: residual_conv column c then skip_conv column c) and d_wdh [2][R][k*2D] (row r, column j*2D+n:
 * [filter;gate].weight[n][r][j]).  d_wrs_rows / d_wfg_bwd of the args are ignored. */
int wn_tc_bwd_supported(int R, int D, int S, int k);
int wn_tc_pack_block_bwd_weights(const float* d_wf, const float* d_wg, const float* d_wr, const float* d_ws,
                                 int R, int D, int S, int k, void* d_wdz, void* d_wdh, void* stream);
int wn_tc_block_bwd_data(const wn_block_bwd_args* a, const void* d_wdz, const void* d_wdh, void* stream);

/* head: given d_dlogits (B*out_len, classes) and the saved skip sum (B, L-skip_start, S) produce
 * d_y1 (B*out_len, E) = relu(W1 relu(skip)+b1) (recomputed), d_dy1 (B*out_len, E) and d_dskip (B, out_len, S).
 * d_w1_t/d_b1: end_conv_1 packed by wn_pack_1x1_weights; d_w2_rows [classes][wn_n2p(E)] = end_conv_2.weight rows;
 * d_w1_rows [E][wn_n2p(S)] = end_conv_1.weight rows. */
typedef struct wn_head_bwd_args {
    const float* d_dlogits; const float* d_skip;
    float* d_y1; float* d_dy1; float* d_dskip;
    const float* d_w1_t; const float* d_b1; const float* d_w2_rows; const float* d_w1_rows;
    int B, L, S, E, classes, skip_start, out_len;
} wn_head_bwd_args;
int wn_head_bwd_data(const wn_head_bwd_args* a, void* stream);

/* weight gradient of one convolution tap -- what autograd's conv1d backward-weight computes for filter/gate
 * (wavenet_model.py:145-151), residual/skip (:156,:164) and the head convolutions (:167-169):
 *     dw[n*dw_n_stride + c*dw_c_stride] = sum_{b<B} sum_{t<rows} g[b*g_seq_stride + t*ldg + n] * x[b*x_seq_stride + t*ldx + c]
 * for n < N, c < C (overwrites, exact fp32, deterministic).  d_g / d_x point at the first paired frame of sequence 0
 * (a tap shift is a pointer offset); strides are in floats, so the result can be written straight into column j of
 * an (out, in, k) weight-gradient tensor (dw_n_stride = in*k, dw_c_stride = k).  d_work: wn_wgrad_workspace_bytes(N, C)
 * bytes of scratch for the split-frames partial sums.  rows == 0 writes zeros. */
typedef struct wn_wgrad_args {
    const float* d_g; const float* d_x; float* d_dw; float* d_work;
    long long g_seq_stride, x_seq_stride, dw_n_stride, dw_c_stride;
    int ldg, ldx, B, rows, N, C;
} wn_wgrad_args;
size_t wn_wgrad_workspace_bytes(int N, int C);
int wn_wgrad(const wn_wgrad_args* a, void* stream);
/* The same contraction on the tensor cores (wgmma on bf16 hi/lo pairs, fp32 accumulation; the operand
 * tiles are transposed to K-major while they are split): C == 256, N % 128 == 0, rows >= 1, ldg / ldx / sequence
 * strides multiples of 4 floats, d_g / d_x 16-byte aligned.  Same argument block and workspace as wn_wgrad. */
int wn_tc_wgrad_supported(int N, int C);
int wn_tc_wgrad(const wn_wgrad_args* a, void* stream);

/* ---------------------------------------------------------------- (T) the rest of a training step
 * What WavenetTrainer.train does around model(x) (reference wavenet_training.py:64-76), as native launches:
 * wn_ce_fwd_bwd: F.cross_entropy(output, target) (:69) AND its gradient in one pass: *d_loss = mean_i(logsumexp(x_i) -
 *   x_i[target_i]), d_dlogits = (softmax(x_i) - onehot(target_i)) / N (may not alias d_logits); deterministic; *d_err
 *   (optional) is set when a target is outside [0, C).  d_work: wn_ce_workspace_bytes().  C <= 1024.
 * wn_adam_step: torch.optim.Adam's update (the reference's default optimizer, :24) of every tensor in one launch.  d_segs
 *   is a DEVICE array of segments, d_chunks a DEVICE array of (segment, chunk-of-4096) int pairs covering them.  All of
 *   them take the same `step` (1-based; each tensor's own count in torch.optim.Adam).  wn_adam_step_f64 takes the
 *   coefficients as double, as torch does (1 - beta2 and the bias corrections are formed in double and rounded once);
 *   wn_adam_step converts its float arguments and calls it, so 1 - 0.999f is 1.3e-5 away from 1 - 0.999.
 * wn_scatter_rows: start_conv gradient for index input: table (classes, R) = sum over frames t >= t_begin of dh[b][t][:]
 *   into row idx[b][t] (idx uint8 or int64, (B, L)), optionally also transposed into d_out_t (R, classes) = the layout of
 *   start_conv.weight; wn_colsum: out[c] = sum_r x[r][c] (bias gradients), d_work
 *   wn_colsum_workspace_bytes(rows, C); wn_relu_copy: y = max(x, 0) (the head's relu(skip) operand of a weight gradient). */
size_t wn_ce_workspace_bytes(void);
int    wn_ce_fwd_bwd(const float* d_logits, const int64_t* d_target, float* d_dlogits, float* d_loss, float* d_work, int* d_err,
                     int N, int C, void* stream);
typedef struct wn_adam_seg { float* p; const float* g; float* m; float* v; long long n; } wn_adam_seg;
int    wn_adam_step(const wn_adam_seg* d_segs, const int* d_chunks, int n_chunks, float lr, float beta1, float beta2, float eps,
                    float weight_decay, int step, void* stream);
int    wn_adam_step_f64(const wn_adam_seg* d_segs, const int* d_chunks, int n_chunks, double lr, double beta1, double beta2,
                        double eps, double weight_decay, int step, void* stream);
int    wn_scatter_rows(const void* d_idx, int idx_is_u8, const float* d_dh, float* d_table, float* d_out_t, int B, int L, int R,
                       int classes, int t_begin, void* stream);
size_t wn_colsum_workspace_bytes(long long rows, int C);
int    wn_colsum(const float* d_x, float* d_out, float* d_work, long long rows, int C, int ld, void* stream);
int    wn_relu_copy(const float* d_x, float* d_y, long long n, void* stream);
/* x *= *d_scale in place (d_scale: one float on the device -- the gradient autograd passes into the loss node,
 * wavenet_training.py:71 `loss.backward()`); no pass over x when the scalar is 1.  n % 4 == 0. */
int    wn_scale_by(float* d_x, long long n, const float* d_scale, void* stream);

/* ---------------------------------------------------------------- (G) Fast-WaveNet sampler
 * replaces WaveNetModel.generate_fast's warm-up and sampling loops (wavenet_model.py:250-302) together with
 * DilatedQueue.enqueue/dequeue/reset (wavenet_modules.py:55-77): ONE persistent cooperative kernel runs
 * `n_evals` network evaluations without returning to the host; the per-layer ring buffers live in d_rings.
 *
 * Weights are the reference's own parameter tensors, UNPACKED (state_dict layout); bias pointers may be NULL.
 * n_streams independent streams share the weights (the reference has a single stream, wavenet_model.py:179).
 * Run through the SAME kernel (wn_gen_set_mode), stream s of a multi-stream run equals a single-stream run with the
 * same inputs bit for bit; different kernels split the dot products differently (rounding-level differences). */
typedef struct wn_gen_weights {
    const float* d_start_w; const float* d_start_b;            /* (R,classes,1), (R) */
    const float* const* d_wf; const float* const* d_bf;        /* HOST arrays [n_layers] of device pointers */
    const float* const* d_wg; const float* const* d_bg;        /* (D,R,k), (D)   */
    const float* const* d_wr; const float* const* d_br;        /* (R,D,1), (R)   */
    const float* const* d_ws; const float* const* d_bs;        /* (S,D,1), (S)   */
    const float* d_end1_w; const float* d_end1_b;              /* (E,S,1), (E)   */
    const float* d_end2_w; const float* d_end2_b;              /* (classes,E,1)  */
} wn_gen_weights;

typedef struct wn_gen_shape {
    int n_layers, k, R, D, S, E, classes, n_streams;
    const int* dilations;                                      /* HOST array [n_layers] */
} wn_gen_shape;

/* bytes the caller must provide: rings (all layers, all streams) and scratch (exchange vectors, barrier) */
int wn_gen_workspace_bytes(const wn_gen_shape* s, size_t* ring_bytes, size_t* scratch_bytes);

typedef struct wn_gen_handle wn_gen_handle;
int wn_gen_create(const wn_gen_shape* s, const wn_gen_weights* w, float* d_rings, void* d_scratch,
                  wn_gen_handle** out);
/* zero the rings and the time counter (DilatedQueue.reset, wavenet_modules.py:74-77) */
int wn_gen_reset(wn_gen_handle* h, void* stream);
/* Prefill: start a run at t0 = t_end > 0 from rings written by a forward pass over the prompt instead of by evaluations
 * [0, t_end).  Layer l's input at time t (what evaluation t enqueues in ring l) is read from d_src at frame
 * frame_of_t_end - (t_end - t), stream s = sequence s of the buffer (B = n_streams, L frames), in either layout
 *     WN_GEN_SRC_FRAMES  fp32 frames (B, L, R)                   (wn_start_fwd_index_*, wn_block_fwd*)
 *     WN_GEN_SRC_PAIRS   chunked bf16 pairs (B, 2, R/8, L, 8)    (wn_tb_block_fwd*; the value is float(hi) + float(lo))
 * for the times [max(0, t_end - ring_len_l), t_end) the ring holds; slots of times < 0 keep wn_gen_reset's zeros.  The
 * rings are written in the layout of the kernel wn_gen_run would launch now (wn_gen_kernel_id): plain floats for kernel 1,
 * {value, tag = t + 1} pairs otherwise.  wn_gen_prefill_layer works only right after wn_gen_reset (WN_E_STATE otherwise);
 * wn_gen_prefill_commit(h, t_end) returns WN_E_STATE unless every layer was filled for that t_end, then moves the handle to
 * t = t_end, so the next wn_gen_run starts at t0 = t_end (evaluation t_end must read a given sample: t_end < n_given).
 * wn_gen_run returns WN_E_STATE after a prefill that was not committed, or when the kernel it would launch keeps another
 * ring layout than the one the prefill wrote. */
#define WN_GEN_SRC_FRAMES 0
#define WN_GEN_SRC_PAIRS  1
int wn_gen_prefill_layer(wn_gen_handle* h, int layer, const void* d_src, int layout, int L, int frame_of_t_end, int t_end,
                         void* stream);
int wn_gen_prefill_commit(wn_gen_handle* h, int t_end);
/* Run evaluations [t0, t0+n_evals) of a schedule with n_given given samples per stream:
 *   evaluation e takes as input  d_first[s*n_given + e]            if e <  n_given
 *                                d_forced[s*n_samples + e-n_given] if d_forced != NULL   (teacher forcing)
 *                                the index chosen at evaluation e-1 otherwise,
 *   and, when e >= n_given-1, chooses sample i = e-(n_given-1): argmax of (logits - regularize*(c-classes/2)^2)
 *   if temperature <= 0 (wavenet_model.py:290-294), else inverse-CDF sampling of softmax(./temperature) with the
 *   float64 uniform d_uniforms[s*n_samples + i] exactly as numpy.random.choice does (wavenet_model.py:282-289).
 *   d_out_idx (n_streams, n_samples) int32; d_out_logits optional (n_streams, n_samples, classes) fp32 holding
 *   logits - regularizer.  t0 must continue where the previous call stopped (0 after wn_gen_reset).          */
typedef struct wn_gen_run_args {
    const int32_t* d_first; int n_given;
    const int32_t* d_forced; const double* d_uniforms;
    int32_t* d_out_idx; float* d_out_logits;
    int n_samples;            /* row pitch of forced / uniforms / out_idx                  */
    int t0, n_evals;
    float temperature, regularize;
} wn_gen_run_args;
int wn_gen_run(wn_gen_handle* h, const wn_gen_run_args* a, void* stream);
int wn_gen_destroy(wn_gen_handle* h);
/* Which sampler kernel runs (all implement the same schedule; call right after wn_gen_reset):
 *   0  auto: 256- and 512-wide k = 2 nets of 256 classes -> the tensor-core cluster kernel 6, for any number of streams;
 *            other nets: one stream -> the single-stream L2 kernel 3, several streams -> one cluster per stream
 *            (kernel 4) where it applies, otherwise the generic kernel
 *   1  atomic grid barrier between stages (the simple reference kernel)
 *   2  generic flag-in-data exchange through L2 (any shape, any number of streams)
 *   3  single-stream L2 kernel with register-free cooperative polling (k = 2, power-of-two row split)
 *   4  cluster kernel: one 16-CTA thread-block cluster per stream, exchange through distributed shared memory
 *   6  tensor-core cluster kernel: up to 8 streams per thread-block cluster (R = D = S = E = W with W = 256 or 512,
 *      classes = 256, k = 2).  The weights of a stage enter shared memory once per 8 streams, as bf16 hi/lo pairs
 *      pre-split into MMA fragment order at wn_gen_reset (wn_gen_workspace_bytes includes the images: 1.5 MB per layer
 *      at W = 256, 6 MB per layer at W = 512, so about 505 MB for an 80-layer 512-wide net, per handle;
 *      wn_gen_weights_changed after in-place weight updates); dot products are mma.sync m16n8k16 with three MMAs per
 *      product (fp32-class: ~1e-6 on the logits); the exchange is one 512-byte st.async.v4 block per destination CTA,
 *      credited to an mbarrier there.  W = 256: clusters of 16 CTAs while all of them are co-resident (as reported by
 *      the occupancy query), else clusters of 8 CTAs that own two 16-channel slices each (more clusters per wave);
 *      wn_gen_create fixes the size.  W = 512: clusters of 16 CTAs that own two 16-channel slices each
 * WN_E_BADARG for any other mode (5 included), WN_E_UNSUPP for a kernel that does not apply to the shape.
 * Kernels 2 and 3 sum in the same order (bit-identical results); kernel 4 splits rows differently (rounding-level
 * differences). */
int wn_gen_set_mode(wn_gen_handle* h, int mode);
/* The parameter tensors given to wn_gen_create were written in place (an optimizer step): kernels 1-4 read them on every
 * launch and need nothing; kernel 6 keeps pre-split copies, which the next wn_gen_reset rebuilds after this call. */
int wn_gen_weights_changed(wn_gen_handle* h);
/* Global conditioning of the sampler: d_cond is a condition table [n_layers][n_streams][2D] (see wn_cond_table); every
 * kernel takes entry (layer, stream) as that stream's filter / gate biases.  Because the table holds bf + Vf h | bg + Vg h,
 * it must be rebuilt (wn_cond_table) after ANY change of Vf, Vg, bf or bg -- an optimizer step that updates the biases
 * included -- before the next wn_gen_run.  The table is read on every launch
 * and must stay alive while the handle samples with it; NULL clears it (unconditioned sampling). */
int wn_gen_set_condition(wn_gen_handle* h, const float* d_cond);
/* Local conditioning of the sampler: d_cond is a table window [n_layers][n_streams][n_frames][2D] (wn_cond_table_frames) of the
 * frames [frame0, frame0 + n_frames); evaluation t (position t: it reads sample t and predicts sample t + 1) takes row
 * t / hop - frame0 of its stream as the filter / gate biases.  wn_gen_run returns WN_E_BADARG when an evaluation of the
 * launch falls outside the window, so a long run is sampled window by window, each launch continuing through t0.  The same
 * lifetime rules as wn_gen_set_condition apply; NULL clears the table, and the last wn_gen_set_condition* call wins. */
int wn_gen_set_condition_frames(wn_gen_handle* h, const float* d_cond, int frame0, int n_frames, int hop);
/* Local conditioning with a window per stream (continuous batching: streams at their own positions): d_cond has the layout
 * above, [n_layers][n_streams][n_frames][2D], but stream s's rows hold frames [frame0[s], frame0[s] + n_frames) of its own
 * series; frame0 is a HOST array [n_streams], copied before the call returns.  Evaluation t of stream s reads row
 * (t - origin) / hop - frame0[s] of its stream, origin from wn_gen_set_stream_positions (0 without positions): the frame of
 * the stream's own position.  Per-stream windows need per-stream records: wn_gen_run returns WN_E_STATE without
 * wn_gen_set_stream_params, and WN_E_BADARG, before launching and with t unchanged, when a stream's frames over the launch
 * leave its window.  WN_E_BADARG for frame0[s] < 0, n_frames < 1 or hop < 1.  The lifetime rules of wn_gen_set_condition
 * apply; NULL clears the table, and the last wn_gen_set_condition* call wins (wn_gen_set_condition_frames returns to one
 * shared window). */
int wn_gen_set_condition_stream_frames(wn_gen_handle* h, const float* d_cond, const int* frame0, int n_frames, int hop);
/* Top-k and nucleus (top-p) truncation of the temperature draw, for every stream and every kernel.  Off is top_k = 0,
 * top_p = 1, which wn_gen_create starts with; the values stay on the handle until the next call.  WN_E_BADARG for
 * top_k < 0 or top_p outside (0, 1] (NaN included).  The rule, per stream and selection, on the fp32 logits l that
 * d_out_logits reports (the regularizer already subtracted):
 *   - it applies only when temperature > 0 and 0 < top_k < classes or top_p < 1; otherwise the selection is the
 *     untruncated one above, bit for bit (at temperature <= 0 the argmax is always kept, so truncation is a no-op);
 *   - p_c is the kernel's own fp32 softmax of l / temperature;
 *   - the classes are ranked by l descending, equal logits by lower class index (on l, not on p: exact and reproducible
 *     from the reported logits);
 *   - K1 is the first top_k classes of that ranking (all of them when top_k is 0 or >= classes);
 *   - K is the shortest prefix of K1, in rank order, whose float64 sum of p reaches top_p times the float64 sum of p
 *     over K1 (at least one class; decisions within float64 rounding of the threshold may go either way);
 *   - the draw is the untruncated inverse CDF restricted to K: the float64 cumulative sum of p over K in ascending index
 *     order, normalised by its last element, the number of edges <= u (searchsorted side 'right') mapped back to the
 *     kept class of that rank; a count past the end gives the largest kept index, never a dropped class.
 * Kernel 1 then needs 4 * 8 * classes more bytes of shared memory per CTA (WN_E_UNSUPP if they do not fit). */
int wn_gen_set_truncation(wn_gen_handle* h, int top_k, double top_p);
/* Per-stream sampling settings: stream s's prompt length, truncation, temperature and regularizer. */
typedef struct wn_gen_stream_params {
    int n_given, top_k;
    float temperature, regularize;
    double top_p;
} wn_gen_stream_params;
/* Give every stream its own settings: params is a HOST array [n_streams], copied before the call returns; NULL returns to
 * the scalar path (wn_gen_create starts there).  The setting stays on the handle until the next call.  WN_E_BADARG, and
 * nothing changes, for n_given < 1, top_k < 0, top_p outside (0, 1] or a non-finite temperature or regularize.  The
 * schedule of wn_gen_run then becomes, per stream s (evaluation e is still position e of every stream):
 *   - input of evaluation e: d_first[s*pitch + e] if e < n_given[s], else d_forced[s*n_samples + e - n_given[s]] when
 *     teacher forcing, else the stream's own last choice; pitch = a->n_given, which must equal the largest n_given[s];
 *   - at e >= n_given[s] - 1 the stream chooses sample i = e - (n_given[s] - 1) with its own temperature, regularize,
 *     top_k and top_p, by the rules of wn_gen_run and wn_gen_set_truncation;
 *   - the head runs at every evaluation e >= head_from = min_s n_given[s] - 1; a stream still inside its prompt there
 *     makes no selection: it reads no uniform and writes no index or logits;
 *   - n_samples stays the row pitch of forced / uniforms / out_idx / out_logits, and t0 + n_evals <= head_from + n_samples.
 * A stream that needs fewer samples than the launch runs keeps evaluating; its extra outputs land in its row's padding.
 * While records are set, a->temperature and a->regularize must be 0 and the handle's truncation off (WN_E_BADARG
 * otherwise), and d_uniforms is required when any stream has temperature > 0.  The library keeps a device copy of the
 * records (allocated at the first call, freed by wn_gen_destroy) and uploads it in stream order before the next launch. */
int wn_gen_set_stream_params(wn_gen_handle* h, const wn_gen_stream_params* params);
/* Stream positions (continuous batching): one record per stream, {origin, sample0, first0}; params is a HOST array
 * [n_streams], copied before the call returns; NULL clears them (wn_gen_create starts cleared, which is origin = sample0 =
 * first0 = 0 for every stream: the schedule above exactly).  Positions need per-stream records (WN_E_STATE otherwise);
 * WN_E_BADARG for sample0 < 0 or first0 < 0.  The handle's time t still drives the rings, the exchange and the head; with
 * positions set, per stream s:
 *   - evaluation t is position q = t - origin of the stream;
 *   - its input is d_first[s*pitch + q - first0] for q < n_given[s] (pitch = a->n_given: a row may hold just the prompt
 *     positions the launch reads), else d_forced[s*n_samples + (q - n_given[s]) - sample0] when teacher forcing, else the
 *     stream's own last choice;
 *   - at q >= n_given[s] - 1 it selects sample i = q - (n_given[s] - 1) into column i - sample0 of d_out_idx, d_out_logits
 *     and d_uniforms;
 *   - the head runs from head_from = min_s (origin + n_given[s] - 1).
 * wn_gen_run returns WN_E_BADARG, before launching, for origin > t0, a prompt read outside [0, pitch), a forced read or a
 * selection column outside [0, n_samples), and a first evaluation of a newly seated stream that reads no prompt sample.
 * A stream whose origin differs from the one it last ran with (after wn_gen_reset: 0; after wn_gen_set_time: none) must have
 * been seated at every layer at the current t for that origin (WN_E_STATE otherwise).  With positions set one stream runs
 * kernel 2 (or 4) where auto would pick kernel 3, which reads no records; mode 3 returns WN_E_UNSUPP. */
typedef struct wn_gen_stream_pos {
    int origin, sample0, first0;
} wn_gen_stream_pos;
int wn_gen_set_stream_positions(wn_gen_handle* h, const wn_gen_stream_pos* pos);
/* Seat new jobs in the listed streams ("slots") of a running handle at its current time t, one layer per call: the slot's
 * ring of layer l is written for every time of [t - ring_len_l, t), as the kernel wn_gen_run would launch now keeps it
 * ({value, tag = time + 1} pairs, plain floats for kernel 1).  With q_end[j] the position of slot slots[j] at t (its
 * origin is t - q_end[j]: 0 for a job that starts at its first prompt sample, T for one primed through position T - 1), the
 * value at a time of position q is 0 for q < 0 or when d_src is NULL, else frame frame_of_end - (q_end[j] - q) of sequence j
 * of d_src (B = n, L frames, in either WN_GEN_SRC_* layout, as for wn_gen_prefill_layer).  Every slot time a new position
 * reads is written: a reused slot's previous job wrote the same times with the same tags, so no tag could tell them apart.
 * No other stream is touched.  Works at any t, between launches.  WN_E_BADARG for a bad or repeated slot, q_end < 0, a
 * source frame below 0, or source positions that would lie at times < 0 (every kernel reads those as zero history).
 * wn_gen_set_time(h, t), right after wn_gen_reset only, moves the handle to t without evaluating, so that a primed job's
 * history lies at times >= 0 (t >= the longest ring); every stream must then be seated before the next wn_gen_run. */
int wn_gen_seat_layer(wn_gen_handle* h, int layer, int n, const int* slots, const int* q_end, const void* d_src, int layout,
                      int L, int frame_of_end, void* stream);
int wn_gen_set_time(wn_gen_handle* h, int t);
/* Synchronise the stream and report whether a launch aborted (a CTA waited > ~3 s for a tag): 0 = fine. */
int wn_gen_check(wn_gen_handle* h, void* stream);
/* Debug aid: with WN_GEN_TRACE=1 in the environment at wn_gen_create, CTA 0 stamps clock64() at 8 points of every layer
 * of the LAST evaluation of a launch (single-stream kernel only); this copies the first n stamps to the host. */
int wn_gen_read_trace(wn_gen_handle* h, long long* host_out, int n, void* stream);
/* Which kernel wn_gen_run launches in the handle's current mode: the number (1-4, 6) documented at wn_gen_set_mode, 0 when
 * none fits in shared memory (wn_gen_run then returns WN_E_UNSUPP). */
int wn_gen_kernel_id(const wn_gen_handle* h);
/* how wn_gen_run launches: grid size, block size, dependent exchange stages per evaluation (WN_E_UNSUPP when no kernel
 * fits, as for wn_gen_run) */
int wn_gen_launch_info(const wn_gen_handle* h, int* grid, int* block, int* barriers_per_eval);

#ifdef __cplusplus
}
#endif
#endif /* WAVENET_B200_H */
