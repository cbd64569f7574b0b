"""WaveNetModel with the reference's constructor, attributes, state_dict and methods
(reference wavenet_model.py), running its two hot paths on hand-written sm_90a CUDA kernels:

* ``forward`` / ``wavenet``   -> start gather/GEMM, the residual blocks (R = D = S = 256 or 512 with k = 2: the fused
                                 tensor-core block, wn_tb_*; other shapes the tensor cores cover: two wgmma launches per
                                 block with bf16-pair operands, wn_tc_block_fwd; any other shape: ONE fused fp32 kernel per
                                 block, wn_block_fwd), fused head (wn_start_fwd_*, wn_head_fwd)
* ``loss.backward()``         -> wn_head_bwd_data, per block wn_tb_block_bwd_data / wn_tc_block_bwd_data / wn_block_bwd_data
                                 for the data gradients and wn_tb_wgrad / wn_tc_wgrad / wn_wgrad for the weight gradients
                                 (a custom autograd node)
* ``generate_fast``           -> ONE persistent kernel for the whole sampling loop (wn_gen_run)

Host code is plumbing only (shape planning, buffer ownership, weight packing cache).  There is no eager /
CPU fallback: tensors must live on a CUDA device and the native library must be built, otherwise the calls
raise.  Frames layout and the absolute time axis are described in include/wavenet_b200.h.
"""
import ctypes
import math
import os
import os.path

import numpy as np
import torch
import torch.nn as nn

from wavenet_modules import *          # noqa: F401,F403  (the reference re-exports these names)
from wavenet_modules import DilatedQueue, dilate
from audio_data import *               # noqa: F401,F403
from audio_data import mu_law_expansion
import native


class StackPlan:
    """Valid frame ranges of every layer for an input of L frames (absolute time axis).

    Restates the length bookkeeping of dilate()'s left zero pad (reference wavenet_modules.py:24-27) and the
    k-tap 'valid' conv (wavenet_model.py:147-165): T_pad = ceil(T/d)*d, T_out = T_pad - d*(k-1), everything
    right-aligned to the newest frame, so layer i reads frames [in_start, L) and writes [out_start, L).
    """

    def __init__(self, dilations, kernel_size, L):
        self.L = L
        self.in_start, self.out_start = [], []
        T = L
        for d in dilations:
            t_out = int(math.ceil(T / d) * d) - d * (kernel_size - 1)
            if t_out < 1:
                raise RuntimeError(f"input of {L} frames is too short for dilation {d} with kernel size "
                                   f"{kernel_size} (the reference's conv raises here too)")
            self.in_start.append(L - T)
            self.out_start.append(L - t_out)
            T = t_out
        self.t_final = T
        self.skip_start = L - T


def prefill_window(T, dilations, kernel_size, hop=1):
    """(P0, S, W) of the sampler's ring prefill to T evaluations (_Runtime.prefill): one forward over prompt positions
    [P0, T), W = T - P0 of them, placed at buffer frames [S, S + W) with every layer's history before frame S zero.

    Ring l holds x_l[t] for t in [T - ring_len_l, T), ring_len_l = (k-1) d_l + 1, and x_l[t] depends on positions
    [t - rf_l + 1, t] (rf_0 = 1, rf_{l+1} = rf_l + (k-1) d_l), so the ring needs positions >= T - rf_{l+1} >= T - rf.
    From P0 = max(0, T - rf) the window's zero history reaches no needed value (P0 > 0), or is the reset queues' own zero
    history (P0 = 0): the forward costs at most one receptive field per stream, however long the prompt.  With local
    conditioning at `hop`, P0 is rounded down and S up to multiples of hop so that window frame f reads condition frame
    (P0 - S) / hop + f // hop.  S >= the largest (k-1) d keeps every tap inside the buffer."""
    rf = 1 + (kernel_size - 1) * sum(dilations)
    P0 = max(0, T - rf) // hop * hop
    unit = math.lcm(8, hop)
    S = max(-(-(kernel_size - 1) * max(dilations) // unit) * unit, unit)
    return P0, S, T - P0


class _Packs:
    """Lazily built packed weight groups of one model state (see _Runtime.packed_weights):
      layers              K-outer fp32 copies for the SIMT block kernels
      tc_layers           K-major bf16 (hi, lo) pair arrays for the two-launch tensor-core blocks
      tc_bwd_layers       the same for the tensor-core data-gradient GEMMs
      tb                  all layers' slot images + biases for the fused tensor-core block (wn_tb_block_fwd)
      start / end1 / end2 K-outer 1x1 weights
    """

    def __init__(self, rt):
        self.rt, self.groups = rt, {}

    def __getitem__(self, name):
        if name in ("tb", "tb_bwd", "tb_local") and name in self.groups and self.groups[name][-1] != self.rt.tb_precision():
            del self.groups[name]                       # packed for the other operand precision
        if name not in self.groups:
            rt = self.rt
            stream = torch.cuda.current_stream(rt.device()).cuda_stream
            self.groups[name] = getattr(self, "_build_" + name)(stream)
        return self.groups[name]

    def _dims(self):
        m = self.rt.model
        return (m.residual_channels, m.dilation_channels, m.skip_channels, m.end_conv_1.out_channels, m.classes,
                m.kernel_size, m.layers * m.blocks)

    def _build_layers(self, stream):
        rt, lib = self.rt, native.lib()
        R, D, S, E, Cc, k, nl = self._dims()
        P = rt._params()
        f32 = dict(device=rt.device(), dtype=torch.float32)
        n1p, n2p = lib.wn_n1p(D), lib.wn_n2p(R + S)
        out = []
        for i in range(nl):
            wfg, bfg = torch.empty(k * R, n1p, **f32), torch.empty(n1p, **f32)
            wrs, brs = torch.empty(D, n2p, **f32), torch.empty(n2p, **f32)
            (wf, bf), (wg, bg) = P["filt"][i], P["gate"][i]
            (wr, br), (wsk, bs) = P["res"][i], P["skip"][i]
            native.check(lib.wn_pack_gate_weights(wf.data_ptr(), wg.data_ptr(), native.ptr(bf), native.ptr(bg),
                                                  R, D, k, wfg.data_ptr(), bfg.data_ptr(), stream), "pack gate")
            native.check(lib.wn_pack_res_skip_weights(wr.data_ptr(), wsk.data_ptr(), native.ptr(br), native.ptr(bs),
                                                      R, D, S, wrs.data_ptr(), brs.data_ptr(), stream), "pack res/skip")
            out.append((wfg, bfg, wrs, brs))
        return out

    def _build_tc_layers(self, stream):
        rt, lib = self.rt, native.lib()
        R, D, S, E, Cc, k, nl = self._dims()
        P = rt._params()
        f32 = dict(device=rt.device(), dtype=torch.float32)
        bf16 = dict(device=rt.device(), dtype=torch.bfloat16)
        out = []
        for i in range(nl):
            (wf, bf), (wg, bg) = P["filt"][i], P["gate"][i]
            (wr, br), (wsk, bs) = P["res"][i], P["skip"][i]
            wa, ba = torch.empty(2, 2 * D, k * R, **bf16), torch.empty(2 * D, **f32)
            wb, bb = torch.empty(2, R + S, D, **bf16), torch.empty(R + S, **f32)
            native.check(lib.wn_tc_pack_block_weights(
                wf.data_ptr(), wg.data_ptr(), native.ptr(bf), native.ptr(bg), wr.data_ptr(), wsk.data_ptr(),
                native.ptr(br), native.ptr(bs), R, D, S, k, wa.data_ptr(), ba.data_ptr(), wb.data_ptr(),
                bb.data_ptr(), stream), "pack tc")
            out.append((wa, ba, wb, bb))
        return out

    def _build_tc_bwd_layers(self, stream):
        rt, lib = self.rt, native.lib()
        R, D, S, E, Cc, k, nl = self._dims()
        P = rt._params()
        bf16 = dict(device=rt.device(), dtype=torch.bfloat16)
        out = []
        for i in range(nl):
            wf, wg, wr, wsk = P["filt"][i][0], P["gate"][i][0], P["res"][i][0], P["skip"][i][0]
            wdz, wdh = torch.empty(2, D, R + S, **bf16), torch.empty(2, R, k * 2 * D, **bf16)
            native.check(lib.wn_tc_pack_block_bwd_weights(wf.data_ptr(), wg.data_ptr(), wr.data_ptr(), wsk.data_ptr(),
                                                          R, D, S, k, wdz.data_ptr(), wdh.data_ptr(), stream), "pack tc bwd")
            out.append((wdz, wdh))
        return out

    def _ptr_table(self):
        """DEVICE table [n_layers][8] of parameter pointers {wf, wg, bf, bg, wr, ws, br, bs} (0 = no bias), cached on the
        runtime while the parameters stay where they are."""
        rt = self.rt
        P = rt._params()
        nl = self._dims()[6]
        rows = []
        for i in range(nl):
            (wf, bf), (wg, bg) = P["filt"][i], P["gate"][i]
            (wr, br), (wsk, bs) = P["res"][i], P["skip"][i]
            rows.append([native.ptr(t) or 0 for t in (wf, wg, bf, bg, wr, wsk, br, bs)])
        key = tuple(map(tuple, rows))
        cached = rt.__dict__.get("_ptr_table_cache")
        if cached is None or cached[0] != key:
            cached = (key, torch.tensor(rows, dtype=torch.int64, device=rt.device()))
            rt._ptr_table_cache = cached
        return cached[1]

    def cond_table(self, h, stream):
        """Condition table [n_layers][N][2D] for the (N, G) fp32 condition rows ``h`` (wn_cond_table): every item's filter /
        gate biases bf + Vf h | bg + Vg h, which the conditioned kernels read instead of bf / bg."""
        rt, lib, m = self.rt, native.lib(), self.rt.model
        nl, D = m.layers * m.blocks, m.dilation_channels
        P = rt._params()
        rows = [[native.ptr(t) or 0 for t in (m.filter_cond_convs[i].weight, m.gate_cond_convs[i].weight,
                                              P["filt"][i][1], P["gate"][i][1])] for i in range(nl)]
        key = tuple(map(tuple, rows))
        cached = rt.__dict__.get("_cond_ptr_cache")
        if cached is None or cached[0] != key:
            cached = (key, torch.tensor(rows, dtype=torch.int64, device=rt.device()))
            rt._cond_ptr_cache = cached
        out = torch.empty(nl, h.shape[0], 2 * D, device=rt.device(), dtype=torch.float32)
        native.check(lib.wn_cond_table(cached[1].data_ptr(), nl, D, h.shape[1], h.data_ptr(), h.shape[0], out.data_ptr(),
                                       stream), "condition table")
        return out

    def _build_local_u(self, stream):
        """Every layer's local-conditioning weights Uf | Ug, packed [n_layers][C][wn_n1p(D)] for wn_cond_table_frames."""
        rt, lib, m = self.rt, native.lib(), self.rt.model
        nl, D, C = m.layers * m.blocks, m.dilation_channels, m.local_condition_channels
        n1p = lib.wn_n1p(D)
        out = torch.empty(nl, C, n1p, device=rt.device(), dtype=torch.float32)
        bias = torch.empty(n1p, device=rt.device(), dtype=torch.float32)
        for i in range(nl):
            native.check(lib.wn_pack_gate_weights(m.filter_local_convs[i].weight.data_ptr(), m.gate_local_convs[i].weight.data_ptr(),
                                                  None, None, C, D, 1, out[i].data_ptr(), bias.data_ptr(), stream), "pack local U")
        return out

    def cond_table_frames(self, h, y, f0, n_frames, stream, out=None):
        """Condition table [n_layers][N][n_frames][2D] of a locally conditioned model (wn_cond_table_frames) for frames
        [f0, f0 + n_frames) of the (N, C, F) fp32 series ``y``, with the (N, G) condition rows ``h`` of a globally conditioned
        one (else None): bf + Vf h + Uf y_f | bg + Vg h + Ug y_f for every item and frame.  The global part is the global
        table (cond_table), built once per item.  ``out``: a contiguous fp32 tensor of that shape to build it into."""
        rt, lib, m = self.rt, native.lib(), self.rt.model
        nl, D = m.layers * m.blocks, m.dilation_channels
        P = rt._params()
        base = None if h is None else self.cond_table(h, stream)
        rows = [[0, 0, native.ptr(P["filt"][i][1]) or 0, native.ptr(P["gate"][i][1]) or 0] for i in range(nl)]
        key = tuple(map(tuple, rows))
        cached = rt.__dict__.get("_lcond_ptr_cache")
        if cached is None or cached[0] != key:
            cached = (key, torch.tensor(rows, dtype=torch.int64, device=rt.device()))
            rt._lcond_ptr_cache = cached
        N, C, F = y.shape
        if out is None:
            out = torch.empty(nl, N, n_frames, 2 * D, device=rt.device(), dtype=torch.float32)
        elif tuple(out.shape) != (nl, N, n_frames, 2 * D) or out.dtype != torch.float32 or not out.is_contiguous():
            raise RuntimeError(f"wavenet_b200: a condition table of shape {tuple(out.shape)} for {N} items x {n_frames} frames")
        native.check(lib.wn_cond_table_frames(cached[1].data_ptr(), self["local_u"].data_ptr(), nl, D, native.ptr(base), C,
                                              y.data_ptr() + 4 * f0, F, N, n_frames, out.data_ptr(), stream),
                     "local condition table")
        return out

    def _build_tb(self, stream, prec=None):
        rt, lib = self.rt, native.lib()
        R, nl = self._dims()[0], self._dims()[6]
        prec, dev = prec or rt.tb_precision(), rt.device()
        tb_w = torch.empty(nl, lib.wn_tb_weight_bytes_per_layer(R, prec), device=dev, dtype=torch.uint8)
        tb_b = torch.empty(nl, 4 * R, device=dev, dtype=torch.float32)
        native.check(lib.wn_tb_pack_all_weights(self._ptr_table().data_ptr(), nl, R, prec, tb_w.data_ptr(), tb_b.data_ptr(),
                                                stream), "pack tb")
        return tb_w, tb_b, prec

    def _build_tb_local(self, stream, prec=None):
        """Every layer's [Uf; Ug] for the K-slabs of the audio-rate local conditioning (wn_tb_pack_local_weights)."""
        rt, lib, m = self.rt, native.lib(), self.rt.model
        R, nl, C = m.residual_channels, m.layers * m.blocks, m.local_condition_channels
        prec, dev = prec or rt.tb_precision(), rt.device()
        u = torch.empty(nl, lib.wn_tb_local_weight_bytes_per_layer(C, R, prec), device=dev, dtype=torch.uint8)
        ptrs = torch.tensor([[m.filter_local_convs[i].weight.data_ptr(), m.gate_local_convs[i].weight.data_ptr()]
                             for i in range(nl)], dtype=torch.int64, device=dev)
        native.check(lib.wn_tb_pack_local_weights(ptrs.data_ptr(), nl, C, R, prec, u.data_ptr(), stream), "pack tb local")
        return u, ptrs, prec

    def _build_tb_pairs(self, stream):
        """"tb" packed for bf16 pairs whatever tc_precision says (the sampler's ring prefill, _Runtime.prefill)."""
        return self["tb"] if self.rt.tb_precision() == native.PREC_BF16_PAIRS else self._build_tb(stream, native.PREC_BF16_PAIRS)

    def _build_tb_local_pairs(self, stream):
        return self["tb_local"] if self.rt.tb_precision() == native.PREC_BF16_PAIRS else \
            self._build_tb_local(stream, native.PREC_BF16_PAIRS)

    def _build_tb_bwd(self, stream):
        rt, lib = self.rt, native.lib()
        R, nl = self._dims()[0], self._dims()[6]
        prec = rt.tb_precision()
        wb = torch.empty(nl, lib.wn_tb_bwd_weight_bytes_per_layer(R, prec), device=rt.device(), dtype=torch.uint8)
        native.check(lib.wn_tb_pack_all_bwd_weights(self._ptr_table().data_ptr(), nl, R, prec, wb.data_ptr(), stream),
                     "pack tb bwd")
        return wb, prec

    def _build_head_rows(self, stream):
        """end_conv_2 / end_conv_1 weight rows zero-padded to the SIMT kernels' column pitch (wn_head_bwd_data)."""
        lib = native.lib()
        R, D, S, E, Cc, k, nl = self._dims()
        P = self.rt._params()
        pad = lambda w2d, n: torch.nn.functional.pad(w2d, (0, n - w2d.shape[1])).contiguous()
        return (pad(P["end2"][0].detach()[:, :, 0], lib.wn_n2p(E)), pad(P["end1"][0].detach()[:, :, 0], lib.wn_n2p(S)))

    def _pack1x1(self, wb, N, K, stream):
        lib = native.lib()
        f32 = dict(device=self.rt.device(), dtype=torch.float32)
        w, b = wb
        wt, bp = torch.empty(K, lib.wn_n2p(N), **f32), torch.empty(lib.wn_n2p(N), **f32)
        native.check(lib.wn_pack_1x1_weights(w.data_ptr(), native.ptr(b), N, K, wt.data_ptr(), bp.data_ptr(), stream), "pack 1x1")
        return wt, bp

    def _build_start(self, stream):
        R, D, S, E, Cc, k, nl = self._dims()
        return self._pack1x1(self.rt._params()["start"], R, Cc, stream)

    def _build_end1(self, stream):
        R, D, S, E, Cc, k, nl = self._dims()
        return self._pack1x1(self.rt._params()["end1"], E, S, stream)

    def _build_end2(self, stream):
        R, D, S, E, Cc, k, nl = self._dims()
        return self._pack1x1(self.rt._params()["end2"], Cc, E, stream)


class _Runtime:
    """Device-side state bound to one model: packed weights, workspaces, sampler handles."""

    def __init__(self, model):
        self.model = model
        self.pack_key = None
        self.packed = None
        self.ws = {}
        self.samplers = {}
        self.weights_epoch = 0                # bumped by invalidate(): parameters were written behind the version counters
        self.block_mode = "auto"     # "auto": tensor-core blocks when the shape allows, "ffma": exact-fp32 SIMT, "tc"
        self.tc_precision = "bf16x2"  # "bf16x2" (bf16 pairs, fp32-class) or "bf16" (single-pass on the fused blocks, tb_precision)
        self.wgrad_mode = "tc"        # weight gradients: "tc" (tensor cores where the shape allows) or "native" (fp32 FMA)
        self.local_table_bytes = 256 << 20   # sampler: largest local-conditioning table window (at least one frame is built)

    # ------------------------------------------------------------------ weights
    def _params(self):
        m = self.model
        n = m.layers * m.blocks
        g = lambda conv: (conv.weight, conv.bias)
        return dict(start=g(m.start_conv), filt=[g(m.filter_convs[i]) for i in range(n)],
                    gate=[g(m.gate_convs[i]) for i in range(n)], res=[g(m.residual_convs[i]) for i in range(n)],
                    skip=[g(m.skip_convs[i]) for i in range(n)], end1=g(m.end_conv_1), end2=g(m.end_conv_2))

    def tb_precision(self):
        """Operand precision of the fused tensor-core kernels for this model: ``tc_precision`` "bf16x2" -> bf16 (hi, lo)
        pairs (fp32-class; 256 channels), "bf16" -> single-pass bf16 operands with fp32 accumulation and an fp32-class
        residual / skip stream (256 or 512 channels).  512-channel nets always run single pass (the resident z image of a
        512-channel pair does not fit on the SM)."""
        R = self.model.residual_channels
        if self.tc_precision == "bf16" or R == 512:
            return native.PREC_BF16
        return native.PREC_BF16_PAIRS

    def invalidate(self):
        """Forget the packed weight copies.  The cache is keyed on (data_ptr, tensor version); writes through ``p.data``
        (the reference's optimizers.py:100, ``dist.broadcast(p.data)``) do not bump the version, so every backward and
        make_data_parallel call this, and code that edits ``p.data`` by hand between no-grad forwards must too
        (``model.invalidate_packed_weights()``)."""
        self.pack_key = None
        self.weights_epoch += 1

    def device(self):
        dev = self.model.start_conv.weight.device
        if dev.type != "cuda":
            raise RuntimeError("wavenet_b200: the model must be on a CUDA device (model.cuda()); "
                               "there is no CPU path in this implementation")
        return dev

    def packed_weights(self, stream):
        """The packed weight copies, built per group on first use (a path packs only what it reads) and forgotten when a
        parameter's (data_ptr, version) changes or after invalidate()."""
        m = self.model
        key = tuple((p.data_ptr(), p._version) for p in m.parameters())
        if key != self.pack_key or self.packed is None:
            self.device()
            for name, p in m.named_parameters():
                if p.dtype != torch.float32 or not p.is_contiguous():
                    raise RuntimeError(f"wavenet_b200: parameter {name} must be a contiguous float32 tensor "
                                       f"(got {p.dtype}, contiguous={p.is_contiguous()}); the kernels read raw fp32 memory")
            self.packed, self.pack_key = _Packs(self), key
        return self.packed

    # ------------------------------------------------------------------ training-path forward
    def stack_forward(self, x, out_len, index_input=False, save=None, cond=None, local=None, upsampled=None):
        """x: (B, classes, L) float32 one-hot/dense, or (B, L) uint8/int64 indices when index_input.
        Returns logits (B*out_len, classes) for the last out_len frames (out_len=None: all T_final frames).
        save: optional dict; filled with what the backward needs (every layer's input, tanh/sigmoid outputs, skip).
        cond: the (B, G) fp32 condition rows of a conditioned model (WaveNetModel._condition), else None.
        local: (y, hop) of a locally conditioned model, y the (B, C, F) fp32 series (WaveNetModel._local_condition), else None.
        upsampled: the (B, C, L) fp32 audio-rate features of a model with a learned upsampler (WaveNetModel._upsample), else
        None: K-slabs of pass A on the fused tensor-core blocks, the local path at hop 1 on the FFMA blocks."""
        m, lib = self.model, native.lib()
        dev = self.device()
        if x.device != dev:
            raise RuntimeError(f"wavenet_b200: input is on {x.device}, model on {dev}")
        x = x.contiguous()
        if index_input:
            if x.dim() != 2 or x.dtype not in (torch.uint8, torch.int64):
                raise RuntimeError("index input must be a (B, L) uint8 or int64 tensor")
            B, L = x.shape
        else:
            if x.dim() != 3 or x.size(1) != m.classes or x.dtype != torch.float32:
                raise RuntimeError(f"input must be a (N, {m.classes}, L) float32 tensor, got {tuple(x.shape)} {x.dtype}")
            B, _, L = x.shape
        stream = torch.cuda.current_stream(dev).cuda_stream
        W = self.packed_weights(stream)
        R, D, S = m.residual_channels, m.dilation_channels, m.skip_channels
        E, Cc, k = m.end_conv_1.out_channels, m.classes, m.kernel_size
        dil = [d for d, _ in m.dilations]
        plan = StackPlan(dil, k, L)
        if out_len is None:
            out_len = plan.t_final
        if out_len > plan.t_final:
            raise RuntimeError(f"output_length {out_len} exceeds the {plan.t_final} frames this input yields "
                               f"(shape '[{B * out_len}, {Cc}]' is invalid for input of size {B * plan.t_final * Cc})")
        f32 = dict(device=dev, dtype=torch.float32)
        n_layers = len(dil)
        if os.environ.get("WN_CHECK_INDICES") and index_input and (int(x.min()) < 0 or int(x.max()) >= Cc):
            raise RuntimeError(f"wavenet_b200: class index outside [0, {Cc}) (the reference's one-hot scatter raises here)")
        if self.tc_precision not in ("bf16x2", "bf16"):
            raise ValueError(f"tc_precision must be 'bf16x2' or 'bf16', not {self.tc_precision!r}")
        if self.block_mode not in ("auto", "tb", "tc", "ffma"):
            raise ValueError(f"block_mode must be 'auto', 'tb', 'tc' or 'ffma', not {self.block_mode!r}")
        use_tb = self.block_mode in ("auto", "tb") and bool(lib.wn_tb_supported(R, D, S, k))
        if self.block_mode == "tb" and not use_tb:
            raise RuntimeError("wavenet_b200: the fused tensor-core block needs R = D = S in (256, 512), kernel_size = 2 "
                               f"(got {R},{D},{S},{k})")
        ctab, frames = None, None
        if cond is not None or local is not None or upsampled is not None:
            if self.block_mode == "tc":
                raise RuntimeError("wavenet_b200: a conditioned model runs on the fused tensor-core blocks (block_mode 'tb' / "
                                   "'auto') or the FFMA blocks ('ffma'); the two-launch 'tc' blocks have no conditioned kernel")
            if cond is not None and cond.shape[0] != B:
                raise RuntimeError(f"wavenet_b200: {cond.shape[0]} condition rows for a batch of {B}")
            if upsampled is not None:
                if tuple(upsampled.shape) != (B, m.local_condition_channels, L):
                    raise RuntimeError(f"wavenet_b200: upsampled local features of shape {tuple(upsampled.shape)} for a batch of "
                                       f"{B} x {L} positions")
                local = (upsampled, 1)
            if local is None or (upsampled is not None and use_tb):
                ctab = None if cond is None else W.cond_table(cond, stream)
            else:
                y, hop = local
                if y.shape[0] != B or y.shape[2] < -(-L // hop):
                    raise RuntimeError(f"wavenet_b200: a local condition of shape {tuple(y.shape)} does not cover a batch of {B} "
                                       f"x {L} positions at hop {hop}")
                frames = (-(-L // hop), hop)          # the table holds the frames the L positions read
                ctab = W.cond_table_frames(cond, y, 0, frames[0], stream)
            if save is not None:
                save["cond"] = cond
                if local is not None:
                    save["local"] = local
        if use_tb:
            if save is not None and upsampled is not None:
                save["kslab"] = True          # the backward reduces dU and dc on the chunked dfg (wn_local_*_grad*)
            return self._forward_tb(x, index_input, B, L, plan, out_len, W, stream, save, ctab, frames, upsampled)
        if save is not None:
            h_all = torch.empty(n_layers + 1, B, L, R, **f32)      # h_all[i] = input of layer i
            fg_all = torch.empty(n_layers, B, L, 2 * D, **f32)     # tanh / sigmoid outputs
            skip = torch.empty(B, plan.t_final, S, **f32)
            h0 = h_all[0]
        else:
            key = (B, L)
            if key not in self.ws:
                self.ws.clear()
                self.ws[key] = (torch.empty(B, L, R, **f32), torch.empty(B, L, R, **f32),
                                torch.empty(B, plan.t_final, S, **f32))
            h0, h1, skip = self.ws[key]
        ws_t, bs_p = W["start"]
        if index_input:
            fn = lib.wn_start_fwd_index_u8 if x.dtype == torch.uint8 else lib.wn_start_fwd_index_i64
            native.check(fn(x.data_ptr(), ws_t.data_ptr(), bs_p.data_ptr(), h0.data_ptr(), B, Cc, L, R, stream), "start")
        else:
            native.check(lib.wn_start_fwd_dense(x.data_ptr(), ws_t.data_ptr(), bs_p.data_ptr(), h0.data_ptr(),
                                                B, Cc, L, R, stream), "start")
        use_tc = self.block_mode != "ffma" and ctab is None and bool(lib.wn_tc_supported(R, D, S, k))     # "auto" / "tb" n/a
        if self.block_mode == "tc" and not use_tc:
            raise RuntimeError(f"wavenet_b200: tensor-core blocks need R%256==0, S%256==0, D%128==0 (got {R},{S},{D})")
        self.last_block_mode = "tc" if use_tc else "ffma"
        if use_tc:
            zkey = ("z", B, L, D)
            if zkey not in self.ws:
                self.ws[zkey] = torch.empty(B, L, D, **f32)
            zws = self.ws[zkey]
            a = native.TcBlockArgs()
            a.B, a.L, a.R, a.D, a.S, a.k = B, L, R, D, S, k
            a.d_z = zws.data_ptr()
        else:
            a = native.BlockArgs()
            a.B, a.L, a.R, a.D, a.S, a.k, a.mode = B, L, R, D, S, k, 0
        a.d_skip, a.skip_start = skip.data_ptr(), plan.skip_start
        src, dst = (h0, h1) if save is None else (h_all[0], h_all[1])
        ev = getattr(self, "block_events", None)      # optional (start, end) CUDA events around the block launches
        if ev is not None:
            ev[0].record(torch.cuda.current_stream(dev))
        for i, d in enumerate(dil):
            a.d_h_in, a.d_h_out = src.data_ptr(), dst.data_ptr()
            a.dilation, a.in_start, a.out_start, a.skip_init = d, plan.in_start[i], plan.out_start[i], int(i == 0)
            a.d_fg_save = None if save is None else fg_all[i].data_ptr()
            if use_tc:
                wa, ba, wb, bb = W["tc_layers"][i]
                a.d_wa, a.d_ba, a.d_wb, a.d_bb = wa.data_ptr(), ba.data_ptr(), wb.data_ptr(), bb.data_ptr()
                native.check(lib.wn_tc_block_fwd(ctypes.byref(a), stream), f"tc block {i}")
            else:
                wfg, bfg, wrs, brs = W["layers"][i]
                a.d_wfg_t, a.d_bfg, a.d_wrs_t, a.d_brs = wfg.data_ptr(), bfg.data_ptr(), wrs.data_ptr(), brs.data_ptr()
                if ctab is None:
                    native.check(lib.wn_block_fwd(ctypes.byref(a), stream), f"block {i}")
                elif frames is not None:
                    native.check(lib.wn_block_fwd_cond_frames(ctypes.byref(a), ctab[i].data_ptr(), frames[0], frames[1], stream),
                                 f"block {i}")
                else:
                    native.check(lib.wn_block_fwd_cond(ctypes.byref(a), ctab[i].data_ptr(), stream), f"block {i}")
            if save is None:
                src, dst = dst, src
            elif i + 1 < n_layers:
                src, dst = h_all[i + 1], h_all[i + 2]
        if ev is not None:
            ev[1].record(torch.cuda.current_stream(dev))
        logits = torch.empty(B * out_len, Cc, device=dev, dtype=torch.float32)
        hd = native.HeadArgs()
        hd.d_skip, hd.d_logits = skip.data_ptr(), logits.data_ptr()
        (w1, b1), (w2, b2) = W["end1"], W["end2"]
        hd.d_w1_t, hd.d_b1, hd.d_w2_t, hd.d_b2 = w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr()
        hd.B, hd.L, hd.S, hd.E, hd.classes, hd.skip_start, hd.out_len, hd.mode = B, L, S, E, Cc, plan.skip_start, out_len, 0
        native.check(lib.wn_head_fwd(ctypes.byref(hd), stream), "head")
        self.launches_last_forward = 1 + len(dil) * (2 if use_tc else 1) + 1
        if save is not None:
            save.update(h_all=h_all, fg_all=fg_all, skip=skip, plan=plan, out_len=out_len, x=x,
                        index_input=index_input, B=B, L=L)
        return logits

    def _forward_tb(self, x, index_input, B, L, plan, out_len, W, stream, save=None, ctab=None, frames=None, upsampled=None):
        """Forward on the fused tensor-core blocks (wn_tb_block_fwd): chunked bf16-pair activations, one launch per residual
        block, z resident on the SM (csrc/tc_block.cu).  With ``save`` every layer's input pair and tanh/sigmoid outputs are
        kept for _backward_tb.  ``upsampled`` (B, C, L): audio-rate local features, K-slabs of pass A (wn_tb_*_fwd_local)."""
        m, lib = self.model, native.lib()
        dev = self.device()
        R, S, Cc = m.residual_channels, m.skip_channels, m.classes
        E = m.end_conv_1.out_channels
        dil = [d for d, _ in m.dilations]
        n_layers = len(dil)
        bf16 = dict(device=dev, dtype=torch.bfloat16)
        if save is not None:
            h_all = torch.empty(n_layers + 1, B, 2, R // 8, L, 8, **bf16)       # h_all[i] = input of layer i
            fg_all = torch.empty(n_layers, B, 2 * R // 4, L, 4, device=dev, dtype=torch.float32)
            skip = torch.empty(B, S // 4, plan.t_final, 4, device=dev, dtype=torch.float32)
            h0 = h_all[0]
        else:
            key = ("tb", B, L)
            if key not in self.ws:
                self.ws.clear()
                self.ws[key] = (torch.empty(3, B, 2, R // 8, L, 8, **bf16),          # three rotating activation buffers
                                torch.empty(B, S // 4, plan.t_final, 4, device=dev, dtype=torch.float32))
            hbuf, skip = self.ws[key]
            h0, h1 = hbuf[0], hbuf[1]
        ws_t, bs_p = W["start"]
        if index_input:
            fn = lib.wn_tb_start_index_u8 if x.dtype == torch.uint8 else lib.wn_tb_start_index_i64
            native.check(fn(x.data_ptr(), ws_t.data_ptr(), bs_p.data_ptr(), h0.data_ptr(), B, Cc, L, R, None, stream), "tb start")
        else:
            frames = torch.empty(B, L, R, device=dev, dtype=torch.float32)
            native.check(lib.wn_start_fwd_dense(x.data_ptr(), ws_t.data_ptr(), bs_p.data_ptr(), frames.data_ptr(),
                                                B, Cc, L, R, stream), "start")
            native.check(lib.wn_pair_from_frames(frames.data_ptr(), h0.data_ptr(), B, L, R, 0, stream), "pair from frames")
            del frames
        tb_w, tb_b, prec = W["tb"]
        if upsampled is not None:
            Cl = m.local_condition_channels
            cpad = lib.wn_tb_local_padded_channels(Cl, prec)
            c_pair = torch.empty(B, 2, cpad // 8, L, 8, **bf16)
            native.check(lib.wn_tb_local_from_channels(upsampled.data_ptr(), c_pair.data_ptr(), B, Cl, L, prec, stream),
                         "local features to pairs")
            u_all = W["tb_local"][0]
        ev = getattr(self, "block_events", None)
        if ev is not None:
            ev[0].record(torch.cuda.current_stream(dev))
        if getattr(self, "stack_launch", True):
            # all blocks in ONE persistent launch (wn_tb_stack_fwd): items of layer i+1 start as soon as the frames they read exist
            hs = [h_all[i] for i in range(n_layers + 1)] if save is not None else [hbuf[i % 3] for i in range(n_layers + 1)]
            ints = lambda v: (ctypes.c_int * n_layers)(*v)
            outs = ints(plan.out_start)
            n_items = lib.wn_tb_stack_items(n_layers, B, L, outs)
            skey = ("tb_stack", n_layers, n_items)
            if skey not in self.ws:
                self.ws[skey] = (torch.empty(n_layers * lib.wn_tb_stack_desc_bytes() + 128, device=dev, dtype=torch.uint8),
                                 torch.empty(n_items + n_layers, device=dev, dtype=torch.int32))
            desc, flags = self.ws[skey]
            sa = native.TbStackArgs()
            hp = native.ptr_array(hs)
            sa.h_ptrs = ctypes.cast(hp, native.c_void_pp)
            sa.d_skip, sa.d_w_all, sa.d_bias_all = skip.data_ptr(), tb_w.data_ptr(), tb_b.data_ptr()
            sa.d_fg_all = None if save is None else fg_all.data_ptr()
            sa.d_desc = (desc.data_ptr() + 127) // 128 * 128
            sa.d_flags = flags.data_ptr()
            sa.n_layers, sa.channels, sa.precision, sa.B, sa.L, sa.skip_start = n_layers, R, prec, B, L, plan.skip_start
            sa.dilations, sa.in_start, sa.out_start = ints(dil), ints(plan.in_start), outs
            if upsampled is not None:
                native.check(lib.wn_tb_stack_fwd_local(ctypes.byref(sa), native.ptr(ctab), c_pair.data_ptr(), Cl, u_all.data_ptr(),
                                                       stream), "tb stack")
            elif ctab is None:
                native.check(lib.wn_tb_stack_fwd(ctypes.byref(sa), stream), "tb stack")
            elif frames is not None:
                native.check(lib.wn_tb_stack_fwd_cond_frames(ctypes.byref(sa), ctab.data_ptr(), frames[0], frames[1], stream),
                             "tb stack")
            else:
                native.check(lib.wn_tb_stack_fwd_cond(ctypes.byref(sa), ctab.data_ptr(), stream), "tb stack")
            n_block_launches = 1
        else:
            a = native.TbBlockArgs()
            a.B, a.L, a.n_layers, a.channels, a.precision = B, L, n_layers, R, prec
            a.d_skip, a.skip_start, a.d_w_all = skip.data_ptr(), plan.skip_start, tb_w.data_ptr()
            a.d_fg_save = None
            src, dst = (h0, h1) if save is None else (h_all[0], h_all[1])
            for i, d in enumerate(dil):
                a.d_h_in, a.d_h_out, a.layer, a.d_bias4 = src.data_ptr(), dst.data_ptr(), i, tb_b[i].data_ptr()
                a.dilation, a.in_start, a.out_start, a.skip_init = d, plan.in_start[i], plan.out_start[i], int(i == 0)
                if save is not None:
                    a.d_fg_save = fg_all[i].data_ptr()
                if upsampled is not None:
                    native.check(lib.wn_tb_block_fwd_local(ctypes.byref(a), None if ctab is None else ctab[i].data_ptr(),
                                                           c_pair.data_ptr(), Cl, u_all.data_ptr(), stream), f"tb block {i}")
                elif ctab is None:
                    native.check(lib.wn_tb_block_fwd(ctypes.byref(a), stream), f"tb block {i}")
                elif frames is not None:
                    native.check(lib.wn_tb_block_fwd_cond_frames(ctypes.byref(a), ctab[i].data_ptr(), frames[0], frames[1], stream),
                                 f"tb block {i}")
                else:
                    native.check(lib.wn_tb_block_fwd_cond(ctypes.byref(a), ctab[i].data_ptr(), stream), f"tb block {i}")
                if save is None:
                    src, dst = dst, src
                elif i + 1 < n_layers:
                    src, dst = h_all[i + 1], h_all[i + 2]
            n_block_launches = n_layers
        if ev is not None:
            ev[1].record(torch.cuda.current_stream(dev))
        # head: the last out_len frames of skip, back in the frames layout of wn_head_fwd
        sk_frames = torch.empty(B, out_len, S, device=dev, dtype=torch.float32)
        native.check(lib.wn_frames_from_chunks4(skip.data_ptr(), sk_frames.data_ptr(), B, plan.t_final, S,
                                                plan.t_final - out_len, out_len, stream), "skip to frames")
        logits = torch.empty(B * out_len, Cc, device=dev, dtype=torch.float32)
        hd = native.HeadArgs()
        hd.d_skip, hd.d_logits = sk_frames.data_ptr(), logits.data_ptr()
        (w1, b1), (w2, b2) = W["end1"], W["end2"]
        hd.d_w1_t, hd.d_b1, hd.d_w2_t, hd.d_b2 = w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr()
        hd.B, hd.L, hd.S, hd.E, hd.classes, hd.skip_start, hd.out_len, hd.mode = B, L, S, E, Cc, L - out_len, out_len, 0
        native.check(lib.wn_head_fwd(ctypes.byref(hd), stream), "head")
        self.last_block_mode = "tb"
        self.launches_last_forward = (1 if index_input else 2) + n_block_launches + 2
        self.last_block_launches = n_block_launches
        if save is not None:
            save.update(mode="tb", h_all=h_all, fg_all=fg_all, sk_frames=sk_frames, plan=plan, out_len=out_len, x=x,
                        index_input=index_input, B=B, L=L, precision=prec)
        self.last_precision = {native.PREC_BF16: "bf16", native.PREC_BF16_PAIRS: "bf16x2"}[prec]
        return logits

    def _backward_tb(self, saved, dlogits):
        """Backward on the chunked pair layout: head (SIMT kernels on the frames layout), then per block two wgmma data-
        gradient launches (wn_tb_block_bwd_data) and one weight-gradient launch (wn_tb_wgrad).  Same frame-range logic as
        stack_backward."""
        m, lib = self.model, native.lib()
        dev = self.device()
        stream = torch.cuda.current_stream(dev).cuda_stream
        W = self.packed_weights(stream)
        P = self._params()
        plan, B, L, OL = saved["plan"], saved["B"], saved["L"], saved["out_len"]
        h_all, fg_all, sk_frames = saved["h_all"], saved["fg_all"], saved["sk_frames"]
        R, D, S = m.residual_channels, m.dilation_channels, m.skip_channels
        E, Cc, k = m.end_conv_1.out_channels, m.classes, m.kernel_size
        dil = [d for d, _ in m.dilations]
        n_layers = len(dil)
        f32 = dict(device=dev, dtype=torch.float32)
        bf16 = dict(device=dev, dtype=torch.bfloat16)
        grads = {}
        dlogits = dlogits.contiguous().view(B, OL, Cc)
        # ---------------- head (frames layout; its skip input is the (B, OL, S) slice the forward made)
        y1, dy1, dskip = torch.empty(B, OL, E, **f32), torch.empty(B, OL, E, **f32), torch.empty(B, OL, S, **f32)
        w2_rows, w1_rows = W["head_rows"]
        hb = native.HeadBwdArgs()
        hb.d_dlogits, hb.d_skip = dlogits.data_ptr(), sk_frames.data_ptr()
        hb.d_y1, hb.d_dy1, hb.d_dskip = y1.data_ptr(), dy1.data_ptr(), dskip.data_ptr()
        hb.d_w1_t, hb.d_b1 = W["end1"][0].data_ptr(), W["end1"][1].data_ptr()
        hb.d_w2_rows, hb.d_w1_rows = w2_rows.data_ptr(), w1_rows.data_ptr()
        hb.B, hb.L, hb.S, hb.E, hb.classes, hb.skip_start, hb.out_len = B, L, S, E, Cc, L - OL, OL
        native.check(lib.wn_head_bwd_data(ctypes.byref(hb), stream), "head bwd")
        ds_start = L - OL
        rskip = torch.empty_like(sk_frames)
        native.check(lib.wn_relu_copy(sk_frames.data_ptr(), rskip.data_ptr(), sk_frames.numel(), stream), "relu(skip)")
        cs_work = torch.empty(lib.wn_colsum_workspace_bytes(B * OL, max(Cc, E, S)) // 4 + 4, **f32)

        def colsum(x2d, C):
            out = torch.empty(C, **f32)
            native.check(lib.wn_colsum(x2d.data_ptr(), out.data_ptr(), cs_work.data_ptr(), B * OL, C, C, stream), "column sums")
            return out

        wg_work = torch.empty(max(lib.wn_wgrad_workspace_bytes(n_, c_) for n_, c_ in ((Cc, E), (E, S))) // 4, **f32)
        wa = native.WgradArgs()
        wa.d_work, wa.B = wg_work.data_ptr(), B
        self.wgrad_tc_calls = 0

        def head_wgrad(out, g, ldg, x, ldx, N, C):
            wa.d_g, wa.d_x, wa.d_dw = g.data_ptr(), x.data_ptr(), out.data_ptr()
            wa.ldg, wa.ldx, wa.g_seq_stride, wa.x_seq_stride = ldg, ldx, OL * ldg, OL * ldx
            wa.rows, wa.N, wa.C, wa.dw_n_stride, wa.dw_c_stride = OL, N, C, C, 1
            if OL >= 64 and lib.wn_tc_wgrad_supported(N, C):
                native.check(lib.wn_tc_wgrad(ctypes.byref(wa), stream), "tc wgrad")
                self.wgrad_tc_calls += 1
            else:
                native.check(lib.wn_wgrad(ctypes.byref(wa), stream), "wgrad")

        gw2, gw1 = torch.empty(Cc, E, 1, **f32), torch.empty(E, S, 1, **f32)
        head_wgrad(gw2, dlogits, Cc, y1, E, Cc, E)
        head_wgrad(gw1, dy1, E, rskip, S, E, S)
        grads["end_conv_2.weight"], grads["end_conv_1.weight"] = gw2, gw1
        grads["end_conv_2.bias"] = colsum(dlogits, Cc)
        grads["end_conv_1.bias"] = colsum(dy1, E)
        reducer = getattr(self, "grad_reducer", None)
        if reducer is not None:
            reducer.reduce_async([grads[n] for n in ("end_conv_2.weight", "end_conv_2.bias", "end_conv_1.weight",
                                                     "end_conv_1.bias")])
        # ---------------- residual blocks, last to first
        dskip_pair = torch.empty(B, 2, S // 8, OL, 8, **bf16)
        native.check(lib.wn_pair_from_frames(dskip.data_ptr(), dskip_pair.data_ptr(), B, OL, S, 0, stream), "dskip pair")
        dskip_bias = colsum(dskip, S) if P["skip"][0][1] is not None else None
        dfg = torch.empty(B, 2, 2 * D // 8, L, 8, **bf16)
        zbuf = torch.empty(B, 2, D // 8, L, 8, **bf16)
        dh_a, dh_b = torch.empty(B, 2, R // 8, L, 8, **bf16), torch.empty(B, 2, R // 8, L, 8, **bf16)
        work = torch.empty(lib.wn_tb_wgrad_workspace_bytes() // 4, **f32)
        wb_all, prec = W["tb_bwd"]
        if prec != saved["precision"]:
            raise RuntimeError("wavenet_b200: tc_precision changed between the forward and its backward")
        a = native.TbBwdArgs()
        a.B, a.L, a.n_layers, a.ds_start, a.channels, a.precision = B, L, n_layers, ds_start, R, prec
        a.d_dskip, a.d_dfg, a.d_z, a.d_wb_all = dskip_pair.data_ptr(), dfg.data_ptr(), zbuf.data_ptr(), wb_all.data_ptr()
        g = native.TbWgradArgs()
        g.B, g.L, g.ds_start, g.channels, g.precision = B, L, ds_start, R, prec
        g.d_dskip, g.d_dfg, g.d_z, g.d_work = dskip_pair.data_ptr(), dfg.data_ptr(), zbuf.data_ptr(), work.data_ptr()
        dh_out, gs_out = None, L
        self.last_bwd_mode = "tb"
        for i in range(n_layers - 1, -1, -1):
            d = dil[i]
            in_s, out_s = plan.in_start[i], plan.out_start[i]
            (wf, bf), (wgt, bg) = P["filt"][i], P["gate"][i]
            (wr, br), (wsk, bs) = P["res"][i], P["skip"][i]
            gz = max(out_s, min(gs_out, ds_start))
            id_start = max(out_s, gs_out)
            gs_in = max(in_s, min(id_start, gz - (k - 1) * d))
            dh_in = dh_a if dh_out is not dh_a else dh_b
            a.d_dh_out = None if dh_out is None else dh_out.data_ptr()
            a.d_fg, a.d_dh_in, a.layer = fg_all[i].data_ptr(), dh_in.data_ptr(), i
            a.dilation, a.in_start, a.out_start = d, in_s, out_s
            a.gs_out, a.gz, a.gs_in = gs_out, gz, gs_in
            native.check(lib.wn_tb_block_bwd_data(ctypes.byref(a), stream), f"tb block bwd {i}")
            # the block's four weight gradients are views of ONE bucket: the all-reduce runs in place on it
            bucket = torch.empty(S * D + R * D + 2 * D * R * k, **f32)
            gws, gwr = bucket[:S * D].view(S, D, 1), bucket[S * D:S * D + R * D].view(R, D, 1)
            gwf = bucket[S * D + R * D:S * D + R * D + D * R * k].view(D, R, k)
            gwg = bucket[S * D + R * D + D * R * k:].view(D, R, k)
            g.d_dh_out, g.d_h_in = a.d_dh_out, h_all[i].data_ptr()
            g.d_gws, g.d_gwr, g.d_gwf, g.d_gwg = gws.data_ptr(), gwr.data_ptr(), gwf.data_ptr(), gwg.data_ptr()
            g.dilation, g.in_start, g.id_start, g.gz = d, in_s, id_start, gz
            native.check(lib.wn_tb_wgrad(ctypes.byref(g), stream), f"tb wgrad {i}")
            grads[f"skip_convs.{i}.weight"], grads[f"residual_convs.{i}.weight"] = gws, gwr
            grads[f"filter_convs.{i}.weight"], grads[f"gate_convs.{i}.weight"] = gwf, gwg
            if bs is not None:
                grads[f"skip_convs.{i}.bias"] = dskip_bias.clone()
            if br is not None:
                grads[f"residual_convs.{i}.bias"] = (dh_out[:, :, :, id_start:, :].float().sum((0, 1, 3)).reshape(R)
                                                     if dh_out is not None and id_start < L else torch.zeros_like(br))
            if bf is not None:
                bsum = dfg[:, :, :, gz:, :].float().sum((0, 1, 3)).reshape(2 * D)
                grads[f"filter_convs.{i}.bias"], grads[f"gate_convs.{i}.bias"] = bsum[:D].clone(), bsum[D:].clone()
            cgrads = self.cond_weight_grads(saved, grads, i, dfg, 1, gz, stream) + \
                self.local_weight_grads(saved, grads, i, dfg, 1, gz, stream)
            if reducer is not None:
                reducer.reduce_flat_async(bucket)
                reducer.reduce_async(cgrads)
                if bf is not None or br is not None or bs is not None:
                    reducer.reduce_async([grads.get(f"{n}.{i}.bias") for n in ("filter_convs", "gate_convs", "residual_convs",
                                                                              "skip_convs")])
            dh_out, gs_out = dh_in, gs_in
        # ---------------- start conv
        dh0_frames = torch.empty(B, L, R, **f32)
        native.check(lib.wn_frames_from_pair(dh_out.data_ptr(), dh0_frames.data_ptr(), B, L, R, gs_out, stream), "dh0 frames")
        dh0 = dh0_frames[:, gs_out:, :]
        x = saved["x"]
        if saved["index_input"]:
            table, gw = torch.empty(Cc, R, **f32), torch.empty(R, Cc, 1, **f32)
            native.check(lib.wn_scatter_rows(x.data_ptr(), int(x.dtype == torch.uint8), dh0_frames.data_ptr(), table.data_ptr(),
                                             gw.data_ptr(), B, L, R, Cc, gs_out, stream), "start conv gradient")
            grads["start_conv.weight"] = gw
        else:
            grads["start_conv.weight"] = torch.einsum("btr,bct->rc", dh0, x[:, :, gs_out:]).unsqueeze(-1)
        if P["start"][1] is not None:
            grads["start_conv.bias"] = dh0.sum((0, 1))
        if reducer is not None:
            reducer.reduce_async([grads["start_conv.weight"], grads.get("start_conv.bias")])
            reducer.wait_all()
        return grads

    def cond_weight_grads(self, saved, grads, i, dfg, pair, gz, stream):
        """Gradients of layer i's conditioning weights: dV[n][g] = sum_b h[b][g] * sum_{t >= gz} dfg[b][t][n]
        (wn_cond_frame_sums per sequence, then the contraction over the batch).  Returns them, or [] when unconditioned."""
        h = saved.get("cond")
        if h is None:
            return []
        B, L, D = saved["B"], saved["L"], self.model.dilation_channels
        sums = torch.empty(B, 2 * D, device=h.device, dtype=torch.float32)
        native.check(native.lib().wn_cond_frame_sums(dfg.data_ptr(), pair, B, L, 2 * D, gz, sums.data_ptr(), stream),
                     "condition frame sums")
        dv = torch.einsum("bn,bg->ng", sums, h)
        gf, gg = dv[:D].unsqueeze(-1).contiguous(), dv[D:].unsqueeze(-1).contiguous()
        grads[f"filter_cond_convs.{i}.weight"], grads[f"gate_cond_convs.{i}.weight"] = gf, gg
        return [gf, gg]

    def local_weight_grads(self, saved, grads, i, dfg, pair, gz, stream):
        """Gradients of layer i's local-conditioning weights, dU[n][k] = sum_b sum_f y[b][k][f] * S[b][f][n] with S the
        per-frame sums of dfg over the positions >= gz (wn_cond_segment_sums), and this layer's share of the gradient of the
        series, dy[b][k][f] += sum_n S[b][f][n] * U[n][k] (kept in saved["local_dy"]; layers add in a fixed order, last to
        first).  Returns [dUf, dUg], or [] when the model is not locally conditioned."""
        local = saved.get("local")
        if local is None:
            return []
        y, hop = local
        m = self.model
        B, L, D = saved["B"], saved["L"], m.dilation_channels
        if saved.get("kslab"):
            # audio-rate features c = y (B, C, L) of the K-slab forward: both contractions read the chunked dfg in place
            lib, C = native.lib(), y.shape[1]
            du = torch.empty(2 * D, C, device=y.device, dtype=torch.float32)
            work = torch.empty(lib.wn_local_weight_grad_workspace_bytes(2 * D, C) // 4, device=y.device, dtype=torch.float32)
            native.check(lib.wn_local_weight_grad(dfg.data_ptr(), B, L, 2 * D, gz, y.data_ptr(), C, work.data_ptr(),
                                                  du.data_ptr(), stream), "local weight gradient")
            gf, gg = du[:D].unsqueeze(-1), du[D:].unsqueeze(-1)
            grads[f"filter_local_convs.{i}.weight"], grads[f"gate_local_convs.{i}.weight"] = gf, gg
            if "local_dy" in saved:
                U = torch.cat([m.filter_local_convs[i].weight.detach(), m.gate_local_convs[i].weight.detach()], 0)[:, :, 0]
                native.check(lib.wn_local_data_grad_add(dfg.data_ptr(), B, L, 2 * D, gz, U.contiguous().data_ptr(), C,
                                                        saved["local_dy"].data_ptr(), stream), "local data gradient")
            return [gf, gg]
        nf = -(-L // hop)
        S = torch.empty(B, nf, 2 * D, device=y.device, dtype=torch.float32)
        native.check(native.lib().wn_cond_segment_sums(dfg.data_ptr(), pair, B, L, 2 * D, gz, hop, nf, S.data_ptr(), stream),
                     "condition segment sums")
        yf = y[:, :, :nf]
        du = torch.einsum("bfn,bkf->nk", S, yf)
        gf, gg = du[:D].unsqueeze(-1).contiguous(), du[D:].unsqueeze(-1).contiguous()
        grads[f"filter_local_convs.{i}.weight"], grads[f"gate_local_convs.{i}.weight"] = gf, gg
        if "local_dy" in saved:
            U = torch.cat([m.filter_local_convs[i].weight.detach(), m.gate_local_convs[i].weight.detach()], 0)[:, :, 0]
            saved["local_dy"][:, :, :nf] += torch.einsum("bfn,nk->bkf", S, U)
        return [gf, gg]

    # ------------------------------------------------------------------ training-path backward
    def ffma_bwd_weights(self, i):
        """Weight rows of layer i for wn_block_bwd_data: d_wrs_rows [(R+S)][wn_n2p(D)] (residual_conv.weight rows, then
        skip_conv.weight rows) and d_wfg_bwd [k*2D][wn_n2p(R)] (row j*2D + n: [filter; gate].weight[n, :, j]), zero padded."""
        lib, P = native.lib(), self._params()
        m = self.model
        R, D, k = m.residual_channels, m.dilation_channels, m.kernel_size
        pad_cols = lambda w2d, n: torch.nn.functional.pad(w2d, (0, n - w2d.shape[1])).contiguous()
        (wf, _), (wg, _), (wr, _), (wsk, _) = P["filt"][i], P["gate"][i], P["res"][i], P["skip"][i]
        wrs_rows = pad_cols(torch.cat([wr.detach()[:, :, 0], wsk.detach()[:, :, 0]], 0), lib.wn_n2p(D))
        wfg_bwd = pad_cols(torch.cat([wf.detach(), wg.detach()], 0).permute(2, 0, 1).reshape(k * 2 * D, R), lib.wn_n2p(R))
        return wrs_rows, wfg_bwd

    def stack_backward(self, saved, dlogits):
        """Gradients of all parameters given d(loss)/d(logits) (B*out_len, classes).  Data gradients run on the
        wn_*_bwd_data kernels, the weight gradients on wn_tc_wgrad / wn_wgrad over the buffers those kernels produce
        (bias gradients are row sums; the start-conv gradient is a scatter-add of dh over the input indices).
        Returns a dict name -> gradient tensor shaped like the parameter."""
        if saved.get("mode") == "tb":
            return self._backward_tb(saved, dlogits)
        m, lib = self.model, native.lib()
        dev = self.device()
        stream = torch.cuda.current_stream(dev).cuda_stream
        W = self.packed_weights(stream)
        P = self._params()
        plan, B, L, OL = saved["plan"], saved["B"], saved["L"], saved["out_len"]
        h_all, fg_all, skip = saved["h_all"], saved["fg_all"], saved["skip"]
        R, D, S = m.residual_channels, m.dilation_channels, m.skip_channels
        E, Cc, k = m.end_conv_1.out_channels, m.classes, m.kernel_size
        dil = [d for d, _ in m.dilations]
        n_layers = len(dil)
        f32 = dict(device=dev, dtype=torch.float32)
        pad_cols = lambda w2d, n: torch.nn.functional.pad(w2d, (0, n - w2d.shape[1])).contiguous()
        grads = {}
        dlogits = dlogits.contiguous().view(B, OL, Cc)
        # ---------------- head
        w1, b1 = P["end1"]
        w2, b2 = P["end2"]
        y1 = torch.empty(B, OL, E, **f32)
        dy1 = torch.empty(B, OL, E, **f32)
        dskip = torch.empty(B, OL, S, **f32)
        w2_rows = pad_cols(w2.detach()[:, :, 0], lib.wn_n2p(E))
        w1_rows = pad_cols(w1.detach()[:, :, 0], lib.wn_n2p(S))
        hb = native.HeadBwdArgs()
        hb.d_dlogits, hb.d_skip = dlogits.data_ptr(), skip.data_ptr()
        hb.d_y1, hb.d_dy1, hb.d_dskip = y1.data_ptr(), dy1.data_ptr(), dskip.data_ptr()
        hb.d_w1_t, hb.d_b1 = W["end1"][0].data_ptr(), W["end1"][1].data_ptr()
        hb.d_w2_rows, hb.d_w1_rows = w2_rows.data_ptr(), w1_rows.data_ptr()
        hb.B, hb.L, hb.S, hb.E, hb.classes, hb.skip_start, hb.out_len = B, L, S, E, Cc, plan.skip_start, OL
        native.check(lib.wn_head_bwd_data(ctypes.byref(hb), stream), "head bwd")
        ds_start = L - OL
        rskip = torch.relu(skip[:, ds_start - plan.skip_start:, :])
        # weight gradients: wgrad_mode "native" = wn_wgrad (split-frames fp32 FMA kernel, wgrad.cu); "tc" = wn_tc_wgrad
        # (tensor cores, bf16 pairs) where the shape allows, else wn_wgrad
        wgrad_mode = getattr(self, "wgrad_mode", "tc")
        if wgrad_mode not in ("native", "tc"):
            raise ValueError(f"wgrad_mode must be 'native' or 'tc', not {wgrad_mode!r}")
        self.wgrad_tc_calls = 0
        wg_work = torch.empty(max(lib.wn_wgrad_workspace_bytes(n_, c_) for n_, c_ in
                                  ((Cc, E), (E, S), (S, D), (R, D), (2 * D, R))) // 4, **f32)
        wa = native.WgradArgs()
        wa.d_work, wa.B = wg_work.data_ptr(), B

        def wgrad(out, g, g_off, ldg, g_seq, x, x_off, ldx, x_seq, rows, N, C, n_stride=None, c_stride=1, out_off=0):
            """out[n, c] (+ strides) = sum_b sum_t g[b, t, n] * x[b, t, c]; offsets in floats from the tensors' bases"""
            wa.d_g, wa.d_x = g.data_ptr() + 4 * g_off, x.data_ptr() + 4 * x_off
            wa.d_dw = out.data_ptr() + 4 * out_off
            wa.ldg, wa.ldx, wa.g_seq_stride, wa.x_seq_stride = ldg, ldx, g_seq, x_seq
            wa.rows, wa.N, wa.C = rows, N, C
            wa.dw_n_stride, wa.dw_c_stride = (C * c_stride if n_stride is None else n_stride), c_stride
            if (wgrad_mode == "tc" and rows >= 64 and lib.wn_tc_wgrad_supported(N, C) and ldg % 4 == 0 and ldx % 4 == 0
                    and g_seq % 4 == 0 and x_seq % 4 == 0 and wa.d_g % 16 == 0 and wa.d_x % 16 == 0):
                native.check(lib.wn_tc_wgrad(ctypes.byref(wa), stream), "tc wgrad")
                self.wgrad_tc_calls += 1
            else:
                native.check(lib.wn_wgrad(ctypes.byref(wa), stream), "wgrad")

        rskip = rskip.contiguous()
        gw2, gw1 = torch.empty(Cc, E, 1, **f32), torch.empty(E, S, 1, **f32)
        wgrad(gw2, dlogits, 0, Cc, OL * Cc, y1, 0, E, OL * E, OL, Cc, E)
        wgrad(gw1, dy1, 0, E, OL * E, rskip, 0, S, OL * S, OL, E, S)
        grads["end_conv_2.weight"], grads["end_conv_1.weight"] = gw2, gw1
        grads["end_conv_2.bias"] = dlogits.sum((0, 1))
        grads["end_conv_1.bias"] = dy1.sum((0, 1))
        reducer = getattr(self, "grad_reducer", None)      # data_parallel.GradientAverager or None
        if reducer is not None:
            reducer.reduce_async([grads[n] for n in ("end_conv_2.weight", "end_conv_2.bias", "end_conv_1.weight",
                                                     "end_conv_1.bias")])
        # ---------------- residual blocks, last to first
        dfg = torch.empty(B, L, 2 * D, **f32)
        zbuf = torch.empty(B, L, D, **f32)
        dh_a, dh_b = torch.empty(B, L, R, **f32), torch.empty(B, L, R, **f32)
        dh_out, gs_out = None, L
        use_tc_bwd = self.block_mode != "ffma" and bool(lib.wn_tc_bwd_supported(R, D, S, k))
        self.last_bwd_mode = "tc" if use_tc_bwd else "ffma"
        a = native.BlockBwdArgs()
        a.B, a.L, a.R, a.D, a.S, a.k, a.ds_start = B, L, R, D, S, k, ds_start
        a.d_dskip, a.d_dfg, a.d_z = dskip.data_ptr(), dfg.data_ptr(), zbuf.data_ptr()
        for i in range(n_layers - 1, -1, -1):
            d = dil[i]
            in_s, out_s = plan.in_start[i], plan.out_start[i]
            (wf, bf), (wg, bg) = P["filt"][i], P["gate"][i]
            (wr, br), (wsk, bs) = P["res"][i], P["skip"][i]
            gz = max(out_s, min(gs_out, ds_start))
            id_start = max(out_s, gs_out)
            gs_in = max(in_s, min(id_start, gz - (k - 1) * d))
            dh_in = dh_a if dh_out is not dh_a else dh_b
            a.d_dh_out = None if dh_out is None else dh_out.data_ptr()
            a.d_fg, a.d_dh_in = fg_all[i].data_ptr(), dh_in.data_ptr()
            a.dilation, a.in_start, a.out_start = d, in_s, out_s
            a.gs_out, a.gz, a.gs_in = gs_out, gz, gs_in
            if use_tc_bwd:
                wdz, wdh = W["tc_bwd_layers"][i]
                native.check(lib.wn_tc_block_bwd_data(ctypes.byref(a), wdz.data_ptr(), wdh.data_ptr(), stream), f"tc block bwd {i}")
            else:
                wrs_rows, wfg_bwd = self.ffma_bwd_weights(i)
                a.d_wrs_rows, a.d_wfg_bwd = wrs_rows.data_ptr(), wfg_bwd.data_ptr()
                native.check(lib.wn_block_bwd_data(ctypes.byref(a), stream), f"block bwd {i}")
            # weight gradients: plain GEMMs over (frames x channels) slices
            h_in = h_all[i]
            gws = torch.empty(S, D, 1, **f32)
            wgrad(gws, dskip, 0, S, OL * S, zbuf, ds_start * D, D, L * D, OL, S, D)
            grads[f"skip_convs.{i}.weight"] = gws
            if dh_out is not None and id_start < L:
                gwr = torch.empty(R, D, 1, **f32)
                wgrad(gwr, dh_out, id_start * R, R, L * R, zbuf, id_start * D, D, L * D, L - id_start, R, D)
                grads[f"residual_convs.{i}.weight"] = gwr
            else:
                grads[f"residual_convs.{i}.weight"] = torch.zeros_like(wr)
            gfg = torch.empty(2 * D, R, k, **f32)          # filter rows then gate rows, like the packed dfg columns
            for j in range(k):
                sh = (k - 1 - j) * d
                lo = min(L, max(gz, in_s + sh))           # frames whose tap j lands on real (non-padded) input
                wgrad(gfg, dfg, lo * 2 * D, 2 * D, L * 2 * D, h_in, (lo - sh) * R, R, L * R, L - lo, 2 * D, R,
                      n_stride=R * k, c_stride=k, out_off=j)
            gwf, gwg = gfg[:D], gfg[D:]
            if bs is not None:
                grads[f"skip_convs.{i}.bias"] = dskip.sum((0, 1))
            if br is not None:
                grads[f"residual_convs.{i}.bias"] = (dh_out[:, id_start:, :].sum((0, 1)) if dh_out is not None and id_start < L
                                                     else torch.zeros_like(br))
            grads[f"filter_convs.{i}.weight"], grads[f"gate_convs.{i}.weight"] = gwf, gwg
            if bf is not None:
                bsum = dfg[:, gz:, :].sum((0, 1))
                grads[f"filter_convs.{i}.bias"], grads[f"gate_convs.{i}.bias"] = bsum[:D].clone(), bsum[D:].clone()
            cgrads = self.cond_weight_grads(saved, grads, i, dfg, 0, gz, stream) + \
                self.local_weight_grads(saved, grads, i, dfg, 0, gz, stream)
            if reducer is not None:
                reducer.reduce_async([grads.get(f"{n}.{i}.{wb}") for n in ("filter_convs", "gate_convs", "residual_convs",
                                                                         "skip_convs") for wb in ("weight", "bias")] + cgrads)
            dh_out, gs_out = dh_in, gs_in
        # ---------------- start conv
        dh0 = dh_out[:, gs_out:, :]
        x = saved["x"]
        if saved["index_input"]:
            table = torch.zeros(Cc, R, **f32)
            table.index_add_(0, x[:, gs_out:].reshape(-1).long(), dh0.reshape(-1, R))
            grads["start_conv.weight"] = table.t().contiguous().unsqueeze(-1)
        else:
            grads["start_conv.weight"] = torch.einsum("btr,bct->rc", dh0, x[:, :, gs_out:]).unsqueeze(-1)
        if P["start"][1] is not None:
            grads["start_conv.bias"] = dh0.sum((0, 1))
        if reducer is not None:
            reducer.reduce_async([grads["start_conv.weight"], grads.get("start_conv.bias")])
            reducer.wait_all()
        return grads

    # ------------------------------------------------------------------ sampler
    def sampler_keys(self, n_streams):
        """(key, wkey) of a sampler handle: the parameter tensors it reads, and the state of their values"""
        m = self.model
        return ((n_streams, tuple(p.data_ptr() for p in m.parameters())),
                (tuple(p._version for p in m.parameters()), self.weights_epoch))

    def sampler(self, n_streams):
        lib = native.lib()
        key, wkey = self.sampler_keys(n_streams)
        s = self.samplers.get(n_streams)
        if s is not None and s["key"] == key:
            if s["wkey"] != wkey:                 # same tensors, new values: the batched kernel re-splits its weight images
                native.check(lib.wn_gen_weights_changed(s["handle"]), "gen weights changed")
                s["wkey"] = wkey
            return s
        if s is not None:
            lib.wn_gen_destroy(s["handle"])
        s = self.new_sampler(n_streams)
        self.samplers[n_streams] = s
        return s

    def new_sampler(self, n_streams):
        """A fresh sampler handle for n_streams streams with its workspaces (the caller owns it: wn_gen_destroy)."""
        m, lib = self.model, native.lib()
        dev = self.device()
        P = self._params()
        key, wkey = self.sampler_keys(n_streams)
        n = m.layers * m.blocks
        dil = (ctypes.c_int * n)(*[d for d, _ in m.dilations])
        shape = native.GenShape(n, m.kernel_size, m.residual_channels, m.dilation_channels, m.skip_channels,
                                m.end_conv_1.out_channels, m.classes, n_streams, dil)
        rb, sb = ctypes.c_size_t(), ctypes.c_size_t()
        native.check(lib.wn_gen_workspace_bytes(ctypes.byref(shape), ctypes.byref(rb), ctypes.byref(sb)), "gen ws")
        rings = torch.zeros(rb.value // 4, device=dev, dtype=torch.float32)
        scratch = torch.zeros(sb.value, device=dev, dtype=torch.uint8)
        for grp in ("filt", "gate", "res", "skip"):
            for w, b in P[grp]:
                if not w.is_contiguous() or (b is not None and not b.is_contiguous()):
                    raise RuntimeError("wavenet_b200: parameters must be contiguous")
        keep = [native.ptr_array([w.data for w, _ in P[g]]) for g in ("filt", "gate", "res", "skip")]
        keepb = [native.ptr_array([None if b is None else b.data for _, b in P[g]]) for g in ("filt", "gate", "res", "skip")]
        cast = lambda arr: ctypes.cast(arr, native.c_void_pp)
        wts = native.GenWeights(P["start"][0].data_ptr(), native.ptr(P["start"][1]),
                                cast(keep[0]), cast(keepb[0]), cast(keep[1]), cast(keepb[1]),
                                cast(keep[2]), cast(keepb[2]), cast(keep[3]), cast(keepb[3]),
                                P["end1"][0].data_ptr(), P["end1"][1].data_ptr(),
                                P["end2"][0].data_ptr(), P["end2"][1].data_ptr())
        handle = ctypes.c_void_p()
        native.check(lib.wn_gen_create(ctypes.byref(shape), ctypes.byref(wts), rings.data_ptr(), scratch.data_ptr(),
                                       ctypes.byref(handle)), "gen create")
        return dict(key=key, wkey=wkey, handle=handle, rings=rings, scratch=scratch, n_streams=n_streams)

    def reset_sampler(self, s, stream):
        lib = native.lib()
        native.check(lib.wn_gen_reset(s["handle"], stream), "gen reset")
        mode = getattr(self, "gen_mode", None)            # None: library default (wn_gen_set_mode 0: the tensor-core cluster kernel for 256- and 512-wide nets)
        if mode is not None:
            native.check(lib.wn_gen_set_mode(s["handle"], int(mode)), "gen mode")

    def prefill(self, s, d_first, T, cond=None, ctab=None, local=None):
        """Write the rings of the freshly reset sampler ``s`` as evaluations [0, T) would, from one forward over the prompt
        window of prefill_window (prefill_forward), and move the handle to t = T (wn_gen_prefill_*)."""
        lib, h = native.lib(), s["handle"]

        def scatter(layer, src, layout, L, stream):
            native.check(lib.wn_gen_prefill_layer(h, layer, src, layout, L, L, T, stream), f"prefill layer {layer}")
        self.prefill_forward(d_first, T, scatter, cond=cond, ctab=ctab, local=local)
        native.check(lib.wn_gen_prefill_commit(h, T), "prefill commit")

    def prefill_forward(self, d_first, T, scatter, cond=None, ctab=None, local=None):
        """One forward over the prompt window of prefill_window(T): scatter(layer, src, layout, L, stream) receives every
        layer's input over the window (sequence b of src = prompt b, frame L - 1 = position T - 1) right after it is
        computed.  d_first: the (B, >= T + 1) int32 prompts on the device; cond: the (B, G) condition rows, ctab their table;
        local: the sampler's (series, hop).  256-channel nets run the fused tensor-core blocks in bf16 pairs whatever
        tc_precision says (fp32-class, the sampler's parity class); every other net, 512 channels included (single-pass bf16
        there, ~1e-3), the FFMA blocks.  One launch per layer, each followed by the scatter of its output; layer 0's input
        comes from the fp32 start conv, which is the sampler's own gather w[:, c] + b."""
        m, lib = self.model, native.lib()
        dev = self.device()
        stream = torch.cuda.current_stream(dev).cuda_stream
        R, D, Sk, Cc, k = m.residual_channels, m.dilation_channels, m.skip_channels, m.classes, m.kernel_size
        dil = [d for d, _ in m.dilations]
        NS, nl = d_first.shape[0], len(dil)
        upsampled = local is not None and getattr(m, "local_upsample", None) is not None
        P0, S, W = prefill_window(T, dil, k, 1 if local is None else local[1])
        L = S + W
        Wp = self.packed_weights(stream)
        use_tb = R == 256 and bool(lib.wn_tb_supported(R, D, Sk, k))
        f32 = dict(device=dev, dtype=torch.float32)
        idx = torch.zeros(NS, L, device=dev, dtype=torch.int64)
        idx[:, S:] = d_first[:, P0:T]
        buf = torch.empty(2, NS, L, R, **f32)               # the two activation buffers (fp32 frames or bf16 pairs)
        ws_t, bs_p = Wp["start"]
        native.check(lib.wn_start_fwd_index_i64(idx.data_ptr(), ws_t.data_ptr(), bs_p.data_ptr(), buf[0].data_ptr(),
                                                NS, Cc, L, R, stream), "prefill start")
        scatter(0, buf[0].data_ptr(), native.GEN_SRC_FRAMES, L, stream)
        frames = None                                       # (table, n_frames, hop) of repeat-upsampled local conditioning
        if local is not None and not (upsampled and use_tb):
            y, hop = local
            nfw = -(-W // hop)
            y_win = torch.zeros(NS, y.shape[1], S // hop + nfw, **f32)      # zero frames before S: never read
            y_win[:, :, S // hop:] = y[:, :, P0 // hop:P0 // hop + nfw]
            frames = (Wp.cond_table_frames(cond, y_win, 0, y_win.shape[2], stream), y_win.shape[2], hop)
        elif upsampled:
            c, Cl = local[0], m.local_condition_channels
            c_win = torch.zeros(NS, Cl, L, **f32)
            c_win[:, :, S:] = c[:, :, P0:T]
            cpad = lib.wn_tb_local_padded_channels(Cl, native.PREC_BF16_PAIRS)
            c_pair = torch.empty(NS, 2, cpad // 8, L, 8, device=dev, dtype=torch.bfloat16)
            native.check(lib.wn_tb_local_from_channels(c_win.data_ptr(), c_pair.data_ptr(), NS, Cl, L, native.PREC_BF16_PAIRS,
                                                       stream), "prefill local features")
            u_all = Wp["tb_local_pairs"][0]
            ctab = None if cond is None else Wp.cond_table(cond, stream)
        if use_tb:
            tb_w, tb_b, _ = Wp["tb_pairs"]
            pairs = [buf[i].view(torch.bfloat16) for i in range(2)]
            native.check(lib.wn_pair_from_frames(buf[0].data_ptr(), pairs[1].data_ptr(), NS, L, R, 0, stream), "prefill pairs")
            skip = torch.empty(NS, Sk // 4, 1, 4, **f32)
            a = native.TbBlockArgs()
            a.B, a.L, a.n_layers, a.channels, a.precision = NS, L, nl, R, native.PREC_BF16_PAIRS
            a.d_w_all, a.d_fg_save = tb_w.data_ptr(), None
            src = 1
        else:
            skip = torch.empty(NS, 1, Sk, **f32)
            a = native.BlockArgs()
            a.R, a.D, a.S, a.k, a.mode = R, D, Sk, k, 0
            a.B, a.L = NS, L
            src = 0
        a.d_skip, a.in_start, a.out_start, a.skip_start, a.skip_init = skip.data_ptr(), S, S, L - 1, 1
        for i in range(nl - 1):                             # the last layer's output feeds no ring
            a.d_h_in, a.d_h_out, a.dilation = buf[src].data_ptr(), buf[1 - src].data_ptr(), dil[i]
            if use_tb:
                a.layer, a.d_bias4 = i, tb_b[i].data_ptr()
                if upsampled:
                    rc = lib.wn_tb_block_fwd_local(ctypes.byref(a), native.ptr(None if ctab is None else ctab[i]),
                                                   c_pair.data_ptr(), Cl, u_all.data_ptr(), stream)
                elif frames is not None:
                    rc = lib.wn_tb_block_fwd_cond_frames(ctypes.byref(a), frames[0][i].data_ptr(), frames[1], frames[2], stream)
                elif ctab is not None:
                    rc = lib.wn_tb_block_fwd_cond(ctypes.byref(a), ctab[i].data_ptr(), stream)
                else:
                    rc = lib.wn_tb_block_fwd(ctypes.byref(a), stream)
            else:
                wfg, bfg, wrs, brs = Wp["layers"][i]
                a.d_wfg_t, a.d_bfg, a.d_wrs_t, a.d_brs = wfg.data_ptr(), bfg.data_ptr(), wrs.data_ptr(), brs.data_ptr()
                if frames is not None:
                    rc = lib.wn_block_fwd_cond_frames(ctypes.byref(a), frames[0][i].data_ptr(), frames[1], frames[2], stream)
                elif ctab is not None:
                    rc = lib.wn_block_fwd_cond(ctypes.byref(a), ctab[i].data_ptr(), stream)
                else:
                    rc = lib.wn_block_fwd(ctypes.byref(a), stream)
            native.check(rc, f"prefill block {i}")
            src = 1 - src
            scatter(i + 1, buf[src].data_ptr(), native.GEN_SRC_PAIRS if use_tb else native.GEN_SRC_FRAMES, L, stream)
        self.last_prefill = dict(P0=P0, S=S, W=W, blocks="tb" if use_tb else "ffma")

    def generate_resident(self, s, d_first, n_given, num_samples, temperature, regularize, d_out, d_uni=None,
                          d_forced=None, d_logits=None, t0=0, n_evals=None, reset=True):
        """Launch the sampler on buffers that already live on the device (no host<->device traffic, no sync)."""
        lib = native.lib()
        stream = torch.cuda.current_stream(self.device()).cuda_stream
        if reset:
            self.reset_sampler(s, stream)
        args = native.GenRunArgs()
        args.d_first, args.n_given = d_first.data_ptr(), n_given
        args.d_forced, args.d_uniforms = native.ptr(d_forced), native.ptr(d_uni)
        args.d_out_idx, args.d_out_logits = d_out.data_ptr(), native.ptr(d_logits)
        args.n_samples = num_samples
        args.temperature, args.regularize = float(temperature), float(regularize)
        total = n_given - 1 + num_samples
        args.t0, args.n_evals = t0, (total - t0 if n_evals is None else n_evals)
        if args.n_evals > 0:
            native.check(lib.wn_gen_run(s["handle"], ctypes.byref(args), stream), "gen run")
        return t0 + args.n_evals

    def generate(self, num_samples, first, temperature, regularize, uniforms=None, forced=None,
                 want_logits=False, callbacks=None, cond=None, local=None, top_k=0, top_p=1.0, prefill=False):
        """first: (NS, n_given) int array.  Returns (indices (NS, num_samples) int64 ndarray, logits or None, t_end).
        top_k, top_p: the truncation of the temperature draw (wn_gen_set_truncation), set on the handle by every call.
        Per-stream form (see _stream_plan): first a list of NS 1-D prompts of any lengths, num_samples and the four settings
        scalars or NS values each, uniforms / forced (NS, >= n_s) matrices or lists.  The prompts are padded into a matrix
        whose pitch is the longest prompt, the records go to wn_gen_set_stream_params, and the rows of the returned arrays
        have the launch's pitch (t_end - head_from): row s holds stream s's samples first, then padding.
        callbacks: optional list of (eval_index, fn) -- fn() is called once evaluations <= eval_index are done.
        cond: the (NS, G) fp32 condition rows of a conditioned model, else None.
        local: (y, hop) of a locally conditioned model, y the (NS, C, F) fp32 series, else None.  The condition table is
        built window by window (at most ``local_table_bytes`` each), and launches are split at the window boundaries.
        prefill: write the rings for the first head_from evaluations (the common prompt prefix) with one forward (prefill())
        instead of evaluating them one by one; callbacks of those evaluations fire, in order, right after it."""
        plan = _stream_plan(first, num_samples, temperature, regularize, top_k, top_p)
        m = self.model
        dev = self.device()
        self.step_session = None             # a generate_fast run restarts the device queues (wavenet_model.py:250)
        first, NS = plan.first, plan.n_streams
        if plan.per_stream:
            # the launch's scalars: the pitch of first, the row pitch, no scalar settings (the records hold them)
            n_given, num_samples, temperature, regularize, top_k, top_p = plan.pitch, plan.n_samples, 0.0, 0.0, 0, 1.0
        else:
            n_given, temperature, regularize, top_k, top_p = first.shape[1], plan.temperature[0], plan.regularize[0], \
                plan.top_k[0], plan.top_p[0]
        s = self.sampler(NS)
        # on every call, so that one call's setting never reaches the next
        native.check(native.lib().wn_gen_set_truncation(s["handle"], top_k, top_p), "gen truncation")
        native.check(native.lib().wn_gen_set_stream_params(s["handle"], plan.records() if plan.per_stream else None),
                     "gen stream params")
        stream = torch.cuda.current_stream(dev).cuda_stream
        # the condition table is read by every launch of this run: the sampler entry keeps it alive
        if local is None:
            s["cond"] = None if cond is None else self.packed_weights(stream).cond_table(cond, stream)
            native.check(native.lib().wn_gen_set_condition(s["handle"], native.ptr(s["cond"])), "gen condition")
        d_out = torch.zeros(NS, max(num_samples, 1), device=dev, dtype=torch.int32)
        d_uni = d_forced = d_logits = None
        if plan.per_stream:
            if any(t > 0 for t in plan.temperature):
                if uniforms is None:
                    # generate_fast's draws, stream by stream in order; a temperature-0 stream draws nothing
                    uniforms = [np.random.random_sample(n) if t > 0 else np.zeros(0)
                                for n, t in zip(plan.counts, plan.temperature)]
                uniforms = plan.rows(uniforms, np.float64, "uniforms", need=[t > 0 for t in plan.temperature])
                d_uni = torch.from_numpy(uniforms).to(dev, non_blocking=True)
            if forced is not None:
                forced = plan.rows(forced, np.int32, "forced")
                d_forced = torch.from_numpy(forced).to(dev, non_blocking=True)
        else:
            if temperature > 0:
                if uniforms is None:
                    # exactly the draws np.random.choice would make: one random_sample() per drawn sample
                    uniforms = np.stack([np.random.random_sample(num_samples) for _ in range(NS)])
                uniforms = np.ascontiguousarray(np.asarray(uniforms, dtype=np.float64).reshape(NS, num_samples))
                d_uni = torch.from_numpy(uniforms).to(dev, non_blocking=True)
            if forced is not None:
                forced = np.ascontiguousarray(np.asarray(forced, dtype=np.int32).reshape(NS, num_samples))
                d_forced = torch.from_numpy(forced).to(dev, non_blocking=True)
        d_first = torch.from_numpy(first).to(dev, non_blocking=True)
        if want_logits:
            d_logits = torch.zeros(NS, max(num_samples, 1), m.classes, device=dev, dtype=torch.float32)
        total_evals = plan.n_evals
        common = dict(d_uni=d_uni, d_forced=d_forced, d_logits=d_logits)
        window = [None]                       # (first frame, frames) of the local-conditioning table the handle holds

        def launch(t, n, reset):
            """evaluations [t, t + n); under local conditioning split at the table windows' boundaries"""
            if local is None or n <= 0:
                return self.generate_resident(s, d_first, n_given, num_samples, temperature, regularize, d_out,
                                              t0=t, n_evals=max(n, 0), reset=reset, **common)
            y, hop = local
            m = self.model
            per_frame = m.layers * m.blocks * NS * 2 * m.dilation_channels * 4
            max_frames = max(1, self.local_table_bytes // per_frame)
            end = t + n
            while t < end:
                f = t // hop
                if window[0] is None or not window[0][0] <= f < window[0][0] + window[0][1]:
                    nf = min(max_frames, -(-total_evals // hop) - f)
                    s["cond"] = None          # the previous window's launches are ordered before this stream's new work
                    s["cond"] = self.packed_weights(stream).cond_table_frames(cond, y, f, nf, stream)
                    native.check(native.lib().wn_gen_set_condition_frames(s["handle"], s["cond"].data_ptr(), f, nf, hop),
                                 "gen local condition")
                    window[0] = (f, nf)
                stop = min(end, (window[0][0] + window[0][1]) * hop)
                t = self.generate_resident(s, d_first, n_given, num_samples, temperature, regularize, d_out,
                                           t0=t, n_evals=stop - t, reset=reset, **common)
                reset = False
            return t

        t, first_launch = 0, True
        if prefill and plan.head_from > 0:
            self.reset_sampler(s, stream)
            self.prefill(s, d_first, plan.head_from, cond=cond, ctab=s.get("cond") if local is None else None, local=local)
            t, first_launch = plan.head_from, False
        for upto, fn in sorted(callbacks or [], key=lambda c: c[0]):
            n = min(upto + 1, total_evals) - t
            if n > 0 or first_launch:
                t = launch(t, n, first_launch)
                first_launch = False
            torch.cuda.current_stream(dev).synchronize()
            fn()
        if total_evals - t > 0 or first_launch:
            launch(t, total_evals - t, first_launch)
        idx = d_out[:, :num_samples].cpu().numpy().astype(np.int64)      # device->host read; synchronises
        native.check(native.lib().wn_gen_check(s["handle"], torch.cuda.current_stream(dev).cuda_stream), "gen check")
        logits = d_logits[:, :num_samples].cpu().numpy() if want_logits else None
        self.last_run = dict(evals=total_evals, sampler=s)
        self.h2d_bytes_last = first.nbytes + (uniforms.nbytes if d_uni is not None else 0) + \
            (forced.nbytes if d_forced is not None else 0)
        self.d2h_bytes_last = NS * num_samples * 4 + (logits.nbytes if want_logits else 0)
        return idx, logits, total_evals


class _Job:
    """One submitted sampling job of a SamplingSession and what it has produced so far."""

    def __init__(self, jid, prompt, count, temperature, regularize, top_k, top_p, cond, uniforms, local=None):
        self.id, self.prompt, self.count = jid, prompt, count
        self.temperature, self.regularize, self.top_k, self.top_p = temperature, regularize, top_k, top_p
        self.cond, self.uniforms = cond, uniforms
        self.local = local              # (C, F) device series the sampler reads (learned upsampler: its hop-1 features)
        self.idx, self.logits = [], []
        self.made = 0


class SamplingSession:
    """Continuous batching on one sampler handle of ``n_slots`` streams (WaveNetModel.sampling_session).

    Jobs queue FIFO (submit); every step() seats queued jobs into free slots, runs ``n_evals`` evaluations of all slots in
    one launch and hands each job its new samples.  A slot whose job is done takes the next queued job at the next step, at
    its own position: the handle's time t is global, a job's position is t - origin (wn_gen_set_stream_positions), and
    seating writes the slot's rings for the times its new positions read (wn_gen_seat_layer), zeros or, with
    ``prefill=True``, the values of one forward over the job's prompt window (as generate_fast(prefill=True) computes them).
    An empty slot runs a parked temperature-0 job whose outputs are discarded.  Each job gives, bit for bit, what a
    generate_fast_batch launch of the same slot count carrying that job in every stream gives, with the same uniforms and
    the same ``prefill``.  The session owns its handle: generate_fast* calls on the model never touch it.  Global
    conditioning is per job.  Local conditioning is per job too: every slot reads its own frame window, indexed by its own
    position (wn_gen_set_condition_stream_frames); a step runs in launches of at most ``local_window`` evaluations, and
    before each one the slots' windows are gathered from their jobs' series and built into one table buffer allocated at
    creation (_session_windows)."""

    _T_MAX = 2 ** 31 - 1

    def __init__(self, model, n_slots, prefill=False, return_logits=False, local_window=None):
        if isinstance(n_slots, (bool, np.bool_)) or not isinstance(n_slots, (int, np.integer)) or n_slots < 1:
            raise ValueError(f"n_slots must be an integer >= 1, got {n_slots!r}")
        _check_prefill(prefill)
        self.Cl = getattr(model, "local_condition_channels", 0)
        if self.Cl:
            if isinstance(local_window, (bool, np.bool_)) or not isinstance(local_window, (int, np.integer)) or local_window < 1:
                raise ValueError("a locally conditioned model needs local_window= (an integer >= 1: the evaluations one "
                                 f"condition-table build covers per slot), got {local_window!r}")
        elif local_window is not None:
            raise ValueError("local_window applies to a locally conditioned model only (this one has local_condition_channels=0)")
        self.model, self.n_slots, self.prefill, self.return_logits = model, int(n_slots), prefill, bool(return_logits)
        self.rt = rt = model._runtime()
        self.dev = rt.device()
        self.queue, self.jobs, self.next_id = [], {}, 0
        self.slot_job = [None] * self.n_slots          # the job in each slot, None: parked
        self.origin = [0] * self.n_slots
        self.seated = [False] * self.n_slots           # False: the slot must be (re)seated at the next step
        dil = [d for d, _ in model.dilations]
        self.t_start = (model.kernel_size - 1) * max(dil) + 1     # past the longest ring: primed history lies at t >= 0
        with torch.cuda.device(self.dev):
            self.s = rt.new_sampler(self.n_slots)
            self.G = getattr(model, "condition_channels", 0)
            self.ctab = self.hrows = None
            if self.Cl:
                # one table buffer for the session: n_layers x n_slots x nf x 2D floats (see sampling_session)
                self.window = int(local_window)
                self.hop = 1 if getattr(model, "local_upsample", None) is not None else model.local_condition_hop
                self.nf = _session_frames(self.window, self.hop)
                nl, D = model.layers * model.blocks, model.dilation_channels
                f32 = dict(device=self.dev, dtype=torch.float32)
                self.ltab = torch.empty(nl, self.n_slots, self.nf, 2 * D, **f32)
                self.ywin = torch.zeros(self.n_slots, self.Cl, self.nf, **f32)     # the slots' gathered frames
                if self.G:                             # each slot's global condition row (parked: zero)
                    self.hrows = torch.zeros(self.n_slots, self.G, **f32)
            elif self.G:                               # rows of parked slots: the zero condition (the biases)
                stream = torch.cuda.current_stream(self.dev).cuda_stream
                zero = torch.zeros(self.n_slots, self.G, device=self.dev, dtype=torch.float32)
                self.ctab = rt.packed_weights(stream).cond_table(zero, stream)
            self.reset()

    def __del__(self):
        s = self.__dict__.get("s")
        if s is not None:
            native.lib().wn_gen_destroy(s["handle"])

    # ------------------------------------------------------------------ public
    @property
    def pending(self):
        """jobs submitted and not yet seated"""
        return len(self.queue)

    @property
    def active(self):
        """jobs seated and not yet done"""
        return sum(j is not None for j in self.slot_job)

    def reset(self):
        """Restart the handle's time (allowed only while no job is active); queued jobs stay queued."""
        if self.active:
            raise RuntimeError(f"reset() with {self.active} active jobs")
        lib, h = native.lib(), self.s["handle"]
        with torch.cuda.device(self.dev):
            self.rt.reset_sampler(self.s, torch.cuda.current_stream(self.dev).cuda_stream)
        native.check(lib.wn_gen_set_time(h, self.t_start), "session time")
        native.check(lib.wn_gen_set_condition(h, native.ptr(self.ctab)), "session condition")
        self.t = self.t_start
        self.seated = [False] * self.n_slots

    def submit(self, first_samples, num_samples, temperature=1., regularize=0., top_k=0, top_p=1.0, condition=None,
               uniforms=None, local_condition=None):
        """Queue one job: generate_fast(num_samples, first_samples, temperature, regularize, top_k=, top_p=, condition=,
        local_condition=) with ``uniforms`` (num_samples,) float64 for its draws; None draws them from numpy's global RNG
        now when temperature > 0.  ``local_condition``: a locally conditioned model's (C, F) series for this job, F >=
        ceil((n_given - 1 + num_samples) / hop) (required there, refused elsewhere); a learned upsampler runs on it here, at
        the job's own length.  Returns the job id.  ValueError for a malformed argument, before any device work."""
        if torch.is_tensor(first_samples):
            first_samples = first_samples.detach().cpu().numpy()
        prompt = np.asarray(first_samples)
        if prompt.ndim == 0:
            prompt = prompt.reshape(1)
        plan = _stream_plan([prompt], [num_samples], [temperature], [regularize], [top_k], [top_p])
        count = plan.counts[0]
        cond = self.model._condition(self.model._one_condition(condition), 1)
        if plan.temperature[0] > 0:
            if uniforms is None:
                uniforms = np.random.random_sample(count)
            u = np.asarray(uniforms.detach().cpu().numpy() if torch.is_tensor(uniforms) else uniforms, dtype=np.float64)
            if u.ndim != 1 or u.shape[0] < count:
                raise ValueError(f"uniforms must be a 1-D array of at least {count} values, got shape {u.shape}")
            uniforms = u[:count].copy()
        else:
            uniforms = None
        positions = plan.n_given[0] - 1 + count
        if local_condition is not None:
            local_condition = local_condition[None] if torch.is_tensor(local_condition) else np.asarray(local_condition)[None]
        y = self.model._local_condition(local_condition, 1, positions)
        if y is not None and count > 0:
            # as _per_stream_local: a learned upsampler runs on the job alone, at its own length
            with torch.no_grad(), torch.cuda.device(self.dev):
                y = y.detach()
                if getattr(self.model, "local_upsample", None) is not None:
                    y = self.model._upsample(y, positions)
                y = y[0].contiguous()
        jid = self.next_id
        self.next_id += 1
        job = _Job(jid, plan.first[0, :plan.n_given[0]].copy(), count, plan.temperature[0], plan.regularize[0],
                   plan.top_k[0], plan.top_p[0], cond, uniforms, local=y)
        self.jobs[jid] = job
        self.queue.append(job)
        return jid

    def result(self, job_id):
        """A done job's indices (int64 (n,)) [and logits (n, classes)]; None while it is queued or running."""
        job = self.jobs[job_id]
        if job.made < job.count:
            return None
        idx = np.concatenate(job.idx).astype(np.int64) if job.idx else np.zeros(0, dtype=np.int64)
        if not self.return_logits:
            return idx
        C = self.model.classes
        return idx, (np.concatenate(job.logits) if job.logits else np.zeros((0, C), dtype=np.float32))

    def step(self, n_evals):
        """Seat queued jobs into free slots, run n_evals evaluations of every slot, return {job_id: new indices} (with
        return_logits: {job_id: (indices, logits)}) for the jobs that ran."""
        if isinstance(n_evals, (bool, np.bool_)) or not isinstance(n_evals, (int, np.integer)) or n_evals < 1:
            raise ValueError(f"n_evals must be an integer >= 1, got {n_evals!r}")
        n_evals = int(n_evals)
        key, wkey = self.rt.sampler_keys(self.n_slots)
        if (key, wkey) != (self.s["key"], self.s["wkey"]):
            raise RuntimeError("the model's parameters changed after the session was created; create a new session")
        if self.t + n_evals >= self._T_MAX:
            raise RuntimeError(f"step({n_evals}) would move the session's time past 2^31 - 1; reset() it between jobs")
        with torch.cuda.device(self.dev):
            return self._step(n_evals)

    # ------------------------------------------------------------------ internals
    def _seat(self, seats, stream):
        lib, h = native.lib(), self.s["handle"]
        nl = self.model.layers * self.model.blocks
        zeros, primed = [], {}
        for b, job in seats:
            self.slot_job[b] = job
            T = 0 if job is None or not self.prefill else job.prompt.shape[0] - 1
            self.origin[b] = self.t - T
            if T == 0:
                zeros.append(b)
            else:
                primed.setdefault(T, []).append((b, job))    # windows line up: one forward per prompt length
            if self.hrows is not None:
                self.hrows[b] = 0.0 if job is None else job.cond[0]
            elif job is not None and job.cond is not None:
                self.ctab[:, b, :] = self.rt.packed_weights(stream).cond_table(job.cond, stream)[:, 0, :]
            self.seated[b] = True
        if zeros:
            sl = (ctypes.c_int * len(zeros))(*zeros)
            qe = (ctypes.c_int * len(zeros))(*([0] * len(zeros)))
            for l in range(nl):
                native.check(lib.wn_gen_seat_layer(h, l, len(zeros), sl, qe, None, 0, 1, 0, stream), "seat")
        for T, group in primed.items():
            slots = [b for b, _ in group]
            sl = (ctypes.c_int * len(slots))(*slots)
            qe = (ctypes.c_int * len(slots))(*([T] * len(slots)))
            d_first = torch.from_numpy(np.stack([j.prompt for _, j in group]).astype(np.int32)).to(self.dev)
            cond = ctab = local = None
            if self.G:
                cond = torch.cat([j.cond for _, j in group])
                ctab = self.rt.packed_weights(stream).cond_table(cond, stream)
            if self.Cl:
                # each job's own series, zero-padded to the frames the prompt window reads
                P0, _, W = prefill_window(T, [d for d, _ in self.model.dilations], self.model.kernel_size, self.hop)
                width = max(P0 // self.hop + -(-W // self.hop), max(j.local.shape[1] for _, j in group))
                y = torch.zeros(len(group), self.Cl, width, device=self.dev, dtype=torch.float32)
                for i, (_, j) in enumerate(group):
                    y[i, :, :j.local.shape[1]] = j.local
                local = (y, self.hop)

            def scatter(layer, src, layout, L, st, sl=sl, qe=qe, n=len(slots)):
                native.check(lib.wn_gen_seat_layer(h, layer, n, sl, qe, src, layout, L, L, st), f"seat layer {layer}")
            self.rt.prefill_forward(d_first, T, scatter, cond=cond, ctab=ctab, local=local)

    def _step(self, n_evals):
        stream = torch.cuda.current_stream(self.dev).cuda_stream
        seats = _session_admit(self.slot_job, self.seated, self.queue)
        if seats:
            self._seat(seats, stream)
        if not self.Cl:
            out = self._launch(self.t, n_evals, stream)
        else:
            got = []
            for t0, n, frame0 in _session_windows(self.t, n_evals, self.origin, self.hop, self.window):
                self._set_windows(frame0, stream)
                got.append(self._launch(t0, n, stream))
            out = {}
            for part in got:                                 # a job's samples of the step, launch after launch
                for jid, v in part.items():
                    out.setdefault(jid, []).append(v)
            cat = lambda vs: np.concatenate(vs) if len(vs) > 1 else vs[0]
            out = {jid: ((cat([v[0] for v in vs]), cat([v[1] for v in vs])) if self.return_logits else cat(vs))
                   for jid, vs in out.items()}
        for b in range(self.n_slots):                        # done jobs give their slot to the next step's admission
            job = self.slot_job[b]
            if job is not None and job.made >= job.count:
                self.slot_job[b] = None
                self.seated[b] = False
        return out

    def _set_windows(self, frame0, stream):
        """Slot b's window: frames [frame0[b], frame0[b] + nf) of its job's series (zeros for a parked slot and past the
        series' end: only discarded outputs read those), built into the session's table buffer and set on the handle.
        The build is ordered on the stream after the previous launch, which still reads the buffer, so one buffer serves
        every launch."""
        lib, h, nf = native.lib(), self.s["handle"], self.nf
        self.ywin.zero_()
        for b, job in enumerate(self.slot_job):
            if job is None:
                continue
            f0, F = frame0[b], job.local.shape[1]
            if f0 < F:
                self.ywin[b, :, :min(nf, F - f0)] = job.local[:, f0:f0 + nf]
        self.rt.packed_weights(stream).cond_table_frames(self.hrows, self.ywin, 0, nf, stream, out=self.ltab)
        f0s = (ctypes.c_int * self.n_slots)(*frame0)
        native.check(lib.wn_gen_set_condition_stream_frames(h, self.ltab.data_ptr(), f0s, nf, self.hop),
                     "session local condition")

    def _launch(self, t, n_evals, stream):
        """One launch of every slot over evaluations [t, t + n_evals): {job_id: new indices [, logits]}."""
        lib, h = native.lib(), self.s["handle"]
        NS = self.n_slots
        recs, pos, first, uni, plans = _session_records(t, n_evals, self.slot_job, self.origin)
        native.check(lib.wn_gen_set_stream_params(h, recs), "session stream params")
        native.check(lib.wn_gen_set_stream_positions(h, pos), "session positions")
        d_first = torch.from_numpy(first).to(self.dev, non_blocking=True)
        d_uni = torch.from_numpy(uni).to(self.dev, non_blocking=True)
        d_out = torch.zeros(NS, n_evals, device=self.dev, dtype=torch.int32)
        d_logits = torch.zeros(NS, n_evals, self.model.classes, device=self.dev, dtype=torch.float32) \
            if self.return_logits else None
        args = native.GenRunArgs()
        args.d_first, args.n_given = d_first.data_ptr(), first.shape[1]
        args.d_forced, args.d_uniforms = None, d_uni.data_ptr()
        args.d_out_idx, args.d_out_logits = d_out.data_ptr(), native.ptr(d_logits)
        args.n_samples, args.t0, args.n_evals = n_evals, t, n_evals
        args.temperature, args.regularize = 0.0, 0.0
        native.check(lib.wn_gen_run(h, ctypes.byref(args), stream), "session run")
        self.t = t + n_evals
        idx = d_out.cpu().numpy().astype(np.int64)          # synchronises
        native.check(lib.wn_gen_check(h, stream), "session check")
        logits = d_logits.cpu().numpy() if self.return_logits else None
        out = {}
        for b, job, c0, n in plans:
            new = idx[b, c0:c0 + n]
            job.idx.append(new)
            job.made += n
            if self.return_logits:
                lg = logits[b, c0:c0 + n]
                job.logits.append(lg)
                out[job.id] = (new, lg)
            else:
                out[job.id] = new
        return out


def _session_admit(slot_job, seated, queue):
    """A session step's admission: queued jobs (FIFO) go to the free slots, lowest slot first; a job of 0 samples is done
    without a slot; a free slot left over is parked (seated with no job) unless it is parked already.  Pops the admitted
    jobs off ``queue``; returns [(slot, job or None)], the slots to seat."""
    seats = []
    for b, job in enumerate(slot_job):
        if job is not None:
            continue
        nxt = None
        while queue:
            cand = queue.pop(0)
            if cand.count > 0:
                nxt = cand
                break
        if nxt is None and seated[b]:
            continue
        seats.append((b, nxt))
    return seats


def _session_frames(window, hop):
    """Frames one slot's table window holds: any run of ``window`` consecutive positions touches at most
    ceil((window - 1) / hop) + 1 frames of ``hop`` positions."""
    return -(-(window - 1) // hop) + 1


def _session_windows(t, n_evals, origin, hop, window):
    """The launches of a session step of n_evals evaluations from time t under local conditioning: [(t0, n, frame0)], each
    at most ``window`` evaluations, frame0[b] = q0 // hop the first frame of slot b (origin[b]) at its position q0 = t0 -
    origin[b].  Its positions [q0, q0 + n) then read frames [frame0[b], frame0[b] + _session_frames(window, hop))."""
    out = []
    while n_evals > 0:
        n = min(window, n_evals)
        out.append((t, n, [(t - o) // hop for o in origin]))
        t, n_evals = t + n, n_evals - n
    return out


def _session_records(t, n_evals, slot_job, origin):
    """The launch of a session step of n_evals evaluations from time t: (stream params, stream positions, (NS, pitch) int32
    prompt rows, (NS, n_evals) float64 uniforms, [(slot, job, first column, new samples)]).  Slot b's job is at position
    q0 = t - origin[b]: its prompt row holds positions [first0, min(n_given, q0 + n_evals)) with first0 = q0 while the
    launch still reads the prompt; its output columns start at sample sample0 = max(0, q0 - (n_given - 1)).  A parked slot
    (job None) runs a temperature-0 job of the prompt [0]."""
    NS = len(slot_job)
    recs = (native.GenStreamParams * NS)()
    pos = (native.GenStreamPos * NS)()
    rows, plans = [], []
    uni = np.zeros((NS, n_evals), dtype=np.float64)
    for b, job in enumerate(slot_job):
        prompt = job.prompt if job is not None else np.zeros(1, dtype=np.int32)
        ng = prompt.shape[0]
        q0 = t - origin[b]
        first0 = q0 if q0 < ng else 0
        rows.append(prompt[first0:min(ng, q0 + n_evals)] if q0 < ng else prompt[:0])
        i0 = q0 - (ng - 1)
        sample0 = max(i0, 0)
        pos[b] = native.GenStreamPos(origin[b], sample0, first0)
        if job is None:
            recs[b] = native.GenStreamParams(1, 0, 0.0, 0.0, 1.0)
            continue
        recs[b] = native.GenStreamParams(ng, job.top_k, job.temperature, job.regularize, job.top_p)
        hi = min(job.count, i0 + n_evals)               # the job's new samples [sample0, hi) in columns [0, hi - sample0)
        if hi > sample0:
            plans.append((b, job, 0, hi - sample0))
            if job.uniforms is not None:
                uni[b, :hi - sample0] = job.uniforms[sample0:hi]
    first = np.zeros((NS, max(1, max(r.shape[0] for r in rows))), dtype=np.int32)
    for b, r in enumerate(rows):
        first[b, :r.shape[0]] = r
    return recs, pos, first, uni, plans


class _StreamPlan:
    """The schedule of one sampler call (see wn_gen_set_stream_params): first the (NS, pitch) int32 prompt matrix (row s
    holds prompt s, then padding that is never read), n_given / counts the prompt lengths and sample counts, head_from
    the first evaluation that runs the head, n_samples the row pitch of uniforms / forced / the outputs, n_evals the
    evaluations of the call; temperature / regularize / top_k / top_p one value per stream.  per_stream: the call needs
    per-stream records (settings or prompt lengths that differ, or counts given per stream); otherwise it is today's
    scalar call."""

    def records(self):
        recs = (native.GenStreamParams * self.n_streams)()
        for s in range(self.n_streams):
            recs[s] = native.GenStreamParams(self.n_given[s], self.top_k[s], self.temperature[s], self.regularize[s],
                                             self.top_p[s])
        return recs

    def rows(self, v, dtype, name, need=None):
        """v -- an (NS, >= n_s) matrix or a list of NS 1-D arrays, row s holding stream s's first n_s values -- as the
        contiguous (NS, n_samples) matrix the kernels read; padding is zero.  need[s] False: stream s's row is not read
        (a temperature-0 stream's uniforms) and may be short."""
        out = np.zeros((self.n_streams, self.n_samples), dtype=dtype)
        if isinstance(v, (list, tuple)):
            if len(v) != self.n_streams:
                raise ValueError(f"{name} must hold {self.n_streams} rows, got {len(v)}")
            rows_ = [np.asarray(r.detach().cpu().numpy() if torch.is_tensor(r) else r).reshape(-1) for r in v]
        else:
            a = np.asarray(v.detach().cpu().numpy() if torch.is_tensor(v) else v)
            if a.ndim != 2 or a.shape[0] != self.n_streams:
                raise ValueError(f"{name} must be an ({self.n_streams}, >= {max(self.counts, default=0)}) array or a list "
                                 f"of {self.n_streams} rows, got shape {a.shape}")
            rows_ = list(a)
        for s, (r, n) in enumerate(zip(rows_, self.counts)):
            if need is not None and not need[s]:
                continue
            if r.shape[0] < n:
                raise ValueError(f"{name} row {s} holds {r.shape[0]} values, stream {s} needs {n}")
            out[s, :n] = r[:n]
        return out


def _is_seq(v):
    """a per-stream sequence (list, tuple, or an array / tensor of at least one dimension), not a scalar"""
    return isinstance(v, (list, tuple)) or ((isinstance(v, np.ndarray) or torch.is_tensor(v)) and v.ndim > 0)


def _per_stream_values(name, v, n, check):
    """(values, given per stream): a scalar repeated n times, or a length-n sequence, every value checked"""
    if not _is_seq(v):
        if isinstance(v, np.ndarray) or torch.is_tensor(v):
            v = v.item()
        return [check(v)] * n, False
    a = v.detach().cpu().numpy() if torch.is_tensor(v) else v
    if np.ndim(a) != 1 or len(a) != n:
        raise ValueError(f"{name} must be a scalar or a sequence of {n} values (one per stream), got shape {np.shape(a)}")
    return [check(x.item() if isinstance(x, np.generic) else x) for x in a], True


def _finite(name):
    def check(x):
        if isinstance(x, (bool, np.bool_)) or not isinstance(x, (int, float, np.integer, np.floating)) \
                or not np.isfinite(float(x)):
            raise ValueError(f"{name} must be a finite real number, got {x!r}")
        return float(x)
    return check


def _stream_plan(first_samples, num_samples, temperature, regularize, top_k, top_p):
    """The checked _StreamPlan of a sampler call; ValueError before any device work.  first_samples: an (NS, n_given) int
    array, or a list of NS 1-D int arrays of any lengths >= 1.  num_samples: an int, or a sequence of NS ints >= 0.
    temperature, regularize (finite numbers), top_k, top_p (see _truncation): scalars or NS values each.  A scalar
    call (rectangular prompt, every argument a scalar) keeps today's unchecked scalar temperature and regularize."""
    plan = _StreamPlan()
    if isinstance(first_samples, (list, tuple)) and any(
            (torch.is_tensor(r) and r.dim() != 0) or np.ndim(r) != 0 for r in first_samples):
        prompts = []
        for s, r in enumerate(first_samples):
            a = np.asarray(r.detach().cpu().numpy() if torch.is_tensor(r) else r)
            if a.ndim != 1 or a.shape[0] < 1 or not (np.issubdtype(a.dtype, np.integer) and a.dtype != np.bool_):
                raise ValueError(f"first_samples[{s}] must be a 1-D int array of at least one sample, got "
                                 f"{a.dtype} {a.shape}")
            prompts.append(a.astype(np.int64))
    else:
        first = np.asarray(first_samples.detach().cpu().numpy() if torch.is_tensor(first_samples) else first_samples)
        first = first.astype(np.int64).reshape(first.shape[0], -1) if first.ndim > 1 else first.astype(np.int64)[None, :]
        if first.shape[1] < 1:
            raise RuntimeError("first_samples must hold at least one sample")
        prompts = list(first)
    NS = plan.n_streams = len(prompts)
    plan.n_given = [int(r.shape[0]) for r in prompts]

    def count(x):
        if isinstance(x, (bool, np.bool_)) or not isinstance(x, (int, np.integer)) or x < 0:
            raise ValueError(f"num_samples must hold integers >= 0, got {x!r}")
        return int(x)
    if _is_seq(num_samples):
        plan.counts, counts_given = _per_stream_values("num_samples", num_samples, NS, count)
    else:
        plan.counts, counts_given = [int(num_samples)] * NS, False
    plan.temperature, t_given = _per_stream_values("temperature", temperature, NS,
                                                   _finite("temperature") if _is_seq(temperature) else float)
    plan.regularize, r_given = _per_stream_values("regularize", regularize, NS,
                                                  _finite("regularize") if _is_seq(regularize) else float)
    plan.top_k, k_given = _per_stream_values("top_k", top_k, NS, lambda k: _truncation(k, 1.0)[0])
    plan.top_p, p_given = _per_stream_values("top_p", top_p, NS, lambda q: _truncation(0, q)[1])
    ragged = len(set(plan.n_given)) > 1
    plan.ragged = ragged or counts_given
    plan.per_stream = plan.ragged or t_given or r_given or k_given or p_given
    plan.head_from = min(plan.n_given) - 1
    plan.pitch = max(plan.n_given)
    plan.n_evals = max(g - 1 + n for g, n in zip(plan.n_given, plan.counts))
    plan.n_samples = plan.n_evals - plan.head_from
    plan.first = np.zeros((NS, plan.pitch), dtype=np.int32)
    for s, r in enumerate(prompts):
        plan.first[s, :r.shape[0]] = r
    return plan


def _truncation(top_k, top_p):
    """Checked (top_k, top_p) of the sampler's truncated draw: top_k an integer >= 0 (0: off), top_p a real number in
    (0, 1] (1: off).  Raises ValueError otherwise, bools included."""
    if isinstance(top_k, (bool, np.bool_)) or not isinstance(top_k, (int, np.integer)):
        raise ValueError(f"top_k must be an integer >= 0 (0: off), got {top_k!r}")
    if isinstance(top_p, (bool, np.bool_)) or not isinstance(top_p, (int, float, np.integer, np.floating)):
        raise ValueError(f"top_p must be a number in (0, 1] (1: off), got {top_p!r}")
    if top_k < 0:
        raise ValueError(f"top_k must be >= 0 (0: off), got {top_k}")
    if not 0.0 < float(top_p) <= 1.0:
        raise ValueError(f"top_p must lie in (0, 1] (1: off), got {top_p}")
    return int(top_k), float(top_p)


def _check_prefill(prefill):
    if not isinstance(prefill, bool):
        raise ValueError(f"prefill must be True or False, got {prefill!r}")


def _exact_convolutions():
    """cuDNN convolutions in full fp32 and deterministic (torch lets them use TF32 by default, ~1e-3 relative): the learned
    upsampler's output feeds every layer."""
    return torch.backends.cudnn.flags(enabled=torch.backends.cudnn.enabled, benchmark=False, deterministic=True,
                                      allow_tf32=False)


class _StackFunction(torch.autograd.Function):
    """forward()/wavenet() as one autograd node: parameters in, logits out; the input carries no gradient."""

    @staticmethod
    def forward(ctx, model, x, out_len, index_input, cond, local_y, local_hop, *params):
        saved = {}
        rt = model._runtime()
        local = None if local_y is None else (local_y.detach(), local_hop)
        ctx.upsampler = None
        if local is not None and getattr(model, "local_upsample", None) is not None:
            # the learned upsampler runs inside this node, so that its gradients exist while the backward still averages
            # gradients across ranks (see backward)
            with torch.enable_grad():
                y_in = local[0].requires_grad_(ctx.needs_input_grad[5])
                c = model._upsample(y_in, x.size(-1))
            ctx.upsampler = (y_in, c)
            with torch.no_grad(), torch.cuda.device(rt.device()):
                y = rt.stack_forward(x, out_len, index_input=index_input, save=saved, cond=cond, upsampled=c.detach())
            saved["local_dy"] = torch.zeros_like(c)              # gradient of c: every layer adds its share
        else:
            with torch.no_grad(), torch.cuda.device(rt.device()):
                y = rt.stack_forward(x, out_len, index_input=index_input, save=saved, cond=cond, local=local)
            if local is not None and ctx.needs_input_grad[5]:
                saved["local_dy"] = torch.zeros_like(local[0])          # the backward adds every layer's share
        ctx.model, ctx.saved = model, saved
        ctx.names = [n for n, _ in model.named_parameters()]
        return y

    @staticmethod
    def backward(ctx, dlogits):
        if ctx.saved is None:
            raise RuntimeError("wavenet_b200: the saved activations of this forward were freed by a previous backward "
                               "(retain_graph=True is not supported: run the forward again)")
        rt = ctx.model._runtime()
        with torch.no_grad(), torch.cuda.device(rt.device()):
            g = rt.stack_backward(ctx.saved, dlogits)
        dy = ctx.saved.get("local_dy")
        if ctx.upsampler is not None:
            # c = upsample(y): its gradient dy comes from dc; the upsampler's parameter gradients are averaged across ranks
            # like every other parameter's before they reach p.grad
            y_in, c = ctx.upsampler
            named = [(f"local_upsample.{n}", p) for n, p in ctx.model.local_upsample.named_parameters() if p.requires_grad]
            inputs = ([y_in] if y_in.requires_grad else []) + [p for _, p in named]
            got = []
            if inputs:
                with torch.cuda.device(rt.device()), _exact_convolutions():
                    got = torch.autograd.grad(c, inputs, dy)
            dy = got[0] if y_in.requires_grad else None
            ug = got[len(got) - len(named):]
            g.update(zip([n for n, _ in named], ug))
            reducer = getattr(rt, "grad_reducer", None)
            if reducer is not None:
                reducer.reduce_async(list(ug))
                reducer.wait_all()
            ctx.upsampler = None
        ctx.saved = None
        rt.invalidate()          # an optimizer step follows; it may write through p.data, which no version counter sees
        return (None, None, None, None, None, dy, None) + tuple(g.get(n) for n in ctx.names)


class WaveNetModel(nn.Module):
    """
    A Complete Wavenet Model (constructor arguments as in the reference, wavenet_model.py:28-39)

    Args:
        layers (Int):               Number of layers in each block
        blocks (Int):               Number of wavenet blocks of this model
        dilation_channels (Int):    Number of channels for the dilated convolution
        residual_channels (Int):    Number of channels for the residual connection
        skip_channels (Int):        Number of channels for the skip connections
        end_channels (Int):         Number of channels of the first 1x1 conv of the head
        classes (Int):              Number of possible values each sample can have
        output_length (Int):        Number of samples that are generated for each input
        kernel_size (Int):          Size of the dilation kernel
        dtype:                      Parameter type of this model (kept for API compatibility)
        bias (Bool):                bias on start/filter/gate/residual/skip convs (the head always has bias)
        condition_channels (Int):   G > 0: global conditioning (WaveNet paper section 2.5) on one (G,) vector h per
                                    sequence, a class label or a dense embedding; every layer adds Vf h / Vg h to its
                                    filter / gate pre-activations (``filter_cond_convs`` / ``gate_cond_convs``, 1x1, no bias)
        local_condition_channels (Int): C > 0: local conditioning (paper section 2.5) on a (C, F) series y at one frame per
                                    ``local_condition_hop`` samples (repeat upsampling): position t adds Uf y[:, t // hop] /
                                    Ug y[:, t // hop] (``filter_local_convs`` / ``gate_local_convs``, 1x1, no bias)
        local_condition_hop (Int):  samples per frame of the local condition (>= 1; required when C > 0)
        local_condition_upsample_scales (tuple of Int): a learned upsampler instead of repetition: ``local_upsample[i]`` is a
                                    ConvTranspose1d(C, C, 2 s_i, stride=s_i) that maps F frames to F * s_i (no nonlinearity
                                    between stages); the product of the s_i must be the hop.  Initialised to exact repetition.
                                    Position t then adds Uf c[:, t] / Ug c[:, t], c = the upsampled series.

    Shape:
        - Input: (N, classes, L) float32 one-hot, L >= receptive_field + output_length - 1 recommended
        - Output: (N * output_length, classes)
    """

    def __init__(self, layers=10, blocks=4, dilation_channels=32, residual_channels=32, skip_channels=256,
                 end_channels=256, classes=256, output_length=32, kernel_size=2, dtype=torch.FloatTensor, bias=False,
                 condition_channels=0, local_condition_channels=0, local_condition_hop=None,
                 local_condition_upsample_scales=None):
        super(WaveNetModel, self).__init__()
        self.layers = layers
        self.blocks = blocks
        self.dilation_channels = dilation_channels
        self.residual_channels = residual_channels
        self.skip_channels = skip_channels
        self.classes = classes
        self.kernel_size = kernel_size
        self.dtype = dtype

        self.dilations = []          # (dilation, init_dilation) per layer, as the reference stores them
        self.dilated_queues = []
        self.filter_convs = nn.ModuleList()
        self.gate_convs = nn.ModuleList()
        self.residual_convs = nn.ModuleList()
        self.skip_convs = nn.ModuleList()

        # parameter creation order == the reference's (start; filter, gate, residual, skip per layer; end_1; end_2)
        # so that a seeded construction reproduces its initial weights
        self.start_conv = nn.Conv1d(classes, residual_channels, kernel_size=1, bias=bias)
        receptive_field, previous = 1, 1
        for _ in range(blocks):
            d = 1
            for _ in range(layers):
                self.dilations.append((d, previous))
                self.dilated_queues.append(DilatedQueue(max_length=(kernel_size - 1) * d + 1,
                                                        num_channels=residual_channels, dilation=d, dtype=dtype))
                self.filter_convs.append(nn.Conv1d(residual_channels, dilation_channels, kernel_size, bias=bias))
                self.gate_convs.append(nn.Conv1d(residual_channels, dilation_channels, kernel_size, bias=bias))
                self.residual_convs.append(nn.Conv1d(dilation_channels, residual_channels, 1, bias=bias))
                self.skip_convs.append(nn.Conv1d(dilation_channels, skip_channels, 1, bias=bias))
                receptive_field += (kernel_size - 1) * d
                previous = d
                d *= 2
        self.end_conv_1 = nn.Conv1d(skip_channels, end_channels, 1, bias=True)
        self.end_conv_2 = nn.Conv1d(end_channels, classes, 1, bias=True)
        # created last, so that a seeded construction gives every other parameter the value an unconditioned net gets
        self.condition_channels = condition_channels
        if condition_channels > 0:
            self.filter_cond_convs = nn.ModuleList()
            self.gate_cond_convs = nn.ModuleList()
            for _ in range(layers * blocks):
                self.filter_cond_convs.append(nn.Conv1d(condition_channels, dilation_channels, 1, bias=False))
                self.gate_cond_convs.append(nn.Conv1d(condition_channels, dilation_channels, 1, bias=False))
        # created after the global ones, for the same reason
        if local_condition_channels > 0 and (isinstance(local_condition_hop, bool) or not isinstance(local_condition_hop, int)
                                             or local_condition_hop < 1):
            raise ValueError(f"local_condition_hop must be an int >= 1 when local_condition_channels > 0, got {local_condition_hop!r}")
        self.local_condition_channels = local_condition_channels
        self.local_condition_hop = local_condition_hop if local_condition_channels > 0 else None
        if local_condition_channels > 0:
            self.filter_local_convs = nn.ModuleList()
            self.gate_local_convs = nn.ModuleList()
            for _ in range(layers * blocks):
                self.filter_local_convs.append(nn.Conv1d(local_condition_channels, dilation_channels, 1, bias=False))
                self.gate_local_convs.append(nn.Conv1d(local_condition_channels, dilation_channels, 1, bias=False))
        # created after the local ones, for the same reason
        if local_condition_upsample_scales is not None:
            scales = local_condition_upsample_scales
            if local_condition_channels <= 0:
                raise ValueError("local_condition_upsample_scales needs local_condition_channels > 0")
            try:
                scales = tuple(scales)
            except TypeError:
                raise ValueError(f"local_condition_upsample_scales must be a sequence of ints >= 1, got {scales!r}") from None
            if not scales or any(isinstance(s, bool) or not isinstance(s, int) or s < 1 for s in scales):
                raise ValueError(f"local_condition_upsample_scales must be a sequence of ints >= 1, got {scales!r}")
            if math.prod(scales) != local_condition_hop:
                raise ValueError(f"the product of local_condition_upsample_scales {scales} must equal local_condition_hop "
                                 f"{local_condition_hop}")
            C = local_condition_channels
            self.local_condition_upsample_scales = scales
            self.local_upsample = nn.ModuleList(nn.ConvTranspose1d(C, C, 2 * s, stride=s) for s in scales)
            with torch.no_grad():                   # exact repetition: stage i copies frame f to positions [f s, (f + 1) s)
                for conv, s in zip(self.local_upsample, scales):
                    conv.weight.zero_()
                    conv.bias.zero_()
                    for c in range(C):
                        conv.weight[c, c, s // 2:s // 2 + s] = 1.0

        self.output_length = output_length
        self.receptive_field = receptive_field

    # ------------------------------------------------------------------ runtime plumbing
    def _runtime(self):
        # created lazily so that objects restored from a pickle (torch.load of a whole model) work too
        rt = self.__dict__.get("_rt")
        if rt is None:
            rt = _Runtime(self)
            self.__dict__["_rt"] = rt
        return rt

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop("_rt", None)               # device workspaces / native handles are not part of a snapshot
        state.pop("_shadow", None)
        return state

    # ------------------------------------------------------------------ training-time path
    def wavenet(self, input, dilation_func=None, condition=None, local_condition=None):
        """All T_final output columns, (N, classes, T_final), like the reference's wavenet() with wavenet_dilate.
        With ``dilation_func=self.queue_dilate`` it advances the fast-generation state by the one-hot column(s)
        in ``input`` and returns the logits of the last one as (1, classes, 1)."""
        if dilation_func is not None and getattr(dilation_func, "__func__", None) is WaveNetModel.queue_dilate:
            if getattr(self, "condition_channels", 0) or getattr(self, "local_condition_channels", 0):
                raise NotImplementedError("wavenet_b200: wavenet(x, queue_dilate) exists for the reference's unconditioned "
                                          "models; sample a conditioned model with generate_fast(..., condition=, "
                                          "local_condition=)")
            return self._queue_step(input)
        n = input.size(0)
        y = self._stack(input, None, condition=condition, local_condition=local_condition)
        return y.view(n, -1, self.classes).transpose(1, 2).contiguous()

    def wavenet_dilate(self, input, dilation, init_dilation, i):
        return dilate(input, dilation, init_dilation)

    def queue_dilate(self, input, dilation, init_dilation, i):
        queue = self.dilated_queues[i]
        queue.enqueue(input.data[0])
        return queue.dequeue(num_deq=self.kernel_size, dilation=dilation).unsqueeze(0)

    def _condition(self, condition, n):
        """The (n, G) float32 condition rows on the model's device for ``condition`` -- an int array / tensor (n,) of
        labels in [0, G) (one-hot rows) or a float (n, G) of dense vectors -- or None for an unconditioned model.  Raises
        when a conditioned model gets no condition, an unconditioned one gets one, or the shape / labels are wrong."""
        G = getattr(self, "condition_channels", 0)          # whole-model pickles made before conditioning existed lack it
        if not G:
            if condition is not None:
                raise ValueError("this model has no conditioning (condition_channels=0) but a condition was given")
            return None
        if condition is None:
            raise ValueError(f"this model is conditioned on {G} channels: pass condition= (labels (N,) or vectors (N, {G}))")
        if torch.is_tensor(condition) and condition.requires_grad and torch.is_grad_enabled():
            raise NotImplementedError("wavenet_b200: no gradient with respect to the condition (the backward computes the "
                                      "conditioning weights' gradients only); detach it, or learn the embedding as V itself "
                                      "by passing labels")
        try:
            c = condition.detach() if torch.is_tensor(condition) else torch.as_tensor(np.asarray(condition))
        except (TypeError, ValueError, RuntimeError) as e:
            raise ValueError(f"condition must hold int labels or float vectors: {e}") from None
        if c.dtype.is_floating_point:
            if tuple(c.shape) != (n, G):
                raise ValueError(f"a dense condition must be a float ({n}, {G}) array, got shape {tuple(c.shape)}")
            c = c.to(torch.float32)
        elif c.dtype in (torch.uint8, torch.int8, torch.int16, torch.int32, torch.int64):
            if tuple(c.shape) != (n,):
                raise ValueError(f"condition labels must be an int ({n},) array, got shape {tuple(c.shape)}")
            c = c.to(torch.int64)
            if n and (int(c.min()) < 0 or int(c.max()) >= G):
                raise ValueError(f"condition labels must lie in [0, {G}), got [{int(c.min())}, {int(c.max())}]")
            c = torch.nn.functional.one_hot(c, G).to(torch.float32)
        else:
            raise ValueError(f"condition must hold int labels or float vectors, got {c.dtype}")
        return c.to(self._runtime().device()).contiguous()

    def _local_condition(self, local_condition, n, positions):
        """The (n, C, F) float32 local condition series on the model's device for ``local_condition`` (a float array /
        tensor), or None for a model without local conditioning.  F must cover ``positions`` positions: F >= ceil(positions /
        hop).  A tensor that requires grad is returned as it is (moved / cast through autograd), so that it receives its
        gradient.  Raises like _condition."""
        C = getattr(self, "local_condition_channels", 0)    # whole-model pickles made before local conditioning lack it
        if not C:
            if local_condition is not None:
                raise ValueError("this model has no local conditioning (local_condition_channels=0) but a local_condition "
                                 "was given")
            return None
        hop = self.local_condition_hop
        need = -(-positions // hop)
        if local_condition is None:
            raise ValueError(f"this model is locally conditioned on {C} channels: pass local_condition= (a float "
                             f"({n}, {C}, F) series, F >= {need} frames of {hop} samples)")
        try:
            y = local_condition if torch.is_tensor(local_condition) else torch.as_tensor(np.asarray(local_condition))
        except (TypeError, ValueError, RuntimeError) as e:
            raise ValueError(f"local_condition must be a float array: {e}") from None
        if not y.dtype.is_floating_point:
            raise ValueError(f"local_condition must be a float ({n}, {C}, F) array, got {y.dtype}")
        if y.dim() != 3 or y.shape[0] != n or y.shape[1] != C:
            raise ValueError(f"local_condition must be a float ({n}, {C}, F) array, got shape {tuple(y.shape)}")
        if y.shape[2] < need:
            raise ValueError(f"local_condition has {y.shape[2]} frames; {positions} positions at hop {hop} need at least {need}")
        if not (y.requires_grad and torch.is_grad_enabled()):
            y = y.detach()
        return y.to(self._runtime().device(), torch.float32).contiguous()

    def _upsample(self, y, positions):
        """The learned upsampler: (N, C, F) frame-rate series -> (N, C, positions) contiguous audio-rate features c.  Stage i
        maps F frames to (F + 1) s_i and keeps [s_i // 2, s_i // 2 + F s_i), so c has F * hop positions before the crop and
        position t is still "frame t // hop"."""
        c = y
        with _exact_convolutions():
            for conv in self.local_upsample:
                s, n = conv.stride[0], c.shape[2]
                c = conv(c)[:, :, s // 2:s // 2 + n * s]
        return c[:, :, :positions].contiguous()

    def _stack(self, input, out_len, index_input=False, condition=None, local_condition=None):
        cond = self._condition(condition, input.size(0))
        y = self._local_condition(local_condition, input.size(0), input.size(-1))
        hop = None if y is None else self.local_condition_hop
        if torch.is_grad_enabled() and (any(p.requires_grad for p in self.parameters()) or (y is not None and y.requires_grad)):
            if input.requires_grad:
                raise NotImplementedError("wavenet_b200: no gradient with respect to the input (it is one-hot data)")
            return _StackFunction.apply(self, input, out_len, index_input, cond, y, hop, *self.parameters())
        rt = self._runtime()
        with torch.cuda.device(rt.device()):       # native launches go to the CURRENT device: make it the model's
            if y is not None and getattr(self, "local_upsample", None) is not None:
                return rt.stack_forward(input, out_len, index_input=index_input, cond=cond,
                                        upsampled=self._upsample(y, input.size(-1)))
            return rt.stack_forward(input, out_len, index_input=index_input, cond=cond,
                                    local=None if y is None else (y, hop))

    def forward(self, input, condition=None, local_condition=None):
        """(N, classes, L) -> (N * output_length, classes): logits of the last ``output_length`` frames.
        condition: for a conditioned model, labels (N,) or vectors (N, G) (see _condition).
        local_condition: for a locally conditioned model, a float (N, C, F) series; frame f conditions input positions
        [f * hop, (f + 1) * hop), and the output at position t predicts sample t + 1 (see _local_condition)."""
        return self._stack(input, self.output_length, condition=condition, local_condition=local_condition)

    def forward_indices(self, indices, condition=None, local_condition=None):
        """Same as ``forward(one_hot(indices))`` bit for bit, from (N, L) uint8 / int64 mu-law indices:
        start_conv on a one-hot column is a gather of one weight column (SURVEY.md section 8, row a4 / f2)."""
        return self._stack(indices, self.output_length, index_input=True, condition=condition,
                           local_condition=local_condition)

    # ------------------------------------------------------------------ generation
    def generate(self, num_samples, first_samples=None, temperature=1., condition=None):
        """The slow sampler (reference wavenet_model.py:198-235): every new sample re-evaluates the whole stack on a window
        of the last ``receptive_field`` samples.  The reference's own body cannot run (``self.scope`` at :209 does not exist
        and :230-235 concatenates Long and Float tensors); this restates its evident intent with the same schedule: the
        given samples are left-padded with zeros (class 0) to one receptive field, each step takes the last column of the
        training-path forward on the window, draws with numpy's global RNG (or the argmax for ``temperature == 0``) and
        appends.  Returns the mu-law expanded float64 waveform of the WHOLE sequence (padding + given + generated), as the
        reference's closing lines do.  One device->host sync per sample: use generate_fast for anything but cross-checks."""
        if getattr(self, "local_condition_channels", 0):
            raise NotImplementedError("wavenet_b200: the slow generate() has no local conditioning; use "
                                      "generate_fast(..., local_condition=)")
        self.eval()
        first = np.zeros(1, dtype=np.int64) if first_samples is None else self._first_array(first_samples)
        rf = self.receptive_field
        if first.shape[0] < rf:
            first = np.concatenate([np.zeros(rf - first.shape[0], dtype=np.int64), first])
        seq = list(first.tolist())
        rt = self._runtime()
        dev = rt.device()
        cond = self._condition(self._one_condition(condition), 1)
        with torch.no_grad(), torch.cuda.device(dev):
            for _ in range(num_samples):
                window = torch.tensor(seq[-rf:], dtype=torch.int64, device=dev).view(1, rf)
                x = rt.stack_forward(window, 1, index_input=True, cond=cond)[0]
                if temperature > 0:
                    prob = torch.softmax(x / temperature, dim=0).cpu().numpy()
                    seq.append(int(np.random.choice(self.classes, p=prob)))
                else:
                    seq.append(int(torch.argmax(x)))
        self.train()
        generated = (np.asarray(seq, dtype=np.float64) / self.classes) * 2. - 1
        return mu_law_expansion(generated, self.classes)

    @staticmethod
    def _one_condition(condition):
        """The condition of ONE stream (a label, or a (G,) vector) as a batch of one: (1,) or (1, G)."""
        if condition is None:
            return None
        c = condition.detach().cpu().numpy() if torch.is_tensor(condition) else np.asarray(condition)
        return c.reshape(1) if c.ndim == 0 else (c.reshape(1, -1) if c.ndim == 1 and c.dtype.kind == "f" else c)

    def _first_array(self, first_samples):
        if first_samples is None:
            return np.full((1,), self.classes // 2, dtype=np.int64)
        if torch.is_tensor(first_samples):
            first_samples = first_samples.detach().cpu().numpy()
        return np.asarray(first_samples).astype(np.int64).reshape(-1)

    def _cuda_shadow(self):
        """A CUDA copy of a CPU-resident model, refreshed when the parameters change.  The reference's own scripts
        generate from a *CPU copy* of the model in a logging thread (train_script.py:48, model_logging.py:55-58); that
        call lands here and still runs the persistent CUDA sampler -- only the weights are copied over."""
        if not torch.cuda.is_available():
            raise RuntimeError("wavenet_b200: generate_fast needs a CUDA device (there is no CPU sampler)")
        key = tuple((p.data_ptr(), p._version) for p in self.parameters())
        sh = self.__dict__.get("_shadow")
        if sh is None or sh[0] != key:
            twin = WaveNetModel(layers=self.layers, blocks=self.blocks, dilation_channels=self.dilation_channels,
                                residual_channels=self.residual_channels, skip_channels=self.skip_channels,
                                end_channels=self.end_conv_1.out_channels, classes=self.classes,
                                output_length=self.output_length, kernel_size=self.kernel_size,
                                bias=self.start_conv.bias is not None,
                                condition_channels=getattr(self, "condition_channels", 0),
                                local_condition_channels=getattr(self, "local_condition_channels", 0),
                                local_condition_hop=getattr(self, "local_condition_hop", None),
                                local_condition_upsample_scales=getattr(self, "local_condition_upsample_scales", None))
            twin.load_state_dict(self.state_dict())
            sh = (key, twin.cuda())
            self.__dict__["_shadow"] = sh
        else:
            sh[1].load_state_dict(self.state_dict())       # cheap, and immune to writes through p.data
        return sh[1]

    def generate_fast(self, num_samples, first_samples=None, temperature=1., regularize=0.,
                      progress_callback=None, progress_interval=100, condition=None, local_condition=None,
                      top_k=0, top_p=1.0, prefill=False):
        """Fast-WaveNet sampling; returns the mu-law expanded waveform, float64 ndarray of ``num_samples`` values.

        Same schedule as the reference (wavenet_model.py:237-315): the queues are reset, the given samples warm
        them up, then every step feeds the chosen sample back.  ``temperature > 0`` draws from the softmax with
        numpy's GLOBAL RNG (one ``random_sample()`` per sample, which is what ``np.random.choice`` consumes), so
        ``np.random.seed(s)`` reproduces the reference's stream; ``temperature == 0`` takes the argmax.
        ``top_k`` / ``top_p`` truncate the draw (0 / 1.0: off): the classes are ranked by logit (ties: lower index), the
        first ``top_k`` are kept, of those the shortest ranked prefix holding ``top_p`` of their probability, and the
        draw is the same inverse CDF over the kept classes only.  No effect at ``temperature == 0``; ValueError for a
        negative or non-integer ``top_k`` or a ``top_p`` outside (0, 1].
        ``condition``: a conditioned model's label or (G,) vector for this stream.
        ``local_condition``: a locally conditioned model's (C, F) series for this stream; evaluation e (which reads sample
        e, the given samples first, and predicts sample e + 1) takes frame e // hop, so F >= ceil((n_given - 1 +
        num_samples) / hop).
        ``prefill=True``: the queues are filled from the prompt by one parallel forward over its last receptive field
        instead of one sequential evaluation per prompt sample (much faster for long prompts).  The history then comes
        from other (fp32-class) arithmetic, so a draw within rounding of a CDF edge, or an argmax near-tie, may go the
        other way; the default False keeps the sequential warm-up.  ValueError unless a bool.
        """
        top_k, top_p = _truncation(top_k, top_p)
        _check_prefill(prefill)
        if self.start_conv.weight.device.type != "cuda":
            twin = self._cuda_shadow()
            audio = twin.generate_fast(num_samples, first_samples=first_samples, temperature=temperature,
                                       regularize=regularize, progress_callback=progress_callback,
                                       progress_interval=progress_interval, condition=condition,
                                       local_condition=local_condition, top_k=top_k, top_p=top_p, prefill=prefill)
            for q, tq in zip(self.dilated_queues, twin.dilated_queues):
                q.data, q.in_pos, q.out_pos = tq.data, tq.in_pos, tq.out_pos
            self.train()
            return audio
        cond = self._condition(self._one_condition(condition), 1)
        first = self._first_array(first_samples)
        num_given = first.shape[0]
        if local_condition is not None:
            local_condition = local_condition[None] if torch.is_tensor(local_condition) else np.asarray(local_condition)[None]
        local = self._sampler_local(self._local_condition(local_condition, 1, num_given - 1 + num_samples),
                                    num_given - 1 + num_samples)
        self.eval()
        total = num_given + num_samples
        callbacks = []
        if progress_callback is not None:
            for i in range(num_given - 1):                               # warm-up loop, wavenet_model.py:266-269
                if i % progress_interval == 0:
                    callbacks.append((i, lambda i=i: progress_callback(i, total)))
            for i in range(num_samples):                                 # sampling loop, :309-311
                if (i + num_given) % progress_interval == 0:
                    callbacks.append((num_given - 1 + i, lambda i=i: progress_callback(i + num_given, total)))
        rt = self._runtime()
        with torch.cuda.device(rt.device()):
            idx, _, _ = rt.generate(num_samples, first[None, :], temperature, regularize, callbacks=callbacks, cond=cond,
                                    local=local, top_k=top_k, top_p=top_p, prefill=prefill)
        self._export_queues()
        self.train()
        generated = (idx[0] / self.classes) * 2. - 1
        return mu_law_expansion(generated, self.classes)

    def generate_fast_batch(self, num_samples, first_samples, temperature=1., regularize=0., uniforms=None,
                            forced=None, return_logits=False, condition=None, local_condition=None, top_k=0, top_p=1.0,
                            prefill=False):
        """``n_streams`` independent generate_fast runs batched in one kernel (the reference has a single stream,
        wavenet_model.py:179).  first_samples: (n_streams, n_given) ints.  Returns int64 indices
        (n_streams, num_samples) [and the per-step logits].  Run through the same sampler kernel, stream s equals a
        single-stream run bit for bit (256- and 512-wide nets of 256 classes run the tensor-core cluster kernel for any
        number of streams; on a 512-wide net every handle holds its own 6 MB of pre-split weight images per layer, about
        505 MB at cfg 5; other nets a latency kernel for one stream and one thread-block cluster per stream otherwise,
        which differ at rounding level).  condition: a conditioned model's labels (n_streams,) or vectors (n_streams, G), one per stream.
        local_condition: a locally conditioned model's (n_streams, C, F) series, one per stream (see generate_fast).
        top_k, top_p: the truncated draw of generate_fast.

        Every stream may have its own job: ``first_samples`` may be a list of n_streams 1-D int arrays of any lengths >= 1,
        ``num_samples`` a sequence of n_streams counts, ``temperature``, ``regularize``, ``top_k`` and ``top_p`` sequences
        of n_streams values, ``uniforms`` / ``forced`` (n_streams, >= n_s) arrays or lists whose row s supplies the first
        n_s entries, and ``local_condition`` a list of (C, F_s) series.  Stream s then gives what
        ``generate_fast(n_s, first_samples[s], ...)`` with its own settings gives; with ``uniforms=None`` the streams with
        temperature > 0 draw their n_s uniforms from numpy's global RNG in stream order, so a seeded batch equals seeded
        generate_fast calls in order.  With a sequence of counts or prompts of different lengths the return is a list of
        per-stream index arrays (n_s,) [and a list of (n_s, classes) logits]; otherwise it is the arrays above.  Streams
        that finish early keep running until the longest job is done.  ValueError for a malformed argument, before any
        device work.  prefill: as for generate_fast, over the prompts' common length (a longer prompt's remainder is
        still evaluated sample by sample)."""
        _check_prefill(prefill)
        plan = _stream_plan(first_samples, num_samples, temperature, regularize, top_k, top_p)
        NS = plan.n_streams
        cond = self._condition(condition, NS)
        positions = [g - 1 + n for g, n in zip(plan.n_given, plan.counts)]
        if plan.per_stream:
            local = self._per_stream_local(local_condition, positions, plan.n_evals)
            if uniforms is not None:          # the rows are checked here, before any device work
                plan.rows(uniforms, np.float64, "uniforms", need=[t > 0 for t in plan.temperature])
            if forced is not None:
                plan.rows(forced, np.int32, "forced")
            first, counts = [r[:g] for r, g in zip(plan.first, plan.n_given)], plan.counts
        else:
            local = self._sampler_local(self._local_condition(local_condition, NS, plan.n_evals), plan.n_evals)
            first, counts = plan.first.astype(np.int64), plan.counts[0]
        self.eval()
        rt = self._runtime()
        with torch.cuda.device(rt.device()):
            idx, logits, _ = rt.generate(counts, first, temperature, regularize, uniforms=uniforms,
                                         forced=forced, want_logits=return_logits, cond=cond, local=local,
                                         top_k=top_k, top_p=top_p, prefill=prefill)
        self._export_queues()
        self.train()
        if plan.ragged:
            idx = [idx[s, :n] for s, n in enumerate(plan.counts)]
            logits = [logits[s, :n] for s, n in enumerate(plan.counts)] if return_logits else None
        elif plan.per_stream:
            idx = idx[:, :plan.counts[0]]
            logits = logits[:, :plan.counts[0]] if return_logits else None
        return (idx, logits) if return_logits else idx

    def sampling_session(self, n_slots, prefill=False, return_logits=False, local_window=None):
        """Continuous batching: a SamplingSession of ``n_slots`` streams on its own sampler handle.  ``submit(first_samples,
        num_samples, temperature=1., regularize=0., top_k=0, top_p=1.0, condition=None, uniforms=None,
        local_condition=None)`` queues a job and returns its id; ``step(n_evals)`` seats queued jobs into free slots, runs
        n_evals evaluations of every slot and returns {job_id: new indices} (with return_logits: {job_id: (indices,
        logits)}); ``result(job_id)`` gives a done job's output; ``pending`` / ``active`` count queued and running jobs.  Each
        job gives, bit for bit, what a generate_fast_batch call of n_slots copies of that job gives (same uniforms, same
        prefill); with uniforms=None a seeded sequence of submits draws what seeded generate_fast calls in the same order
        draw.  ``prefill=True`` primes each job's rings from its prompt with one forward (see generate_fast).  Global
        conditioning is per job.  The model's parameters must not change while the session lives (RuntimeError at the next
        step).

        A locally conditioned model (a vocoder) needs ``local_window``, an int >= 1, and every job its own (C, F) series
        (``submit(..., local_condition=y)``); ValueError otherwise, and for ``local_window`` on any other model.  Each slot
        reads its own frames at its own position.  A step runs in launches of at most ``local_window`` evaluations, each
        after one table build of every slot's nf = ceil((local_window - 1) / hop) + 1 frames (hop 1 under a learned
        upsampler: nf = local_window) into one buffer of n_layers x n_slots x nf x 2 x dilation_channels floats, allocated
        here.  On the cfg-2 net (50 layers of 256 dilation channels): 64 slots at hop 80 and local_window 1 000 take about
        90 MB; 64 slots of a learned upsampler at local_window 64 about 420 MB.  A larger window builds less often and
        holds more memory."""
        return SamplingSession(self, n_slots, prefill=prefill, return_logits=return_logits, local_window=local_window)

    def _per_stream_local(self, local_condition, positions, n_evals):
        """The sampler's (series, hop) for per-stream jobs (None: no local conditioning).  local_condition: an (NS, C, F)
        array or a list of NS (C, F_s) series, stream s needing ceil(positions[s] / hop) frames.  Each series is checked
        and upsampled at its own length (an upsampled position near a series' end depends on the next frame, so a padded
        batch would change it), then the frame axis is padded with zeros to cover the call's n_evals evaluations; only
        the discarded outputs of a stream past its own job read the padding."""
        if not getattr(self, "local_condition_channels", 0) or local_condition is None:
            return self._sampler_local(self._local_condition(local_condition, len(positions), max(positions)), n_evals)
        if isinstance(local_condition, (list, tuple)):
            if len(local_condition) != len(positions):
                raise ValueError(f"local_condition must hold {len(positions)} series (one per stream), got "
                                 f"{len(local_condition)}")
            series = list(local_condition)
        else:
            y = local_condition if torch.is_tensor(local_condition) else np.asarray(local_condition)
            if y.ndim != 3 or y.shape[0] != len(positions):
                raise ValueError(f"local_condition must be an ({len(positions)}, C, F) array or a list of (C, F_s) series, "
                                 f"got shape {tuple(y.shape)}")
            series = [y[s] for s in range(len(positions))]
        ys = []
        for s, (y, pos) in enumerate(zip(series, positions)):
            y = y if torch.is_tensor(y) else np.asarray(y)
            ys.append(self._local_condition(y[None], 1, pos))
        upsample = getattr(self, "local_upsample", None) is not None
        with torch.no_grad(), torch.cuda.device(self._runtime().device()):
            if upsample:
                ys = [self._upsample(y.detach(), pos) for y, pos in zip(ys, positions)]
                hop, width = 1, n_evals
            else:
                hop = self.local_condition_hop
                width = max(max(y.shape[2] for y in ys), -(-n_evals // hop))
            out = torch.zeros(len(ys), ys[0].shape[1], max(width, 1), device=ys[0].device, dtype=torch.float32)
            for s, y in enumerate(ys):
                out[s, :, :min(y.shape[2], out.shape[2])] = y[0, :, :out.shape[2]]
        return out, hop

    def _sampler_local(self, y, evals):
        """The sampler's (series, hop) for the validated frame-rate series ``y`` (None: no local conditioning).  A learned
        upsampler runs once here, and the sampler reads its output at hop 1 (one table row per evaluation)."""
        if y is None:
            return None
        if getattr(self, "local_upsample", None) is None:
            return y.detach(), self.local_condition_hop
        with torch.no_grad(), torch.cuda.device(self._runtime().device()):
            return self._upsample(y.detach(), evals), 1

    def _export_queues(self):
        """Point ``dilated_queues[i].data`` at stream 0 of the sampler's device rings (a (C, max_length) view).
        Ring elements are 8-byte {value, tag} pairs (see csrc/gen.cu; plain floats under the grid-barrier kernel); the view
        picks the values."""
        rt = self._runtime()
        s, evals = rt.last_run["sampler"], rt.last_run["evals"]
        R, NS, off = self.residual_channels, s["n_streams"], 0
        # the grid-barrier kernel (1) keeps plain floats in the ring memory, every other kernel {value, tag} pairs
        plain = native.lib().wn_gen_kernel_id(s["handle"]) == 1
        pairs = s["rings"].view(-1, 1) if plain else s["rings"].view(-1, 2)
        for q in self.dilated_queues:
            n = q.max_length * NS * R
            q.data = pairs[off:off + n, 0].view(q.max_length, NS, R)[:, 0, :].t()
            q.in_pos = q.out_pos = evals % q.max_length
            off += n

    def _queue_step(self, input):
        """``wavenet(input, self.queue_dilate)`` (reference wavenet_model.py:177-184, the body of generate_fast's loops):
        push the one-hot column(s) of ``input`` (1, classes, n) through the cached queues, one evaluation of the
        persistent sampler kernel each, and return the logits of the last column as (1, classes, 1).  The device rings
        are the queue state; a new session starts when every ``dilated_queues[i].reset()`` has been called since the
        last step (what generate_fast does first, wavenet_model.py:250), or on the first call."""
        rt = self._runtime()
        dev = rt.device()
        if input.dim() != 3 or input.size(0) != 1 or input.size(1) != self.classes:
            raise RuntimeError(f"queue_dilate handles a single stream: input must be (1, {self.classes}, n), "
                               f"got {tuple(input.shape)} (the reference enqueues input.data[0] only)")
        col = input.detach().to(dev, torch.float32)[0]                        # (classes, n)
        idx = col.argmax(0)
        if not bool(((col.max(0).values == 1) & (col.sum(0) == 1) & (col.min(0).values == 0)).all()):
            raise NotImplementedError("wavenet(input, queue_dilate) needs one-hot columns (the sampler gathers the "
                                      "start_conv column of the sample index)")
        ses = rt.__dict__.get("step_session")
        with torch.cuda.device(dev):
            if ses is None or all(getattr(q, "was_reset", False) for q in self.dilated_queues) \
                    or ses["sampler"] is not rt.samplers.get(1):
                s = rt.sampler(1)
                native.check(native.lib().wn_gen_reset(s["handle"], torch.cuda.current_stream(dev).cuda_stream), "gen reset")
                native.check(native.lib().wn_gen_set_condition(s["handle"], None), "gen condition")
                # sampler handles are cached per stream count: a per-stream setting of an earlier call must not reach
                # the queue step's scalar launches
                native.check(native.lib().wn_gen_set_stream_params(s["handle"], None), "gen stream params")
                s["cond"] = None
                ses = dict(sampler=s, t=0, inp=torch.zeros(1, dtype=torch.int32, device=dev),
                           out=torch.zeros(1, dtype=torch.int32, device=dev),
                           logits=torch.zeros(self.classes, dtype=torch.float32, device=dev))
                rt.step_session = ses
                for q in self.dilated_queues:
                    q.was_reset = False
            lib, stream = native.lib(), torch.cuda.current_stream(dev).cuda_stream
            for j in range(col.size(1)):
                t = ses["t"]
                ses["inp"].copy_(idx[j:j + 1].to(torch.int32))
                a = native.GenRunArgs()
                # schedule "1 given sample, t+1 samples": evaluation t reads first[0] (t == 0) or forced[t-1] and writes
                # sample t; the buffers hold ONE element each, so the pointers are biased to put element t at their start
                a.d_first, a.n_given = ses["inp"].data_ptr(), 1
                a.d_forced = ses["inp"].data_ptr() - 4 * (t - 1) if t > 0 else None
                a.d_uniforms = None
                a.d_out_idx = ses["out"].data_ptr() - 4 * t
                a.d_out_logits = ses["logits"].data_ptr() - 4 * self.classes * t
                a.n_samples, a.t0, a.n_evals = t + 1, t, 1
                a.temperature, a.regularize = 0.0, 0.0
                native.check(lib.wn_gen_run(ses["sampler"]["handle"], ctypes.byref(a), stream), "gen run (queue step)")
                ses["t"] = t + 1
            rt.last_run = dict(evals=ses["t"], sampler=ses["sampler"])
        self._export_queues()
        return ses["logits"].clone().view(1, self.classes, 1)

    def invalidate_packed_weights(self):
        """Call after writing parameters through ``p.data`` outside a training step (see _Runtime.invalidate)."""
        self._runtime().invalidate()

    # ------------------------------------------------------------------ utilities (reference wavenet_model.py:318-346)
    def parameter_count(self):
        return sum(int(np.prod(list(p.size()))) for p in self.parameters())

    def cpu(self, type=torch.FloatTensor):
        self.dtype = type
        for q in self.dilated_queues:
            q.dtype = self.dtype
        super().cpu()


def load_latest_model_from(location, use_cuda=True):
    files = [location + "/" + f for f in os.listdir(location)]
    newest_file = max(files, key=os.path.getctime)
    print("load model " + newest_file)
    if use_cuda:
        model = torch.load(newest_file, weights_only=False)
    else:
        model = load_to_cpu(newest_file)
    return model


def load_to_cpu(path):
    model = torch.load(path, map_location=lambda storage, loc: storage, weights_only=False)
    model.cpu()
    return model
