"""Every whole-stack forward kernel through the C ABI, layer by layer against the float64 block reference (tests/block_ref.py),
in the style of tests/test_gpu_kernels_f64.py.

The whole-stack launch runs all residual blocks of a forward in one persistent kernel: a layer-major item list (256 frames of
one sequence per item) is dealt round-robin to at most sms / 2 CTA pairs, and an item waits on device-side counters for the
previous layer's items that wrote the frames it reads.  There are 15 kernels: {plain (wn_tb_stack_fwd), global condition
table (wn_tb_stack_fwd_cond), frame table (wn_tb_stack_fwd_cond_frames, which also serves a table with a global term),
K-slab (wn_tb_stack_fwd_local), K-slab + global table} x {256 channels bf16 pairs, 256 bf16, 512 bf16}.

The test builds the launch arguments itself, as _Runtime._forward_tb does, so it chooses B, L, the frame plan and the
buffers.  Every layer's saved output is compared with block_forward applied to that layer's saved input, so errors do not
compound; the skip sum is chained through the reference and checked at the end.  A condition enters the reference as
per-position filter / gate biases: the fp32 table the test hands the kernel (global, frames), or U c[t] formed on the
emulated operands (K-slab).  Bars are those of the per-layer kernel tests (helpers.kernel_check), K = 2C (+ Cpad).

Shapes:
  (a) the runtime's plan of a 10-layer net (d = 1 ... 512), B = 3, L = 1 500;
  (b) wrap: a hand-made plan whose out_start values sit one frame off the previous layer's tile boundaries, dilations up
      to 512 (more than one item, so the producer's lower wait bound clamps to the previous layer's first frame), and B, L
      sized from the SM count so that every layer has more than twice as many items as there are CTA pairs, with a ragged
      remainder: pairs then reach layer l + 1 while others are still in layer l;
  (c) frame tables with hops that put frame boundaries on, and one frame beside, the 128 / 256-frame tile edges, and more
      frames than L needs;
  (d) K-slabs of C = 1, 80 and 200 condition channels.
Every h buffer, fg_all and skip start as NaN: frames left of a layer's out_start must still hold it, and a kernel that read
such a frame would carry NaN into the checked outputs, which no bar passes.  The no-grad path (three rotating h buffers,
no fg_all, a write-after-read wait on the layer that last read a buffer) must give the save-mode launch's last h and skip
bit for bit, three launches in a row on one flag buffer."""
import ctypes
import functools

import pytest
import torch

import block_ref as BR
from helpers import kernel_check as _check, kernel_miss as _miss
from test_gpu_kernels_f64 import _gen, _nan, _pair, _planes, _sentinel_kept, _stream

pytestmark = pytest.mark.gpu
PRECS = [("pairs", 256), ("bf16", 256), ("bf16", 512)]
ENTRY = {"plain": "wn_tb_stack_fwd", "global": "wn_tb_stack_fwd_cond", "frames": "wn_tb_stack_fwd_cond_frames",
         "kslab": "wn_tb_stack_fwd_local", "kslab+global": "wn_tb_stack_fwd_local"}
BASE_DIL = [2 ** i for i in range(10)]


@functools.lru_cache(maxsize=None)
def _model(C, prec, Cl=0):
    """a 10-layer net (biases O(1)); with Cl > 0 it has a learned upsampler, whose U packs the K-slab kernels read"""
    import wavenet_model as wmod
    kw = dict(local_condition_channels=Cl, local_condition_hop=4, local_condition_upsample_scales=(4,)) if Cl else {}
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(C + Cl)
        m = wmod.WaveNetModel(layers=10, blocks=1, dilation_channels=C, residual_channels=C, skip_channels=C, end_channels=256,
                              classes=256, output_length=8, kernel_size=2, bias=True, **kw)
    g = _gen(17)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith(".bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
            if "_local_convs." in n:
                p.copy_(torch.randn(p.shape, generator=g) * Cl ** -0.5)
    m = m.cuda()
    m._runtime().tc_precision = "bf16x2" if prec == "pairs" else "bf16"
    return m


def _pairs():
    import native
    return native.device_info()["sm_count"] // 2


def _plan(shape):
    """B, L, dilations, in_start, out_start, skip_start"""
    if shape == "a":
        import wavenet_model as wmod
        B, L = 3, 1500
        plan = wmod.StackPlan(BASE_DIL, 2, L)
        return B, L, BASE_DIL, plan.in_start, plan.out_start, plan.skip_start
    if shape == "b":
        out = [1, 256, 513, 768, 1023, 1280]             # each one frame off the previous layer's tile boundaries
        B = 8
        tiles = -(-5 * _pairs() // (2 * B))              # the last (shortest) layer: >= 2.5x as many items as pairs
        L = out[-1] + 256 * (tiles - 1) + 100            # ragged last tile
        return B, L, [1, 128, 255, 512, 2, 256], [0] + out[:-1], out, 1300
    # c: every layer's tiles start on a multiple of 128, so frame boundaries of hop 128 / 256 sit on CTA / item edges
    out = [0, 128, 256, 384]
    return 2, 1100, [1, 256, 3, 129], [0] + out[:-1], out, 400


class _Case:
    """inputs, packed weights and condition operands of one whole-stack launch"""

    def __init__(self, variant, prec, C, shape, Cl=80, hop=80):
        import native
        self.lib, self.variant, self.prec, self.C = native.lib(), variant, prec, C
        self.B, self.L, self.dil, self.ins, self.outs, self.sk_s = _plan(shape)
        self.nl = len(self.dil)
        self.Cl = Cl if variant.startswith("kslab") else 0
        m = _model(C, prec, self.Cl)
        packs = m._runtime().packed_weights(_stream())
        self.tb_w, self.tb_b, self.p_id = packs["tb"]
        sd = {n: v.detach().cpu() for n, v in m.state_dict().items()}
        self.W = [BR.layer_weights(sd, i) for i in range(self.nl)]
        g = _gen(1000 + C + len(variant) + self.nl)
        B, L = self.B, self.L
        self.h0 = torch.randn(B, L, C, generator=g)
        self.table, self.hop, self.nf = None, None, None
        if variant in ("global", "kslab+global"):
            self.table = torch.randn(self.nl, B, 2 * C, generator=g) * 0.5
        if variant == "frames":
            self.hop, self.nf = hop, -(-L // hop) + 3          # more frames than the L positions read
            self.table = torch.randn(self.nl, B, self.nf, 2 * C, generator=g) * 0.5
        self.table_d = None if self.table is None else self.table.cuda()
        if self.Cl:
            self.u_all = packs["tb_local"][0]
            self.U = [torch.cat([sd[f"filter_local_convs.{i}.weight"], sd[f"gate_local_convs.{i}.weight"]], 0)[:, :, 0]
                      for i in range(self.nl)]
            self.c = torch.randn(B, self.Cl, L, generator=g)
            self.cpad = self.lib.wn_tb_local_padded_channels(self.Cl, self.p_id)
            self.c_pair = _nan(B, 2, self.cpad // 8, L, 8, dtype=torch.bfloat16)
            native.check(self.lib.wn_tb_local_from_channels(self.c.cuda().data_ptr(), self.c_pair.data_ptr(), B, self.Cl, L,
                                                            self.p_id, _stream()), "convert c")
        ints = lambda v: (ctypes.c_int * self.nl)(*v)
        self.c_dil, self.c_ins, self.c_outs = ints(self.dil), ints(self.ins), ints(self.outs)
        self.items = [B * -(-(L - o) // 256) for o in self.outs]
        total = self.lib.wn_tb_stack_items(self.nl, B, L, self.c_outs)
        assert total == sum(self.items)
        self.desc = torch.empty(self.nl * self.lib.wn_tb_stack_desc_bytes() + 128, device="cuda", dtype=torch.uint8)
        self.flags = torch.empty(total + self.nl, device="cuda", dtype=torch.int32)
        self.pairs = min(_pairs(), total)

    def launch(self, hs, fg_all, skip):
        """layer i reads hs[i] and writes hs[i + 1]; returns the entry point's code (0 or a refusal)"""
        import native
        sa = native.TbStackArgs()
        hp = native.ptr_array(hs)
        sa.h_ptrs = ctypes.cast(hp, native.c_void_pp)
        sa.d_skip, sa.d_w_all, sa.d_bias_all = skip.data_ptr(), self.tb_w.data_ptr(), self.tb_b.data_ptr()
        sa.d_fg_all = native.ptr(fg_all)
        sa.d_desc = (self.desc.data_ptr() + 127) // 128 * 128
        sa.d_flags = self.flags.data_ptr()
        sa.n_layers, sa.channels, sa.precision, sa.B, sa.L, sa.skip_start = self.nl, self.C, self.p_id, self.B, self.L, self.sk_s
        sa.dilations, sa.in_start, sa.out_start = self.c_dil, self.c_ins, self.c_outs
        fn, st, v = getattr(self.lib, ENTRY[self.variant]), _stream(), self.variant
        if v == "plain":
            return fn(ctypes.byref(sa), st)
        if v == "global":
            return fn(ctypes.byref(sa), self.table_d.data_ptr(), st)
        if v == "frames":
            return fn(ctypes.byref(sa), self.table_d.data_ptr(), self.nf, self.hop, st)
        return fn(ctypes.byref(sa), native.ptr(self.table_d), self.c_pair.data_ptr(), self.Cl, self.u_all.data_ptr(), st)

    def new_skip(self):
        return _nan(self.B, self.C // 4, self.L - self.sk_s, 4)

    def layer_weights(self, i, mode, table=None, u_scale=1.0, frame_shift=0, dilation=None):
        """layer i's weights with its condition as per-position filter / gate biases, operands formed as `mode` forms them"""
        W, L = self.W[i], self.L
        table = self.table if table is None else table
        if self.variant == "plain":
            return W
        if self.variant == "global":
            return BR.with_position_biases(W, BR.expand_table(table[i], L), self.outs[i])
        if self.variant == "frames":
            t = torch.arange(L)
            return BR.with_position_biases(W, table[i].double()[:, (t - frame_shift).clamp(min=0) // self.hop], self.outs[i])
        pre = BR.mm(self.c.transpose(1, 2), self.U[i] * u_scale, mode)
        if self.variant == "kslab":
            return BR.with_position_biases(W, pre, self.outs[i], keep_bias=True)
        return BR.with_position_biases(W, pre + BR.expand_table(table[i], L), self.outs[i])

    def header(self, shape):
        extra = {"frames": f" hop={self.hop} n_frames={self.nf}", "kslab": f" C={self.Cl}", "kslab+global": f" C={self.Cl}"}
        print(f"\n{ENTRY[self.variant]} ({self.variant}) {self.prec} {self.C} shape {shape}: B={self.B} L={self.L} "
              f"layers={self.nl} items/layer={self.items} CTA pairs={self.pairs} skip_start={self.sk_s}"
              + extra.get(self.variant, ""))


def _save_mode(cs):
    """the save-mode launch (every layer its own h buffer, fg_all kept), everything NaN first; returns hs, fg_all, skip"""
    B, L, C = cs.B, cs.L, cs.C
    hs = [_pair(cs.h0)] + [_nan(B, 2, C // 8, L, 8, dtype=torch.bfloat16) for _ in range(cs.nl)]
    fg_all = _nan(cs.nl, B, 2 * C // 4, L, 4)
    skip = cs.new_skip()
    import native
    native.check(cs.launch(hs, fg_all, skip), ENTRY[cs.variant])
    torch.cuda.synchronize()
    return hs, fg_all, skip


def _check_layers(cs, hs, fg_all, skip, control=None):
    """every layer's h_out, tanh and sigmoid, then the final skip, against the reference on that layer's saved input"""
    mode = cs.prec
    kind = "emu" if mode == "pairs" else "bf16"
    K = 2 * cs.C + (cs.cpad if cs.Cl else 0)
    sk_ex = sk_em = None
    for i, d in enumerate(cs.dil):
        in_s, out_s = cs.ins[i], cs.outs[i]
        _sentinel_kept(f"layer {i} h_out", hs[i + 1], out_s)
        _sentinel_kept(f"layer {i} fg", fg_all[i], out_s)
        hp = _planes(hs[i])
        ex = BR.block_forward(hp, cs.layer_weights(i, "exact"), d, in_s, out_s, cs.sk_s, sk_ex)
        em = BR.block_forward(hp, cs.layer_weights(i, mode), d, in_s, out_s, cs.sk_s, sk_em, mode=mode, pair_out=True)
        sk_ex, sk_em = ex["skip"], em["skip"]
        got_h = BR.value(_planes(hs[i + 1]))[:, out_s:]
        fg = BR.frames_from_chunks4(fg_all[i].cpu())[:, out_s:]
        bar = _check(f"layer {i} (d={d} in={in_s} out={out_s}) h_out", got_h, ex["h_out"], em["h_out"], kind, K=K)
        _check(f"layer {i} tanh", fg[..., :cs.C], ex["f"], em["f"], kind, K=K)
        _check(f"layer {i} sigmoid", fg[..., cs.C:], ex["g"], em["g"], kind, K=K)
        if control is not None and i == 1:
            what, Wm, dd = control(cs, i)
            _miss(what, got_h, BR.block_forward(hp, Wm, dd, in_s, out_s, cs.sk_s, None)["h_out"], bar)
    _check("skip", BR.frames_from_chunks4(skip.cpu()), sk_ex, sk_em, kind, K=K)


def _control(cs, i):
    """one deliberate mistake per variant in layer i's reference: (what, weights, dilation)"""
    d = cs.dil[i]
    if cs.variant == "plain":
        return "dilation + 1", cs.W[i], d + 1
    if cs.variant == "global":
        return "sequences 0 and 1 swapped in the table", cs.layer_weights(i, "exact", table=cs.table[:, [1, 0] + list(range(2, cs.B))]), d
    if cs.variant == "frames":
        return "frame index one position late", cs.layer_weights(i, "exact", frame_shift=1), d
    return "U zeroed", cs.layer_weights(i, "exact", u_scale=0.0), d


def _rotating_matches_save_mode(cs, hs, skip):
    """the no-grad path: hs[i] = hbuf[i % 3], no fg_all, three launches on one flag buffer, each bit-identical to save mode"""
    B, L, C = cs.B, cs.L, cs.C
    hbuf = [_nan(B, 2, C // 8, L, 8, dtype=torch.bfloat16) for _ in range(3)]
    last = cs.outs[-1]
    import native
    for run in range(3):
        hbuf[0].copy_(hs[0])                               # layer 2 overwrites the input buffer
        sk = cs.new_skip()
        native.check(cs.launch([hbuf[i % 3] for i in range(cs.nl + 1)], None, sk), ENTRY[cs.variant])
        torch.cuda.synchronize()
        assert torch.equal(sk, skip), f"rotating buffers, launch {run}: skip differs from the save-mode launch"
        assert torch.equal(hbuf[cs.nl % 3][:, :, :, last:], hs[cs.nl][:, :, :, last:]), \
            f"rotating buffers, launch {run}: last h differs from the save-mode launch"
    print(f"  rotating buffers: last h and skip bit-identical to save mode in 3 launches on one flag buffer")


@pytest.mark.parametrize("prec,C", PRECS)
@pytest.mark.parametrize("variant", list(ENTRY))
@pytest.mark.parametrize("shape", ["a", "b"])
def test_stack_kernel_layer_by_layer(shape, variant, prec, C):
    torch.set_num_threads(min(8, torch.get_num_threads()))
    cs = _Case(variant, prec, C, shape, hop=80 if shape == "a" else 257)
    cs.header(shape)
    if shape == "b":
        assert all(n > 2 * cs.pairs for n in cs.items), (cs.items, cs.pairs)
        assert cs.dil[3] > 256 and cs.outs[3] - cs.dil[3] < cs.outs[2]         # the lower wait bound clamps
    hs, fg_all, skip = _save_mode(cs)
    _check_layers(cs, hs, fg_all, skip, control=_control if (shape == "a" and prec == "pairs") else None)
    _rotating_matches_save_mode(cs, hs, skip)


@pytest.mark.parametrize("prec,C", PRECS)
@pytest.mark.parametrize("hop", [128, 129, 255, 256])
def test_stack_frames_kernel_at_tile_edges(hop, prec, C):
    torch.set_num_threads(min(8, torch.get_num_threads()))
    cs = _Case("frames", prec, C, "c", hop=hop)
    cs.header("c")
    hs, fg_all, skip = _save_mode(cs)
    _check_layers(cs, hs, fg_all, skip)


@pytest.mark.parametrize("prec,C", PRECS)
@pytest.mark.parametrize("variant,Cl", [("kslab", 1), ("kslab", 200), ("kslab+global", 1), ("kslab+global", 200)])
def test_stack_kslab_kernel_condition_widths(variant, Cl, prec, C):
    torch.set_num_threads(min(8, torch.get_num_threads()))
    cs = _Case(variant, prec, C, "c", Cl=Cl)
    cs.header("d")
    hs, fg_all, skip = _save_mode(cs)
    _check_layers(cs, hs, fg_all, skip)


@pytest.mark.parametrize("variant", list(ENTRY))
def test_stack_kernel_refuses_two_rotating_buffers(variant):
    """layer i + 1 would overwrite the buffer layer i is still reading: the entry point's guard refuses before any launch"""
    cs = _Case(variant, "pairs", 256, "c")
    hb = [_nan(cs.B, 2, cs.C // 8, cs.L, 8, dtype=torch.bfloat16) for _ in range(2)]
    rc = cs.launch([hb[i % 2] for i in range(cs.nl + 1)], None, cs.new_skip())
    msg = cs.lib.wn_last_error_string().decode()
    print(f"\n{ENTRY[variant]} ({variant}): two-buffer rotation -> code {rc}: {msg}")
    assert rc != 0 and "rotate three buffers" in msg
