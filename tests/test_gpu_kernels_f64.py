"""Each training-path block kernel alone, through the C ABI, against the float64 block references of tests/block_ref.py.

Inputs are seeded O(1) random tensors in the kernels' own layouts (every element matters equally); packed weights are the
model runtime's own packs; frame ranges are chosen by the test and placed at 0, on the 128-frame CTA and 256-frame item
boundaries and one frame either side, with dilations up to 512 so the taps cross CTA and item boundaries.  Output buffers
are filled with a sentinel (NaN) first: frames outside a kernel's write range must still hold it.

Bars follow from the operand widths (block_ref's emulation of exactly these inputs):
    rel_err(kernel, exact) <= 2 e_emu + acc(K),     e_emu = rel_err(emulated, exact)
    single-pass bf16 also   rel_err(kernel, emulated) <= 0.25 e_emu   (a wrong operand plane or a dropped term fails this)
    FFMA kernels            rel_err(kernel, exact) <= 1e-5
acc(K) = 2^-16 sqrt(K / 256) allows for the tensor cores' fp32 accumulation over a contraction of length K, which the
emulation (float64 sums) leaves out; see helpers.tc_acc.
rel_err is max|a - b| / max|b| per output tensor (per tap for weight gradients).  Every measured value is printed (-s)."""
import ctypes
import functools

import pytest
import torch

import block_ref as BR
from helpers import kernel_rel as _rel, kernel_check as _check, kernel_miss as _miss

pytestmark = pytest.mark.gpu
TB_PRECS = [("pairs", 256), ("bf16", 256), ("bf16", 512)]


def _sentinel_kept(what, t, lo):
    """frames [0, lo) along dim `t.dim() - 2` (the frame axis of every chunked layout here) still hold NaN"""
    if lo > 0:
        assert bool(torch.isnan(t.narrow(t.dim() - 2, 0, lo).float()).all()), f"{what}: wrote frames left of {lo}"


def _gen(seed):
    return torch.Generator().manual_seed(seed)


@functools.lru_cache(maxsize=None)
def _model(R, D, S, k, prec="bf16x2", layers=2):
    """a 2-layer net of the shape (biases O(1) so a dropped bias shows); the kernels run `layer` 1 of its packs"""
    import wavenet_model as wmod
    with torch.random.fork_rng(devices=[]):                 # seeded weights without touching the global RNG of other tests
        torch.manual_seed(R + 3 * D + 7 * S + k)
        m = wmod.WaveNetModel(layers=layers, blocks=1, dilation_channels=D, residual_channels=R, skip_channels=S,
                              end_channels=256, classes=256, output_length=8, kernel_size=k, bias=True)
    g = _gen(17)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith(".bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
    m = m.cuda()
    m._runtime().tc_precision = prec
    return m


def _weights(m, i):
    return BR.layer_weights({n: v.detach().cpu() for n, v in m.state_dict().items()}, i)


def _tb_model(prec, C):
    return _model(C, C, C, 2, "bf16x2" if prec == "pairs" else "bf16")


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _pair(x):
    return BR.pair_from_frames(x).cuda()


def _planes(p):
    return BR.planes_from_pair(p.cpu())


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _fg(B, L, D, seed):
    g = _gen(seed)
    return torch.cat([torch.rand(B, L, D, generator=g) * 2 - 1, torch.rand(B, L, D, generator=g)], 2)   # f in (-1,1), g in (0,1)


# ================================================================================================ fused chunked-pair kernels
FWD_CASES = [  # B, L, dilation, in_start, out_start, skip_start, skip_init
    (1, 200, 1, 0, 1, 1, 1),                 # one partial item
    (3, 1100, 128, 127, 255, 256, 0),        # tap crosses the CTA boundary; out_start one frame before an item boundary
    (1, 1100, 129, 129, 258, 511, 1),
    (3, 900, 255, 1, 256, 257, 0),
    (1, 1300, 256, 0, 256, 768, 0),          # tap = one item
    (3, 1037, 257, 256, 513, 513, 1),        # ragged tail
    (1, 1500, 512, 0, 512, 1023, 0),
    (3, 700, 127, 128, 129, 300, 1),         # out_start < in_start + d: reads the zero history
]


@pytest.mark.parametrize("prec,C", TB_PRECS)
@pytest.mark.parametrize("case", range(len(FWD_CASES)))
def test_tb_block_fwd(prec, C, case):
    import native
    lib = native.lib()
    B, L, d, in_s, out_s, sk_s, sk_init = FWD_CASES[case]
    m = _tb_model(prec, C)
    rt = m._runtime()
    tb_w, tb_b, p_id = rt.packed_weights(_stream())["tb"]
    W = _weights(m, 1)
    g = _gen(100 + case)
    h = torch.randn(B, L, C, generator=g)
    skip0 = None if sk_init else torch.randn(B, L - sk_s, C, generator=g)
    h_in, h_out = _pair(h), _nan(B, 2, C // 8, L, 8, dtype=torch.bfloat16)
    skip = _nan(B, C // 4, L - sk_s, 4) if sk_init else BR.chunks4_from_frames(skip0).cuda()
    fg = _nan(B, 2 * C // 4, L, 4)
    a = native.TbBlockArgs()
    a.d_h_in, a.d_h_out, a.d_skip, a.d_w_all, a.d_bias4 = h_in.data_ptr(), h_out.data_ptr(), skip.data_ptr(), tb_w.data_ptr(), tb_b[1].data_ptr()
    a.layer, a.n_layers, a.channels, a.precision, a.B, a.L = 1, tb_w.shape[0], C, p_id, B, L
    a.dilation, a.in_start, a.out_start, a.skip_start, a.skip_init, a.d_fg_save = d, in_s, out_s, sk_s, sk_init, fg.data_ptr()
    native.check(lib.wn_tb_block_fwd(ctypes.byref(a), _stream()), "tb block fwd")
    torch.cuda.synchronize()
    _sentinel_kept("h_out", h_out, out_s)
    _sentinel_kept("fg_save", fg, out_s)
    hp = _planes(h_in)
    got_h = BR.value(_planes(h_out))[:, out_s:]
    got_fg = BR.frames_from_chunks4(fg.cpu())[:, out_s:]
    got_sk = BR.frames_from_chunks4(skip.cpu())
    ex = BR.block_forward(hp, W, d, in_s, out_s, sk_s, skip0)
    em = BR.block_forward(hp, W, d, in_s, out_s, sk_s, skip0, mode=prec, pair_out=True)
    kind = "emu" if prec == "pairs" else "bf16"
    print(f"\nwn_tb_block_fwd {prec} {C}: B={B} L={L} d={d} in={in_s} out={out_s} skip={sk_s} init={sk_init}")
    bar = _check("h_out", got_h, ex["h_out"], em["h_out"], kind, K=2 * C)
    _check("skip", got_sk, ex["skip"], em["skip"], kind, K=2 * C)
    _check("tanh", got_fg[..., :C], ex["f"], em["f"], kind, K=2 * C)
    _check("sigmoid", got_fg[..., C:], ex["g"], em["g"], kind, K=2 * C)
    if case == 1 and prec == "pairs":
        _miss("dilation + 1", got_h, BR.block_forward(hp, W, d + 1, in_s, out_s, sk_s, skip0)["h_out"], bar)
        _miss("in_start + 1", got_h, BR.block_forward(hp, W, d, in_s + 1, out_s, sk_s, skip0)["h_out"], bar)
    if case == 1 and prec == "bf16":
        # the pairs emulation is ~exact, so the single-pass kernel misses it by about e_emu = 4x the 0.25 e_emu bar
        e_emu = _rel(em["h_out"], ex["h_out"])
        pe = BR.block_forward(hp, W, d, in_s, out_s, sk_s, skip0, mode="pairs", pair_out=True)["h_out"]
        e = _rel(got_h, pe)
        print(f"  control pairs emulation: rel_err {e:.2e} = {e / (0.25 * e_emu):.1f}x the emulation bar")
        assert e >= 2 * 0.25 * e_emu


BWD_CASES = [  # B, L, dilation, in_start, out_start, gs_out (= L: no dh_out, the last layer), ds_start
    (1, 200, 1, 0, 1, 200, 100),
    (3, 1100, 128, 127, 255, 256, 700),      # gz = 256 on an item boundary, gs_in = 128 on a CTA boundary
    (1, 1100, 129, 129, 258, 300, 512),      # gs_out > out_start, ds_start > gz
    (3, 900, 255, 1, 256, 200, 257),         # gs_out < out_start
    (1, 1300, 256, 0, 256, 1300, 767),       # no dh_out; anti-causal tap = one item
    (3, 1037, 257, 256, 513, 512, 1000),
    (1, 1500, 512, 0, 512, 1024, 1025),
    (3, 700, 127, 128, 129, 129, 385),
]


def _bwd_inputs(B, L, C, gs_out, ds_s, seed):
    g = _gen(seed)
    dh = None if gs_out >= L else torch.randn(B, L, C, generator=g)     # garbage left of gs_out: must not be read
    return dh, torch.randn(B, L - ds_s, C, generator=g), _fg(B, L, C, seed + 1)


@pytest.mark.parametrize("prec,C", TB_PRECS)
@pytest.mark.parametrize("case", range(len(BWD_CASES)))
def test_tb_block_bwd_data(prec, C, case):
    import native
    lib = native.lib()
    B, L, d, in_s, out_s, gs_out, ds_s = BWD_CASES[case]
    gz, id_s, gs_in = BR.backward_ranges(L, 2, d, in_s, out_s, gs_out, ds_s)
    m = _tb_model(prec, C)
    wb_all, p_id = m._runtime().packed_weights(_stream())["tb_bwd"]
    W = _weights(m, 1)
    dh, ds, fgf = _bwd_inputs(B, L, C, gs_out, ds_s, 200 + case)
    dh_c, ds_c, fg_c = (None if dh is None else _pair(dh)), _pair(ds), BR.chunks4_from_frames(fgf).cuda()
    dfg, z, dh_in = (_nan(B, 2, n // 8, L, 8, dtype=torch.bfloat16) for n in (2 * C, C, C))
    a = native.TbBwdArgs()
    a.d_dh_out, a.d_dskip, a.d_fg = (None if dh_c is None else dh_c.data_ptr()), ds_c.data_ptr(), fg_c.data_ptr()
    a.d_dfg, a.d_z, a.d_dh_in, a.d_wb_all = dfg.data_ptr(), z.data_ptr(), dh_in.data_ptr(), wb_all.data_ptr()
    a.layer, a.n_layers, a.channels, a.precision, a.B, a.L, a.dilation = 1, wb_all.shape[0], C, p_id, B, L, d
    a.in_start, a.out_start, a.gs_out, a.ds_start, a.gz, a.gs_in = in_s, out_s, gs_out, ds_s, gz, gs_in
    native.check(lib.wn_tb_block_bwd_data(ctypes.byref(a), _stream()), "tb block bwd")
    torch.cuda.synchronize()
    for n, t, lo in (("dFG", dfg, gz), ("z", z, gz), ("dh_in", dh_in, gs_in)):
        _sentinel_kept(n, t, lo)
    dhp = None if dh_c is None else _planes(dh_c)
    dsp = _planes(ds_c)
    args = (fgf, dhp, dsp, W, d, in_s, out_s, gs_out, ds_s)
    ex = BR.block_backward_data(*args, gz, gs_in)
    em = BR.block_backward_data(*args, gz, gs_in, mode=prec, pair_out=True)
    got = dict(dfg=BR.value(_planes(dfg))[:, gz:], z=BR.value(_planes(z))[:, gz:], dh_in=BR.value(_planes(dh_in))[:, gs_in:])
    kind = "emu" if prec == "pairs" else "bf16"
    print(f"\nwn_tb_block_bwd_data {prec} {C}: B={B} L={L} d={d} in={in_s} out={out_s} gs_out={gs_out} ds={ds_s} "
          f"gz={gz} gs_in={gs_in}")
    bars = {n: _check(n, got[n], ex[n], em[n], kind, K=4 * C) for n in ("dfg", "z", "dh_in")}
    if case == 1 and prec == "pairs":
        wrong = BR.block_backward_data(*args, gz + 1, gs_in)["dh_in"]
        _miss("gz + 1", got["dh_in"], wrong, bars["dh_in"])
        wrong = BR.block_backward_data(fgf, dhp, dsp, W, d + 1, in_s, out_s, gs_out, ds_s, gz, gs_in)["dh_in"]
        _miss("dilation + 1", got["dh_in"], wrong, bars["dh_in"])


WGRAD_CASES = BWD_CASES + [(1, 700, 512, 200, 300, 700, 400)]      # last: tap 0 range [712, 700) is empty


@pytest.mark.parametrize("prec,C", TB_PRECS)
@pytest.mark.parametrize("case", range(len(WGRAD_CASES)))
def test_tb_wgrad(prec, C, case):
    import native
    lib = native.lib()
    B, L, d, in_s, out_s, gs_out, ds_s = WGRAD_CASES[case]
    gz, id_s, _ = BR.backward_ranges(L, 2, d, in_s, out_s, gs_out, ds_s)
    m = _tb_model(prec, C)
    p_id = m._runtime().packed_weights(_stream())["tb_bwd"][1]
    dh, ds, _ = _bwd_inputs(B, L, C, gs_out, ds_s, 300 + case)
    g = _gen(400 + case)
    dfg_f, z_f, h_f = torch.randn(B, L, 2 * C, generator=g), torch.randn(B, L, C, generator=g), torch.randn(B, L, C, generator=g)
    ins = [None if dh is None else _pair(dh), _pair(ds), _pair(dfg_f), _pair(z_f), _pair(h_f)]
    outs = dict(gws=_nan(C, C, 1), gwr=_nan(C, C, 1), gwf=_nan(C, C, 2), gwg=_nan(C, C, 2))
    work = torch.empty(lib.wn_tb_wgrad_workspace_bytes() // 4, device="cuda")
    a = native.TbWgradArgs()
    a.d_dh_out = None if ins[0] is None else ins[0].data_ptr()
    a.d_dskip, a.d_dfg, a.d_z, a.d_h_in = (t.data_ptr() for t in ins[1:])
    a.d_gws, a.d_gwr, a.d_gwf, a.d_gwg = (outs[n].data_ptr() for n in ("gws", "gwr", "gwf", "gwg"))
    a.d_work, a.channels, a.precision, a.B, a.L, a.dilation = work.data_ptr(), C, p_id, B, L, d
    a.in_start, a.ds_start, a.id_start, a.gz = in_s, ds_s, id_s, gz
    native.check(lib.wn_tb_wgrad(ctypes.byref(a), _stream()), "tb wgrad")
    torch.cuda.synchronize()
    got = {n: t.cpu() for n, t in outs.items()}
    pl = [None if t is None else _planes(t) for t in ins]
    args = (pl[1], pl[0], pl[2], pl[3], pl[4], 2, d, in_s, ds_s, id_s, gz)
    ex, em = BR.block_wgrad(*args), BR.block_wgrad(*args, mode=prec)
    kind = "emu" if prec == "pairs" else "bf16"
    print(f"\nwn_tb_wgrad {prec} {C}: B={B} L={L} d={d} in={in_s} ds={ds_s} id={id_s} gz={gz}")
    _check("gws", got["gws"], ex["gws"], em["gws"], kind, K=B * L)
    if pl[0] is None or id_s >= L:
        assert float(got["gwr"].abs().max()) == 0                          # no dh_out: exact zeros
    else:
        _check("gwr", got["gwr"], ex["gwr"], em["gwr"], kind, K=B * L)
    for n in ("gwf", "gwg"):
        for j in range(2):
            if max(gz, in_s + (1 - j) * d) >= L:
                assert float(got[n][:, :, j].abs().max()) == 0, f"{n} tap {j}: empty range must give exact zeros"
                print(f"  {n} tap {j}: empty frame range, exact zeros")
            else:
                _check(f"{n} tap {j}", got[n][:, :, j], ex[n][:, :, j], em[n][:, :, j], kind, K=B * L)


# ================================================================================================ two-launch / FFMA kernels
TC_SHAPES = [(256, 256, 256, 3), (512, 256, 256, 2), (256, 256, 512, 2), (256, 128, 256, 2), (256, 384, 256, 2),
             (1024, 1024, 1024, 2)]
TC_FWD_CASES = [  # B, L, dilation, in_start, out_start, skip_start, skip_init
    (3, 700, 129, 1, 257, 300, 0),
    (1, 1100, 256, 0, 255, 767, 1),
    (3, 900, 128, 127, 255, 256, 0),         # tap crosses the 128-frame tile boundary
    (1, 1300, 512, 0, 512, 1023, 1),
]
TC_BWD_CASES = [  # B, L, dilation, in_start, out_start, gs_out (= L: no dh_out), ds_start
    (3, 700, 129, 1, 257, 300, 400),
    (1, 1100, 256, 0, 256, 1100, 767),       # no dh_out
    (3, 900, 128, 127, 255, 256, 700),       # gz = 256, gs_in = 128: both on tile boundaries
    (1, 1300, 512, 0, 512, 1024, 1025),      # gz = 1024, gs_in = 512
]


@pytest.mark.parametrize("impl", ["pairs", "ffma"])
@pytest.mark.parametrize("case", range(len(TC_FWD_CASES)))
@pytest.mark.parametrize("shape", TC_SHAPES)
def test_two_launch_and_ffma_block_fwd(shape, case, impl):
    import native
    lib = native.lib()
    R, D, S, k = shape
    B, L, d, in_s, out_s, sk_s, sk_init = TC_FWD_CASES[case]
    m = _model(R, D, S, k)
    W = _weights(m, 1)
    packs = m._runtime().packed_weights(_stream())
    g = _gen(500 + case)
    h = torch.randn(B, L, R, generator=g)
    skip0 = None if sk_init else torch.randn(B, L - sk_s, S, generator=g)
    h_in, h_out, z, fg = h.cuda(), _nan(B, L, R), _nan(B, L, D), _nan(B, L, 2 * D)
    skip = _nan(B, L - sk_s, S) if sk_init else skip0.cuda()
    if impl == "ffma":
        a = native.BlockArgs()
        wfg, bfg, wrs, brs = packs["layers"][1]
        a.d_wfg_t, a.d_bfg, a.d_wrs_t, a.d_brs, a.mode = wfg.data_ptr(), bfg.data_ptr(), wrs.data_ptr(), brs.data_ptr(), 0
    else:
        a = native.TcBlockArgs()
        wa, ba, wb, bb = packs["tc_layers"][1]
        a.d_wa, a.d_ba, a.d_wb, a.d_bb, a.d_z = wa.data_ptr(), ba.data_ptr(), wb.data_ptr(), bb.data_ptr(), z.data_ptr()
    a.d_h_in, a.d_h_out, a.d_skip, a.d_fg_save = h_in.data_ptr(), h_out.data_ptr(), skip.data_ptr(), fg.data_ptr()
    a.B, a.L, a.R, a.D, a.S, a.k = B, L, R, D, S, k
    a.dilation, a.in_start, a.out_start, a.skip_start, a.skip_init = d, in_s, out_s, sk_s, sk_init
    fn = lib.wn_block_fwd if impl == "ffma" else lib.wn_tc_block_fwd
    native.check(fn(ctypes.byref(a), _stream()), f"{impl} block fwd")
    torch.cuda.synchronize()
    _sentinel_kept("h_out", h_out, out_s)
    _sentinel_kept("fg_save", fg, out_s)
    ex = BR.block_forward(h, W, d, in_s, out_s, sk_s, skip0)
    em = None if impl == "ffma" else BR.block_forward(h, W, d, in_s, out_s, sk_s, skip0, mode=impl)
    kind = "ffma" if impl == "ffma" else "emu"
    print(f"\n{'wn_block_fwd' if impl == 'ffma' else 'wn_tc_block_fwd ' + impl} R={R} D={D} S={S} k={k}: "
          f"B={B} L={L} d={d} in={in_s} out={out_s} skip={sk_s} init={sk_init}")
    get = lambda n: None if em is None else em[n]
    KK = max(k * R, D)
    bar = _check("h_out", h_out.cpu()[:, out_s:], ex["h_out"], get("h_out"), kind, K=KK)
    _check("skip", skip.cpu(), ex["skip"], get("skip"), kind, K=KK)
    _check("tanh", fg.cpu()[:, out_s:, :D], ex["f"], get("f"), kind, K=KK)
    _check("sigmoid", fg.cpu()[:, out_s:, D:], ex["g"], get("g"), kind, K=KK)
    if impl != "ffma":
        _sentinel_kept("z", z, out_s)
        _check("z", z.cpu()[:, out_s:], ex["z"], get("z"), kind, K=KK)
    if impl == "pairs" and case == 0 and shape == TC_SHAPES[0]:
        _miss("dilation + 1", h_out.cpu()[:, out_s:], BR.block_forward(h, W, d + 1, in_s, out_s, sk_s, skip0)["h_out"], bar)
        _miss("in_start + 1", h_out.cpu()[:, out_s:], BR.block_forward(h, W, d, in_s + 1, out_s, sk_s, skip0)["h_out"], bar)
    if impl == "pairs" and case == 0 and shape == TC_SHAPES[0]:
        # operand-term controls: the same products with the weights' lo plane dropped (hi*hi + lo*hi only), and with
        # the activations' lo plane dropped (hi*hi + hi*lo only).  The bar catches both (measured on an H100: 10.8x and
        # 7.5x the bar).
        W_hi = {n: BR.split_bf16(v)[0] if n[0] == "w" else v for n, v in W.items()}
        got_h = h_out.cpu()[:, out_s:]
        h_hi = BR.split_bf16(h)[0]
        wrongs = {"weights' lo plane dropped": BR.block_forward(h, W_hi, d, in_s, out_s, sk_s, skip0, mode=impl)["h_out"],
                  "activations' lo plane dropped": (BR.block_forward(h_hi, W, d, in_s, out_s, sk_s, skip0, mode=impl)["h_out"]
                                                    + (h - h_hi)[:, out_s:].double())}
        for what, wrong in wrongs.items():
            _miss(what, got_h, wrong, bar, factor=5)


@pytest.mark.parametrize("impl", ["pairs", "ffma"])
@pytest.mark.parametrize("case", range(len(TC_BWD_CASES)))
@pytest.mark.parametrize("shape", [s for s in TC_SHAPES if s[1] % 256 == 0])
def test_two_launch_and_ffma_block_bwd_data(shape, case, impl):
    import native
    lib = native.lib()
    R, D, S, k = shape
    B, L, d, in_s, out_s, gs_out, ds_s = TC_BWD_CASES[case]
    gz, id_s, gs_in = BR.backward_ranges(L, k, d, in_s, out_s, gs_out, ds_s)
    m = _model(R, D, S, k)
    W = _weights(m, 1)
    g = _gen(700 + case)
    dh = None if gs_out >= L else torch.randn(B, L, R, generator=g)
    ds, fgf = torch.randn(B, L - ds_s, S, generator=g), _fg(B, L, D, 800 + case)
    dh_c, ds_c, fg_c = (None if dh is None else dh.cuda()), ds.cuda(), fgf.cuda()
    dfg, z, dh_in = _nan(B, L, 2 * D), _nan(B, L, D), _nan(B, L, R)
    a = native.BlockBwdArgs()
    a.d_dh_out, a.d_dskip, a.d_fg = (None if dh_c is None else dh_c.data_ptr()), ds_c.data_ptr(), fg_c.data_ptr()
    a.d_dfg, a.d_z, a.d_dh_in = dfg.data_ptr(), z.data_ptr(), dh_in.data_ptr()
    a.B, a.L, a.R, a.D, a.S, a.k, a.dilation = B, L, R, D, S, k, d
    a.in_start, a.out_start, a.gs_out, a.ds_start, a.gz, a.gs_in = in_s, out_s, gs_out, ds_s, gz, gs_in
    if impl == "ffma":
        wrs_rows, wfg_bwd = m._runtime().ffma_bwd_weights(1)
        a.d_wrs_rows, a.d_wfg_bwd = wrs_rows.data_ptr(), wfg_bwd.data_ptr()
        native.check(lib.wn_block_bwd_data(ctypes.byref(a), _stream()), "ffma block bwd")
    else:
        packs = m._runtime().packed_weights(_stream())
        wdz, wdh = packs["tc_bwd_layers"][1]
        native.check(lib.wn_tc_block_bwd_data(ctypes.byref(a), wdz.data_ptr(), wdh.data_ptr(), _stream()), f"{impl} block bwd")
    torch.cuda.synchronize()
    for n, t, lo in (("dFG", dfg, gz), ("z", z, gz), ("dh_in", dh_in, gs_in)):
        _sentinel_kept(n, t, lo)
    args = (fgf, dh, ds, W, d, in_s, out_s, gs_out, ds_s, gz, gs_in)
    ex = BR.block_backward_data(*args)
    em = None if impl == "ffma" else BR.block_backward_data(*args, mode=impl)
    kind = "ffma" if impl == "ffma" else "emu"
    print(f"\n{'wn_block_bwd_data' if impl == 'ffma' else 'wn_tc_block_bwd_data ' + impl} R={R} D={D} S={S} k={k}: "
          f"B={B} L={L} d={d} in={in_s} out={out_s} gs_out={gs_out} ds={ds_s} gz={gz} gs_in={gs_in}")
    got = dict(dfg=dfg.cpu()[:, gz:], z=z.cpu()[:, gz:], dh_in=dh_in.cpu()[:, gs_in:])
    for n in ("dfg", "z", "dh_in"):
        _check(n, got[n], ex[n], None if em is None else em[n], kind, K=max(R + S, k * 2 * D))


# ================================================================================================ whole-stack launch
@pytest.mark.parametrize("C,prec", [(256, "bf16x2"), (512, "bf16")])
def test_whole_stack_launch_layer_by_layer(C, prec):
    """wn_tb_stack_fwd through the runtime (which sizes its flag / descriptor buffers and grid): every layer's saved output
    against the block reference applied to that layer's saved input, so errors do not compound; d = 1 ... 512."""
    torch.set_num_threads(min(8, torch.get_num_threads()))
    m = _model(C, C, C, 2, prec, layers=10)
    rt = m._runtime()
    B, L, out_len = 3, 1500, 300
    idx = torch.randint(0, 256, (B, L), generator=_gen(900)).cuda()
    s = {}
    with torch.no_grad():
        rt.stack_forward(idx, out_len, index_input=True, save=s)
    assert rt.last_block_mode == "tb" and rt.last_block_launches == 1
    plan, mode = s["plan"], ("pairs" if prec == "bf16x2" else "bf16")
    kind = "emu" if mode == "pairs" else "bf16"
    dil = [dd for dd, _ in m.dilations]
    sk_ex = sk_em = None
    print(f"\nwn_tb_stack_fwd {mode} {C}: B={B} L={L}")
    for i, d in enumerate(dil):
        W = _weights(m, i)
        hp = _planes(s["h_all"][i])
        in_s, out_s = plan.in_start[i], plan.out_start[i]
        ex = BR.block_forward(hp, W, d, in_s, out_s, plan.skip_start, sk_ex)
        em = BR.block_forward(hp, W, d, in_s, out_s, plan.skip_start, sk_em, mode=mode, pair_out=True)
        sk_ex, sk_em = ex["skip"], em["skip"]
        fg = BR.frames_from_chunks4(s["fg_all"][i].cpu())[:, out_s:]
        _check(f"layer {i} (d={d}) h_out", BR.value(_planes(s["h_all"][i + 1]))[:, out_s:], ex["h_out"], em["h_out"], kind, K=2 * C)
        _check(f"layer {i} tanh", fg[..., :C], ex["f"], em["f"], kind, K=2 * C)
        _check(f"layer {i} sigmoid", fg[..., C:], ex["g"], em["g"], kind, K=2 * C)
    _check("skip (last out_len frames)", s["sk_frames"].cpu(), sk_ex[:, -out_len:], sk_em[:, -out_len:], kind, K=2 * C)
