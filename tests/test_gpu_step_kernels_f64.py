"""The entry points of a training step around the residual blocks, each alone through the C ABI, against the float64
references of tests/step_ref.py: start conv (dense, index, tensor-core pair planes), head forward and data backward,
cross-entropy and its in-place scaling, Adam, scatter-add of rows, column sums and relu_copy.

Weights are packed by the model runtime; class counts other than 256 (1 to 1 000 for the head and start conv, up to the
1 024-class cap of the loss) and sizes past every grid cap (so the grid-stride loops run) are covered.  Output buffers are
filled with a sentinel (NaN) and are one row longer than the write range: the extra row must still hold it.

Bars:
    FFMA kernels (start conv dense, head): max-relative 1e-5 per output tensor (helpers.kernel_check, kind "ffma");
    index start conv, its pair planes, scale_by, relu_copy: bit-exact;
    cross-entropy: loss within 1e-6 relative, dlogits within 1e-6 max-relative;
    Adam: m, v and the update (new - old parameter) within 1e-6 max-relative of float64 Adam, per segment;
    column sums / scatter-add: 1e-6 relative to the sum of absolute values added into each output (the sums cancel).
Every measured value is printed (-s)."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import step_ref as SR
from helpers import kernel_check as _check, kernel_miss as _miss, kernel_rel as _rel

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def _tail_kept(what, buf, n):
    """elements [n, end) of a flat view still hold the NaN sentinel"""
    assert bool(torch.isnan(buf.reshape(-1)[n:]).all()), f"{what}: wrote past its {n} elements"


def _lib():
    import native
    return native.lib()


def _check_native(rc, what):
    import native
    native.check(rc, what)


@functools.lru_cache(maxsize=None)
def _model(R, S, E, classes):
    """a one-layer net with these start / head shapes (biases O(1) so a dropped bias shows)"""
    import wavenet_model as wmod
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(R + 3 * S + 7 * E + 11 * classes)
        m = wmod.WaveNetModel(layers=1, blocks=1, dilation_channels=8, residual_channels=R, skip_channels=S,
                              end_channels=E, classes=classes, output_length=1, kernel_size=2, bias=True)
    g = _gen(17)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith(".bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
    return m.cuda()


def _packs(m):
    return m._runtime().packed_weights(_stream())


def _cpu(m, name):
    return dict(m.named_parameters())[name].detach().cpu()


# ================================================================================================ head
HEAD_CASES = [  # B, S, E, classes, L, skip_start, out_len
    (1, 5, 7, 1, 400, 10, 1),
    (3, 256, 256, 3, 600, 50, 127),
    (1, 1024, 512, 100, 700, 100, 128),
    (3, 5, 1000, 256, 800, 200, 129),           # E = 1 000: 32-frame tile
    (1, 256, 2048, 257, 900, 100, 300),         # E = 2 048: 16-frame tile
    (3, 1024, 7, 1000, 500, 20, 300),
    (1, 256, 1000, 1000, 400, 0, 129),
    (3, 5, 2048, 257, 300, 10, 128),
]


def _head_inputs(B, S, L, skip_start, out_len, seed):
    """skip (B, L - skip_start, S) with every |value| >= 0.01 (no relu(skip) tie); NaN left of the output window, which the
    head must not read"""
    g = _gen(seed)
    x = torch.randn(B, L - skip_start, S, generator=g)
    x = torch.sign(x) * (0.01 + x.abs())
    x[:, :L - skip_start - out_len] = float("nan")
    return x


def _separate_pre1_ties(m, skip, out_len, margin=1e-3):
    """shift end_conv_1's bias per channel until no input of the second head ReLU lies within `margin` of zero (float64)"""
    w1, b1 = _cpu(m, "end_conv_1.weight"), _cpu(m, "end_conv_1.bias").double()
    taps = {}
    SR.head_forward(skip, w1, b1, torch.zeros(1, w1.shape[0], 1), torch.zeros(1), out_len, taps)
    pre = taps["pre1"].reshape(-1, w1.shape[0])
    for c in range(pre.shape[1]):
        off = 0.0
        while float((pre[:, c] + off).abs().min()) < margin:
            off += 5 * margin
        b1[c] += off
    with torch.no_grad():
        m.end_conv_1.bias.copy_(b1.float())
    assert SR.head_relu_margin(skip, w1, _cpu(m, "end_conv_1.bias"), out_len) >= margin


def _head_fwd(m, skip_d, B, L, S, E, classes, skip_start, out_len):
    import native
    W = _packs(m)
    logits = _nan(B * out_len + 1, classes)
    hd = native.HeadArgs()
    hd.d_skip, hd.d_logits = skip_d.data_ptr(), logits.data_ptr()
    (w1, b1), (w2, b2) = W["end1"], W["end2"]
    hd.d_w1_t, hd.d_b1, hd.d_w2_t, hd.d_b2 = w1.data_ptr(), b1.data_ptr(), w2.data_ptr(), b2.data_ptr()
    hd.B, hd.L, hd.S, hd.E, hd.classes, hd.skip_start, hd.out_len, hd.mode = B, L, S, E, classes, skip_start, out_len, 0
    rc = _lib().wn_head_fwd(ctypes.byref(hd), _stream())
    return rc, logits


@pytest.mark.parametrize("case", range(len(HEAD_CASES)))
def test_head_fwd(case):
    B, S, E, classes, L, sk_s, OL = HEAD_CASES[case]
    m = _model(8, S, E, classes)
    skip = _head_inputs(B, S, L, sk_s, OL, 100 + case)
    rc, logits = _head_fwd(m, skip.cuda(), B, L, S, E, classes, sk_s, OL)
    _check_native(rc, "head fwd")
    torch.cuda.synchronize()
    _tail_kept("logits", logits, B * OL * classes)
    args = [_cpu(m, n) for n in ("end_conv_1.weight", "end_conv_1.bias", "end_conv_2.weight", "end_conv_2.bias")]
    ex = SR.head_forward(skip, *args, OL)
    print(f"\nwn_head_fwd B={B} S={S} E={E} classes={classes} L={L} skip_start={sk_s} out_len={OL}")
    got = logits.cpu()[:B * OL]
    bar = _check("logits", got, ex, kind="ffma")
    if case == 1:
        _miss("window one frame early", got, SR.head_forward(skip[:, :-1].nan_to_num(), *args, OL), bar)


def test_head_fwd_refuses_end_channels_past_shared_memory():
    m = _model(8, 5, 4096, 3)
    rc, _ = _head_fwd(m, torch.zeros(1, 10, 5, device="cuda"), 1, 10, 5, 4096, 3, 0, 1)
    assert rc != 0 and b"end_channels=4096" in _lib().wn_last_error_string()


@pytest.mark.parametrize("case", range(len(HEAD_CASES)))
def test_head_bwd_data(case):
    import native
    B, S, E, classes, L, sk_s, OL = HEAD_CASES[case]
    m = _model(8, S, E, classes)
    skip = _head_inputs(B, S, L, sk_s, OL, 200 + case)
    _separate_pre1_ties(m, skip, OL)
    dlogits = torch.randn(B * OL, classes, generator=_gen(300 + case))
    W = _packs(m)
    w2_rows, w1_rows = W["head_rows"]
    y1, dy1, dskip = _nan(B * OL + 1, E), _nan(B * OL + 1, E), _nan(B * OL + 1, S)
    dl_d, skip_d = dlogits.cuda(), skip.cuda()
    hb = native.HeadBwdArgs()
    hb.d_dlogits, hb.d_skip = dl_d.data_ptr(), skip_d.data_ptr()
    hb.d_y1, hb.d_dy1, hb.d_dskip = y1.data_ptr(), dy1.data_ptr(), dskip.data_ptr()
    hb.d_w1_t, hb.d_b1 = W["end1"][0].data_ptr(), W["end1"][1].data_ptr()
    hb.d_w2_rows, hb.d_w1_rows = w2_rows.data_ptr(), w1_rows.data_ptr()
    hb.B, hb.L, hb.S, hb.E, hb.classes, hb.skip_start, hb.out_len = B, L, S, E, classes, sk_s, OL
    _check_native(_lib().wn_head_bwd_data(ctypes.byref(hb), _stream()), "head bwd")
    torch.cuda.synchronize()
    for n, t, c in (("y1", y1, E), ("dy1", dy1, E), ("dskip", dskip, S)):
        _tail_kept(n, t, B * OL * c)
    w1, b1, w2 = _cpu(m, "end_conv_1.weight"), _cpu(m, "end_conv_1.bias"), _cpu(m, "end_conv_2.weight")
    ex = SR.head_backward_data(dlogits, skip, w1, b1, w2, OL)
    print(f"\nwn_head_bwd_data B={B} S={S} E={E} classes={classes} L={L} skip_start={sk_s} out_len={OL} "
          f"(relu margin {SR.head_relu_margin(skip, w1, b1, OL):.1e})")
    got = dict(y1=y1.cpu()[:B * OL].view(B, OL, E), dy1=dy1.cpu()[:B * OL].view(B, OL, E),
               dskip=dskip.cpu()[:B * OL].view(B, OL, S))
    bars = {n: _check(n, got[n], ex[n], kind="ffma") for n in ("y1", "dy1", "dskip")}
    if case == 1:
        _miss("skip mask left out", got["dskip"], ex["dy1"] @ w1[:, :, 0].double(), bars["dskip"])


# ================================================================================================ start conv
START_CASES = [  # classes, R, index dtype
    (1, 8, torch.int64),
    (11, 40, torch.uint8),
    (256, 256, torch.uint8),
    (257, 256, torch.int64),
    (1000, 64, torch.int64),
]


def _start_call(fn_name, idx_d, W, out, B, classes, L, R, err=None):
    lib = _lib()
    ws_t, bs_p = W["start"]
    args = [idx_d.data_ptr(), ws_t.data_ptr(), bs_p.data_ptr(), out.data_ptr(), B, classes, L, R]
    if fn_name.startswith("wn_tb"):
        args.append(None if err is None else err.data_ptr())
    _check_native(getattr(lib, fn_name)(*args, _stream()), fn_name)


@pytest.mark.parametrize("case", range(len(START_CASES)))
def test_start_conv(case):
    from block_ref import planes_from_pair
    classes, R, dt = START_CASES[case]
    m = _model(R, 8, 8, classes)
    W = _packs(m)
    w, b = _cpu(m, "start_conv.weight"), _cpu(m, "start_conv.bias")
    sfx = "u8" if dt == torch.uint8 else "i64"
    B, L = 3, 1_000_000 // R + 131                  # past the grid caps of both index kernels
    g = _gen(400 + case)
    idx = torch.randint(0, classes, (B, L), generator=g).to(dt)
    idx[0, 0], idx[-1, -1] = 0, classes - 1
    print(f"\nstart conv classes={classes} R={R} {sfx}: B={B} L={L}")
    # index form: bit-equal to the fp32 sum w[c] + b
    want = SR.start_index_fp32(idx, w, b)
    h = _nan(B * L + 1, R)
    _start_call(f"wn_start_fwd_index_{sfx}", idx.cuda(), W, h, B, classes, L, R)
    torch.cuda.synchronize()
    _tail_kept("h (index)", h, B * L * R)
    got = h.cpu()[:B * L].view(B, L, R)
    assert torch.equal(got, want), f"index form: {int((got != want).sum())} elements differ from w[c] + b"
    assert not torch.equal(got, SR.start_index_fp32((idx.long() + 1) % classes, w, b)) or classes == 1
    print("  index form: bit-equal to w[c] + b")
    # tensor-core pair planes: bit-equal to split_bf16(w[c] + b)
    pair = _nan(B, 2, R // 8, L, 8, dtype=torch.bfloat16)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    _start_call(f"wn_tb_start_index_{sfx}", idx.cuda(), W, pair, B, classes, L, R, err)
    torch.cuda.synchronize()
    hi, lo = planes_from_pair(pair.cpu())
    whi, wlo = SR.start_pair_planes(idx, w, b)
    assert torch.equal(hi, whi) and torch.equal(lo, wlo) and int(err) == 0
    print("  tb pair planes: bit-equal to split(w[c] + b), no error flag")
    # dense: one-hot bit-equal to the index form; non-one-hot within the FFMA bar (L small: no grid cap here)
    Ld = 300
    oh = torch.zeros(B, classes, Ld).scatter_(1, idx[:, :Ld].long().view(B, 1, Ld), 1.0)
    hd = _nan(B * Ld + 1, R)
    _start_call("wn_start_fwd_dense", oh.cuda(), W, hd, B, classes, Ld, R)
    torch.cuda.synchronize()
    _tail_kept("h (dense)", hd, B * Ld * R)
    assert torch.equal(hd.cpu()[:B * Ld].view(B, Ld, R), want[:, :Ld]), "dense one-hot differs from the index form"
    print("  dense one-hot: bit-equal to the index form")
    x = torch.randn(B, classes, Ld, generator=g)
    _start_call("wn_start_fwd_dense", x.cuda(), W, hd, B, classes, Ld, R)
    torch.cuda.synchronize()
    got_d = hd.cpu()[:B * Ld].view(B, Ld, R)
    bar = _check("dense (randn input)", got_d, SR.start_dense(x, w, b), kind="ffma")
    _miss("bias left out", got_d, SR.start_dense(x, w, None), bar)


@pytest.mark.parametrize("classes,dt,bad", [(11, torch.uint8, 255), (256, torch.int64, -1), (257, torch.int64, 257),
                                            (1000, torch.int64, 1 << 40)])
def test_start_conv_out_of_range_index_clamps_and_flags(classes, dt, bad):
    from block_ref import planes_from_pair
    R = 64
    m = _model(R, 8, 8, classes)
    W = _packs(m)
    w, b = _cpu(m, "start_conv.weight"), _cpu(m, "start_conv.bias")
    sfx = "u8" if dt == torch.uint8 else "i64"
    B, L = 2, 50
    idx = torch.randint(0, classes, (B, L), generator=_gen(classes)).to(dt)
    idx[1, 7] = bad
    want = SR.start_index_fp32(idx, w, b)                           # clamped
    h = _nan(B * L, R)
    _start_call(f"wn_start_fwd_index_{sfx}", idx.cuda(), W, h, B, classes, L, R)
    pair = _nan(B, 2, R // 8, L, 8, dtype=torch.bfloat16)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    _start_call(f"wn_tb_start_index_{sfx}", idx.cuda(), W, pair, B, classes, L, R, err)
    torch.cuda.synchronize()
    assert torch.equal(h.cpu().view(B, L, R), want)
    hi, lo = planes_from_pair(pair.cpu())
    assert torch.equal(hi, SR.start_pair_planes(idx, w, b)[0]) and torch.equal(lo, SR.start_pair_planes(idx, w, b)[1])
    assert int(err) == 1, "an index outside [0, classes) must set the error flag"
    print(f"\nstart conv classes={classes} index {bad}: clamped to {min(max(bad, 0), classes - 1)}, flag set")


# ================================================================================================ cross-entropy
CE_CASES = [  # N, C, logits: "randn" (3 randn), "pm80" (+-80 + randn), "off1e4" (1e4 + 3 randn)
    (1, 1, "randn"),
    (9471, 31, "randn"),
    (9472, 33, "randn"),
    (9473, 256, "randn"),
    (20011, 1000, "randn"),
    (9473, 1024, "randn"),
    (4000, 256, "pm80"),
    (1, 256, "off1e4"),
    (3, 256, "off1e4"),
    (1, 1024, "off1e4"),
]


def _ce(x, t, err=None):
    lib = _lib()
    N, C = x.shape
    xd, td = x.cuda(), t.cuda()
    d = _nan(N * C + 4)
    loss = _nan(1)
    work = torch.empty(lib.wn_ce_workspace_bytes() // 4, device="cuda")
    rc = lib.wn_ce_fwd_bwd(xd.data_ptr(), td.data_ptr(), d.data_ptr(), loss.data_ptr(), work.data_ptr(),
                           None if err is None else err.data_ptr(), N, C, _stream())
    torch.cuda.synchronize()
    return rc, float(loss.cpu()), d


def _ce_inputs(N, C, kind, seed):
    g = _gen(seed)
    x = torch.randn(N, C, generator=g)
    if kind == "randn":
        x = 3 * x
    elif kind == "pm80":
        x = 80 * torch.sign(torch.randn(N, C, generator=g)) + x
    else:
        x = 1e4 + 3 * x
    t = torch.randint(0, C, (N,), generator=g)
    t[0], t[-1] = C - 1, 0
    return x.float(), t


@pytest.mark.parametrize("case", range(len(CE_CASES)))
def test_cross_entropy(case):
    N, C, kind = CE_CASES[case]
    x, t = _ce_inputs(N, C, kind, 500 + case)
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    rc, loss, d = _ce(x, t, err)
    _check_native(rc, "cross entropy")
    _tail_kept("dlogits", d, N * C)
    ref_loss, ref_d = SR.cross_entropy(x, t)
    e_loss = abs(loss - float(ref_loss)) / max(abs(float(ref_loss)), 1e-300) if ref_loss != 0 else abs(loss)
    got_d = d.cpu()[:N * C].view(N, C)
    e_d = _rel(got_d, ref_d)
    print(f"\nwn_ce_fwd_bwd N={N} C={C} {kind}: loss {loss:.7g} rel_err {e_loss:.2e} bar 1.0e-06; dlogits rel_err {e_d:.2e} "
          f"bar 1.0e-06")
    assert int(err) == 0
    assert e_loss <= 1e-6, f"loss {loss!r} vs {float(ref_loss)!r}: {e_loss:.3e}"
    assert e_d <= 1e-6
    if case == 2:
        wrong_loss, wrong_d = SR.cross_entropy(x, (t + 1) % C)
        e = abs(loss - float(wrong_loss)) / abs(float(ref_loss))
        print(f"  control targets + 1: loss {e:.2e} = {e / 1e-6:.1f}x bar")
        assert e >= 10 * 1e-6
        _miss("targets + 1 (dlogits)", got_d, wrong_d, 1e-6)


def test_cross_entropy_bad_target_and_class_cap():
    x, t = _ce_inputs(50, 33, "randn", 600)
    t[5], t[9] = -1, 33
    err = torch.zeros(1, dtype=torch.int32, device="cuda")
    rc, loss, d = _ce(x, t, err)
    _check_native(rc, "cross entropy")
    ref_loss, ref_d = SR.cross_entropy(x, t)                         # clamped targets
    assert int(err) == 1
    assert abs(loss - float(ref_loss)) <= 1e-6 * abs(float(ref_loss)) and _rel(d.cpu()[:50 * 33].view(50, 33), ref_d) <= 1e-6
    x2, t2 = _ce_inputs(4, 1025, "randn", 601)
    rc, _, _ = _ce(x2, t2)
    assert rc != 0 and b"classes <= 1024" in _lib().wn_last_error_string()
    print("\nwn_ce_fwd_bwd: targets -1 and C clamp and set the flag; 1 025 classes refused")


@pytest.mark.parametrize("scale", [1.0, 2.5, -0.3])
def test_scale_by(scale):
    lib = _lib()
    n = 1184 * 256 * 4 * 2 + 8                  # past the grid cap
    x = torch.randn(n + 4, generator=_gen(700))
    x[n:] = float("nan")
    xd, s = x.cuda(), torch.tensor([scale], device="cuda")
    _check_native(lib.wn_scale_by(xd.data_ptr(), n, s.data_ptr(), _stream()), "scale_by")
    torch.cuda.synchronize()
    got = xd.cpu()
    want = x[:n] * torch.tensor(scale, dtype=torch.float32)
    assert torch.equal(got[:n], want) and bool(torch.isnan(got[n:]).all())
    assert lib.wn_scale_by(xd.data_ptr(), 6, s.data_ptr(), _stream()) != 0
    print(f"\nwn_scale_by {scale}: bit-exact" + (" (no-op)" if scale == 1.0 else ""))


# ================================================================================================ Adam
def _adam_table(sizes):
    chunks = []
    for i, n in enumerate(sizes):
        chunks += [(i, c) for c in range((n + 4095) // 4096)]
    return chunks


def _run_adam(tensors, step, hyper, f64=True):
    """tensors: list of (p, g, m, v) CUDA fp32; one launch over all of them"""
    lib = _lib()
    segs = np.array([(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel()) for p, g, m, v in tensors],
                    dtype=np.int64)
    chunks = _adam_table([p.numel() for p, _, _, _ in tensors])
    sd, cd = torch.from_numpy(segs).cuda(), torch.tensor(chunks, dtype=torch.int32, device="cuda")
    fn = lib.wn_adam_step_f64 if f64 else lib.wn_adam_step
    _check_native(fn(sd.data_ptr(), cd.data_ptr(), len(chunks), hyper["lr"], hyper["betas"][0], hyper["betas"][1], hyper["eps"],
                     hyper["weight_decay"], step, _stream()), "adam")
    torch.cuda.synchronize()


SIZES = [4096, 4095, 4097, 1, 3 * 4096 + 5, 777]
GSCALES = [1.0, 1e-3, 1e-6, 1e-9]          # 1e-9: eps dominates the denominator


def _adam_inputs(sizes, step, seed):
    g = _gen(seed)
    out = []
    for i, n in enumerate(sizes):
        gs = GSCALES[i % len(GSCALES)]
        p = torch.randn(n, generator=g) * 1e-7                       # much smaller than lr: the update is resolved
        gr = torch.randn(n, generator=g) * gs
        if step == 1:
            m, v = torch.zeros(n), torch.zeros(n)
        else:
            m = torch.randn(n, generator=g) * gs
            v = (torch.randn(n, generator=g) * gs) ** 2
        out.append((p, gr, m, v))
    return out


@pytest.mark.parametrize("wd", [0.0, 0.5])
@pytest.mark.parametrize("step", [1, 2, 10, 1000])
@pytest.mark.parametrize("layout", ["chunk_edges", "many_segments"])
def test_adam_step(layout, step, wd):
    sizes = SIZES if layout == "chunk_edges" else [int(n) for n in torch.randint(1, 300, (300,), generator=_gen(800))]
    hyper = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=wd)
    host = _adam_inputs(sizes, step, 900 + step)
    dev = [tuple(t.cuda() for t in q) for q in host]
    _run_adam(dev, step, hyper)
    errs = dict(m=0.0, v=0.0, update=0.0)
    for (p, gr, m, v), (pd, _, md, vd) in zip(host, dev):
        rp, rm, rv = SR.adam_update(p, gr, m, v, step, **hyper)
        errs["m"] = max(errs["m"], _rel(md.cpu(), rm))
        errs["v"] = max(errs["v"], _rel(vd.cpu(), rv))
        errs["update"] = max(errs["update"], _rel(pd.cpu().double() - p.double(), rp - p.double()))
    print(f"\nwn_adam_step_f64 {layout} ({len(sizes)} segments) step={step} wd={wd}: "
          + ", ".join(f"{n} rel_err {e:.2e}" for n, e in errs.items()) + " bar 1.0e-06 (worst segment)")
    for n, e in errs.items():
        assert e <= 1e-6, f"{n}: {e:.3e}"
    if layout == "chunk_edges" and wd == 0.0 and step in (1, 2):
        # controls: eps inside the square root (on the eps-dominated segment), and the float-coefficient entry point
        p, gr, m, v = host[3]
        g2 = gr.double()
        mm = m.double() + 0.1 * (g2 - m.double())
        vv = 0.999 * v.double() + 1e-3 * g2 * g2
        wrong = -1e-3 / (1 - 0.9 ** step) * mm / ((vv / (1 - 0.999 ** step) + 1e-8).sqrt())
        _miss("eps inside the square root", dev[3][0].cpu().double() - p.double(), wrong, 1e-6)
        dev2 = [tuple(t.cuda() for t in q) for q in host]
        _run_adam(dev2, step, hyper, f64=False)
        e_v = max(_rel(vd.cpu(), SR.adam_update(p, gr, m, v, step, **hyper)[2]) for (p, gr, m, v), (_, _, _, vd) in zip(host, dev2))
        e_u = max(_rel(pd.cpu().double() - p.double(), SR.adam_update(p, gr, m, v, step, **hyper)[0] - p.double())
                  for (p, gr, m, v), (pd, _, _, _) in zip(host, dev2))
        print(f"  float-coefficient entry point wn_adam_step: v rel_err {e_v:.2e}, update rel_err {e_u:.2e}")
        if step == 1:
            assert e_v >= 10 * 1e-6, "1 - 0.999f should put v 1.3e-5 away from float64 Adam"


def test_fused_adam_per_parameter_steps_and_precision():
    """FusedAdam against float64 Adam with a step count per parameter: parameter 1 has no gradient on steps 1, 2 and 5.
    Each step is compared from the same fp32 state (errors do not compound): m, v and the update within 1e-6."""
    import wavenet_training as wt
    g = _gen(1000)
    sizes = [(300, 7), (4097,), (5,)]
    params = [torch.nn.Parameter((torch.randn(s, generator=g) * 1e-7).cuda()) for s in sizes]
    hyper = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    opt = wt.FusedAdam(params, **hyper)
    steps = [0] * len(params)
    worst = dict(m=0.0, v=0.0, update=0.0)
    for it in range(6):
        grads = [torch.randn(s, generator=g) * 10.0 ** -(3 * i) for i, s in enumerate(sizes)]
        if it in (0, 1, 4):
            grads[1] = None
        before = []
        for i, (p, gr) in enumerate(zip(params, grads)):
            st = opt.state[p]
            before.append((p.detach().cpu().clone(), st["exp_avg"].cpu().clone() if "exp_avg" in st else torch.zeros(p.shape),
                           st["exp_avg_sq"].cpu().clone() if "exp_avg_sq" in st else torch.zeros(p.shape)))
            p.grad = None if gr is None else gr.cuda()
        opt.step()
        for i, (p, gr) in enumerate(zip(params, grads)):
            if gr is None:
                assert torch.equal(p.detach().cpu(), before[i][0])
                continue
            steps[i] += 1
            st = opt.state[p]
            assert int(st["step"]) == steps[i]
            p0, m0, v0 = before[i]
            rp, rm, rv = SR.adam_update(p0, gr, m0, v0, steps[i], **hyper)
            worst["m"] = max(worst["m"], _rel(st["exp_avg"].cpu(), rm))
            worst["v"] = max(worst["v"], _rel(st["exp_avg_sq"].cpu(), rv))
            worst["update"] = max(worst["update"], _rel(p.detach().cpu().double() - p0.double(), rp - p0.double()))
    print("\nFusedAdam, per-parameter steps " + str(steps) + ": "
          + ", ".join(f"{n} rel_err {e:.2e}" for n, e in worst.items()) + " bar 1.0e-06")
    assert steps == [6, 3, 6]
    for n, e in worst.items():
        assert e <= 1e-6, f"{n}: {e:.3e}"


# ================================================================================================ reductions
@pytest.mark.parametrize("rows", [0, 1, 255, 256, 257, 511, 4097])
@pytest.mark.parametrize("C,ld", [(1, 4), (7, 9), (300, 300), (256, 260)])
def test_colsum(rows, C, ld):
    lib = _lib()
    g = _gen(rows + C)
    x = torch.randn(max(rows, 1), ld, generator=g)
    x[:, C:] = float("nan")                                           # columns past C must not be read
    xd = x.cuda()
    out = _nan(C + 4)
    work = torch.empty(max(lib.wn_colsum_workspace_bytes(rows, C) // 4, 1), device="cuda")
    _check_native(lib.wn_colsum(xd.data_ptr(), out.data_ptr(), work.data_ptr(), rows, C, ld, _stream()), "colsum")
    torch.cuda.synchronize()
    _tail_kept("colsum", out, C)
    got = out.cpu()[:C].double()
    if rows == 0:
        assert bool((got == 0).all())
        print(f"\nwn_colsum rows=0 C={C}: zeros")
        return
    s, a = SR.colsum(x, rows, C)
    e = float(((got - s).abs() / a).max())
    print(f"\nwn_colsum rows={rows} C={C} ld={ld}: rel_err (to sum |x|) {e:.2e} bar 1.0e-06")
    assert e <= 1e-6
    if rows == 4097 and C == 300:
        s_wrong, _ = SR.colsum(x, rows - 1, C)
        ew = float(((got - s_wrong).abs() / a).max())
        print(f"  control rows - 1: {ew:.2e} = {ew / 1e-6:.1f}x bar")
        assert ew >= 10 * 1e-6


@pytest.mark.parametrize("classes,R,dt,t_begin", [(11, 5, torch.uint8, 1), (256, 256, torch.uint8, 700),
                                                  (257, 40, torch.int64, 3), (1000, 256, torch.int64, 1999)])
def test_scatter_rows(classes, R, dt, t_begin):
    lib = _lib()
    B, L = 3, 2000
    g = _gen(classes + R)
    idx = torch.randint(0, classes, (B, L), generator=g)
    idx[:, t_begin::7] = idx[0, t_begin]                              # one class repeated many times
    idx[1, -1] = 255 if dt == torch.uint8 and classes < 256 else (-1 if dt == torch.int64 else 0)   # clamps
    idx = idx.to(dt)
    dh = torch.randn(B, L, R, generator=g)
    dh[:, :t_begin] = float("nan")                                    # frames left of t_begin must not be read
    table, out_t = _nan(classes * R + 4), _nan(classes * R + 4)
    idx_d, dh_d = idx.cuda(), dh.cuda()
    _check_native(lib.wn_scatter_rows(idx_d.data_ptr(), int(dt == torch.uint8), dh_d.data_ptr(), table.data_ptr(),
                                      out_t.data_ptr(), B, L, R, classes, t_begin, _stream()), "scatter rows")
    torch.cuda.synchronize()
    _tail_kept("table", table, classes * R)
    _tail_kept("transposed", out_t, classes * R)
    got = table.cpu()[:classes * R].view(classes, R)
    assert torch.equal(out_t.cpu()[:classes * R].view(R, classes), got.T)
    ref, mag = SR.scatter_rows(idx, dh, classes, t_begin)
    hit = mag > 0
    assert bool((got[~hit] == 0).all()), "rows that no frame routes to must be zero"
    e = float(((got.double() - ref).abs()[hit] / mag[hit]).max())
    print(f"\nwn_scatter_rows classes={classes} R={R} {dt} t_begin={t_begin}: rel_err (to routed sum |dh|) {e:.2e} "
          f"bar 1.0e-06; transposed copy bit-equal")
    assert e <= 1e-6
    if classes == 257:
        dh2 = dh.clone()
        dh2[:, t_begin - 1] = 1.0
        wrong, _ = SR.scatter_rows(idx, dh2, classes, t_begin - 1)
        ew = float(((got.double() - wrong).abs()[hit] / mag[hit]).max())
        print(f"  control t_begin - 1: {ew:.2e} = {ew / 1e-6:.1f}x bar")
        assert ew >= 10 * 1e-6


def test_relu_copy():
    lib = _lib()
    n = 1184 * 256 * 4 * 3 + 12                 # past the grid cap
    x = torch.randn(n + 4, generator=_gen(1100))
    xd, y = x.cuda(), _nan(n + 4)
    _check_native(lib.wn_relu_copy(xd.data_ptr(), y.data_ptr(), n, _stream()), "relu_copy")
    torch.cuda.synchronize()
    got = y.cpu()
    assert torch.equal(got[:n], torch.relu(x[:n])) and bool(torch.isnan(got[n:]).all())
    assert lib.wn_relu_copy(xd.data_ptr(), y.data_ptr(), 6, _stream()) != 0
    print("\nwn_relu_copy: bit-exact")
