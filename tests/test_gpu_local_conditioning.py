"""Local conditioning (WaveNetModel(local_condition_channels=C, local_condition_hop=hop)) on the GPU, against the float64
reference of tests/local_ref.py (pinned against the oracle on the CPU by test_local_conditioning_host.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import local_ref
from oracle import wavenet_oracle as O
from helpers import assert_stream_parity, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _kw(ch, layers, blocks, out_len, bias=True, end=256):
    return dict(layers=layers, blocks=blocks, dilation_channels=ch, residual_channels=ch, skip_channels=ch,
                end_channels=end, classes=256, output_length=out_len, kernel_size=2, bias=bias)


def _model(kw, seed, C=0, hop=None, G=0, scale=None):
    import wavenet_model as wmod
    torch.manual_seed(seed)
    m = wmod.WaveNetModel(**kw, condition_channels=G, local_condition_channels=C, local_condition_hop=hop)
    if scale is not None:
        with torch.no_grad():                              # conditioning terms of the size of the biases
            for k, v in m.named_parameters():
                if "_local_convs." in k or "_cond_convs." in k:
                    v.normal_(0, scale)
    return m


def _run(m, idx, tgt, mode, prec, stack=True, **cond):
    m.cuda()
    rt = m._runtime()
    rt.block_mode, rt.tc_precision, rt.stack_launch = mode, prec, stack
    for p in m.parameters():
        p.grad = None
    y = m.forward_indices(idx, **cond)
    F.cross_entropy(y, tgt).backward()
    assert rt.last_block_mode == ("tb" if mode == "auto" else "ffma")
    return y.detach(), {k: p.grad.clone() for k, p in m.named_parameters()}


def _assert_shared_identical(a, b):
    assert torch.equal(a[0], b[0])
    for k, g in a[1].items():
        if k not in b[1]:
            continue
        if k == "start_conv.weight":        # a scatter-add over the input indices with atomics: not bit-reproducible run to run
            assert rel_err(b[1][k].cpu().numpy(), g.cpu().numpy()) < 1e-6
            continue
        assert torch.equal(g, b[1][k]), k


CASES = [(256, "bf16x2", "auto"), (256, "bf16", "auto"), (512, "bf16", "auto"), (64, "bf16x2", "ffma")]


# ---------------------------------------------------------------------------------------------- 1. zero local conditioning
@pytest.mark.parametrize("ch,prec,mode", CASES)
def test_zero_local_condition_is_identity_in_training(ch, prec, mode):
    kw = _kw(ch, 3, 2, 100)
    idx = torch.randint(0, 256, (3, 600), generator=torch.Generator().manual_seed(1)).cuda()
    tgt = torch.randint(0, 256, (300,), generator=torch.Generator().manual_seed(2)).cuda()
    y = torch.randn(3, 4, 600 // 7 + 1, generator=torch.Generator().manual_seed(3)).cuda()
    for G in (0, 5):
        m0 = _model(kw, 3, G=G)
        m1 = _model(kw, 3, C=4, hop=7, G=G)
        with torch.no_grad():
            for k, v in m1.named_parameters():
                if "_local_convs." in k:
                    v.zero_()
        cond = dict(condition=[4, 0, 2]) if G else {}
        a = _run(m0, idx, tgt, mode, prec, **cond)
        b = _run(m1, idx, tgt, mode, prec, local_condition=y, **cond)
        _assert_shared_identical(a, b)


# ---------------------------------------------------------------------------------------------- 2. frames kernels, one frame
@pytest.mark.parametrize("ch,prec,mode,stack", [c + (True,) for c in CASES] + [(256, "bf16x2", "auto", False)])
def test_one_frame_equals_the_global_kernels(ch, prec, mode, stack):
    """hop >= L: one frame, and the frames table (0 + U y) + b has the global table's V h + b bit for bit (the same
    sequential fp32 sum), so a local-only net with U = V is the global-only net with h = y[:, :, 0]."""
    kw = _kw(ch, 3, 2, 100)
    L = 600
    idx = torch.randint(0, 256, (3, L), generator=torch.Generator().manual_seed(1)).cuda()
    tgt = torch.randint(0, 256, (300,), generator=torch.Generator().manual_seed(2)).cuda()
    y = torch.randn(3, 4, 1, generator=torch.Generator().manual_seed(3)).cuda()
    mg = _model(kw, 5, G=4, scale=0.3)
    ml = _model(kw, 5, C=4, hop=L + 5)
    sd = dict(mg.state_dict())
    ml.load_state_dict({k.replace("_cond_convs.", "_local_convs."): v for k, v in sd.items()})
    a = _run(mg, idx, tgt, mode, prec, stack, condition=y[:, :, 0])
    b = _run(ml, idx, tgt, mode, prec, stack, local_condition=y)
    _assert_shared_identical(a, b)
    for k, g in a[1].items():
        if "_cond_convs." in k:
            assert rel_err(b[1][k.replace("_cond_convs.", "_local_convs.")].cpu().numpy(), g.cpu().numpy()) < 1e-6, k


# ---------------------------------------------------------------------------------------------- 3. training parity
def _untie(m, spec, idx, y, hop, h, out_len, margin):
    """helpers.separate_head_relu_ties on the conditioned reference: nudge the last skip bias and the end_conv_1 bias (per
    channel, float64) until no head ReLU input lies within `margin` of zero."""
    step = 5 * margin
    p = {k: v.detach().clone().double() for k, v in m.state_dict().items()}
    last = spec.layers * spec.blocks - 1
    taps = {}
    local_ref.stack_direct(p, spec, O.one_hot(idx, 256).double(), y, hop, h, taps)
    sk = taps["skip"][..., -out_len:].clone()
    for name, pre_of in ((f"skip_convs.{last}.bias", lambda: sk),
                         ("end_conv_1.bias", lambda: F.conv1d(torch.relu(sk), p["end_conv_1.weight"], p["end_conv_1.bias"]))):
        pre = pre_of()
        for c in range(pre.shape[1]):
            v, off = pre[:, c, :], 0.0
            while float((v + off).abs().min()) < margin:
                off += step
            p[name][c] += off
            pre[:, c, :] += off
    m.load_state_dict({k: v.float() for k, v in p.items()}, strict=True)


@pytest.mark.parametrize("ch,prec,mode,stack,hop,G", [
    (256, "bf16x2", "auto", True, 1, 0), (256, "bf16x2", "auto", True, 5, 3), (256, "bf16x2", "auto", True, 128, 0),
    (256, "bf16x2", "auto", True, 200, 3), (256, "bf16x2", "auto", True, 800, 0),
    (256, "bf16x2", "auto", False, 5, 3), (256, "bf16x2", "auto", False, 128, 0),
    (64, "bf16x2", "ffma", True, 1, 0), (64, "bf16x2", "ffma", True, 5, 3), (64, "bf16x2", "ffma", True, 200, 0),
    (256, "bf16", "auto", True, 5, 0), (512, "bf16", "auto", True, 128, 3), (512, "bf16", "auto", False, 200, 0)])
def test_local_training_matches_reference(ch, prec, mode, stack, hop, G):
    _parity(ch, prec, mode, stack, hop, G, 2, 700)


def test_odd_shapes_on_the_ffma_blocks():
    """D, B and the frame count all odd: the per-layer table slices the FFMA blocks read are only 4-byte aligned."""
    _parity(63, "bf16x2", "ffma", True, 7, 3, 3, 701)


def _parity(ch, prec, mode, stack, hop, G, B, L):
    out_len, C = 200, 4
    kw = _kw(ch, 3, 2, out_len)
    spec = O.NetSpec(**kw)
    m = _model(kw, 13, C=C, hop=hop, G=G, scale=0.3)
    rng = np.random.RandomState(5)
    y = torch.tensor(rng.randn(B, C, -(-L // hop) + 2).astype(np.float32))
    h = torch.tensor(rng.randn(B, G).astype(np.float32)) if G else None
    idx = torch.randint(0, 256, (B, L), generator=torch.Generator().manual_seed(8))
    tgt = torch.randint(0, 256, (B * out_len,), generator=torch.Generator().manual_seed(9))
    pair = prec == "bf16x2"
    _untie(m, spec, idx, y.double(), hop, None if h is None else h.double(), out_len, 2e-5 if pair else 2e-3)
    p = {k: v.detach().clone().double().requires_grad_(True) for k, v in m.state_dict().items()}
    yd = y.double().requires_grad_(True)
    want = local_ref.forward(p, spec, O.one_hot(idx, 256).double(), yd, hop, None if h is None else h.double())
    F.cross_entropy(want, tgt).backward()
    m = m.cuda()
    rt = m._runtime()
    rt.block_mode, rt.tc_precision, rt.stack_launch = mode, prec, stack
    yg = y.cuda().requires_grad_(True)
    cond = dict(condition=h) if G else {}
    out = m.forward_indices(idx.cuda(), local_condition=yg, **cond)
    assert rt.last_block_mode == ("tb" if mode == "auto" else "ffma")
    F.cross_entropy(out, tgt.cuda()).backward()
    e = rel_err(out.detach().cpu().numpy(), want.detach().numpy())
    errs = {k: rel_err(v.grad.cpu().numpy(), p[k].grad.numpy()) for k, v in m.named_parameters()
            if p[k].grad is not None and float(p[k].grad.abs().max()) > 0}
    errs["local_condition"] = rel_err(yg.grad.cpu().numpy(), yd.grad.numpy())
    assert any("_local_convs." in k for k in errs) and (not G or any("_cond_convs." in k for k in errs))
    worst = max(errs.values())
    print(f"local {ch} ch {prec} {mode} stack={stack} hop={hop} G={G} B={B} L={L}: logits {e:.2e}, worst gradient {worst:.2e} "
          f"(dy {errs['local_condition']:.2e})")
    if pair:
        assert e < TOL and worst < TOL, (e, sorted(errs.items(), key=lambda kv: -kv[1])[:5])
    else:
        assert e < 3e-2 and worst < 6e-2, (e, worst)


def test_local_condition_errors_on_gpu():
    m = _model(_kw(64, 2, 1, 10), 0, C=3, hop=10).cuda()
    idx = torch.randint(0, 256, (2, 100)).cuda()
    with pytest.raises(ValueError):
        m.forward_indices(idx)
    with pytest.raises(ValueError):
        m.forward_indices(idx, local_condition=torch.zeros(2, 3, 9, device="cuda"))
    m._runtime().block_mode = "tc"
    with pytest.raises(RuntimeError):
        m.forward_indices(idx, local_condition=torch.zeros(2, 3, 10, device="cuda"))


# ---------------------------------------------------------------------------------------------- 5. segment sums
@pytest.mark.parametrize("pair", [0, 1])
def test_segment_sums(pair):
    import native
    lib = native.lib()
    B, L, C = 3, 1000, 64
    g = torch.Generator().manual_seed(3)
    vals = torch.randn(B, L, C, generator=g)
    if pair:
        hi = vals.to(torch.bfloat16)
        lo = (vals - hi.float()).to(torch.bfloat16)
        exact = hi.double() + lo.double()
        src = torch.stack([hi, lo], 1).view(B, 2, L, C // 8, 8).permute(0, 1, 3, 2, 4).contiguous().cuda()
    else:
        exact = vals.double()
        src = vals.cuda()
    stream = torch.cuda.current_stream().cuda_stream
    for gz, hop in ((37, 1), (333, 50), (0, 7), (400, L - 400 + 3), (990, 128)):
        nf = -(-L // hop) + 1
        out = torch.full((B, nf, C), float("nan"), device="cuda")
        native.check(lib.wn_cond_segment_sums(src.data_ptr(), pair, B, L, C, gz, hop, nf, out.data_ptr(), stream), "segment sums")
        out2 = torch.full_like(out, float("nan"))
        native.check(lib.wn_cond_segment_sums(src.data_ptr(), pair, B, L, C, gz, hop, nf, out2.data_ptr(), stream), "segment sums")
        assert torch.equal(out, out2)
        want = torch.zeros(B, nf, C, dtype=torch.float64)
        for f in range(nf):
            lo_, hi_ = max(gz, f * hop), min(L, (f + 1) * hop)
            if hi_ > lo_:
                want[:, f] = exact[:, lo_:hi_].sum(1)
            else:
                assert torch.equal(out[:, f].cpu(), torch.zeros(B, C)), (gz, hop, f)
        err = float((out.cpu().double() - want).abs().max())
        assert err < 1e-5 * max(1.0, float(want.abs().max())), (gz, hop, err)


# ---------------------------------------------------------------------------------------------- 6. sampler
def _sampler_setup(seed=7, hop=3, G=0, NS=3):
    kw = _kw(256, 3, 1, 16)
    spec = O.NetSpec(**kw)
    m = _model(kw, seed, C=4, hop=hop, G=G, scale=0.3).cuda()
    n_given, n = 12, 30
    rng = np.random.RandomState(seed)
    first = rng.randint(0, 256, (NS, n_given))
    forced = rng.randint(0, 256, (NS, n))
    y = rng.randn(NS, 4, -(-(n_given - 1 + n) // hop)).astype(np.float32)
    h = rng.randn(NS, G).astype(np.float32) if G else None
    return m, spec, first, forced, y, h, n


def _ref_logits(m, spec, first, forced, y, hop, h, n):
    """Teacher-forced logits from the float64 reference: the output at position n_given - 1 + i predicts sample i."""
    p = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    seq = np.concatenate([first, forced[:, :-1]], 1)
    x = O.one_hot(torch.tensor(seq), 256).double()
    out = local_ref.stack_direct(p, spec, x, torch.tensor(y).double(), hop, None if h is None else torch.tensor(h).double())
    ng = first.shape[1]
    L = seq.shape[1]
    cols = [ng - 1 + i - (L - out.shape[2]) for i in range(n)]
    return out[:, :, cols].transpose(1, 2).numpy()


@pytest.mark.parametrize("cs", ["16", "8"])
def test_sampler_kernels_match_reference(cs, monkeypatch):
    monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    hop = 3
    m, spec, first, forced, y, h, n = _sampler_setup(hop=hop, G=2)
    want = _ref_logits(m, spec, first, forced, y, hop, h, n)
    free = [_ref_free(m, spec, first[s:s + 1], y[s:s + 1], hop, h[s:s + 1], n) for s in range(3)]
    ran = []
    for mode in (1, 2, 3, 4, 6):
        for ns in (1, 3):
            m._runtime().gen_mode = mode
            try:
                _, lg = m.generate_fast_batch(n, first[:ns], temperature=0.0, forced=forced[:ns], return_logits=True,
                                              condition=h[:ns], local_condition=y[:ns])
            except RuntimeError as e:
                assert "does not apply" in str(e) or "flag exchange" in str(e) or "need a cluster" in str(e), e
                continue
            ran.append((mode, ns))
            err = rel_err(lg, want[:ns])
            assert err < TOL, (mode, ns, err)
            idx = m.generate_fast_batch(n, first[:ns], temperature=0.0, condition=h[:ns], local_condition=y[:ns])
            for s in range(ns):
                assert_stream_parity(idx[s], free[s][0], free[s][1])
    assert (6, 3) in ran and len(ran) >= 4, ran


def _ref_free(m, spec, first, y, hop, h, n):
    """Argmax stream of the float64 reference (one stream), with its logits: re-run the reference per sample."""
    p = {k: v.detach().cpu().double() for k, v in m.state_dict().items()}
    seq = list(first[0])
    yy, hh = torch.tensor(y).double(), torch.tensor(h).double()
    out_idx, logits = [], []
    for i in range(n):
        out = local_ref.stack_direct(p, spec, O.one_hot(torch.tensor([seq]), 256).double(), yy, hop, hh)[0, :, -1]
        logits.append(out.numpy())
        out_idx.append(int(out.argmax()))
        seq.append(out_idx[-1])
    return np.array(out_idx), np.array(logits)


@pytest.mark.parametrize("cs", ["16", "8"])
def test_batched_streams_equal_single_streams(cs, monkeypatch):
    monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    m, spec, first, forced, y, h, n = _sampler_setup(hop=5, NS=9)
    m._runtime().gen_mode = 6
    idx, lg = m.generate_fast_batch(n, first, temperature=0.0, return_logits=True, local_condition=y)
    for s in (0, 4, 8):
        i1, l1 = m.generate_fast_batch(n, first[s:s + 1], temperature=0.0, return_logits=True, local_condition=y[s:s + 1])
        assert np.array_equal(i1[0], idx[s]) and np.array_equal(l1[0], lg[s]), s


@pytest.mark.parametrize("mode", [6, 3, 4])
def test_windows_and_callbacks_are_bit_identical(mode):
    m, spec, first, forced, y, h, n = _sampler_setup(hop=4, NS=1)
    rt = m._runtime()
    rt.gen_mode = mode
    try:
        whole = m.generate_fast(n, first[0], temperature=0.0, local_condition=y[0])
    except RuntimeError as e:
        assert "does not apply" in str(e), e
        pytest.skip(f"mode {mode} does not apply")
    rt.local_table_bytes = 1                 # one frame per window: a launch every 4 evaluations
    calls = []
    split = m.generate_fast(n, first[0], temperature=0.0, local_condition=y[0], progress_interval=7,
                            progress_callback=lambda i, t: calls.append(i))
    assert calls and np.array_equal(whole, split)
    rt.local_table_bytes = 3 * 2 * 256 * 4 * 3 - 1          # two frames per window
    assert np.array_equal(whole, m.generate_fast(n, first[0], temperature=0.0, local_condition=y[0]))


def test_sampler_window_is_checked():
    import ctypes
    import native
    m, spec, first, forced, y, h, n = _sampler_setup(hop=4, NS=1)
    m.generate_fast(n, first[0], temperature=0.0, local_condition=y[0])
    lib, s = native.lib(), m._runtime().sampler(1)
    stream = torch.cuda.current_stream().cuda_stream
    table = torch.zeros(3, 1, 2, 512, device="cuda")
    native.check(lib.wn_gen_set_condition_frames(s["handle"], table.data_ptr(), 1, 2, 4), "set frames")
    native.check(lib.wn_gen_reset(s["handle"], stream), "reset")
    d_first = torch.tensor(first[:, :1], dtype=torch.int32, device="cuda")
    d_out = torch.zeros(1, 8, dtype=torch.int32, device="cuda")
    a = native.GenRunArgs()
    a.d_first, a.n_given, a.d_out_idx, a.n_samples, a.t0, a.n_evals = d_first.data_ptr(), 1, d_out.data_ptr(), 8, 0, 4
    assert lib.wn_gen_run(s["handle"], ctypes.byref(a), stream) != 0          # frame 0 lies before the window
    native.check(lib.wn_gen_set_condition(s["handle"], None), "clear")


# ---------------------------------------------------------------------------------------------- 7. trainer
def test_trainer_with_local_condition_dicts():
    import wavenet_training as wt

    class Items(torch.utils.data.Dataset):
        target_length = 64

        def __init__(self):
            g = torch.Generator().manual_seed(0)
            self.feats = torch.randn(16, 3, 40, generator=g)
            self.x = [torch.randint(0, 256, (400,), generator=g) for _ in range(16)]

        def __len__(self):
            return 16

        def __getitem__(self, i):
            x = self.x[i]
            tgt = ((self.feats[i, 0].repeat_interleave(10)[1:] > 0).long() * 200)[-64:]   # learnable from the features
            return x, {"local_condition": self.feats[i]}, tgt

    kw = dict(layers=3, blocks=2, dilation_channels=32, residual_channels=32, skip_channels=32, end_channels=32,
              classes=256, output_length=64, kernel_size=2, bias=True)
    torch.manual_seed(0)
    import wavenet_model as wmod
    m = wmod.WaveNetModel(**kw, local_condition_channels=3, local_condition_hop=10).cuda()
    ds = Items()
    tr = wt.WavenetTrainer(m, ds, lr=3e-3, snapshot_path=None, num_workers=0)
    losses = []
    x, c, t = torch.utils.data.default_collate([ds[i] for i in range(8)])
    with torch.no_grad():
        losses.append(float(F.cross_entropy(tr._logits(x, c), t.view(-1).cuda())))
    tr.train(batch_size=8, epochs=15)
    with torch.no_grad():
        losses.append(float(F.cross_entropy(tr._logits(x, c), t.view(-1).cuda())))
    assert losses[1] < 0.5 * losses[0], losses
    v = tr.validate()
    assert all(np.isfinite(np.asarray(v, dtype=np.float64)).ravel())


# ---------------------------------------------------------------------------------------------- 4. kernel level
# wn_tb_block_fwd_cond_frames / wn_block_fwd_cond_frames alone on layer 1 of a 2-layer locally conditioned net, two sequences
# with different series, at the frame ranges of test_gpu_conditioning.py's kernel tests (on and beside the 128-frame CTA and
# 256-frame item boundaries).  One block's output at position t depends on the biases of t's frame only, so the reference runs
# block_ref.block_forward once per frame with that frame's term folded into bf / bg and stitches the rows (float64), at the
# bars of test_gpu_kernels_f64.py.  The hops put frame boundaries on tile edges, one row beside them and between a thread's
# rows r0 and r0 + 8.  Negative controls: the frame index shifted by one position, and the two sequences' series swapped.
FRAMES_FWD_CASES = [  # L, dilation, in_start, out_start, skip_start, skip_init, hop
    (1100, 128, 127, 255, 256, 0, 128),
    (900, 255, 1, 256, 257, 1, 128),
    (1037, 257, 256, 513, 513, 0, 97),
]


def _frames_kernel_model(R, D, S, prec, hop):
    import wavenet_model as wmod
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(R + D + S)
        m = wmod.WaveNetModel(layers=2, blocks=1, dilation_channels=D, residual_channels=R, skip_channels=S, end_channels=256,
                              classes=256, output_length=8, kernel_size=2, bias=True, local_condition_channels=4,
                              local_condition_hop=hop)
    g = torch.Generator().manual_seed(17)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith(".bias") or "_local_convs." in n:
                p.copy_(torch.randn(p.shape, generator=g) * (1.0 if "_local_convs." in n else 0.5))
    m = m.cuda()
    m._runtime().tc_precision = prec
    return m


class _FramesRef:
    """block_ref.block_forward per (sequence, series, frame), cached, stitched row by row"""

    def __init__(self, m, h, y, d, in_s, out_s, sk_s, skip0, L):
        import block_ref as BR
        self.BR = BR
        sd = {n: v.detach().cpu() for n, v in m.state_dict().items()}
        self.W = BR.layer_weights(sd, 1)
        self.Uf = sd["filter_local_convs.1.weight"][:, :, 0].double()
        self.Ug = sd["gate_local_convs.1.weight"][:, :, 0].double()
        self.h, self.y, self.args, self.skip0, self.L = h, y.double(), (d, in_s, out_s, sk_s), skip0, L
        self.cache = {}

    def _one(self, b, yb, f, mode):
        key = (b, yb, f, mode)
        if key not in self.cache:
            d, in_s, out_s, sk_s = self.args
            Wb = dict(self.W)
            Wb["bf"] = self.W["bf"].double() + self.Uf @ self.y[yb, :, f]
            Wb["bg"] = self.W["bg"].double() + self.Ug @ self.y[yb, :, f]
            hb = tuple(v[b:b + 1] for v in self.h) if isinstance(self.h, tuple) else self.h[b:b + 1]
            self.cache[key] = self.BR.block_forward(hb, Wb, d, in_s, out_s, sk_s,
                                                    None if self.skip0 is None else self.skip0[b:b + 1], mode=mode,
                                                    pair_out=mode != "exact")
        return self.cache[key]

    def __call__(self, hop, mode, shift=0, series=(0, 1)):
        d, in_s, out_s, sk_s = self.args
        nf = self.y.shape[2]
        fr = lambda t: min((t + shift) // hop, nf - 1)
        out = {}
        for name, t0 in (("h_out", out_s), ("f", out_s), ("g", out_s), ("skip", sk_s)):
            seqs = []
            for b, yb in enumerate(series):
                rows = [self._one(b, yb, fr(t), mode)[name][0, t - t0] for t in range(t0, self.L)]
                seqs.append(torch.stack(rows))
            out[name] = torch.stack(seqs)
        return out


@pytest.mark.parametrize("prec,C", [("pairs", 256), ("bf16", 256), ("bf16", 512)])
@pytest.mark.parametrize("case", range(len(FRAMES_FWD_CASES)))
def test_tb_block_fwd_cond_frames_kernel(prec, C, case):
    import ctypes
    import block_ref as BR
    import native
    import test_gpu_kernels_f64 as KF
    lib = native.lib()
    L, d, in_s, out_s, sk_s, sk_init, hop = FRAMES_FWD_CASES[case]
    B, nf = 2, -(-L // hop)
    m = _frames_kernel_model(C, C, C, "bf16x2" if prec == "pairs" else "bf16", hop)
    st = torch.cuda.current_stream().cuda_stream
    W = m._runtime().packed_weights(st)
    tb_w, tb_b, p_id = W["tb"]
    g = torch.Generator().manual_seed(300 + case)
    y = torch.randn(B, 4, nf, generator=g)
    ctab = W.cond_table_frames(None, y.cuda(), 0, nf, st)            # exactly the frames L positions read
    h = torch.randn(B, L, C, generator=g)
    skip0 = None if sk_init else torch.randn(B, L - sk_s, C, generator=g)
    h_in, h_out = BR.pair_from_frames(h).cuda(), KF._nan(B, 2, C // 8, L, 8, dtype=torch.bfloat16)
    skip = KF._nan(B, C // 4, L - sk_s, 4) if sk_init else BR.chunks4_from_frames(skip0).cuda()
    fg = KF._nan(B, 2 * C // 4, L, 4)
    a = native.TbBlockArgs()
    a.d_h_in, a.d_h_out, a.d_skip, a.d_w_all, a.d_bias4 = h_in.data_ptr(), h_out.data_ptr(), skip.data_ptr(), tb_w.data_ptr(), tb_b[1].data_ptr()
    a.layer, a.n_layers, a.channels, a.precision, a.B, a.L = 1, tb_w.shape[0], C, p_id, B, L
    a.dilation, a.in_start, a.out_start, a.skip_start, a.skip_init, a.d_fg_save = d, in_s, out_s, sk_s, sk_init, fg.data_ptr()
    native.check(lib.wn_tb_block_fwd_cond_frames(ctypes.byref(a), ctab[1].data_ptr(), nf, hop, st), "tb block fwd cond frames")
    torch.cuda.synchronize()
    KF._sentinel_kept("h_out", h_out, out_s)
    hp = BR.planes_from_pair(h_in.cpu())
    got_h = BR.value(BR.planes_from_pair(h_out.cpu()))[:, out_s:]
    got_fg = BR.frames_from_chunks4(fg.cpu())[:, out_s:]
    ref = _FramesRef(m, hp, y, d, in_s, out_s, sk_s, skip0, L)
    ex, em = ref(hop, "exact"), ref(hop, prec)
    kind = "emu" if prec == "pairs" else "bf16"
    print(f"\nwn_tb_block_fwd_cond_frames {prec} {C}: L={L} d={d} in={in_s} out={out_s} skip={sk_s} init={sk_init} hop={hop}")
    bar = KF._check("h_out", got_h, ex["h_out"], em["h_out"], kind, K=2 * C)
    KF._check("skip", BR.frames_from_chunks4(skip.cpu()), ex["skip"], em["skip"], kind, K=2 * C)
    KF._check("tanh", got_fg[..., :C], ex["f"], em["f"], kind, K=2 * C)
    KF._check("sigmoid", got_fg[..., C:], ex["g"], em["g"], kind, K=2 * C)
    KF._miss("frame index shifted by one position", got_h, ref(hop, "exact", shift=1)["h_out"], bar)
    KF._miss("series swapped", got_h, ref(hop, "exact", series=(1, 0))["h_out"], bar)


@pytest.mark.parametrize("shape", [(256, 128, 256), (64, 96, 80), (64, 63, 80)])
@pytest.mark.parametrize("case", range(len(FRAMES_FWD_CASES)))
def test_ffma_block_fwd_cond_frames_kernel(shape, case):
    import ctypes
    import native
    import test_gpu_kernels_f64 as KF
    lib = native.lib()
    R, D, S = shape
    L, d, in_s, out_s, sk_s, sk_init, hop = FRAMES_FWD_CASES[case]
    B, nf = 2, -(-L // hop)
    m = _frames_kernel_model(R, D, S, "bf16x2", hop)
    st = torch.cuda.current_stream().cuda_stream
    W = m._runtime().packed_weights(st)
    wfg, bfg, wrs, brs = W["layers"][1]
    g = torch.Generator().manual_seed(400 + case)
    y = torch.randn(B, 4, nf, generator=g)
    ctab = W.cond_table_frames(None, y.cuda(), 0, nf, st)
    h = torch.randn(B, L, R, generator=g)
    skip0 = None if sk_init else torch.randn(B, L - sk_s, S, generator=g)
    h_out, fg = KF._nan(B, L, R), KF._nan(B, L, 2 * D)
    skip = KF._nan(B, L - sk_s, S) if sk_init else skip0.cuda()
    h_in = h.cuda()
    a = native.BlockArgs()
    a.d_wfg_t, a.d_bfg, a.d_wrs_t, a.d_brs, a.mode = wfg.data_ptr(), bfg.data_ptr(), wrs.data_ptr(), brs.data_ptr(), 0
    a.d_h_in, a.d_h_out, a.d_skip, a.d_fg_save = h_in.data_ptr(), h_out.data_ptr(), skip.data_ptr(), fg.data_ptr()
    a.B, a.L, a.R, a.D, a.S, a.k = B, L, R, D, S, 2
    a.dilation, a.in_start, a.out_start, a.skip_start, a.skip_init = d, in_s, out_s, sk_s, sk_init
    native.check(lib.wn_block_fwd_cond_frames(ctypes.byref(a), ctab[1].data_ptr(), nf, hop, st), "ffma block fwd cond frames")
    torch.cuda.synchronize()
    KF._sentinel_kept("h_out", h_out, out_s)
    ref = _FramesRef(m, h, y, d, in_s, out_s, sk_s, skip0, L)
    ex = ref(hop, "exact")
    print(f"\nwn_block_fwd_cond_frames R={R} D={D} S={S}: L={L} d={d} in={in_s} out={out_s} skip={sk_s} init={sk_init} hop={hop}")
    bar = KF._check("h_out", h_out.cpu()[:, out_s:], ex["h_out"], kind="ffma")
    KF._check("skip", skip.cpu(), ex["skip"], kind="ffma")
    KF._check("tanh", fg.cpu()[:, out_s:, :D], ex["f"], kind="ffma")
    KF._check("sigmoid", fg.cpu()[:, out_s:, D:], ex["g"], kind="ffma")
    KF._miss("frame index shifted by one position", h_out.cpu()[:, out_s:], ref(hop, "exact", shift=1)["h_out"], bar)
    KF._miss("series swapped", h_out.cpu()[:, out_s:], ref(hop, "exact", series=(1, 0))["h_out"], bar)


# ---------------------------------------------------------------------------------------------- 6b. sampler identities
def _gen_all_modes(m, first, n, **cond):
    """{(mode, ns): (indices, logits)} over every sampler kernel that applies, for 1 and all streams"""
    out = {}
    for mode in (1, 2, 3, 4, 6):
        for ns in (1, first.shape[0]):
            m._runtime().gen_mode = mode
            kw = {k: v[:ns] for k, v in cond.items()}
            try:
                out[(mode, ns)] = m.generate_fast_batch(n, first[:ns], temperature=0.0, return_logits=True, **kw)
            except RuntimeError as e:
                assert "does not apply" in str(e) or "flag exchange" in str(e) or "need a cluster" in str(e), e
    return out


@pytest.mark.parametrize("cs", ["16", "8"])
@pytest.mark.parametrize("G", [0, 3])
def test_zero_local_condition_is_identity_in_every_sampler(cs, G, monkeypatch):
    monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    kw = _kw(256, 3, 1, 16)
    m0 = _model(kw, 7, G=G, scale=0.3 if G else None).cuda()
    m1 = _model(kw, 7, C=4, hop=3, G=G).cuda()
    with torch.no_grad():
        for k, v in m1.named_parameters():
            v.copy_(torch.zeros_like(v) if "_local_convs." in k else m0.state_dict()[k])
    rng = np.random.RandomState(0)
    first = rng.randint(0, 256, (3, 20))
    y = rng.randn(3, 4, 15).astype(np.float32)
    cond = dict(condition=rng.randn(3, G).astype(np.float32)) if G else {}
    a, b = _gen_all_modes(m0, first, 24, **cond), _gen_all_modes(m1, first, 24, local_condition=y, **cond)
    assert set(a) == set(b) and (6, 3) in a and len(a) >= 6, sorted(a)
    for k in a:
        assert np.array_equal(a[k][0], b[k][0]) and np.array_equal(a[k][1], b[k][1]), k


@pytest.mark.parametrize("cs", ["16", "8"])
def test_one_frame_sampler_equals_the_global_sampler(cs, monkeypatch):
    """hop >= every evaluation: the frames path with a one-frame window reads the same table the global path reads"""
    monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    kw = _kw(256, 3, 1, 16)
    mg = _model(kw, 9, G=4, scale=0.3).cuda()
    ml = _model(kw, 9, C=4, hop=64).cuda()
    ml.load_state_dict({k.replace("_cond_convs.", "_local_convs."): v for k, v in mg.state_dict().items()})
    rng = np.random.RandomState(1)
    first = rng.randint(0, 256, (3, 20))
    y = rng.randn(3, 4, 1).astype(np.float32)
    a, b = _gen_all_modes(mg, first, 24, condition=y[:, :, 0]), _gen_all_modes(ml, first, 24, local_condition=y)
    assert set(a) == set(b) and (6, 3) in a and len(a) >= 6, sorted(a)
    for k in a:
        assert np.array_equal(a[k][0], b[k][0]) and np.array_equal(a[k][1], b[k][1]), k


@pytest.mark.parametrize("mode,cs", [(2, "16"), (4, "16")])
def test_batched_streams_equal_single_streams_other_kernels(mode, cs, monkeypatch):
    monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    m, spec, first, forced, y, h, n = _sampler_setup(hop=5, NS=9)
    m._runtime().gen_mode = mode
    idx, lg = m.generate_fast_batch(n, first, temperature=0.0, return_logits=True, local_condition=y)
    for s in range(9):
        i1, l1 = m.generate_fast_batch(n, first[s:s + 1], temperature=0.0, return_logits=True, local_condition=y[s:s + 1])
        assert np.array_equal(i1[0], idx[s]) and np.array_equal(l1[0], lg[s]), s
    assert len({tuple(r) for r in idx}) > 1
