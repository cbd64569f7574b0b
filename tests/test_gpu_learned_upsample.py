"""Learned local-conditioning upsampler (WaveNetModel(..., local_condition_upsample_scales=...)) on the GPU: the K-slab
forward of the fused tensor-core blocks, the hop-1 local path of the FFMA blocks and the sampler, against the unconditioned
net, an explicit hop-1 twin fed the upsampled features, the repeat-upsampled net and the float64 reference
(tests/upsample_ref.py)."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import upsample_ref
from oracle import wavenet_oracle as O
from helpers import rel_err
from test_gpu_local_conditioning import _untie

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _kw(ch, layers, blocks, out_len, bias=True, end=256):
    return dict(layers=layers, blocks=blocks, dilation_channels=ch, residual_channels=ch, skip_channels=ch,
                end_channels=end, classes=256, output_length=out_len, kernel_size=2, bias=bias)


def _model(kw, seed, C=0, scales=None, G=0, scale=None, up_scale=None):
    import wavenet_model as wmod
    torch.manual_seed(seed)
    m = wmod.WaveNetModel(**kw, condition_channels=G, local_condition_channels=C,
                          local_condition_hop=None if scales is None else math.prod(scales),
                          local_condition_upsample_scales=scales)
    with torch.no_grad():
        for k, v in m.named_parameters():
            if scale is not None and ("_local_convs." in k or "_cond_convs." in k):
                # conditioning terms of the size of the biases: the C = 4 scale of the frame-rate tests, per sqrt(fan-in)
                v.normal_(0, scale * (2 / v.shape[1]) ** 0.5 if "_local_convs." in k else scale)
            if up_scale is not None and k.startswith("local_upsample."):
                fan = v.shape[0] * v.shape[2] if v.dim() == 3 else 1            # keeps c of the size of y
                v.add_(torch.randn(v.shape, generator=torch.Generator().manual_seed(len(k))) * up_scale / fan ** 0.5)
    return m


def _twin(m):
    """The explicit hop-1 local model with m's parameters (no upsampler)."""
    import wavenet_model as wmod
    kw = dict(layers=m.layers, blocks=m.blocks, dilation_channels=m.dilation_channels, residual_channels=m.residual_channels,
              skip_channels=m.skip_channels, end_channels=m.end_conv_1.out_channels, classes=m.classes,
              output_length=m.output_length, kernel_size=m.kernel_size, bias=m.start_conv.bias is not None)
    t = wmod.WaveNetModel(**kw, condition_channels=m.condition_channels, local_condition_channels=m.local_condition_channels,
                          local_condition_hop=1)
    t.load_state_dict({k: v for k, v in m.state_dict().items() if not k.startswith("local_upsample.")})
    return t


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


TB = [(256, "bf16x2"), (256, "bf16"), (512, "bf16")]


# ---------------------------------------------------------------------------------------------- 1. zero U is the identity
@pytest.mark.parametrize("ch,prec", TB)
@pytest.mark.parametrize("stack", [True, False])
def test_zero_u_is_identity(ch, prec, stack):
    kw = _kw(ch, 3, 2, 100)
    idx = torch.randint(0, 256, (3, 600), generator=torch.Generator().manual_seed(1)).cuda()
    tgt = torch.randint(0, 256, (300,), generator=torch.Generator().manual_seed(2)).cuda()
    y = torch.randn(3, 4, 600 // 6 + 1, generator=torch.Generator().manual_seed(3)).cuda()
    for G in (0, 5):
        m0 = _model(kw, 3, G=G)
        m1 = _model(kw, 3, C=4, scales=(2, 3), G=G, up_scale=0.3)
        with torch.no_grad():
            for k, v in m1.named_parameters():
                if "_local_convs." in k:
                    v.zero_()
        cond = dict(condition=[4, 0, 2]) if G else {}
        a = _run(m0, idx, tgt, "auto", prec, stack, **cond)
        b = _run(m1, idx, tgt, "auto", prec, stack, local_condition=y, **cond)
        _assert_shared_identical(a, b)


# ---------------------------------------------------------------------------------------------- 2. the explicit hop-1 twin
@pytest.mark.parametrize("ch,prec,mode,stack", [(64, "bf16x2", "ffma", True), (256, "bf16x2", "auto", True),
                                                (256, "bf16x2", "auto", False), (256, "bf16", "auto", True),
                                                (512, "bf16", "auto", False)])
def test_same_as_the_hop1_twin(ch, prec, mode, stack):
    kw = _kw(ch, 3, 2, 100)
    L = 600
    idx = torch.randint(0, 256, (3, L), generator=torch.Generator().manual_seed(1)).cuda()
    tgt = torch.randint(0, 256, (300,), generator=torch.Generator().manual_seed(2)).cuda()
    y = torch.randn(3, 5, 60, generator=torch.Generator().manual_seed(3))
    m = _model(kw, 4, C=5, scales=(2, 5), G=3, scale=0.3, up_scale=0.3)
    h = torch.randn(3, 3, generator=torch.Generator().manual_seed(4))
    if mode != "ffma":                  # no head ReLU input near zero, where two fp32-class paths could differ in a branch
        c64 = upsample_ref.upsample({k: v.double() for k, v in m.state_dict().items()}, (2, 5), y.double())[:, :, :L]
        _untie(m, O.NetSpec(**kw), idx.cpu(), c64, 1, h.double(), 100, 2e-5 if prec == "bf16x2" else 2e-3)
    m, y, h = m.cuda(), y.cuda(), h.cuda()
    t = _twin(m).cuda()
    with torch.no_grad():
        c = m._upsample(y, L)
    a = _run(m, idx, tgt, mode, prec, stack, condition=h, local_condition=y)
    b = _run(t, idx, tgt, mode, prec, stack, condition=h, local_condition=c)
    assert any(float(g.abs().max()) > 0 for k, g in a[1].items() if k.startswith("local_upsample."))
    if mode == "ffma":
        _assert_shared_identical(a, b)
        return
    bar = (TOL, TOL) if prec == "bf16x2" else (3e-2, 6e-2)
    assert rel_err(a[0].cpu().numpy(), b[0].cpu().numpy()) < bar[0]
    for k, g in b[1].items():
        if float(g.abs().max()) > 0:
            assert rel_err(a[1][k].cpu().numpy(), g.cpu().numpy()) < bar[1], k


@pytest.mark.parametrize("ns", [1, 8, 64])
def test_sampler_same_as_the_hop1_twin(ns):
    kw = _kw(64, 3, 2, 1)
    m = _model(kw, 6, C=3, scales=(4, 5), scale=0.3, up_scale=0.3).cuda()
    t = _twin(m).cuda()
    n_given, n = 5, 300
    first = np.random.RandomState(1).randint(0, 256, (ns, n_given))
    y = torch.randn(ns, 3, -(-(n_given - 1 + n) // 20), generator=torch.Generator().manual_seed(2)).cuda()
    with torch.no_grad():
        c = m._upsample(y, n_given - 1 + n)
    for mm in (m, t):
        mm._runtime().local_table_bytes = 6 * ns * 2 * 64 * 4 * 37          # 37-evaluation windows of the hop-1 table
    uni = np.random.RandomState(3).random_sample((ns, n))
    ia, la = m.generate_fast_batch(n, first, temperature=1.0, uniforms=uni, return_logits=True, local_condition=y)
    ib, lb = t.generate_fast_batch(n, first, temperature=1.0, uniforms=uni, return_logits=True, local_condition=c)
    assert np.array_equal(ia, ib) and np.array_equal(la, lb)


def test_repetition_init_is_the_repeat_model_on_ffma():
    kw = _kw(64, 3, 2, 100)
    mr = _model(kw, 8, C=4, scales=(2, 3)).cuda()
    torch.manual_seed(8)
    import wavenet_model as wmod
    mp = wmod.WaveNetModel(**kw, local_condition_channels=4, local_condition_hop=6).cuda()
    for mm in (mr, mp):
        mm._runtime().block_mode = "ffma"
    idx = torch.randint(0, 256, (2, 400), generator=torch.Generator().manual_seed(1)).cuda()
    y = torch.randn(2, 4, 67, generator=torch.Generator().manual_seed(2)).cuda()
    with torch.no_grad():
        assert torch.equal(mr.forward_indices(idx, local_condition=y), mp.forward_indices(idx, local_condition=y))
    first = np.random.RandomState(1).randint(0, 256, (8, 3))
    yy = torch.randn(8, 4, 60, generator=torch.Generator().manual_seed(3)).cuda()
    uni = np.random.RandomState(3).random_sample((8, 200))
    assert np.array_equal(mr.generate_fast_batch(200, first, temperature=1.0, uniforms=uni, local_condition=yy),
                          mp.generate_fast_batch(200, first, temperature=1.0, uniforms=uni, local_condition=yy))


# ---------------------------------------------------------------------------------------------- 3. parity with float64
@pytest.mark.parametrize("ch,prec,stack,C,G", [
    (256, "bf16x2", True, 1, 0), (256, "bf16x2", True, 80, 3), (256, "bf16x2", False, 96, 0), (256, "bf16x2", True, 200, 0),
    (256, "bf16x2", False, 200, 3), (256, "bf16", True, 80, 0), (512, "bf16", True, 96, 3), (512, "bf16", False, 200, 0),
    (64, "bf16x2", True, 80, 3)])
def test_learned_training_matches_reference(ch, prec, stack, C, G):
    B, L, out_len, scales = 2, 700, 200, (4, 5)
    hop = math.prod(scales)
    kw = _kw(ch, 3, 2, out_len)
    spec = O.NetSpec(**kw)
    m = _model(kw, 13, C=C, scales=scales, G=G, scale=0.3, up_scale=0.3)
    rng = np.random.RandomState(5)
    y = torch.tensor(rng.randn(B, C, -(-L // hop) + 1).astype(np.float32))
    h = torch.tensor(rng.randn(B, G).astype(np.float32)) if G else None
    idx = torch.randint(0, 256, (B, L), generator=torch.Generator().manual_seed(8))
    tgt = torch.randint(0, 256, (B * out_len,), generator=torch.Generator().manual_seed(9))
    pair = prec == "bf16x2"
    p0 = {k: v.double() for k, v in m.state_dict().items()}
    c64 = upsample_ref.upsample(p0, scales, y.double())[:, :, :L]
    _untie(m, spec, idx, c64, 1, None if h is None else h.double(), out_len, 2e-5 if pair else 2e-3)
    p = {k: v.detach().clone().double().requires_grad_(True) for k, v in m.state_dict().items()}
    yd = y.double().requires_grad_(True)
    want = upsample_ref.forward(p, spec, O.one_hot(idx, 256).double(), yd, scales, None if h is None else h.double())
    F.cross_entropy(want, tgt).backward()
    m = m.cuda()
    rt = m._runtime()
    mode = "auto" if ch >= 256 else "ffma"
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
    assert any(k.startswith("local_upsample.") for k in errs) and any("_local_convs." in k for k in errs)
    worst = max(errs.values())
    print(f"learned {ch} ch {prec} stack={stack} C={C} G={G}: logits {e:.2e}, worst gradient {worst:.2e}")
    if pair:
        assert e < TOL and worst < TOL, (e, sorted(errs.items(), key=lambda kv: -kv[1])[:5])
    else:
        assert e < 3e-2 and worst < 6e-2, (e, worst)


# ---------------------------------------------------------------------------------------------- 4. kernels alone
def test_local_pairs_conversion_pads_with_zeros():
    import native
    lib = native.lib()
    B, C, L = 2, 13, 300
    for prec, width in ((native.PREC_BF16_PAIRS, 32), (native.PREC_BF16, 64)):
        cpad = lib.wn_tb_local_padded_channels(C, prec)
        assert cpad == width
        x = torch.randn(B, C, L, generator=torch.Generator().manual_seed(1)).cuda()
        out = torch.full((B, 2, cpad // 8, L, 8), float("nan"), dtype=torch.bfloat16, device="cuda")
        native.check(lib.wn_tb_local_from_channels(x.data_ptr(), out.data_ptr(), B, C, L, prec, None), "convert")
        torch.cuda.synchronize()
        v = (out[:, 0].float() + out[:, 1].float()).permute(0, 1, 3, 2).reshape(B, cpad, L)
        assert torch.equal(v[:, C:], torch.zeros_like(v[:, C:]))
        assert torch.equal(out[:, 0].float().permute(0, 1, 3, 2).reshape(B, cpad, L)[:, :C], x.to(torch.bfloat16).float())
        assert float((v[:, :C] - x).abs().max()) <= 2.0 ** -16 * float(x.abs().max())


def test_series_gradient_is_deterministic():
    kw = _kw(256, 2, 2, 100)
    m = _model(kw, 5, C=80, scales=(4, 5), scale=0.3, up_scale=0.3).cuda()
    idx = torch.randint(0, 256, (2, 500), generator=torch.Generator().manual_seed(1)).cuda()
    tgt = torch.randint(0, 256, (200,), generator=torch.Generator().manual_seed(2)).cuda()
    y0 = torch.randn(2, 80, 25, generator=torch.Generator().manual_seed(3)).cuda()
    got = []
    for _ in range(2):
        y = y0.clone().requires_grad_(True)
        F.cross_entropy(m.forward_indices(idx, local_condition=y), tgt).backward()
        got.append(y.grad.clone())
    assert torch.equal(got[0], got[1])


# ---------------------------------------------------------------------------------------------- 6. errors
def test_learned_upsampler_errors_on_gpu():
    m = _model(_kw(64, 2, 1, 10), 0, C=3, scales=(2, 5)).cuda()
    idx = torch.randint(0, 256, (2, 100)).cuda()
    with pytest.raises(ValueError, match=r"locally conditioned on 3 channels: pass local_condition= \(a float \(2, 3, F\) series, "
                                         r"F >= 10 frames of 10 samples\)"):
        m.forward_indices(idx)
    with pytest.raises(ValueError, match=r"local_condition has 9 frames; 100 positions at hop 10 need at least 10"):
        m.forward_indices(idx, local_condition=torch.zeros(2, 3, 9, device="cuda"))
    with pytest.raises(ValueError, match=r"local_condition must be a float \(2, 3, F\) array, got shape \(2, 4, 10\)"):
        m.forward_indices(idx, local_condition=torch.zeros(2, 4, 10, device="cuda"))
    with pytest.raises(ValueError, match=r"local_condition must be a float \(2, 3, F\) array, got torch.int64"):
        m.forward_indices(idx, local_condition=torch.zeros(2, 3, 10, device="cuda", dtype=torch.int64))
    m._runtime().block_mode = "tc"
    with pytest.raises(RuntimeError, match="two-launch 'tc' blocks have no conditioned kernel"):
        m.forward_indices(idx, local_condition=torch.zeros(2, 3, 10, device="cuda"))


# ---------------------------------------------------------------------------------------------- 5. trainer
def test_trainer_with_a_learned_upsampler():
    """Several optimizer steps through WavenetTrainer on (x, {"local_condition": y}, target) items, on the K-slab path: the
    upsampler's graph is built in each forward and consumed in its backward, and the packs (U included) are rebuilt after
    every step, so the loss can only fall if all of that holds."""
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
            tgt = ((self.feats[i, 0].repeat_interleave(10)[1:] > 0).long() * 200)[-64:]   # learnable from the features
            return self.x[i], {"local_condition": self.feats[i]}, tgt

    torch.manual_seed(0)
    m = _model(_kw(256, 3, 2, 64), 0, C=3, scales=(2, 5)).cuda()
    ds = Items()
    tr = wt.WavenetTrainer(m, ds, lr=1e-3, snapshot_path=None, num_workers=0)
    x, c, t = torch.utils.data.default_collate([ds[i] for i in range(8)])
    w0 = m.local_upsample[0].weight.detach().clone()
    with torch.no_grad():
        before = float(F.cross_entropy(tr._logits(x, c), t.view(-1).cuda()))
    tr.train(batch_size=8, epochs=15)
    assert m._runtime().last_block_mode == "tb"
    with torch.no_grad():
        after = float(F.cross_entropy(tr._logits(x, c), t.view(-1).cuda()))
    assert after < 0.5 * before, (before, after)
    assert not torch.equal(w0, m.local_upsample[0].weight.detach())       # the upsampler was trained too
