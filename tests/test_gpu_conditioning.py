"""Global conditioning (WaveNetModel(condition_channels=G)) on the GPU.  There is no reference counterpart, but an exact one:
for sequence b a conditioned net IS the unconditioned net with filter_convs.i.bias += Vf_i h_b and gate_convs.i.bias +=
Vg_i h_b, so every check folds the condition into the biases and runs the CPU oracle per sequence."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import wavenet_oracle as O
from helpers import assert_stream_parity, rel_err, separate_head_relu_ties

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _kw(ch, layers, blocks, out_len, bias=True, end=256):
    return dict(layers=layers, blocks=blocks, dilation_channels=ch, residual_channels=ch, skip_channels=ch,
                end_channels=end, classes=256, output_length=out_len, kernel_size=2, bias=bias)


def _h(cond, G):
    c = torch.as_tensor(np.asarray(cond))
    return c.double() if c.dtype.is_floating_point else F.one_hot(c.long(), G).double()


def _folded(p, spec, hb):
    """Unconditioned parameters of sequence b: the condition folded into the filter / gate biases (differentiable)."""
    n, D = spec.layers * spec.blocks, spec.dilation_channels
    q = {k: v for k, v in p.items() if "_cond_convs." not in k}
    for i in range(n):
        for conv, cc in (("filter_convs", "filter_cond_convs"), ("gate_convs", "gate_cond_convs")):
            base = p.get(f"{conv}.{i}.bias")
            shift = p[f"{cc}.{i}.weight"][:, :, 0] @ hb.to(p[f"{cc}.{i}.weight"].dtype)
            q[f"{conv}.{i}.bias"] = shift if base is None else base + shift
    return q


def _spec(kw):
    return O.NetSpec(**kw)


def _conditioned_model(kw, G, seed):
    import wavenet_model as wmod
    torch.manual_seed(seed)
    return wmod.WaveNetModel(**kw, condition_channels=G)


def _untie(m, spec, idx, h, out_len, margin):
    """separate_head_relu_ties for every sequence's folded net (the nudged biases are shared by all sequences)."""
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for _ in range(2):
        for b in range(idx.shape[0]):
            q = separate_head_relu_ties(_folded(sd, spec, h[b]), spec, O.one_hot(idx[b:b + 1], 256), out_len, margin=margin)
            last = spec.layers * spec.blocks - 1
            for k in (f"skip_convs.{last}.bias", "end_conv_1.bias"):
                sd[k] = q[k].float()
    m.load_state_dict(sd, strict=True)


# ---------------------------------------------------------------------------------------------- 1. zero conditioning
@pytest.mark.parametrize("ch,prec,mode", [(256, "bf16x2", "auto"), (256, "bf16", "auto"), (512, "bf16", "auto"), (64, "bf16x2", "ffma")])
def test_zero_condition_is_identity_in_training(ch, prec, mode):
    import wavenet_model as wmod
    kw = _kw(ch, 3, 2, 100)
    torch.manual_seed(3)
    m0 = wmod.WaveNetModel(**kw)
    m1 = _conditioned_model(kw, 5, 3)
    sd0 = m0.state_dict()
    for k, v in m1.state_dict().items():
        if "_cond_convs." in k:
            assert k not in sd0
            v.zero_()
        else:
            assert torch.equal(v, sd0[k]), k                 # a seeded construction shares every unconditioned value
    idx = torch.randint(0, 256, (3, 600), generator=torch.Generator().manual_seed(1)).cuda()
    tgt = torch.randint(0, 256, (300,), generator=torch.Generator().manual_seed(2)).cuda()
    out = []
    for m, cond in ((m0, None), (m1, [4, 0, 2])):
        m.cuda()
        rt = m._runtime()
        rt.block_mode, rt.tc_precision = mode, prec
        y = m.forward_indices(idx, condition=cond)
        F.cross_entropy(y, tgt).backward()
        assert rt.last_block_mode == ("tb" if mode == "auto" else "ffma")
        out.append((y.detach(), {k: p.grad.clone() for k, p in m.named_parameters()}))
    assert torch.equal(out[0][0], out[1][0])
    for k, g in out[0][1].items():
        if k == "start_conv.weight":        # a scatter-add over the input indices with atomics: not bit-reproducible run to run
            assert rel_err(out[1][1][k].cpu().numpy(), g.cpu().numpy()) < 1e-6
            continue
        assert torch.equal(g, out[1][1][k]), k


@pytest.mark.parametrize("cs", ["16", "8"])
def test_zero_condition_is_identity_in_every_sampler(cs, monkeypatch):
    import wavenet_model as wmod
    monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    kw = _kw(256, 3, 1, 16)
    torch.manual_seed(7)
    m0 = wmod.WaveNetModel(**kw).cuda()
    m1 = _conditioned_model(kw, 3, 7).cuda()
    with torch.no_grad():
        for k, v in m1.named_parameters():
            if "_cond_convs." in k:
                v.zero_()
    first = np.random.RandomState(0).randint(0, 256, (3, 20))
    for ns in (1, 3):
        for mode in (1, 2, 3, 4, 6):
            res = []
            for m, cond in ((m0, None), (m1, [2, 0, 1][:ns])):
                m._runtime().gen_mode = mode
                try:
                    res.append(m.generate_fast_batch(24, first[:ns], temperature=0.0, return_logits=True, condition=cond))
                except RuntimeError as e:
                    assert "does not apply" in str(e) or "flag exchange" in str(e), e
            if res:
                assert len(res) == 2
                assert np.array_equal(res[0][0], res[1][0]) and np.array_equal(res[0][1], res[1][1]), (ns, mode)


# ---------------------------------------------------------------------------------------------- 2. training parity
@pytest.mark.parametrize("ch,prec,mode,dense,stack", [(256, "bf16x2", "auto", False, True), (256, "bf16x2", "auto", True, True),
                                                      (256, "bf16x2", "auto", True, False),      # one wn_tb_block_fwd_cond per layer
                                                      (64, "bf16x2", "ffma", False, True), (64, "bf16x2", "ffma", True, True),
                                                      (512, "bf16", "auto", False, True), (512, "bf16", "auto", False, False)])
def test_conditioned_training_matches_folded_oracle(ch, prec, mode, dense, stack):
    G, B, L, out_len = 6, 3, 700, 200
    kw = _kw(ch, 3, 2, out_len)
    spec = _spec(kw)
    m = _conditioned_model(kw, G, 13)
    with torch.no_grad():                                  # conditioning terms of the size of the biases
        for k, v in m.named_parameters():
            if "_cond_convs." in k:
                v.normal_(0, 0.3)
    rng = np.random.RandomState(5)
    cond = rng.randn(B, G).astype(np.float32) if dense else np.array([5, 0, 3])
    h = _h(cond, G)
    idx = torch.randint(0, 256, (B, L), generator=torch.Generator().manual_seed(8))
    tgt = torch.randint(0, 256, (B * out_len,), generator=torch.Generator().manual_seed(9))
    pair = prec == "bf16x2"
    _untie(m, spec, idx, h, out_len, 2e-5 if pair else 2e-3)
    p = {k: v.detach().clone().double().requires_grad_(True) for k, v in m.state_dict().items()}
    want = torch.cat([O.forward(_folded(p, spec, h[b]), spec, O.one_hot(idx[b:b + 1], 256).double()) for b in range(B)])
    F.cross_entropy(want, tgt).backward()
    m = m.cuda()
    rt = m._runtime()
    rt.block_mode, rt.tc_precision, rt.stack_launch = mode, prec, stack
    y = m.forward_indices(idx.cuda(), condition=cond)
    assert rt.last_block_mode == ("tb" if mode == "auto" else "ffma")
    if mode == "auto":
        assert rt.last_block_launches == (1 if stack else spec.layers * spec.blocks)
    F.cross_entropy(y, tgt.cuda()).backward()
    e = rel_err(y.detach().cpu().numpy(), want.detach().numpy())
    errs = {k: rel_err(v.grad.cpu().numpy(), p[k].grad.numpy()) for k, v in m.named_parameters()
            if p[k].grad is not None and float(p[k].grad.abs().max()) > 0}
    assert any("_cond_convs." in k for k in errs)
    worst = max(errs.values())
    print(f"conditioned {ch} ch {prec} {mode} dense={dense} stack={stack}: logits {e:.2e}, worst gradient {worst:.2e}")
    if pair:
        assert e < TOL and worst < TOL, (e, sorted(errs.items(), key=lambda kv: -kv[1])[:5])
    else:
        assert e < 3e-2 and worst < 6e-2, (e, worst)


def test_condition_argument_errors_on_gpu():
    m = _conditioned_model(_kw(64, 2, 1, 10), 4, 0).cuda()
    idx = torch.randint(0, 256, (2, 100)).cuda()
    with pytest.raises(ValueError):
        m.forward_indices(idx)
    with pytest.raises(ValueError):
        m.forward_indices(idx, condition=[1, 4])
    with pytest.raises(NotImplementedError):
        m.wavenet(torch.zeros(1, 256, 1).cuda(), dilation_func=m.queue_dilate)
    with pytest.raises(NotImplementedError):              # a trainable embedding would silently get no gradient
        m.forward_indices(idx, condition=torch.randn(2, 4, device="cuda", requires_grad=True))
    m._runtime().block_mode = "tc"
    with pytest.raises(RuntimeError):
        m.forward_indices(idx, condition=[1, 2])


# ---------------------------------------------------------------------------------------------- 3. kernel level
# wn_tb_block_fwd_cond / wn_block_fwd_cond alone on layer 1 of a 2-layer conditioned net, two sequences with different labels,
# frame ranges on and beside the 128-frame CTA and 256-frame item boundaries; the reference is block_ref.block_forward per
# sequence with that sequence's condition folded into bf / bg (float64), at the bars of test_gpu_kernels_f64.py.  Negative
# control: the same reference with the two sequences' conditions swapped.
COND_FWD_CASES = [  # L, dilation, in_start, out_start, skip_start, skip_init
    (1100, 128, 127, 255, 256, 0),
    (900, 255, 1, 256, 257, 1),
    (1037, 257, 256, 513, 513, 0),
]
LABELS = [1, 3]


def _cond_kernel_model(R, D, S, prec):
    import wavenet_model as wmod
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(R + D + S)
        m = wmod.WaveNetModel(layers=2, blocks=1, dilation_channels=D, residual_channels=R, skip_channels=S, end_channels=256,
                              classes=256, output_length=8, kernel_size=2, bias=True, condition_channels=4)
    g = torch.Generator().manual_seed(17)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith(".bias") or "_cond_convs." in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
    m = m.cuda()
    m._runtime().tc_precision = prec
    return m


def _cond_refs(m, h, d, in_s, out_s, sk_s, skip0, labels, mode):
    """block_ref.block_forward per sequence with its condition folded into layer 1's biases, concatenated over sequences"""
    import block_ref as BR
    sd = {n: v.detach().cpu() for n, v in m.state_dict().items()}
    W = BR.layer_weights(sd, 1)
    outs = []
    for b, lab in enumerate(labels):
        Wb = dict(W)
        Wb["bf"] = W["bf"].double() + sd["filter_cond_convs.1.weight"][:, lab, 0].double()
        Wb["bg"] = W["bg"].double() + sd["gate_cond_convs.1.weight"][:, lab, 0].double()
        hb = tuple(v[b:b + 1] for v in h) if isinstance(h, tuple) else h[b:b + 1]      # h: fp32 frames or a stored (hi, lo) pair
        outs.append(BR.block_forward(hb, Wb, d, in_s, out_s, sk_s, None if skip0 is None else skip0[b:b + 1], mode=mode,
                                     pair_out=mode != "exact"))
    return {k: torch.cat([o[k] for o in outs]) for k in outs[0]}


@pytest.mark.parametrize("prec,C", [("pairs", 256), ("bf16", 256), ("bf16", 512)])
@pytest.mark.parametrize("case", range(len(COND_FWD_CASES)))
def test_tb_block_fwd_cond_kernel(prec, C, case):
    import ctypes
    import block_ref as BR
    import native
    import test_gpu_kernels_f64 as KF
    lib = native.lib()
    L, d, in_s, out_s, sk_s, sk_init = COND_FWD_CASES[case]
    B = len(LABELS)
    m = _cond_kernel_model(C, C, C, "bf16x2" if prec == "pairs" else "bf16")
    st = torch.cuda.current_stream().cuda_stream
    W = m._runtime().packed_weights(st)
    tb_w, tb_b, p_id = W["tb"]
    ctab = W.cond_table(m._condition(LABELS, B), st)
    g = torch.Generator().manual_seed(300 + case)
    h = torch.randn(B, L, C, generator=g)
    skip0 = None if sk_init else torch.randn(B, L - sk_s, C, generator=g)
    h_in, h_out = BR.pair_from_frames(h).cuda(), KF._nan(B, 2, C // 8, L, 8, dtype=torch.bfloat16)
    skip = KF._nan(B, C // 4, L - sk_s, 4) if sk_init else BR.chunks4_from_frames(skip0).cuda()
    fg = KF._nan(B, 2 * C // 4, L, 4)
    a = native.TbBlockArgs()
    a.d_h_in, a.d_h_out, a.d_skip, a.d_w_all, a.d_bias4 = h_in.data_ptr(), h_out.data_ptr(), skip.data_ptr(), tb_w.data_ptr(), tb_b[1].data_ptr()
    a.layer, a.n_layers, a.channels, a.precision, a.B, a.L = 1, tb_w.shape[0], C, p_id, B, L
    a.dilation, a.in_start, a.out_start, a.skip_start, a.skip_init, a.d_fg_save = d, in_s, out_s, sk_s, sk_init, fg.data_ptr()
    native.check(lib.wn_tb_block_fwd_cond(ctypes.byref(a), ctab[1].data_ptr(), st), "tb block fwd cond")
    torch.cuda.synchronize()
    KF._sentinel_kept("h_out", h_out, out_s)
    hp = BR.planes_from_pair(h_in.cpu())
    got_h = BR.value(BR.planes_from_pair(h_out.cpu()))[:, out_s:]
    got_fg = BR.frames_from_chunks4(fg.cpu())[:, out_s:]
    ex = _cond_refs(m, hp, d, in_s, out_s, sk_s, skip0, LABELS, "exact")
    em = _cond_refs(m, hp, d, in_s, out_s, sk_s, skip0, LABELS, prec)
    kind = "emu" if prec == "pairs" else "bf16"
    print(f"\nwn_tb_block_fwd_cond {prec} {C}: L={L} d={d} in={in_s} out={out_s} skip={sk_s} init={sk_init}")
    bar = KF._check("h_out", got_h, ex["h_out"], em["h_out"], kind, K=2 * C)
    KF._check("skip", BR.frames_from_chunks4(skip.cpu()), ex["skip"], em["skip"], kind, K=2 * C)
    KF._check("tanh", got_fg[..., :C], ex["f"], em["f"], kind, K=2 * C)
    KF._check("sigmoid", got_fg[..., C:], ex["g"], em["g"], kind, K=2 * C)
    KF._miss("conditions swapped", got_h, _cond_refs(m, hp, d, in_s, out_s, sk_s, skip0, LABELS[::-1], "exact")["h_out"], bar)


@pytest.mark.parametrize("shape", [(256, 128, 256), (64, 96, 80)])
@pytest.mark.parametrize("case", range(len(COND_FWD_CASES)))
def test_ffma_block_fwd_cond_kernel(shape, case):
    import ctypes
    import native
    import test_gpu_kernels_f64 as KF
    lib = native.lib()
    R, D, S = shape
    L, d, in_s, out_s, sk_s, sk_init = COND_FWD_CASES[case]
    B = len(LABELS)
    m = _cond_kernel_model(R, D, S, "bf16x2")
    st = torch.cuda.current_stream().cuda_stream
    W = m._runtime().packed_weights(st)
    ctab = W.cond_table(m._condition(LABELS, B), st)
    wfg, bfg, wrs, brs = W["layers"][1]
    g = torch.Generator().manual_seed(400 + case)
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
    native.check(lib.wn_block_fwd_cond(ctypes.byref(a), ctab[1].data_ptr(), st), "ffma block fwd cond")
    torch.cuda.synchronize()
    KF._sentinel_kept("h_out", h_out, out_s)
    ex = _cond_refs(m, h, d, in_s, out_s, sk_s, skip0, LABELS, "exact")
    print(f"\nwn_block_fwd_cond R={R} D={D} S={S}: L={L} d={d} in={in_s} out={out_s} skip={sk_s} init={sk_init}")
    bar = KF._check("h_out", h_out.cpu()[:, out_s:], ex["h_out"], kind="ffma")
    KF._check("skip", skip.cpu(), ex["skip"], kind="ffma")
    KF._check("tanh", fg.cpu()[:, out_s:, :D], ex["f"], kind="ffma")
    KF._check("sigmoid", fg.cpu()[:, out_s:, D:], ex["g"], kind="ffma")
    KF._miss("conditions swapped", h_out.cpu()[:, out_s:], _cond_refs(m, h, d, in_s, out_s, sk_s, skip0, LABELS[::-1], "exact")["h_out"], bar)


# ---------------------------------------------------------------------------------------------- 4. sampler
@pytest.mark.parametrize("mode,cs", [(6, "16"), (6, "8"), (2, "16"), (4, "16")])
def test_batched_streams_equal_single_stream_runs(mode, cs, monkeypatch):
    monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    G, NS = 16, 16
    m = _conditioned_model(_kw(256, 3, 1, 16), G, 21).cuda()
    with torch.no_grad():
        for k, v in m.named_parameters():
            if "_cond_convs." in k:
                v.normal_(0, 0.3)
    m._runtime().gen_mode = mode
    first = np.random.RandomState(1).randint(0, 256, (NS, 12))
    labels = np.random.RandomState(2).permutation(G)
    idx, logits = m.generate_fast_batch(20, first, temperature=0.0, return_logits=True, condition=labels)
    for s in range(NS):
        i1, l1 = m.generate_fast_batch(20, first[s:s + 1], temperature=0.0, return_logits=True, condition=labels[s:s + 1])
        assert np.array_equal(idx[s], i1[0]) and np.array_equal(logits[s], l1[0]), s
    assert len({tuple(r) for r in idx}) > 1                # distinct conditions give distinct streams


@pytest.mark.parametrize("mode", [1, 2, 3, 4, 6])
def test_sampler_matches_folded_oracle(mode):
    G, NS = 4, 3
    kw = _kw(256, 3, 1, 16)
    spec = _spec(kw)
    m = _conditioned_model(kw, G, 31)
    with torch.no_grad():
        for k, v in m.named_parameters():
            if "_cond_convs." in k:
                v.normal_(0, 0.3)
    p = {k: v.detach().clone() for k, v in m.state_dict().items()}
    m = m.cuda()
    m._runtime().gen_mode = mode
    first = np.random.RandomState(3).randint(0, 256, (NS, 10))
    cond = np.random.RandomState(4).randn(NS, G).astype(np.float32)
    refs = [O.generate_fast({k: v.float() for k, v in _folded(p, spec, _h(cond, G)[s]).items()}, spec, 24,
                            first_samples=first[s], temperature=0.0, keep_logits=True) for s in range(NS)]
    ns = 1 if mode == 3 else NS
    forced = np.stack([r.indices for r in refs[:ns]])
    try:
        _, logits = m.generate_fast_batch(24, first[:ns], temperature=0.0, forced=forced, return_logits=True,
                                          condition=cond[:ns])
    except RuntimeError as e:
        pytest.skip(f"kernel {mode} does not apply: {e}")
    for s in range(ns):
        assert rel_err(logits[s], refs[s].logits) < TOL, (mode, s)
        got = m.generate_fast_batch(24, first[s:s + 1], temperature=0.0, condition=cond[s:s + 1])
        assert_stream_parity(got[0], refs[s].indices, refs[s].logits)
    g1 = m.generate_fast(8, first_samples=first[0], temperature=0.0, condition=cond[0])
    assert g1.shape == (8,)


# ---------------------------------------------------------------------------------------------- 5. trainer and dataset
def test_trainer_on_file_labels():
    import os
    import audio_data
    import wavenet_training as wt
    golden_dir = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    ds = audio_data.WavenetDataset(os.path.join(golden_dir, "tiny_dataset.npz"), item_length=300, target_length=64,
                                   one_hot=False, condition_on_file=True, test_stride=5)
    n_files = len(ds.start_samples) - 1
    m = _conditioned_model(_kw(32, 3, 2, 64, end=32), n_files, 0).cuda()
    tr = wt.WavenetTrainer(m, ds, lr=3e-3, num_workers=0, logger=wt.Logger(log_interval=10 ** 9))
    losses = []
    tr.logger.log = lambda step, loss: losses.append(loss)
    tr.train(batch_size=4, epochs=50, max_steps=30)
    assert np.mean(losses[-5:]) < np.mean(losses[:5]), losses
    vl, va = tr.validate()
    assert np.isfinite(vl) and 0 <= va <= 1
