"""The sampler's ring prefill (generate_fast(..., prefill=True), _Runtime.prefill, wn_gen_prefill_*) on the GPU.

Rings after a prefill to T against the rings after T sequential evaluations (tags and layer 0 bit-identical, every value
within 1e-4 of the float64 layer inputs of tests/prefill_ref.py) on kernels 1, 2, 3, 4 and 6 at clusters of 16 and 8;
teacher-forced runs after prompts around the ring lengths and the receptive field against tests/sampler_ref.py; free
running against the sequential warm-up; batches, per-stream settings, conditioning, a 512-channel net; and the state rules
of the C ABI.  Each case prints its measured errors (pytest -s)."""
import ctypes

import numpy as np
import pytest
import torch

import native
import prefill_ref as P
import sampler_ref as R
import wavenet_model as wmod
from helpers import build_model, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
CFG2_DIL = R.dilations_of(10, 5)
RF = 5116

# (id, gen_mode, WN_GEN_CL8_CS, streams, kernel that must run, CTAs per cluster)
KERNELS = [("k1", 1, None, 1, 1, 0), ("k2", 2, None, 1, 2, 0), ("k3", 3, None, 1, 3, 0), ("k4", 4, None, 2, 4, 16),
           ("k6-cs16", 6, "16", 8, 6, 16), ("k6-cs8", 6, "8", 8, 6, 8)]
_ids = lambda cases: [c[0] for c in cases]
_refs = {}


def _model(golden, monkeypatch, mode=None, cs=None, name="net_cfg2.npz"):
    if cs is not None:
        monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    m = build_model(golden(name))
    m._runtime().gen_mode = mode
    return m


def _kernel(m, ns):
    h = m._runtime().sampler(ns)["handle"]
    kid = native.lib().wn_gen_kernel_id(h)
    g, b, x = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    native.check(native.lib().wn_gen_launch_info(h, ctypes.byref(g), ctypes.byref(b), ctypes.byref(x)), "launch info")
    return kid, (g.value // -(-ns // 8) if kid == 6 else 16 if kid == 4 else 0)


def _check_kernel(m, ns, kid_want, cs_want):
    kid, cs = _kernel(m, ns)
    assert (kid, cs) == (kid_want, cs_want), f"ran kernel {kid} at cluster {cs}"
    return kid, cs


def _rings(m, s, plain):
    """[(values (len, NS, R), tags (len, NS, R) int32 or None)] per layer, on the host"""
    Rr, NS, k, off, out = m.residual_channels, s["n_streams"], m.kernel_size, 0, []
    for d, _ in m.dilations:
        ln = (k - 1) * d + 1
        n = ln * NS * Rr
        if plain:
            out.append((s["rings"][off:off + n].view(ln, NS, Rr).cpu().numpy(), None))
        else:
            pr = s["rings"].view(-1, 2)[off:off + n]
            out.append((pr[:, 0].reshape(ln, NS, Rr).cpu().numpy(), pr[:, 1].contiguous().view(torch.int32).reshape(ln, NS, Rr).cpu().numpy()))
        off += n
    return out


def _ref_logits(m, seq, **cond):
    key = (float(m.start_conv.weight.detach().abs().sum()), np.asarray(seq).tobytes(), tuple(sorted(cond)))
    if key not in _refs:
        _refs[key] = R.logits(R.weights(m.state_dict()), [d for d, _ in m.dilations], seq, **cond)
    return _refs[key]


def _errs(tag, got, want):
    whole, last = rel_err(got, want), rel_err(got[..., -500:, :], want[..., -500:, :])
    print(f"\n[{tag}] rel_err {whole:.3e}, last 500 {last:.3e}")
    assert np.isfinite(got).all() and whole < TOL and last < TOL, (tag, whole, last)


# ---------------------------------------------------------------------------------------------- rings
@pytest.mark.parametrize("case", KERNELS, ids=_ids(KERNELS))
def test_prefilled_rings_match_sequential_rings(golden, monkeypatch, case):
    """T = 700: past the 513-slot ring's first lap.  Sequential rings from evaluations [0, T), then prefilled ones."""
    _, mode, cs, ns, kid_want, cs_want = case
    m = _model(golden, monkeypatch, mode, cs)
    rt, T = m._runtime(), 700
    first = np.random.RandomState(200).randint(0, 256, (ns, T + 1)).astype(np.int32)
    with torch.cuda.device(rt.device()):
        s = rt.sampler(ns)
        stream = torch.cuda.current_stream().cuda_stream
        d_first = torch.from_numpy(first).cuda()
        d_out = torch.zeros(ns, 1, device="cuda", dtype=torch.int32)
        rt.reset_sampler(s, stream)
        rt.generate_resident(s, d_first, T + 1, 1, 0.0, 0.0, d_out, t0=0, n_evals=T, reset=False)
        kid, cs_ = _check_kernel(m, ns, kid_want, cs_want)
        seq = _rings(m, s, kid == 1)
        rt.reset_sampler(s, stream)
        rt.prefill(s, d_first, T)
        pre = _rings(m, s, kid == 1)
        torch.cuda.synchronize()
    assert rt.last_prefill["blocks"] == "tb"
    w = R.weights(m.state_dict())
    xs = {st: P.layer_inputs(w, CFG2_DIL, first[st, :T])[0] for st in sorted({0, ns - 1})}
    worst = 0.0
    for l, ((vs, ts), (vp, tp)) in enumerate(zip(seq, pre)):
        if ts is not None:
            assert np.array_equal(ts, tp), f"layer {l}: tags differ"
        if l == 0:
            assert np.array_equal(vs.view(np.int32), vp.view(np.int32)), "layer 0 values differ"
        ln = vs.shape[0]
        times = np.arange(max(0, T - ln), T)
        for st, x in xs.items():
            want = x[l][:, times].T
            worst = max(worst, rel_err(vp[times % ln, st], want))
            assert rel_err(vs[times % ln, st], want) < TOL
    print(f"\n[rings {case[0]}] kernel {kid} cluster {cs_}: prefilled ring values max rel err {worst:.3e} vs float64")
    assert worst < TOL


# ---------------------------------------------------------------------------------------------- teacher forcing
TF = [("k6", 6, None, 6, 16), ("k3", 3, None, 3, 0), ("k1", 1, None, 1, 0)]
PROMPTS = [2, 3, 514, 515, RF, RF + 1, RF + 2, 3 * RF + 18]       # n_given = T + 1 for T in {1, 2, 513, 514, rf-1, rf, rf+1, 3rf+17}


@pytest.mark.parametrize("case", TF, ids=_ids(TF))
def test_teacher_forced_after_prefill(golden, monkeypatch, case):
    _, mode, cs, kid_want, cs_want = case
    m = _model(golden, monkeypatch, mode, cs)
    rng = np.random.RandomState(201)
    N = 600
    seq = rng.randint(0, 256, 3 * RF + 18 + N)
    want_all = _ref_logits(m, seq)
    for ng in PROMPTS:
        first, forced = seq[None, :ng], seq[None, ng:ng + N]
        idx, lg = m.generate_fast_batch(N, first, temperature=0.0, forced=forced, return_logits=True, prefill=True)
        _check_kernel(m, 1, kid_want, cs_want)
        _errs(f"tf {case[0]} T={ng - 1}", lg[0], want_all[ng - 1:ng - 1 + N])
        assert np.array_equal(idx[0], lg[0].argmax(axis=1))


# ---------------------------------------------------------------------------------------------- free running, T = 0 / 1
@pytest.mark.parametrize("temperature", [1.0, 0.0])
@pytest.mark.parametrize("ng", [1, 2])
def test_free_running_against_sequential(golden, monkeypatch, ng, temperature):
    m = _model(golden, monkeypatch)
    rng = np.random.RandomState(202)
    n = 400
    first, uni = rng.randint(0, 256, (1, ng)), rng.random_sample((1, n))
    kw = dict(temperature=temperature, uniforms=uni if temperature > 0 else None, return_logits=True)
    i0, l0 = m.generate_fast_batch(n, first, prefill=False, **kw)
    i1, l1 = m.generate_fast_batch(n, first, prefill=True, **kw)
    for idx, lg in ((i0, l0), (i1, l1)):
        assert np.array_equal(R.choose(lg[0], temperature, 0.0, uni[0] if temperature > 0 else None)[0], idx[0])
    if ng == 1:                                            # T = 0: nothing to prefill
        assert np.array_equal(i0, i1) and np.array_equal(l0, l1)
        return
    bad = np.nonzero(i0[0] != i1[0])[0]
    if len(bad):
        j = int(bad[0])
        _, margin, edge = R.choose(l0[0][j:j + 1], temperature, 0.0, uni[0][j:j + 1] if temperature > 0 else None)
        assert (edge[0] < 1e-5) if temperature > 0 else (margin[0] < TOL * np.abs(l0[0][j]).max()), (j, margin, edge)
    print(f"\n[free T={ng - 1} temp {temperature}] first divergence: {int(bad[0]) if len(bad) else None}")


# ---------------------------------------------------------------------------------------------- batches
@pytest.mark.parametrize("ns", [8, 64, 120])
@pytest.mark.parametrize("cs", ["16", "8"])
def test_batched_prefill_equals_8_stream_prefill(golden, monkeypatch, ns, cs):
    m = _model(golden, monkeypatch, None, cs)
    rng = np.random.RandomState(203)
    n, T = 120, 900
    first = rng.randint(0, 256, (ns, T + 1))
    idx, lg = m.generate_fast_batch(n, first, temperature=0.0, return_logits=True, prefill=True)
    for g in range(0, ns, 8):
        i8, l8 = m.generate_fast_batch(n, first[g:g + 8], temperature=0.0, return_logits=True, prefill=True)
        assert np.array_equal(idx[g:g + 8], i8) and np.array_equal(lg[g:g + 8], l8), (ns, g)


# ---------------------------------------------------------------------------------------------- per-stream settings
PS = [("k2", 2, 2, 0), ("k4", 4, 4, 16), ("k6", 6, 6, 16)]


@pytest.mark.parametrize("case", PS, ids=_ids(PS))
def test_ragged_prompts_per_stream_settings(golden, monkeypatch, case):
    """Prompts of 700, 950 and 1 300 samples: 699 prefilled evaluations, the longer prompts' rest sequential."""
    _, mode, kid_want, cs_want = case
    m = _model(golden, monkeypatch, mode)
    rng = np.random.RandomState(204)
    lens, counts = [700, 950, 1300], [300, 200, 100]
    seqs = [rng.randint(0, 256, g + c) for g, c in zip(lens, counts)]
    first, forced = [q[:g] for q, g in zip(seqs, lens)], [q[g:] for q, g in zip(seqs, lens)]
    idx, lg = m.generate_fast_batch(counts, first, temperature=[0.0, 0.0, 0.0], regularize=[0.0, 1e-5, 0.0], forced=forced,
                                    return_logits=True, prefill=True)
    _check_kernel(m, 3, kid_want, cs_want)
    assert m._runtime().last_prefill["W"] == 699
    for st, (q, g, c) in enumerate(zip(seqs, lens, counts)):
        want = _ref_logits(m, R.inputs(q[:g], q[g:]))[g - 1:g - 1 + c]
        if st == 1:
            want = want - R.regularizer(256, 1e-5)[None, :]
        _errs(f"per-stream {case[0]} stream {st}", lg[st], want)


# ---------------------------------------------------------------------------------------------- conditioning
COND_KERNELS = [("k2", 2, 2), ("k3", 3, 3), ("k6", 6, 6)]


def _cond_model(kind):
    kw = dict(layers=10, blocks=1, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
              classes=256, output_length=16, kernel_size=2, bias=True)
    if kind == "global":
        kw.update(condition_channels=16)
    elif kind == "local":
        kw.update(local_condition_channels=8, local_condition_hop=80)
    else:
        kw.update(local_condition_channels=8, local_condition_hop=80, local_condition_upsample_scales=(4, 4, 5))
    torch.manual_seed(5)
    m = wmod.WaveNetModel(**kw)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "cond_convs" in n or "local_convs" in n or "local_upsample" in n:
                p.add_(0.05 * torch.randn_like(p))
    return m.cuda()


@pytest.mark.parametrize("kind", ["global", "local", "upsample"])
@pytest.mark.parametrize("case", COND_KERNELS, ids=_ids(COND_KERNELS))
def test_conditioned_prefill(monkeypatch, case, kind):
    """rf = 1 024; prompts of 1 501 samples: T = 1 500, and under repeat local conditioning P0 = 476 -> 400, are off the
    80-sample frames."""
    _, mode, kid_want = case
    m = _cond_model(kind)
    m._runtime().gen_mode = mode
    ns = 1 if mode == 3 else 2
    rng = np.random.RandomState(205)
    ng, n = 1501, 300
    seq = rng.randint(0, 256, (ns, ng + n))
    kw, ref_kw = {}, [{} for _ in range(ns)]
    if kind == "global":
        h = rng.randint(0, 16, ns)
        kw["condition"] = h
        ref_kw = [dict(h=np.eye(16)[h[s]]) for s in range(ns)]
    else:
        y = rng.standard_normal((ns, 8, -(-(ng + n) // 80))).astype(np.float32)
        kw["local_condition"] = y
        sc = (4, 4, 5) if kind == "upsample" else None
        ref_kw = [dict(y=y[s], hop=80, scales=sc) for s in range(ns)]
    idx, lg = m.generate_fast_batch(n, seq[:, :ng], temperature=0.0, forced=seq[:, ng:], return_logits=True, prefill=True,
                                    **kw)
    assert _kernel(m, ns)[0] == kid_want
    assert m._runtime().last_prefill["P0"] == (400 if kind == "local" else 476)     # the upsampled features are read at hop 1
    w = R.weights(m.state_dict())
    dil = [d for d, _ in m.dilations]
    for s in range(ns):
        want = R.logits(w, dil, R.inputs(seq[s, :ng], seq[s, ng:]), **ref_kw[s])[ng - 1:]
        _errs(f"cond {kind} {case[0]} stream {s}", lg[s], want)


# ---------------------------------------------------------------------------------------------- 512 channels
def test_512_channel_net_ffma_prefill():
    torch.manual_seed(6)
    m = wmod.WaveNetModel(layers=8, blocks=1, dilation_channels=512, residual_channels=512, skip_channels=512,
                          end_channels=256, classes=256, output_length=16, kernel_size=2, bias=True).cuda()
    m._runtime().gen_mode = 2
    rng = np.random.RandomState(206)
    ng, n = 600, 300
    seq = rng.randint(0, 256, ng + n)
    idx, lg = m.generate_fast_batch(n, seq[None, :ng], temperature=0.0, forced=seq[None, ng:], return_logits=True,
                                    prefill=True)
    assert _kernel(m, 1)[0] == 2 and m._runtime().last_prefill["blocks"] == "ffma"
    want = R.logits(R.weights(m.state_dict()), [d for d, _ in m.dilations], R.inputs(seq[:ng], seq[ng:]))[ng - 1:]
    _errs("512 channels k2", lg[0], want)


# ---------------------------------------------------------------------------------------------- state rules
def test_state_rules(golden, monkeypatch):
    m = _model(golden, monkeypatch)
    rt, lib = m._runtime(), native.lib()
    T = 300
    first = torch.from_numpy(np.random.RandomState(207).randint(0, 256, (1, T + 1)).astype(np.int32)).cuda()
    with torch.cuda.device(rt.device()):
        s = rt.sampler(1)
        h, stream = s["handle"], torch.cuda.current_stream().cuda_stream
        d_out = torch.zeros(1, 4, device="cuda", dtype=torch.int32)
        rt.reset_sampler(s, stream)
        rt.generate_resident(s, first, T + 1, 4, 0.0, 0.0, d_out, t0=0, n_evals=5, reset=False)
        buf = torch.zeros(1, 2 * T, 256, device="cuda")
        assert lib.wn_gen_prefill_layer(h, 0, buf.data_ptr(), native.GEN_SRC_FRAMES, 2 * T, 2 * T, T, stream) == -4
        rt.reset_sampler(s, stream)
        assert lib.wn_gen_prefill_layer(h, 0, buf.data_ptr(), native.GEN_SRC_FRAMES, 2 * T, 2 * T, T, stream) == 0
        assert lib.wn_gen_prefill_commit(h, T) == -4                     # the other layers are not filled
        rt.reset_sampler(s, stream)
        rt.prefill(s, first, T)
        a = native.GenRunArgs()
        a.d_first, a.n_given, a.d_out_idx, a.n_samples, a.t0, a.n_evals = first.data_ptr(), T + 1, d_out.data_ptr(), 4, 0, 1
        assert lib.wn_gen_run(h, ctypes.byref(a), stream) == -4          # t0 = 0 after a commit to T
        a.t0 = T
        assert lib.wn_gen_run(h, ctypes.byref(a), stream) == 0
        torch.cuda.synchronize()


def test_queues_after_prefill(golden, monkeypatch):
    """The exported queues of a prefilled call meet those of a sequential one at 1e-4; the queue step that follows (a new
    session from reset queues) is bit-identical."""
    m = _model(golden, monkeypatch)
    first = np.random.RandomState(208).randint(0, 256, 1200)
    col = torch.zeros(1, 256, 1)
    col[0, 17, 0] = 1.0
    out = {}
    for pf in (False, True):
        m.generate_fast(50, first, temperature=0.0, prefill=pf)
        qs = [(q.data.cpu().numpy().copy(), q.in_pos) for q in m.dilated_queues]
        out[pf] = (qs, m.wavenet(col.cuda(), dilation_func=m.queue_dilate).cpu().numpy())
    for (a, pa), (b, pb) in zip(out[False][0], out[True][0]):
        assert pa == pb and rel_err(b, a) < TOL
    assert np.array_equal(out[False][1], out[True][1])
