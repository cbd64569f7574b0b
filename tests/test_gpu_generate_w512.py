"""The batched tensor-core sampler (kernel 6, gen_kernel_cl8) on 512-wide nets (R = D = S = E = 512, 256 classes), the
width of the cfg-5 deep stack: a short seeded net (layers=10, blocks=2, receptive field 2 047, with and without biases)
against the float64 whole-sequence reference (sampler_ref), and the cfg-5 shape itself (80 layers) for the kernel choice
and one short run.

  1. kernel choice: wn_gen_kernel_id, cluster size and wn_gen_launch_info at 1, 8, 11, 64 and 120 streams (a 64-stream
     cfg-5 handle is created and runs);
  2. teacher-forced logits over 4 200 evaluations (two receptive fields: ring wrap, tags one lap old) at rel_err < 1e-4;
  3. launches ending at ring-boundary evaluations give the bits of one launch;
  4. every stream of a 64- and a 120-stream launch equals itself in an 8-stream launch, bit for bit;
  5. free-running selection, 4 000 samples: the kernel's index is the selection rule's on the kernel's own logits
     (temperature 0 and > 0, regularizer, top-k / top-p, uniforms at 0 and 1 - 2^-53);
  6. global (labels and dense), local (hop 80) and learned-upsampler conditioning against float64;
  7. a mixed generate_fast_batch equals uniform launches of each stream; a 4-slot session, with and without prefill,
     gives each job the bits of a static launch; a vocoder session (local_window);
  8. kernel 2 on the same net agrees with kernel 6 to the float64 bar.
Each case prints its kernel, cluster size, streams and errors (pytest -s)."""
import ctypes

import numpy as np
import pytest
import torch

import native
import sampler_ref as R
from helpers import rel_err
from test_gpu_generate_long import SPLITS, _errs, _kernel, _selection, _uniforms
from test_gpu_generate_session import _identity, _inputs, _session_kernel
from test_gpu_generate_truncated import _selections

pytestmark = pytest.mark.gpu
TOL = 1e-4
W512 = dict(dilation_channels=512, residual_channels=512, skip_channels=512, end_channels=512, classes=256,
            output_length=16, kernel_size=2)
SHORT_DIL = R.dilations_of(10, 2)                    # receptive field 2 047
CFG5_KW = dict(W512, layers=10, blocks=8, bias=False)

_models, _weights, _refs = {}, {}, {}


def _short(bias=False, **extra):
    """the seeded 20-layer 512-wide net, one per (bias, conditioning) and module"""
    key = (bias, tuple(sorted(extra.items())))
    if key not in _models:
        import wavenet_model as wmod
        torch.manual_seed(11 + bias)
        m = wmod.WaveNetModel(layers=10, blocks=2, bias=bias, **W512, **extra)
        if "local_condition_upsample_scales" in extra:
            with torch.no_grad():                    # away from exact repetition
                for p in m.local_upsample.parameters():
                    p.add_(0.05 * torch.randn(p.shape, generator=torch.Generator().manual_seed(8)))
        _models[key] = m.cuda()
    m = _models[key]
    m._runtime().gen_mode = 0                        # auto, also on handles a test ran in another mode
    return m


def _ref(m, seq, **cond):
    """float64 logits (T, 256) of one input sequence, once per module"""
    mk = id(m)
    if mk not in _weights:
        _weights[mk] = R.weights(m.state_dict())
    key = (mk, np.asarray(seq, dtype=np.int64).tobytes(),
           tuple((k, None if v is None else np.asarray(v).tobytes()) for k, v in sorted(cond.items())))
    if key not in _refs:
        _refs[key] = R.logits(_weights[mk], [d for d, _ in m.dilations], seq, **cond)
    return _refs[key]


def _info(m, ns):
    h = m._runtime().sampler(ns)["handle"]
    g, b, x = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    rc = native.lib().wn_gen_launch_info(h, ctypes.byref(g), ctypes.byref(b), ctypes.byref(x))
    return native.lib().wn_gen_kernel_id(h), rc, g.value, b.value, x.value


# ---------------------------------------------------------------------------------------------- 1. kernel choice
def test_kernel_choice_and_a_short_run_on_cfg5():
    """cfg 5 (80 layers of 512 channels): kernel 6 in clusters of 16 CTAs of 352 threads at every stream count, 162
    exchange stages per evaluation; 64 streams run 24 teacher-forced evaluations that meet the float64 reference."""
    import wavenet_model as wmod
    torch.manual_seed(5)
    m = wmod.WaveNetModel(**CFG5_KW).cuda()
    rng = np.random.RandomState(500)
    for ns in (1, 8, 11, 64, 120):
        first, forced = rng.randint(0, 256, (ns, 1)), rng.randint(0, 256, (ns, 3))
        m.generate_fast_batch(3, first, temperature=0.0, forced=forced)
        kid, rc, g, b, x = _info(m, ns)
        print(f"\n[1 cfg5] streams {ns}: kernel {kid}, grid {g}, block {b}, stages {x}, cluster {g // -(-ns // 8)}")
        assert (kid, rc, g, b, x) == (6, 0, -(-ns // 8) * 16, 352, 162), ns
        native.lib().wn_gen_destroy(m._runtime().samplers.pop(ns)["handle"])       # one 505 MB image at a time
    first, forced = rng.randint(0, 256, (64, 1)), rng.randint(0, 256, (64, 24))
    idx, lg = m.generate_fast_batch(24, first, temperature=0.0, forced=forced, return_logits=True)
    assert _info(m, 64)[0] == 6
    pick = [0, 7, 56, 63]
    want = np.stack([_ref(m, R.inputs(first[s], forced[s])) for s in pick])
    _errs("1 cfg5 short run", 6, 16, 64, 24, lg[pick], want)
    assert np.array_equal(idx, lg.argmax(axis=2))


@pytest.mark.parametrize("ns", [1, 8, 11, 64, 120])
def test_kernel_choice_short_net(ns):
    m = _short()
    m.generate_fast_batch(2, np.zeros((ns, 1), np.int64), temperature=0.0)
    kid, rc, g, b, x = _info(m, ns)
    assert (kid, rc, g, b, x) == (6, 0, -(-ns // 8) * 16, 352, 42), ns


def test_cluster_size_8_is_not_taken_at_512(monkeypatch):
    """WN_GEN_CL8_CS=8 only applies where clusters of 8 fit: 512-wide nets keep clusters of 16"""
    monkeypatch.setenv("WN_GEN_CL8_CS", "8")
    m = _short()
    if 64 in m._runtime().samplers:                  # the environment is read when a handle is created
        native.lib().wn_gen_destroy(m._runtime().samplers.pop(64)["handle"])
    m.generate_fast_batch(2, np.zeros((64, 1), np.int64), temperature=0.0)
    assert _info(m, 64)[:3] == (6, 0, 128)
    native.lib().wn_gen_destroy(m._runtime().samplers.pop(64)["handle"])


# ---------------------------------------------------------------------------------------------- 2, 8. float64 parity
@pytest.mark.parametrize("mode", [6, 2], ids=["k6", "k2"])
@pytest.mark.parametrize("bias", [False, True], ids=["nobias", "bias"])
def test_teacher_forced_past_two_receptive_fields(bias, mode):
    """1 given and 4 200 forced samples (2.05 receptive fields, 4 laps of the 513-slot rings), 1 and 8 streams, kernel 6
    and kernel 2 on the same net, against float64"""
    m = _short(bias)
    m._runtime().gen_mode = mode
    rng = np.random.RandomState(201 + bias)
    first, forced = rng.randint(0, 256, (8, 1)), rng.randint(0, 256, (8, 4200))
    for ns in (1, 8):
        idx, lg = m.generate_fast_batch(4200, first[:ns], temperature=0.0, forced=forced[:ns], return_logits=True)
        kid, cs = _kernel(m, ns)
        assert kid == mode
        pick = [0] if ns == 1 else [0, 7]
        want = np.stack([_ref(m, R.inputs(first[s], forced[s])) for s in pick])
        _errs(f"2 bias={bias}", kid, cs, ns, 4200, lg[pick], want)
        assert np.array_equal(idx, lg.argmax(axis=2))
    m._runtime().gen_mode = 0


# ---------------------------------------------------------------------------------------------- 3. launch splits
def test_launch_boundaries_on_ring_laps():
    """4 400 evaluations in launches that end around the laps of the 129- and 513-slot rings and at the receptive field
    (2 047): bit-identical to one launch"""
    m = _short()
    rt = m._runtime()
    rng = np.random.RandomState(203)
    n = 4398
    first, forced, uni = rng.randint(0, 256, (1, 3)).astype(np.int32), rng.randint(0, 256, (1, n)), rng.random_sample((1, n))
    splits = tuple(e for e in SPLITS if e < 2100) + (2046, 2047, 2048, 4094)
    calls = []
    with torch.cuda.device(rt.device()):
        a, la, ta = rt.generate(n, first, 1.0, 0.0, uniforms=uni, forced=forced, want_logits=True,
                                callbacks=[(e, lambda: calls.append(1)) for e in splits])
        b, lb, tb = rt.generate(n, first, 1.0, 0.0, uniforms=uni, forced=forced, want_logits=True)
    kid, cs = _kernel(m, 1)
    assert kid == 6 and ta == tb == n + 2 and len(calls) == len(splits)
    assert np.array_equal(a, b) and np.array_equal(la.view(np.uint32), lb.view(np.uint32))
    want = _ref(m, R.inputs(first, forced))[2:]
    _errs("3 splits", kid, cs, 1, n + 2, lb[0], want)


# ---------------------------------------------------------------------------------------------- 4. stream independence
@pytest.mark.parametrize("ns", [64, 120])
def test_every_stream_equals_itself_in_an_8_stream_launch(ns):
    m = _short(True)
    rng = np.random.RandomState(204)
    first, uni = rng.randint(0, 256, (ns, 700)), rng.random_sample((ns, 300))
    idx, lg = m.generate_fast_batch(300, first, temperature=1.0, uniforms=uni, return_logits=True)
    assert _kernel(m, ns) == (6, 16)
    for s0 in range(0, ns, 8):
        sub = slice(s0, s0 + 8)
        i8, l8 = m.generate_fast_batch(300, first[sub], temperature=1.0, uniforms=uni[sub], return_logits=True)
        assert np.array_equal(i8, idx[sub]) and np.array_equal(l8.view(np.uint32), lg[sub].view(np.uint32)), s0
    pick = [0, 7, ns - 8, ns - 1]
    want = np.stack([_ref(m, R.inputs(first[s], idx[s]))[699:] for s in pick])
    _errs(f"4 streams {pick}", 6, 16, ns, 999, lg[pick], want)


# ---------------------------------------------------------------------------------------------- 5. selection
@pytest.mark.parametrize("ns", [1, 8])
def test_selection_thousands_of_times(ns):
    m = _short(True)
    _selection(f"w512 mode 6 streams {ns}", m, "w512-bias", SHORT_DIL, 6, ns, 4000, [0] if ns == 1 else [0, 7])


@pytest.mark.parametrize("top_k,top_p", [(40, 1.0), (0, 0.9), (20, 0.95)])
def test_truncated_selection(top_k, top_p):
    m = _short()
    rng = np.random.RandomState(205)
    ns, n = 8, 4000
    first, uni = rng.randint(0, 256, (ns, 1)), _uniforms(rng, ns, n)
    idx, lg = m.generate_fast_batch(n, first, temperature=1.2, uniforms=uni, top_k=top_k, top_p=top_p,
                                    return_logits=True)
    assert _kernel(m, ns)[0] == 6
    _selections(f"5 top_k={top_k} top_p={top_p}", idx, lg, uni, 1.2, top_k, top_p)


# ---------------------------------------------------------------------------------------------- 6. conditioning
@pytest.mark.parametrize("kind", ["labels", "dense", "local", "learned"])
def test_conditioning_against_float64(kind):
    extra = {"labels": dict(condition_channels=16), "dense": dict(condition_channels=16),
             "local": dict(local_condition_channels=80, local_condition_hop=80),
             "learned": dict(local_condition_channels=80, local_condition_hop=80,
                             local_condition_upsample_scales=(4, 4, 5))}[kind]
    m = _short(**extra)
    rng = np.random.RandomState(206)
    ns, n, ng = 8, 1298, 3
    first, forced = rng.randint(0, 256, (ns, ng)), rng.randint(0, 256, (ns, n))
    labels = rng.randint(0, 16, ns)
    h = {"labels": np.eye(16, dtype=np.float32)[labels], "dense": rng.randn(ns, 16).astype(np.float32)}.get(kind)
    y = rng.randn(ns, 80, -(-1300 // 80)).astype(np.float32) if kind in ("local", "learned") else None
    scales = extra.get("local_condition_upsample_scales")
    idx, lg = m.generate_fast_batch(n, first, temperature=0.0, forced=forced, return_logits=True,
                                    condition=labels if kind == "labels" else h, local_condition=y)
    kid, cs = _kernel(m, ns)
    assert kid == 6
    pick = [0, 7]
    want = np.stack([_ref(m, R.inputs(first[s], forced[s]), h=None if h is None else h[s], y=None if y is None else y[s],
                          hop=80, scales=scales)[ng - 1:] for s in pick])
    _errs(f"6 {kind}", kid, cs, ns, ng - 1 + n, lg[pick], want)


# ---------------------------------------------------------------------------------------------- 7. per-stream jobs, sessions
def test_mixed_batch_equals_uniform_launches():
    """ragged prompts and per-stream settings in one 11-stream launch; each stream equals an 11-stream launch carrying
    its job in every stream"""
    m = _short(True)
    rng = np.random.RandomState(207)
    ns, n = 11, 600
    prompts = [rng.randint(0, 256, int(g)) for g in rng.choice([1, 2, 300, 2100], ns)]
    temps = rng.choice([0.0, 0.8, 1.0], ns)
    regs = rng.choice([0.0, 1e-4], ns)
    top_k = rng.choice([0, 20], ns)
    top_p = rng.choice([1.0, 0.9], ns)
    counts = rng.randint(1, n + 1, ns)
    uni = rng.random_sample((ns, n))
    idx, lg = m.generate_fast_batch(counts, prompts, temperature=temps, regularize=regs, top_k=top_k, top_p=top_p,
                                    uniforms=uni, return_logits=True)
    assert _kernel(m, ns)[0] == 6
    for s in range(ns):
        i1, l1 = m.generate_fast_batch(int(counts[s]), np.stack([prompts[s]] * ns), temperature=float(temps[s]),
                                       regularize=float(regs[s]), top_k=int(top_k[s]), top_p=float(top_p[s]),
                                       uniforms=np.stack([uni[s, :counts[s]]] * ns), return_logits=True)
        c = int(counts[s])
        assert np.array_equal(idx[s][:c], i1[0]) and np.array_equal(lg[s][:c].view(np.uint32), l1[0].view(np.uint32)), s


JOBS = [(600, 500, 1.0, 0.0, 0, 1.0), (1, 700, 0.0, 1e-4, 0, 1.0), (2100, 300, 0.8, 0.0, 40, 0.95),
        (2, 1, 1.2, 0.0, 0, 0.9), (2, 0, 1.0, 0.0, 0, 1.0), (1, 600, 0.7, 1e-4, 10, 1.0), (2, 400, 1.0, 0.0, 0, 1.0)]


@pytest.mark.parametrize("prefill", [False, True], ids=["seq", "prefill"])
def test_session_equals_static_launches(prefill):
    m = _short(True)
    first, uni = _inputs(208, JOBS)
    sess = m.sampling_session(4, prefill=prefill, return_logits=True)
    got, kid = _identity("7 w512", m, sess, 4, first, uni, JOBS, prefill)
    assert kid == 6
    g, n, t, r, *_ = JOBS[2]
    idx, lg = got[2]
    want = _ref(m, R.inputs(first[2], idx))[g - 1:]
    _errs("7 job 2 (prompt 2100)", kid, 16, 4, g - 1 + n, lg + R.regularizer(256, r), want)


def test_vocoder_session():
    """a locally conditioned 512-wide net in a 4-slot session (local_window 300): each job equals its static launch"""
    m = _short(local_condition_channels=80, local_condition_hop=80)
    rng = np.random.RandomState(209)
    jobs = [(1, 500, 1.0, 0.0, 0, 1.0), (300, 200, 0.0, 0.0, 0, 1.0), (2, 700, 0.9, 1e-4, 0, 0.95),
            (1, 300, 1.0, 0.0, 20, 1.0), (5, 400, 1.0, 0.0, 0, 1.0)]
    first, uni = _inputs(210, jobs)
    ys = [rng.randn(80, -(-(g + n) // 80) + 1).astype(np.float32) for g, n, *_ in jobs]
    sess = m.sampling_session(4, return_logits=True, local_window=300)
    ids = [sess.submit(f, n, temperature=t, regularize=r, top_k=k, top_p=p, uniforms=u, local_condition=y)
           for f, u, y, (_, n, t, r, k, p) in zip(first, uni, ys, jobs)]
    k = 0
    while sess.pending or sess.active:
        sess.step((1, 7, 513, 1000)[k % 4])
        k += 1
    assert _session_kernel(sess) == 6
    for j, (f, u, y, (_, n, t, r, kk, p)) in enumerate(zip(first, uni, ys, jobs)):
        idx, lg = sess.result(ids[j])
        si, sl = m.generate_fast_batch(n, np.stack([f] * 4), temperature=t, regularize=r, top_k=kk, top_p=p,
                                       uniforms=None if u is None else np.stack([u] * 4), return_logits=True,
                                       local_condition=np.stack([y] * 4))
        assert np.array_equal(idx, si[0]) and np.array_equal(lg.view(np.uint32), sl[0].view(np.uint32)), j
    print(f"\n[7 vocoder] kernel 6 slots 4: {len(jobs)} jobs in {k} steps")


# ---------------------------------------------------------------------------------------------- 8. kernel 2 cross-check
@pytest.mark.parametrize("ns", [1, 8, 30])
def test_kernel_2_agrees_with_kernel_6(ns):
    m = _short(True)
    rng = np.random.RandomState(211)
    first, forced = rng.randint(0, 256, (ns, 1)), rng.randint(0, 256, (ns, 2200))
    out = {}
    for mode in (6, 2):
        m._runtime().gen_mode = mode
        idx, lg = m.generate_fast_batch(2200, first, temperature=0.0, forced=forced, return_logits=True)
        assert _kernel(m, ns)[0] == mode
        out[mode] = lg
    m._runtime().gen_mode = 0
    err = rel_err(out[6], out[2])
    print(f"\n[8 k2 vs k6] streams {ns}: rel_err {err:.3e}")
    assert err < TOL
