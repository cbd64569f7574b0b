"""Every sampler kernel against the float64 whole-sequence reference (tests/sampler_ref.py, pinned on the CPU by
test_sampler_ref.py) on runs longer than the receptive field.  The cfg-2 net has dilations 1..512 and a receptive field of
5 116; in a run of 48 evaluations from reset rings every layer of dilation >= 64 multiplies a zero history, so the history
tap at t >= dil, the ring wrap at ring_len = dil + 1, the tag of a slot written one lap earlier and the ring position of
a launch that continues at a large t0 only meet a reference here.

All comparisons with the reference are teacher-forced (rounding cannot fork a stream, every evaluation is comparable)
at rel_err < 1e-4 over the whole run and over its last 500 evaluations; each case prints one line with the kernel,
cluster size, streams, evaluations and the two observed errors (pytest -s)."""
import ctypes

import numpy as np
import pytest
import torch

import sampler_ref as R
from helpers import build_model, rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4
CFG2_DIL = R.dilations_of(10, 5)
CFG2_KW = dict(layers=10, blocks=5, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
               classes=256, output_length=16, kernel_size=2, bias=False)

# (id, gen_mode, WN_GEN_CL8_CS, kernel that must run, other environment)
K256 = [("default", None, None, 6, {}), ("k3", 3, None, 3, {}), ("k4", 4, None, 4, {}),
        ("k6-cs16", 6, "16", 6, {}), ("k6-cs8", 6, "8", 6, {}), ("k2", 2, None, 2, {}), ("k1", 1, None, 1, {}),
        ("k3-noprefetch", 3, None, 3, {"WN_GEN_NOPREFETCH": "1"}), ("k2-noprefetch", 2, None, 2, {"WN_GEN_NOPREFETCH": "1"})]
_ids = lambda cases: [c[0] for c in cases]

_weights, _refs = {}, {}


def _w(name, m):
    """float64 weights of a net, once per module"""
    if name not in _weights:
        _weights[name] = R.weights(m.state_dict())
    return _weights[name]


def _ref(name, m, dil, seq, **cond):
    """reference logits (T, classes) of one input sequence, computed once per module"""
    key = (name, np.asarray(seq, dtype=np.int64).tobytes())
    if key not in _refs:
        _refs[key] = R.logits(_w(name, m), dil, seq, **cond)
    return _refs[key]


def _model(golden, monkeypatch, case, name="net_cfg2.npz"):
    """A fresh model per case: the environment is read when its sampler handle is created."""
    _, mode, cs, _, env = case
    if cs is not None:
        monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    m = build_model(golden(name))
    m._runtime().gen_mode = mode
    return m


def _kernel(m, ns):
    """(kernel id, CTAs per cluster or 0) of the sampler handle that served the last ns-stream run"""
    import native
    h = m._runtime().sampler(ns)["handle"]
    kid = native.lib().wn_gen_kernel_id(h)
    g, b, x = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    native.check(native.lib().wn_gen_launch_info(h, ctypes.byref(g), ctypes.byref(b), ctypes.byref(x)), "launch info")
    return kid, (g.value // -(-ns // 8) if kid == 6 else 16 if kid == 4 else 0)


def _check_kernel(m, ns, case):
    kid, cs = _kernel(m, ns)
    assert kid == case[3], f"case {case[0]} ran kernel {kid}"
    if case[2] is not None:
        assert cs == int(case[2]), f"case {case[0]} ran clusters of {cs}"
    return kid, cs


def _errs(tag, kid, cs, ns, evals, got, want):
    """the bar, over the whole run and over its last 500 evaluations; got / want (..., n, classes)"""
    whole, last = rel_err(got, want), rel_err(got[..., -500:, :], want[..., -500:, :])
    print(f"\n[{tag}] kernel {kid} cluster {cs} streams {ns} evaluations {evals}: rel_err {whole:.3e}, last 500 {last:.3e}")
    assert np.isfinite(got).all() and whole < TOL and last < TOL, (tag, kid, cs, whole, last)
    return whole, last


# ---------------------------------------------------------------------------------------------- a. past the receptive field
@pytest.mark.parametrize("case", K256, ids=_ids(K256))
def test_every_256_wide_kernel_past_the_receptive_field(golden, monkeypatch, case):
    """One given sample and 6 400 forced ones: 1.25 receptive fields, 12 laps of the deepest ring (513 slots)."""
    m = _model(golden, monkeypatch, case)
    rng = np.random.RandomState(101)
    first, forced = rng.randint(0, 256, (1, 1)), rng.randint(0, 256, (1, 6400))
    idx, lg = m.generate_fast_batch(6400, first, temperature=0.0, forced=forced, return_logits=True)
    kid, cs = _check_kernel(m, 1, case)
    want = _ref("cfg2", m, CFG2_DIL, R.inputs(first, forced))
    _errs("a " + case[0], kid, cs, 1, 6400, lg[0], want)
    assert np.array_equal(idx[0], lg[0].argmax(axis=1))            # the reported choice is the argmax of the reported logits


# ---------------------------------------------------------------------------------------------- b. long warm-up
B_CASES = [K256[i] for i in (0, 1, 2, 4, 5)]


@pytest.mark.parametrize("case", B_CASES, ids=_ids(B_CASES))
def test_head_switches_on_after_a_long_warm_up(golden, monkeypatch, case):
    """5 200 given samples, then 300: the warm-up evaluations run without the head for more than a receptive field."""
    m = _model(golden, monkeypatch, case)
    rng = np.random.RandomState(102)
    first, forced = rng.randint(0, 256, (1, 5200)), rng.randint(0, 256, (1, 300))
    idx, lg = m.generate_fast_batch(300, first, temperature=0.0, forced=forced, return_logits=True)
    kid, cs = _check_kernel(m, 1, case)
    want = _ref("cfg2", m, CFG2_DIL, R.inputs(first, forced))[5199:]
    _errs("b " + case[0], kid, cs, 1, 5499, lg[0], want)
    assert np.array_equal(idx[0], lg[0].argmax(axis=1))


# ---------------------------------------------------------------------------------------------- c. launch boundaries
C_CASES = [K256[i] for i in (1, 2, 3, 4, 5)]
SPLITS = (0, 1, 127, 128, 129, 511, 512, 513, 514, 1025, 1026, 5115, 5116)


@pytest.mark.parametrize("case", C_CASES, ids=_ids(C_CASES))
def test_launch_boundaries_on_ring_laps(golden, monkeypatch, case):
    """5 400 evaluations in 14 launches that end around the laps of the 129-, 513-slot rings and at the receptive field:
    each continuing launch recomputes its ring positions from t0.  Bit-identical to the single launch, which meets the
    reference.  Three given samples (the head switches on inside the third launch), sampling with temperature."""
    m = _model(golden, monkeypatch, case)
    rt = m._runtime()
    rng = np.random.RandomState(103)
    n = 5398
    first, forced, uni = rng.randint(0, 256, (1, 3)).astype(np.int32), rng.randint(0, 256, (1, n)), rng.random_sample((1, n))
    calls = []
    with torch.cuda.device(rt.device()):
        a, la, ta = rt.generate(n, first, 1.0, 0.0, uniforms=uni, forced=forced, want_logits=True,
                                callbacks=[(e, lambda: calls.append(1)) for e in SPLITS])
        b, lb, tb = rt.generate(n, first, 1.0, 0.0, uniforms=uni, forced=forced, want_logits=True)
    kid, cs = _check_kernel(m, 1, case)
    assert ta == tb == 5400 and len(calls) == len(SPLITS)
    assert np.array_equal(a, b) and np.array_equal(la, lb)
    want = _ref("cfg2", m, CFG2_DIL, R.inputs(first, forced))[2:]
    _errs("c " + case[0], kid, cs, 1, 5400, lb[0], want)
    got, _, edge = R.choose(lb[0], 1.0, 0.0, uni[0])
    assert np.all(edge[got != b[0]] < 1e-5) and (got != b[0]).mean() < 0.01


# ---------------------------------------------------------------------------------------------- d. many streams
@pytest.mark.parametrize("ns", [11, 64, 120])
def test_many_streams_two_laps_deep(golden, ns):
    """The default kernel with 11, 64 and 120 streams, each its own sequence: 1 100 given samples (two laps of the deepest
    ring) and 100 forced ones.  Every stream equals, bit for bit, the same stream in an 8-stream launch; the first and
    last slot of the first and last clusters and five seeded others meet the reference."""
    m = build_model(golden("net_cfg2.npz"))
    rng = np.random.RandomState(104)
    first, forced = rng.randint(0, 256, (120, 1100)), rng.randint(0, 256, (120, 100))
    idx, lg = m.generate_fast_batch(100, first[:ns], temperature=0.0, forced=forced[:ns], return_logits=True)
    kid, cs = _kernel(m, ns)
    assert kid == 6
    for s0 in range(0, ns, 8):
        sub = slice(s0, min(s0 + 8, ns))
        i8, l8 = m.generate_fast_batch(100, first[sub], temperature=0.0, forced=forced[sub], return_logits=True)
        assert np.array_equal(i8, idx[sub]) and np.array_equal(l8, lg[sub]), s0
    pick = sorted({0, 7, 8, 15, 63, 64, 119} | set(np.random.RandomState(5).choice(120, 5, replace=False).tolist()))
    pick = [s for s in pick if s < ns]
    want = np.stack([_ref("cfg2", m, CFG2_DIL, R.inputs(first[s], forced[s]))[1099:] for s in pick])
    _errs(f"d {len(pick)} of the streams", kid, cs, ns, 1199, lg[pick], want)
    assert np.array_equal(idx, lg.argmax(axis=2))


# ---------------------------------------------------------------------------------------------- e. generic kernels, odd shapes
_class_models = {}


def _class_model(name):
    """seeded nets with class counts other than 256 ("c100", "c257", "c1000"): ragged channels, biases everywhere"""
    if name not in _class_models:
        import wavenet_model as wmod
        with torch.random.fork_rng(devices=[]):
            torch.manual_seed(int(name[1:]))
            _class_models[name] = wmod.WaveNetModel(layers=4, blocks=2, dilation_channels=24, residual_channels=20,
                                                    skip_channels=40, end_channels=72, classes=int(name[1:]),
                                                    output_length=8, kernel_size=2, bias=True).cuda()
    return _class_models[name]


@pytest.mark.parametrize("name", ["k3", "odd_bias", "deep", "c100", "c257", "c1000"])
def test_generic_kernels_on_odd_shapes(golden, name):
    """kernel_size 3 (rings of 2 dil + 1 slots, two history taps), biases on every convolution with ragged channel
    counts, a deeper net, and class counts other than 256 (the selection step with idle lanes and with more than 8
    classes per lane): 3 streams, three receptive fields from one given sample.  With biases a reset queue (zeros) is not
    the layers' response to silence; the reference models the queue.  On the class-count nets each of modes 1 to 4 either
    runs its kernel or refuses the shape, and kernels 1 and 2 must run."""
    m = _class_model(name) if name[0] == "c" else build_model(golden(f"net_{name}.npz"))
    C = m.classes
    dil = [d for d, _ in m.dilations]
    n = 3 * m.receptive_field
    rng = np.random.RandomState(105)
    first, forced = rng.randint(0, C, (3, 1)), rng.randint(0, C, (3, n))
    forced[:, 7], forced[:, 8] = 0, C - 1
    want = np.stack([_ref(name, m, dil, R.inputs(first[s], forced[s])) for s in range(3)])
    ran = []
    for mode in ((1, 2, 3, 4) if name[0] == "c" else (None, 1, 2, 4)):
        for ns in (1, 3):
            m._runtime().gen_mode = mode
            try:
                idx, lg = m.generate_fast_batch(n, first[:ns], temperature=0.0, forced=forced[:ns], return_logits=True)
            except RuntimeError as e:
                assert "does not apply" in str(e) or "flag exchange" in str(e) or "need a cluster" in str(e), e
                continue
            kid, cs = _kernel(m, ns)
            assert mode in (None, 2) or kid == mode
            ran.append(kid)
            _errs(f"e {name} mode {mode}", kid, cs, ns, n, lg, want[:ns])
            assert np.array_equal(idx, lg.argmax(axis=2))
    m._runtime().gen_mode = None
    assert 1 in ran and len(set(ran)) >= 2, ran
    if name[0] == "c":
        assert {1, 2} <= set(ran), ran


# ---------------------------------------------------------------------------------------------- f. conditioned
def _cond_model(kind):
    import wavenet_model as wmod
    torch.manual_seed(7)
    kw = dict(CFG2_KW)
    if kind in ("global", "global+repeat"):
        kw["condition_channels"] = 16
    if kind in ("global+repeat", "learned"):
        kw.update(local_condition_channels=80, local_condition_hop=80)
    if kind == "learned":
        kw["local_condition_upsample_scales"] = (4, 4, 5)
    m = wmod.WaveNetModel(**kw)
    if kind == "learned":
        with torch.no_grad():                       # away from exact repetition
            for p in m.local_upsample.parameters():
                p.add_(0.05 * torch.randn(p.shape, generator=torch.Generator().manual_seed(8)))
    return m.cuda()


@pytest.mark.parametrize("kind", ["global", "global+repeat", "learned"])
def test_conditioned_sampling_over_windows_and_frames(kind, monkeypatch):
    """cfg-2 shape with a 16-channel global and / or an 80-channel local condition at hop 80 (repeated, or through the
    learned upsampler of scales 4, 4, 5): 1 300 evaluations, so 17 frames and two laps of the deepest ring.  The table
    window is set to 3 frames for the repeat model and to 43 evaluations for the hop-1 table of the learned upsampler
    (windows end at 129 = one lap of the 129-slot ring, and off every lap elsewhere); the result is that of the
    default window bit for bit and meets the reference at every evaluation, the last row of each window included."""
    n, ng = 1298, 3
    rng = np.random.RandomState(106)
    first, forced = rng.randint(0, 256, (3, ng)), rng.randint(0, 256, (3, n))
    h = rng.randn(3, 16).astype(np.float32) if kind != "learned" else None
    y = rng.randn(3, 80, -(-1300 // 80)).astype(np.float32) if kind != "global" else None
    scales = (4, 4, 5) if kind == "learned" else None
    want = None
    for cs in ("16", "8"):
        monkeypatch.setenv("WN_GEN_CL8_CS", cs)
        m = _cond_model(kind)
        if want is None:
            w = R.weights(m.state_dict())
            want = np.stack([R.logits(w, CFG2_DIL, R.inputs(first[s], forced[s]), h=None if h is None else h[s],
                                      y=None if y is None else y[s], hop=80, scales=scales)[ng - 1:] for s in range(3)])
        rt = m._runtime()
        for mode in ((3, 2, 6) if cs == "16" else (6,)):
            for ns in (1, 3):
                rt.gen_mode = mode
                kw = dict(temperature=0.0, forced=forced[:ns], return_logits=True,
                          condition=None if h is None else h[:ns], local_condition=None if y is None else y[:ns])
                rt.local_table_bytes = 256 << 20
                try:
                    idx, lg = m.generate_fast_batch(n, first[:ns], **kw)
                except RuntimeError as e:
                    assert "does not apply" in str(e) and mode == 3 and ns == 3, e
                    continue
                kid, ccs = _kernel(m, ns)
                assert kid == mode and (kid != 6 or ccs == int(cs))
                _errs(f"f {kind} mode {mode}", kid, ccs, ns, 1300, lg, want[:ns])
                if y is not None:
                    per_row = 50 * ns * 2 * 256 * 4                       # bytes of one table row: layers x streams x 2D floats
                    rt.local_table_bytes = per_row * (43 if scales else 3)
                    i2, l2 = m.generate_fast_batch(n, first[:ns], **kw)
                    assert np.array_equal(i2, idx) and np.array_equal(l2, lg), (kind, mode, ns)
        rt.gen_mode = None


# ---------------------------------------------------------------------------------------------- g. the selection step
SETTINGS = [(0.0, 0.0), (0.0, 1e-4), (0.5, 0.0), (1.0, 1e-4)]


def _uniforms(rng, ns, n):
    uni = rng.random_sample((ns, n))
    uni[:, 5::397] = 0.0
    uni[:, 11::401] = 1.0 - 2.0 ** -53
    return uni


def _selection(tag, m, name, dil, mode, ns, n, ref_streams):
    """Free-running runs at every setting: the kernel's index is what the selection rule gives on the kernel's own
    logits at every step (bar a draw within 1e-5 of a CDF edge or an argmax margin below 1e-4 of the logit scale), and
    the logits of the produced stream meet the reference."""
    rt = m._runtime()
    rt.gen_mode = mode
    rng = np.random.RandomState(107)
    first = rng.randint(0, m.classes, (ns, 1))
    for temperature, regularize in SETTINGS:
        uni = _uniforms(rng, ns, n)
        idx, lg = m.generate_fast_batch(n, first, temperature=temperature, regularize=regularize, uniforms=uni,
                                        return_logits=True)
        kid, cs = _kernel(m, ns)
        assert kid == mode
        scale = np.abs(lg).max()
        bad = close = 0
        for s in range(ns):
            got, margin, edge = R.choose(lg[s], temperature, 0.0, uni[s])        # the kernel reports logits - regularizer
            near = margin < TOL * scale if edge is None else edge < 1e-5
            bad += int(((got != idx[s]) & ~near).sum())
            close += int(((got != idx[s]) & near).sum())
        assert bad == 0 and close < 0.01 * ns * n, (tag, temperature, regularize, bad, close)
        reg = R.regularizer(m.classes, regularize).astype(np.float64)
        want = np.stack([_ref(name, m, dil, R.inputs(first[s], idx[s])) for s in ref_streams])
        whole, last = _errs(f"g {tag} T={temperature} reg={regularize}", kid, cs, ns, n, lg[ref_streams] + reg, want)
        print(f"    {ns * n} selections, {close} within rounding of an edge, {len(np.unique(idx))} distinct classes chosen")
    rt.gen_mode = None


@pytest.mark.parametrize("mode,ns", [(3, 1), (6, 1), (6, 8)])
def test_selection_thousands_of_times_cfg2(golden, mode, ns):
    m = build_model(golden("net_cfg2.npz"))
    _selection(f"cfg2 mode {mode}", m, "cfg2", CFG2_DIL, mode, ns, 4000, [0] if ns == 1 else [0, 7])


def test_selection_thousands_of_times_odd_bias(golden):
    m = build_model(golden("net_odd_bias.npz"))
    _selection("odd_bias mode 2", m, "odd_bias", [d for d, _ in m.dilations], 2, 1, 4000, [0])


@pytest.mark.parametrize("name", ["c100", "c1000"])
def test_selection_at_other_class_counts(name):
    """the selection step with idle lanes (100 classes) and with more than 8 classes per lane (1 000), free running at
    every setting (temperature 1 included) with uniforms at 0 and at 1 - 2^-53"""
    m = _class_model(name)
    _selection(f"{name} mode 2", m, name, [d for d, _ in m.dilations], 2, 1, 3000, [0])
