"""Top-k / nucleus (top-p) truncation in every sampler kernel (wn_gen_set_truncation), against the float64 rule of
truncation_ref.choose_truncated (pinned on the CPU by test_truncation_ref.py) applied to each kernel's own reported logits.

  a. free-running runs of 4 000 samples through kernels 1 to 6 (6 at clusters of 16 and 8) on cfg 2 and kernels 1, 2 at
     100 and 1 000 classes, at four (temperature, top_k, top_p) settings with and without the regularizer; uniforms with
     planted 0, 1 - 2^-53 and 1 (the only value whose count runs past the kept edges);
  b. exact identities, no tolerance: explicit off values, top_k = 1 and top_p = 1e-12 (= the argmax run), top_k >= classes;
  c. kernel 6 at 8, 64 and 120 streams: every stream equals itself in an 8-stream launch;
  d. global and local conditioning through kernel 6 (every gen_kernel_cl8 instantiation sees the flag);
  e. a net with end_conv_2 rows copied in pairs, so that exact logit ties at the k-th place occur.
Each case prints kernel, cluster size, streams, selections, near-edge counts and the logit error (pytest -s)."""
import numpy as np
import pytest
import torch

import sampler_ref as R
import truncation_ref as T
from helpers import build_model
from test_gpu_generate_long import CFG2_DIL, K256, TOL, _check_kernel, _class_model, _cond_model, _errs, _ids, _kernel, \
    _model, _ref

pytestmark = pytest.mark.gpu
SETTINGS = [(1.0, 40, 1.0), (1.0, 0, 0.9), (0.7, 50, 0.95), (1.3, 255, 0.999)]
NEAR = 1e-5


def _uniforms(rng, ns, n):
    uni = rng.random_sample((ns, n))
    uni[:, 5::397] = 0.0
    uni[:, 11::401] = 1.0 - 2.0 ** -53
    uni[:, 17::409] = 1.0
    return uni


def _selections(tag, idx, lg, uni, temperature, top_k, top_p):
    """The kernel's index against the rule on its own logits at every selection: equal, or the draw within NEAR of a CDF
    edge / the top-p prefix within NEAR of its threshold (under 1 % of the selections).  A chosen class outside the kept
    set fails, unless the top-p decision itself was within rounding (then the kernel's kept set may hold one more class).
    Returns (selections, near-edge disagreements)."""
    ns, n = idx.shape
    bad = close = outside = 0
    for s in range(ns):
        got, kept, edge, pgap = T.choose_truncated(lg[s], temperature, 0.0, uni[s], top_k, top_p)
        near = (edge < NEAR) | (pgap < NEAR)
        out = ~kept[np.arange(n), idx[s]]
        outside += int((out & ~(pgap < NEAR)).sum())
        bad += int(((got != idx[s]) & ~near).sum())
        close += int(((got != idx[s]) & near).sum())
    print(f"    [{tag}] {ns * n} selections, {close} within {NEAR:g} of an edge or threshold, {outside} outside the kept set, "
          f"{len(np.unique(idx))} distinct classes")
    assert outside == 0 and bad == 0 and close < 0.01 * ns * n, (tag, outside, bad, close)
    return ns * n, close


def _free_runs(tag, m, name, dil, mode, ns, n, ref_streams, settings=SETTINGS, regs=(0.0, 1e-4)):
    rt = m._runtime()
    rt.gen_mode = mode
    rng = np.random.RandomState(201)
    first = rng.randint(0, m.classes, (ns, 1))
    worst = 0.0
    for temperature, top_k, top_p in settings:
        for reg in regs:
            uni = _uniforms(rng, ns, n)
            idx, lg = m.generate_fast_batch(n, first, temperature=temperature, regularize=reg, uniforms=uni,
                                            return_logits=True, top_k=top_k, top_p=top_p)
            kid, cs = _kernel(m, ns)
            assert mode is None or kid == mode
            st = f"{tag} T={temperature} k={top_k} p={top_p} reg={reg}"
            _selections(st, idx, lg, uni, temperature, top_k, top_p)
            want = np.stack([_ref(name, m, dil, R.inputs(first[s], idx[s])) for s in ref_streams])
            whole, _ = _errs("trunc " + st, kid, cs, ns, n, lg[ref_streams] + R.regularizer(m.classes, reg), want)
            worst = max(worst, whole)
    rt.gen_mode = None
    return worst


# ---------------------------------------------------------------------------------------------- a. the rule, every kernel
A_CASES = [c for c in K256 if "noprefetch" not in c[0]]


@pytest.mark.parametrize("case", A_CASES, ids=_ids(A_CASES))
def test_rule_against_every_kernel_cfg2(golden, monkeypatch, case):
    m = _model(golden, monkeypatch, case)
    m.generate_fast_batch(2, np.zeros((1, 1), dtype=np.int64), temperature=0.0)
    _check_kernel(m, 1, case)
    _free_runs(case[0], m, "cfg2", CFG2_DIL, case[1], 1, 4000, [0])


@pytest.mark.parametrize("name,mode", [("c100", 1), ("c100", 2), ("c1000", 1), ("c1000", 2)])
def test_rule_at_other_class_counts(name, mode):
    """idle lanes (100 classes) and more than 8 classes per lane (1 000): the four settings (at 100 classes top_k = 255
    leaves only the top-p bound), plus top_k = classes - 1 and a small k with p = 0.5"""
    m = _class_model(name)
    _free_runs(f"{name} mode {mode}", m, name, [d for d, _ in m.dilations], mode, 1, 4000, [0],
               settings=SETTINGS + [(1.0, m.classes - 1, 1.0), (1.0, 3, 0.5)])


# ---------------------------------------------------------------------------------------------- b. exact identities
@pytest.mark.parametrize("case", A_CASES, ids=_ids(A_CASES))
def test_exact_identities(golden, monkeypatch, case):
    m = _model(golden, monkeypatch, case)
    n = 600
    rng = np.random.RandomState(202)
    first = rng.randint(0, 256, (1, 1))
    uni = _uniforms(rng, 1, n)
    run = lambda **kw: m.generate_fast_batch(n, first, uniforms=uni, return_logits=True, **kw)
    base_i, base_l = run(temperature=1.0)
    _check_kernel(m, 1, case)
    for kw in (dict(top_k=0, top_p=1.0), dict(top_k=256, top_p=1.0), dict(top_k=1000, top_p=1.0)):
        i, l = run(temperature=1.0, **kw)
        assert np.array_equal(i, base_i) and np.array_equal(l, base_l), (case[0], kw)
    arg_i, arg_l = run(temperature=0.0)
    for kw in (dict(top_k=1), dict(top_p=1e-12), dict(top_k=1, top_p=1e-12)):
        i, l = run(temperature=1.0, **kw)
        assert np.array_equal(i, arg_i) and np.array_equal(l, arg_l), (case[0], kw)
    i, l = run(temperature=0.0, top_k=5, top_p=0.5)                # no effect at temperature 0
    assert np.array_equal(i, arg_i) and np.array_equal(l, arg_l)
    _check_kernel(m, 1, case)


# ---------------------------------------------------------------------------------------------- c. many streams
@pytest.mark.parametrize("ns", [8, 64, 120])
def test_many_streams_truncated(golden, ns):
    m = build_model(golden("net_cfg2.npz"))
    n = 400
    rng = np.random.RandomState(203)
    first, uni = rng.randint(0, 256, (120, 1)), _uniforms(rng, 120, n)
    kw = dict(temperature=1.0, top_k=50, top_p=0.95, return_logits=True)
    idx, lg = m.generate_fast_batch(n, first[:ns], uniforms=uni[:ns], **kw)
    kid, cs = _kernel(m, ns)
    assert kid == 6
    for s0 in range(0, ns, 8):
        sub = slice(s0, min(s0 + 8, ns))
        i8, l8 = m.generate_fast_batch(n, first[sub], uniforms=uni[sub], **kw)
        assert np.array_equal(i8, idx[sub]) and np.array_equal(l8, lg[sub]), s0
    pick = sorted({0, 7, ns - 1} | set(np.random.RandomState(6).choice(ns, min(ns, 5), replace=False).tolist()))
    _selections(f"c {ns} streams", idx[pick], lg[pick], uni[pick], 1.0, 50, 0.95)
    want = np.stack([_ref("cfg2", m, CFG2_DIL, R.inputs(first[s], idx[s])) for s in pick])
    _errs(f"c {ns} streams, {len(pick)} checked", kid, cs, ns, n, lg[pick], want)


# ---------------------------------------------------------------------------------------------- d. conditioning
@pytest.mark.parametrize("kind", ["global", "global+repeat"])
@pytest.mark.parametrize("cs", ["16", "8"])
def test_conditioned_truncated(kind, cs, monkeypatch):
    monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    m = _cond_model(kind)
    n, ns = 1000, 3
    rng = np.random.RandomState(204)
    first = rng.randint(0, 256, (ns, 1))
    h = rng.randn(ns, 16).astype(np.float32)
    y = rng.randn(ns, 80, -(-n // 80)).astype(np.float32) if kind != "global" else None
    uni = _uniforms(rng, ns, n)
    idx, lg = m.generate_fast_batch(n, first, temperature=0.7, regularize=1e-4, uniforms=uni, return_logits=True,
                                    condition=h, local_condition=y, top_k=50, top_p=0.95)
    kid, ccs = _kernel(m, ns)
    assert kid == 6 and ccs == int(cs)
    _selections(f"d {kind} cluster {cs}", idx, lg, uni, 0.7, 50, 0.95)
    w = R.weights(m.state_dict())
    want = np.stack([R.logits(w, CFG2_DIL, R.inputs(first[s], idx[s]), h=h[s], y=None if y is None else y[s], hop=80)
                     for s in range(ns)])
    _errs(f"d {kind}", kid, ccs, ns, n, lg + R.regularizer(256, 1e-4), want)


# ---------------------------------------------------------------------------------------------- e. ties at the k-th place
@pytest.mark.parametrize("mode", [6, 3, 2, 1])
def test_ties_keep_the_lower_index(golden, mode):
    """end_conv_2 rows and biases copied in pairs (2j + 1 <- 2j): wherever a kernel computes the two rows identically the
    logits tie exactly, and with an odd top_k the k-th place often splits a pair.  The lower index must be kept."""
    m = build_model(golden("net_cfg2.npz"))
    with torch.no_grad():
        m.end_conv_2.weight[1::2] = m.end_conv_2.weight[0::2]
        m.end_conv_2.bias[1::2] = m.end_conv_2.bias[0::2]
    m._runtime().gen_mode = mode
    n, top_k = 2000, 41
    rng = np.random.RandomState(205)
    first, uni = rng.randint(0, 256, (1, 1)), _uniforms(rng, 1, n)
    idx, lg = m.generate_fast_batch(n, first, temperature=1.3, uniforms=uni, return_logits=True, top_k=top_k)
    assert _kernel(m, 1)[0] == mode
    srt = -np.sort(-lg[0], axis=1)
    tie_rows = np.flatnonzero(srt[:, top_k - 1] == srt[:, top_k])
    _, kept, _, _ = T.choose_truncated(lg[0], 1.3, 0.0, uni[0], top_k, 1.0)
    for r in tie_rows:                                           # of the tied classes at the k-th place, the lower is kept
        tied = np.flatnonzero(lg[0, r] == srt[r, top_k - 1])
        assert kept[r, tied[0]] and not kept[r, tied[-1]], r
    print(f"    [e mode {mode}] {n} selections, {len(tie_rows)} with an exact tie at place {top_k}")
    assert len(tie_rows) > 0
    _selections(f"e mode {mode}", idx, lg, uni, 1.3, top_k, 1.0)
