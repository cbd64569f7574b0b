"""Per-stream sampling (wn_gen_set_stream_params; generate_fast_batch with per-stream prompts, counts, temperature,
regularizer, top-k and top-p) on the cfg-2 net, against the uniform launches it must reproduce and the float64 references.

  a. a mixed launch of 11 streams -- temperature 0 and > 0, regularizer on and off, truncation off / top-k / top-p / both,
     prompts of 1, 2, 5, 600 and 5 200 samples (the receptive field is 5 116), 0 to 1 000 samples -- through kernels 1, 2,
     4 and 6 (clusters of 16 and of 8): every stream's indices and logits equal, bit for bit, those of an 11-stream uniform
     launch in which every stream carries that stream's prompt, uniforms and settings;
  b. on the same launch, every selection against truncation_ref / sampler_ref with the stream's own settings on the
     kernel's own logits, and the logits of four streams (the longest prompt included) against the float64 reference;
  c. identities: one value per stream in per-stream arrays gives the scalar call's bytes, and equal prompt lengths given
     as a ragged list give the rectangular call's bytes;
  d. teacher forcing with ragged prompts reads forced[s][e - n_given[s]];
  e. 120 streams on kernel 6 with random settings and ragged prompts: every stream equals itself in 8-stream launches;
  f. the public API on the default kernel: a seeded generate_fast_batch equals seeded generate_fast calls stream by
     stream, unconditioned, with global labels plus repeat local conditioning at hop 80, and through the learned
     upsampler (4, 4, 5) on series of different lengths;
  g. no leakage: after a per-stream call, a scalar call at the same stream count and a queue_dilate step give exactly
     what a fresh model gives.
Each case prints its kernel, cluster size, streams, evaluations and observed errors (pytest -s)."""
import numpy as np
import pytest
import torch

import sampler_ref as R
from audio_data import mu_law_expansion
from helpers import build_model
from test_gpu_generate_long import CFG2_DIL, K256, _check_kernel, _cond_model, _errs, _ids, _kernel, _model, _ref
from test_gpu_generate_truncated import _selections, _uniforms

pytestmark = pytest.mark.gpu

# kernels 1, 2, 4 and 6 at clusters of 16 and of 8
PS_CASES = [K256[i] for i in (6, 5, 2, 3, 4)]
# (temperature, regularize, top_k, top_p, prompt length, samples) of the 11 streams of the mixed launch
MIXED = [(0.0, 0.0, 0, 1.0, 1, 1000), (1.0, 0.0, 0, 1.0, 2, 700), (0.8, 1e-4, 50, 1.0, 5, 400),
         (1.2, 0.0, 0, 0.9, 600, 300), (1.0, 1e-4, 40, 0.95, 5200, 5), (0.0, 1e-4, 0, 1.0, 5, 0),
         (0.7, 0.0, 1, 1.0, 1, 250), (1.3, 0.0, 255, 0.999, 2, 1), (0.5, 1e-4, 0, 1.0, 600, 150),
         (1.0, 0.0, 10, 0.5, 1, 800), (0.0, 0.0, 5, 1.0, 2, 60)]
REF_STREAMS = (0, 3, 4, 8)


def _mixed_inputs():
    rng = np.random.RandomState(301)
    ns = len(MIXED)
    first = [rng.randint(0, 256, g) for *_, g, _ in MIXED]
    counts = [n for *_, n in MIXED]
    uni = _uniforms(rng, ns, max(counts))
    cols = list(zip(*MIXED))
    kw = dict(temperature=list(cols[0]), regularize=list(cols[1]), top_k=list(cols[2]), top_p=list(cols[3]))
    return first, counts, uni, kw


@pytest.mark.parametrize("case", PS_CASES, ids=_ids(PS_CASES))
def test_mixed_launch_equals_uniform_launches(golden, monkeypatch, case):
    m = _model(golden, monkeypatch, case)
    first, counts, uni, kw = _mixed_inputs()
    ns = len(first)
    idx, lg = m.generate_fast_batch(counts, first, uniforms=uni, return_logits=True, **kw)
    kid, cs = _check_kernel(m, ns, case)
    assert [len(i) for i in idx] == counts and [l.shape for l in lg] == [(n, 256) for n in counts]
    evals = max(len(f) - 1 + n for f, n in zip(first, counts))
    # b. every selection by the stream's own rule on the kernel's own logits
    for s, (t, reg, k, p, g, n) in enumerate(MIXED):
        if n == 0:
            continue
        if t > 0:
            _selections(f"b {case[0]} stream {s}", idx[s][None], lg[s][None], uni[s:s + 1, :n], t, k, p)
        else:
            assert np.array_equal(idx[s], lg[s].argmax(axis=1)), s
    for s in REF_STREAMS:
        t, reg, k, p, g, n = MIXED[s]
        want = _ref("cfg2", m, CFG2_DIL, R.inputs(first[s], idx[s]))[g - 1:]
        _errs(f"b {case[0]} stream {s} (prompt {g}, {n} samples)", kid, cs, ns, evals,
              lg[s] + R.regularizer(256, reg), want)
    # a. stream s against an 11-stream launch of copies of stream s (the scalar call)
    for s, (t, reg, k, p, g, n) in enumerate(MIXED):
        iu, lu = m.generate_fast_batch(n, np.stack([first[s]] * ns), temperature=t, regularize=reg, top_k=k, top_p=p,
                                       uniforms=np.stack([uni[s, :n]] * ns), return_logits=True)
        assert _kernel(m, ns) == (kid, cs)
        for r in (0, s, ns - 1):
            assert np.array_equal(iu[r], idx[s]) and np.array_equal(lu[r], lg[s]), (case[0], s, r)
    print(f"    [a {case[0]}] kernel {kid} cluster {cs}: {ns} streams, {evals} evaluations, every stream equals its "
          f"uniform launch")


@pytest.mark.parametrize("case", PS_CASES, ids=_ids(PS_CASES))
def test_identities_and_teacher_forcing(golden, monkeypatch, case):
    m = _model(golden, monkeypatch, case)
    rng = np.random.RandomState(302)
    ns, n = 3, 300
    first = rng.randint(0, 256, (ns, 4))
    uni = _uniforms(rng, ns, n)
    # c. one value per stream, as arrays, against the scalar call
    for t, reg, k, p in ((0.0, 0.0, 0, 1.0), (1.0, 1e-4, 0, 1.0), (0.9, 0.0, 40, 0.9)):
        i0, l0 = m.generate_fast_batch(n, first, temperature=t, regularize=reg, top_k=k, top_p=p, uniforms=uni,
                                       return_logits=True)
        i1, l1 = m.generate_fast_batch([n] * ns, first, temperature=[t] * ns, regularize=np.full(ns, reg),
                                       top_k=[k] * ns, top_p=torch.full((ns,), p, dtype=torch.float64), uniforms=uni,
                                       return_logits=True)
        assert np.array_equal(np.stack(i1), i0) and np.array_equal(np.stack(l1), l0), (case[0], t, reg, k, p)
        i2, l2 = m.generate_fast_batch(n, list(first), temperature=[t] * ns, regularize=reg, top_k=k, top_p=p,
                                       uniforms=list(uni), return_logits=True)
        assert np.array_equal(i2, i0) and np.array_equal(l2, l0), (case[0], t, reg, k, p)
    kid, cs = _check_kernel(m, ns, case)
    # d. teacher forcing with prompts of 1, 3 and 40: stream s reads forced[s][e - n_given[s]] after its prompt
    prompts = [rng.randint(0, 256, g) for g in (1, 3, 40)]
    counts = [200, 37, 120]
    forced = [rng.randint(0, 256, 250) for _ in range(ns)]
    idx, lg = m.generate_fast_batch(counts, prompts, temperature=0.0, forced=forced, return_logits=True)
    evals = max(len(f) - 1 + c for f, c in zip(prompts, counts))
    for s in range(ns):
        g, c = len(prompts[s]), counts[s]
        want = _ref("cfg2", m, CFG2_DIL, R.inputs(prompts[s], forced[s][:c]))[g - 1:]
        _errs(f"d {case[0]} stream {s} (prompt {g}, {c} forced)", kid, cs, ns, evals, lg[s], want)
        assert np.array_equal(idx[s], lg[s].argmax(axis=1))


def test_120_streams_equal_their_8_stream_launches(golden):
    m = build_model(golden("net_cfg2.npz"))
    ns = 120
    rng = np.random.RandomState(303)
    first = [rng.randint(0, 256, g) for g in rng.randint(1, 300, ns)]
    counts = rng.randint(0, 400, ns).tolist()
    uni = _uniforms(rng, ns, 400)
    kw = dict(temperature=np.where(rng.rand(ns) < 0.3, 0.0, rng.uniform(0.5, 1.5, ns)),
              regularize=np.where(rng.rand(ns) < 0.5, 0.0, 1e-4), top_k=rng.choice([0, 1, 10, 50, 255], ns),
              top_p=rng.choice([1.0, 0.5, 0.9, 0.99], ns))
    idx, lg = m.generate_fast_batch(counts, first, uniforms=uni, return_logits=True, **kw)
    kid, cs = _kernel(m, ns)
    assert kid == 6
    for s0 in range(0, ns, 8):
        sub = slice(s0, s0 + 8)
        i8, l8 = m.generate_fast_batch(counts[sub], first[sub], uniforms=uni[sub], return_logits=True,
                                       **{k: v[sub] for k, v in kw.items()})
        for j in range(8):
            assert np.array_equal(i8[j], idx[s0 + j]) and np.array_equal(l8[j], lg[s0 + j]), s0 + j
    print(f"    [e] kernel {kid} cluster {cs}: {ns} streams, {max(len(f) - 1 + c for f, c in zip(first, counts))} "
          f"evaluations, every stream equals itself in its 8-stream launch")


@pytest.mark.parametrize("kind", ["none", "global+repeat", "learned"])
def test_seeded_batch_equals_seeded_generate_fast_calls(golden, kind):
    m = build_model(golden("net_cfg2.npz")) if kind == "none" else _cond_model(kind)
    rng = np.random.RandomState(304)
    prompts = [rng.randint(0, 256, g) for g in (1, 7, 90, 3)]
    counts = [400, 0, 250, 130]
    # a temperature-0 stream draws nothing; stream 1 only warms up (generate_fast needs no uniforms for 0 samples then)
    settings = [(1.0, 0.0, 0, 1.0), (0.0, 0.0, 0, 1.0), (0.0, 1e-4, 0, 1.0), (0.9, 1e-4, 50, 0.95)]
    cond = dict()
    if kind != "none":
        hop = 80
        series = [rng.randn(80, -(-(len(f) - 1 + c) // hop) + e).astype(np.float32)
                  for f, c, e in zip(prompts, counts, (0, 2, 1, 0))]
        cond["local_condition"] = series
    if kind == "global+repeat":
        cond["condition"] = np.array([3, 0, 15, 7])
    t, reg, k, p = (list(c) for c in zip(*settings))
    np.random.seed(77)
    idx = m.generate_fast_batch(counts, prompts, temperature=t, regularize=reg, top_k=k, top_p=p, **cond)
    kid, cs = _kernel(m, 4)
    assert kid == 6
    np.random.seed(77)
    for s in range(4):
        one = {}
        if kind != "none":
            one["local_condition"] = cond["local_condition"][s]
        if kind == "global+repeat":
            one["condition"] = int(cond["condition"][s])
        audio = m.generate_fast(counts[s], first_samples=prompts[s], temperature=t[s], regularize=reg[s], top_k=k[s],
                                top_p=p[s], **one)
        want = mu_law_expansion((idx[s] / 256) * 2. - 1, 256)
        assert _kernel(m, 1)[0] == 6
        assert np.array_equal(audio, want), (kind, s)
    print(f"    [f {kind}] kernel {kid} cluster {cs}: 4 streams equal their seeded generate_fast calls")


def test_no_leakage_into_later_calls(golden):
    rng = np.random.RandomState(305)
    first, n = rng.randint(0, 256, (2, 3)), 200
    uni = rng.random_sample((2, n))
    x = torch.zeros(1, 256, 5)
    x[0, rng.randint(0, 256, 5), np.arange(5)] = 1.0

    def after(m):
        i, l = m.generate_fast_batch(n, first, temperature=1.0, uniforms=uni, return_logits=True)
        for q in m.dilated_queues:
            q.reset()
        y = m.wavenet(x.cuda(), dilation_func=m.queue_dilate)
        return i, l, y.detach().cpu().numpy()

    fresh = after(build_model(golden("net_cfg2.npz")))
    m = build_model(golden("net_cfg2.npz"))
    m.generate_fast_batch([n, 5], [first[0], first[1, :1]], temperature=[0.3, 0.0], regularize=[1e-3, 1e-4],
                          top_k=[3, 0], top_p=[0.5, 1.0], uniforms=uni)
    m.generate_fast_batch([7], [first[0, :2]], temperature=[0.4], regularize=[1e-3], top_k=[2], top_p=[0.5],
                          uniforms=uni[:1])                     # one stream: the handle queue_dilate uses
    got = after(m)
    for a, b in zip(got, fresh):
        assert np.array_equal(a, b)
