"""Sampling sessions (continuous batching: WaveNetModel.sampling_session, wn_gen_set_stream_positions, wn_gen_seat_layer) on
the cfg-2 net, against the static launches every job must reproduce and the float64 reference.

  1. identity: a session of N slots serves a seeded sequence of jobs with ragged prompts (1, 2, 600 and 5 200 samples; the
     receptive field is 5 116) and counts (0, 1, up to 1 000), mixed temperature, regularizer, top-k and top-p, in steps of
     1, 7, 513 and 1 000 evaluations; every job's indices and logits equal, bit for bit, an N-stream generate_fast_batch
     launch carrying that job in every stream (same uniforms, same prefill), through kernels 6 (clusters of 16 and 8), 4, 2
     and 1, with prefill off and on;
  2. reused slots, built on purpose: jobs join slots whose previous job ran more than 513 evaluations (longer than the
     longest ring), some with prompts shorter than that job's rings -- a seat that left one old slot time in place would
     hand the new job the old job's history, which the identity catches;
  3. the logits of three jobs (the 5 200-sample prompt included) against the float64 sampler_ref at 1e-4;
  4. 120 slots on kernel 6 at clusters of 8;
  5. global conditioning per job, labels and dense vectors, a slot passing between jobs of different labels;
  6. seeded submits with uniforms=None equal seeded generate_fast calls in the same order;
  7. the ABI's argument and state errors, a locally conditioned model, a parameter change;
  8. no leakage: after a session the model's own sampler calls and a queue_dilate step give what a fresh model gives.
Each case prints its kernel, slots and steps (pytest -s)."""
import ctypes

import numpy as np
import pytest
import torch

import native
import sampler_ref as R
from audio_data import mu_law_expansion
from helpers import build_model
from test_gpu_generate_long import CFG2_DIL, K256, _cond_model, _errs, _ids, _model, _ref

pytestmark = pytest.mark.gpu

# kernels 6 at clusters of 16 and of 8, 4, 2 and 1
S_CASES = [K256[i] for i in (3, 4, 2, 5, 6)]
STEPS = (1, 7, 513, 1000)
# (prompt length, samples, temperature, regularize, top_k, top_p), submitted in this order to 4 slots:
#   jobs 0-3 fill the slots; job 3 ends after two evaluations, job 4 (0 samples) is done at admission and job 5 takes slot 3;
#   job 1 runs 700 evaluations (> 513, the longest ring) and gives slot 1 to job 6, whose prompt of 2 samples is shorter
#   than most of job 1's rings; job 2 (5 200-sample prompt, 5 499 evaluations) gives slot 2 to job 7, another 5 200-sample
#   prompt, and job 0 gives slot 0 to job 8 (one sample of prompt)
JOBS = [(600, 1000, 1.0, 0.0, 0, 1.0), (1, 700, 0.0, 1e-4, 0, 1.0), (5200, 300, 0.8, 0.0, 40, 0.95),
        (2, 1, 1.2, 0.0, 0, 0.9), (2, 0, 1.0, 0.0, 0, 1.0), (1, 600, 0.7, 1e-4, 10, 1.0),
        (2, 500, 1.0, 0.0, 0, 1.0), (5200, 40, 0.0, 0.0, 0, 1.0), (1, 300, 1.0, 1e-4, 255, 0.999)]
REF_JOBS = (0, 2, 6)


def _inputs(seed=501, jobs=JOBS):
    rng = np.random.RandomState(seed)
    first = [rng.randint(0, 256, g) for g, *_ in jobs]
    uni = [rng.random_sample(n) if t > 0 else None for (_, n, t, *_) in jobs]
    return first, uni


def _serve(sess, first, uni, jobs, steps=STEPS, cond=None):
    ids = [sess.submit(f, n, temperature=t, regularize=r, top_k=k, top_p=p, uniforms=u,
                       condition=None if cond is None else cond[j])
           for j, (f, u, (_, n, t, r, k, p)) in enumerate(zip(first, uni, jobs))]
    k = 0
    while sess.pending or sess.active:
        sess.step(steps[k % len(steps)])
        k += 1
    return [sess.result(i) for i in ids], k


def _static(m, N, f, u, job, prefill, cond=None):
    """the job in every stream of one N-stream generate_fast_batch launch"""
    _, n, t, r, k, p = job
    return m.generate_fast_batch(n, np.stack([f] * N), temperature=t, regularize=r, top_k=k, top_p=p,
                                 uniforms=None if u is None else np.stack([u] * N), return_logits=True, prefill=prefill,
                                 condition=None if cond is None else np.stack([cond] * N))


def _session_kernel(sess):
    return native.lib().wn_gen_kernel_id(sess.s["handle"])


def _identity(tag, m, sess, N, first, uni, jobs, prefill, check=None, cond=None):
    got, n_steps = _serve(sess, first, uni, jobs, cond=cond)
    kid = _session_kernel(sess)
    print(f"\n[{tag}] kernel {kid} slots {N} prefill {prefill}: {len(jobs)} jobs in {n_steps} steps, t = {sess.t}")
    for j, (f, u, job) in enumerate(zip(first, uni, jobs)):
        if check is not None and j not in check:
            continue
        idx, lg = got[j]
        assert idx.shape == (job[1],) and lg.shape == (job[1], 256), j
        if job[1] == 0:                                  # done at admission: nothing to compare
            continue
        si, sl = _static(m, N, f, u, job, prefill, cond=None if cond is None else cond[j])
        assert np.array_equal(idx, si[0]), (tag, j)
        assert np.array_equal(lg.view(np.uint32), sl[0].view(np.uint32)), (tag, j)
    return got, kid


@pytest.mark.parametrize("prefill", [False, True], ids=["seq", "prefill"])
@pytest.mark.parametrize("case", S_CASES, ids=_ids(S_CASES))
def test_session_equals_static_launches(golden, monkeypatch, case, prefill):
    m = _model(golden, monkeypatch, case)
    N = 4
    first, uni = _inputs()
    sess = m.sampling_session(N, prefill=prefill, return_logits=True)
    got, kid = _identity(case[0], m, sess, N, first, uni, JOBS, prefill)
    assert kid == case[3]
    if case[0] == "k6-cs16":
        for j in REF_JOBS:                                 # 3. against float64
            g, n, t, r, *_ = JOBS[j]
            idx, lg = got[j]
            want = _ref("cfg2", m, CFG2_DIL, R.inputs(first[j], idx))[g - 1:]
            _errs(f"3 job {j} (prompt {g}, {n} samples)", kid, 16, N, g - 1 + n, lg + R.regularizer(256, r), want)


def test_session_120_slots_cluster_8(golden, monkeypatch):
    m = _model(golden, monkeypatch, K256[4])
    N = 120
    rng = np.random.RandomState(77)
    jobs = [(int(rng.choice([1, 2, 600])), int(rng.randint(0, 300)), float(rng.choice([0.0, 1.0])), 0.0,
             int(rng.choice([0, 20])), 1.0) for _ in range(150)]
    jobs[0] = (5200, 200, 1.0, 1e-4, 0, 0.9)
    first, uni = _inputs(78, jobs)
    sess = m.sampling_session(N, prefill=True, return_logits=True)
    _identity("4 k6-cs8", m, sess, N, first, uni, jobs, True, check=(0, 1, 130, 149))
    assert _session_kernel(sess) == 6


@pytest.mark.parametrize("dense", [False, True], ids=["labels", "dense"])
def test_session_global_conditioning(dense):
    m = _cond_model("global")
    N = 4
    jobs = JOBS[:1] + [(2, 300, 1.0, 0.0, 0, 1.0), (600, 200, 0.0, 0.0, 0, 1.0), (1, 1, 1.0, 0.0, 0, 1.0),
                       (1, 400, 0.9, 0.0, 0, 1.0), (2, 100, 1.0, 0.0, 0, 1.0)]
    first, uni = _inputs(9, jobs)
    rng = np.random.RandomState(10)
    cond = [rng.randn(16).astype(np.float32) for _ in jobs] if dense else [np.int64(j % 16) for j in range(len(jobs))]
    sess = m.sampling_session(N, prefill=True, return_logits=True)
    _identity("5 " + ("dense" if dense else "labels"), m, sess, N, first, uni, jobs, True, cond=cond)


def test_seeded_submits_equal_generate_fast(golden):
    m = build_model(golden("net_cfg2.npz"))
    jobs = [(3, 200, 1.0), (1, 50, 0.0), (40, 120, 0.8)]
    rng = np.random.RandomState(12)
    first = [rng.randint(0, 256, g) for g, *_ in jobs]
    np.random.seed(1234)
    sess = m.sampling_session(4)
    ids = [sess.submit(f, n, temperature=t) for f, (_, n, t) in zip(first, jobs)]
    while sess.pending or sess.active:
        sess.step(97)
    np.random.seed(1234)
    for i, f, (_, n, t) in zip(ids, first, jobs):
        want = m.generate_fast(n, f, temperature=t)
        assert np.array_equal(mu_law_expansion((sess.result(i) / 256) * 2. - 1, 256), want)


def test_session_errors(golden):
    m = build_model(golden("net_cfg2.npz"))
    lib = native.lib()
    sess = m.sampling_session(2)
    sess.submit([1, 2], 10, temperature=0.0)
    sess.step(3)
    h, t = sess.s["handle"], sess.t
    with pytest.raises(ValueError):
        sess.submit([1], 5, temperature=float("nan"))
    with pytest.raises(ValueError):
        sess.submit([1], 5, top_k=-1)
    with pytest.raises(ValueError):
        sess.submit([1], -1)
    with pytest.raises(ValueError):
        sess.submit([1], 5, temperature=1.0, uniforms=np.zeros(3))
    with pytest.raises(ValueError):
        sess.step(0)
    d_first = torch.zeros(2, 4, dtype=torch.int32, device="cuda")
    d_out = torch.zeros(2, 8, dtype=torch.int32, device="cuda")

    def run(origin, sample0=0, first0=0, n_evals=4, n_given=1):
        pos = (native.GenStreamPos * 2)(native.GenStreamPos(origin, sample0, first0), native.GenStreamPos(origin, 0, 0))
        native.check(lib.wn_gen_set_stream_positions(h, pos), "positions")
        a = native.GenRunArgs()
        a.d_first, a.n_given, a.d_out_idx, a.n_samples, a.t0, a.n_evals = d_first.data_ptr(), 4, d_out.data_ptr(), 8, t, n_evals
        return lib.wn_gen_run(h, ctypes.byref(a), None)

    recs = (native.GenStreamParams * 2)(*[native.GenStreamParams(3, 0, 0.0, 0.0, 1.0)] * 2)
    native.check(lib.wn_gen_set_stream_params(h, recs), "params")
    assert run(t + 1) == -1                                   # origin after t0
    assert run(t - 1) == -4                                   # origin changed, not seated
    slots, qe = (ctypes.c_int * 2)(0, 1), (ctypes.c_int * 2)(0, 0)
    assert lib.wn_gen_seat_layer(h, 0, 2, (ctypes.c_int * 2)(0, 0), qe, None, 0, 1, 0, None) == -1   # slot listed twice
    assert lib.wn_gen_seat_layer(h, 0, 2, (ctypes.c_int * 2)(0, 2), qe, None, 0, 1, 0, None) == -1   # slot out of range
    for l in range(m.layers * m.blocks - 1):
        native.check(lib.wn_gen_seat_layer(h, l, 2, slots, qe, None, 0, 1, 0, None), "seat")
    assert run(t) == -4                                       # the last layer was not seated
    native.check(lib.wn_gen_seat_layer(h, m.layers * m.blocks - 1, 2, slots, qe, None, 0, 1, 0, None), "seat")
    assert run(t, first0=1) == -1                             # prompt read before the row
    assert run(t, n_evals=11) == -1                           # selection column past n_samples
    assert run(t, sample0=1) == -1                            # selection column below 0
    assert run(t) == 0
    native.check(lib.wn_gen_check(h, None), "check")
    assert lib.wn_gen_set_stream_positions(h, (native.GenStreamPos * 2)(*[native.GenStreamPos(0, -1, 0)] * 2)) == -1
    native.check(lib.wn_gen_set_stream_params(h, None), "params")
    assert lib.wn_gen_set_stream_positions(h, (native.GenStreamPos * 2)(*[native.GenStreamPos(0, 0, 0)] * 2)) == -4
    # the first evaluation of a newly seated stream must read a prompt sample: q_end 5 with a 3-sample prompt
    native.check(lib.wn_gen_set_stream_params(h, recs), "params")
    t = t + 4
    for l in range(m.layers * m.blocks):
        native.check(lib.wn_gen_seat_layer(h, l, 2, slots, (ctypes.c_int * 2)(5, 5), None, 0, 1, 0, None), "seat")
    assert run(t - 5) == -1
    with pytest.raises(ValueError):
        _cond_model("global+repeat").sampling_session(2)
    sess2 = m.sampling_session(2)
    sess2.submit([1], 5)
    with torch.no_grad():
        m.end_conv_2.bias.add_(0.0)
    with pytest.raises(RuntimeError):
        sess2.step(5)
    with pytest.raises(RuntimeError):
        sess.reset()                                          # a job is still active


def test_no_leakage(golden):
    fresh = build_model(golden("net_cfg2.npz"))
    m = build_model(golden("net_cfg2.npz"))
    first, uni = _inputs(3)
    sess = m.sampling_session(4, prefill=True)
    _serve(sess, first[:4], uni[:4], JOBS[:4], steps=(300,))
    rng = np.random.RandomState(4)
    f = rng.randint(0, 256, (4, 30))
    u = rng.random_sample((4, 200))
    for model in (m, fresh):
        model._got = (model.generate_fast_batch(200, f, temperature=1.0, uniforms=u, return_logits=True),
                      model.generate_fast(100, f[0], temperature=0.0))
    assert np.array_equal(m._got[0][0], fresh._got[0][0]) and np.array_equal(m._got[0][1], fresh._got[0][1])
    assert np.array_equal(m._got[1], fresh._got[1])
    x = torch.zeros(1, 256, 1, device="cuda")
    x[0, 7, 0] = 1
    a = m.wavenet(x, dilation_func=m.queue_dilate)
    b = fresh.wavenet(x, dilation_func=fresh.queue_dilate)
    assert torch.equal(a, b)
