"""Sampling sessions of locally conditioned models (per-stream frame windows: wn_gen_set_condition_stream_frames,
SamplingSession(local_window=)) on the cfg-2 net with an 80-channel local condition at hop 80, repeated ("global+repeat",
with a 16-channel global condition too) or through the learned (4, 4, 5) upsampler ("learned").

  1. identity: a 4-slot session serves ragged jobs (prompts of 1, 2, 600 and 5 200 samples, each with its own series) in
     steps of 1, 7, 513 and 1 000 evaluations, with slots reused after runs longer than the 513-slot ring and windows of
     3 frames (repeat) or 43 evaluations (learned), so windows roll mid-step and mid-frame; every job's indices and logits
     equal, bit for bit, a per-stream generate_fast_batch launch carrying that job in every stream, through kernels 6
     (clusters of 16 and 8), 4, 2 and 1, with prefill off and on.  Some job sits at an origin that is not a multiple of the
     hop: a kernel that read frames by global time would fail here.  A second session with a large window agrees;
  2. three jobs' logits against the float64 sampler_ref at 1e-4;
  3. 120 slots on kernel 6 at clusters of 8;
  4. a table row built by wn_cond_table_frames is the same bits in two window placements;
  5. the ABI's argument and state errors; 6. the session API's argument errors.
Each case prints its kernel, slots and steps (pytest -s)."""
import ctypes

import numpy as np
import pytest
import torch

import native
import sampler_ref as R
from helpers import build_model
from test_gpu_generate_long import CFG2_DIL, K256, _cond_model, _errs, _ids

pytestmark = pytest.mark.gpu

S_CASES = [K256[i] for i in (3, 4, 2, 5, 6)]        # kernels 6 at clusters of 16 and of 8, 4, 2 and 1
STEPS = (1, 7, 513, 1000)
HOP = 80
WINDOW = {"global+repeat": 3 * HOP, "learned": 43}
# (prompt length, samples, temperature, regularize, top_k, top_p), submitted in this order to 4 slots: job 3 ends after two
# evaluations and job 4 takes slot 3 at t = 514 (an origin 34 past a frame edge); job 1 runs 700 evaluations (> 513) and
# gives slot 1 to job 5 (a 2-sample prompt); job 2 (5 200-sample prompt) gives slot 2 to job 6, another 5 200-sample
# prompt, and job 0 gives slot 0 to job 7
JOBS = [(600, 700, 1.0, 0.0, 0, 1.0), (1, 700, 0.0, 1e-4, 0, 1.0), (5200, 200, 0.8, 0.0, 40, 0.95),
        (2, 1, 1.2, 0.0, 0, 0.9), (1, 500, 0.7, 1e-4, 10, 1.0), (2, 400, 1.0, 0.0, 0, 1.0),
        (5200, 30, 0.0, 0.0, 0, 1.0), (1, 300, 1.0, 1e-4, 255, 0.999)]
REF_JOBS = (0, 2, 4)


def _inputs(seed, jobs, kind):
    rng = np.random.RandomState(seed)
    first = [rng.randint(0, 256, g) for g, *_ in jobs]
    uni = [rng.random_sample(n) if t > 0 else None for (_, n, t, *_) in jobs]
    # each job's series holds just the frames it needs: later slots read zeros past its end
    ys = [rng.randn(80, max(1, -(-(g - 1 + n) // HOP))).astype(np.float32) for g, n, *_ in jobs]
    hs = [rng.randn(16).astype(np.float32) for _ in jobs] if kind == "global+repeat" else [None] * len(jobs)
    return first, uni, ys, hs


def _serve(sess, first, uni, ys, hs, jobs, steps=STEPS):
    origins = {}
    seat = sess._seat

    def recording_seat(seats, stream):
        seat(seats, stream)
        for b, job in seats:
            if job is not None:
                origins[job.id] = sess.origin[b]
    sess._seat = recording_seat
    ids = [sess.submit(f, n, temperature=t, regularize=r, top_k=k, top_p=p, uniforms=u, local_condition=y, condition=h)
           for f, u, y, h, (_, n, t, r, k, p) in zip(first, uni, ys, hs, jobs)]
    k = 0
    while sess.pending or sess.active:
        sess.step(steps[k % len(steps)])
        k += 1
    return [sess.result(i) for i in ids], [origins.get(i) for i in ids], k


def _static(m, N, f, u, y, h, job, prefill):
    """the job in every stream of one per-stream N-stream generate_fast_batch launch"""
    _, n, t, r, k, p = job
    idx, lg = m.generate_fast_batch([n] * N, [f] * N, temperature=[t] * N, regularize=[r] * N, top_k=[k] * N,
                                    top_p=[p] * N, uniforms=None if u is None else [u] * N, return_logits=True,
                                    prefill=prefill, local_condition=[y] * N,
                                    condition=None if h is None else np.stack([h] * N))
    return idx[0], lg[0]


def _model(monkeypatch, case, kind):
    _, mode, cs, _, env = case
    if cs is not None:
        monkeypatch.setenv("WN_GEN_CL8_CS", cs)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    m = _cond_model(kind)
    m._runtime().gen_mode = mode
    return m


def _identity(tag, m, sess, N, inputs, jobs, prefill, check=None, steps=STEPS):
    first, uni, ys, hs = inputs
    got, origins, n_steps = _serve(sess, first, uni, ys, hs, jobs, steps)
    kid = native.lib().wn_gen_kernel_id(sess.s["handle"])
    print(f"\n[{tag}] kernel {kid} slots {N} prefill {prefill} window {sess.window}: {len(jobs)} jobs in {n_steps} steps, "
          f"t = {sess.t}, origins mod {HOP}: {sorted({o % HOP for o in origins if o is not None})}")
    for j, job in enumerate(jobs):
        if check is not None and j not in check:
            continue
        idx, lg = got[j]
        assert idx.shape == (job[1],) and lg.shape == (job[1], 256), j
        si, sl = _static(m, N, first[j], uni[j], ys[j], hs[j], job, prefill)
        assert np.array_equal(idx, si), (tag, j)
        assert np.array_equal(lg.view(np.uint32), sl.view(np.uint32)), (tag, j)
    return got, origins, kid


@pytest.mark.parametrize("kind", ["global+repeat", "learned"])
@pytest.mark.parametrize("prefill", [False, True], ids=["seq", "prefill"])
@pytest.mark.parametrize("case", S_CASES, ids=_ids(S_CASES))
def test_local_session_equals_static_launches(monkeypatch, case, prefill, kind):
    m = _model(monkeypatch, case, kind)
    N = 4
    inputs = _inputs(601, JOBS, kind)
    sess = m.sampling_session(N, prefill=prefill, return_logits=True, local_window=WINDOW[kind])
    got, origins, kid = _identity(f"1 {case[0]} {kind}", m, sess, N, inputs, JOBS, prefill)
    assert kid == case[3]
    assert any(o is not None and o % HOP != 0 for o in origins), origins
    if case[0] == "k6-cs16":
        # a window covering whole steps gives the same bits
        big = m.sampling_session(N, prefill=prefill, return_logits=True, local_window=1000)
        got2, _, _ = _serve(big, *inputs, JOBS)
        for j in range(len(JOBS)):
            assert np.array_equal(got2[j][0], got[j][0]) and np.array_equal(got2[j][1].view(np.uint32),
                                                                             got[j][1].view(np.uint32)), j
        # 2. against float64
        first, _, ys, hs = inputs
        w = R.weights(m.state_dict())
        scales = (4, 4, 5) if kind == "learned" else None
        for j in REF_JOBS:
            g, n, t, r, *_ = JOBS[j]
            idx, lg = got[j]
            want = R.logits(w, CFG2_DIL, R.inputs(first[j], idx), h=hs[j], y=ys[j], hop=HOP, scales=scales)[g - 1:]
            _errs(f"2 {kind} job {j} (prompt {g}, {n} samples)", kid, 16, N, g - 1 + n, lg + R.regularizer(256, r), want)


def test_local_session_120_slots_cluster_8(monkeypatch):
    m = _model(monkeypatch, K256[4], "global+repeat")
    N = 120
    rng = np.random.RandomState(77)
    jobs = [(int(rng.choice([1, 2, 600])), int(rng.randint(1, 300)), float(rng.choice([0.0, 1.0])), 0.0,
             int(rng.choice([0, 20])), 1.0) for _ in range(150)]
    jobs[0] = (5200, 200, 1.0, 1e-4, 0, 0.9)
    sess = m.sampling_session(N, prefill=True, return_logits=True, local_window=200)
    _identity("3 k6-cs8", m, sess, N, _inputs(78, jobs, "global+repeat"), jobs, True, check=(0, 1, 130, 149),
              steps=(97, 513))
    assert native.lib().wn_gen_kernel_id(sess.s["handle"]) == 6


def test_table_rows_independent_of_window_placement():
    m = _cond_model("global+repeat")
    rt = m._runtime()
    stream = torch.cuda.current_stream().cuda_stream
    W = rt.packed_weights(stream)
    rng = np.random.RandomState(3)
    y = torch.from_numpy(rng.randn(5, 80, 12).astype(np.float32)).cuda()
    h = torch.from_numpy(rng.randn(5, 16).astype(np.float32)).cuda()
    a = W.cond_table_frames(h, y, 0, 10, stream)                      # frames [0, 10)
    b = W.cond_table_frames(h, y, 3, 9, stream)                       # frames [3, 12)
    c = W.cond_table_frames(h[[3, 1]], y[[3, 1], :, 5:].contiguous(), 0, 4, stream)   # a session's gather: [5, 9)
    out = torch.empty(m.layers * m.blocks, 2, 4, 512, device="cuda")
    d = W.cond_table_frames(h[[3, 1]], y[[3, 1], :, 5:].contiguous(), 0, 4, stream, out=out)
    assert d is out and torch.equal(c, d)
    assert torch.equal(a[:, :, 3:10], b[:, :, 0:7])
    assert torch.equal(a[:, [3, 1], 5:9], c)


def _handle(m, N):
    rt = m._runtime()
    s = rt.new_sampler(N)
    stream = torch.cuda.current_stream().cuda_stream
    rt.reset_sampler(s, stream)
    return s, stream


def test_local_abi_errors():
    m = _cond_model("global+repeat")
    lib, N, nl = native.lib(), 2, m.layers * m.blocks
    rt = m._runtime()
    rng = np.random.RandomState(4)
    stream = torch.cuda.current_stream().cuda_stream
    y = torch.from_numpy(rng.randn(N, 80, 2).astype(np.float32)).cuda()
    h = torch.from_numpy(rng.randn(N, 16).astype(np.float32)).cuda()
    tab = rt.packed_weights(stream).cond_table_frames(h, y, 0, 2, stream)      # frames [0, 2) of both streams
    d_first = torch.zeros(N, 4, dtype=torch.int32, device="cuda")
    recs = (native.GenStreamParams * N)(*[native.GenStreamParams(4, 0, 0.0, 0.0, 1.0)] * N)
    f0s = lambda *v: (ctypes.c_int * N)(*v)

    def run(s, t0, n, logits=None):
        a = native.GenRunArgs()
        a.d_first, a.n_given, a.n_samples, a.t0, a.n_evals = d_first.data_ptr(), 4, 200, t0, n
        out = torch.zeros(N, 200, dtype=torch.int32, device="cuda")
        a.d_out_idx, a.d_out_logits = out.data_ptr(), native.ptr(logits)
        return lib.wn_gen_run(s["handle"], ctypes.byref(a), stream)

    s, _ = _handle(m, N)
    hd = s["handle"]
    # bad arguments of the new entry
    assert lib.wn_gen_set_condition_stream_frames(hd, tab.data_ptr(), f0s(0, -1), 2, HOP) == -1
    assert lib.wn_gen_set_condition_stream_frames(hd, tab.data_ptr(), f0s(0, 0), 0, HOP) == -1
    assert lib.wn_gen_set_condition_stream_frames(hd, tab.data_ptr(), f0s(0, 0), 2, 0) == -1
    assert lib.wn_gen_set_condition_stream_frames(hd, tab.data_ptr(), None, 2, HOP) == -1
    # a per-stream window needs per-stream records
    native.check(lib.wn_gen_set_condition_stream_frames(hd, tab.data_ptr(), f0s(0, 0), 2, HOP), "windows")
    assert run(s, 0, 4) == -4
    native.check(lib.wn_gen_set_stream_params(hd, recs), "params")
    assert run(s, 0, 4) == 0
    # stream 1's window starts at frame 1: positions [4, 84) read frames 0 and 1; t stays where it was
    native.check(lib.wn_gen_set_condition_stream_frames(hd, tab.data_ptr(), f0s(0, 1), 2, HOP), "windows")
    assert run(s, 4, 80) == -1
    assert b"stream 1" in lib.wn_last_error_string()
    native.check(lib.wn_gen_set_condition_stream_frames(hd, tab.data_ptr(), f0s(0, 0), 2, HOP), "windows")
    assert run(s, 4, 80) == 0                                  # continues at t = 4: the failed run moved nothing
    assert run(s, 84, 80) == -1                                # position 160 reads frame 2, past both windows
    native.check(lib.wn_gen_check(hd, stream), "check")
    # wn_gen_set_condition_frames after the per-stream call is one shared window again, bit for bit
    lg = [torch.zeros(N, 200, 256, device="cuda") for _ in range(2)]
    for i in range(2):
        s, _ = _handle(m, N)
        native.check(lib.wn_gen_set_stream_params(s["handle"], recs), "params")
        if i == 0:                                             # these windows (from frame 1) would refuse positions < 80
            native.check(lib.wn_gen_set_condition_stream_frames(s["handle"], tab.data_ptr(), f0s(1, 1), 2, HOP), "windows")
        native.check(lib.wn_gen_set_condition_frames(s["handle"], tab.data_ptr(), 0, 2, HOP), "shared window")
        assert run(s, 0, 150, lg[i]) == 0
        native.check(lib.wn_gen_check(s["handle"], stream), "check")
        lib.wn_gen_destroy(s["handle"])
    assert torch.equal(lg[0], lg[1]) and bool(lg[0][:, :147].abs().sum(2).gt(0).all())


def test_local_session_api_errors(golden):
    rep, plain = _cond_model("global+repeat"), build_model(golden("net_cfg2.npz"))
    for bad in (None, "8", 0, -3, 2.5, True):
        with pytest.raises(ValueError, match="local_window"):
            rep.sampling_session(2, local_window=bad)
    with pytest.raises(ValueError, match="local_window"):
        plain.sampling_session(2, local_window=10)
    sess = rep.sampling_session(2, local_window=100)
    y = np.zeros((80, 3), dtype=np.float32)
    with pytest.raises(ValueError):
        sess.submit([1, 2], 100, condition=np.zeros(16, dtype=np.float32))                 # no local_condition
    with pytest.raises(ValueError):
        sess.submit([1, 2], 100, condition=np.zeros(16, dtype=np.float32), local_condition=np.zeros((40, 3)))
    with pytest.raises(ValueError):                                                        # 101 positions need 2 frames
        sess.submit([1, 2], 100, condition=np.zeros(16, dtype=np.float32), local_condition=y[:, :1])
    assert sess.pending == 0 and sess.next_id == 0
    sess.submit([1, 2], 100, condition=np.zeros(16, dtype=np.float32), local_condition=y[:, :2])
    psess = plain.sampling_session(2)
    with pytest.raises(ValueError):
        psess.submit([1], 5, local_condition=y)
    assert psess.pending == 0
