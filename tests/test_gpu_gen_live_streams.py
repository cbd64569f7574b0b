"""The batched tensor-core sampler (mode 6) exchanges only the bytes of a cluster's live streams; the columns of empty
stream slots keep stale values.  A stream's indices and logits must not depend on how many of the 8 stream slots of its
cluster are live: streams run n at a time (n = 1..8) equal the same streams inside a full 8-stream launch, bit for bit,
for both cluster sizes (16 CTAs with one block each, 8 CTAs with two)."""
import numpy as np
import pytest

from helpers import build_model

pytestmark = pytest.mark.gpu

N_SAMPLES = 40
CHUNKS = (2, 7, 20)          # evaluation indices after which a chunked run ends a launch and continues the session


def _runs(rt, m, first, uni, forced):
    """(sampled, forced, chunked) results of one launch set: each (indices, logits)."""
    sampled = m.generate_fast_batch(N_SAMPLES, first, temperature=1.0, uniforms=uni, return_logits=True)
    tf = m.generate_fast_batch(N_SAMPLES, first, temperature=0.0, forced=forced, return_logits=True)
    idx, lg, _ = rt.generate(N_SAMPLES, first.astype(np.int32), 1.0, 0.0, uniforms=uni, want_logits=True,
                             callbacks=[(e, lambda: None) for e in CHUNKS])
    return sampled, tf, (idx, lg)


@pytest.mark.parametrize("cs", [16, 8])
def test_live_streams_bitwise_vs_full_cluster(golden, monkeypatch, cs):
    monkeypatch.setenv("WN_GEN_CL8_CS", str(cs))      # read when a sampler handle is created: a fresh model per setting
    m = build_model(golden("net_cfg2.npz"))
    rt = m._runtime()
    rt.gen_mode = 6
    rng = np.random.RandomState(7 + cs)
    first = rng.randint(0, 256, size=(8, 5))          # 5 given samples: 4 warm-up evaluations before the first draw
    uni = rng.random_sample((8, N_SAMPLES))
    forced = rng.randint(0, 256, size=(8, N_SAMPLES))
    full = _runs(rt, m, first, uni, forced)
    for i, l in full:
        assert np.isfinite(l).all()
    # the chunked run continues the session it started: same result as one launch
    assert np.array_equal(full[2][0], full[0][0]) and np.array_equal(full[2][1], full[0][1])
    for n in range(1, 9):
        for s0 in range(0, 8, n):
            sub = list(range(s0, min(s0 + n, 8)))
            got = _runs(rt, m, first[sub], uni[sub], forced[sub])
            for (gi, gl), (fi, fl) in zip(got, full):
                assert np.array_equal(gi, fi[sub]), (cs, n, sub)
                assert np.array_equal(gl, fl[sub]), (cs, n, sub)
    rt.gen_mode = None
