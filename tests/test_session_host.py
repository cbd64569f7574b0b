"""Sampling sessions without a GPU: the admission and launch records a step computes (wavenet_model._session_admit,
_session_records), submit's argument checks, and the float64 proof that the fault seating guards against is visible: a job
that runs on a reused slot's old history instead of zeros moves the logits far past the 1e-4 bar once the run is longer
than a tap's dilation."""
import numpy as np
import pytest

import sampler_ref as R
import wavenet_model as W
from helpers import rel_err
from test_sampler_ref import _cfg2, _dil


class _J:
    def __init__(self, prompt, count, temperature=0.0, uniforms=None):
        self.prompt, self.count = np.asarray(prompt, dtype=np.int32), count
        self.temperature, self.regularize, self.top_k, self.top_p, self.uniforms = temperature, 0.0, 0, 1.0, uniforms


def test_admission_is_fifo_lowest_slot_first():
    a, b, c, d = _J([1], 5), _J([2], 0), _J([3], 2), _J([4], 1)
    queue = [a, b, c, d]
    # slot 1 busy, slot 0 free and unseated, slot 2 parked: a -> 0, b is done without a slot, c -> 2
    seats = W._session_admit([None, _J([9], 3), None], [False, True, True], queue)
    assert seats == [(0, a), (2, c)] and queue == [d]
    # nothing queued: an unseated free slot is parked, a parked one stays
    assert W._session_admit([None, None], [False, True], []) == [(0, None)]


def test_launch_records():
    u = np.arange(10) / 10
    a, c = _J([1, 2, 3], 5, 1.0, u), _J([7, 8], 2)
    recs, pos, first, uni, plans = W._session_records(100, 4, [a, None, c], [100, 90, 98])
    # a: positions 0..3, prompt [0, 3) read from first0 = 0, samples 0, 1 in columns 0, 1 with their uniforms
    # parked slot 1: position 10, no prompt read, columns from sample 10
    # c: positions 2..5, past its prompt, samples from 1: one left
    assert [(p.origin, p.sample0, p.first0) for p in pos] == [(100, 0, 0), (90, 10, 0), (98, 1, 0)]
    assert [(r.n_given, r.temperature) for r in recs] == [(3, 1.0), (1, 0.0), (2, 0.0)]
    assert first.tolist() == [[1, 2, 3], [0, 0, 0], [0, 0, 0]]
    assert np.array_equal(uni[0], [0.0, 0.1, 0.0, 0.0]) and not uni[1:].any()
    assert [(b, j, c0, n) for b, j, c0, n in plans] == [(0, a, 0, 2), (2, c, 0, 1)]
    # a primed job (origin = t - T): the row holds only the prompt positions the launch reads
    p = _J(np.arange(50), 3)
    recs, pos, first, uni, plans = W._session_records(1000, 7, [p], [1000 - 49])
    assert (pos[0].origin, pos[0].sample0, pos[0].first0) == (951, 0, 49) and first.tolist() == [[49]]
    assert plans[0][2:] == (0, 3)
    # later steps: columns restart at 0 at sample sample0
    recs, pos, first, uni, plans = W._session_records(1010, 7, [p], [951])
    assert (pos[0].sample0, pos[0].first0) == (10, 0) and plans == []


@pytest.mark.parametrize("bad", [dict(temperature=float("nan")), dict(top_k=-1), dict(top_p=0.0), dict(num_samples=-1),
                                 dict(first_samples=[]), dict(uniforms=np.zeros(3))])
def test_submit_rejects_bad_arguments(bad):
    sess = W.SamplingSession.__new__(W.SamplingSession)       # host state only: submit checks before any device work
    sess.queue, sess.jobs, sess.next_id = [], {}, 0

    class _M:
        _condition = staticmethod(lambda c, n: None)
        _one_condition = staticmethod(lambda c: None)
    sess.model = _M()
    kw = dict(first_samples=[1, 2], num_samples=5, temperature=1.0)
    kw.update(bad)
    with pytest.raises(ValueError):
        sess.submit(**kw)
    assert sess.queue == []


def test_stale_history_moves_logits(golden):
    """The failure seating prevents: a new job evaluated on the previous job's ring history instead of zeros."""
    g, spec, p = _cfg2(golden)
    w, dil = R.weights(p), _dil(spec)
    rng = np.random.RandomState(5)
    old, new = rng.randint(0, 256, 700), rng.randint(0, 256, 600)
    clean = R.logits(w, dil, new)
    stale = R.logits(w, dil, np.concatenate([old, new]))[len(old):]
    d = min(dil)
    assert rel_err(stale[:1], clean[:1]) > 1e-2            # the first evaluation already reads taps at t - 1
    assert rel_err(stale[d:], clean[d:]) > 100 * 1e-4
    assert rel_err(clean, R.logits(w, dil, new)) == 0.0
