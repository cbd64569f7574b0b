"""Locally conditioned sampling sessions without a GPU: the window plan a step follows (wavenet_model._session_windows,
_session_frames), and the float64 proof that per-stream windows are needed: a job seated at an origin that is not a
multiple of the hop, whose frames were taken by global time instead of by its own position, is far past the 1e-4 bar."""
import numpy as np
import pytest

import sampler_ref as R
import wavenet_model as W
from helpers import rel_err


@pytest.mark.parametrize("hop", [1, 80])
def test_window_plan_covers_every_evaluation(hop):
    rng = np.random.RandomState(hop)
    for trial in range(200):
        n_slots = int(rng.randint(1, 9))
        window = int(rng.choice([1, 2, 3, 43, 79, 80, 81, 160, 241, 1000]))
        nf = W._session_frames(window, hop)
        assert nf == -(-(window - 1) // hop) + 1
        t = int(rng.randint(513, 20000))
        origin = [t - int(rng.randint(0, 6000)) for _ in range(n_slots)]
        # steps that straddle frame and window edges: 1, a window, a window +- 1, and ragged
        n_evals = int(rng.choice([1, window - 1 if window > 1 else 1, window, window + 1, 7, 513, 1000,
                                  int(rng.randint(1, 3000))]))
        plan = W._session_windows(t, n_evals, origin, hop, window)
        assert sum(n for _, n, _ in plan) == n_evals
        t_next = t
        for t0, n, frame0 in plan:
            assert t0 == t_next and 1 <= n <= window and len(frame0) == n_slots
            t_next = t0 + n
            for b in range(n_slots):
                rows = [(tt - origin[b]) // hop - frame0[b] for tt in range(t0, t0 + n)]
                assert frame0[b] >= 0 and min(rows) == 0 and max(rows) < nf, (hop, window, b, rows[:3], nf)
        assert t_next == t + n_evals


def test_window_plan_edges():
    # 64 slots at hop 80 and a 1 000-evaluation window hold 14 frames each; hop 1 holds one frame per evaluation
    assert W._session_frames(1000, 80) == 14 and W._session_frames(64, 1) == 64 and W._session_frames(1, 80) == 1
    assert W._session_frames(81, 80) == 2 and W._session_frames(82, 80) == 3
    # a slot at origin 34: positions 46..125 of the launch at t = 80 read frames 0 and 1 of its own series
    assert W._session_windows(80, 80, [34, 80], 80, 100) == [(80, 80, [0, 0])]
    assert W._session_windows(100, 250, [3, 100], 80, 100) == [(100, 100, [1, 0]), (200, 100, [2, 1]), (300, 50, [3, 2])]


def _local_net(rng, Cl=8, ch=16, classes=64, dil=(1, 2, 4, 8, 16, 32)):
    p = {"start_conv.weight": rng.randn(ch, classes, 1) * 0.5}
    for i in range(len(dil)):
        for nm in ("filter", "gate"):
            p[f"{nm}_convs.{i}.weight"] = rng.randn(ch, ch, 2) * 0.3
            p[f"{nm}_local_convs.{i}.weight"] = rng.randn(ch, Cl, 1) * 0.5
        p[f"skip_convs.{i}.weight"] = rng.randn(ch, ch, 1) * 0.3
        p[f"residual_convs.{i}.weight"] = rng.randn(ch, ch, 1) * 0.3
    p.update({"end_conv_1.weight": rng.randn(ch, ch, 1) * 0.3, "end_conv_1.bias": rng.randn(ch) * 0.1,
              "end_conv_2.weight": rng.randn(classes, ch, 1) * 0.3, "end_conv_2.bias": rng.randn(classes) * 0.1})
    return p, list(dil)


def test_frames_by_global_time_move_logits():
    """A job at origin 1 234 (1 234 % 80 = 34) that read frame t // hop of global time t instead of frame q // hop of its
    own position q = t - origin would cross every frame boundary 34 samples early."""
    rng = np.random.RandomState(11)
    p, dil = _local_net(rng)
    hop, origin, T = 80, 1234, 400
    assert origin % hop != 0
    idx = rng.randint(0, 64, T)
    y = rng.randn(8, -(-(origin + T) // hop) + 1)
    own = R.logits(p, dil, idx, y=y, hop=hop)
    q = np.arange(T)
    by_global = R.logits(p, dil, idx, y=y[:, (q + origin) // hop], hop=1)
    by_position = R.logits(p, dil, idx, y=y[:, q // hop], hop=1)
    assert rel_err(by_position, own) == 0.0                     # the hop-1 restatement is the reference itself
    assert rel_err(by_global, own) > 100 * 1e-4
    # an origin on a frame boundary only shifts the frames: the same job with its series shifted by origin // hop agrees
    assert rel_err(R.logits(p, dil, idx, y=y[:, q // hop + 2], hop=1), R.logits(p, dil, idx, y=y[:, 2:], hop=hop)) == 0.0
