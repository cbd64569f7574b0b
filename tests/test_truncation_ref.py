"""The truncated selection rule of the sampler (top-k / nucleus, wn_gen_set_truncation) in tests/truncation_ref.py, pinned
on the CPU against an independent formulation: a stable torch sort, top-k / top-p filtering on the sorted probabilities,
then numpy.random.choice's inverse CDF over the survivors in index order.  Also: the off values reduce to `choose`
exactly, four deliberately wrong rules are caught, and the API refuses bad arguments before any device work."""
import numpy as np
import pytest
import torch

import sampler_ref as R
import truncation_ref as T

U_LAST = 1.0 - 2.0 ** -53


def _probs(lg, temperature):
    """the rule's p: choose's fp32 softmax"""
    x = lg / np.float32(temperature)
    e = np.exp(x - x.max(axis=1, keepdims=True))
    return (e / e.sum(axis=1, keepdims=True, dtype=np.float32)).astype(np.float32).astype(np.float64)


def _independent(lg, temperature, u, top_k, top_p):
    """sort-based filtering in torch, then np.random.choice-style inverse CDF over the survivors"""
    p = _probs(lg, temperature)
    N, C = lg.shape
    out = np.empty(N, dtype=np.int64)
    for i in range(N):
        _, order = torch.sort(torch.from_numpy(lg[i]), descending=True, stable=True)   # equal logits: lower index first
        order = order.numpy()
        if 0 < top_k < C:
            order = order[:top_k]
        ps = p[i, order]
        if top_p < 1.0:
            before = np.concatenate([[0.0], np.cumsum(ps)[:-1]])
            order = order[before < top_p * ps.sum()]           # keep while the mass before a class is short of the bar
        keep = np.sort(order)
        cdf = np.cumsum(p[i, keep])
        cdf /= cdf[-1]
        out[i] = keep[min(np.searchsorted(cdf, u[i], side="right"), len(keep) - 1)]
    return out


def _logits(C, N, seed, scale=3.0):
    rng = np.random.RandomState(seed)
    lg = (scale * rng.randn(N, C)).astype(np.float32)
    lg[:, rng.randint(0, C, 4)] += np.float32(6.0)             # a few dominant classes, as a trained net has
    return lg


def _uniforms(N, seed):
    u = np.random.RandomState(seed).random_sample(N)
    u[::7], u[3::7] = 0.0, U_LAST
    return u


KS = lambda C: [0, 1, 2, 40, C - 1, C, C + 5]
PS = [1e-12, 0.5, 0.95, 1.0]


@pytest.mark.parametrize("C", [100, 256, 1000])
@pytest.mark.parametrize("temperature", [1.0, 0.7, 1.3, 0.05])
def test_rule_matches_the_sort_based_formulation(C, temperature):
    N = 120
    lg = _logits(C, N, C + int(100 * temperature))
    u = _uniforms(N, C)
    for k in KS(C):
        for p in PS:
            got, kept, edge, pgap = T.choose_truncated(lg, temperature, 0.0, u, k, p)
            want = _independent(lg, temperature, u, k, p)
            near = (edge < 1e-12) | (pgap < 1e-12)
            assert np.all(kept[np.arange(N), got]), (C, k, p)
            assert np.array_equal(got[~near], want[~near]), (C, temperature, k, p)
            if 0 < k < C:
                assert np.all(kept.sum(axis=1) <= k)
            if p == 1e-12 or k == 1:
                assert np.array_equal(got, lg.argmax(axis=1))      # a single class: the argmax, ties to the lower index


def test_regularizer_is_subtracted_first():
    C, N = 256, 64
    lg = _logits(C, N, 3)
    u = _uniforms(N, 4)
    a = T.choose_truncated(lg, 1.0, 1e-4, u, 30, 0.9)
    b = T.choose_truncated(lg - R.regularizer(C, 1e-4)[None, :], 1.0, 0.0, u, 30, 0.9)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_ties_at_the_kth_place_keep_the_lower_index():
    C, N = 256, 50
    lg = _logits(C, N, 5, scale=0.5)
    lg[:, 17] = lg[:, 200] = lg.max(axis=1) + 1.0               # an exact tie for the top place
    lg[:, 30] = lg[:, 90] = lg[:, 17] - 0.5                     # and for the third
    u = _uniforms(N, 6)
    _, kept, _, _ = T.choose_truncated(lg, 1.0, 0.0, u, 1, 1.0)
    assert kept[:, 17].all() and not kept[:, 200].any() and (kept.sum(axis=1) == 1).all()
    _, kept, _, _ = T.choose_truncated(lg, 1.0, 0.0, u, 3, 1.0)
    assert kept[:, [17, 200, 30]].all() and not kept[:, 90].any()
    got, _, _, _ = T.choose_truncated(lg, 1.0, 0.0, u, 1, 1.0)
    assert (got == 17).all()
    assert np.array_equal(got, _independent(lg, 1.0, u, 1, 1.0))


def test_u_zero_gives_the_lowest_kept_class_with_mass():
    """at a low temperature kept classes underflow to p = 0; u = 0 must skip them"""
    C, N = 256, 40
    lg = _logits(C, N, 7)
    u = np.zeros(N)
    got, kept, _, _ = T.choose_truncated(lg, 0.02, 0.0, u, 50, 1.0)
    p = _probs(lg, 0.02)
    assert ((p == 0) & kept).any()                               # the case the test is about does occur
    for i in range(N):
        assert got[i] == np.flatnonzero(kept[i] & (p[i] > 0))[0]
    assert np.array_equal(got, _independent(lg, 0.02, u, 50, 1.0))


def test_u_last_gives_the_highest_kept_class():
    """u = 1 - 2^-53 lies past every kept edge but the last (none of these rows has a tail mass below 2^-53)"""
    C, N = 256, 40
    lg = _logits(C, N, 8)
    u = np.full(N, U_LAST)
    for k, p in [(5, 1.0), (0, 0.5), (40, 0.95), (C - 1, 1.0)]:
        got, kept, _, _ = T.choose_truncated(lg, 1.0, 0.0, u, k, p)
        for i in range(N):
            assert got[i] == np.flatnonzero(kept[i])[-1]


@pytest.mark.parametrize("C", [100, 256, 1000])
def test_off_values_reduce_to_choose(C):
    N = 80
    lg = _logits(C, N, 9)
    u = _uniforms(N, 10)
    for temperature, reg in [(0.0, 0.0), (0.0, 1e-4), (0.5, 0.0), (1.0, 1e-4)]:
        want, _, edge = R.choose(lg, temperature, reg, u)
        for k, p in [(0, 1.0), (C, 1.0), (C + 1, 1.0)] + ([(5, 0.5), (1, 1e-12)] if temperature == 0 else []):
            got, kept, e2, _ = T.choose_truncated(lg, temperature, reg, u, k, p)
            assert np.array_equal(got, want) and kept.all()
            assert (e2 is None and edge is None) or np.array_equal(e2, edge)


def test_every_wrong_rule_is_caught():
    """each mutation changes the index of some selection on these inputs, away from rounding of an edge or threshold"""
    C, N = 256, 400
    lg = _logits(C, N, 11, scale=1.0)
    lg[:, 100] = lg[:, 101] = lg.max(axis=1) + 0.25              # ties at the top ...
    lg[:, 150] = lg[:, 151] = np.sort(lg, axis=1)[:, -6]         # ... and around the k-th place
    u = _uniforms(N, 12)
    u[::5] = 1.0                     # the only way the count runs past the kept edges (numpy's RNG never returns it)
    cases = {"k_off_by_one": (5, 1.0), "ties_high": (1, 1.0), "threshold_all": (20, 0.5), "clamp_last_class": (30, 1.0)}
    for mutate, (k, p) in cases.items():
        right, _, edge, pgap = T.choose_truncated(lg, 1.0, 0.0, u, k, p)
        wrong, _, _, _ = T.choose_truncated(lg, 1.0, 0.0, u, k, p, mutate=mutate)
        far = (pgap > 1e-9) & ((edge > 1e-9) | (u >= 1.0))            # u = 1 is past every edge by construction
        assert (right != wrong)[far].sum() >= 5, mutate
        assert np.array_equal(right, _independent(lg, 1.0, u, k, p))


@pytest.mark.parametrize("kw", [dict(top_k=-1), dict(top_k=True), dict(top_k=2.0), dict(top_k="3"), dict(top_p=0.0),
                                dict(top_p=-0.5), dict(top_p=1.5), dict(top_p=float("nan")), dict(top_p=True),
                                dict(top_p="0.9"), dict(top_k=np.bool_(True))])
def test_api_refuses_bad_arguments_before_device_work(kw):
    import wavenet_model as wmod
    m = wmod.WaveNetModel(layers=2, blocks=1, dilation_channels=8, residual_channels=8, skip_channels=8,
                          end_channels=8, classes=16, output_length=4, kernel_size=2, bias=False)
    with pytest.raises(ValueError):
        m.generate_fast(4, first_samples=np.zeros(2, dtype=np.int64), temperature=1.0, **kw)
    with pytest.raises(ValueError):
        m.generate_fast_batch(4, np.zeros((2, 2), dtype=np.int64), temperature=1.0, **kw)


def test_api_accepts_good_arguments():
    import wavenet_model as wmod
    assert wmod._truncation(0, 1.0) == (0, 1.0)
    assert wmod._truncation(np.int64(40), np.float32(0.5)) == (40, 0.5)
    assert wmod._truncation(300, 1) == (300, 1.0)
    assert wmod._truncation(1, 1e-12) == (1, 1e-12)
