"""Float64 reference of the sampler's truncated selection (top-k / nucleus, wn_gen_set_truncation), beside the
untruncated rule `sampler_ref.choose`, which it reduces to when no bound drops a class.  Nothing here comes from the
sampler's code; the `mutate` variants are deliberately wrong and exist to show that the tests which use this file can
fail."""
import numpy as np

from sampler_ref import choose, regularizer


TRUNCATION_MUTATIONS = ("k_off_by_one", "ties_high", "threshold_all", "clamp_last_class")


def choose_truncated(logits32, temperature, regularize, u, top_k=0, top_p=1.0, mutate=None):
    """The truncated selection rule (wn_gen_set_truncation) for rows of fp32 logits (N, classes).  With temperature <= 0
    or no bound that drops a class it is `choose`.  Otherwise p is choose's fp32 softmax of l / temperature (l = logits -
    regularizer); the classes are ranked by l descending, ties by lower index; K1 = the first top_k (all when top_k is 0 or
    >= classes); K = the shortest ranked prefix of K1 whose float64 sum of p reaches top_p * (sum of p over K1); the draw
    is choose's inverse CDF over K in index order, a count past the end giving the largest kept index.
    Returns (index, kept (N, classes) bool, edge, pgap): edge = distance of u to the nearest CDF edge of K, pgap = the
    distance of the deciding prefix sums (the last one kept and the one before it) to the threshold, relative to K1's
    mass (inf when top-p is off); for `choose`'s cases kept is all True and edge is choose's.
    mutate: one of TRUNCATION_MUTATIONS, deliberately wrong rules the tests must catch."""
    lg = np.atleast_2d(np.asarray(logits32, dtype=np.float32))
    N, C = lg.shape
    u = np.asarray(u, dtype=np.float64).reshape(-1)
    if not (temperature > 0 and (0 < top_k < C or top_p < 1.0)):
        index, _, edge = choose(lg, temperature, regularize, u)
        return index, np.ones((N, C), dtype=bool), edge, np.full(N, np.inf)
    if regularize:
        lg = lg - regularizer(C, regularize)[None, :]
    x = lg / np.float32(temperature)
    e = np.exp(x - x.max(axis=1, keepdims=True))
    p = (e / e.sum(axis=1, keepdims=True, dtype=np.float32)).astype(np.float32).astype(np.float64)
    cls = np.broadcast_to(np.arange(C), (N, C))
    order = np.lexsort((-cls if mutate == "ties_high" else cls, -lg), axis=1)     # rank order: l descending, then index
    k1 = C if top_k == 0 or top_k >= C else top_k
    if mutate == "k_off_by_one":
        k1 = min(k1 + 1, C)
    pr = np.take_along_axis(p, order, axis=1)
    cs = np.cumsum(pr[:, :k1], axis=1)
    mass = cs[:, -1]
    n = np.full(N, k1)
    pgap = np.full(N, np.inf)
    if top_p < 1.0:
        thr = top_p * (np.cumsum(pr, axis=1)[:, -1] if mutate == "threshold_all" else mass)
        n = np.minimum(np.argmax(cs >= thr[:, None], axis=1) + 1, k1)
        rows = np.arange(N)
        before = np.where(n >= 2, cs[rows, np.maximum(n - 2, 0)], 0.0)
        pgap = np.minimum(np.abs(cs[rows, n - 1] - thr), np.abs(before - thr)) / mass
    kept = _unrank(order, np.arange(C)[None, :] < n[:, None])
    q = np.where(kept, p, 0.0)
    cdf = np.cumsum(q, axis=1)
    cdf /= cdf[:, -1:]
    count = ((cdf <= u[:, None]) & kept).sum(axis=1)
    n_kept = kept.sum(axis=1)
    index = np.empty(N, dtype=np.int64)
    for i in range(N):
        ks = np.flatnonzero(kept[i])
        index[i] = (C - 1 if mutate == "clamp_last_class" else ks[-1]) if count[i] >= n_kept[i] else ks[count[i]]
    edge = np.where(kept, np.abs(cdf - u[:, None]), np.inf).min(axis=1)
    return index, kept, edge, pgap


def _unrank(order, ranked):
    """(N, C) values in rank order -> the same values at their classes"""
    out = np.empty_like(ranked)
    np.put_along_axis(out, order, ranked, axis=1)
    return out
