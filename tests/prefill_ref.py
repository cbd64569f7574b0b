"""Float64 layer inputs of the sampler reference (tests/sampler_ref.py) at every position, for the ring prefill: ring l of
a sampler that has run evaluations [0, T) holds x_l[t] for t in [max(0, T - ring_len_l), T), x_l being layer l's input
(the start conv for l = 0) of the teacher-forced sequence.  The same recursion as sampler_ref.logits, which
test_prefill_window.py pins at 1e-12, with zeros shifted in at the left edge of `idx` (a reset queue's history)."""
import numpy as np

import sampler_ref as R


def layer_inputs(p, dilations, idx, h=None, c=None):
    """([x_0, ..., x_{L-1}] each (R, T), logits (T, classes)) of one stream reading idx[0..T); h: (G,) global condition;
    c: (C, T) audio-rate local features (sampler_ref.local_features)."""
    idx = np.asarray(idx, dtype=np.int64).reshape(-1)
    k = p["filter_convs.0.weight"].shape[2]

    def bias(name):
        b = p.get(name + ".bias")
        return 0.0 if b is None else b[:, None]

    x = p["start_conv.weight"][:, idx, 0] + bias("start_conv")
    xs, skip = [], 0.0
    for i, d in enumerate(dilations):
        xs.append(x)
        pre = []
        for nm in ("filter", "gate"):
            w = p[f"{nm}_convs.{i}.weight"]
            a = w[:, :, k - 1] @ x + bias(f"{nm}_convs.{i}")
            for j in range(1, k):
                a += w[:, :, k - 1 - j] @ R._shift(x, j * d)
            if h is not None:
                a += (p[f"{nm}_cond_convs.{i}.weight"][:, :, 0] @ np.asarray(h, dtype=np.float64).reshape(-1))[:, None]
            if c is not None:
                a += p[f"{nm}_local_convs.{i}.weight"][:, :, 0] @ c
            pre.append(a)
        z = np.tanh(pre[0]) / (1.0 + np.exp(-pre[1]))
        skip = skip + p[f"skip_convs.{i}.weight"][:, :, 0] @ z + bias(f"skip_convs.{i}")
        x = p[f"residual_convs.{i}.weight"][:, :, 0] @ z + bias(f"residual_convs.{i}") + x
    y1 = np.maximum(p["end_conv_1.weight"][:, :, 0] @ np.maximum(skip, 0.0) + p["end_conv_1.bias"][:, None], 0.0)
    return xs, (p["end_conv_2.weight"][:, :, 0] @ y1 + p["end_conv_2.bias"][:, None]).T


def ring_slots(dilations, k, T):
    """[(layer, times [lo, T))] the rings hold after evaluations [0, T)"""
    return [(l, max(0, T - ((k - 1) * d + 1)), T) for l, d in enumerate(dilations)]
