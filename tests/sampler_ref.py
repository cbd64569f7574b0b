"""Float64 reference of the sampler: a teacher-forced Fast-WaveNet evaluated for all times at once (numpy only).

With the input indices idx[0..T) known (the given samples followed by the samples fed back), evaluation t reads sample
idx[t] and predicts sample t + 1.  Layer l's input is a matrix x_l (R, T); its tap j (j = 0 the current column, weight
column k - 1 - j) is x_l shifted right by j * dil with ZEROS shifted in: a reset queue holds zeros, not the network's
response to silence, so with biases this is not a forward pass over a zero-padded input.  One layer is

    f = sum_j Wf[:, :, k-1-j] shift(x, j dil) + bf  (+ Vf h)  (+ Uf c[:, t])        g likewise
    z = tanh(f) * sigmoid(g)       skip += Ws z + bs       x <- Wr z + br + x

and the head is W2 relu(W1 relu(skip) + b1) + b2.  c[:, t] is y[:, t // hop] under repeat upsampling and the output of
the learned upsampler (tests/upsample_ref.py) at hop 1 otherwise.  Nothing here comes from the sampler's code; the
`mutate` variants are deliberately wrong and exist to show that the tests which use this file can fail."""
import numpy as np


def weights(params):
    """state_dict / oracle parameter dict -> float64 ndarrays."""
    return {k: np.asarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v, dtype=np.float64) for k, v in params.items()}


def dilations_of(layers, blocks):
    return [2 ** i for _ in range(blocks) for i in range(layers)]


def _shift(x, n):
    """x (R, T) delayed by n columns, zeros shifted in."""
    out = np.zeros_like(x)
    if n < x.shape[1]:
        out[:, n:] = x[:, :x.shape[1] - n]
    return out


def local_features(p, y, hop, T, scales=None, mutate=None):
    """(C, T) audio-rate condition features of one stream's (C, F) frame series."""
    y = np.asarray(y, dtype=np.float64)
    if scales is not None:
        import torch
        import upsample_ref
        up = {k: torch.from_numpy(v) for k, v in p.items() if k.startswith("local_upsample.")}
        y, hop = upsample_ref.upsample(up, scales, torch.from_numpy(y)[None])[0].numpy(), 1
    t = np.arange(T)
    if mutate is not None and mutate[0] == "frame_off_by_one":
        t = t + 1                                   # the frame changes one sample early
    return y[:, np.minimum(t // hop, y.shape[1] - 1)]


def logits(p, dilations, idx, h=None, y=None, hop=None, scales=None, mutate=None):
    """(T, classes) float64 logits of one stream: row t is evaluation t, which has read idx[0..t].
    p: weights(); h: (G,) global condition; y: (C, F) local series at `hop` (or through the learned upsampler of
    `scales`); mutate: None, ("zero_history", layer), ("late_tap", layer) or ("frame_off_by_one",)."""
    idx = np.asarray(idx, dtype=np.int64).reshape(-1)
    T = idx.shape[0]
    k = p["filter_convs.0.weight"].shape[2]

    def bias(name):
        b = p.get(name + ".bias")
        return 0.0 if b is None else b[:, None]

    c = None if y is None else local_features(p, y, hop, T, scales, mutate)
    hv = None if h is None else np.asarray(h, dtype=np.float64).reshape(-1)
    x = p["start_conv.weight"][:, idx, 0] + bias("start_conv")
    skip = 0.0
    for i, d in enumerate(dilations):
        pre = []
        for nm in ("filter", "gate"):
            w = p[f"{nm}_convs.{i}.weight"]
            a = w[:, :, k - 1] @ x + bias(f"{nm}_convs.{i}")
            for j in range(1, k):
                if mutate is not None and mutate[1:] == (i,):
                    if mutate[0] == "zero_history":
                        continue
                    if mutate[0] == "late_tap":
                        a += w[:, :, k - 1 - j] @ _shift(x, j * d + 1)
                        continue
                a += w[:, :, k - 1 - j] @ _shift(x, j * d)
            if hv is not None:
                a += (p[f"{nm}_cond_convs.{i}.weight"][:, :, 0] @ hv)[:, None]
            if c is not None:
                a += p[f"{nm}_local_convs.{i}.weight"][:, :, 0] @ c
            pre.append(a)
        z = np.tanh(pre[0]) / (1.0 + np.exp(-pre[1]))
        skip = skip + p[f"skip_convs.{i}.weight"][:, :, 0] @ z + bias(f"skip_convs.{i}")
        x = p[f"residual_convs.{i}.weight"][:, :, 0] @ z + bias(f"residual_convs.{i}") + x
    y1 = np.maximum(skip, 0.0)
    y1 = np.maximum(p["end_conv_1.weight"][:, :, 0] @ y1 + p["end_conv_1.bias"][:, None], 0.0)
    return (p["end_conv_2.weight"][:, :, 0] @ y1 + p["end_conv_2.bias"][:, None]).T


def inputs(first, fed):
    """The input sequence of a run: the given samples, then the samples fed back (all but the last)."""
    first, fed = np.asarray(first).reshape(-1), np.asarray(fed).reshape(-1)
    return np.concatenate([first, fed[:max(len(fed) - 1, 0)]]).astype(np.int64)


def regularizer(classes, regularize):
    """fp32, as the sampler and the upstream model subtract it: regularize * (c - classes / 2)^2."""
    return (np.arange(classes, dtype=np.float32) - np.float32(classes / 2.0)) ** 2 * np.float32(regularize)


def choose(logits32, temperature, regularize, u=None):
    """The selection rule of the sampler for rows of fp32 logits (N, classes): temperature <= 0 takes the lowest index of
    the largest (logits - regularizer); otherwise the fp32 softmax of (logits - regularizer) / temperature is summed in
    float64, normalised by its last element and searched with side='right' for the uniform u (N,), which is what
    numpy.random.choice does.  Returns (index, margin, edge): margin = top-1 minus top-2 of the regularised logits,
    edge = distance of u to the nearest CDF edge (None for argmax)."""
    lg = np.atleast_2d(np.asarray(logits32, dtype=np.float32))
    C = lg.shape[1]
    if regularize:
        lg = lg - regularizer(C, regularize)[None, :]
    top2 = np.sort(lg, axis=1)[:, -2:]
    margin = (top2[:, 1] - top2[:, 0]).astype(np.float64)
    if not temperature > 0:
        return lg.argmax(axis=1), margin, None
    x = lg / np.float32(temperature)
    e = np.exp(x - x.max(axis=1, keepdims=True))
    prob = (e / e.sum(axis=1, keepdims=True, dtype=np.float32)).astype(np.float32)
    cdf = np.cumsum(prob.astype(np.float64), axis=1)
    cdf /= cdf[:, -1:]
    u = np.asarray(u, dtype=np.float64).reshape(-1, 1)
    index = np.minimum((cdf <= u).sum(axis=1), C - 1)
    return index, margin, np.abs(cdf - u).min(axis=1)
