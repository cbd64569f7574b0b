"""Float64 references of the native entry points of a training step that sit around the residual blocks (CPU only; nothing
here is product code), for the kernel-level tests of test_gpu_step_kernels_f64.py.  Each works on the kernel's own layout
(include/wavenet_b200.h):

    start conv     h[b, t, :] = W[:, x[b, :, t]] + bias                  x (B, classes, L) dense or (B, L) class indices
    head forward   logits = W2 relu(W1 relu(skip) + b1) + b2             last out_len frames of skip (B, L - skip_start, S)
    head backward  y1 = relu(W1 relu(skip) + b1),  dy1 = (dlogits W2) [pre1 > 0],  dskip = (dy1 W1) [skip > 0]
    cross-entropy  loss = mean_i (logsumexp(x_i) - x_i[t_i]),  dlogits = (softmax(x_i) - onehot(t_i)) / N
    Adam           torch.optim.Adam (L2 weight decay, no amsgrad) with one step count per parameter
    scatter rows   table[c, :] = sum of dh[b, t, :] over frames t >= t_begin with idx[b, t] = c
    column sums    out[c] = sum_r x[r, c]

Class indices outside [0, classes) are clamped, as the kernels do."""
import torch

import block_ref as BR


def _clamp(idx, classes):
    return idx.long().clamp(0, classes - 1)


# ---------------------------------------------------------------------------------------------------- start conv
def start_dense(x, w, b):
    """x (B, classes, L), w (R, classes, 1), b (R,) or None -> frames (B, L, R) float64"""
    h = torch.einsum("bcl,rc->blr", x.double(), w[:, :, 0].double())
    return h if b is None else h + b.double()


def start_index(idx, w, b):
    """idx (B, L) -> frames (B, L, R) float64: row idx of the start conv's (classes, R) table plus the bias"""
    h = w[:, :, 0].double().T[_clamp(idx, w.shape[1])]
    return h if b is None else h + b.double()


def start_index_fp32(idx, w, b):
    """what the index kernels compute: the fp32 sum w[c] + b (one rounding), as float32"""
    h = w[:, :, 0].float().T[_clamp(idx, w.shape[1])]
    return h if b is None else h + b.float()


def start_pair_planes(idx, w, b):
    """the (hi, lo) planes wn_tb_start_index_* stores: split_bf16 of the fp32 value w[c] + b"""
    return BR.split_bf16(start_index_fp32(idx, w, b))


def index_out_of_range(idx, classes):
    return bool(((idx.long() < 0) | (idx.long() >= classes)).any())


# ---------------------------------------------------------------------------------------------------- head
def head_forward(skip, w1, b1, w2, b2, out_len, taps=None):
    """skip (B, L - skip_start, S) frames; w1 (E, S, 1), w2 (classes, E, 1) -> logits (B * out_len, classes) float64 for the
    last out_len frames.  taps (a dict) receives the float64 inputs of the two ReLUs: "skip" (B, out_len, S), "pre1"."""
    sk = skip[:, skip.shape[1] - out_len:].double()
    pre1 = torch.relu(sk) @ w1[:, :, 0].double().T + b1.double()
    logits = torch.relu(pre1) @ w2[:, :, 0].double().T + b2.double()
    if taps is not None:
        taps["skip"], taps["pre1"] = sk, pre1
    return logits.reshape(-1, w2.shape[0])


def head_backward_data(dlogits, skip, w1, b1, w2, out_len):
    """dlogits (B * out_len, classes); skip (B, L - skip_start, S) -> float64 y1, dy1 (B, out_len, E) and dskip
    (B, out_len, S), the ReLU masks taken from the float64 pre-activations."""
    B = skip.shape[0]
    taps = {}
    head_forward(skip, w1, b1, w2, torch.zeros(w2.shape[0]), out_len, taps)
    sk, pre1 = taps["skip"], taps["pre1"]
    dl = dlogits.double().reshape(B, out_len, -1)
    dy1 = (dl @ w2[:, :, 0].double()) * (pre1 > 0)
    dskip = (dy1 @ w1[:, :, 0].double()) * (sk > 0)
    return dict(y1=torch.relu(pre1), dy1=dy1, dskip=dskip)


def head_relu_margin(skip, w1, b1, out_len):
    """smallest |input| of either head ReLU over the last out_len frames (float64): how far the masks are from a tie"""
    taps = {}
    head_forward(skip, w1, b1, torch.zeros(1, w1.shape[0], 1), torch.zeros(1), out_len, taps)
    return min(float(taps["skip"].abs().min()), float(taps["pre1"].abs().min()))


# ---------------------------------------------------------------------------------------------------- cross-entropy
def cross_entropy(logits, target):
    """mean cross-entropy of rows (N, C) with targets (N,) -> (loss, dlogits) float64; the maximum is subtracted first"""
    x = logits.double()
    t = _clamp(target, x.shape[1])
    mx = x.max(1, keepdim=True).values
    e = torch.exp(x - mx)
    s = e.sum(1, keepdim=True)
    rows = torch.log(s[:, 0]) + (mx[:, 0] - x.gather(1, t.view(-1, 1))[:, 0])
    d = e / s
    d[torch.arange(x.shape[0]), t] -= 1
    return rows.mean(), d / x.shape[0]


# ---------------------------------------------------------------------------------------------------- Adam
def adam_update(p, g, m, v, step, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
    """one torch.optim.Adam update of one parameter at its own step count (1-based) -> float64 (p, m, v)"""
    p, g, m, v = (t.double() for t in (p, g, m, v))
    b1, b2 = betas
    if weight_decay != 0:
        g = g + weight_decay * p
    m = m + (1 - b1) * (g - m)
    v = b2 * v + (1 - b2) * g * g
    denom = v.sqrt() / (1 - b2 ** step) ** 0.5 + eps
    return p - lr / (1 - b1 ** step) * m / denom, m, v


class Adam:
    """Adam over a list of parameters with a step count per parameter, advanced only on steps where that parameter has a
    gradient (torch.optim.Adam's rule).  State in float64."""

    def __init__(self, params, **hyper):
        self.p = [t.double().clone() for t in params]
        self.m = [torch.zeros_like(t) for t in self.p]
        self.v = [torch.zeros_like(t) for t in self.p]
        self.steps = [0] * len(self.p)
        self.hyper = hyper

    def step(self, grads):
        for i, g in enumerate(grads):
            if g is None:
                continue
            self.steps[i] += 1
            self.p[i], self.m[i], self.v[i] = adam_update(self.p[i], g, self.m[i], self.v[i], self.steps[i], **self.hyper)


# ---------------------------------------------------------------------------------------------------- reductions
def scatter_rows(idx, dh, classes, t_begin):
    """idx (B, L), dh (B, L, R) -> table (classes, R) float64 and the sum of |dh| routed to each row (classes, R)"""
    R = dh.shape[2]
    c = _clamp(idx[:, t_begin:], classes).reshape(-1)
    src = dh[:, t_begin:].double().reshape(-1, R)
    table = torch.zeros(classes, R, dtype=torch.float64).index_add_(0, c, src)
    mag = torch.zeros(classes, R, dtype=torch.float64).index_add_(0, c, src.abs())
    return table, mag


def colsum(x, rows, C):
    """x (>= rows, ld) -> (sum, sum of |x|) over rows [0, rows) of columns [0, C), float64"""
    v = x[:rows, :C].double()
    return v.sum(0), v.abs().sum(0)
