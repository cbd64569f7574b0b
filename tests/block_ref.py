"""Float64 references of ONE residual block (reference wavenet_model.py:142-165), written from the block's definition, for the
kernel-level tests (CPU only; nothing here is product code).

Time is absolute (frames [0, L), as in include/wavenet_b200.h); a tensor is zero left of its first valid frame.  With k taps
and dilation d, tap j reads frame t - (k-1-j)*d:

    forward   z[t]      = tanh(sum_j Wf_j h[t-(k-1-j)d] + bf) * sigmoid(sum_j Wg_j h[t-(k-1-j)d] + bg)   h = 0 left of in_start
              h_out[t]  = Wr z[t] + br + h[t]                                                        t in [out_start, L)
              skip[t]   = Ws z[t] + bs (+ skip[t])                                                   t in [skip_start, L)
    backward  dz[t]     = Wr^T dh_out[t] [t >= gs_out] + Ws^T dskip[t] [t >= ds_start]              t in [gz, L)
              dF = dz g (1 - f^2),  dG = dz f g (1 - g),  z = f g
              dh_in[t]  = dh_out[t] [t >= id_start] + sum_j [Wf_j; Wg_j]^T dFG[t + (k-1-j)d]         t in [gs_in, L)
                          (dFG = 0 outside [gz, L), id_start = max(out_start, gs_out))
    weights   gws = sum_{t >= ds_start} dskip z^T,  gwr = sum_{t >= id_start} dh_out z^T,
              gw{f,g}[:, :, j] = sum_{t >= lo_j} d{F,G}[t] h[t - (k-1-j)d]^T,  lo_j = max(gz, in_start + (k-1-j)d)

Operand precision.  ``mode`` selects how every matrix product is formed; products are summed in float64, so only the operand
rounding of the kernels is modelled:
    "exact"   the float64 value of each operand
    "pairs"   hi*hi + lo*hi + hi*lo over bf16 (hi, lo) splits (stored pair planes are used as they are)
    "bf16"    hi*hi only: the hi plane of a stored pair, bf16(x) of an fp32 operand
An activation operand is either a float tensor (its fp32 value is split) or a tuple (hi, lo) of stored bf16 planes.  Outside
"exact", every output is also rounded the way the kernel stores it: ``pair_out`` -> a bf16 (hi, lo) pair of the fp32 value
(about 16 significant bits), otherwise fp32.

Layout converters between frames (B, L, C) and the kernels' chunked layouts are at the end."""
import torch

MODES = ("exact", "pairs", "bf16")


# ---------------------------------------------------------------------------------------------------- operand splits
def split_bf16(t):
    """fp32 -> (hi, lo) = (bf16(t), bf16(t - hi)) as fp32 tensors (round to nearest even, as __float2bfloat16_rn)."""
    t = t.float()
    hi = t.to(torch.bfloat16).to(torch.float32)
    return hi, (t - hi).to(torch.bfloat16).to(torch.float32)


def split_tf32(t):
    """fp32 -> (hi, lo) with hi = cvt.rna.tf32.f32(t) and lo = t - hi (exact in fp32)."""
    t = t.float().contiguous()
    hi = ((t.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)      # cvt.rna.tf32.f32: nearest, ties away
    return hi, t - hi


def _parts(x, mode):
    """(hi, lo) float64 operand planes of x for `mode` (lo is None where the mode has no second plane)."""
    if isinstance(x, tuple):
        hi, lo = x[0].double(), x[1].double()
        if mode == "exact":
            return hi + lo, None
        if mode == "pairs":
            return hi, lo
        if mode == "bf16":
            return hi, None
        raise ValueError(f"stored bf16 pairs have no {mode} form")
    if mode == "exact":
        return x.double(), None
    hi, lo = split_bf16(x)
    return hi.double(), (None if mode == "bf16" else lo.double())


def mm(x, w, mode):
    """out[..., n] = sum_k x[..., k] w[n, k], each product formed as `mode` forms it, summed in float64."""
    (xh, xl), (wh, wl) = _parts(x, mode), _parts(w, mode)
    y = xh @ wh.T
    if xl is not None:
        y = y + xl @ wh.T + xh @ wl.T
    return y


def contract(g, x, mode):
    """out[n, c] = sum_b sum_t g[b, t, n] x[b, t, c] (a weight gradient), operands formed as in mm."""
    (gh, gl), (xh, xl) = _parts(g, mode), _parts(x, mode)
    f = lambda a, b: a.reshape(-1, a.shape[-1]).T @ b.reshape(-1, b.shape[-1])
    y = f(gh, xh)
    if gl is not None:
        y = y + f(gl, xh) + f(gh, xl)
    return y


def value(x):
    """float64 value of a tensor or of a stored (hi, lo) pair."""
    return x[0].double() + x[1].double() if isinstance(x, tuple) else x.double()


def store(v, mode, pair_out):
    """v as the kernel stores it: unchanged in "exact", else a bf16 (hi, lo) pair of fp32(v) or fp32(v)."""
    if mode == "exact":
        return v
    return split_bf16(v.float()) if pair_out else v.float()


# ---------------------------------------------------------------------------------------------------- frame helpers
def _each(x, fn):
    return tuple(fn(v) for v in x) if isinstance(x, tuple) else fn(x)


def _mask(x, lo):
    """frames left of lo -> 0"""
    def f(v):
        v = v.clone()
        v[:, :max(0, lo)] = 0
        return v
    return _each(x, f)


def _shift(x, s):
    """y[:, t] = x[:, t - s] (zero where t - s is outside [0, L)); s < 0 reads later frames"""
    def f(v):
        y, L = torch.zeros_like(v), v.shape[1]
        if abs(s) < L:
            if s >= 0:
                y[:, s:] = v[:, :L - s]
            else:
                y[:, :L + s] = v[:, -s:]
        return y
    return _each(x, f)


def _from(x, t0):
    return _each(x, lambda v: v[:, t0:])


def _pad_left(x, n):
    """a tensor on its own frame axis starting at frame n -> the absolute axis (zeros in front)"""
    return _each(x, lambda v: torch.cat([v.new_zeros(v.shape[0], n, *v.shape[2:]), v], 1))


def _b(W, name):
    b = W.get(name)
    return 0.0 if b is None else b.double()


def layer_weights(params, i):
    """one layer's parameters (fp32 CPU tensors) from a state dict: wf, wg (D, R, k), wr (R, D, 1), ws (S, D, 1), biases or None"""
    g = lambda n: params.get(n)
    return dict(wf=g(f"filter_convs.{i}.weight"), wg=g(f"gate_convs.{i}.weight"), bf=g(f"filter_convs.{i}.bias"),
                bg=g(f"gate_convs.{i}.bias"), wr=g(f"residual_convs.{i}.weight"), ws=g(f"skip_convs.{i}.weight"),
                br=g(f"residual_convs.{i}.bias"), bs=g(f"skip_convs.{i}.bias"))


# ---------------------------------------------------------------------------------------------------- the block
def block_forward(h, W, d, in_start, out_start, skip_start, skip=None, mode="exact", pair_out=False):
    """h: (B, L, R) input (fp32 or stored pair), skip: (B, L - skip_start, S) running skip sum or None (skip_init).
    Returns float64 values: h_out (B, L - out_start, R), f, g, z (B, L - out_start, D), skip (B, L - skip_start, S); h_out
    stored as a pair if pair_out, everything else as fp32 (outside "exact")."""
    k = W["wf"].shape[2]
    hm = _mask(h, in_start)
    F = G = 0.0
    for j in range(k):
        hs = _from(_shift(hm, (k - 1 - j) * d), out_start)
        F = F + mm(hs, W["wf"][:, :, j], mode)
        G = G + mm(hs, W["wg"][:, :, j], mode)
    f, g = torch.tanh(F + _b(W, "bf")), torch.sigmoid(G + _b(W, "bg"))
    z = f * g
    if mode != "exact":
        z = z.float()                                       # the kernels form z in fp32 before splitting it
    h_out = mm(z, W["wr"][:, :, 0], mode) + _b(W, "br") + value(h)[:, out_start:]
    sk = mm(z[:, skip_start - out_start:], W["ws"][:, :, 0], mode) + _b(W, "bs")
    if skip is not None:
        sk = sk + value(skip)
    return dict(h_out=value(store(h_out, mode, pair_out)), f=value(store(f, mode, False)), g=value(store(g, mode, False)),
                z=value(store(z, mode, False)), skip=value(store(sk, mode, False)))


def expand_table(table, L, hop=None):
    """A condition table on the positions [0, L), float64 (B, L, 2D): a global table (B, 2D) gives every position its
    sequence's row; a frames table (B, F, 2D) gives position t frame t // hop."""
    t = table.double()
    if t.dim() == 2:
        return t[:, None].expand(-1, L, -1)
    return t[:, torch.arange(L) // hop]


def with_position_biases(W, pre, out_start, keep_bias=False):
    """W with per-position filter / gate biases on the block's output frames [out_start, L): pre (B, L, 2D) on the absolute
    axis, [filter | gate].  They replace bf / bg (a condition table already holds the biases) or, with keep_bias, add to them."""
    D = W["wf"].shape[0]
    p = pre[:, out_start:].double()
    Wm = dict(W)
    Wm["bf"] = p[..., :D] + (_b(W, "bf") if keep_bias else 0.0)
    Wm["bg"] = p[..., D:] + (_b(W, "bg") if keep_bias else 0.0)
    return Wm


def backward_ranges(L, k, d, in_start, out_start, gs_out, ds_start):
    """gz, id_start, gs_in of one block as the runtime derives them (wavenet_model._Runtime._backward_tb)"""
    gz = max(out_start, min(gs_out, ds_start))
    id_start = max(out_start, gs_out)
    gs_in = max(in_start, min(id_start, gz - (k - 1) * d))
    return gz, id_start, gs_in


def block_backward_data(fg, dh_out, dskip, W, d, in_start, out_start, gs_out, ds_start, gz, gs_in, mode="exact",
                        pair_out=False):
    """fg: (B, L, 2D) saved [tanh | sigmoid] outputs; dh_out: (B, L, R) or None (last layer); dskip: (B, L - ds_start, S).
    Returns float64 values dfg (B, L - gz, 2D), z (B, L - gz, D), dh_in (B, L - gs_in, R), and dfg_stored (the dF|dG operand
    of the dh_in product, on the absolute axis, as stored)."""
    k = W["wf"].shape[2]
    D = W["wf"].shape[0]
    dz = mm(_from(_pad_left(dskip, ds_start), gz), W["ws"][:, :, 0].T, mode)
    if dh_out is not None and gs_out < fg.shape[1]:
        dz = dz + mm(_from(_mask(dh_out, gs_out), gz), W["wr"][:, :, 0].T, mode)
    if mode != "exact":
        dz = dz.float().double()                            # the fp32 accumulator the epilogue reads
    f, g = fg[:, gz:, :D].double(), fg[:, gz:, D:].double()
    dfg = store(torch.cat([dz * g * (1 - f * f), dz * f * g * (1 - g)], 2), mode, pair_out)
    z = store(f * g, mode, pair_out)
    dfg_abs = _pad_left(dfg, gz)
    acc = 0.0
    for j in range(k):
        wj = torch.cat([W["wf"][:, :, j], W["wg"][:, :, j]], 0).T          # (R, 2D)
        acc = acc + mm(_from(_shift(dfg_abs, -(k - 1 - j) * d), gs_in), wj, mode)
    id_start = max(out_start, gs_out)
    if dh_out is not None and id_start < fg.shape[1]:
        acc = acc + value(_from(_mask(dh_out, id_start), gs_in))
    dh_in = store(acc, mode, pair_out)
    return dict(dfg=value(dfg), z=value(z), dh_in=value(dh_in), dfg_stored=dfg_abs)


def block_wgrad(dskip, dh_out, dfg, z, h, k, d, in_start, ds_start, id_start, gz, mode="exact"):
    """dskip (B, L - ds_start, S); dh_out (B, L, R) or None; dfg (B, L, 2D); z (B, L, D); h (B, L, R) the block input
    (absolute axis; each read from its first valid frame on).  Returns float64 gws (S, D, 1), gwr (R, D, 1), gwf, gwg
    (D, R, k), each rounded to fp32 outside "exact"."""
    L = value(z).shape[1]
    D, R = value(z).shape[2], value(h).shape[2]
    zm = _mask(z, gz)
    out = dict(gws=contract(dskip, _from(zm, ds_start), mode).unsqueeze(-1))
    if dh_out is not None and id_start < L:
        out["gwr"] = contract(_from(dh_out, id_start), _from(zm, id_start), mode).unsqueeze(-1)
    else:
        out["gwr"] = torch.zeros(R, D, 1, dtype=torch.float64)
    gfg = torch.zeros(2 * D, R, k, dtype=torch.float64)
    for j in range(k):
        sh = (k - 1 - j) * d
        lo = max(gz, in_start + sh)
        if lo < L:
            gfg[:, :, j] = contract(_from(dfg, lo), _each(h, lambda v: v[:, lo - sh:L - sh]), mode)
    out["gwf"], out["gwg"] = gfg[:D], gfg[D:]
    return {n: value(store(v, mode, False)) for n, v in out.items()}


# ---------------------------------------------------------------------------------------------------- layouts
def pair_from_frames(x):
    """fp32 frames (B, L, C) -> chunked pair (B, 2, C/8, L, 8) bf16: [b][plane hi, lo][c/8][t][c%8]"""
    B, L, C = x.shape
    hi, lo = split_bf16(x)
    return torch.stack([hi, lo], 1).view(B, 2, L, C // 8, 8).permute(0, 1, 3, 2, 4).to(torch.bfloat16).contiguous()


def planes_from_pair(p):
    """chunked pair (B, 2, C/8, L, 8) -> (hi, lo) fp32 frames (B, L, C)"""
    B, _, C8, L, _ = p.shape
    q = p.float().permute(0, 1, 3, 2, 4).reshape(B, 2, L, C8 * 8)
    return q[:, 0].contiguous(), q[:, 1].contiguous()


def chunks4_from_frames(x):
    """fp32 frames (B, T, C) -> chunked fp32 (B, C/4, T, 4): [b][c/4][t][c%4]"""
    B, T, C = x.shape
    return x.float().reshape(B, T, C // 4, 4).permute(0, 2, 1, 3).contiguous()


def frames_from_chunks4(x):
    """chunked fp32 (B, C/4, T, 4) -> frames (B, T, C)"""
    B, C4, T, _ = x.shape
    return x.permute(0, 2, 1, 3).reshape(B, T, C4 * 4)
