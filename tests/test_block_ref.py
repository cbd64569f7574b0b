"""The float64 single-block references of tests/block_ref.py, composed into a whole net, against the oracle (CPU).

The kernel-level GPU tests (test_gpu_kernels_f64.py) hold every block kernel to these references, so their frame-range rules
(in_start, out_start, skip_start, gs_out, ds_start, gz, id_start, gs_in, the per-tap lo of the weight gradients) are pinned
here: the composed forward must give oracle.forward's logits and the composed backward autograd's gradient of every parameter,
to float64 rounding."""
import pytest
import torch
import torch.nn.functional as F

import block_ref as BR
from oracle import wavenet_oracle as O


def _compose(p, spec, x, cot):
    """forward and backward of the whole net from the block references; cot: d(loss)/d(logits) (B*out_len, classes)"""
    k, L = spec.kernel_size, x.shape[2]
    dil = [d for d, _ in spec.dilation_schedule()]
    T, in_s, out_s = L, [], []
    for d in dil:
        t_out = -(-T // d) * d - d * (k - 1)
        in_s.append(L - T)
        out_s.append(L - t_out)
        T = t_out
    skip_start, OL = L - T, spec.output_length
    b = lambda n: p.get(n)
    h = F.conv1d(x, p["start_conv.weight"], b("start_conv.bias")).transpose(1, 2)          # frames (B, L, R), exact
    hs, fgs, skip = [h], [], None
    for i, d in enumerate(dil):
        W = BR.layer_weights(p, i)
        o = BR.block_forward(hs[-1], W, d, in_s[i], out_s[i], skip_start, skip)
        skip = o["skip"]
        nxt = torch.zeros_like(h)
        nxt[:, out_s[i]:] = o["h_out"]
        fg = torch.zeros(h.shape[0], L, 2 * W["wf"].shape[0], dtype=torch.float64)
        fg[:, out_s[i]:] = torch.cat([o["f"], o["g"]], 2)
        hs.append(nxt)
        fgs.append(fg)
    # head by autograd (not a block): logits and d(loss)/d(skip) of the last out_len frames
    sk = skip[:, -OL:].transpose(1, 2).detach().requires_grad_(True)
    y = F.relu(F.conv1d(F.relu(sk), p["end_conv_1.weight"], p["end_conv_1.bias"]))
    logits = F.conv1d(y, p["end_conv_2.weight"], p["end_conv_2.bias"]).transpose(1, 2).reshape(-1, spec.classes)
    (logits * cot).sum().backward()
    dskip = sk.grad.transpose(1, 2)
    grads, ds_start = {}, L - OL
    dh_out, gs_out = None, L
    for i in range(len(dil) - 1, -1, -1):
        d, W = dil[i], BR.layer_weights(p, i)
        gz, id_start, gs_in = BR.backward_ranges(L, k, d, in_s[i], out_s[i], gs_out, ds_start)
        o = BR.block_backward_data(fgs[i], dh_out, dskip, W, d, in_s[i], out_s[i], gs_out, ds_start, gz, gs_in)
        dfg = torch.zeros(fgs[i].shape, dtype=torch.float64)
        dfg[:, gz:] = o["dfg"]
        z = torch.zeros(dfg.shape[0], L, dfg.shape[2] // 2, dtype=torch.float64)
        z[:, gz:] = o["z"]
        g = BR.block_wgrad(dskip, dh_out, dfg, z, hs[i], k, d, in_s[i], ds_start, id_start, gz)
        grads[f"skip_convs.{i}.weight"], grads[f"residual_convs.{i}.weight"] = g["gws"], g["gwr"]
        grads[f"filter_convs.{i}.weight"], grads[f"gate_convs.{i}.weight"] = g["gwf"], g["gwg"]
        if f"skip_convs.{i}.bias" in p:
            D = W["wf"].shape[0]
            grads[f"skip_convs.{i}.bias"] = dskip.sum((0, 1))
            grads[f"residual_convs.{i}.bias"] = (dh_out[:, id_start:].sum((0, 1)) if dh_out is not None
                                                 else torch.zeros(W["wr"].shape[0], dtype=torch.float64))
            grads[f"filter_convs.{i}.bias"], grads[f"gate_convs.{i}.bias"] = dfg[:, gz:, :D].sum((0, 1)), dfg[:, gz:, D:].sum((0, 1))
        dh_out = torch.zeros_like(h)
        dh_out[:, gs_in:] = o["dh_in"]
        gs_out = gs_in
        grads[f"dh_in.{i}"] = dh_out
    dh0 = dh_out[:, gs_out:]
    grads["start_conv.weight"] = torch.einsum("btr,bct->rc", dh0, x[:, :, gs_out:]).unsqueeze(-1)
    if "start_conv.bias" in p:
        grads["start_conv.bias"] = dh0.sum((0, 1))
    return logits.detach(), grads, hs


def _rel(a, b):
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-300))


@pytest.mark.parametrize("k,bias,layers,blocks,B,L,out_len", [
    (2, True, 4, 2, 2, 60, 7),
    (2, False, 5, 1, 1, 70, 20),
    (3, True, 3, 2, 2, 50, 5),
    (3, False, 4, 1, 1, 80, 33),
])
def test_block_references_compose_to_the_oracle(k, bias, layers, blocks, B, L, out_len):
    torch.set_num_threads(min(8, torch.get_num_threads()))
    spec = O.NetSpec(layers=layers, blocks=blocks, dilation_channels=6, residual_channels=5, skip_channels=7, end_channels=9,
                     classes=11, output_length=out_len, kernel_size=k, bias=bias)
    p = {n: v.double().requires_grad_(True) for n, v in O.init_params(spec, seed=3).items()}
    g = torch.Generator().manual_seed(4)
    x = torch.randn(B, spec.classes, L, generator=g, dtype=torch.float64)        # dense input: every frame and class matters
    cot = torch.randn(B * out_len, spec.classes, generator=g, dtype=torch.float64)
    want = O.forward(p, spec, x)
    taps = {}
    (want * cot).sum().backward()
    with torch.no_grad():
        O.stack_direct({n: v.detach() for n, v in p.items()}, spec, x, taps)
    # the head ReLUs must not sit on a tie, or autograd and the composition may pick different one-sided derivatives
    assert float(taps["skip"][..., -out_len:].abs().min()) > 1e-9 and float(taps["pre1"][..., -out_len:].abs().min()) > 1e-9
    pd = {n: v.detach() for n, v in p.items()}
    got, grads, _ = _compose(pd, spec, x, cot)
    assert _rel(got, want.detach()) < 1e-12
    for n, v in p.items():
        if n.startswith("end_conv"):
            continue                                        # the head is autograd on both sides
        if v.grad is None:                                  # the last layer's residual conv feeds nothing
            assert float(grads[n].abs().max()) == 0, n
        else:
            assert _rel(grads[n], v.grad) < 1e-12, n


def test_block_reference_range_rules_are_tight():
    """The composition checks the rules only through parameters; a per-layer check shows a rule off by one frame changes
    the result (the references would otherwise be allowed to be sloppy where gradients are zero anyway)."""
    torch.set_num_threads(min(8, torch.get_num_threads()))
    spec = O.NetSpec(layers=4, blocks=1, dilation_channels=6, residual_channels=5, skip_channels=7, end_channels=9,
                     classes=11, output_length=9, kernel_size=2, bias=True)
    p = {n: v.double() for n, v in O.init_params(spec, seed=5).items()}
    x = torch.randn(1, spec.classes, 40, generator=torch.Generator().manual_seed(6), dtype=torch.float64)
    _, _, hs = _compose(p, spec, x, torch.ones(9, spec.classes, dtype=torch.float64))
    W, d = BR.layer_weights(p, 3), 8
    in_s, out_s = 4, 8                       # layer 3 of this net: input frames [4, 40), output frames [8, 40)
    ok = BR.block_forward(hs[3], W, d, in_s, out_s, out_s)["h_out"]
    assert _rel(ok, hs[4][:, out_s:]) < 1e-14
    assert _rel(BR.block_forward(hs[3], W, d + 1, in_s, out_s, out_s)["h_out"], ok) > 1e-3
    garbage = hs[3].clone()
    garbage[:, :in_s] = 100.0                # frames left of in_start must not be read
    assert _rel(BR.block_forward(garbage, W, d, in_s, out_s, out_s)["h_out"], ok) == 0
    assert _rel(BR.block_forward(garbage, W, d, in_s - 1, out_s, out_s)["h_out"], ok) > 1e-3


@pytest.mark.parametrize("term", ["global", "frames", "frames+global", "kslab", "kslab+global"])
def test_position_biases_compose_to_the_conditioned_references(term):
    """The whole-stack kernel tests (test_gpu_stack_kernels_f64.py) give block_forward each conditioned layer's term as
    per-position filter / gate biases: a global or frames condition table replacing bf / bg (expand_table), or the K-slab
    product U c[t] on top of the biases or of the global table.  Composed over a small net, that must reproduce the skip
    sum of local_ref.stack_direct / upsample_ref.stack_direct."""
    import local_ref
    import upsample_ref
    torch.set_num_threads(min(8, torch.get_num_threads()))
    spec = O.NetSpec(layers=3, blocks=2, dilation_channels=6, residual_channels=6, skip_channels=6, end_channels=9,
                     classes=11, output_length=9, kernel_size=2, bias=True)
    p = {n: v.double() for n, v in O.init_params(spec, seed=9).items()}
    g = torch.Generator().manual_seed(10)
    rnd = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64) * 0.5
    B, L, G, C, hop, D = 2, 70, 3, 4, 5, spec.dilation_channels
    dil = [d for d, _ in spec.dilation_schedule()]
    for i in range(len(dil)):
        for n in ("filter", "gate"):
            p[f"{n}_cond_convs.{i}.weight"], p[f"{n}_local_convs.{i}.weight"] = rnd(D, G, 1), rnd(D, C, 1)
    p["local_upsample.0.weight"], p["local_upsample.0.bias"] = rnd(C, C, 2 * hop), rnd(C)
    x = torch.randn(B, spec.classes, L, generator=g, dtype=torch.float64)
    h = rnd(B, G) if "global" in term else None
    y = rnd(B, C, -(-L // hop) + 2)
    taps = {}
    if term.startswith("kslab"):
        upsample_ref.stack_direct(p, spec, x, y, (hop,), h, taps)
        c = upsample_ref.upsample(p, (hop,), y)[:, :, :L].transpose(1, 2)
    else:
        local_ref.stack_direct(p, spec, x, y if term.startswith("frames") else None, hop, h, taps)
    want = taps["skip"].transpose(1, 2)
    T, in_s, out_s = L, [], []
    for d in dil:
        t_out = -(-T // d) * d - d
        in_s.append(L - T)
        out_s.append(L - t_out)
        T = t_out
    hs = F.conv1d(x, p["start_conv.weight"], p["start_conv.bias"]).transpose(1, 2)
    skip = None
    for i, d in enumerate(dil):
        W = BR.layer_weights(p, i)
        u = lambda n: torch.cat([p[f"filter_{n}_convs.{i}.weight"], p[f"gate_{n}_convs.{i}.weight"]], 0)[:, :, 0]
        table = torch.cat([W["bf"], W["bg"]]).double().expand(B, -1)                 # (B, 2D): the biases
        if h is not None:
            table = table + h @ u("cond").T
        if term.startswith("frames"):
            table = table[:, None] + (y.transpose(1, 2) @ u("local").T)              # (B, F, 2D): + U y_f per frame
        pre = BR.expand_table(table, L, hop)
        if term.startswith("kslab"):
            pre = pre + BR.mm(c, u("local"), "exact")
        o = BR.block_forward(hs, BR.with_position_biases(W, pre, out_s[i]), d, in_s[i], out_s[i], L - T, skip)
        skip = o["skip"]
        hs = torch.zeros_like(hs)
        hs[:, out_s[i]:] = o["h_out"]
    assert _rel(skip, want) < 1e-12


def test_layout_converters_round_trip():
    x = torch.randn(2, 37, 24, generator=torch.Generator().manual_seed(7)) * 3
    p = BR.pair_from_frames(x)
    assert p.shape == (2, 2, 3, 37, 8) and p.dtype == torch.bfloat16
    hi, lo = BR.planes_from_pair(p)
    assert torch.equal(hi, x.to(torch.bfloat16).float()) and torch.equal(p[1, 0, 2, 5], hi[1, 5, 16:24].to(torch.bfloat16))
    assert float(((hi + lo - x).abs() / x.abs()).max()) <= 2.0 ** -16
    c = BR.chunks4_from_frames(x)
    assert c.shape == (2, 6, 37, 4) and torch.equal(c[0, 1, 3], x[0, 3, 4:8])
    assert torch.equal(BR.frames_from_chunks4(c), x)


@pytest.mark.parametrize("mode", ["pairs", "bf16"])
def test_emulated_block_error_has_the_operand_width(mode):
    """Emulation of one 256-channel block on O(1) inputs: its distance from exact tracks the operand width (bf16: 8 bits,
    pairs: about 16 bits)."""
    torch.set_num_threads(min(8, torch.get_num_threads()))
    g = torch.Generator().manual_seed(8)
    C, L = 256, 96
    W = dict(wf=torch.randn(C, C, 2, generator=g) / 16, wg=torch.randn(C, C, 2, generator=g) / 16, bf=None, bg=None,
             wr=torch.randn(C, C, 1, generator=g) / 16, ws=torch.randn(C, C, 1, generator=g) / 16, br=None, bs=None)
    h = torch.randn(1, L, C, generator=g)
    ex = BR.block_forward(h, W, 3, 0, 3, 3)
    em = BR.block_forward(h, W, 3, 0, 3, 3, mode=mode)
    e = _rel(em["h_out"], ex["h_out"])
    lo, hi = {"pairs": (1e-7, 3e-5), "bf16": (3e-4, 3e-2)}[mode]
    assert lo < e < hi, e
