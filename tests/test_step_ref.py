"""The float64 references of tests/step_ref.py against the oracle, float64 autograd and float64 torch.optim / F.cross_entropy
(CPU).  The kernel-level GPU tests (test_gpu_step_kernels_f64.py) hold the start-conv, head, loss, optimizer and reduction
kernels to these references, so each is pinned here on a ragged net with 11 classes, and each deliberately wrong variant
must miss."""
import pytest
import torch
import torch.nn.functional as F

import step_ref as SR
from oracle import wavenet_oracle as O


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / max(float(b.double().abs().max()), 1e-300))


def _net(classes=11):
    spec = O.NetSpec(layers=3, blocks=2, dilation_channels=6, residual_channels=5, skip_channels=7, end_channels=9,
                     classes=classes, output_length=5, kernel_size=2, bias=True)
    return spec, {k: v.double() for k, v in O.init_params(spec, seed=3).items()}


def test_start_conv_matches_oracle():
    spec, p = _net()
    w, b = p["start_conv.weight"], p["start_conv.bias"]
    g = torch.Generator().manual_seed(0)
    idx = torch.randint(0, spec.classes, (2, 40), generator=g)
    want = F.conv1d(O.one_hot(idx, spec.classes).double(), w, b).transpose(1, 2)
    assert _rel(SR.start_index(idx, w, b), want) < 1e-15
    assert _rel(SR.start_dense(O.one_hot(idx, spec.classes), w, b), want) < 1e-15
    x = torch.randn(2, spec.classes, 40, generator=g, dtype=torch.float64)            # dense, not one-hot
    assert _rel(SR.start_dense(x, w, b), F.conv1d(x, w, b).transpose(1, 2)) < 1e-14
    # out-of-range indices clamp to the nearest class; the flag sees them
    bad = idx.clone()
    bad[0, 0], bad[1, 3] = -1, spec.classes
    fixed = bad.clamp(0, spec.classes - 1)
    assert torch.equal(SR.start_index(bad, w, b), SR.start_index(fixed, w, b))
    assert SR.index_out_of_range(bad, spec.classes) and not SR.index_out_of_range(idx, spec.classes)
    # the stored pair planes: the fp32 value w[c] + b split once into bf16 (hi, lo), about 16 significant bits
    hi, lo = SR.start_pair_planes(idx, w.float(), b.float())
    assert torch.equal(hi, SR.start_index_fp32(idx, w.float(), b.float()).bfloat16().float())
    assert _rel(hi.double() + lo.double(), want) < 2 ** -16
    # wrong variants: bias left out, classes off by one
    assert _rel(SR.start_index(idx, w, None), want) > 1e-2
    assert _rel(SR.start_index((idx + 1) % spec.classes, w, b), want) > 1e-2


def _head_case():
    spec, p = _net()
    g = torch.Generator().manual_seed(1)
    idx = torch.randint(0, spec.classes, (2, 60), generator=g)
    taps = {}
    x = O.one_hot(idx, spec.classes).double()
    y = O.stack_direct(p, spec, x, taps)
    return spec, p, taps, y, idx


def test_head_forward_matches_oracle():
    spec, p, taps, y, idx = _head_case()
    OL, L = spec.output_length, idx.shape[1]
    skip = taps["skip"].transpose(1, 2)                         # (B, T_final, S): frames of skip from skip_start = L - T_final
    args = (p["end_conv_1.weight"], p["end_conv_1.bias"], p["end_conv_2.weight"], p["end_conv_2.bias"])
    got = SR.head_forward(skip, *args, OL)
    want = O.forward(p, spec, O.one_hot(idx, spec.classes).double())
    assert got.shape == (2 * OL, spec.classes)
    assert _rel(got, want) < 1e-13
    assert _rel(got, O.forward_direct(p, spec, O.one_hot(idx, spec.classes).double())) < 1e-13
    # wrong variants: no relu on skip, frames one early
    w1, b1, w2, b2 = args
    no_relu = ((skip[:, -OL:] @ w1[:, :, 0].T + b1).relu() @ w2[:, :, 0].T + b2).reshape(-1, spec.classes)
    assert _rel(no_relu, want) > 1e-3
    assert _rel(SR.head_forward(skip[:, :-1], *args, OL), want) > 1e-3


def test_head_backward_matches_autograd():
    spec, p, _, _, idx = _head_case()
    OL = spec.output_length
    x = O.one_hot(idx, spec.classes).double().requires_grad_(True)
    taps = {}
    y = O.stack_direct(p, spec, x, taps)
    sk, pre1 = taps["skip"], taps["pre1"]
    cot = torch.randn(2 * OL, spec.classes, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    logits = y[:, :, -OL:].transpose(1, 2).reshape(-1, spec.classes)
    dsk, dpre1 = torch.autograd.grad((logits * cot).sum(), [sk, pre1])
    skip = sk.detach().transpose(1, 2)
    assert SR.head_relu_margin(skip, p["end_conv_1.weight"], p["end_conv_1.bias"], OL) > 1e-6
    got = SR.head_backward_data(cot, skip, p["end_conv_1.weight"], p["end_conv_1.bias"], p["end_conv_2.weight"], OL)
    assert _rel(got["dskip"], dsk.transpose(1, 2)[:, -OL:]) < 1e-13
    assert float(dsk[:, :, :-OL].abs().max()) == 0                 # frames left of the output window get no gradient
    assert _rel(got["dy1"], dpre1.transpose(1, 2)[:, -OL:]) < 1e-13
    assert _rel(got["y1"], pre1.detach().relu().transpose(1, 2)[:, -OL:]) < 1e-15
    # wrong variant: the skip ReLU's mask left out
    wrong = got["dy1"] @ p["end_conv_1.weight"][:, :, 0]
    assert _rel(wrong, dsk.transpose(1, 2)[:, -OL:]) > 1e-3


@pytest.mark.parametrize("N,C,scale,offset", [(1, 1, 1.0, 0.0), (37, 11, 3.0, 0.0), (5, 1025, 3.0, 0.0), (3, 256, 80.0, 0.0),
                                              (4, 100, 3.0, 1e4)])
def test_cross_entropy_matches_torch_f64(N, C, scale, offset):
    g = torch.Generator().manual_seed(N + C)
    x = torch.randn(N, C, generator=g, dtype=torch.float64) * scale + offset
    t = torch.randint(0, C, (N,), generator=g)
    t[0] = C - 1
    xr = x.clone().requires_grad_(True)
    want = F.cross_entropy(xr, t)
    want.backward()
    want = want.detach()
    loss, d = SR.cross_entropy(x, t)
    assert abs(float(loss) - float(want)) <= 1e-13 * max(1.0, abs(float(want)))
    assert _rel(d, xr.grad) < 1e-12
    if C > 1:    # wrong variant: the mean over classes instead of rows
        assert abs(float(loss) * N / C - float(want)) > 1e-3 * abs(float(want))


def test_cross_entropy_offset_row_rounding():
    """the float32 form logf(s) + mx - x[t] rounds at the ulp of the largest logit; logf(s) + (mx - x[t]) does not"""
    g = torch.Generator().manual_seed(5)
    x = (1e4 + 3 * torch.randn(64, 256, generator=g)).float()
    t = torch.randint(0, 256, (64,), generator=g)
    loss, _ = SR.cross_entropy(x, t)
    rows = []
    for fused_first in (True, False):
        mx = x.max(1).values
        s = torch.exp(x - mx[:, None]).sum(1)
        xt = x.gather(1, t.view(-1, 1))[:, 0]
        r = (torch.log(s) + mx) - xt if fused_first else torch.log(s) + (mx - xt)
        rows.append(r.double())
    want = torch.stack([SR.cross_entropy(x[i:i + 1], t[i:i + 1])[0] for i in range(64)])
    assert float((rows[0] - want).abs().max()) > 1e-4
    assert float((rows[1] - want).abs().max()) < 1e-5
    assert abs(float(want.mean()) - float(loss)) < 1e-12


def test_adam_matches_torch_f64_with_per_parameter_steps():
    g = torch.Generator().manual_seed(7)
    shapes = [(5, 3), (7,), (4, 2, 2)]
    init = [torch.randn(s, generator=g, dtype=torch.float64) for s in shapes]
    hyper = dict(lr=3e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    ref = SR.Adam(init, **hyper)
    tp = [torch.nn.Parameter(t.clone()) for t in init]
    opt = torch.optim.Adam(tp, **hyper)
    for step in range(6):
        grads = [torch.randn(s, generator=g, dtype=torch.float64) * (step + 1) for s in shapes]
        grads[1] = None if step < 2 or step == 4 else grads[1]            # parameter 1: first gradient at step 3, none at 5
        for q, gr in zip(tp, grads):
            q.grad = None if gr is None else gr.clone()
        opt.step()
        ref.step(grads)
    for i, q in enumerate(tp):
        st = opt.state[q]
        assert ref.steps[i] == int(st["step"])
        assert _rel(ref.p[i], q.detach()) < 1e-14
        assert _rel(ref.m[i], st["exp_avg"]) < 1e-14 and _rel(ref.v[i], st["exp_avg_sq"]) < 1e-14
    assert ref.steps == [6, 3, 6]
    # wrong variant: one step count for the group, as if parameter 1 were at step 6 -- its first updates were 0.64x
    p1 = init[1].clone()
    m1 = v1 = torch.zeros_like(p1)
    u_own = SR.adam_update(p1, torch.ones(7, dtype=torch.float64), m1, v1, 1, **hyper)[0] - p1
    u_grp = SR.adam_update(p1, torch.ones(7, dtype=torch.float64), m1, v1, 3, **hyper)[0] - p1
    assert _rel(u_grp, u_own) > 0.3


def test_scatter_rows_and_colsum():
    g = torch.Generator().manual_seed(9)
    idx = torch.randint(-1, 12, (2, 30), generator=g)
    dh = torch.randn(2, 30, 4, generator=g)
    table, mag = SR.scatter_rows(idx, dh, 11, 5)
    want = torch.zeros(11, 4, dtype=torch.float64)
    for b in range(2):
        for t in range(5, 30):
            want[min(max(int(idx[b, t]), 0), 10)] += dh[b, t].double()
    assert _rel(table, want) < 1e-15 and bool((mag >= table.abs()).all())
    assert _rel(SR.scatter_rows(idx, dh, 11, 4)[0], want) > 1e-3         # wrong variant: t_begin one early
    x = torch.randn(300, 9, generator=g)
    s, a = SR.colsum(x, 257, 7)
    assert _rel(s, x[:257, :7].double().sum(0)) < 1e-15 and bool((a >= s.abs()).all())
