"""Training-path gradients on the GPU vs torch autograd over the CPU oracle (which follows the reference op for op).
Tolerance: max|a-b| / max|b| <= 1e-4 per parameter tensor."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import wavenet_oracle as O
from helpers import build_model, spec_from_golden, params_from_golden, rel_err, one_hot_cuda

pytestmark = pytest.mark.gpu
TOL = 1e-4


def oracle_grads(p, spec, x, target):
    p = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    loss = F.cross_entropy(O.forward(p, spec, x), target)
    loss.backward()
    return float(loss.detach()), {k: v.grad for k, v in p.items()}


@pytest.mark.parametrize("name,out_len", [("odd_bias", 5), ("odd_bias", 40), ("k3", 4), ("deep", 100), ("deep", 3)])
def test_gradients_match_oracle_autograd(golden, name, out_len):
    g = golden(f"net_{name}.npz")
    spec = spec_from_golden(g, output_length=out_len)
    p = params_from_golden(g)
    idx = torch.from_numpy(g["idx"])
    B = idx.shape[0]
    x = O.one_hot(idx, 256)
    target = torch.randint(0, 256, (B * out_len,), generator=torch.Generator().manual_seed(3))
    want_loss, want = oracle_grads(p, spec, x, target)
    m = build_model(g, output_length=out_len)
    m.zero_grad()
    loss = F.cross_entropy(m(x.cuda()), target.cuda())
    loss.backward()
    assert abs(float(loss) - want_loss) < 1e-5
    got = {k: v.grad.cpu() for k, v in m.named_parameters()}
    assert set(got) == set(want)
    for k in want:
        if want[k] is None:                 # unused by the loss (the last block's residual conv): autograd gives None
            assert float(got[k].abs().max()) == 0.0, k
            want[k] = torch.zeros_like(got[k])
            continue
        assert got[k].shape == want[k].shape
        assert rel_err(got[k].numpy(), want[k].numpy()) < TOL, k
    # index-input path gives the same gradients
    m.zero_grad()
    F.cross_entropy(m.forward_indices(idx.cuda()), target.cuda()).backward()
    for k, v in m.named_parameters():
        if float(want[k].abs().max()) == 0.0:
            assert float(v.grad.abs().max()) == 0.0, k
        else:
            assert rel_err(v.grad.cpu().numpy(), want[k].numpy()) < TOL, k
    # gradients accumulate like autograd's
    F.cross_entropy(m.forward_indices(idx.cuda()), target.cuda()).backward()
    assert rel_err(m.end_conv_2.weight.grad.cpu().numpy(), 2 * want["end_conv_2.weight"].numpy()) < TOL


@pytest.mark.parametrize("classes", [100, 257, 1000])
@pytest.mark.parametrize("mode", ["ffma", "tb"])
def test_gradients_at_other_class_counts(classes, mode):
    """Class counts other than 256 through the whole training path -- index start conv (uint8 up to 256 classes, int64
    above), the head's ragged logits and dlogits, fused_cross_entropy and the start-conv scatter -- on the FFMA blocks and
    on the fused 256-wide tensor-core blocks, against float64 autograd over the oracle."""
    import wavenet_model as wmod
    import wavenet_training as wt
    from helpers import separate_head_relu_ties
    C = 256 if mode == "tb" else 24
    kw = dict(layers=3, blocks=1, dilation_channels=C, residual_channels=C, skip_channels=C, end_channels=72, classes=classes,
              output_length=40, kernel_size=2, bias=True)
    spec = O.NetSpec(**kw)
    torch.manual_seed(classes)
    m = wmod.WaveNetModel(**kw)
    B, L = 2, spec.receptive_field + spec.output_length - 1 + 30
    g = torch.Generator().manual_seed(classes + 1)
    idx = torch.randint(0, classes, (B, L), generator=g)
    idx[0, -1], idx[1, -2] = classes - 1, 0
    target = torch.randint(0, classes, (B * spec.output_length,), generator=g)
    x = O.one_hot(idx, classes)
    p = separate_head_relu_ties({k: v.detach() for k, v in m.state_dict().items()}, spec, x, spec.output_length)
    m.load_state_dict(p)
    pd = {k: v.double().requires_grad_(True) for k, v in p.items()}
    want_loss = F.cross_entropy(O.forward_direct(pd, spec, x.double()), target)
    want_loss.backward()
    m = m.cuda()
    rt = m._runtime()
    rt.block_mode = "ffma" if mode == "ffma" else "auto"
    xi = idx.to(torch.uint8 if classes <= 256 else torch.int64).cuda()
    loss = wt.fused_cross_entropy(m.forward_indices(xi), target.cuda())
    loss.backward()
    assert rt.last_block_mode == mode
    assert abs(float(loss) - float(want_loss)) < 1e-5 * float(want_loss)
    for k, v in m.named_parameters():
        if pd[k].grad is None:              # the last block's residual conv does not reach the loss
            assert float(v.grad.abs().max()) == 0.0, k
            continue
        assert rel_err(v.grad.cpu().numpy(), pd[k].grad.numpy()) < TOL, k


def test_training_step_reduces_loss(golden):
    """A few SGD steps on a fixed batch through the CUDA forward+backward lower the loss (wavenet_training.py:64-76)."""
    g = golden("net_deep.npz")
    m = build_model(g, output_length=64)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    idx = torch.from_numpy(g["idx"]).cuda()
    target = idx[:, -64:].reshape(-1)
    losses = []
    for _ in range(8):
        opt.zero_grad()
        loss = F.cross_entropy(m.forward_indices(idx), target)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0] - 0.05, losses


def test_backward_full_size_smoke():
    """cfg 3 shape, B=2: backward runs, gradients are finite and non-trivial, per-sample gradients add up."""
    import wavenet_model as wmod
    torch.manual_seed(0)
    m = wmod.WaveNetModel(layers=10, blocks=5, dilation_channels=256, residual_channels=256, skip_channels=256,
                          end_channels=256, classes=256, output_length=2000, kernel_size=2).cuda()
    idx = torch.randint(0, 256, (2, 9000), generator=torch.Generator().manual_seed(1)).cuda()
    tgt = torch.randint(0, 256, (2, 2000), generator=torch.Generator().manual_seed(2)).cuda()

    def grads(rows):
        m.zero_grad()
        F.cross_entropy(m.forward_indices(idx[rows]), tgt[rows].reshape(-1), reduction="sum").backward()
        return {k: v.grad.clone() for k, v in m.named_parameters()}

    both, g0, g1 = grads([0, 1]), grads([0]), grads([1])
    for k in both:
        assert bool(torch.isfinite(both[k]).all())
        assert rel_err((g0[k] + g1[k]).cpu().numpy(), both[k].cpu().numpy()) < 1e-4, k
    assert float(both["filter_convs.0.weight"].abs().max()) > 0


@pytest.mark.parametrize("B,rows,N,C,ldg,ldx,k,j", [
    (3, 37, 17, 5, 19, 7, 1, 0),            # ragged channel counts and pitches: scalar loads, partial tiles
    (2, 3001, 512, 256, 512, 256, 2, 1),    # the 256-channel filter+gate shape, strided scatter into (out, in, k)
    (2, 100, 130, 132, 136, 140, 3, 2),     # tiles that straddle 128 in both directions
    (1, 9, 8, 8, 8, 8, 1, 0),               # fewer frames than one slab
    (4, 0, 16, 12, 16, 12, 2, 0),           # no frames: zeros
])
def test_wn_wgrad_matches_float64_contraction(B, rows, N, C, ldg, ldx, k, j):
    """wn_wgrad through the C ABI: dw[n, c, j] = sum_b sum_t g[b, t, n] * x[b, t, c] with pitched, offset operands."""
    import ctypes, native
    lib = native.lib()
    gen = torch.Generator().manual_seed(5)
    g_off, x_off = 4, 8                                      # floats; keeps 16-byte alignment for the vector path
    gbuf = torch.randn(g_off + B * (rows + 2) * ldg, generator=gen).cuda()
    xbuf = torch.randn(x_off + B * (rows + 3) * ldx, generator=gen).cuda()
    g_seq, x_seq = (rows + 2) * ldg, (rows + 3) * ldx
    gv = gbuf[g_off:g_off + B * g_seq].view(B, rows + 2, ldg)[:, :rows, :N].double()
    xv = xbuf[x_off:x_off + B * x_seq].view(B, rows + 3, ldx)[:, :rows, :C].double()
    want = torch.einsum("btn,btc->nc", gv, xv).cpu().numpy()
    out = torch.full((N, C, k), 7.0, device="cuda")
    work = torch.empty(lib.wn_wgrad_workspace_bytes(N, C) // 4, device="cuda")
    a = native.WgradArgs()
    a.d_g, a.d_x = gbuf.data_ptr() + 4 * g_off, xbuf.data_ptr() + 4 * x_off
    a.d_dw, a.d_work = out.data_ptr() + 4 * j, work.data_ptr()
    a.g_seq_stride, a.x_seq_stride, a.dw_n_stride, a.dw_c_stride = g_seq, x_seq, C * k, k
    a.ldg, a.ldx, a.B, a.rows, a.N, a.C = ldg, ldx, B, rows, N, C
    native.check(lib.wn_wgrad(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), "wgrad")
    got = out.cpu().numpy()
    if rows == 0:
        assert np.abs(got[:, :, j]).max() == 0.0
    else:
        assert rel_err(got[:, :, j], want) < 1e-5
    for jj in range(k):                                      # the other taps' columns are untouched
        if jj != j:
            assert (got[:, :, jj] == 7.0).all()
    # bad arguments are reported, not launched
    a.ldg = N - 1
    assert lib.wn_wgrad(ctypes.byref(a), None) < 0


@pytest.mark.parametrize("B,rows,N,ldg,ldx,k,j", [
    (2, 3001, 512, 512, 256, 2, 1),         # the filter+gate shape: 4 row tiles, ragged last slab, strided scatter
    (3, 100, 128, 136, 260, 1, 0),          # one row tile, pitched operands, few slabs per split
    (1, 16, 256, 256, 256, 1, 0),           # a single slab
    (5, 37, 256, 256, 256, 3, 2),           # sequences shorter than three slabs, zero fill at every sequence end
])
def test_wn_tc_wgrad_matches_float64_contraction(B, rows, N, ldg, ldx, k, j):
    """wn_tc_wgrad (tensor cores, bf16 pairs) against the float64 contraction and against wn_wgrad."""
    import ctypes, native
    lib = native.lib()
    C = 256
    assert lib.wn_tc_wgrad_supported(N, C) and not lib.wn_tc_wgrad_supported(N, 128) and not lib.wn_tc_wgrad_supported(100, C)
    gen = torch.Generator().manual_seed(7)
    g_off, x_off = 4, 8
    gbuf = torch.randn(g_off + B * (rows + 2) * ldg, generator=gen).cuda()
    xbuf = torch.randn(x_off + B * (rows + 3) * ldx, generator=gen).cuda()
    g_seq, x_seq = (rows + 2) * ldg, (rows + 3) * ldx
    gv = gbuf[g_off:g_off + B * g_seq].view(B, rows + 2, ldg)[:, :rows, :N].double()
    xv = xbuf[x_off:x_off + B * x_seq].view(B, rows + 3, ldx)[:, :rows, :C].double()
    want = torch.einsum("btn,btc->nc", gv, xv).cpu().numpy()
    work = torch.empty(lib.wn_wgrad_workspace_bytes(N, C) // 4, device="cuda")
    outs = {}
    for name, fn in (("tc", lib.wn_tc_wgrad), ("fma", lib.wn_wgrad)):
        out = torch.full((N, C, k), 7.0, device="cuda")
        a = native.WgradArgs()
        a.d_g, a.d_x = gbuf.data_ptr() + 4 * g_off, xbuf.data_ptr() + 4 * x_off
        a.d_dw, a.d_work = out.data_ptr() + 4 * j, work.data_ptr()
        a.g_seq_stride, a.x_seq_stride, a.dw_n_stride, a.dw_c_stride = g_seq, x_seq, C * k, k
        a.ldg, a.ldx, a.B, a.rows, a.N, a.C = ldg, ldx, B, rows, N, C
        native.check(fn(ctypes.byref(a), torch.cuda.current_stream().cuda_stream), name)
        outs[name] = out.cpu().numpy()
    assert rel_err(outs["fma"][:, :, j], want) < 1e-5
    assert rel_err(outs["tc"][:, :, j], want) < 5e-5, rel_err(outs["tc"][:, :, j], want)
    for jj in range(k):
        if jj != j:
            assert (outs["tc"][:, :, jj] == 7.0).all()
    a.ldx = 258                                              # pitch not a multiple of 4 floats: rejected, not launched
    assert lib.wn_tc_wgrad(ctypes.byref(a), None) < 0
