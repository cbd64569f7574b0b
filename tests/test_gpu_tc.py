"""Tensor-core (wgmma) residual blocks vs the exact-fp32 SIMT blocks, the golden reference outputs and the CPU oracle.
The bf16-pair operand split must hold the 1e-4 parity bar (expected around 1e-6)."""
import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from helpers import build_model, one_hot_cuda, rel_err, separate_head_relu_ties

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("precision", ["bf16x2"])
def test_tc_blocks_match_ffma_and_oracle(precision):
    import wavenet_model as wmod
    kw = dict(layers=4, blocks=2, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
              classes=256, output_length=300, kernel_size=2, bias=True)
    torch.manual_seed(5)
    m = wmod.WaveNetModel(**kw)
    spec = O.NetSpec(**kw)
    p = {k: v.detach().clone() for k, v in m.state_dict().items()}
    idx = torch.randint(0, 256, (2, 700), generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        want = O.forward(p, spec, O.one_hot(idx, 256)).numpy()
    m = m.cuda()
    rt = m._runtime()
    assert rt.tc_precision == "bf16x2"                          # the default operand split
    for unknown in ("fp8", "tf32x3"):
        rt.tc_precision = unknown
        with pytest.raises(ValueError), torch.no_grad():
            m.forward_indices(idx.cuda())
    rt.tc_precision = precision
    with torch.no_grad():
        rt.block_mode = "ffma"
        y0 = m.forward_indices(idx.cuda()).cpu().numpy()
        assert rt.last_block_mode == "ffma"
        rt.block_mode = "tc"
        y1 = m.forward_indices(idx.cuda()).cpu().numpy()
        assert rt.last_block_mode == "tc"
        full = m.wavenet(one_hot_cuda(idx.numpy()), m.wavenet_dilate).cpu().numpy()
    assert rel_err(y0, want) < 1e-4
    assert rel_err(y1, want) < 1e-4, f"tc vs oracle {rel_err(y1, want):.3e}"
    assert rel_err(y1, y0) < 2e-5, f"tc vs ffma {rel_err(y1, y0):.3e}"
    with torch.no_grad():
        want_full = O.stack_folded(p, spec, O.one_hot(idx, 256), lambda h, d, i0, i: O.fold_time(h, d, i0)).numpy()
    assert rel_err(full, want_full) < 1e-4                      # incl. the zero-history (padding) region


def test_tc_cfg2_golden_and_auto_mode(golden):
    g = golden("net_cfg2.npz")
    m = build_model(g)
    rt = m._runtime()
    assert rt.block_mode == "auto"
    with torch.no_grad():
        y = m(one_hot_cuda(g["idx"]))
    assert rt.last_block_mode == "tb"                           # 256-channel nets take the fused tensor-core path by default
    assert rel_err(y.cpu().numpy(), g["fwd"]) < 1e-4
    small = build_model(golden("net_deep.npz"))
    with torch.no_grad():
        small(one_hot_cuda(golden("net_deep.npz")["idx"]))
    assert small._runtime().last_block_mode == "ffma"           # 64 channels: SIMT path


def test_tc_full_size_batch_independence():
    import wavenet_model as wmod
    torch.manual_seed(0)
    m = wmod.WaveNetModel(layers=10, blocks=5, dilation_channels=256, residual_channels=256, skip_channels=256,
                          end_channels=256, classes=256, output_length=5000, kernel_size=2).cuda()
    idx = torch.randint(0, 256, (4, 16000), generator=torch.Generator().manual_seed(1234)).cuda()
    rt = m._runtime()
    with torch.no_grad():
        rt.block_mode = "tc"
        y = m.forward_indices(idx).view(4, -1, 256)
        y2 = m.forward_indices(idx[2:3]).view(1, -1, 256)
        rt.block_mode = "ffma"
        y_ref = m.forward_indices(idx[2:3]).view(1, -1, 256)
    assert bool(torch.isfinite(y).all())
    assert torch.equal(y[2], y2[0])
    assert rel_err(y2.cpu().numpy(), y_ref.cpu().numpy()) < 2e-5          # bf16 pairs, 50 layers deep


def test_tc_backward_matches_simt_backward_and_oracle():
    """256-channel net: tensor-core data gradients vs the fp32 SIMT kernels and vs autograd over the CPU oracle."""
    import torch.nn.functional as F
    import wavenet_model as wmod
    kw = dict(layers=3, blocks=2, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
              classes=256, output_length=150, kernel_size=2, bias=True)
    torch.manual_seed(11)
    m = wmod.WaveNetModel(**kw)
    spec = O.NetSpec(**kw)
    idx = torch.randint(0, 256, (2, 420), generator=torch.Generator().manual_seed(2))
    tgt = torch.randint(0, 256, (2 * 150,), generator=torch.Generator().manual_seed(3))
    # keep every head ReLU input of this case away from zero (see helpers.separate_head_relu_ties): a mask flipped by
    # a 1e-7 difference is a discontinuity of the gradient itself, not an error of either kernel family
    sep = separate_head_relu_ties(m.state_dict(), spec, O.one_hot(idx, 256), 150)
    m.load_state_dict(sep, strict=True)
    p = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    F.cross_entropy(O.forward(p, spec, O.one_hot(idx, 256)), tgt).backward()
    m = m.cuda()
    rt = m._runtime()
    grads = {}
    for mode, wgrad in (("tc", "tc"), ("ffma", "native")):
        rt.block_mode, rt.wgrad_mode = mode, wgrad
        m.zero_grad()
        F.cross_entropy(m.forward_indices(idx.cuda()), tgt.cuda()).backward()
        assert rt.last_bwd_mode == rt.block_mode
        assert (rt.wgrad_tc_calls > 0) == (wgrad == "tc")        # tensor-core weight gradients ran iff asked for
        grads[mode] = {k: v.grad.detach().cpu().numpy().copy() for k, v in m.named_parameters()}
    rt.block_mode, rt.wgrad_mode = "auto", "tc"
    bad = []
    for k, v in p.items():
        want = np.zeros_like(grads["tc"][k]) if v.grad is None else v.grad.numpy()
        scale = np.abs(want).max()
        if scale == 0:
            assert np.abs(grads["tc"][k]).max() == 0 and np.abs(grads["ffma"][k]).max() == 0, k
            continue
        e_f = np.abs(grads["ffma"][k] - want).max() / scale
        e_t = np.abs(grads["tc"][k] - want).max() / scale
        e_tf = np.abs(grads["tc"][k] - grads["ffma"][k]).max() / scale
        if not (e_f < 1e-4 and e_t < 1e-4 and e_tf < 1e-4):
            bad.append((k, float(scale), float(e_f), float(e_t), float(e_tf)))
    assert not bad, bad[:12]


@pytest.mark.parametrize("R,D,S,k,bwd", [
    (256, 256, 256, 3, "tc"),          # three taps
    (512, 256, 256, 2, "tc"),          # R != S: the residual / skip split of the output tiles
    (256, 256, 512, 2, "tc"),
    (256, 128, 256, 2, "ffma"),        # D % 256 != 0: tensor-core forward, FFMA backward
])
def test_auto_mode_two_launch_shapes_match_oracle(R, D, S, k, bwd):
    """Nets the fused block does not cover take the two-launch tensor-core blocks under block_mode="auto"; a training step
    through the runtime (dispatch, packs, buffers, the per-layer backward) against the oracle and its autograd."""
    import torch.nn.functional as F
    import wavenet_model as wmod
    B, L, out_len = 2, 500, 90
    kw = dict(layers=3, blocks=2, dilation_channels=D, residual_channels=R, skip_channels=S, end_channels=256,
              classes=256, output_length=out_len, kernel_size=k, bias=True)
    torch.manual_seed(13)
    m = wmod.WaveNetModel(**kw)
    spec = O.NetSpec(**kw)
    idx = torch.randint(0, 256, (B, L), generator=torch.Generator().manual_seed(6))
    tgt = torch.randint(0, 256, (B * out_len,), generator=torch.Generator().manual_seed(7))
    m.load_state_dict(separate_head_relu_ties(m.state_dict(), spec, O.one_hot(idx, 256), out_len), strict=True)
    p = {n: v.detach().clone().requires_grad_(True) for n, v in m.state_dict().items()}
    want = O.forward(p, spec, O.one_hot(idx, 256))
    F.cross_entropy(want, tgt).backward()
    m = m.cuda()
    rt = m._runtime()
    assert rt.block_mode == "auto"
    y = m.forward_indices(idx.cuda())
    F.cross_entropy(y, tgt.cuda()).backward()
    assert rt.last_block_mode == "tc" and rt.last_bwd_mode == bwd
    e = rel_err(y.detach().cpu().numpy(), want.detach().numpy())
    bad = []
    for n, v in m.named_parameters():
        g = p[n].grad
        if g is None or float(g.abs().max()) == 0:
            assert float(v.grad.abs().max()) == 0, n
            continue
        eg = rel_err(v.grad.cpu().numpy(), g.numpy())
        if not eg < 1e-4:
            bad.append((n, eg))
    print(f"auto mode R={R} D={D} S={S} k={k}: logits {e:.2e}, backward {rt.last_bwd_mode}")
    assert e < 1e-4, e
    assert not bad, bad[:10]


def test_packed_weights_follow_parameter_writes():
    """ADVICE r1: the packed-weight cache is keyed on tensor versions, which writes through ``p.data`` do not bump (the
    reference's optimizers.py:100 updates that way).  A backward invalidates the cache; so does the explicit call."""
    import torch.nn.functional as F
    import wavenet_model as wmod
    kw = dict(layers=2, blocks=1, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
              classes=256, output_length=32, kernel_size=2, bias=False)
    torch.manual_seed(3)
    m = wmod.WaveNetModel(**kw).cuda()
    idx = torch.randint(0, 256, (1, 200), generator=torch.Generator().manual_seed(1)).cuda()
    tgt = torch.randint(0, 256, (32,), generator=torch.Generator().manual_seed(2)).cuda()
    with torch.no_grad():
        y0 = m.forward_indices(idx).clone()
    w = m.residual_convs[0].weight
    # (1) a training step whose "optimizer" writes through .data, then a no-grad forward (train -> validate)
    F.cross_entropy(m.forward_indices(idx), tgt).backward()
    w.data.mul_(1.5)
    with torch.no_grad():
        y1 = m.forward_indices(idx).clone()
    assert not torch.equal(y1, y0)
    # (2) a hand edit between no-grad forwards needs the explicit invalidate
    w.data.mul_(1.0 / 1.5)
    m.invalidate_packed_weights()
    with torch.no_grad():
        y2 = m.forward_indices(idx)
    assert rel_err(y2.cpu().numpy(), y0.cpu().numpy()) < 1e-5
    # (3) a second backward through a freed graph raises a clear error
    loss = F.cross_entropy(m.forward_indices(idx), tgt)
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="saved activations"):
        loss.backward()
