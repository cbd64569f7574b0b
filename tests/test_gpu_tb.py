"""The fused tensor-core block (csrc/tc_block.cu: wgmma, chunked bf16-pair activations, one launch per
residual block) against the CPU oracle, the golden outputs of the unmodified reference and the exact-fp32 SIMT blocks."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from helpers import build_model, one_hot_cuda, rel_err, separate_head_relu_ties, tie_free_indices

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _pair_emulation(x):
    hi = x.to(torch.bfloat16)
    lo = (x - hi.float()).to(torch.bfloat16)
    return hi, lo


def test_pair_layout_converters():
    """fp32 frames (B, L, C) <-> chunked pair [b][plane][c/8][t][c%8]: element placement, the split itself, the origin."""
    import native
    lib = native.lib()
    B, L, C, t_begin = 2, 333, 256, 17
    x = (torch.randn(B, L, C, generator=torch.Generator().manual_seed(1)) * 3).cuda()
    pair = torch.zeros(B, 2, C // 8, L, 8, device="cuda", dtype=torch.bfloat16)
    st = torch.cuda.current_stream().cuda_stream
    native.check(lib.wn_pair_from_frames(x.data_ptr(), pair.data_ptr(), B, L, C, t_begin, st), "to pair")
    hi, lo = _pair_emulation(x)
    want_hi = hi.view(B, L, C // 8, 8).permute(0, 2, 1, 3)
    want_lo = lo.view(B, L, C // 8, 8).permute(0, 2, 1, 3)
    assert torch.equal(pair[:, 0, :, t_begin:], want_hi[:, :, t_begin:]) and torch.equal(pair[:, 1, :, t_begin:], want_lo[:, :, t_begin:])
    assert float(pair[:, :, :, :t_begin].abs().max()) == 0                 # frames left of t_begin are not touched
    back = torch.full((B, L, C), 7.0, device="cuda")
    native.check(lib.wn_frames_from_pair(pair.data_ptr(), back.data_ptr(), B, L, C, t_begin, st), "from pair")
    assert torch.equal(back[:, t_begin:], (hi.float() + lo.float())[:, t_begin:]) and bool((back[:, :t_begin] == 7.0).all())
    assert rel_err(back[:, t_begin:].cpu().numpy(), x[:, t_begin:].cpu().numpy()) < 2.0 ** -16
    # chunked fp32 (B, C/4, T, 4) -> frames
    sk = torch.randn(B, C // 4, L, 4, device="cuda")
    out = torch.empty(B, 50, C, device="cuda")
    native.check(lib.wn_frames_from_chunks4(sk.data_ptr(), out.data_ptr(), B, L, C, L - 50, 50, st), "chunks4")
    assert torch.equal(out, sk[:, :, L - 50:].permute(0, 2, 1, 3).reshape(B, 50, C))


@pytest.mark.parametrize("B,L,layers,blocks,bias,out_len", [
    (1, 300, 3, 1, False, 64),        # a single 256-frame item and a 44-frame tail
    (2, 700, 4, 2, True, 300),        # several items per sequence, skip starts inside an item
    (3, 1203, 6, 2, True, 40),        # dilation 32 > tile overlap cases; most items lie left of skip_start
    (2, 515, 2, 3, False, 500),
])
def test_fused_blocks_match_oracle_and_simt(B, L, layers, blocks, bias, out_len):
    import wavenet_model as wmod
    kw = dict(layers=layers, blocks=blocks, dilation_channels=256, residual_channels=256, skip_channels=256,
              end_channels=256, classes=256, output_length=out_len, kernel_size=2, bias=bias)
    torch.manual_seed(5)
    m = wmod.WaveNetModel(**kw)
    spec = O.NetSpec(**kw)
    p = {k: v.detach().clone() for k, v in m.state_dict().items()}
    idx = torch.randint(0, 256, (B, L), generator=torch.Generator().manual_seed(9))
    with torch.no_grad():
        want = O.forward(p, spec, O.one_hot(idx, 256)).numpy()
        want_full = O.stack_folded(p, spec, O.one_hot(idx, 256), lambda h, d, i0, i: O.fold_time(h, d, i0)).numpy()
    m = m.cuda()
    rt = m._runtime()
    with torch.no_grad():
        y = m.forward_indices(idx.cuda())
        assert rt.last_block_mode == "tb"
        yu = m.forward_indices(idx.to(torch.uint8).cuda())
        yd = m(one_hot_cuda(idx.numpy()))                               # dense (one-hot float) input path
        full = m.wavenet(one_hot_cuda(idx.numpy()), m.wavenet_dilate)
        rt.block_mode = "ffma"
        y0 = m.forward_indices(idx.cuda())
        rt.block_mode = "auto"
        rows = [m.forward_indices(idx[b:b + 1].cuda()) for b in range(B)]
    assert torch.equal(y, yu) and torch.equal(y, yd)
    e = rel_err(y.cpu().numpy(), want)
    assert e < TOL, f"fused blocks vs oracle {e:.3e}"
    assert rel_err(y.cpu().numpy(), y0.cpu().numpy()) < 3e-5
    assert rel_err(full.cpu().numpy(), want_full) < TOL                  # all T_final columns incl. the zero-history region
    yb = y.view(B, out_len, 256)
    for b in range(B):
        assert torch.equal(yb[b], rows[b].view(out_len, 256))            # batch rows are independent, bit for bit


def test_fused_blocks_dense_non_one_hot_input():
    import wavenet_model as wmod
    kw = dict(layers=3, blocks=2, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
              classes=256, output_length=100, kernel_size=2, bias=True)
    torch.manual_seed(2)
    m = wmod.WaveNetModel(**kw)
    spec = O.NetSpec(**kw)
    p = {k: v.detach().clone() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(4)
    x = torch.rand(2, 256, 400, generator=g) * (torch.rand(2, 256, 400, generator=g) < 0.05)
    with torch.no_grad():
        want = O.forward(p, spec, x).numpy()
        got = m.cuda()(x.cuda())
    assert m._runtime().last_block_mode == "tb"
    assert rel_err(got.cpu().numpy(), want) < TOL


def test_fused_blocks_cfg2_golden(golden):
    g = golden("net_cfg2.npz")
    m = build_model(g)
    with torch.no_grad():
        y = m(one_hot_cuda(g["idx"]))
    assert m._runtime().last_block_mode == "tb"
    e = rel_err(y.cpu().numpy(), g["fwd"])
    assert e < TOL, e


def test_tb_mode_requires_supported_shape(golden):
    small = build_model(golden("net_deep.npz"))
    small._runtime().block_mode = "tb"
    with torch.no_grad(), pytest.raises(RuntimeError):
        small(one_hot_cuda(golden("net_deep.npz")["idx"]))


@pytest.mark.parametrize("B,L,layers,blocks,bias,out_len", [
    (2, 420, 3, 2, True, 150),
    (3, 700, 4, 2, True, 300),         # several 256-frame items, gradients start inside an item
    (1, 1100, 6, 1, False, 37),        # no biases; most frames lie outside the receptive cone of the outputs
    (2, 2200, 10, 1, True, 300),       # the benchmark's depth: dilations to 512 cross CTA and item boundaries; the
                                       # gradients start at frame 1900, inside an item (the reference needs a folded
                                       # length >= 2 at d = 512, so L >= ~2050)
])
def test_fused_backward_matches_oracle_and_simt(B, L, layers, blocks, bias, out_len):
    """Training step through the chunked-pair kernels (forward with saved activations, wgmma data gradients, MN-major
    wgmma weight gradients) vs autograd over the CPU oracle and vs the exact-fp32 SIMT kernels."""
    import torch.nn.functional as F
    import wavenet_model as wmod
    kw = dict(layers=layers, blocks=blocks, dilation_channels=256, residual_channels=256, skip_channels=256,
              end_channels=256, classes=256, output_length=out_len, kernel_size=2, bias=bias)
    torch.manual_seed(11)
    m = wmod.WaveNetModel(**kw)
    spec = O.NetSpec(**kw)
    idx = torch.randint(0, 256, (B, L), generator=torch.Generator().manual_seed(2))
    tgt = torch.randint(0, 256, (B * out_len,), generator=torch.Generator().manual_seed(3))
    # keep head ReLU inputs away from zero: a mask flipped by rounding noise is a discontinuity of the gradient itself (one
    # flipped element perturbs EVERY gradient by ~1e-3 through dskip).  Biases are nudged where they exist; a net without
    # skip biases gets an input whose relu(skip) arguments all stay clear of zero.
    if not bias:
        idx = tie_free_indices(m.state_dict(), spec, B, L, out_len)
    m.load_state_dict(separate_head_relu_ties(m.state_dict(), spec, O.one_hot(idx, 256), out_len), strict=True)
    p = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    F.cross_entropy(O.forward(p, spec, O.one_hot(idx, 256)), tgt).backward()
    m = m.cuda()
    rt = m._runtime()
    grads = {}
    for mode in ("auto", "ffma"):
        rt.block_mode = mode
        rt.wgrad_mode = "tc" if mode == "auto" else "native"
        m.zero_grad()
        loss = F.cross_entropy(m.forward_indices(idx.cuda()), tgt.cuda())
        loss.backward()
        assert rt.last_block_mode == ("tb" if mode == "auto" else "ffma") and rt.last_bwd_mode == rt.last_block_mode
        grads[mode] = {k: v.grad.detach().cpu().numpy().copy() for k, v in m.named_parameters()}
    rt.block_mode, rt.wgrad_mode = "auto", "tc"
    bad = []
    for k, v in p.items():
        want = np.zeros_like(grads["auto"][k]) if v.grad is None else v.grad.numpy()
        scale = np.abs(want).max()
        if scale == 0:
            assert np.abs(grads["auto"][k]).max() == 0, k
            continue
        e_t, e_f = np.abs(grads["auto"][k] - want).max() / scale, np.abs(grads["ffma"][k] - want).max() / scale
        if not (e_t < 1e-4 and e_f < 1e-4):
            bad.append((k, float(scale), float(e_t), float(e_f)))
    assert not bad, bad[:10]


# ------------------------------------------------------------------------------------------------ single-pass bf16 operands
# BASELINE.json configs[4] ("bf16 training", 512 channels).  The reference has no bf16 path, so the bar is stated here: the
# matrix products see bf16 operands (8 mantissa bits) with fp32 accumulation while the residual stream, skip and all
# gradients-of-activations stay fp32-class; logits must stay within 3e-2 and weight gradients within 6e-2 (max-relative) of
# the fp32 oracle on these nets.  Measured values are printed.
@pytest.mark.parametrize("channels,B,L,layers,blocks,out_len", [
    (256, 2, 700, 4, 2, 300),
    (512, 2, 600, 3, 2, 200),
    (512, 1, 1300, 6, 1, 64),
    (512, 2, 2200, 10, 1, 300),        # dilations to 512, gradients from frame 1900 (inside an item)
])
def test_single_pass_bf16_forward_backward(channels, B, L, layers, blocks, out_len):
    import torch.nn.functional as F
    import wavenet_model as wmod
    kw = dict(layers=layers, blocks=blocks, dilation_channels=channels, residual_channels=channels, skip_channels=channels,
              end_channels=256, classes=256, output_length=out_len, kernel_size=2, bias=True)
    torch.manual_seed(21)
    m = wmod.WaveNetModel(**kw)
    spec = O.NetSpec(**kw)
    idx = torch.randint(0, 256, (B, L), generator=torch.Generator().manual_seed(4))
    tgt = torch.randint(0, 256, (B * out_len,), generator=torch.Generator().manual_seed(5))
    m.load_state_dict(separate_head_relu_ties(m.state_dict(), spec, O.one_hot(idx, 256), out_len, margin=2e-3), strict=True)
    p = {k: v.detach().clone().requires_grad_(True) for k, v in m.state_dict().items()}
    want = O.forward(p, spec, O.one_hot(idx, 256))
    F.cross_entropy(want, tgt).backward()
    m = m.cuda()
    rt = m._runtime()
    rt.tc_precision = "bf16"
    with torch.no_grad():
        y = m.forward_indices(idx.cuda())
    assert rt.last_block_mode == "tb" and rt.last_precision == "bf16"
    e = rel_err(y.cpu().numpy(), want.detach().numpy())
    F.cross_entropy(m.forward_indices(idx.cuda()), tgt.cuda()).backward()
    assert rt.last_bwd_mode == "tb"
    worst = 0.0
    for k, v in m.named_parameters():
        g = p[k].grad
        if g is None or float(g.abs().max()) == 0:
            continue
        worst = max(worst, rel_err(v.grad.cpu().numpy(), g.numpy()))
    print(f"single-pass bf16, {channels} ch: logits {e:.2e}, worst gradient {worst:.2e}")
    assert 1e-5 < e < 3e-2, e
    assert worst < 6e-2, worst
    if channels == 256:                      # the same net through the pair kernels is two orders of magnitude closer
        rt.tc_precision = "bf16x2"
        with torch.no_grad():
            y2 = m.forward_indices(idx.cuda())
        assert rt.last_precision == "bf16x2" and rel_err(y2.cpu().numpy(), want.detach().numpy()) < 1e-4


def test_512_channels_take_the_fused_path_by_default():
    import wavenet_model as wmod
    torch.manual_seed(0)
    m = wmod.WaveNetModel(layers=2, blocks=1, dilation_channels=512, residual_channels=512, skip_channels=512, end_channels=256,
                          classes=256, output_length=32, kernel_size=2).cuda()
    idx = torch.randint(0, 256, (1, 300), generator=torch.Generator().manual_seed(1)).cuda()
    rt = m._runtime()
    with torch.no_grad():
        y = m.forward_indices(idx)
        assert rt.last_block_mode == "tb" and rt.last_precision == "bf16"
        rt.block_mode = "ffma"
        y0 = m.forward_indices(idx)
    assert rel_err(y.cpu().numpy(), y0.cpu().numpy()) < 3e-2


def test_whole_stack_launch_equals_per_layer_launches():
    """wn_tb_stack_fwd (all layers in one persistent launch, items chained by device-side flags) does the same arithmetic as
    one wn_tb_block_fwd launch per layer: identical bits, for the no-grad forward (three rotating buffers) and for the
    training step (saved activations, gradients), several items per layer and dilations larger than an item."""
    import torch.nn.functional as F
    import wavenet_model as wmod
    kw = dict(layers=10, blocks=2, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
              classes=256, output_length=700, kernel_size=2, bias=True)
    torch.manual_seed(8)
    m = wmod.WaveNetModel(**kw).cuda()
    rt = m._runtime()
    idx = torch.randint(0, 256, (5, 3000), generator=torch.Generator().manual_seed(3)).cuda()
    tgt = torch.randint(0, 256, (5 * 700,), generator=torch.Generator().manual_seed(4)).cuda()
    outs, grads = {}, {}
    for stack in (True, False):
        rt.stack_launch = stack
        with torch.no_grad():
            for _ in range(3):                                  # repeated launches reuse (and must reset) the flag buffer
                outs[stack] = m.forward_indices(idx).clone()
        assert rt.last_block_launches == (1 if stack else 20)
        m.zero_grad()
        F.cross_entropy(m.forward_indices(idx), tgt).backward()
        grads[stack] = {k: v.grad.clone() for k, v in m.named_parameters()}
    rt.stack_launch = True
    assert torch.equal(outs[True], outs[False])
    for k in grads[True]:
        if k == "start_conv.weight":         # a scatter-add with float atomics: equal up to summation order
            assert rel_err(grads[True][k].cpu().numpy(), grads[False][k].cpu().numpy()) < 1e-5
        else:
            assert torch.equal(grads[True][k], grads[False][k]), k
