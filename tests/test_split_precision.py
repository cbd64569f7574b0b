"""Precision model of the tensor-core operand splits (CPU, float64 emulation on the oracle's stack).

The tensor-core blocks (csrc/tc_gemm.cu) write both GEMM operands as x = hi + lo and accumulate hi*hi + lo*hi + hi*lo in
fp32.  This test evaluates the cfg-2 stack (10x5 layers, 256 channels) with every block convolution replaced by that
three-product form -- products summed in float64, so only the operand rounding is modelled -- and checks the ordering the
design rests on: bf16 pairs and 3xTF32 stay two orders of magnitude inside the 1e-4 parity bar, a single TF32 pass
does not."""
import math

import torch
import torch.nn.functional as F

from block_ref import split_bf16, split_tf32
from oracle import wavenet_oracle as O


def conv(inp, w, dilation, mode):
    if mode == "fp32":
        return F.conv1d(inp, w, dilation=dilation)
    split = split_bf16 if mode == "bf16x2" else split_tf32
    (ah, al), (wh, wl) = split(inp), split(w)
    f = lambda a, b: F.conv1d(a.double(), b.double(), dilation=dilation)
    if mode == "tf32x1":
        return f(ah, wh).float()
    return (f(ah, wh) + f(al, wh) + f(ah, wl)).float()


def stack(p, spec, x, mode, out_len):
    k = spec.kernel_size
    h = F.conv1d(x, p["start_conv.weight"])
    skip = None
    for i, (d, _) in enumerate(spec.dilation_schedule()):
        T = h.size(2)
        hp = F.pad(h, (int(math.ceil(T / d) * d) - T, 0))
        z = torch.tanh(conv(hp, p[f"filter_convs.{i}.weight"], d, mode)) * torch.sigmoid(conv(hp, p[f"gate_convs.{i}.weight"], d, mode))
        s = conv(z, p[f"skip_convs.{i}.weight"], 1, mode)
        skip = s if skip is None else s + skip[:, :, -s.size(2):]
        h = conv(z, p[f"residual_convs.{i}.weight"], 1, mode) + hp[:, :, d * (k - 1):]
    y = F.relu(F.conv1d(F.relu(skip), p["end_conv_1.weight"], p["end_conv_1.bias"]))
    return F.conv1d(y, p["end_conv_2.weight"], p["end_conv_2.bias"])[:, :, -out_len:]


def test_split_helpers_are_exact_decompositions():
    x = torch.randn(4096, generator=torch.Generator().manual_seed(0)) * 3
    for split, bits in ((split_bf16, 8), (split_tf32, 11)):
        hi, lo = split(x)
        assert float(((hi - x).abs() / x.abs()).max()) <= 2.0 ** -bits           # hi keeps `bits` significant bits
        assert float(((hi + lo - x).abs() / x.abs()).max()) <= 2.0 ** -(2 * bits)   # the pair keeps about twice as many
    hi, lo = split_tf32(x)
    assert torch.equal(hi + lo, x)                                               # tf32: x - rna(x) is exact in fp32


def test_three_product_splits_hold_the_parity_bar_through_50_layers():
    torch.set_num_threads(min(8, torch.get_num_threads()))
    kw = dict(layers=10, blocks=5, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
              classes=256, output_length=32, kernel_size=2, bias=False)
    spec = O.NetSpec(**kw)
    p = O.init_params(spec, seed=0)
    rf = sum(d for d, _ in spec.dilation_schedule()) + 1
    idx = torch.randint(0, 256, (1, rf + 31), generator=torch.Generator().manual_seed(1234))
    x = O.one_hot(idx, 256)
    with torch.no_grad():
        ref = stack(p, spec, x, "fp32", 32)
        assert torch.allclose(ref, O.stack_direct(p, spec, x)[:, :, -32:], rtol=0, atol=1e-6)   # same maths as the oracle
        err = {m: float((stack(p, spec, x, m, 32) - ref).abs().max() / ref.abs().max()) for m in ("bf16x2", "tf32x3", "tf32x1")}
    assert err["tf32x3"] < 5e-6 and err["bf16x2"] < 2e-5, err
    assert err["tf32x1"] > 10 * err["bf16x2"], err
    assert err["tf32x1"] > 5e-5, err                                # the single pass is what does not fit under 1e-4 at scale
