"""Training-path parity on the GPU: CUDA kernels (through the C ABI) vs the golden outputs of the unmodified
reference and vs the CPU oracle.  fp32 tolerance: max|a-b| / max|b| <= 1e-4 (BASELINE.json north_star)."""
import numpy as np
import pytest
import torch

from oracle import wavenet_oracle as O
from helpers import (build_model, snapshot_model, one_hot_cuda, rel_err, spec_from_golden, params_from_golden)

pytestmark = pytest.mark.gpu
TOL = 1e-4


@pytest.mark.parametrize("name", ["cfg1", "odd_bias", "k3", "deep"])
def test_forward_matches_reference_golden(golden, name):
    g = golden(f"net_{name}.npz")
    m = build_model(g)
    x = one_hot_cuda(g["idx"])
    with torch.no_grad():
        y = m(x)
        full = m.wavenet(x, m.wavenet_dilate)
    assert y.shape == g["fwd"].shape and full.shape == g["full"].shape
    assert rel_err(y.cpu().numpy(), g["fwd"]) < TOL
    assert rel_err(full.cpu().numpy(), g["full"]) < TOL          # incl. the padding-contaminated early columns
    with torch.no_grad():
        yi = m.forward_indices(torch.from_numpy(g["idx"]).cuda())
        yu = m.forward_indices(torch.from_numpy(g["idx"].astype(np.uint8)).cuda())
    assert torch.equal(yi, y) and torch.equal(yu, y)              # gather == dense conv on one-hot, bit for bit


def test_forward_cfg2_net(golden):
    g = golden("net_cfg2.npz")
    m = build_model(g)
    with torch.no_grad():
        y = m(one_hot_cuda(g["idx"]))
    assert rel_err(y.cpu().numpy(), g["fwd"]) < TOL


def test_forward_snapshot_real_audio(golden):
    gs, gio = golden("snapshot_chaconne_state.npz"), golden("snapshot_chaconne_io.npz")
    m = snapshot_model(gs)
    rf = int(gs["receptive_field"])
    with torch.no_grad():
        y = m(one_hot_cuda(gio["clip"][None, :rf + 63].astype(np.int64)))
    assert rel_err(y.cpu().numpy(), gio["fwd64"]) < TOL
    assert np.array_equal(y.argmax(1).cpu().numpy(), gio["fwd64"].argmax(1))


@pytest.mark.parametrize("B,L,kw", [
    (2, 193, dict(layers=4, blocks=2, dilation_channels=24, residual_channels=20, skip_channels=36, end_channels=28,
                  kernel_size=2, bias=True, output_length=40)),
    (1, 300, dict(layers=5, blocks=1, dilation_channels=64, residual_channels=64, skip_channels=128, end_channels=64,
                  kernel_size=2, bias=False, output_length=200)),
    (3, 90, dict(layers=3, blocks=2, dilation_channels=6, residual_channels=10, skip_channels=5, end_channels=7,
                 kernel_size=3, bias=True, output_length=9)),
    (2, 140, dict(layers=2, blocks=2, dilation_channels=130, residual_channels=4, skip_channels=260, end_channels=132,
                  kernel_size=2, bias=True, output_length=64)),
    (2, 150, dict(layers=3, blocks=2, dilation_channels=24, residual_channels=20, skip_channels=36, end_channels=28,
                  classes=11, kernel_size=2, bias=True, output_length=33)),
    (1, 200, dict(layers=4, blocks=1, dilation_channels=32, residual_channels=32, skip_channels=64, end_channels=48,
                  classes=257, kernel_size=3, bias=True, output_length=129)),
    (3, 100, dict(layers=3, blocks=1, dilation_channels=16, residual_channels=16, skip_channels=40, end_channels=1000,
                  classes=1000, kernel_size=2, bias=False, output_length=50)),
])
def test_forward_matches_oracle_random_nets(B, L, kw):
    """Seeded random nets incl. ragged channel and class counts, k=3, dense (non one-hot) input."""
    import wavenet_model as wmod
    torch.manual_seed(3)
    m = wmod.WaveNetModel(**kw)
    spec = O.NetSpec(**kw)
    p = {k: v.detach().clone() for k, v in m.state_dict().items()}
    C = spec.classes
    x = torch.rand(B, C, L) * (torch.rand(B, C, L) < 0.05)           # sparse dense input, not one-hot
    with torch.no_grad():
        want = O.forward(p, spec, x).numpy()
        want_direct = O.forward_direct(p, spec, x).numpy()
        got = m.cuda()(x.cuda()).cpu().numpy()
    assert rel_err(want_direct, want) < 1e-5
    assert rel_err(got, want) < TOL


def test_output_length_too_long_raises(golden):
    g = golden("net_odd_bias.npz")
    m = build_model(g, output_length=10 ** 4)
    with torch.no_grad(), pytest.raises(RuntimeError):
        m(one_hot_cuda(g["idx"]))
    m = build_model(g)
    with torch.no_grad(), pytest.raises(RuntimeError):
        m(one_hot_cuda(g["idx"][:, :5]))                              # too short for the dilations


def test_full_size_properties_cfg3():
    """cfg 3 shape (10x5 layers, 256 ch, B=8, L=16000): size-independent properties instead of an oracle run."""
    import wavenet_model as wmod
    torch.manual_seed(0)
    m = wmod.WaveNetModel(layers=10, blocks=5, dilation_channels=256, residual_channels=256, skip_channels=256,
                          end_channels=256, classes=256, output_length=16000 - 5116 + 1, kernel_size=2).cuda()
    idx = torch.randint(0, 256, (8, 16000), generator=torch.Generator().manual_seed(1234))
    with torch.no_grad():
        y = m.forward_indices(idx.cuda()).view(8, -1, 256)
        assert y.shape == (8, 10885, 256) and bool(torch.isfinite(y).all())
        # (1) batch elements are independent: row 5 alone gives the same bits
        y5 = m.forward_indices(idx[5:6].cuda()).view(1, -1, 256)
        assert torch.equal(y5[0], y[5])
        # (2) causality: changing the last 100 input samples leaves all but the last 100 outputs untouched
        idx2 = idx.clone()
        idx2[:, -100:] = (idx2[:, -100:] + 1) % 256
        y2 = m.forward_indices(idx2.cuda()).view(8, -1, 256)
        assert torch.equal(y2[:, :-100], y[:, :-100]) and not torch.equal(y2[:, -100:], y[:, -100:])
        # (3) shift equivariance in the fully-valid region: dropping the first 7 input frames shifts nothing
        m.output_length = 4000
        ya = m.forward_indices(idx[:1].cuda())
        yb = m.forward_indices(idx[:1, 7:].cuda())
        assert rel_err(yb.cpu().numpy(), ya.cpu().numpy()) < 1e-5
        # (4) the one-hot API path equals the index path
        m.output_length = 64
        x = one_hot_cuda(idx[:2].numpy())
        assert torch.equal(m(x), m.forward_indices(idx[:2].cuda()))


def test_cfg3_full_size_vs_oracle():
    """The benchmarked shape itself against the CPU oracle: cfg-3 net (10x5 layers, 256 ch), one L=16000 sequence,
    output_length = 10885, default (fused tensor-core) blocks; then B=8 where every row must equal its B=1 run bit for bit."""
    import wavenet_model as wmod
    kw = dict(layers=10, blocks=5, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
              classes=256, output_length=16000 - 5116 + 1, kernel_size=2, bias=False)
    torch.manual_seed(0)
    m = wmod.WaveNetModel(**kw)
    spec = O.NetSpec(**kw)
    p = {k: v.detach().clone() for k, v in m.state_dict().items()}
    idx = torch.randint(0, 256, (8, 16000), generator=torch.Generator().manual_seed(1234))
    with torch.no_grad():
        want = O.forward(p, spec, O.one_hot(idx[3:4], 256)).numpy()           # ~2 s of CPU
    m = m.cuda()
    rt = m._runtime()
    with torch.no_grad():
        y1 = m.forward_indices(idx[3:4].cuda())
        assert rt.last_block_mode == "tb"                      # the fused wgmma block kernel is the default here
        err = rel_err(y1.cpu().numpy(), want)
        assert err < TOL, f"cfg3 full size vs oracle: {err:.3e}"
        y8 = m.forward_indices(idx.cuda()).view(8, -1, 256)
        assert torch.equal(y8[3], y1.view(-1, 256))
        y0 = m.forward_indices(idx[0:1].cuda())
        assert torch.equal(y8[0], y0.view(-1, 256))
