"""Learned local-conditioning upsampler, host side: constructor checks, parameter order and seeded values, old pickles, the
repetition initialisation, and the float64 reference (tests/upsample_ref.py) against the model's own upsampler."""
import pickle

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import local_ref
import upsample_ref
from oracle import wavenet_oracle as O


def _kw(**over):
    kw = dict(layers=3, blocks=2, dilation_channels=32, residual_channels=32, skip_channels=32, end_channels=32,
              classes=256, output_length=16, kernel_size=2, bias=True)
    kw.update(over)
    return kw


@pytest.mark.parametrize("C,hop,scales", [
    (4, 80, (4, 4)), (4, 80, (80, 0)), (4, 80, (4, 4, 5.0)), (4, 80, (True, 80)), (4, 80, ()), (4, 80, 80),
    (4, 80, (-4, -20)), (0, None, (4,)), (4, 6, ("2", 3))])
def test_bad_scales_raise(C, hop, scales):
    import wavenet_model as wmod
    with pytest.raises(ValueError):
        wmod.WaveNetModel(**_kw(), local_condition_channels=C, local_condition_hop=hop, local_condition_upsample_scales=scales)


def test_upsampler_comes_last_and_keeps_seeded_values():
    import wavenet_model as wmod
    torch.manual_seed(4)
    m0 = wmod.WaveNetModel(**_kw(), condition_channels=5, local_condition_channels=7, local_condition_hop=80)
    torch.manual_seed(4)
    m1 = wmod.WaveNetModel(**_kw(), condition_channels=5, local_condition_channels=7, local_condition_hop=80,
                           local_condition_upsample_scales=(4, 4, 5))
    k0, k1 = list(m0.state_dict()), list(m1.state_dict())
    assert k1[:len(k0)] == k0
    assert k1[len(k0):] == [f"local_upsample.{j}.{w}" for j in range(3) for w in ("weight", "bias")]
    for k in k0:
        assert torch.equal(m0.state_dict()[k], m1.state_dict()[k]), k
    assert tuple(m1.local_upsample[2].weight.shape) == (7, 7, 10) and m1.local_upsample[2].stride == (5,)
    assert getattr(m0, "local_upsample", None) is None


def test_pickle_without_the_upsampler_still_loads():
    import wavenet_model as wmod
    m = wmod.WaveNetModel(**_kw(), local_condition_channels=3, local_condition_hop=10)
    m2 = pickle.loads(pickle.dumps(m))
    assert getattr(m2, "local_upsample", None) is None and not hasattr(m2, "local_condition_upsample_scales")
    m2._runtime().device = lambda: torch.device("cpu")
    y = m2._local_condition(np.zeros((2, 3, 10), np.float32), 2, 100)
    assert m2._sampler_local(y, 100)[1] == 10                # repetition: the series at its own hop


@pytest.mark.parametrize("scales", [(80,), (4, 4, 5), (3, 5), (1, 7)])
def test_initialisation_is_exact_repetition(scales):
    import math
    import wavenet_model as wmod
    hop = math.prod(scales)
    m = wmod.WaveNetModel(**_kw(), local_condition_channels=6, local_condition_hop=hop, local_condition_upsample_scales=scales)
    y = torch.randn(2, 6, 9, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    L = 9 * hop - hop // 2
    p = {k: v.double() for k, v in m.state_dict().items()}
    want = local_ref.upsample(y, hop, L)
    assert torch.equal(upsample_ref.upsample(p, scales, y)[:, :, :L], want)
    with torch.no_grad():
        got = m._upsample(y.float(), L)
    assert got.is_contiguous() and torch.equal(got, want.float())


def test_reference_at_repetition_init_is_the_repeat_net():
    import wavenet_model as wmod
    kw = _kw(output_length=40)
    spec = O.NetSpec(**kw)
    torch.manual_seed(3)
    m = wmod.WaveNetModel(**kw, condition_channels=2, local_condition_channels=4, local_condition_hop=15,
                          local_condition_upsample_scales=(3, 5))
    p = {k: v.double() for k, v in m.state_dict().items()}
    with torch.no_grad():
        for k, v in p.items():
            if "_local_convs." in k:
                v.normal_(0, 0.3)
    g = torch.Generator().manual_seed(2)
    x = O.one_hot(torch.randint(0, 256, (2, 130), generator=g), 256).double()
    y = torch.randn(2, 4, 9, generator=g, dtype=torch.float64)
    h = torch.randn(2, 2, generator=g, dtype=torch.float64)
    assert torch.equal(upsample_ref.forward(p, spec, x, y, (3, 5), h), local_ref.forward(p, spec, x, y, 15, h))


def test_model_upsampler_gradients_match_the_reference():
    """Arbitrary upsampler weights: the model's _upsample (what the GPU paths run before the stack) composed with the float64
    reference gives the same logits and gradients, upsampler and series included, as upsample_ref."""
    import wavenet_model as wmod
    kw = _kw(output_length=40)
    spec = O.NetSpec(**kw)
    torch.manual_seed(5)
    m = wmod.WaveNetModel(**kw, local_condition_channels=3, local_condition_hop=12, local_condition_upsample_scales=(4, 3))
    m = m.double()
    with torch.no_grad():
        for k, v in m.named_parameters():
            if "local_" in k:
                v.normal_(0, 0.3)
    g = torch.Generator().manual_seed(6)
    idx = torch.randint(0, 256, (2, 110), generator=g)
    tgt = torch.randint(0, 256, (80,), generator=g)
    x = O.one_hot(idx, 256).double()
    y0 = torch.randn(2, 3, 10, generator=g, dtype=torch.float64)
    p = {k: v.detach().clone().requires_grad_(True) for k, v in m.named_parameters()}
    ya = y0.clone().requires_grad_(True)
    want = upsample_ref.forward(p, spec, x, ya, (4, 3))
    F.cross_entropy(want, tgt).backward()
    yb = y0.clone().requires_grad_(True)
    c = m._upsample(yb, 110)
    q = dict(m.named_parameters())
    out = local_ref.stack_direct(q, spec, x, c, 1)
    got = out[:, :, -40:].transpose(1, 2).contiguous().view(80, 256)
    F.cross_entropy(got, tgt).backward()
    assert float((got - want).detach().abs().max()) <= 1e-12
    assert float((yb.grad - ya.grad).abs().max()) <= 1e-12 * max(1.0, float(ya.grad.abs().max()))
    for k, v in q.items():
        ref = p[k].grad
        if ref is None:                    # parameters the loss does not reach (no path to the output window)
            assert v.grad is None or not v.grad.any(), k
            continue
        assert float((v.grad - ref).abs().max()) <= 1e-12 * max(1.0, float(ref.abs().max())), k
    assert any(float(q[k].grad.abs().max()) > 0 for k in q if k.startswith("local_upsample."))
