"""The window rule of the sampler's ring prefill (wavenet_model.prefill_window) against the float64 reference: a forward
over prompt positions [P0, T) alone, with zero history at P0, reproduces every value the rings hold after evaluations
[0, T) -- on the k = 3, biased, deep and cfg-2 nets and at T around the 512-dilation ring length and the receptive field --
while a window one position shorter misses.  Plus the argument check of generate_fast(prefill=) before any device work."""
import numpy as np
import pytest

import prefill_ref as P
import sampler_ref as R
import wavenet_model as wmod
from oracle import wavenet_oracle as O
from helpers import spec_from_golden, params_from_golden, weight_checksum

NETS = ["k3", "odd_bias", "deep", "cfg2"]
_cache = {}


def _net(golden, name):
    if name not in _cache:
        g = golden(f"net_{name}.npz")
        spec = spec_from_golden(g)
        p = params_from_golden(g)
        if not p:
            p = O.init_params(spec, seed=0)
            assert weight_checksum(p) == float(g["w_checksum"])
        dil = [d for d, _ in spec.dilation_schedule()]
        rf = spec.receptive_field
        idx = np.random.RandomState(7).randint(0, spec.classes, 3 * rf + 17)
        w = R.weights(p)
        _cache[name] = (spec, w, dil, rf, idx, P.layer_inputs(w, dil, idx)[0])
    return _cache[name]


def _ts(rf):
    """the T of the issue's list that the net's 3 rf + 17 positions reach"""
    return sorted(t for t in {1, 2, 513, 514, rf - 1, rf, rf + 1, 3 * rf + 17} if 1 <= t <= 3 * rf + 17)


@pytest.mark.parametrize("name", NETS)
def test_layer_inputs_pinned_to_sampler_ref(golden, name):
    spec, w, dil, rf, idx, _ = _net(golden, name)
    seq = idx[:min(len(idx), rf + 40)]
    got = P.layer_inputs(w, dil, seq)[1]
    want = R.logits(w, dil, seq)
    assert np.abs(got - want).max() <= 1e-12 * np.abs(want).max()


@pytest.mark.parametrize("name", NETS)
def test_window_reproduces_every_ring_slot(golden, name):
    spec, w, dil, rf, idx, full = _net(golden, name)
    k = spec.kernel_size
    for T in _ts(rf):
        P0, S, W = wmod.prefill_window(T, dil, k)
        assert W == T - P0 <= rf and P0 == max(0, T - rf) and S >= (k - 1) * max(dil)
        win = P.layer_inputs(w, dil, idx[P0:T])[0]
        err = 0.0
        for l, lo, hi in P.ring_slots(dil, k, T):
            a, b = win[l][:, lo - P0:hi - P0], full[l][:, lo:hi]
            err = max(err, float(np.abs(a - b).max() / np.abs(b).max()))
        assert err <= 1e-12, f"{name} T={T}: {err:.3e}"


@pytest.mark.parametrize("name", ["k3", "odd_bias", "deep"])
def test_window_one_shorter_misses(golden, name):
    """From P0 + 1 the oldest slot of the last ring loses position T - rf: the rule is tight.  Measured misses: above 1e-9
    on k3 and odd_bias, 2.5e-11 on deep (12 layers), both over the 1e-12 bar above; on cfg-2 the path from T - rf through
    all 50 history taps to that slot carries about 1e-15 at its random init, below float64 resolution, so it is not
    tested there."""
    spec, w, dil, rf, idx, full = _net(golden, name)
    k, T = spec.kernel_size, 3 * rf + 17
    P0 = wmod.prefill_window(T, dil, k)[0] + 1
    win = P.layer_inputs(w, dil, idx[P0:T])[0]
    l, lo, hi = P.ring_slots(dil, k, T)[-1]
    a, b = win[l][:, lo - P0], full[l][:, lo]
    assert np.abs(a - b).max() > 1e-11 * np.abs(b).max()


@pytest.mark.parametrize("hop", [1, 80])
def test_window_on_hop_multiples(hop):
    dil = R.dilations_of(10, 5)
    for T in (1, 5115, 5116, 20017):
        P0, S, W = wmod.prefill_window(T, dil, 2, hop)
        assert P0 % hop == 0 and S % hop == 0 and S % 8 == 0 and S >= 512
        assert P0 <= max(0, T - 5116) < P0 + hop and W == T - P0


@pytest.mark.parametrize("bad", [1, 0, "yes", None, np.bool_(True)])
def test_prefill_argument_errors_before_device_work(bad):
    m = wmod.WaveNetModel(layers=2, blocks=1, dilation_channels=8, residual_channels=8, skip_channels=8, end_channels=8,
                          classes=16)
    with pytest.raises(ValueError, match="prefill"):
        m.generate_fast(4, [1, 2, 3], prefill=bad)
    with pytest.raises(ValueError, match="prefill"):
        m.generate_fast_batch(4, [[1, 2, 3]], prefill=bad)
