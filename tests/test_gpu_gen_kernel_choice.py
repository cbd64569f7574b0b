"""Which sampler kernel every mode of wn_gen_set_mode runs, on the shapes where the kernels' eligibility changes: the cfg-2
net (256 wide) from 1 to 120 streams, the small golden nets, a 1-layer net and a 128-wide net (cluster kernel 4 applies,
the 256-wide batched kernel 6 does not).  Per mode the table holds what wn_gen_set_mode returns, wn_gen_kernel_id and
wn_gen_launch_info (return code, grid, block, exchange stages per evaluation), read on a fresh handle right after
wn_gen_create and wn_gen_reset, before any launch; a launch in that mode must then leave them as they were, and a handle
whose mode was never set must pick what mode 0 picks."""
import ctypes

import numpy as np
import pytest
import torch

import native
from helpers import build_model

pytestmark = pytest.mark.gpu
OK, BADARG, UNSUPP = 0, -1, -2
MODES = (0, 1, 2, 3, 4, 5, 6)


def _net(golden, name):
    if name in ("cfg2", "odd_bias", "deep", "k3"):
        return build_model(golden(f"net_{name}.npz"))
    import wavenet_model as wmod
    torch.manual_seed(0)
    ch, layers = {"one_layer": (32, 1), "w128": (128, 3)}[name]
    return wmod.WaveNetModel(layers=layers, blocks=1, dilation_channels=ch, residual_channels=ch, skip_channels=ch,
                             end_channels=ch, classes=256, output_length=16, kernel_size=2, bias=False).cuda()


# (net, streams) -> per mode 0..6: (wn_gen_set_mode, wn_gen_kernel_id, wn_gen_launch_info rc, grid, block, stages), as
# observed on an H100 80GB HBM3 (132 SMs): the grids of kernels 1-3 and the cluster size of kernel 6 (grid / clusters)
# follow the SM count and the occupancy query.  At 120 streams the cfg-2 net fits neither kernel 1 nor 2 (mode 1 and 2
# rows: id 0, WN_E_UNSUPP).
TABLE = {
    ("cfg2", 1): [(0, 6, 0, 16, 320, 102), (0, 1, 0, 64, 256, 102), (0, 2, 0, 64, 256, 102), (0, 3, 0, 64, 288, 102),
                  (0, 4, 0, 16, 288, 102), (-1, 6, 0, 16, 320, 102), (0, 6, 0, 16, 320, 102)],
    ("cfg2", 3): [(0, 6, 0, 16, 320, 102), (0, 1, 0, 64, 256, 102), (0, 2, 0, 64, 256, 102), (-2, 6, 0, 16, 320, 102),
                  (0, 4, 0, 48, 288, 102), (-1, 6, 0, 16, 320, 102), (0, 6, 0, 16, 320, 102)],
    ("cfg2", 11): [(0, 6, 0, 32, 320, 102), (0, 1, 0, 64, 256, 102), (0, 2, 0, 64, 256, 102), (-2, 6, 0, 32, 320, 102),
                   (0, 4, 0, 176, 288, 102), (-1, 6, 0, 32, 320, 102), (0, 6, 0, 32, 320, 102)],
    ("cfg2", 64): [(0, 6, 0, 64, 352, 102), (0, 1, 0, 64, 256, 102), (0, 2, 0, 64, 256, 102), (-2, 6, 0, 64, 352, 102),
                   (0, 4, 0, 1024, 288, 102), (-1, 6, 0, 64, 352, 102), (0, 6, 0, 64, 352, 102)],
    ("cfg2", 120): [(0, 6, 0, 120, 352, 102), (0, 0, -2, 0, 0, 0), (0, 0, -2, 0, 0, 0), (-2, 6, 0, 120, 352, 102),
                    (0, 4, 0, 1920, 288, 102), (-1, 6, 0, 120, 352, 102), (0, 6, 0, 120, 352, 102)],
    ("odd_bias", 1): [(0, 2, 0, 2, 256, 14), (0, 1, 0, 2, 256, 14), (0, 2, 0, 2, 256, 14), (-2, 2, 0, 2, 256, 14),
                      (-2, 2, 0, 2, 256, 14), (-1, 2, 0, 2, 256, 14), (-2, 2, 0, 2, 256, 14)],
    ("odd_bias", 3): [(0, 2, 0, 2, 256, 14), (0, 1, 0, 2, 256, 14), (0, 2, 0, 2, 256, 14), (-2, 2, 0, 2, 256, 14),
                      (-2, 2, 0, 2, 256, 14), (-1, 2, 0, 2, 256, 14), (-2, 2, 0, 2, 256, 14)],
    ("deep", 1): [(0, 2, 0, 16, 256, 26), (0, 1, 0, 16, 256, 26), (0, 2, 0, 16, 256, 26), (-2, 2, 0, 16, 256, 26),
                  (-2, 2, 0, 16, 256, 26), (-1, 2, 0, 16, 256, 26), (-2, 2, 0, 16, 256, 26)],
    ("deep", 3): [(0, 2, 0, 16, 256, 26), (0, 1, 0, 16, 256, 26), (0, 2, 0, 16, 256, 26), (-2, 2, 0, 16, 256, 26),
                  (-2, 2, 0, 16, 256, 26), (-1, 2, 0, 16, 256, 26), (-2, 2, 0, 16, 256, 26)],
    ("k3", 1): [(0, 2, 0, 2, 256, 14), (0, 1, 0, 2, 256, 14), (0, 2, 0, 2, 256, 14), (-2, 2, 0, 2, 256, 14),
                (-2, 2, 0, 2, 256, 14), (-1, 2, 0, 2, 256, 14), (-2, 2, 0, 2, 256, 14)],
    ("k3", 3): [(0, 2, 0, 2, 256, 14), (0, 1, 0, 2, 256, 14), (0, 2, 0, 2, 256, 14), (-2, 2, 0, 2, 256, 14),
                (-2, 2, 0, 2, 256, 14), (-1, 2, 0, 2, 256, 14), (-2, 2, 0, 2, 256, 14)],
    ("one_layer", 1): [(-2, 1, 0, 8, 256, 4), (0, 1, 0, 8, 256, 4), (-2, 1, 0, 8, 256, 4), (-2, 1, 0, 8, 256, 4),
                       (-2, 1, 0, 8, 256, 4), (-1, 1, 0, 8, 256, 4), (-2, 1, 0, 8, 256, 4)],
    ("one_layer", 3): [(-2, 1, 0, 8, 256, 4), (0, 1, 0, 8, 256, 4), (-2, 1, 0, 8, 256, 4), (-2, 1, 0, 8, 256, 4),
                       (-2, 1, 0, 8, 256, 4), (-1, 1, 0, 8, 256, 4), (-2, 1, 0, 8, 256, 4)],
    ("w128", 1): [(0, 3, 0, 32, 288, 8), (0, 1, 0, 32, 256, 8), (0, 2, 0, 32, 256, 8), (0, 3, 0, 32, 288, 8),
                  (0, 4, 0, 16, 288, 8), (-1, 3, 0, 32, 288, 8), (-2, 3, 0, 32, 288, 8)],
    ("w128", 3): [(0, 4, 0, 48, 288, 8), (0, 1, 0, 32, 256, 8), (0, 2, 0, 32, 256, 8), (-2, 4, 0, 48, 288, 8),
                  (0, 4, 0, 48, 288, 8), (-1, 4, 0, 48, 288, 8), (-2, 4, 0, 48, 288, 8)],
}


def _fresh_handle(m, ns):
    """a new sampler handle for ns streams (wn_gen_create), reset"""
    rt, lib = m._runtime(), native.lib()
    old = rt.samplers.pop(ns, None)
    if old is not None:
        lib.wn_gen_destroy(old["handle"])
    h = rt.sampler(ns)["handle"]
    native.check(lib.wn_gen_reset(h, torch.cuda.current_stream().cuda_stream), "gen reset")
    return h


def _choice(h):
    """(wn_gen_kernel_id, wn_gen_launch_info rc, grid, block, stages)"""
    lib = native.lib()
    g, b, x = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    rc = lib.wn_gen_launch_info(h, ctypes.byref(g), ctypes.byref(b), ctypes.byref(x))
    return (lib.wn_gen_kernel_id(h), rc) + ((g.value, b.value, x.value) if rc == OK else (0, 0, 0))


def _observe(m, ns):
    """[(mode, row before any launch, row after a 2-evaluation launch or None, launch error or None)] and the choice of a
    handle whose mode was never set"""
    rt, out = m._runtime(), []
    default = _choice(_fresh_handle(m, ns))
    for mode in MODES:
        h = _fresh_handle(m, ns)
        row = (native.lib().wn_gen_set_mode(h, mode),) + _choice(h)
        after, err = None, None
        if row[0] == OK:
            rt.gen_mode = mode
            try:
                m.generate_fast_batch(2, np.zeros((ns, 1), np.int64), temperature=0.0)
                after = (row[0],) + _choice(rt.sampler(ns)["handle"])
            except RuntimeError as e:
                err = str(e)
            rt.gen_mode = None
        out.append((mode, row, after, err))
    return out, default


CASES = [("cfg2", ns) for ns in (1, 3, 11, 64, 120)] + [(n, ns) for n in ("odd_bias", "deep", "k3", "one_layer", "w128")
                                                          for ns in (1, 3)]


@pytest.mark.parametrize("net,ns", CASES, ids=[f"{n}-{ns}" for n, ns in CASES])
def test_kernel_choice(golden, net, ns):
    m = _net(golden, net)
    rows, default = _observe(m, ns)
    want = TABLE[(net, ns)]
    for mode, row, after, err in rows:
        assert row == want[mode], (mode, row, want[mode])
        if mode == 5:
            assert row[0] == BADARG
        if row[0] == OK and row[1] != 0:
            assert err is None and after == row, (mode, err, after, row)   # the launch ran and reports what it said
        elif row[0] == OK:
            assert row[2] == UNSUPP and "need a cluster kernel" in err, (mode, err)   # nothing fits: wn_gen_run refuses too
    assert default == want[0][1:], default
