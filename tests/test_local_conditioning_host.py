"""Local conditioning, host side: parameters and their order, old pickles, constructor and argument errors, and the float64
reference (tests/local_ref.py) pinned against the oracle without a GPU."""
import os
import pickle

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import local_ref
from oracle import wavenet_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _kw(**over):
    kw = dict(layers=3, blocks=2, dilation_channels=32, residual_channels=32, skip_channels=32, end_channels=32,
              classes=256, output_length=16, kernel_size=2, bias=True)
    kw.update(over)
    return kw


def _cpu_model(**kw):
    import wavenet_model as wmod
    m = wmod.WaveNetModel(**kw)
    m._runtime().device = lambda: torch.device("cpu")     # argument checks only; the kernels need a CUDA model
    return m


def test_local_parameters_come_last_and_keep_seeded_values():
    import wavenet_model as wmod
    torch.manual_seed(4)
    m0 = wmod.WaveNetModel(**_kw(), condition_channels=5)
    torch.manual_seed(4)
    m1 = wmod.WaveNetModel(**_kw(), condition_channels=5, local_condition_channels=7, local_condition_hop=80)
    k0, k1 = list(m0.state_dict()), list(m1.state_dict())
    n = 6
    assert k1[:len(k0)] == k0
    assert k1[len(k0):] == [f"filter_local_convs.{i}.weight" for i in range(n)] + [f"gate_local_convs.{i}.weight" for i in range(n)]
    for k in k0:
        assert torch.equal(m0.state_dict()[k], m1.state_dict()[k]), k
    assert tuple(m1.filter_local_convs[0].weight.shape) == (32, 7, 1) and m1.gate_local_convs[0].bias is None
    torch.manual_seed(4)
    m2 = wmod.WaveNetModel(**_kw(), local_condition_channels=7, local_condition_hop=80)      # local only
    torch.manual_seed(4)
    m3 = wmod.WaveNetModel(**_kw())
    for k, v in m3.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k
    assert m3.local_condition_channels == 0 and not hasattr(m3, "filter_local_convs")


def test_pickle_without_the_attributes_still_loads():
    import wavenet_model as wmod
    m = wmod.WaveNetModel(**_kw())
    del m.__dict__["local_condition_channels"]            # what a whole-object pickle made before local conditioning holds
    del m.__dict__["local_condition_hop"]
    m2 = pickle.loads(pickle.dumps(m))
    assert m2._local_condition(None, 2, 100) is None
    with pytest.raises(ValueError):
        m2._local_condition(np.zeros((2, 3, 10), np.float32), 2, 100)
    snap = torch.load(os.path.join(ROOT, "tests", "golden", "tiny_snapshot.pt"), weights_only=False)
    assert snap._local_condition(None, 1, 10) is None


@pytest.mark.parametrize("hop", [None, 0, -3, 2.5, "8", True])
def test_constructor_needs_a_hop(hop):
    import wavenet_model as wmod
    with pytest.raises(ValueError):
        wmod.WaveNetModel(**_kw(), local_condition_channels=4, local_condition_hop=hop)


@pytest.mark.parametrize("y,n,positions", [
    (None, 2, 100),                                         # missing
    (np.zeros((2, 4, 10), np.float32), 2, 100),             # hop 10: 10 frames cover 100 positions; 4 channels, not 5
    (np.zeros((3, 5, 10), np.float32), 2, 100),             # wrong N
    (np.zeros((2, 5), np.float32), 2, 100),                 # wrong rank
    (np.zeros((2, 5, 9), np.float32), 2, 100),              # too few frames
    (np.zeros((2, 5, 10), np.int64), 2, 100),               # not float
    ([["a"]], 2, 100),
])
def test_local_condition_argument_errors(y, n, positions):
    m = _cpu_model(**_kw(), local_condition_channels=5, local_condition_hop=10)
    with pytest.raises(ValueError):
        m._local_condition(y, n, positions)


def test_local_condition_rows():
    m = _cpu_model(**_kw(), local_condition_channels=5, local_condition_hop=10)
    y = np.arange(2 * 5 * 12, dtype=np.float64).reshape(2, 5, 12)
    got = m._local_condition(y, 2, 101)                     # 11 frames needed, extra frames are allowed
    assert got.dtype == torch.float32 and torch.equal(got, torch.tensor(y, dtype=torch.float32))
    with pytest.raises(ValueError):
        _cpu_model(**_kw())._local_condition(y, 2, 100)     # unexpected


def test_slow_generate_and_queue_step_refuse_local_models():
    m = _cpu_model(**_kw(), local_condition_channels=5, local_condition_hop=10)
    with pytest.raises(NotImplementedError):
        m.generate(4)
    with pytest.raises(NotImplementedError):
        m.wavenet(torch.zeros(1, 256, 1), dilation_func=m.queue_dilate)


# ---------------------------------------------------------------------------------------------- the reference, pinned
def _small(C=3, G=0, seed=0):
    kw = dict(layers=3, blocks=2, dilation_channels=8, residual_channels=8, skip_channels=8, end_channels=8, classes=16,
              output_length=8, kernel_size=2, bias=True)
    spec = O.NetSpec(**kw)
    g = torch.Generator().manual_seed(seed)
    p = {k: (0.4 * torch.randn(v.shape, generator=g)).double() for k, v in O.init_params(spec, seed).items()}
    for i in range(spec.layers * spec.blocks):
        for nm in ("filter", "gate"):
            p[f"{nm}_local_convs.{i}.weight"] = 0.5 * torch.randn(8, C, 1, generator=g).double()
            if G:
                p[f"{nm}_cond_convs.{i}.weight"] = 0.5 * torch.randn(8, G, 1, generator=g).double()
    return spec, p


def test_reference_with_zero_u_is_the_oracle_bit_for_bit():
    spec, p = _small()
    for k in p:
        if "_local_convs." in k:
            p[k] = torch.zeros_like(p[k])
    x = O.one_hot(torch.randint(0, 16, (2, 50), generator=torch.Generator().manual_seed(1)), 16).double()
    y = torch.randn(2, 3, 50, generator=torch.Generator().manual_seed(2)).double()
    assert torch.equal(local_ref.stack_direct(p, spec, x, y, 1), O.stack_direct(p, spec, x))


def test_reference_with_one_frame_is_the_folded_oracle():
    spec, p = _small(G=4)
    x = O.one_hot(torch.randint(0, 16, (2, 50), generator=torch.Generator().manual_seed(1)), 16).double()
    y = torch.randn(2, 3, 1, generator=torch.Generator().manual_seed(2)).double()
    h = torch.randn(2, 4, generator=torch.Generator().manual_seed(3)).double()
    for hop in (50, 64):
        got = local_ref.forward(p, spec, x, y, hop, h)
        want = torch.cat([O.forward(local_ref.folded(p, spec, y[b, :, 0], h[b]), spec, x[b:b + 1]) for b in range(2)])
        assert float((got - want).abs().max()) < 1e-12 * float(want.abs().max())


@pytest.mark.parametrize("hop", [1, 3, 7, 64])
def test_reference_matches_a_per_position_folded_queue_run(hop):
    """Teacher-forced fast-generation run of the oracle (stack_folded on dilated queues), each position's biases folded
    for that position's frame: at every position >= receptive_field - 1 its logits equal the reference's."""
    spec, p = _small(G=2)
    L = 140
    idx = torch.randint(0, 16, (1, L), generator=torch.Generator().manual_seed(4))
    y = torch.randn(1, 3, -(-L // hop), generator=torch.Generator().manual_seed(5)).double()
    h = torch.randn(1, 2, generator=torch.Generator().manual_seed(6)).double()
    want = local_ref.stack_direct(p, spec, O.one_hot(idx, 16).double(), y, hop, h)[0]      # (classes, T_final)
    t_final = want.shape[1]
    k = spec.kernel_size
    queues = [O.RingQueue((k - 1) * d + 1, spec.residual_channels) for d, _ in spec.dilation_schedule()]
    for q in queues:
        q.data = q.data.double()

    def queue_fn(hq, d, init_d, i):
        q = queues[i]
        q.enqueue(hq[0])
        return q.dequeue(num_deq=k, dilation=d).unsqueeze(0)

    rf = 1 + sum((k - 1) * d for d, _ in spec.dilation_schedule())
    checked = 0
    with torch.no_grad():
        for t in range(L):
            q = local_ref.folded(p, spec, y[0, :, t // hop], h[0])
            out = O.stack_folded(q, spec, O.one_hot(idx[:, t:t + 1], 16).double(), queue_fn)[0, :, 0]
            if t >= rf - 1:
                ref = want[:, t - (L - t_final)]
                assert float((out - ref).abs().max()) < 1e-12 * float(ref.abs().max()), t
                checked += 1
    assert checked == L - rf + 1
