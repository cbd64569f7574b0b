"""Global conditioning, host side: parameters and their order, old pickles, argument errors, the dataset's file labels."""
import os
import pickle

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _kw(**over):
    kw = dict(layers=3, blocks=2, dilation_channels=32, residual_channels=32, skip_channels=32, end_channels=32,
              classes=256, output_length=16, kernel_size=2, bias=True)
    kw.update(over)
    return kw


def test_conditioned_parameters_come_last_and_keep_seeded_values():
    import wavenet_model as wmod
    torch.manual_seed(4)
    m0 = wmod.WaveNetModel(**_kw())
    torch.manual_seed(4)
    m1 = wmod.WaveNetModel(**_kw(), condition_channels=5)
    k0, k1 = list(m0.state_dict()), list(m1.state_dict())
    n = 6
    assert k1[:len(k0)] == k0
    assert k1[len(k0):] == [f"filter_cond_convs.{i}.weight" for i in range(n)] + [f"gate_cond_convs.{i}.weight" for i in range(n)]
    for k in k0:
        assert torch.equal(m0.state_dict()[k], m1.state_dict()[k]), k
    assert tuple(m1.filter_cond_convs[0].weight.shape) == (32, 5, 1) and m1.gate_cond_convs[0].bias is None
    assert m0.condition_channels == 0 and not hasattr(m0, "filter_cond_convs")


def test_unconditioned_pickle_without_the_attribute_still_loads():
    import wavenet_model as wmod
    m = wmod.WaveNetModel(**_kw())
    del m.__dict__["condition_channels"]                  # what a whole-object pickle made before conditioning holds
    m2 = pickle.loads(pickle.dumps(m))
    assert m2._condition(None, 2) is None
    with pytest.raises(ValueError):
        m2._condition([1, 2], 2)
    snap = torch.load(os.path.join(ROOT, "tests", "golden", "tiny_snapshot.pt"), weights_only=False)
    assert snap._condition(None, 1) is None


@pytest.mark.parametrize("cond,n", [(None, 2), ([0, 5], 2), ([0, 1, 2], 2), (np.zeros((2, 4), np.float32), 2),
                                    (np.zeros(2, np.float32), 2), (["a", "b"], 2), ([-1, 0], 2)])
def test_condition_argument_errors(cond, n):
    import wavenet_model as wmod
    m = wmod.WaveNetModel(**_kw(), condition_channels=5)
    with pytest.raises(ValueError):
        m._condition(cond, n)


def test_condition_rows():
    import wavenet_model as wmod
    m = wmod.WaveNetModel(**_kw(), condition_channels=3)
    m._runtime().device = lambda: torch.device("cpu")     # the rows only; the kernels need a CUDA model
    assert torch.equal(m._condition(np.array([2, 0]), 2), torch.tensor([[0., 0., 1.], [1., 0., 0.]]))
    dense = np.arange(6, dtype=np.float64).reshape(2, 3)
    assert torch.equal(m._condition(dense, 2), torch.tensor(dense, dtype=torch.float32))
    assert m._one_condition(1).shape == (1,) and m._one_condition(np.ones(3, np.float32)).shape == (1, 3)


def test_dataset_file_labels():
    import audio_data
    path = os.path.join(ROOT, "tests", "golden", "tiny_dataset.npz")
    ds = audio_data.WavenetDataset(path, item_length=300, target_length=64, one_hot=False, condition_on_file=True)
    plain = audio_data.WavenetDataset(path, item_length=300, target_length=64, one_hot=False)
    data = np.load(path)
    lengths = [len(data[f"arr_{i}"]) for i in range(len(data.files))]
    ends = np.cumsum(lengths)
    seen = set()
    for i in range(len(ds)):
        x, label, target = ds[i]
        x0, t0 = plain[i]
        assert torch.equal(x, x0) and torch.equal(target, t0) and label.dtype == torch.int64
        last = ds._sample_index(i) + 300                       # position of the item's last target sample
        assert int(label) == int(np.searchsorted(ends, last, side="right"))
        seen.add(int(label))
    assert seen == set(range(len(lengths)))


def test_condition_that_needs_a_gradient_is_refused():
    import wavenet_model as wmod
    m = wmod.WaveNetModel(**_kw(), condition_channels=5)
    with pytest.raises(NotImplementedError):
        m._condition(torch.randn(2, 5, requires_grad=True), 2)
