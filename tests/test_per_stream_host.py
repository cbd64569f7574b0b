"""Host side of per-stream sampling (generate_fast_batch with per-stream prompts, counts and settings;
wn_gen_set_stream_params): the schedule derived from ragged inputs, the padded matrices the kernels read, and every
argument error, raised before any device work."""
import ctypes

import numpy as np
import pytest
import torch


def _plan(first, counts, temperature=1.0, regularize=0.0, top_k=0, top_p=1.0):
    import wavenet_model as wmod
    return wmod._stream_plan(first, counts, temperature, regularize, top_k, top_p)


def test_schedule_of_ragged_prompts_and_counts():
    """head_from = shortest prompt - 1, pitch of first = longest prompt, evaluations = the longest job, row pitch =
    evaluations - head_from (every stream's samples fit in its row)"""
    prompts = [np.arange(5), np.array([7]), np.arange(600) % 256, np.arange(2)]
    p = _plan(prompts, [10, 0, 3, 1000])
    assert p.per_stream and p.ragged and p.n_streams == 4
    assert p.n_given == [5, 1, 600, 2] and p.counts == [10, 0, 3, 1000]
    assert p.head_from == 0 and p.pitch == 600
    assert p.n_evals == max(4 + 10, 0 + 0, 599 + 3, 1 + 1000) == 1001
    assert p.n_samples == 1001
    assert p.first.shape == (4, 600) and p.first.dtype == np.int32
    for s, r in enumerate(prompts):
        assert np.array_equal(p.first[s, :len(r)], r) and not p.first[s, len(r):].any()
    # the evaluations each stream needs all fall inside the launch, and its samples inside its row
    for g, n in zip(p.n_given, p.counts):
        assert g - 1 + n <= p.n_evals and (g - 1 + n - 1) - (g - 1) < p.n_samples
    # all prompts longer than one sample: the head starts at the shortest one's end
    p = _plan([np.arange(5), np.arange(3)], [4, 4])
    assert (p.head_from, p.pitch, p.n_evals, p.n_samples) == (2, 5, 8, 6)


def test_scalar_calls_keep_the_old_schedule():
    p = _plan(np.zeros((3, 7), dtype=np.int64), 20, temperature=0.7, regularize=1e-4, top_k=5, top_p=0.5)
    assert not p.per_stream and not p.ragged
    assert (p.head_from, p.pitch, p.n_evals, p.n_samples) == (6, 7, 26, 20)
    assert p.temperature == [0.7] * 3 and p.top_k == [5] * 3
    # equal-length prompts as a list are the rectangular call, 1-D prompts one stream
    p = _plan([np.arange(4), np.arange(4)], 9)
    assert not p.per_stream and p.first.shape == (2, 4)
    p = _plan([3, 4, 5], 9)
    assert not p.per_stream and p.first.shape == (1, 3)
    # one value per stream: the per-stream path, but the same rectangular shapes
    p = _plan(np.zeros((2, 3), dtype=np.int64), 9, temperature=[0.0, 1.0], top_p=np.array([1.0, 0.9]))
    assert p.per_stream and not p.ragged and p.temperature == [0.0, 1.0] and p.top_p == [1.0, 0.9]
    assert (p.head_from, p.n_samples) == (2, 9)
    p = _plan(np.zeros((2, 3), dtype=np.int64), [9, 9])
    assert p.per_stream and p.ragged                          # counts given per stream: per-stream lists come back


def test_rows_and_records():
    import native
    p = _plan([np.arange(3), np.arange(1)], [2, 4], temperature=[0.0, 1.5], regularize=[1e-4, 0.0], top_k=[0, 7],
              top_p=[1.0, 0.25])
    assert p.n_samples == 4
    u = p.rows([np.zeros(0), np.array([0.1, 0.2, 0.3, 0.4, 0.5])], np.float64, "uniforms", need=[False, True])
    assert u.shape == (2, 4) and np.array_equal(u[1], [0.1, 0.2, 0.3, 0.4]) and not u[0].any()
    f = p.rows(np.array([[1, 2, 3, 4], [5, 6, 7, 8]]), np.int32, "forced")
    assert np.array_equal(f, [[1, 2, 0, 0], [5, 6, 7, 8]])
    recs = p.records()
    assert [(r.n_given, r.top_k, r.temperature, r.top_p) for r in recs] == [(3, 0, 0.0, 1.0), (1, 7, 1.5, 0.25)]
    assert abs(recs[0].regularize - 1e-4) < 1e-10
    # the record layout of include/wavenet_b200.h
    assert ctypes.sizeof(native.GenStreamParams) == 24
    assert [getattr(native.GenStreamParams, f).offset for f in ("n_given", "top_k", "temperature", "regularize", "top_p")] \
        == [0, 4, 8, 12, 16]


def _small(**kw):
    import wavenet_model as wmod
    return wmod.WaveNetModel(layers=2, blocks=1, dilation_channels=8, residual_channels=8, skip_channels=8,
                             end_channels=8, classes=16, output_length=4, kernel_size=2, bias=False, **kw)


RAGGED = [np.arange(3), np.arange(1)]
BAD = [
    ("prompt 2-D", dict(first_samples=[np.zeros((2, 2), dtype=np.int64), np.arange(1)])),
    ("prompt empty", dict(first_samples=[np.zeros(0, dtype=np.int64), np.arange(1)])),
    ("prompt float", dict(first_samples=[np.zeros(3), np.arange(1)])),
    ("prompt bool", dict(first_samples=[np.ones(3, dtype=bool), np.arange(1)])),
    ("counts length", dict(num_samples=[4, 4, 4])),
    ("counts negative", dict(num_samples=[4, -1])),
    ("counts float", dict(num_samples=[4, 2.0])),
    ("counts bool", dict(num_samples=[4, True])),
    ("counts 2-D", dict(num_samples=np.ones((2, 1), dtype=np.int64))),
    ("temperature length", dict(temperature=[1.0, 1.0, 1.0])),
    ("temperature nan", dict(temperature=[1.0, float("nan")])),
    ("temperature inf", dict(temperature=[float("inf"), 1.0])),
    ("temperature bool", dict(temperature=[True, 1.0])),
    ("temperature str", dict(temperature=["1.0", 1.0])),
    ("regularize nan", dict(regularize=[0.0, float("nan")])),
    ("regularize length", dict(regularize=[0.0])),
    ("top_k negative", dict(top_k=[0, -1])),
    ("top_k float", dict(top_k=[0, 2.0])),
    ("top_k bool", dict(top_k=np.array([True, False]))),
    ("top_k length", dict(top_k=[5, 5, 5])),
    ("top_p zero", dict(top_p=[1.0, 0.0])),
    ("top_p above one", dict(top_p=[1.5, 1.0])),
    ("top_p nan", dict(top_p=torch.tensor([float("nan"), 1.0], dtype=torch.float64))),
    ("uniforms short row", dict(uniforms=[np.zeros(4), np.zeros(3)])),
    ("uniforms rows", dict(uniforms=[np.zeros(4)])),
    ("uniforms shape", dict(uniforms=np.zeros((3, 6)))),
    ("forced short row", dict(forced=np.zeros((2, 3), dtype=np.int64))),
    ("forced rows", dict(forced=[np.zeros(6, dtype=np.int64)] * 3)),
]


@pytest.mark.parametrize("case", BAD, ids=[c[0] for c in BAD])
def test_bad_per_stream_arguments_raise_before_any_launch(monkeypatch, case):
    import wavenet_model as wmod

    def no_launch(*a, **k):
        raise AssertionError("the sampler ran")
    monkeypatch.setattr(wmod._Runtime, "generate", no_launch)
    kw = dict(num_samples=[4, 4], first_samples=RAGGED, temperature=1.0)
    kw.update(case[1])
    with pytest.raises(ValueError):
        _small().generate_fast_batch(**kw)


def test_bad_local_conditions_raise_before_any_launch(monkeypatch):
    import wavenet_model as wmod
    monkeypatch.setattr(wmod._Runtime, "generate", lambda *a, **k: (_ for _ in ()).throw(AssertionError("ran")))
    m = _small(local_condition_channels=3, local_condition_hop=4)
    kw = dict(num_samples=[8, 2], first_samples=RAGGED, temperature=0.0)
    y_ok = [np.zeros((3, 3), dtype=np.float32), np.zeros((3, 1), dtype=np.float32)]   # 10 and 2 positions
    with pytest.raises(ValueError):                                   # one series per stream
        m.generate_fast_batch(local_condition=y_ok[:1], **kw)
    with pytest.raises(ValueError):                                   # stream 0 needs ceil(10 / 4) = 3 frames
        m.generate_fast_batch(local_condition=[y_ok[0][:, :2], y_ok[1]], **kw)
    with pytest.raises(ValueError):                                   # channels
        m.generate_fast_batch(local_condition=[np.zeros((2, 3), dtype=np.float32), y_ok[1]], **kw)
    with pytest.raises(ValueError):                                   # a rectangular series must have one row per stream
        m.generate_fast_batch(local_condition=np.zeros((3, 3, 3), dtype=np.float32), **kw)
    with pytest.raises(ValueError):                                   # missing
        m.generate_fast_batch(**kw)


def test_setter_is_exported_and_refuses_a_null_handle():
    import native
    lib = native.lib()
    assert "wn_gen_set_stream_params" in native.SIGNATURES
    assert lib.wn_gen_set_stream_params(None, None) < 0 and b"null handle" in lib.wn_last_error_string()
    rec = (native.GenStreamParams * 1)(native.GenStreamParams(1, 0, 1.0, 0.0, 1.0))
    assert lib.wn_gen_set_stream_params(None, rec) < 0
    with open(_header()) as f:
        header = f.read()
    assert "int wn_gen_set_stream_params(wn_gen_handle* h, const wn_gen_stream_params* params);" in header


def _header():
    import os
    return os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "wavenet_b200.h")
