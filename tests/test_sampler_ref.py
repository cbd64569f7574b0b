"""tests/sampler_ref.py (the float64 whole-sequence reference the long sampler tests compare against) pinned on the CPU:
against the oracle's queue-by-queue generate_fast, against the stored golden logits, against the per-position folded
queue run for conditioned nets; and the proof that a comparison with it can fail: a reference with one deep tap wrong
moves the logits by hundreds of times the 1e-4 bar once the run is longer than that tap's dilation, and by nothing at
all in the first 64 evaluations."""
import math

import numpy as np
import pytest
import torch

import local_ref
import sampler_ref as R
import upsample_ref
from oracle import wavenet_oracle as O
from helpers import spec_from_golden, params_from_golden, rel_err, weight_checksum

TOL = 1e-4
SMALL = ["cfg1", "odd_bias", "k3", "deep"]


def _dil(spec):
    return [d for d, _ in spec.dilation_schedule()]


def _net(golden, name):
    g = golden(f"net_{name}.npz")
    spec = spec_from_golden(g)
    p = params_from_golden(g)
    if not p:                                   # seeded weights: the file stores their checksum
        p = O.init_params(spec, seed=0)
        assert weight_checksum(p) == float(g["w_checksum"])
    return g, spec, p


def _cfg2(golden):
    return _net(golden, "cfg2")


# ---------------------------------------------------------------------------------------------- the oracle's queues
@pytest.mark.parametrize("start", ["one", "first"])
@pytest.mark.parametrize("name", SMALL)
def test_matches_oracle_generate_fast(golden, name, start):
    """Runs of 2.5 receptive fields from reset queues: the oracle steps its ring queues sample by sample in fp32."""
    g, spec, p = _net(golden, name)
    first = g["first"][:1] if start == "one" else g["first"]
    n = math.ceil(2.5 * spec.receptive_field) + 1
    w = R.weights(p)
    # argmax, free running
    tr = O.generate_fast(p, spec, n, first_samples=first, temperature=0.0, keep_logits=True)
    ref = R.logits(w, _dil(spec), R.inputs(first, tr.indices))[len(first) - 1:]
    assert ref.shape == tr.logits.shape and rel_err(tr.logits, ref) < 1e-5
    got, margin, _ = R.choose(ref.astype(np.float32), 0.0, 0.0)
    bad = got != tr.indices
    assert np.all(margin[bad] < TOL * np.abs(ref).max()) and bad.sum() <= 1
    assert np.array_equal(R.choose(tr.logits, 0.0, 0.0)[0], tr.indices)
    # sampled with temperature and regularizer: the oracle keeps logits - regularizer
    uni = np.random.RandomState(3).random_sample(n)
    tr = O.generate_fast(p, spec, n, first_samples=first, temperature=0.8, regularize=1e-4, uniforms=uni, keep_logits=True)
    ref = R.logits(w, _dil(spec), R.inputs(first, tr.indices))[len(first) - 1:]
    assert rel_err(tr.logits, ref - R.regularizer(256, 1e-4)[None, :]) < 1e-5
    got, _, edge = R.choose(tr.logits, 0.8, 0.0, uni)            # the oracle's own fp32 logits: the same draw
    assert np.all(edge[got != tr.indices] < 1e-6) and (got != tr.indices).sum() <= 1
    got, _, edge = R.choose(ref.astype(np.float32), 0.8, 1e-4, uni)
    assert np.all(edge[got != tr.indices] < 1e-5) and (got != tr.indices).sum() <= 2


# ---------------------------------------------------------------------------------------------- stored golden logits
@pytest.mark.parametrize("name", SMALL)
def test_matches_golden_streams_small(golden, name):
    g, spec, p = _net(golden, name)
    w, first = R.weights(p), g["first"]
    for kind in ("argmax", "sample"):           # the files store the logits before the regularizer
        ref = R.logits(w, _dil(spec), R.inputs(first, g[f"gen_{kind}_idx"]))[len(first) - 1:]
        assert rel_err(g[f"gen_{kind}_logits"], ref) < 1e-5, kind
    got, _, edge = R.choose(g["gen_sample_logits"], 0.8, 1e-4, g["gen_sample_uniforms"])
    assert np.all(edge[got != g["gen_sample_idx"]] < 1e-6) and (got != g["gen_sample_idx"]).sum() <= 1
    assert np.array_equal(R.choose(g["gen_argmax_logits"], 0.0, 0.0)[0], g["gen_argmax_idx"])


def test_matches_golden_streams_cfg2(golden):
    g, spec, p = _cfg2(golden)
    w = R.weights(p)
    ref = R.logits(w, _dil(spec), R.inputs([128], g["gen_argmax_idx"]))
    assert rel_err(g["gen_argmax_logits"], ref) < 1e-5
    first = g["gen_sample_first"]
    ref = R.logits(w, _dil(spec), R.inputs(first, g["gen_sample_idx"]))[len(first) - 1:]
    assert rel_err(g["gen_sample_logits"], ref) < 1e-5
    got, _, edge = R.choose(g["gen_sample_logits"], 1.0, 0.0, g["gen_sample_uniforms"])
    assert np.all(edge[got != g["gen_sample_idx"]] < 1e-6) and (got != g["gen_sample_idx"]).sum() <= 1


def test_matches_golden_snapshot_with_real_history(golden):
    """The chaconne snapshot: a full receptive field of real audio given, then 200 argmax samples."""
    gs, gio = golden("snapshot_chaconne_state.npz"), golden("snapshot_chaconne_io.npz")
    rf = int(gs["receptive_field"])
    first = gio["clip"].astype(np.int64)[:rf]
    dil = R.dilations_of(int(gs["layers"]), int(gs["blocks"]))
    ref = R.logits(R.weights(params_from_golden(gs)), dil, R.inputs(first, gio["gen_argmax_idx"]))[rf - 1:]
    assert rel_err(gio["gen_argmax_logits"], ref) < 1e-5
    assert np.array_equal(R.choose(ref.astype(np.float32), 0.0, 0.0)[0][:8], gio["gen_argmax_idx"][:8])


# ---------------------------------------------------------------------------------------------- conditioned nets
def _small_cond(k=2, C=3, G=2, scales=None, seed=0):
    kw = dict(layers=3, blocks=2, dilation_channels=8, residual_channels=6, skip_channels=10, end_channels=8, classes=16,
              output_length=8, kernel_size=k, bias=True)
    spec = O.NetSpec(**kw)
    g = torch.Generator().manual_seed(seed)
    p = {n: (0.4 * torch.randn(v.shape, generator=g)).double() for n, v in O.init_params(spec, seed).items()}
    for i in range(spec.n_layers):
        for nm in ("filter", "gate"):
            p[f"{nm}_local_convs.{i}.weight"] = 0.5 * torch.randn(8, C, 1, generator=g).double()
            p[f"{nm}_cond_convs.{i}.weight"] = 0.5 * torch.randn(8, G, 1, generator=g).double()
    for j, s in enumerate(scales or ()):
        p[f"local_upsample.{j}.weight"] = 0.5 * torch.randn(C, C, 2 * s, generator=g).double()
        p[f"local_upsample.{j}.bias"] = 0.5 * torch.randn(C, generator=g).double()
    return spec, p


@pytest.mark.parametrize("k,hop,scales", [(2, 1, None), (2, 3, None), (2, 7, None), (3, 5, None), (2, 6, (2, 3)), (3, 20, (4, 5))])
def test_conditioned_matches_per_position_folded_queue_run(k, hop, scales):
    """The oracle's fast-generation step on reset ring queues, each position's condition terms folded into that
    position's filter / gate biases: every evaluation from the first, over 2.5 receptive fields and more."""
    spec, p = _small_cond(k=k, scales=scales)
    L = max(140, math.ceil(2.5 * spec.receptive_field))
    idx = torch.randint(0, 16, (1, L), generator=torch.Generator().manual_seed(4))
    y = torch.randn(1, 3, -(-L // hop), generator=torch.Generator().manual_seed(5)).double()
    h = torch.randn(1, 2, generator=torch.Generator().manual_seed(6)).double()
    got = R.logits(R.weights(p), _dil(spec), idx[0].numpy(), h=h[0].numpy(), y=y[0].numpy(), hop=hop, scales=scales)
    c = y[0].repeat_interleave(hop, dim=1) if scales is None else upsample_ref.upsample(p, scales, y)[0]
    queues = [O.RingQueue((k - 1) * d + 1, spec.residual_channels) for d in _dil(spec)]
    for q in queues:
        q.data = q.data.double()

    def queue_fn(hq, d, init_d, i):
        queues[i].enqueue(hq[0])
        return queues[i].dequeue(num_deq=k, dilation=d).unsqueeze(0)

    with torch.no_grad():
        for t in range(L):
            q = local_ref.folded(p, spec, c[:, t], h[0])
            out = O.stack_folded(q, spec, O.one_hot(idx[:, t:t + 1], 16).double(), queue_fn)[0, :, 0].numpy()
            assert np.abs(out - got[t]).max() < 1e-12 * np.abs(got).max(), t
    # past the receptive field the whole-sequence training reference says the same
    x = O.one_hot(idx, 16).double()
    want = (local_ref.stack_direct(p, spec, x, y, hop, h) if scales is None
            else upsample_ref.stack_direct(p, spec, x, y, scales, h))[0].numpy().T
    n = L - spec.receptive_field + 1
    assert np.abs(want[-n:] - got[-n:]).max() < 1e-12 * np.abs(got).max()


def test_reset_queues_are_not_a_zero_padded_forward(golden):
    """With biases, zeros in the queues differ from the layers' response to a silent input: the reference models the
    queues, and a forward pass over the run is a different function before the receptive field is full."""
    g, spec, p = _net(golden, "odd_bias")
    rf = spec.receptive_field
    idx = np.random.RandomState(0).randint(0, 256, 3 * rf)
    ref = R.logits(R.weights(p), _dil(spec), idx)
    x = torch.cat([torch.zeros(1, 256, rf - 1), O.one_hot(torch.tensor(idx[None]), 256)], 2).double()      # silence first
    fwd = O.stack_direct({k: v.double() for k, v in p.items()}, spec, x)[0].numpy().T[-len(idx):]
    assert fwd.shape == ref.shape
    assert rel_err(fwd[rf - 1:], ref[rf - 1:]) < 1e-12 and rel_err(fwd[:rf - 1], ref[:rf - 1]) > 1e-2


# ---------------------------------------------------------------------------------------------- the tests can fail
def test_mutated_references_differ_only_on_long_runs(golden):
    """cfg-2 weights, 1 500 teacher-forced evaluations.  One layer's history replaced by zeros, or read one step late,
    moves the logits of evaluations >= 1 100 by more than 100 times the bar and those of evaluations < 64 by nothing:
    runs shorter than the dilation cannot see such a bug, whatever they compare with."""
    g, spec, p = _cfg2(golden)
    w, dil = R.weights(p), _dil(spec)
    idx = np.random.RandomState(0).randint(0, 256, 1500)
    base = R.logits(w, dil, idx)
    scale = np.abs(base).max()
    for layer in (7, 8, 9, 47, 48, 49):
        assert dil[layer] in (128, 256, 512)
        for kind in ("zero_history", "late_tap"):
            bad = R.logits(w, dil, idx, mutate=(kind, layer))
            late = np.abs(bad - base)[1100:].max() / scale
            early = np.abs(bad - base)[:64].max() / scale
            assert late > 100 * TOL and early < TOL, (kind, layer, late, early)
    # local conditioning: the frame changing one sample early
    rng = np.random.RandomState(1)
    for i in range(spec.n_layers):
        for nm in ("filter", "gate"):
            w[f"{nm}_local_convs.{i}.weight"] = rng.uniform(-1, 1, (256, 8, 1)) / math.sqrt(8)
    y = rng.randn(8, -(-1500 // 80))
    base = R.logits(w, dil, idx, y=y, hop=80)
    bad = R.logits(w, dil, idx, y=y, hop=80, mutate=("frame_off_by_one",))
    assert np.abs(bad - base)[1100:].max() / np.abs(base).max() > 100 * TOL


def test_choose_edges():
    lg = np.zeros((4, 8), dtype=np.float32)
    lg[:, 3] = lg[:, 5] = 2.0                                                     # a tie: the lowest index wins
    idx, margin, edge = R.choose(lg, 0.0, 0.0)
    assert idx.tolist() == [3, 3, 3, 3] and np.all(margin == 0) and edge is None
    assert R.choose(lg, 0.0, 1.0)[0].tolist() == [3] * 4                          # (3 - 4)^2 = (5 - 4)^2: still a tie
    lg[:, 0] = -200.0                                                             # probability 0 in fp32: u = 0 skips it
    idx, _, edge = R.choose(lg, 1.0, 0.0, np.array([0.0, 1 - 2.0 ** -53, 0.5, 0.25]))
    assert idx[0] == 1 and idx[1] == 7 and edge[0] == 0.0
    for i, u in enumerate((0.5, 0.25)):
        e = np.exp(lg[0] - lg[0].max())
        assert idx[2 + i] == O.choice_from_probs((e / e.sum()).astype(np.float32), u)
