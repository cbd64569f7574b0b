"""Helpers shared by the parity tests (oracle side only; nothing here is product code)."""
import numpy as np
import torch

from oracle import wavenet_oracle as O


def spec_from_golden(g, output_length=None):
    kw = {k[3:]: g[k].item() for k in g.files if k.startswith("kw_")}
    kw["bias"] = bool(kw["bias"])
    if output_length is not None:
        kw["output_length"] = output_length
    return O.NetSpec(**kw)


def params_from_golden(g):
    return {k[2:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("w:")}


def weight_checksum(params):
    return sum(float(np.abs(v.detach().cpu().numpy()).astype(np.float64).sum()) for v in params.values())


def rel_err(a, b):
    """max |a-b| / max |b|: the relative measure all fp32 parity gates use (tolerance 1e-4)."""
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def classify_stream(got_idx, ref_idx, ref_margins, tol=1e-4):
    """Compare two argmax streams.  Returns (n_equal_prefix, first_mismatch_is_near_tie)."""
    got_idx, ref_idx = np.asarray(got_idx), np.asarray(ref_idx)
    neq = np.nonzero(got_idx != ref_idx)[0]
    if len(neq) == 0:
        return len(ref_idx), True
    i = int(neq[0])
    return i, bool(ref_margins[i] < tol)


def separate_head_relu_ties(params, spec, x, out_len, margin=2e-5, step=None):
    """Gradients are discontinuous where a head ReLU input is exactly zero: an fp32-class difference (tensor cores
    vs FFMA, or just another summation order) that flips the sign of a pre-activation of size 1e-7 switches one
    mask element and moves a weight gradient by percent.  The analogue of the argmax near-tie rule for the backward
    tests: nudge the last skip bias and the end_conv_1 bias (per channel, in float64 on the oracle) until no head ReLU
    input of this test case lies within `margin` of zero.  Returns a new fp32 parameter dict."""
    step = 5 * margin if step is None else step
    p = {k: v.detach().clone().double() for k, v in params.items()}
    last = spec.layers * spec.blocks - 1
    taps = {}
    O.stack_direct(p, spec, x.double(), taps)
    sk = taps["skip"][..., -out_len:].clone()                           # (B, S, out_len)
    for name, pre_of in ((f"skip_convs.{last}.bias", lambda: sk),
                         ("end_conv_1.bias", lambda: F_conv1d(torch.relu(sk), p["end_conv_1.weight"], p["end_conv_1.bias"]))):
        if name not in p:              # bias=False nets have no skip bias to nudge: see tie_free_indices
            continue
        pre = pre_of()
        for c in range(pre.shape[1]):
            v, off = pre[:, c, :], 0.0
            while float((v + off).abs().min()) < margin:
                off += step
            p[name][c] += off
            pre[:, c, :] += off
    return {k: v.float() for k, v in p.items()}


def tie_free_indices(params, spec, B, L, out_len, margin=5e-6, seed0=2, tries=30):
    """(B, L) class indices for which no relu(skip) input of the oracle lies within `margin` of zero: the alternative to a
    bias nudge for nets without skip biases.  Feasible only for small B * out_len (the chance of a miss grows with it)."""
    p = {k: v.detach().double() for k, v in params.items()}
    for s in range(seed0, seed0 + tries):
        idx = torch.randint(0, spec.classes, (B, L), generator=torch.Generator().manual_seed(s))
        taps = {}
        O.stack_direct(p, spec, O.one_hot(idx, spec.classes).double(), taps)
        if float(taps["skip"][..., -out_len:].abs().min()) > margin:
            return idx
    raise RuntimeError("no tie-free input found")


def F_conv1d(x, w, b):
    return torch.nn.functional.conv1d(x, w, b)


# ---------------------------------------------------------------- kernel-level float64 bars (test_gpu_*_f64.py)
def kernel_rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-30))


def tc_acc(K):
    """Allowance for the fp32 accumulation of a K-long contraction on the tensor cores, which the float64 emulation does not
    model: measured on an H100 it reaches ~1e-5 (max-relative) at K = 512 and grows with K, also where the operand error
    is tiny, while spread over all frames and channels rather than on a range boundary.

    What the bar then still catches, per output tensor (~4e-5 to 7e-5 for the K of these tests): any frame-range, tap,
    tile, plane or bias error (the controls miss by 10^3 or more); for bf16 pairs, a dropped lo-plane product of either
    operand (the operand-term controls of test_two_launch_and_ffma_block_fwd); single-pass bf16 against its own emulation
    at 0.25 e_emu.  What it cannot catch: an error below about 2^-16 of the output scale -- one missing lo-plane product on
    a single k-slab."""
    return 2.0 ** -16 * (max(K, 256) / 256) ** 0.5


def worst_element(got, exact):
    """(index, |error|) of the worst element, to localize a failure (frame axis = dim 1 of the frames layouts)"""
    diff = (torch.as_tensor(got).double() - torch.as_tensor(exact).double()).abs()
    i = int(diff.argmax())
    return tuple(int(v) for v in torch.unravel_index(torch.tensor(i), diff.shape)), float(diff.flatten()[i])


def kernel_check(what, got, exact, emu=None, kind="emu", K=256):
    """Assert the bar of `kind` ("emu": operand-split kernels, "bf16": single pass, "ffma"); returns the bar.
    K: the longest contraction feeding the output (sets the accumulation allowance of the tensor-core kernels)."""
    e = kernel_rel(got, exact)
    if kind == "ffma":
        bar, msg = 1e-5, ""
    else:
        e_emu = kernel_rel(emu, exact)
        bar, msg = 2 * e_emu + tc_acc(K), f" e_emu {e_emu:.2e}"
        if kind == "bf16":
            e_ke = kernel_rel(got, emu)
            msg += f" vs-emulation {e_ke:.2e} (bar {0.25 * e_emu:.2e})"
            assert e_ke <= 0.25 * e_emu, f"{what}: kernel vs emulated operands {e_ke:.3e} > {0.25 * e_emu:.3e}"
    idx, ad = worst_element(got, exact)
    print(f"  {what}: rel_err {e:.2e} bar {bar:.2e}{msg} worst at {idx}")
    assert e <= bar, f"{what}: rel_err {e:.3e} > bar {bar:.3e} (worst element {idx}, |error| {ad:.3e})"
    return bar


def kernel_miss(what, got, wrong, bar, factor=10):
    """negative control: a reference with one deliberate mistake must be missed by >= factor x the bar"""
    e = kernel_rel(got, wrong)
    print(f"  control {what}: rel_err {e:.2e} = {e / bar:.1f}x bar")
    assert e >= factor * bar, f"control {what}: only {e:.3e} from a wrong reference (bar {bar:.3e})"


# ---------------------------------------------------------------- product-side helpers (GPU tests)
def build_model(g, device="cuda", output_length=None):
    """WaveNetModel (product) with the constructor args / weights stored in a golden file."""
    import wavenet_model as wmod
    kw = {k[3:]: (bool(g[k]) if k == "kw_bias" else int(g[k])) for k in g.files if k.startswith("kw_")}
    if output_length is not None:
        kw["output_length"] = output_length
    torch.manual_seed(0)
    m = wmod.WaveNetModel(**kw)
    ref = params_from_golden(g)
    if ref:
        m.load_state_dict(ref, strict=True)
    else:
        assert weight_checksum(m.state_dict()) == float(g["w_checksum"])
    return m.to(device)


def snapshot_model(gs, device="cuda", output_length=64):
    import wavenet_model as wmod
    m = wmod.WaveNetModel(layers=int(gs["layers"]), blocks=int(gs["blocks"]), dilation_channels=32,
                          residual_channels=32, skip_channels=1024, end_channels=512, classes=256,
                          output_length=output_length, kernel_size=2, bias=True)
    m.load_state_dict(params_from_golden(gs), strict=True)
    return m.to(device)


def one_hot_cuda(idx, classes=256):
    idx = torch.as_tensor(np.asarray(idx)).long().cuda()
    b, l = idx.shape
    return torch.zeros(b, classes, l, device="cuda").scatter_(1, idx.view(b, 1, l), 1.0)


def assert_stream_parity(got_idx, ref_idx, ref_logits, tol=1e-4):
    """Bit-exact index stream, except that a first mismatch is accepted only where the reference's own top-1/top-2
    logit gap is below tol (a tie-break divergence, SURVEY.md section 7 hard part 3).  Returns the agreed prefix."""
    got_idx, ref_idx = np.asarray(got_idx), np.asarray(ref_idx)
    neq = np.nonzero(got_idx != ref_idx)[0]
    if len(neq) == 0:
        return len(ref_idx)
    i = int(neq[0])
    top2 = np.sort(ref_logits[i])[-2:]
    assert top2[1] - top2[0] < tol * max(1.0, float(np.abs(ref_logits[i]).max())), (
        f"stream diverges at step {i}: got {got_idx[i]} want {ref_idx[i]}, reference margin {top2[1] - top2[0]:.3e}")
    return i
