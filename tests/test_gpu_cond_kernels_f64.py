"""The condition-table kernels (wn_cond_table, wn_cond_table_frames) and the frame sums behind the gradient of V
(wn_cond_frame_sums) alone, through the C ABI, against float64.

These tables are the input of every conditioned block kernel and sampler.  The cases reach the edges the model-level tests do
not: wn_cond_table past its 256-block grid cap (300 items x 2D = 512 at D = 256), table_frames_kernel's 64-frame tiles with
windows at f0 > 0 inside a longer series (y_ld > n_frames, as the sampler passes them), D not a multiple of 64 (FFMA nets),
null bias pointers, and frame sums on both dfg layouts with NaN in the frames the kernel must not read.

Bars: both tables are sequential fp32 sums, so an element is held to 1e-6 of the sum of the absolute values of its terms,
and the identity cases (one-hot rows, U = 0) must be bit-exact.  Frame sums: 1e-5 of max(1, max |sum|), as
test_gpu_local_conditioning.py::test_segment_sums.  Every kernel has a control that the bar misses by at least 10x."""
import pytest
import torch

from test_gpu_kernels_f64 import _gen, _stream

pytestmark = pytest.mark.gpu
NL = 2


def _ptr_table(Vf, Vg, bf, bg):
    """the DEVICE table [n_layers][4] of {Vf, Vg, bf, bg} pointers (0 = null); keeps the tensors alive in its second item"""
    rows = [[0 if t is None else t[i].data_ptr() for t in (Vf, Vg, bf, bg)] for i in range(NL)]
    return torch.tensor(rows, dtype=torch.int64, device="cuda"), (Vf, Vg, bf, bg)


def _scaled_err(got, exact, scale):
    """max over elements of |got - exact| / (sum of |terms|) -- the bar is 1e-6"""
    return float(((got.double() - exact).abs() / scale.clamp(min=1e-30)).max())


def _miss(what, e_wrong, bar=1e-6):
    print(f"  control {what}: {e_wrong:.2e} = {e_wrong / bar:.0f}x the bar")
    assert e_wrong >= 10 * bar, what


@pytest.mark.parametrize("bias", [True, False])
@pytest.mark.parametrize("D", [63, 96, 256, 512])
@pytest.mark.parametrize("n_items", [1, 120, 300])
@pytest.mark.parametrize("G", [1, 3, 80, 1000])
def test_cond_table(G, n_items, D, bias):
    import native
    lib = native.lib()
    g = _gen(G + 7 * n_items + D)
    V = [torch.randn(NL, D, G, 1, generator=g) * G ** -0.5 for _ in range(2)]
    b = [torch.randn(NL, D, generator=g) if bias else None for _ in range(2)]
    h = torch.randn(n_items, G, generator=g)
    hot = torch.arange(n_items) % 2 == 0                       # even rows one-hot (class labels), odd rows dense
    cls = torch.randint(0, G, (n_items,), generator=g)
    rows = hot.nonzero().squeeze(1)
    h[rows] = 0.0
    h[rows, cls[rows]] = 1.0
    tab, keep = _ptr_table(*(None if t is None else t.cuda() for t in (V[0], V[1], b[0], b[1])))
    out = torch.full((NL, n_items, 2 * D), float("nan"), device="cuda")
    native.check(lib.wn_cond_table(tab.data_ptr(), NL, D, G, h.cuda().data_ptr(), n_items, out.data_ptr(), _stream()), "table")
    torch.cuda.synchronize()
    got = out.cpu()
    Vc = torch.cat([V[0], V[1]], 1)[..., 0]                      # (NL, 2D, G)
    bc = torch.zeros(NL, 2 * D) if not bias else torch.cat([b[0], b[1]], 1)
    terms = torch.einsum("lcg,ig->licg", Vc.double(), h.double())
    exact = terms.sum(-1) + bc.double()[:, None]
    scale = terms.abs().sum(-1) + bc.double().abs()[:, None]
    # one-hot rows: exactly bias + one column of V, in fp32
    want_hot = (Vc.permute(0, 2, 1)[:, cls] + bc[:, None])[:, hot]
    assert torch.equal(got[:, hot], want_hot), "one-hot rows must be exactly bias + V[:, g]"
    e = _scaled_err(got, exact, scale)
    print(f"\nwn_cond_table G={G} items={n_items} D={D} bias={bias}: one-hot rows exact, dense rel {e:.2e} (bar 1e-6)")
    assert e <= 1e-6
    if n_items > 1:
        _miss("rows of the next item", _scaled_err(got[:, :-1], exact[:, 1:], scale[:, :-1]))


def _pack_u(U, D, C):
    """every layer's [Uf; Ug] (2D, C) packed by wn_pack_gate_weights (R = C, k = 1): [NL][C][wn_n1p(D)]"""
    import native
    lib = native.lib()
    n1p = lib.wn_n1p(D)
    out = torch.empty(NL, C, n1p, device="cuda")
    bias = torch.empty(n1p, device="cuda")
    for i in range(NL):
        uf, ug = U[i, :D, :, None].contiguous().cuda(), U[i, D:, :, None].contiguous().cuda()
        native.check(lib.wn_pack_gate_weights(uf.data_ptr(), ug.data_ptr(), None, None, C, D, 1, out[i].data_ptr(),
                                              bias.data_ptr(), _stream()), "pack U")
    return out


FRAME_CASES = [  # n_frames, f0 (window start in y), C, D
    (1, 0, 4, 63), (63, 5, 80, 96), (64, 0, 1, 256), (65, 3, 200, 512), (200, 37, 80, 63), (200, 0, 4, 256),
    (65, 64, 200, 96), (64, 1, 80, 512),
]


@pytest.mark.parametrize("with_base", [False, True])
@pytest.mark.parametrize("case", range(len(FRAME_CASES)))
def test_cond_table_frames(case, with_base):
    import native
    lib = native.lib()
    nf, f0, C, D = FRAME_CASES[case]
    n_items, F = 3, f0 + nf + 11                                 # y_ld = F > n_frames: a window inside a longer series
    g = _gen(100 + case)
    U = torch.randn(NL, 2 * D, C, generator=g) * C ** -0.5
    y = torch.randn(n_items, C, F, generator=g)
    bias = case % 2 == 0 or with_base                            # null bias pointers on some of the base-less cases
    bf, bg = (torch.randn(NL, D, generator=g), torch.randn(NL, D, generator=g)) if bias else (None, None)
    base = torch.randn(NL, n_items, 2 * D, generator=g) if with_base else None
    tab, keep = _ptr_table(None, None, None if bf is None else bf.cuda(), None if bg is None else bg.cuda())
    y_d, base_d = y.cuda(), None if base is None else base.cuda()

    def run(Upk, f_start):
        out = torch.full((NL, n_items, nf, 2 * D), float("nan"), device="cuda")
        native.check(lib.wn_cond_table_frames(tab.data_ptr(), Upk.data_ptr(), NL, D, native.ptr(base_d), C,
                                              y_d.data_ptr() + 4 * f_start, F, n_items, nf, out.data_ptr(), _stream()),
                     "table frames")
        torch.cuda.synchronize()
        return out.cpu()

    if base is not None:
        b0 = base
    elif bias:
        b0 = torch.cat([bf, bg], 1)[:, None].expand(NL, n_items, 2 * D)
    else:
        b0 = torch.zeros(NL, n_items, 2 * D)
    zero = run(_pack_u(torch.zeros_like(U), D, C), f0)
    assert torch.equal(zero, b0[:, :, None].expand_as(zero)), "U = 0 must give exactly the base"
    got = run(_pack_u(U, D, C), f0)

    def ref(fs, with_b=True):
        terms = torch.einsum("lck,ikf->lifck", U.double(), y.double()[:, :, fs:fs + nf])
        b = b0.double()[:, :, None, :] if with_b else 0.0
        return terms.sum(-1) + b, terms.abs().sum(-1) + (b0.double().abs()[:, :, None, :] if with_b else 0.0)

    exact, scale = ref(f0)
    e = _scaled_err(got, exact, scale)
    print(f"\nwn_cond_table_frames n_frames={nf} f0={f0} y_ld={F} C={C} D={D} base={with_base} bias={bias}: "
          f"U = 0 exact, rel {e:.2e} (bar 1e-6)")
    assert e <= 1e-6
    _miss("frame offset f0 + 1", _scaled_err(got, ref(f0 + 1)[0], scale))
    if with_base:
        _miss("base omitted", _scaled_err(got, ref(f0, with_b=False)[0], scale))


def _dfg(B, L, C, gz, pair, seed):
    """dfg on the frames layout (B, L, C) fp32 or the chunked pair layout, NaN in the frames < gz; and its float64 value"""
    v = torch.randn(B, L, C, generator=_gen(seed))
    if pair:
        hi = v.to(torch.bfloat16)
        lo = (v - hi.float()).to(torch.bfloat16)
        val = hi.double() + lo.double()
        src = torch.stack([hi, lo], 1).view(B, 2, L, C // 8, 8).permute(0, 1, 3, 2, 4).contiguous()
        src[:, :, :, :gz] = float("nan")
    else:
        val = v.double()
        src = v.clone()
        src[:, :gz] = float("nan")
    return src.cuda(), val


@pytest.mark.parametrize("pair,B,L,C", [(p, 1, 300, 512) for p in (0, 1)] + [(p, 8, 700, 200) for p in (0, 1)] +
                         [(p, 5, 64, 1024) for p in (0, 1)] + [(0, 3, 1037, 126), (0, 8, 500, 63)])   # C % 32 != 0: frames only
def test_cond_frame_sums(pair, B, L, C):
    import native
    lib = native.lib()
    for gz in (0, 37, L - 1):
        src, val = _dfg(B, L, C, gz, pair, B + L + C + gz)
        outs = []
        for _ in range(2):
            out = torch.full((B, C), float("nan"), device="cuda")
            native.check(lib.wn_cond_frame_sums(src.data_ptr(), pair, B, L, C, gz, out.data_ptr(), _stream()), "frame sums")
            torch.cuda.synchronize()
            outs.append(out.cpu())
        assert torch.equal(outs[0], outs[1]), "repeated calls must be bit-identical"
        want = val[:, gz:].sum(1)
        bar = 1e-5 * max(1.0, float(want.abs().max()))
        err = float((outs[0].double() - want).abs().max())
        print(f"\nwn_cond_frame_sums pair={pair} B={B} L={L} C={C} gz={gz}: |err| {err:.2e} (bar {bar:.2e})")
        assert err <= bar
        wrong = float((outs[0].double() - val[:, gz + 1:].sum(1)).abs().max())
        print(f"  control gz + 1: {wrong:.2e} = {wrong / bar:.0f}x the bar")
        assert wrong >= 10 * bar
