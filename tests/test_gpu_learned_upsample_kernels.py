"""The kernels of the learned local-conditioning upsampler alone, through the C ABI, against float64 references in the style
of tests/test_gpu_kernels_f64.py: the K-slab block forward (wn_tb_block_fwd_local, with the features converted by
wn_tb_local_from_channels and U packed by wn_tb_pack_local_weights) at tile-boundary frame ranges with NaN sentinels, and the
backward's dU (wn_local_weight_grad) and dc (wn_local_data_grad_add) contractions on the chunked dfg."""
import ctypes
import functools

import pytest
import torch

import block_ref as BR
from test_gpu_kernels_f64 import FWD_CASES, TB_PRECS, _check, _gen, _miss, _nan, _pair, _planes, _rel, _sentinel_kept, _stream

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _model(C, Cl, prec):
    import wavenet_model as wmod
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(C + Cl)
        m = wmod.WaveNetModel(layers=2, blocks=1, dilation_channels=C, residual_channels=C, skip_channels=C, end_channels=256,
                              classes=256, output_length=8, kernel_size=2, bias=True, local_condition_channels=Cl,
                              local_condition_hop=4, local_condition_upsample_scales=(4,))
    g = _gen(17)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith(".bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.5)
            if "_local_convs." in n:
                p.copy_(torch.randn(p.shape, generator=g) * Cl ** -0.5)
    m = m.cuda()
    m._runtime().tc_precision = "bf16x2" if prec == "pairs" else "bf16"
    return m


@pytest.mark.parametrize("prec,C", TB_PRECS)
@pytest.mark.parametrize("case,Cl", [(0, 80), (1, 80), (3, 80), (5, 80), (7, 80), (1, 1), (5, 200), (6, 96)])
def test_kslab_block_fwd(prec, C, case, Cl):
    import native
    lib = native.lib()
    B, L, d, in_s, out_s, sk_s, sk_init = FWD_CASES[case]
    m = _model(C, Cl, prec)
    rt_packs = m._runtime().packed_weights(_stream())
    tb_w, tb_b, p_id = rt_packs["tb"]
    u_all = rt_packs["tb_local"][0]
    sd = {n: v.detach().cpu() for n, v in m.state_dict().items()}
    W = BR.layer_weights(sd, 1)
    uf, ug = sd["filter_local_convs.1.weight"][:, :, 0], sd["gate_local_convs.1.weight"][:, :, 0]
    g = _gen(300 + case)
    h = torch.randn(B, L, C, generator=g)
    c = torch.randn(B, Cl, L, generator=g)
    skip0 = None if sk_init else torch.randn(B, L - sk_s, C, generator=g)
    cpad = lib.wn_tb_local_padded_channels(Cl, p_id)
    c_pair = _nan(B, 2, cpad // 8, L, 8, dtype=torch.bfloat16)
    native.check(lib.wn_tb_local_from_channels(c.cuda().data_ptr(), c_pair.data_ptr(), B, Cl, L, p_id, _stream()), "convert")
    h_in, h_out = _pair(h), _nan(B, 2, C // 8, L, 8, dtype=torch.bfloat16)
    skip = _nan(B, C // 4, L - sk_s, 4) if sk_init else BR.chunks4_from_frames(skip0).cuda()
    fg = _nan(B, 2 * C // 4, L, 4)
    a = native.TbBlockArgs()
    a.d_h_in, a.d_h_out, a.d_skip, a.d_w_all, a.d_bias4 = h_in.data_ptr(), h_out.data_ptr(), skip.data_ptr(), tb_w.data_ptr(), tb_b[1].data_ptr()
    a.layer, a.n_layers, a.channels, a.precision, a.B, a.L = 1, tb_w.shape[0], C, p_id, B, L
    a.dilation, a.in_start, a.out_start, a.skip_start, a.skip_init, a.d_fg_save = d, in_s, out_s, sk_s, sk_init, fg.data_ptr()
    native.check(lib.wn_tb_block_fwd_local(ctypes.byref(a), None, c_pair.data_ptr(), Cl, u_all.data_ptr(), _stream()), "fwd local")
    torch.cuda.synchronize()
    _sentinel_kept("h_out", h_out, out_s)
    _sentinel_kept("fg_save", fg, out_s)
    hp = _planes(h_in)
    ct = c.transpose(1, 2)[:, out_s:]                     # (B, T, Cl) on the output frames

    def ref(mode, pair_out, u_scale=1.0):
        # the K-slabs are Uf c[t] / Ug c[t] on top of the pass-A sum: a per-position term of the filter / gate biases
        Wm = dict(W)
        Wm["bf"] = W["bf"].double() + BR.mm(ct, uf * u_scale, mode)
        Wm["bg"] = W["bg"].double() + BR.mm(ct, ug * u_scale, mode)
        return BR.block_forward(hp, Wm, d, in_s, out_s, sk_s, skip0, mode=mode, pair_out=pair_out)

    ex, em = ref("exact", False), ref(prec, True)
    got_h = BR.value(_planes(h_out))[:, out_s:]
    got_fg = BR.frames_from_chunks4(fg.cpu())[:, out_s:]
    got_sk = BR.frames_from_chunks4(skip.cpu())
    kind, K = ("emu" if prec == "pairs" else "bf16"), 2 * C + cpad
    print(f"\nwn_tb_block_fwd_local {prec} {C} C={Cl}: B={B} L={L} d={d} in={in_s} out={out_s} skip={sk_s} init={sk_init}")
    bar = _check("h_out", got_h, ex["h_out"], em["h_out"], kind, K=K)
    _check("skip", got_sk, ex["skip"], em["skip"], kind, K=K)
    _check("tanh", got_fg[..., :C], ex["f"], em["f"], kind, K=K)
    _check("sigmoid", got_fg[..., C:], ex["g"], em["g"], kind, K=K)
    if case == 1 and prec == "pairs":
        _miss("no local term", got_h, ref("exact", False, 0.0)["h_out"], bar)


def _dfg(B, L, N, gz, seed):
    """random chunked pair dfg (B, 2, N/8, L, 8) with NaN in the frames < gz (the kernels must not read them), and its value"""
    v = torch.randn(B, L, N, generator=_gen(seed))
    hi, lo = BR.split_bf16(v)
    p = BR.pair_from_frames(v)
    p[:, :, :, :gz] = float("nan")
    return p.cuda(), (hi.double() + lo.double())


DW_CASES = [(1, 200, 0, 1), (3, 1037, 127, 80), (2, 1100, 256, 200), (3, 700, 129, 96), (1, 300, 300, 80)]


@pytest.mark.parametrize("B,L,gz,C", DW_CASES)
@pytest.mark.parametrize("N", [512, 1024])
def test_local_weight_grad(B, L, gz, C, N):
    import native
    lib = native.lib()
    dfg, val = _dfg(B, L, N, gz, 5 + C)
    c = torch.randn(B, C, L, generator=_gen(6 + C))
    work = torch.empty(lib.wn_local_weight_grad_workspace_bytes(N, C) // 4, device="cuda")
    du = _nan(N, C)
    native.check(lib.wn_local_weight_grad(dfg.data_ptr(), B, L, N, gz, c.cuda().data_ptr(), C, work.data_ptr(), du.data_ptr(),
                                          _stream()), "dU")
    torch.cuda.synchronize()
    exact = torch.einsum("btn,bkt->nk", val[:, gz:], c.double()[:, :, gz:])
    if gz >= L:
        assert torch.equal(du.cpu(), torch.zeros(N, C))
        return
    print(f"\nwn_local_weight_grad B={B} L={L} gz={gz} N={N} C={C}")
    bar = _check("dU", du.cpu(), exact, kind="ffma")
    if gz > 0:
        _miss("gz - 1", du.cpu(), torch.einsum("btn,bkt->nk", val[:, gz - 1:], c.double()[:, :, gz - 1:]), bar)
    du2 = _nan(N, C)
    native.check(lib.wn_local_weight_grad(dfg.data_ptr(), B, L, N, gz, c.cuda().data_ptr(), C, work.data_ptr(), du2.data_ptr(),
                                          _stream()), "dU")
    assert torch.equal(du, du2)                          # deterministic


@pytest.mark.parametrize("B,L,gz,C", DW_CASES)
@pytest.mark.parametrize("N", [512, 1024])
def test_local_data_grad_add(B, L, gz, C, N):
    import native
    lib = native.lib()
    dfg, val = _dfg(B, L, N, gz, 7 + C)
    u = torch.randn(N, C, generator=_gen(8 + C))
    dc0 = torch.randn(B, C, L, generator=_gen(9 + C))
    runs = []
    for _ in range(2):
        dc = dc0.cuda()
        native.check(lib.wn_local_data_grad_add(dfg.data_ptr(), B, L, N, gz, u.cuda().data_ptr(), C, dc.data_ptr(), _stream()),
                     "dc")
        torch.cuda.synchronize()
        runs.append(dc.cpu())
    assert torch.equal(runs[0], runs[1])                 # deterministic: the same bits on two runs
    got = runs[0]
    assert torch.equal(got[:, :, :gz], dc0[:, :, :gz])   # frames < gz untouched
    if gz >= L:
        return
    exact = torch.einsum("nk,btn->bkt", u.double(), val[:, gz:])
    print(f"\nwn_local_data_grad_add B={B} L={L} gz={gz} N={N} C={C}")
    _check("dc", got[:, :, gz:].double() - dc0[:, :, gz:].double(), exact, kind="ffma")


def test_converter_pads_to_the_forward_slab_width():
    import native
    lib = native.lib()
    for prec, width in ((native.PREC_BF16_PAIRS, 32), (native.PREC_BF16, 64)):
        for C in (1, 32, 33, 80, 200):
            assert lib.wn_tb_local_padded_channels(C, prec) == -(-C // width) * width
    assert lib.wn_tb_local_padded_channels(80, 7) == 0
    x = torch.zeros(1, 3, 10, device="cuda")
    out = torch.empty(1, 2, 4, 10, 8, dtype=torch.bfloat16, device="cuda")
    assert lib.wn_tb_local_from_channels(x.data_ptr(), out.data_ptr(), 1, 3, 10, 7, None) != 0     # unknown precision
