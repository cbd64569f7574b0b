"""Float64 reference of a locally (and optionally globally) conditioned net: oracle.stack_direct with the condition terms.

Local conditioning with repeat upsampling adds Uf y[:, t // hop] / Ug y[:, t // hop] to the filter / gate pre-activations
of position t (the absolute input position, the same axis as the output position t that predicts sample t + 1); global
conditioning adds Vf h / Vg h.  Everything else is oracle.stack_direct line for line, so with U = 0 (and no global term)
the result is stack_direct's bit for bit."""
import math

import torch
import torch.nn.functional as F

from oracle.wavenet_oracle import _b


def upsample(y, hop, L):
    """(N, C, F) frame-rate series -> (N, C, L) at the sample rate: position t takes frame t // hop."""
    return y.repeat_interleave(hop, dim=2)[:, :, :L]


def stack_direct(p, spec, x, y=None, hop=None, h=None, taps=None):
    """oracle.stack_direct plus the local term of the (N, C, F) series ``y`` at ``hop`` and the global term of the (N, G)
    rows ``h``; p holds filter_local_convs.{i}.weight / gate_local_convs.{i}.weight (and *_cond_convs for h).  ``taps``
    (a dict) receives the input of the first head ReLU ("skip")."""
    k = spec.kernel_size
    L = x.size(2)
    yu = None if y is None else upsample(y, hop, L)
    hh = None if h is None else h[:, :, None]
    hs = x
    hs = F.conv1d(hs, p["start_conv.weight"], _b(p, "start_conv"))
    skip = None
    for i, (d, _) in enumerate(spec.dilation_schedule()):
        T = hs.size(2)
        T_pad = int(math.ceil(T / d) * d)
        hp = F.pad(hs, (T_pad - T, 0))
        pf = F.conv1d(hp, p[f"filter_convs.{i}.weight"], _b(p, f"filter_convs.{i}"), dilation=d)
        pg = F.conv1d(hp, p[f"gate_convs.{i}.weight"], _b(p, f"gate_convs.{i}"), dilation=d)
        To = pf.size(2)
        if hh is not None:
            pf = pf + F.conv1d(hh, p[f"filter_cond_convs.{i}.weight"])
            pg = pg + F.conv1d(hh, p[f"gate_cond_convs.{i}.weight"])
        if yu is not None:
            pf = pf + F.conv1d(yu[:, :, L - To:], p[f"filter_local_convs.{i}.weight"])
            pg = pg + F.conv1d(yu[:, :, L - To:], p[f"gate_local_convs.{i}.weight"])
        z = torch.tanh(pf) * torch.sigmoid(pg)
        s = F.conv1d(z, p[f"skip_convs.{i}.weight"], _b(p, f"skip_convs.{i}"))
        skip = s if skip is None else s + skip[:, :, -s.size(2):]
        hs = F.conv1d(z, p[f"residual_convs.{i}.weight"], _b(p, f"residual_convs.{i}")) + hp[:, :, d * (k - 1):]
    if taps is not None:
        taps["skip"] = skip
    y1 = F.relu(skip)
    y1 = F.relu(F.conv1d(y1, p["end_conv_1.weight"], p["end_conv_1.bias"]))
    return F.conv1d(y1, p["end_conv_2.weight"], p["end_conv_2.bias"])


def forward(p, spec, x, y=None, hop=None, h=None):
    """WaveNetModel.forward of the conditioned net: (N * output_length, classes)."""
    out = stack_direct(p, spec, x, y, hop, h)
    n, c, _ = out.shape
    l = spec.output_length
    return out[:, :, -l:].transpose(1, 2).contiguous().view(n * l, c)


def folded(p, spec, yf=None, hb=None):
    """Unconditioned parameters of ONE sequence at ONE frame: the local term of frame vector ``yf`` (C,) and the global
    term of ``hb`` (G,) folded into the filter / gate biases."""
    q = {k: v for k, v in p.items() if "_local_convs." not in k and "_cond_convs." not in k}
    for i in range(spec.layers * spec.blocks):
        for conv, lc, gc in (("filter_convs", "filter_local_convs", "filter_cond_convs"),
                             ("gate_convs", "gate_local_convs", "gate_cond_convs")):
            base = p.get(f"{conv}.{i}.bias")
            shift = 0
            if yf is not None:
                shift = shift + p[f"{lc}.{i}.weight"][:, :, 0] @ yf.to(p[f"{lc}.{i}.weight"].dtype)
            if hb is not None:
                shift = shift + p[f"{gc}.{i}.weight"][:, :, 0] @ hb.to(p[f"{gc}.{i}.weight"].dtype)
            q[f"{conv}.{i}.bias"] = shift if base is None else base + shift
    return q
