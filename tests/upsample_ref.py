"""Float64 reference of a net with a learned local-conditioning upsampler: every stage is conv_transpose1d(stride s, kernel
2s) cropped to [s // 2, s // 2 + F s), and the audio-rate result c conditions the stack as local_ref does at hop 1."""
import torch.nn.functional as F

import local_ref


def upsample(p, scales, y):
    """(N, C, F) -> (N, C, F * prod(scales)) with the upsampler weights local_upsample.{j}.weight / bias of ``p``."""
    c = y
    for j, s in enumerate(scales):
        n = c.shape[2]
        c = F.conv_transpose1d(c, p[f"local_upsample.{j}.weight"], p[f"local_upsample.{j}.bias"], stride=s)
        c = c[:, :, s // 2:s // 2 + n * s]
    return c


def stack_direct(p, spec, x, y, scales, h=None, taps=None):
    c = upsample(p, scales, y)[:, :, :x.size(2)]
    return local_ref.stack_direct(p, spec, x, c, 1, h, taps)


def forward(p, spec, x, y, scales, h=None):
    """WaveNetModel.forward of the net: (N * output_length, classes)."""
    out = stack_direct(p, spec, x, y, scales, h)
    n, c, _ = out.shape
    l = spec.output_length
    return out[:, :, -l:].transpose(1, 2).contiguous().view(n * l, c)
