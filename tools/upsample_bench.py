"""Cost of the learned local-conditioning upsampler: cfg 3 training forward and step (B = 8, L = 16000, 10x5 layers of 256
channels, C = 80) for an unconditioned net, repeat upsampling at hop 80, the learned (4, 4, 5) upsampler on the K-slab path,
and the explicit hop-1 twin that reads an audio-rate condition table (its OOM is reported); the cfg 2 sampler at 1 and 64
streams, learned against repeat; and the upsampler alone.  Variants alternate within one run; times are CUDA-event means,
peak memory is torch's peak allocation.  Prints one JSON line with the card and its power limit beside the numbers.

    python tools/upsample_bench.py [--steps 5] [--warmup 2] [--samples 4000]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-wavenet_b200")]
import wavenet_model as wmod  # noqa: E402

KW = dict(layers=10, blocks=5, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
          classes=256, kernel_size=2, bias=True)
C, HOP, SCALES = 80, 80, (4, 4, 5)
VARIANTS = {"unconditioned": {}, "repeat": dict(local_condition_channels=C, local_condition_hop=HOP),
            "learned": dict(local_condition_channels=C, local_condition_hop=HOP, local_condition_upsample_scales=SCALES),
            "hop1_twin": dict(local_condition_channels=C, local_condition_hop=1)}


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--samples", type=int, default=4000)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    B, L = 8, 16000
    out = {}
    models = {}
    for name, kw in VARIANTS.items():
        torch.manual_seed(0)
        models[name] = wmod.WaveNetModel(**KW, output_length=L - 5116 + 1, **kw).cuda()
    g = torch.Generator(device="cuda").manual_seed(1)
    idx = torch.randint(0, 256, (B, L), device="cuda", generator=g)
    tgt = torch.randint(0, 256, (B * (L - 5116 + 1),), device="cuda", generator=g)
    y = torch.randn(B, C, L // HOP, device="cuda", generator=g)
    with torch.no_grad():
        c = models["learned"]._upsample(y, L)
    inputs = {"unconditioned": {}, "repeat": dict(local_condition=y), "learned": dict(local_condition=y),
              "hop1_twin": dict(local_condition=c)}
    for rnd in range(args.rounds):                                   # variants alternate within each round
        for name, m in models.items():
            res = out.setdefault(name, {})
            kw = inputs[name]
            try:
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats()
                with torch.no_grad():
                    res.setdefault("cfg3_forward_ms", []).append(timed(lambda: m.forward_indices(idx, **kw), args.steps, args.warmup))
                res.setdefault("cfg3_forward_peak_gb", []).append(torch.cuda.max_memory_allocated() / 2 ** 30)
                torch.cuda.reset_peak_memory_stats()

                def step():
                    m.zero_grad(set_to_none=True)
                    F.cross_entropy(m.forward_indices(idx, **kw), tgt).backward()
                res.setdefault("cfg3_step_ms", []).append(timed(step, args.steps, args.warmup))
                res.setdefault("cfg3_step_peak_gb", []).append(torch.cuda.max_memory_allocated() / 2 ** 30)
            except torch.OutOfMemoryError as e:
                res["oom"] = str(e).splitlines()[0]
                m.zero_grad(set_to_none=True)
            torch.cuda.empty_cache()
    with torch.no_grad():
        up = models["learned"]
        out["upsampler_alone_ms"] = timed(lambda: up._upsample(y, L), args.steps * 4, args.warmup)
    for name in ("repeat", "learned"):
        torch.manual_seed(0)
        gen = wmod.WaveNetModel(**KW, output_length=1, **VARIANTS[name]).cuda()
        for ns in (1, 64):
            first = np.random.RandomState(0).randint(0, 256, (ns, 8))
            yy = torch.randn(ns, C, -(-(7 + args.samples) // HOP), device="cuda")
            ms = timed(lambda: gen.generate_fast_batch(args.samples, first, temperature=1.0, local_condition=yy),
                       args.steps, args.warmup)
            out.setdefault(f"gen_{name}", {})[f"{ns}_streams_us_per_sample"] = 1e3 * ms / args.samples
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    out["gpu"] = q
    print(json.dumps(out))


if __name__ == "__main__":
    main()
