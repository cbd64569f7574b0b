"""Whole-call time of generate_fast_batch with and without the ring prefill (prefill=True): the cfg 2 net (10x5 layers,
256 channels, 256 classes, receptive field 5 116) at its random init, prompts of 1 000, 5 116, 16 000 and 160 000 samples,
1 000 generated samples at temperature 1 with fixed uniforms, 1 and 64 streams, on the default sampler kernel (6).  The
two variants alternate within each round; times are CUDA-event means over whole calls (host work, the prefill forward
and the sampler launch, ending in the call's own device-to-host read); the first prompt length of each stream count is
warmed up.  Prints one JSON line with the card and its power limit beside the numbers.

    python tools/prefill_bench.py [--samples 1000] [--steps 2] [--warmup 1] [--rounds 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "pytorch-wavenet_b200")]
import wavenet_model as wmod  # noqa: E402

KW = dict(layers=10, blocks=5, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
          classes=256, output_length=16, kernel_size=2, bias=False)
PROMPTS = (1000, 5116, 16000, 160000)


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
    ap.add_argument("--samples", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 64])
    ap.add_argument("--prompts", type=int, nargs="+", default=list(PROMPTS))
    args = ap.parse_args()
    torch.manual_seed(0)
    m = wmod.WaveNetModel(**KW).cuda()
    rng = np.random.RandomState(0)
    out = {}
    for ns in args.streams:
        uni = rng.random_sample((ns, args.samples))
        for g in args.prompts:
            first = rng.randint(0, 256, (ns, g))
            res = out.setdefault(f"{ns}_streams", {}).setdefault(f"prompt_{g}", {})
            for _ in range(args.rounds):
                for pf in (False, True):
                    ms = timed(lambda: m.generate_fast_batch(args.samples, first, temperature=1.0, uniforms=uni, prefill=pf),
                               args.steps, args.warmup if g == args.prompts[0] else 0)
                    res.setdefault("prefill_ms" if pf else "sequential_ms", []).append(round(ms, 2))
            res["speedup"] = round(min(res["sequential_ms"]) / min(res["prefill_ms"]), 2)
            print(ns, g, res, file=sys.stderr, flush=True)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    print(json.dumps(dict(tool="prefill_bench", gpu=torch.cuda.get_device_name(), nvidia_smi=q, samples=args.samples,
                          results=out)))


if __name__ == "__main__":
    main()
