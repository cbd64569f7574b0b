"""Cost of top-k / nucleus truncation in the sampler: the cfg 2 net (10x5 layers, 256 channels, 256 classes), temperature 1,
at four settings -- off, top_k = 50, top_p = 0.95, both -- on the default kernel (6) at 1, 64 and 120 streams and on the
single-stream kernel 3.  Settings alternate within each round; times are CUDA-event means over whole generate_fast_batch
calls with fixed uniforms (µs per sample at 1 stream, µs per step of all streams otherwise).  Prints one JSON line with the
card and its power limit beside the numbers.

    python tools/truncation_bench.py [--samples 4000] [--steps 3] [--warmup 1] [--rounds 3]
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
import native  # noqa: E402
import wavenet_model as wmod  # noqa: E402

KW = dict(layers=10, blocks=5, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
          classes=256, output_length=16, kernel_size=2, bias=False)
SETTINGS = {"off": dict(top_k=0, top_p=1.0), "top_k=50": dict(top_k=50, top_p=1.0), "top_p=0.95": dict(top_k=0, top_p=0.95),
            "top_k=50,top_p=0.95": dict(top_k=50, top_p=0.95)}


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
    ap.add_argument("--samples", type=int, default=4000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    torch.manual_seed(0)
    m = wmod.WaveNetModel(**KW).cuda()
    n = args.samples
    rng = np.random.RandomState(0)
    out = {}
    for kernel, ns in (("default", 1), ("k3", 1), ("default", 64), ("default", 120)):
        first, uni = rng.randint(0, 256, (ns, 8)), rng.random_sample((ns, n))
        m._runtime().gen_mode = 3 if kernel == "k3" else None
        res = out.setdefault(f"{kernel}_{ns}_streams_us_per_{'sample' if ns == 1 else 'step'}", {})
        for _ in range(args.rounds):
            for name, kw in SETTINGS.items():
                ms = timed(lambda: m.generate_fast_batch(n, first, temperature=1.0, uniforms=uni, **kw), args.steps,
                           args.warmup)
                res.setdefault(name, []).append(round(1e3 * ms / n, 2))
        out[f"{kernel}_{ns}_streams_kernel_id"] = native.lib().wn_gen_kernel_id(m._runtime().sampler(ns)["handle"])
    m._runtime().gen_mode = None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    out["gpu"] = q
    print(json.dumps(out))


if __name__ == "__main__":
    main()
