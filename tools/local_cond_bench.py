"""Cost of local conditioning: unconditioned, global, local (C = 80, hop = 80) and global + local nets of the same shape,
timed with CUDA events.

    python tools/local_cond_bench.py [--steps 5] [--warmup 2] [--samples 4000]

Workloads (BASELINE.json shapes): the cfg 2 sampler (10x5 layers, 256 channels) with 1 and 64 streams, the cfg 3 training
forward and training step (B = 8, L = 16000), and the cfg 3 condition table build alone.  The global term has G = 16
labels, the local one a random (C, F) series per sequence / stream.  Prints one JSON line with the card and its power limit
beside the numbers.
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
G, C, HOP = 16, 80, 80


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
    args = ap.parse_args()
    out = {}
    for name, g, c in (("unconditioned", 0, 0), ("global", G, 0), ("local", 0, C), ("global_local", G, C)):
        hop = HOP if c else None
        torch.manual_seed(0)
        gen = wmod.WaveNetModel(**KW, output_length=1, condition_channels=g, local_condition_channels=c,
                                local_condition_hop=hop).cuda()
        res = {}
        for ns in (1, 64):
            first = np.random.RandomState(0).randint(0, 256, (ns, 8))
            kw = {}
            if g:
                kw["condition"] = np.arange(ns) % G
            if c:
                kw["local_condition"] = torch.randn(ns, c, -(-(7 + args.samples) // hop), device="cuda")
            ms = timed(lambda: gen.generate_fast_batch(args.samples, first, temperature=1.0, **kw), args.steps, args.warmup)
            res[f"gen_{ns}_streams_us_per_sample"] = 1e3 * ms / args.samples
        B, L = 8, 16000
        torch.manual_seed(0)
        m = wmod.WaveNetModel(**KW, output_length=L - gen.receptive_field + 1, condition_channels=g,
                              local_condition_channels=c, local_condition_hop=hop).cuda()
        idx = torch.randint(0, 256, (B, L), device="cuda")
        tgt = torch.randint(0, 256, (B * m.output_length,), device="cuda")
        kw = {}
        if g:
            kw["condition"] = torch.arange(B) % G
        if c:
            kw["local_condition"] = torch.randn(B, c, -(-L // hop), device="cuda")
        with torch.no_grad():
            res["cfg3_forward_ms"] = timed(lambda: m.forward_indices(idx, **kw), args.steps, args.warmup)

        def step():
            m.zero_grad(set_to_none=True)
            F.cross_entropy(m.forward_indices(idx, **kw), tgt).backward()
        res["cfg3_step_ms"] = timed(step, args.steps, args.warmup)
        if c:
            rt = m._runtime()
            stream = torch.cuda.current_stream().cuda_stream
            h = m._condition(kw.get("condition"), B)
            y = kw["local_condition"]
            W = rt.packed_weights(stream)
            res["cfg3_table_ms"] = timed(lambda: W.cond_table_frames(h, y, 0, y.shape[2], stream), args.steps, args.warmup)
        out[name] = res
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    out["gpu"] = q
    print(json.dumps(out))


if __name__ == "__main__":
    main()
