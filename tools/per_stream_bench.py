"""Cost of per-stream sampling settings (generate_fast_batch with per-stream prompts, counts and settings): the cfg 2 net
(10x5 layers, 256 channels, 256 classes), 2 000 samples per stream at temperature 1, on the default kernel (6) at 1, 64
and 120 streams.  Four calls per stream count, alternated within each round:
  scalar   -- today's call: one prompt length, one setting for every stream;
  arrays   -- the same values passed as per-stream arrays (the per-stream path with uniform settings);
  mixed    -- every stream its own temperature (0 or 0.6-1.4), regularizer (0 or 1e-4), top_k (0, 50) and top_p (1, 0.95);
  ragged   -- the scalar settings with prompts of 1 to 1 000 samples: the launch runs until the longest prompt's stream
              is done, so it is also reported as samples per second of the kept samples only.
Times are CUDA-event means over whole calls with fixed uniforms, as µs per evaluation step of all streams.  Prints one
JSON line with the card and its power limit beside the numbers.

    python tools/per_stream_bench.py [--samples 2000] [--steps 3] [--warmup 1] [--rounds 3]
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


def calls(m, ns, n, rng):
    """name -> (call, evaluations per call, kept samples per call)"""
    first = rng.randint(0, 256, (ns, 8))
    uni = rng.random_sample((ns, n))
    mixed = dict(temperature=np.where(np.arange(ns) % 4 == 3, 0.0, rng.uniform(0.6, 1.4, ns)),
                 regularize=np.where(np.arange(ns) % 2 == 1, 1e-4, 0.0), top_k=np.where(np.arange(ns) % 3 == 1, 50, 0),
                 top_p=np.where(np.arange(ns) % 3 == 2, 0.95, 1.0))
    ragged = [rng.randint(0, 256, g) for g in rng.randint(1, 1001, ns)]
    evals = 7 + n
    ragged_evals = max(len(r) for r in ragged) - 1 + n
    return {
        "scalar": (lambda: m.generate_fast_batch(n, first, temperature=1.0, uniforms=uni), evals, ns * n),
        "arrays": (lambda: m.generate_fast_batch([n] * ns, first, temperature=[1.0] * ns, regularize=[0.0] * ns,
                                                 top_k=[0] * ns, top_p=[1.0] * ns, uniforms=uni), evals, ns * n),
        "mixed": (lambda: m.generate_fast_batch(n, first, uniforms=uni, **mixed), evals, ns * n),
        "ragged": (lambda: m.generate_fast_batch(n, ragged, temperature=[1.0] * ns, uniforms=uni), ragged_evals, ns * n),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    torch.manual_seed(0)
    m = wmod.WaveNetModel(**KW).cuda()
    rng = np.random.RandomState(0)
    out = {}
    for ns in (1, 64, 120):
        res = out.setdefault(f"{ns}_streams", {})
        for _ in range(args.rounds):
            for name, (fn, evals, kept) in calls(m, ns, args.samples, rng).items():
                ms = timed(fn, args.steps, args.warmup)
                res.setdefault(f"{name}_us_per_step", []).append(round(1e3 * ms / evals, 2))
                if name == "ragged":
                    res.setdefault("ragged_evaluations", []).append(evals)
                    res.setdefault("ragged_kept_samples_per_s", []).append(round(kept / (ms * 1e-3)))
                    res.setdefault("scalar_kept_samples_per_s", []).append(
                        round(ns * args.samples / (res["scalar_us_per_step"][-1] * 1e-6 * (7 + args.samples))))
        res["kernel_id"] = native.lib().wn_gen_kernel_id(m._runtime().sampler(ns)["handle"])
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    out["gpu"] = q
    print(json.dumps(out))


if __name__ == "__main__":
    main()
