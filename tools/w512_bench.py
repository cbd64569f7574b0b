"""Sampling the cfg-5 shape (80 layers of 512 channels, skip and end 512, 256 classes) on a random-init net.

  - which sampler kernel wn_gen_create / wn_gen_kernel_id give at 1, 8, 33, 36 and 64 streams (or the error code);
  - microseconds per evaluation step (T = 1: every evaluation samples, temperature 1) of kernel 6 at --streams, and of
    kernel 2 at the stream counts it supports (--k2-streams), each over a timed window of --evals evaluations after a
    warm-up launch, host clock around launches that end in a device synchronise;
  - the weight-streaming figure of kernel 6: the bytes of its weight images read per step (all clusters share one copy
    when their L2 reads coincide) over the step time, against the 3.35 TB/s of the H100 SXM data sheet (a derived bound,
    not a measurement).
Prints one JSON line with the card's name, power limit and SM clock read in the same run.
--lib PATH loads another build of the library (e.g. the parent commit's) for the kernel-choice table."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pytorch-wavenet_b200"))
import native  # noqa: E402

CFG5 = dict(layers=10, blocks=8, dilation_channels=512, residual_channels=512, skip_channels=512, end_channels=512,
            classes=256, output_length=16, kernel_size=2, bias=False)
HBM_BPS = 3.35e12                                     # H100 SXM data sheet


def image_bytes(n_layers, width):
    """kernel 6's weight images: 3 kinds x (W/16)^2 x 2 KB per layer, end_conv_1 (W/16)^2 KB, end_conv_2 16 x W/16 KB"""
    nvr = width // 16
    return 1024 * (6 * nvr * nvr * n_layers + nvr * nvr + 16 * nvr)


def kernel_table(m, counts):
    rt = m._runtime()
    out = {}
    for ns in counts:
        try:
            s = rt.new_sampler(ns)
        except RuntimeError as e:
            out[ns] = {"create": str(e).split("code ")[1].split(")")[0] if "code " in str(e) else str(e)}
            continue
        out[ns] = {"create": 0, "kernel": native.lib().wn_gen_kernel_id(s["handle"])}
        native.lib().wn_gen_destroy(s["handle"])
        del s
        torch.cuda.empty_cache()
    return out


def time_steps(m, mode, ns, n_evals):
    rt = m._runtime()
    rt.gen_mode = mode
    rng = np.random.RandomState(ns)
    first = rng.randint(0, 256, (ns, 1))
    m.generate_fast_batch(16, first, temperature=1.0, uniforms=rng.random_sample((ns, 16)))       # warm-up, handle
    uni = rng.random_sample((ns, n_evals))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    m.generate_fast_batch(n_evals, first, temperature=1.0, uniforms=uni)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    h = rt.samplers[ns]["handle"]
    kid = native.lib().wn_gen_kernel_id(h)
    native.lib().wn_gen_destroy(rt.samplers.pop(ns)["handle"])
    torch.cuda.empty_cache()
    rt.gen_mode = None
    return kid, dt / n_evals * 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 8, 64, 120])
    ap.add_argument("--k2-streams", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--evals", type=int, default=4000)
    ap.add_argument("--k2-evals", type=int, default=1000)
    ap.add_argument("--lib", help="library to load instead of the package's build")
    ap.add_argument("--table-only", action="store_true")
    args = ap.parse_args()
    if args.lib:
        native.LIB_PATH = os.path.abspath(args.lib)
    import wavenet_model as W
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    torch.manual_seed(0)
    m = W.WaveNetModel(**CFG5).cuda()
    res = {"card": q[0] if q else "unknown", "lib": args.lib or "package build",
           "create": kernel_table(m, (1, 8, 33, 36, 64))}
    if not args.table_only:
        nb = image_bytes(CFG5["layers"] * CFG5["blocks"], 512)
        rows = []
        for ns in args.streams:
            kid, us = time_steps(m, None, ns, args.evals)
            rows.append({"kernel": kid, "streams": ns, "us_per_step": round(us, 1),
                         "samples_per_s": round(ns / us * 1e6), "image_bytes_per_s": nb / (us * 1e-6),
                         "of_3.35TB/s": round(nb / (us * 1e-6) / HBM_BPS, 3)})
        for ns in args.k2_streams:
            kid, us = time_steps(m, 2, ns, args.k2_evals)
            rows.append({"kernel": kid, "streams": ns, "us_per_step": round(us, 1), "samples_per_s": round(ns / us * 1e6)})
        res.update(image_bytes=nb, min_us_at_3_35TBps=round(nb / HBM_BPS * 1e6, 1), rows=rows)
        q2 = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True,
                            text=True).stdout.strip()
        res["sm_clock_after"] = q2
    print(json.dumps(res))


if __name__ == "__main__":
    main()
