"""Continuous batching of a vocoder-shaped workload: locally conditioned sessions against static batches on the cfg-2 net
(50 layers of 256 channels) with an 80-channel local condition at hop 80, repeated ("repeat") or through the learned
(4, 4, 5) upsampler ("learned").

A seeded workload of --jobs jobs (1-sample prompts, 0.5 to 4 s at 16 kHz = 8 000 to 64 000 samples each, temperature 1,
each with its own (80, ceil(n / 80)) frame series) is served three ways per model, and the kept rate (samples the jobs
asked for, per second of wall time, host work included) is reported for each:
  - sampling sessions of 64 and 120 slots (local_window 1 000 for repeat, 64 for learned), stepping 200 to 1 000
    evaluations at a time (seeded), with the share of wall time spent gathering and building the condition tables;
  - the same jobs in FIFO per-stream static batches of 64 through generate_fast_batch with a list of series, each batch
    lasting as long as its longest job.
Prints one JSON line, with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "pytorch-wavenet_b200"))
import wavenet_model as W  # noqa: E402

CFG2 = dict(layers=10, blocks=5, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
            classes=256, output_length=16, kernel_size=2, bias=False)
WINDOW = {"repeat": 1000, "learned": 64}


def model(kind):
    torch.manual_seed(0)
    kw = dict(CFG2, local_condition_channels=80, local_condition_hop=80)
    if kind == "learned":
        kw["local_condition_upsample_scales"] = (4, 4, 5)
    return W.WaveNetModel(**kw).cuda()


def workload(n_jobs, seed):
    rng = np.random.RandomState(seed)
    jobs = []
    for _ in range(n_jobs):
        n = int(rng.randint(8000, 64001))
        jobs.append(dict(first=rng.randint(0, 256, 1), n=n, uniforms=rng.random_sample(n),
                         y=rng.randn(80, -(-n // 80)).astype(np.float32)))
    return jobs


def sync():
    torch.cuda.synchronize()


def serve_session(m, jobs, slots, window, seed):
    rng = np.random.RandomState(seed)
    sess = m.sampling_session(slots, local_window=window)
    build = [0.0]
    set_windows = sess._set_windows

    def timed(frame0, stream):                     # launches synchronise anyway: the table build is timed alone
        sync()
        t = time.perf_counter()
        set_windows(frame0, stream)
        sync()
        build[0] += time.perf_counter() - t
    sess._set_windows = timed
    sync()
    t0 = time.perf_counter()
    for j in jobs:
        sess.submit(j["first"], j["n"], temperature=1.0, uniforms=j["uniforms"], local_condition=j["y"])
    steps = 0
    while sess.pending or sess.active:
        sess.step(int(rng.randint(200, 1001)))
        steps += 1
    sync()
    return time.perf_counter() - t0, steps, build[0]


def serve_static(m, jobs, batch):
    sync()
    t0 = time.perf_counter()
    for i in range(0, len(jobs), batch):
        b = jobs[i:i + batch]
        m.generate_fast_batch([j["n"] for j in b], [j["first"] for j in b], temperature=1.0,
                              uniforms=[j["uniforms"] for j in b], local_condition=[j["y"] for j in b])
    sync()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=256)
    ap.add_argument("--seed", type=int, default=2026)
    ap.add_argument("--kinds", default="repeat,learned")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("session_local_bench: needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    jobs = workload(args.jobs, args.seed)
    kept = sum(j["n"] for j in jobs)
    out = dict(card=card, jobs=len(jobs), kept_samples=kept)
    for kind in args.kinds.split(","):
        m = model(kind)
        warm = workload(4, 1)                       # warm-up: every path once on a few short jobs
        for j in warm:
            j["n"] = 300
            j["y"] = j["y"][:, :4]
            j["uniforms"] = j["uniforms"][:300]
        serve_session(m, warm, 64, WINDOW[kind], 0)
        serve_static(m, warm, 64)
        for slots in (64, 120):
            wall, steps, build = serve_session(m, jobs, slots, WINDOW[kind], args.seed + slots)
            out[f"{kind}_session{slots}_samples_per_s"] = round(kept / wall)
            out[f"{kind}_session{slots}_wall_s"] = round(wall, 3)
            out[f"{kind}_session{slots}_steps"] = steps
            out[f"{kind}_session{slots}_table_share"] = round(build / wall, 4)
        wall = serve_static(m, jobs, 64)
        out[f"{kind}_static64_samples_per_s"] = round(kept / wall)
        out[f"{kind}_static64_wall_s"] = round(wall, 3)
        del m
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
