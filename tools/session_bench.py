"""Continuous batching against static batches on the cfg-2 net (50 layers of 256 channels, receptive field 5 116).

A seeded workload of --jobs jobs (prompts of 1 to 16 000 samples, 500 to 8 000 samples each, temperature 0 or 0.7-1.3, top-k
/ top-p on a third of them, a regularizer on a quarter) is served two ways, and the kept rate (samples the jobs asked for,
per second of wall time, host work included) is reported for each:
  - a sampling session of 64 slots (and one of 120) with prefill=True, stepping 200 to 1 000 evaluations at a time (seeded);
  - the same jobs in FIFO static batches of 64 through generate_fast_batch(prefill=True), each batch lasting as long as its
    longest job.
It also reports the wall time of one seat (the prefill forward of a 16 000-sample prompt plus the ring scatter) and of a
1-evaluation step of a full 64-slot session (host work per step plus one evaluation).  Prints one JSON line, with the
card's name and power limit read in the same run."""
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


def workload(n_jobs, seed):
    rng = np.random.RandomState(seed)
    jobs = []
    for _ in range(n_jobs):
        g = int(np.exp(rng.uniform(0, np.log(16000))))
        n = int(rng.randint(500, 8001))
        t = 0.0 if rng.rand() < 0.25 else float(rng.uniform(0.7, 1.3))
        k, p = (int(rng.choice([0, 40])), float(rng.choice([1.0, 0.9]))) if rng.rand() < 1 / 3 else (0, 1.0)
        r = 1e-4 if rng.rand() < 0.25 else 0.0
        jobs.append(dict(first=rng.randint(0, 256, max(g, 1)), n=n, temperature=t, regularize=r, top_k=k, top_p=p,
                         uniforms=rng.random_sample(n)))
    return jobs


def sync():
    torch.cuda.synchronize()


def serve_session(m, jobs, slots, seed):
    rng = np.random.RandomState(seed)
    sess = m.sampling_session(slots, prefill=True)
    sync()
    t0 = time.perf_counter()
    for j in jobs:
        sess.submit(j["first"], j["n"], temperature=j["temperature"], regularize=j["regularize"], top_k=j["top_k"],
                    top_p=j["top_p"], uniforms=j["uniforms"])
    steps = 0
    while sess.pending or sess.active:
        sess.step(int(rng.randint(200, 1001)))
        steps += 1
    sync()
    return time.perf_counter() - t0, steps


def serve_static(m, jobs, batch):
    sync()
    t0 = time.perf_counter()
    for i in range(0, len(jobs), batch):
        b = jobs[i:i + batch]
        m.generate_fast_batch([j["n"] for j in b], [j["first"] for j in b], temperature=[j["temperature"] for j in b],
                              regularize=[j["regularize"] for j in b], top_k=[j["top_k"] for j in b],
                              top_p=[j["top_p"] for j in b], uniforms=[j["uniforms"] for j in b], prefill=True)
    sync()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=256)
    ap.add_argument("--seed", type=int, default=2026)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("session_bench: needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    torch.manual_seed(0)
    m = W.WaveNetModel(**CFG2).cuda()
    jobs = workload(args.jobs, args.seed)
    kept = sum(j["n"] for j in jobs)
    # warm-up: every path once on a few short jobs
    warm = workload(4, 1)
    for j in warm:
        j["n"] = 300
        j["first"] = j["first"][:600]
    serve_session(m, warm, 64, 0)
    serve_static(m, warm, 64)
    out = dict(card=card, jobs=len(jobs), kept_samples=kept)
    for slots in (64, 120):
        wall, steps = serve_session(m, jobs, slots, args.seed + slots)
        out[f"session{slots}_samples_per_s"] = round(kept / wall)
        out[f"session{slots}_wall_s"] = round(wall, 3)
        out[f"session{slots}_steps"] = steps
    wall = serve_static(m, jobs, 64)
    out["static64_samples_per_s"] = round(kept / wall)
    out["static64_wall_s"] = round(wall, 3)
    # one seat: the prefill forward of a 16 000-sample prompt plus the scatter into one slot
    sess = m.sampling_session(64, prefill=True)
    sess.step(1)                                    # parks every slot
    stream = torch.cuda.current_stream().cuda_stream
    seat_ms = []
    for r in range(6):
        sess.submit(np.random.RandomState(r).randint(0, 256, 16000), 1, temperature=0.0)
        job = sess.queue.pop(0)
        sync()
        t0 = time.perf_counter()
        sess._seat([(r, job)], stream)
        sync()
        seat_ms.append((time.perf_counter() - t0) * 1e3)
        sess.slot_job[r] = None
    out["seat_16000_prompt_ms"] = round(float(np.median(seat_ms[1:])), 3)
    # a full 64-slot session stepping one evaluation at a time
    sess = m.sampling_session(64)
    for r in range(64):
        sess.submit([r], 10 ** 6, temperature=1.0, uniforms=np.zeros(10 ** 6))
    sess.step(1)
    step_ms = []
    for _ in range(50):
        t0 = time.perf_counter()
        sess.step(1)
        step_ms.append((time.perf_counter() - t0) * 1e3)
    out["step1_64_slots_ms"] = round(float(np.median(step_ms)), 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
