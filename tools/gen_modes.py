#!/usr/bin/env python
"""Time the single-stream sampler kernels against each other on the bench net (cfg 2): samples/s per mode, and whether
the index streams agree.  usage: gen_modes.py [n_samples] [modes...]"""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-wavenet_b200")):
    sys.path.insert(0, p)
import numpy as np
import torch
import bench

n = int(sys.argv[1]) if len(sys.argv) > 1 else 4000
modes = [int(a) for a in sys.argv[2:]] or [3, 2]
model = bench.build_model(bench.GEN_KW).cuda()
rt = model._runtime()
ref = None
for mode in modes:
    rt.gen_mode = mode
    uni = np.random.RandomState(0).random_sample((1, n))
    first = np.array([[128]])
    best = None
    for rep in range(3):
        torch.cuda.synchronize()
        t0 = time.time()
        idx = model.generate_fast_batch(n, first, temperature=1.0, uniforms=uni, return_logits=False)
        torch.cuda.synchronize()
        dt = time.time() - t0
        best = dt if best is None else min(best, dt)
    idx = np.asarray(idx[0] if isinstance(idx, tuple) else idx)
    same = None if ref is None else bool(np.array_equal(idx, ref))
    if ref is None:
        ref = idx
    print(f"mode {mode}: {n / best:9.1f} samples/s  {best / n * 1e6:7.2f} us/sample  equal_to_first_mode={same}", flush=True)
