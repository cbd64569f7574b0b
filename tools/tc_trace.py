#!/usr/bin/env python
"""Per-stage timeline of the tensor-core block kernel (CTA 0, first 512 stages of the last traced launch).
WN_TC_TRACE_PASS=A keeps the conv+gate launch of the last layer instead of its 1x1 launch."""
import ctypes, os, sys
os.environ["WN_TC_TRACE"] = "1"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "pytorch-wavenet_b200")):
    sys.path.insert(0, p)
import numpy as np, torch, bench, native
model = bench.build_model(bench.GEN_KW).cuda()
pass_a = os.environ.get("WN_TC_TRACE_PASS", "B")[0] == "A"
slabs = 32 if pass_a else 16                                       # K slabs per output tile (k*R/16 or D/16 at 256 channels)
idx = torch.randint(0, 256, (8, 16000), generator=torch.Generator().manual_seed(1)).to(torch.uint8).cuda()
with torch.no_grad():
    for _ in range(2):
        model.forward_indices(idx)
torch.cuda.synchronize()
buf = (ctypes.c_longlong * 4096)()
native.check(native.lib().wn_tc_read_trace(buf, 4096), "trace")
t = np.array(buf[:], dtype=np.int64).reshape(512, 8)
lo, hi = 2 * slabs, 2 * slabs * (400 // (2 * slabs))               # skip the pipeline fill, whole tiles only
t = t[lo:hi]
prod_wait = t[:, 1] - t[:, 0]
mma_wait = t[:, 3] - t[:, 2]
mma_issue = t[:, 4] - t[:, 3]
split_work = t[:, 6] - t[:, 5]
tma_to_full = t[:, 5] - t[:, 1]
split_to_mma = t[:, 3] - t[:, 6]
period = np.diff(t[:, 4])
pos = (np.arange(lo, hi)[1:]) % slabs
print(f"pass {'A (conv+gate)' if pass_a else 'B (1x1)'}: {slabs} slabs per tile")
print(f"stage period (MMA issue to MMA issue)     mean {period.mean():7.0f}  median {np.median(period):7.0f}")
print(f"  ... first slab of a tile (incl. waiting for a free accumulator)  mean {period[pos == 0].mean():7.0f}")
print(f"  ... other slabs                                                   mean {period[pos != 0].mean():7.0f}")
print(f"producer waiting for an empty stage       mean {prod_wait.mean():7.0f}")
print(f"TMA issue -> full barrier (load latency)  mean {tma_to_full.mean():7.0f}  median {np.median(tma_to_full):7.0f}")
print(f"splitter work incl. proxy fence           mean {split_work.mean():7.0f}")
print(f"splitter start-to-start                   mean {np.diff(t[:, 5]).mean():7.0f}")
print(f"splitter done -> MMA warp released        mean {split_to_mma.mean():7.0f}  median {np.median(split_to_mma):7.0f}")
print(f"splitter warp 9 done - warp 2 done        mean {(t[:, 7] - t[:, 6]).mean():7.0f}  median {np.median(t[:, 7] - t[:, 6]):7.0f}")
print(f"MMA warp waiting for operands             mean {mma_wait.mean():7.0f}")
print(f"MMA warp issuing (MMAs + commits)         mean {mma_issue.mean():7.0f}")
