#!/usr/bin/env python
"""Write tiny_snapshot.pt: a whole-object pickle of a small WaveNetModel of the UNMODIFIED reference, saved the way
the reference's trainer saves snapshots (torch.save(self.model, path), reference wavenet_training.py:88), plus
tiny_snapshot_io.npz (its seeded weights' forward on a fixed one-hot input, computed by the reference).

Run on the CPU with the reference checkout at REF (it imports the reference sources from there; nothing is copied):
    python tests/golden/make_tiny_snapshot.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import import_reference, indices, one_hot  # noqa: E402

KW = dict(layers=3, blocks=2, dilation_channels=16, residual_channels=16, skip_channels=32, end_channels=32,
          classes=256, output_length=8, kernel_size=2, bias=True)


def main():
    _, wmod = import_reference()
    torch.set_num_threads(8)
    torch.manual_seed(0)
    model = wmod.WaveNetModel(**KW)
    idx = indices(1, model.receptive_field + KW["output_length"] - 1, seed=4321)
    with torch.no_grad():
        y = model(one_hot(idx))
    torch.save(model, os.path.join(HERE, "tiny_snapshot.pt"))
    np.savez(os.path.join(HERE, "tiny_snapshot_io.npz"), idx=idx.numpy(), fwd=y.numpy(),
             receptive_field=np.int64(model.receptive_field))
    print("tiny snapshot:", os.path.getsize(os.path.join(HERE, "tiny_snapshot.pt")), "bytes, receptive field",
          model.receptive_field, "forward", tuple(y.shape))


if __name__ == "__main__":
    main()
