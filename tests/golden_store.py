"""Golden fixtures on disk: one ``<name>.npz``, or, for a fixture larger than ``SHARD_BYTES``, the shards
``<stem>.part<i>.npz`` that together hold its arrays (an array larger than a shard is stored in row blocks
``<key>@<j>`` along axis 0).  No file of the repository exceeds 1 MB this way; the arrays come back bit-identical."""
import glob
import os

import numpy as np

SHARD_BYTES = 900_000


class Golden(dict):
    """The arrays of one fixture; ``files`` lists the keys like ``numpy.lib.npyio.NpzFile``."""

    @property
    def files(self):
        return list(self.keys())


def save(path, arrays, compressed=False):
    """Write ``arrays`` to ``path`` (``<stem>.npz``), sharding when they exceed SHARD_BYTES."""
    write = np.savez_compressed if compressed else np.savez
    stem = path[:-4] if path.endswith(".npz") else path
    for old in glob.glob(stem + ".part*.npz"):
        os.remove(old)
    arrays = {k: np.asarray(v) for k, v in arrays.items()}
    if sum(a.nbytes for a in arrays.values()) <= SHARD_BYTES:
        write(stem + ".npz", **arrays)
        return
    if os.path.exists(stem + ".npz"):
        os.remove(stem + ".npz")
    pieces = []
    for k, a in arrays.items():
        if a.nbytes <= SHARD_BYTES:
            pieces.append((k, a))
        else:
            rows = max(1, SHARD_BYTES // max(1, a.nbytes // a.shape[0]))
            pieces += [(f"{k}@{j}", a[i:i + rows]) for j, i in enumerate(range(0, a.shape[0], rows))]
    shard, size, n = {}, 0, 0
    for k, a in pieces:
        if shard and size + a.nbytes > SHARD_BYTES:
            write(f"{stem}.part{n}.npz", **shard)
            shard, size, n = {}, 0, n + 1
        shard[k], size = a, size + a.nbytes
    write(f"{stem}.part{n}.npz", **shard)


def load(path):
    """Read a fixture written by ``save`` (or any plain ``.npz``)."""
    stem = path[:-4] if path.endswith(".npz") else path
    files = [stem + ".npz"] if os.path.exists(stem + ".npz") else \
        sorted(glob.glob(stem + ".part*.npz"), key=lambda f: int(f[len(stem) + 5:-4]))
    if not files:
        raise FileNotFoundError(path)
    out, blocks = Golden(), {}
    for f in files:
        with np.load(f, allow_pickle=False) as z:
            for k in z.files:
                if "@" in k:
                    base, j = k.rsplit("@", 1)
                    blocks.setdefault(base, {})[int(j)] = z[k]
                else:
                    out[k] = z[k]
    for k, parts in blocks.items():
        out[k] = np.concatenate([parts[j] for j in sorted(parts)], axis=0)
    return out
