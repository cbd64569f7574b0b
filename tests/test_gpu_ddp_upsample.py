"""Batch-sharded training of a net with a learned local-conditioning upsampler on 2 GPUs (NCCL): the rank-averaged
gradients of the upsampler and of U (and every other gradient) equal the single-process gradients of the whole batch, while the gradient
of each rank's local condition series is its own shard of the whole-batch one.  Skipped on boxes with fewer than 2 GPUs."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from conftest import PKG, ROOT

pytestmark = pytest.mark.gpu
KW = dict(layers=4, blocks=2, dilation_channels=256, residual_channels=256, skip_channels=256, end_channels=256,
          classes=256, output_length=96, kernel_size=2, bias=True)
LOCAL = dict(local_condition_channels=5, local_condition_hop=40, local_condition_upsample_scales=(8, 5))


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _batch():
    g = torch.Generator().manual_seed(11)
    idx = torch.randint(0, 256, (4, 400), generator=g)
    tgt = torch.randint(0, 256, (4, KW["output_length"]), generator=g)
    y = torch.randn(4, 5, 10, generator=g)
    return idx, tgt, y


def _worker(rank, world, port, q):
    import sys
    for p in (ROOT, PKG):
        if p not in sys.path:
            sys.path.insert(0, p)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    try:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    except Exception as e:                                # report instead of leaving the parent waiting
        q.put((rank, repr(e), None, None))
        return
    try:
        import data_parallel as dp
        import wavenet_model as wmod
        torch.manual_seed(7 + rank)                       # replicas start different; make_data_parallel aligns them
        m = wmod.WaveNetModel(**KW, **LOCAL).cuda()
        dp.make_data_parallel(m)
        idx, tgt, y = _batch()
        mine, mine_t = dp.shard_batch(idx, rank, world).cuda(), dp.shard_batch(tgt, rank, world).cuda()
        my_y = dp.shard_batch(y, rank, world).cuda().requires_grad_(True)
        loss = F.cross_entropy(m.forward_indices(mine, local_condition=my_y), mine_t.reshape(-1))
        loss.backward()
        torch.cuda.synchronize()
        grads = {k: v.grad.detach().cpu() for k, v in m.named_parameters()}
        grads["local_condition"] = my_y.grad.detach().cpu()
        weights = {k: v.detach().cpu() for k, v in m.named_parameters()}
        q.put((rank, grads, weights, None))
    except Exception:
        import traceback
        q.put((rank, "worker failed: " + traceback.format_exc(), None, None))
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_rank_learned_upsampler_gradients_equal_single_process():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = {}
    for _ in range(2):
        r, grads, weights, _ = q.get(timeout=300)
        assert not isinstance(grads, str), grads
        res[r] = (grads, weights)
    for p in procs:
        p.join(timeout=60)
    g0, w0 = res[0]
    g1, w1 = res[1]
    assert any(k.startswith("local_upsample.") for k in w0)
    for k in w0:
        assert torch.equal(w0[k], w1[k]), k
        d = float((g0[k] - g1[k]).abs().max())
        assert d <= 1e-6 * max(float(g0[k].abs().max()), 1e-30), (k, d)     # the same averaged gradients on both ranks
    import data_parallel as dp
    import wavenet_model as wmod
    m = wmod.WaveNetModel(**KW, **LOCAL)
    m.load_state_dict(w0)
    m = m.cuda()
    idx, tgt, y = _batch()
    yg = y.cuda().requires_grad_(True)
    F.cross_entropy(m.forward_indices(idx.cuda(), local_condition=yg), tgt.cuda().reshape(-1)).backward()
    for k, v in m.named_parameters():
        ref = v.grad.cpu().numpy()
        err = np.abs(g0[k].numpy() - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err < 1e-4, (k, err)
    # dy is not reduced: rank r holds the gradient of its own shard, which is the whole-batch gradient scaled by the world
    # size (each rank's loss is a mean over half the batch)
    for r, (g, _) in res.items():
        ref = dp.shard_batch(yg.grad.cpu(), r, 2).numpy() * 2
        err = np.abs(g["local_condition"].numpy() - ref).max() / max(np.abs(ref).max(), 1e-30)
        assert err < 1e-4, (r, err)
