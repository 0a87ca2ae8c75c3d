"""Multi-GPU training equivalence (SURVEY.md section 8c item 5, 8e): one process per GPU over NCCL, the batch sharded over
the ranks, ONE gradient all-reduce per step -- the averaged gradients must equal those of a single process on the concatenated
batch (every normalisation is a per-sample GroupNorm, the loss a mean over equal shards).  Also the reference's own mechanism,
single-process nn.DataParallel (tools/engine.py:63-64), on the same two GPUs.  Needs >= 2 GPUs; skipped on a single-GPU machine."""
import os
import socket
import types

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
needs2 = pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
ARGS = types.SimpleNamespace(corr_levels=3, base_scales=0.25, truncate_k=64)
N, ITERS = 512, 2


def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _clouds(b):
    g = torch.Generator().manual_seed(41)
    pc1 = 4.0 * torch.rand(b, N, 3, generator=g)
    pc2 = pc1 + 0.1 * torch.randn(b, N, 3, generator=g)
    return pc1, pc2


def _loss(flows, gt, gamma=0.8):
    n = len(flows)
    return sum(gamma ** (n - i - 1) * (flows[i] - gt).abs().sum(-1).mean() for i in range(n))


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from pvraft_b200 import RSF
    from pvraft_b200 import dist as D
    r, w, local = D.init_from_env(backend='nccl')
    dev = torch.device('cuda', local)
    torch.manual_seed(0)
    model = RSF(ARGS).to(dev).train()
    pc1, pc2 = _clouds(2 * world)
    lo, hi = D.shard_range(2 * world, r, w)
    a, b = pc1[lo:hi].to(dev), pc2[lo:hi].to(dev)
    wrapped = D.ddp(model, local)
    _loss(wrapped([a, b], num_iters=ITERS), b - a).backward()
    got = {k: p.grad.detach().cpu().clone() for k, p in model.named_parameters()}
    res = {'n_params': len(got)}
    if r == 0:
        model.zero_grad()
        fa, fb = pc1.to(dev), pc2.to(dev)
        _loss(model([fa, fb], num_iters=ITERS), fb - fa).backward()        # the concatenated batch on one GPU
        worst = 0.0
        for k, p in model.named_parameters():
            ref = p.grad.detach().cpu().double()
            worst = max(worst, float((got[k].double() - ref).norm() / ref.norm().clamp_min(1e-30)))
        res['worst_rel_l2'] = worst
    out[rank] = res
    dist.destroy_process_group()


@needs2
def test_two_rank_ddp_step_equals_single_process():
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), out), nprocs=world, join=True)
    assert out[0]['n_params'] == 95
    print('DDP (2 ranks, NCCL) vs single process, worst relative L2 over 95 gradients:', out[0]['worst_rel_l2'])
    assert out[0]['worst_rel_l2'] < 2e-3


@needs2
def test_data_parallel_like_the_reference_engine():
    """tools/engine.py:63-64 wraps the model in nn.DataParallel when several GPUs are visible: inference and a training step
    through that wrapper (replicas on other devices, one thread per replica) agree with the single-GPU model."""
    from pvraft_b200 import RSF
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    model = RSF(ARGS).to(dev)
    pc1, pc2 = [t.to(dev) for t in _clouds(4)]
    dp = torch.nn.DataParallel(model, device_ids=[0, 1])
    model.eval()
    with torch.no_grad():
        single = model([pc1, pc2], ITERS)[-1]
        multi = dp([pc1, pc2], ITERS)[-1]
    assert multi.shape == single.shape and float((multi - single).abs().mean()) < 1e-5 * float(single.abs().mean())
    model.train()
    model.zero_grad()
    _loss(model([pc1, pc2], num_iters=ITERS), pc2 - pc1).backward()
    ref = {k: p.grad.clone() for k, p in model.named_parameters()}
    model.zero_grad()
    _loss(dp([pc1, pc2], num_iters=ITERS), pc2 - pc1).backward()
    worst = max(float((p.grad - ref[k]).norm() / ref[k].norm().clamp_min(1e-30)) for k, p in model.named_parameters())
    print('nn.DataParallel step vs single GPU, worst relative L2:', worst)
    assert worst < 2e-3
