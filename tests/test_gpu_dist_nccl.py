"""FlatGradSync on NCCL (2 ranks, one GPU each): the gradient exchange of the data-parallel step -- blocking, and with the
bucketed all-reduces started from post-accumulate-grad hooks while backward is still running -- gives every rank the
mean gradient the reference's utils.sync_grads computes (utils.py:104-125), NaN / Inf handling included, and replicas
stay bit-identical through several optimiser steps. Needs 2 GPUs; skipped otherwise."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')]


def _net(device):
    torch.manual_seed(0)
    return torch.nn.Sequential(torch.nn.Conv2d(3, 32, 3, padding=1), torch.nn.LeakyReLU(0.2), torch.nn.Conv2d(32, 32, 3, padding=1),
                               torch.nn.LeakyReLU(0.2), torch.nn.Flatten(), torch.nn.Linear(32 * 16 * 16, 1)).to(device)


def _worker(rank, world, port, ret):
    sys.path.insert(0, os.path.join(ROOT, 'long-video-gan_b200'))
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    try:
        from lvg_dist.grad_sync import FlatGradSync
        out = {}
        for mode in ('reference', 'blocking', 'overlap'):
            net = _net(dev)
            opt = torch.optim.Adam(net.parameters(), lr=1e-3)
            sync = None
            if mode == 'blocking':
                sync = FlatGradSync(net)
            elif mode == 'overlap':
                sync = FlatGradSync(net, overlap=True, buckets=3, backwards_per_sync=2)
            gen = torch.Generator().manual_seed(100 + rank)
            poison = {'on': False}
            first = next(net.parameters())

            def spoil(g):          # a NaN born INSIDE backward on rank 0 (before the bucket leaves): must come out as 0 everywhere
                if poison['on']:
                    g = g.clone()
                    g.view(-1)[0] = float('nan') if rank == 0 else 1.0
                return g
            first.register_hook(spoil)
            for it in range(3):
                xa, xb = torch.randn(4, 3, 16, 16, generator=gen).to(dev), torch.randn(4, 3, 16, 16, generator=gen).to(dev)
                poison['on'] = it == 1
                net(xa).square().mean().backward()          # two backward passes per update, as update_D does
                net(xb).tanh().mean().backward()
                if mode == 'reference':                      # utils.py:116-124 restated on NCCL
                    ps = [p for p in net.parameters() if p.grad is not None]
                    flat = torch.cat([p.grad.flatten() for p in ps])
                    dist.all_reduce(flat)
                    flat = flat / world * 0.5
                    torch.nan_to_num(flat, nan=0, posinf=1e5, neginf=-1e5, out=flat)
                    for p, g in zip(ps, flat.split([p.numel() for p in ps])):
                        p.grad = g.reshape(p.shape)
                else:
                    sync.sync(gain=0.5)
                opt.step()
                if sync is not None:
                    sync.zero_grad()
                else:
                    opt.zero_grad(set_to_none=True)
            out[mode] = torch.cat([p.detach().flatten() for p in net.parameters()]).cpu()
        ret[rank] = out
    finally:
        dist.destroy_process_group()


def test_flat_grad_sync_on_nccl_two_ranks():
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, 29700 + os.getpid() % 1000, ret), nprocs=world, join=True)
    for mode in ('blocking', 'overlap'):
        for r in range(world):
            # NCCL's reduction order differs from cat-all_reduce-split only in fp32 rounding
            assert torch.allclose(ret[r][mode], ret[r]['reference'], rtol=1e-4, atol=1e-6), mode
        assert torch.equal(ret[0][mode], ret[1][mode]), f'{mode}: replicas diverged'
    assert torch.isfinite(ret[0]['overlap']).all()
