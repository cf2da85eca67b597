"""Helper of test_gblock_tail_host.py / test_gpu_gblock_tail.py (run as a subprocess): the UNMODIFIED reference low-res
generator (staged at oracle/_ref/src) with torch_utils.ops.gblock_tail.

  cpu      every block of the default G, of a 64 x 64 G and of standalone blocks with odd crops: the reference forward
           against block_forward (the tail through the torch composition) at magnitude-EMA beta 1 and 0.9
  install  install() is idempotent, reaches classes persistence rebuilt from a pickle and runs the original method
           outside the envelope
  cuda     the default G forward + backward on cuda, installed and not, at beta 1 and 0.999; no host sync; the kernels
           the profiler sees
"""
import copy
import os
import pickle
import sys
import types
import warnings

import torch

warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))

from model import generator_lres as gl           # noqa: E402
from torch_utils.ops import gblock_tail as gt    # noqa: E402

out_file, mode = sys.argv[1], sys.argv[2]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
ORIG = gl.Synthesis3dResBlock.forward


def capture(G, *args, **kw):
    """(block, input, latent, out_seq_length) of every block call of G(*args)."""
    calls = []

    def spy(self, input, latent, magnitude_ema_beta=1.0, out_seq_length=None, dtype=None):
        calls.append((self, input.detach().clone(), latent.detach().clone(), out_seq_length))
        return ORIG(self, input, latent, magnitude_ema_beta, out_seq_length, dtype)
    gl.Synthesis3dResBlock.forward = spy
    try:
        with torch.no_grad():
            G(*args, **kw)
    finally:
        gl.Synthesis3dResBlock.forward = ORIG
    return calls


def compare_block(blk, x, lat, osl):
    """reference forward vs block_forward on copies of the block at beta 1 (exact) and beta 0.9."""
    r = {}
    for beta in (1.0, 0.9):
        a, b = copy.deepcopy(blk), copy.deepcopy(blk)
        with torch.no_grad():
            ref = ORIG(a, x, lat, beta, osl)
            ours = gt.block_forward(b, gl.__dict__, x, lat, beta, osl)
        bufs = [torch.equal(p, q) for p, q in zip(a.buffers(), b.buffers())]
        r[beta] = dict(ref=ref, ours=ours, same_buffers=all(bufs),
                       buf_err=max([float((p - q).abs().max()) for p, q in zip(a.buffers(), b.buffers())] + [0.0]))
    return dict(sig=(blk.in_channels, blk.out_channels, tuple(x.shape[2:]), osl, blk.temporal_up, blk.spatial_up,
                     blk.out_height, blk.out_width), res=r)


if mode == 'cpu':
    res = []
    for kw, seq in ((dict(out_height=36, out_width=64), 8), (dict(out_height=64, out_width=64), 6)):
        torch.manual_seed(0)
        G = gl.VideoGenerator(**kw)
        torch.manual_seed(1)
        for blk, x, lat, osl in capture(G, 1, seq):
            res.append(compare_block(blk, x, lat, osl))
    # standalone blocks: both flags, odd crop differences on every axis, small channel counts
    g = torch.Generator().manual_seed(5)
    for (tup, sup, t, h, w, osl, oh, ow) in ((True, True, 5, 5, 7, 7, 9, 13), (True, False, 6, 3, 5, 9, None, None),
                                            (False, True, 4, 6, 5, 3, 11, 9), (False, False, 9, 4, 6, 6, 3, 5),
                                            (True, True, 3, 4, 4, 4, 7, 7)):
        torch.manual_seed(7)
        blk = gl.Synthesis3dResBlock(16, 8, 6, out_height=oh or (2 * h if sup else h), out_width=ow or (2 * w if sup else w),
                                     temporal_ksize=3, spatial_ksize=3, temporal_up=tup, spatial_up=sup)
        with torch.no_grad():
            for p in blk.parameters():
                p.add_(torch.randn(p.shape, generator=g) * 0.3)
        x = torch.randn(2, 8, t, h, w, generator=g) * 3
        lat = torch.randn(2, 16, t, generator=g)
        res.append(compare_block(blk, x, lat, osl))
elif mode == 'install':
    assert gt.install(gl) == [gl.Synthesis3dResBlock]
    fwd = gl.Synthesis3dResBlock.forward
    assert fwd is not ORIG and fwd.lvg_gblock_tail is ORIG
    assert gt.install(gl) == [gl.Synthesis3dResBlock] and gl.Synthesis3dResBlock.forward is fwd
    torch.manual_seed(0)
    blk = gl.Synthesis3dResBlock(16, 8, 6, temporal_ksize=3, spatial_ksize=3, temporal_up=True, spatial_up=True, out_height=7, out_width=8)
    assert gt.install(blk) == [gl.Synthesis3dResBlock] and gl.Synthesis3dResBlock.forward is fwd
    # a block that persistence rebuilds from its pickled source has a class of its own
    data = pickle.dumps(blk)
    gl.persistence._src_to_module_dict.clear()           # as in a fresh process: the source runs in a module of its own
    blk2 = pickle.loads(data)
    cls2 = type(blk2)
    assert cls2 is not gl.Synthesis3dResBlock and cls2.__name__ == 'Synthesis3dResBlock'
    assert gt.install(torch.nn.ModuleList([blk2])) == [cls2] and cls2.forward.lvg_gblock_tail is not None
    orig2 = cls2.forward.lvg_gblock_tail
    assert gt.install(blk2) == [cls2] and cls2.forward.lvg_gblock_tail is orig2
    # outside the envelope the original method runs: CPU tensors, padded resamplers, other activations
    calls = []

    def spy(self, *a, **k):
        calls.append(1)
        return ORIG(self, *a, **k)
    patched = gt._forward(spy)
    x = torch.randn(1, 8, 3, 4, 4)
    lat = torch.randn(1, 16, 3)
    got = patched(blk, x, lat, 1.0, 5)
    assert torch.equal(got, ORIG(blk, x, lat, 1.0, 5)) and len(calls) == 1
    blk_pad = copy.deepcopy(blk)
    blk_pad.temporal_upsample.padding = 1
    blk_relu = copy.deepcopy(blk)
    blk_relu.activation = 'relu'
    for b in (blk, blk_pad, blk_relu):
        assert not gt.applies(b, x, torch.float32, 5)
    assert not gt.applies(blk, x.double(), torch.float64, 5)
    gl.Synthesis3dResBlock.forward = ORIG
    res = 'ok'
elif mode == 'cuda':
    from torch_utils.ops import conv_nd, modulated_conv
    conv_nd.install_functional(gl)
    modulated_conv.install(gl)
    dev = torch.device('cuda')

    def step(G, beta, seed=1):
        torch.manual_seed(seed)
        v = G(2, 32, magnitude_ema_beta=beta)
        tgt = torch.randn(v.shape, generator=torch.Generator().manual_seed(11)).to(dev)
        (v * tgt).mean().backward()
        grads = torch.cat([p.grad.flatten().float() for p in G.parameters() if p.grad is not None])
        for p in G.parameters():
            p.grad = None
        return v.detach(), grads

    res = {}
    torch.manual_seed(0)
    G0 = gl.VideoGenerator(out_height=36, out_width=64).to(dev)
    for beta in (1.0, 0.999):
        outs = []
        for installed in (False, True):
            gl.Synthesis3dResBlock.forward = ORIG
            if installed:
                gt.install(gl)
            G = copy.deepcopy(G0)
            v, g = step(G, beta)
            outs.append(dict(v=v.cpu(), g=g.cpu(), bufs=[b.cpu() for b in G.buffers()], cpu_rng=torch.get_rng_state(),
                             cuda_rng=torch.cuda.get_rng_state()))
        res[beta] = outs
    # installed: no host synchronisation in forward + backward, and the kernels the profiler sees
    gl.Synthesis3dResBlock.forward = ORIG
    gt.install(gl)
    G = copy.deepcopy(G0)
    step(G, 0.999)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        torch.manual_seed(1)
        v = G(2, 32, magnitude_ema_beta=0.999)
        v.square().mean().backward()
        res['nosync'] = True
    except RuntimeError as e:
        res['nosync'] = str(e)
    torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()

    def profile(installed):
        gl.Synthesis3dResBlock.forward = ORIG
        if installed:
            gt.install(gl)
        G = copy.deepcopy(G0)
        step(G, 0.999)
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
            step(G, 0.999)
            torch.cuda.synchronize()
        names = {}
        for e in prof.events():
            names[e.name] = names.get(e.name, 0) + 1
        return names
    res['prof_ref'] = profile(False)
    res['prof_ours'] = profile(True)
    gl.Synthesis3dResBlock.forward = ORIG
torch.save(res, out_file)
