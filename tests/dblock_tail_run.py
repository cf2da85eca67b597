"""Helper of test_dblock_tail_host.py and test_gpu_dblock_tail.py (run as a subprocess): builds the UNMODIFIED reference
low-res discriminator (staged at oracle/_ref/src) with this repository's ops and compares DiscriminatorBlock.forward with
dblock_tail.install against the original method. argv: <out file> <mode>:
  cpu        every block of the default D and of a seq_length 2 / max_edge 32 D on small CPU inputs: output, first-order
             gradients and the R1 pattern, original and installed
  install_a  install() conventions, dblock_tail.install before conv3d_down.install
  install_b  the same with conv3d_down.install first
  cuda       the whole D (seq_length 16, 64 x 64, batch 2) on the GPU in fp32 and with num_fp16_res=4: without install, with
             install (the conv_bias_act layers) and with install(tail=True) (also every block on the op);
             conv_nd.install_functional and conv3d_down.install on all sides; the kernel names torch.profiler sees in one
             R1 step and one forward without grad of the last
  orient     the whole fp32 D as in cuda with every Downsample3d filter set to the asymmetric [1, 2, 4, 1] / 8: without
             conv3d_down / dblock_tail, then with both installed (tail=True); the kernel names of one installed R1 step"""
import sys
import types
import warnings

import torch

warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))
from model import discriminator_lres as dl          # noqa: E402
from torch_utils.ops import conv_nd, conv3d_down, dblock_tail      # noqa: E402

out_file, mode = sys.argv[1], sys.argv[2]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def block_step(fn, blk, x, r1):
    """Output, input gradient and parameter gradients of one block through ``fn``; r1: the gradient-penalty pattern."""
    for p in blk.parameters():
        p.grad = None
    xi = x.clone().requires_grad_(True)
    out = fn(blk, xi)
    if r1:
        gx, = torch.autograd.grad(out.square().sum(), [xi], create_graph=True)
        (gx.square().sum() + out.sum()).backward()
    else:
        gx = None
        out.square().sum().backward()
    grads = [p.grad.clone() for p in blk.parameters() if p.grad is not None]
    return [out.detach(), xi.grad.clone()] + ([gx.detach()] if r1 else []) + grads


if mode == 'cpu':
    assert dblock_tail.install(dl) == [dl.DiscriminatorBlock, dl.Conv3dLayer]
    orig = dl.DiscriminatorBlock.forward.lvg_dblock_tail
    calls = []
    ref_fn = dblock_tail._reference
    dblock_tail._reference = lambda *a, **k: (calls.append(1), ref_fn(*a, **k))[1]
    res = []
    for seq, edge in ((128, 64), (2, 32)):
        torch.manual_seed(seq)
        D = dl.VideoDiscriminator(seq_length=seq, max_edge=edge)
        for i, blk in enumerate(D.blocks):
            for p in blk.parameters():
                if p.ndim == 1:
                    torch.nn.init.normal_(p, std=0.5)
            cin = blk.vid_channels or blk.in_channels
            x = torch.randn(2, cin, 4, 8, 8, generator=torch.Generator().manual_seed(i)) * (40 if i == 1 else 1)
            for r1 in (False, True):
                n0 = len(calls)
                ours = block_step(dl.DiscriminatorBlock.forward, blk, x, r1)
                took = len(calls) - n0
                ref = block_step(orig, blk, x, r1)
                res.append({'cfg': (seq, edge, i, r1), 'down': (blk.conv_1.spatial_down, blk.conv_1.temporal_down), 'took': took,
                            'ours': ours, 'ref': ref})
    torch.save(res, out_file)
    sys.exit(0)

if mode in ('install_a', 'install_b'):
    torch.manual_seed(0)
    D = dl.VideoDiscriminator(seq_length=4, max_edge=64)
    x = torch.randn(1, 3, 4, 64, 64, generator=torch.Generator().manual_seed(1))
    want = D(x)
    plain, plain_layer = dl.DiscriminatorBlock.forward, dl.Conv3dLayer.forward
    both = [dl.DiscriminatorBlock, dl.Conv3dLayer]
    if mode == 'install_b':
        assert conv3d_down.install(dl) == [dl.Conv3dLayer]
    assert dblock_tail.install(dl) == both
    first = dl.DiscriminatorBlock.forward
    assert first is not plain and first.lvg_dblock_tail is plain and first.tail is False
    if mode == 'install_a':
        assert conv3d_down.install(dl) == [dl.Conv3dLayer]
    # the two Conv3dLayer patches wrap each other in either order; installing either again changes nothing
    layer = dl.Conv3dLayer.forward
    outer, inner = ('lvg_conv3d_down', 'lvg_conv_bias_act') if mode == 'install_a' else ('lvg_conv_bias_act', 'lvg_conv3d_down')
    assert getattr(getattr(layer, outer), inner) is plain_layer
    assert dblock_tail.install(dl, D) == both and conv3d_down.install(dl, D) == [dl.Conv3dLayer]
    assert dl.DiscriminatorBlock.forward is first and dl.Conv3dLayer.forward is layer                        # idempotent
    assert dblock_tail.install(D.blocks[0]) == both and dblock_tail.install(torch.nn.Linear(1, 1)) == []
    assert dblock_tail.install(dl, tail=True) == both and first.tail is True and dl.DiscriminatorBlock.forward is first
    seen = []
    run = dblock_tail.block_forward
    dblock_tail.block_forward = lambda blk, inp: (seen.append(tuple(inp.shape)), run(blk, inp))[1]
    got = D(x)
    assert len(seen) == 4 and torch.equal(got, want), float((got - want).abs().max())
    # outside the envelope: odd extents on a halved axis, and a conv_1 that the conv3d_down decomposition takes
    blk = D.blocks[1]
    odd = torch.randn(1, 64, 4, 7, 8)
    del seen[:]
    assert torch.equal(blk(odd), plain(blk, odd)) and not seen
    pw = dl.DiscriminatorBlock(8, 8, spatial_ksize=1, temporal_ksize=1)
    xs = torch.randn(1, 8, 4, 8, 8)
    assert torch.equal(pw(xs), plain(pw, xs)) and not seen
    # CUDA inputs take the op only where it is faster (nowhere) or with tail=True; CPU layers never take the epilogue
    fake = types.SimpleNamespace(is_cuda=True, shape=(1, 64, 4, 8, 8))
    real_applies, dblock_tail.applies = dblock_tail.applies, lambda b, i: True
    assert dblock_tail.routed(blk, fake, True) and not dblock_tail.routed(blk, fake, False)
    dblock_tail.applies = real_applies
    assert not dblock_tail.epilogue_applies(blk.conv_0, xs) and not dblock_tail.epilogue_applies(blk.conv_skip, xs)
    torch.save('ok', out_file)
    sys.exit(0)

assert mode in ('cuda', 'orient')
conv_nd.install_functional(dl)
if mode == 'cuda':
    conv3d_down.install(dl)
x = (torch.rand(2, 3, 16, 64, 64, generator=torch.Generator().manual_seed(12)) * 2 - 1).cuda().requires_grad_(True)


def step(D):
    for p in D.parameters():
        p.grad = None
    x.grad = None
    logits = D(x)
    gx, = torch.autograd.grad(logits.sum(), [x], create_graph=True)
    (gx.square().sum() + torch.nn.functional.softplus(logits).mean()).backward()
    grads = torch.cat([p.grad.flatten().double() for p in D.parameters() if p.grad is not None])
    with torch.no_grad():
        plain = D(x.detach())
    return {'logits': logits.detach().double().cpu(), 'r1_gx': gx.detach().double().cpu(), 'gx': x.grad.double().cpu(),
            'grad': grads.cpu(), 'nograd_logits': plain.double().cpu()}


if mode == 'orient':
    torch.manual_seed(2)
    D = dl.VideoDiscriminator(seq_length=16, max_edge=64).cuda()
    filters = [m._downsample_filter for m in D.modules() if type(m).__name__ == 'Downsample3d']
    with torch.no_grad():
        for f in filters:
            f.copy_(torch.tensor([1., 2., 4., 1.]) / 8)
    out = {'filters': len(filters), 'ref': step(D)}
    conv3d_down.install(dl)
    dblock_tail.install(dl, tail=True)
    out['ours'] = step(D)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        step(D)
        torch.cuda.synchronize()
    out['kernels'] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    torch.save(out, out_file)
    sys.exit(0)

out, nets = {}, {}
for name, nfp16 in (('fp32', 0), ('fp16', 4)):
    torch.manual_seed(2)
    nets[name] = dl.VideoDiscriminator(seq_length=16, max_edge=64, num_fp16_res=nfp16).cuda()
    out[name + '_ref'] = step(nets[name])
for tail in (False, True):                      # the epilogue layers alone, then also every block on the op
    dblock_tail.install(dl, tail=tail)
    epi, blocks = [], []
    cba, bf = conv_nd.conv_bias_act, dblock_tail.block_forward
    conv_nd.conv_bias_act = lambda *a, **k: (epi.append(torch.is_grad_enabled()), cba(*a, **k))[1]
    dblock_tail.block_forward = lambda *a: (blocks.append(1), bf(*a))[1]
    key = '_ours' if tail else '_epilogue'
    for name, D in nets.items():
        out[name + key] = step(D)
        if name == 'fp32':
            again = step(D)
            out['bitwise' + key] = all(torch.equal(again[k], out['fp32' + key][k]) for k in ('logits', 'r1_gx', 'nograd_logits'))
        if tail:
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                step(D)
                with torch.no_grad():
                    D(x)
                torch.cuda.synchronize()
            out[name + '_kernels'] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    conv_nd.conv_bias_act, dblock_tail.block_forward = cba, bf
    out['calls' + key] = (len(epi), sum(epi), len(blocks))        # conv_bias_act calls, of them with grad mode on, blocks on the op
torch.save(out, out_file)
