"""Helper of test_gpu_sres_dblock.py (run as a subprocess): builds the UNMODIFIED reference super-res discriminator (staged
at oracle/_ref/src) with this repository's ops and compares it with and without sres_dblock.install. argv: <out file> <mode>:
  cuda     VideoDiscriminator (default channels, 64 x 64, seq_length 4, batch 2) with num_fp16_res 2 (two fp16 and two
           fp32 blocks) and 0 (all fp32), without and with install: logits, parameter gradients and the R1 pattern
           (create_graph); which blocks
           the installed forward took; kernel names torch.profiler sees in one installed R1 step
  run_D    SuperResVideoGAN.run_D + R1 with augment_pipe.install, then also sres_dblock.install, on the same GAN object
  kernels  kernel names torch.profiler sees in forward + backward passes of four block shapes (fp16 / fp32, 64- / 128-row skips)
  cpu      install() conventions and the CPU forward of the installed D (bitwise the original)
  orient   the all-fp32 D of cuda with every resample_filter set to setup_filter([1, 2, 4, 1]), without and with install;
           which blocks the installed forward took; kernel names of one installed forward + first-order backward"""
import pickle
import sys
import types
import warnings

import torch

warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))
sys.modules.setdefault('utils', types.ModuleType('utils'))
from model import discriminator_sres as ds          # noqa: E402
from torch_utils.ops import sres_dblock             # noqa: E402

out_file, mode = sys.argv[1], sys.argv[2]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def make_D(seed, **kw):
    torch.manual_seed(seed)
    D = ds.VideoDiscriminator(**kw)
    with torch.no_grad():
        for p in D.parameters():
            if p.ndim == 1:
                p.normal_(std=0.2)
    return D


def step(D, lr, hr, r1):
    for p in D.parameters():
        p.grad = None
    hr = hr.clone().requires_grad_(True)
    logits = D(lr, hr)
    if r1:
        gx, = torch.autograd.grad(logits.sum(), [hr], create_graph=True)
        (gx.square().sum() + torch.nn.functional.softplus(logits).mean()).backward()
    else:
        gx = None
        torch.nn.functional.softplus(-logits).mean().backward()
    out = dict(logits=logits.detach().cpu(), hr=hr.grad.cpu())
    if r1:
        out['gx'] = gx.detach().cpu()
    out.update({n: p.grad.cpu() for n, p in D.named_parameters() if p.grad is not None})
    return out


def videos(n, seed, dev, t=4, hr=64, lr=16):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 3, t, lr, lr, generator=g).to(dev), torch.randn(n, 3, t, hr, hr, generator=g).to(dev)


res = {}
if mode == 'cuda':
    kw = dict(seq_length=4, lr_height=16, lr_width=16, hr_height=64, hr_width=64, num_fp16_res=2)
    D = make_D(0, **kw).cuda()
    D32 = make_D(0, **dict(kw, num_fp16_res=0)).cuda()
    lr, hr = videos(2, 1, 'cuda')
    res['ref'] = [step(D, lr, hr, r1) for r1 in (False, True)]
    res['ref32'] = [step(D32, lr, hr, r1) for r1 in (False, True)]
    assert sres_dblock.install(D) == [ds.DiscriminatorBlock, ds.Conv2dLayer]
    took = []
    orig_op = sres_dblock.sres_dblock

    def counted(x, *a, **k):
        took.append((tuple(x.shape), str(x.dtype), sres_dblock.native(x, a[0], a[1], a[3], a[5], a[6], k.get('act', 'lrelu'))))
        return orig_op(x, *a, **k)
    sres_dblock.sres_dblock = counted
    res['ours'] = [step(D, lr, hr, r1) for r1 in (False, True)]
    res['ours32'] = [step(D32, lr, hr, r1) for r1 in (False, True)]
    sres_dblock.sres_dblock = orig_op
    res['took'] = took
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(D, lr, hr, True)
        torch.cuda.synchronize()
    res['kernels'] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    ds.DiscriminatorBlock.forward = ds.DiscriminatorBlock.forward.lvg_sres_dblock
    ds.Conv2dLayer.forward = ds.Conv2dLayer.forward.lvg_sres_dblock
elif mode == 'orient':
    from torch.profiler import ProfilerActivity, profile
    from torch_utils.ops import upfirdn2d
    D = make_D(0, seq_length=4, lr_height=16, lr_width=16, hr_height=64, hr_width=64, num_fp16_res=0).cuda()
    filters = [m.resample_filter for m in D.modules() if getattr(m, 'resample_filter', None) is not None]
    with torch.no_grad():
        for f in filters:
            f.copy_(upfirdn2d.setup_filter([1, 2, 4, 1]))
    res['filters'] = len(filters)
    lr, hr = videos(2, 1, 'cuda')
    res['ref'] = [step(D, lr, hr, r1) for r1 in (False, True)]
    sres_dblock.install(D)
    took = []
    orig_op = sres_dblock.sres_dblock

    def counted(x, *a, **k):
        took.append(sres_dblock.native(x, a[0], a[1], a[3], a[5], a[6], k.get('act', 'lrelu')))
        return orig_op(x, *a, **k)
    sres_dblock.sres_dblock = counted
    res['ours'] = [step(D, lr, hr, r1) for r1 in (False, True)]
    sres_dblock.sres_dblock = orig_op
    res['took'] = took
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(D, lr, hr, False)
        torch.cuda.synchronize()
    res['kernels'] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
elif mode == 'run_D':
    from model import video_gan_sres as vs
    from model import ada_augment
    from torch_utils.ops import augment_pipe as ap
    from torch_utils.ops import grid_sample_gradfix
    grid_sample_gradfix.enabled = True              # as train_sres.py sets it: the reference's R1 pass needs it
    kw = dict(seq_length=4, lr_height=16, lr_width=16, hr_height=64, hr_width=64, num_fp16_res=0)

    def gan():
        g = vs.SuperResVideoGAN.__new__(vs.SuperResVideoGAN)      # no __post_init__: it builds G / D and broadcasts
        g.channels, g.seq_length, g.lr_height, g.lr_width, g.hr_height, g.hr_width = 3, 4, 16, 16, 64, 64
        g.lr_cond_prob = 1.0
        g.D = make_D(0, **kw).cuda()
        g.augment = ada_augment.AugmentPipe(xflip=1, rotate90=1, xint=1, scale=1, rotate=1, aniso=1, xfrac=1).cuda()
        g.augment.p.fill_(0.5)
        return g

    def r1_step(g, lr, hr0):
        for p in g.D.parameters():
            p.grad = None
        hr = hr0.clone().requires_grad_(True)
        torch.manual_seed(7)
        logits = g.run_D(lr, hr)
        gx, = torch.autograd.grad(logits.sum(), [hr], create_graph=True)
        (gx.square().sum() + torch.nn.functional.softplus(logits).mean()).backward()
        return dict(logits=logits.detach().cpu(), hr=hr.grad.cpu(), gx=gx.detach().cpu(),
                    **{n: p.grad.cpu() for n, p in g.D.named_parameters() if p.grad is not None})

    lr, hr = videos(2, 5, 'cuda')
    ap.install(ada_augment)
    g = gan()
    res['ref'] = r1_step(g, lr, hr)                   # augment_pipe installed, the D as it is
    sres_dblock.install(g.D)
    res['ours'] = r1_step(g, lr, hr)                  # both installed on the same GAN object
elif mode == 'kernels':
    import numpy as np
    from torch.profiler import ProfilerActivity, profile
    from torch_utils.ops import upfirdn2d
    f = upfirdn2d.setup_filter([1, 3, 3, 1]).cuda()
    calls = []
    for cin, cout, r, dtype in ((64, 128, 32, torch.float16), (512, 512, 16, torch.float32), (24, 40, 16, torch.float32),
                                (24, 40, 16, torch.float16)):
        g = torch.Generator().manual_seed(cin)
        t = lambda *s: (torch.randn(*s, generator=g) / 8).cuda().to(dtype)      # noqa: E731
        calls.append((t(2, cin, r, r), t(cout, cin, 1, 1), t(cin, cin, 3, 3), t(cin), t(cout, cin, 3, 3), t(cout)))
    for a in calls:                                  # warm-up outside the trace
        sres_dblock.sres_dblock(*a, f, f, gain=float(np.sqrt(2)), clamp=256)
    torch.cuda.synchronize()
    calls = [tuple(t.requires_grad_(True) for t in a) for a in calls]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for a in calls:
            sres_dblock.sres_dblock(*a, f, f, gain=float(np.sqrt(2)), clamp=256).float().sum().backward()
        torch.cuda.synchronize()
    res['kernels'] = sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
elif mode == 'cpu':
    plain_b, plain_l = ds.DiscriminatorBlock.forward, ds.Conv2dLayer.forward
    D = make_D(0, seq_length=2, lr_height=8, lr_width=8, hr_height=32, hr_width=32, channels_base=512, channels_max=32)
    lr, hr = videos(2, 3, 'cpu', t=2, hr=32, lr=8)
    want = step(D, lr, hr, True)
    assert sres_dblock.install(ds) == [ds.DiscriminatorBlock, ds.Conv2dLayer]
    first = ds.DiscriminatorBlock.forward, ds.Conv2dLayer.forward
    assert sres_dblock.install(ds, D) == [ds.DiscriminatorBlock, ds.Conv2dLayer]
    assert (ds.DiscriminatorBlock.forward, ds.Conv2dLayer.forward) == first, 'install is not idempotent'
    assert first[0].lvg_sres_dblock is plain_b and first[1].lvg_sres_dblock is plain_l
    got = step(D, lr, hr, True)
    res['cpu_equal'] = all(torch.equal(want[k], got[k]) for k in want)
    # a pickled network: persistence rebuilds its classes from the source; install reaches them through the instance
    D2 = pickle.loads(pickle.dumps(D))
    res['pickled'] = [c.__name__ for c in sres_dblock.install(D2)]
    res['pickled_patched'] = all(getattr(type(m).forward, 'lvg_sres_dblock', None) is not None
                                 for m in D2.modules() if type(m).__name__ in ('DiscriminatorBlock', 'Conv2dLayer'))
torch.save(res, out_file)
