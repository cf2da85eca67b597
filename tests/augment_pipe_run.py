"""Helper of test_augment_pipe_host.py and test_gpu_augment_pipe.py (run as a subprocess): the UNMODIFIED reference
``AugmentPipe`` (staged at oracle/_ref/src) in the two configurations ``SuperResVideoGAN`` builds (video_gan_sres.py:110-136,
train_sres.py:360-373), against this repository's ``augment_pipe`` under the same seeds.

argv: <out file> <mode>
  cpu      per case: the reference's output, RNG state and F.pad arguments, and draw_params + the torch composition
  cuda     per case: y and dx of a fixed dy from the original and the installed forward, and the RNG states; one case
           through the unmodified SuperResVideoGAN.run_D with a small D, with the R1 create_graph pattern; the installed
           run_D + R1 under torch.cuda.set_sync_debug_mode('error'); two runs under torch.use_deterministic_algorithms
  install  the install logic: patched class, idempotence, fallback to the original on calls the op does not take
"""
import sys
import types
import warnings

import torch

warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))
sys.modules.setdefault('utils', types.ModuleType('utils'))
from model import ada_augment                        # noqa: E402
from torch_utils.ops import augment_pipe as ap      # noqa: E402
from torch_utils.ops import grid_sample_gradfix     # noqa: E402

grid_sample_gradfix.enabled = True                  # as train_sres.py:84 sets it: the reference's R1 pass needs it

out_file, mode = sys.argv[1], sys.argv[2]

AUGMENT = dict(xflip=1, rotate90=1, xint=1, scale=1, rotate=1, aniso=1, xfrac=1, brightness=1, contrast=1, lumaflip=1, hue=1,
               saturation=1)
S = 8                                               # in_augment_strength
IN_AUGMENT = dict(scale=1, scale_std=0.01 * S, rotate=1, rotate_max=0.002 * S, aniso=1, aniso_std=0.01 * S, xfrac=1,
                  xfrac_std=0.002 * S, noise=1, noise_std=0.01 * S)
CONFIGS = {'augment': AUGMENT, 'in_augment': IN_AUGMENT}


def pipe(name, p, device):
    m = ada_augment.AugmentPipe(**CONFIGS[name]).to(device).requires_grad_(False).train()
    m.p.fill_(p)
    return m


def video(n, t, h, w, seed, device):
    """A smooth random clip in [-1, 1]: noise at a quarter of the resolution, upsampled bilinearly."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.rand(n * 3 * t, 1, (h + 3) // 4 + 1, (w + 3) // 4 + 1, generator=g) * 2 - 1
    x = torch.nn.functional.interpolate(lo, size=(h, w), mode='bilinear', align_corners=False)
    return x.view(n, 3, t, h, w).to(device)


# (config, p, N, T, H, W)
CASES = [(c, p, 2, 4, 18, 32) for c in CONFIGS for p in (0.0, 0.5, 1.0)] + [('augment', 1.0, 1, 3, 13, 21), ('in_augment', 0.5, 3, 2, 9, 15)]

res = []
if mode == 'cpu':
    real_pad = torch.nn.functional.pad
    for k, (name, p, n, t, h, w) in enumerate(CASES):
        x = video(n, t, h, w, k, 'cpu')
        m = pipe(name, p, 'cpu')
        pads = []

        def spy(input, pad, mode='constant', value=None):
            if mode == 'reflect':
                pads.append(list(pad))
            return real_pad(input, pad, mode=mode) if value is None else real_pad(input, pad, mode=mode, value=value)
        torch.nn.functional.pad = spy
        torch.manual_seed(100 + k)
        ref = m(x)
        torch.nn.functional.pad = real_pad
        state_ref = torch.get_rng_state()
        torch.manual_seed(100 + k)
        params, noise, flags = ap.draw_params(m, x)
        state_ours = torch.get_rng_state()
        ours = ap._reference(x, params, noise, m.Hz_geom, flags)
        res.append(dict(case=(name, p, n, t, h, w), ref=ref, ours=ours, params=params, pads=pads, flags=flags,
                        same_state=torch.equal(state_ref, state_ours)))
elif mode == 'cuda':
    orig = ada_augment.AugmentPipe.forward
    for k, (name, p, n, t, h, w) in enumerate(CASES):
        x0 = video(n, t, h, w, k, 'cuda')
        dy = torch.randn(x0.shape, generator=torch.Generator().manual_seed(k)).cuda()
        outs = []
        for installed in (False, True):
            if installed:
                ap.install(ada_augment)
            m = pipe(name, p, 'cuda')
            x = x0.clone().requires_grad_(True)
            torch.manual_seed(100 + k)
            y = m(x)
            gx, = torch.autograd.grad(y, [x], dy)
            outs.append(dict(y=y.detach().cpu(), gx=gx.cpu(), cuda_state=torch.cuda.get_rng_state(), cpu_state=torch.get_rng_state()))
            ada_augment.AugmentPipe.forward = orig
        res.append(dict(case=(name, p, n, t, h, w), ref=outs[0], ours=outs[1]))

    # the unmodified SuperResVideoGAN.run_D with a small D: the stacked clip goes through `augment`
    from model import video_gan_sres as vs

    class SmallD(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.w = torch.nn.Parameter(torch.randn(3, generator=torch.Generator().manual_seed(3)))

        def upsample(self, lr):
            return torch.nn.functional.interpolate(lr.flatten(1, 2), scale_factor=4, mode='nearest').view(*lr.shape[:3], lr.shape[3] * 4, lr.shape[4] * 4)

        def forward(self, lr, hr):
            wt = self.w.view(1, 3, 1, 1, 1)
            return ((hr * wt).square().mean((1, 2, 3, 4)) + (lr * hr).mean((1, 2, 3, 4))).unsqueeze(1)

    def gan():
        g = vs.SuperResVideoGAN.__new__(vs.SuperResVideoGAN)      # no __post_init__: it builds G / D and broadcasts
        g.channels, g.seq_length, g.lr_height, g.lr_width, g.hr_height, g.hr_width = 3, 4, 9, 16, 36, 64
        g.lr_cond_prob = 1.0
        g.D = SmallD().cuda()
        g.augment = pipe('augment', 0.5, 'cuda')
        return g

    def r1_step(g, lr, hr0):
        hr = hr0.clone().requires_grad_(True)
        torch.manual_seed(7)
        logits = g.run_D(lr, hr)
        gx, = torch.autograd.grad(logits.sum(), [hr], create_graph=True)
        (gx.square().sum() + torch.nn.functional.softplus(logits).mean()).backward()
        return logits.detach(), hr.grad

    lr = video(2, 4, 9, 16, 50, 'cuda')
    hr = video(2, 4, 36, 64, 51, 'cuda')
    run_d = []
    for installed in (False, True):
        if installed:
            ap.install(vs)
        logits, g_hr = r1_step(gan(), lr, hr)
        run_d.append(dict(logits=logits.cpu(), gx=g_hr.cpu()))
    g = gan()
    r1_step(g, lr, hr)                                        # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    _, dx_nosync = r1_step(g, lr, hr)
    torch.cuda.set_sync_debug_mode(0)
    torch.use_deterministic_algorithms(True)
    det = [r1_step(g, lr, hr)[1].cpu() for _ in range(2)]
    torch.use_deterministic_algorithms(False)
    ada_augment.AugmentPipe.forward = orig
    res = dict(cases=res, run_D=run_d, nosync=dx_nosync.cpu(), det=det)
elif mode == 'install':
    orig = ada_augment.AugmentPipe.forward
    assert ap.install(ada_augment) == [ada_augment.AugmentPipe]
    assert ada_augment.AugmentPipe.forward is not orig and ada_augment.AugmentPipe.forward.lvg_augment_pipe is orig
    assert ap.install(ada_augment) == [ada_augment.AugmentPipe] and ada_augment.AugmentPipe.forward.lvg_augment_pipe is orig
    m = pipe('augment', 0.5, 'cpu')
    assert ap.install(m) == [ada_augment.AugmentPipe] and ada_augment.AugmentPipe.forward.lvg_augment_pipe is orig
    from model import video_gan_sres as vs
    assert ap.install(vs) == [ada_augment.AugmentPipe] and ada_augment.AugmentPipe.forward.lvg_augment_pipe is orig
    # pipes inside a container are reached; a module of another name is not, whatever its attributes
    assert ap.install(torch.nn.ModuleList([m])) == [ada_augment.AugmentPipe]
    other = torch.nn.Module()
    other.register_buffer('Hz_geom', m.Hz_geom)
    assert ap.install(other) == []
    calls = []

    def spy(self, v, debug_percentile=None):
        calls.append(v.shape)
        return orig(self, v, debug_percentile)
    patched = ap._forward(spy)
    x = video(1, 1, 48, 48, 0, 'cpu')       # the reference's imgfilter step takes one frame of at least 22 x 22 pixels
    for m, kw in ((pipe('augment', 0.5, 'cpu'), {}),                                      # a CPU video
                  (ada_augment.AugmentPipe(xflip=1, imgfilter=1), {}),                      # image-space filtering
                  (ada_augment.AugmentPipe(cutout=1), {}),                                  # cutout
                  (pipe('augment', 0.5, 'cpu'), dict(debug_percentile=0.3))):               # debug_percentile
        torch.manual_seed(5)
        got = patched(m, x, **kw)
        torch.manual_seed(5)
        assert torch.equal(got, orig(m, x, **kw))
    assert len(calls) == 4, calls
    ada_augment.AugmentPipe.forward = orig
    res = 'ok'
torch.save(res, out_file)
