"""Helper of test_video_augment_host.py and test_gpu_video_augment.py (run as a subprocess): the UNMODIFIED reference
``LowResVideoGAN.run_D`` (staged at oracle/_ref/src, ``utils`` / ``imageio`` stubbed) with a stub D that records its input,
against this repository's ``video_augment`` under the same seeds.

argv: <out file> <mode>
  cpu      per case: the reference's D input and RNG states after run_D, and the same from draw_params + apply on the CPU
  cuda     per case: D input, logits and video gradient of the reference run_D and of the installed one, on cuda; then
           the installed run_D under torch.cuda.set_sync_debug_mode('error'), and forward + backward + the R1 pattern under
           torch.use_deterministic_algorithms(True), twice (dx of both runs)
  install  the install logic on the CPU: patched class, idempotence, fallback to the original on unsupported input
"""
import sys
import types
import warnings

import torch

warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))
sys.modules.setdefault('utils', types.ModuleType('utils'))
from model import video_gan_lres as vg               # noqa: E402
from torch_utils.ops import video_augment as va      # noqa: E402

out_file, mode = sys.argv[1], sys.argv[2]
POLICIES = ['color,translation,cutout', '', 'color', 'translation', 'cutout', 'color,translation', 'translation,cutout',
            'color,cutout']
# (policy, temp_scale_augment, N, C, T, H, W)
CASES = ([(p, ts, 3, 3, 16, 12, 20) for p in POLICIES for ts in (0.0, 1.0)]
         + [(p, 1.0, 2, 1, 12, 9, 15) for p in ('color,translation,cutout', 'color')]
         + [('color,translation,cutout', 0.5, 2, 3, 20, 7, 11), ('color,translation,cutout', 2.0, 4, 3, 16, 10, 12)])


class StubD(torch.nn.Module):
    """Records its input; logits = a fixed quadratic function of it (so that the R1 gradient depends on the video)."""

    def __init__(self):
        super().__init__()
        self.seen = []

    def forward(self, video):
        self.seen.append(video)
        wgt = torch.linspace(-1, 1, video[0].numel(), dtype=video.dtype, device=video.device).view(video.shape[1:])
        return (video * wgt + 0.25 * video.square() * wgt.flip(0)).flatten(1).sum(1, keepdim=True)


def gan(policy, ts, c, t, h, w):
    g = vg.LowResVideoGAN.__new__(vg.LowResVideoGAN)     # no __post_init__: it builds G / D on cuda and broadcasts
    g.seq_length, g.height, g.width, g.channels = t, h, w, c
    g.temp_scale_augment, g.diffaug_policy = ts, policy
    g.D = StubD()
    return g


def video(n, c, t, h, w, seed, device='cpu'):
    return (torch.rand(n, c, t, h, w, generator=torch.Generator().manual_seed(seed)) * 2 - 1).to(device)


res = []
if mode == 'cpu':
    # then 40 seeds of one configuration: scales whose clip keeps T frames (copied by upsample_linear) occur among them
    for k, (policy, ts, n, c, t, h, w) in enumerate(CASES + [('cutout', 1.0, 3, 3, 16, 12, 20)] * 40):
        x = video(n, c, t, h, w, k)
        g = gan(policy, ts, c, t, h, w)
        torch.manual_seed(100 + k)
        g.run_D(x)
        ref, state_ref = g.D.seen[0], torch.get_rng_state()
        torch.manual_seed(100 + k)
        params = va.draw_params(x, policy, ts, t)
        state_ours = torch.get_rng_state()
        res.append(dict(case=(policy, ts, n, c, t, h, w), ref=ref, ours=va.apply(x, params, t), params=params,
                        same_state=torch.equal(state_ref, state_ours)))
elif mode == 'cuda':
    for k, (policy, ts, n, c, t, h, w) in enumerate(CASES):
        x0 = video(n, c, t, h, w, k, 'cuda')
        outs = []
        for installed in (False, True):
            cls = vg.LowResVideoGAN
            if installed:
                va.install(vg)
            g = gan(policy, ts, c, t, h, w)
            x = x0.clone().requires_grad_(True)
            torch.manual_seed(100 + k)
            logits = g.run_D(x)
            gx, = torch.autograd.grad(logits.sum(), [x])
            outs.append(dict(d_in=g.D.seen[0].detach().cpu(), logits=logits.detach().cpu(), gx=gx.cpu(),
                             cuda_state=torch.cuda.get_rng_state(), cpu_state=torch.get_rng_state()))
            if installed:
                cls.run_D = cls.run_D.lvg_video_augment
        res.append(dict(case=(policy, ts, n, c, t, h, w), ref=outs[0], ours=outs[1]))

    def r1_step(g, x0):
        x = x0.clone().requires_grad_(True)
        torch.manual_seed(7)
        logits = g.run_D(x)
        gx, = torch.autograd.grad(logits.sum(), [x], create_graph=True)
        (gx.square().sum() + torch.nn.functional.softplus(logits).mean()).backward()
        return x.grad

    x0 = video(8, 3, 32, 36, 64, 99, 'cuda')
    orig = vg.LowResVideoGAN.run_D
    va.install(vg)
    g = gan('color,translation,cutout', 1.0, 3, 32, 36, 64)
    r1_step(g, x0)                                            # warm-up: pinned host blocks, library load
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    dx_nosync = r1_step(g, x0)
    torch.cuda.set_sync_debug_mode(0)
    torch.use_deterministic_algorithms(True)
    det = [r1_step(g, x0).cpu() for _ in range(2)]
    vg.LowResVideoGAN.run_D = orig
    torch.use_deterministic_algorithms(False)
    res = dict(cases=res, nosync=dx_nosync.cpu(), det=det)
elif mode == 'install':
    orig = vg.LowResVideoGAN.run_D
    assert va.install(vg) == [vg.LowResVideoGAN]
    assert vg.LowResVideoGAN.run_D is not orig and vg.LowResVideoGAN.run_D.lvg_video_augment is orig
    assert va.install(vg) == [vg.LowResVideoGAN] and vg.LowResVideoGAN.run_D.lvg_video_augment is orig    # idempotent
    g = gan('color,translation,cutout', 1.0, 3, 8, 6, 10)
    assert va.install(g) == [vg.LowResVideoGAN] and vg.LowResVideoGAN.run_D.lvg_video_augment is orig
    # another class with a run_D (the super-res GAN's takes other arguments) is not reached
    assert va.install(type('SuperResVideoGAN', (), {'run_D': lambda self, lr, hr: None})()) == []
    calls = []

    def spy(self, v):
        calls.append(v.shape)
        return orig(self, v)
    # unsupported inputs reach the original method: a CPU video, a policy out of order or unknown
    patched = va._run_D(spy)
    for policy, x in (('color,translation,cutout', video(2, 3, 8, 6, 10, 0)),
                      ('cutout,color', video(2, 3, 8, 6, 10, 0)),
                      ('color,zoom', video(2, 3, 8, 6, 10, 0))):
        g = gan(policy, 1.0, 3, 8, 6, 10)
        if policy == 'color,zoom':
            try:
                patched(g, x)
            except KeyError:
                pass
        else:
            torch.manual_seed(5)
            patched(g, x)
            got = g.D.seen[-1]
            g2 = gan(policy, 1.0, 3, 8, 6, 10)
            torch.manual_seed(5)
            orig(g2, x)
            assert torch.equal(got, g2.D.seen[-1])
    assert len(calls) == 3, calls
    res = 'ok'
torch.save(res, out_file)
