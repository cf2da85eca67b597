"""Input augmentation of the low-res discriminator as one native, deterministic op.

Not a module of the reference's ``torch_utils.ops``. ``LowResVideoGAN.run_D`` (video_gan_lres.py:237-266) feeds D

  DiffAugment(video, policy)                                      color, translation, cutout (diff_augment.py)
  then, with temp_scale_augment > 0, per sample: F.interpolate along T by 2^u, a random zero pad p0, a crop at i0

For sample n this is an affine map of the video x [N, C, T, H, W] -> y [N, C, T_out, H, W] (DESIGN.md 7d):

  z = kappa sigma x + kappa (1 - sigma) m + (1 - kappa) mu + beta       m: channel mean per pixel, mu: mean of the sample
  y[t, h, w] = mask(h, w) * ((1 - l1) z[h1] + l1 z[h2])[h + dh, w + dw]  for u = t + off in [0, L), 0 elsewhere

(the reference's contrast mean is mu + beta, so its two means fold into mu). ``draw_params`` makes the reference's random
draws, in its order, and packs them as fp32 [N, 12]: beta, sigma, kappa, dh, dw, r0, r1, c0, c1, r, L, off.
``apply`` runs lvg_video_augment / lvg_video_augment_adjoint for CUDA fp32 tensors and the torch composition
``_reference`` for every other tensor; gradients of any order (the adjoint's backward is the linear forward).
``install(...)`` makes an unmodified ``LowResVideoGAN.run_D`` use it.
"""
import math

import torch

from .. import custom_ops
from . import _install

NPAR = 12
STEPS = ('color', 'translation', 'cutout')
_BIG = 3.0e38


def steps_of(policy):
    """The DiffAugment steps a policy string names, as (color, translation, cutout) flags, or None when the policy is not a
    subset of those three in that order (the op keeps the reference's order of steps)."""
    names = policy.split(',') if policy else []
    if any(n not in STEPS for n in names) or len(set(names)) != len(names) or names != sorted(names, key=STEPS.index):
        return None
    return tuple(s in names for s in STEPS)


def draw_params(video, policy, temp_scale_augment, seq_length):
    """The per-sample parameters of ``run_D``'s augmentation, from exactly the RNG calls the reference makes: on the video's
    device the three ``torch.rand(N, 1, 1, 1)`` of the color step, the two ``torch.randint`` of the translation and the two
    of the cutout; on the CPU, per sample, ``uniform_`` for the scale exponent, then ``randint`` for the pad p0 and for the
    crop i0. Returns fp32 [N, 12] on the video's device; the host-side values reach it in one non-blocking copy from pinned
    memory, and nothing waits for the device."""
    steps = steps_of(policy)
    if steps is None:
        raise ValueError(f'video_augment: unsupported policy {policy!r}')
    color, translation, cutout = steps
    n, _, t, h, w = video.shape
    dev = video.device
    # rows 0..n-1: host-side values; rows n..n+3: scale, shift, lower and upper bound of each column's affine map from
    # the raw device draws (brightness rand - 0.5, saturation 2 rand, contrast rand + 0.5; cutout: clamped rectangle)
    host = torch.zeros([n + 4, NPAR], dtype=torch.float32, pin_memory=video.is_cuda)
    host[:n, 1] = host[:n, 2] = 1.0                    # sigma = kappa = 1 without the color step
    host[:n, 6] = host[:n, 8] = -1.0                   # empty cutout
    host[n] = 1.0
    host[n + 2] = -_BIG
    host[n + 3] = _BIG
    pieces = []
    if color:
        draws = [torch.rand(n, 1, 1, 1, dtype=video.dtype, device=dev) for _ in range(3)]
        pieces.append(torch.cat(draws, 1).view(n, 3).float())
        host[n, 1] = 2.0
        host[n + 1, 0], host[n + 1, 2] = -0.5, 0.5
    else:
        pieces.append(None)
    if translation:
        shift = round(max(h, w) * 0.25)
        tx = torch.randint(-shift, shift + 1, size=[n, 1, 1], device=dev)
        ty = torch.randint(-shift, shift + 1, size=[n, 1, 1], device=dev)
        pieces.append(torch.cat([tx, ty], 1).view(n, 2))
    else:
        pieces.append(None)
    if cutout:
        ch, cw = int(h * 0.5 + 0.5), int(w * 0.5 + 0.5)
        ox = torch.randint(0, h + (1 - ch % 2), size=[n, 1, 1], device=dev)
        oy = torch.randint(0, w + (1 - cw % 2), size=[n, 1, 1], device=dev)
        pieces.append(torch.cat([ox, ox, oy, oy], 1).view(n, 4))
        host[n + 1, 5:9] = torch.tensor([-(ch // 2), ch - 1 - ch // 2, -(cw // 2), cw - 1 - cw // 2], dtype=torch.float32)
        host[n + 2, 5:9] = 0.0
        host[n + 3, 5:7] = h - 1
        host[n + 3, 7:9] = w - 1
    else:
        pieces.append(None)
    host[:n, 9] = 1.0
    host[:n, 10] = t
    if temp_scale_augment > 0:
        for i in range(n):
            scale = 2 ** torch.empty(()).uniform_(-temp_scale_augment, temp_scale_augment)
            length = math.floor(t * float(scale))           # F.interpolate's output size for a scale factor
            if length < 1:
                raise RuntimeError(f'video_augment: a clip of {t} frames scaled by {float(scale)} is empty')
            p0 = torch.randint(max(0, seq_length - length) + 1, ()).item()
            p1 = max(0, seq_length - length - p0)
            i0 = torch.randint(p0 + length + p1 - seq_length + 1, ()).item()
            # rounded to fp32, as upsample_linear's scale; a clip that keeps its length is copied (upsample_linear's
            # shortcut for equal sizes), whatever the scale
            host[i, 9] = 1.0 / float(scale) if length != t else 1.0
            host[i, 10] = length
            host[i, 11] = i0 - p0
    dev_host = host.to(dev, non_blocking=True)
    cols = [(0, 3), (3, 5), (5, 9)]
    raw = torch.cat([dev_host[:n, a:b] if p is None else p for p, (a, b) in zip(pieces, cols)] + [dev_host[:n, 9:]], 1)
    return torch.addcmul(dev_host[n + 1], raw, dev_host[n]).clamp_(dev_host[n + 2], dev_host[n + 3])


# ---------------------------------------------------------------------------------------------------- torch composition

def _reference(x, params, t_out, linear=False):
    """The map of the module docstring in torch ops, in x's dtype (the index arithmetic of the temporal taps in fp32, as
    upsample_linear's). Differentiable; the oracle of the tests and the path of CPU and non-fp32 tensors."""
    n, c, t, h, w = x.shape
    p = params.to(x.device, torch.float32)
    col = lambda k: p[:, k].to(x.dtype).view(n, 1, 1, 1, 1)          # noqa: E731
    beta, sigma, kappa = col(0), col(1), col(2)
    dh, dw, r0, r1, c0, c1 = p[:, 3:9].round().long().unbind(1)
    r, length, off = p[:, 9], p[:, 10].round().long(), p[:, 11].round().long()
    z = kappa * sigma * x + kappa * (1 - sigma) * x.mean(1, keepdim=True) + (1 - kappa) * x.mean((1, 2, 3, 4), keepdim=True)
    if not linear:
        z = z + beta
    # translation and cutout: output pixel (oh, ow) reads (oh + dh, ow + dw)
    oh = torch.arange(h, device=x.device)[None]
    ow = torch.arange(w, device=x.device)[None]
    sh, sw = oh + dh[:, None], ow + dw[:, None]
    keep_h, keep_w = (sh >= 0) & (sh < h), (sw >= 0) & (sw < w)
    cut = ((oh >= r0[:, None]) & (oh <= r1[:, None]))[:, :, None] & ((ow >= c0[:, None]) & (ow <= c1[:, None]))[:, None, :]
    mask = keep_h[:, :, None] & keep_w[:, None, :] & ~cut                                    # [n, h, w]
    ni = torch.arange(n, device=x.device).view(n, 1, 1)
    z = z[ni, :, :, sh.clamp(0, h - 1)[:, :, None], sw.clamp(0, w - 1)[:, None, :]]         # [n, h, w, c, t]
    z = z.permute(0, 3, 4, 1, 2) * mask[:, None, None].to(x.dtype)
    # temporal taps of clip frame u = t + off
    u = torch.arange(t_out, device=x.device)[None] + off[:, None]
    src = (r[:, None] * (u.float() + 0.5) - 0.5).clamp_min(0)
    h1 = src.long().clamp(0, t - 1)
    l1 = (src - h1.float()).to(x.dtype)
    h2 = (h1 + 1).clamp(max=t - 1)
    keep_t = ((u >= 0) & (u < length[:, None])).to(x.dtype)
    take = lambda i: z.gather(2, i.view(n, 1, t_out, 1, 1).expand(n, c, t_out, h, w))     # noqa: E731
    wt = lambda v: v.view(n, 1, t_out, 1, 1)                                                  # noqa: E731
    return (wt(1 - l1) * take(h1) + wt(l1) * take(h2)) * wt(keep_t)


def _reference_adjoint(dy, params, t_in):
    """A^T dy of the linear part: the vector-Jacobian product of the linear composition (exact, it is linear)."""
    n, c, _, h, w = dy.shape
    with torch.enable_grad():
        x0 = torch.zeros([n, c, t_in, h, w], dtype=dy.dtype, device=dy.device, requires_grad=True)
        y = _reference(x0, params, dy.shape[2], linear=True)
        return torch.autograd.grad(y, [x0], dy)[0]


def _native(x):
    return x.is_cuda and x.dtype == torch.float32


def _plugin():
    return custom_ops.get_plugin('video_augment_plugin')


def _forward(x, params, t_out, linear):
    if _native(x):
        y = _plugin().run(x, params, t_out, linear=linear)
        if y is None:
            raise RuntimeError(f'video_augment: no kernel for {x.shape[1]} channels (at most 4)')
        return y
    return _reference(x, params, t_out, linear)


def _adjoint(dy, params, t_in):
    if _native(dy):
        dx = _plugin().run(dy, params, t_in, adjoint=True)
        if dx is None:
            raise RuntimeError(f'video_augment: no kernel for {dy.shape[1]} channels (at most 4)')
        return dx
    return _reference_adjoint(dy, params, t_in)


class _Augment(torch.autograd.Function):
    """y = A x (+ beta unless linear); backward A^T, whose backward is the linear A again. Saves only the parameters."""

    @staticmethod
    def forward(ctx, x, params, t_out, linear):
        ctx.save_for_backward(params)
        ctx.t_in = x.shape[2]
        return _forward(x, params, t_out, linear)

    @staticmethod
    def backward(ctx, dy):
        params, = ctx.saved_tensors
        dx = _AugmentAdjoint.apply(dy, params, ctx.t_in) if ctx.needs_input_grad[0] else None
        return dx, None, None, None


class _AugmentAdjoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dy, params, t_in):
        ctx.save_for_backward(params)
        ctx.t_out = dy.shape[2]
        return _adjoint(dy, params, t_in)

    @staticmethod
    def backward(ctx, ddx):
        params, = ctx.saved_tensors
        return (_Augment.apply(ddx, params, ctx.t_out, True) if ctx.needs_input_grad[0] else None), None, None


def apply(video, params, seq_length):
    """The augmented video [N, C, seq_length, H, W] for parameters from ``draw_params``. Gradients of any order with respect
    to ``video``."""
    return _Augment.apply(video, params.detach(), int(seq_length), False)


def augment(video, policy='color,translation,cutout', temp_scale_augment=0.0, seq_length=None):
    """``draw_params`` + ``apply``: what ``run_D`` feeds D."""
    seq_length = video.shape[2] if seq_length is None else seq_length
    return apply(video, draw_params(video, policy, temp_scale_augment, seq_length), seq_length)


# ---------------------------------------------------------------------------------------------------- install

def applies(video, policy, temp_scale_augment, seq_length):
    """The native op takes run_D's input: a CUDA fp32 video, a policy ``steps_of`` accepts, at most 4 channels (the library's
    LVG_UNSUPPORTED), and no scale that could empty the clip."""
    if not (video.is_cuda and video.dtype == torch.float32 and video.ndim == 5) or steps_of(policy) is None:
        return False
    if temp_scale_augment > 0 and seq_length * 2.0 ** -temp_scale_augment < 2:
        return False
    n, c, t, h, w = video.shape
    return _plugin().workspace(n, c, t, h, w, seq_length) >= 0


def _run_D(orig):
    g = _install.reference_function(orig).__globals__

    def run_D(self, video):
        if not applies(video, self.diffaug_policy, self.temp_scale_augment, self.seq_length):
            return orig(self, video)
        g['misc'].assert_shape(video, (None, self.channels, self.seq_length, self.height, self.width))
        params = draw_params(video, self.diffaug_policy, self.temp_scale_augment, self.seq_length)
        return self.D(apply(video, params, self.seq_length))
    return run_D


def install(*targets):
    """Make ``LowResVideoGAN.run_D`` build D's input with this op. ``targets``: the module ``model.video_gan_lres`` or
    LowResVideoGAN instances, found by ``_install.find_classes``. Inputs ``applies`` rejects run the original method.
    Idempotent; the original stays reachable as ``.run_D.lvg_video_augment``. Returns the patched classes."""
    classes = _install.find_classes(targets, 'LowResVideoGAN')
    for cls in classes:
        _install.wrap(cls, 'run_D', 'lvg_video_augment', _run_D)
    return classes
