"""ADA's ``AugmentPipe`` of the super-res step as one native, deterministic op without host synchronisation.

Not a module of the reference's ``torch_utils.ops``. ``AugmentPipe.forward`` (ada_augment.py:180-439) with
``imgfilter == 0`` and ``cutout == 0`` is, for sample n of a video x [N, 3, T, H, W], the affine map (DESIGN.md 7e)

  y = C_n[:3,:3] . downsample2d(grid_sample(upsample2d(reflect_pad(x, margins), Hz), affine_grid(theta_n)), Hz)
      + C_n[:3,3] + sigma_n * noise

over the planes of one frame's 3 channels; without geometric steps the resampling is the identity. ``draw_params`` makes
the reference's random draws in its order and builds the margins, theta_n and C_n with its op sequence on the video's
device, packed as fp32 [N, 23]: mx0, my0, mx1, my1, theta[2][3], C[3][4], sigma. ``apply`` runs lvg_augment_pipe /
lvg_augment_pipe_adjoint for CUDA fp32 tensors and the torch composition ``_reference`` for every other tensor; gradients
of any order (the adjoint's backward is the linear forward). ``install(...)`` makes an unmodified ``AugmentPipe.forward``
use it.
"""
import numpy as np
import torch

from .. import custom_ops
from . import _install, grid_sample_gradfix, upfirdn2d

NPAR = 23
GEOM = 1            # LVG_AUGMENT_PIPE_GEOM
LINEAR = 2          # LVG_AUGMENT_PIPE_LINEAR
GEOM_STEPS = ('xflip', 'rotate90', 'xint', 'scale', 'rotate', 'aniso', 'xfrac')

_constants = {}


def _const(value, device, shape=None):
    """An fp32 constant on ``device`` (cached), built as the reference builds its constants: from a float64 numpy array."""
    value = np.asarray(value)
    key = (value.shape, value.tobytes(), None if shape is None else tuple(shape), str(device))
    t = _constants.get(key)
    if t is None:
        t = torch.as_tensor(value.copy(), dtype=torch.float32, device=device)
        if shape is not None:
            t, _ = torch.broadcast_tensors(t, torch.empty(shape))
        t = _constants[key] = t.contiguous()
    return t


def _matrix(*rows, device=None):
    elems = [x for row in rows for x in row]
    ref = [x for x in elems if isinstance(x, torch.Tensor)]
    if not ref:
        return _const(np.asarray(rows), device)
    elems = [x if isinstance(x, torch.Tensor) else _const(x, ref[0].device, ref[0].shape) for x in elems]
    return torch.stack(elems, dim=-1).reshape(ref[0].shape + (len(rows), -1))


def _translate2d(tx, ty, **kw):
    return _matrix([1, 0, tx], [0, 1, ty], [0, 0, 1], **kw)


def _scale2d(sx, sy, **kw):
    return _matrix([sx, 0, 0], [0, sy, 0], [0, 0, 1], **kw)


def _rotate2d(theta, **kw):
    return _matrix([torch.cos(theta), torch.sin(-theta), 0], [torch.sin(theta), torch.cos(theta), 0], [0, 0, 1], **kw)


def _translate2d_inv(tx, ty, **kw):
    return _translate2d(-tx, -ty, **kw)


def _scale2d_inv(sx, sy, **kw):
    return _scale2d(1 / sx, 1 / sy, **kw)


def _rotate2d_inv(theta, **kw):
    return _rotate2d(-theta, **kw)


def _translate3d(tx, ty, tz, **kw):
    return _matrix([1, 0, 0, tx], [0, 1, 0, ty], [0, 0, 1, tz], [0, 0, 0, 1], **kw)


def _scale3d(sx, sy, sz, **kw):
    return _matrix([sx, 0, 0, 0], [0, sy, 0, 0], [0, 0, sz, 0], [0, 0, 0, 1], **kw)


def _rotate3d(v, theta, **kw):
    vx, vy, vz = v[..., 0], v[..., 1], v[..., 2]
    s, c = torch.sin(theta), torch.cos(theta)
    cc = 1 - c
    return _matrix([vx * vx * cc + c, vx * vy * cc - vz * s, vx * vz * cc + vy * s, 0],
                   [vy * vx * cc + vz * s, vy * vy * cc + c, vy * vz * cc - vx * s, 0],
                   [vz * vx * cc - vy * s, vz * vy * cc + vx * s, vz * vz * cc + c, 0],
                   [0, 0, 0, 1], **kw)


def flags_of(pipe):
    """GEOM when the pipe has a geometric step (the reference's ``G_inv is not I_3``)."""
    return GEOM if any(getattr(pipe, s) > 0 for s in GEOM_STEPS) else 0


def draw_params(pipe, video):
    """The per-sample parameters of ``pipe.forward(video)``, from exactly the RNG calls the reference makes, in its order,
    shapes, dtypes and devices (the draws that ``p`` masks to identity and the noise tensor included). The margins
    (``ceil().to(int32)``), theta and C come from the reference's torch op sequence on the video's device, with the
    margins kept there. Returns (params fp32 [N, 23], noise [N, C, T, H, W] or None, flags); nothing waits for the device."""
    n, c, t, h, w = video.shape
    dev = video.device
    p = pipe.p
    i3 = torch.eye(3, device=dev)
    g = i3
    if pipe.xflip > 0:
        i = torch.floor(torch.rand([n], device=dev) * 2)
        i = torch.where(torch.rand([n], device=dev) < pipe.xflip * p, i, torch.zeros_like(i))
        g = g @ _scale2d_inv(1 - 2 * i, 1)
    if pipe.rotate90 > 0:
        i = torch.floor(torch.rand([n], device=dev) * 4)
        i = torch.where(torch.rand([n], device=dev) < pipe.rotate90 * p, i, torch.zeros_like(i))
        g = g @ _rotate2d_inv(-np.pi / 2 * i)
    if pipe.xint > 0:
        s = (torch.rand([n, 2], device=dev) * 2 - 1) * pipe.xint_max
        s = torch.where(torch.rand([n, 1], device=dev) < pipe.xint * p, s, torch.zeros_like(s))
        g = g @ _translate2d_inv(torch.round(s[:, 0] * w), torch.round(s[:, 1] * h))
    if pipe.scale > 0:
        s = torch.exp2(torch.randn([n], device=dev) * pipe.scale_std)
        s = torch.where(torch.rand([n], device=dev) < pipe.scale * p, s, torch.ones_like(s))
        g = g @ _scale2d_inv(s, s)
    p_rot = 1 - torch.sqrt((1 - pipe.rotate * p).clamp(0, 1))
    if pipe.rotate > 0:
        th = (torch.rand([n], device=dev) * 2 - 1) * np.pi * pipe.rotate_max
        th = torch.where(torch.rand([n], device=dev) < p_rot, th, torch.zeros_like(th))
        g = g @ _rotate2d_inv(-th)
    if pipe.aniso > 0:
        s = torch.exp2(torch.randn([n], device=dev) * pipe.aniso_std)
        s = torch.where(torch.rand([n], device=dev) < pipe.aniso * p, s, torch.ones_like(s))
        g = g @ _scale2d_inv(s, 1 / s)
    if pipe.rotate > 0:
        th = (torch.rand([n], device=dev) * 2 - 1) * np.pi * pipe.rotate_max
        th = torch.where(torch.rand([n], device=dev) < p_rot, th, torch.zeros_like(th))
        g = g @ _rotate2d_inv(-th)
    if pipe.xfrac > 0:
        s = torch.randn([n, 2], device=dev) * pipe.xfrac_std
        s = torch.where(torch.rand([n, 1], device=dev) < pipe.xfrac * p, s, torch.zeros_like(s))
        g = g @ _translate2d_inv(s[:, 0] * w, s[:, 1] * h)

    flags = flags_of(pipe)
    geo = torch.zeros([n, 10], device=dev)
    if flags & GEOM:
        cx, cy = (w - 1) / 2, (h - 1) / 2
        cp = _matrix([-cx, -cy, 1], [cx, -cy, 1], [cx, cy, 1], [-cx, cy, 1], device=dev)
        cp = g @ cp.t()
        hz_pad = pipe.Hz_geom.shape[0] // 4
        margin = cp[:, :2, :].permute(1, 0, 2).flatten(1)
        margin = torch.cat([-margin, margin]).max(dim=1).values
        margin = margin + _const([hz_pad * 2 - cx, hz_pad * 2 - cy] * 2, dev)
        margin = margin.max(_const([0, 0] * 2, dev))
        margin = margin.min(_const([w - 1, h - 1] * 2, dev))
        margins = margin.ceil().to(torch.int32)
        mx0, my0, mx1, my1 = margins
        g = _translate2d((mx0 - mx1) / 2, (my0 - my1) / 2) @ g
        g = _scale2d(2, 2, device=dev) @ g @ _scale2d_inv(2, 2, device=dev)
        g = _translate2d(-0.5, -0.5, device=dev) @ g @ _translate2d_inv(-0.5, -0.5, device=dev)
        # the reference's scale2d(2 / u.shape[3], 2 / u.shape[2]) from the device-resident margins: the float64 quotient
        # rounded to fp32, as its constant is
        uw, uh = 2 * (w + mx0 + mx1), 2 * (h + my0 + my1)
        su = _scale2d((2 / uw.double()).float(), (2 / uh.double()).float())
        sv = _scale2d_inv(2 / ((w + hz_pad * 2) * 2), 2 / ((h + hz_pad * 2) * 2), device=dev)
        g = su @ g @ sv
        geo = torch.cat([margins.float().expand(n, 4), g[:, :2, :].reshape(n, 6)], 1)

    i4 = torch.eye(4, device=dev)
    cm = i4
    if pipe.brightness > 0:
        b = torch.randn([n], device=dev) * pipe.brightness_std
        b = torch.where(torch.rand([n], device=dev) < pipe.brightness * p, b, torch.zeros_like(b))
        cm = _translate3d(b, b, b) @ cm
    if pipe.contrast > 0:
        s = torch.exp2(torch.randn([n], device=dev) * pipe.contrast_std)
        s = torch.where(torch.rand([n], device=dev) < pipe.contrast * p, s, torch.ones_like(s))
        cm = _scale3d(s, s, s) @ cm
    v = _const(np.asarray([1, 1, 1, 0]) / np.sqrt(3), dev)
    if pipe.lumaflip > 0:
        i = torch.floor(torch.rand([n, 1, 1], device=dev) * 2)
        i = torch.where(torch.rand([n, 1, 1], device=dev) < pipe.lumaflip * p, i, torch.zeros_like(i))
        cm = (i4 - 2 * v.ger(v) * i) @ cm
    if pipe.hue > 0 and c > 1:
        th = (torch.rand([n], device=dev) * 2 - 1) * np.pi * pipe.hue_max
        th = torch.where(torch.rand([n], device=dev) < pipe.hue * p, th, torch.zeros_like(th))
        cm = _rotate3d(v, th) @ cm
    if pipe.saturation > 0 and c > 1:
        s = torch.exp2(torch.randn([n, 1, 1], device=dev) * pipe.saturation_std)
        s = torch.where(torch.rand([n, 1, 1], device=dev) < pipe.saturation * p, s, torch.ones_like(s))
        cm = (v.ger(v) + (i4 - v.ger(v)) * s) @ cm
    cm = cm.expand(n, 4, 4)[:, :3, :].reshape(n, 12)

    noise = None
    sigma = torch.zeros([n, 1], device=dev)
    if pipe.noise > 0:
        sg = torch.randn([n, 1, 1, 1], device=dev).abs() * pipe.noise_std
        sg = torch.where(torch.rand([n, 1, 1, 1], device=dev) < pipe.noise * p, sg, torch.zeros_like(sg))
        noise = torch.randn([n, c * t, h, w], device=dev).view(n, c, t, h, w)
        sigma = sg.view(n, 1)
    return torch.cat([geo, cm, sigma], 1), noise, flags


# ---------------------------------------------------------------------------------------------------- torch composition

def _margins(params):
    return [int(v) for v in params[0, :4].round().tolist()]


def _reference(x, params, noise, f, flags, linear=False):
    """The map of the module docstring in torch ops (reflect pad, upfirdn2d, affine_grid + grid_sample, upfirdn2d, colour,
    noise), in x's dtype. Differentiable; the oracle of the tests and the path of CPU and non-fp32 tensors (it reads the
    margins on the host)."""
    n, c, t, h, w = x.shape
    p = params.to(x.device, x.dtype)
    y = x.reshape(n, c * t, h, w)
    if flags & GEOM:
        mx0, my0, mx1, my1 = _margins(params)
        hz_pad = f.shape[0] // 4
        fx = f.to(x.device)
        y = torch.nn.functional.pad(y, [mx0, mx1, my0, my1], mode='reflect')
        y = upfirdn2d.upsample2d(y, fx, up=2)
        grid = torch.nn.functional.affine_grid(p[:, 4:10].view(n, 2, 3), [n, c * t, (h + hz_pad * 2) * 2, (w + hz_pad * 2) * 2],
                                               align_corners=False)
        y = grid_sample_gradfix.grid_sample(y, grid)
        y = upfirdn2d.downsample2d(y, fx, down=2, padding=-hz_pad * 2, flip_filter=True)
    cm = p[:, 10:22].view(n, 3, 4)
    y = cm[:, :, :3] @ y.reshape(n, c, t * h * w)
    if not linear:
        y = y + cm[:, :, 3:]
        if noise is not None:
            y = y.reshape(n, c * t, h, w) + noise.reshape(n, c * t, h, w).to(x.dtype) * p[:, 22].view(n, 1, 1, 1)
    return y.reshape(n, c, t, h, w)


def _reference_adjoint(dy, params, f, flags):
    """A^T dy of the linear part: the vector-Jacobian product of the linear composition (exact, it is linear)."""
    with torch.enable_grad():
        x0 = torch.zeros(dy.shape, dtype=dy.dtype, device=dy.device, requires_grad=True)
        y = _reference(x0, params, None, f, flags, linear=True)
        return torch.autograd.grad(y, [x0], dy)[0]


def _native(x):
    return x.is_cuda and x.dtype == torch.float32


def _plugin():
    return custom_ops.get_plugin('augment_pipe_plugin')


def _run(src, params, noise, f, flags, adjoint):
    out = _plugin().run(src, params, f, noise, flags, adjoint=adjoint)
    if out is None:
        raise RuntimeError(f'augment_pipe: no kernel for {src.shape[1]} channels and {f.numel()} filter taps (3 and 12)')
    return out


class _Augment(torch.autograd.Function):
    """y = A x (+ C[:3,3] and the noise unless linear); backward A^T, whose backward is the linear A again. Saves only the
    parameters and the filter."""

    @staticmethod
    def forward(ctx, x, params, noise, f, flags, linear):
        ctx.save_for_backward(params, f)
        ctx.flags = flags
        if _native(x):
            return _run(x, params, None if linear else noise, f, flags | (LINEAR if linear else 0), False)
        return _reference(x, params, noise, f, flags, linear)

    @staticmethod
    def backward(ctx, dy):
        params, f = ctx.saved_tensors
        dx = _AugmentAdjoint.apply(dy, params, f, ctx.flags) if ctx.needs_input_grad[0] else None
        return dx, None, None, None, None, None


class _AugmentAdjoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dy, params, f, flags):
        ctx.save_for_backward(params, f)
        ctx.flags = flags
        if _native(dy):
            return _run(dy.contiguous(), params, None, f, flags, True)
        return _reference_adjoint(dy, params, f, flags)

    @staticmethod
    def backward(ctx, ddx):
        params, f = ctx.saved_tensors
        return (_Augment.apply(ddx, params, None, f, ctx.flags, True) if ctx.needs_input_grad[0] else None), None, None, None


def apply(video, params, noise, f, flags):
    """The augmented video for parameters from ``draw_params`` (``f``: the pipe's ``Hz_geom``). Gradients of any order
    with respect to ``video``."""
    return _Augment.apply(video, params.detach(), None if noise is None else noise.detach(), f.detach(), int(flags), False)


def augment(pipe, video):
    """``draw_params`` + ``apply``: what the installed ``pipe.forward(video)`` returns."""
    params, noise, flags = draw_params(pipe, video)
    return apply(video, params, noise, pipe.Hz_geom, flags)


# ---------------------------------------------------------------------------------------------------- install

def applies(pipe, video, debug_percentile=None):
    """The native op takes the call: a CUDA fp32 5-D video with 3 channels, no image-space filtering, no cutout, no
    ``debug_percentile``, and a 12-tap ``Hz_geom``. Both super-res pipes (``video_gan_sres.py:110-136``) qualify."""
    if debug_percentile is not None or not (isinstance(video, torch.Tensor) and video.is_cuda and video.dtype == torch.float32
                                            and video.ndim == 5):
        return False
    if pipe.imgfilter != 0 or pipe.cutout != 0:
        return False
    f = pipe.Hz_geom
    if f.ndim != 1 or f.numel() != 12 or f.device != video.device or f.dtype != torch.float32:
        return False
    n, c, t, h, w = video.shape
    return _plugin().workspace(n, c, t, h, w, flags_of(pipe)) >= 0


def _forward(orig):
    def forward(self, videos, debug_percentile=None):
        if not applies(self, videos, debug_percentile):
            return orig(self, videos, debug_percentile)
        return augment(self, videos)
    return forward


def install(*targets):
    """Make ``AugmentPipe.forward`` run this op. ``targets``: the module ``model.ada_augment`` or ``model.video_gan_sres``,
    or pipes and modules holding them, found by ``_install.find_classes``. Calls ``applies`` rejects run the original
    method. Idempotent; the original stays reachable as ``.forward.lvg_augment_pipe``. Returns the patched classes."""
    classes = _install.find_classes(targets, 'AugmentPipe')
    for cls in classes:
        _install.wrap(cls, 'forward', 'lvg_augment_pipe', _forward)
    return classes
