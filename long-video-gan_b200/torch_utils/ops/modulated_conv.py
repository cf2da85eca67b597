"""Modulated convolutions of the two generators as ONE convolution with a shared weight and two small factor tensors.

Not a module of the reference's ``torch_utils.ops``. The reference builds the style modulation / demodulation around its
convolutions from generic tensor ops:

  modulated_conv2d            generator_sres.py:28-67    per-sample weights [N, Cout, Cin, k, k] (fp32), grouped conv
  temporal_modulated_conv3d   generator_lres.py:83-125   input * style, F.conv3d, output * demodulation

Both are  y = d * conv(a * x, w~)  with one weight w~, an input factor a[n, ci, t] and an output factor d[n, co, t]
(t = 1 for 2-D). ``a``, ``d`` and ``w~`` are computed here with ordinary differentiable torch ops, as the reference does;
the convolution runs on the wgmma engine (csrc/conv_igemm.cu): ``a`` is applied while x is re-tiled, ``d`` in the
epilogue, and the first-order backward pass is one native call (dx, dw summed over samples, the row sums that give the
gradients of a and d). Autograd carries those back through the normalisations to w, s and input_gain.

fp16 (super-res layers): x * a is rounded to fp16 when it is re-tiled, w~ is fp16 and d is applied to the fp32
accumulator; the reference instead rounds the per-sample weight w * s * d * g to fp16, so the two agree to fp16 rounding,
not bit for bit. Range: the generator clamps activations to |x| <= 256 and a = s^ * g with s^ = s / rms(s), so |x * a|
stays within a few thousand, far inside fp16's 65504 for styles of ordinary spread.

``install(model.generator_sres, model.generator_lres)`` (or a generator instance) makes an unmodified model file call
these functions. Outside the engine's envelope (CPU tensors, fp64, LVG_NATIVE_CONV=0, kernels it rejects) the functions
compute the reference's own formulation over ``conv_nd``.
"""
import math
import sys

import numpy as np
import torch

from . import conv_nd


def _plugin():
    return conv_nd._get_plugin()


def _bc(f, nd):
    """[N, C, T] factor -> broadcastable over [N, C, (T,) H, W]."""
    return f[..., None, None] if nd == 3 else f[..., None]


def _spatial_dot(u, v, nd):
    """sum over H, W of u * v, [N, C, (T,) H, W] -> [N, C, T] (T = 1 for 2-D), at least in fp32."""
    ft = torch.promote_types(u.dtype, torch.float32)
    s = (u.to(ft) * v.to(ft)).sum(dim=(-2, -1))
    return s if nd == 3 else s[..., None]


def _native(x, w, padding):
    if not conv_nd.enabled_for(x) or x.dtype not in (torch.float16, torch.float32) or x.ndim not in (4, 5):
        return False
    plug = _plugin()
    return plug.supported(x, w, 1, padding, 1, 1) and plug.modconv_supported(x, w, padding)


class _ModulatedConv(torch.autograd.Function):
    """y = d * conv(a * x, w): x [N, Cin, (T,) H, W], w [Cout, Cin, (kt,) kh, kw] (dtype of x), a [N, Cin, T], d [N, Cout, T]
    or None (fp32). First-order backward: one native call. With create_graph=True the backward pass is recorded from the
    differentiable conv_nd Functions and torch ops instead."""

    @staticmethod
    def forward(ctx, x, w, a, d, padding):
        y = _plugin().modconv_fprop(x, w, a, d, padding)
        ctx.save_for_backward(x, w, a, d, y)
        ctx.padding = padding
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, a, d, y = ctx.saved_tensors
        padding = ctx.padding
        want_dw = ctx.needs_input_grad[1] and not conv_nd._weights_off()
        if not torch.is_grad_enabled():
            dx, dw, da, dyy = _plugin().modconv_backward(x, w, a, d, y, dy, padding, want_dw=want_dw)
            dd = dyy / d if (d is not None and ctx.needs_input_grad[3]) else None
            return (dx if ctx.needs_input_grad[0] else None), dw, (da if ctx.needs_input_grad[2] else None), dd, None
        # differentiable composition (double backward through the generator)
        dx, dw, da, dd = backward_graph(x, w, a, d, dy, padding, ctx.needs_input_grad[0] or ctx.needs_input_grad[2], want_dw,
                                        d is not None and ctx.needs_input_grad[3])
        return dx, dw, da, dd, None


def backward_graph(x, w, a, d, dy, padding, want_dx_da, want_dw, want_dd):
    """(dx, dw, da, dd) of y = d * conv(a * x, w) recorded from the differentiable conv_nd Functions and torch ops, so that
    gradients of any order work (the create_graph=True backward pass); None where not wanted."""
    nd = x.ndim - 2
    dyd = dy if d is None else dy * _bc(d, nd).to(dy.dtype)
    dx = dw = da = dd = None
    if want_dx_da:
        dxp = conv_nd._ConvNdDgrad.apply(dyd, w, x.shape, padding, 1, 1)
        dx = dxp * _bc(a, nd).to(dxp.dtype)
        da = _spatial_dot(dxp, x, nd)
    if want_dw:
        dw = conv_nd._ConvNdWgrad.apply(dyd, x * _bc(a, nd).to(x.dtype), w.shape, padding, 1, 1)
    if want_dd:
        z = conv_nd._ConvNd.apply(x * _bc(a, nd).to(x.dtype), w, padding, 1, 1)
        dd = _spatial_dot(dy, z, nd)
    return dx, dw, da, dd


def modulated_conv(x, w, a, d, padding):
    """y = d * conv(a * x, w) (groups 1, stride 1) on the engine: a [N, Cin, T] and d [N, Cout, T] (or None) as fp32, T = 1
    for 2-D. Callers check the envelope (``_native``) first."""
    if x.is_cuda:
        a, d = a.float(), (None if d is None else d.float())
    return _ModulatedConv.apply(x, w, a, d, padding)


def _pad_tuple(padding, nd):
    return tuple(int(p) for p in padding) if isinstance(padding, (list, tuple)) else (int(padding),) * nd


# ---------------------------------------------------------------------------------------------------- super-res

def _demodulated(w, s, demodulate):
    if demodulate:
        w = w * w.square().mean([1, 2, 3], keepdim=True).rsqrt()
        s = s * s.square().mean().rsqrt()
    return w, s


def factors2d(w, s, gain, demodulate):
    """(a [N, Cin, 1], d [N, Cout, 1] or None) of modulated_conv2d from the normalised w and s and the expanded gain."""
    a = s if gain is None else s * gain
    d = None
    if demodulate:
        d = (s.square() @ w.square().sum(dim=[2, 3]).t() + 1e-8).rsqrt()            # [N, Cout]
    return a[..., None], None if d is None else d[..., None]


def factors(w, s, demodulate=True, input_gain=None):
    """(w~ (fp32), a, d) of ``modulated_conv2d(x, w, s, demodulate, input_gain=input_gain)``: the convolution it runs is
    d * conv(a * x, w~.to(x.dtype)) (the same torch ops, so the same autograd graph)."""
    w, s = _demodulated(w, s, demodulate)
    gain = None if input_gain is None else input_gain.expand(s.shape[0], s.shape[1])
    return (w,) + factors2d(w, s, gain, demodulate)

def modulated_conv2d(x, w, s, demodulate=True, padding=0, input_gain=None):
    """generator_sres.modulated_conv2d: x [N, Cin, H, W], w [Cout, Cin, kh, kw], s [N, Cin], input_gain [], [Cin] or
    [N, Cin]; the weight is cast to x's dtype for the convolution."""
    batch_size = int(x.shape[0])
    out_channels, in_channels, kh, kw = w.shape
    assert tuple(x.shape[:2]) == (batch_size, in_channels) and tuple(s.shape) == (batch_size, in_channels)
    w, s = _demodulated(w, s, demodulate)
    gain = None if input_gain is None else input_gain.expand(batch_size, in_channels)
    pad = _pad_tuple(padding, 2)
    wx = w.to(x.dtype)
    if _native(x, wx, pad):
        return modulated_conv(x, wx, *factors2d(w, s, gain, demodulate), pad)
    # the reference's formulation: per-sample weights, one grouped convolution
    wn = w.unsqueeze(0) * s[:, None, :, None, None]
    if demodulate:
        wn = wn * (wn.square().sum(dim=[2, 3, 4]) + 1e-8).rsqrt()[:, :, None, None, None]
    if gain is not None:
        wn = wn * gain[:, None, :, None, None]
    y = conv_nd.conv2d(x.reshape(1, -1, *x.shape[2:]), wn.reshape(-1, in_channels, kh, kw).to(x.dtype), padding=pad, groups=batch_size)
    return y.reshape(batch_size, -1, *y.shape[2:])


# ---------------------------------------------------------------------------------------------------- low-res

def temporal_factors(weight, style, demodulate=True):
    """(w~ (fp32), the normalised style, d [N, Cout, T] or None) of ``temporal_modulated_conv3d``: its convolution is
    d * conv(style * input_gain * input, w~.type(input.dtype)) (the same torch ops, so the same autograd graph)."""
    if demodulate:
        weight = weight / weight.abs().amax(dim=(1, 2, 3, 4), keepdim=True)
        style = style / style.abs().amax(dim=(1, 2), keepdim=True)
    weight = weight / math.sqrt(int(np.prod(weight.shape[1:])))
    demod = None
    if demodulate:
        demod = torch.einsum('oizyx,nit->not', weight.square(), style.square()).add(1e-8).rsqrt()
    return weight, style, demod


def temporal_modulated_conv3d(input, weight, style, input_gain=None, padding=(0, 0, 0), demodulate=True):
    """generator_lres.temporal_modulated_conv3d: input [N, Cin, T, H, W], weight [Cout, Cin, kt, kh, kw], style [N, Cin, T],
    input_gain a 0-dim tensor or None. Demodulation uses the style of output frame t only (the reference's definition),
    so the output must have the input's frame count."""
    assert input.dim() == 5
    batch_size, in_channels = input.size(0), input.size(1)
    assert weight.shape[1] == in_channels and tuple(style.shape[:2]) == (batch_size, in_channels)
    weight, style, demod = temporal_factors(weight, style, demodulate)
    if input_gain is not None:
        assert input_gain.dim() == 0
    pad = _pad_tuple(padding, 3)
    wx = weight.type(input.dtype)
    t_out = input.shape[2] + 2 * pad[0] - weight.shape[2] + 1
    if _native(input, wx, pad) and t_out == input.shape[2]:
        a = style if input_gain is None else style * input_gain
        return modulated_conv(input, wx, a, demod, pad)
    # the reference's formulation over conv_nd
    if input_gain is not None:
        input = input * input_gain
    output = conv_nd.conv3d(input * style[..., None, None].type(input.dtype), wx, padding=pad)
    if demodulate:
        output = output * demod[..., None, None].type(output.dtype)
    return output


# ---------------------------------------------------------------------------------------------------- install

_OURS = {'modulated_conv2d': modulated_conv2d, 'temporal_modulated_conv3d': temporal_modulated_conv3d}


def install(*targets):
    """Replace ``modulated_conv2d`` / ``temporal_modulated_conv3d`` in reference model modules by the functions above.

    ``targets``: modules (``model.generator_sres``, ``model.generator_lres``) or ``nn.Module`` instances; for an instance
    every submodule's defining module ``sys.modules[type(m).__module__]`` is patched, which reaches unpickled generators
    whose class source ``persistence`` executed into a module of its own. Only attributes that are the reference functions
    (same name) or already these are replaced; ``F`` is left alone. Idempotent. Returns the modules patched."""
    mods = []
    for t in targets:
        if isinstance(t, torch.nn.Module):
            for m in t.modules():
                mod = sys.modules.get(type(m).__module__)
                if mod is not None:
                    mods.append(mod)
        else:
            mods.append(t)
    done = []
    for mod in mods:
        if any(mod is m for m in done):
            continue
        hit = False
        for name, ours in _OURS.items():
            cur = getattr(mod, name, None)
            if cur is ours or (callable(cur) and getattr(cur, '__name__', None) == name):
                setattr(mod, name, ours)
                hit = True
        if hit:
            done.append(mod)
    return done
