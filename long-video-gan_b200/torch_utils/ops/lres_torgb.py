"""The low-res generator's ToRGB layer as one native op.

Not a module of the reference's ``torch_utils.ops``. ``ToRGB.forward`` (generator_lres.py:618-641) makes several full
passes over its input for a 3-channel output: the magnitude statistic (``MagnitudeEMA``: ``square()`` writes a tensor the
size of the input, ``mean()`` reads it), ``input * gain``, ``input * style``, the 1x1x1 convolution and ``bias_act``.
``lres_torgb`` computes

  y = dtype(clamp(dtype(sum_c w[o][c] a[n][c][t] r(x[c])) + dtype(b), +-clamp))     w = weight / sqrt(cin), a = style * gain

in one pass over x on the CUDA cores (csrc/lres_torgb.cu: lvg_lres_torgb_*), with r() the rounding of ``x.type(dtype)``
applied in registers: x is read once in its own dtype and never cast or copied. The products are summed in fp32, so y
agrees with the reference to one rounding of the layer dtype, not bit for bit. The first-order backward is one pass over x
and dy (dx, and the per-plane Gram sums that give da, dw and db, folded in a fixed order: bitwise reproducible); only y is
saved, for bias_act's clamp rule. With create_graph=True the backward is recorded from the reference formulation
(``temporal_modulated_conv3d``'s conv_nd path, then ``bias_act``), so gradients of any order work.

A forward pass that updates the magnitude EMA and records no backward (``update_D``'s generated pass) takes the statistic
from the same pass: the kernel writes u = sum_c w a r(x) in fp32 and a fixed-order sum of r(x)^2; the EMA is updated on the
device as ``MagnitudeEMA.forward`` does it, and a finishing kernel applies the new gain, the bias and the clamp. There is no
host synchronisation.

``install(...)`` makes an unmodified ``ToRGB.forward`` run ``layer_forward`` in the calls ``_takes`` routes to it (DESIGN.md
7l); every other call runs the method the wrapper replaced.
"""
import math

import numpy as np
import torch

from .. import custom_ops
from . import _install, bias_act, conv_nd

_MODES = ('backward', 'stat', 'forward')    # the calls install routes to the op (DESIGN.md 7l)


def _plugin():
    return custom_ops.get_plugin('lres_torgb_plugin')


def supported(x, dtype, weight_shape):
    """The kernels take the call: x [N, Cin, T, H, W] on CUDA in fp16 / fp32, the layer dtype fp16 / fp32 and a [3, Cin,
    1, 1, 1] weight (size query of lvg_lres_torgb), native convolutions not switched off (LVG_NATIVE_CONV=0)."""
    if not (isinstance(x, torch.Tensor) and x.ndim == 5 and conv_nd.enabled_for(x) and len(weight_shape) == 5):
        return False
    if x.dtype not in (torch.float16, torch.float32) or dtype not in (torch.float16, torch.float32):
        return False
    n, cin, t, h, w = x.shape
    if int(weight_shape[1]) != cin:
        return False
    return _plugin().workspace(x.dtype, dtype, n, cin, t, h, w, int(weight_shape[0]), tuple(weight_shape[2:])) >= 0


def composition(x, w, a, b, dtype, clamp):
    """The reference formulation the op replaces: ``temporal_modulated_conv3d(demodulate=False)``'s conv_nd path with the
    gain folded into a, then ``bias_act``. x [N, Cin, T, H, W], w [3, Cin] and a [N, Cin, T] fp32, b [3]."""
    xd = x.type(dtype)
    u = conv_nd.conv3d(xd * a[..., None, None].type(dtype), w.type(dtype)[:, :, None, None, None])
    return bias_act.bias_act(u, b.type(dtype), act='linear', clamp=clamp)


class _LresTorgb(torch.autograd.Function):
    """y = dtype(clamp(dtype(sum_c w a r(x)) + dtype(b))): x [N, Cin, T, H, W] (fp16 / fp32), w [3, Cin], a [N, Cin, T] and
    b [3] fp32. Saves y (bias_act's clamp rule)."""

    @staticmethod
    def forward(ctx, x, w, a, b, dtype, clamp):
        y = _plugin().fprop(x, w, a, b, dtype, clamp)
        ctx.save_for_backward(x, w, a, b, y)
        ctx.dtype, ctx.clamp = dtype, clamp
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, a, b, y = ctx.saved_tensors
        need = ctx.needs_input_grad
        if not torch.is_grad_enabled():
            dx, dw, da, db = _plugin().backward(x, w, a, y, dy, ctx.dtype, ctx.clamp, want_dx=need[0],
                                                want_dw=need[1] and not conv_nd._weights_off(), want_db=need[3])
            return dx, dw, (da if need[2] else None), db, None, None
        # differentiable composition (double backward through the generator)
        inputs = [(i, v) for i, v in ((0, x), (1, w), (2, a), (3, b)) if need[i]]
        with torch.enable_grad():
            yr = composition(x, w, a, b, ctx.dtype, ctx.clamp)
            grads = torch.autograd.grad(yr, [v for _, v in inputs], dy, create_graph=True, allow_unused=True)
        out = [None] * 6
        for (i, _), gr in zip(inputs, grads):
            out[i] = gr
        return tuple(out)


def lres_torgb(x, w, a, b, dtype, clamp):
    """``bias_act(conv3d(x.type(dtype) * a, w), b, act='linear', clamp=clamp)`` in one pass over x: w [3, Cin] (or [3,
    Cin, 1, 1, 1]), a [N, Cin, T] and b [3], cast to fp32; clamp a number or None. CUDA only: callers check
    ``supported``."""
    w = w.float().reshape(w.shape[0], w.shape[1])
    return _LresTorgb.apply(x, w, a.float(), b.float(), dtype, None if clamp is None else float(clamp))


def records_backward(L, input, latent):
    """The call records a backward pass: grad mode on and the input, the latent or a parameter of L requires a gradient."""
    return torch.is_grad_enabled() and (input.requires_grad or latent.requires_grad or any(p.requires_grad for p in L.parameters()))


def track_sumsq(ema, g, sumsq, numel, beta):
    """``MagnitudeEMA.forward``'s update from a sum of squares on the device: the mean, its all_reduce over the world when
    ``dist_sync`` (``dist`` / ``dist_utils`` from the model module's globals ``g``), ``lerp_``. Returns the gain."""
    magnitude = sumsq / numel
    if ema.dist_sync and g['dist_utils'].get_world_size() > 1:
        g['dist'].all_reduce(magnitude, g['dist'].ReduceOp.SUM)
        magnitude = magnitude / g['dist_utils'].get_world_size()
    ema.magnitude_ema.lerp_(magnitude, 1.0 - beta)
    return ema.magnitude_ema.rsqrt()


def layer_forward(L, g, input, latent, magnitude_ema_beta=1.0, dtype=None):
    """ToRGB.forward with the layer as ``lres_torgb``: the same affine, dtype and MagnitudeEMA logic as the reference, in
    its order. ``g``: the globals of the model module (its ``misc``, ``einops``, ``dist`` and ``dist_utils``, whatever they
    are patched to). A magnitude-EMA update in a call that records no backward takes its statistic from the op's pass."""
    misc, einops = g['misc'], g['einops']
    misc.assert_shape(input, (None, L.in_channels, None, None, None))
    batch_size, in_seq_length = input.size(0), input.size(2)
    misc.assert_shape(latent, (batch_size, L.latent_dim, in_seq_length))

    latent_nt = einops.rearrange(latent, "n c t -> (n t) c")
    style = L.affine(latent_nt)
    style = einops.rearrange(style, "(n t) c -> n c t", t=in_seq_length)

    dtype = dtype if dtype is not None else (torch.float16 if L.use_float16 and input.is_cuda else torch.float32)
    w = L.weight / math.sqrt(int(np.prod(L.weight.shape[1:])))
    clamp = L.activation_clamp
    if L.magnitude_ema and magnitude_ema_beta != 1 and not records_backward(L, input, latent):
        plug = _plugin()
        u, sumsq = plug.fprop_sumsq(input, w.detach().float().reshape(w.shape[0], -1), style.detach().float(), dtype)
        gain = track_sumsq(L.input_magnitude_ema, g, sumsq, input.numel(), magnitude_ema_beta)
        return plug.finish(u, gain, L.bias.detach().float(), dtype, None if clamp is None else float(clamp))
    a = style
    if L.magnitude_ema:
        gain = L.input_magnitude_ema(input.type(dtype) if magnitude_ema_beta != 1 else input, magnitude_ema_beta)
        a = style * gain
    return lres_torgb(input, w, a, L.bias, dtype, clamp)


# ---------------------------------------------------------------------------------------------------- install

def _is_torgb(m):
    return getattr(m, 'weight', None) is not None and m.weight.ndim == 5 and hasattr(m, 'affine')


def mode(L, input, latent, magnitude_ema_beta):
    """Which of the layer's three calls this is: 'backward' (records a backward pass at beta 1: update_G), 'stat' (updates
    the magnitude EMA and records none: update_D's generated pass), 'forward' (neither: inference), or None (a backward
    pass with an EMA update, which no training step makes)."""
    update = L.magnitude_ema and magnitude_ema_beta != 1
    if records_backward(L, input, latent):
        return None if update else 'backward'
    return 'stat' if update else 'forward'


def _takes(L, input, latent, magnitude_ema_beta=1.0, dtype=None):
    """The installed forward takes the call: inside ``supported`` and one of the modes the op measured faster in on the
    H100 (``_MODES``, DESIGN.md 7l)."""
    if not (isinstance(input, torch.Tensor) and isinstance(latent, torch.Tensor) and input.ndim == 5 and input.is_cuda):
        return False
    dt = dtype if dtype is not None else (torch.float16 if L.use_float16 else torch.float32)
    if not supported(input, dt, tuple(L.weight.shape)):
        return False
    return mode(L, input, latent, magnitude_ema_beta) in _MODES


def _forward(orig):
    g = _install.reference_function(orig).__globals__

    def forward(self, input, latent, magnitude_ema_beta=1.0, dtype=None):
        if not _takes(self, input, latent, magnitude_ema_beta, dtype):
            return orig(self, input, latent, magnitude_ema_beta, dtype)
        return layer_forward(self, g, input, latent, magnitude_ema_beta, dtype)
    forward.takes = _takes
    return forward


def install(*targets):
    """Make ``ToRGB.forward`` of generator_lres run ``layer_forward`` in the calls ``_takes`` routes to it. ``targets``: the
    module ``model.generator_lres`` or generator / layer instances, found by ``_install.find_classes`` (which reaches
    classes ``persistence`` rebuilt from a pickle). Other calls (CPU tensors, fp64, LVG_NATIVE_CONV=0, shapes the size
    query rejects, modes not routed) run the method this wrapper replaced. Composes with ``modulated_conv.install`` and
    ``gblock_tail.install`` in any order. Idempotent; the replaced method stays reachable as ``.forward.lvg_lres_torgb``.
    Returns the patched classes."""
    classes = _install.find_classes(targets, 'ToRGB', _is_torgb)
    for cls in classes:
        _install.wrap(cls, 'forward', 'lvg_lres_torgb', _forward)
    return classes
