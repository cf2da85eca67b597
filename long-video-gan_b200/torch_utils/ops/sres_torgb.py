"""The super-res generator's ToRGB layer as one native op.

Not a module of the reference's ``torch_utils.ops``. With ``sres_cond`` and ``modulated_conv`` the last layer of the
super-res generator (``SynthesisLayer`` with ``is_torgb``: a 1x1 modulated convolution to 3 channels without
demodulation, then ``filtered_lrelu``'s bias and clamp with gain 1 and slope 1) writes its input z = cat(x_prev,
cond(lr)).to(dtype) to HBM, the convolution engine reads it back for 3 output channels, and ``filtered_lrelu`` makes a
third pass. ``sres_torgb`` computes

  y = dtype(clamp(dtype(conv1x1(r(a * z), w)) + b, +-clamp))      r: fp16 rounding in fp16 layers

in one pass over x_prev on the CUDA cores (csrc/sres_torgb.cu: lvg_sres_torgb_fprop / _backward), with the conditioning
evaluated in place by the layer's plan (csrc/sres_cond.cuh, the sums ``cond_concat`` writes) and a·z rounded as the
engine's re-tiling pass rounds it. The products are summed in fp32 in another order than the engine's wgmma, so y agrees
with the composition to one rounding of the layer dtype, not bit for bit. The forward keeps a one-byte clamp mask per
pixel when a gradient is recorded; the first-order backward is one pass over x_prev and dy (dx_prev, da, and the Gram
sums that give dw and db, folded in a fixed order: bitwise reproducible). With create_graph=True the backward is recorded
from the composition (``cond_concat`` -> ``modulated_conv`` -> ``filtered_lrelu``), so gradients of any order work.
``update_emas`` keeps ``sres_layer``'s statistic pass (``sres_layer.mean_sq``, then ``sres_cond.track_magnitude``).

``install(...)`` makes an unmodified ``Generator.forward`` of generator_sres run its ToRGB layer through this op
(opt-in, idempotent) in the calls where it measured faster (DESIGN.md 7k): every call that records a backward pass, and
forward passes without one that neither update the magnitude EMA (update_D's generated pass) nor run with
``sres_layer`` installed (chained inference with it). The other layers run the step the other installs give them
(``sres_layer``'s where that op takes the call, else ``sres_cond.conv_step``); calls the op does not take run the method
this wrapper replaced.
"""
import numpy as np
import torch

from .. import custom_ops
from . import _install, conv_nd, filtered_lrelu, modulated_conv
from . import sres_cond as sc
from . import sres_layer as sl


def _plugin():
    return custom_ops.get_plugin('sres_cond_plugin')


def supported(n, t, c, c_lr, t_lr, plan, dtype, cout):
    """The kernels take the call (size query of lvg_sres_torgb): n low-res videos of t_lr frames and c_lr channels, c x_prev
    channels, cout output channels."""
    if plan.h.ntaps > sc.MAX_TAPS or plan.w.ntaps > sc.MAX_TAPS:
        return False
    return _plugin().torgb_workspace(n, t, c, c_lr, plan.window, t_lr, plan.h.len, plan.w.len, dtype, sc._ints(plan.h),
                                     sc._ints(plan.w), cout) >= 0


def composition(x_prev, lr, plan, dtype, w, a, b, clamp):
    """What the op replaces: ``cond_concat``, ``modulated_conv`` (the 1x1 convolution on the engine) and
    ``filtered_lrelu``'s bias and clamp with gain 1 and slope 1. w [Cout, Cin] and b [Cout] in dtype, a [N T, Cin, 1]."""
    z, _ = sc.cond_concat(x_prev, lr, plan, dtype, False)
    u = modulated_conv.modulated_conv(z, w[:, :, None, None], a, None, (0, 0))
    return filtered_lrelu.filtered_lrelu(u, b=b, gain=1, slope=1, clamp=clamp)


class _SresTorgb(torch.autograd.Function):
    """y = dtype(clamp(dtype(conv1x1(r(a * cat(x_prev, cond(lr)).to(dtype)), w)) + b)): x_prev [N T, C, H, W] (fp16 /
    fp32), w [Cout, Cin] and b [Cout] in dtype, a [N T, Cin, 1] (fp32)."""

    @staticmethod
    def forward(ctx, x_prev, lr, plan, dtype, w, a, b, clamp):
        f = plan.filter
        y, mask = _plugin().torgb_fprop(x_prev, lr, f if plan.h.ntaps else None, f if plan.w.ntaps else None, sc._ints(plan.h),
                                        sc._ints(plan.w), plan.h.gain, plan.w.gain, plan.window, dtype, w, a, b, clamp,
                                        any(ctx.needs_input_grad))
        ctx.save_for_backward(x_prev, lr, w, a, b, mask)
        ctx.plan, ctx.dtype, ctx.clamp = plan, dtype, clamp
        return y

    @staticmethod
    def backward(ctx, dy):
        x_prev, lr, w, a, b, mask = ctx.saved_tensors
        plan, dtype, clamp = ctx.plan, ctx.dtype, ctx.clamp
        need = ctx.needs_input_grad
        if not torch.is_grad_enabled():
            f = plan.filter
            dx, dw, da, db = _plugin().torgb_backward(x_prev, lr, f if plan.h.ntaps else None, f if plan.w.ntaps else None,
                                                      sc._ints(plan.h), sc._ints(plan.w), plan.h.gain, plan.w.gain, plan.window,
                                                      dtype, w, a, b, mask, dy, want_dx=need[0],
                                                      want_dw=need[4] and not conv_nd._weights_off(), want_db=need[6])
            return dx, None, None, None, dw, (da.view(a.shape) if need[5] else None), db, None
        # differentiable composition (double backward through the generator): the three ops this one replaces
        inputs = [(i, v) for i, v in ((0, x_prev), (4, w), (5, a), (6, b)) if need[i]]
        with torch.enable_grad():
            y = composition(x_prev, lr, plan, dtype, w, a, b, clamp)
            grads = torch.autograd.grad(y, [v for _, v in inputs], dy, create_graph=True, allow_unused=True)
        out = [None] * 8
        for (i, _), gr in zip(inputs, grads):
            out[i] = gr
        return tuple(out)


def sres_torgb(x_prev, lr, plan, dtype, wn, a, b, clamp):
    """``filtered_lrelu(modulated_conv(cond_concat(x_prev, lr, plan, dtype)[0], wn, a), b, gain=1, slope=1, clamp)``
    without z: wn [Cout, Cin] or [Cout, Cin, 1, 1] and b [Cout] in dtype, a [N T, Cin] or [N T, Cin, 1], clamp a number or
    None. CUDA only: callers check ``supported``."""
    f = plan.filter
    if f is not None and f.device != lr.device:
        raise RuntimeError('sres_torgb: the filter must be on the device of lr')
    w = wn.reshape(wn.shape[0], wn.shape[1])
    return _SresTorgb.apply(x_prev, lr, plan, dtype, w, a.float().reshape(a.shape[0], a.shape[1], 1), b, clamp)


def fused_forward(L, g, x_prev, lr, plan, w, force_fp32=False, update_emas=False):
    """``sres_cond.layer_forward`` of the ToRGB layer ``L`` as one op: the same magnitude EMA (its statistic from
    ``sres_layer.mean_sq``), styles and factors (``modulated_conv.factors``, the torch ops of modulated_conv2d), then
    ``sres_torgb``."""
    misc, distributed = g['misc'], g['distributed']
    dtype = torch.float16 if (L.use_fp16 and not force_fp32 and lr.device.type == 'cuda') else torch.float32
    misc.assert_shape(w, [lr.shape[0] * (lr.shape[2] - plan.window + 1), L.w_dim])
    if update_emas:
        sc.track_magnitude(L, distributed, sl.mean_sq(x_prev, lr, plan, dtype, L.weight.detach().to(dtype), (0, 0)))
    input_gain = L.magnitude_ema.rsqrt()
    styles = sc.layer_styles(L, w)
    wn, a, _ = modulated_conv.factors(L.weight, styles, demodulate=False, input_gain=input_gain)
    x = sres_torgb(x_prev, lr, plan, dtype, wn.to(dtype), a, L.bias.to(dtype), L.conv_clamp)
    misc.assert_shape(x, [None, L.out_channels, int(L.out_size[1]), int(L.out_size[0])])
    return x


def layer_forward(L, g, x_prev, lr, plan, w, force_fp32=False, update_emas=False, **unused):
    """The installed ToRGB forward (``fused_forward``; ``unused``: the other layers' step)."""
    return fused_forward(L, g, x_prev, lr, plan, w, force_fp32, update_emas)


# ---------------------------------------------------------------------------------------------------- install

def _is_plain_torgb(L):
    """A ToRGB layer the op computes: a 1x1 convolution, no resampling or filters in filtered_lrelu, no padding."""
    return (L.is_torgb and int(L.conv_kernel) == 1 and L.up_factor == 1 and L.down_factor == 1 and L.up_filter is None
            and L.down_filter is None and list(L.padding) == [0, 0, 0, 0] and np.array_equal(L.in_size, L.out_size)
            and L.weight.ndim == 4 and tuple(L.weight.shape[2:]) == (1, 1))


def rejection(G, cond, lr_plans=None):
    """Why the installed forward does not take the call, or None when it does: ``sres_cond.rejection``'s reasons, 'layer'
    (the last layer is not a plain ToRGB layer: 1x1, unfiltered, unpadded), 'shape' also where the op's or the statistic's
    size query rejects it in fp16 or fp32, and 'conv' (native convolutions are off, LVG_NATIVE_CONV=0). The device check
    ('cpu') still comes after the shape checks."""
    why = sc.rejection(G, cond, lr_plans)
    if why not in (None, 'cpu'):
        return why
    n, c_lr, t_lr, lr_h, lr_w = cond.shape
    lr_plans = sc.plans(G, lr_h, lr_w) if lr_plans is None else lr_plans
    S = G.synthesis
    L, p = getattr(S, S.layer_names[-1]), lr_plans[-1]
    if not _is_plain_torgb(L):
        return 'layer'
    t = t_lr - 2 * G.cond_context
    c = L.in_channels - c_lr * p.window
    if c < 1:
        return 'shape'
    for dt in (torch.float16, torch.float32):
        if not (supported(n, t, c, c_lr, t_lr, p, dt, L.out_channels)
                and sl.supported(n, t, c, c_lr, t_lr, p, dt, L.weight.shape, (0, 0))):
            return 'shape'
    if why is None and not conv_nd.enabled_for(cond):
        return 'conv'
    return why


def records_backward(G):
    """The call records a backward pass through G's parameters."""
    return torch.is_grad_enabled() and any(p.requires_grad for p in G.parameters())


def _layer_wrapper(G):
    """sres_layer.install's wrapper anywhere in the chain of G's forward, or None."""
    return _install.find(type(G).forward, 'lvg_sres_layer')


def _takes(G, cond, update_emas=False):
    """The installed forward takes the call: inside ``rejection``, and routed by where the op measured faster on the H100
    (DESIGN.md 7k): every call that records a backward pass, and forward passes without one only when they do not update
    the magnitude EMA (the statistic is a pass of its own) and ``sres_layer`` is not installed (its fused forward is
    faster at this layer)."""
    if not (isinstance(cond, torch.Tensor) and cond.ndim == 5):
        return False
    if not records_backward(G) and (update_emas or _layer_wrapper(G) is not None):
        return False
    return rejection(G, cond) is None


def _forward(orig):
    g = _install.reference_function(orig).__globals__

    def forward(self, z, cond, truncation_psi=1, truncation_cutoff=None, update_emas=False, **synthesis_kwargs):
        if not _takes(self, cond, update_emas):
            return orig(self, z, cond, truncation_psi, truncation_cutoff, update_emas, **synthesis_kwargs)
        # the other layers: sres_layer's step where its install (anywhere in the chain) takes the call
        layer = _layer_wrapper(self)
        step = sl.conv_step if (layer is not None and layer.takes(self, cond, update_emas)) else sc.conv_step
        return sc.generator_forward(self, g, z, cond, truncation_psi, truncation_cutoff, update_emas,
                                    lr_plans=sc.plans(self, cond.size(3), cond.size(4)), step=step, torgb=layer_forward,
                                    **synthesis_kwargs)
    forward.takes = _takes
    return forward


def install(*targets):
    """Make ``Generator.forward`` of generator_sres run ``sres_cond.generator_forward`` with the ToRGB layer from
    ``sres_torgb`` in the calls ``_takes`` routes to it. ``targets`` as ``sres_cond.install``. Other calls and calls
    outside ``rejection`` run the method this wrapper replaced. Composes with ``sres_cond.install``,
    ``sres_layer.install`` and ``modulated_conv.install`` in any order. Idempotent; the replaced method stays reachable as ``.forward.lvg_sres_torgb``. Returns the patched classes."""
    classes = _install.find_classes(targets, 'Generator', sc._is_generator)
    for cls in classes:
        _install.wrap(cls, 'forward', 'lvg_sres_torgb', _forward)
    return classes
