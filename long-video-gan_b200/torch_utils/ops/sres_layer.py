"""A super-res generator layer's input and modulated convolution as one native op.

Not a module of the reference's ``torch_utils.ops``. With ``sres_cond`` and ``modulated_conv`` each layer of the super-res
generator writes its input z = cat(x_prev, cond(lr)).to(dtype) to HBM (``cond_concat``) and the convolution reads it back
to re-tile it. ``sres_layer`` computes

  y = d * conv(a * z, w)        with z never formed

on the convolution engine (csrc/sres_layer.cu: lvg_sres_layer_fprop / _backward): the re-tiling pass reads x_prev and
evaluates the conditioning from the low-res video by the layer's plan with the same sums as sres_cond's kernel
(csrc/sres_cond.cuh), so y and every gradient are bit for bit those of ``modulated_conv(cond_concat(...))``. The autograd
Function saves x_prev, lr, the plan, w, a, d and y, not z; the first-order backward pass is one native call (dx_prev in
x_prev's dtype, dw, da and the row sums that give dd). With create_graph=True it is recorded from ``cond_concat`` and
``modulated_conv``'s differentiable composition instead, so gradients of any order work. ``mean_sq`` gives the mean square
of the fp32 z from the same re-tiling pass without its stores: a = s * rsqrt(magnitude_ema) depends on it, so with
``update_emas`` it is a pass of its own before the convolution; its fold order differs from ``cond_concat``'s, so the two
agree to float rounding.

``install(...)`` makes an unmodified ``Generator.forward`` of generator_sres run each layer's input and modulated
convolution through this op (opt-in, idempotent), over ``sres_cond``'s restated forwards, in the calls where it measured
faster: forward passes that record no backward and do not update the magnitude EMA (chained inference). The others run
``sres_cond.conv_step`` (DESIGN.md 7j).
"""
import torch

from .. import custom_ops
from . import _install, conv_nd, modulated_conv
from . import sres_cond as sc


def _plugin():
    return custom_ops.get_plugin('sres_cond_plugin')


def _filters(plan):
    f = plan.filter
    return (f if plan.h.ntaps else None), (f if plan.w.ntaps else None)


def supported(n, t, c, c_lr, t_lr, plan, dtype, w_shape, padding):
    """The kernels take the call (size query of lvg_sres_layer): n low-res videos of t_lr frames and c_lr channels, c x_prev
    channels, a weight of shape ``w_shape`` [Cout, c + c_lr window, kh, kw] and ``padding`` (ph, pw)."""
    if plan.h.ntaps > sc.MAX_TAPS or plan.w.ntaps > sc.MAX_TAPS:
        return False
    cout, cin, kh, kw = (int(v) for v in w_shape)
    if cin != c + c_lr * plan.window:
        return False
    return _plugin().layer_workspace(n, t, c, c_lr, plan.window, t_lr, plan.h.len, plan.w.len, dtype, sc._ints(plan.h),
                                     sc._ints(plan.w), cout, kh, kw, int(padding[0]), int(padding[1])) >= 0


class _SresLayer(torch.autograd.Function):
    """y = d * conv(a * cat(x_prev, cond(lr)).to(dtype), w): x_prev [N T, C, H, W] (fp16 / fp32) or None, w [Cout, Cin, kh,
    kw] in dtype, a [N T, Cin, 1], d [N T, Cout, 1] or None (fp32)."""

    @staticmethod
    def forward(ctx, x_prev, lr, plan, dtype, w, a, d, padding):
        f_h, f_w = _filters(plan)
        y, _ = _plugin().layer_fprop(x_prev, lr, f_h, f_w, sc._ints(plan.h), sc._ints(plan.w), plan.h.gain, plan.w.gain,
                                     plan.window, dtype, w, a, d, padding, False)
        ctx.save_for_backward(x_prev, lr, w, a, d, y)
        ctx.plan, ctx.dtype, ctx.padding = plan, dtype, padding
        return y

    @staticmethod
    def backward(ctx, dy):
        x_prev, lr, w, a, d, y = ctx.saved_tensors
        plan, dtype, padding = ctx.plan, ctx.dtype, ctx.padding
        need = ctx.needs_input_grad
        want_dw = need[4] and not conv_nd._weights_off()
        if not torch.is_grad_enabled():
            f_h, f_w = _filters(plan)
            dx, dw, da, dyy = _plugin().layer_backward(x_prev, lr, f_h, f_w, sc._ints(plan.h), sc._ints(plan.w), plan.h.gain,
                                                       plan.w.gain, plan.window, dtype, w, a, d, y, dy, padding,
                                                       want_dx=need[0], want_dw=want_dw)
            dd = dyy / d if (d is not None and need[6]) else None
            return dx, None, None, None, dw, (da if need[5] else None), dd, None
        # differentiable composition (double backward through the generator): the two ops this one replaces
        z, _ = sc.cond_concat(x_prev, lr, plan, dtype, False)
        dz, dw, da, dd = modulated_conv.backward_graph(z, w, a, d, dy, padding, need[0] or need[5], want_dw,
                                                       d is not None and need[6])
        dx = dz[:, :x_prev.shape[1]].to(x_prev.dtype) if (need[0] and x_prev is not None) else None
        return dx, None, None, None, dw, (da if need[5] else None), dd, None


def sres_layer(x_prev, lr, plan, dtype, w, a, d, padding):
    """``modulated_conv.modulated_conv(cond_concat(x_prev, lr, plan, dtype, False)[0], w, a, d, padding)`` without z. CUDA
    only: callers check ``supported``."""
    f = plan.filter
    if f is not None and f.device != lr.device:
        raise RuntimeError('sres_layer: the filter must be on the device of lr')
    return _SresLayer.apply(x_prev, lr, plan, dtype, w, a.float(), None if d is None else d.float(), tuple(padding))


def mean_sq(x_prev, lr, plan, dtype, w, padding):
    """The mean square of the fp32 concatenation cat(x_prev, cond) (``cond_concat``'s statistic, folded in another fixed
    order) from the layer op's re-tiling pass, without its stores."""
    f_h, f_w = _filters(plan)
    _, ms = _plugin().layer_fprop(x_prev, lr, f_h, f_w, sc._ints(plan.h), sc._ints(plan.w), plan.h.gain, plan.w.gain,
                                  plan.window, dtype, w, None, None, padding, True)
    return ms


def _records_backward(L, x_prev, w):
    return torch.is_grad_enabled() and (any(p.requires_grad for p in L.parameters()) or w.requires_grad
                                        or (x_prev is not None and x_prev.requires_grad))


def fused_step(L, g, x_prev, lr, plan, w, dtype, update_emas):
    """``sres_cond.conv_step`` as one op: the same magnitude EMA (its statistic from ``mean_sq``), styles and factors
    (``modulated_conv.factors``, the torch ops of modulated_conv2d), then ``sres_layer``."""
    misc, distributed = g['misc'], g['distributed']
    misc.assert_shape(w, [lr.shape[0] * (lr.shape[2] - plan.window + 1), L.w_dim])
    k = int(L.conv_kernel)
    padding = (k - 1, k - 1)
    if update_emas:
        sc.track_magnitude(L, distributed, mean_sq(x_prev, lr, plan, dtype, L.weight.detach().to(dtype), padding))
    input_gain = L.magnitude_ema.rsqrt()
    styles = sc.layer_styles(L, w)
    wn, a, d = modulated_conv.factors(L.weight, styles, demodulate=(not L.is_torgb), input_gain=input_gain)
    return sres_layer(x_prev, lr, plan, dtype, wn.to(dtype), a, d, padding)


def _records_backward(L, x_prev, w):
    return torch.is_grad_enabled() and (any(p.requires_grad for p in L.parameters()) or w.requires_grad
                                        or (x_prev is not None and x_prev.requires_grad))


def conv_step(L, g, x_prev, lr, plan, w, dtype, update_emas):
    """The installed layer step: ``fused_step`` for forward passes that record no backward and do not update the
    magnitude EMA, ``sres_cond.conv_step`` for the others, which measured slower through the op on the H100 (DESIGN.md
    7j)."""
    if update_emas or _records_backward(L, x_prev, w):
        return sc.conv_step(L, g, x_prev, lr, plan, w, dtype, update_emas)
    return fused_step(L, g, x_prev, lr, plan, w, dtype, update_emas)


# ---------------------------------------------------------------------------------------------------- install

def rejection(G, cond, lr_plans=None):
    """Why the installed forward does not take the call, or None when it does: ``sres_cond.rejection``'s reasons, 'shape'
    also where the layer op's size query rejects a layer in fp16 or fp32, and 'conv' (native convolutions are off,
    LVG_NATIVE_CONV=0). The device check ('cpu') still comes after the shape checks."""
    why = sc.rejection(G, cond, lr_plans)
    if why not in (None, 'cpu'):
        return why
    n, c_lr, t_lr, lr_h, lr_w = cond.shape
    lr_plans = sc.plans(G, lr_h, lr_w) if lr_plans is None else lr_plans
    t = t_lr - 2 * G.cond_context
    S = G.synthesis
    for name, p in zip(S.layer_names, lr_plans):
        L = getattr(S, name)
        c = L.in_channels - c_lr * p.window
        k = int(L.conv_kernel)
        if not all(supported(n, t, c, c_lr, t_lr, p, dt, L.weight.shape, (k - 1, k - 1)) for dt in (torch.float16, torch.float32)):
            return 'shape'
    if why is None and not conv_nd.enabled_for(cond):
        return 'conv'
    return why


def _takes(G, cond):
    return isinstance(cond, torch.Tensor) and cond.ndim == 5 and rejection(G, cond) is None


def _forward(orig):
    g = _install.reference_function(orig).__globals__

    def forward(self, z, cond, truncation_psi=1, truncation_cutoff=None, update_emas=False, **synthesis_kwargs):
        lr_plans = sc.plans(self, cond.size(3), cond.size(4)) if isinstance(cond, torch.Tensor) and cond.ndim == 5 else None
        if lr_plans is None or rejection(self, cond, lr_plans) is not None:
            return orig(self, z, cond, truncation_psi, truncation_cutoff, update_emas, **synthesis_kwargs)
        return sc.generator_forward(self, g, z, cond, truncation_psi, truncation_cutoff, update_emas, lr_plans=lr_plans,
                                    step=conv_step, **synthesis_kwargs)
    forward.takes = _takes
    return forward


def install(*targets):
    """Make ``Generator.forward`` of generator_sres run ``sres_cond.generator_forward`` with every layer's input and
    modulated convolution from ``sres_layer``. ``targets`` as ``sres_cond.install``. Calls outside ``rejection`` run the
    method this wrapper replaced. Composes with ``sres_cond.install`` and ``modulated_conv.install`` in either order.
    Idempotent; the replaced method stays reachable as ``.forward.lvg_sres_layer``. Returns the patched classes."""
    classes = _install.find_classes(targets, 'Generator', sc._is_generator)
    for cls in classes:
        _install.wrap(cls, 'forward', 'lvg_sres_layer', _forward)
    return classes
