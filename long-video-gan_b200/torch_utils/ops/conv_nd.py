"""1-D / 2-D / 3-D grouped convolution on the TMA-fed wgmma engine (csrc/conv_igemm.cu), with autograd of any order.

Not a module of the reference's ``torch_utils.ops`` -- the reference calls ``torch.nn.functional.conv1d / conv2d / conv3d``
(cuDNN) directly at these sites:

  conv2d_gradfix.conv2d / conv_transpose2d    conv2d_gradfix.py:37-45          (this package routes them here)
  F.conv3d in the low-res networks            generator_lres.py:119,578; discriminator_lres.py:172
  F.conv1d in the low-res discriminator       discriminator_lres.py:108-127

``conv1d / conv2d / conv3d / conv_transpose2d`` below keep torch.nn.functional's argument lists. To run an UNMODIFIED
reference model file on them, ``install_functional(model.generator_lres, model.discriminator_lres)`` replaces the
module-level name ``F`` of those modules by a proxy that forwards everything else to ``torch.nn.functional``.

fp16 tensors: fp16 operands, fp32 accumulation. fp32 tensors: bf16 hi/lo split operands, three tensor-core products,
fp32 accumulation (relative error ~2^-16; the reference trains these layers with TF32 off, train_lres.py:269).
Calls outside the engine's envelope (dilation, kernels beyond 3x3 / kt 7, CPU tensors, fp64) fall through to
``torch.nn.functional``; CUDA calls inside it never do.
"""
import os

import torch

_plugin = None


def _get_plugin():
    global _plugin
    if _plugin is None:
        from .. import custom_ops
        _plugin = custom_ops.get_plugin('convnd_plugin')
    return _plugin


def _tup(v, nd):
    return tuple(int(a) for a in v) if isinstance(v, (list, tuple)) else (int(v),) * nd


def enabled_for(x):
    return x.device.type == 'cuda' and os.environ.get('LVG_NATIVE_CONV', '1') != '0'


def _weights_off():
    from . import conv2d_gradfix
    return conv2d_gradfix.weight_gradients_disabled


def _fused_backward_ok(dy):
    """First-order backward pass asking for both gradients: one call that re-tiles dy once (lvg_convnd_backward). With
    create_graph=True (the R1 penalty's double backward) the two gradient Functions below are recorded instead."""
    return not torch.is_grad_enabled() and hasattr(_get_plugin(), 'backward')


class _ConvNd(torch.autograd.Function):
    """y = conv(x, w); gradients of any order through the two classes below."""

    @staticmethod
    def forward(ctx, x, w, padding, groups, stride):
        ctx.save_for_backward(x, w)
        ctx.cfg = (padding, groups, stride)
        return _get_plugin().fprop(x, w, padding, groups, stride=stride)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        padding, groups, stride = ctx.cfg
        dx = dw = None
        want_dw = ctx.needs_input_grad[1] and not _weights_off()
        if ctx.needs_input_grad[0] and want_dw and _fused_backward_ok(dy):
            dx, dw = _get_plugin().backward(x, dy, w, padding, groups, stride=stride)
            return dx, dw, None, None, None
        if ctx.needs_input_grad[0]:
            dx = _ConvNdDgrad.apply(dy, w, x.shape, padding, groups, stride)
        if want_dw:
            dw = _ConvNdWgrad.apply(dy, x, w.shape, padding, groups, stride)
        return dx, dw, None, None, None


class _ConvNdDgrad(torch.autograd.Function):
    """dx = conv^T(dy, w): the forward kernel on dy (spread over the stride lattice) with the weights re-tiled transposed
    and mirrored."""

    @staticmethod
    def forward(ctx, dy, w, x_shape, padding, groups, stride):
        ctx.save_for_backward(dy, w)
        ctx.cfg = (tuple(x_shape), padding, groups, stride)
        return _get_plugin().dgrad(dy, w, tuple(x_shape), padding, groups, stride=stride)

    @staticmethod
    def backward(ctx, ggx):
        dy, w = ctx.saved_tensors
        x_shape, padding, groups, stride = ctx.cfg
        d_dy = d_w = None
        if ctx.needs_input_grad[0]:
            d_dy = _ConvNd.apply(ggx, w, padding, groups, stride)
        if ctx.needs_input_grad[1] and not _weights_off():
            d_w = _ConvNdWgrad.apply(dy, ggx, w.shape, padding, groups, stride)
        return d_dy, d_w, None, None, None, None


class _ConvNdWgrad(torch.autograd.Function):
    """dw = sum over samples and output pixels of dy (x) shifted x (output pixels as the GEMM K axis)."""

    @staticmethod
    def forward(ctx, dy, x, w_shape, padding, groups, stride):
        ctx.save_for_backward(dy, x)
        ctx.cfg = (tuple(w_shape), padding, groups, stride)
        return _get_plugin().wgrad(x, dy, tuple(w_shape), padding, groups, stride=stride)

    @staticmethod
    def backward(ctx, ggw):
        dy, x = ctx.saved_tensors
        w_shape, padding, groups, stride = ctx.cfg
        d_dy = d_x = None
        if ctx.needs_input_grad[0]:
            d_dy = _ConvNd.apply(x, ggw, padding, groups, stride)
        if ctx.needs_input_grad[1]:
            d_x = _ConvNdDgrad.apply(dy, ggw, x.shape, padding, groups, stride)
        return d_dy, d_x, None, None, None, None


def _native_ok(x, w, stride, padding, dilation, groups):
    if not enabled_for(x) or not isinstance(padding, (int, list, tuple)):
        return None
    nd = x.ndim - 2
    st, pd, dl = _tup(stride, nd), _tup(padding, nd), _tup(dilation, nd)
    plug = _get_plugin()
    if w.dtype != x.dtype or not plug.supported(x, w, st, pd, dl, groups):
        return None
    return pd, st[-1]


def conv_nd(x, w, bias=None, stride=1, padding=0, dilation=1, groups=1):
    """torch.nn.functional.conv{1,2,3}d semantics; the tensor-core engine for every CUDA call inside its envelope."""
    ok = _native_ok(x, w, stride, padding, dilation, groups)
    if ok is None:
        f = (torch.nn.functional.conv1d, torch.nn.functional.conv2d, torch.nn.functional.conv3d)[x.ndim - 3]
        return f(x, w, bias, stride, padding, dilation, groups)
    pd, st = ok
    y = _ConvNd.apply(x, w, pd, groups, st)
    if bias is not None:
        y = y + bias.reshape([1, -1] + [1] * (x.ndim - 2)).to(y.dtype)
    return y


def _is_long_depthwise_fir(x, w, bias, stride, padding, dilation, groups):
    """BlurredNoise.blur (generator_lres.py:378-387): conv1d with one channel per group and a long kernel on a noise input --
    no gradient flows into it (noise input, buffer filters)."""
    return (enabled_for(x) and x.ndim == 3 and x.dtype == torch.float32 and w.dtype == torch.float32 and bias is None
            and groups == x.shape[1] == w.shape[0] and w.shape[1] == 1 and w.shape[2] >= 16 and x.shape[2] >= w.shape[2]
            and _tup(stride, 1) == (1,) and _tup(dilation, 1) == (1,) and isinstance(padding, int) and padding == 0
            and groups <= 65535 and x.shape[0] <= 65535
            and not (torch.is_grad_enabled() and (x.requires_grad or w.requires_grad)))


def conv1d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
    if _is_long_depthwise_fir(input, weight, bias, stride, padding, dilation, groups):
        return _get_plugin().fir1d_depthwise(input, weight)
    return conv_nd(input, weight, bias, stride, padding, dilation, groups)


def conv2d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
    return conv_nd(input, weight, bias, stride, padding, dilation, groups)


def conv3d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
    return conv_nd(input, weight, bias, stride, padding, dilation, groups)


def conv_transpose2d(input, weight, bias=None, stride=1, padding=0, output_padding=0, groups=1, dilation=1):
    """Transposed convolution = the input gradient of the convolution whose weight is `weight` ([Cin, Cout/groups, kh, kw]):
    output extent (H - 1) * stride - 2 * padding + k + output_padding."""
    from .. import custom_ops
    nd = 2
    st, pd, op, dl = _tup(stride, nd), _tup(padding, nd), _tup(output_padding, nd), _tup(dilation, nd)
    kh, kw = weight.shape[2], weight.shape[3]
    out_h = (input.shape[2] - 1) * st[0] - 2 * pd[0] + kh + op[0]
    out_w = (input.shape[3] - 1) * st[1] - 2 * pd[1] + kw + op[1]
    x_shape = (input.shape[0], weight.shape[1] * groups, out_h, out_w)
    # the forward convolution of that extent (whose gradients the backward pass takes) lies in the engine's envelope and
    # reproduces the input's extent
    native = (enabled_for(input) and weight.dtype == input.dtype and max(op) < st[0]
              and custom_ops.ConvNdPlugin._in_envelope(x_shape, tuple(weight.shape), input.dtype, st, pd, dl, groups)
              and (out_h + 2 * pd[0] - kh) // st[0] + 1 == input.shape[2] and (out_w + 2 * pd[1] - kw) // st[1] + 1 == input.shape[3])
    if not native:
        return torch.nn.functional.conv_transpose2d(input, weight, bias, stride, padding, output_padding, groups, dilation)
    y = _ConvNdDgrad.apply(input, weight, x_shape, pd, groups, st[0])
    if bias is not None:
        y = y + bias.reshape(1, -1, 1, 1).to(y.dtype)
    return y


class _BiasActGrad(torch.autograd.Function):
    """dz = G(y) * dy, G the slope of linear / lrelu with gain and clamp decided from the saved output y (bias_act's grad-1
    kernel; the sign of y is the sign of the pre-activation). Linear in dy with a piecewise constant G, so it is its own
    backward."""

    @staticmethod
    def forward(ctx, dy, y, cfg):
        from . import bias_act as ba
        act, alpha, gain, clamp = cfg
        ctx.save_for_backward(y)
        ctx.cfg = cfg
        return ba._plugin.bias_act(dy.contiguous(), None, None, y, None, 1, 1, ba.activation_funcs[act].cuda_idx, alpha, gain,
                                   -1.0 if clamp is None else clamp)

    @staticmethod
    def backward(ctx, g):
        y, = ctx.saved_tensors
        return (_BiasActGrad.apply(g, y, ctx.cfg) if ctx.needs_input_grad[0] else None), None, None


class _ConvBiasAct(torch.autograd.Function):
    """conv -> bias_act in ONE kernel: the convolution's epilogue adds the bias, applies linear / lrelu, gain and clamp while
    the accumulators leave the registers (no write + re-read of the pre-activation tensor). Backward: the activation
    gradient from the saved output (``_BiasActGrad``), then the convolution gradients; with create_graph=True every step is
    a recorded Function, so gradients of any order work."""

    @staticmethod
    def forward(ctx, x, w, b, padding, groups, stride, act, alpha, gain, clamp):
        y = _get_plugin().fprop(x, w, padding, groups, bias=b, act=2 if act == 'lrelu' else 1, alpha=alpha, gain=gain,
                                clamp=-1.0 if clamp is None else clamp, stride=stride)
        ctx.save_for_backward(x, w, y)
        ctx.cfg = (padding, groups, stride, act, alpha, gain, clamp, b is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        padding, groups, stride, act, alpha, gain, clamp, has_b = ctx.cfg
        dz = _BiasActGrad.apply(dy, y, (act, alpha, gain, clamp))        # d(pre-activation)
        dx = dw = db = None
        want_dw = ctx.needs_input_grad[1] and not _weights_off()
        if ctx.needs_input_grad[0] and want_dw and _fused_backward_ok(dz):
            dx, dw = _get_plugin().backward(x, dz, w, padding, groups, stride=stride)
        else:
            if ctx.needs_input_grad[0]:
                dx = _ConvNdDgrad.apply(dz, w, x.shape, padding, groups, stride)
            if want_dw:
                dw = _ConvNdWgrad.apply(dz, x, w.shape, padding, groups, stride)
        if has_b and ctx.needs_input_grad[2]:
            db = (dz.float() if dz.dtype == torch.float16 else dz).sum([0] + list(range(2, dz.ndim))).to(dz.dtype)
        return dx, dw, db, None, None, None, None, None, None, None


def conv_bias_act(x, w, b=None, stride=1, padding=0, groups=1, act='linear', alpha=None, gain=None, clamp=None):
    """``bias_act(conv(x, w), b, act=act, alpha=alpha, gain=gain, clamp=clamp)`` for act in ('linear', 'lrelu') -- what
    Conv3dLayer / Conv2dLayer compute (discriminator_lres.py:135-213, discriminator_sres.py:192-204, generator_lres.py:578-589)
    -- with the bias / activation / gain / clamp fused into the convolution's epilogue on CUDA. Gradients of any order.
    Falls back to the two separate ops outside the engine's envelope."""
    from . import bias_act as ba
    assert act in ('linear', 'lrelu')
    spec = ba.activation_funcs[act]
    alpha = float(alpha if alpha is not None else spec.def_alpha)
    gain = float(gain if gain is not None else spec.def_gain)
    ok = _native_ok(x, w, stride, padding, 1, groups)
    if ok is None or not ba._init():
        return ba.bias_act(conv_nd(x, w, None, stride, padding, 1, groups), b, act=act, alpha=alpha, gain=gain, clamp=clamp)
    pd, st = ok
    return _ConvBiasAct.apply(x, w, b, pd, groups, st, act, alpha, gain, clamp)


class _FunctionalProxy:
    """Stands in for the module-level name ``F`` of a reference model file: conv1d / conv2d / conv3d / conv_transpose2d go
    to the tensor-core engine, every other attribute to torch.nn.functional."""
    conv1d = staticmethod(conv1d)
    conv2d = staticmethod(conv2d)
    conv3d = staticmethod(conv3d)
    conv_transpose2d = staticmethod(conv_transpose2d)

    def __getattr__(self, name):
        return getattr(torch.nn.functional, name)


functional = _FunctionalProxy()


def install_functional(*modules):
    """``install_functional(model.generator_lres, model.discriminator_lres)``: their ``F.conv3d`` / ``F.conv1d`` calls run on
    the tensor-core engine from now on (the model source stays as it is). Returns the modules that were patched."""
    done = []
    for m in modules:
        if getattr(m, 'F', None) is torch.nn.functional or isinstance(getattr(m, 'F', None), _FunctionalProxy):
            m.F = functional
            done.append(m)
    return done
