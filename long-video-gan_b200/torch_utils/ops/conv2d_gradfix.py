"""``conv2d`` / ``conv_transpose2d`` entry points (``torch_utils.ops.conv2d_gradfix``).

Same functions and module switches as the reference (conv2d_gradfix.py:22-45):
``enabled``, ``weight_gradients_disabled``, ``no_weight_gradients()``. In the
reference the custom autograd path is inert on torch >= 1.11 (:49-58) and every
call lands in cuDNN. Here this module is the tensor-core boundary: CUDA calls
inside the envelope of the wgmma implicit-GEMM kernel (csrc/conv2d_tc.cu;
grouped "modulated" 3x3 / 1x1 convolutions in fp16) are routed to it through
``_native`` below; everything else goes to ``torch.nn.functional``.
"""
import contextlib
import os

import torch

enabled = False                     # kept for API compatibility (train_lres.py:80 sets it)
weight_gradients_disabled = False   # forcefully skip weight gradients (R1 penalty, see no_weight_gradients)

# Native convolution backend: None = library convolution only (what the reference does). `install_native()`
# binds the wgmma engine; `LVG_NATIVE_CONV=0` in the environment keeps it off.
_native = None


@contextlib.contextmanager
def no_weight_gradients(disable=True):
    global weight_gradients_disabled
    old = weight_gradients_disabled
    if disable:
        weight_gradients_disabled = True
    yield
    weight_gradients_disabled = old


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def install_native(enable=True):
    """Route the convolutions inside the tensor-core kernel's envelope (CUDA, fp16, stride 1, 3x3 / 1x1) to it."""
    global _native
    if not enable:
        _native = None
        return None
    from .. import custom_ops
    _native = custom_ops.get_plugin('conv2d_plugin')
    return _native


def _auto_install():
    import os
    if os.environ.get('LVG_NATIVE_CONV', '1') != '0' and torch.cuda.is_available():
        try:
            install_native(True)
        except (RuntimeError, OSError, AttributeError):
            pass


def _engine():
    """'nd' (default): the TMA-fed engine of csrc/conv_igemm.cu for every dtype / stride it covers; 'r1': the round-1
    kernels (fp16, stride 1) first."""
    return os.environ.get('LVG_CONV_ENGINE', 'nd')


def conv2d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
    if input.device.type == 'cuda' and _engine() == 'nd' and os.environ.get('LVG_NATIVE_CONV', '1') != '0':
        from . import conv_nd
        return conv_nd.conv2d(input, weight, bias, stride, padding, dilation, groups)
    if _native is None and input.device.type == 'cuda' and not _auto_install.done:
        _auto_install.done = True
        _auto_install()
    if _native is not None and input.device.type == 'cuda':
        st, pd, dl = _pair(stride), _pair(padding), _pair(dilation)
        if _native.supported(input, weight, st, pd, dl, groups):
            out = _Conv2d.apply(input, weight, pd, groups)
            return out if bias is None else out + bias.reshape(1, -1, 1, 1).to(out.dtype)
    return torch.nn.functional.conv2d(input=input, weight=weight, bias=bias, stride=stride, padding=padding,
                                      dilation=dilation, groups=groups)


_auto_install.done = False


class _Conv2d(torch.autograd.Function):
    """y = conv2d(x, w) on the tensor-core kernel; gradients of any order through the two classes below."""

    @staticmethod
    def forward(ctx, x, w, padding, groups):
        ctx.save_for_backward(x, w)
        ctx.cfg = (padding, groups)
        return _native.fprop(x, w, padding, groups)

    @staticmethod
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        padding, groups = ctx.cfg
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = _Conv2dDgrad.apply(dy, w, x.shape, padding, groups)
        if ctx.needs_input_grad[1] and not weight_gradients_disabled:
            dw = _Conv2dWgrad.apply(dy, x, w.shape, padding, groups)
        return dx, dw, None, None


class _Conv2dDgrad(torch.autograd.Function):
    """dx = conv2d^T(dy, w): the same kernel with the weights repacked transposed and mirrored."""

    @staticmethod
    def forward(ctx, dy, w, x_shape, padding, groups):
        ctx.save_for_backward(dy, w)
        ctx.cfg = (x_shape, padding, groups)
        return _native.dgrad(dy, w, x_shape, padding, groups)

    @staticmethod
    def backward(ctx, ggx):
        dy, w = ctx.saved_tensors
        x_shape, padding, groups = ctx.cfg
        d_dy = d_w = None
        if ctx.needs_input_grad[0]:
            d_dy = _Conv2d.apply(ggx, w, padding, groups)
        if ctx.needs_input_grad[1] and not weight_gradients_disabled:
            d_w = _Conv2dWgrad.apply(dy, ggx, w.shape, padding, groups)
        return d_dy, d_w, None, None, None


class _Conv2dWgrad(torch.autograd.Function):
    """dw = sum over samples and pixels of dy (x) shifted x: lvg_conv2d_wgrad (wgmma, pixels as the GEMM K axis).
    LVG_NATIVE_WGRAD = 1: always the native kernel (what the GPU tests set); 0: always ATen / cuDNN; unset ("auto"):
    native for few input channels per group (<= 64), where cuDNN's grouped weight gradient is far off the tensor-core
    rate, and ATen for the wide layers. The split has not been re-measured on the H100."""

    @staticmethod
    def forward(ctx, dy, x, w_shape, padding, groups):
        ctx.save_for_backward(dy, x)
        ctx.cfg = (w_shape, padding, groups)
        mode = os.environ.get('LVG_NATIVE_WGRAD', 'auto')
        if _native is not None and hasattr(_native, 'wgrad') and (mode == '1' or (mode != '0' and w_shape[1] <= 64)):
            return _native.wgrad(x, dy, tuple(w_shape), padding, groups)
        w_stub = torch.empty(w_shape, dtype=x.dtype, device=x.device)
        return torch.ops.aten.convolution_backward(dy, x, w_stub, None, [1, 1], list(padding), [1, 1], False, [0, 0], groups,
                                                   [False, True, False])[1]

    @staticmethod
    def backward(ctx, ggw):
        dy, x = ctx.saved_tensors
        w_shape, padding, groups = ctx.cfg
        d_dy = d_x = None
        if ctx.needs_input_grad[0]:
            d_dy = _Conv2d.apply(x, ggw, padding, groups)
        if ctx.needs_input_grad[1]:
            d_x = _Conv2dDgrad.apply(dy, ggw, x.shape, padding, groups)
        return d_dy, d_x, None, None, None


def conv_transpose2d(input, weight, bias=None, stride=1, padding=0, output_padding=0, groups=1, dilation=1):
    if input.device.type == 'cuda' and os.environ.get('LVG_NATIVE_CONV', '1') != '0':
        from . import conv_nd
        return conv_nd.conv_transpose2d(input, weight, bias, stride, padding, output_padding, groups, dilation)
    return torch.nn.functional.conv_transpose2d(input=input, weight=weight, bias=bias, stride=stride, padding=padding,
                                                output_padding=output_padding, groups=groups, dilation=dilation)
