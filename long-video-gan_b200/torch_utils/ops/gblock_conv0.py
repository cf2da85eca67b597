"""The first layer of the low-res generator's residual block as one native op.

Not a module of the reference's ``torch_utils.ops``. ``Synthesis3dResBlock.forward`` (generator_lres.py:568-575) begins

  hidden = temporal_modulated_conv3d(input, weight_0, style_0, ...)     y' = d * conv(a * x, w)
  hidden = bias_act(hidden, bias_0, act='lrelu', clamp=256)             a full pass: read y', write y
  input_gain_1 = input_magnitude_ema_1(hidden, beta)                    beta != 1: square() and mean(), two more passes

``gblock_conv0`` computes y = clamp(act(d * conv(a * x, w) + b) * gain) on the convolution engine (csrc/gblock_conv0.cu,
lvg_gblock_conv0_*): the bias, the activation, the gain and the clamp are applied in the epilogue that applies d, so the
pre-activation is never stored. On request one more pass reads y back and sums its squares as stored (fixed-order fold, no
host synchronisation): the statistic ``input_magnitude_ema_1`` needs, in place of its ``square()`` and ``mean()``. The
first-order backward is one native call: one pass over (dy, y) gives db and the gradient of d, and the convolution gradients
re-tile dy with bias_act's gradient G(y) and d, so dz = G(y) dy is never written; db is summed in a fixed order (bitwise
reproducible). Only y is saved. With
create_graph=True the backward is recorded as ``conv_nd._BiasActGrad`` followed by ``modulated_conv.backward_graph``, so
gradients of any order work.

fp16: the reference rounds d * conv to fp16 before the bias; the op does not, so the two agree to one rounding of fp16.

``install(...)`` makes an unmodified ``Synthesis3dResBlock.forward`` run the op in the calls ``_takes`` routes to it
(DESIGN.md 7m); with ``gblock_tail.install`` as well, the block runs the fused first layer and the fused tail.
"""
import functools
import math

import torch

from .. import custom_ops
from . import _install, bias_act, conv_nd, gblock_tail, lres_torgb, modulated_conv

_MODES = ('backward', 'stat', 'forward')    # the calls install routes to the op (DESIGN.md 7m)
_BACKWARD_MAX_CHANNELS = 128                # ... 'backward' only for blocks of at most this many channels (DESIGN.md 7m)
_ACTS = {'linear': 1, 'lrelu': 2}           # the engine epilogue's codes


def _plugin():
    return custom_ops.get_plugin('gblock_conv0_plugin')


def _act_params(act):
    spec = bias_act.activation_funcs[act]
    return float(spec.def_alpha), float(spec.def_gain)


def supported(x, dtype, weight_shape, padding, act):
    """The op takes the call: x [N, Cin, T, H, W] on CUDA computed in fp16 / fp32 (``dtype``, x's after the block's cast),
    linear or lrelu, and a shape inside the engine's modulated-convolution envelope with the input's frame count (size
    query of lvg_gblock_conv0), native convolutions not switched off (LVG_NATIVE_CONV=0)."""
    if not (isinstance(x, torch.Tensor) and x.ndim == 5 and conv_nd.enabled_for(x) and len(weight_shape) == 5):
        return False
    if dtype not in (torch.float16, torch.float32) or act not in _ACTS:
        return False
    n, cin, t, h, w = x.shape
    if int(weight_shape[1]) != cin:
        return False
    return _plugin().workspace(dtype, n, cin, int(weight_shape[0]), t, h, w, tuple(weight_shape[2:]), tuple(padding)) >= 0


def composition(x, w, a, d, b, padding, act, clamp):
    """The formulation the op replaces: ``modulated_conv`` (d * conv(a * x, w) on the engine), then ``bias_act``."""
    y = modulated_conv.modulated_conv(x, w, a, d, tuple(padding))
    return bias_act.bias_act(y, b, act=act, clamp=clamp)


class _Conv0(torch.autograd.Function):
    """y = clamp(act(d * conv(a * x, w) + b) * gain): x [N, Cin, T, H, W] and w in one dtype (fp16 / fp32), a [N, Cin, T],
    d [N, Cout, T] and b [Cout] (or None) fp32. Saves y (bias_act's gradient rule)."""

    @staticmethod
    def forward(ctx, x, w, a, d, b, cfg):
        padding, act, clamp = cfg
        alpha, gain = _act_params(act)
        y, _ = _plugin().fprop(x, w, a, d, b, padding, _ACTS[act], alpha, gain, -1.0 if clamp is None else clamp)
        ctx.save_for_backward(x, w, a, d, b, y)
        ctx.cfg = cfg
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, a, d, b, y = ctx.saved_tensors
        padding, act, clamp = ctx.cfg
        alpha, gain = _act_params(act)
        need = ctx.needs_input_grad
        want_dw = need[1] and not conv_nd._weights_off()
        if not torch.is_grad_enabled():
            dx, dw, da, dd, db = _plugin().backward(x, w, a, d, b, y, dy, padding, _ACTS[act], alpha, gain, -1.0 if clamp is None else clamp,
                                                    want_dw=want_dw, want_dd=need[3], want_db=need[4])
            return (dx if need[0] else None), dw, (da if need[2] else None), dd, db, None
        # differentiable composition (double backward through the generator): dz = G(y) dy, then the modulated
        # convolution's gradients of dz
        bias_act._init()
        dz = conv_nd._BiasActGrad.apply(dy, y, (act, alpha, gain, clamp))
        dx, dw, da, dd = modulated_conv.backward_graph(x, w, a, d, dz, padding, need[0] or need[2], want_dw, need[3])
        db = dz.float().sum(dim=(0, 2, 3, 4)) if need[4] else None
        return (dx if need[0] else None), dw, (da if need[2] else None), dd, db, None


def gblock_conv0(x, w, a, d, b, padding, act='lrelu', clamp=256.0):
    """``bias_act(modulated_conv(x, w, a, d, padding), b, act=act, clamp=clamp)`` in one pass: w [Cout, Cin, kt, kh, kw] in
    x's dtype, a [N, Cin, T] and d [N, Cout, T] (cast to fp32), b [Cout] (cast to fp32) or None, clamp a number or None.
    CUDA only: callers check ``supported``."""
    return _Conv0.apply(x, w, a.float(), d.float(), None if b is None else b.float(),
                        (tuple(int(p) for p in padding), act, None if clamp is None else float(clamp)))


def head(block, g, input, style_0, input_gain_0, magnitude_ema_beta, mode):
    """The block's first layer as the op, called as ``gblock_tail.head``: (y, the gain input_magnitude_ema_1 takes from y or
    None). ``mode`` 'stat' takes the statistic from the op's pass over y and updates the EMA on the device
    (``lres_torgb.track_sumsq``); the other modes run the autograd Function and the EMA module as the reference does."""
    weight, style, demod = modulated_conv.temporal_factors(block.weight_0, style_0)
    a = style if input_gain_0 is None else style * input_gain_0
    wx = weight.type(input.dtype)
    bias_0 = block.bias_0.type(input.dtype)
    clamp = block.activation_clamp
    if mode == 'stat':
        alpha, gain = _act_params(block.activation)
        y, sumsq = _plugin().fprop(input, wx.detach(), a.detach().float(), demod.detach().float(), bias_0.detach().float(), block.padding,
                                   _ACTS[block.activation], alpha, gain, -1.0 if clamp is None else float(clamp), want_sumsq=True)
        return y, lres_torgb.track_sumsq(block.input_magnitude_ema_1, g, sumsq, y.numel(), magnitude_ema_beta)
    y = gblock_conv0(input, wx, a, demod, bias_0, block.padding, block.activation, clamp)
    return y, (block.input_magnitude_ema_1(y, magnitude_ema_beta) if block.magnitude_ema else None)


def block_forward(block, g, input, latent, magnitude_ema_beta=1.0, out_seq_length=None, dtype=None, head=None):
    """Synthesis3dResBlock.forward with its first layer as ``head`` (above, with the mode bound) and the rest as the
    reference's op sequence, for installs without ``gblock_tail``. ``g``: the globals of the model module (its ``misc``,
    ``einops``, ``F``, ``center_crop``, ``temporal_modulated_conv3d`` and ``bias_act_wrapper``, whatever they are patched
    to)."""
    misc, einops = g['misc'], g['einops']
    misc.assert_shape(input, (None, block.in_channels, None, None, None))
    batch_size, in_seq_length = input.size(0), input.size(2)
    misc.assert_shape(latent, (batch_size, block.latent_dim, in_seq_length))

    latent = einops.rearrange(latent, "n c t -> (n t) c")
    style_0 = block.affine_0(latent)
    style_0 = einops.rearrange(style_0, "(n t) c -> n c t", t=in_seq_length)

    dtype = dtype if dtype is not None else (torch.float16 if block.use_float16 and input.is_cuda else torch.float32)
    input = input.type(dtype)
    if block.magnitude_ema:
        input_gain_0 = block.input_magnitude_ema_0(input, magnitude_ema_beta)
        input = input * input_gain_0

    hidden, input_gain_1 = head(block, g, input, style_0, None, magnitude_ema_beta)

    style_1 = block.affine_1(latent)
    style_1 = einops.rearrange(style_1, "(n t) c -> n c t", t=in_seq_length)
    hidden = g['temporal_modulated_conv3d'](hidden, block.weight_1, style_1, input_gain_1, block.padding, demodulate=True)

    weight_skip = (block.weight_skip * block.weight_skip_gain).type(input.dtype)
    input = g['F'].conv3d(input, weight_skip)
    hidden = (input + hidden) * math.sqrt(0.5)

    if block.temporal_up:
        hidden = block.temporal_upsample(hidden)
    hidden = g['center_crop'](hidden, seq_length=out_seq_length)
    if block.spatial_up:
        hidden = block.spatial_upsample(hidden)
    hidden = g['center_crop'](hidden, width=block.out_width, height=block.out_height)

    bias_1 = block.bias_1.type(hidden.dtype)
    output = g['bias_act_wrapper'](hidden, bias_1, act=block.activation, clamp=block.activation_clamp)
    misc.assert_shape(output, (None, block.out_channels, None, block.out_height, block.out_width))
    return output


# ---------------------------------------------------------------------------------------------------- install

mode = lres_torgb.mode      # which of the block's three calls this is: 'backward', 'stat', 'forward' or None


def _takes(block, input, latent, magnitude_ema_beta=1.0, dtype=None):
    """The mode of the call when the op takes it (inside ``supported`` and one of the modes the op measured faster in on
    the H100, ``_MODES``; a backward only in blocks of at most ``_BACKWARD_MAX_CHANNELS`` channels, DESIGN.md 7m), else
    None."""
    if not (isinstance(input, torch.Tensor) and isinstance(latent, torch.Tensor) and input.ndim == 5 and input.is_cuda):
        return None
    if not getattr(block, 'demodulate', True):
        return None
    dt = dtype if dtype is not None else (torch.float16 if block.use_float16 else torch.float32)
    if not supported(input, dt, tuple(block.weight_0.shape), block.padding, block.activation):
        return None
    m = mode(block, input, latent, magnitude_ema_beta)
    if m == 'backward' and block.in_channels > _BACKWARD_MAX_CHANNELS:
        return None
    return m if m in _MODES else None


def _forward(orig):
    g = _install.reference_function(orig).__globals__

    def head_for(self, input, latent, magnitude_ema_beta=1.0, dtype=None):
        m = _takes(self, input, latent, magnitude_ema_beta, dtype)
        return None if m is None else functools.partial(head, mode=m)

    def forward(self, input, latent, magnitude_ema_beta=1.0, out_seq_length=None, dtype=None):
        h = head_for(self, input, latent, magnitude_ema_beta, dtype)
        if h is None:
            return orig(self, input, latent, magnitude_ema_beta, out_seq_length, dtype)
        dt = dtype if dtype is not None else (torch.float16 if self.use_float16 else torch.float32)
        # with gblock_tail installed (below this wrapper; above it, it would have taken the call) the fused tail as well
        if _install.find(orig, 'lvg_gblock_tail') is not None and gblock_tail.applies(self, input, dt, out_seq_length):
            return gblock_tail.block_forward(self, g, input, latent, magnitude_ema_beta, out_seq_length, dtype, head=h)
        return block_forward(self, g, input, latent, magnitude_ema_beta, out_seq_length, dtype, head=h)
    forward.head_for = head_for
    return forward


def install(*targets):
    """Make ``Synthesis3dResBlock.forward`` of generator_lres run the fused first layer in the calls ``_takes`` routes to
    it. ``targets``: the module ``model.generator_lres`` or generator / block instances, found by ``_install.find_classes``
    (which reaches classes ``persistence`` rebuilt from a pickle). Other calls (CPU tensors, fp64, LVG_NATIVE_CONV=0, shapes
    the size query rejects, modes not routed) run the method this wrapper replaced. Composes with ``gblock_tail.install``
    (the block then runs both fused ops), ``modulated_conv.install`` and ``lres_torgb.install`` in any order. Idempotent;
    the replaced method stays reachable as ``.forward.lvg_gblock_conv0``. Returns the patched classes."""
    classes = _install.find_classes(targets, 'Synthesis3dResBlock')
    for cls in classes:
        _install.wrap(cls, 'forward', 'lvg_gblock_conv0', _forward)
    return classes
