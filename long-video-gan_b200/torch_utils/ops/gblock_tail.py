"""Tail of the low-res generator's residual block as one native op.

Not a module of the reference's ``torch_utils.ops``. After its two modulated convolutions ``Synthesis3dResBlock.forward``
(generator_lres.py:577-589) runs

  hidden = (skip + hidden) * sqrt(0.5)                 ATen add + mul
  hidden = TemporalLinearUpsample(hidden)              upfirdn2d, up (1, 2), [1,3,3,1]/8, gain 2     (temporal_up)
  hidden = center_crop(hidden, seq_length=...)
  hidden = SpatialBilinearUpsample(hidden)             upfirdn2d, up 2, gain 4                       (spatial_up)
  hidden = center_crop(hidden, width=..., height=...)
  output = bias_act(hidden, bias_1, act, clamp=256)

each a full pass over memory, the crops discarding part of what the upsamplings computed. ``gblock_tail`` computes the
output only at kept positions in one pass (csrc/gblock_tail.cu): it reads ``skip`` and ``hidden`` once and writes the
output and, when a backward pass follows, 2-bit codes of the activation (bias_act's). The backward pass is one native call
that returns the common gradient of ``skip`` and ``hidden`` and a deterministic bias gradient; only the codes are saved.
With ``create_graph=True`` the backward pass is recorded from differentiable torch ops, so gradients of any order work.
CPU tensors, fp64 and other activations run ``_reference``, the reference's own op sequence (also the tests' oracle).

``install(...)`` makes an unmodified ``Synthesis3dResBlock.forward`` run this op, with the magnitude-EMA gain of the block
input folded into the first modulated convolution and the skip weight instead of a pass over the input.
"""
import math

import torch

from .. import custom_ops
from . import _install
from . import bias_act as _bias_act
from . import conv_nd
from . import upfirdn2d

TUP, SUP = custom_ops.GblockTailPlugin.TUP, custom_ops.GblockTailPlugin.SUP
_ACTS = {'lrelu': 3, 'linear': 1}           # LVG_ACT_LRELU, LVG_ACT_LINEAR
_FILTER = (0.125, 0.375, 0.375, 0.125)      # LinearResample(scale=2).filter


def _plugin():
    return custom_ops.get_plugin('gblock_tail_plugin')


def out_shape(in_size, temporal_up, spatial_up, seq_length, height, width):
    """(T_out, H_out, W_out) of the tail for an input of (T, H, W), and the crop offsets, as center_crop computes them."""
    t, h, w = in_size
    tu, hu, wu = (2 * t if temporal_up else t), (2 * h if spatial_up else h), (2 * w if spatial_up else w)
    to = tu if seq_length is None else int(seq_length)
    ho = hu if height is None else int(height)
    wo = wu if width is None else int(width)
    return (to, ho, wo), ((tu - to) // 2, (hu - ho) // 2, (wu - wo) // 2)


def _crop(x, width=None, height=None, seq_length=None):
    """generator_lres.center_crop on [N, C, T, H, W]."""
    if width is not None:
        x0 = (x.size(4) - width) // 2
        x = x[:, :, :, :, x0:x0 + width]
    if height is not None:
        y0 = (x.size(3) - height) // 2
        x = x[:, :, :, y0:y0 + height]
    if seq_length is not None:
        t0 = (x.size(2) - seq_length) // 2
        x = x[:, :, t0:t0 + seq_length]
    return x


def _linear_map(m, temporal_up, spatial_up, seq_length, height, width):
    """crop_HW(U_HW crop_T(U_T m)) with the reference's ops (TemporalLinearUpsample, SpatialBilinearUpsample)."""
    f = torch.tensor(_FILTER, dtype=torch.float32, device=m.device)
    if temporal_up:
        n, c, t, h, w = m.shape
        m = upfirdn2d.upsample2d(m.reshape(n, c, t, h * w), f[:, None], up=(1, 2), padding=(0, 0)).reshape(n, c, 2 * t, h, w)
    m = _crop(m, seq_length=seq_length)
    if spatial_up:
        n, c, t, h, w = m.shape
        m = upfirdn2d.upsample2d(m.reshape(n, c * t, h, w), f, up=2, padding=0).reshape(n, c, t, 2 * h, 2 * w)
    return _crop(m, width=width, height=height)


def _reference(s, h, b, temporal_up, spatial_up, seq_length, height, width, act, clamp):
    """The reference's op sequence (generator_lres.py:579-589). Differentiable; the oracle of the tests and the path of
    CPU tensors, fp64 and activations other than lrelu / linear."""
    m = (s + h) * math.sqrt(0.5)
    v = _linear_map(m, temporal_up, spatial_up, seq_length, height, width)
    return _bias_act.bias_act(v, b, act=act, clamp=clamp)


def _decode_codes(codes, numel, dtype):
    """The 2-bit code of every element of z from lvg_bias_act_fwd_codes' layout (see code_byte in csrc/gblock_tail.cu)."""
    e = torch.arange(numel, device=codes.device)
    g = e >> 2
    if dtype == torch.float16:
        pk = g >> 1
        byte = (((pk >> 10) << 8) + (pk & 255)) * 8 + ((pk >> 8) & 3) * 2 + (g & 1)
    else:
        pk = g
        byte = (((pk >> 10) << 8) + (pk & 255)) * 4 + ((pk >> 8) & 3)
    return (codes[byte].long() >> (2 * (e & 3))) & 3


def _act_params(act):
    spec = _bias_act.activation_funcs[act]
    return float(spec.def_alpha), float(spec.def_gain)


class _Tail(torch.autograd.Function):
    """z = bias_act(L((s + h) sqrt(1/2)), b) with L the upsamplings and crops. Saves only the codes."""

    @staticmethod
    def forward(ctx, s, h, b, cfg):
        flags, out_size, act, clamp = cfg
        alpha, gain = _act_params(act)
        want = any(ctx.needs_input_grad[:3])
        z, codes = _plugin().forward(s, h, None if b is None else b.float(), out_size, flags, _ACTS[act], alpha, gain,
                                     -1.0 if clamp is None else clamp, want)
        ctx.save_for_backward(codes)
        ctx.cfg = cfg
        ctx.in_size = tuple(s.shape[2:])
        ctx.b_dtype = None if b is None else b.dtype
        return z

    @staticmethod
    def backward(ctx, dz):
        codes, = ctx.saved_tensors
        flags, out_size, act, clamp = ctx.cfg
        alpha, gain = _act_params(act)
        if not torch.is_grad_enabled():
            dm, db = _plugin().adjoint(dz, codes, ctx.in_size, flags, _ACTS[act], alpha, gain)
        else:
            # differentiable composition (gradients of higher order): dv = dz * bias_act'(codes), dm = sqrt(1/2) L^T dv
            code = _decode_codes(codes, dz.numel(), dz.dtype).view(dz.shape)
            slope = torch.where((code & 1).bool(), alpha, 1.0) if act == 'lrelu' else torch.ones_like(code, dtype=torch.float32)
            mask = torch.where((code & 2).bool(), 0.0, slope * gain).to(dz.dtype)
            dv = dz * mask
            n, c = dz.shape[:2]
            with torch.enable_grad():
                x0 = torch.zeros([n, c, *ctx.in_size], dtype=dz.dtype, device=dz.device, requires_grad=True)
                y = _linear_map(x0, bool(flags & TUP), bool(flags & SUP), *out_size)
                dm = torch.autograd.grad(y, [x0], dv, create_graph=True)[0] * math.sqrt(0.5)
            db = dv.sum(dim=(0, 2, 3, 4), dtype=torch.float32)
        gs = dm if ctx.needs_input_grad[0] else None
        gh = dm if ctx.needs_input_grad[1] else None
        gb = db.to(ctx.b_dtype) if (ctx.b_dtype is not None and ctx.needs_input_grad[2]) else None
        return gs, gh, gb, None


def native(s, act):
    """The native kernels take the call: CUDA fp16 / fp32 tensors and lrelu or linear."""
    return s.is_cuda and s.dtype in (torch.float16, torch.float32) and act in _ACTS


def gblock_tail(s, h, b, *, temporal_up, spatial_up, seq_length=None, height=None, width=None, act='lrelu', clamp=256.0):
    """bias_act(crop_HW(U_HW crop_T(U_T (s + h) sqrt(1/2))), b, act, clamp=clamp) for s, h [N, C, T, H, W] and b [C]:
    the tail of Synthesis3dResBlock.forward. seq_length / height / width: the centre crops (None = keep the axis)."""
    if not native(s, act) or s.dtype != h.dtype or s.device != h.device:
        return _reference(s, h, b, temporal_up, spatial_up, seq_length, height, width, act, clamp)
    (to, ho, wo), _ = out_shape(tuple(s.shape[2:]), temporal_up, spatial_up, seq_length, height, width)
    flags = (TUP if temporal_up else 0) | (SUP if spatial_up else 0)
    return _Tail.apply(s, h, b, (flags, (to, ho, wo), act, None if clamp is None else float(clamp)))


# ---------------------------------------------------------------------------------------------------- install

def applies(block, input, dtype, out_seq_length):
    """The installed forward takes the call: a CUDA 5-D input computed in fp16 / fp32, lrelu or linear, resamplers with
    scale 2 and no padding, crops no larger than their axes, and a shape the kernels plan (workspace query)."""
    if not (isinstance(input, torch.Tensor) and input.is_cuda and input.ndim == 5 and dtype in (torch.float16, torch.float32)):
        return False
    if block.activation not in _ACTS:
        return False
    for flag, name in ((block.temporal_up, 'temporal_upsample'), (block.spatial_up, 'spatial_upsample')):
        r = getattr(block, name, None) if flag else None
        if flag and (r is None or r.scale != 2 or r.padding != 0):
            return False
    n, _, t, h, w = input.shape
    tu, hu, wu = (2 * t if block.temporal_up else t), (2 * h if block.spatial_up else h), (2 * w if block.spatial_up else w)
    (to, ho, wo), _ = out_shape((t, h, w), block.temporal_up, block.spatial_up, out_seq_length, block.out_height, block.out_width)
    if not (1 <= to <= tu and 1 <= ho <= hu and 1 <= wo <= wu):
        return False
    flags = (TUP if block.temporal_up else 0) | (SUP if block.spatial_up else 0)
    return _plugin().workspace(n, block.out_channels, t, h, w, to, ho, wo, flags) >= 0


def block_forward(block, g, input, latent, magnitude_ema_beta=1.0, out_seq_length=None, dtype=None):
    """Synthesis3dResBlock.forward with the tail as ``gblock_tail`` and the block input's magnitude-EMA gain folded into the
    first modulated convolution (``input_gain=``) and the skip weight. ``g``: the globals of the model module (its
    ``misc``, ``einops``, ``temporal_modulated_conv3d`` and ``bias_act_wrapper``, whatever they are patched to). The same
    MagnitudeEMA calls and affine layers as the reference, in its order."""
    misc, einops = g['misc'], g['einops']
    misc.assert_shape(input, (None, block.in_channels, None, None, None))
    batch_size, in_seq_length = input.size(0), input.size(2)
    misc.assert_shape(latent, (batch_size, block.latent_dim, in_seq_length))

    latent = einops.rearrange(latent, "n c t -> (n t) c")
    style_0 = block.affine_0(latent)
    style_0 = einops.rearrange(style_0, "(n t) c -> n c t", t=in_seq_length)

    dtype = dtype if dtype is not None else (torch.float16 if block.use_float16 and input.is_cuda else torch.float32)
    input = input.type(dtype)
    input_gain_0 = block.input_magnitude_ema_0(input, magnitude_ema_beta) if block.magnitude_ema else None

    hidden = g['temporal_modulated_conv3d'](input, block.weight_0, style_0, input_gain_0, block.padding, demodulate=True)
    bias_0 = block.bias_0.type(hidden.dtype)
    hidden = g['bias_act_wrapper'](hidden, bias_0, act=block.activation, clamp=block.activation_clamp)

    style_1 = block.affine_1(latent)
    style_1 = einops.rearrange(style_1, "(n t) c -> n c t", t=in_seq_length)
    input_gain_1 = block.input_magnitude_ema_1(hidden, magnitude_ema_beta) if block.magnitude_ema else None
    hidden = g['temporal_modulated_conv3d'](hidden, block.weight_1, style_1, input_gain_1, block.padding, demodulate=True)

    weight_skip = block.weight_skip * block.weight_skip_gain
    if input_gain_0 is not None:
        weight_skip = weight_skip * input_gain_0
    skip = conv_nd.conv3d(input, weight_skip.type(input.dtype))

    bias_1 = block.bias_1.type(hidden.dtype)
    output = gblock_tail(skip, hidden, bias_1, temporal_up=block.temporal_up, spatial_up=block.spatial_up,
                         seq_length=out_seq_length, height=block.out_height, width=block.out_width, act=block.activation,
                         clamp=block.activation_clamp)
    misc.assert_shape(output, (None, block.out_channels, None, block.out_height, block.out_width))
    return output


def _forward(orig):
    g = _install.reference_function(orig).__globals__

    def forward(self, input, latent, magnitude_ema_beta=1.0, out_seq_length=None, dtype=None):
        dt = dtype if dtype is not None else (torch.float16 if self.use_float16 and input.is_cuda else torch.float32)
        if not applies(self, input, dt, out_seq_length):
            return orig(self, input, latent, magnitude_ema_beta, out_seq_length, dtype)
        return block_forward(self, g, input, latent, magnitude_ema_beta, out_seq_length, dtype)
    return forward


def install(*targets):
    """Make ``Synthesis3dResBlock.forward`` run ``block_forward``. ``targets``: the module ``model.generator_lres`` or
    generator / block instances, found by ``_install.find_classes``. Calls outside ``applies`` (CPU tensors, fp64, other
    activations, resamplers with padding or another scale) run the original method. Idempotent; the original stays
    reachable as ``.forward.lvg_gblock_tail``. Returns the patched classes."""
    classes = _install.find_classes(targets, 'Synthesis3dResBlock')
    for cls in classes:
        _install.wrap(cls, 'forward', 'lvg_gblock_tail', _forward)
    return classes
