"""Tail of the low-res discriminator's residual block as one native op.

Not a module of the reference's ``torch_utils.ops``. After ``conv_1``'s ``F.conv3d`` a ``DiscriminatorBlock``
(discriminator_lres.py:321-333, Conv3dLayer.forward :169-179, Downsample3d.forward :197-213) runs

  y = upfirdn2d.downsample2d(y, f, down=2)             over H, W       (spatial_down)
  y = upfirdn2d.downsample2d(y, f[:, None], down=[1, 2])  over T       (temporal_down)
  hidden = bias_act(y, b, lrelu, clamp=256)
  output = (hidden + skip) * sqrt(0.5)                  ATen add + mul

each a pass over memory, the first over the full-resolution tensor. ``dblock_tail`` reads y and skip once and writes the
output and, when a backward pass follows, 2-bit codes of the activation (csrc/dblock_tail.cu). The map is piecewise
linear, so three Functions over two kernels close its gradients of every order: ``_Tail`` (the forward), ``_TailAdjoint``
(dy, dskip and a deterministic db from dz and the codes) and ``_TailLinear`` (the forward with the slopes read from the
codes), each the backward of the other. Only the codes and the filter are saved; y is not. CPU tensors, fp64, other
activations, other filter lengths and odd extents run ``_reference``, the reference's own op sequence.

``install(...)`` does two things to an unmodified discriminator. Its ``Conv3dLayer``s without downsampling (``conv_0``) run
``conv_nd.conv_bias_act``, bias_act in the convolution's epilogue, where the engine takes the layer anyway and the
measurement says it pays (``epilogue_faster``: calls that record no gradient). Its ``DiscriminatorBlock.forward`` runs this op after ``conv_1``'s
convolution where that is measured faster (``faster``: nowhere on an H100 so far, DESIGN.md 7g) or, with ``tail=True``,
wherever the op takes the block: the caller then pays the measured cost for a bias gradient summed in a fixed order.
"""
import math

import torch

from .. import custom_ops
from . import bias_act as _bias_act
from . import conv3d_down, conv_nd, upfirdn2d

_P = custom_ops.DblockTailPlugin
_ACTS = {'lrelu': 3, 'linear': 1}           # LVG_ACT_LRELU, LVG_ACT_LINEAR


def _plugin():
    return custom_ops.get_plugin('dblock_tail_plugin')


def _reference(y, s, b, f, spatial_down, temporal_down, act, clamp, alpha=None, gain=None):
    """The reference's op sequence, in its order. Differentiable; the path of CPU tensors, fp64, other activations, other
    filter lengths and odd extents."""
    n, c, t, h, w = y.shape
    if spatial_down:
        y = upfirdn2d.downsample2d(y.reshape(n, c * t, h, w), f, down=2)
        h, w = y.shape[2:]
        y = y.reshape(n, c, t, h, w)
    if temporal_down:
        y = upfirdn2d.downsample2d(y.reshape(n, c, t, h * w), f[:, None], down=[1, 2])
        y = y.reshape(n, c, y.shape[2], h, w)
    y = _bias_act.bias_act(y, b, act=act, alpha=alpha, gain=gain, clamp=clamp)
    if s is not None:
        y = (y + s) * math.sqrt(0.5)
    return y


# cfg: (flags, act id, alpha, gain, clamp) as the plugin takes them

class _Tail(torch.autograd.Function):
    """z = scale (bias_act(P y, b) + s). Saves the codes and f."""

    @staticmethod
    def forward(ctx, y, s, b, f, cfg):
        flags, act, alpha, gain, clamp = cfg
        want = any(ctx.needs_input_grad[:3])
        z, codes = _plugin().forward(y, s, b, f, flags, act, alpha, gain, clamp,
                                     _P.WRITE if want else _P.NONE)
        if want:
            ctx.save_for_backward(codes, f)
        ctx.cfg = cfg
        ctx.in_size = tuple(y.shape[2:])
        ctx.b_dtype = None if b is None else b.dtype
        return z

    @staticmethod
    def backward(ctx, dz):
        codes, f = ctx.saved_tensors
        want_ds = ctx.needs_input_grad[1]
        dy, ds, db = _TailAdjoint.apply(dz, codes, f, ctx.cfg, ctx.in_size, want_ds)
        return (dy if ctx.needs_input_grad[0] else None, ds if want_ds else None,
                db.to(ctx.b_dtype) if ctx.needs_input_grad[2] else None, None, None)


class _TailAdjoint(torch.autograd.Function):
    """dy = P^T dv, ds = scale dz, db = sum of dv with dv = scale G dz and G from the codes. Linear in dz: its backward is
    ``_TailLinear``."""

    @staticmethod
    def forward(ctx, dz, codes, f, cfg, in_size, want_ds):
        flags, act, alpha, gain, _ = cfg
        ctx.save_for_backward(codes, f)
        ctx.cfg = cfg
        dy, ds, db = _plugin().adjoint(dz, codes, f, in_size, flags, act, alpha, gain, want_ds)
        return dy, ds, db

    @staticmethod
    def backward(ctx, g_dy, g_ds, g_db):
        if not ctx.needs_input_grad[0]:
            return None, None, None, None, None, None
        codes, f = ctx.saved_tensors
        return _TailLinear.apply(g_dy, g_ds, g_db, codes, f, ctx.cfg), None, None, None, None, None


class _TailLinear(torch.autograd.Function):
    """scale (G (P u + beta) + sigma) with G from the codes. Linear in u, sigma and beta: its backward is ``_TailAdjoint``."""

    @staticmethod
    def forward(ctx, u, sigma, beta, codes, f, cfg):
        flags, act, alpha, gain, _ = cfg
        ctx.save_for_backward(codes, f)
        ctx.cfg = cfg
        ctx.in_size = tuple(u.shape[2:])
        ctx.beta_dtype = None if beta is None else beta.dtype
        z, _ = _plugin().forward(u, sigma, beta, f, flags, act, alpha, gain, -1.0, _P.READ, codes)
        return z

    @staticmethod
    def backward(ctx, g):
        codes, f = ctx.saved_tensors
        want_ds = ctx.needs_input_grad[1]
        dy, ds, db = _TailAdjoint.apply(g, codes, f, ctx.cfg, ctx.in_size, want_ds)
        return (dy if ctx.needs_input_grad[0] else None, ds if want_ds else None,
                db.to(ctx.beta_dtype) if ctx.needs_input_grad[2] else None, None, None, None)


def _flags(spatial_down, temporal_down, merge):
    return (_P.TDOWN if temporal_down else 0) | (_P.SDOWN if spatial_down else 0) | (_P.MERGE if merge else 0)


def native(y, s, f, spatial_down, temporal_down, act):
    """The native kernels take the call: CUDA fp16 / fp32 tensors of one dtype and device, lrelu or linear, 4 taps, and a
    shape the kernels plan (even extents on the filtered axes)."""
    if not (y.is_cuda and y.ndim == 5 and y.dtype in (torch.float16, torch.float32) and act in _ACTS):
        return False
    if (spatial_down or temporal_down) and (f is None or f.ndim != 1 or f.numel() != 4 or f.device != y.device):
        return False
    flags = _flags(spatial_down, temporal_down, s is not None)
    if _plugin().codes_bytes(*y.shape, flags) < 0:
        return False
    return s is None or (s.dtype == y.dtype and s.device == y.device
                         and tuple(s.shape) == (*y.shape[:2], *_P.out_size(tuple(y.shape[2:]), flags)))


def dblock_tail(y, s, b, f, *, spatial_down, temporal_down, act='lrelu', clamp=256.0, alpha=None, gain=None):
    """``(bias_act(Downsample3d(spatial_down, temporal_down)(y), b, act, clamp=clamp) + s) * sqrt(0.5)`` for the convolution
    output y [N, C, T, H, W], the skip tensor s at the output resolution, b [C] or None and Downsample3d's filter f (None where no axis is halved): the
    tail of DiscriminatorBlock.forward. ``s=None``: no merge and no sqrt(0.5), the tail of a Conv3dLayer. alpha / gain
    default per activation as in bias_act. Gradients of any order with respect to y, s and b."""
    if not native(y, s, f, spatial_down, temporal_down, act):
        return _reference(y, s, b, f, spatial_down, temporal_down, act, clamp, alpha, gain)
    _, alpha, gain, clamp = _bias_act._resolve(act, alpha, gain, clamp)
    cfg = (_flags(spatial_down, temporal_down, s is not None), _ACTS[act], alpha, gain, clamp)
    return _Tail.apply(y, s, b, f.float() if spatial_down or temporal_down else None, cfg)


# ---------------------------------------------------------------------------------------------------- install

def faster(y_shape):
    """Which conv_1 outputs [N, C, T, H, W] take the op for speed. None so far: on an H100 (700 W) the four blocks of the
    default VideoDiscriminator(seq_length=128, max_edge=64) at batch 8 measured 2-12 % slower on the op in forward,
    forward + backward and the R1 pattern (DESIGN.md 7g): the tiled upfirdn2d kernels of the reference composition move the
    full-resolution tensor faster than this op's walk does."""
    return False


def applies(block, input):
    """The op can take the block: a 5-D input, a conv_1 with odd kernels that keeps the reference composition
    (``conv3d_down.faster`` layers run the decomposition instead), a 4-tap filter and even extents on the axes it
    halves."""
    c1 = block.conv_1
    if not (isinstance(input, torch.Tensor) and input.ndim == 5) or any(k % 2 == 0 for k in c1.weight.shape[2:]):
        return False
    down = c1.spatial_down or c1.temporal_down
    if down and (conv3d_down.faster(c1.weight.shape) or c1.downsample._downsample_filter.numel() != 4):
        return False
    _, _, t, h, w = input.shape
    return not (c1.temporal_down and t % 2) and not (c1.spatial_down and (h % 2 or w % 2))


def routed(block, input, tail):
    """The installed forward runs ``block_forward``: inside ``applies``, and for CUDA inputs only where the op is ``faster``
    or the caller of ``install`` asked for it (``tail``)."""
    if not applies(block, input):
        return False
    if not input.is_cuda:
        return True                                  # the composition, the reference's own ops
    return bool(tail) or faster((input.shape[0], block.conv_1.out_channels, *input.shape[2:]))


def block_forward(block, input):
    """DiscriminatorBlock.forward with the tail as ``dblock_tail``: the same modules, casts and order as the reference up to
    conv_1's convolution."""
    assert input.dim() == 5
    dtype = torch.float16 if block.use_fp16 else torch.float32
    input = input.type(dtype)
    if block.vid_channels > 0:
        input = block.conv_vid(input)
    hidden = block.conv_0(input)
    skip = block.conv_skip(input)
    c1 = block.conv_1
    weight = (c1.weight * c1.weight_gain).type(hidden.dtype)
    y = conv_nd.conv3d(hidden, weight, padding=c1.padding)
    f = c1.downsample._downsample_filter if c1.spatial_down or c1.temporal_down else None
    bias = c1._bias.type(hidden.dtype) if c1.bias else None
    return dblock_tail(y, skip, bias, f, spatial_down=c1.spatial_down, temporal_down=c1.temporal_down, act=c1.activation,
                       clamp=c1.conv_clamp)


def _forward(orig):
    def forward(self, input):
        if not routed(self, input, forward.tail):
            return orig(self, input)
        return block_forward(self, input)
    forward.lvg_dblock_tail = orig
    forward.tail = False
    return forward


def epilogue_faster(layer, input):
    """Which full-resolution layers take bias_act in the convolution's epilogue for speed: those whose call records no
    gradient. On an H100 (700 W, DESIGN.md 7g) the forward of blocks 0 and 1 of the default D at batch 8 gained 1 % (8.86 ->
    8.77, 9.64 -> 9.53 ms) and the others did not move, but forward + backward and the R1 pattern lost up to 1.5 % (block 0:
    25.27 -> 25.64, 51.90 -> 52.55 ms; whole D 75.98 -> 76.77, 179.39 -> 180.08 ms): conv_bias_act's backward sums the bias
    gradient in a pass of its own, which bias_act's fused gradient kernel does not need."""
    params = [layer.weight] + ([layer._bias] if layer.bias else [])
    return not (torch.is_grad_enabled() and (input.requires_grad or any(p.requires_grad for p in params)))


def epilogue_applies(layer, input):
    """``Conv3dLayer.forward`` runs ``conv_nd.conv_bias_act``: a layer without downsampling, lrelu or linear, a CUDA fp16 /
    fp32 input, and a convolution the engine takes without being asked for the epilogue (route ``engine`` of
    ``lvg_convnd_route``), so that asking for it never takes a layer off a faster route: the 1x1x1 ``conv_vid`` stays on the
    streaming kernels, which have no epilogue."""
    if layer.spatial_down or layer.temporal_down or layer.activation not in _ACTS:
        return False
    if not (isinstance(input, torch.Tensor) and input.ndim == 5 and input.dtype in (torch.float16, torch.float32)
            and conv_nd.enabled_for(input)):
        return False
    pad = tuple(int(p) for p in layer.padding)
    if not custom_ops.ConvNdPlugin._in_envelope(tuple(input.shape), tuple(layer.weight.shape), input.dtype, 1, pad, 1, 1):
        return False
    if conv_nd._get_plugin().route('fprop', tuple(input.shape), tuple(layer.weight.shape), pad, 1, input.dtype, epilogue=False) != 'engine':
        return False
    return epilogue_faster(layer, input)


def _layer_forward(orig):
    def forward(self, input):
        if not epilogue_applies(self, input):
            return orig(self, input)
        weight = (self.weight * self.weight_gain).type(input.dtype)
        bias = self._bias.type(input.dtype) if self.bias else None
        return conv_nd.conv_bias_act(input, weight, bias, padding=self.padding, act=self.activation, clamp=self.conv_clamp)
    forward.lvg_conv_bias_act = orig
    return forward


def install(*targets, tail=False):
    """Patch the classes of an unmodified low-res discriminator. ``targets``: the module ``model.discriminator_lres`` or
    ``nn.Module`` instances (the classes of their submodules are found by name, which reaches networks that ``persistence``
    reconstructed from a pickle).

    ``Conv3dLayer.forward``: layers inside ``epilogue_applies`` run ``conv_nd.conv_bias_act``; every other layer runs the
    method this one replaced, so ``conv3d_down.install`` (the layers with downsampling) wraps or is wrapped by it in either
    order. ``DiscriminatorBlock.forward``: blocks inside ``routed`` run ``block_forward`` with ``conv_vid``, ``conv_0`` and
    ``conv_skip`` as the block's modules; ``tail=True`` routes every block the op takes to it although it measured slower
    (DESIGN.md 7g), for its bitwise reproducible bias gradient. Opt-in and idempotent (a later call sets ``tail`` anew); the
    originals stay reachable as ``.forward.lvg_dblock_tail`` and ``.forward.lvg_conv_bias_act``. Returns the patched
    classes, blocks first."""
    blocks, layers = [], []
    for t in targets:
        for name, into in (('DiscriminatorBlock', blocks), ('Conv3dLayer', layers)):
            if isinstance(t, torch.nn.Module):
                found = [type(m) for m in t.modules() if type(m).__name__ == name]
            else:
                found = [getattr(t, name)] if getattr(t, name, None) is not None else []
            for cls in found:
                if not any(cls is c for c in into):
                    into.append(cls)
    for cls in blocks:
        if getattr(cls.forward, 'lvg_dblock_tail', None) is None:
            cls.forward = _forward(cls.forward)
        cls.forward.tail = bool(tail)
    for cls in layers:
        if not conv3d_down.wrapped_by(cls.forward, 'lvg_conv_bias_act'):
            cls.forward = _layer_forward(cls.forward)
    return blocks + layers
