"""Residual block of the super-res discriminator as native layers.

Not a module of the reference's ``torch_utils.ops``. A ``DiscriminatorBlock`` with ``architecture='resnet'``
(discriminator_sres.py:300-349, Conv2dLayer.forward :184-206, conv2d_resample's plan) runs

  y  = conv2d(upfirdn2d(x, f, down=2, padding=1), w_skip)                                 skip (1x1, no bias, linear)
  h0 = bias_act(conv2d(x, w0, padding=1), b0, lrelu, gain, clamp)                           conv0
  h1 = bias_act(conv2d(upfirdn2d(h0, f, padding=2), w1, stride=2), b1, lrelu, gain, clamp)   conv1
  out = (h1 + y) * sqrt(0.5)                                                                 ATen add + mul

``sres_dblock`` computes the same block with three native calls after the skip's FIR, in one autograd Function:

  conv0  the convolution engine with bias_act in its epilogue.
  conv1  ``lvg_sres_dblock_conv1``: the FIR runs inside the convolution's re-tiling pass, so the filtered
         Cin x (H + 1) x (W + 1) image is never written; bias_act in the strided convolution's epilogue.
  skip   ``lvg_sres_dblock_skip``: the 1x1 convolution on the pointwise wgmma kernels with the residual merge
         ``(acc + h1) * sqrt(0.5)`` in its epilogue.

The first-order backward is native (``_Block``): conv1's weight gradient re-tiles the filtered image from h0 through the FIR
pass (``lvg_sres_dblock_conv1_backward``), the FIR adjoint runs fused with conv0's activation gradient and a fixed-order
bias gradient (``lvg_sres_dblock_fir_adjoint_act``), and sqrt(0.5) is folded into conv1's activation-gradient gain and the
skip's weights. With create_graph=True the backward is recorded from differentiable Functions that exist already
(``conv_nd``'s convolution gradients and ``_BiasActGrad``, ``upfirdn2d``), as ``conv_nd._ConvBiasAct`` does, so gradients
of any order work. ``conv2d_gradfix.no_weight_gradients`` is honoured.

``install(...)`` patches ``DiscriminatorBlock.forward`` (resnet blocks, where ``faster`` says the op pays) and
``Conv2dLayer.forward`` (the layers outside the blocks that the convolution engine takes: the epilogue's 3x3 ``conv``) of
an unmodified discriminator.
"""
import numpy as np
import torch

from .. import custom_ops
from . import bias_act as _bias_act
from . import _install, conv2d_resample, conv_nd, upfirdn2d

_SQRT_HALF = float(np.sqrt(0.5))             # the reference's factor, np.sqrt(0.5)


def _plugin():
    return custom_ops.get_plugin('sres_dblock_plugin')


class _Native:
    """The kernels behind ``_Block``. Tests substitute a torch stand-in with the same methods (float64 on the CPU) to check
    its gradients of every order."""

    @staticmethod
    def conv0(x, w, b, act, alpha, gain, clamp):
        return conv_nd._get_plugin().fprop(x, w, (1, 1), 1, bias=b, act=2 if act == 'lrelu' else 1, alpha=alpha, gain=gain,
                                           clamp=-1.0 if clamp is None else clamp)

    @staticmethod
    def conv1(x, fx, fy, flip, w, b, act, alpha, gain, clamp):
        return _plugin().conv1(x, fx, fy, flip, w, b, 2 if act == 'lrelu' else 1, alpha, gain, -1.0 if clamp is None else clamp)

    @staticmethod
    def skip(x, w, r, rscale):
        return _plugin().skip(x, w, r, rscale)

    @staticmethod
    def act_grad(dy, y, cfg):
        return conv_nd._BiasActGrad.apply(dy, y, cfg)

    @staticmethod
    def conv_grads(x, dz, w, stride, pad, want_dx, want_dw):
        """(dx, dw) of conv2d(x, w, stride=stride, padding=pad); one call that re-tiles dz once when both are wanted and no
        graph is recorded, else the recorded gradient Functions."""
        if want_dx and want_dw and conv_nd._fused_backward_ok(dz):
            return conv_nd._get_plugin().backward(x, dz, w, (pad, pad), 1, stride=stride)
        dx = conv_nd._ConvNdDgrad.apply(dz, w, x.shape, (pad, pad), 1, stride) if want_dx else None
        dw = conv_nd._ConvNdWgrad.apply(dz, x, w.shape, (pad, pad), 1, stride) if want_dw else None
        return dx, dw

    @staticmethod
    def conv1_backward(h0, fx, fy, flip, dz, w, want_dx, want_dw):
        return _plugin().conv1_backward(h0, fx, fy, flip, dz, w, want_dx, want_dw)

    @staticmethod
    def fir_adjoint_act(dhf, h0, fx, fy, flip, act, alpha, gain, clamp, want_db):
        return _plugin().fir_adjoint_act(dhf, h0, fx, fy, flip, 2 if act == 'lrelu' else 1, alpha, gain, -1.0 if clamp is None else clamp, want_db)


_backend = _Native


def _bias_grad(dz, dtype):
    return (dz.float() if dz.dtype == torch.float16 else dz).sum([0, 2, 3]).to(dtype)


class _Block(torch.autograd.Function):
    """out = (conv2d(xd, w_skip) + h1) * rscale with h0 = bias_act(conv2d(x, w0, padding=1), b0) and h1 =
    bias_act(conv2d(upfirdn2d(h0, f, padding=2), w1, stride=2), b1), f = outer(fy, fx); xd = the skip's down-sampled x.
    Saves x, xd, h0, h1, the weights and b0.

    First-order backward (no graph recorded), natively: conv1's activation gradient with rscale folded into its gain; conv1's
    input gradient and its weight gradient with the filtered image re-tiled from h0 by the FIR pass
    (``lvg_sres_dblock_conv1_backward``); the FIR adjoint fused with conv0's activation gradient and a fixed-order db0
    (``lvg_sres_dblock_fir_adjoint_act``); conv0's gradients; the skip's input gradient with rscale folded into its weight
    and its weight gradient scaled by rscale (tiny tensors: no pass over the block's gradient). With create_graph=True every
    step is a recorded differentiable Function (conv_nd's gradients, _BiasActGrad, upfirdn2d), so gradients of any order
    work."""

    @staticmethod
    def forward(ctx, x, xd, w_skip, w0, b0, w1, b1, f, fx, fy, cfg):
        flip, act, alpha, gain, clamp, rscale = cfg
        h0 = _backend.conv0(x, w0, b0, act, alpha, gain, clamp)
        h1 = _backend.conv1(h0, fx, fy, flip, w1, b1, act, alpha, gain, clamp)
        out = _backend.skip(xd, w_skip, h1, rscale)
        ctx.save_for_backward(x, xd, w_skip, w0, b0, h0, w1, h1, f, fx, fy)
        ctx.cfg = cfg
        ctx.bias_dtypes = (None if b0 is None else b0.dtype, None if b1 is None else b1.dtype)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, xd, w_skip, w0, ctx.b0, h0, w1, h1, f, fx, fy = ctx.saved_tensors
        flip, act, alpha, gain, clamp, s = ctx.cfg
        need = ctx.needs_input_grad
        off = conv_nd._weights_off()
        want_h0 = need[0] or (need[3] and not off) or need[4]
        dx = dxd = dws = dw0 = db0 = dw1 = db1 = None
        if not torch.is_grad_enabled():
            dz1 = _backend.act_grad(dout, h1, (act, alpha, gain * s, clamp))
            if need[6] and ctx.bias_dtypes[1] is not None:
                db1 = _bias_grad(dz1, ctx.bias_dtypes[1])
            if want_h0 or (need[5] and not off):
                dhf, dw1 = _backend.conv1_backward(h0, fx, fy, flip, dz1, w1, want_h0, need[5] and not off)
                if want_h0:
                    dz0, db0 = _backend.fir_adjoint_act(dhf, h0, fx, fy, flip, act, alpha, gain, clamp,
                                                        need[4] and ctx.bias_dtypes[0] is not None)
                    if db0 is not None:
                        db0 = db0.to(ctx.bias_dtypes[0])
                    dx, dw0 = _backend.conv_grads(x, dz0, w0, 1, 1, need[0], need[3] and not off)
            if need[1] or (need[2] and not off):
                dxd, dws = _backend.conv_grads(xd, dout, w_skip * s, 1, 0, need[1], need[2] and not off)
                if dws is not None:
                    dws = dws * s
        else:
            g = dout * s                                  # the gradient of the reference's `* np.sqrt(0.5)`
            dz1 = _backend.act_grad(g, h1, (act, alpha, gain, clamp))
            if need[6] and ctx.bias_dtypes[1] is not None:
                db1 = _bias_grad(dz1, ctx.bias_dtypes[1])
            if want_h0 or (need[5] and not off):
                # h0 recomputed as a recorded function of x, w0 and b0 (the saved h0 is not connected to them)
                h0 = conv_nd.conv_bias_act(x, w0, ctx.b0, padding=1, act=act, alpha=alpha, gain=gain, clamp=clamp)
                hf = upfirdn2d.upfirdn2d(h0, f, padding=2, flip_filter=flip)
                dhf, dw1 = _backend.conv_grads(hf, dz1, w1, 2, 0, want_h0, need[5] and not off)
                if want_h0:
                    # upfirdn2d's adjoint: the mirrored filter, padding fw - 2 - 1 = 1 on every side
                    dz0 = _backend.act_grad(upfirdn2d.upfirdn2d(dhf, f, padding=1, flip_filter=not flip), h0, (act, alpha, gain, clamp))
                    if need[4] and ctx.bias_dtypes[0] is not None:
                        db0 = _bias_grad(dz0, ctx.bias_dtypes[0])
                    dx, dw0 = _backend.conv_grads(x, dz0, w0, 1, 1, need[0], need[3] and not off)
            if need[1] or (need[2] and not off):
                dxd, dws = _backend.conv_grads(xd, g, w_skip, 1, 0, need[1], need[2] and not off)
        return dx, dxd, dws, dw0, db0, dw1, db1, None, None, None, None


# ---------------------------------------------------------------------------------------------------- the block op

def _composition(x, w_skip, w0, b0, w1, b1, f_skip, f1, act, gain, clamp):
    """The reference's op sequence (conv2d_resample + bias_act per layer, then the merge)."""
    y = conv2d_resample.conv2d_resample(x, w_skip, f=f_skip, down=2)
    y = _bias_act.bias_act(y, None, act='linear')
    h = _bias_act.bias_act(conv2d_resample.conv2d_resample(x, w0, padding=1), b0, act=act, gain=gain, clamp=clamp)
    h = _bias_act.bias_act(conv2d_resample.conv2d_resample(h, w1, f=f1, down=2, padding=1), b1, act=act, gain=gain, clamp=clamp)
    return (h + y) * np.sqrt(0.5)


def plan_shapes(n, cin, cout, h, w):
    """Output [N, Cout, H', W'] of every layer of the block as conv2d_resample plans it (stride-2 3x3 after a FIR with
    padding 2; 1x1 after a decimating FIR with padding 1): both branches end at ((H - 2) // 2 + 1, (W - 2) // 2 + 1)."""
    ho, wo = (h + 1 - 3) // 2 + 1, (w + 1 - 3) // 2 + 1
    return dict(filtered=(n, cin, h + 1, w + 1), conv1=(n, cout, ho, wo), skip=(n, cout, (h + 2 - 4) // 2 + 1, (w + 2 - 4) // 2 + 1))


def native(x, w_skip, w0, w1, f_skip, f1, act):
    """The native layers take the block: CUDA fp16 / fp32 NCHW tensors with LVG_NATIVE_CONV on, weights of x's dtype,
    lrelu / linear, 4 x 4 rank-1 filters (conv1's factors known outside CUDA-graph capture), and shapes the size queries
    of both kernels and the engine (conv0) accept."""
    if not (isinstance(x, torch.Tensor) and x.ndim == 4 and x.is_cuda and x.dtype in (torch.float16, torch.float32)
            and x.is_contiguous() and conv_nd.enabled_for(x) and act in ('lrelu', 'linear')):
        return False
    if any(t.dtype != x.dtype or t.device != x.device for t in (w_skip, w0, w1)):
        return False
    if any(t is None or t.ndim != 2 or tuple(t.shape) != (4, 4) or t.device != x.device for t in (f_skip, f1)):
        return False
    n, cin, h, w = x.shape
    cout = w1.shape[0]
    if tuple(w0.shape) != (cin, cin, 3, 3) or tuple(w1.shape) != (cout, cin, 3, 3) or tuple(w_skip.shape) != (cout, cin, 1, 1):
        return False
    p = _plugin()
    _, _, ho, wo = plan_shapes(n, cin, cout, h, w)['conv1']
    if p.conv1_workspace(x.dtype, n, cin, cout, h, w) < 0 or p.skip_workspace(x.dtype, n, cin, cout, ho * wo) < 0:
        return False
    if not custom_ops.ConvNdPlugin._in_envelope(tuple(x.shape), tuple(w0.shape), x.dtype, 1, (1, 1), 1, 1):
        return False
    return _bias_act._init() and upfirdn2d._rank1_factors(f1) is not None


def sres_dblock(x, w_skip, w0, b0, w1, b1, f_skip, f1, *, act='lrelu', gain=None, clamp=None):
    """``(conv1(conv0(x)) + skip(x)) * sqrt(0.5)`` of a resnet ``DiscriminatorBlock``: x [N, C, H, W]; w_skip [Cout, C, 1,
    1], w0 [C, C, 3, 3], w1 [Cout, C, 3, 3] with ``weight_gain`` applied and in x's dtype, b0 / b1 in x's dtype (or None);
    f_skip / f1 the skip's and conv1's ``resample_filter``; act, gain (default: the activation's) and clamp as conv0 and
    conv1 pass them to bias_act. Gradients of any order with respect to x, the weights and the biases. Outside ``native``
    the reference's op sequence runs."""
    gain = float(gain if gain is not None else _bias_act.activation_funcs[act].def_gain)
    if not native(x, w_skip, w0, w1, f_skip, f1, act):
        return _composition(x, w_skip, w0, b0, w1, b1, f_skip, f1, act, gain, clamp)
    alpha = float(_bias_act.activation_funcs[act].def_alpha or 0.0)
    xd = upfirdn2d.upfirdn2d(x, f_skip, down=2, padding=1)
    fx, fy = upfirdn2d._rank1_factors(f1)
    return _Block.apply(x, xd, w_skip, w0, b0, w1, b1, f1, fx, fy, (False, act, alpha, gain, clamp, _SQRT_HALF))


# ---------------------------------------------------------------------------------------------------- install

def block_applies(block, force_fp32=False):
    """The block's structure the op computes: architecture 'resnet' without ``negate_half``, layers without dropout or
    up-sampling, 3x3 conv0 / conv1 and a 1x1 skip, conv1 and the skip down-sampling by 2 with 4 x 4 filters, and not
    channels-last."""
    if getattr(block, 'architecture', None) != 'resnet' or getattr(block, 'negate_half', False):
        return False
    if block.channels_last and not force_fp32:
        return False
    layers = [block.conv0, block.conv1, block.skip] + ([block.fromrgb] if block.in_channels == 0 else [])
    if any(l.dropout_p > 0 or l.up != 1 for l in layers) or block.conv0.down != 1 or block.conv1.down != 2 or block.skip.down != 2:
        return False
    if block.conv0.weight.shape[2:] != (3, 3) or block.conv1.weight.shape[2:] != (3, 3) or block.skip.weight.shape[2:] != (1, 1):
        return False
    return all(tuple(l.resample_filter.shape) == (4, 4) for l in (block.conv1, block.skip))


def applies(block, x, img, force_fp32=False):
    """The installed forward takes the block: ``block_applies`` and a CUDA fp16 / fp32 input with LVG_NATIVE_CONV on.
    Everything else runs the original method."""
    t = x if x is not None else img
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype in (torch.float16, torch.float32) and conv_nd.enabled_for(t)):
        return False
    return block_applies(block, force_fp32)


def _layer_args(layer, dtype):
    w = (layer.weight * layer.weight_gain).to(dtype)
    b = layer.bias.to(dtype) if layer.bias is not None else None
    return w, b


def block_forward(block, x, img, force_fp32=False):
    """DiscriminatorBlock.forward (resnet) with the main layers as ``sres_dblock``: the same casts, fromrgb and order."""
    dtype = torch.float16 if block.use_fp16 and not force_fp32 else torch.float32
    if x is not None:
        x = x.to(dtype=dtype, memory_format=torch.contiguous_format)
    if block.in_channels == 0:
        img = img.to(dtype=dtype, memory_format=torch.contiguous_format)
        y = block.fromrgb(img)
        x = x + y if x is not None else y
        img = None
    c0, c1, sk = block.conv0, block.conv1, block.skip
    w0, b0 = _layer_args(c0, dtype)
    w1, b1 = _layer_args(c1, dtype)
    ws, _ = _layer_args(sk, dtype)
    clamp = c0.conv_clamp
    if c1.conv_clamp != clamp or c0.activation != c1.activation or sk.activation != 'linear' or c0.act_gain != c1.act_gain:
        x = (c1(c0(x)) + sk(x)) * np.sqrt(0.5)
    else:
        x = sres_dblock(x, ws, w0, b0, w1, b1, sk.resample_filter, c1.resample_filter, act=c0.activation, gain=c0.act_gain,
                        clamp=clamp)
    assert x.dtype == dtype
    return x, img


def faster(resolution):
    """Which blocks take the op for speed, from the block's input resolution: b16 and b8. Measured on an H100 (700 W) with
    the default D at batch 8 (DESIGN.md 7i): there the op was faster in the forward without a gradient, forward + backward
    and the R1 pattern. At b32 and above it was slower in the R1 pattern (b32 3.88 -> 4.43 ms) and at b64 and above also in
    forward + backward (b256 3.38 -> 3.83 ms): conv1's input and weight gradients each re-tile dy (the composition's
    shares one re-tiling), and the recorded R1 backward recomputes h0 and the filtered image."""
    return resolution <= 16


def _forward(orig):
    def forward(self, x, img, force_fp32=False):
        if not applies(self, x, img, force_fp32) or not faster(self.resolution):
            return orig(self, x, img, force_fp32)
        return block_forward(self, x, img, force_fp32)
    return forward


def layer_applies(layer, x):
    """``Conv2dLayer.forward`` runs ``conv_nd.conv_bias_act``: no resampling or dropout, lrelu / linear, and a contiguous
    NCHW input whose convolution ``conv_nd.engine_takes`` (``fromrgb`` stays on the pointwise kernels)."""
    if layer.up != 1 or layer.down != 1 or layer.dropout_p > 0 or layer.activation not in ('lrelu', 'linear'):
        return False
    if not (isinstance(x, torch.Tensor) and x.ndim == 4 and x.is_contiguous()):
        return False
    return conv_nd.engine_takes(x, layer.weight.shape, (layer.padding, layer.padding))


def _layer_forward(orig):
    def forward(self, x, gain=1):
        if not layer_applies(self, x):
            return orig(self, x, gain)
        w, b = _layer_args(self, x.dtype)
        clamp = self.conv_clamp * gain if self.conv_clamp is not None else None
        return conv_nd.conv_bias_act(x, w, b, padding=self.padding, act=self.activation, gain=self.act_gain * gain, clamp=clamp)
    return forward


def _roots(module):
    return [m for m in module.modules() if type(m).__name__ == 'VideoDiscriminator'] or [module]


def _has_filter(module):
    return hasattr(module, 'resample_filter')          # the low-res D's DiscriminatorBlock has none


def install(*targets):
    """Patch ``DiscriminatorBlock.forward`` and ``Conv2dLayer.forward`` of an unmodified super-res discriminator.
    ``targets``: the module ``model.discriminator_sres`` or discriminator / block instances, found by
    ``_install.find_classes`` among the modules with a ``resample_filter``, below every ``VideoDiscriminator`` of a target
    that holds one. Idempotent; the originals stay reachable as ``.forward.lvg_sres_dblock``. Returns the patched classes,
    blocks first."""
    blocks = _install.find_classes(targets, 'DiscriminatorBlock', _has_filter, _roots)
    layers = _install.find_classes(targets, 'Conv2dLayer', _has_filter, _roots)
    for cls in blocks:
        _install.wrap(cls, 'forward', 'lvg_sres_dblock', _forward)
    for cls in layers:
        _install.wrap(cls, 'forward', 'lvg_sres_dblock', _layer_forward)
    return blocks + layers
