"""Input of a super-res generator layer as one native op.

Not a module of the reference's ``torch_utils.ops``. Between every pair of layers the super-res generator runs

  Generator.prep_cond             generator_sres.py:581-610   replicate pad, unfold the +-context frames into C (c s)
                                                             channels, per layer a replicate pad + upfirdn2d
                                                             (KaiserDownsample / KaiserUpsample), a crop and a second
                                                             replicate pad; all 15 results stay alive for the pass
  torch.cat((x, cond), 1)         :462-464                   fp16 x with fp32 cond -> an fp32 tensor
  x.to(dtype), magnitude EMA      :307-325                   the cast back to fp16, and with update_emas a square-mean

``cond_concat`` writes the layer's whole input in the layer's dtype in one launch (csrc/sres_cond.cu): x_prev copied with
its cast, the conditioning evaluated from the low-res video by each layer's ``plan`` (below) in fp32 and rounded once, and
optionally the mean square of the fp32 concatenation (what the reference squares) without atomics. The conditioning has no
gradient; the gradient of x_prev is ``dz[:, :C].to(x_prev.dtype)``, bit for bit what the reference's ToCopyBackward +
CatBackward produce, and written with torch ops, so gradients of any order work.

The plan. Along an axis (H or W) of a layer, the reference's conditioning value at output index i is
  m   = x0 + clamp(i - px0, 0, mhi)                                  the crop, then the replicate pad to in_size
  out = gain * sum_k f[K - 1 - k] * u[m * down + k - pad0]           upfirdn2d: u = the frame upsampled by `up` (zeros
                                                                     inserted), zero outside [0, zlen)
  u[j * up] = lr[clamp(j - shift, 0, len - 1)]                       prep_cond's pad and the resampler's pad: one clamp
Identity resamplers are the same plan with one tap of 1 (K = 0 in the plan). ``plan`` derives it from the attributes
``prep_cond`` reads: ``cond_width``, ``cond_height``, ``margin_size``, each resampler's ``scale``, ``filter`` and ``pad``
and each layer's ``in_size``.

``install(...)`` makes an unmodified ``Generator.forward`` of generator_sres use the op (opt-in, idempotent).
"""
import collections

import numpy as np
import torch

from .. import custom_ops
from . import _install

MAX_TAPS = 64                                      # kMaxTaps of csrc/sres_cond.cu

# one axis of a layer's plan: the ints of lvg_sres_cond's plan arrays, the per-axis gain and the low-res extent
AxisPlan = collections.namedtuple('AxisPlan', 'out px0 mhi x0 up down pad0 zlen shift ntaps gain len')
# a layer's plan: the two axes, the 1-D filter (a device buffer of the resampler, None for Identity) and the context window
Plan = collections.namedtuple('Plan', 'h w filter window')


def _plugin():
    return custom_ops.get_plugin('sres_cond_plugin')


def _kind(resample):
    name = type(resample).__name__
    return {'KaiserDownsample': 'down', 'KaiserUpsample': 'up', 'Identity': 'id'}.get(name)


def axis_plan(lr_len, square, margin, kind, scale, ntaps, pad, in_len):
    """One axis: lr_len low-res samples, prep_cond's padded square ``square + 2 margin`` (square = max(cond_width,
    cond_height)), resampler ``kind`` ('down' / 'up' / 'id') with ``scale``, ``ntaps`` filter taps and its ``pad`` flag, and
    the layer's input extent ``in_len``."""
    p0 = (square - lr_len) // 2 + margin
    p1 = (square - lr_len + 1) // 2 + margin
    n_pad = lr_len + p0 + p1                                             # prep_cond's replicate-padded frame
    if kind == 'id':
        up = down = 1
        pad0, k, gain, q = 0, 0, 1.0, 0
        n_in = n_pad
        m_len = n_pad
    elif kind == 'down':
        q = int(pad) * scale                                             # KaiserDownsample's replicate pad
        n_in = n_pad + 2 * q
        up, down, k, gain = 1, scale, ntaps, 1.0
        pad0 = -q + (ntaps - scale + 1) // 2                             # upfirdn2d.downsample2d(padding=-q)
        pad1 = -q + (ntaps - scale) // 2
        m_len = (n_in + pad0 + pad1 - ntaps) // down + 1
    elif kind == 'up':
        q = int(pad)                                                     # KaiserUpsample's replicate pad
        n_in = n_pad + 2 * q
        up, down, k, gain = scale, 1, ntaps, float(scale)                # upsample2d's gain up^2, per axis up
        pad0 = -q * scale + (ntaps + scale - 1) // 2                     # upfirdn2d.upsample2d(padding=-q*scale)
        pad1 = -q * scale + (ntaps - scale) // 2
        m_len = n_in * up + pad0 + pad1 - ntaps + 1
    else:
        raise ValueError(f'unknown resampler kind {kind}')
    x0 = max(0, (m_len - in_len) // 2)                                   # prep_cond's crop ...
    kept = min(x0 + in_len, m_len) - x0
    px0 = (in_len - kept) // 2                                           # ... and replicate pad
    return AxisPlan(out=int(in_len), px0=px0, mhi=kept - 1, x0=x0, up=up, down=down, pad0=pad0, zlen=n_in * up,
                    shift=q + p0, ntaps=k, gain=gain, len=int(lr_len))


def plans(G, lr_h, lr_w):
    """The plan of every layer of generator_sres.Generator ``G`` for a low-res video of lr_h x lr_w (None for a layer whose
    resampler is not KaiserDownsample / KaiserUpsample / Identity)."""
    square = max(G.cond_width, G.cond_height)
    window = 2 * G.cond_context + 1
    out = []
    for name, r in zip(G.synthesis.layer_names, G.resamples):
        kind = _kind(r)
        if kind is None:
            out.append(None)
            continue
        in_w, in_h = (int(v) for v in getattr(G.synthesis, name).in_size)
        f = None if kind == 'id' else r.filter
        if f is not None and f.ndim != 1:
            out.append(None)
            continue
        scale, nt, pad = (1, 0, False) if kind == 'id' else (int(r.scale), int(f.numel()), bool(r.pad))
        out.append(Plan(h=axis_plan(lr_h, square, G.margin_size, kind, scale, nt, pad, in_h),
                        w=axis_plan(lr_w, square, G.margin_size, kind, scale, nt, pad, in_w), filter=f, window=window))
    return out


def _ints(a):
    return [a.out, a.px0, a.mhi, a.x0, a.up, a.down, a.pad0, a.zlen, a.shift, a.ntaps]


def axis_matrix(a, f, dtype=torch.float64):
    """The axis map as a dense [out, len] matrix (float64 by default): the restatement the tests evaluate."""
    m = torch.zeros([a.out, a.len], dtype=dtype)
    taps = [1.0] if a.ntaps == 0 else [float(v) for v in f.detach().cpu().double()]
    k_n = max(a.ntaps, 1)
    for i in range(a.out):
        mm = a.x0 + min(max(i - a.px0, 0), a.mhi)
        for k in range(k_n):
            j = mm * a.down + k - a.pad0
            if j < 0 or j >= a.zlen or j % a.up:
                continue
            src = min(max(j // a.up - a.shift, 0), a.len - 1)
            m[i, src] += a.gain * taps[k_n - 1 - k]
    return m


def evaluate(lr, plan):
    """The layer's conditioning [N T, C (c s), H, W] from lr [N, C, T_lr, h, w] by the plan, in float64 (reference of the
    tests; no kernel)."""
    a_h, a_w = axis_matrix(plan.h, plan.filter), axis_matrix(plan.w, plan.filter)
    x = lr.double().cpu().unfold(2, plan.window, 1)                                  # [N, C, T, h, w, S]
    n, c, t = x.shape[:3]
    y = torch.einsum('yh,ncthws,xw->ntcsyx', a_h, x, a_w)
    return y.reshape(n * t, c * plan.window, plan.h.out, plan.w.out)


def supported(n, t, c, c_lr, t_lr, plan, dtype):
    """The kernel takes the call (size query of lvg_sres_cond)."""
    if plan.h.ntaps > MAX_TAPS or plan.w.ntaps > MAX_TAPS:
        return False
    return _plugin().workspace(n, t, c, c_lr, plan.window, t_lr, plan.h.len, plan.w.len, dtype, _ints(plan.h), _ints(plan.w)) >= 0


class _CondConcat(torch.autograd.Function):
    """z = cat(x_prev, cond).to(dtype) (and the mean square). Saves nothing but the channel count and dtype of x_prev."""

    @staticmethod
    def forward(ctx, x_prev, lr, plan, dtype, want_sumsq):
        f = plan.filter
        z, ms = _plugin().forward(x_prev, lr, f if plan.h.ntaps else None, f if plan.w.ntaps else None, _ints(plan.h),
                                  _ints(plan.w), plan.h.gain, plan.w.gain, plan.window, dtype, want_sumsq)
        ctx.c = 0 if x_prev is None else x_prev.shape[1]
        ctx.x_dtype = None if x_prev is None else x_prev.dtype
        if ms is None:
            return z
        ctx.mark_non_differentiable(ms)
        return z, ms

    @staticmethod
    def backward(ctx, dz, *unused):
        dx = None
        if ctx.needs_input_grad[0]:
            dx = dz[:, :ctx.c].to(ctx.x_dtype).contiguous()
        return dx, None, None, None, None


def cond_concat(x_prev, lr, plan, dtype, want_sumsq):
    """(z, mean_sq | None): z = cat((x_prev, cond), 1).to(dtype) with cond the layer's conditioning of lr by ``plan``
    (x_prev None: z = cond), mean_sq = the mean of the squares of the fp32 concatenation (``want_sumsq``). CUDA only:
    callers check ``applies``."""
    f = plan.filter
    if f is not None and f.device != lr.device:
        raise RuntimeError('sres_cond: the filter must be on the device of lr')
    out = _CondConcat.apply(x_prev, lr, plan, dtype, bool(want_sumsq))
    return (out[0], out[1]) if want_sumsq else (out, None)


# ---------------------------------------------------------------------------------------------------- install

def rejection(G, cond, lr_plans=None):
    """Why the installed forward does not take the call, or None when it does: 'dtype' (the low-res video is not a 5-D fp32
    tensor), 'grad' (it needs a gradient and grad mode is on), 'resampler' (not KaiserDownsample / KaiserUpsample /
    Identity with a 1-D filter), 'taps' (a filter longer than MAX_TAPS), 'shape' (the kernel's size query rejects a layer),
    'cpu' (not a CUDA tensor)."""
    if not (isinstance(cond, torch.Tensor) and cond.dtype == torch.float32 and cond.ndim == 5):
        return 'dtype'
    if cond.requires_grad and torch.is_grad_enabled():
        return 'grad'
    n, c_lr, t_lr, lr_h, lr_w = cond.shape
    lr_plans = plans(G, lr_h, lr_w) if lr_plans is None else lr_plans
    if any(p is None for p in lr_plans):
        return 'resampler'
    if any(p.h.ntaps > MAX_TAPS or p.w.ntaps > MAX_TAPS for p in lr_plans):
        return 'taps'
    t = t_lr - 2 * G.cond_context
    S = G.synthesis
    for i, (name, p) in enumerate(zip(S.layer_names, lr_plans)):
        c = getattr(S, name).in_channels - c_lr * p.window
        if t < 1 or c < 0 or (c == 0) != (i == 0 and not S.fourfeats):
            return 'shape'
        if not all(supported(n, t, c, c_lr, t_lr, p, dt) for dt in (torch.float16, torch.float32)):
            return 'shape'
    if not cond.is_cuda:
        return 'cpu'
    return None


def applies(G, cond, lr_plans=None):
    """The installed forward takes the call: a CUDA fp32 low-res video that needs no gradient, resamplers KaiserDownsample /
    KaiserUpsample / Identity with 1-D filters of at most MAX_TAPS taps, and every layer's shape and plan taken by the
    kernel (size query). See ``rejection``."""
    return rejection(G, cond, lr_plans) is None


def track_magnitude(L, distributed, magnitude_cur):
    """SynthesisLayer.forward's magnitude EMA update from the layer input's mean square ``magnitude_cur``."""
    with torch.autograd.profiler.record_function('update_magnitude_ema'):
        if distributed.get_world_size() > 1:
            torch.distributed.all_reduce(magnitude_cur)
            magnitude_cur = magnitude_cur / distributed.get_world_size()
        L.magnitude_ema.copy_(magnitude_cur.lerp(L.magnitude_ema, L.magnitude_ema_beta))


def layer_styles(L, w):
    """SynthesisLayer.forward's styles (the affine layer, ToRGB's weight gain)."""
    styles = L.affine(w)
    if L.is_torgb:
        weight_gain = 1 / np.sqrt(L.in_channels * (L.conv_kernel ** 2))
        styles = styles * weight_gain
    return styles


def conv_step(L, g, x_prev, lr, plan, w, dtype, update_emas):
    """The step of SynthesisLayer.forward from the layer's input to its modulated convolution's output: the input
    ``cat((x_prev, cond), 1).to(dtype)`` from ``cond_concat`` with the magnitude statistic from the same pass, the
    magnitude EMA, the styles and ``modulated_conv2d`` (whatever the model module's global is patched to)."""
    misc, distributed = g['misc'], g['distributed']
    x, magnitude_cur = cond_concat(x_prev, lr, plan, dtype, update_emas)
    misc.assert_shape(x, [None, L.in_channels, int(L.in_size[1]), int(L.in_size[0])])
    misc.assert_shape(w, [x.shape[0], L.w_dim])

    # Track input magnitude.
    if update_emas:
        track_magnitude(L, distributed, magnitude_cur)
    input_gain = L.magnitude_ema.rsqrt()

    # Execute affine layer.
    styles = layer_styles(L, w)

    # Execute modulated conv2d.
    return g['modulated_conv2d'](x=x, w=L.weight, s=styles, padding=L.conv_kernel - 1, demodulate=(not L.is_torgb),
                                 input_gain=input_gain)


def layer_forward(L, g, x_prev, lr, plan, w, force_fp32=False, update_emas=False, step=conv_step):
    """SynthesisLayer.forward with its input ``cat((x_prev, cond), 1).to(dtype)`` from ``cond_concat`` and the magnitude
    statistic from the same pass. ``g``: the globals of the model module (its ``misc``, ``distributed``,
    ``modulated_conv2d`` and ``filtered_lrelu``, whatever they are patched to). ``step``: the part from the input to the
    modulated convolution's output (``conv_step``; torch_utils/ops/sres_layer.py replaces it by one fused op)."""
    misc = g['misc']
    dtype = torch.float16 if (L.use_fp16 and not force_fp32 and lr.device.type == 'cuda') else torch.float32
    x = step(L, g, x_prev, lr, plan, w, dtype, update_emas)

    # Execute bias, filtered leaky ReLU, and clamping.
    gain = 1 if L.is_torgb else np.sqrt(2)
    slope = 1 if L.is_torgb else 0.2
    x = g['filtered_lrelu'].filtered_lrelu(x=x, fu=L.up_filter, fd=L.down_filter, b=L.bias.to(x.dtype), up=L.up_factor,
                                           down=L.down_factor, padding=L.padding, gain=gain, slope=slope, clamp=L.conv_clamp)

    # Ensure correct shape and dtype.
    misc.assert_shape(x, [None, L.out_channels, int(L.out_size[1]), int(L.out_size[0])])
    assert x.dtype == dtype
    return x


def synthesis_forward(S, g, ws, lr, lr_plans, torgb=None, **layer_kwargs):
    """SynthesisNetwork.forward with each layer's input from ``cond_concat``. ``torgb``: the forward of the ToRGB layer
    (``layer_forward``'s arguments; torch_utils/ops/sres_torgb.py runs it as one op), None for ``layer_forward``."""
    misc = g['misc']
    misc.assert_shape(ws, [None, S.num_ws, S.w_dim])
    ws = ws.to(torch.float32).unbind(dim=1)

    x = S.input(ws[0].size(0)) if S.fourfeats else None
    for name, w, plan in zip(S.layer_names, ws, lr_plans):
        L = getattr(S, name)
        x = (torgb if (torgb is not None and L.is_torgb) else layer_forward)(L, g, x, lr, plan, w, **layer_kwargs)
    if S.output_scale != 1:
        x = x * S.output_scale

    misc.assert_shape(x, [None, S.img_channels, S.img_height, S.img_width])
    x = x.to(torch.float32)
    return x


def generator_forward(G, g, z, cond, truncation_psi=1, truncation_cutoff=None, update_emas=False, lr_plans=None,
                      **synthesis_kwargs):
    """Generator.forward of generator_sres with the conditioning of every layer built inside ``cond_concat`` instead of
    ``prep_cond``. The same mapping call, w_avg update, affine layers and magnitude-EMA updates as the reference."""
    misc, einops = g['misc'], g['einops']
    misc.assert_shape(cond, [z.size(0), G.img_channels, None, G.cond_height, G.cond_width])
    out_seq_length = cond.size(2) - 2 * G.cond_context
    assert out_seq_length > 0
    lr_plans = plans(G, cond.size(3), cond.size(4)) if lr_plans is None else lr_plans
    z = einops.repeat(z, "n c -> (n t) c", t=out_seq_length)
    ws = G.mapping(z, c=None, truncation_psi=truncation_psi, truncation_cutoff=truncation_cutoff, update_emas=update_emas)
    img = synthesis_forward(G.synthesis, g, ws, cond, lr_plans, update_emas=update_emas, **synthesis_kwargs)
    vid = einops.rearrange(img, "(n t) c h w -> n c t h w", t=out_seq_length)
    return vid


def _forward(orig):
    g = _install.reference_function(orig).__globals__
    # sres_layer.install's and sres_torgb.install's wrappers below this one
    fused = [f for f in (_install.find(orig, 'lvg_sres_layer'), _install.find(orig, 'lvg_sres_torgb')) if f is not None]

    def forward(self, z, cond, truncation_psi=1, truncation_cutoff=None, update_emas=False, **synthesis_kwargs):
        if any(f.takes(self, cond, update_emas) for f in fused):
            return orig(self, z, cond, truncation_psi, truncation_cutoff, update_emas, **synthesis_kwargs)
        lr_plans = plans(self, cond.size(3), cond.size(4)) if isinstance(cond, torch.Tensor) and cond.ndim == 5 else None
        if lr_plans is None or not applies(self, cond, lr_plans):
            return orig(self, z, cond, truncation_psi, truncation_cutoff, update_emas, **synthesis_kwargs)
        return generator_forward(self, g, z, cond, truncation_psi, truncation_cutoff, update_emas, lr_plans=lr_plans,
                                 **synthesis_kwargs)
    return forward


def _is_generator(m):
    return all(hasattr(m, a) for a in ('prep_cond', 'synthesis', 'resamples'))


def install(*targets):
    """Make ``Generator.forward`` of generator_sres run ``generator_forward``. ``targets``: the module
    ``model.generator_sres`` or instances holding a ``Generator`` with ``prep_cond``, ``synthesis`` and ``resamples``,
    found by ``_install.find_classes``. Calls outside ``applies`` (CPU tensors, a low-res video that is not fp32 or needs a
    gradient, other resamplers, longer filters, shapes the kernel rejects) run the original method, and so do calls that a
    ``sres_layer.install`` wrapper installed below this one takes. Idempotent; the original stays reachable as
    ``.forward.lvg_sres_cond``. Returns the patched classes."""
    classes = _install.find_classes(targets, 'Generator', _is_generator)
    for cls in classes:
        _install.wrap(cls, 'forward', 'lvg_sres_cond', _forward)
    return classes
