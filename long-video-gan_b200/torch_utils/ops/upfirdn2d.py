"""Pad / up-sample / FIR-filter / down-sample of 2-D images (``torch_utils.ops.upfirdn2d``).

Same public functions and argument conventions as the reference module
(torch_utils/ops/upfirdn2d.py: setup_filter :70, upfirdn2d :118, filter2d :277,
upsample2d :313, downsample2d :352, helpers :35-66). CUDA tensors run in
``liblvg_ops.so`` (csrc/upfirdn2d*.cu); a separable filter is applied in ONE
kernel launch (the reference issues two, with the intermediate in HBM,
upfirdn2d.py:244-245).
"""
import math

import numpy as np
import torch

from .. import custom_ops
from . import conv2d_gradfix

_plugin = None


def _init():
    global _plugin
    if _plugin is None:
        _plugin = custom_ops.get_plugin('upfirdn2d_plugin')
    return True


def _parse_scaling(scaling):
    if isinstance(scaling, int):
        scaling = [scaling, scaling]
    assert isinstance(scaling, (list, tuple))
    assert all(isinstance(v, int) for v in scaling)
    sx, sy = scaling
    assert sx >= 1 and sy >= 1
    return sx, sy


def _parse_padding(padding):
    if isinstance(padding, int):
        padding = [padding, padding]
    assert isinstance(padding, (list, tuple))
    assert all(isinstance(v, int) for v in padding)
    if len(padding) == 2:
        px, py = padding
        padding = [px, px, py, py]
    px0, px1, py0, py1 = padding
    return px0, px1, py0, py1


def _get_filter_size(f):
    if f is None:
        return 1, 1
    assert isinstance(f, torch.Tensor) and f.ndim in [1, 2]
    fw, fh = int(f.shape[-1]), int(f.shape[0])
    assert fw >= 1 and fh >= 1
    return fw, fh


def setup_filter(f, device=torch.device('cpu'), normalize=True, flip_filter=False, gain=1, separable=None):
    """Build the float32 FIR tensor the ops expect: ``[taps]`` (separable) or ``[fh, fw]``.

    f: tensor / array / list, rank 0-2, or None (identity). 1-D inputs with >= 8 taps stay
    separable unless `separable` says otherwise; shorter ones become their outer product.
    """
    if f is None:
        f = 1
    f = torch.as_tensor(f, dtype=torch.float32)
    assert f.ndim in [0, 1, 2]
    assert f.numel() > 0
    if f.ndim == 0:
        f = f[np.newaxis]
    if separable is None:
        separable = (f.ndim == 1 and f.numel() >= 8)
    if f.ndim == 1 and not separable:
        f = f.ger(f)
    assert f.ndim == (1 if separable else 2)
    if normalize:
        f = f / f.sum()
    if flip_filter:
        f = f.flip(list(range(f.ndim)))
    f = f * (gain ** (f.ndim / 2))
    return f.to(device=device)


def upfirdn2d(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """x: ``[N, C, H, W]`` float16/32/64. f: float32 ``[fh, fw]``, ``[taps]`` (separable) or None.

    Per channel: insert ``up-1`` zeros after each pixel, pad (negative = crop), convolve with f
    (``flip_filter=True`` = correlate), keep every ``down``-th pixel, scale by gain.
    up / down: int or ``[x, y]``; padding: int, ``[x, y]`` or ``[x0, x1, y0, y1]``.
    """
    assert isinstance(x, torch.Tensor)
    assert impl in ['ref', 'cuda']
    if impl == 'cuda' and x.device.type == 'cuda' and _init():
        return _upfirdn2d_cuda(up=up, down=down, padding=padding, flip_filter=flip_filter, gain=gain).apply(x, f)
    return _upfirdn2d_ref(x, f, up=up, down=down, padding=padding, flip_filter=flip_filter, gain=gain)


def _upfirdn2d_ref(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1):
    """Composition of standard torch ops (CPU tensors, ``impl='ref'``)."""
    assert isinstance(x, torch.Tensor) and x.ndim == 4
    if f is None:
        f = torch.ones([1, 1], dtype=torch.float32, device=x.device)
    assert isinstance(f, torch.Tensor) and f.ndim in [1, 2]
    assert f.dtype == torch.float32 and not f.requires_grad
    n, c, ih, iw = x.shape
    upx, upy = _parse_scaling(up)
    downx, downy = _parse_scaling(down)
    px0, px1, py0, py1 = _parse_padding(padding)
    assert iw * upx + px0 + px1 >= f.shape[-1] and ih * upy + py0 + py1 >= f.shape[0]

    # zero-insertion: each pixel becomes the top-left corner of an upy x upx cell
    x = x.reshape([n, c, ih, 1, iw, 1])
    x = torch.nn.functional.pad(x, [0, upx - 1, 0, 0, 0, upy - 1])
    x = x.reshape([n, c, ih * upy, iw * upx])
    # positive padding pads, negative padding crops
    x = torch.nn.functional.pad(x, [max(px0, 0), max(px1, 0), max(py0, 0), max(py1, 0)])
    x = x[:, :, max(-py0, 0): x.shape[2] - max(-py1, 0), max(-px0, 0): x.shape[3] - max(-px1, 0)]

    f = f * (gain ** (f.ndim / 2))
    f = f.to(x.dtype)
    if not flip_filter:
        f = f.flip(list(range(f.ndim)))
    f = f[np.newaxis, np.newaxis].repeat([c, 1] + [1] * f.ndim)
    if f.ndim == 4:
        x = conv2d_gradfix.conv2d(input=x, weight=f, groups=c)
    else:
        x = conv2d_gradfix.conv2d(input=x, weight=f.unsqueeze(2), groups=c)
        x = conv2d_gradfix.conv2d(input=x, weight=f.unsqueeze(3), groups=c)
    return x[:, :, ::downy, ::downx]


class _Config:
    """One (up, down, padding, flip, gain) flavour; ``.apply(x, f)`` runs it."""
    __slots__ = ('upx', 'upy', 'downx', 'downy', 'px0', 'px1', 'py0', 'py1', 'flip', 'gain')

    def __init__(self, up, down, padding, flip_filter, gain):
        self.upx, self.upy = _parse_scaling(up)
        self.downx, self.downy = _parse_scaling(down)
        self.px0, self.px1, self.py0, self.py1 = _parse_padding(padding)
        self.flip, self.gain = bool(flip_filter), gain

    def key(self):
        return tuple(getattr(self, k) for k in self.__slots__)

    def apply(self, x, f):
        return _Upfirdn2d.apply(x, f, self)

    def run(self, x, f):
        """Launch for a rank-2 (full) or rank-1 (separable) filter."""
        c = self
        sep = getattr(_plugin, 'upfirdn2d_sep', None)
        if f.ndim == 2:
            # `setup_filter([1,3,3,1])` (< 8 taps) hands the networks the OUTER PRODUCT as a full 4x4 filter
            # (upfirdn2d.py:103-108; every conv2d_resample of the super-res discriminator): rank 1, so the two 1-D passes
            # of the single-launch separable kernels apply
            fac = _rank1_factors(f) if (sep is not None and min(f.shape) > 1) else None
            if fac is not None:
                y = sep(x, fac[0], fac[1], c.upx, c.upy, c.downx, c.downy, c.px0, c.px1, c.py0, c.py1, c.flip, c.gain)
                if y is not None:
                    return y
            return _plugin.upfirdn2d(x, f, c.upx, c.upy, c.downx, c.downy, c.px0, c.px1, c.py0, c.py1, c.flip, c.gain)
        if sep is not None:
            y = sep(x, f, f, c.upx, c.upy, c.downx, c.downy, c.px0, c.px1, c.py0, c.py1, c.flip, c.gain)
            if y is not None:
                return y
        y = _plugin.upfirdn2d(x, f.unsqueeze(0), c.upx, 1, c.downx, 1, c.px0, c.px1, 0, 0, c.flip, 1.0)
        return _plugin.upfirdn2d(y, f.unsqueeze(1), 1, c.upy, 1, c.downy, 0, 0, c.py0, c.py1, c.flip, c.gain)


_rank1_cache = dict()     # (device, data_ptr, shape, stride, version) -> (storage kept alive, (fx, fy) or None)


def _rank1_factors(f):
    """(fx, fy) with f == outer(fy, fx) for a full 2-D filter of rank 1, else None. Decided ONCE per filter tensor on the
    host (one small device->host copy; the entry keeps the filter's storage alive so its address cannot be recycled, an
    in-place update changes `_version`), never during CUDA-graph capture."""
    key = (f.device, f.data_ptr(), tuple(f.shape), tuple(f.stride()), f._version)
    hit = _rank1_cache.get(key)
    if hit is not None:
        return hit[1]
    if f.is_cuda and torch.cuda.is_current_stream_capturing():
        return None
    a = f.detach().to('cpu', torch.float64)
    i, j = divmod(int(a.abs().argmax()), a.shape[1])
    fac = None
    if float(a[i, j]) != 0.0:
        # Balanced split first: both factors scaled by sqrt|a[i, j]|, the sign on fx. For the filters of setup_filter
        # (outer(k, k) / sum^2, dyadic) it gives float32 factors whose products ARE the filter's taps, so the two 1-D
        # passes compute the 2-D operator exactly. The unbalanced split a[:, j] x a[i, :] / a[i, j] does not always
        # (setup_filter([1,3,3,1]): fx = [1/3, 1, 1, 1/3] misses the taps by 1e-9); it is the fallback.
        s = abs(float(a[i, j])) ** 0.5
        fy, fx = (a[:, j] / s).float(), (a[i, :] * (math.copysign(1.0, float(a[i, j])) / s)).float()
        if not torch.equal(torch.outer(fy.double(), fx.double()), a):
            fy, fx = a[:, j].clone(), a[i, :] / a[i, j]
            if float((torch.outer(fy, fx) - a).abs().max()) > 1e-6 * float(a.abs().max()):
                fy = fx = None
        if fx is not None:
            fac = (fx.to(torch.float32).to(f.device).contiguous(), fy.to(torch.float32).to(f.device).contiguous())
    if len(_rank1_cache) >= 64:
        _rank1_cache.pop(next(iter(_rank1_cache)))
    _rank1_cache[key] = (f.untyped_storage(), fac)
    return fac


_upfirdn2d_cuda_cache = dict()


def _upfirdn2d_cuda(up=1, down=1, padding=0, flip_filter=False, gain=1):
    cfg = _Config(up, down, padding, flip_filter, gain)
    return _upfirdn2d_cuda_cache.setdefault(cfg.key(), cfg)


class _Upfirdn2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, f, cfg):
        assert isinstance(x, torch.Tensor) and x.ndim == 4
        if f is None:
            f = torch.ones([1, 1], dtype=torch.float32, device=x.device)
        if f.ndim == 1 and f.shape[0] == 1:
            f = f.square().unsqueeze(0)  # a separable 1-tap filter is the full 1x1 filter f*f
        assert isinstance(f, torch.Tensor) and f.ndim in [1, 2]
        y = cfg.run(x, f)
        ctx.save_for_backward(f)
        ctx.cfg = cfg
        ctx.x_shape = x.shape
        return y

    @staticmethod
    def backward(ctx, dy):
        f, = ctx.saved_tensors
        cfg = ctx.cfg
        _, _, ih, iw = ctx.x_shape
        _, _, oh, ow = dy.shape
        fw, fh = _get_filter_size(f)
        dx = None
        if ctx.needs_input_grad[0]:
            # the adjoint is the same operator with up <-> down, the filter mirrored, and this padding
            p = [fw - cfg.px0 - 1,
                 iw * cfg.upx - ow * cfg.downx + cfg.px0 - cfg.upx + 1,
                 fh - cfg.py0 - 1,
                 ih * cfg.upy - oh * cfg.downy + cfg.py0 - cfg.upy + 1]
            adj = _upfirdn2d_cuda(up=[cfg.downx, cfg.downy], down=[cfg.upx, cfg.upy], padding=p,
                                  flip_filter=(not cfg.flip), gain=cfg.gain)
            dx = adj.apply(dy, f)
        assert not ctx.needs_input_grad[1]
        return dx, None, None


def filter2d(x, f, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """FIR-filter keeping the image size (extra `padding` on top; negative crops)."""
    px0, px1, py0, py1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [px0 + fw // 2, px1 + (fw - 1) // 2, py0 + fh // 2, py1 + (fh - 1) // 2]
    return upfirdn2d(x, f, padding=p, flip_filter=flip_filter, gain=gain, impl=impl)


def upsample2d(x, f, up=2, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """Up-sample by `up` (int or ``[x, y]``): output size is ``in * up`` (+ padding)."""
    upx, upy = _parse_scaling(up)
    px0, px1, py0, py1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [px0 + (fw + upx - 1) // 2, px1 + (fw - upx) // 2, py0 + (fh + upy - 1) // 2, py1 + (fh - upy) // 2]
    return upfirdn2d(x, f, up=up, padding=p, flip_filter=flip_filter, gain=gain * upx * upy, impl=impl)


def downsample2d(x, f, down=2, padding=0, flip_filter=False, gain=1, impl='cuda'):
    """Down-sample by `down` (int or ``[x, y]``): output size is ``in / down`` (+ padding)."""
    downx, downy = _parse_scaling(down)
    px0, px1, py0, py1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [px0 + (fw - downx + 1) // 2, px1 + (fw - downx) // 2, py0 + (fh - downy + 1) // 2, py1 + (fh - downy) // 2]
    return upfirdn2d(x, f, down=down, padding=p, flip_filter=flip_filter, gain=gain, impl=impl)
