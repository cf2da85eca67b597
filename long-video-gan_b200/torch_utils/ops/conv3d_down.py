"""Downsampling Conv3dLayers of the low-res discriminator computed at the output resolution.

Not a module of the reference's ``torch_utils.ops``. ``Conv3dLayer.forward`` (discriminator_lres.py:169-179) computes

  z = bias_act(Downsample3d(F.conv3d(x, w, padding=k // 2)), b, act, clamp)

where Downsample3d filters the full-resolution output with f = [1,3,3,1]/8 (padding 1, step 2) on H and W and/or T and
keeps 1/4 or 1/8 of it. Convolution and FIR commute, so ``conv3d_down`` filters the Cin-channel input instead and runs
the convolution only at the kept positions. Per axis of size S, kernel k, p = k // 2:

  not down          the convolution's own padding p, stride 1
  down, k = 1       x filtered with step 2 (FIR|down), then the convolution: exact
  down, k > 1       u = x filtered at full rate over S + 2p positions (positions -p-1 .. S+p-2 of the zero-padded x),
                    then the convolution with padding 0 and step 2 (H, W), or over the two temporal phases of u folded
                    into 2 Cin channels (T: a kt-tap stride-2 convolution is a (p+1)-tap stride-1 one, the engine keeps T
                    stride 1). That gives v = FIR|down(y_ext), y_ext the convolution continued one sample beyond the extent.

  z = v - FIR|down(ring), ring = y_ext on the one-sample shell outside the extent. The shell splits into faces: along
  ring axis a at position -1 (resp. S) with earlier ring axes inside the extent and later ones over the extended range.
  y_ext on a face needs only the first (last) min(p, S) input samples and as many kernel taps along a: a thin convolution. Its filtered
  value touches only the first (last) output sample along a, with the filter's first (last) tap.

All pieces are differentiable of any order (the FIR pair below are each other's backward; conv_nd's Functions; in-place
slice updates; bias_act), as the R1 penalty needs. ``install(...)`` makes an unmodified discriminator use it.
"""
import torch

from . import bias_act, conv_nd, upfirdn2d
from .. import custom_ops

# ---------------------------------------------------------------------------------------------------- FIR pair


def _fir_reference(x, f, axes, fold):
    """P x in torch ops (differentiable; CPU tensors and tests). axes: per T, H, W (filt, step, off, n_in, n_out)."""
    g = f.flip(0).to(x.dtype)
    for d, (filt, step, off, n_in, n_out) in zip((2, 3, 4), axes):
        if not filt:
            continue
        lo = max(0, -off)
        hi = max(0, step * (n_out - 1) + off + 4 - n_in)
        pad = [0] * (2 * (4 - d)) + [lo, hi]
        xp = torch.nn.functional.pad(x, pad)
        idx = [slice(None)] * 5
        acc = 0
        for j in range(4):
            s = off + lo + j
            idx[d] = slice(s, s + step * (n_out - 1) + 1, step)
            acc = acc + g[j] * xp[tuple(idx)]
        x = acc
    if fold:
        n, c, t, h, w = x.shape
        x = x.reshape(n, c, t // 2, 2, h, w).permute(0, 3, 1, 2, 4, 5).reshape(n, 2 * c, t // 2, h, w)
    return x


def _fir_adjoint_reference(y, f, axes, fold):
    """P^T y in torch ops: the gather the adjoint kernel runs (input index base(m) + r, tap per output m)."""
    g = f.flip(0).to(y.dtype)
    if fold:
        n, c2, t2, h, w = y.shape
        y = y.reshape(n, 2, c2 // 2, t2, h, w).permute(0, 2, 3, 1, 4, 5).reshape(n, c2 // 2, 2 * t2, h, w)
    for d, (filt, step, off, n_in, n_out) in zip((2, 3, 4), axes):
        if not filt:
            continue
        out = []
        for m in range(n_in):
            if step == 1:
                terms = [(m - off - 3 + r, g[3 - r]) for r in range(4)]
            else:
                q, odd = (m - off) >> 1, (m - off) & 1
                terms = [(q - 1, g[3] if odd else g[2]), (q, g[1] if odd else g[0])]
            acc = torch.zeros_like(y.select(d, 0))
            for i, tap in terms:
                if 0 <= i < n_out:
                    acc = acc + tap * y.select(d, i)
            out.append(acc)
        y = torch.stack(out, d)
    return y


def _fir_apply(x, f, axes, fold, adjoint):
    if x.is_cuda:
        return custom_ops.get_plugin('fir3d_plugin').fir3d(x, f, axes, fold, adjoint)
    return (_fir_adjoint_reference if adjoint else _fir_reference)(x, f, axes, fold)


class _Fir3d(torch.autograd.Function):
    """y = P x (lvg_fir3d); backward P^T (lvg_fir3d_adjoint), whose backward is P again."""

    @staticmethod
    def forward(ctx, x, f, axes, fold):
        ctx.save_for_backward(f)
        ctx.cfg = (axes, fold)
        return _fir_apply(x, f, axes, fold, False)

    @staticmethod
    def backward(ctx, dy):
        f, = ctx.saved_tensors
        return (_Fir3dAdjoint.apply(dy, f, *ctx.cfg) if ctx.needs_input_grad[0] else None), None, None, None


class _Fir3dAdjoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dy, f, axes, fold):
        ctx.save_for_backward(f)
        ctx.cfg = (axes, fold)
        return _fir_apply(dy, f, axes, fold, True)

    @staticmethod
    def backward(ctx, ddx):
        f, = ctx.saved_tensors
        return (_Fir3d.apply(ddx, f, *ctx.cfg) if ctx.needs_input_grad[0] else None), None, None, None


def fir3d(x, f, axes, fold=False):
    """P x for axes ((filt, step, off, n_in, n_out) per T, H, W) and 4 taps f (upfirdn2d's convolution order)."""
    return _Fir3d.apply(x, f, tuple(tuple(int(v) for v in a) for a in axes), bool(fold))


# ---------------------------------------------------------------------------------------------------- decomposition

_COPY = lambda s: (0, 1, 0, s, s)                  # noqa: E731
_DOWN = lambda s: (1, 2, -1, s, s // 2)            # FIR|down over [0, S): Downsample3d's padding 1, step 2
_DOWN_EXT = lambda s: (1, 2, 0, s + 2, s // 2)     # FIR|down over the extended positions -1 .. S


def _plan(x_shape, w_shape, spatial_down, temporal_down):
    """Per axis T, H, W: (down, k, p, ring)."""
    down = (bool(temporal_down), bool(spatial_down), bool(spatial_down))
    return [(dn, k, k // 2, dn and k > 1) for dn, k in zip(down, w_shape[2:])]


def _calls(x_shape, w_shape, spatial_down, temporal_down):
    """The FIR and convolution calls of the decomposition: (main, faces). main = (fir axes, fold, folded weight shape, conv
    padding, conv stride); faces = [(axis, side, x slice, w slice, conv padding, fir axes)]."""
    plan = _plan(x_shape, w_shape, spatial_down, temporal_down)
    sizes = x_shape[2:]
    fir, pad = [], []
    for (dn, k, p, ring), s in zip(plan, sizes):
        if not dn:
            fir.append(_COPY(s)), pad.append(p)
        elif k == 1:
            fir.append(_DOWN(s)), pad.append(0)
        else:
            fir.append((1, 1, -p - 1, s, s + 2 * p)), pad.append(0)
    fold = plan[0][3]
    cout, cin = w_shape[:2]
    wf_shape = (cout, 2 * cin, plan[0][2] + 1) + tuple(w_shape[3:]) if fold else tuple(w_shape)
    stride = 2 if plan[1][3] else 1
    main = (tuple(fir), fold, wf_shape, tuple(pad), stride)
    faces = []
    rings = [a for a in range(3) if plan[a][3]]
    for a in rings:
        p_a, k_a, s_a = plan[a][2], plan[a][1], sizes[a]
        for side in (0, 1):
            m = min(p_a, s_a)                                  # input samples within reach of the face
            xs = slice(0, m) if side == 0 else slice(s_a - m, s_a)
            ws = slice(p_a + 1, p_a + 1 + m) if side == 0 else slice(p_a - m, p_a)
            cpad, faxes = [], []
            for b in range(3):
                dn, k, p, ring = plan[b]
                if b == a:
                    cpad.append(0), faxes.append(_COPY(1))
                elif ring and b < a:
                    cpad.append(p), faxes.append(_DOWN(sizes[b]))
                elif ring:
                    cpad.append(p + 1), faxes.append(_DOWN_EXT(sizes[b]))
                elif dn:
                    cpad.append(0), faxes.append(_DOWN(sizes[b]))
                else:
                    cpad.append(p), faxes.append(_COPY(sizes[b]))
            faces.append((a, side, xs, ws, tuple(cpad), tuple(faxes)))
    return main, faces


def _fold_weight(w):
    """[Cout, Cin, kt, kh, kw] -> [Cout, 2 Cin, kt // 2 + 1, kh, kw]: phase 0 takes the even taps, phase 1 the odd ones and a
    trailing zero tap."""
    odd = torch.nn.functional.pad(w[:, :, 1::2], (0, 0, 0, 0, 0, 1))
    return torch.cat([w[:, :, 0::2], odd], dim=1)


def _decomposed(x, w, f, spatial_down, temporal_down):
    """Downsample3d(conv3d(x, w, padding=k // 2)) by the decomposition above (no bias / activation)."""
    (fir, fold, _, pad, stride), faces = _calls(tuple(x.shape), tuple(w.shape), spatial_down, temporal_down)
    u = fir3d(x, f, fir, fold)
    z = conv_nd.conv3d(u, _fold_weight(w) if fold else w, padding=pad, stride=(1, stride, stride))
    for a, side, xs, ws, cpad, faxes in faces:
        d = 2 + a
        idx_x = [slice(None)] * 5
        idx_w = [slice(None)] * 5
        idx_x[d], idx_w[d] = xs, ws
        face = conv_nd.conv3d(x[tuple(idx_x)], w[tuple(idx_w)].contiguous(), padding=cpad)
        corr = fir3d(face, f, faxes)
        tap = f[3] if side == 0 else f[0]              # convolution order: position -1 meets g[0] = f[3], position S g[3] = f[0]
        z.narrow(d, 0 if side == 0 else z.shape[d] - 1, 1).sub_(corr * tap.to(corr.dtype))
    return z


def _reference(x, w, f, spatial_down, temporal_down, padding):
    """Downsample3d(conv_nd.conv3d(x, w)) as the reference composes it (discriminator_lres.py:172-175, 197-213)."""
    y = conv_nd.conv3d(x, w, padding=padding)
    n, c, t, h, wd = y.shape
    if spatial_down:
        y = upfirdn2d.downsample2d(y.reshape(n, c * t, h, wd), f, down=2).reshape(n, c, t, h // 2, wd // 2)
        h, wd = h // 2, wd // 2
    if temporal_down:
        y = upfirdn2d.downsample2d(y.reshape(n, c, t, h * wd), f[:, None], down=[1, 2]).reshape(n, c, t // 2, h, wd)
    return y


def in_envelope(x, w, padding, spatial_down, temporal_down, f):
    """conv3d_down takes the decomposition: CUDA fp16 / fp32, a 4-tap f on the same device, LVG_NATIVE_CONV not 0, and
    ``shapes_ok``."""
    return (conv_nd.enabled_for(x) and f.device == x.device and w.dtype == x.dtype and f.ndim == 1
            and shapes_ok(tuple(x.shape), tuple(w.shape), x.dtype, padding, spatial_down, temporal_down, f.numel()))


def shapes_ok(x_shape, w_shape, dtype, padding, spatial_down, temporal_down, taps=4):
    """Odd kernels with padding k // 2, even extents on the down axes, a 4-tap filter, and every convolution of the
    decomposition inside the engine's envelope."""
    if not (spatial_down or temporal_down) or dtype not in (torch.float16, torch.float32) or taps != 4:
        return False
    if len(x_shape) != 5 or len(w_shape) != 5:
        return False
    k = tuple(w_shape[2:])
    if any(kk % 2 == 0 for kk in k) or tuple(int(p) for p in padding) != tuple(kk // 2 for kk in k):
        return False
    if spatial_down and (k[1] > 1) != (k[2] > 1):
        return False
    down = (temporal_down, spatial_down, spatial_down)
    if any(dn and (s % 2 or s < 2) for dn, s in zip(down, x_shape[2:])):
        return False
    (fir, fold, wf_shape, pad, stride), faces = _calls(x_shape, w_shape, spatial_down, temporal_down)
    u_shape = (x_shape[0], x_shape[1] * (2 if fold else 1), fir[0][4] // (2 if fold else 1), fir[1][4], fir[2][4])
    env = custom_ops.ConvNdPlugin._in_envelope
    if not env(u_shape, wf_shape, dtype, (1, stride, stride), pad, 1, 1):
        return False
    for a, side, xs, ws, cpad, faxes in faces:
        xsh, wsh = list(x_shape), list(w_shape)
        xsh[2 + a], wsh[2 + a] = xs.stop - xs.start, ws.stop - ws.start
        if not env(tuple(xsh), tuple(wsh), dtype, 1, cpad, 1, 1):
            return False
    tiles = lambda h, wd: -(-h // 8) * -(-wd // 32)        # noqa: E731  (lvg_fir3d's grid)
    return tiles(fir[1][4], fir[2][4]) <= 65535 and tiles(x_shape[3], x_shape[4]) <= 65535


def faster(w_shape):
    """Which shapes take the decomposition. 1x1x1 kernels (the skip layers): filtering Cin channels before the convolution
    instead of 2 Cin after it is 1.1-3.1x faster in every direction. Larger kernels: the strided main convolution plus up
    to six thin face convolutions and their filters measured 1.5-2.7x slower than the full-resolution convolution
    (DESIGN.md 7c, H100), so they keep the reference composition."""
    return all(k == 1 for k in w_shape[2:])


def conv3d_down(x, w, b, padding, spatial_down, temporal_down, f, act='linear', clamp=None):
    """``bias_act(Downsample3d(spatial_down, temporal_down)(F.conv3d(x, w, padding=padding)), b, act=act, clamp=clamp)``,
    with Downsample3d's filter ``f`` (4 taps, sum 1). x [N, Cin, T, H, W], w [Cout, Cin, kt, kh, kw] of x's dtype, b [Cout]
    or None. Gradients of any order. Outside ``in_envelope`` or ``faster`` the reference composition over conv_nd."""
    if faster(w.shape) and in_envelope(x, w, padding, spatial_down, temporal_down, f):
        y = _decomposed(x, w, f, spatial_down, temporal_down)
    else:
        y = _reference(x, w, f, spatial_down, temporal_down, padding)
    return bias_act.bias_act(y, b, act=act, clamp=clamp)


# ---------------------------------------------------------------------------------------------------- install

def _conv3d_layer_forward(orig):
    def forward(self, input):
        if not (self.spatial_down or self.temporal_down):
            return orig(self, input)
        weight = (self.weight * self.weight_gain).type(input.dtype)
        bias = self._bias.type(input.dtype) if self.bias else None
        return conv3d_down(input, weight, bias, self.padding, self.spatial_down, self.temporal_down,
                           self.downsample._downsample_filter, act=self.activation, clamp=self.conv_clamp)
    forward.lvg_conv3d_down = orig
    return forward


_WRAPPERS = ('lvg_conv3d_down', 'lvg_conv_bias_act')      # attributes under which an install keeps the method it replaced


def wrapped_by(forward, attr):
    """``forward`` or a method below it in the chain of installed wrappers carries ``attr``. conv3d_down.install (layers with
    downsampling) and dblock_tail.install (layers without) both replace Conv3dLayer.forward, each calling the method it
    replaced for the other's layers, in either order."""
    while forward is not None:
        if hasattr(forward, attr):
            return True
        forward = next((getattr(forward, a) for a in _WRAPPERS if hasattr(forward, a)), None)
    return False


def _patch(cls):
    if not wrapped_by(cls.forward, 'lvg_conv3d_down'):
        cls.forward = _conv3d_layer_forward(cls.forward)


def install(*targets):
    """Make the downsampling ``Conv3dLayer``s of reference discriminators run ``conv3d_down``.

    ``targets``: modules (``model.discriminator_lres``, whose ``Conv3dLayer`` class is patched) or ``nn.Module`` instances
    (the class of every submodule named ``Conv3dLayer`` is patched, which reaches unpickled discriminators whose class
    source ``persistence`` executed into a module of its own). The new ``forward`` reads the attributes the reference's
    does; layers without ``spatial_down`` / ``temporal_down`` run the original method. Idempotent. Returns the classes
    that run it."""
    classes = []
    for t in targets:
        if isinstance(t, torch.nn.Module):
            classes += [type(m) for m in t.modules() if type(m).__name__ == 'Conv3dLayer']
        elif getattr(t, 'Conv3dLayer', None) is not None:
            classes.append(t.Conv3dLayer)
    done = []
    for cls in classes:
        if not any(cls is c for c in done):
            _patch(cls)
            done.append(cls)
    return done
