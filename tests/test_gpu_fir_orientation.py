"""The fused FIR kernels with asymmetric taps, so that a reversed tap order, fx and fy exchanged, an ignored flip, an
adjoint that does not mirror its taps or a filter applied along the wrong axis changes the result.

Every GPU test of fir3d (conv3d_down), dblock_tail, sres_dblock's conv1 / FIR adjoint and sres_cond elsewhere uses the
palindrome [1, 3, 3, 1], with which none of those mistakes shows. Here the taps are A = [1, 2, 4, 1] / 8, B = [2, 1, 3, 2] / 8
and, for direct kernel calls, the signed and unnormalised S = [-1, 3, 5, 2] / 8. The references are float64 and built from
the definitions the networks use (upfirdn2d / downsample2d / upsample2d on the CPU, replicate pads, autograd for adjoints),
not from the modules' own restatements; tests/test_fir_orientation_host.py pins those restatements to them and checks that
every case here changes under each of the mistakes above.

Exact tier: sparse small integers, dyadic taps, biases, gains and clamps keep every intermediate exact in fp16 and in the fp32
path's bf16 hi / lo split, so results equal the float64 reference element for element. Random values: whole sres_dblock
blocks, dblock_tail and conv3d_down with A against float64 / the reference composition."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F_

import test_gpu_conv3d_down as tcd
import test_gpu_dblock_tail as tdb
import test_gpu_sres_dblock as tsd
from torch_utils.ops import bias_act, conv3d_down as cd, dblock_tail as dt, sres_cond as sc, sres_dblock as sd, upfirdn2d

pytestmark = pytest.mark.gpu
DEV = 'cuda'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
DT = {'f32': torch.float32, 'f16': torch.float16}

A = (1 / 8, 2 / 8, 4 / 8, 1 / 8)
B = (2 / 8, 1 / 8, 3 / 8, 2 / 8)
S = (-1 / 8, 3 / 8, 5 / 8, 2 / 8)
TAP_IDS = {A: 'A', B: 'B', S: 'S'}
ints, check_repr = tcd.ints, tcd.check_repr


def taps(t):
    return torch.tensor(t, dtype=torch.float32)


def check_exact(t, dtype, what):
    """Precondition of an exact comparison where products with alpha or a gain leave the 2^-9 grid: t is exactly
    representable in fp32 and in the storage type."""
    assert torch.equal(t.float().double(), t) and torch.equal(t.to(dtype).double(), t), f'{what}: not exact in {dtype}'


def differs(a, b):
    """A mutated reference differs from the reference; None stands for a mutation not defined on the case's inputs."""
    return a is None or b is None or a.shape != b.shape or not torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------- float64 references

def fir_axis(x, f, d, step, off, n_out):
    """Along dim d: out[m] = sum_k f[k] x[step m + off + 3 - k], zero outside x -- upfirdn2d (convolution order,
    flip_filter=False) with padding -off before and step ``down``."""
    x = x.movedim(d, -1)
    lead, n_in = x.shape[:-1], x.shape[-1]
    p0 = -off
    p1 = (n_out - 1) * step + 4 - n_in - p0
    y = upfirdn2d.upfirdn2d(x.reshape(-1, 1, 1, n_in), taps(f)[None, :], down=[step, 1], padding=[p0, p1, 0, 0])
    return y.reshape(*lead, n_out).movedim(-1, d)


def fir3d_ref(x, f, axes, fold):
    """fir3d's P: per T, H, W (filt, step, off, n_in, n_out); ``fold`` stores t = 2 t' + p as channel p C + c."""
    for d, (filt, step, off, n_in, n_out) in zip((2, 3, 4), axes):
        assert x.shape[d] == n_in
        if filt:
            x = fir_axis(x, f, d, step, off, n_out)
    if fold:
        x = torch.cat([x[:, :, p::2] for p in (0, 1)], 1)
    return x


def fir3d_adjoint_ref(y, f, axes, fold):
    """P^T y: the autograd of fir3d_ref."""
    x0 = torch.zeros((y.shape[0], y.shape[1] // (2 if fold else 1)) + tuple(a[3] for a in axes), dtype=torch.float64,
                     requires_grad=True)
    with torch.enable_grad():
        return torch.autograd.grad(fir3d_ref(x0, f, axes, fold), [x0], y)[0]


def downsample3d_ref(y, f, spatial_down, temporal_down):
    """Downsample3d (discriminator_lres.py) as the reference writes it: downsample2d over H, W of (c t) h w, then over T of
    t (h w) with the [4, 1] filter."""
    n, c, t, h, w = y.shape
    f = taps(f)
    if spatial_down:
        y = upfirdn2d.downsample2d(y.reshape(n, c * t, h, w), f, down=2)
        h, w = y.shape[2:]
        y = y.reshape(n, c, t, h, w)
    if temporal_down:
        y = upfirdn2d.downsample2d(y.reshape(n, c, t, h * w), f[:, None], down=[1, 2])
        y = y.reshape(n, c, y.shape[2], h, w)
    return y


def down_axes_ref(y, f, down):
    """Downsample3d's filter with step 2 on the axes of ``down`` (per T, H, W), any subset: the mutations of the axis tests."""
    for d, dn in zip((2, 3, 4), down):
        if dn:
            y = fir_axis(y, f, d, 2, -1, y.shape[d] // 2)
    return y


def halvable(shape, down):
    """Downsample3d's filter with step 2 is defined on the axes of ``down``: even extents."""
    return all(not dn or (n >= 2 and n % 2 == 0) for dn, n in zip(down, shape[2:]))


def transpose_ref(fwd, x_shape, dy):
    """The adjoint of the linear map ``fwd`` at dy (autograd, float64)."""
    x0 = torch.zeros(x_shape, dtype=torch.float64, requires_grad=True)
    with torch.enable_grad():
        return torch.autograd.grad(fwd(x0), [x0], dy)[0]


def conv1_fir_ref(x, fx, fy, flip):
    """conv1's filtered image: upfirdn2d(x, outer(fy, fx), padding=2, flip_filter=flip)."""
    return upfirdn2d.upfirdn2d(x, torch.outer(taps(fy), taps(fx)), padding=2, flip_filter=bool(flip))


def _replicate(v, a, b):
    lead, n = v.shape[:-1], v.shape[-1]
    return F_.pad(v.reshape(-1, 1, n), (a, b), mode='replicate').reshape(*lead, n + a + b)


def cond_axis_ref(v, f, kind, scale, pad, square, margin, in_len):
    """One axis (the last) of Generator.prep_cond: the replicate pad to the square plus margins, KaiserDownsample /
    KaiserUpsample (replicate pad, then downsample2d / upsample2d with the filter along this axis and padding -p), the
    centre crop to the layer's in_size and the replicate pad up to it."""
    n = v.shape[-1]
    v = _replicate(v, (square - n) // 2 + margin, (square - n + 1) // 2 + margin)
    lead = v.shape[:-1]
    q = int(pad) * (scale if kind == 'down' else 1)
    v = _replicate(v, q, q).reshape(-1, 1, 1, v.shape[-1] + 2 * q)
    f2 = taps(f)[None, :]
    if kind == 'down':
        v = upfirdn2d.downsample2d(v, f2, down=[scale, 1], padding=[-q, -q, 0, 0])
    else:
        v = upfirdn2d.upsample2d(v, f2, up=[scale, 1], padding=[-q * scale, -q * scale, 0, 0])
    v = v.reshape(*lead, v.shape[-1])
    x0 = max(0, (v.shape[-1] - in_len) // 2)
    v = v[..., x0:x0 + in_len]
    return _replicate(v, (in_len - v.shape[-1]) // 2, (in_len - v.shape[-1] + 1) // 2)


# ---------------------------------------------------------------------------------------------------- fir3d

# (name, axes per T, H, W: (filt, step, off, n_in, n_out), fold): every axis alone and in combination, steps 1 and 2,
# negative, zero and positive offsets, fold on and off, non-square planes and more than one 8 x 32 tile
FIR3D_CASES = [
    ('t_down', ((1, 2, -1, 8, 4), (0, 1, 0, 5, 5), (0, 1, 0, 7, 7)), False),
    ('h_down', ((0, 1, 0, 3, 3), (1, 2, -1, 18, 9), (0, 1, 0, 9, 9)), False),
    ('w_down', ((0, 1, 0, 3, 3), (0, 1, 0, 6, 6), (1, 2, -1, 70, 35)), False),
    ('h_full_w_full', ((0, 1, 0, 2, 2), (1, 1, -2, 9, 11), (1, 1, -1, 33, 34)), False),
    ('hw_offsets', ((0, 1, 0, 2, 2), (1, 1, -1, 12, 12), (1, 1, -3, 12, 12)), False),
    ('t_full_h_down', ((1, 1, -2, 7, 9), (1, 2, -1, 20, 10), (0, 1, 0, 5, 5)), False),
    ('thw_down', ((1, 2, -1, 6, 3), (1, 2, -1, 64, 32), (1, 2, -1, 66, 33)), False),
    ('thw_down_ext', ((1, 2, 0, 6, 2), (1, 2, 0, 10, 4), (1, 2, 1, 12, 5)), False),
    ('full_fold', ((1, 1, -3, 6, 10), (1, 1, -2, 34, 36), (1, 1, -2, 70, 72)), True),
    ('t_fold', ((1, 1, -1, 5, 6), (0, 1, 0, 4, 4), (0, 1, 0, 40, 40)), True),
]
FIR3D_TAPS = [A, S]


def fir3d_case(case):
    """(x, y) of a case: P's input and a cotangent laid out as P's output."""
    name, axes, fold = case
    x = ints((2, 3) + tuple(a[3] for a in axes), 11, vmax=2, density=0.5)
    out = (2, 3 * (2 if fold else 1), axes[0][4] // (2 if fold else 1), axes[1][4], axes[2][4])
    return x, ints(out, 12, vmax=2, density=0.5)


def fir3d_refs(case, f, axes=None):
    name, axes0, fold = case
    axes = axes0 if axes is None else axes
    x, y = fir3d_case(case)
    return fir3d_ref(x, f, axes, fold), fir3d_adjoint_ref(y, f, axes, fold)


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('f', FIR3D_TAPS, ids=lambda f: TAP_IDS[f])
@pytest.mark.parametrize('case', FIR3D_CASES, ids=[c[0] for c in FIR3D_CASES])
def test_fir3d_exact(case, f, dt):
    dtype = DT[dt]
    name, axes, fold = case
    x, y = fir3d_case(case)
    want, want_t = fir3d_refs(case, f)
    check_repr(want, dtype, name)
    check_repr(want_t, dtype, name + ' adjoint')
    plug = cd.custom_ops.get_plugin('fir3d_plugin')
    got = plug.fir3d(x.to(DEV, dtype), taps(f).to(DEV), axes, fold)
    got_t = plug.fir3d(y.to(DEV, dtype), taps(f).to(DEV), axes, fold, adjoint=True)
    assert torch.equal(got.cpu().double(), want), f'{name}: {int((got.cpu().double() != want).sum())} of {want.numel()} differ'
    assert torch.equal(got_t.cpu().double(), want_t), f'{name} adjoint: {int((got_t.cpu().double() != want_t).sum())} differ'
    # <P x, y> = <x, P^T y> on the device results
    assert float((got.double() * y.to(DEV)).sum()) == float((x.to(DEV) * got_t.double()).sum())


# ---------------------------------------------------------------------------------------------------- dblock_tail

P = tdb.P
DB_FLAGS = [P.SDOWN, P.TDOWN, P.TDOWN | P.SDOWN]
DB_OUTS = [(1, 7, 1), (2, 9, 33), (3, 4, 40)]
DB_ALPHA, DB_GAIN, DB_CLAMP = 0.25, 2.0, 2.0
DB_B = (0.5, -0.25, 0.0)


def dblock_case(flags, out):
    """(y, s, u, sig, dz) of a case: the convolution output, the skip, a read-mode input and skip, and a cotangent."""
    to, ho, wo = out
    t, h, w = to * (2 if flags & P.TDOWN else 1), ho * (2 if flags & P.SDOWN else 1), wo * (2 if flags & P.SDOWN else 1)
    n, c = 2, 3
    return (ints((n, c, t, h, w), 21, vmax=3, density=0.3), ints((n, c, to, ho, wo), 22, vmax=3, density=0.6),
            ints((n, c, t, h, w), 23, vmax=3, density=0.3), ints((n, c, to, ho, wo), 24, vmax=3, density=0.3),
            ints((n, c, to, ho, wo), 25, vmax=2, density=0.5))


def dblock_refs(flags, out, f, down=None):
    """(o, G, lin, dy) in float64 without the merge: o = clamp(lrelu(P y + b) gain), G its slopes (0 where clamped), lin
    = G (P u + b), dy = P^T (G dz). ``down``: the filtered axes (T, H, W), by default those of ``flags``."""
    y, _, u, _, dz = dblock_case(flags, out)
    down = (bool(flags & P.TDOWN), bool(flags & P.SDOWN), bool(flags & P.SDOWN)) if down is None else down
    if not halvable(y.shape, down):
        return None, None, None, None
    if down[1] == down[2]:
        fwd = lambda v: downsample3d_ref(v, f, down[1], down[0])      # noqa: E731
    else:
        fwd = lambda v: down_axes_ref(v, f, down)                     # noqa: E731
    b = torch.tensor(DB_B, dtype=torch.float64).view(1, -1, 1, 1, 1)
    x = fwd(y) + b
    o = torch.where(x > 0, x, x * DB_ALPHA) * DB_GAIN
    G = torch.where(o.abs() < DB_CLAMP, torch.where(x > 0, DB_GAIN, DB_ALPHA * DB_GAIN), 0.0)
    lin = G * (fwd(u) + b)
    dy = transpose_ref(fwd, y.shape, G * dz) if G.shape == dz.shape else None     # None: not defined on this case's dz
    return o.clamp(-DB_CLAMP, DB_CLAMP), G, lin, dy


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('out', DB_OUTS, ids=[f'{a}x{b}x{c}' for a, b, c in DB_OUTS])
@pytest.mark.parametrize('flags', DB_FLAGS)
def test_dblock_tail_exact(flags, out, dt):
    """Write mode (with and without the merge), the codes, read mode and the adjoint (dy and db exact without the merge; ds
    with it) with the taps A: element for element the float64 references."""
    dtype = DT[dt]
    y, s, u, sig, dz = dblock_case(flags, out)
    o, G, lin, dy64 = dblock_refs(flags, out, A)
    f = taps(A).to(DEV)
    b = torch.tensor(DB_B, device=DEV)
    t, h, w = y.shape[2:]
    for what, v in (('o', o), ('lin', lin), ('dy', dy64)):
        check_exact(v, dtype, what)
    plug = tdb.plug()
    want_code = (~(o > 0)).long() | ((~(G != 0)).long() << 1)
    z, codes = plug.forward(y.to(DEV, dtype), None, b, f, flags, 3, DB_ALPHA, DB_GAIN, DB_CLAMP, P.WRITE)
    assert torch.equal(z.cpu().double(), o) and torch.equal(tdb.decode(codes, z.shape).cpu(), want_code)
    zm, codes_m = plug.forward(y.to(DEV, dtype), s.to(DEV, dtype), b, f, flags | P.MERGE, 3, DB_ALPHA, DB_GAIN, DB_CLAMP, P.WRITE)
    assert torch.equal(zm.cpu(), ((o + s) * tdb.SQH).float().to(dtype)) and torch.equal(codes_m, codes)
    zr, _ = plug.forward(u.to(DEV, dtype), None, b, f, flags, 3, DB_ALPHA, DB_GAIN, -1.0, P.READ, codes)
    assert torch.equal(zr.cpu().double(), lin)
    zrm, _ = plug.forward(u.to(DEV, dtype), sig.to(DEV, dtype), b, f, flags | P.MERGE, 3, DB_ALPHA, DB_GAIN, -1.0, P.READ, codes)
    assert torch.equal(zrm.cpu(), ((lin + sig) * tdb.SQH).float().to(dtype))
    dy, ds, db = plug.adjoint(dz.to(DEV, dtype), codes, f, (t, h, w), flags, 3, DB_ALPHA, DB_GAIN, False)
    assert ds is None and torch.equal(dy.cpu().double(), dy64)
    assert torch.equal(db.cpu().double(), (G * dz).sum((0, 2, 3, 4)))


@pytest.mark.parametrize('flags', DB_FLAGS)
def test_dblock_tail_adjoint_is_the_transpose_with_asymmetric_taps(flags):
    """The adjoint's matrix against the read-mode forward's, with A (the transpose of the unmirrored operator differs)."""
    t, h, w = 4, 6, 10
    to, ho, wo = P.out_size((t, h, w), flags)
    k_in, k_out = t * h * w, to * ho * wo
    f = taps(A).to(DEV)
    yv = torch.randn(1, 1, t, h, w, generator=torch.Generator(device=DEV).manual_seed(7), device=DEV) * 2
    plug = tdb.plug()
    _, codes1 = plug.forward(yv, None, None, f, flags | P.MERGE, 3, 0.2, 2.0, 1.0, P.WRITE)
    fwd, _ = plug.forward(torch.eye(k_in, device=DEV).view(k_in, 1, t, h, w), None, None, f, flags | P.MERGE, 3, 0.2, 2.0, -1.0,
                          P.READ, codes1.repeat(k_in))
    a = fwd.reshape(k_in, k_out).t()
    adj, _, _ = plug.adjoint(torch.eye(k_out, device=DEV).view(k_out, 1, to, ho, wo), codes1.repeat(k_out), f, (t, h, w),
                             flags | P.MERGE, 3, 0.2, 2.0, True)
    assert torch.allclose(adj.reshape(k_out, k_in), a, atol=1e-7, rtol=0) and float(a.abs().max()) > 0.05
    G = tdb.slope64(tdb.decode(codes1, (to, ho, wo)), 0.2, 2.0).flatten().cpu()
    sd_, td_ = bool(flags & P.SDOWN), bool(flags & P.TDOWN)
    a64 = downsample3d_ref(torch.eye(k_in, dtype=torch.float64).view(k_in, 1, t, h, w), A, sd_, td_).reshape(k_in, k_out).t()
    assert torch.allclose(a.cpu().double(), a64 * G.view(-1, 1) * tdb.SQH, atol=1e-6, rtol=0)


# ---------------------------------------------------------------------------------------------------- conv3d_down

C3_LAYERS = [l for l in tcd.LAYERS if l[0].endswith('_skip')]


def c3_case(layer):
    name, cin, cout, kt, ks, t, h, w, sd_, td_ = layer
    x = ints((1, cin, t, h, w), 31)
    wt = ints((cout, cin, kt, ks, ks), 32, density=min(0.15, 3 / (cin * kt * ks * ks)))
    b = ints((cout,), 33, vmax=2, density=0.5)
    return x, wt, b


def c3_refs(layer, f, down=None, dtype=torch.float32):
    """(z, dx, dw, db) of Downsample3d(conv3d(x, w)) + b in float64; ``down`` overrides the filtered axes (T, H, W)."""
    name, cin, cout, kt, ks, t, h, w, sd_, td_ = layer
    x, wt, b = c3_case(layer)
    down = (td_, sd_, sd_) if down is None else down
    if not halvable(x.shape, down):
        return None, None, None, None
    xg, wg, bg = (v.clone().requires_grad_(True) for v in (x, wt, b))
    with torch.enable_grad():
        y = F_.conv3d(xg, wg, padding=(kt // 2, ks // 2, ks // 2))
        z = (downsample3d_ref(y, f, down[1], down[0]) if down[1] == down[2] else down_axes_ref(y, f, down)) + bg.view(1, -1, 1, 1, 1)
        dz = ints(z.shape, 34, density=0.1 if dtype == torch.float32 else 0.001)
        return (z.detach(),) + torch.autograd.grad(z, [xg, wg, bg], dz)


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('layer', C3_LAYERS, ids=[l[0] for l in C3_LAYERS])
def test_conv3d_down_exact(layer, dt):
    """conv3d_down's decomposition (fir3d, then the convolution at the output resolution) with A: forward, dx, dw and db
    element for element against the float64 reference composition."""
    dtype = DT[dt]
    name, cin, cout, kt, ks, t, h, w, sd_, td_ = layer
    x, wt, b = c3_case(layer)
    refs = c3_refs(layer, A, dtype=dtype)
    xg, wg, bg = (v.to(DEV, dtype).requires_grad_(True) for v in (x, wt, b))
    f = taps(A).to(DEV)
    assert cd.in_envelope(xg, wg, (kt // 2, ks // 2, ks // 2), sd_, td_, f)
    z = bias_act.bias_act(cd._decomposed(xg, wg, f, sd_, td_), bg)
    dz = ints(z.shape, 34, density=0.1 if dtype == torch.float32 else 0.001).to(DEV, dtype)
    got = (z,) + torch.autograd.grad(z, [xg, wg, bg], dz)
    for what, ref, g in zip(('z', 'dx', 'dw', 'db'), refs, got):
        check_repr(ref, dtype, f'{name} {what}')
        g = g.detach().cpu().double()
        assert torch.equal(g, ref), f'{name} {dt} {what}: {int((g != ref).sum())} of {ref.numel()} differ'


# ---------------------------------------------------------------------------------------------------- sres_dblock

SD_SHAPES = [(2, 20, 24, 18, 22), (1, 64, 128, 33, 40), (3, 8, 40, 10, 260), (1, 136, 72, 9, 9)]
SD_PAIRS = [(A, B), (B, A), (S, B)]                     # (fx, fy)
SD_IDS = [f'fx{TAP_IDS[p[0]]}_fy{TAP_IDS[p[1]]}' for p in SD_PAIRS]


def sd_case(shape, dtype):
    """(x, w, b, dz, dhf, h0) of a case; dz is sparse enough that the fp16 weight gradient is exact."""
    n, cin, cout, h, w = shape
    ho, wo = (h - 2) // 2 + 1, (w - 2) // 2 + 1
    dens = (3 if dtype == torch.float16 else 12) / (n * ho * wo)
    return (ints((n, cin, h, w), 41, vmax=2, density=0.5), tsd.ints((cout, cin, 3, 3), -3, 3, 42), tsd.ints((cout,), -8, 8, 43) / 4,
            ints((n, cout, ho, wo), 44, vmax=2, density=min(1.0, dens)), tsd.ints((n, cin, h + 1, w + 1), -4, 4, 45),
            tsd.ints((n, cin, h, w), -3, 3, 46) / 2)


def sd_refs(shape, dtype, fx, fy, flip, clamp=1.5):
    """(conv1 output, filtered image, dw, dz0) in float64: conv1 = bias_act(conv2d(hf, w, stride=2), b) with the engine's fp32
    epilogue roundings, dw = conv1's weight gradient from the float64 filtered image, dz0 = conv0's activation gradient of
    the FIR adjoint of dhf (the autograd of conv1_fir_ref) with the fp32 constants."""
    x, wt, b, dz, dhf, h0 = sd_case(shape, dtype)
    hf = conv1_fir_ref(x, fx, fy, flip)
    y = tsd.act_f32(F_.conv2d(hf, wt, stride=2), b, 256.0).double()
    dw = torch.nn.grad.conv2d_weight(hf, wt.shape, dz, stride=2)
    t = transpose_ref(lambda v: conv1_fir_ref(v, fx, fy, flip), h0.shape, dhf).numpy().astype(np.float32)
    hv = h0.numpy()
    o = np.where(hv > 0, t, (t * tsd.ALPHA).astype(np.float32))
    o = (o * tsd.GAIN).astype(np.float32)
    o = np.where((hv > -clamp) & (hv < clamp), o, np.float32(0))
    return y, hf, dw, torch.from_numpy(o).double()


def _sd_taps(fx, fy):
    return taps(fx).to(DEV), taps(fy).to(DEV)


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('flip', [0, 1])
@pytest.mark.parametrize('fxy', SD_PAIRS, ids=SD_IDS)
@pytest.mark.parametrize('shape', SD_SHAPES, ids=['x'.join(map(str, s)) for s in SD_SHAPES])
def test_sres_conv1_exact(shape, fxy, flip, dt):
    """lvg_sres_dblock_conv1 (the FIR in conv_pack_fir4_kernel) bit for bit: ragged channel blocks, odd extents, a 260-pixel
    row."""
    dtype = DT[dt]
    x, wt, b, *_ = sd_case(shape, dtype)
    y, hf, _, _ = sd_refs(shape, dtype, *fxy, flip)
    check_repr(hf, dtype, 'filtered image')
    got = sd._Native.conv1(x.to(DEV, dtype), *_sd_taps(*fxy), flip, wt.to(DEV, dtype), b.to(DEV, dtype), 'lrelu', 0.2,
                           float(tsd.GAIN), 256.0)
    want = y.float().to(dtype)
    assert torch.equal(got.cpu(), want), f'{int((got.cpu() != want).sum())} of {want.numel()} differ'


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('flip', [0, 1])
@pytest.mark.parametrize('fxy', SD_PAIRS, ids=SD_IDS)
@pytest.mark.parametrize('shape', SD_SHAPES, ids=['x'.join(map(str, s)) for s in SD_SHAPES])
def test_sres_conv1_backward_dw_exact(shape, fxy, flip, dt):
    """conv1's weight gradient from the image conv_pack_fir4_kernel re-tiles from h0 equals the weight gradient of the float64
    filtered image."""
    dtype = DT[dt]
    x, wt, _, dz, _, _ = sd_case(shape, dtype)
    _, _, dw64, _ = sd_refs(shape, dtype, *fxy, flip)
    check_repr(dw64, dtype, 'dw')
    _, dw = sd._Native.conv1_backward(x.to(DEV, dtype), *_sd_taps(*fxy), flip, dz.to(DEV, dtype), wt.to(DEV, dtype), False, True)
    assert torch.equal(dw.cpu().double(), dw64), f'{int((dw.cpu().double() != dw64).sum())} of {dw64.numel()} differ'


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('flip', [0, 1])
@pytest.mark.parametrize('fxy', SD_PAIRS, ids=SD_IDS)
@pytest.mark.parametrize('shape', SD_SHAPES, ids=['x'.join(map(str, s)) for s in SD_SHAPES])
def test_sres_fir_adjoint_act_exact(shape, fxy, flip, dt):
    """lvg_sres_dblock_fir_adjoint_act: G(h0) (.) FIR^T(dhf) bit for bit, and db0 within fp32 summation of its float64 sum."""
    dtype = DT[dt]
    _, _, _, _, dhf, h0 = sd_case(shape, dtype)
    _, _, _, dz64 = sd_refs(shape, dtype, *fxy, flip)
    dz, db = sd._Native.fir_adjoint_act(dhf.to(DEV, dtype), h0.to(DEV, dtype), *_sd_taps(*fxy), flip, 'lrelu', 0.2, float(tsd.GAIN),
                                        1.5, True)
    want = dz64.float().to(dtype)
    assert torch.equal(dz.cpu(), want), f'{int((dz.cpu() != want).sum())} of {want.numel()} differ'
    db64 = want.double().sum([0, 2, 3])
    assert float((db.cpu().double() - db64).abs().max()) <= 1e-5 * max(float(db64.abs().max()), 1.0)


# ---------------------------------------------------------------------------------------------------- sres_cond

LR = (2, 3, 4, 9, 16)                # N, C_lr, T_lr, h, w of the low-res video
SQUARE, MARGIN, WINDOW = 16, 2, 3
# (kind, scale, pad, in_h, in_w): an up layer whose output is cropped along H and replicate-padded along W, and a down layer
COND_LAYERS = [('up', 2, True, 36, 44), ('down', 2, True, 8, 12)]
COND_PAIRS = [(A, B), (S, A)]        # (f_h, f_w)


def cond_plan(layer, f_h, f_w):
    kind, scale, pad, in_h, in_w = layer
    ah = sc.axis_plan(LR[3], SQUARE, MARGIN, kind, scale, 4, pad, in_h)
    aw = sc.axis_plan(LR[4], SQUARE, MARGIN, kind, scale, 4, pad, in_w)
    return ah, aw


def cond_lr():
    return ints(LR, 51, vmax=3, density=0.5)


def cond_ref(layer, f_h, f_w):
    """The layer's conditioning [N T, C_lr window, in_h, in_w] from the low-res video in float64: the window unfolded into
    channels (c s), then prep_cond along W with f_w and along H with f_h."""
    kind, scale, pad, in_h, in_w = layer
    v = cond_lr().unfold(2, WINDOW, 1)                                         # [N, C, T, h, w, S]
    n, c, t, h, w, s = v.shape
    v = v.permute(0, 2, 1, 5, 3, 4).reshape(n * t, c * s, h, w)
    v = cond_axis_ref(v, f_w, kind, scale, pad, SQUARE, MARGIN, in_w)
    v = cond_axis_ref(v.transpose(2, 3), f_h, kind, scale, pad, SQUARE, MARGIN, in_h).transpose(2, 3)
    return v.contiguous()


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('fhw', COND_PAIRS, ids=[f'fh{TAP_IDS[p[0]]}_fw{TAP_IDS[p[1]]}' for p in COND_PAIRS])
@pytest.mark.parametrize('layer', COND_LAYERS, ids=[l[0] for l in COND_LAYERS])
def test_sres_cond_exact(layer, fhw, dt):
    """lvg_sres_cond with different asymmetric filters on H and W: the conditioning bit for bit."""
    dtype = DT[dt]
    f_h, f_w = fhw
    ah, aw = cond_plan(layer, f_h, f_w)
    want = cond_ref(layer, f_h, f_w)
    check_repr(want, dtype, 'conditioning')
    z, _ = sc._plugin().forward(None, cond_lr().float().to(DEV), taps(f_h).to(DEV), taps(f_w).to(DEV), sc._ints(ah), sc._ints(aw),
                                ah.gain, aw.gain, WINDOW, dtype, False)
    assert tuple(z.shape) == tuple(want.shape)
    assert torch.equal(z.cpu().double(), want), f'{int((z.cpu().double() != want).sum())} of {want.numel()} differ'


# ---------------------------------------------------------------------------------------------------- random values

@pytest.mark.parametrize('r1', [False, True], ids=['grad', 'r1'])
@pytest.mark.parametrize('cin,cout,res,dtype', [(512, 512, 32, torch.float16), (512, 512, 16, torch.float32)], ids=['b32_f16', 'b16_f32'])
def test_sres_dblock_block_with_asymmetric_filter(cin, cout, res, dtype, r1):
    """One block per dtype with f1 = f_skip = setup_filter([1, 2, 4, 1]) (rank 1, split exactly): the native first-order
    backward (the FIR adjoint's mirrored taps included) and the R1 pattern within test_gpu_sres_dblock's budget against
    float64."""
    f = upfirdn2d.setup_filter([1, 2, 4, 1]).to(DEV)
    n = 8
    x = torch.randn(n, cin, res, res, generator=torch.Generator().manual_seed(res)).to(DEV) * 0.5
    p = tsd.block_params(cin, cout, dtype, res)
    assert sd.native(x.to(dtype), p['w_skip'], p['w0'], p['w1'], f, f, 'lrelu')
    ours = tsd.run_block(sd.sres_dblock, x.to(dtype), p, r1, f=f)
    comp = tsd.run_block(lambda *a, **k: sd._composition(*a[:8], 'lrelu', k['gain'], k['clamp']), x.to(dtype), p, r1, f=f)
    ref = tsd.run_block(tsd.comp64, x.double(), {k: v.double() for k, v in p.items()}, r1, f=f)
    extra = 1e-5 if dtype == torch.float32 else 2e-3
    for k in ref:
        scale = float(ref[k].abs().max())
        e_ours = float((ours[k] - ref[k]).abs().max()) / scale
        e_comp = float((comp[k] - ref[k]).abs().max()) / scale
        assert e_ours <= 1.5 * e_comp + extra, f'{k}: {e_ours:.3e} vs composition {e_comp:.3e}'


def test_dblock_tail_random_values_with_asymmetric_filter():
    """dblock_tail with A against dt._reference (the reference's op sequence) in fp32: output, first-order gradients and the
    gradients of the R1 pattern."""
    flags = P.TDOWN | P.SDOWN
    y, s, b = tdb._inputs(2, 6, 8, 12, 20, flags, torch.float32, seed=5)
    f = taps(A).to(DEV)
    outs = []
    for native in (True, False):
        yi, si, bi = (v.clone().requires_grad_(True) for v in (y, s, b))
        if native:
            z = dt.dblock_tail(yi, si, bi, f, spatial_down=True, temporal_down=True)
        else:
            z = dt._reference(yi, si, bi, f, True, True, 'lrelu', 256.0)
        dz = torch.randn(z.shape, generator=torch.Generator(device=DEV).manual_seed(6), device=DEV)
        g1 = torch.autograd.grad(z, [yi, si, bi], dz, retain_graph=True)
        gy, gs = torch.autograd.grad(z.square().sum(), [yi, si], create_graph=True)
        gg = torch.autograd.grad(gy.square().sum() + gs.square().sum() + z.sum(), [yi, si, bi])
        outs.append((z.detach(),) + g1 + (gy.detach(), gs.detach()) + gg)
    for a, bb in zip(*outs):
        assert tdb._rel(a, bb) <= 1e-5


@pytest.mark.parametrize('dt', ['f32', 'f16'])
def test_conv3d_down_random_values_with_asymmetric_filter(dt):
    """conv3d_down with A on b1's skip layer: the error of output and gradients against float64 at most 1.5x that of the
    reference composition (conv_nd.conv3d, Downsample3d, bias_act)."""
    dtype = DT[dt]
    name, cin, cout, kt, ks, t, h, w, sd_, td_ = next(l for l in tcd.LAYERS if l[0] == 'b1_skip')
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, cin, t, h, w, generator=g, dtype=torch.float64)
    wt = torch.randn(cout, cin, kt, ks, ks, generator=g, dtype=torch.float64) / cin ** 0.5
    b = torch.randn(cout, generator=g, dtype=torch.float64)
    pad = (0, 0, 0)
    outs = {}
    for path in ('ref64', 'composition', 'op'):
        d, ty = ('cpu', torch.float64) if path == 'ref64' else (DEV, dtype)
        f = taps(A).to(d)
        xg, wg, bg = (v.to(d, ty).requires_grad_(True) for v in (x, wt, b))
        if path == 'op':
            assert cd.faster(wg.shape) and cd.in_envelope(xg, wg, pad, sd_, td_, f)
            z = cd.conv3d_down(xg, wg, bg, pad, sd_, td_, f, act='lrelu', clamp=256)
        else:
            z = bias_act.bias_act(cd._reference(xg, wg, f, sd_, td_, pad), bg, act='lrelu', clamp=256)
        dz = torch.randn(z.shape, generator=torch.Generator().manual_seed(10), dtype=torch.float64).to(d, ty)
        outs[path] = [z] + list(torch.autograd.grad(z, [xg, wg, bg], dz))
    for i, what in enumerate(('z', 'dx', 'dw', 'db')):
        ref = outs['ref64'][i].detach()
        e_op, e_comp = tcd._err(outs['op'][i].detach().cpu(), ref), tcd._err(outs['composition'][i].detach().cpu(), ref)
        slack = 1e-7 if dtype == torch.float32 else 1e-4
        assert e_op <= 1.5 * e_comp + slack, f'{what}: op {e_op:.3e}, composition {e_comp:.3e}'


# ---------------------------------------------------------------------------------------------------- whole networks

def _run_dblock(mode, tmp_path):
    if not os.path.isdir(os.path.join(SRC, 'model')):
        pytest.skip('oracle/_ref not staged')
    out = str(tmp_path / f'{mode}.pt')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.join(ROOT, 'long-video-gan_b200'), SRC]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'dblock_tail_run.py'), out, mode], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out, weights_only=False)


def test_low_res_discriminator_with_asymmetric_filter(tmp_path):
    """The unmodified fp32 VideoDiscriminator with every Downsample3d filter [1, 2, 4, 1] / 8: with conv3d_down and
    dblock_tail (tail=True) installed against without, within test_gpu_dblock_tail's fp32 tolerances; fir3d and the tail
    kernels ran."""
    r = _run_dblock('orient', tmp_path)
    assert r['filters'] > 0
    for key, (tol_max, tol_l2) in tdb.TAIL_TOL.items():
        a, b = r['ours'][key], r['ref'][key]
        assert a.shape == b.shape and torch.isfinite(a).all() and float(b.abs().max()) > 0
        emax, el2 = float((a - b).abs().max() / b.abs().max()), float((a - b).norm() / b.norm())
        assert emax <= tol_max and el2 <= tol_l2, f'{key}: max {emax:.3e}, L2 {el2:.3e}'
    for k in ('fir3d_down_kernel', 'fir3d_adjoint_kernel', 'dblock_tail_fwd_kernel', 'dblock_tail_adj_kernel'):
        assert any(k in n for n in r['kernels']), (k, r['kernels'])


def test_super_res_discriminator_with_asymmetric_filter(tmp_path):
    """The unmodified all-fp32 super-res VideoDiscriminator with every resample_filter setup_filter([1, 2, 4, 1]): installed
    against not, logits, parameter and input gradients and the R1 pattern within 1e-3 of each tensor's largest magnitude
    (test_gpu_sres_dblock's fp32 tolerance); every routed block took the native layers and their FIR kernels ran."""
    r = tsd._helper('orient', tmp_path)
    assert r['filters'] > 0 and r['took'] and all(r['took']), r['took']
    for ours, ref in zip(r['ours'], r['ref']):
        assert ours.keys() == ref.keys()
        for k in ref:
            tsd._close(ours[k], ref[k], k, 1e-3)
    for k in ('conv_pack_fir4_kernel', 'sres_fir_adjoint_act_kernel'):
        assert any(k in n for n in r['kernels']), (k, r['kernels'])
