"""Bit-exact checks of the resampling and activation kernels: upfirdn2d (csrc/upfirdn2d.cu, upfirdn2d_stream.cu,
upfirdn2d_tiled.cu + fir_passes.cuh), filtered_lrelu (filtered_lrelu_v3.cuh, filtered_lrelu.cu,
filtered_lrelu_act.cu) and bias_act (bias_act.cu).

Operands are sparse small integers (about 40 % zeros) and filters have dyadic taps k / 2^m with small k of both signs,
so a flipped or shifted filter changes the result. Gains, slopes and clamps are dyadic; filtered_lrelu folds
sqrt(up^2 * gain) into its up-sampling taps, so gain is 1 or 4 there, which keeps that root (and the one of the
adjoint's gain * up^2 / down^2) exact. Every product and partial sum is then a multiple of the operands' combined unit
u, and each test asserts its own precondition: the float64 oracle run on |x|, |f|, |b| stays below 2^p u, p = 24 for
the fp32 accumulators and shared-memory tiles and p = 11 for the fp16 intermediates of the composed paths (the
two-pass separable fallback of upfirdn2d.py, the composed filtered_lrelu), and every reference value is representable
in the output type. Whatever the summation order, FMA pairing or split into passes, each kernel must then equal the
oracle (oracle/oracle.py) element for element; a wrong tap, halo row, tile seam or sign byte changes at least one
element by at least one unit. Sign tensors are compared as whole uint8 tensors, padding columns included.

The case lists are plain data so that tests/test_ops_exact_host.py can check the operands and preconditions without a
GPU. `test_kernel_routes_reached` runs every case under torch.profiler and asserts that each kernel family and template
instance named in the case comments was launched."""
import re
import zlib

import numpy as np
import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu
DEV = 'cuda'
P_ACC = 24              # fp32 accumulators and shared-memory tiles
P_F16 = 11              # fp16 intermediates of the composed paths
DT = {'f16': torch.float16, 'f32': torch.float32, 'f64': torch.float64}


# ---------------------------------------------------------------------------------------------------------------------
# operands and exactness

def ints(shape, seed, vmax=2, density=0.6):
    """Sparse integers in [-vmax, vmax], float64 numpy."""
    rng = np.random.default_rng(seed)
    v = rng.integers(-vmax, vmax + 1, size=shape).astype(np.float64)
    return v * (rng.random(shape) < density)


def seed_of(name):
    return zlib.crc32(name.encode()) % 100003


def taps(n, seed, m=2, kmax=2, density=0.7):
    """n dyadic taps k / 2^m, k in [-kmax, kmax]; the end taps are non-zero and differ, so flips and shifts show."""
    rng = np.random.default_rng(seed + 7919)
    k = rng.integers(1, kmax + 1, size=n) * rng.choice([-1, 1], size=n) * (rng.random(n) < density)
    k[0], k[-1] = 1, -kmax if n > 1 else 1
    return (k / 2.0 ** m).astype(np.float64)


def unit_of(*arrays):
    """Product of the dyadic units of the operands: the largest 2^-k of which every value is a multiple."""
    u = 1.0
    for a in arrays:
        a = np.abs(np.asarray(a, np.float64)).ravel()
        k = 0
        while not np.all(np.mod(a * 2.0 ** k, 1.0) == 0):
            k += 1
            assert k < 60, 'operand is not dyadic'
        u *= 2.0 ** -k
    return u


def full(f):
    f = np.asarray(f, np.float64)
    return np.outer(f, f) if f.ndim == 1 else f


def check_bound(abs_ref, unit, p, what):
    m = float(np.max(np.abs(abs_ref))) if np.size(abs_ref) else 0.0
    assert m < 2.0 ** p * unit, f'{what}: precondition: |result| bound {m} >= 2^{p} units of {unit}'


def check_repr(ref, dtype, what):
    r = torch.as_tensor(np.asarray(ref, np.float64))
    assert torch.equal(r.to(dtype).double(), r), f'{what}: precondition: the exact result is not representable in {dtype}'


def assert_exact(got, ref, dtype, what):
    """got: kernel result (any device / dtype), ref: exact float64 values (numpy)."""
    check_repr(ref, dtype, what)
    ref = torch.as_tensor(np.asarray(ref, np.float64))
    got = got.detach().double().cpu()
    assert tuple(got.shape) == tuple(ref.shape), f'{what}: shape {tuple(got.shape)} != {tuple(ref.shape)}'
    if not torch.equal(got, ref):
        d = (got - ref).abs()
        i = int(torch.nonzero(d.flatten() > 0)[0])
        idx = tuple(int(j) for j in torch.unravel_index(torch.tensor(i), ref.shape))
        raise AssertionError(f'{what}: first mismatch at {idx}: got {float(got.flatten()[i])}, expected '
                             f'{float(ref.flatten()[i])}; {int((d > 0).sum())} of {ref.numel()} elements differ')


def assert_signs(got, ref, what):
    got = got.cpu().numpy()
    assert got.shape == ref.shape, f'{what}: sign tensor shape {got.shape} != {ref.shape}'
    if not np.array_equal(got, ref):
        idx = tuple(int(v[0]) for v in np.nonzero(got != ref))
        raise AssertionError(f'{what}: sign byte {idx}: got {got[idx]:#04x}, expected {ref[idx]:#04x}; '
                             f'{int((got != ref).sum())} of {ref.size} bytes differ')


def to_dev(a, dtype, layout='nchw'):
    """numpy -> device tensor in the requested memory layout: 'nchw', 'cl' (channels_last), 'off' (storage offset of
    one element: not 16-byte aligned)."""
    t = torch.as_tensor(np.asarray(a, np.float64)).to(DEV, dtype)
    if layout == 'cl':
        return t.contiguous(memory_format=torch.channels_last)
    if layout == 'off':
        buf = torch.zeros(t.numel() + 1, dtype=dtype, device=DEV)
        buf[1:].copy_(t.flatten())
        return buf[1:].view(t.shape).detach()
    return t.contiguous()


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def _pad4(p):
    return orc._pad4(p)


# ---------------------------------------------------------------------------------------------------------------------
# upfirdn2d cases. Every case runs forward and autograd backward (the adjoint: up <-> down, mirrored filter), compared
# with orc.upfirdn2d / orc.upfirdn2d_adjoint. `f` is a separable tap vector ([taps]) or a full 2-D filter.

F4, F8, F12, F24, F5 = taps(4, 1), taps(8, 2, m=3), taps(12, 3, m=2, density=0.5), taps(24, 4, m=2, density=0.35), taps(5, 5)
FY4 = F4[:, None]                 # [4, 1]: a 1-D pass along y
FX4 = F4[None, :]                 # [1, 4]: along x
FY12, FX12 = F12[:, None], F12[None, :]


def ucase(name, shape, f, up=1, down=1, pad=0, flip=False, gain=1, layout='nchw', dtypes=('f32', 'f16'), dbl=False,
          family=''):
    return dict(name=name, shape=tuple(shape), f=np.asarray(f, np.float64), up=up, down=down, pad=pad, flip=flip,
                gain=gain, layout=layout, dtypes=dtypes, dbl=dbl, family=family)


def _stream_cases():
    """upfirdn2d_stream.cu: 4 taps, UP2 = up 2 / pad0 2 / out 2 in, DOWN2 = down 2 / pad0 1 / out in / 2, per axis.
    dispatch(): (UP2, UP2) and (UP2, ID) take K_UP2N when iw <= 64 (2-sample strips), else K_UP2; strips = iw / NI
    must be a power of two <= 32 when x is filtered (NI = 2 UP2N, 4 UP2, 8 DOWN2). launch(): segments of
    seg_rows = (ceil(oh / nseg) + 1) & ~1 output rows, nseg <= oh / 8 -- oh = 42 gives 10-row segments, whose first
    input rows (UP2: o / 2 = 5, 10, ...) are odd and even."""
    c = []
    for iw in (2, 4, 8, 16, 32, 64, 128):                  # UP2N strips 1..32; iw 128: K_UP2 with 32 strips
        c.append(ucase(f'up2_up2_w{iw}', (1, 3, 6, iw), F4, up=2, pad=[2, 1, 2, 1], family='stream'))
    c.append(ucase('up2_up2_flip_gain', (2, 3, 21, 16), F4, up=2, pad=[2, 1, 2, 1], flip=True, gain=4, dbl=True,
                   family='stream'))
    for iw in (8, 16, 64, 256):                            # DOWN2 strips 1, 2, 8, 32
        c.append(ucase(f'down2_down2_w{iw}', (1, 3, 8, iw), F4, down=2, pad=1, family='stream'))
    c.append(ucase('down2_down2_seg', (1, 2, 84, 32), F4, down=2, pad=1, flip=True, gain=0.5, family='stream'))
    c.append(ucase('id_up2_seg', (1, 3, 21, 12), FY4, up=[1, 2], pad=[0, 0, 2, 1], family='stream'))
    c.append(ucase('id_down2_seg', (1, 3, 84, 20), FY4, down=[1, 2], pad=[0, 0, 1, 1], gain=2, family='stream'))
    c.append(ucase('up2n_id', (3, 1, 5, 8), FX4, up=[2, 1], pad=[2, 1, 0, 0], family='stream'))
    c.append(ucase('up2_id', (1, 1, 3, 128), FX4, up=[2, 1], pad=[2, 1, 0, 0], flip=True, family='stream'))
    c.append(ucase('down2_id', (1, 3, 5, 16), FX4, down=[2, 1], pad=[1, 1, 0, 0], family='stream'))
    return c


def _fallthrough_cases():
    """Streamed signatures the streamed kernel refuses; the tiled kernel must give the same exact result."""
    return [
        ucase('ft_strips3', (1, 2, 6, 12), F4, up=2, pad=[2, 1, 2, 1], family='tiled'),           # UP2N: 6 strips
        ucase('ft_strips64', (1, 1, 4, 512), F4, down=2, pad=1, family='tiled'),                  # DOWN2: 64 strips
        ucase('ft_ow_odd', (1, 2, 8, 14), FY4, down=[1, 2], pad=[0, 0, 1, 1], family='tiled'),     # ow % 4 != 0
        ucase('ft_offset', (2, 3, 6, 16), F4, up=2, pad=[2, 1, 2, 1], layout='off', family='tiled'),
        ucase('ft_channels_last', (2, 3, 8, 16), F4, down=2, pad=1, layout='cl', family='tiled'),
    ]


def _row12_cases():
    """upfirdn2d_row12_kernel: 12 taps, up 2 (pad0 6) / down 2 (pad0 5) along the contiguous axis, iw % 4 == 0 and
    ow % 4 == 0, fp16 up additionally ow % 8 == 0. Reached through [N, C, L, 1] tensors with [12, 1] filters (the
    transposed route of lvg_upfirdn2d) and through [1, 12] filters; the lengths straddle each condition."""
    c = []
    # up: ow = 2 L. With iw % 4 == 0, ow is always a multiple of 8, so the fp16 condition only fails with iw % 4 (L = 10)
    for L in (8, 10, 12, 16, 20):
        c.append(ucase(f'row12_up_t{L}', (2, 3, L, 1), FY12, up=[1, 2], pad=[0, 0, 6, 5], family='row12'))
        c.append(ucase(f'row12_up_x{L}', (1, 3, 2, L), FX12, up=[2, 1], pad=[6, 5, 0, 0], flip=True, family='row12'))
    for L in (16, 24, 40, 12):         # down: ow = L / 2 (L = 12: ow % 4 != 0 -> tiled)
        c.append(ucase(f'row12_down_t{L}', (2, 3, L, 1), FY12, down=[1, 2], pad=[0, 0, 5, 5], family='row12'))
        c.append(ucase(f'row12_down_x{L}', (1, 2, 3, L), FX12, down=[2, 1], pad=[5, 5, 0, 0], gain=2, family='row12'))
    c.append(ucase('row12_iw_odd', (1, 2, 1, 18), FX12, down=[2, 1], pad=[5, 5, 0, 0], family='row12'))   # iw % 4 != 0
    return c


# (name, f, up, down, pad) of the 15 LVG_TILED_CASE instances of upfirdn2d_tiled.cu; paddings avoid the streamed
# and row12 signatures
TILED = [
    ('U3_up2_f4', F4, 2, 1, [1, 2, 1, 2]),
    ('U4_down2_f4', F4, 1, 2, [2, 0, 2, 0]),
    ('U2_id_up2_f4', FY4, [1, 2], 1, [0, 0, 1, 2]),
    ('U5_id_down2_f4', FY4, 1, [1, 2], [0, 0, 2, 0]),
    ('U1_id_down2_f12', FY12, 1, [1, 2], [0, 0, 4, 6]),
    ('U1a_id_up2_f12', FY12, [1, 2], 1, [0, 0, 5, 6]),
    ('U1t_down2_f12_id', FX12, 1, [2, 1], [4, 6, 0, 0]),
    ('U1ta_up2_f12_id', FX12, [2, 1], 1, [5, 6, 0, 0]),
    ('U6_down4_f24', F24, 1, 4, [10, 10, 10, 10]),
    ('U9_down2_f12', F12, 1, 2, [5, 5, 5, 5]),
    ('U9_up2_f12', F12, 2, 1, [6, 5, 6, 5]),
    ('U6_up4_f24', F24, 4, 1, [12, 11, 12, 11]),
    ('U7_up4_f8', F8, 4, 1, [5, 2, 5, 2]),
    ('U7a_down4_f8', F8, 1, 4, [2, 2, 2, 2]),
    ('U8_blur_f4', F4, 1, 1, [1, 2, 1, 2]),
]


def _in_for(o, up, down, p0, p1, t):
    """Smallest input length whose output along one axis is at least o."""
    n = 1
    while (n * up + p0 + p1 - t + down) // down < o:
        n += 1
    return n


def _axis_taps(f):
    """(taps along x, taps along y) of a case filter: 1 on an axis it does not span."""
    return (f.shape[0], f.shape[0]) if f.ndim == 1 else (f.shape[1], f.shape[0])


# 'big' cases whose row tile is halved because a tile of round_up(16384 / tow, 4) rows exceeds 56 KB of shared memory
# (kept equal to what tiled_plan() computes by tests/test_ops_exact_host.py)
TILED_HALVED = {'U1_id_down2_f12', 'U1t_down2_f12_id', 'U1ta_up2_f12_id', 'U3_up2_f4', 'U4_down2_f4', 'U5_id_down2_f4',
                'U6_down4_f24', 'U7a_down4_f8', 'U8_blur_f4', 'U9_down2_f12', 'U9_up2_f12'}


def _tiled_cases():
    """launch_tiled() decides at run time, per call (tiled_plan() below replays it on the host):
      tow = ow if ow <= 256 else a width in 64..128            -> tiles_x = ceil(ow / tow) > 1 needs ow > 256
      toh = round_up(16384 / tow, 4) <= oh; = oh when tow == ow and the whole plane fits 56 KB of shared memory,
            else halved while the tile does not fit          -> tiles_y = ceil(oh / toh)
      pb  = min(16384 / (ow oh), 64, planes), then lowered until pb planes fit 56 KB; only when tiles_x == tiles_y == 1,
            planes > 1 and the planes are uniformly spaced (x.stride(0) == C x.stride(1), same for y)
      flat = 1 when the single tile's planes are dense NCHW, iw % V == 0 (V = 4 fp32, 8 fp16), aligned; flat = 2 when
            additionally every input sample lies inside the tile (no negative padding).
    Per instance, in fp32 and fp16: 'whole' (one plane, one tile, flat 2), 'batch' (89 small planes: pb > 1, and 89 is
    prime, so not a multiple of pb), 'crop' (every padding negative, pad - (taps // 2 + 3 + up): one tile, flat 1),
    'cl' (channels_last: non-flat loader, pb 1), 'odd' (iw % V != 0: non-flat loader), and in fp32 'big' (ow, oh >= 300:
    tiles_x, tiles_y > 1; toh is halved for the instances in TILED_HALVED). tests/test_ops_exact_host.py checks each of
    these claims against tiled_plan()."""
    c = []
    for name, f, up, down, pad in TILED:
        (ux, uy), (dx, dy) = _pair(up), _pair(down)
        tx, ty = _axis_taps(f)

        def ins(ow, oh, p):         # input size whose output is at least (oh, ow); width a multiple of 8
            return (_in_for(oh, uy, dy, p[2], p[3], ty),
                    -(-_in_for(ow, ux, dx, p[0], p[1], tx) // 8) * 8)
        h, w = ins(24, 16, pad)
        c.append(ucase(f'{name}_whole', (1, 1, h, w), f, up, down, pad, family='tiled'))
        h, w = ins(8, 6, pad)
        c.append(ucase(f'{name}_batch', (1, 89, h, w), f, up, down, pad, flip=True, gain=2, family='tiled'))
        # crop by more than half the filter plus one input sample, so the first input sample lies before the tile
        cx, cy = tx // 2 + 3 + ux, ty // 2 + 3 + uy
        cpad = [pad[0] - cx, pad[1] - cx, pad[2] - cy, pad[3] - cy]
        h, w = ins(16, 12, cpad)
        c.append(ucase(f'{name}_crop', (1, 1, h, w), f, up, down, cpad, family='tiled'))
        h, w = ins(16, 12, pad)
        c.append(ucase(f'{name}_cl', (2, 3, h, w), f, up, down, pad, layout='cl', family='tiled'))
        h, w = ins(13, 9, pad)
        c.append(ucase(f'{name}_odd', (1, 2, h, w + 5), f, up, down, pad, family='tiled'))
        h, w = ins(300, 300, pad)
        c.append(ucase(f'{name}_big', (1, 1, h, w), f, up, down, pad, gain=0.5, family='tiled', dtypes=('f32',)))
    return c


def tiled_plan(case, dtn):
    """Host replay of launch_tiled() (csrc/upfirdn2d_tiled.cu) for a case that reaches the tiled kernel through
    upfirdn2d.py's separable or one-axis route: tile sizes, whether toh was halved, plane batching and loader kind."""
    rup = lambda a, b: (a + b - 1) // b * b
    f = case['f']
    (ux, uy), (dx, dy) = _pair(case['up']), _pair(case['down'])
    px0, px1, py0, py1 = _pad4(case['pad'])
    tx, ty = _axis_taps(f)

    def axis(taps_, u, d):
        if taps_ == 1 and u == 1 and d == 1:
            return 'ID', 1, 1
        if u > 1 and d == 1 and taps_ % u == 0:
            return 'UP', u, taps_
        assert u == 1, 'no tiled instance'
        return 'DOWN', d, taps_
    (kx, sx, fx), (ky, sy, fy) = axis(tx, ux, dx), axis(ty, uy, dy)
    n, c, ih, iw = case['shape']
    oh, ow = (ih * uy + py0 + py1 - ty + dy) // dy, (iw * ux + px0 + px1 - tx + dx) // dx

    def in_extent(k, s, t, m):
        return m if k == 'ID' else (rup(m, 4) - 1) * s + t if k == 'DOWN' else rup((m + 2 * s - 2) // s, 4) + t // s

    def mid_extent(k, s, m):
        return rup((m + 2 * s - 2) // s, 4) * s if k == 'UP' else rup(m, 4)
    if ow <= 256:
        tow = ow
    else:
        best, waste_best = 64, None
        for cand in range(128, 63, -32):
            tiles = -(-ow // cand)
            last = ow - (tiles - 1) * cand
            waste = tiles * cand - ow + (rup(last, 32) - last)
            if waste_best is None or waste < waste_best:
                best, waste_best = cand, waste
        tow = best

    def smem(toh_, pb_):
        p_in = in_extent(kx, sx, fx, tow) | 1
        p_mid = (mid_extent(kx, sx, tow) + (sx if kx == 'UP' else 0)) | 1
        in_h = in_extent(ky, sy, fy, toh_)
        return (pb_ * in_h * p_in + (0 if kx == 'ID' else pb_ * in_h * p_mid) + fx + fy) * 4
    budget = 56 * 1024
    toh = min(rup(max(16384 // tow, 4), 4), oh)
    if tow == ow and smem(oh, 1) <= budget:
        toh = oh
    toh0 = toh
    while smem(toh, 1) > budget and toh > 4:
        toh = rup(toh // 2, 4)
    tiles_x, tiles_y = -(-ow // tow), -(-oh // toh)
    if case['layout'] == 'cl':
        xs, ys = (ih * iw * c, 1, iw * c, c), (oh * ow * c, 1, ow * c, c)
    else:
        xs, ys = (c * ih * iw, ih * iw, iw, 1), (c * oh * ow, oh * ow, ow, 1)
    uniform = xs[0] == c * xs[1] and ys[0] == c * ys[1]
    pb = 1
    if tiles_x == 1 and tiles_y == 1 and uniform and n * c > 1:
        pb = min(16384 // (ow * oh), 64, n * c)
        while pb > 1 and smem(toh, pb) > budget:
            pb -= 1
        pb = max(pb, 1)
    v = 8 if dtn == 'f16' else 4
    flat = int(tiles_x == 1 and tiles_y == 1 and xs[3] == 1 and xs[2] == iw and xs[1] == ih * iw and
               (pb == 1 or uniform) and iw % v == 0 and xs[0] % v == 0 and case['layout'] != 'off' and
               pb * ih * iw < (1 << 24))
    if flat:
        in_x0 = -px0 // sx if kx == 'UP' else -px0
        in_y0 = -py0 // sy if ky == 'UP' else -py0
        in_w = (rup((ow + (-px0 - in_x0 * sx) + sx - 1) // sx, 4) + fx // sx if kx == 'UP' else
                (ow - 1) * sx + fx if kx == 'DOWN' else ow)
        in_h = (rup((oh + (-py0 - in_y0 * sy) + sy - 1) // sy, 4) + fy // sy if ky == 'UP' else
                (oh - 1) * sy + fy if ky == 'DOWN' else oh)
        if in_x0 <= 0 and in_y0 <= 0 and iw - in_x0 <= in_w and ih - in_y0 <= in_h:
            flat = 2
    return dict(instance=(kx, sx, fx, ky, sy, fy), tow=tow, toh=toh, halved=toh < toh0, tiles_x=tiles_x,
                tiles_y=tiles_y, pb=pb, flat=flat, planes=n * c)


F35 = np.outer(taps(3, 11), taps(5, 12)) + np.pad(np.eye(3, 5), 0) / 4      # rank 2
RANK1_ASYM = np.outer(np.array([1, 3, 3, 1]) / 8, np.array([1, -1, 3, 2]) / 8)   # rank 1, factors not symmetric
RANK1_NEG = -np.outer(np.array([1, 3, 3, 1]) / 8, np.array([2, 1, 3, -1]) / 8)   # rank 1, negative peak


def _setup_filter_131():
    k = np.array([1, 3, 3, 1], np.float64)
    return np.outer(k, k) / 64.0        # setup_filter([1, 3, 3, 1]) of every conv2d_resample


def _generic_cases():
    """upfirdn2d_any_kernel (rank-2 filters, fp64, c_minor outputs) and the two-pass fallback of upfirdn2d.py (a
    separable filter without a tiled instance: two lvg_upfirdn2d calls, fp16 intermediate), and rank-1 full filters that
    go through the single-launch separable path and must equal the 2-D filter."""
    f131 = _setup_filter_131()
    return [
        ucase('any_rank2_3x5', (2, 3, 9, 11), F35, up=2, down=1, pad=[2, 3, 1, 2], dbl=True, family='any'),
        ucase('any_rank2_cl', (2, 3, 7, 8), F35, up=1, down=2, pad=[2, 2, 1, 1], layout='cl', family='any'),
        ucase('any_f64_sep', (2, 3, 8, 8), F4, up=2, pad=[2, 1, 2, 1], dtypes=('f64',), family='any'),
        ucase('any_f64_rank2', (1, 2, 6, 7), F35, down=2, pad=[1, 1, 1, 1], flip=True, dtypes=('f64',), family='any'),
        ucase('twopass_f5', (2, 3, 10, 12), F5, up=2, down=1, pad=[2, 2, 2, 2], family='any'),
        ucase('twopass_mixed', (1, 3, 9, 10), F4, up=[3, 2], down=[2, 3], pad=[1, 2, 2, 1], flip=True, family='any'),
        ucase('rank1_131_down2', (2, 3, 16, 16), f131, down=2, pad=[1, 1, 1, 1], family='tiled'),
        ucase('rank1_131_blur', (2, 3, 12, 12), f131, pad=[2, 2, 2, 2], family='tiled'),
        ucase('rank1_asym', (1, 3, 10, 12), RANK1_ASYM, pad=[1, 2, 1, 1], family='tiled'),
        ucase('rank1_neg_down2', (1, 2, 12, 16), RANK1_NEG, down=2, pad=[1, 2, 2, 1], gain=4, family='tiled'),
    ]


UPFIRDN_CASES = _stream_cases() + _fallthrough_cases() + _row12_cases() + _tiled_cases() + _generic_cases()


def is_two_pass(case):
    """A separable filter without a single-launch kernel: upfirdn2d.py runs two lvg_upfirdn2d passes with an
    intermediate in the input dtype."""
    return case['name'].startswith('twopass_')


def upfirdn_inputs(case):
    x = ints(case['shape'], seed_of(case['name']))
    ref = orc.upfirdn2d(x, full(case['f']), case['up'], case['down'], case['pad'], case['flip'], case['gain'])
    dy = ints(ref.shape, seed_of(case['name']) + 1)
    return x, dy


def upfirdn_refs(case, x, dy):
    """(y, dx) exact references plus the precondition checks of the case."""
    f = full(case['f'])
    up, down, pad, flip, gain = case['up'], case['down'], case['pad'], case['flip'], case['gain']
    y = orc.upfirdn2d(x, f, up, down, pad, flip, gain).astype(np.float64)
    dx = orc.upfirdn2d_adjoint(dy, f, x.shape, up, down, pad, flip, gain).astype(np.float64)
    u_f = unit_of(f, [min(gain, 1.0)])
    for a, r, what in ((x, y, 'forward'), (dy, dx, 'adjoint')):
        ab = (orc.upfirdn2d(np.abs(a), np.abs(f), up, down, pad, flip, gain) if what == 'forward' else
              orc.upfirdn2d_adjoint(np.abs(a), np.abs(f), x.shape, up, down, pad, flip, gain))
        check_bound(ab, unit_of(a) * u_f, P_ACC, f"{case['name']} {what}")
    if is_two_pass(case) and 'f16' in case['dtypes']:
        # the x pass ends in an fp16 tensor: its exact values need at most 11 significant bits
        fv = case['f']
        (ux, _), (dxs, _) = _pair(up), _pair(down)
        px0, px1, _, _ = _pad4(pad)
        mid = orc.upfirdn2d(np.abs(x), np.abs(fv)[None, :], [ux, 1], [dxs, 1], [px0, px1, 0, 0], flip, 1)
        check_bound(mid, unit_of(x, fv), P_F16, f"{case['name']} forward x pass (fp16)")
        check_bound(np.abs(dy).max() * np.abs(fv).sum(), unit_of(dy, fv), P_F16, f"{case['name']} adjoint x pass (fp16)")
    return y, dx


def _case_id(c):
    return c['name']


def _dt_cases(cases):
    return [pytest.param(c, d, id=f"{c['name']}-{d}") for c in cases for d in c['dtypes']]


def run_upfirdn(case, dtn, check=True):
    from torch_utils.ops import upfirdn2d as U
    dtype = DT[dtn]
    x_np, dy_np = upfirdn_inputs(case)
    x = to_dev(x_np, dtype, case['layout']).requires_grad_(True)
    f = torch.tensor(case['f'], dtype=torch.float32, device=DEV)
    y = U.upfirdn2d(x, f, up=case['up'], down=case['down'], padding=case['pad'], flip_filter=case['flip'],
                    gain=case['gain'])
    dy = to_dev(dy_np, dtype).requires_grad_(case['dbl'])
    dx, = torch.autograd.grad(y, x, dy, create_graph=case['dbl'])
    if not check:
        return
    y_ref, dx_ref = upfirdn_refs(case, x_np, dy_np)
    what = f"{case['name']} {dtn}"
    assert_exact(y, y_ref, dtype, what + ' forward')
    assert_exact(dx, dx_ref, dtype, what + ' adjoint')
    if case['dbl']:
        # d<dx, v>/d(dy) = A v: the forward operator again, through the adjoint's own backward pass
        v_np = ints(x_np.shape, 99)
        g, = torch.autograd.grad(dx, dy, to_dev(v_np, dtype))
        ref = orc.upfirdn2d(v_np, full(case['f']), case['up'], case['down'], case['pad'], case['flip'], case['gain'])
        assert_exact(g, ref, dtype, what + ' double backward')


@pytest.mark.parametrize('case,dtn', _dt_cases(UPFIRDN_CASES))
def test_upfirdn2d_exact(case, dtn):
    run_upfirdn(case, dtn)


# ---------------------------------------------------------------------------------------------------------------------
# filtered_lrelu cases. cfg: (up, down, fu taps, fd taps); configurations 1-3 have a fused kernel (v3 tiles 56 x 24,
# and 31 x 16 for configuration 3) for slope <= 1; slope > 1 takes the composed path.

FU12, FD12 = taps(12, 21, m=2, density=0.5), taps(12, 22, m=2, density=0.5)
FU24, FD24 = taps(24, 23, m=2, density=0.3), taps(24, 24, m=2, density=0.3)
CFGS = {1: (2, 2, FU12, FD12), 2: (4, 2, FU24, FD12), 3: (2, 4, FU12, FD24)}
FU8 = taps(8, 25, m=2)
FU2D = np.outer(taps(4, 26), taps(4, 27)) + np.eye(4) / 4                     # rank 2: no fused kernel


def flcase(name, cfg, n, c, oh, ow, px0, py0, flip=False, gain=1, slope=0.25, clamp='pick', dtypes=('f32', 'f16'),
           fu=None, fd=None, up=None, down=None, family='v3'):
    if cfg in CFGS:
        up, down, fu, fd = CFGS[cfg]
    return dict(name=name, cfg=cfg, n=n, c=c, oh=oh, ow=ow, px0=px0, py0=py0, flip=flip, gain=gain, slope=slope,
                clamp=clamp, dtypes=dtypes, fu=np.asarray(fu), fd=np.asarray(fd), up=up, down=down, family=family)


def fl_geometry(case):
    """Input size and padding that give exactly (oh, ow): px1 / py1 follow from the output size (either parity,
    negative when the model pads negatively)."""
    up, down = case['up'], case['down']
    fu, fd = full(case['fu']), full(case['fd'])
    out = []
    for o, p0, ft_u, ft_d in ((case['ow'], case['px0'], fu.shape[1] - 1, fd.shape[1] - 1),
                              (case['oh'], case['py0'], fu.shape[0] - 1, fd.shape[0] - 1)):
        need = o * down - (down - 1) + ft_u + ft_d          # up-sampled samples consumed
        i = max(1, -(-(need - 2 * p0) // up))
        p1 = need - i * up - p0
        out.append((i, p0, p1))
    (iw, px0, px1), (ih, py0, py1) = out
    return (case['n'], case['c'], ih, iw), [px0, px1, py0, py1]


def _fl_cases():
    c = []
    sizes = {1: ((24, 56), (24, 64), (32, 64)), 2: ((24, 56), (24, 64), (32, 64)), 3: ((16, 31), (16, 32))}
    for cfg, tiles in sizes.items():
        k = 0
        for th, tw in tiles:
            for o in (1, tw - 1, tw, tw + 1, 2 * tw + 1):
                oh = (1, th - 1, th, th + 1, 2 * th + 1)[k % 5]
                px0, py0 = ((9, 9), (-6, -6), (-11, -12), (10, 5), (3, -7))[k % 5]
                c.append(flcase(f'c{cfg}_{oh}x{o}_p{px0}', cfg, 1 + (k % 2) * 2, 1 + (k % 3), oh, o, px0, py0,
                                flip=bool(k % 2), gain=(1, 4)[k % 2]))
                k += 1
        # slope 2: the fused kernel declines (rc = -1), the composed path runs in every mode
        for oh in ((24, 32) if cfg != 3 else (16,)):
            c.append(flcase(f'c{cfg}_slope2_rc_oh{oh}', cfg, 1, 3, oh, 40, 9, 8, slope=2, family='composed'))
        c.append(flcase(f'c{cfg}_noclamp', cfg, 2, 3, 9, 17, 9, 9, clamp=None))
        c.append(flcase(f'c{cfg}_slope_half', cfg, 1, 2, 13, 20, -6, 9, slope=0.5, flip=True))
        c.append(flcase(f'c{cfg}_slope0_1', cfg, 1, 2, 7, 9, 9, -6, slope=0, gain=4))
        c.append(flcase(f'c{cfg}_slope1', cfg, 1, 1, 5, 6, 0, 1, slope=1))
    c.append(flcase('fl_1x1', None, 2, 3, 6, 13, 1, 0, fu=[[1.0]], fd=[[1.0]], up=1, down=1, family='1x1'))
    c.append(flcase('fl_1x1_slope2', None, 1, 2, 5, 9, -1, -1, fu=[[1.0]], fd=[[1.0]], up=1, down=1, slope=2, gain=4,
                    clamp=None, family='1x1'))
    c.append(flcase('fl_composed_f8', None, 1, 3, 9, 14, 4, 3, fu=FU8, fd=taps(4, 28), up=2, down=2, family='composed'))
    c.append(flcase('fl_composed_2d', None, 2, 2, 7, 10, 2, 2, fu=FU2D, fd=taps(4, 29), up=2, down=2, flip=True,
                    family='composed'))
    return c


FL_CASES = _fl_cases()


def fl_inputs(case):
    shape, pad = fl_geometry(case)
    seed = seed_of(case['name'])
    x = ints(shape, seed)
    b = ints([shape[1]], seed + 1, vmax=1, density=0.7)
    return x, b, pad


def fl_dy(case, shape):
    return ints(shape, seed_of(case['name']) + 2, vmax=1, density=0.5)


def fl_scale(case):
    """Positive factor in front of the activation: up^2 * gain."""
    return case['up'] ** 2 * case['gain']


def fl_pick_clamp(case, x, b, pad):
    """A clamp that many samples hit exactly: a value of |lrelu(v)| over the consumed pre-activation samples (the
    oracle run with clamp=None and 1x1 down filter reports v on the up-sampled grid)."""
    if case['clamp'] is None:
        return None
    fu = full(case['fu'])
    v = orc.upfirdn2d(x + b[None, :, None, None], fu, case['up'], 1, pad, case['flip'], fl_scale(case))
    v = np.where(v < 0, v * case['slope'], v)
    a = np.unique(np.abs(v[v != 0]))
    return float(a[len(a) * 2 // 3]) if len(a) else 1.0


def fl_refs(case, x, b, pad, clamp, signs=None, sx=0, sy=0, dy=None):
    """Exact forward (y, signs) or, with dy, the read-mode adjoint dx; with the precondition checks."""
    fu, fd, up, down = case['fu'], case['fd'], case['up'], case['down']
    slope, gain, flip = case['slope'], case['gain'], case['flip']
    smax = max(slope, 1.0)
    u_act = unit_of([min(slope, 1.0)] if slope else [1.0])
    if dy is None:
        res = orc.filtered_lrelu(x, fu, fd, b, up, down, pad, gain, slope, clamp, flip, signs_in=signs, sx=sx, sy=sy,
                                 return_signs=signs is None)
        y, s = res if signs is None else (res, None)
        ab = orc.filtered_lrelu(np.abs(x), np.abs(fu), np.abs(fd), np.abs(b), up, down, pad, gain * smax, 1.0, None, flip)
        check_bound(ab, unit_of(x + b[None, :, None, None], full(fu), full(fd)) * u_act, P_ACC, case['name'] + ' forward')
        if case['family'] == 'composed':
            mid = orc.upfirdn2d(np.abs(x) + np.abs(b)[None, :, None, None], np.abs(full(fu)), up, 1, pad, flip, up * up)
            check_bound(mid * gain * smax, unit_of(x + b[None, :, None, None], full(fu)) * u_act, P_F16,
                        case['name'] + ' up-sampled intermediate (fp16)')
        return y.astype(np.float64), s
    ia = adjoint_args(case, x.shape, dy.shape, pad, sx, sy)
    dx = orc.filtered_lrelu(dy, fd, fu, None, down, up, ia['pad'], ia['gain'], slope, None, not flip, signs_in=signs,
                            sx=ia['sx'], sy=ia['sy'])
    ab = orc.filtered_lrelu(np.abs(dy), np.abs(fd), np.abs(fu), None, down, up, ia['pad'], ia['gain'] * smax, 1.0, None,
                            not flip)
    check_bound(ab, unit_of(dy, full(fu), full(fd), [min(ia['gain'] * down ** 2, 1.0)]) * u_act, P_ACC,
                case['name'] + ' adjoint')
    return dx.astype(np.float64)


def adjoint_args(case, x_shape, y_shape, pad, sx, sy):
    """Padding, gain and sign offsets of the backward pass (filtered_lrelu.py backward())."""
    fu, fd = full(case['fu']), full(case['fd'])
    up, down = case['up'], case['down']
    px0, px1, py0, py1 = pad
    (_, _, xh, xw), (_, _, yh, yw) = x_shape, y_shape
    pp = [(fu.shape[1] - 1) + (fd.shape[1] - 1) - px0, xw * up - yw * down + px0 - (up - 1),
          (fu.shape[0] - 1) + (fd.shape[0] - 1) - py0, xh * up - yh * down + py0 - (up - 1)]
    return dict(pad=pp, gain=case['gain'] * up ** 2 / down ** 2, sx=sx - (fu.shape[1] - 1) + px0,
                sy=sy - (fu.shape[0] - 1) + py0)


def poisoned_blocks(*nbytes):
    """Allocate 0xFF-filled blocks of these byte sizes, in this order, on the current stream and free them again. Freeing
    merges the blocks back, so the caching allocator's free lists are as before and the next requests of the same sizes
    in the same order get exactly these blocks. Returns their addresses: the caller checks that its tensors landed there."""
    blocks = [torch.full([n], 255, dtype=torch.uint8, device=DEV) for n in nbytes]
    ptrs = [t.data_ptr() for t in blocks]
    del blocks
    return ptrs


def fl_plugin():
    """Binds the native library (the direct `_filtered_lrelu_cuda(...).apply` calls bypass filtered_lrelu()'s _init)."""
    from torch_utils.ops import filtered_lrelu as FL
    FL._init()
    return FL._plugin


def _fl_tensors(case, dtype, x_np, b_np):
    fu = torch.tensor(case['fu'], dtype=torch.float32, device=DEV)
    fd = torch.tensor(case['fd'], dtype=torch.float32, device=DEV)
    return to_dev(x_np, dtype), to_dev(b_np, dtype), fu, fd


def run_fl(case, dtn, check=True):
    """Write mode (forward with requires_grad), none mode (no_grad), read mode (the backward pass, and a direct call
    fed the oracle's signs)."""
    from torch_utils.ops import filtered_lrelu as FL
    dtype = DT[dtn]
    x_np, b_np, pad = fl_inputs(case)
    clamp = fl_pick_clamp(case, x_np, b_np, pad)
    x, b, fu, fd = _fl_tensors(case, dtype, x_np, b_np)
    fn = FL._filtered_lrelu_cuda(up=case['up'], down=case['down'], padding=pad, gain=case['gain'], slope=case['slope'],
                                 clamp=clamp, flip_filter=case['flip'])
    fl_plugin()
    what = f"{case['name']} {dtn}"
    # write mode. The fused kernels' forward allocates y, then the sign tensor, and nothing before them: both land in
    # 0xFF-poisoned memory, so a sign byte the kernel does not write shows up. (The composed path allocates its
    # intermediates first; there the poisoning is not guaranteed to reach the sign tensor.)
    ssh = orc.sign_shape(x_np.shape, case['fu'], case['fd'], case['up'], case['down'], pad)
    y_bytes = int(np.prod(orc.filtered_lrelu_out_shape(x_np.shape, case['fu'], case['fd'], case['up'], case['down'],
                                                       pad))) * torch.finfo(dtype).bits // 8
    xg, bg = x.clone().requires_grad_(True), b.clone().requires_grad_(True)
    ptrs = poisoned_blocks(y_bytes, int(np.prod(ssh)))
    y = fn.apply(xg, fu, fd, bg, None, 0, 0)
    signs = fl_saved_signs(y)
    if case['family'] != 'composed' and signs is not None:
        assert (y.data_ptr(), signs.data_ptr()) == tuple(ptrs), what + ': y / signs did not land in the poisoned blocks'
    with torch.no_grad():
        y_none = fn.apply(x, fu, fd, b, None, 0, 0)
    dy_np = fl_dy(case, tuple(y.shape))
    dy = to_dev(dy_np, dtype)
    dx, db = torch.autograd.grad(y, [xg, bg], dy)
    if not check:
        if signs is not None:
            with torch.no_grad():
                fn.apply(x, fu, fd, b, signs, 0, 0)
        return
    y_ref, s_ref = fl_refs(case, x_np, b_np, pad, clamp)
    assert_exact(y, y_ref, dtype, what + ' write-mode forward')
    assert_exact(y_none, y_ref, dtype, what + ' forward without signs')
    assert signs is not None, what + ': no sign tensor saved'
    assert_signs(signs, s_ref, what + ' signs')
    dx_ref = fl_refs(case, x_np, b_np, pad, clamp, signs=s_ref, dy=dy_np)
    assert_exact(dx, dx_ref, dtype, what + ' dx (read mode)')
    # db = dx.sum([0, 2, 3]) accumulates in fp32 (exact below 2^24 units) and rounds once to the dtype
    check_bound(np.abs(dx_ref).sum(axis=(0, 2, 3)), unit_of(dx_ref), P_ACC, what + ' db')
    assert_exact(db, torch.as_tensor(dx_ref.sum(axis=(0, 2, 3))).to(dtype).double().numpy(), dtype, what + ' db')
    # read mode directly: the forward operator with the oracle's signs replayed
    with torch.no_grad():
        y_read = fn.apply(x, fu, fd, b,
                          torch.as_tensor(s_ref).to(DEV).contiguous(), 0, 0)
    y_read_ref = fl_refs(case, x_np, b_np, pad, clamp, signs=s_ref)[0]
    assert_exact(y_read, y_read_ref, dtype, what + ' read-mode forward')


def fl_saved_signs(y):
    """The sign tensor the forward pass saved for backward (third saved tensor of _FilteredLRelu)."""
    s = y.grad_fn.saved_tensors[2]
    return s if s.numel() else None


@pytest.mark.parametrize('case,dtn', _dt_cases(FL_CASES))
def test_fl_exact(case, dtn):
    run_fl(case, dtn)


# read mode with random sign tensors: codes 0..3, tensors smaller / larger than the consumed extent, offsets of every
# sign and residue. Rows of s_wb % 4 == 0 bytes at a word-aligned address go to the v3 kernel as they are (entries 0,
# 6-9); for s_wb % 4 != 0 or a 1-3 byte storage offset the plugin passes a zero-padded, aligned copy (entries 1-5).
# fl_read_route() tells which.
FL_READ = []
for _cfg in (1, 2, 3):
    for _k, (_sx, _sy, _dh, _dwb, _off) in enumerate(((0, 0, 0, 0, 0), (-5, 3, -3, 1, 0), (6, -2, 4, 3, 0),
                                                      (-8, 7, 0, -2, 1), (3, 0, 2, 0, 3), (13, -9, -7, 5, 2),
                                                      (5, 3, 2, 4, 0), (-7, -5, -3, -4, 0), (2, -1, 5, 8, 0),
                                                      (-12, 9, -6, 4, 0))):
        FL_READ.append(dict(case=flcase(f'read_c{_cfg}_{_k}', _cfg, 1, 3, 20 + _k, 30 - _k, 9, -6, flip=bool(_k % 2),
                                        slope=(0.25, 0.5)[_k % 2], clamp=None),
                            sx=_sx, sy=_sy, dh=_dh, dwb=_dwb, off=_off))
FL_READ.append(dict(case=flcase('read_1x1', None, 2, 2, 5, 11, 0, 1, fu=[1.0], fd=[1.0], up=1, down=1, clamp=None,
                                family='1x1'), sx=-3, sy=1, dh=1, dwb=1, off=0))
FL_READ.append(dict(case=flcase('read_composed', None, 1, 2, 6, 9, 4, 3, fu=FU8, fd=taps(4, 28), up=2, down=2,
                                clamp=None, family='composed'), sx=5, sy=-2, dh=-1, dwb=2, off=0))


def fl_read_route(rc):
    """'v3' or 'padded' for configurations 1-3: whether FilteredLReluPlugin.filtered_lrelu passes the sign tensor to
    the v3 kernel as it is or as a zero-padded, aligned copy (custom_ops.py)."""
    case = rc['case']
    x, b, pad = fl_inputs(case)
    swb = max(1, orc.sign_shape(x.shape, case['fu'], case['fd'], case['up'], case['down'], pad)[3] + rc['dwb'])
    if case['cfg'] not in CFGS:
        return case['family']
    return 'v3' if swb % 4 == 0 and rc['off'] % 4 == 0 else 'padded'


def fl_read_inputs(rc):
    case = rc['case']
    x, b, pad = fl_inputs(case)
    n, c, sh, swb = orc.sign_shape(x.shape, case['fu'], case['fd'], case['up'], case['down'], pad)
    rng = np.random.default_rng(seed_of(case['name']))
    s = rng.integers(0, 256, size=(n, c, max(1, sh + rc['dh']), max(1, swb + rc['dwb']))).astype(np.uint8)
    return x, b, pad, s


def run_fl_read(rc, dtn, check=True):
    case = rc['case']
    dtype = DT[dtn]
    x_np, b_np, pad, s_np = fl_read_inputs(rc)
    x, b, fu, fd = _fl_tensors(case, dtype, x_np, b_np)
    buf = torch.zeros(s_np.size + 4, dtype=torch.uint8, device=DEV)
    s = buf[rc['off']: rc['off'] + s_np.size].view(s_np.shape)
    s.copy_(torch.as_tensor(s_np))
    from torch_utils.ops import filtered_lrelu as FL
    fl_plugin()
    fn = FL._filtered_lrelu_cuda(up=case['up'], down=case['down'], padding=pad, gain=case['gain'], slope=case['slope'],
                                 clamp=None, flip_filter=case['flip'])
    with torch.no_grad():
        y = fn.apply(x, fu, fd, b, s, rc['sx'], rc['sy'])
    if check:
        ref, _ = fl_refs(case, x_np, b_np, pad, None, signs=s_np, sx=rc['sx'], sy=rc['sy'])
        assert_exact(y, ref, dtype, f"{case['name']} {dtn} read mode sx={rc['sx']} sy={rc['sy']}")


@pytest.mark.parametrize('rc,dtn', [pytest.param(r, d, id=f"{r['case']['name']}-{d}") for r in FL_READ
                                     for d in ('f32', 'f16')])
def test_fl_read_random_signs(rc, dtn):
    run_fl_read(rc, dtn)


@pytest.mark.parametrize('cfg', sorted(CFGS))
def test_fl_fused_kernel_limits(cfg):
    """Configurations 1-3: with slope > 1 the plugin reports rc = -1, so the caller runs the composed path; and the
    library itself (no padded copy in between) refuses read-mode signs that do not start on a 4-byte boundary."""
    from torch_utils import custom_ops as co
    case = flcase(f'limits_c{cfg}', cfg, 1, 2, 7, 9, 9, 8)
    x_np, b_np, pad = fl_inputs(case)
    x, b, fu, fd = _fl_tensors(case, torch.float32, x_np, b_np)
    up, down = case['up'], case['down']
    _, _, rc = fl_plugin().filtered_lrelu(x, fu, fd, b, None, up, down, *pad, 0, 0, 1.0, 2.0, float('inf'), False, True)
    assert rc == -1, f'configuration {cfg}: slope 2 reached a fused kernel'
    n, c, sh, swb = orc.sign_shape(x_np.shape, case['fu'], case['fd'], up, down, pad)
    assert swb % 4 == 0
    s = torch.zeros(n * c * sh * swb + 4, dtype=torch.uint8, device=DEV)[1:1 + n * c * sh * swb].view(n, c, sh, swb)
    y = torch.empty(orc.filtered_lrelu_out_shape(x_np.shape, case['fu'], case['fd'], up, down, pad), device=DEV)
    lib = co.load_library()
    rc = lib.lvg_filtered_lrelu(x.data_ptr(), fu.data_ptr(), fd.data_ptr(), b.data_ptr(), s.data_ptr(), y.data_ptr(),
                                None, co._DTYPE_CODE[torch.float32], co._i4(x.shape), co._i4(x.stride()),
                                co._i4(y.shape), co._i4(y.stride()), len(case['fu']), 0, len(case['fd']), 0, up, down,
                                pad[0], pad[2], sh, swb, 0, 0, 1.0, 0.25, float('inf'), 0, 0, co._stream(x))
    assert rc > 0 and b'4-byte boundary' in lib.lvg_last_error(), (rc, lib.lvg_last_error())


# ---------------------------------------------------------------------------------------------------------------------
# bias_act: linear / relu / lrelu, the exact subset the networks use.

def bacase(name, shape, dim, act, alpha=None, gain=1.0, clamp=None, layout='nchw', dtypes=('f32', 'f16'), codes='1',
           fused='1', has_b=True):
    return dict(name=name, shape=tuple(shape), dim=dim, act=act, alpha=alpha, gain=gain, clamp=clamp, layout=layout,
                dtypes=dtypes, codes=codes, fused=fused, has_b=has_b)


def _ba_cases():
    """bias_act_vec_kernel bias modes (bias_act.cu launch_typed): BIAS_PER_PACK when step_b % N == 0 (N = 4 fp32,
    8 fp16), BIAS_PACKED when step_b == 1 and size_b % N == 0, BIAS_PER_ELEM otherwise; the scalar kernel takes fp64,
    unaligned operands and the tail under one pack. lvg_bias_act_grad_db falls back to bias_act(grad=1) + a sum when
    step_b % N != 0. The steps are not multiples of a warp's 128 (fp32) / 256 (fp16) elements, so one warp's packs span
    several channels, except lrelu_big, whose step of 4608 = 36 x 128 = 18 x 256 gives it rows longer than a
    4096-element tile and tiles that straddle rows."""
    c = []
    for codes in ('1', '0'):
        for fused in ('1', '0'):
            tag = f'c{codes}f{fused}'
            c += [
                bacase(f'lrelu_perpack_{tag}', (2, 12, 5, 4), 1, 'lrelu', 0.25, 2.0, 'pick', codes=codes, fused=fused),
                bacase(f'relu_perelem_{tag}', (4, 6, 5, 3), 1, 'relu', None, 0.5, None, codes=codes, fused=fused),
                bacase(f'lrelu_packed_{tag}', (16, 24), 1, 'lrelu', 0.5, 1.0, 'pick', codes=codes, fused=fused),
                bacase(f'linear_gain_{tag}', (3, 10, 6, 6), 1, 'linear', None, 2.0, None, codes=codes, fused=fused),
                bacase(f'lrelu_big_{tag}', (2, 20, 64, 72), 1, 'lrelu', 0.25, 1.0, None, codes=codes, fused=fused,
                       dtypes=('f32',)),
                # rows of 1025 packs against tiles of 1024 packs: the second tile starts with the last pack of a row
                bacase(f'relu_tile_edge_f32_{tag}', (2, 6, 41, 100), 1, 'relu', None, 2.0, None, codes=codes,
                       fused=fused, dtypes=('f32',)),
                bacase(f'relu_tile_edge_f16_{tag}', (2, 4, 41, 200), 1, 'relu', None, 1.0, None, codes=codes,
                       fused=fused, dtypes=('f16',)),
            ]
    c += [
        bacase('lrelu_tail', (3, 5, 7, 9), 1, 'lrelu', 0.5, 2.0, 'pick'),                    # n % N != 0
        bacase('relu_unaligned', (2, 8, 4, 4), 1, 'relu', None, 1.0, 'pick', layout='off'),
        bacase('lrelu_f64', (2, 6, 3, 5), 1, 'lrelu', 0.25, 0.5, 'pick', dtypes=('f64',)),
        bacase('linear_f64_nob', (2, 6, 3, 5), 1, 'linear', None, 2.0, None, dtypes=('f64',), has_b=False),
        bacase('relu_dim2', (2, 3, 24, 5), 2, 'relu', None, 2.0, None),
        bacase('lrelu_nob', (2, 7, 5, 8), 1, 'lrelu', 0.5, 1.0, 'pick', has_b=False),
    ]
    return c


BA_CASES = _ba_cases()


def ba_inputs(case):
    seed = seed_of(case['name'])
    x = ints(case['shape'], seed, vmax=3)
    b = ints([case['shape'][case['dim']]], seed + 1, vmax=2, density=0.8) if case['has_b'] else None
    dy = ints(case['shape'], seed + 2, vmax=3)
    v = ints(case['shape'], seed + 3, vmax=2)
    clamp = case['clamp']
    if clamp == 'pick':
        y = orc.bias_act(x, b, case['dim'], case['act'], case['alpha'], case['gain'], None).astype(np.float64)
        a = np.unique(np.abs(y[y != 0]))
        clamp = float(a[len(a) // 2]) if len(a) else 1.0
    return x, b, dy, v, clamp


def run_ba(case, dtn, monkeypatch=None, check=True):
    from torch_utils.ops import bias_act as BA
    if monkeypatch is not None:
        monkeypatch.setenv('LVG_BIAS_ACT_CODES', case['codes'])
        monkeypatch.setenv('LVG_BIAS_ACT_FUSED_DB', case['fused'])
    dtype = DT[dtn]
    x_np, b_np, dy_np, v_np, clamp = ba_inputs(case)
    kw = dict(dim=case['dim'], act=case['act'], alpha=case['alpha'], gain=case['gain'], clamp=clamp)
    x = to_dev(x_np, dtype, case['layout']).requires_grad_(True)
    b = to_dev(b_np, dtype).requires_grad_(True) if b_np is not None else None
    with torch.no_grad():
        y0 = BA.bias_act(x, b, **kw)
    y = BA.bias_act(x, b, **kw)
    dy = to_dev(dy_np, dtype, case['layout'])
    grads = torch.autograd.grad(y, [x] + ([b] if b is not None else []), dy)
    dyg = dy.clone().requires_grad_(True)
    dx2, = torch.autograd.grad(BA.bias_act(x, b, **kw), x, dyg, create_graph=True)
    g2 = torch.autograd.grad(dx2, dyg, to_dev(v_np, dtype, case['layout']), allow_unused=True)[0] if dx2.requires_grad else None
    if not check:
        return
    what = f"{case['name']} {dtn}"
    y_ref = orc.bias_act(x_np, b_np, case['dim'], case['act'], case['alpha'], case['gain'], clamp).astype(np.float64)
    check_bound(np.abs(x_np) + (np.abs(b_np).max() if b_np is not None else 0), unit_of(x_np), P_F16, what)
    assert_exact(y0, y_ref, dtype, what + ' forward (no grad)')
    assert_exact(y, y_ref, dtype, what + ' forward')
    gk = dict(y=y_ref.astype(np.float32), b=b_np, dim=case['dim'], act=case['act'], alpha=case['alpha'],
              gain=case['gain'], clamp=clamp)
    dx_ref = orc.bias_act_grad(dy_np, **gk).astype(np.float64)
    assert_exact(grads[0], dx_ref, dtype, what + ' dx')
    assert_exact(dx2, dx_ref, dtype, what + ' dx (create_graph)')
    if b is not None:
        axes = tuple(i for i in range(x_np.ndim) if i != case['dim'])
        db_ref = dx_ref.sum(axis=axes)
        check_bound(np.abs(dx_ref).sum(axis=axes), unit_of(dx_ref), P_ACC, what + ' db')
        assert_exact(grads[1], torch.as_tensor(db_ref).to(dtype).double().numpy(), dtype, what + ' db')
    if g2 is not None:
        assert_exact(g2, orc.bias_act_grad(v_np, **gk).astype(np.float64), dtype, what + ' d(dx)/d(dy)')


@pytest.mark.parametrize('case,dtn', _dt_cases(BA_CASES))
def test_bias_act_exact(case, dtn, monkeypatch):
    run_ba(case, dtn, monkeypatch)


# ---------------------------------------------------------------------------------------------------------------------
# route coverage, observed with torch.profiler

def expected_kernels():
    """Regexes over the demangled kernel names (spaces removed); T = float | __half."""
    T = r'(float|__half)'
    k = {}
    for kx, ky in ((1, 1), (2, 2), (0, 1), (0, 2), (1, 0), (2, 0), (3, 1), (3, 0)):     # K_UP2N = 3 (x axis only)
        k[f'stream<{kx},{ky}>'] = rf'upfirdn2d_stream_kernel<{T},{kx},{ky}>'
    for up in ('true', 'false'):
        k[f'row12<{up}>'] = rf'upfirdn2d_row12_kernel<{T},{up}>'
    axis = {'UP': 1, 'DOWN': 2, 'ID': 0}
    inst = [('UP', 2, 4, 'UP', 2, 4), ('DOWN', 2, 4, 'DOWN', 2, 4), ('ID', 1, 1, 'UP', 2, 4), ('ID', 1, 1, 'DOWN', 2, 4),
            ('ID', 1, 1, 'DOWN', 2, 12), ('ID', 1, 1, 'UP', 2, 12), ('DOWN', 2, 12, 'ID', 1, 1), ('UP', 2, 12, 'ID', 1, 1),
            ('DOWN', 4, 24, 'DOWN', 4, 24), ('DOWN', 2, 12, 'DOWN', 2, 12), ('UP', 2, 12, 'UP', 2, 12),
            ('UP', 4, 24, 'UP', 4, 24), ('UP', 4, 8, 'UP', 4, 8), ('DOWN', 4, 8, 'DOWN', 4, 8), ('DOWN', 1, 4, 'DOWN', 1, 4)]
    for kx, sx, fx, ky, sy, fy in inst:
        k[f'tiled<{kx}{sx}x{fx},{ky}{sy}x{fy}>'] = rf'upfirdn2d_tiled_kernel<{T},{axis[kx]},{sx},{fx},{axis[ky]},{sy},{fy}>'
    for t in ('float', '__half', 'double'):
        k[f'any<{t}>'] = rf'upfirdn2d_any_kernel<{t}>'
    geoms = ('2,12,2,12,56,24,6,2,4,4', '4,24,2,12,56,24,2,2,4,4', '2,12,4,24,31,16,8,6,4,2')
    for g in geoms:
        for mode in (0, 1, 2):
            k[f'v3<{g}>,{mode}'] = rf'filtered_lrelu_v3_kernel<{T},lvg::flv3::Geom<{g}>,{mode}>'
    for mode in (0, 1, 2):
        k[f'1x1,{mode}'] = rf'filtered_lrelu_1x1_kernel<{T},{mode}>'
        k[f'act,{mode}'] = rf'filtered_lrelu_act_kernel<{T},{mode}>'
    k['bias_act_vec'] = r'bias_act_vec_kernel<'
    k['bias_act_scalar'] = r'bias_act_scalar_kernel<'
    return k


def all_runs():
    for c in UPFIRDN_CASES:
        for d in c['dtypes']:
            yield run_upfirdn, (c, d)
    for c in FL_CASES:
        for d in c['dtypes']:
            yield run_fl, (c, d)
    for r in FL_READ:
        for d in ('f32', 'f16'):
            yield run_fl_read, (r, d)
    for c in BA_CASES:
        for d in c['dtypes']:
            yield run_ba, (c, d)


def test_kernel_routes_reached(monkeypatch):
    from torch.profiler import ProfilerActivity, profile
    names = set()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for fn, args in all_runs():
            if fn is run_ba:
                monkeypatch.setenv('LVG_BIAS_ACT_CODES', args[0]['codes'])
                monkeypatch.setenv('LVG_BIAS_ACT_FUSED_DB', args[0]['fused'])
            fn(*args, check=False)
        torch.cuda.synchronize()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            names.add(re.sub(r'\s+', '', e.name))
    if not names:
        pytest.skip('torch.profiler reported no CUDA kernels on this machine, so launches cannot be observed')
    missed = [k for k, rx in expected_kernels().items() if not any(re.search(rx, n) for n in names)]
    print('kernels seen:', len(names))
    assert not missed, 'kernel instances never launched: ' + ', '.join(missed)
