"""Bit-exact checks of the convolution kernels (csrc/conv_igemm.cu, conv_pointwise.cu, fir1d.cu) over the
envelope `ConvNdPlugin._in_envelope` declares.

The operands are sparse small integers (x in {-1, 0, 1}, w in {-2, ..., 2}) or, for the fp32 split path, dyadic values
whose bf16 lo half is not zero (1 + 2^-8 -> hi 1, lo 2^-8). Every product and every partial sum is then a multiple of a
unit u far below 2^24 u, so the fp32 accumulator is exact in any order and under any alignment of the tensor core's
adder, and the result is representable in the output type: the kernel must equal the float64 reference bit for bit.
The fp32 reference is what the split path computes, hi*hi + hi*lo + lo*hi with hi / lo from torch's round-to-nearest-even
bf16 conversion: a missing, duplicated or misplaced product, halo column or tile edge changes at least one element by at
least one unit, which a norm-wise tolerance would dilute. Each test asserts its own precondition (the sum of |products|
per output is at most 2048 u for fp16 outputs and 2^20 u otherwise); a failing precondition is a wrong test, not a wrong
kernel. Shapes sample the envelope pairwise: every (kh, kw), kt 1..7, strides 1-4, paddings 0..k-1, groups, 64-row mode /
one 128-row tile / several m-tiles, column-tile and stride-lattice edges, sizes of 1; the tiling knobs of the engine are
re-run on a subset and must give the same bits."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from torch_utils import custom_ops

pytestmark = pytest.mark.gpu
DEV = 'cuda'
DT_IDS = {torch.float16: 'f16', torch.float32: 'f32split'}
BOUND = {torch.float16: 2048.0, torch.float32: float(2 ** 20)}
UNIT_DYADIC = 2.0 ** -8          # hi*lo products of the dyadic operands below are multiples of 2^-8


@pytest.fixture(scope='module')
def plug():
    return custom_ops.get_plugin('convnd_plugin')


def ints(shape, seed, vmax, density=0.5):
    """Sparse integers in [-vmax, vmax] (float64, on the device)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    v = torch.randint(-vmax, vmax + 1, shape, generator=g, device=DEV).double()
    keep = torch.rand(shape, generator=g, device=DEV) < density
    return v * keep


def dyadic(shape, seed, vmax, density=0.5):
    """Integers as above, a third of them moved by one bf16 half-step: v (1 + 2^-8) -> bf16 hi = v, lo = v 2^-8 (v = +-1, +-2)."""
    g = torch.Generator(device=DEV).manual_seed(seed + 1000)
    v = ints(shape, seed, vmax, density)
    bump = torch.rand(shape, generator=g, device=DEV) < 1 / 3
    return torch.where(bump, v * (1 + 2.0 ** -8), v)


def lo_half(v):
    """The bf16 lo half of fp32 values: v - bf16_rn(v), rounded to bf16 (what the split path's re-tiling computes)."""
    return (v - v.to(torch.bfloat16).double()).to(torch.bfloat16).double()


def operands(shapes, seeds, vmaxes, dtype, dyad, density=0.5):
    make = dyadic if dyad else ints
    return [make(s, seed, vm, density) for s, seed, vm in zip(shapes, seeds, vmaxes)]


def first_mismatch(got, exp, unit):
    d = (got.double() - exp).abs()
    bad = ~(d == 0)                         # NaN included: an element the kernel never wrote into a NaN-filled output
    i = int(torch.nonzero(bad.flatten())[0])
    idx = list(torch.unravel_index(torch.tensor(i), exp.shape))
    return (f'first mismatch at {tuple(int(j) for j in idx)} (n, c, [t,] [y,] x): got {float(got.flatten()[i])}, '
            f'expected {float(exp.flatten()[i])}, difference {float(d.flatten()[i]) / unit:g} units; '
            f'{int(bad.sum())} of {exp.numel()} elements differ')


def assert_exact(got, exp, absum, dtype, unit, what):
    """got (kernel output), exp (float64 reference), absum (float64 sum of |products| per output element)."""
    assert float(absum.max()) <= BOUND[dtype] * unit, f'{what}: precondition: sum |products| {float(absum.max())} > {BOUND[dtype]} units'
    assert torch.equal(exp.to(got.dtype).double(), exp), f'{what}: precondition: the exact result is not representable'
    assert got.shape == exp.shape and got.dtype == dtype, (what, got.shape, exp.shape, got.dtype)
    assert torch.equal(got, exp.to(dtype)), f'{what}: ' + first_mismatch(got, exp, unit)


def conv5(x, w, stride, pad, groups):
    """float64 convolution of 3-/4-/5-D tensors with (1, s, s) stride (torch.nn.functional, any rank)."""
    nd = x.ndim - 2
    st = (1, stride, stride)[3 - nd:]
    return (F.conv1d, F.conv2d, F.conv3d)[nd - 1](x, w, stride=st, padding=tuple(pad)[-nd:], groups=groups)


def grads(x, w, dy, stride, pad, groups):
    """(y, dx, dw) of y = conv(x, w) with output gradient dy, float64."""
    x, w = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = conv5(x, w, stride, pad, groups)
    if dy is None:
        return y.detach(), None, None
    dx, dw = torch.autograd.grad(y, [x, w], dy)
    return y.detach(), dx, dw


def split_exact(x, w, dy, stride, pad, groups, dtype):
    """Expected (y, dx, dw) of the engine: all products for fp16 (exact operands), hi*hi + hi*lo + lo*hi for split fp32 --
    by bilinearity the full product minus lo*lo -- and the sums of |products| (preconditions)."""
    full = grads(x, w, dy, stride, pad, groups)
    ab = grads(x.abs(), w.abs(), None if dy is None else dy.abs(), stride, pad, groups)
    if dtype == torch.float16:
        return full, ab
    lolo = grads(lo_half(x), lo_half(w), None if dy is None else lo_half(dy), stride, pad, groups)
    return tuple(None if f is None else f - l for f, l in zip(full, lolo)), ab


def plan_flags(plug, xs, ws, pad, groups, stride, dtype):
    """(forward, input gradient) run by the streaming 1x1x1 kernels instead of the engine?"""
    args, _, _, _ = plug._args(tuple(xs), tuple(ws), pad, groups, dtype)
    out = (ctypes.c_int * 48)()
    flags = []
    for mode in (0, 1):
        assert plug._lib.lvg_convnd_plan(mode, *args, stride, out, 48) == 0, plug._lib.lvg_last_error().decode()
        flags.append(bool(out[47]))
    return flags


# ---- shapes: (x shape, w shape, padding (t, h, w), stride, groups), pairwise over the envelope's axes
KERNELS_2D = [(kh, kw) for kh in range(1, 10) for kw in range(1, 4) if kh * kw <= 9]
CHANNELS = [(3, 17), (17, 65), (65, 130), (130, 3), (24, 40), (16, 200), (40, 64), (1, 1)]
EXTENTS = [(9, 100), (1, 130), (5, 256), (17, 64), (3, 253), (6, 70), (12, 127), (2, 252), (1, 1), (7, 129)]
GROUPS = [1, 1, 3, 1]


def _cases():
    cases = []
    for i, (kh, kw) in enumerate(KERNELS_2D):
        stride = 1 + i % 4
        cin, cout = CHANNELS[i % len(CHANNELS)]
        groups = GROUPS[i % len(GROUPS)]
        H, W = EXTENTS[i % len(EXTENTS)]
        pad = (0, (i // 2) % kh, (i // 3) % kw)
        H, W = max(H, kh - 2 * pad[1]), max(W, kw - 2 * pad[2])
        cases.append(((2, groups * cin, H, W), (groups * cout, cin, kh, kw), pad, stride, groups))
    for kt in range(1, 8):
        kh, kw = [(3, 3), (1, 1), (3, 1), (1, 3), (2, 2), (3, 3), (1, 1)][kt - 1]
        cin, cout = CHANNELS[(kt + 2) % len(CHANNELS)]
        T = [1, 4, 7, 2, 11, 8, 9][kt - 1]
        H, W = [(5, 16), (9, 20), (1, 40), (6, 130), (3, 7), (4, 5), (1, 1)][kt - 1]
        pad = ((kt - 1) - (kt // 2) % kt if T < kt else kt // 2, kh // 2, kw // 2)
        groups = 3 if kt == 3 else 1
        cases.append(((1, groups * cin, T, H, W), (groups * cout, cin, kt, kh, kw), pad, 1, groups))
    cases += [((3, 64, 31), (48, 64, 3), (0, 0, 1), 1, 1), ((2, 5, 1), (7, 5, 1), (0, 0, 0), 1, 1), ((1, 130, 300), (65, 130, 2), (0, 0, 1), 1, 1)]
    # several tiles per persistent CTA (hundreds of tiles), and the 64-row mode next to a single 128-row tile
    cases += [((4, 32, 40, 96), (64, 32, 3, 3), (0, 1, 1), 1, 1), ((2, 48, 33, 40), (128, 48, 3, 3), (0, 1, 1), 1, 1)]
    return cases


CASES = _cases()


def case_id(c):
    xs, ws, pad, stride, groups = c
    return f"x{'x'.join(map(str, xs[1:]))}-k{'x'.join(map(str, ws[2:]))}-p{''.join(map(str, pad))}-s{stride}-g{groups}"


def run_engine(plug, xs, ws, pad, stride, groups, dtype, dyad, seed=0, entry='separate'):
    nd = len(xs) - 2
    ys = tuple(conv5(torch.zeros(1, *xs[1:], device=DEV, dtype=torch.float64), torch.zeros(*ws, device=DEV, dtype=torch.float64),
                     stride, pad, groups).shape[1:])
    fan = math.prod(ws[1:])
    dens = min(0.5, 300.0 / fan)          # sum |x||w| per output stays ~ 300 * E|w|
    x, w, dy = operands([xs, ws, (xs[0],) + ys], [seed + 1, seed + 2, seed + 3], [1, 2, 1], dtype, dyad, dens)
    x, w, dy = (v.to(dtype).double() for v in (x, w, dy))              # the values are representable: no change
    pd = list(pad[3 - nd:])
    out = {}
    if entry == 'backward':
        y = plug.fprop(x.to(dtype), w.to(dtype), pd, groups, stride=stride)
        out['dx'], out['dw'] = plug.backward(x.to(dtype), dy.to(dtype), w.to(dtype), pd, groups, stride=stride)
    else:
        y = plug.fprop(x.to(dtype), w.to(dtype), pd, groups, stride=stride)
        out['dx'] = plug.dgrad(dy.to(dtype), w.to(dtype), tuple(xs), pd, groups, stride=stride)
        out['dw'] = plug.wgrad(x.to(dtype), dy.to(dtype), tuple(ws), pd, groups, stride=stride)
    out['y'] = y
    return x, w, dy, out


def check_engine(plug, case, dtype, dyad, entry='separate', seed=0):
    xs, ws, pad, stride, groups = case
    nd = len(xs) - 2
    assert plug._in_envelope(xs, ws, dtype, stride, list(pad[3 - nd:]), 1, groups), 'shape outside the envelope'
    pw = plan_flags(plug, xs, ws, list(pad[3 - nd:]), groups, stride, dtype)
    if dyad and any(pw):
        pytest.skip('the streaming 1x1x1 kernels compute full fp32 products: checked with integers')
    x, w, dy, out = run_engine(plug, xs, ws, pad, stride, groups, dtype, dyad, seed, entry)
    (y, dx, dw), (ay, adx, adw) = split_exact(x, w, dy, stride, pad, groups, dtype)
    unit = UNIT_DYADIC if dyad else 1.0
    assert_exact(out['y'], y, ay, dtype, unit, f'{entry} forward')
    assert_exact(out['dx'], dx, adx, dtype, unit, f'{entry} input gradient')
    assert_exact(out['dw'], dw, adw, dtype, unit, f'{entry} weight gradient')
    return out


@pytest.mark.parametrize('dtype,dyad', [(torch.float16, False), (torch.float32, False), (torch.float32, True)],
                         ids=['f16', 'f32split-int', 'f32split-dyadic'])
@pytest.mark.parametrize('case', CASES, ids=[case_id(c) for c in CASES])
def test_engine_exact(plug, case, dtype, dyad):
    check_engine(plug, case, dtype, dyad)


# the one-call backward (dy re-tiled once when the paddings agree) on a subset, both re-tiling layouts
BACKWARD_CASES = [CASES[i] for i in (0, 2, 5, 9, 14)] + [CASES[len(KERNELS_2D) + 2], CASES[-2], CASES[-1]]


@pytest.mark.parametrize('dtype,dyad', [(torch.float16, False), (torch.float32, True)], ids=['f16', 'f32split-dyadic'])
@pytest.mark.parametrize('case', BACKWARD_CASES, ids=[case_id(c) for c in BACKWARD_CASES])
def test_one_call_backward_exact(plug, case, dtype, dyad):
    check_engine(plug, case, dtype, dyad, entry='backward')


# ---- tiling invariance: every knob re-tiles the same sums, so every variant equals the same exact answer
KNOBS = [('LVG_CONV_COLS', v) for v in ('64', '128', '192')] + [('LVG_CONV_CTAS', v) for v in ('1', '5')] + \
        [('LVG_CONV_M64', '0'), ('LVG_CONV_RESIDENT_W', '0'), ('LVG_PACKW_CHUNKS', '1'), ('LVG_PACKW_CHUNKS', '8'),
         ('LVG_WGRAD_NSPLIT', '1'), ('LVG_WGRAD_NSPLIT', '7'), ('LVG_WGRAD_FOLD', '0'), ('LVG_WGRAD_COMPACT', '0'), ('LVG_WGRAD_M64', '0')]
KNOB_CASES = [CASES[i] for i in (0, 1, 3, 12)] + [CASES[len(KERNELS_2D)], CASES[-2]]


@pytest.mark.parametrize('knob,value', KNOBS, ids=[f'{k}={v}' for k, v in KNOBS])
@pytest.mark.parametrize('dtype,dyad', [(torch.float16, False), (torch.float32, True)], ids=['f16', 'f32split-dyadic'])
def test_tiling_knobs_exact(plug, monkeypatch, knob, value, dtype, dyad):
    monkeypatch.setenv(knob, value)
    for case in KNOB_CASES:
        xs, ws, pad, stride, groups = case
        if dyad and any(plan_flags(plug, xs, ws, list(pad[3 - (len(xs) - 2):]), groups, stride, dtype)):
            continue
        check_engine(plug, case, dtype, dyad)


# ---- the fused epilogue: integer bias, lrelu alpha 0.25, gain 2 or 0.5, integer clamp
@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
@pytest.mark.parametrize('act,gain,clamp', [(1, 2.0, -1.0), (2, 0.5, 6.0), (2, 2.0, -1.0), (1, 0.5, 3.0)])
def test_fused_epilogue_exact(plug, act, gain, clamp, dtype):
    for case in (CASES[0], CASES[4], CASES[len(KERNELS_2D) + 1]):
        xs, ws, pad, stride, groups = case
        nd = len(xs) - 2
        x, w = ints(xs, 7, 1, 0.3), ints(ws, 8, 2, 0.3)
        b = ints((ws[0],), 9, 5, 1.0)
        y = plug.fprop(x.to(dtype), w.to(dtype), list(pad[3 - nd:]), groups, bias=b.float(), act=act, alpha=0.25, gain=gain,
                       clamp=clamp, stride=stride)
        z = conv5(x, w, stride, pad, groups) + b.view([1, -1] + [1] * nd)
        if act == 2:
            z = torch.where(z < 0, z * 0.25, z)
        z = z * gain
        if clamp >= 0:
            z = z.clamp(-clamp, clamp)
        absum = conv5(x.abs(), w.abs(), stride, pad, groups)
        assert_exact(y, z, absum, dtype, 1.0, f'epilogue {case_id(case)}')


# ---- conv_nd autograd, conv_transpose2d, and the F proxy at strides 3 / 4 over rows wider than one 256-column tile row
@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
def test_conv_nd_autograd_exact(dtype):
    from torch_utils.ops import conv_nd
    for (xs, ws, pad, stride, groups) in (CASES[1], CASES[6], CASES[len(KERNELS_2D) + 3], CASES[len(KERNELS_2D) + 7]):
        nd = len(xs) - 2
        x, w = ints(xs, 11, 1, 0.4), ints(ws, 12, 2, min(0.5, 300 / math.prod(ws[1:])))
        xa, wa = x.to(dtype).requires_grad_(True), w.to(dtype).requires_grad_(True)
        fn = (conv_nd.conv1d, conv_nd.conv2d, conv_nd.conv3d)[nd - 1]
        st = stride if nd == 2 else 1
        y = fn(xa, wa, None, st, list(pad[3 - nd:]), 1, groups)
        dy = ints(tuple(y.shape), 13, 1, 0.5)
        y.backward(dy.to(dtype))
        (ye, dxe, dwe), (ay, adx, adw) = split_exact(x, w, dy, st, pad, groups, dtype)
        assert_exact(y.detach(), ye, ay, dtype, 1.0, 'conv_nd forward')
        assert_exact(xa.grad, dxe, adx, dtype, 1.0, 'conv_nd input gradient')
        assert_exact(wa.grad, dwe, adw, dtype, 1.0, 'conv_nd weight gradient')


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
@pytest.mark.parametrize('k,pad', [((3, 3), 1), ((2, 2), 0), ((3, 1), 1)])
def test_conv_transpose2d_stride2_output_padding_exact(dtype, k, pad):
    from torch_utils.ops import conv_nd
    xs, ws = (2, 24, 9, 66), (24, 40, *k)
    x, w = ints(xs, 21, 1, 0.4), ints(ws, 22, 2, 0.4)
    xa, wa = x.to(dtype).requires_grad_(True), w.to(dtype).requires_grad_(True)
    y = conv_nd.conv_transpose2d(xa, wa, None, 2, pad, 1)
    dy = ints(tuple(y.shape), 23, 1, 0.5)
    y.backward(dy.to(dtype))
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    yr = F.conv_transpose2d(xr, wr, None, 2, pad, 1)
    dxr, dwr = torch.autograd.grad(yr, [xr, wr], dy)
    xb, wb = x.abs().requires_grad_(True), w.abs().requires_grad_(True)
    yb = F.conv_transpose2d(xb, wb, None, 2, pad, 1)
    adx, adw = torch.autograd.grad(yb, [xb, wb], dy.abs())
    assert_exact(y.detach(), yr.detach(), yb.detach(), dtype, 1.0, 'conv_transpose2d')
    assert_exact(xa.grad, dxr, adx, dtype, 1.0, 'conv_transpose2d input gradient')
    assert_exact(wa.grad, dwr, adw, dtype, 1.0, 'conv_transpose2d weight gradient')


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
@pytest.mark.parametrize('stride,W,k', [(3, 100, (3, 3)), (3, 256, (1, 1)), (4, 70, (3, 3)), (4, 200, (2, 3)), (2, 252, (2, 2))])
def test_functional_proxy_strided_wide_rows_exact(dtype, stride, W, k):
    from torch_utils.ops import conv_nd
    xs, ws, pad = (2, 16, 11, W), (24, 16, *k), (k[0] // 2, k[1] // 2)
    assert conv_nd._native_ok(torch.empty(xs, device=DEV, dtype=dtype), torch.empty(ws, device=DEV, dtype=dtype), stride, pad, 1, 1)
    x, w = ints(xs, 31, 1, 0.5), ints(ws, 32, 2, 0.5)
    xa, wa = x.to(dtype).requires_grad_(True), w.to(dtype).requires_grad_(True)
    y = conv_nd.functional.conv2d(xa, wa, None, stride, pad)
    dy = ints(tuple(y.shape), 33, 1, 0.5)
    y.backward(dy.to(dtype))
    (ye, dxe, dwe), (ay, adx, adw) = split_exact(x, w, dy, stride, (0,) + pad, 1, dtype)
    assert_exact(y.detach(), ye, ay, dtype, 1.0, 'F.conv2d forward')
    assert_exact(xa.grad, dxe, adx, dtype, 1.0, 'F.conv2d input gradient')
    assert_exact(wa.grad, dwe, adw, dtype, 1.0, 'F.conv2d weight gradient')


# ---- conv2d_gradfix.conv2d (the reference's entry point) in fp16: forward, then both gradients through autograd
@pytest.mark.parametrize('xs,ws,pad,groups', [((1, 4 * 24, 20, 26), (4 * 40, 24, 3, 3), (2, 2), 4), ((2, 40, 17, 130), (24, 40, 1, 1), (0, 0), 1),
                                              ((2, 16, 1, 9), (70, 16, 3, 3), (1, 1), 1)])
def test_conv2d_gradfix_exact(xs, ws, pad, groups):
    from torch_utils.ops import conv2d_gradfix, conv_nd
    x, w = ints(xs, 41, 1, 0.5), ints(ws, 42, 2, 0.5)
    xa, wa = x.half().requires_grad_(True), w.half().requires_grad_(True)
    assert conv_nd._native_ok(xa, wa, 1, pad, 1, groups), 'expected the engine'
    y = conv2d_gradfix.conv2d(xa, wa, padding=pad, groups=groups)
    dy = ints(tuple(y.shape), 43, 1, 0.5)
    dx, dw = torch.autograd.grad(y, [xa, wa], dy.half())
    y = y.detach()
    (ye, dxe, dwe), (ay, adx, adw) = split_exact(x, w, dy, 1, (0,) + pad, groups, torch.float16)
    assert_exact(y, ye, ay, torch.float16, 1.0, 'conv2d fprop')
    assert_exact(dx, dxe, adx, torch.float16, 1.0, 'conv2d dgrad')
    assert_exact(dw, dwe, adw, torch.float16, 1.0, 'conv2d wgrad')


# (the fused modulated convolution: tests/test_gpu_modconv_exact.py)


# ---- fp32 streaming kernels: pointwise 1x1x1 forward / input gradient (the weight gradient of these shapes: the engine),
# depthwise long FIR
@pytest.mark.parametrize('xs,ws', [((2, 3, 5, 16, 20), (32, 3, 1, 1, 1)), ((2, 64, 3, 36, 64), (3, 64, 1, 1, 1)), ((3, 16, 2, 6, 8), (24, 16, 1, 1, 1))])
def test_pointwise_kernels_and_engine_wgrad_exact(plug, xs, ws):
    assert all(plan_flags(plug, xs, ws, [0, 0, 0], 1, 1, torch.float32)), 'expected the streaming kernels'
    x, w = ints(xs, 61, 1, 0.5), ints(ws, 62, 2, 0.5)
    dy = ints((xs[0], ws[0]) + xs[2:], 63, 1, 0.5)
    y = plug.fprop(x.float(), w.float(), [0, 0, 0], 1)
    dx = plug.dgrad(dy.float(), w.float(), tuple(xs), [0, 0, 0], 1)
    dw = plug.wgrad(x.float(), dy.float(), tuple(ws), [0, 0, 0], 1)
    (ye, dxe, dwe), (ay, adx, adw) = split_exact(x, w, dy, 1, (0, 0, 0), 1, torch.float16)       # full products
    assert_exact(y, ye, ay, torch.float32, 1.0, 'pw_conv forward')
    assert_exact(dx, dxe, adx, torch.float32, 1.0, 'pw_conv input gradient')
    assert_exact(dw, dwe, adw, torch.float32, 1.0, 'engine weight gradient')


@pytest.mark.parametrize('lead', range(6))
def test_fir1d_depthwise_exact(plug, lead):
    n, g, k, lout = 3, 8, 40, 2100
    x = ints((n, g, lout + k - 1), 71, 1, 0.7)
    w = ints((g, 1, k), 72 + lead, 3, 0.8)
    w[:, :, :lead] = 0                                      # leading zero taps: the kernel starts at first & ~3
    w[:, :, lead] = torch.where(w[:, :, lead] == 0, torch.ones_like(w[:, :, lead]), w[:, :, lead])
    y = plug.fir1d_depthwise(x.float(), w.float())
    ye = F.conv1d(x, w, groups=g)
    assert_exact(y, ye, F.conv1d(x.abs(), w.abs(), groups=g), torch.float32, 1.0, f'fir1d lead {lead}')
