"""Bit-exact checks of the forward / input-gradient kernel's epilogue (csrc/conv_igemm.cu): the column map that places each
accumulator column, the paired 8-byte fp32 / 4-byte half2 stores and the one-element stores, on shapes on both sides of
the pair selection (`lvg_convnd_epilogue_plan` reports which one a shape takes).

Operands are sparse small integers (and, for the fp32 split path, dyadic values with a non-zero bf16 lo half), as in
tests/test_gpu_conv_exact.py, so the kernel must equal the float64 reference bit for bit. Every output is written into
the middle of a NaN-filled guard buffer: an element the kernel misses stays NaN, and a store past either end changes a
guard byte. The same call is repeated with y one element off the pair alignment, which must take the one-element stores
and give the same bits."""
import ctypes

import pytest
import torch

from torch_utils import custom_ops
from test_gpu_conv_exact import conv5, ints, dyadic, lo_half, first_mismatch

pytestmark = pytest.mark.gpu
DEV = 'cuda'
GUARD = 64                      # elements of NaN on each side of the output


@pytest.fixture(scope='module')
def plug():
    return custom_ops.get_plugin('convnd_plugin')


def epilogue_plan(plug, mode, args, stride):
    out = (ctypes.c_int * 4)()
    assert plug._lib.lvg_convnd_epilogue_plan(mode, *args, stride, out, 4) == 0, plug._lib.lvg_last_error().decode()
    return list(out)


class Guarded:
    """An output tensor at element `offset` past a 16-byte aligned start inside a NaN-filled buffer."""

    def __init__(self, shape, dtype, offset):
        n = 1
        for s in shape:
            n *= s
        self.buf = torch.full((GUARD + offset + n + GUARD,), float('nan'), dtype=dtype, device=DEV)
        self.lo, self.n = GUARD + offset, n
        self.t = self.buf[self.lo:self.lo + n].view(shape)
        self.before = self.buf.clone()

    def check(self, what):
        es = self.buf.element_size()
        raw, ref = self.buf.view(torch.uint8), self.before.view(torch.uint8)
        lo, hi = self.lo * es, (self.lo + self.n) * es
        assert torch.equal(raw[:lo], ref[:lo]) and torch.equal(raw[hi:], ref[hi:]), f'{what}: a guard element was written'


def operands(xs, ws, dys, dtype, dyad, seed):
    make = dyadic if dyad else ints
    x, w, dy = make(xs, seed + 1, 1, 0.4), make(ws, seed + 2, 2, 0.4), make(dys, seed + 3, 1, 0.4)
    return [v.to(dtype).double() for v in (x, w, dy)]


def expected(x, w, stride, pad, groups, dtype, dyad):
    y = conv5(x, w, stride, pad, groups)
    if dtype == torch.float32 and dyad:
        y = y - conv5(lo_half(x), lo_half(w), stride, pad, groups)
    return y


def assert_bits(got, exp, what):
    assert torch.equal(exp.to(got.dtype).double(), exp), f'{what}: precondition: the exact result is not representable'
    assert torch.equal(got, exp.to(got.dtype)), f'{what}: ' + first_mismatch(got, exp, 1.0)


def fprop_into(plug, x, w, pad, groups, stride, offset, bias=None, act=0, alpha=0.25, gain=1.0, clamp=-1.0):
    nd = x.ndim - 2
    a, sp, k, p = plug._args(tuple(x.shape), tuple(w.shape), list(pad[3 - nd:]), groups, x.dtype)
    st3 = [1, stride, stride] if nd >= 2 else [1, 1, 1]
    osp = [(s + 2 * q - kk) // t + 1 for s, q, kk, t in zip(sp, p, k, st3)][3 - nd:]
    y = Guarded([x.shape[0], w.shape[0]] + osp, x.dtype, offset)
    ws = custom_ops._workspace(x.device, plug._lib.lvg_convnd_workspace(*a))
    P = custom_ops._ptr
    rc = plug._lib.lvg_convnd_fprop(P(x), P(w), P(y.t), *a, int(stride), P(bias), int(act), float(alpha), float(gain), float(clamp), P(ws),
                                    ws.numel(), custom_ops._stream(x))
    assert rc == 0, plug._lib.lvg_last_error().decode()
    torch.cuda.synchronize()
    return y, a


def dgrad_into(plug, dy, w, xs, pad, groups, stride, offset):
    nd = dy.ndim - 2
    a, _, _, _ = plug._args(tuple(xs), tuple(w.shape), list(pad[3 - nd:]), groups, dy.dtype)
    dx = Guarded(list(xs), dy.dtype, offset)
    ws = custom_ops._workspace(dy.device, plug._lib.lvg_convnd_workspace(*a))
    P = custom_ops._ptr
    rc = plug._lib.lvg_convnd_dgrad(P(dy), P(w), P(dx.t), *a, int(stride), P(ws), ws.numel(), custom_ops._stream(dy))
    assert rc == 0, plug._lib.lvg_last_error().decode()
    torch.cuda.synchronize()
    return dx


# (x shape, w shape, padding (t, h, w), stride, groups): 64-row mode, one full m-tile, several m-tiles, cout 3 and 45, groups,
# tiles clipped in t (several frames per tile), h and w (column tiles), an output row of 16 bytes (wo = 4 fp32 / 8 fp16),
# odd widths (one-element stores), strided calls
CASES = [
    ((2, 32, 3, 18, 40), (32, 32, 1, 3, 3), (0, 1, 1), 1, 1),        # 64-row mode, even widths
    ((2, 24, 5, 7, 9), (45, 24, 1, 3, 3), (0, 1, 1), 1, 1),          # 64-row mode, cout 45, odd widths, frames per tile
    ((1, 16, 9, 5, 8), (3, 16, 3, 3, 3), (1, 1, 1), 1, 1),           # cout 3, several frames per tile clipped in t
    ((2, 40, 1, 37, 60), (128, 40, 1, 3, 3), (0, 1, 1), 1, 1),       # one full m-tile, row tiles clipped in h
    ((1, 48, 2, 9, 250), (200, 48, 1, 3, 3), (0, 1, 1), 1, 1),       # two m-tiles, column tiles clipped in w
    ((2, 3 * 16, 4, 6, 10), (3 * 20, 16, 1, 3, 3), (0, 1, 1), 1, 3), # groups
    ((1, 24, 3, 5, 4), (40, 24, 1, 3, 3), (0, 1, 1), 1, 1),          # wo = 4: 16-byte fp32 rows
    ((1, 24, 3, 5, 8), (40, 24, 1, 3, 3), (0, 1, 1), 1, 1),          # wo = 8: 16-byte fp16 rows
    ((2, 16, 21, 66), (24, 16, 3, 3), (0, 1, 1), 2, 1),              # strided
    ((1, 16, 30, 100), (70, 16, 3, 3), (0, 1, 1), 3, 1),             # strided, column tiles
]


def case_id(c):
    xs, ws, pad, stride, groups = c
    return f"x{'x'.join(map(str, xs[1:]))}-k{'x'.join(map(str, ws[2:]))}-s{stride}-g{groups}"


@pytest.mark.parametrize('dtype,dyad', [(torch.float16, False), (torch.float32, True)], ids=['f16', 'f32split-dyadic'])
@pytest.mark.parametrize('case', CASES, ids=[case_id(c) for c in CASES])
def test_epilogue_paths_exact(plug, case, dtype, dyad):
    xs, ws, pad, stride, groups = case
    nd = len(xs) - 2
    ys = (xs[0],) + tuple(conv5(torch.zeros(1, *xs[1:], device=DEV, dtype=torch.float64),
                                torch.zeros(*ws, device=DEV, dtype=torch.float64), stride, pad, groups).shape[1:])
    x, w, dy = operands(xs, ws, ys, dtype, dyad, seed=len(xs) * 10 + ws[0])
    y_exp = expected(x, w, stride, pad, groups, dtype, dyad)
    for offset in (0, 1):                                         # 1: y off the pair alignment
        y, a = fprop_into(plug, x.to(dtype), w.to(dtype), pad, groups, stride, offset)
        y.check('forward')
        assert_bits(y.t, y_exp, f'forward, y offset {offset}')
    if stride == 1:
        # split: the kernel sums hi*hi + hi*lo + lo*hi of (dy, w), the full input gradient minus the lo*lo one
        xr = x.clone().requires_grad_(True)
        yr = conv5(xr, w, stride, pad, groups)
        (gx,) = torch.autograd.grad(yr, [xr], dy)
        if dtype == torch.float32 and dyad:
            xl = torch.zeros_like(x).requires_grad_(True)
            yl = conv5(xl, lo_half(w), stride, pad, groups)
            (gl,) = torch.autograd.grad(yl, [xl], lo_half(dy))
            gx = gx - gl
        for offset in (0, 1):
            dx = dgrad_into(plug, dy.to(dtype), w.to(dtype), xs, pad, groups, stride, offset)
            dx.check('input gradient')
            assert_bits(dx.t, gx, f'input gradient, dx offset {offset}')


def test_pair_selection_covered(plug):
    """The cases above include shapes on both sides of the pair selection, forward and input gradient."""
    seen = set()
    for xs, ws, pad, stride, groups in CASES:
        for dtype in (torch.float16, torch.float32):
            a, _, _, _ = plug._args(tuple(xs), tuple(ws), list(pad[3 - (len(xs) - 2):]), groups, dtype)
            seen.add(('fprop', epilogue_plan(plug, 0, a, stride)[0]))
            if stride == 1:
                seen.add(('dgrad', epilogue_plan(plug, 1, a, 1)[0]))
    assert seen >= {('fprop', 0), ('fprop', 1), ('dgrad', 0), ('dgrad', 1)}, seen


# ---- [bias, act, gain, clamp] on both store paths: integer bias, lrelu alpha 0.25, gain 2 or 0.5, integer clamp
@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
@pytest.mark.parametrize('act,gain,clamp', [(0, 1.0, -1.0), (1, 2.0, -1.0), (2, 0.5, 6.0), (2, 2.0, -1.0), (1, 0.5, 3.0), (1, 1.0, 0.0)])
def test_epilogue_act_exact(plug, act, gain, clamp, dtype):
    for case in (CASES[0], CASES[1], CASES[4], CASES[8]):
        xs, ws, pad, stride, groups = case
        nd = len(xs) - 2
        x, w = ints(xs, 81, 1, 0.3), ints(ws, 82, 2, 0.3)
        b = ints((ws[0],), 83, 5, 1.0)
        z = conv5(x, w, stride, pad, groups)
        if act:
            z = z + b.view([1, -1] + [1] * nd)
            if act == 2:
                z = torch.where(z < 0, z * 0.25, z)
            z = z * gain
            if clamp >= 0:
                z = z.clamp(-clamp, clamp)
        for offset in (0, 1):
            y, _ = fprop_into(plug, x.to(dtype), w.to(dtype), pad, groups, stride, offset, bias=b.float(), act=act, alpha=0.25, gain=gain,
                              clamp=clamp)
            y.check('forward')
            assert_bits(y.t, z, f'act {act} gain {gain} clamp {clamp} {case_id(case)} offset {offset}')


# ---- the output scale of the modulated convolution (out_scale on the accumulator), paired and one-element stores
@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
@pytest.mark.parametrize('xs,ws,pad', [((2, 32, 3, 10, 16), (32, 32, 1, 3, 3), (0, 1, 1)), ((2, 24, 4, 5, 7), (45, 24, 1, 3, 3), (0, 1, 1)),
                                       ((1, 16, 12, 30), (140, 16, 3, 3), (0, 1, 1))])
def test_epilogue_out_scale_exact(plug, xs, ws, pad, dtype):
    nd = len(xs) - 2
    x, w = ints(xs, 91, 1, 0.4), ints(ws, 92, 2, 0.4)
    t = xs[2] if nd == 3 else 1
    g = torch.Generator(device=DEV).manual_seed(93)
    a = torch.randint(1, 3, (xs[0], xs[1], t), generator=g, device=DEV).double()
    ys = conv5(torch.zeros(1, *xs[1:], device=DEV, dtype=torch.float64), torch.zeros(*ws, device=DEV, dtype=torch.float64), 1, pad, 1).shape
    to = ys[2] if nd == 3 else 1
    d = torch.randint(0, 3, (xs[0], ws[0], to), generator=g, device=DEV).double() * 0.5
    xa = x * (a.view(xs[0], xs[1], t, 1, 1) if nd == 3 else a.view(xs[0], xs[1], 1, 1))
    z = conv5(xa, w, 1, pad, 1) * (d.view(xs[0], ws[0], to, 1, 1) if nd == 3 else d.view(xs[0], ws[0], 1, 1))
    y = plug.modconv_fprop(x.to(dtype), w.to(dtype), a.float(), d.float(), list(pad[3 - nd:]))
    torch.cuda.synchronize()
    assert_bits(y, z, 'modconv forward')
