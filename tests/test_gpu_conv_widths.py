"""Every MMA width of the convolution engine (csrc/conv_igemm.cu) against torch in float64, at the tolerances of
test_gpu_convnd.py: the forward / input-gradient kernel at N = 16, 32, ..., 256 columns per consumer warpgroup (128-row
images) and N = 16, ..., 128 in 64-row mode (GEMMs with at most 64 rows), the weight-gradient kernel at every (taps per
CTA, NT) pair it is instantiated for, and the 64-row mode through the modulated convolution's input and output factors.
Each case first checks, with the library's own plan, that it runs the width it is named for."""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from torch_utils import custom_ops

pytestmark = pytest.mark.gpu
DEV = 'cuda'
DTYPES = [torch.float16, torch.float32]
DT_IDS = ['f16', 'f32split']


@pytest.fixture(scope='module')
def plug():
    return custom_ops.get_plugin('convnd_plugin')


def rnd(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV, dtype=torch.float64) * scale


def tol_of(dtype):
    return 2e-3 if dtype == torch.float16 else 5e-5


def fwd_plan(plug, mode, xs, ws, pad, dtype):
    args, _, _, _ = plug._args(tuple(xs), tuple(ws), pad, 1, dtype)
    out = (ctypes.c_int * 48)()
    assert plug._lib.lvg_convnd_plan(mode, *args, 1, out, 48) == 0
    return out[38], out[39]                                   # 64-row mode, MMA width per consumer warpgroup


def check_conv(plug, xs, ws, pad, dtype):
    fan = math.prod(ws[1:])
    x, w = rnd(xs, 1).to(dtype), rnd(ws, 2, 1.0 / math.sqrt(fan)).to(dtype)
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yr = F.conv3d(xr, wr, padding=pad)
    tol = tol_of(dtype)
    y = plug.fprop(x, w, pad, 1)
    assert float((y.double() - yr.detach()).abs().max()) <= tol * float(yr.detach().abs().max()), 'fprop'
    dy = rnd(tuple(yr.shape), 3).to(dtype)
    gx, gw = torch.autograd.grad(yr, [xr, wr], dy.double())
    dx = plug.dgrad(dy, w, tuple(xs), pad, 1)
    assert float((dx.double() - gx).abs().max()) <= tol * float(gx.abs().max()), 'dgrad'
    dw = plug.wgrad(x, dy, tuple(ws), pad, 1)
    assert float((dw.double() - gw).abs().max()) <= tol * float(gw.abs().max()), 'wgrad'


# 3x3 kernels over 14-pixel rows: a tile row is 16 accumulator columns, so H rows give N = 16 H columns
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('width', range(16, 257, 16))
def test_forward_and_input_gradient_width_128_rows(plug, width, dtype):
    xs, ws, pad = (2, 80, 1, width // 16, 14), (80, 80, 1, 3, 3), (0, 1, 1)
    for mode in (0, 1):
        assert fwd_plan(plug, mode, xs, ws, pad, dtype) == (0, width)
    check_conv(plug, xs, ws, pad, dtype)


# 64-row mode: the two warpgroups take N columns each of a 2 N-column tile (fprop M = 40, dgrad M = 24)
@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('width', range(16, 129, 16))
def test_forward_and_input_gradient_width_64_rows(plug, width, dtype):
    xs, ws, pad = (2, 24, 1, width // 8, 14), (40, 24, 1, 3, 3), (0, 1, 1)
    for mode in (0, 1):
        assert fwd_plan(plug, mode, xs, ws, pad, dtype) == (1, width)
    check_conv(plug, xs, ws, pad, dtype)


def test_64_row_mode_odd_tile(plug):
    # 5 rows of 16 columns: 80 columns, 48 per warpgroup -- the second one's last 16 columns lie past the tile
    xs, ws, pad = (2, 16, 1, 5, 14), (3, 16, 1, 3, 3), (0, 1, 1)
    assert fwd_plan(plug, 0, xs, ws, pad, torch.float32) == (1, 48)
    check_conv(plug, xs, ws, pad, torch.float32)


# (taps per CTA, NT) -> kernel, cin, env: kh = 1 or cin > 32 keeps the tap rows apart (taps = kw); kh > 1 with
# cin <= 32 folds them (taps = kh * kw); LVG_WGRAD_FOLD_CIN widens the folding to 64 input channels
WGRAD_PAIRS = [((1, nt), (2, 1, 1), nt, None) for nt in range(32, 257, 32)] + \
              [((2, nt), (1, 1, 2), nt, None) for nt in range(32, 129, 32)] + \
              [((3, 32), (1, 1, 3), 32, None), ((3, 64), (1, 1, 3), 64, None),
               ((4, 32), (1, 2, 2), 32, None), ((4, 64), (1, 2, 2), 64, '64'),
               ((5, 32), (1, 5, 1), 32, None), ((6, 32), (1, 3, 2), 32, None), ((7, 32), (1, 7, 1), 32, None), ((8, 32), (1, 4, 2), 32, None)]


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('pair,k3,cin,fold_cin', WGRAD_PAIRS, ids=[f'taps{p[0][0]}_nt{p[0][1]}' for p in WGRAD_PAIRS])
def test_weight_gradient_pair(plug, monkeypatch, pair, k3, cin, fold_cin, dtype):
    if dtype == torch.float32 and pair[1] > 128:
        pytest.skip('split operands cap NT at 128')
    if fold_cin:
        monkeypatch.setenv('LVG_WGRAD_FOLD_CIN', fold_cin)
    xs, ws = (2, cin, 3, 9, 10), (48, cin) + k3
    pad = tuple(k // 2 for k in k3)
    args, _, _, _ = plug._args(xs, ws, pad, 1, dtype)
    out = (ctypes.c_int * 32)()
    assert plug._lib.lvg_convnd_wgrad_plan(*args, out, 32) == 0
    assert (out[8] * k3[2], out[3]) == pair
    x = rnd(xs, 4).to(dtype)
    xr = x.double()
    w = rnd(ws, 5, 1.0 / math.sqrt(math.prod(ws[1:]))).double().requires_grad_(True)
    yr = F.conv3d(xr, w, padding=pad)
    dy = rnd(tuple(yr.shape), 6).to(dtype)
    gw, = torch.autograd.grad(yr, [w], dy.double())
    dw = plug.wgrad(x, dy, ws, pad, 1)
    assert float((dw.double() - gw).abs().max()) <= tol_of(dtype) * float(gw.abs().max())


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('cout', [3, 32, 64])
def test_modulated_forward_64_row_mode(plug, cout, dtype):
    n, cin, k3, pad = 2, 24, (3, 3, 3), (1, 1, 1)
    xs, ws = (n, cin, 5, 9, 16), (cout, cin) + k3
    assert fwd_plan(plug, 0, xs, ws, pad, dtype)[0] == 1
    x = rnd(xs, 7).to(dtype)
    w = rnd(ws, 8, 1.0 / math.sqrt(cin * 27)).to(dtype)
    a = (rnd((n, cin, xs[2]), 9).abs() + 0.5).float()
    d = (rnd((n, cout, xs[2]), 10).abs() + 0.5).float()
    y = plug.modconv_fprop(x, w, a, d, pad)
    xa = (x.double() * a.double()[..., None, None]).to(dtype).double()     # the kernel rounds a * x to the operand type
    yr = F.conv3d(xa, w.double(), padding=pad) * d.double()[..., None, None]
    assert float((y.double() - yr).abs().max()) <= tol_of(dtype) * float(yr.abs().max())
