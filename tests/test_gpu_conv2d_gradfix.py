"""The wgmma implicit-GEMM convolution (conv2d_gradfix.conv2d -> conv_nd -> lvg_convnd_*) against torch's own convolution
evaluated in fp32 on the same fp16-rounded operands."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import oracle as orc
from torch_utils import custom_ops
from torch_utils.ops import conv2d_gradfix, conv2d_resample, conv_nd
from _common import assert_close, golden, cases, t

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOL = 2e-3          # fp16 output rounding (4.9e-4) + fp32 accumulation order; relative to max |ref|

CASES = [
    # (n, groups, cin, cout, h, w, k, pad)
    (1, 3, 27, 40, 29, 36, 3, 2),       # sres L0-like: cin not a multiple of 16, one m-tile
    (1, 2, 64, 200, 31, 38, 3, 2),      # two m-tiles, the second partial
    (1, 4, 155, 3, 20, 40, 1, 0),       # ToRGB 1x1
    (1, 2, 48, 128, 58, 86, 3, 2),      # two x tiles
    (3, 1, 32, 64, 16, 16, 3, 1),       # discriminator style: batch shares the weights, pad 1 (odd row start)
    (2, 2, 16, 16, 9, 7, 3, 0),         # tiny odd image, batch and groups
    (1, 1, 16, 128, 70, 150, 3, 1),     # several tiles in both directions
]


@pytest.mark.parametrize('n,g,cin,cout,h,w,k,pad', CASES)
def test_conv2d_forward_and_input_gradient(n, g, cin, cout, h, w, k, pad):
    gen = torch.Generator().manual_seed(n * 1000 + cin)
    x = torch.randn(n, g * cin, h, w, generator=gen).half().to(DEV).requires_grad_(True)
    wt = (torch.randn(g * cout, cin, k, k, generator=gen) / np.sqrt(cin * k * k)).half().to(DEV).requires_grad_(True)
    assert conv_nd._native_ok(x, wt, 1, pad, 1, g)
    y = conv2d_gradfix.conv2d(x, wt, padding=pad, groups=g)
    ref = F.conv2d(x.detach().float(), wt.detach().float(), padding=pad, groups=g)
    assert y.dtype == torch.float16 and y.shape == ref.shape
    assert_close(y, ref, TOL, 'fprop')
    dy = torch.randn(*y.shape, generator=gen).half().to(DEV)
    dx, dw = torch.autograd.grad(y, [x, wt], dy)
    xr, wr = x.detach().float().requires_grad_(True), wt.detach().float().requires_grad_(True)
    rdx, rdw = torch.autograd.grad(F.conv2d(xr, wr, padding=pad, groups=g), [xr, wr], dy.float())
    assert_close(dx, rdx, TOL, 'dgrad')
    assert_close(dw, rdw, 5e-3, 'wgrad')


def test_wgrad_modes_agree():
    # the native weight gradient against the ATen one on a ragged shape: odd width (no pixel pairs), partial last stage,
    # Cin not a multiple of 16, two n-tiles (Cin > 160), batch accumulation
    gen = torch.Generator().manual_seed(5)
    for (n, g, cin, cout, h, w, k, pad) in ((2, 1, 170, 130, 11, 71, 3, 1), (1, 2, 20, 24, 9, 131, 3, 2), (2, 3, 40, 8, 5, 6, 1, 0)):
        x = torch.randn(n, g * cin, h, w, generator=gen).half().to(DEV)
        dy = torch.randn(n, g * cout, h + 2 * pad - k + 1, w + 2 * pad - k + 1, generator=gen).half().to(DEV)
        dw = custom_ops.get_plugin('convnd_plugin').wgrad(x, dy, (g * cout, cin, k, k), (pad, pad), g)
        wr = torch.zeros(g * cout, cin, k, k, device=DEV, requires_grad=True)
        ref, = torch.autograd.grad(F.conv2d(x.float(), wr, padding=pad, groups=g), [wr], dy.float())
        assert_close(dw, ref, 5e-3, f'wgrad {(n, g, cin, cout, h, w, k, pad)}')


def test_conv2d_against_cpu_oracle():
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(1, 2 * 20, 13, 18, generator=gen).half()
    wt = (torch.randn(2 * 24, 20, 3, 3, generator=gen) / 13).half()
    y = conv2d_gradfix.conv2d(x.to(DEV), wt.to(DEV), padding=2, groups=2)
    assert_close(y, orc.conv2d(x.float().numpy(), wt.float().numpy(), padding=2, groups=2), TOL)


def test_conv2d_double_backward_matches_torch():
    # R1-style: gradient of |d y / d x|^2 with respect to the weights and dy
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(2, 16, 12, 12, generator=gen).half().to(DEV).requires_grad_(True)
    wt = (torch.randn(32, 16, 3, 3, generator=gen) / 12).half().to(DEV).requires_grad_(True)
    y = conv2d_gradfix.conv2d(x, wt, padding=1)
    gx, = torch.autograd.grad(y.float().square().sum(), [x], create_graph=True)
    gw, = torch.autograd.grad(gx.float().square().sum(), [wt])
    xr, wr = x.detach().float().requires_grad_(True), wt.detach().float().requires_grad_(True)
    yr = F.conv2d(xr, wr, padding=1)
    gxr, = torch.autograd.grad(yr.square().sum(), [xr], create_graph=True)
    gwr, = torch.autograd.grad(gxr.square().sum(), [wr])
    assert_close(gx, gxr, 5e-3, 'first order')
    assert_close(gw, gwr, 2e-2, 'second order')


def test_engine_takes_fp32_and_strides_and_leaves_dilation_to_torch():
    x = torch.randn(1, 8, 16, 16, device=DEV)
    w = torch.randn(8, 8, 3, 3, device=DEV)
    xh, wh = x.half(), w.half()
    # the TMA-fed engine behind conv2d_gradfix.conv2d takes fp32 (bf16 hi/lo split) and strides ...
    torch.backends.cudnn.allow_tf32 = False
    y = conv2d_gradfix.conv2d(x, w, padding=1)
    r = F.conv2d(x.double(), w.double(), padding=1)
    assert not torch.equal(y, F.conv2d(x, w, padding=1)) and float((y.double() - r).abs().max()) <= 1e-4 * float(r.abs().max())
    ys = conv2d_gradfix.conv2d(xh, wh, stride=2, padding=1)
    assert float((ys.double() - F.conv2d(xh.double(), wh.double(), stride=2, padding=1)).abs().max()) <= 3e-3 * float(r.abs().max())
    # ... and leaves dilation to the library, bit for bit
    assert torch.equal(conv2d_gradfix.conv2d(x, w, padding=2, dilation=2), F.conv2d(x, w, padding=2, dilation=2))


_CV = golden('conv')


@pytest.mark.parametrize('name', ['plain_3x3', 'fromrgb_1x1', 'grouped_mod'])
def test_conv2d_resample_fp16_through_native_conv(name):
    xs, ws, kw, has_f = cases(_CV)[name]
    x, w = t(_CV[f'{name}/x'], DEV, torch.float16), t(_CV[f'{name}/w'], DEV, torch.float16)
    y = conv2d_resample.conv2d_resample(x, w, **kw)
    ref = conv2d_resample.conv2d_resample(x.float().cpu(), w.float().cpu(), **kw)
    assert_close(y, ref, 3e-3, name)


@pytest.mark.parametrize('cin', [256, 512])
def test_wgrad_1x1_wide_input_channels(cin):
    # ADVICE r1: 1x1 kernels with more than 160 input channels per n-tile left B rows 160.. unstaged
    g, cout, h, w = 1, 64, 12, 20
    x = (torch.randn(1, g * cin, h, w, device=DEV) / 4).half()
    dy = torch.randn(1, g * cout, h, w, device=DEV).half()
    dw = custom_ops.get_plugin('convnd_plugin').wgrad(x, dy, (g * cout, cin, 1, 1), (0, 0), g)
    ref = torch.einsum('nohw,nihw->oi', dy.float(), x.float())[:, :, None, None]
    assert_close(dw, ref, 5e-3, 'dw')
