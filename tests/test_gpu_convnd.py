"""The TMA-fed wgmma implicit-GEMM convolution engine (csrc/conv_igemm.cu) through the C ABI, against torch's own
convolutions in float64 on the same inputs: 1-D / 2-D / 3-D, fp16 and fp32 (bf16 hi/lo split), forward with and
without the fused bias_act epilogue, input gradient, weight gradient (with and without split-K, one and two column
segments). Shapes follow the call sites: conv2d_gradfix.py:37-45 (generator_sres.py:63-65, conv2d_resample.py:29-41),
generator_lres.py:119,578, discriminator_lres.py:121,172."""
import math

import pytest
import torch
import torch.nn.functional as F

from torch_utils import custom_ops

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.fixture(scope='module')
def plug():
    return custom_ops.get_plugin('convnd_plugin')


def rnd(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, generator=g, device=DEV, dtype=torch.float64) * scale


def conv_ref(x, w, padding, groups):
    nd = x.ndim - 2
    return (F.conv1d, F.conv2d, F.conv3d)[nd - 1](x, w, padding=padding, groups=groups)


CASES = [
    # name, x shape, w shape, padding, groups
    ('2d modulated 3x3 pad2 ragged', (1, 4 * 24, 20, 26), (4 * 40, 24, 3, 3), (2, 2), 4),
    ('2d 1x1', (3, 40, 17, 23), (24, 40, 1, 1), (0, 0), 1),
    ('2d 3x3 pad1 batch', (3, 64, 33, 40), (130, 64, 3, 3), (1, 1), 1),
    ('2d wide row 150', (1, 2 * 27, 10, 148), (2 * 72, 27, 3, 3), (2, 2), 2),
    ('2d two column tiles 278', (1, 16, 7, 276), (24, 16, 3, 3), (2, 2), 1),
    ('2d tiny 4x4', (2, 32, 4, 4), (32, 32, 3, 3), (1, 1), 1),
    ('2d many k-steps', (1, 539, 12, 20), (130, 539, 3, 3), (2, 2), 1),
    ('3d 3x3x3', (2, 32, 6, 9, 16), (48, 32, 3, 3, 3), (1, 1, 1), 1),
    ('3d 1x3x3', (1, 24, 5, 18, 32), (20, 24, 1, 3, 3), (0, 1, 1), 1),
    ('3d 5x3x3', (1, 16, 9, 8, 8), (24, 16, 5, 3, 3), (2, 1, 1), 1),
    ('3d 1x1x1', (2, 48, 4, 5, 8), (136, 48, 1, 1, 1), (0, 0, 0), 1),
    ('3d 3x3x3 3x4 image', (2, 40, 7, 3, 4), (40, 40, 3, 3, 3), (1, 1, 1), 1),
    ('1d k3', (2, 64, 16), (32, 64, 3), (1,), 1),
    ('1d k1', (3, 200, 16), (50, 200, 1), (0,), 1),
    # few channels, 1x1x1, fp32: the streaming SIMT kernels of csrc/conv_pointwise.cu (fp16 / more channels: the engine)
    ('3d 1x1x1 pointwise 3->32', (2, 3, 5, 16, 20), (32, 3, 1, 1, 1), (0, 0, 0), 1),
    ('3d 1x1x1 pointwise 64->3', (2, 64, 3, 36, 64), (3, 64, 1, 1, 1), (0, 0, 0), 1),
    ('3d 1x1x1 pointwise 64->64', (2, 64, 7, 18, 30), (64, 64, 1, 1, 1), (0, 0, 0), 1),
    ('3d 1x1x1 pointwise 61->128 ragged', (3, 61, 3, 9, 12), (128, 61, 1, 1, 1), (0, 0, 0), 1),
    ('3d 1x1x1 pointwise 128->33', (1, 128, 2, 10, 14), (33, 128, 1, 1, 1), (0, 0, 0), 1),
    ('2d 1x1 pointwise 5->7 tiny', (4, 5, 2, 2), (7, 5, 1, 1), (0, 0), 1),
]


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
@pytest.mark.parametrize('name,xs,ws,pad,groups', CASES, ids=[c[0] for c in CASES])
def test_convnd_forward_and_gradients(plug, name, xs, ws, pad, groups, dtype):
    fan = math.prod(ws[1:])
    x64, w64 = rnd(xs, 1), rnd(ws, 2, 1.0 / math.sqrt(fan))
    x, w = x64.to(dtype), w64.to(dtype)
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)     # the reference sees the rounded operands
    yr = conv_ref(xr, wr, pad, groups)
    assert plug.supported(x, w, 1, pad, 1, groups)
    y = plug.fprop(x, w, pad, groups)
    assert y.shape == yr.shape and y.dtype == dtype
    tol = 2e-3 if dtype == torch.float16 else 5e-5          # fp16: result rounding; split fp32: ~2^-16 per product
    scale = float(yr.detach().abs().max())
    assert float((y.double() - yr).abs().max()) <= tol * scale, f'fprop {float((y.double() - yr).abs().max()) / scale:.3e}'
    dy64 = rnd(tuple(yr.shape), 3)
    dy = dy64.to(dtype)
    gx, gw = torch.autograd.grad(yr, [xr, wr], dy.double())
    dx = plug.dgrad(dy, w, tuple(x.shape), pad, groups)
    assert float((dx.double() - gx).abs().max()) <= tol * float(gx.abs().max()), f'dgrad {float((dx.double() - gx).abs().max() / gx.abs().max()):.3e}'
    dw = plug.wgrad(x, dy, tuple(w.shape), pad, groups)
    assert dw.shape == w.shape and dw.dtype == dtype
    assert float((dw.double() - gw).abs().max()) <= tol * float(gw.abs().max()), f'wgrad {float((dw.double() - gw).abs().max() / gw.abs().max()):.3e}'


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32])
def test_convnd_fused_bias_act_epilogue(plug, dtype):
    x, w, b = rnd((2, 24, 6, 9, 16), 4).to(dtype), rnd((40, 24, 3, 3, 3), 5, 0.05).to(dtype), rnd((40,), 6).float()
    for act, alpha, gain, clamp in ((2, 0.2, math.sqrt(2), 0.8), (1, 0.0, 1.0, 256.0), (2, 0.2, 1.0, -1.0)):
        y = plug.fprop(x, w, (1, 1, 1), 1, bias=b, act=act, alpha=alpha, gain=gain, clamp=clamp)
        r = F.conv3d(x.double(), w.double(), padding=1) + b.double().view(1, -1, 1, 1, 1)
        if act == 2:
            r = F.leaky_relu(r, alpha)
        r = r * gain
        if clamp >= 0:
            r = r.clamp(-clamp, clamp)
        tol = 2e-3 if dtype == torch.float16 else 5e-5
        assert float((y.double() - r).abs().max()) <= tol * float(r.abs().max())


STRIDED = [
    ('3x3 s2 pad0 (conv2d_resample down path)', (2, 32, 35, 42), (48, 32, 3, 3), 0, 2, 1),
    ('3x3 s2 pad1 even', (3, 24, 32, 32), (40, 24, 3, 3), 1, 2, 1),
    ('1x1 s2', (2, 64, 31, 17), (24, 64, 1, 1), 0, 2, 1),
    ('3x3 s2 wide, row tiles', (1, 16, 40, 300), (16, 16, 3, 3), 1, 2, 1),
    ('3x3 s2 grouped', (1, 3 * 16, 21, 22), (3 * 24, 16, 3, 3), 1, 2, 3),
]


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
@pytest.mark.parametrize('name,xs,ws,pad,stride,groups', STRIDED, ids=[c[0] for c in STRIDED])
def test_convnd_strided(plug, name, xs, ws, pad, stride, groups, dtype):
    fan = math.prod(ws[1:])
    x, w = rnd(xs, 11).to(dtype), rnd(ws, 12, 1.0 / math.sqrt(fan)).to(dtype)
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yr = F.conv2d(xr, wr, stride=stride, padding=pad, groups=groups)
    assert plug.supported(x, w, stride, pad, 1, groups)
    tol = 2e-3 if dtype == torch.float16 else 5e-5
    y = plug.fprop(x, w, (pad, pad), groups, stride=stride)
    assert y.shape == yr.shape
    assert float((y.double() - yr).abs().max()) <= tol * float(yr.detach().abs().max()), 'fprop'
    dy = rnd(tuple(yr.shape), 13).to(dtype)
    gx, gw = torch.autograd.grad(yr, [xr, wr], dy.double())
    dx = plug.dgrad(dy, w, tuple(x.shape), (pad, pad), groups, stride=stride)
    assert float((dx.double() - gx).abs().max()) <= tol * float(gx.abs().max()), 'dgrad'
    dw = plug.wgrad(x, dy, tuple(w.shape), (pad, pad), groups, stride=stride)
    assert float((dw.double() - gw).abs().max()) <= tol * float(gw.abs().max()), 'wgrad'


def test_convnd_wgrad_split_k_matches_single_pass(plug):
    # one group, 16 samples: the pixel range is cut over the grid and the fp32 partial sums are folded by a second kernel
    x, dy = rnd((16, 32, 24, 24), 7).half(), rnd((16, 48, 24, 24), 8).half()
    dw = plug.wgrad(x, dy, (48, 32, 3, 3), (1, 1), 1)
    xr = x.double()
    wr = torch.zeros(48, 32, 3, 3, device=DEV, dtype=torch.float64, requires_grad=True)
    gw, = torch.autograd.grad(F.conv2d(xr, wr, padding=1), [wr], dy.double())
    assert float((dw.double() - gw).abs().max()) <= 2e-3 * float(gw.abs().max())


def test_convnd_is_used_for_nan_free_padding(plug):
    # zero * garbage must not leak NaN from uninitialised shared memory or workspace tails into the result
    for _ in range(3):
        x, w = rnd((1, 17, 5, 6), 9).half(), rnd((19, 17, 3, 3), 10, 0.1).half()
        junk = torch.full((1 << 22,), float('nan'), device=DEV)
        del junk
        y = plug.fprop(x, w, (2, 2), 1)
        dw = plug.wgrad(x, torch.ones_like(y), (19, 17, 3, 3), (2, 2), 1)
        assert torch.isfinite(y).all() and torch.isfinite(dw).all()


def _trace_convs():
    import json
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    tr = json.load(open(os.path.join(root, 'workloads', 'lres_step.json')))
    seen, out = set(), []
    for key in ('lres_G', 'lres_D'):
        for c in tr[key]:
            if c['op'] in ('conv3d', 'conv1d') and c['groups'] == 1:
                sig = (tuple(c['x']), tuple(c['w']), str(c['padding']))
                if sig not in seen:
                    seen.add(sig)
                    out.append(c)
    return out


@pytest.mark.parametrize('c', _trace_convs(), ids=lambda c: f"{c['op']}-{'x'.join(map(str, c['x'][1:]))}-w{'x'.join(map(str, c['w']))}")
def test_every_lowres_convolution_signature(plug, c):
    # every F.conv3d / F.conv1d call of one G + D pass of the low-res networks (workloads/lres_step.json, recorded from the
    # reference modules), fp32, at batch 1 with the time axis cut to <= 24 frames: forward, input and weight gradient
    xs, ws = list(c['x']), list(c['w'])
    pad = c['padding'] if isinstance(c['padding'], (list, tuple)) else [c['padding']] * (len(xs) - 2)
    if len(xs) == 5 and xs[2] > 24:
        xs[2] = 24
    x = rnd(xs, 31).float()
    w = rnd(ws, 32, 1.0 / math.sqrt(math.prod(ws[1:]))).float()
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    yr = conv_ref(xr, wr, tuple(pad), 1)
    y = plug.fprop(x, w, tuple(pad), 1)
    # split-precision products are exact to ~2^-16; the tensor core's fp32 accumulation adds an error that grows with the
    # length of the sum (measured 6e-6 at K = 576 ... 7e-5 at K = 13824 products per output) -- still 15x inside 1e-3
    tol = 5e-5 if math.prod(ws[1:]) < 4096 else 2e-4
    assert float((y.double() - yr).abs().max()) <= tol * float(yr.detach().abs().max()), 'fprop'
    dy = rnd(tuple(yr.shape), 33).float()
    gx, gw = torch.autograd.grad(yr, [xr, wr], dy.double())
    dx = plug.dgrad(dy, w, tuple(xs), tuple(pad), 1)
    assert float((dx.double() - gx).abs().max()) <= tol * float(gx.abs().max()), 'dgrad'
    dw = plug.wgrad(x, dy, tuple(ws), tuple(pad), 1)
    assert float((dw.double() - gw).abs().max()) <= tol * float(gw.abs().max()), f'wgrad {float((dw.double() - gw).abs().max() / gw.abs().max()):.3e}'


# ---- weight gradient with few channels: folded tap rows (one CTA takes all ky) and the compact dy8 operand (cout < 128)

FEWCH = [
    # name, x shape, w shape, padding -- the low-res discriminator / generator layers at reduced extent, plus ragged ones
    ('D 32->32 1x3x3 64x64', (2, 32, 3, 64, 64), (32, 32, 1, 3, 3), (0, 1, 1)),
    ('D 32->64 1x3x3', (1, 32, 4, 40, 64), (64, 32, 1, 3, 3), (0, 1, 1)),
    ('D 64->64 5x3x3 (two n-tiles of 32)', (1, 64, 7, 32, 32), (64, 64, 5, 3, 3), (2, 1, 1)),
    ('D 64->128 5x3x3', (1, 64, 6, 16, 32), (128, 64, 5, 3, 3), (2, 1, 1)),
    ('G 64->64 1x3x3 36x64', (1, 64, 5, 36, 64), (64, 64, 1, 3, 3), (0, 1, 1)),
    ('48 channels (n-tile 48), odd rows, pitch 8 mod 16', (2, 48, 2, 9, 20), (40, 48, 1, 3, 3), (0, 1, 1)),
    ('8 -> 16 channels, tiny', (3, 8, 1, 5, 7), (16, 8, 1, 3, 3), (0, 1, 1)),
    ('3 -> 24 channels 3x3x3', (2, 3, 4, 12, 18), (24, 3, 3, 3, 3), (1, 1, 1)),
    ('27 channels, two column segments', (1, 27, 1, 6, 150), (72, 27, 1, 3, 3), (0, 2, 2)),
    ('3x1 kernel (kw 1)', (2, 32, 2, 16, 24), (32, 32, 1, 3, 1), (0, 1, 0)),
    ('no padding', (2, 16, 3, 14, 30), (20, 16, 3, 3, 3), (0, 0, 0)),
]


def _wgrad_ref(x, dy, ws, pad):
    wr = torch.zeros(*ws, device=DEV, dtype=torch.float64, requires_grad=True)
    gw, = torch.autograd.grad(F.conv3d(x.double(), wr, padding=pad), [wr], dy.double())
    return gw


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
@pytest.mark.parametrize('name,xs,ws,pad', FEWCH, ids=[c[0] for c in FEWCH])
def test_convnd_wgrad_few_channels_all_variants(plug, monkeypatch, name, xs, ws, pad, dtype):
    """Default (folded + compact), each switched off, both off: all four against float64 -- the knobs select different
    tilings of the same sums, so they also agree with each other to rounding."""
    x = rnd(xs, 21).to(dtype)
    ys = tuple(F.conv3d(torch.zeros(1, *xs[1:], device=DEV), torch.zeros(*ws, device=DEV), padding=pad).shape[1:])
    dy = rnd((xs[0],) + ys, 22).to(dtype)
    gw = _wgrad_ref(x, dy, ws, pad)
    tol = 2e-3 if dtype == torch.float16 else 5e-5
    monkeypatch.setenv('LVG_WGRAD_FOLD_CIN', '64')        # fold wherever the accumulators fit (default: up to 32 input channels)
    for fold, compact, m64 in ((1, 1, 1), (0, 1, 1), (1, 1, 0), (0, 1, 0), (1, 0, 0), (0, 0, 0)):
        monkeypatch.setenv('LVG_WGRAD_FOLD', str(fold))
        monkeypatch.setenv('LVG_WGRAD_COMPACT', str(compact))
        monkeypatch.setenv('LVG_WGRAD_M64', str(m64))          # 64-row MMAs where cout <= 64
        dw = plug.wgrad(x, dy, ws, pad, 1)
        err = float((dw.double() - gw).abs().max()) / float(gw.abs().max())
        assert err <= tol, f'fold={fold} compact={compact} m64={m64}: {err:.3e}'


BACKWARD = [
    ('3d 1x3x3 32->32', (2, 32, 3, 20, 32), (32, 32, 1, 3, 3), (0, 1, 1), 1, 1),
    ('3d 3x3x3 40->130 (two m-tiles, padded dy8: separate re-tiling)', (1, 40, 4, 6, 8), (130, 40, 3, 3, 3), (1, 1, 1), 1, 1),
    ('3d 3x3x3 64->128', (1, 64, 3, 9, 16), (128, 64, 3, 3, 3), (1, 1, 1), 1, 1),
    ('3d 1x1x1 pointwise 64->64 (streaming kernels)', (2, 64, 3, 8, 10), (64, 64, 1, 1, 1), (0, 0, 0), 1, 1),
    ('3d 1x1x1 256->128 (engine)', (1, 256, 2, 8, 16), (128, 256, 1, 1, 1), (0, 0, 0), 1, 1),
    ('2d modulated groups 4', (1, 4 * 24, 20, 26), (4 * 40, 24, 3, 3), (1, 1), 4, 1),
    ('2d stride 2', (2, 32, 35, 42), (48, 32, 3, 3), (0, 0), 1, 2),
    ('1d k3', (2, 64, 16), (32, 64, 3), (1,), 1, 1),
]


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
@pytest.mark.parametrize('name,xs,ws,pad,groups,stride', BACKWARD, ids=[c[0] for c in BACKWARD])
def test_convnd_backward_one_call_equals_the_two_gradients(plug, name, xs, ws, pad, groups, stride, dtype):
    """lvg_convnd_backward (dy re-tiled once) returns exactly what lvg_convnd_dgrad + lvg_convnd_wgrad return."""
    x, w = rnd(xs, 31).to(dtype), rnd(ws, 32, 1.0 / math.sqrt(math.prod(ws[1:]))).to(dtype)
    y = plug.fprop(x, w, pad, groups, stride=stride)
    dy = rnd(tuple(y.shape), 33).to(dtype)
    dx0 = plug.dgrad(dy, w, tuple(x.shape), pad, groups, stride=stride)
    dw0 = plug.wgrad(x, dy, tuple(w.shape), pad, groups, stride=stride)
    dx, dw = plug.backward(x, dy, w, pad, groups, stride=stride)
    assert torch.equal(dx, dx0) and torch.equal(dw, dw0)
    # and through autograd: a plain backward pass takes the fused call
    from torch_utils.ops import conv_nd
    xa, wa = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    nd = x.ndim - 2
    st = stride if nd == 2 else 1
    ya = (conv_nd.conv1d, conv_nd.conv2d, conv_nd.conv3d)[nd - 1](xa, wa, None, st, pad, 1, groups)
    ya.backward(dy)
    assert torch.equal(xa.grad, dx0) and torch.equal(wa.grad, dw0)


RESIDENT = [
    ('3d 1x3x3 32->32 (two k-steps = two slots)', (2, 32, 3, 40, 64), (32, 32, 1, 3, 3), (0, 1, 1)),
    ('3d 1x1x1 128->128 (k-chunks of four steps)', (1, 128, 4, 18, 32), (128, 128, 1, 1, 1), (0, 0, 0)),
    ('3d 1x3x3 16->24 (one slot period)', (1, 16, 3, 20, 24), (24, 16, 1, 3, 3), (0, 1, 1)),
    ('3d 3x3x3 16->16 (kt stages)', (1, 16, 5, 12, 16), (16, 16, 3, 3, 3), (1, 1, 1)),
    ('2d 3x3 64->64', (4, 64, 33, 40), (64, 64, 3, 3), (1, 1)),
]


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32], ids=['f16', 'f32split'])
@pytest.mark.parametrize('name,xs,ws,pad', RESIDENT, ids=[c[0] for c in RESIDENT])
def test_convnd_resident_weight_slots_change_nothing(plug, monkeypatch, name, xs, ws, pad, dtype):
    """Short K loops keep the weight images in their ring slots across tiles (LVG_CONV_RESIDENT_W, default on): same bits as
    re-fetching them per tile, and right against float64."""
    x, w = rnd(xs, 41).to(dtype), rnd(ws, 42, 1.0 / math.sqrt(math.prod(ws[1:]))).to(dtype)
    yr = conv_ref(x.double(), w.double(), pad, 1)
    out = {}
    for flag in ('1', '0'):
        monkeypatch.setenv('LVG_CONV_RESIDENT_W', flag)
        y = plug.fprop(x, w, pad, 1)
        dx = plug.dgrad(y, w, tuple(x.shape), pad, 1)
        out[flag] = (y, dx)
    tol = 2e-3 if dtype == torch.float16 else 5e-5
    assert float((out['1'][0].double() - yr).abs().max()) <= tol * float(yr.abs().max())
    assert torch.equal(out['1'][0], out['0'][0]) and torch.equal(out['1'][1], out['0'][1])


@pytest.mark.parametrize('xs,ws', [((2, 3, 5, 16, 20), (32, 3, 1, 1, 1)), ((2, 64, 3, 36, 64), (3, 64, 1, 1, 1)), ((3, 16, 2, 6, 8), (24, 16, 1, 1, 1))])
def test_pointwise_weight_gradient_both_paths(plug, xs, ws):
    """1x1x1 fp32 weight gradients of few-channel layers (the forward and input gradient take the streaming kernels, the
    weight gradient the engine) against float64, through both entry points that produce one: lvg_convnd_wgrad and the
    one-call lvg_convnd_backward."""
    x = rnd(xs, 51).float()
    dy = rnd((xs[0], ws[0]) + xs[2:], 52).float()
    gw = _wgrad_ref(x, dy, ws, (0, 0, 0))
    w = rnd(ws, 53).float()
    for path, dw in (('wgrad', plug.wgrad(x, dy, ws, (0, 0, 0), 1)), ('backward', plug.backward(x, dy, w, (0, 0, 0), 1)[1])):
        assert float((dw.double() - gw).abs().max()) <= 5e-5 * float(gw.abs().max()), path
