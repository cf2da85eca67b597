"""The first layer of the low-res generator's residual block as one op (torch_utils/ops/gblock_conv0.py,
lvg_gblock_conv0_* in csrc/gblock_conv0.cu) on the GPU: every conv_0 signature of the default generator (channels, kernel,
padding; frames and image sizes reduced) and an odd shape (40 channels, T = 1), in fp16 and fp32, with inputs scaled so that
some outputs clamp and some are negative.

Numerical contract:
- the forward against float64 of the same operands: integer x and w, power-of-two a and d, dyadic b, so that the
  convolution is exact and only the epilogue's fp32 arithmetic and the rounding to the layer dtype remain (one ulp);
- random operands against the composition modulated_conv + bias_act: within one rounding of the layer dtype (the fp16
  composition rounds d * conv before the bias, the op does not);
- the statistic against a float64 sum of the squares of y as stored, 1e-5 relative;
- dx, dw, da, dd and db against float64 on the op's own activation decisions, within 1e-4 of each tensor's largest
  magnitude in fp32 and 2^-9 in fp16 (dz d is rounded to fp16 when it is re-tiled), and in fp32 against the composition's
  gradients within 1e-4; two calls bitwise identical; create_graph second order; CUDA-graph capture; no host
  synchronisation.
The whole default G with modulated_conv, gblock_tail, lres_torgb and gblock_conv0 installed against the G without the
fused installs and the G with the three others, in the three modes, within test_gpu_lres_torgb.py's whole-G bounds.
"""
import os
import subprocess
import sys

import pytest
import torch

from torch_utils.ops import gblock_conv0 as gc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
DEV = torch.device('cuda')
F16, F32 = torch.float16, torch.float32
GAIN = 2 ** 0.5
_CACHE = {}

# (n, c, t, h, w, kernel, padding): the default G's conv_0 layers (512 / 256 channels 3x3x3, 256 / 128 / 64 channels 1x3x3)
# with fewer frames and smaller images, and an odd shape
SHAPES = [(2, 512, 4, 5, 6, (3, 3, 3), (1, 1, 1)), (2, 256, 4, 9, 16, (3, 3, 3), (1, 1, 1)),
          (2, 256, 3, 9, 16, (1, 3, 3), (0, 1, 1)), (2, 128, 3, 18, 32, (1, 3, 3), (0, 1, 1)),
          (2, 64, 2, 36, 64, (1, 3, 3), (0, 1, 1)), (3, 40, 1, 7, 9, (3, 3, 3), (1, 1, 1))]
IDS = ['c512k333', 'c256k333', 'c256k133', 'c128k133', 'c64k133', 'odd40']


def _run(mode, tmp_path_factory):
    if mode not in _CACHE:
        out = str(tmp_path_factory.mktemp('gblock_conv0') / f'{mode}.pt')
        env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]))
        r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'gblock_conv0_run.py'), out, mode], env=env, cwd=SRC,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
        assert r.returncode == 0, r.stdout[-3000:]
        _CACHE[mode] = torch.load(out, weights_only=False)
    return _CACHE[mode]


def _ulp(v, dtype):
    mant, tiny = (10, 2.0 ** -24) if dtype == F16 else (23, 2.0 ** -149)
    e = torch.floor(torch.log2(v.abs().clamp_min(tiny)))
    return torch.maximum(torch.exp2(e - mant), torch.full_like(v, tiny))


def _random(shape, dt, seed, scale):
    n, c, t, h, w, k, pad = shape
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.randn(n, c, t, h, w, generator=g, device=DEV) * scale).to(dt)
    wt = (torch.randn(c, c, *k, generator=g, device=DEV) / (c * k[0] * k[1] * k[2]) ** 0.5).to(dt)
    a = torch.rand(n, c, t, generator=g, device=DEV) + 0.5
    d = torch.rand(n, c, t, generator=g, device=DEV) + 0.5
    b = torch.randn(c, generator=g, device=DEV) * 0.5
    return x, wt, a, d, b.to(dt).float(), pad


@pytest.mark.parametrize('shape', SHAPES, ids=IDS)
@pytest.mark.parametrize('dt', [F16, F32], ids=['f16', 'f32'])
def test_forward_exact_operands_against_float64(shape, dt):
    n, c, t, h, w, k, pad = shape
    g = torch.Generator(device=DEV).manual_seed(1)
    x = torch.randint(-4, 5, (n, c, t, h, w), generator=g, device=DEV).to(dt)
    wt = torch.randint(-2, 3, (c, c, *k), generator=g, device=DEV).to(dt)
    a = 2.0 ** torch.randint(-1, 2, (n, c, t), generator=g, device=DEV).float()
    conv = torch.nn.functional.conv3d(x.double() * a.double()[..., None, None], wt.double(), padding=pad)
    # power-of-two d around 150 / std(conv): some outputs clamp at 256, some are small, half are negative
    e0 = round(float(torch.log2(150 / conv.std())))
    d = 2.0 ** (e0 + torch.randint(-3, 2, (n, c, t), generator=g, device=DEV).float())
    b = torch.randint(-64, 65, (c,), generator=g, device=DEV).float() / 8
    y = gc.gblock_conv0(x, wt, a, d, b, pad)
    assert y.dtype == dt and y.shape == x.shape
    u = conv * d.double()[..., None, None]
    z = u + b.double()[None, :, None, None, None]
    ref = (torch.where(z > 0, z, 0.2 * z) * GAIN).clamp(-256, 256)
    bound = _ulp(ref, dt) + 2.0 ** -21 * z.abs() * GAIN
    err = (y.double() - ref).abs()
    assert bool((err <= bound).all()), f'max err / bound {float((err / bound).max()):.3f}'
    assert bool((y.abs() == 256).any()) and bool((y < 0).any()) and bool((y.abs() < 256).any())


@pytest.mark.parametrize('shape', SHAPES, ids=IDS)
@pytest.mark.parametrize('dt', [F16, F32], ids=['f16', 'f32'])
def test_forward_and_statistic_against_the_composition(shape, dt):
    x, wt, a, d, b, pad = _random(shape, dt, 2, 150.0)
    y, sumsq = gc._plugin().fprop(x, wt, a, d, b, pad, 2, 0.2, GAIN, 256.0, want_sumsq=True)
    y2 = gc.gblock_conv0(x, wt, a, d, b, pad)
    assert torch.equal(y, y2)                                   # the statistic does not change y
    u = gc.modulated_conv.modulated_conv(x, wt, a, d, pad)
    ref = gc.composition(x, wt, a, d, b.to(dt), pad, 'lrelu', 256.0)
    bound = GAIN * _ulp(u.double(), dt) + 2 * _ulp(ref.double(), dt) + 2.0 ** -20 * (u.double().abs() + b.abs().double()[:, None, None, None])
    err = (y.double() - ref.double()).abs()
    assert bool((err <= bound).all()), f'max err / bound {float((err / bound).max()):.3f}'
    assert bool((y.abs() == 256).any()) and bool((y < 0).any())
    sq = y.double().square().sum()
    assert abs(float(sumsq) - float(sq)) <= 1e-5 * float(sq)


def _grads(fn, x, wt, a, d, b, dy):
    xs, ws, as_, ds, bs = (v.clone().requires_grad_(True) for v in (x, wt, a, d, b))
    y = fn(xs, ws, as_, ds, bs)
    y.backward(dy)
    return dict(x=xs.grad, w=ws.grad, a=as_.grad, d=ds.grad, b=bs.grad)


def _grads_float64(x, wt, a, d, y, dy, pad):
    """Gradients of y = clamp(lrelu(d conv(a x, w) + b) gain) in float64 from the op's own y: its activation and clamp
    decisions (bias_act's rule), the rounded operands x, w, a, d, dy."""
    yd = y.double()
    dz = dy.double() * torch.where(yd > 0, 1.0, 0.2) * GAIN * (yd.abs() < 256)
    x64, w64, a64, d64 = x.double(), wt.double(), a.double()[..., None, None], d.double()[..., None, None]
    dzd = dz * d64
    dxp = torch.nn.grad.conv3d_input(x.shape, w64, dzd, padding=pad)
    conv = torch.nn.functional.conv3d(x64 * a64, w64, padding=pad)
    return dict(x=dxp * a64, w=torch.nn.grad.conv3d_weight(x64 * a64, w64.shape, dzd, padding=pad), a=(dxp * x64).sum(dim=(3, 4)),
                d=(dz * conv).sum(dim=(3, 4)), b=dz.sum(dim=(0, 2, 3, 4)))


@pytest.mark.parametrize('shape', SHAPES, ids=IDS)
@pytest.mark.parametrize('dt', [F16, F32], ids=['f16', 'f32'])
def test_gradients_and_bitwise_repeatable(shape, dt):
    """dx, dw, da, dd, db: against float64 on the op's own activation decisions (fp16 and fp32), and against the
    composition's gradients (fp32: in fp16 the two paths' outputs round differently, so elements near 0 or the clamp take
    different activation branches)."""
    x, wt, a, d, b, pad = _random(shape, dt, 3, 60.0)
    dy = torch.randn(x.shape, generator=torch.Generator(device=DEV).manual_seed(4), device=DEV).to(dt)
    op = [_grads(lambda *v: gc.gblock_conv0(*v, pad), x, wt, a, d, b, dy) for _ in range(2)]
    y = gc.gblock_conv0(x, wt, a, d, b, pad)
    refs = [_grads_float64(x, wt, a, d, y, dy, pad)]
    if dt == F32:
        refs.append(_grads(lambda xs, ws, as_, ds, bs: gc.composition(xs, ws, as_, ds, bs, pad, 'lrelu', 256.0), x, wt, a, d, b, dy))
    tol = 1e-4 if dt == F32 else 2.0 ** -9
    for k in ('x', 'w', 'a', 'd', 'b'):
        assert torch.equal(op[0][k], op[1][k]), k
        for ref in refs:
            err = float((op[0][k].double() - ref[k].double()).abs().max() / ref[k].double().abs().max())
            assert err <= tol, f'{k}: {err:.3e}'


def test_second_order_graph_capture_and_no_host_sync():
    shape = SHAPES[2]
    x, wt, a, d, b, pad = _random(shape, F32, 5, 60.0)
    dy = torch.randn(x.shape, generator=torch.Generator(device=DEV).manual_seed(6), device=DEV)
    second = {}
    for name, fn in (('op', lambda *v: gc.gblock_conv0(*v, pad)), ('ref', lambda *v: gc.composition(*v, pad, 'lrelu', 256.0))):
        xs, ws = x.clone().requires_grad_(True), wt.clone().requires_grad_(True)
        y = fn(xs, ws, a, d, b)
        gx, = torch.autograd.grad((y * dy).sum(), [xs], create_graph=True)
        gw, = torch.autograd.grad(gx.square().sum(), [ws])
        second[name] = gw
    assert float((second['op'] - second['ref']).abs().max() / second['ref'].abs().max()) <= 1e-4
    # CUDA-graph capture of forward + backward
    xs, ws = x.clone().requires_grad_(True), wt.clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            gc.gblock_conv0(xs, ws, a, d, b, pad).backward(dy)
    torch.cuda.current_stream().wait_stream(s)
    xs.grad = ws.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        yg = gc.gblock_conv0(xs, ws, a, d, b, pad)
        yg.backward(dy)
    graph.replay()
    torch.cuda.synchronize()
    eager = _grads(lambda *v: gc.gblock_conv0(*v, pad), x, wt, a, d, b, dy)
    assert torch.equal(yg.detach(), gc.gblock_conv0(x, wt, a, d, b, pad))
    assert torch.equal(xs.grad, eager['x']) and torch.equal(ws.grad, eager['w'])
    # no host synchronisation in the forward with the statistic and the backward
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        gc._plugin().fprop(x, wt, a, d, b, pad, 2, 0.2, GAIN, 256.0, want_sumsq=True)
        _grads(lambda *v: gc.gblock_conv0(*v, pad), x, wt, a, d, b, dy)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def _close(a, b, tol):
    return float((a.float() - b.float()).abs().max()) <= tol * max(float(b.float().abs().max()), 1e-30)


def _rel(a, b):
    return float((a.float() - b.float()).abs().max()) / max(float(b.float().abs().max()), 1e-30)


def test_whole_generator_installed(tmp_path_factory):
    """All four installs against none: outputs within 1e-4 and buffers within 1e-6 in every mode. Parameter gradients:
    within 1e-3 of the G with the three other installs (the op's own share), and no further from the uninstalled G than
    that G with the three other installs is, plus 1e-3 (the gradient of the first parameters passes every block, and the
    modulated_conv install alone moves it by a few 1e-3 relative)."""
    res = _run('G', tmp_path_factory)
    base, three, ours = res['none'], res['three'], res['four']
    p, t, q = base['train'], three['train'], ours['train']
    assert _close(q['v'], p['v'], 1e-4)
    for n in p['g']:
        assert _close(q['g'][n], t['g'][n], 1e-3), (n, _rel(q['g'][n], t['g'][n]))
        assert _rel(q['g'][n], p['g'][n]) <= _rel(t['g'][n], p['g'][n]) + 1e-3, n
    for n in p['bufs']:
        assert _close(q['bufs'][n], p['bufs'][n], 1e-6), n
    p, q = base['gen'], ours['gen']
    assert _close(q['v'], p['v'], 1e-4)
    for n in p['bufs']:
        assert _close(q['bufs'][n], p['bufs'][n], 1e-6), n
    assert _close(ours['infer']['v'], base['infer']['v'], 1e-4)
    assert res['nosync'] is True, res['nosync']
    # with the tail on gblock_tail's kernels, a bias_act kernel runs in a mode exactly when conv_0 is not routed to the op;
    # the op's own kernels show in the modes that have them (the backward's row pass, the statistic's fold)
    own = {'train': 'conv0_rows', 'gen': 'conv0_fold', 'infer': None}
    assert res['routed'] == {'train': True, 'gen': True, 'infer': True}            # the 64-channel block
    # update_G: the op takes the blocks of at most 128 channels (DESIGN.md 7m)
    assert res['routed_train'] == [False] * 6 + [False, True, True, True]
    for mode, names in res['prof'].items():
        routed = res['routed'][mode]
        assert routed != any('bias_act' in n for n in names), (mode, names)
        if own[mode] is not None:
            assert routed == any(own[mode] in n for n in names), (mode, names)
