"""The ToRGB op of the low-res generator (torch_utils/ops/lres_torgb.py, lvg_lres_torgb_* in csrc/lres_torgb.cu) on the
GPU: the default generator's layer (64 channels, 36 x 64) and an odd shape (45 channels, 23 x 37, T = 1: planes that do
not start on a 16-byte boundary), with fp16 and fp32 x and layer dtype, and inputs scaled so that some outputs clamp.

Numerical contract. The op sums w a r(x) in fp32 on the CUDA cores, so:
- y against float64 of the same rounded operands (w = weight / sqrt(cin) and a in fp32, r(x) = x.type(dtype)): half an ulp
  of the layer dtype at u (its rounding to dtype) and half an ulp at y (the rounding after the bias), plus
  2^-22 sum_c |w a r(x)| per element;
- the beta != 1 forward-only path: one more rounding of the layer dtype (the gain applied to u, not to x); the EMA buffer
  within 1e-6 relative of the reference module's;
- gradients (dx, dw, db, and the style gradient as it reaches the affine layer) against the reference's within 1e-4 of
  each tensor's largest magnitude; two calls bitwise identical; create_graph second order; CUDA-graph capture.
The whole default G with modulated_conv + gblock_tail installed, with and without lres_torgb, within those bounds.
"""
import os
import subprocess
import sys

import pytest
import torch

from torch_utils.ops import lres_torgb as lt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
DEV = torch.device('cuda')
F16, F32 = torch.float16, torch.float32
_CACHE = {}


def _run(mode, tmp_path_factory):
    if mode not in _CACHE:
        out = str(tmp_path_factory.mktemp('lres_torgb') / f'{mode}.pt')
        env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]))
        r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'lres_torgb_run.py'), out, mode], env=env, cwd=SRC,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
        assert r.returncode == 0, r.stdout[-3000:]
        _CACHE[mode] = torch.load(out, weights_only=False)
    return _CACHE[mode]


def _ulp(v, dtype):
    mant, tiny = (10, 2.0 ** -24) if dtype == F16 else (23, 2.0 ** -149)
    e = torch.floor(torch.log2(v.abs().clamp_min(tiny)))
    return torch.maximum(torch.exp2(e - mant), torch.full_like(v, tiny))


def _operands(n, cin, t, h, w, xd, seed, scale):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = (torch.randn(n, cin, t, h, w, generator=g, device=DEV) * scale).to(xd)
    wt = torch.randn(3, cin, generator=g, device=DEV) / cin ** 0.5
    a = torch.randn(n, cin, t, generator=g, device=DEV) + 1
    b = torch.randn(3, generator=g, device=DEV) * 0.5
    return x, wt, a, b


def _exact(x, wt, a, dtype):
    """u in float64 of the rounded operands, and sum |w a r(x)|."""
    z = x.to(dtype).double()
    wa = wt.double()[None, :, :, None] * a.double()[:, None]                      # [n, 3, cin, t]
    u = torch.einsum('nocy,ncyhw->noyhw', wa, z)
    s = torch.einsum('nocy,ncyhw->noyhw', wa.abs(), z.abs())
    return u, s


SHAPES = [(2, 64, 6, 36, 64), (3, 45, 1, 23, 37)]


@pytest.mark.parametrize('shape', SHAPES, ids=['default', 'odd'])
@pytest.mark.parametrize('xd,dt', [(F16, F16), (F16, F32), (F32, F16), (F32, F32)], ids=['x16-f16', 'x16-f32', 'x32-f16', 'x32-f32'])
@pytest.mark.parametrize('scale', [1.0, 200.0], ids=['plain', 'clamping'])
def test_forward_against_float64(shape, xd, dt, scale):
    clamp = 256.0
    x, wt, a, b = _operands(*shape, xd, 1, scale)
    y = lt.lres_torgb(x, wt, a, b, dt, clamp)
    assert y.dtype == dt and tuple(y.shape) == (shape[0], 3) + shape[2:]
    u, s = _exact(x, wt, a, dt)
    ref = (u + b.to(dt).double()[None, :, None, None, None]).clamp(-clamp, clamp)
    bound = 0.5 * _ulp(u, dt) + 0.5 * _ulp(ref, dt) + 2.0 ** -22 * s
    err = (y.double() - ref).abs()
    assert bool((err <= bound).all()), f'max err / bound {float((err / bound).max()):.3f}'
    if scale > 1:
        assert bool((y.abs() == clamp).any()) and bool((y.abs() < clamp).any())


@pytest.mark.parametrize('shape', SHAPES, ids=['default', 'odd'])
@pytest.mark.parametrize('xd,dt', [(F16, F16), (F32, F32), (F32, F16)], ids=['x16-f16', 'x32-f32', 'x32-f16'])
def test_sumsq_path_against_float64(shape, xd, dt):
    x, wt, a, b = _operands(*shape, xd, 2, 3.0)
    plug = lt._plugin()
    u, sumsq = plug.fprop_sumsq(x, wt, a, dt)
    uref, s = _exact(x, wt, a, dt)
    assert bool(((u.double() - uref).abs() <= 2.0 ** -22 * s + 1e-30).all())
    sq = x.to(dt).double().square().sum()
    assert abs(float(sumsq) - float(sq)) <= 1e-6 * float(sq)
    gain = torch.tensor(0.37, device=DEV)
    y = plug.finish(u, gain, b, dt, 256.0)
    ref = (uref * 0.37 + b.to(dt).double()[None, :, None, None, None]).clamp(-256, 256)
    bound = 0.5 * _ulp(uref, dt) + _ulp(ref, dt) + 2.0 ** -21 * s
    assert bool(((y.double() - ref).abs() <= bound).all())


@pytest.mark.parametrize('shape', SHAPES, ids=['default', 'odd'])
@pytest.mark.parametrize('xd,dt', [(F16, F16), (F32, F32), (F32, F16)], ids=['x16-f16', 'x32-f32', 'x32-f16'])
def test_gradients_against_float64_and_bitwise_repeatable(shape, xd, dt):
    """dx, dw, da, db of the op against float64 of the same rounded operands and the op's own clamp decisions."""
    x, wt, a, b = _operands(*shape, xd, 3, 20.0)
    g = torch.Generator(device=DEV).manual_seed(4)
    runs = []
    for _ in range(2):
        xs, ws, as_, bs = (v.clone().requires_grad_(True) for v in (x, wt, a, b))
        y = lt.lres_torgb(xs, ws, as_, bs, dt, 256.0)
        dy = torch.randn(y.shape, generator=g.manual_seed(4), device=DEV).to(dt)
        y.backward(dy)
        runs.append((y.detach(), dy, xs.grad, ws.grad, as_.grad, bs.grad))
    for p, q in zip(runs[0][2:], runs[1][2:]):
        assert torch.equal(p, q)
    y, dy, dx, dw, da, db = runs[0]
    dyp = torch.where(y.abs() < 256, dy, torch.zeros_like(dy)).double()
    z = x.to(dt).double()
    dxr = torch.einsum('oc,noyhw->ncyhw', wt.double(), dyp) * a.double()[..., None, None]
    gram = torch.einsum('noyhw,ncyhw->nocy', dyp, z)
    dar = torch.einsum('oc,nocy->ncy', wt.double(), gram)
    dwr = torch.einsum('ncy,nocy->oc', a.double(), gram)
    dbr = dyp.sum(dim=(0, 2, 3, 4))
    for name, got, ref in (('dx', dx, dxr), ('dw', dw, dwr), ('da', da, dar), ('db', db, dbr)):
        err = float((got.double() - ref).abs().max() / ref.abs().max())
        tol = 1e-5 if name != 'dx' or xd == F32 else 2.0 ** -10
        assert err <= tol, f'{name}: {err:.3e}'


def test_layer_against_the_reference_in_every_mode(tmp_path_factory):
    res = _run('layer', tmp_path_factory)
    for dt in (F32, F16):
        for beta in (1.0, 0.999):
            r = res[('fwd', dt, beta)]
            assert r['dtype'] == dt
            ref, ours = r['ref'], r['ours']
            # the reference rounds x gain and x gain style to the layer dtype; the op rounds once
            tol = (2.0 ** -18 if dt == F32 else 2.0 ** -8) * float(ref.abs().max())
            assert float((ours - ref).abs().max()) <= tol, (dt, beta)
            assert abs(r['ema_ours'] - r['ema_ref']) <= 1e-6 * abs(r['ema_ref']), (dt, beta)
    d = res['dist']
    assert d['calls'] == ['sum'] and abs(d['ema'] - d['ema_ref']) <= 1e-6 * abs(d['ema_ref'])
    ref, ours = res['grads']['ref'][0], res['grads']['ours']
    for k in ('x', 'lat', 'w', 'b', 'aff'):
        err = float((ours[0][k] - ref[k]).abs().max() / ref[k].abs().max())
        assert err <= 1e-4, f'{k}: {err:.3e}'
        assert torch.equal(ours[0][k], ours[1][k]), k
    s = res['second']
    assert float((s['ours'] - s['ref']).abs().max() / s['ref'].abs().max()) <= 1e-4
    gph = res['graph']
    assert torch.equal(gph['y'], gph['y_ref']) and torch.equal(gph['x'], gph['x_ref'])


def _close(a, b, tol):
    return float((a.float() - b.float()).abs().max()) <= tol * max(float(b.float().abs().max()), 1e-30)


def test_whole_generator_installed(tmp_path_factory):
    res = _run('G', tmp_path_factory)
    base, ours = res[False], res[True]
    for beta in (1.0, 0.999):
        p, q = base[('train', beta)], ours[('train', beta)]
        assert _close(q['v'], p['v'], 1e-4), beta
        for n in p['g']:
            assert _close(q['g'][n], p['g'][n], 1e-3), (beta, n)
        for n in p['bufs']:
            assert _close(q['bufs'][n], p['bufs'][n], 1e-6), (beta, n)
    p, q = base[('gen', 0.999)], ours[('gen', 0.999)]
    assert _close(q['v'], p['v'], 1e-4)
    for n in p['bufs']:
        assert _close(q['bufs'][n], p['bufs'][n], 1e-6), n
    assert len(base['segments']) == len(ours['segments'])
    for s, t in zip(base['segments'], ours['segments']):
        assert _close(t, s, 1e-4)
    assert res['nosync'] is True, res['nosync']
    for mode, names in res['prof'].items():
        assert any('lres_torgb' in n for n in names), mode
        assert not any(('conv' in n.lower() or 'bias_act' in n.lower()) and 'lres_torgb' not in n for n in names), (mode, names)
