"""The ToRGB op of the super-res generator (torch_utils/ops/sres_torgb.py, lvg_sres_torgb_* in csrc/sres_torgb.cu) on the
GPU, on the default generator's layer 14 at N T = 64, on a small odd shape (37 columns: rows that do not start on a
16-byte boundary; 45 x_prev channels) and on two shapes of several row tiles with a shorter last tile (23 rows of 200
and 203 columns), with fp16 and fp32 x_prev and layer dtype.

Numerical contract. The op sums the products in fp32 on the CUDA cores, the composition (cond_concat -> modulated_conv
on the wgmma engine -> filtered_lrelu) in another order, so:
- y against float64 of the same rounded operands r(a z) and dtype(w): half an ulp of the layer dtype plus
  2^-22 sum_c |w a z| per element;
- y against the composition: two ulps of the layer dtype (at the larger of |y| and |y - b|, the convolution's rounding)
  plus 2^-17 sum_c |w a z| in fp16 layers, 2^-15 in fp32 layers (the engine's three-product bf16 split). The op is
  within half an ulp of the exact value (above); the composition is not: on layer 14's fp16 inputs it is off by up to
  about 1.6 ulps, measured on an H100, so the two may differ by more than one ulp;
- gradients against the composition's taken with the op's clamp mask (near the clamp the two may round u to either
  side; the mask itself is checked against float64 wherever u is clear of the clamp);
- dx_prev: one rounding of dx' (scaled by a) and one of dx_prev, plus 2^-12 of sum_o |w dy| a in fp32 layers (the
  engine's split input gradient); dw, da, db within 1e-4 of each tensor's largest magnitude, plus one ulp of the layer
  dtype per element for dw and db, which both sides round to the layer dtype, and in fp32 layers 2^-15 of
  sum |dy' r(a z)| per element of dw (the split weight gradient);
- two calls bitwise identical; create_graph second-order gradients as the composition's; CUDA-graph capture.
The whole installed generator against modulated_conv + sres_cond (+ sres_layer in chained inference) within those bounds.
"""
import os
import subprocess
import sys

import pytest
import torch

from torch_utils.ops import sres_cond as sc
from torch_utils.ops import sres_torgb as st

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
DEV = torch.device('cuda')
CLAMP = 256.0
_CACHE = {}


def _run(script, mode, out_file):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', script), out_file, mode], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out_file, weights_only=False)


def _layers(tmp_path_factory):
    if 'layers' not in _CACHE:
        _CACHE['layers'] = _run('sres_cond_run.py', 'layers', str(tmp_path_factory.mktemp('torgb') / 'layers.pt'))
    return _CACHE['layers']


def _randn(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=DEV) * scale).to(dtype)


def _case(d, shape, xdt, dtype):
    """(plan, lr, x_prev, w [3, Cin] fp32, a [N T, Cin, 1], b [3] fp32): layer 14's plan and low-res video, or the odd
    shape. w is scaled so that about a fifth of the outputs pass the clamp."""
    f = d['filters'][14].to(DEV)
    if shape == 'L14':
        h, w_, window = d['plans'][14]
        p = sc.Plan(h=h, w=w_, filter=f, window=window)
        lr = d['lr'].to(DEV)
        c = d['layers'][14][0] - 27
    elif shape == 'odd':
        p = sc.Plan(h=sc.axis_plan(9, 15, 4, 'up', 4, 24, True, 23), w=sc.axis_plan(15, 15, 4, 'up', 4, 24, True, 37),
                    filter=f, window=3)
        lr = _randn([2, 3, 4, 9, 15], torch.float32, seed=7)
        c = 45
    else:
        # 23 rows in tiles of 10 (2048 // width): two full tiles and a last tile of 3 rows; width 200 takes the 16-byte
        # loads, 203 the scalar ones
        wd = 200 if shape == 'tiles' else 203
        p = sc.Plan(h=sc.axis_plan(9, 60, 4, 'up', 4, 24, True, 23), w=sc.axis_plan(60, 60, 4, 'up', 4, 24, True, wd),
                    filter=f, window=3)
        lr = _randn([2, 3, 4, 9, 60], torch.float32, seed=7)
        c = 45
    nt = lr.shape[0] * (lr.shape[2] - p.window + 1)
    cin = c + 3 * p.window
    x = _randn([nt, c, p.h.out, p.w.out], xdt, seed=1, scale=3)
    w = _randn([3, cin], torch.float32, seed=2, scale=16)
    a = (_randn([nt, cin, 1], torch.float32, seed=3) * 0.3 + 1) * cin ** -0.5 * 4
    b = _randn([3], torch.float32, seed=4)
    return p, lr, x, w, a, b


def _ulp(v, dtype):
    fi = torch.finfo(dtype)
    mant = 10 if dtype == torch.float16 else 23
    e = torch.floor(torch.log2(v.double().abs().clamp_min(fi.tiny)))
    return torch.exp2(e - mant)


def _mask(p, lr, x, w, a, b, dtype):
    f = p.filter
    _, mask = st._plugin().torgb_fprop(x, lr, f, f, sc._ints(p.h), sc._ints(p.w), p.h.gain, p.w.gain, p.window, dtype,
                                       w, a, b, CLAMP, True)
    return mask


def _run_op(fused, p, lr, x, w, a, b, dtype, dy=None):
    xl = x.detach().clone().requires_grad_(True)
    wl = w.to(dtype).detach().clone().requires_grad_(True)
    al = a.detach().clone().requires_grad_(True)
    bl = b.to(dtype).detach().clone().requires_grad_(True)
    fn = st.sres_torgb if fused else st.composition
    y = fn(xl, lr, p, dtype, wl, al, bl, CLAMP)
    if dy is None:
        return y.detach(), None
    if not fused:
        # near the clamp the two paths may round u to different sides of it; take the composition's gradients with
        # the op's clamp mask (filtered_lrelu without a clamp passes dy through), so they differ by rounding alone
        mask = _mask(p, lr, x, w.to(dtype), a, b.to(dtype), dtype)
        keep = torch.stack([((mask >> o) & 1) == 0 for o in range(3)], 1)
        y_nc = fn(xl, lr, p, dtype, wl, al, bl, None)
        return y.detach(), torch.autograd.grad(y_nc, [xl, wl, al, bl], dy * keep.to(dy.dtype))
    return y.detach(), torch.autograd.grad(y, [xl, wl, al, bl], dy)


SHAPES = ('L14', 'odd', 'tiles', 'tiles_odd')
CASES = [(s, xdt, dt) for s in SHAPES for xdt in (torch.float16, torch.float32) for dt in (torch.float16, torch.float32)]
IDS = [f'{s}_x{16 if x == torch.float16 else 32}_{16 if d == torch.float16 else 32}' for s, x, d in CASES]


@pytest.mark.parametrize('shape,xdt,dtype', CASES, ids=IDS)
def test_forward_against_float64(tmp_path_factory, shape, xdt, dtype):
    p, lr, x, w, a, b = _case(_layers(tmp_path_factory), shape, xdt, dtype)
    zero = torch.zeros(3, device=DEV)
    y = st.sres_torgb(x, lr, p, dtype, w.to(dtype), a, zero.to(dtype), CLAMP)
    z, _ = sc.cond_concat(x, lr, p, dtype, False)
    az = (z.float() * a[..., None]).to(dtype).double()                 # r(a z): the engine's re-tiling rounding
    wd = w.to(dtype).double()
    u = torch.einsum('oc,nchw->nohw', wd, az)
    mag = torch.einsum('oc,nchw->nohw', wd.abs(), az.abs())
    want = u.clamp(-CLAMP, CLAMP)
    err = (y.double() - want).abs()
    bound = 0.5 * _ulp(want, dtype) + 2.0 ** -22 * mag
    assert bool((err <= bound).all()), float((err / bound).max())
    assert float((u.abs() > CLAMP).double().mean()) > 0.05                # the clamp is exercised
    # the clamp mask the backward applies: bit o where |dtype(u) + b| > clamp, wherever u is clear of the clamp by more
    # than the bound above
    mask = _mask(p, lr, x, w.to(dtype), a, zero.to(dtype), dtype)
    bits = torch.stack([(mask >> o) & 1 for o in range(3)], 1).bool()
    clear = (u.abs() - CLAMP).abs() > 2 * bound
    assert torch.equal(bits[clear], (u.abs() > CLAMP)[clear]) and float(clear.double().mean()) > 0.99


@pytest.mark.parametrize('shape,xdt,dtype', CASES, ids=IDS)
def test_against_composition(tmp_path_factory, shape, xdt, dtype):
    p, lr, x, w, a, b = _case(_layers(tmp_path_factory), shape, xdt, dtype)
    dy = _randn([x.shape[0], 3, p.h.out, p.w.out], dtype, seed=5)
    y0, g0 = _run_op(False, p, lr, x, w, a, b, dtype, dy)
    y1, g1 = _run_op(True, p, lr, x, w, a, b, dtype, dy)
    y2, g2 = _run_op(True, p, lr, x, w, a, b, dtype, dy)
    assert torch.equal(y1, y2) and all(torch.equal(u, v) for u, v in zip(g1, g2))     # bitwise reproducible
    assert y1.dtype == dtype and y1.shape == y0.shape
    # y: one ulp of the layer dtype at the convolution's output, plus the engine's split in fp32
    z, _ = sc.cond_concat(x, lr, p, dtype, False)
    mag = torch.einsum('oc,nchw->nohw', w.to(dtype).double().abs(), (z.float() * a[..., None]).to(dtype).double().abs())
    bd = b.to(dtype).double()[None, :, None, None]
    at = torch.maximum(y0.double().abs(), (y0.double() - bd).abs())
    bound = 2 * _ulp(at, dtype) + (2.0 ** -15 if dtype == torch.float32 else 2.0 ** -17) * mag
    err = (y1.double() - y0.double()).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    # dx_prev: one rounding of dx' scaled by a, one of dx_prev (and the engine's split in fp32)
    dx0, dx1 = g0[0].double(), g1[0].double()
    dxp = torch.einsum('oc,nohw->nchw', w.to(dtype).double().abs(), dy.double().abs())[:, :x.shape[1]]
    ad = a[:, :x.shape[1], :, None].double().abs()
    dxm = torch.maximum(dx0.abs(), dx1.abs())                           # the ulp of the larger: rounding across a binade
    bound = _ulp(dxm, xdt) + _ulp(dxm, dtype) + ad * (_ulp(dxp, dtype) + (2.0 ** -12 * dxp if dtype == torch.float32 else 0))
    err = (dx1 - dx0).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    # dw, da, db; fp32 layers add the split's 2^-15 of sum |dy' r(a z)| to dw
    split = 0
    if dtype == torch.float32:
        keep = torch.stack([((_mask(p, lr, x, w, a, b, dtype) >> o) & 1) == 0 for o in range(3)], 1)
        az = (z.float() * a[..., None]).abs().double()
        split = 2.0 ** -15 * torch.einsum('nohw,nchw->oc', dy.double().abs() * keep, az)
    for name, u, v, rounded in (('dw', g1[1], g0[1], True), ('da', g1[2], g0[2], False), ('db', g1[3], g0[3], True)):
        assert u.dtype == v.dtype and u.shape == v.shape, name
        v64, u64 = v.double(), u.double()
        bound = 1e-4 * float(v64.abs().max()) + (_ulp(v64, dtype) if rounded else 0) + (split if name == 'dw' else 0)
        assert bool(((u64 - v64).abs() <= bound).all()), (name, float((u64 - v64).abs().max()), float(v64.abs().max()))


def test_create_graph_matches_composition(tmp_path_factory):
    p, lr, x, w, a, b = _case(_layers(tmp_path_factory), 'L14', torch.float16, torch.float32)
    lr = lr[:2]
    nt = 2 * (lr.shape[2] - p.window + 1)
    x, a = x[:nt], a[:nt]
    res = {}
    for fused in (False, True):
        xl = x.detach().clone().requires_grad_(True)
        wl = w.detach().clone().requires_grad_(True)
        al = a.detach().clone().requires_grad_(True)
        bl = b.detach().clone().requires_grad_(True)
        y = (st.sres_torgb if fused else st.composition)(xl, lr, p, torch.float32, wl, al, bl, CLAMP)
        dy = _randn(y.shape, y.dtype, seed=8)
        gx, = torch.autograd.grad(y, [xl], dy, create_graph=True)
        g2 = torch.autograd.grad(gx.float().square().mean(), [wl, al])
        res[fused] = [gx.detach()] + list(g2)
    assert torch.equal(res[True][0], res[False][0])
    for u, v in zip(res[True][1:], res[False][1:]):
        assert bool(torch.isfinite(u).all()) and bool(v.abs().max() > 0)
        err = float((u.double() - v.double()).abs().max() / v.double().abs().max())
        assert err <= 1e-5, err


def test_cuda_graph_capture(tmp_path_factory):
    p, lr, x, w, a, b = _case(_layers(tmp_path_factory), 'L14', torch.float16, torch.float16)
    dtype = torch.float16
    wl = w.to(dtype).requires_grad_(True)
    al = a.clone().requires_grad_(True)
    bl = b.to(dtype).requires_grad_(True)
    xl = x.clone().requires_grad_(True)
    dy = _randn([x.shape[0], 3, p.h.out, p.w.out], dtype, seed=9)

    def step():
        y = st.sres_torgb(xl, lr, p, dtype, wl, al, bl, CLAMP)
        return [y.detach()] + list(torch.autograd.grad(y, [xl, wl, al, bl], dy))
    want = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = step()
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(u, v) for u, v in zip(got, want))


def _close(u, v, rounded_to=None):
    """Within 1e-4 of the largest magnitude, plus one ulp of ``rounded_to`` per element where both sides round the
    gradient to that dtype."""
    u, v = u.double(), v.double()
    bound = 1e-4 * float(v.abs().max()) + (_ulp(v, rounded_to) if rounded_to is not None else 0)
    return bool(((u - v).abs() <= bound).all())


def test_whole_generator_installed_matches(tmp_path):
    res = _run('sres_torgb_run.py', 'model', str(tmp_path / 'model.pt'))
    ref, ours = res[False], res[True]
    sc_ = res['output_scale']
    for k in ('v0', 'v', 'chained'):
        u, v = ours[k].double(), ref[k].double()
        bound = _ulp(v / sc_, torch.float16) * abs(sc_) * 2 + 1e-6
        assert bool(((u - v).abs() <= bound).all()), (k, float((u - v).abs().max()))
    # buffers: every one bit for bit but the ToRGB magnitude EMA, which is sres_layer.mean_sq's statistic bit for bit
    ema = f'SG3.synthesis.{ours["torgb_name"]}.magnitude_ema'
    for k, b in ref['bufs'].items():
        if k == ema:
            assert torch.equal(ours['bufs'][k], ours['torgb_ema'])
            assert abs(float(ours['bufs'][k]) - float(b)) <= 1e-6 * abs(float(b))
        else:
            assert torch.equal(ours['bufs'][k], b), k
    assert set(ours['grads']) == set(ref['grads'])
    # the ToRGB weight and bias gradients are rounded to the layer dtype (fp16) on both sides; all others are fp32
    torgb = f'SG3.synthesis.{ours["torgb_name"]}.'
    for k in ref['grads']:
        rounded = torch.float16 if k in (torgb + 'weight', torgb + 'bias') else None
        assert _close(ours['grads'][k], ref['grads'][k], rounded), (k, float((ours['grads'][k] - ref['grads'][k]).abs().max()),
                                                                    float(ref['grads'][k].abs().max()))
