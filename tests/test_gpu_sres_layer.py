"""The fused super-res layer op (torch_utils/ops/sres_layer.py, lvg_sres_layer_* in csrc/sres_layer.cu) on the GPU.

Per layer, for all 15 layers of the default generator (hr 144 x 256, lr 36 x 64) at N T = 64 and for a layer whose x_prev
channel count is not a multiple of 8, with fp32 and fp16 x_prev: the output and the gradients of x_prev, w, a and d bit
for bit those of modulated_conv(cond_concat(...)), the statistic against float64 and across two calls, the create_graph
backward against the composition's, and a call captured in a CUDA graph. The whole installed generator (modulated_conv +
sres_cond + sres_layer) against modulated_conv + sres_cond: outputs, buffers and parameter gradients bit for bit, in the
update_emas forward, in forward + backward (both routed to the composition) and in chained inference (the fused op)."""
import os
import subprocess
import sys

import pytest
import torch

from torch_utils.ops import modulated_conv as mc
from torch_utils.ops import sres_cond as sc
from torch_utils.ops import sres_layer as sl

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
DEV = torch.device('cuda')
_CACHE = {}


def _run(script, mode, out_file):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', script), out_file, mode], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out_file, weights_only=False)


def _layers(tmp_path_factory):
    if 'layers' not in _CACHE:
        _CACHE['layers'] = _run('sres_cond_run.py', 'layers', str(tmp_path_factory.mktemp('sres') / 'layers.pt'))
    return _CACHE['layers']


def _plan(d, i):
    h, w, window = d['plans'][i]
    f = d['filters'][i]
    return sc.Plan(h=h, w=w, filter=None if f is None else f.to(DEV), window=window)


def _randn(shape, dtype, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(shape, generator=g, device=DEV) * scale).to(dtype)


# the 3x3 layers of the default G have conv_kernel 3 (padding 2); layer 14 is ToRGB (1x1, no demodulation)
def _case(d, layer, xdt, c_override=None):
    cin, fp16 = d['layers'][layer]
    dtype = torch.float16 if fp16 else torch.float32
    p = _plan(d, layer)
    c = cin - 27 if c_override is None else c_override
    n = 64
    torgb = layer == 14
    k = 1 if torgb else 3
    cout = 3 if torgb else d['layers'][layer + 1][0] - 27            # layer i's output is layer i + 1's x_prev
    x = None if (c == 0 or xdt is None) else _randn([n, c, p.h.out, p.w.out], xdt, seed=layer, scale=3)
    w = _randn([cout, c + 27, k, k], torch.float32, seed=50 + layer)
    s = _randn([n, c + 27], torch.float32, seed=60 + layer) + 1
    gain = torch.rand([], generator=torch.Generator(device=DEV).manual_seed(70 + layer), device=DEV) + 0.5
    return p, dtype, x, w, s, gain, torgb, (k - 1, k - 1)


def _both(p, dtype, x, lr, w, s, gain, torgb, pad, fused):
    """(y, [dx, dw, ds]) of one layer through the fused op or the composition, from leaf copies of the inputs."""
    xl = None if x is None else x.detach().clone().requires_grad_(True)
    wl = w.detach().clone().requires_grad_(True)
    sl_ = s.detach().clone().requires_grad_(True)
    wn, a, d = mc.factors(wl, sl_, demodulate=not torgb, input_gain=gain)
    if fused:
        y = sl.sres_layer(xl, lr, p, dtype, wn.to(dtype), a, d, pad)
    else:
        z, _ = sc.cond_concat(xl, lr, p, dtype, False)
        assert mc._native(z, wn.to(dtype), pad)
        y = mc.modulated_conv(z, wn.to(dtype), a, d, pad)
    return y, [t for t in (xl, wl, sl_) if t is not None]


LAYER_CASES = [(i, xdt) for i in range(15) for xdt in (torch.float32, torch.float16)]


@pytest.mark.parametrize('layer,xdt', LAYER_CASES + [(10, 'c357'), (12, 'c181_odd')],
                         ids=[f'L{i}_{"x32" if x == torch.float32 else "x16"}' for i, x in LAYER_CASES] + ['L10_c357', 'L12_c181'])
def test_layer_matches_composition(tmp_path_factory, layer, xdt):
    d = _layers(tmp_path_factory)
    c_override = None
    if isinstance(xdt, str):                      # x_prev channel counts that are not multiples of 8
        c_override = 357 if layer == 10 else 181
        xdt = torch.float16
    p, dtype, x, w, s, gain, torgb, pad = _case(d, layer, xdt, c_override)
    if c_override is not None:
        w = _randn([w.shape[0], c_override + 27, 3, 3], torch.float32, seed=99)
        s = _randn([64, c_override + 27], torch.float32, seed=98) + 1
    lr = d['lr'].to(DEV)
    dy = None
    res = {}
    for fused in (False, True):
        y, leaves = _both(p, dtype, x, lr, w, s, gain, torgb, pad, fused)
        if dy is None:
            dy = _randn(y.shape, y.dtype, seed=200 + layer)
        grads = torch.autograd.grad(y, leaves, dy)
        res[fused] = (y.detach(), grads)
    y0, g0 = res[False]
    y1, g1 = res[True]
    assert y1.dtype == y0.dtype and torch.equal(y1, y0)
    for a, b in zip(g1, g0):
        assert a.dtype == b.dtype and torch.equal(a, b)
    # the statistic: float64, and bitwise across two calls
    c = 0 if x is None else x.shape[1]
    ms1 = sl.mean_sq(x, lr, p, dtype, w[:, :c + 27].to(dtype), pad)
    ms2 = sl.mean_sq(x, lr, p, dtype, w[:, :c + 27].to(dtype), pad)
    assert torch.equal(ms1, ms2)
    z64 = torch.cat(([x.double()] if x is not None else []) + [sc.cond_concat(None, lr, p, torch.float32, False)[0].double()], 1)
    want = float(z64.square().mean())
    assert abs(float(ms1) - want) <= 1e-6 * want, (float(ms1), want)


# fp32 layers (0-2): the second-order terms of random fp16 layers overflow or underflow in fp16 on both paths
@pytest.mark.parametrize('layer,xdt', [(1, torch.float32), (2, torch.float16)])
def test_create_graph_matches_composition(tmp_path_factory, layer, xdt):
    d = _layers(tmp_path_factory)
    p, dtype, x, w, s, gain, torgb, pad = _case(d, layer, xdt)
    lr = d['lr'].to(DEV)[:2]
    x = x[:2 * (lr.shape[2] - p.window + 1)]
    s = s[:x.shape[0]]
    res = {}
    for fused in (False, True):
        y, leaves = _both(p, dtype, x, lr, w, s, gain, torgb, pad, fused)
        dy = _randn(y.shape, y.dtype, seed=300 + layer)
        gx, = torch.autograd.grad(y, [leaves[0]], dy, create_graph=True)
        g2 = torch.autograd.grad(gx.float().square().mean(), leaves[1:])
        res[fused] = [gx.detach()] + list(g2)
    assert torch.equal(res[True][0], res[False][0])
    # second order: the same terms, which autograd may accumulate in another order
    for a, b in zip(res[True][1:], res[False][1:]):
        assert bool(torch.isfinite(a).all()) and bool(b.abs().max() > 0)
        err = float((a.double() - b.double()).abs().max() / b.double().abs().max())
        assert err <= 1e-5, err


def test_cuda_graph_capture(tmp_path_factory):
    d = _layers(tmp_path_factory)
    p, dtype, x, w, s, gain, torgb, pad = _case(d, 11, torch.float16)
    lr = d['lr'].to(DEV)
    wn, a, dd = mc.factors(w, s, demodulate=True, input_gain=gain)
    wx = wn.to(dtype)
    want = sl.sres_layer(x, lr, p, dtype, wx, a, dd, pad)
    want_ms = sl.mean_sq(x, lr, p, dtype, wx, pad)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        sl.sres_layer(x, lr, p, dtype, wx, a, dd, pad)
        sl.mean_sq(x, lr, p, dtype, wx, pad)
    torch.cuda.current_stream().wait_stream(st)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = sl.sres_layer(x, lr, p, dtype, wx, a, dd, pad)
        got_ms = sl.mean_sq(x, lr, p, dtype, wx, pad)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(got, want) and torch.equal(got_ms, want_ms)


def test_whole_generator_installed_matches(tmp_path):
    res = _run('sres_layer_run.py', 'model', str(tmp_path / 'model.pt'))
    ref, ours = res[False], res[True]
    assert torch.equal(ours['v'], ref['v'])
    assert set(ours['grads']) == set(ref['grads'])
    for k in ref['grads']:
        assert torch.equal(ours['grads'][k], ref['grads'][k]), k
    assert torch.equal(ours['v0'], ref['v0'])
    for k, b in ref['bufs'].items():
        assert torch.equal(ours['bufs'][k], b), k
    assert torch.equal(ours['chained'], ref['chained'])
