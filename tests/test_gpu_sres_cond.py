"""The super-res layer input (torch_utils/ops/sres_cond.py, csrc/sres_cond.cu) on the GPU: for each of the 15 layers of the
default generator (hr 144 x 256, lr 36 x 64) at N T = 64, in fp32 and fp16, with and without x_prev, the conditioning
channels against the float64 plan, the x_prev channels and dx_prev against the reference's cat + .to bit for bit, the
mean square against float64 and across calls; guard bands around z; CUDA-graph capture; the whole installed generator
against the not-installed one (both with modulated_conv.install); and lvg_infer.chained.generate_video installed and not."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import sres_cond as sc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
DEV = torch.device('cuda')
_CACHE = {}


def _run(mode, out_file):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'sres_cond_run.py'), out_file, mode], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out_file, weights_only=False)


def _layers(tmp_path_factory):
    if 'layers' not in _CACHE:
        _CACHE['layers'] = _run('layers', str(tmp_path_factory.mktemp('sres') / 'layers.pt'))
    return _CACHE['layers']


def _plan(d, i):
    h, w, window = d['plans'][i]
    f = d['filters'][i]
    return sc.Plan(h=h, w=w, filter=None if f is None else f.to(DEV), window=window)


def _ref64(d, i):
    """The float64 plan evaluated on the device: [64, 27, H, W]."""
    key = ('ref64', i)
    if key not in _CACHE:
        _CACHE.pop(next((k for k in _CACHE if k[0] == 'ref64'), None), None)
        p = _plan(d, i)
        a_h = sc.axis_matrix(p.h, p.filter).to(DEV)
        a_w = sc.axis_matrix(p.w, p.filter).to(DEV)
        x = d['lr'].to(DEV).double().unfold(2, p.window, 1)
        n, c, t = x.shape[:3]
        y = torch.einsum('yh,ncthws,xw->ntcsyx', a_h, x, a_w)
        _CACHE[key] = y.reshape(n * t, c * p.window, p.h.out, p.w.out)
    return _CACHE[key]


def _x(n, c, h, w, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(n, c, h, w, generator=g, device=DEV) * 3).to(dtype)


def _fp16_ulps(got, ref64):
    """|got - fp16(ref)| in units of fp16(ref)'s ulp, and whether got is the fp16 rounding of a value within the fp32
    tolerance (2e-6 of the largest |ref|) of ref: where the FIR cancels to values far below the layer's largest, the fp32
    accumulation error alone spans more than one ulp of fp16, for the reference's own fp32 prep_cond as for the kernel."""
    want = ref64.to(torch.float16)
    e = torch.floor(torch.log2(want.double().abs().clamp_min(2.0 ** -14)))
    ulp = torch.exp2(e - 10)
    ulps = (got.double() - want.double()).abs() / ulp
    tol = 2e-6 * float(ref64.abs().max())
    ok = (got.double() - ref64).abs() <= ulp / 2 + tol
    return ulps, bool(ok.all())


COMBOS = [(torch.float32, None), (torch.float32, torch.float32), (torch.float16, None), (torch.float16, torch.float16),
          (torch.float16, torch.float32)]


@pytest.mark.parametrize('combo', COMBOS, ids=['f32', 'f32_x32', 'f16', 'f16_x16', 'f16_x32'])
@pytest.mark.parametrize('layer', range(15), ids=[f'L{i}' for i in range(15)])
def test_layer_input(tmp_path_factory, layer, combo):
    dtype, xdt = combo
    d = _layers(tmp_path_factory)
    cin, _ = d['layers'][layer]
    c = cin - 27
    if xdt is not None and c == 0:
        pytest.skip('layer 0 has no x_prev without fourfeats')
    p = _plan(d, layer)
    lr = d['lr'].to(DEV)
    ref = _ref64(d, layer)
    n = ref.shape[0]
    assert n == 64
    x = None if xdt is None else _x(n, c, p.h.out, p.w.out, xdt, seed=layer).requires_grad_(True)
    z, ms = sc.cond_concat(x, lr, p, dtype, True)
    c0 = 0 if x is None else c
    assert z.dtype == dtype and tuple(z.shape) == (n, c0 + 27, p.h.out, p.w.out)
    cond = z[:, c0:]
    if dtype == torch.float32:
        err = float((cond.detach().double() - ref).abs().max())
        assert err <= 2e-6 * float(ref.abs().max()), err
    else:
        ulps, ok = _fp16_ulps(cond, ref)
        big = ref.abs() >= 1e-2 * float(ref.abs().max())
        assert ok and float(ulps[big].max()) <= 1, (float(ulps.max()), float(ulps[big].max()))
    # the mean square of the fp32 concatenation against float64, and bitwise across calls
    total = ref.square().sum()
    if x is not None:
        total = total + x.detach().double().square().sum()
    want = float(total / z.numel())
    assert abs(float(ms) - want) <= 1e-6 * want, (float(ms), want)
    z2, ms2 = sc.cond_concat(x, lr, p, dtype, True)
    assert torch.equal(ms, ms2) and torch.equal(z, z2)
    if x is None:
        return
    # x_prev channels and dx_prev: the reference's cat(...).to(dtype) and its autograd, bit for bit
    xr = x.detach().clone().requires_grad_(True)
    zr = torch.cat((xr, ref.float()), 1).to(dtype)
    assert torch.equal(z[:, :c], zr[:, :c])
    dz = _x(n, c + 27, p.h.out, p.w.out, dtype, seed=100 + layer)
    gx, = torch.autograd.grad(z, [x], dz)
    gr, = torch.autograd.grad(zr, [xr], dz)
    assert gx.dtype == x.dtype and gx.is_contiguous() and torch.equal(gx, gr)


@pytest.mark.parametrize('layer,xdt', [(3, torch.float32), (11, torch.float16), (0, None)])
def test_nothing_written_outside_z(tmp_path_factory, layer, xdt):
    d = _layers(tmp_path_factory)
    p = _plan(d, layer)
    cin, fp16 = d['layers'][layer]
    dtype = torch.float16 if fp16 else torch.float32
    lr = d['lr'].to(DEV)[:2]
    n = 2 * (lr.shape[2] - p.window + 1)
    c = 0 if xdt is None else cin - 27
    x = None if xdt is None else _x(n, c, p.h.out, p.w.out, xdt, seed=7)
    numel = n * (c + 27) * p.h.out * p.w.out
    guard = 4096
    buf = torch.full([numel + 2 * guard], -12345.0, dtype=dtype, device=DEV)
    z = buf[guard:guard + numel]
    assert z.data_ptr() % 16 == 0
    lib = custom_ops.load_library()
    ph = (ctypes.c_int * 10)(*sc._ints(p.h))
    pw = (ctypes.c_int * 10)(*sc._ints(p.w))
    strides = (ctypes.c_int64 * 5)(*lr.stride())
    ms = torch.empty([], dtype=torch.float32, device=DEV)
    nb = lib.lvg_sres_cond_workspace(2, n // 2, c, 3, p.window, lr.shape[2], 36, 64, custom_ops._DTYPE_CODE[dtype], ph, pw)
    ws = torch.empty([nb // 8], dtype=torch.float64, device=DEV)
    f = p.filter
    rc = lib.lvg_sres_cond(None if x is None else x.data_ptr(), lr.data_ptr(), None if f is None else f.data_ptr(),
                           None if f is None else f.data_ptr(), z.data_ptr(), ms.data_ptr(), ws.data_ptr(), nb,
                           custom_ops._DTYPE_CODE[xdt or dtype], custom_ops._DTYPE_CODE[dtype], 2, n // 2, c, 3, p.window,
                           lr.shape[2], 36, 64, strides, ph, pw, float(p.h.gain), float(p.w.gain),
                           torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    assert bool((buf[:guard] == -12345.0).all()) and bool((buf[guard + numel:] == -12345.0).all())
    want, _ = sc.cond_concat(x, lr, p, dtype, False)
    assert torch.equal(z.view(want.shape), want)


def test_non_contiguous_low_res_segments(tmp_path_factory):
    # the windows of sample_video_segments are strided views: the same result as from a contiguous copy
    d = _layers(tmp_path_factory)
    p = _plan(d, 12)
    full = d['lr'].to(DEV)
    seg = full.permute(0, 2, 1, 3, 4).contiguous().permute(0, 2, 1, 3, 4)
    assert not seg.is_contiguous()
    a, _ = sc.cond_concat(None, seg, p, torch.float16, False)
    b, _ = sc.cond_concat(None, full.contiguous(), p, torch.float16, False)
    assert torch.equal(a, b)


def test_cuda_graph_capture(tmp_path_factory):
    d = _layers(tmp_path_factory)
    p = _plan(d, 11)
    lr = d['lr'].to(DEV)
    x = _x(64, 256, p.h.out, p.w.out, torch.float16, seed=3)
    want = sc.cond_concat(x, lr, p, torch.float16, True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        sc.cond_concat(x, lr, p, torch.float16, True)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        got = sc.cond_concat(x, lr, p, torch.float16, True)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-30))


def test_whole_generator_installed_matches(tmp_path):
    res = _run('model', str(tmp_path / 'model.pt'))
    ref, ours = res[False], res[True]
    errs = {k: _rel(ours[k], ref[k]) for k in ('v0', 'v', 'g2')}
    errs['grads'] = max(_rel(ours['grads'][k], ref['grads'][k]) for k in ref['grads'])
    errs['magnitude_ema'] = max(_rel(ours['bufs'][k], b) for k, b in ref['bufs'].items() if k.endswith('magnitude_ema'))
    print('whole generator, installed vs not (max rel diff):', {k: f'{v:.2e}' for k, v in errs.items()})
    assert _rel(ours['v0'], ref['v0']) <= 5e-3
    assert _rel(ours['v'], ref['v']) <= 5e-3
    assert set(ours['grads']) == set(ref['grads'])
    for k in ref['grads']:
        assert _rel(ours["grads"][k], ref["grads"][k]) <= 2e-2, k      # H100: 1.7e-2 at most (fp16 layers, cond rounded once)
    assert _rel(ours['g2'], ref['g2']) <= 2e-2
    for k, b in ref['bufs'].items():
        if k.endswith('w_avg'):
            assert torch.equal(ours['bufs'][k], b), k
        elif k.endswith('magnitude_ema'):
            assert _rel(ours['bufs'][k], b) <= 1e-4, k


def test_chained_inference_installed_matches(tmp_path):
    res = _run('chained', str(tmp_path / 'chained.pt'))
    for graph in (False, True):
        err = _rel(res[(True, graph)], res[(False, graph)])
        print(f'chained graph={graph}: installed vs not, max rel diff {err:.2e}')
        assert err <= 2e-3
    assert _rel(res[(True, True)], res[(True, False)]) <= 1e-6
