"""Fused modulated convolution (torch_utils/ops/modulated_conv.py on lvg_modconv_*) on the GPU: every modulated-convolution
signature of the two generators against the reference definitions in float64, the unmodified generators with install()
against the reference on its own CUDA ops, CUDA graph replay, and the super-res G's peak memory."""
import math
import os
import subprocess
import sys

import pytest
import torch

from torch_utils.ops import conv_nd, modulated_conv as mc
from test_modconv_host import ref_modulated_conv2d, ref_temporal_modulated_conv3d

pytestmark = pytest.mark.gpu
DEV = 'cuda'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

# super-res G (generator_sres.py:325): per-sample (cin, cout, k, h, w, padding, fp16) of L0-L14 (workloads/sres_step.json)
SRES = [(27, 512, 3, 29, 36, 2, False), (539, 512, 3, 29, 36, 2, False), (539, 512, 3, 38, 52, 2, True), (539, 512, 3, 56, 84, 2, True),
        (539, 512, 3, 92, 148, 2, True), (539, 362, 3, 92, 148, 2, True), (389, 256, 3, 92, 148, 2, True), (283, 181, 3, 164, 276, 2, True),
        (208, 128, 3, 164, 276, 2, True), (155, 128, 3, 164, 276, 2, True), (155, 3, 1, 144, 256, 0, True)]
# low-res G (generator_lres.py:568,575,637): (cin, cout, kernel, h, w, padding) of conv0 / conv1 / ToRGB
LRES = [(512, 512, (3, 3, 3), 3, 4, (1, 1, 1)), (512, 512, (3, 3, 3), 5, 8, (1, 1, 1)), (512, 512, (3, 3, 3), 9, 16, (1, 1, 1)),
        (512, 256, (3, 3, 3), 9, 16, (1, 1, 1)), (256, 256, (3, 3, 3), 9, 16, (1, 1, 1)), (256, 256, (1, 3, 3), 9, 16, (0, 1, 1)),
        (256, 128, (1, 3, 3), 9, 16, (0, 1, 1)), (128, 128, (1, 3, 3), 18, 32, (0, 1, 1)), (128, 64, (1, 3, 3), 18, 32, (0, 1, 1)),
        (64, 64, (1, 3, 3), 36, 64, (0, 1, 1)), (64, 3, (1, 1, 1), 36, 64, (0, 0, 0))]


def rnd(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(tuple(shape), generator=g, device=DEV, dtype=torch.float64) * scale


def _run(fn, x, w, s, g, kw, dtype, dy):
    """y, dx, dw, ds of fn with x in `dtype` (fp32 weights / styles / gain, as the networks hold them)."""
    xa = x.to(dtype).requires_grad_(True)
    wa, sa = w.float().requires_grad_(True), s.float().requires_grad_(True)
    y = fn(xa, wa, sa, input_gain=g.float(), **kw)
    gx, gw, gs = torch.autograd.grad(y, [xa, wa, sa], dy.to(y.dtype))
    return [t.double() for t in (y.detach(), gx, gw, gs)]


def _exact(fn, x, w, s, g, kw, dy):
    xa, wa, sa = x.clone().requires_grad_(True), w.clone().requires_grad_(True), s.clone().requires_grad_(True)
    y = fn(xa, wa, sa, input_gain=g, **kw)
    return [y.detach()] + list(torch.autograd.grad(y, [xa, wa, sa], dy))


def _tols(fan):
    """the per-layer tolerances of tests/test_gpu_convnd.py by length of the sum: y and dx sum fan = Cin * taps products,
    dw and ds sum over every output pixel (always >= 4096 products here)"""
    short = 5e-5 if fan < 4096 else 2e-4
    return dict(y=short, dx=short, dw=2e-4, ds=2e-4)


def _rel(a, b):
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)


def _today_sres(x, w, s, demodulate=True, padding=0, input_gain=None):
    """the reference's per-sample formulation over this repository's engine (grouped conv_nd)."""
    f = ref_modulated_conv2d.__globals__['F']
    try:
        ref_modulated_conv2d.__globals__['F'] = conv_nd.functional
        return ref_modulated_conv2d(x, w, s, demodulate, padding, input_gain)
    finally:
        ref_modulated_conv2d.__globals__['F'] = f


def _today_lres(x, w, s, input_gain=None, padding=(0, 0, 0), demodulate=True):
    """the reference's formulation over this repository's engine (conv_nd.conv3d)."""
    f = ref_temporal_modulated_conv3d.__globals__['F']
    try:
        ref_temporal_modulated_conv3d.__globals__['F'] = conv_nd.functional
        return ref_temporal_modulated_conv3d(x, w, s, input_gain, padding, demodulate)
    finally:
        ref_temporal_modulated_conv3d.__globals__['F'] = f


@pytest.mark.parametrize('sig', SRES, ids=lambda c: f'{c[0]}-{c[1]}-k{c[2]}-{c[3]}x{c[4]}-{"f16" if c[6] else "f32"}')
def test_every_sres_signature(sig):
    cin, cout, k, h, wd, pad, fp16 = sig
    n = 2                                             # N*T samples
    x, w, s = rnd((n, cin, h, wd), 1), rnd((cout, cin, k, k), 2), rnd((n, cin), 3) + 1.0
    g = rnd((), 4).abs() + 0.5
    kw = dict(demodulate=k == 3, padding=pad)
    y = ref_modulated_conv2d(x, w, s, input_gain=g, **kw)
    dy = rnd(tuple(y.shape), 5)
    exact = _exact(ref_modulated_conv2d, x, w, s, g, kw, dy)
    dtype = torch.float16 if fp16 else torch.float32
    assert mc._native(x.to(dtype), w.to(dtype), (pad, pad))
    ours = _run(mc.modulated_conv2d, x, w, s, g, kw, dtype, dy)
    names = ('y', 'dx', 'dw', 'ds')
    if not fp16:
        tol = _tols(cin * k * k)
        for nm, a, b in zip(names, ours, exact):
            assert _rel(a, b) <= tol[nm], f'{nm}: {_rel(a, b):.3e}'
    else:
        today = _run(_today_sres, x, w, s, g, kw, dtype, dy)
        for nm, a, t, b in zip(names, ours, today, exact):
            assert _rel(a, b) <= 1.5 * _rel(t, b) + 1e-3, f'{nm}: fused {_rel(a, b):.3e}, today {_rel(t, b):.3e}'


@pytest.mark.parametrize('sig', LRES, ids=lambda c: f'{c[0]}-{c[1]}-k{"x".join(map(str, c[2]))}-{c[3]}x{c[4]}')
def test_every_lres_signature(sig):
    cin, cout, k, h, wd, pad = sig
    n, t = 1, 32
    x, w, s = rnd((n, cin, t, h, wd), 11), rnd((cout, cin) + k, 12), rnd((n, cin, t), 13)
    demod = cout != 3
    g = rnd((), 14).abs() + 0.5
    kw = dict(padding=pad, demodulate=demod)
    y = ref_temporal_modulated_conv3d(x, w, s, g, **kw)
    dy = rnd(tuple(y.shape), 15)
    exact = _exact(ref_temporal_modulated_conv3d, x, w, s, g, kw, dy)
    assert mc._native(x.float(), w.float(), pad)
    ours = _run(mc.temporal_modulated_conv3d, x, w, s, g, kw, torch.float32, dy)
    today = _run(_today_lres, x, w, s, g, kw, torch.float32, dy)
    tol = _tols(cin * math.prod(k))
    for nm, a, t, b in zip(('y', 'dx', 'dw', 'ds'), ours, today, exact):
        if nm in ('dw', 'ds') and demod:
            # demodulation makes y invariant to each output channel's weight scale and (with the amax normalisation) to
            # each sample's style scale: the raw weight's and style's gradients are what is left after the normalisations'
            # terms cancel, so the engine's ~2^-16 product error shows up magnified, in today's path as much as here --
            # judged against it as the fp16 calls are
            assert _rel(a, b) <= 1.5 * _rel(t, b) + 1e-5, f'{nm}: fused {_rel(a, b):.3e}, today {_rel(t, b):.3e}'
        else:
            assert _rel(a, b) <= tol[nm], f'{nm}: fused {_rel(a, b):.3e}, today {_rel(t, b):.3e}'


def test_cuda_graph_replay_is_bit_identical():
    x = rnd((4, 64, 20, 24), 21).half()
    w, s, g = rnd((96, 64, 3, 3), 22).float().requires_grad_(True), (rnd((4, 64), 23) + 1).float().requires_grad_(True), torch.tensor(0.7, device=DEV)
    dy = rnd((4, 96, 20, 24), 24).half()
    xs = x.clone().requires_grad_(True)

    def step():
        y = mc.modulated_conv2d(xs, w, s, padding=1, input_gain=g)
        gx, gw, gsty = torch.autograd.grad(y, [xs, w, s], dy)
        return y, gx, gw, gsty
    s_ = torch.cuda.Stream()
    s_.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s_):
        for _ in range(2):
            eager = [t.detach().clone() for t in step()]
    torch.cuda.current_stream().wait_stream(s_)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(outs, eager):
        assert torch.equal(a, b)


# ---- the unmodified generators with install()

def _net(tmp, name, ref_plugins=False, install=False, fp32=False):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([SRC] if ref_plugins else [PKG, SRC]), LVG_REF_PLUGINS='1' if ref_plugins else '0',
               LVG_MODCONV_INSTALL='1' if install else '0', LVG_FP32='1' if fp32 else '0')
    out = str(tmp / (name + '.pt'))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'modconv_dropin_run.py'), out], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out)


@pytest.fixture(scope='module')
def nets(tmp_path_factory):
    if not os.path.isdir(os.path.join(SRC, 'model')):
        pytest.skip('oracle/_ref not staged')
    d = tmp_path_factory.mktemp('modconv')
    return dict(ours=_net(d, 'ours', install=True), plain=_net(d, 'plain'), theirs=_net(d, 'ref', ref_plugins=True),
                truth=_net(d, 'ref32', ref_plugins=True, fp32=True))


def test_install_patched_both_generators(nets):
    assert sorted(nets['ours']['installed']) == ['model.generator_lres', 'model.generator_sres'] and nets['plain']['installed'] == []


# the tolerances of tests/test_gpu_dropin_cuda.py
@pytest.mark.parametrize('key,tol_max,tol_l2', [('lres_G', 1e-3, 5e-4), ('lres_G_grad', 3e-2, 2e-2)])
def test_lres_generator_with_install_matches_reference_cuda(nets, key, tol_max, tol_l2):
    a, b = nets['ours'][key].double(), nets['theirs'][key].double()
    assert a.shape == b.shape and torch.isfinite(a).all()
    emax, el2 = float((a - b).abs().max() / b.abs().max()), float((a - b).norm() / b.norm())
    assert emax <= tol_max and el2 <= tol_l2, f'{key}: max {emax:.3e}, L2 {el2:.3e}'


@pytest.mark.parametrize('key', ['sres_G', 'sres_G_grad'])
def test_sres_generator_with_install_is_as_close_to_fp32_as_the_reference(nets, key):
    a, b, t = nets['ours'][key].double(), nets['theirs'][key].double(), nets['truth'][key].double()
    assert a.shape == t.shape and torch.isfinite(a).all()
    e_ours, e_ref = float((a - t).norm() / t.norm()), float((b - t).norm() / t.norm())
    m_ours, m_ref = float((a - t).abs().max() / t.abs().max()), float((b - t).abs().max() / t.abs().max())
    assert e_ours <= 1.5 * e_ref + 2e-3, f'{key}: L2 error vs fp32 {e_ours:.3e} (reference fp16: {e_ref:.3e})'
    assert m_ours <= 1.5 * m_ref + 5e-3, f'{key}: max error vs fp32 {m_ours:.3e} (reference fp16: {m_ref:.3e})'


def test_sres_generator_peak_memory_is_lower_with_install(nets):
    assert nets['ours']['sres_peak_bytes'] < nets['plain']['sres_peak_bytes'], (nets['ours']['sres_peak_bytes'], nets['plain']['sres_peak_bytes'])
