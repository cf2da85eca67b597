"""Host logic of torch_utils/ops/modulated_conv.py on CPU: a float64 torch-backed stand-in for the convnd plugin applies the
input factor a and the output factor d exactly where the kernels do (x * a before the convolution, d on its result), and the
fused op, its gradients for x, w, s and input_gain, its create_graph path, the no_weight_gradients switch, the composition
outside the envelope and install() are checked against the reference definitions written out below in float64."""
import math
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from torch_utils.ops import conv2d_gradfix, conv_nd, modulated_conv as mc


def ref_modulated_conv2d(x, w, s, demodulate=True, padding=0, input_gain=None):
    """generator_sres.modulated_conv2d: per-sample weights, one grouped convolution."""
    n, cin = x.shape[:2]
    cout, _, kh, kw = w.shape
    if demodulate:
        w = w * w.square().mean([1, 2, 3], keepdim=True).rsqrt()
        s = s * s.square().mean().rsqrt()
    w = w.unsqueeze(0) * s.unsqueeze(1).unsqueeze(3).unsqueeze(4)
    if demodulate:
        w = w * (w.square().sum(dim=[2, 3, 4]) + 1e-8).rsqrt().unsqueeze(2).unsqueeze(3).unsqueeze(4)
    if input_gain is not None:
        w = w * input_gain.expand(n, cin).unsqueeze(1).unsqueeze(3).unsqueeze(4)
    y = F.conv2d(x.reshape(1, -1, *x.shape[2:]), w.reshape(-1, cin, kh, kw).to(x.dtype), padding=padding, groups=n)
    return y.reshape(n, -1, *y.shape[2:])


def ref_temporal_modulated_conv3d(x, weight, style, input_gain=None, padding=(0, 0, 0), demodulate=True):
    """generator_lres.temporal_modulated_conv3d."""
    if demodulate:
        weight = weight / weight.abs().amax(dim=(1, 2, 3, 4), keepdim=True)
        style = style / style.abs().amax(dim=(1, 2), keepdim=True)
    weight = weight / math.sqrt(int(np.prod(weight.shape[1:])))
    if demodulate:
        dm = torch.einsum('oizyx,nit->not', weight.square(), style.square()).add(1e-8).rsqrt()[..., None, None]
    if input_gain is not None:
        x = x * input_gain
    y = F.conv3d(x * style[..., None, None].type(x.dtype), weight.type(x.dtype), padding=padding)
    return y * dm.type(y.dtype) if demodulate else y


class TorchBackedPlugin:
    """convnd_plugin stand-in (float64 CPU torch arithmetic). Test-only."""

    def __init__(self):
        self.calls = dict(fprop=0, dgrad=0, wgrad=0, backward=0, modconv_fprop=0, modconv_backward=0)

    def supported(self, x, w, stride, padding, dilation, groups):
        return x.ndim in (3, 4, 5)

    def modconv_supported(self, x, w, padding):
        return True

    @staticmethod
    def _conv(nd):
        return (F.conv1d, F.conv2d, F.conv3d)[nd - 1]

    @staticmethod
    def _bc(f, nd):
        return f[..., None, None] if nd == 3 else f[..., None]

    def fprop(self, x, w, padding, groups, stride=1, **kw):
        self.calls['fprop'] += 1
        return self._conv(x.ndim - 2)(x, w, None, 1, padding, 1, groups)

    def dgrad(self, dy, w, x_shape, padding, groups, stride=1):
        self.calls['dgrad'] += 1
        x = torch.zeros(x_shape, dtype=dy.dtype, requires_grad=True)
        with torch.enable_grad():
            return torch.autograd.grad(self._conv(dy.ndim - 2)(x, w, None, 1, padding, 1, groups), [x], dy)[0]

    def wgrad(self, x, dy, w_shape, padding, groups, stride=1):
        self.calls['wgrad'] += 1
        w = torch.zeros(w_shape, dtype=x.dtype, requires_grad=True)
        with torch.enable_grad():
            return torch.autograd.grad(self._conv(x.ndim - 2)(x, w, None, 1, padding, 1, groups), [w], dy)[0]

    def modconv_fprop(self, x, w, a, d, padding):
        self.calls['modconv_fprop'] += 1
        nd = x.ndim - 2
        y = self._conv(nd)(x * self._bc(a, nd), w, None, 1, padding)
        return y if d is None else y * self._bc(d, nd)

    def modconv_backward(self, x, w, a, d, y, dy, padding, want_dw=True):
        self.calls['modconv_backward'] += 1
        nd = x.ndim - 2
        dyd = dy if d is None else dy * self._bc(d, nd)
        dxp = torch.nn.grad.conv2d_input(x.shape, w, dyd, padding=padding) if nd == 2 else torch.nn.grad.conv3d_input(x.shape, w, dyd, padding=padding)
        xa = x * self._bc(a, nd)
        dw = None
        if want_dw:
            dw = torch.nn.grad.conv2d_weight(xa, w.shape, dyd, padding=padding) if nd == 2 else torch.nn.grad.conv3d_weight(xa, w.shape, dyd, padding=padding)
        da = mc._spatial_dot(dxp, x, nd)
        dyy = None if d is None else mc._spatial_dot(dy, y, nd)
        return dxp * self._bc(a, nd), dw, da, dyy


@pytest.fixture
def plug(monkeypatch):
    p = TorchBackedPlugin()
    monkeypatch.setattr(conv_nd, '_plugin', p)
    monkeypatch.setattr(conv_nd, 'enabled_for', lambda x: True)
    monkeypatch.setattr(mc, '_native', lambda x, w, padding: True)
    return p


def rnd(*shape, seed):
    return torch.randn(tuple(shape), generator=torch.Generator().manual_seed(seed), dtype=torch.float64)


def _gain(form, n, cin, seed):
    return {None: None, 'scalar': rnd(seed=seed).abs() + 0.5, 'cin': rnd(cin, seed=seed) + 1.5, 'n_cin': rnd(n, cin, seed=seed) + 1.5}[form]


def _check(fn, ref, args, kwargs, diff, tol=1e-9):
    """forward + gradients of every tensor in `diff` (indices into args / names in kwargs) against ref."""
    outs = []
    for f in (fn, ref):
        a = [t.clone().requires_grad_(True) if i in diff and t is not None else t for i, t in enumerate(args)]
        k = {n: (t.clone().requires_grad_(True) if n in diff and t is not None else t) for n, t in kwargs.items()}
        y = f(*a, **k)
        v = rnd(*y.shape, seed=99)
        leaves = [a[i] for i in diff if isinstance(i, int)] + [k[n] for n in diff if isinstance(n, str) and k[n] is not None]
        outs.append([y.detach()] + list(torch.autograd.grad((y * v).sum(), leaves)))
    for g, r in zip(*outs):
        assert float((g - r).abs().max()) <= tol * max(float(r.abs().max()), 1e-30)


@pytest.mark.parametrize('demodulate', [True, False])
@pytest.mark.parametrize('gain', [None, 'scalar', 'cin', 'n_cin'])
@pytest.mark.parametrize('k,pad', [(1, 0), (3, 1)])
def test_modulated_conv2d_matches_reference(plug, demodulate, gain, k, pad):
    n, cin, cout = 3, 5, 4
    x, w, s = rnd(n, cin, 7, 6, seed=1), rnd(cout, cin, k, k, seed=2), rnd(n, cin, seed=3)
    g = _gain(gain, n, cin, 4)
    if gain == 'scalar':
        g = g.reshape([])
    _check(mc.modulated_conv2d, ref_modulated_conv2d, (x, w, s), dict(demodulate=demodulate, padding=pad, input_gain=g), (0, 1, 2, 'input_gain'))
    assert plug.calls['modconv_fprop'] == 1 and plug.calls['modconv_backward'] == 1


@pytest.mark.parametrize('demodulate', [True, False])
@pytest.mark.parametrize('gain', [None, 'scalar'])
@pytest.mark.parametrize('k,pad', [((1, 1, 1), (0, 0, 0)), ((1, 3, 3), (0, 1, 1)), ((3, 3, 3), (1, 1, 1))])
def test_temporal_modulated_conv3d_matches_reference(plug, demodulate, gain, k, pad):
    n, cin, cout, t = 2, 4, 3, 5
    x, w, s = rnd(n, cin, t, 6, 5, seed=5), rnd(cout, cin, *k, seed=6), rnd(n, cin, t, seed=7)
    g = None if gain is None else _gain('scalar', n, cin, 8).reshape([])
    _check(mc.temporal_modulated_conv3d, ref_temporal_modulated_conv3d, (x, w, s), dict(input_gain=g, padding=pad, demodulate=demodulate),
           (0, 1, 2, 'input_gain'))
    assert plug.calls['modconv_fprop'] == 1 and plug.calls['modconv_backward'] == 1


@pytest.mark.parametrize('nd', [2, 3])
def test_create_graph_path_is_differentiable(plug, nd):
    """With create_graph=True the backward pass is recorded from differentiable Functions: gradcheck / gradgradcheck of the
    fused Function itself, and no native first-order call."""
    if nd == 2:
        x, w, a, d, pad = rnd(2, 3, 5, 4, seed=11), rnd(2, 3, 3, 3, seed=12), rnd(2, 3, 1, seed=13), rnd(2, 2, 1, seed=14).abs() + 0.5, (1, 1)
    else:
        x, w, a, d, pad = rnd(2, 3, 3, 4, 4, seed=11), rnd(2, 3, 3, 3, 3, seed=12), rnd(2, 3, 3, seed=13), rnd(2, 2, 3, seed=14).abs() + 0.5, (1, 1, 1)
    args = tuple(t.requires_grad_(True) for t in (x, w, a, d))
    f = lambda x, w, a, d: mc._ModulatedConv.apply(x, w, a, d, pad)       # noqa: E731
    assert torch.autograd.gradgradcheck(f, args)
    n0 = plug.calls['modconv_backward']
    y = f(*args)
    gs = torch.autograd.grad(y.square().sum(), args, create_graph=True)
    assert plug.calls['modconv_backward'] == n0 and all(g.requires_grad for g in gs)


def test_no_weight_gradients(plug):
    x, w, s = rnd(2, 3, 6, 6, seed=21).requires_grad_(True), rnd(4, 3, 3, 3, seed=22).requires_grad_(True), rnd(2, 3, seed=23).requires_grad_(True)
    with conv2d_gradfix.no_weight_gradients():
        y = mc.modulated_conv2d(x, w, s, padding=1)
        gx, gs, gw = torch.autograd.grad(y.sum(), [x, s, w], allow_unused=True)
    assert gx is not None and gs is not None
    # the weight still reaches y through the demodulation coefficients: only the convolution's own dw is skipped
    gd = torch.autograd.grad(ref_modulated_conv2d(x, w.detach(), s, padding=1).sum(), [x])[0]
    assert torch.allclose(gx, gd, rtol=1e-9, atol=1e-12)


def test_outside_the_envelope_takes_the_composition(monkeypatch):
    """CPU float64 with the real envelope check: no plugin call, the reference's own formulation over conv_nd."""
    called = []
    monkeypatch.setattr(mc, 'modulated_conv', lambda *a, **k: called.append(1))
    x, w, s = rnd(2, 3, 6, 6, seed=31), rnd(4, 3, 3, 3, seed=32), rnd(2, 3, seed=33)
    assert torch.equal(mc.modulated_conv2d(x, w, s, padding=1), ref_modulated_conv2d(x, w, s, padding=1))
    x3, w3, s3 = rnd(2, 3, 4, 5, 5, seed=34), rnd(4, 3, 3, 3, 3, seed=35), rnd(2, 3, 4, seed=36)
    g = torch.tensor(0.7, dtype=torch.float64)
    r = ref_temporal_modulated_conv3d(x3, w3, s3, g, (1, 1, 1))
    assert torch.equal(mc.temporal_modulated_conv3d(x3, w3, s3, g, (1, 1, 1)), r)
    assert not called


def _fake_reference_module(name):
    mod = types.ModuleType(name)

    def modulated_conv2d(*a, **k):
        return 'reference'

    def temporal_modulated_conv3d(*a, **k):
        return 'reference'
    mod.modulated_conv2d = modulated_conv2d
    mod.temporal_modulated_conv3d = temporal_modulated_conv3d
    mod.F = F
    return mod


def test_install_patches_modules_idempotently_and_leaves_F(monkeypatch):
    sres, lres = _fake_reference_module('fake_sres'), _fake_reference_module('fake_lres')
    lres.other = lambda: None
    assert mc.install(sres, lres) == [sres, lres]
    assert sres.modulated_conv2d is mc.modulated_conv2d and lres.temporal_modulated_conv3d is mc.temporal_modulated_conv3d
    assert sres.F is F and lres.F is F
    assert mc.install(sres, lres) == [sres, lres]               # idempotent
    assert sres.modulated_conv2d is mc.modulated_conv2d
    assert mc.install(types.ModuleType('unrelated')) == []
    unrelated = types.ModuleType('unrelated2')
    unrelated.modulated_conv2d = lambda *a: None                # a different function of that name is not the reference's
    unrelated.modulated_conv2d.__name__ = '<lambda>'
    assert mc.install(unrelated) == []


def test_install_reaches_unpickled_instances_through_sys_modules(monkeypatch):
    """persistence execs a pickled class's source into a module of its own: the instance's type names that module."""
    mod = _fake_reference_module('_imported_module_for_test')
    src = 'import torch\nclass Block(torch.nn.Module):\n    def forward(self, x):\n        return modulated_conv2d(x)\n'
    exec(compile(src, '<persisted>', 'exec'), mod.__dict__)
    monkeypatch.setitem(sys.modules, mod.__name__, mod)
    net = torch.nn.Sequential(mod.Block(), torch.nn.Linear(1, 1))
    assert net[0](None) == 'reference'
    done = mc.install(net)
    assert done == [mod] and mod.modulated_conv2d is mc.modulated_conv2d
    assert mc.install(net) == [mod]
