"""Host logic of torch_utils/ops/dblock_tail.py on the CPU: the composition path against an independent float64 evaluation of
the definition; the installed DiscriminatorBlock.forward against the UNMODIFIED reference method bit for bit (output,
gradients, the R1 pattern) for every block of the default discriminator and of one without temporal / spatial
downsampling; the three autograd Functions wired over a torch stand-in for the plugin (gradcheck and gradgradcheck in
float64); install()'s conventions; and the ABI's size queries, which answer without a GPU."""
import math
import os
import subprocess
import sys

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import bias_act, conv_nd
from torch_utils.ops import dblock_tail as dt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
P = custom_ops.DblockTailPlugin

needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')


def down64(x, dim, f):
    """Downsample3d's filter along dim, from the definition: out[m] = sum_j f[3 - j] in[2 m - 1 + j], zero outside."""
    n = x.shape[dim]
    xp = torch.nn.functional.pad(x, [0, 0] * (x.ndim - 1 - dim) + [1, 2])
    idx = torch.arange(n // 2) * 2
    return sum(float(f[3 - j]) * xp.index_select(dim, idx + j) for j in range(4))


def tail64(y, s, b, f, sd, td, act, alpha, gain, clamp):
    """The definition in the dtype of y, independent of upfirdn2d and bias_act. Returns (z, slope G)."""
    v = y
    if sd:
        v = down64(down64(v, 3, f), 4, f)
    if td:
        v = down64(v, 2, f)
    if b is not None:
        v = v + b.view(1, -1, 1, 1, 1)
    a = alpha if act == 'lrelu' else 1.0
    o = torch.where(v > 0, v, v * a) * gain
    g = torch.where(v > 0, gain, gain * a) * torch.ones_like(v)
    if clamp is not None:
        g = torch.where(o.abs() < clamp, g, torch.zeros_like(g))
        o = o.clamp(-clamp, clamp)
    if s is not None:
        o = (o + s) * math.sqrt(0.5)
    return o, g


F4 = torch.tensor([0.125, 0.375, 0.375, 0.125])


@pytest.mark.parametrize('sd,td', [(False, False), (True, False), (False, True), (True, True)])
@pytest.mark.parametrize('act', ['lrelu', 'linear'])
@pytest.mark.parametrize('has_b,has_s,clamp', [(True, True, 2.0), (False, True, None), (True, False, 2.0), (False, False, None)])
def test_composition_matches_the_definition(sd, td, act, has_b, has_s, clamp):
    g = torch.Generator().manual_seed(1)
    y = torch.randn(2, 3, 6, 8, 10, generator=g, dtype=torch.float64) * 3
    out = (6 // (1 + td), 8 // (1 + sd), 10 // (1 + sd))
    s = torch.randn(2, 3, *out, generator=g, dtype=torch.float64) if has_s else None
    b = torch.randn(3, generator=g, dtype=torch.float64) if has_b else None
    z = dt.dblock_tail(y, s, b, F4, spatial_down=sd, temporal_down=td, act=act, clamp=clamp)
    want, _ = tail64(y, s, b, F4, sd, td, act, 0.2, math.sqrt(2) if act == 'lrelu' else 1.0, clamp)
    assert z.shape == want.shape and z.dtype == torch.float64
    assert torch.allclose(z, want, rtol=1e-12, atol=1e-12)


# ---- the installed block against the reference method

def _run(mode, out_file):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'dblock_tail_run.py'), out_file, mode], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out_file, weights_only=False)


@needs_ref
def test_installed_block_equals_the_reference_block_bit_for_bit(tmp_path):
    res = _run('cpu', str(tmp_path / 'cpu.pt'))
    assert len(res) == 2 * 4 * 2
    downs = set()
    for r in res:
        downs.add(r['down'])
        assert r['took'] == 1, r['cfg']                      # the installed forward ran the tail, not the original method
        assert len(r['ours']) == len(r['ref']) >= 6
        for a, b in zip(r['ours'], r['ref']):
            assert a.shape == b.shape and torch.equal(a, b), f'{r["cfg"]}: {float((a - b).abs().max()):.3e}'
    assert downs == {(True, False), (True, True), (False, False)}


@needs_ref
@pytest.mark.parametrize('mode', ['install_a', 'install_b'])
def test_install_conventions_and_composition_with_conv3d_down(tmp_path, mode):
    assert _run(mode, str(tmp_path / 'install.pt')) == 'ok'


# ---- wiring of the three Functions over a torch stand-in for the plugin

class StandIn:
    """The plugin's two calls in torch ops, any dtype and device. Its codes are one byte per output."""

    @staticmethod
    def _p(x, flags, f):
        if flags & P.SDOWN:
            x = down64(down64(x, 3, f), 4, f)
        if flags & P.TDOWN:
            x = down64(x, 2, f)
        return x

    @staticmethod
    def _slope(codes, act, alpha, gain, like):
        a = alpha if act == 3 else 1.0
        g = torch.where((codes & 1).bool(), gain * a, gain) * torch.ones_like(like)
        return torch.where((codes & 2).bool(), torch.zeros_like(g), g)

    def forward(self, y, s, b, f, flags, act, alpha, gain, clamp, mode, codes=None):
        scale = math.sqrt(0.5) if flags & P.MERGE else 1.0
        v = self._p(y, flags, f)
        if b is not None:
            v = v + b.view(1, -1, 1, 1, 1)
        if mode == P.READ:
            o = v * self._slope(codes, act, alpha, gain, v)
        else:
            o = torch.where(v > 0, v, v * (alpha if act == 3 else 1.0)) * gain
            codes = (~(o > 0)).to(torch.uint8)
            if clamp >= 0:
                codes = codes | ((~(o.abs() < clamp)).to(torch.uint8) << 1)
                o = o.clamp(-clamp, clamp)
            codes = codes if mode == P.WRITE else None
        if s is not None:
            o = o + s
        return o * scale, codes

    def adjoint(self, dz, codes, f, in_size, flags, act, alpha, gain, want_ds):
        scale = math.sqrt(0.5) if flags & P.MERGE else 1.0
        dv = dz * scale * self._slope(codes, act, alpha, gain, dz)
        with torch.enable_grad():
            x0 = torch.zeros([*dz.shape[:2], *in_size], dtype=dz.dtype, requires_grad=True)
            dy, = torch.autograd.grad(self._p(x0, flags, f), [x0], dv)
        return dy, (dz * scale if want_ds else None), dv.sum((0, 2, 3, 4))


@pytest.fixture
def standin(monkeypatch):
    monkeypatch.setattr(dt, '_plugin', lambda: StandIn())


def _wiring_inputs(flags, seed=0):
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(1, 2, 4, 4, 6, generator=g, dtype=torch.float64, requires_grad=True)
    out = P.out_size((4, 4, 6), flags)
    s = torch.randn(1, 2, *out, generator=g, dtype=torch.float64, requires_grad=True) if flags & P.MERGE else None
    b = torch.randn(2, generator=g, dtype=torch.float64, requires_grad=True)
    return y, s, b


@pytest.mark.parametrize('flags', [P.MERGE, P.MERGE | P.SDOWN, P.MERGE | P.TDOWN | P.SDOWN, P.TDOWN])
@pytest.mark.parametrize('act', [3, 1])
def test_functions_gradcheck_and_gradgradcheck(standin, flags, act):
    y, s, b = _wiring_inputs(flags)
    f = F4.double()
    cfg = (flags, act, 0.2, 1.5, 1.0)
    if s is None:
        fn, lin, args = (lambda y_, b_: dt._Tail.apply(y_, None, b_, f, cfg)), None, (y, b)
    else:
        fn, lin, args = (lambda y_, s_, b_: dt._Tail.apply(y_, s_, b_, f, cfg)), None, (y, s, b)
    # the map is piecewise linear: inputs away from its kinks by more than the probe step
    v, _ = StandIn().forward(y.detach(), None, b.detach(), f, flags & ~P.MERGE, 1, 0.0, 1.0, -1.0, P.NONE)
    o = torch.where(v > 0, v, v * (0.2 if act == 3 else 1.0)) * 1.5
    assert (v.abs() > 1e-4).all() and ((o.abs() - 1.0).abs() > 1e-4).all()
    assert torch.autograd.gradcheck(fn, args, eps=1e-6, atol=1e-7)
    assert torch.autograd.gradgradcheck(fn, args, eps=1e-6, atol=1e-7)
    # the adjoint and the read-mode map on their own, and as each other's transpose
    _, codes = StandIn().forward(y.detach(), s if s is None else s.detach(), b.detach(), f, flags, act, 0.2, 1.5, 1.0, P.WRITE)
    dz = torch.randn(1, 2, *P.out_size((4, 4, 6), flags), dtype=torch.float64, requires_grad=True)
    adj = lambda d: tuple(o for o in dt._TailAdjoint.apply(d, codes, f, cfg, (4, 4, 6), s is not None) if o is not None)   # noqa: E731
    assert torch.autograd.gradcheck(adj, (dz,), eps=1e-6, atol=1e-7)
    assert torch.autograd.gradgradcheck(adj, (dz,), eps=1e-6, atol=1e-7)
    if s is None:
        lin = lambda u, bt: dt._TailLinear.apply(u, None, bt, codes, f, cfg)        # noqa: E731
    else:
        lin = lambda u, sg, bt: dt._TailLinear.apply(u, sg, bt, codes, f, cfg)      # noqa: E731
    assert torch.autograd.gradcheck(lin, args, eps=1e-6, atol=1e-7)
    u = torch.randn_like(y)
    lhs = (dt._TailLinear.apply(u, None, None, codes, f, cfg) * dz).sum().detach()
    rhs = (dt._TailAdjoint.apply(dz, codes, f, cfg, (4, 4, 6), False)[0] * u).sum().detach()
    assert abs(float(lhs - rhs)) <= 1e-12 * max(1.0, abs(float(lhs)))


def test_tail_matches_the_composition_through_second_order(standin):
    flags = P.MERGE | P.TDOWN | P.SDOWN
    y, s, b = _wiring_inputs(flags, seed=4)
    outs = []
    for fused in (True, False):
        if fused:
            z = dt._Tail.apply(y, s, b, F4.double(), (flags, 3, 0.2, math.sqrt(2), 1.0))
        else:
            z = dt._reference(y, s, b, F4, True, True, 'lrelu', 1.0)
        gy, gs = torch.autograd.grad(z.square().sum(), [y, s], create_graph=True)
        gg = torch.autograd.grad(gy.square().sum() + gs.sum() + z.sum(), [y, s, b])
        outs.append((z.detach(), gy.detach(), gs.detach()) + gg)
    for a, bb in zip(*outs):
        assert torch.allclose(a, bb, rtol=1e-6, atol=1e-7)        # the composition's own backward carries float32 constants


def test_only_the_codes_and_the_filter_are_saved(standin):
    y, s, b = _wiring_inputs(P.MERGE | P.SDOWN)
    saved = []
    with torch.autograd.graph.saved_tensors_hooks(lambda t: (saved.append(t), t)[1], lambda t: t):
        dt._Tail.apply(y, s, b, F4.double(), (P.MERGE | P.SDOWN, 3, 0.2, 1.0, -1.0))
    assert sorted(t.dtype == torch.uint8 for t in saved) == [False, True] and min(t.numel() for t in saved) == 4


# ---- conv_bias_act: gradients of any order, with torch stand-ins for the convolution and bias_act plugins

class ConvStandIn:
    """convnd_plugin's calls in torch ops (float64 CPU); fprop applies the epilogue."""

    def supported(self, x, w, stride, padding, dilation, groups):
        return True

    def fprop(self, x, w, padding, groups, bias=None, act=0, alpha=0.2, gain=1.0, clamp=-1.0, stride=1):
        y = torch.nn.functional.conv3d(x, w, None, 1, padding, 1, groups)
        if act == 0:
            return y
        return bias_act._bias_act_ref(y, bias, act='lrelu' if act == 2 else 'linear', alpha=alpha, gain=gain,
                                      clamp=None if clamp < 0 else clamp)

    def dgrad(self, dy, w, x_shape, padding, groups, stride=1):
        with torch.enable_grad():
            x = torch.zeros(x_shape, dtype=dy.dtype, requires_grad=True)
            return torch.autograd.grad(torch.nn.functional.conv3d(x, w, None, 1, padding, 1, groups), [x], dy)[0]

    def wgrad(self, x, dy, w_shape, padding, groups, stride=1):
        with torch.enable_grad():
            w = torch.zeros(w_shape, dtype=x.dtype, requires_grad=True)
            return torch.autograd.grad(torch.nn.functional.conv3d(x, w, None, 1, padding, 1, groups), [w], dy)[0]

    def backward(self, x, dy, w, padding, groups, stride=1):
        return self.dgrad(dy, w, tuple(x.shape), padding, groups), self.wgrad(x, dy, tuple(w.shape), padding, groups)


class BiasActStandIn:
    """bias_act_plugin.bias_act for grad = 1 with yref: dx = dy * gain * act'(.), zero where yref is clamped."""

    @staticmethod
    def bias_act(x, b, xref, yref, dy, grad, dim, act, alpha, gain, clamp):
        assert grad == 1 and b is None and xref is None and dy is None and act in (1, 3)
        slope = torch.where(yref > 0, 1.0, alpha if act == 3 else 1.0) * gain
        if clamp >= 0:
            slope = torch.where(yref.abs() < clamp, slope, torch.zeros_like(slope))
        return x * slope


@pytest.fixture
def conv_standins(monkeypatch):
    monkeypatch.setattr(conv_nd, '_plugin', ConvStandIn())
    monkeypatch.setattr(conv_nd, 'enabled_for', lambda x: True)
    monkeypatch.setattr(bias_act, '_plugin', BiasActStandIn())
    monkeypatch.setattr(bias_act, '_init', lambda: True)


@pytest.mark.parametrize('act,clamp', [('lrelu', 0.6), ('linear', None), ('lrelu', None)])
def test_conv_bias_act_second_order_matches_the_two_ops(conv_standins, act, clamp):
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 3, 3, 5, 4, generator=g, dtype=torch.float64, requires_grad=True)
    w = (torch.randn(4, 3, 3, 3, 3, generator=g, dtype=torch.float64) * 0.2).requires_grad_(True)
    b = torch.randn(4, generator=g, dtype=torch.float64, requires_grad=True)
    outs = []
    for fused in (True, False):
        if fused:
            y = conv_nd.conv_bias_act(x, w, b, padding=(1, 1, 1), act=act, clamp=clamp)
            assert type(y.grad_fn).__name__ == '_ConvBiasActBackward'
        else:
            y = bias_act._bias_act_ref(torch.nn.functional.conv3d(x, w, padding=1), b, act=act, clamp=clamp)
        gx, gw, gb = torch.autograd.grad(y.square().sum(), [x, w, b], create_graph=True)
        gg = torch.autograd.grad(gx.square().sum() + gw.square().sum() + gb.square().sum(), [x, w, b])       # the R1 pattern
        outs.append((y.detach(), gx.detach(), gw.detach(), gb.detach()) + gg)
    for a, bb in zip(*outs):
        assert float((a - bb).abs().max()) <= 1e-6 * float(bb.abs().max())     # torch's leaky_relu backward carries its slope in float32
    fn = lambda x_, w_, b_: conv_nd.conv_bias_act(x_, w_, b_, padding=(1, 1, 1), act=act, clamp=clamp)        # noqa: E731
    assert torch.autograd.gradcheck(fn, (x, w, b), eps=1e-6, atol=1e-6)
    assert torch.autograd.gradgradcheck(fn, (x, w, b), eps=1e-6, atol=1e-6)


def test_conv_bias_act_first_order_is_the_same_with_and_without_create_graph(conv_standins):
    g = torch.Generator().manual_seed(6)
    x = torch.randn(1, 2, 3, 4, 4, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(3, 2, 1, 3, 3, generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(3, generator=g, dtype=torch.float64, requires_grad=True)
    y = conv_nd.conv_bias_act(x, w, b, padding=(0, 1, 1), act='lrelu', clamp=1.0)
    a = torch.autograd.grad(y.sum(), [x, w, b], retain_graph=True)
    c = torch.autograd.grad(y.sum(), [x, w, b], create_graph=True)
    assert all(torch.equal(p, q.detach()) for p, q in zip(a, c)) and all(q.requires_grad for q in c[:2])


# ---- the ABI without a GPU

def test_size_queries_and_envelope():
    lib = custom_ops.load_library()
    # y [8, 64, 128, 64, 64], H and W halved: one byte per 4 outputs along W, 8 x 2 tiles of 8 x 32 per full-resolution plane
    assert lib.lvg_dblock_tail_codes_bytes(8, 64, 128, 64, 64, P.SDOWN | P.MERGE) == 8 * 64 * 128 * 32 * 8
    assert lib.lvg_dblock_tail_workspace(8, 64, 128, 64, 64, P.SDOWN | P.MERGE) == 8 * 64 * 16 * 4
    assert lib.lvg_dblock_tail_codes_bytes(2, 3, 4, 6, 10, P.TDOWN | P.SDOWN) == 2 * 3 * 2 * 3 * 2        # rows padded to 2 bytes
    assert lib.lvg_dblock_tail_codes_bytes(1, 1, 3, 5, 7, 0) == 3 * 5 * 2
    assert lib.lvg_dblock_tail_workspace(1, 3, 1, 1, 1, 0) == 16                                          # rounded up to 16 bytes
    for bad in ((1, 1, 3, 4, 4, P.TDOWN), (1, 1, 4, 5, 4, P.SDOWN), (1, 1, 4, 4, 5, P.SDOWN), (0, 1, 4, 4, 4, 0), (1, 1, 4, 4, 4, 8),
                (1, 1, 2, 8 * 300, 32 * 300, 0)):
        assert lib.lvg_dblock_tail_codes_bytes(*bad) == -1 and lib.lvg_dblock_tail_workspace(*bad) == -1, bad
    # out of the envelope and bad arguments never launch
    assert lib.lvg_dblock_tail(1, None, None, 1, 1, None, 0, 0, 1, 1, 3, 4, 4, P.TDOWN, 3, 0.2, 1.0, -1.0, None) == -1
    assert lib.lvg_dblock_tail(1, None, None, 1, 1, None, 0, 0, 1, 1, 4, 4, 4, 0, 2, 0.2, 1.0, -1.0, None) == -1       # relu
    assert lib.lvg_dblock_tail(None, None, None, 1, 1, None, 0, 0, 1, 1, 4, 4, 4, 0, 3, 0.2, 1.0, -1.0, None) == 1
    assert b'NULL' in lib.lvg_last_error()
    assert lib.lvg_dblock_tail(1, None, None, 1, 1, None, 1, 0, 1, 1, 4, 4, 4, 0, 3, 0.2, 1.0, -1.0, None) == 1         # write, no codes
    assert lib.lvg_dblock_tail(1, 1, None, 1, 1, None, 0, 0, 1, 1, 4, 4, 4, 0, 3, 0.2, 1.0, -1.0, None) == 1            # s without MERGE
    assert lib.lvg_dblock_tail_adjoint(1, 1, 1, 1, None, 1, 1, 8, 0, 1, 1, 4, 4, 4, 0, 3, 0.2, 1.0, None) == 1          # workspace too small
    assert b'workspace' in lib.lvg_last_error()


def test_cpu_tensors_never_reach_the_plugin():
    with pytest.raises(RuntimeError, match='CUDA'):
        custom_ops.get_plugin('dblock_tail_plugin').forward(torch.zeros(1, 1, 2, 2, 2), None, None, F4, 0, 3, 0.2, 1.0, -1.0, 0)
