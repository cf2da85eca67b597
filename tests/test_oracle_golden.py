"""The oracle reproduces every golden vector generated from the reference's own _ref ops
(tests/golden/*.npz, made by oracle/pin_against_reference.py)."""
import numpy as np
import pytest

from oracle import oracle as orc
from _common import golden, cases, rel_err

ACTS = ['linear', 'relu', 'lrelu', 'tanh', 'sigmoid', 'elu', 'selu', 'softplus', 'swish']
REF_KEEPS = {'linear': '', 'swish': 'x'}   # everything else keeps y (bias_act.py:21-31)


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('clamp', [None, 0.7])
def test_bias_act(act, clamp):
    g = golden('bias_act')
    tag = f'{act}_c{"n" if clamp is None else "y"}'
    x, b, y, dy, dx = (g[f'{tag}/{k}'] for k in ('x', 'b', 'y', 'dy', 'dx'))
    assert rel_err(orc.bias_act(x, b, 1, act, clamp=clamp), y) < 2e-6
    keeps = REF_KEEPS.get(act, 'y')
    got = orc.bias_act_grad(dy, x=x if keeps == 'x' else None, b=b if keeps == 'x' else None,
                            y=y if keeps == 'y' else None, dim=1, act=act, clamp=clamp, order=1)
    if not (act == 'linear' and clamp is not None):
        assert rel_err(got, dx) < 5e-6
    assert rel_err(got.sum(axis=(0, 2, 3)), g[f'{tag}/db']) < 1e-4 or (act == 'linear' and clamp is not None)
    # second order: d<dx, v>/d(dy) is the first-order operator applied to v
    v = g[f'{tag}/v']
    got = orc.bias_act_grad(v, x=x if keeps == 'x' else None, b=b if keeps == 'x' else None,
                            y=y if keeps == 'y' else None, dim=1, act=act, clamp=clamp, order=1)
    if not (act == 'linear' and clamp is not None):
        assert rel_err(got, g[f'{tag}/ddy']) < 5e-6


def test_bias_act_fc():
    g = golden('bias_act')
    assert rel_err(orc.bias_act(g['fc/x'], g['fc/b'], 1, 'lrelu'), g['fc/y']) < 2e-6


_UP = golden('upfirdn2d')


@pytest.mark.parametrize('name', sorted(cases(_UP)))
def test_upfirdn2d(name):
    shape, kw = cases(_UP)[name]
    f = _UP[f'{name}/f'] if f'{name}/f' in _UP else None
    assert rel_err(orc.upfirdn2d(_UP[f'{name}/x'], f, **kw), _UP[f'{name}/y']) < 2e-6
    assert rel_err(orc.upfirdn2d_adjoint(_UP[f'{name}/dy'], f, shape, **kw), _UP[f'{name}/dx']) < 5e-6


_FL = golden('filtered_lrelu')


@pytest.mark.parametrize('name', sorted(cases(_FL)))
def test_filtered_lrelu(name):
    _, kw = cases(_FL)[name]
    fu = _FL[f'{name}/fu'] if f'{name}/fu' in _FL else None
    fd = _FL[f'{name}/fd'] if f'{name}/fd' in _FL else None
    y, so = orc.filtered_lrelu(_FL[f'{name}/x'], fu, fd, _FL[f'{name}/b'], return_signs=True, **kw)
    assert rel_err(y, _FL[f'{name}/y']) < 5e-6
    # the composed reference path rounds to fp32 between stages; the oracle can mimic it
    y2 = orc.filtered_lrelu(_FL[f'{name}/x'], fu, fd, _FL[f'{name}/b'], stage_round=True, **kw)
    assert rel_err(y2, _FL[f'{name}/y']) < 5e-6
    assert so.dtype == np.uint8 and so.shape == orc.sign_shape(_FL[f'{name}/x'].shape, fu, fd, kw['up'], kw['down'], kw['padding'])
    assert orc.unpack_signs(so).max() <= 2


def test_conv_and_fma():
    g = golden('conv')
    assert rel_err(orc.conv2d(g['grouped_mod/x'], g['grouped_mod/w'], padding=2, groups=2), g['grouped_mod/y']) < 5e-6
    assert rel_err(orc.conv2d(g['plain_3x3/x'], g['plain_3x3/w'], padding=1), g['plain_3x3/y']) < 5e-6
    assert rel_err(orc.conv2d(g['fromrgb_1x1/x'], g['fromrgb_1x1/w']), g['fromrgb_1x1/y']) < 5e-6
    assert rel_err(orc.fma(g['fma/a'], g['fma/b'], g['fma/c']), g['fma/o']) < 1e-6


def test_conv2d_wgrad_restatement_matches_torch_autograd():
    # the oracle's float64 weight gradient (smoke() checks the engine's against it) equals the one torch derives for F.conv2d
    import torch
    gen = torch.Generator().manual_seed(1)
    for (n, g, cin, cout, h, w, k, pad) in ((2, 2, 3, 4, 5, 7, 3, 1), (1, 1, 5, 2, 6, 4, 3, 2), (3, 2, 4, 4, 5, 5, 1, 0)):
        x = torch.randn(n, g * cin, h, w, generator=gen)
        dy = torch.randn(n, g * cout, h + 2 * pad - k + 1, w + 2 * pad - k + 1, generator=gen)
        wt = torch.zeros(g * cout, cin, k, k, requires_grad=True)
        ref, = torch.autograd.grad(torch.nn.functional.conv2d(x, wt, padding=pad, groups=g), [wt], dy)
        got = orc.conv2d_wgrad(x.numpy(), dy.numpy(), tuple(wt.shape), padding=pad, groups=g)
        assert rel_err(got, ref.numpy()) < 1e-5
