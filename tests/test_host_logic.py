"""Host side of the ops (argument handling, autograd functions, adjoint padding algebra, sign
offsets, the 'ref' path) checked on CPU against the golden vectors from the reference.

The native plugins are replaced by oracle-backed stand-ins (tests/_common.py) so that the SAME
Python code that drives the CUDA kernels is executed here: what is verified is everything above
the C ABI."""
import numpy as np
import pytest
import torch

from torch_utils.ops import bias_act, upfirdn2d, filtered_lrelu, conv2d_resample, conv2d_gradfix, fma, grid_sample_gradfix
from _common import (golden, cases, assert_close, t, OracleBiasActPlugin, OracleBiasActCodesPlugin, OracleUpfirdn2dPlugin,
                     OracleFilteredLReluPlugin)

ACTS = sorted(bias_act.activation_funcs)


@pytest.fixture
def oracle_plugins(monkeypatch):
    monkeypatch.setattr(bias_act, '_plugin', OracleBiasActPlugin())
    monkeypatch.setattr(upfirdn2d, '_plugin', OracleUpfirdn2dPlugin())
    monkeypatch.setattr(filtered_lrelu, '_plugin', OracleFilteredLReluPlugin(fused=True))


def test_activation_table_matches_reference_contract():
    # values the models read: def_gain, def_alpha, cuda_idx numbering (bias_act.py:21-31)
    tab = bias_act.activation_funcs
    assert [tab[a].cuda_idx for a in ['linear', 'relu', 'lrelu', 'tanh', 'sigmoid', 'elu', 'selu', 'softplus', 'swish']] == list(range(1, 10))
    assert tab['lrelu'].def_alpha == 0.2 and abs(tab['lrelu'].def_gain - np.sqrt(2)) < 1e-12
    assert tab['linear'].def_gain == 1 and tab['swish'].ref == 'x' and tab['linear'].ref == ''
    assert all(tab[a].has_2nd_grad == (a not in ('linear', 'relu', 'lrelu')) for a in tab)


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('clamp', [None, 0.7])
def test_bias_act_autograd(oracle_plugins, act, clamp):
    g = golden('bias_act')
    tag = f'{act}_c{"n" if clamp is None else "y"}'
    x, b, dy = t(g[f'{tag}/x'], grad=True), t(g[f'{tag}/b'], grad=True), t(g[f'{tag}/dy'], grad=True)
    y = bias_act._bias_act_cuda(dim=1, act=act, clamp=clamp).apply(x, b)
    assert_close(y, g[f'{tag}/y'], 2e-6, 'forward')
    dx, db = torch.autograd.grad(y, [x, b], dy, create_graph=True)
    if act == 'linear' and clamp is not None:
        return  # the reference plugin path does not mask linear+clamp gradients (no saved y); _ref autograd does
    assert_close(dx, g[f'{tag}/dx'], 5e-6, 'dx')
    assert_close(db, g[f'{tag}/db'], 1e-5, 'db')
    v = t(g[f'{tag}/v'])
    if dx.requires_grad:
        ddy, ddx = torch.autograd.grad((dx * v).sum(), [dy, x], allow_unused=True)
        assert_close(ddy, g[f'{tag}/ddy'], 5e-6, 'second order wrt dy')
        if bias_act.activation_funcs[act].has_2nd_grad:
            assert_close(ddx, g[f'{tag}/ddx'], 2e-5, 'second order wrt x')
        else:
            assert ddx is None or float(ddx.abs().max()) == 0.0


@pytest.mark.parametrize('act', ['relu', 'lrelu'])
@pytest.mark.parametrize('clamp', [None, 0.7])
@pytest.mark.parametrize('create_graph', [False, True])
def test_bias_act_autograd_through_codes(monkeypatch, act, clamp, create_graph):
    # relu / lrelu: the forward of a call that needs gradients hands 2-bit codes to the backward instead of saving y
    plug = OracleBiasActCodesPlugin()
    monkeypatch.setattr(bias_act, '_plugin', plug)
    g = golden('bias_act')
    tag = f'{act}_c{"n" if clamp is None else "y"}'
    x, b, dy = t(g[f'{tag}/x'], grad=True), t(g[f'{tag}/b'], grad=True), t(g[f'{tag}/dy'], grad=True)
    y = bias_act._bias_act_cuda(dim=1, act=act, clamp=clamp).apply(x, b)
    assert plug.fwd_calls == 1
    assert_close(y, g[f'{tag}/y'], 2e-6, 'forward')
    dx, db = torch.autograd.grad(y, [x, b], dy, create_graph=create_graph)
    assert plug.bwd_calls == 1
    assert_close(dx, g[f'{tag}/dx'], 5e-6, 'dx')
    assert_close(db, g[f'{tag}/db'], 1e-5, 'db')
    if create_graph:
        v = t(g[f'{tag}/v'])
        ddy, ddx = torch.autograd.grad((dx * v).sum(), [dy, x], allow_unused=True)
        assert_close(ddy, g[f'{tag}/ddy'], 5e-6, 'second order wrt dy')
        assert ddx is None or float(ddx.abs().max()) == 0.0
    # no gradient needed -> no codes are produced
    with torch.no_grad():
        bias_act._bias_act_cuda(dim=1, act=act, clamp=clamp).apply(x.detach(), b.detach())
    assert plug.fwd_calls == 1
    # opting out restores the save-y path
    monkeypatch.setenv('LVG_BIAS_ACT_CODES', '0')
    y2 = bias_act._bias_act_cuda(dim=1, act=act, clamp=clamp).apply(x, b)
    dx2, = torch.autograd.grad(y2, [x], dy.detach())
    assert plug.fwd_calls == 1
    assert_close(dx2, g[f'{tag}/dx'], 5e-6, 'dx without codes')


@pytest.mark.parametrize('act', ACTS)
def test_bias_act_ref_path(act):
    g = golden('bias_act')
    for clamp, tag in ((None, f'{act}_cn'), (0.7, f'{act}_cy')):
        y = bias_act.bias_act(t(g[f'{tag}/x']), t(g[f'{tag}/b']), act=act, clamp=clamp, impl='ref')
        assert_close(y, g[f'{tag}/y'], 1e-6)


def test_bias_act_identity_and_layouts(oracle_plugins):
    x = torch.randn(2, 3, 4, 5)
    assert bias_act._bias_act_cuda(act='linear').apply(x, None).data_ptr() == x.data_ptr()   # nothing to do: no kernel, no copy
    xc = x.to(memory_format=torch.channels_last).requires_grad_(True)
    b = torch.randn(3, requires_grad=True)
    y = bias_act._bias_act_cuda(act='lrelu').apply(xc, b)
    assert y.stride() == xc.stride()
    assert_close(y, bias_act.bias_act(xc, b, act='lrelu', impl='ref'), 1e-6)
    y.sum().backward()
    assert xc.grad.shape == xc.shape and b.grad.shape == b.shape


_UP = golden('upfirdn2d')


@pytest.mark.parametrize('name', sorted(cases(_UP)))
def test_upfirdn2d_autograd(oracle_plugins, name):
    _, kw = cases(_UP)[name]
    f = t(_UP[f'{name}/f']) if f'{name}/f' in _UP else None
    x = t(_UP[f'{name}/x'], grad=True)
    y = upfirdn2d._upfirdn2d_cuda(**kw).apply(x, f)
    assert_close(y, _UP[f'{name}/y'], 2e-6, 'forward')
    dx, = torch.autograd.grad(y, [x], t(_UP[f'{name}/dy']), create_graph=True)
    assert_close(dx, _UP[f'{name}/dx'], 5e-6, 'adjoint via swapped up/down')
    assert_close(upfirdn2d.upfirdn2d(t(_UP[f'{name}/x']), f, impl='ref', **kw), _UP[f'{name}/y'], 1e-6, 'ref path')


def test_upfirdn2d_double_backward(oracle_plugins):
    # R1 penalty path: d/d(dy) of <dx, w> equals the forward operator applied to w
    name = 'U4_sdown'
    _, kw = cases(_UP)[name]
    f = t(_UP[f'{name}/f'])
    x = t(_UP[f'{name}/x'], grad=True)
    dy = t(_UP[f'{name}/dy'], grad=True)
    y = upfirdn2d._upfirdn2d_cuda(**kw).apply(x, f)
    dx, = torch.autograd.grad(y, [x], dy, create_graph=True)
    w = torch.randn_like(x)
    ddy, = torch.autograd.grad((dx * w).sum(), [dy])
    assert_close(ddy, upfirdn2d.upfirdn2d(w, f, impl='ref', **kw), 5e-6)


def test_upfirdn2d_wrappers_and_filters():
    f = upfirdn2d.setup_filter([1, 3, 3, 1])
    assert f.shape == (4, 4) and abs(float(f.sum()) - 1) < 1e-6
    fs = upfirdn2d.setup_filter([1, 2, 3, 4, 4, 3, 2, 1], gain=4)
    assert fs.shape == (8,) and abs(float(fs.sum()) - 2) < 1e-6       # gain ** (ndim / 2)
    assert upfirdn2d.setup_filter(None).shape == (1, 1)
    assert torch.equal(upfirdn2d.setup_filter([1, 2, 3], flip_filter=True, normalize=False, separable=True), torch.tensor([3., 2., 1.]))
    x = torch.randn(1, 2, 6, 7)
    assert upfirdn2d.upsample2d(x, f, up=2).shape == (1, 2, 12, 14)
    assert upfirdn2d.downsample2d(x, f, down=2).shape == (1, 2, 3, 3)
    assert upfirdn2d.filter2d(x, f).shape == x.shape
    assert upfirdn2d._parse_scaling(3) == (3, 3) and upfirdn2d._parse_padding([1, 2]) == (1, 1, 2, 2)
    assert upfirdn2d._get_filter_size(None) == (1, 1) and upfirdn2d._get_filter_size(torch.zeros(5, 3)) == (3, 5)


_FL = golden('filtered_lrelu')


@pytest.mark.parametrize('fused', [True, False])
@pytest.mark.parametrize('name', sorted(cases(_FL)))
def test_filtered_lrelu_autograd(oracle_plugins, monkeypatch, name, fused):
    monkeypatch.setattr(filtered_lrelu, '_plugin', OracleFilteredLReluPlugin(fused=fused))
    _, kw = cases(_FL)[name]
    fu = t(_FL[f'{name}/fu']) if f'{name}/fu' in _FL else None
    fd = t(_FL[f'{name}/fd']) if f'{name}/fd' in _FL else None
    x, b = t(_FL[f'{name}/x'], grad=True), t(_FL[f'{name}/b'], grad=True)
    y = filtered_lrelu._filtered_lrelu_cuda(**kw).apply(x, fu, fd, b, None, 0, 0)
    assert_close(y, _FL[f'{name}/y'], 5e-6, 'forward')
    dx, db = torch.autograd.grad(y, [x, b], t(_FL[f'{name}/dy']))
    # backward = the same operator on dy with swapped filters, reading the packed signs at an offset
    assert_close(dx, _FL[f'{name}/dx'], 2e-5, 'dx')
    assert_close(db, _FL[f'{name}/db'], 2e-5, 'db')
    y_ref = filtered_lrelu.filtered_lrelu(t(_FL[f'{name}/x']), fu, fd, t(_FL[f'{name}/b']), impl='ref', **kw)
    assert_close(y_ref, _FL[f'{name}/y'], 1e-6, 'ref path')


def test_filtered_lrelu_no_grad_skips_signs(oracle_plugins, monkeypatch):
    calls = []

    class Spy(OracleFilteredLReluPlugin):
        def filtered_lrelu(self, *a):
            calls.append(a[-1])
            return super().filtered_lrelu(*a)
    monkeypatch.setattr(filtered_lrelu, '_plugin', Spy())
    x = torch.randn(1, 2, 6, 6)
    filtered_lrelu._filtered_lrelu_cuda().apply(x, None, None, None, None, 0, 0)
    filtered_lrelu._filtered_lrelu_cuda().apply(x.requires_grad_(True), None, None, None, None, 0, 0)
    assert calls == [False, True]


_CV = golden('conv')


@pytest.mark.parametrize('name', sorted(cases(_CV)))
def test_conv2d_resample(name):
    xs, ws, kw, has_f = cases(_CV)[name]
    if has_f:
        kw = dict(kw, f=t(_CV['f4']))
    x, w = t(_CV[f'{name}/x'], grad=True), t(_CV[f'{name}/w'], grad=True)
    y = conv2d_resample.conv2d_resample(x, w, **kw)
    assert_close(y, _CV[f'{name}/y'], 1e-5, 'forward')
    dx, dw = torch.autograd.grad(y, [x, w], t(_CV[f'{name}/dy']))
    assert_close(dx, _CV[f'{name}/dx'], 1e-5, 'dx')
    assert_close(dw, _CV[f'{name}/dw'], 1e-5, 'dw')


def test_conv2d_gradfix_surface():
    assert conv2d_gradfix.enabled is False and conv2d_gradfix.weight_gradients_disabled is False
    with conv2d_gradfix.no_weight_gradients():
        assert conv2d_gradfix.weight_gradients_disabled is True
    assert conv2d_gradfix.weight_gradients_disabled is False
    x, w = torch.randn(1, 4, 5, 5), torch.randn(6, 2, 3, 3)
    assert torch.equal(conv2d_gradfix.conv2d(x, w, padding=1, groups=2), torch.nn.functional.conv2d(x, w, padding=1, groups=2))
    wt = torch.randn(4, 3, 3, 3)
    assert torch.equal(conv2d_gradfix.conv_transpose2d(x, wt, stride=2), torch.nn.functional.conv_transpose2d(x, wt, stride=2))


def test_fma_and_unbroadcast():
    g = _CV
    a, b, c = t(g['fma/a'], grad=True), t(g['fma/b'], grad=True), t(g['fma/c'], grad=True)
    o = fma.fma(a, b, c)
    assert_close(o, g['fma/o'], 1e-6)
    da, db, dc = torch.autograd.grad(o, [a, b, c], t(g['fma/do']))
    assert_close(da, g['fma/da'], 1e-6)
    assert_close(db, g['fma/db'], 1e-6)
    assert_close(dc, g['fma/dc'], 1e-6)


def test_grid_sample_gradfix_double_backward():
    grid_sample_gradfix.enabled = True
    try:
        img = torch.randn(1, 2, 5, 5, dtype=torch.float64, requires_grad=True)
        grid = (torch.rand(1, 4, 4, 2, dtype=torch.float64) * 1.6 - 0.8)
        out = grid_sample_gradfix.grid_sample(img, grid)
        ref = torch.nn.functional.grid_sample(img, grid, mode='bilinear', padding_mode='zeros', align_corners=False)
        assert torch.allclose(out, ref)
        wgt = torch.randn_like(out, requires_grad=True)
        gi, = torch.autograd.grad((out * wgt).sum(), [img], create_graph=True)
        gg, = torch.autograd.grad(gi.square().sum(), [wgt])      # second order flows back through grad_output
        # stock grid_sample has no double backward; the adjoint of "scatter wgt" is "sample", so:
        gg_ref = torch.nn.functional.grid_sample(2 * gi.detach(), grid, mode='bilinear', padding_mode='zeros', align_corners=False)
        assert torch.allclose(gg, gg_ref)
    finally:
        grid_sample_gradfix.enabled = False


def test_workload_traces_are_consistent():
    """bench.py replays workloads/*.json: every recorded call must name a hot-path op with usable arguments."""
    import json
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    seen = set()
    for fname, keys in (('lres_step.json', ('lres_G', 'lres_D')), ('sres_step.json', ('sres_G', 'sres_D'))):
        tr = json.load(open(os.path.join(root, 'workloads', fname)))
        for k in keys:
            assert len(tr[k]) > 20
            for c in tr[k]:
                seen.add(c['op'])
                assert len(c['x']) >= 2 and all(isinstance(v, int) and v > 0 for v in c['x'])
                if c['op'] == 'upfirdn2d':
                    upfirdn2d._parse_scaling(c['up']), upfirdn2d._parse_scaling(c['down']), upfirdn2d._parse_padding(c['padding'])
                if c['op'] == 'bias_act':
                    assert c['act'] in bias_act.activation_funcs
    # call counts of SURVEY.md Appendix A
    lres = json.load(open(os.path.join(root, 'workloads', 'lres_step.json')))
    assert sum(c['op'] == 'bias_act' for c in lres['lres_G']) == 23 and sum(c['op'] == 'upfirdn2d' for c in lres['lres_G']) == 14
    assert sum(c['op'] == 'bias_act' for c in lres['lres_D']) == 18
    sres = json.load(open(os.path.join(root, 'workloads', 'sres_step.json')))
    assert sum(c['op'] == 'filtered_lrelu' for c in sres['sres_G']) == 15 and sum(c['op'] == 'conv2d' for c in sres['sres_G']) == 15
    assert sum(c['op'] == 'conv2d_resample' for c in sres['sres_D']) == 20
    assert {'bias_act', 'upfirdn2d', 'filtered_lrelu', 'conv2d', 'conv2d_resample'} <= seen


def test_bench_reference_arm_runs_on_cpu():
    """`bench.py --impl reference` (the oracle on host cores) prints one well-formed JSON line without a GPU."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, 'bench.py'), '--impl', 'reference', '--steps', '1', '--warmup', '0',
                          '--cpu-budget', '1'], capture_output=True, text=True, timeout=600,
                         env=dict(os.environ, OMP_NUM_THREADS='1'))      # torchrun exports this; the arm must still use every core
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line['impl'] == 'reference' and line['unit'] == 'frames/s' and line['value'] > 0
    assert line['cpu_baseline']['kind'] in ('port', 'reference') and line['cpu_baseline']['cores'] == os.cpu_count()
    assert line['e2e']['h2d_bytes_per_step'] == 0 and line['higher_is_better'] is True
