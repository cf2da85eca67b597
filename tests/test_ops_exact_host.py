"""CPU checks that go with tests/test_gpu_ops_exact.py: its operand generators and exactness preconditions hold for
every case (run through the float64 oracle, no GPU needed), and `upfirdn2d._rank1_factors` splits the rank-1 filters
the networks use into factors whose outer product IS the filter, so the single-launch separable path computes the
same operator as the 2-D filter."""
import numpy as np
import pytest
import torch

import test_gpu_ops_exact as gx
from torch_utils.ops import upfirdn2d


@pytest.mark.parametrize('case', gx.UPFIRDN_CASES, ids=lambda c: c['name'])
def test_upfirdn2d_case_preconditions(case):
    x, dy = gx.upfirdn_inputs(case)
    assert np.mean(x == 0) > 0.25 and np.mean(dy == 0) > 0.25, 'operands must be sparse'
    y, dx = gx.upfirdn_refs(case, x, dy)
    for d in case['dtypes']:
        gx.check_repr(y, gx.DT[d], case['name'] + ' forward')
        gx.check_repr(dx, gx.DT[d], case['name'] + ' adjoint')
    # a flipped filter must give a different operator, or the case cannot tell orientations apart
    # (the symmetric setup_filter([1, 3, 3, 1]) of the networks excepted)
    f = gx.full(case['f'])
    if f.size > 1 and not np.array_equal(f, f[::-1, ::-1]):
        yf = gx.orc.upfirdn2d(x, f, case['up'], case['down'], case['pad'], not case['flip'], case['gain'])
        assert not np.array_equal(yf, y), case['name'] + ': flip_filter does not change the result'


@pytest.mark.parametrize('case', gx.FL_CASES, ids=lambda c: c['name'])
def test_filtered_lrelu_case_preconditions(case):
    x, b, pad = gx.fl_inputs(case)
    shape, _ = gx.fl_geometry(case)
    assert gx.orc.filtered_lrelu_out_shape(shape, case['fu'], case['fd'], case['up'], case['down'], pad)[2:] == \
        (case['oh'], case['ow'])
    # the fused kernels fold sqrt(up^2 gain) into the up-sampling taps; it must be exact. The backward pass folds
    # sqrt(down^2 gg) with gg = gain up^2 / down^2 (its up factor is the forward's down), which is the same value.
    scale = case['up'] ** 2 * case['gain']
    assert float(np.sqrt(np.float32(scale))) ** 2 == scale
    clamp = gx.fl_pick_clamp(case, x, b, pad)
    y, s = gx.fl_refs(case, x, b, pad, clamp)
    dx = gx.fl_refs(case, x, b, pad, clamp, signs=s, dy=gx.fl_dy(case, y.shape))
    for d in case['dtypes']:
        gx.check_repr(y, gx.DT[d], case['name'] + ' forward')
        gx.check_repr(dx, gx.DT[d], case['name'] + ' dx')
    codes = gx.orc.unpack_signs(s)
    assert (codes == 1).any() and (codes == 0).any(), case['name'] + ': needs both negative and non-negative samples'
    if clamp is not None:
        assert (codes == 2).any(), case['name'] + ': the clamp is never hit'


def test_filtered_lrelu_read_routes():
    """Sign tensors passed to the v3 kernel as they are and as zero-padded, aligned copies both come with random
    codes, non-zero, odd and negative offsets, and sizes smaller and larger than the consumed extent."""
    for route in ('v3', 'padded'):
        rcs = [r for r in gx.FL_READ if gx.fl_read_route(r) == route]
        assert {r['case']['cfg'] for r in rcs} == {1, 2, 3}, route
        assert any(r['sx'] > 0 and r['sx'] % 2 for r in rcs) and any(r['sx'] < 0 for r in rcs), route
        assert any(r['sy'] > 0 for r in rcs) and any(r['sy'] < 0 and r['sy'] % 2 for r in rcs), route
        assert any(r['sx'] % 4 and r['sy'] % 4 for r in rcs), route
        assert any(r['dh'] < 0 for r in rcs) and any(r['dh'] > 0 for r in rcs), route
        assert any(r['dwb'] < 0 for r in rcs) and any(r['dwb'] > 0 for r in rcs), route


@pytest.mark.parametrize('rc', gx.FL_READ, ids=lambda r: r['case']['name'])
def test_filtered_lrelu_read_preconditions(rc):
    x, b, pad, s = gx.fl_read_inputs(rc)
    assert ((s & 3) == 3).any(), 'code 3 must occur'
    for d in ('f32', 'f16'):
        y, _ = gx.fl_refs(rc['case'], x, b, pad, None, signs=s, sx=rc['sx'], sy=rc['sy'])
        gx.check_repr(y, gx.DT[d], rc['case']['name'])


@pytest.mark.parametrize('case', gx.BA_CASES, ids=lambda c: c['name'])
def test_bias_act_case_preconditions(case):
    x, b, dy, v, clamp = gx.ba_inputs(case)
    y = gx.orc.bias_act(x, b, case['dim'], case['act'], case['alpha'], case['gain'], clamp).astype(np.float64)
    for d in case['dtypes']:
        gx.check_repr(y, gx.DT[d], case['name'])
    if clamp is not None:
        assert (np.abs(y) == clamp).any(), case['name'] + ': no value sits exactly at the clamp'


def _tiled_plans():
    out = {}
    for c in gx.UPFIRDN_CASES:
        inst, _, variant = c['name'].rpartition('_')
        if inst in {t[0] for t in gx.TILED}:
            for d in c['dtypes']:
                out[(inst, variant, d)] = (c, gx.tiled_plan(c, d))
    return out


@pytest.mark.parametrize('inst', [t[0] for t in gx.TILED])
def test_tiled_cases_reach_what_they_claim(inst):
    """Replays launch_tiled() for each case of a tiled instance and checks the claims of _tiled_cases()'s docstring."""
    plans = _tiled_plans()
    for d in ('f32', 'f16'):
        c, p = plans[(inst, 'whole', d)]
        assert (p['tiles_x'], p['tiles_y'], p['pb'], p['flat']) == (1, 1, 1, 2), (c['name'], d, p)
        c, p = plans[(inst, 'batch', d)]
        assert p['pb'] > 1 and p['planes'] % p['pb'] != 0 and p['flat'] >= 1, (c['name'], d, p)
        c, p = plans[(inst, 'crop', d)]
        assert all(v < 0 for v in c['pad']), c['pad']
        assert (p['tiles_x'], p['tiles_y'], p['flat']) == (1, 1, 1), (c['name'], d, p)
        for v in ('cl', 'odd'):
            c, p = plans[(inst, v, d)]
            assert p['flat'] == 0, (c['name'], d, p)
    c, p = plans[(inst, 'big', 'f32')]
    assert p['tiles_x'] > 1 and p['tiles_y'] > 1, (c['name'], p)
    assert p['halved'] == (inst in gx.TILED_HALVED), (c['name'], p)
    assert all(p['instance'] == plans[(inst, v, 'f32')][1]['instance'] for v in ('whole', 'batch', 'crop', 'cl', 'odd'))


def test_route_list_names_every_instance():
    k = gx.expected_kernels()
    assert sum(n.startswith('tiled<') for n in k) == 15
    assert sum(n.startswith('stream<') for n in k) == 8
    assert sum(n.startswith('v3<') for n in k) == 9


def _split_candidates(a):
    """The splits `_rank1_factors` tries: balanced (sqrt|peak| on both factors), then column x row / peak."""
    i, j = divmod(int(np.abs(a).argmax()), a.shape[1])
    p = a[i, j]
    s = np.sqrt(abs(p))
    return [(a[:, j] / s, a[i, :] * np.sign(p) / s), (a[:, j], a[i, :] / p)]


def _exact(fy, fx, a):
    fy32, fx32 = np.float32(fy).astype(np.float64), np.float32(fx).astype(np.float64)
    return np.array_equal(np.outer(fy32, fx32), a)


RANK1 = {
    'setup_filter_1331': lambda: upfirdn2d.setup_filter([1, 3, 3, 1]),
    'setup_filter_121': lambda: upfirdn2d.setup_filter([1, 2, 1]),
    'setup_filter_1331_gain4': lambda: upfirdn2d.setup_filter([1, 3, 3, 1], gain=4),
    'setup_filter_13310_flip': lambda: upfirdn2d.setup_filter([1, 3, 3, 1], flip_filter=True, gain=0.25),
    'asym': lambda: torch.tensor(gx.RANK1_ASYM, dtype=torch.float32),
    'neg_peak': lambda: torch.tensor(gx.RANK1_NEG, dtype=torch.float32),
    'unnormalized': lambda: upfirdn2d.setup_filter([1, 3, 3, 1], normalize=False),
    'third': lambda: torch.outer(torch.tensor([1.0, 3.0, 1.0]), torch.tensor([1.0, 2.0, 1.0])) / 3,
}


@pytest.mark.parametrize('name', sorted(RANK1))
def test_rank1_factors_exact(name):
    """Whenever one of the candidate splits reproduces the filter exactly in float32, the returned factors must."""
    f = RANK1[name]()
    a = f.double().numpy()
    fac = upfirdn2d._rank1_factors(f)
    assert fac is not None, f'{name}: rank-1 filter not recognised'
    fx, fy = (t.double().numpy() for t in fac)
    assert fx.dtype == np.float64 and fac[0].dtype == torch.float32
    err = np.abs(np.outer(fy, fx) - a).max()
    if any(_exact(cy, cx, a) for cy, cx in _split_candidates(a)):
        assert err == 0, f'{name}: outer(fy, fx) misses the filter by {err:g} although an exact split exists'
    else:
        assert err <= 1e-6 * np.abs(a).max()


def test_rank1_factors_rejects_rank2():
    assert upfirdn2d._rank1_factors(torch.tensor(gx.F35, dtype=torch.float32)) is None
