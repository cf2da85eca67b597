"""CPU checks that go with tests/test_gpu_fir_orientation.py: the modules' own restatements of the fused FIR operators
(conv3d_down's FIR pair, sres_cond's axis matrix) equal the float64 references built from the definitions; every GPU case
can tell the orientation mistakes apart (its reference changes with the taps reversed, fx and fy exchanged, flip toggled,
and for the 3-D ops with the filtered axes permuted); sres_dblock's autograd Function with a flipped, asymmetric filter
over the torch stand-in of its kernels; and which rank-1 filters upfirdn2d._rank1_factors splits exactly."""
import itertools

import numpy as np
import pytest
import torch

import test_gpu_fir_orientation as gx
import test_sres_dblock_host as tsh
from torch_utils.ops import conv3d_down as cd, sres_cond as sc, sres_dblock as sd, upfirdn2d

A, B, S = gx.A, gx.B, gx.S


def rev(f):
    return tuple(reversed(f))


def f64(f):
    return torch.tensor(f, dtype=torch.float64)


def _all_differ(refs, mutated, what):
    for i, (a, b) in enumerate(zip(refs, mutated)):
        assert gx.differs(a, b), f'{what}: output {i} does not change'


# ---------------------------------------------------------------------------------------------------- restatements

@pytest.mark.parametrize('f', gx.FIR3D_TAPS, ids=lambda f: gx.TAP_IDS[f])
@pytest.mark.parametrize('case', gx.FIR3D_CASES, ids=[c[0] for c in gx.FIR3D_CASES])
def test_fir3d_restatements_match_the_definition(case, f):
    """conv3d_down._fir_reference / _fir_adjoint_reference (the CPU path of the FIR pair) on every axis subset, step, offset
    and fold."""
    name, axes, fold = case
    x, y = gx.fir3d_case(case)
    want, want_t = gx.fir3d_refs(case, f)
    assert torch.equal(cd._fir_reference(x, f64(f), axes, fold), want)
    assert torch.equal(cd._fir_adjoint_reference(y, f64(f), axes, fold), want_t)


@pytest.mark.parametrize('down', [d for d in itertools.product((False, True), repeat=3) if any(d)])
def test_downsample3d_is_the_down_configuration_of_fir3d(down):
    """Downsample3d as the reference writes it (H and W together) equals fir3d's step-2 configuration per axis, which the
    decomposition and the axis mutations use."""
    y = gx.ints((2, 3, 6, 8, 10), 61, vmax=3, density=0.5)
    got = gx.down_axes_ref(y, A, down)
    axes = [cd._DOWN(s) if dn else cd._COPY(s) for dn, s in zip(down, y.shape[2:])]
    assert torch.equal(got, cd._fir_reference(y, f64(A), axes, False))
    if down[1] == down[2]:
        assert torch.equal(got, gx.downsample3d_ref(y, A, down[1], down[0]))


@pytest.mark.parametrize('fhw', gx.COND_PAIRS, ids=lambda p: f'fh{gx.TAP_IDS[p[0]]}_fw{gx.TAP_IDS[p[1]]}')
@pytest.mark.parametrize('layer', gx.COND_LAYERS, ids=[l[0] for l in gx.COND_LAYERS])
def test_sres_cond_axis_matrix_matches_prep_cond(layer, fhw):
    """sres_cond.axis_matrix (the restatement the other sres_cond tests evaluate) equals prep_cond's pads, resampler and
    crop applied to each unit vector, on every row: the crop and the replicate pads at the ends included."""
    kind, scale, pad, in_h, in_w = layer
    for a, f, n, in_len in zip(gx.cond_plan(layer, *fhw), fhw, gx.LR[3:], (in_h, in_w)):
        want = gx.cond_axis_ref(torch.eye(n, dtype=torch.float64), f, kind, scale, pad, gx.SQUARE, gx.MARGIN, in_len).t()
        got = sc.axis_matrix(a, gx.taps(f))
        assert got.shape == want.shape and torch.equal(got, want), (kind, n)


# ---------------------------------------------------------------------------------------------------- discrimination

def _axis_perms(cfg):
    """The permutations of the per-axis configurations (T, H, W) that give another operator."""
    return [p for p in itertools.permutations(range(3)) if tuple(cfg[i] for i in p) != tuple(cfg)]


@pytest.mark.parametrize('f', gx.FIR3D_TAPS, ids=lambda f: gx.TAP_IDS[f])
@pytest.mark.parametrize('case', gx.FIR3D_CASES, ids=[c[0] for c in gx.FIR3D_CASES])
def test_fir3d_cases_discriminate(case, f):
    name, axes, fold = case
    refs = gx.fir3d_refs(case, f)
    _all_differ(refs, gx.fir3d_refs(case, rev(f)), f'{name} reversed taps')
    x, y = gx.fir3d_case(case)
    for p in _axis_perms(axes):
        pa = tuple(axes[i] for i in p)
        fwd = gx.fir3d_ref(x, f, pa, fold) if all(a[3] == s for a, s in zip(pa, x.shape[2:])) else None
        adj = gx.fir3d_adjoint_ref(y, f, pa, fold) if gx.fir3d_ref(torch.zeros((1, 1) + tuple(a[3] for a in pa)), f, pa, fold).shape[2:] \
            == y.shape[2:] else None
        _all_differ(refs, (fwd, adj), f'{name} axes {p}')


@pytest.mark.parametrize('out', gx.DB_OUTS, ids=[f'{a}x{b}x{c}' for a, b, c in gx.DB_OUTS])
@pytest.mark.parametrize('flags', gx.DB_FLAGS)
def test_dblock_tail_cases_discriminate(flags, out):
    o, _, lin, dy = gx.dblock_refs(flags, out, A)
    refs = (o, lin, dy)
    m = gx.dblock_refs(flags, out, rev(A))
    _all_differ(refs, (m[0], m[2], m[3]), 'reversed taps')
    down = (bool(flags & gx.P.TDOWN), bool(flags & gx.P.SDOWN), bool(flags & gx.P.SDOWN))
    for p in _axis_perms(down):
        m = gx.dblock_refs(flags, out, A, down=tuple(down[i] for i in p))
        _all_differ(refs, (m[0], m[2], m[3]), f'axes {p}')


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('layer', gx.C3_LAYERS, ids=[l[0] for l in gx.C3_LAYERS])
def test_conv3d_down_cases_discriminate(layer, dt):
    """z, dx and dw change (db is the sum of dz: no filter reaches it)."""
    dtype = gx.DT[dt]
    refs = gx.c3_refs(layer, A, dtype=dtype)[:3]
    _all_differ(refs, gx.c3_refs(layer, rev(A), dtype=dtype)[:3], 'reversed taps')
    down = (layer[9], layer[8], layer[8])
    for p in _axis_perms(down):
        _all_differ(refs, gx.c3_refs(layer, A, down=tuple(down[i] for i in p), dtype=dtype)[:3], f'axes {p}')


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('flip', [0, 1])
@pytest.mark.parametrize('fxy', gx.SD_PAIRS, ids=gx.SD_IDS)
@pytest.mark.parametrize('shape', gx.SD_SHAPES, ids=['x'.join(map(str, s)) for s in gx.SD_SHAPES])
def test_sres_dblock_cases_discriminate(shape, fxy, flip, dt):
    """conv1's output, its weight gradient and the FIR adjoint's dz0 each change."""
    dtype = gx.DT[dt]
    fx, fy = fxy
    refs = gx.sd_refs(shape, dtype, fx, fy, flip)
    refs = (refs[0], refs[2], refs[3])
    for what, args in (('fx reversed', (rev(fx), fy, flip)), ('fy reversed', (fx, rev(fy), flip)), ('fx, fy exchanged', (fy, fx, flip)),
                       ('flip toggled', (fx, fy, 1 - flip))):
        m = gx.sd_refs(shape, dtype, *args)
        _all_differ(refs, (m[0], m[2], m[3]), what)


@pytest.mark.parametrize('fhw', gx.COND_PAIRS, ids=lambda p: f'fh{gx.TAP_IDS[p[0]]}_fw{gx.TAP_IDS[p[1]]}')
@pytest.mark.parametrize('layer', gx.COND_LAYERS, ids=[l[0] for l in gx.COND_LAYERS])
def test_sres_cond_cases_discriminate(layer, fhw):
    f_h, f_w = fhw
    ref = gx.cond_ref(layer, f_h, f_w)
    for what, args in (('f_h reversed', (rev(f_h), f_w)), ('f_w reversed', (f_h, rev(f_w))), ('f_h, f_w exchanged', (f_w, f_h))):
        assert gx.differs(ref, gx.cond_ref(layer, *args)), what


# ---------------------------------------------------------------------------------------------------- sres_dblock's Function

@pytest.mark.parametrize('flip', [False, True])
def test_block_function_gradients_asymmetric_filter(monkeypatch, flip):
    """_Block over the torch stand-in of its kernels with f1 = outer(fy, fx), fx != fy both asymmetric: equals the
    composition with conv1's filter flipped when ``flip``, passes gradcheck (the native first-order backward's FIR adjoint)
    and gradgradcheck (the recorded backward's upfirdn2d)."""
    monkeypatch.setattr(sd, '_backend', tsh._TorchStandIn)
    g = torch.Generator().manual_seed(1)
    fx, fy = gx.taps(B), gx.taps(A)
    f1 = torch.outer(fy, fx)
    f_skip = upfirdn2d.setup_filter([1, 2, 4, 1])
    t = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64, requires_grad=True)     # noqa: E731
    x, ws, w0, b0, w1, b1 = t(2, 3, 6, 7), t(4, 3, 1, 1), t(3, 3, 3, 3), t(3), t(4, 3, 3, 3), t(4)
    cfg = (flip, 'lrelu', 0.2, float(np.sqrt(2)), 0.6, sd._SQRT_HALF)

    def fn(x, ws, w0, b0, w1, b1):
        xd = upfirdn2d.upfirdn2d(x, f_skip, down=2, padding=1)
        return sd._Block.apply(x, xd, ws, w0, b0, w1, b1, f1, fx, fy, cfg)
    ref = sd._composition(x, ws, w0, b0, w1, b1, f_skip, f1.flip([0, 1]) if flip else f1, 'lrelu', float(np.sqrt(2)), 0.6)
    assert torch.allclose(fn(x, ws, w0, b0, w1, b1), ref)
    other = sd._composition(x, ws, w0, b0, w1, b1, f_skip, f1 if flip else f1.flip([0, 1]), 'lrelu', float(np.sqrt(2)), 0.6)
    assert not torch.allclose(other, ref)
    assert torch.autograd.gradcheck(fn, (x, ws, w0, b0, w1, b1))
    assert torch.autograd.gradgradcheck(fn, (x, ws, w0, b0, w1, b1))


# ---------------------------------------------------------------------------------------------------- _rank1_factors

@pytest.mark.parametrize('k', [[1, 2, 4, 1], [2, 1, 3, 2], [1, 1, 5, 1], [3, 1, 2, 2]])
def test_rank1_factors_split_asymmetric_setup_filters_exactly(k):
    """setup_filter of an asymmetric integer kernel with a power-of-two sum: the balanced split, dyadic factors whose outer
    product IS the filter, oriented as outer(fy, fx)."""
    f = upfirdn2d.setup_filter(k)
    fx, fy = upfirdn2d._rank1_factors(f)
    assert torch.equal(torch.outer(fy.double(), fx.double()), f.double())
    assert torch.equal(fx, fy) and torch.equal(fx.double(), torch.tensor(k, dtype=torch.float64) / sum(k))


def test_rank1_factors_of_a_product_of_two_filters_fall_back():
    """outer(fy, fx) / 64 with fy = [1, 2, 4, 1], fx = [2, 1, 3, 2]: the balanced split does not reproduce it, the fallback's
    fx = [2/3, 1/3, 1, 2/3] is not dyadic and misses the taps within 1e-6 -- exact kernel tests pass fx and fy directly."""
    fy, fx = torch.tensor([1., 2., 4., 1.]), torch.tensor([2., 1., 3., 2.])
    f = torch.outer(fy, fx) / 64
    gx_, gy_ = upfirdn2d._rank1_factors(f)
    assert torch.allclose(gx_.double(), torch.tensor([2 / 3, 1 / 3, 1, 2 / 3], dtype=torch.float64), rtol=0, atol=1e-7)
    err = torch.outer(gy_.double(), gx_.double()) - f.double()
    assert not torch.equal(err, torch.zeros_like(err)) and float(err.abs().max()) <= 1e-6 * float(f.abs().max())
