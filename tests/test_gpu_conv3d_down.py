"""conv3d_down on the H100 (torch_utils/ops/conv3d_down.py, csrc/fir3d.cu).

Exact tier: sparse small-integer x, w, b, dz and the dyadic filter [1,3,3,1]/8 keep every intermediate of both the float64
reference and the native path exactly representable (each case asserts that precondition), so forward, dx, dw and db must
equal the float64 reference element for element -- for every downsampling layer of the low-res discriminator at reduced
batch and frames, border-sized extents, fp32 and fp16, and the FIR kernels alone in both directions.
Random values: the error against float64 is at most 1.5x that of today's path (conv_nd.conv3d -> Downsample3d -> bias_act).
Whole discriminator: the unmodified reference model with install() against without, both judged against a float64 run.
Profile: the installed layers launch the FIR kernels, and no engine call produces the full-resolution output of a layer
that takes the decomposition (conv3d_down.faster)."""
import os
import subprocess
import sys

import pytest
import torch

from torch_utils.ops import bias_act, conv3d_down as cd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

pytestmark = pytest.mark.gpu
DEV = 'cuda'
F = torch.tensor([1., 3., 3., 1.]) / 8
DT = {'f32': torch.float32, 'f16': torch.float16}

# (name, Cin, Cout, kt, ks, T, H, W, spatial_down, temporal_down): the downsampling layers of one D pass (batch 8, T = 128,
# 64 x 64) at batch 1 and 4 frames, and border-sized extents
LAYERS = [
    ('b0_skip', 32, 64, 1, 1, 4, 64, 64, True, False),
    ('b0_conv1', 32, 64, 1, 3, 4, 64, 64, True, False),
    ('b1_skip', 64, 128, 1, 1, 4, 32, 32, True, True),
    ('b1_conv1', 64, 128, 5, 3, 4, 32, 32, True, True),
    ('b2_skip', 128, 256, 1, 1, 4, 16, 16, True, True),
    ('b2_conv1', 128, 256, 5, 3, 4, 16, 16, True, True),
    ('b3_skip', 256, 512, 1, 1, 4, 8, 8, True, True),
    ('b3_conv1', 256, 512, 5, 3, 4, 8, 8, True, True),
    ('border_533', 8, 16, 5, 3, 2, 2, 2, True, True),
    ('border_333_t', 8, 16, 3, 3, 2, 2, 2, False, True),
    ('border_733_s', 8, 16, 7, 3, 2, 2, 2, True, False),
]


def ints(shape, seed, vmax=1, density=0.1):
    g = torch.Generator().manual_seed(seed)
    v = torch.randint(-vmax, vmax + 1, shape, generator=g).double()
    return v * (torch.rand(shape, generator=g) < density).double()


def check_repr(t, dtype, what):
    """Precondition of an exact comparison: every value is a multiple of 2^-9 (the dyadic filter's three axes) that fp16
    holds exactly, or, for fp32, one within 2^24 units of 2^-9. The engine's operands (x, w, dz: small integers; the
    filtered input: multiples of 2^-9 below 4) then also fit fp16 and the fp32 path's bf16 hi/lo split exactly."""
    assert torch.equal(torch.round(t * 512), t * 512), f'{what}: not a multiple of 2^-9'
    if dtype == torch.float16:
        assert torch.equal(t.half().double(), t), f'{what}: not exactly representable in fp16'
    else:
        assert float(t.abs().max()) * 512 < 2 ** 24, f'{what}: beyond 2^24 units'


def reference64(x, w, b, sd, td, act='linear', clamp=None):
    pad = tuple(k // 2 for k in w.shape[2:])
    return bias_act.bias_act(cd._reference(x, w, F, sd, td, pad), b, act=act, clamp=clamp)     # upfirdn2d takes fp32 taps


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('layer', LAYERS, ids=[l[0] for l in LAYERS])
def test_exact_forward_and_gradients(layer, dt):
    name, cin, cout, kt, ks, t, h, w, sd, td = layer
    dtype = DT[dt]
    x = ints((1, cin, t, h, w), 1)
    wt = ints((cout, cin, kt, ks, ks), 2, density=min(0.15, 3 / (cin * kt * ks * ks)))     # ~3 products per output
    b = ints((cout,), 3, vmax=2, density=0.5)
    pad = (kt // 2, ks // 2, ks // 2)
    res = []
    for d, ty in (('cpu', torch.float64), (DEV, dtype)):
        xg = x.to(d, ty).requires_grad_(True)
        wg = wt.to(d, ty).requires_grad_(True)
        bg = b.to(d, ty).requires_grad_(True)
        if d == 'cpu':
            z = reference64(xg, wg, bg, sd, td)
        else:
            assert cd.in_envelope(xg, wg, pad, sd, td, F.to(d))
            # the decomposition itself, also for the kernel sizes conv3d_down routes to the reference composition
            z = bias_act.bias_act(cd._decomposed(xg, wg, F.to(d), sd, td), bg)
        dz = ints(z.shape, 4, density=0.1 if dtype == torch.float32 else 0.001).to(d, ty)     # fp16: dw stays exact
        gx, gw, gb = torch.autograd.grad(z, [xg, wg, bg], dz)
        res.append([z, gx, gw, gb])
    for what, ref, got in zip(('z', 'dx', 'dw', 'db'), *res):
        ref = ref.detach()
        check_repr(ref, dtype, f'{name} {what}')
        got = got.detach().cpu().double()
        assert got.shape == ref.shape, what
        assert torch.equal(got, ref), f'{name} {dt} {what}: {int((got != ref).sum())} of {ref.numel()} differ, max {(got - ref).abs().max():.3e}'


FIR_CASES = [
    ('full_fold', ((1, 1, -3, 6, 10), (1, 1, -2, 34, 36), (1, 1, -2, 70, 72)), True),
    ('down', ((1, 2, -1, 6, 3), (1, 2, -1, 64, 32), (1, 2, -1, 66, 33)), False),
    ('down_ext', ((1, 2, 0, 6, 2), (1, 2, 0, 10, 4), (0, 1, 0, 5, 5)), False),
    ('copy_t', ((0, 1, 0, 3, 3), (1, 1, -2, 9, 11), (1, 2, -1, 40, 20)), False),
]


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('name,axes,fold', FIR_CASES, ids=[c[0] for c in FIR_CASES])
def test_fir_kernels_exact(name, axes, fold, dt):
    dtype = DT[dt]
    x = ints((2, 3) + tuple(a[3] for a in axes), 5, vmax=2, density=0.5)
    ref = cd._fir_reference(x, F.double(), axes, fold)
    check_repr(ref, dtype, name)
    got = cd.fir3d(x.to(DEV, dtype), F.to(DEV), axes, fold)
    assert torch.equal(got.cpu().double(), ref), name
    y = ints(ref.shape, 6, vmax=2, density=0.5)
    ref_t = cd._fir_adjoint_reference(y, F.double(), axes, fold)
    check_repr(ref_t, dtype, name + ' adjoint')
    got_t = custom_ops_adjoint(y.to(DEV, dtype), axes, fold)
    assert torch.equal(got_t.cpu().double(), ref_t), name + ' adjoint'
    # <P x, y> = <x, P^T y> on the device results
    assert float((got.double() * y.to(DEV)).sum()) == float((x.to(DEV) * got_t.double()).sum())


def custom_ops_adjoint(y, axes, fold):
    from torch_utils import custom_ops
    return custom_ops.get_plugin('fir3d_plugin').fir3d(y, F.to(DEV), axes, fold, adjoint=True)


def _err(a, b):
    return float((a.double() - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize('dt', ['f32', 'f16'])
@pytest.mark.parametrize('layer', [l for l in LAYERS if l[0].startswith('b')], ids=[l[0] for l in LAYERS if l[0].startswith('b')])
def test_random_values_no_less_accurate_than_today(layer, dt):
    name, cin, cout, kt, ks, t, h, w, sd, td = layer
    dtype = DT[dt]
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, cin, t, h, w, generator=g, dtype=torch.float64)
    wt = torch.randn(cout, cin, kt, ks, ks, generator=g, dtype=torch.float64) / (cin * kt * ks * ks) ** 0.5
    b = torch.randn(cout, generator=g, dtype=torch.float64)
    act = 'linear' if ks == 1 else 'lrelu'
    pad = (kt // 2, ks // 2, ks // 2)
    outs = {}
    for path in ('ref64', 'today', 'new'):
        d, ty = ('cpu', torch.float64) if path == 'ref64' else (DEV, dtype)
        xg, wg, bg = (v.to(d, ty).requires_grad_(True) for v in (x, wt, b))
        if path == 'new':
            z = cd.conv3d_down(xg, wg, bg, pad, sd, td, F.to(d), act=act, clamp=256)
        else:
            z = bias_act.bias_act(cd._reference(xg, wg, F.to(d), sd, td, pad), bg, act=act, clamp=256)
        dz = torch.randn(z.shape, generator=torch.Generator().manual_seed(8), dtype=torch.float64).to(d, ty)
        outs[path] = [z] + list(torch.autograd.grad(z, [xg, wg, bg], dz))
    for i, what in enumerate(('z', 'dx', 'dw', 'db')):
        ref = outs['ref64'][i].detach()
        e_new, e_old = _err(outs['new'][i].detach().cpu(), ref), _err(outs['today'][i].detach().cpu(), ref)
        slack = 1e-7 if dtype == torch.float32 else 1e-4
        assert e_new <= 1.5 * e_old + slack, f'{name} {dt} {what}: new {e_new:.3e}, today {e_old:.3e}'


def _run(mode, out_file):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'conv3d_down_dropin_run.py'), out_file, mode], env=env,
                       cwd=SRC, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out_file)


needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')


@needs_ref
def test_whole_discriminator_installed_vs_not_against_float64(tmp_path):
    base, ours, truth = (_run(m, str(tmp_path / f'{m}.pt')) for m in ('base', 'ours', 'truth'))
    # (key, max-norm tolerance, L2 tolerance) as for the low-res discriminator in test_gpu_dropin_cuda.py
    for key, tol_max, tol_l2 in (('logits', 1e-3, 5e-4), ('r1_gx', 1e-1, 2e-2), ('grad', 2e-2, 1e-2)):
        ref = truth[key]
        errs = {}
        for name, run in (('base', base), ('ours', ours)):
            a = run[key]
            assert a.shape == ref.shape and torch.isfinite(a).all(), (name, key)
            errs[name] = (float((a - ref).abs().max() / ref.abs().max()), float((a - ref).norm() / ref.norm()))
        (m_o, l_o), (m_b, l_b) = errs['ours'], errs['base']
        assert m_o <= tol_max and l_o <= tol_l2, f'{key}: max {m_o:.3e}, L2 {l_o:.3e}'
        assert m_o <= 1.5 * m_b + 1e-6 and l_o <= 1.5 * l_b + 1e-6, f'{key}: ours {errs["ours"]}, today {errs["base"]}'


@needs_ref
def test_profile_installed_layers_launch_fir_kernels_and_no_full_resolution_convolution(tmp_path):
    """(the 3x3 layers keep the reference composition by conv3d_down.faster)"""
    p = _run('profile', str(tmp_path / 'profile.pt'))
    kernels = ' '.join(p['kernels'])
    assert 'fir3d_down_kernel' in kernels and 'fir3d_adjoint_kernel' in kernels, p['kernels']
    assert p['full'] and p['fprop']
    full = {tuple(s) for s in p['full']}
    assert not full & {tuple(s) for s in p['fprop']}, full & {tuple(s) for s in p['fprop']}
