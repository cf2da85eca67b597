"""Host logic of torch_utils/ops/conv3d_down.py on CPU, in float64: the decomposition (FIR of the input, strided or
phase-folded convolution at the output resolution, border faces) run over torch stand-ins of the FIR kernels equals the
reference composition conv3d -> Downsample3d (upfirdn2d) in value, first and second order; the stand-in of the adjoint
kernel's gather is the exact adjoint; install() patches the staged reference model and falls back outside the envelope."""
import itertools
import os
import subprocess
import sys

import pytest
import torch

from torch_utils.ops import conv3d_down as cd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

F_ASYM = torch.tensor([1., 2., 4., 1.], dtype=torch.float32) / 8       # asymmetric: catches a flipped tap order
F_DOWN = torch.tensor([1., 3., 3., 1.], dtype=torch.float32) / 8       # Downsample3d's filter

DOWNS = [(True, False), (False, True), (True, True)]                   # (spatial_down, temporal_down)


def _operands(kt, ks, sd, td, t, h, w, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(2, 3, t, h, w, generator=g, dtype=torch.float64)
    wt = torch.randn(4, 3, kt, ks, ks, generator=g, dtype=torch.float64)
    return x, wt


def _both(x, wt, f, sd, td):
    pad = (wt.shape[2] // 2, wt.shape[3] // 2, wt.shape[4] // 2)
    return cd._decomposed(x, wt, f, sd, td), cd._reference(x, wt, f, sd, td, pad)


@pytest.mark.parametrize('kt,ks', list(itertools.product((1, 3, 5, 7), (1, 3))))
@pytest.mark.parametrize('sd,td', DOWNS)
@pytest.mark.parametrize('ext', [(2, 2, 2), (6, 4, 6), (8, 10, 6)])
def test_decomposition_equals_reference_forward(kt, ks, sd, td, ext):
    x, wt = _operands(kt, ks, sd, td, *ext)
    for f in (F_DOWN, F_ASYM):
        got, ref = _both(x, wt, f, sd, td)
        assert got.shape == ref.shape
        torch.testing.assert_close(got, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize('kt,ks', [(1, 3), (3, 3), (5, 3), (7, 1), (5, 1)])
@pytest.mark.parametrize('sd,td', DOWNS)
def test_decomposition_gradients_first_and_second_order(kt, ks, sd, td):
    x0, w0 = _operands(kt, ks, sd, td, 4, 6, 4, seed=1)
    res = []
    for fn in (cd._decomposed, lambda x, w, f, s, t: cd._reference(x, w, f, s, t, (kt // 2, ks // 2, ks // 2))):
        x, w = x0.clone().requires_grad_(True), w0.clone().requires_grad_(True)
        z = fn(x, w, F_ASYM, sd, td)
        dz = torch.linspace(-1, 1, z.numel(), dtype=torch.float64).reshape(z.shape)
        gx, gw = torch.autograd.grad(z, [x, w], dz, create_graph=True)
        hx, hw = torch.autograd.grad(gx.square().sum() + (gw * gw.flip(0)).sum(), [x, w])
        res.append((z, gx, gw, hx, hw))
    for got, ref in zip(*res):
        torch.testing.assert_close(got, ref, rtol=1e-11, atol=1e-11)


@pytest.mark.parametrize('axes,fold', [
    (((1, 1, -3, 6, 10), (1, 1, -2, 5, 7), (1, 1, -2, 4, 6)), True),          # full rate on every axis, T folded
    (((1, 2, -1, 6, 3), (1, 2, -1, 4, 2), (1, 2, 0, 6, 2)), False),           # step 2 (padded and extended ranges)
    (((0, 1, 0, 3, 3), (1, 2, -1, 2, 1), (0, 1, 0, 5, 5)), False),            # copy axes
])
def test_fir_adjoint_reference_is_exact(axes, fold):
    g = torch.Generator().manual_seed(3)
    shape_in = (2, 3) + tuple(a[3] for a in axes)
    x = torch.randn(shape_in, generator=g, dtype=torch.float64)
    px = cd._fir_reference(x, F_ASYM, axes, fold)
    y = torch.randn(px.shape, generator=g, dtype=torch.float64)
    pty = cd._fir_adjoint_reference(y, F_ASYM, axes, fold)
    assert pty.shape == x.shape
    torch.testing.assert_close((px * y).sum(), (x * pty).sum(), rtol=1e-13, atol=0)
    # and it is what autograd makes of the forward
    xg = x.clone().requires_grad_(True)
    vjp, = torch.autograd.grad(cd._fir_reference(xg, F_ASYM, axes, fold), [xg], y)
    torch.testing.assert_close(pty, vjp, rtol=1e-13, atol=1e-13)


def test_envelope():
    x, wt = _operands(5, 3, True, True, 4, 6, 6)
    assert not cd.in_envelope(x, wt, (2, 1, 1), True, True, F_DOWN)                # CPU tensors
    ok = lambda xs, ws=(4, 3, 5, 3, 3), pad=(2, 1, 1), sd=True, td=True, dt=torch.float32, taps=4: cd.shapes_ok(  # noqa: E731
        xs, ws, dt, pad, sd, td, taps)
    assert ok((2, 3, 4, 6, 6)) and ok((2, 3, 4, 6, 6), dt=torch.float16)
    assert not ok((2, 3, 4, 5, 6))                                                 # odd H
    assert not ok((2, 3, 3, 6, 6), sd=False)                                       # odd T
    assert ok((2, 3, 3, 6, 6), td=False)                                           # odd T is fine when T is kept
    assert not ok((2, 3, 4, 6, 6), pad=(2, 1, 0))                                  # padding other than k // 2
    assert not ok((2, 3, 4, 6, 6), sd=False, td=False)                             # nothing to downsample
    assert not ok((2, 3, 4, 6, 6), taps=5)
    assert not ok((2, 3, 4, 6, 6), dt=torch.float64)
    assert not ok((2, 3, 4, 6, 6), ws=(4, 3, 4, 3, 3), pad=(2, 1, 1))              # even kernel
    assert not ok((2, 3, 4, 6, 6), ws=(4, 3, 9, 3, 3), pad=(4, 1, 1))              # kt beyond the engine's 7


_INSTALL_SCRIPT = r'''
import torch
from torch_utils.ops import conv3d_down as cd
assert 'long-video-gan_b200' in cd.__file__, cd.__file__
from model import discriminator_lres as dl
orig = dl.Conv3dLayer.forward
done = cd.install(dl)
assert done == [dl.Conv3dLayer], done
assert dl.Conv3dLayer.forward is not orig and dl.Conv3dLayer.forward.lvg_conv3d_down is orig
again = cd.install(dl)
assert again == done and dl.Conv3dLayer.forward.lvg_conv3d_down is orig           # idempotent
torch.manual_seed(0)
D = dl.VideoDiscriminator(seq_length=16, max_edge=64, channels_max=64)
assert cd.install(D) == [dl.Conv3dLayer]
x = torch.randn(1, 3, 16, 64, 64)
# CPU tensors are outside the envelope: the installed forward is the reference composition, bit for bit
y_new = D(x)
dl.Conv3dLayer.forward = orig
y_old = D(x)
assert torch.equal(y_new, y_old), (y_new - y_old).abs().max()
# a persistence-style copy of the class in a module of its own is reached through the instance
class Conv3dLayer(dl.Conv3dLayer):
    pass
Conv3dLayer.forward = orig
m = Conv3dLayer(3, 4, 3, 3, spatial_down=True)
assert cd.install(m) == [Conv3dLayer] and Conv3dLayer.forward.lvg_conv3d_down is orig
print('ok')
'''


@pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')
def test_install_patches_the_reference_model_and_falls_back_outside_the_envelope(tmp_path):
    script = tmp_path / 'install_run.py'          # run as a file: `-c` would put the reference's torch_utils first
    script.write_text(_INSTALL_SCRIPT)
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, str(script)], env=env, cwd=SRC, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith('ok'), r.stdout[-3000:]
