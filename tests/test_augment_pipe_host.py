"""Host logic of torch_utils/ops/augment_pipe.py on the CPU: under the same seeds, draw_params + the torch composition give
the output of the UNMODIFIED reference AugmentPipe in both super-res configurations and leave the generator as it does;
the margins equal the reference's F.pad arguments; the composition's adjoint is exact and its gradients of any order are
those of the map; install() patches the reference class and falls back to the original method; the ABI entries answer
without a GPU; and the host build of the kernels' coordinate / weight function shows that the adjoint's enumeration box
holds every point with a non-zero weight."""
import math
import os
import shutil
import subprocess
import sys

import pytest
import torch

from torch_utils.ops import augment_pipe as ap
from torch_utils.ops import upfirdn2d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')


def _run(mode, out_file):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'augment_pipe_run.py'), out_file, mode], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out_file, weights_only=False)


@needs_ref
def test_composition_equals_the_reference_pipe_and_its_pad_arguments(tmp_path):
    res = _run('cpu', str(tmp_path / 'cpu.pt'))
    assert len(res) == 8
    for r in res:
        ref, ours = r['ref'], r['ours']
        assert ours.shape == ref.shape, r['case']
        err = float((ours - ref).abs().max() / ref.abs().max())
        assert err <= 1e-6, f'{r["case"]}: {err:.3e}'
        assert r['same_state'], r['case']
        assert r['flags'] == ap.GEOM
        # the reference's F.pad(videos, [mx0, mx1, my0, my1], mode='reflect') against the native margins
        m = [int(v) for v in r['params'][0, :4]]
        assert r['pads'] == [[m[0], m[2], m[1], m[3]]], r['case']
        assert torch.equal(r['params'][:, :4], r['params'][:1, :4].expand(r['params'].shape[0], 4))


@needs_ref
def test_install_is_idempotent_and_falls_back_to_the_original(tmp_path):
    assert _run('install', str(tmp_path / 'install.pt')) == 'ok'


def _filter():
    return upfirdn2d.setup_filter([0.0154041093, 0.0034907121, -0.1179901111, -0.0483117426, 0.4910559419, 0.7876411410,
                                   0.3379294217, -0.0726375228, -0.0210602925, 0.0447249018, 0.0017677119, -0.0078007083])


def _params(n, h, w, seed, rot=0.3, scale=1.2, margins=None):
    """theta of a rotation + scale + translation through the reference's conjugation chain, random colour and noise."""
    g = torch.Generator().manual_seed(seed)
    m = margins or [int(v) for v in torch.randint(0, min(h, w) - 1, (4,), generator=g)]
    m[0], m[2] = min(m[0], w - 1), min(m[2], w - 1)
    m[1], m[3] = min(m[1], h - 1), min(m[3], h - 1)
    p = torch.zeros(n, ap.NPAR, dtype=torch.float64)
    p[:, :4] = torch.tensor(m, dtype=torch.float64)
    uw, uh, vw, vh = 2 * (w + m[0] + m[2]), 2 * (h + m[1] + m[3]), 2 * w + 12, 2 * h + 12
    for i in range(n):
        a = rot * (i + 1)
        c, s = math.cos(a) * scale, math.sin(a) * scale
        G = torch.tensor([[c, -s, 0.7 * i - 0.4], [s, c, -0.3 * i + 0.2], [0, 0, 1]], dtype=torch.float64)
        T = lambda tx, ty: torch.tensor([[1, 0, tx], [0, 1, ty], [0, 0, 1]], dtype=torch.float64)   # noqa: E731
        S = lambda sx, sy: torch.diag(torch.tensor([sx, sy, 1.0], dtype=torch.float64))             # noqa: E731
        G = T((m[0] - m[2]) / 2, (m[1] - m[3]) / 2) @ G
        G = S(2, 2) @ G @ S(0.5, 0.5)
        G = T(-0.5, -0.5) @ G @ T(0.5, 0.5)
        G = S(2 / uw, 2 / uh) @ G @ S(vw / 2, vh / 2)
        p[i, 4:10] = G[:2].reshape(6)
    p[:, 10:22] = (torch.eye(4, dtype=torch.float64)[:3] + 0.3 * torch.randn(n, 3, 4, generator=g, dtype=torch.float64)).view(n, 12)
    p[:, 22] = torch.rand(n, generator=g, dtype=torch.float64)
    return p.float()


@pytest.mark.parametrize('flags', [0, ap.GEOM])
def test_adjoint_of_the_composition_is_exact(flags):
    n, t, h, w = 2, 2, 9, 13
    p = _params(n, h, w, 1)
    f = _filter()
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, 3, t, h, w, generator=g, dtype=torch.float64)
    y = torch.randn(n, 3, t, h, w, generator=g, dtype=torch.float64)
    ax = ap._reference(x, p, None, f, flags, linear=True)
    aty = ap._reference_adjoint(y, p, f, flags)
    torch.testing.assert_close((ax * y).sum(), (x * aty).sum(), rtol=1e-12, atol=0)
    # the affine constant is C[:3,3] + sigma noise alone
    noise = torch.randn(x.shape, generator=g, dtype=torch.float64)
    torch.testing.assert_close(ap._reference(x, p, noise, f, flags) - ax, ap._reference(torch.zeros_like(x), p, noise, f, flags),
                               rtol=0, atol=1e-12)


def test_apply_gradients_of_any_order_on_the_cpu():
    n, t, h, w = 2, 2, 9, 11
    p = _params(n, h, w, 3, margins=[8, 8, 10, 3])
    f = _filter()
    x = torch.randn(n, 3, t, h, w, dtype=torch.float64, requires_grad=True)
    noise = torch.randn(n, 3, t, h, w, dtype=torch.float64)
    y = ap.apply(x, p, noise, f, ap.GEOM)
    torch.testing.assert_close(y, ap._reference(x, p, noise, f, ap.GEOM))
    dy = torch.randn_like(y)
    gx, = torch.autograd.grad(y, [x], dy, create_graph=True)
    torch.testing.assert_close(gx, ap._reference_adjoint(dy, p, f, ap.GEOM))
    # second order through the adjoint: d/d(dy) |A^T dy|^2 = 2 A (A^T dy), the linear forward
    gdy, = torch.autograd.grad(y, [x], dy.requires_grad_(True), create_graph=True)
    hdy, = torch.autograd.grad(gdy.square().sum(), [dy])
    torch.testing.assert_close(hdy, ap._reference(2 * gdy.detach(), p, None, f, ap.GEOM, linear=True))


def test_envelope_rules_on_the_cpu():
    class Pipe:                         # the attributes applies() and flags_of() read
        imgfilter = cutout = 0
        Hz_geom = _filter()
        xflip = rotate90 = xint = scale = rotate = aniso = xfrac = 0.0
    pipe = Pipe()
    assert ap.flags_of(pipe) == 0
    pipe.xfrac = 1.0
    assert ap.flags_of(pipe) == ap.GEOM
    assert not ap.applies(pipe, torch.zeros(2, 3, 4, 9, 15))                  # CPU video: the original runs


def test_abi_entries_answer_without_a_gpu():
    from torch_utils import custom_ops
    lib = custom_ops.load_library()
    # (n, c, t, h, w, flags): the adjoint's D^T C^T dy on the (2h + 12) x (2w + 12) grid, fp32
    assert lib.lvg_augment_pipe_workspace(8, 3, 8, 144, 256, ap.GEOM) == 8 * 3 * 8 * 300 * 524 * 4
    assert lib.lvg_augment_pipe_workspace(8, 3, 8, 144, 256, 0) == 0
    assert lib.lvg_augment_pipe_workspace(8, 4, 8, 144, 256, ap.GEOM) == -1
    assert lib.lvg_augment_pipe(None, None, None, 12, None, None, 1, 4, 2, 3, 5, 1, None) == -1
    assert lib.lvg_augment_pipe(None, None, None, 11, None, None, 1, 3, 2, 3, 5, 1, None) == -1
    assert lib.lvg_augment_pipe(None, None, None, 12, None, None, 1, 3, 2, 3, 5, 1, None) == 1
    assert lib.lvg_augment_pipe_adjoint(None, None, None, 12, None, None, 1, 3, 2, 3, 5, 1, None) == 1


@pytest.mark.skipif(shutil.which('nvcc') is None, reason='nvcc not on PATH')
def test_enumeration_box_holds_every_point_with_a_non_zero_weight(tmp_path):
    exe = str(tmp_path / 'augment_pipe_emul')
    build = subprocess.run(['nvcc', '-O2', '-std=c++17', '-o', exe, os.path.join(ROOT, 'tools', 'augment_pipe_emul.cu')],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert build.returncode == 0, build.stdout[-3000:]
    run = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert run.returncode == 0 and 'all ok' in run.stdout, run.stdout[-3000:]
    for name in ('rot45_clamped', 'scale_0.25', 'scale_4', 'aniso', 'xflip1_rot90x3', 'random_11', 'train_shape_rot'):
        assert f'{name} ' in run.stdout
