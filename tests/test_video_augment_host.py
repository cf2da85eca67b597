"""Host logic of torch_utils/ops/video_augment.py on the CPU: under the same seeds, draw_params + the torch composition give
the input the UNMODIFIED reference LowResVideoGAN.run_D feeds D and leave both generators as the reference leaves them;
the composition's adjoint is exact and its gradients of any order are those of the map; install() patches the reference
class and falls back to the original method on input the op does not take."""
import os
import subprocess
import sys

import pytest
import torch

from torch_utils.ops import video_augment as va

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')


def _run(mode, out_file):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'video_augment_run.py'), out_file, mode], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out_file)


@needs_ref
def test_composition_equals_reference_run_D_and_leaves_the_generators_as_it_does(tmp_path):
    res = _run('cpu', str(tmp_path / 'cpu.pt'))
    assert len(res) == 60
    assert any(r['case'][1] > 0 and bool((r['params'][:, 10] == r['case'][4]).any()) for r in res)      # a clip that keeps T
    for r in res:
        ref, ours = r['ref'], r['ours']
        assert ours.shape == ref.shape, r['case']
        err = float((ours - ref).abs().max() / ref.abs().max())
        assert err <= 1e-6, f'{r["case"]}: {err:.3e}'
        assert r['same_state'], r['case']


@needs_ref
def test_install_is_idempotent_and_falls_back_to_the_original(tmp_path):
    assert _run('install', str(tmp_path / 'install.pt')) == 'ok'


def _params(n, t, t_out, seed, neutral=False):
    """Random parameters in the op's ranges (translation up to 3, cutout anywhere, scale 2^[-1.5, 1.5])."""
    g = torch.Generator().manual_seed(seed)
    p = torch.zeros(n, va.NPAR)
    if not neutral:
        p[:, 0] = torch.rand(n, generator=g) - 0.5
        p[:, 1] = torch.rand(n, generator=g) * 2
        p[:, 2] = torch.rand(n, generator=g) + 0.5
    else:
        p[:, 1:3] = 1
    p[:, 3:5] = torch.randint(-3, 4, (n, 2), generator=g).float()
    p[:, 5] = torch.randint(0, 4, (n,), generator=g).float()
    p[:, 6] = p[:, 5] + torch.randint(-1, 3, (n,), generator=g).float()
    p[:, 7] = torch.randint(0, 4, (n,), generator=g).float()
    p[:, 8] = p[:, 7] + torch.randint(-1, 3, (n,), generator=g).float()
    s = 2 ** (torch.rand(n, generator=g) * 3 - 1.5)
    length = (t * s).floor().clamp_min(1)
    p[:, 9] = (1 / s.double()).float()
    p[:, 10] = length
    p[:, 11] = torch.randint(-3, 4, (n,), generator=g).float() + (length - t_out).clamp_min(0) // 2
    return p


@pytest.mark.parametrize('c', [1, 3, 4])
def test_adjoint_of_the_composition_is_exact(c):
    n, t, h, w, t_out = 3, 9, 7, 8, 11
    p = _params(n, t, t_out, c)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, c, t, h, w, generator=g, dtype=torch.float64)
    y = torch.randn(n, c, t_out, h, w, generator=g, dtype=torch.float64)
    ax = va._reference(x, p, t_out, linear=True)
    aty = va._reference_adjoint(y, p, t)
    torch.testing.assert_close((ax * y).sum(), (x * aty).sum(), rtol=1e-12, atol=0)
    # the affine constant is beta alone
    torch.testing.assert_close(va._reference(x, p, t_out) - ax, va._reference(torch.zeros_like(x), p, t_out), rtol=0, atol=1e-12)


def test_apply_gradients_of_any_order_on_the_cpu():
    n, c, t, h, w = 2, 3, 6, 5, 7
    p = _params(n, t, t, 3)
    x = torch.randn(n, c, t, h, w, dtype=torch.float64, requires_grad=True)
    y = va.apply(x, p, t)
    torch.testing.assert_close(y, va._reference(x, p, t))
    dy = torch.randn_like(y)
    gx, = torch.autograd.grad(y, [x], dy, create_graph=True)
    torch.testing.assert_close(gx, va._reference_adjoint(dy, p, t))
    # second order through the adjoint: d/d(dy) |A^T dy|^2 = 2 A (A^T dy), the linear forward
    gdy, = torch.autograd.grad(y, [x], dy.requires_grad_(True), create_graph=True)
    hdy, = torch.autograd.grad(gdy.square().sum(), [dy])
    torch.testing.assert_close(hdy, va._reference(2 * gdy.detach(), p, t, linear=True))


def test_policy_and_envelope_rules():
    assert va.steps_of('color,translation,cutout') == (True, True, True)
    assert va.steps_of('') == (False, False, False)
    assert va.steps_of('translation') == (False, True, False)
    assert va.steps_of('cutout,color') is None and va.steps_of('color,color') is None and va.steps_of('zoom') is None
    x = torch.zeros(2, 3, 16, 6, 8)
    assert not va.applies(x, 'color', 0.0, 16)                               # CPU video
    with pytest.raises(ValueError):
        va.draw_params(x, 'cutout,color', 0.0, 16)
    p = va.draw_params(x, 'translation', 0.0, 16)                             # defaults of the absent steps are neutral
    assert p.shape == (2, va.NPAR)
    assert torch.equal(p[:, [0, 1, 2, 5, 6, 7, 8, 9, 10, 11]], torch.tensor([0., 1., 1., 0., -1., 0., -1., 1., 16., 0.]).expand(2, 10))
    assert p[:, 3:5].abs().max() <= 2                                         # round(max(6, 8) / 4)


def test_abi_entries_answer_without_a_gpu():
    from torch_utils import custom_ops
    lib = custom_ops.load_library()
    # (n, c, t_in, h, w, t_out): per-sample partial sums of at most 256 CTAs, 4 bytes each
    assert lib.lvg_video_augment_workspace(8, 3, 128, 36, 64, 128) == 8 * 108 * 4
    assert lib.lvg_video_augment_workspace(1, 4, 2, 3, 5, 7) == 4
    assert lib.lvg_video_augment_workspace(1, 5, 2, 3, 5, 7) == -1
    assert lib.lvg_video_augment(None, None, None, None, 1, 5, 2, 3, 5, 7, 0, None) == -1
    assert lib.lvg_video_augment(None, None, None, None, 1, 3, 2, 3, 5, 7, 0, None) == 1
    assert lib.lvg_video_augment_adjoint(None, None, None, None, 1, 3, 2, 3, 5, 7, None) == 1
