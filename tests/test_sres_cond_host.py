"""Host logic of torch_utils/ops/sres_cond.py on the CPU: each layer's plan, evaluated in float64, equals the UNMODIFIED
reference's prep_cond to fp32 rounding (the default and the class-default generator, temporal_context 2, another
margin_size, fourfeats and a third geometry); install() is idempotent, reaches persistence-rebuilt classes and leaves
CPU forwards bitwise unchanged; applies() rejects each case it must; the ABI size query answers without a GPU."""
import os
import subprocess
import sys

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import sres_cond as sc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')


def _run(mode, out_file):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'sres_cond_run.py'), out_file, mode], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out_file, weights_only=False)


@needs_ref
def test_plan_equals_prep_cond(tmp_path):
    res = _run('plan', str(tmp_path / 'plan.pt'))
    assert len(res) == 6 * 15
    kinds = set()
    for r in res:
        assert r['shape_ok'], r
        kinds.add(r['kind'])
        # prep_cond runs in fp32: its rounding, a few ulps of the largest value
        assert r['err'] <= 1e-6 * r['scale'], r
    assert kinds == {'KaiserDownsample', 'KaiserUpsample', 'Identity'}


@needs_ref
def test_install_is_idempotent_reaches_persistence_classes_and_rejects(tmp_path):
    r = _run('install', str(tmp_path / 'install.pt'))
    assert r == {'cpu': 'cpu', 'fp64': 'dtype', 'fp16': 'dtype', 'requires_grad': 'grad', 'requires_grad_no_grad_mode': 'cpu',
                 'resampler': 'resampler', 'taps': 'taps', 'shape': 'shape', 'short_video': 'shape', 'fallback_calls': 1}


def test_axis_matrix_of_hand_built_plans():
    # identity with a crop of 2 and a replicate pad of 1 on each side, over a padded frame 2 wider than the low-res one
    a = sc.axis_plan(4, 4, 1, 'id', 1, 0, False, 4)
    m = sc.axis_matrix(a, None)
    assert (a.x0, a.mhi, a.px0, a.shift) == (1, 3, 0, 1)
    assert torch.equal(m, torch.eye(4, dtype=torch.float64))
    # 2x upsampling by a 4-tap filter [1, 3, 3, 1] / 4 (gain 2 per axis): interior rows hold the polyphase taps
    f = torch.tensor([1., 3., 3., 1.]) / 4
    a = sc.axis_plan(6, 6, 0, 'up', 2, 4, True, 12)
    m = sc.axis_matrix(a, f)
    assert m.shape == (12, 6)
    assert torch.allclose(m.sum(1), torch.full([12], 2.0, dtype=torch.float64))     # every output sees the full gain
    # 2x downsampling: each output row sums to the filter's sum (replicate pads: no zero taps inside the frame)
    a = sc.axis_plan(8, 8, 0, 'down', 2, 4, True, 4)
    m = sc.axis_matrix(a, f)
    assert torch.allclose(m.sum(1), torch.full([4], 2.0, dtype=torch.float64))


def test_abi_size_query_answers_without_a_gpu():
    lib = custom_ops.load_library()
    assert lib.lvg_sres_cond_workspace is not None
    # layer 12 of the default G (up 4, 24 taps) at batch 8 x 8 frames, with and without x_prev
    a_h = sc.axis_plan(36, 64, 10, 'up', 4, 24, True, 164)
    a_w = sc.axis_plan(64, 64, 10, 'up', 4, 24, True, 276)
    f = torch.zeros(24)
    p = sc.Plan(h=a_h, w=a_w, filter=f, window=9)
    for c in (0, 181):
        for dt in (torch.float16, torch.float32):
            assert sc.supported(8, 8, c, 3, 16, p, dt)
    plug = custom_ops.get_plugin('sres_cond_plugin')
    assert plug.workspace(8, 8, 181, 3, 9, 16, 36, 64, torch.float16, sc._ints(a_h), sc._ints(a_w)) % 16 == 0
    assert not sc.supported(8, 9, 181, 3, 16, p, torch.float16)                   # 9 + 8 frames > 16
    assert not sc.supported(8, 8, 181, 3, 16, p, torch.float64)
    assert not sc.supported(8, 8, 181, 3, 16, p._replace(w=a_w._replace(out=30000)), torch.float16)   # tap table too large
    assert not sc.supported(8, 8, 181, 3, 16, p._replace(h=a_h._replace(ntaps=65)), torch.float16)
    with pytest.raises(RuntimeError, match='CUDA'):
        plug.forward(None, torch.zeros(1, 3, 9, 36, 64), f, f, sc._ints(a_h), sc._ints(a_w), 4.0, 4.0, 9, torch.float16, False)
