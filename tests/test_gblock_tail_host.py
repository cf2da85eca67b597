"""Host logic of torch_utils/ops/gblock_tail.py on the CPU: the installed block forward with the tail as the torch
composition gives the UNMODIFIED reference Synthesis3dResBlock.forward exactly (magnitude-EMA beta 1) or to rounding
(beta 0.9, the input gain folded into the convolution weights) for every block of the default and a 64 x 64 generator and
for standalone blocks with both flags and odd crops, and leaves the same buffers; install() is idempotent, reaches
persistence-rebuilt classes and falls back outside the envelope; the crop offsets and output sizes are center_crop's; the
composition's gradients of any order are those of the map; and the ABI size query answers without a GPU."""
import os
import subprocess
import sys

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import gblock_tail as gt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')


def _run(mode, out_file):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'gblock_tail_run.py'), out_file, mode], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out_file, weights_only=False)


@needs_ref
def test_composition_equals_the_reference_block_forward(tmp_path):
    res = _run('cpu', str(tmp_path / 'cpu.pt'))
    assert len(res) == 10 + 10 + 5
    flags = set()
    for r in res:
        sig = r['sig']
        flags.add(sig[4:6])
        exact = r['res'][1.0]
        assert exact['ours'].shape == exact['ref'].shape, sig
        assert torch.equal(exact['ours'], exact['ref']), f'{sig}: {float((exact["ours"] - exact["ref"]).abs().max()):.3e}'
        assert exact['same_buffers'], sig
        ema = r['res'][0.9]
        err = float((ema['ours'] - ema['ref']).abs().max() / ema['ref'].abs().max())
        assert err <= 1e-5, f'{sig}: {err:.3e}'
        assert ema['buf_err'] <= 1e-6, sig
    assert flags == {(True, True), (True, False), (False, True), (False, False)}


@needs_ref
def test_install_is_idempotent_reaches_persistence_classes_and_falls_back(tmp_path):
    assert _run('install', str(tmp_path / 'install.pt')) == 'ok'


def _center_crop(x, width=None, height=None, seq_length=None):
    # generator_lres.center_crop (model/generator_lres.py:131-155)
    if width is not None:
        x0 = (x.size(4) - width) // 2
        x = x[:, :, :, :, x0:x0 + width]
    if height is not None:
        y0 = (x.size(3) - height) // 2
        x = x[:, :, :, y0:y0 + height]
    if seq_length is not None:
        t0 = (x.size(2) - seq_length) // 2
        x = x[:, :, t0:t0 + seq_length]
    return x


def test_crop_offsets_and_sizes_are_center_crops():
    for t in range(1, 9):
        for h in range(1, 7):
            for w in (1, 2, 5, 8):
                for tup in (False, True):
                    for sup in (False, True):
                        tu, hu, wu = t * (1 + tup), h * (1 + sup), w * (1 + sup)
                        x = torch.arange(tu * hu * wu).view(1, 1, tu, hu, wu)
                        for to in {None, 1, tu // 2 + 1, tu}:
                            for ho, wo in ((None, None), (hu, wu), (max(1, hu - 1), max(1, wu - 3))):
                                (a, b, c), (ot, oh, ow) = gt.out_shape((t, h, w), tup, sup, to, ho, wo)
                                y = _center_crop(x, width=wo, height=ho, seq_length=to)
                                assert tuple(y.shape[2:]) == (a, b, c)
                                assert int(y[0, 0, 0, 0, 0]) == (ot * hu + oh) * wu + ow
                                assert torch.equal(gt._crop(x, wo, ho, to), y)


def _small(dtype=torch.float64):
    g = torch.Generator().manual_seed(3)
    s = torch.randn(2, 3, 4, 3, 5, generator=g, dtype=dtype)
    h = torch.randn(2, 3, 4, 3, 5, generator=g, dtype=dtype)
    b = torch.randn(3, generator=g, dtype=dtype)
    return s, h, b


@pytest.mark.parametrize('tup,sup,crop', [(True, True, (7, 5, 9)), (False, True, (3, 6, 7)), (True, False, (6, None, None)),
                                          (False, False, (3, 2, 4))])
def test_composition_is_the_reference_op_sequence_and_differentiable(tup, sup, crop):
    s, h, b = _small()
    s.requires_grad_(True)
    b.requires_grad_(True)
    z = gt.gblock_tail(s, h, b, temporal_up=tup, spatial_up=sup, seq_length=crop[0], height=crop[1], width=crop[2], act='lrelu',
                       clamp=None)
    (to, ho, wo), _ = gt.out_shape(tuple(s.shape[2:]), tup, sup, *crop)
    assert tuple(z.shape) == (2, 3, to, ho, wo)
    # the map is piecewise linear: gradients of any order through the torch composition
    assert torch.autograd.gradcheck(lambda s_, b_: gt.gblock_tail(s_, h, b_, temporal_up=tup, spatial_up=sup, seq_length=crop[0],
                                                                  height=crop[1], width=crop[2], act='linear', clamp=None), (s, b))
    assert torch.autograd.gradgradcheck(lambda s_: gt.gblock_tail(s_, h, b, temporal_up=tup, spatial_up=sup, seq_length=crop[0],
                                                                  height=crop[1], width=crop[2], act='swish', clamp=None), (s,))


def test_abi_size_query_answers_without_a_gpu():
    lib = custom_ops.load_library()
    # (n, c, t, h, w, t_out, h_out, w_out, flags): the largest block of the default G and its crops
    assert lib.lvg_gblock_tail_workspace(8, 64, 160, 18, 32, 160, 36, 64, 2) > 0
    assert lib.lvg_gblock_tail_workspace(8, 512, 26, 3, 4, 36, 5, 8, 3) > 0
    assert lib.lvg_gblock_tail_workspace(8, 256, 176, 9, 16, 160, 9, 16, 0) > 0
    assert lib.lvg_gblock_tail_workspace(8, 64, 160, 18, 32, 161, 36, 64, 2) == -1       # crop larger than the axis
    assert lib.lvg_gblock_tail_workspace(8, 64, 160, 18, 32, 160, 37, 64, 2) == -1
    assert lib.lvg_gblock_tail_workspace(8, 64, 160, 18, 32, 160, 36, 64, 4) == -1       # unknown flag
    assert lib.lvg_gblock_tail_workspace(1, 1, 4, 4, 4096, 8, 8, 8192, 3) == -1          # a dv row beyond the adjoint's tile
    p = custom_ops.get_plugin('gblock_tail_plugin')
    assert p.workspace(8, 64, 160, 18, 32, 160, 36, 64, 2) % 16 == 0
    with pytest.raises(RuntimeError, match='CUDA'):
        p.forward(torch.zeros(1, 1, 2, 2, 4), torch.zeros(1, 1, 2, 2, 4), None, (2, 2, 4), 0, 3, 0.2, 1.0, -1.0, False)
