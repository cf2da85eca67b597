"""Host logic of torch_utils/ops/gblock_conv0.py on the CPU: the size query and argument checks of lvg_gblock_conv0 through
ctypes, the mode of each call, install() idempotence and composition with gblock_tail, modulated_conv and lres_torgb in
every order, classes rebuilt by persistence, calls outside the envelope running the replaced method bit for bit, and the
block forwards the install runs reproducing the reference bit for bit around the reference's first layer."""
import itertools
import os
import subprocess
import sys
import types

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import gblock_conv0 as gc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')
F16, F32, F64 = torch.float16, torch.float32, torch.float64
K3, K1 = ((3, 3, 3), (1, 1, 1)), ((1, 3, 3), (0, 1, 1))


def test_size_query_answers_without_a_gpu():
    plug = custom_ops.get_plugin('gblock_conv0_plugin')
    for dt in (F16, F32):
        assert plug.workspace(dt, 8, 512, 512, 96, 9, 16, *K3) > 0                # the default G's 512-channel conv_0
        assert plug.workspace(dt, 8, 64, 64, 128, 36, 64, *K1) > 0                 # its last block
        assert plug.workspace(dt, 1, 40, 40, 1, 7, 9, *K3) % 256 == 0              # odd shape: 40 channels, T = 1
    assert plug.workspace(F64, 8, 64, 64, 16, 36, 64, *K1) == -1                  # fp16 / fp32 only
    assert plug.workspace(F32, 8, 64, 64, 16, 36, 64, (3, 3, 3), (0, 1, 1)) == -1  # the output keeps the frame count
    assert plug.workspace(F32, 8, 64, 64, 16, 36, 64, (1, 5, 5), (0, 2, 2)) == -1  # at most 9 spatial taps
    assert plug.workspace(F32, 0, 64, 64, 16, 36, 64, *K1) == -1
    # the forward's room holds one partial per (tile, warp): it grows with the frames
    assert plug.workspace(F32, 8, 64, 64, 128, 36, 64, *K1) > plug.workspace(F32, 8, 64, 64, 16, 36, 64, *K1)


def test_argument_errors_without_a_gpu():
    plug = custom_ops.get_plugin('gblock_conv0_plugin')
    x = torch.zeros(2, 64, 4, 9, 16)
    w = torch.zeros(64, 64, 1, 3, 3)
    with pytest.raises(RuntimeError, match='CUDA'):
        plug.fprop(x, w, torch.zeros(2, 64, 4), torch.zeros(2, 64, 4), None, (0, 1, 1), 2, 0.2, 2 ** 0.5, 256.0)
    lib = custom_ops.load_library()
    dims = (0, 2, 64, 64, 4, 9, 16, 1, 3, 3, 0, 1, 1)
    rc = lib.lvg_gblock_conv0_fprop(*([None] * 7), *dims, 2, 0.2, 1.4, 256.0, None, 0, None)
    assert rc != 0 and b'must not be NULL' in lib.lvg_last_error()
    rc = lib.lvg_gblock_conv0_fprop(*([None] * 7), *dims, 3, 0.2, 1.4, 256.0, None, 0, None)        # act: linear / lrelu only
    assert rc == custom_ops.LVG_UNSUPPORTED
    rc = lib.lvg_gblock_conv0_fprop(*([None] * 7), 2, *dims[1:], 2, 0.2, 1.4, 256.0, None, 0, None)  # fp64
    assert rc == custom_ops.LVG_UNSUPPORTED
    rc = lib.lvg_gblock_conv0_backward(*([None] * 12), *dims, 2, 0.2, 1.4, 256.0, None, 0, None)
    assert rc != 0 and b'must not be NULL' in lib.lvg_last_error()
    rc = lib.lvg_gblock_conv0_backward(*([None] * 12), *dims[:7], 3, 3, 3, 0, 1, 1, 2, 0.2, 1.4, 256.0, None, 0, None)
    assert rc == custom_ops.LVG_UNSUPPORTED


def test_cpu_and_fp64_calls_are_outside_the_envelope():
    x = torch.zeros(2, 64, 4, 9, 16)
    assert not gc.supported(x, F32, (64, 64, 1, 3, 3), (0, 1, 1), 'lrelu')
    assert not gc.supported(x.double(), F64, (64, 64, 1, 3, 3), (0, 1, 1), 'lrelu')


def test_mode_of_each_call():
    B = types.SimpleNamespace(magnitude_ema=True, parameters=lambda: iter([torch.zeros(1, requires_grad=True)]))
    x, lat = torch.zeros(1), torch.zeros(1)
    assert gc.mode(B, x, lat, 1.0) == 'backward'                                  # update_G
    assert gc.mode(B, x, lat, 0.999) is None
    with torch.no_grad():
        assert gc.mode(B, x, lat, 1.0) == 'forward'                               # inference
        assert gc.mode(B, x, lat, 0.999) == 'stat'
    frozen = types.SimpleNamespace(magnitude_ema=True, parameters=lambda: iter([torch.zeros(1)]))
    assert gc.mode(frozen, x, lat, 0.999) == 'stat'                               # update_D's generated pass
    assert gc.mode(frozen, x.requires_grad_(True), lat, 1.0) == 'backward'
    assert set(gc._MODES) <= {'backward', 'stat', 'forward'}


@needs_ref
def test_install_composes_reaches_persistence_classes_and_falls_back(tmp_path):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUDA_VISIBLE_DEVICES='')
    out = str(tmp_path / 'install.pt')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'gblock_conv0_run.py'), out, 'install'], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:]
    res = torch.load(out, weights_only=False)
    for order in itertools.permutations(('conv0', 'tail', 'modconv', 'torgb')):
        # one wrapper of each block op on Synthesis3dResBlock.forward whatever was installed twice and in which order
        assert res[order] == (['lvg_gblock_conv0', 'lvg_gblock_tail', 'model'], True, True), order
    assert res['pickled']
    assert res['cpu_bitwise'] and res['fallback_calls'] == 3
    assert res['supported'] == [False, False]
    assert res['block_forward_bitwise']
