"""Host logic of torch_utils/ops/lres_torgb.py on the CPU: the size query and argument checks of lvg_lres_torgb through
ctypes, the mode of each call, install() idempotence and composition with modulated_conv and gblock_tail in every order,
classes rebuilt by persistence, and calls outside the envelope running the replaced method bit for bit."""
import itertools
import os
import subprocess
import sys
import types

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import lres_torgb as lt

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')
F16, F32, F64 = torch.float16, torch.float32, torch.float64


def test_size_query_answers_without_a_gpu():
    plug = custom_ops.get_plugin('lres_torgb_plugin')
    for xd, dt in itertools.product((F16, F32), (F16, F32)):
        assert plug.workspace(xd, dt, 8, 64, 160, 36, 64, 3) > 0                  # the default G's layer
        assert plug.workspace(xd, dt, 1, 45, 1, 23, 37, 3) % 256 == 0              # odd shape: scalar loads
    assert plug.workspace(F32, F32, 8, 64, 160, 36, 64, 4) == -1                  # 3 output channels only
    assert plug.workspace(F32, F32, 8, 64, 160, 36, 64, 3, (1, 3, 3)) == -1       # a 1 x 1 x 1 kernel only
    assert plug.workspace(F32, F32, 8, 64, 160, 36, 64, 3, (3, 1, 1)) == -1
    assert plug.workspace(F64, F32, 8, 64, 160, 36, 64, 3) == -1                  # fp16 / fp32 only
    assert plug.workspace(F32, F64, 8, 64, 160, 36, 64, 3) == -1
    assert plug.workspace(F32, F32, 8, 513, 16, 36, 64, 3) == -1                  # at most 512 input channels
    assert plug.workspace(F32, F32, 0, 64, 16, 36, 64, 3) == -1
    # the workspace holds every CTA's partial Gram sums and every plane's fold
    small = plug.workspace(F32, F32, 1, 64, 1, 36, 64, 3)
    assert plug.workspace(F32, F32, 8, 64, 160, 36, 64, 3) >= 8 * 160 * small // 2


def test_argument_errors_without_a_gpu():
    plug = custom_ops.get_plugin('lres_torgb_plugin')
    x = torch.zeros(2, 64, 4, 36, 64)
    with pytest.raises(RuntimeError, match='CUDA'):
        plug.fprop(x, torch.zeros(3, 64), torch.zeros(2, 64, 4), torch.zeros(3), F32, 256.0)
    lib = custom_ops.load_library()
    rc = lib.lvg_lres_torgb_fprop(None, None, None, None, None, None, None, 0, 0, 2, 64, 4, 36, 64, 3, 256.0, None, 0, None)
    assert rc != 0 and b'must not be NULL' in lib.lvg_last_error()
    rc = lib.lvg_lres_torgb_fprop(None, None, None, None, None, None, None, 0, 0, 2, 64, 4, 36, 64, 4, 256.0, None, 0, None)
    assert rc == custom_ops.LVG_UNSUPPORTED
    rc = lib.lvg_lres_torgb_fprop(None, None, None, None, None, None, None, 2, 0, 2, 64, 4, 36, 64, 3, 256.0, None, 0, None)
    assert rc == custom_ops.LVG_UNSUPPORTED
    rc = lib.lvg_lres_torgb_backward(*([None] * 9), 0, 0, 2, 64, 4, 36, 64, 3, 256.0, None, 0, None)
    assert rc != 0 and b'must not be NULL' in lib.lvg_last_error()
    rc = lib.lvg_lres_torgb_finish(None, None, None, None, 0, 2, 4, 36, 64, 256.0, None)
    assert rc != 0 and b'must not be NULL' in lib.lvg_last_error()


def test_cpu_and_fp64_calls_are_outside_the_envelope():
    x = torch.zeros(2, 64, 4, 36, 64)
    assert not lt.supported(x, F32, (3, 64, 1, 1, 1))
    assert not lt.supported(x.double(), F64, (3, 64, 1, 1, 1))


def test_mode_of_each_call():
    L = types.SimpleNamespace(magnitude_ema=True, parameters=lambda: iter([torch.zeros(1, requires_grad=True)]))
    x, lat = torch.zeros(1), torch.zeros(1)
    assert lt.mode(L, x, lat, 1.0) == 'backward'
    assert lt.mode(L, x, lat, 0.999) is None
    with torch.no_grad():
        assert lt.mode(L, x, lat, 1.0) == 'forward'
        assert lt.mode(L, x, lat, 0.999) == 'stat'
    frozen = types.SimpleNamespace(magnitude_ema=True, parameters=lambda: iter([torch.zeros(1)]))
    assert lt.mode(frozen, x, lat, 0.999) == 'stat'                                # update_D: G's parameters frozen
    assert lt.mode(frozen, x.requires_grad_(True), lat, 1.0) == 'backward'
    no_ema = types.SimpleNamespace(magnitude_ema=False, parameters=lambda: iter([torch.zeros(1)]))
    assert lt.mode(no_ema, torch.zeros(1), lat, 0.999) == 'forward'


@needs_ref
def test_install_composes_reaches_persistence_classes_and_falls_back(tmp_path):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUDA_VISIBLE_DEVICES='')
    out = str(tmp_path / 'install.pt')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'lres_torgb_run.py'), out, 'install'], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:]
    res = torch.load(out, weights_only=False)
    for order in itertools.permutations(('torgb', 'modconv', 'tail')):
        # one wrapper on ToRGB.forward whatever was installed twice and in which order; the other installs in place
        assert res[order] == (['lvg_lres_torgb', 'model'], True, True), order
    assert res['pickled']
    assert res['cpu_bitwise'] and res['fallback_calls'] == 3
    assert res['supported'] == [False, False]
