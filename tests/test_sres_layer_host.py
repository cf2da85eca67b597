"""Host logic of torch_utils/ops/sres_layer.py on the CPU: install() is idempotent, reaches persistence-rebuilt classes,
composes with sres_cond.install and modulated_conv.install in either order and leaves CPU forwards bitwise unchanged;
rejection() names each case it must; the channel -> source mapping of the fused re-tiling pass; the ABI size query
answers without a GPU."""
import os
import subprocess
import sys

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import sres_cond as sc
from torch_utils.ops import sres_layer as sl

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')


@needs_ref
def test_install_composes_falls_through_and_rejects(tmp_path):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUDA_VISIBLE_DEVICES='')
    out = str(tmp_path / 'install.pt')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'sres_layer_run.py'), out, 'install'], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:]
    res = torch.load(out, weights_only=False)
    # one wrapper each, in install order, whatever was installed twice
    assert res[('layer', 'cond')] == ['lvg_sres_cond', 'lvg_sres_layer', 'model']
    assert res[('cond', 'layer')] == ['lvg_sres_layer', 'lvg_sres_cond', 'model']
    assert res['cpu_bitwise'] and res['pickled']
    assert res['reasons'] == {'cpu': 'cpu', 'fp64': 'dtype', 'requires_grad': 'grad', 'resampler': 'resampler',
                              'shape': 'shape', 'fused_shape': ('shape', 'cpu')}
    assert res['fallback_calls'] == 1


def _source(ch, c, window):
    """Where channel ``ch`` of a layer input with ``c`` x_prev channels comes from: ('x', channel) or ('cond', low-res
    channel, frame offset) -- cat((x_prev, cond), 1) with cond's channels (k s) (sres_cond.evaluate's layout)."""
    return ('x', ch) if ch < c else ('cond', (ch - c) // window, (ch - c) % window)


def _block_sources(blk, c, cin, window):
    """conv_pack_cond_kernel's split of 8-channel block ``blk``: j < k0 from x_prev, k0 <= j < k1 conditioning, rest padding."""
    c0 = blk * 8
    k0 = min(max(c - c0, 0), 8)
    k1 = min(max(cin - c0, 0), 8)
    return [('x', c0 + j) if j < k0 else ('cond', (c0 + j - c) // window, (c0 + j - c) % window) if j < k1 else None
            for j in range(8)]


@pytest.mark.parametrize('c', [0, 128, 181, 256, 362, 512, 357])
def test_channel_source_mapping(c):
    window, c_lr = 9, 3
    cin = c + c_lr * window
    cblk = (cin + 15) // 16 * 2                     # the forward's channel blocks (16-channel padding)
    seen = []
    for blk in range(cblk):
        for j, src in enumerate(_block_sources(blk, c, cin, window)):
            ch = blk * 8 + j
            if ch < cin:
                assert src == _source(ch, c, window)
                seen.append(src)
            else:
                assert src is None
    assert seen == [_source(ch, c, window) for ch in range(cin)]
    assert seen[c:] == [('cond', k, s) for k in range(c_lr) for s in range(window)]
    straddles = [b for b in range(cblk) if b * 8 < c < b * 8 + 8]
    assert len(straddles) == (1 if c % 8 else 0)     # layers 10 and 12 (C = 362, 181) have a block of both kinds


def _plan12():
    a_h = sc.axis_plan(36, 64, 10, 'up', 4, 24, True, 164)
    a_w = sc.axis_plan(64, 64, 10, 'up', 4, 24, True, 276)
    return sc.Plan(h=a_h, w=a_w, filter=torch.zeros(24), window=9)


def test_size_query_answers_without_a_gpu():
    p = _plan12()
    for dt in (torch.float16, torch.float32):
        assert sl.supported(8, 8, 181, 3, 16, p, dt, (128, 208, 3, 3), (2, 2))
        assert sl.supported(8, 8, 0, 3, 16, p, dt, (128, 27, 3, 3), (2, 2))
        assert sl.supported(8, 8, 181, 3, 16, p, dt, (3, 208, 1, 1), (0, 0))
    plug = custom_ops.get_plugin('sres_cond_plugin')
    ints = (sc._ints(p.h), sc._ints(p.w))
    assert plug.layer_workspace(8, 8, 181, 3, 9, 16, 36, 64, torch.float16, *ints, 128, 3, 3, 2, 2) % 16 == 0
    assert not sl.supported(8, 8, 181, 3, 16, p, torch.float16, (128, 209, 3, 3), (2, 2))       # Cin != C + 27
    assert not sl.supported(8, 9, 181, 3, 16, p, torch.float16, (128, 208, 3, 3), (2, 2))       # 9 + 8 frames > 16
    assert not sl.supported(8, 8, 181, 3, 16, p, torch.float64, (128, 208, 3, 3), (2, 2))
    assert not sl.supported(8, 8, 181, 3, 16, p, torch.float16, (128, 208, 5, 5), (4, 4))       # > 9 taps per frame
    assert not sl.supported(8, 8, 181, 3, 16, p, torch.float16, (128, 208, 3, 3), (3, 3))       # padding > k - 1
    assert not sl.supported(8, 8, 181, 3, 16, p._replace(h=p.h._replace(ntaps=65)), torch.float16, (128, 208, 3, 3), (2, 2))
    with pytest.raises(RuntimeError, match='CUDA'):
        plug.layer_fprop(None, torch.zeros(8, 3, 16, 36, 64), p.filter, p.filter, *ints, 4.0, 4.0, 9, torch.float16,
                         torch.zeros(128, 27, 3, 3, dtype=torch.float16), torch.zeros(64, 27), None, (2, 2), False)
