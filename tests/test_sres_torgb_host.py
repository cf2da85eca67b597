"""Host logic of torch_utils/ops/sres_torgb.py on the CPU: the size query and argument checks of lvg_sres_torgb through
ctypes, rejection() reasons, install() idempotence and composition with sres_cond, sres_layer and modulated_conv in any
order, and that without the install the generator's forward calls exactly what it called before."""
import itertools
import os
import subprocess
import sys

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import sres_cond as sc
from torch_utils.ops import sres_torgb as st

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

SC, SL, ST = 'torch_utils.ops.sres_cond', 'torch_utils.ops.sres_layer', 'torch_utils.ops.sres_torgb'
needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')


def _plan14():
    a_h = sc.axis_plan(36, 64, 10, 'up', 4, 24, True, 144)
    a_w = sc.axis_plan(64, 64, 10, 'up', 4, 24, True, 256)
    return sc.Plan(h=a_h, w=a_w, filter=torch.zeros(24), window=9)


def test_size_query_answers_without_a_gpu():
    p = _plan14()
    ints = (sc._ints(p.h), sc._ints(p.w))
    plug = custom_ops.get_plugin('sres_cond_plugin')
    for dt in (torch.float16, torch.float32):
        assert st.supported(8, 8, 128, 3, 16, p, dt, 3)
        assert st.supported(1, 1, 45, 3, 9, p, dt, 3)                     # x_prev channels not a multiple of 8
        assert plug.torgb_workspace(8, 8, 128, 3, 9, 16, 36, 64, dt, *ints, 3) % 256 == 0
    assert not st.supported(8, 8, 128, 3, 16, p, torch.float16, 4)         # 3 output channels only
    assert not st.supported(8, 8, 1000, 3, 16, p, torch.float16, 3)        # more than 1024 input channels
    assert not st.supported(8, 9, 128, 3, 16, p, torch.float16, 3)         # 9 + 8 frames > 16
    assert not st.supported(8, 8, 128, 3, 16, p, torch.float64, 3)
    assert not st.supported(8, 8, 128, 3, 16, p._replace(h=p.h._replace(ntaps=65)), torch.float16, 3)
    wide = p._replace(w=sc.axis_plan(64, 64, 10, 'up', 4, 24, True, 2056))  # an output row wider than one CTA's tile
    assert plug.torgb_workspace(8, 8, 128, 3, 9, 16, 36, 64, torch.float16, sc._ints(wide.h), sc._ints(wide.w), 3) == -1
    with pytest.raises(RuntimeError, match='ints per axis'):
        plug.torgb_workspace(8, 8, 128, 3, 9, 16, 36, 64, torch.float16, ints[0][:9], ints[1], 3)


def test_argument_errors_without_a_gpu():
    p = _plan14()
    ints = (sc._ints(p.h), sc._ints(p.w))
    plug = custom_ops.get_plugin('sres_cond_plugin')
    lr = torch.zeros(8, 3, 16, 36, 64)
    x = torch.zeros(64, 128, 144, 256, dtype=torch.float16)
    w = torch.zeros(3, 155, dtype=torch.float16)
    with pytest.raises(RuntimeError, match='CUDA'):
        plug.torgb_fprop(x, lr, p.filter, p.filter, *ints, 4.0, 4.0, 9, torch.float16, w, torch.zeros(64, 155),
                         torch.zeros(3, dtype=torch.float16), 256, False)
    # the C entry points check their arguments before any launch
    lib = custom_ops.load_library()
    ph, pw = (ctypes_ints(q) for q in ints)
    st5 = (custom_ops._c_i64 * 5)(*lr.stride())
    rc = lib.lvg_sres_torgb_fprop(None, None, None, None, None, None, None, None, None, 1, 1, 8, 8, 128, 3, 9, 16, 36, 64,
                                  st5, ph, pw, 4.0, 4.0, 3, 256.0, None)
    assert rc != 0 and b'must not be NULL' in lib.lvg_last_error()
    rc = lib.lvg_sres_torgb_fprop(None, None, None, None, None, None, None, None, None, 1, 1, 8, 8, 128, 3, 9, 16, 36, 64,
                                  st5, ph, pw, 4.0, 4.0, 4, 256.0, None)
    assert rc == custom_ops.LVG_UNSUPPORTED
    rc = lib.lvg_sres_torgb_backward(*([None] * 12), 1, 1, 8, 8, 128, 3, 9, 16, 36, 64, st5, ph, pw, 4.0, 4.0, 3, None, 0, None)
    assert rc != 0 and b'must not be NULL' in lib.lvg_last_error()


def ctypes_ints(q):
    return (custom_ops._c_int * len(q))(*q)


def test_synthesis_forward_hook_defaults_to_todays_path(monkeypatch):
    """Without a ``torgb`` forward every layer, the ToRGB one included, runs ``layer_forward`` with the same arguments."""
    calls = []

    def spy(L, g, x, lr, plan, w, **kw):
        calls.append((L.name, 'layer', tuple(sorted(kw))))
        return x
    monkeypatch.setattr(sc, 'layer_forward', spy)

    class Layer:
        def __init__(self, name, torgb):
            self.name, self.is_torgb = name, torgb

    class S:
        layer_names = ['L0', 'L1', 'L2_rgb']
        num_ws, w_dim, fourfeats, output_scale = 3, 4, False, 1
        img_channels, img_height, img_width = 3, 2, 2
        L0, L1, L2_rgb = Layer('L0', False), Layer('L1', False), Layer('L2_rgb', True)

    class Misc:
        @staticmethod
        def assert_shape(*a):
            pass
    g = {'misc': Misc}
    ws = torch.zeros(1, 3, 4)
    lr = torch.zeros(1, 3, 3, 2, 2)
    with pytest.raises(AttributeError):                      # x is None at the end: the layers were all reached
        sc.synthesis_forward(S, g, ws, lr, [None] * 3, update_emas=True, step='step')
    assert calls == [(n, 'layer', ('step', 'update_emas')) for n in ('L0', 'L1', 'L2_rgb')]
    calls.clear()

    def torgb(L, g, x, lr, plan, w, **kw):
        calls.append((L.name, 'torgb', tuple(sorted(kw))))
        return x
    with pytest.raises(AttributeError):
        sc.synthesis_forward(S, g, ws, lr, [None] * 3, torgb=torgb, update_emas=True, step='step')
    assert calls == [('L0', 'layer', ('step', 'update_emas')), ('L1', 'layer', ('step', 'update_emas')),
                     ('L2_rgb', 'torgb', ('step', 'update_emas'))]


@needs_ref
def test_install_composes_falls_through_and_rejects(tmp_path):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUDA_VISIBLE_DEVICES='')
    out = str(tmp_path / 'install.pt')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'sres_torgb_run.py'), out, 'install'], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:]
    res = torch.load(out, weights_only=False)
    attr = {'torgb': 'lvg_sres_torgb', 'layer': 'lvg_sres_layer', 'cond': 'lvg_sres_cond'}
    for order in itertools.permutations(('torgb', 'layer', 'cond')):
        # one wrapper each, last install on top, whatever was installed twice ...
        assert res['chains'][order] == [attr[o] for o in reversed(order)] + ['model']
        # ... and in every order a call that records a backward runs the ToRGB layer through the op and the other layers
        # through sres_layer's step; forward-only calls run as without sres_torgb.install (sres_layer's fused forward)
        assert res['routes'][order] == [(SL, ST), (SL, None), (SL, None)], order
    # without sres_layer.install a forward-only call also takes the op, unless it updates the magnitude EMA
    for order in (('torgb', 'cond'), ('cond', 'torgb')):
        assert res['routes'][order] == [(SC, ST), (SC, ST), (None, None)], order
    # without sres_torgb.install nothing changes: sres_layer's step and no ToRGB forward
    assert res['routes'][('layer', 'cond')] == [(SL, None)] * 3
    assert res['cpu_bitwise'] and res['pickled']
    assert res['reasons'] == {'cpu': 'cpu', 'fp64': 'dtype', 'requires_grad': 'grad', 'layer': 'layer',
                              'torgb_shape': ('shape', 'cpu')}
    assert res['fallback_calls'] == 1
