"""Host-side checks of torch_utils/ops/sres_dblock.py: the layer plan against conv2d_resample in float64, which blocks the
installed forward takes, install() on the unmodified reference discriminator (tests/sres_dblock_run.py, CPU mode), and
the autograd Functions' gradients of every order over a torch stand-in of the kernels."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from torch_utils.ops import conv2d_resample, conv_nd, sres_dblock as sd, upfirdn2d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')


def f4():
    return upfirdn2d.setup_filter([1, 3, 3, 1])


@pytest.mark.parametrize('h,w', [(8, 8), (9, 12), (256, 256), (5, 7)])
def test_plan_matches_conv2d_resample(h, w):
    """conv1 = FIR with padding 2, then a stride-2 3x3 convolution; the skip = FIR decimating by 2 with padding 1, then the
    1x1 convolution: conv2d_resample's own plan, and in float64 the same values as conv2d_resample, at the extents
    plan_shapes gives."""
    assert conv2d_resample._plan(3, 3, 4, 4, 1, 2, 1) == [('fir', dict(padding=[2, 2, 2, 2])), ('conv', dict(stride=2))]
    assert conv2d_resample._plan(1, 1, 4, 4, 1, 2, 0) == [('fir', dict(down=2, padding=[1, 1, 1, 1])), ('conv', dict())]
    if h * w > 4096:
        return
    g = torch.Generator().manual_seed(h * w)
    x = torch.randn(2, 5, h, w, generator=g, dtype=torch.float64)
    w1 = torch.randn(6, 5, 3, 3, generator=g, dtype=torch.float64)
    ws = torch.randn(6, 5, 1, 1, generator=g, dtype=torch.float64)
    f = f4()
    shapes = sd.plan_shapes(2, 5, 6, h, w)
    hf = upfirdn2d.upfirdn2d(x, f, padding=2)
    assert tuple(hf.shape) == shapes['filtered']
    c1 = torch.nn.functional.conv2d(hf, w1, stride=2)
    want1 = conv2d_resample.conv2d_resample(x, w1, f=f, down=2, padding=1)
    assert tuple(c1.shape) == tuple(want1.shape) == shapes['conv1']
    assert torch.allclose(c1, want1, rtol=0, atol=1e-12)
    sk = torch.nn.functional.conv2d(upfirdn2d.upfirdn2d(x, f, down=2, padding=1), ws)
    wants = conv2d_resample.conv2d_resample(x, ws, f=f, down=2)
    assert tuple(sk.shape) == tuple(wants.shape) == shapes['skip']
    assert torch.allclose(sk, wants, rtol=0, atol=1e-12)


# ---------------------------------------------------------------------------------------------------- routing

class _Layer(torch.nn.Module):
    def __init__(self, k, down=1):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.zeros(4, 4, k, k))
        self.up, self.down, self.dropout_p = 1, down, 0.0
        self.register_buffer('resample_filter', f4())


def _block(**kw):
    b = types.SimpleNamespace(architecture='resnet', negate_half=False, channels_last=False, in_channels=4,
                              conv0=_Layer(3), conv1=_Layer(3, 2), skip=_Layer(1, 2))
    for k, v in kw.items():
        setattr(b, k, v)
    return b


def test_block_applies_rejects_each_case_on_its_own():
    assert sd.block_applies(_block())
    assert not sd.block_applies(_block(architecture='resnet2'))
    assert not sd.block_applies(_block(architecture='orig'))
    assert not sd.block_applies(_block(negate_half=True))
    assert not sd.block_applies(_block(channels_last=True))
    assert sd.block_applies(_block(channels_last=True), force_fp32=True)
    b = _block()
    b.conv0.dropout_p = 0.1
    assert not sd.block_applies(b)
    b = _block()
    b.conv1.up = 2
    assert not sd.block_applies(b)
    b = _block()
    b.skip.resample_filter = upfirdn2d.setup_filter([1, 2, 1])
    assert not sd.block_applies(b)
    b = _block()
    b.conv1.resample_filter = upfirdn2d.setup_filter([1, 3, 3, 1], separable=True)
    assert not sd.block_applies(b)


def test_applies_rejects_cpu_fp64_and_the_switch(monkeypatch):
    b = _block()
    x = torch.zeros(1, 4, 8, 8)
    assert not sd.applies(b, x, None)                                       # CPU
    assert not sd.applies(b, None, x.double())
    assert not sd.native(x, b.skip.weight, b.conv0.weight, b.conv1.weight, f4(), f4(), 'lrelu')
    # the switch applies() and native() consult
    fake = types.SimpleNamespace(device=types.SimpleNamespace(type='cuda'))
    monkeypatch.setenv('LVG_NATIVE_CONV', '0')
    assert not conv_nd.enabled_for(fake)
    monkeypatch.setenv('LVG_NATIVE_CONV', '1')
    assert conv_nd.enabled_for(fake)


def test_install_on_the_reference_discriminator(tmp_path):
    """install() is idempotent, keeps the originals, reaches the classes of a pickled network and leaves the CPU forward,
    gradients and R1 pattern bitwise unchanged."""
    if not os.path.isdir(SRC):
        pytest.skip('oracle/_ref not staged')
    out = str(tmp_path / 'cpu.pt')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'sres_dblock_run.py'), out, 'cpu'], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:]
    res = torch.load(out)
    assert res['cpu_equal'] and res['pickled_patched'] and res['pickled'] == ['DiscriminatorBlock', 'Conv2dLayer']


# ---------------------------------------------------------------------------------------------------- gradients

class _TorchStandIn:
    """The kernels of sd._Native restated with differentiable torch ops (float64 on the CPU)."""

    @staticmethod
    def _act(y, act, alpha, gain, clamp):
        y = torch.where(y < 0, y * alpha, y) * gain if act == 'lrelu' else y * gain
        return y.clamp(-clamp, clamp) if clamp is not None else y

    @staticmethod
    def conv0(x, w, b, act, alpha, gain, clamp):
        return _TorchStandIn._act(torch.nn.functional.conv2d(x, w, padding=1) + b.view(1, -1, 1, 1), act, alpha, gain, clamp)

    @staticmethod
    def conv1(x, fx, fy, flip, w, b, act, alpha, gain, clamp):
        hf = upfirdn2d.upfirdn2d(x, torch.outer(fy, fx).float(), padding=2, flip_filter=flip)
        return _TorchStandIn._act(torch.nn.functional.conv2d(hf, w, stride=2) + b.view(1, -1, 1, 1), act, alpha, gain, clamp)

    @staticmethod
    def skip(x, w, r, rscale):
        return (torch.nn.functional.conv2d(x, w) + r) * rscale

    @staticmethod
    def act_grad(dy, y, cfg):
        act, alpha, gain, clamp = cfg
        slope = torch.where(y < 0, alpha * gain, gain) if act == 'lrelu' else torch.full_like(y, gain)
        if clamp is not None:
            slope = torch.where(y.abs() < clamp, slope, torch.zeros_like(slope))
        return dy * slope.detach()

    @staticmethod
    def conv_grads(x, dz, w, stride, pad, want_dx, want_dw):
        dx = dw = None
        if want_dx:
            k = w.shape[2]
            op = [x.shape[d] + 2 * pad - ((dz.shape[d] - 1) * stride + k) for d in (2, 3)]
            dx = torch.nn.functional.conv_transpose2d(dz, w, stride=stride, padding=pad, output_padding=op)
        if want_dw:
            dw = torch.nn.grad.conv2d_weight(x, w.shape, dz, stride=stride, padding=pad)
        return dx, dw

    @staticmethod
    def conv1_backward(h0, fx, fy, flip, dz, w, want_dx, want_dw):
        hf = upfirdn2d.upfirdn2d(h0, torch.outer(fy, fx).float(), padding=2, flip_filter=flip)
        return _TorchStandIn.conv_grads(hf, dz, w, 2, 0, want_dx, want_dw)

    @staticmethod
    def fir_adjoint_act(dhf, h0, fx, fy, flip, act, alpha, gain, clamp, want_db):
        dh0 = upfirdn2d.upfirdn2d(dhf, torch.outer(fy, fx).float(), padding=1, flip_filter=not flip)
        dz = _TorchStandIn.act_grad(dh0, h0, (act, alpha, gain, clamp))
        return dz, (dz.sum([0, 2, 3]) if want_db else None)


@pytest.fixture
def stand_in(monkeypatch):
    monkeypatch.setattr(sd, '_backend', _TorchStandIn)


@pytest.mark.parametrize('clamp', [None, 0.6])
def test_block_function_gradients(stand_in, clamp):
    """_Block over the stand-in equals the composition and passes gradcheck (the native first-order backward: rscale
    folded into conv1's gain and the skip's weights, the fused FIR adjoint) and gradgradcheck (the recorded backward)."""
    g = torch.Generator().manual_seed(0)
    f = f4()
    fx, fy = (torch.tensor([1., 3., 3., 1.]) / 8,) * 2
    t = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64, requires_grad=True)     # noqa: E731
    x, ws, w0, b0, w1, b1 = t(2, 3, 6, 7), t(4, 3, 1, 1), t(3, 3, 3, 3), t(3), t(4, 3, 3, 3), t(4)
    cfg = (False, 'lrelu', 0.2, float(np.sqrt(2)), clamp, sd._SQRT_HALF)

    def fn(x, ws, w0, b0, w1, b1):
        xd = upfirdn2d.upfirdn2d(x, f, down=2, padding=1)
        return sd._Block.apply(x, xd, ws, w0, b0, w1, b1, f, fx, fy, cfg)
    ref = sd._composition(x, ws, w0, b0, w1, b1, f, f, 'lrelu', float(np.sqrt(2)), clamp)
    assert torch.allclose(fn(x, ws, w0, b0, w1, b1), ref)
    assert torch.autograd.gradcheck(fn, (x, ws, w0, b0, w1, b1))
    assert torch.autograd.gradgradcheck(fn, (x, ws, w0, b0, w1, b1))


def test_faster_rule():
    assert [sd.faster(r) for r in (256, 128, 64, 32, 16, 8)] == [False, False, False, False, True, True]
