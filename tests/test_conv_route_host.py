"""The route query `lvg_convnd_route` (host arithmetic only, no device needed): which kernels a convolution call takes.

Over an enumeration of the engine's envelope (every accepted (kt, kh, kw) with strides, paddings, groups and ragged
channel counts, as tests/test_conv_envelope.py walks it) every shape gets a route in every direction; 1x1x1 calls with
stride 1, no padding, one group and no epilogue leave the engine -- for the streaming SIMT kernels when they are few-channel
fp32 layers (the flag `lvg_convnd_plan` reports in slot 47), for the pointwise wgmma kernels otherwise, given a 16-byte
pixel-row pitch -- and every other call stays on the engine. Weight gradients run on the engine."""
import ctypes
import itertools
import types

import pytest
import torch

from torch_utils import custom_ops

KERNELS = [(kt, kh, kw) for kt in (1, 3) for kh in range(1, 4) for kw in range(1, 4)] + [(1, 1, 1)]
CHANNELS = [(1, 1), (3, 17), (32, 64), (64, 128), (17, 513), (130, 65), (512, 512), (128, 3)]
SPATIAL = [(1, 1, 4), (1, 1, 6), (2, 3, 4), (1, 5, 5), (4, 8, 8), (3, 7, 9)]


@pytest.fixture(scope='module')
def lib():
    return custom_ops.load_library()


def simt_flag(lib, mode, args, stride):
    out = (ctypes.c_int * 48)()
    assert lib.lvg_convnd_plan(mode, *args, stride, out, 48) == 0, lib.lvg_last_error().decode()
    return bool(out[47])


def expected_route(mode, code, groups, cin, cout, sp, k, pad, stride, epilogue, simt):
    P = sp[0] * sp[1] * sp[2]
    pointwise = k == (1, 1, 1) and pad == (0, 0, 0) and stride == 1 and groups == 1 and (mode == 1 or not epilogue)
    if mode == 2 or not pointwise:
        return 0
    if simt:
        return 1
    return 2 if P % (4 if code == 0 else 8) == 0 else 0


def test_route_over_envelope(lib):
    n_pointwise = 0
    for code, k, (cin, cout), sp, groups, stride in itertools.product((0, 1), KERNELS, CHANNELS, SPATIAL, (1, 2), (1, 2)):
        if groups > 1 and (cin % groups or cout % groups):
            continue
        for pad in {(0, 0, 0), tuple(kk - 1 for kk in k)}:
            if any(s + 2 * p - kk + 1 < 1 for s, p, kk in zip(sp, pad, k)):
                continue
            args = [code, 2, groups, cin // groups, cout // groups] + list(sp) + list(k) + list(pad)
            for mode in (0, 1, 2):
                for epilogue in ((0, 1) if mode == 0 else (0,)):
                    r = lib.lvg_convnd_route(mode, *args, stride, epilogue)
                    simt = mode < 2 and simt_flag(lib, mode, args, stride) and not epilogue
                    exp = expected_route(mode, code, groups, cin // groups, cout // groups, sp, k, pad, stride, epilogue, simt)
                    assert r == exp, (mode, epilogue, args, stride, r, exp)
                    n_pointwise += r == 2
    assert n_pointwise > 100


def test_route_outside_envelope(lib):
    assert lib.lvg_convnd_route(3, 0, 1, 1, 8, 8, 1, 1, 8, 1, 1, 1, 0, 0, 0, 1, 0) == -1           # no such mode
    assert lib.lvg_convnd_route(0, 2, 1, 1, 8, 8, 1, 1, 8, 1, 1, 1, 0, 0, 0, 1, 0) == -1           # fp64
    assert lib.lvg_convnd_route(0, 0, 1, 1, 8, 8, 1, 8, 8, 1, 5, 2, 0, 0, 0, 1, 0) == -1           # kh * kw > 9
    assert lib.lvg_convnd_route(1, 0, 1, 1, 8, 8, 1, 8, 8, 1, 3, 3, 0, 3, 3, 1, 0) == -1           # dgrad padding > k - 1


def test_engine_takes(monkeypatch):
    """conv_nd.engine_takes, which decides where the installed Conv3dLayer / Conv2dLayer forwards move bias_act into the
    epilogue: engine-routed calls only, never a 1x1 layer of the pointwise kernels, fp64 or the switch turned off."""
    from torch_utils.ops import conv_nd

    def x(*shape, dtype=torch.float16):
        return types.SimpleNamespace(device=types.SimpleNamespace(type='cuda'), shape=shape, dtype=dtype)
    assert conv_nd.engine_takes(x(2, 16, 4, 8, 8), (32, 16, 3, 3, 3), (1, 1, 1))
    assert conv_nd.engine_takes(x(2, 16, 8, 8, dtype=torch.float32), (32, 16, 3, 3), (1, 1))
    assert not conv_nd.engine_takes(x(2, 16, 4, 8, 8), (32, 16, 1, 1, 1), (0, 0, 0))            # pointwise kernels
    assert not conv_nd.engine_takes(x(2, 16, 4, 8, 8, dtype=torch.float64), (32, 16, 3, 3, 3), (1, 1, 1))
    assert not conv_nd.engine_takes(x(2, 16, 4, 8, 8), (32, 16, 3, 3, 3), (3, 1, 1))             # padding > k - 1
    assert not conv_nd.engine_takes(types.SimpleNamespace(device=torch.device('cpu'), shape=(2, 16, 8, 8),
                                                          dtype=torch.float16), (32, 16, 3, 3), (1, 1))
    monkeypatch.setenv('LVG_NATIVE_CONV', '0')
    assert not conv_nd.engine_takes(x(2, 16, 4, 8, 8), (32, 16, 3, 3, 3), (1, 1, 1))
