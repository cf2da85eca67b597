"""custom_ops._launch, the one path every plugin launch takes, on the CPU: the stream goes last, an error code raises with the
op's name, and LVG_UNSUPPORTED raises unless the caller asked for it as an answer (the device guard, the stream and the
library are stand-ins)."""
import contextlib

import pytest
import torch

from torch_utils import custom_ops


class _StubLib:
    @staticmethod
    def lvg_last_error():
        return b'stub error'


@pytest.fixture
def launch(monkeypatch):
    monkeypatch.setattr(custom_ops, '_lib', _StubLib())
    monkeypatch.setattr(custom_ops, '_stream', lambda t: 1234)
    monkeypatch.setattr(custom_ops, '_DeviceGuard', lambda t: contextlib.nullcontext())
    return custom_ops._launch


def test_launch_return_codes(launch):
    anchor = torch.zeros(1)
    calls = []

    def fn(rc):
        def call(*args):
            calls.append(args)
            return rc
        return call

    assert launch('op', fn(0), anchor, 7, None) is True
    assert calls == [(7, None, 1234)]
    for rc in (1, custom_ops.LVG_UNSUPPORTED):
        with pytest.raises(RuntimeError, match='^op: stub error$'):
            launch('op', fn(rc), anchor, 7)
    with pytest.raises(RuntimeError, match='^op: stub error$'):
        launch('op', fn(1), anchor, 7, optional=True)
    assert launch('op', fn(custom_ops.LVG_UNSUPPORTED), anchor, 7, optional=True) is False
    assert len(calls) == 5
