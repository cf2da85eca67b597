"""The C-ABI library loads without a GPU and exports exactly what include/lvg_ops.h declares."""
import ctypes
import os
import re

import pytest

from torch_utils import custom_ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, 'include', 'lvg_ops.h')).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(lvg_[a-z0-9_]+)\s*\(', text)))


def test_library_exports_every_declared_symbol():
    path = custom_ops.library_path()
    assert os.path.isfile(path), f'{path} missing: run __graft_entry__.build()'
    lib = ctypes.CDLL(path)
    decl = declared_symbols()
    assert len(decl) >= 12
    for name in decl:
        assert hasattr(lib, name), f'{name} declared in lvg_ops.h but not exported'
    assert sorted(custom_ops.exported_symbols()) == decl, 'python binding table and header disagree'


def test_abi_version_and_error_string():
    lib = custom_ops.load_library()
    assert lib.lvg_abi_version() == 2
    assert b'sm_90a' in lib.lvg_build_info()
    assert isinstance(lib.lvg_last_error(), bytes)


def test_argument_errors_are_reported_without_a_gpu():
    lib = custom_ops.load_library()
    # NULL x: rejected before any CUDA call
    rc = lib.lvg_bias_act(None, None, None, None, None, None, 0, 16, 1, 1, 0, 3, 0.2, 1.0, -1.0, None)
    assert rc == 1 and b'NULL' in lib.lvg_last_error()
    rc = lib.lvg_bias_act(None, None, None, None, None, None, 7, 16, 1, 1, 0, 3, 0.2, 1.0, -1.0, None)
    assert rc == 1


def test_host_size_queries_answer_without_a_gpu():
    lib = custom_ops.load_library()
    # size of the opaque relu / lrelu code buffer: one 4-byte (fp32) or 8-byte (fp16) word per thread and 1024-pack tile
    assert lib.lvg_bias_act_codes_bytes(0, 4 * 1024 * 7) == 7 * 256 * 4
    assert lib.lvg_bias_act_codes_bytes(0, 4 * 1024 * 7 + 4) == 8 * 256 * 4
    assert lib.lvg_bias_act_codes_bytes(1, 8 * 1024 * 3) == 3 * 256 * 8
    assert lib.lvg_bias_act_codes_bytes(2, 100) == -1                      # fp64 has no code path
    for n in (4, 1000, 1 << 20, (1 << 31) + 4096):
        assert lib.lvg_bias_act_codes_bytes(0, n) * 4 >= n                 # at least 2 bits per element
    # envelope of the tensor-core convolution: fp16 (dtype code 1) and fp32 (code 0), not fp64 (code 2), kh * kw <= 9
    # (dtype, n, groups, cin, cout, t, h, w, kt, kh, kw, pad_t, pad_h, pad_w)
    assert lib.lvg_convnd_workspace(1, 1, 4, 32, 64, 1, 20, 20, 1, 3, 3, 0, 1, 1) > 0
    assert lib.lvg_convnd_workspace(0, 1, 4, 32, 64, 1, 20, 20, 1, 3, 3, 0, 1, 1) > 0
    assert lib.lvg_convnd_workspace(1, 1, 4, 32, 64, 1, 20, 20, 1, 5, 2, 0, 1, 1) == -1
    assert lib.lvg_convnd_workspace(2, 1, 4, 32, 64, 1, 20, 20, 1, 3, 3, 0, 1, 1) == -1


def test_plugins_reject_cpu_tensors():
    import torch
    p = custom_ops.get_plugin('bias_act_plugin')
    with pytest.raises(RuntimeError, match='CUDA'):
        p.bias_act(torch.zeros(4), torch.zeros(0), torch.zeros(0), torch.zeros(0), torch.zeros(0), 0, 1, 3, 0.2, 1.0, -1.0)
    u = custom_ops.get_plugin('upfirdn2d_plugin')
    with pytest.raises(RuntimeError, match='CUDA'):
        u.upfirdn2d(torch.zeros(1, 1, 4, 4), torch.ones(1, 1), 1, 1, 1, 1, 0, 0, 0, 0, False, 1.0)
    with pytest.raises(RuntimeError):
        custom_ops.get_plugin('no_such_plugin')


def test_missing_library_fails_loudly(monkeypatch):
    monkeypatch.setattr(custom_ops, '_lib', None)
    monkeypatch.setenv('LVG_OPS_LIBRARY', '/nonexistent/liblvg_ops.so')
    with pytest.raises(RuntimeError, match='no fallback'):
        custom_ops.load_library()
