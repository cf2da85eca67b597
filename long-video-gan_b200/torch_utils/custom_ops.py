"""Plugin loader for the sm_90a operator library (replaces the JIT loader).

The reference builds three pybind11 modules at first use
(``torch_utils/custom_ops.py:59-157`` -> ``torch.utils.cpp_extension.load``).
Here there is ONE ahead-of-time built C-ABI shared library, ``liblvg_ops.so``
(``include/lvg_ops.h``), opened with ``ctypes``; ``get_plugin(name)`` returns an
object exposing the same functions, argument order and return values as the
reference's pybind module of that name:

    bias_act_plugin.bias_act            bias_act.cpp:32,96
    upfirdn2d_plugin.upfirdn2d          upfirdn2d.cpp:16,104
    filtered_lrelu_plugin.filtered_lrelu / filtered_lrelu_act_   filtered_lrelu.cpp:16,213,296

Tensors are allocated here with torch; the library only sees raw device
pointers, shapes, strides and the current CUDA stream. There is no CPU
implementation behind these objects: a missing library or a non-CUDA tensor
raises.
"""
import ctypes
import math
import os

import torch

from .ops._util import is_absent, is_dense

verbosity = 'brief'  # kept for API compatibility ('none' | 'brief' | 'full')

_LIB_NAME = 'liblvg_ops.so'
_lib = None
_plugins = {}

_c_void_p = ctypes.c_void_p
_c_int = ctypes.c_int
_c_i64 = ctypes.c_int64
_c_float = ctypes.c_float
_I64x4 = ctypes.c_int64 * 4
_I64x6 = ctypes.c_int64 * 6

_DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.float64: 2}

# every exported symbol of include/lvg_ops.h with its C signature
_SIGNATURES = {
    'lvg_abi_version': (_c_int, []),
    'lvg_last_error': (ctypes.c_char_p, []),
    'lvg_build_info': (ctypes.c_char_p, []),
    'lvg_launch_count': (_c_i64, []),
    'lvg_grad_postprocess': (_c_int, [_c_void_p, _c_i64, _c_float, _c_float, _c_void_p]),
    'lvg_adam_step': (_c_int, [_c_void_p] * 5 + [_c_i64] + [_c_float] * 4 + [_c_i64, _c_float, _c_float, _c_int, _c_float, _c_void_p]),
    'lvg_lerp': (_c_int, [_c_void_p, _c_void_p, _c_i64, _c_float, _c_void_p]),
    'lvg_bias_act': (_c_int, [_c_void_p] * 6 + [_c_int, _c_i64, _c_i64, _c_i64, _c_int, _c_int, _c_float, _c_float, _c_float, _c_void_p]),
    'lvg_bias_act_grad_db': (_c_int, [_c_void_p] * 6 + [_c_int, _c_i64, _c_i64, _c_i64, _c_int, _c_float, _c_float, _c_float, _c_void_p]),
    'lvg_bias_act_fwd_codes': (_c_int, [_c_void_p] * 4 + [_c_int, _c_i64, _c_i64, _c_i64, _c_int, _c_float, _c_float, _c_float, _c_void_p]),
    'lvg_bias_act_codes_bytes': (_c_i64, [_c_int, _c_i64]),
    'lvg_bias_act_bwd_codes': (_c_int, [_c_void_p] * 4 + [_c_int, _c_i64, _c_i64, _c_i64, _c_int, _c_float, _c_float, _c_float, _c_void_p]),
    'lvg_upfirdn2d': (_c_int, [_c_void_p, _c_void_p, _c_void_p, _c_int, _I64x4, _I64x4, _I64x4, _I64x4, _c_int, _c_int, _c_i64, _c_i64]
                      + [_c_int] * 7 + [_c_float, _c_void_p]),
    'lvg_upfirdn2d_sep': (_c_int, [_c_void_p] * 4 + [_c_int, _I64x4, _I64x4, _I64x4, _I64x4] + [_c_int] * 9 + [_c_float, _c_void_p]),
    'lvg_filtered_lrelu': (_c_int, [_c_void_p] * 7 + [_c_int, _I64x4, _I64x4, _I64x4, _I64x4] + [_c_int] * 12
                           + [_c_float, _c_float, _c_float, _c_int, _c_int, _c_void_p]),
    'lvg_filtered_lrelu_supported': (_c_int, [_c_int] * 7),
    'lvg_filtered_lrelu_act': (_c_int, [_c_void_p] * 3 + [_c_int, _I64x4, _I64x4] + [_c_int] * 4 + [_c_float] * 3 + [_c_int, _c_void_p]),
    'lvg_fma': (_c_int, [_c_void_p] * 4 + [_c_int, _c_int, _I64x6, _I64x6, _I64x6, _I64x6, _c_void_p]),
    'lvg_fir1d_depthwise_workspace': (_c_i64, [_c_int]),
    'lvg_fir1d_depthwise': (_c_int, [_c_void_p] * 3 + [_c_int] * 4 + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_convnd_workspace': (_c_i64, [_c_int] * 14),
    'lvg_convnd_fprop': (_c_int, [_c_void_p] * 3 + [_c_int] * 15 + [_c_void_p, _c_int, _c_float, _c_float, _c_float, _c_void_p, _c_i64, _c_void_p]),
    'lvg_convnd_dgrad': (_c_int, [_c_void_p] * 3 + [_c_int] * 15 + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_convnd_wgrad_workspace': (_c_i64, [_c_int] * 14),
    'lvg_convnd_wgrad': (_c_int, [_c_void_p] * 3 + [_c_int] * 15 + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_convnd_plan': (_c_int, [_c_int] * 16 + [ctypes.POINTER(_c_int), _c_int]),
    'lvg_convnd_epilogue_plan': (_c_int, [_c_int] * 16 + [ctypes.POINTER(_c_int), _c_int]),
    'lvg_convnd_wgrad_plan': (_c_int, [_c_int] * 14 + [ctypes.POINTER(_c_int), _c_int]),
    'lvg_convnd_wgrad_ksteps': (_c_int, [_c_int] * 16 + [ctypes.POINTER(_c_int), _c_int]),
    'lvg_convnd_route': (_c_int, [_c_int] * 17),
    'lvg_convnd_backward_workspace': (_c_i64, [_c_int] * 14),
    'lvg_convnd_backward': (_c_int, [_c_void_p] * 5 + [_c_int] * 15 + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_modconv_workspace': (_c_i64, [_c_int] * 13),
    'lvg_modconv_fprop': (_c_int, [_c_void_p] * 5 + [_c_int] * 13 + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_modconv_backward': (_c_int, [_c_void_p] * 10 + [_c_int] * 13 + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_fir3d': (_c_int, [_c_void_p] * 3 + [_c_int] * 19 + [_c_void_p]),
    'lvg_fir3d_adjoint': (_c_int, [_c_void_p] * 3 + [_c_int] * 19 + [_c_void_p]),
    'lvg_video_augment_workspace': (_c_i64, [_c_int] * 6),
    'lvg_video_augment': (_c_int, [_c_void_p] * 4 + [_c_int] * 7 + [_c_void_p]),
    'lvg_video_augment_adjoint': (_c_int, [_c_void_p] * 4 + [_c_int] * 6 + [_c_void_p]),
    'lvg_augment_pipe_workspace': (_c_i64, [_c_int] * 6),
    'lvg_augment_pipe': (_c_int, [_c_void_p] * 3 + [_c_int] + [_c_void_p] * 2 + [_c_int] * 6 + [_c_void_p]),
    'lvg_augment_pipe_adjoint': (_c_int, [_c_void_p] * 3 + [_c_int] + [_c_void_p] * 2 + [_c_int] * 6 + [_c_void_p]),
    'lvg_gblock_tail_workspace': (_c_i64, [_c_int] * 9),
    'lvg_gblock_tail': (_c_int, [_c_void_p] * 5 + [_c_int] * 11 + [_c_float] * 3 + [_c_void_p]),
    'lvg_gblock_tail_adjoint': (_c_int, [_c_void_p] * 5 + [_c_i64] + [_c_int] * 11 + [_c_float] * 2 + [_c_void_p]),
    'lvg_dblock_tail_workspace': (_c_i64, [_c_int] * 6),
    'lvg_dblock_tail_codes_bytes': (_c_i64, [_c_int] * 6),
    'lvg_dblock_tail': (_c_int, [_c_void_p] * 6 + [_c_int] * 9 + [_c_float] * 3 + [_c_void_p]),
    'lvg_dblock_tail_adjoint': (_c_int, [_c_void_p] * 7 + [_c_i64] + [_c_int] * 8 + [_c_float] * 2 + [_c_void_p]),
    'lvg_sres_cond_workspace': (_c_i64, [_c_int] * 9 + [_c_void_p] * 2),
    'lvg_sres_cond': (_c_int, [_c_void_p] * 7 + [_c_i64] + [_c_int] * 10 + [_c_void_p] * 3 + [_c_float] * 2 + [_c_void_p]),
    'lvg_sres_layer_workspace': (_c_i64, [_c_int] * 9 + [_c_void_p] * 2 + [_c_int] * 5),
    'lvg_sres_layer_fprop': (_c_int, [_c_void_p] * 9 + [_c_int] * 10 + [_c_void_p] * 3 + [_c_float] * 2 + [_c_int] * 5
                             + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_sres_layer_backward': (_c_int, [_c_void_p] * 13 + [_c_int] * 10 + [_c_void_p] * 3 + [_c_float] * 2 + [_c_int] * 5
                                + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_sres_torgb_workspace': (_c_i64, [_c_int] * 9 + [_c_void_p] * 2 + [_c_int]),
    'lvg_sres_torgb_fprop': (_c_int, [_c_void_p] * 9 + [_c_int] * 10 + [_c_void_p] * 3 + [_c_float] * 2 + [_c_int, _c_float, _c_void_p]),
    'lvg_sres_torgb_backward': (_c_int, [_c_void_p] * 12 + [_c_int] * 10 + [_c_void_p] * 3 + [_c_float] * 2 + [_c_int]
                                + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_lres_torgb_workspace': (_c_i64, [_c_int] * 11),
    'lvg_lres_torgb_fprop': (_c_int, [_c_void_p] * 7 + [_c_int] * 8 + [_c_float, _c_void_p, _c_i64, _c_void_p]),
    'lvg_lres_torgb_finish': (_c_int, [_c_void_p] * 4 + [_c_int] * 5 + [_c_float, _c_void_p]),
    'lvg_lres_torgb_backward': (_c_int, [_c_void_p] * 9 + [_c_int] * 8 + [_c_float, _c_void_p, _c_i64, _c_void_p]),
    'lvg_gblock_conv0_workspace': (_c_i64, [_c_int] * 13),
    'lvg_gblock_conv0_fprop': (_c_int, [_c_void_p] * 7 + [_c_int] * 14 + [_c_float] * 3 + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_gblock_conv0_backward': (_c_int, [_c_void_p] * 12 + [_c_int] * 14 + [_c_float] * 3 + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_sres_dblock_conv1_workspace': (_c_i64, [_c_int] * 6),
    'lvg_sres_dblock_conv1': (_c_int, [_c_void_p] * 3 + [_c_int] + [_c_void_p] * 3 + [_c_int] * 7 + [_c_float] * 3 + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_sres_dblock_conv1_backward_workspace': (_c_i64, [_c_int] * 6),
    'lvg_sres_dblock_conv1_backward': (_c_int, [_c_void_p] * 3 + [_c_int] + [_c_void_p] * 4 + [_c_int] * 6 + [_c_void_p, _c_i64, _c_void_p]),
    'lvg_sres_dblock_fir_adjoint_act_workspace': (_c_i64, [_c_int] * 5),
    'lvg_sres_dblock_fir_adjoint_act': (_c_int, [_c_void_p] * 4 + [_c_int] + [_c_void_p] * 3 + [_c_i64] + [_c_int] * 6 + [_c_float] * 3 + [_c_void_p]),
    'lvg_sres_dblock_skip_workspace': (_c_i64, [_c_int] * 4 + [_c_i64]),
    'lvg_sres_dblock_skip': (_c_int, [_c_void_p] * 4 + [_c_int] * 4 + [_c_i64, _c_float, _c_void_p, _c_i64, _c_void_p]),
}

LVG_UNSUPPORTED = -1


def library_path():
    """Absolute path where liblvg_ops.so is expected (next to this package)."""
    return os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), _LIB_NAME)


def load_library():
    """Open liblvg_ops.so once and declare every entry point. Raises if it is missing."""
    global _lib
    if _lib is None:
        path = os.environ.get('LVG_OPS_LIBRARY', library_path())
        if not os.path.isfile(path):
            raise RuntimeError(
                f'{_LIB_NAME} not found at {path}: build it with `python -c "import __graft_entry__ as g; g.build()"` '
                f'or `make -C long-video-gan_b200/csrc`. There is no fallback for CUDA tensors.')
        lib = ctypes.CDLL(path)
        for name, (restype, argtypes) in _SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError here = header / library mismatch
            fn.restype = restype
            fn.argtypes = argtypes
        if lib.lvg_abi_version() != 2:
            raise RuntimeError(f'{path}: unexpected ABI version {lib.lvg_abi_version()}')
        _lib = lib
    return _lib


def exported_symbols():
    return sorted(_SIGNATURES)


def launch_count():
    """Kernels launched by liblvg_ops in this process so far."""
    return int(load_library().lvg_launch_count())


def _ptr(t):
    """Device pointer of a tensor, or NULL for None / empty ("absent" in the reference API)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


_raw_stream = getattr(torch._C, '_cuda_getCurrentRawStream', None)


def _stream(t):
    """cudaStream_t of torch's current stream on t's device (the raw-handle accessor skips building a Stream object)."""
    if _raw_stream is not None and t.device.index is not None:
        return _raw_stream(t.device.index)
    return torch.cuda.current_stream(t.device).cuda_stream


def _i4(seq):
    return _I64x4(*[int(v) for v in seq])


def _dtype_code(t, what):
    try:
        return _DTYPE_CODE[t.dtype]
    except KeyError:
        raise RuntimeError(f'{what}: unsupported dtype {t.dtype}') from None


def _same_layout(a, b):
    return a.shape == b.shape and a.stride() == b.stride()


class _DeviceGuard:
    """Makes t's device current for the duration of a launch (like OptionalCUDAGuard)."""

    def __init__(self, t):
        self.idx = t.device.index
        self.prev = None

    def __enter__(self):
        cur = torch.cuda.current_device()
        if self.idx is not None and self.idx != cur:
            self.prev = cur
            torch.cuda.set_device(self.idx)

    def __exit__(self, *exc):
        if self.prev is not None:
            torch.cuda.set_device(self.prev)


def _launch(what, fn, anchor, *args, optional=False):
    """fn(*args, stream) on anchor's device and current stream. Returns True once launched. LVG_UNSUPPORTED (no kernel for
    the configuration) returns False when ``optional``, so the caller can compose other ops; it raises otherwise, as every
    error code does."""
    with _DeviceGuard(anchor):
        rc = fn(*args, _stream(anchor))
    if rc == LVG_UNSUPPORTED and optional:
        return False
    if rc != 0:
        raise RuntimeError(f'{what}: {_lib.lvg_last_error().decode()}')
    return True


_ws = {}


def _workspace(device, need):
    """The convolution engine's workspace on ``device``: one buffer of at least ``need`` bytes (and 4 MiB), grown on
    demand and shared by every ConvNdPlugin, SresDblockPlugin and GblockConv0Plugin call, the SresCondPlugin layer calls and the
    LresTorgbPlugin calls that need one."""
    if need < 0:
        raise RuntimeError('convnd: configuration outside the tensor-core kernel envelope')
    buf = _ws.get(device)
    if buf is None or buf.numel() < need:
        buf = torch.empty(max(int(need), 1 << 22), dtype=torch.uint8, device=device)
        _ws[device] = buf      # stream-ordered reuse: every call re-tiles its operands before it reads them
    return buf


# ----------------------------------------------------------------------------

class BiasActPlugin:
    """``bias_act_plugin`` (bias_act.cpp:32-96)."""

    def __init__(self, lib):
        self._lib = lib

    def bias_act(self, x, b, xref, yref, dy, grad, dim, act, alpha, gain, clamp):
        if not x.is_cuda:
            raise RuntimeError('x must reside on CUDA device')
        code = _dtype_code(x, 'bias_act')
        for name, t in (('xref', xref), ('yref', yref), ('dy', dy)):
            if not is_absent(t) and not (t.dtype == x.dtype and t.device == x.device and _same_layout(t, x)):
                raise RuntimeError(f'{name} must have the same shape, dtype, device and layout as x')
        if grad < 0:
            raise RuntimeError('grad must be non-negative')
        size_b, step_b = 1, 1
        if not is_absent(b):
            if b.dtype != x.dtype or b.device != x.device:
                raise RuntimeError('b must have the same dtype and device as x')
            if b.ndim != 1:
                raise RuntimeError('b must have rank 1')
            if not (0 <= dim < x.ndim):
                raise RuntimeError('dim is out of bounds')
            if b.numel() != x.shape[dim]:
                raise RuntimeError('b has wrong number of elements')
            if not b.is_contiguous():
                raise RuntimeError('b must be contiguous')
            size_b, step_b = b.numel(), x.stride(dim)
        if not is_dense(x):
            raise RuntimeError('x must be non-overlapping and dense')
        y = torch.empty_like(x)
        if not _same_layout(y, x):
            raise RuntimeError('y must have the same layout as x')
        _launch('bias_act', self._lib.lvg_bias_act, x, _ptr(x), _ptr(b), _ptr(xref), _ptr(yref), _ptr(dy), _ptr(y), code,
                x.numel(), size_b, max(step_b, 1), int(grad), int(act), float(alpha), float(gain), float(clamp))
        return y

    def bias_act_grad_db(self, dy, b, xref, yref, dim, act, alpha, gain, clamp):
        """Backward pass with the bias-gradient reduction fused in. Returns (dx, db) with db in dy.dtype,
        or None when the fused kernel does not cover the layout (bias along the contiguous dimension)."""
        if not dy.is_cuda:
            raise RuntimeError('dy must reside on CUDA device')
        code = _dtype_code(dy, 'bias_act_grad_db')
        if not is_dense(dy):
            raise RuntimeError('dy must be non-overlapping and dense')
        for name, t in (('xref', xref), ('yref', yref)):
            if not is_absent(t) and not (t.dtype == dy.dtype and _same_layout(t, dy)):
                raise RuntimeError(f'{name} must have the same shape, dtype and layout as dy')
        size_b, step_b = dy.shape[dim], max(dy.stride(dim), 1)
        dx = torch.empty_like(dy)
        db = torch.zeros([size_b], dtype=torch.float32, device=dy.device)
        if not _launch('bias_act_grad_db', self._lib.lvg_bias_act_grad_db, dy, _ptr(dy), _ptr(b), _ptr(xref), _ptr(yref), _ptr(dx),
                       _ptr(db), code, dy.numel(), size_b, step_b, int(act), float(alpha), float(gain), float(clamp), optional=True):
            return None     # layout not covered by the fused kernel: caller runs bias_act(grad=1) + sum
        return dx, db.to(dy.dtype)


    def bias_act_fwd_codes(self, x, b, dim, act, alpha, gain, clamp):
        """relu / lrelu forward that also emits 2-bit sign / clamp codes (uint8 [numel / 4]) for the backward pass.
        Returns (y, codes), or None when the kernel does not cover the call (other activations, odd sizes, fp64)."""
        if not x.is_cuda or x.dtype not in (torch.float16, torch.float32) or x.numel() == 0 or not is_dense(x):
            return None
        size_b, step_b = 1, 1
        if not is_absent(b):
            if b.dtype != x.dtype or b.device != x.device or b.ndim != 1 or b.numel() != x.shape[dim] or not b.is_contiguous():
                return None         # let the general entry point produce the reference's error message
            size_b, step_b = b.numel(), max(x.stride(dim), 1)
        y = torch.empty_like(x)
        nbytes = self._lib.lvg_bias_act_codes_bytes(_dtype_code(x, 'bias_act'), x.numel())
        if nbytes < 0:
            return None
        codes = torch.empty([int(nbytes)], dtype=torch.uint8, device=x.device)
        if not _launch('bias_act_fwd_codes', self._lib.lvg_bias_act_fwd_codes, x, _ptr(x), _ptr(b), _ptr(y), _ptr(codes),
                       _dtype_code(x, 'bias_act'), x.numel(), size_b, step_b, int(act), float(alpha), float(gain), float(clamp),
                       optional=True):
            return None
        return y, codes

    def bias_act_bwd_codes(self, dy, codes, dim, act, alpha, gain, clamp, want_db):
        """dx (and the bias gradient when want_db and the layout allows fusing it) from dy and the forward's codes.
        dy must have the memory layout of the forward's x. Returns (dx, db or None)."""
        code = _dtype_code(dy, 'bias_act_bwd_codes')
        dx = torch.empty_like(dy)
        size_b, step_b = dy.shape[dim], max(dy.stride(dim), 1)
        pack = 8 if dy.dtype == torch.float16 else 4
        db = torch.zeros([size_b], dtype=torch.float32, device=dy.device) if (want_db and step_b % pack == 0) else None
        _launch('bias_act_bwd_codes', self._lib.lvg_bias_act_bwd_codes, dy, _ptr(dy), _ptr(codes), _ptr(dx), _ptr(db), code,
                dy.numel(), size_b, step_b, int(act), float(alpha), float(gain), float(clamp))
        return dx, (db.to(dy.dtype) if db is not None else None)


class Upfirdn2dPlugin:
    """``upfirdn2d_plugin`` (upfirdn2d.cpp:16-104), plus the single-launch separable entry point."""

    def __init__(self, lib):
        self._lib = lib

    @staticmethod
    def _out_size(x, fw, fh, upx, upy, downx, downy, padx0, padx1, pady0, pady1):
        ow = (x.shape[3] * upx + padx0 + padx1 - fw + downx) // downx
        oh = (x.shape[2] * upy + pady0 + pady1 - fh + downy) // downy
        if ow < 1 or oh < 1:
            raise RuntimeError('output must be at least 1x1')
        return oh, ow

    @staticmethod
    def _alloc_like(x, oh, ow):
        fmt = torch.channels_last if (x.shape[1] > 1 and x.stride(1) == 1) else torch.contiguous_format
        return torch.empty([x.shape[0], x.shape[1], oh, ow], dtype=x.dtype, device=x.device, memory_format=fmt)

    @staticmethod
    def _validate(x, f):
        if not x.is_cuda:
            raise RuntimeError('x must reside on CUDA device')
        if f.device != x.device:
            raise RuntimeError('f must reside on the same device as x')
        if f.dtype != torch.float32:
            raise RuntimeError('f must be float32')
        if x.numel() == 0:
            raise RuntimeError('x has zero size')
        if f.numel() == 0:
            raise RuntimeError('f has zero size')
        if x.ndim != 4:
            raise RuntimeError('x must be rank 4')

    def upfirdn2d(self, x, f, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip, gain):
        self._validate(x, f)
        if f.ndim != 2:
            raise RuntimeError('f must be rank 2')
        if upx < 1 or upy < 1:
            raise RuntimeError('upsampling factor must be at least 1')
        if downx < 1 or downy < 1:
            raise RuntimeError('downsampling factor must be at least 1')
        code = _dtype_code(x, 'upfirdn2d')
        fh, fw = f.shape
        oh, ow = self._out_size(x, fw, fh, upx, upy, downx, downy, padx0, padx1, pady0, pady1)
        y = self._alloc_like(x, oh, ow)
        _launch('upfirdn2d', self._lib.lvg_upfirdn2d, x, _ptr(x), _ptr(f), _ptr(y), code, _i4(x.shape), _i4(x.stride()), _i4(y.shape),
                _i4(y.stride()), fw, fh, f.stride(1), f.stride(0), upx, upy, downx, downy, padx0, pady0, int(bool(flip)), float(gain))
        return y

    def upfirdn2d_sep(self, x, fx, fy, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip, gain):
        """Both passes of a separable filter in one launch (fx along W, fy along H; None = no filter
        on that axis). Returns None when the tiled kernel does not cover the configuration."""
        f_any = fx if fx is not None else fy
        self._validate(x, f_any)
        for f in (fx, fy):
            if f is not None and (f.ndim != 1 or not f.is_contiguous() or f.dtype != torch.float32):
                raise RuntimeError('separable filters must be contiguous float32 vectors')
        code = _dtype_code(x, 'upfirdn2d_sep')
        fw = fx.numel() if fx is not None else 1
        fh = fy.numel() if fy is not None else 1
        oh, ow = self._out_size(x, fw, fh, upx, upy, downx, downy, padx0, padx1, pady0, pady1)
        y = self._alloc_like(x, oh, ow)
        if not _launch('upfirdn2d_sep', self._lib.lvg_upfirdn2d_sep, x, _ptr(x), _ptr(fx), _ptr(fy), _ptr(y), code, _i4(x.shape),
                       _i4(x.stride()), _i4(y.shape), _i4(y.stride()), fw, fh, upx, upy, downx, downy, padx0, pady0, int(bool(flip)),
                       float(gain), optional=True):
            return None
        return y


class FilteredLReluPlugin:
    """``filtered_lrelu_plugin`` (filtered_lrelu.cpp:16-297)."""

    def __init__(self, lib):
        self._lib = lib

    def filtered_lrelu(self, x, fu, fd, b, si, up, down, px0, px1, py0, py1, sx, sy, gain, slope, clamp, flip_filters, writeSigns):
        if not x.is_cuda:
            raise RuntimeError('x must reside on CUDA device')
        if not (fu.device == x.device and fd.device == x.device and b.device == x.device):
            raise RuntimeError('all input tensors must reside on the same device')
        if fu.dtype != torch.float32 or fd.dtype != torch.float32:
            raise RuntimeError('fu and fd must be float32')
        if b.dtype != x.dtype:
            raise RuntimeError('x and b must have the same dtype')
        if x.dtype not in (torch.float16, torch.float32):
            raise RuntimeError('x and b must be float16 or float32')
        if x.ndim != 4:
            raise RuntimeError('x must be rank 4')
        if x.numel() == 0:
            raise RuntimeError('x is empty')
        if fu.ndim not in (1, 2) or fd.ndim not in (1, 2):
            raise RuntimeError('fu and fd must be rank 1 or 2')
        if fu.numel() == 0 or fd.numel() == 0:
            raise RuntimeError('fu and fd must not be empty')
        if b.ndim != 1 or b.shape[0] != x.shape[1]:
            raise RuntimeError('b must be a vector with the same number of channels as x')
        if up < 1 or down < 1:
            raise RuntimeError('up and down must be at least 1')
        code = _dtype_code(x, 'filtered_lrelu')

        fu_w, fu_h = fu.shape[-1], (fu.shape[0] if fu.ndim == 2 else 0)   # height 0 marks a separable filter
        fd_w, fd_h = fd.shape[-1], (fd.shape[0] if fd.ndim == 2 else 0)
        if self._lib.lvg_filtered_lrelu_supported(code, fu_w, fu_h, fd_w, fd_h, up, down) != 0:
            return None, None, -1   # same contract as the reference: caller runs the generic path

        fut_w, fut_h = fu.shape[-1] - 1, fu.shape[0] - 1
        fdt_w, fdt_h = fd.shape[-1] - 1, fd.shape[0] - 1
        cw = x.shape[3] * up + (px0 + px1) - fut_w      # logical size of the up-sampled buffer
        ch = x.shape[2] * up + (py0 + py1) - fut_h
        if not (cw > fdt_w and ch > fdt_h):
            raise RuntimeError('upsampled buffer must be at least the size of downsampling filter')
        yw = (cw - fdt_w + (down - 1)) // down
        yh = (ch - fdt_h + (down - 1)) // down
        if yw < 1 or yh < 1:
            raise RuntimeError('output must be at least 1x1')
        fmt = torch.channels_last if (x.shape[1] > 1 and x.stride(1) == 1) else torch.contiguous_format
        y = torch.empty([x.shape[0], x.shape[1], yh, yw], dtype=x.dtype, device=x.device, memory_format=fmt)

        so = None
        s = si if not is_absent(si) else None
        read_signs = s is not None
        if writeSigns:
            if read_signs:
                raise RuntimeError('cannot read and write signs in the same call')
            sw_active = yw * down - (down - 1) + fdt_w
            sh = yh * down - (down - 1) + fdt_h
            sw = (sw_active + 15) & ~15
            s = so = torch.empty([x.shape[0], x.shape[1], sh, sw >> 2], dtype=torch.uint8, device=x.device)
        if s is not None:
            if not (s.is_contiguous() and s.dtype == torch.uint8 and s.device == x.device and s.ndim == 4
                    and s.shape[0] == x.shape[0] and s.shape[1] == x.shape[1]):
                raise RuntimeError('signs must be a contiguous uint8 [N, C, H, W/4] tensor on the same device as x')
        if read_signs and up * down > 1 and (s.shape[3] % 4 or s.data_ptr() % 4):
            # the resampling kernel reads sign rows as aligned 32-bit words: copy into zero-filled rows of a multiple of
            # 4 bytes. A zero byte is code 0 ("unchanged"), as for samples outside the tensor, so the operator is the same.
            padded = torch.zeros([*s.shape[:3], (s.shape[3] + 3) & ~3], dtype=torch.uint8, device=x.device)
            padded[..., :s.shape[3]] = s
            s = padded
        s_h, s_wb = (s.shape[2], s.shape[3]) if s is not None else (0, 0)
        fu_c, fd_c, b_c = fu.contiguous(), fd.contiguous(), b.contiguous()
        if not _launch('filtered_lrelu', self._lib.lvg_filtered_lrelu, x,
                       _ptr(x), _ptr(fu_c), _ptr(fd_c), _ptr(b_c), _ptr(s) if read_signs else None, _ptr(y),
                       _ptr(so) if writeSigns else None, code, _i4(x.shape), _i4(x.stride()), _i4(y.shape), _i4(y.stride()),
                       fu_w, fu_h, fd_w, fd_h, up, down, px0, py0, s_h, s_wb, sx, sy, float(gain), float(slope),
                       float(clamp), int(bool(flip_filters)), int(bool(writeSigns)), optional=True):
            return None, None, -1
        return y, so, 0

    def filtered_lrelu_act_(self, x, si, sx, sy, gain, slope, clamp, writeSigns):
        if not x.is_cuda:
            raise RuntimeError('x must reside on CUDA device')
        if x.ndim != 4:
            raise RuntimeError('x must be rank 4')
        if x.numel() == 0:
            raise RuntimeError('x is empty')
        code = _dtype_code(x, 'filtered_lrelu_act_')
        so = None
        s = si if not is_absent(si) else None
        read_signs = s is not None
        if writeSigns:
            sw = (x.shape[3] + 15) & ~15
            s = so = torch.empty([x.shape[0], x.shape[1], x.shape[2], sw >> 2], dtype=torch.uint8, device=x.device)
        if s is not None:
            if not (s.is_contiguous() and s.dtype == torch.uint8 and s.device == x.device and s.ndim == 4
                    and s.shape[0] == x.shape[0] and s.shape[1] == x.shape[1]):
                raise RuntimeError('signs must be a contiguous uint8 [N, C, H, W/4] tensor on the same device as x')
        s_h, s_wb = (s.shape[2], s.shape[3]) if s is not None else (0, 0)
        _launch('filtered_lrelu_act_', self._lib.lvg_filtered_lrelu_act, x, _ptr(x), _ptr(s) if (read_signs and not writeSigns) else None,
                _ptr(so) if writeSigns else None, code, _i4(x.shape), _i4(x.stride()), s_h, s_wb, sx, sy, float(gain), float(slope),
                float(clamp), int(bool(writeSigns)))
        return so


class FmaPlugin:
    """Elementwise a * b + c with broadcasting (no reference plugin: fma.py uses torch.addcmul)."""

    def __init__(self, lib):
        self._lib = lib

    def fma(self, a, b, c):
        if not (a.is_cuda and b.device == a.device and c.device == a.device):
            raise RuntimeError('fma operands must reside on one CUDA device')
        dtype = torch.promote_types(torch.promote_types(a.dtype, b.dtype), c.dtype)
        a, b, c = a.to(dtype), b.to(dtype), c.to(dtype)
        code = _dtype_code(a, 'fma')
        shape = torch.broadcast_shapes(a.shape, b.shape, c.shape)
        if len(shape) > 6:
            raise RuntimeError('fma supports at most 6 dimensions')
        out = torch.empty(shape, dtype=dtype, device=a.device)
        if out.numel() == 0:
            return out
        ae, be, ce = a.expand(shape), b.expand(shape), c.expand(shape)
        pad = [0] * (6 - len(shape))
        _launch('fma', self._lib.lvg_fma, out, _ptr(ae), _ptr(be), _ptr(ce), _ptr(out), code, len(shape),
                _I64x6(*(list(shape) + [1] * len(pad))), _I64x6(*(list(ae.stride()) + pad)),
                _I64x6(*(list(be.stride()) + pad)), _I64x6(*(list(ce.stride()) + pad)))
        return out


class ConvNdPlugin:
    """TMA-fed wgmma implicit-GEMM convolution for 1-D / 2-D / 3-D NC(T)HW tensors, fp16 or fp32 (bf16 hi/lo split),
    stride 1: forward (optionally with the bias_act epilogue fused), input gradient, weight gradient. No reference
    plugin: the reference hands these to cuDNN (conv2d_gradfix.py:37-45, generator_lres.py:119, discriminator_lres.py:121,172)."""

    def __init__(self, lib):
        self._lib = lib

    @staticmethod
    def _pad3(padding, nd):
        p = list(padding) if isinstance(padding, (list, tuple)) else [padding] * nd
        return [0] * (3 - nd) + [int(v) for v in p]

    def supported(self, x, w, stride, padding, dilation, groups):
        return x.is_cuda and self._in_envelope(tuple(x.shape), tuple(w.shape), x.dtype if w.dtype == x.dtype else None, stride, padding,
                                               dilation, groups)

    @staticmethod
    def _in_envelope(x_shape, w_shape, dtype, stride, padding, dilation, groups):
        """The shapes the engine plans and runs in every direction (forward, input gradient, weight gradient): fp16 / fp32,
        1-D / 2-D / 3-D, kh * kw <= 9 with kw <= 3, kt <= 7, 0 <= padding <= k - 1, dilation 1, the same stride 1-4 on H and W
        (1 on T and on 1-D tensors), and a stride-1 output width the weight gradient's at most 4 column segments of
        128 - (kw - 1) pixels cover (ConvShape::wgrad_ok in csrc/conv_igemm.cu)."""
        if not (dtype in (torch.float16, torch.float32) and len(x_shape) == len(w_shape) and len(x_shape) in (3, 4, 5)):
            return False
        nd = len(x_shape) - 2
        as_t = lambda v: tuple(v) if isinstance(v, (list, tuple)) else (v,) * nd       # noqa: E731
        st = as_t(stride)
        if as_t(dilation) != (1,) * nd or len(set(st[-2:])) != 1 or not (1 <= st[-1] <= 4) or (nd == 3 and st[0] != 1) or (nd == 1 and st[0] != 1):
            return False
        sp = [1] * (3 - nd) + list(x_shape[2:])
        k = [1] * (3 - nd) + list(w_shape[2:])
        pad = ConvNdPlugin._pad3(padding, nd)
        if k[1] * k[2] > 9 or k[0] > 7 or k[2] > 3 or min(pad) < 0 or any(p > kk - 1 for p, kk in zip(pad, k)):
            return False
        if x_shape[1] != w_shape[1] * groups or w_shape[0] % groups != 0 or x_shape[0] * groups > 65535 or math.prod(x_shape) == 0:
            return False
        out = [s + 2 * p - kk + 1 for s, p, kk in zip(sp, pad, k)]
        return min(out) >= 1 and out[2] <= 4 * (128 - k[2] + 1)

    def _args(self, x_shape, w_shape, padding, groups, dtype):
        nd = len(x_shape) - 2
        sp = [1] * (3 - nd) + list(x_shape[2:])
        k = [1] * (3 - nd) + list(w_shape[2:])
        pad = self._pad3(padding, nd)
        code = 1 if dtype == torch.float16 else 0
        return [code, x_shape[0], groups, w_shape[1], w_shape[0] // groups] + sp + k + pad, sp, k, pad

    ROUTES = ('engine', 'simt', 'pointwise_wgmma')

    def route(self, mode, x_shape, w_shape, padding, groups, dtype, stride=1, epilogue=False):
        """Which kernels a call takes: mode 'fprop' / 'dgrad' / 'wgrad' (shapes of the forward convolution) -> one of ROUTES,
        or None outside the envelope (lvg_convnd_route)."""
        a, _, _, _ = self._args(tuple(x_shape), tuple(w_shape), padding, groups, dtype)
        r = self._lib.lvg_convnd_route(('fprop', 'dgrad', 'wgrad').index(mode), *a, int(stride), int(bool(epilogue)))
        return None if r < 0 else self.ROUTES[r]

    def fprop(self, x, w, padding, groups, bias=None, act=0, alpha=0.2, gain=1.0, clamp=-1.0, stride=1):
        x, w = x.contiguous(), w.contiguous()
        a, sp, k, pad = self._args(tuple(x.shape), tuple(w.shape), padding, groups, x.dtype)
        st3 = [1, stride, stride] if x.ndim >= 4 else [1, 1, 1]
        out_sp = [(s + 2 * p - kk) // q + 1 for s, p, kk, q in zip(sp, pad, k, st3)][3 - (x.ndim - 2):]
        y = torch.empty([x.shape[0], w.shape[0]] + out_sp, dtype=x.dtype, device=x.device)
        ws = _workspace(x.device, self._lib.lvg_convnd_workspace(*a))
        if bias is not None:
            bias = bias.to(torch.float32).contiguous()
        _launch('convnd_fprop', self._lib.lvg_convnd_fprop, x, _ptr(x), _ptr(w), _ptr(y), *a, int(stride), _ptr(bias), int(act), float(alpha),
                float(gain), float(clamp), _ptr(ws), ws.numel())
        return y

    def dgrad(self, dy, w, x_shape, padding, groups, stride=1):
        dy, w = dy.contiguous(), w.contiguous()
        a, sp, k, pad = self._args(tuple(x_shape), tuple(w.shape), padding, groups, dy.dtype)
        dx = torch.empty(list(x_shape), dtype=dy.dtype, device=dy.device)
        ws = _workspace(dy.device, self._lib.lvg_convnd_workspace(*a))
        _launch('convnd_dgrad', self._lib.lvg_convnd_dgrad, dy, _ptr(dy), _ptr(w), _ptr(dx), *a, int(stride), _ptr(ws), ws.numel())
        return dx

    def fir1d_depthwise(self, x, w):
        """y[n][g][t] = sum_k w[g][0][k] * x[n][g][t + k]: F.conv1d(x, w, groups = G) with one channel per group, fp32."""
        x, w = x.contiguous(), w.contiguous()
        n, g, lin = x.shape
        k = w.shape[2]
        y = torch.empty([n, g, lin - k + 1], dtype=x.dtype, device=x.device)
        ws = torch.empty([g + 4], dtype=torch.int32, device=x.device)
        _launch('fir1d_depthwise', self._lib.lvg_fir1d_depthwise, x, _ptr(x), _ptr(w), _ptr(y), n, g, lin, k, _ptr(ws), ws.numel() * 4)
        return y

    def wgrad(self, x, dy, w_shape, padding, groups, stride=1):
        x, dy = x.contiguous(), dy.contiguous()
        a, sp, k, pad = self._args(tuple(x.shape), tuple(w_shape), padding, groups, x.dtype)
        dw = torch.empty(list(w_shape), dtype=x.dtype, device=x.device)
        ws = _workspace(x.device, self._lib.lvg_convnd_wgrad_workspace(*a))
        _launch('convnd_wgrad', self._lib.lvg_convnd_wgrad, x, _ptr(x), _ptr(dy), _ptr(dw), *a, int(stride), _ptr(ws), ws.numel())
        return dw

    def backward(self, x, dy, w, padding, groups, stride=1):
        """(dx, dw) of y = conv(x, w) in one call: dy is re-tiled once for the input- and the weight-gradient kernels."""
        x, dy, w = x.contiguous(), dy.contiguous(), w.contiguous()
        a, sp, k, pad = self._args(tuple(x.shape), tuple(w.shape), padding, groups, x.dtype)
        dx = torch.empty_like(x)
        dw = torch.empty_like(w)
        ws = _workspace(x.device, self._lib.lvg_convnd_backward_workspace(*a))
        _launch('convnd_backward', self._lib.lvg_convnd_backward, x, _ptr(x), _ptr(dy), _ptr(w), _ptr(dx), _ptr(dw), *a, int(stride), _ptr(ws),
                ws.numel())
        return dx, dw

    def _modconv_args(self, x, w, padding):
        a, sp, k, pad = self._args(tuple(x.shape), tuple(w.shape), padding, 1, x.dtype)
        del a[2]                                            # groups = 1
        return a, sp, k, pad

    def modconv_supported(self, x, w, padding):
        """Inside the envelope of lvg_modconv_fprop / lvg_modconv_backward (given supported(x, w, 1, padding, 1, 1))."""
        return self._lib.lvg_modconv_workspace(*self._modconv_args(x, w, padding)[0]) >= 0

    @staticmethod
    def _factor(f, shape, what):
        if f.dtype != torch.float32 or tuple(f.shape) != tuple(shape):
            raise RuntimeError(f'{what}: expected a float32 tensor of shape {list(shape)}, got {f.dtype} {list(f.shape)}')
        return f.contiguous()

    def modconv_fprop(self, x, w, a, d, padding):
        """y = d * conv(a * x, w), groups = 1, stride 1: a [N, Cin, T] scales x, d [N, Cout, To] (or None) the output;
        T = To = 1 for 2-D tensors."""
        x, w = x.contiguous(), w.contiguous()
        args, sp, k, pad = self._modconv_args(x, w, padding)
        out_sp = [s + 2 * p - kk + 1 for s, p, kk in zip(sp, pad, k)]
        a = self._factor(a, (x.shape[0], x.shape[1], sp[0]), 'modconv_fprop: a')
        if d is not None:
            d = self._factor(d, (x.shape[0], w.shape[0], out_sp[0]), 'modconv_fprop: d')
        y = torch.empty([x.shape[0], w.shape[0]] + out_sp[3 - (x.ndim - 2):], dtype=x.dtype, device=x.device)
        ws = _workspace(x.device, self._lib.lvg_modconv_workspace(*args))
        _launch('modconv_fprop', self._lib.lvg_modconv_fprop, x, _ptr(x), _ptr(w), _ptr(a), _ptr(d), _ptr(y), *args, _ptr(ws), ws.numel())
        return y

    def modconv_backward(self, x, w, a, d, y, dy, padding, want_dw=True):
        """Gradients of y = d * conv(a * x, w) in one call: (dx, dw or None, da [N, Cin, T], sum_hw dy * y [N, Cout, To] or
        None when d is None)."""
        x, w, dy = x.contiguous(), w.contiguous(), dy.contiguous()
        args, sp, k, pad = self._modconv_args(x, w, padding)
        a = self._factor(a, (x.shape[0], x.shape[1], sp[0]), 'modconv_backward: a')
        dx = torch.empty_like(x)
        dw = torch.empty_like(w) if want_dw else None
        da = torch.empty(a.shape, dtype=torch.float32, device=x.device)
        dyy = None
        if d is not None:
            d = self._factor(d, (x.shape[0], w.shape[0], dy.shape[2] if dy.ndim == 5 else 1), 'modconv_backward: d')
            y = y.contiguous()
            dyy = torch.empty(d.shape, dtype=torch.float32, device=x.device)
        ws = _workspace(x.device, self._lib.lvg_modconv_workspace(*args))
        _launch('modconv_backward', self._lib.lvg_modconv_backward, x, _ptr(x), _ptr(w), _ptr(a), _ptr(d), _ptr(y) if d is not None else None,
                _ptr(dy), _ptr(dx), _ptr(dw), _ptr(da), _ptr(dyy), *args, _ptr(ws), ws.numel())
        return dx, dw, da, dyy


class Fir3dPlugin:
    """Separable 4-tap FIR over T, H, W of NCTHW tensors and its adjoint (no reference plugin: Downsample3d runs upfirdn2d
    twice, discriminator_lres.py:197-213). ``axes``: per T, H, W a tuple (filt, step, off, n_in, n_out) of the operator P
    (see lvg_fir3d in include/lvg_ops.h)."""

    def __init__(self, lib):
        self._lib = lib

    def fir3d(self, x, f, axes, fold, adjoint=False):
        """y = P x (adjoint=False, x laid out as P's input) or P^T x (x laid out as P's output)."""
        if not x.is_cuda or f.device != x.device:
            raise RuntimeError('fir3d: x and f must reside on one CUDA device')
        if f.dtype != torch.float32 or f.numel() != 4 or x.ndim != 5:
            raise RuntimeError('fir3d: needs a 5-D x and 4 float32 taps')
        code = _dtype_code(x, 'fir3d')
        x, f = x.contiguous(), f.contiguous()
        n, c = x.shape[0], x.shape[1] // (2 if (fold and adjoint) else 1)
        ins = [a[3] for a in axes]
        outs = [a[4] for a in axes]
        src, dst = (outs, ins) if adjoint else (ins, outs)
        fold_src, fold_dst = (fold and adjoint), (fold and not adjoint)
        want = [n, c * (2 if fold_src else 1), src[0] // (2 if fold_src else 1), src[1], src[2]]
        if list(x.shape) != want:
            raise RuntimeError(f'fir3d: x has shape {list(x.shape)}, expected {want}')
        y = torch.empty([n, c * (2 if fold_dst else 1), dst[0] // (2 if fold_dst else 1), dst[1], dst[2]], dtype=x.dtype, device=x.device)
        fn = self._lib.lvg_fir3d_adjoint if adjoint else self._lib.lvg_fir3d
        _launch('fir3d', fn, x, _ptr(x), _ptr(f), _ptr(y), code, n, c, *ins, *outs, *[a[0] for a in axes], *[a[1] for a in axes],
                *[a[2] for a in axes], int(bool(fold)))
        return y


class VideoAugmentPlugin:
    """The low-res discriminator's input augmentation as one affine map per sample and its adjoint (no reference plugin:
    LowResVideoGAN.run_D composes DiffAugment and F.interpolate, video_gan_lres.py:237-266). ``params``: fp32 [N, 12] on the
    device (see lvg_video_augment in include/lvg_ops.h)."""

    def __init__(self, lib):
        self._lib = lib

    def workspace(self, n, c, t_in, h, w, t_out):
        """Workspace bytes of one call, or -1 where the kernels do not take the shape (c > 4)."""
        return int(self._lib.lvg_video_augment_workspace(n, c, t_in, h, w, t_out))

    def run(self, x, params, t_other, linear=False, adjoint=False):
        """y = A x (x [N, C, T, H, W], y with t_other frames) or, adjoint=True, dx = A^T x (x with the output's frames, dx with
        t_other). linear drops the brightness offset. Returns None where the library has no kernel (LVG_UNSUPPORTED)."""
        if not (x.is_cuda and params.device == x.device and x.dtype == torch.float32 and params.dtype == torch.float32):
            raise RuntimeError('video_augment: x and params must be float32 tensors on one CUDA device')
        n, c, t, h, w = x.shape
        if tuple(params.shape) != (n, 12):
            raise RuntimeError(f'video_augment: params must have shape [{n}, 12], got {list(params.shape)}')
        t_in, t_out = (t_other, t) if adjoint else (t, t_other)
        nbytes = self.workspace(n, c, t_in, h, w, t_out)
        if nbytes < 0:
            return None
        x, params = x.contiguous(), params.contiguous()
        y = torch.empty([n, c, t_other, h, w], dtype=x.dtype, device=x.device)
        ws = torch.empty([nbytes // 4], dtype=torch.float32, device=x.device)
        if adjoint:
            ok = _launch('video_augment', self._lib.lvg_video_augment_adjoint, x, _ptr(x), _ptr(params), _ptr(y), _ptr(ws), n, c, t_in, h, w,
                         t_out, optional=True)
        else:
            ok = _launch('video_augment', self._lib.lvg_video_augment, x, _ptr(x), _ptr(params), _ptr(y), _ptr(ws), n, c, t_in, h, w, t_out,
                         int(bool(linear)), optional=True)
        return y if ok else None


class AugmentPipePlugin:
    """ADA's AugmentPipe without imgfilter and cutout as one affine map per sample and its adjoint (no reference plugin:
    AugmentPipe.forward composes F.pad, upfirdn2d, affine_grid / grid_sample and a colour bmm, ada_augment.py:180-439).
    ``params``: fp32 [N, 23] on the device, ``f``: the 12 taps of Hz_geom (see lvg_augment_pipe in include/lvg_ops.h)."""

    def __init__(self, lib):
        self._lib = lib

    def workspace(self, n, c, t, h, w, flags):
        """Workspace bytes of the adjoint, or -1 where the kernels do not take the shape (c != 3)."""
        return int(self._lib.lvg_augment_pipe_workspace(n, c, t, h, w, flags))

    def run(self, x, params, f, noise, flags, adjoint=False):
        """y = A x (+ C[:3,3] + sigma noise unless flags has LINEAR) or, adjoint=True, dx = A^T x; x [N, C, T, H, W]. Returns
        None where the library has no kernel (LVG_UNSUPPORTED)."""
        if not (x.is_cuda and params.device == x.device and f.device == x.device and x.dtype == torch.float32
                and params.dtype == torch.float32 and f.dtype == torch.float32):
            raise RuntimeError('augment_pipe: x, params and the filter must be float32 tensors on one CUDA device')
        n, c, t, h, w = x.shape
        if tuple(params.shape) != (n, 23):
            raise RuntimeError(f'augment_pipe: params must have shape [{n}, 23], got {list(params.shape)}')
        if noise is not None and (tuple(noise.shape) != tuple(x.shape) or noise.dtype != torch.float32 or noise.device != x.device):
            raise RuntimeError('augment_pipe: noise must be a float32 tensor of the shape of x on its device')
        nbytes = self.workspace(n, c, t, h, w, flags)
        if nbytes < 0 or f.numel() != 12:
            return None
        x, params, f = x.contiguous(), params.contiguous(), f.contiguous()
        noise = None if noise is None else noise.contiguous()
        y = torch.empty_like(x)
        if adjoint:
            ws = torch.empty([max(nbytes // 4, 1)], dtype=torch.float32, device=x.device)
            ok = _launch('augment_pipe', self._lib.lvg_augment_pipe_adjoint, x, _ptr(x), _ptr(params), _ptr(f), f.numel(), _ptr(y), _ptr(ws),
                         n, c, t, h, w, int(flags), optional=True)
        else:
            ok = _launch('augment_pipe', self._lib.lvg_augment_pipe, x, _ptr(x), _ptr(params), _ptr(f), f.numel(), _ptr(noise), _ptr(y),
                         n, c, t, h, w, int(flags), optional=True)
        return y if ok else None


def _check_5d(op, what, x):
    if not x.is_cuda or x.dtype not in (torch.float16, torch.float32) or x.ndim != 5:
        raise RuntimeError(f'{op}: {what} must be a 5-D float16 / float32 CUDA tensor')


class GblockTailPlugin:
    """Tail of the low-res generator's residual block, z = bias_act(crop(U_HW crop(U_T (s + h) sqrt(1/2))), b), and its
    adjoint (no reference plugin: Synthesis3dResBlock.forward composes ATen add / mul, two upfirdn2d calls, slices and
    bias_act, generator_lres.py:577-589). ``flags``: LVG_GBLOCK_TAIL_TUP | LVG_GBLOCK_TAIL_SUP (see lvg_gblock_tail in
    include/lvg_ops.h)."""

    TUP, SUP = 1, 2

    def __init__(self, lib):
        self._lib = lib

    def workspace(self, n, c, t, h, w, t_out, h_out, w_out, flags):
        """Workspace bytes of the adjoint, or -1 where the kernels do not take the shape."""
        return int(self._lib.lvg_gblock_tail_workspace(n, c, t, h, w, t_out, h_out, w_out, flags))

    def forward(self, s, h, b, out_size, flags, act, alpha, gain, clamp, want_codes):
        """(z [N, C, *out_size], codes or None) from s and h [N, C, T, H, W] (one dtype and shape) and b (fp32 [C] or None)."""
        _check_5d('gblock_tail', 's', s)
        if h.dtype != s.dtype or h.shape != s.shape or h.device != s.device:
            raise RuntimeError('gblock_tail: s and h must have one shape, dtype and device')
        n, c, t, hh, ww = s.shape
        if b is not None and (b.dtype != torch.float32 or tuple(b.shape) != (c,) or b.device != s.device):
            raise RuntimeError(f'gblock_tail: b must be a float32 [{c}] tensor on the device of s')
        to, ho, wo = (int(v) for v in out_size)
        if self.workspace(n, c, t, hh, ww, to, ho, wo, flags) < 0:
            raise RuntimeError(f'gblock_tail: no kernel for {list(s.shape)} -> {[to, ho, wo]} (flags {flags})')
        s, h = s.contiguous(), h.contiguous()
        b = None if b is None else b.contiguous()
        z = torch.empty([n, c, to, ho, wo], dtype=s.dtype, device=s.device)
        codes = None
        if want_codes:
            codes = torch.empty([int(self._lib.lvg_bias_act_codes_bytes(_dtype_code(s, 'gblock_tail'), z.numel()))], dtype=torch.uint8,
                                device=s.device)
        _launch('gblock_tail', self._lib.lvg_gblock_tail, s, _ptr(s), _ptr(h), _ptr(b), _ptr(z), _ptr(codes), _dtype_code(s, 'gblock_tail'),
                n, c, t, hh, ww, to, ho, wo, int(flags), int(act), float(alpha), float(gain), float(clamp))
        return z, codes

    def adjoint(self, dz, codes, in_size, flags, act, alpha, gain):
        """(dm [N, C, *in_size], db fp32 [C]) from dz [N, C, T_out, H_out, W_out] and the forward's codes."""
        _check_5d('gblock_tail', 'dz', dz)
        n, c, to, ho, wo = dz.shape
        t, hh, ww = (int(v) for v in in_size)
        nbytes = self.workspace(n, c, t, hh, ww, to, ho, wo, flags)
        if nbytes < 0:
            raise RuntimeError(f'gblock_tail_adjoint: no kernel for {[t, hh, ww]} -> {list(dz.shape)} (flags {flags})')
        need = int(self._lib.lvg_bias_act_codes_bytes(_dtype_code(dz, 'gblock_tail'), dz.numel()))
        if codes.dtype != torch.uint8 or codes.device != dz.device or codes.numel() < need or not codes.is_contiguous():
            raise RuntimeError(f'gblock_tail_adjoint: codes must be a contiguous uint8 buffer of {need} bytes on the device of dz')
        dz = dz.contiguous()
        dm = torch.empty([n, c, t, hh, ww], dtype=dz.dtype, device=dz.device)
        db = torch.empty([c], dtype=torch.float32, device=dz.device)
        ws = torch.empty([nbytes // 4], dtype=torch.float32, device=dz.device)
        _launch('gblock_tail_adjoint', self._lib.lvg_gblock_tail_adjoint, dz, _ptr(dz), _ptr(codes), _ptr(dm), _ptr(db), _ptr(ws), nbytes,
                _dtype_code(dz, 'gblock_tail'), n, c, t, hh, ww, to, ho, wo, int(flags), int(act), float(alpha), float(gain))
        return dm, db


class DblockTailPlugin:
    """Tail of the low-res discriminator's residual block, z = scale (bias_act(P y, b) + s) with P Downsample3d's filter, its
    read-mode linear map and its adjoint (no reference plugin: DiscriminatorBlock.forward composes two upfirdn2d calls,
    bias_act and ATen add / mul, discriminator_lres.py:321-333). ``flags``: TDOWN | SDOWN | MERGE, ``mode``: NONE / WRITE /
    READ (see lvg_dblock_tail in include/lvg_ops.h)."""

    TDOWN, SDOWN, MERGE = 1, 2, 4
    NONE, WRITE, READ = 0, 1, 2

    def __init__(self, lib):
        self._lib = lib

    def workspace(self, n, c, t, h, w, flags):
        """Workspace bytes of the adjoint for y [n, c, t, h, w], or -1 where the kernels do not take the shape."""
        return int(self._lib.lvg_dblock_tail_workspace(n, c, t, h, w, flags))

    def codes_bytes(self, n, c, t, h, w, flags):
        """Bytes of the codes of one forward call, or -1 where the kernels do not take the shape."""
        return int(self._lib.lvg_dblock_tail_codes_bytes(n, c, t, h, w, flags))

    @staticmethod
    def out_size(in_size, flags):
        t, h, w = in_size
        return (t // 2 if flags & 1 else t, h // 2 if flags & 2 else h, w // 2 if flags & 2 else w)

    def _check_codes(self, codes, ref, need):
        if codes.dtype != torch.uint8 or codes.device != ref.device or codes.numel() != need or not codes.is_contiguous():
            raise RuntimeError(f'dblock_tail: codes must be a contiguous uint8 buffer of {need} bytes on the device of the data')

    def _check_taps(self, op, f, flags, ref, name):
        if f is None and flags & (self.TDOWN | self.SDOWN) or f is not None and (f.dtype != torch.float32 or f.numel() != 4
                                                                                  or f.device != ref.device):
            raise RuntimeError(f'{op}: f must hold 4 float32 taps on the device of {name} (None where no axis is filtered)')

    def forward(self, y, s, b, f, flags, act, alpha, gain, clamp, mode, codes=None):
        """(z, codes) from y [N, C, T, H, W], s [N, C, T', H', W'] or None, b ([C], passed as fp32, or None) and the 4 fp32 taps f. WRITE
        returns new codes, READ takes ``codes``, NONE returns None for them."""
        _check_5d('dblock_tail', 'y', y)
        n, c, t, h, w = y.shape
        nbytes = self.codes_bytes(n, c, t, h, w, flags)
        if nbytes < 0:
            raise RuntimeError(f'dblock_tail: no kernel for {list(y.shape)} (flags {flags})')
        out = [n, c, *self.out_size((t, h, w), flags)]
        if s is not None and (list(s.shape) != out or s.dtype != y.dtype or s.device != y.device or not flags & self.MERGE):
            raise RuntimeError(f'dblock_tail: s must be a {y.dtype} tensor of shape {out} on the device of y, with MERGE')
        if b is not None and (tuple(b.shape) != (c,) or b.device != y.device):
            raise RuntimeError(f'dblock_tail: b must be a [{c}] tensor on the device of y')
        self._check_taps('dblock_tail', f, flags, y, 'y')
        y, f = y.contiguous(), (None if f is None else f.contiguous())
        s = None if s is None else s.contiguous()
        b = None if b is None else b.float().contiguous()
        if mode == self.WRITE:
            codes = torch.empty([nbytes], dtype=torch.uint8, device=y.device)
        elif mode == self.READ:
            self._check_codes(codes, y, nbytes)
        else:
            codes = None
        z = torch.empty(out, dtype=y.dtype, device=y.device)
        _launch('dblock_tail', self._lib.lvg_dblock_tail, y, _ptr(y), _ptr(s), _ptr(b), _ptr(f), _ptr(z), _ptr(codes), int(mode),
                _dtype_code(y, 'dblock_tail'), n, c, t, h, w, int(flags), int(act), float(alpha), float(gain), float(clamp))
        return z, codes

    def adjoint(self, dz, codes, f, in_size, flags, act, alpha, gain, want_ds):
        """(dy [N, C, *in_size], ds like dz or None, db fp32 [C]) from dz [N, C, T', H', W'] and the forward's codes."""
        _check_5d('dblock_tail', 'dz', dz)
        n, c = dz.shape[:2]
        t, h, w = (int(v) for v in in_size)
        nbytes = self.workspace(n, c, t, h, w, flags)
        if nbytes < 0 or list(dz.shape[2:]) != list(self.out_size((t, h, w), flags)):
            raise RuntimeError(f'dblock_tail_adjoint: no kernel for {[t, h, w]} -> {list(dz.shape)} (flags {flags})')
        self._check_codes(codes, dz, self.codes_bytes(n, c, t, h, w, flags))
        self._check_taps('dblock_tail_adjoint', f, flags, dz, 'dz')
        dz, f = dz.contiguous(), (None if f is None else f.contiguous())
        dy = torch.empty([n, c, t, h, w], dtype=dz.dtype, device=dz.device)
        ds = torch.empty_like(dz) if want_ds else None
        db = torch.empty([c], dtype=torch.float32, device=dz.device)
        ws = torch.empty([nbytes // 4], dtype=torch.float32, device=dz.device)
        _launch('dblock_tail_adjoint', self._lib.lvg_dblock_tail_adjoint, dz, _ptr(dz), _ptr(codes), _ptr(f), _ptr(dy), _ptr(ds), _ptr(db),
                _ptr(ws), nbytes, _dtype_code(dz, 'dblock_tail'), n, c, t, h, w, int(flags), int(act), float(alpha), float(gain))
        return dy, ds, db


class SresCondPlugin:
    """Input of a super-res generator layer: x_prev cast to the layer's dtype, concatenated with the layer's conditioning
    built from the low-res video, and optionally the mean square of the fp32 concatenation (no reference plugin:
    Generator.prep_cond, torch.cat and Tensor.to, generator_sres.py:581-610, 462-464, 307-325). ``plan_h`` / ``plan_w``:
    LVG_SRES_COND_NPLAN ints per axis (see lvg_sres_cond in include/lvg_ops.h and torch_utils/ops/sres_cond.py)."""

    NPLAN = 10

    def __init__(self, lib):
        self._lib = lib

    @classmethod
    def _plan(cls, q):
        if len(q) != cls.NPLAN:
            raise RuntimeError(f'sres_cond: a plan holds {cls.NPLAN} ints per axis')
        return (_c_int * cls.NPLAN)(*[int(v) for v in q])

    def workspace(self, n, t, c, c_lr, window, t_lr, h_lr, w_lr, dtype, plan_h, plan_w):
        """Workspace bytes of a call with the mean square, or -1 where the kernel does not take the shape and plan."""
        return int(self._lib.lvg_sres_cond_workspace(n, t, c, c_lr, window, t_lr, h_lr, w_lr, _DTYPE_CODE.get(dtype, -1),
                                                     self._plan(plan_h), self._plan(plan_w)))

    def forward(self, x, lr, f_h, f_w, plan_h, plan_w, gain_h, gain_w, window, dtype, want_sumsq):
        """(z [N T, C + C_lr window, H, W] in ``dtype``, mean square (fp32 0-dim) or None) from x [N T, C, H, W] (fp16 /
        fp32, or None) and lr [N, C_lr, T_lr, h, w] (fp32, any strides), T = T_lr - window + 1."""
        if not lr.is_cuda or lr.dtype != torch.float32 or lr.ndim != 5:
            raise RuntimeError('sres_cond: lr must be a 5-D float32 CUDA tensor')
        if dtype not in (torch.float16, torch.float32):
            raise RuntimeError(f'sres_cond: unsupported layer dtype {dtype}')
        n, c_lr, t_lr, h_lr, w_lr = lr.shape
        t = t_lr - window + 1
        c = 0
        if x is not None:
            if not x.is_cuda or x.dtype not in (torch.float16, torch.float32) or x.ndim != 4 or x.device != lr.device:
                raise RuntimeError('sres_cond: x must be a 4-D float16 / float32 tensor on the device of lr')
            if x.shape[0] != n * t or list(x.shape[2:]) != [int(plan_h[0]), int(plan_w[0])]:
                raise RuntimeError(f'sres_cond: x of shape {list(x.shape)} does not match the plan ({n * t} samples, '
                                   f'{int(plan_h[0])} x {int(plan_w[0])})')
            x = x.contiguous()
            c = x.shape[1]
        for f, q in ((f_h, plan_h), (f_w, plan_w)):
            k = int(q[9])
            if (k == 0) != (f is None) or f is not None and (f.dtype != torch.float32 or f.numel() != k or f.device != lr.device):
                raise RuntimeError(f'sres_cond: a filter of {k} float32 taps on the device of lr (None for an identity axis)')
        f_h = None if f_h is None else f_h.contiguous()
        f_w = None if f_w is None else f_w.contiguous()
        ph, pw = self._plan(plan_h), self._plan(plan_w)
        nbytes = int(self._lib.lvg_sres_cond_workspace(n, t, c, c_lr, window, t_lr, h_lr, w_lr, _DTYPE_CODE[dtype], ph, pw))
        if nbytes < 0:
            raise RuntimeError(f'sres_cond: no kernel for {list(lr.shape)}, window {window}, plan {list(plan_h)} / {list(plan_w)}')
        z = torch.empty([n * t, c + c_lr * window, int(plan_h[0]), int(plan_w[0])], dtype=dtype, device=lr.device)
        ms = ws = None
        if want_sumsq:
            ms = torch.empty([], dtype=torch.float32, device=lr.device)
            ws = torch.empty([nbytes // 8], dtype=torch.float64, device=lr.device)
        strides = (_c_i64 * 5)(*lr.stride())
        _launch('sres_cond', self._lib.lvg_sres_cond, lr, _ptr(x), _ptr(lr), _ptr(f_h), _ptr(f_w), _ptr(z), _ptr(ms), _ptr(ws), nbytes,
                _DTYPE_CODE[x.dtype] if x is not None else _DTYPE_CODE[dtype], _DTYPE_CODE[dtype], n, t, c, c_lr, window, t_lr, h_lr, w_lr,
                strides, ph, pw, float(gain_h), float(gain_w))
        return z, ms

    # ---- the layer's modulated convolution with z built in its re-tiling pass (lvg_sres_layer_*)

    def layer_workspace(self, n, t, c, c_lr, window, t_lr, h_lr, w_lr, dtype, plan_h, plan_w, cout, kh, kw, pad_h, pad_w):
        """Workspace bytes of lvg_sres_layer_fprop / _backward, or -1 where the kernels do not take the call."""
        return int(self._lib.lvg_sres_layer_workspace(_DTYPE_CODE.get(dtype, -1), n, t, c, c_lr, window, t_lr, h_lr, w_lr,
                                                      self._plan(plan_h), self._plan(plan_w), cout, kh, kw, pad_h, pad_w))

    def _layer_args(self, x, lr, f_h, f_w, plan_h, plan_w, window, dtype, w, a, d, padding):
        """Checked arguments shared by layer_fprop and layer_backward."""
        if not lr.is_cuda or lr.dtype != torch.float32 or lr.ndim != 5:
            raise RuntimeError('sres_layer: lr must be a 5-D float32 CUDA tensor')
        n, c_lr, t_lr, h_lr, w_lr = lr.shape
        t = t_lr - window + 1
        h, wd = int(plan_h[0]), int(plan_w[0])
        c = 0 if x is None else x.shape[1]
        if x is not None and (x.dtype not in (torch.float16, torch.float32) or x.device != lr.device
                              or tuple(x.shape) != (n * t, c, h, wd)):
            raise RuntimeError(f'sres_layer: x must be a float16 / float32 [{n * t}, C, {h}, {wd}] tensor on the device of lr')
        cin = c + c_lr * window
        if w.dtype != dtype or w.ndim != 4 or w.shape[1] != cin or w.device != lr.device:
            raise RuntimeError(f'sres_layer: w must be a {dtype} [Cout, {cin}, kh, kw] tensor on the device of lr')
        cout, kh, kw = int(w.shape[0]), int(w.shape[2]), int(w.shape[3])
        if a is not None and (a.dtype != torch.float32 or a.numel() != n * t * cin) or d is not None and (d.dtype != torch.float32 or
                                                                                                    d.numel() != n * t * cout):
            raise RuntimeError('sres_layer: a must be float32 [N T, Cin], d float32 [N T, Cout] or None')
        for f, q in ((f_h, plan_h), (f_w, plan_w)):
            k = int(q[9])
            if (k == 0) != (f is None) or f is not None and (f.dtype != torch.float32 or f.numel() != k or f.device != lr.device):
                raise RuntimeError(f'sres_layer: a filter of {k} float32 taps on the device of lr (None for an identity axis)')
        ph, pw = self._plan(plan_h), self._plan(plan_w)
        dims = (n, t, c, c_lr, window, t_lr, h_lr, w_lr)
        conv = (cout, kh, kw, int(padding[0]), int(padding[1]))
        need = int(self._lib.lvg_sres_layer_workspace(_DTYPE_CODE[dtype], *dims, ph, pw, *conv))
        if need < 0:
            raise RuntimeError(f'sres_layer: no kernel for {list(lr.shape)}, window {window}, C {c}, w {list(w.shape)}, '
                               f'padding {list(padding)}')
        return dict(x=None if x is None else x.contiguous(), f_h=None if f_h is None else f_h.contiguous(),
                    f_w=None if f_w is None else f_w.contiguous(), w=w.contiguous(), a=None if a is None else a.contiguous(),
                    d=None if d is None else d.contiguous(), dims=dims, conv=conv, ph=ph, pw=pw, need=need,
                    strides=(_c_i64 * 5)(*lr.stride()), out=(n * t, cout, h + 2 * conv[3] - kh + 1, wd + 2 * conv[4] - kw + 1))

    def layer_fprop(self, x, lr, f_h, f_w, plan_h, plan_w, gain_h, gain_w, window, dtype, w, a, d, padding, want_sumsq):
        """(y = d * conv(a * z, w) [N T, Cout, Ho, Wo] in ``dtype``, mean square of the fp32 z (0-dim) or None) with
        z = cat(x, cond(lr)).to(dtype) as ``forward`` builds it, never stored. a [N T, Cin], d [N T, Cout] or None: fp32.
        a None: (None, mean square) from the same pass without the convolution."""
        q = self._layer_args(x, lr, f_h, f_w, plan_h, plan_w, window, dtype, w, a, d, padding)
        if a is None and not want_sumsq:
            raise RuntimeError('sres_layer_fprop: a call without a computes the mean square alone')
        y = torch.empty(q['out'], dtype=dtype, device=lr.device) if a is not None else None
        ms = torch.empty([], dtype=torch.float32, device=lr.device) if want_sumsq else None
        ws = _workspace(lr.device, q['need'])
        xt = q['x']
        _launch('sres_layer_fprop', self._lib.lvg_sres_layer_fprop, lr, _ptr(xt), _ptr(lr), _ptr(q['f_h']), _ptr(q['f_w']), _ptr(q['w']),
                _ptr(q['a']), _ptr(q['d']), _ptr(y), _ptr(ms), _DTYPE_CODE[xt.dtype] if xt is not None else _DTYPE_CODE[dtype],
                _DTYPE_CODE[dtype], *q['dims'], q['strides'], q['ph'], q['pw'], float(gain_h), float(gain_w), *q['conv'], _ptr(ws),
                ws.numel())
        return y, ms

    def layer_backward(self, x, lr, f_h, f_w, plan_h, plan_w, gain_h, gain_w, window, dtype, w, a, d, y, dy, padding, want_dx=True,
                       want_dw=True):
        """Gradients of ``layer_fprop``'s y in one call: (dx in x's dtype or None, dw or None, da [N T, Cin], sum_hw dy * y
        [N T, Cout] or None when d is None)."""
        q = self._layer_args(x, lr, f_h, f_w, plan_h, plan_w, window, dtype, w, a, d, padding)
        dy = dy.contiguous()
        if dy.dtype != dtype or tuple(dy.shape) != q['out'] or dy.device != lr.device:
            raise RuntimeError(f'sres_layer_backward: dy must be a {dtype} tensor of shape {list(q["out"])}')
        xt = q['x']
        dx = torch.empty_like(xt) if (want_dx and xt is not None) else None
        dw = torch.empty_like(q['w']) if want_dw else None
        da = torch.empty(q['a'].shape, dtype=torch.float32, device=lr.device)
        dyy = None
        if d is not None:
            y = y.contiguous()
            dyy = torch.empty(q['d'].shape, dtype=torch.float32, device=lr.device)
        ws = _workspace(lr.device, q['need'])
        _launch('sres_layer_backward', self._lib.lvg_sres_layer_backward, lr, _ptr(xt), _ptr(lr), _ptr(q['f_h']), _ptr(q['f_w']),
                _ptr(q['w']), _ptr(q['a']), _ptr(q['d']), _ptr(y) if d is not None else None, _ptr(dy), _ptr(dx), _ptr(dw), _ptr(da),
                _ptr(dyy), _DTYPE_CODE[xt.dtype] if xt is not None else _DTYPE_CODE[dtype], _DTYPE_CODE[dtype], *q['dims'],
                q['strides'], q['ph'], q['pw'], float(gain_h), float(gain_w), *q['conv'], _ptr(ws), ws.numel())
        return dx, dw, da, dyy

    # ---- the ToRGB layer in one pass over its input (lvg_sres_torgb_*)

    def torgb_workspace(self, n, t, c, c_lr, window, t_lr, h_lr, w_lr, dtype, plan_h, plan_w, cout):
        """Workspace bytes of lvg_sres_torgb_backward, or -1 where the kernels do not take the call."""
        return int(self._lib.lvg_sres_torgb_workspace(_DTYPE_CODE.get(dtype, -1), n, t, c, c_lr, window, t_lr, h_lr, w_lr,
                                                      self._plan(plan_h), self._plan(plan_w), cout))

    def _torgb_args(self, x, lr, f_h, f_w, plan_h, plan_w, window, dtype, w, a, b):
        """Checked arguments shared by torgb_fprop and torgb_backward."""
        if not lr.is_cuda or lr.dtype != torch.float32 or lr.ndim != 5:
            raise RuntimeError('sres_torgb: lr must be a 5-D float32 CUDA tensor')
        n, c_lr, t_lr, h_lr, w_lr = lr.shape
        t = t_lr - window + 1
        h, wd = int(plan_h[0]), int(plan_w[0])
        if (x is None or x.dtype not in (torch.float16, torch.float32) or x.device != lr.device or x.ndim != 4
                or x.shape[0] != n * t or tuple(x.shape[2:]) != (h, wd)):
            raise RuntimeError(f'sres_torgb: x must be a float16 / float32 [{n * t}, C, {h}, {wd}] tensor on the device of lr')
        c = x.shape[1]
        cin = c + c_lr * window
        if w.dtype != dtype or w.ndim != 2 or w.shape[1] != cin or w.device != lr.device:
            raise RuntimeError(f'sres_torgb: w must be a {dtype} [Cout, {cin}] tensor on the device of lr')
        cout = int(w.shape[0])
        if a.dtype != torch.float32 or a.numel() != n * t * cin or a.device != lr.device:
            raise RuntimeError(f'sres_torgb: a must be a float32 [{n * t}, {cin}] tensor on the device of lr')
        if b.dtype != dtype or tuple(b.shape) != (cout,) or b.device != lr.device:
            raise RuntimeError(f'sres_torgb: b must be a {dtype} [{cout}] tensor on the device of lr')
        for f, q in ((f_h, plan_h), (f_w, plan_w)):
            k = int(q[9])
            if (k == 0) != (f is None) or f is not None and (f.dtype != torch.float32 or f.numel() != k or f.device != lr.device):
                raise RuntimeError(f'sres_torgb: a filter of {k} float32 taps on the device of lr (None for an identity axis)')
        ph, pw = self._plan(plan_h), self._plan(plan_w)
        dims = (n, t, c, c_lr, window, t_lr, h_lr, w_lr)
        need = int(self._lib.lvg_sres_torgb_workspace(_DTYPE_CODE[dtype], *dims, ph, pw, cout))
        if need < 0:
            raise RuntimeError(f'sres_torgb: no kernel for {list(lr.shape)}, window {window}, C {c}, w {list(w.shape)}')
        return dict(x=x.contiguous(), f_h=None if f_h is None else f_h.contiguous(), f_w=None if f_w is None else f_w.contiguous(),
                    w=w.contiguous(), a=a.contiguous(), b=b.contiguous(), dims=dims, cout=cout, ph=ph, pw=pw, need=need,
                    strides=(_c_i64 * 5)(*lr.stride()), out=(n * t, cout, h, wd))

    def torgb_fprop(self, x, lr, f_h, f_w, plan_h, plan_w, gain_h, gain_w, window, dtype, w, a, b, clamp, want_mask):
        """(y [N T, Cout, H, W] in ``dtype``, clamp mask [N T, H, W] uint8 or None): y = dtype(clamp(dtype(w r(a z)) + b))
        with z = cat(x, cond(lr)).to(dtype) as ``forward`` builds it, never stored. w [Cout, Cin] and b [Cout] in dtype, a
        [N T, Cin] fp32, clamp None for no clamp."""
        q = self._torgb_args(x, lr, f_h, f_w, plan_h, plan_w, window, dtype, w, a, b)
        y = torch.empty(q['out'], dtype=dtype, device=lr.device)
        mask = torch.empty([q['out'][0], q['out'][2], q['out'][3]], dtype=torch.uint8, device=lr.device) if want_mask else None
        xt = q['x']
        _launch('sres_torgb_fprop', self._lib.lvg_sres_torgb_fprop, lr, _ptr(xt), _ptr(lr), _ptr(q['f_h']), _ptr(q['f_w']), _ptr(q['w']),
                _ptr(q['a']), _ptr(q['b']), _ptr(y), _ptr(mask), _DTYPE_CODE[xt.dtype], _DTYPE_CODE[dtype], *q['dims'], q['strides'],
                q['ph'], q['pw'], float(gain_h), float(gain_w), q['cout'], float('inf') if clamp is None else float(clamp))
        return y, mask

    def torgb_backward(self, x, lr, f_h, f_w, plan_h, plan_w, gain_h, gain_w, window, dtype, w, a, b, mask, dy, want_dx=True,
                       want_dw=True, want_db=True):
        """Gradients of ``torgb_fprop``'s y in one call: (dx in x's dtype or None, dw [Cout, Cin] in dtype or None, da
        [N T, Cin] fp32, db [Cout] in dtype or None)."""
        q = self._torgb_args(x, lr, f_h, f_w, plan_h, plan_w, window, dtype, w, a, b)
        dy = dy.contiguous()
        if dy.dtype != dtype or tuple(dy.shape) != q['out'] or dy.device != lr.device:
            raise RuntimeError(f'sres_torgb_backward: dy must be a {dtype} tensor of shape {list(q["out"])}')
        if mask is None or mask.dtype != torch.uint8 or tuple(mask.shape) != (q['out'][0],) + q['out'][2:]:
            raise RuntimeError('sres_torgb_backward: the clamp mask of the forward call is needed')
        xt = q['x']
        dx = torch.empty_like(xt) if want_dx else None
        dw = torch.empty_like(q['w']) if want_dw else None
        da = torch.empty(q['a'].shape, dtype=torch.float32, device=lr.device)
        db = torch.empty_like(q['b']) if want_db else None
        ws = _workspace(lr.device, q['need'])
        _launch('sres_torgb_backward', self._lib.lvg_sres_torgb_backward, lr, _ptr(xt), _ptr(lr), _ptr(q['f_h']), _ptr(q['f_w']),
                _ptr(q['w']), _ptr(q['a']), _ptr(mask.contiguous()), _ptr(dy), _ptr(dx), _ptr(dw), _ptr(da), _ptr(db),
                _DTYPE_CODE[xt.dtype], _DTYPE_CODE[dtype], *q['dims'], q['strides'], q['ph'], q['pw'], float(gain_h), float(gain_w),
                q['cout'], _ptr(ws), ws.numel())
        return dx, dw, da, db


class LresTorgbPlugin:
    """The low-res generator's ToRGB layer in one pass over its input (DESIGN.md 7l; no reference plugin: ToRGB.forward
    composes MagnitudeEMA, ATen muls, F.conv3d and bias_act, generator_lres.py:618-641). x [N, Cin, T, H, W] fp16 / fp32
    is read in its own dtype; w fp32 [3, Cin], a fp32 [N, Cin, T], b fp32 [3]; ``dtype`` is the layer's."""

    def __init__(self, lib):
        self._lib = lib

    def workspace(self, x_dtype, dtype, n, cin, t, h, w, cout, kernel=(1, 1, 1)):
        """Workspace bytes of lvg_lres_torgb_backward (and of the forward's sum of squares), or -1 where the kernels do not
        take the call."""
        return int(self._lib.lvg_lres_torgb_workspace(_DTYPE_CODE.get(x_dtype, -1), _DTYPE_CODE.get(dtype, -1), n, cin, t, h, w,
                                                      cout, *(int(k) for k in kernel)))

    def _args(self, x, w, a, b, dtype):
        """Checked, dense arguments shared by every entry point, and the workspace the call needs."""
        if not x.is_cuda or x.dtype not in (torch.float16, torch.float32) or x.ndim != 5:
            raise RuntimeError('lres_torgb: x must be a 5-D float16 / float32 CUDA tensor')
        n, cin, t, h, wd = x.shape
        if w.dtype != torch.float32 or w.ndim != 2 or w.shape[1] != cin or w.device != x.device:
            raise RuntimeError(f'lres_torgb: w must be a float32 [3, {cin}] tensor on the device of x')
        if a.dtype != torch.float32 or tuple(a.shape) != (n, cin, t) or a.device != x.device:
            raise RuntimeError(f'lres_torgb: a must be a float32 [{n}, {cin}, {t}] tensor on the device of x')
        cout = int(w.shape[0])
        if b is not None and (b.dtype != torch.float32 or tuple(b.shape) != (cout,) or b.device != x.device):
            raise RuntimeError(f'lres_torgb: b must be a float32 [{cout}] tensor on the device of x')
        need = self.workspace(x.dtype, dtype, n, cin, t, h, wd, cout)
        if need < 0:
            raise RuntimeError(f'lres_torgb: no kernel for x {list(x.shape)} ({x.dtype}), w {list(w.shape)}, layer dtype {dtype}')
        return (x.contiguous(), w.contiguous(), a.contiguous(), None if b is None else b.contiguous(),
                (_DTYPE_CODE[x.dtype], _DTYPE_CODE[dtype], n, cin, t, h, wd, cout), need)

    def fprop(self, x, w, a, b, dtype, clamp):
        """y [N, 3, T, H, W] in dtype: dtype(clamp(dtype(sum_c w a r(x)) + dtype(b))), clamp None for none."""
        x, w, a, b, dims, _ = self._args(x, w, a, b, dtype)
        y = torch.empty([dims[2], dims[7], *x.shape[2:]], dtype=dtype, device=x.device)
        _launch('lres_torgb_fprop', self._lib.lvg_lres_torgb_fprop, x, _ptr(x), _ptr(w), _ptr(a), _ptr(b), _ptr(y), None, None,
                *dims, -1.0 if clamp is None else float(clamp), None, 0)
        return y

    def fprop_sumsq(self, x, w, a, dtype):
        """(u [N, 3, T, H, W] fp32 = sum_c w a r(x), sum of r(x)^2 over x as a 0-dim fp32 tensor), from one pass over x."""
        x, w, a, _, dims, need = self._args(x, w, a, None, dtype)
        u = torch.empty([dims[2], dims[7], *x.shape[2:]], dtype=torch.float32, device=x.device)
        sumsq = torch.empty([], dtype=torch.float32, device=x.device)
        ws = _workspace(x.device, need)
        _launch('lres_torgb_fprop', self._lib.lvg_lres_torgb_fprop, x, _ptr(x), _ptr(w), _ptr(a), None, None, _ptr(u), _ptr(sumsq),
                *dims, -1.0, _ptr(ws), ws.numel())
        return u, sumsq

    def finish(self, u, gain, b, dtype, clamp):
        """y = dtype(clamp(dtype(gain u) + dtype(b))) from fprop_sumsq's u, gain a 0-dim fp32 tensor on the device."""
        if not u.is_cuda or u.dtype != torch.float32 or u.ndim != 5 or u.shape[1] != 3:
            raise RuntimeError('lres_torgb_finish: u must be a float32 [N, 3, T, H, W] CUDA tensor')
        if gain.dtype != torch.float32 or gain.numel() != 1 or gain.device != u.device:
            raise RuntimeError('lres_torgb_finish: gain must be one float32 value on the device of u')
        if b.dtype != torch.float32 or tuple(b.shape) != (3,) or b.device != u.device:
            raise RuntimeError('lres_torgb_finish: b must be a float32 [3] tensor on the device of u')
        u, gain, b = u.contiguous(), gain.contiguous(), b.contiguous()
        n, _, t, h, wd = u.shape
        y = torch.empty(u.shape, dtype=dtype, device=u.device)
        _launch('lres_torgb_finish', self._lib.lvg_lres_torgb_finish, u, _ptr(u), _ptr(gain), _ptr(b), _ptr(y), _dtype_code(y, 'lres_torgb'),
                n, t, h, wd, -1.0 if clamp is None else float(clamp))
        return y

    def backward(self, x, w, a, y, dy, dtype, clamp, want_dx=True, want_dw=True, want_db=True):
        """(dx in x's dtype or None, dw fp32 [3, Cin] or None, da fp32 [N, Cin, T], db fp32 [3] or None) of fprop's y."""
        x, w, a, _, dims, need = self._args(x, w, a, None, dtype)
        shape = (dims[2], dims[7]) + tuple(x.shape[2:])
        for name, v in (('y', y), ('dy', dy)):
            if v.dtype != dtype or tuple(v.shape) != shape or v.device != x.device:
                raise RuntimeError(f'lres_torgb_backward: {name} must be a {dtype} tensor of shape {list(shape)}')
        y, dy = y.contiguous(), dy.contiguous()
        dx = torch.empty_like(x) if want_dx else None
        dw = torch.empty_like(w) if want_dw else None
        da = torch.empty_like(a)
        db = torch.empty([dims[7]], dtype=torch.float32, device=x.device) if want_db else None
        ws = _workspace(x.device, need)
        _launch('lres_torgb_backward', self._lib.lvg_lres_torgb_backward, x, _ptr(x), _ptr(w), _ptr(a), _ptr(y), _ptr(dy), _ptr(dx),
                _ptr(dw), _ptr(da), _ptr(db), *dims, -1.0 if clamp is None else float(clamp), _ptr(ws), ws.numel())
        return dx, dw, da, db


class GblockConv0Plugin:
    """The first modulated convolution of the low-res generator's residual block with its bias_act (DESIGN.md 7m; no
    reference plugin: Synthesis3dResBlock.forward composes temporal_modulated_conv3d, bias_act and MagnitudeEMA,
    generator_lres.py:568-575). x [N, Cin, T, H, W] fp16 / fp32, w [Cout, Cin, kt, kh, kw] in x's dtype, a fp32 [N, Cin, T],
    d fp32 [N, Cout, T], b fp32 [Cout] or None; act 1 linear, 2 lrelu."""

    def __init__(self, lib):
        self._lib = lib

    def workspace(self, dtype, n, cin, cout, t, h, w, kernel, padding):
        """Workspace bytes of lvg_gblock_conv0_fprop / _backward, or -1 where the op does not take the call."""
        return int(self._lib.lvg_gblock_conv0_workspace(_DTYPE_CODE.get(dtype, -1), n, cin, cout, t, h, w, *(int(k) for k in kernel),
                                                        *(int(p) for p in padding)))

    def _args(self, x, w, a, d, b, padding):
        """Checked, dense arguments shared by both entry points, and the workspace the call needs."""
        if not x.is_cuda or x.dtype not in (torch.float16, torch.float32) or x.ndim != 5:
            raise RuntimeError('gblock_conv0: x must be a 5-D float16 / float32 CUDA tensor')
        n, cin, t, h, wd = x.shape
        if w.dtype != x.dtype or w.ndim != 5 or w.shape[1] != cin or w.device != x.device:
            raise RuntimeError(f'gblock_conv0: w must be a {x.dtype} [Cout, {cin}, kt, kh, kw] tensor on the device of x')
        cout = int(w.shape[0])
        for name, f, shape in (('a', a, (n, cin, t)), ('d', d, (n, cout, t))):
            if f is None or f.dtype != torch.float32 or tuple(f.shape) != shape or f.device != x.device:
                raise RuntimeError(f'gblock_conv0: {name} must be a float32 {list(shape)} tensor on the device of x')
        if b is not None and (b.dtype != torch.float32 or tuple(b.shape) != (cout,) or b.device != x.device):
            raise RuntimeError(f'gblock_conv0: b must be a float32 [{cout}] tensor on the device of x')
        pad = tuple(int(p) for p in padding)
        need = self.workspace(x.dtype, n, cin, cout, t, h, wd, w.shape[2:], pad)
        if need < 0:
            raise RuntimeError(f'gblock_conv0: no kernel for x {list(x.shape)} ({x.dtype}), w {list(w.shape)}, padding {list(pad)}')
        dims = (_DTYPE_CODE[x.dtype], n, cin, cout, t, h, wd) + tuple(int(k) for k in w.shape[2:]) + pad
        return (x.contiguous(), w.contiguous(), a.contiguous(), d.contiguous(), None if b is None else b.contiguous(), dims, need)

    def fprop(self, x, w, a, d, b, padding, act, alpha, gain, clamp, want_sumsq=False):
        """(y [N, Cout, T, Ho, Wo] in x's dtype = clamp(act(d conv(a x, w) + b) gain), sum of y^2 as stored (0-dim fp32) or
        None); clamp < 0: none."""
        x, w, a, d, b, dims, need = self._args(x, w, a, d, b, padding)
        ho, wo = [s + 2 * p - k + 1 for s, p, k in zip(x.shape[3:], dims[11:], dims[8:10])]
        y = torch.empty([dims[1], dims[3], dims[4], ho, wo], dtype=x.dtype, device=x.device)
        sumsq = torch.empty([], dtype=torch.float32, device=x.device) if want_sumsq else None
        ws = _workspace(x.device, need)
        _launch('gblock_conv0_fprop', self._lib.lvg_gblock_conv0_fprop, x, _ptr(x), _ptr(w), _ptr(a), _ptr(d), _ptr(b), _ptr(y), _ptr(sumsq),
                *dims, int(act), float(alpha), float(gain), float(clamp), _ptr(ws), ws.numel())
        return y, sumsq

    def backward(self, x, w, a, d, b, y, dy, padding, act, alpha, gain, clamp, want_dw=True, want_dd=True, want_db=True):
        """(dx, dw or None, da fp32 [N, Cin, T], dd fp32 [N, Cout, T] or None, db fp32 [Cout] or None) of fprop's y, with
        bias_act's gradient decided from y."""
        x, w, a, d, b, dims, need = self._args(x, w, a, d, b, padding)
        if y.dtype != x.dtype or dy.dtype != x.dtype or dy.shape != y.shape or y.device != x.device or dy.device != x.device:
            raise RuntimeError(f'gblock_conv0_backward: y and dy must be {x.dtype} tensors of one shape on the device of x')
        y, dy = y.contiguous(), dy.contiguous()
        dx = torch.empty_like(x)
        dw = torch.empty_like(w) if want_dw else None
        da = torch.empty_like(a)
        dd = torch.empty_like(d) if want_dd else None
        db = torch.empty([dims[3]], dtype=torch.float32, device=x.device) if want_db else None
        ws = _workspace(x.device, need)
        _launch('gblock_conv0_backward', self._lib.lvg_gblock_conv0_backward, x, _ptr(x), _ptr(w), _ptr(a), _ptr(d), _ptr(b), _ptr(y), _ptr(dy),
                _ptr(dx), _ptr(dw), _ptr(da), _ptr(dd), _ptr(db), *dims, int(act), float(alpha), float(gain), float(clamp), _ptr(ws), ws.numel())
        return dx, dw, da, dd, db


class SresDblockPlugin:
    """The two native layers of a super-res discriminator block (DESIGN.md 7i): ``conv1`` (the 4-tap FIR in the
    convolution's re-tiling pass, the stride-2 3x3 convolution with its bias_act epilogue) and ``skip`` (the 1x1 convolution
    of the down-sampled input with the residual merge in its epilogue)."""

    def __init__(self, lib):
        self._lib = lib

    def conv1_workspace(self, dtype, n, cin, cout, h, w):
        return int(self._lib.lvg_sres_dblock_conv1_workspace(_DTYPE_CODE.get(dtype, -1), n, cin, cout, h, w))

    def skip_workspace(self, dtype, n, cin, cout, p):
        return int(self._lib.lvg_sres_dblock_skip_workspace(_DTYPE_CODE.get(dtype, -1), n, cin, cout, p))

    def conv1(self, x, fx, fy, flip, w, b, act, alpha, gain, clamp):
        """bias_act(conv2d(upfirdn2d(x, outer(fy, fx), padding=2, flip_filter=flip), w, stride=2), b, ...): act 1 linear, 2 lrelu."""
        x, w = x.contiguous(), w.contiguous()
        n, cin, h, wd = x.shape
        cout = w.shape[0]
        need = self.conv1_workspace(x.dtype, n, cin, cout, h, wd)
        if need < 0:
            raise RuntimeError('sres_dblock_conv1: outside the kernels\' envelope')
        y = torch.empty([n, cout, (h - 2) // 2 + 1, (wd - 2) // 2 + 1], dtype=x.dtype, device=x.device)
        ws = _workspace(x.device, need)
        if b is not None:
            b = b.to(torch.float32).contiguous()
        _launch('sres_dblock_conv1', self._lib.lvg_sres_dblock_conv1, x, _ptr(x), _ptr(fx), _ptr(fy), int(bool(flip)), _ptr(w), _ptr(b), _ptr(y),
                _DTYPE_CODE[x.dtype], n, cin, cout, h, wd, int(act), float(alpha), float(gain), float(clamp), _ptr(ws), ws.numel())
        return y

    def conv1_backward(self, x, fx, fy, flip, dy, w, want_dx=True, want_dw=True):
        """(d filtered image, dw) of conv1 from dy, the gradient of its pre-activation; dw's x operand is re-tiled from x
        through the FIR (the filtered image is not stored)."""
        x, dy, w = x.contiguous(), dy.contiguous(), w.contiguous()
        n, cin, h, wd = x.shape
        cout = w.shape[0]
        need = int(self._lib.lvg_sres_dblock_conv1_backward_workspace(_DTYPE_CODE.get(x.dtype, -1), n, cin, cout, h, wd))
        if need < 0:
            raise RuntimeError('sres_dblock_conv1_backward: outside the kernels\' envelope')
        dhf = torch.empty([n, cin, h + 1, wd + 1], dtype=x.dtype, device=x.device) if want_dx else None
        dw = torch.empty_like(w) if want_dw else None
        ws = _workspace(x.device, need)
        _launch('sres_dblock_conv1_backward', self._lib.lvg_sres_dblock_conv1_backward, x, _ptr(x), _ptr(fx), _ptr(fy), int(bool(flip)), _ptr(dy),
                _ptr(w), _ptr(dhf), _ptr(dw), _DTYPE_CODE[x.dtype], n, cin, cout, h, wd, _ptr(ws), ws.numel())
        return dhf, dw

    def fir_adjoint_act_workspace(self, dtype, n, c, h, w):
        return int(self._lib.lvg_sres_dblock_fir_adjoint_act_workspace(_DTYPE_CODE.get(dtype, -1), n, c, h, w))

    def fir_adjoint_act(self, dhf, h0, fx, fy, flip, act, alpha, gain, clamp, want_db=True):
        """(G(h0) * FIR^T(dhf), fp32 db or None): act 1 linear, 2 lrelu; db from per-CTA partials folded in a fixed order."""
        dhf, h0 = dhf.contiguous(), h0.contiguous()
        n, c, h, w = h0.shape
        need = self.fir_adjoint_act_workspace(h0.dtype, n, c, h, w)
        if need < 0:
            raise RuntimeError('sres_dblock_fir_adjoint_act: outside the kernel\'s envelope')
        dz = torch.empty_like(h0)
        db = torch.empty([c], dtype=torch.float32, device=h0.device) if want_db else None
        ws = torch.empty([need], dtype=torch.uint8, device=h0.device)
        _launch('sres_dblock_fir_adjoint_act', self._lib.lvg_sres_dblock_fir_adjoint_act, h0, _ptr(dhf), _ptr(h0), _ptr(fx), _ptr(fy),
                int(bool(flip)), _ptr(dz), _ptr(db), _ptr(ws), ws.numel(), _DTYPE_CODE[h0.dtype], n, c, h, w, int(act), float(alpha),
                float(gain), float(clamp))
        return dz, db

    def skip(self, x, w, r, rscale):
        """(conv2d(x, w) + r) * rscale for a 1x1 weight w [cout, cin, 1, 1]; r has the output's shape and x's dtype."""
        x, w, r = x.contiguous(), w.contiguous(), r.contiguous()
        n, cin, h, wd = x.shape
        cout = w.shape[0]
        need = self.skip_workspace(x.dtype, n, cin, cout, h * wd)
        if need < 0:
            raise RuntimeError('sres_dblock_skip: outside the kernel\'s envelope')
        y = torch.empty([n, cout, h, wd], dtype=x.dtype, device=x.device)
        ws = _workspace(x.device, need)
        _launch('sres_dblock_skip', self._lib.lvg_sres_dblock_skip, x, _ptr(x), _ptr(w), _ptr(r), _ptr(y), _DTYPE_CODE[x.dtype], n, cin, cout,
                h * wd, float(rscale), _ptr(ws), ws.numel())
        return y


_PLUGIN_CLASSES = {
    'gblock_conv0_plugin': GblockConv0Plugin,
    'lres_torgb_plugin': LresTorgbPlugin,
    'sres_dblock_plugin': SresDblockPlugin,
    'sres_cond_plugin': SresCondPlugin,
    'dblock_tail_plugin': DblockTailPlugin,
    'gblock_tail_plugin': GblockTailPlugin,
    'augment_pipe_plugin': AugmentPipePlugin,
    'video_augment_plugin': VideoAugmentPlugin,
    'convnd_plugin': ConvNdPlugin,
    'fir3d_plugin': Fir3dPlugin,
    'bias_act_plugin': BiasActPlugin,
    'upfirdn2d_plugin': Upfirdn2dPlugin,
    'filtered_lrelu_plugin': FilteredLReluPlugin,
    'fma_plugin': FmaPlugin,
}


def get_plugin(module_name, sources=None, headers=None, source_dir=None, **build_kwargs):
    """Same call shape as the reference loader (custom_ops.py:59); sources/headers/build flags
    are accepted and ignored because the library is prebuilt for sm_90a."""
    if module_name not in _plugins:
        if module_name not in _PLUGIN_CLASSES:
            raise RuntimeError(f'unknown plugin "{module_name}"')
        _plugins[module_name] = _PLUGIN_CLASSES[module_name](load_library())
    return _plugins[module_name]
