"""``conv2d`` / ``conv_transpose2d`` entry points (``torch_utils.ops.conv2d_gradfix``).

Same functions and module switches as the reference (conv2d_gradfix.py:22-45):
``enabled``, ``weight_gradients_disabled``, ``no_weight_gradients()``. In the
reference the custom autograd path is inert on torch >= 1.11 (:49-58) and every
call lands in cuDNN. Here both functions are those of ``conv_nd``: CUDA calls
inside the envelope of the wgmma implicit-GEMM engine (csrc/conv_igemm.cu) run
on it, everything else goes to ``torch.nn.functional``.
"""
import contextlib

from .conv_nd import conv2d, conv_transpose2d  # noqa: F401

enabled = False                     # kept for API compatibility (train_lres.py:80 sets it)
weight_gradients_disabled = False   # forcefully skip weight gradients (R1 penalty, see no_weight_gradients)


@contextlib.contextmanager
def no_weight_gradients(disable=True):
    global weight_gradients_disabled
    old = weight_gradients_disabled
    if disable:
        weight_gradients_disabled = True
    yield
    weight_gradients_disabled = old
