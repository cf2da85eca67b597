"""Timing of the TMA-fed wgmma convolution engine against cuDNN (torch.nn.functional / aten::convolution_backward) on
the convolution shapes of the two training configurations. CUDA events, L2 flushed, median of 7.
    python tools/bench_convnd.py [filter] > profiles/r02_convnd.txt"""
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'long-video-gan_b200'))
from torch_utils import custom_ops  # noqa: E402

DEV = 'cuda'
_flush = None


def timeit(fn, iters=7, warmup=2):
    global _flush
    if _flush is None:
        _flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=DEV)
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        _flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    pat = sys.argv[1] if len(sys.argv) > 1 else ''
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    plug = custom_ops.get_plugin('convnd_plugin')
    old = custom_ops.get_plugin('conv2d_plugin')
    print(f'# {torch.cuda.get_device_name()}; TFLOP/s = 2*N*Cout*Cin*taps*out_pixels / time; cuDNN fp32 runs with TF32 off (as the reference)')
    print(f'# {"shape":58s} {"fprop":>22s} {"dgrad":>22s} {"wgrad":>22s}   ms (TFLOP/s): ours | cudnn')
    cases = [
        # name, x, w, pad, groups, dtype
        ('sres G L4 539->512 38x52 G=64 f16', (1, 64 * 539, 38, 52), (64 * 512, 539, 3, 3), (2, 2), 64, torch.float16),
        ('sres G L8 539->512 92x148 G=16 f16', (1, 16 * 539, 92, 148), (16 * 512, 539, 3, 3), (2, 2), 16, torch.float16),
        ('sres G L10 389->256 92x148 G=16 f16', (1, 16 * 389, 92, 148), (16 * 256, 389, 3, 3), (2, 2), 16, torch.float16),
        ('sres G L12 208->128 164x276 G=4 f16', (1, 4 * 208, 164, 276), (4 * 128, 208, 3, 3), (2, 2), 4, torch.float16),
        ('sres G L0 27->512 29x36 G=64 f32', (1, 64 * 27, 29, 36), (64 * 512, 27, 3, 3), (2, 2), 64, torch.float32),
        ('sres G L1 539->512 29x36 G=64 f32', (1, 64 * 539, 29, 36), (64 * 512, 539, 3, 3), (2, 2), 64, torch.float32),
        ('sres D b256 conv0 64->64 256x256 N=16 f16', (16, 64, 256, 256), (64, 64, 3, 3), (1, 1), 1, torch.float16),
        ('sres D b64 conv0 256->256 64x64 N=16 f16', (16, 256, 64, 64), (256, 256, 3, 3), (1, 1), 1, torch.float16),
        ('sres D b16 conv0 512->512 16x16 N=16 f32', (16, 512, 16, 16), (512, 512, 3, 3), (1, 1), 1, torch.float32),
        ('lres G 512->512 3x3x3 T96 9x16 N=8 f32', (8, 512, 96, 9, 16), (512, 512, 3, 3, 3), (1, 1, 1), 1, torch.float32),
        ('lres G 256->256 3x3x3 T176 9x16 N=8 f32', (8, 256, 176, 9, 16), (256, 256, 3, 3, 3), (1, 1, 1), 1, torch.float32),
        ('lres G 128->128 1x3x3 T160 18x32 N=8 f32', (8, 128, 160, 18, 32), (128, 128, 1, 3, 3), (0, 1, 1), 1, torch.float32),
        ('lres G 64->64 1x3x3 T160 36x64 N=8 f32', (8, 64, 160, 36, 64), (64, 64, 1, 3, 3), (0, 1, 1), 1, torch.float32),
        ('lres G 512->512 1x1x1 T56 5x8 N=8 f32', (8, 512, 56, 5, 8), (512, 512, 1, 1, 1), (0, 0, 0), 1, torch.float32),
        ('lres D 64->128 5x3x3 T128 32x32 N=8 f32', (8, 64, 128, 32, 32), (128, 64, 5, 3, 3), (2, 1, 1), 1, torch.float32),
        ('lres D 32->64 1x3x3 T128 64x64 N=8 f32', (8, 32, 128, 64, 64), (64, 32, 1, 3, 3), (0, 1, 1), 1, torch.float32),
        ('lres D conv1d 1024->1024 k3 L16 N=8 f32', (8, 1024, 16), (1024, 1024, 3), (1,), 1, torch.float32),
    ]
    for name, xs, ws, pad, groups, dt in cases:
        if pat not in name:
            continue
        nd = len(xs) - 2
        x = torch.randn(*xs, device=DEV, dtype=dt)
        w = torch.randn(*ws, device=DEV, dtype=dt) / math.sqrt(math.prod(ws[1:]))
        conv = (F.conv1d, F.conv2d, F.conv3d)[nd - 1]
        y = plug.fprop(x, w, pad, groups)
        ref = conv(x, w, padding=pad, groups=groups)
        err = float((y.float() - ref.float()).abs().max() / ref.float().abs().max())
        dy = torch.randn_like(y)
        flops = 2.0 * y.numel() * math.prod(ws[1:])
        slow_cudnn = groups > 1 and ws[1] == 208
        cells = []
        for ours, theirs in (
            (lambda: plug.fprop(x, w, pad, groups), lambda: conv(x, w, padding=pad, groups=groups)),
            (lambda: plug.dgrad(dy, w, xs, pad, groups),
             lambda: torch.ops.aten.convolution_backward(dy, x, w, None, [1] * nd, list(pad), [1] * nd, False, [0] * nd, groups, [True, False, False])),
            (lambda: plug.wgrad(x, dy, ws, pad, groups),
             lambda: torch.ops.aten.convolution_backward(dy, x, w, None, [1] * nd, list(pad), [1] * nd, False, [0] * nd, groups, [False, True, False])),
        ):
            a = timeit(ours)
            b = timeit(theirs, iters=3, warmup=1) if not slow_cudnn else float('nan')
            cells.append(f'{a:7.3f} ({flops / a / 1e9:5.0f}) |{b:7.3f}')
        extra = ''
        if nd == 2 and dt == torch.float16 and old.supported(x, w, (1, 1), pad, (1, 1), groups):
            extra = f'  r1 kernels: {timeit(lambda: old.fprop(x, w, pad, groups)):.3f} / {timeit(lambda: old.dgrad(dy, w, xs, pad, groups)):.3f}' \
                    f' / {timeit(lambda: old.wgrad(x, dy, ws, pad, groups)) if (groups > 1) else float("nan"):.3f}'
        print(f'{name:60s} {cells[0]:>22s} {cells[1]:>22s} {cells[2]:>22s}  err {err:.1e}{extra}', flush=True)
        del x, w, y, dy, ref


if __name__ == '__main__':
    main()
