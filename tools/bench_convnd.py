"""Timing of the TMA-fed wgmma convolution engine against cuDNN (torch.nn.functional / aten::convolution_backward) on
the convolution shapes of the two training configurations. CUDA events, L2 flushed, median of 7.
    python tools/bench_convnd.py [filter] > profiles/r02_convnd.txt
    python tools/bench_convnd.py --lres [filter]
--lres: every distinct conv3d / conv1d signature of the low-res G and D step (workloads/lres_step.json, batch 8) with its
calls per step, engine only. Per pass: ms, algorithmic TFLOP/s (2 * N * Cout * Cin * taps * output pixels) and executed
TFLOP/s (the tensor-core products the planned tiles issue: padded rows and columns, K padded to 16, three bf16 products
per fp32 product), both over the same time."""
import argparse
import collections
import ctypes
import json
import math
import os
import subprocess
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


def card():
    """name and power limit of the card the timings ran on"""
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = 'power limit unknown'
    return f'{torch.cuda.get_device_name()}, power limit / max SM clock {q}'


def executed_flops(lib, args, mode, split):
    """tensor-core multiply-adds x 2 that the planned launch issues for one pass (mode 0 forward, 1 input gradient,
    2 weight gradient), or None when the forward or input gradient runs on the streaming 1x1x1 kernels. args = the plugin's [dtype, n, groups, cin, cout, t, h, w,
    kt, kh, kw, pad_t, pad_h, pad_w]."""
    dt, n, groups, cin, cout, t, h, wd, kt, kh, kw, pt, ph, pw = args
    prods = 3 if split else 1
    if mode < 2:
        out = (ctypes.c_int * 48)()
        assert lib.lvg_convnd_plan(mode, *args, 1, out, 48) == 0, lib.lvg_last_error().decode()
        if out[47]:
            return None
        ncols, total_tiles, kc = out[22], out[26], out[3]
        ncw = out[39] if out[39] else -(-ncols // 64) * 64         # libraries without the field: 64-column chunks
        return 2.0 * total_tiles * (2 * 64 * ncw) * (kc * 16 * kt * kh * kw) * prods
    out = (ctypes.c_int * 32)()
    assert lib.lvg_convnd_wgrad_plan(*args, out, 32) == 0, lib.lvg_last_error().decode()
    nt, ntiles, mt, nseg, ps, rh, mrows = out[3], out[4], out[5], out[9], out[10], out[11], out[27]
    to, ho = t + 2 * pt - kt + 1, h + 2 * ph - kh + 1
    kpix = sum(-(-min(rh, ho - r0) * ps // 16) * 16 for r0 in range(0, ho, rh))
    return 2.0 * groups * mt * mrows * ntiles * nt * kt * kh * kw * n * to * nseg * kpix * prods


def lres_table(pat):
    tr = json.load(open(os.path.join(ROOT, 'workloads', 'lres_step.json')))
    plug = custom_ops.get_plugin('convnd_plugin')
    lib = custom_ops.load_library()
    batch = 8
    # passes per step: G forward x2 + backward x1, D forward x3 + backward x3
    mult = {'lres_G': (2, 1), 'lres_D': (3, 3)}
    tot = collections.Counter()
    print(f'# {card()}; batch {batch}; ms per call (algorithmic / executed TFLOP/s); calls per step = layers x passes')
    print(f'# {"net signature":62s} {"fwd":>6s} {"bwd":>4s} {"fprop":>21s} {"dgrad":>21s} {"wgrad":>21s}   per-step ms f / d / w')
    for net in ('lres_G', 'lres_D'):
        agg = collections.OrderedDict()
        for c in tr[net]:
            if c['op'] not in ('conv3d', 'conv1d'):
                continue
            key = (c['op'], tuple(c['x']), tuple(c['w']), tuple(c['padding']) if isinstance(c['padding'], list) else (c['padding'],), c['groups'])
            agg[key] = agg.get(key, 0) + 1
        for (op, xs, ws, pad, groups), layers in agg.items():
            xs = (batch,) + tuple(xs[1:])
            pad = tuple(pad) * (len(xs) - 2) if len(pad) == 1 else tuple(pad)
            name = f'{net[5:]} {op} {"x".join(map(str, xs[1:]))} w {"x".join(map(str, ws))}' + (f' G={groups}' if groups > 1 else '')
            if pat not in name:
                continue
            nf, nb = mult[net]
            x = torch.randn(*xs, device=DEV)
            w = torch.randn(*ws, device=DEV) / math.sqrt(math.prod(ws[1:]))
            if not plug.supported(x, w, 1, pad, 1, groups):
                print(f'{name:64s} {layers * nf:6d} {layers * nb:4d}   not on the engine', flush=True)
                continue
            y = plug.fprop(x, w, pad, groups)
            dy = torch.randn_like(y)
            flops = 2.0 * y.numel() * math.prod(ws[1:])
            args, _, _, _ = plug._args(tuple(xs), tuple(ws), pad, groups, x.dtype)
            cells, per = [], []
            for mode, fn, calls in ((0, lambda: plug.fprop(x, w, pad, groups), layers * nf),
                                    (1, lambda: plug.dgrad(dy, w, xs, pad, groups), layers * nb),
                                    (2, lambda: plug.wgrad(x, dy, ws, pad, groups), layers * nb)):
                ms = timeit(fn)
                ex = executed_flops(lib, args, mode, True)
                cells.append(f'{ms:7.3f} ({flops / ms / 1e9:4.0f} / {ex / ms / 1e9:4.0f})' if ex else f'{ms:7.3f} ({flops / ms / 1e9:4.0f} /  pw)')
                per.append(ms * calls)
            tot['f'] += per[0]; tot['d'] += per[1]; tot['w'] += per[2]
            print(f'{name:64s} {layers * nf:6d} {layers * nb:4d} {cells[0]:>21s} {cells[1]:>21s} {cells[2]:>21s}   {per[0]:7.2f} {per[1]:7.2f} {per[2]:7.2f}',
                  flush=True)
            del x, w, y, dy
    print(f'# per step: forward {tot["f"]:.1f} ms, input gradients {tot["d"]:.1f} ms, weight gradients {tot["w"]:.1f} ms')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('filter', nargs='?', default='')
    ap.add_argument('--lres', action='store_true', help='the signatures of the low-res training step, engine only')
    a = ap.parse_args()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    if a.lres:
        return lres_table(a.filter)
    pat = a.filter
    plug = custom_ops.get_plugin('convnd_plugin')
    print(f'# {card()}; TFLOP/s = 2*N*Cout*Cin*taps*out_pixels / time; cuDNN fp32 runs with TF32 off (as the reference)')
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
        print(f'{name:60s} {cells[0]:>22s} {cells[1]:>22s} {cells[2]:>22s}  err {err:.1e}', flush=True)
        del x, w, y, dy, ref


if __name__ == '__main__':
    main()
