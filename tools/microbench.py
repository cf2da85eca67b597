"""Per-op achieved bandwidth on the GPU box: `python tools/microbench.py [filter]`.
Times each op signature with CUDA events (L2 flushed between iterations) and prints
algorithmic GB/s = (inputs read once + outputs written once) / time  (SURVEY.md 8d)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'long-video-gan_b200'))
from torch_utils.ops import bias_act, upfirdn2d, filtered_lrelu  # noqa: E402

DEV = 'cuda'
_flush = None


def flush_l2():
    global _flush
    if _flush is None:
        _flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=DEV)
    _flush.zero_()


def timeit(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        flush_l2()
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
    peak = 3350.0       # H100 SXM data sheet HBM3 rate (GB/s); a measured MEASURED_PEAKS.json replaces it
    try:
        peak = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs']
    except Exception:
        pass
    rows = []

    def run(name, fn, nbytes):
        if pat not in name:
            return
        ms = timeit(fn)
        gbs = nbytes / ms / 1e6
        rows.append((name, ms, gbs))
        print(f'{name:58s} {ms:8.3f} ms {gbs:8.1f} GB/s  {gbs / peak:5.2f} of measured copy peak', flush=True)

    for dt, sz in ((torch.float32, 4), (torch.float16, 2)):
        tag = 'f32' if sz == 4 else 'f16'
        # bias_act: lres G largest (N=8: 8x64x160x36x64), D first block
        for shape in ((8, 64, 160, 36, 64), (8, 32, 128, 64, 64), (8, 512, 24, 3, 4), (640, 1024)):
            x = torch.randn(*shape, device=DEV, dtype=dt)
            b = torch.randn(shape[1], device=DEV, dtype=dt)
            n = x.numel()
            run(f'bias_act fwd lrelu {tag} {shape}', lambda: bias_act.bias_act(x, b, act='lrelu', clamp=256), 2 * n * sz)
            run(f'bias_act fwd ref(torch) {tag} {shape}', lambda: bias_act.bias_act(x, b, act='lrelu', clamp=256, impl='ref'), 2 * n * sz)
            xg = x.clone().requires_grad_(True)
            bg = b.clone().requires_grad_(True)
            run(f'bias_act fwd lrelu (+2-bit codes for bwd) {tag} {shape}', lambda: bias_act.bias_act(xg, bg, act='lrelu', clamp=256), 2 * n * sz + n // 4)
            y = bias_act.bias_act(xg, bg, act='lrelu', clamp=256)
            dy = torch.randn_like(y)
            run(f'bias_act bwd dx+db (from codes) {tag} {shape}', lambda: torch.autograd.grad(y, [xg, bg], dy, retain_graph=True), 2 * n * sz + n // 4)
            if len(shape) == 5:
                from torch_utils import custom_ops
                plug = custom_ops.get_plugin('bias_act_plugin')
                yd = y.detach()
                run(f'bias_act bwd dx only (grad=1 kernel) {tag} {shape}',
                    lambda: plug.bias_act(dy, b, None, yd, None, 1, 1, 3, 0.2, 2 ** 0.5, 256.0), 3 * n * sz)
                out = torch.empty_like(x)
                run(f'bias_act ref 2R1W torch.add {tag} {shape}', lambda: torch.add(x, dy, out=out), 3 * n * sz)
                run(f'bias_act ref 1R1W torch.copy {tag} {shape}', lambda: out.copy_(x), 2 * n * sz)
            del x, xg, y, dy
        f4 = upfirdn2d.setup_filter([1, 3, 3, 1], separable=True).to(DEV)
        lin = (torch.tensor([1., 3., 3., 1.], device=DEV) / 8)[:, None]
        ups = [
            ('U3 up2 (8,8192,18,32)', (8, 8192, 18, 32), f4, dict(up=2, padding=[2, 1, 2, 1], gain=4)),
            ('U3 up2 tiny (8,16384,3,4)', (8, 16384, 3, 4), f4, dict(up=2, padding=[2, 1, 2, 1], gain=4)),
            ('U4 down2 (8,8192,64,64)', (8, 8192, 64, 64), f4, dict(down=2, padding=[1, 1, 1, 1])),
            ('U2 tup (8,256,80,144)', (8, 256, 80, 144), lin, dict(up=[1, 2], padding=[0, 0, 2, 1], gain=2)),
            ('U5 tdown (8,128,128,256)', (8, 128, 128, 256), lin, dict(down=[1, 2], padding=[0, 0, 1, 1])),
        ]
        for name, shape, f, kw in ups:
            x = torch.randn(*shape, device=DEV, dtype=dt)
            y = upfirdn2d.upfirdn2d(x, f, **kw)
            run(f'upfirdn2d {name} {tag}', lambda: upfirdn2d.upfirdn2d(x, f, **kw), (x.numel() + y.numel()) * sz)
            del x, y
        k12 = torch.randn(12, device=DEV) / 3
        k24 = torch.randn(24, device=DEV) / 5
        fls = [
            ('L4 up2/down2 (64,512,40,54)', (64, 512, 40, 54), k12, k12, dict(up=2, down=2, padding=[9, 8, 9, 8])),
            ('L5 up4/down2 (64,512,40,54)', (64, 512, 40, 54), k24, k12, dict(up=4, down=2, padding=[-6, -9, -6, -9])),
            ('L12 up2/down2 (64,128,166,278)', (64, 128, 166, 278), k12, k12, dict(up=2, down=2, padding=[9, 8, 9, 8])),
        ]
        for name, shape, fu, fd, kw in fls:
            x = torch.randn(*shape, device=DEV, dtype=dt)
            b = torch.randn(shape[1], device=DEV, dtype=dt)
            y = filtered_lrelu.filtered_lrelu(x, fu, fd, b, clamp=256, **kw)
            run(f'filtered_lrelu {name} {tag}', lambda: filtered_lrelu.filtered_lrelu(x, fu, fd, b, clamp=256, **kw), (x.numel() + y.numel()) * sz)
            del x, y
    # the conv boundary as the reference runs it today (cuDNN grouped conv through F.conv2d), for orientation
    for name, nt, cin, cout, h, w in (('L4 539->512 38x52', 64, 539, 512, 38, 52), ('L8 539->512 92x148', 16, 539, 512, 92, 148),
                                      ('L12 208->128 164x276', 16, 208, 128, 164, 276), ('L12 208->128 164x276', 4, 208, 128, 164, 276),
                                      ('L10 389->256 92x148', 16, 389, 256, 92, 148), ('L0 27->512 29x36', 64, 27, 512, 29, 36)):
        if pat not in 'conv2d cudnn':
            continue
        from torch_utils import custom_ops
        from torch_utils.ops import conv2d_gradfix
        x = torch.randn(1, nt * cin, h, w, device=DEV, dtype=torch.float16)
        wt = torch.randn(nt * cout, cin, 3, 3, device=DEV, dtype=torch.float16) / 70
        flops = 2.0 * nt * cout * cin * 9 * (h + 2) * (w + 2)
        ms = timeit(lambda: conv2d_gradfix.conv2d(x, wt, padding=2, groups=nt))
        print(f'conv2d engine grouped fp16 {name} NT={nt}: {ms:8.3f} ms {flops / ms / 1e9:8.1f} TFLOP/s', flush=True)
        if not (cin == 208 and nt > 4):     # cuDNN takes ~0.2 s on this shape: time it once at small NT only
            ms = timeit(lambda: torch.nn.functional.conv2d(x, wt, padding=2, groups=nt), iters=3, warmup=1)
            print(f'conv2d cudnn   grouped fp16 {name} NT={nt}: {ms:8.3f} ms {flops / ms / 1e9:8.1f} TFLOP/s', flush=True)
        # weight gradient: the engine vs aten::convolution_backward (cuDNN)
        plug = custom_ops.get_plugin('convnd_plugin')
        y = conv2d_gradfix.conv2d(x, wt, padding=2, groups=nt)
        dy = torch.randn_like(y)
        ms = timeit(lambda: plug.wgrad(x, dy, tuple(wt.shape), (2, 2), nt))
        print(f'conv2d wgrad engine fp16 {name} NT={nt}: {ms:8.3f} ms {flops / ms / 1e9:8.1f} TFLOP/s', flush=True)
        if not (cin == 208 and nt > 4):
            ms = timeit(lambda: torch.ops.aten.convolution_backward(dy, x, wt, None, [1, 1], [2, 2], [1, 1], False, [0, 0], nt,
                                                                    [False, True, False]), iters=3, warmup=1)
            print(f'conv2d wgrad cudnn   fp16 {name} NT={nt}: {ms:8.3f} ms {flops / ms / 1e9:8.1f} TFLOP/s', flush=True)
        del x, wt, y, dy
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    json.dump(rows, open(os.path.join(ROOT, 'gpurun_out', 'microbench.json'), 'w'), indent=1)


if __name__ == '__main__':
    main()
