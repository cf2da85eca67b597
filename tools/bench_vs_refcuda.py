"""Per-op timing of this repository's CUDA ops NEXT TO the reference's own CUDA ops (oracle/_ref, built unmodified for
sm_90a by oracle/build_ref.py) on the same H100, same inputs, at the full sizes of the two training configurations
(lres per-GPU batch 8; sres NT = 64). Forward, and forward+backward through autograd (dx [+db]) -- the public API on
both sides. CUDA events, L2 flushed between iterations, median of 10.

    python tools/bench_vs_refcuda.py [filter] > profiles/r02_vs_refcuda.txt
"""
import math
import os
import sys

import scipy.signal
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'long-video-gan_b200'))
sys.path.insert(0, ROOT)
from torch_utils.ops import bias_act, upfirdn2d, filtered_lrelu, conv2d_resample, conv2d_gradfix  # noqa: E402
from oracle import ref_cuda  # noqa: E402

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


def kaiser(taps, scale):
    return torch.tensor(scipy.signal.firwin(numtaps=taps, cutoff=0.5, width=0.6, fs=2.0 * scale), dtype=torch.float32, device=DEV)


def main():
    pat = sys.argv[1] if len(sys.argv) > 1 else ''
    ref = ref_cuda.load()
    assert ref.bias_act._init() and ref.upfirdn2d._init() and ref.filtered_lrelu._init()
    print(f'# {torch.cuda.get_device_name()}  torch {torch.__version__}; reference = its own plugins (oracle/_ref) + its own Python wrappers')
    print(f'# {"op / signature":64s} {"ours fwd":>9s} {"ref fwd":>9s} {"x":>6s} | {"ours f+b":>9s} {"ref f+b":>9s} {"x":>6s}   (ms)')
    worst = []

    def row(name, make):
        if pat not in name:
            return
        t = []
        for mod in ('ours', 'ref'):
            fwd, fb = make(mod)
            t.append((timeit(fwd), timeit(fb) if fb else float('nan')))
        (of, ob), (rf, rb) = t
        worst.append((rf / of, name + ' fwd'))
        if ob == ob:
            worst.append((rb / ob, name + ' fwd+bwd'))
        print(f'{name:66s} {of:9.3f} {rf:9.3f} {rf / of:6.2f} | {ob:9.3f} {rb:9.3f} {rb / ob:6.2f}', flush=True)

    F4 = [1., 3., 3., 1.]

    # ---- bias_act
    for shape, act, gain, dt in (((8, 64, 160, 36, 64), 'lrelu', None, torch.float32), ((8, 32, 128, 64, 64), 'lrelu', None, torch.float32),
                                 ((8, 256, 144, 9, 16), 'lrelu', None, torch.float32), ((8, 512, 24, 3, 4), 'lrelu', None, torch.float32),
                                 ((640, 1024), 'lrelu', None, torch.float32), ((16, 64, 256, 256), 'lrelu', math.sqrt(2), torch.float16),
                                 ((16, 512, 32, 32), 'lrelu', math.sqrt(2), torch.float16)):
        def make(which, shape=shape, act=act, gain=gain, dt=dt):
            m = bias_act if which == 'ours' else ref.bias_act
            x = torch.randn(*shape, device=DEV, dtype=dt).requires_grad_(True)
            b = torch.randn(shape[1], device=DEV, dtype=dt).requires_grad_(True)
            dy = torch.randn(*shape, device=DEV, dtype=dt)
            xd = x.detach()
            bd = b.detach()

            def fb():
                y = m.bias_act(x, b, act=act, gain=gain, clamp=256)
                torch.autograd.grad(y, [x, b], dy)
            return (lambda: m.bias_act(xd, bd, act=act, gain=gain, clamp=256)), fb
        row(f'bias_act {act} {"f32" if dt == torch.float32 else "f16"} {shape}', make)

    # ---- upfirdn2d
    lin = (torch.tensor(F4, device=DEV) / 8)[:, None]
    f4 = upfirdn2d.setup_filter(F4, separable=True).to(DEV)      # the low-res networks pass the 1-D taps (generator_lres.py:171-174)
    f44 = upfirdn2d.setup_filter(F4, separable=False).to(DEV)
    ups = [
        ('U1 kaiser tdown (8,1024,640,1)', (8, 1024, 640, 1), kaiser(12, 2)[:, None], dict(down=[1, 2], padding=[0, 0, 5, 5]), torch.float32),
        ('U2 tup (8,256,80,144)', (8, 256, 80, 144), lin, dict(up=[1, 2], padding=[0, 0, 2, 1], gain=2), torch.float32),
        ('U3 up2 (8,8192,18,32)', (8, 8192, 18, 32), f4, dict(up=2, padding=[2, 1, 2, 1], gain=4), torch.float32),
        ('U3 up2 (8,16384,3,4)', (8, 16384, 3, 4), f4, dict(up=2, padding=[2, 1, 2, 1], gain=4), torch.float32),
        ('U4 down2 (8,8192,64,64)', (8, 8192, 64, 64), f4, dict(down=2, padding=[1, 1, 1, 1]), torch.float32),
        ('U5 tdown (8,128,128,256)', (8, 128, 128, 256), lin, dict(down=[1, 2], padding=[0, 0, 1, 1]), torch.float32),
        ('U6 kaiser down4 (64,27,92,92)', (64, 27, 92, 92), kaiser(24, 4), dict(down=4, padding=6), torch.float32),
        ('U6 kaiser up4 (64,27,86,86)', (64, 27, 86, 86), kaiser(24, 4), dict(up=4, padding=[9, 6, 9, 6], gain=16), torch.float32),
        ('U7 lr up4 (16,24,36,64)', (16, 24, 36, 64), kaiser(8, 2), dict(up=4, padding=[5, 2, 5, 2], gain=16), torch.float32),
        ('U8 2-D pad2 f16 (16,64,256,256)', (16, 64, 256, 256), f44, dict(padding=2), torch.float16),
        ('U8 2-D down2 f16 (16,64,256,256)', (16, 64, 256, 256), f44, dict(down=2, padding=1), torch.float16),
    ]
    for name, shape, f, kw, dt in ups:
        def make(which, shape=shape, f=f, kw=kw, dt=dt):
            m = upfirdn2d if which == 'ours' else ref.upfirdn2d
            x = torch.randn(*shape, device=DEV, dtype=dt).requires_grad_(True)
            xd = x.detach()
            y0 = m.upfirdn2d(xd, f, **kw)
            dy = torch.randn_like(y0)

            def fb():
                torch.autograd.grad(m.upfirdn2d(x, f, **kw), [x], dy)
            return (lambda: m.upfirdn2d(xd, f, **kw)), fb
        row('upfirdn2d ' + name, make)

    # ---- filtered_lrelu (sres G, NT = 64)
    fls = [
        ('L1 up2/down2 f32 (64,512,31,38)', (64, 512, 31, 38), 2, 2, [9, 8, 9, 8], torch.float32),
        ('L3 up4/down2 f16 (64,512,31,38)', (64, 512, 31, 38), 4, 2, [-6, -9, -6, -9], torch.float16),
        ('L4 up2/down2 f16 (64,512,40,54)', (64, 512, 40, 54), 2, 2, [9, 8, 9, 8], torch.float16),
        ('L5 up4/down2 f16 (64,512,40,54)', (64, 512, 40, 54), 4, 2, [-6, -9, -6, -9], torch.float16),
        ('L8 up2/down2 f16 (64,512,94,150)', (64, 512, 94, 150), 2, 2, [9, 8, 9, 8], torch.float16),
        ('L10 up4/down2 f16 (64,256,94,150)', (64, 256, 94, 150), 4, 2, [-6, -9, -6, -9], torch.float16),
        ('L12 up2/down2 f16 (64,128,166,278)', (64, 128, 166, 278), 2, 2, [9, 8, 9, 8], torch.float16),
        ('L13 crop f16 (64,128,166,278)', (64, 128, 166, 278), 2, 2, [-11, -12, -11, -12], torch.float16),
        ('ToRGB 1x1 f16 (64,3,144,256)', (64, 3, 144, 256), 1, 1, [0, 0, 0, 0], torch.float16),
    ]
    for name, shape, up, down, pad, dt in fls:
        def make(which, shape=shape, up=up, down=down, pad=pad, dt=dt):
            m = filtered_lrelu if which == 'ours' else ref.filtered_lrelu
            fu = kaiser(6 * up, up) if up > 1 else None
            fd = kaiser(6 * down, down) if down > 1 else None
            x = torch.randn(*shape, device=DEV, dtype=dt).requires_grad_(True)
            b = torch.randn(shape[1], device=DEV, dtype=dt).requires_grad_(True)
            xd, bd = x.detach(), b.detach()
            g, s = (1.0, 1.0) if up == 1 else (math.sqrt(2), 0.2)
            y0 = m.filtered_lrelu(xd, fu, fd, bd, up=up, down=down, padding=pad, gain=g, slope=s, clamp=256)
            dy = torch.randn_like(y0)

            def fb():
                y = m.filtered_lrelu(x, fu, fd, b, up=up, down=down, padding=pad, gain=g, slope=s, clamp=256)
                torch.autograd.grad(y, [x, b], dy)
            return (lambda: m.filtered_lrelu(xd, fu, fd, bd, up=up, down=down, padding=pad, gain=g, slope=s, clamp=256)), fb
        row('filtered_lrelu ' + name, make)

    # ---- conv2d_resample (sres D, N = 16) and the modulated grouped conv (sres G): reference = its Python over cuDNN
    crs = [
        ('b256 conv0 3x3 f16 (16,64,256,256)', (16, 64, 256, 256), (64, 64, 3, 3), dict(padding=1), False, torch.float16),
        ('b256 conv1 down2 f16 (16,64,256,256)', (16, 64, 256, 256), (128, 64, 3, 3), dict(down=2, padding=1), True, torch.float16),
        ('b256 skip 1x1 down2 f16', (16, 64, 256, 256), (128, 64, 1, 1), dict(down=2), True, torch.float16),
        ('b64 conv1 down2 f16 (16,256,64,64)', (16, 256, 64, 64), (512, 256, 3, 3), dict(down=2, padding=1), True, torch.float16),
        ('b16 conv0 f32 (16,512,16,16)', (16, 512, 16, 16), (512, 512, 3, 3), dict(padding=1), False, torch.float32),
        ('b16 conv1 down2 f32 (16,512,16,16)', (16, 512, 16, 16), (512, 512, 3, 3), dict(down=2, padding=1), True, torch.float32),
    ]
    torch.backends.cudnn.allow_tf32 = False
    for name, xs, ws, kw, usef, dt in crs:
        def make(which, xs=xs, ws=ws, kw=kw, usef=usef, dt=dt):
            m = conv2d_resample if which == 'ours' else ref.conv2d_resample
            x = torch.randn(*xs, device=DEV, dtype=dt).requires_grad_(True)
            w = (torch.randn(*ws, device=DEV, dtype=dt) / math.sqrt(ws[1] * ws[2] * ws[3])).requires_grad_(True)
            f = f44 if usef else None
            xd, wd = x.detach(), w.detach()
            y0 = m.conv2d_resample(xd, wd, f=f, **kw)
            dy = torch.randn_like(y0)

            def fb():
                torch.autograd.grad(m.conv2d_resample(x, w, f=f, **kw), [x, w], dy)
            return (lambda: m.conv2d_resample(xd, wd, f=f, **kw)), fb
        row('conv2d_resample ' + name, make)
    for name, nt, cin, cout, h, w_ in (('L4 539->512 38x52 NT=64', 64, 539, 512, 38, 52), ('L8 539->512 92x148 NT=16', 16, 539, 512, 92, 148),
                                       ('L10 389->256 92x148 NT=16', 16, 389, 256, 92, 148), ('L0 27->512 29x36 NT=64', 64, 27, 512, 29, 36)):
        def make(which, nt=nt, cin=cin, cout=cout, h=h, w_=w_):
            m = conv2d_gradfix if which == 'ours' else ref.conv2d_gradfix
            x = torch.randn(1, nt * cin, h, w_, device=DEV, dtype=torch.float16).requires_grad_(True)
            w = (torch.randn(nt * cout, cin, 3, 3, device=DEV, dtype=torch.float16) / 70).requires_grad_(True)
            xd, wd = x.detach(), w.detach()
            dy = torch.randn(1, nt * cout, h + 2, w_ + 2, device=DEV, dtype=torch.float16)

            def fb():
                torch.autograd.grad(m.conv2d(x, w, padding=2, groups=nt), [x, w], dy)
            return (lambda: m.conv2d(xd, wd, padding=2, groups=nt)), fb
        row('conv2d modulated grouped f16 ' + name, make)

    worst.sort()
    print('# slowest relative to the reference: ' + '; '.join(f'{n} {r:.2f}x' for r, n in worst[:6]))


if __name__ == '__main__':
    main()
