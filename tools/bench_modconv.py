"""Modulated convolutions of the two generators: today's path (the reference's own modulated_conv2d /
temporal_modulated_conv3d, staged under oracle/_ref/src, over this repository's convolution engine) against the fused op
(torch_utils.ops.modulated_conv), per layer signature and for the whole unmodified generators with and without install().

    python tools/bench_modconv.py [--iters 20] [--warmup 3] [--skip-nets]

Per layer: forward and forward + backward times from CUDA events after warm-up, the two variants alternating in the same
process, and torch.cuda.max_memory_allocated above the inputs. Super-res: per-GPU batch 8 x 8 frames = 64 samples, the
network's fp16 / fp32 layer dtypes (workloads/sres_step.json). Low-res: per-GPU batch 8, T = 160 frames, fp32. Prints one
JSON line per measurement with the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import types
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
for p in (SRC, PKG):
    sys.path.insert(0, p)
warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))

from model import generator_lres, generator_sres          # noqa: E402
from torch_utils.ops import conv_nd, modulated_conv as mc  # noqa: E402

REF_SRES, REF_LRES = generator_sres.modulated_conv2d, generator_lres.temporal_modulated_conv3d
conv_nd.install_functional(generator_lres)                 # today's path: the reference function's F.conv3d on the engine

# (cin, cout, k, h, w, padding, fp16, calls per forward) -- super-res G L0-L14 per sample
SRES = [(27, 512, 3, 29, 36, 2, False, 1), (539, 512, 3, 29, 36, 2, False, 1), (539, 512, 3, 38, 52, 2, True, 2),
        (539, 512, 3, 56, 84, 2, True, 2), (539, 512, 3, 92, 148, 2, True, 2), (539, 362, 3, 92, 148, 2, True, 1),
        (389, 256, 3, 92, 148, 2, True, 1), (283, 181, 3, 164, 276, 2, True, 1), (208, 128, 3, 164, 276, 2, True, 1),
        (155, 128, 3, 164, 276, 2, True, 2), (155, 3, 1, 144, 256, 0, True, 1)]
# (cin, cout, kernel, t, h, w, padding) -- low-res G conv0 / conv1 / ToRGB at the T = 160 layer lengths
LRES = [(512, 512, (3, 3, 3), 21, 3, 4, (1, 1, 1)), (512, 512, (3, 3, 3), 26, 3, 4, (1, 1, 1)), (512, 512, (3, 3, 3), 36, 5, 8, (1, 1, 1)),
        (512, 512, (3, 3, 3), 56, 5, 8, (1, 1, 1)), (512, 512, (3, 3, 3), 96, 9, 16, (1, 1, 1)), (512, 256, (3, 3, 3), 96, 9, 16, (1, 1, 1)),
        (256, 256, (3, 3, 3), 176, 9, 16, (1, 1, 1)), (256, 256, (1, 3, 3), 160, 9, 16, (0, 1, 1)), (256, 128, (1, 3, 3), 160, 9, 16, (0, 1, 1)),
        (128, 128, (1, 3, 3), 160, 18, 32, (0, 1, 1)), (128, 64, (1, 3, 3), 160, 18, 32, (0, 1, 1)), (64, 64, (1, 3, 3), 160, 36, 64, (0, 1, 1)),
        (64, 3, (1, 1, 1), 160, 36, 64, (0, 0, 0))]


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'], capture_output=True, text=True, timeout=30)
        name, plim = [v.strip() for v in q.stdout.strip().split(',')[:2]]
    except Exception:       # noqa: BLE001 -- the name from torch, the limit unknown
        name, plim = torch.cuda.get_device_name(0), 'unknown'
    return dict(gpu=name, power_limit=plim)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def layer(kind, sig, args, iters, warmup, meta):
    x, w, s, g, kw = args
    fns = {'today': REF_SRES if kind == 'sres' else REF_LRES, 'fused': mc.modulated_conv2d if kind == 'sres' else mc.temporal_modulated_conv3d}

    def call(f):
        if kind == 'sres':
            return f(x=x, w=w, s=s, input_gain=g, **kw)
        return f(x, w, s, g, **kw)

    def fwd(f):
        with torch.no_grad():
            call(f)

    def fwd_bwd(f):
        y = call(f)
        torch.autograd.grad(y, [x, w, s], torch.ones_like(y))

    res = {v: {} for v in fns}
    for rep in range(2):                                  # alternate the variants, twice
        for v, f in fns.items():
            res[v].setdefault('fwd_ms', []).append(timed(lambda: fwd(f), iters, warmup))
            res[v].setdefault('fwd_bwd_ms', []).append(timed(lambda: fwd_bwd(f), iters, warmup))
    for v, f in fns.items():
        res[v]['peak_fwd_bwd_bytes'] = peak(lambda: fwd_bwd(f))
        res[v]['fwd_ms'] = min(res[v]['fwd_ms'])
        res[v]['fwd_bwd_ms'] = min(res[v]['fwd_bwd_ms'])
    print(json.dumps(dict(meta, kind=kind, sig=list(map(str, sig)), today=res['today'], fused=res['fused'],
                          speedup_fwd_bwd=res['today']['fwd_bwd_ms'] / res['fused']['fwd_bwd_ms'])), flush=True)


def nets(iters, warmup, meta):
    dev = torch.device('cuda')
    installed = False
    for install in (False, True):
        if install and not installed:
            mc.install(generator_sres, generator_lres)
            installed = True
        torch.manual_seed(3)
        S = generator_sres.VideoGenerator(hr_height=144, hr_width=256, lr_height=36, lr_width=64, temporal_context=4, num_fp16_res=4,
                                          fourfeats=False).to(dev)
        lr = (torch.rand(8, 3, 8 + 8, 36, 64, generator=torch.Generator().manual_seed(13)) * 2 - 1).to(dev)

        def sres_step():
            S(lr).float().square().mean().backward()
        t = timed(sres_step, max(3, iters // 4), warmup)
        m = peak(sres_step)
        print(json.dumps(dict(meta, kind='sres_G_step', batch=8, frames=8, install=install, step_ms=t, peak_bytes=m)), flush=True)
        del S, lr
        torch.manual_seed(0)
        G = generator_lres.VideoGenerator(out_height=36, out_width=64, num_fp16_layers=0, temporal_padding=8, temporal_emb_dim=1024).to(dev)

        def lres_step():
            G(8, 128).square().mean().backward()
        t = timed(lres_step, max(3, iters // 4), warmup)
        m = peak(lres_step)
        print(json.dumps(dict(meta, kind='lres_G_step', batch=8, frames=128, install=install, step_ms=t, peak_bytes=m)), flush=True)
        del G
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--skip-nets', action='store_true')
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_modconv needs a CUDA device'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    meta = card()
    dev = torch.device('cuda')
    gen = torch.Generator(device=dev).manual_seed(0)
    for (cin, cout, k, h, wd, pad, fp16, calls) in SRES:
        n = 64
        dt = torch.float16 if fp16 else torch.float32
        x = torch.randn(n, cin, h, wd, device=dev, generator=gen).to(dt).requires_grad_(True)
        w = torch.randn(cout, cin, k, k, device=dev, generator=gen).requires_grad_(True)
        s = (torch.randn(n, cin, device=dev, generator=gen) + 1).requires_grad_(True)
        g = torch.tensor(0.5, device=dev)
        layer('sres', (cin, cout, k, h, wd, 'f16' if fp16 else 'f32', f'x{calls}'), (x, w, s, g, dict(demodulate=k == 3, padding=pad)),
              args.iters, args.warmup, meta)
        del x, w, s
    for (cin, cout, k, t, h, wd, pad) in LRES:
        n = 8
        x = torch.randn(n, cin, t, h, wd, device=dev, generator=gen).requires_grad_(True)
        w = torch.randn(cout, cin, *k, device=dev, generator=gen).requires_grad_(True)
        s = torch.randn(n, cin, t, device=dev, generator=gen).requires_grad_(True)
        g = torch.tensor(0.5, device=dev)
        layer('lres', (cin, cout, 'x'.join(map(str, k)), t, h, wd), (x, w, s, g, dict(padding=pad, demodulate=cout != 3)), args.iters, args.warmup, meta)
        del x, w, s
    torch.cuda.empty_cache()
    if not args.skip_nets:
        nets(args.iters, args.warmup, meta)


if __name__ == '__main__':
    main()
