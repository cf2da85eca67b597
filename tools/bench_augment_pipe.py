"""ADA's AugmentPipe of the super-res step: the reference forward (staged at oracle/_ref/src by build()) against the same
method with augment_pipe.install, in the two configurations SuperResVideoGAN builds (video_gan_sres.py:110-136):

  augment      train_sres.py:360-373 kwargs on the stacked clip [8, 3, 8, 144, 256] fp32, at p = 0 and p = 0.5
  augment_clamp  the same shape with scale_std = 3 at p = 1, so that the margins reach their clamp (W - 1, H - 1)
  in_augment   strength 8, p = 0.5 on the conditioning clip [8, 3, 12, 36, 64]

and three modes per configuration, with a stub loss 0.5 * sum(y^2):

  fwd   forward only
  bwd   forward + backward
  r1    forward, create_graph gradient, backward of its square (update_r1)

Per configuration, mode and side: ms per call (median over alternating rounds of CUDA-event timed calls), kernels and
copies per call and device-to-host synchronisations per call (torch.profiler, a run of its own), and peak memory above the
inputs. The GPU name, power limit and SM clocks are read in the same run.

  python tools/bench_augment_pipe.py [--rounds 7] [--calls 10]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
sys.path[:0] = [os.path.join(ROOT, 'long-video-gan_b200'), SRC]
warnings.filterwarnings('ignore')
sys.modules.setdefault('imageio', types.ModuleType('imageio'))
sys.modules.setdefault('utils', types.ModuleType('utils'))

import torch                                          # noqa: E402
from model import ada_augment                         # noqa: E402
from torch_utils.ops import augment_pipe as ap        # noqa: E402
from torch_utils.ops import grid_sample_gradfix       # noqa: E402

grid_sample_gradfix.enabled = True                    # as train_sres.py:84 sets it: the reference's R1 pass needs it

AUGMENT = dict(xflip=1, rotate90=1, xint=1, scale=1, rotate=1, aniso=1, xfrac=1, brightness=1, contrast=1, lumaflip=1, hue=1,
               saturation=1)
IN_AUGMENT = dict(scale=1, scale_std=0.08, rotate=1, rotate_max=0.016, aniso=1, aniso_std=0.08, xfrac=1, xfrac_std=0.016, noise=1,
                  noise_std=0.08)
# name: (kwargs, p, shape)
CONFIGS = {
    'augment p=0': (AUGMENT, 0.0, (8, 3, 8, 144, 256)),
    'augment p=0.5': (AUGMENT, 0.5, (8, 3, 8, 144, 256)),
    'augment clamp': (dict(AUGMENT, scale_std=3.0), 1.0, (8, 3, 8, 144, 256)),
    'in_augment p=0.5': (IN_AUGMENT, 0.5, (8, 3, 12, 36, 64)),
}
MODES = ('fwd', 'bwd', 'r1')


def call(pipe, x, mode):
    if mode == 'fwd':
        with torch.no_grad():
            return pipe(x)
    loss = 0.5 * pipe(x).square().sum()
    if mode == 'bwd':
        loss.backward()
    else:
        gx, = torch.autograd.grad(loss, [x], create_graph=True)
        gx.square().sum().backward()


def gpu_facts():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    a = argparse.ArgumentParser()
    a.add_argument('--rounds', type=int, default=7)
    a.add_argument('--calls', type=int, default=10)
    a = a.parse_args()
    assert torch.cuda.is_available(), 'bench_augment_pipe needs a CUDA device'
    orig = ada_augment.AugmentPipe.forward
    ap.install(ada_augment)
    sides = {'reference': orig, 'augment_pipe': ada_augment.AugmentPipe.forward}
    facts_before = gpu_facts()
    res = {}
    margins = {}
    for cname, (kw, p, shape) in CONFIGS.items():
        pipe = ada_augment.AugmentPipe(**kw).cuda().requires_grad_(False).train()
        pipe.p.fill_(p)
        x = torch.rand(shape, device='cuda') * 2 - 1
        xg = x.clone().requires_grad_(True)
        torch.manual_seed(0)
        margins[cname] = [int(v) for v in ap.draw_params(pipe, x)[0][0, :4].tolist()]
        for mode in MODES:
            xin = x if mode == 'fwd' else xg
            times = {s: [] for s in sides}
            for s, fn in sides.items():                # warm-up
                ada_augment.AugmentPipe.forward = fn
                for _ in range(2):
                    call(pipe, xin, mode)
                    xg.grad = None
            torch.cuda.synchronize()
            for r in range(a.rounds):
                for s, fn in sides.items():
                    ada_augment.AugmentPipe.forward = fn
                    torch.manual_seed(r)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(a.calls):
                        call(pipe, xin, mode)
                        xg.grad = None
                    e1.record()
                    e1.synchronize()
                    times[s].append(e0.elapsed_time(e1) / a.calls)
            for s, fn in sides.items():
                ada_augment.AugmentPipe.forward = fn
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                call(pipe, xin, mode)
                torch.cuda.synchronize()
                peak = torch.cuda.max_memory_allocated() - base
                xg.grad = None
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
                    call(pipe, xin, mode)
                    torch.cuda.synchronize()
                xg.grad = None
                ev = prof.events()
                dev = [e for e in ev if e.device_type == torch.autograd.DeviceType.CUDA]
                kernels = sum(1 for e in dev if 'memcpy' not in e.name.lower() and 'memset' not in e.name.lower())
                syncs = sum(1 for e in ev if e.name in ('cudaStreamSynchronize', 'cudaMemcpy'))
                dtoh = sum(1 for e in dev if 'dtoh' in e.name.lower().replace(' ', ''))
                res[(cname, mode, s)] = dict(ms=statistics.median(times[s]), runs=[round(v, 3) for v in times[s]], kernels=kernels,
                                             copies=len(dev) - kernels, syncs=syncs, dtoh=dtoh, peak_mb=peak / 2 ** 20)
        del pipe, x, xg
        torch.cuda.empty_cache()
    ada_augment.AugmentPipe.forward = orig
    facts_after = gpu_facts()
    print(f'GPU (name, power limit, SM clock, max SM clock): before {facts_before}; after {facts_after}')
    print(f'{a.rounds} alternating rounds x {a.calls} calls; margins (mx0, my0, mx1, my1) of seed 0: {margins}')
    print('| configuration | mode | side | ms / call (median) | kernels + copies / call | D2H syncs / call | peak MB above inputs |')
    print('|---|---|---|---|---|---|---|')
    for (c, m, s), r in res.items():
        print(f'| {c} | {m} | {s} | {r["ms"]:.3f} | {r["kernels"]} + {r["copies"]} | {r["syncs"]} ({r["dtoh"]} D2H copies) | {r["peak_mb"]:.1f} |')
    print(json.dumps({f'{c}/{m}/{s}': r for (c, m, s), r in res.items()}))


if __name__ == '__main__':
    main()
