"""The low-res discriminator's input path: the reference LowResVideoGAN.run_D (staged at oracle/_ref/src by build()) against
the same method with video_augment.install, both with a stub D, at the low-res training shape (batch 8, 3 x 128 x 36 x 64
fp32, policy color,translation,cutout, temp_scale_augment = 1; train_lres.py:300-301). Three modes:

  fwd   forward only (update_D's real / generated pass)
  bwd   forward + backward of the logits (update_G)
  r1    forward, create_graph gradient of the logits, backward of its square (update_r1)

Per mode and side: ms per call (median over alternating rounds of CUDA-event timed calls), kernel launches and copies per
call (torch.profiler, a run of its own), peak memory above the inputs, and GB/s of the whole call against the map's
algorithmic bytes (per pass of the map or its adjoint: the source read, the destination written, and the reduction's
read of the source, 3 n 4 bytes). The GPU name, SM clock and power limit are read in the same run.

  python tools/bench_video_augment.py [--rounds 7] [--calls 20]
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
from model import video_gan_lres as vg                # noqa: E402
from torch_utils.ops import video_augment as va       # noqa: E402

N, C, T, H, W = 8, 3, 128, 36, 64
PASSES = {'fwd': 1, 'bwd': 2, 'r1': 4}                # passes of the map or its adjoint per call


class StubD(torch.nn.Module):
    def forward(self, video):
        return 0.5 * video.square().flatten(1).sum(1, keepdim=True)


def make_gan():
    g = vg.LowResVideoGAN.__new__(vg.LowResVideoGAN)
    g.seq_length, g.height, g.width, g.channels = T, H, W, C
    g.temp_scale_augment, g.diffaug_policy = 1.0, 'color,translation,cutout'
    g.D = StubD()
    return g


def call(g, x, mode):
    if mode == 'fwd':
        with torch.no_grad():
            return g.run_D(x)
    logits = g.run_D(x)
    if mode == 'bwd':
        logits.sum().backward()
    else:
        gx, = torch.autograd.grad(logits.sum(), [x], create_graph=True)
        gx.square().sum().backward()


def gpu_facts():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--calls', type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_video_augment needs a CUDA device'
    orig = vg.LowResVideoGAN.run_D
    va.install(vg)
    patched = vg.LowResVideoGAN.run_D
    sides = {'reference': orig, 'video_augment': patched}
    g = make_gan()
    x = torch.rand(N, C, T, H, W, device='cuda', generator=None) * 2 - 1
    xg = x.clone().requires_grad_(True)
    n_bytes = x.numel() * 4
    facts_before = gpu_facts()
    res = {}
    for mode in PASSES:
        xin = x if mode == 'fwd' else xg
        times = {s: [] for s in sides}
        for s, fn in sides.items():                    # warm-up
            vg.LowResVideoGAN.run_D = fn
            for _ in range(3):
                call(g, xin, mode)
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for s, fn in sides.items():
                vg.LowResVideoGAN.run_D = fn
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.calls):
                    call(g, xin, mode)
                    xg.grad = None
                e1.record()
                e1.synchronize()
                times[s].append(e0.elapsed_time(e1) / a.calls)
        for s, fn in sides.items():
            vg.LowResVideoGAN.run_D = fn
            xg.grad = None
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            call(g, xin, mode)
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            xg.grad = None
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                call(g, xin, mode)
                torch.cuda.synchronize()
            ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            kernels = sum(1 for e in ev if 'memcpy' not in e.name.lower() and 'memset' not in e.name.lower())
            copies = len(ev) - kernels
            xg.grad = None
            ms = statistics.median(times[s])
            res[(mode, s)] = dict(ms=ms, runs=[round(v, 4) for v in times[s]], kernels=kernels, copies=copies, peak_mb=peak / 2 ** 20,
                                  gbs=PASSES[mode] * 3 * n_bytes / (ms * 1e-3) / 1e9)
    vg.LowResVideoGAN.run_D = orig
    facts_after = gpu_facts()
    print(f'GPU (name, power limit, SM clock, max SM clock): before {facts_before}; after {facts_after}')
    print(f'batch {N}, {C}x{T}x{H}x{W} fp32, policy color,translation,cutout, temp_scale_augment 1; {a.rounds} rounds x {a.calls} calls')
    print('| mode | side | ms / call (median) | kernels + copies / call | peak MB above inputs | GB/s of the map\'s bytes |')
    print('|---|---|---|---|---|---|')
    for (mode, s), r in res.items():
        print(f'| {mode} | {s} | {r["ms"]:.3f} | {r["kernels"]} + {r["copies"]} | {r["peak_mb"]:.1f} | {r["gbs"]:.0f} |')
    print(json.dumps({f'{m}/{s}': r for (m, s), r in res.items()}))


if __name__ == '__main__':
    main()
