"""The low-res generator's residual blocks: the reference Synthesis3dResBlock.forward (staged at oracle/_ref/src by build())
against the same method with gblock_tail.install, in the default VideoGenerator (36 x 64, batch 8, 128 frames, fp32, TF32
off), both sides with the generator's convolutions on this repository's engine (conv_nd.install_functional and
modulated_conv.install, as a training run configures them). Magnitude-EMA beta 1 (G's default call).

  per block   forward (no grad) and forward + backward of one block on the inputs the generator feeds it
  whole G     forward without grad (update_D's generated pass) and forward + backward (update_G)
  memory      peak memory of the whole-G forward + backward above the parameters

ms per call: median over alternating rounds of CUDA-event timed calls, the two sides interleaved. The GPU name, power
limit and SM clocks are read before and after the run.

  python tools/bench_gblock_tail.py [--rounds 5] [--calls 5] [--seq 128] [--batch 8]
"""
import argparse
import copy
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

import torch                                           # noqa: E402
from model import generator_lres as gl                 # noqa: E402
from torch_utils.ops import conv_nd, gblock_tail, modulated_conv   # noqa: E402


def gpu_facts():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def timed(sides, fn, rounds, calls):
    """median ms per call of fn() for each side (a callable that installs it), the sides alternating."""
    times = {s: [] for s in sides}
    for s, use in sides.items():
        use()
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for s, use in sides.items():
            use()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(calls):
                fn()
            e1.record()
            e1.synchronize()
            times[s].append(e0.elapsed_time(e1) / calls)
    return {s: statistics.median(v) for s, v in times.items()}, times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--calls', type=int, default=5)
    ap.add_argument('--seq', type=int, default=128)
    ap.add_argument('--batch', type=int, default=8)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_gblock_tail needs a CUDA device'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    conv_nd.install_functional(gl)
    modulated_conv.install(gl)
    orig = gl.Synthesis3dResBlock.forward
    gblock_tail.install(gl)
    patched = gl.Synthesis3dResBlock.forward
    gl.Synthesis3dResBlock.forward = orig

    def use(f):
        def go():
            gl.Synthesis3dResBlock.forward = f
        return go
    sides = {'reference': use(orig), 'gblock_tail': use(patched)}
    facts_before = gpu_facts()

    torch.manual_seed(0)
    G = gl.VideoGenerator(out_height=36, out_width=64).cuda()
    calls = []

    def spy(self, input, latent, magnitude_ema_beta=1.0, out_seq_length=None, dtype=None):
        calls.append((self, input.detach(), latent.detach(), out_seq_length))
        return orig(self, input, latent, magnitude_ema_beta, out_seq_length, dtype)
    gl.Synthesis3dResBlock.forward = spy
    with torch.no_grad():
        torch.manual_seed(1)
        G(a.batch, a.seq)
    gl.Synthesis3dResBlock.forward = orig

    rows = []
    for i, (blk, x, lat, osl) in enumerate(calls):
        xg = x.clone().requires_grad_(True)

        def fwd():
            with torch.no_grad():
                blk(x, lat, 1.0, osl)

        def fwd_bwd():
            y = blk(xg, lat, 1.0, osl)
            y.square().mean().backward()
            xg.grad = None
            for p in blk.parameters():
                p.grad = None
        with torch.no_grad():
            shape = tuple(blk(x, lat, 1.0, osl).shape)
        f, _ = timed(sides, fwd, a.rounds, a.calls)
        fb, _ = timed(sides, fwd_bwd, a.rounds, a.calls)
        rows.append(dict(block=i, cin=blk.in_channels, inp=tuple(x.shape), out=shape, fwd=f, fwd_bwd=fb))

    tgt = None

    def g_fwd():
        with torch.no_grad():
            torch.manual_seed(1)
            G(a.batch, a.seq)

    def g_fwd_bwd():
        nonlocal tgt
        torch.manual_seed(1)
        v = G(a.batch, a.seq)
        if tgt is None:
            tgt = torch.randn_like(v)
        (v * tgt).mean().backward()
        for p in G.parameters():
            p.grad = None
    gf, gf_runs = timed(sides, g_fwd, a.rounds, 2)
    gfb, gfb_runs = timed(sides, g_fwd_bwd, a.rounds, 1)
    peak = {}
    for s, u in sides.items():
        u()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        g_fwd_bwd()
        torch.cuda.synchronize()
        peak[s] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    gl.Synthesis3dResBlock.forward = orig
    facts_after = gpu_facts()

    print(f'GPU (name, power limit, SM clock, max SM clock): before {facts_before}; after {facts_after}')
    print(f'VideoGenerator 36x64, batch {a.batch}, {a.seq} frames, fp32; {a.rounds} alternating rounds')
    print('| block | input -> output | fwd ms ref -> installed | fwd+bwd ms ref -> installed |')
    print('|---|---|---|---|')
    for r in rows:
        print(f'| {r["block"]} | {list(r["inp"][1:])} -> {list(r["out"][1:])} | {r["fwd"]["reference"]:.3f} -> {r["fwd"]["gblock_tail"]:.3f} '
              f'| {r["fwd_bwd"]["reference"]:.3f} -> {r["fwd_bwd"]["gblock_tail"]:.3f} |')
    print(f'| whole G forward (no grad) | | {gf["reference"]:.2f} -> {gf["gblock_tail"]:.2f} | |')
    print(f'| whole G forward + backward | | | {gfb["reference"]:.2f} -> {gfb["gblock_tail"]:.2f} |')
    print(f'| peak MB, whole G forward + backward | | | {peak["reference"]:.0f} -> {peak["gblock_tail"]:.0f} |')
    print(json.dumps(dict(blocks=[dict(r, inp=list(r['inp']), out=list(r['out'])) for r in rows], g_fwd=gf, g_fwd_runs=gf_runs,
                          g_fwd_bwd=gfb, g_fwd_bwd_runs=gfb_runs, peak_mb=peak, gpu_before=facts_before, gpu_after=facts_after)))


if __name__ == '__main__':
    main()
