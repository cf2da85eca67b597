"""The super-res generator's layers with the input built inside the modulated convolution's re-tiling pass (sres_layer)
against the two-op composition (sres_cond's cond_concat, then modulated_conv), in the default VideoGenerator (hr 144 x 256,
lr 36 x 64, temporal_context 4; staged at oracle/_ref/src by build()) at batch 8 x 8 frames (N T = 64), TF32 off.

  whole G     modulated_conv + sres_cond installed ('composition') against modulated_conv + sres_cond + sres_layer
              ('sres_layer'): forward without gradient at magnitude_ema_beta 0.999 (update_D's generated pass), forward +
              backward (update_G), and the chained-inference forward (SG3 under no_grad, eval, no EMA update)
  per layer   sres_cond.conv_step against sres_layer.fused_step (the layer from its x_prev to the modulated convolution's
              output, styles and factors included; the op on every call, without install's routing) on the layer's real
              x_prev: forward without gradient, and forward + backward (gradients of x_prev and the layer's parameters)
  memory      peak max_memory_allocated of each whole-G mode above what was allocated before it

ms per call: median (min..max) over alternating rounds of CUDA-event timed calls, the two sides interleaved. The GPU name,
power limit and SM clocks are read before and after the run, in the same process.

  python tools/bench_sres_layer.py [--rounds 5] [--calls 3]
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

import torch                                                       # noqa: E402
from model import generator_sres as gs                             # noqa: E402
from torch_utils.ops import modulated_conv, sres_cond, sres_layer  # noqa: E402


def gpu_facts():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def timed(sides, rounds, calls):
    """(median, min, max) ms per call of each side's callable, the sides alternating."""
    times = {s: [] for s in sides}
    for fn in sides.values():
        for _ in range(2):
            fn()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for s, fn in sides.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(calls):
                fn()
            e1.record()
            e1.synchronize()
            times[s].append(e0.elapsed_time(e1) / calls)
    return {s: (statistics.median(v), min(v), max(v)) for s, v in times.items()}


def fmt(t):
    return f'{t[0]:.3f} ({t[1]:.3f}..{t[2]:.3f})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--calls', type=int, default=3)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--frames', type=int, default=8)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_sres_layer needs a CUDA device'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    modulated_conv.install(gs)
    orig = gs.Generator.forward
    sres_cond.install(gs)
    composition = gs.Generator.forward
    sres_layer.install(gs)
    fused = gs.Generator.forward
    gs.Generator.forward = orig
    facts_before = gpu_facts()
    dev = torch.device('cuda')

    torch.manual_seed(0)
    V = gs.VideoGenerator(hr_height=144, hr_width=256, lr_height=36, lr_width=64, temporal_context=4).to(dev)
    G = V.SG3
    g = torch.Generator().manual_seed(1)
    lr = torch.randn(a.batch, 3, a.frames + 2 * V.temporal_context, 36, 64, generator=g).to(dev)
    z = torch.randn(a.batch, V.latent_z_dim, generator=g).to(dev)

    # ------------------------------------------------------------------ whole G
    Vi = copy.deepcopy(V).eval().requires_grad_(False)
    tgt = None

    def fwd_emas():
        with torch.no_grad():
            V(lr, magnitude_ema_beta=0.999)

    def fwd_bwd():
        nonlocal tgt
        v = V.SG3(z, lr)
        if tgt is None:
            tgt = torch.randn_like(v)
        (v * tgt).mean().backward()
        for p in V.parameters():
            p.grad = None

    def chained():
        with torch.no_grad():
            Vi.SG3(z, lr)

    def on(f, fn):
        def go():
            gs.Generator.forward = f
            fn()
        return go
    modes = {'forward, no grad, beta 0.999': fwd_emas, 'forward + backward': fwd_bwd, 'chained-inference forward': chained}
    whole, peak = {}, {}
    for name, fn in modes.items():
        whole[name] = timed({'composition': on(composition, fn), 'sres_layer': on(fused, fn)}, a.rounds, a.calls)
        peak[name] = {}
        for s, f in (('composition', composition), ('sres_layer', fused)):
            gs.Generator.forward = f
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fn()
            torch.cuda.synchronize()
            peak[name][s] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    gs.Generator.forward = orig

    # ------------------------------------------------------------------ per layer
    S = G.synthesis
    glb = vars(gs)
    plans = sres_cond.plans(G, 36, 64)
    prev = {}
    with torch.no_grad():
        ws = G.mapping(z.repeat_interleave(a.frames, 0), c=None).unbind(1)
        x = None
        for name, w, plan in zip(S.layer_names, ws, plans):
            prev[name] = x
            x = sres_cond.layer_forward(getattr(S, name), glb, x, lr, plan, w)
    rows = []
    for i, (name, w, plan) in enumerate(zip(S.layer_names, ws, plans)):
        L = getattr(S, name)
        dtype = torch.float16 if L.use_fp16 else torch.float32
        xp = prev[name]
        xg = None if xp is None else xp.detach().clone().requires_grad_(True)
        dy = {}

        def fwd(step):
            def go():
                with torch.no_grad():
                    step(L, glb, xp, lr, plan, w, dtype, False)
            return go

        def bwd(step):
            def go():
                y = step(L, glb, xg, lr, plan, w, dtype, False)
                if 'dy' not in dy:
                    dy['dy'] = torch.randn_like(y)
                y.backward(dy['dy'])
                for p in L.parameters():
                    p.grad = None
                if xg is not None:
                    xg.grad = None
            return go
        t_f = timed({'composition': fwd(sres_cond.conv_step), 'sres_layer': fwd(sres_layer.fused_step)}, a.rounds, 10)
        t_b = timed({'composition': bwd(sres_cond.conv_step), 'sres_layer': bwd(sres_layer.fused_step)}, a.rounds, 5)
        rows.append(dict(layer=i, c=0 if xp is None else xp.shape[1], x_dtype=None if xp is None else str(xp.dtype).split('.')[-1],
                         dtype=str(dtype).split('.')[-1], h=int(L.in_size[1]), w=int(L.in_size[0]), cout=int(L.out_channels),
                         k=int(L.conv_kernel), fwd=t_f, fwd_bwd=t_b))
    facts_after = gpu_facts()

    print(f'GPU (name, power limit, SM clock, max SM clock): before {facts_before}; after {facts_after}')
    print(f'VideoGenerator hr 144x256, lr 36x64, batch {a.batch} x {a.frames} frames; {a.rounds} alternating rounds; '
          f'ms median (min..max)')
    print('| whole G | composition | sres_layer | peak MB composition -> sres_layer |')
    print('|---|---|---|---|')
    for name in modes:
        print(f'| {name} | {fmt(whole[name]["composition"])} | {fmt(whole[name]["sres_layer"])} | '
              f'{peak[name]["composition"]:.0f} -> {peak[name]["sres_layer"]:.0f} |')
    print('| layer | x_prev -> z, conv | fwd composition | fwd sres_layer | fwd+bwd composition | fwd+bwd sres_layer |')
    print('|---|---|---|---|---|---|')
    for r in rows:
        print(f'| {r["layer"]} | {r["c"]} {r["x_dtype"]} -> {r["c"] + 27} {r["dtype"]}, {r["h"]}x{r["w"]}, {r["k"]}x{r["k"]} -> '
              f'{r["cout"]} | {fmt(r["fwd"]["composition"])} | {fmt(r["fwd"]["sres_layer"])} | '
              f'{fmt(r["fwd_bwd"]["composition"])} | {fmt(r["fwd_bwd"]["sres_layer"])} |')
    print(json.dumps(dict(whole=whole, peak_mb=peak, layers=rows, gpu_before=facts_before, gpu_after=facts_after)))


if __name__ == '__main__':
    main()
