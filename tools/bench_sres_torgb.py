"""The super-res generator's ToRGB layer as one op (sres_torgb) against the composition it replaces (sres_cond's
cond_concat, modulated_conv on the engine, filtered_lrelu's bias and clamp), in the default VideoGenerator (hr 144 x 256,
lr 36 x 64, temporal_context 4; staged at oracle/_ref/src by build()) at batch 8 x 8 frames (N T = 64), TF32 off.

  layer 14    sres_cond.layer_forward (conv_step + filtered_lrelu) against sres_torgb.fused_forward (the op on every call,
              without install's routing) on the layer's real
              x_prev: forward without gradient, forward with update_emas, forward + backward (gradients of x_prev and the
              layer's parameters) without and with update_emas; algorithmic GB/s from the bytes the op must move (x_prev and y forward; x_prev, dy and
              dx_prev backward)
  whole G     modulated_conv + sres_cond installed ('composition') against the same + sres_torgb: forward without gradient
              at magnitude_ema_beta 0.999, forward + backward, and the chained-inference forward, without and with
              sres_layer installed on both sides; peak max_memory_allocated above what was allocated before each mode

ms per call: median (min..max) over alternating rounds of CUDA-event timed calls, the two sides interleaved. The GPU name,
power limit and SM clocks are read before and after the run, in the same process.

  python tools/bench_sres_torgb.py [--rounds 5] [--calls 3]
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

import torch                                                                   # noqa: E402
from model import generator_sres as gs                                         # noqa: E402
from torch_utils.ops import modulated_conv, sres_cond, sres_layer, sres_torgb  # noqa: E402


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


def peak_mb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def fmt(t):
    return f'{t[0]:.3f} ({t[1]:.3f}..{t[2]:.3f})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--calls', type=int, default=3)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--frames', type=int, default=8)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_sres_torgb needs a CUDA device'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    modulated_conv.install(gs)
    orig = gs.Generator.forward
    sres_cond.install(gs)
    composition = gs.Generator.forward
    sres_torgb.install(gs)
    ours = gs.Generator.forward
    gs.Generator.forward = orig
    facts_before = gpu_facts()
    dev = torch.device('cuda')

    torch.manual_seed(0)
    V = gs.VideoGenerator(hr_height=144, hr_width=256, lr_height=36, lr_width=64, temporal_context=4).to(dev)
    G = V.SG3
    g = torch.Generator().manual_seed(1)
    lr = torch.randn(a.batch, 3, a.frames + 2 * V.temporal_context, 36, 64, generator=g).to(dev)
    z = torch.randn(a.batch, V.latent_z_dim, generator=g).to(dev)

    # ------------------------------------------------------------------ layer 14 on its real x_prev
    S = G.synthesis
    glb = vars(gs)
    plans = sres_cond.plans(G, 36, 64)
    with torch.no_grad():
        ws = G.mapping(z.repeat_interleave(a.frames, 0), c=None).unbind(1)
        x = None
        for name, w, plan in list(zip(S.layer_names, ws, plans))[:-1]:
            x = sres_cond.layer_forward(getattr(S, name), glb, x, lr, plan, w)
    name, w, plan = S.layer_names[-1], ws[-1], plans[-1]
    L = getattr(S, name)
    xp = x
    xg = xp.detach().clone().requires_grad_(True)
    dy = {}

    def fwd(f, emas):
        def go():
            with torch.no_grad():
                f(L, glb, xp, lr, plan, w, update_emas=emas)
        return go

    def bwd(f, emas=False):
        def go():
            y = f(L, glb, xg, lr, plan, w, update_emas=emas)
            if 'dy' not in dy:
                dy['dy'] = torch.randn_like(y)
            y.backward(dy['dy'])
            for p in L.parameters():
                p.grad = None
            xg.grad = None
        return go
    comp_f, op_f = sres_cond.layer_forward, sres_torgb.fused_forward
    layer = {'forward, no grad': timed({'composition': fwd(comp_f, False), 'sres_torgb': fwd(op_f, False)}, a.rounds, 10),
             'forward, update_emas': timed({'composition': fwd(comp_f, True), 'sres_torgb': fwd(op_f, True)}, a.rounds, 10),
             'forward + backward': timed({'composition': bwd(comp_f), 'sres_torgb': bwd(op_f)}, a.rounds, 5),
             'forward + backward, update_emas': timed({'composition': bwd(comp_f, True), 'sres_torgb': bwd(op_f, True)},
                                                      a.rounds, 5)}
    layer_peak = {k: {s: peak_mb(fn) for s, fn in sides.items()} for k, sides in
                  (('forward, no grad', {'composition': fwd(comp_f, False), 'sres_torgb': fwd(op_f, False)}),
                   ('forward + backward', {'composition': bwd(comp_f), 'sres_torgb': bwd(op_f)}))}
    es = xp.element_size()
    y_bytes = xp.shape[0] * 3 * xp.shape[2] * xp.shape[3] * (2 if L.use_fp16 else 4)
    gbytes = {'forward, no grad': (xp.numel() * es + y_bytes) / 1e9,
              'forward, update_emas': (2 * xp.numel() * es + y_bytes) / 1e9,            # the statistic pass reads x_prev too
              'forward + backward': (3 * xp.numel() * es + 2 * y_bytes) / 1e9,       # x_prev twice, dx_prev, y, dy
              'forward + backward, update_emas': (4 * xp.numel() * es + 2 * y_bytes) / 1e9}

    # ------------------------------------------------------------------ whole G
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

    Vi = copy.deepcopy(V).eval().requires_grad_(False)

    def chained():
        with torch.no_grad():
            Vi.SG3(z, lr)

    def on(f, fn):
        def go():
            gs.Generator.forward = f
            fn()
        return go
    modes = {'forward, no grad, beta 0.999': (fwd_emas, composition, ours), 'forward + backward': (fwd_bwd, composition, ours),
             'chained-inference forward': (chained, composition, ours)}
    gs.Generator.forward = ours
    sres_layer.install(gs)                                   # on top: chained inference with sres_layer on both sides
    ours_layer = gs.Generator.forward
    gs.Generator.forward = composition
    sres_layer.install(gs)
    comp_layer = gs.Generator.forward
    modes['chained-inference forward (+ sres_layer)'] = (chained, comp_layer, ours_layer)
    whole, peak = {}, {}
    for mname, (fn, fc, fo) in modes.items():
        whole[mname] = timed({'composition': on(fc, fn), 'sres_torgb': on(fo, fn)}, a.rounds, a.calls)
        peak[mname] = {}
        for s, f in (('composition', fc), ('sres_torgb', fo)):
            gs.Generator.forward = f
            peak[mname][s] = peak_mb(fn)
    gs.Generator.forward = orig
    facts_after = gpu_facts()

    print(f'GPU (name, power limit, SM clock, max SM clock): before {facts_before}; after {facts_after}')
    print(f'VideoGenerator hr 144x256, lr 36x64, batch {a.batch} x {a.frames} frames; {a.rounds} alternating rounds; '
          f'ms median (min..max)')
    print(f'| layer {len(S.layer_names) - 1}: {xp.shape[1]} {str(xp.dtype).split(".")[-1]} -> 3 | composition | sres_torgb | '
          f'sres_torgb GB/s | peak MB composition -> sres_torgb |')
    print('|---|---|---|---|---|')
    for k, t in layer.items():
        pk = layer_peak.get(k)
        print(f'| {k} | {fmt(t["composition"])} | {fmt(t["sres_torgb"])} | {gbytes[k] / (t["sres_torgb"][0] / 1e3):.0f} | '
              + (f'{pk["composition"]:.0f} -> {pk["sres_torgb"]:.0f} |' if pk else '|'))
    print('| whole G | composition | sres_torgb | peak MB composition -> sres_torgb |')
    print('|---|---|---|---|')
    for mname in modes:
        print(f'| {mname} | {fmt(whole[mname]["composition"])} | {fmt(whole[mname]["sres_torgb"])} | '
              f'{peak[mname]["composition"]:.0f} -> {peak[mname]["sres_torgb"]:.0f} |')
    print(json.dumps(dict(layer=layer, layer_peak_mb=layer_peak, layer_gbytes=gbytes, whole=whole, peak_mb=peak,
                          gpu_before=facts_before, gpu_after=facts_after)))


if __name__ == '__main__':
    main()
