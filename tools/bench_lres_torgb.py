"""The low-res generator's ToRGB layer as one op (lres_torgb) against the reference's ToRGB.forward, with and without
modulated_conv.install, in the default VideoGenerator (36 x 64; staged at oracle/_ref/src by build()), TF32 off.

  layer    on the layer's real input ([N, 64, T, 36, 64] fp32 from the generator), in its three calls: forward + backward
           at magnitude_ema_beta 1 (update_G: gradients of the input and the layer's parameters), forward at 0.999 with
           G's parameters frozen (update_D's generated pass), forward without gradient at 1 (inference). Sides: 'ref'
           (the model's method), 'modconv' (the same with modulated_conv installed), 'op' (lres_torgb.layer_forward, on
           every call). Algorithmic GB/s from the bytes the op must move (x and y forward, plus u written and read in the
           0.999 pass; x, y, dy and dx backward)
  whole G  modulated_conv + gblock_tail installed ('base') against the same + lres_torgb ('op'): the same three calls of
           the whole generator; peak max_memory_allocated above what was allocated before each call

ms per call: median (min..max) over alternating rounds of CUDA-event timed calls, the sides interleaved. The GPU name,
power limit and SM clocks are read before and after the run, in the same process.

  python tools/bench_lres_torgb.py [--rounds 5] [--calls 3] [--batch 8] [--frames 160]
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
from model import generator_lres as gl                                         # noqa: E402
from torch_utils.ops import gblock_tail, lres_torgb, modulated_conv           # noqa: E402

ORIG, ORIG_BLOCK, ORIG_TMC = gl.ToRGB.forward, gl.Synthesis3dResBlock.forward, gl.temporal_modulated_conv3d


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


def reset():
    gl.ToRGB.forward, gl.Synthesis3dResBlock.forward, gl.temporal_modulated_conv3d = ORIG, ORIG_BLOCK, ORIG_TMC


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--calls', type=int, default=3)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--frames', type=int, default=160)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_lres_torgb needs a CUDA device'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device('cuda')
    facts = {'gpu_before': gpu_facts()}
    torch.manual_seed(0)
    G0 = gl.VideoGenerator(out_height=36, out_width=64).to(dev)

    # the layer's real input and latent
    feats = {}

    def grab(self, input, latent, *args, **kw):
        feats['in'] = (input.detach(), latent.detach())
        return ORIG(self, input, latent, *args, **kw)
    gl.ToRGB.forward = grab
    with torch.no_grad():
        G0(a.batch, a.frames)
    reset()
    x, lat = feats.pop('in')
    L = copy.deepcopy(G0.to_rgb)
    Lf = copy.deepcopy(L).requires_grad_(False)
    dy = torch.randn([x.shape[0], 3, *x.shape[2:]], device=dev)
    xg = x.clone().requires_grad_(True)
    es, ys = x.element_size(), 4
    nb = x.numel() * es
    ny = dy.numel() * ys
    out = {'shape': list(x.shape), 'layer': {}, 'whole_G': {}}

    def side(name):
        def run(fn):
            def call():
                reset()
                if name == 'modconv':
                    modulated_conv.install(gl)
                return fn()
            return call
        return run

    def op_train():
        y = lres_torgb.layer_forward(L, gl.__dict__, xg, lat, 1.0)
        y.backward(dy)

    def ref_train():
        y = L(xg, lat, 1.0)
        y.backward(dy)

    def op_gen():
        return lres_torgb.layer_forward(Lf, gl.__dict__, x, lat, 0.999)

    def ref_gen():
        return Lf(x, lat, 0.999)

    def op_infer():
        with torch.no_grad():
            return lres_torgb.layer_forward(L, gl.__dict__, x, lat, 1.0)

    def ref_infer():
        with torch.no_grad():
            return L(x, lat, 1.0)

    modes = {'update_G fwd+bwd (beta 1)': (ref_train, op_train, nb + ny + nb + ny + ny + nb),
             'update_D gen fwd (beta 0.999)': (ref_gen, op_gen, nb + 4 * dy.numel() * 2 + ny),
             'inference fwd (beta 1)': (ref_infer, op_infer, nb + ny)}
    for mode, (ref_fn, op_fn, nbytes) in modes.items():
        sides = {'ref': side('ref')(ref_fn), 'modconv': side('modconv')(ref_fn), 'op': side('op')(op_fn)}
        t = timed(sides, a.rounds, a.calls)
        out['layer'][mode] = {s: fmt(v) for s, v in t.items()}
        out['layer'][mode]['op_GB/s'] = round(nbytes / (t['op'][0] * 1e-3) / 1e9, 1)
        out['layer'][mode]['peak_MB'] = {s: round(peak_mb(fn), 1) for s, fn in sides.items()}
        print(mode, json.dumps(out['layer'][mode]), flush=True)
    reset()

    # whole G
    def installed(ours):
        reset()
        modulated_conv.install(gl)
        gblock_tail.install(gl)
        if ours:
            lres_torgb.install(gl)

    G = copy.deepcopy(G0)
    Gf = copy.deepcopy(G0).requires_grad_(False)

    def g_train():
        G(a.batch, a.frames).square().mean().backward()
        for p in G.parameters():
            p.grad = None

    def g_gen():
        Gf(a.batch, a.frames, magnitude_ema_beta=0.999)

    def g_infer():
        with torch.no_grad():
            G(a.batch, a.frames)

    for mode, fn in (('update_G fwd+bwd', g_train), ('update_D gen fwd', g_gen), ('inference fwd', g_infer)):
        def with_install(ours, fn=fn):
            def call():
                installed(ours)
                fn()
            return call
        sides = {'base': with_install(False), 'op': with_install(True)}
        t = timed(sides, a.rounds, 1)
        out['whole_G'][mode] = {s: fmt(v) for s, v in t.items()}
        out['whole_G'][mode]['peak_MB'] = {s: round(peak_mb(f), 1) for s, f in sides.items()}
        print('whole G', mode, json.dumps(out['whole_G'][mode]), flush=True)
    reset()
    facts['gpu_after'] = gpu_facts()
    out['gpu'] = facts
    print(json.dumps(out))


if __name__ == '__main__':
    main()
