"""The first layer of every residual block of the default low-res VideoGenerator (36 x 64; staged at oracle/_ref/src by
build()) as one op (gblock_conv0) against the composition it replaces, TF32 off.

For each block, on the block's real input at --batch x --frames (fp32, as the generator computes it), the layer
  hidden = bias_act(temporal_modulated_conv3d(input, weight_0, style_0, input_gain_0), bias_0); input_gain_1 = EMA_1(hidden)
in the block's three calls: forward + backward at magnitude_ema_beta 1 (update_G: gradients of the input, the style and the
layer's parameters), forward at 0.999 with G's parameters frozen (update_D's generated pass), forward without gradient at 1
(inference). Sides: 'comp' (gblock_tail.head with modulated_conv installed: the engine's modulated convolution, bias_act,
MagnitudeEMA) and 'op' (gblock_conv0.head in the call's mode).

ms per call: median (min..max) over alternating rounds of CUDA-event timed calls, the sides interleaved. 'MB' is the HBM
traffic of the activation-sized passes outside the convolution's own operand reads, from the shapes (x the input, y the
output, each pass one tensor):
  forward      comp: write y', read y', write y                         op: write y
  statistic    comp: + read y, write y^2 (fp32), read y^2                op: (the squares are read back from L2)
  backward     comp: bias_act's gradient reads dy, y and writes dz; db reads dz; the d gradient reads dz, y'; dgrad's
               re-tiling reads dz (shared with dw)                       op: the row pass reads dy, y; the re-tiling reads
               dy, y
'peak_MB': max_memory_allocated above what was allocated before the call. The GPU name, power limit and SM clocks are read
before and after the run, in the same process.

  python tools/bench_gblock_conv0.py [--rounds 5] [--calls 3] [--batch 8] [--frames 128]
"""
import argparse
import copy
import functools
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
from torch_utils.ops import gblock_conv0, gblock_tail, modulated_conv         # noqa: E402

ORIG_BLOCK, ORIG_TMC = gl.Synthesis3dResBlock.forward, gl.temporal_modulated_conv3d


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
    ap.add_argument('--frames', type=int, default=128)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_gblock_conv0 needs a CUDA device'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device('cuda')
    facts = {'gpu_before': gpu_facts()}
    torch.manual_seed(0)
    G0 = gl.VideoGenerator(out_height=36, out_width=64).to(dev)
    gl.temporal_modulated_conv3d = modulated_conv.temporal_modulated_conv3d
    g = gl.__dict__

    # every block's real input, latent and dtype
    feats = []

    def grab(self, input, latent, *args, **kw):
        feats.append((self, input.detach(), latent.detach()))
        return ORIG_BLOCK(self, input, latent, *args, **kw)
    gl.Synthesis3dResBlock.forward = grab
    with torch.no_grad():
        G0(a.batch, a.frames)
    gl.Synthesis3dResBlock.forward = ORIG_BLOCK
    out = {'batch': a.batch, 'frames': a.frames, 'blocks': []}
    for i, (B0, x, lat) in enumerate(feats):
        B = copy.deepcopy(B0)
        Bf = copy.deepcopy(B0).requires_grad_(False)
        t = x.shape[2]
        with torch.no_grad():
            style = B.affine_0(lat.permute(0, 2, 1).reshape(-1, lat.shape[1])).reshape(x.shape[0], t, -1).permute(0, 2, 1).contiguous()
        gain0 = B.input_magnitude_ema_0.magnitude_ema.rsqrt()
        xg, sg = x.clone().requires_grad_(True), style.clone().requires_grad_(True)
        dy = torch.randn(x.shape, device=dev)
        heads = {'comp': {m: gblock_tail.head for m in ('backward', 'stat', 'forward')},
                 'op': {m: functools.partial(gblock_conv0.head, mode=m) for m in ('backward', 'stat', 'forward')}}

        def train(h):
            y, _ = h['backward'](B, g, xg, sg, gain0, 1.0)
            y.backward(dy)

        def gen(h):
            Bf.input_magnitude_ema_1.magnitude_ema.fill_(1.0)
            h['stat'](Bf, g, x, style, gain0, 0.999)

        def infer(h):
            with torch.no_grad():
                h['forward'](B, g, x, style, gain0, 1.0)

        ny, nx = x.numel() * x.element_size(), x.numel() * x.element_size()
        traffic = {'update_G fwd+bwd': (3 * ny + 3 * ny + ny + 2 * ny + ny, ny + 2 * ny + 2 * ny),
                   'update_D gen fwd (beta 0.999)': (3 * ny + 3 * ny, ny),
                   'inference fwd': (3 * ny, ny)}
        row = {'block': i, 'shape': list(x.shape), 'kernel': list(B.weight_0.shape[2:]), 'modes': {}}
        for mode, fn in (('update_G fwd+bwd', train), ('update_D gen fwd (beta 0.999)', gen), ('inference fwd', infer)):
            sides = {s: functools.partial(fn, heads[s]) for s in ('comp', 'op')}
            tm = timed(sides, a.rounds, a.calls)
            r = {s: fmt(v) for s, v in tm.items()}
            r['MB'] = {'comp': round(traffic[mode][0] / 1e6), 'op': round(traffic[mode][1] / 1e6)}
            if mode.startswith('update_G'):
                r['peak_MB'] = {s: round(peak_mb(f), 1) for s, f in sides.items()}
            row['modes'][mode] = r
            print(i, mode, json.dumps(r), flush=True)
        out['blocks'].append(row)
        xg.grad = sg.grad = None
        for p in B.parameters():
            p.grad = None
    gl.temporal_modulated_conv3d = ORIG_TMC
    facts['gpu_after'] = gpu_facts()
    out['gpu'] = facts
    print(json.dumps(out))


if __name__ == '__main__':
    main()
