"""Times the downsampling Conv3dLayers of the low-res discriminator (batch 8, T = 128, 64 x 64, fp32, as in the training
step) two ways: today's path (conv_nd.conv3d -> Downsample3d -> bias_act) and conv3d_down (FIR of the input, convolution at
the output resolution, border faces). Per layer: forward, forward + backward, and the double backward of the R1 penalty;
the paths alternate and every figure is the median over --rounds rounds. Then the whole reference discriminator (staged at
oracle/_ref/src) forward + backward and R1 step with and without conv3d_down.install, with peak memory. Prints the card
and its power limit read in the same run, one JSON line per measurement, and a markdown table.

    python tools/bench_dconv.py [--rounds 5] [--iters 5] [--out <markdown file for the table>]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
for p in (SRC, PKG):                                # this package's torch_utils.ops ahead of the reference's
    if p not in sys.path:
        sys.path.insert(0, p)
sys.modules.setdefault('imageio', types.ModuleType('imageio'))

import torch                                        # noqa: E402

from torch_utils.ops import bias_act, conv3d_down as cd     # noqa: E402

LAYERS = [   # (name, Cin, Cout, kt, ks, T, H, W, temporal_down), spatial_down everywhere, batch 8
    ('b0 conv_skip', 32, 64, 1, 1, 128, 64, 64, False),
    ('b0 conv_1', 32, 64, 1, 3, 128, 64, 64, False),
    ('b1 conv_skip', 64, 128, 1, 1, 128, 32, 32, True),
    ('b1 conv_1', 64, 128, 5, 3, 128, 32, 32, True),
    ('b2 conv_skip', 128, 256, 1, 1, 64, 16, 16, True),
    ('b2 conv_1', 128, 256, 5, 3, 64, 16, 16, True),
    ('b3 conv_skip', 256, 512, 1, 1, 32, 8, 8, True),
    ('b3 conv_1', 256, 512, 5, 3, 32, 8, 8, True),
]


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def timed(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def layer_fns(path, layer):
    name, cin, cout, kt, ks, t, h, w, td = layer
    g = torch.Generator(device='cuda').manual_seed(0)
    x = torch.randn(8, cin, t, h, w, device='cuda', generator=g).requires_grad_(True)
    wt = (torch.randn(cout, cin, kt, ks, ks, device='cuda', generator=g) / (cin * kt * ks * ks) ** 0.5).requires_grad_(True)
    b = torch.zeros(cout, device='cuda').requires_grad_(ks > 1)
    f = torch.tensor([1., 3., 3., 1.], device='cuda') / 8
    pad = (kt // 2, ks // 2, ks // 2)
    act = 'lrelu' if ks > 1 else 'linear'
    bb = b if ks > 1 else None

    def fwd():
        if path == 'new':
            return cd.conv3d_down(x, wt, bb, pad, True, td, f, act=act, clamp=256)
        return bias_act.bias_act(cd._reference(x, wt, f, True, td, pad), bb, act=act, clamp=256)

    params = [x, wt] + ([b] if ks > 1 else [])

    def fwd_bwd():
        z = fwd()
        torch.autograd.grad(z, params, torch.ones_like(z))

    def double_bwd():
        z = fwd()
        gx, = torch.autograd.grad(z.square().sum(), [x], create_graph=True)
        torch.autograd.grad(gx.square().sum(), params)

    return {'fwd': lambda: fwd(), 'fwd+bwd': fwd_bwd, 'double bwd': double_bwd}


def whole_d(install, rounds, iters):
    from model import discriminator_lres
    from torch_utils.ops import conv_nd
    conv_nd.install_functional(discriminator_lres)
    cls = discriminator_lres.Conv3dLayer
    orig = getattr(cls.forward, 'lvg_conv3d_down', None) or cls.forward
    if install:
        cd.install(discriminator_lres)
    else:
        cls.forward = orig
    torch.manual_seed(0)
    D = discriminator_lres.VideoDiscriminator(seq_length=128, max_edge=64).cuda()
    x = torch.randn(8, 3, 128, 64, 64, device='cuda').requires_grad_(True)

    def step():
        D(x).sum().backward()

    def r1():
        logits = D(x)
        gx, = torch.autograd.grad(logits.sum(), [x], create_graph=True)
        gx.square().sum().backward()

    res = {}
    for what, fn in (('D fwd+bwd', step), ('D R1 step', r1)):
        fn()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ts = [timed(fn, iters) for _ in range(rounds)]
        res[what] = (statistics.median(ts), torch.cuda.max_memory_allocated() / 2 ** 30)
    cls.forward = orig
    del D, x
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--out', default=None)
    ap.add_argument('--no-whole', action='store_true')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_dconv measures on a CUDA device'
    dev = card()
    print(json.dumps({'card': dev}), flush=True)
    rows = []
    for layer in LAYERS:
        fns = {p: layer_fns(p, layer) for p in ('today', 'new')}
        times = {(p, k): [] for p in fns for k in fns[p]}
        for k in fns['today']:
            for p in fns:
                fns[p][k]()                       # warm-up
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for k in fns['today']:
                for p in ('today', 'new'):        # alternating
                    times[(p, k)].append(timed(fns[p][k], a.iters))
        med = {key: statistics.median(v) for key, v in times.items()}
        rec = {'layer': layer[0], **{f'{p} {k} ms': round(v, 3) for (p, k), v in med.items()}}
        print(json.dumps(rec), flush=True)
        rows.append((layer[0], med))
        del fns
        torch.cuda.empty_cache()
    whole = {}
    if not a.no_whole and os.path.isdir(os.path.join(SRC, 'model')):
        for inst in (False, True, False, True):   # alternating
            for k, (ms, gib) in whole_d(inst, a.rounds, 2).items():
                whole.setdefault((k, inst), []).append((ms, gib))
        for (k, inst), v in sorted(whole.items()):
            print(json.dumps({'what': k, 'install': inst, 'ms': [round(m, 2) for m, _ in v], 'peak GiB': round(max(g for _, g in v), 2)}), flush=True)
    lines = [f'Card: {dev} (name, power limit, max SM clock; read in the same run). Batch 8, fp32, median of {a.rounds} rounds '
             f'x {a.iters} calls, paths alternating. ms today -> conv3d_down.', '',
             '| layer | fwd | fwd+bwd | double bwd |', '|---|---|---|---|']
    for name, med in rows:
        cells = [f"{med[('today', k)]:.2f} → {med[('new', k)]:.2f}" for k in ('fwd', 'fwd+bwd', 'double bwd')]
        lines.append(f'| {name} | ' + ' | '.join(cells) + ' |')
    if whole:
        lines += ['', '| whole D (batch 8, T 128, 64×64) | without install ms (peak GiB) | with install ms (peak GiB) |', '|---|---|---|']
        for k in ('D fwd+bwd', 'D R1 step'):
            cell = lambda inst: f"{statistics.median(m for m, _ in whole[(k, inst)]):.1f} ({max(g for _, g in whole[(k, inst)]):.1f})"  # noqa: E731
            lines.append(f'| {k} | {cell(False)} | {cell(True)} |')
    text = '\n'.join(lines)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as fh:
            fh.write(text + '\n')


if __name__ == '__main__':
    main()
