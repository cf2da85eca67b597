"""The super-res generator's layer inputs: the reference Generator.forward (prep_cond, torch.cat, .to, square().mean(); staged
at oracle/_ref/src by build()) against the same method with sres_cond.install, in the default VideoGenerator (hr 144 x 256,
lr 36 x 64, temporal_context 4) at batch 8 x 8 frames (N T = 64), both sides with modulated_conv.install, TF32 off.

  whole G     forward without gradient at magnitude_ema_beta 0.999 (update_D's generated pass), forward + backward
              (update_G), and the chained-inference forward (SG3 under no_grad, eval, no EMA update)
  per layer   cond_concat against the reference's share of the layer input: the layer's resampler call, crop and pad
              of prep_cond, torch.cat, .to(dtype) and (with the statistic) .float().square().mean()
  memory      peak max_memory_allocated of each whole-G mode above what was allocated before it

ms per call: median (min..max) over alternating rounds of CUDA-event timed calls, the two sides interleaved. Bytes are
algorithmic (from the shapes: x_prev read, z written, the low-res frames read once). The GPU name, power limit and SM
clocks are read before and after the run.

  python tools/bench_sres_cond.py [--rounds 5] [--calls 3]
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
from model import generator_sres as gs                 # noqa: E402
from torch_utils.ops import modulated_conv, sres_cond  # noqa: E402


def gpu_facts():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def timed(sides, fn, rounds, calls):
    """(median, min, max) ms per call of fn() for each side (a callable that installs it), the sides alternating."""
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
    assert torch.cuda.is_available(), 'bench_sres_cond needs a CUDA device'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    modulated_conv.install(gs)
    orig = gs.Generator.forward
    sres_cond.install(gs)
    patched = gs.Generator.forward
    gs.Generator.forward = orig

    def use(f):
        def go():
            gs.Generator.forward = f
        return go
    sides = {'reference': use(orig), 'sres_cond': use(patched)}
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
    modes = {'forward, no grad, beta 0.999': fwd_emas, 'forward + backward': fwd_bwd, 'chained-inference forward': chained}
    whole, peak = {}, {}
    for name, fn in modes.items():
        whole[name] = timed(sides, fn, a.rounds, a.calls)
        peak[name] = {}
        for s, u in sides.items():
            u()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fn()
            torch.cuda.synchronize()
            peak[name][s] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    gs.Generator.forward = orig

    # ------------------------------------------------------------------ per layer
    S = G.synthesis
    prev = {}                                                   # each layer's x_prev, as the reference feeds it
    with torch.no_grad():
        conds = G.prep_cond(lr)
        ws = G.mapping(z.repeat_interleave(a.frames, 0), c=None)
        x = None
        for name, w, cond in zip(S.layer_names, ws.unbind(1), conds):
            prev[name] = x
            inp = cond if x is None else torch.cat((x, cond), 1)
            x = getattr(S, name)(inp, w)
    del conds
    plans = sres_cond.plans(G, 36, 64)
    n_t = a.batch * a.frames
    lr_bytes = lr.numel() * 4
    rows = []

    def ref_unfold():
        # prep_cond's shared replicate pad and unfold, restated
        m = max(G.cond_width, G.cond_height)
        px0 = (m - lr.size(4)) // 2 + G.margin_size
        px1 = (m - lr.size(4) + 1) // 2 + G.margin_size
        py0 = (m - lr.size(3)) // 2 + G.margin_size
        py1 = (m - lr.size(3) + 1) // 2 + G.margin_size
        cnd = torch.nn.functional.pad(lr, (px0, px1, py0, py1, 0, 0), mode='replicate')
        cnd = cnd.unfold(dimension=2, size=(1 + 2 * G.cond_context), step=1)
        return cnd.permute(0, 2, 1, 5, 3, 4).reshape(n_t, 3 * (1 + 2 * G.cond_context), cnd.shape[3], cnd.shape[4])
    with torch.no_grad():
        unf = ref_unfold()
    with torch.no_grad():
        t_unfold = timed({'reference': lambda: None}, ref_unfold, a.rounds, a.calls)['reference']
    for i, (name, r, plan) in enumerate(zip(S.layer_names, G.resamples, plans)):
        L = getattr(S, name)
        dtype = torch.float16 if L.use_fp16 else torch.float32
        xp = prev[name]
        in_w, in_h = (int(v) for v in L.in_size)

        def ref_layer(stat):
            lc = r(unf)
            x0 = max(0, (lc.size(3) - in_w) // 2)
            y0 = max(0, (lc.size(2) - in_h) // 2)
            lc = lc[:, :, y0:y0 + in_h, x0:x0 + in_w]
            px0, px1 = (in_w - lc.size(3)) // 2, (in_w - lc.size(3) + 1) // 2
            py0, py1 = (in_h - lc.size(2)) // 2, (in_h - lc.size(2) + 1) // 2
            lc = torch.nn.functional.pad(lc, (px0, px1, py0, py1), mode='replicate')
            cat = lc if xp is None else torch.cat((xp, lc), 1)
            if stat:
                cat.detach().to(torch.float32).square().mean()
            return cat.to(dtype)

        def op(stat):
            return sres_cond.cond_concat(xp, lr, plan, dtype, stat)
        res = {}
        for stat in (False, True):
            with torch.no_grad():
                t_ref = timed({'reference': lambda: None}, lambda: ref_layer(stat), a.rounds, 10)['reference']
                t_op = timed({'sres_cond': lambda: None}, lambda: op(stat), a.rounds, 10)['sres_cond']
            res[stat] = (t_ref, t_op)
        c = 0 if xp is None else xp.shape[1]
        hw = in_h * in_w
        nbytes = (0 if xp is None else xp.numel() * xp.element_size()) + n_t * (c + 27) * hw * (2 if dtype == torch.float16 else 4) + lr_bytes
        rows.append(dict(layer=i, kind=type(r).__name__, c=c, h=in_h, w=in_w, dtype=str(dtype).split('.')[-1],
                         x_dtype=None if xp is None else str(xp.dtype).split('.')[-1], bytes=nbytes,
                         ref=res[False][0], op=res[False][1], ref_stat=res[True][0], op_stat=res[True][1]))
    facts_after = gpu_facts()

    print(f'GPU (name, power limit, SM clock, max SM clock): before {facts_before}; after {facts_after}')
    print(f'VideoGenerator hr 144x256, lr 36x64, batch {a.batch} x {a.frames} frames; {a.rounds} alternating rounds; '
          f'ms median (min..max)')
    print('| whole G | reference | sres_cond | peak MB reference -> sres_cond |')
    print('|---|---|---|---|')
    for name in modes:
        print(f'| {name} | {fmt(whole[name]["reference"])} | {fmt(whole[name]["sres_cond"])} | '
              f'{peak[name]["reference"]:.0f} -> {peak[name]["sres_cond"]:.0f} |')
    print(f'shared pad + unfold of prep_cond (reference, once per forward): {fmt(t_unfold)} ms')
    print('| layer | resampler | x_prev -> z | MB moved | ref ms | op ms | op GB/s | ref ms, stat | op ms, stat |')
    print('|---|---|---|---|---|---|---|---|---|')
    for r in rows:
        print(f'| {r["layer"]} | {r["kind"]} | {r["c"]} {r["x_dtype"]} -> {r["c"] + 27} {r["dtype"]}, {r["h"]}x{r["w"]} | '
              f'{r["bytes"] / 1e6:.0f} | {fmt(r["ref"])} | {fmt(r["op"])} | {r["bytes"] / r["op"][0] / 1e6:.0f} | '
              f'{fmt(r["ref_stat"])} | {fmt(r["op_stat"])} |')
    print(json.dumps(dict(whole=whole, peak_mb=peak, layers=rows, unfold=t_unfold, gpu_before=facts_before,
                          gpu_after=facts_after)))


if __name__ == '__main__':
    main()
