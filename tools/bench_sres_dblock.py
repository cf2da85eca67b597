"""The super-res discriminator's resnet blocks: the reference composition (conv2d_resample + bias_act per layer, then the
merge) against sres_dblock (conv0 with bias_act in its epilogue, conv1 with the FIR in its re-tiling pass, the skip with the
residual merge in its epilogue), at per-GPU batch 8 with the default VideoDiscriminator (hr 256 x 256, seq_length 8,
num_fp16_res 4: blocks b256-b32 fp16, b16 and b8 fp32), TF32 off.

  block     one block on a random input of its shape: sd._composition against sd.sres_dblock
  whole D   the unmodified reference VideoDiscriminator (staged at oracle/_ref/src by build()) without and with
            sres_dblock.install

each in three modes: forward (no grad), forward + backward, and the R1 pattern (input gradient with create_graph, then the
backward of its square sum). ms per call: median over alternating rounds of CUDA-event timed calls, with the spread (min ..
max) of both sides; peak memory above what was allocated before the call; kernels launched through liblvg_ops per call
(custom_ops.launch_count, eager launches). The GPU name, power limit and SM clocks are read in the same run. Needs a CUDA
device.

  python tools/bench_sres_dblock.py [--rounds 7] [--calls 10] [--batch 8] [--out file.json]
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

import numpy as np                                     # noqa: E402
import torch                                           # noqa: E402
from torch_utils import custom_ops                     # noqa: E402
from torch_utils.ops import sres_dblock as sd          # noqa: E402
from torch_utils.ops import upfirdn2d                  # noqa: E402

MODES = ('fwd', 'fwd_bwd', 'r1')


def gpu_facts():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def run(fn, mode, x, params):
    """One pass of fn(x) in the given mode."""
    for p in params:
        p.grad = None
    if mode == 'fwd':
        with torch.no_grad():
            fn(x)
        return
    xi = x.detach().requires_grad_(mode == 'r1')
    out = fn(xi)
    if mode == 'fwd_bwd':
        out.float().square().sum().backward()
    else:
        gx, = torch.autograd.grad(out.float().sum(), [xi], create_graph=True)
        (gx.float().square().sum() + out.float().sum()).backward()


def measure(sides, mode, x, params, rounds, calls):
    """{side: (median ms, min, max, peak MB, launches per call)}, the sides alternating round by round."""
    times = {s: [] for s in sides}
    peak, launches = {}, {}
    for name, fn in sides.items():                     # warm-up, peak memory and launch count
        run(fn, mode, x, params)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        n0 = custom_ops.launch_count()
        run(fn, mode, x, params)
        torch.cuda.synchronize()
        launches[name] = custom_ops.launch_count() - n0
        peak[name] = (torch.cuda.max_memory_allocated() - base) / 2**20
    for _ in range(rounds):
        for name, fn in sides.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(calls):
                run(fn, mode, x, params)
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b) / calls)
    return {s: dict(ms=statistics.median(t), lo=min(t), hi=max(t), peak_mb=round(peak[s], 1), launches=launches[s])
            for s, t in times.items()}


BLOCKS = [(64, 128, 256, torch.float16), (128, 256, 128, torch.float16), (256, 512, 64, torch.float16),
          (512, 512, 32, torch.float16), (512, 512, 16, torch.float32), (512, 512, 8, torch.float32)]


def bench_blocks(batch, rounds, calls):
    rows = []
    f = upfirdn2d.setup_filter([1, 3, 3, 1]).cuda()
    gain = float(np.sqrt(2))
    for cin, cout, res, dtype in BLOCKS:
        g = torch.Generator().manual_seed(res)
        t = lambda *s: torch.randn(*s, generator=g).cuda().to(dtype).requires_grad_(True)       # noqa: E731
        ws, w0, b0, w1, b1 = t(cout, cin, 1, 1) / cin ** .5, t(cin, cin, 3, 3) / (9 * cin) ** .5, t(cin), t(cout, cin, 3, 3) / (9 * cin) ** .5, t(cout)
        params = [p.detach().requires_grad_(True) for p in (ws, w0, b0, w1, b1)]
        x = torch.randn(batch, cin, res, res, generator=g).cuda().to(dtype)
        sides = {'composition': lambda xi: sd._composition(xi, *params, f, f, 'lrelu', gain, 256),
                 'op': lambda xi: sd.sres_dblock(xi, *params, f, f, act='lrelu', gain=gain, clamp=256)}
        assert sd.native(x, params[0], params[1], params[3], f, f, 'lrelu')
        for mode in MODES:
            r = measure(sides, mode, x, params, rounds, calls)
            rows.append(dict(block=f'b{res}', shape=[batch, cin, res, res], dtype=str(dtype).split('.')[-1], mode=mode, **r))
            print(json.dumps(rows[-1]), flush=True)
    return rows


def bench_whole(batch, rounds, calls):
    from model import discriminator_sres as ds
    torch.manual_seed(0)
    D = ds.VideoDiscriminator().cuda()
    plain = ds.DiscriminatorBlock.forward, ds.Conv2dLayer.forward
    sd.install(ds)
    patched = ds.DiscriminatorBlock.forward, ds.Conv2dLayer.forward
    g = torch.Generator().manual_seed(1)
    lr = torch.randn(batch, 3, 8, 32, 32, generator=g).cuda()
    hr = torch.randn(batch, 3, 8, 256, 256, generator=g).cuda()

    def side(fwds):
        def fn(h):
            ds.DiscriminatorBlock.forward, ds.Conv2dLayer.forward = fwds
            return D(lr, h)
        return fn
    params = list(D.parameters())
    rows = []
    for mode in MODES:
        r = measure({'composition': side(plain), 'op': side(patched)}, mode, hr, params, rounds, calls)
        rows.append(dict(block='whole D', shape=[batch, 3, 8, 256, 256], mode=mode, **r))
        print(json.dumps(rows[-1]), flush=True)
    ds.DiscriminatorBlock.forward, ds.Conv2dLayer.forward = plain
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--calls', type=int, default=10)
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_sres_dblock needs a CUDA device'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    facts = [gpu_facts()]
    print(json.dumps(dict(gpu=facts[0])), flush=True)
    rows = bench_blocks(a.batch, a.rounds, a.calls) + bench_whole(a.batch, a.rounds, a.calls)
    facts.append(gpu_facts())
    print(json.dumps(dict(gpu_after=facts[1])), flush=True)
    if a.out:
        with open(a.out, 'w') as fh:
            json.dump(dict(gpu=facts, rows=rows), fh, indent=1)


if __name__ == '__main__':
    main()
