"""The low-res discriminator's residual blocks: the reference DiscriminatorBlock.forward (staged at oracle/_ref/src by
build()) against dblock_tail.block_forward and conv_bias_act layers (what
dblock_tail.install can route to), in the default VideoDiscriminator(seq_length=128, max_edge=64) at batch 8, fp32, TF32 off, both sides with conv_nd.install_functional and conv3d_down.install (as a training run configures
them).

  tail        from conv_1's convolution output y and the skip tensor: the reference's op sequence against dblock_tail
  block       one DiscriminatorBlock on the input the discriminator feeds it, with its tail on the op, and (separately) with
              conv_0 through conv_nd.conv_bias_act (bias_act in the convolution's epilogue)
  whole D     all of it, the same two ways; peak memory above the parameters and the input
  kernels     lvg_dblock_tail (write mode) and lvg_dblock_tail_adjoint (with ds) called through the Python plugin, so output
              allocation and argument checks are included: achieved GB/s over their algorithmic bytes (forward |y| + |s| +
              |z| + codes, adjoint |dz| + codes + |dy| + |ds|, computed from the shapes here)

each in three modes: forward (no grad), forward + backward, and the R1 pattern (input gradient with create_graph, then the
backward of its square sum). ms per call: median over alternating rounds of CUDA-event timed calls with the spread (min ..
max) of the installed side. The GPU name, power limit and SM clocks are read before and after the run. Needs a CUDA device.

  python tools/bench_dblock_tail.py [--rounds 3] [--calls 4] [--seq 128] [--batch 8]
"""
import argparse
import json
import math
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
from model import discriminator_lres as dl             # noqa: E402
from torch_utils import custom_ops                     # noqa: E402
from torch_utils.ops import conv_nd, conv3d_down, dblock_tail   # noqa: E402

HBM_DATA_SHEET_GBS = 3350.0       # H100 SXM data sheet, not a measurement
MODES = ('fwd', 'fwd_bwd', 'r1')


def gpu_facts():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def timed(sides, fn, rounds, calls):
    """ms per call of fn() for each side (a callable that selects it), the sides alternating: (medians, all rounds)."""
    times = {s: [] for s in sides}
    for use in sides.values():
        use()
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


def three_modes(run, inputs, params):
    """fn per mode for out = run(*inputs): inputs are leaf tensors, params the parameters whose .grad is dropped."""
    def clear():
        for p in list(inputs) + list(params):
            p.grad = None

    def fwd():
        with torch.no_grad():
            run(*[v.detach() for v in inputs])

    def fwd_bwd():
        run(*inputs).square().mean().backward()
        clear()

    def r1():
        out = run(*inputs)
        g, = torch.autograd.grad(out.sum(), [inputs[0]], create_graph=True)
        (g.square().sum() + out.mean()).backward()
        clear()
    return dict(fwd=fwd, fwd_bwd=fwd_bwd, r1=r1)


def cell(med, runs, ours):
    return f'{med["reference"]:.2f} -> {med[ours]:.2f} ({min(runs[ours]):.2f} .. {max(runs[ours]):.2f})'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--calls', type=int, default=4)
    ap.add_argument('--seq', type=int, default=128)
    ap.add_argument('--batch', type=int, default=8)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_dblock_tail needs a CUDA device'
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    conv_nd.install_functional(dl)
    conv3d_down.install(dl)
    orig = dl.DiscriminatorBlock.forward

    def patched(self, input):          # every block on the op, whatever install()'s routing rule says
        assert dblock_tail.applies(self, input)
        return dblock_tail.block_forward(self, input)

    layer_orig = dl.Conv3dLayer.forward
    # conv_bias_act on every layer the engine takes, whatever install()'s routing rule (epilogue_faster) says
    dblock_tail.epilogue_faster = lambda layer, input: True
    layer_epi = dblock_tail._layer_forward(layer_orig)

    def use(f, layer=layer_orig):
        def go():
            dl.DiscriminatorBlock.forward = f
            dl.Conv3dLayer.forward = layer
        return go
    sides = {'reference': use(orig), 'installed': use(patched)}
    esides = {'reference': use(orig), 'installed': use(orig, layer_epi)}
    facts_before = gpu_facts()

    torch.manual_seed(0)
    D = dl.VideoDiscriminator(seq_length=a.seq, max_edge=64).cuda()
    x = (torch.rand(a.batch, 3, a.seq, 64, 64, device='cuda') * 2 - 1).requires_grad_(True)
    seen = []

    def spy(self, input):
        seen.append((self, input.detach()))
        return orig(self, input)
    dl.DiscriminatorBlock.forward = spy
    with torch.no_grad():
        D(x)
    dl.DiscriminatorBlock.forward = orig

    plug = custom_ops.get_plugin('dblock_tail_plugin')
    P = custom_ops.DblockTailPlugin
    rows = []
    for i, (blk, inp) in enumerate(seen):
        c1 = blk.conv_1
        sd, td = c1.spatial_down, c1.temporal_down
        f = c1.downsample._downsample_filter
        with torch.no_grad():
            h = blk.conv_0(blk.conv_vid(inp) if blk.vid_channels > 0 else inp)
            y0 = conv_nd.conv3d(h, c1.weight * c1.weight_gain, padding=c1.padding)
            s0 = blk.conv_skip(blk.conv_vid(inp) if blk.vid_channels > 0 else inp)
            del h
        row = dict(block=i, y=list(y0.shape), z=list(s0.shape))
        for dtype in ((torch.float32, torch.float16) if i == 0 else (torch.float32,)):
            y, s = y0.to(dtype).requires_grad_(True), s0.to(dtype).requires_grad_(True)
            b = c1._bias.detach().to(dtype).requires_grad_(True)
            which = {}
            tsides = {'reference': lambda: which.__setitem__('f', dblock_tail._reference),
                      'installed': lambda: which.__setitem__('f', None)}

            def tail(y_, s_, b_):
                if which['f'] is None:
                    return dblock_tail.dblock_tail(y_, s_, b_, f, spatial_down=sd, temporal_down=td, act=c1.activation, clamp=c1.conv_clamp)
                return which['f'](y_, s_, b_, f, sd, td, c1.activation, c1.conv_clamp)
            key = 'tail' if dtype == torch.float32 else 'tail_fp16'
            for m, fn in three_modes(tail, [y, s, b], []).items():
                row[f'{key}_{m}'] = timed(tsides, fn, a.rounds, a.calls * (1 if i == 0 else 5))
            if dtype == torch.float32:
                # the two kernels alone
                flags = (P.TDOWN if td else 0) | (P.SDOWN if sd else 0) | P.MERGE
                gain = math.sqrt(2)
                yd, sd_, bd = y.detach(), s.detach(), b.detach()
                _, codes = plug.forward(yd, sd_, bd, f, flags, 3, 0.2, gain, 256.0, P.WRITE)
                dz = torch.randn_like(sd_)
                k = {'reference': lambda: which.__setitem__('k', 'fwd'), 'installed': lambda: which.__setitem__('k', 'adj')}

                def kern():
                    if which['k'] == 'fwd':
                        plug.forward(yd, sd_, bd, f, flags, 3, 0.2, gain, 256.0, P.WRITE)
                    else:
                        plug.adjoint(dz, codes, f, tuple(yd.shape[2:]), flags, 3, 0.2, gain, True)
                med, _ = timed(k, kern, a.rounds, 50)
                esz = 4
                fwd_bytes = (yd.numel() + 2 * sd_.numel()) * esz + codes.numel()
                adj_bytes = (yd.numel() + 2 * sd_.numel()) * esz + codes.numel()
                row['kernel_fwd'] = dict(ms=med['reference'], bytes=fwd_bytes, gbs=fwd_bytes / med['reference'] / 1e6)
                row['kernel_adj'] = dict(ms=med['installed'], bytes=adj_bytes, gbs=adj_bytes / med['installed'] / 1e6)
                del codes, dz
            del y, s, b
        del y0, s0
        xin = inp.clone().requires_grad_(True)
        for m, fn in three_modes(lambda v: blk(v), [xin], list(blk.parameters())).items():
            row[f'block_{m}'] = timed(sides, fn, a.rounds, a.calls)
            row[f'epi_{m}'] = timed(esides, fn, a.rounds, a.calls)
        del xin
        rows.append(row)
        torch.cuda.empty_cache()

    whole, whole_epi, peak = {}, {}, {}
    for m, fn in three_modes(lambda v: D(v), [x], list(D.parameters())).items():
        whole[m] = timed(sides, fn, a.rounds, 1)
        whole_epi[m] = timed(esides, fn, a.rounds, 1)
        peak[m] = {}
        for sname, u in sides.items():
            u()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            fn()
            torch.cuda.synchronize()
            peak[m][sname] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    use(orig)()
    facts_after = gpu_facts()

    print(f'GPU (name, power limit, SM clock, max SM clock): before {facts_before}; after {facts_after}')
    print(f'VideoDiscriminator(seq_length={a.seq}, max_edge=64), batch {a.batch}, fp32, TF32 off; {a.rounds} alternating rounds; '
          'ms reference -> installed (min .. max of the installed rounds)')
    print('| | y -> z | forward | forward + backward | R1 pattern |')
    print('|---|---|---|---|---|')
    for r in rows:
        for key, label in (('tail', 'tail'), ('tail_fp16', 'tail fp16'), ('block', 'block, tail on the op'),
                           ('epi', 'block, conv_0 with the epilogue')):
            if f'{key}_fwd' in r:
                print(f'| {label} {r["block"]} | {r["y"][1:]} -> {r["z"][1:]} | '
                      + ' | '.join(cell(*r[f'{key}_{m}'], 'installed') for m in MODES) + ' |')
    print('| whole D, tails on the op | | ' + ' | '.join(cell(*whole[m], 'installed') for m in MODES) + ' |')
    print('| whole D, conv_0 with the epilogue | | ' + ' | '.join(cell(*whole_epi[m], 'installed') for m in MODES) + ' |')
    print('| peak MB, whole D | | ' + ' | '.join(f'{peak[m]["reference"]:.0f} -> {peak[m]["installed"]:.0f}' for m in MODES) + ' |')
    print(f'lvg_dblock_tail / lvg_dblock_tail_adjoint through the Python plugin (output allocation and argument checks included), fp32 (data-sheet HBM bandwidth of the H100 SXM, not measured: {HBM_DATA_SHEET_GBS:.0f} GB/s)')
    print('| block | forward (write) ms | MB | GB/s | adjoint (with ds) ms | MB | GB/s |')
    print('|---|---|---|---|---|---|---|')
    for r in rows:
        kf, ka = r['kernel_fwd'], r['kernel_adj']
        print(f'| {r["block"]} | {kf["ms"]:.3f} | {kf["bytes"] / 1e6:.0f} | {kf["gbs"]:.0f} | {ka["ms"]:.3f} | {ka["bytes"] / 1e6:.0f} | {ka["gbs"]:.0f} |')
    print(json.dumps(dict(rows=rows, whole=whole, whole_epilogue=whole_epi, peak_mb=peak, gpu_before=facts_before, gpu_after=facts_after)))


if __name__ == '__main__':
    main()
