"""video_augment on the H100 (torch_utils/ops/video_augment.py, csrc/video_augment.cu).

Accuracy: forward, adjoint and double backward against the float64 composition (scales below, at and above 1 with padded
and cropped clips, translations of +-shift and 0, cutouts on every edge, odd extents, C = 1, 3, 4, N = 1).
Exact tier: color neutral, small-integer video and dy, dyadic reciprocal scales -- every intermediate is exact, so the
library's results must equal float64 bit for bit; outputs are NaN-filled and followed by guards, and the workspace has
exactly lvg_video_augment_workspace bytes. <A x, y> = <x, A^T y>. The installed unmodified run_D against the reference's
under the same seeds; no host synchronisation; determinism; CUDA-graph capture; the profiler sees the kernels."""
import os
import subprocess
import sys

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import video_augment as va

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def params(n, t, t_out, h, w, scale=1.0, off=0, dh=0, dw=0, rect=(0, -1, 0, -1), color=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    p = torch.zeros(n, va.NPAR)
    if color:
        p[:, 0] = torch.rand(n, generator=g) - 0.5
        p[:, 1] = torch.rand(n, generator=g) * 2
        p[:, 2] = torch.rand(n, generator=g) + 0.5
    else:
        p[:, 1:3] = 1
    p[:, 3], p[:, 4] = dh, dw
    p[:, 5:9] = torch.tensor(rect, dtype=torch.float32)
    p[:, 9] = float(torch.tensor(1.0 / scale, dtype=torch.float32))
    p[:, 10] = int(t * scale)
    p[:, 11] = off
    return p


# (name, N, C, T, H, W, scale, off, dh, dw, cutout rows / columns)
CASES = [
    ('down_padded', 2, 3, 16, 12, 20, 0.6, -3, 3, -5, (2, 7, 4, 13)),
    ('unit', 2, 3, 16, 12, 20, 1.0, 0, 0, 0, (0, 5, 0, 9)),
    ('up_cropped', 2, 3, 16, 12, 20, 1.7, 6, -3, 5, (6, 11, 10, 19)),
    ('down_strong', 2, 3, 24, 8, 16, 0.51, -5, 2, 4, (0, 7, 0, 3)),
    ('up_strong', 2, 3, 12, 8, 16, 1.98, 11, -2, -4, (0, 7, 12, 15)),
    ('odd_c1_n1', 1, 1, 13, 9, 15, 1.37, 2, 2, -4, (0, 0, 0, 14)),
    ('odd_c4', 2, 4, 11, 9, 15, 0.77, -1, -2, 4, (8, 8, 3, 9)),
    ('shift_edges', 2, 3, 16, 12, 20, 1.2, 1, 5, 5, (11, 11, 0, 19)),
    ('shift_edges_neg', 2, 3, 16, 12, 20, 0.9, -1, -5, -5, (0, 11, 19, 19)),
]


def _err(a, b):
    return float((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_forward_adjoint_and_double_backward_against_float64(case):
    name, n, c, t, h, w, scale, off, dh, dw, rect = case
    p = params(n, t, t, h, w, scale, off, dh, dw, rect, seed=len(name))
    g = torch.Generator().manual_seed(1)
    x = torch.rand(n, c, t, h, w, generator=g, dtype=torch.float64) * 2 - 1
    dy = torch.randn(n, c, t, h, w, generator=g, dtype=torch.float64)
    res = []
    for d, ty in ((DEV, torch.float32), ('cpu', torch.float64)):
        xg, dyg = x.to(d, ty).requires_grad_(True), dy.to(d, ty).requires_grad_(True)
        y = va.apply(xg, p.to(d), t)
        gx, = torch.autograd.grad(y, [xg], dyg, create_graph=True)
        hdy, = torch.autograd.grad(gx.square().sum(), [dyg])            # 2 A (A^T dy): the linear forward
        res.append((y, gx, hdy))
    for what, got, ref in zip(('y', 'dx', 'ddy'), *res):
        assert got.shape == ref.shape
        e = _err(got.detach(), ref.detach())
        assert e <= 1e-5, f'{name} {what}: {e:.3e}'


def _guarded(numel, dtype, fill):
    buf = torch.empty(numel + 4096, dtype=dtype, device=DEV)
    buf[:numel] = fill
    buf[numel:] = 12345.0 if dtype == torch.float32 else 0xA5
    return buf


EXACT = [('unit', 1.0, 0), ('half', 0.5, -4), ('double', 2.0, 9), ('three_quarters', 1.25, 2), ('five_quarters', 0.75, -1),
         ('eighths', 1.625, 3)]


@pytest.mark.parametrize('c', [1, 3, 4])
@pytest.mark.parametrize('name,r,off', EXACT, ids=[e[0] for e in EXACT])
def test_exact_tier_bit_for_bit_with_guards(name, r, off, c):
    n, t, h, w = 2, 12, 9, 15
    t_out = 12
    p = params(n, t, t_out, h, w, 1 / r, off, 2, -3, (1, 3, 8, 14), color=False)
    p[:, 9] = r
    p[:, 10] = int(t / r)
    g = torch.Generator().manual_seed(4)
    x = torch.randint(-8, 9, (n, c, t, h, w), generator=g).double()
    dy = torch.randint(-8, 9, (n, c, t_out, h, w), generator=g).double()
    ref_y = va._reference(x, p, t_out)
    ref_dx = va._reference_adjoint(dy, p, t)
    for ref in (ref_y, ref_dx):                 # precondition: multiples of 1/64 within fp32's exact range
        assert torch.equal(torch.round(ref * 64), ref * 64) and float(ref.abs().max()) * 64 < 2 ** 24
    lib = custom_ops.load_library()
    ws_bytes = lib.lvg_video_augment_workspace(n, c, t, h, w, t_out)
    assert ws_bytes > 0 and ws_bytes % 4 == 0
    for adjoint, src, ref in ((False, x, ref_y), (True, dy, ref_dx)):
        xs, pd = src.float().to(DEV), p.to(DEV)
        xs_copy, pd_copy = xs.clone(), pd.clone()
        out = _guarded(ref.numel(), torch.float32, float('nan'))
        ws = _guarded(ws_bytes, torch.uint8, 0xFF)
        stream = torch.cuda.current_stream().cuda_stream
        if adjoint:
            rc = lib.lvg_video_augment_adjoint(xs.data_ptr(), pd.data_ptr(), out.data_ptr(), ws.data_ptr(), n, c, t, h, w, t_out, stream)
        else:
            rc = lib.lvg_video_augment(xs.data_ptr(), pd.data_ptr(), out.data_ptr(), ws.data_ptr(), n, c, t, h, w, t_out, 0, stream)
        assert rc == 0, lib.lvg_last_error()
        torch.cuda.synchronize()
        got = out[:ref.numel()].view(ref.shape).double().cpu()
        bad = (got != ref) | torch.isnan(got)
        assert not bad.any(), f'{name} c={c} adjoint={adjoint}: {int(bad.sum())} of {ref.numel()} differ'
        assert torch.equal(out[ref.numel():].cpu(), torch.full([4096], 12345.0)), 'output guard overwritten'
        assert torch.equal(ws[ws_bytes:].cpu(), torch.full([4096], 0xA5, dtype=torch.uint8)), 'workspace guard overwritten'
        assert torch.equal(xs, xs_copy) and torch.equal(pd, pd_copy), 'inputs modified'


@pytest.mark.parametrize('case', CASES[:3] + CASES[5:7], ids=[c[0] for c in CASES[:3] + CASES[5:7]])
def test_adjoint_identity_on_the_device(case):
    name, n, c, t, h, w, scale, off, dh, dw, rect = case
    p = params(n, t, t, h, w, scale, off, dh, dw, rect, seed=3).to(DEV)
    plugin = custom_ops.get_plugin('video_augment_plugin')
    x = torch.randn(n, c, t, h, w, device=DEV)
    y = torch.randn(n, c, t, h, w, device=DEV)
    ax = plugin.run(x, p, t, linear=True)
    aty = plugin.run(y, p, t, adjoint=True)
    lhs, rhs = float((ax.double() * y.double()).sum()), float((x.double() * aty.double()).sum())
    assert abs(lhs - rhs) <= 1e-5 * (ax.double().abs() * y.double().abs()).sum().item(), (lhs, rhs)


def test_unsupported_channels_fall_back():
    assert not va.applies(torch.zeros(2, 5, 8, 6, 10, device=DEV), 'color', 1.0, 8)
    assert va.applies(torch.zeros(2, 4, 8, 6, 10, device=DEV), 'color', 1.0, 8)
    assert custom_ops.get_plugin('video_augment_plugin').run(torch.zeros(1, 5, 4, 3, 3, device=DEV), torch.zeros(1, 12, device=DEV), 4) is None


def test_cuda_graph_capture_replays_equal_to_eager():
    n, c, t, h, w = 4, 3, 32, 36, 64
    p = params(n, t, t, h, w, 1.3, 4, 3, -2, (3, 20, 5, 40), seed=9).to(DEV)
    x = torch.rand(n, c, t, h, w, device=DEV).requires_grad_(True)
    dy = torch.randn(n, c, t, h, w, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            y = va.apply(x, p, t)
            gx, = torch.autograd.grad(y, [x], dy)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_static = va.apply(x, p, t)
        gx_static, = torch.autograd.grad(y_static, [x], dy)
    x.data.copy_(torch.rand(n, c, t, h, w, device=DEV))
    dy.copy_(torch.randn(n, c, t, h, w, device=DEV))
    graph.replay()
    y_eager = va.apply(x, p, t)
    gx_eager, = torch.autograd.grad(y_eager, [x], dy)
    torch.cuda.synchronize()
    assert torch.equal(y_static, y_eager) and torch.equal(gx_static, gx_eager)


def test_profiler_sees_every_kernel():
    """Each kernel instance shows up under torch.profiler. Each instance launches once per sequence, and a profile taken
    late in a long single-process run of the suite has missed such a single launch, so the sequence runs three times in
    the session; the library's own launch counter checks the launches independently of the profiler."""
    n, c, t, h, w = 2, 3, 16, 12, 20
    p = params(n, t, t, h, w, 0.8, -2, 1, 1, (2, 5, 2, 5)).to(DEV)
    x = torch.rand(n, c, t, h, w, device=DEV).requires_grad_(True)
    dy = torch.randn(n, c, t, h, w, device=DEV).requires_grad_(True)

    def sequence():                 # forward, adjoint, and the adjoint's backward (the linear forward): 3 calls, 6 launches
        y = va.apply(x, p, t)
        gx, = torch.autograd.grad(y, [x], dy, create_graph=True)
        torch.autograd.grad(gx.square().sum(), [dy])

    sequence()
    torch.cuda.synchronize()
    before = custom_ops.launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            sequence()
        torch.cuda.synchronize()
    assert custom_ops.launch_count() - before == 3 * 6
    names = sorted({e.name.replace(' ', '') for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
    if not names:
        pytest.skip('torch.profiler reported no CUDA kernels on this machine, so launches cannot be observed')
    for k in ('video_augment_reduce_kernel<0>', 'video_augment_reduce_kernel<1>', 'video_augment_fwd_kernel<3,false>',
              'video_augment_fwd_kernel<3,true>', 'video_augment_adjoint_kernel<3>'):
        assert any(k in nm for nm in names), (k, names)


needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')


@needs_ref
def test_installed_run_D_matches_the_reference_without_sync_and_deterministically(tmp_path):
    out = str(tmp_path / 'cuda.pt')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUBLAS_WORKSPACE_CONFIG=':4096:8')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'video_augment_run.py'), out, 'cuda'], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    res = torch.load(out)
    assert len(res['cases']) == 20
    for case in res['cases']:
        ref, ours = case['ref'], case['ours']
        for key in ('d_in', 'logits', 'gx'):
            assert ours[key].shape == ref[key].shape
            e = _err(ours[key], ref[key].double())
            assert e <= 1e-5, f'{case["case"]} {key}: {e:.3e}'
        assert torch.equal(ours['cuda_state'], ref['cuda_state']) and torch.equal(ours['cpu_state'], ref['cpu_state']), case['case']
    assert torch.isfinite(res['nosync']).all()
    a, b = res['det']
    assert torch.equal(a, b), 'two deterministic runs differ'
