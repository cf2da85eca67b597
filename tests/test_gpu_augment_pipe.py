"""augment_pipe on the H100 (torch_utils/ops/augment_pipe.py, csrc/augment_pipe.cu).

Accuracy: forward, adjoint and double backward against the float64 composition on extreme transforms (45 degrees, scale
0.25 and 4, aniso, every xflip / rotate90, margins at their clamp, odd extents, N = 1), with NaN-filled outputs followed by
guards and a workspace of exactly lvg_augment_pipe_workspace bytes. The dense matrix of the forward kernel equals the
transpose of the adjoint kernel's. The installed unmodified AugmentPipe.forward against the original under the same seeds
(both super-res configurations, p = 0, 0.5, 1), one case through the unmodified SuperResVideoGAN.run_D with the R1
pattern, no host synchronisation, determinism; CUDA-graph capture; the profiler sees every kernel instance."""
import json
import math
import os
import subprocess
import sys

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import augment_pipe as ap
from torch_utils.ops import upfirdn2d

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')

pytestmark = pytest.mark.gpu
DEV = 'cuda'

SYM6 = [0.015404109327027373, 0.0034907120842174702, -0.11799011114819057, -0.048311742585633, 0.4910559419267466,
        0.787641141030194, 0.3379294217276218, -0.07263752278646252, -0.021060292512300564, 0.04472490177066578,
        0.0017677118642428036, -0.007800708325034148]


def _filter():
    return upfirdn2d.setup_filter(SYM6)


def _rot(a):
    return torch.tensor([[math.cos(a), -math.sin(a), 0], [math.sin(a), math.cos(a), 0], [0, 0, 1]], dtype=torch.float64)


def _diag(sx, sy):
    return torch.diag(torch.tensor([sx, sy, 1.0], dtype=torch.float64))


def params(gs, h, w, clamp=False, seed=0):
    """[N, 23] from per-sample G_inv (output pixel -> input pixel) through the reference's margin rule and conjugations."""
    gen = torch.Generator().manual_seed(seed)
    n = len(gs)
    cx, cy = (w - 1) / 2, (h - 1) / 2
    corners = torch.tensor([[-cx, -cy, 1], [cx, -cy, 1], [cx, cy, 1], [-cx, cy, 1]], dtype=torch.float64).t()
    mg = torch.stack([(g @ corners)[:2] for g in gs]).permute(1, 0, 2).flatten(1)
    mg = torch.cat([-mg, mg]).max(1).values + torch.tensor([6 - cx, 6 - cy] * 2, dtype=torch.float64)
    lim = torch.tensor([w - 1, h - 1] * 2, dtype=torch.float64)
    m = [int(v) for v in (lim if clamp else mg.clamp(min=0).minimum(lim).ceil())]
    uw, uh, vw, vh = 2 * (w + m[0] + m[2]), 2 * (h + m[1] + m[3]), 2 * w + 12, 2 * h + 12
    T = lambda tx, ty: torch.tensor([[1, 0, tx], [0, 1, ty], [0, 0, 1]], dtype=torch.float64)     # noqa: E731
    p = torch.zeros(n, ap.NPAR, dtype=torch.float64)
    for i, g in enumerate(gs):
        g = T((m[0] - m[2]) / 2, (m[1] - m[3]) / 2) @ g
        g = _diag(2, 2) @ g @ _diag(0.5, 0.5)
        g = T(-0.5, -0.5) @ g @ T(0.5, 0.5)
        g = _diag(2 / uw, 2 / uh) @ g @ _diag(vw / 2, vh / 2)
        p[i, 4:10] = g[:2].reshape(6)
    p[:, :4] = torch.tensor(m, dtype=torch.float64)
    p[:, 10:22] = (torch.eye(4, dtype=torch.float64)[:3] + 0.3 * torch.randn(n, 3, 4, generator=gen, dtype=torch.float64)).view(n, 12)
    p[:, 22] = torch.rand(n, generator=gen, dtype=torch.float64) * 0.1
    return p.float()


def _r90(k, flip):
    c, s = float(torch.cos(torch.tensor(math.pi / 2 * k))), float(torch.sin(torch.tensor(math.pi / 2 * k)))
    return _diag(-1 if flip else 1, 1) @ torch.tensor([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=torch.float64)


# (name, transforms per sample, T, H, W, margins at the clamp)
CASES = [
    ('rot45', [_rot(math.pi / 4), _rot(-math.pi / 4) @ _diag(1.1, 0.9)], 2, 13, 21, False),
    ('rot_any_clamped', [_rot(2.1), _rot(-0.4)], 2, 12, 17, True),
    ('scale_0.25_n1', [_diag(0.25, 0.25)], 3, 9, 15, False),
    ('scale_4', [_diag(4, 4), _rot(0.5) @ _diag(4, 4)], 2, 11, 14, False),
    ('aniso', [_rot(-1.1) @ _diag(2.3, 1 / 2.3) @ _rot(0.7), _diag(0.5, 2)], 2, 12, 20, False),
    ('xflip_rot90', [_r90(k, f) for f in (0, 1) for k in range(4)], 1, 9, 15, False),
    ('xflip_rot90_clamped', [_r90(k, f) for f in (0, 1) for k in range(4)], 1, 10, 13, True),
    ('identity_odd', [torch.eye(3, dtype=torch.float64)], 2, 7, 9, False),
]


def _err(a, b):
    return float((a.double().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-30))


@pytest.mark.parametrize('case', CASES, ids=[c[0] for c in CASES])
def test_forward_adjoint_and_double_backward_against_float64(case):
    name, gs, t, h, w, clamp = case
    p = params(gs, h, w, clamp, seed=len(name))
    n = len(gs)
    f = _filter()
    g = torch.Generator().manual_seed(1)
    x = torch.rand(n, 3, t, h, w, generator=g, dtype=torch.float64) * 2 - 1
    dy = torch.randn(n, 3, t, h, w, generator=g, dtype=torch.float64)
    noise = torch.randn(n, 3, t, h, w, generator=g, dtype=torch.float64)
    res = []
    for d, ty in ((DEV, torch.float32), ('cpu', torch.float64)):
        xg, dyg = x.to(d, ty).requires_grad_(True), dy.to(d, ty).requires_grad_(True)
        y = ap.apply(xg, p.to(d), noise.to(d, ty), f.to(d), ap.GEOM)
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


@pytest.mark.parametrize('flags', [0, ap.GEOM])
@pytest.mark.parametrize('case', [CASES[1], CASES[6]], ids=[CASES[1][0], CASES[6][0]])
def test_raw_entries_with_guards_and_an_exact_workspace(case, flags):
    name, gs, t, h, w, clamp = case
    n = len(gs)
    p = params(gs, h, w, clamp, seed=5).to(DEV)
    f = _filter().to(DEV)
    g = torch.Generator().manual_seed(4)
    x = (torch.rand(n, 3, t, h, w, generator=g) * 2 - 1).to(DEV)
    dy = torch.randn(n, 3, t, h, w, generator=g).to(DEV)
    noise = torch.randn(n, 3, t, h, w, generator=g).to(DEV)
    ref_y = ap._reference(x.double().cpu(), p.cpu(), noise.double().cpu(), f.cpu(), flags)
    ref_dx = ap._reference_adjoint(dy.double().cpu(), p.cpu(), f.cpu(), flags)
    lib = custom_ops.load_library()
    ws_bytes = lib.lvg_augment_pipe_workspace(n, 3, t, h, w, flags)
    assert ws_bytes == (n * 3 * t * (2 * h + 12) * (2 * w + 12) * 4 if flags else 0)
    stream = torch.cuda.current_stream().cuda_stream
    copies = [v.clone() for v in (x, dy, noise, p, f)]
    out = _guarded(x.numel(), torch.float32, float('nan'))
    rc = lib.lvg_augment_pipe(x.data_ptr(), p.data_ptr(), f.data_ptr(), 12, noise.data_ptr(), out.data_ptr(), n, 3, t, h, w, flags, stream)
    assert rc == 0, lib.lvg_last_error()
    out2 = _guarded(x.numel(), torch.float32, float('nan'))
    ws = _guarded(ws_bytes, torch.uint8, 0xFF)
    rc = lib.lvg_augment_pipe_adjoint(dy.data_ptr(), p.data_ptr(), f.data_ptr(), 12, out2.data_ptr(), ws.data_ptr(), n, 3, t, h, w, flags,
                                      stream)
    assert rc == 0, lib.lvg_last_error()
    torch.cuda.synchronize()
    for buf, ref in ((out, ref_y), (out2, ref_dx)):
        got = buf[:ref.numel()].view(ref.shape)
        assert not torch.isnan(got).any()
        assert _err(got, ref) <= 1e-5
        assert torch.equal(buf[ref.numel():].cpu(), torch.full([4096], 12345.0)), 'output guard overwritten'
    assert torch.equal(ws[ws_bytes:].cpu(), torch.full([4096], 0xA5, dtype=torch.uint8)), 'workspace guard overwritten'
    for a, b in zip((x, dy, noise, p, f), copies):
        assert torch.equal(a, b), 'inputs modified'


@pytest.mark.parametrize('case', [CASES[0], CASES[3], CASES[5]], ids=[CASES[0][0], CASES[3][0], CASES[5][0]])
def test_dense_forward_matrix_is_the_transpose_of_the_adjoint(case):
    """One frame of 9 x 15 per sample: columns of A from unit inputs, rows of A^T from unit outputs."""
    name, gs, _, _, _, clamp = case
    h, w = 9, 15
    gs = gs[:2]
    n, m = len(gs), 3 * h * w
    p = params(gs, h, w, clamp, seed=2).to(DEV)
    f = _filter().to(DEV)
    plugin = custom_ops.get_plugin('augment_pipe_plugin')
    eye = torch.eye(m, device=DEV).view(m, 3, 1, h, w)
    for i in range(n):
        pi = p[i:i + 1].expand(m, ap.NPAR).contiguous()
        a = plugin.run(eye, pi, f, None, ap.GEOM | ap.LINEAR).view(m, m).t()           # A[:, j] = A e_j
        at = plugin.run(eye, pi, f, None, ap.GEOM, adjoint=True).view(m, m).t()         # A^T[:, j] = A^T e_j
        scale = float(a.abs().max())
        assert float((a - at.t()).abs().max()) <= 1e-6 * scale, name


def test_envelope_and_fallback_on_the_device():
    class Pipe:
        imgfilter = cutout = 0
        Hz_geom = _filter().to(DEV)
        xflip = rotate90 = xint = scale = rotate = aniso = 0.0
        xfrac = 1.0
    pipe = Pipe()
    assert ap.applies(pipe, torch.zeros(2, 3, 4, 9, 15, device=DEV))
    assert not ap.applies(pipe, torch.zeros(2, 3, 4, 9, 15, device=DEV, dtype=torch.float64))
    assert not ap.applies(pipe, torch.zeros(2, 4, 4, 9, 15, device=DEV))
    assert not ap.applies(pipe, torch.zeros(2, 3, 4, 9, 15, device=DEV), debug_percentile=0.5)
    pipe.cutout = 1
    assert not ap.applies(pipe, torch.zeros(2, 3, 4, 9, 15, device=DEV))
    pipe.cutout, pipe.imgfilter = 0, 1
    assert not ap.applies(pipe, torch.zeros(2, 3, 4, 9, 15, device=DEV))
    pipe.imgfilter, pipe.Hz_geom = 0, upfirdn2d.setup_filter([1, 3, 3, 1]).to(DEV)
    assert not ap.applies(pipe, torch.zeros(2, 3, 4, 9, 15, device=DEV))
    assert custom_ops.get_plugin('augment_pipe_plugin').run(torch.zeros(1, 4, 2, 5, 5, device=DEV), torch.zeros(1, 23, device=DEV),
                                                            _filter().to(DEV), None, ap.GEOM) is None


def test_cuda_graph_capture_replays_equal_to_eager():
    gs = [_rot(0.3) @ _diag(1.1, 0.9), _r90(1, 1), _diag(0.8, 0.8), _rot(-2.0)]
    n, t, h, w = 4, 4, 36, 64
    p = params(gs, h, w, seed=9).to(DEV)
    f = _filter().to(DEV)
    x = torch.rand(n, 3, t, h, w, device=DEV).requires_grad_(True)
    noise = torch.randn(n, 3, t, h, w, device=DEV)
    dy = torch.randn(n, 3, t, h, w, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            y = ap.apply(x, p, noise, f, ap.GEOM)
            gx, = torch.autograd.grad(y, [x], dy)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y_static = ap.apply(x, p, noise, f, ap.GEOM)
        gx_static, = torch.autograd.grad(y_static, [x], dy)
    x.data.copy_(torch.rand(n, 3, t, h, w, device=DEV))
    dy.copy_(torch.randn(n, 3, t, h, w, device=DEV))
    noise.copy_(torch.randn(n, 3, t, h, w, device=DEV))
    graph.replay()
    y_eager = ap.apply(x, p, noise, f, ap.GEOM)
    gx_eager, = torch.autograd.grad(y_eager, [x], dy)
    torch.cuda.synchronize()
    assert torch.equal(y_static, y_eager) and torch.equal(gx_static, gx_eager)


_PROFILE = r"""
import json, sys, torch
sys.path[:0] = sys.argv[1:]
from torch_utils import custom_ops
from torch_utils.ops import augment_pipe as ap
from test_gpu_augment_pipe import DEV, _diag, _filter, _rot, params
n, t, h, w = 2, 2, 12, 20
p = params([_rot(0.4), _diag(1.2, 0.7)], h, w).to(DEV)
f = _filter().to(DEV)
x = torch.rand(n, 3, t, h, w, device=DEV).requires_grad_(True)
dy = torch.randn(n, 3, t, h, w, device=DEV).requires_grad_(True)
noise = torch.randn(n, 3, t, h, w, device=DEV)

def sequence():     # per flag set: forward, adjoint (2 kernels with GEOM), the adjoint's backward (linear forward)
    for flags in (0, ap.GEOM):
        y = ap.apply(x, p, noise, f, flags)
        gx, = torch.autograd.grad(y, [x], dy, create_graph=True)
        torch.autograd.grad(gx.square().sum(), [dy])

sequence()
torch.cuda.synchronize()
before = custom_ops.launch_count()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(3):
        sequence()
    torch.cuda.synchronize()
launches = custom_ops.launch_count() - before
names = sorted({e.name.replace(' ', '') for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA})
print(json.dumps(dict(launches=launches, names=names)))
"""


def test_profiler_sees_every_kernel():
    """Every kernel instance shows up under torch.profiler, and the library's launch counter counts 7 launches per sequence.
    The profile runs in a process of its own, so that it neither depends on nor disturbs the profiler state of a long
    single-process run of the suite."""
    r = subprocess.run([sys.executable, '-c', _PROFILE, os.path.dirname(os.path.abspath(__file__)), PKG], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res['launches'] == 3 * 7
    names = res['names']
    if not names:
        pytest.skip('torch.profiler reported no CUDA kernels on this machine, so launches cannot be observed')
    for k in ('augment_pipe_color_kernel<false,false>', 'augment_pipe_color_kernel<false,true>', 'augment_pipe_color_kernel<true,true>',
              'augment_pipe_fwd_kernel<false>', 'augment_pipe_fwd_kernel<true>', 'augment_pipe_dv_kernel', 'augment_pipe_adjoint_kernel'):
        assert any(k in nm for nm in names), (k, names)


needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(SRC, 'model')), reason='oracle/_ref not staged')


@needs_ref
def test_installed_pipe_matches_the_reference_without_sync_and_deterministically(tmp_path):
    out = str(tmp_path / 'cuda.pt')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]), CUBLAS_WORKSPACE_CONFIG=':4096:8')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'augment_pipe_run.py'), out, 'cuda'], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:]
    res = torch.load(out, weights_only=False)
    assert len(res['cases']) == 8
    for case in res['cases']:
        ref, ours = case['ref'], case['ours']
        for key in ('y', 'gx'):
            assert ours[key].shape == ref[key].shape
            e = _err(ours[key], ref[key].double())
            assert e <= 1e-5, f'{case["case"]} {key}: {e:.3e}'
        assert torch.equal(ours['cuda_state'], ref['cuda_state']) and torch.equal(ours['cpu_state'], ref['cpu_state']), case['case']
    ref, ours = res['run_D']
    for key in ('logits', 'gx'):
        e = _err(ours[key], ref[key].double())
        assert e <= 1e-5, f'run_D {key}: {e:.3e}'
    assert torch.isfinite(res['nosync']).all()
    a, b = res['det']
    assert torch.equal(a, b), 'two deterministic runs differ'
