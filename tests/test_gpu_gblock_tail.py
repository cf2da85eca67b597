"""The residual-block tail (torch_utils/ops/gblock_tail.py, csrc/gblock_tail.cu) on the GPU: the forward against a float64
evaluation of the same map for all ten block signatures of the default low-res G at batch 8 (fp32 and fp16), the codes
against the float64 activation decision, the adjoint against float64 and as the transpose of the forward's matrix, guard
bands around every output, bitwise reproducibility, CUDA-graph capture, gradients of higher order, and the unmodified
VideoGenerator with install() against the same generator without it."""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import gblock_tail as gt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
DEV = torch.device('cuda')
CLAMP = 256.0

# (C, T, H, W, temporal_up, spatial_up, T_out, H_out, W_out): the ten blocks of the default VideoGenerator (36 x 64) at the
# low-res step's 160 frames (workloads/lres_step.json)
BLOCKS = [
    (512, 21, 3, 4, True, False, 26, 3, 4),
    (512, 26, 3, 4, True, True, 36, 5, 8),
    (512, 36, 5, 8, True, False, 56, 5, 8),
    (512, 56, 5, 8, True, True, 96, 9, 16),
    (256, 96, 9, 16, True, False, 176, 9, 16),
    (256, 176, 9, 16, False, False, 160, 9, 16),
    (128, 160, 9, 16, False, True, 160, 18, 32),
    (128, 160, 18, 32, False, False, 160, 18, 32),
    (64, 160, 18, 32, False, True, 160, 36, 64),
    (64, 160, 36, 64, False, False, 160, 36, 64),
]
IDS = [f'b{i}' for i in range(len(BLOCKS))]


def _up(x, dim):
    """2x linear upsampling along dim: out[2m] = x[m-1]/4 + 3x[m]/4, out[2m+1] = 3x[m]/4 + x[m+1]/4, zero outside."""
    n = x.shape[dim]
    pad = [0, 0] * (x.ndim - 1 - dim) + [1, 1]
    xp = torch.nn.functional.pad(x, pad)
    lo, mid, hi = xp.narrow(dim, 0, n), xp.narrow(dim, 1, n), xp.narrow(dim, 2, n)
    even, odd = 0.25 * lo + 0.75 * mid, 0.75 * mid + 0.25 * hi
    return torch.stack([even, odd], dim + 1).flatten(dim, dim + 1)


def _lin64(m, tup, sup, to, ho, wo):
    """The linear part in float64, independent of upfirdn2d."""
    if tup:
        m = _up(m, 2)
    t0 = (m.shape[2] - to) // 2
    m = m[:, :, t0:t0 + to]
    if sup:
        m = _up(_up(m, 3), 4)
    h0, w0 = (m.shape[3] - ho) // 2, (m.shape[4] - wo) // 2
    return m[:, :, :, h0:h0 + ho, w0:w0 + wo]


def _inputs(n, c, t, h, w, dtype, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    s = torch.randn(n, c, t, h, w, generator=g, device=DEV)
    hh = torch.randn(n, c, t, h, w, generator=g, device=DEV)
    s[:, :2] *= 150                                    # reach the clamp in a few channels
    b = torch.randn(c, generator=g, device=DEV) * 0.3
    return s.to(dtype), hh.to(dtype), b.to(dtype)


def _call(s, h, b, sig, act='lrelu', clamp=CLAMP):
    _, _, _, _, tup, sup, to, ho, wo = sig
    return gt.gblock_tail(s, h, b, temporal_up=tup, spatial_up=sup, seq_length=to, height=ho, width=wo, act=act, clamp=clamp)


def _rel(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


@pytest.mark.parametrize('sig', BLOCKS, ids=IDS)
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_forward_and_codes_match_float64(sig, dtype):
    c, t, h, w, tup, sup, to, ho, wo = sig
    s, hh, b = _inputs(8, c, t, h, w, dtype)
    plug = custom_ops.get_plugin('gblock_tail_plugin')
    flags = (gt.TUP if tup else 0) | (gt.SUP if sup else 0)
    z, codes = plug.forward(s, hh, b.float(), (to, ho, wo), flags, 3, 0.2, math.sqrt(2), CLAMP, True)
    v = _lin64((s.double() + hh.double()) * math.sqrt(0.5), tup, sup, to, ho, wo) + b.double().view(1, -1, 1, 1, 1)
    del s, hh
    y = torch.where(v > 0, v, 0.2 * v) * math.sqrt(2)
    ref = y.clamp(-CLAMP, CLAMP)
    if dtype == torch.float32:
        assert (z.double() - ref).abs().max() <= 2e-6 * ref.abs().max()
    else:
        # fp16 storage: one rounding of the result (2^-11 relative) plus fp16 inputs
        assert ((z.double() - ref).abs() <= ref.abs() * 2 ** -10 + 2e-3).all()
    # the codes against the float64 decision, away from the decision boundaries
    code = gt._decode_codes(codes, z.numel(), dtype).view(z.shape)
    # fp32: within the forward's tolerance; fp16: the one rounding of the stored value (2^-11 relative) moves no element
    # that far from 0 across it and none that far from the clamp onto it
    tz, tc = (2e-6 * float(ref.abs().max()),) * 2 if dtype == torch.float32 else (1e-6, CLAMP * 2 ** -10)
    certain = (y.abs() > tz) & ((y.abs() - CLAMP).abs() > tc)
    want = (~(y > 0)).long() | ((y.abs() >= CLAMP).long() << 1)
    assert torch.equal(code[certain], want[certain])
    assert certain.float().mean() > 0.99


@pytest.mark.parametrize('sig', BLOCKS, ids=IDS)
def test_adjoint_matches_float64(sig):
    c, t, h, w, tup, sup, to, ho, wo = sig
    n = 8 if c * t * h * w <= 128 * 160 * 18 * 32 else 4
    s, hh, b = _inputs(n, c, t, h, w, torch.float32, seed=1)
    s.requires_grad_(True)
    hh.requires_grad_(True)
    b.requires_grad_(True)
    z = _call(s, hh, b, sig)
    dz = torch.randn(z.shape, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV)
    ds, dh, db = torch.autograd.grad(z, [s, hh, b], dz)
    assert ds.data_ptr() == dh.data_ptr()                        # one tensor for both
    # float64: dv from the forward's codes, then the transposed linear map
    _, codes = custom_ops.get_plugin('gblock_tail_plugin').forward(s.detach(), hh.detach(), b.detach(), (to, ho, wo),
                                                                   (gt.TUP if tup else 0) | (gt.SUP if sup else 0), 3, 0.2,
                                                                   math.sqrt(2), CLAMP, True)
    code = gt._decode_codes(codes, z.numel(), torch.float32).view(z.shape)
    dv = dz.double() * torch.where((code & 1).bool(), 0.2, 1.0).double() * math.sqrt(2) * (code < 2).double()
    x0 = torch.zeros(s.shape, dtype=torch.float64, device=DEV, requires_grad=True)
    dm = torch.autograd.grad(_lin64(x0, tup, sup, to, ho, wo), [x0], dv)[0] * math.sqrt(0.5)
    assert _rel(ds, dm) <= 1e-5
    assert _rel(db, dv.sum((0, 2, 3, 4))) <= 1e-5


SMALL = [(1, 3, 3, 5, True, True, 5, 5, 9), (1, 4, 3, 3, True, False, 7, 3, 3), (1, 3, 4, 5, False, True, 2, 7, 7),
         (1, 5, 2, 6, False, False, 3, 2, 5), (1, 2, 3, 4, True, True, 4, 6, 8)]


@pytest.mark.parametrize('sig', SMALL)
def test_adjoint_matrix_is_the_transpose_of_the_forward_matrix(sig):
    c, t, h, w, tup, sup, to, ho, wo = sig
    plug = custom_ops.get_plugin('gblock_tail_plugin')
    flags = (gt.TUP if tup else 0) | (gt.SUP if sup else 0)
    k_in, k_out = t * h * w, to * ho * wo
    eye_in = torch.eye(k_in, device=DEV).view(k_in, 1, t, h, w)
    fwd, _ = plug.forward(eye_in, torch.zeros_like(eye_in), None, (to, ho, wo), flags, 1, 0.0, 1.0, -1.0, False)
    a = fwd.reshape(k_in, k_out).t()                              # column j = forward of basis vector j
    eye_out = torch.eye(k_out, device=DEV).view(k_out, 1, to, ho, wo)
    _, codes = plug.forward(torch.ones(k_out, 1, t, h, w, device=DEV), torch.zeros(k_out, 1, t, h, w, device=DEV), None,
                            (to, ho, wo), flags, 1, 0.0, 1.0, -1.0, True)
    adj, db = plug.adjoint(eye_out, codes, (t, h, w), flags, 1, 0.0, 1.0)
    at = adj.reshape(k_out, k_in)                                 # row i = adjoint of basis vector i
    assert torch.allclose(at, a, atol=1e-7, rtol=0)
    assert torch.equal(db, torch.ones(1, device=DEV) * k_out)
    # and both against the float64 matrix of the map
    a64 = _lin64(torch.eye(k_in, dtype=torch.float64, device=DEV).view(k_in, 1, t, h, w), tup, sup, to, ho, wo)
    assert torch.allclose(a.double(), a64.reshape(k_in, k_out).t() * math.sqrt(0.5), atol=1e-7, rtol=0)


_G = 64     # guard elements before and after every output


def _guarded(numel, dtype, fill):
    buf = torch.full([numel + 2 * _G], fill, dtype=dtype, device=DEV)
    return buf, buf[_G:_G + numel]


@pytest.mark.parametrize('sig', [BLOCKS[1], BLOCKS[5], (8, 5, 3, 5, True, True, 7, 5, 9), (6, 4, 3, 3, False, True, 4, 5, 5)])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_no_stray_writes(sig, dtype):
    c, t, h, w, tup, sup, to, ho, wo = sig
    lib = custom_ops.load_library()
    code = 0 if dtype == torch.float32 else 1
    flags = (gt.TUP if tup else 0) | (gt.SUP if sup else 0)
    s, hh, b = _inputs(2, c, t, h, w, dtype)
    nz = 2 * c * to * ho * wo
    zbuf, z = _guarded(nz, dtype, 7.0)
    ncode = int(lib.lvg_bias_act_codes_bytes(code, nz))
    cbuf, codes = _guarded(ncode, torch.uint8, 0xA5)
    stream = torch.cuda.current_stream().cuda_stream
    rc = lib.lvg_gblock_tail(s.data_ptr(), hh.data_ptr(), b.float().data_ptr(), z.data_ptr(), codes.data_ptr(), code, 2, c, t, h, w,
                             to, ho, wo, flags, 3, 0.2, math.sqrt(2), CLAMP, ctypes.c_void_p(stream))
    assert rc == 0
    ref = _call(s, hh, b, sig)
    assert torch.equal(z, ref.flatten())
    assert (zbuf[:_G] == 7).all() and (zbuf[-_G:] == 7).all()
    assert (cbuf[:_G] == 0xA5).all() and (cbuf[-_G:] == 0xA5).all()
    dz = torch.randn(nz, device=DEV).to(dtype)
    nm = 2 * c * t * h * w
    mbuf, dm = _guarded(nm, dtype, 7.0)
    bbuf, db = _guarded(c, torch.float32, 7.0)
    nws = int(lib.lvg_gblock_tail_workspace(2, c, t, h, w, to, ho, wo, flags))
    wbuf, ws = _guarded(nws // 4, torch.float32, 7.0)
    rc = lib.lvg_gblock_tail_adjoint(dz.data_ptr(), codes.data_ptr(), dm.data_ptr(), db.data_ptr(), ws.data_ptr(), nws, code, 2, c, t,
                                     h, w, to, ho, wo, flags, 3, 0.2, math.sqrt(2), ctypes.c_void_p(stream))
    assert rc == 0
    torch.cuda.synchronize()
    for buf in (mbuf, bbuf, wbuf):
        assert (buf[:_G] == 7).all() and (buf[-_G:] == 7).all()
    assert torch.isfinite(dm).all() and torch.isfinite(db).all()


@pytest.mark.parametrize('sig', [BLOCKS[3], BLOCKS[8]], ids=['b3', 'b8'])
def test_bitwise_reproducible_and_graph_capture(sig):
    c, t, h, w, *_ = sig
    s, hh, b = _inputs(4, c, t, h, w, torch.float32, seed=3)
    dz = torch.randn(_call(s, hh, b, sig).shape, generator=torch.Generator(device=DEV).manual_seed(4), device=DEV)

    def step():
        si, hi, bi = s.clone().requires_grad_(True), hh.clone().requires_grad_(True), b.clone().requires_grad_(True)
        z = _call(si, hi, bi, sig)
        gs, gb = torch.autograd.grad(z, [si, bi], dz)
        return z.detach(), gs, gb
    runs = [step() for _ in range(2)]
    for a, bb in zip(*runs):
        assert torch.equal(a, bb)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, bb in zip(outs, runs[0]):
        assert torch.equal(a, bb)


def test_double_backward_matches_the_composition():
    sig = (6, 4, 3, 5, True, True, 7, 5, 9)
    c, t, h, w, *_ = sig
    s, hh, b = _inputs(2, c, t, h, w, torch.float32, seed=5)
    outs = []
    for native in (True, False):
        si, bi = s.clone().requires_grad_(True), b.clone().requires_grad_(True)
        if native:
            z = _call(si, hh, bi, sig)
        else:
            z = gt._reference(si, hh, bi, True, True, 7, 5, 9, 'lrelu', CLAMP)
        gs, = torch.autograd.grad(z.square().sum(), [si], create_graph=True)
        gg = torch.autograd.grad(gs.square().sum(), [si, bi])
        outs.append((gs.detach(),) + gg)
    for a, bb in zip(*outs):
        assert _rel(a, bb) <= 1e-5


# ---- the unmodified generator with install()

@pytest.fixture(scope='module')
def gen(tmp_path_factory):
    if not os.path.isdir(os.path.join(SRC, 'model')):
        pytest.skip('oracle/_ref not staged')
    out = str(tmp_path_factory.mktemp('gblock') / 'cuda.pt')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'gblock_tail_run.py'), out, 'cuda'], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out, weights_only=False)


# the tolerances of tests/test_gpu_modconv.py (and test_gpu_dropin_cuda.py)
@pytest.mark.parametrize('beta', [1.0, 0.999])
@pytest.mark.parametrize('key,tol_max,tol_l2', [('v', 1e-3, 5e-4), ('g', 3e-2, 2e-2)])
def test_generator_with_install_matches_without(gen, beta, key, tol_max, tol_l2):
    ref, ours = gen[beta]
    a, b = ours[key].double(), ref[key].double()
    assert a.shape == b.shape and torch.isfinite(a).all()
    emax, el2 = float((a - b).abs().max() / b.abs().max()), float((a - b).norm() / b.norm())
    assert emax <= tol_max and el2 <= tol_l2, f'{key}: max {emax:.3e}, L2 {el2:.3e}'


@pytest.mark.parametrize('beta', [1.0, 0.999])
def test_generator_state_and_rng_after_install(gen, beta):
    ref, ours = gen[beta]
    assert torch.equal(ref['cpu_rng'], ours['cpu_rng']) and torch.equal(ref['cuda_rng'], ours['cuda_rng'])
    assert len(ref['bufs']) == len(ours['bufs'])
    for a, b in zip(ours['bufs'], ref['bufs']):
        assert torch.allclose(a, b, rtol=1e-5, atol=0), float((a - b).abs().max())
    if beta == 1.0:
        assert all(torch.equal(a, b) for a, b in zip(ours['bufs'], ref['bufs']))


def test_generator_with_install_makes_no_host_sync(gen):
    assert gen['nosync'] is True, gen['nosync']


def test_profiler_sees_the_kernels_and_fewer_generic_ops(gen):
    ours, ref = gen['prof_ours'], gen['prof_ref']
    k = lambda names, part: sum(v for n, v in names.items() if part in n)      # noqa: E731
    assert k(ours, 'gblock_tail_fwd_kernel') == 10 and k(ours, 'gblock_tail_adj_kernel') == 10
    assert k(ours, 'gblock_tail_fold_kernel') == 10 and k(ref, 'gblock_tail') == 0
    # the reference's tails run an ATen add per block forward and a slice_backward per crop backward, and upfirdn2d for
    # their upsamplings; installed, the crops of the latents (compute_latent_ws) are what is left of slice_backward
    assert k(ref, 'aten::slice_backward') - k(ours, 'aten::slice_backward') >= 7
    assert k(ref, 'aten::add') - k(ours, 'aten::add') >= 10
    assert k(ours, 'upfirdn2d') < k(ref, 'upfirdn2d')
