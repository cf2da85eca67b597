"""The discriminator-block tail (torch_utils/ops/dblock_tail.py, csrc/dblock_tail.cu) on the GPU: exact arithmetic over every
down-sampling subset and the tile edges, random inputs at the four block shapes of the default low-res D at batch 8 against
float64, guard bands around every output, the adjoint as the transpose of the read-mode forward, bitwise reproducibility,
CUDA-graph capture, every instantiated kernel seen by torch.profiler, and the unmodified VideoDiscriminator with install()
against the same network without it."""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import dblock_tail as dt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
DEV = torch.device('cuda')
P = custom_ops.DblockTailPlugin
SQH = float(torch.tensor(0.5).sqrt())                 # sqrt(1/2) rounded to float32, the kernels' constant
TAPS = (0.125, 0.375, 0.375, 0.125)
SUBSETS = [0, P.SDOWN, P.TDOWN, P.TDOWN | P.SDOWN]


_F4 = []


def f4():
    if not _F4:
        _F4.append(torch.tensor(TAPS, device=DEV))
    return _F4[0]


def plug():
    return custom_ops.get_plugin('dblock_tail_plugin')


def down64(x, dim):
    """Downsample3d's filter along dim from the definition: out[m] = sum_j f[3 - j] in[2 m - 1 + j], zero outside."""
    n = x.shape[dim]
    xp = torch.nn.functional.pad(x, [0, 0] * (x.ndim - 1 - dim) + [1, 2])
    idx = [slice(None)] * x.ndim
    acc = 0
    for j in range(4):
        idx[dim] = slice(j, j + n - 1, 2)
        acc = acc + TAPS[3 - j] * xp[tuple(idx)]
    return acc


def p64(x, flags):
    if flags & P.SDOWN:
        x = down64(down64(x, 3), 4)
    if flags & P.TDOWN:
        x = down64(x, 2)
    return x


def pt64(dv, in_shape, flags):
    """P^T dv in float64 (autograd of the definition)."""
    with torch.enable_grad():
        x0 = torch.zeros(in_shape, dtype=torch.float64, device=DEV, requires_grad=True)
        return torch.autograd.grad(p64(x0, flags), [x0], dv)[0]


def decode(codes, shape):
    """The 2-bit code of every output from the layout of lvg_dblock_tail: one byte per 4 outputs along W, padded rows."""
    w = shape[-1]
    rows = codes.view(-1, (w + 3) // 4).long()
    c = torch.stack([(rows >> (2 * k)) & 3 for k in range(4)], -1).flatten(1)[:, :w]
    return c.reshape(shape)


def slope64(code, alpha, gain):
    return torch.where(code >= 2, 0.0, torch.where((code & 1).bool(), alpha * gain, gain)).double()


def r32(x):
    return x.float().double()


def sparse_ints(shape, seed, density=0.3, hi=3):
    g = torch.Generator(device=DEV).manual_seed(seed)
    v = torch.randint(-hi, hi + 1, shape, generator=g, device=DEV).double()
    return v * (torch.rand(shape, generator=g, device=DEV) < density)


OUTS = [(1, 7, 1), (2, 8, 4), (2, 9, 31), (1, 8, 32), (2, 9, 33), (3, 17, 70)]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16], ids=['fp32', 'fp16'])
@pytest.mark.parametrize('out', OUTS, ids=[f'{a}x{b}x{c}' for a, b, c in OUTS])
@pytest.mark.parametrize('flags', SUBSETS)
@pytest.mark.parametrize('act,gain', [('lrelu', 2.0), ('linear', 1.0)])
def test_exact_arithmetic(flags, out, dtype, act, gain):
    """Inputs on which every fp32 operation of the kernels is exact except the final multiplication by sqrt(1/2), which
    rounds once: small sparse integers, the taps (1, 3, 3, 1) / 8, dyadic b, alpha, gain and clamp. The results must equal
    the float64 evaluation element for element."""
    n, c = 2, 3
    alpha, clamp = 0.25, 2.0
    to, ho, wo = out
    t, h, w = to * (2 if flags & P.TDOWN else 1), ho * (2 if flags & P.SDOWN else 1), wo * (2 if flags & P.SDOWN else 1)
    y = sparse_ints((n, c, t, h, w), 1)
    s = sparse_ints((n, c, to, ho, wo), 2, density=0.6)
    b = torch.tensor([0.5, -0.25, 0.0], device=DEV, dtype=torch.float64)
    a_eff = alpha if act == 'lrelu' else 1.0
    for merge in (True, False):
        fl = flags | (P.MERGE if merge else 0)
        scale = SQH if merge else 1.0
        x = p64(y, flags) + b.view(1, -1, 1, 1, 1)
        o = torch.where(x > 0, x, x * a_eff) * gain
        assert torch.equal(r32(x), x) and torch.equal(r32(o), o) and torch.equal(o.to(dtype).double(), o)      # precondition
        want_code = (~(o > 0)).long() | ((~(o.abs() < clamp)).long() << 1)
        o = o.clamp(-clamp, clamp)
        pre = o + s if merge else o
        assert torch.equal(r32(pre), pre)
        want = (pre * scale).float().to(dtype)
        yy, ss = y.to(dtype), (s.to(dtype) if merge else None)
        y0, s0 = yy.clone(), (None if ss is None else ss.clone())
        z, codes = plug().forward(yy, ss, b.float(), f4(), fl, dt._ACTS[act], alpha, gain, clamp, P.WRITE)
        z_none, none = plug().forward(yy, ss, b.float(), f4(), fl, dt._ACTS[act], alpha, gain, clamp, P.NONE)
        assert none is None and torch.equal(z, want) and torch.equal(z_none, want)
        assert codes.numel() == custom_ops.load_library().lvg_dblock_tail_codes_bytes(n, c, t, h, w, fl)
        code = decode(codes, z.shape)
        assert torch.equal(code, want_code)
        assert {int(v) for v in want_code.unique()} >= ({0, 1, 2} if flags == 0 and out == OUTS[-1] else {0, 1})
        # the read-mode map on other inputs
        u, sig = sparse_ints((n, c, t, h, w), 3), sparse_ints((n, c, to, ho, wo), 4)
        G = slope64(code, a_eff, gain)
        lin = G * (p64(u, flags) + b.view(1, -1, 1, 1, 1))
        lin = lin + sig if merge else lin
        assert torch.equal(r32(lin), lin)
        zr, _ = plug().forward(u.to(dtype), sig.to(dtype) if merge else None, b.float(), f4(), fl, dt._ACTS[act], alpha, gain, -1.0,
                               P.READ, codes)
        assert torch.equal(zr, (lin * scale).float().to(dtype))
        # the adjoint: ds rounds once; dy and db are exact without the merge's sqrt(1/2), and within fp32 rounding with it
        dz = sparse_ints((n, c, to, ho, wo), 5, density=0.5, hi=2)
        d = (dz * scale).float().double()
        dv = d * G
        dy64, db64 = pt64(dv, (n, c, t, h, w), flags), dv.sum((0, 2, 3, 4))
        dzz = dz.to(dtype)
        dz0 = dzz.clone()
        dy, ds, db = plug().adjoint(dzz, codes, f4(), (t, h, w), fl, dt._ACTS[act], alpha, gain, merge)
        if merge:
            assert torch.equal(ds, d.float().to(dtype))
            assert (dy.double() - dy64).abs().max() <= (1e-6 if dtype == torch.float32 else 1e-3) * max(1.0, float(dy64.abs().max()))
            assert (db.double() - db64).abs().max() <= 1e-5 * max(1.0, float(db64.abs().max()))
        else:
            assert ds is None
            assert torch.equal(r32(dy64), dy64)                                                                 # precondition
            assert torch.equal(dy, dy64.to(dtype)) and torch.equal(db, db64.float())
        assert torch.equal(yy, y0) and torch.equal(dzz, dz0) and (ss is None or torch.equal(ss, s0))


# y of conv_1 in the four blocks of VideoDiscriminator(seq_length=128, max_edge=64) at batch 8: (C, T, H, W, flags)
BLOCKS = [(64, 128, 64, 64, P.SDOWN), (128, 128, 32, 32, P.TDOWN | P.SDOWN), (256, 64, 16, 16, P.TDOWN | P.SDOWN),
          (512, 32, 8, 8, P.TDOWN | P.SDOWN)]
IDS = [f'b{i}' for i in range(4)]


def _inputs(n, c, t, h, w, flags, dtype, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    y = torch.randn(n, c, t, h, w, generator=g, device=DEV)
    y[:, :2] *= 400                                     # reach the clamp in a few channels
    s = torch.randn(n, c, *P.out_size((t, h, w), flags), generator=g, device=DEV)
    b = torch.randn(c, generator=g, device=DEV) * 0.3
    return y.to(dtype), s.to(dtype), b.to(dtype)


def _call(y, s, b, flags, **kw):
    return dt.dblock_tail(y, s, b, f4(), spatial_down=bool(flags & P.SDOWN), temporal_down=bool(flags & P.TDOWN), **kw)


def _rel(a, b):
    return float((a.detach().double() - b.detach().double()).abs().max() / b.detach().double().abs().max())


@pytest.mark.parametrize('sig', BLOCKS, ids=IDS)
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16], ids=['fp32', 'fp16'])
def test_block_shapes_match_float64(sig, dtype):
    c, t, h, w, flags = sig
    y, s, b = _inputs(8, c, t, h, w, flags, dtype)
    y.requires_grad_(True), s.requires_grad_(True), b.requires_grad_(True)
    z = _call(y, s, b, flags)
    dz = torch.randn(z.shape, generator=torch.Generator(device=DEV).manual_seed(2), device=DEV).to(dtype)
    dy, ds, db = torch.autograd.grad(z, [y, s, b], dz)
    gain = math.sqrt(2)
    x = p64(y.detach().double(), flags) + b.detach().double().view(1, -1, 1, 1, 1)
    o = (torch.where(x > 0, x, 0.2 * x) * gain).clamp(-256, 256)
    assert (o.abs() == 256).any()
    ref = (o + s.detach().double()) * math.sqrt(0.5)
    del x, o
    assert _rel(z, ref) <= (1e-3 if dtype == torch.float32 else 4e-3)
    del ref
    # gradients through the decisions the kernel took (its codes), in float64
    _, codes = plug().forward(y.detach(), s.detach(), b.detach(), f4(), flags | P.MERGE, 3, 0.2, gain, 256.0, P.WRITE)
    dv = dz.double() * math.sqrt(0.5) * slope64(decode(codes, z.shape), 0.2, gain)
    tol = 1e-2 if dtype == torch.float32 else 4e-3
    assert _rel(db, dv.sum((0, 2, 3, 4))) <= tol
    assert _rel(ds, dz.double() * math.sqrt(0.5)) <= tol
    want = pt64(dv, y.shape, flags)
    assert _rel(dy, want) <= tol


_G = 64     # guard elements before and after every output


def _guarded(numel, dtype, fill):
    buf = torch.full([numel + 2 * _G], fill, dtype=dtype, device=DEV)
    return buf, buf[_G:_G + numel]


@pytest.mark.parametrize('shape,flags', [((2, 5, 6, 18, 66), P.SDOWN), ((2, 5, 6, 18, 66), P.TDOWN | P.SDOWN), ((3, 2, 5, 9, 33), 0),
                                         ((1, 4, 8, 7, 5), P.TDOWN)])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16], ids=['fp32', 'fp16'])
def test_no_stray_writes(shape, flags, dtype):
    n, c, t, h, w = shape
    fl = flags | P.MERGE
    lib = custom_ops.load_library()
    dcode = 0 if dtype == torch.float32 else 1
    y, s, b = _inputs(n, c, t, h, w, flags, dtype)
    b = b.float()
    f = f4()
    y0, s0 = y.clone(), s.clone()
    nz = s.numel()
    zbuf, z = _guarded(nz, dtype, 7.0)
    ncode = int(lib.lvg_dblock_tail_codes_bytes(n, c, t, h, w, fl))
    cbuf, codes = _guarded(ncode, torch.uint8, 0xA5)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rc = lib.lvg_dblock_tail(y.data_ptr(), s.data_ptr(), b.data_ptr(), f.data_ptr(), z.data_ptr(), codes.data_ptr(), P.WRITE, dcode,
                             n, c, t, h, w, fl, 3, 0.2, math.sqrt(2), 256.0, stream)
    assert rc == 0
    ref = _call(y, s, b, flags)
    assert torch.equal(z, ref.flatten())
    assert (zbuf[:_G] == 7).all() and (zbuf[-_G:] == 7).all()
    assert (cbuf[:_G] == 0xA5).all() and (cbuf[-_G:] == 0xA5).all()
    z2buf, z2 = _guarded(nz, dtype, 7.0)
    rc = lib.lvg_dblock_tail(y.data_ptr(), s.data_ptr(), b.data_ptr(), f.data_ptr(), z2.data_ptr(), codes.data_ptr(), P.READ, dcode,
                             n, c, t, h, w, fl, 3, 0.2, math.sqrt(2), -1.0, stream)
    assert rc == 0 and (z2buf[:_G] == 7).all() and (z2buf[-_G:] == 7).all() and torch.isfinite(z2).all()
    codes0 = codes.clone()
    dz = torch.randn(nz, device=DEV).to(dtype)
    dz0 = dz.clone()
    ybuf, dy = _guarded(y.numel(), dtype, 7.0)
    sbuf, ds = _guarded(nz, dtype, 7.0)
    bbuf, db = _guarded(c, torch.float32, 7.0)
    nws = int(lib.lvg_dblock_tail_workspace(n, c, t, h, w, fl))
    wbuf, ws = _guarded(nws // 4, torch.float32, 7.0)
    rc = lib.lvg_dblock_tail_adjoint(dz.data_ptr(), codes.data_ptr(), f.data_ptr(), dy.data_ptr(), ds.data_ptr(), db.data_ptr(),
                                     ws.data_ptr(), nws, dcode, n, c, t, h, w, fl, 3, 0.2, math.sqrt(2), stream)
    assert rc == 0
    torch.cuda.synchronize()
    for buf in (ybuf, sbuf, bbuf, wbuf):
        assert (buf[:_G] == 7).all() and (buf[-_G:] == 7).all()
    for out in (dy, ds, db):
        assert torch.isfinite(out).all() and not (out == 7).all()
    assert torch.equal(y, y0) and torch.equal(s, s0) and torch.equal(dz, dz0) and torch.equal(codes, codes0)


@pytest.mark.parametrize('flags', SUBSETS)
def test_adjoint_matrix_is_the_transpose_of_the_read_mode_matrix(flags):
    t, h, w = 4, 6, 10
    to, ho, wo = P.out_size((t, h, w), flags)
    k_in, k_out = t * h * w, to * ho * wo
    y = torch.randn(1, 1, t, h, w, generator=torch.Generator(device=DEV).manual_seed(7), device=DEV) * 2
    _, codes1 = plug().forward(y, None, None, f4(), flags | P.MERGE, 3, 0.2, 2.0, 1.0, P.WRITE)
    assert {int(v) for v in decode(codes1, (1, 1, to, ho, wo)).unique()} >= {0, 1, 2}
    fwd, _ = plug().forward(torch.eye(k_in, device=DEV).view(k_in, 1, t, h, w), None, None, f4(), flags | P.MERGE, 3, 0.2, 2.0, -1.0,
                            P.READ, codes1.repeat(k_in))
    a = fwd.reshape(k_in, k_out).t()                              # column j = the map of basis vector j
    adj, ds, db = plug().adjoint(torch.eye(k_out, device=DEV).view(k_out, 1, to, ho, wo), codes1.repeat(k_out), f4(), (t, h, w),
                                 flags | P.MERGE, 3, 0.2, 2.0, True)
    at = adj.reshape(k_out, k_in)                                 # row i = the adjoint of basis vector i
    assert torch.allclose(at, a, atol=1e-7, rtol=0) and float(a.abs().max()) > 0.05
    assert torch.equal(ds.reshape(k_out, k_out), torch.eye(k_out, device=DEV) * SQH)
    G = slope64(decode(codes1, (to, ho, wo)), 0.2, 2.0).flatten()
    assert torch.allclose(db.double(), (G * SQH).sum().view(1), rtol=1e-4)       # an fp32 sum of k_out terms
    a64 = p64(torch.eye(k_in, dtype=torch.float64, device=DEV).view(k_in, 1, t, h, w), flags).reshape(k_in, k_out).t()
    assert torch.allclose(a.double(), a64 * G.view(-1, 1) * SQH, atol=1e-6, rtol=0)


def _three_steps(y, s, b, flags, dz):
    """forward, forward + backward and the R1 pattern."""
    with torch.no_grad():
        z0 = _call(y, s, b, flags)
    yi, si, bi = (v.clone().requires_grad_(True) for v in (y, s, b))
    z = _call(yi, si, bi, flags)
    first = torch.autograd.grad(z, [yi, si, bi], dz)
    yi, si, bi = (v.clone().requires_grad_(True) for v in (y, s, b))
    z = _call(yi, si, bi, flags)
    gy, gs = torch.autograd.grad(z.square().sum(), [yi, si], create_graph=True)
    second = torch.autograd.grad(gy.square().sum() + gs.square().sum() + z.sum(), [yi, si, bi])
    return (z0, z.detach(), gy.detach(), gs.detach()) + first + second


@pytest.mark.parametrize('sig', [(32, 16, 64, 64, P.SDOWN), (64, 16, 32, 32, P.TDOWN | P.SDOWN)], ids=['s', 'ts'])
def test_bitwise_reproducible_deterministic_mode_and_graph_capture(sig):
    c, t, h, w, flags = sig
    y, s, b = _inputs(4, c, t, h, w, flags, torch.float32, seed=3)
    dz = torch.randn(s.shape, generator=torch.Generator(device=DEV).manual_seed(4), device=DEV)
    runs = [_three_steps(y, s, b, flags, dz) for _ in range(2)]
    torch.use_deterministic_algorithms(True)
    try:
        runs.append(_three_steps(y, s, b, flags, dz))
    finally:
        torch.use_deterministic_algorithms(False)
    for other in runs[1:]:
        for a, bb in zip(runs[0], other):
            assert torch.equal(a, bb)

    def step():
        yi, si, bi = (v.clone().requires_grad_(True) for v in (y, s, b))
        z = _call(yi, si, bi, flags)
        return (z.detach(),) + torch.autograd.grad(z, [yi, si, bi], dz)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = step()
    graph.replay()
    torch.cuda.synchronize()
    for a, bb in zip(outs, eager):
        assert torch.equal(a, bb)


def test_higher_order_matches_the_composition():
    flags = P.TDOWN | P.SDOWN
    y, s, b = _inputs(2, 6, 8, 12, 20, flags, torch.float32, seed=5)
    outs = []
    for native in (True, False):
        yi, si, bi = (v.clone().requires_grad_(True) for v in (y, s, b))
        z = _call(yi, si, bi, flags) if native else dt._reference(yi, si, bi, f4(), True, True, 'lrelu', 256.0)
        gy, gs = torch.autograd.grad(z.square().sum(), [yi, si], create_graph=True)
        gg = torch.autograd.grad(gy.square().sum() + gs.square().sum() + z.sum(), [yi, si, bi])
        outs.append((z.detach(), gy.detach(), gs.detach()) + gg)
    for a, bb in zip(*outs):
        assert _rel(a, bb) <= 1e-5


def test_plain_layer_tail_without_skip_and_the_fallbacks():
    y, s, b = _inputs(2, 4, 6, 10, 12, P.SDOWN, torch.float32, seed=6)
    z = _call(y, None, b, P.SDOWN, act='linear', clamp=None)
    assert _rel(z, p64(y.double(), P.SDOWN) + b.double().view(1, -1, 1, 1, 1)) <= 1e-6
    none = dict(spatial_down=False, temporal_down=False)                       # no axis filtered: the taps may be absent
    assert torch.equal(dt.dblock_tail(y, None, b, None, **none), dt.dblock_tail(y, None, b, f4(), **none))
    odd = y[:, :, :, :9]                                   # odd extent on a halved axis: the composition takes the call
    assert torch.equal(_call(odd, None, b, P.SDOWN), dt._reference(odd, None, b, f4(), True, False, 'lrelu', 256.0))
    assert _call(y.double(), s.double(), b.double(), P.SDOWN).dtype == torch.float64
    assert _rel(_call(y, s, b, P.SDOWN, act='relu'), dt._reference(y, s, b, f4(), True, False, 'relu', 256.0)) == 0


def test_profiler_sees_every_instantiated_kernel():
    def cases():
        for dtype in (torch.float32, torch.float16):
            y, s, b = _inputs(1, 3, 4, 8, 12, P.SDOWN, dtype)
            with torch.no_grad():
                _call(y, s, b, P.SDOWN)                                                     # none
            for s_grad in (True, False):
                yi, si, bi = y.clone().requires_grad_(True), s.clone().requires_grad_(s_grad), b.clone().requires_grad_(True)
                z = _call(yi, si, bi, P.SDOWN)                                              # write
                gy, = torch.autograd.grad(z.float().square().sum(), [yi], create_graph=True)    # adjoint with / without ds
                gy.float().square().sum().backward()                                        # read
        torch.cuda.synchronize()
    cases()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        cases()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and 'dblock_tail' in e.name}
    assert len({n for n in names if 'dblock_tail_fwd_kernel' in n}) == 6, names     # 2 dtypes x none / write / read
    assert len({n for n in names if 'dblock_tail_adj_kernel' in n}) == 4, names     # 2 dtypes x with / without ds
    assert len({n for n in names if 'dblock_tail_fold_kernel' in n}) == 1, names


# ---- the unmodified discriminator with install()

@pytest.fixture(scope='module')
def disc(tmp_path_factory):
    if not os.path.isdir(os.path.join(SRC, 'model')):
        pytest.skip('oracle/_ref not staged')
    out = str(tmp_path_factory.mktemp('dblock') / 'cuda.pt')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'dblock_tail_run.py'), out, 'cuda'], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-3000:]
    return torch.load(out, weights_only=False)


# fp32. Without tail=True, install() moves bias_act into the convolution's epilogue in calls that record no gradient (the
# no-grad logits) and nothing else: every tensor within 1e-5 of its largest magnitude. With every block on the op as well the two paths filter in different orders, so a pre-activation
# within rounding of zero can take the other lrelu slope: the output is continuous there, a gradient changes locally by up
# to its own size. Measured on an H100 (this network, seed and input), max / L2 error relative to the tensor: logits
# 1.2e-5 / 9.2e-6, gx 5.4e-3 / 2.2e-4, grad 2.5e-6 / 2.1e-6, r1_gx 5.4e-3 / 2.2e-4; the bounds are about four times that.
@pytest.mark.parametrize('key', ['logits', 'gx', 'grad', 'r1_gx', 'nograd_logits'])
def test_discriminator_with_the_epilogue_layers_matches_without_fp32(disc, key):
    a, b = disc['fp32_epilogue'][key], disc['fp32_ref'][key]
    assert a.shape == b.shape and torch.isfinite(a).all() and float(b.abs().max()) > 0
    assert float((a - b).abs().max()) <= 1e-5 * float(b.abs().max()), float((a - b).abs().max() / b.abs().max())
    n_epi, n_epi_grad, n_blocks = disc['calls_epilogue']
    assert disc['bitwise_epilogue'] is True and n_epi > 0 and n_epi_grad == 0 and n_blocks == 0


TAIL_TOL = {'logits': (5e-5, 4e-5), 'gx': (2e-2, 1e-3), 'grad': (1e-5, 1e-5), 'r1_gx': (2e-2, 1e-3)}


@pytest.mark.parametrize('key', ['logits', 'gx', 'grad', 'r1_gx'])
def test_discriminator_with_install_matches_without_fp32(disc, key):
    a, b = disc['fp32_ours'][key], disc['fp32_ref'][key]
    assert a.shape == b.shape and torch.isfinite(a).all() and float(b.abs().max()) > 0
    emax, el2 = float((a - b).abs().max() / b.abs().max()), float((a - b).norm() / b.norm())
    tol_max, tol_l2 = TAIL_TOL[key]
    assert emax <= tol_max and el2 <= tol_l2, f'{key}: max {emax:.3e}, L2 {el2:.3e}'
    assert disc['bitwise_ours'] is True


# fp16 blocks (num_fp16_res=4): as close to the fp32 network as the same fp16 network without install is (the tolerance of
# tests/test_gpu_dropin_cuda.py)
@pytest.mark.parametrize('key', ['logits', 'gx', 'grad', 'r1_gx'])
def test_discriminator_with_install_matches_without_fp16(disc, key):
    t, a, r = disc['fp32_ref'][key], disc['fp16_ours'][key], disc['fp16_ref'][key]
    assert a.shape == t.shape and torch.isfinite(a).all()
    e_ours, e_ref = float((a - t).norm() / t.norm()), float((r - t).norm() / t.norm())
    m_ours, m_ref = float((a - t).abs().max() / t.abs().max()), float((r - t).abs().max() / t.abs().max())
    assert e_ours <= 1.5 * e_ref + 2e-3, f'{key}: L2 error vs fp32 {e_ours:.3e} (without install: {e_ref:.3e})'
    assert m_ours <= 1.5 * m_ref + 5e-3, f'{key}: max error vs fp32 {m_ours:.3e} (without install: {m_ref:.3e})'


def test_discriminator_runs_the_kernels(disc):
    assert disc['calls_ours'][2] > 0 and disc['calls_ours'][0] > 0       # tail=True: every block on the op; without it none
    for name in ('fp32', 'fp16'):
        k = [n for n in disc[name + '_kernels'] if 'dblock_tail' in n]
        assert any('fwd_kernel' in n for n in k) and any('adj_kernel' in n for n in k) and any('fold_kernel' in n for n in k), k


# ---- conv_bias_act with create_graph=True (gradients of any order)

def _cba_inputs(dtype):
    g = torch.Generator(device=DEV).manual_seed(20)
    x = torch.randn(2, 24, 6, 9, 16, generator=g, device=DEV).to(dtype).requires_grad_(True)
    w = (torch.randn(40, 24, 3, 3, 3, generator=g, device=DEV) * 0.05).to(dtype).requires_grad_(True)
    b = torch.randn(40, generator=g, device=DEV).to(dtype).requires_grad_(True)
    return x, w, b


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16], ids=['fp32', 'fp16'])
@pytest.mark.parametrize('act,clamp', [('lrelu', 0.875), ('linear', 256), ('lrelu', None)])
def test_conv_bias_act_create_graph_matches_the_two_ops(dtype, act, clamp):
    from torch_utils.ops import bias_act, conv_nd
    x, w, b = _cba_inputs(dtype)
    outs = []
    for fused in (True, False):
        if fused:
            y = conv_nd.conv_bias_act(x, w, b, padding=(1, 1, 1), act=act, clamp=clamp)
            assert type(y.grad_fn).__name__ == '_ConvBiasActBackward'
        else:
            y = bias_act.bias_act(conv_nd.conv3d(x, w, padding=(1, 1, 1)), b, act=act, clamp=clamp)
        gx, gw, gb = torch.autograd.grad(y.float().square().sum(), [x, w, b], create_graph=True)
        # the R1 pattern; in fp16 its second-order values leave the format's range for both paths, so fp16 stops at first order
        gg = () if dtype == torch.float16 else torch.autograd.grad(
            gx.square().sum() + gw.square().sum() + gb.square().sum(), [x, w, b])
        outs.append((y.detach(), gx.detach(), gw.detach(), gb.detach()) + gg)
    tol = 1e-4 if dtype == torch.float32 else 2e-2
    for name, a, bb in zip(('y', 'gx', 'gw', 'gb', 'ggx', 'ggw', 'ggb'), *outs):
        err = float((a.double() - bb.double()).norm() / bb.double().norm())
        assert err <= tol, f'{name}: {err:.3e}'


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16], ids=['fp32', 'fp16'])
def test_conv_bias_act_first_order_is_bitwise_the_same_with_create_graph(dtype):
    from torch_utils.ops import conv_nd
    x, w, b = _cba_inputs(dtype)
    y = conv_nd.conv_bias_act(x, w, b, padding=(1, 1, 1), act='lrelu', clamp=0.875)
    dy = torch.randn(y.shape, generator=torch.Generator(device=DEV).manual_seed(23), device=DEV).to(dtype)
    plain = torch.autograd.grad(y, [x, w, b], dy, retain_graph=True)
    graph = torch.autograd.grad(y, [x, w, b], dy, create_graph=True)
    for name, a, c in zip('xwb', plain, graph):
        assert torch.equal(a, c.detach()), f'd{name}: {float((a.float() - c.detach().float()).abs().max()):.3e}'
