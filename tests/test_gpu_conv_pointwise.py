"""The pointwise wgmma kernels (csrc/conv_pw_tc.cu): every 1x1x1 forward / input gradient outside the streaming SIMT
kernels' envelope runs on them, straight from the NC(T)HW tensors.

They issue the engine's products (bf16 hi*hi, hi*lo, lo*hi per 16-channel k step for fp32; one fp16 product for fp16) in
the engine's order, so their results must equal the engine's (LVG_CONV_PW_TC=0, read on every call) bit for bit on
random operands -- over the 1x1x1 signatures of the low-res step, ragged channel counts, pixel counts that are not a
multiple of the 128-pixel tile, and samples whose last channel chunk is partial (the next sample's channels are NaN: the
3-D tensor map must zero-fill, never read across the sample). Output guards, exact-size workspaces, unchanged inputs,
the route query against the kernels the profiler sees, and CUDA-graph capture are checked too. The exact-arithmetic
checks of tests/test_gpu_conv_exact.py cover these layers as well (they run on this path by default)."""
import math
import os

import pytest
import torch

from torch_utils import custom_ops

pytestmark = pytest.mark.gpu
DEV = 'cuda'
DTYPES = [torch.float32, torch.float16]
DT_IDS = ['f32', 'f16']


@pytest.fixture(scope='module')
def plug():
    return custom_ops.get_plugin('convnd_plugin')


class engine_only:
    """LVG_CONV_PW_TC=0 inside the block: the same calls run on the implicit-GEMM engine."""

    def __enter__(self):
        self.old = os.environ.get('LVG_CONV_PW_TC')
        os.environ['LVG_CONV_PW_TC'] = '0'

    def __exit__(self, *exc):
        if self.old is None:
            del os.environ['LVG_CONV_PW_TC']
        else:
            os.environ['LVG_CONV_PW_TC'] = self.old


def operands(n, cin, cout, sp, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn((n, cin) + tuple(sp), generator=g, device=DEV).to(dtype)
    w = (torch.randn((cout, cin) + (1,) * len(sp), generator=g, device=DEV) / math.sqrt(cin)).to(dtype)
    dy = torch.randn((n, cout) + tuple(sp), generator=g, device=DEV).to(dtype)
    return x, w, dy


def pad0(nd):
    return [0] * nd


def assert_same(got, exp, what):
    assert got.shape == exp.shape and got.dtype == exp.dtype, (what, got.shape, exp.shape)
    same = (got == exp) | (torch.isnan(got) & torch.isnan(exp))
    if not bool(same.all()):
        i = int(torch.nonzero(~same.flatten())[0])
        raise AssertionError(f'{what}: {int((~same).sum())} of {got.numel()} elements differ; first at flat index {i}: '
                             f'{float(got.flatten()[i])} vs the engine\'s {float(exp.flatten()[i])}')


def both_paths(plug, x, w, dy):
    nd = x.ndim - 2
    routes = (plug.route('fprop', x.shape, w.shape, pad0(nd), 1, x.dtype), plug.route('dgrad', x.shape, w.shape, pad0(nd), 1, x.dtype))
    y = plug.fprop(x, w, pad0(nd), 1)
    dx = plug.dgrad(dy, w, x.shape, pad0(nd), 1)
    with engine_only():
        assert plug.route('fprop', x.shape, w.shape, pad0(nd), 1, x.dtype) != 'pointwise_wgmma'
        ye = plug.fprop(x, w, pad0(nd), 1)
        dxe = plug.dgrad(dy, w, x.shape, pad0(nd), 1)
    return routes, (y, dx), (ye, dxe)


def lres_pointwise_signatures():
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    tr = json.load(open(os.path.join(root, 'workloads', 'lres_step.json')))
    sigs = set()
    for net in ('lres_G', 'lres_D'):
        for c in tr[net]:
            if c['op'] == 'conv3d' and tuple(c['w'][2:]) == (1, 1, 1):
                sigs.add((tuple(c['x'][1:]), c['w'][0]))
    return sorted(sigs)


LRES = lres_pointwise_signatures()


def test_lres_signatures_exist():
    assert len(LRES) >= 8, LRES


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('sig', LRES, ids=lambda s: f'{s[0][0]}to{s[1]}_{"x".join(map(str, s[0][1:]))}')
def test_lres_signature_matches_engine(plug, sig, dtype):
    (cin, t, h, w_), cout = sig
    n = 1 if cin * t * h * w_ > 2 ** 22 else 2
    x, w, dy = operands(n, cin, cout, (t, h, w_), dtype, seed=cin * 7 + cout)
    routes, got, exp = both_paths(plug, x, w, dy)
    pitch_ok = (t * h * w_) % (4 if dtype == torch.float32 else 8) == 0     # fp16 rows of 4 mod 8 elements stay on the engine
    for r, g, e, what in zip(routes, got, exp, ('forward', 'input gradient')):
        assert r in (('simt', 'pointwise_wgmma') if pitch_ok else ('engine',)), (what, r)
        if r == 'pointwise_wgmma':
            assert_same(g, e, what)


RAGGED = [1, 3, 17, 65, 130, 257, 513]
RAGGED_PAIRS = [(a, b) for i, a in enumerate(RAGGED) for b in RAGGED[i % 3::3]]


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('cin,cout', RAGGED_PAIRS)
def test_ragged_channels_match_engine(plug, cin, cout, dtype):
    P = 328 if dtype == torch.float32 else 200               # not a multiple of the 128-pixel tile
    x, w, dy = operands(2, cin, cout, (P,), dtype, seed=cin * 1000 + cout)
    routes, got, exp = both_paths(plug, x, w, dy)
    for r, g, e, what in zip(routes, got, exp, ('forward', 'input gradient')):
        if r == 'pointwise_wgmma':
            assert_same(g, e, what)
    if dtype == torch.float16 or cin * cout > 4096:
        assert routes == ('pointwise_wgmma', 'pointwise_wgmma'), routes


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('P', [8, 120, 128, 136, 1032])
def test_pixel_edges_match_engine(plug, P, dtype):
    x, w, dy = operands(3, 70, 150, (P,), dtype, seed=P)
    routes, got, exp = both_paths(plug, x, w, dy)
    assert routes == ('pointwise_wgmma', 'pointwise_wgmma')
    for g, e, what in zip(got, exp, ('forward', 'input gradient')):
        assert_same(g, e, what)


def test_four_pixels(plug):
    x, w, dy = operands(2, 100, 90, (1, 2, 2), torch.float32, seed=4)
    routes, got, exp = both_paths(plug, x, w, dy)
    assert routes == ('pointwise_wgmma', 'pointwise_wgmma')
    for g, e, what in zip(got, exp, ('forward', 'input gradient')):
        assert_same(g, e, what)


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('cin', [17, 40, 97])
def test_partial_chunk_zero_fill(plug, cin, dtype):
    """The last 32-channel chunk of a sample runs past its channels: NaN planted in the following sample's channels must
    not reach the output."""
    n, P, cout = 3, 256, 300
    g = torch.Generator(device=DEV).manual_seed(cin)
    x = torch.randn(n, cin, P, generator=g, device=DEV).to(dtype)
    w = (torch.randn(cout, cin, 1, generator=g, device=DEV) / math.sqrt(cin)).to(dtype)
    x[1:, :] = float('nan')                        # every sample after the first is NaN: sample 0 must stay finite
    y = plug.fprop(x, w, [0], 1)
    assert plug.route('fprop', x.shape, w.shape, [0], 1, dtype) == 'pointwise_wgmma'
    assert bool(torch.isfinite(y[0]).all())
    assert bool(torch.isnan(y[1:]).all())
    x[1:] = torch.randn(n - 1, cin, P, generator=g, device=DEV).to(dtype)
    y = plug.fprop(x, w, [0], 1)
    with engine_only():
        ye = plug.fprop(x, w, [0], 1)
    assert_same(y, ye, 'forward')


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
def test_guards_workspace_inputs(plug, dtype):
    lib = plug._lib
    n, cin, cout, P = 2, 96, 200, 392
    x, w, dy = operands(n, cin, cout, (P,), dtype, seed=9)
    code = 0 if dtype == torch.float32 else 1
    args = [code, n, 1, cin, cout, 1, 1, P, 1, 1, 1, 0, 0, 0]
    for mode in (0, 1):
        src, m = (x, cout) if mode == 0 else (dy, cin)
        assert lib.lvg_convnd_route(mode, *args, 1, 0) == 2
        need = lib.lvg_convnd_workspace(*args)
        assert need > 0
        guard = 4096
        ws = torch.full((need + guard,), 0xFF, dtype=torch.uint8, device=DEV)
        out_full = torch.full((n * m * P + guard,), float('nan'), dtype=dtype, device=DEV)
        out = out_full[:n * m * P].view(n, m, P)
        keep = [t.clone() for t in (src, w)]
        ws_guard = ws[need:].clone()
        stream = torch.cuda.current_stream().cuda_stream
        fn = lib.lvg_convnd_fprop if mode == 0 else lib.lvg_convnd_dgrad
        extra = [1, None, 0, 0.0, 1.0, -1.0] if mode == 0 else [1]
        rc = fn(src.data_ptr(), w.data_ptr(), out.data_ptr(), *args, *extra, ws.data_ptr(), need, stream)
        assert rc == 0, lib.lvg_last_error().decode()
        torch.cuda.synchronize()
        assert bool(torch.isfinite(out).all()), 'an output element was not written'
        assert bool(torch.isnan(out_full[n * m * P:]).all()), 'the kernel wrote past the output'
        assert torch.equal(ws[need:], ws_guard), 'the kernel wrote past the workspace'
        for a, b in zip((src, w), keep):
            assert torch.equal(a, b), 'an input changed'


def test_routing_envelope(plug):
    f32 = torch.float32
    # unaligned pixel pitch (P % 4 != 0), stride, padding, groups, a bias / act epilogue: the engine
    assert plug.route('fprop', (2, 96, 3, 5, 7), (128, 96, 1, 1, 1), [0, 0, 0], 1, f32) == 'engine'
    assert plug.route('fprop', (2, 96, 16, 16), (128, 96, 1, 1), [0, 0], 1, f32, stride=2) == 'engine'
    assert plug.route('fprop', (2, 96, 16, 16), (128, 48, 1, 1), [0, 0], 2, f32) == 'engine'
    assert plug.route('fprop', (2, 96, 16, 16), (128, 96, 1, 1), [0, 0], 1, f32, epilogue=True) == 'engine'
    assert plug.route('fprop', (2, 96, 16, 16), (128, 96, 1, 1), [0, 0], 1, f32) == 'pointwise_wgmma'
    assert plug.route('dgrad', (2, 96, 16, 16), (128, 96, 1, 1), [0, 0], 1, f32) == 'pointwise_wgmma'
    assert plug.route('fprop', (2, 96, 6, 6), (128, 96, 1, 1), [0, 0], 1, torch.float16) == 'engine'       # 36 % 8 != 0
    assert plug.route('fprop', (2, 32, 16, 16), (64, 32, 1, 1), [0, 0], 1, f32) == 'simt'
    assert plug.route('fprop', (2, 32, 16, 16), (64, 32, 1, 1), [0, 0], 1, torch.float16) == 'pointwise_wgmma'
    assert plug.route('fprop', (2, 32, 16, 16), (64, 32, 3, 3), [1, 1], 1, f32) == 'engine'
    assert plug.route('wgrad', (2, 96, 16, 16), (128, 96, 1, 1), [0, 0], 1, f32) == 'engine'
    # a bias epilogue runs on the engine and still matches the unfused result's route-independent definition
    x, w, _ = operands(2, 96, 128, (64,), f32, seed=3)
    b = torch.randn(128, device=DEV)
    y = plug.fprop(x, w, [0], 1, bias=b, act=1)
    with engine_only():
        ye = plug.fprop(x, w, [0], 1, bias=b, act=1)
    assert_same(y, ye, 'forward with bias')


def kernel_names(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize('dtype', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('cout', [48, 300])
def test_route_matches_profiler(plug, cout, dtype):
    """Every kernel instance (split / fp16 x 64-row / 128-row) launches, and only when the route query says so."""
    x, w, dy = operands(2, 100, cout, (512,), dtype, seed=cout)             # 100 x 48 > 4096: not a SIMT layer
    plug.fprop(x, w, [0], 1)
    names = kernel_names(lambda: plug.fprop(x, w, [0], 1))
    nw = 64 if cout <= 64 else 128
    want = f'conv_pw_tc_kernel<{"true" if dtype == torch.float32 else "false"}, {nw}>'
    assert plug.route('fprop', x.shape, w.shape, [0], 1, dtype) == 'pointwise_wgmma'
    assert any(want in nm for nm in names), names
    assert not any('conv_igemm_kernel' in nm or 'conv_pack_act' in nm for nm in names), names
    with engine_only():
        names = kernel_names(lambda: plug.fprop(x, w, [0], 1))
    assert not any('conv_pw_tc' in nm for nm in names), names
    assert any('conv_igemm_kernel' in nm for nm in names), names


def test_graph_capture(plug):
    x, w, dy = operands(2, 128, 256, (16, 8, 8), torch.float32, seed=11)
    y0 = plug.fprop(x, w, [0, 0, 0], 1)
    dx0 = plug.dgrad(dy, w, x.shape, [0, 0, 0], 1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        plug.fprop(x, w, [0, 0, 0], 1)
        plug.dgrad(dy, w, x.shape, [0, 0, 0], 1)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        y = plug.fprop(x, w, [0, 0, 0], 1)
        dx = plug.dgrad(dy, w, x.shape, [0, 0, 0], 1)
    y.fill_(float('nan'))
    dx.fill_(float('nan'))
    g.replay()
    torch.cuda.synchronize()
    assert_same(y, y0, 'forward (graph)')
    assert_same(dx, dx0, 'input gradient (graph)')


def test_backward_matches_engine(plug):
    """lvg_convnd_backward: the input gradient on this path, the weight gradient on the engine (dy is not shared)."""
    x, w, dy = operands(2, 128, 256, (8, 8, 16), torch.float32, seed=12)
    dx, dw = plug.backward(x, dy, w, [0, 0, 0], 1)
    with engine_only():
        dxe, dwe = plug.backward(x, dy, w, [0, 0, 0], 1)
    assert_same(dx, dxe, 'input gradient')
    assert_same(dw, dwe, 'weight gradient')
