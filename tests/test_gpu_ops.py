"""Parity of the CUDA path (through the public torch_utils.ops API -> C ABI -> sm_90a kernels)
against the golden vectors from the reference and against the CPU oracle on seeded inputs.

Tolerances are the north_star's: 1e-3 relative for fp32 activations, 1e-2 for gradients (fp16
storage adds its own half-ulp rounding, stated per test)."""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from torch_utils import custom_ops
from torch_utils.ops import bias_act, upfirdn2d, filtered_lrelu, conv2d_resample, fma
from _common import golden, cases, assert_close, t, RTOL_ACT, RTOL_GRAD

pytestmark = pytest.mark.gpu
DEV = 'cuda'
ACTS = sorted(bias_act.activation_funcs)
F16_TOL = 3e-3      # fp16 storage: half-ulp 4.9e-4 per rounding, a few roundings per op


def tol(dtype, base):
    return max(base, F16_TOL) if dtype == torch.float16 else base


def test_native_library_is_loaded():
    lib = custom_ops.load_library()
    assert b'sm_90a' in lib.lvg_build_info()
    assert bias_act._init() and upfirdn2d._init() and filtered_lrelu._init()
    assert type(bias_act._plugin).__name__ == 'BiasActPlugin'


# ------------------------------------------------------------------ bias_act

@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.float64])
@pytest.mark.parametrize('clamp', [None, 0.7])
@pytest.mark.parametrize('act', ACTS)
def test_bias_act_golden(act, clamp, dtype):
    g = golden('bias_act')
    tag = f'{act}_c{"n" if clamp is None else "y"}'
    x, b, dy = (t(g[f'{tag}/{k}'], DEV, dtype, grad=True) for k in ('x', 'b', 'dy'))
    y = bias_act.bias_act(x, b, act=act, clamp=clamp)
    assert y.dtype == dtype and y.is_cuda
    assert_close(y, g[f'{tag}/y'], tol(dtype, 1e-5), 'forward')
    if dtype == torch.float16 or (act == 'linear' and clamp is not None):
        return   # fp16 saved activations move the clamp/sign decisions; covered by the oracle tests below
    dx, db = torch.autograd.grad(y, [x, b], dy, create_graph=True)
    assert_close(dx, g[f'{tag}/dx'], 1e-4, 'dx')
    assert_close(db, g[f'{tag}/db'], 1e-4, 'db')
    if dx.requires_grad:
        v = t(g[f'{tag}/v'], DEV, dtype)
        ddy, ddx = torch.autograd.grad((dx * v).sum(), [dy, x], allow_unused=True)
        assert_close(ddy, g[f'{tag}/ddy'], 1e-4, 'second order wrt dy')
        if bias_act.activation_funcs[act].has_2nd_grad:
            assert_close(ddx, g[f'{tag}/ddx'], 1e-3, 'second order wrt x')


SHAPES = [
    ((3, 7, 5, 6, 9), 1),        # 5-D video tensor, odd sizes (tail + per-element bias path: step 270 % 4 != 0)
    ((2, 16, 20, 12, 16), 1),    # vector path, one bias index per 16-byte pack
    ((37, 1024), 1),             # fully connected: bias along the contiguous dim (packed bias loads)
    ((5, 13), 1),                # tiny, unaligned tail only
    ((2, 8, 33, 17), 1),
    ((4, 6, 10), 2),             # bias on the last dim of a 3-D tensor
    ((2, 3, 4, 5), 0),           # bias on the batch dim
]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('shape,dim', SHAPES)
def test_bias_act_shapes_vs_oracle(shape, dim, dtype):
    gen = torch.Generator().manual_seed(hash((shape, dim)) % 2**31)
    x = torch.randn(*shape, generator=gen).to(dtype)
    b = torch.randn(shape[dim], generator=gen).to(dtype)
    for act, clamp, gain in (('lrelu', 256, None), ('lrelu', 0.5, None), ('linear', None, None), ('swish', 1.0, 0.7), ('tanh', None, 2.0)):
        xg, bg = x.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
        y = bias_act.bias_act(xg, bg, dim=dim, act=act, gain=gain, clamp=clamp)
        ref = orc.bias_act(x.float().numpy(), b.float().numpy(), dim, act, gain=gain, clamp=clamp)
        assert_close(y, ref, tol(dtype, 1e-5), f'forward {act}')
        dy = torch.randn(*shape, generator=gen).to(dtype)
        y.backward(dy.to(DEV))      # plain backward: exercises the fused dx + db kernel
        keep_x = bias_act.activation_funcs[act].ref == 'x'
        yk = None if (keep_x or act == 'linear') else y.detach().float().cpu().numpy()
        rdx = orc.bias_act_grad(dy.float().numpy(), x=x.float().numpy() if keep_x else None, b=b.float().numpy() if keep_x else None,
                                y=yk, dim=dim, act=act, gain=gain, clamp=clamp, order=1)
        assert_close(xg.grad, rdx, tol(dtype, 1e-5), f'dx {act}')
        # db must equal the sum of the dx that was actually stored
        rdb = xg.grad.double().sum([i for i in range(len(shape)) if i != dim]).cpu().numpy()
        assert_close(bg.grad, rdb, tol(dtype, 1e-4), f'db {act}')


def test_bias_act_layouts_and_alignment():
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(2, 8, 9, 10, generator=gen)
    b = torch.randn(8, generator=gen)
    ref = orc.bias_act(x.numpy(), b.numpy(), 1, 'lrelu')
    xc = x.to(DEV).to(memory_format=torch.channels_last)
    y = bias_act.bias_act(xc, b.to(DEV), act='lrelu')
    assert y.stride() == xc.stride()
    assert_close(y, ref, 1e-6, 'channels_last')
    # non-dense view: copied to dense first
    big = torch.zeros(2, 8, 9, 12, device=DEV)
    big[..., 1:11] = x.to(DEV)
    assert_close(bias_act.bias_act(big[..., 1:11], b.to(DEV), act='lrelu'), ref, 1e-6, 'strided view')
    # dense but only 4-byte aligned storage offset: scalar kernel
    flat = torch.zeros(x.numel() + 1, device=DEV)
    flat[1:] = x.to(DEV).flatten()
    xo = flat[1:].view(x.shape)
    assert xo.data_ptr() % 16 != 0
    assert_close(bias_act.bias_act(xo, b.to(DEV), act='lrelu'), ref, 1e-6, 'unaligned')
    # no bias, identity shortcut
    z = torch.randn(4, 4, device=DEV)
    assert bias_act.bias_act(z).data_ptr() == z.data_ptr()
    assert_close(bias_act.bias_act(z, act='relu', gain=1), z.clamp(min=0), 1e-7)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('act,clamp', [('lrelu', 0.7), ('lrelu', None), ('relu', 0.5)])
def test_bias_act_code_path_is_bitwise_the_saved_output_path(act, clamp, dtype, monkeypatch):
    # relu / lrelu keep 2-bit sign / clamp codes for the backward pass (lvg_bias_act_fwd_codes / _bwd_codes) instead of
    # re-reading y; forward, dx, db and the double-backward must be the very same numbers as with the y-based kernels
    gen = torch.Generator().manual_seed(17)
    x = (torch.randn(3, 8, 5, 6, 8, generator=gen) * 0.6).to(dtype).to(DEV)
    x[0, 0, 0, 0, :4] = 0                       # exact zeros: "not positive" must agree on both paths
    b = torch.randn(8, generator=gen).to(dtype).to(DEV)
    b[0] = 0
    dy = torch.randn(x.shape, generator=gen).to(dtype).to(DEV)
    out = {}
    for mode in ('1', '0'):
        monkeypatch.setenv('LVG_BIAS_ACT_CODES', mode)
        xg, bg = x.clone().requires_grad_(True), b.clone().requires_grad_(True)
        y = bias_act.bias_act(xg, bg, act=act, clamp=clamp)
        dx, db = torch.autograd.grad(y, [xg, bg], dy, retain_graph=True)
        dyg = dy.clone().requires_grad_(True)
        gx2, = torch.autograd.grad(y, [xg], dyg, create_graph=True)
        d_dy, = torch.autograd.grad(gx2.float().sum(), [dyg])
        out[mode] = (y, dx, db, d_dy)
    for a, c, what in zip(out['1'], out['0'], ('y', 'dx', 'db', 'd(dx)/d(dy)')):
        if what == 'db':
            assert_close(a, c, tol(dtype, 1e-5), what)      # different summation order of the fused reduction
        else:
            assert torch.equal(a, c), what


def test_bias_act_matches_torch_at_scale():
    # lres generator's largest call (SURVEY.md 8a): (N, 64, T, 36, 64); checked against torch's own kernels
    x = torch.randn(1, 64, 160, 36, 64, device=DEV)
    b = torch.randn(64, device=DEV)
    y = bias_act.bias_act(x, b, act='lrelu', clamp=256)
    assert_close(y, bias_act.bias_act(x, b, act='lrelu', clamp=256, impl='ref'), 1e-6)
    # property: the op is odd-homogeneous in the gain
    y2 = bias_act.bias_act(x, b, act='lrelu', gain=2 * np.sqrt(2), clamp=None)
    assert_close(y2, 2 * bias_act.bias_act(x, b, act='lrelu', clamp=None), 1e-6)


def test_bias_act_beyond_2_31_elements():
    # The reference indexes with 32-bit ints and chunks its tensors below 2^31 elements (generator_lres.py:30-70);
    # these kernels index with 64 bits. 2^31 + 2^21 fp16 elements (4.3 GB), forward and code-passing backward, checked
    # on slices from both ends and around the 2^31 boundary against the same op on the slices alone.
    n_ch, inner = 64, (1 << 25) + (1 << 15)
    free, _ = torch.cuda.mem_get_info()
    if free < 24 * (1 << 30):
        pytest.skip('needs ~20 GB of free device memory')
    x = torch.empty(1, n_ch, inner, device=DEV, dtype=torch.float16)
    assert x.numel() > (1 << 31)
    for c0 in range(0, n_ch, 8):
        x[:, c0:c0 + 8].normal_()
    b = torch.randn(n_ch, device=DEV, dtype=torch.float16)
    xg = x.requires_grad_(True)
    y = bias_act.bias_act(xg, b, act='lrelu', clamp=2.0)
    dy = torch.empty_like(y)
    for c0 in range(0, n_ch, 8):
        dy[:, c0:c0 + 8].normal_()
    dx, = torch.autograd.grad(y, [xg], dy)
    for ch, lo in ((0, 0), (31, inner - 4096), (32, 0), (63, inner - 4096), (17, 12345 * 8)):
        xs = x.detach()[:, ch:ch + 1, lo:lo + 4096].clone().requires_grad_(True)
        ys = bias_act.bias_act(xs, b[ch:ch + 1], act='lrelu', clamp=2.0)
        assert torch.equal(ys, y[:, ch:ch + 1, lo:lo + 4096]), (ch, lo)
        dxs, = torch.autograd.grad(ys, [xs], dy[:, ch:ch + 1, lo:lo + 4096].clone())
        assert torch.equal(dxs, dx[:, ch:ch + 1, lo:lo + 4096]), (ch, lo)


def test_ops_are_cuda_graph_capturable():
    # bench.py replays a whole training step from CUDA graphs: every op (forward and autograd backward) must capture --
    # no synchronisation, no host-side reads -- and the replay must reproduce the eager results
    f = upfirdn2d.setup_filter([1, 3, 3, 1], separable=True).to(DEV)
    k = (torch.randn(12) / 3).to(DEV)
    x = torch.randn(2, 8, 18, 32, device=DEV)
    b = torch.randn(8, device=DEV)

    def forward(xg, bg):
        y = bias_act.bias_act(upfirdn2d.upsample2d(xg, f, up=2), bg, act='lrelu', clamp=256)
        return filtered_lrelu.filtered_lrelu(y, k, k, bg, up=2, down=2, padding=[9, 8, 9, 8], clamp=256)

    with torch.no_grad():
        dy = torch.randn_like(forward(x, b))

    def step():
        xg, bg = x.detach().requires_grad_(True), b.detach().requires_grad_(True)
        y = forward(xg, bg)
        return (y,) + torch.autograd.grad(y, [xg, bg], dy)

    ref = [v.clone() for v in step()]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()                                              # warm-up on the capture stream
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side, capture_error_mode='thread_local'):
            out = step()
    torch.cuda.current_stream().wait_stream(side)
    for v in out:
        v.zero_()
    g.replay()
    torch.cuda.synchronize()
    for got, want, what in zip(out, ref, ('y', 'dx', 'db')):
        assert_close(got, want, 1e-6, what)


# ------------------------------------------------------------------ upfirdn2d

_UP = golden('upfirdn2d')


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.float64])
@pytest.mark.parametrize('name', sorted(cases(_UP)))
def test_upfirdn2d_golden(name, dtype):
    _, kw = cases(_UP)[name]
    f = t(_UP[f'{name}/f'], DEV) if f'{name}/f' in _UP else None
    x = t(_UP[f'{name}/x'], DEV, dtype, grad=True)
    y = upfirdn2d.upfirdn2d(x, f, **kw)
    assert y.dtype == dtype
    ref_y = _UP[f'{name}/y']
    if dtype == torch.float16:   # compare against the oracle on the fp16-rounded input
        ref_y = orc.upfirdn2d(x.detach().float().cpu().numpy(), None if f is None else f.cpu().numpy(), **kw)
    assert_close(y, ref_y, tol(dtype, 1e-5), 'forward')
    dy = t(_UP[f'{name}/dy'], DEV, dtype)
    dx, = torch.autograd.grad(y, [x], dy)
    ref_dx = _UP[f'{name}/dx']
    if dtype == torch.float16:
        ref_dx = orc.upfirdn2d_adjoint(dy.float().cpu().numpy(), None if f is None else f.cpu().numpy(), x.shape, **kw)
    assert_close(dx, ref_dx, tol(dtype, 1e-5), 'dx')


UP_SHAPES = [
    # (x shape, taps, kwargs): model signatures at moderate size (SURVEY.md Appendix A)
    ((2, 64, 18, 32), 4, dict(up=2, padding=[2, 1, 2, 1], gain=4)),                 # U3 bilinear up
    ((2, 512, 3, 4), 4, dict(up=2, padding=[2, 1, 2, 1], gain=4)),                  # U3 tiny planes
    ((1, 96, 64, 64), 4, dict(down=2, padding=[1, 1, 1, 1])),                       # U4
    ((2, 27, 44, 46), 12, dict(down=2, padding=[3, 3, 3, 3])),                      # U6 kaiser down 2
    ((2, 27, 46, 46), 24, dict(down=4, padding=[6, 6, 6, 6])),                      # U6 kaiser down 4
    ((2, 27, 23, 25), 12, dict(up=2, padding=[4, 3, 4, 3], gain=4)),                # U6 up 2
    ((1, 27, 21, 22), 24, dict(up=4, padding=[9, 6, 9, 6], gain=16)),               # U6 up 4
    ((2, 12, 36, 64), 8, dict(up=4, padding=[5, 2, 5, 2], gain=16)),                # U7
    ((1, 3, 40, 40), 12, dict(up=2, padding=[-6, -6, -6, -6], flip_filter=True, gain=4)),   # U9
    ((1, 5, 31, 29), 5, dict(up=[3, 2], down=[2, 3], padding=[4, 1, -1, 3])),       # nothing special about it
]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('shape,taps,kw', UP_SHAPES)
def test_upfirdn2d_separable_vs_oracle(shape, taps, kw, dtype):
    gen = torch.Generator().manual_seed(taps * 1000 + shape[1])
    x = torch.randn(*shape, generator=gen).to(dtype)
    f = torch.randn(taps, generator=gen) / taps
    y = upfirdn2d.upfirdn2d(x.to(DEV), f.to(DEV), **kw)
    ref = orc.upfirdn2d(x.float().numpy(), f.numpy(), **kw)
    assert_close(y, ref, tol(dtype, 1e-5), 'separable forward')
    # channels_last input gives channels_last output with the same values
    ycl = upfirdn2d.upfirdn2d(x.to(DEV).to(memory_format=torch.channels_last), f.to(DEV), **kw)
    assert_close(ycl, ref, tol(dtype, 1e-5), 'channels_last')


STREAM_SHAPES = [
    # (x shape, kwargs): signatures of the register-streaming kernel (upfirdn2d_stream.cu) -- strips per row 1..32,
    # plane counts that leave part of a warp idle, planes tall enough to be split into row segments
    ((1, 3, 18, 32), dict(up=2, padding=[2, 1, 2, 1], gain=4)),
    ((2, 5, 5, 8), dict(up=2, padding=[2, 1, 2, 1], gain=4)),
    ((1, 7, 9, 16), dict(up=2, padding=[2, 1, 2, 1], gain=4, flip_filter=True)),
    ((1, 2, 200, 128), dict(up=2, padding=[2, 1, 2, 1], gain=4)),
    ((1, 3, 64, 64), dict(down=2, padding=[1, 1, 1, 1])),
    ((3, 11, 8, 8), dict(down=2, padding=[1, 1, 1, 1], flip_filter=True)),
    ((1, 1, 36, 64), dict(down=2, padding=[1, 1, 1, 1], gain=0.5)),
    ((1, 2, 300, 256), dict(down=2, padding=[1, 1, 1, 1])),
    ((1, 5, 32, 16), dict(down=2, padding=[1, 1, 1, 1])),
]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('shape,kw', STREAM_SHAPES)
def test_upfirdn2d_streamed_signatures_vs_oracle(shape, kw, dtype):
    gen = torch.Generator().manual_seed(shape[1] * 31 + shape[2])
    x = torch.randn(*shape, generator=gen).to(dtype)
    f = torch.rand(4, generator=gen) + 0.1          # asymmetric: catches orientation / phase mix-ups
    xd = x.to(DEV).requires_grad_(True)
    y = upfirdn2d.upfirdn2d(xd, f.to(DEV), **kw)
    ref = orc.upfirdn2d(x.float().numpy(), f.numpy(), **kw)
    assert_close(y, ref, tol(dtype, 1e-5), 'forward')
    # backward = the adjoint signature (UP2 <-> DOWN2), also streamed
    dy = torch.randn(y.shape, generator=gen).to(dtype)
    dx, = torch.autograd.grad(y, [xd], dy.to(DEV))
    ref_dx = orc.upfirdn2d_adjoint(dy.float().numpy(), f.numpy(), x.shape, **kw)
    assert_close(dx, ref_dx, tol(dtype, 1e-5), 'adjoint')
    # one-axis variants (temporal resampling of [N, C, T, H*W] tensors)
    kw1 = dict(kw)
    kw1['padding'] = [0, 0] + list(kw['padding'][2:])
    for key in ('up', 'down'):
        if key in kw1:
            kw1[key] = [1, kw1[key]]
    if 'gain' in kw1 and 'up' in kw1:
        kw1['gain'] = 2
    y1 = upfirdn2d.upfirdn2d(x.to(DEV), f[:, None].to(DEV), **kw1)
    assert_close(y1, orc.upfirdn2d(x.float().numpy(), f[:, None].numpy(), **kw1), tol(dtype, 1e-5), 'y axis only')


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('shape', [(2, 16, 672, 1), (1, 5, 84, 1), (3, 7, 168, 1), (1, 4, 42, 1), (2, 3, 6, 40)])
def test_upfirdn2d_kaiser12_rows_vs_oracle(shape, dtype):
    # TemporalKaiserDownsample (generator_lres.py:219-262): 12 taps, down 2 along T on [N, C, T, 1] (and [N, C, T, H*W]) tensors,
    # forward and adjoint (up 2, pad 6); lengths that are / are not multiples of the vector width (42 -> 21 takes the tiled kernel)
    gen = torch.Generator().manual_seed(shape[2])
    f = (torch.rand(12, 1, generator=gen) - 0.3) / 4
    kw = dict(down=[1, 2], padding=[0, 0, 5, 5])
    x = torch.randn(*shape, generator=gen).to(dtype)
    xd = x.to(DEV).requires_grad_(True)
    y = upfirdn2d.upfirdn2d(xd, f.to(DEV), **kw)
    assert_close(y, orc.upfirdn2d(x.float().numpy(), f.numpy(), **kw), tol(dtype, 1e-5), 'down 2')
    dy = torch.randn(y.shape, generator=gen).to(dtype)
    dx, = torch.autograd.grad(y, [xd], dy.to(DEV))
    assert_close(dx, orc.upfirdn2d_adjoint(dy.float().numpy(), f.numpy(), x.shape, **kw), tol(dtype, 1e-5), 'adjoint (up 2)')
    yf = upfirdn2d.upfirdn2d(x.to(DEV), f.to(DEV), flip_filter=True, gain=1.5, **kw)
    assert_close(yf, orc.upfirdn2d(x.float().numpy(), f.numpy(), flip_filter=True, gain=1.5, **kw), tol(dtype, 1e-5), 'flipped, gain')


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_upfirdn2d_temporal_axis_vs_oracle(dtype):
    # filters along H only on [N, C, T, H*W] tensors (U1, U2, U5)
    gen = torch.Generator().manual_seed(11)
    lin = torch.tensor([1., 3., 3., 1.]) / 8
    for shape, f, kw in (((2, 32, 20, 144), lin[:, None], dict(up=[1, 2], padding=[0, 0, 2, 1], gain=2)),
                         ((2, 16, 32, 256), lin[:, None] * 2, dict(down=[1, 2], padding=[0, 0, 1, 1])),
                         ((2, 128, 80, 1), torch.randn(12, 1, generator=gen) / 12, dict(down=[1, 2], padding=[0, 0, 5, 5])),
                         ((2, 9, 7, 33), torch.randn(1, 6, generator=gen), dict(up=[2, 1], padding=[3, 2, 0, 0]))):
        x = torch.randn(*shape, generator=gen).to(dtype)
        y = upfirdn2d.upfirdn2d(x.to(DEV), f.to(DEV), **kw)
        assert_close(y, orc.upfirdn2d(x.float().numpy(), f.numpy(), **kw), tol(dtype, 1e-5), str(shape))


def test_upfirdn2d_properties_at_scale():
    # full lres size (U3 largest: (N, 8192, 18, 32) -> (36, 64)); linearity + agreement with torch's conv path
    f = upfirdn2d.setup_filter([1, 3, 3, 1], separable=True).to(DEV)
    x1 = torch.randn(1, 8192, 18, 32, device=DEV)
    x2 = torch.randn(1, 8192, 18, 32, device=DEV)
    y1, y2 = upfirdn2d.upsample2d(x1, f, up=2), upfirdn2d.upsample2d(x2, f, up=2)
    assert y1.shape == (1, 8192, 36, 64)
    assert_close(upfirdn2d.upsample2d(0.5 * x1 - 3 * x2, f, up=2), 0.5 * y1 - 3 * y2, 1e-5, 'linearity')
    assert_close(y1, upfirdn2d.upsample2d(x1, f, up=2, impl='ref'), 1e-5, 'vs torch conv composition')
    # a normalised low-pass filter keeps DC: constant in -> same constant out (away from the borders)
    c = upfirdn2d.upsample2d(torch.ones(1, 4, 18, 32, device=DEV), f, up=2)
    assert_close(c[..., 2:-2, 2:-2], torch.ones_like(c[..., 2:-2, 2:-2]), 1e-6, 'DC gain')
    # adjoint identity <A x, y> == <x, A^T y>
    xd = torch.randn(2, 64, 64, 64, device=DEV, dtype=torch.float64, requires_grad=True)
    yd = upfirdn2d.downsample2d(xd, f, down=2)
    w = torch.randn_like(yd)
    gx, = torch.autograd.grad(yd, [xd], w)
    assert abs(float((yd * w).sum() - (xd * gx).sum())) < 1e-8 * float(yd.abs().sum())


# ------------------------------------------------------------------ filtered_lrelu

_FL = golden('filtered_lrelu')


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('name', sorted(cases(_FL)))
def test_filtered_lrelu_golden(name, dtype):
    _, kw = cases(_FL)[name]
    fu = t(_FL[f'{name}/fu'], DEV) if f'{name}/fu' in _FL else None
    fd = t(_FL[f'{name}/fd'], DEV) if f'{name}/fd' in _FL else None
    x, b = t(_FL[f'{name}/x'], DEV, dtype, grad=True), t(_FL[f'{name}/b'], DEV, dtype, grad=True)
    y = filtered_lrelu.filtered_lrelu(x, fu=fu, fd=fd, b=b, **kw)
    assert y.dtype == dtype
    if dtype == torch.float32:
        assert_close(y, _FL[f'{name}/y'], 1e-4 if name == 'clamp_active' else 2e-5, 'forward')
        dx, db = torch.autograd.grad(y, [x, b], t(_FL[f'{name}/dy'], DEV, dtype))
        assert_close(dx, _FL[f'{name}/dx'], 1e-4, 'dx')
        assert_close(db, _FL[f'{name}/db'], 1e-4, 'db')
    else:
        ref = orc.filtered_lrelu(x.detach().float().cpu().numpy(), None if fu is None else fu.cpu().numpy(),
                                 None if fd is None else fd.cpu().numpy(), b.detach().float().cpu().numpy(), **kw)
        assert_close(y, ref, F16_TOL, 'forward fp16')
        dy = t(_FL[f'{name}/dy'], DEV, dtype)
        dx, db = torch.autograd.grad(y, [x, b], dy)
        assert torch.isfinite(dx).all() and torch.isfinite(db).all()


FL_SHAPES = [
    # sres generator layer geometries at reduced channel count (SURVEY.md Appendix A)
    ((2, 5, 31, 38), 12, 12, dict(up=2, down=2, padding=[9, 8, 9, 8])),
    ((2, 3, 31, 38), 24, 12, dict(up=4, down=2, padding=[-6, -9, -6, -9])),
    ((1, 2, 94, 150), 12, 12, dict(up=2, down=2, padding=[9, 8, 9, 8])),
    ((1, 2, 58, 86), 24, 12, dict(up=4, down=2, padding=[-6, -9, -6, -9])),
    ((1, 2, 166, 278), 12, 12, dict(up=2, down=2, padding=[-11, -12, -11, -12])),
    ((2, 3, 144, 256), 1, 1, dict(up=1, down=1, padding=0, gain=1.0, slope=1.0, clamp=256)),
]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('shape,fut,fdt,kw', FL_SHAPES)
def test_filtered_lrelu_model_shapes_vs_oracle(shape, fut, fdt, kw, dtype):
    gen = torch.Generator().manual_seed(fut * 100 + shape[2])
    x = (torch.randn(*shape, generator=gen) * 2).to(dtype)
    b = torch.randn(shape[1], generator=gen).to(dtype)
    fu = None if fut == 1 else (torch.randn(fut, generator=gen) / np.sqrt(fut))
    fd = None if fdt == 1 else (torch.randn(fdt, generator=gen) / np.sqrt(fdt))
    kw = dict(kw)
    kw.setdefault('clamp', 1.5)      # make the clamp bite so that both sign codes occur
    xg, bg = x.to(DEV).requires_grad_(True), b.to(DEV).requires_grad_(True)
    y = filtered_lrelu.filtered_lrelu(xg, None if fu is None else fu.to(DEV), None if fd is None else fd.to(DEV), bg, **kw)
    fun, fdn = (None if fu is None else fu.numpy()), (None if fd is None else fd.numpy())
    ref, so = orc.filtered_lrelu(x.float().numpy(), fun, fdn, b.float().numpy(), return_signs=True, **kw)
    assert_close(y, ref, tol(dtype, 2e-5) * 5, 'forward')
    # backward: the oracle in read mode with the oracle's own signs, swapped filters (filtered_lrelu.py:252-263)
    dy = torch.randn(*y.shape, generator=gen).to(dtype)
    dx, db = torch.autograd.grad(y, [xg, bg], dy.to(DEV))
    fu_w = 1 if fu is None else fut
    fd_w = 1 if fd is None else fdt
    px0, px1, py0, py1 = orc._pad4(kw['padding'])
    up, down = kw['up'], kw['down']
    pp = [(fu_w - 1) + (fd_w - 1) - px0, shape[3] * up - y.shape[3] * down + px0 - (up - 1),
          (fu_w - 1) + (fd_w - 1) - py0, shape[2] * up - y.shape[2] * down + py0 - (up - 1)]
    rdx = orc.filtered_lrelu(dy.float().numpy(), fdn, fun, None, up=down, down=up, padding=pp,
                             gain=kw.get('gain', np.sqrt(2)) * up ** 2 / down ** 2, slope=kw.get('slope', 0.2), clamp=None,
                             flip_filter=True, signs_in=so, sx=-(fu_w - 1) + px0, sy=-(fu_w - 1) + py0)
    # a handful of samples sit within rounding of the lrelu kink / clamp edge and may flip code: compare in L2
    num = np.linalg.norm(dx.float().cpu().numpy().ravel() - rdx.ravel())
    assert num / np.linalg.norm(rdx.ravel()) < (2e-2 if dtype == torch.float16 else 2e-3), 'dx'
    assert_close(db, dx.double().sum([0, 2, 3]), tol(dtype, 1e-4), 'db')


def test_filtered_lrelu_generic_path_matches_fused():
    # force the composed path (separate native kernels) and compare with whatever the default picks
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(2, 6, 20, 24, generator=gen).to(DEV).requires_grad_(True)
    b = torch.randn(6, generator=gen).to(DEV).requires_grad_(True)
    f = (torch.randn(12, generator=gen) / 3).to(DEV)
    kw = dict(up=2, down=2, padding=[9, 8, 9, 8], clamp=0.8)
    y = filtered_lrelu.filtered_lrelu(x, f, f, b, **kw)
    gx, gb = torch.autograd.grad(y, [x, b], torch.ones_like(y))

    class NoFused:
        def __init__(self, inner): self.inner = inner
        def filtered_lrelu(self, *a): return None, None, -1
        def filtered_lrelu_act_(self, *a): return self.inner.filtered_lrelu_act_(*a)
    real = filtered_lrelu._plugin
    filtered_lrelu._plugin = NoFused(real)
    try:
        with _null():
            y2 = filtered_lrelu.filtered_lrelu(x, f, f, b, **kw)
            gx2, gb2 = torch.autograd.grad(y2, [x, b], torch.ones_like(y2))
    finally:
        filtered_lrelu._plugin = real
    assert_close(y2, y, 1e-5)
    assert_close(gx2, gx, 1e-4)
    assert_close(gb2, gb, 1e-4)


class _null:
    def __enter__(self): return self
    def __exit__(self, *a): return False


# ------------------------------------------------------------------ conv2d_resample, fma

_CV = golden('conv')


@pytest.mark.parametrize('name', sorted(cases(_CV)))
def test_conv2d_resample_golden(name):
    xs, ws, kw, has_f = cases(_CV)[name]
    if has_f:
        kw = dict(kw, f=t(_CV['f4'], DEV))
    x, w = t(_CV[f'{name}/x'], DEV, grad=True), t(_CV[f'{name}/w'], DEV, grad=True)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        y = conv2d_resample.conv2d_resample(x, w, **kw)
        assert_close(y, _CV[f'{name}/y'], RTOL_ACT, 'forward')
        dx, dw = torch.autograd.grad(y, [x, w], t(_CV[f'{name}/dy'], DEV))
    finally:
        torch.backends.cudnn.allow_tf32 = old
    assert_close(dx, _CV[f'{name}/dx'], RTOL_GRAD, 'dx')
    assert_close(dw, _CV[f'{name}/dw'], RTOL_GRAD, 'dw')


def test_fma_gpu():
    g = _CV
    a, b, c = t(g['fma/a'], DEV, grad=True), t(g['fma/b'], DEV, grad=True), t(g['fma/c'], DEV, grad=True)
    o = fma.fma(a, b, c)
    assert_close(o, g['fma/o'], 1e-6)
    da, db, dc = torch.autograd.grad(o, [a, b, c], t(g['fma/do'], DEV))
    assert_close(da, g['fma/da'], 1e-6)
    assert_close(db, g['fma/db'], 1e-6)
    assert_close(dc, g['fma/dc'], 1e-6)
    big = torch.randn(3, 1000, 257, device=DEV)
    assert_close(fma.fma(big, big, big), torch.addcmul(big, big, big), 1e-6)
    h = torch.randn(64, 33, device=DEV, dtype=torch.float16)
    assert_close(fma.fma(h, h[:1], h[:, :1]), torch.addcmul(h[:, :1].float(), h.float(), h[:1].float()), 2e-3)


def test_grad_postprocess_matches_nan_to_num():
    from lvg_dist.grad_sync import postprocess_
    g = torch.randn(1_000_003, device=DEV) * 1e3
    g[::1001] = float('nan')
    g[1::1001] = float('inf')
    g[2::1001] = -float('inf')
    g[3::1001] = 3e5
    for view in (g.clone(), g.clone()[1:]):          # aligned and unaligned start
        ref = torch.nan_to_num(view * 0.125, nan=0.0, posinf=1e5, neginf=-1e5)
        postprocess_(view, scale=0.125)
        assert torch.equal(view, ref)


def test_bias_act_backward_accepts_unaligned_upstream_gradient():
    # ADVICE r1: a dy view with the right strides but a 4-byte-aligned storage offset (narrow of a dim-0 cat backward)
    x = torch.randn(3, 8, 5, 7, device=DEV, requires_grad=True)
    b = torch.randn(8, device=DEV, requires_grad=True)
    y = bias_act.bias_act(x, b, act='lrelu', clamp=256)
    flat = torch.randn(y.numel() + 1, device=DEV)
    dy = flat[1:].view(y.shape)
    assert dy.data_ptr() % 16 != 0 and dy.stride() == y.stride()
    gx, gb = torch.autograd.grad(y, [x, b], dy)
    xr, br = x.detach().double().requires_grad_(True), b.detach().double().requires_grad_(True)
    yr = bias_act.bias_act(xr, br, act='lrelu', clamp=256, impl='ref')
    rx, rb = torch.autograd.grad(yr, [xr, br], dy.double())
    assert_close(gx, rx, 1e-5, 'dx')
    assert_close(gb, rb, 1e-4, 'db')


def test_bias_act_reproducible_bias_gradient_switch(monkeypatch):
    """LVG_BIAS_ACT_FUSED_DB=0: db is the separate reduction of dx (bitwise equal to dx.sum, as the reference computes it);
    the default fused path agrees with it to rounding."""
    x = torch.randn(4, 48, 6, 9, 16, device=DEV)
    b = torch.randn(48, device=DEV)
    dy = torch.randn_like(x)
    out = {}
    for mode in ('1', '0'):
        monkeypatch.setenv('LVG_BIAS_ACT_FUSED_DB', mode)
        xg, bg = x.clone().requires_grad_(True), b.clone().requires_grad_(True)
        y = bias_act.bias_act(xg, bg, act='lrelu', clamp=256)
        dx, db = torch.autograd.grad(y, [xg, bg], dy)
        out[mode] = (dx, db)
    assert torch.equal(out['0'][0], out['1'][0])
    assert torch.equal(out['0'][1], out['0'][0].sum([0, 2, 3, 4]))
    torch.testing.assert_close(out['1'][1], out['0'][1], rtol=1e-5, atol=1e-4)
