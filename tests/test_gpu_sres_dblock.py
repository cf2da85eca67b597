"""The super-res discriminator block op (torch_utils/ops/sres_dblock.py, csrc/conv_igemm.cu conv_pack_fir4_kernel, the
residual epilogue of csrc/conv_pw_tc.cu) on the GPU: exact arithmetic of both native layers in fp32 and fp16, guard bands,
every block shape of the default discriminator at batch 8 against float64 and the composition, CUDA-graph capture, kernel
names, and the whole installed reference discriminator (tests/sres_dblock_run.py) against the original."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import sres_dblock as sd
from torch_utils.ops import upfirdn2d

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'long-video-gan_b200')
SRC = os.path.join(ROOT, 'oracle', '_ref', 'src')
DEV = 'cuda'
F32 = np.float32
ALPHA, GAIN, SQH = F32(0.2), F32(np.sqrt(2)), F32(np.sqrt(0.5))


def filt():
    return upfirdn2d.setup_filter([1, 3, 3, 1]).to(DEV)


def ints(shape, lo, hi, seed):
    return torch.randint(lo, hi + 1, shape, generator=torch.Generator().manual_seed(seed)).double()


def fir_pad2_f64(x):
    """upfirdn2d(x, outer(k, k) / 64, padding=2) in float64, k = [1, 3, 3, 1] (symmetric: orientation does not matter)."""
    k = torch.tensor([1., 3., 3., 1.], dtype=torch.float64) / 8
    f = torch.outer(k, k)[None, None].repeat(x.shape[1], 1, 1, 1)
    return torch.nn.functional.conv2d(torch.nn.functional.pad(x, [2, 2, 2, 2]), f, groups=x.shape[1])


def act_f32(v, b, clamp):
    """The engine's epilogue restated in float64 with its fp32 constants and fp32 roundings: v + b, lrelu, gain, clamp."""
    v = (v + b.view(1, -1, 1, 1)).numpy().astype(F32)
    v = np.where(v < 0, (v * ALPHA).astype(F32), v)
    v = (v * GAIN).astype(F32)
    return torch.from_numpy(np.clip(v, -F32(clamp), F32(clamp)))


def conv1_call(x, w, b, clamp=256.0):
    fx, fy = upfirdn2d._rank1_factors(filt())
    return sd._Native.conv1(x, fx, fy, False, w, b, 'lrelu', 0.2, float(GAIN), clamp)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('n,cin,cout,h,w', [(2, 20, 24, 18, 22), (1, 64, 128, 33, 40), (3, 8, 40, 10, 260), (1, 136, 72, 9, 9)])
def test_conv1_exact(dtype, n, cin, cout, h, w):
    """Small integer inputs and weights and dyadic taps: the FIR re-tiling, the products and the fp32 accumulation are exact,
    so the output equals the float64 restatement with the epilogue's fp32 roundings (fp16: then one rounding to fp16),
    bit for bit. Ragged channel blocks (20, 136 channels), odd extents and a 260-pixel row (three column tiles)."""
    x = ints((n, cin, h, w), -4, 4, 1)
    wt = ints((cout, cin, 3, 3), -3, 3, 2)
    b = ints((cout,), -8, 8, 3) / 4
    ref = act_f32(torch.nn.functional.conv2d(fir_pad2_f64(x), wt, stride=2), b, 256.0)
    got = conv1_call(x.to(DEV, dtype), wt.to(DEV, dtype), b.to(DEV, dtype))
    assert tuple(got.shape) == tuple(ref.shape)
    assert torch.equal(got.cpu(), ref.to(dtype)), float((got.cpu().double() - ref.double()).abs().max())


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('n,cin,cout,hw', [(2, 64, 128, 64 * 64), (3, 24, 40, 8 * 12), (1, 512, 512, 16), (2, 136, 72, 40)])
def test_skip_exact(dtype, n, cin, cout, hw):
    """(W x + r) * sqrt(1/2) in the pointwise epilogue: fp32 add, fp32 multiply by the fp32 constant, one rounding to the
    storage type -- the reference's float operations in its order for fp32."""
    x = ints((n, cin, hw), -4, 4, 4)
    wt = ints((cout, cin), -3, 3, 5)
    r = ints((n, cout, hw), -64, 64, 6) / 8
    acc = torch.einsum('oc,ncp->nop', wt, x)
    s = (acc + r).numpy().astype(F32)
    ref = torch.from_numpy((s * SQH).astype(F32)).to(dtype)
    got = sd._Native.skip(x.view(n, cin, hw, 1).to(DEV, dtype), wt.view(cout, cin, 1, 1).to(DEV, dtype),
                          r.view(n, cout, hw, 1).to(DEV, dtype), float(SQH))
    assert torch.equal(got.view(n, cout, hw).cpu(), ref)


def _guarded(nbytes, guard=4096):
    buf = torch.full([nbytes + 2 * guard], 0x5A, dtype=torch.uint8, device=DEV)
    return buf, buf[guard:guard + nbytes]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_guard_bands(dtype):
    """Both kernels write exactly their output: sentinels before and after it stay as they were."""
    lib = custom_ops.load_library()
    code = custom_ops._DTYPE_CODE[dtype]
    es = torch.finfo(dtype).bits // 8
    n, cin, cout, h, w = 2, 24, 40, 21, 30
    x = torch.randn(n, cin, h, w, device=DEV).to(dtype)
    wt = (torch.randn(cout, cin, 3, 3, device=DEV) / 10).to(dtype)
    fx, fy = upfirdn2d._rank1_factors(filt())
    ho, wo = (h - 2) // 2 + 1, (w - 2) // 2 + 1
    buf, y = _guarded(n * cout * ho * wo * es)
    ws = torch.empty(lib.lvg_sres_dblock_conv1_workspace(code, n, cin, cout, h, w), dtype=torch.uint8, device=DEV)
    assert lib.lvg_sres_dblock_conv1(x.data_ptr(), fx.data_ptr(), fy.data_ptr(), 0, wt.data_ptr(), None, y.data_ptr(), code, n, cin, cout, h, w,
                                     2, 0.2, 1.0, -1.0, ws.data_ptr(), ws.numel(), torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    assert (buf[:4096] == 0x5A).all() and (buf[-4096:] == 0x5A).all()
    want = sd._Native.conv1(x, fx, fy, False, wt, None, 'lrelu', 0.2, 1.0, None)
    assert torch.equal(y.view(dtype).view(want.shape), want)
    p = ho * wo + (8 - (ho * wo) % 8) % 8
    xs = torch.randn(n, cin, p, device=DEV).to(dtype)
    ws1 = (torch.randn(cout, cin, device=DEV) / 5).to(dtype)
    r = torch.randn(n, cout, p, device=DEV).to(dtype)
    buf, y = _guarded(n * cout * p * es)
    wsp = torch.empty(lib.lvg_sres_dblock_skip_workspace(code, n, cin, cout, p), dtype=torch.uint8, device=DEV)
    assert lib.lvg_sres_dblock_skip(xs.data_ptr(), ws1.data_ptr(), r.data_ptr(), y.data_ptr(), code, n, cin, cout, p, ctypes.c_float(0.5),
                                    wsp.data_ptr(), wsp.numel(), torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    assert (buf[:4096] == 0x5A).all() and (buf[-4096:] == 0x5A).all()


def test_unsupported_is_reported():
    lib = custom_ops.load_library()
    assert lib.lvg_sres_dblock_conv1_workspace(2, 1, 8, 8, 16, 16) == -1            # fp64
    assert lib.lvg_sres_dblock_skip_workspace(1, 1, 8, 8, 12) == -1                 # fp16 with P % 8 != 0
    x = torch.zeros(8, device=DEV)
    assert lib.lvg_sres_dblock_skip(x.data_ptr(), x.data_ptr(), x.data_ptr(), x.data_ptr(), 1, 1, 8, 8, 12, ctypes.c_float(1.0), x.data_ptr(),
                                    32, None) == custom_ops.LVG_UNSUPPORTED


# ---------------------------------------------------------------------------------------------------- whole blocks

# (cin = tmp channels, cout, resolution, dtype) of every block of the default VideoDiscriminator (hr 256, num_fp16_res 4)
BLOCKS = [(64, 128, 256, torch.float16), (128, 256, 128, torch.float16), (256, 512, 64, torch.float16),
          (512, 512, 32, torch.float16), (512, 512, 16, torch.float32), (512, 512, 8, torch.float32)]


def block_params(cin, cout, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    t = lambda *s: torch.randn(*s, generator=g)                      # noqa: E731
    p = dict(w_skip=t(cout, cin, 1, 1) / np.sqrt(cin), w0=t(cin, cin, 3, 3) / np.sqrt(9 * cin), b0=t(cin) * 0.2,
             w1=t(cout, cin, 3, 3) / np.sqrt(9 * cin), b1=t(cout) * 0.2)
    return {k: v.to(DEV, dtype) for k, v in p.items()}


def run_block(fn, x, p, r1, f=None):
    x = x.clone().requires_grad_(True)
    q = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    f = filt() if f is None else f
    out = fn(x, q['w_skip'], q['w0'], q['b0'], q['w1'], q['b1'], f, f, act='lrelu', gain=float(np.sqrt(2)), clamp=256)
    if r1:
        gx, = torch.autograd.grad(out.float().square().sum(), [x], create_graph=True)
        # scaled by the output's size: the fp16 weight gradients of a b256 block at batch 8 stay inside fp16's range
        ((gx.float().square().sum() + out.float().sum()) / out.numel()).backward()
    else:
        out.float().square().sum().backward()
    res = dict(out=out.detach(), x=x.grad)
    res.update({k: v.grad for k, v in q.items()})
    return {k: v.double() for k, v in res.items()}


def comp64(x, ws, w0, b0, w1, b1, fs, f1, **kw):
    return sd._composition(x, ws, w0, b0, w1, b1, fs, f1, 'lrelu', kw['gain'], kw['clamp'])


@pytest.mark.parametrize('cin,cout,res,dtype', BLOCKS, ids=[f'b{b[2]}' for b in BLOCKS])
@pytest.mark.parametrize('r1', [False, True], ids=['grad', 'r1'])
def test_block_against_float64_and_composition(cin, cout, res, dtype, r1):
    """Every block of the default D at batch 8: output and first-order gradients (and the R1 pattern: the gradient of
    the input taken with create_graph, then backward through it) of the op against the composition in float64 and in the
    block's dtype. Budget: the op's error against float64 is at most 1.5x the composition's plus 1e-5 (fp32) / 2e-3
    (fp16) of the tensor's largest magnitude."""
    n = 8
    x = torch.randn(n, cin, res, res, generator=torch.Generator().manual_seed(res), device='cpu').to(DEV) * 0.5
    p = block_params(cin, cout, dtype, res)
    assert sd.native(x.to(dtype), p['w_skip'], p['w0'], p['w1'], filt(), filt(), 'lrelu')
    ours = run_block(sd.sres_dblock, x.to(dtype), p, r1)
    comp = run_block(lambda *a, **k: sd._composition(*a[:8], 'lrelu', k['gain'], k['clamp']), x.to(dtype), p, r1)
    ref = run_block(comp64, x.double(), {k: v.double() for k, v in p.items()}, r1)
    extra = 1e-5 if dtype == torch.float32 else 2e-3
    for k in ref:
        scale = float(ref[k].abs().max())
        e_ours = float((ours[k] - ref[k]).abs().max()) / scale
        e_comp = float((comp[k] - ref[k]).abs().max()) / scale
        assert e_ours <= 1.5 * e_comp + extra, f'{k}: {e_ours:.3e} vs composition {e_comp:.3e}'


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('n,cin,cout,h,w', [(2, 20, 24, 18, 22), (1, 64, 128, 33, 40), (2, 136, 72, 9, 9)])
def test_conv1_backward_prepacked(dtype, n, cin, cout, h, w):
    """conv1's backward: dhf is lvg_convnd_dgrad's, and dw from the X8 the FIR pass re-tiles from h0 is bit for bit the
    weight gradient of the same filtered image packed from NCHW (small integers: upfirdn2d's image is exact)."""
    x = ints((n, cin, h, w), -4, 4, 7).to(DEV, dtype)
    wt = ints((cout, cin, 3, 3), -3, 3, 8).to(DEV, dtype)
    dz = ints((n, cout, (h - 2) // 2 + 1, (w - 2) // 2 + 1), -4, 4, 9).to(DEV, dtype)
    f = filt()
    fx, fy = upfirdn2d._rank1_factors(f)
    dhf, dw = sd._Native.conv1_backward(x, fx, fy, False, dz, wt, True, True)
    hf = upfirdn2d.upfirdn2d(x, f, padding=2)
    plug = sd.conv_nd._get_plugin()
    assert torch.equal(dw, plug.wgrad(hf, dz, tuple(wt.shape), (0, 0), 1, stride=2))
    assert torch.equal(dhf, plug.dgrad(dz, wt, tuple(hf.shape), (0, 0), 1, stride=2))
    xr = torch.randn(n, cin, h, w, device=DEV).to(dtype)
    _, dw2 = sd._Native.conv1_backward(xr, fx, fy, False, dz, wt, False, True)
    want = plug.wgrad(upfirdn2d.upfirdn2d(xr, f, padding=2), dz, tuple(wt.shape), (0, 0), 1, stride=2)
    assert float((dw2.double() - want.double()).abs().max()) <= 1e-2 * float(want.double().abs().max())


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('n,c,h,w,clamp', [(2, 20, 18, 22, None), (3, 8, 33, 40, 1.5), (1, 64, 9, 70, None)])
def test_fir_adjoint_act_exact(dtype, n, c, h, w, clamp):
    """dz0 = G(h0) (.) FIR^T(dhf): with small-integer dhf the adjoint is exact, the slope is applied with the fp32
    constants in bias_act's order, one rounding: bit for bit the float64 restatement. db0: the sum of the stored dz0,
    within fp32 summation error of float64, and bitwise the same on every run."""
    dhf = ints((n, c, h + 1, w + 1), -4, 4, 10)
    h0 = ints((n, c, h, w), -3, 3, 11) / 2
    k = torch.tensor([1., 3., 3., 1.], dtype=torch.float64) / 8
    fk = torch.outer(k, k)[None, None].repeat(c, 1, 1, 1)
    t = torch.nn.functional.conv2d(torch.nn.functional.pad(dhf, [1, 1, 1, 1]), fk, groups=c).numpy().astype(F32)
    y = h0.numpy()
    o = np.where(y > 0, t, (t * ALPHA).astype(F32))
    o = (o * GAIN).astype(F32)
    if clamp is not None:
        o = np.where((y > -clamp) & (y < clamp), o, F32(0))
    ref = torch.from_numpy(o).to(dtype)
    fx, fy = upfirdn2d._rank1_factors(filt())
    runs = [sd._Native.fir_adjoint_act(dhf.to(DEV, dtype), h0.to(DEV, dtype), fx, fy, False, 'lrelu', 0.2, float(GAIN), clamp, True)
            for _ in range(2)]
    dz, db = runs[0]
    assert torch.equal(dz.cpu(), ref)
    assert torch.equal(db, runs[1][1]) and torch.equal(dz, runs[1][0])
    want = ref.double().sum([0, 2, 3])
    assert float((db.cpu().double() - want).abs().max()) <= 1e-5 * max(float(want.abs().max()), 1.0)


def test_bias_gradient_reproducible():
    """Every gradient of the block, conv0's bias gradient from the fixed-order fold included, is bitwise the same run to
    run."""
    cin, cout, res, dtype = 128, 256, 64, torch.float16
    x = torch.randn(8, cin, res, res, device=DEV).to(dtype)
    p = block_params(cin, cout, dtype, 1)
    a = run_block(sd.sres_dblock, x, p, False)
    b = run_block(sd.sres_dblock, x, p, False)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_no_weight_gradients():
    from torch_utils.ops import conv2d_gradfix
    cin, cout, res, dtype = 64, 128, 32, torch.float32
    x = torch.randn(2, cin, res, res, device=DEV).requires_grad_(True)
    p = {k: v.requires_grad_(True) for k, v in block_params(cin, cout, dtype, 2).items()}
    with conv2d_gradfix.no_weight_gradients():
        out = sd.sres_dblock(x, p['w_skip'], p['w0'], p['b0'], p['w1'], p['b1'], filt(), filt(), gain=float(np.sqrt(2)), clamp=256)
        out.sum().backward()
    assert x.grad is not None and p['b1'].grad is not None
    assert all(p[k].grad is None or not p[k].grad.any() for k in ('w_skip', 'w0', 'w1'))


def test_cuda_graph_capture():
    cin, cout, res, dtype = 128, 256, 64, torch.float16
    x = torch.randn(8, cin, res, res, device=DEV).to(dtype)
    p = block_params(cin, cout, dtype, 3)
    f = filt()
    call = lambda: sd.sres_dblock(x, p['w_skip'], p['w0'], p['b0'], p['w1'], p['b1'], f, f, gain=float(np.sqrt(2)), clamp=256)  # noqa: E731
    with torch.no_grad():
        want = call()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            call()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            out = call()
        x.copy_(x * 0.5)
        want = call()
        g.replay()
        torch.cuda.synchronize()
    assert torch.equal(out, want)


def test_profiler_names_every_kernel(tmp_path):
    """Every instance of both new kernels appears by name in a torch.profiler trace (in a process of its own)."""
    names = _helper('kernels', tmp_path)['kernels']
    for want in ('conv_pack_fir4_kernel<__half, false>', 'conv_pack_fir4_kernel<float, true>', 'sres_fir_adjoint_act_kernel<float>',
                 'sres_fir_adjoint_act_kernel<__half>', 'sres_fir_adjoint_fold_kernel'):
        assert any(want in n for n in names), (want, names)
    for inst in ('<true, 64>', '<true, 128>', '<false, 64>', '<false, 128>'):
        assert any('conv_pw_tc_res_kernel' + inst in n for n in names), (inst, names)


# ---------------------------------------------------------------------------------------------------- the reference D

def _helper(mode, tmp_path):
    if not os.path.isdir(SRC):
        pytest.skip('oracle/_ref not staged')
    out = str(tmp_path / f'{mode}.pt')
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, SRC]))
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'sres_dblock_run.py'), out, mode], env=env, cwd=SRC,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1500)
    assert r.returncode == 0, r.stdout[-4000:]
    return torch.load(out)


def _close(a, b, key, tol):
    err = float((a.double() - b.double()).abs().max()) / max(float(b.double().abs().max()), 1e-30)
    assert err <= tol, f'{key}: {err:.3e}'


def test_installed_discriminator(tmp_path):
    """The whole installed VideoDiscriminator against the original: logits, parameter and input gradients, and the R1
    pattern. All fp32: within 1e-3 of each tensor's largest magnitude. Two fp16 and two fp32 blocks: the error against the
    all-fp32 network at most 1.5x the original's plus 5e-3 (the fp16 blocks round at other points, DESIGN.md 5). Every
    block ``faster`` routes took the op and the profiler saw its kernels."""
    r = _helper('cuda', tmp_path)
    assert len(r['took']) >= 8 and all(t[2] for t in r['took']), r['took']
    for ours, ref in zip(r['ours32'], r['ref32']):
        assert ours.keys() == ref.keys()
        for k in ref:
            _close(ours[k], ref[k], k, 1e-3)
    for ours, ref, t in zip(r['ours'], r['ref'], r['ref32']):
        assert ours.keys() == ref.keys()
        for k in ref:
            scale = float(t[k].double().abs().max())
            e_ours = float((ours[k].double() - t[k].double()).abs().max()) / scale
            e_ref = float((ref[k].double() - t[k].double()).abs().max()) / scale
            assert e_ours <= 1.5 * e_ref + 5e-3, f'{k}: {e_ours:.3e} against fp32, the original {e_ref:.3e}'
    assert any('conv_pack_fir4_kernel' in n for n in r['kernels'])
    assert any('conv_pw_tc_res_kernel' in n for n in r['kernels'])


def test_installed_run_D_with_augment_pipe(tmp_path):
    """SuperResVideoGAN.run_D + R1 on one GAN with augment_pipe.install, without and then with sres_dblock.install (all
    fp32 blocks: num_fp16_res 0): the two installs compose."""
    r = _helper('run_D', tmp_path)
    for k in r['ref']:
        _close(r['ours'][k], r['ref'][k], k, 1e-3)
