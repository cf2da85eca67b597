"""Bit-exact checks of the fused modulated convolution y = d * conv(a * x, w) (lvg_modconv_fprop / lvg_modconv_backward,
csrc/modconv.cu) over its envelope, and of the two wrappers of torch_utils/ops/modulated_conv.py.

The operands are those of tests/test_gpu_conv_exact.py (sparse small integers; for the fp32 split path also dyadic values
whose bf16 lo half is not zero) and power-of-two factors a in 2^{-1,0,1}, d in 2^{-2..0}: a * x splits into bf16 halves
exactly as x does, scaled by a, and d * dy likewise, so every product and partial sum is exact and each output must equal
its float64 reference bit for bit -- y = d conv(a x, w), dx = a conv^T(d dy, w), dw = sum_n conv_w(a x, d dy),
da = sum_hw conv^T(d dy, w) x and sum_hw dy y, minus the lo*lo products for split fp32. Integer operands make every
result a multiple of 1/8 (dyadic ones of 2^-11). Each output asserts its own precondition (sum of |products| at most 2048
units for fp16 outputs, 2^20 for fp32 ones; da and sum dy*y are always fp32). The dyadic runs skip da and sum dy*y (passed
as NULL): their plain fp32 products carry 16 or more significant bits, more than their sums could hold exactly; the
integer runs of the same cases check them.

The harness calls the library through ctypes. Before each call every output is filled with NaN (a skipped element shows)
and sits at the start of a larger allocation whose tail holds a byte pattern; the workspace is exactly
lvg_modconv_workspace bytes, filled with 0xFF (NaN in every operand format, so a read of anything not re-tiled by this
call shows) and followed by 1 MiB of pattern in the same allocation. After the call the patterns must be intact and x, w,
a, d, y and dy unchanged to the bit (the row-dot pass rescales dx in place and reads dy through a cast-away const).

Cases (a pairwise sample, checked on the CPU by tests/test_modconv_exact_host.py against the library's own planners):
every modulated-convolution signature of both generators; every MMA width of the output-scaled forward kernel (N = 16 ...
256 with 128-row images, 16 ... 128 in 64-row mode); output channels on both sides of the backward-layout predicate
(one re-tiling of d * dy for both gradients when cout < 128 or a multiple of 128) with one and several m-tiles; every
(kh, kw); kt 1-7 with every temporal padding (so To < T); 3-D calls with T = 1; k-step remainders of the batched k-steps
(1x1: 4 per stage, kh * kw <= 3: 2); output widths at the column-tile edges; heights of 1; multi-frame tiles; the four
row-dot instances (vector / scalar rows, rows longer than one pass of the CTA); d = NULL, dw = NULL and sum dy*y = NULL."""
import ctypes
import math

import pytest
import torch

from torch_utils import custom_ops
from torch_utils.ops import modulated_conv as mc
from test_gpu_conv_exact import KNOBS, assert_exact, conv5, dyadic, ints, lo_half, plan_flags
from test_gpu_modconv import LRES, SRES
from test_modconv_host import ref_modulated_conv2d, ref_temporal_modulated_conv3d

pytestmark = pytest.mark.gpu
DEV = 'cuda'
UNIT_INT = 1.0 / 8                 # integer operands, a >= 1/2, d >= 1/4
UNIT_DYADIC = 2.0 ** -11           # dyadic operands (hi*lo products are multiples of 2^-8)
OUT_TAIL = 4096                    # pattern bytes behind every output
WS_TAIL = 1 << 20                  # pattern bytes behind the workspace
MODES = [(torch.float16, False), (torch.float32, False), (torch.float32, True)]
MODE_IDS = ['f16', 'f32split-int', 'f32split-dyadic']


@pytest.fixture(scope='module')
def plug():
    return custom_ops.get_plugin('convnd_plugin')


# ---- cases: (x shape, w shape, padding (t, h, w), claims). Claims: width = (64-row mode, MMA width) of the forward,
# multiframe = tiles span frames, kstep = kc is not a multiple of the k-steps per stage, and the ABI switches
# d / dw / dyy = False (passed as NULL).
def C(xs, ws, pad, **claims):
    return (tuple(xs), tuple(ws), tuple(pad), claims)


def out_shape(xs, ws, pad):
    nd = len(xs) - 2
    return tuple(s + 2 * p - k + 1 for s, p, k in zip(xs[2:], pad[3 - nd:], ws[2:]))


def _cases():
    cases = []
    # every modulated-convolution signature of both generators (super-res: per sample, one sample for the large images)
    for cin, cout, k, h, w, p, fp16 in SRES:
        cases.append(C((1 if h * w > 4000 else 2, cin, h, w), (cout, cin, k, k), (0, p, p), sig='sres'))
    for cin, cout, k, h, w, p in LRES:
        mf = dict(multiframe=True) if h * w <= 12 else {}
        cases.append(C((1, cin, 16 if mf else 3, h, w), (cout, cin) + k, p, sig='lres', **mf))
    # the three shapes of the earlier sample
    cases += [C((2, 24, 5, 9, 16), (40, 24, 3, 3, 3), (1, 1, 1)), C((3, 17, 12, 30), (130, 17, 3, 3), (0, 1, 1)),
              C((2, 32, 1, 7, 129), (3, 32, 1, 1, 1), (0, 0, 0))]
    # every MMA width of the output-scaled forward: 3x3 kernels over 14-pixel rows, one tile row = 16 accumulator columns
    couts = [65, 80, 127, 128, 130, 181, 256, 384]
    cins = [24, 1, 17, 40, 33, 3, 70, 16]
    for i, n_ in enumerate(range(16, 257, 16)):
        cases.append(C((1 + i % 3, cins[i % 8], n_ // 16, 14), (couts[i % 8], cins[i % 8], 3, 3), (0, 1, 1), width=(0, n_)))
    couts64 = [1, 3, 40, 64, 17, 33, 48, 64]
    for i, n_ in enumerate(range(16, 129, 16)):
        cases.append(C((1 + (i + 1) % 3, cins[(i + 3) % 8], n_ // 8, 14), (couts64[i], cins[(i + 3) % 8], 3, 3), (0, 1, 1), width=(1, n_)))
    # every (kh, kw): output widths at the column-tile edges (126-130, 252-256, 504), heights of 1
    kernels = [(kh, kw) for kh in range(1, 10) for kw in range(1, 4) if kh * kw <= 9]
    wos = [126, 127, 128, 129, 130, 252, 253, 254, 255, 256, 504, 7, 64, 1, 33, 100]
    hos = [1, 3, 2, 5, 1, 4, 1, 2, 6, 1, 3, 9, 1, 2, 17, 1]
    chans = [(3, 17), (17, 65), (40, 128), (65, 3), (24, 40), (16, 130), (33, 64), (1, 1), (8, 127), (48, 181)]
    for i, (kh, kw) in enumerate(kernels):
        ph, pw = (i // 2) % kh, (i // 3) % kw
        ho, wo = hos[i], wos[i]
        H, W = ho + kh - 1 - 2 * ph, wo + kw - 1 - 2 * pw
        if H < 1:
            ph, H = 0, ho + kh - 1
        if W < 1:
            pw, W = 0, wo + kw - 1
        cin, cout = chans[i % len(chans)]
        cases.append(C((1 + i % 3, cin, H, W), (cout, cin, kh, kw), (0, ph, pw)))
    # kt 1-7 with every temporal padding: To < T whenever pad_t < (kt - 1) / 2, T = 1 where kt <= 1 + 2 pad_t
    ks2 = [(3, 3), (1, 1), (3, 1), (1, 3), (2, 2), (1, 2), (3, 2)]
    chans3 = [(24, 40), (3, 17), (17, 3), (40, 64), (16, 130), (8, 65), (33, 1)]
    i = 0
    for kt in range(1, 8):
        for pt in range(kt):
            kh, kw = ks2[i % len(ks2)]
            T = 1 if (kt <= 1 + 2 * pt and i % 3 == 0) else max(kt - 2 * pt, 1) + 1 + i % 3
            cin, cout = chans3[i % len(chans3)]
            H, W = [(3, 5), (5, 9), (1, 7), (4, 4), (2, 11)][i % 5]
            cases.append(C((1 + i % 2, cin, T, H, W), (cout, cin, kt, kh, kw), (pt, kh // 2, kw // 2)))
            i += 1
    # k-step remainders: 1x1 (4 k-steps per stage) with kc mod 4 = 1, 2, 3 -- in fp32 these shapes reach the engine through
    # this path only --, kh * kw <= 3 (2 per stage) with an odd kc, and cin = 1
    cases += [C((2, 70, 6, 10), (3, 70, 1, 1), (0, 0, 0), kstep=True), C((1, 90, 5, 8), (40, 90, 1, 1), (0, 0, 0), kstep=True),
              C((2, 100, 3, 12), (40, 100, 1, 1), (0, 0, 0), kstep=True), C((1, 155, 6, 20), (3, 155, 1, 1), (0, 0, 0), kstep=True),
              C((2, 70, 5, 2, 4), (24, 70, 1, 1, 1), (0, 0, 0), kstep=True), C((1, 40, 4, 9), (64, 40, 1, 2), (0, 0, 1), kstep=True),
              C((2, 70, 6, 7), (20, 70, 3, 1), (0, 1, 0), kstep=True), C((1, 33, 3, 30), (130, 33, 1, 3), (0, 0, 1), kstep=True),
              C((2, 80, 7, 5), (3, 80, 2, 1), (0, 1, 0), kstep=True),
              C((3, 1, 9, 21), (5, 1, 1, 1), (0, 0, 0)), C((2, 1, 4, 6, 8), (70, 1, 3, 3, 3), (1, 1, 1))]
    # multi-frame tiles: 3x4 frames over T >= 16, n up to 3; rows for the row-dot kernel: 17 x 19 = 323 elements (scalar
    # fp32 / fp16 rows longer than one pass of 256), 36 x 64 = 2304 (vector rows of several passes in both types)
    cases += [C((3, 24, 17, 3, 4), (40, 24, 3, 3, 3), (1, 1, 1), multiframe=True), C((2, 16, 20, 3, 4), (130, 16, 1, 3, 3), (0, 1, 1), multiframe=True),
              C((2, 24, 17, 19), (40, 24, 3, 3), (0, 1, 1)), C((1, 8, 2, 36, 64), (16, 8, 1, 3, 3), (0, 1, 1))]
    # ABI: d = NULL (unscaled forward kernel, no sum dy*y), dw = NULL, sum dy*y = NULL with d given
    cases += [C((2, 24, 9, 30), (130, 24, 3, 3), (0, 1, 1), d=False), C((1, 17, 4, 5, 6), (3, 17, 3, 3, 3), (1, 1, 1), d=False),
              C((2, 40, 6, 20), (64, 40, 3, 3), (0, 1, 1), dw=False), C((1, 24, 3, 4, 6), (181, 24, 3, 1, 3), (1, 0, 1), dw=False, dyy=False),
              C((2, 33, 5, 16), (256, 33, 2, 2), (0, 1, 0), dyy=False)]
    return cases


CASES = _cases()


def case_id(c):
    xs, ws, pad, claims = c
    tag = ''
    for k, v in claims.items():
        tag += f"-{'m64' if v[0] else 'm128'}n{v[1]}" if k == 'width' else f'-{v}' if k == 'sig' else f'-{k}' if v else f'-no{k}'
    return f"x{'x'.join(map(str, xs))}-w{'x'.join(map(str, ws))}-p{''.join(map(str, pad))}{tag}"


def densities(xs, ws, pad):
    """(x, w, dy) densities: about 48 non-zero products per element of y (cin * taps), dx (cout * taps) and dw (n To Ho Wo),
    the others as dense as that allows (at most 0.5)."""
    taps = math.prod(ws[2:])
    fy, fx, fw = ws[1] * taps, ws[0] * taps, xs[0] * math.prod(out_shape(xs, ws, pad))
    c = 48.0
    r = [min(0.5, math.sqrt(c / fy), math.sqrt(c / fx), math.sqrt(c / fw))] * 3
    for _ in range(2):
        r[0] = min(0.5, c / fy / r[1], c / fw / r[2])
        r[1] = min(0.5, c / fy / r[0], c / fx / r[2])
        r[2] = min(0.5, c / fx / r[1], c / fw / r[0])
    return r


def factors(xs, ws, pad, seed, with_d=True):
    g = torch.Generator(device=DEV).manual_seed(seed)
    n, cin, cout = xs[0], xs[1], ws[0]
    T = xs[2] if len(xs) == 5 else 1
    To = out_shape(xs, ws, pad)[0] if len(xs) == 5 else 1
    a = 2.0 ** torch.randint(-1, 2, (n, cin, T), generator=g, device=DEV).double()
    d = 2.0 ** torch.randint(-2, 1, (n, cout, To), generator=g, device=DEV).double() if with_d else None
    return a, d


def modconv_ref(x, w, a, d, dy, pad):
    """(y, dx, dw, da, sum dy*y) of y = d * conv(a * x, w) in float64 (d None: no output factor)."""
    nd = x.ndim - 2
    ex = (lambda v: v[..., None, None]) if nd == 3 else (lambda v: v[..., 0, None, None])
    sum_hw = (lambda v: v.sum((3, 4))) if nd == 3 else (lambda v: v.sum((2, 3))[..., None])
    xa, wr = (x * ex(a)).requires_grad_(True), w.clone().requires_grad_(True)
    z = conv5(xa, wr, 1, pad, 1)
    dd = 1.0 if d is None else ex(d)
    y = z.detach() * dd
    dxp, dw = torch.autograd.grad(z, [xa, wr], dy * dd)          # dxp: the input gradient before the factor a
    return y, dxp * ex(a), dw, sum_hw(dxp * x), sum_hw(dy * y)


# ---- the harness: poisoned, guarded outputs and an exact-size, guarded workspace
def pattern(nbytes):
    return ((torch.arange(nbytes, device=DEV, dtype=torch.int64) * 37 + 11) % 251).to(torch.uint8)


class Guarded:
    """An output tensor at the start of a larger allocation: NaN before the call, a byte pattern behind it."""

    def __init__(self, shape, dtype):
        self.nbytes = math.prod(shape) * torch.finfo(dtype).bits // 8
        self.raw = torch.empty(self.nbytes + OUT_TAIL, dtype=torch.uint8, device=DEV)
        self.raw[self.nbytes:] = pattern(OUT_TAIL)
        self.t = self.raw[:self.nbytes].view(dtype).view(shape)
        if dtype == torch.float16:
            self.t.view(torch.int16).fill_(0x7E00)
        else:
            self.t.fill_(float('nan'))

    def check(self, what):
        assert torch.equal(self.raw[self.nbytes:], pattern(OUT_TAIL)), f'{what}: bytes behind the output were written'


class Workspace:
    def __init__(self, need):
        assert need > 0
        self.need = need
        self.raw = torch.full((need + WS_TAIL,), 0xFF, dtype=torch.uint8, device=DEV)
        self.raw[need:] = pattern(WS_TAIL)

    def check(self, what):
        assert torch.equal(self.raw[self.need:], pattern(WS_TAIL)), f'{what}: written past the end of the workspace'


def bits(ts):
    return [None if t is None else t.view(torch.uint8).clone() for t in ts]


def assert_unchanged(ts, before, what):
    for i, (t, b) in enumerate(zip(ts, before)):
        assert t is None or torch.equal(t.view(torch.uint8), b), f'{what}: input {"x w a d y dy".split()[i]} was modified'


def run_modconv(plug, x, w, a, d, dy, pad, want_dw=True, want_da=True, want_dyy=True):
    """y, then (dx, dw, da, dyy) through lvg_modconv_fprop / lvg_modconv_backward; x, w, dy in the operand type, a, d fp32."""
    lib, nd = plug._lib, x.ndim - 2
    args, sp, k, p = plug._modconv_args(x, w, list(pad[3 - nd:]))
    need = lib.lvg_modconv_workspace(*args)
    P = custom_ops._ptr
    y = Guarded((x.shape[0], w.shape[0]) + out_shape(tuple(x.shape), tuple(w.shape), pad), x.dtype)
    ins = [x, w, a, d]
    before = bits(ins)
    ws = Workspace(need)
    rc = lib.lvg_modconv_fprop(P(x), P(w), P(a), P(d), P(y.t), *args, ws.raw.data_ptr(), need, custom_ops._stream(x))
    assert rc == 0, 'modconv_fprop: ' + lib.lvg_last_error().decode()
    torch.cuda.synchronize()
    y.check('forward y')
    ws.check('forward')
    assert_unchanged(ins, before, 'forward')
    want_dyy = want_dyy and d is not None
    dx = Guarded(tuple(x.shape), x.dtype)
    dw = Guarded(tuple(w.shape), x.dtype) if want_dw else None
    da = Guarded(tuple(a.shape), torch.float32) if want_da else None
    dyy = Guarded(tuple(d.shape), torch.float32) if want_dyy else None
    ins = [x, w, a, d, y.t, dy]
    before = bits(ins)
    ws = Workspace(need)
    T = lambda g: None if g is None else g.t                # noqa: E731
    rc = lib.lvg_modconv_backward(P(x), P(w), P(a), P(d), P(y.t) if want_dyy else None, P(dy), P(dx.t), P(T(dw)), P(T(da)), P(T(dyy)),
                                  *args, ws.raw.data_ptr(), need, custom_ops._stream(x))
    assert rc == 0, 'modconv_backward: ' + lib.lvg_last_error().decode()
    torch.cuda.synchronize()
    for name, g in (('dx', dx), ('dw', dw), ('da', da), ('sum dy*y', dyy)):
        if g is not None:
            g.check(name)
    ws.check('backward')
    assert_unchanged(ins, before, 'backward')
    return y.t, dx.t, T(dw), T(da), T(dyy)


def check_case(plug, case, dtype, dyad, seed=0, check=True):
    xs, ws_, pad, claims = case
    with_d = claims.get('d', True)
    dens = densities(xs, ws_, pad)
    make = dyadic if dyad else ints
    x, w = make(xs, seed + 1, 1, dens[0]), make(ws_, seed + 2, 2, dens[1])
    a, d = factors(xs, ws_, pad, seed + 3, with_d)
    dy = make((xs[0], ws_[0]) + out_shape(xs, ws_, pad), seed + 4, 1, dens[2])
    x, w, dy = (v.to(dtype).double() for v in (x, w, dy))             # representable: no change
    want_dw, want_dyy = claims.get('dw', True), claims.get('dyy', True) and not dyad
    got = run_modconv(plug, x.to(dtype), w.to(dtype), a.float(), None if d is None else d.float(), dy.to(dtype), pad,
                      want_dw=want_dw, want_da=not dyad, want_dyy=want_dyy)
    if not check:
        return
    exp = modconv_ref(x, w, a, d, dy, pad)
    ab = modconv_ref(x.abs(), w.abs(), a, d, dy.abs(), pad)
    if dtype == torch.float32 and dyad:       # split: hi*hi + hi*lo + lo*hi = all products minus lo*lo (bilinear in (x, w), (dy, w), (x, dy))
        lolo = modconv_ref(lo_half(x), lo_half(w), a, d, lo_half(dy), pad)
        exp = tuple(e - l for e, l in zip(exp[:3], lolo[:3])) + exp[3:]
    unit = UNIT_DYADIC if dyad else UNIT_INT
    names = ('y', 'dx', 'dw', 'da', 'sum dy*y')
    for i, (name, g) in enumerate(zip(names, got)):
        if g is None:
            continue
        assert_exact(g, exp[i], ab[i], dtype if i < 3 else torch.float32, unit, f'modconv {name}')


@pytest.mark.parametrize('dtype,dyad', MODES, ids=MODE_IDS)
@pytest.mark.parametrize('case', CASES, ids=[case_id(c) for c in CASES])
def test_modconv_exact(plug, case, dtype, dyad):
    xs, ws_, pad, claims = case
    nd = len(xs) - 2
    assert plug._in_envelope(xs, ws_, dtype, 1, list(pad[3 - nd:]), 1, 1), 'shape outside the envelope'
    if 'width' in claims and not any(plan_flags(plug, xs, ws_, list(pad[3 - nd:]), 1, 1, dtype)):
        args, _, _, _ = plug._args(xs, ws_, list(pad[3 - nd:]), 1, dtype)
        out = (ctypes.c_int * 48)()
        assert plug._lib.lvg_convnd_plan(0, *args, 1, out, 48) == 0
        assert (out[38], out[39]) == claims['width'], 'the forward runs another MMA width'
    check_case(plug, case, dtype, dyad)


# ---- tiling invariance on a subset: shared / separate backward layout, 64- / 128-row mode, a multi-frame 3-D case; the
# engine's switches and LVG_CONV_SHARED_DY8=0, which re-tiles d dy for each gradient where the backward would share it
KNOB_CASES = [c for c in CASES if c[2] == (0, 1, 1) and c[3].get('width') in ((0, 64), (1, 64), (0, 80))] + \
             [c for c in CASES if c[3].get('multiframe') and c[0][0] == 3]
MODCONV_KNOBS = KNOBS + [('LVG_CONV_SHARED_DY8', '0')]


@pytest.mark.parametrize('knob,value', MODCONV_KNOBS, ids=[f'{k}={v}' for k, v in MODCONV_KNOBS])
@pytest.mark.parametrize('dtype,dyad', [MODES[0], MODES[2]], ids=[MODE_IDS[0], MODE_IDS[2]])
def test_modconv_tiling_knobs_exact(plug, monkeypatch, knob, value, dtype, dyad):
    monkeypatch.setenv(knob, value)
    for case in KNOB_CASES:
        check_case(plug, case, dtype, dyad, seed=100)


# ---- the wrappers with demodulate=False: dyadic styles and input gains keep the fp32 arithmetic around the kernels exact
# (kind, x shape, w shape, padding, dtype): the two ToRGB layers (super-res 155 -> 3 1x1 fp16; low-res 64 -> 3 1x1x1 fp32,
# whose weight / sqrt(64) = / 8 stays exact), a super-res 3x3 layer, and a low-res 1x2x2 layer over 16 channels (weight
# / sqrt(64) again: the 27 taps of a 3x3x3 kernel admit no power-of-two sqrt(fan))
WRAPPER_CASES = [('sres', (2, 155, 36, 64), (3, 155, 1, 1), 0, torch.float16), ('lres', (1, 64, 4, 36, 64), (3, 64, 1, 1, 1), (0, 0, 0), torch.float32),
                 ('sres', (2, 40, 12, 30), (24, 40, 3, 3), 1, torch.float16), ('lres', (2, 16, 5, 6, 8), (24, 16, 1, 2, 2), (0, 1, 1), torch.float32)]
STYLE_EXPONENTS = (-1, 0, 1)
INPUT_GAINS = (0.5, 2.0)


def wrapper_operands(kind, xs, ws, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x, w = ints(xs, seed + 1, 1, 0.3), ints(ws, seed + 2, 2, 0.3)
    shape = (xs[0], xs[1]) if kind == 'sres' else (xs[0], xs[1], xs[2])
    e = torch.tensor(STYLE_EXPONENTS, device=DEV)[torch.randint(0, len(STYLE_EXPONENTS), shape, generator=g, device=DEV)]
    sign = torch.randint(0, 2, shape, generator=g, device=DEV) * 2 - 1
    s = sign * 2.0 ** e.double()
    gain = torch.tensor(INPUT_GAINS[seed % len(INPUT_GAINS)], dtype=torch.float64, device=DEV)
    return x, w, s, gain


def wrapper_grads(fn, x, w, s, gain, pad, dtype, dy, create_graph=False):
    xa = x.to(dtype).requires_grad_(True)
    wa, sa, ga = (t.to(torch.float32 if dtype != torch.float64 else dtype).requires_grad_(True) for t in (w, s, gain))
    if fn is mc.modulated_conv2d or fn is ref_modulated_conv2d:
        y = fn(xa, wa, sa, demodulate=False, padding=pad, input_gain=ga)
    else:
        y = fn(xa, wa, sa, ga, padding=pad, demodulate=False)
    grads = torch.autograd.grad(y, [xa, wa, sa, ga], dy.to(y.dtype), create_graph=create_graph)
    return [y.detach()] + [t.detach() for t in grads]


@pytest.mark.parametrize('create_graph', [False, True], ids=['first-order', 'create-graph'])
@pytest.mark.parametrize('wcase', WRAPPER_CASES, ids=[f'{c[0]}-{c[2][1]}-{c[2][0]}-k{c[2][-1]}' for c in WRAPPER_CASES])
def test_wrappers_exact(wcase, create_graph):
    kind, xs, ws, pad, dtype = wcase
    if create_graph and ws[-1] == 1:
        pytest.skip('the create_graph path is checked once in 2-D and once in 3-D, on the layers with larger kernels')
    fn, ref = (mc.modulated_conv2d, ref_modulated_conv2d) if kind == 'sres' else (mc.temporal_modulated_conv3d, ref_temporal_modulated_conv3d)
    x, w, s, gain = wrapper_operands(kind, xs, ws, 7 + len(xs) + xs[1])
    pd = (0, pad, pad) if kind == 'sres' else pad
    assert mc._native(x.to(dtype), w.to(dtype), pd[3 - (len(xs) - 2):])
    yshape = (xs[0], ws[0]) + out_shape(xs, ws, pd)
    dy = ints(yshape, 9, 1, min(0.3, 200.0 / math.prod(yshape[:1] + yshape[2:])))     # dw sums about 60 products
    ours = wrapper_grads(fn, x, w, s, gain, pad, dtype, dy, create_graph)
    exact = wrapper_grads(ref, x, w, s, gain, pad, torch.float64, dy)
    for name, o, e in zip(('y', 'dx', 'dw', 'ds', 'd(input_gain)'), ours, exact):
        assert o.dtype in (dtype, torch.float32) and o.shape == e.shape, (name, o.dtype, o.shape, e.shape)
        assert torch.equal(o.double(), e), f'{kind} wrapper {name}: max difference {float((o.double() - e).abs().max())}'


# ---- every output-scaled kernel instance the path owns is launched by the case list
def expected_kernels():
    k = {}
    for bf16 in ('false', 'true'):
        for n_ in range(16, 257, 16):
            k[f'igemm<{bf16},{n_},scaled>'] = rf'conv_igemm_kernel<{bf16},{n_},true>'
    k['pack<f32,scaled>'] = r'conv_pack_act_kernel<float,true,true>'
    k['pack<f16,scaled>'] = r'conv_pack_act_kernel<__half,false,true>'
    for t, v in (('float', 4), ('float', 1), ('__half', 8), ('__half', 1)):
        k[f'rowdot<{t},{v}>'] = rf'modconv_rowdot_kernel<{t},{v}>'
    return k


def test_kernel_routes_reached(plug):
    import re
    from torch.profiler import ProfilerActivity, profile
    names = set()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for case in CASES:
            for dtype, dyad in MODES[:2]:
                check_case(plug, case, dtype, dyad, check=False)
        torch.cuda.synchronize()
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            names.add(re.sub(r'\s+', '', e.name))
    if not names:
        pytest.skip('torch.profiler reported no CUDA kernels on this machine, so launches cannot be observed')
    missed = [k for k, rx in expected_kernels().items() if not any(re.search(rx, n) for n in names)]
    assert not missed, 'kernel instances never launched: ' + ', '.join(missed)
