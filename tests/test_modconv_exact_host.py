"""The case list of tests/test_gpu_modconv_exact.py against the library's own planners (host arithmetic, no GPU): each
case reaches what it claims -- MMA width and 64-row mode, multi-frame tiles, a k-step remainder -- and together they cover
every width of the output-scaled forward, both sides of the backward-layout predicate, every kernel and temporal padding,
the tile edges, the four row-dot instances and the ABI switches. The fp32 1x1x1 shapes the streaming kernels take have no
engine plan; their forward runs on the engine only through the modulated convolution, which the GPU route check sees."""
import ctypes
import math

import pytest
import torch

from torch_utils import custom_ops
import test_gpu_modconv_exact as mx

CASES = mx.CASES


@pytest.fixture(scope='module')
def plug():
    return custom_ops.get_plugin('convnd_plugin')


def fwd_plan(plug, case, dtype):
    """lvg_convnd_plan(mode 0, groups 1) of the case (the tiling lvg_modconv_fprop launches), or None for the shapes the
    streaming 1x1x1 kernels take in lvg_convnd_fprop."""
    xs, ws, pad, _ = case
    args, _, _, _ = plug._args(xs, ws, list(pad[3 - (len(xs) - 2):]), 1, dtype)
    out = (ctypes.c_int * 48)()
    assert plug._lib.lvg_convnd_plan(0, *args, 1, out, 48) == 0, plug._lib.lvg_last_error().decode()
    return None if out[47] else list(out)


def test_case_ids_are_unique_and_inside_both_envelopes(plug):
    ids = [mx.case_id(c) for c in CASES]
    assert len(set(ids)) == len(ids)
    for xs, ws, pad, _ in CASES:
        p = list(pad[3 - (len(xs) - 2):])
        for dtype in (torch.float16, torch.float32):
            assert plug._in_envelope(xs, ws, dtype, 1, p, 1, 1), (xs, ws, pad)
            args, _, _, _ = plug._modconv_args(torch.empty(xs, device='meta', dtype=dtype), torch.empty(ws, device='meta', dtype=dtype), p)
            assert plug._lib.lvg_modconv_workspace(*args) > 0, (xs, ws, pad)


def test_width_and_multiframe_claims(plug):
    for case in CASES:
        claims = case[3]
        for dtype in (torch.float16, torch.float32):
            out = fwd_plan(plug, case, dtype)
            if out is None:
                assert dtype == torch.float32 and case[1][2:] in ((1, 1), (1, 1, 1)), case
                continue
            if 'width' in claims:
                assert (out[38], out[39]) == claims['width'], (mx.case_id(case), dtype, out[38], out[39])
            if claims.get('multiframe'):
                assert out[16] > 1, (mx.case_id(case), dtype, 'tt', out[16])


def test_every_scaled_width_is_claimed():
    widths = {c[3]['width'] for c in CASES if 'width' in c[3] and c[3].get('d', True)}
    assert widths == {(0, n) for n in range(16, 257, 16)} | {(1, n) for n in range(16, 129, 16)}
    assert all(c[1][0] > 64 for c in CASES if c[3].get('width', (1,))[0] == 0), 'the 128-row widths with cout > 64'


def test_both_backward_layouts(plug):
    """one re-tiling of d * dy serves both gradients iff the weight gradient pads cout to 16 (cout < 128 or a multiple of 128)"""
    shared = set()
    separate = set()
    for xs, ws, pad, _ in CASES:
        args, _, _, _ = plug._args(xs, ws, list(pad[3 - (len(xs) - 2):]), 1, torch.float16)
        out = (ctypes.c_int * 32)()
        assert plug._lib.lvg_convnd_wgrad_plan(*args, out, 32) == 0
        cout = ws[0]
        is_shared = out[1] == (cout + 15) // 16 * 16
        assert is_shared == (cout < 128 or cout % 128 == 0), cout
        (shared if is_shared else separate).add(cout)
    wanted = {1, 3, 64, 65, 127, 128, 130, 181, 256, 362, 384, 512}
    assert wanted <= shared | separate, sorted(wanted - shared - separate)
    assert any(c <= 128 for c in shared) and any(c > 128 for c in shared) and separate


def test_kernels_and_temporal_paddings():
    k2 = {c[1][2:] for c in CASES if len(c[0]) == 4}
    assert k2 >= {(kh, kw) for kh in range(1, 10) for kw in range(1, 4) if kh * kw <= 9}
    t = {(c[1][2], c[2][0]) for c in CASES if len(c[0]) == 5}
    assert t >= {(kt, p) for kt in range(1, 8) for p in range(kt)}
    three = [c for c in CASES if len(c[0]) == 5]
    assert any(mx.out_shape(*c[:3])[0] < c[0][2] for c in three), 'To < T'
    assert any(c[0][2] == 1 for c in three), 'T = 1'
    assert any(c[0][2] == 1 and c[1][2] > 1 for c in three), 'T = 1 under a temporal kernel'


def test_kstep_remainder_claims(plug):
    """kc = channel k-steps of 16; a stage batches ks of them (4 for 1x1 kernels, 2 for kh * kw <= 3, kt = 1)"""
    seen = set()
    for case in CASES:
        if not case[3].get('kstep'):
            continue
        out = fwd_plan(plug, case, torch.float16)         # the same tiling in fp32 (or, for 1x1x1, no engine plan in fp32)
        kc, ks = out[3], out[27]
        assert kc == (case[1][1] + 15) // 16 and kc % ks != 0, (mx.case_id(case), kc, ks)
        taps = math.prod(case[1][3:] if len(case[0]) == 5 else case[1][2:])
        seen.add((taps == 1, ks, kc % ks))
    assert {(True, 4, 1), (True, 4, 2), (True, 4, 3)} <= seen
    assert any(not one and ks == 2 for one, ks, _ in seen)
    assert any(c[0][1] == 1 for c in CASES), 'cin = 1'
    # fp32 1x1 shapes that only the modulated convolution runs on the engine, with a remainder
    assert any(c[3].get('kstep') and fwd_plan(plug, c, torch.float32) is None for c in CASES)


def test_tile_edges_and_rowdot_rows():
    wos = {mx.out_shape(*c[:3])[-1] for c in CASES}
    assert wos >= set(range(126, 131)) | set(range(252, 257)) | {504}
    assert any(mx.out_shape(*c[:3])[-2] == 1 for c in CASES) and max(c[0][0] for c in CASES) == 3
    # modconv_rowdot_kernel<T, VEC>: vector rows when a row is a multiple of 16 bytes; rows longer than one pass of 256 VEC
    rows = {(es, vec) for c in CASES for es in (2, 4) for length in (c[0][-2] * c[0][-1],)
            for vec in (16 // es if length * es % 16 == 0 else 1,) if length > 256 * vec}
    assert rows >= {(2, 8), (2, 1), (4, 4), (4, 1)}, rows


def test_abi_switches():
    for key in ('d', 'dw', 'dyy'):
        assert any(c[3].get(key) is False for c in CASES), key


def test_wrapper_operands_are_dyadic():
    """styles +-2^e and power-of-two input gains scale integer operands exactly; the low-res wrapper divides the weight by
    sqrt(fan), which must be a power of two"""
    pow2 = lambda v: v > 0 and math.frexp(v)[0] == 0.5         # noqa: E731
    assert all(pow2(g) for g in mx.INPUT_GAINS) and all(isinstance(e, int) for e in mx.STYLE_EXPONENTS)
    for kind, xs, ws, pad, dtype in mx.WRAPPER_CASES:
        if kind == 'lres':
            fan = math.prod(ws[1:])
            assert math.isqrt(fan) ** 2 == fan and pow2(math.isqrt(fan)), (ws, fan)
        s_max = 2.0 ** max(mx.STYLE_EXPONENTS) * max(mx.INPUT_GAINS)
        # |a x| <= 4 with a unit of 1/4: exact in fp16 and in one bf16 half
        assert s_max <= 4 and 2.0 ** min(mx.STYLE_EXPONENTS) * min(mx.INPUT_GAINS) >= 0.25
    assert {c[0] for c in mx.WRAPPER_CASES} == {'sres', 'lres'}
    assert any(c[2][1:] == (155, 1, 1) and c[4] == torch.float16 for c in mx.WRAPPER_CASES)
    assert any(c[2][1:] == (64, 1, 1, 1) and c[4] == torch.float32 for c in mx.WRAPPER_CASES)
