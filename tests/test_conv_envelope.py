"""The convolution engine's declared envelope and its planners agree (host arithmetic only, no device needed).

`ConvNdPlugin._in_envelope` is the shape logic behind `ConvNdPlugin.supported()`: every call it accepts runs on the engine
of csrc/conv_igemm.cu in every direction (conv_nd, the `F` proxy and the modulated convolution rely on that; a call it
refuses goes to torch.nn.functional). Here the envelope is enumerated -- every accepted (kt, kh, kw), strides 1-4, every
padding 0..k-1, groups, ragged channel counts, sizes of 1 and widths on both sides of each tiling threshold -- and for
every accepted shape the library's own planners (`lvg_convnd_plan`, `lvg_convnd_wgrad_plan`, the arithmetic the launches
use) must return a plan whose TMA boxes, MMA widths, shared memory and tiles are valid. tests/test_igemm_emul.py replays
single plans element by element; tests/test_gpu_conv_exact.py runs the envelope on the GPU with exact arithmetic."""
import ctypes
import itertools

import pytest
import torch

from torch_utils import custom_ops

FIELDS = ['wgroups', 'rows', 'mt', 'kc', 'nblk', 'nimg', 'lo_blk', 'to', 'ho', 'wo', 'kt', 'kh', 'kw', 'pad_t', 'pad_h', 'pad_w', 'tt', 'th',
          'wt', 'wtb', 'thb', 'frame_px', 'ncols', 'tiles_x', 'tiles_y', 'tiles_t', 'total_tiles', 'ks', 'stages',
          'a_resident', 'a_stage', 'b_step', 'b_bytes', 'b_box', 'stage_bytes', 'ostride', 'hos', 'wos', 'm64', 'ncw']
WFIELDS = ['split', 'cpad_a', 'cpad_b', 'nt', 'ntiles', 'mt', 'nsplit', 'ablk', 'khc', 'nseg', 'ps', 'rh', 'stages', 'a_stage', 'b_stage',
           'stage_bytes', 'tail_bytes', 'smem', 'seg_w0', 'seg_w1', 'seg_w2', 'seg_w3', 'seg_x00', 'seg_x01', 'seg_x02', 'seg_x03',
           'unused', 'mrows']
SMEM = 227 * 1024                      # dynamic shared memory of one CTA on sm_90
DTYPES = {0: torch.float32, 1: torch.float16}

KERNELS_2D = [(kh, kw) for kh in range(1, 10) for kw in range(1, 4) if kh * kw <= 9]
# widths on both sides of: one TMA box row (126-130), two (252-256), the weight gradient's four segments of a 3x3 kernel
# (504-506), and the strided row tiles that no longer fit 256 columns at stride 3 (84-86) and 4 (62-65)
WIDTHS = [1, 2, 5, 16, 62, 63, 64, 65, 84, 85, 86, 126, 127, 128, 129, 130, 252, 253, 254, 255, 256, 504, 505, 506]


@pytest.fixture(scope='module')
def lib():
    return custom_ops.load_library()


def conv_plan(lib, mode, code, n, groups, cin, cout, sp, k, pad, stride):
    out = (ctypes.c_int * 48)()
    rc = lib.lvg_convnd_plan(mode, code, n, groups, cin, cout, *sp, *k, *pad, stride, out, 48)
    return rc, (lib.lvg_last_error().decode() if rc else None), list(out)


def wgrad_plan(lib, code, n, groups, cin, cout, sp, k, pad):
    out = (ctypes.c_int * 32)()
    rc = lib.lvg_convnd_wgrad_plan(code, n, groups, cin, cout, *sp, *k, *pad, out, 32)
    return rc, (lib.lvg_last_error().decode() if rc else None), list(out)


def conv_plan_problems(q, stride):
    """What is wrong with one forward / input-gradient plan (empty: nothing)."""
    bad = []
    if not (q['wtb'] <= 128 and q['thb'] <= 256 and q['tt'] <= 256):
        bad.append(f"TMA box {q['wtb']} x {q['thb']} x {q['tt']}")
    if not (16 <= q['ncols'] <= 256 and q['ncols'] % 16 == 0 and 16 <= q['ncw'] <= 256 and q['ncw'] % 16 == 0):
        bad.append(f"columns {q['ncols']} / MMA width {q['ncw']}")
    if q['m64'] and q['ncw'] != -(-(q['ncols'] // 2) // 16) * 16 or not q['m64'] and q['ncw'] != q['ncols']:
        bad.append(f"MMA width {q['ncw']} for {q['ncols']} columns (64-row mode {q['m64']})")
    if (q['tt'] - 1) * q['frame_px'] + q['th'] * q['wtb'] > q['ncols'] or q['frame_px'] != q['thb'] * q['wtb']:
        bad.append('the tile does not fit its columns')
    if q['wtb'] != q['wt'] + q['kw'] - 1 or q['thb'] != q['th'] + q['kh'] - 1:
        bad.append('box without its halo')
    if not (q['stages'] >= 2 and q['stages'] * q['stage_bytes'] + 128 <= SMEM):
        bad.append(f"{q['stages']} stages of {q['stage_bytes']} bytes")
    if q['tiles_x'] * q['wt'] < q['wo'] or q['tiles_y'] * q['th'] < q['ho'] or q['tiles_t'] * q['tt'] < q['to']:
        bad.append('tiles do not cover the output')
    if (q['tiles_x'] - 1) * q['wt'] >= q['wo'] or (q['tiles_y'] - 1) * q['th'] >= q['ho'] or (q['tiles_t'] - 1) * q['tt'] >= q['to']:
        bad.append('an empty tile')
    if q['ostride'] != stride:
        bad.append(f"output stride {q['ostride']}")
    if stride > 1 and ((q['tiles_x'] > 1 and q['wt'] % stride) or (q['tiles_y'] > 1 and q['th'] % stride)):
        bad.append(f"tile origins off the stride-{stride} lattice ({q['wt']} x {q['th']})")
    if q['hos'] != (q['ho'] - 1) // stride + 1 or q['wos'] != (q['wo'] - 1) // stride + 1:
        bad.append('strided output extent')
    return bad


def wgrad_kernel_exists(taps, nt, split):
    return nt % 32 == 0 and 32 <= nt and taps * nt <= 256 and (nt <= 128 or not split)


def wgrad_plan_problems(q, wo, kw):
    bad = []
    if not wgrad_kernel_exists(q['khc'] * kw, q['nt'], q['split']):
        bad.append(f"no kernel for {q['khc'] * kw} taps x {q['nt']} columns")
    if q['smem'] > SMEM or q['stages'] < 2:
        bad.append(f"{q['smem']} bytes of shared memory")
    if not (1 <= q['nseg'] <= 4) or sum(q[f'seg_w{j}'] for j in range(4)) != wo:
        bad.append(f"{q['nseg']} segments do not cover {wo} columns")
    if any(q[f'seg_w{j}'] and q[f'seg_x0{j}'] != sum(q[f'seg_w{i}'] for i in range(j)) for j in range(4)):
        bad.append('segments overlap')
    if not (q['ps'] <= 128 and q['ps'] % 8 == 0 and q['ps'] >= max(q[f'seg_w{j}'] for j in range(4)) + kw - 1):
        bad.append(f"tile pitch {q['ps']}")
    if q['rh'] + q['khc'] - 1 > 256 or q['nt'] // 8 > 256 or q['ablk'] > 256:
        bad.append('TMA box too large')
    return bad


def check_shape(lib, code, n, groups, cin, cout, sp, k, pad, stride):
    """Problems of one shape the envelope accepts, as strings naming the shape."""
    name = f"{'f32' if code == 0 else 'f16'} n{n} g{groups} {cin}->{cout} {tuple(sp)} k{tuple(k)} p{tuple(pad)} s{stride}"
    bad = []
    for mode in (0, 1):
        rc, err, out = conv_plan(lib, mode, code, n, groups, cin, cout, sp, k, pad, stride)
        what = ('forward', 'input gradient')[mode]
        if rc:
            bad.append(f'{name}: {what}: {err}')
            continue
        if out[47]:
            continue                    # the streaming 1x1x1 kernels (csrc/conv_pointwise.cu) take the call
        q = dict(zip(FIELDS, out))
        bad += [f'{name}: {what}: {b}' for b in conv_plan_problems(q, stride if mode == 0 else 1)]
    # the weight-gradient planner has no stride argument: it tiles the stride-1 output grid, over which dy is spread for any
    # stride, so the same plan serves every stride
    rc, err, out = wgrad_plan(lib, code, n, groups, cin, cout, sp, k, pad)
    if rc:
        bad.append(f'{name}: weight gradient: {err}')
    else:
        wo = sp[2] + 2 * pad[2] - k[2] + 1
        bad += [f'{name}: weight gradient: {b}' for b in wgrad_plan_problems(dict(zip(WFIELDS, out)), wo, k[2])]
    return bad


def accepted(code, n, groups, cin, cout, sp, k, pad, stride, nd):
    x_shape = (n, groups * cin) + tuple(sp[3 - nd:])
    w_shape = (groups * cout, cin) + tuple(k[3 - nd:])
    st = (1, stride, stride)[3 - nd:]
    return custom_ops.ConvNdPlugin._in_envelope(x_shape, w_shape, DTYPES[code], st, list(pad[3 - nd:]), 1, groups)


def enumerate_2d(stride):
    """2-D shapes at one stride: every kernel and padding, rows of 1 / 9, every threshold width, channel counts pairwise."""
    chans = [(1, 3), (3, 17), (17, 65), (65, 130), (130, 1)]
    for (kh, kw), W, H, (cin, cout), groups in itertools.product(KERNELS_2D, WIDTHS, (1, 9), chans[:1] + chans[3:4], (1,)):
        for ph, pw in itertools.product(range(kh), range(kw)):
            yield (1, groups, cin, cout, (1, H, W), (1, kh, kw), (0, ph, pw), stride, 2)
    # channel counts and groups over a smaller set of kernels and widths
    for (kh, kw), W, (cin, cout), groups in itertools.product([(1, 1), (3, 3), (2, 2), (9, 1), (4, 2)], (16, 85, 129, 256, 505),
                                                              chans, (1, 3)):
        yield (2, groups, cin, cout, (1, 9, W), (1, kh, kw), (0, kh // 2, kw // 2), stride, 2)


def enumerate_3d():
    """3-D (and 1-D) shapes: kt = 1..7 with every temporal padding, frames of 1, a few spatial kernels."""
    for kt, (kh, kw), T, (H, W) in itertools.product(range(1, 8), [(1, 1), (3, 3), (1, 3), (3, 1)], (1, 2, 7, 11), [(1, 1), (5, 16), (9, 130)]):
        for pt in range(kt):
            for code_c in ((3, 17), (65, 130)):
                yield (1, 1, code_c[0], code_c[1], (T, H, W), (kt, kh, kw), (pt, kh // 2, kw // 2), 1, 3)
    for kw, W in itertools.product((1, 2, 3), (1, 3, 127, 128, 129, 256, 505, 513)):
        for pw in range(kw):
            yield (2, 1, 17, 65, (1, 1, W), (1, 1, kw), (0, 0, pw), 1, 1)


@pytest.mark.parametrize('code', [1, 0], ids=['f16', 'f32split'])
@pytest.mark.parametrize('stride', [1, 2, 3, 4])
def test_2d_envelope_plans(lib, code, stride):
    bad, n_ok = [], 0
    for n, groups, cin, cout, sp, k, pad, st, nd in enumerate_2d(stride):
        if not accepted(code, n, groups, cin, cout, sp, k, pad, st, nd):
            continue
        n_ok += 1
        bad += check_shape(lib, code, n, groups, cin, cout, sp, k, pad, st)
    assert n_ok > 1000
    assert not bad, f'{len(bad)} problems, e.g.\n' + '\n'.join(bad[:40])


@pytest.mark.parametrize('code', [1, 0], ids=['f16', 'f32split'])
def test_3d_and_1d_envelope_plans(lib, code):
    bad, n_ok = [], 0
    for n, groups, cin, cout, sp, k, pad, st, nd in enumerate_3d():
        if not accepted(code, n, groups, cin, cout, sp, k, pad, st, nd):
            continue
        n_ok += 1
        bad += check_shape(lib, code, n, groups, cin, cout, sp, k, pad, st)
    assert n_ok > 500
    assert not bad, f'{len(bad)} problems, e.g.\n' + '\n'.join(bad[:40])


def test_envelope_edges():
    """What the envelope refuses, so that those calls go to torch.nn.functional instead of failing in the library."""
    env = custom_ops.ConvNdPlugin._in_envelope
    f16 = torch.float16
    assert env((1, 16, 9, 504), (16, 16, 3, 3), f16, 1, 1, 1, 1)                  # stride-1 output width 504 = 4 x 126
    assert not env((1, 16, 9, 505), (16, 16, 3, 3), f16, 1, 1, 1, 1)              # 505: more than the weight gradient's 4 segments
    assert not env((1, 16, 9, 505), (16, 16, 3, 3), f16, 3, 1, 1, 1)              # whatever the stride
    assert env((1, 16, 9, 512), (16, 16, 1, 1), f16, 1, 0, 1, 1)                  # 1x1: 4 x 128
    assert not env((1, 16, 9, 513), (16, 16, 1, 1), f16, 1, 0, 1, 1)
    assert not env((1, 16, 9, 20), (16, 16, 3, 3), f16, 5, 1, 1, 1)               # stride 5
    assert not env((1, 16, 9, 20), (16, 16, 3, 3), f16, (1, 2), 1, 1, 1)          # unequal strides
    assert not env((1, 16, 3, 9, 20), (16, 16, 3, 3, 3), f16, (2, 1, 1), 1, 1, 1)  # temporal stride
    assert not env((1, 16, 20), (16, 16, 3), f16, 2, 1, 1, 1)                     # strided 1-D
    assert not env((1, 16, 9, 20), (16, 16, 3, 3), f16, 1, 1, 2, 1)               # dilation
    assert not env((1, 16, 9, 20), (16, 16, 1, 4), f16, 1, 0, 1, 1)               # kw 4
    assert not env((1, 16, 9, 20), (16, 16, 5, 2), f16, 1, 0, 1, 1)               # kh * kw 10
    assert env((1, 16, 9, 20), (16, 16, 9, 1), f16, 1, 0, 1, 1)
    assert not env((1, 16, 9, 9, 20), (16, 16, 8, 1, 1), f16, 1, 0, 1, 1)          # kt 8
    assert not env((1, 16, 9, 20), (16, 16, 3, 3), f16, 1, 3, 1, 1)               # padding k
    assert not env((1, 16, 9, 20), (16, 16, 3, 3), f16, 1, -1, 1, 1)
    assert not env((1, 16, 1, 20), (16, 16, 3, 3), f16, 1, 0, 1, 1)               # empty output
    assert not env((1, 16, 9, 20), (16, 16, 3, 3), torch.float64, 1, 1, 1, 1)
    assert not env((1, 16, 9, 20), (16, 16, 3, 3), None, 1, 1, 1, 1)              # (supported(): x and w of different dtypes)
    assert not env((0, 16, 9, 20), (16, 16, 3, 3), f16, 1, 1, 1, 1)
    assert not env((1, 16, 9, 20), (16, 8, 3, 3), f16, 1, 1, 1, 1)               # channels do not match the groups
    assert env((1, 16, 9, 20), (16, 8, 3, 3), f16, 1, 1, 1, 2)
    assert not env((65536, 16, 9, 20), (16, 16, 3, 3), f16, 1, 1, 1, 1)           # instances of a tensor map
