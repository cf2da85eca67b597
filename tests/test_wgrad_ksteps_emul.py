"""The K steps of the weight-gradient kernel (conv_wgrad_v2_kernel, csrc/conv_igemm.cu) over the valid 8-pixel groups of a
stage, replayed on the CPU from the library's own plan and its own step enumeration (`lvg_convnd_wgrad_ksteps`, which
runs the kernel's `wgrad_kstep`).

A stage tile holds rows of `ps` pixels of which only the first `width` hold dy; the rest of each row is zero-filled by the
TMA. The kernel takes only the 8-pixel groups that hold dy pixels, two per wgmma K step. Checked here, for every
weight-gradient shape of the low-res and super-res steps, every shape of the envelope enumeration and a set of widths:
every valid pixel is read exactly once per product term (and so every (pixel, tap) pair, the taps being shifts of the
same offsets); no step reads past the first ceil(rows * ps / 16) * 16 pixels of the tile (what a walk over the whole pitch
reads, which the plan's shared-memory layout is sized for); the only other pixels read are zero-filled ones. The flat
shared-memory replay with garbage in the skipped row padding then matches torch's weight gradient."""
import ctypes
import itertools
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from torch_utils import custom_ops
from test_conv_envelope import accepted, enumerate_2d, enumerate_3d
from test_wgrad_emul import CASES, plan, tma_box, to_blocks8

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def ksteps(lib, shape, rows, seg):
    """[(offset of the first 8-pixel group, distance to the second)] of one stage, in pixels"""
    code, n, groups, cin, cout, sp, k, pad = shape
    out = (ctypes.c_int * 4096)()
    rc = lib.lvg_convnd_wgrad_ksteps(code, n, groups, cin, cout, *sp, *k, *pad, rows, seg, out, 4096)
    assert rc == 0, lib.lvg_last_error().decode()
    return [(int(out[1 + 2 * i]), int(out[2 + 2 * i])) for i in range(out[0])]


def stage_rows(ho, rh):
    """the dy row counts the kernel's stages take: full stages of rh rows and the last, shorter one"""
    return sorted({min(rh, ho)} | {ho - (-(-ho // rh) - 1) * rh})


def step_problems(steps, rows, width, ps):
    """what is wrong with the K steps of one stage (empty: nothing)"""
    bad = []
    gw = -(-width // 8)
    if len(steps) != -(-(rows * gw) // 2):
        bad.append(f'{len(steps)} steps for {rows} x {gw} groups')
    if ps == 8 * gw and steps != [(16 * i, 8) for i in range(len(steps))]:
        bad.append('a pitch without padding groups is not walked linearly (the kernel takes 16 pixels per step there)')
    limit = -(-(rows * ps) // 16) * 16
    count = np.zeros(limit + 16, dtype=np.int64)
    for off, d in steps:
        if not (off % 8 == 0 and d >= 8 and d % 8 == 0 and d < 1 << 14 and off + d + 8 <= limit):
            bad.append(f'step ({off}, {d}) outside the {limit} pixels a stage may read')
            continue
        count[off:off + 8] += 1
        count[off + d:off + d + 8] += 1
    px = np.arange(limit + 16)
    valid = (px // ps < rows) & (px % ps < width)
    if (count[valid] != 1).any():
        bad.append(f'valid pixels read {sorted(set(count[valid].tolist()))} times')
    # the other pixels read are TMA zero fill: row padding, or rows past the image (a stage of fewer than rh rows, or an
    # even rh behind an odd row count)
    if (count[~valid] > 1).any():
        bad.append('a zero-filled pixel read twice')
    return bad


def conv_shapes(path, nets):
    """(code, n, groups, cin, cout, (T, H, W), (kt, kh, kw), pad) of every convolution signature of a workload trace"""
    wl = json.load(open(os.path.join(ROOT, 'workloads', path)))
    out = set()
    for net in nets:
        for c in wl[net]:
            if c['op'] not in ('conv3d', 'conv2d', 'conv2d_resample') or 'w' not in c:
                continue
            xs, ws, g = c['x'], c['w'], c.get('groups', 1)
            nd = len(xs) - 2
            pad = c['padding'] if isinstance(c['padding'], list) else [c['padding']] * nd
            sp, k = (1,) * (3 - nd) + tuple(xs[2:]), (1,) * (3 - nd) + tuple(ws[2:])
            pad = (0,) * (3 - nd) + tuple(pad)
            out.add((1 if c.get('fp16') else 0, 8 if nd == 3 else xs[0], g, ws[1], ws[0] // g, sp, k, pad))
    return sorted(out)


def check_shapes(lib, shapes):
    bad, stages = [], 0
    for shape in shapes:
        code, n, groups, cin, cout, sp, k, pad = shape
        q = plan(code, n, groups, cin, cout, *sp, *k, *pad)
        ho = sp[1] + 2 * pad[1] - k[1] + 1
        for seg in range(q['nseg']):
            for rows in stage_rows(ho, q['rh']):
                stages += 1
                bad += [f'{shape} rows {rows} seg {seg}: {b}' for b in step_problems(ksteps(lib, shape, rows, seg), rows, q['seg_w'][seg], q['ps'])]
    return bad, stages


@pytest.fixture(scope='module')
def lib():
    return custom_ops.load_library()


def test_ksteps_of_the_workloads_cover_every_pixel_once(lib):
    shapes = conv_shapes('lres_step.json', ('lres_G', 'lres_D')) + conv_shapes('sres_step.json', ('sres_G', 'sres_D'))
    ok = []
    for code, n, groups, cin, cout, sp, k, pad in shapes:
        x = (n, groups * cin) + (sp if k[0] > 1 or sp[0] > 1 else sp[1:])
        w = (groups * cout, cin) + (k if k[0] > 1 or sp[0] > 1 else k[1:])
        if custom_ops.ConvNdPlugin._in_envelope(x, w, torch.float16 if code else torch.float32, 1, list(pad[3 - len(x) + 2:]), 1, groups):
            ok.append((code, n, groups, cin, cout, sp, k, pad))
    assert len(ok) >= 40
    bad, stages = check_shapes(lib, ok)
    assert stages >= len(ok)
    assert not bad, f'{len(bad)} problems, e.g.\n' + '\n'.join(bad[:20])


@pytest.mark.parametrize('code', [1, 0], ids=['f16', 'f32split'])
def test_ksteps_of_the_envelope_cover_every_pixel_once(lib, code):
    shapes = set()
    for n, groups, cin, cout, sp, k, pad, st, nd in itertools.chain(enumerate_2d(1), enumerate_3d()):
        if accepted(code, n, groups, cin, cout, sp, k, pad, st, nd):
            shapes.add((code, n, groups, cin, cout, tuple(sp), tuple(k), tuple(pad)))
    assert len(shapes) > 1000
    bad, _ = check_shapes(lib, sorted(shapes))
    assert not bad, f'{len(bad)} problems, e.g.\n' + '\n'.join(bad[:20])


def test_ksteps_of_narrow_rows():
    """width 16 rows: one K step per row; width 8: one per two rows; a partial group and an odd group count"""
    lib = custom_ops.load_library()
    for W, rows, want in ((16, 3, [(0, 8), (24, 8), (48, 8)]), (8, 4, [(0, 16), (32, 16)]), (8, 3, [(0, 16), (32, 8)]),
                          (4, 3, [(0, 8), (16, 8)]), (20, 1, [(0, 8), (16, 8)])):
        shape = (1, 1, 1, 32, 32, (1, 9, W), (1, 3, 3), (0, 1, 1))
        q = plan(*shape[:5], *shape[5], *shape[6], *shape[7])
        if q['rh'] < rows:
            continue
        got = ksteps(lib, shape, rows, 0)
        ps = q['ps']
        # expected offsets written for the pitch of each width: 16 -> 24, 8 -> 16, 4 -> 8, 20 -> 24 (2 halo columns)
        assert ps == {16: 24, 8: 16, 4: 8, 20: 24}[W], q
        assert got == want, (W, rows, got)


def emulate(x, dy, cin, cout, groups, k3, pad3, q, garbage, steps_of):
    """conv_wgrad_v2_kernel's data path on a flat model of shared memory, K steps from steps_of(rows, seg): x
    [n][G*cin][T][H][W], dy [n][G*cout][To][Ho][Wo] (float64) -> dw [G*cout][cin][kt][kh][kw]. Everything the TMA does not
    write holds `garbage`, and so do the zero-filled pitch columns of every dy row but a stage's last, past its last
    8-pixel group: the K steps must skip them."""
    n = x.shape[0]
    kt, kh, kw = k3
    pt, ph, pw = pad3
    T, H, W = x.shape[2:]
    To, Ho, Wo = dy.shape[2:]
    NT, ps, rh, khc, ablk = q['nt'], q['ps'], q['rh'], q['khc'], q['ablk']
    nop = 2 if q['split'] else 1
    dy8 = to_blocks8(dy.reshape(n * groups, cout, To, Ho, Wo), q['cpad_a']).reshape(-1, To, Ho, Wo, 8)
    x8 = to_blocks8(x.reshape(n * groups, cin, T, H, W), q['cpad_b']).reshape(-1, T, H, W, 8)
    nblk_a, nblk_b = q['cpad_a'] // 8, q['cpad_b'] // 8
    stage_px, tail_px = q['stage_bytes'] // 16, q['tail_bytes'] // 16
    a_px, b_px = q['a_stage'] // 16, q['b_stage'] // 16
    smem_px = q['stages'] * stage_px + tail_px
    dw = np.zeros((groups * cout, cin, kt, kh, kw))
    rblocks = -(-Ho // rh)
    total = n * To * q['nseg'] * rblocks
    blk_a, blk_b = rh * ps, (rh + khc - 1) * ps
    MR = q['mrows']
    for g, mti, nti, ktap in itertools.product(range(groups), range(q['mt']), range(q['ntiles']), range(kt)):
        for ky0 in ([0] if khc > 1 else range(kh)):
            D = np.zeros((khc * kw, MR, NT))
            for sp in range(q['nsplit']):
                s0, s1 = total * sp // q['nsplit'], total * (sp + 1) // q['nsplit']
                for it, s in enumerate(range(s0, s1)):
                    slot = it % q['stages']
                    rb, r = s % rblocks, s // rblocks
                    seg, r = r % q['nseg'], r // q['nseg']
                    tt, nn = r % To, r // To
                    inst = nn * groups + g
                    oy0 = rb * rh
                    rows = min(rh, Ho - oy0)
                    width = q['seg_w'][seg]
                    smem = np.full((smem_px, 8), garbage)
                    smem[q['stages'] * stage_px:] = 0.0
                    base = slot * stage_px
                    A = tma_box(dy8[:, :, :, q['seg_x0'][seg]:], inst * nblk_a + mti * 16, ablk, tt, oy0, rh, 0, ps, width)
                    A[:, :rows - 1, -(-width // 8) * 8:] = garbage
                    smem[base:base + a_px] = A.reshape(-1, 8)
                    Bt = tma_box(x8, inst * nblk_b + nti * (NT // 8), NT // 8, tt + ktap - pt, oy0 + ky0 - ph, rh + khc - 1, q['seg_x0'][seg] - pw, ps, W)
                    b_off = base + nop * a_px
                    smem[b_off:b_off + b_px] = Bt.reshape(-1, 8)
                    for off, d in steps_of(rows, seg):
                        pix = np.concatenate([off + np.arange(8), off + d + np.arange(8)])          # the 16 K positions
                        ia = base + (np.arange(MR) // 8)[:, None] * blk_a + pix[None, :]
                        assert ia.max() < smem_px, 'A rows read past the shared-memory allocation'
                        Am = smem[ia, (np.arange(MR) % 8)[:, None]]
                        for kyi, kx in itertools.product(range(khc), range(kw)):
                            ib = b_off + (np.arange(NT) // 8)[:, None] * blk_b + pix[None, :] + kyi * ps + kx
                            assert ib.max() < smem_px, 'x tile read past the shared-memory allocation'
                            D[kyi * kw + kx] += Am @ smem[ib, (np.arange(NT) % 8)[:, None]].T
            for kyi, kx in itertools.product(range(khc), range(kw)):
                for co in range(min(MR, cout - mti * 128)):
                    c = min(NT, cin - nti * NT)
                    dw[g * cout + mti * 128 + co, nti * NT:nti * NT + c, ktap, ky0 + kyi, kx] = D[kyi * kw + kx, co, :c]
    return dw


WIDTH_CASES = [(1, 1, 16, 24, (1, 7, W), (1, 3, 3), (0, 1, 1)) for W in (4, 8, 12, 16, 20, 32, 64, 86)] + \
              [(1, 1, 48, 40, (2, 5, W), (2, 1, 3), (1, 0, 1)) for W in (8, 20, 86)] + \
              [(1, 1, 24, 16, (1, 3, W), (1, 1, 1), (0, 0, 0)) for W in (8, 12)] + \
              [(1, 1, 16, 16, (1, 3, 300), (1, 3, 3), (0, 1, 1))] + list(CASES)


@pytest.mark.parametrize('dtype_code', [0, 1], ids=['f32split', 'f16'])
@pytest.mark.parametrize('case', WIDTH_CASES, ids=[f'{c[2]}->{c[3]} k{c[5]} {c[4]}' for c in WIDTH_CASES])
def test_wgrad_ksteps_replayed_on_cpu(case, dtype_code, monkeypatch):
    n, groups, cin, cout, (T, H, W), k3, pad3 = case
    lib = custom_ops.load_library()
    monkeypatch.setenv('LVG_WGRAD_FOLD_CIN', '64')
    for fold in (1, 0):
        monkeypatch.setenv('LVG_WGRAD_FOLD', str(fold))
        q = plan(dtype_code, n, groups, cin, cout, T, H, W, *k3, *pad3)
        shape = (dtype_code, n, groups, cin, cout, (T, H, W), k3, pad3)
        g = torch.Generator().manual_seed(7)
        x = torch.randn(n, groups * cin, T, H, W, generator=g, dtype=torch.float64)
        w = torch.zeros(groups * cout, cin, *k3, dtype=torch.float64, requires_grad=True)
        y = F.conv3d(x, w, padding=pad3, groups=groups)
        dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
        ref, = torch.autograd.grad(y, [w], dy)
        steps = {}

        def steps_of(rows, seg):
            if (rows, seg) not in steps:
                steps[rows, seg] = ksteps(lib, shape, rows, seg)
            return steps[rows, seg]
        res = [emulate(x.numpy(), dy.numpy(), cin, cout, groups, k3, pad3, q, garbage, steps_of) for garbage in (1e3, -7.0)]
        np.testing.assert_allclose(res[0], ref.numpy(), rtol=1e-9, atol=1e-9, err_msg=f'fold={fold} plan={q}')
        np.testing.assert_array_equal(res[0], res[1])
