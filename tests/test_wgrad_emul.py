"""CPU replay of conv_wgrad_v2_kernel's addressing (csrc/conv_igemm.cu) with the tiling the library itself plans.

There is no GPU in the build container, so the geometry of the weight-gradient kernel -- TMA boxes with hardware zero
fill, the linear pixel index of the MN-major operands, taps as start-address shifts (kx: one pixel, ky: one tile row when
the tap rows are folded into one CTA), the compact dy operand whose missing rows read whatever follows in shared memory,
the split over the pixel range -- is replayed here in numpy on a flat model of the CTA's shared memory, using the numbers
`lvg_convnd_wgrad_plan` returns (host arithmetic of the shipped library, no device needed), and compared with torch's
weight gradient. What it checks: every read stays inside the CTA's shared-memory allocation, garbage rows never reach the
result, and the sums are the right ones. What it cannot check: descriptor bit fields and the tensor-core instruction
itself (the -m gpu tests do). Reference semantics: the weight gradient of F.conv3d (generator_lres.py:119,578,
discriminator_lres.py:172)."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from torch_utils import custom_ops

FIELDS = ['split', 'cpad_a', 'cpad_b', 'nt', 'ntiles', 'mt', 'nsplit', 'ablk', 'khc', 'nseg', 'ps', 'rh', 'stages', 'a_stage', 'b_stage',
          'stage_bytes', 'tail_bytes', 'smem']


def plan(dtype_code, n, groups, cin, cout, t, h, w, kt, kh, kw, pt, ph, pw):
    lib = custom_ops.load_library()
    out = (ctypes.c_int * 32)()
    rc = lib.lvg_convnd_wgrad_plan(dtype_code, n, groups, cin, cout, t, h, w, kt, kh, kw, pt, ph, pw, out, 32)
    assert rc == 0, lib.lvg_last_error().decode()
    q = {k: int(out[i]) for i, k in enumerate(FIELDS)}
    q['seg_w'] = [int(out[18 + j]) for j in range(4)]
    q['seg_x0'] = [int(out[22 + j]) for j in range(4)]
    q['mrows'] = int(out[27])
    return q


def to_blocks8(x, cpad):
    """[inst][c][t][h][w] -> [inst][cpad / 8][t][h][w][8] (zero channels beyond c): conv_pack_act_kernel's layout, one operand image"""
    inst, c = x.shape[:2]
    xp = np.zeros((inst, cpad) + x.shape[2:], dtype=x.dtype)
    xp[:, :c] = x
    return np.ascontiguousarray(xp.reshape(inst, cpad // 8, 8, *x.shape[2:]).transpose(0, 1, 3, 4, 5, 2))


def tma_box(src, blk0, nblk, t, y0, nrows, x0, ncols, w_extent):
    """box [nblk][nrows][ncols][8] of src [blocks][T][H][W][8] at (block blk0, frame t, row y0, column x0); elements outside
    the tensor (W clipped to w_extent) are zero"""
    B, T, H, W = src.shape[:4]
    out = np.zeros((nblk, nrows, ncols, 8), dtype=src.dtype)
    if not 0 <= t < T:
        return out
    for b in range(nblk):
        if not 0 <= blk0 + b < B:
            continue
        for r in range(nrows):
            y = y0 + r
            if not 0 <= y < H:
                continue
            lo, hi = max(0, -x0), min(ncols, min(W, w_extent) - x0)
            if hi > lo:
                out[b, r, lo:hi] = src[blk0 + b, t, y, x0 + lo:x0 + hi]
    return out


def emulate(x, dy, cin, cout, groups, k3, pad3, q, garbage):
    """x [n][G*cin][T][H][W], dy [n][G*cout][To][Ho][Wo] (float64) -> dw [G*cout][cin][kt][kh][kw] through the kernel's data path
    (one operand image per side: the hi/lo split repeats the same addressing on a second image)."""
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
    # shared memory in 16-byte units (= one pixel of one channel block); the lo images / the next stage hold `garbage`
    stage_px, tail_px = q['stage_bytes'] // 16, q['tail_bytes'] // 16
    a_px, b_px = q['a_stage'] // 16, q['b_stage'] // 16
    assert a_px == ablk * rh * ps and b_px == (NT // 8) * (rh + khc - 1) * ps
    assert q['stages'] >= 2 and q['stages'] * q['stage_bytes'] + q['tail_bytes'] + 128 <= q['smem'] <= 227 * 1024
    assert khc * kw * NT <= 256 and NT % 32 == 0 and rh + khc - 1 <= 256 and ps <= 128 and ablk <= 16 and NT // 8 <= 256
    smem_px = q['stages'] * stage_px + tail_px
    dw = np.zeros((groups * cout, cin, kt, kh, kw))
    rblocks = -(-Ho // rh)
    total = n * To * q['nseg'] * rblocks
    blk_a, blk_b = rh * ps, (rh + khc - 1) * ps
    max_read = 0
    for g in range(groups):
        for mti in range(q['mt']):
            for nti in range(q['ntiles']):
                for ktap in range(kt):
                    for ky0 in ([0] if khc > 1 else range(kh)):
                        MR = q['mrows']                                                    # rows of the MMA (64 when cout <= 64)
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
                                smem = np.full((smem_px, 8), garbage)
                                smem[q['stages'] * stage_px:] = 0.0                       # the tail is cleared once and never written
                                base = slot * stage_px
                                # A: dy8 through the map of this column segment (base shifted by seg_x0, W extent seg_w)
                                A = tma_box(dy8[:, :, :, q['seg_x0'][seg]:], inst * nblk_a + mti * 16, ablk, tt, oy0, rh, 0, ps, q['seg_w'][seg])
                                smem[base:base + a_px] = A.reshape(-1, 8)
                                Bt = tma_box(x8, inst * nblk_b + nti * (NT // 8), NT // 8, tt + ktap - pt, oy0 + ky0 - ph, rh + khc - 1,
                                             q['seg_x0'][seg] - pw, ps, W)
                                b_off = base + nop * a_px
                                smem[b_off:b_off + b_px] = Bt.reshape(-1, 8)
                                rows = min(rh, Ho - oy0)
                                ksteps = -(-(rows * ps) // 16)
                                # the lo images of the split (one image further) are read with the same offsets
                                assert base + (nop - 1) * a_px + (MR // 8 - 1) * blk_a + 16 * ksteps <= smem_px, 'lo dy image: rows read past the allocation'
                                assert b_off + (nop - 1) * b_px + (NT // 8 - 1) * blk_b + 16 * ksteps + (khc - 1) * ps + kw - 1 <= smem_px, \
                                    'lo x image read past the allocation'
                                for k in range(ksteps):
                                    # A operand: row m, K index j -> smem[(m / 8) * blk_a + 16 k + j][m % 8]  (all MR rows are read)
                                    ia = base + (np.arange(MR) // 8)[:, None] * blk_a + 16 * k + np.arange(16)[None, :]
                                    max_read = max(max_read, int(ia.max()))
                                    assert ia.max() < smem_px, 'A rows read past the shared-memory allocation'
                                    Am = smem[ia, (np.arange(MR) % 8)[:, None]]              # [MR][16]
                                    for kyi in range(khc):
                                        for kx in range(kw):
                                            ib = b_off + (np.arange(NT) // 8)[:, None] * blk_b + 16 * k + np.arange(16)[None, :] + kyi * ps + kx
                                            assert ib.max() < smem_px, 'x tile read past the shared-memory allocation'
                                            Bm = smem[ib, (np.arange(NT) % 8)[:, None]]      # [NT][16]
                                            D[kyi * kw + kx] += Am @ Bm.T
                        for kyi in range(khc):
                            for kx in range(kw):
                                for co in range(min(MR, cout - mti * 128)):
                                    for c in range(min(NT, cin - nti * NT)):
                                        dw[g * cout + mti * 128 + co, nti * NT + c, ktap, ky0 + kyi, kx] = D[kyi * kw + kx, co, c]
    return dw, max_read


CASES = [
    # n, groups, cin, cout, (T, H, W), (kt, kh, kw), pad
    (2, 1, 32, 32, (2, 6, 20), (1, 3, 3), (0, 1, 1)),          # folded, compact (the low-res discriminator's 32 -> 32 layer, reduced)
    (1, 1, 64, 64, (3, 5, 12), (3, 3, 3), (1, 1, 1)),          # folded: two n-tiles of 32
    (1, 1, 64, 128, (2, 4, 8), (1, 3, 3), (0, 1, 1)),          # folded, full m-tile
    (1, 1, 48, 40, (1, 9, 20), (1, 3, 3), (0, 1, 1)),          # n-tile 48, pitch 8 mod 16 (row pairs), odd row count
    (2, 1, 8, 16, (1, 5, 7), (1, 3, 3), (0, 1, 1)),            # two dy blocks: the longest over-read
    (1, 1, 3, 24, (3, 6, 10), (3, 3, 3), (1, 1, 1)),
    (1, 2, 24, 40, (1, 7, 9), (1, 3, 3), (0, 2, 2)),           # groups (modulated convolution), padding 2
    (1, 1, 16, 20, (3, 8, 30), (3, 3, 3), (0, 0, 0)),          # no padding
    (1, 1, 27, 72, (1, 4, 150), (1, 3, 3), (0, 2, 2)),         # two column segments
    (1, 1, 32, 32, (1, 8, 12), (1, 3, 1), (0, 1, 0)),          # 3x1 kernel
    (1, 1, 80, 130, (1, 5, 9), (1, 3, 3), (0, 1, 1)),          # not folded (cin > 64), two m-tiles, padded dy8
    (1, 1, 64, 32, (1, 4, 16), (1, 1, 3), (0, 0, 1)),          # kh = 1: nothing to fold
]


@pytest.mark.parametrize('dtype_code', [0, 1], ids=['f32split', 'f16'])
@pytest.mark.parametrize('case', CASES, ids=[f'{c[2]}->{c[3]} k{c[5]} {c[4]}' for c in CASES])
def test_wgrad_kernel_addressing_replayed_on_cpu(case, dtype_code, monkeypatch):
    n, groups, cin, cout, (T, H, W), k3, pad3 = case
    monkeypatch.setenv('LVG_WGRAD_FOLD_CIN', '64')        # fold wherever the accumulators fit (default: up to 32 input channels)
    for fold, compact in ((1, 1), (0, 1), (1, 0), (0, 0)):
        monkeypatch.setenv('LVG_WGRAD_FOLD', str(fold))
        monkeypatch.setenv('LVG_WGRAD_COMPACT', str(compact))
        q = plan(dtype_code, n, groups, cin, cout, T, H, W, *k3, *pad3)
        assert q['khc'] == (k3[1] if (fold and k3[1] > 1 and cin <= 64 and k3[1] * k3[2] * 32 <= 256) else 1)
        assert q['ablk'] == (-(-cout // 16) * 2 if (compact and cout < 128) else 16)
        assert q['mrows'] == (64 if (compact and cout <= 64) else 128)
        g = torch.Generator().manual_seed(5)
        x = torch.randn(n, groups * cin, T, H, W, generator=g, dtype=torch.float64)
        w = torch.zeros(groups * cout, cin, *k3, dtype=torch.float64, requires_grad=True)
        y = F.conv3d(x, w, padding=pad3, groups=groups)
        dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
        ref, = torch.autograd.grad(y, [w], dy)
        # two different fillers for everything the TMA did not write: the result must not depend on it
        res = [emulate(x.numpy(), dy.numpy(), cin, cout, groups, k3, pad3, q, garbage)[0] for garbage in (1e3, -7.0)]
        np.testing.assert_allclose(res[0], ref.numpy(), rtol=1e-9, atol=1e-9, err_msg=f'fold={fold} compact={compact} plan={q}')
        np.testing.assert_array_equal(res[0], res[1])


def test_wgrad_plans_of_the_lowres_networks_fit_the_hardware(monkeypatch):
    """Every conv3d signature of one low-res G+D pass (workloads/lres_step.json), batch 8: the plan's shared memory, register
    accumulator columns and TMA boxes are inside the limits, and the few-channel layers are folded where their accumulators fit."""
    import json
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    wl = json.load(open(os.path.join(root, 'workloads', 'lres_step.json')))
    seen = 0
    for c in wl['lres_G'] + wl['lres_D']:
        if c.get('op') != 'conv3d' or c.get('groups', 1) != 1:
            continue
        xs, ws = c['x'], c['w']
        pad = c['padding'] if isinstance(c['padding'], (list, tuple)) else [c['padding']] * 3
        q = plan(0, 8, 1, ws[1], ws[0], xs[2], xs[3], xs[4], ws[2], ws[3], ws[4], *pad)
        seen += 1
        assert q['smem'] <= 227 * 1024 and q['stages'] >= 2, (c, q)
        assert q['khc'] * ws[4] * q['nt'] <= 256 and q['nt'] % 32 == 0 and q['rh'] + q['khc'] - 1 <= 256 and q['ps'] <= 128, (c, q)
        assert q['khc'] == (ws[3] if ws[3] > 1 and ws[1] <= 32 and ws[3] * ws[4] * 32 <= 256 else 1), (c, q)
    assert seen >= 10
