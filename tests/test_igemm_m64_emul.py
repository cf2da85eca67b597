"""CPU replay of the 64-row mode of conv_igemm_kernel (csrc/conv_igemm.cu: forward / input-gradient GEMMs with at most 64
rows) with the tiling the library plans (`lvg_convnd_plan`, host arithmetic only), as tests/test_igemm_emul.py replays the
128-row mode: 64-row weight images with row = channel, both consumer warpgroups reading the same A, warpgroup c computing
accumulator columns [c N, c N + N) with N the planned per-warpgroup MMA width (ncols / 2 rounded up to 16), every read
inside the stage buffer plus its slack, columns >= ncols dropped, every output element written exactly once, and the
values against torch.nn.functional convolutions in float64."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from torch_utils import custom_ops

FIELDS = ['wgroups', 'rows', 'mt', 'kc', 'nblk', 'nimg', 'lo_blk', 'to', 'ho', 'wo', 'kt', 'kh', 'kw', 'pad_t', 'pad_h', 'pad_w', 'tt', 'th',
          'wt', 'wtb', 'thb', 'frame_px', 'ncols', 'tiles_x', 'tiles_y', 'tiles_t', 'total_tiles', 'ks', 'stages',
          'a_resident', 'a_stage', 'b_step', 'b_bytes', 'b_box', 'stage_bytes', 'ostride', 'hos', 'wos', 'm64', 'ncw']


def plan(mode, dtype_code, n, groups, cin, cout, t, h, w, k3, pad3, stride):
    lib = custom_ops.load_library()
    out = (ctypes.c_int * 48)()
    rc = lib.lvg_convnd_plan(mode, dtype_code, n, groups, cin, cout, t, h, w, *k3, *pad3, stride, out, 48)
    assert rc == 0, lib.lvg_last_error().decode()
    q = {k: int(out[i]) for i, k in enumerate(FIELDS)}
    q['pointwise'] = int(out[47])
    return q


def emulate(X, A, q, n, groups, ck, cm, garbage):
    T, H, W = X.shape[2:]
    kt, kh, kw = q['kt'], q['kh'], q['kw']
    tt, th, wt, wtb, thb, fpx, ncols, ncw = q['tt'], q['th'], q['wt'], q['wtb'], q['thb'], q['frame_px'], q['ncols'], q['ncw']
    os_ = q['ostride']
    cpad = q['kc'] * 16
    assert q['m64'] == 1 and q['mt'] == 1 and cm <= 64
    assert ncw % 16 == 0 and ncw == -(-(ncols // 2) // 16) * 16 and ncols <= 256
    # the A part of a stage holds 64-row images: 2048 bytes per (k-step, tap, operand half)
    assert q['a_stage'] == q['ks'] * kh * kw * q['nimg'] * 2048
    assert q['stages'] >= 2 and q['stages'] * q['stage_bytes'] + 128 <= 227 * 1024
    kchunks = -(-q['kc'] // q['ks'])
    Y = np.full((n, groups * cm, q['to'], q['hos'], q['wos']), np.nan)
    cnt = np.zeros(Y.shape, dtype=np.int64)
    blk_px = tt * fpx
    step_px = q['b_step'] // 16
    stage_b_px = (q['stage_bytes'] - q['a_stage']) // 16
    for L in range(q['total_tiles']):
        r = L
        ox0 = (r % q['tiles_x']) * wt; r //= q['tiles_x']
        oy0 = (r % q['tiles_y']) * th; r //= q['tiles_y']
        t0 = (r % q['tiles_t']) * tt; r //= q['tiles_t']
        inst = r // q['mt']
        nn, g = inst // groups, inst % groups
        Xp = np.zeros((cpad, T, H, W))
        Xp[:ck] = X[nn, g * ck:(g + 1) * ck]
        D = [np.zeros((64, ncw)) for _ in range(2)]           # the two consumer warpgroups
        for ktap in range(kt):
            for kcix in range(kchunks):
                k0 = kcix * q['ks']
                nks = min(q['ks'], q['kc'] - k0)
                smem = np.full((stage_b_px, 8), garbage)
                for j in range(nks):
                    for b in range(2):
                        c0 = (k0 + j) * 16 + b * 8
                        box = np.zeros((tt, thb, wtb, 8))
                        for f in range(tt):
                            ft = t0 + ktap - q['pad_t'] + f
                            if not 0 <= ft < T:
                                continue
                            for rr in range(thb):
                                yy = oy0 - q['pad_h'] + rr
                                if not 0 <= yy < H:
                                    continue
                                x0 = ox0 - q['pad_w']
                                lo, hi = max(0, -x0), min(wtb, W - x0)
                                if hi > lo:
                                    box[f, rr, lo:hi] = Xp[c0:c0 + 8, ft, yy, x0 + lo:x0 + hi].T
                        smem[j * step_px + b * blk_px:j * step_px + (b + 1) * blk_px] = box.reshape(-1, 8)
                for j in range(nks):
                    kk = (k0 + j) * 16
                    kv = min(16, ck - kk)
                    for ky in range(kh):
                        for kx in range(kw):
                            Am = np.zeros((64, 16))                  # image row = channel
                            if kv > 0:
                                Am[:cm, :kv] = A[g, :cm, kk:kk + kv, ktap, ky, kx]
                            for cw in range(2):
                                cols = cw * ncw + np.arange(ncw)
                                idx = j * step_px + (np.arange(16) // 8)[None, :] * blk_px + cols[:, None] + ky * wtb + kx
                                assert idx.max() < stage_b_px, 'tap read past the stage buffer'
                                D[cw] += Am @ smem[idx, (np.arange(16) % 8)[None, :]].T
        for cw in range(2):
            for ch in range(cm):
                for lc in range(ncw):
                    col = cw * ncw + lc
                    f, rem = divmod(col, fpx)
                    rr, cc = divmod(rem, wtb)
                    ot, oy, ox = t0 + f, oy0 + rr, ox0 + cc
                    ok = col < ncols and f < tt and rr < th and cc < wt and ot < q['to'] and oy < q['ho'] and ox < q['wo']
                    if os_ > 1:
                        ok = ok and oy % os_ == 0 and ox % os_ == 0
                    if ok:
                        Y[nn, g * cm + ch, ot, oy // os_, ox // os_] = D[cw][ch, lc]
                        cnt[nn, g * cm + ch, ot, oy // os_, ox // os_] += 1
    return Y, cnt


CASES = [
    # n, groups, cin, cout, (T, H, W), (kt, kh, kw), pad, stride   (M = cout forward, cin input gradient)
    (2, 1, 1, 1, (1, 5, 9), (1, 3, 3), (0, 1, 1), 1),          # M = 1
    (1, 1, 3, 3, (3, 6, 7), (3, 3, 3), (1, 1, 1), 1),          # M = 3, several frames per tile
    (2, 1, 30, 30, (2, 9, 20), (1, 3, 3), (0, 1, 1), 1),       # M = 30, two k-steps
    (1, 1, 32, 32, (4, 4, 6), (3, 3, 3), (1, 1, 1), 1),        # M = 32, small frames
    (1, 1, 64, 64, (1, 7, 12), (1, 3, 3), (0, 1, 1), 1),       # M = 64
    (1, 2, 20, 24, (1, 7, 9), (1, 3, 3), (0, 2, 2), 1),        # groups, padding 2
    (2, 1, 40, 24, (1, 9, 11), (1, 3, 3), (0, 0, 0), 2),       # stride 2, no padding
    (1, 1, 16, 16, (1, 12, 14), (1, 3, 3), (0, 1, 1), 2),      # stride 2, padding 1
    (1, 1, 16, 24, (1, 5, 150), (1, 3, 3), (0, 1, 1), 1),      # two column tiles
    (1, 1, 16, 24, (7, 4, 6), (5, 3, 3), (2, 1, 1), 1),        # 5x3x3, multi-frame tiles
]


@pytest.mark.parametrize('mode', [0, 1], ids=['forward', 'input_gradient'])
@pytest.mark.parametrize('dtype_code', [0, 1], ids=['f32split', 'f16'])
@pytest.mark.parametrize('case', CASES, ids=[f'{c[2]}->{c[3]} k{c[5]} {c[4]} g{c[1]} s{c[7]}' for c in CASES])
def test_64_row_mode_replayed_on_cpu(case, dtype_code, mode):
    n, groups, cin, cout, (T, H, W), k3, pad3, stride = case
    q = plan(mode, dtype_code, n, groups, cin, cout, T, H, W, k3, pad3, stride)
    assert not q['pointwise']
    g = torch.Generator().manual_seed(9)
    x = torch.randn(n, groups * cin, T, H, W, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(groups * cout, cin, *k3, generator=g, dtype=torch.float64)
    y = F.conv3d(x, w, stride=(1, stride, stride), padding=pad3, groups=groups)
    wg = w.reshape(groups, cout, cin, *k3).numpy()
    if mode == 0:
        X, A, ck, cm, ref = x.detach().numpy(), wg, cin, cout, y.detach().numpy()
    else:
        dy = torch.randn(y.shape, generator=g, dtype=torch.float64)
        ref = torch.autograd.grad(y, [x], dy)[0].numpy()
        to, ho, wo = T + 2 * pad3[0] - k3[0] + 1, H + 2 * pad3[1] - k3[1] + 1, W + 2 * pad3[2] - k3[2] + 1
        X = np.zeros((n, groups * cout, to, ho, wo))
        X[:, :, :, ::stride, ::stride] = dy.numpy()
        A = np.ascontiguousarray(wg.transpose(0, 2, 1, 3, 4, 5)[:, :, :, ::-1, ::-1, ::-1])
        ck, cm = cout, cin
    assert q['rows'] == cm
    res = [emulate(X, A, q, n, groups, ck, cm, garbage) for garbage in (1e3, -7.0)]
    Y, cnt = res[0]
    assert Y.shape == ref.shape
    assert (cnt == 1).all(), 'an output element was written %d..%d times' % (cnt.min(), cnt.max())
    np.testing.assert_allclose(Y, ref, rtol=1e-9, atol=1e-9, err_msg=str(q))
    np.testing.assert_array_equal(Y, res[1][0])


def test_128_rows_above_64():
    q = plan(0, 0, 1, 1, 16, 65, 1, 7, 12, (1, 3, 3), (0, 1, 1), 1)
    assert q['m64'] == 0 and q['ncw'] == q['ncols']
