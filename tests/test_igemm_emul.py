"""CPU replay of conv_igemm_kernel's addressing (csrc/conv_igemm.cu: forward and input gradient of the convolution engine)
with the tiling the library itself plans (`lvg_convnd_plan`, host arithmetic of the shipped library, no device needed).

What is replayed in numpy: the persistent tile loop and its decode order, the TMA boxes over the channel-block tensor X8
with hardware zero fill (halo rows / columns / frames), the stage layout in shared memory, a filter tap as a shift of the
linear pixel index (ky * tile_width + kx), the MMA over ALL accumulator columns including the halo columns that straddle
rows and frames (one instruction per tap and product at the tile's full width, ncols = 16 ... 256), the row order of the weight images (channels of a partial m-tile spread
over the four 32-row quarters), and the epilogue's map from (accumulator row, column) to (channel, frame, row, column) with the stride lattice of strided
convolutions -- against torch.nn.functional convolutions in float64. Checked besides the values: every read stays inside the
stage buffer (+ its slack), every output element is written exactly once, the shared-memory budget, and the
slot-invariance the resident weight images rely on. Not covered: descriptor bit fields, the instruction itself, the weight
re-tiling kernel's byte layout (the -m gpu tests do). Reference call sites: conv2d_gradfix.py:37-45, generator_lres.py:119,578,
discriminator_lres.py:121,172."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from torch_utils import custom_ops

FIELDS = ['wgroups', 'rows', 'mt', 'kc', 'nblk', 'nimg', 'lo_blk', 'to', 'ho', 'wo', 'kt', 'kh', 'kw', 'pad_t', 'pad_h', 'pad_w', 'tt', 'th',
          'wt', 'wtb', 'thb', 'frame_px', 'ncols', 'tiles_x', 'tiles_y', 'tiles_t', 'total_tiles', 'ks', 'stages',
          'a_resident', 'a_stage', 'b_step', 'b_bytes', 'b_box', 'stage_bytes', 'ostride', 'hos', 'wos']


def plan(mode, dtype_code, n, groups, cin, cout, t, h, w, k3, pad3, stride):
    lib = custom_ops.load_library()
    out = (ctypes.c_int * 48)()
    rc = lib.lvg_convnd_plan(mode, dtype_code, n, groups, cin, cout, t, h, w, *k3, *pad3, stride, out, 48)
    assert rc == 0, lib.lvg_last_error().decode()
    q = {k: int(out[i]) for i, k in enumerate(FIELDS)}
    q['pointwise'] = int(out[47])
    return q


def rows_per_quadrant(channels_left):
    cv = min(max(channels_left, 0), 128)
    return 32 if cv >= 128 else max(1, (cv + 3) // 4)


def row_of_channel(ch, per):
    if per >= 32:
        return ch
    if ch < 4 * per:
        return (ch // per) * 32 + ch % per
    r = ch - 4 * per
    return (r // (32 - per)) * 32 + per + r % (32 - per)


def emulate(X, A, q, n, groups, ck, cm, garbage):
    """X [n][G*ck][T][H][W] (the kernel's input grid, already dilated for strided input gradients); A [G][cm][ck][kt][kh][kw]
    logical weights (already mirrored / transposed for the input gradient) -> Y [n][G*cm][to][hos][wos] + write counts."""
    T, H, W = X.shape[2:]
    kt, kh, kw = q['kt'], q['kh'], q['kw']
    tt, th, wt, wtb, thb, fpx, ncols = q['tt'], q['th'], q['wt'], q['wtb'], q['thb'], q['frame_px'], q['ncols']
    os_ = q['ostride']
    cpad = q['kc'] * 16
    assert fpx == thb * wtb and q['b_box'] == 2 * tt * fpx * 16 and q['b_bytes'] >= q['b_box'] and q['b_bytes'] % 128 == 0
    assert ncols % 16 == 0 and 16 <= ncols <= 256 and wtb <= 128 and thb <= 256 and tt <= 256
    assert q['stages'] >= 2 and q['stages'] * q['stage_bytes'] + 128 <= 227 * 1024
    mma_cols = ncols                                       # one MMA per tap over the tile's full width
    kchunks = -(-q['kc'] // q['ks'])
    if q['a_resident']:
        assert q['stages'] % (kt * kchunks) == 0 and groups == 1 and q['mt'] == 1
    Y = np.full((n, groups * cm, q['to'], q['hos'], q['wos']), np.nan)
    cnt = np.zeros(Y.shape, dtype=np.int64)
    blk_px = tt * fpx                                      # pixels of one channel block of a k-step (LBO of the B descriptor)
    step_px = q['b_step'] // 16
    stage_b_px = (q['stage_bytes'] - q['a_stage']) // 16    # B part of a stage incl. the slack behind the last step
    for L in range(q['total_tiles']):
        r = L
        ox0 = (r % q['tiles_x']) * wt; r //= q['tiles_x']
        oy0 = (r % q['tiles_y']) * th; r //= q['tiles_y']
        t0 = (r % q['tiles_t']) * tt; r //= q['tiles_t']
        mti = r % q['mt']; inst = r // q['mt']
        nn, g = inst // groups, inst % groups
        Xp = np.zeros((cpad, T, H, W))
        Xp[:ck] = X[nn, g * ck:(g + 1) * ck]
        per = rows_per_quadrant(cm - mti * 128)
        D = np.zeros((128, mma_cols))
        for ktap in range(kt):
            for kcix in range(kchunks):
                k0 = kcix * q['ks']
                nks = min(q['ks'], q['kc'] - k0)
                smem = np.full((stage_b_px, 8), garbage)
                for j in range(nks):
                    for b in range(2):                     # the two 8-channel blocks of the k-step, written densely by TMA
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
                    for ky in range(kh):
                        for kx in range(kw):
                            Am = np.zeros((128, 16))
                            for ch in range(min(128, cm - mti * 128)):
                                kv = min(16, ck - kk)
                                if kv > 0:
                                    Am[row_of_channel(ch, per), :kv] = A[g, mti * 128 + ch, kk:kk + kv, ktap, ky, kx]
                            idx = j * step_px + (np.arange(16) // 8)[None, :] * blk_px + np.arange(mma_cols)[:, None] + ky * wtb + kx
                            assert idx.max() < stage_b_px, 'tap read past the stage buffer'
                            Bm = smem[idx, (np.arange(16) % 8)[None, :]]            # [mma_cols][16]
                            D += Am @ Bm.T
        for qd in range(4):
            m0 = mti * 128 + qd * per
            rows_ok = min(per, cm - m0)
            for lane in range(max(0, rows_ok)):
                for col in range(ncols):
                    f, rem = divmod(col, fpx)
                    rr, cc = divmod(rem, wtb)
                    ot, oy, ox = t0 + f, oy0 + rr, ox0 + cc
                    ok = f < tt and rr < th and cc < wt and ot < q['to'] and oy < q['ho'] and ox < q['wo']
                    if os_ > 1:
                        ok = ok and oy % os_ == 0 and ox % os_ == 0
                    if ok:
                        Y[nn, g * cm + m0 + lane, ot, oy // os_, ox // os_] = D[qd * 32 + lane, col]
                        cnt[nn, g * cm + m0 + lane, ot, oy // os_, ox // os_] += 1
    return Y, cnt


CASES = [
    # n, groups, cin, cout, (T, H, W), (kt, kh, kw), pad, stride
    (2, 1, 32, 32, (3, 9, 20), (1, 3, 3), (0, 1, 1), 1),       # few channels: rows spread over the lane quadrants, two k-steps
    (1, 1, 24, 30, (4, 3, 4), (3, 3, 3), (1, 1, 1), 1),        # small frames: several frames per tile, 30 channels (ragged quadrants)
    (1, 2, 20, 40, (1, 7, 9), (1, 3, 3), (0, 2, 2), 1),        # groups (modulated convolution), padding 2
    (1, 1, 16, 130, (1, 6, 10), (1, 3, 3), (0, 1, 1), 1),      # two m-tiles
    (1, 1, 16, 24, (1, 5, 150), (1, 3, 3), (0, 1, 1), 1),      # two column tiles
    (2, 1, 40, 24, (1, 9, 11), (1, 3, 3), (0, 0, 0), 2),       # stride 2, no padding (conv2d_resample down path)
    (1, 1, 16, 16, (1, 12, 14), (1, 3, 3), (0, 1, 1), 2),      # stride 2, padding 1
    (1, 1, 72, 40, (2, 5, 6), (1, 1, 1), (0, 0, 0), 1),        # 1x1x1: four k-steps per stage
    (2, 1, 64, 32, (1, 1, 16), (1, 1, 3), (0, 0, 1), 1),       # conv1d
    (1, 1, 16, 24, (7, 4, 6), (5, 3, 3), (2, 1, 1), 1),        # 5x3x3
    (1, 1, 16, 16, (1, 7, 100), (1, 3, 3), (0, 1, 1), 3),      # stride 3, rows wider than 3 x 85: narrower column tiles on the lattice
    (1, 1, 16, 16, (1, 9, 70), (1, 3, 3), (0, 1, 1), 4),       # stride 4, rows wider than 4 x 64
    (1, 1, 16, 16, (1, 3, 252), (1, 2, 2), (0, 1, 1), 2),      # 2x2 stride 2: column tiles rounded to the lattice stay <= 128 pixels
]


@pytest.mark.parametrize('mode', [0, 1], ids=['forward', 'input_gradient'])
@pytest.mark.parametrize('dtype_code', [0, 1], ids=['f32split', 'f16'])
@pytest.mark.parametrize('case', CASES, ids=[f'{c[2]}->{c[3]} k{c[5]} {c[4]} s{c[7]}' for c in CASES])
def test_forward_kernel_addressing_replayed_on_cpu(case, dtype_code, mode):
    n, groups, cin, cout, (T, H, W), k3, pad3, stride = case
    q = plan(mode, dtype_code, n, groups, cin, cout, T, H, W, k3, pad3, stride)
    if q['pointwise']:
        pytest.skip('this call takes the streaming 1x1x1 kernels')
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
        # the kernel's input: dy spread over every stride-th pixel of the stride-1 output grid; weights channel-transposed and mirrored
        to, ho, wo = T + 2 * pad3[0] - k3[0] + 1, H + 2 * pad3[1] - k3[1] + 1, W + 2 * pad3[2] - k3[2] + 1
        X = np.zeros((n, groups * cout, to, ho, wo))
        X[:, :, :, ::stride, ::stride] = dy.numpy()
        A = np.ascontiguousarray(wg.transpose(0, 2, 1, 3, 4, 5)[:, :, :, ::-1, ::-1, ::-1])
        ck, cm = cout, cin
    assert q['rows'] == cm
    res = [emulate(X, A, q, n, groups, ck, cm, garbage) for garbage in (1e3, -7.0)]
    Y, cnt = res[0]
    assert Y.shape == ref.shape, (Y.shape, ref.shape)
    assert (cnt == 1).all(), 'an output element was written %d..%d times' % (cnt.min(), cnt.max())
    np.testing.assert_allclose(Y, ref, rtol=1e-9, atol=1e-9, err_msg=str(q))
    np.testing.assert_array_equal(Y, res[1][0])              # whatever the TMA did not write never reaches an output
