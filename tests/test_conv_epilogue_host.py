"""The forward / input-gradient kernel's epilogue plan (`lvg_convnd_epilogue_plan`, host arithmetic only, no device needed)
for every convolution of the two training workloads, in both modes and dtypes.

  * The epilogue stores column pairs exactly when the tiling proves them: unit stride, even tile and box widths, an even
    output width and channel stride. Where it does, the column map of the tile (replayed here from `lvg_convnd_plan`)
    places every even column and its right neighbour on adjacent elements starting at an even offset, both stored or
    both dropped, and every tile's clipped width is even, so that no clip splits a pair.
  * The stage count is `lvg_convnd_plan`'s and the ring plus the column map fit the 227 KB of shared memory of a CTA."""
import ctypes
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, 'long-video-gan_b200'), os.path.join(ROOT, 'tests')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from torch_utils import custom_ops  # noqa: E402
import test_conv_host_plans as hp  # noqa: E402
import test_igemm_emul as emul  # noqa: E402

SMEM_PER_CTA = 227 * 1024
BARRIERS = 2 * 6 * 8            # full / empty mbarriers of the stage ring


@pytest.fixture(scope='module')
def lib():
    return custom_ops.load_library()


def calls():
    seen = []
    for c in hp.workload_convs():
        if c not in seen:
            seen.append(c)
    return seen


def plans(lib, mode, c):
    code, n, groups, cin, cout, sp, k, pad, stride = c
    args = (mode, code, n, groups, cin, cout, *sp, *k, *pad, stride)
    plan, epi = (ctypes.c_int * 48)(), (ctypes.c_int * 4)()
    rc_p = lib.lvg_convnd_plan(*args, plan, 48)
    rc_e = lib.lvg_convnd_epilogue_plan(*args, epi, 4)
    return rc_p, rc_e, list(plan), list(epi)


def column_map(q):
    """accumulator column -> (offset past the tile origin on the stored grid, (frame, row, col)) or None (not stored), as
    the kernel builds it"""
    cols = 2 * q['ncw'] if q['m64'] else q['ncw']
    out = []
    for n in range(cols):
        f, rem = divmod(n, q['frame_px'])
        r, cc = divmod(rem, q['wtb'])
        st = n < q['ncols'] and f < q['tt'] and r < q['th'] and cc < q['wt'] and r % q['ostride'] == 0 and cc % q['ostride'] == 0
        out.append(((f * q['hos'] + r // q['ostride']) * q['wos'] + cc // q['ostride'], (f, r, cc)) if st else None)
    return out


def pairs_proven(q):
    return q['ostride'] == 1 and q['wt'] % 2 == 0 and q['wtb'] % 2 == 0 and q['wo'] % 2 == 0 and (q['to'] * q['hos'] * q['wos']) % 2 == 0


@pytest.mark.parametrize('mode', [0, 1], ids=['fprop', 'dgrad'])
def test_workload_epilogue_plans(lib, mode):
    checked = 0
    for c in calls():
        rc_p, rc_e, plan, epi = plans(lib, mode, c)
        assert rc_e == rc_p, (c, rc_p, rc_e)
        if rc_p != 0:
            continue
        if plan[47]:
            assert epi[0] == -1, c
            continue
        q = dict(zip(emul.FIELDS, plan))
        q['m64'], q['ncw'] = plan[38], plan[39]
        assert epi[0] == int(pairs_proven(q)), (c, epi)
        assert epi[1] == q['stages'], (c, epi, q['stages'])
        assert epi[2] == q['stages'] * q['stage_bytes'] + 128, (c, epi)
        assert epi[2] + epi[3] + BARRIERS <= SMEM_PER_CTA, (c, epi)
        if epi[0] == 1:
            m = column_map(q)
            for n in range(0, len(m), 2):
                assert (m[n] is None) == (m[n + 1] is None), (c, n)
                if m[n] is not None:
                    assert m[n][0] % 2 == 0 and m[n + 1][0] == m[n][0] + 1, (c, n, m[n], m[n + 1])
                    assert m[n][1][:2] == m[n + 1][1][:2], (c, n)          # same frame and row
            for ix in range(q['tiles_x']):
                assert min(q['wt'], q['wo'] - ix * q['wt']) % 2 == 0, (c, ix)
        checked += 1
    assert checked > 20
