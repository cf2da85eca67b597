"""The convolution engine's host arithmetic, pinned (no device needed).

tests/golden/conv_host_plans.npz holds what the library answered, for a fixed set of calls, to
  * `lvg_convnd_plan` (forward and input gradient), `lvg_convnd_wgrad_plan` and `lvg_convnd_route`: the tilings and routes
    the launches take. They must not change;
  * the seven workspace size queries (`convnd`, `convnd_wgrad`, `convnd_backward`, `modconv`, `sres_dblock_conv1` and its
    backward, `sres_layer`): a size may shrink where a formula asked for more than the calls carve, but it never grows (the
    plugin layer's workspace cache must not start to allocate where it did not), and a call the library refused stays
    refused and the other way round.
The calls: the shapes of tests/test_conv_envelope.py's enumerators, every convolution of workloads/lres_step.json and
workloads/sres_step.json (in both dtypes, at batch 1 and 4), and modulated-convolution, super-res discriminator conv1 and
super-res generator layer shapes, including the 181- and 362-channel layers whose two gradients tile dy differently.

`python tests/test_conv_host_plans.py --write` rewrites the fixture from the library that is built."""
import ctypes
import itertools
import json
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, 'long-video-gan_b200'), os.path.join(ROOT, 'tests')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from torch_utils import custom_ops  # noqa: E402
from torch_utils.ops import sres_cond as sc  # noqa: E402
import test_conv_envelope as env  # noqa: E402

GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'conv_host_plans.npz')


def workload_convs():
    """(code, n, groups, cin, cout, (t, h, w), (kt, kh, kw), (pt, ph, pw), stride) of every convolution the two training
    workloads run, as the engine sees it; conv2d_resample with down = 2 as its strided 3x3 convolution on the filtered
    (h + 1) x (w + 1) image, or its 1x1 convolution on the down-sampled image."""
    for name in ('lres_step.json', 'sres_step.json'):
        with open(os.path.join(ROOT, 'workloads', name)) as f:
            ops = [o for k, v in json.load(f).items() if k != 'meta' for o in v]
        for o in ops:
            if 'w' not in o or 'conv' not in o['op']:
                continue
            x, w, g = o['x'], o['w'], o['groups']
            pad = o['padding'] if isinstance(o['padding'], list) else [o['padding']] * (len(w) - 2)
            sp, k, p = [1, 1, 1], [1, 1, 1], [0, 0, 0]
            sp[3 - len(x[2:]):], k[3 - len(w[2:]):], p[3 - len(pad):] = x[2:], w[2:], pad
            stride = o['stride'] if isinstance(o.get('stride'), int) else 1
            if o['op'] == 'conv2d_resample' and o['down'] == 2:
                if k[2] == 3:
                    sp, p, stride = [1, sp[1] + 1, sp[2] + 1], [0, 0, 0], 2
                else:
                    sp = [1, sp[1] // 2, sp[2] // 2]
            for code, n in itertools.product((0, 1), (1, 4)):
                yield (code, x[0] * n, g, x[1] // g, w[0] // g, tuple(sp), tuple(k), tuple(p), stride)


def envelope_convs():
    for stride in (1, 2, 3, 4):
        for code in (1, 0):
            for n, groups, cin, cout, sp, k, pad, st, nd in env.enumerate_2d(stride):
                if env.accepted(code, n, groups, cin, cout, sp, k, pad, st, nd):
                    yield (code, n, groups, cin, cout, sp, k, pad, st)
    for code in (1, 0):
        for n, groups, cin, cout, sp, k, pad, st, nd in env.enumerate_3d():
            if env.accepted(code, n, groups, cin, cout, sp, k, pad, st, nd):
                yield (code, n, groups, cin, cout, sp, k, pad, st)


def modconv_convs():
    """Modulated convolutions (groups 1, stride 1): the super-res generator's layers, a 1x1 one, the low-res generator's."""
    for code, (cin, cout, h, w, k, p) in itertools.product((0, 1), [
            (27, 512, 29, 36, 3, 2), (539, 512, 38, 52, 3, 2), (539, 362, 92, 148, 3, 2), (389, 256, 92, 148, 3, 2),
            (283, 181, 164, 276, 3, 2), (208, 128, 164, 276, 3, 2), (155, 128, 164, 276, 3, 1), (155, 3, 144, 256, 1, 0),
            (512, 512, 9, 16, 3, 1), (181, 181, 20, 30, 3, 1), (362, 362, 20, 30, 3, 1), (64, 64, 36, 64, 1, 0)]):
        yield (code, 8, 1, cin, cout, (1, h, w), (1, k, k), (0, p, p), 1)


def conv_cases():
    seen, out = set(), []
    for c in itertools.chain(envelope_convs(), workload_convs(), modconv_convs()):
        flat = (c[0], c[1], c[2], c[3], c[4], *c[5], *c[6], *c[7], c[8])
        if flat not in seen:
            seen.add(flat)
            out.append(flat)
    return np.array(out, dtype=np.int32)


def conv1_cases():
    """(code, n, cin, cout, h, w) of lvg_sres_dblock_conv1: the super-res discriminator's down-sampling 3x3 layers."""
    layers = [(64, 128, 256, 256), (128, 256, 128, 128), (256, 512, 64, 64), (512, 512, 32, 32), (512, 512, 16, 16),
              (512, 512, 8, 8), (24, 40, 9, 13), (3, 181, 20, 30), (181, 362, 17, 33), (16, 16, 2, 2), (16, 16, 1, 8)]
    return np.array([(code, n, *l) for code, n, l in itertools.product((0, 1), (1, 4, 8), layers)], dtype=np.int32)


def layer_cases():
    """lvg_sres_layer_workspace's arguments: (code, n, t, c, c_lr, window, t_lr, h_lr, w_lr, plan_h[10], plan_w[10], cout,
    kh, kw, pad_h, pad_w) for the super-res generator's layers (c x_prev channels and 27 conditioning channels)."""
    rows = []
    for (c, cout, h, w, k), code, n in itertools.product(
            [(0, 512, 29, 36, 3), (512, 512, 38, 52, 3), (512, 362, 92, 148, 3), (362, 256, 92, 148, 3), (256, 181, 164, 276, 3),
             (181, 128, 164, 276, 3), (128, 128, 164, 276, 3), (128, 3, 164, 276, 1), (357, 181, 56, 84, 3)], (0, 1), (1, 8)):
        a_h = sc.axis_plan(36, 64, 10, 'up', 4, 24, True, h)
        a_w = sc.axis_plan(64, 64, 10, 'up', 4, 24, True, w)
        p = k // 2 + 1 if k > 1 else 0
        rows.append((code, n, 8, c, 3, 9, 16, a_h.len, a_w.len, *sc._ints(a_h), *sc._ints(a_w), cout, k, k, p, p))
    return np.array(rows, dtype=np.int32)


def query(lib):
    conv, conv1, layer = conv_cases(), conv1_cases(), layer_cases()
    plan0 = np.zeros((len(conv), 49), np.int32)
    plan1 = np.zeros((len(conv), 49), np.int32)
    wplan = np.zeros((len(conv), 33), np.int32)
    route = np.zeros((len(conv), 4), np.int32)
    ws = np.zeros((len(conv), 4), np.int64)        # convnd, convnd_wgrad, convnd_backward, modconv
    for i, r in enumerate(conv.tolist()):
        code, n, groups, cin, cout, t, h, w, kt, kh, kw, pt, ph, pw, stride = r
        a = (code, n, groups, cin, cout, t, h, w, kt, kh, kw, pt, ph, pw)
        for mode, dst in ((0, plan0), (1, plan1)):
            out = (ctypes.c_int * 48)()
            dst[i, 0] = lib.lvg_convnd_plan(mode, *a, stride, out, 48)
            dst[i, 1:] = list(out)
        out = (ctypes.c_int * 32)()
        wplan[i, 0] = lib.lvg_convnd_wgrad_plan(*a, out, 32)
        wplan[i, 1:] = list(out)
        route[i] = [lib.lvg_convnd_route(0, *a, stride, 0), lib.lvg_convnd_route(0, *a, stride, 1),
                    lib.lvg_convnd_route(1, *a, stride, 0), lib.lvg_convnd_route(2, *a, stride, 0)]
        ws[i] = [lib.lvg_convnd_workspace(*a), lib.lvg_convnd_wgrad_workspace(*a), lib.lvg_convnd_backward_workspace(*a),
                 lib.lvg_modconv_workspace(code, n, cin, cout, t, h, w, kt, kh, kw, pt, ph, pw)]
    ws1 = np.array([[lib.lvg_sres_dblock_conv1_workspace(*r), lib.lvg_sres_dblock_conv1_backward_workspace(*r)]
                    for r in conv1.tolist()], np.int64)
    wsl = []
    for r in layer.tolist():
        ph, pw = (ctypes.c_int * 10)(*r[9:19]), (ctypes.c_int * 10)(*r[19:29])
        wsl.append(lib.lvg_sres_layer_workspace(*r[:9], ph, pw, *r[29:]))
    return dict(conv=conv, plan0=plan0, plan1=plan1, wplan=wplan, route=route, ws=ws, conv1=conv1, ws_conv1=ws1, layer=layer,
                ws_layer=np.array(wsl, np.int64)[:, None])


def to_planes(a):
    """[rows][cols] -> [cols][byte][rows]: columns of sizes and tilings vary slowly, so the fixture compresses ~4x better."""
    a = np.ascontiguousarray(a.T)
    return np.ascontiguousarray(a.view(np.uint8).reshape(a.shape + (a.itemsize,)).transpose(0, 2, 1))


def from_planes(p, dtype):
    return np.ascontiguousarray(p.transpose(0, 2, 1)).view(dtype)[..., 0].T


@pytest.fixture(scope='module')
def pinned():
    with np.load(GOLDEN) as f:
        return {k: from_planes(f[k], np.int64 if k.startswith('ws') else np.int32) for k in f.files}


@pytest.fixture(scope='module')
def now():
    return query(custom_ops.load_library())


def test_same_calls(pinned, now):
    """The calls above are the ones the fixture was written for."""
    for k in ('conv', 'conv1', 'layer'):
        np.testing.assert_array_equal(now[k], pinned[k])


@pytest.mark.parametrize('key', ['plan0', 'plan1', 'wplan', 'route'])
def test_plans_and_routes_unchanged(pinned, now, key):
    bad = np.nonzero((now[key] != pinned[key]).any(axis=1))[0]
    assert not len(bad), f'{len(bad)} calls differ, e.g. {pinned["conv"][bad[0]].tolist()}: {now[key][bad[0]].tolist()} ' \
                         f'instead of {pinned[key][bad[0]].tolist()}'


@pytest.mark.parametrize('key', ['ws', 'ws_conv1', 'ws_layer'])
def test_workspace_sizes_never_grow(pinned, now, key):
    old, new = pinned[key], now[key]
    assert np.array_equal(new < 0, old < 0), f'{key}: a size query changed between a refusal and a size'
    grew = np.argwhere((new > old) & (old >= 0))
    assert not len(grew), f'{key}: {len(grew)} sizes grew, e.g. entry {grew[0].tolist()}: {new[tuple(grew[0])]} > {old[tuple(grew[0])]}'


if __name__ == '__main__':
    if sys.argv[1:] != ['--write']:
        sys.exit('usage: python tests/test_conv_host_plans.py --write')
    res = query(custom_ops.load_library())
    np.savez_compressed(GOLDEN, **{k: to_planes(v) for k, v in res.items()})
    print(GOLDEN, {k: v.shape for k, v in res.items()}, os.path.getsize(GOLDEN), 'bytes')
