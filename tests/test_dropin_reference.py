"""Drop-in rule (DESIGN.md section 1): with `long-video-gan_b200/` ahead of the LongVideoGAN code on PYTHONPATH the
reference's own `model/*` code imports THIS repository's `torch_utils.ops` while `torch_utils.misc`, `dnnlib`, ... still
come from the reference -- and the networks compute what they compute on the reference's own ops. Runs the unmodified
reference generators and discriminator on CPU (where both resolve to compositions of standard torch ops) in a
subprocess over this package and compares the outputs with tests/golden/dropin_reference.npz: the same run over the
reference's own ops (tests/dropin_reference_run.py, same seeds), stored as a fixed sample of every output tensor
(np.unique(default_rng(0).integers(0, n, 16384)) flat indices), the full shape and max |output|. The file was recorded
from the reference's own ops by running this module as a script:

    cd <reference checkout>; PYTHONPATH=. CUDA_VISIBLE_DEVICES= python <repo>/tests/dropin_reference_run.py /tmp/ref.pt
    python <repo>/tests/test_dropin_reference.py --record /tmp/ref.pt

(`--record` refuses a run whose ops did not come from the reference; the npz's `provenance` entry names the ops' files).

The reference's model code comes from a checkout named by LVG_REFERENCE_CHECKOUT, or from the staged copy that
oracle/build_ref.py leaves in oracle/_ref/src; the test skips when neither is present."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'dropin_reference.npz')


def _reference_code():
    for d in (os.environ.get('LVG_REFERENCE_CHECKOUT'), os.path.join(ROOT, 'oracle', '_ref', 'src')):
        if d and os.path.isdir(os.path.join(d, 'model')) and os.path.isdir(os.path.join(d, 'dnnlib')):
            return os.path.abspath(d)
    return None


REFERENCE = _reference_code()
pytestmark = pytest.mark.skipif(REFERENCE is None, reason='no LongVideoGAN model code (checkout or oracle/_ref/src) available')


def _sample(t):
    flat = t.detach().double().numpy().reshape(-1)
    idx = np.unique(np.random.default_rng(0).integers(0, flat.size, size=min(flat.size, 16384)))
    return flat, idx


def record(ref_pt):
    """tests/golden/dropin_reference.npz from a dropin_reference_run.py output of the reference on its own ops."""
    t = torch.load(ref_pt)
    assert 'long-video-gan_b200' not in t['where']['bias_act'] and 'long-video-gan_b200' not in t['where']['upfirdn2d'], t['where']
    root = os.path.dirname(os.path.dirname(t['where']['dnnlib']))        # the checkout the run imported
    out = {'provenance': np.array('tests/dropin_reference_run.py over the reference checkout, ops from ' +
                                  ', '.join(f'{k}={os.path.relpath(v, root)}' for k, v in sorted(t['where'].items())))}
    for name in ('lres_G', 'lres_D', 'sres_G'):
        flat, idx = _sample(t[name])
        out[name + '_shape'] = np.array(t[name].shape, np.int64)
        out[name + '_values'] = flat[idx].astype(np.float32)
        out[name + '_absmax'] = np.array(np.abs(flat).max(), np.float64)
    np.savez_compressed(GOLDEN, **out)


def _run(pythonpath, out_file):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(pythonpath), CUDA_VISIBLE_DEVICES='')
    subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'dropin_reference_run.py'), out_file], check=True, env=env,
                   cwd=REFERENCE, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL, timeout=1200)
    return torch.load(out_file)


def test_reference_networks_run_unchanged_on_the_dropped_in_ops(tmp_path):
    pkg = os.path.join(ROOT, 'long-video-gan_b200')
    ours = _run([pkg, REFERENCE], str(tmp_path / 'ours.pt'))
    # module resolution: ops from here, the rest of torch_utils and dnnlib from the reference
    assert ours['where']['bias_act'].startswith(pkg) and ours['where']['upfirdn2d'].startswith(pkg)
    assert ours['where']['misc'].startswith(REFERENCE) and ours['where']['dnnlib'].startswith(REFERENCE)
    gold = np.load(GOLDEN)
    # same networks, same seeds: low-res generator (32 frames 36x64), low-res discriminator, super-res generator (2 frames 144x256)
    for name in ('lres_G', 'lres_D', 'sres_G'):
        assert tuple(ours[name].shape) == tuple(gold[name + '_shape']), name
        flat, idx = _sample(ours[name])
        assert np.isfinite(flat).all(), name
        a, amax = gold[name + '_values'].astype(np.float64), float(gold[name + '_absmax'])
        err = float(np.abs(flat[idx] - a).max()) / max(amax, 1e-30)
        assert err <= 1e-5, f'{name}: {err:.3e}'
        assert abs(float(np.abs(flat).max()) - amax) <= 1e-5 * max(amax, 1e-30), f'{name}: max |output| differs'


if __name__ == '__main__':
    assert len(sys.argv) == 3 and sys.argv[1] == '--record', 'usage: test_dropin_reference.py --record <reference run .pt>'
    record(sys.argv[2])
