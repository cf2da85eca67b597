"""Oracle #2 recipe (TEST INFRASTRUCTURE, never imported by the product): builds the reference's OWN three CUDA
plugins for sm_90a from the sources where they lie under /root/reference and stages the reference's Python
modules next to them, all under oracle/_ref/ (git-ignored; it goes wherever the built tree goes, like our own .so).

  oracle/_ref/bias_act_plugin.so         <- torch_utils/ops/bias_act.{cpp,cu}          (custom_ops.py:59-157, bias_act.py:38-49)
  oracle/_ref/upfirdn2d_plugin.so        <- torch_utils/ops/upfirdn2d.{cpp,cu}         (upfirdn2d.py:23-33)
  oracle/_ref/filtered_lrelu_plugin.so   <- torch_utils/ops/filtered_lrelu*.{cpp,cu}   (filtered_lrelu.py:23-34)
  oracle/_ref/src/{torch_utils,model,dnnlib}   staged copy of the checkout's Python (build artefact, not repo source)

Same compiler flags as the reference passes to torch.utils.cpp_extension (`--use_fast_math
--allow-unsupported-compiler`) plus torch's own extension defaults; the only difference is that the build is
ahead-of-time (no GPU here) and targets sm_90a explicitly. Nothing is copied into tracked files.

Usage: python oracle/build_ref.py [--reference /root/reference] [--force]
"""
import argparse
import concurrent.futures as cf
import os
import shutil
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, '_ref')

PLUGINS = {
    'bias_act_plugin': ['bias_act.cpp', 'bias_act.cu'],
    'upfirdn2d_plugin': ['upfirdn2d.cpp', 'upfirdn2d.cu'],
    'filtered_lrelu_plugin': ['filtered_lrelu.cpp', 'filtered_lrelu_wr.cu', 'filtered_lrelu_rd.cu', 'filtered_lrelu_ns.cu'],
}
STAGED = ['torch_utils', 'model', 'dnnlib']


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError('command failed: ' + ' '.join(cmd) + '\n' + r.stdout[-4000:])


def _newest(paths):
    return max(os.path.getmtime(p) for p in paths)


def build(reference='/root/reference', force=False, verbose=True):
    """Returns True when oracle/_ref is complete, False when there is no checkout to build from."""
    ops = os.path.join(reference, 'torch_utils', 'ops')
    if not os.path.isdir(ops):
        return all(os.path.exists(os.path.join(OUT, n + '.so')) for n in PLUGINS)
    import torch
    from torch.utils import cpp_extension as ce

    os.makedirs(os.path.join(OUT, 'obj'), exist_ok=True)
    inc = [f'-I{p}' for p in ce.include_paths('cuda')] + [f'-I{sysconfig.get_paths()["include"]}']
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI)
    jobs, links = [], []
    for name, srcs in PLUGINS.items():
        so = os.path.join(OUT, name + '.so')
        paths = [os.path.join(ops, s) for s in srcs]
        deps = [os.path.join(ops, f) for f in os.listdir(ops) if f.endswith(('.h', '.cu', '.cpp'))]
        if not force and os.path.exists(so) and os.path.getmtime(so) >= _newest(deps):
            continue
        common = [f'-DTORCH_EXTENSION_NAME={name}', '-DTORCH_API_INCLUDE_EXTENSION_H', f'-D_GLIBCXX_USE_CXX11_ABI={abi}'] + inc
        objs = []
        for p in paths:
            o = os.path.join(OUT, 'obj', name + '__' + os.path.basename(p) + '.o')
            objs.append(o)
            if p.endswith('.cu'):
                jobs.append(['nvcc', '-c', p, '-o', o, '-std=c++17', '-O3', '-gencode', 'arch=compute_90a,code=sm_90a',
                             '--use_fast_math', '--allow-unsupported-compiler', '--expt-relaxed-constexpr',
                             '-D__CUDA_NO_HALF_OPERATORS__', '-D__CUDA_NO_HALF_CONVERSIONS__',
                             '-D__CUDA_NO_BFLOAT16_CONVERSIONS__', '-D__CUDA_NO_HALF2_OPERATORS__',
                             '--compiler-options', '-fPIC'] + common)
            else:
                jobs.append(['g++', '-c', p, '-o', o, '-std=c++17', '-O3', '-fPIC'] + common)
        lib = [f'-L{p}' for p in ce.library_paths('cuda')]
        links.append(['g++', '-shared', '-o', so] + objs + lib +
                     ['-lc10', '-lc10_cuda', '-ltorch_cpu', '-ltorch_cuda', '-ltorch', '-ltorch_python', '-lcudart'])
    if jobs and verbose:
        print(f'oracle/_ref: compiling {len(jobs)} reference translation units for sm_90a ...', flush=True)
    with cf.ThreadPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1))) as ex:
        list(ex.map(_run, jobs))
    for cmd in links:
        _run(cmd)

    # staged Python (so the UNMODIFIED reference networks and op wrappers can run on a GPU machine)
    src = os.path.join(OUT, 'src')
    for d in STAGED:
        dst = os.path.join(src, d)
        if os.path.isdir(dst):
            shutil.rmtree(dst)
        shutil.copytree(os.path.join(reference, d), dst,
                        ignore=shutil.ignore_patterns('__pycache__', '*.cu', '*.cpp', '*.h', '*.pyc'))
    if verbose:
        print('oracle/_ref: ready (' + ', '.join(sorted(os.listdir(OUT))) + ')')
    return True


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--reference', default='/root/reference')
    ap.add_argument('--force', action='store_true')
    a = ap.parse_args()
    ok = build(a.reference, a.force)
    sys.exit(0 if ok else 1)
