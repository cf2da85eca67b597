"""Oracle #2 loader (TEST INFRASTRUCTURE): the reference's own CUDA ops, side by side with this repository's.

`load()` imports the UNMODIFIED reference `torch_utils` package staged at oracle/_ref/src (see build_ref.py) under
the alias `lvgref_torch_utils`, so it can live in one process with this repository's `torch_utils`, and replaces its
JIT step (`custom_ops.get_plugin`, custom_ops.py:59-157) with a loader of the three plugins prebuilt for sm_90a in
oracle/_ref/*.so. Everything above the plugins -- `bias_act.py:126-207`, `upfirdn2d.py:217-273`,
`filtered_lrelu.py:159-272` (the autograd.Functions, sign-tensor plumbing, fallbacks) -- is the reference's code,
running its kernels. Only tests/, tools/microbench.py (--ref-cuda) and bench.py's reference legs may use this.
"""
import importlib
import importlib.machinery
import importlib.util
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(HERE, '_ref')
SRC = os.path.join(REF, 'src')
ALIAS = 'lvgref_torch_utils'
_plugins = {}


def available():
    return os.path.isdir(os.path.join(SRC, 'torch_utils', 'ops')) and \
        all(os.path.exists(os.path.join(REF, n + '.so')) for n in ('bias_act_plugin', 'upfirdn2d_plugin', 'filtered_lrelu_plugin'))


def load_plugin(name):
    """The prebuilt pybind11 module oracle/_ref/<name>.so (what cpp_extension.load would have produced)."""
    if name not in _plugins:
        import torch  # noqa: F401  (libtorch must be loaded before the extension)
        path = os.path.join(REF, name + '.so')
        loader = importlib.machinery.ExtensionFileLoader(name, path)
        spec = importlib.util.spec_from_loader(name, loader)
        mod = importlib.util.module_from_spec(spec)
        loader.exec_module(mod)
        _plugins[name] = mod
    return _plugins[name]


def _get_plugin(module_name, sources=None, headers=None, source_dir=None, **build_kwargs):
    return load_plugin(module_name)


def patch_custom_ops(custom_ops_module):
    custom_ops_module.get_plugin = _get_plugin
    custom_ops_module.verbosity = 'none'


def load():
    """-> namespace with bias_act, upfirdn2d, filtered_lrelu, conv2d_resample, conv2d_gradfix (reference modules)."""
    if not available():
        raise RuntimeError('oracle/_ref is not built (python oracle/build_ref.py where a reference checkout is present)')
    if ALIAS not in sys.modules:
        sys.modules.setdefault('imageio', types.ModuleType('imageio'))
        if SRC not in sys.path:
            sys.path.append(SRC)          # dnnlib (absolute import of the reference's misc.py); appended: never shadows ours
        pkg_dir = os.path.join(SRC, 'torch_utils')
        spec = importlib.util.spec_from_file_location(ALIAS, os.path.join(pkg_dir, '__init__.py'),
                                                      submodule_search_locations=[pkg_dir])
        pkg = importlib.util.module_from_spec(spec)
        sys.modules[ALIAS] = pkg
        spec.loader.exec_module(pkg)
        patch_custom_ops(importlib.import_module(ALIAS + '.custom_ops'))
    ns = types.SimpleNamespace()
    for name in ('bias_act', 'upfirdn2d', 'filtered_lrelu', 'conv2d_resample', 'conv2d_gradfix', 'fma'):
        setattr(ns, name, importlib.import_module(f'{ALIAS}.ops.{name}'))
    return ns
