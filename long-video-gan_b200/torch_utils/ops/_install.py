"""Bookkeeping shared by the opt-in ``install`` functions of the fused ops: which classes of an unmodified reference model
a call reaches, and replacing a method of such a class by a wrapper.

Each wrapper runs its op inside the op's envelope and calls the method it replaced everywhere else. ``wrap`` keeps that
method as ``wrapper.__wrapped__`` (and as ``wrapper.lvg_<op>``), so the wrappers installed on one method form a chain
that ends at the model's own function. Installs walk this chain: one finds its own wrapper wherever another install put
its wrapper above or below it, so wrappers stack in any order and installing again changes nothing; and a wrapper that
reads the model module's globals takes them from the function at the bottom (``reference_function``).
"""
import inspect
import types

import torch


def find_classes(targets, name, accept=None, roots=None):
    """The classes named ``name`` that ``targets`` reach, each once, in first-seen order. A Python module gives its
    attribute ``name``. An ``nn.Module`` gives the class of every submodule of ``roots(t)`` (default ``[t]``) that is named
    ``name`` and satisfies ``accept``; this reaches the classes that ``persistence`` rebuilt from a pickle into a module
    of their own. Any other object gives its own class under the same two conditions."""
    found = []
    for t in targets:
        if isinstance(t, types.ModuleType):
            classes = [getattr(t, name)] if getattr(t, name, None) is not None else []
        else:
            objs = [m for r in (roots(t) if roots else [t]) for m in r.modules()] if isinstance(t, torch.nn.Module) else [t]
            classes = [type(m) for m in objs if type(m).__name__ == name and (accept is None or accept(m))]
        for cls in classes:
            if cls not in found:
                found.append(cls)
    return found


def find(fn, attr):
    """The wrapper carrying ``attr`` in the chain that starts at ``fn``, or None."""
    while fn is not None:
        if hasattr(fn, attr):
            return fn
        fn = getattr(fn, '__wrapped__', None)
    return None


def wrap(cls, method, attr, make):
    """Replace ``cls.<method>`` by ``make(current)``, unless a wrapper carrying ``attr`` is in the chain below it already.
    The new wrapper keeps ``current`` as ``wrapper.<attr>`` and ``wrapper.__wrapped__``. Returns the wrapper carrying
    ``attr``."""
    found = find(getattr(cls, method), attr)
    if found is not None:
        return found
    current = getattr(cls, method)
    wrapper = make(current)
    setattr(wrapper, attr, current)
    wrapper.__wrapped__ = current
    setattr(cls, method, wrapper)
    return wrapper


def reference_function(fn):
    """The function at the bottom of ``fn``'s chain of wrappers: the model's own method, whose ``__globals__`` are those
    of the model module."""
    return inspect.unwrap(fn)
