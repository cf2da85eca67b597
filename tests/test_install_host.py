"""torch_utils/ops/_install.py, the bookkeeping of every fused op's ``install``, on stub classes (no reference model): which
classes a target reaches, idempotence, wrappers of two ops stacked on one method in either order, and the model module's
globals seen through the chain."""
import types

import torch

from torch_utils.ops import _install


def _layer_class(name='Layer'):
    """A fresh class of the given name each call, as ``persistence`` rebuilds one from a pickle."""
    return type(name, (torch.nn.Module,), {'forward': lambda self, x: ('ref', x)})


class Root(torch.nn.Module):
    def __init__(self, *layers):
        super().__init__()
        self.layers = torch.nn.ModuleList(layers)


def test_module_targets_give_their_attribute():
    Layer = _layer_class()
    mod = types.ModuleType('model_stub')
    mod.Layer = Layer
    assert _install.find_classes([mod], 'Layer') == [Layer]
    assert _install.find_classes([mod], 'Block') == []
    assert _install.find_classes([mod, mod], 'Layer') == [Layer]


def test_module_instances_give_the_classes_of_their_submodules_by_name():
    A, B = _layer_class(), _layer_class()                      # same name, different identity
    net = torch.nn.Sequential(A(), torch.nn.Linear(1, 1), B(), A())
    assert A is not B and _install.find_classes([net], 'Layer') == [A, B]
    assert _install.find_classes([B()], 'Layer') == [B]
    assert _install.find_classes([torch.nn.Linear(1, 1)], 'Layer') == []


def test_other_objects_give_their_own_class():
    GAN = type('GAN', (), {})
    Other = type('Other', (), {'GAN': GAN})
    assert _install.find_classes([GAN()], 'GAN') == [GAN]
    assert _install.find_classes([Other()], 'GAN') == []        # an attribute of a non-module object is not followed
    assert _install.find_classes([GAN()], 'GAN', accept=lambda m: hasattr(m, 'D')) == []


def test_first_seen_order_across_targets():
    A, B, C = _layer_class(), _layer_class(), _layer_class()
    mod = types.ModuleType('model_stub')
    mod.Layer = C
    assert _install.find_classes([torch.nn.Sequential(B(), A()), mod, A(), torch.nn.Sequential(C(), B())], 'Layer') == [B, A, C]


def test_accept_and_roots():
    A, B = _layer_class(), _layer_class()
    a, b = A(), B()
    a.f = 1
    net = torch.nn.Sequential(b, a)
    assert _install.find_classes([net], 'Layer', accept=lambda m: hasattr(m, 'f')) == [A]
    # roots: only what lies below a Root, or the whole target when it holds none
    roots = lambda t: [m for m in t.modules() if type(m).__name__ == 'Root'] or [t]      # noqa: E731
    assert _install.find_classes([torch.nn.Sequential(B(), Root(A()))], 'Layer', roots=roots) == [A]
    assert _install.find_classes([torch.nn.Sequential(B(), A())], 'Layer', roots=roots) == [B, A]


def _make(tag):
    """A wrapper factory: the op takes inputs equal to ``tag`` and passes everything else to the method it replaced."""
    def make(orig):
        def forward(self, x):
            return (tag, x) if x == tag else orig(self, x)
        return forward
    return make


def test_wrap_is_idempotent_and_keeps_the_original():
    Layer = _layer_class()
    orig = Layer.forward
    w = _install.wrap(Layer, 'forward', 'lvg_a', _make('a'))
    assert Layer.forward is w and w.lvg_a is orig and w.__wrapped__ is orig
    assert _install.wrap(Layer, 'forward', 'lvg_a', _make('a')) is w and Layer.forward is w
    assert Layer()('a') == ('a', 'a') and Layer()('c') == ('ref', 'c')


def test_two_wrappers_stack_in_either_order_without_double_wrapping():
    for first, second in (('a', 'b'), ('b', 'a')):
        Layer = _layer_class()
        orig = Layer.forward
        inner = _install.wrap(Layer, 'forward', 'lvg_' + first, _make(first))
        outer = _install.wrap(Layer, 'forward', 'lvg_' + second, _make(second))
        for _ in range(2):
            for tag in (first, second, first):
                got = _install.wrap(Layer, 'forward', 'lvg_' + tag, _make(tag))
                assert got is (inner if tag == first else outer)
        assert Layer.forward is outer and outer.__wrapped__ is inner and inner.__wrapped__ is orig
        assert getattr(outer, 'lvg_' + second) is inner and getattr(inner, 'lvg_' + first) is orig
        assert [Layer()(x) for x in 'abc'] == [('a', 'a'), ('b', 'b'), ('ref', 'c')]
        assert _install.reference_function(Layer.forward) is orig
        assert _install.reference_function(orig) is orig


_MODEL_SRC = '''
misc = "the model module's misc"

class Layer:
    def forward(self, x):
        return x
'''


def test_globals_read_through_the_chain_are_the_model_modules():
    for other_first in (False, True):
        model = types.ModuleType('model_stub')
        exec(_MODEL_SRC, model.__dict__)

        def reads_globals(orig):
            g = _install.reference_function(orig).__globals__

            def forward(self, x):
                return g['misc']
            return forward
        if other_first:
            _install.wrap(model.Layer, 'forward', 'lvg_other', _make('b'))
            assert 'misc' not in model.Layer.forward.__globals__          # the other wrapper's globals are this file's
        _install.wrap(model.Layer, 'forward', 'lvg_reader', reads_globals)
        _install.wrap(model.Layer, 'forward', 'lvg_other', _make('b'))
        assert model.Layer().forward('c') == "the model module's misc"
