"""Drop-in ``torch_utils`` package holding the H100-native ``torch_utils.ops``.

Only the operator path (``torch_utils.ops`` and the plugin loader
``torch_utils.custom_ops``) lives here. When this directory is placed on
``sys.path`` *ahead of* a LongVideoGAN checkout, the remaining reference
sub-modules (``misc``, ``persistence``, ``training_stats``, ``distributed``)
still resolve to the checkout: the package path is extended over every
``torch_utils`` directory found on ``sys.path`` (ours first).
"""
import pkgutil

__path__ = pkgutil.extend_path(__path__, __name__)
