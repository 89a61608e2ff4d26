"""Drop-in alias: ``import infinistore`` resolves to the H100-native package, so code
written against the reference (``infinistore.ClientConfig``, ``python -m
infinistore.server`` ...) runs unchanged."""
import sys as _sys

import infinistore_b200 as _impl
from infinistore_b200 import *  # noqa: F401,F403
from infinistore_b200 import __all__, __version__  # noqa: F401
from infinistore_b200 import lib, _infinistore  # noqa: F401

_sys.modules.setdefault(__name__ + ".lib", lib)
_sys.modules.setdefault(__name__ + "._infinistore", _infinistore)
