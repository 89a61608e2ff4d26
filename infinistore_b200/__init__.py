"""infinistore_b200 — an H100-native KV-cache block store with infiniStore's API.

The package exports the reference's public names (its ``infinistore/__init__.py``) plus the
additions of this implementation; everything lives in ``lib.py``.
"""
from . import lib as _lib

try:  # the installed distribution knows its version (setup.py: git describe)
    from importlib.metadata import PackageNotFoundError as _NotInstalled, version as _version

    __version__ = _version("infinistore-b200")
except _NotInstalled:  # run from the source tree
    __version__ = "0.2.0.dev0"

# what a program written against the reference imports from the package
_REFERENCE_SURFACE = (
    "ClientConfig", "ServerConfig", "InfinityConnection", "DisableTorchCaching", "Logger",
    "TYPE_RDMA", "TYPE_LOCAL_GPU", "LINK_ETHERNET", "LINK_IB",
    "register_server", "purge_kv_map", "get_kvmap_len", "check_supported",
)
# added here: in-process server control, statistics, checkpoint / resume, row-sliced reads
_ADDITIONS = ("stop_server", "server_stats", "dump_kv_map", "load_kv_map", "PartRows")

__all__ = [*_REFERENCE_SURFACE, *_ADDITIONS]
globals().update({_name: getattr(_lib, _name) for _name in __all__})
