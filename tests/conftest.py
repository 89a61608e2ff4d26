import os
import socket
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100)")
    config.addinivalue_line("markers", "benchmark: runs the throughput benchmark")


def _ensure_built():
    from tools import build_native

    if not build_native.module_path().exists():
        build_native.build()


_ensure_built()


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


@pytest.fixture()
def host_server():
    """In-process server with a small host-memory (shm) pool on an ephemeral port."""
    from infinistore_b200 import _infinistore as m

    cfg = m.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "host"
    cfg.prealloc_bytes = 64 << 20
    cfg.minimal_allocate_size = 16
    srv = m.Server(cfg)
    port = srv.start()
    yield srv, port
    srv.stop()


@pytest.fixture()
def hbm_server():
    """In-process server with an HBM pool on cuda:0 (GPU tests)."""
    from infinistore_b200 import _infinistore as m

    cfg = m.ServerConfig()
    cfg.service_port = 0
    cfg.host = "127.0.0.1"
    cfg.pool_backend = "hbm"
    cfg.pool_devices = [0]
    cfg.prealloc_bytes = 1 << 30
    cfg.minimal_allocate_size = 16
    srv = m.Server(cfg)
    port = srv.start()
    yield srv, port
    srv.stop()


def make_conn(port, connection_type="RDMA", **kw):
    import infinistore_b200 as ist

    cfg = ist.ClientConfig(host_addr="127.0.0.1", service_port=port,
                           connection_type=connection_type, log_level="warning", **kw)
    conn = ist.InfinityConnection(cfg)
    conn.connect()
    return conn
