"""`copy_variant="auto"` with the pool in the same GPU's HBM: pages of 64 KB and more move
through the ld/st kernels (kv_copy_ldst, kv_read_fused); an explicit "tma" still takes the TMA
pipeline.  Kernel names come from torch.profiler."""
import pytest
import torch

from conftest import make_conn

pytestmark = pytest.mark.gpu


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize("variant, write_kernel, read_kernel", [
    ("auto", "kv_copy_ldst_kernel", "kv_read_fused_kernel"),
    ("tma", "kv_pipe_copy_kernel", "kv_pipe_read_kernel"),
])
def test_local_pool_variant(hbm_server, variant, write_kernel, read_kernel):
    _, port = hbm_server
    conn = make_conn(port, device_lookup=True, copy_variant=variant)
    n, elems = 256, 64 * 1024  # 128 KB bf16 pages, as the flagship
    src = torch.randn(n * elems, device="cuda:0").to(torch.bfloat16)
    dst = torch.zeros_like(src)
    conn.register_mr(src)
    conn.register_mr(dst)
    keys = [f"local-{variant}-{i}" for i in range(n)]
    blocks = conn.allocate_rdma(keys, elems * 2)

    def write():
        conn.rdma_write_cache(src, [i * elems for i in range(n)], elems, blocks)
        conn.sync()

    def read():
        conn.read_cache(dst, [(k, i * elems) for i, k in enumerate(keys)], elems)
        conn.sync()

    wrote = _kernels(write)
    got = _kernels(read)
    assert torch.equal(src, dst)
    assert any(write_kernel in k for k in wrote), wrote
    assert any(read_kernel in k for k in got), got
    conn.close()
