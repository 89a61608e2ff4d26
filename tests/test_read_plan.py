"""How a read through the device index is launched, checked on the CPU: which kernels run for a
batch (csrc/ctrl/read_plan.h) and how a call's keys are split into launches that fit the
pinned staging ring (csrc/ctrl/staging.h)."""
import random

import pytest

from infinistore_b200 import _infinistore as m

T = m.testing
AUTO, LDST, TMA, LDST256 = 0, 1, 2, 3
SMS = 132
KB, MB = 1 << 10, 1 << 20
FP8_PAGE = 8192 + 4 * 8192 // 128  # bytes of an fp8 page of 8192 elements: e4m3 + scales

# (case, plan_device_read arguments, expected (path, variant, grid_cap));
# variant None: the path runs no launch that takes one
CASES = [
    ("small batch, local", dict(n=16, block_bytes=64 * KB, all_local=True),
     ("fused_copy", LDST256, 0)),
    ("small batch over NVLink", dict(n=16, block_bytes=64 * KB, all_remote=True),
     ("fused_copy", LDST256, 2 * SMS)),
    # an ldst connection reads fused copies with the 16-byte ld/st kernel
    ("small batch, ldst", dict(n=4, block_bytes=64 * KB, copy_variant=LDST, all_local=True),
     ("fused_copy", LDST, 0)),
    ("whole blocks, auto, local", dict(n=2048, block_bytes=128 * KB, all_local=True),
     ("fused_copy", LDST256, 0)),
    ("whole blocks, auto, over NVLink", dict(n=2048, block_bytes=128 * KB, all_remote=True),
     ("fused_copy", AUTO, 2 * SMS)),
    ("whole blocks, auto, mixed pool", dict(n=2048, block_bytes=128 * KB),
     ("fused_copy", AUTO, 0)),
    ("whole blocks, tma, local", dict(n=2048, block_bytes=128 * KB, copy_variant=TMA,
                                      all_local=True),
     ("fused_copy", TMA, 0)),
    ("whole blocks, tma, over NVLink", dict(n=2048, block_bytes=128 * KB, copy_variant=TMA,
                                            all_remote=True),
     ("fused_copy", TMA, 2 * SMS)),
    ("whole blocks, ldst, local", dict(n=2048, block_bytes=128 * KB, copy_variant=LDST,
                                       all_local=True),
     ("fused_copy", LDST, 0)),
    ("whole blocks, max_ctas", dict(n=2048, block_bytes=128 * KB, all_remote=True, max_ctas=8),
     ("fused_copy", AUTO, 8)),
    ("large blocks, local", dict(n=8, block_bytes=2 * MB, all_local=True),
     ("lookup_copy", LDST256, 0)),
    ("large blocks, ldst", dict(n=8, block_bytes=2 * MB, copy_variant=LDST, all_local=True),
     ("lookup_copy", LDST, 0)),
    ("few blocks above 4 MB, over NVLink", dict(n=16, block_bytes=512 * KB, all_remote=True),
     ("lookup_copy", AUTO, 2 * SMS)),
    ("large blocks, tma, max_ctas", dict(n=8, block_bytes=2 * MB, copy_variant=TMA,
                                         all_local=True, max_ctas=20),
     ("lookup_copy", TMA, 20)),
    ("fp8 fused, local", dict(n=512, block_bytes=FP8_PAGE, fp8_elems=8192, fp8_fused_ok=True,
                              all_local=True),
     ("fused_fp8", LDST256, 0)),
    ("fp8 fused, small batch", dict(n=4, block_bytes=FP8_PAGE, fp8_elems=8192,
                                    fp8_fused_ok=True, all_remote=True),
     ("fused_fp8", LDST256, SMS)),
    ("fp8 fused over NVLink", dict(n=512, block_bytes=FP8_PAGE, fp8_elems=8192,
                                   fp8_fused_ok=True, all_remote=True),
     ("fused_fp8", AUTO, SMS)),
    ("fp8 unfused, local", dict(n=512, block_bytes=FP8_PAGE, fp8_elems=8192, all_local=True),
     ("lookup_fp8", 1, 0)),
    ("fp8 unfused over NVLink", dict(n=512, block_bytes=FP8_PAGE, fp8_elems=8192,
                                     all_remote=True),
     ("lookup_fp8", 0, SMS)),
    # not move_blocks' rule (all_local ? 1 : 0): a mixed pool reads with the ld/st kernels
    ("fp8 unfused, mixed pool", dict(n=512, block_bytes=FP8_PAGE, fp8_elems=8192),
     ("lookup_fp8", 1, 0)),
    ("fp8 unfused, small batch", dict(n=4, block_bytes=FP8_PAGE, fp8_elems=8192,
                                      all_local=True),
     ("lookup_fp8", 1, 0)),
    ("gathered, fused, local", dict(n=2048, block_bytes=64 * 32 * KB, gather=True,
                                    scatter_fused_ok=True, all_local=True),
     ("fused_scatter", LDST256, 0)),
    ("gathered, fused, small batch, ldst", dict(n=132, block_bytes=8 * KB, gather=True,
                                                scatter_fused_ok=True, copy_variant=LDST),
     ("fused_scatter", LDST256, 0)),
    ("gathered, fused, over NVLink", dict(n=2048, block_bytes=64 * 32 * KB, gather=True,
                                          scatter_fused_ok=True, all_remote=True),
     ("fused_scatter", AUTO, 2 * SMS)),
    ("gathered, unfused", dict(n=16, block_bytes=64 * 32 * KB, gather=True, all_local=True),
     ("lookup_gather", None, 0)),
    ("gathered, unfused over NVLink", dict(n=16, block_bytes=MB, gather=True, all_remote=True),
     ("lookup_gather", None, 2 * SMS)),
    # a gathered read never takes the fp8 or plain copy paths
    ("gathered, small batch, unfused", dict(n=4, block_bytes=8 * KB, gather=True,
                                            fp8_fused_ok=True),
     ("lookup_gather", None, 0)),
]


@pytest.mark.parametrize("case,kw,want", CASES, ids=[c[0] for c in CASES])
def test_device_read_plans(case, kw, want):
    p = T.plan_device_read(sm_count=SMS, **kw)
    path, variant, grid_cap = want
    assert p["path"] == path
    if variant is not None:
        assert p["variant"] == variant
    assert p["grid_cap"] == grid_cap


def test_every_path_is_covered():
    paths = {c[2][0] for c in CASES}
    assert paths == {"fused_copy", "fused_fp8", "fused_scatter", "lookup_copy", "lookup_fp8",
                     "lookup_gather"}


def _staged(lens):
    return sum((max(n, 1) + 7) // 8 * 8 + 16 for n in lens)


def _check_batches(lens, max_blocks=None):
    cap = T.MAX_BATCH if max_blocks is None else max_blocks
    batches = T.key_batches(lens) if max_blocks is None else T.key_batches(lens, max_blocks)
    bound = T.RING_BYTES // 2
    at = 0
    for n, key_bytes in batches:
        part = lens[at:at + n]
        assert 1 <= n <= cap
        assert key_bytes == sum((max(k, 1) + 7) // 8 * 8 for k in part)
        assert _staged(part) <= bound or n == 1
        at += n
        # each batch is as large as the bounds allow
        if at < len(lens) and n < cap:
            assert _staged(lens[at - n:at + 1]) > bound
    assert at == len(lens)
    return batches


def test_short_keys_fit_one_launch():
    assert _check_batches([8] * 65536) == [(65536, 8 * 65536)]


def test_long_keys_are_split_to_fit_half_the_ring():
    # 300-byte keys stage 304 + 16 bytes each: 26214 of them fit in 8 MB
    assert [n for n, _ in _check_batches([300] * 65536)] == [26214, 26214, 13108]


def test_mixed_keys():
    rng = random.Random(3)
    lens = [rng.choice([0, 8, 40, 300, 1000, 4000]) for _ in range(65536)]
    assert len(_check_batches(lens)) > 1


def test_block_caps_are_kept():
    assert T.gather_max_blocks(256, 64 * KB) == T.MAX_BATCH
    cap = T.gather_max_blocks(256, 16 * MB)  # 2^30 work items of 16 KB chunks
    assert cap == 4096
    assert [n for n, _ in _check_batches([8] * 10000, cap)] == [4096, 4096, 1808]
    assert [n for n, _ in _check_batches([300] * 70000)][0] == 26214
    assert [n for n, _ in _check_batches([8] * 70000)] == [65536, 70000 - 65536]
    assert T.gather_max_blocks(1 << 20, 1 << 31) == 1  # never zero


def test_a_key_above_the_bound_gets_a_launch_of_its_own():
    big = 9 << 20
    assert T.key_batches([big, 8, 8]) == [(1, big), (2, 16)]
    assert T.key_batches([8, big, 8]) == [(1, 8), (1, big), (1, 8)]


def test_bad_arguments_are_refused():
    with pytest.raises(ValueError):
        T.key_batches([8, 8], 0)
    with pytest.raises(ValueError):
        T.gather_max_blocks(0, 4096)
    with pytest.raises(ValueError):
        T.gather_max_blocks(4, 0)
