"""The raw launchers refuse bad index shards, segment lists and fused-read geometries with
ValueError before anything is launched, without a GPU.  No pointer passed here is valid: a call
that got past its checks would fail at the launch with another error, never a ValueError."""
import pytest

from infinistore_b200 import _infinistore as m

K = m.kernels
P = 1 << 12  # a stand-in address, never dereferenced
GOOD_SHARD = (P, 127)  # 1024 slots


def _read(**kw):
    args = dict(key_bytes=P, key_off=P, key_len=P, n=200, table=P, table_mask=127,
                seg_base=[P], dst_base=P, dst_off=P, bytes=4096, status=P)
    args.update(kw)
    return K.read_fused(**args)


BAD_SHARDS = [
    ([GOOD_SHARD] * 8, "at most 8"),  # nine tables in all
    ([(P, 5)], "bucket mask"),        # 48 slots: not a power of two
    ([(P, 1 << 26)], "bucket mask"),  # 2^29 + 8 slots: slot ids would reach the shard bits
    ([(P, (1 << 26) - 1), (0, 127)], "null index table"),
]


@pytest.mark.parametrize("shards,reason", BAD_SHARDS)
def test_every_launcher_refuses_bad_shards(shards, reason):
    calls = [
        lambda: _read(shards=shards),
        lambda: K.index_lookup(P, P, P, 1, P, 127, [P], shards=shards),
        lambda: K.index_validate(P, 1, P, P, shards=shards),
        lambda: K.kv_copy(P, 1, 4096, recs=P, table=P, table_mask=127, done=P, shards=shards),
        lambda: K.kv_gather(P, 1, [P], 4096, recs=P, table=P, table_mask=127, done=P,
                            shards=shards),
    ]
    for call in calls:
        with pytest.raises(ValueError, match=reason):
            call()


def test_segment_lists_past_the_limit():
    with pytest.raises(ValueError, match="at most 16 segment bases"):
        _read(seg_base=[P] * 17)
    with pytest.raises(ValueError, match="at most 16 segment bases"):
        K.index_lookup(P, P, P, 1, P, 127, [P] * 17)


@pytest.mark.parametrize("kw,reason", [
    (dict(elems=500), "multiple of 512"),
    (dict(elems=1024, align_or=8), "16-byte aligned"),
    (dict(elems=1024, part_base=[P], part_bytes=1024), "not both"),
    (dict(validate=True, status=0), "status"),
])
def test_fp8_and_validate_refusals(kw, reason):
    with pytest.raises(ValueError, match=reason):
        _read(**kw)


@pytest.mark.parametrize("kw", [
    dict(part_base=[P] * 257, part_bytes=1024),        # more than GATHER_MAX_PARTS parts
    dict(part_base=[P] * 3, part_bytes=0),             # empty parts
    dict(part_base=[P] * 3, part_bytes=1000),          # not a multiple of 16 bytes
    dict(part_base=[P + 8] * 3, part_bytes=1024),      # a part base off 16 bytes
    dict(part_base=[P] * 3, part_bytes=1024, align_or=4),
    dict(part_base=[P] * 3, part_bytes=1 << 30, first_part=2),  # a block past 2^32 bytes
    dict(part_base=[P] * 3, part_bytes=1024, n=3),     # fewer blocks than the default grid
    dict(part_base=[P] * 3, part_bytes=1024, n=7, max_ctas=8),
])
def test_scatter_geometry_refusals(kw):
    with pytest.raises(ValueError, match="gathered parts"):
        _read(**kw)
