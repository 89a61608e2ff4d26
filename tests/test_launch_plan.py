"""Which kernel a page-mover launcher runs, how it cuts the batch into work items and on how many
CTAs (csrc/kernels/launch_plan.h), checked on the CPU.  Every expected value is the one the
launchers computed before the rules moved into the plan; each case names the launcher line
(kernels/<file>:<line> of that version) it pins."""
import pytest

from infinistore_b200 import _infinistore as m

from test_read_plan import CASES as READ_CASES

T = m.testing
AUTO, LDST, TMA, LDST256 = 0, 1, 2, 3
SMS = 132
R16, R32 = 4, 3  # resident CTAs per SM of the 16- / 32-byte ld/st flavours (arbitrary, distinct)
KB, MB = 1 << 10, 1 << 20
RES = dict(sm_count=SMS, resident16=R16, resident32=R32)


def _check(plan, want):
    if want is None:
        assert not plan["valid"]
        return
    kernel, param, chunk, cpb, ctas, geo = want
    assert plan["valid"]
    assert plan["kernel"] == kernel
    assert plan["param"] == param
    assert (plan["chunk"], plan["cpb"], plan["ctas"]) == (chunk, cpb, ctas)
    if geo is not None:
        assert (plan["stage_bytes"], plan["stages"], plan["smem"]) == geo
    return plan["kernel"], plan["param"]


G16 = (16 * KB, 4, 64 * KB)  # default ring: 16 KB slots, four of them

# (case, plan_copy arguments, (kernel, param, chunk, cpb, ctas, ring geometry) or None = refused)
COPY = [
    ("auto, 128 KB pages: TMA, whole blocks (kv_copy.cu:175, kv_pipe.cu:691)",
     dict(n=512, bytes=128 * KB), ("tma", False, 128 * KB, 1, SMS, G16)),
    ("auto, host descriptors, n <= 256: TMA with parameter descriptors (kv_pipe.cu:704)",
     dict(n=16, bytes=128 * KB, descs_host=True), ("tma", True, 64 * KB, 2, 32, G16)),
    ("tma: max_ctas clamped to the SM count (kv_pipe.cu:690)",
     dict(n=512, bytes=128 * KB, variant=TMA, max_ctas=500), ("tma", False, 128 * KB, 1, SMS, G16)),
    ("tma: max_ctas below the SM count (kv_pipe.cu:690)",
     dict(n=512, bytes=128 * KB, variant=TMA, max_ctas=64), ("tma", False, 128 * KB, 1, 64, G16)),
    ("tma: small blocks stay on TMA when asked, slots shrink to the block (kv_pipe.cu:669)",
     dict(n=10, bytes=4 * KB, variant=TMA), ("tma", False, 4 * KB, 1, 10, (4 * KB, 16, 64 * KB))),
    ("tma: caller's ring geometry (kv_pipe.cu:667-668)",
     dict(n=SMS, bytes=256 * KB, variant=TMA, stage_bytes=32 * KB, ring_bytes=128 * KB),
     ("tma", False, 256 * KB, 1, SMS, (32 * KB, 4, 128 * KB))),
    ("tma: at least kStoreLag + 1 slots (kv_pipe.cu:670)",
     dict(n=1, bytes=64 * KB, variant=TMA, ring_bytes=16 * KB),
     ("tma", False, 64 * KB, 1, 1, (16 * KB, 3, 48 * KB))),
    ("auto below 64 KB, 32-byte aligned: ldst256 (kv_copy.cu:176, :181, :216)",
     dict(n=16, bytes=32 * KB, descs_host=True), ("ldst32", True, 32 * KB, 1, 16, None)),
    ("auto below 64 KB, 16-byte aligned only: ldst, whole blocks (kv_copy.cu:176, :192, :222)",
     dict(n=1000, bytes=48), ("ldst16", False, 48, 1, R16 * SMS, None)),
    ("unaligned: byte kernel, no parameter descriptors (kv_copy.cu:181, :213)",
     dict(n=8, bytes=4 * KB, align_or=2, descs_host=True), ("ldst1", False, 4 * KB, 1, 8, None)),
    ("unaligned tma request falls to ldst, then the byte kernel (kv_copy.cu:177, :213)",
     dict(n=4, bytes=128 * KB + 8, variant=TMA), ("ldst1", False, 32 * KB, 5, 20, None)),
    ("unaligned ldst256 request falls to ldst, then the byte kernel (kv_copy.cu:177, :213)",
     dict(n=2, bytes=64 * KB, align_or=4, variant=LDST256), ("ldst1", False, 32 * KB, 2, 4, None)),
    ("ldst256 without 32-byte alignment falls to ldst (kv_copy.cu:178, :222)",
     dict(n=2, bytes=64 * KB, align_or=16, variant=LDST256), ("ldst16", False, 32 * KB, 2, 4, None)),
    ("ldst256: max_ctas is not clamped to the resident grid (kv_copy.cu:207)",
     dict(n=2000, bytes=64 * KB, variant=LDST256, max_ctas=1000),
     ("ldst32", False, 64 * KB, 1, 1000, None)),
    ("ldst256: the resident grid of the 32-byte flavour (kv_copy.cu:206)",
     dict(n=2000, bytes=64 * KB, variant=LDST256), ("ldst32", False, 64 * KB, 1, R32 * SMS, None)),
    ("blocks above 1 MB are cut into 32 KB chunks even when n >= SMs (kv_copy.cu:191-192)",
     dict(n=200, bytes=2 * MB, variant=LDST), ("ldst16", False, 32 * KB, 64, R16 * SMS, None)),
    ("ldst, host descriptors, 16-byte aligned (kv_copy.cu:181, :220)",
     dict(n=256, bytes=4 * KB, variant=LDST, descs_host=True), ("ldst16", True, 4 * KB, 1, 256, None)),
    ("ldst, more than 256 blocks: descriptors stay in memory (kv_copy.cu:181)",
     dict(n=257, bytes=4 * KB, variant=LDST, descs_host=True),
     ("ldst16", False, 4 * KB, 1, 257, None)),
    ("multicast forces the 16-byte MC kernel, whatever the variant (kv_copy.cu:170, :210)",
     dict(n=4, bytes=128 * KB, variant=TMA, multicast=True, descs_host=True),
     ("ldst16_mc", True, 32 * KB, 4, 16, None)),
    ("multicast, descriptors in memory (kv_copy.cu:212)",
     dict(n=300, bytes=4 * KB, multicast=True), ("ldst16_mc", False, 4 * KB, 1, 300, None)),
    ("unaligned multicast is refused (kv_copy.cu:169)",
     dict(n=4, bytes=4 * KB, align_or=8, multicast=True), None),
]


@pytest.mark.parametrize("case,kw,want", COPY, ids=[c[0] for c in COPY])
def test_plan_copy(case, kw, want):
    _check(T.plan_copy(**kw, **RES), want)


# (case, plan_gather arguments, expected as for COPY)
GATHER = [
    ("64 KB parts: TMA whatever the pool or connection - gathers take no variant (kv_copy.cu:233)",
     dict(n=100, nparts=4, part_bytes=64 * KB), ("tma", False, 64 * KB, 1, SMS, G16)),
    ("TMA: max_ctas clamped to the SM count (kv_pipe.cu:728)",
     dict(n=100, nparts=4, part_bytes=64 * KB, max_ctas=200), ("tma", False, 64 * KB, 1, SMS, G16)),
    ("TMA: large parts of few blocks are split over the grid (kv_pipe.cu:732-736)",
     dict(n=2, nparts=2, part_bytes=MB), ("tma", False, 64 * KB, 16, 64, G16)),
    ("TMA: more than 2^31 - 1 parts are refused (kv_pipe.cu:731)",
     dict(n=1 << 24, nparts=256, part_bytes=64 * KB), None),
    ("TMA: more than 2^31 - 1 items are refused (kv_pipe.cu:738)",
     dict(n=1 << 21, nparts=256, part_bytes=16 * MB), None),
    ("48 KB parts, parts >= SMs: ldst256 with whole parts (kv_copy.cu:241, :262)",
     dict(n=40, nparts=4, part_bytes=48 * KB), ("ldst32", False, 48 * KB, 1, 160, None)),
    ("48 KB parts, parts < SMs: 32 KB chunks (kv_copy.cu:240, :254)",
     dict(n=10, nparts=4, part_bytes=48 * KB), ("ldst32", False, 32 * KB, 2, 80, None)),
    ("ld/st: max_ctas is not clamped to the resident grid (kv_copy.cu:254)",
     dict(n=1000, nparts=4, part_bytes=48 * KB, max_ctas=2000),
     ("ldst32", False, 48 * KB, 1, 2000, None)),
    ("ld/st: the resident grid of the 32-byte flavour (kv_copy.cu:254)",
     dict(n=1000, nparts=4, part_bytes=48 * KB), ("ldst32", False, 48 * KB, 1, R32 * SMS, None)),
    ("16-byte aligned parts only: the 16-byte kernel (kv_copy.cu:264)",
     dict(n=1, nparts=3, part_bytes=4 * KB + 16), ("ldst16", False, 4 * KB + 16, 1, 3, None)),
    ("unaligned 128 KB parts: the byte kernel (kv_copy.cu:233, :258)",
     dict(n=2, nparts=2, part_bytes=128 * KB, align_or=4), ("ldst1", False, 32 * KB, 4, 16, None)),
    ("ld/st: 2^31 - 512 items are launched (kv_copy.cu:244)",
     dict(n=(1 << 22) - 1, nparts=1, part_bytes=16 * MB, align_or=1),
     ("ldst1", False, 32 * KB, 512, R16 * SMS, None)),
    ("ld/st: 2^31 items are refused (kv_copy.cu:244)",
     dict(n=1 << 22, nparts=1, part_bytes=16 * MB, align_or=1), None),
]


@pytest.mark.parametrize("case,kw,want", GATHER, ids=[c[0] for c in GATHER])
def test_plan_gather(case, kw, want):
    _check(T.plan_gather(**kw, **RES), want)


# (case, plan_read_fused arguments, expected as for COPY)
READ = [
    ("auto, 128 KB pages: resolver + TMA pipeline (kv_read_fused.cu:140, kv_pipe.cu:803)",
     dict(n=512, bytes=128 * KB), ("tma", False, 128 * KB, 1, SMS, G16)),
    ("tma: small pages stay on TMA when asked (kv_read_fused.cu:140)",
     dict(n=10, bytes=4 * KB, variant=TMA), ("tma", False, 4 * KB, 1, 10, (4 * KB, 16, 64 * KB))),
    ("tma: max_ctas clamped to the SM count (kv_pipe.cu:801)",
     dict(n=512, bytes=128 * KB, variant=TMA, max_ctas=500), ("tma", False, 128 * KB, 1, SMS, G16)),
    ("tma: a few large pages are split over the grid (kv_pipe.cu:803-806)",
     dict(n=4, bytes=4 * MB, variant=TMA), ("tma", False, 128 * KB, 32, 128, G16)),
    ("unaligned tma request: the byte kernel (kv_read_fused.cu:141, :160)",
     dict(n=4, bytes=128 * KB, align_or=8, variant=TMA), ("ldst1", False, 32 * KB, 4, 16, None)),
    ("auto below 64 KB, 32-byte aligned: 32-byte kernel (kv_read_fused.cu:162)",
     dict(n=16, bytes=32 * KB), ("ldst32", False, 32 * KB, 1, 16, None)),
    ("ldst256, whole blocks once n >= SMs (kv_read_fused.cu:144, :157)",
     dict(n=512, bytes=128 * KB, variant=LDST256), ("ldst32", False, 128 * KB, 1, R32 * SMS, None)),
    ("ldst: the 16-byte kernel on a 32-byte aligned batch (kv_read_fused.cu:157, :164 with "
     "align_or | 16)",
     dict(n=512, bytes=128 * KB, variant=LDST), ("ldst16", False, 128 * KB, 1, 512, None)),
    ("16-byte aligned only: the 16-byte kernel (kv_read_fused.cu:164)",
     dict(n=8, bytes=48), ("ldst16", False, 48, 1, 8, None)),
    ("ld/st: max_ctas is not clamped to the resident grid (kv_read_fused.cu:158)",
     dict(n=2000, bytes=64 * KB, variant=LDST256, max_ctas=1000),
     ("ldst32", False, 64 * KB, 1, 1000, None)),
    ("blocks above 1 MB are cut into 32 KB chunks (kv_read_fused.cu:143-144)",
     dict(n=200, bytes=2 * MB, variant=LDST256), ("ldst32", False, 32 * KB, 64, R32 * SMS, None)),
]


@pytest.mark.parametrize("case,kw,want", READ, ids=[c[0] for c in READ])
def test_plan_read_fused(case, kw, want):
    _check(T.plan_read_fused(**kw, **RES), want)


@pytest.mark.parametrize("max_ctas,ctas", [(0, SMS), (500, SMS), (8, 8)])
def test_scatter_read_grid(max_ctas, ctas):
    # kv_pipe.cu:749: a CTA per SM, a caller's cap bounded by it; not clamped to the blocks
    # (the fused scatter needs at least as many blocks as CTAs)
    p = T.plan_read_fused(n=1, bytes=64 * KB, max_ctas=max_ctas, **RES)
    assert p["scatter_ctas"] == ctas


# (case, plan_fp8 arguments, expected as for COPY; chunk in elements)
FP8 = [
    ("auto, 8192-element pages: the pipeline, 8 compute warps, 2 CTAs per SM "
     "(kv_fp8.cu:197, kv_fp8_pipe.cu:309, :312)",
     dict(n=512, elems=8192), ("tma", False, 8192, 1, 2 * SMS, None)),
    ("variant 2: the pipeline with 4 compute warps (kv_fp8_pipe.cu:312)",
     dict(n=512, elems=8192, variant=2), ("tma4", False, 8192, 1, 2 * SMS, None)),
    ("pipeline: max_ctas clamped to 2 x SMs (kv_fp8_pipe.cu:309)",
     dict(n=2000, elems=8192, max_ctas=1000), ("tma", False, 8192, 1, 2 * SMS, None)),
    ("pipeline: a few large pages are cut into tiles (kv_fp8_pipe.cu:288-291)",
     dict(n=8, elems=1 << 19), ("tma", False, 16384, 32, 256, None)),
    ("pipeline: no more CTAs than items (kv_fp8_pipe.cu:311)",
     dict(n=4, elems=8192), ("tma", False, 8192, 1, 4, None)),
    ("variant 1: the ld/st kernels, whole pages once n >= SMs, 6 CTAs per SM (kv_fp8.cu:197, "
     ":203, :206)",
     dict(n=512, elems=8192, variant=1), ("ldst_fp8", False, 8192, 1, 512, None)),
    # every fp8 kernel moves bf16 in 16-byte vectors: unaligned pages are refused, whatever
    # the variant and page size (the ld/st kernels would fault on them)
    ("unaligned pages: refused",
     dict(n=1000, elems=8192, aligned16=False), None),
    ("unaligned pages, ld/st asked for: refused",
     dict(n=1000, elems=8192, variant=1, aligned16=False), None),
    ("unaligned pages of 384 elements: refused",
     dict(n=4, elems=384, aligned16=False), None),
    # kv_fp8.cu:202 passed 8192 for a page of 384 elements; the kernels clip every item at the
    # page's end, so a chunk of the page's size moves the same rows
    ("elems not a multiple of 512: the ld/st kernels (kv_fp8_pipe.cu:297, kv_fp8.cu:215)",
     dict(n=4, elems=384), ("ldst_fp8", False, 384, 1, 4, None)),
    ("ld/st: pages above 2^19 elements are cut into 8192-element chunks (kv_fp8.cu:202-203)",
     dict(n=200, elems=1 << 20, variant=1), ("ldst_fp8", False, 8192, 128, 6 * SMS, None)),
    ("ld/st: max_ctas is not clamped (kv_fp8.cu:206)",
     dict(n=2000, elems=8192, variant=1, max_ctas=1000), ("ldst_fp8", False, 8192, 1, 1000, None)),
]


@pytest.mark.parametrize("case,kw,want", FP8, ids=[c[0] for c in FP8])
def test_plan_fp8(case, kw, want):
    _check(T.plan_fp8(**kw, sm_count=SMS), want)


def test_every_kernel_is_reached():
    seen = {(w[0], w[1]) for table in (COPY, GATHER, READ, FP8) for _, _, w in table if w}
    assert {k for k, _ in seen} == {"ldst1", "ldst16", "ldst32", "ldst16_mc", "tma", "tma4",
                                    "ldst_fp8"}
    # every instantiation that takes parameter descriptors, with and without them
    for k in ("ldst16", "ldst32", "ldst16_mc", "tma"):
        assert {(k, False), (k, True)} <= seen, k
    assert any(w is None for _, _, w in COPY) and any(w is None for _, _, w in GATHER)


# The kernel the fused read of each fused-copy case of test_read_plan.py ran, with aligned
# destinations.  Before, an ldst connection ORed 16 into the launch's align_or to get the 16-byte
# kernel (client_data.cpp:744 with kv_read_fused.cu:147-165); now plan_device_read hands the
# variant over.  Unaligned destinations always ran the byte kernel.
FUSED_COPY_KERNEL = {
    "small batch, local": "ldst32",
    "small batch over NVLink": "ldst32",
    "small batch, ldst": "ldst16",
    "whole blocks, auto, local": "ldst32",
    "whole blocks, auto, over NVLink": "tma",
    "whole blocks, auto, mixed pool": "tma",
    "whole blocks, tma, local": "tma",
    "whole blocks, tma, over NVLink": "tma",
    "whole blocks, ldst, local": "ldst16",
    "whole blocks, max_ctas": "tma",
}


def test_every_fused_copy_case_is_listed():
    fused = {c[0] for c in READ_CASES if c[2][0] == "fused_copy"}
    assert fused == set(FUSED_COPY_KERNEL)


@pytest.mark.parametrize("case", sorted(FUSED_COPY_KERNEL))
@pytest.mark.parametrize("align_or", [0, 8])
def test_device_read_then_fused_copy(case, align_or):
    kw = next(c[1] for c in READ_CASES if c[0] == case)
    read = T.plan_device_read(sm_count=SMS, **kw)
    assert read["path"] == "fused_copy"
    p = T.plan_read_fused(n=kw["n"], bytes=kw["block_bytes"], align_or=align_or,
                          variant=read["variant"], max_ctas=read["grid_cap"], **RES)
    assert p["kernel"] == (FUSED_COPY_KERNEL[case] if align_or == 0 else "ldst1")
