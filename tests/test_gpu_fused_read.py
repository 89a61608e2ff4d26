"""The fused reads, launched directly (ops.read_fused) and compared with what was published.

Four kernels resolve keys in the device index and copy in one launch: kv_read_fused (byte,
16- and 32-byte flavours), kv_pipe_read, kv_fp8_pipe's resolving read and kv_pipe_scatter_read.
Every test builds its index tables through the kernels' own publish path (kv_copy with
``publish=``; sharded tables are separate tables on cuda:0) and keeps a dict key -> (addr,
size, committed) next to the pool bytes.  That is all the expected answer needs: a key reads its
pool bytes when it was committed, holds at least the bytes asked for, and its address names a
segment with a base; otherwise it is a miss, counted once per block, and leaves its
destination untouched.  fp8 pages are compared bit for bit with the exact dequantiser of
tests/fp8_exact.py (NaN as NaN).  Every destination page has canary bytes around it and the
destination slots are permuted.  Each flavour is forced through the variant and the alignment
of its geometry (Geo); one torch.profiler session confirms which kernel each of them runs."""
import numpy as np
import pytest
import torch

import fp8_exact as fe

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
CANARY = 0xA5
GAP = 64          # canary bytes before every destination page (32-byte multiple)
OFF_MASK = (1 << 44) - 1
MISS_KINDS = ("absent", "uncommitted", "short", "seg_over", "seg_zero", "seg_field0")
# slots of the index tables of shards 0..7: different sizes on purpose
SHARD_SLOTS = (8192, 2048, 4096, 1024, 2048, 4096, 1024, 2048)


def _ops():
    from infinistore_b200 import ops

    return ops


def _native():
    from infinistore_b200 import _infinistore as m

    return m


def _round_up(x, a):
    return (x + a - 1) // a * a


class Geo:
    """A kernel flavour and the page geometry that selects it.  `need`: bytes an entry must
    hold; `block`: bytes stored per pool block; `out`: destination bytes per region and block;
    `regions`: destination regions (parts of a gathered read)."""

    def __init__(self, flavour, big=False, nparts=3, first_part=1, part_bytes=None):
        self.flavour = flavour
        self.elems, self.bytes, self.nparts, self.first_part, self.part_bytes = 0, 0, 0, 0, 0
        self.regions = 1
        self.variant = {"byte": "ldst", "ldst16": "ldst", "ldst32": "ldst256",
                        "pipe": "tma"}.get(flavour, "auto")
        self.kernel = {"byte": "kv_read_fused_kernel<1>", "ldst16": "kv_read_fused_kernel<16>",
                       "ldst32": "kv_read_fused_kernel<32>", "pipe": "kv_pipe_read_kernel",
                       "fp8": "kv_fp8_pipe_kernel<false, 8, true>",
                       "scatter": "kv_pipe_scatter_read_kernel"}[flavour]
        mb = 1 << 20
        if flavour == "fp8":
            self.elems = 512 * 1025 if big else 1024
            self.need = self.block = self.elems + self.elems // 128 * 4
            self.out = 2 * self.elems
        elif flavour == "scatter":
            self.nparts, self.first_part = nparts, first_part
            self.part_bytes = part_bytes or ((mb >> 1) if big else 512)
            self.need = (first_part + nparts) * self.part_bytes
            self.block = self.need + self.part_bytes  # one stored part past the read
            self.out = self.part_bytes
            self.regions = nparts
        else:
            extra = {"byte": 3, "ldst16": 16, "ldst32": 32, "pipe": 48}[flavour]
            self.bytes = (mb if big else 4096) + extra
            if flavour == "byte":
                self.bytes = mb + 3 if big else 1003
            self.need = self.block = self.out = self.bytes
        self.odd = flavour == "byte"  # unaligned pool and destination addresses

    def expect(self, src: np.ndarray):
        """Destination bytes of every region for a block whose pool bytes are `src`."""
        if self.flavour == "fp8":
            e = self.elems
            scales = src[e:e + e // 128 * 4].copy().view(np.float32)
            return [fe.dequantise(src[:e].reshape(-1, 128), scales).reshape(-1).view(np.uint8)]
        if self.flavour == "scatter":
            pb = self.part_bytes
            return [src[(self.first_part + s) * pb:(self.first_part + s + 1) * pb]
                    for s in range(self.nparts)]
        return [src[:self.bytes]]


class Store:
    """Pool bytes in `nbases` segments over one tensor (one base of 0 among several), index
    tables of `nshards` shards, and what was published into them."""

    def __init__(self, geo: Geo, nblocks: int, nbases: int = 1, nshards: int = 1, seed: int = 0):
        ops = _ops()
        self.geo = geo
        self.rng = np.random.default_rng(seed)
        self.nbases = nbases
        self.hole = nbases // 2 if nbases > 1 else None
        usable = [s for s in range(nbases) if s != self.hole]
        slot = _round_up(geo.block + 32, 256)
        self.span = -(-nblocks // len(usable)) * slot + 256
        host = self.rng.integers(0, 256, nbases * self.span, dtype=np.uint8)
        self.loc = []  # (segment, offset in it) of pool block j
        for j in range(nblocks):
            s, k = usable[j % len(usable)], j // len(usable)
            off = k * slot + (1 + (j * 5) % 13 if geo.odd else 0)
            self.loc.append((s, off))
            if geo.flavour == "fp8":  # finite and special scales, every payload code
                at = s * self.span + off + geo.elems
                sc = self.rng.choice(fe.read_scales(), geo.elems // 128).astype(np.float32)
                host[at:at + sc.nbytes] = sc.view(np.uint8)
        self.host = host
        self.pool = torch.from_numpy(host).to(DEV)
        base = self.pool.data_ptr()
        self.seg_base = [0 if s == self.hole else base + s * self.span for s in range(nbases)]
        self.tables = [ops.new_index_table(SHARD_SLOTS[i], DEV) for i in range(nshards)]
        self.published = {}  # key -> (addr, size, committed)
        self.gen = 1
        self.sink = torch.zeros(16, dtype=torch.uint8, device=DEV)

    @property
    def shards(self):
        return self.tables[1:]

    def addr(self, j: int) -> int:
        s, off = self.loc[j]
        return ((s + 1) << 44) | off

    def publish(self, keys, addrs, size, committed=True):
        """Publish `keys` with kv_copy's in-band commit (debug=4 stops before the tag store:
        claimed, never committed).  The copy itself moves 16 bytes to a scratch buffer."""
        ops = _ops()
        n = len(keys)
        if n == 0:
            return
        scratch = torch.zeros(16 * n, dtype=torch.uint8, device=DEV)
        descs = ops.make_descs([self.sink.data_ptr()] * n,
                               [scratch.data_ptr() + 16 * i for i in range(n)], DEV)
        gens = list(range(self.gen, self.gen + n))
        self.gen += n
        status = torch.zeros(8, dtype=torch.int32, device=DEV)
        pub = ops.PublishArgs(self.tables[0], keys, addrs, gens, size, shards=self.shards)
        ops.kv_copy(descs, 16, variant="ldst", publish=pub, status=status,
                    debug=0 if committed else 4)
        torch.cuda.synchronize()
        assert int(status[1]) == 0, "an index table was full"
        for k, a in zip(keys, addrs):
            assert k not in self.published
            self.published[k] = (a, size, committed)

    def source(self, key):
        """The pool bytes `key` reads, or None for a miss."""
        if key not in self.published:
            return None
        addr, size, committed = self.published[key]
        seg = (addr >> 44) - 1
        if not committed or size < self.geo.need or not 0 <= seg < self.nbases:
            return None
        if self.seg_base[seg] == 0:
            return None
        at = seg * self.span + (addr & OFF_MASK)
        return self.host[at:at + self.geo.block]

    def read(self, keys, max_ctas=0, validate=True, stage_bytes=0, ring_bytes=0):
        """Read `keys` into permuted destination slots.  Returns (got, want, status)."""
        ops, g = _ops(), self.geo
        n = len(keys)
        stride = _round_up(g.out + 2 * GAP + 16, 256)
        region = n * stride
        dst = torch.full((g.regions * region,), CANARY, dtype=torch.uint8, device=DEV)
        slots = self.rng.permutation(n)
        shift = [(1 + (i * 3) % 11) if g.odd else 0 for i in range(n)]
        dst_off = [int(slots[i]) * stride + GAP + shift[i] for i in range(n)]
        want = np.full(g.regions * region, CANARY, dtype=np.uint8)
        for i, k in enumerate(keys):
            src = self.source(k)
            if src is None:
                continue
            for r, b in enumerate(g.expect(src)):
                want[r * region + dst_off[i]:r * region + dst_off[i] + b.size] = b
        status = torch.zeros(8, dtype=torch.int32, device=DEV)
        kw = dict(shards=self.shards, variant=g.variant, max_ctas=max_ctas, validate=validate,
                  stage_bytes=stage_bytes, ring_bytes=ring_bytes)
        if g.flavour == "scatter":
            kw.update(part_base=[dst.data_ptr() + r * region for r in range(g.regions)],
                      part_bytes=g.part_bytes, first_part=g.first_part)
            base = 0
        else:
            base = dst.data_ptr()
        if g.flavour == "fp8":
            kw.update(elems=g.elems)

        ops.read_fused(self.tables[0], keys, base, dst_off, g.bytes, self.seg_base, status, **kw)
        torch.cuda.synchronize()
        return dst.cpu().numpy(), want, status.cpu().numpy()

    def check(self, keys, **kw):
        """Read `keys`; the destination must equal the model, every miss must be counted once
        and nothing may be stale.  Returns the number of misses."""
        got, want, status = self.read(keys, **kw)
        _assert_dst(got, want, self.geo.flavour == "fp8")
        misses = sum(self.source(k) is None for k in keys)
        assert int(status[0]) == misses, (int(status[0]), misses)
        assert int(status[3]) == 0
        return misses


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def _assert_dst(got: np.ndarray, want: np.ndarray, bf16: bool):
    if bf16:  # NaN compared as NaN; the canary 0xa5a5 is a finite bf16 value
        g, w = got.view(np.uint16), want.view(np.uint16)
        gn, wn = np.isnan(fe.bf16_to_f64(g)), np.isnan(fe.bf16_to_f64(w))
        assert np.array_equal(gn, wn), f"NaN at {np.flatnonzero(gn != wn)[:8]}"
        bad = np.flatnonzero((g != w) & ~wn)
    else:
        bad = np.flatnonzero(got != want)
    assert bad.size == 0, f"{bad.size} differ, first at {bad[:8]}"


def _keys(rng, n, taken):
    """`n` new distinct keys of 0 to 700 bytes."""
    lens = (0, 1, 5, 7, 8, 9, 31, 63, 64, 65, 255, 256, 257, 700)
    out, attempt = [], 0
    while len(out) < n:
        L = int(lens[attempt % len(lens)])
        attempt += 1
        k = bytes(rng.integers(0, 256, L, dtype=np.uint8))
        if k not in taken:
            taken.add(k)
            out.append(k)
    return out


def _build(store: Store, kinds, taken=None):
    """Publish one key per batch item of kind kinds[i] ("hit" or a MISS_KINDS entry) and return
    the batch.  Item i's entry points at pool block i; a hit holds exactly the bytes read."""
    g = store.geo
    taken = set() if taken is None else taken
    keys = _keys(store.rng, len(kinds), taken)
    groups = {}  # (size, committed) -> ([keys], [addrs])
    for i, kind in enumerate(kinds):
        addr, size, committed = store.addr(i), g.need, True
        off = addr & OFF_MASK
        if kind == "absent":
            continue
        if kind == "uncommitted":
            committed = False
        elif kind == "short":
            size = g.need - 16
        elif kind == "seg_over":  # segment id == nsegs
            addr = ((store.nbases + 1) << 44) | off
        elif kind == "seg_zero":  # a segment whose base is 0 (past nsegs with one base)
            seg = store.hole if store.hole is not None else store.nbases + 3
            addr = ((seg + 1) << 44) | off
        elif kind == "seg_field0":  # segment field 0: the id wraps to 0xffffffff
            addr = off
        ks, ads = groups.setdefault((size, committed), ([], []))
        ks.append(keys[i])
        ads.append(addr)
    for (size, committed), (ks, ads) in groups.items():
        store.publish(ks, ads, size, committed)
    return keys


FLAVOURS = ["byte", "ldst16", "ldst32", "pipe", "fp8", "scatter"]
EDGES = (0, 31, 32, 63, 64)


def test_every_flavour_runs_its_kernel():
    """The geometry of each flavour, small pages and pages above 1 MB, selects the kernel it is
    named for: one profiler session over all of them, each read checked against the model."""
    stores = []
    for big in (False, True):
        for flavour in FLAVOURS:
            g = Geo(flavour, big=big)
            n = 5 if big else 40
            store = Store(g, n, nbases=3, seed=FLAVOURS.index(flavour) + 50 * big)
            kinds = ["hit"] * n
            kinds[1] = "absent"
            stores.append((store, _build(store, kinds)))
    names = _kernels(lambda: [s.check(k, max_ctas=4) for s, k in stores])
    for store, _ in stores:
        assert any(store.geo.kernel in k for k in names), (store.geo.kernel, sorted(set(names)))


@pytest.mark.parametrize("nbases", [1, 3, 16])
@pytest.mark.parametrize("flavour", FLAVOURS)
def test_misses_at_resolver_batch_edges(flavour, nbases):
    """Six CTAs of 97 items each (4 resolver rounds); CTA c has miss kind c at its items 0, 31,
    32, 63, 64 and 96, where the double-buffered resolver queue changes halves.  One key is
    asked twice for two destinations.  Entries are spread over the segments."""
    ctas, per = 6, 97
    g = Geo(flavour)
    n = ctas * per
    store = Store(g, n, nbases=nbases, seed=nbases * 31 + FLAVOURS.index(flavour))
    kinds = ["hit"] * n
    for c, kind in enumerate(MISS_KINDS):
        for p in EDGES + (per - 1,):
            kinds[c + p * ctas] = kind
    keys = _build(store, kinds)
    keys[5 * ctas + 1] = keys[3 * ctas]  # one key, two destinations (item 3 of CTA 0 is a hit)
    assert kinds[3 * ctas] == "hit"
    assert store.check(keys, max_ctas=ctas) == len(MISS_KINDS) * (len(EDGES) + 1)


@pytest.mark.parametrize("rounds", [1, 2, 3, 7, "few"])
@pytest.mark.parametrize("flavour", FLAVOURS)
def test_resolver_rounds_and_small_grids(flavour, rounds):
    """1, 2, 3 and 7 resolver rounds per CTA on a grid of 3 (the CTAs' item counts differ), and
    fewer blocks than the kernel's default grid (not for the scatter read, which needs a block
    per CTA: test_scatter_read_refuses_fewer_blocks_than_ctas)."""
    if rounds == "few" and flavour == "scatter":
        pytest.skip("kv_pipe_scatter_read needs at least as many blocks as CTAs")
    g = Geo(flavour)
    ctas = 0 if rounds == "few" else 3
    n = 3 if rounds == "few" else 3 * 32 * (rounds - 1) + 3 * 17 - 1
    store = Store(g, n, nbases=3, seed=100 + n)
    kinds = ["hit"] * n
    for i in store.rng.choice(n, max(1, n // 9), replace=False):
        kinds[i] = MISS_KINDS[i % len(MISS_KINDS)]
    keys = _build(store, kinds)
    store.check(keys, max_ctas=ctas)


@pytest.mark.parametrize("flavour", FLAVOURS)
def test_chunked_blocks_count_a_miss_once(flavour):
    """Blocks above 1 MB on the default grid, cut into chunks over several CTAs (the scatter
    read: parts of 512 KB on 4 CTAs); the missing block counts once, not once per chunk."""
    g = Geo(flavour, big=True)
    n = 5
    store = Store(g, n, seed=7)
    keys = _build(store, ["hit", "hit", "absent", "hit", "short"])
    store.check(keys, max_ctas=4 if flavour == "scatter" else 0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if flavour in ("byte", "ldst16", "ldst32", "pipe"):
        variant = {"byte": 1, "ldst16": 1, "ldst32": 3, "pipe": 2}[flavour]
        plan = _native().testing.plan_read_fused(n, g.bytes, 1 if g.odd else 0, variant,
                                                 sm_count=sms)
        kernel = {"byte": "ldst1", "ldst16": "ldst16", "ldst32": "ldst32", "pipe": "tma"}
        assert plan["cpb"] > 1 and plan["kernel"] == kernel[flavour], plan


@pytest.mark.parametrize("stage_kb,ring_kb", [(4, 12), (8, 64), (16, 128), (32, 192)])
@pytest.mark.parametrize("flavour", ["pipe", "scatter"])
def test_pipe_ring_geometries(flavour, stage_kb, ring_kb):
    """The TMA reads with the ring geometries of the TMA copy tests: a 3-slot ring, slots that
    do not divide the page, a page split over several slots."""
    g = Geo(flavour, part_bytes=40960 + 16) if flavour == "scatter" else Geo(flavour)
    if flavour == "pipe":
        g.bytes = g.need = g.block = g.out = 40960 + 16
    n = 70
    store = Store(g, n, seed=stage_kb)
    kinds = ["hit"] * n
    kinds[0], kinds[33], kinds[n - 1] = "absent", "short", "uncommitted"
    keys = _build(store, kinds)
    store.check(keys, max_ctas=5, stage_bytes=stage_kb << 10, ring_bytes=ring_kb << 10)


@pytest.mark.parametrize("nparts", [1, 3, 256])
def test_scatter_read_parts(nparts):
    """kv_pipe_scatter_read with 1, 3 and GATHER_MAX_PARTS parts from stored part 2 on, misses
    at resolver batch edges, more blocks than CTAs."""
    assert _native().kernels.GATHER_MAX_PARTS == 256
    g = Geo("scatter", nparts=nparts, first_part=2, part_bytes=64 if nparts == 256 else 1024)
    ctas, n = 4, 4 * 70
    store = Store(g, n, nbases=3, seed=nparts)
    kinds = ["hit"] * n
    for j, p in enumerate((0, 31, 32, 63, 64, 69)):
        kinds[(j % ctas) + p * ctas] = MISS_KINDS[j]
    keys = _build(store, kinds)
    assert store.check(keys, max_ctas=ctas) == 6


def test_scatter_read_refuses_fewer_blocks_than_ctas():
    """Fewer blocks than CTAs is refused with ValueError, and nothing is launched: the
    destination and the status stay as they were."""
    ops = _ops()
    g = Geo("scatter")
    store = Store(g, 3, seed=3)
    keys = _build(store, ["hit"] * 3)
    dst = torch.full((3 * 4096,), CANARY, dtype=torch.uint8, device=DEV)
    status = torch.full((8,), 7, dtype=torch.int32, device=DEV)
    with pytest.raises(ValueError, match="as many blocks as CTAs"):
        ops.read_fused(store.tables[0], keys, 0, [0, 1024, 2048], 0, store.seg_base, status,
                       part_base=[dst.data_ptr() + s * 4096 for s in range(3)],
                       part_bytes=g.part_bytes, first_part=1, max_ctas=8)
    torch.cuda.synchronize()
    assert (dst == CANARY).all() and (status == 7).all()


@pytest.mark.parametrize("nshards", [1, 2, 3, 8])
@pytest.mark.parametrize("flavour", FLAVOURS)
def test_sharded_index(flavour, nshards):
    """1, 2, 3 and 8 index tables of different sizes on cuda:0, published with shards=.  Every
    shard holds keys; every key is found by the fused read; index_lookup's found_at slot ids
    carry the key's shard; index_validate passes them, and after index_erase of some keys on
    the table that holds them counts exactly those; a fused read then misses exactly them."""
    ops, m = _ops(), _native()
    g = Geo(flavour)
    n = 400
    store = Store(g, n, nbases=3, nshards=nshards, seed=nshards * 11 + FLAVOURS.index(flavour))
    keys = _build(store, ["hit"] * n)
    shard_of = [m.testing.index_shard_of(k, nshards) for k in keys]
    assert sorted(set(shard_of)) == list(range(nshards))
    assert store.check(keys, max_ctas=8) == 0

    found = torch.zeros((n, 2), dtype=torch.int32, device=DEV)
    descs, present, _ = ops.index_lookup(store.tables[0], keys, seg_base=store.seg_base,
                                         dst_off=[0] * n, need_bytes=g.need, found_at=found,
                                         shards=store.shards)
    torch.cuda.synchronize()
    assert all(ops.presence_bits(present, n))
    slot = found[:, 0].cpu().numpy().view(np.uint32)
    assert (slot & ((1 << 29) - 1)).all()
    assert ((slot >> 29) == np.array(shard_of, dtype=np.uint32)).all()
    assert ops.index_validate(store.tables[0], found, shards=store.shards) == 0

    erased = [i for i in range(n) if i % 7 == 3]
    for s in range(nshards):
        mine = [i for i in erased if shard_of[i] == s]
        ops.index_erase(store.tables[s], [keys[i] for i in mine], [store.addr(i) for i in mine])
    assert ops.index_validate(store.tables[0], found, shards=store.shards) == len(erased)
    for i in erased:
        del store.published[keys[i]]
    assert store.check(keys, max_ctas=8) == len(erased)
