// Python binding: module infinistore_b200._infinistore.
//
// Surface parity with the reference's pybind module (src/pybind.cpp:36-210): ClientConfig,
// ServerConfig, Connection, register_server, purge_kv_map, get_kvmap_len, log_msg,
// set_log_level; allocate results are a zero-copy numpy structured array with rkey:u4 @0
// and remote_addr:u8 @8 (itemsize 16).  Every blocking call releases the GIL; callbacks
// of the async API re-acquire it on the connection's completion thread.
// Extras: a Server class (several servers per process, SPMD ranks hosting pool shards),
// introspection (stats, segments), and raw launchers of the sm_90a kernels plus the wire
// codec / allocator for unit tests.
#include <pybind11/functional.h>
#include <pybind11/numpy.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include <cuda_runtime_api.h>

#include <unistd.h>

#include <cstring>
#include <memory>
#include <mutex>
#include <string_view>

#include "core/config.h"
#include "core/hash.h"
#include "core/kv_store.h"
#include "core/log.h"
#include "core/mempool.h"
#include "core/trace.h"
#include "ctrl/client.h"
#include "ctrl/client_dev.h"
#include "ctrl/read_plan.h"
#include "ctrl/server.h"
#include "ctrl/staging.h"
#include "fabric/nvls.h"
#include "fabric/segment.h"
#include "kernels/balance.h"
#include "kernels/kernels.h"
#include "kernels/launch_plan.h"
#include "wire/messages.h"

namespace py = pybind11;
using namespace istore;

namespace {

std::mutex g_server_mu;
std::unique_ptr<Server> g_server;

py::array_t<RemoteBlock> blocks_to_array(std::vector<RemoteBlock>&& v) {
    auto* heap = new std::vector<RemoteBlock>(std::move(v));
    py::capsule owner(heap, [](void* p) { delete static_cast<std::vector<RemoteBlock>*>(p); });
    return py::array_t<RemoteBlock>(heap->size(), heap->data(), owner);
}

// Remote blocks arrive as the structured array returned by allocate (possibly sliced):
// used in place when contiguous; otherwise converted into `tmp`.
struct BlockSpan {
    const RemoteBlock* data = nullptr;
    size_t n = 0;
    std::vector<RemoteBlock> tmp;
    py::object keep;
};

void blocks_from_py(const py::object& obj, BlockSpan& out) {
    if (py::isinstance<py::array>(obj)) {
        py::array arr = py::reinterpret_borrow<py::array>(obj);
        if (arr.itemsize() == sizeof(RemoteBlock) && arr.ndim() == 1) {
            if (arr.strides(0) == py::ssize_t(sizeof(RemoteBlock))) {
                out.data = static_cast<const RemoteBlock*>(arr.data());
                out.n = size_t(arr.shape(0));
                out.keep = arr;
                return;
            }
            out.tmp.resize(size_t(arr.shape(0)));
            const char* base = static_cast<const char*>(arr.data());
            for (py::ssize_t i = 0; i < arr.shape(0); ++i)
                std::memcpy(&out.tmp[size_t(i)], base + i * arr.strides(0), sizeof(RemoteBlock));
            out.data = out.tmp.data();
            out.n = out.tmp.size();
            return;
        }
    }
    for (auto item : obj) {  // list of (rkey, remote_addr) or (rkey, gen, remote_addr)
        py::tuple t = py::cast<py::tuple>(item);
        RemoteBlock b{};
        if (t.size() == 2) {
            b.rkey = t[0].cast<uint32_t>();
            b.remote_addr = t[1].cast<uint64_t>();
        } else {
            b.rkey = t[0].cast<uint32_t>();
            b.gen = t[1].cast<uint32_t>();
            b.remote_addr = t[2].cast<uint64_t>();
        }
        out.tmp.push_back(b);
    }
    out.data = out.tmp.data();
    out.n = out.tmp.size();
}

// Offsets: a contiguous int64/uint64 numpy array is used in place, anything else is
// converted element by element with the C API.
struct OffsetSpan {
    const uint64_t* data = nullptr;
    size_t n = 0;
    std::vector<uint64_t> tmp;
    py::object keep;
};

void offsets_from_py(const py::object& obj, OffsetSpan& out) {
    if (py::isinstance<py::array>(obj)) {
        py::array arr = py::reinterpret_borrow<py::array>(obj);
        const char kind = arr.dtype().kind();
        if ((kind == 'i' || kind == 'u') && arr.itemsize() == 8 && arr.ndim() == 1 &&
            arr.strides(0) == 8) {
            out.data = static_cast<const uint64_t*>(arr.data());
            out.n = size_t(arr.shape(0));
            out.keep = arr;
            return;
        }
    }
    PyObject* seq = PySequence_Fast(obj.ptr(), "offsets must be a sequence of integers");
    if (!seq) throw py::error_already_set();
    const Py_ssize_t n = PySequence_Fast_GET_SIZE(seq);
    out.tmp.resize(size_t(n));
    for (Py_ssize_t i = 0; i < n; ++i) {
        const unsigned long long v = PyLong_AsUnsignedLongLong(PySequence_Fast_GET_ITEM(seq, i));
        if (v == (unsigned long long)-1 && PyErr_Occurred()) {
            Py_DECREF(seq);
            throw py::error_already_set();
        }
        out.tmp[size_t(i)] = v;
    }
    Py_DECREF(seq);
    out.data = out.tmp.data();
    out.n = out.tmp.size();
}

// Keys are copied once into a per-thread arena while the GIL is held; the views stay valid
// after the GIL is released for the (possibly blocking) native call.
struct KeyArena {
    // the layout the lookup kernels read (client.h PackedKeys): keys on 8-byte boundaries,
    // zero padded - the data plane copies the arena into its pinned ring as it is
    std::vector<char> bytes;
    std::vector<uint32_t> off, len;
    void clear() {
        bytes.clear();
        off.clear();
        len.clear();
    }
    void add(PyObject* o) {
        const char* p = nullptr;
        Py_ssize_t n = 0;
        if (PyUnicode_Check(o)) {
            p = PyUnicode_AsUTF8AndSize(o, &n);
            if (!p) throw py::error_already_set();
        } else if (PyBytes_Check(o)) {
            p = PyBytes_AS_STRING(o);
            n = PyBytes_GET_SIZE(o);
        } else {
            throw py::type_error("keys must be str or bytes");
        }
        if (bytes.size() + size_t(n) + 8 > 0xffffffffull) throw py::value_error("too many key bytes");
        const size_t at = bytes.size();
        const size_t padded = (std::max<size_t>(size_t(n), 1) + 7) & ~size_t(7);
        off.push_back(uint32_t(at));
        len.push_back(uint32_t(n));
        bytes.resize(at + padded, 0);
        std::memcpy(bytes.data() + at, p, size_t(n));
    }
    std::string_view view(size_t i) const {
        return std::string_view(bytes.data() + off[i], len[i]);
    }
    PackedKeys packed() const {
        return PackedKeys{reinterpret_cast<const uint8_t*>(bytes.data()), bytes.size(), off.data(),
                          len.data(), off.size()};
    }
};

thread_local KeyArena t_arena;

// A gathered call's row geometry from its native list, in bytes: (rows, row_bytes, src_pitch,
// src_col, dst_pitch) or the same followed by (slices, dst_slice_pitch); an empty list is whole
// parts.  `pieces` comes from its own argument.  False unless the list has 0, 5 or 7 entries.
bool parse_rows(const std::vector<uint32_t>& v, uint32_t pieces, kernels::PartRows& r) {
    if (!v.empty() && v.size() != 5 && v.size() != 7) return false;
    r = kernels::PartRows{};
    r.pieces = pieces;
    if (v.empty()) return true;
    r.rows = v[0];
    r.row_bytes = v[1];
    r.src_pitch = v[2];
    r.src_col = v[3];
    r.dst_pitch = v[4];
    if (v.size() == 7) {
        r.slices = v[5];
        r.dst_slice_pitch = v[6];
    }
    return true;
}

// fp8 token records from their native list: (latent, rope) elements, or empty for none.
kernels::Fp8Records parse_records(const std::vector<uint32_t>& v) {
    if (v.empty()) return {};
    if (v.size() != 2 || v[0] == 0)
        throw py::value_error("records is (latent, rope) with latent > 0, or empty");
    return kernels::Fp8Records{v[0], v[1]};
}

// A RoPE shift from its native form: None (no shift, false) or (head_elems, rot_offset,
// rot_dim, interleaved, even_parts, cos, sin) with rot_dim / 2 cosines and sines.  The
// connection and the launcher check the geometry and the values.
bool parse_rope(const py::object& o, kernels::RopeShift& r) {
    if (o.is_none()) return false;
    const auto t = o.cast<py::tuple>();
    if (t.size() != 7)
        throw py::value_error("rope is (head_elems, rot_offset, rot_dim, interleaved, "
                              "even_parts, cos, sin)");
    r = kernels::RopeShift{};
    r.head_elems = t[0].cast<uint32_t>();
    r.rot_offset = t[1].cast<uint32_t>();
    r.rot_dim = t[2].cast<uint32_t>();
    r.interleaved = t[3].cast<bool>() ? 1 : 0;
    r.even_parts = t[4].cast<bool>() ? 1 : 0;
    const auto c = t[5].cast<std::vector<float>>(), s = t[6].cast<std::vector<float>>();
    if (r.rot_dim % 2 || c.size() != r.rot_dim / 2 || s.size() != c.size() ||
        c.size() > kernels::kRopeMaxPairs)
        throw py::value_error("rope: rot_dim / 2 (at most 128) cosines and as many sines");
    for (size_t i = 0; i < c.size(); ++i) {
        r.c[i] = c[i];
        r.s[i] = s[i];
    }
    return true;
}

// A gathered call's parts: part s at part_base[s] (which must outlive the spec); elems > 0:
// bf16 parts of elems elements stored as fp8 pages, or with records (parse_records) as token
// records.  rows: a row-sliced read's or write's geometry (parse_rows); empty: whole parts.
// scales: one per part for e4m3 parts (GatherSpec::part_scale), or empty.  scales and
// part_base must outlive the spec.  The connection checks the values.
Connection::GatherSpec gather_spec(const std::vector<uint64_t>& part_base, uint32_t part_bytes,
                                   uint32_t elems, uint32_t first_part,
                                   const std::vector<uint32_t>& rows = {},
                                   const std::vector<uint64_t>* piece_off = nullptr,
                                   uint32_t pieces = 1,
                                   const std::vector<uint32_t>& records = {},
                                   const std::vector<float>& scales = {}) {
    Connection::GatherSpec g;
    g.records = parse_records(records);
    if (!scales.empty()) {
        if (scales.size() != part_base.size())
            throw py::value_error("scales holds one scale per part");
        g.part_scale = scales.data();
    }
    if (pieces > 1) g.piece_off = piece_off->data();
    g.part_base = part_base.data();
    g.nparts = uint32_t(part_base.size());
    g.part_bytes = part_bytes;
    g.fp8_elems = elems;
    g.first_part = first_part;
    if (!parse_rows(rows, pieces, g.rows))
        throw py::value_error("rows is (rows, row_bytes, src_pitch, src_col, dst_pitch[, "
                              "slices, dst_slice_pitch])");
    return g;
}

// A gathered call's piece table: `pieces` local offsets per block of n blocks (a flat int64
// ndarray or list, n * pieces values), times `scale`.  pieces <= 1: none (empty).
std::vector<uint64_t> piece_table(const py::object& obj, size_t n, uint32_t pieces,
                                  uint64_t scale) {
    std::vector<uint64_t> out;
    if (pieces <= 1) return out;
    if (obj.is_none()) throw py::value_error("pieces > 1 need piece_off");
    OffsetSpan off;
    offsets_from_py(obj, off);
    if (off.n != n * pieces)
        throw py::value_error("piece_off holds `pieces` offsets for every block");
    out.resize(off.n);
    for (size_t i = 0; i < off.n; ++i) out[i] = off.data[i] * scale;
    return out;
}

// A row-sliced launch as the plan bindings of _infinistore.testing describe it: part_bytes is
// rows * src_pitch, and group_parts > 0 makes it a layered read (the plans only ask whether
// group_flags is set).
kernels::GatherLaunch rows_launch(uint32_t n, uint32_t nparts, bool write,
                                  const kernels::PartRows& rows, uint64_t align_or,
                                  uint32_t group_parts, int max_ctas) {
    static uint32_t flags[1];
    kernels::GatherLaunch a;
    a.n = n;
    a.nparts = nparts;
    a.write = write;
    a.part_bytes = uint32_t(uint64_t(rows.rows) * rows.src_pitch);
    a.rows = rows;
    a.align_or = align_or;
    a.group_flags = group_parts ? flags : nullptr;
    a.group_parts = group_parts;
    a.max_ctas = max_ctas;
    return a;
}

// [(key, offset), ...] -> KeyOffset views (offset * scale bytes).  Also accepted: the pair
// (keys, offsets) with `keys` a sequence of str / bytes and `offsets` an integer ndarray of the
// same length - callers that hold their offsets in numpy anyway skip one heap object and one
// integer conversion per block (the walk below is bound by exactly those cache misses).
void blocks_list_from_py(const py::object& obj, uint64_t scale, std::vector<KeyOffset>& out) {
    KeyArena& a = t_arena;
    a.clear();
    if (PyTuple_Check(obj.ptr()) && PyTuple_GET_SIZE(obj.ptr()) == 2 &&
        py::isinstance<py::array>(py::handle(PyTuple_GET_ITEM(obj.ptr(), 1)))) {
        auto offs = py::array_t<int64_t, py::array::c_style | py::array::forcecast>::ensure(
            py::reinterpret_borrow<py::object>(PyTuple_GET_ITEM(obj.ptr(), 1)));
        if (!offs || offs.ndim() != 1) throw py::type_error("offsets must be a 1-D integer array");
        PyObject* seq = PySequence_Fast(PyTuple_GET_ITEM(obj.ptr(), 0), "keys must be a sequence of str");
        if (!seq) throw py::error_already_set();
        const Py_ssize_t n = PySequence_Fast_GET_SIZE(seq);
        if (n != offs.shape(0)) {
            Py_DECREF(seq);
            throw py::value_error("keys and offsets differ in length");
        }
        PyObject** items = PySequence_Fast_ITEMS(seq);
        try {
            for (Py_ssize_t i = 0; i < n; ++i) {
                if (i + 8 < n) __builtin_prefetch(items[i + 8]);
                a.add(items[i]);
            }
        } catch (...) {
            Py_DECREF(seq);
            throw;
        }
        Py_DECREF(seq);
        const int64_t* o = offs.data();
        out.resize(size_t(n));
        for (size_t i = 0; i < size_t(n); ++i) {
            if (o[i] < 0) throw py::value_error("negative offset");
            out[i] = KeyOffset{a.view(i), uint64_t(o[i]) * scale};
        }
        return;
    }
    PyObject* seq = PySequence_Fast(obj.ptr(), "blocks must be a sequence of (key, offset)");
    if (!seq) throw py::error_already_set();
    const Py_ssize_t n = PySequence_Fast_GET_SIZE(seq);
    std::vector<uint64_t> offs;
    offs.resize(size_t(n));
    // The walk is bound by cache misses, not instructions: every pair, key and offset is its
    // own heap object (three dependent misses per block when a layer's list has gone cold).
    // Two-stage software prefetch: the pair 16 ahead, the members of the pair 8 ahead.
    PyObject** items = PySequence_Fast_ITEMS(seq);
    for (Py_ssize_t i = 0; i < n; ++i) {
        if (i + 16 < n) __builtin_prefetch(items[i + 16]);
        if (i + 8 < n) {
            PyObject* ahead = items[i + 8];
            if (PyTuple_Check(ahead) && PyTuple_GET_SIZE(ahead) == 2) {
                __builtin_prefetch(PyTuple_GET_ITEM(ahead, 0));
                __builtin_prefetch(reinterpret_cast<char*>(PyTuple_GET_ITEM(ahead, 0)) + 64);
                __builtin_prefetch(PyTuple_GET_ITEM(ahead, 1));
            }
        }
        PyObject* item = items[i];
        PyObject *k, *o;
        if (PyTuple_Check(item) && PyTuple_GET_SIZE(item) == 2) {
            k = PyTuple_GET_ITEM(item, 0);
            o = PyTuple_GET_ITEM(item, 1);
        } else if (PyList_Check(item) && PyList_GET_SIZE(item) == 2) {
            k = PyList_GET_ITEM(item, 0);
            o = PyList_GET_ITEM(item, 1);
        } else {
            Py_DECREF(seq);
            throw py::type_error("each block must be a (key, offset) pair");
        }
        const unsigned long long v = PyLong_AsUnsignedLongLong(o);
        if (v == (unsigned long long)-1 && PyErr_Occurred()) {
            Py_DECREF(seq);
            throw py::error_already_set();
        }
        try {
            a.add(k);
        } catch (...) {
            Py_DECREF(seq);
            throw;
        }
        offs[size_t(i)] = v * scale;
    }
    Py_DECREF(seq);
    out.resize(size_t(n));
    for (size_t i = 0; i < size_t(n); ++i) out[i] = KeyOffset{a.view(i), offs[i]};
}

void keys_from_py(const py::object& obj, std::vector<std::string_view>& out) {
    KeyArena& a = t_arena;
    a.clear();
    PyObject* seq = PySequence_Fast(obj.ptr(), "keys must be a sequence of str");
    if (!seq) throw py::error_already_set();
    const Py_ssize_t n = PySequence_Fast_GET_SIZE(seq);
    try {
        for (Py_ssize_t i = 0; i < n; ++i) a.add(PySequence_Fast_GET_ITEM(seq, i));
    } catch (...) {
        Py_DECREF(seq);
        throw;
    }
    Py_DECREF(seq);
    out.resize(size_t(n));
    for (size_t i = 0; i < size_t(n); ++i) out[i] = a.view(i);
}

py::dict segment_dict(const SegmentInfo& s) {
    py::dict d;
    d["id"] = s.id;
    d["kind"] = s.kind == kSegDeviceIpc ? "hbm" : (s.kind == kSegReplica ? "nvls-replica" : "host");
    d["device"] = s.device;
    d["granule"] = s.granule;
    d["bytes"] = s.bytes;
    d["index_slots"] = s.index_slots;
    d["map_bytes"] = s.map_bytes;
    return d;
}

py::dict stats_dict(const ServerStats& s) {
    py::dict d;
    d["connections"] = s.connections;
    d["accepted"] = s.accepted;
    d["requests"] = s.requests;
    d["bad_requests"] = s.bad_requests;
    d["keys"] = s.keys;
    d["inflight"] = s.inflight;
    d["pool_bytes"] = s.pool_bytes;
    d["used_bytes"] = s.used_bytes;
    d["segments"] = s.segments;
    d["evicted"] = s.evicted;
    d["lookup_hits"] = s.lookup_hits;
    d["lookup_misses"] = s.lookup_misses;
    d["dedup_skips"] = s.dedup_skips;
    d["index_overflows"] = s.index_overflows;
    py::dict ops;
    for (int i = 0; i < 128; ++i)
        if (s.ops[i]) ops[py::str(op_name(char(i)))] = s.ops[i];
    d["ops"] = ops;
    py::dict lat;  // service time of the control-plane ops, microseconds (log2 buckets)
    for (int i = 0; i < 128; ++i) {
        const OpTiming& t = s.timing[i];
        if (!t.count) continue;
        py::dict e;
        e["count"] = t.count;
        e["mean_us"] = double(t.sum_us) / double(t.count);
        e["p50_us"] = t.quantile_us(0.5);
        e["p99_us"] = t.quantile_us(0.99);
        e["max_us"] = t.max_us;
        lat[py::str(op_name(char(i)))] = e;
    }
    d["op_latency_us"] = lat;
    return d;
}

template <typename T>
T* as_ptr(uint64_t p) {
    return reinterpret_cast<T*>(p);
}

// Index shards 1, 2, ... of a launch from their native list of (table address, bucket mask);
// the launch's own table is shard 0.  An empty list leaves the launch unsharded.  Refused
// before any launch: more than kMaxIndexShards tables in all, a null table, and a mask that is
// not slots / 8 - 1 of a power-of-two table whose slot ids fit under the shard bits.
kernels::IndexShards parse_shards(const std::vector<std::pair<uint64_t, uint64_t>>& v) {
    kernels::IndexShards s;
    if (v.empty()) return s;
    if (v.size() + 1 > kernels::kMaxIndexShards)
        throw py::value_error("shards: at most " + std::to_string(kernels::kMaxIndexShards) +
                              " index tables in all");
    constexpr uint64_t kMaxBuckets = (1ull << kernels::kSlotShardShift) / kernels::kIndexWays;
    for (size_t i = 0; i < v.size(); ++i) {
        const auto [table, mask] = v[i];
        if (!table) throw py::value_error("shards: a null index table");
        if (mask >= kMaxBuckets || ((mask + 1) & mask) != 0)
            throw py::value_error("shards: a bucket mask is slots / 8 - 1 of a power-of-two "
                                  "table of at most 2^29 slots");
        s.table[i] = as_ptr<kernels::IndexBucket>(table);
        s.mask[i] = mask;
    }
    s.n = uint32_t(v.size() + 1);
    return s;
}

// Segment bases of a launch that resolves pool addresses, refused past kMaxSegs.
template <typename Launch>
void set_segments(Launch& a, const std::vector<uint64_t>& seg_base) {
    if (seg_base.size() > size_t(Launch::kMaxSegs))
        throw py::value_error("seg_base: at most " + std::to_string(Launch::kMaxSegs) +
                              " segment bases");
    a.nsegs = uint32_t(seg_base.size());
    for (uint32_t i = 0; i < a.nsegs; ++i) a.seg_base[i] = seg_base[i];
}

using ShardList = std::vector<std::pair<uint64_t, uint64_t>>;

}  // namespace

PYBIND11_MODULE(_infinistore, m) {
    m.doc() = "H100-native KV-cache store: control plane, fabric and sm_90a kernels";

    PYBIND11_NUMPY_DTYPE(RemoteBlock, rkey, gen, remote_addr);

    py::class_<ClientConfig>(m, "ClientConfig")
        .def(py::init<>())
        .def_readwrite("service_port", &ClientConfig::service_port)
        .def_readwrite("log_level", &ClientConfig::log_level)
        .def_readwrite("dev_name", &ClientConfig::dev_name)
        .def_readwrite("host_addr", &ClientConfig::host_addr)
        .def_readwrite("ib_port", &ClientConfig::ib_port)
        .def_readwrite("link_type", &ClientConfig::link_type)
        .def_readwrite("device", &ClientConfig::device)
        .def_readwrite("timeout_ms", &ClientConfig::timeout_ms)
        .def_readwrite("pool_hint", &ClientConfig::pool_hint)
        .def_readwrite("posted_commit", &ClientConfig::posted_commit)
        .def_readwrite("doorbell", &ClientConfig::doorbell)
        .def_readwrite("doorbell_idle_us", &ClientConfig::doorbell_idle_us);

    py::class_<ServerConfig>(m, "ServerConfig")
        .def(py::init<>())
        .def_readwrite("service_port", &ServerConfig::service_port)
        .def_readwrite("log_level", &ServerConfig::log_level)
        .def_readwrite("dev_name", &ServerConfig::dev_name)
        .def_readwrite("prealloc_size", &ServerConfig::prealloc_size)
        .def_readwrite("ib_port", &ServerConfig::ib_port)
        .def_readwrite("link_type", &ServerConfig::link_type)
        .def_readwrite("minimal_allocate_size", &ServerConfig::minimal_allocate_size)
        .def_readwrite("num_stream", &ServerConfig::num_stream)
        .def_readwrite("auto_increase", &ServerConfig::auto_increase)
        .def_readwrite("host", &ServerConfig::host)
        .def_readwrite("pool_backend", &ServerConfig::pool_backend)
        .def_readwrite("pool_devices", &ServerConfig::pool_devices)
        .def_readwrite("extend_size", &ServerConfig::extend_size)
        .def_readwrite("prealloc_bytes", &ServerConfig::prealloc_bytes)
        .def_readwrite("index_slots", &ServerConfig::index_slots)
        .def_readwrite("replica_bytes", &ServerConfig::replica_bytes)
        .def_readwrite("evict", &ServerConfig::evict)
        .def_readwrite("evict_ratio", &ServerConfig::evict_ratio)
        .def_readwrite("max_pending_reply_bytes", &ServerConfig::max_pending_reply_bytes)
        .def_readwrite("replica_devices", &ServerConfig::replica_devices);

    // ------------------------------------------------------------ client
    py::class_<Connection, std::shared_ptr<Connection>>(m, "Connection")
        .def(py::init<>())
        .def("close", &Connection::close, py::call_guard<py::gil_scoped_release>())
        .def("init_connection", &Connection::init_connection,
             py::call_guard<py::gil_scoped_release>())
        .def("setup_rdma", &Connection::setup_rdma, py::call_guard<py::gil_scoped_release>())
        .def("check_exist", &Connection::check_exist, py::call_guard<py::gil_scoped_release>())
        .def("get_match_last_index",
             [](Connection& c, const py::object& keys) {
                 std::vector<std::string_view> kv;
                 keys_from_py(keys, kv);
                 py::gil_scoped_release rel;
                 return c.get_match_last_index(kv);
             })
        .def("touch",
             [](Connection& c, const py::object& keys) {
                 std::vector<std::string_view> kv;
                 keys_from_py(keys, kv);
                 py::gil_scoped_release rel;
                 return c.touch(kv);
             })
        .def("sync_local", &Connection::sync_local, py::call_guard<py::gil_scoped_release>())
        .def("sync_rdma", &Connection::sync_rdma, py::call_guard<py::gil_scoped_release>())
        .def("register_mr", &Connection::register_mr, py::arg("ptr"), py::arg("size"),
             py::arg("device") = -1, py::call_guard<py::gil_scoped_release>())
        .def("unregister_mr", &Connection::unregister_mr, py::call_guard<py::gil_scoped_release>())
        .def(
            "allocate_rdma",
            [](Connection& c, const py::object& keys, int block_size, int hint) {
                std::vector<std::string_view> kv;
                keys_from_py(keys, kv);
                std::vector<RemoteBlock> out;
                {
                    py::gil_scoped_release rel;
                    if (c.allocate(kv, block_size, out, hint) != 0) out.clear();
                }
                return blocks_to_array(std::move(out));
            },
            py::arg("keys"), py::arg("block_size"), py::arg("hint") = Connection::kHintDefault,
            "Reserve pool blocks for keys; returns a structured array (rkey, gen, remote_addr), "
            "empty on failure.  hint = -2 allocates in the NVLS-replicated region")
        .def(
            "allocate_rdma_async",
            [](Connection& c, const std::vector<std::string>& keys, int block_size,
               py::function cb) {
                auto holder = std::make_shared<py::function>(std::move(cb));
                c.allocate_async(keys, block_size, [holder](std::vector<RemoteBlock> v) {
                    py::gil_scoped_acquire acq;
                    (*holder)(blocks_to_array(std::move(v)));
                    holder->release().dec_ref();
                });
            })
        .def(
            "w_rdma",
            [](Connection& c, const py::object& offsets, int block_size,
               const py::object& remote_blocks, uint64_t base_ptr, int device, uint64_t stream,
               uint64_t scale) {
                BlockSpan rb;
                OffsetSpan off;
                blocks_from_py(remote_blocks, rb);
                offsets_from_py(offsets, off);
                py::gil_scoped_release rel;
                return c.w_rdma(off.data, off.n, scale, block_size, rb.data, rb.n, base_ptr,
                                device, stream);
            },
            py::arg("offsets"), py::arg("block_size"), py::arg("remote_blocks"),
            py::arg("base_ptr"), py::arg("device") = -1, py::arg("stream") = 0,
            py::arg("scale") = 1)
        .def(
            "w_rdma_async",
            [](Connection& c, const py::object& offsets, int block_size,
               const py::object& remote_blocks, uint64_t base_ptr, py::function cb, int device,
               uint64_t stream, uint64_t scale) {
                BlockSpan rb;
                OffsetSpan off;
                blocks_from_py(remote_blocks, rb);
                offsets_from_py(offsets, off);
                std::vector<uint64_t> bytes(off.n);
                for (size_t i = 0; i < off.n; ++i) bytes[i] = off.data[i] * scale;
                auto holder = std::make_shared<py::function>(std::move(cb));
                py::gil_scoped_release rel;
                return c.w_rdma_async(bytes, block_size, rb.data, rb.n, base_ptr, device, stream,
                                      [holder](int status) {
                                          py::gil_scoped_acquire acq;
                                          (*holder)(status);
                                          holder->release().dec_ref();
                                      });
            },
            py::arg("offsets"), py::arg("block_size"), py::arg("remote_blocks"),
            py::arg("base_ptr"), py::arg("callback"), py::arg("device") = -1,
            py::arg("stream") = 0, py::arg("scale") = 1)
        .def(
            "r_rdma",
            [](Connection& c, const py::object& blocks, int block_size, uint64_t base_ptr,
               int device, uint64_t stream, uint64_t scale) {
                std::vector<KeyOffset> kb;
                blocks_list_from_py(blocks, scale, kb);
                const PackedKeys packed = t_arena.packed();  // this thread's arena: still ours
                py::gil_scoped_release rel;
                return c.r_rdma(kb, block_size, base_ptr, device, stream, nullptr, &packed);
            },
            py::arg("blocks"), py::arg("block_size"), py::arg("base_ptr"),
            py::arg("device") = -1, py::arg("stream") = 0, py::arg("scale") = 1)
        .def(
            "r_rdma_multi",
            [](Connection& c, const py::object& blocks, int block_size,
               const std::vector<uint64_t>& bases, int device, uint64_t stream, uint64_t scale) {
                std::vector<KeyOffset> kb;
                blocks_list_from_py(blocks, scale, kb);
                py::gil_scoped_release rel;
                return c.r_rdma_multi(kb, block_size, bases, device, stream);
            },
            py::arg("blocks"), py::arg("block_size"), py::arg("bases"), py::arg("device") = -1,
            py::arg("stream") = 0, py::arg("scale") = 1)
        .def(
            "r_rdma_hnd",
            [](Connection& c, const py::object& blocks, int tokens, int heads, int dim,
               int elem_size, uint64_t base_ptr, uint64_t num_pages, int device, uint64_t stream) {
                std::vector<KeyOffset> kb;
                blocks_list_from_py(blocks, 1, kb);  // (key, page index)
                py::gil_scoped_release rel;
                return c.r_rdma_hnd(kb, tokens, heads, dim, elem_size, base_ptr, num_pages, device,
                                    stream);
            },
            py::arg("blocks"), py::arg("tokens"), py::arg("heads"), py::arg("dim"),
            py::arg("elem_size"), py::arg("base_ptr"), py::arg("num_pages"),
            py::arg("device") = -1, py::arg("stream") = 0)
        .def(
            "r_rdma_async",
            [](Connection& c, const py::object& blocks, int block_size, uint64_t base_ptr,
               py::function cb, int device, uint64_t stream, uint64_t scale) {
                std::vector<KeyOffset> kb;
                blocks_list_from_py(blocks, scale, kb);
                auto holder = std::make_shared<py::function>(std::move(cb));
                py::gil_scoped_release rel;
                return c.r_rdma_async(kb, block_size, base_ptr, device, stream,
                                      [holder](int status) {
                                          py::gil_scoped_acquire acq;
                                          (*holder)(status);
                                          holder->release().dec_ref();
                                      });
            },
            py::arg("blocks"), py::arg("block_size"), py::arg("base_ptr"), py::arg("callback"),
            py::arg("device") = -1, py::arg("stream") = 0, py::arg("scale") = 1)
        .def(
            "w_rdma_fp8",
            [](Connection& c, const py::object& offsets, int elems, const py::object& remote_blocks,
               uint64_t base_ptr, int device, uint64_t stream, uint64_t scale) {
                BlockSpan rb;
                OffsetSpan off;
                blocks_from_py(remote_blocks, rb);
                offsets_from_py(offsets, off);
                py::gil_scoped_release rel;
                return c.w_rdma_fp8(off.data, off.n, scale, elems, rb.data, rb.n, base_ptr, device,
                                    stream);
            },
            py::arg("offsets"), py::arg("elems"), py::arg("remote_blocks"), py::arg("base_ptr"),
            py::arg("device") = -1, py::arg("stream") = 0, py::arg("scale") = 1)
        .def(
            "r_rdma_fp8",
            [](Connection& c, const py::object& blocks, int elems, uint64_t base_ptr, int device,
               uint64_t stream, uint64_t scale) {
                std::vector<KeyOffset> kb;
                blocks_list_from_py(blocks, scale, kb);
                py::gil_scoped_release rel;
                return c.r_rdma_fp8(kb, elems, base_ptr, device, stream);
            },
            py::arg("blocks"), py::arg("elems"), py::arg("base_ptr"), py::arg("device") = -1,
            py::arg("stream") = 0, py::arg("scale") = 1)
        .def(
            "w_rdma_gather",
            [](Connection& c, const std::vector<uint64_t>& part_base, uint32_t part_bytes,
               uint32_t elems, const py::object& offsets, const py::object& remote_blocks,
               int device, uint64_t stream, uint64_t scale, const std::vector<uint32_t>& rows,
               const py::object& piece_off, uint32_t pieces, const std::vector<uint32_t>& records,
               const std::vector<float>& scales, const py::object& rope) {
                BlockSpan rb;
                OffsetSpan off;
                blocks_from_py(remote_blocks, rb);
                offsets_from_py(offsets, off);
                std::vector<uint64_t> bytes(off.n);
                for (size_t i = 0; i < off.n; ++i) bytes[i] = off.data[i] * scale;
                const std::vector<uint64_t> table = piece_table(piece_off, off.n, pieces, scale);
                Connection::GatherSpec g =
                    gather_spec(part_base, part_bytes, elems, 0, rows, &table, pieces, records,
                                scales);
                kernels::RopeShift rs;
                if (parse_rope(rope, rs)) g.rope = &rs;
                py::gil_scoped_release rel;
                return c.w_rdma_gather(g, bytes.data(), bytes.size(), rb.data, rb.n, device, stream);
            },
            py::arg("part_base"), py::arg("part_bytes"), py::arg("elems"), py::arg("offsets"),
            py::arg("remote_blocks"), py::arg("device") = -1, py::arg("stream") = 0,
            py::arg("scale") = 1, py::arg("rows") = std::vector<uint32_t>{},
            py::arg("piece_off") = py::none(), py::arg("pieces") = 1,
            py::arg("records") = std::vector<uint32_t>{}, py::arg("scales") = std::vector<float>{},
            py::arg("rope") = py::none(),
            "gathered write: block i = part s at part_base[s] + offsets[i] * scale, s = 0..S-1; "
            "elems > 0: bf16 parts of elems elements, quantised into fp8 page s of block i, or "
            "with records = (latent, rope) into elems / (latent + rope) fp8 token records "
            "(with pieces > 1 and no rows: run t of pieces runs of whole tokens from "
            "part_base[s] + offset + piece_off[i * pieces + t]); "
            "rows = (rows, row_bytes, src_pitch, 0, dst_pitch[, slices, dst_slice_pitch]) filling "
            "each stored part: slice j of stored row r from part_base[s] + offset + r * "
            "dst_pitch + j * dst_slice_pitch; pieces > 1 (with rows): piece_off holds pieces "
            "offsets per block (times scale), and run t of rows / pieces rows comes from "
            "part_base[s] + offset + piece_off[i * pieces + t]; scales (one per part, elems > "
            "0, whole parts): the parts are elems bytes of e4m3 of those scales, stored verbatim "
            "as fp8 pages whose group scales are the part's; rope = (head_elems, rot_offset, "
            "rot_dim, interleaved, even_parts, cos, sin) (bf16 whole parts): the rotary pairs of "
            "every head of the rotating parts are turned by the table as they are stored")
        .def(
            "r_rdma_scatter",
            [](Connection& c, const std::vector<uint64_t>& part_base, uint32_t part_bytes,
               uint32_t elems, uint32_t first_part, const py::object& blocks, int device,
               uint64_t stream, uint64_t scale, const std::vector<uint32_t>& rows,
               Connection::ScatterReader* reader, uint32_t group_parts, const py::object& piece_off,
               uint32_t pieces, const std::vector<uint32_t>& records,
               const std::vector<float>& scales, const py::object& rope) {
                std::vector<KeyOffset> kb;
                blocks_list_from_py(blocks, scale, kb);
                const std::vector<uint64_t> table = piece_table(piece_off, kb.size(), pieces, scale);
                Connection::GatherSpec g = gather_spec(part_base, part_bytes, elems, first_part,
                                                       rows, &table, pieces, records, scales);
                kernels::RopeShift rs;
                if (parse_rope(rope, rs)) g.rope = &rs;
                g.reader = reader;
                g.group_parts = group_parts;
                py::gil_scoped_release rel;
                return c.r_rdma_scatter(g, kb, device, stream);
            },
            py::arg("part_base"), py::arg("part_bytes"), py::arg("elems"), py::arg("first_part"),
            py::arg("blocks"), py::arg("device") = -1, py::arg("stream") = 0,
            py::arg("scale") = 1, py::arg("rows") = std::vector<uint32_t>{},
            py::arg("reader") = py::none(), py::arg("group_parts") = 0,
            py::arg("piece_off") = py::none(), py::arg("pieces") = 1,
            py::arg("records") = std::vector<uint32_t>{}, py::arg("scales") = std::vector<float>{},
            py::arg("rope") = py::none(),
            "scattered read: stored part first_part + s of each block -> part_base[s] + offset; "
            "elems > 0: fp8 pages (or with records, token records) dequantised into bf16 parts "
            "of elems elements; rows = (rows, "
            "row_bytes, src_pitch, src_col, dst_pitch[, slices, dst_slice_pitch]): only those "
            "rows of each part, slice j of row r to part_base[s] + offset + r * dst_pitch + j * "
            "dst_slice_pitch; reader: a layered read whose parts are "
            "released in groups of group_parts (check reader.failed); pieces as for "
            "w_rdma_gather; scales (one per part): e4m3 parts, each stored group requantised to "
            "its part's scale (verbatim when the scales are equal); rope as for w_rdma_gather, "
            "turning the pairs as they land")
        .def(
            "wait_layered",
            [](Connection& c, const Connection::ScatterReader& r, uint32_t group, uint64_t stream) {
                std::string err;
                int rc;
                {
                    py::gil_scoped_release rel;
                    rc = c.wait_layered(r, group, stream, &err);
                }
                if (rc == -1) throw py::value_error(err);
                if (rc != 0) throw std::runtime_error(err);
            },
            py::arg("reader"), py::arg("group"), py::arg("stream"),
            "later work on `stream` waits on the GPU until `group` of the reader has landed; "
            "ValueError when refused (failed reader, group outside the read, connection closed "
            "since the read)")
        .def(
            "gather_writer",
            [](Connection& c, const py::object& remote_blocks, const py::object& offsets,
               uint32_t nparts, const py::object& piece_off, uint32_t pieces) {
                BlockSpan rb;
                OffsetSpan off;
                blocks_from_py(remote_blocks, rb);
                offsets_from_py(offsets, off);
                if (off.n != rb.n) throw std::invalid_argument("one offset per remote block");
                if (nparts < 1 || nparts > kernels::kGatherMaxParts)
                    throw std::invalid_argument("a block holds 1 to GATHER_MAX_PARTS parts");
                if (pieces < 1) throw std::invalid_argument("pieces must be at least 1");
                const std::vector<uint64_t> table = piece_table(piece_off, off.n, pieces, 1);
                py::gil_scoped_release rel;
                return c.gather_writer(rb.data, off.data, rb.n, nparts,
                                       pieces > 1 ? table.data() : nullptr, pieces);
            },
            py::arg("remote_blocks"), py::arg("offsets"), py::arg("nparts"),
            py::arg("piece_off") = py::none(), py::arg("pieces") = 1,
            "layered gathered writer over allocated blocks (offsets in elements); pieces > 1: "
            "piece_off (elements) as for w_rdma_gather, used by every call")
        .def(
            "w_rdma_layered",
            [](Connection& c, Connection::GatherWriter& w, const std::vector<uint64_t>& part_base,
               uint32_t part_bytes, uint32_t elems, uint32_t first_part, int device,
               uint64_t stream, uint64_t scale, const std::vector<uint32_t>& rows,
               const std::vector<uint32_t>& records, const std::vector<float>& scales,
               const py::object& rope) {
                Connection::GatherSpec g = gather_spec(
                    part_base, part_bytes, elems, first_part, rows, nullptr, 1, records, scales);
                kernels::RopeShift rs;
                if (parse_rope(rope, rs)) g.rope = &rs;
                py::gil_scoped_release rel;
                return c.write_layered(w, g, scale, device, stream);
            },
            py::arg("writer"), py::arg("part_base"), py::arg("part_bytes"), py::arg("elems"),
            py::arg("first_part"), py::arg("device") = -1, py::arg("stream") = 0,
            py::arg("scale") = 1, py::arg("rows") = std::vector<uint32_t>{},
            py::arg("records") = std::vector<uint32_t>{}, py::arg("scales") = std::vector<float>{},
            py::arg("rope") = py::none(),
            "layered write: stored part first_part + s of every block of the writer <- "
            "part_base[s] + offset * scale; elems > 0: fp8 parts of elems bf16 elements; rows, "
            "records, scales and rope as for w_rdma_gather (every call with scales or none, and "
            "with rope or none)")
        .def(
            "rw_local",
            [](Connection& c, const std::string& op, const py::object& blocks, int block_size,
               uint64_t base_ptr, int device, uint64_t stream, uint64_t scale) {
                std::vector<KeyOffset> kb;
                blocks_list_from_py(blocks, scale, kb);
                py::gil_scoped_release rel;
                return c.rw_local(op.empty() ? 0 : op[0], kb, block_size, base_ptr, device,
                                  stream);
            },
            py::arg("op"), py::arg("blocks"), py::arg("block_size"), py::arg("base_ptr"),
            py::arg("device") = -1, py::arg("stream") = 0, py::arg("scale") = 1)
        .def("set_copy_variant", &Connection::set_copy_variant)
        .def("set_max_ctas", &Connection::set_max_ctas)
        .def("set_pipe_geometry", &Connection::set_pipe_geometry, py::arg("stage_bytes"),
             py::arg("ring_bytes"))
        .def("set_device_lookup", &Connection::set_device_lookup)
        .def("set_streams", &Connection::set_streams)
        .def("device_lookup", &Connection::device_lookup)
        .def("server_has_hbm", &Connection::server_has_hbm)
        .def("server_evicts", &Connection::server_evicts)
        .def("index_incomplete", &Connection::index_incomplete)
        .def("last_error", &Connection::last_error)
        .def("segments",
             [](Connection& c) {
                 py::list l;
                 for (auto& s : c.segments()) l.append(segment_dict(s));
                 return l;
             })
        .def("stats", [](Connection& c) {
            const ClientStats s = c.stats();
            py::dict d;
            d["kernel_launches"] = s.kernel_launches;
            d["doorbell_ops"] = s.doorbell_ops;
            d["doorbell_launches"] = s.doorbell_launches;
            d["bytes_written"] = s.bytes_written;
            d["bytes_read"] = s.bytes_read;
            d["ctrl_requests"] = s.ctrl_requests;
            d["host_copies"] = s.host_copies;
            d["ns_build"] = s.ns_build;
            d["ns_streams"] = s.ns_streams;
            d["ns_launch"] = s.ns_launch;
            d["calls"] = s.calls;
            d["drains"] = s.drains;
            return d;
        });

    // ------------------------------------------------------------ server
    py::class_<Connection::GatherWriter, std::shared_ptr<Connection::GatherWriter>>(
        m, "GatherWriter")
        .def_property_readonly("complete", &Connection::GatherWriter::complete)
        .def_readonly("failed", &Connection::GatherWriter::failed)
        .def_readonly("nparts", &Connection::GatherWriter::nparts)
        .def_property_readonly("nblocks",
                               [](const Connection::GatherWriter& w) { return w.blocks.size(); })
        .def_property_readonly("written", [](const Connection::GatherWriter& w) {
            return std::vector<bool>(w.written.begin(), w.written.end());
        });
    py::class_<Connection::ScatterReader, std::shared_ptr<Connection::ScatterReader>>(
        m, "ScatterReader")
        .def(py::init<>())
        .def_readonly("groups", &Connection::ScatterReader::groups)
        .def_readonly("group_parts", &Connection::ScatterReader::group_parts)
        .def_readonly("seq", &Connection::ScatterReader::seq)
        .def_readonly("failed", &Connection::ScatterReader::failed)
        .def_property_readonly("flags", [](const Connection::ScatterReader& r) {
            return reinterpret_cast<uint64_t>(r.flags);
        });

    py::class_<Server, std::shared_ptr<Server>>(m, "Server")
        .def(py::init<const ServerConfig&>())
        .def(
            "start",
            [](Server& s) {
                std::string err;
                int rc;
                {
                    py::gil_scoped_release rel;
                    rc = s.start(&err);
                }
                if (rc != 0) throw std::runtime_error("server start failed: " + err);
                return s.port();
            })
        .def("stop", &Server::stop, py::call_guard<py::gil_scoped_release>())
        .def("port", &Server::port)
        .def("running", &Server::running)
        .def("kvmap_len", &Server::kvmap_len, py::call_guard<py::gil_scoped_release>())
        .def("purge", &Server::purge, py::call_guard<py::gil_scoped_release>())
        .def("inject_delay", &Server::inject_delay, py::arg("ms"), py::arg("count") = 1,
             "fault injection: stall the reactor `ms` before each of the next `count` requests")
        .def("inject_delay", &Server::inject_delay, py::arg("ms"), py::arg("count") = 1,
             "fault injection: stall the reactor `ms` before each of the next `count` requests")
        .def("inject_drop_after", &Server::inject_drop_after)
        .def(
            "dump",
            [](Server& s, const std::string& path) {
                std::string err;
                long n;
                {
                    py::gil_scoped_release rel;
                    n = s.dump(path, &err);
                }
                if (n < 0) throw std::runtime_error("dump failed: " + err);
                return n;
            },
            "Write every committed block to a checkpoint file; returns the block count")
        .def(
            "load",
            [](Server& s, const std::string& path) {
                std::string err;
                long n;
                {
                    py::gil_scoped_release rel;
                    n = s.load(path, &err);
                }
                if (n < 0) throw std::runtime_error("load failed: " + err);
                return n;
            },
            "Load a checkpoint file into the pool (existing keys win); returns blocks loaded")
        .def("stats", [](Server& s) { return stats_dict(s.stats()); })
        .def("index_table", &Server::index_table,
             "(address on the pool GPU, slots) of device-index shard 0; (0, 0) without one")
        .def("segments", [](Server& s) {
            py::list l;
            for (auto& i : s.segments()) l.append(segment_dict(i));
            return l;
        });

    m.def(
        "register_server",
        [](uint64_t /*loop_ptr*/, const ServerConfig& cfg) {
            std::lock_guard<std::mutex> lk(g_server_mu);
            if (g_server && g_server->running()) return 0;
            g_server = std::make_unique<Server>(cfg);
            std::string err;
            int rc;
            {
                py::gil_scoped_release rel;
                rc = g_server->start(&err);
            }
            if (rc != 0) {
                LOG_ERROR("register_server: %s", err.c_str());
                g_server.reset();
                return -1;
            }
            return 0;
        },
        "Start the process-wide store server (reactor thread); the event-loop pointer of the "
        "reference API is accepted and ignored");
    m.def("stop_server", [] {
        std::lock_guard<std::mutex> lk(g_server_mu);
        if (g_server) {
            py::gil_scoped_release rel;
            g_server->stop();
        }
        g_server.reset();
    });
    m.def("purge_kv_map", [] {
        std::lock_guard<std::mutex> lk(g_server_mu);
        if (g_server) g_server->purge();
    });
    m.def("get_kvmap_len", [] {
        std::lock_guard<std::mutex> lk(g_server_mu);
        return g_server ? g_server->kvmap_len() : size_t(0);
    });
    m.def("dump_kv_map", [](const std::string& path) {
        std::lock_guard<std::mutex> lk(g_server_mu);
        if (!g_server) throw std::runtime_error("no server in this process");
        std::string err;
        const long n = g_server->dump(path, &err);
        if (n < 0) throw std::runtime_error("dump failed: " + err);
        return n;
    });
    m.def("load_kv_map", [](const std::string& path) {
        std::lock_guard<std::mutex> lk(g_server_mu);
        if (!g_server) throw std::runtime_error("no server in this process");
        std::string err;
        const long n = g_server->load(path, &err);
        if (n < 0) throw std::runtime_error("load failed: " + err);
        return n;
    });
    m.def("server_stats", [] {
        std::lock_guard<std::mutex> lk(g_server_mu);
        return g_server ? stats_dict(g_server->stats()) : py::dict();
    });
    m.def("server_port", [] {
        std::lock_guard<std::mutex> lk(g_server_mu);
        return g_server ? g_server->port() : 0;
    });

    m.def("install_crash_handler", &install_crash_handler,
          "Print a backtrace on SIGSEGV/SIGBUS/SIGFPE/SIGABRT, then take the default action");
    m.def("log_msg", &log_msg);
    m.def("set_log_level", [](const std::string& l) { set_log_level(l); });
    m.def("cuda_available", &fabric::cuda_available);
    m.def(
        "enable_peer_access",
        [](int device, int peer) {
            int prev = -1, can = 0;
            cudaGetDevice(&prev);
            cudaDeviceCanAccessPeer(&can, device, peer);
            if (!can) return false;
            cudaSetDevice(device);
            const cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
            (void)cudaGetLastError();
            if (prev >= 0) cudaSetDevice(prev);
            return e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled;
        },
        "Let kernels running on `device` address memory of `peer` (single-process use)");
    m.def("cuda_device_count", &fabric::cuda_device_count);

    // ------------------------------------------------------------ fabric (NVLS)
    py::class_<fabric::NvlsProbe>(m, "NvlsProbe")
        .def_readonly("driver_ok", &fabric::NvlsProbe::driver_ok)
        .def_readonly("multicast_supported", &fabric::NvlsProbe::multicast_supported)
        .def_readonly("vmm_supported", &fabric::NvlsProbe::vmm_supported)
        .def_readonly("posix_fd_supported", &fabric::NvlsProbe::posix_fd_supported)
        .def_readonly("fabric_handle_supported", &fabric::NvlsProbe::fabric_handle_supported)
        .def_readonly("granularity", &fabric::NvlsProbe::granularity)
        .def_readonly("detail", &fabric::NvlsProbe::detail);
    m.def("nvls_probe", &fabric::nvls_probe, py::arg("device") = 0);
    py::class_<fabric::NvlsGroup, std::shared_ptr<fabric::NvlsGroup>>(m, "NvlsGroup")
        .def_static(
            "create",
            [](const std::vector<int>& devices, size_t bytes) {
                std::string err;
                auto g = fabric::NvlsGroup::create(devices, bytes, &err);
                if (!g) throw std::runtime_error("NVLS group: " + err);
                return g;
            },
            "Single-process multicast group over `devices` with `bytes` of replica per GPU")
        .def("mc_ptr", &fabric::NvlsGroup::mc_ptr, "multicast VA as seen from devices[i]")
        .def("uc_ptr", &fabric::NvlsGroup::uc_ptr, "local replica VA on devices[i]")
        .def("bytes", &fabric::NvlsGroup::bytes)
        .def("size", &fabric::NvlsGroup::size);

    // ------------------------------------------------------------ raw kernel launchers
    py::module_ k = m.def_submodule("kernels", "raw launchers of the sm_90a kernels");
    k.attr("COPY_AUTO") = int(kernels::kCopyAuto);
    k.attr("COPY_LDST") = int(kernels::kCopyLdSt);
    k.attr("COPY_TMA") = int(kernels::kCopyTma);
    k.attr("COPY_LDST256") = int(kernels::kCopyLdSt256);
    k.attr("STAT_MISS") = int(kernels::kStatMiss);
    k.attr("STAT_PUBLISH_FAIL") = int(kernels::kStatPublishFail);
    k.attr("STAT_MATCH") = int(kernels::kStatMatch);
    k.attr("STAT_STALE") = int(kernels::kStatStale);
    k.attr("INDEX_WAYS") = int(kernels::kIndexWays);
    k.attr("STAT_WORDS") = int(kernels::kStatWords);
    k.def(
        "kv_copy",
        [](uint64_t descs, uint32_t n, uint32_t bytes, int variant, int max_ctas, uint64_t stream,
           uint64_t recs, uint64_t table, uint64_t table_mask, uint64_t done, uint64_t status,
           uint64_t align_or, uint64_t trace, bool all_local, uint32_t debug,
           uint32_t stage_bytes, uint32_t ring_bytes, const std::vector<int64_t>& fan_delta,
           const ShardList& shards) {
            kernels::CopyLaunch L;
            L.shards = parse_shards(shards);
            L.stage_bytes = stage_bytes;
            L.ring_bytes = ring_bytes;
            if (!fan_delta.empty()) {
                if (fan_delta.size() > 4) throw std::runtime_error("at most 4 destinations");
                L.fan_n = int(fan_delta.size());
                for (size_t i = 0; i < fan_delta.size(); ++i) L.fan_delta[i] = fan_delta[i];
            }
            L.descs = as_ptr<const kernels::CopyDesc>(descs);
            L.n = n;
            L.bytes = bytes;
            L.align_or = align_or;
            L.recs = as_ptr<const kernels::IndexEntry>(recs);
            L.table = as_ptr<kernels::IndexBucket>(table);
            L.table_mask = table_mask;
            L.done = as_ptr<uint32_t>(done);
            L.status = as_ptr<uint32_t>(status);
            L.variant = variant;
            L.max_ctas = max_ctas;
            L.trace = as_ptr<unsigned long long>(trace);
            L.all_local = all_local;
            L.debug = debug;
            const cudaError_t e = kernels::launch_kv_copy(L, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("descs"), py::arg("n"), py::arg("bytes"), py::arg("variant") = 0,
        py::arg("max_ctas") = 0, py::arg("stream") = 0, py::arg("recs") = 0,
        py::arg("table") = 0, py::arg("table_mask") = 0, py::arg("done") = 0,
        py::arg("status") = 0, py::arg("align_or") = 0, py::arg("trace") = 0,
        py::arg("all_local") = false, py::arg("debug") = 0, py::arg("stage_bytes") = 0,
        py::arg("ring_bytes") = 0, py::arg("fan_delta") = std::vector<int64_t>(),
        py::arg("shards") = ShardList(),
        "shards: (table, bucket mask) of index shards 1, 2, ... for the publish; a key is "
        "published in the table its fingerprint selects (index_shard_of)");
    k.attr("GATHER_MAX_PARTS") = int(kernels::kGatherMaxParts);
    k.def(
        "kv_gather",
        [](uint64_t descs, uint32_t n, const std::vector<uint64_t>& part_base, uint32_t part_bytes,
           uint32_t first_part, bool write, int max_ctas, uint64_t stream, uint64_t recs,
           uint64_t table, uint64_t table_mask, uint64_t done, uint64_t status, uint64_t align_or,
           uint32_t stage_bytes, uint32_t ring_bytes, uint64_t layer_state, uint32_t layer_parts,
           bool layer_claim, uint64_t group_flags, uint64_t group_counters, uint32_t group_seq,
           uint32_t group_parts, const std::vector<uint32_t>& rows, uint64_t piece_off,
           uint32_t pieces, const ShardList& shards, const py::object& rope) {
            if (part_base.empty() || part_base.size() > kernels::kGatherMaxParts)
                throw std::runtime_error("kv_gather: 1 to GATHER_MAX_PARTS parts");
            kernels::RopeShift rs;
            const bool has_rope = parse_rope(rope, rs);
            const kernels::IndexShards sh = parse_shards(shards);
            if (layer_state && first_part + part_base.size() > layer_parts)
                throw std::runtime_error("kv_gather: first_part + parts > layer_parts");
            if (group_flags && (write || !group_counters || !group_parts ||
                                part_base.size() % group_parts))
                throw std::runtime_error(
                    "kv_gather: a layered read needs counters and group_parts dividing the parts");
            kernels::GatherLaunch G;
            G.descs = as_ptr<const kernels::CopyDesc>(descs);
            G.n = n;
            G.write = write;
            G.part_base = part_base.data();
            G.nparts = uint32_t(part_base.size());
            G.part_bytes = part_bytes;
            G.first_part = first_part;
            G.align_or = align_or;
            G.recs = as_ptr<const kernels::IndexEntry>(recs);
            G.table = as_ptr<kernels::IndexBucket>(table);
            G.table_mask = table_mask;
            G.done = as_ptr<uint32_t>(done);
            G.status = as_ptr<uint32_t>(status);
            G.max_ctas = max_ctas;
            G.stage_bytes = stage_bytes;
            G.ring_bytes = ring_bytes;
            G.layer_state = as_ptr<uint32_t>(layer_state);
            G.layer_parts = layer_parts;
            G.layer_claim = layer_claim;
            G.group_flags = as_ptr<uint32_t>(group_flags);
            G.group_counters = as_ptr<uint32_t>(group_counters);
            G.group_seq = group_seq;
            G.group_parts = group_parts;
            if (!parse_rows(rows, pieces, G.rows))
                throw std::runtime_error("kv_gather: rows is 5 or 7 values");
            G.piece_off = as_ptr<const uint64_t>(piece_off);
            G.shards = sh;
            G.rope = has_rope ? &rs : nullptr;
            const cudaError_t e = kernels::launch_kv_gather(G, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("descs"), py::arg("n"), py::arg("part_base"), py::arg("part_bytes"),
        py::arg("first_part") = 0, py::arg("write") = true, py::arg("max_ctas") = 0,
        py::arg("stream") = 0, py::arg("recs") = 0, py::arg("table") = 0,
        py::arg("table_mask") = 0, py::arg("done") = 0, py::arg("status") = 0,
        py::arg("align_or") = 0, py::arg("stage_bytes") = 0, py::arg("ring_bytes") = 0,
        py::arg("layer_state") = 0, py::arg("layer_parts") = 0, py::arg("layer_claim") = false,
        py::arg("group_flags") = 0, py::arg("group_counters") = 0, py::arg("group_seq") = 0,
        py::arg("group_parts") = 0, py::arg("rows") = std::vector<uint32_t>{},
        py::arg("piece_off") = 0, py::arg("pieces") = 1, py::arg("shards") = ShardList(),
        py::arg("rope") = py::none(),
        "gathered blocks: descs[i] = write {local byte offset, block address} / read {block "
        "address or 0, local byte offset}; part s of block i at part_base[s] + local offset is "
        "stored part first_part + s.  layer_state (3 zeroed u32 per block, kept across the "
        "launches of one layered write): the block is published by the launch that lands the "
        "last of its layer_parts parts; layer_claim: this launch claims the index ways.  "
        "group_flags (reads): a layered read that stores group_seq to group_flags[g] once "
        "group g (group_parts parts of every block) has landed; group_counters: one zeroed "
        "u32 per group.  rows (5 or 7 values): a row-sliced read, or a write whose rows fill "
        "each stored part.  pieces > 1 (with rows): piece_off is the device address of n * "
        "pieces byte offsets, and run t of block i's rows / pieces rows is at part_base[s] + "
        "local offset + piece_off[i * pieces + t].  shards as for kv_copy.  rope = (head_elems, "
        "rot_offset, rot_dim, interleaved, even_parts, cos, sin): whole bf16 parts whose rotary "
        "pairs are turned as they move (kv_write_rope_gather, kv_read_rope_scatter; a table of "
        "(1, 0) pairs copies verbatim)");
    k.def(
        "kv_gather_fp8",
        [](uint64_t descs, uint32_t n, const std::vector<uint64_t>& part_base, uint32_t elems,
           uint32_t first_part, bool write, int variant, int max_ctas, uint64_t stream,
           uint64_t recs, uint64_t table, uint64_t table_mask, uint64_t done, uint64_t status,
           uint64_t align_or, uint64_t layer_state, uint32_t layer_parts, bool layer_claim,
           uint64_t group_flags, uint64_t group_counters, uint32_t group_seq,
           uint32_t group_parts, const std::vector<uint32_t>& rows, uint64_t piece_off,
           uint32_t pieces, const std::vector<uint32_t>& records, const std::vector<float>& scales) {
            if (part_base.empty() || part_base.size() > kernels::kGatherMaxParts)
                throw std::runtime_error("kv_gather_fp8: 1 to GATHER_MAX_PARTS parts");
            if (!scales.empty() && scales.size() != part_base.size())
                throw std::runtime_error("kv_gather_fp8: one scale per part");
            if (layer_state && first_part + part_base.size() > layer_parts)
                throw std::runtime_error("kv_gather_fp8: first_part + parts > layer_parts");
            if (group_flags && (write || !group_counters || !group_parts ||
                                part_base.size() % group_parts))
                throw std::runtime_error("kv_gather_fp8: a layered read needs counters and "
                                         "group_parts dividing the parts");
            kernels::GatherLaunch G;
            G.descs = as_ptr<const kernels::CopyDesc>(descs);
            G.n = n;
            G.write = write;
            G.part_base = part_base.data();
            G.nparts = uint32_t(part_base.size());
            G.first_part = first_part;
            G.align_or = align_or;
            G.recs = as_ptr<const kernels::IndexEntry>(recs);
            G.table = as_ptr<kernels::IndexBucket>(table);
            G.table_mask = table_mask;
            G.done = as_ptr<uint32_t>(done);
            G.status = as_ptr<uint32_t>(status);
            G.max_ctas = max_ctas;
            G.layer_state = as_ptr<uint32_t>(layer_state);
            G.layer_parts = layer_parts;
            G.layer_claim = layer_claim;
            G.group_flags = as_ptr<uint32_t>(group_flags);
            G.group_counters = as_ptr<uint32_t>(group_counters);
            G.group_seq = group_seq;
            G.group_parts = group_parts;
            if (!parse_rows(rows, pieces, G.rows))
                throw std::runtime_error("kv_gather_fp8: rows is 5 or 7 values");
            if (!rows.empty()) G.part_bytes = 2 * elems;  // bytes of the parts' bf16 view
            G.piece_off = as_ptr<const uint64_t>(piece_off);
            G.records = parse_records(records);
            G.part_scale = scales.empty() ? nullptr : scales.data();
            const cudaError_t e =
                kernels::launch_kv_gather_fp8(G, elems, variant, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("descs"), py::arg("n"), py::arg("part_base"), py::arg("elems"),
        py::arg("first_part") = 0, py::arg("write") = true, py::arg("variant") = 0,
        py::arg("max_ctas") = 0, py::arg("stream") = 0, py::arg("recs") = 0, py::arg("table") = 0,
        py::arg("table_mask") = 0, py::arg("done") = 0, py::arg("status") = 0,
        py::arg("align_or") = 0, py::arg("layer_state") = 0, py::arg("layer_parts") = 0,
        py::arg("layer_claim") = false, py::arg("group_flags") = 0, py::arg("group_counters") = 0,
        py::arg("group_seq") = 0, py::arg("group_parts") = 0,
        py::arg("rows") = std::vector<uint32_t>{}, py::arg("piece_off") = 0, py::arg("pieces") = 1,
        py::arg("records") = std::vector<uint32_t>{}, py::arg("scales") = std::vector<float>{},
        "gathered fp8 blocks: descs as for kv_gather; records = (latent, rope): every part is "
        "elems / (latent + rope) bf16 tokens stored as fp8 token records (kv_write_fp8_records, "
        "kv_read_fp8_records; no rows, any variant; with pieces > 1 and piece_off, run t of "
        "the elems / (latent + rope) / pieces tokens of each part at its local offset + "
        "piece_off[i * pieces + t]: kv_{write,read}_fp8_records_pieces); pieces as for "
        "kv_gather; part s (elems bf16 elements at "
        "part_base[s] + local offset) <-> fp8 page first_part + s of the block; layer_* and "
        "group_* as for kv_gather (a layered read always runs the ld/st kernel); rows as for "
        "kv_gather, in bytes of the parts' bf16 view: a read dequantises those rows of each "
        "fp8 page (kv_read_fp8_rows), a write quantises stored pages whose rows it loads from "
        "the strided parts (kv_write_fp8_rows); scales (one per part): every part is elems "
        "bytes of e4m3 of that scale (kv_write_e4m3_gather, kv_read_e4m3_scatter; whole parts, "
        "any variant): a write keeps the bytes with every group scale the part's, a read "
        "requantises each stored group to it");
    k.def(
        "stream_wait_value",
        [](uint64_t addr, uint32_t value, uint64_t stream) {
            const cudaError_t e = kernels::stream_wait_geq(as_ptr<const uint32_t>(addr), value,
                                                           as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("addr"), py::arg("value"), py::arg("stream"),
        "later work on `stream` waits on the GPU until the u32 at `addr` is >= value");
    k.def(
        "kv_pipe_mcast",
        [](uint64_t descs, uint32_t n, uint32_t bytes, const std::vector<int64_t>& delta,
           int max_clusters, uint64_t stream, uint64_t status, uint32_t stage_bytes,
           uint32_t ring_bytes) {
            kernels::McastLaunch M;
            M.descs = as_ptr<const kernels::CopyDesc>(descs);
            M.n = n;
            M.bytes = bytes;
            M.ndst = int(delta.size());
            for (size_t i = 0; i < delta.size() && i < 4; ++i) M.delta[i] = delta[i];
            M.status = as_ptr<uint32_t>(status);
            M.src_local = true;  // raw launcher: the caller vouches for local sources
            M.max_clusters = max_clusters;
            M.stage_bytes = stage_bytes;
            M.ring_bytes = ring_bytes;
            const cudaError_t e = kernels::launch_kv_pipe_mcast(M, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("descs"), py::arg("n"), py::arg("bytes"), py::arg("delta"),
        py::arg("max_clusters") = 0, py::arg("stream") = 0, py::arg("status") = 0,
        py::arg("stage_bytes") = 0, py::arg("ring_bytes") = 0,
        "one pool block -> 2 or 4 destinations through a thread-block cluster (TMA multicast)");
    k.def(
        "kv_pipe_hnd",
        [](uint64_t descs, uint32_t n, uint32_t tokens, uint32_t heads, uint32_t dim,
           uint32_t elem_size, uint64_t dst_base, uint32_t num_pages, int max_ctas, uint64_t stream,
           uint64_t status, uint32_t stage_bytes, uint32_t ring_bytes) {
            kernels::HndLaunch H;
            H.descs = as_ptr<const kernels::CopyDesc>(descs);
            H.n = n;
            H.tokens = tokens;
            H.heads = heads;
            H.dim = dim;
            H.elem_size = elem_size;
            H.dst_base = dst_base;
            H.num_pages = num_pages;
            H.max_ctas = max_ctas;
            H.status = as_ptr<uint32_t>(status);
            H.stage_bytes = stage_bytes;
            H.ring_bytes = ring_bytes;
            const cudaError_t e = kernels::launch_kv_pipe_hnd(H, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("descs"), py::arg("n"), py::arg("tokens"), py::arg("heads"), py::arg("dim"),
        py::arg("elem_size"), py::arg("dst_base"), py::arg("num_pages"), py::arg("max_ctas") = 0,
        py::arg("stream") = 0, py::arg("status") = 0, py::arg("stage_bytes") = 0,
        py::arg("ring_bytes") = 0,
        "token-major pages -> head-major paged KV cache; transposition by a 4-D TMA tensor store");
    k.def(
        "index_lookup",
        [](uint64_t key_bytes, uint64_t key_off, uint64_t key_len, uint32_t n, uint64_t table,
           uint64_t table_mask, const std::vector<uint64_t>& seg_base, uint64_t out_descs,
           uint64_t dst_off, uint64_t dst_base, uint32_t need_bytes, uint64_t present,
           uint64_t status, uint64_t ticket, bool want_match, uint64_t stream,
           uint64_t found_at, bool accept_claimed, const ShardList& shards) {
            kernels::LookupLaunch Q;
            Q.shards = parse_shards(shards);
            set_segments(Q, seg_base);
            Q.accept_claimed = accept_claimed;
            Q.found_at = as_ptr<kernels::LookupLaunch::FoundAt>(found_at);
            Q.key_bytes = as_ptr<const uint8_t>(key_bytes);
            Q.key_off = as_ptr<const uint32_t>(key_off);
            Q.key_len = as_ptr<const uint32_t>(key_len);
            Q.n = n;
            Q.table = as_ptr<const kernels::IndexBucket>(table);
            Q.table_mask = table_mask;
            Q.out_descs = as_ptr<kernels::CopyDesc>(out_descs);
            Q.dst_off = as_ptr<const uint64_t>(dst_off);
            Q.dst_base = dst_base;
            Q.need_bytes = need_bytes;
            Q.present = as_ptr<uint32_t>(present);
            Q.status = as_ptr<uint32_t>(status);
            Q.ticket = as_ptr<uint32_t>(ticket);
            Q.want_match = want_match;
            const cudaError_t e = kernels::launch_index_lookup(Q, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("key_bytes"), py::arg("key_off"), py::arg("key_len"), py::arg("n"),
        py::arg("table"), py::arg("table_mask"), py::arg("seg_base") = std::vector<uint64_t>(),
        py::arg("out_descs") = 0, py::arg("dst_off") = 0, py::arg("dst_base") = 0,
        py::arg("need_bytes") = 0, py::arg("present") = 0, py::arg("status") = 0,
        py::arg("ticket") = 0, py::arg("want_match") = false, py::arg("stream") = 0,
        py::arg("found_at") = 0, py::arg("accept_claimed") = false,
        py::arg("shards") = ShardList(),
        "shards as for kv_copy: found_at slot ids carry the shard in their top 3 bits");
    k.def(
        "index_validate",
        [](uint64_t found_at, uint32_t n, uint64_t table, uint64_t status, uint64_t stream,
           const ShardList& shards) {
            kernels::ValidateLaunch V;
            V.shards = parse_shards(shards);
            V.found_at = as_ptr<const kernels::LookupLaunch::FoundAt>(found_at);
            V.n = n;
            V.table = as_ptr<const kernels::IndexBucket>(table);
            V.status = as_ptr<uint32_t>(status);
            const cudaError_t e = kernels::launch_index_validate(V, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("found_at"), py::arg("n"), py::arg("table"), py::arg("status"),
        py::arg("stream") = 0, py::arg("shards") = ShardList(),
        "shards: the tables index_lookup resolved found_at in (as for kv_copy)");
    k.def(
        "read_fused",
        [](uint64_t key_bytes, uint64_t key_off, uint64_t key_len, uint32_t n, uint64_t table,
           uint64_t table_mask, const std::vector<uint64_t>& seg_base, uint64_t dst_base,
           uint64_t dst_off, uint32_t bytes, uint64_t align_or, uint64_t status, int max_ctas,
           bool validate, int variant, uint32_t stage_bytes, uint32_t ring_bytes, uint64_t stream,
           const ShardList& shards, uint32_t elems, const std::vector<uint64_t>& part_base,
           uint32_t part_bytes, uint32_t first_part) {
            kernels::ReadFusedLaunch R;
            R.shards = parse_shards(shards);
            set_segments(R, seg_base);
            if (validate && !status)
                throw py::value_error("read_fused: validate counts into a status array");
            if (elems && !part_base.empty())
                throw py::value_error("read_fused: fp8 pages or gathered parts, not both");
            R.key_bytes = as_ptr<const uint8_t>(key_bytes);
            R.key_off = as_ptr<const uint32_t>(key_off);
            R.key_len = as_ptr<const uint32_t>(key_len);
            R.n = n;
            R.table = as_ptr<const kernels::IndexBucket>(table);
            R.table_mask = table_mask;
            R.dst_base = dst_base;
            R.dst_off = as_ptr<const uint64_t>(dst_off);
            R.bytes = bytes;
            R.align_or = align_or;
            R.status = as_ptr<uint32_t>(status);
            R.max_ctas = max_ctas;
            R.validate = validate;
            R.variant = variant;
            R.stage_bytes = stage_bytes;
            R.ring_bytes = ring_bytes;
            const auto s = as_ptr<CUstream_st>(stream);
            cudaError_t e;
            if (!part_base.empty()) {
                kernels::GatherLaunch G;
                G.n = n;
                G.write = false;
                G.part_base = part_base.data();
                G.nparts = uint32_t(part_base.size());
                G.part_bytes = part_bytes;
                G.first_part = first_part;
                G.align_or = align_or;
                for (const uint64_t b : part_base) G.align_or |= b;
                G.status = R.status;
                G.max_ctas = max_ctas;
                if (part_base.size() > kernels::kGatherMaxParts ||
                    !kernels::scatter_read_fused_supported(R, G) ||
                    (uint64_t(first_part) + G.nparts) * part_bytes > 0xffffffffull ||
                    uint64_t(n) * G.nparts > 0x7fffffffull)
                    throw py::value_error(
                        "read_fused: gathered parts need 1 to GATHER_MAX_PARTS 16-byte aligned "
                        "parts of a nonzero multiple of 16 bytes, blocks within 2^32 bytes, and at "
                        "least as many blocks as CTAs");
                e = kernels::launch_kv_pipe_scatter_read(R, G, s);
            } else if (elems) {
                if (!kernels::fp8_read_fused_supported(R, elems))
                    throw py::value_error("read_fused: fp8 pages need a multiple of 512 "
                                          "elements and 16-byte aligned destinations");
                e = kernels::launch_kv_fp8_read_fused(R, elems, s);
            } else {
                e = kernels::launch_kv_read_fused(R, s);
            }
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("key_bytes"), py::arg("key_off"), py::arg("key_len"), py::arg("n"),
        py::arg("table"), py::arg("table_mask"), py::arg("seg_base"), py::arg("dst_base"),
        py::arg("dst_off"), py::arg("bytes"), py::arg("align_or") = 0, py::arg("status") = 0,
        py::arg("max_ctas") = 0, py::arg("validate") = true, py::arg("variant") = 0,
        py::arg("stage_bytes") = 0, py::arg("ring_bytes") = 0, py::arg("stream") = 0,
        py::arg("shards") = ShardList(), py::arg("elems") = 0,
        py::arg("part_base") = std::vector<uint64_t>(), py::arg("part_bytes") = 0,
        py::arg("first_part") = 0,
        "read_cache through the device index in one launch: key i (packed as for index_lookup) "
        "is resolved and its pool page of `bytes` lands at dst_base + dst_off[i] "
        "(kv_read_fused, or kv_pipe_read by variant and alignment).  elems > 0: fp8 pages "
        "dequantised to bf16 (kv_fp8_pipe).  part_base: gathered blocks, stored part "
        "first_part + s of part_bytes landing at part_base[s] + dst_off[i] "
        "(kv_pipe_scatter_read).  A miss is counted once per block in status[STAT_MISS]; "
        "validate re-checks every entry after its copy.  shards as for kv_copy");
    k.def(
        "index_erase",
        [](uint64_t recs, uint32_t n, uint64_t table, uint64_t table_mask, uint64_t stream) {
            kernels::EraseLaunch E;
            E.recs = as_ptr<const kernels::EraseRec>(recs);
            E.n = n;
            E.table = as_ptr<kernels::IndexBucket>(table);
            E.table_mask = table_mask;
            const cudaError_t e = kernels::launch_index_erase(E, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("recs"), py::arg("n"), py::arg("table"), py::arg("table_mask"),
        py::arg("stream") = 0);
    auto fp8 = [](bool write) {
        return [write](uint64_t descs, uint32_t n, uint32_t elems, uint32_t group, int max_ctas,
                       uint64_t stream, uint64_t recs, uint64_t table, uint64_t table_mask,
                       uint64_t done, uint64_t status, int variant, uint64_t align_or) {
            kernels::Fp8Launch L;
            L.variant = variant;
            L.aligned16 = (align_or & 15) == 0;
            L.descs = as_ptr<const kernels::CopyDesc>(descs);
            L.n = n;
            L.elems = elems;
            L.group = group;
            L.recs = as_ptr<const kernels::IndexEntry>(recs);
            L.table = as_ptr<kernels::IndexBucket>(table);
            L.table_mask = table_mask;
            L.done = as_ptr<uint32_t>(done);
            L.status = as_ptr<uint32_t>(status);
            L.max_ctas = max_ctas;
            const cudaError_t e = write
                                      ? kernels::launch_kv_write_fp8(L, as_ptr<CUstream_st>(stream))
                                      : kernels::launch_kv_read_fp8(L, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        };
    };
    k.def("kv_write_fp8", fp8(true), py::arg("descs"), py::arg("n"), py::arg("elems"),
          py::arg("group") = 128, py::arg("max_ctas") = 0, py::arg("stream") = 0,
          py::arg("recs") = 0, py::arg("table") = 0, py::arg("table_mask") = 0,
          py::arg("done") = 0, py::arg("status") = 0, py::arg("variant") = 0,
          py::arg("align_or") = 0);
    k.def("kv_read_fp8", fp8(false), py::arg("descs"), py::arg("n"), py::arg("elems"),
          py::arg("group") = 128, py::arg("max_ctas") = 0, py::arg("stream") = 0,
          py::arg("recs") = 0, py::arg("table") = 0, py::arg("table_mask") = 0,
          py::arg("done") = 0, py::arg("status") = 0, py::arg("variant") = 0,
          py::arg("align_or") = 0);
    k.def("fp8_block_bytes", &kernels::fp8_block_bytes);
    k.def("fp8_gather_bytes", &kernels::fp8_gather_bytes, py::arg("nparts"), py::arg("elems"),
          "bytes of nparts fp8 pages of elems elements end to end (a gathered fp8 block)");
    k.def(
        "fp8_records_bytes",
        [](uint32_t nparts, uint32_t elems, uint32_t latent, uint32_t rope) {
            return kernels::fp8_records_bytes(nparts, elems, kernels::Fp8Records{latent, rope});
        },
        py::arg("nparts"), py::arg("elems"), py::arg("latent"), py::arg("rope"),
        "bytes of a gathered block of nparts parts of elems bf16 elements stored as fp8 token "
        "records of latent + rope elements");
    k.def(
        "kv_bcast_nvls",
        [](uint64_t descs, uint32_t n, uint32_t bytes, int max_ctas, uint64_t stream,
           uint64_t flags_mc) {
            kernels::BcastLaunch L;
            L.descs = as_ptr<const kernels::CopyDesc>(descs);
            L.n = n;
            L.bytes = bytes;
            L.max_ctas = max_ctas;
            L.flags_mc = as_ptr<uint32_t>(flags_mc);
            const cudaError_t e = kernels::launch_kv_bcast_nvls(L, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("descs"), py::arg("n"), py::arg("bytes"), py::arg("max_ctas") = 0,
        py::arg("stream") = 0, py::arg("flags_mc") = 0);
    k.def("bcast_chunks_per_block", &kernels::bcast_chunks_per_block);
    k.def(
        "kv_read_when_ready",
        [](uint64_t descs, uint32_t n, uint32_t bytes, uint64_t flags_local, uint32_t ready_value,
           int max_ctas, uint64_t stream, uint64_t status) {
            kernels::ReadyLaunch L;
            L.descs = as_ptr<const kernels::CopyDesc>(descs);
            L.n = n;
            L.bytes = bytes;
            L.flags_local = as_ptr<const uint32_t>(flags_local);
            L.ready_value = ready_value;
            L.max_ctas = max_ctas;
            L.status = as_ptr<uint32_t>(status);
            const cudaError_t e = kernels::launch_kv_read_when_ready(L, as_ptr<CUstream_st>(stream));
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("descs"), py::arg("n"), py::arg("bytes"), py::arg("flags_local"),
        py::arg("ready_value"), py::arg("max_ctas") = 0, py::arg("stream") = 0,
        py::arg("status") = 0);

    // ------------------------------------------------------------ comparison baselines
    // The reference's data-movement pattern, reproduced for bench/ only (never on the
    // product path): one cudaMemcpyAsync per block on a stream + event created for the
    // request and destroyed after it (reference: src/infinistore.cpp:581-586,623-624,
    // 667-681,723-729,747-748).
    py::module_ bl = m.def_submodule("baseline", "library-call baselines for bench/");
    bl.def(
        "memcpy_blocks",
        [](const std::vector<uint64_t>& dst, const std::vector<uint64_t>& src, size_t bytes,
           bool fresh_stream, int device) {
            py::gil_scoped_release rel;
            int prev = -1;
            cudaGetDevice(&prev);
            if (device >= 0) cudaSetDevice(device);
            cudaStream_t st = nullptr;
            cudaEvent_t ev = nullptr;
            if (fresh_stream) {
                cudaStreamCreate(&st);
                cudaEventCreate(&ev);
            }
            cudaError_t e = cudaSuccess;
            for (size_t i = 0; i < dst.size() && e == cudaSuccess; ++i)
                e = cudaMemcpyAsync(as_ptr<void>(dst[i]), as_ptr<void>(src[i]), bytes,
                                    cudaMemcpyDefault, st);
            if (fresh_stream) {
                cudaEventRecord(ev, st);
                cudaEventSynchronize(ev);
                cudaEventDestroy(ev);
                cudaStreamDestroy(st);
            } else {
                cudaStreamSynchronize(st);
            }
            if (prev >= 0) cudaSetDevice(prev);
            if (e != cudaSuccess) throw std::runtime_error(cudaGetErrorString(e));
        },
        py::arg("dst"), py::arg("src"), py::arg("bytes"), py::arg("fresh_stream") = true,
        py::arg("device") = -1);

    // ------------------------------------------------------------ unit-test access to the core
    py::module_ t = m.def_submodule("testing", "wire codec, allocator and hash for unit tests");
    t.def("parse_blocks",
          [](const py::object& blocks) {
              std::vector<KeyOffset> kb;
              blocks_list_from_py(blocks, 1, kb);
              return kb.size();
          },
          "only the [(key, offset)] parsing step of the read calls (host-cost micro-benchmarks)");
    t.def("plan_chunks",
          [](uint32_t n, uint32_t units, uint32_t min_units, uint32_t max_units, uint32_t ctas) {
              const kernels::ChunkPlan p = kernels::plan_chunks(n, units, min_units, max_units, ctas);
              return py::make_tuple(p.chunk, p.cpb);
          },
          "work-item split of a batch for a persistent grid (kernels/balance.h)");
    t.def("index_shard_of", [](py::bytes key, uint32_t nshards) {
        const std::string k = key;
        const KeyHash h = hash_key(reinterpret_cast<const uint8_t*>(k.data()), k.size());
        return kernels::index_shard_of(h.h2, nshards);
    });
    t.def("hash_key", [](py::bytes key) {
        const std::string s = key;
        const KeyHash h = hash_key(reinterpret_cast<const uint8_t*>(s.data()), s.size());
        return py::make_tuple(h.h1, h.h2);
    });
    t.def("fd_pass_selftest", [] {
        // SCM_RIGHTS round trip over the abstract unix socket used for VMM handles: the
        // "server" hands out the read end of a pipe, the "client" reads through it.
        int p[2];
        if (pipe(p) != 0) return false;
        (void)!write(p[1], "hello", 5);
        fabric::FdServer srv;
        std::string err;
        const std::string name = "istore_b200_selftest_" + std::to_string(getpid());
        const int rd = p[0];
        bool ok = srv.start(name,
                            [rd](int req, std::vector<int>* fds, uint64_t* payload) {
                                fds->push_back(dup(rd));
                                *payload = uint64_t(req) * 2;
                                return true;
                            },
                            &err);
        std::vector<int> fds;
        uint64_t payload = 0;
        ok = ok && fabric::fd_request(name, 21, &fds, &payload, &err) && fds.size() == 1 &&
             payload == 42;
        char buf[8] = {0};
        ok = ok && read(fds[0], buf, 5) == 5 && std::memcmp(buf, "hello", 5) == 0;
        for (int fd : fds) close(fd);
        srv.stop();
        close(p[0]);
        close(p[1]);
        return ok;
    });
    t.def("header_size", [] { return sizeof(Header); });
    t.def("conn_info_size", [] { return sizeof(ConnInfo); });
    t.def("segment_info_size", [] { return sizeof(SegmentInfo); });
    t.def("encode_remote_meta",
          [](const std::vector<std::string>& keys, int block_size, uint32_t rkey,
             const std::vector<uint64_t>& addrs, const std::string& op, int hint) {
              std::vector<std::string_view> kv(keys.begin(), keys.end());
              std::vector<uint8_t> buf(remote_meta_bound(kv, addrs.size()));
              fb::Builder b(buf.data(), buf.size());
              encode_remote_meta(b, kv, block_size, rkey, addrs.data(), addrs.size(),
                                 op.empty() ? 0 : op[0], hint);
              return py::bytes(reinterpret_cast<const char*>(b.data()), b.size());
          },
          py::arg("keys"), py::arg("block_size"), py::arg("rkey"), py::arg("addrs"),
          py::arg("op"), py::arg("hint") = -1);
    t.def("decode_remote_meta", [](py::bytes data) {
        const std::string s = data;
        RemoteMetaRequest r = decode_remote_meta(s.data(), s.size());
        py::dict d;
        py::list keys;
        for (auto k : r.keys) keys.append(py::bytes(k.data(), k.size()));
        d["keys"] = keys;
        d["block_size"] = r.block_size;
        d["rkey"] = r.rkey;
        d["remote_addrs"] = r.remote_addrs;
        d["op"] = std::string(1, char(r.op));
        d["hint"] = r.hint;
        return d;
    });
    t.def("encode_allocate_response", [](const std::vector<std::tuple<uint32_t, uint32_t, uint64_t>>& blocks) {
        std::vector<RemoteBlock> rb;
        for (auto& b : blocks) rb.push_back(RemoteBlock{std::get<0>(b), std::get<1>(b), std::get<2>(b)});
        std::vector<uint8_t> buf((rb.size() * 16 + 64 + 7) & ~size_t(7));
        fb::Builder b(buf.data(), buf.size());
        encode_allocate_response(b, rb.data(), rb.size());
        return py::bytes(reinterpret_cast<const char*>(b.data()), b.size());
    });
    t.def("decode_allocate_response", [](py::bytes data) {
        const std::string s = data;
        return blocks_to_array(decode_allocate_response(s.data(), s.size()));
    });
    t.def("encode_local_meta",
          [](int device, py::bytes ipc, int block_size,
             const std::vector<std::pair<std::string, uint64_t>>& blocks) {
              const std::string ipc_s = ipc;
              std::vector<LocalBlock> lb;
              for (auto& b : blocks) lb.push_back(LocalBlock{b.first, b.second});
              std::vector<uint8_t> buf(local_meta_bound(lb) + ((ipc_s.size() + 15) & ~size_t(7)));
              fb::Builder b(buf.data(), buf.size());
              encode_local_meta(b, device, ipc_s, block_size, lb);
              return py::bytes(reinterpret_cast<const char*>(b.data()), b.size());
          });
    t.def("decode_local_meta", [](py::bytes data) {
        const std::string s = data;
        LocalMetaRequest r = decode_local_meta(s.data(), s.size());
        py::dict d;
        d["device"] = r.device;
        d["ipc_handle"] = py::bytes(r.ipc_handle.data(), r.ipc_handle.size());
        d["block_size"] = r.block_size;
        py::list blocks;
        for (auto& b : r.blocks)
            blocks.append(py::make_tuple(py::bytes(b.key.data(), b.key.size()), b.offset));
        d["blocks"] = blocks;
        return d;
    });
    t.def("encode_match_request", [](const std::vector<std::string>& keys) {
        std::vector<std::string_view> kv(keys.begin(), keys.end());
        std::vector<uint8_t> buf(remote_meta_bound(kv, 0));
        fb::Builder b(buf.data(), buf.size());
        encode_match_request(b, kv);
        return py::bytes(reinterpret_cast<const char*>(b.data()), b.size());
    });
    t.def("decode_match_request", [](py::bytes data) {
        const std::string s = data;
        py::list keys;
        for (auto k : decode_match_request(s.data(), s.size())) keys.append(py::bytes(k.data(), k.size()));
        return keys;
    });

    py::class_<MemoryPool>(t, "MemoryPool")
        .def(py::init<size_t, size_t, int>(), py::arg("pool_bytes"), py::arg("granule"),
             py::arg("device") = -1)
        .def("allocate", &MemoryPool::allocate)
        .def("allocate_n",
             [](MemoryPool& p, size_t size, size_t n) -> py::object {
                 std::vector<uint64_t> out;
                 if (!p.allocate_n(size, n, out)) return py::none();
                 return py::cast(out);
             })
        .def("deallocate", &MemoryPool::deallocate)
        .def("used_blocks", &MemoryPool::used_blocks)
        .def("total_blocks", &MemoryPool::total_blocks)
        .def("usage", &MemoryPool::usage);
    // staging-space reuse of a client device context (ctrl/staging.h), events as integers
    using Staging = StagingFifo<int64_t, 3>;
    py::class_<Staging>(t, "StagingFifo")
        .def(py::init<>())
        .def("place",
             [](Staging& f, int region, size_t bytes, size_t size) {
                 if (region < 0 || region >= 3 || size == 0 || bytes > size)
                     throw py::value_error("needs region in [0, 3) and bytes <= size");
                 py::list waited;
                 const uint64_t at = f.place(region, bytes, size, [&](int64_t ev) { waited.append(ev); });
                 return py::make_tuple(at, waited);
             })
        .def("push", &Staging::push)
        .def("retire_all", &Staging::retire_all)
        .def("take_free",
             [](Staging& f) -> py::object {
                 int64_t ev;
                 if (!f.take_free(&ev)) return py::none();
                 return py::int_(ev);
             })
        .def("in_flight", &Staging::in_flight);
    // flag slots of layered reads (ctrl/staging.h), events as integers
    using Readers = ReaderSlots<int64_t, kReaderSlots>;
    t.attr("READER_SLOTS") = kReaderSlots;
    py::class_<Readers>(t, "ReaderSlots")
        .def(py::init<>())
        .def("take",
             [](Readers& r) {
                 py::list waited;
                 const uint64_t seq = r.take([&](int64_t ev) { waited.append(ev); });
                 return py::make_tuple(seq, Readers::slot_of(seq), waited);
             })
        .def("launched", &Readers::launched)
        .def("retire_all", &Readers::retire_all);
    // layered reads' work-item numbering (kernels/launch_plan.h)
    t.def("layered_item", [](uint32_t item, uint32_t n, uint32_t gp, uint32_t cpp) {
        if (!n || !gp || !cpp) throw py::value_error("needs n, gp, cpp > 0");
        const kernels::LayeredItem it = kernels::layered_item(item, n, gp, cpp);
        return py::make_tuple(it.group, it.block, it.part, it.chunk);
    });
    t.def("cta_items", [](uint32_t lo, uint32_t hi, uint32_t first, uint32_t stride) {
        if (!stride || hi < lo) throw py::value_error("needs stride > 0 and lo <= hi");
        return kernels::cta_items(lo, hi, first, stride);
    });
    // row geometry (kernels::PartRows): where (slice, row) pair q of a part goes, where byte o
    // of a covered stored part comes from (with pieces: which piece, and where inside it), and
    // the geometry the plans and the connection accept
    using kernels::PartRows;
    t.def("slice_pair",
          [](uint32_t q, uint32_t rows, uint32_t row, uint32_t src_pitch, uint32_t src_col,
             uint32_t dst_pitch, uint32_t dst_slice_pitch) {
              if (!rows) throw py::value_error("needs rows > 0");
              const kernels::PairOffsets o =
                  PartRows{.rows = rows, .row_bytes = row, .src_pitch = src_pitch,
                           .src_col = src_col, .dst_pitch = dst_pitch,
                           .dst_slice_pitch = dst_slice_pitch}
                      .pair(q);
              return py::make_tuple(o.src, o.dst);
          },
          py::arg("q"), py::arg("rows"), py::arg("row"), py::arg("src_pitch"),
          py::arg("src_col"), py::arg("dst_pitch"), py::arg("dst_slice_pitch"));
    t.def("row_write_offset",
          [](uint32_t o, uint32_t row_bytes, uint32_t src_pitch, uint32_t dst_pitch,
             uint32_t dst_slice_pitch) {
              if (!row_bytes || !src_pitch) throw py::value_error("needs row_bytes, src_pitch > 0");
              return PartRows{.row_bytes = row_bytes, .src_pitch = src_pitch,
                              .dst_pitch = dst_pitch, .dst_slice_pitch = dst_slice_pitch}
                  .write_offset(o);
          },
          py::arg("o"), py::arg("row_bytes"), py::arg("src_pitch"), py::arg("dst_pitch"),
          py::arg("dst_slice_pitch"));
    t.def("row_write_covers",
          [](uint32_t row_bytes, uint32_t src_pitch, uint32_t src_col, uint32_t slices) {
              return PartRows{.row_bytes = row_bytes, .src_pitch = src_pitch, .src_col = src_col,
                              .slices = slices}
                  .covers();
          },
          py::arg("row_bytes"), py::arg("src_pitch"), py::arg("src_col"), py::arg("slices"));
    t.def("row_geometry_ok",
          [](uint32_t rows, uint32_t row_bytes, uint32_t src_pitch, uint32_t src_col,
             uint32_t dst_pitch, uint32_t slices, uint32_t dst_slice_pitch, uint64_t part_bytes,
             uint32_t pieces) {
              return PartRows{rows,   row_bytes,       src_pitch, src_col, dst_pitch,
                              slices, dst_slice_pitch, pieces}
                  .ok(part_bytes);
          },
          py::arg("rows"), py::arg("row_bytes"), py::arg("src_pitch"), py::arg("src_col"),
          py::arg("dst_pitch"), py::arg("slices"), py::arg("dst_slice_pitch"),
          py::arg("part_bytes"), py::arg("pieces") = 1);
    t.def("piece_pair",
          [](uint32_t q, uint32_t rows, uint32_t row, uint32_t src_pitch, uint32_t src_col,
             uint32_t dst_pitch, uint32_t dst_slice_pitch, uint32_t piece_rows) {
              if (!rows || !piece_rows) throw py::value_error("needs rows, piece_rows > 0");
              const kernels::PairOffsets o =
                  PartRows{.rows = rows, .row_bytes = row, .src_pitch = src_pitch,
                           .src_col = src_col, .dst_pitch = dst_pitch,
                           .dst_slice_pitch = dst_slice_pitch}
                      .pair(q, piece_rows);
              return py::make_tuple(o.src, o.dst, o.piece);
          },
          py::arg("q"), py::arg("rows"), py::arg("row"), py::arg("src_pitch"),
          py::arg("src_col"), py::arg("dst_pitch"), py::arg("dst_slice_pitch"),
          py::arg("piece_rows"));
    t.def("piece_write_offset",
          [](uint32_t o, uint32_t row_bytes, uint32_t src_pitch, uint32_t dst_pitch,
             uint32_t dst_slice_pitch, uint32_t piece_rows) {
              if (!row_bytes || !src_pitch || !piece_rows)
                  throw py::value_error("needs row_bytes, src_pitch, piece_rows > 0");
              const kernels::PairOffsets p =
                  PartRows{.row_bytes = row_bytes, .src_pitch = src_pitch,
                           .dst_pitch = dst_pitch, .dst_slice_pitch = dst_slice_pitch}
                      .write_offset(o, piece_rows);
              return py::make_tuple(p.piece, p.dst);
          },
          py::arg("o"), py::arg("row_bytes"), py::arg("src_pitch"), py::arg("dst_pitch"),
          py::arg("dst_slice_pitch"), py::arg("piece_rows"));
    t.attr("PIECE_RING_BYTES") = kPieceRingBytes;
    // how a read call is split into launches (ctrl/staging.h), with the client's limits
    t.attr("RING_BYTES") = kRingBytes;
    t.attr("MAX_BATCH") = kMaxBatch;
    t.def("gather_max_blocks", [](uint32_t nparts, uint32_t part_bytes) {
        if (nparts == 0 || part_bytes == 0) throw py::value_error("needs nparts, part_bytes > 0");
        return gather_max_blocks(kMaxBatch, nparts, part_bytes);
    });
    t.def("key_batches",
          [](const std::vector<size_t>& key_lens, size_t max_blocks) {
              if (max_blocks == 0) throw py::value_error("needs max_blocks > 0");
              py::list out;  // (keys, padded key bytes) of every launch
              for (size_t base = 0; base < key_lens.size();) {
                  const KeyBatch b = key_batch(key_lens.size() - base, max_blocks, kRingBytes / 2,
                                               [&](size_t i) { return key_lens[base + i]; });
                  out.append(py::make_tuple(b.n, b.key_bytes));
                  base += b.n;
              }
              return out;
          },
          py::arg("key_lens"), py::arg("max_blocks") = kMaxBatch);
    // which kernels a read through the device index runs (ctrl/read_plan.h)
    t.def("plan_device_read",
          [](size_t n, uint32_t block_bytes, uint32_t fp8_elems, bool gather, bool fp8_fused_ok,
             bool scatter_fused_ok, int copy_variant, bool all_local, bool all_remote, int max_ctas,
             int sm_count, bool layered, bool rows) {
              const DeviceReadPlan p = plan_device_read(DeviceReadIn{
                  n, block_bytes, fp8_elems, gather, fp8_fused_ok, scatter_fused_ok, copy_variant,
                  all_local, all_remote, max_ctas, sm_count, layered, rows});
              static const char* const kPaths[] = {"fused_copy",    "fused_fp8",
                                                   "fused_scatter", "lookup_copy",
                                                   "lookup_fp8",    "lookup_gather",
                                                   "lookup_gather_fp8"};
              py::dict d;
              d["path"] = kPaths[int(p.path)];
              d["variant"] = p.variant;
              d["grid_cap"] = p.grid_cap;
              return d;
          },
          py::arg("n"), py::arg("block_bytes"), py::arg("fp8_elems") = 0, py::arg("gather") = false,
          py::arg("fp8_fused_ok") = false, py::arg("scatter_fused_ok") = false,
          py::arg("copy_variant") = 0, py::arg("all_local") = false, py::arg("all_remote") = false,
          py::arg("max_ctas") = 0, py::arg("sm_count") = 132, py::arg("layered") = false,
          py::arg("rows") = false);
    // which kernel a page-mover launcher runs, its work split and grid (kernels/launch_plan.h);
    // the resident CTAs per SM of the ld/st kernels are the occupancy API's answer on a GPU
    const auto plan_dict = [](const kernels::LaunchPlan& p) {
        static const char* const kKernels[] = {"ldst1", "ldst16", "ldst32",  "ldst16_mc",
                                               "tma",   "tma4",   "ldst_fp8"};
        py::dict d;
        d["valid"] = p.valid;
        d["kernel"] = kKernels[int(p.kernel)];
        d["param"] = p.param;
        d["chunk"] = p.chunk;
        d["cpb"] = p.cpb;
        d["ctas"] = p.ctas;
        d["stage_bytes"] = p.geo.stage_bytes;
        d["stages"] = p.geo.stages;
        d["smem"] = p.geo.smem;
        return d;
    };
    static const kernels::CopyDesc kHostDescs[1] = {};  // plan_copy only asks whether there are any
    t.def("plan_copy",
          [plan_dict](uint32_t n, uint32_t bytes, uint64_t align_or, int variant, bool multicast,
                      bool descs_host, int max_ctas, uint32_t stage_bytes, uint32_t ring_bytes,
                      int sm_count, int resident16, int resident32) {
              kernels::CopyLaunch a;
              a.n = n;
              a.bytes = bytes;
              a.align_or = align_or;
              a.variant = variant;
              a.multicast = multicast;
              a.descs_host = descs_host ? kHostDescs : nullptr;
              a.max_ctas = max_ctas;
              a.stage_bytes = stage_bytes;
              a.ring_bytes = ring_bytes;
              return plan_dict(kernels::plan_copy(a, sm_count, {resident16, resident32}));
          },
          py::arg("n"), py::arg("bytes"), py::arg("align_or") = 0, py::arg("variant") = 0,
          py::arg("multicast") = false, py::arg("descs_host") = false, py::arg("max_ctas") = 0,
          py::arg("stage_bytes") = 0, py::arg("ring_bytes") = 0, py::arg("sm_count") = 132,
          py::arg("resident16") = 1, py::arg("resident32") = 1);
    t.def("plan_gather",
          [plan_dict](uint32_t n, uint32_t nparts, uint32_t part_bytes, uint64_t align_or,
                      int max_ctas, uint32_t stage_bytes, uint32_t ring_bytes, int sm_count,
                      int resident16, int resident32) {
              kernels::GatherLaunch a;
              a.n = n;
              a.nparts = nparts;
              a.part_bytes = part_bytes;
              a.align_or = align_or;
              a.max_ctas = max_ctas;
              a.stage_bytes = stage_bytes;
              a.ring_bytes = ring_bytes;
              return plan_dict(kernels::plan_gather(a, sm_count, {resident16, resident32}));
          },
          py::arg("n"), py::arg("nparts"), py::arg("part_bytes"), py::arg("align_or") = 0,
          py::arg("max_ctas") = 0, py::arg("stage_bytes") = 0, py::arg("ring_bytes") = 0,
          py::arg("sm_count") = 132, py::arg("resident16") = 1, py::arg("resident32") = 1);
    t.def("plan_gather_layered",
          [plan_dict](uint32_t n, uint32_t nparts, uint32_t part_bytes, uint32_t group_parts,
                      uint64_t align_or, int max_ctas, int sm_count, int resident16,
                      int resident32) {
              kernels::GatherLaunch a;
              a.n = n;
              a.nparts = nparts;
              a.part_bytes = part_bytes;
              static uint32_t flags[1];
              a.group_flags = flags;
              a.group_parts = group_parts;
              a.align_or = align_or;
              a.max_ctas = max_ctas;
              return plan_dict(kernels::plan_gather(a, sm_count, {resident16, resident32}));
          },
          py::arg("n"), py::arg("nparts"), py::arg("part_bytes"), py::arg("group_parts") = 2,
          py::arg("align_or") = 0, py::arg("max_ctas") = 0, py::arg("sm_count") = 132,
          py::arg("resident16") = 1, py::arg("resident32") = 1);
    t.def("plan_gather_rows",
          [plan_dict](uint32_t n, uint32_t nparts, uint32_t rows, uint32_t row_bytes,
                      uint32_t src_pitch, uint32_t src_col, uint32_t dst_pitch, uint64_t align_or,
                      uint32_t group_parts, int max_ctas, int sm_count, int resident16,
                      int resident32, uint32_t slices, uint32_t dst_slice_pitch, uint32_t pieces) {
              const kernels::GatherLaunch a = rows_launch(
                  n, nparts, false,
                  {rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dst_slice_pitch, pieces},
                  align_or, group_parts, max_ctas);
              return plan_dict(kernels::plan_gather_rows(a, sm_count, {resident16, resident32}));
          },
          py::arg("n"), py::arg("nparts"), py::arg("rows"), py::arg("row_bytes"),
          py::arg("src_pitch"), py::arg("src_col") = 0, py::arg("dst_pitch") = 0,
          py::arg("align_or") = 0, py::arg("group_parts") = 0, py::arg("max_ctas") = 0,
          py::arg("sm_count") = 132, py::arg("resident16") = 1, py::arg("resident32") = 1,
          py::arg("slices") = 1, py::arg("dst_slice_pitch") = 0, py::arg("pieces") = 1);
    t.def("plan_read_fused",
          [plan_dict](uint32_t n, uint32_t bytes, uint64_t align_or, int variant, int max_ctas,
                      uint32_t stage_bytes, uint32_t ring_bytes, int sm_count, int resident16,
                      int resident32) {
              kernels::ReadFusedLaunch a;
              a.n = n;
              a.bytes = bytes;
              a.align_or = align_or;
              a.variant = variant;
              a.max_ctas = max_ctas;
              a.stage_bytes = stage_bytes;
              a.ring_bytes = ring_bytes;
              py::dict d = plan_dict(kernels::plan_read_fused(a, sm_count, {resident16, resident32}));
              d["scatter_ctas"] = kernels::scatter_read_ctas(a, sm_count);
              return d;
          },
          py::arg("n"), py::arg("bytes"), py::arg("align_or") = 0, py::arg("variant") = 0,
          py::arg("max_ctas") = 0, py::arg("stage_bytes") = 0, py::arg("ring_bytes") = 0,
          py::arg("sm_count") = 132, py::arg("resident16") = 1, py::arg("resident32") = 1);
    t.def("plan_fp8",
          [plan_dict](uint32_t n, uint32_t elems, int variant, bool aligned16, uint32_t group,
                      int max_ctas, int sm_count) {
              kernels::Fp8Launch a;
              a.n = n;
              a.elems = elems;
              a.variant = variant;
              a.aligned16 = aligned16;
              a.group = group;
              a.max_ctas = max_ctas;
              return plan_dict(kernels::plan_fp8(a, sm_count));
          },
          py::arg("n"), py::arg("elems"), py::arg("variant") = 0, py::arg("aligned16") = true,
          py::arg("group") = 128, py::arg("max_ctas") = 0, py::arg("sm_count") = 132);
    t.def("plan_gather_fp8",
          [plan_dict](uint32_t n, uint32_t nparts, uint32_t elems, int variant, uint64_t align_or,
                      int max_ctas, int sm_count) {
              kernels::GatherLaunch a;
              a.n = n;
              a.nparts = nparts;
              a.align_or = align_or;
              a.max_ctas = max_ctas;
              return plan_dict(kernels::plan_gather_fp8(a, elems, variant, sm_count));
          },
          py::arg("n"), py::arg("nparts"), py::arg("elems"), py::arg("variant") = 0,
          py::arg("align_or") = 0, py::arg("max_ctas") = 0, py::arg("sm_count") = 132);
    t.def("plan_gather_fp8_rows",
          [plan_dict](uint32_t n, uint32_t nparts, uint32_t elems, uint32_t rows,
                      uint32_t row_bytes, uint32_t src_pitch, uint32_t src_col, uint32_t dst_pitch,
                      uint64_t align_or, uint32_t group_parts, bool write, int max_ctas,
                      int sm_count, int resident, uint32_t slices, uint32_t dst_slice_pitch,
                      uint32_t pieces) {
              const kernels::GatherLaunch a = rows_launch(
                  n, nparts, write,
                  {rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dst_slice_pitch, pieces},
                  align_or, group_parts, max_ctas);
              return plan_dict(
                  kernels::plan_gather_fp8_rows(a, elems, sm_count, {resident, resident}));
          },
          py::arg("n"), py::arg("nparts"), py::arg("elems"), py::arg("rows"), py::arg("row_bytes"),
          py::arg("src_pitch"), py::arg("src_col") = 0, py::arg("dst_pitch") = 0,
          py::arg("align_or") = 0, py::arg("group_parts") = 0, py::arg("write") = false,
          py::arg("max_ctas") = 0, py::arg("sm_count") = 132, py::arg("resident") = 1,
          py::arg("slices") = 1, py::arg("dst_slice_pitch") = 0, py::arg("pieces") = 1);
    // row-sliced writes (kernels/launch_plan.h); group_parts > 0 asks for a layered read, which
    // the write plans refuse
    t.def("plan_gather_rows_write",
          [plan_dict](uint32_t n, uint32_t nparts, uint32_t rows, uint32_t row_bytes,
                      uint32_t src_pitch, uint32_t src_col, uint32_t dst_pitch, uint32_t slices,
                      uint32_t dst_slice_pitch, uint64_t align_or, bool write,
                      uint32_t group_parts, int max_ctas, int sm_count, int resident16,
                      int resident32, uint32_t pieces) {
              const kernels::GatherLaunch a = rows_launch(
                  n, nparts, write,
                  {rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dst_slice_pitch, pieces},
                  align_or, group_parts, max_ctas);
              return plan_dict(
                  kernels::plan_gather_rows_write(a, sm_count, {resident16, resident32}));
          },
          py::arg("n"), py::arg("nparts"), py::arg("rows"), py::arg("row_bytes"),
          py::arg("src_pitch"), py::arg("src_col") = 0, py::arg("dst_pitch") = 0,
          py::arg("slices") = 1, py::arg("dst_slice_pitch") = 0, py::arg("align_or") = 0,
          py::arg("write") = true, py::arg("group_parts") = 0, py::arg("max_ctas") = 0,
          py::arg("sm_count") = 132, py::arg("resident16") = 1, py::arg("resident32") = 1,
          py::arg("pieces") = 1);
    t.def("plan_gather_fp8_rows_write",
          [plan_dict](uint32_t n, uint32_t nparts, uint32_t elems, uint32_t rows,
                      uint32_t row_bytes, uint32_t src_pitch, uint32_t src_col, uint32_t dst_pitch,
                      uint32_t slices, uint32_t dst_slice_pitch, uint64_t align_or, bool write,
                      uint32_t group_parts, int max_ctas, int sm_count, int resident,
                      uint32_t pieces) {
              const kernels::GatherLaunch a = rows_launch(
                  n, nparts, write,
                  {rows, row_bytes, src_pitch, src_col, dst_pitch, slices, dst_slice_pitch, pieces},
                  align_or, group_parts, max_ctas);
              return plan_dict(
                  kernels::plan_gather_fp8_rows_write(a, elems, sm_count, {resident, resident}));
          },
          py::arg("n"), py::arg("nparts"), py::arg("elems"), py::arg("rows"), py::arg("row_bytes"),
          py::arg("src_pitch"), py::arg("src_col") = 0, py::arg("dst_pitch") = 0,
          py::arg("slices") = 1, py::arg("dst_slice_pitch") = 0, py::arg("align_or") = 0,
          py::arg("write") = true, py::arg("group_parts") = 0, py::arg("max_ctas") = 0,
          py::arg("sm_count") = 132, py::arg("resident") = 1, py::arg("pieces") = 1);
    // fp8 token records (kernels/launch_plan.h): the geometry the record movers use
    t.def(
        "fp8_records",
        [](uint32_t latent, uint32_t rope) {
            const kernels::Fp8Records r{latent, rope};
            py::dict d;
            d["ok"] = r.ok();
            d["token_elems"] = r.token_elems();
            d["scale_offset"] = r.scale_offset();
            d["rope_offset"] = r.rope_offset();
            d["record_bytes"] = r.record_bytes();
            return d;
        },
        py::arg("latent"), py::arg("rope"));
    t.def(
        "fp8_record_offset",
        [](uint32_t latent, uint32_t rope, uint32_t tokens, uint32_t s, uint32_t t) {
            return kernels::fp8_record_offset(kernels::Fp8Records{latent, rope}, tokens, s, t);
        },
        py::arg("latent"), py::arg("rope"), py::arg("tokens"), py::arg("part"), py::arg("token"));
    t.def(
        "fp8_records_bytes",
        [](uint32_t nparts, uint32_t elems, uint32_t latent, uint32_t rope) {
            return kernels::fp8_records_bytes(nparts, elems, kernels::Fp8Records{latent, rope});
        },
        py::arg("nparts"), py::arg("elems"), py::arg("latent"), py::arg("rope"));
    t.def("plan_gather_fp8_records",
          [plan_dict](uint32_t n, uint32_t nparts, uint32_t elems, uint32_t latent, uint32_t rope,
                      uint64_t align_or, uint32_t group_parts, bool write, int max_ctas,
                      int sm_count, int resident, uint32_t rows, uint32_t pieces) {
              static uint32_t flags[1];
              kernels::GatherLaunch a;
              a.n = n;
              a.nparts = nparts;
              a.write = write;
              a.align_or = align_or;
              a.group_flags = group_parts ? flags : nullptr;
              a.group_parts = group_parts;
              a.max_ctas = max_ctas;
              a.records = kernels::Fp8Records{latent, rope};
              a.rows.rows = rows;  // any row geometry is refused
              a.rows.pieces = pieces;  // piece offsets count in align_or
              return plan_dict(
                  kernels::plan_gather_fp8_records(a, elems, sm_count, {resident, resident}));
          },
          py::arg("n"), py::arg("nparts"), py::arg("elems"), py::arg("latent"), py::arg("rope"),
          py::arg("align_or") = 0, py::arg("group_parts") = 0, py::arg("write") = false,
          py::arg("max_ctas") = 0, py::arg("sm_count") = 132, py::arg("resident") = 1,
          py::arg("rows") = 0, py::arg("pieces") = 1);
    t.def("plan_gather_e4m3",
          [plan_dict](uint32_t n, uint32_t nparts, uint32_t elems, uint64_t align_or,
                      uint32_t group_parts, bool write, int max_ctas, int sm_count, int resident,
                      uint32_t rows, uint32_t pieces, bool records) {
              static uint32_t flags[1];
              kernels::GatherLaunch a;
              a.n = n;
              a.nparts = nparts;
              a.write = write;
              a.align_or = align_or;
              a.group_flags = group_parts ? flags : nullptr;
              a.group_parts = group_parts;
              a.max_ctas = max_ctas;
              a.rows.rows = rows;  // any row geometry is refused
              a.rows.pieces = pieces;
              if (records) a.records = kernels::Fp8Records{512, 64};  // records are refused
              return plan_dict(kernels::plan_gather_e4m3(a, elems, sm_count, {resident, resident}));
          },
          py::arg("n"), py::arg("nparts"), py::arg("elems"), py::arg("align_or") = 0,
          py::arg("group_parts") = 0, py::arg("write") = false, py::arg("max_ctas") = 0,
          py::arg("sm_count") = 132, py::arg("resident") = 1, py::arg("rows") = 0,
          py::arg("pieces") = 1, py::arg("records") = false);
    t.def("plan_gather_rope",
          [plan_dict](uint32_t n, uint32_t nparts, uint32_t part_bytes, uint32_t head_elems,
                      uint32_t rot_offset, uint32_t rot_dim, bool interleaved, uint64_t align_or,
                      uint32_t group_parts, bool write, int max_ctas, int sm_count, int resident,
                      uint32_t rows, uint32_t pieces, bool records, bool scales, bool rope) {
              static uint32_t flags[1];
              static const float scale[kernels::kGatherMaxParts] = {};
              kernels::RopeShift rs;
              rs.head_elems = head_elems;
              rs.rot_offset = rot_offset;
              rs.rot_dim = rot_dim;
              rs.interleaved = interleaved ? 1 : 0;
              kernels::GatherLaunch a;
              a.n = n;
              a.nparts = nparts;
              a.part_bytes = part_bytes;
              a.write = write;
              a.align_or = align_or;
              a.group_flags = group_parts ? flags : nullptr;
              a.group_parts = group_parts;
              a.max_ctas = max_ctas;
              a.rows.rows = rows;  // any row geometry is refused
              a.rows.pieces = pieces;
              if (records) a.records = kernels::Fp8Records{512, 64};  // records are refused
              if (scales) a.part_scale = scale;                       // scales are refused
              a.rope = rope ? &rs : nullptr;
              return plan_dict(kernels::plan_gather_rope(a, sm_count, {resident, resident}));
          },
          py::arg("n"), py::arg("nparts"), py::arg("part_bytes"), py::arg("head_elems"),
          py::arg("rot_offset") = 0, py::arg("rot_dim") = 0, py::arg("interleaved") = false,
          py::arg("align_or") = 0, py::arg("group_parts") = 0, py::arg("write") = false,
          py::arg("max_ctas") = 0, py::arg("sm_count") = 132, py::arg("resident") = 1,
          py::arg("rows") = 0, py::arg("pieces") = 1, py::arg("records") = false,
          py::arg("scales") = false, py::arg("rope") = true,
          "plan_gather_rope of a launch of n blocks of nparts bf16 parts of part_bytes, heads of "
          "head_elems with rot_dim rotary elements from rot_offset (rope=False: no RopeShift)");
    t.def("fp8_rows_read_bytes", &fp8_rows_read_bytes, py::arg("rows"), py::arg("row_bytes"),
          py::arg("src_pitch"), py::arg("src_col") = 0,
          "bytes_read of a row-sliced read of one stored fp8 part (geometry in bf16 bytes)");
    py::class_<MM>(t, "MM")
        .def(py::init<>())
        .def("add_pool", &MM::add_pool)
        .def("allocate",
             [](MM& mm, size_t size, size_t n, int hint) -> py::object {
                 std::vector<Allocation> out;
                 if (!mm.allocate(size, n, hint, out)) return py::none();
                 py::list l;
                 for (auto& a : out) l.append(py::make_tuple(a.seg, a.offset));
                 return l;
             })
        .def("deallocate", &MM::deallocate)
        .def("need_extend", &MM::need_extend)
        .def("used_bytes", &MM::used_bytes)
        .def("total_bytes", &MM::total_bytes);
}
