"""ctypes binding of libfbgpu.so (include/fbgpu.h).  There is no CPU fallback: if the CUDA library is missing or
a call fails, an exception is raised."""
import ctypes as C
import os
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

OP_ROW, OP_INTERSECT, OP_UNION, OP_DIFFERENCE, OP_XOR, OP_NOT, OP_BSI_RANGE, OP_EMPTY, OP_ALL = range(1, 10)
CMP = {"==": 1, "!=": 2, "<": 3, "<=": 4, ">": 5, ">=": 6, "><": 7}
E_INVALID, E_QUERY, E_FORMAT, E_NOSPACE, E_CUDA, E_NOMEM, E_COMM = -1, -2, -3, -4, -5, -6, -7
DEVICE_NONE = -1            # fbgpu_init(FBGPU_DEVICE_NONE): inspection-only context (no device, no queries)


_row_tls = threading.local()


class FbgpuError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"fbgpu error {code}: {msg}")
        self.code = code


class Op(C.Structure):
    _fields_ = [("opcode", C.c_uint32), ("field", C.c_uint32), ("view", C.c_uint32), ("argc", C.c_uint32),
                ("a", C.c_uint64), ("b", C.c_uint64), ("lo", C.c_int64), ("hi", C.c_int64)]


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("fragments", "containers", "array_containers", "bitmap_containers",
                                           "run_containers", "payload_bytes", "device_bytes", "dead_bytes", "full_commits", "patch_commits")]


class Counters(C.Structure):
    _fields_ = [("kernel_launches", C.c_uint64), ("queries", C.c_uint64), ("last_query_gpu_ms", C.c_float),
                ("pair_kernel_queries", C.c_uint32), ("last_algo_bytes", C.c_uint64),
                ("groupby_units", C.c_uint64), ("groupby_fallback_units", C.c_uint64)]


EXPORTS = ["fbgpu_init", "fbgpu_shutdown", "fbgpu_last_error", "fbgpu_abi_version", "fbgpu_load_fragment",
           "fbgpu_load_fragments", "fbgpu_drop_fragment", "fbgpu_commit", "fbgpu_get_stats", "fbgpu_count", "fbgpu_row",
           "fbgpu_row_counts", "fbgpu_row_counts_per_shard", "fbgpu_groupby", "fbgpu_comm_unique_id", "fbgpu_comm_init", "fbgpu_comm_destroy",
           "fbgpu_get_counters", "fbgpu_stream", "fbgpu_rows_payload_bytes", "fbgpu_count_pairs", "fbgpu_columns", "fbgpu_extract", "fbgpu_load_rbf", "fbgpu_load_rbf_dir", "fbgpu_bsi_minmax", "fbgpu_bsi_sum", "fbgpu_compact", "fbgpu_comm_p2p_handle", "fbgpu_comm_p2p_open", "fbgpu_comm_p2p_disable",
           "fbgpu_any", "fbgpu_pair_types", "fbgpu_node_any", "fbgpu_apply_containers", "fbgpu_node_apply_containers",
           "fbgpu_comm_p2p_open_local", "fbgpu_node_init", "fbgpu_node_shutdown", "fbgpu_node_devices", "fbgpu_node_owner", "fbgpu_node_ctx", "fbgpu_node_load_fragment",
           "fbgpu_node_load_fragments", "fbgpu_node_load_rbf_dir", "fbgpu_node_drop_fragment", "fbgpu_node_commit", "fbgpu_node_get_stats", "fbgpu_node_count", "fbgpu_node_row",
           "fbgpu_node_count_pairs", "fbgpu_node_row_counts", "fbgpu_node_groupby", "fbgpu_node_bsi_sum", "fbgpu_node_bsi_minmax"]


def lib_path():
    return os.environ.get("FBGPU_LIB") or os.path.join(_HERE, "libfbgpu.so")   # FBGPU_LIB: another build of the library (the test suite's CPU kernel interpreter)


def load():
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} missing: run `python -m featurebase_b200.build` (no CPU fallback exists)")
    L = C.CDLL(path)
    vp, u32, u64, i32, i64 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int32, C.c_int64
    L.fbgpu_init.argtypes, L.fbgpu_init.restype = [i32, C.POINTER(vp)], C.c_int
    L.fbgpu_shutdown.argtypes, L.fbgpu_shutdown.restype = [vp], None
    L.fbgpu_last_error.argtypes, L.fbgpu_last_error.restype = [], C.c_char_p
    L.fbgpu_abi_version.argtypes, L.fbgpu_abi_version.restype = [], i32
    L.fbgpu_load_fragment.argtypes, L.fbgpu_load_fragment.restype = [vp, u32, u32, u32, u64, vp, u64], C.c_int
    L.fbgpu_load_fragments.argtypes, L.fbgpu_load_fragments.restype = [vp, u32, u32, u32, vp, i64, vp, vp], C.c_int
    L.fbgpu_drop_fragment.argtypes, L.fbgpu_drop_fragment.restype = [vp, u32, u32, u32, u64], C.c_int
    L.fbgpu_apply_containers.argtypes, L.fbgpu_apply_containers.restype = [vp, u32, u32, u32, u64, vp, u64, vp, i64], C.c_int
    L.fbgpu_node_apply_containers.argtypes, L.fbgpu_node_apply_containers.restype = [vp, u32, u32, u32, u64, vp, u64, vp, i64], C.c_int
    L.fbgpu_load_rbf.argtypes, L.fbgpu_load_rbf.restype = [vp, u32, u64, vp, u64, vp, u64, vp, vp, vp, i32, C.POINTER(i32)], C.c_int
    L.fbgpu_load_rbf_dir.argtypes, L.fbgpu_load_rbf_dir.restype = [vp, u32, u64, C.c_char_p, vp, vp, vp, i32, C.POINTER(i32)], C.c_int
    L.fbgpu_commit.argtypes, L.fbgpu_commit.restype = [vp], C.c_int
    L.fbgpu_compact.argtypes, L.fbgpu_compact.restype = [vp], C.c_int
    L.fbgpu_debug_container.argtypes = [vp, u32, u32, u32, u64, u64, i32, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32), vp, u64, C.POINTER(u64)]
    L.fbgpu_debug_container.restype = C.c_int
    L.fbgpu_debug_compile.argtypes, L.fbgpu_debug_compile.restype = [vp, u32, vp, i32, vp, i32, C.POINTER(i32), C.POINTER(i32)], C.c_int
    L.fbgpu_get_stats.argtypes, L.fbgpu_get_stats.restype = [vp, C.POINTER(Stats)], C.c_int
    L.fbgpu_count.argtypes, L.fbgpu_count.restype = [vp, u32, vp, i32, vp, i64, C.POINTER(u64), vp], C.c_int
    L.fbgpu_row.argtypes, L.fbgpu_row.restype = [vp, u32, vp, i32, vp, i64, vp, u64, C.POINTER(u64), C.POINTER(u64)], C.c_int
    L.fbgpu_columns.argtypes, L.fbgpu_columns.restype = [vp, u32, vp, i32, vp, i64, u64, i64, vp, u64, C.POINTER(u64), C.POINTER(u64)], C.c_int
    L.fbgpu_extract.argtypes = [vp, u32, vp, i32, u32, u32, i32, vp, i64, u64, i64, vp, vp, u64, C.POINTER(u64), C.POINTER(u64)]
    L.fbgpu_extract.restype = C.c_int
    L.fbgpu_bsi_minmax.argtypes = [vp, u32, vp, i32, u32, u32, i32, vp, i64, i32, C.POINTER(C.c_int64), C.POINTER(u64)]
    L.fbgpu_bsi_minmax.restype = C.c_int
    L.fbgpu_bsi_sum.argtypes, L.fbgpu_bsi_sum.restype = [vp, u32, vp, i32, u32, u32, i32, vp, i64, C.POINTER(C.c_int64), C.POINTER(u64)], C.c_int
    L.fbgpu_row_counts.argtypes, L.fbgpu_row_counts.restype = [vp, u32, u32, u32, vp, i32, vp, i32, vp, i64, vp, vp, i32, C.POINTER(i32)], C.c_int
    L.fbgpu_row_counts_per_shard.argtypes, L.fbgpu_row_counts_per_shard.restype = [vp, u32, u32, u32, vp, i32, vp, i32, vp, i64, vp], C.c_int
    L.fbgpu_groupby.argtypes, L.fbgpu_groupby.restype = [vp, u32, vp, vp, i32, vp, vp, vp, i32, vp, i64, vp], C.c_int
    L.fbgpu_count_pairs.argtypes, L.fbgpu_count_pairs.restype = [vp, u32, u32, u32, vp, u32, u32, vp, i32, vp, i64, vp], C.c_int
    L.fbgpu_comm_unique_id.argtypes, L.fbgpu_comm_unique_id.restype = [vp], C.c_int
    L.fbgpu_comm_init.argtypes, L.fbgpu_comm_init.restype = [vp, i32, i32, vp], C.c_int
    L.fbgpu_comm_destroy.argtypes, L.fbgpu_comm_destroy.restype = [vp], C.c_int
    L.fbgpu_comm_p2p_handle.argtypes, L.fbgpu_comm_p2p_handle.restype = [vp, vp], C.c_int
    L.fbgpu_comm_p2p_open.argtypes, L.fbgpu_comm_p2p_open.restype = [vp, i32, i32, vp], C.c_int
    L.fbgpu_comm_p2p_disable.argtypes, L.fbgpu_comm_p2p_disable.restype = [vp], C.c_int
    L.fbgpu_get_counters.argtypes, L.fbgpu_get_counters.restype = [vp, C.POINTER(Counters)], C.c_int
    L.fbgpu_stream.argtypes, L.fbgpu_stream.restype = [vp], vp
    L.fbgpu_rows_payload_bytes.argtypes, L.fbgpu_rows_payload_bytes.restype = [vp, u32, u32, u32, vp, i32, vp, i64, C.POINTER(u64), C.POINTER(u64)], C.c_int
    L.fbgpu_comm_p2p_open_local.argtypes, L.fbgpu_comm_p2p_open_local.restype = [vp, i32], C.c_int
    L.fbgpu_any.argtypes, L.fbgpu_any.restype = [vp, u32, vp, i32, vp, i64, C.POINTER(i32)], C.c_int
    L.fbgpu_pair_types.argtypes, L.fbgpu_pair_types.restype = [vp, u32, u32, u32, u64, u32, u32, u64, vp, i64, vp], C.c_int
    # fbgpu_node_*: the fbgpu_* signature of the same name with the node handle in place of the context
    L.fbgpu_node_init.argtypes, L.fbgpu_node_init.restype = [vp, i32, u64, C.POINTER(vp)], C.c_int
    L.fbgpu_node_shutdown.argtypes, L.fbgpu_node_shutdown.restype = [vp], None
    L.fbgpu_node_devices.argtypes, L.fbgpu_node_devices.restype = [vp], i32
    L.fbgpu_node_owner.argtypes, L.fbgpu_node_owner.restype = [vp, u64], i32
    L.fbgpu_node_ctx.argtypes, L.fbgpu_node_ctx.restype = [vp, i32], vp
    for name in ("load_fragment", "load_fragments", "load_rbf_dir", "drop_fragment", "commit", "get_stats", "count", "any", "row", "count_pairs", "groupby", "bsi_sum", "bsi_minmax"):
        src, dst = getattr(L, "fbgpu_" + name), getattr(L, "fbgpu_node_" + name)
        dst.argtypes, dst.restype = src.argtypes, src.restype
    L.fbgpu_node_row_counts.argtypes, L.fbgpu_node_row_counts.restype = [vp, u32, u32, u32, vp, i32, vp, i32, vp, i64, vp], C.c_int
    _LIB = L
    return L


def _u64arr(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.uint64))


def ops_array(ops):
    """list of Op / tuples -> ctypes array (an array built earlier is passed through: a caller that issues the same program
    repeatedly keeps it marshalled, like a Go caller holds its []Op)"""
    if isinstance(ops, C.Array):
        return ops
    arr = (Op * max(len(ops), 1))()
    for i, o in enumerate(ops):
        arr[i] = o
    return arr


class Context:
    """One fbgpu_ctx (one GPU)."""

    def __init__(self, device=0):
        self.L = load()
        self.h = C.c_void_p()
        self._check(self.L.fbgpu_init(device, C.byref(self.h)))

    def _check(self, rc):
        if rc != 0:
            raise FbgpuError(rc, self.L.fbgpu_last_error().decode())

    def close(self):
        if self.h:
            self.L.fbgpu_shutdown(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- residency
    def load_fragment(self, index, field, view, shard, data):
        data = bytes(data) if not isinstance(data, (bytes, bytearray)) else data
        buf = (C.c_uint8 * len(data)).from_buffer_copy(data)
        self._check(self.L.fbgpu_load_fragment(self.h, index, field, view, int(shard), buf, len(data)))

    def load_fragments(self, index, field, view, shards, buf, offsets):
        """buf: numpy uint8 array or (address, nbytes); offsets: n+1 uint64"""
        sh, off = _u64arr(shards), _u64arr(offsets)
        ptr = buf.ctypes.data if isinstance(buf, np.ndarray) else int(buf)
        self._check(self.L.fbgpu_load_fragments(self.h, index, field, view, sh.ctypes.data, len(sh), ptr, off.ctypes.data))

    def load_rbf(self, index, shard, data, names, fields, views, wal=b""):
        """one shard's RBF database bytes (+ WAL) -> fragments; names[i] = "~field;view<" maps to (fields[i], views[i]).
        Returns how many of the names the file held."""
        data, wal = bytes(data), bytes(wal or b"")
        dbuf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
        wbuf = (C.c_uint8 * max(len(wal), 1)).from_buffer_copy(wal or b"\0")
        cn = (C.c_char_p * max(len(names), 1))(*[n.encode() if isinstance(n, str) else n for n in names])
        fl = np.ascontiguousarray(np.asarray(fields, dtype=np.uint32))
        vw = np.ascontiguousarray(np.asarray(views, dtype=np.uint32))
        n = C.c_int32(0)
        self._check(self.L.fbgpu_load_rbf(self.h, index, int(shard), C.addressof(dbuf), len(data), C.addressof(wbuf) if wal else None, len(wal),
                                          C.addressof(cn), fl.ctypes.data, vw.ctypes.data, len(names), C.byref(n)))
        return n.value

    def load_rbf_dir(self, index, shard, path, names, fields, views):
        """same as load_rbf, the library mapping `<path>/data` (+ `<path>/wal`) itself"""
        cn = (C.c_char_p * max(len(names), 1))(*[n.encode() if isinstance(n, str) else n for n in names])
        fl = np.ascontiguousarray(np.asarray(fields, dtype=np.uint32))
        vw = np.ascontiguousarray(np.asarray(views, dtype=np.uint32))
        n = C.c_int32(0)
        self._check(self.L.fbgpu_load_rbf_dir(self.h, index, int(shard), os.fsencode(path), C.addressof(cn), fl.ctypes.data, vw.ctypes.data, len(names), C.byref(n)))
        return n.value

    def debug_container(self, index, field, view, shard, row, slot):
        """inspection-only contexts (Context(DEVICE_NONE)): -> None | (type, card, runs, payload bytes as stored)"""
        typ, card, runs, n = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)
        buf = np.empty(8192, dtype=np.uint8)
        self._check(self.L.fbgpu_debug_container(self.h, index, field, view, int(shard), int(row), int(slot), C.byref(typ), C.byref(card), C.byref(runs),
                                                 buf.ctypes.data, 8192, C.byref(n)))
        return None if typ.value == 0 else (typ.value, card.value, runs.value, buf[: n.value].tobytes())

    def debug_compile(self, index, ops):
        """-> ([(op, view slot, row)], stack depth): the device program for a post-order fbgpu_op program"""
        arr = ops_array(ops)
        buf = np.zeros(4096 * 16, dtype=np.uint8)
        n, depth = C.c_int32(0), C.c_int32(0)
        self._check(self.L.fbgpu_debug_compile(self.h, index, arr, len(ops), buf.ctypes.data, 4096, C.byref(n), C.byref(depth)))
        rec = np.frombuffer(buf[: n.value * 16].tobytes(), dtype=np.dtype([("op", "u1"), ("pad", "u1", 3), ("fv", "<u4"), ("row", "<u8")]))
        return [(int(r["op"]), int(r["fv"]), int(r["row"])) for r in rec], depth.value

    def drop_fragment(self, index, field, view, shard):
        self._check(self.L.fbgpu_drop_fragment(self.h, index, field, view, int(shard)))

    def apply_containers(self, index, field, view, shard, data=b"", removed_keys=()):
        """incremental refresh of one fragment: `data` = roaring bytes of ONLY the written containers, removed_keys = deleted keys"""
        data = bytes(data or b"")
        buf = (C.c_uint8 * max(len(data), 1)).from_buffer_copy(data or b"\0")
        rk = _u64arr(list(removed_keys))
        self._check(self.L.fbgpu_apply_containers(self.h, index, field, view, int(shard), buf if data else None, len(data),
                                                  rk.ctypes.data if len(rk) else None, len(rk)))

    def commit(self):
        self._check(self.L.fbgpu_commit(self.h))

    def compact(self):
        """reclaim the arena space of replaced / dropped fragments (stats()["dead_bytes"])"""
        self._check(self.L.fbgpu_compact(self.h))

    def stats(self):
        s = Stats()
        self._check(self.L.fbgpu_get_stats(self.h, C.byref(s)))
        return {n: getattr(s, n) for n, _ in Stats._fields_}

    def counters(self):
        s = Counters()
        self._check(self.L.fbgpu_get_counters(self.h, C.byref(s)))
        return {"kernel_launches": s.kernel_launches, "queries": s.queries, "last_query_gpu_ms": s.last_query_gpu_ms, "pair_kernel_queries": s.pair_kernel_queries,
                "groupby_units": s.groupby_units, "groupby_fallback_units": s.groupby_fallback_units}

    # ---- queries
    def count(self, index, ops, shards, per_shard=False):
        sh = _u64arr(shards)
        arr = ops_array(ops)
        tot = C.c_uint64(0)
        per = np.zeros(len(sh), dtype=np.uint64) if per_shard else None
        self._check(self.L.fbgpu_count(self.h, index, arr, len(ops), sh.ctypes.data, len(sh), C.byref(tot),
                                       per.ctypes.data if per_shard else None))
        return (tot.value, per) if per_shard else tot.value

    def any(self, index, ops, shards):
        """Row.Any(): True as soon as one block of shards holds a column of the row (fbgpu_any, early exit by shard blocks)"""
        sh = _u64arr(shards)
        arr = ops_array(ops)
        out = C.c_int32(0)
        self._check(self.L.fbgpu_any(self.h, index, arr, len(ops), sh.ctypes.data, len(sh), C.byref(out)))
        return bool(out.value)

    def pair_types(self, index, field_a, view_a, row_a, field_b, view_b, row_b, shards):
        """4 x 4 histogram of container type pairs (0 absent, 1 array, 2 bitmap, 3 run) of Count(Intersect(Row a, Row b))"""
        sh = _u64arr(shards)
        out = np.zeros(16, dtype=np.uint64)
        self._check(self.L.fbgpu_pair_types(self.h, index, field_a, view_a, int(row_a), field_b, view_b, int(row_b), sh.ctypes.data, len(sh), out.ctypes.data))
        return out.reshape(4, 4)

    def row_into(self, index, ops, shards, buf):
        """fbgpu_row into a caller-owned uint8 array (what a Go caller with a reused buffer does): returns (bytes needed, count,
        fits) — when `fits` is False nothing was written and `buf` must be at least `bytes needed` long"""
        sh = _u64arr(shards)
        arr = ops_array(ops)
        need, cnt = C.c_uint64(0), C.c_uint64(0)
        rc = self.L.fbgpu_row(self.h, index, arr, len(ops), sh.ctypes.data, len(sh), buf.ctypes.data, len(buf), C.byref(need), C.byref(cnt))
        if rc == E_NOSPACE:
            return need.value, cnt.value, False
        self._check(rc)
        return need.value, cnt.value, True

    def row(self, index, ops, shards):
        """returns (pilosa roaring bytes, count)"""
        tls = _row_tls                                           # output buffer kept across calls, one per calling thread
        buf = getattr(tls, "buf", None)                          # (its pages stay mapped; the library is re-entrant, a shared buffer is not)
        if buf is None:
            buf = tls.buf = np.empty(1 << 20, dtype=np.uint8)
        while True:
            need, cnt, fits = self.row_into(index, ops, shards, buf)
            if fits:
                return buf[:need].tobytes(), cnt
            buf = tls.buf = np.empty(int(need) + (int(need) >> 3), dtype=np.uint8)

    def columns(self, index, ops, shards, offset=0, limit=None):
        """ascending column ids of the row (Row.Columns()), expanded on the device; offset / limit = executeLimitCall's window.
        Returns (uint64 array, cardinality of the whole row)"""
        sh = _u64arr(shards)
        arr = ops_array(ops)
        n, total = C.c_uint64(0), C.c_uint64(0)
        cap = max(getattr(self, "_col_cap", 0), 1 << 16) if limit is None else max(int(limit), 1)
        while True:
            buf = np.empty(cap, dtype=np.uint64)
            rc = self.L.fbgpu_columns(self.h, index, arr, len(ops), sh.ctypes.data, len(sh), int(offset), -1 if limit is None else int(limit),
                                      buf.ctypes.data, cap, C.byref(n), C.byref(total))
            if rc == E_NOSPACE:
                cap = int(n.value)
                continue
            self._check(rc)
            if limit is None:
                self._col_cap = cap
            return buf[: n.value].copy(), total.value

    def extract(self, index, field, view, bit_depth, shards, filter_ops=None, offset=0, limit=None):
        """(column ids, int64 values relative to the field's Base, number of columns with a value under the filter): the int
        field's values for the columns of <filter> ∩ not-null, ascending by column, gathered from the bit planes on the device"""
        sh = _u64arr(shards)
        arr = ops_array(filter_ops) if filter_ops else None
        nf = len(filter_ops) if filter_ops else 0
        n, total = C.c_uint64(0), C.c_uint64(0)
        cap = max(getattr(self, "_col_cap", 0), 1 << 16) if limit is None else max(int(limit), 1)
        while True:
            cols, vals = np.empty(cap, dtype=np.uint64), np.empty(cap, dtype=np.int64)
            rc = self.L.fbgpu_extract(self.h, index, arr, nf, field, view, int(bit_depth), sh.ctypes.data, len(sh), int(offset), -1 if limit is None else int(limit),
                                      cols.ctypes.data, vals.ctypes.data, cap, C.byref(n), C.byref(total))
            if rc == E_NOSPACE:
                cap = int(n.value)
                continue
            self._check(rc)
            return cols[: n.value].copy(), vals[: n.value].copy(), total.value

    def bsi_minmax(self, index, field, view, bit_depth, shards, want_max, filter_ops=None):
        """(extreme stored value = value - Base, number of columns holding it) over <filter> ∩ not-null; count 0: empty row"""
        sh = _u64arr(shards)
        arr = ops_array(filter_ops) if filter_ops else None
        val, cnt = C.c_int64(0), C.c_uint64(0)
        self._check(self.L.fbgpu_bsi_minmax(self.h, index, arr, len(filter_ops) if filter_ops else 0, field, view, int(bit_depth), sh.ctypes.data, len(sh),
                                            1 if want_max else 0, C.byref(val), C.byref(cnt)))
        return val.value, cnt.value

    def bsi_sum(self, index, field, view, bit_depth, shards, filter_ops=None):
        """(Σ stored values = Σ (value - Base) in wrapping int64, number of columns) over <filter> ∩ not-null"""
        sh = _u64arr(shards)
        arr = ops_array(filter_ops) if filter_ops else None
        tot, cnt = C.c_int64(0), C.c_uint64(0)
        self._check(self.L.fbgpu_bsi_sum(self.h, index, arr, len(filter_ops) if filter_ops else 0, field, view, int(bit_depth), sh.ctypes.data, len(sh),
                                         C.byref(tot), C.byref(cnt)))
        return tot.value, cnt.value

    def row_counts(self, index, field, view, shards, row_ids=None, filter_ops=None, cap=1 << 20):
        sh = _u64arr(shards)
        f = ops_array(filter_ops) if filter_ops else None
        nf = len(filter_ops) if filter_ops else 0
        n = C.c_int32(0)
        if row_ids is not None:
            ids = _u64arr(row_ids)
            out = np.zeros(len(ids), dtype=np.uint64)
            self._check(self.L.fbgpu_row_counts(self.h, index, field, view, ids.ctypes.data, len(ids), f, nf, sh.ctypes.data, len(sh),
                                                None, out.ctypes.data, len(ids), C.byref(n)))
            return out
        cap = min(cap, 1 << 16)
        while True:                                  # the library reports how many rows there are when the buffers are too small
            rid, out = np.zeros(cap, dtype=np.uint64), np.zeros(cap, dtype=np.uint64)
            rc = self.L.fbgpu_row_counts(self.h, index, field, view, None, 0, f, nf, sh.ctypes.data, len(sh),
                                         rid.ctypes.data, out.ctypes.data, cap, C.byref(n))
            if rc == E_NOSPACE and n.value > cap:
                cap = n.value
                continue
            self._check(rc)
            return rid[: n.value], out[: n.value]

    def row_counts_per_shard(self, index, field, view, shards, row_ids, filter_ops=None):
        """[len(shards), len(row_ids)] matrix of per-shard counts (fbgpu_row_counts_per_shard)"""
        sh, ids = _u64arr(shards), _u64arr(row_ids)
        f = ops_array(filter_ops) if filter_ops else None
        out = np.zeros((len(sh), len(ids)), dtype=np.uint64)
        self._check(self.L.fbgpu_row_counts_per_shard(self.h, index, field, view, ids.ctypes.data, len(ids), f, len(filter_ops) if filter_ops else 0,
                                                      sh.ctypes.data, len(sh), out.ctypes.data))
        return out

    def count_pairs(self, index, field_a, view_a, rows_a, field_b, view_b, rows_b, shards):
        sh, ra, rb = _u64arr(shards), _u64arr(rows_a), _u64arr(rows_b)
        assert len(ra) == len(rb)
        out = np.zeros(len(ra), dtype=np.uint64)
        self._check(self.L.fbgpu_count_pairs(self.h, index, field_a, view_a, ra.ctypes.data, field_b, view_b, rb.ctypes.data, len(ra),
                                             sh.ctypes.data, len(sh), out.ctypes.data))
        return out

    def groupby(self, index, fields, views, row_ids, shards, filter_ops=None):
        sh = _u64arr(shards)
        fl = np.ascontiguousarray(np.asarray(fields, dtype=np.uint32))
        vw = np.ascontiguousarray(np.asarray(views, dtype=np.uint32))
        n_rows = np.ascontiguousarray(np.asarray([len(r) for r in row_ids], dtype=np.int32))
        flat = _u64arr(np.concatenate([np.asarray(r, dtype=np.uint64) for r in row_ids]))
        out = np.zeros(int(np.prod(n_rows.astype(np.int64))), dtype=np.uint64)
        f = ops_array(filter_ops) if filter_ops else None
        nf = len(filter_ops) if filter_ops else 0
        self._check(self.L.fbgpu_groupby(self.h, index, fl.ctypes.data, vw.ctypes.data, len(fl), flat.ctypes.data, n_rows.ctypes.data,
                                         f, nf, sh.ctypes.data, len(sh), out.ctypes.data))
        return out.reshape([int(x) for x in n_rows])

    def rows_payload_bytes(self, index, field, view, shards, row_ids=None):
        sh = _u64arr(shards)
        pay, nc = C.c_uint64(0), C.c_uint64(0)
        if row_ids is None:
            self._check(self.L.fbgpu_rows_payload_bytes(self.h, index, field, view, None, 0, sh.ctypes.data, len(sh), C.byref(pay), C.byref(nc)))
        else:
            ids = _u64arr(row_ids)
            self._check(self.L.fbgpu_rows_payload_bytes(self.h, index, field, view, ids.ctypes.data, len(ids), sh.ctypes.data, len(sh), C.byref(pay), C.byref(nc)))
        return pay.value, nc.value

    # ---- comm
    def comm_unique_id(self):
        buf = (C.c_uint8 * 128)()
        self._check(self.L.fbgpu_comm_unique_id(buf))
        return bytes(buf)

    def comm_init(self, n_ranks, rank, uid):
        buf = (C.c_uint8 * 128).from_buffer_copy(uid)
        self._check(self.L.fbgpu_comm_init(self.h, n_ranks, rank, buf))

    def comm_p2p_handle(self):
        buf = (C.c_uint8 * 64)()
        self._check(self.L.fbgpu_comm_p2p_handle(self.h, buf))
        return bytes(buf)

    def comm_p2p_open(self, n_ranks, rank, handles):
        blob = b"".join(handles)
        assert len(blob) == 64 * n_ranks
        buf = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        self._check(self.L.fbgpu_comm_p2p_open(self.h, n_ranks, rank, buf))

    def comm_p2p_disable(self):
        self._check(self.L.fbgpu_comm_p2p_disable(self.h))


class _NodeCalls:
    """routes Context's `self.L.fbgpu_<call>` to `fbgpu_node_<call>` where the node has that call"""

    def __init__(self, real):
        self._real = real

    def __getattr__(self, name):
        if name.startswith("fbgpu_") and not name.startswith("fbgpu_node_") and hasattr(self._real, "fbgpu_node_" + name[6:]):
            return getattr(self._real, "fbgpu_node_" + name[6:])
        return getattr(self._real, name)


class Node(Context):
    """fbgpu_node: every GPU of this process behind one handle.  Residency and query methods are Context's, fanned out over
    the devices by the library; shard s lives on device slot (s // shard_block) % len(devices)."""

    def __init__(self, devices, shard_block):
        real = load()
        self.L = _NodeCalls(real)
        self.h = C.c_void_p()
        devs = (C.c_int32 * len(devices))(*[int(d) for d in devices])
        self._check(real.fbgpu_node_init(devs, len(devices), int(shard_block), C.byref(self.h)))
        self.n_devices = len(devices)

    def close(self):
        if self.h:
            self.L.fbgpu_node_shutdown(self.h)
            self.h = C.c_void_p()

    def owner(self, shard):
        return int(self.L.fbgpu_node_owner(self.h, int(shard)))

    def device_counters(self, slot):
        s = Counters()
        self._check(self.L._real.fbgpu_get_counters(self.L.fbgpu_node_ctx(self.h, slot), C.byref(s)))
        return {"kernel_launches": s.kernel_launches, "queries": s.queries, "last_query_gpu_ms": s.last_query_gpu_ms}

    def counters(self):
        per = [self.device_counters(i) for i in range(self.n_devices)]
        return {"kernel_launches": sum(p["kernel_launches"] for p in per), "queries": sum(p["queries"] for p in per),
                "last_query_gpu_ms": max(p["last_query_gpu_ms"] for p in per)}

    def row_counts(self, index, field, view, shards, row_ids=None, filter_ops=None, cap=1 << 20):
        if row_ids is None:
            raise NotImplementedError("fbgpu_node_row_counts takes explicit row ids (TopN(ids=..) / TopK candidates)")
        sh, ids = _u64arr(shards), _u64arr(row_ids)
        f = ops_array(filter_ops) if filter_ops else None
        out = np.zeros(len(ids), dtype=np.uint64)
        self._check(self.L.fbgpu_node_row_counts(self.h, index, field, view, ids.ctypes.data, len(ids), f, len(filter_ops) if filter_ops else 0,
                                                 sh.ctypes.data, len(sh), out.ctypes.data))
        return out


def p2p_open_local(contexts):
    """wire the Count mailboxes of contexts living in this process to each other (fbgpu_comm_p2p_open_local)"""
    L = load()
    arr = (C.c_void_p * len(contexts))(*[c.h for c in contexts])
    rc = L.fbgpu_comm_p2p_open_local(arr, len(contexts))
    if rc != 0:
        raise FbgpuError(rc, L.fbgpu_last_error().decode())
