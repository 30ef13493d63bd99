"""fbgpu_bsi_sort (Sort over an int field, with offset / limit, in one device call) and the Sort path built on it.

Entry-point tests compare the call with the columns and stored values the test wrote, sorted in Python by (value, column) or
(-value, column) and sliced; a filter's columns come from an oracle-backed context holding the same fragments.  Query-level
tests compare the executor's Sort and Extract(Sort(..)) on the device with the composition it replaced (every value extracted
and sorted on the host), which contexts without the call still run, and with a node.  The CPU tests check the argument errors
on a context without a device and run this file's gpu tests on the interpreted kernels."""
import ctypes as C
import os

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from oracle import oracle as O
from tests import archetypes as A
from tests.oracle_ctx import OracleCtx

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR"))
SW, W = 1 << 20, 1 << 16
IDX, VV = 0, 7
V, SETF, EX = 5, 2, 3                  # the int field (BSI view VV), a set field for filters, an existence-like row for Not
NEG0 = "-0"                            # a column stored as sign with magnitude 0
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
ENCODINGS = (O.ARRAY, O.BITMAP, O.RUN)
gpu = pytest.mark.gpu


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def row_op(field, row):
    return L.Op(L.OP_ROW, field, 0, 0, row, 0, 0, 0)


def _val(v):
    return 0 if v is NEG0 else v


def bsi_frag(colval, depth, rng):
    """one shard's BSI fragment (exists row 0, sign row 1, magnitude bit i in row 2 + i; NEG0: sign row only), every container in
    a random encoding whatever its cardinality: arrays above 4096 elements, bitmaps of a few bits, runs of single columns"""
    conts = {}
    for c, v in colval:
        o = int(c) % SW
        neg, mag = (True, 0) if v is NEG0 else (v < 0, abs(int(v)))
        for r in [0] + ([1] if neg else []) + [2 + i for i in range(depth) if (mag >> i) & 1]:
            conts.setdefault(r * 16 + (o >> 16), []).append(o & 0xffff)
    b = O.Bitmap()
    for k, lows in sorted(conts.items()):
        b.put(k, A.container_of(np.unique(lows), ENCODINGS[int(rng.integers(0, 3))]))
    return b.to_bytes(optimize=False)


def load(ctxs, colval, depth, seed, field=V):
    """colval: {absolute column: stored value or NEG0}; one BSI fragment per shard that holds a column, loaded into every context"""
    per = {}
    for c, v in colval.items():
        per.setdefault(c // SW, []).append((c, v))
    rng = np.random.default_rng(seed)
    frags = {s: bsi_frag(cv, depth, rng) for s, cv in per.items()}
    for x in ctxs:
        for s, data in frags.items():
            x.load_fragment(IDX, field, VV, s, data)
        x.commit()


def expect(colval, desc, offset, limit, keep=None):
    """(the window's (column, stored value) pairs, |row|)"""
    items = [(c, _val(v)) for c, v in colval.items() if keep is None or c in keep]
    items.sort(key=lambda p: (-p[1] if desc else p[1], p[0]))
    return (items[offset:] if limit is None else items[offset:offset + limit]), len(items)


def windows(total):
    return [(0, None), (0, 0), (0, 1), (0, 10), (7, 13), (0, total + 5), (total, None), (total + 3, 2), (max(total - 1, 0), 10)]


def check(ctx, depth, shards, colval, filter_ops=None, keep=None, what=""):
    total = len(colval) if keep is None else sum(1 for c in colval if c in keep)
    for desc in (False, True):
        for off, lim in windows(total):
            cols, vals, t = ctx.bsi_sort(IDX, V, VV, depth, shards, desc=desc, filter_ops=filter_ops, offset=off, limit=lim)
            want, wt = expect(colval, desc, off, lim, keep)
            assert list(zip(cols.tolist(), vals.tolist())) == want, (what, desc, off, lim)
            assert t == wt, (what, desc, off, lim)


def spread(rng, n, shards, slots=(0, 5, 15)):
    """n distinct columns over the shards, in a few slots of each"""
    cols = set()
    while len(cols) < n:
        cols.add(int(rng.choice(shards)) * SW + int(rng.choice(slots)) * W + int(rng.integers(0, W)))
    return sorted(cols)


def pool_values(rng, depth):
    """few distinct values, so that ties span units and shards and window boundaries fall inside tie groups: the depth's edges
    (INT64_MIN / INT64_MAX at depth 64), 0, sign with magnitude 0, and a few others"""
    hi = (1 << depth) - 1 if depth < 64 else I64_MAX
    lo = -hi if depth < 64 else I64_MIN
    return [hi, lo, 0, NEG0, 1, -1] + [int(x) for x in rng.integers(lo, hi, 3, endpoint=True)]


# ------------------------------------------------------------------ entry point
@gpu
@pytest.mark.parametrize("depth", [1, 8, 21, 63, 64])
def test_depths_with_edge_values(ctx, depth):
    """each depth holding its edge values over three shards; the shard list is unsorted and repeated and lists a shard without
    the field's fragment"""
    rng = np.random.default_rng(300 + depth)
    cols = spread(rng, 120 if ON_EMU else 900, [0, 1, 3])
    pool = pool_values(rng, depth)
    colval = {c: pool[int(rng.integers(0, len(pool)))] for c in cols}
    load([ctx], colval, depth, depth)
    check(ctx, depth, [3, 0, 2, 1, 0], colval, what=depth)


@gpu
def test_depth_zero(ctx):
    """depth 0: every value is 0 (or a sign with magnitude 0), so the order is the column order in both directions"""
    rng = np.random.default_rng(7)
    colval = {c: (NEG0 if rng.random() < 0.3 else 0) for c in spread(rng, 200, [0, 2])}
    load([ctx], colval, 0, 7)
    check(ctx, 0, [0, 1, 2], colval)


@gpu
def test_many_tiles(ctx):
    """more pairs than one radix-sort tile holds (4096), dense columns whose planes are bitmaps, values in long runs"""
    rng = np.random.default_rng(8)
    n = 5000 if ON_EMU else 40000
    cols = [SW + 3 * W + i for i in range(n // 2)] + [2 * SW + k for k in rng.choice(SW, n - n // 2, replace=False).tolist()]
    vals = np.repeat(rng.integers(-2000, 2000, n // 100 + 1), 100)[:n]
    colval = dict(zip(cols, [int(v) for v in vals]))
    load([ctx], colval, 11, 8)
    for desc in (False, True):
        for off, lim in ((0, None), (0, 10), (4090, 20), (n - 3, None)):
            cols_, vals_, t = ctx.bsi_sort(IDX, V, VV, 11, [1, 2], desc=desc, offset=off, limit=lim)
            want, wt = expect(colval, desc, off, lim)
            assert list(zip(cols_.tolist(), vals_.tolist())) == want and t == wt, (desc, off, lim)


def _filter_world(ctxs, seed, depth=16, n=600):
    rng = np.random.default_rng(seed)
    shards = [0, 1, 4]
    cols = spread(rng, n, shards)
    pool = [int(x) for x in rng.integers(-300, 300, 12)] + [NEG0]
    colval = {c: pool[int(rng.integers(0, len(pool)))] for c in cols}
    sets = {r: [c for c in cols if rng.random() < 0.4] + spread(rng, 30, shards) for r in (0, 1)}
    for s in shards:
        b, e = O.Bitmap(), O.Bitmap()
        for r, cs in sets.items():
            for slot in range(16):
                lows = sorted({c % W for c in cs if c // SW == s and (c % SW) // W == slot})
                if lows:
                    b.put(r * 16 + slot, A.container_of(np.asarray(lows), ENCODINGS[(r + slot) % 3]))
        for slot in (0, 5, 15):
            e.put(slot, A.container_of(np.arange(0, W, 2), O.BITMAP))
        for x in ctxs:
            x.load_fragment(IDX, SETF, 0, s, b.to_bytes(optimize=False))
            x.load_fragment(IDX, EX, 0, s, e.to_bytes(optimize=False))
    load(ctxs, colval, depth, seed)
    return shards, colval


def filter_programs(depth=16):
    """{name: filter program}: a row, a Union, a BSI range on the sorted field and a Not"""
    return {
        "row": [row_op(SETF, 0)],
        "union": [row_op(SETF, 0), row_op(SETF, 1), L.Op(L.OP_UNION, 0, 0, 2, 0, 0, 0, 0)],
        "range": [L.Op(L.OP_BSI_RANGE, V, VV, 0, depth, L.CMP[">"], 17, 0)],
        "not": [row_op(SETF, 1), L.Op(L.OP_NOT, EX, 0, 1, 0, 0, 0, 0)],
    }


@gpu
def test_filters(ctx):
    """no filter, a row, a Union, a BSI range and a Not: the row is filter ∩ not-null, its columns taken from the oracle"""
    oc = OracleCtx()
    shards, colval = _filter_world([ctx, oc], 41)
    listed = shards + [9]
    check(ctx, 16, listed, colval, what="none")
    for name, ops in filter_programs().items():
        keep = {int(c) for c in oc.columns(IDX, ops, listed)[0].tolist()}
        assert 0 < len(keep & colval.keys()) < len(colval), name
        check(ctx, 16, listed, colval, filter_ops=ops, keep=keep, what=name)


def _sorts(chunks, k):
    """how many sorts run for chunks of these sizes: before a chunk that would take the buffer past 2K pairs, and at the end"""
    kept = sorts = 0
    for cn in chunks:
        if k is not None and kept > k and kept + cn > 2 * k:
            sorts, kept = sorts + 1, k
        kept += cn
    return sorts + (kept > 0)


@gpu
def test_one_query_and_its_launches(ctx):
    """one call is one library query: one evaluation, one chunk of three launches and one sort of ceil((depth + 1) / 8) passes
    of three launches (a 32-bit field: 5 passes)"""
    rng = np.random.default_rng(9)
    for depth in (1, 21, 32, 64):
        colval = {c: int(rng.integers(-(1 << min(depth, 62)) + 1, 1 << min(depth, 62))) for c in spread(rng, 100, [0, 1])}
        load([ctx], colval, depth, depth, field=V + depth)
        before = ctx.counters()
        got = ctx.bsi_sort(IDX, V + depth, VV, depth, [0, 1], desc=True, limit=10)
        after = ctx.counters()
        want, _ = expect(colval, True, 0, 10)
        assert list(zip(got[0].tolist(), got[1].tolist())) == want, depth
        assert after["queries"] - before["queries"] == 1, depth
        passes = (min(depth + 1, 64) + 7) // 8
        assert after["kernel_launches"] - before["kernel_launches"] == 1 + 3 + 3 * passes, depth
    before = ctx.counters()
    assert ctx.bsi_sort(IDX, V, VV, 8, [0, 1])[2] == 0                     # no such field: the evaluation only
    assert ctx.counters()["kernel_launches"] - before["kernel_launches"] == 1


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: every shard is its own batch and chunk, so that with a small limit the kept pairs are sorted and cut
    between chunks"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    ctx = L.Context(0)
    try:
        oc = OracleCtx()
        shards, colval = _filter_world([ctx, oc], 42)
        check(ctx, 16, shards, colval)
        per_shard = [sum(1 for c in colval if c // SW == s) for s in sorted(shards)]
        for off, lim in ((0, 10), (7, 13), (0, 1)):
            k = off + lim
            assert _sorts(per_shard, k) > 1, (off, lim)                      # at least one cut between chunks
            before = ctx.counters()["kernel_launches"]
            cols, vals, _ = ctx.bsi_sort(IDX, V, VV, 16, shards, offset=off, limit=lim)
            assert list(zip(cols.tolist(), vals.tolist())) == expect(colval, False, off, lim)[0]
            got = ctx.counters()["kernel_launches"] - before
            assert got == len(shards) + 3 * len(per_shard) + 3 * 3 * _sorts(per_shard, k), (off, lim)
        for name, ops in filter_programs().items():
            keep = {int(c) for c in oc.columns(IDX, ops, shards)[0].tolist()}
            check(ctx, 16, shards, colval, filter_ops=ops, keep=keep, what=name)
    finally:
        ctx.close()


def _raw(ctx, shards, offset, limit, cap, null_outputs=False):
    sh = np.asarray(shards, dtype=np.uint64)
    cols, vals = np.zeros(max(cap, 1), dtype=np.uint64), np.zeros(max(cap, 1), dtype=np.int64)
    n, total = C.c_uint64(12345), C.c_uint64(12345)
    rc = ctx.L.fbgpu_bsi_sort(ctx.h, IDX, None, 0, V, VV, 16, sh.ctypes.data, len(sh), 0, offset, limit,
                              None if null_outputs else cols.ctypes.data, None if null_outputs else vals.ctypes.data, cap, C.byref(n), C.byref(total))
    return rc, n.value, total.value, cols, vals


@gpu
def test_nospace_round_trip(ctx):
    """a cap smaller than the window writes nothing and reports the window's size; the retry returns it; *out_total is
    reported in every case"""
    oc = OracleCtx()
    shards, colval = _filter_world([ctx, oc], 43)
    T = len(colval)
    for off, lim in ((0, -1), (5, 40), (T - 2, 10)):
        want, _ = expect(colval, False, off, None if lim < 0 else lim)
        rc, n, t, cols, vals = _raw(ctx, shards, off, lim, len(want) - 1)
        assert (rc, n, t) == (L.E_NOSPACE, len(want), T), (off, lim)
        assert not cols.any() and not vals.any()
        rc, n, t, cols, vals = _raw(ctx, shards, off, lim, 0, null_outputs=True)
        assert (rc, n, t) == (L.E_NOSPACE, len(want), T), (off, lim)
        rc, n, t, cols, vals = _raw(ctx, shards, off, lim, n)
        assert (rc, n, t) == (0, len(want), T) and list(zip(cols[:n].tolist(), vals[:n].tolist())) == want, (off, lim)
    rc, n, t, _, _ = _raw(ctx, shards, T, 5, 0, null_outputs=True)
    assert (rc, n, t) == (0, 0, T)


@gpu
def test_node_equals_the_context(ctx):
    """a node over the same device listed twice with a small shard block, so that both devices' lists merge, answers what the
    single context answers"""
    node = L.Node([0, 0], 1)
    try:
        oc = OracleCtx()
        shards, colval = _filter_world([ctx, node, oc], 44)
        assert {node.owner(s) for s in shards} == {0, 1}
        for name, ops in [("none", None)] + list(filter_programs().items()):
            for desc in (False, True):
                for off, lim in windows(len(colval))[:6]:
                    a = ctx.bsi_sort(IDX, V, VV, 16, shards, desc=desc, filter_ops=ops, offset=off, limit=lim)
                    b = node.bsi_sort(IDX, V, VV, 16, shards, desc=desc, filter_ops=ops, offset=off, limit=lim)
                    assert a[0].tolist() == b[0].tolist() and a[1].tolist() == b[1].tolist() and a[2] == b[2], (name, desc, off, lim)
        keep = {int(c) for c in oc.columns(IDX, filter_programs()["union"], shards)[0].tolist()}
        check(node, 16, shards, colval, filter_ops=filter_programs()["union"], keep=keep)
    finally:
        node.close()


# ------------------------------------------------------------------ query level
class _Composition:
    """the device context without bsi_sort: the executor extracts every value and sorts on the host"""

    def __init__(self, ctx):
        self._ctx = ctx

    def __getattr__(self, name):
        if name == "bsi_sort":
            raise AttributeError(name)
        return getattr(self._ctx, name)


def _holder(ctx, seed):
    h = X.Holder(ctx=ctx)
    idx = h.create_index("i")
    idx.create_field("f")
    idx.create_field("v", "int", min=-40, max=40)
    idx.create_field("w", "int", min=1000, max=1100)                     # Base 1000
    idx.create_field("z", "int", min=I64_MIN, max=I64_MAX)              # depth 64
    rng = np.random.default_rng(seed)
    for s in (0, 1, 2, 4):
        for c in rng.choice(3000, size=400, replace=False):
            col = s * SW + int(c)
            if rng.random() < 0.8:
                h.set_value("i", "v", col, int(rng.integers(-40, 41)))
            if rng.random() < 0.6:
                h.set_value("i", "w", col, int(rng.integers(1000, 1005)))
            if rng.random() < 0.5:
                h.set_value("i", "z", col, [I64_MIN, I64_MAX, 0, -1, 5][int(rng.integers(0, 5))])
            for r in range(3):
                if rng.random() < 0.3:
                    h.set_bit("i", "f", r, col)
    h.sync()
    return h


QUERIES = [
    "Sort(Row(f=0), field=v)",
    "Sort(Row(f=0), field=v, sort-desc=true, limit=10)",
    "Sort(Row(v >= 0), field=v, sort-desc=true, limit=10)",
    "Sort(Union(Row(f=1), Row(f=2)), field=w, limit=25, offset=7)",
    "Sort(Not(Row(f=0)), field=w, sort-desc=true, offset=100)",
    "Sort(All(), field=z, limit=30, offset=3)",
    "Sort(All(), field=z, sort-desc=true, limit=12)",
    "Sort(Row(f=2), field=v, offset=100000)",
    "Sort(Row(f=1), field=w, limit=0)",
    "Sort(Row(f=1), field=v, sort-desc=true, limit=1000000000000)",
    "Extract(Sort(Row(f=0), field=v, sort-desc=true, limit=8, offset=2), Rows(v), Rows(w), Rows(f))",
    "Extract(Sort(Row(v > -5), field=z, limit=20), Rows(z), Rows(v))",
]


@gpu
def test_executor_on_three_contexts():
    """Sort and Extract(Sort(..)) give the same result through the call and through the composition on the same context; Sort
    gives it on a node too, where it used to raise NotImplementedError"""
    dev = _holder(L.Context(0), 51)
    node = _holder(L.Node([0, 0], 1), 51)
    try:
        ed, en = X.Executor(dev), X.Executor(node)
        ec = X.Executor(dev)
        ec.ctx = _Composition(dev.ctx)
        nonempty = 0
        for q in QUERIES:
            before = dev.ctx.counters()["queries"]
            got = ed.execute("i", q)[0]
            if q.startswith("Sort"):
                assert dev.ctx.counters()["queries"] - before == 1, q
                assert got == en.execute("i", q)[0], q                   # (Extract's int cells have no node form)
            assert got == ec.execute("i", q)[0], q
            nonempty += bool(got["columns"] if isinstance(got, dict) else got)
        assert nonempty >= len(QUERIES) - 2
    finally:
        dev.ctx.close()
        node.ctx.close()


# ------------------------------------------------------------------ CPU
ARG_ERRORS = [
    ({"null": "out_n"}, "null argument"),
    ({"null": "shards"}, "null argument"),
    ({"null": "out_cols"}, "null argument"),
    ({"null": "out_vals"}, "null argument"),
    ({"null": "ops"}, "null argument"),
    ({"n_shards": -1}, "null argument"),
    ({"n_ops": -1}, "null argument"),
    ({"depth": -1}, "bit depth -1 outside 0..64"),
    ({"depth": 65}, "bit depth 65 outside 0..64"),
]


def _raw_args(L_, h, n_ops=1, depth=8, n_shards=1, cap=4, null=None):
    sh = np.asarray([0], dtype=np.uint64)
    cols, vals = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.int64)
    ops = L.ops_array([row_op(SETF, 0)])
    n, total = C.c_uint64(0), C.c_uint64(0)
    return L_.fbgpu_bsi_sort(h, IDX, None if null == "ops" else ops, n_ops, V, VV, depth, None if null == "shards" else sh.ctypes.data, n_shards,
                             1, 0, 10, None if null == "out_cols" else cols.ctypes.data, None if null == "out_vals" else vals.ctypes.data, cap,
                             None if null == "out_n" else C.byref(n), C.byref(total))


def test_argument_errors_before_the_device_check():
    """argument errors come before the device check, on a context and on a node; valid arguments reach it"""
    ctx = L.Context(L.DEVICE_NONE)
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        for L_, h in ((ctx.L, ctx.h), (node.L, node.h)):
            for kw, msg in ARG_ERRORS:
                rc = _raw_args(L_, h, **kw)
                assert rc == L.E_INVALID and L_.fbgpu_last_error().decode() == msg, (kw, msg)
            for kw in ({}, {"depth": 0}, {"depth": 64}, {"n_ops": 0, "null": "ops"}, {"cap": 0, "null": "out_cols"}):
                rc = _raw_args(L_, h, **kw)
                assert rc == L.E_CUDA and "no device" in L_.fbgpu_last_error().decode(), kw
        with pytest.raises(L.FbgpuError) as e:
            ctx.bsi_sort(IDX, V, VV, 8, [0], limit=3)
        assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()
        node.close()


def test_bsi_sort_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_bsi_sort.py"], timeout=3000)
