"""fbgpu_bsi_distinct (the distinct values of an int field in one device call) and the Distinct, Count(Distinct) and GroupBy
paths built on it.

Entry-point tests compare the call with the set of stored values the test wrote (the writer, the filter world and the value pools
are test_bsi_sort.py's); a filter's columns come from an oracle-backed context holding the same fragments.  Query-level tests
compare the executor on the device and on a node with an oracle-backed holder, whose context has no bsi_distinct and so runs the
composition (every value extracted, then np.unique).  The CPU tests check the argument errors on a context without a device,
the node routing of the new call, and run this file's gpu tests on the interpreted kernels."""
import ctypes as C
import os

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from featurebase_b200 import roaring_io
from tests.oracle_ctx import OracleCtx
from tests.test_bsi_sort import (I64_MAX, I64_MIN, IDX, NEG0, SETF, SW, V, VV, W, _filter_world, _val, filter_programs, load,
                                 pool_values, row_op, spread)

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR"))
gpu = pytest.mark.gpu


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def expect(colval, keep=None):
    """(the distinct stored values, ascending, |row|)"""
    vals = [_val(v) for c, v in colval.items() if keep is None or c in keep]
    return sorted(set(vals)), len(vals)


def check(ctx, depth, shards, colval, filter_ops=None, keep=None, what=""):
    vals, total = ctx.bsi_distinct(IDX, V, VV, depth, shards, filter_ops=filter_ops)
    want, wt = expect(colval, keep)
    assert vals.dtype == np.int64 and vals.tolist() == want, what
    assert total == wt, what
    if not isinstance(ctx, L.Node):                                      # (fbgpu_extract has no node form)
        _, xv, _ = ctx.extract(IDX, V, VV, depth, shards, filter_ops=filter_ops)
        assert np.array_equal(vals, np.unique(xv)), what                # bit for bit what extract + np.unique give


# ------------------------------------------------------------------ entry point
@gpu
@pytest.mark.parametrize("depth", [0, 1, 8, 21, 63, 64])
def test_depths_with_edge_values(ctx, depth):
    """few distinct values (the depth's edges, INT64_MIN / INT64_MAX at 64, 0 and sign with magnitude 0) over three shards, so
    that duplicates cross units and shards; the shard list is unsorted and repeated and lists a shard without the fragment"""
    rng = np.random.default_rng(500 + depth)
    cols = spread(rng, 120 if ON_EMU else 900, [0, 1, 3])
    pool = pool_values(rng, depth) if depth else [0, NEG0]
    colval = {c: pool[int(rng.integers(0, len(pool)))] for c in cols}
    load([ctx], colval, depth, depth)
    check(ctx, depth, [3, 0, 2, 1, 0], colval, what=depth)
    if depth == 64:
        assert ctx.bsi_distinct(IDX, V, VV, 64, [0, 1, 3])[0][0] == I64_MIN


@gpu
def test_all_distinct_over_many_tiles(ctx):
    """every value distinct, more keys than one sort tile (4096), dense columns whose planes are bitmaps"""
    rng = np.random.default_rng(8)
    n = 5000 if ON_EMU else 60000
    cols = [SW + 3 * W + i for i in range(n // 2)] + [2 * SW + k for k in rng.choice(SW, n - n // 2, replace=False).tolist()]
    vals = rng.choice(1 << 30, n, replace=False) - (1 << 29)
    colval = dict(zip(cols, [int(v) for v in vals]))
    load([ctx], colval, 30, 8)
    check(ctx, 30, [1, 2], colval)


@gpu
def test_filters_and_empty_rows(ctx):
    """no filter, a row, a Union, a BSI range and a Not (the row is filter ∩ not-null, its columns taken from the oracle); an
    empty row, a shard list of shards without the fragment and an empty shard list give no values"""
    oc = OracleCtx()
    shards, colval = _filter_world([ctx, oc], 41)
    listed = shards + [9]
    check(ctx, 16, listed, colval, what="none")
    for name, ops in filter_programs().items():
        keep = {int(c) for c in oc.columns(IDX, ops, listed)[0].tolist()}
        assert 0 < len(keep & colval.keys()) < len(colval), name
        check(ctx, 16, listed, colval, filter_ops=ops, keep=keep, what=name)
    for ops, sh in (([row_op(SETF, 7)], listed), (None, [9, 11]), (None, [])):
        vals, total = ctx.bsi_distinct(IDX, V, VV, 16, sh, filter_ops=ops)
        assert vals.tolist() == [] and total == 0, (ops, sh)


@gpu
def test_one_query_and_its_launches(ctx):
    """one call is one library query: one evaluation, one chunk of two launches (values, keys), one sort of ceil((depth + 1) / 8)
    passes of three launches and one dedupe of three"""
    rng = np.random.default_rng(9)
    for depth in (1, 21, 32, 64):
        m = min(5, (1 << depth) - 1)
        colval = {c: int(rng.integers(-m, m + 1)) for c in spread(rng, 100, [0, 1])}
        load([ctx], colval, depth, depth, field=V + depth)
        before = ctx.counters()
        vals, total = ctx.bsi_distinct(IDX, V + depth, VV, depth, [0, 1])
        after = ctx.counters()
        assert (vals.tolist(), total) == expect(colval), depth
        assert after["queries"] - before["queries"] == 1, depth
        passes = (min(depth + 1, 64) + 7) // 8
        assert after["kernel_launches"] - before["kernel_launches"] == 1 + 2 + 3 * passes + 3, depth
    before = ctx.counters()
    assert ctx.bsi_distinct(IDX, V, VV, 8, [0, 1])[1] == 0                  # no such field: the evaluation only
    assert ctx.counters()["kernel_launches"] - before["kernel_launches"] == 1


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: every shard is its own batch and chunk, so the kept keys are sorted and deduped between chunks"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    ctx = L.Context(0)
    try:
        oc = OracleCtx()
        shards, colval = _filter_world([ctx, oc], 42)
        check(ctx, 16, shards, colval)
        for name, ops in filter_programs().items():
            keep = {int(c) for c in oc.columns(IDX, ops, shards)[0].tolist()}
            check(ctx, 16, shards, colval, filter_ops=ops, keep=keep, what=name)
    finally:
        ctx.close()


def bitmap_fragment(value_of, shard, depth):
    """a full shard of an int field whose column c holds value_of(c) (int64 numpy), every container a bitmap"""
    lows = np.arange(W, dtype=np.int64)
    full = np.full(1024, ~np.uint64(0), dtype=np.uint64)
    conts = []
    for slot in range(16):
        v = value_of(shard * SW + slot * W + lows)
        mag, neg = np.abs(v), v < 0
        planes = [(0, full), (1, np.packbits(neg.astype(np.uint8), bitorder="little").view("<u8"))]
        planes += [(2 + i, np.packbits(((mag >> i) & 1).astype(np.uint8), bitorder="little").view("<u8")) for i in range(depth)]
        conts += [(r * 16 + slot, w) for r, w in planes if w.any()]
    conts.sort(key=lambda kw: kw[0])
    out = bytearray(np.array([roaring_io.MAGIC, len(conts)], dtype="<u4").tobytes())
    for key, w in conts:
        n = int(np.unpackbits(w.view(np.uint8)).sum())
        out += np.array([key], dtype="<u8").tobytes() + np.array([roaring_io.BITMAP, n - 1], dtype="<u2").tobytes()
    off = 8 + 16 * len(conts)
    for k in range(len(conts)):
        out += np.array([off + 8192 * k], dtype="<u4").tobytes()
    for _, w in conts:
        out += w.astype("<u8").tobytes()
    return bytes(out)


@gpu
@pytest.mark.parametrize("kind", ["three_values", "column_ids"])
def test_more_than_one_chunk(ctx, kind):
    """17 full shards: a row of more than 2^24 columns is emitted in two chunks, and the keys of the first are sorted and deduped
    before the second is appended.  Three distinct values (each repeated across both chunks), or every column its own value."""
    if ON_EMU:
        pytest.skip("2^24 columns: too large for the interpreter")
    S = 17
    if kind == "three_values":
        depth, pick = 3, np.array([-5, 0, 7], dtype=np.int64)
        value_of, want = (lambda c: pick[c % 3]), [-5, 0, 7]
    else:
        depth, value_of, want = 25, (lambda c: c), None
    for s in range(S):
        ctx.load_fragment(IDX, V, VV, s, bitmap_fragment(value_of, s, depth))
    ctx.commit()
    before = ctx.counters()["queries"]
    vals, total = ctx.bsi_distinct(IDX, V, VV, depth, list(range(S)))
    # one query; 17 M values are more than the binding's first 2^16-value buffer holds: one NOSPACE answer, then the retry
    assert ctx.counters()["queries"] - before == (1 if want is not None else 2)
    assert total == S * SW
    if want is not None:
        assert vals.tolist() == want
    else:
        assert np.array_equal(vals, np.arange(S * SW, dtype=np.int64))
    f = [L.Op(L.OP_BSI_RANGE, V, VV, 0, depth, L.CMP[">"], 0, 0)]                # the positive values only
    vals, total = ctx.bsi_distinct(IDX, V, VV, depth, list(range(S)), filter_ops=f)
    assert vals.tolist() == ([7] if want is not None else list(range(1, S * SW)))


def _raw(ctx, shards, cap, null_outputs=False):
    sh = np.asarray(shards, dtype=np.uint64)
    vals = np.zeros(max(cap, 1), dtype=np.int64)
    n, total = C.c_uint64(12345), C.c_uint64(12345)
    rc = ctx.L.fbgpu_bsi_distinct(ctx.h, IDX, None, 0, V, VV, 16, sh.ctypes.data, len(sh), None if null_outputs else vals.ctypes.data, cap,
                                  C.byref(n), C.byref(total))
    return rc, n.value, total.value, vals


@gpu
def test_nospace_round_trip(ctx):
    """cap 0 and cap U - 1 write nothing and report U; cap U returns the list; *out_total is reported in every case"""
    oc = OracleCtx()
    shards, colval = _filter_world([ctx, oc], 43)
    want, T = expect(colval)
    U = len(want)
    for cap, null in ((0, True), (0, False), (U - 1, False)):
        rc, n, t, vals = _raw(ctx, shards, cap, null_outputs=null)
        assert (rc, n, t) == (L.E_NOSPACE, U, T), cap
        assert not vals.any(), cap
    rc, n, t, vals = _raw(ctx, shards, U)
    assert (rc, n, t) == (0, U, T) and vals[:n].tolist() == want
    rc, n, t, _ = _raw(ctx, [9], 0, null_outputs=True)                       # an empty list fits cap 0
    assert (rc, n, t) == (0, 0, 0)


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
            for sh in (shards, shards[:1], [9], []):
                a, b = ctx.bsi_distinct(IDX, V, VV, 16, sh, filter_ops=ops), node.bsi_distinct(IDX, V, VV, 16, sh, filter_ops=ops)
                assert a[0].tolist() == b[0].tolist() and a[1] == b[1], (name, sh)
        keep = {int(c) for c in oc.columns(IDX, filter_programs()["union"], shards)[0].tolist()}
        check(node, 16, shards, colval, filter_ops=filter_programs()["union"], keep=keep)
        with pytest.raises(L.FbgpuError) as e:                              # no shard listed: the program is still checked
            node.bsi_distinct(IDX, V, VV, 16, [], filter_ops=[L.Op(L.OP_UNION, 0, 0, 2, 0, 0, 0, 0)])
        assert e.value.code == L.E_INVALID
    finally:
        node.close()


# ------------------------------------------------------------------ query level
def _world(h, seed):
    """index i: a set field f, int fields a (five values: a GroupBy child that runs on a node too), v, w (Base 1000), u and z
    (depth 64); index j: a set field f and an int field v"""
    idx = h.create_index("i")
    idx.create_field("f")
    idx.create_field("a", "int", min=0, max=4)
    idx.create_field("v", "int", min=-40, max=40)
    idx.create_field("w", "int", min=1000, max=1100)
    idx.create_field("u", "int", min=-1000, max=1000)
    idx.create_field("z", "int", min=I64_MIN, max=I64_MAX)
    j = h.create_index("j")
    j.create_field("f")
    j.create_field("v", "int", min=-500, max=500)
    rng = np.random.default_rng(seed)
    n = 120 if ON_EMU else 400
    for s in (0, 1, 2, 4):
        for c in rng.choice(3000, size=n, replace=False):
            col = s * SW + int(c)
            for name, lo, hi, p in (("a", 0, 4, 0.9), ("v", -40, 40, 0.8), ("w", 1000, 1004, 0.6), ("u", -1000, 1000, 0.7)):
                if rng.random() < p:
                    h.set_value("i", name, col, int(rng.integers(lo, hi + 1)))
            if rng.random() < 0.5:
                h.set_value("i", "z", col, [I64_MIN, I64_MAX, 0, -1, 5][int(rng.integers(0, 5))])
            for r in range(3):
                if rng.random() < 0.3:
                    h.set_bit("i", "f", r, col)
            if rng.random() < 0.3:
                h.set_value("j", "v", col, int(rng.integers(-500, 501)))
                if rng.random() < 0.5:
                    h.set_bit("j", "f", 0, col)
    h.sync()
    return h


QUERIES = [
    "Distinct(field=v)",
    "Distinct(Row(f=0), field=v)",
    "Distinct(Union(Row(f=1), Row(f=2)), field=w)",
    "Distinct(Row(v > 10), field=u)",
    "Distinct(field=z)",
    "Distinct(Row(f=0), field=v, index=j)",
    "Distinct(Row(f=9), field=v)",
    "Count(Distinct(field=v))",
    "Count(Distinct(Row(f=1), field=u))",
    "Count(Distinct(Row(f=1), field=z))",
    "Intersect(Row(f=0), Distinct(Row(f=1), index=j, field=v))",         # a Distinct operand: j's values as columns of i
    "GroupBy(Rows(a), Rows(v))",
    "GroupBy(Rows(v), Rows(w), aggregate=Sum(field=u))",
    "GroupBy(Rows(a), aggregate=Count(Distinct(field=v)))",
    "GroupBy(Rows(a), Rows(w), aggregate=Count(Distinct(Row(f=0), field=u)), filter=Row(f=1))",
]
CONTEXT_ONLY = [                                                          # a set field's Rows has no node form
    "GroupBy(Rows(f), Rows(v))",
    "GroupBy(Rows(f), aggregate=Count(Distinct(field=w)))",
]


def _result(r):
    return [int(c) for c in r.columns()] if hasattr(r, "columns") else r


@gpu
def test_queries_against_the_oracle():
    """Distinct (with a filter and with index=), Count(Distinct), a Distinct operand and GroupBy with int children or
    Count(Distinct) give on the device and on a node what an oracle-backed holder gives; on the node these used to raise
    NotImplementedError.  Distinct(field=v) is one library query."""
    ref = _world(X.Holder(ctx=OracleCtx()), 61)
    assert not hasattr(ref.ctx, "bsi_distinct")
    dev = _world(X.Holder(ctx=L.Context(0)), 61)
    node = _world(X.Holder(ctx=L.Node([0, 0], 1)), 61)
    try:
        er, ed, en = X.Executor(ref), X.Executor(dev), X.Executor(node)
        nonempty = 0
        for q in QUERIES + CONTEXT_ONLY:
            want = _result(er.execute("i", q)[0])
            assert _result(ed.execute("i", q)[0]) == want, q
            if q in QUERIES:
                assert _result(en.execute("i", q)[0]) == want, q
            nonempty += bool(want)
        assert nonempty >= len(QUERIES) + len(CONTEXT_ONLY) - 1
        for h, n in ((dev, 1), (node, 2)):                                  # (a node's counters add up its devices' queries)
            before = h.ctx.counters()["queries"]
            X.Executor(h).execute("i", "Distinct(field=v)")
            assert h.ctx.counters()["queries"] - before == n
    finally:
        dev.ctx.close()
        node.ctx.close()


# ------------------------------------------------------------------ CPU
ARG_ERRORS = [
    ({"null": "out_n"}, "null argument"),
    ({"null": "shards"}, "null argument"),
    ({"null": "out_vals"}, "null argument"),
    ({"null": "ops"}, "null argument"),
    ({"n_shards": -1}, "null argument"),
    ({"n_ops": -1}, "null argument"),
    ({"depth": -1}, "bit depth -1 outside 0..64"),
    ({"depth": 65}, "bit depth 65 outside 0..64"),
]


def _raw_args(L_, h, n_ops=1, depth=8, n_shards=1, cap=4, null=None):
    sh = np.asarray([0], dtype=np.uint64)
    vals = np.zeros(4, dtype=np.int64)
    ops = L.ops_array([row_op(SETF, 0)])
    n, total = C.c_uint64(0), C.c_uint64(0)
    return L_.fbgpu_bsi_distinct(h, IDX, None if null == "ops" else ops, n_ops, V, VV, depth, None if null == "shards" else sh.ctypes.data, n_shards,
                                 None if null == "out_vals" else vals.ctypes.data, cap, None if null == "out_n" else C.byref(n), C.byref(total))


def test_argument_errors_before_the_device_check():
    """argument errors come before the device check, on a context and on a node; valid arguments reach it"""
    ctx = L.Context(L.DEVICE_NONE)
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        for L_, h in ((ctx.L, ctx.h), (node.L, node.h)):
            for kw, msg in ARG_ERRORS:
                rc = _raw_args(L_, h, **kw)
                assert rc == L.E_INVALID and L_.fbgpu_last_error().decode() == msg, (kw, msg)
            rc = L_.fbgpu_bsi_distinct(None, IDX, None, 0, V, VV, 8, None, 0, None, 0, C.byref(C.c_uint64()), None)
            assert rc == L.E_INVALID and L_.fbgpu_last_error().decode() == "null argument"
            for kw in ({}, {"depth": 0}, {"depth": 64}, {"n_ops": 0, "null": "ops"}, {"cap": 0, "null": "out_vals"}, {"n_shards": 0, "null": "shards"}):
                rc = _raw_args(L_, h, **kw)
                assert rc == L.E_CUDA and "no device" in L_.fbgpu_last_error().decode(), kw
        for c in (ctx, node):
            with pytest.raises(L.FbgpuError) as e:
                c.bsi_distinct(IDX, V, VV, 8, [0])
            assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()
        node.close()


def test_node_routes_the_call():
    """Node inherits bsi_distinct, and its library handle routes fbgpu_bsi_distinct to the node form"""
    real = L.load()
    calls = L._NodeCalls(real)
    assert calls.fbgpu_bsi_distinct is real.fbgpu_node_bsi_distinct
    assert real.fbgpu_node_bsi_distinct.argtypes == real.fbgpu_bsi_distinct.argtypes
    assert "fbgpu_bsi_distinct" in L.EXPORTS and "fbgpu_node_bsi_distinct" in L.EXPORTS
    assert L.Node.bsi_distinct is L.Context.bsi_distinct


def test_bsi_distinct_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_bsi_distinct.py"], timeout=3000)
