"""fbgpu_extract_rows (the rows of a set, mutex, bool or time field for every column of a row, in one device call) and the Extract
and Sort paths built on it.

Entry-point tests compare the call with Python dicts of the bits the test wrote: for every column of the window, the ascending
rows of the field that hold it.  The window's columns come from an oracle-backed context holding the same fragments, and must
equal fbgpu_columns' for the same arguments.  Containers are stored in random encodings whatever their cardinality, so a slot
mixes arrays above 4096 elements, bitmaps of a few bits and runs of single columns.  Query-level tests compare the executor's
Extract and Sort on the device with an oracle-backed holder, which runs the per-row composition the call replaces.  The CPU
tests check the argument errors on a context without a device and the node routing, and run this file's gpu tests on the
interpreted kernels."""
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
IDX = 0
SETF, SPARSE, MUTEX, BOOL, FILT, EX = 1, 2, 3, 4, 5, 6
NEVER = 40                              # a field that is never loaded
SPARSE_ROWS = [5] + [(1 << 33) + 977 * j for j in range(12)]      # row ids above 2^32, too spread for the dense directory
ENCODINGS = (O.ARRAY, O.BITMAP, O.RUN)
SHARDS = [0, 1, 3]                      # shard 2 holds the filter field only
LISTED = [3, 0, 2, 1, 0]                # unsorted, repeated, with a shard without the fields' fragments
gpu = pytest.mark.gpu


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def row_op(field, row):
    return L.Op(L.OP_ROW, field, 0, 0, row, 0, 0, 0)


def frag_bytes(rows_cols, rng):
    """{row: local columns of one shard} -> the shard's fragment, every container in a random encoding"""
    conts = {}
    for r, cs in rows_cols.items():
        for c in cs:
            conts.setdefault(r * 16 + (c >> 16), []).append(c & 0xffff)
    b = O.Bitmap()
    for k, lows in sorted(conts.items()):
        b.put(k, A.container_of(np.unique(lows), ENCODINGS[int(rng.integers(0, 3))]))
    return b.to_bytes(optimize=False)


def load_field(ctxs, field, model, rng):
    """model {column: rows}: one fragment per shard that holds a bit, loaded into every context"""
    per = {}
    for col, rows in model.items():
        for r in rows:
            per.setdefault(col // SW, {}).setdefault(r, []).append(col % SW)
    for s, rc in sorted(per.items()):
        data = frag_bytes(rc, rng)
        for x in ctxs:
            x.load_fragment(IDX, field, 0, s, data)


def spread(rng, n, shards, slots=(0, 5, 15)):
    cols = set()
    while len(cols) < n:
        cols.add(int(rng.choice(shards)) * SW + int(rng.choice(slots)) * W + int(rng.integers(0, W)))
    return sorted(cols)


def world(ctxs, seed, n=None):
    """{field: {column: ascending rows}}: a set field with dense row ids (0 .. 39; columns with none, one, a few and 30 rows),
    a set field with sparse row ids above 2^32, a mutex field (one row, none, or two rows in a non-canonical column) and a bool
    field; filter rows 0 and 1 of FILT, and an existence row for Not"""
    rng = np.random.default_rng(seed)
    n = n or (150 if ON_EMU else 800)
    cols = spread(rng, n, SHARDS)
    models = {SETF: {}, SPARSE: {}, MUTEX: {}, BOOL: {}}
    for c in cols:
        u = rng.random()
        k = 0 if u < 0.25 else 1 if u < 0.5 else 30 if u < 0.55 else int(rng.integers(2, 12))
        models[SETF][c] = sorted(rng.choice(40, k, replace=False).tolist())
        models[SPARSE][c] = sorted(int(r) for r in rng.choice(SPARSE_ROWS, int(rng.integers(0, 4)), replace=False))
        u = rng.random()
        models[MUTEX][c] = [] if u < 0.2 else sorted(rng.choice(8, 2, replace=False).tolist()) if u < 0.3 else [int(rng.integers(0, 8))]
        u = rng.random()
        models[BOOL][c] = [] if u < 0.15 else [0, 1] if u < 0.2 else [int(u < 0.6)]
    for f, m in models.items():
        load_field(ctxs, f, {c: r for c, r in m.items() if r}, rng)
    extra = spread(rng, 40, [2])
    filt = {c: [r for r in (0, 1) if rng.random() < 0.5] for c in cols + extra}
    load_field(ctxs, FILT, {c: r for c, r in filt.items() if r}, rng)
    load_field(ctxs, EX, {c: [0] for c in cols + extra}, rng)
    for x in ctxs:
        x.commit()
    return models


def filter_programs():
    return {
        "row": [row_op(FILT, 0)],
        "union": [row_op(FILT, 0), row_op(FILT, 1), L.Op(L.OP_UNION, 0, 0, 2, 0, 0, 0, 0)],
        "not": [row_op(FILT, 1), L.Op(L.OP_NOT, EX, 0, 1, 0, 0, 0, 0)],
        "set row": [row_op(SETF, 3)],
        "empty": [L.Op(L.OP_EMPTY, 0, 0, 0, 0, 0, 0, 0)],
    }


def windows(total):
    return [(0, None), (0, 0), (0, 1), (total // 2, 10), (total // 3, None), (max(total - 1, 0), 5), (total + 3, None)]


def check(ctx, oc, field, model, ops, shards, what=""):
    total = len(oc.columns(IDX, ops, shards)[0])
    for off, lim in windows(total):
        want = [int(c) for c in oc.columns(IDX, ops, shards, offset=off, limit=lim)[0].tolist()]
        cols, offs, rows, t = ctx.extract_rows(IDX, field, 0, shards, ops, offset=off, limit=lim)
        assert cols.tolist() == want, (what, off, lim)
        assert cols.tolist() == ctx.columns(IDX, ops, shards, offset=off, limit=lim)[0].tolist(), (what, off, lim)
        assert t == total and len(offs) == len(cols) + 1 and offs[0] == 0 and offs[-1] == len(rows), (what, off, lim)
        got = [rows[offs[i]:offs[i + 1]].tolist() for i in range(len(cols))]
        assert got == [model.get(c, []) for c in want], (what, off, lim)


# ------------------------------------------------------------------ entry point
@gpu
def test_lists_against_the_written_bits(ctx):
    """set fields with dense and sparse row ids, a mutex and a bool field, under every filter and window, over an unsorted,
    repeated shard list with a shard that holds none of the fields; a field that was never loaded gives empty lists"""
    oc = OracleCtx()
    models = world([ctx, oc], 11)
    for name, ops in filter_programs().items():
        for field, model in models.items():
            check(ctx, oc, field, model, ops, LISTED, what=(name, field))
        check(ctx, oc, NEVER, {}, ops, LISTED, what=(name, "never loaded"))
    lens = [len(r) for r in models[SETF].values()]
    assert 0 in lens and 1 in lens and 30 in lens


def _raw(ctx, ops, shards, offset, limit, cap_cols, cap_rows, null_outputs=False):
    sh = np.asarray(shards, dtype=np.uint64)
    arr = L.ops_array(ops)
    cols, offs, rows = np.zeros(max(cap_cols, 1), dtype=np.uint64), np.zeros(cap_cols + 1, dtype=np.uint64), np.zeros(max(cap_rows, 1), dtype=np.uint64)
    nc, nr, total = C.c_uint64(12345), C.c_uint64(12345), C.c_uint64(12345)
    rc = ctx.L.fbgpu_extract_rows(ctx.h, IDX, arr, len(ops), SETF, 0, sh.ctypes.data, len(sh), offset, limit,
                                  None if null_outputs else cols.ctypes.data, None if null_outputs else offs.ctypes.data, cap_cols,
                                  None if null_outputs else rows.ctypes.data, cap_rows, C.byref(nc), C.byref(nr), C.byref(total))
    return rc, nc.value, nr.value, total.value, cols, offs, rows


@gpu
def test_nospace_round_trip(ctx):
    """a cap smaller than either size, or both, writes nothing and reports both sizes; the retry with them succeeds"""
    oc = OracleCtx()
    world([ctx, oc], 12)
    ops = filter_programs()["union"]
    for off, lim in ((0, -1), (5, 40)):
        want_c, want_o, want_r, T = ctx.extract_rows(IDX, SETF, 0, SHARDS, ops, offset=off, limit=None if lim < 0 else lim)
        nc, nr = len(want_c), len(want_r)
        assert nc > 1 and nr > 1
        for cc, cr in ((nc - 1, nr), (nc, nr - 1), (nc - 1, nr - 1)):
            rc, gc, gr, t, cols, offs, rows = _raw(ctx, ops, SHARDS, off, lim, cc, cr)
            assert (rc, gc, gr, t) == (L.E_NOSPACE, nc, nr, T), (off, lim, cc, cr)
            assert not cols.any() and not offs.any() and not rows.any()
        rc, gc, gr, t, _, _, _ = _raw(ctx, ops, SHARDS, off, lim, 0, 0, null_outputs=True)
        assert (rc, gc, gr, t) == (L.E_NOSPACE, nc, nr, T)
        rc, gc, gr, t, cols, offs, rows = _raw(ctx, ops, SHARDS, off, lim, gc, gr)
        assert (rc, gc, gr, t) == (0, nc, nr, T)
        assert cols[:nc].tolist() == want_c.tolist() and offs[:nc + 1].tolist() == want_o.tolist() and rows[:nr].tolist() == want_r.tolist()
    rc, gc, gr, t, _, _, _ = _raw(ctx, ops, SHARDS, 10 ** 9, 5, 0, 0, null_outputs=True)
    assert (rc, gc, gr) == (0, 0, 0)


@gpu
def test_one_query_per_call(ctx):
    world([ctx], 13)
    for field in (SETF, MUTEX, NEVER):
        before = ctx.counters()["queries"]
        ctx.extract_rows(IDX, field, 0, LISTED, filter_programs()["union"], offset=3, limit=50)
        assert ctx.counters()["queries"] - before == 1, field


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: every shard is its own evaluation batch, so windows and lists cross batches"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    ctx = L.Context(0)
    try:
        oc = OracleCtx()
        models = world([ctx, oc], 14)
        for name, ops in filter_programs().items():
            for field in (SETF, SPARSE, MUTEX):
                check(ctx, oc, field, models[field], ops, SHARDS, what=(name, field))
    finally:
        ctx.close()


@gpu
def test_more_than_one_chunk(ctx):
    """one full shard holding 17 full rows: 2^20 columns of 17 rows are more than 2^24 pairs, so the batch is cut into two
    chunks at a column boundary"""
    if ON_EMU:
        pytest.skip("2^24 pairs: too large for the interpreter")
    n_rows = 17
    b = O.Bitmap()
    for r in range(n_rows):
        for slot in range(16):
            b.put(r * 16 + slot, A.container_of(np.arange(W), ENCODINGS[(r + slot) % 3]))
    ctx.load_fragment(IDX, SETF, 0, 0, b.to_bytes(optimize=False))
    ctx.commit()
    cols, offs, rows, t = ctx.extract_rows(IDX, SETF, 0, [0], [row_op(SETF, 0)])
    assert n_rows * SW > 1 << 24 and t == SW
    assert np.array_equal(cols, np.arange(SW, dtype=np.uint64))
    assert np.array_equal(offs, np.arange(SW + 1, dtype=np.uint64) * n_rows)
    assert np.array_equal(rows, np.tile(np.arange(n_rows, dtype=np.uint64), SW))
    cols, offs, rows, _ = ctx.extract_rows(IDX, SETF, 0, [0], [row_op(SETF, 0)], offset=SW - 3, limit=10)
    assert cols.tolist() == [SW - 3, SW - 2, SW - 1] and rows.tolist() == list(range(n_rows)) * 3


@gpu
def test_store_after_updates_drop_and_compact(ctx):
    """containers rewritten and removed by apply_containers, a fragment dropped, then the arena compacted: the lists follow the
    store"""
    oc = OracleCtx()
    models = world([ctx, oc], 15)
    model = {c: list(r) for c, r in models[SETF].items()}
    rng = np.random.default_rng(16)
    ops = filter_programs()["union"]
    for step in range(3):
        shard = SHARDS[step % 2]
        written, removed = {}, []
        for r in rng.choice(40, 6, replace=False).tolist():
            slot = int(rng.choice([0, 5, 15]))
            if rng.random() < 0.3:
                removed.append(r * 16 + slot)
                for c in model:
                    if c // SW == shard and (c % SW) // W == slot and r in model[c]:
                        model[c].remove(r)
                continue
            lows = sorted(int(x) for x in rng.choice(W, int(rng.integers(1, 3000)), replace=False))
            written[r * 16 + slot] = lows
            for c in list(model):
                if c // SW == shard and (c % SW) // W == slot and r in model[c]:
                    model[c].remove(r)
            for lo in lows:
                c = shard * SW + slot * W + lo
                model[c] = sorted(set(model.get(c, [])) | {r})
        b = O.Bitmap()
        for k, lows in sorted(written.items()):
            b.put(k, A.container_of(np.asarray(lows), ENCODINGS[int(rng.integers(0, 3))]))
        for x in (ctx, oc):
            x.apply_containers(IDX, SETF, 0, shard, b.to_bytes(optimize=False), removed)
            x.commit()
        check(ctx, oc, SETF, model, ops, SHARDS, what=("update", step))
    ctx.drop_fragment(IDX, SETF, 0, 1)                                  # (the oracle only lists the filter's columns)
    ctx.commit()
    model = {c: r for c, r in model.items() if c // SW != 1}
    check(ctx, oc, SETF, model, ops, SHARDS, what="drop")
    ctx.compact()
    check(ctx, oc, SETF, model, ops, SHARDS, what="compact")


# ------------------------------------------------------------------ query level
def _holder(ctx):
    h = X.Holder(ctx=ctx)
    idx = h.create_index("i")
    for name, typ, kw in (("set", "set", {}), ("mutex", "mutex", {}), ("time", "time", {"quantum": "YMDH"}), ("bsint", "int", {"min": -100, "max": 100}),
                          ("bool", "bool", {}), ("f", "set", {}), ("a", "set", {}), ("m", "mutex", {}), ("b", "bool", {})):
        idx.create_field(name, typ, **kw)
    # executor_test.go TestExecutor_Execute_Extract's table (without the translated columns)
    for row, col in ((0, 1), (0, 2), (3, 1), (4, 1), (4, 4 * SW)):
        h.set_bit("i", "set", row, col)
    for row, col in ((0, 1), (0, 2), (4, 4 * SW)):
        h.set_bit("i", "mutex", row, col)
    for col, row, ts in ((0, 1, "2016-01-01T00:00"), (1, 2, "2017-01-01T00:00"), (3, 3, "2018-01-01T00:00")):
        h.set_bit("i", "time", row, col, timestamp=ts)
    for col, v in ((0, 1), (1, -1), (3, 2)):
        h.set_value("i", "bsint", col, v)
    for col, v in ((0, True), (1, False), (3, True)):
        h.set_bit("i", "bool", 1 if v else 0, col)
    h.set_bit("i", "set", 0, SW)
    # a larger table on shards 5..7: a 64-row set field, a mutex field with a column in two rows, a bool field
    rng = np.random.default_rng(21)
    for s in (5, 6, 7):
        for c in rng.choice(4000, 500, replace=False).tolist():
            col = s * SW + c
            if rng.random() < 0.3:
                h.set_bit("i", "f", 0, col)
            for r in rng.choice(64, int(rng.integers(0, 6)), replace=False).tolist():
                h.set_bit("i", "a", r, col)
            if rng.random() < 0.8:
                h.set_bit("i", "m", int(rng.integers(0, 16)), col)
            if rng.random() < 0.7:
                h.set_bit("i", "b", int(rng.random() < 0.5), col)
    h.set_bit("i", "m", 3, 5 * SW + 4001)
    h.set_bit("i", "m", 9, 5 * SW + 4001)       # (set_bit keeps both rows of a mutex column: a non-canonical fragment)
    h.set_bit("i", "f", 0, 5 * SW + 4001)
    h.sync()
    return h


QUERIES = [
    "Extract(All(), Rows(set), Rows(mutex), Rows(time), Rows(bsint), Rows(bool))",
    "Extract(Limit(All(), limit=2, offset=1), Rows(set), Rows(bsint))",
    "Extract(Limit(All(), limit=3, offset=1), Rows(set), Rows(mutex), Rows(bool))",
    "Extract(Row(set=4), Rows(mutex))",
    "Extract(Row(set=9), Rows(mutex))",
    "Extract(Row(f=0), Rows(a), Rows(m), Rows(b))",
    "Extract(Limit(Row(f=0), limit=40, offset=100), Rows(a), Rows(m))",
    "Extract(Limit(All(), limit=1000, offset=700), Rows(a))",
    "Extract(Limit(All(), limit=0), Rows(a))",
    "Extract(Limit(All(), offset=100000), Rows(a))",
    "Extract(Sort(Row(f=0), field=m, sort-desc=true, limit=25, offset=3), Rows(a), Rows(b))",
    "Extract(Sort(All(), field=bsint, limit=3), Rows(set), Rows(time))",
    "Sort(Row(f=0), field=m, limit=10)",
    "Sort(Row(f=0), field=m, sort-desc=true)",
    "Sort(All(), field=b, limit=30, offset=5)",
    "Sort(Not(Row(f=0)), field=b, sort-desc=true, limit=50)",
    "Sort(All(), field=bool)",
    "Sort(All(), field=mutex, sort-desc=true)",
]


@gpu
def test_executor_against_the_composition():
    """Extract and Sort over set-like fields on the device equal the oracle-backed holder, which runs the per-row composition;
    Extract(filter, Rows(a)) is one columns call and one extract_rows call instead of 1 + 1 + R, and Sort over a mutex field one
    extract_rows call"""
    ref, dev = _holder(OracleCtx()), _holder(L.Context(0))
    assert not hasattr(ref.ctx, "extract_rows")
    try:
        er, ed = X.Executor(ref), X.Executor(dev)
        nonempty = 0
        for q in QUERIES:
            want = er.execute("i", q)[0]
            assert ed.execute("i", q)[0] == want, q
            nonempty += bool(want["columns"] if isinstance(want, dict) else want)
        assert nonempty >= len(QUERIES) - 3
        table = ed.execute("i", QUERIES[0])[0]["columns"]
        assert table[:6] == [(0, [[], None, [1], 1, True]), (1, [[0, 3, 4], 0, [2], -1, False]), (2, [[0], 0, [], None, None]),
                             (3, [[], None, [3], 2, True]), (SW, [[0], None, [], None, None]), (4 * SW, [[4], 4, [], None, None])]
        for q, n in (("Extract(Row(f=0), Rows(a))", 2), ("Extract(Row(f=0), Rows(a), Rows(m), Rows(b))", 4), ("Sort(Row(f=0), field=m)", 1)):
            before = dev.ctx.counters()["queries"]
            ed.execute("i", q)
            assert dev.ctx.counters()["queries"] - before == n, q
    finally:
        dev.ctx.close()


# ------------------------------------------------------------------ CPU
ARG_ERRORS = [
    {"null": "handle"}, {"null": "out_n_cols"}, {"null": "out_n_rows"}, {"null": "out_cols"}, {"null": "out_offsets"},
    {"null": "out_rows"}, {"null": "ops"}, {"null": "shards"}, {"n_ops": -1}, {"n_shards": -1},
]


def _raw_args(L_, h, n_ops=1, n_shards=1, cap_cols=4, cap_rows=4, null=None):
    sh = np.asarray([0], dtype=np.uint64)
    cols, offs, rows = np.zeros(4, dtype=np.uint64), np.zeros(5, dtype=np.uint64), np.zeros(4, dtype=np.uint64)
    ops = L.ops_array([row_op(FILT, 0)])
    nc, nr, total = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    return L_.fbgpu_extract_rows(None if null == "handle" else h, IDX, None if null == "ops" else ops, n_ops, SETF, 0,
                                 None if null == "shards" else sh.ctypes.data, n_shards, 0, 10,
                                 None if null == "out_cols" else cols.ctypes.data, None if null == "out_offsets" else offs.ctypes.data, cap_cols,
                                 None if null == "out_rows" else rows.ctypes.data, cap_rows,
                                 None if null == "out_n_cols" else C.byref(nc), None if null == "out_n_rows" else C.byref(nr), C.byref(total))


def test_argument_errors_before_the_device_check():
    """argument errors come before the device check; valid arguments (null outputs with zero caps, no program) reach it"""
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for kw in ARG_ERRORS:
            assert _raw_args(ctx.L, ctx.h, **kw) == L.E_INVALID and ctx.L.fbgpu_last_error().decode() == "null argument", kw
        for kw in ({}, {"cap_cols": 0, "null": "out_cols"}, {"cap_cols": 0, "null": "out_offsets"}, {"cap_rows": 0, "null": "out_rows"},
                   {"n_ops": 0, "null": "ops"}, {"n_shards": 0, "null": "shards"}):
            rc = _raw_args(ctx.L, ctx.h, **kw)
            assert rc == L.E_CUDA and "no device" in ctx.L.fbgpu_last_error().decode(), kw
        with pytest.raises(L.FbgpuError) as e:
            ctx.extract_rows(IDX, SETF, 0, [0], [row_op(FILT, 0)], limit=3)
        assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()


def test_node_has_no_form():
    """there is no node form: Node.extract_rows raises NotImplementedError, and so do Extract and Sort over a set-like field
    on a node, as they did before the call"""
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        with pytest.raises(NotImplementedError):
            node.extract_rows(IDX, SETF, 0, [0], [row_op(FILT, 0)])
    finally:
        node.close()


def test_extract_rows_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_extract_rows.py"], timeout=3000)
