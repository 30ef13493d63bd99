"""fbgpu_groupby_values (GroupBy whose last dimension is the values of an int field) and the GroupBy path built on it.

Entry-point tests compare every count tensor with one the test computes from the columns and values it wrote, as plain Python
integers.  Query-level tests compare the executor's GroupBy with an oracle-backed holder, which has no groupby_values and so runs
the Row(v == value)-per-value composition.  The CPU tests check the argument errors and the refusal on a context without a
device, and run this file's gpu tests on the interpreted kernels."""
import itertools
import os

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from featurebase_b200 import roaring_io
from tests.oracle_ctx import OracleCtx

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR"))
SW = 1 << 20
IDX, VF, VV = 0, 5, 7                  # index, int field, its BSI view
SF = (6, 8, 9)                         # set fields (view 0)
FILT = 10                              # set field of the filters
NEG0 = "-0"                            # a column stored as sign with magnitude 0
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
gpu = pytest.mark.gpu


def bsi_bytes(cols, vals, depth):
    """one shard's BSI fragment: exists row 0, sign row 1, magnitude bit i in row 2 + i (NEG0: sign row only)"""
    bits = []
    for c, v in zip(cols, vals):
        o = int(c) % SW
        neg, mag = (True, 0) if v is NEG0 else (v < 0, abs(int(v)))
        bits.append(o)
        if neg:
            bits.append(SW + o)
        bits += [(2 + i) * SW + o for i in range(depth) if (mag >> i) & 1]
    return roaring_io.encode(np.unique(np.asarray(bits, dtype=np.uint64)))


def load_values(ctx, colval, depth):
    """colval: {absolute column: stored value or NEG0}; one BSI fragment per shard that holds a column"""
    per = {}
    for c, v in colval.items():
        per.setdefault(c // SW, []).append((c, v))
    for s, cv in per.items():
        ctx.load_fragment(IDX, VF, VV, s, bsi_bytes([c for c, _ in cv], [v for _, v in cv], depth))


def load_set(ctx, field, rows):
    """rows: {row id: absolute columns}; one fragment per shard"""
    per = {}
    for row, cols in rows.items():
        for c in cols:
            per.setdefault(int(c) // SW, []).append(row * SW + int(c) % SW)
    for s, bits in per.items():
        ctx.load_fragment(IDX, field, 0, s, roaring_io.encode(np.unique(np.asarray(bits, dtype=np.uint64))))


def expect(colval, dims, values, keep=None):
    """the count tensor from the written data: dims = [(row list, {row: columns})], keep = the filter's columns"""
    shape = [len(r) for r, _ in dims] + [len(values)]
    out = np.zeros(shape, dtype=np.uint64)
    pos = {v: j for j, v in enumerate(values)}
    member = [{r: set(int(c) for c in cols) for r, cols in m.items()} for _, m in dims]
    for c, v in colval.items():
        if v is NEG0 or v not in pos or (keep is not None and c not in keep):
            continue
        for ix in itertools.product(*[[i for i, r in enumerate(rows) if c in m.get(r, ())] for (rows, _), m in zip(dims, member)]):
            out[ix + (pos[v],)] += 1
    return out


def gbv(ctx, dims, values, depth, shards, filter_ops=None):
    return ctx.groupby_values(IDX, [SF[k] for k in range(len(dims))], [0] * len(dims), [r for r, _ in dims], VF, VV, depth, values, shards,
                              filter_ops=filter_ops)


def filt(row):
    return [L.Op(L.OP_ROW, FILT, 0, 0, row, 0, 0, 0)]


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


# ------------------------------------------------------------------ entry point
def _depth_values(rng, depth, n):
    if depth == 64:
        edge = [I64_MIN, I64_MAX, I64_MIN + 1, -1, 0, 1]
        rnd = [int(x) for x in rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)]
    else:
        top = (1 << depth) - 1
        edge = [-top, top, 0, -1 if depth else 0, 1 if depth else 0]
        rnd = [int(x) for x in rng.integers(-top, top + 1, n, dtype=np.int64)] if depth < 63 else \
              [max(-top, int(rng.integers(-(1 << 62), 1 << 62)) * 2 + int(rng.integers(0, 2))) for _ in range(n)]
    return edge + rnd


@gpu
@pytest.mark.parametrize("depth", [1, 8, 31, 32, 33, 63, 64])
def test_depths_with_edge_values(ctx, depth):
    """random and edge values (INT64_MIN / INT64_MAX at depth 64) over two shards, grouped alone and by one set field; the
    value list includes absent values and omits present ones; a listed shard holds no fragment at all"""
    rng = np.random.default_rng(depth)
    n = 60 if ON_EMU else 400
    cols = rng.choice(2 * SW, n, replace=False).tolist()
    vals = _depth_values(rng, depth, n)[:n]
    colval = dict(zip(cols, vals))
    load_values(ctx, colval, depth)
    b = {r: rng.choice(cols, n // 3, replace=False).tolist() for r in range(4)}
    load_set(ctx, SF[0], b)
    ctx.commit()
    present = sorted(set(vals))
    absent = [x for x in (I64_MIN, -7777, 3, 12345, I64_MAX) if x not in present]
    values = sorted(set(present[::2] + absent))                                # every other present value
    shards = [0, 1, 4]
    assert np.array_equal(gbv(ctx, [], values, depth, shards), expect(colval, [], values))
    dims = [([0, 1, 2, 3, 9], b)]                                              # row 9 holds nothing
    assert np.array_equal(gbv(ctx, dims, values, depth, shards), expect(colval, dims, values))


@gpu
@pytest.mark.parametrize("layout", ["bitmap", "run", "array"])
def test_container_encodings(ctx, layout):
    """planes and b rows stored as bitmaps (dense random columns), runs (contiguous columns, values in long stretches) and arrays
    (scattered columns)"""
    rng = np.random.default_rng(11)
    n = 20000 if ON_EMU else 60000
    if layout == "bitmap":
        cols = (np.sort(rng.choice(SW // 8, n, replace=False)) + 3 * 65536).tolist()
        vals = rng.integers(-3000, 3000, n).tolist()
        b = {r: [c for c in cols if rng.random() < 0.5] for r in range(2)}
    elif layout == "run":
        cols = list(range(100, 100 + n))
        vals = np.repeat(rng.integers(-(1 << 20), 1 << 20, n // 1000), 1000).tolist()
        b = {0: cols[: n // 2], 1: cols[n // 3: n // 3 + 7000], 2: cols[5000: 5100]}
    else:
        cols = rng.choice(3 * SW, 3000 if ON_EMU else 9000, replace=False).tolist()
        vals = rng.integers(-300, 300, len(cols)).tolist()
        b = {r: rng.choice(cols, len(cols) // 2, replace=False).tolist() for r in range(3)}      # >= 64 per slot: stored bank-striped
    colval = dict(zip(cols, vals))
    load_values(ctx, colval, 21)
    load_set(ctx, SF[0], b)
    ctx.commit()
    values = sorted(set(vals))
    dims = [(sorted(b), b)]
    shards = [0, 1, 2]
    assert np.array_equal(gbv(ctx, dims, values, 21, shards), expect(colval, dims, values))
    assert np.array_equal(gbv(ctx, [], values, 21, shards), expect(colval, [], values))


@gpu
def test_filters(ctx):
    """no filter, a sparse, a dense and an empty filter, with 1 and 0 set dimensions"""
    rng = np.random.default_rng(12)
    n = 1500 if ON_EMU else 5000
    cols = rng.choice(2 * SW, n, replace=False).tolist()
    vals = rng.integers(-50, 50, n).tolist()
    colval = dict(zip(cols, vals))
    load_values(ctx, colval, 6)
    b = {r: rng.choice(cols, n // 4, replace=False).tolist() for r in range(5)}
    load_set(ctx, SF[0], b)
    outside = (3 * SW + np.arange(40)).tolist()
    rows = {1: [c for c in cols if rng.random() < 0.01], 2: [c for c in cols if rng.random() < 0.9], 3: outside}
    load_set(ctx, FILT, rows)
    ctx.commit()
    values = sorted(set(vals))
    dims = [(sorted(b), b)]
    shards = [0, 1, 3]
    for row, keep in ((None, None), (1, set(rows[1])), (2, set(rows[2])), (3, set())):
        fo = None if row is None else filt(row)
        assert np.array_equal(gbv(ctx, dims, values, 6, shards, fo), expect(colval, dims, values, keep)), row
        assert np.array_equal(gbv(ctx, [], values, 6, shards, fo), expect(colval, [], values, keep)), row
    assert gbv(ctx, dims, values, 6, shards, filt(3)).sum() == 0


@gpu
def test_set_dimensions_zero_to_three(ctx):
    """0, 1, 2 and 3 set dimensions; the leading ones are peeled into the filter on the host"""
    rng = np.random.default_rng(13)
    n = 300 if ON_EMU else 2000
    cols = rng.choice(2 * SW, n, replace=False).tolist()
    vals = rng.integers(-20, 20, n).tolist()
    colval = dict(zip(cols, vals))
    load_values(ctx, colval, 5)
    sets = []
    for k, nr in enumerate((3, 4, 2)):
        m = {r: rng.choice(cols, n // 2, replace=False).tolist() for r in range(nr)}
        load_set(ctx, SF[k], m)
        sets.append((list(range(nr)), m))
    load_set(ctx, FILT, {1: cols[::2]})
    ctx.commit()
    values = sorted(set(vals))
    for nd in range(4):
        dims = sets[:nd]
        got = gbv(ctx, dims, values, 5, [0, 1])
        assert got.shape == tuple(len(r) for r, _ in dims) + (len(values),)
        assert np.array_equal(got, expect(colval, dims, values)), nd
        assert np.array_equal(gbv(ctx, dims, values, 5, [0, 1], filt(1)), expect(colval, dims, values, set(cols[::2]))), nd


@gpu
def test_sign_with_zero_magnitude_counts_nowhere(ctx):
    colval = {1: 0, 2: NEG0, 3: -1, 4: 0, 5: NEG0, 6: 1, SW + 7: NEG0}
    load_values(ctx, colval, 3)
    load_set(ctx, SF[0], {0: list(colval)})
    ctx.commit()
    got = gbv(ctx, [([0], {0: list(colval)})], [-1, 0, 1], 3, [0, 1])
    assert got.tolist() == [[1, 2, 1]]
    assert gbv(ctx, [], [0], 3, [0, 1]).tolist() == [2]


@gpu
def test_shards_missing_a_fragment(ctx):
    """shard 0 holds both fields, shard 1 only the int field, shard 2 only the set field"""
    colval = {5: 3, 6: 4, SW + 5: 3, SW + 6: 4}
    load_values(ctx, colval, 4)
    b = {0: [5, 6, 2 * SW + 5], 1: [6, 2 * SW + 6]}
    load_set(ctx, SF[0], b)
    ctx.commit()
    got = gbv(ctx, [([0, 1], b)], [3, 4], 4, [0, 1, 2])
    assert got.tolist() == [[1, 1], [0, 1]]
    assert gbv(ctx, [], [3, 4], 4, [0, 1, 2]).tolist() == [2, 2]


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch and kernel launch"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        rng = np.random.default_rng(14)
        n_sh = 3 if ON_EMU else 6
        cols = rng.choice(n_sh * SW, 900, replace=False).tolist()
        vals = rng.integers(-9, 9, len(cols)).tolist()
        colval = dict(zip(cols, vals))
        load_values(c, colval, 4)
        b = {r: rng.choice(cols, 300, replace=False).tolist() for r in range(3)}
        load_set(c, SF[0], b)
        load_set(c, FILT, {1: cols[::3]})
        c.commit()
        values = sorted(set(vals))
        dims = [(sorted(b), b)]
        shards = list(range(n_sh))
        assert np.array_equal(gbv(c, dims, values, 4, shards), expect(colval, dims, values))
        assert np.array_equal(gbv(c, [], values, 4, shards, filt(1)), expect(colval, [], values, set(cols[::3])))
    finally:
        c.close()


def _raw_call(lib, h, values, n_values=None, depth=4, n_fields=1, fields=None, n_rows=None, out=True, shards=True, n_shards=1, n_ops=0, ops=None):
    keep = [np.ascontiguousarray(np.asarray(values if values is not None else [], dtype=np.int64)), np.ones(8, dtype=np.uint32) * SF[0], np.zeros(8, dtype=np.uint32),
            np.zeros(8, dtype=np.uint64), np.zeros(1 << 16, dtype=np.uint64), np.zeros(1, dtype=np.uint64)]
    v, fl, vw, rows, o, sh = keep
    nr = np.ascontiguousarray(np.asarray(n_rows if n_rows is not None else [1] * 8, dtype=np.int32))
    return lib.fbgpu_groupby_values(h, IDX, fl.ctypes.data if fields is None else fields, vw.ctypes.data, n_fields, rows.ctypes.data, nr.ctypes.data,
                                    VF, VV, depth, v.ctypes.data if values is not None else None, len(v) if n_values is None else n_values, ops, n_ops,
                                    sh.ctypes.data if shards else None, n_shards, o.ctypes.data if out else None), o


ARG_ERRORS = [
    ({"values": [1, 1]}, "values are not strictly ascending at position 1"),
    ({"values": [3, 2]}, "values are not strictly ascending at position 1"),
    ({"values": [1], "n_values": 0}, "n_values=0 outside 1..65535"),
    ({"values": [1], "n_values": 65536}, "n_values=65536 outside 1..65535"),
    ({"values": [1], "depth": -1}, "bit depth -1 outside 0..64"),
    ({"values": [1], "depth": 65}, "bit depth 65 outside 0..64"),
    ({"values": [1], "n_fields": -1}, "bad argument"),
    ({"values": [1], "n_fields": 8}, "bad argument"),
    ({"values": None}, "bad argument"),
    ({"values": [1], "out": False}, "bad argument"),
    ({"values": [1], "shards": False}, "bad argument"),
    ({"values": [1], "n_shards": -1}, "bad argument"),
    ({"values": [1], "n_ops": 1}, "bad argument"),
    ({"values": [1], "n_ops": -1}, "bad argument"),
]


def test_argument_errors_before_the_device_check():
    """every argument error but n_rows is reported before the device check, on a context and on a node without a device"""
    ctx = L.Context(L.DEVICE_NONE)
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        for h, lib in ((ctx.h, ctx.L), (node.h, node.L)):
            for kw, msg in ARG_ERRORS:
                kw = dict(kw)
                rc, _ = _raw_call(lib, h, kw.pop("values"), **kw)
                assert rc == L.E_INVALID and lib.fbgpu_last_error().decode() == msg, (kw, msg)
        # n_fields == 0 takes no set-field arrays; the node checks n_rows before fanning out
        rc, _ = _raw_call(node.L, node.h, [1], n_fields=1, n_rows=[65536])
        assert rc == L.E_INVALID and node.L.fbgpu_last_error().decode() == "n_rows[0]=65536 out of range"
    finally:
        node.close()
        ctx.close()


def test_refused_on_an_inspection_only_context():
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for dims in ([], [[0, 1]]):
            with pytest.raises(L.FbgpuError) as e:
                ctx.groupby_values(IDX, [SF[0]] * len(dims), [0] * len(dims), dims, VF, VV, 4, [1, 2], [0])
            assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()


@gpu
def test_argument_errors_on_a_device(ctx):
    load_values(ctx, {1: 3}, 4)
    ctx.commit()
    rc, o = _raw_call(ctx.L, ctx.h, [3], n_fields=0, fields=0)                # no set field: the set-field arrays may be NULL
    assert rc == 0 and int(o[0]) == 1
    for kw, msg in ARG_ERRORS + [({"values": [1], "n_rows": [65536]}, "n_rows[0]=65536 out of range"), ({"values": [1], "n_rows": [-1]}, "n_rows[0]=-1 out of range")]:
        kw = dict(kw)
        rc, _ = _raw_call(ctx.L, ctx.h, kw.pop("values"), **kw)
        assert rc == L.E_INVALID and ctx.L.fbgpu_last_error().decode() == msg, (kw, msg)
    rc, o = _raw_call(ctx.L, ctx.h, [3], n_rows=[0])                          # an empty tensor: nothing written, no error
    assert rc == 0


# ------------------------------------------------------------------ query level
def _world(holder, seed, n):
    """index "g": set fields a (6 rows), b (4 rows), c (filter rows), int fields v over [-60, 60] and w over [1000, 1040]
    (Base 1000), some columns without a value, over three shards"""
    rng = np.random.default_rng(seed)
    idx = holder.create_index("g")
    for name in ("a", "b", "c"):
        idx.create_field(name)
    idx.create_field("v", "int", min=-60, max=60)
    idx.create_field("w", "int", min=1000, max=1040)
    cols = rng.choice(3 * SW, n, replace=False).tolist()
    for col in cols:
        for name, nr in (("a", 6), ("b", 4)):
            for r in range(nr):
                if rng.random() < 0.3:
                    holder.set_bit("g", name, r, col)
        if rng.random() < 0.4:
            holder.set_bit("g", "c", 0, col)
        if rng.random() < 0.9:
            holder.set_value("g", "v", col, int(rng.integers(-60, 61)))
        if rng.random() < 0.8:
            holder.set_value("g", "w", col, int(rng.integers(1000, 1041)))
    holder.sync()


QUERIES = [
    "GroupBy(Rows(v))",
    "GroupBy(Rows(w))",
    "GroupBy(Rows(v), Rows(a))",
    "GroupBy(Rows(a), Rows(v))",
    "GroupBy(Rows(a), Rows(w), Rows(b))",
    "GroupBy(Rows(a), Rows(b), Rows(v))",
    "GroupBy(Rows(v), Rows(a), Rows(b), filter=Row(c=0))",
    "GroupBy(Rows(a), Rows(v), filter=Row(c=0), limit=7)",
    "GroupBy(Rows(a, previous=2), Rows(v, previous=5), limit=9)",
    "GroupBy(Rows(v, previous=-3), Rows(b, previous=1), limit=4)",
    "GroupBy(Rows(a), Rows(w), having=Condition(count > 2))",
    'GroupBy(Rows(v), Rows(b), sort="count desc", limit=5)',
    'GroupBy(Rows(w), Rows(a), sort="count asc", offset=3, limit=6)',
    "GroupBy(Rows(b), Rows(w), aggregate=Sum(field=v), having=Condition(sum > 20))",
    'GroupBy(Rows(v), aggregate=Sum(field=w), sort="sum desc", limit=10)',
    "GroupBy(Rows(a), Rows(b), Rows(c), Rows(v), filter=Row(c=0))",
]


@gpu
def test_queries_match_the_composition():
    """the device path against an oracle-backed holder running the Row(v == value) composition: the int child first, in the
    middle and last, with filter, previous, limit, offset, having, sort and aggregate"""
    n = 150 if ON_EMU else 1500
    dev, ref = X.Holder(), X.Holder(ctx=OracleCtx())
    _world(dev, 21, n)
    _world(ref, 21, n)
    ed, er = X.Executor(dev), X.Executor(ref)
    assert not hasattr(ref.ctx, "groupby_values")
    try:
        for q in (QUERIES[:6] if ON_EMU else QUERIES):
            got = ed.execute("g", q)[0]
            assert got == er.execute("g", q)[0], q
            assert got or "having" in q, q
    finally:
        dev.ctx.close()


@gpu
def test_two_queries_and_no_scratch_rows():
    """GroupBy(Rows(v)) asks the library twice (the Distinct values, the counts) and GroupBy(Rows(a), Rows(v)) once more (a's
    row list), whatever the number of values; neither loads nor embeds anything"""
    h = X.Holder()
    try:
        _world(h, 22, 100 if ON_EMU else 600)
        ex = X.Executor(h)
        before_s = h.ctx.stats()
        for q, n_queries in (("GroupBy(Rows(v))", 2), ("GroupBy(Rows(a), Rows(v))", 3)):
            before_q = h.ctx.counters()["queries"]
            assert len(ex.execute("g", q)[0]) > 20, q
            assert h.ctx.counters()["queries"] - before_q == n_queries, q
        after = h.ctx.stats()
        assert (after["fragments"], after["payload_bytes"]) == (before_s["fragments"], before_s["payload_bytes"])
        assert X.SCRATCH_FIELD not in h.indexes["g"].fields
    finally:
        h.ctx.close()


@gpu
def test_node_answers_what_the_context_answers():
    """lib.Node with one device listed twice (shards alternate between its two contexts) sums the per-device tensors"""
    node, ctx = L.Node([0, 0], 1), L.Context(0)
    try:
        rng = np.random.default_rng(23)
        cols = rng.choice(4 * SW, 600 if ON_EMU else 4000, replace=False).tolist()
        vals = rng.integers(-30, 30, len(cols)).tolist()
        colval = dict(zip(cols, vals))
        sets = [{r: rng.choice(cols, len(cols) // 3, replace=False).tolist() for r in range(nr)} for nr in (3, 2)]
        for c in (node, ctx):
            load_values(c, colval, 5)
            for k, m in enumerate(sets):
                load_set(c, SF[k], m)
            load_set(c, FILT, {1: cols[::2]})
            c.commit()
        assert {node.owner(s) for s in range(4)} == {0, 1}
        values = sorted(set(vals))[1:]
        for nd in range(3):
            dims = [(sorted(m), m) for m in sets[:nd]]
            for fo, keep in ((None, None), (filt(1), set(cols[::2]))):
                got = gbv(node, dims, values, 5, [0, 1, 2, 3], fo)
                assert np.array_equal(got, gbv(ctx, dims, values, 5, [0, 1, 2, 3], fo)), nd
                assert np.array_equal(got, expect(colval, dims, values, keep)), nd
    finally:
        node.close()
        ctx.close()


# ------------------------------------------------------------------ CPU
def test_groupby_values_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_groupby_values.py"], timeout=3000)
