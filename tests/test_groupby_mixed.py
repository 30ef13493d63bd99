"""fbgpu_groupby_mixed (GroupBy over set dimensions and one or more int dimensions in one device call) and the GroupBy path built
on it.

Entry-point tests compare every count tensor with one the test computes from the columns and values it wrote, as plain Python
integers.  Query-level tests compare the executor's GroupBy with an oracle-backed holder, which has no groupby_mixed and so runs
the Row(v == value)-per-value composition over scratch rows.  The CPU tests check the argument errors and the refusal on a
context without a device, and run this file's gpu tests on the interpreted kernels."""
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
IDX, VV = 0, 7                         # index, the int fields' BSI view
VF = (5, 11, 12)                       # int fields
SF = (6, 8, 9)                         # set fields
VIEWS = (0, 3, 4)                      # views of the set fields
FILT = 10                              # set field of the filters
NEG0 = "-0"                            # a column stored as sign with magnitude 0
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
gpu = pytest.mark.gpu


def bsi_bytes(colval, depth):
    """one shard's BSI fragment: exists row 0, sign row 1, magnitude bit i in row 2 + i (NEG0: sign row only)"""
    bits = []
    for c, v in colval:
        o = int(c) % SW
        neg, mag = (True, 0) if v is NEG0 else (v < 0, abs(int(v)))
        bits.append(o)
        if neg:
            bits.append(SW + o)
        bits += [(2 + i) * SW + o for i in range(depth) if (mag >> i) & 1]
    return roaring_io.encode(np.unique(np.asarray(bits, dtype=np.uint64)))


def load_values(ctx, field, colval, depth):
    """colval: {absolute column: stored value or NEG0}; one BSI fragment per shard that holds a column"""
    per = {}
    for c, v in colval.items():
        per.setdefault(c // SW, []).append((c, v))
    for s, cv in per.items():
        ctx.load_fragment(IDX, field, VV, s, bsi_bytes(cv, depth))


def load_set(ctx, field, rows, view=0):
    """rows: {row id: absolute columns}; one fragment per shard"""
    per = {}
    for row, cols in rows.items():
        for c in cols:
            per.setdefault(int(c) // SW, []).append(row * SW + int(c) % SW)
    for s, bits in per.items():
        ctx.load_fragment(IDX, field, view, s, roaring_io.encode(np.unique(np.asarray(bits, dtype=np.uint64))))


class Dim:
    """a set dimension: field, its row list and, per listed view, {row: columns}; a row is its union over the views"""

    def __init__(self, field, rows, per_view, views=VIEWS):
        self.field, self.rows, self.per_view = field, rows, per_view
        self.views = [views[k] for k in range(len(per_view))]
        self.union = {}
        for m in per_view:
            for r, cols in m.items():
                self.union.setdefault(r, set()).update(int(c) for c in cols)

    def load(self, ctx):
        for view, m in zip(self.views, self.per_view):
            load_set(ctx, self.field, m, view)


def expect(ints, dims, values, keep=None):
    """the count tensor from the written data: ints = [{column: value}] per int field, values = their listed value lists"""
    out = np.zeros([len(d.rows) for d in dims] + [len(v) for v in values], dtype=np.uint64)
    pos = [{v: j for j, v in enumerate(vals)} for vals in values]
    for c in set(ints[0]).intersection(*ints[1:]):
        if keep is not None and c not in keep:
            continue
        js = []
        for cv, p in zip(ints, pos):
            v = cv[c]
            if v is NEG0 or v not in p:
                break
            js.append(p[v])
        else:
            for ix in itertools.product(*[[i for i, r in enumerate(d.rows) if c in d.union.get(r, ())] for d in dims]):
                out[ix + tuple(js)] += 1
    return out


def gbm(ctx, dims, depths, values, shards, filter_ops=None):
    return ctx.groupby_mixed(IDX, [(d.field, d.views, d.rows) for d in dims], [(VF[k], VV, depths[k], values[k]) for k in range(len(values))],
                             shards, filter_ops=filter_ops)


def filt(row):
    return [L.Op(L.OP_ROW, FILT, 0, 0, row, 0, 0, 0)]


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


# ------------------------------------------------------------------ entry point
def _pool(rng, depth, n):
    """n distinct values of a depth-bit field, its edge values first (INT64_MIN / INT64_MAX at depth 64)"""
    if depth == 64:
        edge = [I64_MIN, I64_MAX, -1, 0, 1]
    else:
        top = (1 << depth) - 1
        edge = sorted({-top, top, 0, -1, 1})
    pool = list(edge)
    n = min(n, 3) if depth == 1 else n                                       # a 1-bit field holds -1, 0 and 1 only
    while len(pool) < n:
        x = int(rng.integers(I64_MIN, I64_MAX, dtype=np.int64, endpoint=True)) if depth >= 63 else int(rng.integers(-((1 << depth) - 1), 1 << depth))
        if depth == 63:
            x = max(-((1 << 63) - 1), x)
        if x not in pool:
            pool.append(x)
    return pool[:n]


def _listed(rng, pool):
    """every other value of the pool (present ones left out) and some absent ones, ascending"""
    absent = [x for x in (I64_MIN, -7777, 3, 12345, I64_MAX) if x not in pool]
    return sorted(set(pool[::2] + absent[:3]))


@gpu
@pytest.mark.parametrize("depth", [1, 8, 32, 63, 64])
def test_depths_with_edge_values(ctx, depth):
    """2 and 3 int fields of one depth over two shards (a third listed shard holds nothing), grouped alone and under one
    and two set dimensions; value lists include absent values and leave present ones out, some columns are stored as sign
    with magnitude 0.  Three fields of depth 63 or 64 have more planes than the per-unit table holds and are resolved per
    range; two of depth 64 fit it."""
    rng = np.random.default_rng(depth)
    n = 150 if ON_EMU else 600
    cols = rng.choice(2 * SW, n, replace=False).tolist()
    ints = []
    for k in range(3):
        pool = _pool(rng, depth, 6)
        cv = {c: pool[int(rng.integers(len(pool)))] for c in cols if rng.random() < 0.9}
        for c in list(cv)[:3]:
            cv[c] = NEG0
        ints.append((cv, _listed(rng, pool)))
        load_values(ctx, VF[k], cv, depth)
    dims = [Dim(SF[0], [0, 1, 2, 9], [{r: rng.choice(cols, n // 3, replace=False).tolist() for r in range(3)}]),
            Dim(SF[1], [0, 1], [{r: rng.choice(cols, n // 2, replace=False).tolist() for r in range(2)}])]
    for d in dims:
        d.load(ctx)
    ctx.commit()
    shards = [0, 1, 4]
    for ni in (2, 3):
        cv, vals = [c for c, _ in ints[:ni]], [v for _, v in ints[:ni]]
        for nd in (0, 1, 2):
            got = gbm(ctx, dims[:nd], [depth] * ni, vals, shards)
            want = expect(cv, dims[:nd], vals)
            assert np.array_equal(got, want), (ni, nd)
            assert want.sum() > 0


@gpu
@pytest.mark.parametrize("layout", ["bitmap", "run", "array"])
def test_container_encodings(ctx, layout):
    """planes and set rows stored as bitmaps (dense random columns), runs (contiguous columns, values in long stretches) and
    arrays (scattered columns, bank-striped); the set dimension has two views"""
    rng = np.random.default_rng(11)
    n = 20000 if ON_EMU else 60000
    if layout == "bitmap":
        cols = (np.sort(rng.choice(SW // 8, n, replace=False)) + 3 * 65536).tolist()
        vs = [rng.integers(-30, 30, n).tolist(), rng.integers(0, 40, n).tolist()]
        views = [{r: [c for c in cols if rng.random() < 0.5] for r in range(2)} for _ in range(2)]
    elif layout == "run":
        cols = list(range(100, 100 + n))
        vs = [np.repeat(rng.integers(-(1 << 20), 1 << 20, n // 1000), 1000).tolist(), np.repeat(rng.integers(0, 9, n // 2500), 2500).tolist()]
        views = [{0: cols[: n // 2], 1: cols[n // 3: n // 3 + 7000]}, {0: cols[n // 4: n // 2 + 3000], 1: cols[5000: 5100]}]
    else:
        cols = rng.choice(3 * SW, 3000 if ON_EMU else 9000, replace=False).tolist()
        vs = [rng.integers(-300, 300, len(cols)).tolist(), rng.integers(0, 30, len(cols)).tolist()]
        views = [{r: rng.choice(cols, len(cols) // 2, replace=False).tolist() for r in range(3)} for _ in range(2)]      # >= 64 per slot: bank-striped
    ints = [dict(zip(cols, v)) for v in vs]
    for k, cv in enumerate(ints):
        load_values(ctx, VF[k], cv, 21)
    d = Dim(SF[0], sorted(views[0]), views)
    d.load(ctx)
    ctx.commit()
    values = [sorted(set(v)) for v in vs]
    values[0] = values[0][: 65535 // len(values[1])]
    shards = [0, 1, 2]
    for dims in ([d], []):
        got = gbm(ctx, dims, [21, 21], values, shards)
        assert np.array_equal(got, expect(ints, dims, values)), len(dims)


def _set_world(ctx, rng, n):
    """two int fields over two shards, three set fields with 1, 2 and 3 views (a column in several views of one row), a filter
    field with a sparse, a dense and an empty row"""
    cols = rng.choice(2 * SW, n, replace=False).tolist()
    ints = [{c: int(rng.integers(-6, 6)) for c in cols if rng.random() < 0.9}, {c: int(rng.integers(100, 105)) for c in cols if rng.random() < 0.85}]
    for k, cv in enumerate(ints):
        load_values(ctx, VF[k], cv, 8)
    dims = []
    for k, (nr, nv) in enumerate(((3, 1), (4, 2), (2, 3))):
        base = {r: rng.choice(cols, n // 3, replace=False).tolist() for r in range(nr)}
        per_view = [{r: [c for c in cs if rng.random() < 0.6] for r, cs in base.items()} for _ in range(nv)]
        d = Dim(SF[k], list(range(nr)) + [7], per_view)              # row 7 holds nothing
        d.load(ctx)
        dims.append(d)
    outside = (3 * SW + np.arange(40)).tolist()
    rows = {1: [c for c in cols if rng.random() < 0.02], 2: [c for c in cols if rng.random() < 0.9], 3: outside}
    load_set(ctx, FILT, rows)
    ctx.commit()
    values = [sorted(set(ints[0].values()))[1:] + [50], sorted(set(ints[1].values()))]
    return ints, dims, values, rows


@gpu
def test_set_dimensions_views_and_filters(ctx):
    """0-2 set dimensions with 1-3 views each, in every order (so a multi-view dimension is peeled and is the kernel's last
    one), under no filter and a sparse, a dense and an empty filter"""
    rng = np.random.default_rng(13)
    ints, dims, values, rows = _set_world(ctx, rng, 300 if ON_EMU else 2000)
    shards = [0, 1, 3]
    orders = [(), (0,), (1,), (2,), (0, 2), (2, 1)] if ON_EMU else [()] + [p for k in (1, 2) for p in itertools.permutations(range(3), k)]
    for order in orders:
        ds = [dims[k] for k in order]
        for row, keep in ((None, None), (1, set(rows[1])), (2, set(rows[2])), (3, set())):
            got = gbm(ctx, ds, [8, 8], values, shards, None if row is None else filt(row))
            assert got.shape == tuple(len(d.rows) for d in ds) + tuple(len(v) for v in values)
            assert np.array_equal(got, expect(ints, ds, values, keep)), (order, row)


@gpu
def test_more_views_than_a_warp_resolves_at_once(ctx):
    """a set dimension of 40 views (the kernel resolves a row's views 32 at a time, so two rounds), every column of a row in
    one to three of them and some views empty in a shard; as the last dimension and peeled before another one"""
    rng = np.random.default_rng(17)
    n = 300 if ON_EMU else 3000
    ints, dims, values, rows = _set_world(ctx, rng, n)
    cols = sorted(set(ints[0]) | set(ints[1]))
    per_view = [{} for _ in range(40)]
    for r in range(4):
        for c in rng.choice(cols, len(cols) // 3, replace=False).tolist():
            for k in rng.choice(40, int(rng.integers(1, 4)), replace=False).tolist():
                per_view[k].setdefault(r, []).append(c)
    per_view[33] = {0: [c for c in cols if c >= SW][:50]}                  # a view of the second round with columns in one shard only
    wide = Dim(SF[2] + 20, [0, 1, 2, 3, 5], per_view, views=list(range(20, 60)))
    wide.load(ctx)
    ctx.commit()
    for ds in ([wide], [wide, dims[0]], [dims[1], wide]):
        for fo, keep in ((None, None), (filt(2), set(rows[2]))):
            got = gbm(ctx, ds, [8, 8], values, [0, 1, 2], fo)
            assert np.array_equal(got, expect(ints, ds, values, keep)), ([d.field for d in ds], keep is None)


@gpu
def test_shards_missing_a_fragment(ctx):
    """shard 0 holds everything, shard 1 lacks w's fragment, shard 2 lacks the set field in both of its views; shard 3 lacks
    the set field in one view only and still counts"""
    cols = [5, 6, SW + 5, SW + 6, 2 * SW + 5, 3 * SW + 5]
    v = {c: 3 for c in cols}
    w = {c: 4 for c in cols if c // SW != 1}
    load_values(ctx, VF[0], v, 4)
    load_values(ctx, VF[1], w, 4)
    d = Dim(SF[0], [0], [{0: [5, 6, SW + 5, SW + 6]}, {0: [6, SW + 6, 3 * SW + 5]}])
    d.load(ctx)
    ctx.commit()
    got = gbm(ctx, [d], [4, 4], [[3], [4]], [0, 1, 2, 3])
    assert got.tolist() == [[[3]]]
    assert gbm(ctx, [], [4, 4], [[3], [4]], [0, 1, 2, 3]).tolist() == [[4]]


@gpu
def test_zero_rows(ctx):
    load_values(ctx, VF[0], {1: 3}, 4)
    load_values(ctx, VF[1], {1: 3}, 4)
    ctx.commit()
    d = Dim(SF[0], [], [{}])
    got = gbm(ctx, [d], [4, 4], [[3], [3]], [0])
    assert got.shape == (0, 1, 1)
    assert gbm(ctx, [Dim(SF[0], [0], [{}]), d], [4, 4], [[3], [3]], [0]).shape == (1, 0, 1, 1)


@gpu
def test_one_int_field_is_groupby_values(ctx):
    """n_ints == 1 with single views: bit for bit what fbgpu_groupby_values returns, with 0-2 set dimensions and filters, and
    both equal to the tensor computed from the written data"""
    rng = np.random.default_rng(14)
    ints, dims, values, rows = _set_world(ctx, rng, 300 if ON_EMU else 2000)
    single = [dims[0], Dim(SF[1], dims[1].rows, dims[1].per_view[:1])]
    for nd in range(3):
        ds = single[:nd]
        for fo, keep in ((None, None), (filt(1), set(rows[1])), (filt(2), set(rows[2]))):
            got = gbm(ctx, ds, [8], values[:1], [0, 1, 2], fo)
            ref = ctx.groupby_values(IDX, [d.field for d in ds], [d.views[0] for d in ds], [d.rows for d in ds], VF[0], VV, 8, values[0], [0, 1, 2], filter_ops=fo)
            assert got.dtype == ref.dtype and got.shape == ref.shape and got.tobytes() == ref.tobytes(), nd
            assert np.array_equal(got, expect(ints[:1], ds, values[:1], keep)), nd


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch and kernel launch"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        rng = np.random.default_rng(15)
        ints, dims, values, rows = _set_world(c, rng, 300 if ON_EMU else 1500)
        assert np.array_equal(gbm(c, dims[1:2], [8, 8], values, [0, 1, 2]), expect(ints, dims[1:2], values))
        assert np.array_equal(gbm(c, [], [8, 8], values, [0, 1, 2], filt(2)), expect(ints, [], values, set(rows[2])))
    finally:
        c.close()


@gpu
def test_node_answers_what_the_context_answers():
    """lib.Node with one device listed twice (shards alternate between its two contexts) sums the per-device tensors"""
    node, ctx = L.Node([0, 0], 1), L.Context(0)
    try:
        for c in (node, ctx):
            ints, dims, values, rows = _set_world(c, np.random.default_rng(16), 300 if ON_EMU else 2000)
        assert {node.owner(s) for s in range(2)} == {0, 1}
        for ds in ([], dims[1:2], dims[:2]):
            for fo, keep in ((None, None), (filt(2), set(rows[2]))):
                got = gbm(node, ds, [8, 8], values, [0, 1, 2], fo)
                assert np.array_equal(got, gbm(ctx, ds, [8, 8], values, [0, 1, 2], fo)), len(ds)
                assert np.array_equal(got, expect(ints, ds, values, keep)), len(ds)
    finally:
        node.close()
        ctx.close()


# ------------------------------------------------------------------ argument errors
def _raw_call(lib, h, n_fields=1, n_views=None, n_rows=None, n_ints=2, depths=None, n_values=None, values=None, null=None, n_shards=1):
    keep = dict(fields=np.full(8, SF[0], dtype=np.uint32), views=np.zeros(64, dtype=np.uint32),
                n_views=np.asarray(n_views if n_views is not None else [1] * 8, dtype=np.int32),
                rows=np.zeros(64, dtype=np.uint64), n_rows=np.asarray(n_rows if n_rows is not None else [1] * 8, dtype=np.int32),
                vfields=np.asarray(VF + VF + VF[:2], dtype=np.uint32), vviews=np.full(8, VV, dtype=np.uint32),
                depths=np.asarray(depths if depths is not None else [4] * 8, dtype=np.int32),
                values=np.asarray(values if values is not None else list(range(1 << 17)), dtype=np.int64),
                n_values=np.asarray(n_values if n_values is not None else [2] * 8, dtype=np.int32),
                shards=np.zeros(1, dtype=np.uint64), out=np.zeros(1 << 16, dtype=np.uint64))
    p = {k: (None if k == null else a.ctypes.data) for k, a in keep.items()}
    rc = lib.fbgpu_groupby_mixed(h, IDX, p["fields"], p["views"], p["n_views"], n_fields, p["rows"], p["n_rows"], p["vfields"], p["vviews"], p["depths"], n_ints,
                                 p["values"], p["n_values"], None, 0, p["shards"], n_shards, p["out"])
    return rc, keep["out"]


ARG_ERRORS = [
    ({"n_values": [300, 300]}, "product of n_values 90000 exceeds 65535"),
    ({"n_values": [65535, 2]}, "product of n_values 131070 exceeds 65535"),
    ({"n_fields": 5, "n_ints": 4}, "n_fields + n_ints = 9 exceeds 8"),
    ({"n_fields": 0, "n_ints": 9}, "n_ints=9 outside 1..8"),
    ({"n_ints": 0}, "n_ints=0 outside 1..8"),
    ({"n_fields": 8, "n_ints": 1}, "n_fields=8 outside 0..7"),
    ({"n_fields": -1}, "n_fields=-1 outside 0..7"),
    ({"n_fields": 2, "n_views": [1, 0]}, "n_views[1]=0 < 1"),
    ({"values": [1, 2, 5, 5]}, "values[1] are not strictly ascending at position 1"),
    ({"values": [1, 2, 5, 6, 7, 9, 8], "n_values": [2, 5]}, "values[1] are not strictly ascending at position 4"),
    ({"values": [2, 1]}, "values[0] are not strictly ascending at position 1"),
    ({"n_values": [2, 0]}, "n_values[1]=0 outside 1..65535"),
    ({"n_values": [65536, 1]}, "n_values[0]=65536 outside 1..65535"),
    ({"depths": [4, 65]}, "bit_depths[1]=65 outside 0..64"),
    ({"depths": [-1, 4]}, "bit_depths[0]=-1 outside 0..64"),
    ({"n_shards": -1}, "bad argument"),
] + [({"null": k}, "bad argument") for k in ("fields", "views", "n_views", "rows", "n_rows", "vfields", "vviews", "depths", "values", "n_values", "shards", "out")]


def test_argument_errors_before_the_device_check():
    """every argument error but n_rows is reported before the device check, on a context and on a node without a device"""
    ctx = L.Context(L.DEVICE_NONE)
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        for h, lib in ((ctx.h, ctx.L), (node.h, node.L)):
            for kw, msg in ARG_ERRORS:
                rc, _ = _raw_call(lib, h, **kw)
                assert rc == L.E_INVALID and lib.fbgpu_last_error().decode() == msg, (kw, msg)
        rc, _ = _raw_call(ctx.L, ctx.h, n_fields=0, null="fields")             # no set dimension: the set arrays may be NULL
        assert rc == L.E_CUDA and "no device" in ctx.L.fbgpu_last_error().decode()
        rc, _ = _raw_call(node.L, node.h, n_rows=[65536])                        # the node checks n_rows before fanning out
        assert rc == L.E_INVALID and node.L.fbgpu_last_error().decode() == "n_rows[0]=65536 out of range"
    finally:
        node.close()
        ctx.close()


def test_refused_on_an_inspection_only_context():
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for dims in ([], [(SF[0], [0], [0, 1])]):
            with pytest.raises(L.FbgpuError) as e:
                ctx.groupby_mixed(IDX, dims, [(VF[0], VV, 4, [1, 2]), (VF[1], VV, 4, [3])], [0])
            assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()


@gpu
def test_argument_errors_on_a_device(ctx):
    load_values(ctx, VF[0], {1: 0}, 4)
    load_values(ctx, VF[1], {1: 3}, 4)
    ctx.commit()
    rc, o = _raw_call(ctx.L, ctx.h, n_fields=0, null="fields")             # values [0, 1] x [2, 3]: the column is in group (0, 1)
    assert rc == 0 and o[:4].tolist() == [0, 1, 0, 0]
    for kw, msg in ARG_ERRORS + [({"n_rows": [65536]}, "n_rows[0]=65536 out of range"), ({"n_rows": [-1]}, "n_rows[0]=-1 out of range")]:
        rc, _ = _raw_call(ctx.L, ctx.h, **kw)
        assert rc == L.E_INVALID and ctx.L.fbgpu_last_error().decode() == msg, (kw, msg)
    rc, _ = _raw_call(ctx.L, ctx.h, n_rows=[0])                              # an empty tensor: nothing written, no error
    assert rc == 0


# ------------------------------------------------------------------ query level
def _world(holder, seed, n):
    """index "g": set fields a (5 rows), b (3 rows), c (filter rows), int fields v over [-8, 8], w over [1000, 1012] (Base 1000)
    and u over [0, 5], a quantum-YMD time field t (4 rows), some columns without a value, over three shards"""
    rng = np.random.default_rng(seed)
    idx = holder.create_index("g")
    for name in ("a", "b", "c"):
        idx.create_field(name)
    idx.create_field("t", "time", quantum="YMD")
    idx.create_field("v", "int", min=-8, max=8)
    idx.create_field("w", "int", min=1000, max=1012)
    idx.create_field("u", "int", min=0, max=5)
    cols = rng.choice(3 * SW, n, replace=False).tolist()
    for col in cols:
        for name, nr in (("a", 5), ("b", 3)):
            for r in range(nr):
                if rng.random() < 0.3:
                    holder.set_bit("g", name, r, col)
        for r in range(4):
            if rng.random() < 0.35:
                holder.set_bit("g", "t", r, col, timestamp=f"2019-{int(rng.integers(1, 5)):02d}-{int(rng.integers(1, 28)):02d}T00:00")
        if rng.random() < 0.4:
            holder.set_bit("g", "c", 0, col)
        for name, lo, hi, p in (("v", -8, 8, 0.9), ("w", 1000, 1012, 0.8), ("u", 0, 5, 0.7)):
            if rng.random() < p:
                holder.set_value("g", name, col, int(rng.integers(lo, hi + 1)))
    holder.sync()


TR = "from=2019-01-20T00:00, to=2019-03-10T00:00"
QUERIES = [
    "GroupBy(Rows(v), Rows(w))",
    "GroupBy(Rows(a), Rows(v), Rows(w))",
    "GroupBy(Rows(a), Rows(v), Rows(w), filter=Row(c=0))",
    "GroupBy(Rows(v), Rows(a), Rows(w))",
    "GroupBy(Rows(v), Rows(w), Rows(a))",
    "GroupBy(Rows(w), Rows(a), Rows(b), Rows(u))",
    "GroupBy(Rows(u), Rows(v), Rows(w))",
    f"GroupBy(Rows(t, {TR}), Rows(v))",
    f"GroupBy(Rows(v), Rows(t, {TR}), filter=Row(c=0))",
    f"GroupBy(Rows(t, {TR}), Rows(a), Rows(v), Rows(w))",
    "GroupBy(Rows(a, previous=2), Rows(v, previous=3), Rows(w, previous=1005), limit=9)",
    "GroupBy(Rows(v), Rows(w), limit=7, offset=3)",
    "GroupBy(Rows(a), Rows(w), Rows(v), having=Condition(count > 2))",
    'GroupBy(Rows(v), Rows(u), sort="count desc", limit=5)',
    "GroupBy(Rows(b), Rows(w), Rows(u), aggregate=Sum(field=v), having=Condition(sum > 5))",
    'GroupBy(Rows(v), Rows(w), aggregate=Sum(field=u), sort="sum desc", limit=10)',
]


def _pair(seed, n):
    dev, ref = X.Holder(), X.Holder(ctx=OracleCtx())
    _world(dev, seed, n)
    _world(ref, seed, n)
    assert not hasattr(ref.ctx, "groupby_mixed")
    return dev, X.Executor(dev), X.Executor(ref)


@gpu
def test_queries_match_the_composition():
    """the device path against an oracle-backed holder running the composition: two and three int children first, in the
    middle and last, beside set and time-range children, with filter, previous, limit, offset, having, sort and aggregate"""
    dev, ed, er = _pair(21, 150 if ON_EMU else 1500)
    try:
        for q in (QUERIES[:3] + QUERIES[7:8] if ON_EMU else QUERIES):
            got = ed.execute("g", q)[0]
            assert got == er.execute("g", q)[0], q
            assert got or "having" in q, q
    finally:
        dev.ctx.close()


@gpu
def test_slices_tile_the_tensor(monkeypatch):
    """with the groups-per-call cap lowered, the value lists are cut into slices and every combination is one call; the
    result is the composition's"""
    dev, ed, er = _pair(22, 150 if ON_EMU else 1000)
    calls = []
    real = dev.ctx.groupby_mixed
    monkeypatch.setattr(dev.ctx, "groupby_mixed", lambda *a, **kw: calls.append(a[2]) or real(*a, **kw), raising=False)
    try:
        for cap in ((40,) if ON_EMU else (7, 40)):
            monkeypatch.setattr(X.Executor, "GROUPBY_MIXED_MAX", cap)
            for q in ("GroupBy(Rows(a), Rows(v), Rows(w))", "GroupBy(Rows(u), Rows(w), Rows(v), filter=Row(c=0))")[:1 if ON_EMU else 2]:
                calls.clear()
                got = ed.execute("g", q)[0]
                assert got == er.execute("g", q)[0], (cap, q)
                assert len(calls) > 1 and all(np.prod([len(d[3]) for d in c]) <= cap for c in calls), (cap, q)
    finally:
        dev.ctx.close()


@gpu
def test_bounded_calls_and_no_scratch_rows():
    """GroupBy(Rows(v), Rows(w)) asks the library three times (two Distincts, the counts) and GroupBy(Rows(a), Rows(v), Rows(w))
    once more (a's row list), whatever the number of values; neither loads nor embeds anything"""
    h = X.Holder()
    try:
        _world(h, 23, 100 if ON_EMU else 600)
        ex = X.Executor(h)
        before_s = h.ctx.stats()
        for q, n_queries in (("GroupBy(Rows(v), Rows(w))", 3), ("GroupBy(Rows(a), Rows(v), Rows(w))", 4)):
            before_q = h.ctx.counters()["queries"]
            assert len(ex.execute("g", q)[0]) > 20, q
            assert h.ctx.counters()["queries"] - before_q == n_queries, q
        after = h.ctx.stats()
        assert (after["fragments"], after["payload_bytes"]) == (before_s["fragments"], before_s["payload_bytes"])
        assert X.SCRATCH_FIELD not in h.indexes["g"].fields
    finally:
        h.ctx.close()


# ------------------------------------------------------------------ CPU
def test_groupby_mixed_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_groupby_mixed.py"], timeout=3000)
