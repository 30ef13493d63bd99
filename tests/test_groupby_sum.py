"""fbgpu_groupby_sum (GroupBy(..., aggregate=Sum(field=x)) in one device call) and the GroupBy path built on it.

Entry-point tests compare the count and sum tensors with ones the test computes from the columns and values it wrote, as plain
Python integers, and every cell of a small world with fbgpu_bsi_sum under the cell's filter.  Query-level tests compare the
executor's GroupBy with an oracle-backed holder, which has no groupby_sum and so runs one Sum per non-empty group.  The CPU
tests check the argument errors and the refusal on a context without a device, and run this file's gpu tests on the
interpreted kernels."""
import itertools

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from tests.oracle_ctx import OracleCtx
from tests.test_groupby_mixed import I64_MAX, IDX, NEG0, ON_EMU, SF, SW, VF, VV, Dim, _pool, _set_world, _world, filt, load_values

AF = 13                                # the aggregate field (BSI view VV)
gpu = pytest.mark.gpu


def _wrap(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


def expect(agg, ints, dims, values, keep=None):
    """(counts, sums) from the written data: agg = {column: stored value or NEG0} of the aggregate field, ints = [{column: value}]
    per int dimension with `values` its listed value lists"""
    shape = [len(d.rows) for d in dims] + [len(v) for v in values]
    counts = np.zeros(shape, dtype=np.uint64)
    sums = np.zeros(shape, dtype=object)
    sums.fill(0)
    pos = [{v: j for j, v in enumerate(vals)} for vals in values]
    for c, x in agg.items():
        if keep is not None and c not in keep:
            continue
        js = []
        for cv, p in zip(ints, pos):
            v = cv.get(c)
            if v is None or v is NEG0 or v not in p:
                break
            js.append(p[v])
        else:
            for ix in itertools.product(*[[i for i, r in enumerate(d.rows) if c in d.union.get(r, ())] for d in dims]):
                counts[ix + tuple(js)] += 1
                sums[ix + tuple(js)] += 0 if x is NEG0 else x
    return counts, np.vectorize(_wrap, otypes=[np.int64])(sums) if sums.size else sums.astype(np.int64)


def gbs(ctx, dims, int_depths, values, depth, shards, filter_ops=None, afield=AF):
    return ctx.groupby_sum(IDX, [(d.field, d.views, d.rows) for d in dims], [(VF[k], VV, int_depths[k], values[k]) for k in range(len(values))],
                           (afield, VV, depth), shards, filter_ops=filter_ops)


def check(got, want, what):
    assert got[0].shape == want[0].shape and got[1].shape == want[1].shape, what
    assert got[0].dtype == np.uint64 and got[1].dtype == np.int64, what
    assert np.array_equal(got[0], want[0]), what
    assert np.array_equal(got[1], want[1]), what


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


# ------------------------------------------------------------------ entry point
@gpu
@pytest.mark.parametrize("depth", [1, 8, 32, 63, 64])
def test_depths_with_edge_values(ctx, depth):
    """an aggregate of each depth holding its edge values (INT64_MIN / INT64_MAX at depth 64) and sign with magnitude 0, over two
    shards (a third listed shard holds nothing), grouped by 0-2 set dimensions and 0-2 int dimensions; at depths 63 and 64 one
    group's sum wraps"""
    rng = np.random.default_rng(100 + depth)
    n = 150 if ON_EMU else 600
    cols = rng.choice(2 * SW, n, replace=False).tolist()
    pool = _pool(rng, depth, 8)
    agg = {c: pool[int(rng.integers(len(pool)))] for c in cols if rng.random() < 0.9}
    for c in list(agg)[:3]:
        agg[c] = NEG0
    ints = [{c: int(rng.integers(-3, 3)) for c in cols if rng.random() < 0.9}, {c: int(rng.integers(0, 4)) for c in cols if rng.random() < 0.9}]
    if depth >= 63:                                             # group (-3, 7) holds five columns of the largest value and no other
        for c in cols[-5:]:
            agg[c], ints[0][c], ints[1][c] = I64_MAX, -3, 7
    load_values(ctx, AF, agg, depth)
    for k, cv in enumerate(ints):
        load_values(ctx, VF[k], cv, 8)
    dims = [Dim(SF[0], [0, 1, 2, 9], [{r: rng.choice(cols, n // 3, replace=False).tolist() for r in range(3)}]),
            Dim(SF[1], [0, 1], [{r: rng.choice(cols, n // 2, replace=False).tolist() for r in range(2)}])]
    for d in dims:
        d.load(ctx)
    ctx.commit()
    values = [[-3, -2, -1, 0, 1, 2], [0, 1, 3, 7]]
    shards = [0, 1, 4]
    for ni in (0, 1, 2):
        for nd in (0, 1, 2):
            if ni + nd == 0:
                continue
            got = gbs(ctx, dims[:nd], [8] * ni, values[:ni], depth, shards)
            check(got, expect(agg, ints[:ni], dims[:nd], values[:ni]), (ni, nd))
            assert got[0].sum() > 0
    if depth >= 63:
        c, s = gbs(ctx, [], [8, 8], values, depth, shards)
        assert (int(c[0, 3]), int(s[0, 3])) == (5, _wrap(5 * I64_MAX)) == (5, I64_MAX - 4)


@gpu
@pytest.mark.parametrize("layout", ["bitmap", "run", "array"])
def test_container_encodings(ctx, layout):
    """the aggregate's planes, an int dimension's planes and set rows stored as bitmaps (dense random columns), runs (contiguous
    columns, values in long stretches) and arrays (scattered columns, bank-striped); the set dimension has two views"""
    rng = np.random.default_rng(111)
    n = 20000 if ON_EMU else 60000
    if layout == "bitmap":
        cols = (np.sort(rng.choice(SW // 8, n, replace=False)) + 3 * 65536).tolist()
        xs, vs = rng.integers(-(1 << 20), 1 << 20, n).tolist(), rng.integers(0, 40, n).tolist()
        views = [{r: [c for c in cols if rng.random() < 0.5] for r in range(2)} for _ in range(2)]
    elif layout == "run":
        cols = list(range(100, 100 + n))
        xs, vs = np.repeat(rng.integers(-(1 << 20), 1 << 20, n // 1000), 1000).tolist(), np.repeat(rng.integers(0, 9, n // 2500), 2500).tolist()
        views = [{0: cols[: n // 2], 1: cols[n // 3: n // 3 + 7000]}, {0: cols[n // 4: n // 2 + 3000], 1: cols[5000: 5100]}]
    else:
        cols = rng.choice(3 * SW, 3000 if ON_EMU else 9000, replace=False).tolist()
        xs, vs = rng.integers(-300, 300, len(cols)).tolist(), rng.integers(0, 30, len(cols)).tolist()
        views = [{r: rng.choice(cols, len(cols) // 2, replace=False).tolist() for r in range(3)} for _ in range(2)]      # >= 64 per slot: bank-striped
    agg, ints = dict(zip(cols, xs)), [dict(zip(cols, vs))]
    load_values(ctx, AF, agg, 21)
    load_values(ctx, VF[0], ints[0], 21)
    d = Dim(SF[0], sorted(views[0]), views)
    d.load(ctx)
    ctx.commit()
    values = [sorted(set(vs))]
    shards = [0, 1, 2]
    for dims, ni in (([d], 1), ([d], 0), ([], 1)):
        check(gbs(ctx, dims, [21] * ni, values[:ni], 21, shards), expect(agg, ints[:ni], dims, values[:ni]), (len(dims), ni))


def _agg_world(ctx, rng, n):
    """_set_world (two int fields, three set fields of 1-3 views, filter rows) plus an aggregate field of depth 40 on most columns"""
    ints, dims, values, rows = _set_world(ctx, rng, n)
    cols = sorted(set(ints[0]) | set(ints[1]))
    agg = {c: int(rng.integers(-(1 << 40) + 1, 1 << 40)) for c in cols if rng.random() < 0.85}
    for c in cols[:4]:
        agg[c] = NEG0
    load_values(ctx, AF, agg, 40)
    ctx.commit()
    return agg, ints, dims, values, rows


@gpu
def test_set_dimensions_views_and_filters(ctx):
    """0-3 set dimensions with 1-3 views each in several orders, beside 0-2 int dimensions, under no filter and a sparse, a dense
    and an empty filter"""
    rng = np.random.default_rng(113)
    agg, ints, dims, values, rows = _agg_world(ctx, rng, 300 if ON_EMU else 2000)
    shards = [0, 1, 3]
    orders = [(0,), (2,), (1, 2), (2, 1, 0)] if ON_EMU else [p for k in (1, 2, 3) for p in itertools.permutations(range(3), k)]
    filters = ((None, None), (2, set(rows[2]))) if ON_EMU else ((None, None), (1, set(rows[1])), (2, set(rows[2])), (3, set()))
    for order in [()] + orders:
        ds = [dims[k] for k in order]
        for ni in ((1, 2) if not ds else (0, 1, 2)):
            for row, keep in filters:
                got = gbs(ctx, ds, [8] * ni, values[:ni], 40, shards, None if row is None else filt(row))
                check(got, expect(agg, ints[:ni], ds, values[:ni], keep), (order, ni, row))


@gpu
def test_aggregate_is_also_a_group_dimension(ctx):
    """GroupBy(Rows(a), Rows(v), aggregate=Sum(field=v)): every cell sums its own value"""
    rng = np.random.default_rng(114)
    ints, dims, values, rows = _set_world(ctx, rng, 300 if ON_EMU else 2000)
    for ds in ([], dims[:1], dims[1:2]):
        got = gbs(ctx, ds, [8], values[:1], 8, [0, 1, 2], afield=VF[0])
        check(got, expect(ints[0], ints[:1], ds, values[:1]), len(ds))
        want_sums = got[0].astype(object) * np.asarray(values[0], dtype=object)
        assert np.array_equal(got[1], want_sums.astype(np.int64))


@gpu
def test_plane_table_overflow(ctx):
    """two depth-64 int dimensions and a depth-64 aggregate need 195 plane-table entries, more than the 184 the kernel holds:
    every field's planes are resolved per range.  Two depth-64 int fields with a depth-8 aggregate (139 entries) fit."""
    rng = np.random.default_rng(115)
    n = 200 if ON_EMU else 1500
    cols = rng.choice(2 * SW, n, replace=False).tolist()
    pools = [_pool(rng, 64, 5), _pool(rng, 64, 4)]
    ints = [{c: p[int(rng.integers(len(p)))] for c in cols if rng.random() < 0.9} for p in pools]
    big = {c: _pool(rng, 64, 6)[int(rng.integers(6))] for c in cols if rng.random() < 0.9}
    small = {c: int(rng.integers(-255, 256)) for c in cols}
    for k, cv in enumerate(ints):
        load_values(ctx, VF[k], cv, 64)
    load_values(ctx, AF, big, 64)
    load_values(ctx, AF + 1, small, 8)
    d = Dim(SF[0], [0, 1], [{r: rng.choice(cols, n // 2, replace=False).tolist() for r in range(2)}])
    d.load(ctx)
    ctx.commit()
    values = [sorted(p) for p in pools]
    for ds in ([], [d]):
        check(gbs(ctx, ds, [64, 64], values, 64, [0, 1]), expect(big, ints, ds, values), ("195", len(ds)))
        check(gbs(ctx, ds, [64, 64], values, 8, [0, 1], afield=AF + 1), expect(small, ints, ds, values), ("139", len(ds)))


def _cell_ops(dims, depths, values, ix, base=None):
    """the program of filter ∩ the cell's rows: each set row as its union over the views, each int value as Row(v == value)"""
    ops = list(base or [])
    n = 1 if base else 0
    for d, i in zip(dims, ix):
        for v in d.views:
            ops.append(L.Op(L.OP_ROW, d.field, v, 0, d.rows[i], 0, 0, 0))
        if len(d.views) > 1:
            ops.append(L.Op(L.OP_UNION, 0, 0, len(d.views), 0, 0, 0, 0))
        n += 1
    for k, (depth, vals) in enumerate(zip(depths, values)):
        ops.append(L.Op(L.OP_BSI_RANGE, VF[k], VV, 0, depth, L.CMP["=="], vals[ix[len(dims) + k]], 0))
        n += 1
    if n > 1:
        ops.append(L.Op(L.OP_INTERSECT, 0, 0, n, 0, 0, 0, 0))
    return ops


@gpu
def test_every_cell_is_bsi_sum(ctx):
    """on a small world, every cell's (count, sum) is what fbgpu_bsi_sum returns under filter ∩ the cell's rows"""
    rng = np.random.default_rng(116)
    agg, ints, dims, values, rows = _agg_world(ctx, rng, 200 if ON_EMU else 600)
    small_vals = [values[0][:3], values[1][:2]]
    for ds, ni, fo in (([dims[1]], 0, None), ([dims[0], dims[2]], 1, filt(2)), ([dims[2]], 2, None), ([], 2, filt(2))):
        counts, sums = gbs(ctx, ds, [8] * ni, small_vals[:ni], 40, [0, 1], fo)
        for ix in np.ndindex(counts.shape):
            s, n = ctx.bsi_sum(IDX, AF, VV, 40, [0, 1], filter_ops=_cell_ops(ds, [8] * ni, small_vals[:ni], ix, fo))
            assert (int(counts[ix]), int(sums[ix])) == (n, s), (len(ds), ni, ix)
        assert counts.sum() > 0


@gpu
def test_shards_missing_a_fragment(ctx):
    """shard 0 holds everything; shard 1 lacks the aggregate's fragment, shard 2 the int field's, shard 3 the set field in both
    of its views; shard 4 lacks the set field in one view only and still counts"""
    cols = [5, 6, SW + 5, 2 * SW + 5, 3 * SW + 5, 4 * SW + 5]
    load_values(ctx, AF, {c: 10 * (c // SW + 1) for c in cols if c // SW != 1}, 8)
    load_values(ctx, VF[0], {c: 3 for c in cols if c // SW != 2}, 4)
    d = Dim(SF[0], [0], [{0: [5, 6, SW + 5, 2 * SW + 5]}, {0: [6, SW + 5, 2 * SW + 5, 4 * SW + 5]}])
    d.load(ctx)
    ctx.commit()
    sh = [0, 1, 2, 3, 4]
    c, s = gbs(ctx, [d], [4], [[3]], 8, sh)
    assert (c.tolist(), s.tolist()) == ([[3]], [[70]])                 # columns 5, 6 (10 each) and 4·SW + 5 (50)
    c, s = gbs(ctx, [d], [], [], 8, sh)
    assert (c.tolist(), s.tolist()) == ([4], [100])                    # and 2·SW + 5 (30): no int dimension to miss
    c, s = gbs(ctx, [], [4], [[3]], 8, sh)
    assert (c.tolist(), s.tolist()) == ([4], [110])                    # 5, 6, 3·SW + 5, 4·SW + 5


@gpu
def test_zero_rows(ctx):
    load_values(ctx, AF, {1: 3}, 4)
    load_values(ctx, VF[0], {1: 3}, 4)
    ctx.commit()
    d = Dim(SF[0], [], [{}])
    c, s = gbs(ctx, [d], [4], [[3]], 4, [0])
    assert c.shape == s.shape == (0, 1)
    c, s = gbs(ctx, [Dim(SF[0], [0], [{}]), d], [], [], 4, [0])
    assert c.shape == s.shape == (1, 0)


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch and kernel launch"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        agg, ints, dims, values, rows = _agg_world(c, np.random.default_rng(117), 300 if ON_EMU else 1500)
        check(gbs(c, dims[1:2], [8, 8], values, 40, [0, 1, 2]), expect(agg, ints, dims[1:2], values), "b")
        check(gbs(c, [], [8], values[:1], 40, [0, 1, 2], filt(2)), expect(agg, ints[:1], [], values[:1], set(rows[2])), "no b")
        check(gbs(c, dims[2:], [], [], 40, [0, 1, 2]), expect(agg, [], dims[2:], []), "no int")
    finally:
        c.close()


@gpu
def test_node_answers_what_the_context_answers():
    """lib.Node with one device listed twice (shards alternate between its two contexts) sums the per-device tensors"""
    node, ctx = L.Node([0, 0], 1), L.Context(0)
    try:
        for c in (node, ctx):
            agg, ints, dims, values, rows = _agg_world(c, np.random.default_rng(118), 300 if ON_EMU else 2000)
        assert {node.owner(s) for s in range(2)} == {0, 1}
        for ds, ni in (([], 2), (dims[1:2], 1), (dims[:2], 0)):
            for fo, keep in ((None, None), (filt(2), set(rows[2]))):
                got = gbs(node, ds, [8] * ni, values[:ni], 40, [0, 1, 2], fo)
                check(got, gbs(ctx, ds, [8] * ni, values[:ni], 40, [0, 1, 2], fo), (len(ds), ni))
                check(got, expect(agg, ints[:ni], ds, values[:ni], keep), (len(ds), ni))
    finally:
        node.close()
        ctx.close()


# ------------------------------------------------------------------ argument errors
def _raw_call(lib, h, n_fields=1, n_views=None, n_rows=None, n_ints=2, depths=None, n_values=None, values=None, a_depth=4, null=None, n_shards=1):
    keep = dict(fields=np.full(8, SF[0], dtype=np.uint32), views=np.zeros(64, dtype=np.uint32),
                n_views=np.asarray(n_views if n_views is not None else [1] * 8, dtype=np.int32),
                rows=np.zeros(64, dtype=np.uint64), n_rows=np.asarray(n_rows if n_rows is not None else [1] * 8, dtype=np.int32),
                vfields=np.asarray(VF + VF + VF[:2], dtype=np.uint32), vviews=np.full(8, VV, dtype=np.uint32),
                depths=np.asarray(depths if depths is not None else [4] * 8, dtype=np.int32),
                values=np.asarray(values if values is not None else list(range(1 << 17)), dtype=np.int64),
                n_values=np.asarray(n_values if n_values is not None else [2] * 8, dtype=np.int32),
                shards=np.zeros(1, dtype=np.uint64), out=np.zeros(1 << 16, dtype=np.uint64), sums=np.zeros(1 << 16, dtype=np.int64))
    p = {k: (None if k == null else a.ctypes.data) for k, a in keep.items()}
    rc = lib.fbgpu_groupby_sum(h, IDX, p["fields"], p["views"], p["n_views"], n_fields, p["rows"], p["n_rows"], p["vfields"], p["vviews"], p["depths"], n_ints,
                               p["values"], p["n_values"], AF, VV, a_depth, None, 0, p["shards"], n_shards, p["out"], p["sums"])
    return rc, keep["out"], keep["sums"]


ARG_ERRORS = [
    ({"n_values": [300, 300]}, "product of n_values 90000 exceeds 65535"),
    ({"n_fields": 5, "n_ints": 4}, "n_fields + n_ints = 9 exceeds 8"),
    ({"n_fields": 8, "n_ints": 1}, "n_fields + n_ints = 9 exceeds 8"),
    ({"n_fields": 0, "n_ints": 9}, "n_ints=9 outside 0..8"),
    ({"n_ints": -1}, "n_ints=-1 outside 0..8"),
    ({"n_fields": 9, "n_ints": 0}, "n_fields=9 outside 0..8"),
    ({"n_fields": -1}, "n_fields=-1 outside 0..8"),
    ({"n_fields": 0, "n_ints": 0}, "no dimension: n_fields + n_ints = 0"),
    ({"n_fields": 2, "n_views": [1, 0]}, "n_views[1]=0 < 1"),
    ({"values": [1, 2, 5, 5]}, "values[1] are not strictly ascending at position 1"),
    ({"n_values": [2, 0]}, "n_values[1]=0 outside 1..65535"),
    ({"depths": [4, 65]}, "bit_depths[1]=65 outside 0..64"),
    ({"a_depth": 65}, "a_depth=65 outside 0..64"),
    ({"a_depth": -1}, "a_depth=-1 outside 0..64"),
    ({"n_shards": -1}, "bad argument"),
] + [({"null": k}, "bad argument") for k in ("fields", "views", "n_views", "rows", "n_rows", "vfields", "vviews", "depths", "values", "n_values", "shards", "out", "sums")]


def test_argument_errors_before_the_device_check():
    """every argument error but n_rows is reported before the device check, on a context and on a node without a device"""
    ctx = L.Context(L.DEVICE_NONE)
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        for h, lib in ((ctx.h, ctx.L), (node.h, node.L)):
            for kw, msg in ARG_ERRORS:
                rc, _, _ = _raw_call(lib, h, **kw)
                assert rc == L.E_INVALID and lib.fbgpu_last_error().decode() == msg, (kw, msg)
        for kw in ({"n_fields": 0, "null": "fields"}, {"n_ints": 0, "null": "vfields"}, {"n_ints": 0, "null": "values"}):
            rc, _, _ = _raw_call(ctx.L, ctx.h, **kw)                     # a kind of dimension that is absent may have NULL arrays
            assert rc == L.E_CUDA and "no device" in ctx.L.fbgpu_last_error().decode(), kw
        rc, _, _ = _raw_call(node.L, node.h, n_rows=[65536])               # the node checks n_rows before fanning out
        assert rc == L.E_INVALID and node.L.fbgpu_last_error().decode() == "n_rows[0]=65536 out of range"
    finally:
        node.close()
        ctx.close()


def test_refused_on_an_inspection_only_context():
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for dims, ints in (([], [(VF[0], VV, 4, [1, 2])]), ([(SF[0], [0], [0, 1])], [])):
            with pytest.raises(L.FbgpuError) as e:
                ctx.groupby_sum(IDX, dims, ints, (AF, VV, 4), [0])
            assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()


@gpu
def test_argument_errors_on_a_device(ctx):
    load_values(ctx, VF[0], {1: 0}, 4)
    load_values(ctx, VF[1], {1: 3}, 4)
    load_values(ctx, AF, {1: -9}, 4)
    ctx.commit()
    rc, o, s = _raw_call(ctx.L, ctx.h, n_fields=0, null="fields")          # values [0, 1] x [2, 3]: the column is in group (0, 1)
    assert rc == 0 and o[:4].tolist() == [0, 1, 0, 0] and s[:4].tolist() == [0, -9, 0, 0]
    for kw, msg in ARG_ERRORS + [({"n_rows": [65536]}, "n_rows[0]=65536 out of range"), ({"n_rows": [-1]}, "n_rows[0]=-1 out of range")]:
        rc, _, _ = _raw_call(ctx.L, ctx.h, **kw)
        assert rc == L.E_INVALID and ctx.L.fbgpu_last_error().decode() == msg, (kw, msg)
    rc, _, _ = _raw_call(ctx.L, ctx.h, n_rows=[0])                         # an empty tensor: nothing written, no error
    assert rc == 0


# ------------------------------------------------------------------ query level
TR = "from=2019-01-20T00:00, to=2019-03-10T00:00"
QUERIES = [
    "GroupBy(Rows(a), aggregate=Sum(field=v))",
    "GroupBy(Rows(a), Rows(b), aggregate=Sum(field=w))",
    "GroupBy(Rows(v), aggregate=Sum(field=w))",
    "GroupBy(Rows(a), Rows(v), aggregate=Sum(field=v), filter=Row(c=0))",
    "GroupBy(Rows(w), Rows(a), Rows(u), aggregate=Sum(field=v))",
    f"GroupBy(Rows(t, {TR}), aggregate=Sum(field=w))",
    f"GroupBy(Rows(a), Rows(t, {TR}), Rows(v), aggregate=Sum(field=u), filter=Row(c=0))",
    "GroupBy(Rows(a, previous=2), Rows(b, previous=1), aggregate=Sum(field=w), limit=4)",
    "GroupBy(Rows(a), Rows(u), aggregate=Sum(field=w), limit=5, offset=3)",
    "GroupBy(Rows(a), Rows(b), aggregate=Sum(field=v), having=Condition(sum > 3))",
    "GroupBy(Rows(a), Rows(v), aggregate=Sum(field=w), having=Condition(count >= 4))",
    'GroupBy(Rows(b), Rows(u), aggregate=Sum(field=w), sort="sum desc", limit=6)',
    'GroupBy(Rows(a), Rows(b), aggregate=Sum(field=v), sort="aggregate asc, count desc")',
    "GroupBy(Rows(a), aggregate=Sum(field=c))",                       # not an int field: no group has a value
]


def _pair(seed, n):
    dev, ref = X.Holder(), X.Holder(ctx=OracleCtx())
    _world(dev, seed, n)
    _world(ref, seed, n)
    assert not hasattr(ref.ctx, "groupby_sum")
    return dev, X.Executor(dev), X.Executor(ref)


@gpu
def test_queries_match_the_composition():
    """the device path against an oracle-backed holder running one Sum per group: Sum beside set, int and time-range children,
    with filter, previous, limit, offset, having on sum and count, and sort; a missing or unknown aggregate field is the same
    error on both"""
    dev, ed, er = _pair(31, 150 if ON_EMU else 1500)
    try:
        for q in (QUERIES[:4] + QUERIES[5:6] if ON_EMU else QUERIES):
            got = ed.execute("g", q)[0]
            assert got == er.execute("g", q)[0], q
            assert got or "having" in q or "field=c" in q, q
        for q in ("GroupBy(Rows(a), aggregate=Sum())", "GroupBy(Rows(a), aggregate=Sum(field=nope))"):
            with pytest.raises(X.QueryError) as e1:
                ed.execute("g", q)
            with pytest.raises(X.QueryError) as e2:
                er.execute("g", q)
            assert str(e1.value) == str(e2.value), q
    finally:
        dev.ctx.close()


@gpu
def test_slices_tile_the_tensors(monkeypatch):
    """with the groups-per-call cap lowered, the value lists are cut into slices and every combination is one call; the result is
    the composition's"""
    dev, ed, er = _pair(32, 150 if ON_EMU else 1000)
    calls = []
    real = dev.ctx.groupby_sum
    monkeypatch.setattr(dev.ctx, "groupby_sum", lambda *a, **kw: calls.append(a[2]) or real(*a, **kw), raising=False)
    monkeypatch.setattr(X.Executor, "GROUPBY_MIXED_MAX", 7)
    try:
        for q in ("GroupBy(Rows(a), Rows(v), Rows(w), aggregate=Sum(field=u))", "GroupBy(Rows(u), Rows(w), aggregate=Sum(field=v), filter=Row(c=0))"):
            calls.clear()
            got = ed.execute("g", q)[0]
            assert got and got == er.execute("g", q)[0], q
            assert len(calls) > 1 and all(np.prod([len(d[3]) for d in c]) <= 7 for c in calls), q
    finally:
        dev.ctx.close()


@gpu
def test_bounded_queries():
    """a 256-group Sum GroupBy asks the library twice (a's row list, then the groups), and with an int child once more (its
    Distinct), not once per group"""
    h = X.Holder()
    try:
        idx = h.create_index("s")
        idx.create_field("a")
        idx.create_field("v", "int", min=-1000, max=1000)
        idx.create_field("w", "int", min=0, max=3)
        rng = np.random.default_rng(33)
        for col in range(0, 4096 if ON_EMU else 20000, 3):
            h.set_bit("s", "a", col % 256, col)
            h.set_value("s", "v", col, int(rng.integers(-1000, 1001)))
            h.set_value("s", "w", col, col % 4)
        h.sync()
        ex = X.Executor(h)
        for q, n_queries, n_groups in (("GroupBy(Rows(a), aggregate=Sum(field=v))", 2, 256), ("GroupBy(Rows(a), Rows(w), aggregate=Sum(field=v))", 3, 256)):
            before = h.ctx.counters()["queries"]
            res = ex.execute("s", q)[0]
            assert len(res) == n_groups, q
            assert h.ctx.counters()["queries"] - before == n_queries, q
    finally:
        h.ctx.close()


# ------------------------------------------------------------------ CPU
def test_groupby_sum_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_groupby_sum.py"], timeout=3000)
