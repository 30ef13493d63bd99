"""fbgpu_groupby_distinct (GroupBy(..., aggregate=Count(Distinct(field=x))) in one device call) and the GroupBy path built on it.

Entry-point tests compare the distinct tensor with one the test computes from the columns and values it wrote, as Python sets,
and every cell of a small world with fbgpu_extract + unique under the cell's filter.  Query-level tests compare the executor's
GroupBy with an oracle-backed holder, which has no groupby_distinct and so runs one Distinct per group.  The CPU tests check the
argument errors and the refusal on a context without a device, and run this file's gpu tests on the interpreted kernels."""
import itertools

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from tests.oracle_ctx import OracleCtx
from tests.test_groupby_mixed import I64_MAX, I64_MIN, IDX, NEG0, ON_EMU, SF, SW, VF, VV, Dim, _pool, _set_world, _world, filt, load_values
from tests.test_groupby_sum import _cell_ops

XF = 14                                # the aggregate field x (BSI view VV)
gpu = pytest.mark.gpu


def _val(v):
    return 0 if v is NEG0 else v       # x's sign with magnitude 0 is the value 0


def expect(x, ints, dims, values, xs, keep=None):
    """the distinct tensor from the written data: x = {column: stored value or NEG0}, ints = [{column: value}] per int dimension
    with `values` its listed value lists, xs the listed values of x"""
    shape = [len(d.rows) for d in dims] + [len(v) for v in values]
    seen = {}
    pos = [{v: j for j, v in enumerate(vals)} for vals in values]
    listed = set(xs)
    for c, xv in x.items():
        if (keep is not None and c not in keep) or _val(xv) not in listed:
            continue
        js = []
        for cv, p in zip(ints, pos):
            v = cv.get(c)
            if v is None or v is NEG0 or v not in p:
                break
            js.append(p[v])
        else:
            for ix in itertools.product(*[[i for i, r in enumerate(d.rows) if c in d.union.get(r, ())] for d in dims]):
                seen.setdefault(ix + tuple(js), set()).add(_val(xv))
    out = np.zeros(shape, dtype=np.uint64)
    for ix, s in seen.items():
        out[ix] = len(s)
    return out


def gbd(ctx, dims, int_depths, values, depth, xs, shards, filter_ops=None, xfield=XF):
    return ctx.groupby_distinct(IDX, [(d.field, d.views, d.rows) for d in dims], [(VF[k], VV, int_depths[k], values[k]) for k in range(len(values))],
                                (xfield, VV, depth, xs), shards, filter_ops=filter_ops)


def check(got, want, what):
    assert got.shape == want.shape and got.dtype == np.uint64, what
    assert np.array_equal(got, want), what


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def _present(x):
    return sorted({_val(v) for v in x.values()})


# ------------------------------------------------------------------ entry point
@gpu
@pytest.mark.parametrize("depth", [1, 8, 32, 63, 64])
def test_depths_with_edge_values(ctx, depth):
    """x of each depth holding its edge values (INT64_MIN / INT64_MAX at depth 64), 0 and sign with magnitude 0 (the same value
    0), over two shards (a third listed shard holds nothing), grouped by 0-2 set and 0-2 int dimensions; x's list leaves out a
    present value and holds absent ones"""
    rng = np.random.default_rng(200 + depth)
    n = 150 if ON_EMU else 600
    cols = rng.choice(2 * SW, n, replace=False).tolist()
    pool = _pool(rng, depth, 8)
    x = {c: pool[int(rng.integers(len(pool)))] for c in cols if rng.random() < 0.9}
    xc = list(x)
    for c in xc[:3]:
        x[c] = NEG0
    x[xc[3]] = 0
    ints = [{c: int(rng.integers(-3, 3)) for c in cols if rng.random() < 0.9}, {c: int(rng.integers(0, 4)) for c in cols if rng.random() < 0.9}]
    load_values(ctx, XF, x, depth)
    for k, cv in enumerate(ints):
        load_values(ctx, VF[k], cv, 8)
    dims = [Dim(SF[0], [0, 1, 2, 9], [{r: rng.choice(cols, n // 3, replace=False).tolist() for r in range(3)}]),
            Dim(SF[1], [0, 1], [{r: rng.choice(cols, n // 2, replace=False).tolist() for r in range(2)}])]
    for d in dims:
        d.load(ctx)
    ctx.commit()
    values = [[-3, -2, -1, 0, 1, 2], [0, 1, 3, 7]]
    present = _present(x)
    assert 0 in present and (depth < 64 or {I64_MIN, I64_MAX} <= set(present))
    cut = [v for v in present if v != present[1]]                  # one present value is not listed: it counts nowhere
    absent = [v for v in (I64_MIN, -7777, 12345, I64_MAX) if v not in present][:2]
    for xs in (present, sorted(cut + absent)):
        for ni in (0, 1, 2):
            for nd in (0, 1, 2):
                if ni + nd == 0:
                    continue
                got = gbd(ctx, dims[:nd], [8] * ni, values[:ni], depth, xs, [0, 1, 4])
                check(got, expect(x, ints[:ni], dims[:nd], values[:ni], xs), (len(xs), ni, nd))
                assert got.sum() > 0
    got = gbd(ctx, [], [8], [[-3, -2, -1, 0, 1, 2]], depth, present, [0, 1])
    assert got.max() > 1


@gpu
@pytest.mark.parametrize("layout", ["bitmap", "run", "array"])
def test_container_encodings(ctx, layout):
    """x's planes, an int dimension's planes and set rows stored as bitmaps (dense random columns), runs (contiguous columns,
    values in long stretches) and arrays (scattered columns, bank-striped); the set dimension has two views.  Hundreds to
    thousands of listed values: many presence words per cell, the last one partly used"""
    rng = np.random.default_rng(211)
    n = 20000 if ON_EMU else 60000
    if layout == "bitmap":
        cols = (np.sort(rng.choice(SW // 8, n, replace=False)) + 3 * 65536).tolist()
        xs, vs = rng.integers(-3000, 3000, n).tolist(), rng.integers(0, 40, n).tolist()
        views = [{r: [c for c in cols if rng.random() < 0.5] for r in range(2)} for _ in range(2)]
    elif layout == "run":
        cols = list(range(100, 100 + n))
        xs, vs = np.repeat(rng.integers(-(1 << 20), 1 << 20, n // 1000), 1000).tolist(), np.repeat(rng.integers(0, 9, n // 2500), 2500).tolist()
        views = [{0: cols[: n // 2], 1: cols[n // 3: n // 3 + 7000]}, {0: cols[n // 4: n // 2 + 3000], 1: cols[5000: 5100]}]
    else:
        cols = rng.choice(3 * SW, 3000 if ON_EMU else 9000, replace=False).tolist()
        xs, vs = rng.integers(-300, 300, len(cols)).tolist(), rng.integers(0, 30, len(cols)).tolist()
        views = [{r: rng.choice(cols, len(cols) // 2, replace=False).tolist() for r in range(3)} for _ in range(2)]      # >= 64 per slot: bank-striped
    x, ints = dict(zip(cols, xs)), [dict(zip(cols, vs))]
    load_values(ctx, XF, x, 21)
    load_values(ctx, VF[0], ints[0], 21)
    d = Dim(SF[0], sorted(views[0]), views)
    d.load(ctx)
    ctx.commit()
    values = [sorted(set(vs))]
    listed = _present(x)
    for dims, ni in (([d], 1), ([d], 0), ([], 1)):
        check(gbd(ctx, dims, [21] * ni, values[:ni], 21, listed, [0, 1, 2]), expect(x, ints[:ni], dims, values[:ni], listed), (len(dims), ni))


def _x_world(ctx, rng, n):
    """_set_world (two int fields, three set fields of 1-3 views, filter rows) plus x of depth 40 on most columns, drawn from
    70 values so that cells share values"""
    ints, dims, values, rows = _set_world(ctx, rng, n)
    cols = sorted(set(ints[0]) | set(ints[1]))
    pool = [int(v) for v in rng.integers(-(1 << 40) + 1, 1 << 40, 69)] + [0]
    x = {c: pool[int(rng.integers(len(pool)))] for c in cols if rng.random() < 0.85}
    for c in cols[:4]:
        x[c] = NEG0
    load_values(ctx, XF, x, 40)
    ctx.commit()
    return x, ints, dims, values, rows


@gpu
def test_set_dimensions_views_and_filters(ctx):
    """0-3 set dimensions with 1-3 views each in several orders, beside 0-2 int dimensions, under no filter and a sparse, a dense
    and an empty filter; 70 listed values (two presence words per cell, the second partly used)"""
    rng = np.random.default_rng(213)
    x, ints, dims, values, rows = _x_world(ctx, rng, 300 if ON_EMU else 2000)
    xs = _present(x)
    shards = [0, 1, 3]
    orders = [(0,), (2,), (1, 2), (2, 1, 0)] if ON_EMU else [p for k in (1, 2, 3) for p in itertools.permutations(range(3), k)]
    filters = ((None, None), (2, set(rows[2]))) if ON_EMU else ((None, None), (1, set(rows[1])), (2, set(rows[2])), (3, set()))
    for order in [()] + orders:
        ds = [dims[k] for k in order]
        for ni in ((1, 2) if not ds else (0, 1, 2)):
            for row, keep in filters:
                got = gbd(ctx, ds, [8] * ni, values[:ni], 40, xs, shards, None if row is None else filt(row))
                check(got, expect(x, ints[:ni], ds, values[:ni], xs, keep), (order, ni, row))


@gpu
@pytest.mark.parametrize("n_x", [1, 63, 64, 65, 130])
def test_listed_value_counts(ctx, n_x):
    """lists of 1 to 130 values, whole and partial presence words; the other present values are not listed"""
    rng = np.random.default_rng(214 + n_x)
    x, ints, dims, values, rows = _x_world(ctx, rng, 300 if ON_EMU else 1500)
    more = [int(v) for v in rng.integers(-(1 << 40) + 1, 1 << 40, 200)]
    xs = sorted(set(_present(x)[::2] + more))[:n_x]
    for ds, ni in (([], 1), (dims[1:2], 1), (dims[2:], 0)):
        check(gbd(ctx, ds, [8] * ni, values[:ni], 40, xs, [0, 1, 2]), expect(x, ints[:ni], ds, values[:ni], xs), (n_x, len(ds), ni))


@gpu
def test_x_is_also_a_group_dimension(ctx):
    """GroupBy(Rows(a), Rows(v), aggregate=Count(Distinct(field=v))): every non-empty cell holds one value, its own"""
    rng = np.random.default_rng(215)
    ints, dims, values, rows = _set_world(ctx, rng, 300 if ON_EMU else 2000)
    xs = sorted(set(ints[0].values()))
    for ds in ([], dims[:1], dims[1:2]):
        got = gbd(ctx, ds, [8], values[:1], 8, xs, [0, 1, 2], xfield=VF[0])
        check(got, expect(ints[0], ints[:1], ds, values[:1], xs), len(ds))
        counts = ctx.groupby_mixed(IDX, [(d.field, d.views, d.rows) for d in ds], [(VF[0], VV, 8, values[0])], [0, 1, 2])
        assert np.array_equal(got, (counts > 0).astype(np.uint64)) and counts.sum() > 0


@gpu
def test_plane_table_overflow(ctx):
    """two depth-64 int dimensions and a depth-64 x need 195 plane-table entries, more than the 184 the kernel holds: every
    field's planes are resolved per range.  With a depth-8 x (139 entries) they fit."""
    rng = np.random.default_rng(216)
    n = 200 if ON_EMU else 1500
    cols = rng.choice(2 * SW, n, replace=False).tolist()
    pools = [_pool(rng, 64, 5), _pool(rng, 64, 4)]
    ints = [{c: p[int(rng.integers(len(p)))] for c in cols if rng.random() < 0.9} for p in pools]
    bigpool = _pool(rng, 64, 6)
    big = {c: bigpool[int(rng.integers(6))] for c in cols if rng.random() < 0.9}
    small = {c: int(rng.integers(-20, 21)) for c in cols}
    for k, cv in enumerate(ints):
        load_values(ctx, VF[k], cv, 64)
    load_values(ctx, XF, big, 64)
    load_values(ctx, XF + 1, small, 8)
    d = Dim(SF[0], [0, 1], [{r: rng.choice(cols, n // 2, replace=False).tolist() for r in range(2)}])
    d.load(ctx)
    ctx.commit()
    values = [sorted(p) for p in pools]
    for ds in ([], [d]):
        check(gbd(ctx, ds, [64, 64], values, 64, _present(big), [0, 1]), expect(big, ints, ds, values, _present(big)), ("195", len(ds)))
        check(gbd(ctx, ds, [64, 64], values, 8, _present(small), [0, 1], xfield=XF + 1), expect(small, ints, ds, values, _present(small)), ("139", len(ds)))


@gpu
def test_every_cell_is_extract_unique(ctx):
    """on a small world, every cell is the number of listed values among fbgpu_extract(x)'s values under filter ∩ the cell's
    rows"""
    rng = np.random.default_rng(217)
    x, ints, dims, values, rows = _x_world(ctx, rng, 200 if ON_EMU else 600)
    small_vals = [values[0][:3], values[1][:2]]
    xs = _present(x)[1::2]
    for ds, ni, fo in (([dims[1]], 0, None), ([dims[0], dims[2]], 1, filt(2)), ([dims[2]], 2, None), ([], 2, filt(2))):
        got = gbd(ctx, ds, [8] * ni, small_vals[:ni], 40, xs, [0, 1], fo)
        for ix in np.ndindex(got.shape):
            _, vals, _ = ctx.extract(IDX, XF, VV, 40, [0, 1], filter_ops=_cell_ops(ds, [8] * ni, small_vals[:ni], ix, fo))
            assert int(got[ix]) == len(set(np.unique(vals).tolist()) & set(xs)), (len(ds), ni, ix)
        assert got.sum() > 0


@gpu
def test_shards_missing_a_fragment(ctx):
    """shard 0 holds everything; shard 1 lacks x's fragment, shard 2 the int field's, shard 3 the set field in both of its
    views; shard 4 lacks the set field in one view only and still counts"""
    cols = [5, 6, SW + 5, 2 * SW + 5, 3 * SW + 5, 4 * SW + 5]
    load_values(ctx, XF, {c: 10 * (c // SW + 1) for c in cols if c // SW != 1}, 8)
    load_values(ctx, VF[0], {c: 3 for c in cols if c // SW != 2}, 4)
    d = Dim(SF[0], [0], [{0: [5, 6, SW + 5, 2 * SW + 5]}, {0: [6, SW + 5, 2 * SW + 5, 4 * SW + 5]}])
    d.load(ctx)
    ctx.commit()
    sh, xs = [0, 1, 2, 3, 4], [10, 20, 30, 40, 50]
    assert gbd(ctx, [d], [4], [[3]], 8, xs, sh).tolist() == [[2]]         # 10 (columns 5, 6) and 50
    assert gbd(ctx, [d], [], [], 8, xs, sh).tolist() == [3]               # and 30: no int dimension to miss
    assert gbd(ctx, [], [4], [[3]], 8, xs, sh).tolist() == [3]            # 10, 40, 50


@gpu
def test_zero_rows(ctx):
    load_values(ctx, XF, {1: 3}, 4)
    load_values(ctx, VF[0], {1: 3}, 4)
    ctx.commit()
    d = Dim(SF[0], [], [{}])
    assert gbd(ctx, [d], [4], [[3]], 4, [3], [0]).shape == (0, 1)
    assert gbd(ctx, [Dim(SF[0], [0], [{}]), d], [], [], 4, [3], [0]).shape == (1, 0)


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch and kernel launch, every batch marking the same bitset"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        x, ints, dims, values, rows = _x_world(c, np.random.default_rng(218), 300 if ON_EMU else 1500)
        xs = _present(x)
        check(gbd(c, dims[1:2], [8, 8], values, 40, xs, [0, 1, 2]), expect(x, ints, dims[1:2], values, xs), "b")
        check(gbd(c, [], [8], values[:1], 40, xs, [0, 1, 2], filt(2)), expect(x, ints[:1], [], values[:1], xs, set(rows[2])), "no b")
        check(gbd(c, dims[2:], [], [], 40, xs, [0, 1, 2]), expect(x, [], dims[2:], [], xs), "no int")
        check(gbd(c, dims[:2], [], [], 40, xs, [0, 1, 2]), expect(x, [], dims[:2], [], xs), "peeled")
    finally:
        c.close()


@gpu
def test_refused_with_ranks_attached():
    """two contexts wired as ranks: a distinct set does not merge by the sum the ranks' tensors are reduced with"""
    a, b = L.Context(0), L.Context(0)
    try:
        L.p2p_open_local([a, b])
        for c in (a, b):
            with pytest.raises(L.FbgpuError) as e:
                c.groupby_distinct(IDX, [], [(VF[0], VV, 4, [1, 2])], (XF, VV, 4, [1]), [0])
            assert e.value.code == L.E_COMM and "union" in str(e.value)
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ argument errors
def _raw_call(lib, h, n_fields=1, n_views=None, n_rows=None, n_ints=2, depths=None, n_values=None, values=None, x_depth=4, x_values=None,
              n_x=None, null=None, n_shards=1):
    xv = x_values if x_values is not None else [1, 2, 3]
    keep = dict(fields=np.full(8, SF[0], dtype=np.uint32), views=np.zeros(64, dtype=np.uint32),
                n_views=np.asarray(n_views if n_views is not None else [1] * 8, dtype=np.int32),
                rows=np.zeros(64, dtype=np.uint64), n_rows=np.asarray(n_rows if n_rows is not None else [1] * 8, dtype=np.int32),
                vfields=np.asarray(VF + VF + VF[:2], dtype=np.uint32), vviews=np.full(8, VV, dtype=np.uint32),
                depths=np.asarray(depths if depths is not None else [4] * 8, dtype=np.int32),
                values=np.asarray(values if values is not None else list(range(1 << 17)), dtype=np.int64),
                n_values=np.asarray(n_values if n_values is not None else [2] * 8, dtype=np.int32),
                x_values=np.asarray(xv, dtype=np.int64), shards=np.zeros(1, dtype=np.uint64), out=np.zeros(1 << 16, dtype=np.uint64))
    p = {k: (None if k == null else a.ctypes.data) for k, a in keep.items()}
    rc = lib.fbgpu_groupby_distinct(h, IDX, p["fields"], p["views"], p["n_views"], n_fields, p["rows"], p["n_rows"], p["vfields"], p["vviews"], p["depths"],
                                    n_ints, p["values"], p["n_values"], XF, VV, x_depth, p["x_values"], len(xv) if n_x is None else n_x, None, 0,
                                    p["shards"], n_shards, p["out"])
    return rc, keep["out"]


ARG_ERRORS = [
    ({"n_values": [300, 300]}, "product of n_values 90000 exceeds 65535"),
    ({"n_fields": 5, "n_ints": 4}, "n_fields + n_ints = 9 exceeds 8"),
    ({"n_fields": 0, "n_ints": 9}, "n_ints=9 outside 0..8"),
    ({"n_fields": 9, "n_ints": 0}, "n_fields=9 outside 0..8"),
    ({"n_fields": 0, "n_ints": 0}, "no dimension: n_fields + n_ints = 0"),
    ({"n_fields": 2, "n_views": [1, 0]}, "n_views[1]=0 < 1"),
    ({"values": [1, 2, 5, 5]}, "values[1] are not strictly ascending at position 1"),
    ({"depths": [4, 65]}, "bit_depths[1]=65 outside 0..64"),
    ({"x_depth": 65}, "x_depth=65 outside 0..64"),
    ({"x_depth": -1}, "x_depth=-1 outside 0..64"),
    ({"n_x": 0}, "n_x=0 < 1"),
    ({"n_x": -3}, "n_x=-3 < 1"),
    ({"x_values": [1, 4, 4]}, "x_values are not strictly ascending at position 2"),
    ({"x_values": [5, -1]}, "x_values are not strictly ascending at position 1"),
    ({"n_shards": -1}, "bad argument"),
] + [({"null": k}, "bad argument") for k in ("fields", "views", "n_views", "rows", "n_rows", "vfields", "values", "x_values", "shards", "out")]


def test_argument_errors_before_the_device_check():
    """every argument error but n_rows is reported before the device check"""
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for kw, msg in ARG_ERRORS:
            rc, _ = _raw_call(ctx.L, ctx.h, **kw)
            assert rc == L.E_INVALID and ctx.L.fbgpu_last_error().decode() == msg, (kw, msg)
        for kw in ({"n_fields": 0, "null": "fields"}, {"n_ints": 0, "null": "vfields"}, {"n_ints": 0, "null": "values"}, {}):
            rc, _ = _raw_call(ctx.L, ctx.h, **kw)                        # a kind of dimension that is absent may have NULL arrays
            assert rc == L.E_CUDA and "no device" in ctx.L.fbgpu_last_error().decode(), kw
    finally:
        ctx.close()


def test_refused_on_an_inspection_only_context():
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for dims, ints in (([], [(VF[0], VV, 4, [1, 2])]), ([(SF[0], [0], [0, 1])], [])):
            with pytest.raises(L.FbgpuError) as e:
                ctx.groupby_distinct(IDX, dims, ints, (XF, VV, 4, [-1, 7]), [0])
            assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()


def test_no_node_form():
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        with pytest.raises(NotImplementedError):
            node.groupby_distinct(IDX, [], [(VF[0], VV, 4, [1, 2])], (XF, VV, 4, [1]), [0])
    finally:
        node.close()


@gpu
def test_argument_errors_on_a_device(ctx):
    load_values(ctx, VF[0], {1: 0}, 4)
    load_values(ctx, VF[1], {1: 3}, 4)
    load_values(ctx, XF, {1: 2}, 4)
    ctx.commit()
    rc, o = _raw_call(ctx.L, ctx.h, n_fields=0, null="fields")              # values [0, 1] x [2, 3]: the column is in group (0, 1)
    assert rc == 0 and o[:4].tolist() == [0, 1, 0, 0]
    for kw, msg in ARG_ERRORS + [({"n_rows": [65536]}, "n_rows[0]=65536 out of range"), ({"n_rows": [-1]}, "n_rows[0]=-1 out of range")]:
        rc, _ = _raw_call(ctx.L, ctx.h, **kw)
        assert rc == L.E_INVALID and ctx.L.fbgpu_last_error().decode() == msg, (kw, msg)
    rc, _ = _raw_call(ctx.L, ctx.h, n_rows=[0])                             # an empty tensor: nothing written, no error
    assert rc == 0


# ------------------------------------------------------------------ query level
TR = "from=2019-01-20T00:00, to=2019-03-10T00:00"
QUERIES = [
    "GroupBy(Rows(a), aggregate=Count(Distinct(field=v)))",
    "GroupBy(Rows(a), Rows(b), aggregate=Count(Distinct(field=w)))",
    "GroupBy(Rows(a), aggregate=Count(Distinct(field=u)), filter=Row(c=0))",
    "GroupBy(Rows(a), Rows(b), aggregate=Count(Distinct(Row(c=0), field=v)))",
    "GroupBy(Rows(b), aggregate=Count(Distinct(Row(v > 0), field=w)), filter=Row(c=0))",
    "GroupBy(Rows(v), aggregate=Count(Distinct(field=w)))",
    "GroupBy(Rows(a), Rows(v), aggregate=Count(Distinct(field=v)))",
    "GroupBy(Rows(w), Rows(a), Rows(u), aggregate=Count(Distinct(field=v)))",
    f"GroupBy(Rows(t, {TR}), aggregate=Count(Distinct(field=w)))",
    f"GroupBy(Rows(a), Rows(t, {TR}), Rows(v), aggregate=Count(Distinct(field=u)), filter=Row(c=0))",
    "GroupBy(Rows(a, previous=2), Rows(b, previous=1), aggregate=Count(Distinct(field=w)), limit=4)",
    "GroupBy(Rows(a), Rows(u), aggregate=Count(Distinct(field=w)), limit=5, offset=3)",
    "GroupBy(Rows(a), Rows(b), aggregate=Count(Distinct(field=v)), having=Condition(sum > 3))",
    "GroupBy(Rows(a), Rows(v), aggregate=Count(Distinct(field=w)), having=Condition(count >= 4))",
    'GroupBy(Rows(b), Rows(u), aggregate=Count(Distinct(field=w)), sort="aggregate desc", limit=6)',
    'GroupBy(Rows(a), Rows(b), aggregate=Count(Distinct(field=v)), sort="aggregate desc, count asc")',
    "GroupBy(Rows(a), aggregate=Count(Distinct(Row(c=5), field=v)))",       # an empty x list: every distinct count is 0
    "GroupBy(Rows(a), aggregate=Count(Distinct(field=b)))",                 # not an int field: the per-group composition
]


def _pair(seed, n):
    dev, ref = X.Holder(), X.Holder(ctx=OracleCtx())
    _world(dev, seed, n)
    _world(ref, seed, n)
    assert not hasattr(ref.ctx, "groupby_distinct")
    return dev, X.Executor(dev), X.Executor(ref)


@gpu
def test_queries_match_the_composition():
    """the device path against an oracle-backed holder running one Distinct per group: Count(Distinct) beside set, int and
    time-range children, with filter, a Distinct child, previous, limit, offset, having, sort; a missing or unknown field is the
    same error on both"""
    dev, ed, er = _pair(41, 150 if ON_EMU else 1500)
    try:
        for q in (QUERIES[:4] + QUERIES[8:9] if ON_EMU else QUERIES):
            got = ed.execute("g", q)[0]
            assert got == er.execute("g", q)[0], q
            assert got or "having" in q, q
        assert all(g[2] == 0 for g in ed.execute("g", QUERIES[-2])[0])
        for q in ("GroupBy(Rows(a), aggregate=Count(Distinct()))", "GroupBy(Rows(a), aggregate=Count(Distinct(field=nope)))"):
            with pytest.raises(X.QueryError) as e1:
                ed.execute("g", q)
            with pytest.raises(X.QueryError) as e2:
                er.execute("g", q)
            assert str(e1.value) == str(e2.value), q
    finally:
        dev.ctx.close()


@gpu
def test_slices_add_up(monkeypatch):
    """with the groups-per-call and bits-per-call caps lowered, the int children's lists and x's list are cut into slices; the
    result is the composition's"""
    dev, ed, er = _pair(42, 150 if ON_EMU else 1000)
    calls = []
    real = dev.ctx.groupby_distinct
    monkeypatch.setattr(dev.ctx, "groupby_distinct", lambda *a, **kw: calls.append((a[2], a[3])) or real(*a, **kw), raising=False)
    monkeypatch.setattr(X.Executor, "GROUPBY_MIXED_MAX", 7)
    monkeypatch.setattr(X.Executor, "GROUPBY_DISTINCT_BITS", 24)
    try:
        for q, rows_last in (("GroupBy(Rows(a), Rows(v), Rows(w), aggregate=Count(Distinct(field=u)))", 5),
                             ("GroupBy(Rows(u), Rows(w), aggregate=Count(Distinct(field=v)), filter=Row(c=0))", 1),
                             ("GroupBy(Rows(b), aggregate=Count(Distinct(field=w)))", 3)):
            calls.clear()
            got = ed.execute("g", q)[0]
            assert got and got == er.execute("g", q)[0], q
            assert len(calls) > 1, q
            for ints, x in calls:
                groups = int(np.prod([len(d[3]) for d in ints]))
                assert groups <= 7 and (rows_last * groups * len(x[3]) <= 24 or len(x[3]) == 1), q
    finally:
        dev.ctx.close()


@gpu
def test_falls_back_on_comm_and_node(monkeypatch):
    """FBGPU_E_COMM from the call, or the NotImplementedError of a node (no node form), leaves the per-group composition, which
    answers the same"""
    dev, ed, er = _pair(43, 150 if ON_EMU else 600)
    q = "GroupBy(Rows(a), Rows(b), aggregate=Count(Distinct(field=v)), filter=Row(c=0))"
    try:
        want = er.execute("g", q)[0]
        assert ed.execute("g", q)[0] == want
        for exc in (L.FbgpuError(L.E_COMM, "local to one context"), NotImplementedError("no node form")):
            def refuse(*a, exc=exc, **kw):
                raise exc
            monkeypatch.setattr(dev.ctx, "groupby_distinct", refuse, raising=False)
            assert ed.execute("g", q)[0] == want, exc
    finally:
        dev.ctx.close()


@gpu
def test_bounded_queries():
    """a 256-group Count(Distinct) GroupBy asks the library four times (a's row list, the counts, x's values, the distinct
    counts), and with an int child once more (its Distinct), not once per group"""
    h = X.Holder()
    try:
        idx = h.create_index("s")
        idx.create_field("a")
        idx.create_field("v", "int", min=-1000, max=1000)
        idx.create_field("w", "int", min=0, max=3)
        rng = np.random.default_rng(44)
        for col in range(0, 4096 if ON_EMU else 20000, 3):
            h.set_bit("s", "a", col % 256, col)
            h.set_value("s", "v", col, int(rng.integers(-1000, 1001)))
            h.set_value("s", "w", col, col % 4)
        h.sync()
        ex = X.Executor(h)
        for q, n_queries, n_groups in (("GroupBy(Rows(a), aggregate=Count(Distinct(field=v)))", 4, 256),
                                       ("GroupBy(Rows(a), Rows(w), aggregate=Count(Distinct(field=v)))", 5, 256)):
            before = h.ctx.counters()["queries"]
            res = ex.execute("s", q)[0]
            assert len(res) == n_groups and all(len(g) == 3 and 0 < g[2] <= g[1] for g in res), q
            assert h.ctx.counters()["queries"] - before == n_queries, q
    finally:
        h.ctx.close()


# ------------------------------------------------------------------ CPU
def test_groupby_distinct_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_groupby_distinct.py"], timeout=3000)
