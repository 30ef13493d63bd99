"""fbgpu_groupby_distinct_rows (GroupBy(..., aggregate=Count(Distinct(field=x))) over a set, mutex, bool or time field x in one
device call) and the GroupBy path built on it.

Entry-point tests compare the distinct tensor with one the test computes from the bits it wrote, as Python sets, and every cell
of a small world with the all-rows row counts of x under the cell's filter.  Query-level tests compare the executor's GroupBy with
an oracle-backed holder, which has neither distinct call and so runs one Distinct per group.  The CPU tests check the argument
errors and the refusals on a context without a device and on a node, and run this file's gpu tests on the interpreted kernels."""
import itertools

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from tests.oracle_ctx import OracleCtx
from tests.test_groupby_mixed import IDX, ON_EMU, SF, SW, VF, VV, Dim, _pool, _set_world, _world, filt, load_set, load_values
from tests.test_groupby_sum import _cell_ops

XF, XV = 14, 0                         # the aggregate field x and its view
BIG = 1 << 32                          # row ids at and above 2^32
gpu = pytest.mark.gpu


def expect(xr, ints, dims, values, xs, keep=None):
    """the distinct tensor from the written data: xr = {column: set of x rows}, ints = [{column: value}] per int dimension with
    `values` its listed value lists, xs the listed rows of x"""
    shape = [len(d.rows) for d in dims] + [len(v) for v in values]
    seen = {}
    pos = [{v: j for j, v in enumerate(vals)} for vals in values]
    listed = set(xs)
    for c, rs in xr.items():
        rs = rs & listed
        if not rs or (keep is not None and c not in keep):
            continue
        js = []
        for cv, p in zip(ints, pos):
            v = cv.get(c)
            if v is None or v not in p:
                break
            js.append(p[v])
        else:
            for ix in itertools.product(*[[i for i, r in enumerate(d.rows) if c in d.union.get(r, ())] for d in dims]):
                seen.setdefault(ix + tuple(js), set()).update(rs)
    out = np.zeros(shape, dtype=np.uint64)
    for ix, s in seen.items():
        out[ix] = len(s)
    return out


def gbr(ctx, dims, depths, values, xs, shards, filter_ops=None, xfield=XF, xview=XV):
    return ctx.groupby_distinct_rows(IDX, [(d.field, d.views, d.rows) for d in dims], [(VF[k], VV, depths[k], values[k]) for k in range(len(values))],
                                     (xfield, xview, xs), shards, filter_ops=filter_ops)


def load_x(ctx, xr, field=XF):
    rows = {}
    for c, rs in xr.items():
        for r in rs:
            rows.setdefault(r, []).append(c)
    load_set(ctx, field, rows, XV)


def check(got, want, what):
    assert got.shape == want.shape and got.dtype == np.uint64, what
    assert np.array_equal(got, want), what


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def _x_data(rng, cols, shape):
    """x's rows per column: `set` holds 0 to about 40 rows of 60 (ids below and at or above 2^32), `mutex` one row of 30 on most
    columns, `bool` row 0 or 1"""
    if shape == "set":
        pool = list(range(30)) + [BIG + r for r in range(30)]
        xr = {c: {pool[int(i)] for i in rng.choice(60, int(rng.integers(0, 41)), replace=False)} for c in cols}
    elif shape == "mutex":
        pool = list(range(15)) + [BIG + 7 * r for r in range(15)]
        xr = {c: {pool[int(rng.integers(30))]} for c in cols if rng.random() < 0.85}
    else:
        xr = {c: {int(rng.integers(2))} for c in cols if rng.random() < 0.9}
    return {c: rs for c, rs in xr.items() if rs}


def _present(xr):
    return sorted(set().union(*xr.values()))


# ------------------------------------------------------------------ entry point
@gpu
@pytest.mark.parametrize("shape", ["set", "mutex", "bool"])
def test_shapes_dimensions_and_filters(ctx, shape):
    """x holding many rows per column (many rounds), one (mutex: one round) or a bool; 0-2 set dimensions of 1-3 views beside 0-2
    int dimensions, under no filter, a sparse and a dense filter; x's list leaves out a present row and holds absent ones, some
    at or above 2^32; shard 3 is listed and holds nothing"""
    rng = np.random.default_rng({"set": 300, "mutex": 301, "bool": 302}[shape])
    ints, dims, values, rows = _set_world(ctx, rng, 200 if ON_EMU else 1500)
    cols = sorted(set(ints[0]) | set(ints[1]))
    xr = _x_data(rng, cols, shape)
    load_x(ctx, xr)
    ctx.commit()
    present = _present(xr)
    lists = [present, sorted(set(present[1:]) | {5000, BIG + 99999})] if shape != "bool" else [present, [1], [0, 1, 2, BIG]]
    orders = [(0,), (1, 2)] if ON_EMU else [p for k in (1, 2) for p in itertools.permutations(range(3), k)]
    filters = ((None, None), (2, set(rows[2]))) if ON_EMU else ((None, None), (1, set(rows[1])), (2, set(rows[2])))
    for xs in lists:
        for order in [()] + orders:
            ds = [dims[k] for k in order]
            for ni in ((1, 2) if not ds else (0, 1, 2)):
                for row, keep in filters:
                    got = gbr(ctx, ds, [8] * ni, values[:ni], xs, [0, 1, 3], None if row is None else filt(row))
                    check(got, expect(xr, ints[:ni], ds, values[:ni], xs, keep), (shape, len(xs), order, ni, row))
    assert gbr(ctx, dims[1:2], [], [], present, [0, 1]).max() > (1 if shape == "bool" else 3)


@gpu
@pytest.mark.parametrize("layout", ["bitmap", "run", "array"])
def test_container_encodings(ctx, layout):
    """x's rows, a set dimension's rows (two views) and a depth-64 int dimension's planes stored as bitmaps (dense random
    columns), runs (contiguous columns) and arrays (scattered columns, bank-striped)"""
    rng = np.random.default_rng(310)
    n = 20000 if ON_EMU else 60000
    if layout == "bitmap":
        cols = (np.sort(rng.choice(SW // 8, n, replace=False)) + 3 * 65536).tolist()
        xr = {c: {int(r) for r in rng.choice(6, int(rng.integers(1, 4)), replace=False)} for c in cols}
        views = [{r: [c for c in cols if rng.random() < 0.5] for r in range(2)} for _ in range(2)]
    elif layout == "run":
        cols = list(range(100, 100 + n))
        xr = {c: {c // 5000, BIG + c // 7000} for c in cols}
        views = [{0: cols[: n // 2], 1: cols[n // 3: n // 3 + 7000]}, {0: cols[n // 4: n // 2 + 3000], 1: cols[5000: 5100]}]
    else:
        cols = rng.choice(3 * SW, 3000 if ON_EMU else 9000, replace=False).tolist()
        xr = {c: {int(r) for r in rng.choice(4, int(rng.integers(1, 3)), replace=False)} for c in cols}
        views = [{r: rng.choice(cols, len(cols) // 2, replace=False).tolist() for r in range(3)} for _ in range(2)]
    pool = _pool(rng, 64, 5)
    ints = [{c: pool[int(rng.integers(5))] for c in cols if rng.random() < 0.9}]
    load_x(ctx, xr)
    load_values(ctx, VF[0], ints[0], 64)
    d = Dim(SF[0], sorted(views[0]), views)
    d.load(ctx)
    ctx.commit()
    values = [sorted(pool)]
    xs = _present(xr)
    for dims, ni in (([d], 1), ([d], 0), ([], 1)):
        check(gbr(ctx, dims, [64] * ni, values[:ni], xs, [0, 1, 2]), expect(xr, ints[:ni], dims, values[:ni], xs), (layout, len(dims), ni))


@gpu
def test_x_is_also_a_group_dimension(ctx):
    """GroupBy(Rows(s), Rows(v), aggregate=Count(Distinct(field=s))): a cell of row r holds r and, through the columns it
    shares, the other rows of those columns"""
    rng = np.random.default_rng(311)
    ints, dims, values, rows = _set_world(ctx, rng, 300 if ON_EMU else 2000)
    d = dims[0]                                                          # single view: x is this field's view
    xr = {}
    for r, cs in d.per_view[0].items():
        for c in cs:
            xr.setdefault(c, set()).add(r)
    xs = sorted(d.per_view[0])
    for ds, ni in (([d], 1), ([d], 0), ([d, dims[1]], 0)):
        got = gbr(ctx, ds, [8] * ni, values[:ni], xs, [0, 1, 2], xfield=d.field, xview=d.views[0])
        check(got, expect(xr, ints[:ni], ds, values[:ni], xs), (len(ds), ni))
        assert got.sum() > 0


@gpu
def test_every_cell_is_row_counts(ctx):
    """on a small world, every cell is the number of listed rows among those the all-rows row counts of x find under filter ∩
    the cell's rows"""
    rng = np.random.default_rng(312)
    ints, dims, values, rows = _set_world(ctx, rng, 200 if ON_EMU else 600)
    cols = sorted(set(ints[0]) | set(ints[1]))
    xr = _x_data(rng, cols, "set")
    load_x(ctx, xr)
    ctx.commit()
    small_vals = [values[0][:3], values[1][:2]]
    xs = _present(xr)[1::2]
    for ds, ni, fo in (([dims[1]], 0, None), ([dims[0], dims[2]], 1, filt(2)), ([dims[2]], 2, None), ([], 2, filt(2))):
        got = gbr(ctx, ds, [8] * ni, small_vals[:ni], xs, [0, 1], fo)
        for ix in np.ndindex(got.shape):
            rid, cnt = ctx.row_counts(IDX, XF, XV, [0, 1], filter_ops=_cell_ops(ds, [8] * ni, small_vals[:ni], ix, fo))
            assert int(got[ix]) == len({int(r) for r, n in zip(rid, cnt) if n} & set(xs)), (len(ds), ni, ix)
        assert got.sum() > 0


@gpu
def test_shards_missing_a_fragment(ctx):
    """shard 0 holds everything; shard 1 lacks x's fragment, shard 2 the int field's, shard 3 the set field in both of its
    views; shard 4 lacks the set field in one view only and still counts"""
    cols = [5, 6, SW + 5, 2 * SW + 5, 3 * SW + 5, 4 * SW + 5]
    load_x(ctx, {c: {10 * (c // SW + 1)} | ({BIG} if c == 6 else set()) for c in cols if c // SW != 1})
    load_values(ctx, VF[0], {c: 3 for c in cols if c // SW != 2}, 4)
    d = Dim(SF[0], [0], [{0: [5, 6, SW + 5, 2 * SW + 5]}, {0: [6, SW + 5, 2 * SW + 5, 4 * SW + 5]}])
    d.load(ctx)
    ctx.commit()
    sh, xs = [0, 1, 2, 3, 4], [10, 20, 30, 40, 50, BIG]
    assert gbr(ctx, [d], [4], [[3]], xs, sh).tolist() == [[3]]           # 10 and 2^32 (columns 5, 6) and 50
    assert gbr(ctx, [d], [], [], xs, sh).tolist() == [4]                 # and 30: no int dimension to miss
    assert gbr(ctx, [], [4], [[3]], xs, sh).tolist() == [4]              # 10, 2^32, 40, 50
    assert gbr(ctx, [], [4], [[3]], xs, [1]).tolist() == [0]             # x's fragment only is missing


@gpu
def test_zero_rows(ctx):
    load_x(ctx, {1: {3}})
    load_values(ctx, VF[0], {1: 3}, 4)
    ctx.commit()
    d = Dim(SF[0], [], [{}])
    assert gbr(ctx, [d], [4], [[3]], [3], [0]).shape == (0, 1)
    assert gbr(ctx, [Dim(SF[0], [0], [{}]), d], [], [], [3], [0]).shape == (1, 0)


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch and kernel launch, every batch marking the same bitset"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        rng = np.random.default_rng(313)
        ints, dims, values, rows = _set_world(c, rng, 300 if ON_EMU else 1500)
        xr = _x_data(rng, sorted(set(ints[0]) | set(ints[1])), "set")
        load_x(c, xr)
        c.commit()
        xs = _present(xr)
        check(gbr(c, dims[1:2], [8, 8], values, xs, [0, 1, 2]), expect(xr, ints, dims[1:2], values, xs), "b")
        check(gbr(c, [], [8], values[:1], xs, [0, 1, 2], filt(2)), expect(xr, ints[:1], [], values[:1], xs, set(rows[2])), "no b")
        check(gbr(c, dims[2:], [], [], xs, [0, 1, 2]), expect(xr, [], dims[2:], [], xs), "no int")
        check(gbr(c, dims[:2], [], [], xs, [0, 1, 2]), expect(xr, [], dims[:2], [], xs), "peeled")
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
                c.groupby_distinct_rows(IDX, [], [(VF[0], VV, 4, [1, 2])], (XF, XV, [1]), [0])
            assert e.value.code == L.E_COMM and "union" in str(e.value)
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ argument errors
def _raw_call(lib, h, n_fields=1, n_views=None, n_rows=None, n_ints=2, depths=None, n_values=None, values=None, x_rows=None, n_x=None,
              null=None, n_shards=1):
    xv = x_rows if x_rows is not None else [1, 2, 3]
    keep = dict(fields=np.full(8, SF[0], dtype=np.uint32), views=np.zeros(64, dtype=np.uint32),
                n_views=np.asarray(n_views if n_views is not None else [1] * 8, dtype=np.int32),
                rows=np.zeros(64, dtype=np.uint64), n_rows=np.asarray(n_rows if n_rows is not None else [1] * 8, dtype=np.int32),
                vfields=np.asarray(VF + VF + VF[:2], dtype=np.uint32), vviews=np.full(8, VV, dtype=np.uint32),
                depths=np.asarray(depths if depths is not None else [4] * 8, dtype=np.int32),
                values=np.asarray(values if values is not None else list(range(1 << 17)), dtype=np.int64),
                n_values=np.asarray(n_values if n_values is not None else [2] * 8, dtype=np.int32),
                x_rows=np.asarray(xv, dtype=np.uint64), shards=np.zeros(1, dtype=np.uint64), out=np.zeros(1 << 16, dtype=np.uint64))
    p = {k: (None if k == null else a.ctypes.data) for k, a in keep.items()}
    rc = lib.fbgpu_groupby_distinct_rows(h, IDX, p["fields"], p["views"], p["n_views"], n_fields, p["rows"], p["n_rows"], p["vfields"], p["vviews"],
                                         p["depths"], n_ints, p["values"], p["n_values"], XF, XV, p["x_rows"], len(xv) if n_x is None else n_x, None, 0,
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
    ({"n_x": 0}, "n_x=0 < 1"),
    ({"n_x": -3}, "n_x=-3 < 1"),
    ({"x_rows": [1, 4, 4]}, "x_rows are not strictly ascending at position 2"),
    ({"x_rows": [BIG, 5]}, "x_rows are not strictly ascending at position 1"),
    ({"n_shards": -1}, "bad argument"),
] + [({"null": k}, "bad argument") for k in ("fields", "views", "n_views", "rows", "n_rows", "vfields", "values", "x_rows", "shards", "out")]


def test_argument_errors_before_the_device_check():
    """every argument error but n_rows is reported before the device check"""
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for kw, msg in ARG_ERRORS:
            rc, _ = _raw_call(ctx.L, ctx.h, **kw)
            assert rc == L.E_INVALID and ctx.L.fbgpu_last_error().decode() == msg, (kw, msg)
        for kw in ({"n_fields": 0, "null": "fields"}, {"n_ints": 0, "null": "vfields"}, {"n_ints": 0, "null": "values"}, {"x_rows": [0, BIG, (1 << 64) - 1]}, {}):
            rc, _ = _raw_call(ctx.L, ctx.h, **kw)                        # a kind of dimension that is absent may have NULL arrays
            assert rc == L.E_CUDA and "no device" in ctx.L.fbgpu_last_error().decode(), kw
    finally:
        ctx.close()


def test_refused_on_an_inspection_only_context():
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for dims, ints in (([], [(VF[0], VV, 4, [1, 2])]), ([(SF[0], [0], [0, 1])], [])):
            with pytest.raises(L.FbgpuError) as e:
                ctx.groupby_distinct_rows(IDX, dims, ints, (XF, XV, [1, BIG]), [0])
            assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()


def test_no_node_form():
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        with pytest.raises(NotImplementedError):
            node.groupby_distinct_rows(IDX, [], [(VF[0], VV, 4, [1, 2])], (XF, XV, [1]), [0])
    finally:
        node.close()


@gpu
def test_argument_errors_on_a_device(ctx):
    load_values(ctx, VF[0], {1: 0}, 4)
    load_values(ctx, VF[1], {1: 3}, 4)
    load_x(ctx, {1: {2}})
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
    "GroupBy(Rows(a), aggregate=Count(Distinct(field=m)))",
    "GroupBy(Rows(a), Rows(b), aggregate=Count(Distinct(field=s)))",
    "GroupBy(Rows(a), aggregate=Count(Distinct(field=bo)), filter=Row(c=0))",
    "GroupBy(Rows(a), aggregate=Count(Distinct(field=t)))",
    "GroupBy(Rows(a), Rows(b), aggregate=Count(Distinct(Row(c=0), field=m)))",
    "GroupBy(Rows(b), aggregate=Count(Distinct(Row(v > 0), field=s)), filter=Row(c=0))",
    "GroupBy(Rows(v), aggregate=Count(Distinct(field=s)))",
    "GroupBy(Rows(a), Rows(v), aggregate=Count(Distinct(field=m)))",
    "GroupBy(Rows(s), aggregate=Count(Distinct(field=s)))",
    f"GroupBy(Rows(t, {TR}), aggregate=Count(Distinct(field=m)))",
    f"GroupBy(Rows(a), Rows(t, {TR}), Rows(v), aggregate=Count(Distinct(field=s)), filter=Row(c=0))",
    "GroupBy(Rows(a, previous=2), Rows(b, previous=1), aggregate=Count(Distinct(field=s)), limit=4)",
    "GroupBy(Rows(a), Rows(u), aggregate=Count(Distinct(field=m)), limit=5, offset=3)",
    "GroupBy(Rows(a), Rows(b), aggregate=Count(Distinct(field=s)), having=Condition(count >= 4))",
    'GroupBy(Rows(b), Rows(u), aggregate=Count(Distinct(field=m)), sort="aggregate desc", limit=6)',
    'GroupBy(Rows(a), Rows(b), aggregate=Count(Distinct(field=bo)), sort="aggregate desc, count asc")',
    "GroupBy(Rows(a), aggregate=Count(Distinct(Row(c=5), field=s)))",       # an empty x list: every distinct count is 0
]


def _xworld(holder, seed, n):
    """_world's index "g" plus, on the same columns, a mutex field m (one of 40 rows, some at or above 2^32), a bool field bo and
    a set field s (0-6 of 12 rows per column)"""
    _world(holder, seed, n)
    rng = np.random.default_rng(seed)
    cols = rng.choice(3 * SW, n, replace=False).tolist()                 # _world's columns (its first draw)
    idx = holder.indexes["g"]
    idx.create_field("m", "mutex")
    idx.create_field("bo", "bool")
    idx.create_field("s")
    mrows = list(range(20)) + [BIG + r for r in range(20)]
    for col in cols:
        if rng.random() < 0.8:
            holder.set_bit("g", "m", mrows[int(rng.integers(40))], col)
        if rng.random() < 0.7:
            holder.set_bit("g", "bo", int(rng.integers(2)), col)
        for r in rng.choice(12, int(rng.integers(0, 7)), replace=False):
            holder.set_bit("g", "s", int(r), col)
    holder.sync()


def _pair(seed, n):
    dev, ref = X.Holder(), X.Holder(ctx=OracleCtx())
    _xworld(dev, seed, n)
    _xworld(ref, seed, n)
    assert not hasattr(ref.ctx, "groupby_distinct_rows")
    return dev, X.Executor(dev), X.Executor(ref)


@gpu
def test_queries_match_the_composition():
    """the device path against an oracle-backed holder running one Distinct per group: Count(Distinct) over mutex, set, bool and
    time x beside set, int and time-range children, with filter, a Distinct child, previous, limit, offset, having, sort; a
    missing or unknown field is the same error on both"""
    dev, ed, er = _pair(51, 150 if ON_EMU else 1500)
    try:
        for q in (QUERIES[:4] + QUERIES[9:10] if ON_EMU else QUERIES):
            got = ed.execute("g", q)[0]
            assert got == er.execute("g", q)[0], q
            assert got, q
        assert all(g[2] == 0 for g in ed.execute("g", QUERIES[-1])[0])
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
    """with the groups-per-call and bits-per-call caps lowered, the int children's lists and x's row list are cut into slices;
    the result is the composition's"""
    dev, ed, er = _pair(52, 150 if ON_EMU else 1000)
    calls = []
    real = dev.ctx.groupby_distinct_rows
    monkeypatch.setattr(dev.ctx, "groupby_distinct_rows", lambda *a, **kw: calls.append((a[2], a[3])) or real(*a, **kw), raising=False)
    monkeypatch.setattr(X.Executor, "GROUPBY_MIXED_MAX", 7)
    monkeypatch.setattr(X.Executor, "GROUPBY_DISTINCT_BITS", 24)
    try:
        for q, rows_last in (("GroupBy(Rows(a), Rows(v), Rows(w), aggregate=Count(Distinct(field=m)))", 5),
                             ("GroupBy(Rows(u), Rows(w), aggregate=Count(Distinct(field=s)), filter=Row(c=0))", 1),
                             ("GroupBy(Rows(b), aggregate=Count(Distinct(field=s)))", 3)):
            calls.clear()
            got = ed.execute("g", q)[0]
            assert got and got == er.execute("g", q)[0], q
            assert len(calls) > 1, q
            for ints, x in calls:
                groups = int(np.prod([len(d[3]) for d in ints]))
                assert groups <= 7 and (rows_last * groups * len(x[2]) <= 24 or len(x[2]) == 1), q
    finally:
        dev.ctx.close()


@gpu
def test_falls_back_on_comm_and_node(monkeypatch):
    """FBGPU_E_COMM from the call, or the NotImplementedError of a node (no node form), leaves the per-group composition, which
    answers the same"""
    dev, ed, er = _pair(53, 150 if ON_EMU else 600)
    q = "GroupBy(Rows(a), Rows(b), aggregate=Count(Distinct(field=m)), filter=Row(c=0))"
    try:
        want = er.execute("g", q)[0]
        assert ed.execute("g", q)[0] == want
        for exc in (L.FbgpuError(L.E_COMM, "local to one context"), NotImplementedError("no node form")):
            def refuse(*a, exc=exc, **kw):
                raise exc
            monkeypatch.setattr(dev.ctx, "groupby_distinct_rows", refuse, raising=False)
            assert ed.execute("g", q)[0] == want, exc
    finally:
        dev.ctx.close()


@gpu
def test_bounded_queries():
    """a 256-group Count(Distinct) GroupBy over a mutex field asks the library four times (a's row list, the counts, x's rows,
    the distinct counts), not once per group"""
    h = X.Holder()
    try:
        idx = h.create_index("s")
        idx.create_field("a")
        idx.create_field("m", "mutex")
        for col in range(0, 4096 if ON_EMU else 20000, 3):
            h.set_bit("s", "a", col % 256, col)
            h.set_bit("s", "m", (col * 7) % 1000, col)
        h.sync()
        ex = X.Executor(h)
        q = "GroupBy(Rows(a), aggregate=Count(Distinct(field=m)))"
        before = h.ctx.counters()["queries"]
        res = ex.execute("s", q)[0]
        assert len(res) == 256 and all(len(g) == 3 and 0 < g[2] <= g[1] for g in res)
        assert h.ctx.counters()["queries"] - before == 4
    finally:
        h.ctx.close()


# ------------------------------------------------------------------ CPU
def test_groupby_distinct_rows_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_groupby_distinct_rows.py"], timeout=3000)
