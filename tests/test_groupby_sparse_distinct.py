"""fbgpu_groupby_sparse_distinct and fbgpu_groupby_sparse_distinct_rows (GroupBy(..., aggregate=Count(Distinct(field=x))) over
set, mutex, bool or time dimensions of any size, as the sorted list of the cells in a range where some listed value or row of x
is present, with how many are, in one device call) and the GroupBy path built on them.

Entry-point tests compare (cells, distinct) with a Python model built from the bits and values the test wrote, and, where the
dense tensor fits, with the non-zero cells of fbgpu_groupby_distinct / fbgpu_groupby_distinct_rows.  Query-level tests compare
the executor's GroupBy on the sparse path with an oracle-backed holder, which has no distinct call and so runs one Distinct per
group.  The CPU tests check the argument errors and the refusals on a context without a device, the node's refusal and the
executor's fall-back, and run this file's gpu tests on the interpreted kernels."""
import itertools
import math
import types

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from tests.oracle_ctx import OracleCtx
from tests.test_groupby_mixed import I64_MAX, I64_MIN, IDX, NEG0, ON_EMU, SW, VV, Dim, _pool, filt, load_set, load_values
from tests.test_groupby_sparse import ARG_ERRORS, BIG, FIELDS, SHARDS, _lists, _random_world
from tests.test_groupby_sparse import gbs as gbs_counts
from tests.test_groupby_sparse_sum import _nworld

XF = 14                                # the int x (BSI view VV)
XR, XRV = 15, 0                        # the set-like x and its view
gpu = pytest.mark.gpu


def model(dims, lists, xmap, xs, keep=None, start=0, end=None):
    """(cells, distinct) from the written data: dims[i].union = {row: columns}, lists[i] the listed rows of dimension i,
    xmap = {column: set of x's stored values (NEG0 as 0) or rows}, xs x's listed values or rows"""
    per_col = []
    for d, rows in zip(dims, lists):
        pos = {r: i for i, r in enumerate(rows)}
        m = {}
        for r, cols in d.union.items():
            if r in pos:
                for c in cols:
                    m.setdefault(c, []).append(pos[r])
        per_col.append(m)
    stride = [math.prod(len(x) for x in lists[i + 1:]) for i in range(len(lists))]
    listed = set(xs)
    seen = {}
    for c, j0 in per_col[0].items():
        xv = xmap.get(c, set()) & listed
        if not xv or (keep is not None and c not in keep):
            continue
        rest = [m.get(c) for m in per_col[1:]]
        if any(r is None for r in rest):
            continue
        for js in itertools.product(j0, *rest):
            seen.setdefault(sum(j * s for j, s in zip(js, stride)), set()).update(xv)
    cells = sorted(x for x in seen if x >= start and (end is None or x < end))
    return cells, [len(seen[x]) for x in cells]


def int_map(vals):
    return {c: {0 if v is NEG0 else v} for c, v in vals.items()}


def gbsd(ctx, dims, lists, x, shards, filter_ops=None, start=0, end=None):
    """x: (field, BSI view, depth, values) calls the int form, (field, view, rows) the rows form"""
    set_dims = [(d.field, d.views, r) for d, r in zip(dims, lists)]
    call = ctx.groupby_sparse_distinct if len(x) == 4 else ctx.groupby_sparse_distinct_rows
    cells, dist = call(IDX, set_dims, x, shards, filter_ops=filter_ops, start=start, end=end)
    assert cells.dtype == np.uint64 and dist.dtype == np.uint64
    return [int(v) for v in cells], [int(v) for v in dist]


def dense(ctx, dims, lists, x, shards, filter_ops=None):
    set_dims = [(d.field, d.views, r) for d, r in zip(dims, lists)]
    if len(x) == 4:
        t = ctx.groupby_distinct(IDX, set_dims, [], x, shards, filter_ops=filter_ops)
    else:
        t = ctx.groupby_distinct_rows(IDX, set_dims, [], x, shards, filter_ops=filter_ops)
    t = t.reshape(-1)
    nz = np.flatnonzero(t)
    return [int(v) for v in nz], [int(v) for v in t[nz]]


def load_x(ctx, xr, field=XR, view=XRV):
    rows = {}
    for c, rs in xr.items():
        for r in rs:
            rows.setdefault(r, []).append(c)
    load_set(ctx, field, rows, view)


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def _x_data(rng, cols):
    """x on the columns: int values (depth 21) on about 80 % of them, constant over stretches of 200 columns in shard 1 (run
    containers in the planes), a few signs with magnitude 0; set rows 0-3 of 20 per column (a quarter at or above 2^32), one
    row per stretch of 300 columns in shard 1 (run containers)"""
    pool = [int(v) for v in rng.integers(-3000, 3001, 40)]
    vals = {}
    for c in cols:
        if rng.random() < 0.8:
            vals[c] = pool[(c // 200) % 40] if c // SW == 1 else pool[int(rng.integers(40))]
    for c in list(vals)[::97]:
        vals[c] = NEG0
    xpool = list(range(15)) + [BIG + 5 * r for r in range(5)]
    xr = {}
    for c in cols:
        picks = {xpool[(c // 300) % 20]} if c // SW == 1 else {xpool[int(i)] for i in rng.choice(20, int(rng.integers(0, 4)), replace=False)}
        if picks:
            xr[c] = picks
    return vals, xr


def _int_list(vals):
    """every other present stored value, 0 (the sign with magnitude 0) and absent ones, ascending"""
    present = sorted({0 if v is NEG0 else v for v in vals.values()})
    return sorted(set(present[::2]) | {0, -99999, 77777})


def _row_list(xr):
    """x's present rows but one, and absent ones"""
    present = sorted(set().union(*xr.values()))
    return sorted(set(present[1:]) | {999, BIG + 999})


def _distinct_world(ctx, seed, n):
    rng, dims, keep = _random_world(ctx, seed, n)
    cols = sorted(set().union(*[c for d in dims for c in d.union.values()]))
    vals, xr = _x_data(rng, cols)
    load_values(ctx, XF, vals, 21)
    load_x(ctx, xr)
    ctx.commit()
    xi, xs = _int_list(vals), _row_list(xr)
    return rng, dims, keep, [((XF, VV, 21, xi), int_map(vals), xi), ((XR, XRV, xs), xr, xs)]


# ------------------------------------------------------------------ entry point
@gpu
@pytest.mark.parametrize("seed", [0, 1])
def test_random_worlds(ctx, seed):
    """1-3 set, mutex and two-view time dimensions over bitmap, run and array containers, columns past 2^32 and a shard without
    a fragment; an int x and a set x, each with unlisted values or rows; with and without a filter: the model and the dense
    calls' non-zero cells.  Cells whose columns hold no listed x are the ones the counts-only call lists and these do not."""
    rng, dims, keep, xs = _distinct_world(ctx, 700 + seed, 600 if ON_EMU else 6000)
    orders = [(0,), (1, 2), (2, 0, 3)] if ON_EMU else [p for k in (1, 2, 3) for p in itertools.permutations(range(4), k)][::2]
    dropped = 0
    for order in orders:
        ds = [dims[k] for k in order]
        lists = [_lists(rng, d) for d in ds]
        for x, xmap, xl in xs:
            for fo, kp in ((None, None), (filt(0), keep)):
                want = model(ds, lists, xmap, xl, kp)
                assert want[0], (order, len(x))
                got = gbsd(ctx, ds, lists, x, SHARDS, fo)
                assert got == want, (order, len(x), fo is None)
                if len(ds) <= 2 or not ON_EMU:                  # (the dense calls peel 3+ dimensions on the host: slow when interpreted)
                    assert got == dense(ctx, ds, lists, x, SHARDS, fo), (order, len(x), fo is None)
                plain = gbs_counts(ctx, ds, lists, SHARDS, fo)[0]
                assert set(got[0]) <= set(plain)
                dropped += len(set(plain) - set(got[0]))
    assert dropped > 0


@gpu
@pytest.mark.parametrize("depth", [0, 1, 32, 63, 64])
def test_int_depths_with_edge_values(ctx, depth):
    """an int x of each depth with its edge values (INT64_MIN / INT64_MAX at depth 64), signs with magnitude 0 (the value 0)
    and values that are not listed, over columns past 2^32"""
    rng = np.random.default_rng(710 + depth)
    n = 200 if ON_EMU else 2000
    cols = sorted(rng.choice(2 * SW, n, replace=False).tolist() + [4100 * SW + 333 + k for k in range(20)])
    pool = [0] if depth == 0 else _pool(rng, depth, 8)
    vals = {c: pool[int(rng.integers(len(pool)))] for c in cols if rng.random() < 0.9}
    for c in list(vals)[:5]:
        vals[c] = NEG0
    d0 = Dim(FIELDS[0], [3, 9, BIG + 1], [{r: [c for c in cols if rng.random() < 0.4] for r in (3, 9, BIG + 1)}], views=(0,))
    d1 = Dim(FIELDS[1], [0, 1, 2], [{r: [] for r in (0, 1, 2)}], views=(0,))
    for c in cols:
        d1.per_view[0][int(rng.integers(3))].append(c)
    d1 = Dim(FIELDS[1], [0, 1, 2], d1.per_view, views=(0,))
    load_values(ctx, XF, vals, depth)
    for d in (d0, d1):
        d.load(ctx)
    ctx.commit()
    shards = [0, 1, 4, 4100]
    present = sorted({0 if v is NEG0 else v for v in vals.values()})
    edge = [v for v in (I64_MIN, I64_MAX, 0) if v in present]
    assert depth < 64 or I64_MIN in edge
    for listed in (present, sorted(set(present[1::2]) | set(edge))):
        for ds in ([d0], [d1], [d0, d1], [d1, d0]):
            lists = [d.rows for d in ds]
            x = (XF, VV, depth, listed)
            want = model(ds, lists, int_map(vals), listed)
            assert want[0]
            got = gbsd(ctx, ds, lists, x, shards)
            assert got == want == dense(ctx, ds, lists, x, shards), (len(ds), len(listed))


@gpu
def test_set_x_held_several_times_and_x_as_a_dimension(ctx):
    """a column held by several listed x rows counts toward each of them; x may also be one of the group dimensions, where the
    cell of row r counts every listed row that r's columns hold"""
    rng = np.random.default_rng(720)
    cols = rng.choice(3 * SW, 400 if ON_EMU else 4000, replace=False).tolist()
    xr = {c: {int(r) for r in rng.choice(12, int(rng.integers(1, 6)), replace=False)} for c in cols}
    load_x(ctx, xr)
    d0 = Dim(FIELDS[0], [0, 1], [{0: cols[::2], 1: cols[1::3]}], views=(0,))
    d0.load(ctx)
    ctx.commit()
    xs = list(range(12))
    xdim = Dim(XR, xs, [{r: [c for c in cols if r in xr[c]] for r in xs}], views=(XRV,))
    for ds in ([d0], [xdim], [d0, xdim], [xdim, d0]):
        lists = [d.rows for d in ds]
        want = model(ds, lists, xr, xs)
        got = gbsd(ctx, ds, lists, (XR, XRV, xs), [0, 1, 2])
        assert got == want == dense(ctx, ds, lists, (XR, XRV, xs), [0, 1, 2]), len(ds)
        assert max(got[1]) > 1
    held = [len(set().union(*[xr[c] for c in cols if r in xr[c]])) for r in xs]
    assert gbsd(ctx, [xdim], [xs], (XR, XRV, xs), [0, 1, 2]) == (xs, held)
    assert gbsd(ctx, [d0], [[0, 1]], (XR, XRV, xs), [0, 1, 2])[1] == [12, 12]


@gpu
@pytest.mark.parametrize("layout", ["bitmap", "run", "array"])
def test_container_encodings(ctx, layout):
    """x's planes and rows, and a two-view dimension's rows, stored as bitmaps (dense random columns), runs (contiguous columns,
    values and rows in long stretches) and arrays (scattered columns)"""
    rng = np.random.default_rng(730)
    n = 20000 if ON_EMU else 60000
    if layout == "bitmap":
        cols = (np.sort(rng.choice(SW // 8, n, replace=False)) + 3 * 65536).tolist()
        xv = rng.integers(-40, 40, n).tolist()
        xrows = [{int(r) for r in rng.choice(6, int(rng.integers(1, 3)), replace=False)} for _ in range(n)]
        views = [{r: [c for c in cols if rng.random() < 0.5] for r in range(2)} for _ in range(2)]
    elif layout == "run":
        cols = list(range(100, 100 + n))
        xv = np.repeat(rng.integers(-40, 40, n // 1000), 1000).tolist()
        xrows = [{(i // 3000) % 5} for i in range(n)]
        views = [{0: cols[: n // 2], 1: cols[n // 3: n // 3 + 7000]}, {0: cols[n // 4: n // 2 + 3000], 1: cols[5000: 5100]}]
    else:
        cols = rng.choice(3 * SW, 3000 if ON_EMU else 9000, replace=False).tolist()
        xv = rng.integers(-300, 300, len(cols)).tolist()
        xrows = [{int(rng.integers(40))} for _ in cols]
        views = [{r: rng.choice(cols, len(cols) // 2, replace=False).tolist() for r in range(3)} for _ in range(2)]
    vals = dict(zip(cols, xv))
    xr = dict(zip(cols, xrows))
    load_values(ctx, XF, vals, 21)
    load_x(ctx, xr)
    d = Dim(FIELDS[0], sorted(views[0]), views, views=(0, 3))
    d.load(ctx)
    ctx.commit()
    shards = [0, 1, 2]
    xi = sorted(set(xv))[::2]
    xs = sorted(set().union(*xrows))
    for x, xmap, xl in (((XF, VV, 21, xi), int_map(vals), xi), ((XR, XRV, xs), xr, xs)):
        want = model([d], [d.rows], xmap, xl)
        assert want[0]
        assert gbsd(ctx, [d], [d.rows], x, shards) == want == dense(ctx, [d], [d.rows], x, shards), len(x)


@gpu
def test_ranges(ctx):
    """[start, end) inside, between and past the cells, an empty range, and a range whose only cells with columns have no
    listed x (so distinct 0: nothing listed); the NOSPACE contract of the raw call and the wrapper's retry"""
    rng, dims, keep, xs = _distinct_world(ctx, 740, 500 if ON_EMU else 3000)
    ds = [dims[0], dims[1]]
    lists = [_lists(rng, d) for d in ds]
    for x, xmap, xl in xs:
        full = model(ds, lists, xmap, xl)
        cells = full[0]
        assert len(cells) > 20
        gap = next(a + 1 for a, b in zip(cells, cells[1:]) if b > a + 1)
        for start, end in ((0, None), (cells[5], cells[12]), (cells[5] + 1, cells[12] + 1), (gap, cells[-1]), (cells[-1], cells[-1] + 1),
                           (cells[-1] + 1, None), (cells[7], cells[7]), (0, 0), (1 << 63, None)):
            want = model(ds, lists, xmap, xl, start=start, end=end)
            assert gbsd(ctx, ds, lists, x, SHARDS, start=start, end=end) == want, (len(x), start, end)
            assert gbsd(ctx, ds, lists, x, SHARDS, filt(0), start, end) == model(ds, lists, xmap, xl, keep, start, end), (len(x), start, end)
        plain = gbs_counts(ctx, ds, lists, SHARDS)[0]
        zero = [c for c in plain if c not in set(cells)]                   # cells with columns but no listed x
        assert zero
        assert gbsd(ctx, ds, lists, x, SHARDS, start=zero[0], end=zero[0] + 1) == ([], [])
    x, xmap, xl = xs[1]
    full = model(ds, lists, xmap, xl)
    g = L._groupby_args([(d.field, d.views, r) for d, r in zip(ds, lists)], [], SHARDS, None)
    xa = np.asarray(xl, dtype=np.uint64)
    oc, od, n = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64), L.C.c_uint64(0)
    rc = ctx.L.fbgpu_groupby_sparse_distinct_rows(ctx.h, IDX, g.fields, g.views, g.n_views, g.n_fields, g.rows, g.n_rows, XR, XRV, xa.ctypes.data, len(xa),
                                                  None, 0, g.shards, g.n_shards, 0, (1 << 64) - 1, oc.ctypes.data, od.ctypes.data, 4, L.C.byref(n))
    assert rc == L.E_NOSPACE and n.value == len(full[0]) and not oc.any() and not od.any()
    e = full[0][3] + 1
    rc = ctx.L.fbgpu_groupby_sparse_distinct_rows(ctx.h, IDX, g.fields, g.views, g.n_views, g.n_fields, g.rows, g.n_rows, XR, XRV, xa.ctypes.data, len(xa),
                                                  None, 0, g.shards, g.n_shards, 0, e, oc.ctypes.data, od.ctypes.data, 4, L.C.byref(n))
    assert rc == 0 and n.value == 4 and (oc.tolist(), od.tolist()) == (full[0][:4], full[1][:4])
    ctx._sparse_cap = 2                                                      # the wrapper grows its buffers and calls again
    assert gbsd(ctx, ds, lists, x, SHARDS) == full


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch, so a (cell, x) pair met in several batches and shards (x's rows and
    values recur across shards) is merged into the running list and still counted once"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        rng, dims, keep, xs = _distinct_world(c, 750, 500 if ON_EMU else 3000)
        for order in ((0, 1), (2, 3, 1)):
            ds = [dims[k] for k in order]
            lists = [_lists(rng, d) for d in ds]
            for x, xmap, xl in xs:
                for fo, kp in ((None, None), (filt(0), keep)):
                    want = model(ds, lists, xmap, xl, kp)
                    assert gbsd(c, ds, lists, x, SHARDS, fo) == want, (order, len(x))
                    lo, hi = want[0][3], want[0][-3]
                    assert gbsd(c, ds, lists, x, SHARDS, fo, lo, hi) == model(ds, lists, xmap, xl, kp, lo, hi), (order, len(x))
    finally:
        c.close()


@gpu
def test_seven_dimensions(ctx):
    """seven set dimensions beside x, the join's eighth slot"""
    rng = np.random.default_rng(760)
    cols = rng.choice(2 * SW, 300 if ON_EMU else 3000, replace=False).tolist()
    dims = []
    for k in range(7):
        rows = [10 * k + r for r in range(3)]
        dims.append(Dim((FIELDS + (16, 17, 18))[k], rows, [{r: [c for c in cols if rng.random() < 0.6] for r in rows}], views=(0,)))
    for d in dims:
        d.load(ctx)
    vals = {c: int(rng.integers(-5, 6)) for c in cols if rng.random() < 0.9}
    xr = {c: {int(rng.integers(7))} for c in cols}
    load_values(ctx, XF, vals, 8)
    load_x(ctx, xr)
    ctx.commit()
    lists = [d.rows for d in dims]
    for x, xmap, xl in (((XF, VV, 8, list(range(-5, 6))), int_map(vals), list(range(-5, 6))), ((XR, XRV, list(range(7))), xr, list(range(7)))):
        want = model(dims, lists, xmap, xl)
        assert want[0]
        got = gbsd(ctx, dims, lists, x, [0, 1])
        assert got == want, len(x)
        if not ON_EMU:
            assert got == dense(ctx, dims, lists, x, [0, 1]), len(x)
        lo, hi = want[0][len(want[0]) // 3], want[0][-1]
        assert gbsd(ctx, dims, lists, x, [0, 1], start=lo, end=hi) == model(dims, lists, xmap, xl, start=lo, end=hi), len(x)


@gpu
def test_refused_with_ranks_attached():
    a, b = L.Context(0), L.Context(0)
    try:
        L.p2p_open_local([a, b])
        for c in (a, b):
            for call, x in ((c.groupby_sparse_distinct, (XF, VV, 8, [1, 2])), (c.groupby_sparse_distinct_rows, (XR, XRV, [1, 2]))):
                with pytest.raises(L.FbgpuError) as e:
                    call(IDX, [(FIELDS[0], [0], [1, 2])], x, [0])
                assert e.value.code == L.E_COMM
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ argument errors
def _raw_call(lib, h, rows_form, n_fields=1, n_views=None, n_rows=None, rows=None, null=None, n_shards=1, cap=4, xs=None, n_x=2, x_depth=8,
              start=0, end=(1 << 64) - 1):
    keep = dict(fields=np.full(8, FIELDS[0], dtype=np.uint32), views=np.zeros(64, dtype=np.uint32),
                n_views=np.asarray(n_views if n_views is not None else [1] * 8, dtype=np.int32),
                rows=np.asarray(rows if rows is not None else list(range(64)), dtype=np.uint64),
                n_rows=np.asarray(n_rows if n_rows is not None else [2] * 8, dtype=np.int32),
                x=np.asarray(xs if xs is not None else [1, 2], dtype=np.uint64 if rows_form else np.int64),
                shards=np.zeros(1, dtype=np.uint64), cells=np.zeros(4, dtype=np.uint64), counts=np.zeros(4, dtype=np.uint64),
                out_n=np.zeros(1, dtype=np.uint64))
    p = {k: (None if k == null else a.ctypes.data) for k, a in keep.items()}
    p["out_n"] = None if null == "out_n" else keep["out_n"].ctypes.data_as(L.C.POINTER(L.C.c_uint64))
    head = (h, IDX, p["fields"], p["views"], p["n_views"], n_fields, p["rows"], p["n_rows"])
    tail = (None, 0, p["shards"], n_shards, start, end, p["cells"], p["counts"], cap, p["out_n"])
    if rows_form:
        return lib.fbgpu_groupby_sparse_distinct_rows(*head, XR, XRV, p["x"], n_x, *tail)
    return lib.fbgpu_groupby_sparse_distinct(*head, XF, VV, x_depth, p["x"], n_x, *tail)


BIG_ROWS = dict(n_fields=4, n_rows=[1 << 16] * 3 + [(1 << 16) - 1], rows=list(range(1 << 16)) * 3 + list(range((1 << 16) - 1)))
DISTINCT_ERRORS = ARG_ERRORS + [
    ({"n_fields": 8}, "n_fields=8 outside 1..7"),
    ({"null": "x"}, "bad argument"),
    ({"n_x": 0}, "n_x=0 < 1"),
    ({"start": 5, "end": 4}, "start=5 > end=4"),
    (dict(BIG_ROWS, n_x=2), "product of n_rows times 2^1 exceeds 2^64 - 1"),
]
INT_ERRORS = DISTINCT_ERRORS + [({"xs": [2, 2]}, "x_values are not strictly ascending at position 1"),
                                ({"xs": [0, -1]}, "x_values are not strictly ascending at position 1"),
                                ({"x_depth": -1}, "bit depth -1 outside 0..64"), ({"x_depth": 65}, "bit depth 65 outside 0..64")]
ROWS_ERRORS = DISTINCT_ERRORS + [({"xs": [BIG, 3]}, "x_rows are not strictly ascending at position 1")]


def test_argument_errors_before_the_device_check():
    """every argument error is reported before the device check; with cap 0 the outputs may be NULL; one listed x leaves every
    bit of the key to the cell"""
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for rows_form, errors in ((False, INT_ERRORS), (True, ROWS_ERRORS)):
            for kw, msg in errors:
                rc = _raw_call(ctx.L, ctx.h, rows_form, **kw)
                assert rc == L.E_INVALID and ctx.L.fbgpu_last_error().decode() == msg, (rows_form, kw, msg)
            for kw in ({}, {"null": "counts", "cap": 0}, {"n_fields": 7}, {"start": 4, "end": 4}, {"xs": [0, (1 << 64) - 1] if rows_form else [I64_MIN, I64_MAX]},
                       dict(BIG_ROWS, n_x=1), {"x_depth": 0}, {"x_depth": 64}):
                rc = _raw_call(ctx.L, ctx.h, rows_form, **kw)
                assert rc == L.E_CUDA and "no device" in ctx.L.fbgpu_last_error().decode(), (rows_form, kw)
    finally:
        ctx.close()


def test_refused_on_an_inspection_only_context():
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for call, x in ((ctx.groupby_sparse_distinct, (XF, VV, 8, [1, 2])), (ctx.groupby_sparse_distinct_rows, (XR, XRV, [1, BIG]))):
            with pytest.raises(L.FbgpuError) as e:
                call(IDX, [(FIELDS[0], [0, 3], [1, BIG])], x, [0], start=1, end=3)
            assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()


def test_no_node_form_and_the_executor_falls_back():
    """a node raises NotImplementedError for both calls; the executor then returns None, and the per-group composition runs"""
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        for call in (node.groupby_sparse_distinct, node.groupby_sparse_distinct_rows):
            with pytest.raises(NotImplementedError):
                call(IDX, [(FIELDS[0], [0], [1, 2])], (XR, XRV, [1]), [0])
    finally:
        node.close()

    class Refusing:
        def __init__(self, exc):
            self.exc, self.calls = exc, 0

        def row_counts(self, *a, **kw):
            return np.asarray([1, 4], dtype=np.uint64), np.asarray([3, 1], dtype=np.uint64)

        def groupby_sparse_distinct_rows(self, *a, **kw):
            self.calls += 1
            raise self.exc

    ex = X.Executor.__new__(X.Executor)
    f = types.SimpleNamespace(id=1, type="set", name="k")
    idx = types.SimpleNamespace(id=0, fields={"k": f, "x": types.SimpleNamespace(id=2, type="set", name="x")})
    agg = X.pql.Call("Distinct", {"field": "x"})
    for exc in (NotImplementedError("no node form"), L.FbgpuError(L.E_COMM, "local to one context")):
        ex.ctx = Refusing(exc)
        got = ex._groupby_sparse_distinct(idx, [f], [[1, 2]], [{}], None, agg, [(0, None), (1, None)], ([0, 1], [2, 2]), [0])
        assert got is None and ex.ctx.calls == 1, exc
    ex.ctx = Refusing(L.FbgpuError(L.E_INVALID, "bad argument"))
    with pytest.raises(L.FbgpuError):
        ex._groupby_sparse_distinct(idx, [f], [[1, 2]], [{}], None, agg, [(0, None)], ([0], [2]), [0])
    assert ex._groupby_sparse_distinct(idx, [f] * 8, [[1]] * 8, [{}] * 8, None, agg, [(0, None)], ([0], [2]), [0]) is None     # 8 children
    assert ex._groupby_sparse_distinct(idx, [f], [[1]], [{}], None, X.pql.Call("Distinct", {"field": "x", "index": "i"}), [(0, None)], ([0], [2]), [0]) is None


# ------------------------------------------------------------------ query level
TR = "from=2019-01-20T00:00, to=2019-03-10T00:00"
QUERIES = [                                                      # (query, its Rows pre-passes, distinct calls)
    ("GroupBy(Rows(k), aggregate=Count(Distinct(field=v)))", ("Rows(k)",), 1),
    ("GroupBy(Rows(k), Rows(a), aggregate=Count(Distinct(field=b)))", ("Rows(k)", "Rows(a)"), 1),
    ("GroupBy(Rows(a), Rows(k), aggregate=Count(Distinct(field=w)), filter=Row(c=0))", ("Rows(a)", "Rows(k)"), 1),
    ("GroupBy(Rows(k), aggregate=Count(Distinct(Row(c=0), field=a)))", ("Rows(k)",), 1),
    ("GroupBy(Rows(k, previous=250), Rows(a, previous=2), aggregate=Count(Distinct(field=v)), limit=20)", ("Rows(k)", "Rows(a)"), 1),
    ("GroupBy(Rows(k), Rows(b), aggregate=Count(Distinct(field=a)), limit=15, offset=7)", ("Rows(k)", "Rows(b)"), 1),
    ('GroupBy(Rows(k), aggregate=Count(Distinct(field=n)), sort="aggregate desc", limit=10)', ("Rows(k)",), 1),
    ("GroupBy(Rows(k), Rows(a), aggregate=Count(Distinct(field=b)), having=Condition(count > 1))", ("Rows(k)", "Rows(a)"), 1),
    (f"GroupBy(Rows(t, {TR}), Rows(k), aggregate=Count(Distinct(field=v)))", (f"Rows(t, {TR})", "Rows(k)"), 1),
    ("GroupBy(Rows(k), Rows(b), aggregate=Count(Distinct(field=n)), filter=Row(c=0))", ("Rows(k)", "Rows(b)"), 1),
    ("GroupBy(Rows(k), aggregate=Count(Distinct(field=t)), limit=40)", ("Rows(k)",), 1),
    ("GroupBy(Rows(k), aggregate=Count(Distinct(Row(c=5), field=a)), limit=30)", ("Rows(k)",), 0),     # x's list is empty: every count is 0
]


def _pair(seed, n, n_k):
    """test_groupby_sparse_sum's world: k of n_k rows beside a, b, c, t, int fields v, w (Base 1000) and n (Base -10, negative
    stored values)"""
    dev, ref = X.Holder(), X.Holder(ctx=OracleCtx())
    _nworld(dev, seed, n, n_k)
    _nworld(ref, seed, n, n_k)
    assert not hasattr(ref.ctx, "groupby_sparse_distinct") and not hasattr(ref.ctx, "groupby_sparse_distinct_rows")
    return dev, X.Executor(dev), X.Executor(ref)


def _spy(dev, monkeypatch):
    calls = []
    for name in ("groupby_sparse", "groupby_sparse_distinct", "groupby_sparse_distinct_rows"):
        real = getattr(dev.ctx, name)
        monkeypatch.setattr(dev.ctx, name, lambda *a, real=real, name=name, **kw: calls.append((name, a, kw)) or real(*a, **kw), raising=False)
    return calls


def _check_queries(dev, ed, er, queries, monkeypatch):
    """each query against the oracle, asking the library for its Rows pre-passes, the sparse list, x's list (when there are
    groups) and the given number of distinct calls, whatever the number of groups"""
    calls = _spy(dev, monkeypatch)
    for q, pre, n_dist in queries:
        before = dev.ctx.counters()["queries"]
        for p in pre:
            ed.execute("g", p)
        mid = dev.ctx.counters()["queries"]
        calls.clear()
        got = ed.execute("g", q)[0]
        assert got == er.execute("g", q)[0], q
        assert got and all(len(g) == 3 for g in got), q
        assert [c[0] for c in calls if c[0] != "groupby_sparse"] == ["groupby_sparse_distinct" if "field=v" in q or "field=w" in q or "field=n" in q
                                                                     else "groupby_sparse_distinct_rows"] * n_dist, q
        assert dev.ctx.counters()["queries"] - mid == mid - before + 2 + n_dist, q


@gpu
def test_queries_match_the_oracle(monkeypatch):
    """Count(Distinct) on the sparse path against the oracle-backed holder, over k of 300 rows with the dense cap lowered so that
    the queries take it: int and set-like x (a time field too), a filter, a Distinct child, previous, limit, offset, sort on the
    aggregate, having on the count, a time-range child, an int x with a non-zero Base and negative values, and an empty x list"""
    monkeypatch.setattr(X.Executor, "GROUPBY_DENSE_MAX_CELLS", 64)
    dev, ed, er = _pair(81, 150 if ON_EMU else 600, 300)
    try:
        _check_queries(dev, ed, er, QUERIES[:3] + QUERIES[4:5] + QUERIES[10:] if ON_EMU else QUERIES, monkeypatch)
        assert all(g[2] == 0 for g in ed.execute("g", QUERIES[-1][0])[0])
    finally:
        dev.ctx.close()


@gpu
def test_pair_bound_cuts_ranges_and_slices(monkeypatch):
    """with GROUPBY_SPARSE_DISTINCT_PAIRS lowered, the window's cells are cut into several ranges and x's list into several
    slices; the pieces add up to the oracle's answer, and no call may produce more pairs than the bound"""
    monkeypatch.setattr(X.Executor, "GROUPBY_DENSE_MAX_CELLS", 64)
    monkeypatch.setattr(X.Executor, "GROUPBY_SPARSE_DISTINCT_PAIRS", 6)
    dev, ed, er = _pair(82, 150 if ON_EMU else 600, 300)
    calls = _spy(dev, monkeypatch)
    try:
        for q in ("GroupBy(Rows(k), Rows(a), aggregate=Count(Distinct(field=b)), limit=40)", "GroupBy(Rows(k), aggregate=Count(Distinct(field=v)))",
                  "GroupBy(Rows(a), Rows(k), aggregate=Count(Distinct(field=n)), filter=Row(c=0), offset=5, limit=30)"):
            calls.clear()
            got = ed.execute("g", q)[0]
            assert got and got == er.execute("g", q)[0], q
            dist = [c for c in calls if c[0] != "groupby_sparse"]
            assert len(dist) > 2, q
            slices = {tuple(c[1][2][-1]) for c in dist}
            assert len(slices) > 1 or "field=b" in q, q                    # (b has 3 rows: one slice of 3 <= 6)
            assert all(len(s) <= 6 for s in slices), q
            assert all(c[2]["start"] < c[2]["end"] for c in dist), q
    finally:
        dev.ctx.close()


@gpu
def test_more_than_65535_rows(monkeypatch):
    """k of 70,000 rows, which takes the sparse path by its row count, for queries whose limit stops the oracle's per-group
    Distincts early"""
    if ON_EMU:
        pytest.skip("70,000 rows: covered at 300 rows by test_queries_match_the_oracle on the interpreted kernels")
    dev, ed, er = _pair(83, 1500, 70_000)
    try:
        _check_queries(dev, ed, er, [("GroupBy(Rows(k), Rows(a), aggregate=Count(Distinct(field=v)), limit=20)", ("Rows(k)", "Rows(a)"), 1),
                                     ("GroupBy(Rows(k, previous=30000), aggregate=Count(Distinct(field=b)), filter=Row(c=0), limit=10)", ("Rows(k)",), 1)],
                       monkeypatch)
    finally:
        dev.ctx.close()


@gpu
def test_falls_back_on_comm(monkeypatch):
    """FBGPU_E_COMM or NotImplementedError from the calls leaves the per-group composition, which answers the same"""
    monkeypatch.setattr(X.Executor, "GROUPBY_DENSE_MAX_CELLS", 64)
    dev, ed, er = _pair(84, 150 if ON_EMU else 600, 300)
    qs = ["GroupBy(Rows(k), Rows(a), aggregate=Count(Distinct(field=n)), filter=Row(c=0), limit=30)",
          "GroupBy(Rows(k), Rows(b), aggregate=Count(Distinct(field=a)), limit=25)"]
    try:
        want = [er.execute("g", q)[0] for q in qs]
        assert all(want) and [ed.execute("g", q)[0] for q in qs] == want
        for exc in (L.FbgpuError(L.E_COMM, "local to one context"), NotImplementedError("no node form")):
            def refuse(*a, exc=exc, **kw):
                raise exc
            monkeypatch.setattr(dev.ctx, "groupby_sparse_distinct", refuse, raising=False)
            monkeypatch.setattr(dev.ctx, "groupby_sparse_distinct_rows", refuse, raising=False)
            assert [ed.execute("g", q)[0] for q in qs] == want, exc
    finally:
        dev.ctx.close()


# ------------------------------------------------------------------ CPU
def test_groupby_sparse_distinct_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_groupby_sparse_distinct.py"], timeout=3000)
