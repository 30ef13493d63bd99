"""fbgpu_groupby_sparse_sum (GroupBy(..., aggregate=Sum(field=x)) over set, mutex, bool or time dimensions of any size, as the
sorted list of the groups whose columns hold a value of x, with counts and sums, in one device call) and the GroupBy path built
on it.

Entry-point tests compare (cells, counts, sums) with a Python model built from the bits and values the test wrote, and, where the
dense tensor fits, with the non-zero cells of fbgpu_groupby_sum and its sums there.  Query-level tests compare the executor's
GroupBy over a field of more than 65,535 rows with an oracle-backed holder, which has no sparse call.  The CPU tests check the
argument errors and the refusals on a context without a device, the routing of a node, and run this file's gpu tests on the
interpreted kernels."""
import itertools
import math

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from featurebase_b200 import roaring_io
from tests.oracle_ctx import OracleCtx
from tests.test_groupby_mixed import I64_MAX, IDX, NEG0, ON_EMU, SW, VV, Dim, _pool, filt, load_values
from tests.test_groupby_sparse import ARG_ERRORS, BIG, FIELDS, SHARDS, _kworld, _lists, _random_world, window
from tests.test_groupby_sparse import gbs as gbs_counts
from tests.test_groupby_sum import _wrap

AF = 13                                # the aggregate field (BSI view VV)
FAR_COL = 4100 * SW + 333              # columns past 2^32
gpu = pytest.mark.gpu


def model(dims, lists, agg, keep=None):
    """(cells, counts, sums) from the written data: dims[i].union = {row: columns}, lists[i] the listed rows of dimension i,
    agg = {column: stored value or NEG0} of x; only columns holding a value count"""
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
    cnt, tot = {}, {}
    for c, j0 in per_col[0].items():
        if c not in agg or (keep is not None and c not in keep):
            continue
        rest = [m.get(c) for m in per_col[1:]]
        if any(r is None for r in rest):
            continue
        x = 0 if agg[c] is NEG0 else agg[c]
        for js in itertools.product(j0, *rest):
            cell = sum(j * s for j, s in zip(js, stride))
            cnt[cell] = cnt.get(cell, 0) + 1
            tot[cell] = tot.get(cell, 0) + x
    cells = sorted(cnt)
    return cells, [cnt[x] for x in cells], [_wrap(tot[x]) for x in cells]


def gbss(ctx, dims, lists, depth, shards, filter_ops=None, start=0, limit=None):
    cells, counts, sums = ctx.groupby_sparse(IDX, [(d.field, d.views, r) for d, r in zip(dims, lists)], shards, filter_ops=filter_ops,
                                             start=start, limit=limit, agg=(AF, VV, depth))
    assert cells.dtype == np.uint64 and counts.dtype == np.uint64 and sums.dtype == np.int64
    return [int(x) for x in cells], [int(x) for x in counts], [int(x) for x in sums]


def dense(ctx, dims, lists, depth, shards, filter_ops=None):
    counts, sums = ctx.groupby_sum(IDX, [(d.field, d.views, r) for d, r in zip(dims, lists)], [], (AF, VV, depth), shards, filter_ops=filter_ops)
    counts, sums = counts.reshape(-1), sums.reshape(-1)
    nz = np.flatnonzero(counts)
    return [int(x) for x in nz], [int(x) for x in counts[nz]], [int(x) for x in sums[nz]]


def window3(got, start=0, limit=None):
    cells, counts = window(got[0], got[1], start, limit)
    return cells, counts, [got[2][got[0].index(x)] for x in cells]


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def _values(rng, cols, depth=21, skip_shard=2):
    """stored values of x on about 80 % of cols, none in skip_shard (it has no fragment of x); in shard 1 constant over stretches
    of 200 columns (run containers in the planes), a few signs with magnitude 0"""
    agg = {}
    stretch = {}
    top = (1 << depth) - 1
    for c in cols:
        if c // SW == skip_shard or rng.random() >= 0.8:
            continue
        if c // SW == 1:
            agg[c] = stretch.setdefault(c // 200, int(rng.integers(-top, top + 1)))
        else:
            agg[c] = int(rng.integers(-top, top + 1))
    for c in list(agg)[::97]:
        agg[c] = NEG0
    return agg


def _sum_world(ctx, seed, n, depth=21):
    rng, dims, keep = _random_world(ctx, seed, n)
    cols = sorted(set().union(*[c for d in dims for c in d.union.values()]))
    agg = _values(rng, cols, depth)
    load_values(ctx, AF, agg, depth)
    ctx.commit()
    return rng, dims, keep, agg


# ------------------------------------------------------------------ entry point
@gpu
@pytest.mark.parametrize("seed", [0, 1])
def test_random_worlds(ctx, seed):
    """1-4 set, mutex and two-view time dimensions over bitmap, run and array containers, columns past 2^32, a shard without a
    fragment of x and columns without a value, with and without a filter: the model and the dense call's non-zero cells; the
    groups whose columns hold no value are the ones the counts-only call lists and this one does not"""
    rng, dims, keep, agg = _sum_world(ctx, 500 + seed, 600 if ON_EMU else 6000)
    orders = [(0,), (1, 2), (2, 0, 3), (3, 1, 2, 0)] if ON_EMU else [p for k in (1, 2, 3, 4) for p in itertools.permutations(range(4), k)][::3]
    dropped = 0
    for order in orders:
        ds = [dims[k] for k in order]
        lists = [_lists(rng, d) for d in ds]
        for fo, kp in ((None, None), (filt(0), keep)):
            want = model(ds, lists, agg, kp)
            assert want[0], order
            got = gbss(ctx, ds, lists, 21, SHARDS, fo)
            assert got == want, (order, fo is None)
            if len(ds) <= 2 or not ON_EMU:                      # (the dense call peels 3+ dimensions on the host: slow when interpreted)
                assert got == dense(ctx, ds, lists, 21, SHARDS, fo), (order, fo is None)
            plain = gbs_counts(ctx, ds, lists, SHARDS, fo)
            assert set(got[0]) <= set(plain[0])
            dropped += len(set(plain[0]) - set(got[0]))
    assert dropped > 0


@gpu
@pytest.mark.parametrize("depth", [0, 1, 32, 63, 64])
def test_depths_with_edge_values(ctx, depth):
    """x of each depth with its edge values (INT64_MIN / INT64_MAX at depth 64), negative values and signs with magnitude 0; at
    depths 63 and 64 one group's sum wraps"""
    rng = np.random.default_rng(600 + depth)
    n = 200 if ON_EMU else 2000
    cols = sorted(rng.choice(2 * SW, n, replace=False).tolist() + [FAR_COL + k for k in range(20)])
    pool = [0] if depth == 0 else _pool(rng, depth, 8)
    agg = {c: pool[int(rng.integers(len(pool)))] for c in cols if rng.random() < 0.9}
    for c in list(agg)[:5]:
        agg[c] = NEG0
    d0 = Dim(FIELDS[0], [], [{r: [c for c in cols if rng.random() < 0.4] for r in (3, 9, BIG + 1)}])
    d0 = Dim(FIELDS[0], sorted(d0.per_view[0]), d0.per_view, views=(0,))
    wrap_row = 77
    d1 = Dim(FIELDS[1], [], [{r: [] for r in (0, 1, wrap_row)}])
    for c in cols:
        d1.per_view[0][int(rng.integers(2))].append(c)
    if depth >= 63:                                             # row 77 holds five columns of the largest value and no other
        for c in cols[-5:]:
            for r in (0, 1):
                if c in d1.per_view[0][r]:
                    d1.per_view[0][r].remove(c)
            d1.per_view[0][wrap_row].append(c)
            agg[c] = I64_MAX
    d1 = Dim(FIELDS[1], sorted(d1.per_view[0]), d1.per_view, views=(0,))
    load_values(ctx, AF, agg, depth)
    for d in (d0, d1):
        d.load(ctx)
    ctx.commit()
    shards = [0, 1, 4, FAR_COL // SW]
    for ds in ([d0], [d1], [d0, d1], [d1, d0]):
        lists = [d.rows for d in ds]
        want = model(ds, lists, agg)
        assert want[0]
        got = gbss(ctx, ds, lists, depth, shards)
        assert got == want, len(ds)
        assert got == dense(ctx, ds, lists, depth, shards), len(ds)
    if depth == 0:
        assert all(s == 0 for s in gbss(ctx, [d1], [d1.rows], 0, shards)[2])
    if depth >= 63:
        cells, counts, sums = gbss(ctx, [d1], [d1.rows], depth, shards)
        assert (counts[-1], sums[-1]) == (5, _wrap(5 * I64_MAX)) == (5, I64_MAX - 4)


@gpu
@pytest.mark.parametrize("layout", ["bitmap", "run", "array"])
def test_container_encodings(ctx, layout):
    """x's planes and a two-view dimension's rows stored as bitmaps (dense random columns), runs (contiguous columns, values in
    long stretches) and arrays (scattered columns)"""
    rng = np.random.default_rng(611)
    n = 20000 if ON_EMU else 60000
    if layout == "bitmap":
        cols = (np.sort(rng.choice(SW // 8, n, replace=False)) + 3 * 65536).tolist()
        xs = rng.integers(-(1 << 20), 1 << 20, n).tolist()
        views = [{r: [c for c in cols if rng.random() < 0.5] for r in range(2)} for _ in range(2)]
    elif layout == "run":
        cols = list(range(100, 100 + n))
        xs = np.repeat(rng.integers(-(1 << 20), 1 << 20, n // 1000), 1000).tolist()
        views = [{0: cols[: n // 2], 1: cols[n // 3: n // 3 + 7000]}, {0: cols[n // 4: n // 2 + 3000], 1: cols[5000: 5100]}]
    else:
        cols = rng.choice(3 * SW, 3000 if ON_EMU else 9000, replace=False).tolist()
        xs = rng.integers(-300, 300, len(cols)).tolist()
        views = [{r: rng.choice(cols, len(cols) // 2, replace=False).tolist() for r in range(3)} for _ in range(2)]
    agg = dict(zip(cols, xs))
    load_values(ctx, AF, agg, 21)
    d = Dim(FIELDS[0], sorted(views[0]), views, views=(0, 3))
    d.load(ctx)
    ctx.commit()
    shards = [0, 1, 2]
    want = model([d], [d.rows], agg)
    assert gbss(ctx, [d], [d.rows], 21, shards) == want == dense(ctx, [d], [d.rows], 21, shards)


@gpu
def test_windows(ctx):
    """start inside a run of groups, between groups and past the last one; limit 0, 1, exact and past the end (a limit counts
    listed groups); the NOSPACE contract of the raw call and the wrapper's retry"""
    rng, dims, keep, agg = _sum_world(ctx, 520, 500 if ON_EMU else 3000)
    ds = [dims[0], dims[1]]
    lists = [_lists(rng, d) for d in ds]
    full = model(ds, lists, agg)
    cells = full[0]
    assert len(cells) > 20
    gap = next(x + 1 for x, y in zip(cells, cells[1:]) if y > x + 1)
    for start in (0, cells[5], cells[5] + 1, gap, cells[-1], cells[-1] + 1, 1 << 63):
        for limit in (None, 0, 1, 7, len(cells), len(cells) + 5):
            assert gbss(ctx, ds, lists, 21, SHARDS, start=start, limit=limit) == window3(full, start, limit), (start, limit)
            assert gbss(ctx, ds, lists, 21, SHARDS, filt(0), start, limit) == window3(model(ds, lists, agg, keep), start, limit), (start, limit)
    g = L._groupby_args([(d.field, d.views, r) for d, r in zip(ds, lists)], [], SHARDS, None)
    oc, on, os_, n = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.int64), L.C.c_uint64(0)
    args = (ctx.h, IDX, g.fields, g.views, g.n_views, g.n_fields, g.rows, g.n_rows, AF, VV, 21, None, 0, g.shards, g.n_shards, 0)
    rc = ctx.L.fbgpu_groupby_sparse_sum(*args, -1, oc.ctypes.data, on.ctypes.data, os_.ctypes.data, 4, L.C.byref(n))
    assert rc == L.E_NOSPACE and n.value == len(cells) and not oc.any() and not on.any() and not os_.any()
    rc = ctx.L.fbgpu_groupby_sparse_sum(*args, 4, oc.ctypes.data, on.ctypes.data, os_.ctypes.data, 4, L.C.byref(n))
    assert rc == 0 and n.value == 4 and (oc.tolist(), on.tolist(), os_.tolist()) == window3(full, 0, 4)
    ctx._sparse_cap = 2                                                      # the wrapper grows its buffers and calls again
    assert gbss(ctx, ds, lists, 21, SHARDS) == full


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch, the running lists merged across batches, with and without a limit"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        rng, dims, keep, agg = _sum_world(c, 530, 500 if ON_EMU else 3000)
        for order in ((0, 1), (2, 3, 1)):
            ds = [dims[k] for k in order]
            lists = [_lists(rng, d) for d in ds]
            for fo, kp in ((None, None), (filt(0), keep)):
                want = model(ds, lists, agg, kp)
                assert gbss(c, ds, lists, 21, SHARDS, fo) == want, order
                assert gbss(c, ds, lists, 21, SHARDS, fo, start=want[0][3], limit=5) == window3(want, want[0][3], 5), order
    finally:
        c.close()


def _full_rows(ctx, field, rows, shard, lo, hi):
    """rows of `field` holding every column [lo, hi) of `shard` (run containers)"""
    bits = np.concatenate([r * SW + np.arange(lo, hi, dtype=np.uint64) for r in rows])
    ctx.load_fragment(IDX, field, 0, shard, roaring_io.encode(bits))


@gpu
def test_size_limits(ctx):
    """one shard where every column holds a value and every listed row: 1 x 5 x 5 cells of 2^20 columns each, 26 M
    (cell, column) pairs, so the join takes several ranges and the running lists merge across them"""
    if ON_EMU:
        pytest.skip("2^24 pairs and more: too large for the interpreted kernels")
    shard = 5
    _full_rows(ctx, FIELDS[0], [4], shard, 0, SW)
    _full_rows(ctx, FIELDS[1], range(5), shard, 0, SW)
    _full_rows(ctx, FIELDS[2], [BIG + r for r in range(5)], shard, 0, SW)
    depth = 40
    slot_vals = [(-1) ** s * (s + 1) * 987_654_321 for s in range(16)]      # one value per 65,536-column slot
    bits = [np.arange(SW, dtype=np.uint64)]                              # exists
    for s, v in enumerate(slot_vals):
        cs = np.arange(s * 65536, (s + 1) * 65536, dtype=np.uint64)
        if v < 0:
            bits.append(SW + cs)
        bits += [(2 + i) * SW + cs for i in range(depth) if (abs(v) >> i) & 1]
    ctx.load_fragment(IDX, AF, VV, shard, roaring_io.encode(np.concatenate(bits)))
    ctx.commit()
    dims = [(FIELDS[0], [0], [4]), (FIELDS[1], [0], list(range(5))), (FIELDS[2], [0], [BIG + r for r in range(5)])]
    total = 65536 * sum(slot_vals)
    cells, counts, sums = ctx.groupby_sparse(IDX, dims, [shard], agg=(AF, VV, depth))
    assert cells.tolist() == list(range(25)) and counts.tolist() == [SW] * 25 and sums.tolist() == [total] * 25
    cells, counts, sums = ctx.groupby_sparse(IDX, dims, [shard], start=7, limit=3, agg=(AF, VV, depth))
    assert cells.tolist() == [7, 8, 9] and counts.tolist() == [SW] * 3 and sums.tolist() == [total] * 3
    c1, n1, s1 = ctx.groupby_sparse(IDX, dims[:1], [shard], agg=(AF, VV, depth))
    assert (c1.tolist(), n1.tolist(), s1.tolist()) == ([0], [SW], [total])
    counts_d, sums_d = ctx.groupby_sum(IDX, dims, [], (AF, VV, depth), [shard])
    assert counts_d.reshape(-1).tolist() == [SW] * 25 and sums_d.reshape(-1).tolist() == [total] * 25


@gpu
def test_node_equals_context(ctx):
    """a node of two device slots over one GPU lists each slot's shards and merges counts and sums: the context's answer,
    windows included"""
    node = L.Node([0, 0], 1)
    try:
        _sum_world(node, 540, 500 if ON_EMU else 3000)
        rng, dims, keep, agg = _sum_world(ctx, 540, 500 if ON_EMU else 3000)
        for order in ((0,), (1, 3), (2, 0, 1)):
            ds = [dims[k] for k in order]
            lists = [_lists(rng, d) for d in ds]
            cells = model(ds, lists, agg)[0]
            for fo in (None, filt(0)):
                for start, limit in ((0, None), (0, 3), (cells[len(cells) // 2], 4), (cells[-1] + 1, None), (0, 0)):
                    want = gbss(ctx, ds, lists, 21, SHARDS, fo, start, limit)
                    assert gbss(node, ds, lists, 21, SHARDS, fo, start, limit) == want, (order, start, limit)
    finally:
        node.close()


@gpu
def test_refused_with_ranks_attached():
    a, b = L.Context(0), L.Context(0)
    try:
        L.p2p_open_local([a, b])
        for c in (a, b):
            with pytest.raises(L.FbgpuError) as e:
                c.groupby_sparse(IDX, [(FIELDS[0], [0], [1, 2])], [0], agg=(AF, VV, 8))
            assert e.value.code == L.E_COMM
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ argument errors
def _raw_call(lib, h, n_fields=1, n_views=None, n_rows=None, rows=None, null=None, n_shards=1, cap=4, a_depth=8):
    keep = dict(fields=np.full(8, FIELDS[0], dtype=np.uint32), views=np.zeros(64, dtype=np.uint32),
                n_views=np.asarray(n_views if n_views is not None else [1] * 8, dtype=np.int32),
                rows=np.asarray(rows if rows is not None else list(range(64)), dtype=np.uint64),
                n_rows=np.asarray(n_rows if n_rows is not None else [2] * 8, dtype=np.int32),
                shards=np.zeros(1, dtype=np.uint64), cells=np.zeros(4, dtype=np.uint64), counts=np.zeros(4, dtype=np.uint64),
                sums=np.zeros(4, dtype=np.int64), out_n=np.zeros(1, dtype=np.uint64))
    p = {k: (None if k == null else a.ctypes.data) for k, a in keep.items()}
    p["out_n"] = None if null == "out_n" else keep["out_n"].ctypes.data_as(L.C.POINTER(L.C.c_uint64))
    return lib.fbgpu_groupby_sparse_sum(h, IDX, p["fields"], p["views"], p["n_views"], n_fields, p["rows"], p["n_rows"], AF, VV, a_depth, None, 0,
                                        p["shards"], n_shards, 0, -1, p["cells"], p["counts"], p["sums"], cap, p["out_n"])


SUM_ARG_ERRORS = ARG_ERRORS + [({"a_depth": -1}, "bit depth -1 outside 0..64"), ({"a_depth": 65}, "bit depth 65 outside 0..64"),
                               ({"null": "sums"}, "bad argument")]


def _check_errors(lib, h):
    for kw, msg in SUM_ARG_ERRORS:
        rc = _raw_call(lib, h, **kw)
        assert rc == L.E_INVALID and lib.fbgpu_last_error().decode() == msg, (kw, msg)


def test_argument_errors_before_the_device_check():
    """every argument error is reported before the device check, on a context and on a node; with cap 0 the outputs may be NULL"""
    ctx = L.Context(L.DEVICE_NONE)
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        _check_errors(ctx.L, ctx.h)
        _check_errors(node.L, node.h)
        for kw in ({}, {"null": "sums", "cap": 0}, {"a_depth": 0}, {"a_depth": 64}, {"rows": [0, (1 << 64) - 1]}):
            rc = _raw_call(ctx.L, ctx.h, **kw)
            assert rc == L.E_CUDA and "no device" in ctx.L.fbgpu_last_error().decode(), kw
    finally:
        ctx.close()
        node.close()


def test_refused_on_an_inspection_only_context():
    ctx = L.Context(L.DEVICE_NONE)
    try:
        with pytest.raises(L.FbgpuError) as e:
            ctx.groupby_sparse(IDX, [(FIELDS[0], [0, 3], [1, BIG])], [0], agg=(AF, VV, 8))
        assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()


def test_node_routing():
    """Node inherits the agg form of groupby_sparse, and its calls go to fbgpu_node_groupby_sparse_sum"""
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        assert node.L.fbgpu_groupby_sparse_sum is node.L._real.fbgpu_node_groupby_sparse_sum
        with pytest.raises(L.FbgpuError) as e:
            node.groupby_sparse(IDX, [(FIELDS[0], [0], [1, 2])], [0], start=1, limit=3, agg=(AF, VV, 8))
        assert e.value.code == L.E_CUDA and "no device" in str(e.value)
        with pytest.raises(L.FbgpuError) as e:
            node.groupby_sparse(IDX, [(FIELDS[0], [0], [1, 2])], [0], agg=(AF, VV, 65))
        assert e.value.code == L.E_INVALID and "bit depth 65" in str(e.value)
    finally:
        node.close()


# ------------------------------------------------------------------ query level
TR = "from=2019-01-20T00:00, to=2019-03-10T00:00"
QUERIES = [                                                      # (query, its Rows pre-passes)
    ("GroupBy(Rows(k), Rows(a), aggregate=Sum(field=v))", ("Rows(k)", "Rows(a)")),
    ("GroupBy(Rows(a), Rows(k), aggregate=Sum(field=w), filter=Row(c=0))", ("Rows(a)", "Rows(k)")),
    ("GroupBy(Rows(k, previous=250), Rows(a, previous=2), aggregate=Sum(field=v), limit=20)", ("Rows(k)", "Rows(a)")),
    ("GroupBy(Rows(k), Rows(b), aggregate=Sum(field=v), limit=15, offset=7)", ("Rows(k)", "Rows(b)")),
    ('GroupBy(Rows(k), aggregate=Sum(field=v), sort="aggregate desc", limit=10)', ("Rows(k)",)),
    ('GroupBy(Rows(a), Rows(k), aggregate=Sum(field=w), sort="sum asc, count desc", limit=30)', ("Rows(a)", "Rows(k)")),
    ("GroupBy(Rows(k), Rows(a), aggregate=Sum(field=v), having=Condition(sum > 0))", ("Rows(k)", "Rows(a)")),
    (f"GroupBy(Rows(t, {TR}), Rows(k), aggregate=Sum(field=v))", (f"Rows(t, {TR})", "Rows(k)")),
    ("GroupBy(Rows(k), Rows(b), aggregate=Sum(field=n), filter=Row(c=0))", ("Rows(k)", "Rows(b)")),
]


def _nworld(holder, seed, n, n_k):
    """test_groupby_sparse's world plus an int field n over [-50, -10] (Base -10, negative stored values) on most columns"""
    _kworld(holder, seed, n, n_k)
    holder.indexes["g"].create_field("n", "int", min=-50, max=-10)
    cols = np.random.default_rng(seed).choice(3 * SW, n, replace=False).tolist()       # _world's columns (its first draw)
    rng = np.random.default_rng(seed + 1)
    for c in cols[: n * 4 // 5] + [(i * 23) % (2 * SW) for i in range(0, n_k, 7)]:
        holder.set_value("g", "n", c, int(rng.integers(-50, -9)))
    holder.sync()


def _pair(seed, n, n_k):
    dev, ref = X.Holder(), X.Holder(ctx=OracleCtx())
    _nworld(dev, seed, n, n_k)
    _nworld(ref, seed, n, n_k)
    assert not hasattr(ref.ctx, "groupby_sparse")
    assert dev.indexes["g"].fields["n"].base == -10
    return dev, X.Executor(dev), X.Executor(ref)


def _check_queries(dev, ed, er, queries, monkeypatch):
    calls = []
    real = dev.ctx.groupby_sparse
    monkeypatch.setattr(dev.ctx, "groupby_sparse", lambda *a, **kw: calls.append(kw) or real(*a, **kw), raising=False)
    for q, pre in queries:
        before = dev.ctx.counters()["queries"]
        for p in pre:
            ed.execute("g", p)
        mid = dev.ctx.counters()["queries"]
        calls.clear()
        got = ed.execute("g", q)[0]
        assert dev.ctx.counters()["queries"] - mid == mid - before + 1, q          # the Rows pre-passes, then one call
        assert got == er.execute("g", q)[0], q
        assert got and len(calls) == 1 and calls[0].get("agg") is not None, q


@gpu
def test_queries_match_the_oracle(monkeypatch):
    """aggregate=Sum on the sparse path against the oracle-backed holder, over k of 300 rows with the dense cap lowered so that
    the queries take it (the oracle runs one Sum per group, so every group of a 70,000-row k would cost one oracle query): Rows(a)
    beside it, a filter, previous, limit, offset, sort on the aggregate, having on the sum, a time-range child and an int field
    with a non-zero Base and negative values.  Each query asks the library once beyond its Rows pre-passes, through the agg form
    of groupby_sparse."""
    monkeypatch.setattr(X.Executor, "GROUPBY_DENSE_MAX_CELLS", 64)
    dev, ed, er = _pair(71, 150 if ON_EMU else 600, 300)
    try:
        _check_queries(dev, ed, er, QUERIES, monkeypatch)
    finally:
        dev.ctx.close()


@gpu
def test_more_than_65535_rows(monkeypatch):
    """the same over k of 70,000 rows, which takes the sparse path by its row count, for queries whose limit stops the oracle's
    per-group Sums early"""
    if ON_EMU:
        pytest.skip("70,000 rows: covered at 300 rows by test_queries_match_the_oracle on the interpreted kernels")
    dev, ed, er = _pair(72, 1500, 70_000)
    try:
        _check_queries(dev, ed, er, [("GroupBy(Rows(k), Rows(a), aggregate=Sum(field=v), limit=20)", ("Rows(k)", "Rows(a)")),
                                     ("GroupBy(Rows(k, previous=30000), aggregate=Sum(field=n), filter=Row(c=0), limit=10)", ("Rows(k)",))],
                       monkeypatch)
    finally:
        dev.ctx.close()


@gpu
def test_falls_back_on_comm(monkeypatch):
    """FBGPU_E_COMM or NotImplementedError from the call leaves the dense fbgpu_groupby_sum path, which answers the same when the
    tensor fits"""
    monkeypatch.setattr(X.Executor, "GROUPBY_DENSE_MAX_CELLS", 64)
    dev, ed, er = _pair(73, 150 if ON_EMU else 600, 300)
    q = "GroupBy(Rows(k), Rows(a), aggregate=Sum(field=n), filter=Row(c=0), limit=30)"
    try:
        want = er.execute("g", q)[0]
        assert want and ed.execute("g", q)[0] == want
        for exc in (L.FbgpuError(L.E_COMM, "local to one context"), NotImplementedError("no node form")):
            def refuse(*a, exc=exc, **kw):
                raise exc
            monkeypatch.setattr(dev.ctx, "groupby_sparse", refuse, raising=False)
            assert ed.execute("g", q)[0] == want, exc
    finally:
        dev.ctx.close()


# ------------------------------------------------------------------ CPU
def test_groupby_sparse_sum_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_groupby_sparse_sum.py"], timeout=3000)
