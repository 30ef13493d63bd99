"""fbgpu_groupby_sparse (GroupBy over set, mutex, bool or time dimensions of any size as a sorted list of its non-empty groups, in
one device call) and the GroupBy path built on it.

Entry-point tests compare (cells, counts) with np.flatnonzero of fbgpu_groupby_views' dense tensor where it fits, and always with
a Python model built from the bits the test wrote.  Query-level tests compare the executor's GroupBy over a field of more than
65,535 rows with an oracle-backed holder, which is dense and has no row cap.  The CPU tests check the argument errors and the
refusals on a context without a device, the routing of a node, and run this file's gpu tests on the interpreted kernels."""
import itertools
import math

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from tests.oracle_ctx import OracleCtx
from tests.test_groupby_mixed import FILT, IDX, ON_EMU, SW, Dim, _world, filt, load_set

BIG = 1 << 32                          # row ids at and above 2^32
FAR = 4100                             # a shard whose columns lie past 2^32
FIELDS = (6, 8, 9, 13)                 # one set field per dimension
gpu = pytest.mark.gpu


def model(dims, lists, keep=None):
    """(cells, counts) from the written data: dims[i].union = {row: columns}, lists[i] the listed rows of dimension i"""
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
    cnt = {}
    for c, j0 in per_col[0].items():
        if keep is not None and c not in keep:
            continue
        rest = [m.get(c) for m in per_col[1:]]
        if any(r is None for r in rest):
            continue
        for js in itertools.product(j0, *rest):
            cell = sum(j * s for j, s in zip(js, stride))
            cnt[cell] = cnt.get(cell, 0) + 1
    cells = sorted(cnt)
    return cells, [cnt[x] for x in cells]


def window(cells, counts, start=0, limit=None):
    k = [i for i, x in enumerate(cells) if x >= start]
    k = k if limit is None else k[:limit]
    return [cells[i] for i in k], [counts[i] for i in k]


def gbs(ctx, dims, lists, shards, filter_ops=None, start=0, limit=None):
    cells, counts = ctx.groupby_sparse(IDX, [(d.field, d.views, r) for d, r in zip(dims, lists)], shards, filter_ops=filter_ops, start=start, limit=limit)
    assert cells.dtype == np.uint64 and counts.dtype == np.uint64
    return [int(x) for x in cells], [int(x) for x in counts]


def dense(ctx, dims, lists, shards, filter_ops=None):
    t = ctx.groupby_views(IDX, [d.field for d in dims], [d.views for d in dims], lists, shards, filter_ops=filter_ops).reshape(-1)
    nz = np.flatnonzero(t)
    return [int(x) for x in nz], [int(x) for x in t[nz]]


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def _columns(rng, n):
    """n columns: dense random ones in shard 0 (bitmap containers), clustered runs in shard 1, scattered ones in shard 2 (arrays)
    and a few past 2^32 in shard FAR; shard 3 holds nothing"""
    a = rng.choice(65536, n // 2, replace=False)
    run0 = SW + 1000 + 3 * int(rng.integers(1000))
    b = np.arange(run0, run0 + n // 4)
    c = 2 * SW + rng.choice(SW, n // 8, replace=False)
    d = FAR * SW + rng.choice(SW, n // 8, replace=False)
    return sorted(set(np.concatenate([a, b, c, d]).tolist()))


def _dim(rng, k, kind, cols, n_rows):
    """dimension k over cols: `set` 0-3 rows per column, `mutex` one row per column, `time` 0-2 rows per column in each of two
    views; a quarter of the row ids lie at or above 2^32"""
    pool = [int(r) for r in rng.choice(n_rows, min(n_rows, 40), replace=False)]
    pool = [r + BIG if i % 4 == 0 else r for i, r in enumerate(pool)]
    views = [{}, {}] if kind == "time" else [{}]
    for c in cols:
        for m in views:
            if kind == "mutex":
                picks = [pool[int(rng.integers(len(pool)))]] if rng.random() < 0.9 else []
            else:
                picks = [pool[int(i)] for i in rng.choice(len(pool), int(rng.integers(0, 3 if kind == "time" else 4)), replace=False)]
            for r in picks:
                m.setdefault(r, []).append(c)
    return Dim(FIELDS[k], sorted(set(pool)), views, views=(0, 3))


def _lists(rng, d):
    """the dimension's row list: its present rows but one, plus absent ones (some at or above 2^32)"""
    present = sorted(d.union)
    return sorted(set(present[1:]) | {7_000_003, BIG + 123_456, int(rng.integers(100))})


SHARDS = [0, 1, 2, 3, FAR]


def _random_world(ctx, seed, n):
    rng = np.random.default_rng(seed)
    cols = _columns(rng, n)
    dims = [_dim(rng, k, kind, cols, 60) for k, kind in enumerate(("set", "mutex", "time", "set"))]
    for d in dims:
        d.load(ctx)
    keep = [c for c in cols if rng.random() < 0.5]
    load_set(ctx, FILT, {0: keep})
    ctx.commit()
    return rng, dims, set(keep)


# ------------------------------------------------------------------ entry point
@gpu
@pytest.mark.parametrize("seed", [0, 1])
def test_random_worlds(ctx, seed):
    """1-4 set, mutex and two-view time dimensions over bitmap, run and array containers, columns past 2^32, a shard without a
    fragment, listed rows that are absent and present rows that are not listed, with and without a filter: the dense tensor's
    non-zero cells and the model"""
    rng, dims, keep = _random_world(ctx, 400 + seed, 600 if ON_EMU else 6000)
    orders = [(0,), (1, 2), (2, 0, 3), (3, 1, 2, 0)] if ON_EMU else [p for k in (1, 2, 3, 4) for p in itertools.permutations(range(4), k)][::3]
    for order in orders:
        ds = [dims[k] for k in order]
        lists = [_lists(rng, d) for d in ds]
        for fo, kp in ((None, None), (filt(0), keep)):
            want = model(ds, lists, kp)
            assert want[0], order
            got = gbs(ctx, ds, lists, SHARDS, fo)
            assert got == want, (order, fo is None)
            if len(ds) <= 2 or not ON_EMU:                      # (fbgpu_groupby_views peels 3+ dimensions on the host: slow when interpreted)
                assert got == dense(ctx, ds, lists, SHARDS, fo), (order, fo is None)


@gpu
def test_large_dimensions(ctx):
    """a dimension of 100,000 listed rows beside a small one, and two dimensions whose product exceeds 2^32: beyond what the dense
    tensor holds, against the model"""
    rng = np.random.default_rng(410)
    n = 3000 if ON_EMU else 40000
    cols = _columns(rng, n)
    big = Dim(FIELDS[0], [], [{}])
    rows = rng.choice(100_000, len(cols), replace=True)
    for c, r in zip(cols, rows):
        big.per_view[0].setdefault(int(r) + (BIG if r % 3 == 0 else 0), []).append(c)
    big = Dim(FIELDS[0], sorted(big.per_view[0]), big.per_view)
    small = _dim(rng, 1, "set", cols, 50)
    other = Dim(FIELDS[2], [], [{}])
    for c in cols:
        other.per_view[0].setdefault(int(rng.integers(70_000)), []).append(c)
    other = Dim(FIELDS[2], sorted(other.per_view[0]), other.per_view)
    for d in (big, small, other):
        d.load(ctx)
    load_set(ctx, FILT, {0: cols[::3]})
    ctx.commit()
    lbig = sorted(set(range(100_000)) | {r for r in big.union})            # 100,000 ids and more, most of them absent
    lother = list(range(70_000))
    assert len(lbig) >= 100_000 and len(lbig) * len(lother) > 1 << 32
    for ds, lists, fo, kp in (([big], [lbig], None, None), ([big, small], [lbig, small.rows], None, None),
                              ([small, big], [small.rows, lbig], filt(0), set(cols[::3])), ([big, other], [lbig, lother], None, None),
                              ([other, small, big], [lother, small.rows, lbig], filt(0), set(cols[::3]))):
        want = model(ds, lists, kp)
        assert want[0]
        assert gbs(ctx, ds, lists, SHARDS, fo) == want, len(ds)
    assert max(model([big, other], [lbig, lother])[0]) >= 1 << 32


@gpu
def test_windows(ctx):
    """start inside a run of groups, between groups and past the last one; limit 0, 1, exact and past the end; the NOSPACE
    contract of the raw call and the wrapper's retry"""
    rng, dims, keep = _random_world(ctx, 420, 500 if ON_EMU else 3000)
    ds = [dims[0], dims[1]]
    lists = [_lists(rng, d) for d in ds]
    cells, counts = model(ds, lists)
    assert len(cells) > 20
    gap = next(x + 1 for x, y in zip(cells, cells[1:]) if y > x + 1)      # a start between two groups
    for start in (0, cells[5], cells[5] + 1, gap, cells[-1], cells[-1] + 1, 1 << 63):
        for limit in (None, 0, 1, 7, len(cells), len(cells) + 5):
            assert gbs(ctx, ds, lists, SHARDS, start=start, limit=limit) == window(cells, counts, start, limit), (start, limit)
            assert gbs(ctx, ds, lists, SHARDS, filt(0), start, limit) == window(*model(ds, lists, keep), start, limit), (start, limit)
    g = L._groupby_args([(d.field, d.views, r) for d, r in zip(ds, lists)], [], SHARDS, None)
    out_c, out_n, n = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64), L.C.c_uint64(0)
    rc = ctx.L.fbgpu_groupby_sparse(ctx.h, IDX, g.fields, g.views, g.n_views, g.n_fields, g.rows, g.n_rows, None, 0, g.shards, g.n_shards, 0, -1,
                                    out_c.ctypes.data, out_n.ctypes.data, 4, L.C.byref(n))
    assert rc == L.E_NOSPACE and n.value == len(cells) and not out_c.any() and not out_n.any()
    rc = ctx.L.fbgpu_groupby_sparse(ctx.h, IDX, g.fields, g.views, g.n_views, g.n_fields, g.rows, g.n_rows, None, 0, g.shards, g.n_shards, 0, 4,
                                    out_c.ctypes.data, out_n.ctypes.data, 4, L.C.byref(n))
    assert rc == 0 and n.value == 4 and out_c.tolist() == cells[:4] and out_n.tolist() == counts[:4]
    ctx._sparse_cap = 2                                                      # the wrapper grows its buffers and calls again
    assert gbs(ctx, ds, lists, SHARDS) == (cells, counts)


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch, the running list merged across batches, with and without a limit"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        rng, dims, keep = _random_world(c, 430, 500 if ON_EMU else 3000)
        for order in ((0, 1), (2, 3, 1)):
            ds = [dims[k] for k in order]
            lists = [_lists(rng, d) for d in ds]
            for fo, kp in ((None, None), (filt(0), keep)):
                want = model(ds, lists, kp)
                assert gbs(c, ds, lists, SHARDS, fo) == want, order
                assert gbs(c, ds, lists, SHARDS, fo, start=want[0][3], limit=5) == window(*want, want[0][3], 5), order
    finally:
        c.close()


@gpu
def test_node_equals_context(ctx):
    """a node of two device slots over one GPU lists each slot's shards and merges them: the context's answer, windows included"""
    node = L.Node([0, 0], 1)
    try:
        _random_world(node, 440, 500 if ON_EMU else 3000)
        rng, dims, keep = _random_world(ctx, 440, 500 if ON_EMU else 3000)
        for order in ((0,), (1, 3), (2, 0, 1)):
            ds = [dims[k] for k in order]
            lists = [_lists(rng, d) for d in ds]
            cells = model(ds, lists)[0]
            for fo in (None, filt(0)):
                for start, limit in ((0, None), (0, 3), (cells[len(cells) // 2], 4), (cells[-1] + 1, None), (0, 0)):
                    want = gbs(ctx, ds, lists, SHARDS, fo, start, limit)
                    assert gbs(node, ds, lists, SHARDS, fo, start, limit) == want, (order, start, limit)
    finally:
        node.close()


@gpu
def test_refused_with_ranks_attached():
    a, b = L.Context(0), L.Context(0)
    try:
        L.p2p_open_local([a, b])
        for c in (a, b):
            with pytest.raises(L.FbgpuError) as e:
                c.groupby_sparse(IDX, [(FIELDS[0], [0], [1, 2])], [0])
            assert e.value.code == L.E_COMM
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ argument errors
def _raw_call(lib, h, n_fields=1, n_views=None, n_rows=None, rows=None, null=None, n_shards=1, cap=4):
    keep = dict(fields=np.full(8, FIELDS[0], dtype=np.uint32), views=np.zeros(64, dtype=np.uint32),
                n_views=np.asarray(n_views if n_views is not None else [1] * 8, dtype=np.int32),
                rows=np.asarray(rows if rows is not None else list(range(64)), dtype=np.uint64),
                n_rows=np.asarray(n_rows if n_rows is not None else [2] * 8, dtype=np.int32),
                shards=np.zeros(1, dtype=np.uint64), cells=np.zeros(4, dtype=np.uint64), counts=np.zeros(4, dtype=np.uint64), out_n=np.zeros(1, dtype=np.uint64))
    p = {k: (None if k == null else a.ctypes.data) for k, a in keep.items()}
    p["out_n"] = None if null == "out_n" else keep["out_n"].ctypes.data_as(L.C.POINTER(L.C.c_uint64))
    return lib.fbgpu_groupby_sparse(h, IDX, p["fields"], p["views"], p["n_views"], n_fields, p["rows"], p["n_rows"], None, 0, p["shards"], n_shards,
                                    0, -1, p["cells"], p["counts"], cap, p["out_n"])


ARG_ERRORS = [
    ({"n_fields": 0}, "n_fields=0 outside 1..8"),
    ({"n_fields": 9}, "n_fields=9 outside 1..8"),
    ({"n_fields": 2, "n_views": [1, 0]}, "n_views[1]=0 < 1"),
    ({"n_fields": 2, "n_rows": [2, 0]}, "n_rows[1]=0 < 1"),
    ({"n_rows": [-1]}, "n_rows[0]=-1 < 1"),
    ({"rows": [3, 3]}, "row_ids[0] are not strictly ascending at position 1"),
    ({"n_fields": 2, "rows": [1, 2, BIG, 5]}, "row_ids[1] are not strictly ascending at position 1"),
    ({"n_shards": -1}, "bad argument"),
] + [({"null": k}, "bad argument") for k in ("fields", "views", "n_views", "rows", "n_rows", "cells", "counts", "out_n")]


def _check_errors(lib, h):
    for kw, msg in ARG_ERRORS:
        rc = _raw_call(lib, h, **kw)
        assert rc == L.E_INVALID and lib.fbgpu_last_error().decode() == msg, (kw, msg)


def test_argument_errors_before_the_device_check():
    """every argument error is reported before the device check, on a context and on a node; with cap 0 the outputs may be NULL"""
    ctx = L.Context(L.DEVICE_NONE)
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        _check_errors(ctx.L, ctx.h)
        _check_errors(node.L, node.h)
        for kw in ({}, {"null": "cells", "cap": 0}, {"rows": [0, (1 << 64) - 1]}, {"n_fields": 2, "n_rows": [65536, 1], "rows": list(range(65537))}):
            rc = _raw_call(ctx.L, ctx.h, **kw)
            assert rc == L.E_CUDA and "no device" in ctx.L.fbgpu_last_error().decode(), kw
    finally:
        ctx.close()
        node.close()


def test_product_overflow_is_an_argument_error():
    """four dimensions of 2^16 rows make 2^64 cells, one too many; with one row fewer the product fits"""
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for last, code, msg in ((1 << 16, L.E_INVALID, "product of n_rows exceeds 2^64 - 1"), ((1 << 16) - 1, L.E_CUDA, "no device")):
            with pytest.raises(L.FbgpuError) as e:
                ctx.groupby_sparse(IDX, [(FIELDS[0], [0], np.arange(1 << 16))] * 3 + [(FIELDS[1], [0], np.arange(last))], [0])
            assert e.value.code == code and msg in str(e.value), last
    finally:
        ctx.close()


def test_refused_on_an_inspection_only_context():
    ctx = L.Context(L.DEVICE_NONE)
    try:
        with pytest.raises(L.FbgpuError) as e:
            ctx.groupby_sparse(IDX, [(FIELDS[0], [0, 3], [1, BIG])], [0])
        assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()


def test_node_routing():
    """Node inherits groupby_sparse, and its calls go to fbgpu_node_groupby_sparse"""
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        assert node.L.fbgpu_groupby_sparse is node.L._real.fbgpu_node_groupby_sparse
        with pytest.raises(L.FbgpuError) as e:
            node.groupby_sparse(IDX, [(FIELDS[0], [0], [1, 2])], [0], start=1, limit=3)
        assert e.value.code == L.E_CUDA and "no device" in str(e.value)
        with pytest.raises(L.FbgpuError) as e:
            node.groupby_sparse(IDX, [(FIELDS[0], [0], [2, 1])], [0])
        assert e.value.code == L.E_INVALID and "not strictly ascending" in str(e.value)
    finally:
        node.close()


# ------------------------------------------------------------------ query level
TR = "from=2019-01-20T00:00, to=2019-03-10T00:00"
QUERIES = [
    "GroupBy(Rows(k))",
    "GroupBy(Rows(k), Rows(a))",
    "GroupBy(Rows(a), Rows(k), filter=Row(c=0))",
    "GroupBy(Rows(k, previous=250), Rows(a, previous=2), limit=20)",
    "GroupBy(Rows(k), Rows(b), limit=15, offset=7)",
    "GroupBy(Rows(b), Rows(k), offset=3)",
    'GroupBy(Rows(a), Rows(k), sort="count desc", limit=10)',
    "GroupBy(Rows(k), Rows(a), having=Condition(count >= 2))",
    f"GroupBy(Rows(t, {TR}), Rows(k))",
    "GroupBy(Rows(k), Rows(a), aggregate=Sum(field=v), limit=12)",
    "GroupBy(Rows(a), Rows(k), aggregate=Count(Distinct(field=b)), filter=Row(c=0), limit=25)",
]


def _kworld(holder, seed, n, n_k):
    """_world's index "g" plus a set field k holding n_k rows: row i on column i of a run over shards 0 and 1, and on a few of
    _world's columns"""
    _world(holder, seed, n)
    rng = np.random.default_rng(seed)
    holder.indexes["g"].create_field("k")
    cols = rng.choice(3 * SW, n, replace=False).tolist()                 # _world's columns (its first draw)
    for i in range(n_k):
        holder.set_bit("g", "k", i if i % 5 else BIG + i, (i * 23) % (2 * SW))
    for c in cols:
        holder.set_bit("g", "k", int(rng.integers(n_k)), c)
    holder.sync()


def _pair(seed, n, n_k):
    dev, ref = X.Holder(), X.Holder(ctx=OracleCtx())
    _kworld(dev, seed, n, n_k)
    _kworld(ref, seed, n, n_k)
    assert not hasattr(ref.ctx, "groupby_sparse")
    return dev, X.Executor(dev), X.Executor(ref)


@gpu
def test_queries_match_the_oracle(monkeypatch):
    """the sparse path against the oracle-backed holder over k of more than 65,535 rows (on the interpreted kernels: 300 rows,
    with the dense cap lowered so that they take it): filter, previous, limit, offset, sort, having, a time-range child, Sum and
    Count(Distinct); plain ones ask the library once for the groups beyond the Rows pre-passes"""
    n_k = 300 if ON_EMU else 70_000
    if ON_EMU:
        monkeypatch.setattr(X.Executor, "GROUPBY_DENSE_MAX_CELLS", 64)
    dev, ed, er = _pair(61, 150 if ON_EMU else 1500, n_k)
    calls = []
    real = dev.ctx.groupby_sparse
    monkeypatch.setattr(dev.ctx, "groupby_sparse", lambda *a, **kw: calls.append(kw) or real(*a, **kw), raising=False)
    try:
        for q in (QUERIES[:4] + QUERIES[8:10] if ON_EMU else QUERIES):
            calls.clear()
            got = ed.execute("g", q)[0]
            assert got == er.execute("g", q)[0], q
            assert got and len(calls) == 1, q
        for q, pre in (("GroupBy(Rows(k), Rows(a), limit=20)", ("Rows(k)", "Rows(a)")), ("GroupBy(Rows(k), filter=Row(c=0))", ("Rows(k)",))):
            before = dev.ctx.counters()["queries"]
            for p in pre:
                ed.execute("g", p)
            mid = dev.ctx.counters()["queries"]
            got = ed.execute("g", q)[0]
            assert got == er.execute("g", q)[0], q
            assert dev.ctx.counters()["queries"] - mid == mid - before + 1, q          # the Rows pre-passes, then one call
    finally:
        dev.ctx.close()


@gpu
def test_limits_pushed_down(monkeypatch):
    """offset + limit is the device limit without sort, having or Sum; previous= is its start"""
    monkeypatch.setattr(X.Executor, "GROUPBY_DENSE_MAX_CELLS", 64)
    dev, ed, er = _pair(62, 150 if ON_EMU else 600, 300)
    calls = []
    real = dev.ctx.groupby_sparse
    monkeypatch.setattr(dev.ctx, "groupby_sparse", lambda *a, **kw: calls.append(kw) or real(*a, **kw), raising=False)
    try:
        for q, limit in (("GroupBy(Rows(k), Rows(a), limit=15, offset=7)", 22), ("GroupBy(Rows(k), Rows(a), limit=5)", 5),
                         ('GroupBy(Rows(k), Rows(a), sort="count desc", limit=5)', None), ("GroupBy(Rows(k), Rows(a), having=Condition(count > 1), limit=5)", None),
                         ("GroupBy(Rows(k), Rows(a), aggregate=Sum(field=v), limit=5)", None), ("GroupBy(Rows(k, previous=40), Rows(a, previous=3))", None)):
            calls.clear()
            assert ed.execute("g", q)[0] == er.execute("g", q)[0], q
            assert len(calls) == 1 and calls[0]["limit"] == limit, q
        assert calls[0]["start"] > 0
    finally:
        dev.ctx.close()


@gpu
def test_falls_back_on_comm(monkeypatch):
    """FBGPU_E_COMM or NotImplementedError from the call leaves the dense path, which answers the same when the tensor fits"""
    monkeypatch.setattr(X.Executor, "GROUPBY_DENSE_MAX_CELLS", 64)
    dev, ed, er = _pair(63, 150 if ON_EMU else 600, 300)
    q = "GroupBy(Rows(k), Rows(a), filter=Row(c=0), limit=30)"
    try:
        want = er.execute("g", q)[0]
        assert ed.execute("g", q)[0] == want
        for exc in (L.FbgpuError(L.E_COMM, "local to one context"), NotImplementedError("no node form")):
            def refuse(*a, exc=exc, **kw):
                raise exc
            monkeypatch.setattr(dev.ctx, "groupby_sparse", refuse, raising=False)
            assert ed.execute("g", q)[0] == want, exc
    finally:
        dev.ctx.close()


# ------------------------------------------------------------------ CPU
def test_groupby_sparse_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_groupby_sparse.py"], timeout=3000)
