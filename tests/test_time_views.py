"""fbgpu_row_counts_views / fbgpu_groupby_views (a row taken as its union over several views) and the TopK, Rows and GroupBy
paths with from= / to= built on them.

Entry-point tests load each view's fragments themselves, with every container in an encoding chosen per container (array,
bitmap, run; arrays of 64 elements or more in array-only fragments are stored bank-striped), and compare every result with
one computed from the columns they wrote.  Query-level tests compare the executor with an oracle-backed holder, which has
neither call and so runs the composition (one operand row per row id, stored in the scratch field).  The CPU tests check
the argument errors and the refusal on a context without a device, and run this file's gpu tests on the interpreted kernels."""
import ctypes as C
import itertools
import os

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from featurebase_b200 import roaring_io
from oracle import oracle as O
from tests import archetypes as A
from tests.oracle_ctx import OracleCtx

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR"))
SW, W = 1 << 20, 1 << 16
IDX = 0
FT, FG = 1, 2                          # fields whose views 2.. are loaded one by one (time views)
SA, SB = 3, 4                          # set fields (view 0)
FILT = 5                               # set field of the filters (view 0)
NEVER = 60000                          # a view id that is never loaded
SLOTS = (0, 3, 15)                     # the slots the test data occupies
N_SHARDS = 4
ENCS = (O.ARRAY, O.BITMAP, O.RUN)
gpu = pytest.mark.gpu


# ------------------------------------------------------------------ data
def _pools(seed):
    """per (shard, slot): 4000 in-slot values the random containers draw from, so that views overlap"""
    rng = np.random.default_rng(seed)
    return {(s, k): np.sort(rng.choice(W, 4000, replace=False)) for s in range(N_SHARDS) for k in SLOTS}


def _values(rng, pool, small):
    if rng.random() < 0.25:                                   # a contiguous block: long runs
        n = int(rng.integers(1, 300 if small else 6000))
        s = int(rng.integers(0, W - n))
        return np.arange(s, s + n)
    k = int(rng.choice([1, 20, 70, 300] if small else [1, 20, 70, 300, 1500, 3800]))
    return np.sort(rng.choice(pool, k, replace=False))


def load_views(ctx, rng, field, views, rows, shards_of=None, small=False, pools=None):
    """one fragment per (view, shard) — a view skips some shards — each (row, slot) container in a random encoding; every
    third view is array-only (its arrays of 64 elements or more are stored bank-striped).  Returns {view: {row: abs columns}}."""
    pools = pools or _pools(7)
    model = {}
    for k, v in enumerate(views):
        array_only = k % 3 == 2
        m = model.setdefault(v, {})
        for s in (shards_of(v) if shards_of else range(N_SHARDS)):
            if rng.random() < 0.2:
                continue
            b, any_c = O.Bitmap(), False
            for r in rows:
                if rng.random() < 0.4:
                    continue
                for slot in SLOTS:
                    if rng.random() < 0.5:
                        continue
                    vals = _values(rng, pools[(s, slot)], small)
                    if array_only and len(vals) < 64:
                        vals = np.sort(rng.choice(pools[(s, slot)], 64, replace=False))
                    enc = O.ARRAY if array_only else ENCS[int(rng.integers(3))]
                    b.put(r * 16 + slot, A.container_of(vals, enc))
                    m.setdefault(r, []).append(s * SW + slot * W + vals)
                    any_c = True
            if any_c:
                ctx.load_fragment(IDX, field, v, s, b.to_bytes(optimize=False))
    return {v: {r: np.unique(np.concatenate(c)) for r, c in m.items()} for v, m in model.items()}


def load_set(ctx, field, rows):
    """rows: {row id: absolute columns}; one canonical fragment per shard (view 0)"""
    per = {}
    for row, cols in rows.items():
        for c in np.asarray(cols, dtype=np.int64):
            per.setdefault(int(c) // SW, []).append(row * SW + int(c) % SW)
    for s, bits in per.items():
        ctx.load_fragment(IDX, field, 0, s, roaring_io.encode(np.unique(np.asarray(bits, dtype=np.uint64))))


def union_cols(model, views, row, shards, keep=None):
    parts = [model[v][row] for v in set(views) if v in model and row in model[v]]
    cols = np.unique(np.concatenate(parts)) if parts else np.zeros(0, dtype=np.int64)
    cols = cols[np.isin(cols // SW, shards)]
    return cols if keep is None else cols[keep[cols]]


def filters(rng, pools):
    """{filter row: keep mask over the columns of N_SHARDS + 4 shards}: 1 sparse, 2 dense, 3 only in an unlisted shard"""
    rows = {1: [], 2: [], 3: (7 * SW + np.arange(0, 5000, 3)).tolist()}
    for (s, slot), pool in pools.items():
        base = s * SW + slot * W
        rows[1] += (base + rng.choice(pool, 40, replace=False)).tolist()
        rows[2] += (base + np.flatnonzero(rng.random(W) < 0.9)).tolist()
    keep = {}
    for r, cols in rows.items():
        m = np.zeros((N_SHARDS + 4) * SW, dtype=bool)
        m[np.asarray(cols, dtype=np.int64)] = True
        keep[r] = m
    return rows, keep


def filt(row):
    return [L.Op(L.OP_ROW, FILT, 0, 0, row, 0, 0, 0)]


def expect_all(model, views, shards, keep, rows):
    pairs = [(r, len(union_cols(model, views, r, shards, keep))) for r in rows]
    return sorted([p for p in pairs if p[1]], key=lambda p: (-p[1], p[0]))


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


# ------------------------------------------------------------------ fbgpu_row_counts_views
ROWS = [0, 1, 2, 5, 9, 1 << 33]
VIEW_COUNTS = [1, 2, 7, 40, 100] if ON_EMU else [1, 2, 7, 40, 400]


@gpu
@pytest.mark.parametrize("n_views", VIEW_COUNTS)
def test_row_counts_views_against_sets(ctx, n_views):
    """both forms over n_views views of mixed encodings, one of them never loaded and one listed twice, views missing in some
    shards, with no filter and with sparse, dense and empty filters; n_views == 1 against fbgpu_row_counts"""
    rng = np.random.default_rng(100 + n_views)
    pools = _pools(n_views)
    views = list(range(2, 2 + n_views))
    rows = ROWS[:4] if ON_EMU and n_views > 40 else ROWS
    model = load_views(ctx, rng, FT, views, rows, shards_of=lambda v: [s for s in range(N_SHARDS) if (v + s) % 5], small=n_views > 40, pools=pools)
    frows, keep = filters(rng, pools)
    load_set(ctx, FILT, frows)
    ctx.commit()
    listed = views + ([NEVER, views[0]] if n_views > 1 else [])
    shards = [0, 1, 3]
    ids = rows + [77, 1 << 40]                                   # absent rows
    for fr in (None, 1, 2, 3):
        fo, km = (None, None) if fr is None else (filt(fr), keep[fr])
        got = ctx.row_counts_views(IDX, FT, listed, shards, row_ids=ids, filter_ops=fo)
        assert [int(x) for x in got] == [len(union_cols(model, views, r, shards, km)) for r in ids], fr
        rid, cnt = ctx.row_counts_views(IDX, FT, listed, shards, filter_ops=fo)
        assert list(zip(rid.tolist(), cnt.tolist())) == expect_all(model, views, shards, km, rows), fr
        if fr == 3:
            assert len(rid) == 0 and not got.any()
        if n_views == 1:
            assert np.array_equal(got, ctx.row_counts(IDX, FT, views[0], shards, row_ids=ids, filter_ops=fo))
            rid1, cnt1 = ctx.row_counts(IDX, FT, views[0], shards, filter_ops=fo)
            assert np.array_equal(rid, rid1) and np.array_equal(cnt, cnt1)
    if n_views == 1:                                             # the same view twice is the same view
        assert np.array_equal(ctx.row_counts_views(IDX, FT, views * 2, shards, row_ids=ids), ctx.row_counts(IDX, FT, views[0], shards, row_ids=ids))
    assert not ctx.row_counts_views(IDX, FT, [NEVER, NEVER + 1], shards, row_ids=ids).any()
    assert len(ctx.row_counts_views(IDX, FT, [NEVER, NEVER + 1], shards)[0]) == 0


@gpu
def test_one_slot_in_every_encoding(ctx):
    """one (shard, slot) holding the same row in three views: every pair and triple of array / bank-striped array / bitmap / run,
    overlapping, each counted once per column, with and without a filter"""
    rng = np.random.default_rng(5)
    sets = [np.sort(rng.choice(W, 3000, replace=False)), np.arange(1000, 9000), np.sort(rng.choice(W, 90, replace=False)),
            np.concatenate([np.arange(0, 100), np.arange(60000, W)])]
    encs = [O.ARRAY, O.BITMAP, O.RUN]
    combos = list(itertools.product(range(len(sets)), encs))
    fcols = np.flatnonzero(rng.random(W) < 0.3)
    load_set(ctx, FILT, {1: 2 * SW + 4 * W + fcols})
    for k, (si, enc) in enumerate(combos):                      # view 2 + k holds set si in encoding enc, row 0, shard 2 slot 4
        b = O.Bitmap()
        b.put(4, A.container_of(sets[si], enc))
        ctx.load_fragment(IDX, FT, 2 + k, 2, b.to_bytes(optimize=False))
    ctx.commit()
    picks = list(itertools.combinations(range(len(combos)), 2)) + list(itertools.combinations(range(len(combos)), 3))[:: 1 if not ON_EMU else 7]
    for p in picks:
        u = np.unique(np.concatenate([sets[combos[k][0]] for k in p]))
        views = [2 + k for k in p]
        assert int(ctx.row_counts_views(IDX, FT, views, [2], row_ids=[0])[0]) == len(u), p
        assert int(ctx.row_counts_views(IDX, FT, views, [2], row_ids=[0], filter_ops=filt(1))[0]) == len(np.intersect1d(u, fcols)), p


def _raw_rcv(lib, h, views=True, n_views=2, rows=True, n_rows=1, out=True, shards=True, n_shards=1, ops=None, n_ops=0, cap=4):
    keep = [np.array([2, 3], dtype=np.uint32), np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64), np.zeros(1, dtype=np.uint64)]
    vw, ids, o, sh = keep
    n = C.c_int32(-1)
    rc = lib.fbgpu_row_counts_views(h, IDX, FT, vw.ctypes.data if views else None, n_views, ids.ctypes.data if rows else None, n_rows, ops, n_ops,
                                    sh.ctypes.data if shards else None, n_shards, None, o.ctypes.data if out else None, cap, C.byref(n))
    return rc, o, n.value


def _raw_node_rcv(lib, h, views=True, n_views=2, rows=True, n_rows=1, out=True, shards=True, n_shards=1, ops=None, n_ops=0):
    vw, ids, o, sh = np.array([2, 3], dtype=np.uint32), np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64), np.zeros(1, dtype=np.uint64)
    return lib.fbgpu_node_row_counts_views(h, IDX, FT, vw.ctypes.data if views else None, n_views, ids.ctypes.data if rows else None, n_rows, ops, n_ops,
                                           sh.ctypes.data if shards else None, n_shards, o.ctypes.data if out else None)


RCV_ERRORS = [
    ({"views": False}, "bad argument"),
    ({"n_views": 0}, "n_views=0 < 1"),
    ({"n_views": -3}, "n_views=-3 < 1"),
    ({"out": False}, "bad argument"),
    ({"n_rows": -1}, "bad argument"),
    ({"shards": False}, "bad argument"),
    ({"n_shards": -1}, "bad argument"),
    ({"n_ops": 1}, "bad argument"),
    ({"n_ops": -1}, "bad argument"),
]


def _raw_gbv(lib, h, fields=True, views=True, n_views=(2, 1), n_fields=2, rows=True, n_rows=(1, 1), out=True, shards=True, n_shards=1, ops=None, n_ops=0):
    fl, vw = np.array([FT, SA] * 4, dtype=np.uint32), np.array([2, 3, 0] * 8, dtype=np.uint32)
    nv = np.ascontiguousarray(np.asarray(list(n_views or ()) + [1] * 8, dtype=np.int32))
    nr = np.ascontiguousarray(np.asarray(list(n_rows or ()) + [1] * 8, dtype=np.int32))
    ids, o, sh = np.zeros(1 << 16, dtype=np.uint64), np.zeros(1 << 16, dtype=np.uint64), np.zeros(1, dtype=np.uint64)
    return lib.fbgpu_groupby_views(h, IDX, fl.ctypes.data if fields else None, vw.ctypes.data if views else None, nv.ctypes.data if n_views is not None else None,
                                   n_fields, ids.ctypes.data if rows else None, nr.ctypes.data if n_rows is not None else None, ops, n_ops,
                                   sh.ctypes.data if shards else None, n_shards, o.ctypes.data if out else None), o


GBV_ERRORS = [
    ({"n_fields": 0}, "n_fields=0 outside 1..8"),
    ({"n_fields": 9}, "n_fields=9 outside 1..8"),
    ({"n_views": (2, 0)}, "n_views[1]=0 < 1"),
    ({"n_views": (-1, 1)}, "n_views[0]=-1 < 1"),
    ({"n_rows": (1, 65536)}, "n_rows[1]=65536 out of range"),
    ({"n_rows": (-1, 1)}, "n_rows[0]=-1 out of range"),
    ({"fields": False}, "bad argument"),
    ({"views": False}, "bad argument"),
    ({"n_views": None}, "bad argument"),
    ({"rows": False}, "bad argument"),
    ({"n_rows": None}, "bad argument"),
    ({"out": False}, "bad argument"),
    ({"shards": False}, "bad argument"),
    ({"n_shards": -1}, "bad argument"),
    ({"n_ops": 1}, "bad argument"),
    ({"n_ops": -1}, "bad argument"),
]


def _check_errors(lib, h, node):
    for kw, msg in RCV_ERRORS:
        rc = _raw_node_rcv(lib, h, **kw) if node else _raw_rcv(lib, h, **kw)[0]
        assert rc == L.E_INVALID and lib.fbgpu_last_error().decode() == msg, (kw, msg)
    for kw, msg in GBV_ERRORS:
        rc, _ = _raw_gbv(lib, h, **kw)
        assert rc == L.E_INVALID and lib.fbgpu_last_error().decode() == msg, (kw, msg)
    if node:                                                     # the node form takes explicit row ids only
        assert _raw_node_rcv(lib, h, rows=False) == L.E_INVALID and lib.fbgpu_last_error().decode() == "bad argument"


def test_argument_errors_before_the_device_check():
    """every argument error is reported before the device check, on a context and on a node without a device"""
    ctx = L.Context(L.DEVICE_NONE)
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        _check_errors(ctx.L, ctx.h, False)
        _check_errors(node.L, node.h, True)
    finally:
        node.close()
        ctx.close()


def test_refused_on_an_inspection_only_context():
    ctx = L.Context(L.DEVICE_NONE)
    try:
        for call in (lambda: ctx.row_counts_views(IDX, FT, [2, 3], [0], row_ids=[1]), lambda: ctx.row_counts_views(IDX, FT, [2, 3], [0]),
                     lambda: ctx.row_counts_views(IDX, FT, [2], [0]), lambda: ctx.groupby_views(IDX, [FT, SA], [[2, 3], [0]], [[1], [1]], [0])):
            with pytest.raises(L.FbgpuError) as e:
                call()
            assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()


@gpu
def test_argument_errors_on_a_device(ctx):
    load_views(ctx, np.random.default_rng(1), FT, [2, 3], [0], small=True)
    ctx.commit()
    _check_errors(ctx.L, ctx.h, False)
    rc, _, _ = _raw_rcv(ctx.L, ctx.h, n_rows=0)                  # no rows: nothing to count, no error
    assert rc == 0


@gpu
def test_all_rows_nospace_and_retry(ctx):
    """the all-rows form writes nothing past cap: FBGPU_E_NOSPACE with *out_n = the number of rows, and row_counts_views grows its
    buffers and calls again"""
    rng = np.random.default_rng(3)
    rows = list(range(12))
    model = load_views(ctx, rng, FT, [2, 3, 4], rows, small=True)
    ctx.commit()
    exp = expect_all(model, [2, 3, 4], [0, 1, 2, 3], None, rows)
    assert len(exp) > 4
    vw, sh = np.array([2, 3, 4], dtype=np.uint32), np.arange(4, dtype=np.uint64)
    rid, cnt, n = np.zeros(4, dtype=np.uint64), np.zeros(4, dtype=np.uint64), C.c_int32(0)
    rc = ctx.L.fbgpu_row_counts_views(ctx.h, IDX, FT, vw.ctypes.data, 3, None, 0, None, 0, sh.ctypes.data, 4, rid.ctypes.data, cnt.ctypes.data, 4, C.byref(n))
    assert rc == L.E_NOSPACE and n.value == len(exp) and not rid.any() and not cnt.any()
    r2, c2 = ctx.row_counts_views(IDX, FT, [2, 3, 4], [0, 1, 2, 3], cap=1)
    assert list(zip(r2.tolist(), c2.tolist())) == exp


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: the filter is evaluated one shard per batch, and the counts still add up"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        rng = np.random.default_rng(4)
        pools = _pools(4)
        model = load_views(c, rng, FT, list(range(2, 9)), ROWS, small=True, pools=pools)
        frows, keep = filters(rng, pools)
        load_set(c, FILT, frows)
        c.commit()
        views, shards = list(range(2, 9)), [0, 1, 2, 3]
        for fr in (1, 2):
            got = c.row_counts_views(IDX, FT, views, shards, row_ids=ROWS, filter_ops=filt(fr))
            assert [int(x) for x in got] == [len(union_cols(model, views, r, shards, keep[fr])) for r in ROWS]
            rid, cnt = c.row_counts_views(IDX, FT, views, shards, filter_ops=filt(fr))
            assert list(zip(rid.tolist(), cnt.tolist())) == expect_all(model, views, shards, keep[fr], ROWS)
    finally:
        c.close()


# ------------------------------------------------------------------ fbgpu_groupby_views
def _gb_world(c, seed):
    """FT over views 2..(2+nt), FG over views 2..6, SA / SB with rows 0..2: shard 2 holds SA / SB columns but no time-view
    fragment at all"""
    rng = np.random.default_rng(seed)
    pools = _pools(seed)
    nt = 6 if ON_EMU else 30
    rows = [0, 1, 4]
    mt = load_views(c, rng, FT, list(range(2, 2 + nt)), rows, shards_of=lambda v: [0, 1, 3], small=True, pools=pools)
    mg = load_views(c, rng, FG, list(range(2, 7)), rows, shards_of=lambda v: [0, 1, 3], small=True, pools=pools)
    sets = []
    for f in (SA, SB):
        m = {}
        for r in range(3):
            cols = [s * SW + k * W + rng.choice(pools[(s, k)], 2500, replace=False) for s in range(N_SHARDS) for k in SLOTS]
            m[r] = np.unique(np.concatenate(cols))
        load_set(c, f, m)
        sets.append(m)
    frows, keep = filters(rng, pools)
    load_set(c, FILT, frows)
    c.commit()
    return {FT: (mt, list(range(2, 2 + nt)), rows), FG: (mg, list(range(2, 7)), rows), SA: ({0: sets[0]}, [0], [0, 1, 2]), SB: ({0: sets[1]}, [0], [2, 0])}, keep


def _expect_gb(world, fields, shards, keep):
    per = []
    for f in fields:
        model, views, rows = world[f]
        per.append([union_cols(model, views, r, shards, keep) for r in rows])
    out = np.zeros([len(p) for p in per], dtype=np.uint64)
    for ix in itertools.product(*[range(len(p)) for p in per]):
        cols = per[0][ix[0]]
        for d in range(1, len(per)):
            cols = np.intersect1d(cols, per[d][ix[d]], assume_unique=True)
        out[ix] = len(cols)
    return out


def _gbv(c, world, fields, shards, fo=None):
    return c.groupby_views(IDX, fields, [world[f][1] for f in fields], [world[f][2] for f in fields], shards, filter_ops=fo)


GB_SHAPES = [(FT,), (FT, SA), (SA, FT), (SA, FT, SB), (FT, SA, SB), (SA, SB, FT), (FT, FG), (SA, FT, FG), (FG, SA, SB, FT)]


@gpu
def test_groupby_views_against_sets(ctx):
    """1-4 dimensions with the multi-view one first, in the middle and last, and two multi-view dimensions, with and without a
    filter; shard 2 holds set-field columns but no fragment of any listed view of FT / FG, so it adds nothing where those group"""
    world, keep = _gb_world(ctx, 21)
    shards = [0, 1, 2, 3]
    assert _gbv(ctx, world, [SA], [2]).sum() > 0
    for fields in (GB_SHAPES[:6] if ON_EMU else GB_SHAPES):
        for fr in (None, 2):
            fo, km = (None, None) if fr is None else (filt(fr), keep[fr])
            got = _gbv(ctx, world, list(fields), shards, fo)
            assert got.shape == tuple(len(world[f][2]) for f in fields)
            assert np.array_equal(got, _expect_gb(world, fields, shards, km)), (fields, fr)
            assert got.any() or fr is not None, fields


@gpu
def test_single_view_groupby_views_is_groupby(ctx):
    """every n_views == 1: bit-identical to fbgpu_groupby, dimension counts 1-3, with and without a filter"""
    world, _ = _gb_world(ctx, 22)
    rows = {FT: [0, 1, 4], SA: [0, 1, 2], SB: [2, 0]}
    for fields in ([SA], [FT], [SA, SB], [FT, SA], [SA, SB, FT], [FT, SB, SA]):
        views = [5 if f == FT else 0 for f in fields]
        for fo in (None, filt(1), filt(2)):
            a = ctx.groupby_views(IDX, fields, [[v] for v in views], [rows[f] for f in fields], [0, 1, 2, 3], filter_ops=fo)
            b = ctx.groupby(IDX, fields, views, [rows[f] for f in fields], [0, 1, 2, 3], filter_ops=fo)
            assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), fields
            assert a.any() or fo is not None or len(fields) == 3, fields


@gpu
def test_node_answers_what_the_context_answers():
    """lib.Node with one device listed twice (shards alternate between its two contexts): explicit-ids row counts and GroupBy
    summed over the devices; the all-rows form has no node form"""
    node, ctx = L.Node([0, 0], 1), L.Context(0)
    try:
        worlds = [_gb_world(c, 23) for c in (node, ctx)]
        world, keep = worlds[1]
        assert {node.owner(s) for s in range(4)} == {0, 1}
        shards = [0, 1, 2, 3]
        model, views, rows = world[FT]
        for fo, km in ((None, None), (filt(2), keep[2])):
            got = node.row_counts_views(IDX, FT, views + [NEVER], shards, row_ids=rows + [99], filter_ops=fo)
            assert np.array_equal(got, ctx.row_counts_views(IDX, FT, views + [NEVER], shards, row_ids=rows + [99], filter_ops=fo))
            assert [int(x) for x in got] == [len(union_cols(model, views, r, shards, km)) for r in rows + [99]]
            for fields in ([FT], [SA, FT], [FT, FG]):
                g = _gbv(node, world, fields, shards, fo)
                assert np.array_equal(g, _gbv(ctx, world, fields, shards, fo)) and np.array_equal(g, _expect_gb(world, fields, shards, km)), fields
        with pytest.raises(NotImplementedError):
            node.row_counts_views(IDX, FT, views, shards)
    finally:
        node.close()
        ctx.close()


# ------------------------------------------------------------------ query level
SPANS = {"YMDH": (20, 24), "YMD": (120, 1), "YM": (400, 1), "D": (90, 1), "H": (6, 24)}       # days spread, timestamps per day granularity


def _ts(day, hour):
    import datetime
    t = datetime.datetime(2019, 1, 1) + datetime.timedelta(days=day, hours=hour)
    return t.strftime("%Y-%m-%dT%H:%M")


def _time_world(holder, quantum, seed, n):
    """index "t": time field f (rows 0..7), set field a (rows 0..4), filter field c, over three shards"""
    rng = np.random.default_rng(seed)
    idx = holder.create_index("t")
    idx.create_field("f", "time", quantum=quantum)
    idx.create_field("a")
    idx.create_field("c")
    days, per = SPANS[quantum]
    cols = rng.choice(3 * SW, n, replace=False).tolist()
    for col in cols:
        for r in range(8):
            if rng.random() < 0.35:
                for _ in range(int(rng.integers(1, 3))):
                    holder.set_bit("t", "f", r, col, timestamp=_ts(int(rng.integers(days)), int(rng.integers(24)) if per > 1 else 0))
        for r in range(5):
            if rng.random() < 0.3:
                holder.set_bit("t", "a", r, col)
        if rng.random() < 0.3:
            holder.set_bit("t", "c", 0, col)
    holder.sync()


def _ranges(quantum):
    days = SPANS[quantum][0]
    lo, hi = _ts(days // 5, 3), _ts(days * 3 // 5, 17)
    return [f"from={lo}, to={hi}", f"from={_ts(days // 2, 5)}", f"to={_ts(days // 3, 0)}"]


QUERIES = [
    "TopK(f, {R})",
    "TopK(f, k=3, {R})",
    "TopK(f, k=2, {R}, filter=Row(c=0))",
    "Rows(f, {R})",
    "Rows(f, {R}, previous=2)",
    "Rows(f, {R}, limit=3)",
    "Rows(f, {R}, in=[1, 4, 6])",
    "GroupBy(Rows(a), Rows(f, {R}))",
    "GroupBy(Rows(f, {R}), Rows(a), filter=Row(c=0))",
    "GroupBy(Rows(a), Rows(f, {R}), limit=5, offset=2)",
    "GroupBy(Rows(a, previous=1), Rows(f, {R}, previous=2), limit=6)",
    "GroupBy(Rows(f, {R}), having=Condition(count > 3))",
    'GroupBy(Rows(a), Rows(f, {R}), sort="count desc", limit=4)',
    "GroupBy(Rows(f, {R}), Rows(f, {R2}), Rows(a))",
]


@gpu
@pytest.mark.parametrize("quantum", ["YMDH", "YMD", "YM", "D", "H"])
def test_queries_match_the_composition(quantum):
    """TopK, Rows and GroupBy with from= / to= against an oracle-backed holder, which runs the composition"""
    n = 120 if ON_EMU else 1200
    dev, ref = X.Holder(), X.Holder(ctx=OracleCtx())
    _time_world(dev, quantum, 31, n)
    _time_world(ref, quantum, 31, n)
    ed, er = X.Executor(dev), X.Executor(ref)
    assert not hasattr(ref.ctx, "row_counts_views") and not hasattr(ref.ctx, "groupby_views")
    rs = _ranges(quantum)
    n_run, n_empty = 0, 0
    try:
        for q in (QUERIES[::3] if ON_EMU else QUERIES):
            for k, r in enumerate(rs[:1] if ON_EMU else rs):
                qq = q.format(R=r, R2=rs[(k + 1) % len(rs)])
                got = ed.execute("t", qq)[0]
                assert got == er.execute("t", qq)[0], qq
                n_run, n_empty = n_run + 1, n_empty + (not got)
        assert n_empty * 4 < n_run, (n_empty, n_run)
    finally:
        dev.ctx.close()


class _Counting:
    """the executor's context, counting the method calls made on it"""

    def __init__(self, ctx):
        self._ctx, self.calls = ctx, []

    def __getattr__(self, name):
        a = getattr(self._ctx, name)
        if not callable(a):
            return a

        def call(*args, **kw):
            self.calls.append(name)
            return a(*args, **kw)
        return call


@gpu
def test_one_library_call_and_no_scratch_rows():
    """TopK(f, from=, to=) and Rows(f, from=, to=) make one library call each, GroupBy(Rows(a), Rows(f, from=, to=)) three (a's row
    list, f's row list, the counts); none of them loads or embeds anything"""
    h = X.Holder()
    try:
        _time_world(h, "YMD", 32, 100 if ON_EMU else 800)
        ex = X.Executor(h)
        ex.ctx = proxy = _Counting(h.ctx)
        r = _ranges("YMD")[0]
        before = h.ctx.stats()
        for q, n_calls in ((f"TopK(f, {r})", 1), (f"TopK(f, k=2, {r}, filter=Row(c=0))", 1), (f"Rows(f, {r})", 1), (f"GroupBy(Rows(a), Rows(f, {r}))", 3)):
            proxy.calls.clear()
            assert ex.execute("t", q)[0], q
            assert len(proxy.calls) == n_calls, (q, proxy.calls)
        after = h.ctx.stats()
        assert (after["fragments"], after["payload_bytes"]) == (before["fragments"], before["payload_bytes"])
        assert X.SCRATCH_FIELD not in h.indexes["t"].fields
    finally:
        h.ctx.close()


# ------------------------------------------------------------------ CPU
def test_time_views_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_time_views.py"], timeout=3000)
