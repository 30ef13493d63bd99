"""fbgpu_bsi_select (order statistics of an int field over a row) and the Percentile built on it.

Entry-point tests compare every answer with the values the test itself wrote, sorted with numpy.  Query-level tests compare
Percentile through the select path with the same executor forced onto the reference's query-driven bisection, and with
executePercentile restated over a plain list.  The CPU tests run this file's gpu tests on the interpreted kernels and check
the host-side bisection over order statistics against the query-driven one on the oracle-backed context."""
import os

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from featurebase_b200 import roaring_io
from tests.oracle_ctx import OracleCtx

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR"))
SW = 1 << 20
IDX, FLD, VIEW, SETF = 0, 5, 7, 6          # index, int field, its BSI view, a set field for filters (view 0)
gpu = pytest.mark.gpu


def bsi_bytes(cols, vals, depth):
    """one shard's BSI fragment: exists row 0, sign row 1, magnitude bit i in row 2 + i"""
    o = np.asarray(cols, dtype=np.uint64) % np.uint64(SW)
    v = np.asarray(vals, dtype=object)
    mag = np.array([abs(int(x)) for x in v], dtype=np.uint64)
    neg = np.array([int(x) < 0 for x in v], dtype=bool)
    parts = [o, np.uint64(SW) + o[neg]]
    for i in range(depth):
        parts.append(np.uint64((2 + i) * SW) + o[((mag >> np.uint64(i)) & np.uint64(1)) == 1])
    return roaring_io.encode(np.unique(np.concatenate(parts)))


def load_field(ctx, cols, vals, depth):
    """cols: absolute column ids; loads one BSI fragment per shard that holds a column"""
    cols, vals = np.asarray(cols, dtype=np.int64), list(vals)
    for s in sorted(set((cols // SW).tolist())):
        m = (cols // SW) == s
        ctx.load_fragment(IDX, FLD, VIEW, s, bsi_bytes(cols[m], [v for v, k in zip(vals, m) if k], depth))


def load_filters(ctx, rows):
    """rows: {row id: absolute column ids} of the set field SETF, one fragment per shard"""
    per = {}
    for row, cols in rows.items():
        cols = np.asarray(cols, dtype=np.int64)
        for s in set((cols // SW).tolist()):
            o = (cols[(cols // SW) == s] % SW).astype(np.uint64)
            per.setdefault(s, []).append(np.uint64(row * SW) + o)
    for s, parts in per.items():
        ctx.load_fragment(IDX, SETF, 0, s, roaring_io.encode(np.unique(np.concatenate(parts))))


def filt(row):
    return [L.Op(L.OP_ROW, SETF, 0, 0, row, 0, 0, 0)]


def select_all(ctx, depth, shards, T, filter_ops=None):
    """every rank 0..T-1, 8 per call -> (values, counts)"""
    vals, cnts = [], []
    for r0 in range(0, T, L.SELECT_MAX_RANKS):
        v, c, t = ctx.bsi_select(IDX, FLD, VIEW, depth, shards, list(range(r0, min(T, r0 + L.SELECT_MAX_RANKS))), filter_ops=filter_ops)
        assert t == T
        vals += v.tolist()
        cnts += c.tolist()
    return vals, cnts


def check_ranks(ctx, depth, shards, expect, ranks, filter_ops=None):
    s = np.sort(np.asarray(expect, dtype=np.int64))
    v, c, t = ctx.bsi_select(IDX, FLD, VIEW, depth, shards, ranks, filter_ops=filter_ops)
    assert t == len(s)
    assert v.tolist() == [int(s[r]) for r in ranks]
    assert c.tolist() == [int((s == s[r]).sum()) for r in ranks]


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


# ------------------------------------------------------------------ entry point
@gpu
def test_every_rank_with_duplicates_and_count(ctx):
    """a few hundred signed values with many duplicates (0 included) over two shards, plus a listed shard without a BSI
    fragment: every rank's value and multiplicity, and the total equals fbgpu_count of the same row"""
    rng = np.random.default_rng(1)
    n = 160 if ON_EMU else 400
    cols = rng.choice(2 * SW, n, replace=False)
    vals = rng.integers(-40, 41, n).tolist()
    vals[:5] = [0, 0, 0, -40, 40]
    load_field(ctx, cols, vals, 6)
    ctx.commit()
    shards = [0, 1, 5]
    got_v, got_c = select_all(ctx, 6, shards, n)
    s = np.sort(vals)
    assert got_v == s.tolist()
    assert got_c == [int((s == x).sum()) for x in s]
    assert ctx.count(IDX, [L.Op(L.OP_ROW, FLD, VIEW, 0, 0, 0, 0, 0)], shards) == n


@gpu
@pytest.mark.parametrize("kind", ["negative", "positive"])
def test_one_sign_side(ctx, kind):
    rng = np.random.default_rng(2)
    vals = rng.integers(1, 5000, 120)
    vals = (-vals if kind == "negative" else vals).tolist()
    load_field(ctx, rng.choice(SW, 120, replace=False), vals, 13)
    ctx.commit()
    check_ranks(ctx, 13, [0], vals, [0, 1, 59, 60, 118, 119, 7, 33])


@gpu
def test_offset_base_field():
    """a field whose Base is its min (1000): the call returns value - Base"""
    h = X.Holder()
    idx = h.create_index("i")
    f = idx.create_field("v", "int", min=1000, max=1400)
    assert f.base == 1000
    rng = np.random.default_rng(3)
    vals = rng.integers(1000, 1401, 90).tolist()
    for col, v in zip(rng.choice(3 * SW, 90, replace=False).tolist(), vals):
        h.set_value("i", "v", col, v)
    h.sync()
    s = np.sort(vals)
    got, cnt, t = h.ctx.bsi_select(idx.id, f.id, X.VIEW_BSI, f.bit_depth, sorted(idx.shards), [0, 45, 89])
    assert t == 90 and (got + f.base).tolist() == [s[0], s[45], s[89]]
    h.ctx.close()


@gpu
def test_depth_one_and_depth_63(ctx):
    load_field(ctx, [1, 2, 3, 4, 5], [1, 0, -1, 1, 0], 1)
    ctx.commit()
    check_ranks(ctx, 1, [0], [1, 0, -1, 1, 0], [0, 1, 2, 3, 4])
    big = [(1 << 62) + 5, -(1 << 62) - 3, (1 << 62) - 1, 7, -(1 << 62) - 3, (1 << 63) - 1, -((1 << 63) - 1)]
    ctx.load_fragment(IDX, FLD, VIEW, 0, bsi_bytes(list(range(10, 17)), big, 63))
    ctx.commit()
    check_ranks(ctx, 63, [0], big, [0, 1, 2, 3, 4, 5, 6])


@gpu
@pytest.mark.parametrize("layout", ["dense", "clustered", "sparse"])
def test_container_encodings(ctx, layout):
    """planes stored as bitmap containers (dense columns, random values), run containers (a contiguous column range with
    values in long constant stretches) and array containers (scattered columns)"""
    rng = np.random.default_rng(4)
    if layout == "dense":
        cols = np.arange(0, 50000) + SW // 2
        vals = rng.integers(-3000, 3000, len(cols))
    elif layout == "clustered":
        cols = np.arange(100, 40100)
        vals = np.repeat(rng.integers(-1 << 20, 1 << 20, 40), 1000)
    else:
        cols = rng.choice(4 * SW, 3000, replace=False)
        vals = rng.integers(-1 << 30, 1 << 30, len(cols))
    if ON_EMU:
        cols, vals = cols[: len(cols) // 4], vals[: len(vals) // 4]
    load_field(ctx, cols, vals.tolist(), 31)
    ctx.commit()
    n = len(vals)
    check_ranks(ctx, 31, [0, 1, 2, 3], vals, [0, n // 7, n // 2, n - 1, 5, n - 6])


@gpu
def test_filters_and_empty_row(ctx):
    rng = np.random.default_rng(5)
    cols = rng.choice(2 * SW, 2000, replace=False)
    vals = rng.integers(-100000, 100000, 2000)
    load_field(ctx, cols, vals.tolist(), 17)
    outside = rng.choice(np.arange(3 * SW, 4 * SW), 50, replace=False)             # a shard with no valued column
    rows = {row: np.concatenate([cols[rng.random(len(cols)) < p], outside]) for row, p in ((1, 0.01), (2, 0.2), (3, 0.9))}
    load_filters(ctx, {**rows, 4: outside})
    ctx.commit()
    shards = [0, 1, 3]
    for row in (1, 2, 3):
        f = ctx.columns(IDX, filt(row), shards)[0].astype(np.int64)
        keep = np.isin(cols, f)
        n = int(keep.sum())
        assert n > 0
        check_ranks(ctx, 17, shards, vals[keep], sorted({0, n // 3, n // 2, n - 1}), filter_ops=filt(row))
        ops = filt(row) + [L.Op(L.OP_ROW, FLD, VIEW, 0, 0, 0, 0, 0), L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)]
        assert ctx.bsi_select(IDX, FLD, VIEW, 17, shards, [], filter_ops=filt(row))[2] == ctx.count(IDX, ops, shards) == n
    v, c, t = ctx.bsi_select(IDX, FLD, VIEW, 17, shards, [], filter_ops=filt(4))
    assert t == 0 and len(v) == 0
    with pytest.raises(L.FbgpuError) as e:
        ctx.bsi_select(IDX, FLD, VIEW, 17, shards, [0], filter_ops=filt(4))
    assert e.value.code == L.E_INVALID
    assert ctx.bsi_select(IDX, FLD, VIEW, 17, [], [])[2] == 0


@gpu
def test_unsorted_and_duplicate_ranks(ctx):
    rng = np.random.default_rng(6)
    vals = rng.integers(-500, 500, 300)
    load_field(ctx, rng.choice(SW, 300, replace=False), vals.tolist(), 9)
    ctx.commit()
    check_ranks(ctx, 9, [0], vals, [299, 3, 150, 3, 0, 299, 77, 150])


@gpu
def test_steps_cross_unit_batches(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch; the select steps run over the units of every batch"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        rng = np.random.default_rng(7)
        n_sh = 3 if ON_EMU else 6
        cols = rng.choice(n_sh * SW, 600, replace=False)
        vals = rng.integers(-(1 << 20), 1 << 20, 600)
        load_field(c, cols, vals.tolist(), 21)
        load_filters(c, {1: cols[::3]})
        c.commit()
        shards = list(range(n_sh))
        check_ranks(c, 21, shards, vals, [0, 1, 299, 300, 598, 599])
        check_ranks(c, 21, shards, vals[::3], [0, 100, 199], filter_ops=filt(1))
    finally:
        c.close()


@gpu
def test_argument_errors(ctx):
    import ctypes as C
    load_field(ctx, [1, 2, 3], [5, -5, 0], 3)
    ctx.commit()
    Lb, sh, rk = ctx.L, np.zeros(1, dtype=np.uint64), np.zeros(9, dtype=np.uint64)
    vals, cnts, tot = np.zeros(9, dtype=np.int64), np.zeros(9, dtype=np.uint64), C.c_uint64(0)

    def call(ops=None, n_ops=0, depth=3, shards=sh.ctypes.data, n_shards=1, ranks=rk.ctypes.data, n_ranks=1, out_vals=vals.ctypes.data, out_total=True):
        return Lb.fbgpu_bsi_select(ctx.h, IDX, ops, n_ops, FLD, VIEW, depth, shards, n_shards, ranks, n_ranks, out_vals, cnts.ctypes.data,
                                   C.byref(tot) if out_total else None)
    assert call() == 0 and tot.value == 3 and vals[0] == -5
    assert call(out_vals=None, n_ranks=0) == 0 and tot.value == 3
    for kw in ({"depth": -1}, {"depth": 64}, {"n_ops": -1}, {"n_ops": 1}, {"shards": None}, {"n_shards": -1}, {"ranks": None},
               {"out_vals": None}, {"out_total": False}, {"n_ranks": -1}, {"n_ranks": L.SELECT_MAX_RANKS + 1}):
        assert call(**kw) == L.E_INVALID, kw
    rk[0] = 3
    assert call() == L.E_INVALID and tot.value == 3                          # rank >= total: the total is still reported
    with pytest.raises(L.FbgpuError):
        ctx.bsi_select(IDX, FLD, VIEW, 3, [0], [0, 3])


# ------------------------------------------------------------------ Percentile
def percentile_of_list(nums, nth):
    """executePercentile (executor.go:1310-1600) restated over a plain list: (ValCount as a tuple, converged)"""
    def go_div(a, b):
        q = abs(a) // abs(b)
        return q if (a >= 0) == (b > 0) else -q

    def go_mod(a, b):
        return a - b * go_div(a, b)
    if not nums:
        return None, True
    mn, mx = min(nums), max(nums)
    less, greater = int(len(nums) * nth / 100.0), int(len(nums) * (100 - nth) / 100.0)
    if greater != 0 and less == 0:
        return (mn, nums.count(mn)), True
    if greater == 0:
        return (mx, nums.count(mx)), True
    lo, hi, guess = mn, mx, mn
    while lo < hi:
        guess = go_div(lo, 2) + go_div(hi, 2) + go_div(go_mod(lo, 2) + go_mod(hi, 2), 2)
        if sum(1 for x in nums if x < guess) > less:
            hi = guess - 1
        elif sum(1 for x in nums if x > guess) > greater:
            lo = guess + 1
        else:
            return (guess, 1), True
    return (guess, 1), False


NTHS = [0, 100, 99.9, 0.1, 50, 12.5, 33.3, 66.7, 99, 1, 25, 75, 90, 10, 0.5, 99.5]


def _percentile_world(holder, datasets):
    """one index per dataset: field v (int, over the dataset's range), set field f (row 0: the filter)"""
    out = []
    for k, (vals, cols, in_filter) in enumerate(datasets):
        idx = holder.create_index(f"p{k}")
        idx.create_field("f")
        idx.create_field("v", "int", min=min(vals), max=max(vals))
        for c, v, fl in zip(cols, vals, in_filter):
            holder.set_value(idx.name, "v", c, v)
            if fl:
                holder.set_bit(idx.name, "f", 0, c)
        out.append((idx.name, vals, in_filter))
    holder.sync()
    return out


def _datasets(seed, n):
    rng = np.random.default_rng(seed)
    ds = [([0, 2, 2], [1, 2, 3], [True, True, True]),                  # the bisection runs out of range at nth=50 (returns 1)
          ([-7, -7, 3, 3, 3, 9], [5, SW + 5, 6, 7, 2 * SW, 8], [True, False, True, True, True, False])]
    for spread in (1 << 4, 1 << 31):
        vals = rng.integers(-spread, spread, n).tolist()
        cols = rng.choice(3 * SW, n, replace=False).tolist()
        ds.append((vals, cols, (rng.random(n) < 0.3).tolist()))
    vals = (rng.integers(0, 3, n) * 1000003 - 7).tolist()                # few distinct values far apart
    ds.append((vals, rng.choice(2 * SW, n, replace=False).tolist(), (rng.random(n) < 0.5).tolist()))
    return ds


def _check_percentiles(ex, world, forced=None):
    """select path == plain-list restatement (== the forced bisection when given); returns how many cases did not converge"""
    not_conv = 0
    for name, vals, in_filter in world:
        for q_filter in (False, True):
            nums = [v for v, fl in zip(vals, in_filter) if fl or not q_filter]
            for nth in NTHS:
                q = f"Percentile(field=v, nth={nth}" + (", filter=Row(f=0))" if q_filter else ")")
                got = ex.execute(name, q)[0]
                exp, conv = percentile_of_list(nums, float(nth))
                not_conv += not conv
                assert (got if got is None else (got.val, got.count)) == exp, (name, q, got, exp)
                if forced is not None:
                    assert forced.execute(name, q)[0] == got, (name, q)
    return not_conv


@gpu
def test_percentile_select_vs_bisection_and_plain_list():
    h = X.Holder()
    world = _percentile_world(h, _datasets(8, 60 if ON_EMU else 300))
    ex, forced = X.Executor(h), X.Executor(h)
    forced.percentile_select = False
    assert _check_percentiles(ex, world, forced) > 0                     # the non-converging corner is covered
    # a bounded number of library queries per Percentile (one Count, one select), whatever the value range
    for name, vals, _ in world:
        before = h.ctx.counters()["queries"]
        ex.execute(name, "Percentile(field=v, nth=37)")
        assert h.ctx.counters()["queries"] - before == 2, name
    name = world[3][0]                                                   # 2^31 spread: the bisection asks dozens of Counts
    before = h.ctx.counters()["queries"]
    forced.execute(name, "Percentile(field=v, nth=37)")
    assert h.ctx.counters()["queries"] - before > 10
    h.ctx.close()


@gpu
def test_percentile_through_node_takes_the_bisection():
    """a node handle has no select: Percentile through lib.Node (one device listed twice) falls back to the bisection and
    answers what the select path answers on a plain context"""
    node, ctx = L.Node([0, 0], 1), L.Context(0)
    try:
        ds = _datasets(9, 40 if ON_EMU else 150)
        hn, hc = X.Holder(ctx=node), X.Holder(ctx=ctx)
        world = _percentile_world(hn, ds)
        _percentile_world(hc, ds)
        en, ec = X.Executor(hn), X.Executor(hc)
        for k, nth in enumerate(NTHS):
            name = world[k % len(world)][0]
            q = f"Percentile(field=v, nth={nth}, filter=Row(f=0))"
            assert en.execute(name, q)[0] == ec.execute(name, q)[0], (name, nth)
        with pytest.raises(NotImplementedError):
            node.bsi_select(0, 1, X.VIEW_BSI, 4, [0], [0])
    finally:
        node.close()
        ctx.close()


# ------------------------------------------------------------------ CPU
class SelectOracleCtx(OracleCtx):
    """OracleCtx with a bsi_select built from the oracle's values (sorted with numpy)"""

    def bsi_select(self, index, field, view, bit_depth, shards, ranks, filter_ops=None):
        _, vals, total = self.extract(index, field, view, bit_depth, shards, filter_ops=filter_ops)
        s = np.sort(vals)
        if any(int(r) >= total for r in ranks):
            raise L.FbgpuError(L.E_INVALID, "rank outside the sorted values")
        return (np.array([s[int(r)] for r in ranks], dtype=np.int64), np.array([int((s == s[int(r)]).sum()) for r in ranks], dtype=np.uint64), total)


def test_host_bisection_over_order_statistics_matches_query_driven():
    h = X.Holder(ctx=SelectOracleCtx())
    world = _percentile_world(h, _datasets(10, 40))
    ex, forced = X.Executor(h), X.Executor(h)
    forced.percentile_select = False
    assert _check_percentiles(ex, world, forced) > 0


def test_bsi_select_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_bsi_select.py"], timeout=3000)
