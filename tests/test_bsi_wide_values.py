"""Int-field values across the whole int64 range: fbgpu_extract, fbgpu_bsi_sum, fbgpu_bsi_minmax, fbgpu_bsi_select and the
OP_BSI_RANGE programs at the depths and values where sign-magnitude code breaks.

A field created over [MinInt64, MaxInt64] has base 0 and bit depth 64; it stores INT64_MIN as the sign row plus magnitude
2^63 in plane 63 (row 65), which fragment.value / min / max / sum read like any other plane.  Every expectation here is
plain Python integers over the values the test itself wrote (sums wrapped to int64 as the reference's arithmetic does),
never the oracle.  Entry-point tests cover depths 1, 2, 31, 32, 33, 62, 63 and 64 over array, bitmap and run planes, shards
without a fragment or without a sign row, and filters of every density; query-level tests run Sum / Min / Max / FieldValue /
Extract / Distinct / Sort / Percentile on fields over [MinInt64, MaxInt64], [MinInt64, -1] and [1, MaxInt64].  The CPU tests
run the query-level bodies on the oracle-backed context, this file's gpu tests on the interpreted kernels, and the node
call routing with a stand-in library."""
import operator
import os
import types

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from tests.golden import vectors as V
from tests.oracle_ctx import OracleCtx
from tests.test_bsi_select import FLD, IDX, SW, VIEW, bsi_bytes, check_ranks, filt, load_field, load_filters, percentile_of_list

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR"))
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
DEPTHS = [1, 2, 31, 32, 33, 62, 63, 64]
DENSE_FLD = 8                                   # a second int field (same BSI view id) whose planes are all bitmaps
UNIT = 1 << 16
CMPS = {"==": operator.eq, "!=": operator.ne, "<": operator.lt, "<=": operator.le, ">": operator.gt, ">=": operator.ge}
gpu = pytest.mark.gpu


def wrap64(x):
    return ((x + 2**63) % 2**64) - 2**63


def edge_values(d):
    """0, ±1, ±(2^(d-1) ± 1), ±2^(d-1), ±(2^d - 1): those that fit depth d and int64 (at d = 64: INT64_MIN and INT64_MAX)"""
    h, top = 1 << (d - 1), (1 << d) - 1
    c = {0, 1, -1, h - 1, h + 1, h, top, -(h - 1), -(h + 1), -h, -top}
    return sorted(v for v in c if abs(v) <= top and I64_MIN <= v <= I64_MAX)


def rand_vals(rng, d, n, odd=False, nonneg=False):
    """n random values of depth d; magnitudes below 2^min(d, 63), so a depth-64 value stays inside int64"""
    mag = rng.integers(0, 1 << min(d, 63), n, dtype=np.uint64)
    if odd:
        mag |= np.uint64(1)
    neg = np.zeros(n, dtype=bool) if nonneg else rng.random(n) < 0.5
    return [-int(m) if s else int(m) for m, s in zip(mag.tolist(), neg.tolist())]


def mixed_world(ctx, d, seed):
    """loads FLD at depth d and filter rows 1..3 of the set field; returns ({column: value}, shards, {row: set of columns}).
    shard 0: slot 0 scattered columns holding every edge value three times plus a random fill (array planes), slot 1 dense
    columns with odd random values (bitmap planes: plane 0 is an array in slot 0 and a bitmap here), slot 2 three stretches
    of one value over consecutive columns (run planes); shard 1: listed, no BSI fragment; shard 2: non-negative values only
    (a fragment without a sign row); shard 3: the edge values again over two slots."""
    rng = np.random.default_rng(seed)
    edges = edge_values(d)
    want = {}
    vals = edges * 3 + rand_vals(rng, d, 150)
    want.update(zip(rng.choice(UNIT, len(vals), replace=False).tolist(), vals))
    n = 4200 if ON_EMU else 9000
    want.update(zip((UNIT + 7 * np.arange(n)).tolist(), rand_vals(rng, d, n, odd=True)))
    stretch = 1000 if ON_EMU else 1500
    for k, v in enumerate((edges[-1], edges[0], edges[len(edges) // 2 + 1])):
        for col in range(2 * UNIT + k * stretch, 2 * UNIT + (k + 1) * stretch):
            want[col] = v
    nonneg = [v for v in edges if v >= 0] + rand_vals(rng, d, 40, nonneg=True)
    want.update(zip((2 * SW + rng.choice(3 * UNIT, len(nonneg), replace=False)).tolist(), nonneg))
    want.update(zip((3 * SW + 5 * UNIT + rng.choice(2 * UNIT, len(edges), replace=False)).tolist(), edges))
    load_field(ctx, list(want), list(want.values()), d)
    valued = np.array(sorted(want), dtype=np.int64)
    unvalued = np.concatenate([SW + rng.choice(SW, 40, replace=False), 9 * UNIT + rng.choice(UNIT, 20, replace=False)])
    edge_cols = [c for c, v in want.items() if c < UNIT and v in (edges[0], edges[-1])]
    rows = {1: np.concatenate([valued[rng.random(len(valued)) < 0.02], edge_cols, unvalued[:10]]),
            2: np.concatenate([valued[rng.random(len(valued)) < 0.9], unvalued]),
            3: unvalued}
    load_filters(ctx, rows)
    ctx.commit()
    return want, [0, 1, 2, 3], {r: set(c.tolist()) for r, c in rows.items()}


def windows(keys):
    """(offset, limit) windows that start and end in different (shard, slot) units, plus the ends"""
    n = len(keys)
    bnd = [i for i in range(1, n) if keys[i] >> 16 != keys[i - 1] >> 16]
    out = [(0, 1), (max(n - 1, 0), 10), (n + 2, 3), (3, None)]
    if bnd:
        out.append((max(bnd[0] - 2, 0), 5))
    if len(bnd) >= 2:
        out.append((bnd[0] - 1, bnd[1] - bnd[0] + 2))
        out.append((bnd[-2] + 1, n))
    return out


def check_value_entry_points(ctx, d, want, shards, rows, field=FLD):
    """rows: {filter row: its columns}; filter row 9 holds no column at all"""
    for row in [None, 9] + sorted(rows):
        fo = None if row is None else filt(row)
        keys = sorted(c for c in want if row is None or c in rows.get(row, ()))
        exp = [want[c] for c in keys]
        cols, vals, total = ctx.extract(IDX, field, VIEW, d, shards, filter_ops=fo)
        assert total == len(keys) and cols.tolist() == keys and vals.tolist() == exp, (d, row)
        for off, lim in windows(keys):
            end = None if lim is None else off + lim
            cols, vals, total = ctx.extract(IDX, field, VIEW, d, shards, filter_ops=fo, offset=off, limit=lim)
            assert total == len(keys) and cols.tolist() == keys[off:end] and vals.tolist() == exp[off:end], (d, row, off, lim)
        assert ctx.bsi_sum(IDX, field, VIEW, d, shards, filter_ops=fo) == (wrap64(sum(exp)), len(exp)), (d, row)
        for want_max in (False, True):
            got = ctx.bsi_minmax(IDX, field, VIEW, d, shards, want_max, filter_ops=fo)
            e = (max(exp) if want_max else min(exp)) if exp else 0
            assert got == ((e, exp.count(e)) if exp else (0, 0)), (d, row, want_max)
        if d <= 63 and exp and field == FLD:
            check_ranks(ctx, d, shards, exp, sorted({0, len(exp) // 2, len(exp) - 1}), filter_ops=fo)


def range_programs(d, vals, rng):
    """(cmp, lo, hi): every comparison at ±(2^d - 1), one past each end, the stored extremes ± 1, INT64_MIN / INT64_MAX, and
    between-ranges, several of them sharing their high bits"""
    top, h = (1 << d) - 1, 1 << (d - 1)
    mn, mx = min(vals), max(vals)
    preds = {0, 1, -1, top, -top, top + 1, -top - 1, h, -h, mn - 1, mn, mn + 1, mx - 1, mx, mx + 1, I64_MIN, I64_MAX}
    out = [(c, p, 0) for c in CMPS for p in sorted(preds)]
    pairs = [(mn, mx), (mn, mn + 1), (mx - 1, mx), (top - 2, top), (-top, -top + 2), (-1, 1), (0, top), (-top, 0), (h - 1, h + 1),
             (-h - 1, -h + 1), (-top - 1, 5), (I64_MIN, I64_MAX), (I64_MIN, I64_MIN + 1), (I64_MAX - 1, I64_MAX), (0xf0, 0xf1)]
    for v in rng.choice(np.array(vals, dtype=object), 4, replace=False).tolist():
        pairs += [(v, v + 1), (v - 2, v), (v & ~0xff, v | 0xff) if v >= 0 else (-(abs(v) | 0xff), -(abs(v) & ~0xff))]
    out += [("><", lo, hi) for lo, hi in pairs if lo <= hi]
    return [(c, lo, hi) for c, lo, hi in out if I64_MIN <= lo <= I64_MAX and I64_MIN <= hi <= I64_MAX]


def check_range_programs(ctx, field, d, want, shards, seed):
    """Count (eval_wordpar_kernel on bitmap-heavy planes, else eval_kernel) and Row columns (eval_kernel) of every program
    against the Python filter over the stored values"""
    keys = sorted(want)
    vals = [want[c] for c in keys]
    for c, lo, hi in range_programs(d, vals, np.random.default_rng(seed)):
        match = (lambda v: lo <= v <= hi) if c == "><" else (lambda v: CMPS[c](v, lo))
        exp = [k for k, v in zip(keys, vals) if match(v)]
        op = [L.Op(L.OP_BSI_RANGE, field, VIEW, 0, d, L.CMP[c], lo, hi)]
        assert ctx.count(IDX, op, shards) == len(exp), (d, c, lo, hi)
        assert ctx.columns(IDX, op, shards)[0].tolist() == exp, (d, c, lo, hi)


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


# ------------------------------------------------------------------ entry points
@gpu
@pytest.mark.parametrize("d", DEPTHS)
def test_value_entry_points(ctx, d):
    """extract (all columns and windows across units), sum, min / max with multiplicity and (d <= 63) select, under no
    filter, a sparse, a dense, an empty filter and one that holds only columns without a value"""
    want, shards, rows = mixed_world(ctx, d, 100 + d)
    if d == 64:
        assert I64_MIN in want.values() and I64_MAX in want.values()
    check_value_entry_points(ctx, d, want, shards, rows)


@gpu
@pytest.mark.parametrize("d", DEPTHS)
def test_range_programs(ctx, d):
    """OP_BSI_RANGE for every comparison over the mixed planes and over a field whose planes are all bitmaps"""
    want, shards, _ = mixed_world(ctx, d, 200 + d)
    check_range_programs(ctx, FLD, d, want, shards, d)
    rng = np.random.default_rng(300 + d)
    n = 4200 if ON_EMU else 9000
    vals = rand_vals(rng, d, n, odd=True)
    edges = edge_values(d)
    for k, p in enumerate(rng.choice(n, 3 * len(edges), replace=False).tolist()):
        vals[p] = edges[k % len(edges)]
    dense = dict(zip((UNIT + 7 * np.arange(n)).tolist(), vals))
    ctx.load_fragment(IDX, DENSE_FLD, VIEW, 0, bsi_bytes(list(dense), vals, d))
    ctx.commit()
    check_range_programs(ctx, DENSE_FLD, d, dense, [0, 1], d + 1)
    check_value_entry_points(ctx, d, dense, [0, 1], {}, field=DENSE_FLD)


@gpu
def test_between_common_bits_regression_depth_64(ctx):
    """fragment_internal_test.go BetweenCommonBitsRegression (depth 64, values 0xf0 / 0xf1, >< [0xf0, 0xf1]) at the C ABI"""
    (values, depth, checks), = [c for c in V.BSI_RANGE_CASES if c[1] == 64]
    load_field(ctx, list(values), list(values.values()), depth)
    ctx.commit()
    for c, (lo, hi), exp in checks:
        op = [L.Op(L.OP_BSI_RANGE, FLD, VIEW, 0, depth, L.CMP[c], lo, hi)]
        assert ctx.count(IDX, op, [0]) == len(exp)
        assert ctx.columns(IDX, op, [0])[0].tolist() == exp


@gpu
def test_depth_argument_range(ctx):
    """extract / sum / minmax take depth 0..64; select stays at 0..63 (its sort key takes depth + 1 bits)"""
    load_field(ctx, [1, 2], [I64_MIN, 3], 64)
    ctx.commit()
    calls = (lambda d: ctx.extract(IDX, FLD, VIEW, d, [0]), lambda d: ctx.bsi_sum(IDX, FLD, VIEW, d, [0]),
             lambda d: ctx.bsi_minmax(IDX, FLD, VIEW, d, [0], False))
    for call in calls:
        for d in (-1, 65):
            with pytest.raises(L.FbgpuError) as e:
                call(d)
            assert e.value.code == L.E_INVALID, d
    assert ctx.extract(IDX, FLD, VIEW, 64, [0])[1].tolist() == [I64_MIN, 3]
    with pytest.raises(L.FbgpuError) as e:
        ctx.bsi_select(IDX, FLD, VIEW, 64, [0], [0])
    assert e.value.code == L.E_INVALID


@gpu
@pytest.mark.parametrize("d, vals", [
    (63, [(1 << 62) + 1] * 5),                                        # true sum above INT64_MAX
    (63, [-((1 << 62) + 3)] * 5),                                     # true sum below INT64_MIN
    (63, [(1 << 62) + 1] * 5 + [-((1 << 62) + 3)] * 5 + [I64_MAX, -I64_MAX]),
    (64, [I64_MIN] * 3 + [I64_MAX] * 2 + [-1]),
    (64, [I64_MIN, I64_MIN, 5]),
    (64, [I64_MAX] * 7),
])
def test_sum_wraps_int64(ctx, d, vals):
    """Σ in wrapping int64 with the columns spread over two shards and several slots"""
    cols = [k * 40009 for k in range(len(vals))]
    load_field(ctx, cols, vals, d)
    ctx.commit()
    assert ctx.bsi_sum(IDX, FLD, VIEW, d, [0, 1]) == (wrap64(sum(vals)), len(vals))
    mn, mx = min(vals), max(vals)
    assert ctx.bsi_minmax(IDX, FLD, VIEW, d, [0, 1], False) == (mn, vals.count(mn))
    assert ctx.bsi_minmax(IDX, FLD, VIEW, d, [0, 1], True) == (mx, vals.count(mx))
    assert ctx.extract(IDX, FLD, VIEW, d, [0, 1])[1].tolist() == vals


@gpu
def test_depth_64_across_unit_batches(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per batch; INT64_MIN sits in a later batch than INT64_MAX and the other extremes"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    c = L.Context(0)
    try:
        rng = np.random.default_rng(11)
        want = {3: I64_MAX, UNIT + 4: -I64_MAX, 5 * UNIT: I64_MAX, 7: 0}
        want.update(zip((SW + rng.choice(SW, 60, replace=False)).tolist(), rand_vals(rng, 64, 60)))
        want.update({3 * SW + 9: I64_MIN, 3 * SW + 4 * UNIT: I64_MIN, 3 * SW + 11: -1})
        load_field(c, list(want), list(want.values()), 64)
        load_filters(c, {1: [3, UNIT + 4, 3 * SW + 9, 3 * SW + 11, 2 * SW + 1]})
        c.commit()
        shards = [0, 1, 2, 3]
        keys = sorted(want)
        exp = [want[k] for k in keys]
        cols, vals, total = c.extract(IDX, FLD, VIEW, 64, shards)
        assert total == len(keys) and cols.tolist() == keys and vals.tolist() == exp
        cols, vals, _ = c.extract(IDX, FLD, VIEW, 64, shards, offset=len(keys) - 4, limit=10)
        assert cols.tolist() == keys[-4:] and vals.tolist() == exp[-4:]
        assert c.bsi_sum(IDX, FLD, VIEW, 64, shards) == (wrap64(sum(exp)), len(exp))
        assert c.bsi_minmax(IDX, FLD, VIEW, 64, shards, False) == (I64_MIN, 2)
        assert c.bsi_minmax(IDX, FLD, VIEW, 64, shards, True) == (I64_MAX, 2)
        sub = [I64_MAX, -I64_MAX, I64_MIN, -1]
        assert c.bsi_sum(IDX, FLD, VIEW, 64, shards, filter_ops=filt(1)) == (wrap64(sum(sub)), 4)
        assert c.bsi_minmax(IDX, FLD, VIEW, 64, shards, False, filter_ops=filt(1)) == (I64_MIN, 1)
        assert c.extract(IDX, FLD, VIEW, 64, shards, filter_ops=filt(1))[1].tolist() == [I64_MAX, -I64_MAX, I64_MIN, -1]
    finally:
        c.close()


@gpu
def test_node_sum_and_minmax_at_depth_64():
    """lib.Node (one device listed twice, shards alternate between its slots): Sum and Min / Max at depth 64 equal the plain
    context's; Node.extract has no node form and raises"""
    node, ctx = L.Node([0, 0], 1), L.Context(0)
    try:
        want, shards, rows = mixed_world(ctx, 64, 400)
        mixed_world(node, 64, 400)
        for row in (None, 1, 2, 3, 9):
            fo = None if row is None else filt(row)
            exp = [v for c, v in want.items() if row is None or c in rows.get(row, ())]
            got = node.bsi_sum(IDX, FLD, VIEW, 64, shards, filter_ops=fo)
            assert got == ctx.bsi_sum(IDX, FLD, VIEW, 64, shards, filter_ops=fo) == (wrap64(sum(exp)), len(exp)), row
            for want_max in (False, True):
                got = node.bsi_minmax(IDX, FLD, VIEW, 64, shards, want_max, filter_ops=fo)
                assert got == ctx.bsi_minmax(IDX, FLD, VIEW, 64, shards, want_max, filter_ops=fo), (row, want_max)
        with pytest.raises(NotImplementedError):
            node.extract(IDX, FLD, VIEW, 64, shards)
    finally:
        node.close()
        ctx.close()


# ------------------------------------------------------------------ queries
WIDE = {                                                 # field: (PQL options, base, depth)
    "a": ({}, 0, 64),                                    # [MinInt64, MaxInt64]
    "b": ({"min": I64_MIN, "max": -1}, -1, 63),
    "c": ({"min": 1, "max": I64_MAX}, 1, 63),            # count * Base wraps in Sum
}


def _wide_world(holder, seed, n):
    rng = np.random.default_rng(seed)
    idx = holder.create_index("w")
    idx.create_field("f")
    for name, (opts, base, depth) in WIDE.items():
        f = idx.create_field(name, "int", **opts)
        assert (f.base, f.bit_depth) == (base, depth), name
    vals = {
        "a": [I64_MIN, I64_MIN, I64_MAX, -5, 7, 0, I64_MIN + 1, -I64_MAX, 1 << 62] + rand_vals(rng, 64, n),
        "b": [I64_MIN, -1, -1, I64_MIN + 1, -(1 << 62), -2] + [-1 - abs(v) for v in rand_vals(rng, 62, n)],
        "c": [1, I64_MAX, I64_MAX, I64_MAX - 1, 2, 1 << 62] + [1 + abs(v) for v in rand_vals(rng, 62, n)],
    }
    data = {}
    for name, vs in vals.items():
        cols = rng.choice(3 * SW, len(vs), replace=False).tolist()
        data[name] = dict(zip(cols, vs))
        for col, v in data[name].items():
            holder.set_value("w", name, col, v)
    in_f = set()
    for name, d in data.items():
        cols = sorted(d)
        in_f.update(cols[::3])
        in_f.add(min(d, key=lambda c: (d[c], c)))                  # the column of the field's minimum is in the filter
    for col in in_f:
        holder.set_bit("w", "f", 0, col)
    holder.sync()
    return data, in_f


def _check_wide_queries(h, n):
    data, in_f = _wide_world(h, 21, n)
    ex = X.Executor(h)
    run = lambda q: ex.execute("w", q)[0]
    for name, d in data.items():
        for flt in (None, "Row(f=0)"):
            vs = [v for c, v in d.items() if flt is None or c in in_f]
            arg = "" if flt is None else flt + ", "
            assert run(f"Sum({arg}field={name})") == (wrap64(sum(vs)), len(vs)), (name, flt)
            mn, mx = min(vs), max(vs)
            assert run(f"Min({arg}field={name})") == (mn, vs.count(mn)), (name, flt)
            assert run(f"Max({arg}field={name})") == (mx, vs.count(mx)), (name, flt)
            pf = "" if flt is None else ", filter=" + flt
            for nth in ([0, 50, 99.9] if ON_EMU else [0, 100, 99.9, 0.1, 50, 12.5, 33.3, 90]):
                got = run(f"Percentile(field={name}, nth={nth}{pf})")
                exp, _ = percentile_of_list(vs, float(nth))
                assert (got.val, got.count) == exp, (name, flt, nth)
        c_min = min(d, key=lambda c: (d[c], c))
        assert run(f"FieldValue(field={name}, column={c_min})") == (d[c_min], 1), name
        assert run(f"Distinct(field={name})").values() == sorted(set(d.values())), name
        by_val = sorted(d.items(), key=lambda kv: (kv[1], kv[0]))
        assert run(f"Sort(All(), field={name})") == by_val, name
        assert run(f"Sort(All(), field={name}, sort-desc=true)") == sorted(d.items(), key=lambda kv: (-kv[1], kv[0])), name
    got = run("Extract(All(), Rows(a), Rows(b), Rows(c))")
    assert got["fields"] == [("a", "int64"), ("b", "int64"), ("c", "int64")]
    cols = sorted(set().union(*data.values()))
    assert got["columns"] == [(c, [data[k].get(c) for k in ("a", "b", "c")]) for c in cols]


@gpu
def test_queries_on_full_range_fields():
    """Sum / Min / Max (with and without a filter), Percentile, FieldValue on the minimum's column, Distinct, Sort both ways
    and Extract over fields [MinInt64, MaxInt64] (depth 64: Percentile takes the bisection), [MinInt64, -1] and [1, MaxInt64]"""
    h = X.Holder()
    try:
        _check_wide_queries(h, 8 if ON_EMU else 40)
    finally:
        h.ctx.close()


# ------------------------------------------------------------------ CPU
def test_queries_on_full_range_fields_host_mirror():
    """the query-level body on the oracle-backed context: the executor's own calls with their unclamped depths"""
    _check_wide_queries(X.Holder(ctx=OracleCtx()), 20)


def test_node_calls_route_refuse_and_pass_through():
    """lib._NodeCalls over a stand-in library that exports every name of lib.EXPORTS: a call with a node form is routed to
    it, a call that takes no handle passes through, any other context call raises instead of reading the node handle as
    a context"""
    lib = types.SimpleNamespace(**{name: (lambda name=name: lambda *a: name)() for name in L.EXPORTS})
    nc = L._NodeCalls(lib)
    assert nc.fbgpu_count() == "fbgpu_node_count" and nc.fbgpu_bsi_sum() == "fbgpu_node_bsi_sum" and nc.fbgpu_bsi_minmax() == "fbgpu_node_bsi_minmax"
    assert nc.fbgpu_node_shutdown() == "fbgpu_node_shutdown" and nc.fbgpu_node_ctx() == "fbgpu_node_ctx"
    for name in ("fbgpu_last_error", "fbgpu_abi_version", "fbgpu_comm_unique_id"):
        assert getattr(nc, name)() == name
    for name in ("fbgpu_extract", "fbgpu_columns", "fbgpu_row_counts_per_shard", "fbgpu_pair_types", "fbgpu_rows_payload_bytes", "fbgpu_compact",
                 "fbgpu_load_rbf", "fbgpu_bsi_select"):
        with pytest.raises(NotImplementedError):
            getattr(nc, name)(None)
    with pytest.raises(AttributeError):
        nc.not_a_library_call


def test_bsi_wide_values_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_bsi_wide_values.py"], timeout=3000)
