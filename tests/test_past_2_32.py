"""Every counting entry point on a world of 2^32 + 2^20 columns: counts, ranks, offsets and sums past 2^32, over more shards
than one evaluation batch holds.

The world has S shards (0 .. S-1, 2^20 columns each): N = S * 2^20 columns, B = (S-1) * 2^20 of them outside shard 0.  On the
device S = 4097, so N = 2^32 + 2^20, B = 2^32, and the 65,552 (shard, slot) units are four full batches of the default
16,384 units plus a batch of one shard.  Full rows are one run container per (shard, slot), so the world is cheap, and every
expectation is a closed form in S checked with plain Python integers: N mod 2^32 is 2^20 (the count of row 3), B mod 2^32 is
0, so an accumulator, rank or offset narrowed to 32 bits answers visibly wrong.  (That holds for what sums across units: the
query totals the kernels add into, the host's merges, ranks and offsets.  One block's share of a count launch, at most a few
hundred units, and one (shard, row) count, at most 2^20, stay below 2^32 at any shard count a test can load.)

    field  id  content
    EX      0  row 0 full in every shard (the filter, and the executor's existence row)
    F       1  row 5 full everywhere; row 3 full in shard 0 only; rows 9 / 10 the odd / even columns everywhere (bitmaps)
    G       2  row 0 full everywhere; row 1 full in shards 1 .. S-1 (a count of B)
    T       3  row 0 full, in view 1 on even shards and in view 2 on odd shards
    A, B  4, 5  rows 0..3: the columns with col % 256 == row (array containers of 256)
    V       6  int, depth 63: every column holds 2^62 + 1 (Sum wraps)
    U       7  int, depth 3: -5 in shards 0 .. S-2, 7 in shard S-1 (the -5 / 7 boundary sits at rank B)

The field ids are those an executor Holder gives index 0 with existence tracking, so the executor runs on the same store.
Each distinct fragment is built once and loaded for every shard that holds it.  The CPU tests check the closed forms at
S = 3 with the oracle-backed context, and run this file's gpu tests on the interpreted kernels at S = 3 with
FBGPU_UNIT_BATCH=16 (several full batches, then one more); the full-size world runs on the device only."""
import os
import threading

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from featurebase_b200 import roaring_io
from oracle import oracle as O
from tests.oracle_ctx import OracleCtx
from tests.test_bsi_select import percentile_of_list

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR"))
SW = 1 << 20
SLOTS = SW >> 16
IDX = 0
EX, F, G, T, A, B, V, U = range(8)
BSI = X.VIEW_BSI
V_DEPTH, U_DEPTH = 63, 3
VAL = (1 << 62) + 1
S_DEVICE = 3 if ON_EMU else 4097
gpu = pytest.mark.gpu


def _i64(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


class Sizes:
    def __init__(self, S):
        self.S, self.N, self.B, self.H = S, S * SW, (S - 1) * SW, S * SW // 2
        self.shards = list(range(S))


# ------------------------------------------------------------------ the world
def _full(row):
    return np.uint64(row * SW) + np.arange(SW, dtype=np.uint64)


def _bsi(value, depth):
    """one shard's fragment of an int field whose every column holds `value`: exists row 0, sign row 1, magnitude bit i in row 2 + i"""
    rows = [0] + ([1] if value < 0 else []) + [2 + i for i in range(depth) if (abs(value) >> i) & 1]
    return roaring_io.encode(np.concatenate([_full(r) for r in rows]))


def fragments(S):
    """[(field, view, fragment bytes, shards that hold it)]: every distinct fragment once"""
    enc = roaring_io.encode
    odd, even = np.arange(1, SW, 2, dtype=np.uint64), np.arange(0, SW, 2, dtype=np.uint64)
    f_all = [_full(5), np.uint64(9 * SW) + odd, np.uint64(10 * SW) + even]
    c = np.arange(SW, dtype=np.uint64)
    ab = enc(np.concatenate([np.uint64(r * SW) + c[c % np.uint64(256) == np.uint64(r)] for r in range(4)]))
    everywhere, rest = list(range(S)), list(range(1, S))
    return [
        (EX, 0, enc(_full(0)), everywhere),
        (F, 0, enc(np.concatenate(f_all + [_full(3)])), [0]),
        (F, 0, enc(np.concatenate(f_all)), rest),
        (G, 0, enc(_full(0)), [0]),
        (G, 0, enc(np.concatenate([_full(0), _full(1)])), rest),
        (T, 1, enc(_full(0)), everywhere[0::2]),
        (T, 2, enc(_full(0)), everywhere[1::2]),
        (A, 0, ab, everywhere),
        (B, 0, ab, everywhere),
        (V, BSI, _bsi(VAL, V_DEPTH), everywhere),
        (U, BSI, _bsi(-5, U_DEPTH), everywhere[:-1]),
        (U, BSI, _bsi(7, U_DEPTH), everywhere[-1:]),
    ]


def load_world(ctx, S):
    for field, view, data, shards in fragments(S):
        for s in shards:
            ctx.load_fragment(IDX, field, view, s, data)
    ctx.commit()
    return Sizes(S)


def full_row_bytes(k0, k1):
    """the canonical Pilosa-roaring bytes of the columns [k0 * 2^16, k1 * 2^16): one full run container per key (cookie,
    key / type / n-1 headers, 32-bit offsets, payloads of one run [0, 65535])"""
    n = k1 - k0
    hdr = np.zeros(n, dtype=np.dtype([("key", "<u8"), ("typ", "<u2"), ("n1", "<u2")]))
    hdr["key"], hdr["typ"], hdr["n1"] = np.arange(k0, k1, dtype=np.uint64), roaring_io.RUN, 0xFFFF
    offs = (8 + 16 * n + 6 * np.arange(n, dtype=np.uint64)).astype("<u4")
    payload = np.tile(np.array([1, 0, 0xFFFF], dtype="<u2"), n)
    return np.array([roaring_io.MAGIC, n], dtype="<u4").tobytes() + hdr.tobytes() + offs.tobytes() + payload.tobytes()


# ------------------------------------------------------------------ programs
def row(field, r, view=0):
    return L.Op(L.OP_ROW, field, view, 0, r, 0, 0, 0)


def nary(op, n):
    return L.Op(op, 0, 0, n, 0, 0, 0, 0)


def count_programs(z):
    """(name, program, expected count, expected per-shard counts).  Programs over F, G and EX alone (runs and bitmaps) take
    eval_wordpar_kernel, Count(Intersect(Row, Row)) pair_count_kernel, and programs that also read A's array containers
    eval_kernel."""
    S, every, a_row = z.S, [SW] * z.S, SW // 256
    return [
        ("Union(F=5, A=0)", [row(F, 5), row(A, 0), nary(L.OP_UNION, 2)], z.N, every),
        ("Xor(G=1, A=0)", [row(G, 1), row(A, 0), nary(L.OP_XOR, 2)], a_row + (S - 1) * (SW - a_row), [a_row] + [SW - a_row] * (S - 1)),
        ("Row(F=5)", [row(F, 5)], z.N, every),
        ("Intersect(F=5, G=0)", [row(F, 5), row(G, 0), nary(L.OP_INTERSECT, 2)], z.N, every),
        ("Union(F=9, F=10)", [row(F, 9), row(F, 10), nary(L.OP_UNION, 2)], z.N, every),
        ("Row(G=1)", [row(G, 1)], z.B, [0] + [SW] * (S - 1)),
        ("Difference(F=5, F=3)", [row(F, 5), row(F, 3), nary(L.OP_DIFFERENCE, 2)], z.B, [0] + [SW] * (S - 1)),
        ("Xor(F=9, G=0)", [row(F, 9), row(G, 0), nary(L.OP_XOR, 2)], z.H, [SW // 2] * S),
    ]


# ------------------------------------------------------------------ checks (each names the context calls it makes)
def check_count(ctx, z):
    for name, prog, exp, per_exp in count_programs(z):
        assert ctx.count(IDX, prog, z.shards) == exp, name
        total, per = ctx.count(IDX, prog, z.shards, per_shard=True)
        assert total == exp and per.tolist() == per_exp, name
        assert ctx.any(IDX, prog, z.shards), name
    assert ctx.any(IDX, [row(F, 3)], z.shards[::-1])                    # row 3's only shard is the last one listed
    assert not ctx.any(IDX, [row(F, 3)], z.shards[1:])


def check_count_pairs(ctx, z):
    got = ctx.count_pairs(IDX, F, 0, [5, 5, 9], G, 0, [0, 1, 0], z.shards)
    assert got.tolist() == [z.N, z.B, z.H]


def check_row_counts(ctx, z):
    ids, exp = [3, 5, 9, 10], [SW, z.N, z.H, z.H]
    assert ctx.row_counts(IDX, F, 0, z.shards, row_ids=ids).tolist() == exp
    exp_g1 = [0, z.B, z.B // 2, z.B // 2]
    assert ctx.row_counts(IDX, F, 0, z.shards, row_ids=ids, filter_ops=[row(G, 1)]).tolist() == exp_g1
    if isinstance(ctx, L.Node):                                         # (no per-shard or all-rows node form)
        return
    m = ctx.row_counts_per_shard(IDX, F, 0, z.shards, ids)
    assert m.shape == (z.S, 4) and m.sum(axis=0, dtype=object).tolist() == exp
    assert m[0].tolist() == [SW, SW, SW // 2, SW // 2] and (m[1:] == np.array([0, SW, SW // 2, SW // 2], dtype=np.uint64)).all()
    m = ctx.row_counts_per_shard(IDX, F, 0, z.shards, ids, filter_ops=[row(G, 1)])
    assert m.sum(axis=0, dtype=object).tolist() == exp_g1 and not m[0].any()
    rid, cnt = ctx.row_counts(IDX, F, 0, z.shards)
    assert list(zip(rid.tolist(), cnt.tolist())) == [(5, z.N), (9, z.H), (10, z.H), (3, SW)]     # count desc, then row id


def check_row_counts_views(ctx, z):
    assert ctx.row_counts_views(IDX, T, [1, 2], z.shards, row_ids=[0]).tolist() == [z.N]
    assert ctx.row_counts_views(IDX, T, [1, 2], z.shards, row_ids=[0], filter_ops=[row(G, 1)]).tolist() == [z.B]
    if not isinstance(ctx, L.Node):
        rid, cnt = ctx.row_counts_views(IDX, T, [1, 2], z.shards)
        assert rid.tolist() == [0] and cnt.tolist() == [z.N]


def check_row(ctx, z):
    for prog, k0, exp in (([row(F, 5)], 0, z.N), ([row(G, 1)], SLOTS, z.B)):
        want = full_row_bytes(k0, z.N >> 16)
        data, cnt = ctx.row(IDX, prog, z.shards)
        assert cnt == exp and data == want
        if not hasattr(ctx, "row_into"):                                # (the oracle-backed context)
            continue
        need, cnt, fits = ctx.row_into(IDX, prog, z.shards, np.empty(len(want) - 1, dtype=np.uint8))
        assert (need, fits) == (len(want), False)
        buf = np.empty(len(want), dtype=np.uint8)
        need, cnt, fits = ctx.row_into(IDX, prog, z.shards, buf)
        assert (need, cnt, fits) == (len(want), exp, True) and buf.tobytes() == want


def check_columns(ctx, z):
    def window(prog, offset, limit, first):
        cols, total = ctx.columns(IDX, prog, z.shards, offset=offset, limit=limit)
        assert cols.tolist() == list(range(first, min(first + limit, z.N))), (offset, limit)
        return total
    f5 = [row(F, 5)]                                                    # contiguous shards from 0: the r-th column is r
    for off, lim in ((0, 5), (z.B - 3, 7), (z.B + SW // 2 + 7, 5), (z.H - 2, 4), (z.N - 2, 5)):
        assert window(f5, off, lim, off) == z.N
    cols, total = ctx.columns(IDX, f5, z.shards, offset=z.N, limit=3)
    assert len(cols) == 0 and total == z.N
    g1 = [row(G, 1)]                                                    # the r-th column is 2^20 + r
    for off, lim in ((0, 3), (z.B // 2 - 1, 4), (z.B - 2, 5)):
        assert window(g1, off, lim, SW + off) == z.B


def check_extract(ctx, z):
    cols, vals, total = ctx.extract(IDX, U, BSI, U_DEPTH, z.shards, offset=z.B - 3, limit=6)
    assert total == z.N and cols.tolist() == list(range(z.B - 3, z.B + 3)) and vals.tolist() == [-5] * 3 + [7] * 3
    cols, vals, total = ctx.extract(IDX, U, BSI, U_DEPTH, z.shards, filter_ops=[row(G, 1)], offset=z.B - SW - 2, limit=4)
    assert total == z.B and cols.tolist() == list(range(z.B - 2, z.B + 2)) and vals.tolist() == [-5, -5, 7, 7]
    cols, vals, total = ctx.extract(IDX, V, BSI, V_DEPTH, z.shards, offset=z.N - 1, limit=4)
    assert total == z.N and cols.tolist() == [z.N - 1] and vals.tolist() == [VAL]


def check_bsi_sum_minmax(ctx, z):
    u_sum = -5 * z.B + 7 * SW
    assert ctx.bsi_sum(IDX, V, BSI, V_DEPTH, z.shards) == (_i64(z.N * VAL), z.N)
    assert ctx.bsi_sum(IDX, U, BSI, U_DEPTH, z.shards) == (u_sum, z.N)
    g1 = [row(G, 1)]
    assert ctx.bsi_sum(IDX, V, BSI, V_DEPTH, z.shards, filter_ops=g1) == (_i64(z.B * VAL), z.B)
    assert ctx.bsi_sum(IDX, U, BSI, U_DEPTH, z.shards, filter_ops=g1) == (u_sum + 5 * SW, z.B)
    assert ctx.bsi_minmax(IDX, U, BSI, U_DEPTH, z.shards, False) == (-5, z.B)
    assert ctx.bsi_minmax(IDX, U, BSI, U_DEPTH, z.shards, True) == (7, SW)
    assert ctx.bsi_minmax(IDX, U, BSI, U_DEPTH, z.shards, False, filter_ops=g1) == (-5, z.B - SW)
    for want_max in (False, True):
        assert ctx.bsi_minmax(IDX, V, BSI, V_DEPTH, z.shards, want_max) == (VAL, z.N)
        assert ctx.bsi_minmax(IDX, V, BSI, V_DEPTH, z.shards, want_max, filter_ops=g1) == (VAL, z.B)


def check_bsi_select(ctx, z):
    vals, cnts, total = ctx.bsi_select(IDX, U, BSI, U_DEPTH, z.shards, [0, z.B - 1, z.B, z.N - 1])
    assert vals.tolist() == [-5, -5, 7, 7] and cnts.tolist() == [z.B, z.B, SW, SW] and total == z.N
    vals, cnts, total = ctx.bsi_select(IDX, U, BSI, U_DEPTH, z.shards, [z.B - SW - 1, z.B - SW], filter_ops=[row(G, 1)])
    assert vals.tolist() == [-5, 7] and cnts.tolist() == [z.B - SW, SW] and total == z.B


def check_groupby(ctx, z):
    ids = [[3, 5, 9, 10], [0, 1]]
    exp = [[SW, 0], [z.N, z.B], [z.H, z.B // 2], [z.H, z.B // 2]]
    assert ctx.groupby(IDX, [F, G], [0, 0], ids, z.shards).tolist() == exp
    assert ctx.groupby(IDX, [F, G], [0, 0], ids, z.shards, filter_ops=[row(EX, 0)]).tolist() == exp       # groupby_kernel, filter batches


def check_groupby_direct(ctx, z):
    """A x B (array containers only: groupby_direct_kernel) under the full filter row"""
    before = ctx.counters()
    got = ctx.groupby(IDX, [A, B], [0, 0], [[0, 1, 2, 3], [0, 1, 2, 3]], z.shards, filter_ops=[row(EX, 0)])
    assert got.tolist() == (np.eye(4, dtype=object) * (z.N // 256)).tolist()
    after = ctx.counters()
    if not os.environ.get("FBGPU_GROUPBY_CTA"):
        assert after["groupby_units"] - before["groupby_units"] == z.S * SLOTS
        assert after["groupby_fallback_units"] == before["groupby_fallback_units"]


def check_groupby_views(ctx, z):
    assert ctx.groupby_views(IDX, [T, G], [[1, 2], [0]], [[0], [0, 1]], z.shards).tolist() == [[z.N, z.B]]


def check_groupby_values(ctx, z):
    got = ctx.groupby_values(IDX, [G], [0], [[0, 1]], U, BSI, U_DEPTH, [-5, 7], z.shards)
    assert got.tolist() == [[z.B, SW], [z.B - SW, SW]]


def check_groupby_mixed(ctx, z):
    u, v = (U, BSI, U_DEPTH, [-5, 7]), (V, BSI, V_DEPTH, [VAL])
    assert ctx.groupby_mixed(IDX, [], [u, v], z.shards).tolist() == [[z.B], [SW]]
    got = ctx.groupby_mixed(IDX, [(F, [0], [3, 5])], [u, v], z.shards, filter_ops=[row(EX, 0)])
    assert got.tolist() == [[[SW], [0]], [[z.B], [SW]]]


def check_groupby_sum(ctx, z):
    counts, sums = ctx.groupby_sum(IDX, [(G, [0], [0, 1])], [], (V, BSI, V_DEPTH), z.shards)
    assert counts.tolist() == [z.N, z.B] and sums.tolist() == [_i64(z.N * VAL), _i64(z.B * VAL)]
    counts, sums = ctx.groupby_sum(IDX, [], [(U, BSI, U_DEPTH, [-5, 7])], (V, BSI, V_DEPTH), z.shards)
    assert counts.tolist() == [z.B, SW] and sums.tolist() == [_i64(z.B * VAL), _i64(SW * VAL)]


def check_groupby_distinct(ctx, z):
    got = ctx.groupby_distinct(IDX, [(F, [0], [3, 5, 9, 10])], [], (U, BSI, U_DEPTH, [-5, 7]), z.shards)
    assert got.tolist() == [1, 2, 2, 2]


CHECKS = [check_count, check_count_pairs, check_row_counts, check_row_counts_views, check_row, check_columns, check_extract,
          check_bsi_sum_minmax, check_bsi_select, check_groupby, check_groupby_direct, check_groupby_views, check_groupby_values,
          check_groupby_mixed, check_groupby_sum, check_groupby_distinct]
NODE_CHECKS = [check_count, check_count_pairs, check_row_counts, check_row_counts_views, check_row, check_bsi_sum_minmax, check_groupby,
               check_groupby_views, check_groupby_values, check_groupby_mixed, check_groupby_sum]
ORACLE_CHECKS = [check_count, check_count_pairs, check_row_counts, check_row, check_columns, check_extract, check_bsi_sum_minmax,
                 check_groupby]          # the calls tests/oracle_ctx.py has


# ------------------------------------------------------------------ the executor on the same store
def percentile_of_counts(mult, nth):
    """percentile_of_list (executePercentile restated) over {value: multiplicity} instead of a list"""
    def go_div(a, b):
        q = abs(a) // abs(b)
        return q if (a >= 0) == (b > 0) else -q
    total = sum(mult.values())
    mn, mx = min(mult), max(mult)
    less, greater = int(total * nth / 100.0), int(total * (100 - nth) / 100.0)
    if greater != 0 and less == 0:
        return mn, mult[mn]
    if greater == 0:
        return mx, mult[mx]
    lo, hi, guess = mn, mx, mn
    while lo < hi:
        guess = go_div(lo, 2) + go_div(hi, 2) + go_div(lo - 2 * go_div(lo, 2) + hi - 2 * go_div(hi, 2), 2)
        if sum(n for v, n in mult.items() if v < guess) > less:
            hi = guess - 1
        elif sum(n for v, n in mult.items() if v > guess) > greater:
            lo = guess + 1
        else:
            return guess, 1
    return guess, 1


def nth_at_rank(total, rank):
    """a percentile whose desiredLess (int(total * nth / 100) in float64) is exactly `rank`"""
    nth = 100.0 * rank / total
    for _ in range(64):
        got = int(total * nth / 100.0)
        if got == rank:
            return nth
        nth = np.nextafter(nth, np.inf if got < rank else -np.inf)
    raise AssertionError("no nth lands on the rank")


def executor_on(ctx, S):
    """a Holder over a context that holds the world: index 0 with existence tracking, whose field ids are the world's"""
    h = X.Holder(ctx=ctx)
    idx = h.create_index("i")
    for name in ("f", "g", "t", "a", "b"):
        idx.create_field(name)
    idx.create_field("v", "int", min=0, max=(1 << 63) - 1)
    idx.create_field("u", "int", min=-5, max=7)
    got = {n: (f.id, getattr(f, "bit_depth", None), getattr(f, "base", None)) for n, f in idx.fields.items()}
    assert got == {X.EXISTENCE_FIELD: (EX, None, None), "f": (F, None, None), "g": (G, None, None), "t": (T, None, None), "a": (A, None, None),
                   "b": (B, None, None), "v": (V, V_DEPTH, 0), "u": (U, U_DEPTH, 0)}
    idx.shards.update(range(S))
    return X.Executor(h)


def check_executor(ex, z):
    run = lambda q: ex.execute("i", q)[0]
    N, B, H = z.N, z.B, z.H
    assert run("Count(All())") == N
    assert run("Count(Not(Row(f=3)))") == B
    assert run("TopN(f, n=2)") == [(5, N), (9, H)]                     # a count of N mod 2^32 would tie row 5 with row 3
    assert run("TopN(f)") == [(5, N), (9, H), (10, H), (3, SW)]
    assert run("TopN(f, ids=[3, 5])") == [(5, N), (3, SW)]
    assert run("TopK(f, k=2)") == [(5, N), (9, H)]
    groups = [((f, g), n) for (f, g), n in {(3, 0): SW, (5, 0): N, (5, 1): B, (9, 0): H, (9, 1): B // 2, (10, 0): H, (10, 1): B // 2}.items()]
    exp = sorted(sorted(groups), key=lambda gn: -gn[1])
    got = [((grp[0][1], grp[1][1]), n) for grp, n in run('GroupBy(Rows(f), Rows(g), sort="count desc")')]
    assert got == exp
    got = run("GroupBy(Rows(g), aggregate=Sum(field=v))")
    assert got == [([("g", 0)], N, _i64(N * VAL)), ([("g", 1)], B, _i64(B * VAL))]
    assert run("Sum(field=v)") == (_i64(N * VAL), N)
    assert run("Sum(Row(g=1), field=u)") == (-5 * (B - SW) + 7 * SW, B)
    assert run("Min(field=u)") == (-5, B) and run("Max(field=u)") == (7, SW)
    assert run("Min(field=v)") == (VAL, N) and run("Max(field=v)") == (VAL, N)
    for rank in (B, B - 1):
        nth = nth_at_rank(N, rank)
        got = run(f"Percentile(field=u, nth={nth!r})")
        assert (got.val, got.count) == percentile_of_counts({-5: B, 7: SW}, nth), nth


# ------------------------------------------------------------------ device (interpreted kernels: S = 3)
@pytest.fixture(scope="module")
def world():
    ctx = L.Context(0)
    z = load_world(ctx, S_DEVICE)
    if not ON_EMU:
        assert (z.N, z.B) == ((1 << 32) + SW, 1 << 32)
    yield ctx, z
    ctx.close()


@gpu
@pytest.mark.parametrize("check", CHECKS, ids=lambda c: c.__name__[6:])
def test_entry_point(world, check):
    ctx, z = world
    check(ctx, z)


@gpu
def test_executor_queries(world):
    """Count, TopN, TopK, GroupBy (plain and with aggregate=Sum), Sum / Min / Max and a Percentile whose rank is B, through the
    executor over the same store"""
    ctx, z = world
    check_executor(executor_on(ctx, z.S), z)


@gpu
def test_node_merges_past_2_32():
    """lib.Node with one device listed twice: every device slot holds fewer than 2^32 columns of any row, so only the host merge
    of the two slots' results crosses 2^32"""
    z = Sizes(S_DEVICE)
    block = max(1, (z.S - 1) // 4)                    # S = 4097: slot 0 gets 2049 shards, slot 1 2048
    node = L.Node([0, 0], block)
    try:
        load_world(node, z.S)
        per_slot = [sum(1 for s in z.shards if node.owner(s) == k) for k in (0, 1)]
        assert sum(per_slot) == z.S and 0 < max(per_slot) * SW < 1 << 32
        for check in NODE_CHECKS:
            check(node, z)
    finally:
        node.close()


@gpu
@pytest.mark.skipif(ON_EMU, reason="the interpreted kernels run a launch to completion on the calling thread: no concurrent peer to wait for")
def test_fused_peer_count_past_2_32():
    """two contexts on device 0 with half the shards each, their Count mailboxes wired to each other: both ranks return the 64-bit
    sum of the two halves"""
    z = Sizes(S_DEVICE)
    data = {0: roaring_io.encode(np.concatenate([_full(3), _full(5)])), 1: roaring_io.encode(_full(5))}
    halves = [z.shards[: z.S // 2], z.shards[z.S // 2:]]
    progs = (([row(F, 5)], z.N), ([row(F, 5), row(F, 3), nary(L.OP_DIFFERENCE, 2)], z.B))
    a, b = L.Context(0), L.Context(0)
    try:
        for c, half in zip((a, b), halves):
            for s in half:
                c.load_fragment(IDX, F, 0, s, data[min(s, 1)])
            c.commit()
        # Each rank alone first: its share stays below 2^32, so only the exchange crosses it.  These calls also size the
        # workspaces for the collective ones: two ranks on one device must not grow a buffer while the peer's kernel waits
        # (INTEGRATION.md).
        for prog, exp in progs:
            alone = [c.count(IDX, prog, half) for c, half in zip((a, b), halves)]
            assert sum(alone) == exp and max(alone) < 1 << 32
        L.p2p_open_local([a, b])
        for prog, exp in progs:
            out = {}
            tb = threading.Thread(target=lambda: out.setdefault("b", b.count(IDX, prog, halves[1])))
            tb.start()
            out["a"] = a.count(IDX, prog, halves[0])
            tb.join()
            assert out == {"a": exp, "b": exp}
    finally:
        a.close()
        b.close()


# ------------------------------------------------------------------ CPU
def test_row_writer_matches_the_encoder_and_the_oracle():
    z = Sizes(3)
    for k0 in (0, SLOTS):
        want = full_row_bytes(k0, z.N >> 16)
        cols = np.arange(k0 << 16, z.N, dtype=np.uint64)
        assert want == roaring_io.encode(cols)
        bm = O.Bitmap.from_bytes(want)
        assert bm.count() == z.N - (k0 << 16) and bm.to_bytes() == want


def test_fragments_are_canonical_and_hold_the_model():
    """each distinct fragment is the oracle's canonical encoding, and its rows hold what the table in the docstring says"""
    for S in (2, 3, 4):
        held = {}
        for field, view, data, shards in fragments(S):
            assert O.Bitmap.from_bytes(data).to_bytes() == data
            for s in shards:
                assert (field, view, s) not in held
                held[field, view, s] = data
        assert sorted(s for f, v, s in held if f == U) == list(range(S))
        assert sorted(s for f, v, s in held if f == T) == list(range(S))
    ora = OracleCtx()
    z = load_world(ora, 3)
    frag = lambda f, v, s: ora.frags[(IDX, f, v)][s]
    for s in z.shards:
        rows, cnts = frag(F, 0, s).row_counts(s, None)
        assert dict(zip(rows.tolist(), cnts.tolist())) == ({3: SW} if s == 0 else {}) | {5: SW, 9: SW // 2, 10: SW // 2}
        rows, cnts = frag(A, 0, s).row_counts(s, None)
        assert dict(zip(rows.tolist(), cnts.tolist())) == {r: SW // 256 for r in range(4)}
        assert {t for _, t, _, _ in roaring_io.containers(frag(A, 0, s).to_bytes())} == {roaring_io.ARRAY}


@pytest.fixture(scope="module")
def oracle_world():
    ora = OracleCtx()
    return ora, load_world(ora, 3)


@pytest.mark.parametrize("check", ORACLE_CHECKS, ids=lambda c: c.__name__[6:])
def test_closed_forms_on_the_oracle(oracle_world, check):
    """the expectations the device is held to, at S = 3, against the CPU oracle driven through the same calls"""
    ora, z = oracle_world
    check(ora, z)


def test_executor_closed_forms_on_the_oracle(oracle_world):
    ora, z = oracle_world
    check_executor(executor_on(ora, z.S), z)


def test_percentile_of_counts_restates_the_list_form():
    rng = np.random.default_rng(5)
    for _ in range(40):
        mult = {int(v): int(rng.integers(1, 9)) for v in rng.integers(-20, 21, int(rng.integers(1, 5)))}
        nums = [v for v, n in mult.items() for _ in range(n)]
        for nth in (0, 100, 50, 12.5, 99.9, 0.1, float(rng.uniform(0, 100))):
            assert percentile_of_counts(mult, nth) == percentile_of_list(nums, nth)[0], (mult, nth)
    z = Sizes(4097)
    for rank in (z.B, z.B - 1):
        assert int(z.N * nth_at_rank(z.N, rank) / 100.0) == rank


def test_past_2_32_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_past_2_32.py"], env={"FBGPU_UNIT_BATCH": "16"}, timeout=3000)
