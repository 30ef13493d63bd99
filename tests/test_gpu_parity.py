"""GPU parity tests: every result of the CUDA path (through the C ABI) is compared bit-exactly with the CPU
oracle on the same seeded inputs, against the reference's golden vectors, and — at BASELINE sizes — through
size-independent properties."""
import json
import os

import numpy as np
import pytest

from featurebase_b200 import datagen as D
from featurebase_b200 import executor as X
from featurebase_b200 import roaring_io
from oracle import oracle as O
from tests import archetypes as A
from tests.golden import vectors as V
from tests.oracle_exec import Pair

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
SW = 1 << 20


def test_config1_single_shard_plumbing():
    """BASELINE config 1: 1 shard, 2 rows @1 %: Count(Intersect) and the intersection bytes, bit-exact"""
    p = Pair()
    p.field("f")
    p.load("f", X.VIEW_STANDARD, 0, D.fragment(1, 0, [0, 1], 0.01))
    real = hasattr(p.holder.ctx, "counters")                       # (the oracle-backed stand-in of the host-logic tests has no kernels)
    before = p.holder.ctx.counters().get("pair_kernel_queries", 0) if real else 0
    n = p.check_count("Count(Intersect(Row(f=0), Row(f=1)))")
    assert 40 < n < 200
    # the north-star query shape must reach the fused pair_count_kernel (round 2 lost it for a while to a program rewrite: 97 us
    # instead of 17 us per query, with every result still right)
    if real:
        assert p.holder.ctx.counters()["pair_kernel_queries"] == before + 1
    r = p.check_row("Intersect(Row(f=0), Row(f=1))")
    assert r.count == n
    p.check_count("Count(Row(f=0))")
    p.check_count("Count(Union(Row(f=0), Row(f=1)))")
    p.check_row("Row(f=1)")


def test_pair_kernel_padded_array_tails():
    """Count(Intersect(Row, Row)) on arrays whose last 16-byte chunk is padded (1..17, 63..65 elements), with the LAST element present on
    both sides: the fused pair kernel probes the pad copies too and must take them out again — in the right warp of its two-warp team and
    in 64-bit arithmetic (a per-warp share of the count can be negative).  One query per launch and all row pairs in one launch."""
    from featurebase_b200 import lib as L
    p = Pair(track_existence=False)
    p.field("f")
    sizes = list(range(1, 18)) + [63, 64, 65, 255, 257]
    bits = []
    for k, n in enumerate(sizes):
        cols = np.arange(n, dtype=np.uint64) * np.uint64(3) + np.uint64(5)            # row 2k: n columns
        other = np.concatenate([cols[-1:], cols[: n // 2], np.arange(n, dtype=np.uint64) * np.uint64(3) + np.uint64(70000 + 6)])   # row 2k+1 shares the last one and a few more
        for r, cc in ((2 * k, cols), (2 * k + 1, np.unique(other))):
            bits.append(np.uint64(r * SW) + cc)
            bits.append(np.uint64(r * SW) + cc + np.uint64(3 * 65536))               # a second slot with the same pattern
    p.load("f", X.VIEW_STANDARD, 0, roaring_io.encode(np.sort(np.concatenate(bits))))
    fid = p.idx.fields["f"].id
    for k, n in enumerate(sizes):
        for a, b in ((2 * k, 2 * k + 1), (2 * k + 1, 2 * k), (2 * k, 2 * k)):
            got = p.check_count(f"Count(Intersect(Row(f={a}), Row(f={b})))")
            assert got == (2 * n if a == b else 2 * (1 + n // 2)), (n, a, b, got)
    ra, rb = [2 * k for k in range(len(sizes))], [2 * k + 1 for k in range(len(sizes))]
    got = p.holder.ctx.count_pairs(p.idx.id, fid, 0, ra, fid, 0, rb, [0])
    assert [int(x) for x in got] == [2 * (1 + n // 2) for n in sizes]


def test_container_combinations_table_on_gpu():
    """The reference's TestContainerCombinations table (roaring_internal_test.go:2974-3780) evaluated by the CUDA
    kernels: one shard per (x, y, enc_x, enc_y); ops intersect/union/difference/xor; results as sets AND as
    canonical bytes, plus the fused count path."""
    rows = json.load(open(os.path.join(GOLD, "container_combinations.json")))["rows"]
    expected = {}
    for r in rows:
        op = r["op"].replace("InPlaceWrapper", "")
        if op in ("intersect", "union", "difference", "xor"):
            expected[(op, r["x"], r["y"])] = r["exp"]
    pairs = sorted({(x, y) for (_, x, y) in expected})
    p = Pair(track_existence=False)
    p.field("f")
    types = [O.ARRAY, O.BITMAP, O.RUN]
    cache = {(n, t): A.container(n, t) for n in A.NAMES for t in types}
    shard_of, s = {}, 0
    for (x, y) in pairs:
        for tx in types:
            for ty in types:
                frag = O.Bitmap()
                cx, cy = cache[(x, tx)], cache[(y, ty)]
                if cx.n:
                    frag.put(0 * 16 + 5, cx)       # row 0, slot 5
                if cy.n:
                    frag.put(1 * 16 + 5, cy)       # row 1, slot 5
                p.load("f", X.VIEW_STANDARD, s, frag.to_bytes(optimize=False))
                shard_of[(x, y, tx, ty)] = s
                s += 1
    shards = list(range(s))
    qs = {"intersect": "Intersect(Row(f=0), Row(f=1))", "union": "Union(Row(f=0), Row(f=1))",
          "difference": "Difference(Row(f=0), Row(f=1))", "xor": "Xor(Row(f=0), Row(f=1))"}
    for op, q in qs.items():
        got = p.check_row(q, shards)                                  # bytes == oracle canonical bytes over all shards
        cols = got.columns()
        per_shard = {}
        sh = (cols >> np.uint64(20)).astype(np.int64)
        for k in np.unique(sh):
            per_shard[int(k)] = (cols[sh == k] & np.uint64(SW - 1)).astype(np.int64)
        tot, per = p.ex.ctx.count(p.idx.id, p.ex._bitmap_call(p.idx, __import__("featurebase_b200").pql.parse(q)[0]), shards, per_shard=True)
        checked = 0
        for (o, x, y), exp_name in expected.items():
            if o != op:
                continue
            exp = A.archetype_values(exp_name) + 5 * 65536
            for tx in types:
                for ty in types:
                    k = shard_of[(x, y, tx, ty)]
                    g = per_shard.get(k, np.zeros(0, dtype=np.int64))
                    assert np.array_equal(g, exp), (op, x, y, tx, ty)
                    assert int(per[k]) == len(exp), (op, x, y, tx, ty)
                    checked += 1
        assert checked >= 76 * 9
        assert tot == int(per.sum())


@pytest.mark.parametrize("mode", [0, 1])
def test_density_sweep_intersect_count(mode):
    """BASELINE config 5 (reduced shard count): p in 0.01 %..50 %, uniform and clustered generators; fused pair
    kernel, general evaluator and Row bytes all agree with the oracle; container mix recorded"""
    for pi, pdens in enumerate([0.0001, 0.001, 0.01, 0.03, 0.0625, 0.125, 0.25, 0.5]):
        p = Pair(track_existence=False)
        p.field("f")
        shards = list(range(4))
        for s in shards:
            p.load("f", X.VIEW_STANDARD, s, D.fragment(3, s, [0, 1, 2], pdens, mode=mode, mean_run=64.0))
        st = p.holder.ctx.stats()
        if mode == 1 and pdens >= 0.01:
            assert st["run_containers"] > 0
        if mode == 0 and pdens >= 0.0625:
            assert st["bitmap_containers"] > 0
        a = p.check_count("Count(Intersect(Row(f=0), Row(f=1)))")                 # fused pair kernel
        b = p.check_count("Count(Intersect(Row(f=0), Row(f=1), Row(f=0)))")       # general evaluator
        assert a == b
        p.check_row("Intersect(Row(f=0), Row(f=1))")
        p.check_row("Union(Row(f=0), Row(f=1), Row(f=2))")
        p.check_row("Difference(Row(f=0), Row(f=1))")
        p.check_row("Xor(Row(f=0), Row(f=2))")


def test_mixed_encoding_pairs():
    """array x bitmap x run operands in the same query (different densities per row)"""
    p = Pair(track_existence=False)
    p.field("f")
    for s in range(3):
        parts = [D.fragment(9, s, [0], 0.004), D.fragment(9, s, [1], 0.3), D.fragment(9, s, [2], 0.2, mode=1, mean_run=200.0),
                 D.fragment(9, s, [3], 0.9, mode=1, mean_run=5000.0)]
        merged = O.Bitmap()
        for d in parts:
            merged = merged.union(O.Bitmap.from_bytes(d))
        p.load("f", X.VIEW_STANDARD, s, merged.to_bytes())
    for a in range(4):
        for b in range(4):
            p.check_count(f"Count(Intersect(Row(f={a}), Row(f={b})))")
            p.check_row(f"Intersect(Row(f={a}), Row(f={b}))")
            p.check_row(f"Difference(Row(f={a}), Row(f={b}))")
            p.check_row(f"Xor(Row(f={a}), Row(f={b}))")
            p.check_row(f"Union(Row(f={a}), Row(f={b}))")
    p.check_count("Count(Intersect(Union(Row(f=0), Row(f=2)), Xor(Row(f=1), Row(f=3)), Row(f=1)))")


def test_union_intersect_count_config2_small():
    """BASELINE config 2 shape at reduced size: 8 shards, 64 rows @1 %"""
    p = Pair(track_existence=False)
    p.field("f")
    bulk = D.fragments(1, range(8), range(64), 0.01, threads=4)
    for s in range(8):
        p.load("f", X.VIEW_STANDARD, s, bulk.fragment_bytes(s))
    ua = "Union(" + ", ".join(f"Row(f={r})" for r in range(32)) + ")"
    ub = "Union(" + ", ".join(f"Row(f={r})" for r in range(32, 64)) + ")"
    n = p.check_count(f"Count(Intersect({ua}, {ub}))")
    assert n > 0
    p.check_row(f"Intersect({ua}, {ub})")


def test_executor_goldens_and_edge_semantics():
    """executor_test.go:1236-1373 + SURVEY Appendix E"""
    for name, (rows, q, exp) in V.EXEC_SETOPS.items():
        p = Pair()
        p.field("general")
        for row, cols in rows.items():
            for c in cols:
                p.holder.set_bit("i", "general", row, c)
        p.sync_pending()
        got = p.ex.execute("i", q)[0]
        if name == "count":
            assert got == exp
        else:
            assert list(got.columns()) == exp, name
    p = Pair()
    p.field("general")
    p.holder.set_bit("i", "general", 10, 1)
    p.holder.set_bit("i", "general", 11, SW + 2)
    p.sync_pending()
    with pytest.raises(X.QueryError):
        p.ex.execute("i", "Intersect()")                  # executor_test.go:1289-1297
    with pytest.raises(X.QueryError):
        p.ex.execute("i", "Difference()")
    assert p.ex.execute("i", "Union()")[0].count == 0     # executor_test.go:1321-1332
    assert p.ex.execute("i", "Xor()")[0].count == 0
    assert list(p.ex.execute("i", "Not(Row(general=10))")[0].columns()) == [SW + 2]
    assert list(p.ex.execute("i", "All()")[0].columns()) == [1, SW + 2]
    assert p.ex.execute("i", "Count(Row(general=99))")[0] == 0
    p.check_row("Not(Union(Row(general=10), Row(general=11)))")


def _bsi_pair(values, depth, shard=0):
    p = Pair()
    p.field("v", "int", min=-(1 << depth) + 1, max=(1 << depth) - 1, bit_depth=depth)
    for col, val in values.items():
        p.holder.set_value("i", "v", shard * SW + col, val)
    p.sync_pending()
    return p


def test_bsi_range_goldens_on_gpu():
    """fragment_internal_test.go:606-916 literal cases through Row(v <op> k)"""
    for values, depth, checks in V.BSI_RANGE_CASES:
        if depth == 64:
            continue  # covered at the C-ABI level by tests/test_bsi_wide_values.py::test_between_common_bits_regression_depth_64
        p = _bsi_pair(values, depth)
        for op, pred, exp in checks:
            q = f"Row(v >< [{pred[0]},{pred[1]}])" if op == "><" else f"Row(v {op} {pred})"
            got = p.ex.execute("i", q)[0]
            f = p.idx.fields["v"]
            inside = (lambda x: f.bit_depth_min() <= x <= f.bit_depth_max())
            if (op != "><" and inside(pred)) or (op == "><" and inside(pred[0]) and inside(pred[1])):
                assert list(got.columns()) == sorted(exp), (op, pred)
            p.check_row(q)


@pytest.mark.parametrize("signed", [False, True])
def test_bsi_diagonal_exhaustive_on_gpu(signed):
    """fragment_internal_test.go:3768-3948 / 4113-4275"""
    k = 6
    if signed:
        lo, hi = 1 - (1 << k), (1 << k) - 1
        values = {i - lo: i for i in range(lo, hi + 1)}
        checks = range(2 * lo, 2 * hi)
    else:
        values = {i: i for i in range(1 << k)}
        checks = range(-3, 1 << (k + 1))
    p = _bsi_pair(values, k, shard=2)
    base = 2 * SW
    for pr in checks:
        for op, f in (("<", lambda v: v < pr), ("<=", lambda v: v <= pr), (">", lambda v: v > pr),
                      (">=", lambda v: v >= pr), ("==", lambda v: v == pr), ("!=", lambda v: v != pr)):
            exp = sorted(base + c for c, v in values.items() if f(v))
            got = p.ex.execute("i", f"Row(v {op} {pr})")[0]
            assert list(got.columns()) == exp, (op, pr)
        for q in (pr, pr + 1, pr + 7):
            exp = sorted(base + c for c, v in values.items() if pr <= v <= q)
            assert list(p.ex.execute("i", f"Row(v >< [{pr},{q}])")[0].columns()) == exp, (pr, q)


def test_bsi_uniform_u32_config3_small():
    """BASELINE config 3 shape: 32-bit uniform values (bit planes are bitmap containers, exists row is runs)"""
    p = Pair()
    p.field("v", "int", min=0, max=(1 << 32) - 1)
    assert p.idx.fields["v"].bit_depth == 32
    ncols = [SW, 300000]
    for s, n in enumerate(ncols):
        p.load("v", X.VIEW_BSI, s, D.bsi_fragment(7, s, n, 32, 0, (1 << 32) - 1))
    for k in (1 << 31, int(0.99 * (1 << 32)), 0, 1, (1 << 32) - 2, 12345678):
        for op in (">", ">=", "<", "<=", "==", "!="):
            p.check_count(f"Count(Row(v {op} {k}))")
        p.check_row(f"Row(v > {k})")
    p.check_row(f"Row(v >< [{1 << 20},{1 << 31}])")
    # direct value check on a sample
    got = set(p.ex.execute("i", f"Row(v > {1 << 31})", [1])[0].columns().tolist())
    for c in range(0, 300000, 997):
        v = D.bsi_value(7, 1, c, 0, (1 << 32) - 1)
        assert ((SW + c) in got) == (v > (1 << 31))


def test_topk_topn_rowcounts():
    """doTopK (executor.go:2705) / fragment.top with ids: exact per-row counts with and without filter"""
    p = Pair(track_existence=False)
    p.field("f")
    p.field("g")
    shards = [0, 1, 2]
    for s in shards:
        merged = O.Bitmap()
        for r, dens in ((0, 0.02), (1, 0.001), (3, 0.3), (10, 0.08), (11, 0.0004)):
            merged = merged.union(O.Bitmap.from_bytes(D.fragment(4, s, [r], dens, mode=(1 if r == 3 else 0))))
        p.load("f", X.VIEW_STANDARD, s, merged.to_bytes())
        p.load("g", X.VIEW_STANDARD, s, D.fragment(5, s, [7], 0.25))
    exp, expf = {}, {}
    for s in shards:
        rows, cnts = p.ora.frag("f", 0, s).row_counts(s, None)
        for r, c in zip(rows.tolist(), cnts.tolist()):
            exp[r] = exp.get(r, 0) + c
        rows, cnts = p.ora.frag("f", 0, s).row_counts(s, p.ora.row("g", 0, 7, s))
        for r, c in zip(rows.tolist(), cnts.tolist()):
            expf[r] = expf.get(r, 0) + c
    order = lambda d: sorted(d.items(), key=lambda kv: (-kv[1], kv[0]))
    assert p.ex.execute("i", "TopK(f, k=10)")[0] == order(exp)
    assert p.ex.execute("i", "TopK(f, k=2)")[0] == order(exp)[:2]
    assert p.ex.execute("i", "TopK(f, k=10, filter=Row(g=7))")[0] == order(expf)
    assert p.ex.execute("i", "TopN(f, Row(g=7), n=3)")[0] == order(expf)[:3]
    ids = [0, 3, 11, 99]
    got = p.ex.execute("i", "TopN(f, Row(g=7), n=5, ids=[0,3,11,99])")[0]          # plain-Row Src: fused multi-pair kernel
    assert got == order({i: expf[i] for i in ids if expf.get(i)})
    got = p.ex.execute("i", "TopN(f, Intersect(Row(g=7), Row(g=7)), n=5, ids=[0,3,11,99])")[0]   # general Src: filter bitmaps
    assert got == order({i: expf[i] for i in ids if expf.get(i)})
    pc = p.holder.ctx.count_pairs(p.idx.id, p.idx.fields["f"].id, 0, [0, 1, 3, 10, 11, 99, 3], p.idx.fields["g"].id, 0, [7, 7, 7, 7, 7, 7, 8], shards)
    assert pc.tolist() == [expf.get(r, 0) for r in (0, 1, 3, 10, 11, 99)] + [0]
    assert p.ex.execute("i", "Rows(f)")[0] == sorted(exp)


def test_groupby_two_and_three_fields():
    """groupByIterator (executor.go:8617-8934) vs the oracle's nested-loop restatement"""
    p = Pair(track_existence=False)
    for n in ("a", "b", "c"):
        p.field(n)
    shards = [0, 1, 5]
    for s in shards:
        fa, fb = D.groupby_fragments(1, 2, s, 0.02, 16, 8)
        p.load("a", X.VIEW_STANDARD, s, fa)
        p.load("b", X.VIEW_STANDARD, s, fb)
        p.load("c", X.VIEW_STANDARD, s, D.fragment(6, s, [0, 1, 2], 0.3))
    ra, rb, rc = list(range(16)), list(range(8)), [0, 1, 2]

    def oracle_counts(fields, row_ids, filt_call=None):
        out = np.zeros(int(np.prod([len(r) for r in row_ids])), dtype=np.uint64)
        for s in shards:
            filt = p.ora.eval_shard(filt_call, s) if filt_call is not None else None
            O.groupby_shard([p.ora.frag(f, 0, s) for f in fields], s, row_ids, filt, out)
        return out.reshape([len(r) for r in row_ids])

    def to_groups(fields, row_ids, counts):
        out = []
        for flat in np.flatnonzero(counts.reshape(-1)):
            ix = np.unravel_index(int(flat), counts.shape)
            out.append(([(f, row_ids[k][int(i)]) for k, (f, i) in enumerate(zip(fields, ix))], int(counts[ix])))
        return out

    from featurebase_b200 import pql
    got = p.ex.execute("i", "GroupBy(Rows(a), Rows(b))")[0]
    assert got == to_groups(["a", "b"], [ra, rb], oracle_counts(["a", "b"], [ra, rb]))
    assert sum(c for _, c in got) > 1000
    got = p.ex.execute("i", "GroupBy(Rows(a), Rows(b), filter=Row(c=1))")[0]
    assert got == to_groups(["a", "b"], [ra, rb], oracle_counts(["a", "b"], [ra, rb], pql.parse("Row(c=1)")[0]))
    got = p.ex.execute("i", "GroupBy(Rows(a))")[0]
    assert got == to_groups(["a"], [ra], oracle_counts(["a"], [ra]))
    got = p.ex.execute("i", "GroupBy(Rows(c), Rows(a), Rows(b))")[0]
    assert got == to_groups(["c", "a", "b"], [rc, ra, rb], oracle_counts(["c", "a", "b"], [rc, ra, rb]))
    # dense x sparse, multi-valued columns (c rows overlap: a column can be in several rows)
    got = p.ex.execute("i", "GroupBy(Rows(c), Rows(a))")[0]
    assert got == to_groups(["c", "a"], [rc, ra], oracle_counts(["c", "a"], [rc, ra]))
    got = p.ex.execute("i", "GroupBy(Rows(a), Rows(c), filter=Row(b=3))")[0]
    assert got == to_groups(["a", "c"], [ra, rc], oracle_counts(["a", "c"], [ra, rc], pql.parse("Row(b=3)")[0]))


def test_full_size_properties_1024_shards():
    """BASELINE config 5 at full size (1024 shards x 2^20, 1 %): size-independent properties instead of the oracle:
    inclusion-exclusion, idempotence, commutativity, per-shard sums, fused == general path; plus oracle spot checks"""
    from featurebase_b200 import lib as L
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    idx.create_field("f")
    ex = X.Executor(h)
    shards = np.arange(1024, dtype=np.uint64)
    bulk = D.fragments(1, shards, [0, 1, 2], 0.01)
    h.ctx.load_fragments(idx.id, idx.fields["f"].id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
    idx.shards.update(range(1024))
    q = lambda s: ex.execute("i", s)[0]
    a, b = q("Count(Row(f=0))"), q("Count(Row(f=1))")
    i_ab, u_ab, x_ab, d_ab, d_ba = (q("Count(Intersect(Row(f=0), Row(f=1)))"), q("Count(Union(Row(f=0), Row(f=1)))"),
                                    q("Count(Xor(Row(f=0), Row(f=1)))"), q("Count(Difference(Row(f=0), Row(f=1)))"),
                                    q("Count(Difference(Row(f=1), Row(f=0)))"))
    assert abs(a - 0.01 * 1024 * SW) < 0.002 * 1024 * SW
    assert i_ab + u_ab == a + b
    assert x_ab == u_ab - i_ab == d_ab + d_ba
    assert d_ab == a - i_ab
    assert q("Count(Intersect(Row(f=0), Row(f=0)))") == a
    assert q("Count(Intersect(Row(f=1), Row(f=0)))") == i_ab
    assert q("Count(Intersect(Row(f=0), Row(f=1), Row(f=0)))") == i_ab          # general evaluator vs fused pair kernel
    ops = ex._bitmap_call(idx, __import__("featurebase_b200").pql.parse("Intersect(Row(f=0), Row(f=1))")[0])
    tot, per = h.ctx.count(idx.id, ops, shards, per_shard=True)
    assert tot == i_ab == int(per.sum())
    # oracle spot check on 3 shards
    for s in (0, 511, 1023):
        fr = O.Bitmap.from_bytes(bulk.fragment_bytes(s))
        assert int(per[s]) == fr.row(0, s).intersection_count(fr.row(1, s))
    r = ex.execute("i", "Intersect(Row(f=0), Row(f=1))")[0]
    assert r.count == i_ab and len(r.columns()) == i_ab


@pytest.mark.parametrize("env", ["FBGPU_FORCE_WORDPAR"])
def test_alternative_eval_kernels(env, monkeypatch):
    """the word-parallel kernel (bitmap-heavy programs) is normally picked by a heuristic; force it over array, bitmap and
    run operands, counts and filter bitmaps, and compare with the oracle"""
    monkeypatch.setenv(env, "1")
    p = Pair()
    p.field("f")
    p.field("v", "int", min=-2000, max=2000)
    for s in range(3):
        parts = [D.fragment(9, s, [0, 4, 5, 6], 0.004), D.fragment(9, s, [1], 0.3), D.fragment(9, s, [2], 0.2, mode=1, mean_run=200.0),
                 D.fragment(9, s, [3], 0.9, mode=1, mean_run=5000.0)]
        merged = O.Bitmap()
        for d in parts:
            merged = merged.union(O.Bitmap.from_bytes(d))
        p.load("f", X.VIEW_STANDARD, s, merged.to_bytes())
    rng = np.random.default_rng(5)
    for col, val in zip(rng.choice(3 * SW, 5000, replace=False), rng.integers(-2000, 2000, 5000)):
        p.holder.set_value("i", "v", int(col), int(val))
    p.sync_pending()
    for q in ("Count(Union(Row(f=0), Row(f=1), Row(f=2), Row(f=4), Row(f=5), Row(f=6)))",
              "Count(Intersect(Union(Row(f=0), Row(f=4), Row(f=5), Row(f=6), Row(f=2)), Xor(Row(f=1), Row(f=3), Row(f=0), Row(f=4)), Row(f=1)))",
              "Count(Difference(Row(f=3), Row(f=0), Row(f=2), Row(f=4), Row(f=1)))",
              "Count(Not(Union(Row(f=0), Row(f=2))))",
              "Count(Row(v > 17))", "Count(Row(v <= -5))", "Count(Row(v >< [-100, 700]))", "Count(Row(v != 3))"):
        p.check_count(q)
    p.check_row("Union(Row(f=0), Row(f=2), Row(f=4), Row(f=5))")
    # filter bitmaps produced by the alternative kernel feed TopK / GroupBy
    exp = {}
    for s in range(3):
        rows, cnts = p.ora.frag("f", 0, s).row_counts(s, p.ora.eval_shard(__import__("featurebase_b200").pql.parse("Union(Row(f=1), Row(f=2), Row(f=0), Row(f=4))")[0], s))
        for r, c in zip(rows.tolist(), cnts.tolist()):
            exp[r] = exp.get(r, 0) + c
    got = p.ex.execute("i", "TopK(f, k=10, filter=Union(Row(f=1), Row(f=2), Row(f=0), Row(f=4)))")[0]
    assert got == sorted(exp.items(), key=lambda kv: (-kv[1], kv[0]))


def test_full_size_properties_bsi_and_groupby():
    """BASELINE config 3 (10 M records, 32-bit BSI) and one GPU's share of config 4 (512 shards, 256 x 256 GroupBy) at
    full size, checked through size-independent properties: complementary predicates partition the non-null set,
    monotonicity in k, GroupBy total = number of records = Count(All rows of a), marginals = per-row counts."""
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    ex = X.Executor(h)
    idx.create_field("v", "int", min=0, max=(1 << 32) - 1)
    n_rec = 10_000_000
    n_sh = (n_rec + SW - 1) // SW
    for s in range(n_sh):
        h.import_roaring("i", "v", X.VIEW_BSI, s, D.bsi_fragment(20, s, min(SW, n_rec - s * SW), 32, 0, (1 << 32) - 1))
    q = lambda t: ex.execute("i", t)[0]
    notnull = q("Count(Row(v != null))")
    assert notnull == n_rec
    prev = None
    for k in (0, 1, 12345, 1 << 20, 1 << 31, int(0.99 * (1 << 32)), (1 << 32) - 2):
        gt, le, eq, ne, ge = q(f"Count(Row(v > {k}))"), q(f"Count(Row(v <= {k}))"), q(f"Count(Row(v == {k}))"), q(f"Count(Row(v != {k}))"), q(f"Count(Row(v >= {k}))")
        assert gt + le == notnull and eq + ne == notnull and ge == gt + eq
        assert prev is None or gt <= prev
        prev = gt
        assert abs(gt / n_rec - (1 - (k + 1) / (1 << 32))) < 0.002          # uniform values
    assert q(f"Count(Row(v >< [{1 << 30},{1 << 31}]))") == q(f"Count(Row(v >= {1 << 30}))") - q(f"Count(Row(v > {1 << 31}))")

    idx.create_field("a")
    idx.create_field("b")
    S = 512
    for s in range(S):
        da, db = D.groupby_fragments(31, 32, s, 100e6 / (4096 * SW), 256, 256)
        h.import_roaring("i", "a", X.VIEW_STANDARD, s, da)
        h.import_roaring("i", "b", X.VIEW_STANDARD, s, db)
    shards = list(range(S))
    rows = list(range(256))
    fa, fb = idx.fields["a"], idx.fields["b"]
    counts = h.ctx.groupby(idx.id, [fa.id, fb.id], [0, 0], [rows, rows], shards)
    ca = h.ctx.row_counts(idx.id, fa.id, 0, shards, row_ids=rows)
    cb = h.ctx.row_counts(idx.id, fb.id, 0, shards, row_ids=rows)
    total = int(counts.sum())
    assert abs(total - 100e6 / 8) < 0.01 * 100e6 / 8                        # ~12.2 M records on this GPU's share
    assert total == int(ca.sum()) == int(cb.sum())                          # every record has exactly one a-row and one b-row
    assert np.array_equal(counts.sum(axis=1), ca) and np.array_equal(counts.sum(axis=0), cb)
    flt = ex._bitmap_call(idx, __import__("featurebase_b200").pql.parse("Row(b=7)")[0])
    sub = h.ctx.groupby(idx.id, [fa.id, fb.id], [0, 0], [rows, rows], shards, filter_ops=flt)
    assert np.array_equal(sub[:, 7], counts[:, 7]) and int(sub.sum()) == int(counts[:, 7].sum())


def test_full_size_every_shard_against_the_cpu_port():
    """BASELINE config[1] and config[3] at their full sizes, every unit compared (not sampled): the headline 64-row
    Union->Intersect->Count per-shard vector of all 1024 shards, and the complete 256 x 256 GroupBy tensor over all 4096 shards of
    config 4, against the CPU port run on the host's cores (threaded C restatement: groupByIterator's nested loop, executor.go:8617)."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench as B
    if os.environ.get("FBGPU_TEST_ON_EMULATOR"):
        pytest.skip("full BASELINE sizes: device only")
    pool = O.Pool()
    # ---- config[1]
    S = 1024
    shards = np.arange(S, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    fld = idx.create_field("f")
    ex = X.Executor(h)
    bulk = B.gen_headline(shards)
    h.ctx.load_fragments(idx.id, fld.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
    idx.shards.update(range(S))
    ops = ex._bitmap_call(idx, __import__("featurebase_b200").pql.parse(B.query_text())[0].children[0])
    tot, per = h.ctx.count(idx.id, ops, shards, per_shard=True)
    frags = [O.Bitmap.from_bytes(bulk.fragment_bytes(i)) for i in range(S)]
    want = O.union_intersect_per_shard(pool, frags, shards, B.ROWS_A, B.ROWS_B)
    assert np.array_equal(np.asarray(per, dtype=np.uint64), want) and tot == int(want.sum()) > 0
    # the 32 north-star pairs: every pair's count over all shards, fused and one by one
    pw, _ = O.bench_pair_counts(pool, frags, shards, B.PAIRS_A, B.PAIRS_B, materialise=False)
    got = h.ctx.count_pairs(idx.id, fld.id, 0, B.PAIRS_A, fld.id, 0, B.PAIRS_B, shards)
    assert np.array_equal(np.asarray(got, dtype=np.uint64), pw)
    h.ctx.close()
    del frags, bulk
    # ---- config[3]: all 4096 shards on this one GPU
    S = 4096
    h = X.Holder()
    idx = h.create_index("g", track_existence=False)
    fa, fb = idx.create_field("a"), idx.create_field("b")
    fr_a, fr_b = [], []
    for s in range(S):
        da, db = D.groupby_fragments(31, 32, s, 100e6 / (4096 * SW), 256, 256)
        h.import_roaring("g", "a", X.VIEW_STANDARD, s, da)
        h.import_roaring("g", "b", X.VIEW_STANDARD, s, db)
        fr_a.append(O.Bitmap.from_bytes(da))
        fr_b.append(O.Bitmap.from_bytes(db))
    rows = list(range(256))
    shards = np.arange(S, dtype=np.uint64)
    counts = h.ctx.groupby(idx.id, [fa.id, fb.id], [0, 0], [rows, rows], shards)
    want, _ = O.bench_groupby(pool, [fr_a, fr_b], shards, [rows, rows])
    assert np.array_equal(np.asarray(counts, dtype=np.uint64).reshape(-1), want)
    assert abs(int(want.sum()) - 100e6) < 0.01 * 100e6
    h.ctx.close()
    pool.close()


def test_thread_safety_and_api_edges():
    """The C ABI promises re-entrancy from any thread (goroutines migrate between OS threads): 8 threads issue mixed
    queries concurrently (ctypes releases the GIL) and must get the sequential answers; plus argument edge cases."""
    import threading
    from featurebase_b200 import lib as L
    p = Pair(track_existence=False)
    p.field("f")
    shards = list(range(6))
    for s in shards:
        p.load("f", X.VIEW_STANDARD, s, D.fragment(3, s, list(range(8)), 0.02))
    queries = ["Count(Intersect(Row(f=0), Row(f=1)))", "Count(Union(Row(f=0), Row(f=1), Row(f=2), Row(f=3)))",
               "Count(Xor(Row(f=4), Row(f=5)))", "Count(Difference(Row(f=6), Row(f=7), Row(f=0)))", "Intersect(Row(f=2), Row(f=3))",
               "TopK(f, k=4, filter=Row(f=1))"]
    expect = [p.ex.execute("i", q)[0] for q in queries]
    expect[4] = expect[4].roaring
    errors = []

    def worker(tid):
        try:
            for it in range(12):
                k = (tid + it) % len(queries)
                got = p.ex.execute("i", queries[k])[0]
                if k == 4:
                    got = got.roaring
                if got != expect[k]:
                    errors.append((tid, it, queries[k]))
        except Exception as e:  # noqa: BLE001
            errors.append((tid, repr(e)))

    ths = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errors, errors[:3]
    ctx, iid, fid = p.holder.ctx, p.idx.id, p.idx.fields["f"].id
    row = lambda r: L.Op(L.OP_ROW, fid, 0, 0, r, 0, 0, 0)
    # empty shard list, unknown field/view/row, duplicate shards in a Row call, malformed programs
    assert ctx.count(iid, [row(0)], []) == 0
    assert ctx.count(iid, [L.Op(L.OP_ROW, 999, 0, 0, 0, 0, 0, 0)], shards) == 0
    assert ctx.count(iid, [row(12345)], shards) == 0
    assert ctx.count(iid, [row(0)], [77, 78]) == 0
    one = ctx.row(iid, [row(0)], [2])
    assert ctx.row(iid, [row(0)], [2, 2, 2]) == one
    for bad in ([], [row(0), row(1)], [L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)], [row(0), L.Op(42, 0, 0, 0, 0, 0, 0, 0)]):
        with pytest.raises(L.FbgpuError) as ei:
            ctx.count(iid, bad, shards)
        assert ei.value.code == L.E_INVALID
    with pytest.raises(L.FbgpuError) as ei:
        ctx.count(iid, [L.Op(L.OP_INTERSECT, 0, 0, 0, 0, 0, 0, 0)], shards)
    assert ei.value.code == L.E_QUERY
    with pytest.raises(L.FbgpuError) as ei:
        ctx.load_fragment(iid, fid, 0, 9, b"\x00" * 32)
    assert ei.value.code == L.E_FORMAT
    # drop + reload
    before = ctx.count(iid, [row(0)], shards)
    ctx.drop_fragment(iid, fid, 0, 3)
    after = ctx.count(iid, [row(0)], shards)
    assert after == before - p.ora.row("f", 0, 0, 3).count()
    ctx.load_fragment(iid, fid, 0, 3, D.fragment(3, 3, list(range(8)), 0.02))
    assert ctx.count(iid, [row(0)], shards) == before


def test_executor_topk_topn_groupby_goldens_on_gpu():
    """executor_test.go:1758-1809 (TopK), :1846-1889 (TopN exact), :6033-6120 (GroupBy Basic / Filter / error cases)"""
    def pair_with(fields_bits):
        p = Pair()
        for name, bits in fields_bits.items():
            p.field(name)
            for r, c in bits:
                p.holder.set_bit("i", name, r, c)
        p.sync_pending()
        return p
    p = pair_with({"f": V.TOPK_BITS})
    assert p.ex.execute("i", "TopK(f, k=2)")[0] == V.TOPK_EXPECT
    p = pair_with({"f": V.TOPN_BITS, "other": [(0, 0)]})
    assert p.ex.execute("i", "TopN(f, n=2)")[0] == V.TOPN_EXPECT
    assert p.ex.execute("i", "TopN(f, Row(other=0), n=5)")[0] == [(0, 1), (10, 1)]
    p = pair_with({"general": V.GROUPBY_GENERAL, "sub": V.GROUPBY_SUB})
    fmt = lambda res: [(tuple(r for _, r in g), c) for g, c in res]
    assert fmt(p.ex.execute("i", "GroupBy(Rows(general), Rows(sub))")[0]) == V.GROUPBY_BASIC
    assert fmt(p.ex.execute("i", "GroupBy(Rows(general), Rows(sub), filter=Row(general=10))")[0]) == V.GROUPBY_FILTER_GENERAL_10
    assert fmt(p.ex.execute("i", "GroupBy(Rows(general), Rows(sub), limit=2)")[0]) == V.GROUPBY_BASIC[:2]
    with pytest.raises(X.QueryError, match="need at least one child call"):
        p.ex.execute("i", "GroupBy()")
    with pytest.raises(X.QueryError, match="field not found"):
        p.ex.execute("i", "GroupBy(Rows(missing))")


def test_any_early_exit_and_pair_type_histogram():
    """fbgpu_any (Row.Any, row.go:258 — early exit by shard blocks) and fbgpu_pair_types (the statsHit analogue: which of the nine
    container-pair kernels a Count(Intersect(Row, Row)) exercises, roaring.go:4477-4614)"""
    import struct
    from featurebase_b200 import lib as L
    p = Pair(track_existence=False)
    f = p.field("f")
    n_sh, frags = 40, {}
    for s in range(n_sh):
        # row 0 only exists from shard 30 on; rows 1 / 2: uniform and clustered data so that arrays, bitmaps and runs all occur
        rows = ([0] if s >= 30 else []) + [1, 2]
        data = D.fragment(41, s, rows, 0.3 if s % 3 == 0 else 0.01, mode=s % 2)
        p.load("f", X.VIEW_STANDARD, s, data)
        frags[s] = data
    shards = list(range(n_sh))
    ctx, idx = p.ex.ctx, p.idx
    row = lambda r: L.Op(L.OP_ROW, f.id, 0, 0, r, 0, 0, 0)
    q = [row(0), row(1), L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)]
    launches0 = ctx.counters()["kernel_launches"]
    assert ctx.any(idx.id, [row(1)], shards) is True
    assert ctx.counters()["kernel_launches"] - launches0 == 1                   # found in the first block of 8 shards
    assert ctx.any(idx.id, [row(0)], shards[:30]) is False                      # absent: every block was looked at
    assert ctx.any(idx.id, [row(0)], shards) is True
    assert ctx.any(idx.id, q, shards) == (ctx.count(idx.id, q, shards) > 0)
    assert ctx.any(idx.id, [row(7)], shards) is False
    with pytest.raises(L.FbgpuError):
        ctx.any(idx.id, [L.Op(L.OP_INTERSECT, 0, 0, 0, 0, 0, 0, 0)], shards[:0])
    # expected histogram from the container tables of the loaded images (type per key; key = row * 16 + slot)
    want = np.zeros((4, 4), dtype=np.uint64)
    for s in shards:
        raw = frags[s]
        n = struct.unpack_from("<I", raw, 4)[0]
        typ = {}
        for i in range(n):
            key, t, _ = struct.unpack_from("<QHH", raw, 8 + 12 * i)
            typ[key] = t
        for slot in range(16):
            want[typ.get(1 * 16 + slot, 0), typ.get(2 * 16 + slot, 0)] += 1
    got = ctx.pair_types(idx.id, f.id, 0, 1, f.id, 0, 2, shards)
    assert np.array_equal(got, want), (got, want)
    assert int(got.sum()) == 16 * n_sh and (got > 0).sum() >= 3                 # several of the nine kernels are exercised
