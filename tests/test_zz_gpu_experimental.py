"""Device runs of everything written after round 1's GPU budget was spent.

The query-level tests below (BSI aggregates, RBF loader, further reference goldens, GroupBy post-processing, Percentile, time
views, embedded rows, Shift, All/Limit) use only entry points and kernels whose parity was already green on the GPU; their
host side — mirror, program compiler, readers, store tables — has been exercised on the CPU through tests/test_host_mirror.py
(oracle-backed context) and tests/test_store_inspect.py (the library's own compiler and store), so they run by default.
Array payloads are stored in the bank-sorted_order order by default since round 2 (csrc/stripe.h); FBGPU_ARRAY_SORTED=1 keeps the
reference's sorted order.  The *sorted_order* tests re-run the parity bodies under that switch (FBGPU_TEST_EXPERIMENTAL=1: they
repeat the long tables)."""
import os

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from featurebase_b200 import pql
from tests import test_gpu_parity as G
from tests.golden import vectors as V
from tests.oracle_exec import Pair

pytestmark = pytest.mark.gpu
# opt-in part: the parity bodies once more in the other array payload order
experimental = pytest.mark.skipif(not os.environ.get("FBGPU_TEST_EXPERIMENTAL"), reason="experimental layouts: set FBGPU_TEST_EXPERIMENTAL=1")


@pytest.fixture
def sorted_order(monkeypatch):
    monkeypatch.setenv("FBGPU_ARRAY_SORTED", "1")      # read when a context is created


@experimental
def test_sorted_order_set_ops(sorted_order):
    G.test_config1_single_shard_plumbing()
    G.test_container_combinations_table_on_gpu()
    G.test_mixed_encoding_pairs()
    G.test_union_intersect_count_config2_small()
    G.test_executor_goldens_and_edge_semantics()


@experimental
@pytest.mark.parametrize("mode", [0, 1])
def test_sorted_order_density_sweep(sorted_order, mode):
    G.test_density_sweep_intersect_count(mode)


@experimental
def test_sorted_order_bsi_topk_groupby(sorted_order):
    G.test_bsi_range_goldens_on_gpu()
    G.test_bsi_uniform_u32_config3_small()
    G.test_topk_topn_rowcounts()
    G.test_groupby_two_and_three_fields()


@experimental
@pytest.mark.parametrize("env", ["FBGPU_FORCE_WORDPAR"])
def test_sorted_order_alternative_kernels(sorted_order, env, monkeypatch):
    G.test_alternative_eval_kernels(env, monkeypatch)       # FORCE_WORDPAR must be ignored for views that hold arrays


# ---------------------------------------------------------------------------------------------------------------
# BSI aggregates (composition of already-verified entry points; bodies shared with tests/test_host_mirror.py)
# ---------------------------------------------------------------------------------------------------------------
def _setup(setup):
    p = Pair(track_existence=True)
    for name in setup["set"]:
        p.field(name)
    for name, (lo, hi) in setup["ranges"].items():
        p.field(name, "int", min=lo, max=hi, bit_depth=(63 if hi > (1 << 40) else None))
    for name, bits in setup["set"].items():
        for r, c in bits:
            p.holder.set_bit("i", name, r, c)
    for name, vals in setup["int"].items():
        for c, v in vals:
            p.holder.set_value("i", name, c, v)
    p.sync_pending()
    return p


def _check_agg(p, q, exp=None):
    """mirror result == reference flow on the oracle (per shard + ValCount reduce) [== literal expectation]"""
    call = pql.parse(q)[0]
    got = p.ex.execute("i", q)[0]
    ref = p.ora.sum(call, p.shards()) if call.name == "Sum" else p.ora.minmax(call, p.shards(), call.name == "Max")
    assert got == ref, (q, got, ref)
    if exp is not None:
        assert got == exp, (q, got, exp)
    return got


def test_fragment_top_goldens():
    """fragment_internal_test.go:1150-1272,1513-1537 through TopN(f[, Row(src=0)], n=..[, ids=..]) on one shard"""
    for rows, src, n, ids, exp in V.FRAG_TOP_CASES:
        p = Pair(track_existence=False)
        p.field("f")
        p.field("src")
        if rows == "large":
            from oracle import oracle as O
            pos = np.concatenate([np.uint64(i << 20) + np.arange(i, dtype=np.uint64) for i in range(1, 1000)])
            p.load("f", X.VIEW_STANDARD, 0, O.Bitmap.from_values(pos).to_bytes())
        else:
            for r, cols in rows.items():
                for c in cols:
                    p.holder.set_bit("i", "f", r, c)
        for c in (src or []):
            p.holder.set_bit("i", "src", 0, c)
        p.sync_pending()
        q = "TopN(f" + (", Row(src=0)" if src else "") + (f", n={n}" if n else "") + (", ids=[" + ",".join(map(str, ids)) + "]" if ids else "") + ")"
        assert p.ex.execute("i", q, [0])[0] == exp, q


def test_filter_sample_goldens():
    """roaring/filter_internal_test.go:78-138 at executor level, shards 0 and 2: Rows(f), rows holding one column (the
    column filter becomes a one-column filter row), Union of two rows"""
    SW = 1 << 20
    p = Pair(track_existence=False)
    p.field("f")
    p.field("c")                                        # row i = the single column (i << 16) + i
    for shard in (0, 2):
        for r, c in V.filter_sample_bits():
            p.holder.set_bit("i", "f", r, shard * SW + c)
        for i in range(1, 16):
            p.holder.set_bit("i", "c", i, shard * SW + (i << 16) + i)
    p.sync_pending()
    assert p.ex.execute("i", "Rows(f)")[0] == list(range(V.FILTER_SAMPLE_ROWS))
    for shards in ([0], [2], [0, 2]):
        for i in range(1, 16):
            got = p.ex.execute("i", f"TopK(f, k=1000, filter=Row(c={i}))", shards)[0]
            assert sorted(r for r, _ in got) == list(range(0, V.FILTER_SAMPLE_ROWS, i)) and {n for _, n in got} == {len(shards)}
        ids, cols = V.FILTER_ROWS_UNION
        got = p.check_row(f"Union(Row(f={ids[0]}), Row(f={ids[1]}))", shards)
        assert list(got.columns()) == [s * SW + c for s in shards for c in cols]
    rowset, col, exp = V.FILTER_ROWSET
    got = p.ex.execute("i", "TopN(f, Row(c=2), ids=[0,1,2,3])", [0])[0]
    assert sorted(r for r, _ in got) == exp


def test_bench_archetype_matrix():
    """roaring_container_test.go:62-88 shape matrix on the device: the 20 benchmark archetypes (2 draws each) stored in
    their NAMED encodings (unoptimised Pilosa bytes keep them: a 512-bit bitmap container, a 4096-element array, ...),
    all 1600 ordered pairs through the fused pair-count kernel, and the four set ops of a diagonal band as Row bytes"""
    from oracle import oracle as O
    from tests import archetypes as A
    rng = np.random.default_rng(23)
    cs = [(n, *A.bench_archetype(rng, n)) for n in A.BENCH_NAMES for _ in range(2)]
    shard, slot = 1, 3
    frag = O.Bitmap()
    for row, (_, c, v) in enumerate(cs):
        if len(v):
            frag.put(row * 16 + slot, c)
    p = Pair(track_existence=False)
    p.field("f")
    p.load("f", X.VIEW_STANDARD, shard, frag.to_bytes(optimize=False))
    masks = np.zeros((len(cs), 1 << 16), dtype=bool)
    for i, (_, _, v) in enumerate(cs):
        masks[i, v] = True
    ra, rb = np.divmod(np.arange(len(cs) ** 2), len(cs))
    got = p.holder.ctx.count_pairs(p.idx.id, p.idx.fields["f"].id, 0, ra, p.idx.fields["f"].id, 0, rb, [shard])
    exp = (masks.astype(np.uint32) @ masks.astype(np.uint32).T).reshape(-1)       # |a ∩ b| for every ordered pair
    assert np.array_equal(np.asarray(got, dtype=np.int64), exp.astype(np.int64))
    for i in range(len(cs)):
        for j in (i, (i + 1) % len(cs), (i + 7) % len(cs), (i + 19) % len(cs)):
            assert p.check_count(f"Count(Intersect(Row(f={i}), Row(f={j})))", [shard]) == int(exp[i * len(cs) + j])
            for op in ("Union", "Difference", "Xor"):
                p.check_row(f"{op}(Row(f={i}), Row(f={j}))", [shard])


def test_time_quantum_rows():
    """executor_test.go:470-515, 982-1010: Row(f=x, from=, to=) over a time field = the union of the row over the views
    viewsByTimeRange picks (time.go:158-235); the views are ordinary fragments, the union an ordinary program"""
    for quantum, cases in V.TIME_ROW_CASES.items():
        p = Pair()
        p.field("f", "time", quantum=quantum)
        p.field("plain")
        for row, col, ts in V.TIME_BITS:
            p.holder.set_bit("i", "f", row, col, timestamp=ts)
        p.holder.set_bit("i", "plain", 1, 5)
        p.sync_pending()
        for q, exp in cases:
            got = p.check_row(q)
            assert [int(c) for c in got.columns()] == exp, (quantum, q)
        assert [int(c) for c in p.check_row("Row(f=1)").columns()] == [2, 3, 4, 5, 6, 7]          # no range: the standard view
        if quantum == "YMDH":                                     # executor_test.go:675 legacy spelling (with YMD the last day is not fully covered)
            assert [int(c) for c in p.check_row("Range(f=1, from=1999-12-31T00:00, to=2002-01-01T03:00)").columns()] == [2, 3, 4, 5, 6, 7]
        assert p.check_count("Count(Intersect(Row(f=1, from=2000-01-01T00:00, to=2001-01-01T00:00), Row(f=1)))") == 3
        assert p.check_row("Row(f=1, from=2010-01-01T00:00, to=2011-01-01T00:00)").count == 0
        with pytest.raises(X.QueryError, match="not a time-field"):
            p.ex.execute("i", "Row(plain=1, from=2000-01-01T00:00)")
        # TopN(ids=..) over a time-ranged Src: the Src is the union over the covering views, not the standard view's row
        # (the fused pair path is for a plain Row only)
        narrow = "Row(f=1, from=2000-01-01T00:00, to=2001-01-01T00:00)"
        n_narrow, n_all = p.check_count(f"Count({narrow})"), p.check_count("Count(Row(f=1))")
        assert 0 < n_narrow < n_all
        assert p.ex.execute("i", f"TopN(f, {narrow}, ids=[1])")[0] == [(1, n_narrow)]
        assert p.ex.execute("i", "TopN(f, Row(f=1), ids=[1])")[0] == [(1, n_all)]


def test_kernel_table_goldens_on_device():
    """the 172 literal per-kernel cases of tests/golden/kernel_tables{,2}.json (roaring_internal_test.go table tests) with
    a set-op result, on the device: case k lives in shard k as rows 0 and 1 of one field, in the encodings the reference
    test names (unoptimised Pilosa bytes keep them), and one query per operation covers all of its shards"""
    import json
    import os
    from oracle import oracle as O
    from tests import archetypes as A
    gold = os.path.join(os.path.dirname(__file__), "golden")
    t1 = {"TestIntersectArrayRun": ("Intersect", "array", "runs"), "TestIntersectRunRun": ("Intersect", "aruns", "bruns"),
          "TestUnionInterval16InPlace": ("Union", "a", "b"), "TestUnionRunRun": ("Union", "aruns", "bruns"),
          "TestUnionArrayRun": ("Union", "array", "runs"), "TestDifferenceArrayRun": ("Difference", "array", "runs"),
          "TestDifferenceRunArray": ("Difference", "runs", "array"), "TestDifferenceRunRun": ("Difference", "aruns", "bruns"),
          "TestXorArrayRun": ("Xor", "a", "b"), "TestXorRunRun": ("Xor", "aruns", "bruns"),
          "TestIntersectBitmapRunBitmap": ("Intersect", "bitmap", "runs"), "TestIntersectBitmapRunArray": ("Intersect", "bitmap", "runs"),
          "TestUnionBitmapRun": ("Union", "bitmap", "runs"), "TestDifferenceRunBitmap": ("Difference", "runs", "bitmap"),
          "TestDifferenceBitmapRun": ("Difference", "bitmap", "runs"), "TestDifferenceBitmapArray": ("Difference", "bitmap", "array"),
          "TestDifferenceBitmapBitmap": ("Difference", "abitmap", "bbitmap"), "TestXorBitmapRun": ("Xor", "bitmap", "runs"),
          "TestIntersectArrayBitmap": ("Intersect", "array", "bitmap")}

    def cont(lit):
        if lit["kind"] == "array":
            return O.Container.array(lit["values"])
        if lit["kind"] == "runs":
            return O.Container.run(np.array(lit["values"], dtype=np.uint16).reshape(-1, 2))
        if lit["kind"] == "archetype":
            return A.container(lit["values"], O.BITMAP)
        w = np.zeros(1024, dtype=np.uint64)
        w[: len(lit["values"])] = np.array(lit["values"], dtype=np.uint64)
        return O.Container.bitmap(w)

    def values(lit):
        if lit["kind"] == "array":
            return sorted(lit["values"])
        if lit["kind"] == "runs":
            return [v for s_, l_ in lit["values"] for v in range(s_, l_ + 1)]
        if lit["kind"] == "archetype":
            return A.archetype_values(lit["values"]).tolist()
        return [64 * i + b for i, w in enumerate(lit["values"]) for b in range(64) if (w >> b) & 1]

    cases = []
    for name in ("kernel_tables.json", "kernel_tables2.json"):
        cases += [c for c in json.load(open(os.path.join(gold, name)))["cases"] if c["func"] in t1]
    assert len(cases) == 73 + 47
    p = Pair(track_existence=False)
    p.field("f")
    slot, by_op, expect = 5, {}, {}
    for k, c in enumerate(cases):
        op, fa, fb = t1[c["func"]]
        f = c["fields"]
        a, b = cont(f[fa]), cont(f[fb])
        if c["func"] == "TestDifferenceBitmapArray":
            a = a.intersect(O.Container.run(np.array([[0, 63]], dtype=np.uint16))).convert(O.BITMAP)
        frag = O.Bitmap()
        if a.n:
            frag.put(0 * 16 + slot, a)
        if b.n:
            frag.put(1 * 16 + slot, b)
        if a.n or b.n:
            p.load("f", X.VIEW_STANDARD, k, frag.to_bytes(optimize=False))
        by_op.setdefault(op, []).append(k)
        exp = f.get("exp") or f.get("expected")
        expect[k] = [((k * 16 + slot) << 16) + v for v in values(exp)]
    for op, shards in by_op.items():
        # Sets, not bytes: several of these reference cases use operands with adjacent, unmerged runs ([1,2],[3,4],[5,7]), which
        # no stored fragment contains.  The reference passes such a container through a one-sided union untouched, whereas the
        # device always emits the maximal runs of the result set, so the serialised forms legitimately differ there.
        q = f"{op}(Row(f=0), Row(f=1))"
        got = p.ex.execute("i", q, shards)[0]
        cols = [int(x) for x in got.columns()]
        assert cols == [int(x) for x in p.ora.eval_row(pql.parse(q)[0], shards).slice()], op
        assert cols == [v for k in shards for v in expect[k]], op              # == the reference's literal expectations
        assert got.count == len(cols)
        if op == "Intersect":
            tot, per = p.holder.ctx.count(p.idx.id, [X.L.Op(X.L.OP_ROW, p.idx.fields["f"].id, 0, 0, 0, 0, 0, 0), X.L.Op(X.L.OP_ROW, p.idx.fields["f"].id, 0, 0, 1, 0, 0, 0),
                                                     X.L.Op(X.L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)], shards, per_shard=True)
            assert [int(x) for x in per] == [len(expect[k]) for k in shards] and tot == sum(len(expect[k]) for k in shards)


def test_mixed_container_goldens_on_device():
    """TestUnionMixed / TestIntersectMixed / TestDifferenceMixed / TestXorRunRun1 and the full-container cases
    (roaring_internal_test.go:284-304, 694-735, 918-1022, 2026-2037, 4316-4323) on the device: case k lives in shard k as rows 0
    and 1 of one field in the encodings the reference test builds (unoptimised Pilosa bytes keep them); one query per operation"""
    from oracle import oracle as O
    from tests.test_oracle import _spec_container
    names = {"union": "Union", "intersect": "Intersect", "difference": "Difference", "xor": "Xor"}
    full = {"bitmap": ("bitmap", [0xFFFFFFFFFFFFFFFF] * 1024), "run": ("run", [(0, 65535)])}
    cases = [(op, a, b, exp) for _, op, a, b, exp, _ in V.MIXED_CONTAINER_CASES]
    for ea, eb in V.FULL_CONTAINER_ENCODINGS:
        cases.append(("intersect", full[ea], full[eb], list(range(65536))))
        cases.append(("difference", full[ea], full[eb], []))
    p = Pair(track_existence=False)
    p.field("f")
    slot, by_op, expect = 9, {}, {}
    for k, (op, a, b, exp) in enumerate(cases):
        frag = O.Bitmap()
        frag.put(0 * 16 + slot, _spec_container(a))
        frag.put(1 * 16 + slot, _spec_container(b))
        p.load("f", X.VIEW_STANDARD, k, frag.to_bytes(optimize=False))
        by_op.setdefault(op, []).append(k)
        expect[k] = [((k * 16 + slot) << 16) + v for v in exp]
    fid = p.idx.fields["f"].id
    for op, shards in by_op.items():
        got = p.check_row(f"{names[op]}(Row(f=0), Row(f=1))", shards)           # canonical bytes == the oracle's
        assert [int(x) for x in got.columns()] == [v for k in shards for v in expect[k]], op
        if op == "intersect":
            prog = [X.L.Op(X.L.OP_ROW, fid, 0, 0, 0, 0, 0, 0), X.L.Op(X.L.OP_ROW, fid, 0, 0, 1, 0, 0, 0), X.L.Op(X.L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)]
            tot, per = p.holder.ctx.count(p.idx.id, prog, shards, per_shard=True)
            assert [int(x) for x in per] == [len(expect[k]) for k in shards] and tot == sum(len(expect[k]) for k in shards)
            pairs = p.holder.ctx.count_pairs(p.idx.id, fid, 0, [0], fid, 0, [1], shards)      # the fused Intersect+Count kernel
            assert int(pairs[0]) == tot


def test_bitmap_level_goldens_on_device():
    """roaring/roaring_test.go Bitmap-level cases: operand a = row 0 of field "a", operand b = row 0 of field "b", values are
    columns (so the larger cases span three shards); counts through Count(op(...)), slices through the Row bytes"""
    from tests.test_oracle import _spec_values
    from oracle import oracle as O
    names = {"intersect": "Intersect", "difference": "Difference", "union": "Union", "xor": "Xor"}
    for cite, a, b, op, (kind, exp) in V.BITMAP_LEVEL_CASES:
        p = Pair(track_existence=False)
        p.field("a")
        p.field("b")
        for fld, spec in (("a", a), ("b", b)):
            vals = _spec_values(spec)
            for shard in np.unique(vals >> np.uint64(20)).tolist():
                part = vals[(vals >> np.uint64(20)) == np.uint64(shard)] & np.uint64((1 << 20) - 1)
                p.load(fld, X.VIEW_STANDARD, int(shard), O.Bitmap.from_values(part).to_bytes())
        if not p.idx.shards:
            continue
        q = f"{names[op]}(Row(a=0), Row(b=0))"
        if kind == "count":
            assert p.check_count(f"Count({q})") == exp, cite
            assert p.check_row(q).count == exp, cite
        else:
            assert [int(c) for c in p.check_row(q).columns()] == exp, cite


def test_embedded_rows_constrow_unionrows():
    """executor_test.go:1195-1234 (ConstRow with / without existence tracking), :7264-7287 (UnionRows over Rows / TopN),
    :5339-5340 (Rows(f, column=c)); the caller-provided row is an ordinary fragment of a scratch field on the device
    (what a Precomputed operand becomes, executePrecomputedCallShard :5535)"""
    SW = 1 << 20
    for track, exp in ((False, [2, 6, 7]), (True, [2, 6])):
        p = Pair(track_existence=track)
        p.field("h")
        for r, c in ((1, 2), (3, 4), (5, 6)):
            p.holder.set_bit("i", "h", r, c)
        p.sync_pending()
        assert [int(c) for c in p.check_row("ConstRow(columns=[2,6,7])").columns()] == exp
        assert p.check_count("Count(Intersect(ConstRow(columns=[2,4,9]), Row(h=3)))") == 1
        assert p.ex.execute("i", "ConstRow(columns=[])")[0].count == 0
    p = Pair(track_existence=False)
    p.field("s")
    for c, r in ((0, 1), (1, 2), (2, 3), (3, 1), (3, 5), (SW + 9, 2)):
        p.holder.set_bit("i", "s", r, c)
    p.sync_pending()
    assert p.ex.execute("i", "Count(UnionRows(TopN(s, n=1)))", [0])[0] == 2         # row 1: columns 0, 3
    assert p.check_count("Count(UnionRows(Rows(s)))", [0]) == 4
    assert p.check_count("Count(UnionRows(Rows(s)))") == 5
    assert [int(c) for c in p.check_row("UnionRows(Rows(s))").columns()] == [0, 1, 2, 3, SW + 9]
    assert p.ex.execute("i", "Rows(s, column=3)")[0] == [1, 5]
    assert p.ex.execute("i", f"Rows(s, column={SW + 9})")[0] == [2]
    assert p.ex.execute("i", "Rows(s, column=77)")[0] == []
    q = Pair()
    q.field("general")
    for r, c in [(10, 0), (10, SW + 1), (11, 2), (11, SW + 2), (12, 2), (12, SW + 2), (13, 3)]:
        q.holder.set_bit("i", "general", r, c)
    q.sync_pending()
    assert q.ex.execute("i", "Rows(general, column=2)")[0] == [11, 12]               # executor_test.go:5339


def test_shift_and_includes_column():
    """executor_test.go:6590-6673 (Shift: bit 0, container boundary, shard boundary, nested) and :6678-6706 (IncludesColumn):
    host-side compositions over Row results / embedded operand rows"""
    SW = 1 << 20

    def fresh(cols):
        p = Pair(track_existence=False)
        p.field("general")
        for c in cols:
            p.holder.set_bit("i", "general", 10, c)
        p.sync_pending()
        return p
    cols = lambda p, q: [int(c) for c in p.ex.execute("i", q)[0].columns()]
    p = fresh([0])
    assert cols(p, "Shift(Row(general=10), n=1)") == [1]
    assert cols(p, "Shift(Shift(Row(general=10), n=1), n=1)") == [2]
    p = fresh([65535])
    assert cols(p, "Shift(Row(general=10), n=1)") == [65536]
    p = fresh([1, SW - 1, SW + 1])
    assert cols(p, "Shift(Row(general=10), n=1)") == [2, SW, SW + 2]
    assert cols(p, "Shift(Row(general=10), n=2)") == [3, SW + 1, SW + 3]
    assert cols(p, "Shift(Shift(Row(general=10)))") == [1, SW - 1, SW + 1]
    p = fresh([SW - 2, SW - 1, SW, SW + 2])
    assert cols(p, "Shift(Row(general=10), n=1)") == [SW - 1, SW, SW + 1, SW + 3]
    assert cols(p, "Shift(Shift(Row(general=10), n=1), n=1)") == [SW, SW + 1, SW + 2, SW + 4]
    assert cols(p, "Intersect(Shift(Row(general=10), n=1), Row(general=10))") == [SW - 1, SW]
    p = fresh([1, SW, 2 * SW])
    for col, exp in ((1, True), (2, False), (SW, True), (SW + 1, False), (2 * SW, True), (2 * SW + 1, False)):
        assert p.ex.execute("i", f"IncludesColumn(Row(general=10), column={col})")[0] is exp
    with pytest.raises(X.QueryError, match="must specify a column"):
        p.ex.execute("i", "IncludesColumn(Row(general=10))")
    with pytest.raises(X.QueryError, match="must specify a row query"):
        p.ex.execute("i", "IncludesColumn(column=1)")


def test_all_with_limit_offset():
    """executor_test.go:4406-4485 TestExecutor_Execute_All (ColumnID): 105 existence bits spread over the ends of shards 0-2
    and one in shard 3; All() with every limit / offset window of the reference's table"""
    SW = 1 << 20
    n = 105
    cols = [i + SW - 2 for i in range(n // 2)] + [i + 2 * SW - n + 5 for i in range(n // 2, n - 1)] + [3 * SW + 2]
    p = Pair(track_existence=True)
    p.field("f")
    for c in cols:
        p.holder.set_bit("i", "f", 10, c)
    p.sync_pending()
    assert cols == sorted(cols)
    cases = [("All()", cols), ("All(limit=1)", cols[:1]), ("All(limit=4)", cols[:4]), ("All(limit=4, offset=4)", cols[4:8]),
             (f"All(limit=4, offset={n - 5})", cols[n - 5:n - 1]), (f"All(limit=1, offset={n - 2})", cols[n - 2:n - 1]),
             (f"All(limit=4, offset={n - 2})", cols[n - 2:]), (f"All(limit=4, offset={n + 1})", []), (f"All(limit=2, offset={n - 3})", cols[n - 3:n - 1]),
             (f"All(limit=2, offset={n - 5})", cols[n - 5:n - 3]), ("All(limit=2, offset=2)", cols[2:4]), ("All(limit=1, offset=1)", cols[1:2]),
             (f"All(limit={n - 3}, offset=2)", cols[2:n - 1]), ("Limit(Row(f=10), limit=3, offset=50)", cols[50:53])]
    for q, exp in cases:
        got = p.ex.execute("i", q)[0]
        assert got.count == len(exp) and [int(c) for c in got.columns()] == exp, q


def test_min_max_row():
    """executor_test.go:2662-2712 TestExecutor_Execute_MinMaxRow (RowID) + filtered variants against brute force"""
    SW = 1 << 20
    p = Pair(track_existence=False)
    p.field("f")
    p.field("g")
    for col, row in ((0, 7000), (3, 50), (SW + 1, 10000), (1000, 1), (SW + 2, 5000)):
        p.holder.set_bit("i", "f", row, col)
    for col in (3, SW + 2, 5 * SW):
        p.holder.set_bit("i", "g", 0, col)
    p.sync_pending()
    assert p.ex.execute("i", "MinRow(field=f)")[0] == (1, 1)
    assert p.ex.execute("i", "MaxRow(field=f)")[0] == (10000, 1)
    assert p.ex.execute("i", "MinRow(Row(g=0), field=f)")[0] == (50, 1)          # rows meeting the filter: 50 (col 3), 5000 (col SW+2)
    assert p.ex.execute("i", "MaxRow(Row(g=0), field=f)")[0] == (5000, 1)
    assert p.ex.execute("i", "MinRow(Row(g=7), field=f)")[0] == (0, 0)
    for bad in ("MinRow(field=fake)", "MaxRow(field=fake)"):
        with pytest.raises(X.QueryError, match="field not found"):
            p.ex.execute("i", bad)
    with pytest.raises(X.QueryError, match="field required"):
        p.ex.execute("i", "MinRow()")


def test_groupby_kernel_pass_shapes():
    """GroupBy over shapes chosen for groupby_kernel's passes: 300 x 270 rows (two a-chunks, two b-chunks) of tiny array
    containers, a 40-element a-row, a bitmap a-row and a bitmap b-row (dense / warp passes), with and without a filter, either
    field order — the dense count tensor against the oracle's nested-loop restatement.  By default groupby_kernel only takes the
    units groupby_direct_kernel declines; FBGPU_GROUPBY_CTA=1 (tests/test_emu_kernels.py) sends it every unit."""
    from oracle import oracle as O
    SW = 1 << 20
    rng = np.random.default_rng(5)
    p = Pair(track_existence=False)
    for n in ("a", "b", "f"):
        p.field(n)
    for c in rng.choice(2 * SW, size=6000, replace=False).tolist():
        p.holder.set_bit("i", "a", int(rng.integers(0, 300)), c)
        p.holder.set_bit("i", "b", int(rng.integers(0, 270)), c)
        if c & 1:
            p.holder.set_bit("i", "f", 1, c)
    for c in range(70000, 79000):                                  # bitmap containers: a row 7 and b row 11, slot 1 of shard 0
        p.holder.set_bit("i", "a", 7, c)
        if c % 3:
            p.holder.set_bit("i", "b", 11, c)
    for c in range(SW + 5, SW + 45):                               # an a-row container of 40 elements
        p.holder.set_bit("i", "a", 299, c)
        p.holder.set_bit("i", "b", c % 270, c)
    p.sync_pending()
    rows = {"a": list(range(300)), "b": list(range(270))}
    for fields, filt in ((("a", "b"), None), (("a", "b"), "Row(f=1)"), (("b", "a"), None), (("b", "a"), "Row(f=1)")):
        call = pql.parse(filt)[0] if filt else None
        ids = [rows[f] for f in fields]
        exp = np.zeros(len(ids[0]) * len(ids[1]), dtype=np.uint64)
        for s in p.shards():
            O.groupby_shard([p.ora.frag(f, 0, s) for f in fields], s, ids, p.ora.eval_shard(call, s) if call is not None else None, exp)
        got = p.holder.ctx.groupby(p.idx.id, [p.idx.fields[f].id for f in fields], [X.VIEW_STANDARD] * 2, ids, p.shards(),
                                   filter_ops=p.ex._bitmap_call(p.idx, call) if call is not None else None)
        assert np.array_equal(np.asarray(got).reshape(-1), exp), (fields, filt)
        assert int(exp.sum()) > 3000


def test_groupby_direct_kernel_shapes():
    """groupby_direct_kernel (byte table indexed by column, one CTA per (shard, slot)): more than 256 a-rows (the host launches it per
    chunk of 256) and more than 256 b-rows (every b-row is vetted before anything is counted), run containers on both sides, columns
    that sit in two a-rows (side list), a b-row whose container is a bitmap (that unit goes to groupby_kernel), a shard that lacks one
    fragment, a filter — the dense count tensor against the oracle's nested loop"""
    from oracle import oracle as O
    from featurebase_b200 import roaring_io
    SW = 1 << 20
    rng = np.random.default_rng(23)
    p = Pair(track_existence=False)
    for n in ("a", "b", "f"):
        p.field(n)
    NA, NB = 300, 280
    for s in (0, 2, 5):
        cols = np.sort(rng.choice(SW, size=30000, replace=False)).astype(np.uint64)
        ra, rb = rng.integers(0, NA, size=len(cols)).astype(np.uint64), rng.integers(0, NB, size=len(cols)).astype(np.uint64)
        dup = rng.choice(len(cols), size=800, replace=False)                                      # 800 columns in two a-rows (~50 per slot: side list)
        a_bits = [ra * np.uint64(SW) + cols, ((ra[dup] + np.uint64(1)) % np.uint64(NA)) * np.uint64(SW) + cols[dup]]
        b_bits = [rb * np.uint64(SW) + cols]
        a_bits.append(np.uint64(17 * SW) + np.arange(70000, 70400, dtype=np.uint64))            # runs: 400 adjacent columns in a-row 17 / b-row 9
        b_bits.append(np.uint64(9 * SW) + np.arange(70100, 70700, dtype=np.uint64))
        a_bits.append(np.uint64(299 * SW) + np.arange(5 * 65536 + 10, 5 * 65536 + 20, dtype=np.uint64))
        if s == 0:
            b_bits.append(np.uint64(7 * SW) + np.uint64(3 * 65536) + rng.choice(65536, size=6000, replace=False).astype(np.uint64))   # bitmap container: (shard 0, slot 3)
        p.load("a", X.VIEW_STANDARD, s, roaring_io.encode(np.unique(np.concatenate(a_bits))))
        if s != 5:
            p.load("b", X.VIEW_STANDARD, s, roaring_io.encode(np.unique(np.concatenate(b_bits))))
        p.load("f", X.VIEW_STANDARD, s, roaring_io.encode(np.uint64(1 * SW) + np.unique(np.concatenate([cols[cols % np.uint64(5) != 0], np.arange(70000, 70350, dtype=np.uint64)]))))
    ids = [list(range(NA)), list(range(NB))]
    shards = [0, 2, 5, 6]
    for filt in (None, "Row(f=1)"):
        call = pql.parse(filt)[0] if filt else None
        exp = np.zeros(NA * NB, dtype=np.uint64)
        for s in (0, 2):
            O.groupby_shard([p.ora.frag(f, 0, s) for f in ("a", "b")], s, ids, p.ora.eval_shard(call, s) if call is not None else None, exp)
        before = p.holder.ctx.counters()
        got = p.holder.ctx.groupby(p.idx.id, [p.idx.fields["a"].id, p.idx.fields["b"].id], [X.VIEW_STANDARD] * 2, ids, shards,
                                   filter_ops=p.ex._bitmap_call(p.idx, call) if call is not None else None)
        assert np.array_equal(np.asarray(got).reshape(-1), exp), filt
        assert int(exp.sum()) > 40000 and int(exp.reshape(NA, NB)[17, 9]) >= (300 if filt is None else 200)
        after = p.holder.ctx.counters()
        if "groupby_fallback_units" in after and not os.environ.get("FBGPU_GROUPBY_CTA"):
            assert after["groupby_units"] - before["groupby_units"] == 2 * 16 * len(shards)            # two launches (256 + 44 a-rows) over 4 shards
            assert after["groupby_fallback_units"] - before["groupby_fallback_units"] == 2, (filt, before, after)   # (shard 0, slot 3), once per launch


def test_groupby_slot_groups():
    """groupby_direct_kernel on denser fields whose 3000 columns in two a-rows fill the side list: the two crowded (shard, slot) units
    overflow it and are declined before anything is counted (groupby_kernel takes them), a row subset, and a filter: the dense count
    tensor against the oracle's nested loop, and the fallback counter says what ran where"""
    from oracle import oracle as O
    SW = 1 << 20
    rng = np.random.default_rng(11)
    p = Pair(track_existence=False)
    for n in ("a", "b", "f"):
        p.field(n)
    cols = {0: rng.choice(SW, size=40000, replace=False), 1: np.concatenate([rng.choice(2 * 65536, size=24000, replace=False), 2 * 65536 + rng.choice(14 * 65536, size=16000, replace=False)]) + SW}
    frs = {"a": {}, "b": {}, "f": {}}
    for s, cc in cols.items():
        ra, rb = rng.integers(0, 64, size=len(cc)), rng.integers(0, 50, size=len(cc))
        rel = cc.astype(np.uint64) - np.uint64(s * SW)
        dup = rel[:3000]                                                     # 3000 columns sit in TWO a-rows: a probe must not stop at its first hit
        frs["a"][s] = np.sort(np.concatenate([ra.astype(np.uint64) * np.uint64(SW) + rel, ((ra[:3000] + 1) % 64).astype(np.uint64) * np.uint64(SW) + dup]))
        frs["b"][s] = np.sort(rb.astype(np.uint64) * np.uint64(SW) + rel)
        frs["f"][s] = np.sort(np.uint64(1 * SW) + rel[rel % np.uint64(3) != 0])
    from featurebase_b200 import roaring_io
    for f in frs:
        for s, bits in frs[f].items():
            p.load(f, X.VIEW_STANDARD, s, roaring_io.encode(bits))
    ids = [list(range(64)), list(range(0, 50, 2)) + [49, 77]]
    for filt in (None, "Row(f=1)"):
        call = pql.parse(filt)[0] if filt else None
        exp = np.zeros(len(ids[0]) * len(ids[1]), dtype=np.uint64)
        for s in p.shards():
            O.groupby_shard([p.ora.frag(f, 0, s) for f in ("a", "b")], s, ids, p.ora.eval_shard(call, s) if call is not None else None, exp)
        before = p.holder.ctx.counters()
        got = p.holder.ctx.groupby(p.idx.id, [p.idx.fields["a"].id, p.idx.fields["b"].id], [X.VIEW_STANDARD] * 2, ids, p.shards(),
                                   filter_ops=p.ex._bitmap_call(p.idx, call) if call is not None else None)
        assert np.array_equal(np.asarray(got).reshape(-1), exp), filt
        assert int(exp.sum()) > 20000
        after = p.holder.ctx.counters()
        if "groupby_fallback_units" in after and not os.environ.get("FBGPU_GROUPBY_CTA"):
            assert after["groupby_units"] - before["groupby_units"] == 32
            assert after["groupby_fallback_units"] - before["groupby_fallback_units"] == 2, (filt, before, after)   # (the crowded slots 0-1 of shard 1: their side lists overflow with or without the filter)


def test_topk_time_range():
    """executor_test.go:1811-1843 TestExecutor_Execute_TopK_Time: TopK over a time range counts a row's union over the covering
    views (column 0 is set on two days and counts once), plus a filter and k"""
    p = Pair()
    p.field("f", "time", quantum="YMD")
    p.field("g")
    for col, row, ts in ((0, 0, "2016-01-02T00:00"), (0, 1, "2016-01-02T00:00"), (0, 0, "2016-01-03T00:00"), (1, 0, "2016-01-10T00:00"),
                         (100000000, 2, "2016-02-02T00:00"), (200000000, 3, "2015-01-02T00:00")):
        p.holder.set_bit("i", "f", row, col, timestamp=ts)
    p.holder.set_bit("i", "g", 5, 1)
    p.holder.set_bit("i", "g", 5, 100000000)
    p.sync_pending()
    run = lambda q: p.ex.execute("i", q)[0]
    assert run("TopK(f, k=3, from=2016-01-01T00:00, to=2016-01-11T00:00)") == [(0, 2), (1, 1)]
    assert run("TopK(f, k=1, from=2016-01-01T00:00, to=2016-01-11T00:00)") == [(0, 2)]
    assert run("TopK(f, from=2016-01-01T00:00, to=2016-03-01T00:00)") == [(0, 2), (1, 1), (2, 1)]
    assert run("TopK(f, from=2016-01-01T00:00, to=2016-03-01T00:00, filter=Row(g=5))") == [(0, 1), (2, 1)]
    assert run("TopK(f, from=2017-01-01T00:00, to=2017-03-01T00:00)") == []
    assert run("TopK(f, k=3)") == [(0, 2), (1, 1), (2, 1)]                        # no range: the standard view


def _random_call(rng, depth):
    """a random bitmap call over the fields of test_random_call_trees_differential (PQL text)"""
    if depth == 0 or rng.random() < 0.3:
        r = rng.random()
        if r < 0.7:
            return f"Row(m={int(rng.integers(0, 9))})"             # rows 0..6 exist (array / bitmap / run / mixed), 7..8 do not
        if r < 0.8:
            return "All()"
        if r < 0.9:
            op = ["<", "<=", ">", ">=", "==", "!="][int(rng.integers(0, 6))]
            return f"Row(v {op} {int(rng.integers(-700, 700))})"
        lo = int(rng.integers(-700, 600))
        return f"Row(v >< [{lo}, {lo + int(rng.integers(0, 500))}])"
    kind = ["Intersect", "Union", "Difference", "Xor", "Not"][int(rng.integers(0, 5))]
    if kind == "Not":
        return f"Not({_random_call(rng, depth - 1)})"
    return f"{kind}({', '.join(_random_call(rng, depth - 1) for _ in range(int(rng.integers(1, 6))))})"


def test_random_call_trees_differential():
    """random call trees (n-ary set ops, Not, All, BSI comparisons as leaves; up to 4 levels) over rows of every encoding —
    sparse arrays, ~4000-element arrays at the array/bitmap boundary, bitmaps, short and long runs, a row mixing all three
    per slot — Row bytes and Count against the oracle on three shards"""
    import featurebase_b200.datagen as D
    from oracle import oracle as O
    rng = np.random.default_rng(int(os.environ.get("FBGPU_FUZZ_SEED", "2024")))
    p = Pair()
    p.field("m")
    p.field("v", "int", min=-600, max=600)
    for s in (0, 1, 4):
        parts = [D.fragment(9, s, [0], 0.004), D.fragment(9, s, [1], 0.0615), D.fragment(9, s, [2], 0.3), D.fragment(9, s, [3], 0.2, mode=1, mean_run=200.0),
                 D.fragment(9, s, [4], 0.9, mode=1, mean_run=5000.0), D.fragment(9, s, [5], 0.02, mode=1, mean_run=3.0)]
        merged = O.Bitmap()
        for d in parts:
            merged = merged.union(O.Bitmap.from_bytes(d))
        mixed = []                                                 # row 6: slot k takes its container from row k % 5
        for k in range(16):
            src = merged.row(k % 5, s)
            cols = roaring_values(src)
            cols = cols[(cols % (1 << 20)) // 65536 == k]
            mixed.append(np.uint64(6 << 20) + (cols % np.uint64(1 << 20)))
        merged = merged.union(O.Bitmap.from_values(np.concatenate(mixed)))
        p.load("m", X.VIEW_STANDARD, s, merged.to_bytes())
        p.load("v", X.VIEW_BSI, s, D.bsi_fragment(12, s, 300000, p.idx.fields["v"].bit_depth, -600, 600, base=0, null_frac=0.2))
        p.load(X.EXISTENCE_FIELD, X.VIEW_STANDARD, s, D.fragment(13, s, [0], 0.7))
    from tests.oracle_ctx import OracleCtx
    twin = OracleCtx()                                             # the same fragments, for the value-level entry points
    vf = p.idx.fields["v"]
    for s in (0, 1, 4):
        twin.load_fragment(p.idx.id, vf.id, X.VIEW_BSI, s, p.ora.frag("v", X.VIEW_BSI, s).to_bytes())
        twin.load_fragment(p.idx.id, p.idx.fields["m"].id, X.VIEW_STANDARD, s, p.ora.frag("m", X.VIEW_STANDARD, s).to_bytes())
        twin.load_fragment(p.idx.id, p.idx.fields[X.EXISTENCE_FIELD].id, X.VIEW_STANDARD, s, p.ora.frag(X.EXISTENCE_FIELD, X.VIEW_STANDARD, s).to_bytes())
    n_checked = 0
    for i in range(int(os.environ.get("FBGPU_FUZZ_TREES", "120"))):
        q = _random_call(rng, 3)
        try:
            if i % 2:
                p.check_row(q)
            else:
                p.check_count(f"Count({q})")
            n_checked += 1
            if i % 8 == 0:                                         # the row as a filter of the value-level entry points
                ops = p.ex._bitmap_call(p.idx, pql.parse(q)[0])
                args = (p.idx.id, vf.id, X.VIEW_BSI, vf.bit_depth, p.shards())
                got, exp = p.holder.ctx.extract(*args, filter_ops=ops), twin.extract(*args, filter_ops=ops)
                assert got[2] == exp[2] and np.array_equal(got[0], exp[0]) and np.array_equal(got[1], exp[1]), q
                assert p.holder.ctx.bsi_sum(*args, filter_ops=ops) == twin.bsi_sum(*args, filter_ops=ops), q
                for want_max in (False, True):
                    assert p.holder.ctx.bsi_minmax(*args, want_max, filter_ops=ops) == twin.bsi_minmax(*args, want_max, filter_ops=ops), q
        except X.QueryError as e:                                  # both sides refuse the same calls (empty Intersect(), > 15 operands deep)
            assert "not supported" in str(e) or "stack depth" in str(e), (q, e)
    assert n_checked > 80


def roaring_values(bm):
    from featurebase_b200 import roaring_io
    return np.asarray(roaring_io.decode(bm.to_bytes()), dtype=np.uint64)


def test_groupby_postprocessing_goldens():
    """executor_test.go:6087-6386: aggregate=Sum, previous / limit paging, wrapping iterators, rows spread over shards — the
    dense count tensor comes from the device, the rest is the mirror's host-side post-processing"""
    p = Pair()
    fields = {"general": V.GROUPBY_GENERAL, "sub": V.GROUPBY_SUB, **V.GB_FIELDS}
    for name, bits in fields.items():
        p.field(name)
        for r, c in bits:
            p.holder.set_bit("i", name, r, c)
    p.field("v", "int", min=0, max=1000)
    for c, val in V.GB_V_VALUES:
        p.holder.set_value("i", "v", c, val)
    p.sync_pending()
    fmt = lambda res: [(tuple(r for _, r in g[0]),) + tuple(g[1:]) for g in res]
    for q, exp in V.GB_CASES:
        assert fmt(p.ex.execute("i", q)[0]) == exp, q
    got = fmt(p.ex.execute("i", "GroupBy(Rows(ppa), Rows(ppb), Rows(ppc), limit=3)")[0])
    total = list(got)
    while len(total) < 64:
        a, b, c = got[-1][0]
        got = fmt(p.ex.execute("i", f"GroupBy(Rows(ppa, previous={a}), Rows(ppb, previous={b}), Rows(ppc, previous={c}), limit=3)")[0])
        assert got, "paging stalled"
        total += got
    assert total == V.GB_PAGING_EXPECT
    # having / sort / offset (executeGroupBy :3388-3421, applyLimitAndOffsetToGroupByResult :3441-3459)
    base = fmt(p.ex.execute("i", "GroupBy(Rows(general), Rows(sub))")[0])
    assert fmt(p.ex.execute("i", "GroupBy(Rows(general), Rows(sub), having=Condition(count > 1))")[0]) == [g for g in base if g[1] > 1]
    assert fmt(p.ex.execute("i", 'GroupBy(Rows(general), Rows(sub), sort="count asc")')[0]) == sorted(base, key=lambda g: g[1])
    assert fmt(p.ex.execute("i", 'GroupBy(Rows(general), Rows(sub), sort="count desc", limit=1)')[0]) == [base[0]]
    assert fmt(p.ex.execute("i", "GroupBy(Rows(general), Rows(sub), offset=1, limit=2)")[0]) == base[1:3]
    assert fmt(p.ex.execute("i", "GroupBy(Rows(general), Rows(sub), offset=9)")[0]) == base
    agg = fmt(p.ex.execute("i", 'GroupBy(Rows(general), Rows(sub), aggregate=Sum(field=v), having=Condition(sum > 50))')[0])
    assert agg == [((10, 100), 2, 110)]
    with pytest.raises(X.QueryError):
        p.ex.execute("i", 'GroupBy(Rows(general), sort="rowid")')
    # executor_test.go:5311-5341 TestExecutor_Execute_Rows (the `column=` form needs a column-literal operand: not mirrored)
    q = Pair()
    q.field("general")
    q.field("integer", "int", min=-1000, max=1000)
    for r, c in [(10, 0), (10, (1 << 20) + 1), (11, 2), (11, (1 << 20) + 2), (12, 2), (12, (1 << 20) + 2), (13, 3)]:
        q.holder.set_bit("i", "general", r, c)
    q.sync_pending()
    for query, exp in (("Rows(general)", [10, 11, 12, 13]), ("Rows(field=general)", [10, 11, 12, 13]), ("Rows(general, limit=2)", [10, 11]),
                       ("Rows(general, previous=10,limit=2)", [11, 12]), ("Rows(general, in=[11, 13, 99])", [11, 13])):
        assert q.ex.execute("i", query)[0] == exp, query
    for bad, msg in (("Rows(integer)", "int fields not supported"), ("GroupBy(Rows())", "missing field in Rows call"),
                     ("Rows(general, in=[1, 2], column=3)", "does not support other arguments")):
        with pytest.raises(X.QueryError, match=msg):
            q.ex.execute("i", bad)


def test_columns_entry_point():
    """fbgpu_columns: the row's ascending column ids straight from the device (Row.Columns row.go:471) with executeLimitCall's
    offset / limit window, against the decoded Row result and the oracle — rows of every encoding, windows that start and
    end inside containers, across containers and across shards, an empty row, a too-small buffer"""
    import featurebase_b200.datagen as D
    from featurebase_b200 import lib as L
    from featurebase_b200 import roaring_io
    from oracle import oracle as O
    p = Pair(track_existence=False)
    p.field("m")
    for s in (0, 2, 3):
        merged = O.Bitmap()
        for d in (D.fragment(9, s, [0], 0.004), D.fragment(9, s, [1], 0.3), D.fragment(9, s, [2], 0.2, mode=1, mean_run=200.0)):
            merged = merged.union(O.Bitmap.from_bytes(d))
        p.load("m", X.VIEW_STANDARD, s, merged.to_bytes())
    ctx = p.holder.ctx
    for q in ("Row(m=0)", "Row(m=1)", "Row(m=2)", "Union(Row(m=0), Row(m=2))", "Difference(Row(m=1), Row(m=2))", "Row(m=7)"):
        ops = p.ex._bitmap_call(p.idx, pql.parse(q)[0])
        want = np.asarray(roaring_io.decode(p.check_row(q).roaring), dtype=np.uint64)
        cols, total = ctx.columns(p.idx.id, ops, p.shards())
        assert total == len(want) and np.array_equal(cols, want), q
        n = len(want)
        for off, lim in ((0, 1), (0, 10), (5, 0), (n // 3, 1000), (max(n - 3, 0), 10), (n, 5), (n + 9, 5), (70000, 70000), (1, None)):
            cols, total = ctx.columns(p.idx.id, ops, p.shards(), offset=off, limit=lim)
            assert total == n and np.array_equal(cols, want[off:] if lim is None else want[off:off + lim]), (q, off, lim)
        cols, _ = ctx.columns(p.idx.id, ops, [3, 0])                       # shard list order does not matter, subsets do
        assert np.array_equal(cols, want[(want >> np.uint64(20) == 0) | (want >> np.uint64(20) == 3)])
    if isinstance(ctx, L.Context):                                         # the C ABI's too-small-buffer contract
        import ctypes as C
        ops = L.ops_array(p.ex._bitmap_call(p.idx, pql.parse("Row(m=1)")[0]))
        sh = np.asarray(p.shards(), dtype=np.uint64)
        n, tot, buf = C.c_uint64(0), C.c_uint64(0), np.empty(10, dtype=np.uint64)
        rc = ctx.L.fbgpu_columns(ctx.h, p.idx.id, ops, len(ops), sh.ctypes.data, len(sh), 0, -1, buf.ctypes.data, 10, C.byref(n), C.byref(tot))
        assert rc == L.E_NOSPACE and n.value == tot.value > 10
        rc = ctx.L.fbgpu_columns(ctx.h, p.idx.id, ops, len(ops), sh.ctypes.data, len(sh), 3, 10, buf.ctypes.data, 10, C.byref(n), None)
        assert rc == 0 and n.value == 10


def test_extract_entry_point():
    """fbgpu_extract: an int field's values for the columns of filter ∩ not-null, gathered from the bit planes on the device
    (the bulk fragment.value, fragment.go:585-617).  Planes of every encoding: uniform values (bitmap / array planes), a
    contiguous block of equal values (run planes), negative values, a Base other than zero, nulls, windows, an empty filter."""
    import featurebase_b200.datagen as D
    SW = 1 << 20
    p = Pair()
    p.field("u", "int", min=-40000, max=40000)
    p.field("w", "int", min=1000, max=9000)                        # Base 1000
    p.field("g")
    depth = p.idx.fields["u"].bit_depth
    want_u, want_w = {}, {}
    for s in (0, 2):
        p.load("u", X.VIEW_BSI, s, D.bsi_fragment(21, s, 200000, depth, -40000, 40000, base=0, null_frac=0.3))
        for col in range(200000):
            v = D.bsi_value(21, s, col, -40000, 40000, null_frac=0.3)
            if v is not None:
                want_u[s * SW + col] = v
    for col in range(3 * SW + 100, 3 * SW + 9000):                 # run planes: a block of equal values, then a ramp
        want_w[col] = 4097 if col < 3 * SW + 5000 else 1000 + (col % 8000)
        p.holder.set_value("i", "w", col, want_w[col])
    p.field("z", "int", min=-200000, max=200000)                   # array planes: scattered columns, small values, a few large ones
    want_z = {}
    for k, col in enumerate(np.random.default_rng(8).choice(2 * SW, size=20000, replace=False).tolist()):
        want_z[col] = (70000 + k % 1000) * (-1 if k % 100 == 0 else 1) if k % 50 == 0 else k % 6
        p.holder.set_value("i", "z", col, want_z[col])
    for col in list(want_u)[::7] + list(want_w)[::3] + list(want_z)[::2]:
        p.holder.set_bit("i", "g", 1, col)
    p.sync_pending()
    ctx, idx = p.holder.ctx, p.idx
    g_cols = {int(c) for c in p.ex.execute("i", "Row(g=1)")[0].columns()}
    for name, want in (("u", want_u), ("w", want_w), ("z", want_z)):
        f = idx.fields[name]
        keys = np.array(sorted(want), dtype=np.uint64)
        cols, vals, total = ctx.extract(idx.id, f.id, X.VIEW_BSI, f.bit_depth, p.shards())
        assert total == len(keys) and np.array_equal(cols, keys)
        assert np.array_equal(vals + f.base, np.array([want[int(c)] for c in keys], dtype=np.int64)), name
        filt = p.ex._bitmap_call(idx, pql.parse("Row(g=1)")[0])
        fk = np.array([c for c in keys.tolist() if c in g_cols], dtype=np.uint64)
        cols, vals, total = ctx.extract(idx.id, f.id, X.VIEW_BSI, f.bit_depth, p.shards(), filter_ops=filt)
        assert total == len(fk) and np.array_equal(cols, fk) and np.array_equal(vals + f.base, np.array([want[int(c)] for c in fk], dtype=np.int64)), name
        for off, lim in ((0, 5), (len(fk) // 2, 4000), (len(fk) - 2, 10), (len(fk) + 3, 4)):
            cols, vals, total = ctx.extract(idx.id, f.id, X.VIEW_BSI, f.bit_depth, p.shards(), filter_ops=filt, offset=off, limit=lim)
            assert total == len(fk) and np.array_equal(cols, fk[off:off + lim]) and np.array_equal(vals + f.base, np.array([want[int(c)] for c in fk[off:off + lim]], dtype=np.int64))
        cols, vals, total = ctx.extract(idx.id, f.id, X.VIEW_BSI, f.bit_depth, p.shards(), filter_ops=p.ex._bitmap_call(idx, pql.parse("Row(g=9)")[0]))
        assert total == 0 and len(cols) == 0 and len(vals) == 0
    # Sum / Min / Max cross-check: the aggregates composed from counts agree with the extracted values
    vc = p.ex.execute("i", "Sum(field=u)")[0]
    assert (vc.val, vc.count) == (sum(want_u.values()), len(want_u))
    assert p.ex.execute("i", "Min(field=w)")[0].val == min(want_w.values()) and p.ex.execute("i", "Max(field=u)")[0].val == max(want_u.values())


def test_extract_table_golden():
    """executor_test.go:4940-5182 TestExecutor_Execute_Extract without the key / decimal / timestamp columns (translation layers):
    set, mutex, time, int and bool cells for every existing column, incl. a column whose only bit was cleared"""
    SW = 1 << 20
    p = Pair()
    p.field("set")
    p.field("mutex", "mutex")
    p.field("time", "time", quantum="YMDH")
    p.field("bsint", "int", min=-100, max=100)
    p.field("bool", "bool")
    for row, col in ((0, 1), (0, 2), (3, 1), (4, 1), (4, 4 * SW)):
        p.holder.set_bit("i", "set", row, col)
    p.holder._pending.setdefault(("i", X.EXISTENCE_FIELD, X.VIEW_STANDARD, 1), set()).add(0)       # Set(SW, set=5) then Clear(): the column stays
    for row, col in ((0, 1), (0, 2), (4, 4 * SW)):
        p.holder.set_bit("i", "mutex", row, col)
    for col, row, ts in ((0, 1, "2016-01-01T00:00"), (1, 2, "2017-01-01T00:00"), (3, 3, "2018-01-01T00:00")):
        p.holder.set_bit("i", "time", row, col, timestamp=ts)
    for col, v in ((0, 1), (1, -1), (3, 2)):
        p.holder.set_value("i", "bsint", col, v)
    for col, v in ((0, True), (1, False), (3, True)):
        p.holder.set_bit("i", "bool", 1 if v else 0, col)
    p.sync_pending()
    got = p.ex.execute("i", "Extract(All(), Rows(set), Rows(mutex), Rows(time), Rows(bsint), Rows(bool))")[0]
    assert got["fields"] == [("set", "[]uint64"), ("mutex", "uint64"), ("time", "[]uint64"), ("bsint", "int64"), ("bool", "bool")]
    assert got["columns"] == [
        (0, [[], None, [1], 1, True]),
        (1, [[0, 3, 4], 0, [2], -1, False]),
        (2, [[0], 0, [], None, None]),
        (3, [[], None, [3], 2, True]),
        (SW, [[], None, [], None, None]),
        (4 * SW, [[4], 4, [], None, None]),
    ]
    assert p.ex.execute("i", "Extract(Limit(All(), limit=2, offset=1), Rows(set), Rows(bsint))")[0]["columns"] == [(1, [[0, 3, 4], -1]), (2, [[0], None])]
    assert p.ex.execute("i", "Extract(Row(set=4), Rows(mutex))")[0]["columns"] == [(1, [0]), (4 * SW, [4])]
    assert p.ex.execute("i", "Extract(Row(set=9), Rows(mutex))")[0]["columns"] == []
    with pytest.raises(X.QueryError, match="missing column filter"):
        p.ex.execute("i", "Extract()")


def test_sort_goldens():
    """executor_test.go:4298-4390 TestExecutor_Sort (the key-translated mutex replaced by an id mutex): Sort by an int / bool /
    mutex field with limit, offset and sort-desc, alone and as Extract's column source"""
    p = Pair()
    p.field("bsint", "int")
    p.field("bool", "bool")
    p.field("mutex", "mutex")
    for col, v in enumerate((1, -1, 2, -2, 3, 4)):
        p.holder.set_value("i", "bsint", col, v)
    for col, v in enumerate((True, False, False, True, False, True)):
        p.holder.set_bit("i", "bool", 1 if v else 0, col)
    for col, r in enumerate((8, 26, 18, 16, 23, 9)):              # "h", "xyzzy", "ra", "plugh", "wl", "ig" by first letter
        p.holder.set_bit("i", "mutex", r, col)
    p.sync_pending()
    run = lambda q: p.ex.execute("i", q)[0]
    assert run("Extract(Sort(Row(bsint > 1), field = bsint, limit = 2, offset = 1), Rows(bsint))") == {"fields": [("bsint", "int64")], "columns": [(4, [3]), (5, [4])]}
    assert run("Extract(Sort(Row(bsint < -1), field = bool, limit = 1, sort-desc = true), Rows(bool))") == {"fields": [("bool", "bool")], "columns": [(3, [True])]}
    assert run("Extract(Sort(All(), field = mutex, limit = 1), Rows(mutex))") == {"fields": [("mutex", "uint64")], "columns": [(0, [8])]}
    assert run("Sort(All(), field=bsint)") == [(3, -2), (1, -1), (0, 1), (2, 2), (4, 3), (5, 4)]
    assert run("Sort(All(), field=bsint, sort-desc=true, limit=3)") == [(5, 4), (4, 3), (2, 2)]
    assert run("Sort(All(), field=bool)") == [(1, False), (2, False), (4, False), (0, True), (3, True), (5, True)]
    assert run("Sort(Row(bsint > 0), field=mutex, sort-desc=true)") == [(4, 23), (2, 18), (5, 9), (0, 8)]
    with pytest.raises(X.QueryError, match="not implemented"):
        p.ex.execute("i", "Sort(All(), field=_exists)")


def test_field_value_and_options():
    """executor_test.go:4066-4123 FieldValue (int cases) and :820-830 Options(shards=)"""
    SW = 1 << 20
    p = Pair()
    p.field("f", "int", min=-1100, max=1000)
    p.field("s")
    for col, v in ((1, 3), (2, -4), (SW + 1, 3)):
        p.holder.set_value("i", "f", col, v)
    for col in (100, SW, 2 * SW):
        p.holder.set_bit("i", "s", 10, col)
    p.sync_pending()
    run = lambda q: p.ex.execute("i", q)[0]
    for q, exp in (("FieldValue(field=f, column=1)", 3), ("FieldValue(field=f, column=2)", -4), (f"FieldValue(field=f, column={SW + 1})", 3)):
        vc = run(q)
        assert (vc.val, vc.count) == (exp, 1), q
    vc = run("FieldValue(field=f, column=7)")
    assert (vc.val, vc.count) == (0, 0)
    for q, msg in (("FieldValue()", "field required"), ("FieldValue(field=f)", "column required")):
        with pytest.raises(X.QueryError, match=msg):
            run(q)
    assert [int(c) for c in run("Options(Row(s=10), shards=[0, 2])").columns()] == [100, 2 * SW]
    assert run("Options(Count(Row(s=10)), shards=[1])") == 1
    assert [int(c) for c in run("Options(Row(s=10))").columns()] == [100, SW, 2 * SW]


def test_various_queries_goldens():
    """executor_test.go:8560-8990 populateTestData / variousQueries with the keys replaced by ids in order of first use (key
    translation is outside the path): Distinct on set and int fields, Count(Distinct), GroupBy over time-range rows, with
    filter / aggregate=Sum / aggregate=Count(Distinct) / having / sort / limit / offset.  The users are spread over three
    shards; userE is alone in the last one."""
    SW = 1 << 20
    U = dict(A=1, B=2, C=SW + 3, D=4, E=2 * SW + 5, F=6, G=SW + 7)
    p = Pair()
    p.field("likenums")
    for rid, u in [(1, "A"), (2, "B"), (3, "C"), (4, "D"), (5, "E"), (6, "F"), (7, "A"), (7, "B"), (7, "C"), (7, "D"), (7, "F")]:
        p.holder.set_bit("i", "likenums", rid, U[u])             # (row 7 leaves userE out, as upstream)
    p.field("likes")                                              # molecula 1, pilosa 2, pangolin 3, zebra 4, toucan 5, dog 6, icecream 7
    for rid, u in [(1, "A"), (2, "B"), (3, "C"), (4, "D"), (5, "E"), (6, "F")] + [(7, u) for u in "ABCDEF"]:
        p.holder.set_bit("i", "likes", rid, U[u])
    p.field("places", "time", quantum="YM")                       # nairobi 1, paris 2, austin 3, toronto 4, mombasa 5, sydney 6
    J19, A19, J20 = "2019-01-01T00:00", "2019-08-01T00:00", "2020-01-01T00:00"
    for rid, u, ts in [(1, "B", J19), (2, "C", J19), (3, "F", J19), (4, "A", J19), (4, "B", A19), (4, "C", A19), (4, "B", J20), (4, "D", J20),
                       (4, "E", J20), (4, "F", J20), (5, "A", J20), (6, "D", J20), (1, "E", J20)]:
        p.holder.set_bit("i", "places", rid, U[u], timestamp=ts)
    p.field("affinity", "int", min=-1000, max=1000)
    for u, v in dict(A=10, B=-10, C=5, D=-5, E=0).items():
        p.holder.set_value("i", "affinity", U[u], v)
    p.field("net_worth", "int", min=-100000000, max=100000000)
    for u, v in dict(A=1, B=10, C=100, D=1000, E=10000, F=100000).items():
        p.holder.set_value("i", "net_worth", U[u], v)
    p.field("zip_code", "int", min=0, max=100000)
    for u, v in dict(A=78739, B=78739, C=19707, D=19707, E=86753, G=78739).items():
        p.holder.set_value("i", "zip_code", U[u], v)
    p.sync_pending()
    run = lambda q: p.ex.execute("i", q)[0]
    gb = lambda q: [tuple(r for _, r in g[0]) + tuple(g[1:]) for g in run(q)]
    Y19, ALL = "from='2019-01-01T00:00', to='2019-12-31T23:59'", "from='2019-01-01T00:00', to='2020-12-31T23:59'"
    NOT_C = "filter=Not(Intersect(Row(likes=3), Row(likes=7)))"
    assert gb(f"GroupBy(Rows(places, {ALL}))") == [(1, 2), (2, 1), (3, 1), (4, 6), (5, 1), (6, 1)]
    assert gb("GroupBy(Rows(places, from='2019-01-01T00:00', to='2019-02-01T00:00'))") == [(1, 1), (2, 1), (3, 1), (4, 1)]
    assert gb(f"GroupBy(Rows(places, {Y19}))") == [(1, 1), (2, 1), (3, 1), (4, 3)]
    assert gb(f"GroupBy(Rows(places, {Y19}), {NOT_C})") == [(1, 1), (3, 1), (4, 2)]
    assert gb(f"GroupBy(Rows(places, {Y19}), {NOT_C}, aggregate=Sum(field=net_worth))") == [(1, 1, 10), (3, 1, 100000), (4, 2, 11)]
    assert run(f"Rows(places, {ALL})") == [1, 2, 3, 4, 5, 6]
    assert run(f"Rows(places, {Y19})") == [1, 2, 3, 4]
    assert run("Rows(places, from='2019-01-01T00:00', to='2019-02-01T00:00')") == [1, 2, 3, 4]
    assert run("Count(All())") == 7
    assert run("Count(Distinct(field=likenums))") == 7
    assert run("Distinct(field=likenums)") == [1, 2, 3, 4, 5, 6, 7]
    assert run("Count(Distinct(field=likes))") == 7
    d = run("Distinct(field=affinity)")
    assert (d.pos, d.neg, d.values()) == ([0, 5, 10], [5, 10], [-10, -5, 0, 5, 10])
    assert run("Count(Distinct(field=affinity))") == 5
    assert run("Distinct(Row(affinity>=0),field=affinity)") == X.SignedRow([0, 5, 10], [])
    assert run("Count(Distinct(Row(affinity>=0),field=affinity))") == 3
    assert run("Distinct(Row(affinity<0),field=likes)") == [2, 4, 7]
    assert run("Distinct(Row(affinity>0),field=likes)") == [1, 3, 7]
    assert run("Distinct(Row(likenums=1),field=likes)") == [1, 7]
    for q in ("Distinct(field=likes)", "Distinct(All(),field=likes)", "Distinct(field=likes )"):
        assert run(q) == [1, 2, 3, 4, 5, 6, 7], q
    assert gb("GroupBy(Rows(field=likes))") == [(1, 1), (2, 1), (3, 1), (4, 1), (5, 1), (6, 1), (7, 6)]
    assert gb("GroupBy(Rows(field=likes), aggregate=Sum(field=net_worth), limit=2, having=Condition(sum>10))") == [(3, 1, 100), (4, 1, 1000)]
    assert gb("GroupBy(Rows(field=likes), having=Condition(count>5))") == [(7, 6)]
    assert gb("GroupBy(Rows(field=likes), filter=Row(affinity>-7))") == [(1, 1), (3, 1), (4, 1), (5, 1), (7, 4)]
    CD = "aggregate=Count(Distinct(field=zip_code))"
    assert gb(f"GroupBy(Rows(field=likes), {CD})") == [(1, 1, 1), (2, 1, 1), (3, 1, 1), (4, 1, 1), (5, 1, 1), (6, 1, 0), (7, 6, 3)]
    assert gb(f"GroupBy(Rows(field=likes), {CD}, having=Condition(sum>2))") == [(7, 6, 3)]
    assert gb(f"GroupBy(Rows(field=likes), filter=Row(affinity>-11), {CD})") == [(1, 1, 1), (2, 1, 1), (3, 1, 1), (4, 1, 1), (5, 1, 1), (7, 5, 3)]
    assert gb("GroupBy(Rows(field=likes), filter=Row(affinity>-11), aggregate=Count(Distinct(Row(affinity>-7), field=zip_code)))") == \
        [(1, 1, 1), (2, 1, 0), (3, 1, 1), (4, 1, 1), (5, 1, 1), (7, 5, 3)]
    assert gb('GroupBy(Rows(field=likes), sort="count desc")') == [(7, 6), (1, 1), (2, 1), (3, 1), (4, 1), (5, 1), (6, 1)]
    SUM = 'aggregate=Sum(field=net_worth), sort="aggregate desc, count asc"'
    full = [(7, 6, 111111), (6, 1, 100000), (5, 1, 10000), (4, 1, 1000), (3, 1, 100), (2, 1, 10), (1, 1, 1)]
    assert gb(f"GroupBy(Rows(field=likes), {SUM})") == full
    assert gb(f"GroupBy(Rows(field=likes), {SUM}, limit=3)") == full[:3]
    assert gb(f"GroupBy(Rows(field=likes), {SUM},limit=3,offset=2)") == full[2:5]
    # groups of an int field are its values (executor_test.go:8980-8990), alone and next to a set field
    assert gb("GroupBy(Rows(field=affinity), aggregate=Count(Distinct(field=zip_code)))") == [(-10, 1, 1), (-5, 1, 1), (0, 1, 1), (5, 1, 1), (10, 1, 1)]
    assert gb("GroupBy(Rows(field=affinity))") == [(-10, 1), (-5, 1), (0, 1), (5, 1), (10, 1)]
    assert gb("GroupBy(Rows(field=zip_code), Rows(field=likes))") == [(19707, 3, 1), (19707, 4, 1), (19707, 7, 2), (78739, 1, 1), (78739, 2, 1), (78739, 7, 2), (86753, 5, 1), (86753, 7, 1)]
    assert gb("GroupBy(Rows(field=zip_code), aggregate=Sum(field=net_worth))") == [(19707, 2, 1100), (78739, 2, 11), (86753, 1, 10000)]
    # TestExecutor_Execute_Distinct / BareDistinct (executor_test.go:5945-5977, 7175-7207): a foreign-index join through Distinct(index=)
    h = p.holder
    par, ch = h.create_index("parent"), h.create_index("child")
    par.create_field("general")
    for row, cols in ((1, (1, 2, 3)), (2, (21, 22, 23)), (SW, (1, 21))):
        for c in cols:
            h.set_bit("parent", "general", row, c)
    ch.create_field("parent_id", "int", min=0, max=(1 << 28) - 1)
    ch.create_field("parent_set_id")
    ch.create_field("color")                                      # red 1, blue 2
    for col, parent, color in ((1, 1, 1), (2, 2, 2), (SW, 1, 2), (4, 21, 1)):
        h.set_value("child", "parent_id", col, parent)
        h.set_bit("child", "parent_set_id", parent, col)
        h.set_bit("child", "color", color, col)
    h.sync()
    ex = X.Executor(h)
    assert ex.execute("child", "Distinct(index=child, field=parent_id)")[0] == X.SignedRow([1, 2, 21], [])
    assert ex.execute("child", "Distinct(field=parent_set_id)")[0] == [1, 2, 21]
    assert ex.execute("child", "Distinct(Row(parent_id=3), field=parent_id)")[0] == X.SignedRow()
    for fld in ("parent_id", "parent_set_id"):
        got = ex.execute("parent", f"Intersect(Row(general={SW}), Distinct(Row(color=2), index=child, field={fld}))")[0]
        assert [int(c) for c in got.columns()] == [1], fld
    with pytest.raises(X.QueryError, match="missing field option"):
        ex.execute("child", "Distinct(Row(color=2))")


def test_distinct_random():
    """Distinct over int fields (zero, positive and negative Base; values on both sides of zero; with and without a filter) and
    set fields against a direct enumeration of the imported values"""
    SW = 1 << 20
    rng = np.random.default_rng(77)
    for lo, hi, n_vals in ((-300, 300, 40), (1000, 90000, 25), (-5000, -10, 30), (0, 1, 2), (-(1 << 40), 1 << 40, 12)):
        p = Pair()
        p.field("v", "int", min=lo, max=hi)
        p.field("s")
        pool = [int(x) for x in rng.integers(lo, hi, size=n_vals, endpoint=True)] + [lo, hi]
        cols = rng.choice(3 * SW, size=400, replace=False)
        vals = {}
        for c in cols.tolist():
            vals[c] = pool[int(rng.integers(len(pool)))]
            p.holder.set_value("i", "v", c, vals[c])
            p.holder.set_bit("i", "s", int(rng.integers(0, 9)) * 1000, c)
        for c in rng.choice(3 * SW, size=100, replace=False).tolist():           # columns without a value
            p.holder.set_bit("i", "s", 3, c)
        p.sync_pending()
        members = {}
        for r in [k * 1000 for k in range(9)] + [3]:
            members[r] = {int(c) for c in p.ex.execute("i", f"Row(s={r})")[0].columns()}
        def expect(keep):
            seen = {vals[c] for c in vals if keep(c)}
            return X.SignedRow([v for v in seen if v >= 0], [-v for v in seen if v < 0])
        assert p.ex.execute("i", "Distinct(field=v)")[0] == expect(lambda c: True), (lo, hi)
        assert p.ex.execute("i", "Count(Distinct(field=v))")[0] == expect(lambda c: True).count()
        for r in (0, 4000, 3):
            assert p.ex.execute("i", f"Distinct(Row(s={r}), field=v)")[0] == expect(lambda c: c in members[r]), (lo, hi, r)
        mid = (lo + hi) // 2
        assert p.ex.execute("i", f"Distinct(Row(v > {mid}), field=v)")[0] == expect(lambda c: vals[c] > mid), (lo, hi)
        assert p.ex.execute("i", f"Distinct(Row(v < {mid}), field=s)")[0] == sorted(r for r in members if any(c in vals and vals[c] < mid for c in members[r]))
        assert p.ex.execute("i", "Distinct(Row(s=12345), field=v)")[0] == X.SignedRow()


def test_bsi_aggregate_goldens():
    """executor_test.go:2192-2286 (Min/Max with offset bases), :2508-2567,2629-2655 (Min/Max with filters over 3 shards),
    :2782-2869 (Sum)"""
    for k, (lo, hi, val) in enumerate(V.EXEC_MINMAX_OFFSET):
        p = Pair()
        p.field(f"f{k}", "int", min=lo, max=hi)
        p.holder.set_value("i", f"f{k}", 10, val)
        p.sync_pending()
        for q in (f"Min(field=f{k})", f"Max(field=f{k})", f'Min(field="f{k}")', f"Max(f{k})", f"Sum(f{k})"):
            _check_agg(p, q, (val, 1))
    p = _setup(V.EXEC_MINMAX_SETUP)
    for q, exp in V.EXEC_MIN_CASES + V.EXEC_MAX_CASES:
        _check_agg(p, q, exp)
    p = _setup(V.EXEC_SUM_SETUP)
    for q, exp in V.EXEC_SUM_CASES:
        _check_agg(p, q, exp)
    with pytest.raises(X.QueryError, match="field not found"):
        p.ex.execute("i", "Sum(field=fake)")                      # executor_test.go:2871-2876
    with pytest.raises(X.QueryError):
        p.ex.execute("i", "Sum(Row(x=0), Row(x=1), field=foo)")
    with pytest.raises(X.QueryError):
        p.ex.execute("i", "Min()")


def test_bsi_aggregates_random():
    """signed / all-negative / all-positive / offset-base fields over several shards, filters of every density"""
    rng = np.random.default_rng(77)
    SW = 1 << 20
    for name, lo, hi, nvals in (("a", -5000, 5000, 6000), ("b", 100, 900, 3000), ("c", -900, -100, 3000), ("d", -3, 3, 500), ("e", -(1 << 40), 1 << 40, 2000)):
        p = Pair()
        p.field("x")
        p.field(name, "int", min=lo, max=hi)
        cols = rng.choice(4 * SW, nvals, replace=False)
        for c, v in zip(cols, rng.integers(lo, hi + 1, nvals)):
            p.holder.set_value("i", name, int(c), int(v))
        for r, frac in ((0, 0.5), (1, 0.02), (2, 0.0005)):
            for c in rng.choice(cols, max(1, int(nvals * frac)), replace=False):
                p.holder.set_bit("i", "x", r, int(c))
        p.holder.set_bit("i", "x", 3, 4 * SW + 5)                   # a filter row with no valued column
        p.sync_pending()
        for agg in ("Sum", "Min", "Max"):
            _check_agg(p, f"{agg}(field={name})")
            for r in range(4):
                _check_agg(p, f"{agg}(Row(x={r}), field={name})")
            _check_agg(p, f"{agg}(Union(Row(x=1), Row(x=2)), field={name})")
            _check_agg(p, f"{agg}(Row({name} > 0), field={name})")
            _check_agg(p, f"{agg}(Row({name} < 0), field={name})")
        assert _check_agg(p, f"Sum(Row(x=3), field={name})") == (0, 0)


# ---------------------------------------------------------------------------------------------------------------
# RBF loader (SURVEY §8 f1): fbgpu_load_rbf must leave the store in a state that answers every query exactly like the
# same fragments loaded through fbgpu_load_fragment (the reader itself is covered on the CPU by tests/test_rbf.py)
# ---------------------------------------------------------------------------------------------------------------
def test_rbf_loader_matches_fragment_loader():
    from featurebase_b200 import datagen as D
    from featurebase_b200 import roaring_io
    from oracle import oracle as O
    from tests import rbf_writer as W
    from tests import test_rbf as TR

    a, b = Pair(), Pair()                         # a: Pilosa-roaring path (+ oracle), b: RBF path
    for p in (a, b):
        p.field("f")
        p.field("g")
        p.field("v", "int", min=-2000, max=2000)
    rng = np.random.default_rng(8)
    shards = [0, 3, 4]
    for s in shards:
        per_view = {}
        for k, name in enumerate(("f", "g")):
            bm, _ = TR._fragment_containers(60 + k, s)
            per_view[(name, X.VIEW_STANDARD)] = bm.to_bytes()
        for col, val in zip(rng.choice(1 << 20, 4000, replace=False), rng.integers(-2000, 2001, 4000)):
            a.holder.set_value("i", "v", s * (1 << 20) + int(col), int(val))
        for (index, field, view, shard), bits in a.holder._pending.items():
            per_view[(field, view)] = roaring_io.encode(np.fromiter(bits, dtype=np.uint64, count=len(bits)))
        a.holder._pending = {}
        bitmaps = {}
        for (field, view), data in per_view.items():
            a.load(field, view, s, data)
            vname = "standard" if view == X.VIEW_STANDARD else "bsig_" + field
            bitmaps["~%s;%s<" % (field, vname)] = W.cells_from_pilosa(data)
        bitmaps["~other;standard<"] = [(0, "array", np.array([1], dtype=np.uint16))]          # a field this index does not know
        n = b.holder.import_rbf("i", s, W.build(bitmaps))
        assert n == len(per_view)
    sa, sb = a.holder.ctx.stats(), b.holder.ctx.stats()
    assert sa["fragments"] == sb["fragments"]
    assert sa["containers"] == sb["containers"]   # (RBF turns 4080..4095-element arrays into bitmaps: types may differ, counts not)
    for q in ("Count(Intersect(Row(f=0), Row(g=1)))", "Count(Union(Row(f=0), Row(f=3), Row(f=5), Row(f=6), Row(f=9), Row(g=40)))",
              "Count(Xor(Row(f=9), Row(g=9)))", "Count(Difference(Row(f=6), Row(g=5), Row(f=3)))", "Count(Not(Row(f=9)))",
              "Count(Row(v > 17))", "Count(Row(v >< [-100, 700]))", "Count(Row(v == null))"):
        assert b.ex.execute("i", q, shards)[0] == a.check_count(q, shards), q
    for q in ("Union(Row(f=0), Row(f=5), Row(f=9))", "Intersect(Row(f=3), Row(g=6))", "Row(v < -1500)"):
        ra = a.check_row(q, shards)
        rb = b.ex.execute("i", q, shards)[0]
        assert (rb.count, rb.roaring) == (ra.count, ra.roaring), q
    assert b.ex.execute("i", "TopK(f, k=20)", shards)[0] == a.ex.execute("i", "TopK(f, k=20)", shards)[0]
    assert b.ex.execute("i", "GroupBy(Rows(f), Rows(g))", shards)[0] == a.ex.execute("i", "GroupBy(Rows(f), Rows(g))", shards)[0]
    assert b.ex.execute("i", "Sum(field=v)", shards)[0] == a.ex.execute("i", "Sum(field=v)", shards)[0]
    with pytest.raises(Exception):
        b.holder.ctx.load_rbf(0, 9, TR.fixture("bad-bitmap"), ["x"], [1], [0])
    assert b.holder.ctx.load_rbf(0, 9, TR.fixture("bad-freelist"), ["x", "y"], [1, 2], [0, 0]) == 1
    assert b.holder.ctx.count(0, [X.L.Op(X.L.OP_ROW, 1, 0, 0, 0, 0, 0, 0)], [9]) == 1


def test_percentile_vs_reference_helper():
    """executor_test.go:7587-7760 variousQueriesOnPercentiles: 100 values of +-uint32 magnitude, half of them under the
    filter row; Percentile(nth) for the reference's nth list.  The reference checks against its own brute-force helper
    (getExpectedPercentile :7631-7678) on values drawn from math/rand seed 42, which cannot be reproduced here; on other
    data that helper and executePercentile differ in one corner (when the bisection runs out of range the executor returns
    its last midpoint, executor.go:1535-1585, the helper returns `min`), so the expectation below is executePercentile's
    control flow restated over a plain list, and the helper is only required to agree where the bisection converged."""
    def go_div(a, b):
        q = abs(a) // abs(b)
        return q if (a >= 0) == (b > 0) else -q

    def go_mod(a, b):
        return a - b * go_div(a, b)

    def expected(nums, nth):                                  # getExpectedPercentile :7631-7678
        mn, mx = min(nums), max(nums)
        less, greater = int(len(nums) * nth / 100.0), int(len(nums) * (100 - nth) / 100.0)
        if greater != 0 and less == 0:
            return mn, True
        if greater == 0:
            return mx, True
        guess = mn
        while mn < mx:
            guess = go_div(mx, 2) + go_div(mn, 2) + go_div(go_mod(mx, 2) + go_mod(mn, 2), 2)
            left, right = sum(1 for x in nums if x < guess), sum(1 for x in nums if x > guess)
            if left > less:
                mx = guess - 1
            elif right > greater:
                mn = guess + 1
            else:
                return guess, True
        return guess, False                                   # (the test helper would return mn here)

    rng = np.random.default_rng(42)
    SW = 1 << 20
    for trial in range(3):
        vals = [int(v) * (1 if rng.random() < 0.5 else -1) for v in rng.integers(0, 1 << 32, 100)]
        cols = [int(c) for c in rng.choice(3 * SW, 100, replace=False)]
        foo = [bool(rng.random() < 0.5) for _ in range(100)]
        p = Pair()
        p.field("val")
        p.field("net_worth", "int", min=min(vals), max=max(vals))
        for c, v, is_foo in zip(cols, vals, foo):
            p.holder.set_value("i", "net_worth", c, v)
            p.holder.set_bit("i", "val", 0 if is_foo else 1, c)
        p.sync_pending()
        nums = [v for v, is_foo in zip(vals, foo) if is_foo]
        for nth in (0, 10, 25, 50, 75, 90, 99, 100, 12.5, 99.9):
            q = f"Percentile(field=net_worth, filter=Row(val=0), nth={nth})"
            got = p.ex.execute("i", q)[0]
            exp, converged = expected(nums, float(nth))
            assert got.val == exp, (trial, nth)
            assert got.count >= 1
            if converged and 0 < nth < 100:                   # a balanced answer: as many smaller / larger values as asked for
                assert sum(1 for x in nums if x < got.val) <= int(len(nums) * nth / 100.0)
                assert sum(1 for x in nums if x > got.val) <= int(len(nums) * (100 - nth) / 100.0)
            got = p.ex.execute("i", f'Percentile(field="net_worth", nth={nth})')[0]
            assert got.val == expected(vals, float(nth))[0], (trial, nth, "no filter")
    assert p.ex.execute("i", "Percentile(field=net_worth, filter=Row(val=7), nth=50)")[0] is None
    for bad in ("Percentile(field=net_worth)", "Percentile(field=net_worth, nth=101)", "Percentile(nth=5)", "Percentile(field=nope, nth=5)"):
        with pytest.raises(X.QueryError):
            p.ex.execute("i", bad)


def test_arena_compaction():
    """fbgpu_compact: fragments are replaced and dropped (dead arena bytes grow), queries stay right before and after the live
    fragments are moved into a fresh arena, further loads land behind them, and the dead bytes are gone"""
    import featurebase_b200.datagen as D
    from oracle import oracle as O
    p = Pair(track_existence=False)
    p.field("m")
    p.field("n")
    ctx = p.holder.ctx

    def frag(seed, s):
        b = O.Bitmap()
        for d in (D.fragment(seed, s, [0, 1], 0.004), D.fragment(seed, s, [2], 0.3), D.fragment(seed, s, [3], 0.2, mode=1, mean_run=200.0)):
            b = b.union(O.Bitmap.from_bytes(d))
        return b.to_bytes()

    def check():
        for q in ("Intersect(Row(m=0), Row(n=1))", "Union(Row(m=2), Row(n=3), Row(m=1))", "Difference(Row(n=2), Row(m=3))", "Xor(Row(m=0), Row(m=3))"):
            p.check_row(q)
            p.check_count(f"Count({q})")
        assert p.ex.execute("i", "TopK(m, k=3)")[0] == sorted(((r, p.ora.count(pql.parse(f"Row(m={r})")[0], p.shards())) for r in range(4)), key=lambda kv: (-kv[1], kv[0]))[:3]

    for s in range(4):
        p.load("m", X.VIEW_STANDARD, s, frag(40, s))
        p.load("n", X.VIEW_STANDARD, s, frag(41, s))
    check()
    assert ctx.stats()["dead_bytes"] == 0
    for rnd in range(3):                                           # write batches: the same fragments re-sent with new content
        for s in (0, 2, 3):
            p.load("m", X.VIEW_STANDARD, s, frag(50 + rnd, s))
        p.load("n", X.VIEW_STANDARD, 1, frag(60 + rnd, 1))
    check()
    before = ctx.stats()
    assert before["dead_bytes"] > before["payload_bytes"]           # three generations of garbage behind the live data
    ctx.compact()
    after = ctx.stats()
    assert after["dead_bytes"] == 0 and after["payload_bytes"] == before["payload_bytes"] and after["containers"] == before["containers"]
    if hasattr(ctx, "L"):                                          # (the real library: the arena shrank)
        assert after["device_bytes"] < before["device_bytes"]
    check()
    p.load("m", X.VIEW_STANDARD, 5, frag(70, 5))                    # loads after a compaction append behind the moved data
    p.load("n", X.VIEW_STANDARD, 0, frag(71, 0))
    check()
    ctx.compact()
    ctx.compact()                                                  # nothing dead: a no-op
    check()


def test_incremental_container_refresh():
    """fbgpu_apply_containers on the device: a fragment's containers are replaced / added / removed one write batch after the other
    (bytes moved = the delta), queries are right after every batch, the commits are table patches, and fbgpu_compact gathers the
    live containers of the holed fragments one by one (arena_gather_kernel) without changing any result"""
    import featurebase_b200.datagen as D
    from oracle import oracle as O
    rng = np.random.default_rng(17)
    p = Pair(track_existence=False)
    p.field("m")
    p.field("n")
    ctx = p.holder.ctx

    def frag(seed, s):
        b = O.Bitmap()
        for d in (D.fragment(seed, s, [0, 1], 0.004), D.fragment(seed, s, [2], 0.3), D.fragment(seed, s, [3], 0.2, mode=1, mean_run=200.0)):
            b = b.union(O.Bitmap.from_bytes(d))
        return b.to_bytes()

    def check():
        for q in ("Intersect(Row(m=0), Row(n=1))", "Union(Row(m=2), Row(n=3), Row(m=1), Row(m=4))", "Difference(Row(n=2), Row(m=3))", "Xor(Row(m=0), Row(m=3))"):
            p.check_row(q)
            p.check_count(f"Count({q})")
        got = p.ex.execute("i", "TopK(m, k=4)")[0]
        assert got == sorted(((r, p.ora.count(pql.parse(f"Row(m={r})")[0], p.shards())) for r in range(6)), key=lambda kv: (-kv[1], kv[0]))[:4]

    for s in range(4):
        p.load("m", X.VIEW_STANDARD, s, frag(40, s))
        p.load("n", X.VIEW_STANDARD, s, frag(41, s))
    check()
    base = ctx.stats()
    for rnd in range(5):
        s = int(rng.integers(0, 4))
        keys = np.unique(p.ora.frag("m", X.VIEW_STANDARD, s).slice() >> np.uint64(16))
        written = sorted(set(int(k) for k in rng.choice(keys, size=3, replace=False)) | {16 * 4 + int(rng.integers(0, 16)), int(rng.integers(0, 64))})   # row 4 is new
        removed = sorted(set(int(k) for k in rng.choice(keys, size=2, replace=False)) - set(written))
        put = []
        for k in written:
            n = int(rng.choice([7, 300, 5000, 40000]))
            put.append((np.uint64(k) << np.uint64(16)) | np.sort(rng.choice(65536, size=n, replace=False)).astype(np.uint64))
        p.apply("m", X.VIEW_STANDARD, s, np.concatenate(put), removed)
        if rnd == 2:                                                # a batch for the other field and a removal-only batch in the same commit
            p.apply("n", X.VIEW_STANDARD, 1, (np.uint64(16 * 1 + 3) << np.uint64(16)) | np.arange(0, 60000, 3, dtype=np.uint64), [])
            p.apply("n", X.VIEW_STANDARD, 2, [], [int(np.unique(p.ora.frag("n", X.VIEW_STANDARD, 2).slice() >> np.uint64(16))[0])])
        check()
    st = ctx.stats()
    assert st["fragments"] == base["fragments"] and st["dead_bytes"] > 0
    if hasattr(ctx, "L"):                                          # (the real library) row 4 is new to the dense directory once; the rest are patches
        assert st["patch_commits"] - base["patch_commits"] >= 3, (base, st)
    ctx.compact()
    after = ctx.stats()
    assert after["dead_bytes"] == 0 and after["payload_bytes"] == st["payload_bytes"] and after["containers"] == st["containers"]
    check()
    p.apply("m", X.VIEW_STANDARD, 0, (np.uint64(5 * 16) << np.uint64(16)) | np.arange(100, dtype=np.uint64), [])      # updates after a compaction
    p.apply("m", X.VIEW_STANDARD, 9, (np.uint64(1 * 16 + 2) << np.uint64(16)) | np.arange(0, 65536, 2, dtype=np.uint64), [])   # a shard that was not resident
    check()
    with pytest.raises(L.FbgpuError):
        p.holder.apply_containers("i", "m", X.VIEW_STANDARD, 0, O.Bitmap.from_values(np.arange(10, dtype=np.uint64)).to_bytes(), [0])
    check()


def test_row_result_threaded_assembly():
    """a Row result above 8 MiB (72 shards of bitmap containers): fbgpu_row splits the payload copies into the caller's buffer over
    several host threads; the bytes must still be the canonical serialisation.  Also with two batches behind one header."""
    import featurebase_b200.datagen as D
    for env in (None, "640"):                            # 640 units = 40 shards per batch
        if env:
            os.environ["FBGPU_UNIT_BATCH"] = env
        try:
            p = Pair(track_existence=False)
            p.field("f")
            shards = list(range(72))
            bulk = D.fragments(5, np.asarray(shards, dtype=np.uint64), [0, 1], 0.5)
            for s in shards:
                p.load("f", X.VIEW_STANDARD, s, bulk.fragment_bytes(s))
            got = p.check_row("Row(f=0)")
            assert len(got.roaring) > (9 << 20)
            p.check_row("Intersect(Row(f=0), Row(f=1))")
        finally:
            os.environ.pop("FBGPU_UNIT_BATCH", None)

def test_topn_cutoff_goldens():
    """threshold= / tanimotoThreshold= through TopN on one shard: fragment_internal_test.go:1490-1537 and the MinThreshold rows of
    tests/golden/vectors.py; argument errors of executeTopNShard :2876,2893,2921"""
    for rows, src, n, ids, thr, tan, exp in V.FRAG_TOP_THRESHOLD_CASES:
        p = Pair(track_existence=False)
        p.field("f")
        p.field("src")
        for r, cols in rows.items():
            for c in cols:
                p.holder.set_bit("i", "f", r, c)
        for c in (src or []):
            p.holder.set_bit("i", "src", 0, c)
        p.sync_pending()
        q = ("TopN(f" + (", Row(src=0)" if src else "") + (f", n={n}" if n else "") + (", ids=[" + ",".join(map(str, ids)) + "]" if ids else "")
             + (f", threshold={thr}" if thr else "") + (f", tanimotoThreshold={tan}" if tan else "") + ")")
        assert p.ex.execute("i", q, [0])[0] == exp, q
    p.field("v", "int", min=0, max=100)
    for q, msg in (("TopN(f, Row(src=0), tanimotoThreshold=101)", "Tanimoto Threshold is from 1 to 100 only"),
                   ("TopN(f, Row(src=0), Row(src=0), n=1)", "TopN() can only have one input bitmap"),
                   ("TopN(v, n=1)", "cannot compute TopN() on integer, decimal, or timestamp field")):
        with pytest.raises(X.QueryError, match=msg.replace("(", r"\(").replace(")", r"\)")):
            p.ex.execute("i", q, [0])
    # explicit ids: n does not truncate (executeTopN :2802-2807, fragment.go:1325-1327)
    assert p.ex.execute("i", "TopN(f, n=1, ids=[100,101,102])", [0])[0] == [(100, 4), (102, 4), (101, 2)]
    assert p.ex.execute("i", "TopN(f, n=1, ids=[])", [0])[0] == [(100, 4)]                       # an empty id list is no id list


def test_topn_cutoffs_random():
    """several shards, random rows: the mirror's per-shard cut-offs == fragment.top per shard (oracle.fragment_top with the
    candidate ids) summed by Pairs.Add and sorted (executeTopNShards :2831-2866)"""
    from oracle import oracle as O
    rng = np.random.default_rng(77)
    SW = 1 << 20
    p = Pair(track_existence=False)
    p.field("f")
    p.field("src")
    shards = [0, 1, 3]
    for s in shards:
        for r in range(12):
            k = int(rng.integers(0, 60))
            for c in rng.choice(400, size=k, replace=False):
                p.holder.set_bit("i", "f", r, s * SW + int(c))
        for c in rng.choice(400, size=int(rng.integers(20, 200)), replace=False):
            p.holder.set_bit("i", "src", 0, s * SW + int(c))
    p.sync_pending()
    src_call = pql.parse("Row(src=0)")[0]
    for with_src in (False, True):
        for thr, tan in ((2, 0), (8, 0), (25, 0), (0, 1), (0, 10), (0, 35), (0, 100), (4, 20)):
            for ids in (None, [0, 3, 5, 7, 11, 40]):
                want = {}
                for s in shards:
                    fr = p.ora.frag("f", X.VIEW_STANDARD, s)
                    src = p.ora.eval_shard(src_call, s) if with_src else None
                    cand = ids if ids is not None else [int(r) for r in fr.rows()]
                    for r, k in O.fragment_top(fr, s, src=src, row_ids=cand, min_threshold=thr or 1, tanimoto_threshold=tan):
                        want[r] = want.get(r, 0) + k
                exp = sorted(want.items(), key=lambda kv: (-kv[1], kv[0]))
                q = ("TopN(f" + (", Row(src=0)" if with_src else "") + (", ids=[" + ",".join(map(str, ids)) + "]" if ids else "")
                     + (f", threshold={thr}" if thr else "") + (f", tanimotoThreshold={tan}" if tan else "") + ")")
                assert p.ex.execute("i", q, shards)[0] == exp, q


def test_row_counts_per_shard_entry_point():
    """fbgpu_row_counts_per_shard (row_count_kernel<true>): the [shard][row] matrix against per-shard oracle counts — rows of
    every encoding, a filter program, a shard without the fragment, a row id the field does not hold, a repeated shard; its
    column sums are what fbgpu_row_counts returns"""
    import featurebase_b200.datagen as D
    from oracle import oracle as O
    p = Pair(track_existence=False)
    p.field("m")
    p.field("flt")
    for s in (0, 2, 3):
        merged = O.Bitmap()
        for d in (D.fragment(9, s, [0], 0.004), D.fragment(9, s, [1], 0.3), D.fragment(9, s, [2], 0.2, mode=1, mean_run=200.0), D.fragment(9, s, [5], 0.02)):
            merged = merged.union(O.Bitmap.from_bytes(d))
        p.load("m", X.VIEW_STANDARD, s, merged.to_bytes())
        if s != 3:
            p.load("flt", X.VIEW_STANDARD, s, D.fragment(4, s, [0, 1], 0.1))
    ctx, mid = p.holder.ctx, p.idx.fields["m"].id
    ids, shards = [0, 1, 2, 5, 77], [3, 0, 1, 2, 0]
    filt_call = pql.parse("Union(Row(flt=0), Row(flt=1))")[0]
    for call in (None, filt_call):
        ops = p.ex._bitmap_call(p.idx, call) if call is not None else None
        got = ctx.row_counts_per_shard(p.idx.id, mid, X.VIEW_STANDARD, shards, ids, filter_ops=ops)
        assert got.shape == (len(shards), len(ids))
        for k, s in enumerate(shards):
            fr = p.ora.frag("m", X.VIEW_STANDARD, s)
            filt = p.ora.eval_shard(call, s) if call is not None else None
            for j, r in enumerate(ids):
                row = fr.row(r, s) if fr is not None else O.Bitmap()
                assert int(got[k, j]) == (row.count() if filt is None else row.intersection_count(filt)), (s, r, call is not None)
        uniq = [0, 2, 3]
        total = ctx.row_counts(p.idx.id, mid, X.VIEW_STANDARD, uniq, row_ids=ids, filter_ops=ops)
        assert [int(x) for x in total] == [int(x) for x in ctx.row_counts_per_shard(p.idx.id, mid, X.VIEW_STANDARD, uniq, ids, filter_ops=ops).sum(axis=0)]
    # the all-rows form never hands back a truncated list: buffers that are too small get FBGPU_E_NOSPACE and the number of rows
    # there are, and the binding calls again with that many entries
    full_ids, full_cnts = ctx.row_counts(p.idx.id, mid, X.VIEW_STANDARD, [0, 2, 3])
    assert sorted(int(r) for r in full_ids) == [0, 1, 2, 5]
    small_ids, small_cnts = ctx.row_counts(p.idx.id, mid, X.VIEW_STANDARD, [0, 2, 3], cap=1)
    assert list(small_ids) == list(full_ids) and list(small_cnts) == list(full_cnts)
    if hasattr(ctx, "L"):
        import ctypes as C
        sh = np.asarray([0, 2, 3], dtype=np.uint64)
        rid, out, n = np.full(2, 99, dtype=np.uint64), np.full(2, 99, dtype=np.uint64), C.c_int32(-1)
        rc = ctx.L.fbgpu_row_counts(ctx.h, p.idx.id, mid, X.VIEW_STANDARD, None, 0, None, 0, sh.ctypes.data, 3, rid.ctypes.data, out.ctypes.data, 2, C.byref(n))
        assert rc == L.E_NOSPACE and n.value == 4 and list(rid) == [99, 99] and list(out) == [99, 99]


def test_multi_batch_paths(monkeypatch):
    """FBGPU_UNIT_BATCH=16 (read when a context is created): one shard per launch, so the batch loops of fbgpu_row (payloads of
    several batches assembled behind one header), fbgpu_columns / fbgpu_extract (a window that starts in one batch and ends in
    another), fbgpu_bsi_sum / fbgpu_bsi_minmax (accumulators and the ValCount merge across batches) and the filtered
    fbgpu_row_counts / fbgpu_groupby passes run with a handful of shards instead of more than 1024"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    G.test_executor_goldens_and_edge_semantics()
    G.test_topk_topn_rowcounts()
    G.test_groupby_two_and_three_fields()
    test_columns_entry_point()
    test_extract_entry_point()
    test_bsi_aggregate_goldens()
    test_filter_sample_goldens()
    test_topn_cutoffs_random()
    test_row_counts_per_shard_entry_point()


def test_launch_and_query_counts(monkeypatch):
    """kernel_launches / queries of one call to each query entry point, one shard per batch (FBGPU_UNIT_BATCH=16): what
    bench.py's gpu_launches and the per-call counters report.  Then the two calls that answer an empty request after the device
    check without committing the pending load."""
    import ctypes as C
    import featurebase_b200.datagen as D
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    ctx = L.Context(0)
    shards = [0, 1, 2]
    for s in shards:
        ctx.load_fragment(0, 1, 0, s, D.fragment(1, s, [0, 1, 2, 3], 0.002))
        ctx.load_fragment(0, 1, 1, s, D.fragment(4, s, [0, 1, 2, 3], 0.002))          # a second (time) view of field 1
        ctx.load_fragment(0, 3, 0, s, D.fragment(3, s, [0, 1], 0.02))
        ctx.load_fragment(0, 2, 0, s, D.fragment(2, s, list(range(10)), 0.002))      # an int field of depth 8: exists, sign, 8 planes
    ctx.commit()
    row = lambda f, r: L.Op(L.OP_ROW, f, 0, 0, r, 0, 0, 0)
    inter = L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)
    union = [row(1, 0), row(1, 1), L.Op(L.OP_UNION, 0, 0, 2, 0, 0, 0, 0)]
    filt = [row(3, 0)]

    def delta(call):
        before = ctx.counters()
        call()
        after = ctx.counters()
        return after["kernel_launches"] - before["kernel_launches"], after["queries"] - before["queries"]
    calls = {
        "count": lambda: ctx.count(0, [row(1, 0), row(1, 1), inter], shards),
        "count_eval": lambda: ctx.count(0, union, shards),
        "any": lambda: ctx.any(0, union, shards),
        "row": lambda: ctx.row(0, union, shards),
        "columns": lambda: ctx.columns(0, union, shards),
        "extract": lambda: ctx.extract(0, 2, 0, 8, shards, filter_ops=filt),
        "bsi_sum": lambda: ctx.bsi_sum(0, 2, 0, 8, shards, filter_ops=filt),
        "bsi_minmax": lambda: ctx.bsi_minmax(0, 2, 0, 8, shards, True),
        "bsi_select": lambda: ctx.bsi_select(0, 2, 0, 8, shards, [0, 3]),
        "row_counts": lambda: ctx.row_counts(0, 1, 0, shards, row_ids=[0, 1, 2], filter_ops=filt),
        "count_pairs": lambda: ctx.count_pairs(0, 1, 0, [0, 1], 3, 0, [0, 1], shards),
        "groupby2": lambda: ctx.groupby(0, [1, 3], [0, 0], [[0, 1, 2], [0, 1]], shards),
        "groupby3": lambda: ctx.groupby(0, [1, 3, 1], [0, 0, 0], [[0, 1], [0, 1], [2, 3]], shards),
        "groupby_views": lambda: ctx.groupby_views(0, [1, 3], [[0, 1], [0]], [[0, 1, 2], [0, 1]], shards),
        "groupby_values": lambda: ctx.groupby_values(0, [1], [0], [[0, 1]], 2, 0, 8, [1, 5, 9], shards),
        "groupby_mixed": lambda: ctx.groupby_mixed(0, [(1, [0], [0, 1]), (3, [0], [0, 1])], [(2, 0, 8, [1, 5, 9])], shards),
        "groupby_sum": lambda: ctx.groupby_sum(0, [(1, [0], [0, 1])], [], (2, 0, 8), shards, filter_ops=filt),
        "groupby_distinct": lambda: ctx.groupby_distinct(0, [(3, [0], [0, 1])], [], (2, 0, 8, [1, 5, 9]), shards),
    }
    got = {name: delta(call) for name, call in calls.items()}
    # row / columns: eval + emit per batch; extract: + the value gather; bsi_sum / bsi_minmax: eval + plane kernel per batch;
    # bsi_select: eval per batch + (step, decide) per 4-bit digit of the 9-bit key; filtered row_counts: eval + count per batch;
    # GroupBy: groupby_direct_kernel + groupby_kernel for the units it declines (field 3's containers are too large for it),
    # behind a filter eval per batch for 3 fields, which run one 2-field pass per row of the first field; a multi-view first
    # dimension is peeled too, one filtered row count per row.  Int dimensions or an aggregate: eval + groupby_values_kernel per
    # batch, one query per row of every set dimension but the last; Count(Distinct) adds the popcount
    assert got == {"count": (1, 1), "count_eval": (1, 1), "any": (1, 1), "row": (6, 1), "columns": (6, 1), "extract": (9, 1),
                   "bsi_sum": (6, 1), "bsi_minmax": (6, 1), "bsi_select": (9, 1), "row_counts": (6, 1), "count_pairs": (1, 1),
                   "groupby2": (2, 1), "groupby3": (18, 2), "groupby_views": (18, 3), "groupby_values": (6, 1), "groupby_mixed": (12, 2),
                   "groupby_sum": (6, 1), "groupby_distinct": (7, 1)}, got
    # a load that is not committed yet: an empty request is answered without committing it
    ctx.load_fragment(0, 1, 0, 5, D.fragment(1, 5, [0], 0.002))
    commits = lambda: ctx.stats()["full_commits"] + ctx.stats()["patch_commits"]
    before, counters = commits(), ctx.counters()
    one = np.zeros(1, dtype=np.uint64)
    assert ctx.L.fbgpu_count_pairs(ctx.h, 0, 1, 0, one.ctypes.data, 1, 0, one.ctypes.data, 0, one.ctypes.data, 1, one.ctypes.data) == 0
    assert ctx.pair_types(0, 1, 0, 0, 1, 0, 1, []).sum() == 0
    assert commits() == before
    assert ctx.counters()["queries"] == counters["queries"] and ctx.counters()["kernel_launches"] == counters["kernel_launches"]
    ctx.close()
