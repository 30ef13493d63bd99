"""fbgpu_topn_cutoffs (TopN with threshold= / tanimotoThreshold= in one device call) and the TopN path built on it.

Entry-point tests compare the call with oracle.fragment_top run per shard over the same fragments, held by an oracle-backed
context, and summed as Pairs.Add sums the shards.  Hand-built worlds put each Tanimoto comparison on its boundary.  Query-level
tests compare the executor's TopN on the device with the composition it replaced (per-shard count matrices cut on the host),
which contexts without the call still run, and with a node.  The CPU tests check the argument errors on a context without a
device and run this file's gpu tests on the interpreted kernels."""
import ctypes as C
import os

import numpy as np
import pytest

from featurebase_b200 import executor as X
from featurebase_b200 import lib as L
from oracle import oracle as O
from tests import archetypes as A
from tests.oracle_ctx import OracleCtx
from tests.test_groupby_mixed import load_values

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR"))
SW, W = 1 << 20, 1 << 16
IDX, VV = 0, 7
F, SRC, EX, V = 1, 2, 3, 5             # the TopN field, Src rows, an existence-like row for Not, an int field (BSI view VV)
V_DEPTH = 8
SLOTS = (0, 9)                         # every shard's columns lie in these two slots
ENCODINGS = (O.ARRAY, O.BITMAP, O.RUN)
THRESHOLDS = [0, 1, 2, 8, 1 << 40]
TANIMOTO = [1, 10, 35, 50, 99, 100]
gpu = pytest.mark.gpu


@pytest.fixture
def ctx():
    c = L.Context(0)
    yield c
    c.close()


def row_op(field, row):
    return L.Op(L.OP_ROW, field, 0, 0, row, 0, 0, 0)


def src_programs():
    """{name: Src program}: a plain row, a Union, a BSI range and a Not"""
    return {
        "row": [row_op(SRC, 0)],
        "union": [row_op(SRC, 0), row_op(SRC, 1), L.Op(L.OP_UNION, 0, 0, 2, 0, 0, 0, 0)],
        "range": [L.Op(L.OP_BSI_RANGE, V, VV, 0, V_DEPTH, L.CMP[">"], 100, 0)],
        "not": [row_op(SRC, 1), L.Op(L.OP_NOT, EX, 0, 1, 0, 0, 0, 0)],
    }


def _bits(rng, n):
    """n distinct in-slot columns: a random set or a contiguous block (many short or few long runs)"""
    n = min(n, W)
    if rng.random() < 0.3:
        start = int(rng.integers(0, W - n + 1))
        return np.arange(start, start + n)
    return np.sort(rng.choice(W, n, replace=False))


def build_world(ctxs, seed, n_rows, shards, no_src=(), no_field=()):
    """loads the same fragments into every context of `ctxs`.  Per shard and slot: Src rows 0 and 1 of SRC, a wide EX row, V's
    values, and n_rows rows of F of varied cardinality in a random encoding (arrays above 4096 elements, bitmaps of a few bits
    and run containers of many runs included), half of them drawn mostly from Src's row 0 so that the Tanimoto band and
    coefficient fall on both sides.  Shards in no_src hold no SRC / EX / V fragments, shards in no_field no F fragment."""
    rng = np.random.default_rng(seed)
    frags = {}
    vals = {}
    for s in shards:
        fb, sb, eb = O.Bitmap(), O.Bitmap(), O.Bitmap()
        for slot in SLOTS:
            src0 = _bits(rng, int(rng.choice([3, 40, 700, 5000])))
            sb.put(0 * 16 + slot, A.container_of(src0, O.ARRAY if len(src0) < 4096 else O.BITMAP))
            src1 = _bits(rng, int(rng.integers(1, 3000)))
            sb.put(1 * 16 + slot, A.container_of(src1, O.RUN))
            eb.put(0 * 16 + slot, A.container_of(np.arange(0, W, 2), O.BITMAP))
            for c in rng.choice(W, 300, replace=False):
                vals[s * SW + slot * W + int(c)] = int(rng.integers(0, 1 << V_DEPTH))
            for r in range(n_rows):
                if rng.random() < 0.15:
                    continue                                   # the row has no container in this slot
                if rng.random() < 0.5:                         # similar to Src row 0: most of it, and a few others
                    keep = src0[rng.random(len(src0)) < rng.uniform(0.5, 1.0)]
                    extra = _bits(rng, int(rng.integers(0, max(2, len(src0) // 4))))
                    cols = np.union1d(keep, extra)
                else:
                    cols = _bits(rng, int(rng.choice([1, 2, 5, 30, 300, 3000, 4500, 9000])))
                if len(cols):
                    fb.put(r * 16 + slot, A.container_of(cols, ENCODINGS[int(rng.integers(0, 3))]))
        frags[s] = (fb, sb, eb)
    for c in ctxs:
        for s, (fb, sb, eb) in frags.items():
            if s not in no_field:
                c.load_fragment(IDX, F, 0, s, fb.to_bytes(optimize=False))
            if s not in no_src:
                c.load_fragment(IDX, SRC, 0, s, sb.to_bytes(optimize=False))
                c.load_fragment(IDX, EX, 0, s, eb.to_bytes(optimize=False))
        load_values(c, V, {col: v for col, v in vals.items() if col // SW not in no_src}, V_DEPTH)
        c.commit()


def expect(oc, shards, cand, src_ops, thr, tan):
    """{row: total}: oracle.fragment_top per shard (candidates `cand`, or every row of the shard's fragment), summed"""
    want = {}
    for s in shards:
        fr = oc._frag(IDX, F, 0, s)
        if fr is None:
            continue
        src = oc._eval(IDX, src_ops, s) if src_ops else None
        c = sorted(set(cand)) if cand is not None else [int(r) for r in fr.rows()]
        if not c:
            continue
        for r, k in O.fragment_top(fr, s, src=src, row_ids=c, min_threshold=max(thr, 1), tanimoto_threshold=tan):
            want[r] = want.get(r, 0) + k
    return want


def ranked(want):
    return sorted(((r, k) for r, k in want.items() if k > 0), key=lambda p: (-p[1], p[0]))


def check_call(ctx, oc, shards, src_ops, thr, tan, ids=None, what=""):
    want = expect(oc, shards, ids, src_ops, thr, tan)
    if ids is None:
        rid, tot = ctx.topn_cutoffs(IDX, F, 0, shards, src_ops=src_ops, min_threshold=thr, tanimoto=tan)
        got = list(zip(rid.tolist(), tot.tolist()))
        assert got == ranked(want), what
    else:
        got = ctx.topn_cutoffs(IDX, F, 0, shards, row_ids=ids, src_ops=src_ops, min_threshold=thr, tanimoto=tan)
        assert got.tolist() == [want.get(int(i), 0) for i in ids], what
    return want


# ------------------------------------------------------------------ entry point
SHARDS = [0, 1, 2, 5]


@gpu
def test_against_fragment_top(ctx):
    """every threshold and Tanimoto level, without a Src and with each Src program, in both output forms; a real share of the
    rows is kept and a real share dropped in the Tanimoto runs"""
    oc = OracleCtx()
    n_rows = 12 if ON_EMU else 40
    build_world([ctx, oc], 11, n_rows, SHARDS)
    progs = src_programs()
    ids = [int(i) for i in np.random.default_rng(3).permutation(n_rows + 4)[: n_rows // 2]]
    kept = dropped = 0
    for name, src in [("none", None)] + list(progs.items() if not ON_EMU else list(progs.items())[:2]):
        for thr in THRESHOLDS:
            check_call(ctx, oc, SHARDS, src, thr, 0, what=(name, thr))
            check_call(ctx, oc, SHARDS, src, thr, 0, ids=ids, what=(name, thr, "ids"))
        for tan in TANIMOTO:
            want = check_call(ctx, oc, SHARDS, src, 0, tan, what=(name, tan))
            check_call(ctx, oc, SHARDS, src, 3, tan, ids=ids, what=(name, tan, "ids"))
            if src is not None:
                kept += sum(1 for k in want.values() if k > 0)
                dropped += n_rows - sum(1 for k in want.values() if k > 0)
    assert kept > 0 and dropped > 0, (kept, dropped)


@gpu
def test_one_query_and_its_launches(ctx):
    """one call is one library query: an evaluation of the Src plus the counting kernel per shard batch (one batch here), or
    the counting kernel alone without a Src"""
    oc = OracleCtx()
    build_world([ctx, oc], 12, 10, SHARDS)
    for name, src in src_programs().items():
        before = ctx.counters()
        check_call(ctx, oc, SHARDS, src, 0, 35, what=name)
        after = ctx.counters()
        assert after["queries"] - before["queries"] == 1, name
        assert after["kernel_launches"] - before["kernel_launches"] == 2, name
    before = ctx.counters()
    check_call(ctx, oc, SHARDS, None, 2, 0, what="no src")
    after = ctx.counters()
    assert (after["queries"] - before["queries"], after["kernel_launches"] - before["kernel_launches"]) == (1, 1)


def _edge_world(ctx):
    """shard 0: |Src| = 100 (columns 0..99), rows 1..4 with cnt 50, 200, 51 and 199; shard 1: |Src| = cnt = 100 and count = 75
    (row 5); shard 2: |Src| = 2 and row 6 = {1, 2}: count 1 over a denominator of 3"""
    def frag(rows):
        b = O.Bitmap()
        for r, cols in rows.items():
            b.put(r * 16, A.container_of(np.asarray(cols), O.ARRAY))
        return b.to_bytes(optimize=False)
    src = {0: range(100), 1: range(100), 2: [0, 1]}
    rows = {0: {1: range(50), 2: range(200), 3: range(51), 4: range(199)},
            1: {5: list(range(75)) + list(range(1000, 1025))},
            2: {6: [1, 2]}}
    for s in range(3):
        ctx.load_fragment(IDX, SRC, 0, s, frag({0: list(src[s])}))
        ctx.load_fragment(IDX, F, 0, s, frag({r: list(c) for r, c in rows[s].items()}))
    ctx.commit()


@gpu
def test_exact_edges(ctx):
    """each Tanimoto comparison on its boundary: the band's ends are exclusive, a coefficient of exactly 60.0 is dropped at t = 60
    and kept at 59, 100 / 3 rounds up to 34"""
    _edge_world(ctx)
    src = [row_op(SRC, 0)]
    ids = [1, 2, 3, 4, 5, 6]

    def totals(shard, tan):
        return ctx.topn_cutoffs(IDX, F, 0, [shard], row_ids=ids, src_ops=src, tanimoto=tan).tolist()
    # shard 0, t = 50: the band is (50, 200); row 3: 51 * 100 / 100 = 51 > 50; row 4: 100 * 100 / 199 = 50.25 -> 51 > 50
    assert totals(0, 50) == [0, 0, 51, 100, 0, 0]
    assert totals(1, 60) == [0] * 6
    assert totals(1, 59) == [0, 0, 0, 0, 75, 0]
    assert totals(2, 33) == [0] * 5 + [1]
    assert totals(2, 34) == [0] * 6
    # summed over the shards: t = 33 keeps row 5 (coefficient 60) and row 6 (34), and in shard 0 rows 3 and 4 (band (33, 303))
    # plus row 2 (cnt 200: 100 * 100 / 200 = 50) and row 1 (50 * 100 / 100 = 50)
    assert ctx.topn_cutoffs(IDX, F, 0, [0, 1, 2], row_ids=ids, src_ops=src, tanimoto=33).tolist() == [50, 100, 51, 100, 75, 1]


@gpu
def test_explicit_ids(ctx):
    """ids unsorted, repeated and absent from the field: each gets its own row's total"""
    oc = OracleCtx()
    build_world([ctx, oc], 13, 16, SHARDS)
    ids = [7, 3, 3, 1000, 0, 15, 7, 99]
    for src, thr, tan in ((None, 2, 0), ([row_op(SRC, 0)], 0, 20), ([row_op(SRC, 0)], 4, 0)):
        check_call(ctx, oc, SHARDS, src, thr, tan, ids=ids, what=(thr, tan))
    assert ctx.topn_cutoffs(IDX, F, 0, SHARDS, row_ids=[], src_ops=[row_op(SRC, 0)], tanimoto=10).tolist() == []


@gpu
def test_missing_fragments(ctx):
    """listed shards without the field's fragment, without the Src's fragments, or holding nothing at all"""
    oc = OracleCtx()
    shards = [0, 1, 2, 3, 4]
    build_world([ctx, oc], 14, 16, [0, 1, 2, 3], no_src=(1,), no_field=(2,))
    listed = shards + [7]
    for name, src in src_programs().items():
        for thr, tan in ((0, 10), (0, 50), (2, 0)):
            check_call(ctx, oc, listed, src, thr, tan, what=(name, thr, tan))
            check_call(ctx, oc, listed, src, thr, tan, ids=list(range(18)), what=(name, thr, tan, "ids"))
    assert ctx.topn_cutoffs(IDX, F, 0, [], src_ops=[row_op(SRC, 0)], tanimoto=10)[0].tolist() == []
    assert ctx.topn_cutoffs(IDX, 77, 0, shards, src_ops=[row_op(SRC, 0)], tanimoto=10)[0].tolist() == []     # no such field


def _raw(ctx, shards, cap, src_ops, tan):
    sh = np.asarray(shards, dtype=np.uint64)
    rid, cnt, n = np.zeros(max(cap, 1), dtype=np.uint64), np.zeros(max(cap, 1), dtype=np.uint64), C.c_int32(-1)
    arr = L.ops_array(src_ops)
    rc = ctx.L.fbgpu_topn_cutoffs(ctx.h, IDX, F, 0, None, 0, arr, len(src_ops), 0, tan, sh.ctypes.data, len(sh),
                                  rid.ctypes.data, cnt.ctypes.data, cap, C.byref(n))
    return rc, n.value, rid, cnt


@gpu
def test_all_rows_nospace_round_trip(ctx):
    """a cap too small writes nothing and reports how many rows there are; the retry returns the list"""
    oc = OracleCtx()
    build_world([ctx, oc], 15, 20, SHARDS)
    src = [row_op(SRC, 0)]
    want = ranked(expect(oc, SHARDS, None, src, 0, 10))
    assert len(want) > 2
    rc, n, rid, cnt = _raw(ctx, SHARDS, len(want) - 1, src, 10)
    assert rc == L.E_NOSPACE and n == len(want)
    assert not rid.any() and not cnt.any()
    rc, n, rid, cnt = _raw(ctx, SHARDS, n, src, 10)
    assert rc == 0 and list(zip(rid[:n].tolist(), cnt[:n].tolist())) == want


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: every shard is its own evaluation batch and counting launch"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    ctx = L.Context(0)
    try:
        oc = OracleCtx()
        build_world([ctx, oc], 16, 12, SHARDS)
        for name, src in src_programs().items():
            before = ctx.counters()["kernel_launches"]
            check_call(ctx, oc, SHARDS, src, 0, 35, what=name)
            assert ctx.counters()["kernel_launches"] - before == 2 * len(SHARDS), name
            check_call(ctx, oc, SHARDS, src, 2, 0, ids=list(range(14)), what=name)
    finally:
        ctx.close()


@gpu
def test_node_equals_the_context(ctx):
    """a node over the same device listed twice, shards spread over both slots, answers what the single context answers in both
    forms"""
    node = L.Node([0, 0], 2)
    try:
        oc = OracleCtx()
        shards = [0, 1, 2, 3, 5, 6]
        build_world([ctx, node, oc], 17, 16, shards)
        assert {node.owner(s) for s in shards} == {0, 1}
        ids = [9, 2, 2, 40, 0]
        for name, src in [("none", None)] + list(src_programs().items()):
            for thr, tan in ((2, 0), (0, 35), (0, 100)):
                a = ctx.topn_cutoffs(IDX, F, 0, shards, src_ops=src, min_threshold=thr, tanimoto=tan)
                b = node.topn_cutoffs(IDX, F, 0, shards, src_ops=src, min_threshold=thr, tanimoto=tan)
                assert a[0].tolist() == b[0].tolist() and a[1].tolist() == b[1].tolist(), (name, thr, tan)
                assert list(zip(a[0].tolist(), a[1].tolist())) == ranked(expect(oc, shards, None, src, thr, tan)), (name, thr, tan)
                a = ctx.topn_cutoffs(IDX, F, 0, shards, row_ids=ids, src_ops=src, min_threshold=thr, tanimoto=tan)
                b = node.topn_cutoffs(IDX, F, 0, shards, row_ids=ids, src_ops=src, min_threshold=thr, tanimoto=tan)
                assert a.tolist() == b.tolist(), (name, thr, tan)
    finally:
        node.close()


# ------------------------------------------------------------------ query level
class _Composition:
    """the device context without topn_cutoffs: the executor composes the cut-offs from per-shard count matrices"""

    def __init__(self, ctx):
        self._ctx = ctx

    def __getattr__(self, name):
        if name == "topn_cutoffs":
            raise AttributeError(name)
        return getattr(self._ctx, name)


QUERIES = [
    "TopN(f, Row(src=0), threshold=2)",
    "TopN(f, Row(src=0), threshold=9, n=3)",
    "TopN(f, threshold=4)",
    "TopN(f, Row(src=0), tanimotoThreshold=10)",
    "TopN(f, Row(src=0), tanimotoThreshold=50, n=2)",
    "TopN(f, Union(Row(src=0), Row(src=1)), tanimotoThreshold=35)",
    "TopN(f, Row(v > 20), tanimotoThreshold=20)",
    "TopN(f, Not(Row(src=1)), threshold=3)",
    "TopN(f, Row(src=0), ids=[5, 1, 3, 77], tanimotoThreshold=20)",
    "TopN(f, Row(src=0), ids=[0, 2, 4, 6, 8], threshold=3)",
]


def _holder(ctx, seed):
    h = X.Holder(ctx=ctx)
    idx = h.create_index("i")
    idx.create_field("f")
    idx.create_field("src")
    idx.create_field("v", "int", min=0, max=100)
    rng = np.random.default_rng(seed)
    for s in (0, 1, 2, 4):
        src = rng.choice(400, size=int(rng.integers(30, 200)), replace=False)
        for c in src:
            h.set_bit("i", "src", 0, s * SW + int(c))
        for c in rng.choice(400, size=60, replace=False):
            h.set_bit("i", "src", 1, s * SW + int(c))
            h.set_value("i", "v", s * SW + int(c), int(rng.integers(0, 101)))
        for r in range(12):
            base = src if r % 2 else rng.choice(400, size=int(rng.integers(0, 80)), replace=False)
            for c in base[rng.random(len(base)) < rng.uniform(0.4, 1.0)]:
                h.set_bit("i", "f", r, s * SW + int(c))
    h.sync()
    return h


@gpu
def test_executor_on_three_contexts():
    """TopN with threshold= and tanimotoThreshold= gives the same pairs through the call, through the composition on the same
    context, and on a node, where it used to raise NotImplementedError"""
    dev = _holder(L.Context(0), 21)
    node = _holder(L.Node([0, 0], 1), 21)
    try:
        ed, en = X.Executor(dev), X.Executor(node)
        ec = X.Executor(dev)
        ec.ctx = _Composition(dev.ctx)
        nonempty = 0
        for q in QUERIES:
            before = dev.ctx.counters()["queries"]
            got = ed.execute("i", q)[0]
            assert dev.ctx.counters()["queries"] - before == 1, q
            assert got == ec.execute("i", q)[0], q
            assert got == en.execute("i", q)[0], q
            nonempty += bool(got)
        assert nonempty >= len(QUERIES) - 2
    finally:
        dev.ctx.close()
        node.ctx.close()


@gpu
@pytest.mark.skipif(not ON_EMU and (__import__("torch").cuda.device_count() < 2), reason="needs two GPUs")
def test_two_ranks_all_reduce():
    """two ranks on two GPUs with a communicator: the explicit-ids form is all-reduced, so each rank returns the total over both
    ranks' shards"""
    if ON_EMU:
        pytest.skip("the interpreted library has no communicator")
    import threading
    oc = OracleCtx()
    ctxs = [L.Context(0), L.Context(1)]
    try:
        shards = [[0, 2], [1, 3]]
        for c, sh in zip(ctxs, shards):
            build_world([c], 18, 16, sh)
        build_world([oc], 18, 16, [0, 1, 2, 3])
        uid = ctxs[0].comm_unique_id()
        out, errs = [None, None], []

        def run(k, fn):
            try:
                out[k] = fn()
            except Exception as e:                      # a rank's failure is reported in the test's thread
                errs.append(e)
        ids = list(range(18))
        src = [row_op(SRC, 0)]
        want = expect(oc, [0, 1, 2, 3], ids, src, 0, 35)
        for fn in (lambda k: ctxs[k].comm_init(2, k, uid),
                   lambda k: ctxs[k].topn_cutoffs(IDX, F, 0, shards[k], row_ids=ids, src_ops=src, tanimoto=35)):
            threads = [threading.Thread(target=run, args=(k, lambda k=k: fn(k))) for k in range(2)]
            [t.start() for t in threads]
            [t.join() for t in threads]
            assert not errs, errs
        for k in range(2):
            assert out[k].tolist() == [want.get(i, 0) for i in ids], k
    finally:
        for c in ctxs:
            c.close()


# ------------------------------------------------------------------ CPU
ARG_ERRORS = [
    ({"tan": 101}, "tanimoto_threshold=101 > 100"),
    ({"tan": 1 << 31}, "tanimoto_threshold=2147483648 > 100"),
    ({"n_rows": -1}, "bad argument"),
    ({"n_src_ops": -1}, "bad argument"),
    ({"null": "src"}, "bad argument"),
    ({"null": "shards"}, "bad argument"),
    ({"null": "out"}, "bad argument"),
    ({"n_shards": -1}, "bad argument"),
]


def _raw_args(L_, h, n_rows=2, n_src_ops=1, tan=10, n_shards=1, null=None):
    ids = np.asarray([1, 2], dtype=np.uint64)
    sh = np.asarray([0], dtype=np.uint64)
    out = np.zeros(4, dtype=np.uint64)
    src = L.ops_array([row_op(SRC, 0)])
    n = C.c_int32(0)
    return L_.fbgpu_topn_cutoffs(h, IDX, F, 0, ids.ctypes.data, n_rows, None if null == "src" else src, n_src_ops, 0, tan,
                                 None if null == "shards" else sh.ctypes.data, n_shards, None, None if null == "out" else out.ctypes.data, 4, C.byref(n))


def test_argument_errors_before_the_device_check():
    """argument errors come before the device check, on a context and on a node"""
    ctx = L.Context(L.DEVICE_NONE)
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    try:
        for L_, h in ((ctx.L, ctx.h), (node.L, node.h)):
            for kw, msg in ARG_ERRORS:
                rc = _raw_args(L_, h, **kw)
                assert rc == L.E_INVALID and L_.fbgpu_last_error().decode() == msg, (kw, msg)
        for kw in ({}, {"tan": 100}, {"tan": 0, "n_src_ops": 0, "null": "src"}):
            rc = _raw_args(ctx.L, ctx.h, **kw)
            assert rc == L.E_CUDA and "no device" in ctx.L.fbgpu_last_error().decode(), kw
        with pytest.raises(L.FbgpuError) as e:
            ctx.topn_cutoffs(IDX, F, 0, [0], src_ops=[row_op(SRC, 0)], tanimoto=5)
        assert e.value.code == L.E_CUDA and "no device" in str(e.value)
    finally:
        ctx.close()
        node.close()


def test_topn_cutoffs_on_interpreted_kernels():
    from tests.test_emu_kernels import run_on_emulator
    run_on_emulator(["tests/test_topn_cutoffs.py"], timeout=3000)
