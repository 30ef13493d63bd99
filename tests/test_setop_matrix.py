"""The set-op kernels on containers of every encoding and on programs at the compiler's limits.

Count, Row, Columns and Any run every bitmap call through eval_kernel / eval_wordpar_kernel (pair_count_kernel for
Count(Intersect(Row, Row)) and fbgpu_count_pairs), then canon_emit_kernel / columns_emit_kernel.  roaring_io.encode() and
datagen optimize() every container, so tests built on them hand these kernels canonical shapes only.  Here the operands are
the container set of tests/test_encoding_matrix.py (every value set in all three encodings, non-canonical ones included:
arrays of up to 65,536 elements, run containers of up to 32,768 intervals, one-bit bitmaps, `full` in every encoding) and
every expectation is a numpy boolean mask over the 65,536 columns of each (shard, slot) unit.  Row results are checked
container by container against a small encoder of the canonical rule (run if runs <= 2048 and runs <= N / 2, else array if
N < 4096, else bitmap), never against the oracle library.

Branches only these shapes reach:
  - warp_icount_runs searching run lists of more than 2048 intervals in global memory; the kFull short cut of
    warp_intersection_count_generic for a full array / run; unstriped array x array above 4096 and its pad correction
    (test_binary_ops_on_every_encoding_pair);
  - pair_count_kernel's per-pair sums in shared memory (<= 256 pairs) and in global memory (test_count_pairs_256_and_257);
  - eval_kernel's per-chunk `has_runs` and row-op batches clipped at a 128-op chunk (test_nary_programs_across_chunks), the
    XOR scatter that must leave an array's padded tail alone, the 15-deep operand stack and the refusal of 16
    (test_stack_depth_limits);
  - wp_slice on sorted arrays of 4097..65,536 elements, run lists above 2048 and one-bit bitmaps, and both sides of the
    word-parallel selection rule (n_ops <= 256, depth <= 4; never for views holding bank-striped arrays), under
    FBGPU_FORCE_WORDPAR;
  - the encoding choice of fbgpu_row at each of its boundaries (test_canonical_emission_boundaries);
  - columns_emit_kernel windows on and inside unit edges, in one and in many evaluation batches (test_columns_windows*).

Every gpu test runs in both array payload orders: the default bank-striped one and FBGPU_ARRAY_SORTED=1.  On the
interpreted kernels (FBGPU_TEST_ON_EMULATOR) a sampled subset of pairs and trees runs; FBGPU_EMU_FULL_SIZE runs all."""
import functools
import os
import struct

import numpy as np
import pytest

from featurebase_b200 import lib as L
from oracle import oracle as O
from tests import archetypes as A
from tests.test_encoding_matrix import SHARDS, SLOTS, abs_cols, container_set, index_of, load, mask_of, masks

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR")) and not os.environ.get("FBGPU_EMU_FULL_SIZE")
SEED = int(os.environ.get("FBGPU_FUZZ_SEED", "2024"))
W = 1 << 16
IDX = 0
FA, FB = 1, 2          # pair fields: pair k of the container set is row 0 of unit (shard k // 16, slot k % 16)
SA, SB = 3, 4          # the same for arrays of 64..4096 elements only (stored bank-striped by default)
R = 5                  # row i = container i of the set, in shard 0 slot 5 and shard 1 slot 11
EM, FULL = 6, 7        # operands of the canonical-emission targets; FULL rows 0..2: `full` as array / bitmap / run
EX = 8                 # existence rows 0..2: one value set in each encoding
ANYF = 9               # row n: one column, in shard n - 1; row 1: columns in every shard
ENCODINGS = (O.ARRAY, O.BITMAP, O.RUN)
OPC = {"and": L.OP_INTERSECT, "or": L.OP_UNION, "andnot": L.OP_DIFFERENCE, "xor": L.OP_XOR}
BIN = {"and": np.logical_and, "or": np.logical_or, "andnot": lambda a, b: a & ~b, "xor": np.logical_xor}
gpu = pytest.mark.gpu


def row_op(field, row):
    return L.Op(L.OP_ROW, field, 0, 0, int(row), 0, 0, 0)


def nary(op, n):
    return L.Op(OPC[op], 0, 0, n, 0, 0, 0, 0)


# ------------------------------------------------------------------ expected results
def canonical(m):
    """(type, N, payload bytes) of the canonical container for the column mask m, None when empty (roaring.go:3412-3426)"""
    v = np.flatnonzero(m)
    n = len(v)
    if n == 0:
        return None
    brk = np.flatnonzero(np.diff(v) != 1)
    runs = len(brk) + 1
    if runs <= 2048 and runs <= n // 2:
        starts = np.concatenate([v[:1], v[brk + 1]])
        lasts = np.concatenate([v[brk], v[-1:]])
        return O.RUN, n, struct.pack("<H", runs) + np.stack([starts, lasts], axis=1).astype("<u2").tobytes()
    if n < 4096:
        return O.ARRAY, n, v.astype("<u2").tobytes()
    return O.BITMAP, n, np.packbits(m, bitorder="little").tobytes()


def parse_row(data):
    """[(key, type, N, payload)] of a Pilosa roaring result written without optimisation (cookie 12348)"""
    cookie, n = struct.unpack_from("<II", data, 0)
    assert cookie == 12348
    out, end = [], 8 + 16 * n
    for i in range(n):
        key, typ, n1 = struct.unpack_from("<QHH", data, 8 + 12 * i)
        off, = struct.unpack_from("<I", data, 8 + 12 * n + 4 * i)
        assert off == end, (i, off, end)
        size = 2 * (n1 + 1) if typ == O.ARRAY else 8192 if typ == O.BITMAP else 2 + 4 * struct.unpack_from("<H", data, off)[0]
        out.append((key, typ, n1 + 1, bytes(data[off: off + size])))
        end = off + size
    assert end == len(data), (end, len(data))
    return out


def expect_row(units):
    """[(key, type, N, payload)] for [(key, column mask)] in key order"""
    out = []
    for key, m in units:
        c = canonical(m)
        if c is not None:
            out.append((key,) + c)
    return out


def check_row(got_data, got_count, exp, what):
    got = parse_row(got_data)
    assert got_count == sum(e[2] for e in exp), what
    assert len(got) == len(exp), (what, len(got), len(exp))
    for g, e in zip(got, exp):
        assert g[:3] == e[:3], (what, "key/type/N", g[:3], e[:3])
        assert g[3] == e[3], (what, "payload", g[:3])


def r_units(m):
    """the two units of R / EM / EX (shard 0 slot 5, shard 1 slot 11) holding the same columns m"""
    return [(s * 16 + slot, m) for s, slot in zip(SHARDS, SLOTS)]


def check_r_program(ctx, ops, m, what, row=True, columns=True):
    """Count, Row and Columns of a program over R-like fields whose result is m in both units"""
    n = int(m.sum())
    assert ctx.count(IDX, ops, SHARDS) == 2 * n, what
    if row:
        data, cnt = ctx.row(IDX, ops, SHARDS)
        check_row(data, cnt, expect_row(r_units(m)), what)
    if columns:
        got, total = ctx.columns(IDX, ops, SHARDS)
        assert total == 2 * n and np.array_equal(got, abs_cols(np.flatnonzero(m)).astype(np.uint64)), what


# ------------------------------------------------------------------ operand sets
@functools.lru_cache(maxsize=None)
def striped_arrays():
    """[(name, values, ARRAY)]: the set's arrays the loader stripes (64..4096 elements) and a few more at the edges of that range
    and of pair_count_kernel's register-window path (768 elements)"""
    rng = np.random.default_rng(31)
    out = [(n, v, t) for n, v, t in container_set() if t == O.ARRAY and 64 <= len(v) <= 4096]
    out += [(f"striped{k}", np.sort(rng.choice(W, k, replace=False)), O.ARRAY) for k in (65, 767, 768, 769, 2049, 4089)]
    out.append(("block@61440", np.arange(W - 4096, W), O.ARRAY))
    return out


EMU_PAIR_PICKS = [("full", t) for t in ENCODINGS] + [("oddBitsSet", t) for t in ENCODINGS] + [
    ("random1", O.ARRAY), ("random1", O.BITMAP), ("random1025", O.ARRAY), ("random5000", O.ARRAY), ("random40000", O.RUN),
    ("block@4096", O.RUN), ("lastBitSet", O.RUN), ("random4097", O.BITMAP)]


class PairSet:
    """pairs[k] = (i, j): conts[i] as row 0 of field fa and conts[j] as row 0 of fb in unit (shard k // 16, slot k % 16)"""

    def __init__(self, fa, fb, conts, m, pairs):
        self.fa, self.fb, self.conts, self.m, self.pairs = fa, fb, conts, m, pairs
        self.shards = list(range((len(pairs) + 15) // 16))
        self.objs = [A.container_of(v, t) for _, v, t in conts]

    def load(self, ctx):
        for f, side in ((self.fa, 0), (self.fb, 1)):
            for s in self.shards:
                b = O.Bitmap()
                for k in range(16 * s, min(16 * s + 16, len(self.pairs))):
                    b.put(k % 16, self.objs[self.pairs[k][side]])
                ctx.load_fragment(IDX, f, 0, s, b.to_bytes(optimize=False))

    def operands(self, s):
        """[16, W] column masks of both sides in shard s (rows past the last pair empty)"""
        ks = range(16 * s, min(16 * s + 16, len(self.pairs)))
        a, b = np.zeros((16, W), dtype=bool), np.zeros((16, W), dtype=bool)
        a[: len(ks)] = self.m[[self.pairs[k][0] for k in ks]]
        b[: len(ks)] = self.m[[self.pairs[k][1] for k in ks]]
        return a, b

    def result(self, op, s):
        a, b = self.operands(s)
        return BIN[op](a, b)

    def program(self, op):
        return [row_op(self.fa, 0), row_op(self.fb, 0), nary(op, 2)]

    def type_hist(self):
        h = np.zeros((4, 4), dtype=np.int64)
        for i, j in self.pairs:
            h[self.conts[i][2], self.conts[j][2]] += 1
        h[0, 0] += 16 * len(self.shards) - len(self.pairs)
        return h


@functools.lru_cache(maxsize=None)
def pair_sets():
    cs = container_set()
    if ON_EMU:
        picks = [index_of(n, t) for n, t in EMU_PAIR_PICKS]
        main = [(i, j) for i in picks for j in picks]
        sa = striped_arrays()
        sp = [(i, j) for i in range(0, len(sa), 3) for j in range(1, len(sa), 4)]
    else:
        main = [(i, j) for i in range(len(cs)) for j in range(len(cs))]
        sa = striped_arrays()
        sp = [(i, j) for i in range(len(sa)) for j in range(len(sa))]
    return [PairSet(FA, FB, cs, masks(), main), PairSet(SA, SB, sa, np.stack([mask_of(v) for _, v, _ in sa]), sp)]


@functools.lru_cache(maxsize=None)
def expected_pair_results(which, op):
    """(per-shard counts, Row containers) of `op` over pair set `which`"""
    ps = pair_sets()[which]
    per, row = [], []
    for s in ps.shards:
        r = ps.result(op, s)
        per.append(int(r.sum()))
        row += expect_row([(s * 16 + slot, r[slot]) for slot in range(16)])
    return per, row


def expected_columns(ps, op, shards):
    """the column ids of `op` over a contiguous range of shards: unit u of the range starts at column (shards[0] << 20) + u * W"""
    assert list(shards) == list(range(shards[0], shards[0] + len(shards)))
    r = np.concatenate([ps.result(op, s) for s in shards])
    return np.flatnonzero(r.ravel()).astype(np.uint64) + (np.uint64(shards[0]) << np.uint64(20))


# ------------------------------------------------------------------ canonical-emission targets
def from_runs(lengths, rng, at_end):
    """sorted values made of runs of the given lengths separated by random gaps of 1..16 columns, starting at column 0 or
    ending at column 65,535"""
    gaps = rng.integers(1, 9, len(lengths))
    gaps[0] = 0
    starts = np.cumsum(gaps + np.concatenate([[0], lengths[:-1]]))
    v = np.concatenate([np.arange(s, s + n) for s, n in zip(starts, lengths)])
    assert v[-1] < W
    return v + (W - 1 - v[-1] if at_end else 0)


@functools.lru_cache(maxsize=None)
def emission_targets():
    """[(name, values, (N, runs))]: result containers at each boundary of the canonical encoding rule, with the N and run count
    each is built to have (runs None: scattered)"""
    rng = np.random.default_rng(17)
    t = [("N=1", np.array([40000]), (1, 1))]
    for n in (4095, 4096, 4097):
        t.append((f"N={n} scattered", np.sort(rng.choice(W, n, replace=False)), (n, None)))
    t.append(("N=65536", np.arange(W), (W, 1)))
    shapes = [((2, 1), [2]), ((3, 2), [2, 1]), ((4000, 2000), [2] * 2000), ((4000, 2001), [2] * 1999 + [1, 1]),
              ((4001, 2000), [2] * 1999 + [3]), ((4001, 2001), [2] * 1999 + [2, 1]), ((4095, 2048), [2] * 2047 + [1]),
              ((4096, 2048), [2] * 2048), ((4098, 2049), [2] * 2049), ((10000, 2048), [5] * 1808 + [4] * 240),
              ((10000, 2049), [5] * 1804 + [4] * 245), ((40000, 2049), [20] * 1069 + [19] * 980)]
    for k, ((n, runs), lens) in enumerate(shapes):
        t.append((f"N={n} runs={runs}", from_runs(np.array(lens), rng, k % 2 == 1), (n, runs)))
    return [(name, np.asarray(v, dtype=np.int64), claim) for name, v, claim in t]


# ------------------------------------------------------------------ the store
@functools.lru_cache(maxsize=None)
def existence_mask():
    return masks()[index_of("random40000", O.ARRAY)] | masks()[index_of("block@0", O.ARRAY)]


def load_world(ctx):
    for ps in pair_sets():
        ps.load(ctx)
    cs = container_set()
    load(ctx, R, 0, [(i, A.container_of(v, t)) for i, (_, v, t) in enumerate(cs)])
    rng = np.random.default_rng(5)
    rows = []
    for k, (_, v, _) in enumerate(emission_targets()):
        m = mask_of(v)
        rows += [(10 * k + e, A.container_of(v, t)) for e, t in enumerate(ENCODINGS)]
        split = np.zeros(W, dtype=bool)
        brk = np.concatenate([[0], np.flatnonzero(np.diff(v) != 1) + 1, [len(v)]])
        for r in range(0, len(brk) - 1, 2):
            split[v[brk[r]: brk[r + 1]]] = True
        if len(brk) == 2:                                     # one run: two overlapping halves
            split[:] = False
            split[v[: len(v) * 2 // 3]] = True
            p2 = mask_of(v[len(v) // 3:])
        else:
            p2 = m & ~split
        extra = mask_of(np.sort(rng.choice(W, 500, replace=False)))
        for e, part in ((3, m & split), (4, p2), (5, m ^ extra), (6, extra)):
            if part.any():                                    # (an empty part is an absent row)
                rows.append((10 * k + e, A.container_of(np.flatnonzero(part), ENCODINGS[(k + e) % 3])))
    load(ctx, EM, 0, rows)
    load(ctx, FULL, 0, [(e, A.container_of(np.arange(W), t)) for e, t in enumerate(ENCODINGS)])
    ex = np.flatnonzero(existence_mask())
    load(ctx, EX, 0, [(e, A.container_of(ex, t)) for e, t in enumerate(ENCODINGS)])
    for s in range(65):
        b = O.Bitmap()
        b.put(1 * 16 + s % 16, A.container_of(np.arange(s, W, 97), O.ARRAY))
        for n in (8, 9, 64, 65):
            if s == n - 1:
                b.put(n * 16 + 15, A.container_of(np.array([W - 1]), O.ARRAY))
        ctx.load_fragment(IDX, ANYF, 0, s, b.to_bytes(optimize=False))
    ctx.commit()


@pytest.fixture(scope="module", params=["striped", "sorted"])
def world(request):
    """a context holding every operand set; `sorted`: created under FBGPU_ARRAY_SORTED=1 (fixed per context)"""
    with pytest.MonkeyPatch.context() as mp:
        if request.param == "sorted":
            mp.setenv("FBGPU_ARRAY_SORTED", "1")
        else:
            mp.delenv("FBGPU_ARRAY_SORTED", raising=False)
        ctx = L.Context(0)
    try:
        load_world(ctx)
        yield ctx
    finally:
        ctx.close()


# ------------------------------------------------------------------ tests
@gpu
def test_binary_ops_on_every_encoding_pair(world, monkeypatch):
    """Intersect, Union, Difference and Xor of every ordered pair of the container set (and of the striped arrays): Count per
    shard (Intersect also in its eval_kernel form, and every op again under FBGPU_FORCE_WORDPAR), Row container by
    container, Columns; pair_count_kernel's launch and pair types for Intersect"""
    ctx = world
    for which, ps in enumerate(pair_sets()):
        for op in OPC:
            per, row = expected_pair_results(which, op)
            prog = ps.program(op)
            before = ctx.counters()["pair_kernel_queries"]
            total, got = ctx.count(IDX, prog, ps.shards, per_shard=True)
            assert (total, got.tolist()) == (sum(per), per), (which, op)
            if op == "and":
                assert ctx.counters()["pair_kernel_queries"] == before + 1
                assert np.array_equal(ctx.pair_types(IDX, ps.fa, 0, 0, ps.fb, 0, 0, ps.shards).astype(np.int64), ps.type_hist()), which
                tri = [row_op(ps.fa, 0), row_op(ps.fb, 0), row_op(ps.fa, 0), nary("and", 3)]       # same result through eval_kernel
                assert ctx.count(IDX, tri, ps.shards, per_shard=True)[1].tolist() == per, which
                assert ctx.counters()["pair_kernel_queries"] == before + 1
            data, cnt = ctx.row(IDX, prog, ps.shards)
            check_row(data, cnt, row, (which, op))
            for g in range(0, len(ps.shards), 32):                  # (a Union over every shard holds ~10^8 columns: 32 shards per call)
                sh = ps.shards[g: g + 32]
                cols, total = ctx.columns(IDX, prog, sh)
                assert total == sum(per[g: g + 32]) and np.array_equal(cols, expected_columns(ps, op, sh)), (which, op, g)
        with monkeypatch.context() as mp:
            mp.setenv("FBGPU_FORCE_WORDPAR", "1")
            for op in OPC:
                per, _ = expected_pair_results(which, op)
                prog = ps.program(op) if op != "and" else [row_op(ps.fa, 0), row_op(ps.fb, 0), row_op(ps.fa, 0), nary("and", 3)]
                assert ctx.count(IDX, prog, ps.shards, per_shard=True)[1].tolist() == per, (which, op, "wordpar")


@gpu
@pytest.mark.parametrize("n_pairs", [256, 257])
def test_count_pairs_256_and_257(world, n_pairs):
    """fbgpu_count_pairs with per-pair sums in shared memory (256 pairs) and in global memory (257), rows of every encoding"""
    ctx = world
    rng = np.random.default_rng(n_pairs)
    n = len(container_set())
    ra, rb = rng.integers(0, n, n_pairs), rng.integers(0, n, n_pairs)
    m = masks()
    exp = [2 * int((m[a] & m[b]).sum()) for a, b in zip(ra, rb)]
    assert ctx.count_pairs(IDX, R, 0, ra, R, 0, rb, SHARDS).tolist() == exp
    assert ctx.count_pairs(IDX, R, 0, ra, R, 0, rb, [1, 0, 7]).tolist() == exp          # a shard list that is not a range


def nary_operands(rng, op, k, runs_in):
    """k row ids of R for an n-ary `op`: run containers only in the 128-op chunks listed in runs_in (the row of operand j is
    op j + 1 of the compiled program), and one row listed twice"""
    cs = container_set()
    pool = [i for i in range(len(cs)) if op == "xor" or len(cs[i][1]) <= 5000]       # (Union / Difference of large sets is all or nothing)
    runs = [i for i in pool if cs[i][2] == O.RUN]
    other = [i for i in pool if cs[i][2] != O.RUN]
    chunk = lambda j: (j + 1) // 128
    rows = [int(rng.choice(pool if chunk(j) in runs_in else other)) for j in range(k)]
    for c in runs_in:                                        # at least one run container in each such chunk
        js = [j for j in range(k) if chunk(j) == c]
        rows[js[len(js) // 2]] = int(rng.choice(runs))
    if op == "andnot":
        rows[0] = index_of("full", O.RUN if 0 in runs_in else O.BITMAP)
    src = next(j for j in range(k - 1, 0, -1) if cs[rows[j]][2] != O.RUN)
    rows[1 if src > 1 else 2] = rows[src]                    # listed twice, in different chunks when k > 128
    return rows


def fold(op, ms):
    out = ms[0].copy()
    if op == "andnot":
        for m in ms[1:]:
            out &= ~m
        return out
    for m in ms[1:]:
        out = BIN[op](out, m)
    return out


@gpu
@pytest.mark.parametrize("k", [127, 128, 129, 300])
def test_nary_programs_across_chunks(world, k):
    """Union, Xor and Difference of k row operands (k + 1 compiled ops: 128 is one 128-op chunk): run containers in the first
    chunk only, or in the last chunk only, a row listed twice (Xor cancels it, Difference does not care)"""
    ctx = world
    rng = np.random.default_rng(SEED + k)
    last = k // 128
    layouts = [{0}] + ([{last}] if last else [])
    for op in ("or", "xor", "andnot"):
        for runs_in in layouts:
            rows = nary_operands(rng, op, k, runs_in)
            ops = [row_op(R, r) for r in rows] + [nary(op, k)]
            prog, depth = ctx.debug_compile(IDX, ops)
            assert (len(prog), depth) == (k + 1, 1), (op, k)
            chunks_with_runs = {j // 128 for j, (_, _, r) in enumerate(prog) if j and container_set()[r][2] == O.RUN}
            assert chunks_with_runs == runs_in, (op, k, chunks_with_runs)
            m = fold(op, [masks()[r] for r in rows])
            check_r_program(ctx, ops, m, (op, k, sorted(runs_in)), columns=not ON_EMU)


def nested(rng, d, ops_cycle=("or", "and", "xor", "andnot")):
    """a tree of compiled stack depth d: P1 = Union(a, b), Pd = op(Union(c, e), P(d-1))"""
    n = len(container_set())
    pick = lambda: ("row", int(rng.integers(n)))
    t = ("or", [pick(), pick()])
    for lvl in range(2, d + 1):
        t = (ops_cycle[lvl % len(ops_cycle)], [("or", [pick(), pick()]), t])
    return t


def tree_ops(t):
    if t[0] == "row":
        return [row_op(R, t[1])]
    if t[0] == "not":
        return tree_ops(t[2]) + [L.Op(L.OP_NOT, EX, 0, 1, t[1], 0, 0, 0)]
    return [o for kid in t[1] for o in tree_ops(kid)] + [nary(t[0], len(t[1]))]


def tree_eval(t):
    if t[0] == "row":
        return masks()[t[1]]
    if t[0] == "not":
        return existence_mask() & ~tree_eval(t[2])
    return fold(t[0], [tree_eval(kid) for kid in t[1]])


@gpu
def test_stack_depth_limits(world, monkeypatch):
    """compiled stack depths 4, 5 and 15 (128 KiB of operand stack) evaluate; 16 is refused with FBGPU_E_INVALID before any
    launch.  Under FBGPU_FORCE_WORDPAR, 256 / 257 compiled ops and depth 4 / 5 lie on both sides of the word-parallel
    selection rule and agree"""
    ctx = world
    rng = np.random.default_rng(SEED)
    for d in (4, 5, 15):
        t = nested(rng, d)
        ops = tree_ops(t)
        prog, depth = ctx.debug_compile(IDX, ops)
        assert (len(prog), depth) == (4 * d - 1, d)
        check_r_program(ctx, ops, tree_eval(t), d, columns=not ON_EMU)
    ops = tree_ops(nested(rng, 16))
    for call in (lambda: ctx.debug_compile(IDX, ops), lambda: ctx.count(IDX, ops, SHARDS), lambda: ctx.row(IDX, ops, SHARDS),
                 lambda: ctx.columns(IDX, ops, SHARDS), lambda: ctx.any(IDX, ops, SHARDS)):
        before = ctx.counters()["kernel_launches"]
        with pytest.raises(L.FbgpuError) as e:
            call()
        assert e.value.code == L.E_INVALID and "depth 16" in str(e.value)
        assert ctx.counters()["kernel_launches"] == before
    monkeypatch.setenv("FBGPU_FORCE_WORDPAR", "1")
    cs = container_set()
    for k in (255, 256):
        rows = [int(r) for r in rng.integers(0, len(cs), k)]
        ops = [row_op(R, r) for r in rows] + [nary("xor", k)]
        assert len(ctx.debug_compile(IDX, ops)[0]) == k + 1
        assert ctx.count(IDX, ops, SHARDS) == 2 * int(fold("xor", [masks()[r] for r in rows]).sum()), k
    for d in (4, 5):
        t = nested(rng, d)
        assert ctx.debug_compile(IDX, tree_ops(t))[1] == d
        assert ctx.count(IDX, tree_ops(t), SHARDS) == 2 * int(tree_eval(t).sum()), d


@gpu
def test_canonical_emission_boundaries(world):
    """results of N = 1, 4095, 4096, 4097, 65,536 and of runs = N/2, N/2 + 1, 2048, 2049, reached by Intersect with `full` in
    each encoding, by Union and by Xor: every container's type and bytes"""
    ctx = world
    for k, (name, v, (n, runs)) in enumerate(emission_targets()):
        assert len(v) == n and runs in (None, 1 + int(np.count_nonzero(np.diff(v) != 1))), name
        m = mask_of(v)
        for e in range(3):
            for f in range(3):
                ops = [row_op(EM, 10 * k + e), row_op(FULL, f), nary("and", 2)]
                check_r_program(ctx, ops, m, (name, "and full", e, f), columns=(e == f and not ON_EMU))
        check_r_program(ctx, [row_op(EM, 10 * k + 3), row_op(EM, 10 * k + 4), nary("or", 2)], m, (name, "or"), columns=not ON_EMU)
        check_r_program(ctx, [row_op(EM, 10 * k + 5), row_op(EM, 10 * k + 6), nary("xor", 2)], m, (name, "xor"), columns=not ON_EMU)


@gpu
def test_not_all_any(world):
    """Not and All with the existence row stored in each encoding; Any over 8, 9, 64 and 65 shards with the only column in the
    last one, launched in blocks of 8, 64, 512 ... shards"""
    ctx = world
    cs = container_set()
    ex = existence_mask()
    picks = range(len(cs)) if not ON_EMU else [index_of(n, t) for n in ("full", "oddBitsSet", "random1", "random40000") for t in ENCODINGS]
    for e in range(3):
        check_r_program(ctx, [L.Op(L.OP_ALL, EX, 0, 0, e, 0, 0, 0)], ex, ("all", e))
        for i in picks:
            check_r_program(ctx, [row_op(R, i), L.Op(L.OP_NOT, EX, 0, 1, e, 0, 0, 0)], ex & ~masks()[i], ("not", e, cs[i][0], cs[i][2]),
                            row=not ON_EMU or i == picks[0], columns=i == picks[0])
        j = index_of("block@4096", ENCODINGS[e])
        t = ("not", e, ("xor", [("row", j), ("row", index_of("random5000", O.ARRAY))]))
        check_r_program(ctx, tree_ops(t), tree_eval(t), ("not of xor", e))
    for n, launches in ((8, 1), (9, 2), (64, 2), (65, 2)):       # blocks [0, 8), [8, 72), ...
        before = ctx.counters()["kernel_launches"]
        assert ctx.any(IDX, [row_op(ANYF, n)], list(range(n))), n
        assert ctx.counters()["kernel_launches"] - before == launches, n
        assert not ctx.any(IDX, [row_op(ANYF, n)], list(range(n - 1))), n
        assert ctx.any(IDX, [row_op(ANYF, 1), row_op(ANYF, n), nary("andnot", 2)], list(range(n))), n
        assert not ctx.any(IDX, [row_op(ANYF, n), row_op(ANYF, 1), nary("and", 2)], list(range(n))), n


def windows(bounds, total):
    """(offset, limit) windows over results whose units end at the ranks in bounds"""
    b1, b2, bl = bounds[0], bounds[1], bounds[-2]
    return [(0, None), (0, 0), (b1, 0), (0, b1), (b1, b2 - b1), (b1 - 1, 2), (b1 + 3, 7), (b1 - 1, b2 - b1 + 2), (bl, None), (max(bl - 5, 0), 5),
            (total - 1, 10), (total, 5), (total + 10, None), (total + 10, 3), (b1 // 2, total)]


def check_windows(ctx, ps, op, shards):
    prog = ps.program(op)
    exp = expected_columns(ps, op, shards)
    sizes = [int(ps.result(op, s)[slot].sum()) for s in shards for slot in range(16)]
    bounds = [b for b in np.cumsum(sizes).tolist() if b]
    assert len(set(bounds)) >= 3, (op, shards)
    bounds = sorted(set(bounds))
    for off, lim in windows(bounds, len(exp)):
        got, total = ctx.columns(IDX, prog, shards, offset=off, limit=lim)
        end = None if lim is None else off + lim
        assert total == len(exp) and np.array_equal(got, exp[off:end]), (op, off, lim)


@gpu
def test_columns_windows(world):
    """Columns windows on unit edges, inside units, limit 0 and offsets at and past the end, over results of every encoding"""
    ps = pair_sets()[0]
    for op in OPC:
        check_windows(world, ps, op, ps.shards[:3])


@gpu
def test_columns_windows_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch, so Row and Columns are assembled from several batches"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    ctx = L.Context(0)
    try:
        main = pair_sets()[0]
        ps = PairSet(FA, FB, main.conts, main.m, main.pairs[: 16 * 4 + 5])
        ps.load(ctx)
        ctx.commit()
        for op in OPC:
            row = []
            for s in ps.shards:
                r = ps.result(op, s)
                row += expect_row([(s * 16 + slot, r[slot]) for slot in range(16)])
            data, cnt = ctx.row(IDX, ps.program(op), ps.shards)
            check_row(data, cnt, row, op)
            check_windows(ctx, ps, op, ps.shards)
    finally:
        ctx.close()


def random_tree(rng, depth, n):
    """a tree of exactly `depth` levels of calls (its first child is the deepest), up to 6 children per call"""
    if depth == 0:
        return ("row", int(rng.integers(n)))
    if rng.random() < 0.1:
        return ("not", int(rng.integers(3)), random_tree(rng, depth - 1, n))
    kids = [random_tree(rng, depth - 1, n)] + [random_tree(rng, int(rng.integers(depth)), n) for _ in range(int(rng.integers(0, 6)))]
    return (["and", "or", "andnot", "xor"][int(rng.integers(4))], kids)


@gpu
def test_random_trees(world, monkeypatch):
    """random call trees of depth 3-4 over the container set (FBGPU_FUZZ_SEED): Count (default and forced word-parallel), Row
    and Columns against numpy"""
    ctx = world
    rng = np.random.default_rng(SEED)
    n = len(container_set())
    for trial in range(4 if ON_EMU else 40):
        t = random_tree(rng, 3 + trial % 2, n)
        ops = tree_ops(t)
        m = tree_eval(t)
        check_r_program(ctx, ops, m, (SEED, trial))
        with monkeypatch.context() as mp:
            mp.setenv("FBGPU_FORCE_WORDPAR", "1")
            assert ctx.count(IDX, ops, SHARDS) == 2 * int(m.sum()), (SEED, trial, "wordpar")


# ------------------------------------------------------------------ CPU
def test_setop_matrix_on_interpreted_kernels():
    """the gpu tests on the interpreted kernels, in both array orders: a sampled subset of pairs and trees, or all of them as on
    a GPU under FBGPU_EMU_FULL=1"""
    from tests.test_emu_kernels import FULL, run_on_emulator
    run_on_emulator(["tests/test_setop_matrix.py"], env={"FBGPU_EMU_FULL_SIZE": "1"} if FULL else None, timeout=3000)
