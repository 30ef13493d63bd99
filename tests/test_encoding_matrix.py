"""The kernels outside the set-op path on containers of every encoding, the non-canonical ones included.

roaring_io.encode() and datagen optimize() every container, so tests built on them only hand the kernels canonical shapes:
arrays below 4096 elements, run containers of at most 2048 runs, bitmaps for the rest.  A fragment written without
optimize(), or an fbgpu_apply_containers batch, may also carry arrays of up to 65,536 elements, run containers of up to
65,535 intervals (odd or even bits: 32,768 one-bit runs), a bitmap holding one bit.  The container set below holds each
value set in all three encodings, loaded with to_bytes(optimize=False), and every test compares an entry point with numpy /
Python-integer results computed from the values it wrote, exactly.

Branches only these shapes reach:
  - groupby_kernel's dense pass for an array a-row of 4096 elements or more (test_groupby_mixed_encodings,
    test_groupby_array_fields), run b-rows of more than 2048 intervals in its probe;
  - groupby_direct_kernel declining arrays above kGdMaxCard and groupby_kernel taking the declined units from its unit list
    (test_groupby_array_fields, which asserts the fallback counter);
  - unit_load_plane (bsi_sum / bsi_minmax / bsi_select_step) scattering arrays of 4096 to 65,536 elements and expanding runs
    above 2048 (bm_expand_runs), extract_values_kernel and the range programs on the same planes (test_bsi_value_entry_points,
    test_bsi_range_programs);
  - gv_for_each and the 16-bit run count in groupby_values_kernel's shuffled meta word (test_groupby_values);
  - row_count_kernel's warp_count_vs_global_bitmap and its shuffled meta word (test_row_counts).

Every case puts all its containers into one (shard, slot) unit and the same fragment into another slot of a second shard,
so each result is also summed across shards.  The CPU tests check that the store keeps every container in the encoding it
was built with, and run the gpu tests on the interpreted kernels."""
import ctypes as C
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

from featurebase_b200 import lib as L
from oracle import oracle as O
from tests import archetypes as A

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR")) and not os.environ.get("FBGPU_EMU_FULL_SIZE")      # fewer filters, rows, trials
CTA = bool(os.environ.get("FBGPU_GROUPBY_CTA"))           # read once per process by the library: groupby_kernel for every unit
SW, W = 1 << 20, 1 << 16
IDX = 0
F, G, FILT = 1, 2, 3                   # set fields holding the whole container set, row i = container i (view 0)
FA, GA = 4, 5                          # array-only set fields, arrays of up to 40,000 elements
FS, GS = 6, 7                          # array-only set fields, arrays of at most kGdMaxCard (1024) elements
V, VZ, VV = 8, 9, 7                    # int fields and their BSI view: V without, VZ with columns stored as sign + magnitude 0
SHARDS = [0, 1]
SLOTS = (5, 11)                        # shard 0 holds the case in slot 5, shard 1 in slot 11
ENCODINGS = (O.ARRAY, O.BITMAP, O.RUN)
ENC_NAME = {O.ARRAY: "array", O.BITMAP: "bitmap", O.RUN: "run"}
DEPTHS = [1, 12, 33, 63, 64]
CMPS = ["==", "!=", "<", "<=", ">", ">=", "><"]
gpu = pytest.mark.gpu


def n_runs(vals):
    return 0 if len(vals) == 0 else 1 + int(np.count_nonzero(np.diff(vals) != 1))


@functools.lru_cache(maxsize=None)
def value_sets():
    """[(name, sorted column values)]: the non-empty reference archetypes, random sets, contiguous blocks touching column 0,
    column 65,535 and the edges of 4096-column ranges"""
    rng = np.random.default_rng(2024)
    sets = [(n, A.archetype_values(n)) for n in A.NAMES if n != "empty"]
    sets += [(f"random{k}", np.sort(rng.choice(W, k, replace=False))) for k in (1, 50, 1025, 4095, 4096, 4097, 5000, 40000)]
    sets += [("block@0", np.arange(0, 3000)), ("block@65535", np.arange(W - 2500, W)), ("block@4096", np.arange(4096 - 700, 4096 + 700)),
             ("block@8191", np.arange(8192 - 1000, 8192))]
    return [(n, np.asarray(v, dtype=np.int64)) for n, v in sets]


@functools.lru_cache(maxsize=None)
def container_set():
    """[(name, values, encoding)]: every value set in all three encodings (a run form above 65,535 intervals would be left
    out), plus a 64-element array, the smallest one stored in bank-striped order"""
    out = [(n, v, t) for n, v in value_sets() for t in ENCODINGS if t != O.RUN or n_runs(v) <= 65535]
    out.append(("striped64", np.sort(np.random.default_rng(7).choice(W, 64, replace=False)), O.ARRAY))
    return out


@functools.lru_cache(maxsize=None)
def masks():
    """[n_containers, 65536] bool: the columns of each container"""
    m = np.zeros((len(container_set()), W), dtype=bool)
    for i, (_, v, _) in enumerate(container_set()):
        m[i, v] = True
    return m


def mask_of(vals):
    m = np.zeros(W, dtype=bool)
    m[vals] = True
    return m


def index_of(name, typ):
    return next(i for i, (n, _, t) in enumerate(container_set()) if n == name and t == typ)


def abs_cols(local):
    """the columns of the local (in-slot) columns in both shards, ascending"""
    local = np.asarray(local, dtype=np.int64)
    return np.concatenate([SLOTS[0] * W + local, SW + SLOTS[1] * W + local])


def load(ctx, field, view, rows):
    """rows: [(row id, container)] -> one fragment per shard, every container in that shard's slot, encodings as built"""
    for shard, slot in zip(SHARDS, SLOTS):
        b = O.Bitmap()
        for r, c in rows:
            b.put(r * 16 + slot, c)
        ctx.load_fragment(IDX, field, view, shard, b.to_bytes(optimize=False))


def row_op(field, row):
    return L.Op(L.OP_ROW, field, 0, 0, row, 0, 0, 0)


def filters(seed, n_emu, n_gpu):
    """[(None | filter row of FILT, its columns mask)]: no filter, then filter rows of the container set, every encoding at least
    once"""
    rng = np.random.default_rng(seed)
    by_enc = {t: [i for i, (_, _, tt) in enumerate(container_set()) if tt == t] for t in ENCODINGS}
    n = n_emu if ON_EMU else n_gpu
    rows = [int(rng.choice(by_enc[ENCODINGS[k % 3]])) for k in range(n)]
    return [(None, None)] + [(r, masks()[r]) for r in rows]


# ------------------------------------------------------------------ set fields
ARRAY_FIELD = ["firstBitSet", "lastBitSet", "outerBitsSet", "oddBitsSet", "random1", "random50", "random1025", "random4095", "random4096",
               "random4097", "random5000", "random40000", "block@0", "block@65535", "block@4096", "block@8191", "striped64"]


def interleaved(idx, field_rows=None):
    """row order with two sparse a-rows (arrays below 4096 elements) before each dense one, so groupby_kernel runs a sparse
    pass, a dense pass and another sparse pass; field_rows[i]: the container-set index of the field's row i (default: i)"""
    cs = container_set()
    at = (lambda i: cs[i]) if field_rows is None else (lambda i: cs[field_rows[i]])
    dense = [i for i in idx if at(i)[2] != O.ARRAY or len(at(i)[1]) >= 4096]
    sparse = [i for i in idx if i not in dense]
    out = []
    while dense or sparse:
        out += sparse[:2] + dense[:1]
        sparse, dense = sparse[2:], dense[1:]
    return out


@functools.lru_cache(maxsize=None)
def small_arrays():
    """(values) of FS / GS: the arrays of the set with at most 1024 elements, and one of exactly 1024"""
    vs = [v for n, v, t in container_set() if t == O.ARRAY and len(v) <= 1024]
    return vs + [np.sort(np.random.default_rng(8).choice(W, 1024, replace=False))]


@pytest.fixture(scope="module")
def world():
    """a context holding F, G and FILT (the container set), FA / GA (its arrays of up to 40,000 elements) and FS / GS (arrays
    groupby_direct_kernel accepts)"""
    ctx = L.Context(0)
    cs = container_set()
    rows = [(i, A.container_of(v, t)) for i, (_, v, t) in enumerate(cs)]
    for f in (F, G, FILT):
        load(ctx, f, 0, rows)
    arr = [i for i, (n, _, t) in enumerate(cs) if t == O.ARRAY and n in ARRAY_FIELD]
    for f in (FA, GA):
        load(ctx, f, 0, [(k, A.container_of(cs[i][1], O.ARRAY)) for k, i in enumerate(arr)])
    for f in (FS, GS):
        load(ctx, f, 0, [(k, A.container_of(v, O.ARRAY)) for k, v in enumerate(small_arrays())])
    ctx.commit()
    yield ctx, arr
    ctx.close()


def expect_pairs(ma, mb, keep):
    """group counts over both shards: 2 * (ma ∩ keep) @ mb^T, in int64"""
    a = (ma & keep) if keep is not None else ma
    return 2 * (a.astype(np.int64) @ mb.astype(np.int64).T)


def check_groupby(ctx, fa, fb, rows_a, rows_b, ma, mb, fl, declined):
    """one GroupBy per filter; `declined`: units groupby_direct_kernel is expected to hand to groupby_kernel per call (None:
    groupby_kernel takes every unit without the direct kernel)"""
    for frow, fmask in fl:
        before = ctx.counters()
        got = ctx.groupby(IDX, [fa, fb], [0, 0], [rows_a, rows_b], SHARDS, filter_ops=None if frow is None else [row_op(FILT, frow)])
        assert np.array_equal(got.astype(np.int64), expect_pairs(ma, mb, fmask)), frow
        after = ctx.counters()
        units, fallback = after["groupby_units"] - before["groupby_units"], after["groupby_fallback_units"] - before["groupby_fallback_units"]
        if declined is None or CTA:
            assert (units, fallback) == (0, 0), frow
        else:
            assert (units, fallback) == (16 * len(SHARDS), declined), frow


@gpu
def test_groupby_mixed_encodings(world):
    """GroupBy(Rows(F), Rows(G)) over the whole container set: bitmap / run heavy fields, so groupby_kernel takes every unit;
    the dense pass meets bitmaps, runs of up to 32,768 intervals and arrays of up to 65,536 elements"""
    ctx, _ = world
    n = len(container_set())
    rows_a = interleaved(list(range(n)))
    rows_b = list(range(n))[::-1]
    m = masks()
    check_groupby(ctx, F, G, rows_a, rows_b, m[rows_a], m[rows_b], filters(1, 3, 9), None)


@gpu
def test_groupby_array_fields(world):
    """array-only fields that groupby_direct_eligible accepts: with arrays above 1024 (and above 4096) elements every non-empty
    unit is declined and counted by groupby_kernel from the unit list, dense array pass included; with arrays of at most 1024
    the direct kernel counts them itself"""
    ctx, arr = world
    cs = container_set()
    ma = masks()[arr]
    rows_a = interleaved(list(range(len(arr))), arr)
    check_groupby(ctx, FA, GA, rows_a, list(range(len(arr))), ma[rows_a], ma, filters(2, 3, 6), len(SHARDS))
    assert any(len(cs[i][1]) > 4096 for i in arr) and any(1024 < len(cs[i][1]) <= 4096 for i in arr)
    sm = np.stack([mask_of(v) for v in small_arrays()])
    rows = list(range(len(sm)))
    check_groupby(ctx, FS, GS, rows[::-1], rows, sm[::-1], sm, filters(3, 3, 6), 0)


@gpu
def test_groupby_kernel_for_every_unit():
    """the two GroupBy tests again with FBGPU_GROUPBY_CTA=1 (fixed per process, so in a child): groupby_kernel takes every
    unit, the array-only fields included"""
    if CTA:
        pytest.skip("this process already runs with FBGPU_GROUPBY_CTA=1")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "-p", "no:cacheprovider", os.path.abspath(__file__), "-k",
                        "groupby_mixed_encodings or groupby_array_fields"], cwd=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                       env=dict(os.environ, FBGPU_GROUPBY_CTA="1"), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=3000)
    tail = "\n".join(r.stdout.splitlines()[-25:])
    assert r.returncode == 0 and "2 passed" in tail, tail


@gpu
def test_row_counts(world):
    """fbgpu_row_counts (listed rows and every row) and fbgpu_row_counts_per_shard over rows of every encoding, with no filter
    and with filter rows of every encoding"""
    ctx, _ = world
    m = masks()
    n = len(m)
    rows = list(range(n))[::-1]
    for frow, fmask in filters(4, 4, 12):
        fo = None if frow is None else [row_op(FILT, frow)]
        per = (m[rows] & fmask).sum(axis=1) if fmask is not None else m[rows].sum(axis=1)
        assert ctx.row_counts(IDX, F, 0, SHARDS, row_ids=rows, filter_ops=fo).tolist() == (2 * per).tolist(), frow
        assert ctx.row_counts_per_shard(IDX, F, 0, SHARDS, rows, filter_ops=fo).tolist() == [per.tolist()] * 2, frow
    rid, cnt = ctx.row_counts(IDX, F, 0, SHARDS)                      # every row, by count descending, then row id
    exp = sorted(((r, 2 * int(c)) for r, c in enumerate(m.sum(axis=1))), key=lambda rc: (-rc[1], rc[0]))
    assert list(zip(rid.tolist(), cnt.tolist())) == exp


def windows(n):
    """(offset, limit) windows over 2n results, n per unit: inside the first unit, across the two units, inside the second,
    the last one, past the end, and no limit from inside the first"""
    h = max(n // 3, 1)
    return [(h, h), (max(n - 2, 0), 5), (n + h, h), (2 * n - 1, 3), (2 * n + 1, 2), (n // 2, None)]


@gpu
def test_columns_and_extract_windows():
    """fbgpu_columns of rows stored in every encoding, and fbgpu_extract with each such row as the filter, whole and in
    offset / limit windows that cut inside a unit"""
    ctx = L.Context(0)
    try:
        cs = container_set()
        load(ctx, F, 0, [(i, A.container_of(v, t)) for i, (_, v, t) in enumerate(cs)])
        rng = np.random.default_rng(5)
        vals = rng.integers(-(1 << 40), 1 << 40, W)
        rows = [(0, A.container_of(np.arange(W), O.BITMAP)), (1, A.container_of(np.nonzero(vals < 0)[0], O.BITMAP))]
        rows += [(2 + i, A.container_of(np.nonzero((np.abs(vals) >> i) & 1)[0], O.BITMAP)) for i in range(41)]
        load(ctx, V, VV, rows)
        ctx.commit()
        picks = range(len(cs)) if not ON_EMU else [index_of(n, t) for n in ("full", "oddBitsSet", "random40000", "random1", "block@4096") for t in ENCODINGS]
        for i in picks:
            local = cs[i][1]
            cols = abs_cols(local).tolist()
            ev = np.concatenate([vals[local], vals[local]]).tolist()
            got, total = ctx.columns(IDX, [row_op(F, i)], SHARDS)
            assert (got.tolist(), total) == (cols, len(cols)), cs[i][:1]
            c, v, total = ctx.extract(IDX, V, VV, 41, SHARDS, filter_ops=[row_op(F, i)])
            assert (c.tolist(), v.tolist(), total) == (cols, ev, len(cols)), cs[i][:1]
            for off, lim in windows(len(local)):
                end = None if lim is None else off + lim
                got, total = ctx.columns(IDX, [row_op(F, i)], SHARDS, offset=off, limit=lim)
                assert (got.tolist(), total) == (cols[off:end], len(cols)), (cs[i][0], off, lim)
                c, v, total = ctx.extract(IDX, V, VV, 41, SHARDS, filter_ops=[row_op(F, i)], offset=off, limit=lim)
                assert (c.tolist(), v.tolist(), total) == (cols[off:end], ev[off:end], len(cols)), (cs[i][0], off, lim)
    finally:
        ctx.close()


# ------------------------------------------------------------------ int fields
class BsiCase:
    """an int field of depth d whose exists row, sign row and magnitude planes are value sets of the container set, each in a
    random encoding.  Columns stored as sign with magnitude 0 are dropped from V's sign row (the comparisons, Min / Max and
    the select order have no rule for them that existing tests pin down); VZ keeps them, and its GroupBy counts them
    nowhere, as Row(v == 0) does not hold them.  At depth 64, plane 63 holds only columns stored as INT64_MIN
    (sign + magnitude 2^63), a few columns cleared of the lower planes for it."""

    def __init__(self, depth, seed):
        rng = np.random.default_rng(seed)
        pool = [v for _, v in value_sets()]
        draw = lambda: mask_of(pool[int(rng.integers(len(pool)))])
        enc = lambda: ENCODINGS[int(rng.integers(3))]
        self.depth = depth
        self.exists, sign0 = draw(), draw()
        planes = [draw() for _ in range(depth)]
        if depth == 64:
            low = np.any(planes[:63], axis=0)
            cand = np.nonzero(self.exists & sign0)[0]
            pick = rng.choice(cand, min(3, len(cand)), replace=False) if len(cand) else []
            for p in planes[:63]:
                p[pick] = False
            planes[63] &= sign0 & ~low
            planes[63][pick] = True
        mag = np.zeros(W, dtype=np.uint64)
        for i, p in enumerate(planes):
            mag |= p.astype(np.uint64) << np.uint64(i)
        self.mag = mag
        self.sign = sign0 & (mag != 0)
        self.sign_z = sign0
        self.rows = [(0, self.exists, enc()), (1, None, enc())] + [(2 + i, p, enc()) for i, p in enumerate(planes)]     # (row, columns, encoding)

    def load(self, ctx):
        for field, sign in ((V, self.sign), (VZ, self.sign_z)):
            rows = []
            for r, m, t in self.rows:
                m = sign if r == 1 else m
                if m.any():
                    rows.append((r, A.container_of(np.nonzero(m)[0], t)))
            load(ctx, field, VV, rows)

    def columns(self, keep_mask):
        """(local columns, Python-int values, negative-zero flags) of exists ∩ keep, ascending"""
        keep = self.exists if keep_mask is None else self.exists & keep_mask
        local = np.nonzero(keep)[0]
        mags = [int(x) for x in self.mag[local].tolist()]
        vals = [-m if s else m for m, s in zip(mags, self.sign[local].tolist())]
        negz = (self.sign_z[local] & (self.mag[local] == 0)).tolist()
        return local, vals, negz


def wrap64(x):
    return ((x + 2**63) % 2**64) - 2**63


def check_values(ctx, case, frow, fmask):
    d = case.depth
    fo = None if frow is None else [row_op(FILT, frow)]
    local, vals, negz = case.columns(fmask)
    cols, both = abs_cols(local).tolist(), vals + vals
    n = len(both)
    assert ctx.bsi_sum(IDX, V, VV, d, SHARDS, filter_ops=fo) == (wrap64(sum(both)), n), (d, frow)
    assert ctx.bsi_sum(IDX, VZ, VV, d, SHARDS, filter_ops=fo) == (wrap64(sum(both)), n), (d, frow)      # sign + 0 adds 0
    for want_max in (False, True):
        e = (max(both) if want_max else min(both)) if both else 0
        assert ctx.bsi_minmax(IDX, V, VV, d, SHARDS, want_max, filter_ops=fo) == ((e, both.count(e)) if both else (0, 0)), (d, frow, want_max)
    c, v, total = ctx.extract(IDX, V, VV, d, SHARDS, filter_ops=fo)
    assert (c.tolist(), v.tolist(), total) == (cols, both, n), (d, frow)
    c, v, _ = ctx.extract(IDX, VZ, VV, d, SHARDS, filter_ops=fo)
    assert v.tolist() == both, (d, frow)                                                                 # sign + 0 reads 0
    for off, lim in windows(len(local))[:2 if ON_EMU else 6]:
        end = None if lim is None else off + lim
        c, v, total = ctx.extract(IDX, V, VV, d, SHARDS, filter_ops=fo, offset=off, limit=lim)
        assert (c.tolist(), v.tolist(), total) == (cols[off:end], both[off:end], n), (d, frow, off, lim)
    if d <= 63 and n:
        s = sorted(both)
        ranks = list(range(n)) if n <= 48 else sorted({0, 1, n // 4, n // 2, n // 2 + 1, 3 * n // 4, n - 2, n - 1})
        for r0 in range(0, len(ranks), L.SELECT_MAX_RANKS):
            rk = ranks[r0: r0 + L.SELECT_MAX_RANKS]
            v, cnt, total = ctx.bsi_select(IDX, V, VV, d, SHARDS, rk, filter_ops=fo)
            assert total == n and v.tolist() == [s[r] for r in rk], (d, frow, rk)
            assert cnt.tolist() == [both.count(s[r]) for r in rk], (d, frow, rk)
    return local, vals, negz


def bsi_filters(seed):
    """no filter, one filter row per encoding and a 50-column one (every rank of its values is selected)"""
    fl = filters(seed, 3, 6)
    rng = np.random.default_rng(seed)
    r = index_of("random50", ENCODINGS[int(rng.integers(3))])
    return fl + [(r, masks()[r])]


def trials(depth):
    return [depth * 10 + t for t in range(1 if ON_EMU else 3)]


@gpu
@pytest.mark.parametrize("depth", DEPTHS)
def test_bsi_value_entry_points(depth):
    """bsi_sum, bsi_minmax both ways, extract (whole and in windows) and bsi_select over planes of every encoding, with no
    filter and with filter rows of every encoding"""
    for seed in trials(depth):
        ctx = L.Context(0)
        try:
            case = BsiCase(depth, seed)
            case.load(ctx)
            load(ctx, FILT, 0, [(i, A.container_of(v, t)) for i, (_, v, t) in enumerate(container_set())])
            ctx.commit()
            for frow, fmask in bsi_filters(seed):
                check_values(ctx, case, frow, fmask)
        finally:
            ctx.close()


def range_matches(c, lo, hi):
    if c == "><":
        return lambda v: lo <= v <= hi
    return {"==": lambda v: v == lo, "!=": lambda v: v != lo, "<": lambda v: v < lo, "<=": lambda v: v <= lo, ">": lambda v: v > lo,
            ">=": lambda v: v >= lo}[c]


@gpu
@pytest.mark.parametrize("depth", DEPTHS)
def test_bsi_range_programs(depth):
    """Count and Row of OP_BSI_RANGE for every comparison at predicate values that are present, alone and intersected with
    filter rows of every encoding"""
    for seed in trials(depth):
        ctx = L.Context(0)
        try:
            case = BsiCase(depth, seed + 5)
            case.load(ctx)
            load(ctx, FILT, 0, [(i, A.container_of(v, t)) for i, (_, v, t) in enumerate(container_set())])
            ctx.commit()
            rng = np.random.default_rng(seed)
            for frow, fmask in filters(seed, 1, 3):
                local, vals, _ = case.columns(fmask)
                if not vals:
                    continue
                cols = abs_cols(local).tolist()
                present = sorted(set(vals))
                p = [present[int(rng.integers(len(present)))] for _ in range(2)]
                for c in CMPS:
                    lo, hi = (min(p), max(p)) if c == "><" else (p[0], 0)
                    m = range_matches(c, lo, hi)
                    exp = [col for col, v in zip(cols, vals + vals) if m(v)]
                    op = [L.Op(L.OP_BSI_RANGE, V, VV, 0, depth, L.CMP[c], lo, hi)]
                    if frow is not None:
                        op = [row_op(FILT, frow)] + op + [L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)]
                    assert ctx.count(IDX, op, SHARDS) == len(exp), (depth, frow, c, lo, hi)
                    data, cnt = ctx.row(IDX, op, SHARDS)
                    assert cnt == len(exp) and O.Bitmap.from_bytes(data).slice().tolist() == exp, (depth, frow, c, lo, hi)
        finally:
            ctx.close()


def value_list(rng, depth, present):
    """a strictly ascending list of more than kGvHist (1024) values: present ones and absent ones"""
    if depth <= 12:
        return list(range(-1500, 1501))
    pick = rng.choice(len(present), min(len(present), 1400), replace=False)
    absent = [x for x in (-(1 << 60), -12345, 3, 1 << 40) if x not in set(present)]
    return sorted(set([present[i] for i in pick.tolist()] + absent))


@gpu
@pytest.mark.parametrize("depth", DEPTHS)
def test_groupby_values(depth):
    """fbgpu_groupby_values over VZ (planes of every encoding, columns stored as sign + magnitude 0 counted nowhere) with no set
    dimension and with rows of the container set as the set dimension, under no filter and filter rows of every encoding"""
    cs = container_set()
    b_rows = list(range(len(cs))) if not ON_EMU else [index_of(n, t) for n in ("full", "oddBitsSet", "random4097", "block@4096", "random1")
                                                     for t in ENCODINGS]
    for seed in trials(depth):
        ctx = L.Context(0)
        try:
            case = BsiCase(depth, seed + 7)
            case.load(ctx)
            load(ctx, G, 0, [(i, A.container_of(v, t)) for i, (_, v, t) in enumerate(cs)])
            load(ctx, FILT, 0, [(i, A.container_of(v, t)) for i, (_, v, t) in enumerate(cs)])
            ctx.commit()
            rng = np.random.default_rng(seed)
            for frow, fmask in filters(seed, 1, 3):
                fo = None if frow is None else [row_op(FILT, frow)]
                local, vals, negz = case.columns(fmask)
                values = value_list(rng, depth, sorted(set(v for v, z in zip(vals, negz) if not z)))
                pos = {v: j for j, v in enumerate(values)}
                k = np.array([-1 if z else pos.get(v, -1) for v, z in zip(vals, negz)], dtype=np.int64)
                hit = k >= 0
                exp0 = 2 * np.bincount(k[hit], minlength=len(values))
                got = ctx.groupby_values(IDX, [], [], [], VZ, VV, depth, values, SHARDS, filter_ops=fo)
                assert np.array_equal(got.astype(np.int64), exp0), (depth, frow)
                exp1 = np.stack([2 * np.bincount(k[hit & masks()[b][local]], minlength=len(values)) for b in b_rows])
                got = ctx.groupby_values(IDX, [G], [0], [b_rows], VZ, VV, depth, values, SHARDS, filter_ops=fo)
                assert np.array_equal(got.astype(np.int64), exp1), (depth, frow)
        finally:
            ctx.close()


@gpu
def test_unit_batch_16(monkeypatch):
    """FBGPU_UNIT_BATCH=16: one shard per evaluation batch, for the filtered GroupBy, row counts and an int field's entry points"""
    monkeypatch.setenv("FBGPU_UNIT_BATCH", "16")
    ctx = L.Context(0)
    try:
        cs = container_set()
        rows = [(i, A.container_of(v, t)) for i, (_, v, t) in enumerate(cs)]
        for f in (F, G, FILT):
            load(ctx, f, 0, rows)
        case = BsiCase(33, 99)
        case.load(ctx)
        ctx.commit()
        m = masks()
        n = len(cs)
        for frow, fmask in filters(6, 1, 3)[1:]:
            fo = [row_op(FILT, frow)]
            got = ctx.groupby(IDX, [F, G], [0, 0], [interleaved(list(range(n))), list(range(n))], SHARDS, filter_ops=fo)
            assert np.array_equal(got.astype(np.int64), expect_pairs(m[interleaved(list(range(n)))], m, fmask)), frow
            assert ctx.row_counts(IDX, F, 0, SHARDS, row_ids=list(range(n)), filter_ops=fo).tolist() == (2 * (m & fmask).sum(axis=1)).tolist()
            check_values(ctx, case, frow, fmask)
    finally:
        ctx.close()


# ------------------------------------------------------------------ CPU
def test_containers_keep_their_encoding():
    """every container of the set reaches the store in the encoding it was built with, whatever its size"""
    ctx = L.Context(L.DEVICE_NONE)
    try:
        cs = container_set()
        load(ctx, F, 0, [(i, A.container_of(v, t)) for i, (_, v, t) in enumerate(cs)])
        buf = np.empty(1 << 18, dtype=np.uint8)
        for shard, slot in zip(SHARDS, SLOTS):
            for i, (name, v, t) in enumerate(cs):
                typ, card, runs, n = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)      # (Context.debug_container's buffer holds 8 KiB)
                rc = ctx.L.fbgpu_debug_container(ctx.h, IDX, F, 0, shard, i, slot, C.byref(typ), C.byref(card), C.byref(runs), buf.ctypes.data, len(buf),
                                                 C.byref(n))
                assert rc == 0, (name, t)
                assert (typ.value, card.value) == (t, len(v)), (name, ENC_NAME[t])
                if t == O.RUN:
                    assert runs.value == n_runs(v), name
    finally:
        ctx.close()
    shapes = {(ENC_NAME[t], "array>4096" if t == O.ARRAY and len(v) > 4096 else "runs>2048" if t == O.RUN and n_runs(v) > 2048 else
               "one-bit bitmap" if t == O.BITMAP and len(v) == 1 else "") for _, v, t in cs}
    assert {("array", "array>4096"), ("run", "runs>2048"), ("bitmap", "one-bit bitmap")} <= shapes


def test_encoding_matrix_on_interpreted_kernels():
    """the gpu tests on the interpreted kernels: with fewer filters, rows and trials (≈30 s), or as on a GPU under
    FBGPU_EMU_FULL=1 (≈2 min)"""
    from tests.test_emu_kernels import FULL, run_on_emulator
    run_on_emulator(["tests/test_encoding_matrix.py"], env={"FBGPU_EMU_FULL_SIZE": "1"} if FULL else None, timeout=3000)
