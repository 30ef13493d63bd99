"""Every query kernel on a store that has been updated, dropped, rolled back and compacted, in every row-directory form.

A plain Python model of the store — (field, view, shard) -> {container key: (sorted column values, encoding)} — is changed
step by step together with the library: fragments replaced by fbgpu_load_fragment and by fbgpu_load_fragments batches (one
of them failing half way), containers put and removed by fbgpu_apply_containers in every encoding (arrays above 4096
elements, run containers above 2048 intervals and one-bit bitmaps included), int values rewritten plane by plane, fragments
dropped, commits explicit and implicit, the arena compacted.  Every fragment and every batch is built from the model with
to_bytes(optimize=False), so the store holds exactly the encodings the test chose, and every result is compared exactly with
numpy / Python integers computed from the model.

The world (index 0):
  FA  array-dominated set field, dense row ids 0..5 (bank-striped arrays; GroupBy FA x FA takes groupby_direct_kernel's
      dense-directory walk), shards 0..3
  FB  bitmap / run heavy set field, dense row ids, shards 0..3 (Count on eval_wordpar_kernel while no array of the view is
      bank-striped; GroupBy on groupby_kernel).  Shard 3 joins array-dominated, so its arrays are bank-striped.
  FC  array-dominated, rows 0..4 in shard 0 and around 10^6 in shards 2 and FAR: every fragment's rows are contiguous, the
      view's are not (the contiguous search chain)
  FD  array-dominated, sparse rows {0, 7, 40000, 2^30} in shards 0, 1 and FAR (the binary-searched row list)
  FM  array-dominated, dense rows, shards 0..2: moves to the search chain when a far row id is put, and stays there after it
      is removed until the next full rebuild
  EX  the existence field (row 0), every shard
  V   int field (BSI view VV: exists, sign, DEPTH magnitude planes; negatives), shards 0, 1, 2 and FAR
FAR = 2^20 + 3 is only held by FC and FD (search chain anyway), EX and V (rows span at most 64, so 64 x (FAR + 1) entries
stay under the dense directory's 64M limit).  Shard 3 holds neither FC nor FD nor V.  Queries run over the contiguous shard
range [0, 3] and over [0, 2, 3, FAR] (pair_count_kernel's two shard-list forms).

Directed cases, each a scripted step that asserts it was reached:
  1. FB's striped fragment turned bitmap-heavy by an apply batch keeps striped arrays of >= 64 elements, so FB's Count stays on
     eval_kernel (test_striped_arrays_keep_count_off_wordpar); a bitmap-heavy fragment that gains arrays keeps them sorted.
  2. a load_fragments batch that fails half way (a shard id >= 2^24 after valid ones) between uncommitted updates: stats,
     routing and answers as before (test_failed_batch_between_updates).
  3. GroupBy FA x FA on groupby_direct_kernel's dense walk right after a patch commit rewrote those rows' directory slices.
  4. compaction with block-moved and gathered fragments, then apply batches on the compacted arena.
  5. FM moves to the search chain (full rebuild) and stays there after the far row is removed (patch commit).
The scripted prefix of the sequence runs all five; random steps follow."""
import ctypes as C
import os

import numpy as np
import pytest

from featurebase_b200 import lib as L
from oracle import oracle as O
from tests import archetypes as A
from tests.test_store_inspect import container_values

ON_EMU = bool(os.environ.get("FBGPU_TEST_ON_EMULATOR")) and not os.environ.get("FBGPU_EMU_FULL_SIZE")      # fewer steps, smaller containers
SW, W = 1 << 20, 1 << 16
IDX = 0
FA, FB, FC, FD, FM, EX, V = 1, 2, 3, 4, 5, 6, 7
VV = 3                                  # V's BSI view
SET_FIELDS = (FA, FB, FC, FD, FM, EX)
DEPTH = 20 if ON_EMU else 24
FAR = (1 << 20) + 3
SHARDS = [0, 1, 2, 3, FAR]
RANGE = [0, 1, 2, 3]                    # a contiguous shard range
GAPPED = [0, 2, 3, FAR]                 # a shard list with gaps and the far shard
C_ROW0 = 1_000_000
D_ROWS = [0, 7, 40000, 1 << 30]
M_FAR_ROW = 3_000_000
V_SLOTS = (0, 9)
BAD_SHARD = (1 << 24) + 5               # past the accepted shard range: the batch fails on it
STRIPE = not os.environ.get("FBGPU_ARRAY_SORTED")
GD_DIRECT = not os.environ.get("FBGPU_GROUPBY_CTA")
N_RANDOM = 6 if ON_EMU else 30
FULL_EVERY = 4
ENC = (O.ARRAY, O.BITMAP, O.RUN)
CMPS = ["==", "!=", "<", "<=", ">", ">=", "><"]
gpu = pytest.mark.gpu


# ------------------------------------------------------------------ containers
def values_of(rng, kind):
    """sorted unique in-container values of a kind"""
    small = ON_EMU
    if kind == "tiny":
        return np.sort(rng.choice(W, int(rng.integers(1, 50)), replace=False))
    if kind == "striped":                                    # stored bank-striped in an array-dominated fragment
        return np.sort(rng.choice(W, int(rng.integers(64, 400 if small else 1000)), replace=False))
    if kind == "bigarray":
        return np.sort(rng.choice(W, int(rng.integers(4097, 4500 if small else 9000)), replace=False))
    if kind == "dense":
        return np.sort(rng.choice(W, int(rng.integers(3000, 8000 if small else 30000)), replace=False))
    if kind == "onebit":
        return np.array([int(rng.integers(W))])
    if kind == "runs":
        starts = np.sort(rng.choice(W // 64, int(rng.integers(1, 12)), replace=False)) * 64
        return np.unique(np.concatenate([np.arange(s, s + int(rng.integers(1, 60))) for s in starts]))
    if kind == "manyruns":                                   # more than 2048 one-bit runs
        s = int(rng.integers(0, 1000))
        return np.arange(s, s + 2 * int(rng.integers(2049, 2300)), 2)
    raise KeyError(kind)


def cont(rng, kind, enc=None):
    """(values, encoding): the encoding drawn when not given"""
    v = np.asarray(values_of(rng, kind), dtype=np.int64)
    if enc is None:
        enc = {"tiny": O.ARRAY, "striped": O.ARRAY, "bigarray": O.ARRAY, "onebit": O.BITMAP, "manyruns": O.RUN}.get(kind) or ENC[int(rng.integers(3))]
    return v, enc


def n_runs(v):
    return 0 if len(v) == 0 else 1 + int(np.count_nonzero(np.diff(v) != 1))


def cont_bytes(v, enc):
    return 2 * len(v) if enc == O.ARRAY else 8192 if enc == O.BITMAP else 4 * n_runs(v)


def frag_bytes(conts):
    b = O.Bitmap()
    for k in sorted(conts):
        v, enc = conts[k]
        b.put(k, A.container_of(v, enc))
    return b.to_bytes(optimize=False)


# ------------------------------------------------------------------ the model
class Model:
    """(field, view, shard) -> {key: (values, encoding)}, each fragment's stripe policy (decided when it is created, kept by
    updates, as the library does) and whether it holds holes (gathered container by container at compaction)"""

    def __init__(self):
        self.frags, self.policy, self.holed = {}, {}, {}
        self._cache = {}

    def _created(self, fk, conts):
        n_arr = sum(1 for v, e in conts.values() if e == O.ARRAY)
        self.policy[fk] = STRIPE and n_arr * 8 > len(conts) - n_arr

    def load(self, f, v, s, conts):
        self._cache.clear()
        fk = (f, v, s)
        self.frags[fk] = dict(conts)
        self._created(fk, conts)
        self.holed[fk] = False

    def apply(self, f, v, s, put, removed):
        self._cache.clear()
        fk = (f, v, s)
        cur = self.frags.get(fk)
        if cur is None:
            if put:
                self.load(f, v, s, put)
            return
        new = {k: c for k, c in cur.items() if k not in removed and k not in put}
        new.update(put)
        if not new:
            self.drop(f, v, s)
            return
        self.frags[fk] = new
        self.holed[fk] = True

    def drop(self, f, v, s):
        self._cache.clear()
        for d in (self.frags, self.policy, self.holed):
            d.pop((f, v, s), None)

    def compacted(self):
        self.holed = {k: False for k in self.holed}

    def stats(self):
        st = dict(fragments=len(self.frags), containers=0, array_containers=0, bitmap_containers=0, run_containers=0, payload_bytes=0)
        name = {O.ARRAY: "array_containers", O.BITMAP: "bitmap_containers", O.RUN: "run_containers"}
        for conts in self.frags.values():
            for v, e in conts.values():
                st["containers"] += 1
                st[name[e]] += 1
                st["payload_bytes"] += cont_bytes(v, e)
        return st

    def frag_stats(self, fk):
        """(arrays, bitmaps + runs, arrays stored bank-striped) of one fragment, as the library counts them"""
        conts = self.frags[fk]
        arr = sum(1 for v, e in conts.values() if e == O.ARRAY)
        striped = sum(1 for v, e in conts.values() if e == O.ARRAY and len(v) >= 64) if self.policy[fk] else 0
        return arr, len(conts) - arr, striped

    def view_stats(self, f, v=0):
        t = np.zeros(3, dtype=np.int64)
        for fk in self.frags:
            if fk[:2] == (f, v):
                t += self.frag_stats(fk)
        return tuple(int(x) for x in t)

    def wordpar(self, fields):
        """eval_wordpar_kernel's condition for a Count program over these set fields (view 0)"""
        arr, other, striped = (sum(x) for x in zip(*[self.view_stats(f) for f in set(fields)]))
        return striped == 0 and other > 0 and arr * 8 <= other

    def direct(self, fa, fb, shards):
        """groupby_direct_eligible for a two-field GroupBy over view 0"""
        if not GD_DIRECT:
            return False
        for f in (fa, fb):
            arr, other, _ = self.view_stats(f)
            if other * 8 > arr:
                return False
        elems = seen = 0
        for s in shards[::max(1, len(shards) // 64)]:
            conts = self.frags.get((fa, 0, s))
            if conts:
                elems += sum(cont_bytes(v, e) for v, e in conts.values()) // 2
                seen += 1
        return not seen or (elems // seen) // 16 <= 8192

    def rows(self, f, v=0, shards=SHARDS):
        out = set()
        for s in shards:
            out |= {k // 16 for k in self.frags.get((f, v, s), {})}
        return sorted(out)

    def cols(self, f, row, shards, v=0):
        """absolute column ids of a row over the shards, ascending (shards ascending)"""
        ck = (f, v, row, tuple(shards))
        if ck not in self._cache:
            parts = []
            for s in shards:
                conts = self.frags.get((f, v, s))
                if not conts:
                    continue
                for slot in range(16):
                    c = conts.get(row * 16 + slot)
                    if c is not None:
                        parts.append(s * SW + slot * W + c[0])
            self._cache[ck] = np.concatenate(parts) if parts else np.zeros(0, dtype=np.int64)
        return self._cache[ck]

    def int_values(self, shards):
        """(columns, Python-int values) of V over the shards, ascending by column"""
        ck = ("int", tuple(shards))
        if ck not in self._cache:
            cols = self.cols(V, 0, shards, VV)
            mag = np.zeros(len(cols), dtype=np.int64)
            for i in range(DEPTH):
                mag |= np.isin(cols, self.cols(V, 2 + i, shards, VV), assume_unique=True).astype(np.int64) << i
            neg = np.isin(cols, self.cols(V, 1, shards, VV), assume_unique=True)
            self._cache[ck] = (cols, np.where(neg, -mag, mag))
        return self._cache[ck]


def slot_values(model, s, slot):
    """{local column: value} of V in one (shard, slot)"""
    cols, vals = model.int_values([s])
    sel = ((cols >> 16) & 15) == slot
    return {int(c) & 0xFFFF: int(x) for c, x in zip(cols[sel], vals[sel])}


def encode_slot(rng, values, slot):
    """{key: container} of V's rows (exists, sign, planes) in one slot holding the {local column: value} map"""
    out = {}
    cols = np.array(sorted(values), dtype=np.int64)
    vals = np.array([values[c] for c in cols.tolist()], dtype=np.int64)
    mag = np.abs(vals)
    rows = [(0, cols), (1, cols[vals < 0])] + [(2 + i, cols[((mag >> i) & 1) == 1]) for i in range(DEPTH)]
    for r, c in rows:
        if len(c):
            out[r * 16 + slot] = (c, ENC[int(rng.integers(3))])
    return out


# ------------------------------------------------------------------ the store under test and the model, side by side
class Store:
    """one library target (Context, Node or inspection-only Context) and the model, changed together"""

    def __init__(self, ctx, kind):
        self.ctx, self.kind, self.m = ctx, kind, Model()
        self.reached = set()

    def load(self, f, s, conts, v=0):
        self.ctx.load_fragment(IDX, f, v, s, frag_bytes(conts))
        self.m.load(f, v, s, conts)

    def load_batch(self, f, items, v=0, fail=False):
        if fail and self.kind == "node":                                 # (each member loads its share: keep the share that fails)
            items = [it for it in items if self.ctx.owner(it[0]) == self.ctx.owner(BAD_SHARD)]
            if not items:
                return
        shards = [s for s, _ in items] + ([BAD_SHARD] if fail else [])
        blobs = [frag_bytes(c) for _, c in items] + ([frag_bytes(items[0][1])] if fail else [])
        offs = np.concatenate([[0], np.cumsum([len(b) for b in blobs])]).astype(np.uint64)
        buf = np.frombuffer(b"".join(blobs), dtype=np.uint8)
        if fail:
            with pytest.raises(L.FbgpuError, match="too large"):
                self.ctx.load_fragments(IDX, f, v, shards, buf, offs)
            self.reached.add("load_fragments_failed")
            return
        self.ctx.load_fragments(IDX, f, v, shards, buf, offs)
        for s, c in items:
            self.m.load(f, v, s, c)
        self.reached.add("load_fragments")

    def apply(self, f, s, put, removed=(), v=0):
        fk = (f, v, s)
        old = self.m.frags.get(fk)
        removed = set(removed) - set(put)                                # (a key both written and removed is refused)
        self.ctx.apply_containers(IDX, f, v, s, frag_bytes(put) if put else b"", sorted(removed))
        rows_before = self.m.rows(f, v, SHARDS)
        self.m.apply(f, v, s, put, set(removed))
        self.reached.add("apply")
        kinds = self.reached
        for val, e in put.values():
            if e == O.ARRAY and len(val) > 4096:
                kinds.add("array>4096")
            if e == O.RUN and n_runs(val) > 2048:
                kinds.add("runs>2048")
            if e == O.BITMAP and len(val) == 1:
                kinds.add("one-bit bitmap")
        if old is None and put:
            kinds.add("apply_not_resident")
        if old is not None and set(removed) & set(old):
            kinds.add("apply_removes")
        if not put and removed:
            kinds.add("apply_removal_only")
        if old is not None and fk not in self.m.frags:
            kinds.add("apply_empties")
        if any(k // 16 not in rows_before for k in put):
            kinds.add("apply_new_row")

    def drop(self, f, s, v=0):
        self.ctx.drop_fragment(IDX, f, v, s)
        self.m.drop(f, v, s)
        self.reached.add("drop")

    def commit(self):
        self.ctx.commit()
        self.reached.add("commit")

    def compact(self):
        self.ctx.compact()
        self.m.compacted()
        self.reached.add("compact")

    def stats(self):
        return self.ctx.stats()

    def check_stats(self, after_compact=False):
        st = self.ctx.stats()
        exp = self.m.stats()
        assert {k: st[k] for k in exp} == exp
        if after_compact and self.kind == "ctx":
            assert st["dead_bytes"] == 0, st


# ------------------------------------------------------------------ the world
def initial_world(st, rng):
    m = lambda *a: cont(rng, *a)
    # FA: arrays (most of 64 or more elements: striped), rows 0..5, a slot or three per row
    for s in RANGE:
        st.load(FA, s, {r * 16 + int(sl): m(str(rng.choice(["striped", "striped", "tiny"])), O.ARRAY)
                        for r in range(6) for sl in rng.choice(16, int(rng.integers(1, 4)), replace=False)})
    # FB: bitmap / run heavy in shards 0..2 (one batch), array-dominated with striped arrays in shard 3
    heavy = lambda: {r * 16 + int(sl): m(str(rng.choice(["dense", "runs", "dense"])), [O.BITMAP, O.RUN][int(rng.integers(2))])
                     for r in range(6) for sl in rng.choice(16, 4, replace=False)}
    st.load_batch(FB, [(s, heavy()) for s in (0, 1, 2)])
    # FC: contiguous rows in each fragment, far apart across the view
    for s, r0 in ((0, 0), (2, C_ROW0), (FAR, C_ROW0 + 2)):
        st.load(FC, s, {(r0 + r) * 16 + int(sl): m(str(rng.choice(["striped", "tiny"])), O.ARRAY) for r in range(5) for sl in rng.choice(16, 2, replace=False)})
    # FD: sparse rows
    for s in (0, 1, FAR):
        st.load(FD, s, {r * 16 + int(sl): m(str(rng.choice(["striped", "tiny"])), O.ARRAY) for r in D_ROWS for sl in rng.choice(16, 2, replace=False)})
    for s in (0, 1, 2):
        st.load(FM, s, {r * 16 + int(sl): m("striped", O.ARRAY) for r in range(5) for sl in rng.choice(16, 2, replace=False)})
    for s in SHARDS:
        st.load(EX, s, {int(sl): m(str(rng.choice(["dense", "runs", "striped"]))) for sl in rng.choice(16, 6, replace=False)})
    n = 200 if ON_EMU else 1500
    for s in (0, 1, 2, FAR):
        conts = {}
        for slot in V_SLOTS:
            cols = rng.choice(W, n, replace=False).tolist()
            conts.update(encode_slot(rng, dict(zip(cols, rand_values(rng, n))), slot))
        st.load(V, s, conts, v=VV)


def rand_values(rng, n):
    """int values of V: the full signed range of the depth, a fifth of them small (repeated values, zeros)"""
    hi = (1 << DEPTH) - 1
    v = rng.integers(-hi, hi + 1, n)
    small = rng.random(n) < 0.2
    v[small] = rng.integers(-40, 40, int(small.sum()))
    return [int(x) for x in v]


# ------------------------------------------------------------------ mutations
def put_in(rng, st, f, s, n, kinds, rows, enc=None):
    """n containers of the given kinds in the given rows of one fragment (replacing or adding)"""
    out = {}
    for _ in range(n):
        r = int(rng.choice(rows))
        out[r * 16 + int(rng.integers(16))] = cont(rng, str(rng.choice(kinds)), enc)
    return out


def change_int_values(rng, st, s=None):
    """rewrite a few values of V in one (shard, slot): changed, new and cleared columns, applied as plane containers"""
    if s is None:
        s = int(rng.choice([x for x in (0, 1, 2, FAR) if (V, VV, x) in st.m.frags] or [0]))
    slot = int(rng.choice(V_SLOTS))
    vals = slot_values(st.m, s, slot)
    cols = list(vals)
    for c in rng.choice(cols, min(len(cols), 20), replace=False).tolist() if cols else []:
        vals[c] = rand_values(rng, 1)[0]
    for c in rng.choice(cols, min(len(cols), 5), replace=False).tolist() if cols else []:
        vals.pop(c, None)
    for c, x in zip(rng.choice(W, 10, replace=False).tolist(), rand_values(rng, 10)):
        vals[c] = x
    put = encode_slot(rng, vals, slot)
    old = {k for k in st.m.frags.get((V, VV, s), {}) if k % 16 == slot}
    st.apply(V, s, put, old - set(put), v=VV)
    st.reached.add("int_values")


def random_step(rng, st, can_compact):
    kinds = ["apply", "apply", "apply", "int", "load", "batch", "drop", "commit"] + (["compact"] if can_compact else [])
    k = str(rng.choice(kinds))
    f = int(rng.choice([FA, FB, FC, FD, FM, EX]))
    own = {FA: RANGE, FB: RANGE, FC: [0, 2, FAR], FD: [0, 1, FAR], FM: [0, 1, 2], EX: SHARDS}[f]
    s = int(rng.choice(own))
    rows = st.m.rows(f) or [0]
    pal = {FB: ["dense", "runs", "onebit", "manyruns", "striped"]}.get(f, ["tiny", "striped", "striped", "bigarray", "onebit", "runs"])
    if k == "apply":
        put = put_in(rng, st, f, s, int(rng.integers(1, 5)), pal, rows + [max(rows) + 1])
        keys = list(st.m.frags.get((f, 0, s), {}))
        removed = set(int(x) for x in rng.choice(keys, min(len(keys), int(rng.integers(0, 3))), replace=False)) - set(put) if keys else set()
        st.apply(f, s, put, removed)
        return f"apply {f}/{s}"
    if k == "int":
        change_int_values(rng, st)
        return "int values"
    if k == "load":
        st.load(f, s, put_in(rng, st, f, s, int(rng.integers(2, 8)), pal, rows))
        st.reached.add("load_fragment")
        return f"load {f}/{s}"
    if k == "batch":
        items = [(x, put_in(rng, st, f, x, int(rng.integers(2, 6)), pal, rows)) for x in sorted(rng.choice(own, min(2, len(own)), replace=False).tolist())]
        st.load_batch(f, items, fail=bool(rng.random() < 0.3))
        return f"batch {f}"
    if k == "drop":
        if len([x for x in own if (f, 0, x) in st.m.frags]) > 1:
            st.drop(f, s)
        return f"drop {f}/{s}"
    if k == "compact":
        st.compact()
        return "compact"
    st.commit()
    return "commit"


# ------------------------------------------------------------------ the battery
def row_op(f, r, v=0):
    return L.Op(L.OP_ROW, f, v, 0, r, 0, 0, 0)


def nary(op, *xs):
    """program node: (ops, expected columns over the shards) from (ops, columns) children"""
    ops = [o for x in xs for o in x[0]] + [L.Op(op, 0, 0, len(xs), 0, 0, 0, 0)]
    cols = xs[0][1]
    for x in xs[1:]:
        if op == L.OP_INTERSECT:
            cols = np.intersect1d(cols, x[1], assume_unique=True)
        elif op == L.OP_UNION:
            cols = np.union1d(cols, x[1])
        elif op == L.OP_DIFFERENCE:
            cols = np.setdiff1d(cols, x[1], assume_unique=True)
        else:
            cols = np.setxor1d(cols, x[1], assume_unique=True)
    return ops, cols


def query_rows(m, f, shards=SHARDS):
    """the field's rows and rows it does not hold: just past its largest row, well past it, and (dense fields) past the rows
    the directory covers, so groupby_direct_kernel's dense walk meets row ids outside its range"""
    rows = m.rows(f, 0, shards) or [0]
    extra = [rows[-1] + 1, rows[-1] + 2, rows[-1] + 5, rows[-1] + 1000]
    return sorted(set(rows) | set(extra))[:14]


def check_counts(st, shards, rng):
    m, ctx = st.m, st.ctx
    R = lambda f, r: ([row_op(f, r)], m.cols(f, r, shards))
    a = [int(x) for x in rng.choice(query_rows(m, FA), 2)]
    b = [int(x) for x in rng.choice(query_rows(m, FB), 3)]
    c, d = int(rng.choice(query_rows(m, FC))), int(rng.choice(query_rows(m, FD)))
    progs = [nary(L.OP_INTERSECT, R(FA, a[0]), R(FB, b[0])),                                   # pair kernel shape
             nary(L.OP_INTERSECT, R(FA, a[0]), R(FA, a[1])),
             nary(L.OP_DIFFERENCE, nary(L.OP_UNION, R(FA, a[1]), R(FC, c), R(FD, d)), R(FB, b[1])),
             nary(L.OP_UNION, nary(L.OP_INTERSECT, R(FB, b[0]), R(FB, b[1])), R(FB, b[2])),    # the bitmap-heavy field alone
             nary(L.OP_XOR, R(FB, 0), R(FB, 3)), R(FB, 0), R(FB, 1),
             nary(L.OP_INTERSECT, R(EX, 0), R(FM, int(rng.choice(query_rows(m, FM)))))]
    for ops, exp in progs:
        assert ctx.count(IDX, ops, shards) == len(exp), (ops[0].field, shards)
    return progs


def check_full(st, shards, rng):
    m, ctx, node = st.m, st.ctx, st.kind == "node"
    progs = check_counts(st, shards, rng)
    # Row bytes (canonical), Columns in windows, Any
    for ops, exp in progs[2:4] + [([row_op(FD, 1 << 30)], m.cols(FD, 1 << 30, shards))]:
        data, cnt = ctx.row(IDX, ops, shards)
        assert cnt == len(exp) and data == O.Bitmap.from_values(exp.astype(np.uint64)).to_bytes(), shards
        assert ctx.any(IDX, ops, shards) == (len(exp) > 0)
        if not node:
            n = len(exp)
            for off, lim in ((0, None), (n // 3, max(n // 3, 1)), (max(n - 2, 0), 5), (n + 1, 2)):
                got, total = ctx.columns(IDX, ops, shards, offset=off, limit=lim)
                assert (got.tolist(), total) == (exp[off: None if lim is None else off + lim].tolist(), n), (off, lim)
    assert not ctx.any(IDX, [row_op(FA, 999)], shards)
    # row counts
    ex = m.cols(EX, 0, shards)
    for f in SET_FIELDS:
        rows = query_rows(m, f, shards)
        per = np.array([[len(m.cols(f, r, [s])) for r in rows] for s in shards], dtype=np.int64)
        assert ctx.row_counts(IDX, f, 0, shards, row_ids=rows).tolist() == per.sum(axis=0).tolist(), f
        filt = np.array([[len(np.intersect1d(m.cols(f, r, [s]), ex, assume_unique=True)) for r in rows] for s in shards], dtype=np.int64)
        assert ctx.row_counts(IDX, f, 0, shards, row_ids=rows, filter_ops=[row_op(EX, 0)]).tolist() == filt.sum(axis=0).tolist(), f
        if not node:
            assert ctx.row_counts_per_shard(IDX, f, 0, shards, rows).tolist() == per.tolist(), f
            assert ctx.row_counts_per_shard(IDX, f, 0, shards, rows, filter_ops=[row_op(EX, 0)]).tolist() == filt.tolist(), f
            rid, cnt = ctx.row_counts(IDX, f, 0, shards)
            exp = sorted(((r, int(x)) for r, x in zip(rows, per.sum(axis=0).tolist()) if x), key=lambda rc: (-rc[1], rc[0]))
            assert list(zip(rid.tolist(), cnt.tolist())) == exp, f
    # count_pairs, pair_types
    for fa, fb in ((FA, FB), (FC, FD), (FM, FA)):
        ra, rb = query_rows(m, fa, shards), query_rows(m, fb, shards)
        pa = [int(x) for x in rng.choice(ra, 6)]
        pb = [int(x) for x in rng.choice(rb, 6)]
        exp = [len(np.intersect1d(m.cols(fa, x, shards), m.cols(fb, y, shards), assume_unique=True)) for x, y in zip(pa, pb)]
        assert ctx.count_pairs(IDX, fa, 0, pa, fb, 0, pb, shards).tolist() == exp, (fa, fb)
        if not node:
            hist = np.zeros((4, 4), dtype=np.int64)
            for s in shards:
                for slot in range(16):
                    ta, tb = (m.frags.get((f, 0, s), {}).get(r * 16 + slot, (None, 0))[1] for f, r in ((fa, pa[0]), (fb, pb[0])))
                    hist[ta, tb] += 1
            assert ctx.pair_types(IDX, fa, 0, pa[0], fb, 0, pb[0], shards).tolist() == hist.tolist(), (fa, fb)
    check_groupby(st, shards, rng)
    check_int(st, shards, rng)


def gb_expect(m, dims, shards, keep=None):
    """GroupBy counts: dims [(field, rows)] -> int64 tensor"""
    out = np.zeros([len(r) for _, r in dims], dtype=np.int64)
    for s in shards:
        sets = [[m.cols(f, r, [s]) for r in rows] for f, rows in dims]
        if keep is not None:
            sets[0] = [np.intersect1d(x, keep, assume_unique=True) for x in sets[0]]

        def rec(level, acc, idx):
            if level == len(sets):
                out[tuple(idx)] += len(acc)
                return
            for j, x in enumerate(sets[level]):
                y = x if acc is None else np.intersect1d(acc, x, assume_unique=True)
                if len(y):
                    rec(level + 1, y, idx + [j])
        rec(0, None, [])
    return out


# directory forms: FA / FB / FM dense, FC the contiguous search chain, FD the binary-searched row list
GB_PAIRS = [(FA, FA), (FA, FB), (FA, FC), (FC, FD), (FD, FA), (FD, FD), (FM, FC)]
GB_TRIPLES = [(FB, FA, FC), (FA, FD, FA)]


def check_groupby(st, shards, rng, pairs=GB_PAIRS, triples=GB_TRIPLES):
    m, ctx = st.m, st.ctx
    ex = m.cols(EX, 0, shards)
    for dims_f in list(pairs) + list(triples):
        dims = [(f, query_rows(m, f, shards)[: 10 if len(dims_f) == 2 else 5]) for f in dims_f]
        for flt, keep in ((None, None), ([row_op(EX, 0)], ex)):
            before = ctx.counters() if st.kind == "ctx" else None
            got = ctx.groupby(IDX, list(dims_f), [0] * len(dims_f), [r for _, r in dims], shards, filter_ops=flt)
            assert np.array_equal(got.astype(np.int64), gb_expect(m, dims, shards, keep)), (dims_f, flt is not None, shards)
            if before is not None and len(dims_f) == 2:
                units = ctx.counters()["groupby_units"] - before["groupby_units"]
                direct = m.direct(dims_f[0], dims_f[1], shards)
                assert units == (16 * len(shards) if direct else 0), (dims_f, direct)
                if direct and dims_f == (FA, FA):
                    st.reached.add("groupby_direct_dense")


def check_int(st, shards, rng):
    m, ctx, node = st.m, st.ctx, st.kind == "node"
    cols, vals = m.int_values(shards)
    a = int(rng.choice(query_rows(m, FA, shards)[:-2]))
    fa = m.cols(FA, a, shards)
    for flt, keep in ((None, None), ([row_op(FA, a)], fa)):
        sel = np.ones(len(cols), dtype=bool) if keep is None else np.isin(cols, keep, assume_unique=True)
        cs, vs = cols[sel].tolist(), [int(x) for x in vals[sel].tolist()]
        n = len(vs)
        assert ctx.bsi_sum(IDX, V, VV, DEPTH, shards, filter_ops=flt) == (sum(vs), n)
        for want_max in (False, True):
            e = (max(vs) if want_max else min(vs)) if vs else 0
            assert ctx.bsi_minmax(IDX, V, VV, DEPTH, shards, want_max, filter_ops=flt) == ((e, vs.count(e)) if vs else (0, 0)), want_max
        if node:
            continue
        c, v, total = ctx.extract(IDX, V, VV, DEPTH, shards, filter_ops=flt)
        assert (c.tolist(), v.tolist(), total) == (cs, vs, n)
        off, lim = n // 3, max(n // 4, 1)
        c, v, total = ctx.extract(IDX, V, VV, DEPTH, shards, filter_ops=flt, offset=off, limit=lim)
        assert (c.tolist(), v.tolist(), total) == (cs[off:off + lim], vs[off:off + lim], n)
        if n:
            s = sorted(vs)
            rk = sorted({0, n // 3, n // 2, n - 1})
            got, cnt, total = ctx.bsi_select(IDX, V, VV, DEPTH, shards, rk, filter_ops=flt)
            assert total == n and got.tolist() == [s[r] for r in rk] and cnt.tolist() == [vs.count(s[r]) for r in rk], rk
    # each comparison, as a filter of Count, of Sum and of row counts
    present = sorted(set(int(x) for x in vals.tolist())) or [0]
    p = sorted(int(x) for x in rng.choice(present, 2))
    for cmp in CMPS:
        lo, hi = (p[0], p[1]) if cmp == "><" else (p[int(rng.integers(2))], 0)
        match = {"==": vals == lo, "!=": vals != lo, "<": vals < lo, "<=": vals <= lo, ">": vals > lo, ">=": vals >= lo, "><": (vals >= lo) & (vals <= hi)}[cmp]
        rop = L.Op(L.OP_BSI_RANGE, V, VV, 0, DEPTH, L.CMP[cmp], lo, hi)
        hit = cols[match]
        assert ctx.count(IDX, [rop], shards) == len(hit), cmp
        assert ctx.count(IDX, [row_op(FA, a), rop, L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)], shards) == len(np.intersect1d(hit, fa, assume_unique=True)), cmp
        assert ctx.bsi_sum(IDX, V, VV, DEPTH, shards, filter_ops=[rop]) == (sum(int(x) for x in vals[match].tolist()), len(hit)), cmp
        rows = query_rows(m, FA, shards)[:6]
        assert ctx.row_counts(IDX, FA, 0, shards, row_ids=rows, filter_ops=[rop]).tolist() == \
            [len(np.intersect1d(m.cols(FA, r, shards), hit, assume_unique=True)) for r in rows], cmp
    # groupby_values: FA rows x values (present ones, absent ones)
    rows = query_rows(m, FA, shards)[:6]
    pick = sorted(set(int(x) for x in rng.choice(present, min(len(present), 150), replace=False)) | {-(1 << DEPTH) + 1, 123456789 % (1 << DEPTH)})
    pos = {x: j for j, x in enumerate(pick)}
    for flt, keep in ((None, None), ([row_op(EX, 0)], m.cols(EX, 0, shards))):
        exp = np.zeros((len(rows), len(pick)), dtype=np.int64)
        for i, r in enumerate(rows):
            rc = m.cols(FA, r, shards) if keep is None else np.intersect1d(m.cols(FA, r, shards), keep, assume_unique=True)
            for x in vals[np.isin(cols, rc, assume_unique=True)].tolist():
                if int(x) in pos:
                    exp[i, pos[int(x)]] += 1
        got = ctx.groupby_values(IDX, [FA], [0], [rows], V, VV, DEPTH, pick, shards, filter_ops=flt)
        assert np.array_equal(got.astype(np.int64), exp), flt is not None


def battery(st, rng, full, step):
    """the full battery on both shard lists, or the Count programs on one of them"""
    if st.kind == "inspect":
        return check_inspect(st)
    if full:
        for shards in (RANGE, GAPPED):
            check_full(st, shards, rng)
    else:
        check_counts(st, RANGE if step % 2 else GAPPED, rng)


# ------------------------------------------------------------------ inspection-only twin
def debug_container(ctx, f, v, s, row, slot, buf=np.empty(1 << 18, dtype=np.uint8)):
    typ, card, runs, n = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)
    rc = ctx.L.fbgpu_debug_container(ctx.h, IDX, f, v, int(s), int(row), int(slot), C.byref(typ), C.byref(card), C.byref(runs), buf.ctypes.data, len(buf), C.byref(n))
    assert rc == 0, ctx.L.fbgpu_last_error()
    return None if typ.value == 0 else (typ.value, card.value, runs.value, buf[: n.value].tobytes())


def check_inspect(st):
    """every container of the model where it belongs, in its encoding; absent keys of every row the field ever held, and past
    them, resolve to nothing"""
    m, ctx = st.m, st.ctx
    for (f, v, s), conts in m.frags.items():
        for k, (vals, enc) in conts.items():
            got = debug_container(ctx, f, v, s, k // 16, k % 16)
            assert got is not None and got[0] == enc and np.array_equal(container_values(got), vals), (f, v, s, k)
    for f, v in [(x, 0) for x in SET_FIELDS] + [(V, VV)]:
        st.seen_rows.setdefault((f, v), set()).update(m.rows(f, v))
        rows = sorted(st.seen_rows[(f, v)])
        for s in SHARDS + [4]:
            conts = m.frags.get((f, v, s), {})
            for r in rows + [rows[-1] + 1 if rows else 0]:
                for slot in range(16):
                    if r * 16 + slot not in conts:
                        assert debug_container(ctx, f, v, s, r, slot) is None, (f, v, s, r, slot)


# ------------------------------------------------------------------ the sequence
def scripted(st, rng, can_compact):
    """the directed steps: yields (name, full battery after it)"""
    m = st.m
    # case 1, reverse: a bitmap-heavy fragment gains arrays of 64 or more elements; they stay sorted, so Count on FB stays on wordpar
    st.apply(FB, 0, {k: cont(rng, "striped", O.ARRAY) for k in list(m.frags[(FB, 0, 0)])[:2]})
    arr, other, striped = m.view_stats(FB)
    assert not m.policy[(FB, 0, 0)] and arr == 2 and striped == 0 and m.wordpar([FB])
    yield "bitmap-heavy fragment gains arrays", False
    # an array-dominated fragment of FB: its arrays are stored bank-striped, which keeps FB's Count off wordpar
    st.load(FB, 3, {r * 16 + 4: cont(rng, "striped", O.ARRAY) for r in range(3)})
    assert m.policy[(FB, 0, 3)] and m.view_stats(FB)[2] == 3 and not m.wordpar([FB])
    yield "striped fragment in a bitmap-heavy view", False
    # case 1: the striped fragment of FB turned bitmap-heavy by an apply batch, its striped arrays left in place
    st.apply(FB, 3, {r * 16 + sl: cont(rng, "dense", [O.BITMAP, O.RUN][sl % 2]) for r in range(6) for sl in (1, 2, 3, 5) + ((4,) if r >= 3 else ())})
    a3, o3, s3 = m.frag_stats((FB, 0, 3))
    arr, other, striped = m.view_stats(FB)
    assert m.policy[(FB, 0, 3)] and a3 * 8 <= o3 and s3 == 3 and other > 0 and arr * 8 <= other
    st.reached.add("case1")
    yield "striped arrays left in a bitmap-heavy view", True
    # a pending update, a batch that fails half way through, another update: all as before, routing included
    before = st.stats()
    st.apply(FA, 1, put_in(rng, st, FA, 1, 2, ["striped"], [0, 1, 2]))
    mid = st.stats()
    st.load_batch(FB, [(3, {r * 16 + 4: cont(rng, "dense", O.BITMAP) for r in range(6)}), (1, {r * 16 + 7: cont(rng, "dense", O.BITMAP) for r in range(6)})], fail=True)
    assert st.stats() == mid and st.stats()["patch_commits"] == before["patch_commits"]
    st.apply(FB, 2, put_in(rng, st, FB, 2, 2, ["dense"], [0, 1]))
    st.reached.add("case2")
    yield "failed batch between updates", True
    # case 3: rows of FA rewritten in place, committed as a patch, then read by groupby_direct_kernel's dense walk
    for s in (1, 2):
        keys = list(m.frags[(FA, 0, s)])
        st.apply(FA, s, put_in(rng, st, FA, s, 3, ["striped", "tiny"], [1, 2, 3, 4], O.ARRAY), set(keys[:2]))
    before = st.stats()
    st.commit()
    after = st.stats()
    assert after["patch_commits"] > before["patch_commits"] and after["full_commits"] == before["full_commits"], (before, after)
    if st.kind != "inspect":
        if st.kind == "ctx":
            assert m.direct(FA, FA, RANGE) and m.direct(FA, FA, GAPPED)
        check_groupby(st, RANGE, rng, pairs=[(FA, FA)], triples=[])
        check_groupby(st, GAPPED, rng, pairs=[(FA, FA)], triples=[])
        assert st.kind != "ctx" or "groupby_direct_dense" in st.reached
    st.reached.add("case3")
    yield "patched rows read by the direct GroupBy", False
    # case 5: a far row id moves FM onto the search chain (a full rebuild); removing it leaves FM there (a patch)
    before = st.stats()
    st.apply(FM, 1, {M_FAR_ROW * 16 + 3: cont(rng, "striped", O.ARRAY)})
    st.commit()
    mid = st.stats()
    assert mid["full_commits"] == before["full_commits"] + 1, (before, mid)
    yield "far row puts FM on the search chain", True
    st.apply(FM, 1, {}, {M_FAR_ROW * 16 + 3})
    st.commit()
    after = st.stats()
    assert after["full_commits"] == mid["full_commits"] and after["patch_commits"] == mid["patch_commits"] + 1, (mid, after)
    st.reached.add("case5")
    yield "far row removed, FM stays on the search chain", True
    # the other mutation kinds once each
    st.load(FC, 2, {(C_ROW0 + r) * 16 + 5: cont(rng, "striped", O.ARRAY) for r in range(4)})
    st.reached.add("load_fragment")
    st.load_batch(FD, [(0, {r * 16 + 2: cont(rng, "tiny") for r in D_ROWS}), (FAR, {r * 16 + 9: cont(rng, "striped", O.ARRAY) for r in D_ROWS[1:]})])
    yield "fragments replaced", False
    st.apply(FA, 0, {0 * 16 + 3: cont(rng, "bigarray"), 1 * 16 + 3: cont(rng, "manyruns"), 2 * 16 + 3: cont(rng, "onebit"), 20 * 16 + 1: cont(rng, "tiny")},
             {list(m.frags[(FA, 0, 0)])[-1]})                             # row 20: outside FA's dense directory (a full rebuild)
    st.apply(FA, 3, {}, set(list(m.frags[(FA, 0, 3)])[:2]))              # removal only
    st.apply(FM, 2, {}, set(m.frags[(FM, 0, 2)]))                       # empties the fragment
    st.apply(FC, 3, {C_ROW0 * 16 + 1: cont(rng, "striped", O.ARRAY)})    # a shard FC does not hold
    change_int_values(rng, st, FAR)
    change_int_values(rng, st, 0)
    yield "apply batches of every kind", True                           # (the queries commit them)
    st.reached.add("implicit_commit")
    st.drop(FD, 1)
    st.commit()
    yield "drop", False
    if can_compact:
        # case 4: clean fragments move as blocks, updated ones are gathered; then batches land on the compacted arena
        assert any(not h for h in m.holed.values()) and any(m.holed.values())
        st.compact()
        st.reached.add("case4")
        yield "compact", True
        st.apply(FA, 2, put_in(rng, st, FA, 2, 3, ["striped", "tiny"], [0, 1, 2, 3]), {list(m.frags[(FA, 0, 2)])[0]})
        st.apply(FB, 1, put_in(rng, st, FB, 1, 2, ["dense", "runs"], [0, 4]))
        change_int_values(rng, st, 1)
        yield "updates on the compacted arena", True


def run_sequence(st, seed, can_compact=True, n_random=N_RANDOM):
    rng = np.random.default_rng(seed)
    qrng = np.random.default_rng(seed + 1)
    st.seen_rows = {}
    initial_world(st, rng)
    st.commit()
    st.check_stats()
    start = st.stats()
    battery(st, qrng, True, 0)
    step = 0
    for name, full in scripted(st, rng, can_compact):
        step += 1
        st.check_stats(after_compact=name == "compact")
        battery(st, qrng, full, step)
    for i in range(n_random):
        step += 1
        name = random_step(rng, st, can_compact)
        st.check_stats(after_compact=name == "compact")
        battery(st, qrng, name == "compact" or i % FULL_EVERY == FULL_EVERY - 1, step)
    st.commit()
    battery(st, qrng, True, step + 1)
    end = st.stats()
    if st.kind != "inspect":
        assert end["patch_commits"] > start["patch_commits"] and end["full_commits"] > start["full_commits"], (start, end)
    want = {"apply", "array>4096", "runs>2048", "one-bit bitmap", "apply_not_resident", "apply_removes", "apply_removal_only", "apply_empties",
            "apply_new_row", "int_values", "load_fragment", "load_fragments", "load_fragments_failed", "drop", "commit", "implicit_commit",
            "case1", "case2", "case3", "case5"} | ({"compact", "case4"} if can_compact else set())
    assert want <= st.reached, want - st.reached


# ------------------------------------------------------------------ tests
@gpu
@pytest.mark.parametrize("seed", [11] if ON_EMU else [11, 12])
def test_store_lifecycle(seed):
    """the whole sequence on one device context: stats after every step, the Count programs after every step, the full battery
    every few steps and after compaction, GroupBy routed to the kernel the model's view statistics predict"""
    ctx = L.Context(0)
    try:
        run_sequence(Store(ctx, "ctx"), seed)
    finally:
        ctx.close()


@gpu
def test_striped_arrays_keep_count_off_wordpar():
    """case 1 alone: Count over FB while its bitmap-heavy view still holds bank-striped arrays (eval_kernel), before and after
    the batch that turned their fragment bitmap-heavy, and after a bitmap-heavy fragment gained sorted arrays"""
    ctx = L.Context(0)
    try:
        st = Store(ctx, "ctx")
        rng, qrng = np.random.default_rng(3), np.random.default_rng(4)
        st.seen_rows = {}
        initial_world(st, rng)
        steps = scripted(st, rng, True)
        for _ in range(3):
            next(steps)
            for shards in (RANGE, GAPPED):
                check_counts(st, shards, qrng)
        assert "case1" in st.reached
    finally:
        ctx.close()


@gpu
def test_failed_batch_between_updates():
    """case 2 alone: the same answers, stats and GroupBy routing after a batch that failed half way between two updates"""
    ctx = L.Context(0)
    try:
        st = Store(ctx, "ctx")
        rng, qrng = np.random.default_rng(5), np.random.default_rng(6)
        st.seen_rows = {}
        initial_world(st, rng)
        steps = scripted(st, rng, True)
        for _ in range(4):
            next(steps)
        st.check_stats()
        for shards in (RANGE, GAPPED):
            check_counts(st, shards, qrng)
            check_groupby(st, shards, qrng)
        assert "case2" in st.reached
    finally:
        ctx.close()


@gpu
def test_store_lifecycle_on_a_node():
    """the sequence without compact (it has no node form) through lib.Node([0, 0], 2): shards 0 and 1 live on one member,
    2, 3 and FAR on the other, each query merges both; the failing batch runs on the member that owns every shard of it"""
    node = L.Node([0, 0], 2)
    try:
        assert {node.owner(s) for s in SHARDS} == {0, 1} and node.owner(3) == node.owner(FAR)
        run_sequence(Store(node, "node"), 21, can_compact=False, n_random=N_RANDOM // 2)
    finally:
        node.close()


def test_store_lifecycle_tables_without_a_device():
    """the same sequence on an inspection-only context: after every step every model container resolves, through the tables a
    commit builds (dense directory, contiguous chain, binary-searched rows), to its values in its encoding, absent keys resolve
    to nothing, and the stats match"""
    ctx = L.Context(L.DEVICE_NONE)
    try:
        run_sequence(Store(ctx, "inspect"), 11)
    finally:
        ctx.close()


def test_store_lifecycle_on_interpreted_kernels():
    """the gpu tests on the interpreted kernels: fewer steps and smaller containers, or as on a GPU under FBGPU_EMU_FULL=1"""
    from tests.test_emu_kernels import FULL, run_on_emulator
    run_on_emulator(["tests/test_store_lifecycle.py"], env={"FBGPU_EMU_FULL_SIZE": "1"} if FULL else None, timeout=3000)
