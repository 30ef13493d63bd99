"""Host-side mirror of the reference's executor interface for the hot path (executor.go), above the C ABI.

Holder/Index/Field carry just the schema facts the path needs (field type, bsiGroup Base/BitDepth/Min/Max,
existence tracking); Executor.execute() walks a pql.Call tree exactly like executor.executeCall /
executeBitmapCallShard do, but instead of mapping a Go closure over shards it compiles each bitmap call into a
post-order fbgpu_op program and hands the whole shard batch to libfbgpu (one C-ABI call per PQL call).

In a real integration this layer stays in Go (INTEGRATION.md); it exists here because the Go toolchain is absent
and the parity tests should read like the reference's executor tests.  All reference cites are executor.go unless
noted."""
import itertools
import math

import numpy as np

from . import lib as L
from . import pql
from . import roaring_io
from . import timeq

SHARD_WIDTH = 1 << 20                    # shardwidth/helper.go:13
VIEW_STANDARD = 0                        # view.go:28 "standard"
VIEW_BSI = 1                             # view.go:30 "bsig_<field>"
EXISTENCE_FIELD = "_exists"              # holder.go:33
SCRATCH_FIELD = "_embedded"              # mirror-only: holds rows embedded in a query (ConstRow / Precomputed operands)


class Field:
    def __init__(self, fid, name, ftype="set", min=None, max=None, bit_depth=None, quantum=""):
        self.id, self.name, self.type = fid, name, ftype
        self.quantum = quantum if ftype == "time" else ""       # TimeQuantum "YMDH" (time.go:17)
        self.view_ids = {"standard": VIEW_STANDARD}              # view name -> the small id used in programs / residency calls
        if ftype == "int":
            self.min = -(1 << 63) if min is None else int(min)
            self.max = (1 << 63) - 1 if max is None else int(max)
            self.base = self.min if self.min > 0 else self.max if self.max < 0 else 0      # bsiBase field.go:2384
            if bit_depth is None:                                                            # field.go:2502-2512 (data driven)
                bit_depth = max_bitlen(abs(self.min - self.base), abs(self.max - self.base))
            self.bit_depth = int(bit_depth)

    def view_id(self, name, create=False):
        if name not in self.view_ids:
            if not create:
                return None
            self.view_ids[name] = 2 + sum(1 for v in self.view_ids.values() if v >= 2)      # 0 standard, 1 bsig, 2.. time views
        return self.view_ids[name]

    def views_by_time_range(self, t_from, t_to):
        """Field.viewsByTimeRange field.go:1063-1110 -> view names (clamped to the views that exist)"""
        if not self.quantum:
            raise QueryError(f"field {self.name} is not a time-field, 'from' and 'to' are not valid options for this field type")
        if t_from is None and t_to is None:
            return ["standard"]
        lo, hi = timeq.min_max_views([v for v in self.view_ids if v != "standard"], self.quantum)
        if not lo or not hi:
            return []
        t_min, t_max = timeq.time_of_view(lo, False), timeq.time_of_view(hi, True)
        if t_from is None or t_from < t_min:
            t_from = t_min
        if t_to is None or t_to > t_max:
            t_to = t_max
        return timeq.views_by_time_range("standard", t_from, t_to, self.quantum)

    # bsiGroup.bitDepthMin / bitDepthMax  field.go:2475-2482
    def bit_depth_min(self):
        return self.base - (1 << self.bit_depth) + 1

    def bit_depth_max(self):
        return self.base + (1 << self.bit_depth) - 1

    def base_value(self, op, value):
        """bsiGroup.baseValue field.go:2412-2446 -> (baseValue, outOfRange)"""
        lo, hi = self.bit_depth_min(), self.bit_depth_max()
        bv = 0
        if op in (">", ">="):
            if value > hi:
                return 0, True
            if value < lo:
                bv = lo - self.base - (1 if op == ">" else 0)
            else:
                bv = value - self.base
        elif op in ("<", "<="):
            if value < lo:
                return 0, True
            if value > hi:
                bv = hi - self.base + (1 if op == "<" else 0)
            else:
                bv = value - self.base
        elif op in ("==", "!="):
            if value < lo or value > hi:
                return 0, True
            bv = value - self.base
        return bv, False

    def base_value_between(self, lo, hi):
        """bsiGroup.baseValueBetween field.go:2449-2463"""
        mn, mx = self.bit_depth_min(), self.bit_depth_max()
        if hi < mn or lo > mx or hi < lo:
            return 0, 0, True
        return max(lo, mn) - self.base, min(hi, mx) - self.base, False


def max_bitlen(*vals):
    return max(int(v).bit_length() for v in vals)


class Index:
    def __init__(self, iid, name, track_existence=True):
        self.id, self.name, self.track_existence = iid, name, track_existence
        self.fields = {}
        self.shards = set()
        if track_existence:
            self.fields[EXISTENCE_FIELD] = Field(0, EXISTENCE_FIELD)

    def create_field(self, name, ftype="set", **kw):
        f = Field(len(self.fields) + (0 if self.track_existence else 1), name, ftype, **kw)
        self.fields[name] = f
        return f


class Holder:
    """Schema + residency front end: owns one libfbgpu context."""

    def __init__(self, ctx=None, device=0):
        self.ctx = ctx or L.Context(device)
        self.indexes = {}
        self._pending = {}

    def create_index(self, name, track_existence=True):
        idx = Index(len(self.indexes), name, track_existence)
        self.indexes[name] = idx
        return idx

    def import_roaring(self, index, field, view, shard, data):
        """API.ImportRoaring analogue: one fragment's Pilosa-roaring bytes (keys row*16+slot)"""
        idx = self.indexes[index]
        self.ctx.load_fragment(idx.id, idx.fields[field].id, view, shard, data)
        idx.shards.add(int(shard))

    def apply_containers(self, index, field, view, shard, data=b"", removed_keys=()):
        """a committed write transaction's container changes to one fragment (Tx.PutContainer / RemoveContainer, tx.go:91-96): `data`
        holds only the written containers, removed_keys the deleted ones; untouched containers stay where they are in HBM"""
        idx = self.indexes[index]
        self.ctx.apply_containers(idx.id, idx.fields[field].id, view, shard, data, removed_keys)
        idx.shards.add(int(shard))

    def import_rbf(self, index, shard, data, wal=b""):
        """residency straight from a shard's RBF database bytes (SURVEY §8 f1): every field/view of this index that the
        file holds under its rbfName "~field;view<" (rbf.go:504; views "standard" view.go:28 and "bsig_<field>" :30)"""
        idx = self.indexes[index]
        names, fields, views = [], [], []
        for f in idx.fields.values():
            view = VIEW_BSI if f.type == "int" else VIEW_STANDARD
            names.append("~%s;%s<" % (f.name, "bsig_" + f.name if view == VIEW_BSI else "standard"))
            fields.append(f.id)
            views.append(view)
        n = self.ctx.load_rbf(idx.id, shard, data, names, fields, views, wal)
        if n:
            idx.shards.add(int(shard))
        return n

    # ---- test conveniences mirroring test helpers (hldr.SetBit / SetValue, test/holder.go)
    def set_bit(self, index, field, row, col, timestamp=None):
        idx = self.indexes[index]
        shard = col // SHARD_WIDTH
        self._pending.setdefault((index, field, VIEW_STANDARD, shard), set()).add(row * SHARD_WIDTH + col % SHARD_WIDTH)
        if timestamp is not None:                                # Set(col, f=row, timestamp): one more bit per quantum unit view (viewsByTime)
            f = idx.fields[field]
            for vname in timeq.views_by_time("standard", timeq.parse_time(timestamp), f.quantum):
                self._pending.setdefault((index, field, f.view_id(vname, create=True), shard), set()).add(row * SHARD_WIDTH + col % SHARD_WIDTH)
        if idx.track_existence:
            self._pending.setdefault((index, EXISTENCE_FIELD, VIEW_STANDARD, shard), set()).add(col % SHARD_WIDTH)

    def set_value(self, index, field, col, value):
        """fragment.setValue fragment.go:619-657: exists row 0, sign row 1, magnitude bits rows 2+i of value-Base"""
        idx = self.indexes[index]
        f = idx.fields[field]
        shard, c = col // SHARD_WIDTH, col % SHARD_WIDTH
        d = int(value) - f.base
        if abs(d).bit_length() > f.bit_depth:
            raise ValueError("value out of bit depth")
        s = self._pending.setdefault((index, field, VIEW_BSI, shard), set())
        s.add(c)
        if d < 0:
            s.add(1 * SHARD_WIDTH + c)
        for i in range(f.bit_depth):
            if (abs(d) >> i) & 1:
                s.add((2 + i) * SHARD_WIDTH + c)
        if idx.track_existence:
            self._pending.setdefault((index, EXISTENCE_FIELD, VIEW_STANDARD, shard), set()).add(c)

    def embed_row(self, index, columns):
        """A caller-provided operand row (pql ConstRow, or the *Row a Precomputed call carries per shard,
        executePrecomputedCallShard :5535): stored as the next row of a hidden scratch field, whose touched shards are
        re-sent through the normal residency call, and then addressed by an ordinary Row op.  Returns (field, row id)."""
        idx = self.indexes[index]
        f = idx.fields.get(SCRATCH_FIELD) or idx.create_field(SCRATCH_FIELD)
        store = self.__dict__.setdefault("_scratch", {}).setdefault(index, {})          # shard -> set of fragment positions
        row = self.__dict__.setdefault("_scratch_rows", {}).get(index, 0)
        self._scratch_rows[index] = row + 1
        touched = set()
        for col in columns:
            col = int(col)
            store.setdefault(col // SHARD_WIDTH, set()).add(row * SHARD_WIDTH + col % SHARD_WIDTH)
            touched.add(col // SHARD_WIDTH)
        for shard in touched:
            bits = store[shard]
            self.ctx.load_fragment(idx.id, f.id, VIEW_STANDARD, shard, roaring_io.encode(np.fromiter(bits, dtype=np.uint64, count=len(bits))))
        return f, row

    def sync(self):
        """serialises pending bits per fragment (merged with nothing: test fragments are written once)"""
        for (index, field, view, shard), bits in self._pending.items():
            self.import_roaring(index, field, view, shard, roaring_io.encode(np.fromiter(bits, dtype=np.uint64, count=len(bits))))
        self._pending = {}


class RowResult:
    """pilosa.Row as returned to clients: roaring bytes (absolute keys) + Columns()"""

    def __init__(self, data, count):
        self.roaring, self.count = data, count

    def columns(self):
        return roaring_io.decode(self.roaring)


class QueryError(Exception):
    pass


class ValCount:
    """pilosa.ValCount (executor.go:8425): integer Val + Count; compares equal to a (val, count) tuple"""

    def __init__(self, val=0, count=0):
        self.val, self.count = int(val), int(count)

    def __eq__(self, o):
        return (self.val, self.count) == ((o.val, o.count) if isinstance(o, ValCount) else tuple(o))

    def __repr__(self):
        return f"ValCount(val={self.val}, count={self.count})"


class SignedRow:
    """pilosa.SignedRow executor.go:8225: the distinct values of an int field, as two id sets (Pos: values >= 0, Neg: |v| of
    the negative ones), Base already added (executeDistinctShardBSI :2125)"""

    def __init__(self, pos=(), neg=()):
        self.pos, self.neg = sorted(pos), sorted(neg)

    def values(self):
        return [-v for v in reversed(self.neg)] + list(self.pos)       # SignedRow.ToRows :8253 order

    def count(self):
        return len(self.pos) + len(self.neg)                            # executeCount :5861

    def __eq__(self, o):
        return isinstance(o, SignedRow) and (self.pos, self.neg) == (o.pos, o.neg)

    def __repr__(self):
        return f"SignedRow(pos={self.pos}, neg={self.neg})"


def _i64(x):
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


class Executor:
    def __init__(self, holder):
        self.holder, self.ctx = holder, holder.ctx

    # ------------------------------------------------------------------ entry (executor.Execute :183 / execute :490)
    def execute(self, index, query, shards=None):
        idx = self.holder.indexes.get(index)
        if idx is None:
            raise QueryError("index not found")
        calls = pql.parse(query) if isinstance(query, str) else ([query] if isinstance(query, pql.Call) else list(query))
        if shards is None:
            shards = sorted(idx.shards)        # idx.AvailableShards :521
        return [self._execute_call(idx, c, shards) for c in calls]

    # executeCall :679
    def _execute_call(self, idx, c, shards):
        self._cur_shards = shards                                # (UnionRows runs its Rows / TopN children over the same shard list)
        try:
            if c.name == "Count":
                return self._count(idx, c, shards)
            if c.name == "TopN":
                return self._topn(idx, c, shards)
            if c.name == "TopK":
                return self._topk(idx, c, shards)
            if c.name == "GroupBy":
                return self._groupby(idx, c, shards)
            if c.name == "Rows":
                return self._rows(idx, c, shards, standalone=True)
            if c.name == "Sum":
                return self._sum(idx, c, shards)
            if c.name in ("Min", "Max"):
                return self._minmax(idx, c, shards, c.name)
            if c.name == "Percentile":
                return self._percentile(idx, c, shards)
            if c.name in ("MinRow", "MaxRow"):
                return self._minmax_row(idx, c, shards, c.name == "MaxRow")
            if c.name == "Distinct":
                return self._distinct(idx, c, shards)
            if c.name == "Extract":
                return self._extract(idx, c, shards)
            if c.name == "Sort":
                return self._sort(idx, c, shards)
            if c.name == "FieldValue":                           # executeFieldValueCall :943: the int value of one column, ValCount(value, 1)
                name = c.args.get("field")
                if not name:
                    raise QueryError("field required")
                if c.args.get("column") in (None, ""):
                    raise QueryError("column required")
                f = self._field(idx, name)
                if f.type != "int":
                    raise QueryError(f"field {name} is not an int field")
                col = int(c.args["column"])
                ef, erow = self.holder.embed_row(idx.name, [col])
                _, vals, n = self.ctx.extract(idx.id, f.id, VIEW_BSI, f.bit_depth, [col // SHARD_WIDTH],
                                              filter_ops=[L.Op(L.OP_ROW, ef.id, VIEW_STANDARD, 0, erow, 0, 0, 0)])
                return ValCount(int(vals[0]) + f.base, 1) if n else ValCount()
            if c.name == "Options":                              # executeOptionsCall :869: shards=[..] narrows the shard list of the child call
                if len(c.children) != 1:
                    raise QueryError("Options() requires a single child call")
                sh = c.args.get("shards")
                return self._execute_call(idx, c.children[0], shards if sh is None else sorted(int(x) for x in sh))
            if c.name == "IncludesColumn":                       # executeIncludesColumnCall: is the column in the row?
                if "column" not in c.args:
                    raise QueryError("IncludesColumn call must specify a column")
                if len(c.children) != 1:
                    raise QueryError("IncludesColumn call must specify a row query")
                col = int(c.args["column"])
                ef, erow = self.holder.embed_row(idx.name, [col])
                ops = self._bitmap_call(idx, c.children[0]) + [L.Op(L.OP_ROW, ef.id, VIEW_STANDARD, 0, erow, 0, 0, 0), L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)]
                return self.ctx.count(idx.id, ops, [col // SHARD_WIDTH]) > 0
            window = None
            if c.name == "Limit":                                # executeLimitCall: a column window over the child's row
                if len(c.children) != 1:
                    raise QueryError("Limit() requires a single bitmap input")
                window, c = (int(c.args.get("offset", 0)), c.args.get("limit")), c.children[0]
            elif c.name == "All" and ("limit" in c.args or "offset" in c.args):      # executeAllCall :5720-5779 with limit / offset
                window = (int(c.args.get("offset", 0)), c.args.get("limit"))
            ops = self._bitmap_call(idx, c)
            data, cnt = self.ctx.row(idx.id, ops, self._cur_shards)       # (Shift may have carried bits into a further shard)
            if window is not None:                               # the window is cut from the merged result on the host
                cols = roaring_io.decode(data)
                off, lim = window
                cols = cols[off:] if lim is None else cols[off:off + int(lim)]
                return RowResult(roaring_io.encode(np.asarray(cols, dtype=np.uint64)), len(cols))
            return RowResult(data, cnt)
        except L.FbgpuError as e:
            if e.code == L.E_QUERY:
                raise QueryError(str(e)) from e
            raise

    # ------------------------------------------------------------------ bitmap calls -> post-order program (executeBitmapCallShard :1782)
    def _bitmap_call(self, idx, c):
        ops = []
        self._emit(idx, c, ops)
        return ops

    def _field(self, idx, name):
        f = idx.fields.get(name)
        if f is None:
            raise QueryError(f"field not found: {name}")       # ErrFieldNotFound
        return f

    def _emit(self, idx, c, ops):
        n = c.name
        if n in ("Row", "Range"):                                # executeBitmapCallShard :1790-1791
            return self._emit_row(idx, c, ops)
        if n in ("Intersect", "Union", "Difference", "Xor"):
            for ch in c.children:
                self._emit(idx, ch, ops)
            code = {"Intersect": L.OP_INTERSECT, "Union": L.OP_UNION, "Difference": L.OP_DIFFERENCE, "Xor": L.OP_XOR}[n]
            ops.append(L.Op(code, 0, 0, len(c.children), 0, 0, 0, 0))
            return
        if n == "Not":                                           # executeNotShard :5554
            if len(c.children) != 1:
                raise QueryError("Not() requires a single bitmap input")
            if not idx.track_existence:
                raise QueryError(f"index does not support existence tracking: {idx.name}")
            self._emit(idx, c.children[0], ops)
            ops.append(L.Op(L.OP_NOT, idx.fields[EXISTENCE_FIELD].id, VIEW_STANDARD, 1, 0, 0, 0, 0))
            return
        if n == "ConstRow":                                      # executeConstRow :5604-5694: the listed columns (∩ existence when tracked)
            cols = c.args.get("columns")
            if not isinstance(cols, (list, tuple)):
                raise QueryError("missing columns list")
            if not cols:
                ops.append(L.Op(L.OP_EMPTY, 0, 0, 0, 0, 0, 0, 0))
                return
            f, row = self.holder.embed_row(idx.name, cols)
            ops.append(L.Op(L.OP_ROW, f.id, VIEW_STANDARD, 0, row, 0, 0, 0))
            if idx.track_existence:
                ops.append(L.Op(L.OP_ALL, idx.fields[EXISTENCE_FIELD].id, VIEW_STANDARD, 0, 0, 0, 0, 0))
                ops.append(L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0))
            return
        if n == "Distinct":                                      # handlePreCalls :396-440: the result's ids become a column row (SignedRow: Pos only)
            res = self._distinct(idx, c, self._cur_shards)
            cols = res.pos if isinstance(res, SignedRow) else res
            if not cols:
                ops.append(L.Op(L.OP_EMPTY, 0, 0, 0, 0, 0, 0, 0))
                return
            f, row = self.holder.embed_row(idx.name, cols)
            ops.append(L.Op(L.OP_ROW, f.id, VIEW_STANDARD, 0, row, 0, 0, 0))
            return
        if n == "Shift":                                         # executeShiftShard (unsupported upstream, row.go Shift): every column + n
            if len(c.children) != 1:
                raise QueryError("Shift() requires a single bitmap input")
            k = int(c.args.get("n", 0))
            data, _ = self.ctx.row(idx.id, self._bitmap_call(idx, c.children[0]), self._cur_shards)
            cols = [int(x) + k for x in roaring_io.decode(data)]
            if not cols:
                ops.append(L.Op(L.OP_EMPTY, 0, 0, 0, 0, 0, 0, 0))
                return
            f, row = self.holder.embed_row(idx.name, cols)       # the shifted row is a caller-provided operand from here on
            self._cur_shards = sorted(set(self._cur_shards) | {col // SHARD_WIDTH for col in cols})
            ops.append(L.Op(L.OP_ROW, f.id, VIEW_STANDARD, 0, row, 0, 0, 0))
            return
        if n == "UnionRows":                                     # executeUnionRows :5696-5779 -> Union(Row(..), ...) over the children's row ids
            leaves = []
            for ch in c.children:
                if ch.name == "Rows":
                    fld = self._field(idx, ch.args.get("_field", ch.args.get("field")))
                    leaves += [(fld, r) for r in self._rows(idx, ch, self._cur_shards, standalone=True)]
                elif ch.name in ("TopN", "TopK"):
                    fld = self._field(idx, ch.args["_field"])
                    pairs = self._topn(idx, ch, self._cur_shards) if ch.name == "TopN" else self._topk(idx, ch, self._cur_shards)
                    leaves += [(fld, r) for r, _ in pairs]
                else:
                    raise QueryError(f"UnionRows doesn't support {ch.name}")
            if not leaves:
                ops.append(L.Op(L.OP_EMPTY, 0, 0, 0, 0, 0, 0, 0))
                return
            for fld, r in leaves:
                ops.append(L.Op(L.OP_ROW, fld.id, VIEW_STANDARD, 0, int(r), 0, 0, 0))
            if len(leaves) > 1:
                ops.append(L.Op(L.OP_UNION, 0, 0, len(leaves), 0, 0, 0, 0))
            return
        if n == "All":                                           # executeAllCallShard :5781
            if not idx.track_existence:
                raise QueryError(f"index does not support existence tracking: {idx.name}")
            ops.append(L.Op(L.OP_ALL, idx.fields[EXISTENCE_FIELD].id, VIEW_STANDARD, 0, 0, 0, 0, 0))
            return
        raise QueryError(f"unknown call: {n}")

    def _emit_row(self, idx, c, ops):                            # executeRowShard :5120
        keys = [k for k in c.args if not k.startswith("_") and k not in ("from", "to")]
        if len(keys) == 0:
            raise QueryError("Row(): condition required")
        if len(keys) > 1:
            raise QueryError("Row(): too many arguments")
        name = keys[0]
        f = self._field(idx, name)
        v = c.args[name]
        if f.type == "int" or isinstance(v, pql.Condition):
            return self._emit_bsi(idx, f, v if isinstance(v, pql.Condition) else pql.Condition("==", v), ops)
        if f.type == "bool":
            v = 1 if v else 0                                    # fragment.go:59-60
        if "from" in c.args or "to" in c.args:                   # :5149-5163, 5209-5241: union of the row over the covering time views
            ids = self._time_view_ids(f, c.args)
            if not ids:
                ops.append(L.Op(L.OP_EMPTY, 0, 0, 0, 0, 0, 0, 0))
                return
            for i in ids:
                ops.append(L.Op(L.OP_ROW, f.id, i, 0, int(v), 0, 0, 0))
            if len(ids) > 1:
                ops.append(L.Op(L.OP_UNION, 0, 0, len(ids), 0, 0, 0, 0))
            return
        ops.append(L.Op(L.OP_ROW, f.id, VIEW_STANDARD, 0, int(v), 0, 0, 0))

    def _time_view_ids(self, f, args):
        """ids of the views that cover from= / to= (Field.viewsByTimeRange); views without a fragment anywhere contribute nothing"""
        try:
            t_from = timeq.parse_time(args["from"]) if "from" in args else None
            t_to = timeq.parse_time(args["to"]) if "to" in args else None
        except ValueError as e:
            raise QueryError(f"parsing time: {e}")
        ids = [f.view_id(name) for name in f.views_by_time_range(t_from, t_to)]
        return [i for i in ids if i is not None]

    def _emit_bsi(self, idx, f, cond, ops):                      # executeRowBSIGroupShard :5249-5354
        if f.type != "int":
            raise QueryError(f"field {f.name} is not an int field")
        op, value = cond.op, cond.value
        not_null = L.Op(L.OP_ROW, f.id, VIEW_BSI, 0, 0, 0, 0, 0)     # frag.notNull fragment.go:1208 == exists row
        if value is None and op == "!=":
            ops.append(not_null)
            return
        if value is None and op == "==":                        # getNullRowShard :5056: existence \ notNull
            if not idx.track_existence:
                raise QueryError(f"index does not support existence tracking: {idx.name}")
            ops.append(L.Op(L.OP_ALL, idx.fields[EXISTENCE_FIELD].id, VIEW_STANDARD, 0, 0, 0, 0, 0))
            ops.append(not_null)
            ops.append(L.Op(L.OP_DIFFERENCE, 0, 0, 2, 0, 0, 0, 0))
            return
        if op == "><":
            if not isinstance(value, (list, tuple)) or len(value) != 2:
                raise QueryError("Row(): BETWEEN condition requires exactly two integer values")
            lo, hi, oor = f.base_value_between(int(value[0]), int(value[1]))
            if oor:
                ops.append(L.Op(L.OP_EMPTY, 0, 0, 0, 0, 0, 0, 0))
            elif value[0] <= f.min and value[1] >= f.max:
                ops.append(not_null)
            else:
                ops.append(L.Op(L.OP_BSI_RANGE, f.id, VIEW_BSI, 0, f.bit_depth, L.CMP["><"], lo, hi))
            return
        value = int(value)
        bv, oor = f.base_value(op, value)
        if oor and op != "!=":
            ops.append(L.Op(L.OP_EMPTY, 0, 0, 0, 0, 0, 0, 0))
        elif (op == "<" and value > f.max) or (op == "<=" and value >= f.max) or (op == ">" and value < f.min) or (op == ">=" and value <= f.min):
            ops.append(not_null)
        elif oor and op == "!=":
            ops.append(not_null)
        else:
            ops.append(L.Op(L.OP_BSI_RANGE, f.id, VIEW_BSI, 0, f.bit_depth, L.CMP[op], bv, 0))

    # ------------------------------------------------------------------ Count (executeCount :5839)
    def _count(self, idx, c, shards):
        if len(c.children) == 0:
            raise QueryError("Count() requires an input bitmap")
        if len(c.children) > 1:
            raise QueryError("Count() only accepts a single bitmap input")
        if c.children[0].name == "Distinct":                     # PrecallGlobal child: run it and count the result (:5852-5868)
            res = self._distinct(idx, c.children[0], shards)
            return res.count() if isinstance(res, SignedRow) else len(res)
        return self.ctx.count(idx.id, self._bitmap_call(idx, c.children[0]), shards)

    # ------------------------------------------------------------------ TopN / TopK (exact modes; SURVEY Appendix D)
    def _topn(self, idx, c, shards):                             # executeTopN :2779 with ids / second pass semantics
        f = self._field(idx, c.args["_field"])
        if f.type in ("int", "decimal", "timestamp"):            # executeTopNShard :2876
            raise QueryError(f'cannot compute TopN() on integer, decimal, or timestamp field: "{f.name}"')
        if len(c.children) > 1:
            raise QueryError("TopN() can only have one input bitmap")
        n = int(c.args.get("n", 0))
        thr = int(c.args.get("threshold", 0)) or 1               # defaultMinThreshold = 1 (:2917-2919)
        tan = int(c.args.get("tanimotoThreshold", 0))
        if tan > 100:
            raise QueryError("Tanimoto Threshold is from 1 to 100 only")
        filt = self._bitmap_call(idx, c.children[0]) if c.children else None
        ids = c.args.get("ids")
        if ids is not None:
            ids = sorted(int(i) for i in ids) or None              # an empty list is "no ids" (len(opt.RowIDs) > 0, fragment.go:1325)
        if thr > 1 or (tan > 0 and filt is not None):            # per-shard cut-offs of fragment.top (fragment.go:1329-1388)
            pairs = self._topn_cutoffs(idx, f, filt, ids, thr, tan, shards)
        elif ids is not None:
            src = c.children[0] if c.children else None
            src_key = [k for k in src.args if not k.startswith("_") and k not in ("from", "to")] if src is not None and src.name == "Row" else []
            if len(src_key) == 1 and "from" not in src.args and "to" not in src.args and not isinstance(src.args[src_key[0]], pql.Condition) and self._field(idx, src_key[0]).type != "int":
                # Src is a plain Row: count = Src.intersectionCount(row) per candidate (fragment.go:1367-1372), fused
                sf = self._field(idx, src_key[0])
                counts = self.ctx.count_pairs(idx.id, f.id, VIEW_STANDARD, ids, sf.id, VIEW_STANDARD, [int(src.args[src_key[0]])] * len(ids), shards)
            else:
                counts = self.ctx.row_counts(idx.id, f.id, VIEW_STANDARD, shards, row_ids=ids, filter_ops=filt)
            pairs = [(i, int(k)) for i, k in zip(ids, counts) if k > 0]
            pairs.sort(key=lambda p: (-p[1], p[0]))              # Pairs sort desc; ties pinned (count desc, id asc)
        else:
            rid, cnt = self.ctx.row_counts(idx.id, f.id, VIEW_STANDARD, shards, filter_ops=filt)
            pairs = [(int(i), int(k)) for i, k in zip(rid, cnt)]
        if ids is not None:                                      # explicit ids: the result is never truncated (:2802-2807, fragment.go:1325)
            return pairs
        return pairs[:n] if n else pairs

    def _topn_cutoffs(self, idx, f, filt, ids, thr, tan, shards):
        """TopN with threshold= / tanimotoThreshold=: fragment.top applies its cut-offs per shard — on the row's own count `cnt`
        in that shard, then on `count` = |Src ∩ row| there (MinThreshold :1357-1362,1384-1388; Tanimoto band and coefficient
        :1329-1338,1351-1356,1378-1383) — and only what passes is summed across shards (Pairs.Add, executeTopNShards :2845).
        So the counts are fetched as [shard][row] matrices (fbgpu_row_counts_per_shard: one launch for the rows' own counts, one
        more with the Src as filter; the Src counts of all shards come from one fbgpu_count).  Candidates: `ids`, else every row of the
        field (what the internal second pass asks for when the first pass missed nothing; SURVEY Appendix D).  A context with
        topn_cutoffs does all of it in one device call, whose all-rows form is already in the answer's order."""
        if hasattr(self.ctx, "topn_cutoffs"):
            if ids is not None:
                totals = self.ctx.topn_cutoffs(idx.id, f.id, VIEW_STANDARD, shards, row_ids=ids, src_ops=filt, min_threshold=thr, tanimoto=tan)
                pairs = [(i, int(k)) for i, k in zip(ids, totals) if k > 0]
                pairs.sort(key=lambda p: (-p[1], p[0]))
                return pairs
            rid, cnt = self.ctx.topn_cutoffs(idx.id, f.id, VIEW_STANDARD, shards, src_ops=filt, min_threshold=thr, tanimoto=tan)
            return [(int(i), int(k)) for i, k in zip(rid, cnt)]
        if ids is None:
            rid, _ = self.ctx.row_counts(idx.id, f.id, VIEW_STANDARD, shards)
            ids = sorted(int(r) for r in rid)
        if not ids:
            return []
        use_tan = tan > 0 and filt is not None
        src_counts = self.ctx.count(idx.id, filt, shards, per_shard=True)[1] if use_tan else None
        total = np.zeros(len(ids), dtype=np.uint64)
        cnt_m = self.ctx.row_counts_per_shard(idx.id, f.id, VIEW_STANDARD, shards, ids)
        count_m = self.ctx.row_counts_per_shard(idx.id, f.id, VIEW_STANDARD, shards, ids, filter_ops=filt) if filt is not None else cnt_m
        for k in range(len(shards)):
            cnt, count = cnt_m[k], count_m[k]
            if not cnt.any():
                continue
            for j in range(len(ids)):
                cj, kj = int(cnt[j]), int(count[j])
                if cj == 0 or kj == 0:
                    continue
                if use_tan:
                    sc = int(src_counts[k])
                    if float(cj) <= float(sc * tan) / 100 or float(cj) >= float(sc * 100) / float(tan):
                        continue
                    if math.ceil(float(kj * 100) / float(cj + sc - kj)) <= float(tan):
                        continue
                elif cj < thr or kj < thr:
                    continue
                total[j] += np.uint64(kj)
        pairs = [(i, int(k)) for i, k in zip(ids, total) if k > 0]
        pairs.sort(key=lambda p: (-p[1], p[0]))
        return pairs

    def _topk(self, idx, c, shards):                             # executeTopK :2357, doTopK :2705
        f = self._field(idx, c.args["_field"])
        k = int(c.args.get("k", 0))
        filt = c.args.get("filter")
        filt = self._bitmap_call(idx, filt) if isinstance(filt, pql.Call) else None
        targs = {a: c.args[a] for a in ("from", "to") if a in c.args} if f.quantum else {}
        if targs and hasattr(self.ctx, "row_counts_views"):     # executeTopKShardTime :2506-2533 / mergerator :2570: a row is the union of
            views = self._time_view_ids(f, targs)                # itself over the covering views, counted in one library call
            if not views:
                return []
            rid, cnt = self.ctx.row_counts_views(idx.id, f.id, views, shards, filter_ops=filt)
            pairs = [(int(i), int(n)) for i, n in zip(rid, cnt)]
            return pairs[:k] if k else pairs
        if targs:
            rows = self._rows(idx, pql.Call("Rows", {"_field": f.name, **targs}), shards)
            if not rows:
                return []
            sf, operands = self._time_rows_as_operands(idx, f, rows, targs, shards)
            cnt = self.ctx.row_counts(idx.id, sf.id, VIEW_STANDARD, shards, row_ids=operands, filter_ops=filt)
            pairs = sorted(((r, int(n)) for r, n in zip(rows, cnt) if n), key=lambda kv: (-kv[1], kv[0]))
            return pairs[:k] if k else pairs
        rid, cnt = self.ctx.row_counts(idx.id, f.id, VIEW_STANDARD, shards, filter_ops=filt)
        pairs = [(int(i), int(n)) for i, n in zip(rid, cnt)]
        return pairs[:k] if k else pairs

    def _time_rows_as_operands(self, idx, f, rows, targs, shards):
        """Rows of a time field restricted to from= / to=, made addressable by the single-view kernels: each row's union over
        the covering views (timeFragmentsRowIterator :8755-8768, mergerator :2570) is evaluated once and stored as an operand
        row of the scratch field.  Returns (scratch field, operand row ids in the order of `rows`).  TopK, Rows and GroupBy
        count such rows with row_counts_views / groupby_views / groupby_mixed instead where the context has them; this remains for
        contexts without those calls."""
        operands = []
        for r in rows:
            data, _ = self.ctx.row(idx.id, self._bitmap_call(idx, pql.Call("Row", {f.name: r, **targs})), shards)
            sf, srow = self.holder.embed_row(idx.name, roaring_io.decode(data))
            operands.append(srow)
        return sf, operands

    def _rows(self, idx, c, shards, standalone=False):           # executeRows (row ids present; limit / previous / in)
        name = c.args["_field"] if "_field" in c.args else c.args.get("field")
        if name is None:
            raise QueryError("missing field in Rows call")
        f = self._field(idx, name)
        if standalone and f.type in ("int", "bool"):
            raise QueryError(f"{f.type} fields not supported by Rows() query")
        if "like" in c.args:
            raise QueryError("Rows(): like is not supported by this mirror")
        if "in" in c.args and "column" in c.args:
            raise QueryError("Rows call with 'in' does not support other arguments")
        filt = None
        if "column" in c.args:                                   # rows that hold this column (BitmapColumnFilter roaring/filter.go:118): a one-column filter row
            col = int(c.args["column"])
            ef, erow = self.holder.embed_row(idx.name, [col])
            filt = [L.Op(L.OP_ROW, ef.id, VIEW_STANDARD, 0, erow, 0, 0, 0)]
            shards = [s for s in shards if s == col // SHARD_WIDTH]
        views = [VIEW_BSI if f.type == "int" else VIEW_STANDARD]
        timed = f.quantum and ("from" in c.args or "to" in c.args)
        if timed:                                                # executeRowsShard :4107-4127: the rows of every covering view, merged
            views = self._time_view_ids(f, c.args)
        if timed and views and hasattr(self.ctx, "row_counts_views"):       # (in one library call)
            rid, _ = self.ctx.row_counts_views(idx.id, f.id, views, shards, filter_ops=filt)
            out = sorted(int(r) for r in rid)
        else:
            out = set()
            for v in views:
                rid, _ = self.ctx.row_counts(idx.id, f.id, v, shards, filter_ops=filt)
                out.update(int(r) for r in rid)
            out = sorted(out)
        if "in" in c.args:
            keep = {int(r) for r in c.args["in"]}
            out = [r for r in out if r in keep]
        if "previous" in c.args:                                 # rows strictly after `previous` (fragment.rows start = previous + 1)
            out = [r for r in out if r > int(c.args["previous"])]
        lim = c.args.get("limit")
        return out[:lim] if lim else out

    # ------------------------------------------------------------------ BSI aggregates (executeSum :1119, executeMin :1225, executeMax :1261)
    # Composed from the library's counting entry points, the way the Go shim would inside executeSumCountShard /
    # Field.MinForShard: every step is one launch over the whole shard batch.
    def _sum(self, idx, c, shards):
        """executeSum :1119 over fragment.sum (fragment.go:722) / BitmapBSICountFilter (filter.go:1106-1165), reduced by
        ValCount.Add (:8438): one library call — the row (filter ∩ not-null) is evaluated once, the planes are walked once,
        Val = Σ (pos_i - neg_i) << i  +  count * Base (executeSumCountShard :2203-2206), all in wrapping int64."""
        name = c.args.get("field", c.args.get("_field"))
        if name is None:
            raise QueryError("Sum(): field required")
        if len(c.children) > 1:
            raise QueryError("Sum() only accepts a single bitmap input")
        f = self._field(idx, name)
        if f.type != "int":
            return ValCount()                                           # bsig == nil (:2187-2190)
        filt = self._bitmap_call(idx, c.children[0]) if c.children else None
        total, count = self.ctx.bsi_sum(idx.id, f.id, VIEW_BSI, f.bit_depth, shards, filter_ops=filt)
        if count == 0:
            return ValCount()                                           # executeSum :1147-1149
        return ValCount(_i64(total + count * f.base), count)

    def _minmax(self, idx, c, shards, what):
        """executeMin :1225 / executeMax :1261 over fragment.min / max (fragment.go:752-838): one library call — the row
        (filter ∩ not-null) is evaluated once and the bit planes are walked once per (shard, slot) unit on the device, the
        per-unit extremes are merged as ValCount.Smaller / Larger do (:8446-8560)."""
        name = c.args.get("field", c.args.get("_field"))
        if name is None:
            raise QueryError(f"{what}(): field required")
        if len(c.children) > 1:
            raise QueryError(f"{what}() only accepts a single bitmap input")
        f = self._field(idx, name)
        if f.type != "int":
            raise QueryError("bsigroup not found")                      # ErrBSIGroupNotFound field.go:1571
        filt = self._bitmap_call(idx, c.children[0]) if c.children else None
        v, n = self.ctx.bsi_minmax(idx.id, f.id, VIEW_BSI, f.bit_depth, shards, what == "Max", filter_ops=filt)
        if n == 0:
            return ValCount()                                           # :1252-1254
        return ValCount(v + f.base, n)                                  # valCountize field.go:1640

    def _minmax_row(self, idx, c, shards, want_max):
        """executeMinRow / executeMaxRow :1604-1672 with fragment.minRow / maxRow fragment.go:862-922: the smallest / largest
        row id that has a bit (under the optional filter).  Per shard the reference reports Count = 1 without a filter, else
        |row ∩ filter| in that shard, and the reduce keeps the pair of ONE shard (on equal ids the later arrival, so the count
        is order dependent upstream); here: the last shard, in ascending order, where the row meets the filter.
        Returns (row id, count), or (0, 0) when nothing qualifies."""
        name = c.args.get("field", c.args.get("_field"))
        if not name:
            raise QueryError(("MaxRow" if want_max else "MinRow") + "(): field required")
        f = self._field(idx, name)
        filt = self._bitmap_call(idx, c.children[0]) if c.children else None
        rid, cnt = self.ctx.row_counts(idx.id, f.id, VIEW_STANDARD, shards, filter_ops=filt)
        ids = [int(r) for r, n in zip(rid, cnt) if n > 0]
        if not ids:
            return (0, 0)
        best = max(ids) if want_max else min(ids)
        if filt is None:
            return (best, 1)
        for s in sorted(shards, reverse=True):
            n = int(self.ctx.row_counts(idx.id, f.id, VIEW_STANDARD, [s], row_ids=[best], filter_ops=filt)[0])
            if n:
                return (best, n)
        return (best, 0)

    def _distinct(self, idx, c, shards):
        """executeDistinct :1173 / executeDistinctShard :1820.  Set-like field: the ids of the rows that have a bit (under the
        optional filter), executeDistinctShardSet :1952 — one row-count launch.  Int field: the set of values present,
        executeDistinctShardBSI :2034, returned as a SignedRow.  The reference transposes the bit planes column by column;
        a context with bsi_distinct lists the distinct values of filter ∩ not-null on the device in one call; a context without
        it gathers every value (fbgpu_extract) and takes the distinct set of the value vector.
        `index=` runs the call on another index (foreign-index joins)."""
        name = c.args.get("field", c.args.get("_field"))
        if name is None:
            raise QueryError("missing field option in Distinct query")
        if len(c.children) > 1:
            raise QueryError("Distinct() only accepts a single bitmap input")
        other = c.args.get("index")
        if other is not None and other != idx.name:
            idx = self.holder.indexes.get(other)
            if idx is None:
                raise QueryError("index not found")
            shards = sorted(idx.shards)
        f = self._field(idx, name)
        saved, self._cur_shards = self._cur_shards, shards
        try:
            filt = self._bitmap_call(idx, c.children[0]) if c.children else None
        finally:
            self._cur_shards = saved
        if f.type != "int":
            rid, cnt = self.ctx.row_counts(idx.id, f.id, VIEW_STANDARD, shards, filter_ops=filt)
            return sorted(int(r) for r, n in zip(rid, cnt) if n > 0)
        pos, neg = set(), set()
        for m in self._int_values(idx, f, shards, filt).tolist():
            v = int(m) + f.base                                        # value += offset (:2125)
            (neg if v < 0 else pos).add(abs(v))
        return SignedRow(pos, neg)

    def _int_values(self, idx, f, shards, filt):
        """the distinct stored values (value - Base) of int field f under filt ∩ not-null, ascending int64"""
        if hasattr(self.ctx, "bsi_distinct"):
            return self.ctx.bsi_distinct(idx.id, f.id, VIEW_BSI, f.bit_depth, shards, filter_ops=filt)[0]
        _, vals, _ = self.ctx.extract(idx.id, f.id, VIEW_BSI, f.bit_depth, shards, filter_ops=filt)
        return np.unique(np.asarray(vals, dtype=np.int64))

    def _extract(self, idx, c, shards):
        """executeExtract :4711 / executeExtractShard :4758: the table {column -> per-field cell} for the columns of the first
        child.  The column list and the int cells come from the device (fbgpu_columns, fbgpu_extract: value + Base, None
        when the column has no value); a set / time cell is the ascending list of the field's rows that hold the column, a
        mutex cell the lowest such row (None if none), a bool cell whether that row is 1 (None if none).  A context with
        extract_rows takes each set-like field's lists from one call with the Extract's filter and window; other contexts
        expand filter ∩ Row(field=r) for every row of the field.  Keys, decimals and timestamps are translation layers above
        the path.  Returns {"fields": [(name, type)], "columns": [(column id, [cell, ...])]}."""
        if not c.children:
            raise QueryError("missing column filter in Extract")
        filt_call = c.children[0]
        sorted_cols = None
        if filt_call.name == "Sort":                             # Extract(Sort(..), ..): rows in the sort's order (ExtractedIDMatrixSorted :9610)
            sorted_cols = [col for col, _ in self._sort(idx, filt_call, shards)]
        win = (0, None)
        if filt_call.name == "Limit":                            # Extract(Limit(x, limit=, offset=), ...): the window is cut on the device
            if len(filt_call.children) != 1:
                raise QueryError("Limit() requires a single bitmap input")
            win, filt_call = (int(filt_call.args.get("offset", 0)), filt_call.args.get("limit")), filt_call.children[0]
        fields = []
        for ch in c.children[1:]:                                # extractFieldsFromRowsCalls :4670-4708
            if ch.name != "Rows":
                raise QueryError(f"child call of Extract is {ch.name} but expected Rows")
            name = ch.args.get("_field", ch.args.get("field"))
            if name is None:
                raise QueryError("missing field in Rows call")
            fields.append(self._field(idx, name))
        if sorted_cols is None:
            filt = self._bitmap_call(idx, filt_call)
            cols, _ = self.ctx.columns(idx.id, filt, shards, offset=win[0], limit=win[1])
            cols = [int(x) for x in cols]
        else:
            cols, filt, win = sorted_cols, [], (1, None)         # (cells for exactly these columns: the narrowed filter below)
        pos = {col: i for i, col in enumerate(cols)}
        by_rows = hasattr(self.ctx, "extract_rows")
        rows_filt, rows_win = filt, win                          # extract_rows cuts the window itself
        if win != (0, None) and cols and (sorted_cols is not None or not by_rows or any(f.type == "int" for f in fields)):
            ef, erow = self.holder.embed_row(idx.name, cols)     # cells are only needed for the window: narrow the filter to it
            filt = [L.Op(L.OP_ROW, ef.id, VIEW_STANDARD, 0, erow, 0, 0, 0)]
            if sorted_cols is not None:
                rows_filt, rows_win = filt, (0, None)
        table = [[None] * len(fields) for _ in cols]
        types = []
        for k, f in enumerate(fields):
            if f.type == "int":
                types.append("int64")
                vc, vv, _ = self.ctx.extract(idx.id, f.id, VIEW_BSI, f.bit_depth, shards, filter_ops=filt)
                for col, v in zip(vc.tolist(), vv.tolist()):
                    if col in pos:
                        table[pos[col]][k] = int(v) + f.base
                continue
            multi = f.type in ("set", "time")
            types.append("[]uint64" if multi else "bool" if f.type == "bool" else "uint64")
            if multi:
                for row in table:
                    row[k] = []
            if by_rows:
                for col, rs in self._cell_rows(idx, f, shards, rows_filt, rows_win) if cols else ():
                    if rs and col in pos:
                        table[pos[col]][k] = rs if multi else (rs[0] == 1) if f.type == "bool" else rs[0]
                continue
            rid, _ = self.ctx.row_counts(idx.id, f.id, VIEW_STANDARD, shards, filter_ops=filt)
            for r in sorted(int(x) for x in rid):
                ops = filt + [L.Op(L.OP_ROW, f.id, VIEW_STANDARD, 0, r, 0, 0, 0), L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)]
                for col in self.ctx.columns(idx.id, ops, shards)[0].tolist():
                    if col not in pos:
                        continue
                    if multi:
                        table[pos[col]][k].append(r)
                    elif table[pos[col]][k] is None:
                        table[pos[col]][k] = (r == 1) if f.type == "bool" else r
        return {"fields": [(f.name, t) for f, t in zip(fields, types)], "columns": list(zip(cols, table))}

    def _cell_rows(self, idx, f, shards, filt, win=(0, None)):
        """[(column, [row, ...])]: every column of the window of filt with the ascending rows of set-like field f that hold it
        (one fbgpu_extract_rows call)"""
        cols, offs, rows, _ = self.ctx.extract_rows(idx.id, f.id, VIEW_STANDARD, shards, filt, offset=win[0], limit=win[1])
        offs, rows = offs.tolist(), rows.tolist()
        return [(col, rows[offs[i]:offs[i + 1]]) for i, col in enumerate(cols.tolist())]

    def _sort(self, idx, c, shards):
        """executeSort :9321 / executeSortShard :9387: the columns of the child row ordered by a field's value — int (values from
        fbgpu_extract), bool (falses then trues), mutex (by row id) — ascending or `sort-desc`, then offset / limit.  The
        reference merges per-shard lists in arrival order, so its order among equal values is unspecified; here ties keep
        ascending column order.  A context with bsi_sort orders an int field on the device and returns only the window; other
        contexts (and a negative offset or limit, which slice the list from its end) extract every value and sort here.  A
        context with extract_rows takes a bool or mutex field's (column, row) pairs from one call.
        Returns [(column, value)]."""
        name = c.args.get("field", c.args.get("_field"))
        if name is None:
            raise QueryError("getting field: Sort(): field required")
        if len(c.children) != 1:
            raise QueryError("Sort() requires a single bitmap input")
        f = self._field(idx, name)
        desc = bool(c.args.get("sort-desc", False))
        filt = self._bitmap_call(idx, c.children[0])
        off, lim = int(c.args.get("offset", 0)), c.args.get("limit")
        if f.type == "int" and hasattr(self.ctx, "bsi_sort") and off >= 0 and (lim is None or int(lim) >= 0):
            cols, vals, _ = self.ctx.bsi_sort(idx.id, f.id, VIEW_BSI, f.bit_depth, shards, desc=desc, filter_ops=filt, offset=off,
                                              limit=None if lim is None else int(lim))
            return [(int(col), int(v) + f.base) for col, v in zip(cols.tolist(), vals.tolist())]
        if f.type == "int":
            cols, vals, _ = self.ctx.extract(idx.id, f.id, VIEW_BSI, f.bit_depth, shards, filter_ops=filt)
            kvs = [(int(col), int(v) + f.base) for col, v in zip(cols.tolist(), vals.tolist())]
        elif f.type in ("bool", "mutex") and hasattr(self.ctx, "extract_rows"):
            kvs = [(col, (r == 1) if f.type == "bool" else r) for col, rs in self._cell_rows(idx, f, shards, filt) for r in rs]
        elif f.type in ("bool", "mutex"):
            kvs = []
            rid, _ = self.ctx.row_counts(idx.id, f.id, VIEW_STANDARD, shards, filter_ops=filt)
            for r in sorted(int(x) for x in rid):
                ops = filt + [L.Op(L.OP_ROW, f.id, VIEW_STANDARD, 0, r, 0, 0, 0), L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)]
                kvs += [(int(col), (r == 1) if f.type == "bool" else r) for col in self.ctx.columns(idx.id, ops, shards)[0].tolist()]
        else:
            raise QueryError(f"Sort of field type {f.type} not implemented yet")
        kvs.sort(key=lambda kv: (-kv[1] if desc else kv[1], kv[0]))
        kvs = kvs[off:]
        return kvs[:int(lim)] if lim is not None else kvs

    percentile_select = True            # False: Percentile always runs the query-driven bisection (the reference's own flow)

    def _percentile(self, idx, c, shards):
        """executePercentile :1310-1600 (int fields): total = Count(filter ∩ notNull); the wanted numbers of smaller / larger
        values (float64 arithmetic, as the reference); Min and Max under the filter; then a bisection on the value.
        The reference asks two Count(Row(f < x) [∩ filter]) style queries per bisection step.  Every guess g lies in
        [min, max], so with v[0..T-1] the sorted values: Count(f < g) > desiredLess exactly when v[desiredLess] < g, and
        Count(f > g) > desiredGreater exactly when v[T-1-desiredGreater] > g.  One fbgpu_bsi_select call for the ranks
        0, T-1, desiredLess, T-1-desiredGreater therefore fixes the answer bit for bit, and the bisection runs on the host.
        Contexts without the call (a node handle, a context with a communicator) and depth-64 fields take the query-driven bisection.
        Returns None ("the median of nothing is NULL") or ValCount(value, 1) / the Min / Max ValCount at the ends."""
        nth = c.args.get("nth")
        if nth is None:
            raise QueryError("Percentile(): nth required")
        if isinstance(nth, bool) or not isinstance(nth, (int, float)):
            raise QueryError(f"Percentile(): invalid nth='{nth}', should be a number between 0 and 100 inclusive")
        nth = float(nth)
        if nth < 0 or nth > 100.0:
            raise QueryError(f"Percentile(): invalid nth value ({nth}), should be a number between 0 and 100 inclusive")
        name = c.args.get("field", c.args.get("_field"))
        if name is None:
            raise QueryError("Percentile(): field required")
        f = self._field(idx, name)
        filt = c.args.get("filter") if isinstance(c.args.get("filter"), pql.Call) else None
        not_null = pql.Call("Row", {name: pql.Condition("!=", None)})
        total = self._count(idx, pql.Call("Count", {}, [not_null if filt is None else pql.Call("Intersect", {}, [filt, not_null])]), shards)
        if total == 0:
            return None
        want_less = int(total * nth / 100.0)
        want_greater = int(total * (100 - nth) / 100.0)
        if self.percentile_select and f.type == "int" and f.bit_depth <= 63 and hasattr(self.ctx, "bsi_select"):      # select keys take depth + 1 bits
            try:
                return self._percentile_select(idx, f, filt, shards, total, want_less, want_greater)
            except NotImplementedError:
                pass
            except L.FbgpuError as e:
                if e.code != L.E_COMM:
                    raise
        return self._percentile_bisect(idx, f, filt, shards, want_less, want_greater)

    @staticmethod
    def _midpoint(lo, hi):
        """the reference's overflow-free midpoint (:1493-1497) in Go's truncating integer arithmetic"""
        tdiv = lambda a, b: int(a / b) if abs(a) < (1 << 52) else (abs(a) // b) * (1 if a >= 0 else -1)      # Go's truncating division
        tmod = lambda a, b: a - b * tdiv(a, b)                                                                  # Go's %: sign of the dividend
        return tdiv(lo, 2) + tdiv(hi, 2) + tdiv(tmod(lo, 2) + tmod(hi, 2), 2)

    def _percentile_select(self, idx, f, filt, shards, total, want_less, want_greater):
        """the bisection over order statistics: one device call, no Count query per step.  A rank >= total (float rounding
        can make desiredLess reach it) or < 0 names a branch that is never taken."""
        wanted = {0, total - 1}
        i_less, i_greater = want_less, total - 1 - want_greater
        for r in (i_less, i_greater):
            if 0 <= r < total:
                wanted.add(r)
        ranks = sorted(wanted)
        filt_ops = self._bitmap_call(idx, filt) if filt is not None else None
        vals, cnts, _ = self.ctx.bsi_select(idx.id, f.id, VIEW_BSI, f.bit_depth, shards, ranks, filter_ops=filt_ops)
        at = {r: (int(v) + f.base, int(n)) for r, v, n in zip(ranks, vals.tolist(), cnts.tolist())}
        mn = ValCount()
        if want_greater != 0:
            mn = ValCount(*at[0])                                       # Min under the filter, with its multiplicity
            if want_less == 0:
                return mn
        mx = ValCount(*at[total - 1])
        if want_greater == 0:
            return mx
        v_less = at[i_less][0] if i_less < total else None
        v_greater = at[i_greater][0] if i_greater >= 0 else None
        lo, hi, guess = mn.val, mx.val, mn.val
        while lo < hi:
            guess = self._midpoint(lo, hi)
            if v_less is not None and v_less < guess:                   # Count(f < guess) > desiredLess
                hi = guess - 1
                continue
            if v_greater is not None and v_greater > guess:             # Count(f > guess) > desiredGreater
                lo = guess + 1
                continue
            break
        return ValCount(guess, 1)

    def _percentile_bisect(self, idx, f, filt, shards, want_less, want_greater):
        """the reference's flow: Min, Max, then two Count(Row(f < x) [∩ filter]) style queries per bisection step, every one a
        whole-batch device query, exactly as every step is a cluster-wide query in the reference"""
        name = f.name

        def count_of(row_call):
            inner = row_call if filt is None else pql.Call("Intersect", {}, [row_call, filt])
            return self._count(idx, pql.Call("Count", {}, [inner]), shards)
        kids = [filt] if filt is not None else []
        mn = ValCount()
        if want_greater != 0:
            mn = self._minmax(idx, pql.Call("Min", {"field": name}, kids), shards, "Min")
            if want_less == 0:
                return mn
        mx = self._minmax(idx, pql.Call("Max", {"field": name}, kids), shards, "Max")
        if want_greater == 0:
            return mx
        lo, hi, guess = mn.val, mx.val, mn.val
        while lo < hi:
            guess = self._midpoint(lo, hi)
            if count_of(pql.Call("Row", {name: pql.Condition("<", guess)})) > want_less:
                hi = guess - 1
                continue
            if count_of(pql.Call("Row", {name: pql.Condition(">", guess)})) > want_greater:
                lo = guess + 1
                continue
            break
        return ValCount(guess, 1)

    # ------------------------------------------------------------------ GroupBy (executeGroupBy :3176)
    def _groupby(self, idx, c, shards):
        """The device returns the dense count tensor over the children's row lists (with aggregate=Sum over an int field, the
        counts of columns holding a value and their sums, from the same call; with aggregate=Count(Distinct), the distinct
        counts from one more call after one Distinct for the field's values or rows; over set-like children too large for the
        dense tensor, the list of non-empty groups from fbgpu_groupby_sparse, _groupby_sparse); everything after it is the host-side
        post-processing executeGroupBy does in Go: previous (iterator start, newGroupByIterator :8779-8826), aggregate=Sum
        (groupByIterator.Next :8893-8911: Count becomes the number of columns holding a value), having (:3388-3406),
        sort (:3130-3162, 3408-3414), offset / limit (:3441-3459).  Results: (group, count) or (group, count, agg)."""
        if not c.children:
            raise QueryError("need at least one child call")
        fields, row_ids, time_args = [], [], []
        for ch in c.children:
            if ch.name != "Rows":
                raise QueryError(f"'{ch.name}' is not a valid child query for GroupBy, must be 'Rows'")
            name = ch.args.get("_field", ch.args.get("field"))
            if name is None:
                raise QueryError("missing field in Rows call")
            f = self._field(idx, name)
            fields.append(f)
            if f.type == "int":                                  # groups of an int field are its values (FieldRow.Value, :8740-8750), ascending
                row_ids.append(self._distinct(idx, pql.Call("Distinct", {"field": f.name}), shards).values())
                time_args.append(None)
                continue
            pre = pql.Call("Rows", {k: v for k, v in ch.args.items() if k != "previous"})     # previous positions the iterator, it does not drop rows
            row_ids.append(self._rows(idx, pre, shards))         # pre-pass executeRows :3263-3287
            time_args.append({k: ch.args[k] for k in ("from", "to") if k in ch.args} if f.quantum else {})
        filt_call = c.args.get("filter")
        filt = self._bitmap_call(idx, filt_call) if isinstance(filt_call, pql.Call) else None
        agg = c.args.get("aggregate")
        distinct_agg = False
        if isinstance(agg, pql.Call):
            if agg.name == "Count":                              # Count(Distinct(..)) is filled in after the groups are known (:3340-3386);
                distinct_agg = bool(agg.children) and agg.children[0].name == "Distinct"      # any other Count is the plain count (:8889)
                agg_distinct, agg = (agg.children[0] if distinct_agg else None), None
            elif agg.name != "Sum":
                raise QueryError(f"aggregate {agg.name} is not supported by this mirror")
        if any(len(r) == 0 for r in row_ids):
            return []
        int_dims = [k for k, f in enumerate(fields) if f.type == "int"]
        sum_f = None                                              # Sum over an int field: counts and sums from one device call
        if isinstance(agg, pql.Call) and hasattr(self.ctx, "groupby_sum"):
            f = idx.fields.get(agg.args.get("field", agg.args.get("_field")))
            if f is not None and f.type == "int":                 # otherwise the per-group Sum below raises or finds no values
                sum_f = f
        has_sort, has_having = "sort" in c.args, isinstance(c.args.get("having"), pql.Call)
        sparse = None                                             # (cells, counts[, sums]) of the non-empty groups from `start` on
        if not int_dims and hasattr(self.ctx, "groupby_sparse") and (
                max(len(r) for r in row_ids) > 65535 or math.prod(len(r) for r in row_ids) > self.GROUPBY_DENSE_MAX_CELLS):
            start = self._groupby_start(c, row_ids)
            if start is None:
                return []
            sparse = self._groupby_sparse(idx, c, fields, row_ids, time_args, filt, start, shards,
                                          device_limit=agg is None and not (has_sort or has_having), sum_f=sum_f)
        if sparse is not None:
            pass                                                  # groups in hand; Count(Distinct) below (_groupby_sparse_distinct), Sum over a non-int field per group
        elif sum_f is not None:
            counts, sums = self._groupby_tensors(idx, fields, row_ids, time_args, int_dims, filt, shards, agg=sum_f)
        elif int_dims and hasattr(self.ctx, "groupby_mixed"):
            counts, = self._groupby_tensors(idx, fields, row_ids, time_args, int_dims, filt, shards)
        elif not int_dims and any(time_args) and hasattr(self.ctx, "groupby_views"):
            # a Rows(f, from=, to=) child groups by its rows' unions over the covering views, in the same call as the other children
            views = [self._time_view_ids(f, targs) if targs else [VIEW_STANDARD] for f, targs in zip(fields, time_args)]
            counts = self.ctx.groupby_views(idx.id, [f.id for f in fields], views, row_ids, shards, filter_ops=filt)
        else:
            # what the device groups over: a field's standard view, or — for Rows(f, from=, to=) on a time field — one operand
            # row per row id holding the union of that row over the covering views (timeFragmentsRowIterator :8755-8768)
            dev_fields, dev_rows = [], []
            for f, rows, targs in zip(fields, row_ids, time_args):
                if targs is not None and not targs:
                    dev_fields.append(f.id)
                    dev_rows.append(rows)
                    continue
                sf, operands = self._time_rows_as_operands(idx, f, rows, targs or {}, shards)      # (int field: Row(f == value) per value)
                dev_fields.append(sf.id)
                dev_rows.append(operands)
            counts = self.ctx.groupby(idx.id, dev_fields, [VIEW_STANDARD] * len(fields), dev_rows, shards, filter_ops=filt)
        if sparse is None:
            start = self._groupby_start(c, row_ids)
            if start is None:
                return []
        dist = None                                               # Count(Distinct) over a field of this index: per-cell counts
        if sparse is None and distinct_agg and "index" not in agg_distinct.args and counts.any():
            f = idx.fields.get(agg_distinct.args.get("field", agg_distinct.args.get("_field")))
            call = None if f is None else "groupby_distinct" if f.type == "int" else "groupby_distinct_rows"
            if call is not None and hasattr(self.ctx, call):      # otherwise the per-group Distinct below raises or runs
                dist = self._groupby_distinct(idx, fields, row_ids, time_args, int_dims, filt_call, agg_distinct, f, counts.shape, shards)
        limit = c.args.get("limit") if not (has_sort or has_having) else None       # :3196-3212: no early limit when sorting / filtering
        out = []
        if sparse is not None:
            groups = ((_unravel(int(flat), [len(r) for r in row_ids]), int(n)) for flat, n in zip(sparse[0], sparse[1]))
        else:
            flat0 = int(np.ravel_multi_index(start, counts.shape))
            flat_counts = counts.reshape(-1)
            groups = ((np.unravel_index(int(flat), counts.shape), int(flat_counts[flat])) for flat in np.flatnonzero(flat_counts) if flat >= flat0)
        for g, (ix, n) in enumerate(groups):                      # only Count > 0, lexicographic (:3960)
            group = [(f.name, row_ids[k][int(i)]) for k, (f, i) in enumerate(zip(fields, ix))]
            if sum_f is not None:                                 # counts here: columns of the group holding a value of the field
                stored = int(sparse[2][g]) if sparse is not None else int(sums[ix])
                out.append((group, n, _i64(stored + n * sum_f.base)))      # executeSumCountShard :2203-2206
            elif isinstance(agg, pql.Call):
                rows = [pql.Call("Row", {name: rid, **(targs or {})}) for (name, rid), targs in zip(group, time_args)]
                if isinstance(filt_call, pql.Call):
                    rows.append(filt_call)
                inter = rows[0] if len(rows) == 1 else pql.Call("Intersect", {}, rows)
                vc = self._sum(idx, pql.Call("Sum", dict(agg.args), [inter]), shards)
                if vc.count == 0:
                    continue                                      # ret.Count == 0 => skipped (:8913-8919)
                out.append((group, vc.count, vc.val))
            elif dist is not None:
                out.append((group, n, int(dist[ix])))             # a distinct count of 0 is kept (:3343-3385)
            else:
                out.append((group, n))
            if limit and len(out) >= limit and "offset" not in c.args:
                break
        sparse_dist = None                                        # Count(Distinct) of the sparse path's listed groups: {cell: count}
        if distinct_agg and sparse is not None:
            pairs = list(zip((int(x) for x in sparse[0][:len(out)]), out))            # (cell, (group, count)) of the listed groups
            if not (has_sort or has_having):                      # limits first, as below
                pairs = self._window(c, pairs)
            sparse_dist = self._groupby_sparse_distinct(idx, fields, row_ids, time_args, filt_call, agg_distinct, pairs, sparse, shards)
            if sparse_dist is not None:
                out = [(group, n, sparse_dist.get(cell, 0)) for cell, (group, n) in pairs]    # a distinct count of 0 is kept (:3343-3385)
                if not (has_sort or has_having):
                    return out
        if distinct_agg and dist is None and sparse_dist is None:
            if not (has_sort or has_having):                      # limits first: the aggregate is expensive per group (:3327-3335)
                out = self._window(c, out)
            for k, (group, n) in enumerate(out):                  # Count(Distinct(Intersect(group rows, filter, Distinct's child), field=..)) :3343-3385
                rows = [pql.Call("Row", {name: rid, **(targs or {})}) for (name, rid), targs in zip(group, time_args)]
                if isinstance(filt_call, pql.Call):
                    rows.append(filt_call)
                rows += agg_distinct.children[:1]
                res = self._distinct(idx, pql.Call("Distinct", dict(agg_distinct.args), [pql.Call("Intersect", {}, rows)]), shards)
                out[k] = (group, n, res.count() if isinstance(res, SignedRow) else len(res))
            if not (has_sort or has_having):
                return out
        if has_having:                                            # Condition(count|sum <op> n)
            having = c.args["having"]
            if having.name != "Condition" or len(having.args) != 1:
                raise QueryError("the only supported having call is Condition() with a single condition")
            (subj, cond), = having.args.items()
            if subj not in ("count", "sum"):
                raise QueryError("Condition() only supports count or sum")
            pick = (lambda g: g[1]) if subj == "count" else (lambda g: g[2] if len(g) > 2 else 0)
            out = [g for g in out if _cond_holds(pick(g), cond)]
        if has_sort:
            keys = []
            for part in str(c.args["sort"]).split(","):
                w = part.split()
                if not w or w[0] not in ("count", "aggregate", "sum") or len(w) > 2 or (len(w) == 2 and w[1] not in ("asc", "desc")):
                    raise QueryError(f"invalid sorting directive: '{part.strip()}'")
                keys.append((1 if w[0] == "count" else 2, len(w) == 2 and w[1] == "asc"))
            for col, asc in reversed(keys):                       # stable sorts, last key first == sort.Stable on the tuple
                out.sort(key=lambda g: (g[col] if len(g) > col else 0), reverse=not asc)
        return self._window(c, out)

    # cells of the dense count tensor above which a GroupBy over set-like children takes fbgpu_groupby_sparse (128 MiB of
    # counts): a bound on memory, not a measured optimum.  A child of more than 65,535 rows takes it whatever the product.
    GROUPBY_DENSE_MAX_CELLS = 1 << 24

    def _groupby_sparse(self, idx, c, fields, row_ids, time_args, filt, start, shards, device_limit, sum_f=None):
        """(cells, counts) of a GroupBy over set-like children from fbgpu_groupby_sparse: the non-empty groups from the iterator's
        start position on, as row-major flat indices over the children's row lists, ascending; with device_limit (no sort, having or
        Sum, which skips groups after the fact) at most offset + limit of them.  With sum_f (the int field of aggregate=Sum),
        (cells, counts, sums) from fbgpu_groupby_sparse_sum in the same call: a count is the group's columns holding a value of
        the field, and a group is listed when it is non-zero.  None when the context answers FBGPU_E_COMM or has no such call:
        the dense tensor is asked for instead.  Count(Distinct) takes _groupby_sparse_distinct after the window is cut; Sum
        over a field that is not int takes the per-group composition, one query per group."""
        sizes = [len(r) for r in row_ids]
        flat0 = 0
        for p, n in zip(start, sizes):
            flat0 = flat0 * n + p
        lim = c.args.get("limit")
        limit = int(lim) + int(c.args.get("offset") or 0) if device_limit and lim else None
        set_dims = [(f.id, self._time_view_ids(f, targs) if targs else [VIEW_STANDARD], rows) for f, rows, targs in zip(fields, row_ids, time_args)]
        try:
            if sum_f is not None:
                return self.ctx.groupby_sparse(idx.id, set_dims, shards, filter_ops=filt, start=flat0, limit=limit,
                                               agg=(sum_f.id, VIEW_BSI, sum_f.bit_depth))
            return self.ctx.groupby_sparse(idx.id, set_dims, shards, filter_ops=filt, start=flat0, limit=limit)
        except NotImplementedError:
            return None
        except L.FbgpuError as e:
            if e.code != L.E_COMM:
                raise
            return None

    # (cell, x) pairs a fbgpu_groupby_sparse_distinct(_rows) call may produce, bounded before the call by Σ min(count, listed
    # x) over its cells: 2 GiB of keys over both halves of the device sort.  A bound on memory, not a measured optimum.
    GROUPBY_SPARSE_DISTINCT_PAIRS = 1 << 27

    def _groupby_sparse_distinct(self, idx, fields, row_ids, time_args, filt_call, agg_distinct, pairs, sparse, shards):
        """{cell: Count(Distinct(field=x))} for the listed groups `pairs` ((cell, group) in ascending cells) of a GroupBy on the
        sparse path, from fbgpu_groupby_sparse_distinct(_rows); cells absent from it have a distinct count of 0.  x's list is
        made once, as _groupby_distinct makes it, and the calls run over filter ∩ Distinct's child.  The cells are cut into
        consecutive ranges whose Σ min(count, listed x) stays within GROUPBY_SPARSE_DISTINCT_PAIRS, and x's list into disjoint
        slices that fit beside the cell in a 64-bit key; the pieces add up per cell.  None (the per-group composition runs
        instead) for Distinct(index=..), an x that is not a field of this index, more than 7 children, or a context that
        answers FBGPU_E_COMM or has no such call (a node)."""
        xf = idx.fields.get(agg_distinct.args.get("field", agg_distinct.args.get("_field")))
        if xf is None or "index" in agg_distinct.args or len(fields) > 7:
            return None
        call = "groupby_sparse_distinct" if xf.type == "int" else "groupby_sparse_distinct_rows"
        if not hasattr(self.ctx, call):
            return None
        if not pairs:
            return {}
        set_dims = [(f.id, self._time_view_ids(f, targs) if targs else [VIEW_STANDARD], rows) for f, rows, targs in zip(fields, row_ids, time_args)]
        counts = dict(zip((int(x) for x in sparse[0]), (int(n) for n in sparse[1])))
        total = math.prod(len(r) for r in row_ids)
        try:
            ops, xs = self._distinct_list(idx, filt_call, agg_distinct, xf, shards)
            got = {}
            if len(xs) == 0:
                return got
            room = self.GROUPBY_SPARSE_DISTINCT_PAIRS
            xbits = 0                                             # the widest x index the key leaves room for
            while xbits < 63 and total <= ((1 << 64) - 1) >> (xbits + 1):
                xbits += 1
            x_step = max(1, min(len(xs), room, 1 << xbits))
            for s in range(0, len(xs), x_step):
                xc = xs[s:s + x_step]
                x = (xf.id, VIEW_STANDARD, xc) if xf.type != "int" else (xf.id, VIEW_BSI, xf.bit_depth, xc)
                a = 0
                while a < len(pairs):
                    b, used = a, 0
                    while b < len(pairs) and (b == a or used + min(counts[pairs[b][0]], len(xc)) <= room):
                        used += min(counts[pairs[b][0]], len(xc))
                        b += 1
                    cells, dist = getattr(self.ctx, call)(idx.id, set_dims, x, shards, filter_ops=ops, start=pairs[a][0], end=pairs[b - 1][0] + 1)
                    for cell, d in zip(cells.tolist(), dist.tolist()):
                        got[cell] = got.get(cell, 0) + d
                    a = b
            return got
        except NotImplementedError:
            return None
        except L.FbgpuError as e:
            if e.code != L.E_COMM:
                raise
            return None

    def _distinct_list(self, idx, filt_call, agg_distinct, xf, shards):
        """(filter ∩ Distinct's child as ops, x's list there): an int field's distinct stored values (one Distinct), a set, mutex,
        bool or time field's rows that hold a column (one row-count call, as Distinct's set branch)"""
        parts = [x for x in (filt_call, *agg_distinct.children[:1]) if isinstance(x, pql.Call)]
        both = (parts[0] if len(parts) == 1 else pql.Call("Intersect", {}, parts)) if parts else None
        ops = self._bitmap_call(idx, both) if both is not None else None
        if xf.type == "int":
            return ops, self._int_values(idx, xf, shards, ops)
        rid, cnt = self.ctx.row_counts(idx.id, xf.id, VIEW_STANDARD, shards, filter_ops=ops)
        return ops, np.asarray(sorted(int(r) for r, n in zip(rid, cnt) if n > 0), dtype=np.uint64)

    GROUPBY_MIXED_MAX = 65535                                     # groups (product of the int children's value counts) per fbgpu_groupby_mixed / _sum / _distinct call
    # presence bits ((rows of the last set child, or 1) x groups x listed values or rows of x) per fbgpu_groupby_distinct(_rows) call: 256 MiB
    # of device workspace.  A choice that bounds the workspace, not a measured optimum.
    GROUPBY_DISTINCT_BITS = 1 << 31

    def _groupby_distinct(self, idx, fields, row_ids, time_args, int_dims, filt_call, agg_distinct, xf, shape, shards):
        """the Count(Distinct(field=xf)) tensor of a GroupBy (shape: the count tensor's), or None when the context answers
        FBGPU_E_COMM or has no such call (a node): the composition runs instead.  x's list is, for an int field, its stored values
        under filter ∩ Distinct's child (one Distinct, as the int children's lists are made), for a set, mutex, bool or time
        field the rows that hold a column there (one row-count call, as Distinct's set branch); the device then counts, per
        cell, those present under filter ∩ Distinct's child ∩ the cell's rows."""
        try:
            ops, xs = self._distinct_list(idx, filt_call, agg_distinct, xf, shards)
            if len(xs) == 0:
                return np.zeros(shape, dtype=np.uint64)
            return self._groupby_tensors(idx, fields, row_ids, time_args, int_dims, ops, shards, distinct=(xf, xs))[0]
        except NotImplementedError:
            return None
        except L.FbgpuError as e:
            if e.code != L.E_COMM:
                raise
            return None

    def _groupby_tensors(self, idx, fields, row_ids, time_args, int_dims, filt, shards, agg=None, distinct=None):
        """[counts] of a GroupBy with int children (positions int_dims), from fbgpu_groupby_mixed, or with agg (the int field of
        aggregate=Sum) [counts, sums] from fbgpu_groupby_sum, or with distinct = (x, its listed stored values) [distinct counts]
        from fbgpu_groupby_distinct (fbgpu_groupby_distinct_rows, with its listed row ids, when x is not an int field), where
        int_dims may be empty: the other children are the set dimensions (a time-range child
        with its covering views), the int children's values the trailing dimensions, moved back to the children's order.  No
        Row(v == value) per value and no scratch rows.  When the value lists' product exceeds GROUPBY_MIXED_MAX, each int child's
        list is cut into slices whose product fits and every combination of slices is one call: a column's value lies in exactly
        one slice per field, so the pieces tile the tensors.  x's list is cut so that each call's presence bits stay within
        GROUPBY_DISTINCT_BITS; the slices are disjoint, so their distinct counts add up per cell (a set-like x's list alike)."""
        set_k = [j for j in range(len(fields)) if j not in int_dims]
        set_dims = [(fields[j].id, self._time_view_ids(fields[j], time_args[j]) if time_args[j] else [VIEW_STANDARD], row_ids[j]) for j in set_k]
        stored = [[v - fields[k].base for v in row_ids[k]] for k in int_dims]      # values as the planes hold them (value - Base)
        step, room = [], self.GROUPBY_MIXED_MAX
        for vals in stored:
            step.append(max(1, min(len(vals), room)))
            room //= step[-1]
        shape = [len(row_ids[j]) for j in set_k] + [len(v) for v in stored]
        outs = [np.zeros(shape, dtype=np.uint64)] + ([np.zeros(shape, dtype=np.int64)] if agg is not None else [])
        x_cuts = [None]
        if distinct is not None:
            xf, xs = distinct
            per_value = (len(row_ids[set_k[-1]]) if set_k else 1) * int(np.prod(step, dtype=np.int64))    # bits per listed value
            x_step = max(1, self.GROUPBY_DISTINCT_BITS // per_value)
            x_cuts = [xs[s:s + x_step] for s in range(0, len(xs), x_step)]
        for starts in itertools.product(*[range(0, len(v), n) for v, n in zip(stored, step)]):
            cut = [slice(s, s + n) for s, n in zip(starts, step)]
            int_part = [(fields[k].id, VIEW_BSI, fields[k].bit_depth, v[c]) for k, v, c in zip(int_dims, stored, cut)]
            for xc in x_cuts:
                if distinct is not None and xf.type != "int":
                    got = [self.ctx.groupby_distinct_rows(idx.id, set_dims, int_part, (xf.id, VIEW_STANDARD, xc), shards, filter_ops=filt)]
                elif distinct is not None:
                    got = [self.ctx.groupby_distinct(idx.id, set_dims, int_part, (xf.id, VIEW_BSI, xf.bit_depth, xc), shards, filter_ops=filt)]
                elif agg is None:
                    got = [self.ctx.groupby_mixed(idx.id, set_dims, int_part, shards, filter_ops=filt)]
                else:
                    got = self.ctx.groupby_sum(idx.id, set_dims, int_part, (agg.id, VIEW_BSI, agg.bit_depth), shards, filter_ops=filt)
                for o, g in zip(outs, got):
                    o[(Ellipsis, *cut)] += g
        order = set_k + list(int_dims)
        return [np.transpose(o, [order.index(j) for j in range(len(fields))]) for o in outs]

    @staticmethod
    def _window(c, out):                                          # applyLimitAndOffsetToGroupByResult :3441-3459
        off = c.args.get("offset")
        if off is not None and int(off) < len(out):               # (an offset beyond the result is ignored, :3446)
            out = out[int(off):]
        lim = c.args.get("limit")
        return out[:lim] if lim else out

    def _groupby_start(self, c, row_ids):
        """position (one index per field) of the first group the iterator yields, or None when `previous` was the last
        group: newGroupByIterator :8779-8826 on one merged row list per field (the reference seeks per shard)"""
        n = len(row_ids)
        pos, ignore = [0] * n, False
        for i, ch in enumerate(c.children):
            rows = row_ids[i]
            prev = ch.args.get("previous")
            if prev is not None and not ignore:
                prev = int(prev) + (1 if i == n - 1 else 0)
                pos[i] = next((k for k, r in enumerate(rows) if r >= prev), len(rows))
            wrapped = pos[i] >= len(rows)
            if wrapped:
                if i == 0:
                    return None                                   # the first field's iterator does not wrap
                pos[i] = 0
            if prev is not None and not ignore and rows[pos[i]] != prev:
                ignore = True
            if wrapped:
                for j in range(i - 1, -1, -1):
                    pos[j] += 1
                    if pos[j] < len(row_ids[j]):
                        break
                    if j == 0:
                        return None
                    pos[j] = 0
        return pos


def _unravel(flat, shape):
    """np.unravel_index for a Python int over a shape whose size may exceed int64"""
    ix = []
    for n in reversed(shape):
        flat, i = divmod(flat, n)
        ix.append(i)
    return tuple(reversed(ix))


def _cond_holds(v, cond):
    op, x = cond.op, cond.value
    if op == "><":
        return x[0] <= v <= x[1]
    return {"==": v == x, "!=": v != x, "<": v < x, "<=": v <= x, ">": v > x, ">=": v >= x}[op]
