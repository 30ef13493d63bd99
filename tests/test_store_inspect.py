"""The shard store on a box without a GPU: an inspection-only context (fbgpu_init(FBGPU_DEVICE_NONE)) accepts the
residency calls and lets fbgpu_debug_container() locate containers with the very resolve() code the kernels inline, over
the host copies of the tables a commit would upload.  This pins, on the CPU: the fragment reader's hand-over to the store
builder, the descriptor / row / dense-directory tables, payload placement, array padding and (opt-in) striping, fragment
replacement and dropping, and fbgpu_load_rbf end to end.  Every query entry point must refuse such a context."""
import os
import subprocess
import sys

import numpy as np
import pytest

from featurebase_b200 import datagen as D
from featurebase_b200 import lib as L
from oracle import oracle as O
from tests import rbf_writer as W
from tests import test_rbf as TR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SW = 1 << 20


def container_values(found):
    typ, card, runs, payload = found
    if typ == 1:
        a = np.frombuffer(payload, dtype="<u2")
        assert len(a) == (card + 7) // 8 * 8 and set(a[card:].tolist()) <= {int(a[card - 1])}       # duplicate-padded tail
        return np.sort(a[:card]).astype(np.int64)
    if typ == 2:
        assert len(payload) == 8192
        v = np.flatnonzero(np.unpackbits(np.frombuffer(payload, dtype=np.uint8), bitorder="little"))
        assert len(v) == card
        return v.astype(np.int64)
    r = np.frombuffer(payload, dtype="<u2")[: 2 * runs].reshape(-1, 2).astype(np.int64)
    v = np.concatenate([np.arange(s, l + 1) for s, l in r.tolist()])
    assert len(v) == card
    return v


def check_fragment(ctx, index, field, view, shard, frag, rows_to_probe):
    """every (row, slot) of the oracle fragment resolves to exactly its container; absent ones resolve to nothing"""
    present = set(frag.rows().tolist())
    n = 0
    for row in rows_to_probe:
        bits = frag.row(row, 0).slice() if row in present else np.zeros(0, dtype=np.uint64)
        for slot in range(16):
            exp = bits[(bits >> np.uint64(16)) == np.uint64(slot)] & np.uint64(0xFFFF)
            got = ctx.debug_container(index, field, view, shard, row, slot)
            if len(exp) == 0:
                assert got is None, (row, slot)
            else:
                assert got is not None, (row, slot)
                assert np.array_equal(container_values(got), exp.astype(np.int64)), (row, slot)
                n += 1
    return n


def mixed_fragment(seed, shard, rows=(0, 1, 2, 3, 5, 6, 9, 40)):
    parts = [D.fragment(seed, shard, [0, 1, 2], 0.01), D.fragment(seed, shard, [3], 0.3), D.fragment(seed, shard, [5], 0.2, mode=1, mean_run=200.0),
             D.fragment(seed, shard, [6], 0.9, mode=1, mean_run=5000.0), D.fragment(seed, shard, [9], 0.0622), D.fragment(seed, shard, [40], 0.0001)]
    merged = O.Bitmap()
    for d in parts:
        merged = merged.union(O.Bitmap.from_bytes(d))
    return merged


def test_store_tables_and_payloads():
    ctx = L.Context(L.DEVICE_NONE)
    frags = {}
    for shard in (0, 3, 7):
        frags[shard] = mixed_fragment(11 + shard, shard)
        ctx.load_fragment(1, 2, 0, shard, frags[shard].to_bytes())
    # a second view with sparse row ids (search chain instead of the dense directory) and an official-format fragment
    sparse = O.Bitmap.from_values(np.concatenate([np.uint64(r * SW) + np.arange(0, 70000, 7, dtype=np.uint64) for r in (0, 5, 1000, 123456, 1 << 30)]))
    ctx.load_fragment(1, 3, 0, 0, sparse.to_bytes())
    ctx.load_fragment(1, 4, 0, 2, open(os.path.join(ROOT, "tests", "golden", "bitmapcontainer.roaringbitmap"), "rb").read())
    ctx.commit()
    st = ctx.stats()
    assert st["fragments"] == 5
    total = 0
    for shard, fr in frags.items():
        total += check_fragment(ctx, 1, 2, 0, shard, fr, [0, 1, 2, 3, 4, 5, 6, 7, 9, 40, 41])
    assert total > 300
    assert check_fragment(ctx, 1, 3, 0, 0, sparse, [0, 1, 5, 999, 1000, 1001, 123456, 1 << 30, (1 << 30) + 1]) == 10
    official = O.Bitmap.from_bytes(open(os.path.join(ROOT, "tests", "golden", "bitmapcontainer.roaringbitmap"), "rb").read())
    assert check_fragment(ctx, 1, 4, 0, 2, official, [0, 1]) == 2
    for args in ((1, 2, 0, 1, 0, 0), (1, 2, 1, 0, 0, 0), (9, 2, 0, 0, 0, 0), (1, 2, 0, 100000, 0, 0)):       # unknown shard / view / index
        assert ctx.debug_container(*args) is None
    # replacing and dropping a fragment
    newer = mixed_fragment(99, 3)
    ctx.load_fragment(1, 2, 0, 3, newer.to_bytes())
    assert check_fragment(ctx, 1, 2, 0, 3, newer, [0, 1, 2, 3, 5, 6, 9, 40]) > 80
    ctx.drop_fragment(1, 2, 0, 0)
    assert ctx.debug_container(1, 2, 0, 0, 0, 0) is None
    assert check_fragment(ctx, 1, 2, 0, 7, frags[7], [0, 3, 5]) > 30
    assert ctx.stats()["fragments"] == 4


def test_queries_are_refused_without_a_device():
    ctx = L.Context(L.DEVICE_NONE)
    ctx.load_fragment(0, 1, 0, 0, D.fragment(1, 0, [0, 1], 0.01))
    row = [L.Op(L.OP_ROW, 1, 0, 0, 0, 0, 0, 0)]
    for call in (lambda: ctx.count(0, row, [0]), lambda: ctx.row(0, row, [0]), lambda: ctx.row_counts(0, 1, 0, [0]),
                 lambda: ctx.count_pairs(0, 1, 0, [0], 1, 0, [1], [0]), lambda: ctx.groupby(0, [1, 1], [0, 0], [[0], [1]], [0]),
                 lambda: ctx.columns(0, row, [0]), lambda: ctx.extract(0, 2, 0, 8, [0], filter_ops=row), lambda: ctx.bsi_sum(0, 2, 0, 8, [0]),
                 lambda: ctx.bsi_minmax(0, 2, 0, 8, [0], True), lambda: ctx.bsi_select(0, 2, 0, 8, [0], [0]), lambda: ctx.any(0, row, [0]),
                 lambda: ctx.pair_types(0, 1, 0, 0, 1, 0, 1, [0]), lambda: ctx.row_counts(0, 1, 0, [0], row_ids=[0, 1], filter_ops=row),
                 lambda: ctx.row_counts_per_shard(0, 1, 0, [0], [0, 1])):
        with pytest.raises(L.FbgpuError) as e:
            call()
        assert e.value.code == L.E_CUDA and "no device" in str(e.value)


def test_query_argument_errors_without_a_device():
    """every query entry point rejects bad arguments with FBGPU_E_INVALID before it looks for a device, so the same table holds
    on a box without one; fbgpu_row_counts_per_shard answers an empty matrix before the device check"""
    import ctypes as C
    ctx = L.Context(L.DEVICE_NONE)
    node = L.Node([L.DEVICE_NONE, L.DEVICE_NONE], 1)
    lib, h = ctx.L, ctx.h
    op = L.ops_array([L.Op(L.OP_ROW, 1, 0, 0, 0, 0, 0, 0)])
    sh, rows, out = _u64([0]), _u64([0, 1]), _u64([0] * 64)
    u64, i64, i32 = C.c_uint64(0), C.c_int64(0), C.c_int32(0)
    p, u, v, w = sh.ctypes.data, C.byref(u64), C.byref(i64), C.byref(i32)
    null = "null argument"
    fields, views, nrow = np.ones(9, dtype=np.uint32), np.zeros(9, dtype=np.uint32), np.ones(9, dtype=np.int32)
    big = np.asarray([65536], dtype=np.int32)
    cases = [
        ("count null total", lib.fbgpu_count, (h, 0, op, 1, p, 1, None, None), null),
        ("count n_shards<0", lib.fbgpu_count, (h, 0, op, 1, p, -1, u, None), null),
        ("count null shards", lib.fbgpu_count, (h, 0, op, 1, None, 1, u, None), null),
        ("any null out", lib.fbgpu_any, (h, 0, op, 1, p, 1, None), null),
        ("any n_shards<0", lib.fbgpu_any, (h, 0, op, 1, p, -1, w), null),
        ("row null len", lib.fbgpu_row, (h, 0, op, 1, p, 1, None, 0, None, None), null),
        ("row n_shards<0", lib.fbgpu_row, (h, 0, op, 1, p, -1, None, 0, u, None), null),
        ("columns null n", lib.fbgpu_columns, (h, 0, op, 1, p, 1, 0, -1, out.ctypes.data, 8, None, None), null),
        ("columns n_shards<0", lib.fbgpu_columns, (h, 0, op, 1, p, -1, 0, -1, out.ctypes.data, 8, u, None), null),
        ("columns null cols", lib.fbgpu_columns, (h, 0, op, 1, p, 1, 0, -1, None, 8, u, None), null),
        ("extract null n", lib.fbgpu_extract, (h, 0, None, 0, 2, 0, 8, p, 1, 0, -1, out.ctypes.data, out.ctypes.data, 8, None, None), null),
        ("extract n_shards<0", lib.fbgpu_extract, (h, 0, None, 0, 2, 0, 8, p, -1, 0, -1, out.ctypes.data, out.ctypes.data, 8, u, None), null),
        ("extract null vals", lib.fbgpu_extract, (h, 0, None, 0, 2, 0, 8, p, 1, 0, -1, out.ctypes.data, None, 8, u, None), null),
        ("extract null ops", lib.fbgpu_extract, (h, 0, None, 1, 2, 0, 8, p, 1, 0, -1, out.ctypes.data, out.ctypes.data, 8, u, None), null),
        ("extract depth 65", lib.fbgpu_extract, (h, 0, None, 0, 2, 0, 65, p, 1, 0, -1, out.ctypes.data, out.ctypes.data, 8, u, None), "bit depth 65 outside 0..64"),
        ("minmax null val", lib.fbgpu_bsi_minmax, (h, 0, None, 0, 2, 0, 8, p, 1, 1, None, u), null),
        ("minmax n_shards<0", lib.fbgpu_bsi_minmax, (h, 0, None, 0, 2, 0, 8, p, -1, 1, v, u), null),
        ("minmax null ops", lib.fbgpu_bsi_minmax, (h, 0, None, 1, 2, 0, 8, p, 1, 1, v, u), null),
        ("minmax depth 65", lib.fbgpu_bsi_minmax, (h, 0, None, 0, 2, 0, 65, p, 1, 1, v, u), "bit depth 65 outside 0..64"),
        ("sum null count", lib.fbgpu_bsi_sum, (h, 0, None, 0, 2, 0, 8, p, 1, v, None), null),
        ("sum n_shards<0", lib.fbgpu_bsi_sum, (h, 0, None, 0, 2, 0, 8, p, -1, v, u), null),
        ("sum null ops", lib.fbgpu_bsi_sum, (h, 0, None, 1, 2, 0, 8, p, 1, v, u), null),
        ("sum depth 65", lib.fbgpu_bsi_sum, (h, 0, None, 0, 2, 0, 65, p, 1, v, u), "bit depth 65 outside 0..64"),
        ("select null total", lib.fbgpu_bsi_select, (h, 0, None, 0, 2, 0, 8, p, 1, rows.ctypes.data, 1, out.ctypes.data, None, None), null),
        ("select n_shards<0", lib.fbgpu_bsi_select, (h, 0, None, 0, 2, 0, 8, p, -1, rows.ctypes.data, 1, out.ctypes.data, None, u), null),
        ("select null ops", lib.fbgpu_bsi_select, (h, 0, None, 1, 2, 0, 8, p, 1, rows.ctypes.data, 1, out.ctypes.data, None, u), null),
        ("select null ranks", lib.fbgpu_bsi_select, (h, 0, None, 0, 2, 0, 8, p, 1, None, 1, out.ctypes.data, None, u), null),
        ("select depth 64", lib.fbgpu_bsi_select, (h, 0, None, 0, 2, 0, 64, p, 1, rows.ctypes.data, 1, out.ctypes.data, None, u), "bit depth 64 outside 0..63"),
        ("select 9 ranks", lib.fbgpu_bsi_select, (h, 0, None, 0, 2, 0, 8, p, 1, out.ctypes.data, 9, out.ctypes.data, None, u), "9 ranks: at most 8 per call"),
        ("row_counts null out", lib.fbgpu_row_counts, (h, 0, 1, 0, rows.ctypes.data, 2, None, 0, p, 1, None, None, 2, w), null),
        ("row_counts n_shards<0", lib.fbgpu_row_counts, (h, 0, 1, 0, rows.ctypes.data, 2, None, 0, p, -1, None, out.ctypes.data, 2, w), null),
        ("row_counts n_rows<0", lib.fbgpu_row_counts, (h, 0, 1, 0, rows.ctypes.data, -1, None, 0, p, 1, None, out.ctypes.data, 2, w), null),
        ("per_shard null out", lib.fbgpu_row_counts_per_shard, (h, 0, 1, 0, rows.ctypes.data, 2, None, 0, p, 1, None), null),
        ("per_shard null rows", lib.fbgpu_row_counts_per_shard, (h, 0, 1, 0, None, 2, None, 0, p, 1, out.ctypes.data), null),
        ("per_shard n_shards<0", lib.fbgpu_row_counts_per_shard, (h, 0, 1, 0, rows.ctypes.data, 2, None, 0, p, -1, out.ctypes.data), null),
        ("per_shard null ops", lib.fbgpu_row_counts_per_shard, (h, 0, 1, 0, rows.ctypes.data, 2, None, 1, p, 1, out.ctypes.data), null),
        ("pairs null out", lib.fbgpu_count_pairs, (h, 0, 1, 0, rows.ctypes.data, 1, 0, rows.ctypes.data, 2, p, 1, None), null),
        ("pairs null rows", lib.fbgpu_count_pairs, (h, 0, 1, 0, None, 1, 0, rows.ctypes.data, 2, p, 1, out.ctypes.data), null),
        ("pairs n_shards<0", lib.fbgpu_count_pairs, (h, 0, 1, 0, rows.ctypes.data, 1, 0, rows.ctypes.data, 2, p, -1, out.ctypes.data), null),
        ("pair_types null out", lib.fbgpu_pair_types, (h, 0, 1, 0, 0, 1, 0, 1, p, 1, None), null),
        ("pair_types n_shards<0", lib.fbgpu_pair_types, (h, 0, 1, 0, 0, 1, 0, 1, p, -1, out.ctypes.data), null),
        ("groupby null out", lib.fbgpu_groupby, (h, 0, fields.ctypes.data, views.ctypes.data, 2, rows.ctypes.data, nrow.ctypes.data, None, 0, p, 1, None), "bad argument"),
        ("groupby 0 fields", lib.fbgpu_groupby, (h, 0, fields.ctypes.data, views.ctypes.data, 0, rows.ctypes.data, nrow.ctypes.data, None, 0, p, 1, out.ctypes.data), "bad argument"),
        ("groupby 9 fields", lib.fbgpu_groupby, (h, 0, fields.ctypes.data, views.ctypes.data, 9, rows.ctypes.data, nrow.ctypes.data, None, 0, p, 1, out.ctypes.data), "bad argument"),
        ("groupby n_shards<0", lib.fbgpu_groupby, (h, 0, fields.ctypes.data, views.ctypes.data, 2, rows.ctypes.data, nrow.ctypes.data, None, 0, p, -1, out.ctypes.data), "bad argument"),
        ("groupby n_filter_ops<0", lib.fbgpu_groupby, (h, 0, fields.ctypes.data, views.ctypes.data, 2, rows.ctypes.data, nrow.ctypes.data, op, -1, p, 1, out.ctypes.data), "bad argument"),
        ("groupby null filter", lib.fbgpu_groupby, (h, 0, fields.ctypes.data, views.ctypes.data, 2, rows.ctypes.data, nrow.ctypes.data, None, 1, p, 1, out.ctypes.data), "bad argument"),
        # (the context form checks n_rows after the device check; the node form checks it before fanning out)
        ("node groupby n_rows 65536", lib.fbgpu_node_groupby, (node.h, 0, fields.ctypes.data, views.ctypes.data, 1, rows.ctypes.data, big.ctypes.data, None, 0, p, 1, out.ctypes.data),
         "n_rows[0]=65536 out of range"),
        ("node groupby 9 fields", lib.fbgpu_node_groupby, (node.h, 0, fields.ctypes.data, views.ctypes.data, 9, rows.ctypes.data, nrow.ctypes.data, None, 0, p, 1, out.ctypes.data), "bad argument"),
        ("node groupby n_filter_ops<0", lib.fbgpu_node_groupby, (node.h, 0, fields.ctypes.data, views.ctypes.data, 2, rows.ctypes.data, nrow.ctypes.data, op, -1, p, 1, out.ctypes.data),
         "bad argument"),
        ("node groupby null filter", lib.fbgpu_node_groupby, (node.h, 0, fields.ctypes.data, views.ctypes.data, 2, rows.ctypes.data, nrow.ctypes.data, None, 1, p, 1, out.ctypes.data),
         "bad argument"),
        ("node pairs n_pairs<0", lib.fbgpu_node_count_pairs, (node.h, 0, 1, 0, rows.ctypes.data, 1, 0, rows.ctypes.data, -1, p, 1, out.ctypes.data), null),
        ("node row_counts null ids", lib.fbgpu_node_row_counts, (node.h, 0, 1, 0, None, 2, None, 0, p, 1, out.ctypes.data), null),
    ]
    for name, fn, args, msg in cases:
        rc = fn(*args)
        assert rc == L.E_INVALID, (name, rc, lib.fbgpu_last_error())
        assert lib.fbgpu_last_error().decode() == msg, name
    # an empty matrix is answered before the device check
    for n_rows, n_shards in ((0, 1), (2, 0)):
        assert lib.fbgpu_row_counts_per_shard(h, 0, 1, 0, rows.ctypes.data, n_rows, None, 0, p, n_shards, out.ctypes.data) == 0
    node.close()
    ctx.close()


def _u64(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.uint64))


def test_rbf_loader_end_to_end():
    ctx = L.Context(L.DEVICE_NONE)
    bitmaps, frs = {}, {}
    for k, (name, fid) in enumerate((("~f;standard<", 5), ("~g;standard<", 6))):
        bm, conts = TR._fragment_containers(30 + k, 7)
        frs[fid], bitmaps[name] = bm, conts
    data = W.build(bitmaps)
    assert ctx.load_rbf(2, 7, data, ["~f;standard<", "~missing;standard<", "~g;standard<"], [5, 8, 6], [0, 0, 0]) == 2
    for fid, bm in frs.items():
        assert check_fragment(ctx, 2, fid, 0, 7, bm, [0, 1, 2, 3, 4, 5, 6, 9, 40]) > 100
    assert ctx.debug_container(2, 8, 0, 7, 0, 0) is None
    # WAL overlay: the newer content wins
    bm2, conts2 = TR._fragment_containers(77, 7)
    wa, wb = W.Writer(), W.Writer()
    wa.add_bitmap("~f;standard<", bitmaps["~f;standard<"])
    wb.add_bitmap("~f;standard<", conts2)
    old, new = wa.finish(1), wb.finish(2)
    assert ctx.load_rbf(2, 8, b"".join(old), ["~f;standard<"], [5], [0], wal=W.wal_between(old, new, wb.raw)) == 1
    assert check_fragment(ctx, 2, 5, 0, 8, bm2, [0, 1, 2, 3, 5, 6, 9, 40]) > 100
    with pytest.raises(L.FbgpuError):
        ctx.load_rbf(2, 9, TR.fixture("bad-bitmap"), ["x"], [1], [0])
    assert ctx.debug_container(2, 1, 0, 9, 0, 0) is None                 # a rejected file leaves the store unchanged
    # the same two databases from a shard directory the library maps itself (<dir>/data, <dir>/wal; wal absent or empty is fine)
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        for sub, d, w in (("a", data, None), ("b", b"".join(old), W.wal_between(old, new, wb.raw)), ("c", data, b"")):
            os.makedirs(os.path.join(tmp, sub))
            open(os.path.join(tmp, sub, "data"), "wb").write(d)
            if w is not None:
                open(os.path.join(tmp, sub, "wal"), "wb").write(w)
        assert ctx.load_rbf_dir(2, 17, os.path.join(tmp, "a"), ["~f;standard<", "~g;standard<"], [5, 6], [0, 0]) == 2
        assert ctx.load_rbf_dir(2, 18, os.path.join(tmp, "b"), ["~f;standard<"], [5], [0]) == 1
        assert ctx.load_rbf_dir(2, 19, os.path.join(tmp, "c"), ["~g;standard<"], [6], [0]) == 1
        with pytest.raises(L.FbgpuError, match="cannot map"):
            ctx.load_rbf_dir(2, 20, os.path.join(tmp, "nope"), ["~f;standard<"], [5], [0])
    for shard, fid, want in ((17, 5, frs[5]), (17, 6, frs[6]), (19, 6, frs[6])):
        got = {r: [ctx.debug_container(2, fid, 0, shard, r, sl) for sl in range(16)] for r in (0, 1, 2, 3)}
        ref = {r: [ctx.debug_container(2, fid, 0, 7, r, sl) for sl in range(16)] for r in (0, 1, 2, 3)}
        assert got == ref and any(x is not None for row in got.values() for x in row)      # (the file's keys are fragment-relative: same containers under any shard id)
    assert [ctx.debug_container(2, 5, 0, 18, r, 3) for r in range(6)] == [ctx.debug_container(2, 5, 0, 8, r, 3) for r in range(6)]


def test_striped_layout_in_a_subprocess():
    """the default payload order: array-dominated fragments are stored bank-striped (same sets), bitmap-heavy ones keep sorted
    arrays; FBGPU_ARRAY_SORTED=1 (read when a context is created) keeps every array sorted"""
    code = r"""
import sys, numpy as np
sys.path.insert(0, %r)
from featurebase_b200 import lib as L, datagen as D
from oracle import oracle as O
from tests.test_store_inspect import check_fragment, mixed_fragment
ctx = L.Context(L.DEVICE_NONE)
arrays = O.Bitmap.from_bytes(D.fragment(5, 0, [0, 1, 2, 3], 0.01))
ctx.load_fragment(0, 1, 0, 0, arrays.to_bytes())
assert check_fragment(ctx, 0, 1, 0, 0, arrays, [0, 1, 2, 3, 4]) == 64
t, card, runs, payload = ctx.debug_container(0, 1, 0, 0, 0, 0)
a = np.frombuffer(payload, dtype='<u2')[:card]
assert t == 1 and not np.all(a[:-1] <= a[1:]), 'array-dominated fragment should be striped'
dense = mixed_fragment(3, 1, rows=())
ctx.load_fragment(0, 2, 0, 1, O.Bitmap.from_bytes(D.fragment(6, 1, [0, 1, 2, 3, 4, 5, 6, 7, 8], 0.3)).union(O.Bitmap.from_bytes(D.fragment(6, 1, [9], 0.002))).to_bytes())
t, card, runs, payload = ctx.debug_container(0, 2, 0, 1, 9, 0)
a = np.frombuffer(payload, dtype='<u2')[:card]
assert t == 1 and card >= 64 and np.all(a[:-1] < a[1:]), 'arrays of a bitmap-heavy fragment stay sorted'
print('striped ok')
""" % ROOT
    env = dict(os.environ)
    env.pop("FBGPU_ARRAY_SORTED", None)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert out.returncode == 0 and "striped ok" in out.stdout, out.stderr[-3000:]


def test_executor_bodies_through_library_compiler_and_store(monkeypatch):
    """the executor-level test bodies once more, with Count / Row answered from the LIBRARY's compiled program and the
    LIBRARY's store (tests/inspect_ctx.InspectCtx); only the kernels' stack machine is modelled in Python"""
    from tests import oracle_exec
    from tests import test_gpu_parity as G
    from tests import test_zz_gpu_executor_goldens as Z
    from tests import test_zz_gpu_experimental as E
    from tests.inspect_ctx import InspectCtx

    def make(*a, **kw):
        return oracle_exec.Pair(*a, ctx=InspectCtx(), **kw)
    for mod in (G, Z, E):
        monkeypatch.setattr(mod, "Pair", make)
    G.test_executor_goldens_and_edge_semantics()
    G.test_config1_single_shard_plumbing()
    G.test_bsi_range_goldens_on_gpu()
    Z.test_executor_bsi_goldens_on_gpu()
    E.test_time_quantum_rows()
    E.test_embedded_rows_constrow_unionrows()
    E.test_rbf_loader_matches_fragment_loader()
    E.test_bsi_aggregate_goldens()
    E.test_fragment_top_goldens()
    E.test_topn_cutoff_goldens()
    E.test_filter_sample_goldens()
    E.test_groupby_postprocessing_goldens()
    E.test_shift_and_includes_column()
    E.test_all_with_limit_offset()
    E.test_min_max_row()
    E.test_various_queries_goldens()
    E.test_distinct_random()
    E.test_columns_entry_point()
    E.test_extract_entry_point()
    E.test_extract_table_golden()
    E.test_sort_goldens()
    E.test_field_value_and_options()
    E.test_topk_time_range()
    E.test_mixed_container_goldens_on_device()
    E.test_kernel_table_goldens_on_device()            # explicit (unoptimised) encodings through the library's reader and store
    E.test_bitmap_level_goldens_on_device()
    E.test_bench_archetype_matrix()


def test_algorithmic_byte_accounting():
    """fbgpu_rows_payload_bytes (the roofline numerator of bench.py, SURVEY §8d) = Σ payload bytes (array 2n, bitmap 8192,
    run 4r) and the container count of the named rows, checked against the stored containers one by one"""
    ctx = L.Context(L.DEVICE_NONE)
    shards = [0, 2, 5]
    for s in shards:
        ctx.load_fragment(0, 1, 0, s, mixed_fragment(40 + s, s).to_bytes())
    for rows in ([0, 1], [3], [5, 6, 9], [0, 1, 2, 3, 5, 6, 9, 40, 77], None):
        pay = cont = 0
        for s in shards:
            for row in (rows if rows is not None else [0, 1, 2, 3, 5, 6, 9, 40]):
                for slot in range(16):
                    found = ctx.debug_container(0, 1, 0, s, row, slot)
                    if found:
                        typ, card, runs, _ = found
                        pay += 2 * card if typ == 1 else 8192 if typ == 2 else 4 * runs
                        cont += 1
        assert ctx.rows_payload_bytes(0, 1, 0, shards, rows) == (pay, cont), rows
    assert ctx.rows_payload_bytes(0, 1, 0, [9], [0]) == (0, 0)
    assert ctx.rows_payload_bytes(0, 7, 0, shards, [0]) == (0, 0)


def test_failed_batch_load_leaves_the_store_unchanged():
    """ADVICE r1: a batch load that fails half way (here: a shard id past the accepted range) must not leave the earlier fragments
    of the batch live with unwritten payloads, nor drop the fragments they were about to replace."""
    from featurebase_b200 import datagen as D
    from featurebase_b200 import lib as L
    ctx = L.Context(L.DEVICE_NONE)
    old = D.fragment(7, 0, [0, 1], 0.01)
    ctx.load_fragment(0, 0, 0, 0, old)
    kept = ctx.debug_container(0, 0, 0, 0, 0, 3)
    assert kept is not None
    before = ctx.stats()
    new0, new1 = D.fragment(8, 0, [0, 1, 2], 0.02), D.fragment(8, 1, [0], 0.02)
    buf = np.frombuffer(new0 + new1, dtype=np.uint8)
    offs = np.array([0, len(new0), len(new0) + len(new1)], dtype=np.uint64)
    with pytest.raises(L.FbgpuError):
        ctx.load_fragments(0, 0, 0, np.array([0, 1 << 40], dtype=np.uint64), buf, offs)
    after = ctx.stats()
    assert after == before
    assert ctx.debug_container(0, 0, 0, 0, 0, 3) == kept          # the replaced fragment is live again, payload intact
    assert ctx.debug_container(0, 0, 0, 0, 2, 0) is None           # nothing of the failed batch is visible
    # and the store still accepts the same data once the bad shard id is gone
    ctx.load_fragments(0, 0, 0, np.array([0, 1], dtype=np.uint64), buf, offs)
    assert ctx.debug_container(0, 0, 0, 0, 2, 0) is not None
    assert ctx.debug_container(0, 0, 0, 1, 0, 0) is not None
    ctx.close()


def _container_bitmap(frag, keys):
    """roaring bytes of ONLY the containers `keys` of an oracle fragment (what a write transaction's PutContainer calls carry)"""
    vals = frag.slice()
    sel = vals[np.isin(vals >> np.uint64(16), np.asarray(sorted(keys), dtype=np.uint64))]
    return O.Bitmap.from_values(sel).to_bytes()


def test_apply_containers_incremental_refresh():
    """fbgpu_apply_containers (Tx.PutContainer / RemoveContainer mirror): written containers replace / add, removed keys vanish, untouched
    containers keep their payload in place; small updates are committed by patching the tables, not by rebuilding them."""
    rng = np.random.default_rng(5)
    ctx = L.Context(L.DEVICE_NONE)
    rows = [0, 1, 2, 3, 4, 5, 6, 7, 9, 40, 41]
    frags = {s: mixed_fragment(21 + s, s) for s in (0, 1, 2)}
    for s, fr in frags.items():
        ctx.load_fragment(1, 2, 0, s, fr.to_bytes())
    ctx.commit()
    st0 = ctx.stats()
    assert st0["full_commits"] == 1 and st0["patch_commits"] == 0
    model = {s: fr.slice() for s, fr in frags.items()}
    for step in range(6):
        s = int(rng.integers(0, 3))
        cur = model[s]
        keys = np.unique(cur >> np.uint64(16))
        written = set(int(k) for k in rng.choice(keys, size=min(4, len(keys)), replace=False))
        written |= {int(rng.integers(0, 16)) + 16 * int(r) for r in rng.choice([1, 8, 40, 41, 42], size=2)}       # keys in existing and in new rows
        removed = set(int(k) for k in rng.choice(keys, size=3, replace=False)) - written
        new_vals = []
        for k in sorted(written):
            kind = int(rng.integers(0, 3))
            n = [int(rng.integers(1, 300)), int(rng.integers(5000, 30000)), 65536][kind]
            lo = rng.choice(65536, size=n, replace=False) if n < 65536 else np.arange(65536)
            if kind == 2:
                lo = np.arange(int(rng.integers(0, 1000)), int(rng.integers(30000, 65536)))                        # one long run
            new_vals.append((np.uint64(k) << np.uint64(16)) | np.sort(lo).astype(np.uint64))
        new_vals = np.concatenate(new_vals)
        keep = cur[~np.isin(cur >> np.uint64(16), np.asarray(sorted(written | removed), dtype=np.uint64))]
        model[s] = np.sort(np.concatenate([keep, new_vals]))
        ctx.apply_containers(1, 2, 0, s, O.Bitmap.from_values(new_vals).to_bytes(), sorted(removed))
        want = O.Bitmap.from_values(model[s])
        assert check_fragment(ctx, 1, 2, 0, s, want, rows + [8, 42]) > 50
        for other in (0, 1, 2):                                                                                   # the neighbours are untouched
            if other != s:
                assert check_fragment(ctx, 1, 2, 0, other, O.Bitmap.from_values(model[other]), [0, 3, 9]) > 10
    st = ctx.stats()
    assert st["fragments"] == 3 and st["dead_bytes"] > 0
    # rows 41 / 42 lie past the dense directory's range the first time they appear (full rebuild); every later update is a patch
    assert st["patch_commits"] >= 3 and st["full_commits"] <= 3, st
    assert st["payload_bytes"] == sum(_payload_bytes(O.Bitmap.from_values(model[s])) for s in model)
    # a key both written and removed, and a malformed delta, change nothing
    before = ctx.stats()
    with pytest.raises(L.FbgpuError):
        ctx.apply_containers(1, 2, 0, 0, _container_bitmap(O.Bitmap.from_values(model[0]), [0]), [0])
    with pytest.raises(L.FbgpuError):
        ctx.apply_containers(1, 2, 0, 0, b"\x3c\x30\x00\x00\xff\xff\xff\x7f", [])
    after = ctx.stats()
    assert {k: v for k, v in after.items() if 'commits' not in k} == {k: v for k, v in before.items() if 'commits' not in k}
    # removing every container drops the fragment; applying to a shard that is not resident creates it
    keys0 = np.unique(model[0] >> np.uint64(16)).tolist()
    ctx.apply_containers(1, 2, 0, 0, b"", keys0)
    assert ctx.stats()["fragments"] == 2 and ctx.debug_container(1, 2, 0, 0, 0, 0) is None
    fresh = mixed_fragment(77, 5)
    ctx.apply_containers(1, 2, 0, 5, fresh.to_bytes(), [123456])
    assert check_fragment(ctx, 1, 2, 0, 5, fresh, rows) > 80


def _payload_bytes(bm):
    data = bm.to_bytes()
    n = int(np.frombuffer(data[4:8], dtype="<u4")[0])
    hdr = np.frombuffer(data[8:8 + 12 * n], dtype=np.dtype([("key", "<u8"), ("typ", "<u2"), ("n1", "<u2")]))
    tot = int(2 * (hdr["n1"][hdr["typ"] == 1].astype(np.int64) + 1).sum()) + 8192 * int((hdr["typ"] == 2).sum())
    for j in np.nonzero(hdr["typ"] == 3)[0]:
        off = int(np.frombuffer(data[8 + 12 * n + 4 * j: 12 + 12 * n + 4 * j], dtype="<u4")[0])
        tot += 4 * int(np.frombuffer(data[off:off + 2], dtype="<u2")[0])
    return tot
