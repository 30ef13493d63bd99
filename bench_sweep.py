#!/usr/bin/env python3
"""bench_sweep.py — secondary measurements on one GPU (BASELINE configs 3, 4, 5); prints one JSON line per point.

  config 5: density sweep p in {0.01 %..50 %} x {uniform, clustered}, Count(Intersect(Row a, Row b)) over 1024 shards
            (fused pair_count_kernel); row pairs are rotated between steps so that the touched data exceeds L2.
  config 3: BSI Count(Row(v > k)) over 10 M records, 32-bit values (eval_kernel plane sweep).
  config 4: GroupBy(Rows(a), Rows(b)) 256 x 256 over this GPU's share (512 shards) of 100 M records / 4096 shards.
  config X: fbgpu_columns / fbgpu_extract (device-side column-id and int-value expansion), wall clock; R: fbgpu_row.
  config P: Percentile over config X's 32-bit field, order statistics (fbgpu_bsi_select) against the query-driven bisection
            (only when named in --configs).
  config V: GroupBy(Rows(a), Rows(v)) with v an int field of 64 / 1000 / 65535 distinct values, fbgpu_groupby_values against the
            Row(v == value)-per-value composition (only when named in --configs).
  config T: TopK(f, from=, to=) and GroupBy(Rows(a), Rows(f, from=, to=)) over 48 views of a quantum-YMD field,
            fbgpu_row_counts_views / fbgpu_groupby_views against the operand-row composition (only when named in --configs).
  config M: GroupBy(Rows(a), Rows(v), Rows(w)) and GroupBy(Rows(t, from=, to=), Rows(v)) with int fields of 8 / 64 / 256
            distinct values each, fbgpu_groupby_mixed against the composition (only when named in --configs).
  config S: GroupBy(Rows(a), aggregate=Sum(field=v)), the same with Rows(b) or Rows(w) beside a, fbgpu_groupby_sum against the
            Sum-per-group composition (only when named in --configs).
  config D: GroupBy(Rows(a), aggregate=Count(Distinct(field=v))), the same with Rows(w) or Rows(b) beside a, on config S's data,
            fbgpu_groupby_distinct against the Distinct-per-group composition (only when named in --configs).
  config K: GroupBy(Rows(a), aggregate=Count(Distinct(field=x))) and the same with Rows(b) beside a, for x a mutex field of
            100,000 rows and a set field of 64 rows, on config D's data, fbgpu_groupby_distinct_rows against the
            Distinct-per-group composition (only when named in --configs).
  config G: fbgpu_groupby_sparse against fbgpu_groupby on config S's 256 x 256 GroupBy(Rows(a), Rows(b)), against the host
            composition (one fbgpu_extract_rows per dimension and a numpy join) for a 1,000,000-row mutex field x a, and paged
            with limit=1000 (only when named in --configs).
  config H: config G's data with aggregate=Sum(field=v): GroupBy(Rows(m), aggregate=Sum(field=v), limit=1000) through the
            executor, fbgpu_groupby_sparse_sum against the sparse list plus one Sum per group; m x a with Sum against the
            counts-only sparse call; a x b with Sum against fbgpu_groupby_sum (only when named in --configs).
  config J: config G's data with aggregate=Count(Distinct): GroupBy(Rows(m), aggregate=Count(Distinct(field=v)), limit=1000)
            through the executor, fbgpu_groupby_sparse_distinct against the sparse list plus one Distinct per group; m x a with
            Count(Distinct(field=b)) against the counts-only sparse call; a x b with Count(Distinct(field=w)) against
            fbgpu_groupby_distinct (only when named in --configs).
  config N: TopN(f, Row(src=0), tanimotoThreshold=50) and TopN(f, Row(src=0), threshold=100) over --topn-rows rows of varied
            cardinality, fbgpu_topn_cutoffs against the per-shard count-matrix composition (only when named in --configs).
  config O: Sort over config X's 32-bit field with and without a limit, fbgpu_bsi_sort against extracting every value and
            sorting on the host (only when named in --configs).
  config E: Extract over a 256-row set field, a 64-row mutex field and a bool field, and Sort over the mutex field, on 512
            shards, fbgpu_extract_rows against the per-row column-expansion composition (only when named in --configs).
Every point is spot-checked against the CPU oracle on a few shards (the checker, not the thing measured)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
SW = 1 << 20


def peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    try:
        return float(json.load(open(p))["hbm_gbs"]), "measured"
    except Exception:
        return 3350.0, "H100 SXM data sheet"


def timed(ctx, fn, steps, warmup=3):
    for i in range(warmup):
        fn(i)
    ms = []
    t0 = time.perf_counter()
    for i in range(steps):
        fn(i)
        ms.append(ctx.counters()["last_query_gpu_ms"])
    wall = (time.perf_counter() - t0) / steps * 1e3
    return float(np.mean(ms)), float(np.min(ms)), wall


def config5(args, out):
    from featurebase_b200 import datagen as D, executor as X, lib as L
    from oracle import oracle as O
    pk, src = peak()
    S = args.shards
    shards = np.arange(S, dtype=np.uint64)
    for mode, mname in ((0, "uniform"), (1, "clustered")):
        if mname not in args.generators.split(","):
            continue
        for p in [float(x) for x in args.densities.split(",")]:
            per_pair = 2 * S * 16 * max(2 * p * 65536, 16)
            n_pairs = int(min(8, max(2, np.ceil(300e6 / max(per_pair, 1)))))
            if p >= 0.0625 and mode == 0:
                n_pairs = 2
            rows = list(range(2 * n_pairs))
            h = X.Holder()
            idx = h.create_index("i", track_existence=False)
            f = idx.create_field("f")
            bulk = D.fragments(11 + mode, shards, rows, p, mode=mode, mean_run=64.0)
            h.ctx.load_fragments(idx.id, f.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
            h.ctx.commit()
            st = h.ctx.stats()
            progs = [[L.Op(L.OP_ROW, f.id, 0, 0, 2 * k, 0, 0, 0), L.Op(L.OP_ROW, f.id, 0, 0, 2 * k + 1, 0, 0, 0), L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)] for k in range(n_pairs)]
            counts = {}

            def step(i):
                k = i % n_pairs
                counts[k] = h.ctx.count(idx.id, progs[k], shards)

            ms, ms_min, wall = timed(h.ctx, step, args.steps)
            pay, nc = h.ctx.rows_payload_bytes(idx.id, f.id, X.VIEW_STANDARD, shards, [0, 1])
            algo = pay + 16 * nc + 8
            # oracle spot check: pair 0 on 2 shards
            tot, per = h.ctx.count(idx.id, progs[0], shards, per_shard=True)
            for s in (0, S - 1):
                fr = O.Bitmap.from_bytes(bulk.fragment_bytes(s))
                assert int(per[s]) == fr.row(0, s).intersection_count(fr.row(1, s)), (mname, p, s)
            assert tot == counts[0]
            gbs = algo / (ms * 1e-3) / 1e9
            out({"config": 5, "generator": mname, "density": p, "shards": S, "kernel": "pair_count_kernel", "ms": ms, "ms_min": ms_min, "wall_ms": wall,
                 "set_ops_per_sec": S / (ms * 1e-3), "count_rows_per_sec": S / (ms * 1e-3), "columns_per_sec": S * SW / (ms * 1e-3),
                 "algorithmic_bytes": int(algo), "achieved_gbs": gbs, "peak_gbs": pk, "peak_source": src, "frac": gbs / pk,
                 "l2_note": f"{n_pairs} row pairs rotated, {n_pairs * algo / 1e6:.0f} MB touched per cycle" + (" (< L2: launch/L2-bound point)" if n_pairs * algo < 50e6 else ""),
                 "containers": {"array": st["array_containers"], "bitmap": st["bitmap_containers"], "run": st["run_containers"]}, "count": int(tot)})
            if args.batched:
                # the same Intersect+Count, N independent row pairs fused in one launch (SURVEY §8d "(ii) batched")
                nb = max(n_pairs, 4)
                ra, rb = [2 * (k % n_pairs) for k in range(nb)], [2 * (k % n_pairs) + 1 for k in range(nb)]
                res = {}

                def bstep(i):
                    res[0] = h.ctx.count_pairs(idx.id, f.id, 0, ra, f.id, 0, rb, shards)

                bms, bmin, bwall = timed(h.ctx, bstep, args.steps)
                for k in range(n_pairs):                         # (fewer timed steps than row pairs: count the ones the rotation did not reach)
                    if k not in counts:
                        counts[k] = h.ctx.count(idx.id, progs[k], shards)
                assert int(res[0][0]) == counts[0] and int(res[0].sum()) == sum(counts[k % n_pairs] for k in range(nb))
                bgbs = nb * algo / (bms * 1e-3) / 1e9
                out({"config": "5b", "generator": mname, "density": p, "shards": S, "pairs_per_launch": nb, "kernel": "pair_count_kernel (multi-pair)", "ms": bms, "ms_min": bmin, "wall_ms": bwall,
                     "set_ops_per_sec": nb * S / (bms * 1e-3), "algorithmic_bytes": int(nb * algo), "achieved_gbs": bgbs, "peak_gbs": pk, "peak_source": src, "frac": bgbs / pk,
                     "l2_note": f"{nb} pairs over {n_pairs} distinct row pairs ({n_pairs * algo / 1e6:.0f} MB distinct data)"})
            h.ctx.close()


def config_row(args, out):
    """Row-returning calls (canonical Pilosa-roaring bytes to the host): fbgpu_row end to end, wall clock"""
    from featurebase_b200 import datagen as D, executor as X, pql
    from oracle import oracle as O
    S = args.shards
    shards = np.arange(S, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    f = idx.create_field("f")
    ex = X.Executor(h)
    bulk = D.fragments(11, shards, [0, 1, 2, 3], 0.01)
    h.ctx.load_fragments(idx.id, f.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
    h.ctx.commit()
    idx.shards.update(range(S))
    for q in ("Intersect(Row(f=0), Row(f=1))", "Union(Row(f=0), Row(f=1), Row(f=2), Row(f=3))", "Row(f=0)"):
        ops = ex._bitmap_call(idx, pql.parse(q)[0])
        data, cnt = h.ctx.row(idx.id, ops, shards)               # (also sizes the buffer below)
        buf = np.zeros(len(data) + 4096, dtype=np.uint8)         # caller-owned and reused, as a Go caller would: pages already mapped
        for _ in range(2):
            h.ctx.row_into(idx.id, ops, shards, buf)
        t0 = time.perf_counter()
        n = 5
        for _ in range(n):
            need, cnt, fits = h.ctx.row_into(idx.id, ops, shards, buf)
        wall = (time.perf_counter() - t0) / n * 1e3
        assert fits and buf[:need].tobytes() == data
        # oracle spot check: the first shard's segment
        fr = O.Bitmap.from_bytes(bulk.fragment_bytes(0))
        call = pql.parse(q)[0]
        from tests.oracle_exec import OracleIndex
        oi = OracleIndex(idx)
        oi.load("f", 0, 0, bulk.fragment_bytes(0))
        sub, _ = h.ctx.row(idx.id, ops, [0])
        assert sub == oi.eval_row(call, [0]).to_bytes()
        out({"config": "R", "query": q, "shards": S, "kernel": "eval_kernel + canon_emit_kernel + host assembly", "ms": wall, "result_bytes": len(data), "result_count": int(cnt),
             "columns_per_sec": S * SW / (wall * 1e-3), "frac": 0.0, "achieved_gbs": 0.0, "note": "wall clock of fbgpu_row() into a reused caller buffer: evaluate, {N,runs} D2H, encoding choice on host, emit, payload D2H, roaring assembly"})
    h.ctx.close()


def config_extract(args, out):
    """Column-id and value expansion on the device: fbgpu_columns over a 1 % row, fbgpu_extract over a 32-bit int field
    (10 M records), wall clock through the C ABI; every result is checked against the data generator"""
    from featurebase_b200 import datagen as D, executor as X, pql, roaring_io
    S = args.shards
    shards = np.arange(S, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    f = idx.create_field("f")
    v = idx.create_field("v", "int", min=0, max=(1 << 32) - 1)
    ex = X.Executor(h)
    bulk = D.fragments(11, shards, [0, 1], 0.01)
    h.ctx.load_fragments(idx.id, f.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
    n_rec = min(10_000_000, S * SW)
    n_sh = (n_rec + SW - 1) // SW
    for s in range(n_sh):
        h.ctx.load_fragment(idx.id, v.id, X.VIEW_BSI, s, D.bsi_fragment(12, s, min(SW, n_rec - s * SW), 32, 0, (1 << 32) - 1))
    h.ctx.commit()
    idx.shards.update(range(S))

    def timed(fn, n=5):
        for _ in range(2):
            r = fn()
        t0 = time.perf_counter()
        for _ in range(n):
            r = fn()
        return r, (time.perf_counter() - t0) / n * 1e3

    ops = ex._bitmap_call(idx, pql.parse("Union(Row(f=0), Row(f=1))")[0])
    (cols, total), wall = timed(lambda: h.ctx.columns(idx.id, ops, shards))
    want = roaring_io.decode(h.ctx.row(idx.id, ops, shards)[0])
    assert total == len(want) and np.array_equal(cols, np.asarray(want, dtype=np.uint64))
    out({"config": "X", "query": "columns of Union(Row(f=0), Row(f=1)) at 1 %", "shards": S, "kernel": "eval_kernel + columns_emit_kernel", "ms": wall, "columns": int(total),
         "columns_per_sec": float(total) / (wall * 1e-3), "frac": 0.0, "achieved_gbs": 0.0, "note": "wall clock of fbgpu_columns(): evaluate, N per unit D2H, expand ids on the device, ids D2H"})
    bsh = np.arange(n_sh, dtype=np.uint64)
    (c2, vals, tot2), wall = timed(lambda: h.ctx.extract(idx.id, v.id, X.VIEW_BSI, 32, bsh), n=3)
    assert tot2 == n_rec and len(c2) == n_rec
    for i in (0, 1, n_rec // 2, n_rec - 1):
        assert int(vals[i]) == D.bsi_value(12, int(c2[i]) // SW, int(c2[i]) % SW, 0, (1 << 32) - 1)
    out({"config": "X", "query": "values of a 32-bit int field, all records", "records": n_rec, "kernel": "eval_kernel + columns_emit_kernel + extract_values_kernel", "ms": wall,
         "records_per_sec": n_rec / (wall * 1e-3), "frac": 0.0, "achieved_gbs": 0.0, "note": "wall clock of fbgpu_extract(): 34 planes read once, 16 B per record D2H"})
    # the one-pass aggregates, cross-checked against the extracted value vector
    (tot, cnt), wall = timed(lambda: h.ctx.bsi_sum(idx.id, v.id, X.VIEW_BSI, 32, bsh))
    assert cnt == n_rec and tot == int(vals.astype(object).sum())
    out({"config": "X", "query": "Sum(field=v), 32-bit, all records", "records": n_rec, "kernel": "eval_kernel + bsi_sum_kernel", "ms": wall, "records_per_sec": n_rec / (wall * 1e-3),
         "frac": 0.0, "achieved_gbs": 0.0, "note": "wall clock of fbgpu_bsi_sum()"})
    for want_max in (False, True):
        (val, n), wall = timed(lambda: h.ctx.bsi_minmax(idx.id, v.id, X.VIEW_BSI, 32, bsh, want_max))
        ref = int(vals.max() if want_max else vals.min())
        assert (val, n) == (ref, int((vals == ref).sum()))
        out({"config": "X", "query": ("Max" if want_max else "Min") + "(field=v), 32-bit, all records", "records": n_rec, "kernel": "eval_kernel + bsi_minmax_kernel", "ms": wall,
             "records_per_sec": n_rec / (wall * 1e-3), "frac": 0.0, "achieved_gbs": 0.0, "note": "wall clock of fbgpu_bsi_minmax()"})
    h.ctx.close()


class _KernelMs:
    """a context proxy that sums last_query_gpu_ms over every library query issued through it"""

    def __init__(self, ctx):
        self.ctx, self.ms = ctx, 0.0

    def __getattr__(self, name):
        fn = getattr(self.ctx, name)
        if name in ("counters", "close", "commit") or not callable(fn):
            return fn

        def call(*a, **kw):
            r = fn(*a, **kw)
            self.ms += self.ctx.counters()["last_query_gpu_ms"]
            return r
        return call


def config_percentile(args, out):
    """Percentile(field=v, nth) over config X's data (10 M records, 32-bit values), with and without a 1 % filter row, through
    the executor: the select arm (one Count + one fbgpu_bsi_select) and the bisection arm (Count, Min, Max, then up to two
    Counts per bisection step), alternated query by query.  Both arms must give the same ValCount."""
    from featurebase_b200 import datagen as D, executor as X
    n_rec = min(10_000_000, args.shards * SW)
    n_sh = (n_rec + SW - 1) // SW
    shards = np.arange(n_sh, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    f = idx.create_field("f")
    v = idx.create_field("v", "int", min=0, max=(1 << 32) - 1)
    bulk = D.fragments(11, shards, [0], 0.01)
    h.ctx.load_fragments(idx.id, f.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
    for s in range(n_sh):
        h.ctx.load_fragment(idx.id, v.id, X.VIEW_BSI, s, D.bsi_fragment(12, s, min(SW, n_rec - s * SW), 32, 0, (1 << 32) - 1))
    h.ctx.commit()
    idx.shards.update(range(n_sh))
    real = h.ctx
    h.ctx = prox = _KernelMs(real)
    arms = {"select": X.Executor(h), "bisection": X.Executor(h)}
    arms["bisection"].percentile_select = False
    for nth in (1, 50, 99.9):
        for q_filter in (False, True):
            q = f"Percentile(field=v, nth={nth}" + (", filter=Row(f=0))" if q_filter else ")")
            rec = {name: {"wall": [], "kernel_ms": [], "queries": []} for name in arms}
            res = {}
            for i in range(2 + args.steps):                  # two warm-up rounds, then alternate the arms
                for name in (("select", "bisection") if i % 2 == 0 else ("bisection", "select")):
                    q0, prox.ms = real.counters()["queries"], 0.0
                    t0 = time.perf_counter()
                    r = arms[name].execute("i", q)[0]
                    wall = (time.perf_counter() - t0) * 1e3
                    res.setdefault(name, r)
                    assert r == res[name], (q, name)
                    if i >= 2:
                        rec[name]["wall"].append(wall)
                        rec[name]["kernel_ms"].append(prox.ms)
                        rec[name]["queries"].append(real.counters()["queries"] - q0)
            assert res["select"] == res["bisection"], (q, res)
            for name, d in rec.items():
                out({"config": "P", "query": q, "arm": name, "records": n_rec, "shards": n_sh, "result": [res[name].val, res[name].count],
                     "wall_ms": float(np.median(d["wall"])), "wall_ms_min": float(np.min(d["wall"])), "wall_ms_max": float(np.max(d["wall"])),
                     "kernel_ms": float(np.median(d["kernel_ms"])), "queries": int(np.median(d["queries"])), "steps": args.steps,
                     "kernel": "eval_kernel + bsi_select_step_kernel + bsi_select_decide_kernel" if name == "select" else "eval_kernel + bsi_minmax_kernel (Count / Min / Max / bisection Counts)",
                     "note": "median over the timed steps of the executor call (wall clock) and of the summed last_query_gpu_ms of its library queries"})
    real.close()


class _NoGroupByValues(_KernelMs):
    """the same proxy without groupby_values / groupby_mixed: the executor takes the Row(v == value)-per-value composition"""

    def __getattr__(self, name):
        if name in ("groupby_values", "groupby_mixed"):
            raise AttributeError(name)
        return super().__getattr__(name)


def config_groupby_values(args, out):
    """GroupBy(Rows(a), Rows(v)) over --groupby-shards shards: int fields v holding one of D values (uniform) for each of the first
    16,384 columns of every shard, D in {64, 1000, 65535}, and a 256-row set field a at 1/256 density per row, without and with a
    1 % filter row, through the executor.  The device arm (one fbgpu_groupby_values) runs at every D.  The composition arm (one
    Row(v == value) and one scratch-row load per value, then fbgpu_groupby) runs only for the unfiltered query at D = 64, for
    --composition-steps steps alternated with the device arm, every one of them reported (no warm-up): it adds D scratch rows to
    the store every step, so each step is slower than the one before (at 512 shards on an H100: about 97 s, 266 s, 387 s).  Both
    arms must return the same groups; every result's total must equal Σ_r Count(Row(a=r) ∩ filter ∩ exists(v)).  Progress goes
    to stderr."""
    from featurebase_b200 import datagen as D, executor as X
    S = args.groupby_shards
    n_cols = 16384
    shards = np.arange(S, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    fa, ff = idx.create_field("a"), idx.create_field("f")
    dvals = (64, 1000, 65535)
    t0 = time.time()
    for fld, rows, p in ((fa, range(256), 1 / 256), (ff, [0], 0.01)):
        bulk = D.fragments(40 + fld.id, shards, list(rows), p)
        h.ctx.load_fragments(idx.id, fld.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
        h.ctx.commit()
        del bulk
    for k, d in enumerate(dvals):
        f = idx.create_field(f"v{d}", "int", min=0, max=d - 1)
        for s in range(S):
            h.ctx.load_fragment(idx.id, f.id, X.VIEW_BSI, s, D.bsi_fragment(50 + k, s, n_cols, f.bit_depth, 0, d - 1))
        h.ctx.commit()
    idx.shards.update(range(S))
    load_s = time.time() - t0
    print(f"config V: loaded {S} shards in {load_s:.1f}s", file=sys.stderr, flush=True)
    real = h.ctx
    from featurebase_b200 import lib as L
    n_rec = S * n_cols
    dev = _KernelMs(real)
    comp = _NoGroupByValues(real)
    for d in dvals:
        for q_filter in (False, True):
            q = f"GroupBy(Rows(a), Rows(v{d})" + (", filter=Row(f=0))" if q_filter else ")")
            exists = [L.Op(L.OP_ROW, idx.fields[f"v{d}"].id, X.VIEW_BSI, 0, 0, 0, 0, 0)]
            if q_filter:
                exists += [L.Op(L.OP_ROW, ff.id, X.VIEW_STANDARD, 0, 0, 0, 0, 0), L.Op(L.OP_INTERSECT, 0, 0, 2, 0, 0, 0, 0)]
            want = int(real.row_counts(idx.id, fa.id, X.VIEW_STANDARD, list(range(S)), row_ids=list(range(256)), filter_ops=exists).sum())
            arms = {"device": dev} if d != 64 or q_filter or args.composition_steps < 1 else {"device": dev, "composition": comp}
            rec = {name: {"wall": [], "kernel_ms": [], "queries": []} for name in arms}
            res = {}
            for i in range(1 + args.steps):                  # one warm-up round of the device arm, then alternate the arms
                for name in (sorted(arms) if i % 2 == 0 else sorted(arms, reverse=True)):
                    if name == "composition" and len(rec[name]["wall"]) >= args.composition_steps:
                        continue
                    h.ctx = arms[name]
                    q0, arms[name].ms = real.counters()["queries"], 0.0
                    t1 = time.perf_counter()
                    r = X.Executor(h).execute("i", q)[0]
                    wall = (time.perf_counter() - t1) * 1e3
                    res.setdefault(name, r)
                    assert r == res[name], (q, name)
                    print(f"config V: {q} {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                    if i >= 1 or name == "composition":
                        rec[name]["wall"].append(wall)
                        rec[name]["kernel_ms"].append(arms[name].ms)
                        rec[name]["queries"].append(real.counters()["queries"] - q0)
            h.ctx = real
            assert all(r == res["device"] for r in res.values()), q
            assert sum(g[1] for g in res["device"]) == want, (q, want)
            for name, dd in rec.items():
                o = {"config": "V", "query": q, "arm": name, "distinct_values": d, "shards": S, "records": n_rec, "groups": len(res[name]),
                     "wall_ms": float(np.median(dd["wall"])), "wall_ms_min": float(np.min(dd["wall"])), "wall_ms_max": float(np.max(dd["wall"])),
                     "kernel_ms": float(np.median(dd["kernel_ms"])), "queries": int(np.median(dd["queries"])), "steps": args.steps, "load_s": round(load_s, 1),
                     "kernel": "eval_kernel + groupby_values_kernel" if name == "device" else "eval_kernel (Row(v == value) per value) + groupby kernels",
                     "note": "median over the timed steps of the executor call (wall clock, Distinct and Rows pre-passes included) and of the summed last_query_gpu_ms of its library queries"}
                if name == "composition":
                    o["wall_ms_per_step"], o["steps"] = [round(x, 2) for x in dd["wall"]], len(dd["wall"])
                out(o)
    real.close()


class _NoTimeViews(_KernelMs):
    """the same proxy without row_counts_views / groupby_views: the executor takes the operand-row composition"""

    def __getattr__(self, name):
        if name in ("row_counts_views", "groupby_views"):
            raise AttributeError(name)
        return super().__getattr__(name)


def _array_fragment(v):
    """Pilosa-roaring bytes of sorted unique values whose containers all hold fewer than 4096 values and are not run-shaped (the
    random sparse bits of config T): every container an array, encoded without a per-container Python loop"""
    keys = v >> np.uint64(16)
    uk, first, cnt = np.unique(keys, return_index=True, return_counts=True)
    hdr = np.zeros(len(uk), dtype=[("key", "<u8"), ("typ", "<u2"), ("n1", "<u2")])
    hdr["key"], hdr["typ"], hdr["n1"] = uk, 1, cnt - 1
    offs = (8 + 16 * len(uk) + 2 * first).astype("<u4")
    return np.array([12348, len(uk)], dtype="<u4").tobytes() + hdr.tobytes() + offs.tobytes() + (v & np.uint64(0xFFFF)).astype("<u2").tobytes()


def _card():
    """the card's name, power limit and maximum SM clock, read in the same run as the numbers they belong to"""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], stdout=subprocess.PIPE,
                           stderr=subprocess.DEVNULL, text=True, timeout=30)
        name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:
        return {"name": None, "error": f"nvidia-smi unavailable: {e}"}


TIME_RANGE = "from=2019-01-05T00:00, to=2019-04-20T00:00"       # configs T and M: 48 views of a quantum-YMD field


def _load_time_field(h, idx, ft, shards, R, per_shard, days):
    """config T's time field: R rows, per_shard bits per shard, each at a random column with a timestamp spread uniformly over
    `days` days from 2019-01-01, in its day, month, year and standard views"""
    import datetime
    from featurebase_b200 import executor as X, roaring_io
    rng = np.random.default_rng(61)
    day0 = datetime.date(2019, 1, 1)
    names = [(day0 + datetime.timedelta(days=d)).strftime("%Y%m%d") for d in range(days)]
    month_of = np.array([int(n[4:6]) for n in names])
    views = {}                                                   # view name -> [per-shard fragment bytes]
    for s in range(len(shards)):
        col = rng.integers(0, SW, per_shard, dtype=np.uint64)
        pos = rng.integers(0, R, per_shard, dtype=np.uint64) * np.uint64(SW) + col
        day = rng.integers(0, days, per_shard)
        every = _array_fragment(np.unique(pos))
        views.setdefault("standard", []).append(every)
        views.setdefault("standard_2019", []).append(every)
        for m in sorted(set(month_of.tolist())):
            views.setdefault("standard_2019%02d" % m, []).append(_array_fragment(np.unique(pos[month_of[day] == m])))
        order = np.argsort(day, kind="stable")
        bounds = np.searchsorted(day[order], np.arange(days + 1))
        for d in range(days):
            views.setdefault("standard_" + names[d], []).append(_array_fragment(np.unique(pos[order[bounds[d]:bounds[d + 1]]])))
        if s == 0:
            assert every == roaring_io.encode(pos)
    for name, blobs in views.items():
        vid = X.VIEW_STANDARD if name == "standard" else ft.view_id(name, create=True)
        offsets = np.concatenate([[0], np.cumsum([len(b) for b in blobs])]).astype(np.uint64)
        h.ctx.load_fragments(idx.id, ft.id, vid, shards, np.frombuffer(b"".join(blobs), dtype=np.uint8), offsets)
    del views


def config_time_views(args, out):
    """TopK(f, from=, to=) and GroupBy(Rows(a), Rows(f, from=, to=)) over a range of 48 views, without and with a 1 % filter row,
    through the executor.  f: a quantum-YMD time field of 256 rows over --groupby-shards shards, 64 Ki bits per shard, each at a
    random column with a timestamp spread uniformly over the 120 days from 2019-01-01 (every bit is in its day, month, year and
    standard views); a: a 256-row set field at 1/256 density per row.  The device arm (fbgpu_row_counts_views /
    fbgpu_groupby_views) runs over all shards.  The composition arm (per row, a Row over the views, read back and stored as a row of
    the scratch field, then one row-count or GroupBy call) re-sends the scratch fragment of every touched shard and commits the
    store again for every row (about two minutes per query on one shard on an H100): it runs over the first --composition-shards
    shards, for
    --composition-steps steps alternated with the device arm over the same shards, every step reported (the scratch field grows
    with each).  Both arms must return the same result.  Progress goes to stderr."""
    from featurebase_b200 import datagen as D, executor as X, lib as L
    S, R, per_shard, days = args.groupby_shards, 256, 1 << 16, 120
    shards = np.arange(S, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    fa, ff, ft = idx.create_field("a"), idx.create_field("c"), idx.create_field("f", "time", quantum="YMD")
    t0 = time.time()
    for fld, rows, p in ((fa, range(R), 1 / 256), (ff, [0], 0.01)):
        bulk = D.fragments(60 + fld.id, shards, list(rows), p)
        h.ctx.load_fragments(idx.id, fld.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
        del bulk
    _load_time_field(h, idx, ft, shards, R, per_shard, days)
    h.ctx.commit()
    idx.shards.update(range(S))
    load_s = time.time() - t0
    rng_q = TIME_RANGE
    n_views = len(X.Executor(h)._time_view_ids(ft, {"from": "2019-01-05T00:00", "to": "2019-04-20T00:00"}))
    print(f"config T: loaded {S} shards in {load_s:.1f}s; the range covers {n_views} views", file=sys.stderr, flush=True)
    real = h.ctx
    card = _card()
    dev, comp = _KernelMs(real), _NoTimeViews(real)
    CS = min(S, args.composition_shards)
    for q in (f"TopK(f, k=10, {rng_q})", f"TopK(f, k=10, {rng_q}, filter=Row(c=0))", f"GroupBy(Rows(a), Rows(f, {rng_q}))",
              f"GroupBy(Rows(a), Rows(f, {rng_q}), filter=Row(c=0))"):
        for n_sh, arms in ((S, {"device": dev}), (CS, {"device": dev, "composition": comp})):
            sh = list(range(n_sh))
            rec = {name: {"wall": [], "kernel_ms": [], "queries": [], "scratch_bytes": []} for name in arms}
            res = {}
            for i in range(1 + args.steps):                  # one warm-up round of the device arm, then alternate the arms
                for name in (sorted(arms) if i % 2 == 0 else sorted(arms, reverse=True)):
                    if name == "composition" and len(rec[name]["wall"]) >= args.composition_steps:
                        continue
                    h.ctx = arms[name]
                    q0, arms[name].ms, b0 = real.counters()["queries"], 0.0, real.stats()["payload_bytes"]
                    t1 = time.perf_counter()
                    r = X.Executor(h).execute("i", q, sh)[0]
                    wall = (time.perf_counter() - t1) * 1e3
                    res.setdefault(name, r)
                    assert r == res[name], (q, name)
                    print(f"config T: {q} over {n_sh} shards, {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                    if i >= 1 or name == "composition":
                        rec[name]["wall"].append(wall)
                        rec[name]["kernel_ms"].append(arms[name].ms)
                        rec[name]["queries"].append(real.counters()["queries"] - q0)
                        rec[name]["scratch_bytes"].append(real.stats()["payload_bytes"] - b0)
            h.ctx = real
            assert all(r == res["device"] for r in res.values()), q
            assert res["device"], q
            for name, dd in rec.items():
                o = {"config": "T", "query": q, "arm": name, "gpu": card, "shards": n_sh, "views": n_views, "rows": R, "results": len(res[name]),
                     "wall_ms": float(np.median(dd["wall"])), "wall_ms_min": float(np.min(dd["wall"])), "wall_ms_max": float(np.max(dd["wall"])),
                     "kernel_ms": float(np.median(dd["kernel_ms"])), "queries": int(np.median(dd["queries"])),
                     "scratch_bytes": int(np.median(dd["scratch_bytes"])), "steps": len(dd["wall"]), "load_s": round(load_s, 1),
                     "kernel": "row_count_views_kernel (+ eval_kernel for filters and peeled GroupBy dimensions)" if name == "device"
                               else "eval_kernel + canonical emission per row, row_count_kernel / groupby kernels over the scratch rows",
                     "note": "median over the timed steps of the executor call (wall clock, Rows pre-passes included), of the summed "
                             "last_query_gpu_ms and of the number of its library queries; scratch_bytes: growth of the store's payload bytes"}
                if name == "composition":
                    o["wall_ms_per_step"] = [round(x, 2) for x in dd["wall"]]
                out(o)
    real.close()


def config_groupby_mixed(args, out):
    """GroupBy(Rows(a), Rows(v), Rows(w)) and GroupBy(Rows(t, from=, to=), Rows(v)) over --groupby-shards shards, without and with
    a 1 % filter row, through the executor.  v and w: int fields holding one of D values (uniform) for each of the first 16,384
    columns of every shard, D x D in {8 x 8, 64 x 64, 256 x 256} (256 x 256 groups exceed one call's 65,535 and take two
    calls); a: a 256-row set field at 1/256 density per row; t: config T's quantum-YMD field (256 rows) over config T's range of
    48 views.  The device arm (fbgpu_groupby_mixed) runs over all shards at every D.  The composition arm (one Row per value and
    per time row, each read back and stored as a row of the scratch field, then fbgpu_groupby) runs over the first
    --composition-shards shards at D = 8 without the filter, for --composition-steps steps alternated with the device arm over
    the same shards: it stores D + D (or 256 time rows + D) scratch rows per step and is slower at every step.  Both arms must
    return the same groups; every device result's total must equal Σ_r Count(Row(a=r) or Row(t=r) ∩ filter ∩ exists(v) (∩
    exists(w))).  Progress goes to stderr."""
    from featurebase_b200 import datagen as D, executor as X, lib as L
    S, R, n_cols = args.groupby_shards, 256, 16384
    shards = np.arange(S, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    fa, ff, ft = idx.create_field("a"), idx.create_field("c"), idx.create_field("t", "time", quantum="YMD")
    dvals = (8, 64, 256)
    t0 = time.time()
    for fld, rows, p in ((fa, range(R), 1 / 256), (ff, [0], 0.01)):
        bulk = D.fragments(70 + fld.id, shards, list(rows), p)
        h.ctx.load_fragments(idx.id, fld.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
        del bulk
    _load_time_field(h, idx, ft, shards, R, 1 << 16, 120)
    for k, d in enumerate(dvals):
        for name in ("v", "w"):
            f = idx.create_field(f"{name}{d}", "int", min=0, max=d - 1)
            for s in range(S):
                h.ctx.load_fragment(idx.id, f.id, X.VIEW_BSI, s, D.bsi_fragment(80 + 2 * k + (name == "w"), s, n_cols, f.bit_depth, 0, d - 1))
    h.ctx.commit()
    idx.shards.update(range(S))
    load_s = time.time() - t0
    tviews = X.Executor(h)._time_view_ids(ft, {"from": "2019-01-05T00:00", "to": "2019-04-20T00:00"})
    print(f"config M: loaded {S} shards in {load_s:.1f}s", file=sys.stderr, flush=True)
    real = h.ctx
    card = _card()
    dev, comp = _KernelMs(real), _NoGroupByValues(real)
    CS = min(S, args.composition_shards)
    op = lambda code, field=0, view=0, argc=0: L.Op(code, field, view, argc, 0, 0, 0, 0)
    for d in dvals:
        v, w = idx.fields[f"v{d}"], idx.fields[f"w{d}"]
        for q_time in (False, True):
            for q_filter in (False, True):
                q = (f"GroupBy(Rows(t, {TIME_RANGE}), Rows(v{d})" if q_time else f"GroupBy(Rows(a), Rows(v{d}), Rows(w{d})") + (", filter=Row(c=0))" if q_filter else ")")
                exists = [op(L.OP_ROW, v.id, X.VIEW_BSI)] + ([] if q_time else [op(L.OP_ROW, w.id, X.VIEW_BSI), op(L.OP_INTERSECT, argc=2)])
                if q_filter:
                    exists += [op(L.OP_ROW, ff.id), op(L.OP_INTERSECT, argc=2)]
                runs = [(S, {"device": dev})]
                if d == dvals[0] and not q_filter and args.composition_steps > 0:
                    runs.append((CS, {"device": dev, "composition": comp}))
                for n_sh, arms in runs:
                    sh = list(range(n_sh))
                    if q_time:
                        want = int(real.row_counts_views(idx.id, ft.id, tviews, sh, row_ids=list(range(R)), filter_ops=exists).sum())
                    else:
                        want = int(real.row_counts(idx.id, fa.id, X.VIEW_STANDARD, sh, row_ids=list(range(R)), filter_ops=exists).sum())
                    rec = {name: {"wall": [], "kernel_ms": [], "queries": []} for name in arms}
                    res = {}
                    for i in range(1 + args.steps):          # one warm-up round of the device arm, then alternate the arms
                        for name in (sorted(arms) if i % 2 == 0 else sorted(arms, reverse=True)):
                            if name == "composition" and len(rec[name]["wall"]) >= args.composition_steps:
                                continue
                            h.ctx = arms[name]
                            q0, arms[name].ms = real.counters()["queries"], 0.0
                            t1 = time.perf_counter()
                            r = X.Executor(h).execute("i", q, sh)[0]
                            wall = (time.perf_counter() - t1) * 1e3
                            res.setdefault(name, r)
                            assert r == res[name], (q, name)
                            print(f"config M: {q} over {n_sh} shards, {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                            if i >= 1 or name == "composition":
                                rec[name]["wall"].append(wall)
                                rec[name]["kernel_ms"].append(arms[name].ms)
                                rec[name]["queries"].append(real.counters()["queries"] - q0)
                    h.ctx = real
                    assert all(r == res["device"] for r in res.values()), q
                    assert sum(g[1] for g in res["device"]) == want > 0, (q, want)
                    for name, dd in rec.items():
                        o = {"config": "M", "query": q, "arm": name, "gpu": card, "distinct_values": [d] if q_time else [d, d], "shards": n_sh,
                             "groups": len(res[name]), "equal_to_composition": ("composition" in res) or None,
                             "wall_ms": float(np.median(dd["wall"])), "wall_ms_min": float(np.min(dd["wall"])), "wall_ms_max": float(np.max(dd["wall"])),
                             "kernel_ms": float(np.median(dd["kernel_ms"])), "queries": int(np.median(dd["queries"])), "steps": len(dd["wall"]), "load_s": round(load_s, 1),
                             "kernel": "eval_kernel + groupby_values_kernel" if name == "device" else "eval_kernel (a Row per value / time row) + groupby kernels",
                             "note": "median over the timed steps of the executor call (wall clock, Distinct and Rows pre-passes included), of the summed "
                                     "last_query_gpu_ms and of the number of its library queries"}
                        if name == "composition":
                            o["wall_ms_per_step"] = [round(x, 2) for x in dd["wall"]]
                        out(o)
    real.close()


class _NoGroupBySum(_KernelMs):
    """the same proxy without groupby_sum: the executor counts the groups on the device, then runs one Sum per non-empty group"""

    def __getattr__(self, name):
        if name == "groupby_sum":
            raise AttributeError(name)
        return super().__getattr__(name)


class _NoGroupByDistinct(_KernelMs):
    """the same proxy without groupby_distinct: the executor counts the groups on the device, then runs one Distinct per group"""

    def __getattr__(self, name):
        if name == "groupby_distinct":
            raise AttributeError(name)
        return super().__getattr__(name)


class _NoGroupByDistinctRows(_KernelMs):
    """the same proxy without groupby_distinct_rows: the executor runs one Distinct per group for a set-like x"""

    def __getattr__(self, name):
        if name == "groupby_distinct_rows":
            raise AttributeError(name)
        return super().__getattr__(name)


def _config_s_world(args, tag):
    """config S's data over --groupby-shards shards: a and b are 256-row set fields at 1/256 density per row, c a 1 % filter row;
    w (64 distinct values) and v (values in ±2^20, 21 bits) are int fields holding a value for each of the first 16,384 columns
    of every shard.  Returns (holder, index, fields a, b, c, w, v, load seconds)."""
    from featurebase_b200 import datagen as D, executor as X
    S, R, n_cols, dw = args.groupby_shards, 256, 16384, 64
    shards = np.arange(S, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    fa, fb, ff = idx.create_field("a"), idx.create_field("b"), idx.create_field("c")
    fw = idx.create_field("w", "int", min=0, max=dw - 1)
    fv = idx.create_field("v", "int", min=-(1 << 20), max=1 << 20)
    t0 = time.time()
    for fld, rows, p in ((fa, range(R), 1 / 256), (fb, range(R), 1 / 256), (ff, [0], 0.01)):
        bulk = D.fragments(90 + fld.id, shards, list(rows), p)
        h.ctx.load_fragments(idx.id, fld.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
        del bulk
    for s in range(S):
        h.ctx.load_fragment(idx.id, fw.id, X.VIEW_BSI, s, D.bsi_fragment(95, s, n_cols, fw.bit_depth, 0, dw - 1))
        h.ctx.load_fragment(idx.id, fv.id, X.VIEW_BSI, s, D.bsi_fragment(96, s, n_cols, fv.bit_depth, -(1 << 20), 1 << 20))
    h.ctx.commit()
    idx.shards.update(range(S))
    load_s = time.time() - t0
    print(f"config {tag}: loaded {S} shards in {load_s:.1f}s", file=sys.stderr, flush=True)
    return h, idx, fa, fb, ff, fw, fv, load_s


def config_groupby_sum(args, out):
    """GroupBy(Rows(a), aggregate=Sum(field=v)), GroupBy(Rows(a), Rows(b), aggregate=Sum(field=v)) and GroupBy(Rows(a), Rows(w),
    aggregate=Sum(field=v)) over --groupby-shards shards (_config_s_world), without and with a 1 % filter row, through the
    executor.  The device arm (one fbgpu_groupby_sum) runs over all shards.  The composition arm (the group counts on the device,
    then one Sum(Intersect(rows, filter)) library query per non-empty group) runs over the first --composition-shards shards, for
    --composition-steps steps alternated with the device arm over the same shards.  Both arms must return the same groups; every
    device result's total count must equal Σ_r Count(Row(a=r) ∩ filter ∩ exists(v) (∩ exists(w))).  Progress goes to stderr."""
    from featurebase_b200 import executor as X, lib as L
    S, R = args.groupby_shards, 256
    h, idx, fa, fb, ff, fw, fv, load_s = _config_s_world(args, "S")
    real = h.ctx
    card = _card()
    dev, comp = _KernelMs(real), _NoGroupBySum(real)
    CS = min(S, args.composition_shards)
    op = lambda code, field=0, view=0, argc=0: L.Op(code, field, view, argc, 0, 0, 0, 0)
    for second in ("", "Rows(b), ", "Rows(w), "):
        for q_filter in (False, True):
            q = f"GroupBy(Rows(a), {second}aggregate=Sum(field=v)" + (", filter=Row(c=0))" if q_filter else ")")
            exists = [op(L.OP_ROW, fv.id, X.VIEW_BSI)] + ([op(L.OP_ROW, fw.id, X.VIEW_BSI), op(L.OP_INTERSECT, argc=2)] if "w" in second else [])
            if q_filter:
                exists += [op(L.OP_ROW, ff.id), op(L.OP_INTERSECT, argc=2)]
            runs = [(S, {"device": dev})] + ([(CS, {"device": dev, "composition": comp})] if args.composition_steps > 0 else [])
            for n_sh, arms in runs:
                sh = list(range(n_sh))
                want = int(real.row_counts(idx.id, fa.id, X.VIEW_STANDARD, sh, row_ids=list(range(R)), filter_ops=exists).sum())
                rec = {name: {"wall": [], "kernel_ms": [], "queries": []} for name in arms}
                res = {}
                for i in range(1 + args.steps):              # one warm-up round of the device arm, then alternate the arms
                    for name in (sorted(arms) if i % 2 == 0 else sorted(arms, reverse=True)):
                        if name == "composition" and len(rec[name]["wall"]) >= args.composition_steps:
                            continue
                        h.ctx = arms[name]
                        q0, arms[name].ms = real.counters()["queries"], 0.0
                        t1 = time.perf_counter()
                        r = X.Executor(h).execute("i", q, sh)[0]
                        wall = (time.perf_counter() - t1) * 1e3
                        res.setdefault(name, r)
                        assert r == res[name], (q, name)
                        print(f"config S: {q} over {n_sh} shards, {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                        if i >= 1 or name == "composition":
                            rec[name]["wall"].append(wall)
                            rec[name]["kernel_ms"].append(arms[name].ms)
                            rec[name]["queries"].append(real.counters()["queries"] - q0)
                h.ctx = real
                assert all(r == res["device"] for r in res.values()), q
                if "b" not in second:                           # a column is in one b-row or several: only a and w partition the columns
                    assert sum(g[1] for g in res["device"]) == want > 0, (q, want)
                for name, dd in rec.items():
                    o = {"config": "S", "query": q, "arm": name, "gpu": card, "shards": n_sh, "groups": len(res[name]),
                         "equal_to_composition": ("composition" in res) or None,
                         "wall_ms": float(np.median(dd["wall"])), "wall_ms_min": float(np.min(dd["wall"])), "wall_ms_max": float(np.max(dd["wall"])),
                         "kernel_ms": float(np.median(dd["kernel_ms"])), "queries": int(np.median(dd["queries"])), "steps": len(dd["wall"]), "load_s": round(load_s, 1),
                         "kernel": "eval_kernel + groupby_values_kernel<true>" if name == "device" else "eval_kernel + groupby kernels, then eval_kernel + bsi_sum_kernel per group",
                         "note": "median over the timed steps of the executor call (wall clock, Rows / Distinct pre-passes included), of the summed "
                                 "last_query_gpu_ms and of the number of its library queries"}
                    if name == "composition":
                        o["wall_ms_per_step"] = [round(x, 2) for x in dd["wall"]]
                    out(o)
    real.close()


def config_groupby_distinct(args, out):
    """GroupBy(Rows(a), aggregate=Count(Distinct(field=v))), the same with Rows(w) and then Rows(b) beside a, over config S's data
    (_config_s_world), without and with a 1 % filter row, through the executor.  The device arm (one Distinct for v's values,
    then fbgpu_groupby_distinct, sliced by GROUPBY_DISTINCT_BITS) runs over all shards.  The composition arm (the group counts on
    the device, then one Distinct(Intersect(rows, filter), field=v) library query per group) runs over the first
    --composition-shards shards, for --composition-steps steps alternated with the device arm over the same shards.  Both arms
    must return the same groups, every distinct count lies in 0 .. the group's count, and without b (a and w partition the
    columns) the counts add up to Σ_r Count(Row(a=r) ∩ filter).  Progress goes to stderr."""
    from featurebase_b200 import executor as X, lib as L
    S, R = args.groupby_shards, 256
    h, idx, fa, fb, ff, fw, fv, load_s = _config_s_world(args, "D")
    real = h.ctx
    card = _card()
    dev, comp = _KernelMs(real), _NoGroupByDistinct(real)
    CS = min(S, args.composition_shards)
    op = lambda code, field=0, view=0, argc=0: L.Op(code, field, view, argc, 0, 0, 0, 0)
    for second in ("", "Rows(w), ", "Rows(b), "):
        for q_filter in (False, True):
            q = f"GroupBy(Rows(a), {second}aggregate=Count(Distinct(field=v))" + (", filter=Row(c=0))" if q_filter else ")")
            need = [op(L.OP_ROW, fw.id, X.VIEW_BSI)] if "w" in second else []
            if q_filter:
                need += [op(L.OP_ROW, ff.id)] + ([op(L.OP_INTERSECT, argc=2)] if "w" in second else [])
            runs = [(S, {"device": dev})] + ([(CS, {"device": dev, "composition": comp})] if args.composition_steps > 0 else [])
            for n_sh, arms in runs:
                sh = list(range(n_sh))
                want = int(real.row_counts(idx.id, fa.id, X.VIEW_STANDARD, sh, row_ids=list(range(R)), filter_ops=need or None).sum())
                rec = {name: {"wall": [], "kernel_ms": [], "queries": []} for name in arms}
                res = {}
                for i in range(1 + args.steps):              # one warm-up round of the device arm, then alternate the arms
                    for name in (sorted(arms) if i % 2 == 0 else sorted(arms, reverse=True)):
                        if name == "composition" and len(rec[name]["wall"]) >= args.composition_steps:
                            continue
                        h.ctx = arms[name]
                        q0, arms[name].ms = real.counters()["queries"], 0.0
                        t1 = time.perf_counter()
                        r = X.Executor(h).execute("i", q, sh)[0]
                        wall = (time.perf_counter() - t1) * 1e3
                        res.setdefault(name, r)
                        assert r == res[name], (q, name)
                        print(f"config D: {q} over {n_sh} shards, {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                        if i >= 1 or name == "composition":
                            rec[name]["wall"].append(wall)
                            rec[name]["kernel_ms"].append(arms[name].ms)
                            rec[name]["queries"].append(real.counters()["queries"] - q0)
                h.ctx = real
                assert all(r == res["device"] for r in res.values()), q
                assert all(0 <= g[2] <= g[1] for g in res["device"]) and any(g[2] for g in res["device"]), q
                if "b" not in second:
                    assert sum(g[1] for g in res["device"]) == want > 0, (q, want)
                for name, dd in rec.items():
                    o = {"config": "D", "query": q, "arm": name, "gpu": card, "shards": n_sh, "groups": len(res[name]),
                         "equal_to_composition": ("composition" in res) or None,
                         "wall_ms": float(np.median(dd["wall"])), "wall_ms_min": float(np.min(dd["wall"])), "wall_ms_max": float(np.max(dd["wall"])),
                         "kernel_ms": float(np.median(dd["kernel_ms"])), "queries": int(np.median(dd["queries"])), "steps": len(dd["wall"]), "load_s": round(load_s, 1),
                         "kernel": ("eval_kernel + groupby kernels, extract_values_kernel once, groupby_values_kernel<GvAgg::kDistinct> + gv_popcount_kernel"
                                    if name == "device" else "eval_kernel + groupby kernels, then eval_kernel + extract_values_kernel per group"),
                         "note": "median over the timed steps of the executor call (wall clock, Rows / Distinct pre-passes included), of the summed "
                                 "last_query_gpu_ms and of the number of its library queries"}
                    if name == "composition":
                        o["wall_ms_per_step"] = [round(x, 2) for x in dd["wall"]]
                    out(o)
    real.close()


def config_groupby_distinct_rows(args, out):
    """GroupBy(Rows(a), aggregate=Count(Distinct(field=x))) and the same with Rows(b) beside a, for x = m, a mutex field of
    100,000 rows (one row per record), and x = s, a set field of 64 rows (0-4 rows per record), without and with a 1 % filter
    row, through the executor.  The data is config D's (_config_s_world); m and s cover the first 16,384 columns of every shard,
    the records that hold config D's int values, and every shard holds the same m and s fragments, encoded once.  The device arm
    (one fbgpu_row_counts for x's rows, then fbgpu_groupby_distinct_rows, sliced by GROUPBY_DISTINCT_BITS) runs over all shards.
    The composition arm (the group counts on the device, then one Distinct(Intersect(rows, filter), field=x) library query per
    group) runs over the first --composition-shards shards, for --composition-steps steps alternated with the device arm over the
    same shards, and only for queries of at most --composition-max-groups groups (a's 256; a x b's 65,536 are not timed).  Both
    arms must return the same groups and every distinct count lies in 0 .. the group's count.  Progress goes to stderr."""
    from featurebase_b200 import executor as X, roaring_io
    S, n_cols = args.groupby_shards, 16384
    h, idx, fa, fb, ff, fw, fv, load_s = _config_s_world(args, "K")
    fm, fs = idx.create_field("m", "mutex"), idx.create_field("s")
    rng = np.random.default_rng(2028)
    cols = np.arange(n_cols, dtype=np.uint64)
    s_bits = np.concatenate([rng.choice(64, int(k), replace=False).astype(np.uint64) * np.uint64(SW) + c for c, k in zip(cols, rng.integers(0, 5, n_cols))])
    data = {fm: roaring_io.encode(np.sort(rng.integers(0, 100000, n_cols).astype(np.uint64) * np.uint64(SW) + cols)),
            fs: roaring_io.encode(np.unique(s_bits))}
    t0 = time.time()
    for s in range(S):
        for f, d in data.items():
            h.ctx.load_fragment(idx.id, f.id, X.VIEW_STANDARD, s, d)
    h.ctx.commit()
    load_s += time.time() - t0
    real = h.ctx
    card = _card()
    dev, comp = _KernelMs(real), _NoGroupByDistinctRows(real)
    CS = min(S, args.composition_shards)
    for second, x in (("", "m"), ("Rows(b), ", "m"), ("", "s"), ("Rows(b), ", "s")):
        for q_filter in (False, True):
            q = f"GroupBy(Rows(a), {second}aggregate=Count(Distinct(field={x}))" + (", filter=Row(c=0))" if q_filter else ")")
            groups = 256 * (256 if second else 1)
            runs = [(S, {"device": dev})]
            if args.composition_steps > 0 and groups <= args.composition_max_groups:
                runs.append((CS, {"device": dev, "composition": comp}))
            for n_sh, arms in runs:
                sh = list(range(n_sh))
                rec = {name: {"wall": [], "kernel_ms": [], "queries": []} for name in arms}
                res = {}
                for i in range(1 + args.steps):              # one warm-up round of the device arm, then alternate the arms
                    for name in (sorted(arms) if i % 2 == 0 else sorted(arms, reverse=True)):
                        if name == "composition" and len(rec[name]["wall"]) >= args.composition_steps:
                            continue
                        h.ctx = arms[name]
                        q0, arms[name].ms = real.counters()["queries"], 0.0
                        t1 = time.perf_counter()
                        r = X.Executor(h).execute("i", q, sh)[0]
                        wall = (time.perf_counter() - t1) * 1e3
                        res.setdefault(name, r)
                        assert r == res[name], (q, name)
                        print(f"config K: {q} over {n_sh} shards, {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                        if i >= 1 or name == "composition":
                            rec[name]["wall"].append(wall)
                            rec[name]["kernel_ms"].append(arms[name].ms)
                            rec[name]["queries"].append(real.counters()["queries"] - q0)
                h.ctx = real
                assert all(r == res["device"] for r in res.values()), q
                assert all(0 <= g[2] <= g[1] for g in res["device"]) and any(g[2] for g in res["device"]), q
                for name, dd in rec.items():
                    o = {"config": "K", "query": q, "arm": name, "gpu": card, "shards": n_sh, "groups": len(res[name]),
                         "equal_to_composition": ("composition" in res) or None,
                         "wall_ms": float(np.median(dd["wall"])), "wall_ms_min": float(np.min(dd["wall"])), "wall_ms_max": float(np.max(dd["wall"])),
                         "kernel_ms": float(np.median(dd["kernel_ms"])), "queries": int(np.median(dd["queries"])), "steps": len(dd["wall"]), "load_s": round(load_s, 1),
                         "kernel": ("eval_kernel + groupby kernels, row_count_kernel once, groupby_values_kernel<GvAgg::kDistinctRows> + gv_popcount_kernel"
                                    if name == "device" else "eval_kernel + groupby kernels, then eval_kernel + row_count_kernel per group"),
                         "note": "median over the timed steps of the executor call (wall clock, Rows / Distinct pre-passes included), of the summed "
                                 "last_query_gpu_ms and of the number of its library queries"}
                    if name == "composition":
                        o["wall_ms_per_step"] = [round(x, 2) for x in dd["wall"]]
                    out(o)
    real.close()


def _config_g_world(args, tag, m_fragments=1):
    """config G's data: _config_s_world plus m, a mutex field of 1,000,000 rows holding one row for each of the first 16,384
    columns of every shard (shard s takes the (s % m_fragments)-th of m_fragments fragments, each encoded once; config G's one
    fragment gives about 16,000 distinct rows, eight give more than 65,535), and e, whose row 0 holds those columns.  Returns
    (holder, index, fields a, b, c, w, v, m, e, load seconds)."""
    from featurebase_b200 import executor as X, roaring_io
    n_cols = 16384
    h, idx, fa, fb, ff, fw, fv, load_s = _config_s_world(args, tag)
    fm, fe = idx.create_field("m", "mutex"), idx.create_field("e")
    rng = np.random.default_rng(2029)
    data = [roaring_io.encode(np.sort(rng.integers(0, 1_000_000, n_cols).astype(np.uint64) * np.uint64(SW) + np.arange(n_cols, dtype=np.uint64)))
            for _ in range(m_fragments)]
    every = roaring_io.encode(np.arange(n_cols, dtype=np.uint64))          # e=0: the columns m covers
    t0 = time.time()
    for s_ in range(args.groupby_shards):
        h.ctx.load_fragment(idx.id, fm.id, X.VIEW_STANDARD, s_, data[s_ % m_fragments])
        h.ctx.load_fragment(idx.id, fe.id, X.VIEW_STANDARD, s_, every)
    h.ctx.commit()
    return h, idx, fa, fb, ff, fw, fv, fm, fe, load_s + time.time() - t0


def config_groupby_sparse(args, out):
    """fbgpu_groupby_sparse over --groupby-shards shards of config S's data (_config_s_world) plus m, a mutex field of 1,000,000
    rows holding one row for each of the first 16,384 columns of every shard (every shard the same fragment, encoded once), as
    library calls (no executor):
      (a) a x b, 256 x 256: the sparse call against fbgpu_groupby (the dense tensor), alternated; the same groups and counts;
      (b) m x a: the sparse call against the host composition, one fbgpu_extract_rows per dimension over Row(e=0) (a row
          holding the columns m covers) and a numpy join of the per-column row lists, alternated; the same groups and counts;
      (c) m x a paged: limit=1000 pages, each starting one past the last cell of the page before, for 8 pages.
    Wall clock per call (each ends in a device synchronise and a copy to the host), with the call's last_query_gpu_ms."""
    from featurebase_b200 import executor as X, lib as L
    S = args.groupby_shards
    h, idx, fa, fb, ff, fw, fv, fm, fe, load_s = _config_g_world(args, "G")
    ctx, card, sh = h.ctx, _card(), list(range(S))
    ra, rm = np.arange(256, dtype=np.uint64), np.arange(1_000_000, dtype=np.uint64)
    dims_ab = [(fa.id, [X.VIEW_STANDARD], ra), (fb.id, [X.VIEW_STANDARD], ra)]
    dims_ma = [(fm.id, [X.VIEW_STANDARD], rm), (fa.id, [X.VIEW_STANDARD], ra)]
    m_cols = [L.Op(L.OP_ROW, fe.id, X.VIEW_STANDARD, 0, 0, 0, 0, 0)]

    def composition():
        cm, om, rows_m, _ = ctx.extract_rows(idx.id, fm.id, X.VIEW_STANDARD, sh, m_cols)
        ca, oa, rows_a, _ = ctx.extract_rows(idx.id, fa.id, X.VIEW_STANDARD, sh, m_cols)
        nm, na = np.diff(om.astype(np.int64)), np.diff(oa.astype(np.int64))
        rep = nm * na                                          # the cells of each column: its m rows x its a rows
        col = np.repeat(np.arange(len(cm)), rep)
        k = np.arange(len(col)) - np.repeat(np.cumsum(rep) - rep, rep)
        im = om[:-1].astype(np.int64)[col] + k // na[col]
        ia = oa[:-1].astype(np.int64)[col] + k % na[col]
        cells, counts = np.unique(np.searchsorted(rm, rows_m[im]).astype(np.uint64) * np.uint64(256) + np.searchsorted(ra, rows_a[ia]).astype(np.uint64),
                                  return_counts=True)
        return cells, counts.astype(np.uint64)

    def paged():
        start, got = 0, 0
        for _ in range(8):
            c, n = ctx.groupby_sparse(idx.id, dims_ma, sh, start=start, limit=1000)
            if len(c) == 0:
                break
            got += len(c)
            start = int(c[-1]) + 1
        return got

    arms = {"a": {"sparse": lambda: ctx.groupby_sparse(idx.id, dims_ab, sh), "dense": lambda: ctx.groupby(idx.id, [fa.id, fb.id], [0, 0], [ra, ra], sh)},
            "b": {"sparse": lambda: ctx.groupby_sparse(idx.id, dims_ma, sh), "composition": composition},
            "c": {"sparse_paged": paged}}
    for part, fns in arms.items():
        rec = {name: {"wall": [], "gpu_ms": [], "queries": []} for name in fns}
        res = {}
        for i in range(1 + args.steps):                          # one warm-up round, then alternate the arms
            for name in (sorted(fns) if i % 2 == 0 else sorted(fns, reverse=True)):
                q0 = ctx.counters()["queries"]
                t1 = time.perf_counter()
                r = fns[name]()
                wall = (time.perf_counter() - t1) * 1e3
                if name == "dense":                              # the dense tensor's non-zero cells, for the comparison
                    flat = r.reshape(-1)
                    nz = np.flatnonzero(flat)
                    r = (nz.astype(np.uint64), flat[nz])
                res.setdefault(name, r)
                print(f"config G ({part}): {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                if i >= 1:
                    rec[name]["wall"].append(wall)
                    rec[name]["gpu_ms"].append(ctx.counters()["last_query_gpu_ms"])
                    rec[name]["queries"].append(ctx.counters()["queries"] - q0)
        vals = list(res.values())
        if part != "c":
            assert all(np.array_equal(v[0], vals[0][0]) and np.array_equal(v[1], vals[0][1]) for v in vals), part
        for name, dd in rec.items():
            r = res[name]
            out({"config": "G", "part": part, "arm": name, "gpu": card, "shards": S, "groups": int(r if part == "c" else len(r[0])),
                 "wall_ms": float(np.median(dd["wall"])), "wall_ms_min": float(np.min(dd["wall"])), "wall_ms_max": float(np.max(dd["wall"])),
                 "last_query_gpu_ms": float(np.median(dd["gpu_ms"])), "queries": int(np.median(dd["queries"])), "steps": len(dd["wall"]),
                 "load_s": round(load_s, 1),
                 "note": "median over the timed steps of the call's wall clock, of the last library query's GPU ms and of the library queries"})
    ctx.close()


def config_groupby_sparse_sum(args, out):
    """aggregate=Sum(field=v) over config G's data (_config_g_world with eight m fragments, so that Rows(m) lists more than
    65,535 rows and the executor takes the sparse path; v holds a value on every column m covers), over --groupby-shards shards:
      (a) GroupBy(Rows(m), aggregate=Sum(field=v), limit=1000) through the executor: fbgpu_groupby_sparse_sum against today's
          composition without it (the sparse list of groups, then one Sum query per group until 1,000 are listed), alternated;
          the same groups, counts and sums;
      (b) GroupBy(Rows(m), Rows(a), aggregate=Sum(field=v)), every group, as library calls: fbgpu_groupby_sparse_sum against the
          counts-only fbgpu_groupby_sparse on the same dimensions, alternated; the same cells and counts (every column of m holds
          a value of v), so the difference is the cost of carrying the aggregate;
      (c) a x b, 256 x 256, with Sum, as library calls: fbgpu_groupby_sparse_sum against the dense fbgpu_groupby_sum, alternated;
          the same cells, counts and sums.
    Per arm: the median wall clock, the summed last_query_gpu_ms of the arm's library queries and their number."""
    from featurebase_b200 import executor as X
    S = args.groupby_shards
    h, idx, fa, fb, ff, fw, fv, fm, fe, load_s = _config_g_world(args, "H", m_fragments=8)
    real, card, sh = h.ctx, _card(), list(range(S))
    dev, comp = _KernelMs(real), _NoGroupBySum(real)
    ra, rm = np.arange(256, dtype=np.uint64), np.arange(1_000_000, dtype=np.uint64)
    agg = (fv.id, X.VIEW_BSI, fv.bit_depth)
    dims_ab = [(fa.id, [X.VIEW_STANDARD], ra), (fb.id, [X.VIEW_STANDARD], ra)]
    dims_ma = [(fm.id, [X.VIEW_STANDARD], rm), (fa.id, [X.VIEW_STANDARD], ra)]
    q = "GroupBy(Rows(m), aggregate=Sum(field=v), limit=1000)"

    def executor(ctx):
        def run():
            h.ctx = ctx
            try:
                return X.Executor(h).execute("i", q, sh)[0]
            finally:
                h.ctx = real
        return run

    def dense_sum():
        counts, sums = dev.groupby_sum(idx.id, dims_ab, [], agg, sh)
        counts, sums = counts.reshape(-1), sums.reshape(-1)
        nz = np.flatnonzero(counts)
        return nz.astype(np.uint64), counts[nz], sums[nz]

    arms = {"a": {"device": (dev, executor(dev)), "composition": (comp, executor(comp))},
            "b": {"sparse_sum": (dev, lambda: dev.groupby_sparse(idx.id, dims_ma, sh, agg=agg)),
                  "sparse_counts": (dev, lambda: dev.groupby_sparse(idx.id, dims_ma, sh))},
            "c": {"sparse_sum": (dev, lambda: dev.groupby_sparse(idx.id, dims_ab, sh, agg=agg)), "dense_sum": (dev, dense_sum)}}
    for part, fns in arms.items():
        rec = {name: {"wall": [], "gpu_ms": [], "queries": []} for name in fns}
        res = {}
        for i in range(1 + args.steps):                          # one warm-up round, then alternate the arms
            for name in (sorted(fns) if i % 2 == 0 else sorted(fns, reverse=True)):
                proxy, fn = fns[name]
                q0, proxy.ms = real.counters()["queries"], 0.0
                t1 = time.perf_counter()
                r = fn()
                wall = (time.perf_counter() - t1) * 1e3
                res.setdefault(name, r)
                print(f"config H ({part}): {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                if i >= 1:
                    rec[name]["wall"].append(wall)
                    rec[name]["gpu_ms"].append(proxy.ms)
                    rec[name]["queries"].append(real.counters()["queries"] - q0)
        v = list(res.values())
        if part == "a":
            assert v[0] == v[1] and len(v[0]) == 1000, part
        else:
            n_cmp = 2 if part == "b" else 3                      # (b): the counts-only call has no sums
            assert all(np.array_equal(x[k], v[0][k]) for x in v for k in range(n_cmp)), part
        for name, dd in rec.items():
            out({"config": "H", "part": part, "arm": name, "gpu": card, "shards": S, "groups": len(res[name] if part == "a" else res[name][0]),
                 "equal_to_other_arm": True, "wall_ms": float(np.median(dd["wall"])), "wall_ms_min": float(np.min(dd["wall"])),
                 "wall_ms_max": float(np.max(dd["wall"])), "gpu_ms": float(np.median(dd["gpu_ms"])), "queries": int(np.median(dd["queries"])),
                 "steps": len(dd["wall"]), "load_s": round(load_s, 1),
                 "note": "median over the timed steps of the wall clock (executor: Rows pre-pass included), of the summed last_query_gpu_ms "
                         "of the arm's library queries and of their number"})
    real.close()


class _NoTopnCutoffs(_KernelMs):
    """the same proxy without topn_cutoffs: the executor fetches per-shard count matrices and applies the cut-offs on the host"""

    def __getattr__(self, name):
        if name == "topn_cutoffs":
            raise AttributeError(name)
        return super().__getattr__(name)


def config_topn_cutoffs(args, out):
    """TopN(f, Row(src=0), tanimotoThreshold=50) and TopN(f, Row(src=0), threshold=100) through the executor.  f is a set field of
    --topn-rows rows in each of --topn-shards shards; Src (row 0 of src) holds 400 random columns of slot 0 per shard.  Half of
    f's rows take each of Src's columns with a probability drawn per row from 0.5..1 plus up to 40 other columns, so their
    Tanimoto coefficient straddles 50; the other half hold 1..300 random columns.  The device arm (fbgpu_topn_cutoffs) runs over
    all shards; the composition arm (fbgpu_count per shard, two fbgpu_row_counts_per_shard matrices, the cut-offs in a Python
    loop over (shard, row)) over the first --composition-shards shards, for --composition-steps steps alternated with the device
    arm over the same shards.  Both arms must return the same pairs, and between 5 % and 95 % of the rows must survive each
    cut-off, so that neither rule is trivially all-pass or all-fail.  Progress goes to stderr."""
    from featurebase_b200 import executor as X, roaring_io
    S, R, n_src = args.topn_shards, args.topn_rows, 400
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    idx.create_field("f")
    idx.create_field("src")
    t0 = time.perf_counter()
    rng = np.random.default_rng(2026)
    for s in range(S):
        src = np.sort(rng.choice(1 << 16, n_src, replace=False)).astype(np.uint64)
        h.import_roaring("i", "src", X.VIEW_STANDARD, s, roaring_io.encode(src))
        half = R // 2
        take = rng.random((half, n_src)) < rng.uniform(0.5, 1.0, size=(half, 1))
        rr, cc = np.nonzero(take)
        n_extra = rng.integers(0, 41, size=half)
        er = np.repeat(np.arange(half), n_extra)
        n_rand = rng.integers(1, 301, size=R - half)
        qr = half + np.repeat(np.arange(R - half), n_rand)
        rows = np.concatenate([rr, er, qr]).astype(np.uint64)
        cols = np.concatenate([src[cc], rng.integers(0, 1 << 16, size=len(er) + len(qr)).astype(np.uint64)])
        h.import_roaring("i", "f", X.VIEW_STANDARD, s, roaring_io.encode(rows * np.uint64(SW) + cols))
        print(f"config N: shard {s} loaded, {time.perf_counter() - t0:.1f} s", file=sys.stderr, flush=True)
    h.ctx.commit()
    load_s = time.perf_counter() - t0
    real = h.ctx
    card = _card()
    dev, comp = _KernelMs(real), _NoTopnCutoffs(real)
    CS = min(S, args.composition_shards)
    for q in ("TopN(f, Row(src=0), tanimotoThreshold=50)", "TopN(f, Row(src=0), threshold=100)"):
        runs = [(S, {"device": dev})] + ([(CS, {"device": dev, "composition": comp})] if args.composition_steps > 0 else [])
        for n_sh, arms in runs:
            sh = list(range(n_sh))
            rec = {name: {"wall": [], "kernel_ms": [], "queries": []} for name in arms}
            res = {}
            for i in range(1 + args.steps):                  # one warm-up round of the device arm, then alternate the arms
                for name in (sorted(arms) if i % 2 == 0 else sorted(arms, reverse=True)):
                    if name == "composition" and len(rec[name]["wall"]) >= args.composition_steps:
                        continue
                    h.ctx = arms[name]
                    q0, arms[name].ms = real.counters()["queries"], 0.0
                    t1 = time.perf_counter()
                    r = X.Executor(h).execute("i", q, sh)[0]
                    wall = (time.perf_counter() - t1) * 1e3
                    res.setdefault(name, r)
                    assert r == res[name], (q, name)
                    print(f"config N: {q} over {n_sh} shards, {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                    if i >= 1 or name == "composition":
                        rec[name]["wall"].append(wall)
                        rec[name]["kernel_ms"].append(arms[name].ms)
                        rec[name]["queries"].append(real.counters()["queries"] - q0)
            h.ctx = real
            assert all(r == res["device"] for r in res.values()), q
            assert 0.05 * R < len(res["device"]) < 0.95 * R, (q, len(res["device"]), R)
            for name, dd in rec.items():
                o = {"config": "N", "query": q, "arm": name, "gpu": card, "shards": n_sh, "rows": R, "pairs": len(res[name]),
                     "equal_to_composition": ("composition" in res) or None,
                     "wall_ms": float(np.median(dd["wall"])), "wall_ms_min": float(np.min(dd["wall"])), "wall_ms_max": float(np.max(dd["wall"])),
                     "kernel_ms": float(np.median(dd["kernel_ms"])), "queries": int(np.median(dd["queries"])), "steps": len(dd["wall"]), "load_s": round(load_s, 1),
                     "kernel": ("eval_kernel + row_count_kernel<RcOut::kCutoff>" if name == "device"
                                else "row_count_kernel (candidates), eval_kernel (Src counts), row_count_kernel<RcOut::kPerShard> x 2, host loop"),
                     "note": "median over the timed steps of the executor call (wall clock), of the summed last_query_gpu_ms and of the "
                             "number of its library queries"}
                if name == "composition":
                    o["wall_ms_per_step"] = [round(x, 2) for x in dd["wall"]]
                out(o)
    real.close()


def config3(args, out, n_rec=10_000_000, nf=4):
    """nf fields are rotated between steps so that the touched planes exceed L2 (the 10 M-record config is 42.5 MB)"""
    from featurebase_b200 import datagen as D, executor as X, pql
    from oracle import oracle as O
    from tests.oracle_exec import OracleIndex
    pk, src = peak()
    n_sh = (n_rec + SW - 1) // SW
    shards = np.arange(n_sh, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    ex = X.Executor(h)
    ora = OracleIndex(idx)
    for k in range(nf):
        fld = idx.create_field(f"v{k}", "int", min=0, max=(1 << 32) - 1)
        for s in range(n_sh):
            ncols = min(SW, n_rec - s * SW)
            data = D.bsi_fragment(20 + k, s, ncols, 32, 0, (1 << 32) - 1)
            h.import_roaring("i", f"v{k}", X.VIEW_BSI, s, data)
            if k == 0 and s in (0, n_sh - 1):
                ora.load("v0", X.VIEW_BSI, s, data)
    h.ctx.commit()
    for kname, kval in (("2^31", 1 << 31), ("0.99*2^32", int(0.99 * (1 << 32)))):
        progs = [ex._bitmap_call(idx, pql.parse(f"Row(v{k} > {kval})")[0]) for k in range(nf)]
        res = {}

        def step(i):
            res[i % nf] = h.ctx.count(idx.id, progs[i % nf], shards)

        ms, ms_min, wall = timed(h.ctx, step, args.steps)
        # planes the compiled program touches: exists, sign, and every bit row down to where the predicate saturates
        pay, nc = h.ctx.rows_payload_bytes(idx.id, idx.fields["v0"].id, X.VIEW_BSI, shards, None)
        algo = pay + 16 * nc + 8
        call = pql.parse(f"Row(v0 > {kval})")[0]
        exp = sum(ora.eval_shard(call, s).count() for s in (0, n_sh - 1))
        tot, per = h.ctx.count(idx.id, progs[0], shards, per_shard=True)
        assert int(per[0]) + int(per[n_sh - 1]) == exp
        gbs = algo / (ms * 1e-3) / 1e9
        out({"config": 3, "query": f"Count(Row(v > {kname}))", "records": n_rec, "shards": n_sh, "kernel": "eval_kernel (BSI plane sweep)", "ms": ms, "ms_min": ms_min, "wall_ms": wall,
             "records_per_sec": n_rec / (ms * 1e-3), "algorithmic_bytes": int(algo), "achieved_gbs": gbs, "peak_gbs": pk, "peak_source": src, "frac": gbs / pk,
             "note": f"algorithmic bytes = all 34 planes of the field (upper bound; the sweep stops early when the predicate saturates); {nf} field(s) rotated",
             "count": int(tot), "selectivity": tot / n_rec})
    h.ctx.close()


def config4(args, out):
    from featurebase_b200 import datagen as D, executor as X
    from oracle import oracle as O
    pk, src = peak()
    S = args.groupby_shards
    p_rec = 100e6 / (4096 * SW)
    shards = np.arange(S, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    fa, fb = idx.create_field("a"), idx.create_field("b")
    keep = {}
    t0 = time.time()
    for s in range(S):
        da, db = D.groupby_fragments(31, 32, s, p_rec, 256, 256)
        h.import_roaring("i", "a", X.VIEW_STANDARD, s, da)
        h.import_roaring("i", "b", X.VIEW_STANDARD, s, db)
        if s in (0, S - 1):
            keep[s] = (da, db)
    h.ctx.commit()
    rows = list(range(256))
    res = {}

    def step(i):
        res[0] = h.ctx.groupby(idx.id, [fa.id, fb.id], [0, 0], [rows, rows], shards)

    ms, ms_min, wall = timed(h.ctx, step, args.steps)
    pa, na = h.ctx.rows_payload_bytes(idx.id, fa.id, 0, shards, None)
    pb, nb = h.ctx.rows_payload_bytes(idx.id, fb.id, 0, shards, None)
    algo = pa + pb + 16 * (na + nb) + 8 * 65536
    # oracle spot check on two shards
    sub = h.ctx.groupby(idx.id, [fa.id, fb.id], [0, 0], [rows, rows], np.array(sorted(keep), dtype=np.uint64))
    exp = np.zeros(65536, dtype=np.uint64)
    for s, (da, db) in keep.items():
        O.groupby_shard([O.Bitmap.from_bytes(da), O.Bitmap.from_bytes(db)], s, [rows, rows], None, exp)
    assert np.array_equal(sub.reshape(-1), exp)
    total = int(res[0].sum())
    gbs = algo / (ms * 1e-3) / 1e9
    out({"config": 4, "query": "GroupBy(Rows(a), Rows(b)) 256x256", "shards": S, "records": total, "kernel": "groupby_direct_kernel", "ms": ms, "ms_min": ms_min, "wall_ms": wall,
         "records_per_sec": total / (ms * 1e-3), "group_counts_per_sec": 65536 * S / (ms * 1e-3), "algorithmic_bytes": int(algo), "payload_bytes": int(pa + pb),
         "achieved_gbs": gbs, "peak_gbs": pk, "peak_source": src, "frac": gbs / pk, "nonzero_groups": int((res[0] > 0).sum()),
         "note": f"this GPU's 1/8 share ({S} of 4096 shards) of the 100 M-record config; load {time.time() - t0:.1f}s"})
    h.ctx.close()


class _NoBsiSort(_KernelMs):
    """the same proxy without bsi_sort: the executor extracts every (column, value) pair and sorts them on the host"""

    def __getattr__(self, name):
        if name == "bsi_sort":
            raise AttributeError(name)
        return super().__getattr__(name)


SORT_QUERIES = ["Sort(Row(v >= 0), field=v, sort-desc=true, limit=10)",       # every record, ten kept
                "Sort(Row(f=0), field=v, limit=10, offset=1000)",              # the 1 % row, a window past its start
                "Sort(Row(f=0), field=v)"]                                     # the 1 % row, no limit: about 100 K pairs returned


def config_sort(args, out):
    """Sort over config X's data (10 M records of a 32-bit field, a 1 % row f=0) through the executor: the device arm (one
    fbgpu_bsi_sort) and the composition arm (fbgpu_extract of every pair of the row, a Python sort, then the window), alternated
    step by step; the composition runs --composition-steps steps.  Both arms must return the same pairs."""
    from featurebase_b200 import datagen as D, executor as X
    n_rec = min(10_000_000, args.shards * SW)
    n_sh = (n_rec + SW - 1) // SW
    shards = np.arange(n_sh, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    f = idx.create_field("f")
    v = idx.create_field("v", "int", min=0, max=(1 << 32) - 1)
    bulk = D.fragments(11, shards, [0], 0.01)
    h.ctx.load_fragments(idx.id, f.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
    for s in range(n_sh):
        h.ctx.load_fragment(idx.id, v.id, X.VIEW_BSI, s, D.bsi_fragment(12, s, min(SW, n_rec - s * SW), 32, 0, (1 << 32) - 1))
    h.ctx.commit()
    idx.shards.update(range(n_sh))
    real = h.ctx
    card = _card()
    arms = {"device": _KernelMs(real), "composition": _NoBsiSort(real)}
    for q in SORT_QUERIES:
        rec = {name: {"wall": [], "kernel_ms": [], "queries": []} for name in arms}
        res = {}
        for i in range(1 + args.steps):                      # one warm-up round of the device arm, then alternate the arms
            for name in (sorted(arms) if i % 2 == 0 else sorted(arms, reverse=True)):
                if name == "composition" and len(rec[name]["wall"]) >= args.composition_steps:
                    continue
                h.ctx = arms[name]
                q0, arms[name].ms = real.counters()["queries"], 0.0
                t0 = time.perf_counter()
                r = X.Executor(h).execute("i", q)[0]
                wall = (time.perf_counter() - t0) * 1e3
                res.setdefault(name, r)
                assert r == res[name], (q, name)
                print(f"config O: {q}, {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                if i >= 1 or name == "composition":
                    rec[name]["wall"].append(wall)
                    rec[name]["kernel_ms"].append(arms[name].ms)
                    rec[name]["queries"].append(real.counters()["queries"] - q0)
        h.ctx = real
        equal = res.get("composition") == res["device"] if "composition" in res else None
        assert equal is not False, q
        for name, d in rec.items():
            if not d["wall"]:
                continue
            out({"config": "O", "query": q, "arm": name, "gpu": card, "records": n_rec, "shards": n_sh, "pairs": len(res[name]),
                 "equal_to_composition": equal, "wall_ms": float(np.median(d["wall"])), "wall_ms_min": float(np.min(d["wall"])),
                 "wall_ms_max": float(np.max(d["wall"])), "kernel_ms": float(np.median(d["kernel_ms"])), "queries": int(np.median(d["queries"])),
                 "steps": len(d["wall"]),
                 "kernel": ("eval_kernel + columns_emit_kernel + extract_values_kernel + sort_keys_kernel + sort_{hist,scan,scatter}_kernel"
                            if name == "device" else "eval_kernel + columns_emit_kernel + extract_values_kernel, host sort"),
                 "note": "median over the timed steps of the executor call (wall clock), of the summed last_query_gpu_ms and of the "
                         "number of its library queries"})
    real.close()


class _NoBsiDistinct(_KernelMs):
    """the same proxy without bsi_distinct: the executor extracts every value of the row and takes the distinct set on the host"""

    def __getattr__(self, name):
        if name == "bsi_distinct":
            raise AttributeError(name)
        return super().__getattr__(name)


DISTINCT_QUERIES = ["Distinct(field=v)",                                  # every record, nearly every value distinct
                    "Distinct(Row(f=0), field=v)",                        # the 1 % row
                    "Count(Distinct(field=w))",                           # every record, 64 values
                    "GroupBy(Rows(w))"]                                   # w's values, then one groupby_mixed call


def config_distinct(args, out):
    """Distinct over config X's data (10 M records of a 32-bit field v, a 1 % row f=0) plus a field w of 64 values on the same
    columns, through the executor: the device arm (one fbgpu_bsi_distinct per value list) and the composition arm (fbgpu_extract
    of every value of the row, then np.unique), alternated step by step; the composition runs --composition-steps steps.  Both
    arms must return the same result."""
    from featurebase_b200 import datagen as D, executor as X
    n_rec = min(10_000_000, args.shards * SW)
    n_sh = (n_rec + SW - 1) // SW
    shards = np.arange(n_sh, dtype=np.uint64)
    h = X.Holder()
    idx = h.create_index("i", track_existence=False)
    f = idx.create_field("f")
    v = idx.create_field("v", "int", min=0, max=(1 << 32) - 1)
    w = idx.create_field("w", "int", min=0, max=63)
    bulk = D.fragments(11, shards, [0], 0.01)
    h.ctx.load_fragments(idx.id, f.id, X.VIEW_STANDARD, shards, bulk.buf, bulk.offsets)
    for s in range(n_sh):
        n_cols = min(SW, n_rec - s * SW)
        h.ctx.load_fragment(idx.id, v.id, X.VIEW_BSI, s, D.bsi_fragment(12, s, n_cols, v.bit_depth, 0, (1 << 32) - 1))
        h.ctx.load_fragment(idx.id, w.id, X.VIEW_BSI, s, D.bsi_fragment(13, s, n_cols, w.bit_depth, 0, 63))
    h.ctx.commit()
    idx.shards.update(range(n_sh))
    real = h.ctx
    card = _card()
    arms = {"device": _KernelMs(real), "composition": _NoBsiDistinct(real)}
    for q in DISTINCT_QUERIES:
        rec = {name: {"wall": [], "kernel_ms": [], "queries": []} for name in arms}
        res = {}
        for i in range(1 + args.steps):                      # one warm-up round of the device arm, then alternate the arms
            for name in (sorted(arms) if i % 2 == 0 else sorted(arms, reverse=True)):
                if name == "composition" and len(rec[name]["wall"]) >= args.composition_steps:
                    continue
                h.ctx = arms[name]
                q0, arms[name].ms = real.counters()["queries"], 0.0
                t0 = time.perf_counter()
                r = X.Executor(h).execute("i", q)[0]
                wall = (time.perf_counter() - t0) * 1e3
                res.setdefault(name, r)
                assert r == res[name], (q, name)
                print(f"config U: {q}, {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                if i >= 1 or name == "composition":
                    rec[name]["wall"].append(wall)
                    rec[name]["kernel_ms"].append(arms[name].ms)
                    rec[name]["queries"].append(real.counters()["queries"] - q0)
        h.ctx = real
        equal = res.get("composition") == res["device"] if "composition" in res else None
        assert equal is not False, q
        r = res["device"]
        size = r.count() if isinstance(r, X.SignedRow) else len(r) if isinstance(r, list) else int(r)
        for name, d in rec.items():
            if not d["wall"]:
                continue
            out({"config": "U", "query": q, "arm": name, "gpu": card, "records": n_rec, "shards": n_sh, "result_size": size,
                 "equal_to_composition": equal, "wall_ms": float(np.median(d["wall"])), "wall_ms_min": float(np.min(d["wall"])),
                 "wall_ms_max": float(np.max(d["wall"])), "kernel_ms": float(np.median(d["kernel_ms"])), "queries": int(np.median(d["queries"])),
                 "steps": len(d["wall"]),
                 "kernel": ("eval_kernel + extract_values_kernel + sort_keys_kernel + sort_{hist,scan,scatter}_kernel + distinct_{heads,compact}_kernel"
                            if name == "device" else "eval_kernel + columns_emit_kernel + extract_values_kernel, host np.unique"),
                 "note": "median over the timed steps of the executor call (wall clock), of the summed last_query_gpu_ms and of the "
                         "number of its library queries; result_size: values listed, the count, or groups"})
    real.close()


class _NoExtractRows(_KernelMs):
    """the same proxy without extract_rows: the executor lists the field's rows under the filter, then expands the columns of
    filter ∩ Row(field=r) for every row r"""

    def __getattr__(self, name):
        if name == "extract_rows":
            raise AttributeError(name)
        return super().__getattr__(name)


EXTRACT_QUERIES = ["Extract(Row(f=0), Rows(a), Rows(m), Rows(b))",        # the 1 % row, three set-like children
                   "Extract(Limit(All(), limit=1000, offset=100000), Rows(a))",   # a window of the existence row
                   "Sort(Row(f=0), field=m, limit=10)"]


def config_extract_rows(args, out):
    """Extract and Sort over set-like fields through the executor, on 512 shards whose first 65,536 columns each hold about 4 of
    the 256 rows of a set field a, one of the 64 rows of a mutex field m and one row of a bool field b; f=0 holds 1 % of those
    columns.  Every shard holds the same fragments, encoded once.  The device arm (one fbgpu_extract_rows per set-like child,
    beside fbgpu_columns for Extract) runs over all shards; the composition arm (fbgpu_row_counts, then fbgpu_columns of
    filter ∩ Row(field=r) for every row r) over the first --composition-shards shards, for --composition-steps steps alternated
    with the device arm over the same shards.  Both arms must return the same result.  Progress goes to stderr."""
    from featurebase_b200 import executor as X, roaring_io
    S, n_cols = 512, 1 << 16
    h = X.Holder()
    idx = h.create_index("i")
    for name, typ in (("f", "set"), ("a", "set"), ("m", "mutex"), ("b", "bool")):
        idx.create_field(name, typ)
    rng = np.random.default_rng(2027)
    cols = np.arange(n_cols, dtype=np.uint64)
    a_rows = rng.integers(0, 256, size=(n_cols, 4)).astype(np.uint64)            # duplicates fold: about 3.98 rows per column
    data = {"a": roaring_io.encode((a_rows * np.uint64(SW) + cols[:, None]).ravel()),
            "m": roaring_io.encode(rng.integers(0, 64, n_cols).astype(np.uint64) * np.uint64(SW) + cols),
            "b": roaring_io.encode(rng.integers(0, 2, n_cols).astype(np.uint64) * np.uint64(SW) + cols),
            "f": roaring_io.encode(np.sort(rng.choice(n_cols, n_cols // 100, replace=False)).astype(np.uint64)),
            X.EXISTENCE_FIELD: roaring_io.encode(cols)}
    t0 = time.perf_counter()
    for s in range(S):
        for name, d in data.items():
            h.import_roaring("i", name, X.VIEW_STANDARD, s, d)
    h.ctx.commit()
    load_s = time.perf_counter() - t0
    real = h.ctx
    card = _card()
    dev, comp = _KernelMs(real), _NoExtractRows(real)
    CS = min(S, args.composition_shards)
    for q in EXTRACT_QUERIES:
        runs = [(S, {"device": dev})] + ([(CS, {"device": dev, "composition": comp})] if args.composition_steps > 0 else [])
        for n_sh, arms in runs:
            sh = list(range(n_sh))
            rec = {name: {"wall": [], "kernel_ms": [], "queries": []} for name in arms}
            res = {}
            for i in range(1 + args.steps):                  # one warm-up round of the device arm, then alternate the arms
                for name in (sorted(arms) if i % 2 == 0 else sorted(arms, reverse=True)):
                    if name == "composition" and len(rec[name]["wall"]) >= args.composition_steps:
                        continue
                    h.ctx = arms[name]
                    q0, arms[name].ms = real.counters()["queries"], 0.0
                    t1 = time.perf_counter()
                    r = X.Executor(h).execute("i", q, sh)[0]
                    wall = (time.perf_counter() - t1) * 1e3
                    res.setdefault(name, r)
                    assert r == res[name], (q, name)
                    print(f"config E: {q} over {n_sh} shards, {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                    if i >= 1 or name == "composition":
                        rec[name]["wall"].append(wall)
                        rec[name]["kernel_ms"].append(arms[name].ms)
                        rec[name]["queries"].append(real.counters()["queries"] - q0)
            h.ctx = real
            equal = res.get("composition") == res["device"] if "composition" in res else None
            assert equal is not False, q
            r = res["device"]
            size = len(r["columns"]) if isinstance(r, dict) else len(r)
            for name, d in rec.items():
                out({"config": "E", "query": q, "arm": name, "gpu": card, "shards": n_sh, "result_size": size, "equal_to_composition": equal,
                     "wall_ms": float(np.median(d["wall"])), "wall_ms_min": float(np.min(d["wall"])), "wall_ms_max": float(np.max(d["wall"])),
                     "kernel_ms": float(np.median(d["kernel_ms"])), "queries": int(np.median(d["queries"])), "steps": len(d["wall"]), "load_s": round(load_s, 1),
                     "kernel": ("eval_kernel + extract_rows_kernel<kCount, kEmit> + columns_emit_kernel + sort_{hist,scan,scatter}_kernel"
                                if name == "device" else "eval_kernel + row_count_kernel + columns_emit_kernel per row, host transposition"),
                     "note": "median over the timed steps of the executor call (wall clock), of the summed last_query_gpu_ms and of the "
                             "number of its library queries; result_size: Extract's columns or Sort's pairs"})
    real.close()


class _NoSparseDistinct(_KernelMs):
    """the same proxy without the sparse distinct calls: the executor lists the groups, then runs one Distinct per group"""

    def __getattr__(self, name):
        if name in ("groupby_sparse_distinct", "groupby_sparse_distinct_rows"):
            raise AttributeError(name)
        return super().__getattr__(name)


def config_groupby_sparse_distinct(args, out):
    """aggregate=Count(Distinct) over config G's data (_config_g_world with eight m fragments, so that Rows(m) lists more than
    65,535 rows and the executor takes the sparse path), over --groupby-shards shards:
      (a) GroupBy(Rows(m), aggregate=Count(Distinct(field=v)), limit=1000) through the executor: fbgpu_groupby_sparse_distinct
          against today's composition without it (the sparse list of groups, then one Distinct per group until 1,000 are
          listed), alternated; the same groups, counts and distinct counts;
      (b) GroupBy(Rows(m), Rows(a), aggregate=Count(Distinct(field=b))), every group, as library calls:
          fbgpu_groupby_sparse_distinct_rows over b's 256 rows against the counts-only fbgpu_groupby_sparse on the same
          dimensions, alternated, to show the cost of carrying x; the distinct call's cells must be among the counts-only
          call's, each with a distinct count of at least 1;
      (c) a x b, 256 x 256, with Count(Distinct(field=w)), as library calls: fbgpu_groupby_sparse_distinct against the dense
          fbgpu_groupby_distinct, alternated; the same cells (the dense tensor's non-zero ones) and distinct counts.
    Per arm: the median wall clock, the summed last_query_gpu_ms of the arm's library queries and their number."""
    from featurebase_b200 import executor as X
    S = args.groupby_shards
    h, idx, fa, fb, ff, fw, fv, fm, fe, load_s = _config_g_world(args, "J", m_fragments=8)
    real, card, sh = h.ctx, _card(), list(range(S))
    dev, comp = _KernelMs(real), _NoSparseDistinct(real)
    ra, rm = np.arange(256, dtype=np.uint64), np.arange(1_000_000, dtype=np.uint64)
    dims_ab = [(fa.id, [X.VIEW_STANDARD], ra), (fb.id, [X.VIEW_STANDARD], ra)]
    dims_ma = [(fm.id, [X.VIEW_STANDARD], rm), (fa.id, [X.VIEW_STANDARD], ra)]
    xw = (fw.id, X.VIEW_BSI, fw.bit_depth, np.arange(64, dtype=np.int64))      # w's stored values (Base 0)
    q = "GroupBy(Rows(m), aggregate=Count(Distinct(field=v)), limit=1000)"

    def executor(ctx):
        def run():
            h.ctx = ctx
            try:
                return X.Executor(h).execute("i", q, sh)[0]
            finally:
                h.ctx = real
        return run

    def dense_distinct():
        t = dev.groupby_distinct(idx.id, dims_ab, [], xw, sh).reshape(-1)
        nz = np.flatnonzero(t)
        return nz.astype(np.uint64), t[nz]

    arms = {"a": {"device": (dev, executor(dev)), "composition": (comp, executor(comp))},
            "b": {"sparse_distinct_rows": (dev, lambda: dev.groupby_sparse_distinct_rows(idx.id, dims_ma, (fb.id, X.VIEW_STANDARD, ra), sh)),
                  "sparse_counts": (dev, lambda: dev.groupby_sparse(idx.id, dims_ma, sh))},
            "c": {"sparse_distinct": (dev, lambda: dev.groupby_sparse_distinct(idx.id, dims_ab, xw, sh)), "dense_distinct": (dev, dense_distinct)}}
    for part, fns in arms.items():
        rec = {name: {"wall": [], "gpu_ms": [], "queries": []} for name in fns}
        res = {}
        for i in range(1 + args.steps):                          # one warm-up round, then alternate the arms
            for name in (sorted(fns) if i % 2 == 0 else sorted(fns, reverse=True)):
                proxy, fn = fns[name]
                q0, proxy.ms = real.counters()["queries"], 0.0
                t1 = time.perf_counter()
                r = fn()
                wall = (time.perf_counter() - t1) * 1e3
                res.setdefault(name, r)
                print(f"config J ({part}): {name} step {i}: {wall:.1f} ms", file=sys.stderr, flush=True)
                if i >= 1:
                    rec[name]["wall"].append(wall)
                    rec[name]["gpu_ms"].append(proxy.ms)
                    rec[name]["queries"].append(real.counters()["queries"] - q0)
        v = list(res.values())
        if part == "a":
            assert v[0] == v[1] and len(v[0]) == 1000, part
        elif part == "b":                                      # a listed cell is a group, and holds at least one row of b
            cells, dist = res["sparse_distinct_rows"]
            assert len(cells) and np.isin(cells, res["sparse_counts"][0]).all() and dist.min() >= 1, part
        else:
            assert all(np.array_equal(x[k], v[0][k]) for x in v for k in range(2)), part
        for name, dd in rec.items():
            out({"config": "J", "part": part, "arm": name, "gpu": card, "shards": S, "groups": len(res[name] if part == "a" else res[name][0]),
                 "checked": True, "wall_ms": float(np.median(dd["wall"])), "wall_ms_min": float(np.min(dd["wall"])),
                 "wall_ms_max": float(np.max(dd["wall"])), "gpu_ms": float(np.median(dd["gpu_ms"])), "queries": int(np.median(dd["queries"])),
                 "steps": len(dd["wall"]), "load_s": round(load_s, 1),
                 "note": "median over the timed steps of the wall clock (executor: Rows pre-pass included), of the summed last_query_gpu_ms "
                         "of the arm's library queries and of their number"})
    real.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="5,3,4")
    ap.add_argument("--steps", type=int, default=16)
    ap.add_argument("--shards", type=int, default=1024)
    ap.add_argument("--groupby-shards", type=int, default=512)
    ap.add_argument("--composition-steps", type=int, default=1, help="configs V, T, M, S, D, K, N, O, U, E: steps of the composition arm")
    ap.add_argument("--composition-shards", type=int, default=1, help="configs T, M, S, D, K, N, E: shards of the composition arm and of the device arm timed beside it")
    ap.add_argument("--composition-max-groups", type=int, default=4096, help="config K: the composition arm runs only for queries of at most this many groups")
    ap.add_argument("--topn-rows", type=int, default=1 << 14, help="config N: rows of the TopN field")
    ap.add_argument("--topn-shards", type=int, default=16, help="config N: shards (the fragments are encoded in Python: ~5 s per shard)")
    ap.add_argument("--generators", default="uniform,clustered")
    ap.add_argument("--batched", action="store_true", help="also time the multi-pair launch (config 5b)")
    ap.add_argument("--densities", default="0.0001,0.001,0.01,0.03,0.0625,0.125,0.25,0.5")
    args = ap.parse_args()

    def out(d):
        print(json.dumps(d), flush=True)

    for c in args.configs.split(","):
        c = c.strip()
        if c == "R":
            config_row(args, out)
        elif c == "X":
            config_extract(args, out)
        elif c == "P":
            config_percentile(args, out)
        elif c == "V":
            config_groupby_values(args, out)
        elif c == "T":
            config_time_views(args, out)
        elif c == "M":
            config_groupby_mixed(args, out)
        elif c == "S":
            config_groupby_sum(args, out)
        elif c == "D":
            config_groupby_distinct(args, out)
        elif c == "K":
            config_groupby_distinct_rows(args, out)
        elif c == "G":
            config_groupby_sparse(args, out)
        elif c == "H":
            config_groupby_sparse_sum(args, out)
        elif c == "J":
            config_groupby_sparse_distinct(args, out)
        elif c == "N":
            config_topn_cutoffs(args, out)
        elif c == "O":
            config_sort(args, out)
        elif c == "U":
            config_distinct(args, out)
        elif c == "E":
            config_extract_rows(args, out)
        elif c == "3L":     # the same BSI query at 256 shards (268 M records, 1.1 GB of planes): shows the kernel away from the launch-bound regime
            config3(args, out, n_rec=256 * SW, nf=1)
        else:
            {"5": config5, "3": config3, "4": config4}[c](args, out)


if __name__ == "__main__":
    main()
