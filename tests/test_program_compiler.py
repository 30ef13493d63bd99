"""featurebase_b200/csrc/program_compiler.h on the CPU: the C++ compiler that turns a post-order fbgpu_op program into the
kernels' stack-machine ops (fold order, fused row batches, the BSI plane-sweep expansions of fragment.go:937-1303) is
host code, so it is compiled with g++ here and its OUTPUT is executed by a small Python stack machine over oracle
bitmaps, then compared with the direct evaluation of the same fbgpu_op program (tests/oracle_ctx.OracleCtx: oracle set
operations and the oracle's own rangeOp restatement).  The CUDA kernels implement exactly this stack machine
(fbgpu_types.h: D_* semantics); they are covered by the -m gpu tests."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from featurebase_b200 import lib as L
from oracle import oracle as O
from tests import helpers as H
from tests.oracle_ctx import OracleCtx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
(D_PUSH_ROW, D_PUSH_EMPTY, D_OR_ROW, D_AND_ROW, D_ANDNOT_ROW, D_XOR_ROW, D_ORAND_ROW, D_ORANDNOT_ROW, D_AND, D_OR, D_ANDNOT, D_XOR,
 D_SWAP, D_POP) = range(1, 15)
NO_VIEW = 0xFFFFFFFF


class DevOp(C.Structure):
    _fields_ = [("op", C.c_uint8), ("pad", C.c_uint8 * 3), ("fv", C.c_uint32), ("row", C.c_uint64)]


@pytest.fixture(scope="module")
def cc():
    out = os.path.join(tempfile.mkdtemp(prefix="compile_check_"), "libcompile_check.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-I", os.path.join(ROOT, "featurebase_b200", "csrc"),
                           os.path.join(ROOT, "tests", "native", "compile_check.cpp"), "-o", out])
    return C.CDLL(out)


def compile_ops(cc, ops):
    arr = L.ops_array(ops)
    out = (DevOp * 4096)()
    n, depth = C.c_int32(0), C.c_int32(0)
    err = C.create_string_buffer(512)
    rc = cc.compile_ops(arr, len(ops), out, 4096, C.byref(n), C.byref(depth), err, 512)
    if rc:
        raise L.FbgpuError(rc, err.value.decode())
    return [(o.op, o.fv, o.row) for o in out[: n.value]], depth.value


def run_devops(ctx, index, prog, depth, shard):
    """the stack machine of fbgpu_types.h / eval_kernel, over oracle bitmaps"""
    st = []

    def row(fv, r):
        return O.Bitmap() if fv == NO_VIEW else ctx._row(index, fv >> 2, fv & 3, r, shard)
    for op, fv, r in prog:
        if op == D_PUSH_ROW:
            st.append(row(fv, r))
        elif op == D_PUSH_EMPTY:
            st.append(O.Bitmap())
        elif op == D_OR_ROW:
            st[-1] = st[-1].union(row(fv, r))
        elif op == D_AND_ROW:
            st[-1] = st[-1].intersect(row(fv, r))
        elif op == D_ANDNOT_ROW:
            st[-1] = st[-1].difference(row(fv, r))
        elif op == D_XOR_ROW:
            st[-1] = st[-1].xor(row(fv, r))
        elif op == D_ORAND_ROW:
            st[-2] = st[-2].union(st[-1].intersect(row(fv, r)))
        elif op == D_ORANDNOT_ROW:
            st[-2] = st[-2].union(st[-1].difference(row(fv, r)))
        elif op in (D_AND, D_OR, D_ANDNOT, D_XOR):
            b = st.pop()
            a = st[-1]
            st[-1] = {D_AND: a.intersect, D_OR: a.union, D_ANDNOT: a.difference, D_XOR: a.xor}[op](b)
        elif op == D_SWAP:
            st[-1], st[-2] = st[-2], st[-1]
        elif op == D_POP:
            st.pop()
        else:
            raise AssertionError(op)
        assert 0 <= len(st) <= depth, (len(st), depth)      # (a POP + PUSH_EMPTY pair may empty the stack transiently)
    assert len(st) == 1
    return st[0]


def check(cc, ctx, ops, shards=(0,)):
    prog, depth = compile_ops(cc, ops)
    for s in shards:
        got = run_devops(ctx, 0, prog, depth, s)
        exp = ctx._eval(0, ops, s)
        assert got.count() == exp.count() and got.to_bytes() == exp.to_bytes(), [(o.opcode, o.argc, o.a, o.b, o.lo, o.hi) for o in ops]
    return prog


def op(code, field=0, view=0, argc=0, a=0, b=0, lo=0, hi=0):
    return L.Op(code, field, view, argc, a, b, lo, hi)


def test_bsi_expansions_exhaustive_diagonal(cc):
    """every comparison and predicate of the reference's diagonal tests (fragment_internal_test.go:3768-3948, 4113-4275),
    signed and unsigned, plus between ranges, through compile -> stack machine"""
    SW = H.SW
    for signed in (False, True):
        k = 6
        values = {i + 70: i for i in (range(1 - (1 << k), 1 << k) if signed else range(1 << k))}
        ctx = OracleCtx()
        ctx.frags[(0, 1, 1)] = {0: H.bsi_fragment(values, k)}
        preds = range(-2 * (1 << k), 2 * (1 << k) + 1)
        for pr in preds:
            for cmp_name in ("==", "!=", "<", "<=", ">", ">="):
                ops = [op(L.OP_BSI_RANGE, 1, 1, 0, k, L.CMP[cmp_name], pr, 0)]
                prog, depth = compile_ops(cc, ops)
                got = run_devops(ctx, 0, prog, depth, 0)
                f = {"==": lambda v: v == pr, "!=": lambda v: v != pr, "<": lambda v: v < pr, "<=": lambda v: v <= pr,
                     ">": lambda v: v > pr, ">=": lambda v: v >= pr}[cmp_name]
                inside = abs(pr) < (1 << k)
                if inside:                                 # literal expectation (predicates the bit depth can represent)
                    assert got.slice().tolist() == sorted(c for c, v in values.items() if f(v)), (signed, cmp_name, pr)
                assert got.to_bytes() == ctx._eval(0, ops, 0).to_bytes(), (signed, cmp_name, pr)     # oracle rangeOp incl. clamped cases
            for hi in (pr, pr + 1, pr + 9, pr + 200):
                ops = [op(L.OP_BSI_RANGE, 1, 1, 0, k, L.CMP["><"], pr, hi)]
                prog, depth = compile_ops(cc, ops)
                got = run_devops(ctx, 0, prog, depth, 0)
                assert got.to_bytes() == ctx._eval(0, ops, 0).to_bytes(), (signed, pr, hi)
                if abs(pr) < (1 << k) and abs(hi) < (1 << k):
                    assert got.slice().tolist() == sorted(c for c, v in values.items() if pr <= v <= hi)


def test_bsi_wide_depths(cc):
    rng = np.random.default_rng(4)
    for depth, lo, hi in ((1, -1, 1), (12, -4000, 4000), (33, -(1 << 32), 1 << 32), (63, -(1 << 62), 1 << 62), (64, -(1 << 63), (1 << 63) - 1)):
        cols = rng.choice(200000, 400, replace=False)
        values = {int(c): int(v) for c, v in zip(cols, rng.integers(lo, hi, 400, dtype=np.int64, endpoint=True))}
        ctx = OracleCtx()
        ctx.frags[(0, 2, 1)] = {0: H.bsi_fragment(values, depth)}
        vs = sorted(values.values())
        preds = [0, 1, -1, lo, hi, vs[0], vs[-1], vs[len(vs) // 2], vs[len(vs) // 3] + 1, (1 << min(depth, 62)) - 1, -(1 << min(depth, 62))]
        for pr in preds:
            pr = max(min(pr, (1 << 63) - 1), -(1 << 63))
            for cmp_name in ("==", "!=", "<", "<=", ">", ">="):
                check(cc, ctx, [op(L.OP_BSI_RANGE, 2, 1, 0, depth, L.CMP[cmp_name], pr, 0)])
        for a, b in ((vs[3], vs[-3]), (0, vs[-1]), (vs[0], 0), (vs[10], vs[10]), (vs[-1], vs[0])):
            check(cc, ctx, [op(L.OP_BSI_RANGE, 2, 1, 0, depth, L.CMP["><"], a, b)])


def _random_tree(rng, fields, depth):
    """post-order fbgpu_op list of a random bitmap call"""
    if depth == 0 or rng.random() < 0.35:
        r = rng.random()
        if r < 0.75:
            f = int(rng.choice(fields))
            return [op(L.OP_ROW, f, 0, 0, int(rng.integers(0, 6)))]
        if r < 0.85:
            return [op(L.OP_EMPTY)]
        if r < 0.93:
            return [op(L.OP_ROW, 1000, 0, 0, 1)]                # a field the store has never seen: empty row
        return [op(L.OP_BSI_RANGE, 9, 1, 0, 10, int(rng.integers(1, 7)), int(rng.integers(-600, 600)), 0)]
    kind = int(rng.choice([L.OP_INTERSECT, L.OP_UNION, L.OP_DIFFERENCE, L.OP_XOR, L.OP_NOT]))
    if kind == L.OP_NOT:
        return _random_tree(rng, fields, depth - 1) + [op(L.OP_NOT, 0, 0, 1, 0)]
    n = int(rng.integers(1, 6))
    out = []
    for _ in range(n):
        out += _random_tree(rng, fields, depth - 1)
    return out + [op(kind, 0, 0, n)]


def test_random_trees_match_direct_evaluation(cc):
    """n-ary folds with complex children first and leaf rows batched, Not over the existence row, unknown views, BSI leaves
    inside set operations: compiled program == direct evaluation, on two shards with different content"""
    rng = np.random.default_rng(12)
    ctx = OracleCtx()
    SW = H.SW
    for shard in (0, 3):
        for f in (0, 1, 2):                                 # field 0 doubles as the existence field of Not (row 0)
            rows = {r: rng.choice(SW, int(rng.integers(50, 3000)), replace=False) for r in range(6)}
            ctx.frags.setdefault((0, f, 0), {})[shard] = O.Bitmap.from_values(
                np.concatenate([np.uint64(r * SW) + c.astype(np.uint64) for r, c in rows.items()]))
        vals = {int(c): int(v) for c, v in zip(rng.choice(SW, 1500, replace=False), rng.integers(-500, 500, 1500))}
        ctx.frags.setdefault((0, 9, 1), {})[shard] = H.bsi_fragment(vals, 10)
    depths = []
    for _ in range(300):
        ops = _random_tree(rng, [0, 1, 2], 3)
        try:
            prog = check(cc, ctx, ops, shards=(0, 3))
        except L.FbgpuError as e:
            assert "stack depth" in str(e)                  # > 15 operands deep: rejected, never mis-compiled
            continue
        depths.append(len(prog))
    assert len(depths) > 250


def test_fold_shape_and_errors(cc):
    """the headline query compiles to PUSH_EMPTY + 32 fused ORs, twice, then one AND: two barrier-free batches"""
    ua = [op(L.OP_ROW, 1, 0, 0, r) for r in range(32)] + [op(L.OP_UNION, argc=32)]
    ub = [op(L.OP_ROW, 1, 0, 0, r) for r in range(32, 64)] + [op(L.OP_UNION, argc=32)]
    prog, depth = compile_ops(cc, ua + ub + [op(L.OP_INTERSECT, argc=2)])
    kinds = [p[0] for p in prog]
    assert kinds == [D_PUSH_EMPTY] + [D_OR_ROW] * 32 + [D_PUSH_EMPTY] + [D_OR_ROW] * 32 + [D_AND] and depth == 2
    prog, depth = compile_ops(cc, [op(L.OP_ROW, 1, 0, 0, 5), op(L.OP_ROW, 1, 0, 0, 6), op(L.OP_INTERSECT, argc=2)])
    assert [p[0] for p in prog] == [D_PUSH_ROW, D_AND_ROW] and depth == 1          # the fused pair-count fast path's shape
    for bad, msg in (([op(L.OP_INTERSECT, argc=0)], "empty Intersect"), ([op(L.OP_DIFFERENCE, argc=0)], "empty Difference"),
                     ([op(L.OP_ROW, 1), op(L.OP_ROW, 1)], "exactly one result"), ([op(L.OP_UNION, argc=3)], "pops 3"),
                     ([op(99)], "unknown opcode"), ([op(L.OP_BSI_RANGE, 1, 1, 0, 65, 1, 0, 0)], "bit depth"),
                     ([op(L.OP_BSI_RANGE, 1, 1, 0, 8, 42, 0, 0)], "invalid range operation")):
        with pytest.raises(L.FbgpuError, match=msg):
            compile_ops(cc, bad)
    assert [p[0] for p in compile_ops(cc, [op(L.OP_UNION, argc=0)])[0]] == [D_PUSH_EMPTY]
    assert [p[0] for p in compile_ops(cc, [op(L.OP_XOR, argc=0)])[0]] == [D_PUSH_EMPTY]


def test_wordpar_unrolled_loop_matches_stack_model(cc):
    """csrc/wp_machine.h (the fixed-register op loop of eval_wordpar_kernel) against a plain
    Python stack machine on 128-bit slices: programs from the real compiler (random call trees with BSI leaves, every
    comparison at several depths), random operand slices incl. all-zero / all-one rows"""
    rng = np.random.default_rng(33)
    M = (1 << 128) - 1

    def model(prog, slices):
        st, ri = [], 0
        for op, fv, row in prog:
            if op in (D_PUSH_ROW, D_OR_ROW, D_AND_ROW, D_ANDNOT_ROW, D_XOR_ROW, D_ORAND_ROW, D_ORANDNOT_ROW):
                x = slices[ri]
                ri += 1
                if op == D_PUSH_ROW:
                    st.append(x)
                elif op == D_OR_ROW:
                    st[-1] |= x
                elif op == D_AND_ROW:
                    st[-1] &= x
                elif op == D_ANDNOT_ROW:
                    st[-1] &= ~x & M
                elif op == D_XOR_ROW:
                    st[-1] ^= x
                elif op == D_ORAND_ROW:
                    st[-2] |= st[-1] & x
                else:
                    st[-2] |= st[-1] & ~x & M
            elif op == D_PUSH_EMPTY:
                st.append(0)
            elif op == D_SWAP:
                st[-1], st[-2] = st[-2], st[-1]
            elif op == D_POP:
                st.pop()
            else:
                b = st.pop()
                st[-1] = {D_AND: st[-1] & b, D_OR: st[-1] | b, D_ANDNOT: st[-1] & ~b & M, D_XOR: st[-1] ^ b}[op]
        return st[-1] if st else 0

    def run(prog):
        n_row = sum(1 for op, _, _ in prog if op in (D_PUSH_ROW, D_OR_ROW, D_AND_ROW, D_ANDNOT_ROW, D_XOR_ROW, D_ORAND_ROW, D_ORANDNOT_ROW))
        words = rng.integers(0, 1 << 32, (max(n_row, 1), 4), dtype=np.uint64).astype(np.uint32)
        for k in range(n_row):
            r = rng.random()
            if r < 0.1:
                words[k] = 0
            elif r < 0.2:
                words[k] = 0xFFFFFFFF
        slices = [int(w[0]) | int(w[1]) << 32 | int(w[2]) << 64 | int(w[3]) << 96 for w in words]
        arr = (DevOp * max(len(prog), 1))()
        for i, (op, fv, row) in enumerate(prog):
            arr[i].op, arr[i].fv, arr[i].row = op, fv, row
        for no_push in (0, 1):                               # 1: PUSH_ROW rewritten to PUSH_EMPTY + OR_ROW first (what the kernel runs)
            out = (C.c_uint32 * 4)()
            cc.wp_run(arr, len(prog), np.ascontiguousarray(words).ctypes.data_as(C.c_void_p), out, no_push)
            got = out[0] | out[1] << 32 | out[2] << 64 | out[3] << 96
            assert got == model(prog, slices), (no_push, prog)

    n = 0
    for depth in (1, 6, 32, 63):
        for cmp_name in ("==", "!=", "<", "<=", ">", ">="):
            for pred in (0, 1, -1, 5, -37, (1 << (depth - 1)), (1 << depth) - 1, -(1 << depth) + 1, 1 << depth):
                prog, d = compile_ops(cc, [op(L.OP_BSI_RANGE, 2, 1, 0, depth, L.CMP[cmp_name], pred, 0)])
                if d <= 4:
                    run(prog)
                    n += 1
        for lo, hi in ((0, 5), (-9, 9), (-(1 << depth) + 1, (1 << depth) - 1), (3, 3), (7, 2)):
            prog, d = compile_ops(cc, [op(L.OP_BSI_RANGE, 2, 1, 0, depth, L.CMP["><"], lo, hi)])
            if d <= 4:
                run(prog)
                n += 1
    for _ in range(400):
        try:
            prog, d = compile_ops(cc, _random_tree(rng, [0, 1, 2], 3))
        except L.FbgpuError:
            continue
        if d <= 4:                                           # kWpMaxDepth
            run(prog)
            n += 1
    run([])                                                  # no ops at all
    run([(D_PUSH_EMPTY, NO_VIEW, 0)])
    assert n > 450
