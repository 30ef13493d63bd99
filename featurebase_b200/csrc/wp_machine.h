// Op loop of the word-parallel program machine (eval_wordpar_kernel), restructured to keep every value in a register with a
// fixed role.  Host-compilable on purpose: tests/test_program_compiler.py::test_wordpar_unrolled_loop_matches_stack_model checks it
// on the CPU against a plain stack-machine model for random programs.
//
// Why: in a loop where the operand prefetch ring (p0 <- p1 <- p2) rotates and the 4-deep register stack shifts inside one
// generic loop body, ptxas emits ~40-60 register moves per op around 4 useful logic instructions (cuobjdump: blocks of
// IMAD.MOV per switch case) — interpretive overhead that limited the first form of the kernel.  Here the loop walks ROW ops
// R at a time; ring slot j always serves row op R*t+j, so there is no rotation, and the ops that do move the stack
// (PUSH_EMPTY / SWAP / POP / binary ops, rare in BSI sweeps) run in a separate small loop between row ops.
#pragma once
#include <stdint.h>

#include "bitaddr.h"        // FBGPU_HD
#include "fbgpu_types.h"

#if defined(__CUDACC__)
#define FBGPU_NO_UNROLL _Pragma("unroll 1")
#else
#define FBGPU_NO_UNROLL
#endif

namespace fbgpu {

template <class V>
struct WpStack {            // T = top, B = below, S2, S3 deeper (the host checks depth <= 4)
    V T, B, S2, S3; int depth;
};

template <class V> FBGPU_HD V wp_and(V a, V b) { V r; r.x = a.x & b.x; r.y = a.y & b.y; r.z = a.z & b.z; r.w = a.w & b.w; return r; }
template <class V> FBGPU_HD V wp_or(V a, V b) { V r; r.x = a.x | b.x; r.y = a.y | b.y; r.z = a.z | b.z; r.w = a.w | b.w; return r; }
template <class V> FBGPU_HD V wp_xor(V a, V b) { V r; r.x = a.x ^ b.x; r.y = a.y ^ b.y; r.z = a.z ^ b.z; r.w = a.w ^ b.w; return r; }
template <class V> FBGPU_HD V wp_andn(V a, V b) { V r; r.x = a.x & ~b.x; r.y = a.y & ~b.y; r.z = a.z & ~b.z; r.w = a.w & ~b.w; return r; }
template <class V> FBGPU_HD V wp_zero() { V r; r.x = 0; r.y = 0; r.z = 0; r.w = 0; return r; }

// ops that take no row operand
template <class V>
FBGPU_HD void wp_stack_op(WpStack<V>& s, uint8_t opc) {
    if (opc == D_PUSH_EMPTY) { s.S3 = s.S2; s.S2 = s.B; s.B = s.T; s.T = wp_zero<V>(); s.depth++; }
    else if (opc == D_SWAP) { V t = s.T; s.T = s.B; s.B = t; }
    else if (opc == D_POP) { s.T = s.B; s.B = s.S2; s.S2 = s.S3; s.depth--; }
    else {
        s.T = opc == D_AND ? wp_and(s.B, s.T) : opc == D_OR ? wp_or(s.B, s.T) : opc == D_ANDNOT ? wp_andn(s.B, s.T) : wp_xor(s.B, s.T);
        s.B = s.S2; s.S2 = s.S3; s.depth--;
    }
}
// ops that take a row operand x.  Every case updates T or B in place; PUSH_ROW is executed as PUSH_EMPTY (the only
// stack shift, kept out of the hot switch) followed by T |= x, so that the switch arms leave all other registers alone
// and the compiler has nothing to copy where they join.
// NO_PUSH: the program was rewritten by expand_push_row() (program_compiler.h) and holds no PUSH_ROW, so the hot switch
// contains no stack shift at all (otherwise the shift is compiled as ~14 predicated moves that issue on every row op).
template <bool NO_PUSH, class V>
FBGPU_HD void wp_row_op(WpStack<V>& s, uint8_t opc, V x) {
    if (!NO_PUSH && opc == D_PUSH_ROW) { wp_stack_op(s, D_PUSH_EMPTY); opc = D_OR_ROW; }
    // one expression per arm, each a single three-input LOP3 per word, each updating T or B in place
    if (opc == D_ORAND_ROW) s.B = wp_or(s.B, wp_and(s.T, x));
    else if (opc == D_ORANDNOT_ROW) s.B = wp_or(s.B, wp_andn(s.T, x));
    else if (opc == D_AND_ROW) s.T = wp_and(s.T, x);
    else if (opc == D_ANDNOT_ROW) s.T = wp_andn(s.T, x);
    else if (opc == D_OR_ROW) s.T = wp_or(s.T, x);
    else s.T = wp_xor(s.T, x);                                      // D_XOR_ROW
}

// opc(k): opcode of program op k; is_row(k); rowops[ri]: program index of the ri-th row op; fetch(ri): its operand slice.
// Returns the top of stack (zero when the program leaves the stack empty).  R = operand slices fetched ahead per thread: ring slot j
// always serves row op R*t + j, so the ring never rotates.  The default R = 1 is what eval_wordpar_kernel runs: its fetch() reads a
// cp.async ring in shared memory that already keeps the loads in flight.
template <class V, bool NO_PUSH, int R = 1, class OpcAt, class IsRowAt, class RowOpAt, class Fetch>
FBGPU_HD V wp_run_unrolled(int n_ops, int nr, OpcAt opc_at, IsRowAt is_row_at, RowOpAt rowop_at, Fetch fetch) {
    WpStack<V> s; s.T = s.B = s.S2 = s.S3 = wp_zero<V>(); s.depth = 0;
    V p[R];
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int j = 0; j < R; j++) { p[j] = wp_zero<V>(); if (j < nr) p[j] = fetch(j); }
    int k = 0;                                         // next program op to execute
    for (int base = 0; base < nr; base += R) {
#if defined(__CUDACC__)
#pragma unroll
#endif
        for (int j = 0; j < R; j++) {
            if (base + j < nr) {
                const int kr = rowop_at(base + j);
                FBGPU_NO_UNROLL for (; k < kr; k++) wp_stack_op(s, opc_at(k));
                wp_row_op<NO_PUSH>(s, opc_at(kr), p[j]); k = kr + 1;
                if (base + j + R < nr) p[j] = fetch(base + j + R);
            }
        }
    }
    FBGPU_NO_UNROLL for (; k < n_ops; k++) wp_stack_op(s, opc_at(k));     // trailing stack ops (and programs without any row op)
    (void)is_row_at;
    return s.depth > 0 ? s.T : wp_zero<V>();
}

}  // namespace fbgpu
