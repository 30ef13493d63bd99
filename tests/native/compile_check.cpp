// Host-only harness around featurebase_b200/csrc/program_compiler.h for tests/test_program_compiler.py (g++, no CUDA).
// View slots are synthesised as (field << 2) | view so that the Python side can map them back.
#include "program_compiler.h"
#include <cstring>
extern "C" int compile_ops(const fbgpu_op* ops, int32_t n_ops, fbgpu::DevOp* out, int32_t cap, int32_t* n_out, int32_t* depth, char* err, int32_t err_cap) {
    fbgpu::Error e; std::vector<fbgpu::DevOp> prog; int d = 0;
    fbgpu::ViewLookup lookup = [](uint32_t field, uint32_t view) { return field >= 1000 ? fbgpu::kNoView : (field << 2) | view; };
    int rc = fbgpu::compile(ops, n_ops, lookup, prog, d, e);
    if (rc) { snprintf(err, err_cap, "%s", e.msg); return rc; }
    *n_out = (int32_t)prog.size(); *depth = d;
    if ((int32_t)prog.size() > cap) return 1;
    memcpy(out, prog.data(), prog.size() * sizeof(fbgpu::DevOp));
    return 0;
}

// featurebase_b200/csrc/wp_machine.h (op loop of the word-parallel kernel) on the host: runs a compiled
// program over caller-provided 128-bit operand slices (one per row op, in program order) and returns the result slice.
#include "wp_machine.h"
struct U4 { uint32_t x, y, z, w; };
extern "C" void wp_run(const fbgpu::DevOp* prog_in, int32_t n_ops_in, const uint32_t* slices /* [n_rowops][4] */, uint32_t out[4], int32_t no_push) {
    std::vector<fbgpu::DevOp> pv(prog_in, prog_in + n_ops_in);
    if (no_push) fbgpu::expand_push_row(pv);           // what compile_program does before launching
    const fbgpu::DevOp* prog = pv.data(); const int n_ops = (int)pv.size();
    std::vector<uint16_t> rowops;
    auto is_row = [&](int k) { uint8_t o = prog[k].op; return o >= fbgpu::D_PUSH_ROW && o <= fbgpu::D_ORANDNOT_ROW && o != fbgpu::D_PUSH_EMPTY; };
    for (int k = 0; k < n_ops; k++) if (is_row(k)) rowops.push_back((uint16_t)k);
    auto opc = [&](int k) { return prog[k].op; };
    auto rop = [&](int ri) { return (int)rowops[ri]; };
    auto fetch = [&](int ri) { U4 v{ slices[4 * ri], slices[4 * ri + 1], slices[4 * ri + 2], slices[4 * ri + 3] }; return v; };
    U4 r = no_push ? fbgpu::wp_run_unrolled<U4, true, 1>(n_ops, (int)rowops.size(), opc, is_row, rop, fetch)     // what the kernel runs
                   : fbgpu::wp_run_unrolled<U4, false, 1>(n_ops, (int)rowops.size(), opc, is_row, rop, fetch);
    out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}
