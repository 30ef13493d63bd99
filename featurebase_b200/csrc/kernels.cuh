// Hand-written sm_90a (H100) kernels of libfbgpu.  Pure integer / bitwise work, HBM-bound: no tensor cores.
//
//   eval_kernel        one CTA per (shard, container slot): runs a compiled bitmap-call program with its
//                      operand stack held as 8 KiB bitmaps in shared memory (replaces executeBitmapCallShard +
//                      Row/roaring set algebra, executor.go:1782, row.go:242-353, roaring.go:736-1623).
//   pair_count_kernel  one warp per container pair: fused Intersect+Count for Count(Intersect(Row,Row))
//                      (replaces roaring.intersectionCount's 9 type-pair kernels, roaring.go:4477-4614).
//   row_count_kernel   one warp per (shard,row): per-row |row ∩ filter| (doTopK executor.go:2705, fragment.top).
//   groupby_kernel     one CTA per (shard, slot): column-keyed join of two fields' rows (groupByIterator :8617).
//   canon_*            canonical (optimize()) container emission for Row results (roaring.go:3412-3461).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "fbgpu_types.h"
#include "bitaddr.h"
#include "wp_machine.h"
#include "resolve.h"

namespace fbgpu {

constexpr int kEvalThreads = 256;
constexpr int kEvalMinBlocks = 6;      // 40 registers: room for three chunk loads in flight per lane (faster on the headline query than 8 CTAs / 32 registers)
constexpr int kEvalU4PerThread = 512 / kEvalThreads;       // uint4 per thread of an 8 KiB bitmap
constexpr int kEvalW64PerThread = 1024 / kEvalThreads;     // consecutive u64 words per thread in scans
constexpr int kResolveChunk = 128;

__device__ __forceinline__ uint4 ldg_nc(const uint4* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ int popc4(uint4 v) { return __popc(v.x) + __popc(v.y) + __popc(v.z) + __popc(v.w); }
__device__ __forceinline__ uint4 and4(uint4 a, uint4 b) { return make_uint4(a.x & b.x, a.y & b.y, a.z & b.z, a.w & b.w); }
__device__ __forceinline__ uint4 or4(uint4 a, uint4 b) { return make_uint4(a.x | b.x, a.y | b.y, a.z | b.z, a.w | b.w); }
__device__ __forceinline__ uint4 xor4(uint4 a, uint4 b) { return make_uint4(a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w); }
__device__ __forceinline__ uint4 andn4(uint4 a, uint4 b) { return make_uint4(a.x & ~b.x, a.y & ~b.y, a.z & ~b.z, a.w & ~b.w); }

// ------------------------------------------------------------------------------------------------
// CTA-level helpers on 8 KiB shared-memory bitmaps (uint4[512]); thread t owns uint4 t and t+256.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void bm_zero(uint4* d) {
#pragma unroll
    for (int h = 0; h < kEvalU4PerThread; h++) d[threadIdx.x + h * kEvalThreads] = make_uint4(0, 0, 0, 0);
}
// scatter an array container into a bitmap with MODE 0: |=  1: &= ~  2: ^=
template <int MODE>
__device__ __forceinline__ void bm_scatter(uint32_t* bm, const uint16_t* arr, uint32_t n) {
    const uint32_t* a32 = reinterpret_cast<const uint32_t*>(arr);
    uint32_t n2 = (n + 1) >> 1;
    for (uint32_t i = threadIdx.x; i < n2; i += kEvalThreads) {
        uint32_t v = __ldg(a32 + i);
        uint32_t lo = v & 0xffffu, hi = v >> 16;
        if (MODE == 0) atomicOr(&bm[lo >> 5], 1u << (lo & 31)); else if (MODE == 1) atomicAnd(&bm[lo >> 5], ~(1u << (lo & 31))); else atomicXor(&bm[lo >> 5], 1u << (lo & 31));
        if (2 * i + 1 < n) {
            if (MODE == 0) atomicOr(&bm[hi >> 5], 1u << (hi & 31)); else if (MODE == 1) atomicAnd(&bm[hi >> 5], ~(1u << (hi & 31))); else atomicXor(&bm[hi >> 5], 1u << (hi & 31));
        }
    }
}
// for each array element present in `src`, set it in `dst`
__device__ __forceinline__ void bm_filter_scatter(uint32_t* dst, const uint32_t* src, const uint16_t* arr, uint32_t n) {
    const uint32_t* a32 = reinterpret_cast<const uint32_t*>(arr);
    uint32_t n2 = (n + 1) >> 1;
    for (uint32_t i = threadIdx.x; i < n2; i += kEvalThreads) {
        uint32_t v = __ldg(a32 + i);
        uint32_t lo = v & 0xffffu, hi = v >> 16;
        if ((src[lo >> 5] >> (lo & 31)) & 1) atomicOr(&dst[lo >> 5], 1u << (lo & 31));
        if (2 * i + 1 < n && ((src[hi >> 5] >> (hi & 31)) & 1)) atomicOr(&dst[hi >> 5], 1u << (hi & 31));
    }
}
// Expand a run container into `dst` (overwrites).  Delta bitmap (toggle at start and last+1) followed by a
// CTA-wide prefix-XOR scan: O(runs + 1024 words), independent of run lengths (runToBitmap roaring.go:3792).
__device__ __noinline__ void bm_expand_runs(uint4* dst4, const uint16_t* runs, uint32_t n_runs, uint32_t* warp_par /*[8]*/) {
    bm_zero(dst4);
    __syncthreads();
    uint32_t* d32 = reinterpret_cast<uint32_t*>(dst4);
    const uint32_t* r32 = reinterpret_cast<const uint32_t*>(runs);
    for (uint32_t i = threadIdx.x; i < n_runs; i += kEvalThreads) {
        uint32_t v = __ldg(r32 + i);
        uint32_t s = v & 0xffffu, e = (v >> 16) + 1;
        atomicXor(&d32[s >> 5], 1u << (s & 31));
        if (e < 65536u) atomicXor(&d32[e >> 5], 1u << (e & 31));
    }
    __syncthreads();
    // thread t owns kEvalW64PerThread consecutive u64 words
    uint64_t* d64 = reinterpret_cast<uint64_t*>(dst4);
    uint64_t w[kEvalW64PerThread]; uint32_t carry = 0;
#pragma unroll
    for (int k = 0; k < kEvalW64PerThread; k++) {
        uint64_t x = d64[kEvalW64PerThread * threadIdx.x + k];
        x ^= x << 1; x ^= x << 2; x ^= x << 4; x ^= x << 8; x ^= x << 16; x ^= x << 32;
        if (carry) x = ~x;
        carry = (uint32_t)(x >> 63);
        w[k] = x;
    }
    unsigned b = __ballot_sync(0xffffffffu, carry);
    int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t excl = __popc(b & ((1u << lane) - 1u)) & 1u;
    if (lane == 0) warp_par[wid] = __popc(b) & 1u;
    __syncthreads();
    for (int k = 0; k < wid; k++) excl ^= warp_par[k];
#pragma unroll
    for (int k = 0; k < kEvalW64PerThread; k++) d64[kEvalW64PerThread * threadIdx.x + k] = excl ? ~w[k] : w[k];
    __syncthreads();
}

enum { K_PUSH = 0, K_OR, K_AND, K_ANDNOT, K_XOR, K_ORAND, K_ORANDNOT };

// top = f(top, g)   or   below |= top & (~)g   with g streamed from global (bitmap container)
__device__ __forceinline__ void bm_apply_global(int kind, uint4* top, uint4* below, const uint4* g) {
#pragma unroll
    for (int h = 0; h < kEvalU4PerThread; h++) {
        int i = threadIdx.x + h * kEvalThreads;
        uint4 x = ldg_nc(g + i);
        switch (kind) {
            case K_PUSH: top[i] = x; break;
            case K_OR: top[i] = or4(top[i], x); break;
            case K_AND: top[i] = and4(top[i], x); break;
            case K_ANDNOT: top[i] = andn4(top[i], x); break;
            case K_XOR: top[i] = xor4(top[i], x); break;
            case K_ORAND: below[i] = or4(below[i], and4(top[i], x)); break;
            default: below[i] = or4(below[i], andn4(top[i], x)); break;
        }
    }
}
__device__ __forceinline__ void bm_apply_smem(int kind, uint4* top, uint4* below, const uint4* s) {
#pragma unroll
    for (int h = 0; h < kEvalU4PerThread; h++) {
        int i = threadIdx.x + h * kEvalThreads;
        uint4 x = s[i];
        switch (kind) {
            case K_PUSH: top[i] = x; break;
            case K_OR: top[i] = or4(top[i], x); break;
            case K_AND: top[i] = and4(top[i], x); break;
            case K_ANDNOT: top[i] = andn4(top[i], x); break;
            case K_XOR: top[i] = xor4(top[i], x); break;
            case K_ORAND: below[i] = or4(below[i], and4(top[i], x)); break;
            default: below[i] = or4(below[i], andn4(top[i], x)); break;
        }
    }
}

template <int MODE>   // 0: |=   1: &= ~   2: ^=
__device__ __forceinline__ void smem_bit_op(uint32_t* bm, uint32_t v) {
    // red.shared (no return value).  `asm volatile` keeps the reductions in program order, which stops ptxas from
    // hoisting dozens of address/mask computations ahead of them (register pressure decides CTA residency here).
    uint32_t addr = (uint32_t)__cvta_generic_to_shared(bm + (v >> 5));
    uint32_t m = 1u << (v & 31);
    if (MODE == 0) asm volatile("red.shared.or.b32 [%0], %1;" :: "r"(addr), "r"(m) : "memory");
    else if (MODE == 1) asm volatile("red.shared.and.b32 [%0], %1;" :: "r"(addr), "r"(~m) : "memory");
    else asm volatile("red.shared.xor.b32 [%0], %1;" :: "r"(addr), "r"(m) : "memory");
}
// one warp applies a whole bitmap container with word atomics (safe against concurrent warps)
template <int MODE>
__device__ __forceinline__ void warp_bitmap_atomic(uint32_t* bm, const uint4* g, int lane) {
    // no "skip zero words" test: a stored bitmap container has >= 4096 bits, so few words are zero, and the test compiled to a
    // branch + reconvergence pair around every reduction (4 instructions per word instead of 1)
    for (int i = lane; i < 512; i += 32) {
        uint4 v = ldg_nc(g + i);
        uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
        for (int q = 0; q < 4; q++) {
            if (MODE == 0) atomicOr(&bm[4 * i + q], w[q]); else if (MODE == 1) atomicAnd(&bm[4 * i + q], ~w[q]); else atomicXor(&bm[4 * i + q], w[q]);
        }
    }
}
// same reduction with the word's byte offset and the bit index given separately (sh: only its low 5 bits are used)
template <int MODE>
__device__ __forceinline__ void smem_bit_op_at(uint32_t addr, uint32_t sh) {
    const uint32_t m = 1u << (sh & 31);
    if (MODE == 0) asm volatile("red.shared.or.b32 [%0], %1;" :: "r"(addr), "r"(m) : "memory");
    else if (MODE == 1) asm volatile("red.shared.and.b32 [%0], %1;" :: "r"(addr), "r"(~m) : "memory");
    else asm volatile("red.shared.xor.b32 [%0], %1;" :: "r"(addr), "r"(m) : "memory");
}
// scatter the (up to) 8 elements of one 16-byte array chunk; sb = shared-space address of the target bitmap
template <int MODE>
__device__ __forceinline__ void scatter_chunk_sb(uint32_t sb, uint4 v, uint32_t base, uint32_t n) {
    uint32_t w[4] = { v.x, v.y, v.z, v.w };
    // OR / AND-NOT: the loader pads the last chunk with copies of the last element (stripe.h pad_array_tail), setting or
    // clearing a bit twice is harmless, so every chunk takes the unguarded path and the warp never diverges on a tail
    if (MODE != 2 || base + 8 <= n) {
#pragma unroll
        for (int q = 0; q < 4; q++) {            // LOP3 + LEA.HI + SHF.L.W (+ SHF.R for the upper element) + ATOMS, see bitaddr.h
            smem_bit_op_at<MODE>(word_addr_lo(sb, w[q]), w[q]);
            smem_bit_op_at<MODE>(word_addr_hi(sb, w[q]), w[q] >> 16);
        }
    } else {
#pragma unroll
        for (int q = 0; q < 4; q++) {
            if (base + 2 * q < n) smem_bit_op_at<MODE>(word_addr_lo(sb, w[q]), w[q]);
            if (base + 2 * q + 1 < n) smem_bit_op_at<MODE>(word_addr_hi(sb, w[q]), w[q] >> 16);
        }
    }
}
template <int MODE>
__device__ __forceinline__ void scatter_chunk_unrolled(uint32_t* bm, uint4 v, uint32_t base, uint32_t n) {
    scatter_chunk_sb<MODE>((uint32_t)__cvta_generic_to_shared(bm), v, base, n);
}
// Batch of commuting row operands (OR / ANDNOT / XOR onto the same target), no barrier in between: warp w takes
// operands w, w+8, ...; arrays are scattered with red.shared, bitmaps applied with word atomics.  (Tried and slower:
// 4 loads in flight per thread, register double-buffering, L2 prefetch, TMA staging.)
static_assert(sizeof(Resolved) == 16, "batch_rows reads a Resolved with one 16-byte shared load");
constexpr int kEvalDeep = 3;
template <int MODE>
__device__ __forceinline__ void batch_rows(uint32_t* T32, const Resolved* res, int n) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t sb = (uint32_t)__cvta_generic_to_shared(T32);
    pin_base(sb);                          // keep the shared address live: ptxas otherwise rebuilds it for every chunk
    for (int j = wid; j < n; j += kEvalThreads / 32) {
        const uint4 raw = *reinterpret_cast<const uint4*>(res + j);        // one LDS.128: {ptr lo, ptr hi, card, typ | cnt << 16}
        const uint4* a4 = reinterpret_cast<const uint4*>(((unsigned long long)raw.y << 32) | raw.x);
        if (a4 == nullptr) continue;
        const uint32_t typ = raw.w & 0xffffu;
        if (typ == kArray) {
            const uint32_t card = raw.z, n8 = (card + 7) >> 3;
            // the first kEvalDeep chunks of the lane are all in flight before the first reduction is issued: a ~650-element
            // container is 82 chunks = at most 3 per lane, so its whole payload costs the warp ONE exposed HBM latency instead of
            // three (most stall samples of the old one-chunk loop sat on its single load)
            // (the loads are unconditional — index clamped to the last chunk — so that no register of v[] is ever undefined:
            // predicated loads made ptxas park the chunks in local memory)
            uint4 v[kEvalDeep];
#pragma unroll
            for (int q = 0; q < kEvalDeep; q++) v[q] = ldg_nc(a4 + min((uint32_t)lane + 32u * q, n8 - 1u));
#pragma unroll
            for (int q = 0; q < kEvalDeep; q++) if (lane + 32 * q < n8) scatter_chunk_sb<MODE>(sb, v[q], (lane + 32 * q) * 8, card);
            for (uint32_t i = lane + 32 * kEvalDeep; i < n8; i += 32) scatter_chunk_sb<MODE>(sb, ldg_nc(a4 + i), i * 8, card);
        } else if (typ == kBitmap) warp_bitmap_atomic<MODE>(T32, a4, lane);
    }
}
// ------------------------------------------------------------------------------------------------
// Fused Count + sum all-reduce over NVLink peer memory (replaces the separate NCCL launch for the 8-byte Count
// merge, executor.go:5880-5883): every rank owns a Mailbox in its HBM that all peers map through CUDA IPC.  The last
// CTA of the counting kernel (atomic ticket) stores this rank's total into every peer's mailbox, publishes it with
// an epoch flag (system-scope fences), then waits for the peers' flags and sums.  Slots are double-buffered by
// epoch parity: a peer can only reach epoch e+2 after this rank has finished epoch e (it needs our e+1 value).
// ------------------------------------------------------------------------------------------------
constexpr int kMaxRanks = 16;
struct Mailbox { unsigned long long value[2][kMaxRanks]; unsigned long long flag[2][kMaxRanks]; };
struct FuseReduce {
    Mailbox* const* peers;          // device array [n_ranks]; peers[rank] is this rank's own mailbox; nullptr => fusion off
    unsigned int* ticket;           // completion counter of the launch (zeroed by the host)
    unsigned long long* result;     // receives the reduced total
    unsigned int* error;            // set to 1 + the rank that never published (bounded wait); zeroed by the host
    unsigned long long epoch;
    long long timeout_cycles;       // bound of the wait for one peer, in SM clock cycles
    int rank, n_ranks;
};
// called by ONE thread per CTA (or per warp) after its atomicAdd into *total; n_callers = how many will call
__device__ __forceinline__ void fused_allreduce_tail(const FuseReduce& fr, unsigned long long* total, unsigned int n_callers) {
    if (fr.peers == nullptr) return;
    __threadfence();
    if (atomicAdd(fr.ticket, 1u) != n_callers - 1) return;
    __threadfence();
    const unsigned long long mine = *reinterpret_cast<volatile unsigned long long*>(total);
    const int par = (int)(fr.epoch & 1ull);
    for (int p = 0; p < fr.n_ranks; p++) *reinterpret_cast<volatile unsigned long long*>(&fr.peers[p]->value[par][fr.rank]) = mine;
    __threadfence_system();
    for (int p = 0; p < fr.n_ranks; p++) *reinterpret_cast<volatile unsigned long long*>(&fr.peers[p]->flag[par][fr.rank]) = fr.epoch;
    __threadfence_system();
    Mailbox* me = fr.peers[fr.rank];
    unsigned long long sum = 0;
    for (int q = 0; q < fr.n_ranks; q++) {
        // exact match: a slot of this parity holds e-2 (or 0) until the peer publishes e; anything else is a protocol error and
        // runs into the same bound.  The wait is bounded: a dead or diverged peer must not hang the GPU (the host turns the
        // error word into FBGPU_E_COMM).
        const long long t0 = clock64();
        while (*reinterpret_cast<volatile unsigned long long*>(&me->flag[par][q]) != fr.epoch) {
            if (clock64() - t0 > fr.timeout_cycles) { *fr.error = 1u + (unsigned int)q; *fr.result = ~0ull; __threadfence_system(); return; }
        }
        __threadfence_system();
        sum += *reinterpret_cast<volatile unsigned long long*>(&me->value[par][q]);
    }
    *fr.result = sum;
}
// a rank with nothing to count still has to take part in the exchange
__global__ void p2p_reduce_only_kernel(FuseReduce fr, unsigned long long* total) { fused_allreduce_tail(fr, total, 1u); }

struct EvalOut {
    unsigned long long* total;      // += count of every unit (may be null)
    unsigned long long* per_shard;  // [n_shards] += (may be null)
    uint4* bitmaps;                 // [n_units][512] result bitmaps (may be null)
    uint2* info;                    // [n_units] {N, runs} (may be null)
    FuseReduce fr;                  // fused cross-GPU reduce of `total` (fr.peers == nullptr => off)
};

// One CTA per (shard, slot) unit, persistent over units.  Dynamic smem: (depth+1) x 8 KiB.
__global__ void __launch_bounds__(kEvalThreads, kEvalMinBlocks)
eval_kernel(StoreRef st, const DevOp* __restrict__ prog, int n_ops, int depth,
            const int2* __restrict__ batches, int n_batches,
            const uint64_t* __restrict__ shards, long long n_units, EvalOut out) {
    extern __shared__ uint4 smem4[];
    __shared__ __align__(16) Resolved res[kResolveChunk];
    __shared__ uint32_t warp_tmp[kEvalThreads / 32];
    __shared__ uint32_t warp_tmp2[kEvalThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    unsigned long long cta_total = 0;

    for (long long unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
        const uint64_t shard = shards[unit >> 4];
        const int slot = (int)(unit & 15);
        // nibble-packed permutation level -> physical bitmap; levels > top are free, index `depth` is the spare
        uint64_t map = 0xFEDCBA9876543210ull;
        int top = -1;
        auto phys = [&](int level) -> uint4* { return smem4 + (size_t)((map >> (4 * level)) & 15u) * 512; };
        auto swap_levels = [&](int a, int b) {
            uint64_t pa = (map >> (4 * a)) & 15u, pb = (map >> (4 * b)) & 15u;
            map &= ~((15ull << (4 * a)) | (15ull << (4 * b)));
            map |= (pb << (4 * a)) | (pa << (4 * b));
        };
        int cur_batch = 0;
        for (int base = 0; base < n_ops; base += kResolveChunk) {
            int chunk = min(kResolveChunk, n_ops - base);
            __syncthreads();
            bool is_run = false;
            if (tid < chunk) {
                DevOp op = prog[base + tid];
                Resolved r; r.ptr = nullptr; r.card = 0; r.typ = 0; r.cnt = 0;
                if (op.op >= D_PUSH_ROW && op.op <= D_ORANDNOT_ROW && op.op != D_PUSH_EMPTY) r = resolve(st, op.fv, shard, op.row, slot);
                res[tid] = r;
                is_run = r.ptr != nullptr && r.typ == kRun;
            }
            const int has_runs = __syncthreads_or(is_run);
            for (int k = 0; k < chunk; k++) {
                const uint8_t opc = prog[base + k].op;
                if (opc == D_PUSH_EMPTY) { top++; bm_zero(phys(top)); __syncthreads(); continue; }
                if (opc == D_SWAP) { swap_levels(top, top - 1); continue; }
                if (opc == D_POP) { top--; continue; }
                if (opc >= D_AND && opc <= D_XOR) {
                    int kind = opc == D_AND ? K_AND : opc == D_OR ? K_OR : opc == D_ANDNOT ? K_ANDNOT : K_XOR;
                    bm_apply_smem(kind, phys(top - 1), nullptr, phys(top));
                    top--; __syncthreads(); continue;
                }
                if (opc == D_OR_ROW || opc == D_ANDNOT_ROW || opc == D_XOR_ROW) {
                    // extent of this batch (host-computed runs of the same commuting row op), clipped to the chunk
                    while (cur_batch < n_batches && batches[cur_batch].y <= base + k) cur_batch++;
                    const int e = min(cur_batch < n_batches ? batches[cur_batch].y - base : k + 1, chunk);
                    uint4* T = phys(top);
                    uint32_t* T32 = reinterpret_cast<uint32_t*>(T);
                    if (opc == D_OR_ROW) batch_rows<0>(T32, res + k, e - k);
                    else if (opc == D_ANDNOT_ROW) batch_rows<1>(T32, res + k, e - k);
                    else batch_rows<2>(T32, res + k, e - k);
                    __syncthreads();
                    if (has_runs) for (int j = k; j < e; j++) {   // run containers: CTA-wide expansion, one at a time
                        const Resolved r = res[j];
                        if (r.ptr == nullptr || r.typ != kRun) continue;
                        uint4* S = phys(depth);
                        bm_expand_runs(S, reinterpret_cast<const uint16_t*>(r.ptr), r.cnt, warp_tmp);
                        bm_apply_smem(opc == D_OR_ROW ? K_OR : opc == D_ANDNOT_ROW ? K_ANDNOT : K_XOR, T, nullptr, S);
                        __syncthreads();
                    }
                    k = e - 1;
                    continue;
                }
                // row-operand ops
                int kind = opc == D_PUSH_ROW ? K_PUSH : opc == D_OR_ROW ? K_OR : opc == D_AND_ROW ? K_AND : opc == D_ANDNOT_ROW ? K_ANDNOT
                         : opc == D_XOR_ROW ? K_XOR : opc == D_ORAND_ROW ? K_ORAND : K_ORANDNOT;
                const Resolved r = res[k];
                if (kind == K_PUSH) top++;
                uint4* T = phys(top);
                uint4* B = (kind == K_ORAND || kind == K_ORANDNOT) ? phys(top - 1) : nullptr;
                if (r.ptr == nullptr) {                      // absent container == empty (container_stash.go:38)
                    if (kind == K_PUSH || kind == K_AND) bm_zero(T);
                    else if (kind == K_ORANDNOT) bm_apply_smem(K_OR, B, nullptr, T);
                    __syncthreads();
                } else if (r.typ == kBitmap) {
                    bm_apply_global(kind, T, B, reinterpret_cast<const uint4*>(r.ptr));
                    __syncthreads();
                } else if (r.typ == kArray) {
                    const uint16_t* arr = reinterpret_cast<const uint16_t*>(r.ptr);
                    uint32_t* T32 = reinterpret_cast<uint32_t*>(T);
                    if (kind == K_PUSH) { bm_zero(T); __syncthreads(); bm_scatter<0>(T32, arr, r.card); }
                    else if (kind == K_OR) bm_scatter<0>(T32, arr, r.card);
                    else if (kind == K_ANDNOT) bm_scatter<1>(T32, arr, r.card);
                    else if (kind == K_XOR) bm_scatter<2>(T32, arr, r.card);
                    else if (kind == K_ORAND) bm_filter_scatter(reinterpret_cast<uint32_t*>(B), T32, arr, r.card);
                    else if (kind == K_AND) {
                        uint4* S = phys(depth);
                        bm_zero(S); __syncthreads();
                        bm_filter_scatter(reinterpret_cast<uint32_t*>(S), T32, arr, r.card);
                        swap_levels(top, depth);
                    } else {  // K_ORANDNOT
                        uint4* S = phys(depth);
                        bm_zero(S); __syncthreads();
                        bm_scatter<0>(reinterpret_cast<uint32_t*>(S), arr, r.card); __syncthreads();
                        bm_apply_smem(K_ORANDNOT, T, B, S);
                    }
                    __syncthreads();
                } else {                                     // run container
                    const uint16_t* runs = reinterpret_cast<const uint16_t*>(r.ptr);
                    if (kind == K_PUSH) bm_expand_runs(T, runs, r.cnt, warp_tmp);
                    else {
                        uint4* S = phys(depth);
                        bm_expand_runs(S, runs, r.cnt, warp_tmp);
                        bm_apply_smem(kind, T, B, S);
                        __syncthreads();
                    }
                }
            }
        }
        // ---- unit epilogue: popcount (+ optional bitmap / run statistics for canonical emission)
        uint32_t cnt = 0, nruns = 0;
        if (top >= 0) {
            const uint4* R = phys(top);
            const uint64_t* R64 = reinterpret_cast<const uint64_t*>(R);
#pragma unroll
            for (int h = 0; h < kEvalU4PerThread; h++) {
                int i = tid + h * kEvalThreads;
                uint4 a = R[i];
                cnt += popc4(a);
                if (out.bitmaps) out.bitmaps[(size_t)unit * 512 + i] = a;
                if (out.info) {
#pragma unroll
                    for (int q = 0; q < 2; q++) {
                        int wi = 2 * i + q;
                        uint64_t v = R64[wi];
                        uint64_t prev = wi ? (R64[wi - 1] >> 63) : 0ull;
                        nruns += __popcll(v & ~((v << 1) | prev));   // bitmapCountRuns roaring.go:3372
                    }
                }
            }
        } else if (out.bitmaps) {
#pragma unroll
            for (int h = 0; h < kEvalU4PerThread; h++) out.bitmaps[(size_t)unit * 512 + tid + h * kEvalThreads] = make_uint4(0, 0, 0, 0);
        }
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        nruns = __reduce_add_sync(0xffffffffu, nruns);
        __syncthreads();
        if (lane == 0) { warp_tmp[wid] = cnt; warp_tmp2[wid] = nruns; }
        __syncthreads();
        if (tid == 0) {
            uint32_t c = 0, rr = 0;
#pragma unroll
            for (int k = 0; k < kEvalThreads / 32; k++) { c += warp_tmp[k]; rr += warp_tmp2[k]; }
            cta_total += c;
            if (out.per_shard && c) atomicAdd(&out.per_shard[unit >> 4], (unsigned long long)c);
            if (out.info) out.info[unit] = make_uint2(c, rr);
        }
    }
    if (tid == 0 && out.total) { if (cta_total) atomicAdd(out.total, cta_total); fused_allreduce_tail(out.fr, out.total, gridDim.x); }
}

// ------------------------------------------------------------------------------------------------
// eval_wordpar_kernel: word-parallel evaluation for bitmap-heavy programs (BSI plane sweeps, dense rows).
// Every thread owns 32 bytes (two adjacent 128-bit slices) of a (shard, slot) stripe and runs the whole program on them with the
// operand stack in registers (wp_machine.h): no shared-memory bitmaps and no barriers between ops.  Arrays and runs are handled by
// a per-thread search for the slice's elements, so any program is valid here; the host only picks this kernel when the referenced
// views are dominated by bitmap/run containers.
// ------------------------------------------------------------------------------------------------
// 32 bytes per thread in CTAs of 64 threads rather than 16 bytes in CTAs of 128: the same 2 KiB per CTA and row op, but the program
// loop's per-op overhead (ring bookkeeping, op decode, branches: ~32 of the ~36 instructions per op and thread; the 16-byte form issued
// 43 % of its cycles with DRAM 30 % busy) is paid once per 32 bytes.
constexpr int kWpThreads = 64;
constexpr int kWpBlocksPerUnit = 512 / (kWpThreads * 2);       // CTAs per (shard, slot) unit
constexpr int kWpMinBlocks = 8;
struct __align__(16) WpV32 { unsigned long long x, y, z, w; };      // 32 bytes of a stripe; member-wise bit ops (wp_machine.h)
constexpr int kWpMaxOps = 256;
constexpr int kWpMaxDepth = 4;

__device__ __forceinline__ uint4 wp_slice(const Resolved& r, int i) {
    if (r.ptr == nullptr) return make_uint4(0, 0, 0, 0);
    if (r.typ == kBitmap) return ldg_nc(reinterpret_cast<const uint4*>(r.ptr) + i);
    const uint32_t lo = (uint32_t)i * 128u, hi = lo + 127u;       // value range of this slice
    uint32_t w[4] = { 0, 0, 0, 0 };
    if (r.typ == kArray) {
        const uint16_t* a = reinterpret_cast<const uint16_t*>(r.ptr);
        uint32_t l = 0, h = r.card;
        while (l < h) { uint32_t m = (l + h) >> 1; if (__ldg(a + m) < lo) l = m + 1; else h = m; }
        for (; l < r.card; l++) { uint32_t v = __ldg(a + l); if (v > hi) break; v -= lo; w[v >> 5] |= 1u << (v & 31); }
    } else {
        const uint32_t* rr = reinterpret_cast<const uint32_t*>(r.ptr);
        uint32_t l = 0, h = r.cnt;                                  // first run with last >= lo
        while (l < h) { uint32_t m = (l + h) >> 1; if ((__ldg(rr + m) >> 16) < lo) l = m + 1; else h = m; }
        for (; l < r.cnt; l++) {
            uint32_t v = __ldg(rr + l); uint32_t s0 = v & 0xffffu, l0 = v >> 16;
            if (s0 > hi) break;
            uint32_t a0 = max(s0, lo) - lo, b0 = min(l0, hi) - lo;  // inclusive bit range inside the slice
#pragma unroll
            for (int q = 0; q < 4; q++) {
                uint32_t qa = q * 32, qb = qa + 31;
                if (b0 < qa || a0 > qb) continue;
                uint32_t x = max(a0, qa) - qa, y = min(b0, qb) - qa;
                w[q] |= (0xffffffffu << x) & (0xffffffffu >> (31 - y));
            }
        }
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
}

struct WpOp { const void* ptr; uint32_t card; uint16_t typ, cnt; uint8_t opc, is_row, pad[6]; };   // pre-decoded op, 24 B

// Operand ring in shared memory, filled by cp.async (LDGSTS): every thread copies ITS 32 bytes of the next kWpAsyncDepth - 1 row
// operands into its own ring slots — no registers and no scoreboard entry per load in flight (a register ring stalled on shared
// scoreboards beyond 3 loads: depth 6 was slower than depth 3 on BASELINE config 3), no barrier (a slot is written and read by the
// same thread), and the depth is a shared-memory size, not a register count.  One commit group per row op, empty when the operand
// is absent or not a bitmap (its slice is computed into the slot right away), so that `wait_group depth - 1` at row op ri always
// means "group ri has landed".
constexpr int kWpAsyncDepth = 8;       // ring slots per thread: depth - 1 operand slices in flight
__device__ __forceinline__ void cp_async_16(uint4* dst_smem, const uint4* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"((uint32_t)__cvta_generic_to_shared(dst_smem)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait_group() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

__global__ void __launch_bounds__(kWpThreads, kWpMinBlocks)
eval_wordpar_kernel(StoreRef st, const DevOp* __restrict__ prog, int n_ops,
                    const uint64_t* __restrict__ shards, long long n_units, EvalOut out) {
    __shared__ WpOp ops[kWpMaxOps];
    __shared__ uint16_t rowops[kWpMaxOps];     // indices of the row ops, in program order
    __shared__ int n_rowops;
    __shared__ uint32_t wsum[kWpThreads / 32];
    __shared__ __align__(16) WpV32 wp_ring[kWpAsyncDepth][kWpThreads];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const long long n_blocks = n_units * kWpBlocksPerUnit;
    for (long long blk = blockIdx.x; blk < n_blocks; blk += gridDim.x) {
        const long long unit = blk / kWpBlocksPerUnit;
        const int i0 = (int)(blk % kWpBlocksPerUnit) * kWpThreads * 2 + 2 * tid;       // the thread's two adjacent uint4 slices: i0, i0 + 1
        __syncthreads();
        for (int k = tid; k < n_ops; k += kWpThreads) {        // decode + resolve: one op per thread
            DevOp op = prog[k];
            Resolved r; r.ptr = nullptr; r.card = 0; r.typ = 0; r.cnt = 0;
            const bool row_op = op.op >= D_PUSH_ROW && op.op <= D_ORANDNOT_ROW && op.op != D_PUSH_EMPTY;
            if (row_op) r = resolve(st, op.fv, shards[unit >> 4], op.row, (int)(unit & 15));
            WpOp w; w.ptr = r.ptr; w.card = r.card; w.typ = r.typ; w.cnt = r.cnt; w.opc = op.op; w.is_row = row_op ? 1 : 0;
            ops[k] = w;
        }
        __syncthreads();
        if (wid == 0) {                        // positions of the row ops: ballot scan, 32 ops per step (was a serial loop of one thread)
            int n = 0;
            for (int base = 0; base < n_ops; base += 32) {
                const int k = base + lane;
                const bool is = k < n_ops && ops[k].is_row != 0;
                const unsigned m = __ballot_sync(0xffffffffu, is);
                if (is) rowops[n + __popc(m & ((1u << lane) - 1u))] = (uint16_t)k;
                n += __popc(m);
            }
            if (lane == 0) n_rowops = n;
        }
        __syncthreads();
        const int nr = n_rowops;
        auto issue = [&](int ri) {
            if (ri < nr) {
                const WpOp w = ops[rowops[ri]];
                uint4* slot = reinterpret_cast<uint4*>(&wp_ring[ri % kWpAsyncDepth][tid]);
                if (w.ptr != nullptr && w.typ == kBitmap) { const uint4* g = reinterpret_cast<const uint4*>(w.ptr) + i0; cp_async_16(slot, g); cp_async_16(slot + 1, g + 1); }
                else { Resolved r; r.ptr = w.ptr; r.card = w.card; r.typ = w.typ; r.cnt = w.cnt; slot[0] = wp_slice(r, i0); slot[1] = wp_slice(r, i0 + 1); }
            }
            cp_async_commit();
        };
        for (int ri = 0; ri < kWpAsyncDepth - 1; ri++) issue(ri);
        const WpV32 T32 = wp_run_unrolled<WpV32, true, 1>(n_ops, nr, [&](int k) { return ops[k].opc; }, [&](int k) { return ops[k].is_row != 0; },
                                         [&](int ri) { return (int)rowops[ri]; },
                                         [&](int ri) {      // called once per row op, in order, after the previous operand has been consumed
                                             issue(ri + kWpAsyncDepth - 1);          // into the slot the previous row op was read from
                                             cp_async_wait_group<kWpAsyncDepth - 1>();
                                             return wp_ring[ri % kWpAsyncDepth][tid];
                                         });
        cp_async_wait_group<0>();
        uint4 T[2];
        T[0] = make_uint4((uint32_t)T32.x, (uint32_t)(T32.x >> 32), (uint32_t)T32.y, (uint32_t)(T32.y >> 32));
        T[1] = make_uint4((uint32_t)T32.z, (uint32_t)(T32.z >> 32), (uint32_t)T32.w, (uint32_t)(T32.w >> 32));
        uint32_t cnt = 0;
#pragma unroll
        for (int q = 0; q < 2; q++) {                   // (wp_run_unrolled already returns zero for an empty stack)
            if (out.bitmaps) out.bitmaps[(size_t)unit * 512 + i0 + q] = T[q];
            cnt += (uint32_t)popc4(T[q]);
        }
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (lane == 0) wsum[wid] = cnt;
        __syncthreads();
        if (tid == 0) {
            uint32_t c = 0;
#pragma unroll
            for (int q = 0; q < kWpThreads / 32; q++) c += wsum[q];
            if (c) { if (out.total) atomicAdd(out.total, (unsigned long long)c); if (out.per_shard) atomicAdd(&out.per_shard[unit >> 4], (unsigned long long)c); }
        }
    }
    if (tid == 0 && out.total) fused_allreduce_tail(out.fr, out.total, gridDim.x);
}

// ------------------------------------------------------------------------------------------------
// Warp-level intersection count of two located containers; `bm` is the warp's private 8 KiB smem bitmap.
// Follows the dispatch of intersectionCount (roaring.go:4477-4512) incl. the full/empty short-circuits.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr)); return v; }
// per-lane partial count of array elements found in a shared-memory bitmap
__device__ __forceinline__ uint32_t warp_probe_smem(const uint32_t* bm, const uint16_t* arr, uint32_t n, int lane) {
    const uint4* a4 = reinterpret_cast<const uint4*>(arr);
    uint32_t n8 = (n + 7) >> 3, c = 0;
    for (uint32_t i = lane; i < n8; i += 32) {
        uint4 v = ldg_nc(a4 + i);
        uint32_t w[4] = { v.x, v.y, v.z, v.w };
        uint32_t base = i * 8;
#pragma unroll
        for (int q = 0; q < 4; q++) {
            uint32_t lo = w[q] & 0xffffu, hi = w[q] >> 16;
            if (base + 2 * q < n) c += (bm[lo >> 5] >> (lo & 31)) & 1u;
            if (base + 2 * q + 1 < n) c += (bm[hi >> 5] >> (hi & 31)) & 1u;
        }
    }
    return c;
}
// per-lane partial count of array elements found in a global-memory bitmap: 16-byte element loads, then the eight
// word probes of a chunk are issued back to back (independent loads in flight)
__device__ __forceinline__ uint32_t warp_probe_global(const uint32_t* g, const uint16_t* arr, uint32_t n, int lane) {
    const uint4* a4 = reinterpret_cast<const uint4*>(arr);
    const uint32_t n8 = (n + 7) >> 3;
    uint32_t c = 0;
    for (uint32_t i = lane; i < n8; i += 32) {
        uint4 v = ldg_nc(a4 + i);
        uint32_t e[8] = { v.x & 0xffffu, v.x >> 16, v.y & 0xffffu, v.y >> 16, v.z & 0xffffu, v.z >> 16, v.w & 0xffffu, v.w >> 16 };
        uint32_t w[8];
        const uint32_t base = i * 8;
#pragma unroll
        for (int q = 0; q < 8; q++) w[q] = (base + q < n) ? __ldg(g + (e[q] >> 5)) : 0u;
#pragma unroll
        for (int q = 0; q < 8; q++) c += (w[q] >> (e[q] & 31)) & 1u;
    }
    return c;
}
// per-lane partial: |bitmap(global) ∩ smem bitmap|
__device__ __forceinline__ uint32_t warp_and_count_gs(const uint4* g, const uint32_t* bm, int lane) {
    const uint4* s4 = reinterpret_cast<const uint4*>(bm);
    uint32_t c = 0;
#pragma unroll 4
    for (int i = lane; i < 512; i += 32) c += popc4(and4(ldg_nc(g + i), s4[i]));
    return c;
}
// per-lane partial: number of set bits of a u32-word bitmap (smem or global) inside [s, l]
__device__ __forceinline__ uint32_t range_count32(const uint32_t* bm, uint32_t s, uint32_t l) {
    uint32_t ws = s >> 5, wl = l >> 5;
    uint32_t ms = 0xffffffffu << (s & 31), ml = 0xffffffffu >> (31 - (l & 31));
    if (ws == wl) return __popc(bm[ws] & ms & ml);
    uint32_t c = __popc(bm[ws] & ms) + __popc(bm[wl] & ml);
    for (uint32_t k = ws + 1; k < wl; k++) c += __popc(bm[k]);
    return c;
}

// shared-memory store of a zero word / probe of one bit at an absolute shared address
__device__ __forceinline__ void sts_zero(uint32_t addr) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(addr), "r"(0u) : "memory"); }
__device__ __forceinline__ void red_or_at(uint32_t addr, uint32_t m) { asm volatile("red.shared.or.b32 [%0], %1;" :: "r"(addr), "r"(m) : "memory"); }
__device__ __forceinline__ uint2 ldg_nc64(const uint2* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
constexpr int kPairWarps = 8;           // row_count_kernel
constexpr int kPcWarps = 8;                                 // warps per CTA of pair_count_kernel, one 8 KiB bitmap each; 3 CTAs per SM (8 warps measured faster than 9)
constexpr int kPcMinBlocks = 3;
constexpr int kPcPairSlots = 256;                           // row pairs per launch whose counts are summed in shared memory first
constexpr int kPcPfDist = 1;                                // how many units ahead the payload lines are prefetched into L2
constexpr int kPcBmUnroll = 8;                              // bitmap x bitmap: pairs of 16-byte loads in flight per lane
constexpr uint32_t kPcFastCard = 768;                       // arrays up to this size take the register-window path (3 chunks per lane)

// Pairs with a run container on at least one side; returns the per-lane partial count.  The searched interval list (<= 2048 runs =
// 8 KiB) is first copied into the warp's shared-memory words, so the per-element / per-run binary searches are ~30-cycle shared-memory
// loads instead of dependent global loads (in global memory, run x run at 20 % clustered density spent six rounds of an eight-deep chain
// of L2 round trips per warp and pair; the shared-memory copy halved its time); the words are zeroed again before returning.
__device__ __noinline__ uint32_t warp_icount_runs(Resolved a, Resolved b, uint32_t* bm, int lane) {
    uint32_t c = 0;
    if (a.typ == kRun && b.typ != kRun) { Resolved t = a; a = b; b = t; }   // make `b` a run side
    if (a.typ == kBitmap) {                                   // bitmap x run: roaring.go:4588 (sum of BitmapCountRange per run), global words
        const uint32_t* g = reinterpret_cast<const uint32_t*>(a.ptr);
        const uint32_t* r32 = reinterpret_cast<const uint32_t*>(b.ptr);
        if (b.cnt >= 32) {                                    // many short runs: one lane per run
            for (uint32_t i = lane; i < b.cnt; i += 32) { uint32_t v = __ldg(r32 + i); c += range_count32(g, v & 0xffffu, v >> 16); }
        } else {                                              // few long runs: the warp walks each run's words together
            for (uint32_t i = 0; i < b.cnt; i++) {
                uint32_t v = __ldg(r32 + i); uint32_t s0 = v & 0xffffu, l0 = v >> 16;
                for (uint32_t w = (s0 >> 5) + lane; w <= (l0 >> 5); w += 32) {
                    uint32_t m = 0xffffffffu;
                    if (w == (s0 >> 5)) m &= 0xffffffffu << (s0 & 31);
                    if (w == (l0 >> 5)) m &= 0xffffffffu >> (31 - (l0 & 31));
                    c += __popc(__ldg(g + w) & m);
                }
            }
        }
        return c;
    }
    if (a.typ == kRun && a.cnt > b.cnt) { Resolved t = a; a = b; b = t; }   // run x run: search the longer list
    const uint32_t* rb = reinterpret_cast<const uint32_t*>(b.ptr);
    // (stored fragments hold at most 2048 runs per container — optimize() turns longer lists into bitmaps — but a hand-built
    // container may carry up to 32768: those are searched where they are, in global memory)
    const bool staged = b.cnt <= 2048u;
    if (staged) { for (uint32_t i = lane; i < b.cnt; i += 32) bm[i] = __ldg(rb + i); }
    __syncwarp();
    auto run_at = [&](uint32_t m) { return staged ? bm[m] : __ldg(rb + m); };
    if (a.typ == kArray) {                                    // array x run: roaring.go:4537
        const uint16_t* arr = reinterpret_cast<const uint16_t*>(a.ptr);
        for (uint32_t i = lane; i < a.card; i += 32) {
            const uint32_t v = __ldg(arr + i);
            uint32_t lo = 0, hi = b.cnt;                      // first run with last >= v
            while (lo < hi) { uint32_t m = (lo + hi) >> 1; if ((run_at(m) >> 16) < v) lo = m + 1; else hi = m; }
            if (lo < b.cnt) c += ((run_at(lo) & 0xffffu) <= v);
        }
    } else {                                                  // run x run: interval overlap, roaring.go:4555
        const uint32_t* ra = reinterpret_cast<const uint32_t*>(a.ptr);
        for (uint32_t i = lane; i < a.cnt; i += 32) {
            const uint32_t v = __ldg(ra + i); const uint32_t s0 = v & 0xffffu, l0 = v >> 16;
            uint32_t lo = 0, hi = b.cnt;                      // first run of b with last >= s0
            while (lo < hi) { uint32_t m = (lo + hi) >> 1; if ((run_at(m) >> 16) < s0) lo = m + 1; else hi = m; }
            for (; lo < b.cnt; lo++) {
                const uint32_t u = run_at(lo); const uint32_t s1 = u & 0xffffu, l1 = u >> 16;
                if (s1 > l0) break;
                c += min(l0, l1) - max(s0, s1) + 1;
            }
        }
    }
    __syncwarp();
    if (staged) { for (uint32_t i = lane; i < b.cnt; i += 32) bm[i] = 0; }
    __syncwarp();
    return c;
}

// Every pair that is not two arrays of at most kPcFastCard elements (kept out of line: the hot path is the inline code of the kernel).
// Follows the dispatch of intersectionCount (roaring.go:4477-4512) incl. the full/empty short-circuits.  `bm` is all zero on entry
// and on exit.  Returns the count (reduced over the warp, valid in all lanes).
__device__ __noinline__ uint32_t warp_intersection_count_generic(Resolved a, Resolved b, uint32_t* bm, int lane) {
    if (a.ptr == nullptr || b.ptr == nullptr) return 0;
    if (a.card == kFull) return b.card;                       // roaring.go:4478-4483
    if (b.card == kFull) return a.card;
    if (a.typ != kArray && b.typ == kArray) { Resolved t = a; a = b; b = t; }      // arrays first
    uint32_t c = 0;
    if (a.typ == kRun || b.typ == kRun) c = warp_icount_runs(a, b, bm, lane);
    else if (a.typ == kArray && b.typ == kArray) {            // long arrays (> kPcFastCard): scatter the smaller, probe the larger, chunk by chunk
        if (a.card > b.card) { Resolved t = a; a = b; b = t; }
        const uint4* a4 = reinterpret_cast<const uint4*>(a.ptr); const uint4* b4 = reinterpret_cast<const uint4*>(b.ptr);
        const uint32_t na8 = (a.card + 7) >> 3, nb8 = (b.card + 7) >> 3;
        const uint32_t sb = (uint32_t)__cvta_generic_to_shared(bm);
        for (uint32_t i = lane; i < na8; i += 32) scatter_chunk_sb<0>(sb, ldg_nc(a4 + i), i * 8, a.card);
        __syncwarp();
        for (uint32_t i = lane; i < nb8; i += 32) {           // whole chunks: the pad copies of b's last element are taken out below
            const uint4 v = ldg_nc(b4 + i); const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
            for (int q = 0; q < 4; q++) {
                c += (lds_u32(word_addr_lo(sb, w[q])) >> (w[q] & 31)) & 1u;
                c += (lds_u32(word_addr_hi(sb, w[q])) >> ((w[q] >> 16) & 31)) & 1u;
            }
        }
        const uint32_t pads = nb8 * 8u - b.card;
        if (pads && lane == 0) { const uint32_t last = __ldg(reinterpret_cast<const uint16_t*>(b.ptr) + b.card - 1); c -= pads * ((bm[last >> 5] >> (last & 31)) & 1u); }
        __syncwarp();
        for (uint32_t i = lane; i < na8; i += 32) {
            const uint4 v = ldg_nc(a4 + i); const uint32_t x[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
            for (int k = 0; k < 4; k++) { sts_zero(word_addr_lo(sb, x[k])); sts_zero(word_addr_hi(sb, x[k])); }
        }
        __syncwarp();
    } else if (a.typ == kArray) {                             // array x bitmap: roaring.go:4596
        c = warp_probe_global(reinterpret_cast<const uint32_t*>(b.ptr), reinterpret_cast<const uint16_t*>(a.ptr), a.card, lane);
    } else {                                                  // bitmap x bitmap: roaring.go:4611
        const uint4* x = reinterpret_cast<const uint4*>(a.ptr); const uint4* y = reinterpret_cast<const uint4*>(b.ptr);
#pragma unroll kPcBmUnroll
        for (int i = lane; i < 512; i += 32) c += popc4(and4(ldg_nc(x + i), ldg_nc(y + i)));
    }
    return __reduce_add_sync(0xffffffffu, c);
}

// Count(Intersect(Row(fvA,rowA), Row(fvB,rowB))): one warp per (shard, slot) container pair, a warp-private 8 KiB bitmap in shared
// memory.  A warp owns the units w, w+W, w+2W, ...; it walks the descriptor chains of up to 16 of its units at once (lane 2k / 2k+1 =
// side a / b of unit k) and classifies them lane-parallel: for two arrays of at most 768 elements — the shape of the 1 % acceptance
// point — lane 2k ends up holding the SMALLER array (scattered), lane 2k+1 the larger (probed), so that the per-unit code has no
// dispatch left: six shuffles, six 16-byte loads per lane, scatter / probe / clear out of a register window.
// The path is bound by the integer ALU pipe (LOP3 / LEA / SHF), about half of whose instructions per pair are the scatter and probe
// arithmetic itself: every instruction that is not per-element work was taken out of the per-unit loop.
__global__ void __launch_bounds__(kPcWarps * 32, kPcMinBlocks)
pair_count_kernel(StoreRef st, uint32_t fvA, uint64_t rowA, uint32_t fvB, uint64_t rowB,
                  const uint64_t* __restrict__ rowsA, const uint64_t* __restrict__ rowsB, long long units_per_pair,
                  const uint64_t* __restrict__ shards, uint64_t shard0, long long n_units,
                  unsigned long long* total, unsigned long long* per_shard, unsigned long long* per_pair, FuseReduce fr) {
    extern __shared__ __align__(128) uint32_t smem32[];
    // per-pair counts of this CTA (multi-pair form): summed here and added to the global vector once per CTA and pair at the end —
    // one global atomicAdd per unit onto per_pair[pair] was ~16 k same-address atomics per pair and launch on one L2 slice
    __shared__ unsigned long long s_pair[kPcPairSlots];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const long long n_pairs = per_pair ? (n_units + units_per_pair - 1) / units_per_pair : 0;
    const bool pairs_in_smem = per_pair && n_pairs <= kPcPairSlots;
    if (pairs_in_smem) { for (int i = threadIdx.x; i < (int)n_pairs; i += blockDim.x) s_pair[i] = 0; __syncthreads(); }
    uint32_t* bm = smem32 + wid * 2048;
    {   uint4* b4 = reinterpret_cast<uint4*>(bm);          // the only full clear: every path leaves the bitmap all-zero again
#pragma unroll 4
        for (int i = lane; i < 512; i += 32) b4[i] = make_uint4(0, 0, 0, 0); }
    __syncwarp();
    uint32_t sb = (uint32_t)__cvta_generic_to_shared(bm);
    pin_base(sb);
    unsigned long long acc = 0, run_sum = 0;               // run_sum: count of the current pair index / shard, flushed when it changes
    long long run_key = -1;
    auto flush = [&]() {
        if (run_key >= 0 && run_sum && lane == 0) {
            if (pairs_in_smem) atomicAdd(&s_pair[run_key], run_sum);
            else if (per_pair) atomicAdd(&per_pair[run_key], run_sum);
            else atomicAdd(&per_shard[run_key], run_sum);
        }
        run_sum = 0;
    };
    const long long stride = (long long)gridDim.x * kPcWarps;
    for (long long base = (long long)blockIdx.x * kPcWarps + wid; base < n_units; base += stride * 16) {
        // ---- resolve up to 16 units of this warp concurrently
        // multi-pair form (rowsA != null): unit = pair * units_per_pair + (shard index * 16 + slot)
        const long long my_unit = base + (long long)(lane >> 1) * stride;
        Resolved r; r.ptr = nullptr; r.card = 0; r.typ = 0; r.cnt = 0;
        if (my_unit < n_units) {
            const long long pr = rowsA ? my_unit / units_per_pair : 0, su = rowsA ? my_unit - pr * units_per_pair : my_unit;
            // shards == nullptr: the caller's list is the contiguous range shard0, shard0 + 1, ... (one dependent load less)
            const uint64_t shard = shards ? shards[su >> 4] : shard0 + (uint64_t)(su >> 4);
            r = (lane & 1) ? resolve(st, fvB, shard, rowsA ? rowsB[pr] : rowB, (int)(su & 15))
                           : resolve(st, fvA, shard, rowsA ? rowsA[pr] : rowA, (int)(su & 15));
        }
        // ---- classify lane-parallel; for the fast class put the smaller array into the even lane
        const uint32_t meta = ((uint32_t)r.typ << 16) | r.cnt;
        unsigned long long my_ptr = (unsigned long long)r.ptr; uint32_t my_card = r.card;
        {
            const uint32_t o_card = __shfl_xor_sync(0xffffffffu, r.card, 1), o_meta = __shfl_xor_sync(0xffffffffu, meta, 1);
            const unsigned long long o_ptr = __shfl_xor_sync(0xffffffffu, my_ptr, 1);
            const bool fast = my_ptr != 0 && o_ptr != 0 && r.typ == kArray && (o_meta >> 16) == kArray && r.card <= kPcFastCard && o_card <= kPcFastCard;
            const bool absent = my_ptr == 0 || o_ptr == 0;
            const uint32_t even_card = (lane & 1) ? o_card : r.card, odd_card = (lane & 1) ? r.card : o_card;
            if (fast && even_card > odd_card) { my_ptr = o_ptr; my_card = o_card; }        // swap the two lanes' containers
            my_card |= fast ? (1u << 20) : absent ? 0u : (2u << 20);                          // bits 20..21: 0 absent, 1 fast, 2 generic
        }
        long long pr = per_pair ? base / units_per_pair : 0, pr_rem = per_pair ? base - pr * units_per_pair : 0;     // pair index of unit k, kept incrementally (one division per round)
        // lanes 0-11 / 16-27 prefetch one 128-byte line each of unit j's two containers (up to 1.5 KiB per side)
        auto prefetch_unit = [&](int j) {
            if (j < 16) {
                const unsigned long long np = __shfl_sync(0xffffffffu, my_ptr, 2 * j + (lane >> 4));
                if (np != 0 && (lane & 15) < 12) asm volatile("prefetch.global.L2 [%0];" :: "l"(np + (unsigned long long)(lane & 15) * 128ull));
            }
        };
#pragma unroll
        for (int j = 1; j < kPcPfDist; j++) prefetch_unit(j);
        const int n_k = (int)min((long long)16, (n_units - base + stride - 1) / stride);      // units of this round (one division per round instead of a 64-bit compare per unit)
        long long unit = base - stride;
        for (int k = 0; k < n_k; k++) {
            unit += stride;
            const uint32_t ca = __shfl_sync(0xffffffffu, my_card, 2 * k), cb = __shfl_sync(0xffffffffu, my_card, 2 * k + 1);
            uint32_t c = 0;
            prefetch_unit(k + kPcPfDist);       // payloads of a later unit on their way to L2 while this one is intersected
            if ((ca >> 20) == 1u) {
                // ---- two small arrays: a (even lane) is scattered, b probed; lane L owns chunks L, L+32, L+64 of both
                const uint4* a4 = reinterpret_cast<const uint4*>(__shfl_sync(0xffffffffu, my_ptr, 2 * k)) + lane;
                const uint4* b4 = reinterpret_cast<const uint4*>(__shfl_sync(0xffffffffu, my_ptr, 2 * k + 1)) + lane;
                const uint32_t card_b = cb & 0xfffffu, na8 = ((ca & 0xfffffu) + 7) >> 3, nb8 = (card_b + 7) >> 3;
                // (chunks past an array's end are loaded too — the arena ends with 4 KiB of slack — and never used)
                const uint4 va0 = ldg_nc(a4), va1 = ldg_nc(a4 + 32), va2 = ldg_nc(a4 + 64);
                const uint4 vb0 = ldg_nc(b4), vb1 = ldg_nc(b4 + 32), vb2 = ldg_nc(b4 + 64);
                const bool pa0 = (uint32_t)lane < na8, pa1 = (uint32_t)lane + 32 < na8, pa2 = (uint32_t)lane + 64 < na8;
                uint32_t addr[3][8];
                auto scatter = [&](const uint4& v, uint32_t (&ad)[8], bool on) {
                    const uint32_t x[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                    for (int q = 0; q < 4; q++) { ad[2 * q] = word_addr_lo(sb, x[q]); ad[2 * q + 1] = word_addr_hi(sb, x[q]); }
                    if (on) {       // (array tails are padded with copies of the last element: setting a bit twice is harmless)
#pragma unroll
                        for (int q = 0; q < 4; q++) { red_or_at(ad[2 * q], 1u << (x[q] & 31)); red_or_at(ad[2 * q + 1], 1u << ((x[q] >> 16) & 31)); }
                    }
                };
                scatter(va0, addr[0], pa0); scatter(va1, addr[1], pa1); scatter(va2, addr[2], pa2);
                __syncwarp();
                // every chunk of b is probed whole: the slots behind its last element hold copies of that element (pad_array_tail),
                // which are taken out of the count again below — no divergent partial-chunk path
                auto probe = [&](const uint4& v) {
                    const uint32_t x[4] = { v.x, v.y, v.z, v.w };
                    uint32_t n = 0;
#pragma unroll
                    for (int q = 0; q < 4; q++) {
                        n += (lds_u32(word_addr_lo(sb, x[q])) >> (x[q] & 31)) & 1u;
                        n += (lds_u32(word_addr_hi(sb, x[q])) >> ((x[q] >> 16) & 31)) & 1u;
                    }
                    return n;
                };
                if ((uint32_t)lane < nb8) c += probe(vb0);
                if ((uint32_t)lane + 32 < nb8) c += probe(vb1);
                if ((uint32_t)lane + 64 < nb8) c += probe(vb2);
                const uint32_t pads = nb8 * 8u - card_b;              // 0..7 copies of b's last element were probed too (warp-uniform)
                if (pads) {
                    const uint32_t ql = (nb8 - 1u) >> 5;               // the chunk holding them: register window slot ql of lane (nb8 - 1) & 31
                    uint32_t wl = ql == 0 ? vb0.w : ql == 1 ? vb1.w : vb2.w;
                    wl = __shfl_sync(0xffffffffu, wl, (int)((nb8 - 1u) & 31u)) >> 16;
                    if (lane == 0) c -= pads * ((bm[wl >> 5] >> (wl & 31)) & 1u);
                }
                __syncwarp();
                if (pa0) {
#pragma unroll
                    for (int q = 0; q < 8; q++) sts_zero(addr[0][q]);
                }
                if (pa1) {
#pragma unroll
                    for (int q = 0; q < 8; q++) sts_zero(addr[1][q]);
                }
                if (pa2) {
#pragma unroll
                    for (int q = 0; q < 8; q++) sts_zero(addr[2][q]);
                }
                __syncwarp();
                c = __reduce_add_sync(0xffffffffu, c);
            } else if ((ca >> 20) == 2u) {
                auto fetch = [&](int src) {     // the original container of lane `src` (the generic class is never swapped)
                    Resolved x;
                    x.ptr = (const void*)__shfl_sync(0xffffffffu, (unsigned long long)r.ptr, src);
                    x.card = __shfl_sync(0xffffffffu, r.card, src);
                    const uint32_t m = __shfl_sync(0xffffffffu, meta, src);
                    x.typ = m >> 16; x.cnt = m & 0xffff;
                    return x;
                };
                c = warp_intersection_count_generic(fetch(2 * k), fetch(2 * k + 1), bm, lane);
            }
            acc += c;
            if (per_pair || per_shard) {                    // (uniform) sums per pair index / per shard: consecutive units mostly share the key
                const long long key = per_pair ? pr : (unit >> 4);
                if (key != run_key) { flush(); run_key = key; }
                run_sum += c;
                if (per_pair) { pr_rem += stride; while (pr_rem >= units_per_pair) { pr_rem -= units_per_pair; pr++; } }
            }
        }
    }
    if (per_pair || per_shard) flush();
    if (pairs_in_smem) {
        __syncthreads();
        for (int i = threadIdx.x; i < (int)n_pairs; i += blockDim.x) { const unsigned long long v = s_pair[i]; if (v) atomicAdd(&per_pair[i], v); }
    }
    if (lane == 0 && total) { if (acc) atomicAdd(total, acc); fused_allreduce_tail(fr, total, gridDim.x * kPcWarps); }
}

// Container-pair-type histogram of a Count(Intersect(Row, Row)) query: hist[4 * ta + tb] += 1 per (shard, slot) unit, t = 0 absent,
// 1 array, 2 bitmap, 3 run.  The device-side analogue of the reference's statsHit("intersectionCount/ArrayRun") counters
// (roaring.go:4477-4614): which of the nine kernels a query exercises, and how often.  Diagnostic: one thread per unit.
__global__ void pair_types_kernel(StoreRef st, uint32_t fvA, uint64_t rowA, uint32_t fvB, uint64_t rowB,
                                  const uint64_t* __restrict__ shards, long long n_units, unsigned long long* hist /* [16] */) {
    __shared__ unsigned int h[16];
    if (threadIdx.x < 16) h[threadIdx.x] = 0;
    __syncthreads();
    for (long long u = (long long)blockIdx.x * blockDim.x + threadIdx.x; u < n_units; u += (long long)gridDim.x * blockDim.x) {
        const Resolved a = resolve(st, fvA, shards[u >> 4], rowA, (int)(u & 15)), b = resolve(st, fvB, shards[u >> 4], rowB, (int)(u & 15));
        atomicAdd(&h[4 * (a.ptr ? a.typ : 0) + (b.ptr ? b.typ : 0)], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 16 && h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], (unsigned long long)h[threadIdx.x]);
}

// ------------------------------------------------------------------------------------------------
// Per-row counts (TopK / TopN-with-ids): one warp per (shard, requested row); filter is an optional
// per-unit bitmap produced by eval_kernel.  doTopK executor.go:2719-2738.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t warp_count_vs_global_bitmap(Resolved a, const uint32_t* fb, uint32_t* bm, int lane) {
    uint32_t c = 0;
    if (a.typ == kArray) c = warp_probe_global(fb, reinterpret_cast<const uint16_t*>(a.ptr), a.card, lane);
    else if (a.typ == kBitmap) {
        const uint4* x = reinterpret_cast<const uint4*>(a.ptr); const uint4* y = reinterpret_cast<const uint4*>(fb);
#pragma unroll 4
        for (int i = lane; i < 512; i += 32) c += popc4(and4(ldg_nc(x + i), y[i]));
    } else {
        const uint32_t* r32 = reinterpret_cast<const uint32_t*>(a.ptr);
        for (uint32_t i = lane; i < a.cnt; i += 32) { uint32_t v = __ldg(r32 + i); c += range_count32(fb, v & 0xffffu, v >> 16); }
    }
    return __reduce_add_sync(0xffffffffu, c);
}

// kPerShard: out_counts is the [n_shards][n_rows] matrix of per-shard counts (what fragment.top's per-shard cut-offs need,
// fragment.go:1329-1388) instead of the [n_rows] vector summed over the shards; every (shard, row) task then owns its slot.
template <bool kPerShard>
__global__ void __launch_bounds__(kPairWarps * 32)
row_count_kernel(StoreRef st, uint32_t fv, const uint64_t* __restrict__ row_ids, int n_rows,
                 const uint64_t* __restrict__ shards, long long n_shards,
                 const uint4* __restrict__ filter_bitmaps /* [n_shards*16][512] or null */,
                 unsigned long long* out_counts /* [n_rows], or [n_shards][n_rows] */) {
    extern __shared__ __align__(128) uint32_t smem32[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t* bm = smem32 + wid * 2048;
    const long long n_tasks = n_shards * (long long)n_rows;
    const long long stride = (long long)gridDim.x * kPairWarps;
    for (long long t = (long long)blockIdx.x * kPairWarps + wid; t < n_tasks; t += stride) {
        const long long si = t / n_rows; const int ri = (int)(t - si * n_rows);
        const uint64_t shard = shards[si], row = row_ids[ri];
        // lanes 0..15 resolve the 16 slots of the row concurrently
        Resolved r; r.ptr = nullptr; r.card = 0; r.typ = 0; r.cnt = 0;
        if (lane < 16) r = resolve(st, fv, shard, row, lane);
        unsigned present = __ballot_sync(0xffffffffu, r.ptr != nullptr);
        unsigned long long acc = 0;
        while (present) {
            int s = __ffs(present) - 1; present &= present - 1;
            Resolved a;
            a.ptr = (const void*)__shfl_sync(0xffffffffu, (unsigned long long)r.ptr, s);
            a.card = __shfl_sync(0xffffffffu, r.card, s);
            uint32_t meta = __shfl_sync(0xffffffffu, ((uint32_t)r.typ << 16) | r.cnt, s);
            a.typ = meta >> 16; a.cnt = meta & 0xffff;
            if (!filter_bitmaps) acc += a.card;
            else acc += warp_count_vs_global_bitmap(a, reinterpret_cast<const uint32_t*>(filter_bitmaps + ((size_t)si * 16 + s) * 512), bm, lane);
        }
        if (lane == 0 && acc) { if (kPerShard) out_counts[(size_t)si * n_rows + ri] = acc; else atomicAdd(&out_counts[ri], acc); }
    }
}

// ------------------------------------------------------------------------------------------------
// Canonical emission of result bitmaps (Row results): optimize() roaring.go:3412-3461 decides the encoding
// on the host from {N, runs}; this kernel writes the payload (array / run / bitmap) at the given offset.
// ------------------------------------------------------------------------------------------------
constexpr int kEmitThreads = 256;   // thread t owns u64 words 4t..4t+3
struct EmitUnit { uint64_t offset; uint32_t unit; uint32_t typ; };

__global__ void __launch_bounds__(kEmitThreads)
canon_emit_kernel(const uint4* __restrict__ bitmaps, const EmitUnit* __restrict__ units, int n_emit, uint8_t* __restrict__ out) {
    __shared__ uint32_t wsum[kEmitThreads / 32], wsum2[kEmitThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int e = blockIdx.x; e < n_emit; e += gridDim.x) {
        EmitUnit u = units[e];
        const uint64_t* src = reinterpret_cast<const uint64_t*>(bitmaps + (size_t)u.unit * 512);
        if (u.typ == kBitmap) {
            uint4* o = reinterpret_cast<uint4*>(out + u.offset);   // offsets of bitmap payloads are only 2-byte aligned in the
            const uint4* s4 = bitmaps + (size_t)u.unit * 512;      // roaring file; the host keeps emit buffers 16 B aligned per unit
            o[tid] = s4[tid]; o[tid + kEmitThreads] = s4[tid + kEmitThreads];
            continue;
        }
        // thread t owns words 4t..4t+3; compute exclusive prefix of element count (array) or start/end counts (run)
        uint64_t w[4]; uint32_t c1 = 0, c2 = 0;
        uint64_t prev = tid ? (src[4 * tid - 1] >> 63) : 0ull;
        uint64_t starts[4], ends[4];
#pragma unroll
        for (int k = 0; k < 4; k++) {
            w[k] = src[4 * tid + k];
            if (u.typ == kArray) c1 += __popcll(w[k]);
            else {
                uint64_t nextbit = (4 * tid + k + 1 < 1024) ? (src[4 * tid + k + 1] & 1ull) : 0ull;
                starts[k] = w[k] & ~((w[k] << 1) | prev);
                ends[k] = w[k] & ~((w[k] >> 1) | (nextbit << 63));
                c1 += __popcll(starts[k]); c2 += __popcll(ends[k]);
                prev = w[k] >> 63;
            }
        }
        // block exclusive scan of c1 (and c2)
        uint32_t i1 = c1, i2 = c2;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t x = __shfl_up_sync(0xffffffffu, i1, d), y = __shfl_up_sync(0xffffffffu, i2, d); if (lane >= d) { i1 += x; i2 += y; } }
        __syncthreads();
        if (lane == 31) { wsum[wid] = i1; wsum2[wid] = i2; }
        __syncthreads();
        uint32_t b1 = 0, b2 = 0;
        for (int k = 0; k < wid; k++) { b1 += wsum[k]; b2 += wsum2[k]; }
        uint32_t p1 = b1 + i1 - c1, p2 = b2 + i2 - c2;
        uint16_t* o16 = reinterpret_cast<uint16_t*>(out + u.offset);
        if (u.typ == kArray) {
#pragma unroll
            for (int k = 0; k < 4; k++) { uint64_t v = w[k]; while (v) { int bit = __ffsll((long long)v) - 1; o16[p1++] = (uint16_t)((4 * tid + k) * 64 + bit); v &= v - 1; } }
        } else {   // run payload: u16 count, then {start,last} pairs (roaring.go:19-51)
            if (tid == 0) o16[0] = (uint16_t)0;  // patched below by the thread holding the total
#pragma unroll
            for (int k = 0; k < 4; k++) {
                uint64_t v = starts[k]; while (v) { int bit = __ffsll((long long)v) - 1; o16[1 + 2 * (p1++)] = (uint16_t)((4 * tid + k) * 64 + bit); v &= v - 1; }
                v = ends[k]; while (v) { int bit = __ffsll((long long)v) - 1; o16[2 + 2 * (p2++)] = (uint16_t)((4 * tid + k) * 64 + bit); v &= v - 1; }
            }
            __syncthreads();
            if (tid == kEmitThreads - 1) o16[0] = (uint16_t)p1;
        }
    }
}

// Column-id expansion of result bitmaps (Row.Columns row.go:471): one CTA per non-empty unit; thread t owns u64 words
// 4t..4t+3, a block scan of the popcounts gives each thread its output position, every set bit becomes one u64 id.
// `first` / `last` clip the unit to the caller's [offset, offset+limit) window (element ranks inside the unit).
struct ColUnit { uint64_t out_off; uint64_t col_base; uint32_t unit; uint32_t first; uint32_t last; uint32_t pad; };

__global__ void __launch_bounds__(kEmitThreads)
columns_emit_kernel(const uint4* __restrict__ bitmaps, const ColUnit* __restrict__ units, int n_units, unsigned long long* __restrict__ out) {
    __shared__ uint32_t wsum[kEmitThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int e = blockIdx.x; e < n_units; e += gridDim.x) {
        const ColUnit u = units[e];
        const uint64_t* src = reinterpret_cast<const uint64_t*>(bitmaps + (size_t)u.unit * 512);
        uint64_t w[4]; uint32_t c = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) { w[k] = src[4 * tid + k]; c += __popcll(w[k]); }
        uint32_t inc = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t x = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += x; }
        __syncthreads();                                   // (wsum of the previous unit has been read)
        if (lane == 31) wsum[wid] = inc;
        __syncthreads();
        uint32_t base = 0;
        for (int k = 0; k < wid; k++) base += wsum[k];
        uint32_t rank = base + inc - c;                    // rank of this thread's first element inside the unit
        if (rank >= u.last || rank + c <= u.first) continue;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            uint64_t v = w[k];
            while (v) {
                const int bit = __ffsll((long long)v) - 1;
                if (rank >= u.first && rank < u.last) out[u.out_off + (rank - u.first)] = u.col_base + (uint64_t)((4 * tid + k) * 64 + bit);
                rank++; v &= v - 1;
            }
        }
    }
}

// Bit-sliced values of the columns of a result row (the bulk form of fragment.value fragment.go:585-617, what Extract and
// executeDistinctShardBSI :2034 transpose column by column): one CTA per non-empty unit.  The unit's base bitmap
// (filter ∩ exists, produced by eval_kernel) is staged in shared memory with a per-word rank table; warp w then walks the
// planes w, w+8, ... — sign row 1 and magnitude rows 2..depth+1 of the BSI view — each container read once, in its own
// encoding, and every base column found in plane b gets bit b (sign: bit 63) or-ed into its output slot
// out[out_off + rank - first].  Ranks match columns_emit_kernel, so the two outputs line up.
constexpr int kExtractThreads = 256;
__global__ void __launch_bounds__(kExtractThreads)
extract_values_kernel(StoreRef st, uint32_t fv, int depth, const uint4* __restrict__ bitmaps, const ColUnit* __restrict__ units, int n_units,
                      unsigned long long* __restrict__ out) {
    __shared__ __align__(16) uint64_t base[1024];
    __shared__ uint32_t rank0[1024];            // number of base bits before word i
    __shared__ uint32_t wsum[kExtractThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nwarps = kExtractThreads / 32;
    for (int e = blockIdx.x; e < n_units; e += gridDim.x) {
        const ColUnit u = units[e];
        const uint64_t* src = reinterpret_cast<const uint64_t*>(bitmaps + (size_t)u.unit * 512);
        __syncthreads();                                   // the previous unit's readers are done
        uint64_t w[4]; uint32_t c = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) { w[k] = src[4 * tid + k]; base[4 * tid + k] = w[k]; c += __popcll(w[k]); }
        uint32_t inc = c;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t x = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += x; }
        if (lane == 31) wsum[wid] = inc;
        __syncthreads();
        uint32_t r = inc - c;
        for (int k = 0; k < wid; k++) r += wsum[k];
#pragma unroll
        for (int k = 0; k < 4; k++) { rank0[4 * tid + k] = r; r += __popcll(w[k]); }
        __syncthreads();
        const uint64_t shard = u.col_base >> 20; const int slot = (int)((u.col_base >> 16) & 15);
        // or `flag` into the slot of base column v (a column outside the base or outside the window is skipped)
        auto hit = [&](uint32_t v, unsigned long long flag) {
            const uint64_t bw = base[v >> 6];
            if (!((bw >> (v & 63)) & 1ull)) return;
            const uint32_t rk = rank0[v >> 6] + __popcll(bw & ((1ull << (v & 63)) - 1ull));
            if (rk >= u.first && rk < u.last) atomicOr(&out[u.out_off + (rk - u.first)], flag);
        };
        for (int pl = wid; pl < depth + 1; pl += nwarps) {                 // pl 0: sign row 1; pl 1..depth: value rows 2..depth+1
            Resolved rc; rc.ptr = nullptr; rc.card = 0; rc.typ = 0; rc.cnt = 0;
            if (lane == 0) rc = resolve(st, fv, shard, (uint64_t)(pl + 1), slot);
            const void* ptr = (const void*)__shfl_sync(0xffffffffu, (unsigned long long)rc.ptr, 0);
            const uint32_t card = __shfl_sync(0xffffffffu, rc.card, 0);
            const uint32_t meta = __shfl_sync(0xffffffffu, ((uint32_t)rc.typ << 16) | rc.cnt, 0);
            if (ptr == nullptr) continue;
            const unsigned long long flag = pl == 0 ? (1ull << 63) : (1ull << (pl - 1));
            const uint32_t typ = meta >> 16, cnt = meta & 0xffffu;
            if (typ == kArray) {
                const uint16_t* a = reinterpret_cast<const uint16_t*>(ptr);
                for (uint32_t i = lane; i < card; i += 32) hit((uint32_t)__ldg(a + i), flag);
            } else if (typ == kBitmap) {
                const uint64_t* g = reinterpret_cast<const uint64_t*>(ptr);
                for (int i = lane; i < 1024; i += 32) {
                    uint64_t v = __ldg(g + i) & base[i];
                    while (v) { const int bit = __ffsll((long long)v) - 1; hit((uint32_t)(i * 64 + bit), flag); v &= v - 1; }
                }
            } else {
                const uint32_t* r32 = reinterpret_cast<const uint32_t*>(ptr);
                for (uint32_t k = 0; k < cnt; k++) {                      // the warp walks each interval's words together
                    const uint32_t iv = __ldg(r32 + k), s0 = iv & 0xffffu, l0 = iv >> 16;
                    for (uint32_t i = (s0 >> 6) + lane; i <= (l0 >> 6); i += 32) {
                        uint64_t m = ~0ull;
                        if (i == (s0 >> 6)) m &= ~0ull << (s0 & 63);
                        if (i == (l0 >> 6)) m &= ~0ull >> (63 - (l0 & 63));
                        uint64_t v = base[i] & m;
                        while (v) { const int bit = __ffsll((long long)v) - 1; hit(i * 64 + (uint32_t)bit, flag); v &= v - 1; }
                    }
                }
            }
        }
    }
}

// Min / Max of an int field over a row (fragment.min / max fragment.go:752-838 with minUnsigned :788 / maxUnsigned :841),
// one CTA per (shard, slot) unit, every plane container read once.  The unit's `consider` bitmap (filter ∩ exists, produced
// by eval_kernel) is split by the sign row; the side that decides the answer is narrowed plane by plane from the top bit:
// largest magnitude keeps R ∩ plane when that is non-empty (bit = 1), smallest magnitude keeps R \ plane when that is
// non-empty (bit = 0).  What is left are the columns holding the extreme value: out = {has, signed value, count} per unit.
// Narrowing a unit on its own is sound because the reduce over units is the executor's ValCount reduce (Smaller / Larger
// executor.go:8446-8560: keep the extreme value, add the counts of equal values), done by the host over the unit results.
// plane `row` of the BSI view `fv` for one (shard, slot) unit as a bitmap, returned as this thread's kEvalU4PerThread uint4
// (CTA-wide call, kEvalThreads threads): bitmap containers are read straight from global memory, arrays / runs are expanded
// into the shared buffer X first, an absent container is empty.  s_res / warp_tmp are CTA-shared scratch.
__device__ __forceinline__ void unit_load_plane(const StoreRef& st, uint32_t fv, uint64_t shard, int slot, uint64_t row,
                                                uint4* X, Resolved* s_res, uint32_t* warp_tmp, uint4 x[kEvalU4PerThread]) {
    const int tid = threadIdx.x;
    __syncthreads();                                       // X and s_res of the previous plane are no longer read
    if (tid == 0) *s_res = resolve(st, fv, shard, row, slot);
    __syncthreads();
    const Resolved r = *s_res;
    if (r.ptr == nullptr) {
#pragma unroll
        for (int h = 0; h < kEvalU4PerThread; h++) x[h] = make_uint4(0, 0, 0, 0);
    } else if (r.typ == kBitmap) {
#pragma unroll
        for (int h = 0; h < kEvalU4PerThread; h++) x[h] = ldg_nc(reinterpret_cast<const uint4*>(r.ptr) + tid + h * kEvalThreads);
    } else {
        if (r.typ == kArray) { bm_zero(X); __syncthreads(); bm_scatter<0>(reinterpret_cast<uint32_t*>(X), reinterpret_cast<const uint16_t*>(r.ptr), r.card); __syncthreads(); }
        else bm_expand_runs(X, reinterpret_cast<const uint16_t*>(r.ptr), r.cnt, warp_tmp);
#pragma unroll
        for (int h = 0; h < kEvalU4PerThread; h++) x[h] = X[tid + h * kEvalThreads];
    }
}
__device__ __forceinline__ bool any_u4(const uint4 v[kEvalU4PerThread]) {
    uint32_t o = 0;
#pragma unroll
    for (int h = 0; h < kEvalU4PerThread; h++) o |= v[h].x | v[h].y | v[h].z | v[h].w;
    return o != 0;
}

struct MinMaxUnit { long long val; unsigned long long cnt; };       // cnt == 0: the unit holds no column of the row

__global__ void __launch_bounds__(kEvalThreads)
bsi_minmax_kernel(StoreRef st, uint32_t fv, int depth, const uint4* __restrict__ consider, const uint64_t* __restrict__ shards, long long n_units, int want_max,
                  MinMaxUnit* __restrict__ out) {
    __shared__ __align__(16) uint4 X[512];
    __shared__ Resolved s_res;
    __shared__ uint32_t warp_tmp[kEvalThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (long long unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
        const uint64_t shard = shards[unit >> 4];
        const int slot = (int)(unit & 15);
        uint4 a[kEvalU4PerThread], x[kEvalU4PerThread], pos[kEvalU4PerThread], neg[kEvalU4PerThread];
#pragma unroll
        for (int h = 0; h < kEvalU4PerThread; h++) a[h] = consider[(size_t)unit * 512 + tid + h * kEvalThreads];
        if (!__syncthreads_or(any_u4(a))) { if (tid == 0) { out[unit].val = 0; out[unit].cnt = 0; } continue; }
        unit_load_plane(st, fv, shard, slot, 1, X, &s_res, warp_tmp, x);                      // bsiSignBit
#pragma unroll
        for (int h = 0; h < kEvalU4PerThread; h++) { pos[h] = andn4(a[h], x[h]); neg[h] = and4(a[h], x[h]); }
        const int has_pos = __syncthreads_or(any_u4(pos)), has_neg = __syncthreads_or(any_u4(neg));
        // which side decides, and in which direction its magnitude is narrowed (fragment.go:760-784, 819-837)
        const bool use_neg = want_max ? !has_pos : has_neg != 0;
        const bool largest = want_max ? !use_neg : use_neg;  // max: largest positive, else smallest |negative|; min: largest |negative|, else smallest positive
        uint4 r[kEvalU4PerThread];
#pragma unroll
        for (int h = 0; h < kEvalU4PerThread; h++) r[h] = use_neg ? neg[h] : pos[h];
        unsigned long long mag = 0;
        for (int i = depth - 1; i >= 0; i--) {
            unit_load_plane(st, fv, shard, slot, (uint64_t)(2 + i), X, &s_res, warp_tmp, x);
            uint4 t[kEvalU4PerThread];
#pragma unroll
            for (int h = 0; h < kEvalU4PerThread; h++) t[h] = largest ? and4(r[h], x[h]) : andn4(r[h], x[h]);
            const int some = __syncthreads_or(any_u4(t));
            if (some) {
#pragma unroll
                for (int h = 0; h < kEvalU4PerThread; h++) r[h] = t[h];
            }
            if ((some != 0) == largest) mag |= 1ull << i;   // largest: bit set when kept; smallest: bit set when no column lacks it
        }
        uint32_t c = 0;
#pragma unroll
        for (int h = 0; h < kEvalU4PerThread; h++) c += popc4(r[h]);
        c = __reduce_add_sync(0xffffffffu, c);
        __syncthreads();
        if (lane == 0) warp_tmp[wid] = c;
        __syncthreads();
        if (tid == 0) {
            uint32_t n = 0;
            for (int k = 0; k < kEvalThreads / 32; k++) n += warp_tmp[k];
            out[unit].val = use_neg ? -(long long)mag : (long long)mag;
            out[unit].cnt = n;
        }
    }
}

// Sum of an int field over a row (fragment.sum fragment.go:722-750 / BitmapBSICountFilter roaring/filter.go:1106-1165), same
// walk: acc[0] += |consider|, acc[1 + 2 i] += |positives ∩ plane i|, acc[2 + 2 i] += |negatives ∩ plane i| — the host forms
// Σ (pos_i - neg_i) << i.  One CTA per (shard, slot) unit, every plane container read once.
__global__ void __launch_bounds__(kEvalThreads)
bsi_sum_kernel(StoreRef st, uint32_t fv, int depth, const uint4* __restrict__ consider, const uint64_t* __restrict__ shards, long long n_units,
               unsigned long long* __restrict__ acc /* [1 + 2 * depth], zeroed by the host */) {
    __shared__ __align__(16) uint4 X[512];
    __shared__ Resolved s_res;
    __shared__ uint32_t warp_tmp[kEvalThreads / 32];
    __shared__ uint32_t wp[kEvalThreads / 32], wn[kEvalThreads / 32];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    // CTA-wide sums of two per-thread counts; thread 0 adds them to acc[k], acc[k + 1] (k + 1 skipped when negative)
    auto add2 = [&](uint32_t p, uint32_t n, int kp, int kn) {
        p = __reduce_add_sync(0xffffffffu, p); n = __reduce_add_sync(0xffffffffu, n);
        __syncthreads();
        if (lane == 0) { wp[wid] = p; wn[wid] = n; }
        __syncthreads();
        if (tid == 0) {
            unsigned long long sp = 0, sn = 0;
            for (int k = 0; k < kEvalThreads / 32; k++) { sp += wp[k]; sn += wn[k]; }
            if (sp) atomicAdd(&acc[kp], sp);
            if (sn && kn >= 0) atomicAdd(&acc[kn], sn);
        }
    };
    for (long long unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
        const uint64_t shard = shards[unit >> 4];
        const int slot = (int)(unit & 15);
        uint4 a[kEvalU4PerThread], x[kEvalU4PerThread], pos[kEvalU4PerThread], neg[kEvalU4PerThread];
#pragma unroll
        for (int h = 0; h < kEvalU4PerThread; h++) a[h] = consider[(size_t)unit * 512 + tid + h * kEvalThreads];
        if (!__syncthreads_or(any_u4(a))) continue;
        unit_load_plane(st, fv, shard, slot, 1, X, &s_res, warp_tmp, x);       // bsiSignBit
        uint32_t ca = 0;
#pragma unroll
        for (int h = 0; h < kEvalU4PerThread; h++) { pos[h] = andn4(a[h], x[h]); neg[h] = and4(a[h], x[h]); ca += (uint32_t)popc4(a[h]); }
        add2(ca, 0u, 0, -1);
        for (int i = 0; i < depth; i++) {
            unit_load_plane(st, fv, shard, slot, (uint64_t)(2 + i), X, &s_res, warp_tmp, x);
            uint32_t cp = 0, cn = 0;
#pragma unroll
            for (int h = 0; h < kEvalU4PerThread; h++) { cp += (uint32_t)popc4(and4(pos[h], x[h])); cn += (uint32_t)popc4(and4(neg[h], x[h])); }
            add2(cp, cn, 1 + 2 * i, 2 + 2 * i);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// GroupBy(Rows(a), Rows(b)) [+ filter]: one CTA per (shard, slot).  Column-keyed hash join instead of the
// reference's |A|x|B| nested intersectionCount loop (executor.go:8880-8934): the elements of field-a rows are inserted
// as (column, row) entries into an open-addressing table in shared memory (linear probing, duplicates allowed, so
// multi-valued columns just occupy several slots), field-b rows are streamed against it and bump counts[i*nB + j].
// Dense (bitmap/run) a-rows take a bitmap pass instead.  Shared memory: 32 KiB table + 8 KiB bitmap => 4 CTAs/SM.
// ------------------------------------------------------------------------------------------------
constexpr int kGbThreads = 256;
constexpr int kGbSlots = 8192;          // open-addressing table slots per CTA (32 KiB)
constexpr int kGbPool = kGbSlots / 2;   // entries per pass (load factor <= 0.5)
constexpr uint32_t kGbEmpty = 0xffffffffu;
constexpr uint32_t kGbDenseCard = 4096; // a-rows at/above this cardinality (or non-array) use the bitmap pass

template <class F>
__device__ __forceinline__ void warp_for_each(const Resolved& c, int lane, F f) {
    if (c.typ == kArray) {
        const uint16_t* a = reinterpret_cast<const uint16_t*>(c.ptr);
        for (uint32_t i = lane; i < c.card; i += 32) f((uint32_t)__ldg(a + i));
    } else if (c.typ == kBitmap) {
        const uint32_t* w = reinterpret_cast<const uint32_t*>(c.ptr);
        for (uint32_t i = lane; i < 2048; i += 32) { uint32_t v = __ldg(w + i); while (v) { int b = __ffs(v) - 1; f(i * 32 + b); v &= v - 1; } }
    } else {
        const uint32_t* r = reinterpret_cast<const uint32_t*>(c.ptr);
        for (uint32_t i = 0; i < c.cnt; i++) { uint32_t v = __ldg(r + i); uint32_t s = v & 0xffffu, l = v >> 16; for (uint32_t x = s + lane; x <= l; x += 32) f(x); }
    }
}

// block-wide exclusive prefix sum of one uint32 per thread (kGbThreads threads); `tmp` holds one word per warp
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* tmp, uint32_t* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t x = __shfl_up_sync(0xffffffffu, inc, d); if (lane >= d) inc += x; }
    __syncthreads();
    if (lane == 31) tmp[wid] = inc;
    __syncthreads();
    uint32_t base = 0, tot = 0;
    for (int k = 0; k < kGbThreads / 32; k++) { if (k < wid) base += tmp[k]; tot += tmp[k]; }
    if (total) *total = tot;
    return base + inc - v;
}

__global__ void __launch_bounds__(kGbThreads)
groupby_kernel(StoreRef st, uint32_t fvA, const uint64_t* __restrict__ rowsA, int nA,
               uint32_t fvB, const uint64_t* __restrict__ rowsB, int nB,
               const uint64_t* __restrict__ shards, long long n_units,
               const uint4* __restrict__ filter_bitmaps /* per unit or null */,
               unsigned long long* counts /* [nA*nB] */, const unsigned int* __restrict__ unit_list /* null, or [0] = n, then unit indices */) {
    extern __shared__ uint8_t gsm[];
    uint32_t* tab = reinterpret_cast<uint32_t*>(gsm);                        // kGbSlots entries: (column << 16) | row index
    uint32_t* fbm = reinterpret_cast<uint32_t*>(gsm + kGbSlots * 4);         // 8 KiB bitmap (dense a-row)
    __shared__ Resolved resA[kGbThreads], resB[kGbThreads];
    __shared__ uint32_t offA[kGbThreads], offB[kGbThreads];
    __shared__ uint32_t scan_tmp[kGbThreads / 32];
    __shared__ uint32_t s_any, s_pass_end;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nwarps = kGbThreads / 32;

    const long long n_work = unit_list ? (long long)unit_list[0] : n_units;     // the units groupby_direct_kernel declined
    for (long long wi = blockIdx.x; wi < n_work; wi += gridDim.x) {
        const long long unit = unit_list ? (long long)unit_list[1 + wi] : wi;
        const uint64_t shard = shards[unit >> 4];
        const int slot = (int)(unit & 15);
        const uint32_t* flt = filter_bitmaps ? reinterpret_cast<const uint32_t*>(filter_bitmaps + (size_t)unit * 512) : nullptr;
        __syncthreads();
        if (tid == 0) {   // executor.go:8769-8772: a shard missing either fragment contributes nothing
            bool ok = fvA < st.n_views && fvB < st.n_views;
            if (ok) { ViewTab va = st.views[fvA], vb = st.views[fvB]; ok = shard < va.n_shards && shard < vb.n_shards && st.shardmap[va.shard_off + shard] >= 0 && st.shardmap[vb.shard_off + shard] >= 0; }
            s_any = ok ? 1u : 0u;
        }
        __syncthreads();
        if (!s_any) continue;

        for (int a0 = 0; a0 < nA; a0 += kGbThreads) {
            const int chunkA = min(kGbThreads, nA - a0);
            // all a-row descriptor chains of this chunk are walked concurrently (one per thread)
            { Resolved r; r.ptr = nullptr; r.card = 0; r.typ = 0; r.cnt = 0;
              if (tid < chunkA) r = resolve(st, fvA, shard, rowsA[a0 + tid], slot);
              __syncthreads(); resA[tid] = r; __syncthreads(); }
            int ia = 0;
            while (ia < chunkA) {
                // ---- sparse pass [ia, pass_end): pool offsets = exclusive prefix over row cardinalities (deterministic)
                const Resolved mine = resA[tid];
                const bool in_range = tid >= ia && tid < chunkA;
                const bool dense = in_range && mine.ptr && (mine.typ != kArray || mine.card >= kGbDenseCard);
                const uint32_t need = (in_range && mine.ptr && !dense) ? mine.card : 0u;
                const uint32_t off = block_excl_scan(need, scan_tmp, nullptr);
                if (tid == 0) s_pass_end = (uint32_t)chunkA;
                __syncthreads();
                if (in_range && (dense || off + need > (uint32_t)kGbPool)) atomicMin(&s_pass_end, (uint32_t)tid);
                offA[tid] = off;
                { uint4* t4 = reinterpret_cast<uint4*>(tab); for (int i = tid; i < kGbSlots / 4; i += kGbThreads) t4[i] = make_uint4(kGbEmpty, kGbEmpty, kGbEmpty, kGbEmpty); }
                __syncthreads();
                const int pass_end = (int)s_pass_end;
                {   // flat: one thread per a-element of the pass; the owning row is found by binary search over offA[]
                    const uint32_t total = pass_end < chunkA ? offA[pass_end] : (offA[chunkA - 1] + ((resA[chunkA - 1].ptr && resA[chunkA - 1].typ == kArray && resA[chunkA - 1].card < kGbDenseCard) ? resA[chunkA - 1].card : 0u));
                    for (uint32_t e = tid; e < total; e += kGbThreads) {
                        int lo = ia, hi = pass_end - 1;           // last row i in [ia, pass_end) with offA[i] <= e
                        while (lo < hi) { int m = (lo + hi + 1) >> 1; if (offA[m] <= e) lo = m; else hi = m - 1; }
                        const Resolved c = resA[lo];
                        const uint32_t k = e - offA[lo];
                        if (!c.ptr || k >= c.card) continue;      // rows without a container have zero width
                        uint32_t col = __ldg(reinterpret_cast<const uint16_t*>(c.ptr) + k);
                        if (flt && !((__ldg(flt + (col >> 5)) >> (col & 31)) & 1u)) continue;
                        const uint32_t ent = (col << 16) | (uint32_t)(a0 + lo);
                        uint32_t h = (col * 40503u) & (kGbSlots - 1);
                        while (atomicCAS(&tab[h], kGbEmpty, ent) != kGbEmpty) h = (h + 1) & (kGbSlots - 1);
                    }
                }
                __syncthreads();
                // ---- probe: stream b rows against the table
                if (pass_end > ia) {
                    for (int b0 = 0; b0 < nB; b0 += kGbThreads) {
                        const int chunkB = min(kGbThreads, nB - b0);
                        { Resolved r; r.ptr = nullptr; r.card = 0; r.typ = 0; r.cnt = 0;
                          if (tid < chunkB) r = resolve(st, fvB, shard, rowsB[b0 + tid], slot);
                          __syncthreads(); resB[tid] = r; __syncthreads(); }
                        {   // arrays: flat thread-per-element (offsets by block scan); bitmap/run rows: warp loop
                            const Resolved mb = resB[tid];
                            const uint32_t nb_ = (tid < chunkB && mb.ptr && mb.typ == kArray) ? mb.card : 0u;
                            uint32_t totalB = 0;
                            const uint32_t ob = block_excl_scan(nb_, scan_tmp, &totalB);
                            __syncthreads();
                            offB[tid] = ob;
                            __syncthreads();
                            for (uint32_t e = tid; e < totalB; e += kGbThreads) {
                                int lo = 0, hi = chunkB - 1;
                                while (lo < hi) { int m = (lo + hi + 1) >> 1; if (offB[m] <= e) lo = m; else hi = m - 1; }
                                const Resolved c = resB[lo];
                                const uint32_t k = e - offB[lo];
                                if (!c.ptr || c.typ != kArray || k >= c.card) continue;
                                uint32_t col = __ldg(reinterpret_cast<const uint16_t*>(c.ptr) + k);
                                for (uint32_t h = (col * 40503u) & (kGbSlots - 1);; h = (h + 1) & (kGbSlots - 1)) {
                                    const uint32_t ent = tab[h];
                                    if (ent == kGbEmpty) break;
                                    if ((ent >> 16) == col) atomicAdd(&counts[(size_t)(ent & 0xffffu) * nB + (b0 + lo)], 1ull);
                                }
                            }
                        }
                        for (int j = wid; j < chunkB; j += nwarps) {
                            const Resolved c = resB[j];
                            if (!c.ptr || c.typ == kArray) continue;
                            const int jj = b0 + j;
                            warp_for_each(c, lane, [&](uint32_t col) {
                                for (uint32_t h = (col * 40503u) & (kGbSlots - 1);; h = (h + 1) & (kGbSlots - 1)) {
                                    const uint32_t ent = tab[h];
                                    if (ent == kGbEmpty) break;
                                    if ((ent >> 16) == col) atomicAdd(&counts[(size_t)(ent & 0xffffu) * nB + jj], 1ull);
                                }
                            });
                        }
                    }
                }
                __syncthreads();
                ia = pass_end;
                // ---- dense pass for the row that ended the sparse pass (bitmap/run container or >= kGbDenseCard elements)
                if (ia < chunkA) {
                    const Resolved c = resA[ia];
                    const bool is_dense = c.ptr && (c.typ != kArray || c.card >= kGbDenseCard);
                    if (is_dense) {
                        uint4* f4 = reinterpret_cast<uint4*>(fbm);
                        for (int i = tid; i < 512; i += kGbThreads) f4[i] = make_uint4(0, 0, 0, 0);
                        __syncthreads();
                        if (c.typ == kBitmap) { const uint4* g = reinterpret_cast<const uint4*>(c.ptr); for (int i = tid; i < 512; i += kGbThreads) f4[i] = ldg_nc(g + i); }
                        else if (c.typ == kArray) { const uint16_t* a = reinterpret_cast<const uint16_t*>(c.ptr); for (uint32_t k = tid; k < c.card; k += kGbThreads) { uint32_t v = __ldg(a + k); atomicOr(&fbm[v >> 5], 1u << (v & 31)); } }
                        else { const uint32_t* r = reinterpret_cast<const uint32_t*>(c.ptr);
                            for (uint32_t k = wid; k < c.cnt; k += nwarps) { uint32_t v = __ldg(r + k); uint32_t s0 = v & 0xffffu, l0 = v >> 16;
                                for (uint32_t w = (s0 >> 5) + lane; w <= (l0 >> 5); w += 32) { uint32_t mask = 0xffffffffu; if (w == (s0 >> 5)) mask &= 0xffffffffu << (s0 & 31); if (w == (l0 >> 5)) mask &= 0xffffffffu >> (31 - (l0 & 31)); atomicOr(&fbm[w], mask); } } }
                        __syncthreads();
                        if (flt) { const uint4* g = reinterpret_cast<const uint4*>(flt); for (int i = tid; i < 512; i += kGbThreads) f4[i] = and4(f4[i], g[i]); __syncthreads(); }
                        for (int b0 = 0; b0 < nB; b0 += kGbThreads) {
                            const int chunkB = min(kGbThreads, nB - b0);
                            { Resolved r; r.ptr = nullptr; r.card = 0; r.typ = 0; r.cnt = 0;
                              if (tid < chunkB) r = resolve(st, fvB, shard, rowsB[b0 + tid], slot);
                              __syncthreads(); resB[tid] = r; __syncthreads(); }
                            for (int j = wid; j < chunkB; j += nwarps) {
                                const Resolved bb = resB[j];
                                if (!bb.ptr) continue;
                                uint32_t cc = 0;
                                if (bb.typ == kArray) cc = warp_probe_smem(fbm, reinterpret_cast<const uint16_t*>(bb.ptr), bb.card, lane);
                                else if (bb.typ == kBitmap) cc = warp_and_count_gs(reinterpret_cast<const uint4*>(bb.ptr), fbm, lane);
                                else { const uint32_t* r = reinterpret_cast<const uint32_t*>(bb.ptr); for (uint32_t k = lane; k < bb.cnt; k += 32) { uint32_t v = __ldg(r + k); cc += range_count32(fbm, v & 0xffffu, v >> 16); } }
                                cc = __reduce_add_sync(0xffffffffu, cc);
                                if (lane == 0 && cc) atomicAdd(&counts[(size_t)(a0 + ia) * nB + (b0 + j)], (unsigned long long)cc);
                            }
                        }
                        __syncthreads();
                        ia++;
                    }
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// groupby_direct_kernel (round 2): GroupBy(Rows(a), Rows(b)) for array-dominated fields — hundreds of rows, a handful of
// columns per container — without a hash table.  One CTA of 256 threads per (shard, slot); the 65,536 columns of the slot index a
// byte table directly: tab[column] = index of the a-row that holds the column (one thread per a-row, at most 256 a-rows per launch:
// the host chunks longer lists), valid where the 8 KiB presence bitmap has the column's bit.  The presence bit is set with one
// atomicOr whose return value tells a second a-row of the same column (fields that are not mutually exclusive): that (column, row)
// goes to a short side list every probe also scans.  Then one thread per b-row looks its columns up: bitmap word, byte, one RED.
// Per element: ~8 instructions to insert, ~10 to probe, no probe chains, no CAS loops, nothing to clear but the 8 KiB bitmap — a
// hash table per group of slots (the kernel this one replaced) took ~70 warp instructions per probed element at 8-17 of 32 lanes.  72 KiB of shared memory:
// three CTAs per SM, so one unit's descriptor chain (views -> row table -> descriptor -> payload) hides behind two other units.
// Descriptors / payloads are read 16 bytes at a stride of one row (the 16 units of a shard run side by side: the sectors are
// shared in L2).  A unit is declined — listed in `fallback` for groupby_kernel before anything of it is counted — when a container
// of either side is a bitmap or holds more than kGdMaxCard columns (one thread walks a container), or the side list overflows.
// Replaces the same reference code as groupby_kernel (groupByIterator executor.go:8617-8867).
// ------------------------------------------------------------------------------------------------
constexpr int kGdThreads = 256;
constexpr uint32_t kGdOver = 256;                 // side-list entries ((column << 8) | a-row index)
constexpr uint32_t kGdMaxCard = 1024;
constexpr size_t kGdSmemBytes = 65536 + 8192;

// one thread walks an array or run container, one column per call; `first` = its first 16 bytes, loaded earlier (all containers start
// 16-byte aligned and are allocated in 16-byte units)
template <class F>
__device__ __forceinline__ void thread_for_each_col(const Resolved& c, const uint4& first, F f) {
    const uint4* p = reinterpret_cast<const uint4*>(c.ptr);
    if (c.typ == kArray) {
        for (uint32_t k0 = 0; k0 < c.card; k0 += 8) {
            const uint4 v = k0 ? ldg_nc(p + (k0 >> 3)) : first;
            const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
            for (int q = 0; q < 8; q++) { if (k0 + q >= c.card) break; f((w[q >> 1] >> ((q & 1) * 16)) & 0xffffu); }
        }
    } else {
        for (uint32_t k0 = 0; k0 < c.cnt; k0 += 4) {
            const uint4 v = k0 ? ldg_nc(p + (k0 >> 2)) : first;
            const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
            for (int q = 0; q < 4; q++) { if (k0 + q >= c.cnt) break; for (uint32_t x = w[q] & 0xffffu, l = w[q] >> 16; x <= l; x++) f(x); }
        }
    }
}

__global__ void __launch_bounds__(kGdThreads, 3)
groupby_direct_kernel(StoreRef st, uint32_t fvA, const uint64_t* __restrict__ rowsA, int nA /* <= kGdThreads */,
                      uint32_t fvB, const uint64_t* __restrict__ rowsB, int nB,
                      const uint64_t* __restrict__ shards, long long n_units /* shards x 16 */,
                      const uint4* __restrict__ filter_bitmaps /* per (shard, slot) unit or null */,
                      unsigned long long* counts /* [nA*nB] */, unsigned int* fallback /* [0] = n, then unit indices */) {
    extern __shared__ __align__(16) uint8_t gd_sm[];
    uint8_t* tab = gd_sm;
    uint32_t* bits = reinterpret_cast<uint32_t*>(gd_sm + 65536);
    __shared__ uint32_t s_over[kGdOver];
    __shared__ uint32_t s_nover;
    const int tid = threadIdx.x;
    const bool multiB = nB > kGdThreads;
    if (fvA >= st.n_views || fvB >= st.n_views) return;
    auto too_big = [](const Resolved& r) { return r.ptr && (r.typ == kBitmap || r.card > kGdMaxCard); };

    // one (shard, slot) unit, its a- and b-row containers located and their first 16 bytes loaded (or on their way); `mid` runs between
    // the two phases (the pipelined caller issues the next unit's loads there)
    auto unit_body = [&](long long unit, uint64_t shard, int slot, const Resolved& ra, Resolved rb, uint4 va, uint4 vb, auto&& mid) {
        const uint32_t* flt = filter_bitmaps ? reinterpret_cast<const uint32_t*>(filter_bitmaps + (size_t)unit * 512) : nullptr;
        bool bad = too_big(ra) || too_big(rb);
        if (multiB)      // every b-row is looked at before anything is counted
            for (int b0 = 0; b0 < nB; b0 += kGdThreads) if (b0 + tid < nB) bad |= too_big(resolve(st, fvB, shard, rowsB[b0 + tid], slot));
        { uint4* b4 = reinterpret_cast<uint4*>(bits); b4[tid] = make_uint4(0, 0, 0, 0); b4[tid + kGdThreads] = make_uint4(0, 0, 0, 0); }
        if (tid == 0) s_nover = 0;
        bool decline = __syncthreads_or(bad ? 1 : 0) != 0;
        if (!decline) {
            // ---- a-rows: column -> row index
            if (ra.ptr) thread_for_each_col(ra, va, [&](uint32_t col) {
                if (flt && !((__ldg(flt + (col >> 5)) >> (col & 31)) & 1u)) return;
                const uint32_t m = 1u << (col & 31);
                if (!(atomicOr(&bits[col >> 5], m) & m)) tab[col] = (uint8_t)tid;
                else { const uint32_t k = atomicAdd(&s_nover, 1u); if (k < kGdOver) s_over[k] = (col << 8) | (uint32_t)tid; }
            });
            __syncthreads();
        }
        mid();
        if (!decline) {
            const uint32_t nover = s_nover;
            decline = nover > kGdOver;
            // ---- b-rows: look every column up
            if (!decline)
                for (int b0 = 0; b0 < nB; b0 += kGdThreads) {
                    if (multiB) { rb.ptr = nullptr; if (b0 + tid < nB) rb = resolve(st, fvB, shard, rowsB[b0 + tid], slot); if (rb.ptr) vb = ldg_nc(reinterpret_cast<const uint4*>(rb.ptr)); }
                    if (!rb.ptr) continue;
                    unsigned long long* cj = counts + (b0 + tid);
                    thread_for_each_col(rb, vb, [&](uint32_t col) {
                        if ((bits[col >> 5] >> (col & 31)) & 1u) atomicAdd(cj + (uint32_t)tab[col] * (uint32_t)nB, 1ull);
                        for (uint32_t k = 0; k < nover; k++) { const uint32_t e = s_over[k]; if ((e >> 8) == col) atomicAdd(cj + (e & 0xffu) * (uint32_t)nB, 1ull); }
                    });
                }
        }
        if (decline && tid == 0) { const unsigned int k = atomicAdd(&fallback[0], 1u); fallback[1 + k] = (unsigned int)unit; }
        __syncthreads();                                       // the bitmap and the side list are reused by the next unit
    };

    const ViewTab vA = st.views[fvA], vB = st.views[fvB];
    if (!multiB && vA.rt_rows && vB.rt_rows) {
        // Both views have the dense (shard, row) directory: the three dependent loads of a unit — directory entry, descriptor, first
        // payload chunk — are issued one unit apart each, so that every level has a whole phase of another unit to arrive in:
        //   iteration i:  shard id(i+3), directory(i+2), descriptor(i+1) <- directory(i+1) | insert(i) | payload(i+1) <- descriptor(i+1) | probe(i)
        // (a shard without one of the fragments has empty directory entries on that side and counts nothing, like the explicit test)
        struct Ent { uint32_t fa, ma, fb, mb; };
        struct D3 { uint32_t x, y, z, w; };
        struct Dsc { D3 a, b; };                               // ContDesc images: x = off16, y = card (0: absent), z = typ | cnt << 16
        const uint64_t rowA = tid < nA ? rowsA[tid] : 0, rowB = tid < nB ? rowsB[tid] : 0;
        const bool inA = tid < nA && rowA >= vA.rmin && rowA - vA.rmin < vA.rt_rows, inB = tid < nB && rowB >= vB.rmin && rowB - vB.rmin < vB.rt_rows;
        const uint64_t offA = vA.rt_off + (rowA - vA.rmin), offB = vB.rt_off + (rowB - vB.rmin);
        auto shard_of = [&](long long u) -> uint64_t { return u < n_units ? shards[u >> 4] : ~0ull; };       // (~0: no such unit)
        auto load_ent = [&](uint64_t sh) {
            Ent e; e.fa = e.ma = e.fb = e.mb = 0;
            if (inA && sh < vA.n_shards) { const RowTabEnt t = st.rowtab[offA + sh * vA.rt_rows]; e.fa = t.first_desc; e.ma = t.mask; }
            if (inB && sh < vB.n_shards) { const RowTabEnt t = st.rowtab[offB + sh * vB.rt_rows]; e.fb = t.first_desc; e.mb = t.mask; }
            return e;
        };
        // (12 of the descriptor's 16 bytes: a 16-byte load would leave a dead fourth register that the allocator reuses at once, and the
        // next write to it then waits for the load — seen as a long-scoreboard stall at the top of the loop)
        auto load_desc = [&](uint32_t first, uint32_t mask, int slot) {
            D3 d; d.x = d.y = d.z = d.w = 0;
            if ((mask >> slot) & 1u) {
                const uint4 v = __ldg(reinterpret_cast<const uint4*>(st.descs + first + __popc(mask & ((1u << slot) - 1u))));
                d.x = v.x; d.y = v.y; d.z = v.z; d.w = v.w;
            }
            return d;
        };
        auto load_dsc = [&](const Ent& e, int slot) { Dsc d; d.a = load_desc(e.fa, e.ma, slot); d.b = load_desc(e.fb, e.mb, slot); return d; };
        // (the descriptor's unused fourth word is kept live until the descriptor is consumed: a dead destination register of the
        // 16-byte load is reused at once by the allocator, and the next write to it then waits for the load)
        auto located = [&](D3 d) {
            asm volatile("" : "+r"(d.w));
            Resolved r; r.ptr = d.y ? st.payload + (size_t)d.x * 16 : nullptr; r.card = d.y; r.typ = (uint16_t)(d.z & 0xffffu); r.cnt = (uint16_t)(d.z >> 16); return r; };
        auto load_first = [&](const D3& d) { return d.y ? ldg_nc(reinterpret_cast<const uint4*>(st.payload + (size_t)d.x * 16)) : make_uint4(0, 0, 0, 0); };
        const long long step = gridDim.x;
        long long unit = blockIdx.x;
        if (unit >= n_units) return;
        uint64_t s2 = shard_of(unit + 2 * step);
        Ent e1 = load_ent(shard_of(unit + step));
        Dsc d0 = load_dsc(load_ent(shard_of(unit)), (int)(unit & 15));
        uint4 va = load_first(d0.a), vb = load_first(d0.b);
        for (; unit < n_units; unit += step) {
            const uint64_t s3 = shard_of(unit + 3 * step);
            const Ent e2 = load_ent(s2);
            const Dsc d1 = load_dsc(e1, (int)((unit + step) & 15));
            uint4 va1, vb1;
            unit_body(unit, 0 /* (the shard id is only needed by the multi-pass b side) */, (int)(unit & 15), located(d0.a), located(d0.b), va, vb, [&] { va1 = load_first(d1.a); vb1 = load_first(d1.b); });
            s2 = s3; e1 = e2; d0 = d1; va = va1; vb = vb1;
        }
        return;
    }
    for (long long unit = blockIdx.x; unit < n_units; unit += gridDim.x) {
        const uint64_t shard = shards[unit >> 4];
        const int slot = (int)(unit & 15);
        // executor.go:8769-8772: a shard missing either fragment contributes nothing (uniform test, broadcast loads)
        if (!(shard < vA.n_shards && shard < vB.n_shards && st.shardmap[vA.shard_off + shard] >= 0 && st.shardmap[vB.shard_off + shard] >= 0)) continue;
        Resolved ra, rb; ra.ptr = nullptr; ra.card = 0; ra.typ = 0; ra.cnt = 0; rb = ra;
        if (tid < nA) ra = resolve(st, fvA, shard, rowsA[tid], slot);
        if (!multiB && tid < nB) rb = resolve(st, fvB, shard, rowsB[tid], slot);
        uint4 va = make_uint4(0, 0, 0, 0), vb = va;
        if (ra.ptr) va = ldg_nc(reinterpret_cast<const uint4*>(ra.ptr));
        if (rb.ptr) vb = ldg_nc(reinterpret_cast<const uint4*>(rb.ptr));
        unit_body(unit, shard, slot, ra, rb, va, vb, [] {});
    }
}

// ------------------------------------------------------------------------------------------------
// arena_gather_kernel (fbgpu_compact): copies containers one by one from the old payload arena into the new one — one warp per
// container, 16 bytes per lane and step.  Used for fragments that fbgpu_apply_containers left with holes.
// ------------------------------------------------------------------------------------------------
struct ArenaMove { uint32_t from16, to16, len16, pad; };
__global__ void __launch_bounds__(256)
arena_gather_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, const ArenaMove* __restrict__ mv, long long n) {
    const int lane = threadIdx.x & 31;
    for (long long i = (long long)blockIdx.x * 8 + (threadIdx.x >> 5); i < n; i += (long long)gridDim.x * 8) {
        const ArenaMove m = mv[i];
        for (uint32_t k = lane; k < m.len16; k += 32) dst[(size_t)m.to16 + k] = src[(size_t)m.from16 + k];
    }
}

}  // namespace fbgpu
