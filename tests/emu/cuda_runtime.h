// TEST INFRASTRUCTURE ONLY — a CPU stand-in for <cuda_runtime.h> that lets the UNMODIFIED sources of libfbgpu
// (featurebase_b200/csrc/fbgpu.cu + kernels.cuh) be compiled with g++ and their kernels be *interpreted* thread by thread,
// so that kernel logic written while no GPU was reachable can still be run against the oracle (tests/test_emu_kernels.py).
// It is never built, loaded or referenced by the product (featurebase_b200/ loads libfbgpu.so only); a library built
// from it is slow (one fibre per CUDA thread) and exists under tests/emu/_build/ only.
//
// Model: blocks run one after another; the threads of a block are fibres (ucontext) that run until they reach a barrier
// (__syncthreads*, or the implicit warp barrier inside a *_sync primitive) and are resumed when every live thread of the
// block / warp has arrived.  A barrier that can never complete (divergent __syncthreads, a lane missing from a full-mask
// shuffle) is reported as a deadlock and aborts.  Atomics are plain read-modify-writes (one fibre runs at a time), so data
// races are NOT detected — compute-sanitizer on the GPU does that.  Shared memory, static
// and dynamic, is re-poisoned for every block; device allocations start as garbage and end at a guard page.
//
// tests/emu/make_emu_source.py rewrites, in a scratch copy of the sources, the three constructs g++ cannot parse:
// kernel<<<...>>>(...) launches, `extern __shared__ T name[];`, and inline PTX (each known statement is mapped to the
// emu:: function below; an unknown one fails the rewrite).
#pragma once
#include <time.h>
#include <ucontext.h>

#include <dlfcn.h>
#include <stdarg.h>
#include <sys/mman.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <map>
#include <memory>
#include <shared_mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <vector>

// (every standard header the sources use is included above: the qualifier macros below must not reach libstdc++'s own
// __attribute__((__noinline__)) spellings)
#define FBGPU_EMU 1
#define __align__(n) __attribute__((aligned(n)))
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __noinline__ __attribute__((noinline))
#define __launch_bounds__(...)
// static shared memory goes into one named section so that launch() can poison all of it before every block: real shared
// memory is not zero at block start, a kernel that reads a __shared__ variable before writing it must not pass here
#ifdef FBGPU_EMU_PLAIN_SHARED            // AddressSanitizer build: ordinary statics get red zones (ASAN leaves named sections alone)
#define __shared__ static
static char* const __start_fbgpu_smem = nullptr;
static char* const __stop_fbgpu_smem = nullptr;
#else
#define __shared__ static __attribute__((section("fbgpu_smem")))
extern "C" char __start_fbgpu_smem[] __attribute__((weak, visibility("hidden")));
extern "C" char __stop_fbgpu_smem[] __attribute__((weak, visibility("hidden")));
#endif
#define __constant__ static

struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; } __attribute__((aligned(16)));
struct int2 { int x, y; };
struct int4 { int x, y, z, w; } __attribute__((aligned(16)));
struct dim3 { unsigned x = 1, y = 1, z = 1; dim3() {} dim3(unsigned a, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
static inline uint2 make_uint2(uint32_t x, uint32_t y) { return uint2{ x, y }; }
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { uint4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }
static inline int2 make_int2(int x, int y) { return int2{ x, y }; }

namespace emu {

constexpr size_t kStack = 256 << 10;
constexpr size_t kDynSmem = 232448;

// ---- fibre switch: glibc's swapcontext makes a signal-mask system call per switch; on x86-64 a six-register switch is used instead
#if defined(__x86_64__) && !defined(FBGPU_EMU_UCONTEXT)
extern "C" void fbgpu_emu_switch(void** save_sp, void* load_sp);
asm(R"(
    .text
    .type fbgpu_emu_switch,@function
fbgpu_emu_switch:
    pushq %rbp
    pushq %rbx
    pushq %r12
    pushq %r13
    pushq %r14
    pushq %r15
    movq %rsp, (%rdi)
    movq %rsi, %rsp
    popq %r15
    popq %r14
    popq %r13
    popq %r12
    popq %rbx
    popq %rbp
    ret
    .size fbgpu_emu_switch,.-fbgpu_emu_switch
)");
struct Ctx { void* sp = nullptr; };
inline void ctx_switch(Ctx& from, Ctx& to) { fbgpu_emu_switch(&from.sp, to.sp); }
inline void ctx_make(Ctx& c, char* stack, size_t size, void (*fn)()) {
    uintptr_t top = ((uintptr_t)stack + size) & ~(uintptr_t)15;
    void** sp = (void**)top;
    *--sp = nullptr;                 // fake return address of fn: fn is entered with rsp = 8 mod 16, like after a call
    *--sp = (void*)fn;               // taken by the switch's ret
    for (int i = 0; i < 6; i++) *--sp = nullptr;
    c.sp = sp;
}
#else
struct Ctx { ucontext_t uc; };
inline void ctx_switch(Ctx& from, Ctx& to) { swapcontext(&from.uc, &to.uc); }
inline void ctx_make(Ctx& c, char* stack, size_t size, void (*fn)()) {
    getcontext(&c.uc); c.uc.uc_stack.ss_sp = stack; c.uc.uc_stack.ss_size = size; c.uc.uc_link = nullptr;
    makecontext(&c.uc, fn, 0);
}
#endif

struct Warp { int alive = 0, arrived = 0; long gen = 0; uint64_t buf[32]; };
struct Fiber {
    Ctx ctx; char* stack = nullptr; bool done = true;
    dim3 tid; int lane = 0, warp = 0;
    long blk_gen = 0, warp_gen = 0;          // barriers this thread has arrived at
    int wait = 0;                             // 0 runnable, 1 block barrier, 2 warp barrier
    unsigned red_n = 0;
};
struct State {
    std::mutex mu;                            // one launch at a time (host code may call from several threads)
    std::vector<Fiber> fibers; std::vector<Warp> warps;
    Ctx sched; Fiber* cur = nullptr;
    dim3 grid, block, bid; int nthreads = 0;
    int alive = 0, arrived = 0; long bar_gen = 0;
    int red_cnt[2] = { 0, 0 };
    const std::function<void()>* body = nullptr;
    unsigned long long launches = 0, switches = 0;
    int order = 0; unsigned salt = 12345u;
    State() { const char* e = getenv("FBGPU_EMU_ORDER"); order = !e ? 0 : !strcmp(e, "reverse") ? 1 : !strcmp(e, "random") ? 2 : 0; }
};
inline State g_state;                                  // (one per library image)
alignas(128) inline uint8_t g_dyn[kDynSmem];           // dynamic shared memory; lives in .bss next to the `__shared__` statics
inline State& S() { return g_state; }

[[noreturn]] inline void die(const char* what) { fprintf(stderr, "[emu] fatal: %s (block %u thread %u)\n", what, S().bid.x, S().cur ? S().cur->tid.x : 0u); abort(); }

inline void yield() { State& s = S(); s.switches++; ctx_switch(s.cur->ctx, s.sched); }

inline void release_block(State& s) { s.arrived = 0; s.bar_gen++; }
inline void release_warp(Warp& w) { w.arrived = 0; w.gen++; }

inline void block_barrier() {
    State& s = S(); Fiber& me = *s.cur;
    const long g = ++me.blk_gen;
    if (++s.arrived == s.alive) { release_block(s); return; }
    me.wait = 1;
    while (s.bar_gen < g) yield();
    me.wait = 0;
}
inline void warp_barrier() {
    State& s = S(); Fiber& me = *s.cur; Warp& w = s.warps[me.warp];
    const long g = ++me.warp_gen;
    if (++w.arrived == w.alive) { release_warp(w); return; }
    me.wait = 2;
    while (w.gen < g) yield();
    me.wait = 0;
}
inline int block_reduce(int pred, int mode /*0 count, 1 and, 2 or*/) {
    State& s = S(); Fiber& me = *s.cur;
    const int par = (int)(me.red_n++ & 1u);
    if (pred) s.red_cnt[par]++;
    block_barrier();
    const int c = s.red_cnt[par], n = s.alive;
    block_barrier();
    s.red_cnt[par] = 0;                       // every thread zeroes it again; nobody accumulates into this parity before all have
    return mode == 0 ? c : mode == 1 ? (c == n) : (c != 0);
}
template <class T> inline T warp_exchange(T v, int src_lane) {     // value of `src_lane` (own value when that lane is gone)
    State& s = S(); Fiber& me = *s.cur; Warp& w = s.warps[me.warp];
    uint64_t raw = 0; memcpy(&raw, &v, sizeof(T));
    w.buf[me.lane] = raw;
    warp_barrier();
    const int idx = me.warp * 32 + src_lane;
    const bool ok = src_lane >= 0 && src_lane < 32 && idx < s.nthreads && !s.fibers[idx].done;
    T r = v; if (ok) memcpy(&r, &w.buf[src_lane], sizeof(T));
    warp_barrier();
    return r;
}
template <class F> inline uint64_t warp_fold(uint64_t v, F f) {    // f folded over the live lanes' values, lane order
    State& s = S(); Fiber& me = *s.cur; Warp& w = s.warps[me.warp];
    w.buf[me.lane] = v;
    warp_barrier();
    uint64_t acc = 0; bool first = true;
    for (int l = 0; l < 32; l++) { const int idx = me.warp * 32 + l; if (idx >= s.nthreads || s.fibers[idx].done) continue; acc = first ? w.buf[l] : f(acc, w.buf[l]); first = false; }
    warp_barrier();
    return acc;
}
inline unsigned warp_ballot(int pred) {
    State& s = S(); Fiber& me = *s.cur; Warp& w = s.warps[me.warp];
    w.buf[me.lane] = pred ? 1 : 0;
    warp_barrier();
    unsigned m = 0;
    for (int l = 0; l < 32; l++) { const int idx = me.warp * 32 + l; if (idx < s.nthreads && !s.fibers[idx].done && w.buf[l]) m |= 1u << l; }
    warp_barrier();
    return m;
}

inline void thread_exit(State& s, Fiber& me) {       // a finished thread no longer counts for any barrier
    me.done = true;
    Warp& w = s.warps[me.warp];
    if (--w.alive > 0 && w.arrived == w.alive) release_warp(w);
    if (--s.alive > 0 && s.arrived == s.alive) release_block(s);
}
inline void trampoline() { State& s = S(); (*s.body)(); thread_exit(s, *s.cur); ctx_switch(s.cur->ctx, s.sched); die("a finished thread was resumed"); }

inline bool runnable(const State& s, const Fiber& f) {
    if (f.done) return false;
    if (f.wait == 1) return s.bar_gen >= f.blk_gen;
    if (f.wait == 2) return s.warps[f.warp].gen >= f.warp_gen;
    return true;
}

inline void launch(dim3 grid, dim3 block, size_t smem, const std::function<void()>& body) {
    State& s = S();
    std::lock_guard<std::mutex> lk(s.mu);
    if (block.y != 1 || block.z != 1 || grid.y != 1 || grid.z != 1) die("only 1-D launches are modelled");
    if (smem > kDynSmem) die("dynamic shared memory request too large");
    const int T = (int)block.x, W = (T + 31) / 32;
    if ((int)s.fibers.size() < T) { size_t o = s.fibers.size(); s.fibers.resize(T); for (size_t i = o; i < (size_t)T; i++) s.fibers[i].stack = (char*)malloc(kStack); }
    s.warps.assign(W, Warp());
    s.grid = grid; s.block = block; s.nthreads = T; s.body = &body; s.launches++;
    for (unsigned b = 0; b < grid.x; b++) {
        s.bid = dim3(b); s.alive = T; s.arrived = 0; s.bar_gen = 0; s.red_cnt[0] = s.red_cnt[1] = 0;
        memset(g_dyn, 0xCD, smem ? smem : 16);
        if (__start_fbgpu_smem && __stop_fbgpu_smem > __start_fbgpu_smem) memset(__start_fbgpu_smem, 0xCD, (size_t)(__stop_fbgpu_smem - __start_fbgpu_smem));
        for (int w = 0; w < W; w++) { s.warps[w] = Warp(); s.warps[w].alive = std::min(32, T - 32 * w); }
        for (int t = 0; t < T; t++) {
            Fiber& f = s.fibers[t];
            f.done = false; f.tid = dim3((unsigned)t); f.lane = t & 31; f.warp = t >> 5; f.blk_gen = f.warp_gen = 0; f.wait = 0; f.red_n = 0;
            ctx_make(f.ctx, f.stack, kStack, trampoline);
        }
        int left = T, idle_scans = 0;
        while (left > 0) {
            bool ran = false;
            for (int k = 0; k < T; k++) {
                // FBGPU_EMU_ORDER=reverse|random: the order in which runnable threads get the CPU between barriers.  Results
                // must not depend on it; a missing barrier between a producer and a consumer phase usually does.
                const int t = s.order == 1 ? T - 1 - k : (s.order == 2 && (T & (T - 1)) == 0) ? (int)((k * 2654435761u + s.salt) % (unsigned)T) : k;   // (odd multiplier: a permutation of a power-of-two block)
                if (s.order == 2 && k == T - 1) s.salt = s.salt * 1664525u + 1013904223u;
                Fiber& f = s.fibers[t];
                if (!runnable(s, f)) continue;
                s.cur = &f; ran = true;
                ctx_switch(s.sched, f.ctx);
                if (f.done) left--;
            }
            if (!ran && ++idle_scans > 1) die("deadlock: no thread of the block can make progress (divergent barrier?)");
            if (ran) idle_scans = 0;
        }
    }
    s.cur = nullptr; s.body = nullptr;
}

// ---- shared-memory "addresses": 32-bit offsets from a base 2 GiB below the dynamic buffer (statics of this library are near it)
inline uintptr_t smem_base() { return (uintptr_t)g_dyn - (1ull << 31); }
inline uint32_t* sptr(uint32_t a) { return (uint32_t*)(smem_base() + a); }
inline void red_or(uint32_t a, uint32_t m) { *sptr(a) |= m; }
inline void red_and(uint32_t a, uint32_t m) { *sptr(a) &= m; }
inline void sts_u32(uint32_t a, uint32_t v) { *sptr(a) = v; }
inline uint32_t lds_u32(uint32_t a) { return *sptr(a); }
inline void red_xor(uint32_t a, uint32_t m) { *sptr(a) ^= m; }

}  // namespace emu

#define threadIdx (emu::S().cur->tid)
#define blockIdx (emu::S().bid)
#define blockDim (emu::S().block)
#define gridDim (emu::S().grid)

// ---- device builtins
static inline void __syncthreads() { emu::block_barrier(); }
static inline int __syncthreads_count(int p) { return emu::block_reduce(p, 0); }
static inline int __syncthreads_and(int p) { return emu::block_reduce(p, 1); }
static inline int __syncthreads_or(int p) { return emu::block_reduce(p, 2); }
static inline void __syncwarp(unsigned = 0xffffffffu) { emu::warp_barrier(); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}
static inline void __threadfence_system() {}
template <class T> static inline T __shfl_sync(unsigned, T v, int src, int = 32) { return emu::warp_exchange(v, src & 31); }
template <class T> static inline T __shfl_up_sync(unsigned, T v, unsigned d, int = 32) { int l = emu::S().cur->lane; return emu::warp_exchange(v, l - (int)d >= 0 ? l - (int)d : l); }
template <class T> static inline T __shfl_down_sync(unsigned, T v, unsigned d, int = 32) { int l = emu::S().cur->lane; return emu::warp_exchange(v, l + (int)d < 32 ? l + (int)d : l); }
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int m, int = 32) { return emu::warp_exchange(v, emu::S().cur->lane ^ m); }
static inline unsigned __ballot_sync(unsigned, int p) { return emu::warp_ballot(p); }
static inline int __any_sync(unsigned, int p) { return emu::warp_ballot(p) != 0; }
static inline unsigned __reduce_add_sync(unsigned, unsigned v) { return (unsigned)emu::warp_fold(v, [](uint64_t a, uint64_t b) { return (uint64_t)(uint32_t)(a + b); }); }
static inline unsigned __reduce_or_sync(unsigned, unsigned v) { return (unsigned)emu::warp_fold(v, [](uint64_t a, uint64_t b) { return a | b; }); }
static inline unsigned __reduce_and_sync(unsigned, unsigned v) { return (unsigned)emu::warp_fold(v, [](uint64_t a, uint64_t b) { return a & b; }); }
static inline unsigned __reduce_max_sync(unsigned, unsigned v) { return (unsigned)emu::warp_fold(v, [](uint64_t a, uint64_t b) { return a > b ? a : b; }); }
static inline unsigned __reduce_min_sync(unsigned, unsigned v) { return (unsigned)emu::warp_fold(v, [](uint64_t a, uint64_t b) { return a < b ? a : b; }); }

static inline long long clock64() { struct timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return (long long)ts.tv_sec * 1000000000ll + ts.tv_nsec; }   // "cycles" = ns
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __ffsll(long long v) { return __builtin_ffsll(v); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline int __clzll(long long v) { return v ? __builtin_clzll((unsigned long long)v) : 64; }
static inline unsigned __brev(unsigned v) { unsigned r = 0; for (int i = 0; i < 32; i++) r |= ((v >> i) & 1u) << (31 - i); return r; }
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((unsigned long long)a * b) >> 32); }
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned s) { s &= 31; return s ? (hi << s) | (lo >> (32 - s)) : hi; }
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) { s &= 31; return s ? (lo >> s) | (hi << (32 - s)) : lo; }
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline size_t __cvta_generic_to_shared(const void* p) { return (size_t)(uint32_t)((uintptr_t)p - emu::smem_base()); }
using std::max;
using std::min;

namespace emu { template <class T> struct same { typedef T type; }; }
#define EMU_V(T) typename emu::same<T>::type
template <class T> static inline T atomicAdd(T* p, EMU_V(T) v) { T o = *p; *p = o + v; return o; }
template <class T> static inline T atomicOr(T* p, EMU_V(T) v) { T o = *p; *p = o | v; return o; }
template <class T> static inline T atomicAnd(T* p, EMU_V(T) v) { T o = *p; *p = o & v; return o; }
template <class T> static inline T atomicXor(T* p, EMU_V(T) v) { T o = *p; *p = o ^ v; return o; }
template <class T> static inline T atomicMin(T* p, EMU_V(T) v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> static inline T atomicMax(T* p, EMU_V(T) v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> static inline T atomicExch(T* p, EMU_V(T) v) { T o = *p; *p = v; return o; }
template <class T> static inline T atomicCAS(T* p, EMU_V(T) c, EMU_V(T) v) { T o = *p; if (o == c) *p = v; return o; }

// ---- host runtime: device memory is host memory, streams are synchronous
typedef int cudaError_t;
typedef struct emuStream* cudaStream_t;
typedef struct emuEvent { std::chrono::steady_clock::time_point t; }* cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorMemoryAllocation = 2, cudaErrorPeerAccessAlreadyEnabled = 704, cudaErrorNotSupported = 801 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum { cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2, cudaIpcMemLazyEnablePeerAccess = 1 };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8 };
struct cudaDeviceProp { char name[256]; size_t totalGlobalMem; int multiProcessorCount, major, minor; size_t sharedMemPerBlockOptin, sharedMemPerMultiprocessor; int l2CacheSize, clockRate; };
struct cudaIpcMemHandle_t { char reserved[64]; };

static inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : e == cudaErrorNotSupported ? "operation not supported by the CPU emulation" : "emulated CUDA error"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceCount(int* n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDeviceProperties(cudaDeviceProp* p, int) {
    memset(p, 0, sizeof(*p)); snprintf(p->name, sizeof(p->name), "fbgpu CPU kernel emulation (tests only)");
    p->totalGlobalMem = 8ull << 30; p->multiProcessorCount = 3; p->major = 10; p->minor = 0; p->sharedMemPerBlockOptin = emu::kDynSmem; p->sharedMemPerMultiprocessor = emu::kDynSmem; p->l2CacheSize = 1 << 20; p->clockRate = 1000000;
    return cudaSuccess;
}
// "Device" allocations end flush against an inaccessible page (size rounded up to 16 bytes, the granularity the kernels'
// vector loads rely on), so a kernel or a copy that runs past the end of a buffer faults at once — the interpreter's
// stand-in for compute-sanitizer's memcheck on over-runs.  Contents start as 0xA5 garbage, like fresh device memory.
namespace emu {
struct Allocs { std::mutex mu; std::unordered_map<void*, std::pair<void*, size_t>> m; };
inline Allocs g_allocs;
}
static inline cudaError_t cudaMalloc(void** p, size_t n) {
    const size_t page = 4096, body = (std::max<size_t>(n, 1) + 15) & ~(size_t)15, len = ((body + page - 1) / page + 1) * page;
    char* base = (char*)mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
    if (base == (char*)MAP_FAILED) return cudaErrorMemoryAllocation;
    mprotect(base + len - page, page, PROT_NONE);
    *p = base + len - page - body;
    memset(*p, 0xA5, body);
    std::lock_guard<std::mutex> lk(emu::g_allocs.mu);
    emu::g_allocs.m[*p] = std::make_pair((void*)base, len);
    return cudaSuccess;
}
template <class T> static inline cudaError_t cudaMalloc(T** p, size_t n) { return cudaMalloc((void**)p, n); }
static inline cudaError_t cudaFree(void* p) {
    if (!p) return cudaSuccess;
    std::lock_guard<std::mutex> lk(emu::g_allocs.mu);
    auto it = emu::g_allocs.m.find(p);
    if (it == emu::g_allocs.m.end()) emu::die("cudaFree of a pointer cudaMalloc did not return");
    munmap(it->second.first, it->second.second);
    emu::g_allocs.m.erase(it);
    return cudaSuccess;
}
static inline cudaError_t cudaMallocHost(void** p, size_t n) { *p = aligned_alloc(256, (n + 255) & ~(size_t)255); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
template <class T> static inline cudaError_t cudaMallocHost(T** p, size_t n) { return cudaMallocHost((void**)p, n); }
static inline cudaError_t cudaFreeHost(void* p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void* d, const void* s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void* d, const void* s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void* d, int v, size_t n) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* d, int v, size_t n, cudaStream_t = nullptr) { if (n) memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) { *s = (cudaStream_t)malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t* e) { *e = new emuEvent(); return cudaSuccess; }
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) { *e = new emuEvent(); return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { delete e; return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t = nullptr) { e->t = std::chrono::steady_clock::now(); return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float* ms, cudaEvent_t a, cudaEvent_t b) { *ms = std::chrono::duration<float, std::milli>(b->t - a->t).count(); return cudaSuccess; }
template <class F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
template <class F> static inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int* n, F, int, size_t) { *n = 2; return cudaSuccess; }
static inline cudaError_t cudaIpcGetMemHandle(cudaIpcMemHandle_t*, void*) { return cudaErrorNotSupported; }
static inline cudaError_t cudaIpcOpenMemHandle(void**, cudaIpcMemHandle_t, unsigned) { return cudaErrorNotSupported; }
static inline cudaError_t cudaIpcCloseMemHandle(void*) { return cudaErrorNotSupported; }
static inline cudaError_t cudaDeviceCanAccessPeer(int* can, int, int) { *can = 1; return cudaSuccess; }
static inline cudaError_t cudaDeviceEnablePeerAccess(int, unsigned) { return cudaSuccess; }
