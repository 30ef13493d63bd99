// libfbgpu host runtime: shard store residency, bitmap-call program compiler, query entry points (C ABI in
// include/fbgpu.h).  C++17 + CUDA runtime only — no torch types, no CPU fallback: every query runs the
// sm_90a kernels in kernels.cuh or fails with FBGPU_E_CUDA.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <condition_variable>
#include <map>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <atomic>
#include <deque>
#include <functional>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/fbgpu.h"
#include "fbgpu_types.h"
#include "kernels.cuh"
#include "stripe.h"
#include "rbf_reader.h"
#include "program_compiler.h"
#include "roaring_parse.h"

using namespace fbgpu;

// ------------------------------------------------------------------ errors
static thread_local std::string g_err;
static int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof buf, fmt, ap); va_end(ap);
    g_err = buf;
    return code;
}
#define CUDA_TRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return fail(FBGPU_E_CUDA, "%s failed: %s (%s:%d)", #x, cudaGetErrorString(_e), __FILE__, __LINE__); } while (0)

// no C++ exception may cross the C boundary (the caller is cgo): every int-returning entry point is a function-try-block
#define FBGPU_CATCH \
    catch (const std::bad_alloc&) { return fail(FBGPU_E_NOMEM, "out of host memory"); } \
    catch (const std::exception& e) { return fail(FBGPU_E_INVALID, "internal error: %s", e.what()); } \
    catch (...) { return fail(FBGPU_E_INVALID, "internal error"); }

// every entry point that needs the GPU: an inspection-only context (FBGPU_DEVICE_NONE) is refused here, loudly
#define USE_DEVICE(c) do { if ((c)->inspect_only) return fail(FBGPU_E_CUDA, "this context was created with FBGPU_DEVICE_NONE: it holds no device and answers no query"); \
                           CUDA_TRY(cudaSetDevice((c)->device)); } while (0)

extern "C" const char* fbgpu_last_error(void) { return g_err.c_str(); }
extern "C" int32_t fbgpu_abi_version(void) { return FBGPU_ABI_VERSION; }

// ------------------------------------------------------------------ small device buffer helper
struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    int ensure(size_t n) {
        if (n <= cap) return 0;
        size_t nc = std::max(n, cap + cap / 2);
        nc = (nc + 255) & ~size_t(255);
        void* q = nullptr;
        if (cudaMalloc(&q, nc) != cudaSuccess) { cudaGetLastError(); if (cudaMalloc(&q, (n + 255) & ~size_t(255)) != cudaSuccess) return fail(FBGPU_E_NOMEM, "cudaMalloc(%zu) failed", n); nc = (n + 255) & ~size_t(255); }
        if (p) cudaFree(p);
        p = q; cap = nc;
        return 0;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};
struct PinBuf {
    void* p = nullptr; size_t cap = 0;
    int ensure(size_t n) {
        if (n <= cap) return 0;
        size_t nc = std::max(n, cap * 2);
        void* q = nullptr;
        if (cudaMallocHost(&q, nc) != cudaSuccess) return fail(FBGPU_E_NOMEM, "cudaMallocHost(%zu) failed", nc);
        if (p) cudaFreeHost(p);
        p = q; cap = nc;
        return 0;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
};

// growable host byte buffer without value-initialisation (std::vector::resize would write every byte twice)
struct RawBuf {
    uint8_t* p = nullptr; size_t len = 0, cap = 0;
    bool empty() const { return len == 0; }
    size_t size() const { return len; }
    int reserve(size_t n) {
        if (n <= cap) return 0;
        size_t nc = std::max(n, cap + cap / 2);
        uint8_t* q = (uint8_t*)realloc(p, nc);
        if (!q) return fail(FBGPU_E_NOMEM, "host staging realloc(%zu) failed", nc);
        p = q; cap = nc; return 0;
    }
    void clear_and_free() { free(p); p = nullptr; len = cap = 0; }
};
struct PayloadCopy { const uint8_t* src; uint64_t dst; uint32_t bytes, padded; uint16_t typ; uint16_t official_run; uint32_t cnt; uint32_t stripe; };   // dst: offset inside the staging buffer

// ------------------------------------------------------------------ NCCL (resolved at run time)
struct Id128 { char b[128]; };   // ncclUniqueId is passed by value (128 bytes)
struct NcclApi {
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, Id128, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
static NcclApi g_nccl; static std::once_flag g_nccl_once;
static bool nccl_load() {
    std::call_once(g_nccl_once, [] {
        const char* names[] = { "libnccl.so.2", "libnccl.so" };
        for (const char* n : names) { g_nccl.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (g_nccl.lib) break; }
        if (!g_nccl.lib) return;
        g_nccl.GetUniqueId = (int (*)(void*))dlsym(g_nccl.lib, "ncclGetUniqueId");
        g_nccl.CommInitRank = (int (*)(void**, int, Id128, int))dlsym(g_nccl.lib, "ncclCommInitRank");
        g_nccl.AllReduce = (int (*)(const void*, void*, size_t, int, int, void*, cudaStream_t))dlsym(g_nccl.lib, "ncclAllReduce");
        g_nccl.CommDestroy = (int (*)(void*))dlsym(g_nccl.lib, "ncclCommDestroy");
        g_nccl.GetErrorString = (const char* (*)(int))dlsym(g_nccl.lib, "ncclGetErrorString");
    });
    return g_nccl.lib && g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.AllReduce && g_nccl.CommDestroy;
}
constexpr int kNcclUint64 = 5, kNcclSum = 0;   // ncclDataType_t / ncclRedOp_t values (nccl.h)

// ------------------------------------------------------------------ context
struct ViewKey { uint32_t index, field, view; bool operator<(const ViewKey& o) const { return index != o.index ? index < o.index : field != o.field ? field < o.field : view < o.view; } };

struct Extent { uint64_t off, len; };
struct HostFrag { uint32_t fv; uint64_t shard; bool live; uint32_t row_off, n_rows; uint64_t payload_bytes; uint32_t n_desc; uint32_t n_arr, n_bmp, n_run; uint32_t n_striped;
                  uint64_t desc_off = 0;               // its descriptors are h_descs[desc_off, desc_off + n_desc)
                  uint64_t arena_off = 0, arena_len = 0;      // the payloads it brought (with their alignment gaps) are arena bytes [arena_off, arena_off + arena_len)
                  // a fragment produced by fbgpu_apply_containers keeps the untouched containers of its predecessor where they are:
                  std::vector<Extent> inherited;       // arena extents taken over from the predecessors (theirs to free with this fragment)
                  uint64_t hole_bytes = 0;             // bytes inside those extents no descriptor points at any more (already counted in dead_arena)
                  bool stripe_policy = false; };       // arrays of this fragment are stored bank-striped (decided at its first load, kept by updates)

struct Workspace {
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    DevBuf d_in, d_counts, d_bitmaps, d_info, d_emit_units, d_emit, d_rows, d_aux;
    DevBuf d_select;                     // fbgpu_bsi_select: per-rank candidate bitmaps of every unit of the call
    DevBuf d_present;                    // fbgpu_groupby_distinct: one leaf's presence bitset, (cell, listed value of x) -> present
    DevBuf d_sort;                       // fbgpu_bsi_sort: (key, column) pairs, two halves (SortPairs)
    DevBuf d_cells;                      // fbgpu_extract_rows: per window column of a batch, its number of rows, then its place in the chunk's pairs
    PinBuf h_in, h_out;
    bool busy = false;
};

struct fbgpu_ctx {
    int device = 0;
    int sm_count = 132;                  // H100 SXM; replaced by the device's own count in fbgpu_init
    // ---- store (host mirrors are the source of truth for metadata; payload lives only in HBM once committed)
    std::shared_mutex store_mu;
    std::map<ViewKey, uint32_t> view_ids;
    std::vector<std::vector<int32_t>> shardmaps;  // per view
    std::vector<uint64_t> view_arr, view_other;   // per view: live array containers / bitmap+run containers
    std::vector<uint64_t> view_striped;           // per view: live array containers stored in bank-striped order (stripe.h)
    std::vector<HostFrag> frags;
    std::vector<FragHdr> h_frags;
    std::vector<RowEnt> h_rows;
    std::vector<ContDesc> h_descs;
    RawBuf staging;                      // payload bytes not yet uploaded, destined for [uploaded, uploaded+staging.len)
    uint64_t uploaded = 0;               // bytes of payload already in HBM
    uint64_t dead_arena = 0;             // arena bytes of replaced / dropped fragments (reclaimed by compact_locked)
    bool meta_dirty = false;
    // incremental commit: the host tables t_* are kept between commits; a commit after a few loads / drops / container updates patches the
    // entries of the touched (view, shard) pairs and uploads the tails of the append-only mirrors instead of rebuilding and re-sending everything
    bool tables_valid = false;            // t_views / t_flat / t_rowtab describe the mirrors except for `dirty_shards`
    bool dev_tables_valid = false;        // the device tables equal the host tables as of the last commit
    std::vector<std::pair<uint32_t, uint64_t>> dirty_shards;
    size_t dev_rows = 0, dev_descs = 0, dev_frags = 0;   // prefix of h_rows / h_descs / h_frags already in HBM
    bool inspect_only = false;           // created with FBGPU_DEVICE_NONE: residency + fbgpu_debug_container only, no device, no queries
    std::vector<ViewTab> t_views; std::vector<int32_t> t_flat; std::vector<RowTabEnt> t_rowtab;   // inspect_only: the tables a commit would upload
    bool stripe_arrays = getenv("FBGPU_ARRAY_SORTED") == nullptr;    // bank-striped array payload order (stripe.h) unless FBGPU_ARRAY_SORTED=1 (fixed per context)
    // (shard, slot) units whose result bitmaps are materialised per launch by the row-returning / aggregate / filtered entry
    // points: 16384 units = 1024 shards = 128 MiB of workspace per lease.  FBGPU_UNIT_BATCH (a multiple of 16, fixed per
    // context) trades workspace for launches; the tests set it small to walk the multi-batch paths with a handful of shards.
    long long unit_batch = [] { const char* e = getenv("FBGPU_UNIT_BATCH"); const long long n = e ? atoll(e) : 0; return n >= 16 ? (n / 16) * 16 : 16384ll; }();
    int gd_ctas_per_sm = 3;               // resident CTAs of groupby_direct_kernel per SM
    int pair_ctas_per_sm = 2;             // resident CTAs of pair_count_kernel per SM (occupancy query at init)
    std::atomic<uint64_t> counters_pair_launches{0};      // Count(Intersect(Row, Row)) queries that took the fused pair kernel
    DevBuf d_payload, d_views, d_shardmap, d_frags, d_rows, d_descs, d_rowtab;
    PinBuf bounce[2];
    uint32_t n_views_dev = 0;
    fbgpu_stats stats{};
    // ---- execution
    std::mutex ws_mu; std::condition_variable ws_cv;
    std::vector<std::unique_ptr<Workspace>> wss;
    // ---- counters
    std::mutex cnt_mu; fbgpu_counters counters{};
    // ---- comm
    void* comm = nullptr; int n_ranks = 1, rank = 0;
    // fused peer-memory reduce (Count)
    Mailbox* mbox = nullptr; Mailbox* peers[kMaxRanks] = {}; DevBuf d_peers; bool p2p = false; bool peers_local = false; unsigned long long epoch = 0; std::mutex coll_mu;
    // bound of the in-kernel wait for one peer's count (FBGPU_P2P_TIMEOUT_MS, default 2000 ms at ~2 GHz)
    long long p2p_timeout_cycles = [] { const char* e = getenv("FBGPU_P2P_TIMEOUT_MS"); const long long ms = e ? atoll(e) : 2000; return (ms > 0 ? ms : 2000) * 2000000ll; }();
};

static StoreRef store_ref(fbgpu_ctx* c) {
    StoreRef s;
    s.views = (const ViewTab*)c->d_views.p; s.shardmap = (const int32_t*)c->d_shardmap.p; s.frags = (const FragHdr*)c->d_frags.p;
    s.rows = (const RowEnt*)c->d_rows.p; s.descs = (const ContDesc*)c->d_descs.p; s.payload = (const uint8_t*)c->d_payload.p; s.rowtab = (const RowTabEnt*)c->d_rowtab.p; s.n_views = c->n_views_dev;
    return s;
}

extern "C" int fbgpu_init(int32_t device_ordinal, fbgpu_ctx** out) try {
    if (!out) return fail(FBGPU_E_INVALID, "out is null");
    if (device_ordinal == FBGPU_DEVICE_NONE) {          // store inspection without a device (tests): no CUDA call is ever made
        auto c = new fbgpu_ctx(); c->inspect_only = true; c->device = -1;
        *out = c;
        return FBGPU_OK;
    }
    int n = 0;
    CUDA_TRY(cudaGetDeviceCount(&n));
    if (device_ordinal < 0 || device_ordinal >= n) return fail(FBGPU_E_INVALID, "device ordinal %d out of range (%d devices)", device_ordinal, n);
    CUDA_TRY(cudaSetDevice(device_ordinal));
    auto c = new fbgpu_ctx();
    struct Guard { fbgpu_ctx* c; ~Guard() { if (c) fbgpu_shutdown(c); } } guard{ c };     // a failing step below must not leak the context
    c->device = device_ordinal;
    cudaDeviceProp p; CUDA_TRY(cudaGetDeviceProperties(&p, device_ordinal));
    c->sm_count = p.multiProcessorCount;
    for (int i = 0; i < 4; i++) {
        auto w = std::make_unique<Workspace>();
        CUDA_TRY(cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking));
        CUDA_TRY(cudaEventCreate(&w->ev0)); CUDA_TRY(cudaEventCreate(&w->ev1));
        c->wss.push_back(std::move(w));
    }
    // opt in to large dynamic shared memory once
    CUDA_TRY(cudaFuncSetAttribute(eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 17 * 8192));
    CUDA_TRY(cudaFuncSetAttribute(pair_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPcWarps * 8192));
    CUDA_TRY(cudaFuncSetAttribute(row_count_kernel<RcOut::kSummed>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPairWarps * 8192));
    CUDA_TRY(cudaFuncSetAttribute(row_count_kernel<RcOut::kPerShard>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPairWarps * 8192));
    CUDA_TRY(cudaFuncSetAttribute(row_count_kernel<RcOut::kCutoff>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPairWarps * 8192));
    CUDA_TRY(cudaFuncSetAttribute(row_count_views_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kPairWarps * 8192));
    CUDA_TRY(cudaFuncSetAttribute(groupby_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGbSlots * 4 + 8192));
    CUDA_TRY(cudaFuncSetAttribute(groupby_direct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kGdSmemBytes));
    { int nb = 0; if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, groupby_direct_kernel, kGdThreads, kGdSmemBytes) == cudaSuccess && nb > 0) c->gd_ctas_per_sm = nb; }
    { int nb = 0; if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, pair_count_kernel, kPcWarps * 32, kPcWarps * 8192) == cudaSuccess && nb > 0) c->pair_ctas_per_sm = nb; }
    guard.c = nullptr;
    *out = c;
    return FBGPU_OK;
} FBGPU_CATCH

extern "C" void fbgpu_shutdown(fbgpu_ctx* c) {
    if (!c) return;
    if (c->inspect_only) { c->staging.clear_and_free(); delete c; return; }
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    if (c->comm && nccl_load()) g_nccl.CommDestroy(c->comm);
    for (auto& w : c->wss) {
        for (DevBuf* b : { &w->d_in, &w->d_counts, &w->d_bitmaps, &w->d_info, &w->d_emit_units, &w->d_emit, &w->d_rows, &w->d_aux, &w->d_select, &w->d_present, &w->d_sort, &w->d_cells }) b->release();
        w->h_in.release(); w->h_out.release();
        if (w->ev0) cudaEventDestroy(w->ev0);
        if (w->ev1) cudaEventDestroy(w->ev1);
        if (w->stream) cudaStreamDestroy(w->stream);
    }
    for (DevBuf* b : { &c->d_payload, &c->d_views, &c->d_shardmap, &c->d_frags, &c->d_rows, &c->d_descs, &c->d_rowtab }) b->release();
    c->bounce[0].release(); c->bounce[1].release(); c->staging.clear_and_free();
    for (int p = 0; p < kMaxRanks; p++) if (c->peers[p] && c->peers[p] != c->mbox && !c->peers_local) cudaIpcCloseMemHandle(c->peers[p]);   // peer mailboxes mapped by fbgpu_comm_p2p_open
    if (c->mbox) cudaFree(c->mbox);
    c->d_peers.release();
    delete c;
}

struct WsLease {
    fbgpu_ctx* c; Workspace* w;
    bool ok = false;        // set on the success path; otherwise the destructor drains the stream, so that work queued
                            // before an error return cannot still be running when the next query reuses the buffers
    explicit WsLease(fbgpu_ctx* ctx) : c(ctx), w(nullptr) {
        std::unique_lock<std::mutex> lk(c->ws_mu);
        for (;;) { for (auto& x : c->wss) if (!x->busy) { x->busy = true; w = x.get(); return; } c->ws_cv.wait(lk); }
    }
    ~WsLease() { if (!ok) cudaStreamSynchronize(w->stream); { std::lock_guard<std::mutex> lk(c->ws_mu); w->busy = false; } c->ws_cv.notify_one(); }
};

// ------------------------------------------------------------------ fragment parsing (roaring_parse.h)
static int parse_roaring(const uint8_t* buf, uint64_t len, std::vector<ParsedCont>& out) {
    Error err;
    int rc = parse_roaring(buf, len, out, err);
    return rc ? fail(rc, "%s", err.msg) : 0;
}

static uint32_t view_id_locked(fbgpu_ctx* c, ViewKey k, bool create) {
    auto it = c->view_ids.find(k);
    if (it != c->view_ids.end()) return it->second;
    if (!create) return kNoView;
    uint32_t id = (uint32_t)c->shardmaps.size();
    c->view_ids[k] = id; c->shardmaps.emplace_back(); c->view_arr.push_back(0); c->view_other.push_back(0); c->view_striped.push_back(0);
    return id;
}

// `successor_keeps_arena`: the fragment is being superseded by fbgpu_apply_containers — its arena extents go to the new fragment
static void drop_locked(fbgpu_ctx* c, uint32_t fv, uint64_t shard, bool successor_keeps_arena = false) {
    auto& sm = c->shardmaps[fv];
    if (shard >= sm.size() || sm[shard] < 0) return;
    HostFrag& f = c->frags[sm[shard]];
    f.live = false;
    if (!successor_keeps_arena) {
        uint64_t own = f.arena_len; for (const Extent& e : f.inherited) own += e.len;
        c->dead_arena += own - f.hole_bytes; c->stats.dead_bytes = c->dead_arena;
    }
    c->stats.fragments--; c->stats.containers -= f.n_desc; c->stats.payload_bytes -= f.payload_bytes;
    c->stats.array_containers -= f.n_arr; c->stats.bitmap_containers -= f.n_bmp; c->stats.run_containers -= f.n_run;
    c->view_arr[fv] -= f.n_arr; c->view_other[fv] -= (uint64_t)f.n_bmp + f.n_run; c->view_striped[fv] -= f.n_striped;
    sm[shard] = -1;
    c->meta_dirty = true;
    c->dirty_shards.emplace_back(fv, shard);
}

// A load is all-or-nothing (ADVICE r1): the entry points open a StoreTxn before the first mutation; unless commit() is reached
// (every fragment appended AND every payload copied), its destructor puts the host mirrors back exactly as they were —
// vector lengths, the claimed staging space, statistics, the shard-map entries and the liveness of replaced fragments.
// store_mu is held exclusively for the whole life of the object.
struct StoreTxn {
    fbgpu_ctx* c;
    size_t n_rows, n_descs, n_frags, n_hfrags; uint64_t staging_len, dead_arena; fbgpu_stats stats; bool meta_dirty;
    std::vector<uint64_t> view_arr, view_other, view_striped;
    struct Undo { uint32_t fv; uint64_t shard; int32_t old_fid; size_t old_size; };
    std::vector<Undo> undo;
    bool done = false;
    explicit StoreTxn(fbgpu_ctx* ctx) : c(ctx), n_rows(ctx->h_rows.size()), n_descs(ctx->h_descs.size()), n_frags(ctx->frags.size()), n_hfrags(ctx->h_frags.size()),
        staging_len(ctx->staging.len), dead_arena(ctx->dead_arena), stats(ctx->stats), meta_dirty(ctx->meta_dirty),
        view_arr(ctx->view_arr), view_other(ctx->view_other), view_striped(ctx->view_striped) {}
    void note(uint32_t fv, uint64_t shard) {
        auto& sm = c->shardmaps[fv];
        undo.push_back(Undo{ fv, shard, shard < sm.size() ? sm[shard] : -1, sm.size() });
    }
    void commit() { done = true; }
    ~StoreTxn() {
        if (done) return;
        for (size_t k = undo.size(); k-- > 0;) {
            const Undo& u = undo[k]; auto& sm = c->shardmaps[u.fv];
            if (sm.size() > u.old_size) sm.resize(u.old_size);
            if (u.shard < sm.size()) sm[u.shard] = u.old_fid;
            if (u.old_fid >= 0) c->frags[(size_t)u.old_fid].live = true;
        }
        c->h_rows.resize(n_rows); c->h_descs.resize(n_descs); c->frags.resize(n_frags); c->h_frags.resize(n_hfrags);
        c->staging.len = staging_len; c->dead_arena = dead_arena; c->stats = stats; c->meta_dirty = meta_dirty;
        // (views created by the failed call stay, empty: resize the snapshots up to the current number of views)
        view_arr.resize(c->view_arr.size(), 0); view_other.resize(c->view_other.size(), 0); view_striped.resize(c->view_striped.size(), 0);
        c->view_arr = view_arr; c->view_other = view_other; c->view_striped = view_striped;
        c->tables_valid = false;            // (dirty_shards may name pairs of the undone call: the next commit rebuilds the tables)
    }
};

// Bytes kept allocated behind the last payload byte of the arena: pair_count_kernel loads three 16-byte chunks per lane of a small array
// without looking at its length (up to 1.5 KiB past a one-chunk array) and only USES the chunks the array has.
constexpr uint64_t kArenaSlack = 4096;

// Shard ids index the dense per-view shard maps: the accepted range is bounded so that one stray id cannot make a load allocate
// gigabytes of map (the reference's shard space is sparse; 2^24 shards = 1.7e13 columns per index is far past its deployments).
constexpr uint64_t kMaxShard = 1ull << 24;

static inline uint64_t cont_bytes(uint16_t typ, uint32_t n, uint32_t cnt) { return typ == kArray ? (uint64_t)n * 2 : typ == kBitmap ? 8192 : (uint64_t)cnt * 4; }

// one container of a fragment being appended: a parsed one (payload to be copied), or one kept from the predecessor fragment
// (descriptor copied, payload stays where it is in the arena)
struct FragItem { uint64_t key; const ParsedCont* pc; ContDesc kept; };

// appends one fragment to the host mirrors + staging (store_mu held exclusively, inside a StoreTxn).  `pred` != null: the fragment
// supersedes *pred (fbgpu_apply_containers): it takes over pred's arena extents, `new_holes` more bytes of them are unreferenced now
static int add_items_locked(fbgpu_ctx* c, StoreTxn& txn, uint32_t fv, uint64_t shard, const std::vector<FragItem>& items, std::vector<PayloadCopy>& copies,
                            const HostFrag* pred, uint64_t new_holes) {
    if (shard >= kMaxShard) return fail(FBGPU_E_INVALID, "shard %llu too large (limit %llu)", (unsigned long long)shard, (unsigned long long)kMaxShard);
    txn.note(fv, shard);
    HostFrag hf{}; hf.fv = fv; hf.shard = shard; hf.live = true; hf.row_off = (uint32_t)c->h_rows.size(); hf.desc_off = c->h_descs.size();
    if (pred) {             // (read before drop_locked / push_back: `pred` points into c->frags)
        hf.inherited = pred->inherited;
        if (pred->arena_len) hf.inherited.push_back(Extent{ pred->arena_off, pred->arena_len });
        hf.hole_bytes = pred->hole_bytes + new_holes; hf.stripe_policy = pred->stripe_policy;
        c->dead_arena += new_holes; c->stats.dead_bytes = c->dead_arena;
    }
    drop_locked(c, fv, shard, pred != nullptr);
    hf.arena_off = c->uploaded + c->staging.len;
    uint64_t prev_row = ~0ull; bool contiguous = true; uint64_t row0 = 0;
    const size_t desc0 = c->h_descs.size();
    // descriptors: row-major (key order), so that a row's slots are adjacent and rank = popc(mask & below)
    for (const FragItem& it : items) {
        uint64_t row = it.key / kSlotsPerRow; int slot = (int)(it.key % kSlotsPerRow);
        if (row != prev_row) {
            if (prev_row == ~0ull) row0 = row; else if (row != prev_row + 1) contiguous = false;
            RowEnt e{}; e.row = row; e.first_desc = (uint32_t)c->h_descs.size(); e.mask = 0;
            c->h_rows.push_back(e); prev_row = row; hf.n_rows++;
        }
        c->h_rows.back().mask |= (uint16_t)(1u << slot);
        ContDesc d = it.kept;
        if (it.pc) { d = ContDesc{}; d.off16 = 0; d.card = it.pc->n; d.typ = it.pc->typ; d.cnt = (uint16_t)it.pc->cnt; }
        c->h_descs.push_back(d);
        hf.n_desc++; hf.payload_bytes += cont_bytes(d.typ, d.card, d.cnt);
        if (d.typ == kArray) hf.n_arr++; else if (d.typ == kBitmap) hf.n_bmp++; else hf.n_run++;
    }
    // payloads: row-major (key order): a row's 16 containers are contiguous, which is what the common
    // few-rows-of-many query streams.
    // striped order: only for array-dominated fragments, so that bitmap-heavy views (BSI planes) keep every
    // array sorted and stay eligible for the word-parallel kernel, whose slice search needs sorted arrays
    if (!pred) hf.stripe_policy = c->stripe_arrays && (uint64_t)hf.n_arr * 8 > (uint64_t)hf.n_bmp + hf.n_run;
    const bool stripe = hf.stripe_policy;
    if (stripe) for (size_t i = 0; i < items.size(); i++) { const ContDesc& d = c->h_descs[desc0 + i]; if (d.typ == kArray && d.card >= fbgpu_stripe::kMinStripe) hf.n_striped++; }
    for (size_t i = 0; i < items.size(); i++) {
        if (!items[i].pc) continue;                             // kept: its descriptor already points at the payload
        const ParsedCont& pc = *items[i].pc;
        uint64_t pos = c->uploaded + c->staging.len;
        uint64_t align = pc.typ == kBitmap ? 128 : 16;
        uint64_t apos = (pos + align - 1) & ~(align - 1);
        uint64_t bytes = cont_bytes(pc.typ, pc.n, pc.cnt);
        uint64_t padded = (bytes + 15) & ~15ull;
        if (apos / 16 > 0xffffffffull) return fail(FBGPU_E_NOMEM, "payload arena exceeds 64 GiB addressable by 32-bit 16 B offsets");
        c->staging.len += (apos - pos) + padded;            // space is claimed now, bytes are copied by run_copies()
        copies.push_back(PayloadCopy{ pc.data, apos - c->uploaded, (uint32_t)bytes, (uint32_t)padded, pc.typ, (uint16_t)(pc.official_run ? 1 : 0), pc.cnt, stripe ? 1u : 0u });
        c->h_descs[desc0 + i].off16 = (uint32_t)(apos / 16);
    }
    hf.arena_len = c->uploaded + c->staging.len - hf.arena_off;
    FragHdr h{}; h.row_off = hf.row_off; h.n_rows = hf.n_rows; h.row0 = row0; h.contiguous = contiguous ? 1u : 0u;
    int32_t fid = (int32_t)c->frags.size();
    c->stats.fragments++; c->stats.containers += hf.n_desc; c->stats.payload_bytes += hf.payload_bytes;
    c->stats.array_containers += hf.n_arr; c->stats.bitmap_containers += hf.n_bmp; c->stats.run_containers += hf.n_run;
    c->view_arr[fv] += hf.n_arr; c->view_other[fv] += (uint64_t)hf.n_bmp + hf.n_run; c->view_striped[fv] += hf.n_striped;
    c->frags.push_back(std::move(hf)); c->h_frags.push_back(h);
    auto& sm = c->shardmaps[fv];
    if (shard >= sm.size()) sm.resize(shard + 1, -1);
    sm[shard] = fid;
    c->meta_dirty = true;
    c->dirty_shards.emplace_back(fv, shard);
    return 0;
}
static int add_fragment_locked(fbgpu_ctx* c, StoreTxn& txn, uint32_t fv, uint64_t shard, const std::vector<ParsedCont>& cs, std::vector<PayloadCopy>& copies) {
    std::vector<FragItem> items(cs.size());
    for (size_t i = 0; i < cs.size(); i++) items[i] = FragItem{ cs[i].key, &cs[i], ContDesc{} };
    return add_items_locked(c, txn, fv, shard, items, copies, nullptr, 0);
}

// copies the planned payloads into the staging buffer (possibly on several host threads); store_mu held exclusively
static int run_copies(fbgpu_ctx* c, const std::vector<PayloadCopy>& copies, int n_threads) {
    if (c->staging.reserve(c->staging.len + 64)) return FBGPU_E_NOMEM;
    uint8_t* base = c->staging.p;
    auto work = [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; i++) {
            const PayloadCopy& pc = copies[i];
            uint8_t* dst = base + pc.dst;
            if (pc.typ == kArray && pc.stripe) fbgpu_stripe::stripe_array(pc.src, (uint16_t*)dst, pc.bytes / 2);
            else memcpy(dst, pc.src, pc.bytes);
            if (pc.typ == kArray) fbgpu_stripe::pad_array_tail((uint16_t*)dst, pc.bytes / 2, pc.padded / 2);      // tail of the last 16-byte chunk: copies of the last element (stripe.h)
            else if (pc.padded > pc.bytes) memset(dst + pc.bytes, 0, pc.padded - pc.bytes);                      // zero tail
            if (pc.typ == kRun && pc.official_run) {     // official format stores (start, length-1): roaring.go:2240-2247
                uint16_t* r = (uint16_t*)dst; for (uint32_t k = 0; k < pc.cnt; k++) r[2 * k + 1] = (uint16_t)(r[2 * k] + r[2 * k + 1]);
            }
        }
    };
    n_threads = (int)std::min<size_t>(std::max(n_threads, 1), copies.size() / 4096 + 1);
    if (n_threads <= 1) { work(0, copies.size()); return 0; }
    std::vector<std::thread> th;
    for (int t = 0; t < n_threads; t++) th.emplace_back(work, copies.size() * t / n_threads, copies.size() * (t + 1) / n_threads);
    for (auto& t : th) t.join();
    return 0;
}

extern "C" int fbgpu_load_fragment(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, uint64_t shard, const uint8_t* roaring, uint64_t nbytes) try {
    if (!c || !roaring) return fail(FBGPU_E_INVALID, "null argument");
    std::vector<ParsedCont> cs;
    int rc = parse_roaring(roaring, nbytes, cs); if (rc) return rc;
    std::unique_lock<std::shared_mutex> lk(c->store_mu);
    uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, true);
    std::vector<PayloadCopy> copies;
    StoreTxn txn(c);
    rc = add_fragment_locked(c, txn, fv, shard, cs, copies); if (rc) return rc;
    rc = run_copies(c, copies, 1); if (rc) return rc;
    txn.commit();
    return FBGPU_OK;
} FBGPU_CATCH

extern "C" int fbgpu_load_fragments(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, const uint64_t* shards, int64_t n,
                                    const uint8_t* buf, const uint64_t* offsets) try {
    if (!c || !shards || !buf || !offsets || n < 0) return fail(FBGPU_E_INVALID, "null argument");
    // parse in parallel (validation + container tables), then append serially (memcpy-bound)
    std::vector<std::vector<ParsedCont>> parsed((size_t)n);
    std::vector<int> rcs((size_t)n, 0); std::vector<std::string> errs((size_t)n);
    int nt = (int)std::min<int64_t>(std::max(1u, std::thread::hardware_concurrency()), std::max<int64_t>(1, n / 8));
    nt = std::min(nt, 32);
    std::vector<std::thread> th;
    for (int t = 0; t < nt; t++) th.emplace_back([&, t] {
        for (int64_t i = n * t / nt; i < n * (t + 1) / nt; i++) { rcs[i] = parse_roaring(buf + offsets[i], offsets[i + 1] - offsets[i], parsed[i]); if (rcs[i]) errs[i] = g_err; }
    });
    for (auto& t : th) t.join();
    for (int64_t i = 0; i < n; i++) if (rcs[i]) { g_err = errs[i]; return rcs[i]; }
    std::unique_lock<std::shared_mutex> lk(c->store_mu);
    uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, true);
    std::vector<PayloadCopy> copies;
    StoreTxn txn(c);
    for (int64_t i = 0; i < n; i++) { int rc = add_fragment_locked(c, txn, fv, shards[i], parsed[i], copies); if (rc) return rc; }
    int rc = run_copies(c, copies, nt); if (rc) return rc;
    txn.commit();
    return FBGPU_OK;
} FBGPU_CATCH

extern "C" int fbgpu_load_rbf(fbgpu_ctx* c, uint32_t index, uint64_t shard, const uint8_t* data, uint64_t data_bytes, const uint8_t* wal, uint64_t wal_bytes,
                              const char* const* names, const uint32_t* fields, const uint32_t* views, int32_t n_names, int32_t* out_loaded) try {
    if (!c || !data || n_names < 0 || (n_names > 0 && (!names || !fields || !views))) return fail(FBGPU_E_INVALID, "null argument");
    if (out_loaded) *out_loaded = 0;
    fbgpu_rbf::File f; std::string err;
    if (!f.open(data, data_bytes, wal, wal_bytes, err)) return fail(FBGPU_E_FORMAT, "%s", err.c_str());
    std::vector<fbgpu_rbf::RootRecord> recs;
    if (!f.root_records(recs, err)) return fail(FBGPU_E_FORMAT, "%s", err.c_str());
    // walk + validate everything before touching the store, so that a bad file leaves it unchanged
    struct Found { uint32_t field, view; std::vector<ParsedCont> cs; };
    std::vector<Found> found;
    std::vector<fbgpu_rbf::Cell> cells;
    for (int32_t i = 0; i < n_names; i++) {
        if (!names[i]) return fail(FBGPU_E_INVALID, "names[%d] is null", i);
        const fbgpu_rbf::RootRecord* rec = nullptr;
        for (const auto& r : recs) if (r.name == names[i]) { rec = &r; break; }
        if (!rec) continue;
        cells.clear();
        if (!f.walk(rec->pgno, cells, err)) return fail(FBGPU_E_FORMAT, "%s (bitmap %s)", err.c_str(), names[i]);
        Found fd{ fields[i], views[i], {} };
        fd.cs.reserve(cells.size());
        for (const auto& cl : cells) {
            if (cl.bit_n == 0) continue;                           // ContainerTypeNone / empty: never written, tolerated
            ParsedCont pc{}; pc.key = cl.key; pc.data = cl.data; pc.official_run = false; pc.n = cl.bit_n;
            if (cl.type == fbgpu_rbf::kCellArray) {
                if (cl.elem_n > 4096) return fail(FBGPU_E_FORMAT, "rbf: array cell with %u elements (bitmap %s)", cl.elem_n, names[i]);   // ArrayMaxSize 4079 rbf.go:39
                if (cl.elem_n != cl.bit_n) return fail(FBGPU_E_FORMAT, "rbf: array cell with elemN %u != bitN %u (bitmap %s)", cl.elem_n, cl.bit_n, names[i]);
                pc.typ = kArray;
            } else if (cl.type == fbgpu_rbf::kCellRLE) {
                if (cl.elem_n == 0 || cl.elem_n > 2048 || cl.bit_n > 65536) return fail(FBGPU_E_FORMAT, "rbf: bad RLE cell (bitmap %s)", names[i]);   // RLEMaxSize 2039 rbf.go:42
                pc.typ = kRun; pc.cnt = cl.elem_n;
            } else {
                if (cl.bit_n > 65536) return fail(FBGPU_E_FORMAT, "rbf: bad bitmap cell (bitmap %s)", names[i]);
                pc.typ = kBitmap;
            }
            fd.cs.push_back(pc);
        }
        found.push_back(std::move(fd));
    }
    std::unique_lock<std::shared_mutex> lk(c->store_mu);
    std::vector<PayloadCopy> copies;
    StoreTxn txn(c);
    for (auto& fd : found) {
        uint32_t fv = view_id_locked(c, ViewKey{ index, fd.field, fd.view }, true);
        int rc = add_fragment_locked(c, txn, fv, shard, fd.cs, copies); if (rc) return rc;
    }
    int rc = run_copies(c, copies, 1); if (rc) return rc;
    txn.commit();
    if (out_loaded) *out_loaded = (int32_t)found.size();
    return FBGPU_OK;
} FBGPU_CATCH

// read-only mapping of one file; empty / missing files map to (nullptr, 0) with ok() still true when `optional`
struct MappedFile {
    const uint8_t* p = nullptr; uint64_t n = 0; bool good = false;
    MappedFile(const std::string& path, bool optional) {
        int fd = open(path.c_str(), O_RDONLY | O_CLOEXEC);
        if (fd < 0) { good = optional; return; }
        struct stat st;
        if (fstat(fd, &st) == 0 && st.st_size > 0) {
            void* m = mmap(nullptr, (size_t)st.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
            if (m != MAP_FAILED) { p = (const uint8_t*)m; n = (uint64_t)st.st_size; good = true; }
        } else good = optional;
        close(fd);
    }
    ~MappedFile() { if (p) munmap((void*)p, (size_t)n); }
    MappedFile(const MappedFile&) = delete; MappedFile& operator=(const MappedFile&) = delete;
};

extern "C" int fbgpu_load_rbf_dir(fbgpu_ctx* c, uint32_t index, uint64_t shard, const char* dir, const char* const* names, const uint32_t* fields,
                                  const uint32_t* views, int32_t n_names, int32_t* out_loaded) try {
    if (!c || !dir) return fail(FBGPU_E_INVALID, "null argument");
    const std::string d(dir);
    MappedFile data(d + "/data", false), wal(d + "/wal", true);
    if (!data.good) return fail(FBGPU_E_FORMAT, "rbf: cannot map %s/data", dir);
    if (!wal.good) return fail(FBGPU_E_FORMAT, "rbf: cannot map %s/wal", dir);
    return fbgpu_load_rbf(c, index, shard, data.p, data.n, wal.p, wal.n, names, fields, views, n_names, out_loaded);
} FBGPU_CATCH

extern "C" int fbgpu_drop_fragment(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, uint64_t shard) try {
    if (!c) return fail(FBGPU_E_INVALID, "null ctx");
    std::unique_lock<std::shared_mutex> lk(c->store_mu);
    uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    if (fv == kNoView) return 0;
    drop_locked(c, fv, shard);
    return 0;
} FBGPU_CATCH

// ------------------------------------------------------------------ incremental refresh (the write path's mirror)
// fbgpu_apply_containers: what a committed write transaction did to ONE fragment, container by container — the mirror of
// Tx.PutContainer / Tx.RemoveContainer (tx.go:91-96, rbf/tx.go:791-860) collected over the transaction.  `roaring` holds only
// the containers that were written (each REPLACES the container under its key, or adds it), `removed_keys` the keys that were
// deleted.  Untouched containers keep their payload where it is in HBM: the call costs the bytes of the changed containers plus the
// fragment's row / descriptor entries, not a re-send of the fragment (fbgpu_load_fragment).  The replaced payloads become holes that
// fbgpu_compact reclaims container by container.  A fragment that is not resident yet is created from the written containers.
extern "C" int fbgpu_apply_containers(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, uint64_t shard, const uint8_t* roaring, uint64_t nbytes,
                                      const uint64_t* removed_keys, int64_t n_removed) try {
    if (!c || n_removed < 0 || (n_removed && !removed_keys) || (nbytes && !roaring)) return fail(FBGPU_E_INVALID, "null argument");
    std::vector<ParsedCont> put;
    if (nbytes) { int rc = parse_roaring(roaring, nbytes, put); if (rc) return rc; }
    for (size_t i = 1; i < put.size(); i++) if (put[i - 1].key >= put[i].key) return fail(FBGPU_E_FORMAT, "container keys not ascending");
    std::vector<uint64_t> removed(removed_keys, removed_keys + n_removed);
    std::sort(removed.begin(), removed.end());
    removed.erase(std::unique(removed.begin(), removed.end()), removed.end());
    for (const ParsedCont& pc : put) if (std::binary_search(removed.begin(), removed.end(), pc.key)) return fail(FBGPU_E_INVALID, "container key %llu is both written and removed", (unsigned long long)pc.key);
    std::unique_lock<std::shared_mutex> lk(c->store_mu);
    uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, true);
    std::vector<PayloadCopy> copies;
    StoreTxn txn(c);
    const auto& sm = c->shardmaps[fv];
    const int32_t old_fid = shard < sm.size() ? sm[shard] : -1;
    std::vector<FragItem> items;
    uint64_t holes = 0;
    if (old_fid >= 0) {
        const HostFrag& of = c->frags[(size_t)old_fid];
        items.reserve((size_t)of.n_desc + put.size());
        size_t pi = 0;
        auto flush_put = [&](uint64_t below) { while (pi < put.size() && put[pi].key < below) { items.push_back(FragItem{ put[pi].key, &put[pi], ContDesc{} }); pi++; } };
        for (uint32_t r = 0; r < of.n_rows; r++) {
            const RowEnt e = c->h_rows[of.row_off + r];
            uint32_t rank = 0;
            for (int slot = 0; slot < kSlotsPerRow; slot++) {
                if (!((e.mask >> slot) & 1)) continue;
                const ContDesc d = c->h_descs[e.first_desc + rank++];
                const uint64_t key = e.row * kSlotsPerRow + (uint64_t)slot;
                flush_put(key);
                const bool replaced = pi < put.size() && put[pi].key == key;
                if (replaced || std::binary_search(removed.begin(), removed.end(), key)) {
                    holes += (cont_bytes(d.typ, d.card, d.cnt) + 15) & ~15ull;
                    if (replaced) { items.push_back(FragItem{ key, &put[pi], ContDesc{} }); pi++; }
                } else items.push_back(FragItem{ key, nullptr, d });
            }
        }
        while (pi < put.size()) { items.push_back(FragItem{ put[pi].key, &put[pi], ContDesc{} }); pi++; }
    } else {
        items.reserve(put.size());
        for (const ParsedCont& pc : put) items.push_back(FragItem{ pc.key, &pc, ContDesc{} });
    }
    int rc;
    if (items.empty()) {                         // every container is gone: the fragment is dropped (its arena becomes dead space)
        if (old_fid >= 0) { txn.note(fv, shard); drop_locked(c, fv, shard); }
        rc = 0;
    } else {
        HostFrag pred_copy; const HostFrag* pred = nullptr;
        if (old_fid >= 0) { pred_copy = c->frags[(size_t)old_fid]; pred = &pred_copy; }
        rc = add_items_locked(c, txn, fv, shard, items, copies, pred, holes);
    }
    if (rc) return rc;
    rc = run_copies(c, copies, 1); if (rc) return rc;
    txn.commit();
    return FBGPU_OK;
} FBGPU_CATCH

// uploads staged payload (append) and refreshes metadata tables; store_mu held exclusively
// flatten shard maps; build the dense (shard,row) directory of every view whose row ids are dense
static void build_tables(fbgpu_ctx* c, std::vector<ViewTab>& views, std::vector<int32_t>& flat, std::vector<RowTabEnt>& rowtab) {
    views.assign(c->shardmaps.size(), ViewTab{}); flat.clear(); rowtab.clear();
    for (size_t v = 0; v < c->shardmaps.size(); v++) {
        const auto& sm = c->shardmaps[v];
        views[v] = ViewTab{}; views[v].shard_off = (uint32_t)flat.size(); views[v].n_shards = (uint32_t)sm.size();
        flat.insert(flat.end(), sm.begin(), sm.end());
        uint64_t rmin = ~0ull, rmax = 0, nrows = 0;
        for (int32_t f : sm) if (f >= 0) { const HostFrag& hf = c->frags[f]; if (!hf.n_rows) continue;
            rmin = std::min(rmin, c->h_rows[hf.row_off].row); rmax = std::max(rmax, c->h_rows[hf.row_off + hf.n_rows - 1].row); nrows = std::max<uint64_t>(nrows, hf.n_rows); }
        if (rmin == ~0ull) continue;
        uint64_t span = rmax - rmin + 1;
        if (span > 4 * nrows + 64 || span * sm.size() > (64ull << 20)) continue;       // sparse row ids or too large: keep the search chain
        views[v].rt_rows = (uint32_t)span; views[v].rt_off = rowtab.size(); views[v].rmin = rmin;
        rowtab.resize(rowtab.size() + span * sm.size(), RowTabEnt{ 0, 0, 0 });
        for (size_t sh = 0; sh < sm.size(); sh++) if (sm[sh] >= 0) { const HostFrag& hf = c->frags[sm[sh]];
            for (uint32_t k = 0; k < hf.n_rows; k++) { const RowEnt& e = c->h_rows[hf.row_off + k]; rowtab[views[v].rt_off + sh * span + (e.row - rmin)] = RowTabEnt{ e.first_desc, e.mask, 0 }; } }
    }
}

// memcpy split over a few host threads (one core moves ~10 GB/s, well below what the H2D DMA behind it takes)
static void par_memcpy(void* dst, const void* src, size_t n) {
    const int nt = (int)std::min<size_t>({ (size_t)std::max(1u, std::thread::hardware_concurrency()), (size_t)4, n / (4u << 20) + 1 });
    if (nt <= 1) { memcpy(dst, src, n); return; }
    std::vector<std::thread> th;
    for (int t = 0; t < nt; t++) {
        const size_t lo = (n * t / nt) & ~size_t(63), hi = t + 1 == nt ? n : (n * (t + 1) / nt) & ~size_t(63);
        th.emplace_back([=] { memcpy((uint8_t*)dst + lo, (const uint8_t*)src + lo, hi - lo); });
    }
    for (auto& t : th) t.join();
}

// Brings the host tables t_views / t_flat / t_rowtab up to date.  Full rebuild, or — when only a few (view, shard) pairs changed and
// none of them changes a table's geometry (a new view, a shard past the view's map, a row outside the dense directory's range) —
// a patch of those pairs' entries.  `patched` receives the patched pairs (empty after a full rebuild).
static bool refresh_tables(fbgpu_ctx* c, std::vector<std::pair<uint32_t, uint64_t>>& patched) {
    patched.clear();
    bool full = !c->tables_valid || c->dirty_shards.size() > 512 || c->t_views.size() != c->shardmaps.size();
    if (!full) {
        std::sort(c->dirty_shards.begin(), c->dirty_shards.end());
        c->dirty_shards.erase(std::unique(c->dirty_shards.begin(), c->dirty_shards.end()), c->dirty_shards.end());
        for (const auto& ds : c->dirty_shards) {
            const uint32_t fv = ds.first; const uint64_t shard = ds.second;
            const ViewTab& v = c->t_views[fv]; const auto& sm = c->shardmaps[fv];
            if (sm.size() != v.n_shards || shard >= v.n_shards) { full = true; break; }
            const int32_t fid = sm[shard];
            if (v.rt_rows && fid >= 0) {
                const HostFrag& hf = c->frags[(size_t)fid];
                if (hf.n_rows && (c->h_rows[hf.row_off].row < v.rmin || c->h_rows[hf.row_off + hf.n_rows - 1].row - v.rmin >= v.rt_rows)) { full = true; break; }
            }       // (a view without a dense directory stays correct through the search chain; it only gets one at the next full rebuild)
        }
    }
    if (full) { build_tables(c, c->t_views, c->t_flat, c->t_rowtab); c->tables_valid = true; c->dirty_shards.clear(); c->stats.full_commits++; return true; }
    c->stats.patch_commits++;
    for (const auto& ds : c->dirty_shards) {
        const uint32_t fv = ds.first; const uint64_t shard = ds.second;
        const ViewTab& v = c->t_views[fv];
        const int32_t fid = c->shardmaps[fv][shard];
        c->t_flat[v.shard_off + shard] = fid;
        if (v.rt_rows) {
            RowTabEnt* slice = c->t_rowtab.data() + v.rt_off + shard * v.rt_rows;
            std::fill(slice, slice + v.rt_rows, RowTabEnt{ 0, 0, 0 });
            if (fid >= 0) { const HostFrag& hf = c->frags[(size_t)fid];
                for (uint32_t k = 0; k < hf.n_rows; k++) { const RowEnt& e = c->h_rows[hf.row_off + k]; slice[e.row - v.rmin] = RowTabEnt{ e.first_desc, e.mask, 0 }; } }
        }
    }
    patched.swap(c->dirty_shards); c->dirty_shards.clear();
    return false;
}

// grows a device table to hold `need` bytes, keeping its first `keep` bytes (DevBuf::ensure alone would drop them)
static int grow_keeping(DevBuf& b, size_t need, size_t keep) {
    if (need <= b.cap) return 0;
    DevBuf nb;
    if (nb.ensure(std::max(need, b.cap + b.cap / 2))) return FBGPU_E_NOMEM;
    if (keep && b.p) { cudaError_t e = cudaMemcpy(nb.p, b.p, keep, cudaMemcpyDeviceToDevice); if (e != cudaSuccess) { nb.release(); return fail(FBGPU_E_CUDA, "table copy failed: %s", cudaGetErrorString(e)); } }
    b.release(); b = nb;
    return 0;
}

static int commit_locked(fbgpu_ctx* c) {
    std::vector<std::pair<uint32_t, uint64_t>> patched;
    if (c->inspect_only) {                  // no device: keep the payload in the staging buffer and the tables on the host
        if (c->meta_dirty || !c->tables_valid) refresh_tables(c, patched);
        c->meta_dirty = false;
        return 0;
    }
    if (!c->meta_dirty && c->staging.empty()) return 0;
    USE_DEVICE(c);
    CUDA_TRY(cudaDeviceSynchronize());   // no query may be reading tables we are about to replace (queries hold the shared lock anyway)
    if (!c->staging.empty()) {
        uint64_t need = c->uploaded + c->staging.len + kArenaSlack;
        if (need > c->d_payload.cap) {
            DevBuf nb; size_t want = std::max<size_t>(need, c->d_payload.cap * 2);
            if (nb.ensure(want)) { if (nb.ensure(need)) return FBGPU_E_NOMEM; }
            if (c->uploaded) CUDA_TRY(cudaMemcpy(nb.p, c->d_payload.p, c->uploaded, cudaMemcpyDeviceToDevice));
            c->d_payload.release(); c->d_payload = nb;
        }
        // pageable -> HBM through two pinned bounce buffers: the host memcpy of chunk k+1 overlaps the DMA of chunk k
        {
            const size_t chunk = 32u << 20, total = c->staging.len;
            if (total <= (4u << 20)) CUDA_TRY(cudaMemcpy((uint8_t*)c->d_payload.p + c->uploaded, c->staging.p, total, cudaMemcpyHostToDevice));
            else {
                if (c->bounce[0].ensure(chunk) || c->bounce[1].ensure(chunk)) return FBGPU_E_NOMEM;
                cudaStream_t st = c->wss[0]->stream;
                cudaEvent_t done[2]; CUDA_TRY(cudaEventCreateWithFlags(&done[0], cudaEventDisableTiming)); CUDA_TRY(cudaEventCreateWithFlags(&done[1], cudaEventDisableTiming));
                int k = 0;
                for (size_t off = 0; off < total; off += chunk, k ^= 1) {
                    size_t n = std::min(chunk, total - off);
                    if (off >= 2 * chunk) CUDA_TRY(cudaEventSynchronize(done[k]));       // bounce buffer k is free again
                    par_memcpy(c->bounce[k].p, c->staging.p + off, n);
                    CUDA_TRY(cudaMemcpyAsync((uint8_t*)c->d_payload.p + c->uploaded + off, c->bounce[k].p, n, cudaMemcpyHostToDevice, st));
                    CUDA_TRY(cudaEventRecord(done[k], st));
                }
                CUDA_TRY(cudaStreamSynchronize(st));
                cudaEventDestroy(done[0]); cudaEventDestroy(done[1]);
            }
        }
        c->uploaded += c->staging.len;
        c->staging.clear_and_free();
    }
    const bool full = refresh_tables(c, patched) || !c->dev_tables_valid;
    auto h2d = [&](void* dst, const void* src, size_t bytes) -> int {
        if (!bytes) return 0;
        cudaError_t e = cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice);
        return e == cudaSuccess ? 0 : fail(FBGPU_E_CUDA, "metadata upload failed: %s", cudaGetErrorString(e));
    };
    auto up = [&](DevBuf& b, const void* src, size_t bytes) -> int {
        if (b.ensure(std::max<size_t>(bytes, 256))) return FBGPU_E_NOMEM;
        return h2d(b.p, src, bytes);
    };
    int rc;
    c->dev_tables_valid = false;            // (a failure below leaves the device tables in an unknown state: the next commit re-sends them)
    if (full) {
        if ((rc = up(c->d_views, c->t_views.data(), c->t_views.size() * sizeof(ViewTab)))) return rc;
        if ((rc = up(c->d_shardmap, c->t_flat.data(), c->t_flat.size() * 4))) return rc;
        if ((rc = up(c->d_frags, c->h_frags.data(), c->h_frags.size() * sizeof(FragHdr)))) return rc;
        if ((rc = up(c->d_rows, c->h_rows.data(), c->h_rows.size() * sizeof(RowEnt)))) return rc;
        if ((rc = up(c->d_descs, c->h_descs.data(), c->h_descs.size() * sizeof(ContDesc)))) return rc;
        if ((rc = up(c->d_rowtab, c->t_rowtab.data(), c->t_rowtab.size() * sizeof(RowTabEnt)))) return rc;
    } else {
        // append-only mirrors: only their new tails travel; then the patched directory entries
        auto tail = [&](DevBuf& b, const void* base, size_t have, size_t now, size_t elem) -> int {
            int r = grow_keeping(b, std::max<size_t>(now * elem, 256), have * elem); if (r) return r;
            return h2d((uint8_t*)b.p + have * elem, (const uint8_t*)base + have * elem, (now - have) * elem);
        };
        if ((rc = tail(c->d_frags, c->h_frags.data(), c->dev_frags, c->h_frags.size(), sizeof(FragHdr)))) return rc;
        if ((rc = tail(c->d_rows, c->h_rows.data(), c->dev_rows, c->h_rows.size(), sizeof(RowEnt)))) return rc;
        if ((rc = tail(c->d_descs, c->h_descs.data(), c->dev_descs, c->h_descs.size(), sizeof(ContDesc)))) return rc;
        for (const auto& ds : patched) {
            const ViewTab& v = c->t_views[ds.first];
            const size_t fi = (size_t)v.shard_off + ds.second;
            if ((rc = h2d((int32_t*)c->d_shardmap.p + fi, c->t_flat.data() + fi, 4))) return rc;
            if (v.rt_rows) { const size_t ri = (size_t)v.rt_off + ds.second * v.rt_rows;
                if ((rc = h2d((RowTabEnt*)c->d_rowtab.p + ri, c->t_rowtab.data() + ri, (size_t)v.rt_rows * sizeof(RowTabEnt)))) return rc; }
        }
    }
    c->dev_frags = c->h_frags.size(); c->dev_rows = c->h_rows.size(); c->dev_descs = c->h_descs.size();
    c->dev_tables_valid = true;
    c->n_views_dev = (uint32_t)c->t_views.size();
    c->meta_dirty = false;
    c->stats.device_bytes = c->d_payload.cap + c->d_views.cap + c->d_shardmap.cap + c->d_frags.cap + c->d_rows.cap + c->d_descs.cap + c->d_rowtab.cap;
    return 0;
}

// Reclaims what replaced / dropped fragments left behind (store_mu held exclusively; everything pending is committed first):
// live fragments are copied device-to-device into a fresh arena in their current order, each keeping its offset modulo 128 so
// that every container keeps its alignment, and the host mirrors (fragment headers, row entries, descriptors, shard maps)
// are rebuilt without the dead entries.  Write batches re-send whole fragments (INTEGRATION.md §3), so without this the
// arena of a long-running node would only grow.
static int compact_locked(fbgpu_ctx* c) {
    int rc = commit_locked(c); if (rc) return rc;
    if (c->inspect_only) return 0;                         // (no device arena: the staging buffer is the store)
    if (c->dead_arena == 0) return 0;
    USE_DEVICE(c);
    CUDA_TRY(cudaDeviceSynchronize());
    std::vector<HostFrag> frags; std::vector<FragHdr> hfr; std::vector<RowEnt> rows; std::vector<ContDesc> descs;
    struct Move { uint64_t from, to, len; };
    std::vector<Move> moves; uint64_t cur = 0;
    std::vector<ArenaMove> gathers;                        // container-granular moves of fragments that hold holes (fbgpu_apply_containers)
    auto maps = c->shardmaps;                              // (built aside: an allocation failure below must leave the store as it was)
    for (auto& sm : maps) std::fill(sm.begin(), sm.end(), -1);
    for (size_t fid = 0; fid < c->frags.size(); fid++) {
        HostFrag f = c->frags[fid];
        if (!f.live) continue;
        FragHdr h = c->h_frags[fid];
        const uint64_t desc_new = descs.size(), row_new = rows.size();
        for (uint32_t r = 0; r < f.n_rows; r++) { RowEnt e = c->h_rows[f.row_off + r]; e.first_desc = (uint32_t)(e.first_desc - f.desc_off + desc_new); rows.push_back(e); }
        if (f.inherited.empty() && f.hole_bytes == 0) {    // one extent, no hole: moved as a block, every container keeps its offset modulo 128
            const uint64_t to = ((cur + 127) & ~127ull) + (f.arena_off & 127ull);
            const int64_t d16 = ((int64_t)to - (int64_t)f.arena_off) / 16;         // both are 16-byte aligned
            for (uint32_t k = 0; k < f.n_desc; k++) { ContDesc d = c->h_descs[f.desc_off + k]; d.off16 = (uint32_t)((int64_t)d.off16 + d16); descs.push_back(d); }
            moves.push_back(Move{ f.arena_off, to, f.arena_len });
            f.arena_off = to;
            cur = to + f.arena_len;
        } else {                                           // updated fragment: its live containers are gathered one by one, the holes stay behind
            const uint64_t start = (cur + 15) & ~15ull;
            cur = start;
            for (uint32_t k = 0; k < f.n_desc; k++) {
                ContDesc d = c->h_descs[f.desc_off + k];
                const uint64_t align = d.typ == kBitmap ? 128 : 16, to = (cur + align - 1) & ~(align - 1);
                const uint64_t padded = (cont_bytes(d.typ, d.card, d.cnt) + 15) & ~15ull;
                gathers.push_back(ArenaMove{ d.off16, (uint32_t)(to / 16), (uint32_t)(padded / 16), 0u });
                d.off16 = (uint32_t)(to / 16); descs.push_back(d);
                cur = to + padded;
            }
            f.arena_off = start; f.arena_len = cur - start; f.inherited.clear(); f.hole_bytes = 0;
        }
        f.row_off = (uint32_t)row_new; f.desc_off = desc_new; h.row_off = (uint32_t)row_new;
        maps[f.fv][f.shard] = (int32_t)frags.size();
        frags.push_back(std::move(f)); hfr.push_back(h);
    }
    if (cur / 16 > 0xffffffffull) return fail(FBGPU_E_NOMEM, "payload arena exceeds 64 GiB addressable by 32-bit 16 B offsets");
    DevBuf nb;
    if (nb.ensure(cur + kArenaSlack)) return FBGPU_E_NOMEM;
    for (const Move& m : moves) if (m.len) CUDA_TRY(cudaMemcpy((uint8_t*)nb.p + m.to, (const uint8_t*)c->d_payload.p + m.from, m.len, cudaMemcpyDeviceToDevice));
    if (!gathers.empty()) {
        DevBuf d_mv;
        if (d_mv.ensure(gathers.size() * sizeof(ArenaMove))) { nb.release(); return FBGPU_E_NOMEM; }
        cudaError_t e = cudaMemcpy(d_mv.p, gathers.data(), gathers.size() * sizeof(ArenaMove), cudaMemcpyHostToDevice);
        if (e == cudaSuccess) {
            const unsigned grid = (unsigned)std::min<size_t>((gathers.size() + 7) / 8, (size_t)c->sm_count * 16);
            arena_gather_kernel<<<grid, 256>>>((const uint4*)c->d_payload.p, (uint4*)nb.p, (const ArenaMove*)d_mv.p, (long long)gathers.size());
            e = cudaGetLastError(); if (e == cudaSuccess) e = cudaDeviceSynchronize();
        }
        d_mv.release();
        if (e != cudaSuccess) { nb.release(); return fail(FBGPU_E_CUDA, "arena gather failed: %s", cudaGetErrorString(e)); }
    }
    c->d_payload.release(); c->d_payload = nb;
    c->frags.swap(frags); c->h_frags.swap(hfr); c->h_rows.swap(rows); c->h_descs.swap(descs); c->shardmaps.swap(maps);
    c->uploaded = cur; c->dead_arena = 0; c->stats.dead_bytes = 0;
    c->meta_dirty = true; c->tables_valid = false; c->dev_tables_valid = false;
    return commit_locked(c);                               // tables for the new layout
}

extern "C" int fbgpu_commit(fbgpu_ctx* c) try {
    if (!c) return fail(FBGPU_E_INVALID, "null ctx");
    std::unique_lock<std::shared_mutex> lk(c->store_mu);
    // a node that keeps re-sending fragments compacts on its own once the dead share is large (never reached by small stores)
    if (!c->inspect_only && c->dead_arena >= (256ull << 20) && c->dead_arena * 2 >= c->uploaded + c->staging.len) return compact_locked(c);
    return commit_locked(c);
} FBGPU_CATCH

extern "C" int fbgpu_compact(fbgpu_ctx* c) try {
    if (!c) return fail(FBGPU_E_INVALID, "null ctx");
    std::unique_lock<std::shared_mutex> lk(c->store_mu);
    return compact_locked(c);
} FBGPU_CATCH
// Takes the store's shared lock for a query with the device tables in sync with the host mirrors: the "is anything
// pending" check and the query run under the SAME lock acquisition, so a load that slips in between a commit and the
// query cannot leave the query reading host mirrors that are newer than what is in HBM.  (After USE_DEVICE.)
static int lock_committed(fbgpu_ctx* c, std::shared_lock<std::shared_mutex>& lk) {
    for (;;) {
        lk = std::shared_lock<std::shared_mutex>(c->store_mu);
        if (!c->meta_dirty && c->staging.empty()) return 0;
        lk.unlock();
        int rc = fbgpu_commit(c); if (rc) return rc;
    }
}

// the start of every query once its arguments are checked: refuses an inspection-only context, selects the device, locks the store
static int begin_query(fbgpu_ctx* c, std::shared_lock<std::shared_mutex>& lk) {
    USE_DEVICE(c);
    return lock_committed(c, lk);
}

extern "C" int fbgpu_get_stats(fbgpu_ctx* c, fbgpu_stats* out) try {
    if (!c || !out) return fail(FBGPU_E_INVALID, "null argument");
    std::shared_lock<std::shared_mutex> lk(c->store_mu);
    *out = c->stats;
    return 0;
} FBGPU_CATCH

// ------------------------------------------------------------------ program compiler (program_compiler.h)
// store_mu must be held (shared) by the caller
static int compile_program(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, std::vector<DevOp>& out, int& depth) {
    Error err;
    ViewLookup lookup = [c, index](uint32_t field, uint32_t view) { return view_id_locked(c, ViewKey{ index, field, view }, false); };
    int rc = compile(ops, n_ops, lookup, out, depth, err);
    if (rc) return fail(rc, "%s", err.msg);
    expand_push_row(out);          // every kernel accepts the rewritten program; the word-parallel op loop (wp_machine.h) requires it
    return 0;
}

// ------------------------------------------------------------------ execution helpers
static void bump(fbgpu_ctx* c, uint64_t launches, float ms) {
    std::lock_guard<std::mutex> lk(c->cnt_mu);
    c->counters.kernel_launches += launches; c->counters.queries++; c->counters.last_query_gpu_ms = ms;
}

static int allreduce_u64(fbgpu_ctx* c, Workspace* w, void* dptr, size_t n) {
    if (!c->comm) return 0;
    // one communicator, many caller threads: enqueueing must be serialised (and the callers must issue collective
    // queries in the same order on every rank, like any NCCL program)
    std::lock_guard<std::mutex> lk(c->coll_mu);
    int r = g_nccl.AllReduce(dptr, dptr, n, kNcclUint64, kNcclSum, c->comm, w->stream);
    if (r != 0) return fail(FBGPU_E_COMM, "ncclAllReduce failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    return 0;
}

// uploads [DevOp prog | u64 shards] with one H2D copy; returns device pointers
static std::vector<int2> find_batches(const std::vector<DevOp>& prog);
static int upload_inputs(Workspace* w, const std::vector<DevOp>& prog, const uint64_t* shards, int64_t n_shards, const DevOp** d_prog, const uint64_t** d_shards) {
    std::vector<int2> batches = find_batches(prog);
    size_t pb = prog.size() * sizeof(DevOp), sb = (size_t)n_shards * 8, bb = batches.size() * sizeof(int2), tot = pb + sb + bb;
    if (w->h_in.ensure(tot + 16)) return FBGPU_E_NOMEM;
    if (w->d_in.ensure(pb + sb + 16)) return FBGPU_E_NOMEM;
    if (w->d_aux.ensure(bb + 16)) return FBGPU_E_NOMEM;
    if (pb) memcpy(w->h_in.p, prog.data(), pb);
    if (sb) memcpy((uint8_t*)w->h_in.p + pb, shards, sb);
    if (bb) memcpy((uint8_t*)w->h_in.p + pb + sb, batches.data(), bb);
    if (pb + sb) CUDA_TRY(cudaMemcpyAsync(w->d_in.p, w->h_in.p, pb + sb, cudaMemcpyHostToDevice, w->stream));
    if (bb) CUDA_TRY(cudaMemcpyAsync(w->d_aux.p, (uint8_t*)w->h_in.p + pb + sb, bb, cudaMemcpyHostToDevice, w->stream));
    *d_prog = (const DevOp*)w->d_in.p; *d_shards = (const uint64_t*)((uint8_t*)w->d_in.p + pb);
    return 0;
}

// runs of commuting row ops ([k,e) of D_OR_ROW / D_ANDNOT_ROW / D_XOR_ROW): eval_kernel applies each run as one batch
static std::vector<int2> find_batches(const std::vector<DevOp>& prog) {
    std::vector<int2> b;
    for (size_t k = 0; k < prog.size();) {
        uint8_t o = prog[k].op;
        if (o == D_OR_ROW || o == D_ANDNOT_ROW || o == D_XOR_ROW) { size_t e = k + 1; while (e < prog.size() && prog[e].op == o) e++; b.push_back(make_int2((int)k, (int)e)); k = e; }
        else k++;
    }
    return b;
}

static int launch_eval(fbgpu_ctx* c, Workspace* w, const std::vector<DevOp>& prog, const DevOp* d_prog, int depth, const uint64_t* d_shards, long long n_units, EvalOut out) {
    if (n_units <= 0) return 0;
    const int n_ops = (int)prog.size();
    std::vector<int2> batches = find_batches(prog);
    // Word-parallel kernel for bitmap-heavy programs (BSI plane sweeps, dense rows): chosen when the views the
    // program references hold few array containers.  Row results (out.info) need cross-slice run counts: not here.
    if (!out.info && n_ops <= kWpMaxOps && depth <= kWpMaxDepth) {
        uint64_t arr = 0, other = 0, striped = 0;
        for (const DevOp& o : prog) if (o.op >= D_PUSH_ROW && o.op <= D_ORANDNOT_ROW && o.op != D_PUSH_EMPTY && o.fv < c->view_arr.size()) { arr += c->view_arr[o.fv]; other += c->view_other[o.fv]; striped += c->view_striped[o.fv]; }
        // (wp_slice searches sorted arrays: a view that holds striped arrays can never take this kernel, forced or not)
        if (striped == 0 && ((other > 0 && arr * 8 <= other) || getenv("FBGPU_FORCE_WORDPAR") != nullptr)) {
            long long blocks = n_units * kWpBlocksPerUnit;
            long long grid = std::min<long long>(blocks, (long long)c->sm_count * kWpMinBlocks * 2);
            eval_wordpar_kernel<<<(unsigned)grid, kWpThreads, 0, w->stream>>>(store_ref(c), d_prog, n_ops, d_shards, n_units, out);
            CUDA_TRY(cudaGetLastError());
            return 0;
        }
    }
    // the batch table travels in front of the program in the same H2D copy (upload_inputs); see d_batches()
    const int2* d_batches = reinterpret_cast<const int2*>(w->d_aux.p);
    size_t smem = (size_t)(depth + 1) * 8192;
    int per_sm = std::max(1, (int)std::min<size_t>(std::min(kEvalMinBlocks, 2048 / kEvalThreads), (227 * 1024) / (smem + 3 * 1024 + 512)));
    long long grid = std::min<long long>(n_units, (long long)c->sm_count * per_sm);
    eval_kernel<<<(unsigned)grid, kEvalThreads, smem, w->stream>>>(store_ref(c), d_prog, n_ops, depth, d_batches, (int)batches.size(), d_shards, n_units, out);
    CUDA_TRY(cudaGetLastError());
    return 0;
}

// pair_count_kernel's shard arguments: the usual shard list is a contiguous range (a node's share, SURVEY §8e), for which the
// kernel is given no list and computes each shard id from the first instead of loading it
struct PairShards { const uint64_t* list; uint64_t first; };
static PairShards pair_shards(const uint64_t* shards, int64_t n, const uint64_t* d_shards) {
    for (int64_t i = 1; i < n; i++) if (shards[i] != shards[0] + (uint64_t)i) return { d_shards, shards[0] };
    return { n > 0 ? nullptr : d_shards, n ? shards[0] : 0 };
}

static std::vector<uint64_t> sorted_unique(const uint64_t* v, int64_t n) {
    std::vector<uint64_t> s(v, v + n);
    std::sort(s.begin(), s.end());
    s.erase(std::unique(s.begin(), s.end()), s.end());
    return s;
}

// the program "<ops> ∩ Union(Row(field, views[0], row), ..., Row(field, views[n_views - 1], row))": one view's row without the
// Union, and the row (or union) alone when there are no ops
static std::vector<fbgpu_op> and_row(const fbgpu_op* ops, int32_t n_ops, uint32_t field, const uint32_t* views, int32_t n_views, uint64_t row) {
    std::vector<fbgpu_op> full(ops, ops + n_ops);
    for (int32_t i = 0; i < n_views; i++) { fbgpu_op r{}; r.opcode = FBGPU_OP_ROW; r.field = field; r.view = views[i]; r.a = row; full.push_back(r); }
    if (n_views > 1) { fbgpu_op u{}; u.opcode = FBGPU_OP_UNION; u.argc = (uint32_t)n_views; full.push_back(u); }
    if (n_ops) { fbgpu_op in{}; in.opcode = FBGPU_OP_INTERSECT; in.argc = 2; full.push_back(in); }
    return full;
}
static std::vector<fbgpu_op> and_row(const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, uint64_t row) {
    return and_row(ops, n_ops, field, &view, 1, row);
}

// One query call on a leased workspace: the device program and its operand stack depth, the uploaded program and shard list,
// and the call's kernel launches and GPU milliseconds, which finish() adds to the counters.
struct Query {
    fbgpu_ctx* c; WsLease lease; Workspace* w;
    std::vector<DevOp> prog; int depth = 1;
    const DevOp* d_prog = nullptr; const uint64_t* d_shards = nullptr;
    long long n_units = 0;                   // (shard, slot) units of the shard list
    uint64_t launches = 0; float ms = 0;
    explicit Query(fbgpu_ctx* ctx) : c(ctx), lease(ctx), w(lease.w) {}

    int open(uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards) {
        int rc = compile_program(c, index, ops, n_ops, prog, depth); if (rc) return rc;
        return open(shards, n_shards);
    }
    int open(const uint64_t* shards, int64_t n_shards) {      // no program
        n_units = (long long)n_shards * kSlotsPerRow;
        return upload_inputs(w, prog, shards, n_shards, &d_prog, &d_shards);
    }
    // evaluates the program for units [u0, u0 + nu) into `bits` (w->d_bitmaps when null), with `info` also their {N, runs} into w->d_info
    int eval(long long u0, long long nu, bool info = false, uint4* bits = nullptr) {
        if (!bits) { if (w->d_bitmaps.ensure((size_t)nu * 8192)) return FBGPU_E_NOMEM; bits = (uint4*)w->d_bitmaps.p; }
        if (info && w->d_info.ensure((size_t)nu * 8)) return FBGPU_E_NOMEM;
        EvalOut eo{ nullptr, nullptr, bits, info ? (uint2*)w->d_info.p : nullptr, FuseReduce{} };
        int rc = launch_eval(c, w, prog, d_prog, depth, d_shards + u0 / kSlotsPerRow, nu, eo); if (rc) return rc;
        launches++;
        return 0;
    }
    // Row / Columns: eval() with the units' {N, runs} read back into h_out; ev0 opens the batch's timed bracket
    int eval_info(long long u0, long long nu, const uint2*& info) {
        // (the buffers are grown before ev0: the bracket holds no allocation)
        if (w->d_bitmaps.ensure((size_t)nu * 8192) || w->d_info.ensure((size_t)nu * 8) || w->h_out.ensure((size_t)nu * 8)) return FBGPU_E_NOMEM;
        CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
        int rc = eval(u0, nu, true); if (rc) return rc;
        CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_info.p, (size_t)nu * 8, cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        info = (const uint2*)w->h_out.p;
        return 0;
    }
    // copies the unit list to d_emit_units and runs launch(d_units, units.size(), grid): emit kernels whose output stays on the device
    template <class Unit, class Launch>
    int emit_on_device(const std::vector<Unit>& units, size_t out_bytes, Launch launch) {
        const size_t ub = units.size() * sizeof(Unit);
        if (w->d_emit_units.ensure(ub) || w->d_emit.ensure(out_bytes) || w->h_in.ensure(ub)) return FBGPU_E_NOMEM;
        CUDA_TRY(cudaStreamSynchronize(w->stream));   // an earlier H2D copy out of h_in may still be pending
        memcpy(w->h_in.p, units.data(), ub);
        CUDA_TRY(cudaMemcpyAsync(w->d_emit_units.p, w->h_in.p, ub, cudaMemcpyHostToDevice, w->stream));
        const int grid = (int)std::min<size_t>(units.size(), (size_t)c->sm_count * 8);
        return launch((const Unit*)w->d_emit_units.p, (int)units.size(), grid);
    }
    // Row / Columns: emit_on_device, then `out_bytes` of d_emit read back into h_in; ev1 closes the batch's timed bracket
    template <class Unit, class Launch>
    int emit(const std::vector<Unit>& units, size_t out_bytes, Launch launch) {
        if (w->h_in.ensure(std::max(units.size() * sizeof(Unit), out_bytes))) return FBGPU_E_NOMEM;
        int rc = emit_on_device(units, out_bytes, launch); if (rc) return rc;
        CUDA_TRY(cudaStreamSynchronize(w->stream));   // h_in is reused as the D2H landing buffer below
        CUDA_TRY(cudaMemcpyAsync(w->h_in.p, w->d_emit.p, out_bytes, cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        add_elapsed();
        return 0;
    }
    void add_elapsed() { float t = 0; cudaEventElapsedTime(&t, w->ev0, w->ev1); ms += t; }
    void finish() { bump(c, launches, ms); lease.ok = true; }
};

// ------------------------------------------------------------------ Count
// collective == false: this context's shards only — no cross-GPU merge (fbgpu_any's early exit must not desynchronise the ranks)
static int count_impl(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards,
                      uint64_t* out_total, uint64_t* out_per_shard, bool collective) {
    if (!c || !out_total || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    Query q(c); Workspace* w = q.w;
    rc = q.open(index, ops, n_ops, shards, n_shards); if (rc) return rc;
    const std::vector<DevOp>& prog = q.prog;
    // layout of d_counts: [total][per-shard counts ...][ticket][reduced result][error]
    const size_t nper = out_per_shard ? (size_t)n_shards : 0, nc = 1 + nper + 3;
    if (w->d_counts.ensure(nc * 8)) return FBGPU_E_NOMEM;
    if (w->h_out.ensure(nc * 8)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, nc * 8, w->stream));
    unsigned long long* d_total = (unsigned long long*)w->d_counts.p;
    unsigned long long* d_per = out_per_shard ? d_total + 1 : nullptr;
    const long long n_units = q.n_units;
    // cross-GPU merge of the count: fused into the kernel over peer memory when the mailboxes are mapped, else NCCL
    std::unique_lock<std::mutex> coll_lk(c->coll_mu, std::defer_lock);
    FuseReduce fr{};
    coll_lk.lock();                          // collective queries are issued in the same order on every rank
    const bool p2p = c->p2p && collective;   // read once, under the lock fbgpu_comm_p2p_open/_disable take
    if (!p2p) coll_lk.unlock();
    if (p2p) {
        fr.peers = (Mailbox* const*)c->d_peers.p; fr.ticket = (unsigned int*)(d_total + 1 + nper); fr.result = d_total + 1 + nper + 1;
        fr.error = (unsigned int*)(d_total + 1 + nper + 2);
        fr.epoch = ++c->epoch; fr.rank = c->rank; fr.n_ranks = c->n_ranks; fr.timeout_cycles = c->p2p_timeout_cycles;
    }
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    if (n_units > 0) {
        // fused Intersect+Count fast path: Count(Intersect(Row, Row))  (executor.go:5357 + row.go:242 + Count)
        // (the compiled form of Row is PUSH_ROW, or PUSH_EMPTY ; OR_ROW after expand_push_row)
        const DevOp* pa = nullptr; const DevOp* pb = nullptr;
        if (prog.size() == 2 && prog[0].op == D_PUSH_ROW && prog[1].op == D_AND_ROW) { pa = &prog[0]; pb = &prog[1]; }
        else if (prog.size() == 3 && prog[0].op == D_PUSH_EMPTY && prog[1].op == D_OR_ROW && prog[2].op == D_AND_ROW) { pa = &prog[1]; pb = &prog[2]; }
        if (pa) {
            long long grid = std::min<long long>((n_units + kPcWarps - 1) / kPcWarps, (long long)c->sm_count * c->pair_ctas_per_sm);
            c->counters_pair_launches++;
            const PairShards ps = pair_shards(shards, n_shards, q.d_shards);
            pair_count_kernel<<<(unsigned)grid, kPcWarps * 32, kPcWarps * 8192, w->stream>>>(store_ref(c), pa->fv, pa->row, pb->fv, pb->row, nullptr, nullptr, n_units,
                ps.list, ps.first, n_units, d_total, d_per, nullptr, fr);
            CUDA_TRY(cudaGetLastError());
        } else {
            EvalOut eo{ d_total, d_per, nullptr, nullptr, fr };
            rc = launch_eval(c, w, prog, q.d_prog, q.depth, q.d_shards, n_units, eo); if (rc) return rc;
        }
    } else if (p2p) {
        p2p_reduce_only_kernel<<<1, 1, 0, w->stream>>>(fr, d_total);
        CUDA_TRY(cudaGetLastError());
    }
    if (!p2p && collective) { rc = allreduce_u64(c, w, d_total, 1); if (rc) return rc; }   // inside the timed bracket: the collective is part of the step
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, nc * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    if (p2p && ((uint64_t*)w->h_out.p)[1 + nper + 2] != 0) {
        q.lease.ok = true;                   // the stream is drained; the exchange state is not: the caller re-opens the peers
        return fail(FBGPU_E_COMM, "rank %d did not publish its count for exchange %llu in time (peer dead, or the ranks issued their collective queries in different orders); re-open with fbgpu_comm_p2p_open",
                    (int)((uint64_t*)w->h_out.p)[1 + nper + 2] - 1, (unsigned long long)fr.epoch);
    }
    *out_total = p2p ? ((uint64_t*)w->h_out.p)[1 + nper + 1] : ((uint64_t*)w->h_out.p)[0];
    if (out_per_shard) memcpy(out_per_shard, (uint64_t*)w->h_out.p + 1, (size_t)n_shards * 8);
    q.add_elapsed();
    q.launches = (n_units > 0 || p2p) ? 1 : 0;
    q.finish();
    return FBGPU_OK;
}
extern "C" int fbgpu_count(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards,
                           uint64_t* out_total, uint64_t* out_per_shard) try {
    return count_impl(c, index, ops, n_ops, shards, n_shards, out_total, out_per_shard, true);
} FBGPU_CATCH
static int fbgpu_count_local(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_total) {
    return count_impl(c, index, ops, n_ops, shards, n_shards, out_total, nullptr, false);
}

// ------------------------------------------------------------------ Row (canonical Pilosa-roaring result)
extern "C" int fbgpu_row(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards,
                         uint8_t* out_buf, uint64_t out_cap, uint64_t* out_len, uint64_t* out_count) try {
    if (!c || !out_len || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    Query q(c); Workspace* w = q.w;
    // Row.Merge concatenates disjoint shard segments (row.go:202); emit in ascending shard order
    const std::vector<uint64_t> sorted = sorted_unique(shards, n_shards);
    rc = q.open(index, ops, n_ops, sorted.data(), (int64_t)sorted.size()); if (rc) return rc;
    const long long n_units = q.n_units;
    struct OutCont { uint64_t key; uint16_t typ; uint32_t n; uint64_t size; uint32_t batch; uint64_t src_off; };
    std::vector<OutCont> conts; std::vector<std::vector<uint8_t>> batch_bufs;   // one host copy of the emitted payloads per batch
    // a single batch (<= 1024 shards, the usual call) needs no such copy: its payloads are assembled straight from the pinned
    // D2H landing buffer, which stays leased until this function returns
    const bool single_batch = n_units <= c->unit_batch;
    const uint8_t* single_src = nullptr;
    uint64_t total_count = 0;
    for (long long u0 = 0; u0 < n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, n_units - u0);
        const uint2* info;
        rc = q.eval_info(u0, nu, info); if (rc) return rc;
        // optimize(): roaring.go:3412-3426
        std::vector<EmitUnit> emits; uint64_t off = 0;
        for (long long u = 0; u < nu; u++) {
            uint32_t N = info[u].x, runs = info[u].y;
            if (!N) continue;
            uint16_t typ = (runs <= 2048 && runs <= N / 2) ? kRun : (N < 4096 ? kArray : kBitmap);
            uint64_t size = typ == kRun ? 2 + 4ull * runs : typ == kArray ? 2ull * N : 8192;
            EmitUnit e{ off, (uint32_t)u, typ };
            emits.push_back(e);
            OutCont oc; oc.key = sorted[(u0 + u) / kSlotsPerRow] * kSlotsPerRow + (uint64_t)((u0 + u) % kSlotsPerRow); oc.typ = typ; oc.n = N; oc.size = size;
            oc.batch = (uint32_t)batch_bufs.size(); oc.src_off = off;
            conts.push_back(oc);
            off += (size + 15) & ~15ull;
            total_count += N;
        }
        if (emits.empty()) batch_bufs.emplace_back();
        if (!emits.empty()) {
            rc = q.emit(emits, off, [&](const EmitUnit* d_units, int n, int grid) {
                canon_emit_kernel<<<grid, kEmitThreads, 0, w->stream>>>((const uint4*)w->d_bitmaps.p, d_units, n, (uint8_t*)w->d_emit.p);
                CUDA_TRY(cudaGetLastError()); q.launches++;
                return 0;
            });
            if (rc) return rc;
            if (single_batch) { single_src = (const uint8_t*)w->h_in.p; batch_bufs.emplace_back(); }
            else batch_bufs.emplace_back((uint8_t*)w->h_in.p, (uint8_t*)w->h_in.p + off);
        }
    }
    bump(c, q.launches, q.ms);
    // writeToUnoptimized layout: roaring.go:1738-1817
    uint64_t need = 8 + conts.size() * 16;
    for (auto& oc : conts) need += oc.size;
    *out_len = need;
    if (out_count) *out_count = total_count;
    if (need > 0xffffffffull) return fail(FBGPU_E_INVALID, "result of %llu bytes exceeds the 32-bit container offsets of the Pilosa roaring format (roaring.go:1790-1800); query fewer shards per call", (unsigned long long)need);
    if (need > out_cap || !out_buf) return fail(FBGPU_E_NOSPACE, "output needs %llu bytes", (unsigned long long)need);
    uint32_t cookie = 12348, cnt = (uint32_t)conts.size();
    memcpy(out_buf, &cookie, 4); memcpy(out_buf + 4, &cnt, 4);
    // header + offset table serially (12 + 4 bytes per container); the payload copies are split over a few host threads when
    // the result is large (one thread moves ~10 GB/s; an 85 MB union of rows otherwise spends most of its time here)
    uint8_t *h = out_buf + 8, *offp = out_buf + 8 + conts.size() * 12; uint64_t off = 8 + conts.size() * 16;
    std::vector<uint64_t> dst_off(conts.size());
    for (size_t i = 0; i < conts.size(); i++) {
        const OutCont& oc = conts[i];
        uint16_t n1 = (uint16_t)(oc.n - 1);
        memcpy(h, &oc.key, 8); memcpy(h + 8, &oc.typ, 2); memcpy(h + 10, &n1, 2); h += 12;
        uint32_t o32 = (uint32_t)off; memcpy(offp, &o32, 4); offp += 4;
        dst_off[i] = off; off += oc.size;
    }
    auto copy_range = [&](size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; i++) {
            const OutCont& oc = conts[i];
            const uint8_t* src = single_batch ? single_src : batch_bufs[oc.batch].data();
            memcpy(out_buf + dst_off[i], src + oc.src_off, oc.size);
        }
    };
    const int n_threads = (int)std::min<uint64_t>({ (uint64_t)std::max(1u, std::thread::hardware_concurrency()), 8ull, need / (8ull << 20) + 1 });
    if (n_threads <= 1) copy_range(0, conts.size());
    else {
        std::vector<std::thread> th;
        for (int t = 0; t < n_threads; t++) th.emplace_back(copy_range, conts.size() * t / n_threads, conts.size() * (t + 1) / n_threads);
        for (auto& t : th) t.join();
    }
    q.lease.ok = true;                       // (not before the size checks above: their error returns drain the stream)
    return FBGPU_OK;
} FBGPU_CATCH

// ------------------------------------------------------------------ Columns (Row.Columns(): ascending ids, with executeLimitCall's window) / Extract
// [offset, offset + limit) as a half-open range of ranks; no limit (limit < 0) and an overflowing end are "to the end"
static uint64_t window_end(uint64_t offset, int64_t limit) {
    return limit < 0 ? ~0ull : (offset + (uint64_t)limit < offset ? ~0ull : offset + (uint64_t)limit);
}

// the emit units of one evaluated batch (units [u0, u0 + nu) of the sorted shard list, `info` their {N, runs}): its non-empty
// units clipped to the ranks [offset, win_end) of the row, packed from out_off 0.  `seen` is the row's rank of the batch's first
// column on entry and of the next batch's on return; the result is the number of columns the units emit.
static uint64_t col_units(const uint2* info, long long u0, long long nu, const std::vector<uint64_t>& sorted, uint64_t offset, uint64_t win_end,
                          uint64_t& seen, std::vector<ColUnit>& units) {
    units.clear();
    uint64_t out = 0;
    for (long long u = 0; u < nu; u++) {
        const uint64_t N = info[u].x;
        if (!N) continue;
        const uint64_t lo = std::max(seen, offset), hi = std::min(seen + N, win_end);    // the unit's ranks are [seen, seen + N)
        if (hi > lo) {
            ColUnit cu{};
            cu.out_off = out; cu.unit = (uint32_t)u; cu.first = (uint32_t)(lo - seen); cu.last = (uint32_t)(hi - seen);
            cu.col_base = (sorted[(u0 + u) / kSlotsPerRow] << 20) + (uint64_t)((u0 + u) % kSlotsPerRow) * 65536ull;
            units.push_back(cu);
            out += hi - lo;
        }
        seen += N;
    }
    return out;
}

// shared body: evaluate the row into per-unit bitmaps, cut the [offset, offset+limit) window into per-unit rank ranges, expand
// the column ids on the device and — for Extract — gather the BSI planes of `fv_vals` for exactly those columns
static int columns_impl(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards,
                        uint64_t offset, int64_t limit, bool want_vals, uint32_t fv_vals, int depth_vals,
                        uint64_t* out_cols, int64_t* out_vals, uint64_t cap, uint64_t* out_n, uint64_t* out_total) {
    Query q(c); Workspace* w = q.w;
    const std::vector<uint64_t> sorted = sorted_unique(shards, n_shards);
    int rc = q.open(index, ops, n_ops, sorted.data(), (int64_t)sorted.size()); if (rc) return rc;
    const long long n_units = q.n_units;
    const uint64_t win_end = window_end(offset, limit);
    uint64_t seen = 0, written = 0;
    std::vector<ColUnit> units;
    for (long long u0 = 0; u0 < n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, n_units - u0);
        const uint2* info;
        rc = q.eval_info(u0, nu, info); if (rc) return rc;
        const uint64_t batch_out = col_units(info, u0, nu, sorted, offset, win_end, seen, units);
        if (batch_out && written + batch_out <= cap) {
            // d_emit: columns [batch_out] u64, then for Extract magnitudes [batch_out] u64 and sign bits [ceil(batch_out / 32)] u32
            const size_t vb = want_vals ? batch_out * 8 + ((batch_out + 31) / 32) * 4 : 0;
            rc = q.emit(units, batch_out * 8 + vb, [&](const ColUnit* d_units, int n, int grid) {
                unsigned long long* d_cols = (unsigned long long*)w->d_emit.p; unsigned long long* d_vals = d_cols + batch_out;
                columns_emit_kernel<<<grid, kEmitThreads, 0, w->stream>>>((const uint4*)w->d_bitmaps.p, d_units, n, d_cols);
                CUDA_TRY(cudaGetLastError()); q.launches++;
                if (want_vals) {
                    CUDA_TRY(cudaMemsetAsync(d_vals, 0, vb, w->stream));
                    extract_values_kernel<<<grid, kExtractThreads, 0, w->stream>>>(store_ref(c), fv_vals, depth_vals, (const uint4*)w->d_bitmaps.p, d_units, n,
                                                                                   d_vals, (unsigned int*)(d_vals + batch_out));
                    CUDA_TRY(cudaGetLastError()); q.launches++;
                }
                return 0;
            });
            if (rc) return rc;
            memcpy(out_cols + written, w->h_in.p, batch_out * 8);
            if (want_vals) {                               // sign-magnitude -> int64, wrapping like fragment.value: sign + 2^63 is INT64_MIN
                const uint64_t* mag = (const uint64_t*)w->h_in.p + batch_out;
                const uint32_t* sgn = (const uint32_t*)(mag + batch_out);
                for (uint64_t i = 0; i < batch_out; i++) out_vals[written + i] = (int64_t)(((sgn[i >> 5] >> (i & 31)) & 1u) ? 0ull - mag[i] : mag[i]);
            }
        }
        written += batch_out;                              // (past cap: counted, not written)
    }
    *out_n = written;
    if (out_total) *out_total = seen;
    q.finish();
    if (written > cap) return fail(FBGPU_E_NOSPACE, "output needs room for %llu columns", (unsigned long long)written);
    return FBGPU_OK;
}

extern "C" int fbgpu_columns(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards,
                             uint64_t offset, int64_t limit, uint64_t* out_cols, uint64_t cap, uint64_t* out_n, uint64_t* out_total) try {
    if (!c || !out_n || n_shards < 0 || (n_shards && !shards) || (cap && !out_cols)) return fail(FBGPU_E_INVALID, "null argument");
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    return columns_impl(c, index, ops, n_ops, shards, n_shards, offset, limit, false, 0, 0, out_cols, nullptr, cap, out_n, out_total);
} FBGPU_CATCH

extern "C" int fbgpu_extract(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                             const uint64_t* shards, int64_t n_shards, uint64_t offset, int64_t limit,
                             uint64_t* out_cols, int64_t* out_vals, uint64_t cap, uint64_t* out_n, uint64_t* out_total) try {
    if (!c || !out_n || n_shards < 0 || (n_shards && !shards) || (cap && (!out_cols || !out_vals)) || n_ops < 0 || (n_ops && !ops)) return fail(FBGPU_E_INVALID, "null argument");
    if (bit_depth < 0 || bit_depth > 64) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..64", bit_depth);
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    const std::vector<fbgpu_op> full = and_row(ops, n_ops, field, view, 0);    // <filter> ∩ exists (bsiExistsBit, row 0 of the bsig_ view; fragment.go:44)
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    return columns_impl(c, index, full.data(), (int32_t)full.size(), shards, n_shards, offset, limit, true, fv, bit_depth, out_cols, out_vals, cap, out_n, out_total);
} FBGPU_CATCH

// ------------------------------------------------------------------ Sort over an int field (sort_keys_kernel and the radix sort, kernels.cuh)
// The row is evaluated batch by batch as for fbgpu_extract.  Each batch's non-empty units are emitted in chunks of at most
// kSortChunk pairs straight into the call's pair buffer, behind the pairs kept so far: the columns by columns_emit_kernel, the
// keys by sort_keys_kernel from extract_values_kernel's output.  With a limit, the buffer is sorted and cut to the K = offset +
// limit first pairs before a chunk that would take it past 2K pairs.  At the end it is sorted once more and only the window is
// read back.
constexpr uint64_t kSortChunk = 1ull << 24;

static uint64_t sat_add(uint64_t a, uint64_t b) { return a + b < a ? ~0ull : a + b; }

// w->d_sort as two halves of `cap` elements for the radix sort's ping-pong; half `cur` holds the n kept so far.  An element is a
// (key, column) pair, [keys | columns] in each half, 32 bytes over both halves, or with keys_only (fbgpu_bsi_distinct) a key
// alone, 16 bytes.  The buffer outlives the call, like the workspace's other buffers; fbgpu_groupby_sparse also sorts in
// buffers of its own (`buf`).
struct SortPairs {
    Workspace* w; DevBuf* buf; uint64_t bound; uint64_t words; uint64_t cap, n = 0; int cur = 0;
    SortPairs(Workspace* ws, uint64_t max_pairs, bool keys_only = false, DevBuf* b = nullptr)
        : w(ws), buf(b ? b : &ws->d_sort), bound(max_pairs), words(keys_only ? 1 : 2), cap(buf->cap / (16 * words)) {}
    bool keys_only() const { return words == 1; }
    unsigned long long* keys(int h) const { return (unsigned long long*)buf->p + (size_t)h * words * cap; }
    unsigned long long* cols(int h) const { return keys_only() ? nullptr : keys(h) + cap; }
    // room for `need` elements (need <= bound); a buffer that has to grow takes the kept ones along into its half 0
    int reserve(uint64_t need) {
        if (need <= cap) return 0;
        if (need > 0xffffffffull) return fail(FBGPU_E_NOMEM, "the sort would hold %llu pairs on the device: more than 2^32", (unsigned long long)need);
        const uint64_t nc = std::min(std::max(need, cap + cap / 2), bound);
        DevBuf nb;
        if (nb.ensure((size_t)nc * 16 * words)) return FBGPU_E_NOMEM;
        if (n) {
            CUDA_TRY(cudaMemcpyAsync(nb.p, keys(cur), n * 8, cudaMemcpyDeviceToDevice, w->stream));
            if (!keys_only()) CUDA_TRY(cudaMemcpyAsync((unsigned long long*)nb.p + nc, cols(cur), n * 8, cudaMemcpyDeviceToDevice, w->stream));
            CUDA_TRY(cudaStreamSynchronize(w->stream));
        }
        buf->release(); *buf = nb; cap = nc; cur = 0;
        return 0;
    }
};

// stable sort of the kept elements by the low `bits` bits of their keys (8-bit digits, least significant first), then the first
// `keep` of them kept
static int sort_pairs(Query& q, SortPairs& sp, int bits, uint64_t keep) {
    Workspace* w = q.w;
    if (sp.n == 0) return 0;
    const uint64_t n_tiles = (sp.n + kSortTile - 1) / kSortTile, m = n_tiles * 256;
    if (w->d_counts.ensure((size_t)m * 4)) return FBGPU_E_NOMEM;
    unsigned int* counts = (unsigned int*)w->d_counts.p;
    for (int shift = 0; shift < bits; shift += 8) {
        sort_hist_kernel<<<(unsigned)n_tiles, kSortThreads, 0, w->stream>>>(sp.keys(sp.cur), sp.n, shift, counts);
        CUDA_TRY(cudaGetLastError());
        sort_scan_kernel<<<1, kSortScanThreads, 0, w->stream>>>(counts, m);
        CUDA_TRY(cudaGetLastError());
        if (sp.keys_only())
            sort_scatter_kernel<true><<<(unsigned)n_tiles, kSortThreads, 0, w->stream>>>(sp.keys(sp.cur), nullptr, sp.n, shift, counts, sp.keys(1 - sp.cur), nullptr);
        else
            sort_scatter_kernel<false><<<(unsigned)n_tiles, kSortThreads, 0, w->stream>>>(sp.keys(sp.cur), sp.cols(sp.cur), sp.n, shift, counts,
                                                                                         sp.keys(1 - sp.cur), sp.cols(1 - sp.cur));
        CUDA_TRY(cudaGetLastError());
        q.launches += 3;
        sp.cur = 1 - sp.cur;
    }
    sp.n = std::min(sp.n, keep);
    return 0;
}

// the chunk of one batch's emit units that starts at units[a]: units [a, b) holding at most kSortChunk columns (at least one
// unit), re-based to out_off 0 in `chunk`.  Returns b; *cn = the chunk's columns.
static size_t next_chunk(const std::vector<ColUnit>& units, size_t a, uint64_t batch_out, std::vector<ColUnit>& chunk, uint64_t* cn) {
    const uint64_t base = units[a].out_off;
    size_t b = a + 1;
    while (b < units.size() && units[b].out_off + (units[b].last - units[b].first) - base <= kSortChunk) b++;
    *cn = (b < units.size() ? units[b].out_off : batch_out) - base;
    chunk.assign(units.begin() + (long)a, units.begin() + (long)b);
    for (ColUnit& cu : chunk) cu.out_off -= base;
    return b;
}

// one chunk's cn sort keys to keys_out (sort_keys_kernel from extract_values_kernel's magnitudes and signs) and, unless
// cols_out is NULL, its columns to cols_out (columns_emit_kernel)
static int emit_sort_keys(Query& q, const std::vector<ColUnit>& chunk, uint64_t cn, uint32_t fv, int depth, bool desc,
                          unsigned long long* keys_out, unsigned long long* cols_out) {
    Workspace* w = q.w;
    // d_emit: magnitudes [cn] u64, then sign bits [ceil(cn / 32)] u32
    const size_t vb = cn * 8 + ((cn + 31) / 32) * 4;
    return q.emit_on_device(chunk, vb, [&](const ColUnit* d_units, int n, int grid) {
        unsigned long long* d_mag = (unsigned long long*)w->d_emit.p;
        unsigned int* d_sign = (unsigned int*)(d_mag + cn);
        if (cols_out) {
            columns_emit_kernel<<<grid, kEmitThreads, 0, w->stream>>>((const uint4*)w->d_bitmaps.p, d_units, n, cols_out);
            CUDA_TRY(cudaGetLastError());
            q.launches++;
        }
        CUDA_TRY(cudaMemsetAsync(d_mag, 0, vb, w->stream));
        extract_values_kernel<<<grid, kExtractThreads, 0, w->stream>>>(store_ref(q.c), fv, depth, (const uint4*)w->d_bitmaps.p, d_units, n, d_mag, d_sign);
        CUDA_TRY(cudaGetLastError());
        const unsigned kgrid = (unsigned)std::min<uint64_t>((cn + kSortThreads - 1) / kSortThreads, (uint64_t)q.c->sm_count * 8);
        sort_keys_kernel<<<kgrid, kSortThreads, 0, w->stream>>>(d_mag, d_sign, cn, depth, desc ? 1 : 0, keys_out);
        CUDA_TRY(cudaGetLastError());
        q.launches += 2;
        return 0;
    });
}

// the pairs [offset, min(win_end, |row|)) of the row <ops> ∩ exists(field) in sort order (store lock held): columns and stored
// values into cols / vals, |row| into *total
static int bsi_sort_run(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int depth,
                        const uint64_t* shards, int64_t n_shards, bool desc, uint64_t offset, uint64_t win_end,
                        std::vector<uint64_t>& cols, std::vector<int64_t>& vals, uint64_t* total) {
    const std::vector<fbgpu_op> full = and_row(ops, n_ops, field, view, 0);    // as for fbgpu_extract
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    Query q(c); Workspace* w = q.w;
    const std::vector<uint64_t> sorted = sorted_unique(shards, n_shards);      // units in ascending column order
    int rc = q.open(index, full.data(), (int32_t)full.size(), sorted.data(), (int64_t)sorted.size()); if (rc) return rc;
    const bool limited = win_end != ~0ull;
    const uint64_t K = win_end, twice_k = sat_add(K, K);
    const int bits = sort_key_bits(depth);
    SortPairs sp(w, limited ? std::max(twice_k, sat_add(K, kSortChunk)) : ~0ull);
    uint64_t seen = 0;
    std::vector<ColUnit> units, chunk;
    for (long long u0 = 0; u0 < q.n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, q.n_units - u0);
        const uint2* info;
        rc = q.eval_info(u0, nu, info); if (rc) return rc;
        const uint64_t batch_out = col_units(info, u0, nu, sorted, 0, ~0ull, seen, units);
        for (size_t a = 0; a < units.size();) {
            uint64_t cn;
            const size_t b = next_chunk(units, a, batch_out, chunk, &cn);
            if (limited && sp.n > K && sp.n + cn > twice_k) { rc = sort_pairs(q, sp, bits, K); if (rc) return rc; }
            rc = sp.reserve(sp.n + cn); if (rc) return rc;
            rc = emit_sort_keys(q, chunk, cn, fv, depth, desc, sp.keys(sp.cur) + sp.n, sp.cols(sp.cur) + sp.n); if (rc) return rc;
            sp.n += cn;
            a = b;
        }
        CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        q.add_elapsed();
    }
    *total = seen;
    // sp.n = min(K, |row|) after the last sort; the window is its part from offset on (offset <= K)
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    rc = sort_pairs(q, sp, bits, K); if (rc) return rc;
    const uint64_t lo = std::min(offset, sp.n), cnt = sp.n - lo;
    if (w->h_out.ensure(std::max<size_t>(cnt * 16, 16))) return FBGPU_E_NOMEM;
    const uint64_t* h_keys = (const uint64_t*)w->h_out.p; const uint64_t* h_cols = h_keys + cnt;
    if (cnt) {
        CUDA_TRY(cudaMemcpyAsync(w->h_out.p, sp.keys(sp.cur) + lo, cnt * 8, cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaMemcpyAsync((uint64_t*)w->h_out.p + cnt, sp.cols(sp.cur) + lo, cnt * 8, cudaMemcpyDeviceToHost, w->stream));
    }
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    q.add_elapsed();
    const uint64_t mask = sort_key_mask(depth);
    cols.assign(h_cols, h_cols + cnt);
    vals.resize(cnt);
    for (uint64_t i = 0; i < cnt; i++) {                 // sort_keys_kernel backwards
        const uint64_t k = desc ? ~h_keys[i] & mask : h_keys[i];
        vals[i] = (int64_t)(depth < 64 ? k - (1ull << depth) : k ^ (1ull << 63));
    }
    q.finish();
    return FBGPU_OK;
}

// the FBGPU_E_INVALID checks of fbgpu_bsi_sort and its node form, with fbgpu_extract's messages
static int bsi_sort_args(const void* handle, const fbgpu_op* ops, int32_t n_ops, int32_t bit_depth, const uint64_t* shards, int64_t n_shards,
                         const uint64_t* out_cols, const int64_t* out_vals, uint64_t cap, const uint64_t* out_n) {
    if (!handle || !out_n || n_shards < 0 || (n_shards && !shards) || (cap && (!out_cols || !out_vals)) || n_ops < 0 || (n_ops && !ops)) return fail(FBGPU_E_INVALID, "null argument");
    if (bit_depth < 0 || bit_depth > 64) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..64", bit_depth);
    return 0;
}

// a window into the caller's arrays under the NOSPACE contract: *out_n = its size, nothing written when it exceeds cap
static int write_window(const std::vector<uint64_t>& cols, const std::vector<int64_t>& vals, uint64_t* out_cols, int64_t* out_vals, uint64_t cap, uint64_t* out_n) {
    *out_n = cols.size();
    if (cols.size() > cap) return fail(FBGPU_E_NOSPACE, "output needs room for %llu columns", (unsigned long long)cols.size());
    if (!cols.empty()) { memcpy(out_cols, cols.data(), cols.size() * 8); memcpy(out_vals, vals.data(), vals.size() * 8); }
    return FBGPU_OK;
}

extern "C" int fbgpu_bsi_sort(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                              const uint64_t* shards, int64_t n_shards, int32_t desc, uint64_t offset, int64_t limit,
                              uint64_t* out_cols, int64_t* out_vals, uint64_t cap, uint64_t* out_n, uint64_t* out_total) try {
    int rc = bsi_sort_args(c, ops, n_ops, bit_depth, shards, n_shards, out_cols, out_vals, cap, out_n); if (rc) return rc;
    std::shared_lock<std::shared_mutex> lk;
    rc = begin_query(c, lk); if (rc) return rc;
    std::vector<uint64_t> cols; std::vector<int64_t> vals; uint64_t total = 0;
    rc = bsi_sort_run(c, index, ops, n_ops, field, view, bit_depth, shards, n_shards, desc != 0, offset, window_end(offset, limit), cols, vals, &total);
    if (rc) return rc;
    if (out_total) *out_total = total;
    return write_window(cols, vals, out_cols, out_vals, cap, out_n);
} FBGPU_CATCH

// ------------------------------------------------------------------ Distinct values of an int field (the sort on keys alone, then one key per run)
// The row is evaluated batch by batch and emitted in chunks as for fbgpu_bsi_sort, keys only (sort_keys_kernel, ascending).  Before
// a chunk that would take the buffer past twice the U distinct keys left by the last dedupe, the buffer is sorted and deduped
// (distinct_heads_kernel, sort_scan_kernel, distinct_compact_kernel); once more at the end, and only the U keys are read back.

// sorts the kept keys and keeps the first of each run of equal keys: sk.n becomes the number of distinct keys
static int distinct_keys(Query& q, SortPairs& sk, int bits) {
    int rc = sort_pairs(q, sk, bits, ~0ull); if (rc) return rc;
    if (sk.n == 0) return 0;
    Workspace* w = q.w;
    const uint64_t n_tiles = (sk.n + kSortTile - 1) / kSortTile;
    if (w->d_counts.ensure((size_t)(n_tiles + 1) * 4) || w->h_out.ensure(8)) return FBGPU_E_NOMEM;
    unsigned int* counts = (unsigned int*)w->d_counts.p;                    // [n_tiles] heads per tile, then their total
    distinct_heads_kernel<<<(unsigned)n_tiles, kSortThreads, 0, w->stream>>>(sk.keys(sk.cur), sk.n, counts);
    CUDA_TRY(cudaGetLastError());
    sort_scan_kernel<<<1, kSortScanThreads, 0, w->stream>>>(counts, n_tiles + 1);
    CUDA_TRY(cudaGetLastError());
    distinct_compact_kernel<<<(unsigned)n_tiles, kSortThreads, 0, w->stream>>>(sk.keys(sk.cur), sk.n, counts, sk.keys(1 - sk.cur));
    CUDA_TRY(cudaGetLastError());
    q.launches += 3;
    sk.cur = 1 - sk.cur;
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, counts + n_tiles, 4, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    sk.n = *(const unsigned int*)w->h_out.p;
    return 0;
}

// the distinct stored values of the row <ops> ∩ exists(field), ascending, into vals (store lock held); |row| into *total
static int bsi_distinct_run(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int depth,
                            const uint64_t* shards, int64_t n_shards, std::vector<int64_t>& vals, uint64_t* total) {
    const std::vector<fbgpu_op> full = and_row(ops, n_ops, field, view, 0);    // as for fbgpu_extract
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    Query q(c); Workspace* w = q.w;
    const std::vector<uint64_t> sorted = sorted_unique(shards, n_shards);
    int rc = q.open(index, full.data(), (int32_t)full.size(), sorted.data(), (int64_t)sorted.size()); if (rc) return rc;
    const int bits = sort_key_bits(depth);
    SortPairs sk(w, kSortChunk, true);              // bound: max(2U, U + kSortChunk) keys, U the distinct keys after the last dedupe
    uint64_t u = 0, seen = 0;
    std::vector<ColUnit> units, chunk;
    for (long long u0 = 0; u0 < q.n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, q.n_units - u0);
        const uint2* info;
        rc = q.eval_info(u0, nu, info); if (rc) return rc;
        const uint64_t batch_out = col_units(info, u0, nu, sorted, 0, ~0ull, seen, units);
        for (size_t a = 0; a < units.size();) {
            uint64_t cn;
            const size_t b = next_chunk(units, a, batch_out, chunk, &cn);
            if (sk.n > u && sk.n + cn > sat_add(u, u)) {
                rc = distinct_keys(q, sk, bits); if (rc) return rc;
                u = sk.n;
                sk.bound = std::max(sat_add(u, u), sat_add(u, kSortChunk));
            }
            rc = sk.reserve(sk.n + cn); if (rc) return rc;
            rc = emit_sort_keys(q, chunk, cn, fv, depth, false, sk.keys(sk.cur) + sk.n, nullptr); if (rc) return rc;
            sk.n += cn;
            a = b;
        }
        CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        q.add_elapsed();
    }
    *total = seen;
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    rc = distinct_keys(q, sk, bits); if (rc) return rc;
    const uint64_t cnt = sk.n;
    if (w->h_out.ensure(std::max<size_t>(cnt * 8, 8))) return FBGPU_E_NOMEM;
    if (cnt) CUDA_TRY(cudaMemcpyAsync(w->h_out.p, sk.keys(sk.cur), cnt * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    q.add_elapsed();
    const uint64_t* h_keys = (const uint64_t*)w->h_out.p;
    vals.resize(cnt);
    for (uint64_t i = 0; i < cnt; i++)                   // sort_keys_kernel backwards, as in bsi_sort_run
        vals[i] = (int64_t)(depth < 64 ? h_keys[i] - (1ull << depth) : h_keys[i] ^ (1ull << 63));
    q.finish();
    return FBGPU_OK;
}

// a value list into the caller's array under the NOSPACE contract: *out_n = its size, nothing written when it exceeds cap
static int write_values(const std::vector<int64_t>& vals, int64_t* out_vals, uint64_t cap, uint64_t* out_n) {
    *out_n = vals.size();
    if (vals.size() > cap) return fail(FBGPU_E_NOSPACE, "output needs room for %llu values", (unsigned long long)vals.size());
    if (!vals.empty()) memcpy(out_vals, vals.data(), vals.size() * 8);
    return FBGPU_OK;
}

extern "C" int fbgpu_bsi_distinct(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                                  const uint64_t* shards, int64_t n_shards, int64_t* out_vals, uint64_t cap, uint64_t* out_n, uint64_t* out_total) try {
    // fbgpu_bsi_sort's checks, out_vals being the only output array
    int rc = bsi_sort_args(c, ops, n_ops, bit_depth, shards, n_shards, (const uint64_t*)out_vals, out_vals, cap, out_n); if (rc) return rc;
    std::shared_lock<std::shared_mutex> lk;
    rc = begin_query(c, lk); if (rc) return rc;
    std::vector<int64_t> vals; uint64_t total = 0;
    rc = bsi_distinct_run(c, index, ops, n_ops, field, view, bit_depth, shards, n_shards, vals, &total); if (rc) return rc;
    if (out_total) *out_total = total;
    return write_values(vals, out_vals, cap, out_n);
} FBGPU_CATCH

// ------------------------------------------------------------------ The rows of a set-like field per column (extract_rows_kernel, kernels.cuh)
// R is evaluated batch by batch and its window cut into per-unit rank ranges as for fbgpu_columns.  Per batch, the count pass
// gives every window column its number of rows; the host turns them into the columns' offsets and cuts the batch into chunks
// at column boundaries, of at most kSortChunk columns and kSortChunk (column, row) pairs each, a column holding more rows than
// that being a chunk of its own.  Per chunk, columns_emit_kernel writes the columns, the emit pass the pairs keyed
// (i << kbits) | k (i the column in the chunk, k the row's rank in its fragment), and the radix sort orders them by column,
// then by row id.  Only the columns and the row ids are read back.

// the parts of a batch's units that fall in its window columns [a, b), re-based to out_off 0
static void chunk_units(const std::vector<ColUnit>& units, uint64_t a, uint64_t b, std::vector<ColUnit>& chunk) {
    chunk.clear();
    for (const ColUnit& u : units) {
        const uint64_t lo = std::max<uint64_t>(u.out_off, a), hi = std::min<uint64_t>(u.out_off + (u.last - u.first), b);
        if (lo >= hi) continue;
        ColUnit cu = u;
        cu.first = u.first + (uint32_t)(lo - u.out_off); cu.last = cu.first + (uint32_t)(hi - lo); cu.out_off = lo - a;
        chunk.push_back(cu);
    }
}

static int bit_width(uint64_t x) { return x ? 64 - __builtin_clzll(x) : 0; }

// the window's columns, the offsets of their lists and the row ids of the lists (store lock held); |R| into *total
static int extract_rows_run(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view,
                            const uint64_t* shards, int64_t n_shards, uint64_t offset, int64_t limit,
                            std::vector<uint64_t>& cols, std::vector<uint64_t>& offs, std::vector<uint64_t>& rows, uint64_t* total) {
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    Query q(c); Workspace* w = q.w;
    const std::vector<uint64_t> sorted = sorted_unique(shards, n_shards);
    int rc = q.open(index, ops, n_ops, sorted.data(), (int64_t)sorted.size()); if (rc) return rc;
    uint32_t max_rows = 0;                               // the most rows of one listed fragment: a row rank takes kbits bits
    if (fv != kNoView)
        for (uint64_t s : sorted) if (s < c->shardmaps[fv].size() && c->shardmaps[fv][s] >= 0) max_rows = std::max(max_rows, c->frags[(size_t)c->shardmaps[fv][s]].n_rows);
    const int kbits = bit_width(max_rows ? max_rows - 1 : 0);
    const uint64_t win_end = window_end(offset, limit);
    SortPairs sp(w, kSortChunk);
    uint64_t seen = 0;
    std::vector<ColUnit> units, chunk;
    std::vector<uint32_t> cnt;
    cols.clear(); rows.clear(); offs.assign(1, 0);
    for (long long u0 = 0; u0 < q.n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, q.n_units - u0);
        const uint2* info;
        rc = q.eval_info(u0, nu, info); if (rc) return rc;
        const uint64_t batch_out = col_units(info, u0, nu, sorted, offset, win_end, seen, units);
        if (batch_out) {
            if (w->d_cells.ensure(batch_out * 4) || w->h_out.ensure(batch_out * 4)) return FBGPU_E_NOMEM;
            unsigned int* d_cells = (unsigned int*)w->d_cells.p;
            uint32_t* h_cells = (uint32_t*)w->h_out.p;
            CUDA_TRY(cudaMemsetAsync(d_cells, 0, batch_out * 4, w->stream));
            rc = q.emit_on_device(units, 0, [&](const ColUnit* d_units, int n, int grid) {
                extract_rows_kernel<ErOut::kCount><<<grid, kExtractThreads, 0, w->stream>>>(store_ref(c), fv, (const uint4*)w->d_bitmaps.p, d_units, n,
                                                                                            d_cells, 0, nullptr, nullptr);
                CUDA_TRY(cudaGetLastError()); q.launches++;
                return 0;
            });
            if (rc) return rc;
            CUDA_TRY(cudaMemcpyAsync(h_cells, d_cells, batch_out * 4, cudaMemcpyDeviceToHost, w->stream));
            CUDA_TRY(cudaStreamSynchronize(w->stream));
            cnt.assign(h_cells, h_cells + batch_out);
            const size_t c0 = cols.size();               // the window rank of the batch's first column
            cols.resize(c0 + batch_out);
            for (uint64_t i = 0; i < batch_out; i++) offs.push_back(offs.back() + cnt[i]);
            rows.resize(offs.back());
            for (uint64_t a = 0; a < batch_out;) {
                uint64_t b = a, pairs = 0;
                while (b < batch_out && b - a < kSortChunk && (b == a || pairs + cnt[b] <= kSortChunk)) pairs += cnt[b++];
                chunk_units(units, a, b, chunk);
                const uint64_t p0 = offs[c0 + a];
                for (uint64_t i = a; i < b; i++) h_cells[i] = (uint32_t)(offs[c0 + i] - p0);     // column i's first place in the chunk's pairs
                CUDA_TRY(cudaMemcpyAsync(d_cells + a, h_cells + a, (b - a) * 4, cudaMemcpyHostToDevice, w->stream));
                sp.n = 0; sp.bound = std::max(kSortChunk, pairs);
                rc = sp.reserve(std::max(pairs, b - a)); if (rc) return rc;
                rc = q.emit_on_device(chunk, 0, [&](const ColUnit* d_units, int n, int grid) {
                    unsigned long long* d_cols = sp.keys(1 - sp.cur);         // the sort's other half: read back before its first pass
                    columns_emit_kernel<<<grid, kEmitThreads, 0, w->stream>>>((const uint4*)w->d_bitmaps.p, d_units, n, d_cols);
                    CUDA_TRY(cudaGetLastError());
                    CUDA_TRY(cudaMemcpyAsync(cols.data() + c0 + a, d_cols, (b - a) * 8, cudaMemcpyDeviceToHost, w->stream));
                    q.launches++;
                    if (pairs) {
                        extract_rows_kernel<ErOut::kEmit><<<grid, kExtractThreads, 0, w->stream>>>(store_ref(c), fv, (const uint4*)w->d_bitmaps.p, d_units, n,
                                                                                                   d_cells + a, kbits, sp.keys(sp.cur), sp.cols(sp.cur));
                        CUDA_TRY(cudaGetLastError()); q.launches++;
                    }
                    return 0;
                });
                if (rc) return rc;
                sp.n = pairs;
                rc = sort_pairs(q, sp, bit_width(b - a - 1) + kbits, ~0ull); if (rc) return rc;
                if (pairs) CUDA_TRY(cudaMemcpyAsync(rows.data() + p0, sp.cols(sp.cur), pairs * 8, cudaMemcpyDeviceToHost, w->stream));
                CUDA_TRY(cudaStreamSynchronize(w->stream));
                a = b;
            }
        }
        CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        q.add_elapsed();
    }
    *total = seen;
    q.finish();
    return FBGPU_OK;
}

extern "C" int fbgpu_extract_rows(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view,
                                  const uint64_t* shards, int64_t n_shards, uint64_t offset, int64_t limit,
                                  uint64_t* out_cols, uint64_t* out_offsets, uint64_t cap_cols, uint64_t* out_rows, uint64_t cap_rows,
                                  uint64_t* out_n_cols, uint64_t* out_n_rows, uint64_t* out_total) try {
    if (!c || !out_n_cols || !out_n_rows || (cap_cols && (!out_cols || !out_offsets)) || (cap_rows && !out_rows) || n_ops < 0 || (n_ops && !ops) ||
        n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    std::vector<uint64_t> cols, offs, rows; uint64_t total = 0;
    rc = extract_rows_run(c, index, ops, n_ops, field, view, shards, n_shards, offset, limit, cols, offs, rows, &total); if (rc) return rc;
    if (out_total) *out_total = total;
    *out_n_cols = cols.size(); *out_n_rows = rows.size();
    if (cols.size() > cap_cols || rows.size() > cap_rows)
        return fail(FBGPU_E_NOSPACE, "output needs room for %llu columns and %llu row ids", (unsigned long long)cols.size(), (unsigned long long)rows.size());
    if (!cols.empty()) memcpy(out_cols, cols.data(), cols.size() * 8);
    if (out_offsets) memcpy(out_offsets, offs.data(), offs.size() * 8);
    if (!rows.empty()) memcpy(out_rows, rows.data(), rows.size() * 8);
    return FBGPU_OK;
} FBGPU_CATCH

// ------------------------------------------------------------------ BSI Min / Max (one pass over the planes)
extern "C" int fbgpu_bsi_minmax(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                                const uint64_t* shards, int64_t n_shards, int32_t want_max, int64_t* out_val, uint64_t* out_count) try {
    if (!c || !out_val || !out_count || n_shards < 0 || (n_shards && !shards) || n_ops < 0 || (n_ops && !ops)) return fail(FBGPU_E_INVALID, "null argument");
    if (bit_depth < 0 || bit_depth > 64) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..64", bit_depth);
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    *out_val = 0; *out_count = 0;
    const std::vector<fbgpu_op> full = and_row(ops, n_ops, field, view, 0);    // consider = <filter> ∩ exists (fragment.go:753-757)
    Query q(c); Workspace* w = q.w;
    rc = q.open(index, full.data(), (int32_t)full.size(), shards, n_shards); if (rc) return rc;
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    bool have = false; int64_t best = 0; uint64_t best_n = 0;
    for (long long u0 = 0; u0 < q.n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, q.n_units - u0);
        // (the buffers are grown before ev0: the bracket holds no allocation)
        if (w->d_bitmaps.ensure((size_t)nu * 8192) || w->d_counts.ensure((size_t)nu * sizeof(MinMaxUnit)) || w->h_out.ensure((size_t)nu * sizeof(MinMaxUnit))) return FBGPU_E_NOMEM;
        CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
        rc = q.eval(u0, nu); if (rc) return rc;
        const long long grid = std::min<long long>(nu, (long long)c->sm_count * 8);
        bsi_minmax_kernel<<<(unsigned)grid, kEvalThreads, 0, w->stream>>>(store_ref(c), fv, bit_depth, (const uint4*)w->d_bitmaps.p, q.d_shards + u0 / kSlotsPerRow, nu, want_max ? 1 : 0, (MinMaxUnit*)w->d_counts.p);
        CUDA_TRY(cudaGetLastError()); q.launches++;
        CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
        CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, (size_t)nu * sizeof(MinMaxUnit), cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        const MinMaxUnit* r = (const MinMaxUnit*)w->h_out.p;
        for (long long u = 0; u < nu; u++) {                // ValCount.Larger / Smaller: keep the extreme, add the counts of equal values
            if (!r[u].cnt) continue;
            if (!have || (want_max ? r[u].val > best : r[u].val < best)) { have = true; best = r[u].val; best_n = r[u].cnt; }
            else if (r[u].val == best) best_n += r[u].cnt;
        }
        q.add_elapsed();
    }
    if (have) { *out_val = best; *out_count = best_n; }
    q.finish();
    return FBGPU_OK;
} FBGPU_CATCH

extern "C" int fbgpu_bsi_sum(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                             const uint64_t* shards, int64_t n_shards, int64_t* out_sum, uint64_t* out_count) try {
    if (!c || !out_sum || !out_count || n_shards < 0 || (n_shards && !shards) || n_ops < 0 || (n_ops && !ops)) return fail(FBGPU_E_INVALID, "null argument");
    if (bit_depth < 0 || bit_depth > 64) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..64", bit_depth);
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    *out_sum = 0; *out_count = 0;
    const std::vector<fbgpu_op> full = and_row(ops, n_ops, field, view, 0);
    Query q(c); Workspace* w = q.w;
    rc = q.open(index, full.data(), (int32_t)full.size(), shards, n_shards); if (rc) return rc;
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    const size_t n_acc = 1 + 2 * (size_t)bit_depth;
    if (w->d_counts.ensure(n_acc * 8) || w->h_out.ensure(n_acc * 8)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, n_acc * 8, w->stream));
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    for (long long u0 = 0; u0 < q.n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, q.n_units - u0);
        rc = q.eval(u0, nu); if (rc) return rc;
        const long long grid = std::min<long long>(nu, (long long)c->sm_count * 8);
        bsi_sum_kernel<<<(unsigned)grid, kEvalThreads, 0, w->stream>>>(store_ref(c), fv, bit_depth, (const uint4*)w->d_bitmaps.p, q.d_shards + u0 / kSlotsPerRow, nu, (unsigned long long*)w->d_counts.p);
        CUDA_TRY(cudaGetLastError()); q.launches++;
    }
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, n_acc * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    const uint64_t* acc = (const uint64_t*)w->h_out.p;
    uint64_t sum = 0;                                       // wrapping, like the reference's int64 arithmetic
    for (int i = 0; i < bit_depth; i++) sum += (acc[1 + 2 * i] - acc[2 + 2 * i]) << i;
    *out_sum = (int64_t)sum; *out_count = acc[0];
    q.add_elapsed();
    q.finish();
    return FBGPU_OK;
} FBGPU_CATCH

// ------------------------------------------------------------------ BSI order statistics (radix select over the planes, kernels.cuh)
// The row is evaluated batch by batch straight into rank 0's slot of the call's candidate buffer (d_select: 8 KiB per unit per
// distinct rank, plus one live mask per unit), then the select steps run over every unit of the call at once, chained on the
// stream: no host round trip until the one D2H copy of the rank states.
static_assert(kSelMaxRanks == FBGPU_SELECT_MAX_RANKS, "kernels.cuh and fbgpu.h disagree on the rank cap");
extern "C" int fbgpu_bsi_select(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                                const uint64_t* shards, int64_t n_shards, const uint64_t* ranks, int32_t n_ranks,
                                int64_t* out_vals, uint64_t* out_counts, uint64_t* out_total) try {
    if (!c || !out_total || n_shards < 0 || (n_shards && !shards) || n_ops < 0 || (n_ops && !ops) || n_ranks < 0 || (n_ranks && (!ranks || !out_vals)))
        return fail(FBGPU_E_INVALID, "null argument");
    if (bit_depth < 0 || bit_depth > 63) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..63", bit_depth);     // the sort key takes depth + 1 bits
    if (n_ranks > FBGPU_SELECT_MAX_RANKS) return fail(FBGPU_E_INVALID, "%d ranks: at most %d per call", n_ranks, FBGPU_SELECT_MAX_RANKS);
    if (c->comm || c->n_ranks > 1) return fail(FBGPU_E_COMM, "fbgpu_bsi_select is local to one context: order statistics of the ranks' shares do not merge");
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    *out_total = 0;
    const std::vector<uint64_t> uniq = sorted_unique(ranks, n_ranks);     // the device works on distinct ranks (at least one: slot 0 holds the row)
    const int nr = std::max(1, (int)uniq.size());
    const std::vector<fbgpu_op> full = and_row(ops, n_ops, field, view, 0);    // the row = <filter> ∩ exists, as for Min / Max
    Query q(c); Workspace* w = q.w;
    rc = q.open(index, full.data(), (int32_t)full.size(), shards, n_shards); if (rc) return rc;
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    const long long n_units = q.n_units;
    // d_counts: [SelRank x kSelMaxRanks][buckets kSelMaxRanks x kSelBuckets][total]
    const size_t st_bytes = kSelMaxRanks * sizeof(SelRank), bk_bytes = kSelMaxRanks * kSelBuckets * 8, ctl_bytes = st_bytes + bk_bytes + 8;
    if (w->d_counts.ensure(ctl_bytes) || w->h_out.ensure(ctl_bytes)) return FBGPU_E_NOMEM;
    const size_t cand_bytes = (size_t)n_units * (size_t)nr * 8192;
    if (n_units > 0 && w->d_select.ensure(cand_bytes + (size_t)n_units * 4)) return FBGPU_E_NOMEM;
    memset(w->h_out.p, 0, ctl_bytes);                       // (h_out is free: the previous user of the lease drained its copies)
    SelRank* hs = (SelRank*)w->h_out.p;
    for (int r = 0; r < (int)uniq.size(); r++) hs[r].rank = uniq[(size_t)r];
    CUDA_TRY(cudaMemcpyAsync(w->d_counts.p, w->h_out.p, ctl_bytes, cudaMemcpyHostToDevice, w->stream));
    SelRank* d_state = (SelRank*)w->d_counts.p;
    unsigned long long* d_buckets = (unsigned long long*)((uint8_t*)w->d_counts.p + st_bytes);
    unsigned long long* d_total = d_buckets + kSelMaxRanks * kSelBuckets;
    uint4* d_cand = (uint4*)w->d_select.p;
    unsigned int* d_live = n_units > 0 ? (unsigned int*)((uint8_t*)w->d_select.p + cand_bytes) : nullptr;
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    if (n_units > 0) {
        for (long long u0 = 0; u0 < n_units; u0 += c->unit_batch) {
            rc = q.eval(u0, std::min(c->unit_batch, n_units - u0), false, d_cand + (size_t)u0 * 512); if (rc) return rc;
        }
        const int n_steps = (bit_depth + 1 + kSelDigit - 1) / kSelDigit;
        const long long grid = std::min<long long>(n_units, (long long)c->sm_count * 4);
        for (int s = 0; s < n_steps; s++) {
            bsi_select_step_kernel<<<(unsigned)grid, kEvalThreads, 0, w->stream>>>(store_ref(c), fv, bit_depth, s, s == n_steps - 1 ? 1 : 0, d_cand, q.d_shards, n_units, nr,
                                                                                   d_state, d_live, d_buckets);
            CUDA_TRY(cudaGetLastError());
            bsi_select_decide_kernel<<<1, 32, 0, w->stream>>>(bit_depth, s, nr, d_state, d_buckets, d_total);
            CUDA_TRY(cudaGetLastError());
            q.launches += 2;
        }
    }
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, ctl_bytes, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    q.add_elapsed();
    q.finish();
    const SelRank* rs = (const SelRank*)w->h_out.p;
    const uint64_t total = *(const uint64_t*)((const uint8_t*)w->h_out.p + st_bytes + bk_bytes);
    *out_total = total;
    const uint64_t low = bit_depth ? ~0ull >> (64 - bit_depth) : 0ull;
    for (int i = 0; i < n_ranks; i++) {
        if (ranks[i] >= total) return fail(FBGPU_E_INVALID, "rank %llu outside the %llu sorted values", (unsigned long long)ranks[i], (unsigned long long)total);
        const SelRank& R = rs[std::lower_bound(uniq.begin(), uniq.end(), ranks[i]) - uniq.begin()];
        const bool neg = ((R.key >> bit_depth) & 1ull) == 0;   // key -> sign-magnitude (kernels.cuh)
        const uint64_t mag = neg ? ~R.key & low : R.key & low;
        out_vals[i] = neg ? -(int64_t)mag : (int64_t)mag;
        if (out_counts) out_counts[i] = R.count;
    }
    return FBGPU_OK;
} FBGPU_CATCH

// ------------------------------------------------------------------ per-row counts (TopK / TopN ids)
// fvs: the view slots each row is the union over.  One slot: row_count_kernel; several: row_count_views_kernel, whose counts
// are always summed over the shards (per_shard and cut need one slot).  cut: TopN's per-shard cut-offs with `filter` as the Src
// (row_count_kernel<kCutoff>, which gets the Src units' {N, runs} from the evaluation pass; cut->info is not read).
static int row_counts_impl(fbgpu_ctx* c, uint32_t index, const std::vector<uint32_t>& fvs, const std::vector<uint64_t>& rows, const fbgpu_op* filter, int32_t n_filter_ops,
                           const uint64_t* shards, int64_t n_shards, std::vector<uint64_t>& counts, bool reduce = true, bool per_shard = false,
                           const RcCut* cut = nullptr) {
    counts.assign(rows.size() * (per_shard ? (size_t)n_shards : 1), 0);
    if (rows.empty()) return 0;
    const bool have_filter = filter && n_filter_ops > 0;
    Query q(c); Workspace* w = q.w;
    int rc = have_filter ? q.open(index, filter, n_filter_ops, shards, n_shards) : q.open(shards, n_shards); if (rc) return rc;
    size_t nr = rows.size(), nv = fvs.size();
    const size_t n_out = counts.size();                     // nr, or n_shards x nr (per_shard: one row of the matrix per listed shard)
    if (w->d_rows.ensure(nr * 8 + nv * 4) || w->d_counts.ensure(n_out * 8) || w->h_out.ensure(n_out * 8)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemcpyAsync(w->d_rows.p, rows.data(), nr * 8, cudaMemcpyHostToDevice, w->stream));       // [rows | view slots]
    const uint32_t* d_fvs = (const uint32_t*)((const uint64_t*)w->d_rows.p + nr);
    if (nv > 1) CUDA_TRY(cudaMemcpyAsync((void*)d_fvs, fvs.data(), nv * 4, cudaMemcpyHostToDevice, w->stream));
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, n_out * 8, w->stream));
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    const int64_t batch = have_filter ? c->unit_batch / kSlotsPerRow : n_shards;
    for (int64_t s0 = 0; s0 < n_shards; s0 += batch) {
        int64_t ns = std::min(batch, n_shards - s0);
        if (have_filter) { rc = q.eval(s0 * kSlotsPerRow, ns * kSlotsPerRow, cut != nullptr); if (rc) return rc; }
        long long tasks = (long long)ns * (long long)nr;
        long long grid = std::min<long long>((tasks + kPairWarps - 1) / kPairWarps, (long long)c->sm_count * 3);
        const uint32_t fv = fvs[0];
        if (nv > 1)
            row_count_views_kernel<<<(unsigned)grid, kPairWarps * 32, kPairWarps * 8192, w->stream>>>(store_ref(c), d_fvs, (int)nv, (const uint64_t*)w->d_rows.p, (int)nr,
                q.d_shards + s0, ns, have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, (unsigned long long*)w->d_counts.p);
        else if (per_shard)
            row_count_kernel<RcOut::kPerShard><<<(unsigned)grid, kPairWarps * 32, kPairWarps * 8192, w->stream>>>(store_ref(c), fv, (const uint64_t*)w->d_rows.p, (int)nr, q.d_shards + s0, ns,
                have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, (unsigned long long*)w->d_counts.p + (size_t)s0 * nr, RcCut{});
        else if (cut)
            row_count_kernel<RcOut::kCutoff><<<(unsigned)grid, kPairWarps * 32, kPairWarps * 8192, w->stream>>>(store_ref(c), fv, (const uint64_t*)w->d_rows.p, (int)nr, q.d_shards + s0, ns,
                have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, (unsigned long long*)w->d_counts.p,
                RcCut{ have_filter ? (const uint2*)w->d_info.p : nullptr, cut->min_threshold, cut->tanimoto });
        else
            row_count_kernel<RcOut::kSummed><<<(unsigned)grid, kPairWarps * 32, kPairWarps * 8192, w->stream>>>(store_ref(c), fv, (const uint64_t*)w->d_rows.p, (int)nr, q.d_shards + s0, ns,
                have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, (unsigned long long*)w->d_counts.p, RcCut{});
        CUDA_TRY(cudaGetLastError()); q.launches++;
    }
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    // every rank must bring the same row list to the collective: only the explicit-ids form is all-reduced (fbgpu.h)
    if (reduce && !per_shard) { rc = allreduce_u64(c, w, w->d_counts.p, nr); if (rc) return rc; }
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, n_out * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    memcpy(counts.data(), w->h_out.p, n_out * 8);
    q.add_elapsed();
    q.finish();
    return 0;
}

// The counts of fbgpu_row_counts / fbgpu_row_counts_views / fbgpu_topn_cutoffs once the store is locked, the rows being their
// unions over the view slots fvs.  row_ids != NULL: rows = row_ids, counts[i] theirs, all-reduced.  row_ids == NULL: the rows of
// the listed shards with a non-zero count and their counts, in no particular order, not all-reduced.
static int row_counts_run(fbgpu_ctx* c, uint32_t index, const std::vector<uint32_t>& fvs, const uint64_t* row_ids, int32_t n_rows,
                          const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards,
                          std::vector<uint64_t>& rows, std::vector<uint64_t>& counts, const RcCut* cut = nullptr) {
    rows.clear();
    if (row_ids) rows.assign(row_ids, row_ids + n_rows);
    else {
        // fragment.rows() (fragment.go:2465-2486): distinct row ids present in the listed shards (of any of the views)
        for (uint32_t fv : fvs) if (fv != kNoView) for (int64_t s = 0; s < n_shards; s++) {
            const auto& sm = c->shardmaps[fv];
            if (shards[s] >= sm.size() || sm[shards[s]] < 0) continue;
            const HostFrag& f = c->frags[sm[shards[s]]];
            for (uint32_t k = 0; k < f.n_rows; k++) rows.push_back(c->h_rows[f.row_off + k].row);
        }
        std::sort(rows.begin(), rows.end()); rows.erase(std::unique(rows.begin(), rows.end()), rows.end());
    }
    int rc = row_counts_impl(c, index, fvs, rows, filter, n_filter_ops, shards, n_shards, counts, row_ids != nullptr, false, cut); if (rc) return rc;
    if (!row_ids) {
        size_t k = 0;
        for (size_t i = 0; i < rows.size(); i++) if (counts[i]) { rows[k] = rows[i]; counts[k++] = counts[i]; }
        rows.resize(k); counts.resize(k);
    }
    return 0;
}

// the all-rows form's output: every (row, count) sorted by (count desc, row id asc), or none
static int write_sorted_rows(const std::vector<uint64_t>& rows, const std::vector<uint64_t>& counts, uint64_t* out_row_ids, uint64_t* out_counts, int32_t cap, int32_t* out_n) {
    std::vector<size_t> order(rows.size());
    for (size_t i = 0; i < rows.size(); i++) order[i] = i;
    std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return counts[a] != counts[b] ? counts[a] > counts[b] : rows[a] < rows[b]; });
    // all rows with a non-zero count, or none: a silently truncated list would make Rows() / the TopN candidate set incomplete
    // (ADVICE r1).  *out_n always receives the number of rows there are, so the caller can size its buffers and call again.
    if (out_n) *out_n = (int32_t)std::min<size_t>(order.size(), (size_t)INT32_MAX);
    if (order.size() > (size_t)std::max(cap, 0)) return fail(FBGPU_E_NOSPACE, "%zu rows have a non-zero count, cap is %d", order.size(), cap);
    for (size_t i = 0; i < order.size(); i++) { if (out_row_ids) out_row_ids[i] = rows[order[i]]; out_counts[i] = counts[order[i]]; }
    return FBGPU_OK;
}

// fbgpu_row_counts / fbgpu_row_counts_views / fbgpu_topn_cutoffs once the store is locked: row_counts_run, then the output form
static int row_counts_query(fbgpu_ctx* c, uint32_t index, const std::vector<uint32_t>& fvs, const uint64_t* row_ids, int32_t n_rows,
                            const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards,
                            uint64_t* out_row_ids, uint64_t* out_counts, int32_t cap, int32_t* out_n, const RcCut* cut = nullptr) {
    std::vector<uint64_t> rows, counts;
    int rc = row_counts_run(c, index, fvs, row_ids, n_rows, filter, n_filter_ops, shards, n_shards, rows, counts, cut); if (rc) return rc;
    if (row_ids) {
        if (cap < n_rows) return fail(FBGPU_E_NOSPACE, "cap %d < n_rows %d", cap, n_rows);
        for (int32_t i = 0; i < n_rows; i++) { out_counts[i] = counts[i]; if (out_row_ids) out_row_ids[i] = rows[i]; }
        if (out_n) *out_n = n_rows;
        return FBGPU_OK;
    }
    return write_sorted_rows(rows, counts, out_row_ids, out_counts, cap, out_n);
}

extern "C" int fbgpu_row_counts(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, const uint64_t* row_ids, int32_t n_rows,
                                const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards,
                                uint64_t* out_row_ids, uint64_t* out_counts, int32_t cap, int32_t* out_n) try {
    if (!c || !out_counts || n_shards < 0 || (n_shards && !shards) || n_rows < 0) return fail(FBGPU_E_INVALID, "null argument");
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    const std::vector<uint32_t> fvs{ view_id_locked(c, ViewKey{ index, field, view }, false) };
    return row_counts_query(c, index, fvs, row_ids, n_rows, filter, n_filter_ops, shards, n_shards, out_row_ids, out_counts, cap, out_n);
} FBGPU_CATCH

// the argument checks fbgpu_row_counts_views and its node form make before any device is touched
static int row_counts_views_args(const void* handle, const uint32_t* views, int32_t n_views, int32_t n_rows, const fbgpu_op* filter, int32_t n_filter_ops,
                                 const uint64_t* shards, int64_t n_shards, const uint64_t* out_counts) {
    if (!handle || !views || !out_counts || n_rows < 0 || n_filter_ops < 0 || (n_filter_ops && !filter) || n_shards < 0 || (n_shards && !shards))
        return fail(FBGPU_E_INVALID, "bad argument");
    if (n_views < 1) return fail(FBGPU_E_INVALID, "n_views=%d < 1", n_views);
    return 0;
}

// the view slots of (index, field, views[i]) that exist, each once: a view never loaded, or listed twice, adds nothing to a
// union.  {kNoView} when none exists, so that every row counts 0.
static std::vector<uint32_t> view_slots(fbgpu_ctx* c, uint32_t index, uint32_t field, const uint32_t* views, int32_t n_views) {
    std::vector<uint32_t> fvs;
    for (int32_t i = 0; i < n_views; i++) { const uint32_t fv = view_id_locked(c, ViewKey{ index, field, views[i] }, false); if (fv != kNoView) fvs.push_back(fv); }
    std::sort(fvs.begin(), fvs.end()); fvs.erase(std::unique(fvs.begin(), fvs.end()), fvs.end());
    if (fvs.empty()) fvs.push_back(kNoView);
    return fvs;
}

// TopK / Rows of a time field with from= / to=: fbgpu_row_counts with each row taken as its union over the covering views.
// executeTopKShardTime (executor.go:2506-2533) counts a row over the mergerator of the views' fragments (:2570), and
// executeRowsShard (:4107-4127) merges the row ids of every covering view; both in one pass over the shards here.
extern "C" int fbgpu_row_counts_views(fbgpu_ctx* c, uint32_t index, uint32_t field, const uint32_t* views, int32_t n_views,
                                      const uint64_t* row_ids, int32_t n_rows, const fbgpu_op* filter, int32_t n_filter_ops,
                                      const uint64_t* shards, int64_t n_shards, uint64_t* out_row_ids, uint64_t* out_counts, int32_t cap, int32_t* out_n) try {
    int rc = row_counts_views_args(c, views, n_views, n_rows, filter, n_filter_ops, shards, n_shards, out_counts); if (rc) return rc;
    if (n_views == 1) return fbgpu_row_counts(c, index, field, views[0], row_ids, n_rows, filter, n_filter_ops, shards, n_shards, out_row_ids, out_counts, cap, out_n);
    std::shared_lock<std::shared_mutex> lk;
    rc = begin_query(c, lk); if (rc) return rc;
    return row_counts_query(c, index, view_slots(c, index, field, views, n_views), row_ids, n_rows, filter, n_filter_ops, shards, n_shards,
                            out_row_ids, out_counts, cap, out_n);
} FBGPU_CATCH

// per-shard counts of explicit rows: out_counts[s * n_rows + i] = |Row(row_ids[i]) [∩ filter]| in shards[s]
extern "C" int fbgpu_row_counts_per_shard(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, const uint64_t* row_ids, int32_t n_rows,
                                          const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    if (!c || !out_counts || !row_ids || n_rows < 0 || n_shards < 0 || (n_shards && !shards) || n_filter_ops < 0 || (n_filter_ops && !filter)) return fail(FBGPU_E_INVALID, "null argument");
    if (n_rows == 0 || n_shards == 0) return FBGPU_OK;
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    const std::vector<uint32_t> fv{ view_id_locked(c, ViewKey{ index, field, view }, false) };
    std::vector<uint64_t> rows(row_ids, row_ids + n_rows), counts;
    // the matrix is produced in blocks of shards so that the device / pinned buffers stay below 512 MiB however many rows are asked for
    const int64_t block = std::max<int64_t>(1, (int64_t)((64ull << 20) / (uint64_t)n_rows));
    for (int64_t s0 = 0; s0 < n_shards; s0 += block) {
        const int64_t ns = std::min(block, n_shards - s0);
        rc = row_counts_impl(c, index, fv, rows, filter, n_filter_ops, shards + s0, ns, counts, false, true); if (rc) return rc;
        memcpy(out_counts + (size_t)s0 * n_rows, counts.data(), counts.size() * 8);
    }
    return FBGPU_OK;
} FBGPU_CATCH

// the argument checks fbgpu_topn_cutoffs and its node form make before any device is touched
static int topn_cutoffs_args(const void* handle, int32_t n_rows, const fbgpu_op* src, int32_t n_src_ops, uint32_t tanimoto_threshold,
                             const uint64_t* shards, int64_t n_shards, const uint64_t* out_counts) {
    if (!handle || !out_counts || n_rows < 0 || n_src_ops < 0 || (n_src_ops && !src) || n_shards < 0 || (n_shards && !shards))
        return fail(FBGPU_E_INVALID, "bad argument");
    if (tanimoto_threshold > 100) return fail(FBGPU_E_INVALID, "tanimoto_threshold=%u > 100", tanimoto_threshold);
    return 0;
}

// TopN(f, Src, threshold= / tanimotoThreshold=): fragment.top's per-shard cut-offs (fragment.go:1329-1388) and the sum over the
// shards of what passes (executeTopNShards executor.go:2831-2866), in one pass over the shards
extern "C" int fbgpu_topn_cutoffs(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, const uint64_t* row_ids, int32_t n_rows,
                                  const fbgpu_op* src, int32_t n_src_ops, uint64_t min_threshold, uint32_t tanimoto_threshold,
                                  const uint64_t* shards, int64_t n_shards, uint64_t* out_row_ids, uint64_t* out_counts, int32_t cap, int32_t* out_n) try {
    int rc = topn_cutoffs_args(c, n_rows, src, n_src_ops, tanimoto_threshold, shards, n_shards, out_counts); if (rc) return rc;
    std::shared_lock<std::shared_mutex> lk;
    rc = begin_query(c, lk); if (rc) return rc;
    const std::vector<uint32_t> fvs{ view_id_locked(c, ViewKey{ index, field, view }, false) };
    const RcCut cut{ nullptr, min_threshold, tanimoto_threshold };
    return row_counts_query(c, index, fvs, row_ids, n_rows, src, n_src_ops, shards, n_shards, out_row_ids, out_counts, cap, out_n, &cut);
} FBGPU_CATCH

// ------------------------------------------------------------------ many fused Intersect+Count pairs in one launch
extern "C" int fbgpu_count_pairs(fbgpu_ctx* c, uint32_t index, uint32_t field_a, uint32_t view_a, const uint64_t* rows_a,
                                 uint32_t field_b, uint32_t view_b, const uint64_t* rows_b, int32_t n_pairs,
                                 const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    if (!c || !rows_a || !rows_b || !out_counts || n_pairs < 0 || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    USE_DEVICE(c);
    if (n_pairs == 0) return FBGPU_OK;
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    uint32_t fa = view_id_locked(c, ViewKey{ index, field_a, view_a }, false), fb = view_id_locked(c, ViewKey{ index, field_b, view_b }, false);
    Query q(c); Workspace* w = q.w;
    rc = q.open(shards, n_shards); if (rc) return rc;
    size_t np = (size_t)n_pairs;
    if (w->d_rows.ensure(np * 16) || w->d_counts.ensure(np * 8) || w->h_out.ensure(np * 16)) return FBGPU_E_NOMEM;
    memcpy(w->h_out.p, rows_a, np * 8); memcpy((uint8_t*)w->h_out.p + np * 8, rows_b, np * 8);
    CUDA_TRY(cudaMemcpyAsync(w->d_rows.p, w->h_out.p, np * 16, cudaMemcpyHostToDevice, w->stream));
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, np * 8, w->stream));
    const long long upp = q.n_units, n_units = upp * n_pairs;
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    if (n_units > 0) {
        long long grid = std::min<long long>((n_units + kPcWarps - 1) / kPcWarps, (long long)c->sm_count * c->pair_ctas_per_sm);
        const PairShards ps = pair_shards(shards, n_shards, q.d_shards);
        pair_count_kernel<<<(unsigned)grid, kPcWarps * 32, kPcWarps * 8192, w->stream>>>(store_ref(c), fa, 0, fb, 0, (const uint64_t*)w->d_rows.p, (const uint64_t*)w->d_rows.p + np,
            upp, ps.list, ps.first, n_units, nullptr, nullptr, (unsigned long long*)w->d_counts.p, FuseReduce{});
        CUDA_TRY(cudaGetLastError()); q.launches++;
    }
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    rc = allreduce_u64(c, w, w->d_counts.p, np); if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(w->stream));      // h_out was the H2D source; now reuse it as the D2H landing buffer
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, np * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    memcpy(out_counts, w->h_out.p, np * 8);
    q.add_elapsed();
    q.finish();
    return FBGPU_OK;
} FBGPU_CATCH

// container-pair-type histogram of Count(Intersect(Row a, Row b)) (statsHit analogue, roaring.go:4477-4614)
extern "C" int fbgpu_pair_types(fbgpu_ctx* c, uint32_t index, uint32_t field_a, uint32_t view_a, uint64_t row_a, uint32_t field_b, uint32_t view_b, uint64_t row_b,
                                const uint64_t* shards, int64_t n_shards, uint64_t out_hist[16]) try {
    if (!c || !out_hist || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    USE_DEVICE(c);
    memset(out_hist, 0, 16 * 8);
    if (n_shards == 0) return FBGPU_OK;
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    const uint32_t fa = view_id_locked(c, ViewKey{ index, field_a, view_a }, false), fb = view_id_locked(c, ViewKey{ index, field_b, view_b }, false);
    Query q(c); Workspace* w = q.w;
    rc = q.open(shards, n_shards); if (rc) return rc;
    if (w->d_counts.ensure(16 * 8) || w->h_out.ensure(16 * 8)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, 16 * 8, w->stream));
    const long long grid = std::min<long long>((q.n_units + 255) / 256, (long long)c->sm_count * 4);
    pair_types_kernel<<<(unsigned)grid, 256, 0, w->stream>>>(store_ref(c), fa, row_a, fb, row_b, q.d_shards, q.n_units, (unsigned long long*)w->d_counts.p);
    CUDA_TRY(cudaGetLastError()); q.launches++;
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, 16 * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    memcpy(out_hist, w->h_out.p, 16 * 8);
    q.finish();                              // (untimed: last_query_gpu_ms reads 0)
    return FBGPU_OK;
} FBGPU_CATCH

// Row.Any() of a bitmap call (row.go:258; the early exit of intersectionAny, roaring.go:4266-4408, lifted to shard granularity):
// the shards are evaluated in blocks of growing size and the walk stops at the first block whose count is not zero, so a row that
// has any column in its first shards costs one small launch instead of a pass over every shard.
extern "C" int fbgpu_any(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards, int32_t* out_any) try {
    if (!c || !out_any || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    *out_any = 0;
    uint64_t cnt = 0;
    if (n_shards == 0) return fbgpu_count(c, index, ops, n_ops, shards, 0, &cnt, nullptr);      // (still validates the program)
    int64_t block = 8;
    for (int64_t s0 = 0; s0 < n_shards; s0 += block, block *= 8) {
        const int64_t ns = std::min(block, n_shards - s0);
        int rc = fbgpu_count_local(c, index, ops, n_ops, shards + s0, ns, &cnt); if (rc) return rc;
        if (cnt) { *out_any = 1; return FBGPU_OK; }
    }
    return FBGPU_OK;
} FBGPU_CATCH

// ------------------------------------------------------------------ GroupBy
// Largest average number of field-a columns per (shard, slot) that groupby_direct_kernel is given: the size its predecessor, a
// hash table per group of slots, was built for.  Whether the direct kernel is also the faster one above it has not been measured.
constexpr uint64_t kGdMaxSlotCols = 8192;

// groupby_direct_kernel's shape: both fields array-dominated, and field a holding at most kGdMaxSlotCols columns per slot on
// average, from the cardinality of a sample of the listed shards' fragments.
static bool groupby_direct_eligible(fbgpu_ctx* c, uint32_t fvA, uint32_t fvB, const uint64_t* shards, int64_t n) {
    if (fvA >= c->shardmaps.size() || fvB >= c->shardmaps.size() || n <= 0) return false;
    if (c->view_other[fvA] * 8 > c->view_arr[fvA] || c->view_other[fvB] * 8 > c->view_arr[fvB]) return false;     // bitmap / run heavy: groupby_kernel
    const auto& sm = c->shardmaps[fvA];
    uint64_t elems = 0, seen = 0;
    const int64_t step = std::max<int64_t>(1, n / 64);
    for (int64_t i = 0; i < n; i += step) {
        const uint64_t sh = shards[i];
        if (sh >= sm.size() || sm[sh] < 0) continue;
        elems += c->frags[(size_t)sm[sh]].payload_bytes / 2; seen++;
    }
    if (!seen) return true;
    const uint64_t avg = elems / seen;                       // columns of field a per shard (all its rows: an upper bound for a row subset)
    return avg / kSlotsPerRow <= kGdMaxSlotCols;
}

static int groupby2(fbgpu_ctx* c, uint32_t index, uint32_t fvA, const uint64_t* rowsA, int nA, uint32_t fvB, const uint64_t* rowsB, int nB,
                    const std::vector<fbgpu_op>& filter, const uint64_t* shards, int64_t n_shards, uint64_t* out) {
    const bool have_filter = !filter.empty();
    Query q(c); Workspace* w = q.w;
    int rc = have_filter ? q.open(index, filter.data(), (int)filter.size(), shards, n_shards) : q.open(shards, n_shards); if (rc) return rc;
    const uint64_t* d_shards = q.d_shards;
    size_t ncnt = (size_t)nA * nB;
    if (w->d_rows.ensure((size_t)(nA + nB) * 8) || w->d_counts.ensure(ncnt * 8) || w->h_out.ensure(ncnt * 8)) return FBGPU_E_NOMEM;
    std::vector<uint64_t> rr(rowsA, rowsA + nA); rr.insert(rr.end(), rowsB, rowsB + nB);
    CUDA_TRY(cudaMemcpyAsync(w->d_rows.p, rr.data(), rr.size() * 8, cudaMemcpyHostToDevice, w->stream));
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, ncnt * 8, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));   // rr is a local
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    uint64_t fb_units = 0, all_units = 0;
    const int64_t batch = have_filter ? c->unit_batch / kSlotsPerRow : n_shards;
    const size_t smem = kGbSlots * 4 + 8192;
    for (int64_t s0 = 0; s0 < n_shards; s0 += batch) {
        int64_t ns = std::min(batch, n_shards - s0);
        if (have_filter) { rc = q.eval(s0 * kSlotsPerRow, ns * kSlotsPerRow); if (rc) return rc; }
        long long units = (long long)ns * kSlotsPerRow;
        long long grid = std::min<long long>(units, (long long)c->sm_count * 4);
        static const bool gb_cta_only = getenv("FBGPU_GROUPBY_CTA") != nullptr; // round-1 path only: one CTA per unit
        if (!gb_cta_only && units < (1ll << 31) && groupby_direct_eligible(c, fvA, fvB, shards + s0, ns)) {
            // array-dominated fields: groupby_direct_kernel, one CTA per (shard, slot), 256 a-rows per launch; what it declines is listed
            // for groupby_kernel, launched only when the list is not empty (its launch alone costs tens of microseconds next to a kernel
            // with another shared-memory carve-out) — the 4-byte count is read back first
            if (w->d_emit_units.ensure((size_t)(units + 1) * 4)) return FBGPU_E_NOMEM;
            unsigned int* d_fb = (unsigned int*)w->d_emit_units.p;
            unsigned int* h_fb = (unsigned int*)w->h_in.p;          // (pinned; upload_inputs sized it, its content is in flight no longer: the stream was synchronised above)
            const long long dgrid = std::min<long long>(units, (long long)c->sm_count * c->gd_ctas_per_sm);
            for (int a0 = 0; a0 < nA; a0 += kGdThreads) {
                const int na = std::min(kGdThreads, nA - a0);
                const uint64_t* d_ra = (const uint64_t*)w->d_rows.p + a0;
                unsigned long long* d_cnt = (unsigned long long*)w->d_counts.p + (size_t)a0 * nB;
                CUDA_TRY(cudaMemsetAsync(d_fb, 0, 4, w->stream));
                groupby_direct_kernel<<<(unsigned)dgrid, kGdThreads, kGdSmemBytes, w->stream>>>(store_ref(c), fvA, d_ra, na, fvB, (const uint64_t*)w->d_rows.p + nA, nB,
                    d_shards + s0, units, have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, d_cnt, d_fb);
                CUDA_TRY(cudaGetLastError()); q.launches++;
                CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
                CUDA_TRY(cudaMemcpyAsync(h_fb, d_fb, 4, cudaMemcpyDeviceToHost, w->stream));
                CUDA_TRY(cudaStreamSynchronize(w->stream));
                const unsigned int n_fb = *h_fb;
                if (n_fb) {
                    groupby_kernel<<<(unsigned)std::min<long long>(n_fb, grid), kGbThreads, smem, w->stream>>>(store_ref(c), fvA, d_ra, na, fvB, (const uint64_t*)w->d_rows.p + nA, nB,
                        d_shards + s0, units, have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, d_cnt, d_fb);
                    CUDA_TRY(cudaGetLastError()); q.launches++;
                    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
                }
                fb_units += n_fb; all_units += (uint64_t)units;
            }
        } else {
            groupby_kernel<<<(unsigned)grid, kGbThreads, smem, w->stream>>>(store_ref(c), fvA, (const uint64_t*)w->d_rows.p, nA, fvB, (const uint64_t*)w->d_rows.p + nA, nB,
                d_shards + s0, units, have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, (unsigned long long*)w->d_counts.p, nullptr);
            CUDA_TRY(cudaGetLastError()); q.launches++;
            CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
        }
    }
    if (n_shards <= 0) CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    rc = allreduce_u64(c, w, w->d_counts.p, ncnt); if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, ncnt * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    memcpy(out, w->h_out.p, ncnt * 8);
    q.add_elapsed();
    { std::lock_guard<std::mutex> lk2(c->cnt_mu); c->counters.groupby_units += all_units; c->counters.groupby_fallback_units += fb_units; }
    q.finish();
    return 0;
}

// one GroupBy dimension: the listed rows of `field`, each taken as its union over views[0..n_views)
struct GbDim { uint32_t field; const uint32_t* views; int32_t n_views; const uint64_t* rows; int32_t n_rows; };

// the argument checks fbgpu_groupby and its node form make before any device is touched (the context form checks n_rows after it)
static int groupby_args(const void* handle, const uint32_t* fields, const uint32_t* views, int32_t n_fields, const uint64_t* row_ids_flat, const int32_t* n_rows,
                        const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, const uint64_t* out_counts) {
    if (!handle || !fields || !views || !row_ids_flat || !n_rows || !out_counts || n_fields < 1 || n_fields > 8 || n_filter_ops < 0 || (n_filter_ops && !filter) ||
        n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "bad argument");
    return 0;
}

// the argument checks fbgpu_groupby_views and its node form make before any device is touched
static int groupby_views_args(const void* handle, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                              const uint64_t* row_ids_flat, const int32_t* n_rows, const fbgpu_op* filter, int32_t n_filter_ops,
                              const uint64_t* shards, int64_t n_shards, const uint64_t* out_counts) {
    if (!handle || !fields || !views_flat || !n_views || !row_ids_flat || !n_rows || !out_counts || n_filter_ops < 0 || (n_filter_ops && !filter) ||
        n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "bad argument");
    if (n_fields < 1 || n_fields > 8) return fail(FBGPU_E_INVALID, "n_fields=%d outside 1..8", n_fields);
    for (int i = 0; i < n_fields; i++) {
        if (n_views[i] < 1) return fail(FBGPU_E_INVALID, "n_views[%d]=%d < 1", i, n_views[i]);
        if (n_rows[i] < 0 || n_rows[i] > 65535) return fail(FBGPU_E_INVALID, "n_rows[%d]=%d out of range", i, n_rows[i]);
    }
    return 0;
}

// ------------------------------------------------------------------ GroupBy over the values of int fields
// one int dimension of fbgpu_groupby_values / fbgpu_groupby_mixed: field, BSI view, depth and the ascending stored values that are its groups.
// As the aggregate field x: values is null for Sum, and for Count(Distinct) the ascending stored values whose presence is counted;
// for Count(Distinct) over a set-like field, rows holds the n_values ascending row ids whose presence is counted (values null)
struct GvInt { uint32_t field, view; int32_t depth; const int64_t* values; int32_t n_values; const uint64_t* rows = nullptr; };

// the argument checks fbgpu_groupby_values and its node form make before any device is touched
static int groupby_values_args(const void* handle, const uint32_t* fields, const uint32_t* views, int32_t n_fields, const uint64_t* row_ids_flat,
                               const int32_t* n_rows, int32_t bit_depth, const int64_t* values, int32_t n_values, const fbgpu_op* filter,
                               int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, const uint64_t* out_counts) {
    if (!handle || !values || !out_counts || n_fields < 0 || n_fields > 7 || (n_fields && (!fields || !views || !row_ids_flat || !n_rows)) ||
        n_filter_ops < 0 || (n_filter_ops && !filter) || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "bad argument");
    if (bit_depth < 0 || bit_depth > 64) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..64", bit_depth);
    if (n_values < 1 || n_values > 65535) return fail(FBGPU_E_INVALID, "n_values=%d outside 1..65535", n_values);
    for (int32_t i = 1; i < n_values; i++)
        if (values[i] <= values[i - 1]) return fail(FBGPU_E_INVALID, "values are not strictly ascending at position %d", i);
    return 0;
}

// the argument checks fbgpu_groupby_mixed and its node form make before any device is touched (n_rows is checked after it);
// fbgpu_groupby_sum's dimensions are the same but for the bounds: 0..8 set and 0..8 int dimensions, the int arrays may then be NULL
static int groupby_mixed_args(const void* handle, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                              const uint64_t* row_ids_flat, const int32_t* n_rows, const uint32_t* vfields, const uint32_t* vviews,
                              const int32_t* bit_depths, int32_t n_ints, const int64_t* values_flat, const int32_t* n_values,
                              const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, const uint64_t* out_counts,
                              int32_t min_ints = 1, int32_t max_fields = 7) {
    if (!handle || ((min_ints || n_ints) && (!vfields || !vviews || !bit_depths || !values_flat || !n_values)) || !out_counts ||
        (n_fields > 0 && (!fields || !views_flat || !n_views || !row_ids_flat || !n_rows)) ||
        n_filter_ops < 0 || (n_filter_ops && !filter) || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "bad argument");
    if (n_fields < 0 || n_fields > max_fields) return fail(FBGPU_E_INVALID, "n_fields=%d outside 0..%d", n_fields, max_fields);
    if (n_ints < min_ints || n_ints > kGvMaxInts) return fail(FBGPU_E_INVALID, "n_ints=%d outside %d..%d", n_ints, min_ints, kGvMaxInts);
    if (n_fields + n_ints > 8) return fail(FBGPU_E_INVALID, "n_fields + n_ints = %d exceeds 8", n_fields + n_ints);
    for (int32_t i = 0; i < n_fields; i++)
        if (n_views[i] < 1) return fail(FBGPU_E_INVALID, "n_views[%d]=%d < 1", i, n_views[i]);
    const int64_t* vals = values_flat;
    double groups = 1;
    for (int32_t k = 0; k < n_ints; k++) {
        if (bit_depths[k] < 0 || bit_depths[k] > 64) return fail(FBGPU_E_INVALID, "bit_depths[%d]=%d outside 0..64", k, bit_depths[k]);
        if (n_values[k] < 1 || n_values[k] > 65535) return fail(FBGPU_E_INVALID, "n_values[%d]=%d outside 1..65535", k, n_values[k]);
        for (int32_t i = 1; i < n_values[k]; i++)
            if (vals[i] <= vals[i - 1]) return fail(FBGPU_E_INVALID, "values[%d] are not strictly ascending at position %d", k, i);
        vals += n_values[k];
        groups *= n_values[k];
    }
    if (groups > 65535) return fail(FBGPU_E_INVALID, "product of n_values %.0f exceeds 65535", groups);
    return 0;
}

// the argument checks fbgpu_groupby_sum, fbgpu_groupby_distinct and fbgpu_groupby_distinct_rows (and the node form of Sum) make
// before any device is touched (n_rows is checked after it): agg_array is out_sums of Sum, x_values / x_rows of Count(Distinct),
// the aggregate field's depth is named depth_name in the message.  Count(Distinct) checks its x list next
static int groupby_agg_args(const void* handle, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                            const uint64_t* row_ids_flat, const int32_t* n_rows, const uint32_t* vfields, const uint32_t* vviews,
                            const int32_t* bit_depths, int32_t n_ints, const int64_t* values_flat, const int32_t* n_values, const void* agg_array,
                            const char* depth_name, int32_t depth, const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards,
                            int64_t n_shards, const uint64_t* out_counts) {
    if (!agg_array) return fail(FBGPU_E_INVALID, "bad argument");
    int rc = groupby_mixed_args(handle, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, vfields, vviews, bit_depths, n_ints, values_flat,
                                n_values, filter, n_filter_ops, shards, n_shards, out_counts, 0, 8);
    if (rc) return rc;
    if (n_fields + n_ints < 1) return fail(FBGPU_E_INVALID, "no dimension: n_fields + n_ints = 0");
    if (depth < 0 || depth > 64) return fail(FBGPU_E_INVALID, "%s=%d outside 0..64", depth_name, depth);
    return 0;
}

// one groupby_values_kernel pass over the shards: counts[nB or 1][groups] of consider = filter ∩ exists(v_1) ∩ ... (∩ Row(b = row));
// with an aggregate x, consider also ∩ exists(x) and sums[nB or 1][groups] the columns' stored values of x (Sum), or out[nB or 1]
// [groups] the number of x's listed values present in the cell (Count(Distinct): x->values set, out_sums null), or with x->rows
// set the number of x's listed rows that hold a column of the cell (consider without exists(x)).  The presence bitset stays on
// the device; only the per-cell counts come back
static int groupby_values_leaf(fbgpu_ctx* c, uint32_t index, const GbDim* b /* null: no set dimension */, const std::vector<GvInt>& v,
                               const GvInt* x /* null: counts only */, const std::vector<fbgpu_op>& filter, const uint64_t* shards, int64_t n_shards,
                               uint64_t* out, uint64_t* out_sums) {
    std::vector<fbgpu_op> full = filter;
    for (const GvInt& f : v) full = and_row(full.data(), (int32_t)full.size(), f.field, f.view, 0);
    const bool rows_x = x && x->rows;                                 // Count(Distinct) over a set-like x: no exists row
    if (x && !rows_x) full = and_row(full.data(), (int32_t)full.size(), x->field, x->view, 0);
    if (full.empty()) {                                              // (rows_x, b alone, no filter) consider: b's listed rows, which b's walk keeps anyway
        for (int r = 0; r < b->n_rows; r++)
            for (int32_t i = 0; i < b->n_views; i++) { fbgpu_op o{}; o.opcode = FBGPU_OP_ROW; o.field = b->field; o.view = b->views[i]; o.a = b->rows[r]; full.push_back(o); }
        if (full.size() > 1) { fbgpu_op u{}; u.opcode = FBGPU_OP_UNION; u.argc = (uint32_t)full.size(); full.push_back(u); }
    }
    Query q(c); Workspace* w = q.w;
    int rc = q.open(index, full.data(), (int32_t)full.size(), shards, n_shards); if (rc) return rc;
    GvInts k{};
    k.n = (int)v.size(); k.n_groups = 1;
    std::vector<uint64_t> in;                                        // [values (as int64) | x's values | b rows | b view slots (u32)]
    for (int i = 0; i < k.n; i++) {
        k.fv[i] = view_id_locked(c, ViewKey{ index, v[(size_t)i].field, v[(size_t)i].view }, false);
        k.depth[i] = v[(size_t)i].depth; k.off[i] = (int)in.size(); k.n_values[i] = v[(size_t)i].n_values;
        k.n_groups *= v[(size_t)i].n_values;
        in.insert(in.end(), v[(size_t)i].values, v[(size_t)i].values + v[(size_t)i].n_values);
    }
    const bool distinct = x && (x->values || rows_x);
    const size_t x_off = in.size();
    if (rows_x) in.insert(in.end(), x->rows, x->rows + x->n_values);
    else if (distinct) in.insert(in.end(), x->values, x->values + x->n_values);
    const size_t n_vals = in.size();
    const uint32_t fvX = x ? view_id_locked(c, ViewKey{ index, x->field, x->view }, false) : kNoView;
    const int nB = b ? b->n_rows : 0;
    const std::vector<uint32_t> fvsB = b ? view_slots(c, index, b->field, b->views, b->n_views) : std::vector<uint32_t>{ kNoView };
    const size_t nvB = fvsB.size();
    if (b) in.insert(in.end(), b->rows, b->rows + nB);
    const size_t n_in = in.size();
    if (nvB > 1) in.resize(n_in + (nvB + 1) / 2);
    if (nvB > 1) memcpy(in.data() + n_in, fvsB.data(), nvB * 4);
    const size_t ncnt = (size_t)(b ? nB : 1) * (size_t)k.n_groups;
    const size_t nout = x && !distinct ? 2 * ncnt : ncnt;            // [counts | sums], or the distinct counts
    const size_t xwords = distinct ? ((size_t)x->n_values + 63) / 64 : 0;       // presence words per cell
    if (distinct && w->d_present.ensure(ncnt * xwords * 8)) return FBGPU_E_NOMEM;
    if (w->d_rows.ensure(in.size() * 8) || w->d_counts.ensure(nout * 8) || w->h_out.ensure(nout * 8)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemcpyAsync(w->d_rows.p, in.data(), in.size() * 8, cudaMemcpyHostToDevice, w->stream));
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, nout * 8, w->stream));
    if (distinct) CUDA_TRY(cudaMemsetAsync(w->d_present.p, 0, ncnt * xwords * 8, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));   // `in` is a local
    const long long* d_values = (const long long*)w->d_rows.p;
    const uint64_t* d_rowsB = b ? (const uint64_t*)w->d_rows.p + n_vals : nullptr;
    const uint32_t* d_fvsB = nvB > 1 ? (const uint32_t*)((const uint64_t*)w->d_rows.p + n_in) : nullptr;
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    for (long long u0 = 0; u0 < q.n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, q.n_units - u0);
        rc = q.eval(u0, nu); if (rc) return rc;
        const long long grid = std::min<long long>(nu, (long long)c->sm_count * kGvCtasPerSm);
        unsigned long long* d_counts = (unsigned long long*)w->d_counts.p;
        if (rows_x)
            groupby_values_kernel<GvAgg::kDistinctRows><<<(unsigned)grid, kGvThreads, 0, w->stream>>>(
                store_ref(c), k, d_values, d_rowsB, nB, fvsB[0], d_fvsB, (int)nvB, (const uint4*)w->d_bitmaps.p, q.d_shards + u0 / kSlotsPerRow, nu, d_counts,
                fvX, 0, nullptr, d_values + x_off, x->n_values, (unsigned long long*)w->d_present.p);
        else if (distinct)
            groupby_values_kernel<GvAgg::kDistinct><<<(unsigned)grid, kGvThreads, 0, w->stream>>>(
                store_ref(c), k, d_values, d_rowsB, nB, fvsB[0], d_fvsB, (int)nvB, (const uint4*)w->d_bitmaps.p, q.d_shards + u0 / kSlotsPerRow, nu, d_counts,
                fvX, x->depth, nullptr, d_values + x_off, x->n_values, (unsigned long long*)w->d_present.p);
        else if (x)
            groupby_values_kernel<GvAgg::kSum><<<(unsigned)grid, kGvThreads, 0, w->stream>>>(store_ref(c), k, d_values, d_rowsB, nB, fvsB[0], d_fvsB, (int)nvB,
                                                                                           (const uint4*)w->d_bitmaps.p, q.d_shards + u0 / kSlotsPerRow, nu, d_counts,
                                                                                           fvX, x->depth, d_counts + ncnt);
        else
            groupby_values_kernel<GvAgg::kCount><<<(unsigned)grid, kGvThreads, 0, w->stream>>>(store_ref(c), k, d_values, d_rowsB, nB, fvsB[0], d_fvsB, (int)nvB,
                                                                                             (const uint4*)w->d_bitmaps.p, q.d_shards + u0 / kSlotsPerRow, nu, d_counts);
        CUDA_TRY(cudaGetLastError()); q.launches++;
    }
    if (distinct) {                                                  // every batch has marked the bitset: count each cell's bits
        const long long grid = std::min<long long>(((long long)ncnt + 7) / 8, (long long)c->sm_count * 8);
        gv_popcount_kernel<<<(unsigned)grid, 256, 0, w->stream>>>((const unsigned long long*)w->d_present.p, (long long)xwords, (long long)ncnt,
                                                                  (unsigned long long*)w->d_counts.p);
        CUDA_TRY(cudaGetLastError()); q.launches++;
    }
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    rc = allreduce_u64(c, w, w->d_counts.p, nout); if (rc) return rc;           // a wrapping int64 sum is a u64 sum
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, nout * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    memcpy(out, w->h_out.p, ncnt * 8);
    if (x && !distinct) memcpy(out_sums, (const uint64_t*)w->h_out.p + ncnt, ncnt * 8);
    q.add_elapsed();
    q.finish();
    return 0;
}

// ------------------------------------------------------------------ one GroupBy request: every GroupBy entry point
// The tensor's axes are the set dimensions, then the int dimensions.  Per cell: the number of columns of filter ∩ the cell's rows
// (∩ exists(x) with an aggregate), and with agg kSum the sum of x's stored values behind it, or with kDistinct, in place of the
// count, how many of x.values the cell holds, or with kDistinctRows how many of the rows x.rows hold a column of the cell
struct GbRequest {
    std::vector<GbDim> dims;
    std::vector<GvInt> ints;
    GvAgg agg; GvInt x;                                             // (x unused for kCount)
    const fbgpu_op* filter; int32_t n_filter_ops;
    const uint64_t* shards; int64_t n_shards;
    int check_rows() const {
        for (size_t i = 0; i < dims.size(); i++)
            if (dims[i].n_rows < 0 || dims[i].n_rows > 65535) return fail(FBGPU_E_INVALID, "n_rows[%d]=%d out of range", (int)i, dims[i].n_rows);
        return 0;
    }
    size_t cells() const {
        size_t n = 1;
        for (const GbDim& d : dims) n *= (size_t)d.n_rows;
        for (const GvInt& v : ints) n *= (size_t)v.n_values;
        return n;
    }
    size_t out_len() const { return agg == GvAgg::kSum ? 2 * cells() : cells(); }     // Sum: [counts | sums]
};

// the set dimensions of the ABI's flat arrays: dimension i has n_views[i] views (one when n_views is null) and n_rows[i] rows
static std::vector<GbDim> gb_set_dims(const uint32_t* fields, const uint32_t* views, const int32_t* n_views, int32_t n_fields,
                                      const uint64_t* row_ids_flat, const int32_t* n_rows) {
    std::vector<GbDim> dims((size_t)n_fields);
    for (int i = 0; i < n_fields; i++) {
        const int32_t nv = n_views ? n_views[i] : 1;
        dims[(size_t)i] = GbDim{ fields[i], views, nv, row_ids_flat, n_rows[i] };
        views += nv; row_ids_flat += n_rows[i];
    }
    return dims;
}

// the int dimensions of the ABI's flat arrays: dimension k has n_values[k] values
static std::vector<GvInt> gb_int_dims(const uint32_t* vfields, const uint32_t* vviews, const int32_t* bit_depths, int32_t n_ints,
                                      const int64_t* values_flat, const int32_t* n_values) {
    std::vector<GvInt> ints((size_t)n_ints);
    for (int k = 0; k < n_ints; k++) { ints[(size_t)k] = GvInt{ vfields[k], vviews[k], bit_depths[k], values_flat, n_values[k] }; values_flat += n_values[k]; }
    return ints;
}

// Peel the leading set dimension on the host, folding Row(f0=r) — over several views, the union of those rows — into the filter
// (groupByIterator keeps the same prefix intersections per level, executor.go:8829-8835,8861-8867), down to a leaf.  Counts over
// set dimensions alone: the last dimension by the row-count kernels, two single-view last dimensions by groupby2.  Otherwise one
// groupby_values_leaf pass once at most one set dimension (the kernel's b) is left
static int groupby_rec(fbgpu_ctx* c, uint32_t index, const GbRequest& q, const GbDim* d, int nf, const std::vector<fbgpu_op>& filter,
                       uint64_t* out, uint64_t* out_sums) {
    if (q.ints.empty() && q.agg == GvAgg::kCount) {
        if (nf == 1) {
            std::vector<uint64_t> r(d[0].rows, d[0].rows + d[0].n_rows), counts;
            int rc = row_counts_impl(c, index, view_slots(c, index, d[0].field, d[0].views, d[0].n_views), r, filter.empty() ? nullptr : filter.data(), (int)filter.size(),
                                     q.shards, q.n_shards, counts); if (rc) return rc;
            memcpy(out, counts.data(), counts.size() * 8);
            return 0;
        }
        if (nf == 2 && d[0].n_views == 1 && d[1].n_views == 1) {
            uint32_t fa = view_id_locked(c, ViewKey{ index, d[0].field, d[0].views[0] }, false), fb = view_id_locked(c, ViewKey{ index, d[1].field, d[1].views[0] }, false);
            return groupby2(c, index, fa, d[0].rows, d[0].n_rows, fb, d[1].rows, d[1].n_rows, filter, q.shards, q.n_shards, out);
        }
    } else if (nf <= 1) {
        return groupby_values_leaf(c, index, nf ? d : nullptr, q.ints, q.agg == GvAgg::kCount ? nullptr : &q.x, filter, q.shards, q.n_shards, out, out_sums);
    }
    size_t sub = 1; for (const GvInt& f : q.ints) sub *= (size_t)f.n_values;
    for (int i = 1; i < nf; i++) sub *= (size_t)d[i].n_rows;
    for (int r = 0; r < d[0].n_rows; r++) {
        int rc = groupby_rec(c, index, q, d + 1, nf - 1, and_row(filter.data(), (int32_t)filter.size(), d[0].field, d[0].views, d[0].n_views, d[0].rows[r]),
                             out + (size_t)r * sub, out_sums ? out_sums + (size_t)r * sub : nullptr); if (rc) return rc;
    }
    return 0;
}

// a GroupBy entry point once its arguments but n_rows are checked: the store locked, the outputs zeroed, the peel.  (Its own
// catch serves the node forms, which run it on their worker threads.)
static int groupby_run(fbgpu_ctx* c, uint32_t index, const GbRequest& q, uint64_t* out_counts, int64_t* out_sums = nullptr) try {
    std::shared_lock<std::shared_mutex> lk;
    int rc = begin_query(c, lk); if (rc) return rc;
    rc = q.check_rows(); if (rc) return rc;
    const size_t cells = q.cells();
    memset(out_counts, 0, cells * 8);
    if (out_sums) memset(out_sums, 0, cells * 8);
    if (cells == 0) return 0;
    // executor.go:8769-8772: the kernels treat a shard with a missing fragment as contributing nothing; for the row_counts
    // leaf a missing fragment naturally yields zeros.  Peeled dimensions enter through the filter, which is empty on shards
    // without that fragment.
    return groupby_rec(c, index, q, q.dims.data(), (int)q.dims.size(), std::vector<fbgpu_op>(q.filter, q.filter + q.n_filter_ops), out_counts, (uint64_t*)out_sums);
} FBGPU_CATCH

extern "C" int fbgpu_groupby(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views, int32_t n_fields, const uint64_t* row_ids_flat, const int32_t* n_rows,
                             const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    int rc = groupby_args(c, fields, views, n_fields, row_ids_flat, n_rows, filter, n_filter_ops, shards, n_shards, out_counts);
    if (rc) return rc;
    return groupby_run(c, index, GbRequest{ gb_set_dims(fields, views, nullptr, n_fields, row_ids_flat, n_rows), {}, GvAgg::kCount, {},
                                            filter, n_filter_ops, shards, n_shards }, out_counts);
} FBGPU_CATCH

// GroupBy(Rows(f1, from=, to=), ...): fbgpu_groupby with dimension i's rows taken as their unions over n_views[i] views
// (timeFragmentsRowIterator, executor.go:8755-8768)
extern "C" int fbgpu_groupby_views(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                   const uint64_t* row_ids_flat, const int32_t* n_rows, const fbgpu_op* filter, int32_t n_filter_ops,
                                   const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    int rc = groupby_views_args(c, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, filter, n_filter_ops, shards, n_shards, out_counts);
    if (rc) return rc;
    return groupby_run(c, index, GbRequest{ gb_set_dims(fields, views_flat, n_views, n_fields, row_ids_flat, n_rows), {}, GvAgg::kCount, {},
                                            filter, n_filter_ops, shards, n_shards }, out_counts);
} FBGPU_CATCH

extern "C" int fbgpu_groupby_values(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views, int32_t n_fields, const uint64_t* row_ids_flat,
                                    const int32_t* n_rows, uint32_t vfield, uint32_t vview, int32_t bit_depth, const int64_t* values, int32_t n_values,
                                    const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    int rc = groupby_values_args(c, fields, views, n_fields, row_ids_flat, n_rows, bit_depth, values, n_values, filter, n_filter_ops, shards, n_shards, out_counts);
    if (rc) return rc;
    return groupby_run(c, index, GbRequest{ gb_set_dims(fields, views, nullptr, n_fields, row_ids_flat, n_rows), gb_int_dims(&vfield, &vview, &bit_depth, 1, values, &n_values),
                                            GvAgg::kCount, {}, filter, n_filter_ops, shards, n_shards }, out_counts);
} FBGPU_CATCH

// GroupBy(Rows(f1), ..., Rows(v1), Rows(v2), ...) with set dimensions (each row a union over views, as fbgpu_groupby_views) and
// one or more int dimensions: fbgpu_groupby_values generalised; with one int field and single views it is that call
extern "C" int fbgpu_groupby_mixed(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                   const uint64_t* row_ids_flat, const int32_t* n_rows, const uint32_t* vfields, const uint32_t* vviews, const int32_t* bit_depths,
                                   int32_t n_ints, const int64_t* values_flat, const int32_t* n_values, const fbgpu_op* filter, int32_t n_filter_ops,
                                   const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    int rc = groupby_mixed_args(c, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, vfields, vviews, bit_depths, n_ints, values_flat, n_values,
                                filter, n_filter_ops, shards, n_shards, out_counts);
    if (rc) return rc;
    return groupby_run(c, index, GbRequest{ gb_set_dims(fields, views_flat, n_views, n_fields, row_ids_flat, n_rows),
                                            gb_int_dims(vfields, vviews, bit_depths, n_ints, values_flat, n_values), GvAgg::kCount, {},
                                            filter, n_filter_ops, shards, n_shards }, out_counts);
} FBGPU_CATCH

// GroupBy(..., aggregate=Sum(field=x)): fbgpu_groupby_mixed's dimensions (none of them int is fine) with, per cell, the number of
// columns holding a value of x and the sum of their stored values: fbgpu_bsi_sum under filter ∩ the cell's rows, for every cell
extern "C" int fbgpu_groupby_sum(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                 const uint64_t* row_ids_flat, const int32_t* n_rows, const uint32_t* vfields, const uint32_t* vviews, const int32_t* bit_depths,
                                 int32_t n_ints, const int64_t* values_flat, const int32_t* n_values, uint32_t afield, uint32_t aview, int32_t a_depth,
                                 const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts, int64_t* out_sums) try {
    int rc = groupby_agg_args(c, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, vfields, vviews, bit_depths, n_ints, values_flat, n_values,
                              out_sums, "a_depth", a_depth, filter, n_filter_ops, shards, n_shards, out_counts);
    if (rc) return rc;
    return groupby_run(c, index, GbRequest{ gb_set_dims(fields, views_flat, n_views, n_fields, row_ids_flat, n_rows),
                                            gb_int_dims(vfields, vviews, bit_depths, n_ints, values_flat, n_values), GvAgg::kSum, GvInt{ afield, aview, a_depth, nullptr, 0 },
                                            filter, n_filter_ops, shards, n_shards }, out_counts, out_sums);
} FBGPU_CATCH

// GroupBy(..., aggregate=Count(Distinct(field=x))): fbgpu_groupby_sum's dimensions with, per cell, how many of x's listed stored
// values some column of filter ∩ the cell's rows holds.  Local to one context: distinct sets merge by union, which the u64 sum
// the ranks' tensors are reduced with is not
extern "C" int fbgpu_groupby_distinct(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                      const uint64_t* row_ids_flat, const int32_t* n_rows, const uint32_t* vfields, const uint32_t* vviews, const int32_t* bit_depths,
                                      int32_t n_ints, const int64_t* values_flat, const int32_t* n_values, uint32_t xfield, uint32_t xview, int32_t x_depth,
                                      const int64_t* x_values, int32_t n_x, const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards,
                                      uint64_t* out_distinct) try {
    int rc = groupby_agg_args(c, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, vfields, vviews, bit_depths, n_ints, values_flat, n_values,
                              x_values, "x_depth", x_depth, filter, n_filter_ops, shards, n_shards, out_distinct);
    if (rc) return rc;
    if (n_x < 1) return fail(FBGPU_E_INVALID, "n_x=%d < 1", n_x);
    for (int32_t i = 1; i < n_x; i++)
        if (x_values[i] <= x_values[i - 1]) return fail(FBGPU_E_INVALID, "x_values are not strictly ascending at position %d", i);
    if (c->comm || c->n_ranks > 1) return fail(FBGPU_E_COMM, "fbgpu_groupby_distinct is local to one context: distinct sets of the ranks merge by union, not by sum");
    return groupby_run(c, index, GbRequest{ gb_set_dims(fields, views_flat, n_views, n_fields, row_ids_flat, n_rows),
                                            gb_int_dims(vfields, vviews, bit_depths, n_ints, values_flat, n_values), GvAgg::kDistinct,
                                            GvInt{ xfield, xview, x_depth, x_values, n_x }, filter, n_filter_ops, shards, n_shards }, out_distinct);
} FBGPU_CATCH

// GroupBy(..., aggregate=Count(Distinct(field=x))) over a set-like x: fbgpu_groupby_distinct's dimensions with, per cell, how
// many of x's listed rows hold at least one column of filter ∩ the cell's rows.  Local to one context, as fbgpu_groupby_distinct
extern "C" int fbgpu_groupby_distinct_rows(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                           const uint64_t* row_ids_flat, const int32_t* n_rows, const uint32_t* vfields, const uint32_t* vviews,
                                           const int32_t* bit_depths, int32_t n_ints, const int64_t* values_flat, const int32_t* n_values, uint32_t xfield,
                                           uint32_t xview, const uint64_t* x_rows, int32_t n_x, const fbgpu_op* filter, int32_t n_filter_ops,
                                           const uint64_t* shards, int64_t n_shards, uint64_t* out_distinct) try {
    int rc = groupby_agg_args(c, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, vfields, vviews, bit_depths, n_ints, values_flat, n_values,
                              x_rows, "x_depth", 0 /* x has no depth */, filter, n_filter_ops, shards, n_shards, out_distinct);
    if (rc) return rc;
    if (n_x < 1) return fail(FBGPU_E_INVALID, "n_x=%d < 1", n_x);
    for (int32_t i = 1; i < n_x; i++)
        if (x_rows[i] <= x_rows[i - 1]) return fail(FBGPU_E_INVALID, "x_rows are not strictly ascending at position %d", i);
    if (c->comm || c->n_ranks > 1) return fail(FBGPU_E_COMM, "fbgpu_groupby_distinct_rows is local to one context: distinct sets of the ranks merge by union, not by sum");
    GvInt x{ xfield, xview, 0, nullptr, n_x };
    x.rows = x_rows;
    return groupby_run(c, index, GbRequest{ gb_set_dims(fields, views_flat, n_views, n_fields, row_ids_flat, n_rows),
                                            gb_int_dims(vfields, vviews, bit_depths, n_ints, values_flat, n_values), GvAgg::kDistinctRows,
                                            x, filter, n_filter_ops, shards, n_shards }, out_distinct);
} FBGPU_CATCH

// ------------------------------------------------------------------ GroupBy as a sorted list of its non-empty groups
// (sparse_rows_kernel, sparse_join_kernel, kernels.cuh).  A cell is the row-major flat index of fbgpu_groupby_views' tensor.
// Per evaluation batch of units: the filter is evaluated (none: every column counts), and the count pass of sparse_rows_kernel
// gives each unit its hits per dimension; units that miss a dimension are dropped, and the rest are cut into chunks of at most
// kSortChunk hits per dimension.  Per chunk, each dimension's (column, list index) keys are emitted, sorted and, over several
// views, deduped.  sparse_join_kernel turns dimension 0's entries, in ranges of at most kSortChunk cells, into the cells
// >= start; the cells are sorted and run-length coded into (cell, count), and merged into the call's running list by a sort of
// (cell, count) pairs and a sum of equal cells.  With a limit, the list is cut to its first `limit` cells after each merge, and
// once it holds that many, cells past its last one are not emitted.
// With an aggregate x (fbgpu_groupby_sparse_sum) the evaluated filter is <filter> ∩ exists(x), so every hit is a column holding
// a value.  Chunks also hold at most kSortChunk filter columns, and each chunk's filter columns get their stored values of x
// (columns_emit_kernel and extract_values_kernel over the chunk's units, in (unit, column) order).  The join emits (cell, value)
// pairs, sorted by cell; each run becomes (cell, count) as before and its wrapping sum (sparse_run_sums_kernel).  The sums form a
// second running list with the same cells, merged by the same deterministic sort and compaction, so the two stay aligned.
// With a distinct x (fbgpu_groupby_sparse_distinct(_rows)) x is one more, trailing, dimension of the join, whose index j is x's
// place in its list, and the join's strides are packed so that it emits the key cell << xbits | j (xbits = bit_width(n_x - 1)),
// within [start << xbits, end << xbits).  A set-like x is walked by sparse_rows_kernel like any dimension.  For an int x the
// filter holds exists(x), and the chunk's value list (as for Sum) becomes x's keys (sparse_xkeys_kernel, then sorted).  Each
// join range's keys are sorted and deduped, and merged into the running list of distinct (cell, j) keys by an append and
// another dedupe.  At the end the keys are shifted down to their cells and run-length coded: a run's length is the cell's
// distinct count.

namespace {                                                         // (internal linkage: not exported beside the C entry points)
// one sparse GroupBy request: the set dimensions, the aggregate as GbRequest carries it (kCount, kSum, kDistinct or kDistinctRows
// with its x), the filter, the shards and the window: the cells >= start, below end and at most `limit` of them (limit < 0: no
// cut).  The distinct pair takes end and no limit, kCount and kSum a limit and no end (~0).
struct SpRequest {
    std::vector<GbDim> dims;
    GvAgg agg; GvInt x;                                             // (x unused for kCount)
    const fbgpu_op* filter; int32_t n_filter_ops;
    const uint64_t* shards; int64_t n_shards;
    uint64_t start, end; int64_t limit;
    bool distinct() const { return agg == GvAgg::kDistinct || agg == GvAgg::kDistinctRows; }
};

// a sparse GroupBy's list: its cells, ascending, their counts (for the distinct pair the distinct counts) and, for kSum only, sums
struct SpResult { std::vector<uint64_t> cells, counts; std::vector<int64_t> sums; };
}  // namespace

// the argument checks every sparse GroupBy entry point and node form makes before any device is touched: the dimensions of the
// ABI's flat arrays and the outputs; for kSum x's depth and out_sums; for the distinct pair at most kSpMaxDims - 1 dimensions (x
// takes the join's last slot), x's list (values for an int x, rows for a set-like one) and depth, the range, and room in a u64
// for cell << bit_width(n_x - 1).  q's dimensions are not read: they are built from the arrays checked here.
static int groupby_sparse_args(const void* handle, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                               const uint64_t* row_ids_flat, const int32_t* n_rows, const SpRequest& q, const uint64_t* out_cells,
                               const uint64_t* out_counts, const int64_t* out_sums, uint64_t cap, const uint64_t* out_n) {
    if (!handle || !fields || !views_flat || !n_views || !row_ids_flat || !n_rows || !out_n || (cap && (!out_cells || !out_counts)) ||
        q.n_filter_ops < 0 || (q.n_filter_ops && !q.filter) || q.n_shards < 0 || (q.n_shards && !q.shards)) return fail(FBGPU_E_INVALID, "bad argument");
    if (n_fields < 1 || n_fields > kSpMaxDims) return fail(FBGPU_E_INVALID, "n_fields=%d outside 1..%d", n_fields, kSpMaxDims);
    const uint64_t* rows = row_ids_flat;
    uint64_t cells = 1;
    for (int32_t i = 0; i < n_fields; i++) {
        if (n_views[i] < 1) return fail(FBGPU_E_INVALID, "n_views[%d]=%d < 1", i, n_views[i]);
        if (n_rows[i] < 1) return fail(FBGPU_E_INVALID, "n_rows[%d]=%d < 1", i, n_rows[i]);
        for (int32_t k = 1; k < n_rows[i]; k++)
            if (rows[k] <= rows[k - 1]) return fail(FBGPU_E_INVALID, "row_ids[%d] are not strictly ascending at position %d", i, k);
        if (cells > ~0ull / (uint64_t)n_rows[i]) return fail(FBGPU_E_INVALID, "product of n_rows exceeds 2^64 - 1");
        cells *= (uint64_t)n_rows[i];
        rows += n_rows[i];
    }
    const GvInt& x = q.x;
    if (q.agg == GvAgg::kSum) {
        if (x.depth < 0 || x.depth > 64) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..64", x.depth);
        if (cap && !out_sums) return fail(FBGPU_E_INVALID, "bad argument");
    }
    if (!q.distinct()) return 0;
    if (n_fields > kSpMaxDims - 1) return fail(FBGPU_E_INVALID, "n_fields=%d outside 1..%d", n_fields, kSpMaxDims - 1);
    if (!x.values && !x.rows) return fail(FBGPU_E_INVALID, "bad argument");
    if (x.n_values < 1) return fail(FBGPU_E_INVALID, "n_x=%d < 1", x.n_values);
    for (int32_t i = 1; i < x.n_values; i++) {
        if (x.values && x.values[i] <= x.values[i - 1]) return fail(FBGPU_E_INVALID, "x_values are not strictly ascending at position %d", i);
        if (x.rows && x.rows[i] <= x.rows[i - 1]) return fail(FBGPU_E_INVALID, "x_rows are not strictly ascending at position %d", i);
    }
    if (x.depth < 0 || x.depth > 64) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..64", x.depth);
    if (q.start > q.end) return fail(FBGPU_E_INVALID, "start=%llu > end=%llu", (unsigned long long)q.start, (unsigned long long)q.end);
    const int xbits = bit_width((uint64_t)x.n_values - 1);
    if (cells > (~0ull >> xbits)) return fail(FBGPU_E_INVALID, "product of n_rows times 2^%d exceeds 2^64 - 1", xbits);
    return 0;
}

// device buffers of one fbgpu_groupby_sparse call, freed when it returns: they can be large, and are not reused by other calls.
// b[d]: dimension d's keys (with a distinct x, x is the last dimension); b[nd]: the cells (with an aggregate, (cell, value)
// pairs; with a distinct x, (cell, x) keys); b[kSpMaxDims + 1]: the cursor, row lists, an int x's listed values and view slots;
// with an aggregate or an int x, b[kSpMaxDims + 2]: a chunk's value list, b[kSpMaxDims + 3]: its two ColUnit lists;
// b[kSpMaxDims + 4]: the running list of sums, or with a distinct x the final (cell, distinct count) list.
struct SparseBufs {
    DevBuf b[kSpMaxDims + 5];
    ~SparseBufs() { for (DevBuf& x : b) x.release(); }
};

// the sorted cells of cs into (cell, count) pairs merged into acc, whose cells are distinct and sorted; then acc cut to its first
// `limit` cells (limit < 0: no cut), and *hi lowered to one past its last cell once it holds that many.  With `sums`, cs holds
// (cell, value) pairs, and each run's wrapping sum of values goes into *sums, a list with acc's cells, merged and cut alike.
static int sparse_merge(Query& q, SortPairs& cs, SortPairs& acc, SortPairs* sums, int bits, int64_t limit, unsigned long long* hi) {
    Workspace* w = q.w;
    const uint64_t n = cs.n, n_tiles = (n + kSortTile - 1) / kSortTile;
    if (w->d_counts.ensure((size_t)(n_tiles + 1) * 4) || w->h_out.ensure(8)) return FBGPU_E_NOMEM;
    unsigned int* counts = (unsigned int*)w->d_counts.p;
    distinct_heads_kernel<<<(unsigned)n_tiles, kSortThreads, 0, w->stream>>>(cs.keys(cs.cur), n, counts);
    CUDA_TRY(cudaGetLastError());
    sort_scan_kernel<<<1, kSortScanThreads, 0, w->stream>>>(counts, n_tiles + 1);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, counts + n_tiles, 4, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    const uint64_t u = *(const unsigned int*)w->h_out.p;
    int rc = acc.reserve(acc.n + u); if (rc) return rc;
    if (sums) { rc = sums->reserve(sums->n + u); if (rc) return rc; }
    unsigned long long* pos = cs.keys(1 - cs.cur);          // the sort's free half: the runs' first positions
    sparse_compact_kernel<false><<<(unsigned)n_tiles, kSortThreads, 0, w->stream>>>(cs.keys(cs.cur), nullptr, n, counts, acc.keys(acc.cur) + acc.n, pos);
    CUDA_TRY(cudaGetLastError());
    const unsigned grid = (unsigned)std::min<uint64_t>((u + 255) / 256, (uint64_t)q.c->sm_count * 8);
    sparse_run_lengths_kernel<<<grid, 256, 0, w->stream>>>(pos, u, n, acc.cols(acc.cur) + acc.n);
    CUDA_TRY(cudaGetLastError());
    q.launches += 4;
    if (sums) {
        CUDA_TRY(cudaMemcpyAsync(sums->keys(sums->cur) + sums->n, acc.keys(acc.cur) + acc.n, u * 8, cudaMemcpyDeviceToDevice, w->stream));
        CUDA_TRY(cudaMemsetAsync(sums->cols(sums->cur) + sums->n, 0, u * 8, w->stream));
        sparse_run_sums_kernel<<<(unsigned)n_tiles, kSortThreads, 0, w->stream>>>(cs.keys(cs.cur), cs.cols(cs.cur), n, counts, sums->cols(sums->cur) + sums->n);
        CUDA_TRY(cudaGetLastError());
        q.launches++;
        sums->n += u;
    }
    const bool merge = acc.n > 0;
    acc.n += u;
    if (merge) {
        rc = sort_pairs(q, acc, bits, ~0ull); if (rc) return rc;
        if (sums) { rc = sort_pairs(q, *sums, bits, ~0ull); if (rc) return rc; }    // the same keys: the same order
        const uint64_t m = acc.n, m_tiles = (m + kSortTile - 1) / kSortTile;
        if (w->d_counts.ensure((size_t)(m_tiles + 1) * 4)) return FBGPU_E_NOMEM;
        counts = (unsigned int*)w->d_counts.p;
        distinct_heads_kernel<<<(unsigned)m_tiles, kSortThreads, 0, w->stream>>>(acc.keys(acc.cur), m, counts);
        CUDA_TRY(cudaGetLastError());
        sort_scan_kernel<<<1, kSortScanThreads, 0, w->stream>>>(counts, m_tiles + 1);
        CUDA_TRY(cudaGetLastError());
        sparse_compact_kernel<true><<<(unsigned)m_tiles, kSortThreads, 0, w->stream>>>(acc.keys(acc.cur), acc.cols(acc.cur), m, counts,
                                                                                      acc.keys(1 - acc.cur), acc.cols(1 - acc.cur));
        CUDA_TRY(cudaGetLastError());
        q.launches += 3;
        acc.cur = 1 - acc.cur;
        if (sums) {
            sparse_compact_kernel<true><<<(unsigned)m_tiles, kSortThreads, 0, w->stream>>>(sums->keys(sums->cur), sums->cols(sums->cur), m, counts,
                                                                                          sums->keys(1 - sums->cur), sums->cols(1 - sums->cur));
            CUDA_TRY(cudaGetLastError());
            q.launches++;
            sums->cur = 1 - sums->cur;
        }
        CUDA_TRY(cudaMemcpyAsync(w->h_out.p, counts + m_tiles, 4, cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        acc.n = *(const unsigned int*)w->h_out.p;
        if (sums) sums->n = acc.n;
    }
    if (limit >= 0 && acc.n >= (uint64_t)limit) {
        acc.n = (uint64_t)limit;
        if (sums) sums->n = (uint64_t)limit;
        CUDA_TRY(cudaMemcpyAsync(w->h_out.p, acc.keys(acc.cur) + acc.n - 1, 8, cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        *hi = *(const uint64_t*)w->h_out.p + 1;
    }
    return 0;
}

// the distinct sorted keys of cs added to acc, a keys-only list of distinct sorted keys: appended, then sorted and deduped
static int sparse_union(Query& q, const SortPairs& cs, SortPairs& acc, int bits) {
    const bool merge = acc.n > 0;
    int rc = acc.reserve(acc.n + cs.n); if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(acc.keys(acc.cur) + acc.n, cs.keys(cs.cur), cs.n * 8, cudaMemcpyDeviceToDevice, q.w->stream));
    acc.n += cs.n;
    return merge ? distinct_keys(q, acc, bits) : 0;
}

namespace {
// one groupby_sparse_run: the request, its query and join, the call's device buffers and what was uploaded into them, and the
// running lists.  The stages below work on it; the batch and the chunk a stage works on are passed to it.
struct SpCall {
    fbgpu_ctx* c;
    uint32_t index;
    const SpRequest& r;
    const bool x_int = r.agg == GvAgg::kDistinct;
    const bool vals = x_int || r.agg == GvAgg::kSum;                // a value list per chunk, of Sum's x or of an int distinct x
    std::vector<GbDim> dims = r.dims;                               // the dimensions sparse_rows_kernel walks: a set-like x is the last one
    const int ng = (int)r.dims.size();
    const int nd = ng + (r.distinct() ? 1 : 0);                     // the join's dimensions
    const int xbits = r.distinct() ? bit_width((uint64_t)r.x.n_values - 1) : 0;
    int cell_bits = 0;                                              // a join key's bits
    Query q{ c };
    Workspace* w = q.w;
    const std::vector<uint64_t> sorted = sorted_unique(r.shards, r.n_shards);
    bool have_filter = false;
    uint32_t fv_x = 0;
    SpJoin jn{};
    SparseBufs sb;
    // sb.b[kSpMaxDims + 1]: [cursor | dimension d's rows at row_at[d] | an int x's values at d_xs | its n_fv[d] view slots at fv_at[d] of d_fv0]
    unsigned long long* cursor = nullptr;
    const long long* d_xs = nullptr;
    const uint32_t* d_fv0 = nullptr;
    std::vector<size_t> row_at, fv_at;
    std::vector<int> n_fv;
    std::vector<SortPairs> dk;                                      // each join dimension's keys
    SortPairs cs{ w, ~0ull, r.agg != GvAgg::kSum, &sb.b[nd] };      // a join range's cells ((cell, value) pairs for kSum)
    SortPairs acc{ w, ~0ull, r.distinct() };                        // the running list: (cell, count) pairs or distinct (cell, x) keys
    SortPairs acc_sums{ w, ~0ull, false, &sb.b[kSpMaxDims + 4] };   // kSum's running sums, or the distinct pair's final list
    SortPairs* sums = nullptr;                                      // acc_sums for kSum
    int (*fold)(SpCall&) = nullptr;                                 // folds cs into the running list
};

// an evaluation batch from unit u0: the units with filter columns (ncol[k] in units[k]), their hits per walked dimension
// (ucnt[d * units.size() + k]) and, as places in `units`, the ones every dimension meets
struct SpBatch {
    long long u0;
    const uint4* bitmaps;
    const uint64_t* shards;
    std::vector<uint32_t> units, ncol, keep;
    std::vector<uint64_t> ucnt;
};

// a chunk: keep[a, b) of its batch, its units, their hits per dimension and filter columns, and their value list
struct SpChunk {
    size_t a, b;
    std::vector<uint32_t> units;
    std::vector<uint64_t> hits;
    uint64_t vn;
    SpVals vl;
};
}  // namespace

// folding a join range into the running list: merge counts (and, for kSum, sums), or union distinct keys; set-up picks which
static int sparse_fold_merge(SpCall& s) {
    int rc = sort_pairs(s.q, s.cs, s.cell_bits, ~0ull); if (rc) return rc;
    return sparse_merge(s.q, s.cs, s.acc, s.sums, s.cell_bits, s.r.limit, &s.jn.hi);
}
static int sparse_fold_union(SpCall& s) {
    int rc = distinct_keys(s.q, s.cs, s.cell_bits); if (rc) return rc;
    return sparse_union(s.q, s.cs, s.acc, s.cell_bits);
}

// set-up: filter ∩ exists(x) (with a value list, as for fbgpu_bsi_sum), the strides, the fold; *empty when the window holds no
// cell, else the metadata uploaded
static int sparse_setup(SpCall& s, bool* empty) {
    const SpRequest& r = s.r;
    const fbgpu_op* filter = r.filter;
    int32_t n_filter_ops = r.n_filter_ops;
    std::vector<fbgpu_op> full;
    if (s.vals) {
        full = and_row(filter, n_filter_ops, r.x.field, r.x.view, 0);
        s.fv_x = view_id_locked(s.c, ViewKey{ s.index, r.x.field, r.x.view }, false);
        filter = full.data(); n_filter_ops = (int32_t)full.size();
    }
    s.have_filter = n_filter_ops > 0;
    int rc = s.have_filter ? s.q.open(s.index, filter, n_filter_ops, s.sorted.data(), (int64_t)s.sorted.size()) : s.q.open(s.sorted.data(), (int64_t)s.sorted.size());
    if (rc) return rc;
    SpJoin& jn = s.jn;
    jn.nd = s.nd; jn.lo = r.start; jn.hi = ~0ull;
    uint64_t total = 1;                              // the group dimensions' cells; x, when there is one, has stride 1
    for (int d = s.ng - 1; d >= 0; d--) { jn.stride[d] = total << s.xbits; total *= (uint64_t)r.dims[d].n_rows; jn.jbits[d] = bit_width((uint64_t)r.dims[d].n_rows - 1); }
    s.sums = r.agg == GvAgg::kSum ? &s.acc_sums : nullptr;
    s.fold = r.distinct() ? sparse_fold_union : sparse_fold_merge;
    if (r.distinct()) {
        jn.stride[s.ng] = 1; jn.jbits[s.ng] = s.xbits;
        const uint64_t e = std::min(r.end, total);
        jn.lo = std::min(r.start, e) << s.xbits; jn.hi = e << s.xbits;
    }
    s.cell_bits = bit_width((total << s.xbits) - 1);
    *empty = r.limit == 0 || jn.lo >= jn.hi;
    if (*empty) return 0;
    if (r.agg == GvAgg::kDistinctRows) s.dims.push_back(GbDim{ r.x.field, &r.x.view, 1, r.x.rows, r.x.n_values });
    std::vector<uint64_t> rows_h(1, 0);              // the cursor, then the rows
    std::vector<uint32_t> fvs_h;
    for (const GbDim& g : s.dims) {
        s.row_at.push_back(rows_h.size()); rows_h.insert(rows_h.end(), g.rows, g.rows + g.n_rows);
        const std::vector<uint32_t> fvs = view_slots(s.c, s.index, g.field, g.views, g.n_views);
        s.fv_at.push_back(fvs_h.size()); s.n_fv.push_back((int)fvs.size()); fvs_h.insert(fvs_h.end(), fvs.begin(), fvs.end());
    }
    const size_t xv_at = rows_h.size();
    if (s.x_int) rows_h.insert(rows_h.end(), r.x.values, r.x.values + r.x.n_values);
    DevBuf& meta = s.sb.b[kSpMaxDims + 1];
    if (meta.ensure(rows_h.size() * 8 + fvs_h.size() * 4)) return FBGPU_E_NOMEM;
    s.cursor = (unsigned long long*)meta.p;
    s.d_xs = (const long long*)s.cursor + xv_at;
    s.d_fv0 = (const uint32_t*)(s.cursor + rows_h.size());
    CUDA_TRY(cudaMemcpyAsync(meta.p, rows_h.data(), rows_h.size() * 8, cudaMemcpyHostToDevice, s.w->stream));
    CUDA_TRY(cudaMemcpyAsync((void*)s.d_fv0, fvs_h.data(), fvs_h.size() * 4, cudaMemcpyHostToDevice, s.w->stream));
    CUDA_TRY(cudaStreamSynchronize(s.w->stream));
    for (int d = 0; d < s.nd; d++) s.dk.emplace_back(s.w, ~0ull, true, &s.sb.b[d]);
    return 0;
}

// sparse_rows_kernel over walked dimension d for the n units at d_units: their hits into counts (kCount) or their keys at the
// cursor into keys (kEmit)
template <SrOut kMode>
static int sparse_rows(SpCall& s, const SpBatch& bt, size_t d, int n, unsigned long long* counts, unsigned long long* keys) {
    const unsigned grid = (unsigned)std::min<size_t>((size_t)n, (size_t)s.c->sm_count * 8);
    sparse_rows_kernel<kMode><<<grid, kSrThreads, 0, s.w->stream>>>(store_ref(s.c), s.d_fv0 + s.fv_at[d], s.n_fv[d], (const uint64_t*)s.cursor + s.row_at[d],
        s.dims[d].n_rows, s.jn.jbits[d], bt.bitmaps, (const uint32_t*)s.w->d_emit_units.p, n, bt.shards, counts, keys ? s.cursor : nullptr, keys);
    CUDA_TRY(cudaGetLastError()); s.q.launches++;
    return 0;
}

// a batch's units [u0, u0 + nu): evaluation, the kCount pass, the units every dimension meets
static int sparse_batch(SpCall& s, long long u0, long long nu, SpBatch& bt) {
    Workspace* w = s.w;
    bt.u0 = u0;
    bt.units.clear(); bt.ncol.clear();
    if (s.have_filter) {
        const uint2* info;
        int rc = s.q.eval_info(u0, nu, info); if (rc) return rc;
        for (long long u = 0; u < nu; u++) if (info[u].x) { bt.units.push_back((uint32_t)u); bt.ncol.push_back(info[u].x); }
    } else {
        for (long long u = 0; u < nu; u++) bt.units.push_back((uint32_t)u);
    }
    if (bt.units.empty()) return 0;
    bt.bitmaps = s.have_filter ? (const uint4*)w->d_bitmaps.p : nullptr;
    bt.shards = s.q.d_shards + u0 / kSlotsPerRow;
    const size_t nun = bt.units.size(), nr = s.dims.size();
    if (w->d_emit_units.ensure(nun * 4) || w->d_cells.ensure(nun * nr * 8) || w->h_out.ensure(nun * nr * 8)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemcpyAsync(w->d_emit_units.p, bt.units.data(), nun * 4, cudaMemcpyHostToDevice, w->stream));
    CUDA_TRY(cudaMemsetAsync(w->d_cells.p, 0, nun * nr * 8, w->stream));
    for (size_t d = 0; d < nr; d++) {
        int rc = sparse_rows<SrOut::kCount>(s, bt, d, (int)nun, (unsigned long long*)w->d_cells.p + d * nun, nullptr); if (rc) return rc;
    }
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_cells.p, nun * nr * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    bt.ucnt.assign((const uint64_t*)w->h_out.p, (const uint64_t*)w->h_out.p + nun * nr);
    bt.keep.clear();
    for (size_t e = 0; e < nun; e++) {
        bool all = true;
        for (size_t d = 0; d < nr && all; d++) all = bt.ucnt[d * nun + e] > 0;
        if (all) bt.keep.push_back((uint32_t)e);
    }
    return 0;
}

// chunk planning: keep[a, b) of at most kSortChunk hits per dimension and, with a value list, filter columns (at least one unit)
static int sparse_plan(SpCall& s, const SpBatch& bt, size_t a, SpChunk& ch) {
    const size_t nun = bt.units.size(), nr = s.dims.size();
    ch.a = a;
    ch.hits.assign(nr, 0);
    ch.vn = 0;
    for (ch.b = a; ch.b < bt.keep.size(); ch.b++) {
        const uint32_t e = bt.keep[ch.b];
        bool fits = !s.vals || ch.vn + bt.ncol[e] <= kSortChunk;
        for (size_t d = 0; d < nr; d++) fits = fits && ch.hits[d] + bt.ucnt[d * nun + e] <= kSortChunk;
        if (!fits && ch.b > a) break;
        for (size_t d = 0; d < nr; d++) ch.hits[d] += bt.ucnt[d * nun + e];
        if (s.vals) ch.vn += bt.ncol[e];
    }
    ch.units.clear();
    for (size_t k = a; k < ch.b; k++) ch.units.push_back(bt.units[bt.keep[k]]);
    if (s.w->d_emit_units.ensure(ch.units.size() * 4)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemcpyAsync(s.w->d_emit_units.p, ch.units.data(), ch.units.size() * 4, cudaMemcpyHostToDevice, s.w->stream));
    return 0;
}

// a chunk's dimension keys
static int sparse_keys(SpCall& s, const SpBatch& bt, const SpChunk& ch) {
    for (size_t d = 0; d < s.dims.size(); d++) {
        SortPairs& k = s.dk[d];
        k.n = 0;
        int rc = k.reserve(ch.hits[d]); if (rc) return rc;
        CUDA_TRY(cudaMemsetAsync(s.cursor, 0, 8, s.w->stream));
        rc = sparse_rows<SrOut::kEmit>(s, bt, d, (int)ch.units.size(), nullptr, k.keys(k.cur)); if (rc) return rc;
        k.n = ch.hits[d];
        const int kbits = bit_width(ch.units.size() - 1) + 16 + s.jn.jbits[d];
        rc = s.n_fv[d] > 1 ? distinct_keys(s.q, k, kbits) : sort_pairs(s.q, k, kbits, ~0ull); if (rc) return rc;
        s.jn.keys[d] = k.keys(k.cur); s.jn.n[d] = k.n;
    }
    return 0;
}

// a chunk's value list (kSum or an int x): its units' filter columns in (unit, column) order as (e << 16 | c) keys, and their
// values' magnitudes and sign bits; for an int x, x's keys from it
static int sparse_values(SpCall& s, const SpBatch& bt, SpChunk& ch) {
    if (!s.vals) return 0;
    Workspace* w = s.w;
    const uint64_t vn = ch.vn;
    const int nc = (int)ch.units.size();
    const unsigned grid = (unsigned)std::min<size_t>((size_t)nc, (size_t)s.c->sm_count * 8);
    std::vector<ColUnit> vunits;
    for (int pass = 0; pass < 2; pass++) {
        uint64_t off = 0;
        for (size_t k = ch.a; k < ch.b; k++) {
            ColUnit cu{};
            const uint32_t u = bt.units[bt.keep[k]];
            cu.out_off = off; cu.unit = u; cu.first = 0; cu.last = bt.ncol[bt.keep[k]];
            cu.col_base = pass == 0 ? (s.sorted[(bt.u0 + u) / kSlotsPerRow] << 20) + (uint64_t)((bt.u0 + u) % kSlotsPerRow) * 65536ull
                                    : (uint64_t)(k - ch.a) << 16;
            vunits.push_back(cu);
            off += cu.last;
        }
    }
    DevBuf& vb = s.sb.b[kSpMaxDims + 2]; DevBuf& ub = s.sb.b[kSpMaxDims + 3];
    const size_t sign_bytes = ((vn + 31) / 32) * 4;
    if (vb.ensure(vn * 16 + sign_bytes) || ub.ensure(vunits.size() * sizeof(ColUnit))) return FBGPU_E_NOMEM;
    unsigned long long* vcols = (unsigned long long*)vb.p; unsigned long long* mag = vcols + vn;
    unsigned int* sign = (unsigned int*)(mag + vn);
    const ColUnit* d_vu = (const ColUnit*)ub.p;
    CUDA_TRY(cudaMemcpyAsync(ub.p, vunits.data(), vunits.size() * sizeof(ColUnit), cudaMemcpyHostToDevice, w->stream));
    CUDA_TRY(cudaMemsetAsync(mag, 0, vn * 8 + sign_bytes, w->stream));
    columns_emit_kernel<<<grid, kEmitThreads, 0, w->stream>>>(bt.bitmaps, d_vu + nc, nc, vcols);
    CUDA_TRY(cudaGetLastError());
    extract_values_kernel<<<grid, kExtractThreads, 0, w->stream>>>(store_ref(s.c), s.fv_x, s.r.x.depth, bt.bitmaps, d_vu, nc, mag, sign);
    CUDA_TRY(cudaGetLastError());
    s.q.launches += 2;
    const SpVals& vl = ch.vl = SpVals{ vcols, mag, sign, vn, nullptr };
    if (!s.x_int) return 0;
    SortPairs& k = s.dk[s.dims.size()];
    k.n = 0;
    int rc = k.reserve(vn); if (rc) return rc;
    CUDA_TRY(cudaMemsetAsync(s.cursor, 0, 8, w->stream));
    const unsigned xgrid = (unsigned)std::min<uint64_t>((vn + 255) / 256, (uint64_t)s.c->sm_count * 8);
    sparse_xkeys_kernel<<<xgrid, 256, 0, w->stream>>>(vl.cols, vl.mag, vl.sign, vn, s.d_xs, s.r.x.n_values, s.xbits, s.cursor, k.keys(k.cur));
    CUDA_TRY(cudaGetLastError()); s.q.launches++;
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, s.cursor, 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    k.n = *(const uint64_t*)w->h_out.p;
    rc = sort_pairs(s.q, k, bit_width((uint64_t)nc - 1) + 16 + s.xbits, ~0ull); if (rc) return rc;
    s.jn.keys[s.dims.size()] = k.keys(k.cur); s.jn.n[s.dims.size()] = k.n;
    return 0;
}

// the join-range search and emit: [e0, n0) of dimension 0's entries halved to [e0, *e1) until it gives at most kSortChunk cells
// (at least one entry), and those cells emitted into cs, with kSum's values taken from the chunk's value list
static int sparse_join_range(SpCall& s, SpChunk& ch, uint64_t e0, uint64_t* e1) {
    Workspace* w = s.w;
    const uint64_t n0 = s.jn.n[0];
    const unsigned grid = (unsigned)std::min<uint64_t>((n0 + 255) / 256, (uint64_t)s.c->sm_count * 8);
    uint64_t got = 0;
    for (*e1 = n0;; *e1 = e0 + (*e1 - e0) / 2) {
        CUDA_TRY(cudaMemsetAsync(s.cursor, 0, 8, w->stream));
        sparse_join_kernel<SrOut::kCount><<<grid, 256, 0, w->stream>>>(s.jn, e0, *e1, s.cursor, nullptr, SpVals{});
        CUDA_TRY(cudaGetLastError()); s.q.launches++;
        CUDA_TRY(cudaMemcpyAsync(w->h_out.p, s.cursor, 8, cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        got = *(const uint64_t*)w->h_out.p;
        if (got <= kSortChunk || *e1 - e0 == 1) break;
    }
    SortPairs& cs = s.cs;
    cs.n = 0;
    if (!got) return 0;
    int rc = cs.reserve(got); if (rc) return rc;
    CUDA_TRY(cudaMemsetAsync(s.cursor, 0, 8, w->stream));
    if (s.r.agg == GvAgg::kSum) {
        ch.vl.out = cs.cols(cs.cur);
        sparse_join_kernel<SrOut::kSum><<<grid, 256, 0, w->stream>>>(s.jn, e0, *e1, s.cursor, cs.keys(cs.cur), ch.vl);
    } else {
        sparse_join_kernel<SrOut::kEmit><<<grid, 256, 0, w->stream>>>(s.jn, e0, *e1, s.cursor, cs.keys(cs.cur), SpVals{});
    }
    CUDA_TRY(cudaGetLastError()); s.q.launches++;
    cs.n = got;
    return 0;
}

// the distinct pair's final run-length coding of its keys' cells into acc_sums; then the read-back
static int sparse_finish(SpCall& s, SpResult& out) {
    Workspace* w = s.w;
    SortPairs& acc = s.acc;
    SortPairs& res = s.r.distinct() ? s.acc_sums : acc;
    if (s.r.distinct() && acc.n) {
        CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
        const unsigned grid = (unsigned)std::min<uint64_t>((acc.n + 255) / 256, (uint64_t)s.c->sm_count * 8);
        sparse_shift_kernel<<<grid, 256, 0, w->stream>>>(acc.keys(acc.cur), acc.n, s.xbits);
        CUDA_TRY(cudaGetLastError()); s.q.launches++;
        unsigned long long no_hi = ~0ull;
        int rc = sparse_merge(s.q, acc, s.acc_sums, nullptr, s.cell_bits, -1, &no_hi); if (rc) return rc;
        CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        s.q.add_elapsed();
    }
    out.cells.resize(res.n); out.counts.resize(res.n);
    if (res.n) {
        CUDA_TRY(cudaMemcpyAsync(out.cells.data(), res.keys(res.cur), res.n * 8, cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaMemcpyAsync(out.counts.data(), res.cols(res.cur), res.n * 8, cudaMemcpyDeviceToHost, w->stream));
        if (s.sums) {
            out.sums.resize(acc.n);
            CUDA_TRY(cudaMemcpyAsync(out.sums.data(), s.sums->cols(s.sums->cur), acc.n * 8, cudaMemcpyDeviceToHost, w->stream));
        }
        CUDA_TRY(cudaStreamSynchronize(w->stream));
    }
    return 0;
}

// r's non-empty cells >= start, ascending, at most `limit` of them, and their counts (store lock held).  For kSum the filter is
// <filter> ∩ exists(x), a cell is non-empty when its count there is, and each listed cell gets its wrapping sum of x's stored
// values.  For the distinct pair, the cells in [start, end) where at least one listed x value (row) is held by a column of the
// filter ∩ the cell's rows, and as counts the number of such x.
static int groupby_sparse_run(fbgpu_ctx* c, uint32_t index, const SpRequest& r, SpResult& out) {
    SpCall s{ c, index, r };
    bool empty = false;
    int rc = sparse_setup(s, &empty); if (rc) return rc;
    if (empty) { s.q.finish(); return FBGPU_OK; }
    const long long batch = std::min<long long>(c->unit_batch, 1ll << 16);     // a unit's place in a chunk takes 16 bits of a key
    SpBatch bt;
    SpChunk ch;
    for (long long u0 = 0; u0 < s.q.n_units; u0 += batch) {
        CUDA_TRY(cudaEventRecord(s.w->ev0, s.w->stream));
        rc = sparse_batch(s, u0, std::min(batch, s.q.n_units - u0), bt); if (rc) return rc;
        if (bt.units.empty()) continue;
        for (size_t a = 0; a < bt.keep.size(); a = ch.b) {
            rc = sparse_plan(s, bt, a, ch); if (rc) return rc;
            rc = sparse_keys(s, bt, ch); if (rc) return rc;
            rc = sparse_values(s, bt, ch); if (rc) return rc;
            for (uint64_t e0 = 0, e1 = 0; e0 < s.jn.n[0]; e0 = e1) {
                rc = sparse_join_range(s, ch, e0, &e1); if (rc) return rc;
                if (s.cs.n) { rc = s.fold(s); if (rc) return rc; }
            }
        }
        CUDA_TRY(cudaEventRecord(s.w->ev1, s.w->stream));
        CUDA_TRY(cudaStreamSynchronize(s.w->stream));
        s.q.add_elapsed();
    }
    rc = sparse_finish(s, out); if (rc) return rc;
    s.q.finish();
    return FBGPU_OK;
}

// a (cell, count) list, with its sums when it has any, into the caller's arrays under the NOSPACE contract: *out_n = its size,
// nothing written when it exceeds cap
static int write_cells(const SpResult& r, uint64_t* out_cells, uint64_t* out_counts, int64_t* out_sums, uint64_t cap, uint64_t* out_n) {
    *out_n = r.cells.size();
    if (r.cells.size() > cap) return fail(FBGPU_E_NOSPACE, "output needs room for %llu cells", (unsigned long long)r.cells.size());
    if (!r.cells.empty()) { memcpy(out_cells, r.cells.data(), r.cells.size() * 8); memcpy(out_counts, r.counts.data(), r.counts.size() * 8); }
    if (!r.sums.empty()) memcpy(out_sums, r.sums.data(), r.sums.size() * 8);
    return FBGPU_OK;
}

// the sparse GroupBy entry point `name`: the argument checks, the refusal with ranks attached (group lists merge by cell and
// distinct sets by union, neither by an all-reduce), then q over the dimensions of the flat arrays, the store locked, and the
// list written out
static int groupby_sparse_call(fbgpu_ctx* c, const char* name, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views,
                               int32_t n_fields, const uint64_t* row_ids_flat, const int32_t* n_rows, SpRequest q,
                               uint64_t* out_cells, uint64_t* out_counts, int64_t* out_sums, uint64_t cap, uint64_t* out_n) {
    int rc = groupby_sparse_args(c, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, q, out_cells, out_counts, out_sums, cap, out_n);
    if (rc) return rc;
    if (c->comm || c->n_ranks > 1)
        return q.distinct() ? fail(FBGPU_E_COMM, "%s is local to one context: distinct sets of the ranks merge by union, not by sum", name)
                            : fail(FBGPU_E_COMM, "%s is local to one context: group lists merge by cell, not by an all-reduce", name);
    q.dims = gb_set_dims(fields, views_flat, n_views, n_fields, row_ids_flat, n_rows);
    std::shared_lock<std::shared_mutex> lk;
    rc = begin_query(c, lk); if (rc) return rc;
    SpResult r;
    rc = groupby_sparse_run(c, index, q, r); if (rc) return rc;
    return write_cells(r, out_cells, out_counts, out_sums, cap, out_n);
}

// GroupBy over set-like dimensions of any number of rows: fbgpu_groupby_views' cells, as the sorted list of the non-empty ones
// from `start` on, at most `limit` of them (executeGroupBy's walk of groupByIterator, executor.go:3176, with previous= / limit=)
extern "C" int fbgpu_groupby_sparse(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                    const uint64_t* row_ids_flat, const int32_t* n_rows, const fbgpu_op* filter, int32_t n_filter_ops,
                                    const uint64_t* shards, int64_t n_shards, uint64_t start, int64_t limit,
                                    uint64_t* out_cells, uint64_t* out_counts, uint64_t cap, uint64_t* out_n) try {
    return groupby_sparse_call(c, "fbgpu_groupby_sparse", index, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows,
                               SpRequest{ {}, GvAgg::kCount, {}, filter, n_filter_ops, shards, n_shards, start, ~0ull, limit },
                               out_cells, out_counts, nullptr, cap, out_n);
} FBGPU_CATCH

// GroupBy(..., aggregate=Sum(field=x)) over set-like dimensions of any number of rows: fbgpu_groupby_sparse's list, where a cell is
// listed when filter ∩ its rows ∩ exists(x) is non-empty, with that count and the wrapping sum of the columns' stored values
// (groupByIterator.Next's Sum, executor.go:8893-8919, which skips a group whose count is 0)
extern "C" int fbgpu_groupby_sparse_sum(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                        const uint64_t* row_ids_flat, const int32_t* n_rows, uint32_t afield, uint32_t aview, int32_t a_depth,
                                        const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t start, int64_t limit,
                                        uint64_t* out_cells, uint64_t* out_counts, int64_t* out_sums, uint64_t cap, uint64_t* out_n) try {
    return groupby_sparse_call(c, "fbgpu_groupby_sparse_sum", index, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows,
                               SpRequest{ {}, GvAgg::kSum, GvInt{ afield, aview, a_depth, nullptr, 0 }, filter, n_filter_ops, shards, n_shards, start, ~0ull, limit },
                               out_cells, out_counts, out_sums, cap, out_n);
} FBGPU_CATCH

// GroupBy(..., aggregate=Count(Distinct(field=x))) over set-like dimensions of any number of rows, x an int field: per cell of
// fbgpu_groupby_sparse's in [start, end), the number of listed stored values of x that a column of filter ∩ the cell's rows
// holds, listed where it is non-zero (executeGroupBy's Count(Distinct), executor.go:3343-3385, for every group at once)
extern "C" int fbgpu_groupby_sparse_distinct(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views,
                                             int32_t n_fields, const uint64_t* row_ids_flat, const int32_t* n_rows, uint32_t xfield, uint32_t xview,
                                             int32_t x_depth, const int64_t* x_values, int32_t n_x, const fbgpu_op* filter, int32_t n_filter_ops,
                                             const uint64_t* shards, int64_t n_shards, uint64_t start, uint64_t end,
                                             uint64_t* out_cells, uint64_t* out_distinct, uint64_t cap, uint64_t* out_n) try {
    return groupby_sparse_call(c, "fbgpu_groupby_sparse_distinct", index, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows,
                               SpRequest{ {}, GvAgg::kDistinct, GvInt{ xfield, xview, x_depth, x_values, n_x }, filter, n_filter_ops, shards, n_shards, start, end, -1 },
                               out_cells, out_distinct, nullptr, cap, out_n);
} FBGPU_CATCH

// the same with a set, mutex, bool or time field x: per cell, the number of listed rows of x holding a column of filter ∩ the
// cell's rows
extern "C" int fbgpu_groupby_sparse_distinct_rows(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views,
                                                  int32_t n_fields, const uint64_t* row_ids_flat, const int32_t* n_rows, uint32_t xfield, uint32_t xview,
                                                  const uint64_t* x_rows, int32_t n_x, const fbgpu_op* filter, int32_t n_filter_ops,
                                                  const uint64_t* shards, int64_t n_shards, uint64_t start, uint64_t end,
                                                  uint64_t* out_cells, uint64_t* out_distinct, uint64_t cap, uint64_t* out_n) try {
    return groupby_sparse_call(c, "fbgpu_groupby_sparse_distinct_rows", index, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows,
                               SpRequest{ {}, GvAgg::kDistinctRows, GvInt{ xfield, xview, 0, nullptr, n_x, x_rows }, filter, n_filter_ops, shards, n_shards,
                                          start, end, -1 },
                               out_cells, out_distinct, nullptr, cap, out_n);
} FBGPU_CATCH

// ------------------------------------------------------------------ comm
extern "C" int fbgpu_comm_unique_id(uint8_t id[FBGPU_NCCL_ID_BYTES]) try {
    if (!nccl_load()) return fail(FBGPU_E_COMM, "libnccl.so.2 not loadable: %s", dlerror());
    int r = g_nccl.GetUniqueId(id);
    if (r) return fail(FBGPU_E_COMM, "ncclGetUniqueId failed (%d)", r);
    return 0;
} FBGPU_CATCH
extern "C" int fbgpu_comm_init(fbgpu_ctx* c, int32_t n_ranks, int32_t rank, const uint8_t id[FBGPU_NCCL_ID_BYTES]) try {
    if (!c || !id || n_ranks < 1 || rank < 0 || rank >= n_ranks) return fail(FBGPU_E_INVALID, "bad argument");
    if (!nccl_load()) return fail(FBGPU_E_COMM, "libnccl.so.2 not loadable");
    USE_DEVICE(c);
    Id128 u; memcpy(u.b, id, 128);
    void* comm = nullptr;
    int r = g_nccl.CommInitRank(&comm, n_ranks, u, rank);
    if (r) return fail(FBGPU_E_COMM, "ncclCommInitRank failed: %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?");
    c->comm = comm; c->n_ranks = n_ranks; c->rank = rank;
    return 0;
} FBGPU_CATCH
extern "C" int fbgpu_comm_destroy(fbgpu_ctx* c) try {
    if (!c) return fail(FBGPU_E_INVALID, "null ctx");
    if (c->comm && nccl_load()) { cudaSetDevice(c->device); cudaDeviceSynchronize(); g_nccl.CommDestroy(c->comm); }
    c->comm = nullptr; c->n_ranks = 1; c->rank = 0;
    return 0;
} FBGPU_CATCH

// ---- fused peer-memory reduce: mailbox exchange through CUDA IPC (one process per GPU)
extern "C" int fbgpu_comm_p2p_handle(fbgpu_ctx* c, uint8_t out[64]) try {
    if (!c || !out) return fail(FBGPU_E_INVALID, "null argument");
    USE_DEVICE(c);
    if (!c->mbox) { CUDA_TRY(cudaMalloc((void**)&c->mbox, sizeof(Mailbox))); CUDA_TRY(cudaMemset(c->mbox, 0, sizeof(Mailbox))); }
    cudaIpcMemHandle_t h;
    CUDA_TRY(cudaIpcGetMemHandle(&h, c->mbox));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    memcpy(out, &h, 64);
    return FBGPU_OK;
} FBGPU_CATCH
extern "C" int fbgpu_comm_p2p_open(fbgpu_ctx* c, int32_t n_ranks, int32_t rank, const uint8_t* handles /* n_ranks x 64 */) try {
    if (!c || !handles || n_ranks < 1 || n_ranks > kMaxRanks || rank < 0 || rank >= n_ranks) return fail(FBGPU_E_INVALID, "bad argument");
    if (!c->mbox) return fail(FBGPU_E_COMM, "call fbgpu_comm_p2p_handle first");
    USE_DEVICE(c);
    std::lock_guard<std::mutex> lk(c->coll_mu);
    c->p2p = false;
    for (int p = 0; p < kMaxRanks; p++) {                        // re-open after a membership change: drop the old mappings first
        if (c->peers[p] && c->peers[p] != c->mbox && !c->peers_local) cudaIpcCloseMemHandle(c->peers[p]);
        c->peers[p] = nullptr;
    }
    c->peers_local = false;
    for (int p = 0; p < n_ranks; p++) {
        if (p == rank) { c->peers[p] = c->mbox; continue; }
        cudaIpcMemHandle_t h; memcpy(&h, handles + (size_t)p * 64, 64);
        void* ptr = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) return fail(FBGPU_E_COMM, "cudaIpcOpenMemHandle(rank %d) failed: %s", p, cudaGetErrorString(e));
        c->peers[p] = (Mailbox*)ptr;
    }
    if (c->d_peers.ensure(sizeof(Mailbox*) * kMaxRanks)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemcpy(c->d_peers.p, c->peers, sizeof(Mailbox*) * kMaxRanks, cudaMemcpyHostToDevice));
    // a re-open restarts the exchange numbering: flags left by the previous membership must not satisfy a new wait.  Every rank
    // clears its OWN mailbox here; the caller separates fbgpu_comm_p2p_open from the first query by a barrier (all ranks opened).
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemset(c->mbox, 0, sizeof(Mailbox)));
    CUDA_TRY(cudaDeviceSynchronize());
    c->n_ranks = n_ranks; c->rank = rank; c->epoch = 0; c->p2p = true;
    return FBGPU_OK;
} FBGPU_CATCH

extern "C" int fbgpu_comm_p2p_disable(fbgpu_ctx* c) try {      // back to the NCCL merge (mappings stay open; harmless)
    if (!c) return fail(FBGPU_E_INVALID, "null ctx");
    std::lock_guard<std::mutex> lk(c->coll_mu);
    c->p2p = false;
    return FBGPU_OK;
} FBGPU_CATCH

// ---- store inspection (tests): the container the kernels would find for (index, field, view, shard, row, slot), located by
// the same resolve() the kernels inline, over the host copies of the tables of an FBGPU_DEVICE_NONE context
extern "C" int fbgpu_debug_container(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, uint64_t shard, uint64_t row, int32_t slot,
                                     uint32_t* out_type, uint32_t* out_card, uint32_t* out_runs, uint8_t* out_payload, uint64_t cap, uint64_t* out_len) try {
    if (!c || !out_type || !out_card || !out_runs || !out_len || slot < 0 || slot >= kSlotsPerRow) return fail(FBGPU_E_INVALID, "bad argument");
    if (!c->inspect_only) return fail(FBGPU_E_INVALID, "fbgpu_debug_container needs a context created with FBGPU_DEVICE_NONE");
    std::unique_lock<std::shared_mutex> lk(c->store_mu);
    if (c->meta_dirty) { int rc = commit_locked(c); if (rc) return rc; }
    StoreRef st{};
    st.views = c->t_views.data(); st.shardmap = c->t_flat.data(); st.frags = c->h_frags.data(); st.rows = c->h_rows.data(); st.descs = c->h_descs.data();
    st.payload = c->staging.p; st.rowtab = c->t_rowtab.data(); st.n_views = (uint32_t)c->t_views.size();
    uint32_t fv = index == 0xffffffffu ? field : view_id_locked(c, ViewKey{ index, field, view }, false);   // (index ~0: `field` is a view slot of a compiled program)
    Resolved r = resolve(st, fv, shard, row, slot);
    *out_type = 0; *out_card = 0; *out_runs = 0; *out_len = 0;
    if (r.ptr == nullptr) return FBGPU_OK;                      // absent
    *out_type = r.typ; *out_card = r.card; *out_runs = r.cnt;
    const uint64_t bytes = r.typ == kArray ? (((uint64_t)r.card * 2 + 15) & ~15ull) : r.typ == kBitmap ? 8192 : (((uint64_t)r.cnt * 4 + 15) & ~15ull);   // padded, as stored
    *out_len = bytes;
    if (bytes > cap || !out_payload) return fail(FBGPU_E_NOSPACE, "payload needs %llu bytes", (unsigned long long)bytes);
    if ((const uint8_t*)r.ptr + bytes > c->staging.p + c->staging.len) return fail(FBGPU_E_INVALID, "descriptor points outside the payload arena");
    memcpy(out_payload, r.ptr, bytes);
    return FBGPU_OK;
} FBGPU_CATCH

// the device program the library would run for a post-order fbgpu_op program (records of 16 bytes: u8 op, 3 pad, u32 view slot, u64 row)
extern "C" int fbgpu_debug_compile(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint8_t* out, int32_t cap_ops, int32_t* out_n, int32_t* out_depth) try {
    if (!c || !out_n || !out_depth) return fail(FBGPU_E_INVALID, "null argument");
    std::shared_lock<std::shared_mutex> lk(c->store_mu);
    std::vector<DevOp> prog; int depth = 1;
    int rc = compile_program(c, index, ops, n_ops, prog, depth); if (rc) return rc;
    *out_n = (int32_t)prog.size(); *out_depth = depth;
    if ((int32_t)prog.size() > cap_ops || (!out && !prog.empty())) return fail(FBGPU_E_NOSPACE, "program has %zu ops", prog.size());
    static_assert(sizeof(DevOp) == 16, "DevOp layout");
    if (!prog.empty()) memcpy(out, prog.data(), prog.size() * sizeof(DevOp));
    return FBGPU_OK;
} FBGPU_CATCH

extern "C" int fbgpu_get_counters(fbgpu_ctx* c, fbgpu_counters* out) try {
    if (!c || !out) return fail(FBGPU_E_INVALID, "null argument");
    std::lock_guard<std::mutex> lk(c->cnt_mu);
    *out = c->counters;
    out->pair_kernel_queries = (uint32_t)c->counters_pair_launches.load();
    return 0;
} FBGPU_CATCH
extern "C" void* fbgpu_stream(fbgpu_ctx* c) { return c && !c->wss.empty() ? (void*)c->wss[0]->stream : nullptr; }

// algorithmic-bytes accounting for bench / DESIGN (SURVEY §8d): payload bytes + 16 B descriptor of every
// container of the given rows over the given shards
extern "C" int fbgpu_rows_payload_bytes(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, const uint64_t* row_ids, int32_t n_rows,
                                        const uint64_t* shards, int64_t n_shards, uint64_t* out_payload, uint64_t* out_containers) try {
    if (!c || !out_payload || !out_containers) return fail(FBGPU_E_INVALID, "null argument");
    std::shared_lock<std::shared_mutex> lk(c->store_mu);
    uint64_t pay = 0, nc = 0;
    uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    if (fv != kNoView) for (int64_t s = 0; s < n_shards; s++) {
        const auto& sm = c->shardmaps[fv];
        if (shards[s] >= sm.size() || sm[shards[s]] < 0) continue;
        const HostFrag& f = c->frags[sm[shards[s]]];
        for (uint32_t k = 0; k < f.n_rows; k++) {
            const RowEnt& e = c->h_rows[f.row_off + k];
            bool want = row_ids == nullptr;
            for (int32_t r = 0; !want && r < n_rows; r++) want = row_ids[r] == e.row;
            if (!want) continue;
            int n = __builtin_popcount(e.mask);
            for (int q = 0; q < n; q++) { const ContDesc& d = c->h_descs[e.first_desc + q]; pay += d.typ == kArray ? 2ull * d.card : d.typ == kBitmap ? 8192 : 4ull * d.cnt; nc++; }
        }
    }
    *out_payload = pay; *out_containers = nc;
    return 0;
} FBGPU_CATCH

// ------------------------------------------------------------------ all GPUs of one process behind one handle
#include "node.h"
