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
    CUDA_TRY(cudaFuncSetAttribute(row_count_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPairWarps * 8192));
    CUDA_TRY(cudaFuncSetAttribute(row_count_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPairWarps * 8192));
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
        for (DevBuf* b : { &w->d_in, &w->d_counts, &w->d_bitmaps, &w->d_info, &w->d_emit_units, &w->d_emit, &w->d_rows, &w->d_aux }) b->release();
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
// query cannot leave the query reading host mirrors that are newer than what is in HBM.
static int lock_committed(fbgpu_ctx* c, std::shared_lock<std::shared_mutex>& lk) {
    if (c->inspect_only) return fail(FBGPU_E_CUDA, "this context was created with FBGPU_DEVICE_NONE: it holds no device and answers no query");
    for (;;) {
        lk = std::shared_lock<std::shared_mutex>(c->store_mu);
        if (!c->meta_dirty && c->staging.empty()) return 0;
        lk.unlock();
        int rc = fbgpu_commit(c); if (rc) return rc;
    }
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

// the usual shard list is a contiguous range (a node's share, SURVEY §8e): kernels then compute the shard id instead of loading it
static bool contiguous_shards(const uint64_t* shards, int64_t n) {
    for (int64_t i = 1; i < n; i++) if (shards[i] != shards[0] + (uint64_t)i) return false;
    return n > 0;
}

// ------------------------------------------------------------------ Count
// collective == false: this context's shards only — no cross-GPU merge (fbgpu_any's early exit must not desynchronise the ranks)
static int count_impl(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards,
                      uint64_t* out_total, uint64_t* out_per_shard, bool collective) {
    if (!c || !out_total || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    USE_DEVICE(c);
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    std::vector<DevOp> prog; int depth = 1;
    rc = compile_program(c, index, ops, n_ops, prog, depth); if (rc) return rc;
    WsLease lease(c); Workspace* w = lease.w;
    const DevOp* d_prog; const uint64_t* d_shards;
    rc = upload_inputs(w, prog, shards, n_shards, &d_prog, &d_shards); if (rc) return rc;
    // layout of d_counts: [total][per-shard counts ...][ticket][reduced result][error]
    const size_t nper = out_per_shard ? (size_t)n_shards : 0, nc = 1 + nper + 3;
    if (w->d_counts.ensure(nc * 8)) return FBGPU_E_NOMEM;
    if (w->h_out.ensure(nc * 8)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, nc * 8, w->stream));
    unsigned long long* d_total = (unsigned long long*)w->d_counts.p;
    unsigned long long* d_per = out_per_shard ? d_total + 1 : nullptr;
    long long n_units = (long long)n_shards * kSlotsPerRow;
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
            pair_count_kernel<<<(unsigned)grid, kPcWarps * 32, kPcWarps * 8192, w->stream>>>(store_ref(c), pa->fv, pa->row, pb->fv, pb->row, nullptr, nullptr, n_units,
                contiguous_shards(shards, n_shards) ? nullptr : d_shards, n_shards ? shards[0] : 0, n_units, d_total, d_per, nullptr, fr);
            CUDA_TRY(cudaGetLastError());
        } else {
            EvalOut eo{ d_total, d_per, nullptr, nullptr, fr };
            rc = launch_eval(c, w, prog, d_prog, depth, d_shards, n_units, eo); if (rc) return rc;
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
        lease.ok = true;                     // the stream is drained; the exchange state is not: the caller re-opens the peers
        return fail(FBGPU_E_COMM, "rank %d did not publish its count for exchange %llu in time (peer dead, or the ranks issued their collective queries in different orders); re-open with fbgpu_comm_p2p_open",
                    (int)((uint64_t*)w->h_out.p)[1 + nper + 2] - 1, (unsigned long long)fr.epoch);
    }
    *out_total = p2p ? ((uint64_t*)w->h_out.p)[1 + nper + 1] : ((uint64_t*)w->h_out.p)[0];
    if (out_per_shard) memcpy(out_per_shard, (uint64_t*)w->h_out.p + 1, (size_t)n_shards * 8);
    float ms = 0; cudaEventElapsedTime(&ms, w->ev0, w->ev1);
    bump(c, (n_units > 0 || p2p) ? 1 : 0, ms);
    lease.ok = true;
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
    USE_DEVICE(c);
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    std::vector<DevOp> prog; int depth = 1;
    rc = compile_program(c, index, ops, n_ops, prog, depth); if (rc) return rc;
    // Row.Merge concatenates disjoint shard segments (row.go:202); emit in ascending shard order
    std::vector<uint64_t> sorted(shards, shards + n_shards);
    std::sort(sorted.begin(), sorted.end());
    sorted.erase(std::unique(sorted.begin(), sorted.end()), sorted.end());
    n_shards = (int64_t)sorted.size();
    WsLease lease(c); Workspace* w = lease.w;
    const DevOp* d_prog; const uint64_t* d_shards;
    rc = upload_inputs(w, prog, sorted.data(), n_shards, &d_prog, &d_shards); if (rc) return rc;
    long long n_units = (long long)n_shards * kSlotsPerRow;
    struct OutCont { uint64_t key; uint16_t typ; uint32_t n; uint64_t size; uint32_t batch; uint64_t src_off; };
    std::vector<OutCont> conts; std::vector<std::vector<uint8_t>> batch_bufs;   // one host copy of the emitted payloads per batch
    // a single batch (<= 1024 shards, the usual call) needs no such copy: its payloads are assembled straight from the pinned
    // D2H landing buffer, which stays leased until this function returns
    const bool single_batch = n_units <= c->unit_batch;
    const uint8_t* single_src = nullptr;
    uint64_t total_count = 0; uint64_t launches = 0; float ms_total = 0;
    for (long long u0 = 0; u0 < n_units; u0 += c->unit_batch) {
        long long nu = std::min(c->unit_batch, n_units - u0);
        if (w->d_bitmaps.ensure((size_t)nu * 8192)) return FBGPU_E_NOMEM;
        if (w->d_info.ensure((size_t)nu * 8)) return FBGPU_E_NOMEM;
        if (w->h_out.ensure((size_t)nu * 8)) return FBGPU_E_NOMEM;
        EvalOut eo{ nullptr, nullptr, (uint4*)w->d_bitmaps.p, (uint2*)w->d_info.p, FuseReduce{} };
        CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
        rc = launch_eval(c, w, prog, d_prog, depth, d_shards + u0 / kSlotsPerRow, nu, eo); if (rc) return rc;
        launches++;
        CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_info.p, (size_t)nu * 8, cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        // optimize(): roaring.go:3412-3426
        std::vector<EmitUnit> emits; uint64_t off = 0; size_t first = conts.size();
        const uint2* info = (const uint2*)w->h_out.p;
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
            if (w->d_emit_units.ensure(emits.size() * sizeof(EmitUnit))) return FBGPU_E_NOMEM;
            if (w->d_emit.ensure(off)) return FBGPU_E_NOMEM;
            if (w->h_in.ensure(std::max<size_t>(emits.size() * sizeof(EmitUnit), off))) return FBGPU_E_NOMEM;
            memcpy(w->h_in.p, emits.data(), emits.size() * sizeof(EmitUnit));
            CUDA_TRY(cudaMemcpyAsync(w->d_emit_units.p, w->h_in.p, emits.size() * sizeof(EmitUnit), cudaMemcpyHostToDevice, w->stream));
            int grid = (int)std::min<size_t>(emits.size(), (size_t)c->sm_count * 8);
            canon_emit_kernel<<<grid, kEmitThreads, 0, w->stream>>>((const uint4*)w->d_bitmaps.p, (const EmitUnit*)w->d_emit_units.p, (int)emits.size(), (uint8_t*)w->d_emit.p);
            CUDA_TRY(cudaGetLastError()); launches++;
            CUDA_TRY(cudaStreamSynchronize(w->stream));   // h_in is reused as the D2H landing buffer below
            CUDA_TRY(cudaMemcpyAsync(w->h_in.p, w->d_emit.p, off, cudaMemcpyDeviceToHost, w->stream));
            CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
            CUDA_TRY(cudaStreamSynchronize(w->stream));
            if (single_batch) { single_src = (const uint8_t*)w->h_in.p; batch_bufs.emplace_back(); }
            else batch_bufs.emplace_back((uint8_t*)w->h_in.p, (uint8_t*)w->h_in.p + off);
            float ms = 0; cudaEventElapsedTime(&ms, w->ev0, w->ev1); ms_total += ms;
        }
    }
    bump(c, launches, ms_total);
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
    lease.ok = true;
    return FBGPU_OK;
} FBGPU_CATCH

// ------------------------------------------------------------------ Columns (Row.Columns(): ascending ids, with executeLimitCall's window) / Extract
// shared body: evaluate the row into per-unit bitmaps, cut the [offset, offset+limit) window into per-unit rank ranges, expand
// the column ids on the device and — for Extract — gather the BSI planes of `fv_vals` for exactly those columns
static int columns_impl(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards,
                        uint64_t offset, int64_t limit, bool want_vals, uint32_t fv_vals, int depth_vals,
                        uint64_t* out_cols, int64_t* out_vals, uint64_t cap, uint64_t* out_n, uint64_t* out_total) {
    std::vector<DevOp> prog; int depth = 1;
    int rc = compile_program(c, index, ops, n_ops, prog, depth); if (rc) return rc;
    std::vector<uint64_t> sorted(shards, shards + n_shards);
    std::sort(sorted.begin(), sorted.end());
    sorted.erase(std::unique(sorted.begin(), sorted.end()), sorted.end());
    n_shards = (int64_t)sorted.size();
    WsLease lease(c); Workspace* w = lease.w;
    const DevOp* d_prog; const uint64_t* d_shards;
    rc = upload_inputs(w, prog, sorted.data(), n_shards, &d_prog, &d_shards); if (rc) return rc;
    const long long n_units = (long long)n_shards * kSlotsPerRow;
    const uint64_t win_end = limit < 0 ? ~0ull : (offset + (uint64_t)limit < offset ? ~0ull : offset + (uint64_t)limit);
    uint64_t seen = 0, written = 0, launches = 0; float ms_total = 0;
    for (long long u0 = 0; u0 < n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, n_units - u0);
        if (w->d_bitmaps.ensure((size_t)nu * 8192) || w->d_info.ensure((size_t)nu * 8) || w->h_out.ensure((size_t)nu * 8)) return FBGPU_E_NOMEM;
        EvalOut eo{ nullptr, nullptr, (uint4*)w->d_bitmaps.p, (uint2*)w->d_info.p, FuseReduce{} };
        CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
        rc = launch_eval(c, w, prog, d_prog, depth, d_shards + u0 / kSlotsPerRow, nu, eo); if (rc) return rc;
        launches++;
        CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_info.p, (size_t)nu * 8, cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        const uint2* info = (const uint2*)w->h_out.p;
        std::vector<ColUnit> units; uint64_t batch_out = 0;
        for (long long u = 0; u < nu; u++) {
            const uint64_t N = info[u].x;
            if (!N) continue;
            const uint64_t lo = std::max(seen, offset), hi = std::min(seen + N, win_end);    // the unit's ranks are [seen, seen + N)
            if (hi > lo) {
                ColUnit cu{};
                cu.out_off = batch_out; cu.unit = (uint32_t)u; cu.first = (uint32_t)(lo - seen); cu.last = (uint32_t)(hi - seen);
                cu.col_base = (sorted[(u0 + u) / kSlotsPerRow] << 20) + (uint64_t)((u0 + u) % kSlotsPerRow) * 65536ull;
                units.push_back(cu);
                batch_out += hi - lo;
            }
            seen += N;
        }
        if (batch_out && written + batch_out <= cap) {
            const size_t ub = units.size() * sizeof(ColUnit), ob = batch_out * 8 * (want_vals ? 2 : 1);
            if (w->d_emit_units.ensure(ub) || w->d_emit.ensure(ob) || w->h_in.ensure(std::max<size_t>(ub, ob))) return FBGPU_E_NOMEM;
            memcpy(w->h_in.p, units.data(), ub);
            CUDA_TRY(cudaMemcpyAsync(w->d_emit_units.p, w->h_in.p, ub, cudaMemcpyHostToDevice, w->stream));
            const int grid = (int)std::min<size_t>(units.size(), (size_t)c->sm_count * 8);
            unsigned long long* d_cols = (unsigned long long*)w->d_emit.p; unsigned long long* d_vals = d_cols + batch_out;
            columns_emit_kernel<<<grid, kEmitThreads, 0, w->stream>>>((const uint4*)w->d_bitmaps.p, (const ColUnit*)w->d_emit_units.p, (int)units.size(), d_cols);
            CUDA_TRY(cudaGetLastError()); launches++;
            if (want_vals) {
                CUDA_TRY(cudaMemsetAsync(d_vals, 0, batch_out * 8, w->stream));
                extract_values_kernel<<<grid, kExtractThreads, 0, w->stream>>>(store_ref(c), fv_vals, depth_vals, (const uint4*)w->d_bitmaps.p, (const ColUnit*)w->d_emit_units.p, (int)units.size(), d_vals);
                CUDA_TRY(cudaGetLastError()); launches++;
            }
            CUDA_TRY(cudaStreamSynchronize(w->stream));   // h_in is reused as the D2H landing buffer below
            CUDA_TRY(cudaMemcpyAsync(w->h_in.p, w->d_emit.p, ob, cudaMemcpyDeviceToHost, w->stream));
            CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
            CUDA_TRY(cudaStreamSynchronize(w->stream));
            memcpy(out_cols + written, w->h_in.p, batch_out * 8);
            if (want_vals) {                               // sign-magnitude (bit 63 = sign row) -> int64
                const uint64_t* raw = (const uint64_t*)w->h_in.p + batch_out;
                for (uint64_t i = 0; i < batch_out; i++) { const int64_t m = (int64_t)(raw[i] & ~(1ull << 63)); out_vals[written + i] = (raw[i] >> 63) ? -m : m; }
            }
            float ms = 0; cudaEventElapsedTime(&ms, w->ev0, w->ev1); ms_total += ms;
        }
        written += batch_out;                              // (past cap: counted, not written)
    }
    bump(c, launches, ms_total);
    *out_n = written;
    if (out_total) *out_total = seen;
    lease.ok = true;
    if (written > cap) return fail(FBGPU_E_NOSPACE, "output needs room for %llu columns", (unsigned long long)written);
    return FBGPU_OK;
}

extern "C" int fbgpu_columns(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards,
                             uint64_t offset, int64_t limit, uint64_t* out_cols, uint64_t cap, uint64_t* out_n, uint64_t* out_total) try {
    if (!c || !out_n || n_shards < 0 || (n_shards && !shards) || (cap && !out_cols)) return fail(FBGPU_E_INVALID, "null argument");
    USE_DEVICE(c);
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    return columns_impl(c, index, ops, n_ops, shards, n_shards, offset, limit, false, 0, 0, out_cols, nullptr, cap, out_n, out_total);
} FBGPU_CATCH

extern "C" int fbgpu_extract(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                             const uint64_t* shards, int64_t n_shards, uint64_t offset, int64_t limit,
                             uint64_t* out_cols, int64_t* out_vals, uint64_t cap, uint64_t* out_n, uint64_t* out_total) try {
    if (!c || !out_n || n_shards < 0 || (n_shards && !shards) || (cap && (!out_cols || !out_vals)) || n_ops < 0 || (n_ops && !ops)) return fail(FBGPU_E_INVALID, "null argument");
    if (bit_depth < 0 || bit_depth > 63) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..63", bit_depth);
    USE_DEVICE(c);
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    // the row: <filter> ∩ exists (bsiExistsBit, row 0 of the bsig_ view; fragment.go:44)
    std::vector<fbgpu_op> full(ops, ops + n_ops);
    fbgpu_op ex{}; ex.opcode = FBGPU_OP_ROW; ex.field = field; ex.view = view; ex.a = 0;
    full.push_back(ex);
    if (n_ops) { fbgpu_op in{}; in.opcode = FBGPU_OP_INTERSECT; in.argc = 2; full.push_back(in); }
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    return columns_impl(c, index, full.data(), (int32_t)full.size(), shards, n_shards, offset, limit, true, fv, bit_depth, out_cols, out_vals, cap, out_n, out_total);
} FBGPU_CATCH

// ------------------------------------------------------------------ BSI Min / Max (one pass over the planes)
extern "C" int fbgpu_bsi_minmax(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                                const uint64_t* shards, int64_t n_shards, int32_t want_max, int64_t* out_val, uint64_t* out_count) try {
    if (!c || !out_val || !out_count || n_shards < 0 || (n_shards && !shards) || n_ops < 0 || (n_ops && !ops)) return fail(FBGPU_E_INVALID, "null argument");
    if (bit_depth < 0 || bit_depth > 63) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..63", bit_depth);
    USE_DEVICE(c);
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    *out_val = 0; *out_count = 0;
    std::vector<fbgpu_op> full(ops, ops + n_ops);           // consider = <filter> ∩ exists (fragment.go:753-757)
    fbgpu_op ex{}; ex.opcode = FBGPU_OP_ROW; ex.field = field; ex.view = view; ex.a = 0;
    full.push_back(ex);
    if (n_ops) { fbgpu_op in{}; in.opcode = FBGPU_OP_INTERSECT; in.argc = 2; full.push_back(in); }
    std::vector<DevOp> prog; int depth = 1;
    rc = compile_program(c, index, full.data(), (int32_t)full.size(), prog, depth); if (rc) return rc;
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    WsLease lease(c); Workspace* w = lease.w;
    const DevOp* d_prog; const uint64_t* d_shards;
    rc = upload_inputs(w, prog, shards, n_shards, &d_prog, &d_shards); if (rc) return rc;
    const long long n_units = (long long)n_shards * kSlotsPerRow;
    bool have = false; int64_t best = 0; uint64_t best_n = 0; uint64_t launches = 0; float ms_total = 0;
    for (long long u0 = 0; u0 < n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, n_units - u0);
        if (w->d_bitmaps.ensure((size_t)nu * 8192) || w->d_counts.ensure((size_t)nu * sizeof(MinMaxUnit)) || w->h_out.ensure((size_t)nu * sizeof(MinMaxUnit))) return FBGPU_E_NOMEM;
        EvalOut eo{ nullptr, nullptr, (uint4*)w->d_bitmaps.p, nullptr, FuseReduce{} };
        CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
        rc = launch_eval(c, w, prog, d_prog, depth, d_shards + u0 / kSlotsPerRow, nu, eo); if (rc) return rc;
        const long long grid = std::min<long long>(nu, (long long)c->sm_count * 8);
        bsi_minmax_kernel<<<(unsigned)grid, kEvalThreads, 0, w->stream>>>(store_ref(c), fv, bit_depth, (const uint4*)w->d_bitmaps.p, d_shards + u0 / kSlotsPerRow, nu, want_max ? 1 : 0, (MinMaxUnit*)w->d_counts.p);
        CUDA_TRY(cudaGetLastError()); launches += 2;
        CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
        CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, (size_t)nu * sizeof(MinMaxUnit), cudaMemcpyDeviceToHost, w->stream));
        CUDA_TRY(cudaStreamSynchronize(w->stream));
        const MinMaxUnit* r = (const MinMaxUnit*)w->h_out.p;
        for (long long u = 0; u < nu; u++) {                // ValCount.Larger / Smaller: keep the extreme, add the counts of equal values
            if (!r[u].cnt) continue;
            if (!have || (want_max ? r[u].val > best : r[u].val < best)) { have = true; best = r[u].val; best_n = r[u].cnt; }
            else if (r[u].val == best) best_n += r[u].cnt;
        }
        float ms = 0; cudaEventElapsedTime(&ms, w->ev0, w->ev1); ms_total += ms;
    }
    bump(c, launches, ms_total);
    if (have) { *out_val = best; *out_count = best_n; }
    lease.ok = true;
    return FBGPU_OK;
} FBGPU_CATCH

extern "C" int fbgpu_bsi_sum(fbgpu_ctx* c, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                             const uint64_t* shards, int64_t n_shards, int64_t* out_sum, uint64_t* out_count) try {
    if (!c || !out_sum || !out_count || n_shards < 0 || (n_shards && !shards) || n_ops < 0 || (n_ops && !ops)) return fail(FBGPU_E_INVALID, "null argument");
    if (bit_depth < 0 || bit_depth > 63) return fail(FBGPU_E_INVALID, "bit depth %d outside 0..63", bit_depth);
    USE_DEVICE(c);
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    *out_sum = 0; *out_count = 0;
    std::vector<fbgpu_op> full(ops, ops + n_ops);
    fbgpu_op ex{}; ex.opcode = FBGPU_OP_ROW; ex.field = field; ex.view = view; ex.a = 0;
    full.push_back(ex);
    if (n_ops) { fbgpu_op in{}; in.opcode = FBGPU_OP_INTERSECT; in.argc = 2; full.push_back(in); }
    std::vector<DevOp> prog; int depth = 1;
    rc = compile_program(c, index, full.data(), (int32_t)full.size(), prog, depth); if (rc) return rc;
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    WsLease lease(c); Workspace* w = lease.w;
    const DevOp* d_prog; const uint64_t* d_shards;
    rc = upload_inputs(w, prog, shards, n_shards, &d_prog, &d_shards); if (rc) return rc;
    const long long n_units = (long long)n_shards * kSlotsPerRow;
    const size_t n_acc = 1 + 2 * (size_t)bit_depth;
    if (w->d_counts.ensure(n_acc * 8) || w->h_out.ensure(n_acc * 8)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, n_acc * 8, w->stream));
    uint64_t launches = 0;
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    for (long long u0 = 0; u0 < n_units; u0 += c->unit_batch) {
        const long long nu = std::min(c->unit_batch, n_units - u0);
        if (w->d_bitmaps.ensure((size_t)nu * 8192)) return FBGPU_E_NOMEM;
        EvalOut eo{ nullptr, nullptr, (uint4*)w->d_bitmaps.p, nullptr, FuseReduce{} };
        rc = launch_eval(c, w, prog, d_prog, depth, d_shards + u0 / kSlotsPerRow, nu, eo); if (rc) return rc;
        const long long grid = std::min<long long>(nu, (long long)c->sm_count * 8);
        bsi_sum_kernel<<<(unsigned)grid, kEvalThreads, 0, w->stream>>>(store_ref(c), fv, bit_depth, (const uint4*)w->d_bitmaps.p, d_shards + u0 / kSlotsPerRow, nu, (unsigned long long*)w->d_counts.p);
        CUDA_TRY(cudaGetLastError()); launches += 2;
    }
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, n_acc * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    const uint64_t* acc = (const uint64_t*)w->h_out.p;
    uint64_t sum = 0;                                       // wrapping, like the reference's int64 arithmetic
    for (int i = 0; i < bit_depth; i++) sum += (acc[1 + 2 * i] - acc[2 + 2 * i]) << i;
    *out_sum = (int64_t)sum; *out_count = acc[0];
    float ms = 0; cudaEventElapsedTime(&ms, w->ev0, w->ev1);
    bump(c, launches, ms);
    lease.ok = true;
    return FBGPU_OK;
} FBGPU_CATCH

// ------------------------------------------------------------------ per-row counts (TopK / TopN ids)
// evaluates `filter` for shards [s0, s0+ns) into w->d_bitmaps (16 bitmaps per shard)
static int eval_filter_batch(fbgpu_ctx* c, Workspace* w, const std::vector<DevOp>& prog, int depth, const DevOp* d_prog, const uint64_t* d_shards, int64_t ns) {
    if (w->d_bitmaps.ensure((size_t)ns * kSlotsPerRow * 8192)) return FBGPU_E_NOMEM;
    EvalOut eo{ nullptr, nullptr, (uint4*)w->d_bitmaps.p, nullptr, FuseReduce{} };
    return launch_eval(c, w, prog, d_prog, depth, d_shards, ns * kSlotsPerRow, eo);
}

static int row_counts_impl(fbgpu_ctx* c, uint32_t index, uint32_t fv, const std::vector<uint64_t>& rows, const fbgpu_op* filter, int32_t n_filter_ops,
                           const uint64_t* shards, int64_t n_shards, std::vector<uint64_t>& counts, bool reduce = true, bool per_shard = false) {
    counts.assign(rows.size() * (per_shard ? (size_t)n_shards : 1), 0);
    if (rows.empty()) return 0;
    std::vector<DevOp> prog; int depth = 1; int rc;
    bool have_filter = filter && n_filter_ops > 0;
    if (have_filter) { rc = compile_program(c, index, filter, n_filter_ops, prog, depth); if (rc) return rc; }
    WsLease lease(c); Workspace* w = lease.w;
    const DevOp* d_prog; const uint64_t* d_shards;
    rc = upload_inputs(w, prog, shards, n_shards, &d_prog, &d_shards); if (rc) return rc;
    size_t nr = rows.size();
    const size_t n_out = counts.size();                     // nr, or n_shards x nr (per_shard: one row of the matrix per listed shard)
    if (w->d_rows.ensure(nr * 8) || w->d_counts.ensure(n_out * 8) || w->h_out.ensure(n_out * 8)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemcpyAsync(w->d_rows.p, rows.data(), nr * 8, cudaMemcpyHostToDevice, w->stream));
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, n_out * 8, w->stream));
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    uint64_t launches = 0;
    const int64_t batch = have_filter ? c->unit_batch / kSlotsPerRow : n_shards;
    for (int64_t s0 = 0; s0 < n_shards; s0 += batch) {
        int64_t ns = std::min(batch, n_shards - s0);
        if (have_filter) { rc = eval_filter_batch(c, w, prog, depth, d_prog, d_shards + s0, ns); if (rc) return rc; launches++; }
        long long tasks = (long long)ns * (long long)nr;
        long long grid = std::min<long long>((tasks + kPairWarps - 1) / kPairWarps, (long long)c->sm_count * 3);
        if (per_shard)
            row_count_kernel<true><<<(unsigned)grid, kPairWarps * 32, kPairWarps * 8192, w->stream>>>(store_ref(c), fv, (const uint64_t*)w->d_rows.p, (int)nr, d_shards + s0, ns,
                have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, (unsigned long long*)w->d_counts.p + (size_t)s0 * nr);
        else
            row_count_kernel<false><<<(unsigned)grid, kPairWarps * 32, kPairWarps * 8192, w->stream>>>(store_ref(c), fv, (const uint64_t*)w->d_rows.p, (int)nr, d_shards + s0, ns,
                have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, (unsigned long long*)w->d_counts.p);
        CUDA_TRY(cudaGetLastError()); launches++;
    }
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    // every rank must bring the same row list to the collective: only the explicit-ids form is all-reduced (fbgpu.h)
    if (reduce && !per_shard) { rc = allreduce_u64(c, w, w->d_counts.p, nr); if (rc) return rc; }
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, n_out * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    memcpy(counts.data(), w->h_out.p, n_out * 8);
    float ms = 0; cudaEventElapsedTime(&ms, w->ev0, w->ev1);
    bump(c, launches, ms);
    lease.ok = true;
    return 0;
}

extern "C" int fbgpu_row_counts(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, const uint64_t* row_ids, int32_t n_rows,
                                const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards,
                                uint64_t* out_row_ids, uint64_t* out_counts, int32_t cap, int32_t* out_n) try {
    if (!c || !out_counts || n_shards < 0 || (n_shards && !shards) || n_rows < 0) return fail(FBGPU_E_INVALID, "null argument");
    USE_DEVICE(c);
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
    std::vector<uint64_t> rows, counts;
    if (row_ids) rows.assign(row_ids, row_ids + n_rows);
    else {
        // fragment.rows() (fragment.go:2465-2486): distinct row ids present in the listed shards
        if (fv != kNoView) for (int64_t s = 0; s < n_shards; s++) {
            const auto& sm = c->shardmaps[fv];
            if (shards[s] >= sm.size() || sm[shards[s]] < 0) continue;
            const HostFrag& f = c->frags[sm[shards[s]]];
            for (uint32_t k = 0; k < f.n_rows; k++) rows.push_back(c->h_rows[f.row_off + k].row);
        }
        std::sort(rows.begin(), rows.end()); rows.erase(std::unique(rows.begin(), rows.end()), rows.end());
    }
    rc = row_counts_impl(c, index, fv, rows, filter, n_filter_ops, shards, n_shards, counts, row_ids != nullptr); if (rc) return rc;
    if (row_ids) {
        if (cap < n_rows) return fail(FBGPU_E_NOSPACE, "cap %d < n_rows %d", cap, n_rows);
        for (int32_t i = 0; i < n_rows; i++) { out_counts[i] = counts[i]; if (out_row_ids) out_row_ids[i] = rows[i]; }
        if (out_n) *out_n = n_rows;
        return FBGPU_OK;
    }
    std::vector<size_t> order;
    for (size_t i = 0; i < rows.size(); i++) if (counts[i]) order.push_back(i);
    std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return counts[a] != counts[b] ? counts[a] > counts[b] : rows[a] < rows[b]; });
    // all rows with a non-zero count, or none: a silently truncated list would make Rows() / the TopN candidate set incomplete
    // (ADVICE r1).  *out_n always receives the number of rows there are, so the caller can size its buffers and call again.
    if (out_n) *out_n = (int32_t)std::min<size_t>(order.size(), (size_t)INT32_MAX);
    if (order.size() > (size_t)std::max(cap, 0)) return fail(FBGPU_E_NOSPACE, "%zu rows have a non-zero count, cap is %d", order.size(), cap);
    for (size_t i = 0; i < order.size(); i++) { if (out_row_ids) out_row_ids[i] = rows[order[i]]; out_counts[i] = counts[order[i]]; }
    return FBGPU_OK;
} FBGPU_CATCH

// per-shard counts of explicit rows: out_counts[s * n_rows + i] = |Row(row_ids[i]) [∩ filter]| in shards[s]
extern "C" int fbgpu_row_counts_per_shard(fbgpu_ctx* c, uint32_t index, uint32_t field, uint32_t view, const uint64_t* row_ids, int32_t n_rows,
                                          const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    if (!c || !out_counts || !row_ids || n_rows < 0 || n_shards < 0 || (n_shards && !shards) || n_filter_ops < 0 || (n_filter_ops && !filter)) return fail(FBGPU_E_INVALID, "null argument");
    if (n_rows == 0 || n_shards == 0) return FBGPU_OK;
    USE_DEVICE(c);
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    const uint32_t fv = view_id_locked(c, ViewKey{ index, field, view }, false);
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
    WsLease lease(c); Workspace* w = lease.w;
    std::vector<DevOp> none; const DevOp* d_prog; const uint64_t* d_shards;
    rc = upload_inputs(w, none, shards, n_shards, &d_prog, &d_shards); if (rc) return rc;
    size_t np = (size_t)n_pairs;
    if (w->d_rows.ensure(np * 16) || w->d_counts.ensure(np * 8) || w->h_out.ensure(np * 16)) return FBGPU_E_NOMEM;
    memcpy(w->h_out.p, rows_a, np * 8); memcpy((uint8_t*)w->h_out.p + np * 8, rows_b, np * 8);
    CUDA_TRY(cudaMemcpyAsync(w->d_rows.p, w->h_out.p, np * 16, cudaMemcpyHostToDevice, w->stream));
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, np * 8, w->stream));
    const long long upp = (long long)n_shards * kSlotsPerRow, n_units = upp * n_pairs;
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    if (n_units > 0) {
        long long grid = std::min<long long>((n_units + kPcWarps - 1) / kPcWarps, (long long)c->sm_count * c->pair_ctas_per_sm);
        pair_count_kernel<<<(unsigned)grid, kPcWarps * 32, kPcWarps * 8192, w->stream>>>(store_ref(c), fa, 0, fb, 0, (const uint64_t*)w->d_rows.p, (const uint64_t*)w->d_rows.p + np,
            upp, contiguous_shards(shards, n_shards) ? nullptr : d_shards, n_shards ? shards[0] : 0, n_units, nullptr, nullptr, (unsigned long long*)w->d_counts.p, FuseReduce{});
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    rc = allreduce_u64(c, w, w->d_counts.p, np); if (rc) return rc;
    CUDA_TRY(cudaStreamSynchronize(w->stream));      // h_out was the H2D source; now reuse it as the D2H landing buffer
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, np * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    memcpy(out_counts, w->h_out.p, np * 8);
    float ms = 0; cudaEventElapsedTime(&ms, w->ev0, w->ev1);
    bump(c, n_units > 0 ? 1 : 0, ms);
    lease.ok = true;
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
    WsLease lease(c); Workspace* w = lease.w;
    std::vector<DevOp> none; const DevOp* d_prog; const uint64_t* d_shards;
    rc = upload_inputs(w, none, shards, n_shards, &d_prog, &d_shards); if (rc) return rc;
    if (w->d_counts.ensure(16 * 8) || w->h_out.ensure(16 * 8)) return FBGPU_E_NOMEM;
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, 16 * 8, w->stream));
    const long long n_units = (long long)n_shards * kSlotsPerRow;
    const long long grid = std::min<long long>((n_units + 255) / 256, (long long)c->sm_count * 4);
    pair_types_kernel<<<(unsigned)grid, 256, 0, w->stream>>>(store_ref(c), fa, row_a, fb, row_b, d_shards, n_units, (unsigned long long*)w->d_counts.p);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, 16 * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    memcpy(out_hist, w->h_out.p, 16 * 8);
    bump(c, 1, 0.f);
    lease.ok = true;
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
    std::vector<DevOp> prog; int depth = 1; int rc;
    bool have_filter = !filter.empty();
    if (have_filter) { rc = compile_program(c, index, filter.data(), (int)filter.size(), prog, depth); if (rc) return rc; }
    WsLease lease(c); Workspace* w = lease.w;
    const DevOp* d_prog; const uint64_t* d_shards;
    rc = upload_inputs(w, prog, shards, n_shards, &d_prog, &d_shards); if (rc) return rc;
    size_t ncnt = (size_t)nA * nB;
    if (w->d_rows.ensure((size_t)(nA + nB) * 8) || w->d_counts.ensure(ncnt * 8) || w->h_out.ensure(ncnt * 8)) return FBGPU_E_NOMEM;
    std::vector<uint64_t> rr(rowsA, rowsA + nA); rr.insert(rr.end(), rowsB, rowsB + nB);
    CUDA_TRY(cudaMemcpyAsync(w->d_rows.p, rr.data(), rr.size() * 8, cudaMemcpyHostToDevice, w->stream));
    CUDA_TRY(cudaMemsetAsync(w->d_counts.p, 0, ncnt * 8, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));   // rr is a local
    CUDA_TRY(cudaEventRecord(w->ev0, w->stream));
    uint64_t launches = 0, fb_units = 0, all_units = 0;
    const int64_t batch = have_filter ? c->unit_batch / kSlotsPerRow : n_shards;
    const size_t smem = kGbSlots * 4 + 8192;
    for (int64_t s0 = 0; s0 < n_shards; s0 += batch) {
        int64_t ns = std::min(batch, n_shards - s0);
        if (have_filter) { rc = eval_filter_batch(c, w, prog, depth, d_prog, d_shards + s0, ns); if (rc) return rc; launches++; }
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
                CUDA_TRY(cudaGetLastError()); launches++;
                CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
                CUDA_TRY(cudaMemcpyAsync(h_fb, d_fb, 4, cudaMemcpyDeviceToHost, w->stream));
                CUDA_TRY(cudaStreamSynchronize(w->stream));
                const unsigned int n_fb = *h_fb;
                if (n_fb) {
                    groupby_kernel<<<(unsigned)std::min<long long>(n_fb, grid), kGbThreads, smem, w->stream>>>(store_ref(c), fvA, d_ra, na, fvB, (const uint64_t*)w->d_rows.p + nA, nB,
                        d_shards + s0, units, have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, d_cnt, d_fb);
                    CUDA_TRY(cudaGetLastError()); launches++;
                    CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
                }
                fb_units += n_fb; all_units += (uint64_t)units;
            }
        } else {
            groupby_kernel<<<(unsigned)grid, kGbThreads, smem, w->stream>>>(store_ref(c), fvA, (const uint64_t*)w->d_rows.p, nA, fvB, (const uint64_t*)w->d_rows.p + nA, nB,
                d_shards + s0, units, have_filter ? (const uint4*)w->d_bitmaps.p : nullptr, (unsigned long long*)w->d_counts.p, nullptr);
            CUDA_TRY(cudaGetLastError()); launches++;
            CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
        }
    }
    if (n_shards <= 0) CUDA_TRY(cudaEventRecord(w->ev1, w->stream));
    rc = allreduce_u64(c, w, w->d_counts.p, ncnt); if (rc) return rc;
    CUDA_TRY(cudaMemcpyAsync(w->h_out.p, w->d_counts.p, ncnt * 8, cudaMemcpyDeviceToHost, w->stream));
    CUDA_TRY(cudaStreamSynchronize(w->stream));
    memcpy(out, w->h_out.p, ncnt * 8);
    float ms = 0; cudaEventElapsedTime(&ms, w->ev0, w->ev1);
    bump(c, launches, ms);
    { std::lock_guard<std::mutex> lk2(c->cnt_mu); c->counters.groupby_units += all_units; c->counters.groupby_fallback_units += fb_units; }
    lease.ok = true;
    return 0;
}

// n-field GroupBy: peel the leading field on the host, folding Row(f0=r) into the filter (groupByIterator keeps
// the same prefix intersections per level, executor.go:8829-8835,8861-8867)
static int groupby_rec(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views, int nf, const uint64_t* const* rows, const int32_t* n_rows,
                       std::vector<fbgpu_op> filter, const uint64_t* shards, int64_t n_shards, uint64_t* out) {
    if (nf == 1) {
        uint32_t fv = view_id_locked(c, ViewKey{ index, fields[0], views[0] }, false);
        std::vector<uint64_t> r(rows[0], rows[0] + n_rows[0]), counts;
        int rc = row_counts_impl(c, index, fv, r, filter.empty() ? nullptr : filter.data(), (int)filter.size(), shards, n_shards, counts); if (rc) return rc;
        memcpy(out, counts.data(), counts.size() * 8);
        return 0;
    }
    if (nf == 2) {
        uint32_t fa = view_id_locked(c, ViewKey{ index, fields[0], views[0] }, false), fb = view_id_locked(c, ViewKey{ index, fields[1], views[1] }, false);
        return groupby2(c, index, fa, rows[0], n_rows[0], fb, rows[1], n_rows[1], filter, shards, n_shards, out);
    }
    size_t sub = 1; for (int i = 1; i < nf; i++) sub *= (size_t)n_rows[i];
    for (int r = 0; r < n_rows[0]; r++) {
        std::vector<fbgpu_op> f2 = filter;
        fbgpu_op ro{}; ro.opcode = FBGPU_OP_ROW; ro.field = fields[0]; ro.view = views[0]; ro.a = rows[0][r];
        f2.push_back(ro);
        if (!filter.empty()) { fbgpu_op in{}; in.opcode = FBGPU_OP_INTERSECT; in.argc = 2; f2.push_back(in); }
        int rc = groupby_rec(c, index, fields + 1, views + 1, nf - 1, rows + 1, n_rows + 1, f2, shards, n_shards, out + (size_t)r * sub); if (rc) return rc;
    }
    return 0;
}

extern "C" int fbgpu_groupby(fbgpu_ctx* c, uint32_t index, const uint32_t* fields, const uint32_t* views, int32_t n_fields, const uint64_t* row_ids_flat, const int32_t* n_rows,
                             const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    if (!c || !fields || !views || !row_ids_flat || !n_rows || !out_counts || n_fields < 1 || n_fields > 8 || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "bad argument");
    USE_DEVICE(c);
    std::shared_lock<std::shared_mutex> lk;
    int rc = lock_committed(c, lk); if (rc) return rc;
    std::vector<const uint64_t*> rows(n_fields); const uint64_t* p = row_ids_flat; size_t total = 1;
    for (int i = 0; i < n_fields; i++) { if (n_rows[i] < 0 || n_rows[i] > 65535) return fail(FBGPU_E_INVALID, "n_rows[%d]=%d out of range", i, n_rows[i]); rows[i] = p; p += n_rows[i]; total *= (size_t)n_rows[i]; }
    memset(out_counts, 0, total * 8);
    if (total == 0) return 0;
    // executor.go:8769-8772: the kernels treat a shard with a missing fragment as contributing nothing; for the
    // row_counts path (n_fields == 1) a missing fragment naturally yields zeros.  For n_fields >= 3 the peeled
    // fields enter through the filter, which is empty on shards without that fragment.
    std::vector<fbgpu_op> f(filter, filter + (filter ? n_filter_ops : 0));
    return groupby_rec(c, index, fields, views, n_fields, rows.data(), n_rows, f, shards, n_shards, out_counts);
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
