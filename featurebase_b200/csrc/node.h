// fbgpu_node: every GPU of ONE process behind one handle (SURVEY §8(b) `fbgpu_init(device_ordinals, n)`).
//
// FeatureBase is a single process per node whose goroutines call the executor concurrently (executor.go:6449-6533 mapReduce,
// :6742-6812 mapperLocal).  A node owns one fbgpu_ctx per device; a shard lives on exactly one device
// (owner = (shard / shard_block) % n_devices: contiguous blocks of shards per GPU, SURVEY §8(e)).  One C call fans a query
// out to the devices that own the listed shards — each on its own worker thread, stream and workspace — and merges the
// per-device results (u64 sums: Count executor.go:5880, Pairs.Add cache.go:464, mergeGroupCounts executor.go:3728) in the
// calling thread.  Every query has its own buffers on every device, so concurrent callers can never mix their results and
// there is no cross-device wait that a failing device could hang: an error on any device is the call's error.
// (The one-process-per-GPU form with NCCL / the fused mailbox exchange stays available for launchers that want it.)
//
// Included at the end of fbgpu.cu (single translation unit).
#pragma once

struct NodeWorker {                       // one OS thread draining a FIFO of closures
    std::thread th; std::mutex mu; std::condition_variable cv; std::deque<std::function<void()>> q; bool quit = false;
    NodeWorker() { th = std::thread([this] { run(); }); }
    ~NodeWorker() { { std::lock_guard<std::mutex> lk(mu); quit = true; } cv.notify_all(); th.join(); }
    void post(std::function<void()> f) { { std::lock_guard<std::mutex> lk(mu); q.push_back(std::move(f)); } cv.notify_one(); }
    void run() {
        for (;;) {
            std::function<void()> f;
            { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [this] { return quit || !q.empty(); }); if (q.empty()) return; f = std::move(q.front()); q.pop_front(); }
            f();
        }
    }
};

struct fbgpu_node {
    std::vector<fbgpu_ctx*> ctx;                                   // one per device slot (the same ordinal may appear twice: tests)
    std::vector<std::vector<std::unique_ptr<NodeWorker>>> workers; // [device][k]
    std::vector<std::atomic<uint32_t>> rr;                         // round-robin cursor per device
    uint64_t shard_block = 1;
    explicit fbgpu_node(size_t n) : rr(n) {}
    int owner(uint64_t shard) const { return (int)((shard / shard_block) % ctx.size()); }
};

constexpr int kNodeWorkersPerDevice = 4;   // = workspaces per context: that many queries of one device can overlap

// completion latch of one fan-out
struct NodeJoin {
    std::mutex mu; std::condition_variable cv; int pending = 0; int rc = 0; std::string err;
    void done(int r, const char* msg) { std::lock_guard<std::mutex> lk(mu); if (r && !rc) { rc = r; err = msg ? msg : ""; } if (--pending == 0) cv.notify_all(); }
    int wait() { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [this] { return pending == 0; }); if (rc) g_err = err; return rc; }
};

// shard list split by owner, order kept; pos[d][k] = index of the k-th shard of device d in the caller's list
struct NodeSplit { std::vector<std::vector<uint64_t>> shards; std::vector<std::vector<int64_t>> pos; };
static NodeSplit node_split(const fbgpu_node* n, const uint64_t* shards, int64_t n_shards) {
    NodeSplit s; s.shards.resize(n->ctx.size()); s.pos.resize(n->ctx.size());
    for (int64_t i = 0; i < n_shards; i++) { int d = n->owner(shards[i]); s.shards[d].push_back(shards[i]); s.pos[d].push_back(i); }
    return s;
}

// runs fn(device) on a worker of every device in `devs` and waits; the first error wins
template <class F>
static int node_fan_out(fbgpu_node* n, const std::vector<int>& devs, F fn) {
    NodeJoin j; j.pending = (int)devs.size();
    if (devs.empty()) return 0;
    for (int d : devs) {
        NodeWorker* w = n->workers[d][n->rr[d].fetch_add(1, std::memory_order_relaxed) % n->workers[d].size()].get();
        w->post([&j, &fn, d] { int rc; try { rc = fn(d); } catch (...) { rc = fail(FBGPU_E_INVALID, "internal error on a node worker"); } j.done(rc, rc ? g_err.c_str() : nullptr); });
    }
    return j.wait();
}
static std::vector<int> node_all(const fbgpu_node* n) { std::vector<int> v(n->ctx.size()); for (size_t i = 0; i < v.size(); i++) v[i] = (int)i; return v; }
static std::vector<int> node_owners(const NodeSplit& s) { std::vector<int> v; for (size_t d = 0; d < s.shards.size(); d++) if (!s.shards[d].empty()) v.push_back((int)d); return v; }

extern "C" int fbgpu_node_init(const int32_t* device_ordinals, int32_t n_devices, uint64_t shard_block, fbgpu_node** out) try {
    if (!device_ordinals || !out || n_devices < 1 || n_devices > 64 || shard_block < 1) return fail(FBGPU_E_INVALID, "bad argument");
    auto node = std::make_unique<fbgpu_node>((size_t)n_devices);
    node->shard_block = shard_block;
    struct Guard { fbgpu_node* n; ~Guard() { if (n) for (fbgpu_ctx* c : n->ctx) fbgpu_shutdown(c); } } guard{ node.get() };
    for (int i = 0; i < n_devices; i++) {
        fbgpu_ctx* c = nullptr;
        int rc = fbgpu_init(device_ordinals[i], &c); if (rc) return rc;
        node->ctx.push_back(c);
    }
    node->workers.resize((size_t)n_devices);
    for (int i = 0; i < n_devices; i++) for (int k = 0; k < kNodeWorkersPerDevice; k++) node->workers[i].push_back(std::make_unique<NodeWorker>());
    guard.n = nullptr;
    *out = node.release();
    return FBGPU_OK;
} FBGPU_CATCH

extern "C" void fbgpu_node_shutdown(fbgpu_node* n) {
    if (!n) return;
    n->workers.clear();                                   // joins the threads (queues are empty: every call waits for its jobs)
    for (fbgpu_ctx* c : n->ctx) fbgpu_shutdown(c);
    delete n;
}
extern "C" int32_t fbgpu_node_devices(const fbgpu_node* n) { return n ? (int32_t)n->ctx.size() : 0; }
extern "C" int32_t fbgpu_node_owner(const fbgpu_node* n, uint64_t shard) { return n ? n->owner(shard) : -1; }
extern "C" fbgpu_ctx* fbgpu_node_ctx(fbgpu_node* n, int32_t i) { return n && i >= 0 && (size_t)i < n->ctx.size() ? n->ctx[(size_t)i] : nullptr; }

// ---- residency: routed by the owner of the shard
extern "C" int fbgpu_node_load_fragment(fbgpu_node* n, uint32_t index, uint32_t field, uint32_t view, uint64_t shard, const uint8_t* roaring, uint64_t nbytes) try {
    if (!n) return fail(FBGPU_E_INVALID, "null node");
    return fbgpu_load_fragment(n->ctx[(size_t)n->owner(shard)], index, field, view, shard, roaring, nbytes);
} FBGPU_CATCH
extern "C" int fbgpu_node_load_fragments(fbgpu_node* n, uint32_t index, uint32_t field, uint32_t view, const uint64_t* shards, int64_t cnt,
                                         const uint8_t* buf, const uint64_t* offsets) try {
    if (!n || !shards || !buf || !offsets || cnt < 0) return fail(FBGPU_E_INVALID, "null argument");
    // per device: the sub-list of fragments with their own offsets table into the caller's buffer (no payload copy here); a
    // device's batch is all-or-nothing (StoreTxn), devices load concurrently
    const NodeSplit sp = node_split(n, shards, cnt);
    return node_fan_out(n, node_owners(sp), [&](int d) -> int {
        // fragments of one device are generally not adjacent in buf: load them as runs of adjacent fragments
        const auto& ix = sp.pos[(size_t)d];
        for (size_t a = 0; a < ix.size();) {
            size_t b = a + 1; while (b < ix.size() && ix[b] == ix[b - 1] + 1) b++;
            std::vector<uint64_t> off(b - a + 1); const uint64_t base = offsets[ix[a]];
            for (size_t k = a; k <= b; k++) off[k - a] = (k < b ? offsets[ix[k]] : offsets[ix[b - 1] + 1]) - base;
            int rc = fbgpu_load_fragments(n->ctx[(size_t)d], index, field, view, sp.shards[(size_t)d].data() + a, (int64_t)(b - a), buf + base, off.data()); if (rc) return rc;
            a = b;
        }
        return 0;
    });
} FBGPU_CATCH
extern "C" int fbgpu_node_load_rbf_dir(fbgpu_node* n, uint32_t index, uint64_t shard, const char* dir, const char* const* names, const uint32_t* fields,
                                       const uint32_t* views, int32_t n_names, int32_t* out_loaded) try {
    if (!n) return fail(FBGPU_E_INVALID, "null node");
    return fbgpu_load_rbf_dir(n->ctx[(size_t)n->owner(shard)], index, shard, dir, names, fields, views, n_names, out_loaded);
} FBGPU_CATCH
extern "C" int fbgpu_node_drop_fragment(fbgpu_node* n, uint32_t index, uint32_t field, uint32_t view, uint64_t shard) try {
    if (!n) return fail(FBGPU_E_INVALID, "null node");
    return fbgpu_drop_fragment(n->ctx[(size_t)n->owner(shard)], index, field, view, shard);
} FBGPU_CATCH
extern "C" int fbgpu_node_apply_containers(fbgpu_node* n, uint32_t index, uint32_t field, uint32_t view, uint64_t shard, const uint8_t* roaring, uint64_t nbytes,
                                           const uint64_t* removed_keys, int64_t n_removed) try {
    if (!n) return fail(FBGPU_E_INVALID, "null node");
    return fbgpu_apply_containers(n->ctx[(size_t)n->owner(shard)], index, field, view, shard, roaring, nbytes, removed_keys, n_removed);
} FBGPU_CATCH
extern "C" int fbgpu_node_commit(fbgpu_node* n) try {
    if (!n) return fail(FBGPU_E_INVALID, "null node");
    return node_fan_out(n, node_all(n), [&](int d) { return fbgpu_commit(n->ctx[(size_t)d]); });
} FBGPU_CATCH
extern "C" int fbgpu_node_get_stats(fbgpu_node* n, fbgpu_stats* out) try {
    if (!n || !out) return fail(FBGPU_E_INVALID, "null argument");
    memset(out, 0, sizeof *out);
    for (fbgpu_ctx* c : n->ctx) {
        fbgpu_stats s{}; int rc = fbgpu_get_stats(c, &s); if (rc) return rc;
        out->fragments += s.fragments; out->containers += s.containers; out->array_containers += s.array_containers; out->bitmap_containers += s.bitmap_containers;
        out->run_containers += s.run_containers; out->payload_bytes += s.payload_bytes; out->device_bytes += s.device_bytes; out->dead_bytes += s.dead_bytes;
        out->full_commits += s.full_commits; out->patch_commits += s.patch_commits;
    }
    return FBGPU_OK;
} FBGPU_CATCH

// ---- queries
extern "C" int fbgpu_node_count(fbgpu_node* n, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards,
                                uint64_t* out_total, uint64_t* out_per_shard) try {
    if (!n || !out_total || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    NodeSplit sp = node_split(n, shards, n_shards);
    std::vector<int> devs = node_owners(sp);
    if (devs.empty()) devs.push_back(0);                 // no shard listed: still validate the program (Intersect() etc. must error)
    std::vector<uint64_t> tot(n->ctx.size(), 0); std::vector<std::vector<uint64_t>> per(n->ctx.size());
    int rc = node_fan_out(n, devs, [&](int d) {
        auto& s = sp.shards[(size_t)d];
        if (out_per_shard) per[(size_t)d].assign(s.size(), 0);
        return fbgpu_count(n->ctx[(size_t)d], index, ops, n_ops, s.data(), (int64_t)s.size(), &tot[(size_t)d], out_per_shard ? per[(size_t)d].data() : nullptr);
    });
    if (rc) return rc;
    uint64_t t = 0; for (int d : devs) t += tot[(size_t)d];
    *out_total = t;
    if (out_per_shard) for (int d : devs) for (size_t k = 0; k < sp.pos[(size_t)d].size(); k++) out_per_shard[sp.pos[(size_t)d][k]] = per[(size_t)d][k];
    return FBGPU_OK;
} FBGPU_CATCH

// Row.Any(): every device walks its own shards with the early exit; the answers are OR-ed
extern "C" int fbgpu_node_any(fbgpu_node* n, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards, int32_t* out_any) try {
    if (!n || !out_any || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    NodeSplit sp = node_split(n, shards, n_shards);
    std::vector<int> devs = node_owners(sp);
    if (devs.empty()) devs.push_back(0);
    std::vector<int32_t> any(n->ctx.size(), 0);
    int rc = node_fan_out(n, devs, [&](int d) { auto& s = sp.shards[(size_t)d]; return fbgpu_any(n->ctx[(size_t)d], index, ops, n_ops, s.data(), (int64_t)s.size(), &any[(size_t)d]); });
    if (rc) return rc;
    *out_any = 0; for (int d : devs) *out_any |= any[(size_t)d];
    return FBGPU_OK;
} FBGPU_CATCH

// runs fn(ctx, its shards, part) on every device that owns listed shards, each filling a zeroed u64 vector of `len`, and writes
// their element-wise sum to out (overwritten; zeros when no shard is listed)
template <class F>
static int node_sum(fbgpu_node* n, const uint64_t* shards, int64_t n_shards, size_t len, uint64_t* out, F fn) {
    const NodeSplit sp = node_split(n, shards, n_shards);
    const std::vector<int> devs = node_owners(sp);
    std::vector<std::vector<uint64_t>> part(n->ctx.size());
    int rc = node_fan_out(n, devs, [&](int d) {
        part[(size_t)d].assign(len, 0);
        return fn(n->ctx[(size_t)d], sp.shards[(size_t)d], part[(size_t)d].data());
    });
    if (rc) return rc;
    memset(out, 0, len * 8);
    for (int d : devs) { const uint64_t* p = part[(size_t)d].data(); for (size_t i = 0; i < len; i++) out[i] += p[i]; }
    return FBGPU_OK;
}

extern "C" int fbgpu_node_count_pairs(fbgpu_node* n, uint32_t index, uint32_t field_a, uint32_t view_a, const uint64_t* rows_a,
                                      uint32_t field_b, uint32_t view_b, const uint64_t* rows_b, int32_t n_pairs,
                                      const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    if (!n || !rows_a || !rows_b || !out_counts || n_pairs < 0 || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    return node_sum(n, shards, n_shards, (size_t)n_pairs, out_counts, [&](fbgpu_ctx* c, const std::vector<uint64_t>& s, uint64_t* part) {
        return fbgpu_count_pairs(c, index, field_a, view_a, rows_a, field_b, view_b, rows_b, n_pairs, s.data(), (int64_t)s.size(), part);
    });
} FBGPU_CATCH

// explicit-ids form only (TopN(ids=...), TopK candidates): the reduced vector is what Pairs.Add produces (cache.go:464)
extern "C" int fbgpu_node_row_counts(fbgpu_node* n, uint32_t index, uint32_t field, uint32_t view, const uint64_t* row_ids, int32_t n_rows,
                                     const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    if (!n || !row_ids || !out_counts || n_rows < 0 || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    return node_sum(n, shards, n_shards, (size_t)n_rows, out_counts, [&](fbgpu_ctx* c, const std::vector<uint64_t>& s, uint64_t* part) {
        int32_t got = 0;
        return fbgpu_row_counts(c, index, field, view, row_ids, n_rows, filter, n_filter_ops, s.data(), (int64_t)s.size(), nullptr, part, n_rows, &got);
    });
} FBGPU_CATCH

extern "C" int fbgpu_node_row_counts_views(fbgpu_node* n, uint32_t index, uint32_t field, const uint32_t* views, int32_t n_views, const uint64_t* row_ids, int32_t n_rows,
                                           const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    int rc = row_counts_views_args(n, views, n_views, n_rows, filter, n_filter_ops, shards, n_shards, out_counts); if (rc) return rc;
    if (!row_ids) return fail(FBGPU_E_INVALID, "bad argument");
    return node_sum(n, shards, n_shards, (size_t)n_rows, out_counts, [&](fbgpu_ctx* c, const std::vector<uint64_t>& s, uint64_t* part) {
        int32_t got = 0;
        return fbgpu_row_counts_views(c, index, field, views, n_views, row_ids, n_rows, filter, n_filter_ops, s.data(), (int64_t)s.size(), nullptr, part, n_rows, &got);
    });
} FBGPU_CATCH

// Explicit ids: the devices' vectors are summed.  All rows: each device's (row, total) list, merged by row id with the totals
// summed, then sorted under fbgpu_row_counts' NOSPACE contract.  Both are exact: a shard lives on one device, and a row's total is
// a sum over shards.
extern "C" int fbgpu_node_topn_cutoffs(fbgpu_node* n, uint32_t index, uint32_t field, uint32_t view, const uint64_t* row_ids, int32_t n_rows,
                                       const fbgpu_op* src, int32_t n_src_ops, uint64_t min_threshold, uint32_t tanimoto_threshold,
                                       const uint64_t* shards, int64_t n_shards, uint64_t* out_row_ids, uint64_t* out_counts, int32_t cap, int32_t* out_n) try {
    int rc = topn_cutoffs_args(n, n_rows, src, n_src_ops, tanimoto_threshold, shards, n_shards, out_counts); if (rc) return rc;
    if (row_ids) {
        rc = node_sum(n, shards, n_shards, (size_t)n_rows, out_counts, [&](fbgpu_ctx* c, const std::vector<uint64_t>& s, uint64_t* part) {
            int32_t got = 0;
            return fbgpu_topn_cutoffs(c, index, field, view, row_ids, n_rows, src, n_src_ops, min_threshold, tanimoto_threshold, s.data(), (int64_t)s.size(),
                                      nullptr, part, n_rows, &got);
        });
        if (rc) return rc;
        if (cap < n_rows) return fail(FBGPU_E_NOSPACE, "cap %d < n_rows %d", cap, n_rows);
        if (out_row_ids) memcpy(out_row_ids, row_ids, (size_t)n_rows * 8);
        if (out_n) *out_n = n_rows;
        return FBGPU_OK;
    }
    const NodeSplit sp = node_split(n, shards, n_shards);
    const std::vector<int> devs = node_owners(sp);
    std::vector<std::vector<uint64_t>> rows(n->ctx.size()), totals(n->ctx.size());
    rc = node_fan_out(n, devs, [&](int d) {
        fbgpu_ctx* c = n->ctx[(size_t)d];
        const auto& s = sp.shards[(size_t)d];
        std::shared_lock<std::shared_mutex> lk;
        int r = begin_query(c, lk); if (r) return r;
        const std::vector<uint32_t> fvs{ view_id_locked(c, ViewKey{ index, field, view }, false) };
        const RcCut cut{ nullptr, min_threshold, tanimoto_threshold };
        return row_counts_run(c, index, fvs, nullptr, 0, src, n_src_ops, s.data(), (int64_t)s.size(), rows[(size_t)d], totals[(size_t)d], &cut);
    });
    if (rc) return rc;
    std::vector<std::pair<uint64_t, uint64_t>> all;
    for (int d : devs) for (size_t i = 0; i < rows[(size_t)d].size(); i++) all.emplace_back(rows[(size_t)d][i], totals[(size_t)d][i]);
    std::sort(all.begin(), all.end());
    std::vector<uint64_t> mr, mt;
    for (const auto& p : all) {
        if (!mr.empty() && mr.back() == p.first) mt.back() += p.second;
        else { mr.push_back(p.first); mt.push_back(p.second); }
    }
    return write_sorted_rows(mr, mt, out_row_ids, out_counts, cap, out_n);
} FBGPU_CATCH

// a GroupBy node form once its arguments but n_rows are checked: n_rows checked before the fan-out, the request run on each device
// over its own shards, the tensors added up (mergeGroupCounts executor.go:3728; Sum's [counts | sums]: wrapping int64 sums add as u64)
static int node_groupby(fbgpu_node* n, uint32_t index, const GbRequest& q, uint64_t* out_counts, int64_t* out_sums = nullptr) {
    int rc = q.check_rows(); if (rc) return rc;
    const size_t cells = q.cells();
    std::vector<uint64_t> both(out_sums ? q.out_len() : 0);
    rc = node_sum(n, q.shards, q.n_shards, q.out_len(), out_sums ? both.data() : out_counts, [&](fbgpu_ctx* c, const std::vector<uint64_t>& s, uint64_t* part) {
        GbRequest qd = q; qd.shards = s.data(); qd.n_shards = (int64_t)s.size();
        return groupby_run(c, index, qd, part, out_sums ? (int64_t*)(part + cells) : nullptr);
    });
    if (rc || !out_sums) return rc;
    memcpy(out_counts, both.data(), cells * 8);
    memcpy(out_sums, both.data() + cells, cells * 8);
    return FBGPU_OK;
}

extern "C" int fbgpu_node_groupby_views(fbgpu_node* n, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                        const uint64_t* row_ids_flat, const int32_t* n_rows, const fbgpu_op* filter, int32_t n_filter_ops,
                                        const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    int rc = groupby_views_args(n, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, filter, n_filter_ops, shards, n_shards, out_counts);
    if (rc) return rc;
    return node_groupby(n, index, GbRequest{ gb_set_dims(fields, views_flat, n_views, n_fields, row_ids_flat, n_rows), {}, GvAgg::kCount, {},
                                             filter, n_filter_ops, shards, n_shards }, out_counts);
} FBGPU_CATCH

extern "C" int fbgpu_node_groupby(fbgpu_node* n, uint32_t index, const uint32_t* fields, const uint32_t* views, int32_t n_fields, const uint64_t* row_ids_flat,
                                  const int32_t* n_rows, const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    int rc = groupby_args(n, fields, views, n_fields, row_ids_flat, n_rows, filter, n_filter_ops, shards, n_shards, out_counts); if (rc) return rc;
    return node_groupby(n, index, GbRequest{ gb_set_dims(fields, views, nullptr, n_fields, row_ids_flat, n_rows), {}, GvAgg::kCount, {},
                                             filter, n_filter_ops, shards, n_shards }, out_counts);
} FBGPU_CATCH

extern "C" int fbgpu_node_groupby_values(fbgpu_node* n, uint32_t index, const uint32_t* fields, const uint32_t* views, int32_t n_fields, const uint64_t* row_ids_flat,
                                         const int32_t* n_rows, uint32_t vfield, uint32_t vview, int32_t bit_depth, const int64_t* values, int32_t n_values,
                                         const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    int rc = groupby_values_args(n, fields, views, n_fields, row_ids_flat, n_rows, bit_depth, values, n_values, filter, n_filter_ops, shards, n_shards, out_counts);
    if (rc) return rc;
    return node_groupby(n, index, GbRequest{ gb_set_dims(fields, views, nullptr, n_fields, row_ids_flat, n_rows), gb_int_dims(&vfield, &vview, &bit_depth, 1, values, &n_values),
                                             GvAgg::kCount, {}, filter, n_filter_ops, shards, n_shards }, out_counts);
} FBGPU_CATCH

extern "C" int fbgpu_node_groupby_mixed(fbgpu_node* n, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                        const uint64_t* row_ids_flat, const int32_t* n_rows, const uint32_t* vfields, const uint32_t* vviews, const int32_t* bit_depths,
                                        int32_t n_ints, const int64_t* values_flat, const int32_t* n_values, const fbgpu_op* filter, int32_t n_filter_ops,
                                        const uint64_t* shards, int64_t n_shards, uint64_t* out_counts) try {
    int rc = groupby_mixed_args(n, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, vfields, vviews, bit_depths, n_ints, values_flat, n_values,
                                filter, n_filter_ops, shards, n_shards, out_counts);
    if (rc) return rc;
    return node_groupby(n, index, GbRequest{ gb_set_dims(fields, views_flat, n_views, n_fields, row_ids_flat, n_rows),
                                             gb_int_dims(vfields, vviews, bit_depths, n_ints, values_flat, n_values), GvAgg::kCount, {},
                                             filter, n_filter_ops, shards, n_shards }, out_counts);
} FBGPU_CATCH

extern "C" int fbgpu_node_groupby_sum(fbgpu_node* n, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                      const uint64_t* row_ids_flat, const int32_t* n_rows, const uint32_t* vfields, const uint32_t* vviews, const int32_t* bit_depths,
                                      int32_t n_ints, const int64_t* values_flat, const int32_t* n_values, uint32_t afield, uint32_t aview, int32_t a_depth,
                                      const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t* out_counts, int64_t* out_sums) try {
    int rc = groupby_agg_args(n, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, vfields, vviews, bit_depths, n_ints, values_flat, n_values,
                              out_sums, "a_depth", a_depth, filter, n_filter_ops, shards, n_shards, out_counts);
    if (rc) return rc;
    return node_groupby(n, index, GbRequest{ gb_set_dims(fields, views_flat, n_views, n_fields, row_ids_flat, n_rows),
                                             gb_int_dims(vfields, vviews, bit_depths, n_ints, values_flat, n_values), GvAgg::kSum, GvInt{ afield, aview, a_depth, nullptr, 0 },
                                             filter, n_filter_ops, shards, n_shards }, out_counts, out_sums);
} FBGPU_CATCH

// a sparse GroupBy node form (kCount or kSum): every device lists its own shards' cells with the same window; the lists merge by
// cell with the counts and the (wrapping) sums added, and the window is cut after the merge.  Exact: a cell is listed on a device
// exactly when its count there is non-zero, so a cell among the first K non-empty cells of the node is among the first K of every
// device where it is non-empty, as for the all-rows branch of fbgpu_node_topn_cutoffs.
static int node_groupby_sparse(fbgpu_node* n, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                               const uint64_t* row_ids_flat, const int32_t* n_rows, SpRequest q,
                               uint64_t* out_cells, uint64_t* out_counts, int64_t* out_sums, uint64_t cap, uint64_t* out_n) {
    int rc = groupby_sparse_args(n, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows, q, out_cells, out_counts, out_sums, cap, out_n);
    if (rc) return rc;
    q.dims = gb_set_dims(fields, views_flat, n_views, n_fields, row_ids_flat, n_rows);
    const NodeSplit sp = node_split(n, q.shards, q.n_shards);
    std::vector<int> devs = node_owners(sp);
    if (devs.empty()) devs.push_back(0);                 // no shard listed: still validate the filter
    std::vector<SpResult> part(n->ctx.size());
    rc = node_fan_out(n, devs, [&](int d) {
        fbgpu_ctx* c = n->ctx[(size_t)d];
        SpRequest qd = q; qd.shards = sp.shards[(size_t)d].data(); qd.n_shards = (int64_t)sp.shards[(size_t)d].size();
        std::shared_lock<std::shared_mutex> lk;
        int r = begin_query(c, lk); if (r) return r;
        return groupby_sparse_run(c, index, qd, part[(size_t)d]);
    });
    if (rc) return rc;
    std::vector<std::pair<uint64_t, std::pair<uint64_t, uint64_t>>> all;          // (cell, (count, sum))
    for (int d : devs) {
        const SpResult& p = part[(size_t)d];
        for (size_t i = 0; i < p.cells.size(); i++) all.push_back({ p.cells[i], { p.counts[i], p.sums.empty() ? 0 : (uint64_t)p.sums[i] } });
    }
    std::sort(all.begin(), all.end(), [](const auto& x, const auto& y) { return x.first < y.first; });
    SpResult m;
    for (const auto& e : all) {
        if (!m.cells.empty() && m.cells.back() == e.first) { m.counts.back() += e.second.first; m.sums.back() = (int64_t)((uint64_t)m.sums.back() + e.second.second); }
        else { m.cells.push_back(e.first); m.counts.push_back(e.second.first); m.sums.push_back((int64_t)e.second.second); }
    }
    const size_t keep = q.limit >= 0 ? std::min(m.cells.size(), (size_t)q.limit) : m.cells.size();
    m.cells.resize(keep); m.counts.resize(keep); m.sums.resize(q.agg == GvAgg::kSum ? keep : 0);
    return write_cells(m, out_cells, out_counts, out_sums, cap, out_n);
}

// fbgpu_groupby_sparse over a node: the non-empty cells from `start` on, at most `limit` of them, merged over the devices
extern "C" int fbgpu_node_groupby_sparse(fbgpu_node* n, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views, int32_t n_fields,
                                         const uint64_t* row_ids_flat, const int32_t* n_rows, const fbgpu_op* filter, int32_t n_filter_ops,
                                         const uint64_t* shards, int64_t n_shards, uint64_t start, int64_t limit,
                                         uint64_t* out_cells, uint64_t* out_counts, uint64_t cap, uint64_t* out_n) try {
    return node_groupby_sparse(n, index, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows,
                               SpRequest{ {}, GvAgg::kCount, {}, filter, n_filter_ops, shards, n_shards, start, ~0ull, limit },
                               out_cells, out_counts, nullptr, cap, out_n);
} FBGPU_CATCH

// fbgpu_groupby_sparse_sum over a node: the same window, with each listed cell's wrapping sum merged beside its count
extern "C" int fbgpu_node_groupby_sparse_sum(fbgpu_node* n, uint32_t index, const uint32_t* fields, const uint32_t* views_flat, const int32_t* n_views,
                                             int32_t n_fields, const uint64_t* row_ids_flat, const int32_t* n_rows, uint32_t afield, uint32_t aview, int32_t a_depth,
                                             const fbgpu_op* filter, int32_t n_filter_ops, const uint64_t* shards, int64_t n_shards, uint64_t start, int64_t limit,
                                             uint64_t* out_cells, uint64_t* out_counts, int64_t* out_sums, uint64_t cap, uint64_t* out_n) try {
    return node_groupby_sparse(n, index, fields, views_flat, n_views, n_fields, row_ids_flat, n_rows,
                               SpRequest{ {}, GvAgg::kSum, GvInt{ afield, aview, a_depth, nullptr, 0 }, filter, n_filter_ops, shards, n_shards, start, ~0ull, limit },
                               out_cells, out_counts, out_sums, cap, out_n);
} FBGPU_CATCH

// Sum / Min / Max of an int field: per-device partials merged as ValCount.Add / Smaller / Larger do (executor.go:8446-8560)
extern "C" int fbgpu_node_bsi_sum(fbgpu_node* n, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                                  const uint64_t* shards, int64_t n_shards, int64_t* out_sum, uint64_t* out_count) try {
    if (!n || !out_sum || !out_count || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    NodeSplit sp = node_split(n, shards, n_shards);
    std::vector<int> devs = node_owners(sp);
    std::vector<int64_t> sums(n->ctx.size(), 0); std::vector<uint64_t> cnts(n->ctx.size(), 0);
    int rc = node_fan_out(n, devs, [&](int d) {
        return fbgpu_bsi_sum(n->ctx[(size_t)d], index, ops, n_ops, field, view, bit_depth, sp.shards[(size_t)d].data(), (int64_t)sp.shards[(size_t)d].size(), &sums[(size_t)d], &cnts[(size_t)d]);
    });
    if (rc) return rc;
    uint64_t s = 0, c = 0; for (int d : devs) { s += (uint64_t)sums[(size_t)d]; c += cnts[(size_t)d]; }     // wrapping, like the per-device sums
    *out_sum = (int64_t)s; *out_count = c;
    return FBGPU_OK;
} FBGPU_CATCH
extern "C" int fbgpu_node_bsi_minmax(fbgpu_node* n, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                                     const uint64_t* shards, int64_t n_shards, int32_t want_max, int64_t* out_val, uint64_t* out_count) try {
    if (!n || !out_val || !out_count || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    NodeSplit sp = node_split(n, shards, n_shards);
    std::vector<int> devs = node_owners(sp);
    std::vector<int64_t> vals(n->ctx.size(), 0); std::vector<uint64_t> cnts(n->ctx.size(), 0);
    int rc = node_fan_out(n, devs, [&](int d) {
        return fbgpu_bsi_minmax(n->ctx[(size_t)d], index, ops, n_ops, field, view, bit_depth, sp.shards[(size_t)d].data(), (int64_t)sp.shards[(size_t)d].size(), want_max, &vals[(size_t)d], &cnts[(size_t)d]);
    });
    if (rc) return rc;
    int64_t v = 0; uint64_t c = 0;
    for (int d : devs) {
        if (!cnts[(size_t)d]) continue;
        if (!c || (want_max ? vals[(size_t)d] > v : vals[(size_t)d] < v)) { v = vals[(size_t)d]; c = cnts[(size_t)d]; }
        else if (vals[(size_t)d] == v) c += cnts[(size_t)d];
    }
    *out_val = v; *out_count = c;
    return FBGPU_OK;
} FBGPU_CATCH

// Sort over an int field: every device sorts its own shards and keeps its first offset + limit pairs; the devices' lists (their
// columns are disjoint) are merged in the same order, as SortedRow.Merge does (executor.go:9574), and the window is cut after the
// merge
extern "C" int fbgpu_node_bsi_sort(fbgpu_node* n, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                                   const uint64_t* shards, int64_t n_shards, int32_t desc, uint64_t offset, int64_t limit,
                                   uint64_t* out_cols, int64_t* out_vals, uint64_t cap, uint64_t* out_n, uint64_t* out_total) try {
    int rc = bsi_sort_args(n, ops, n_ops, bit_depth, shards, n_shards, out_cols, out_vals, cap, out_n); if (rc) return rc;
    const uint64_t win_end = window_end(offset, limit);
    const NodeSplit sp = node_split(n, shards, n_shards);
    std::vector<int> devs = node_owners(sp);
    if (devs.empty()) devs.push_back(0);                 // no shard listed: still validate the program
    std::vector<std::vector<uint64_t>> cols(n->ctx.size()); std::vector<std::vector<int64_t>> vals(n->ctx.size()); std::vector<uint64_t> tot(n->ctx.size(), 0);
    rc = node_fan_out(n, devs, [&](int d) {
        fbgpu_ctx* c = n->ctx[(size_t)d];
        const auto& s = sp.shards[(size_t)d];
        std::shared_lock<std::shared_mutex> lk;
        int r = begin_query(c, lk); if (r) return r;
        return bsi_sort_run(c, index, ops, n_ops, field, view, bit_depth, s.data(), (int64_t)s.size(), desc != 0, 0, win_end,
                            cols[(size_t)d], vals[(size_t)d], &tot[(size_t)d]);
    });
    if (rc) return rc;
    struct Pair { int64_t v; uint64_t col; };
    const auto before = [desc](const Pair& a, const Pair& b) { return a.v != b.v ? (desc ? a.v > b.v : a.v < b.v) : a.col < b.col; };
    std::vector<Pair> all; uint64_t total = 0;
    for (int d : devs) {
        const size_t mid = all.size();
        for (size_t i = 0; i < cols[(size_t)d].size(); i++) all.push_back(Pair{ vals[(size_t)d][i], cols[(size_t)d][i] });
        std::inplace_merge(all.begin(), all.begin() + (long)mid, all.end(), before);
        total += tot[(size_t)d];
    }
    if (out_total) *out_total = total;
    const size_t lo = (size_t)std::min<uint64_t>(offset, all.size()), hi = (size_t)std::min<uint64_t>(win_end, all.size());
    std::vector<uint64_t> wc(hi - lo); std::vector<int64_t> wv(hi - lo);
    for (size_t i = lo; i < hi; i++) { wc[i - lo] = all[i].col; wv[i - lo] = all[i].v; }
    return write_window(wc, wv, out_cols, out_vals, cap, out_n);
} FBGPU_CATCH

// Distinct over an int field: every device lists the distinct values of its own shards; the lists merge by union, as
// SignedRow.Union does (executeDistinct executor.go:1173), and the totals add up
extern "C" int fbgpu_node_bsi_distinct(fbgpu_node* n, uint32_t index, const fbgpu_op* ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                                       const uint64_t* shards, int64_t n_shards, int64_t* out_vals, uint64_t cap, uint64_t* out_n, uint64_t* out_total) try {
    int rc = bsi_sort_args(n, ops, n_ops, bit_depth, shards, n_shards, (const uint64_t*)out_vals, out_vals, cap, out_n); if (rc) return rc;
    const NodeSplit sp = node_split(n, shards, n_shards);
    std::vector<int> devs = node_owners(sp);
    if (devs.empty()) devs.push_back(0);                 // no shard listed: still validate the program
    std::vector<std::vector<int64_t>> vals(n->ctx.size()); std::vector<uint64_t> tot(n->ctx.size(), 0);
    rc = node_fan_out(n, devs, [&](int d) {
        fbgpu_ctx* c = n->ctx[(size_t)d];
        const auto& s = sp.shards[(size_t)d];
        std::shared_lock<std::shared_mutex> lk;
        int r = begin_query(c, lk); if (r) return r;
        return bsi_distinct_run(c, index, ops, n_ops, field, view, bit_depth, s.data(), (int64_t)s.size(), vals[(size_t)d], &tot[(size_t)d]);
    });
    if (rc) return rc;
    std::vector<int64_t> all; uint64_t total = 0;
    for (int d : devs) {
        const size_t mid = all.size();
        all.insert(all.end(), vals[(size_t)d].begin(), vals[(size_t)d].end());
        std::inplace_merge(all.begin(), all.begin() + (long)mid, all.end());
        all.erase(std::unique(all.begin(), all.end()), all.end());
        total += tot[(size_t)d];
    }
    if (out_total) *out_total = total;
    return write_values(all, out_vals, cap, out_n);
} FBGPU_CATCH

// <bitmap call> returning a Row: every device emits the canonical Pilosa-roaring bytes of its own shards (absolute keys);
// Row.Merge (row.go:202) of disjoint shard sets is a merge of the container tables by key.  Two passes over the per-device
// images: sizes, then headers + payloads straight into the caller's buffer.
static inline uint32_t node_rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
static inline uint64_t node_rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }
extern "C" int fbgpu_node_row(fbgpu_node* n, uint32_t index, const fbgpu_op* ops, int32_t n_ops, const uint64_t* shards, int64_t n_shards,
                              uint8_t* out_buf, uint64_t out_cap, uint64_t* out_len, uint64_t* out_count) try {
    if (!n || !out_len || n_shards < 0 || (n_shards && !shards)) return fail(FBGPU_E_INVALID, "null argument");
    NodeSplit sp = node_split(n, shards, n_shards);
    std::vector<int> devs = node_owners(sp);
    if (devs.empty()) devs.push_back(0);
    if (devs.size() == 1) { auto& s = sp.shards[(size_t)devs[0]]; return fbgpu_row(n->ctx[(size_t)devs[0]], index, ops, n_ops, s.data(), (int64_t)s.size(), out_buf, out_cap, out_len, out_count); }
    std::vector<std::vector<uint8_t>> img(n->ctx.size()); std::vector<uint64_t> cnt(n->ctx.size(), 0);
    int rc = node_fan_out(n, devs, [&](int d) {
        auto& s = sp.shards[(size_t)d]; auto& b = img[(size_t)d];
        uint64_t need = 0;
        b.resize(1 << 20);
        int r = fbgpu_row(n->ctx[(size_t)d], index, ops, n_ops, s.data(), (int64_t)s.size(), b.data(), b.size(), &need, &cnt[(size_t)d]);
        if (r == FBGPU_E_NOSPACE) { b.resize(need); r = fbgpu_row(n->ctx[(size_t)d], index, ops, n_ops, s.data(), (int64_t)s.size(), b.data(), b.size(), &need, &cnt[(size_t)d]); }
        if (r) return r;
        b.resize(need);
        return 0;
    });
    if (rc) return rc;
    // image layout (roaring.go:1738-1817): u32 cookie, u32 n, n x {u64 key, u16 type, u16 N-1}, n x u32 offset, payloads
    struct Src { const uint8_t* p; uint64_t len; uint32_t n; uint32_t i; };
    std::vector<Src> src; uint64_t total_n = 0, payload = 0, count = 0;
    for (int d : devs) {
        const auto& b = img[(size_t)d]; count += cnt[(size_t)d];
        if (b.size() < 8) continue;
        uint32_t k = node_rd32(b.data() + 4);
        if (!k) continue;
        src.push_back(Src{ b.data(), b.size(), k, 0 }); total_n += k; payload += b.size() - (8 + 16ull * k);
    }
    const uint64_t need = 8 + 16 * total_n + payload;
    *out_len = need; if (out_count) *out_count = count;
    if (need > out_cap || !out_buf) return fail(FBGPU_E_NOSPACE, "row needs %llu bytes", (unsigned long long)need);
    if (need > 0xffffffffull + 8) return fail(FBGPU_E_NOSPACE, "row image exceeds the 4 GiB offset range of the format");
    const uint32_t cookie = 12348u;
    memcpy(out_buf, &cookie, 4); const uint32_t tn = (uint32_t)total_n; memcpy(out_buf + 4, &tn, 4);
    uint8_t* hdr = out_buf + 8; uint8_t* offs = out_buf + 8 + 12 * total_n; uint64_t pos = 8 + 16 * total_n;
    auto payload_len = [](const Src& s, uint32_t i) -> uint64_t {
        const uint64_t a = node_rd32(s.p + 8 + 12ull * s.n + 4ull * i);
        const uint64_t b = i + 1 < s.n ? node_rd32(s.p + 8 + 12ull * s.n + 4ull * (i + 1)) : s.len;
        return b - a;
    };
    for (uint64_t k = 0; k < total_n; k++) {
        Src* best = nullptr; uint64_t bk = 0;
        for (auto& s : src) if (s.i < s.n) { const uint64_t key = node_rd64(s.p + 8 + 12ull * s.i); if (!best || key < bk) { best = &s; bk = key; } }
        memcpy(hdr + 12 * k, best->p + 8 + 12ull * best->i, 12);
        const uint32_t o = (uint32_t)pos; memcpy(offs + 4 * k, &o, 4);
        const uint64_t len = payload_len(*best, best->i);
        memcpy(out_buf + pos, best->p + node_rd32(best->p + 8 + 12ull * best->n + 4ull * best->i), len);
        pos += len; best->i++;
    }
    return FBGPU_OK;
} FBGPU_CATCH

// ---- in-process form of the fused Count exchange: the mailboxes of contexts living in THIS process are wired to each other
// directly (peer access instead of CUDA IPC).  Used by tests of the bounded wait; a launcher with one thread per GPU may use
// it in place of fbgpu_comm_p2p_handle / _open.
extern "C" int fbgpu_comm_p2p_open_local(fbgpu_ctx* const* ctxs, int32_t n_ranks) try {
    if (!ctxs || n_ranks < 1 || n_ranks > kMaxRanks) return fail(FBGPU_E_INVALID, "bad argument");
    for (int r = 0; r < n_ranks; r++) {
        fbgpu_ctx* c = ctxs[r];
        if (!c || c->inspect_only) return fail(FBGPU_E_INVALID, "context %d holds no device", r);
        CUDA_TRY(cudaSetDevice(c->device));
        if (!c->mbox) CUDA_TRY(cudaMalloc((void**)&c->mbox, sizeof(Mailbox)));
        CUDA_TRY(cudaDeviceSynchronize());
        CUDA_TRY(cudaMemset(c->mbox, 0, sizeof(Mailbox)));
        for (int p = 0; p < n_ranks; p++) if (ctxs[p] && ctxs[p]->device != c->device) {
            int can = 0; CUDA_TRY(cudaDeviceCanAccessPeer(&can, c->device, ctxs[p]->device));
            if (!can) return fail(FBGPU_E_COMM, "device %d cannot access device %d", c->device, ctxs[p]->device);
            cudaError_t e = cudaDeviceEnablePeerAccess(ctxs[p]->device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return fail(FBGPU_E_COMM, "cudaDeviceEnablePeerAccess failed: %s", cudaGetErrorString(e));
            (void)cudaGetLastError();
        }
    }
    for (int r = 0; r < n_ranks; r++) {
        fbgpu_ctx* c = ctxs[r];
        CUDA_TRY(cudaSetDevice(c->device));
        std::lock_guard<std::mutex> lk(c->coll_mu);
        for (int p = 0; p < kMaxRanks; p++) c->peers[p] = p < n_ranks ? ctxs[p]->mbox : nullptr;
        c->peers_local = true;
        if (c->d_peers.ensure(sizeof(Mailbox*) * kMaxRanks)) return FBGPU_E_NOMEM;
        CUDA_TRY(cudaMemcpy(c->d_peers.p, c->peers, sizeof(Mailbox*) * kMaxRanks, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaDeviceSynchronize());
        c->n_ranks = n_ranks; c->rank = r; c->epoch = 0; c->p2p = true;
    }
    return FBGPU_OK;
} FBGPU_CATCH
