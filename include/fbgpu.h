/*
 * fbgpu.h — C ABI of libfbgpu: an H100-native (sm_90a) roaring-bitmap query executor that replaces the
 * per-shard inner loop of FeatureBase's executor.go / fragment.go / roaring/.
 *
 * The reference has no FFI seam on this path (it is 100 % Go).  Each entry point below names the
 * reference function(s) whose per-shard map step + reduce it replaces; a Go maintainer binds them through
 * cgo from executor.mapperLocal (INTEGRATION.md shows the stub).  Paths are relative to the FeatureBase source tree.
 *
 * Conventions: all integers fixed width, little endian; no callbacks; inputs are read-only and never
 * retained after return (cgo pointer rules); outputs are caller-allocated; return 0 on success or a
 * negative FBGPU_E_* (maps to Go `error`; every executor function returns (T, error)).  Thread-safe and
 * re-entrant: any OS thread may call any function on a context (goroutines migrate between threads), the
 * library sets the CUDA device itself on every call.  One context per GPU; a context owns the contiguous
 * shard range its caller loads into it (SURVEY.md §8e).
 */
#ifndef FBGPU_H
#define FBGPU_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FBGPU_ABI_VERSION 2

/* error codes */
#define FBGPU_OK 0
#define FBGPU_E_INVALID (-1)  /* bad argument / malformed program                       */
#define FBGPU_E_QUERY (-2)    /* query the reference rejects (e.g. empty Intersect())    */
#define FBGPU_E_FORMAT (-3)   /* unreadable roaring data                                 */
#define FBGPU_E_NOSPACE (-4)  /* output buffer too small; required size reported         */
#define FBGPU_E_CUDA (-5)     /* CUDA runtime failure (see fbgpu_last_error)             */
#define FBGPU_E_NOMEM (-6)
#define FBGPU_E_COMM (-7)     /* NCCL failure / communicator not initialised             */

typedef struct fbgpu_ctx fbgpu_ctx; /* opaque, one per GPU */

/* fbgpu_init(FBGPU_DEVICE_NONE, ..) creates an INSPECTION-ONLY context: it touches no device, accepts the residency calls
 * (load / drop / commit / stats) and fbgpu_debug_container(), and refuses every query with FBGPU_E_CUDA.  It exists so that the
 * loaders and the store tables can be tested on a machine without a GPU; it is not a CPU execution path. */
#define FBGPU_DEVICE_NONE (-1)

/* lifecycle (what Holder.Open / Holder.Close are to the fragments of a node, holder.go:432, 614): one context per GPU,
 * created once per process.  device_ordinal is the CUDA ordinal this context owns. */
int fbgpu_init(int32_t device_ordinal, fbgpu_ctx **out);
void fbgpu_shutdown(fbgpu_ctx *ctx);
/* thread-local message of the last failing call on this thread */
const char *fbgpu_last_error(void);
int32_t fbgpu_abi_version(void);

/* ---- residency (replaces fragment.row -> tx.OffsetRange -> rbf cursor walk: fragment.go:283-333,
 *      rbf.go:472, rbf/tx.go:1586-1637; data source = tx.RoaringBitmap / Bitmap.WriteTo bytes, tx.go:85) ----
 * `roaring` = Pilosa-roaring bytes (cookie 12348, roaring/roaring.go:1738-1817) or official RoaringBitmap
 * bytes (12346/12347, roaring.go:6943-7006) of ONE fragment with fragment-relative keys row*16+slot
 * (fragment.go:2780-2782).  index/field/view are caller-assigned ids.  Replaces any previous content of
 * (index,field,view,shard).  The library copies; the caller keeps ownership of the bytes. */
int fbgpu_load_fragment(fbgpu_ctx *ctx, uint32_t index, uint32_t field, uint32_t view, uint64_t shard,
                        const uint8_t *roaring, uint64_t nbytes);
/* bulk form (the shape of API.ImportRoaringShard's per-view payloads, api.go:1647; fragment.importRoaringOverwrite
 * fragment.go:2196): n fragments of the same (index,field,view); fragment i is buf[offsets[i], offsets[i+1]) */
int fbgpu_load_fragments(fbgpu_ctx *ctx, uint32_t index, uint32_t field, uint32_t view,
                         const uint64_t *shards, int64_t n, const uint8_t *buf, const uint64_t *offsets);
/* view.deleteFragment (view.go:405): the fragment no longer answers queries; its arena space is reclaimed by fbgpu_compact */
int fbgpu_drop_fragment(fbgpu_ctx *ctx, uint32_t index, uint32_t field, uint32_t view, uint64_t shard);
/* Incremental refresh: what ONE committed write transaction did to ONE fragment, container by container -- the mirror of the
 * Tx.PutContainer / Tx.RemoveContainer calls of the transaction (tx.go:91-96, rbf/tx.go:791-860; the writes reach them through
 * fragment.setBit / importRoaring / ImportRoaringBits, fragment.go:2196, rbf/tx.go:1819).  `roaring` (may be NULL / 0 bytes) holds
 * ONLY the containers that were written, under their fragment-relative keys: each replaces the container stored under its key, or
 * adds it.  removed_keys lists the keys whose containers were deleted.  Containers the transaction did not touch keep their payload
 * where it is in HBM, so the call moves the changed containers' bytes plus the fragment's row / descriptor entries -- not the
 * fragment (fbgpu_load_fragment re-sends it whole); the next fbgpu_commit patches the tables of the touched (view, shard) pairs
 * instead of rebuilding them.  Replaced payloads become holes (fbgpu_stats.dead_bytes) that fbgpu_compact reclaims.  A fragment
 * that is not resident yet is created from the written containers; one whose last container is removed is dropped.  A key that
 * is both written and removed is FBGPU_E_INVALID.  All-or-nothing like the loads. */
int fbgpu_apply_containers(fbgpu_ctx *ctx, uint32_t index, uint32_t field, uint32_t view, uint64_t shard,
                           const uint8_t *roaring, uint64_t nbytes, const uint64_t *removed_keys, int64_t n_removed);
/* (SURVEY §8 f1) Load the fragments of ONE shard straight from its RBF database, i.e. from the bytes of
 * `<index>/backends/rbf/<shard>/data` (and, if it is not empty, `wal`) -- one RBF DB holds every field/view of a
 * shard (dbshard.go:64-71).  Replaces the per-fragment tx.RoaringBitmap().WriteTo re-serialisation: leaf cells (array /
 * RLE / bitmap page, rbf/rbf.go:489-512) become store containers directly.  names[i] is an RBF bitmap name
 * "~field;view<" (rbfName rbf.go:504, short_txkey/txkey.go:129); fields[i] / views[i] are the ids the caller uses for
 * it in programs.  Names that the file does not hold are skipped (a field without data in this shard); *out_loaded
 * (may be NULL) receives how many were found.  Committed WAL pages override data pages (rbf/tx.go:1269-1273); pages
 * after the WAL's last meta page are ignored.  The library copies; the caller keeps the buffers. */
int fbgpu_load_rbf(fbgpu_ctx *ctx, uint32_t index, uint64_t shard, const uint8_t *data, uint64_t data_bytes,
                   const uint8_t *wal, uint64_t wal_bytes, const char *const *names, const uint32_t *fields,
                   const uint32_t *views, int32_t n_names, int32_t *out_loaded);
/* Same, with the library mapping the files itself (read-only mmap of `<dir>/data` and, when present and non-empty,
 * `<dir>/wal`): the caller hands over the shard's RBF directory instead of reading it into its own memory first.  The
 * mappings are released before the call returns.  FBGPU_E_FORMAT when `data` cannot be opened or mapped. */
int fbgpu_load_rbf_dir(fbgpu_ctx *ctx, uint32_t index, uint64_t shard, const char *dir, const char *const *names,
                       const uint32_t *fields, const uint32_t *views, int32_t n_names, int32_t *out_loaded);
/* pushes pending host-side staging to HBM now (otherwise done lazily by the next query): the point at which loaded
 * fragments become visible to queries, as RBFTx.Commit (rbf.go:189) is for writes in the reference */
int fbgpu_commit(fbgpu_ctx *ctx);
/* Replacing or dropping a fragment leaves its old payload in the arena.  fbgpu_compact() commits what is pending, then
 * copies the live fragments into a fresh arena (device to device) and rebuilds the tables; fbgpu_commit() does the same on
 * its own once at least 256 MiB and half of the arena are dead.  Blocks queries for the duration, like a commit. */
int fbgpu_compact(fbgpu_ctx *ctx);
/* Inspection (FBGPU_DEVICE_NONE contexts only): the container the kernels would find for (index, field, view, shard, row,
 * slot), located by the same resolve() code, with its payload exactly as stored (incl. the padding of the last 16-byte
 * chunk).  *out_type = 0 when the container is absent, else 1 array / 2 bitmap / 3 run. */
int fbgpu_debug_container(fbgpu_ctx *ctx, uint32_t index, uint32_t field, uint32_t view, uint64_t shard, uint64_t row,
                          int32_t slot, uint32_t *out_type, uint32_t *out_card, uint32_t *out_runs,
                          uint8_t *out_payload, uint64_t cap, uint64_t *out_len);

typedef struct {
    uint64_t fragments, containers;
    uint64_t array_containers, bitmap_containers, run_containers;
    uint64_t payload_bytes;   /* roaring payload bytes resident in HBM (array 2n, bitmap 8192, run 4r) */
    uint64_t device_bytes;    /* total HBM held by the store incl. descriptors and padding            */
    uint64_t dead_bytes;      /* arena bytes of replaced / dropped fragments and containers, reclaimed by fbgpu_compact */
    uint64_t full_commits;    /* commits that rebuilt (and re-sent) every lookup table                                */
    uint64_t patch_commits;   /* commits that patched the touched (view, shard) entries and sent only those + the new tails */
} fbgpu_stats;
int fbgpu_get_stats(fbgpu_ctx *ctx, fbgpu_stats *out);

/* ---- bitmap-call programs (replaces executeBitmapCallShard and its children, executor.go:1782-1816) ----
 * A program is the post-order walk of the pql.Call tree of one bitmap call. */
enum {
    FBGPU_OP_ROW = 1,        /* Row(field=row)         executeRowShard executor.go:5120 ; field,view,a=row id        */
    FBGPU_OP_INTERSECT = 2,  /* Intersect(c1..cn)      executeIntersectShard :5357 ; argc=n (0 => FBGPU_E_QUERY)      */
    FBGPU_OP_UNION = 3,      /* Union(c1..cn)          executeUnionShard :5382 ; argc=n (0 => empty row)             */
    FBGPU_OP_DIFFERENCE = 4, /* Difference(c1..cn)     executeDifferenceShard :2950 ; left fold; argc 0 => E_QUERY    */
    FBGPU_OP_XOR = 5,        /* Xor(c1..cn)            executeXorShard :5513 ; left fold; argc 0 => empty row         */
    FBGPU_OP_NOT = 6,        /* Not(c)                 executeNotShard :5554 ; field,view = existence field, a = row  */
    FBGPU_OP_BSI_RANGE = 7,  /* Row(v <op> k)          executeRowBSIGroupShard :5249 -> fragment.rangeOp fragment.go:937
                                field,view = bsig view; a = bitDepth; b = FBGPU_CMP_*; lo(,hi) = base-adjusted
                                predicate(s) exactly as passed to rangeOp/rangeBetween                              */
    FBGPU_OP_EMPTY = 8,      /* empty row (out-of-range BSI predicate, executor.go:5331)                               */
    FBGPU_OP_ALL = 9         /* All(): existence row   executeAllCallShard :5781 ; field,view = existence, a = row    */
};
enum { FBGPU_CMP_EQ = 1, FBGPU_CMP_NEQ = 2, FBGPU_CMP_LT = 3, FBGPU_CMP_LTE = 4, FBGPU_CMP_GT = 5,
       FBGPU_CMP_GTE = 6, FBGPU_CMP_BETWEEN = 7 };

typedef struct {
    uint32_t opcode, field, view, argc;
    uint64_t a, b;
    int64_t lo, hi;
} fbgpu_op; /* 48 bytes */

/* Count(<bitmap call>) over the listed shards (executeCount executor.go:5839-5892: map = per-shard
 * Row.Count(), reduce = u64 add).  *out_total is the sum over this context's shards, all-reduced over
 * the communicator when one is attached.  out_per_shard may be NULL, else receives n_shards counts. */
int fbgpu_count(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops,
                const uint64_t *shards, int64_t n_shards, uint64_t *out_total, uint64_t *out_per_shard);

/* Row.Any() of a bitmap call (row.go:258; roaring.go:4266-4408 intersectionAny lifted to shard granularity): *out_any = 1 as soon
 * as one block of shards holds a column.  Shards are evaluated in blocks of growing size (8, 64, 512, ...), so a non-empty row
 * costs one small launch.  Local to this context: never merged across GPUs (fbgpu_node_any walks the devices itself). */
int fbgpu_any(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops,
              const uint64_t *shards, int64_t n_shards, int32_t *out_any);

/* <bitmap call> returning a Row (mapReduce with Row.Merge, executor.go:1694-1780, row.go:202): writes
 * Pilosa-roaring bytes with absolute keys shard*16+slot and canonical (optimize()) encodings, i.e. what
 * Row.Roaring() (row.go:174-180) yields after Optimize.  If out_cap is too small returns FBGPU_E_NOSPACE
 * and sets *out_len to the needed size.  *out_count receives the row's cardinality (may be NULL). */
int fbgpu_row(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops,
              const uint64_t *shards, int64_t n_shards,
              uint8_t *out_buf, uint64_t out_cap, uint64_t *out_len, uint64_t *out_count);

/* <bitmap call> returning the row's column ids (Row.Columns(), row.go:471, what Extract / Limit / API row responses
 * iterate): ascending absolute column ids (shard * 2^20 + position), expanded on the device from the result bitmaps, so
 * a caller that wants ids does not have to decode roaring containers.  Skips the first `offset` columns and writes at
 * most `limit` (limit < 0: no limit) — executeLimitCall's window.  *out_n = columns written, *out_total = the row's
 * cardinality before the window (may be NULL).  FBGPU_E_NOSPACE when cap is smaller than the window; *out_n then holds
 * the needed capacity. */
int fbgpu_columns(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops,
                  const uint64_t *shards, int64_t n_shards, uint64_t offset, int64_t limit,
                  uint64_t *out_cols, uint64_t cap, uint64_t *out_n, uint64_t *out_total);

/* Values of an int field for the columns of a row: the bulk form of fragment.value (fragment.go:585-617) that Extract
 * (executor.go executeExtract) and Distinct on int fields (executeDistinctShardBSI :2034) are built on.  The row is
 * <filter program> ∩ not-null(field) (n_ops == 0: every column that has a value); for its columns, in ascending order and
 * inside the offset / limit window, out_cols[i] receives the column id and out_vals[i] the stored sign-magnitude value as
 * an int64, i.e. value - bsiGroup.Base (the caller adds Base, field.go:1640).  `view` is the field's bsig_ view,
 * bit_depth (0..64) its current depth.  A field over [MinInt64, MaxInt64] has depth 64: INT64_MIN is stored as the sign
 * row plus magnitude 2^63, and -magnitude wraps to INT64_MIN as in fragment.value.  Same capacity contract as fbgpu_columns. */
int fbgpu_extract(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                  const uint64_t *shards, int64_t n_shards, uint64_t offset, int64_t limit,
                  uint64_t *out_cols, int64_t *out_vals, uint64_t cap, uint64_t *out_n, uint64_t *out_total);

/* The rows of a set, mutex, bool or time field for every column of a row: the transposition Extract makes of each Rows(f)
 * child (executeExtractShard executor.go:4758-4960 intersects every row of the fragment with the filter and turns the hits
 * into a column -> rows matrix), and what Sort over a bool or mutex field orders by.
 *   - The row R is <ops>, compiled and evaluated as for fbgpu_columns.  *out_total = |R| (when out_total is not NULL).
 *   - The window is [offset, offset + limit) of R's columns in ascending order (limit < 0: no limit), as for fbgpu_columns:
 *     out_cols[0 .. n_cols) is what fbgpu_columns returns for the same arguments, and *out_n_cols = n_cols.  A column with no
 *     row in the field is listed too, with an empty list.
 *   - For window column i, out_rows[out_offsets[i] .. out_offsets[i + 1]) holds the row ids r, strictly ascending, such that
 *     the column is in Row(field = r) of `view`.  out_offsets receives n_cols + 1 entries (it has room for cap_cols + 1),
 *     out_offsets[0] = 0, and *out_n_rows = out_offsets[n_cols].  A shard without the field's fragment, and a view that was
 *     never loaded, give empty lists.
 *   - cap_cols < n_cols or cap_rows < n_rows is FBGPU_E_NOSPACE with nothing written; *out_n_cols and *out_n_rows then both
 *     hold the sizes needed, so one retry succeeds.
 *   - Local to the context: never reduced over a communicator.
 *   - Device memory: the call holds at most one radix-sort buffer of max(2^24, the most rows of one window column)
 *     (key, row id) pairs of 32 bytes and 4 bytes per window column of one evaluation batch, whatever the window's size;
 *     FBGPU_E_NOMEM when that cannot be allocated.
 *   - A NULL handle, out_n_cols or out_n_rows, a non-zero cap_cols with NULL out_cols or out_offsets, a non-zero cap_rows with
 *     NULL out_rows, n_ops < 0 or n_ops > 0 with NULL ops, n_shards < 0 or n_shards > 0 with NULL shards ("null argument") are
 *     FBGPU_E_INVALID, reported before the device check.
 * There is no node form. */
int fbgpu_extract_rows(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view,
                       const uint64_t *shards, int64_t n_shards, uint64_t offset, int64_t limit,
                       uint64_t *out_cols, uint64_t *out_offsets, uint64_t cap_cols,
                       uint64_t *out_rows, uint64_t cap_rows,
                       uint64_t *out_n_cols, uint64_t *out_n_rows, uint64_t *out_total);

/* Sort(<filter>, field=, sort-desc=, offset=, limit=) over an int field (executeSort / executeSortShard executor.go:9321-9560):
 * the row of fbgpu_extract, put in order on the device, and only a window of it returned.
 *   - The row is <filter program> ∩ not-null(field), exactly as for fbgpu_extract (n_ops == 0: every column that has a value);
 *     *out_total = |row| (when out_total is not NULL).
 *   - The order is ascending by stored value (value - Base, read from the planes as fbgpu_extract reads them, INT64_MIN included
 *     at depth 64), ties in ascending column order.  desc != 0: descending by value, ties still in ascending column order.  A
 *     sign with magnitude 0 is the value 0 and sorts among the other zeros by column.
 *   - The window is [offset, offset + limit) of that order; limit < 0 means no limit.  out_cols[i] / out_vals[i] receive its
 *     i-th (column, stored value) pair, *out_n its size.  Same capacity contract as fbgpu_columns: a cap smaller than the
 *     window is FBGPU_E_NOSPACE with nothing written and *out_n = the size needed.
 *   - bit_depth 0..64.
 *   - Local to the context: never reduced over a communicator.  Ranks merge their lists as SortedRow.Merge does, so a caller
 *     asks each rank for offset 0 and limit offset + limit and cuts the window after the merge.
 *   - Device memory: the call holds at most max(2K, K + 2^24) (key, column) pairs of 32 bytes (both halves of the radix sort),
 *     K = offset + limit, or the whole row without a limit; FBGPU_E_NOMEM when that cannot be allocated.
 *   - NULL pointers, a non-zero cap with NULL outputs, n_shards < 0 or n_ops < 0 ("null argument") and a bit_depth outside
 *     0..64 are FBGPU_E_INVALID, reported before the device check.
 * The node form runs each device with offset 0 and limit offset + limit (saturating), merges the devices' lists in the same
 * order (their columns are disjoint) and cuts the window, under the same contracts. */
int fbgpu_bsi_sort(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                   const uint64_t *shards, int64_t n_shards, int32_t desc, uint64_t offset, int64_t limit,
                   uint64_t *out_cols, int64_t *out_vals, uint64_t cap, uint64_t *out_n, uint64_t *out_total);

/* Distinct(<filter>, field=) over an int field (executeDistinct :1173 / executeDistinctShardBSI executor.go:2034): the distinct
 * stored values of fbgpu_extract's row, found on the device.
 *   - The row is <filter program> ∩ not-null(field), exactly as for fbgpu_extract (n_ops == 0: every column that has a value);
 *     *out_total = |row| (when out_total is not NULL).
 *   - out_vals receives the row's distinct stored values (value - Base, read from the planes as fbgpu_extract reads them),
 *     strictly ascending as int64, and *out_n their number U.  A sign with magnitude 0 is the value 0; at depth 64 INT64_MIN
 *     (sign + magnitude 2^63) is included.  The list equals np.unique of fbgpu_extract's values, bit for bit.  Same capacity
 *     contract as fbgpu_columns: cap < U is FBGPU_E_NOSPACE with nothing written and *out_n = U.
 *   - bit_depth 0..64.
 *   - Local to the context: never reduced over a communicator.  Ranks merge their lists by union, as SignedRow.Union does.
 *   - Device memory: the call holds at most max(2U, U + 2^24) keys of 16 bytes (both halves of the radix sort);
 *     FBGPU_E_NOMEM when that cannot be allocated.
 *   - NULL handle or out_n, a non-zero cap with NULL out_vals, n_shards < 0 or n_ops < 0 ("null argument") and a bit_depth
 *     outside 0..64 are FBGPU_E_INVALID, reported before the device check.
 * The node form lists each device's values, merges the lists into one ascending list without duplicates and adds up the
 * totals, under the same contracts. */
int fbgpu_bsi_distinct(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                       const uint64_t *shards, int64_t n_shards, int64_t *out_vals, uint64_t cap, uint64_t *out_n, uint64_t *out_total);

/* Min / Max of an int field over a row (executeMin :1225 / executeMax :1261, fragment.min / max fragment.go:752-838): the row
 * is <filter program> ∩ not-null(field) (n_ops == 0: every column with a value).  *out_val receives the extreme stored
 * value, i.e. value - bsiGroup.Base (the caller adds Base), *out_count how many columns hold it — the reference's ValCount;
 * *out_count == 0 when the row is empty.  bit_depth 0..64, as for fbgpu_extract.  One evaluation of the row plus one pass over the bit planes, every plane container
 * read once (the composition from fbgpu_count calls re-reads the planes it has kept).  Not reduced over the communicator:
 * the caller merges per-node ValCounts as it does today (ValCount.Smaller / Larger executor.go:8446-8560). */
int fbgpu_bsi_minmax(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                     const uint64_t *shards, int64_t n_shards, int32_t want_max, int64_t *out_val, uint64_t *out_count);

/* Sum of an int field over a row (executeSum :1119, fragment.sum fragment.go:722-750): *out_count = |<filter> ∩ not-null|,
 * *out_sum = Σ (stored value) over those columns in wrapping int64 arithmetic, i.e. Σ (value - Base); the caller adds
 * count * Base (executeSumCountShard :2203-2206).  bit_depth 0..64.  One evaluation of the row, one pass over the planes.  Per-node result,
 * like fbgpu_bsi_minmax (ValCount.Add merges nodes). */
int fbgpu_bsi_sum(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                  const uint64_t *shards, int64_t n_shards, int64_t *out_sum, uint64_t *out_count);

/* Order statistics of an int field over a row: the row is <filter program> ∩ not-null(field) (n_ops == 0: every column with a
 * value).  Sort the stored values (value - bsiGroup.Base, sign-magnitude planes as fbgpu_extract reads them) of its columns
 * ascending, keeping duplicates.  out_vals[i] = the value at 0-based position ranks[i], and out_counts[i] = how many columns hold
 * that value (may be NULL).  *out_total = |row|.  ranks need not be sorted or distinct; n_ranks == 0 only reports the total
 * (out_vals may then be NULL).  At most FBGPU_SELECT_MAX_RANKS ranks per call.  A rank >= *out_total is FBGPU_E_INVALID
 * (*out_total is still set).  One evaluation of the row, then an MSB-first radix select over the bit planes chained on the
 * device (every plane container read at most twice) and one D2H copy.  Device memory held by the call: 8 KiB per (shard, slot)
 * unit per distinct rank (at least one).  Local to this context: a context with a communicator attached returns FBGPU_E_COMM,
 * because per-rank order statistics do not merge.  Percentile (executePercentile :1310-1600) needs the ranks 0, T-1,
 * desiredLess and T-1-desiredGreater: its bisection then runs on the host over these values without further queries.
 * bit_depth 0..63: the sort key takes depth + 1 bits (a depth-64 field takes Percentile's query-driven bisection). */
#define FBGPU_SELECT_MAX_RANKS 8
int fbgpu_bsi_select(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view,
                     int32_t bit_depth, const uint64_t *shards, int64_t n_shards, const uint64_t *ranks, int32_t n_ranks,
                     int64_t *out_vals, uint64_t *out_counts, uint64_t *out_total);

/* Per-row counts of one field, optionally intersected with a filter program: the exact part of TopN
 * (fragment.top with explicit ids, fragment.go:1317-1437) and TopK (doTopK executor.go:2705-2746).
 * row_ids != NULL: counts for exactly those rows (out_counts[i] for row_ids[i]).
 * row_ids == NULL: all rows present in the field over the shards; writes every (row id, count) pair with
 * count > 0 sorted by (count desc, row id asc) — the reference's tie order is unspecified (cache.go:464-482).
 * *out_n receives the number of such rows; when it exceeds cap nothing is written and the call returns
 * FBGPU_E_NOSPACE (never a truncated list: Rows() and the TopN candidate set must be complete) — call again
 * with buffers of *out_n entries.
 * Counts are all-reduced over the communicator in the row_ids form. */
int fbgpu_row_counts(fbgpu_ctx *ctx, uint32_t index, uint32_t field, uint32_t view,
                     const uint64_t *row_ids, int32_t n_rows,
                     const fbgpu_op *filter, int32_t n_filter_ops,
                     const uint64_t *shards, int64_t n_shards,
                     uint64_t *out_row_ids, uint64_t *out_counts, int32_t cap, int32_t *out_n);
/* The same counts kept apart per shard, for explicit rows: out_counts[s * n_rows + i] = |Row(row_ids[i]) [∩ filter]| in
 * shards[s] (a shard without the fragment gives zeros).  fragment.top applies its MinThreshold / Tanimoto cut-offs to each
 * shard's own counts before Pairs.Add sums them (fragment.go:1329-1388, executeTopNShards executor.go:2831-2866), so TopN
 * with threshold= / tanimotoThreshold= needs this matrix, not the reduced vector.  Never all-reduced: a shard belongs to
 * one rank. */
int fbgpu_row_counts_per_shard(fbgpu_ctx *ctx, uint32_t index, uint32_t field, uint32_t view,
                               const uint64_t *row_ids, int32_t n_rows, const fbgpu_op *filter, int32_t n_filter_ops,
                               const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
/* TopN(f, Src, threshold=) and TopN(f, Src, tanimotoThreshold=): fragment.top's per-shard cut-offs for a cache that holds every
 * row, without N-truncation (fragment.go:1317-1437), and the sum over the shards of what passes (Pairs.Add in
 * executeTopNShards, executor.go:2831-2866), in one call.  For every listed shard s and candidate row r: cnt = |Row(field = r)|
 * in s; with a Src program (n_src_ops > 0) S = Src in s, srcCount = |S| and count = |Row(r) ∩ S|, else count = cnt.  The pair
 * is dropped
 *   - Tanimoto mode (tanimoto_threshold t > 0 and a Src): if cnt == 0, (double)cnt <= (double)(srcCount * t) / 100,
 *     (double)cnt >= (double)(srcCount * 100) / (double)t, count == 0, or
 *     ceil((double)(count * 100) / (double)(cnt + srcCount - count)) <= (double)t (products in uint64, as in Go);
 *   - otherwise, with m = max(min_threshold, 1): if cnt < m or count < m (t without a Src is ignored, as in the reference).
 * total[r] = the sum of count over the shards where (s, r) is kept.  The output forms are fbgpu_row_counts': row_ids != NULL
 * (any order, repeats allowed): out_counts[i] = total[row_ids[i]], all-reduced over the communicator.  row_ids == NULL: the
 * candidates are the rows with a container in the field in at least one listed shard; the rows with total > 0 are written
 * sorted by (total desc, row id asc) under the FBGPU_E_NOSPACE / *out_n contract, not all-reduced.
 * tanimoto_threshold > 100 is FBGPU_E_INVALID, like NULL pointers, n_rows < 0 and n_src_ops < 0, all reported before the
 * device check.  The node form takes the same arguments. */
int fbgpu_topn_cutoffs(fbgpu_ctx *ctx, uint32_t index, uint32_t field, uint32_t view,
                       const uint64_t *row_ids, int32_t n_rows,
                       const fbgpu_op *src, int32_t n_src_ops,
                       uint64_t min_threshold, uint32_t tanimoto_threshold,
                       const uint64_t *shards, int64_t n_shards,
                       uint64_t *out_row_ids, uint64_t *out_counts, int32_t cap, int32_t *out_n);
/* fbgpu_row_counts with each row taken as its union over n_views (>= 1, any number) views of the field: the counts of TopK(f,
 * from=, to=) and the row ids of Rows(f, from=, to=) on a time field, whose covering views are listed in `views`
 * (executeTopKShardTime executor.go:2506-2533 over the mergerator :2570; executeRowsShard :4107-4127).
 * count(r) = |(∪_v Row(field = r) in view v) [∩ filter]|.  row_ids != NULL: out_counts[i] for row_ids[i], all-reduced over the
 * communicator.  row_ids == NULL: the candidates are the row ids with a container in at least one listed view in at least one
 * listed shard; the rows with count > 0 are written sorted by (count desc, row id asc), with fbgpu_row_counts' FBGPU_E_NOSPACE /
 * *out_n contract, not all-reduced.  A view never loaded, or without a fragment in a shard, contributes nothing there; a view
 * listed twice counts once.  n_views == 1 is fbgpu_row_counts. */
int fbgpu_row_counts_views(fbgpu_ctx *ctx, uint32_t index, uint32_t field, const uint32_t *views, int32_t n_views,
                           const uint64_t *row_ids, int32_t n_rows, const fbgpu_op *filter, int32_t n_filter_ops,
                           const uint64_t *shards, int64_t n_shards,
                           uint64_t *out_row_ids, uint64_t *out_counts, int32_t cap, int32_t *out_n);

/* Many fused Intersect+Count pairs in ONE launch: out_counts[i] = |Row(field_a = rows_a[i]) ∩ Row(field_b = rows_b[i])| over
 * the shards — the inner loop of fragment.top with a plain-row Src (count = Src.intersectionCount(row) per candidate
 * row, fragment.go:1367-1372,1416-1420), of the GroupBy leaf (executor.go:8893) and of BenchmarkFragment_IntersectionCount
 * (fragment_internal_test.go:1461), without materialising anything.  All-reduced over the communicator. */
int fbgpu_count_pairs(fbgpu_ctx *ctx, uint32_t index, uint32_t field_a, uint32_t view_a, const uint64_t *rows_a,
                      uint32_t field_b, uint32_t view_b, const uint64_t *rows_b, int32_t n_pairs,
                      const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);

/* Which of the nine container-pair kernels Count(Intersect(Row a, Row b)) exercises and how often: out_hist[4 * ta + tb] = number
 * of (shard, slot) units whose a / b containers have types ta / tb (0 absent, 1 array, 2 bitmap, 3 run).  The reference keeps
 * the same information as statsHit("intersectionCount/...") counters (roaring.go:4477-4614).  Computed on the device. */
int fbgpu_pair_types(fbgpu_ctx *ctx, uint32_t index, uint32_t field_a, uint32_t view_a, uint64_t row_a,
                     uint32_t field_b, uint32_t view_b, uint64_t row_b, const uint64_t *shards, int64_t n_shards, uint64_t out_hist[16]);

/* GroupBy(Rows(f1), Rows(f2), ..., filter=...) with Count aggregate (executeGroupBy executor.go:3176,
 * executeGroupByShard :3918, groupByIterator :8617-8934; reduce = mergeGroupCounts :3728).  row_ids_flat holds
 * the per-field row-id lists concatenated (flat on purpose: cgo forbids nested Go pointers).  out_counts is
 * the dense count tensor, row-major, rightmost field fastest; the caller emits groups with Count>0 in
 * lexicographic order (executor.go:3960).  A shard lacking a fragment for any field contributes nothing
 * (executor.go:8769-8772).  All-reduced over the communicator. */
int fbgpu_groupby(fbgpu_ctx *ctx, uint32_t index, const uint32_t *fields, const uint32_t *views, int32_t n_fields,
                  const uint64_t *row_ids_flat, const int32_t *n_rows,
                  const fbgpu_op *filter, int32_t n_filter_ops,
                  const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
/* fbgpu_groupby with dimension i's rows taken as their unions over n_views[i] (>= 1) views of fields[i]: GroupBy(Rows(f,
 * from=, to=), ...) on time fields (timeFragmentsRowIterator executor.go:8755-8768).  The views of all dimensions are listed
 * one dimension after the other in views_flat.  Same dense output tensor (rightmost fastest) and all-reduce as fbgpu_groupby;
 * with every n_views[i] == 1 the result is fbgpu_groupby's.  A shard lacking a dimension's fragment in every listed view
 * contributes nothing.  Argument errors (n_fields outside 1..8, n_views[i] < 1, n_rows[i] outside 0..65535, null pointers)
 * are reported before the device check. */
int fbgpu_groupby_views(fbgpu_ctx *ctx, uint32_t index, const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views,
                        int32_t n_fields, const uint64_t *row_ids_flat, const int32_t *n_rows,
                        const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);

/* GroupBy whose last dimension is the values of an int field: GroupBy(Rows(f1), ..., Rows(v)) with v an int field, whose groups
 * are v's values (FieldRow.Value, executor.go:8740-8750), in one device pass instead of one Row(v == value) per value.
 * fields / views / row_ids_flat / n_rows: n_fields (0..7) set-like dimensions, as for fbgpu_groupby (may be NULL when
 * n_fields == 0).  vfield / vview / bit_depth (0..64): the int field's BSI view.  values: n_values (1..65535) strictly ascending
 * stored values (value - bsiGroup.Base, as fbgpu_extract reports them; at depth 64, INT64_MIN is stored as sign + 2^63).
 * out_counts: the dense tensor [n_rows[0]] ... [n_rows[n_fields-1]] [n_values], row-major, the int dimension last; entry
 * (i..., j) = |{columns of filter ∩ exists(v) ∩ Row(f1 = r1_i) ∩ ... whose stored value is values[j]}|.  A column whose value is
 * not listed is counted nowhere, nor is a column stored as sign with magnitude 0 (Row(v == 0) does not hold it).  A shard lacking
 * the int field's fragment or any set field's fragment contributes nothing (executor.go:8769-8772).  All-reduced over the
 * communicator. */
int fbgpu_groupby_values(fbgpu_ctx *ctx, uint32_t index, const uint32_t *fields, const uint32_t *views, int32_t n_fields,
                         const uint64_t *row_ids_flat, const int32_t *n_rows, uint32_t vfield, uint32_t vview, int32_t bit_depth,
                         const int64_t *values, int32_t n_values, const fbgpu_op *filter, int32_t n_filter_ops,
                         const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
/* GroupBy over set dimensions and one or more int dimensions in one device call: GroupBy(Rows(a), Rows(v), Rows(w)) (SQL GROUP BY
 * int_a, int_b) or GroupBy(Rows(t, from=, to=), Rows(v)).
 * fields / views_flat / n_views / row_ids_flat / n_rows: n_fields (0..7) set dimensions, as for fbgpu_groupby_views: dimension i
 * has n_views[i] >= 1 views and n_rows[i] (0..65535) rows, each row its union over those views (may be NULL when n_fields == 0).
 * vfields / vviews / bit_depths / values_flat / n_values: n_ints (1..8, n_fields + n_ints <= 8) int dimensions, each a BSI view of
 * depth 0..64 with n_values[k] (1..65535) strictly ascending stored values (as for fbgpu_groupby_values), listed one dimension
 * after the other in values_flat; the product of the n_values is at most 65535.
 * out_counts: the dense tensor [n_rows[0]] ... [n_rows[n_fields-1]] [n_values[0]] ... [n_values[n_ints-1]], row-major, set
 * dimensions first, rightmost fastest.  A column is counted in a cell when it is in the filter, in every set row of the cell, in
 * exists(v_k) of every int field and its stored value of every v_k is the listed one; sign with magnitude 0 is no value.  A shard
 * lacking any int field's fragment, or a set dimension's fragment in every listed view, contributes nothing.  All-reduced over
 * the communicator.  With n_ints == 1 and every n_views[i] == 1 the result is fbgpu_groupby_values'.  Argument errors other than
 * n_rows are reported before the device check; a counts workspace (rows of the last set dimension x groups x 8 bytes) that
 * cannot be allocated gives FBGPU_E_NOMEM. */
int fbgpu_groupby_mixed(fbgpu_ctx *ctx, uint32_t index,
                        const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                        const uint64_t *row_ids_flat, const int32_t *n_rows,
                        const uint32_t *vfields, const uint32_t *vviews, const int32_t *bit_depths, int32_t n_ints,
                        const int64_t *values_flat, const int32_t *n_values,
                        const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
/* GroupBy(..., aggregate=Sum(field=x)) in one device call (SQL SELECT a, SUM(x) ... GROUP BY a).
 * The dimensions are fbgpu_groupby_mixed's, except that n_fields is 0..8 and n_ints 0..8 with 1 <= n_fields + n_ints <= 8 (with
 * n_ints == 0 the int arrays may be NULL).  afield / aview / a_depth (0..64): the aggregate's BSI view and its depth.
 * out_counts / out_sums: tensors of fbgpu_groupby_mixed's shape and layout.  Per cell, out_counts = |cell ∩ filter ∩ exists(x)|
 * and out_sums = the sum of those columns' stored values of x (value - Base) in wrapping int64: for every cell the pair
 * fbgpu_bsi_sum returns under the filter `filter ∩ the cell's rows` (sign with magnitude 0 counts, with value 0; the caller adds
 * count x Base).  A shard lacking x's fragment contributes nothing; missing set or int fragments as for fbgpu_groupby_mixed.
 * Both tensors are all-reduced over the communicator as u64 sums.  Argument errors other than n_rows are reported before the
 * device check; a workspace (rows of the last set dimension x groups x 16 bytes) that cannot be allocated gives FBGPU_E_NOMEM. */
int fbgpu_groupby_sum(fbgpu_ctx *ctx, uint32_t index,
                      const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                      const uint64_t *row_ids_flat, const int32_t *n_rows,
                      const uint32_t *vfields, const uint32_t *vviews, const int32_t *bit_depths, int32_t n_ints,
                      const int64_t *values_flat, const int32_t *n_values, uint32_t afield, uint32_t aview, int32_t a_depth,
                      const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards,
                      uint64_t *out_counts, int64_t *out_sums);
/* GroupBy(..., aggregate=Count(Distinct(field=x))) in one device call (SQL SELECT a, COUNT(DISTINCT x) ... GROUP BY a).
 * The dimensions are fbgpu_groupby_sum's.  xfield / xview / x_depth (0..64): x's BSI view and its depth; x_values: n_x >= 1
 * strictly ascending stored values (value - Base) as fbgpu_extract reports them.  out_distinct: a tensor of
 * fbgpu_groupby_mixed's shape and layout.  Per cell, the number of listed x_values[j] that at least one column of
 * filter ∩ the cell's rows ∩ exists(x) holds as its stored value of x: the listed values among fbgpu_extract(x)'s values under
 * `filter ∩ the cell's rows`.  x's sign with magnitude 0 is the value 0 (as in fbgpu_extract), the int dimensions' is no
 * value (as in fbgpu_groupby_mixed); a column whose x value is not listed counts nowhere.  A shard lacking x's fragment
 * contributes nothing; missing set or int fragments as for fbgpu_groupby_mixed.  Argument errors other than n_rows are
 * reported before the device check; a presence workspace (rows of the last set dimension, or 1) x groups x ceil(n_x / 64)
 * x 8 bytes that cannot be allocated gives FBGPU_E_NOMEM.  A context with a communicator attached returns FBGPU_E_COMM:
 * distinct sets merge by union, not by the u64 sum the other GroupBy tensors are all-reduced with. */
int fbgpu_groupby_distinct(fbgpu_ctx *ctx, uint32_t index,
                           const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                           const uint64_t *row_ids_flat, const int32_t *n_rows,
                           const uint32_t *vfields, const uint32_t *vviews, const int32_t *bit_depths, int32_t n_ints,
                           const int64_t *values_flat, const int32_t *n_values,
                           uint32_t xfield, uint32_t xview, int32_t x_depth, const int64_t *x_values, int32_t n_x,
                           const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards,
                           uint64_t *out_distinct);
/* GroupBy(..., aggregate=Count(Distinct(field=x))) over a set, mutex, bool or time field x in one device call (SQL
 * SELECT a, COUNT(DISTINCT s) ... GROUP BY a over a string, id, stringset or idset column).  The dimensions, limits and
 * out_distinct's shape and layout are fbgpu_groupby_distinct's.  xfield / xview: a set-like view of x (executeDistinctShardSet
 * reads the standard view); x_rows: n_x >= 1 strictly ascending row ids, any u64.  Per cell, the number of listed rows x_rows[j]
 * for which filter ∩ the cell's rows ∩ Row(x = x_rows[j]) holds at least one column: the listed rows among those
 * fbgpu_row_counts(x, all rows) counts as non-zero under `filter ∩ the cell's rows`.  A column held by several listed rows
 * counts toward each of them; the data need not be mutex-shaped.  A shard lacking x's fragment contributes nothing; missing set
 * or int fragments as for fbgpu_groupby_mixed.  Argument errors other than n_rows (those of fbgpu_groupby_distinct, n_x < 1,
 * x_rows not strictly ascending) are reported before the device check; a presence workspace (rows of the last set dimension,
 * or 1) x groups x ceil(n_x / 64) x 8 bytes that cannot be allocated gives FBGPU_E_NOMEM.  A context with a communicator
 * attached returns FBGPU_E_COMM, as fbgpu_groupby_distinct does.  Device cost per 4,096-column range (16 per container
 * slot): one scan of x's row-directory entries whose ids lie between x_rows[0] and x_rows[n_x - 1], reading the containers of
 * the listed ones in the range, and one walk of the dimensions' last set field, plus one more of each for every further
 * listed row a column of the range holds. */
int fbgpu_groupby_distinct_rows(fbgpu_ctx *ctx, uint32_t index,
                                const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                                const uint64_t *row_ids_flat, const int32_t *n_rows,
                                const uint32_t *vfields, const uint32_t *vviews, const int32_t *bit_depths, int32_t n_ints,
                                const int64_t *values_flat, const int32_t *n_values,
                                uint32_t xfield, uint32_t xview, const uint64_t *x_rows, int32_t n_x,
                                const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards,
                                uint64_t *out_distinct);
/* GroupBy over set, mutex, bool or time dimensions of any size, as the sorted list of its non-empty groups (executeGroupBy's
 * walk of groupByIterator, with previous= and limit=).  The dimensions are fbgpu_groupby_views': 1..8, dimension i the rows
 * row_ids_flat[..n_rows[i]] of fields[i], each taken as its union over n_views[i] >= 1 views; the filter is optional.  n_rows[i]
 * may be 1..2^31-1, and each list must be strictly ascending; the product of the n_rows must fit in u64.  A cell is the
 * row-major flat index Σ idx_i · Π_{j>i} n_rows[j] of the dense tensor fbgpu_groupby_views would fill (the last dimension
 * fastest, the reference's iteration order), and its count is what that call would put there: |filter ∩ ⋂_i row_i|.
 * Output: the cells with a non-zero count and cell >= start, ascending, at most `limit` of them (limit < 0: no limit), into
 * out_cells / out_counts under fbgpu_columns' NOSPACE contract (cap too small: nothing written, FBGPU_E_NOSPACE, *out_n = the
 * size needed).  Argument errors (null pointers, n_fields outside 1..8, n_views < 1, n_rows < 1, a list not strictly ascending,
 * an overflowing product) are reported before the device check.  A context with a communicator attached returns FBGPU_E_COMM:
 * lists of cells do not all-reduce.  Device memory: 16 bytes per (column, listed row) hit of each dimension in a chunk of at
 * most 2^24 hits per dimension, 16 bytes per cell of a join range of at most 2^24 cells (one column's cross product may exceed
 * that), and 32 bytes per cell of the running list, which the limit bounds. */
int fbgpu_groupby_sparse(fbgpu_ctx *ctx, uint32_t index,
                         const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                         const uint64_t *row_ids_flat, const int32_t *n_rows,
                         const fbgpu_op *filter, int32_t n_filter_ops,
                         const uint64_t *shards, int64_t n_shards,
                         uint64_t start, int64_t limit,
                         uint64_t *out_cells, uint64_t *out_counts, uint64_t cap, uint64_t *out_n);
/* GroupBy(..., aggregate=Sum(field=x)) over fbgpu_groupby_sparse's dimensions, in one call.  Dimensions, cells, start, limit
 * and the NOSPACE contract are fbgpu_groupby_sparse's.  x: the int field afield, its BSI view aview and bit depth a_depth
 * (0..64).  Per listed cell, out_counts = |filter ∩ the cell's rows ∩ exists(x)| and out_sums = the wrapping int64 sum of those
 * columns' stored values of x (value - Base): the pair fbgpu_groupby_sum puts in that cell, and the pair fbgpu_bsi_sum returns
 * under `filter ∩ the cell's rows`.  A sign with magnitude 0 counts, with value 0.  The caller adds count x Base.  A cell is
 * listed when that count is non-zero, so a group whose columns hold no value of x is absent (the reference skips a group whose
 * Sum count is 0), and `limit` counts listed cells.  A shard lacking x's fragments contributes nothing.  Argument errors
 * (fbgpu_groupby_sparse's, a_depth outside 0..64, a null out_sums with cap > 0) are reported before the device check.  A context
 * with a communicator attached returns FBGPU_E_COMM.  Device memory: fbgpu_groupby_sparse's bounds, with a chunk also holding
 * at most 2^24 columns of filter ∩ exists(x), which take about 16 bytes each (column and magnitude, plus a sign bit); 32 bytes
 * instead of 16 per (cell, value) pair of a join range of at most 2^24 pairs; and 64 bytes instead of 32 per cell of the
 * running list, whose sums are a second list beside the counts. */
int fbgpu_groupby_sparse_sum(fbgpu_ctx *ctx, uint32_t index,
                             const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                             const uint64_t *row_ids_flat, const int32_t *n_rows,
                             uint32_t afield, uint32_t aview, int32_t a_depth,
                             const fbgpu_op *filter, int32_t n_filter_ops,
                             const uint64_t *shards, int64_t n_shards, uint64_t start, int64_t limit,
                             uint64_t *out_cells, uint64_t *out_counts, int64_t *out_sums, uint64_t cap, uint64_t *out_n);
/* GroupBy(..., aggregate=Count(Distinct(field=x))) over set-like dimensions of any size, in one call (SQL SELECT k,
 * COUNT(DISTINCT x) ... GROUP BY k over a column of more than 65,535 values).  Dimensions and cells are fbgpu_groupby_sparse's,
 * but at most 7 dimensions: x takes the eighth place of the join.  xfield / xview / x_depth (0..64): x's BSI view and depth;
 * x_values: n_x >= 1 strictly ascending stored values (value - Base), as for fbgpu_groupby_distinct.  For every cell in
 * [start, end), the number of listed x_values[j] held by at least one column of filter ∩ the cell's rows ∩ exists(x) (a sign
 * with magnitude 0 is the value 0; a column whose value is not listed counts nowhere).  Only the cells where that number is
 * non-zero are written, ascending, into out_cells / out_distinct under fbgpu_columns' NOSPACE contract.  Where the dense tensor
 * fits, these are the non-zero cells of fbgpu_groupby_distinct.  Argument errors (fbgpu_groupby_sparse's with out_distinct in
 * the place of out_counts, n_fields > 7, n_x < 1, x_values not strictly ascending, x_depth outside 0..64, start > end, a
 * product of n_rows that does not fit in u64 once shifted left by bit_width(n_x - 1)) are reported before the device check.  A
 * context with a communicator attached returns FBGPU_E_COMM: distinct sets merge by union.  There is no node form.  Device
 * memory: fbgpu_groupby_sparse_sum's bounds per chunk (its value list, and 16 bytes per listed value a column holds); 16 bytes
 * per (cell, x) pair of a join range of at most 2^24 pairs (one column's cross product may exceed that); 16 bytes per
 * distinct (cell, x) pair of the running list, which has no limit: a caller bounds it by the range and x's list (the pairs
 * are at most Σ over the range's cells of min(count, n_x)); and at the end 32 bytes per listed cell. */
int fbgpu_groupby_sparse_distinct(fbgpu_ctx *ctx, uint32_t index,
                                  const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                                  const uint64_t *row_ids_flat, const int32_t *n_rows,
                                  uint32_t xfield, uint32_t xview, int32_t x_depth, const int64_t *x_values, int32_t n_x,
                                  const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards,
                                  uint64_t start, uint64_t end,
                                  uint64_t *out_cells, uint64_t *out_distinct, uint64_t cap, uint64_t *out_n);
/* The same over a set, mutex, bool or time field x: xfield / xview a set-like view of x, x_rows n_x >= 1 strictly ascending
 * row ids (any u64).  Per cell in [start, end), the number of listed rows x_rows[j] that hold at least one column of
 * filter ∩ the cell's rows; a column held by several listed rows counts toward each of them.  Where the dense tensor fits,
 * these are the non-zero cells of fbgpu_groupby_distinct_rows.  Argument errors as for fbgpu_groupby_sparse_distinct (x_rows
 * not strictly ascending in the place of x_values; no depth), and FBGPU_E_COMM alike.  Device memory: fbgpu_groupby_sparse's
 * per chunk, x counted as one more dimension, then as for fbgpu_groupby_sparse_distinct from the join on. */
int fbgpu_groupby_sparse_distinct_rows(fbgpu_ctx *ctx, uint32_t index,
                                       const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                                       const uint64_t *row_ids_flat, const int32_t *n_rows,
                                       uint32_t xfield, uint32_t xview, const uint64_t *x_rows, int32_t n_x,
                                       const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards,
                                       uint64_t start, uint64_t end,
                                       uint64_t *out_cells, uint64_t *out_distinct, uint64_t cap, uint64_t *out_n);

/* ---- multi-GPU reduce (replaces the HTTP fan-in of mapReduce/remoteExec, executor.go:6392-6533) ----
 * One context (process) per GPU; rank 0 creates the id, every rank joins.  When a communicator is attached,
 * count / row_counts / groupby results are summed with one ncclAllReduce(uint64,sum) on the device before
 * the single D2H copy.  NCCL is resolved at run time (dlopen libnccl.so.2). */
#define FBGPU_NCCL_ID_BYTES 128
int fbgpu_comm_unique_id(uint8_t id[FBGPU_NCCL_ID_BYTES]);
int fbgpu_comm_init(fbgpu_ctx *ctx, int32_t n_ranks, int32_t rank, const uint8_t id[FBGPU_NCCL_ID_BYTES]);
int fbgpu_comm_destroy(fbgpu_ctx *ctx);
/* Fused Count merge over NVLink peer memory (optional, Count only): every rank exports a small mailbox through CUDA IPC
 * (fbgpu_comm_p2p_handle), the host exchanges the 64-byte handles (any transport), every rank maps its peers
 * (fbgpu_comm_p2p_open).  From then on fbgpu_count() sums the per-GPU totals inside the counting kernel itself (last CTA
 * stores to all peers' mailboxes, waits for theirs) instead of launching a separate all-reduce. */
int fbgpu_comm_p2p_handle(fbgpu_ctx *ctx, uint8_t out_handle[64]);
int fbgpu_comm_p2p_open(fbgpu_ctx *ctx, int32_t n_ranks, int32_t rank, const uint8_t *handles /* n_ranks x 64 bytes */);
int fbgpu_comm_p2p_disable(fbgpu_ctx *ctx);   /* fall back to the NCCL merge (e.g. when a peer could not be mapped) */

/* In-process form of the same exchange: the contexts of ONE process (one per GPU, one caller thread each) are wired to each
 * other through peer access instead of CUDA IPC.  ctxs[r] becomes rank r. */
int fbgpu_comm_p2p_open_local(fbgpu_ctx *const *ctxs, int32_t n_ranks);
/* The wait for a peer's count inside the kernel is bounded (FBGPU_P2P_TIMEOUT_MS, default 2000): a peer that died, or ranks
 * that issued their collective queries in different orders, make fbgpu_count() return FBGPU_E_COMM instead of hanging the GPU.
 * The multi-process forms keep NCCL's precondition: every rank issues its collective queries in the same order, from one thread
 * at a time.  A process whose threads query concurrently (FeatureBase: executor.go:6449-6533) uses fbgpu_node below. */

/* ---- every GPU of one process behind one handle (SURVEY §8(b) fbgpu_init(device_ordinals, n); replaces mapReduce's local
 *      fan-out + reduce, executor.go:6449-6533, 6742-6812) ----
 * A node owns one context per listed device.  Shard s lives on device slot (s / shard_block) % n_devices: contiguous blocks of
 * shard_block shards per GPU (SURVEY §8(e); shard_block = ceil(total shards / n_devices) gives one range per GPU).  Every
 * fbgpu_node_* query takes the caller's whole shard list, runs each device's share concurrently on that device (own worker
 * thread, stream and workspace per call) and merges the per-device results on the host with the reference's reducers (u64
 * add: Count executor.go:5880, Pairs.Add cache.go:464, mergeGroupCounts executor.go:3728; Row.Merge row.go:202).  Any number
 * of threads may call concurrently; calls never share result buffers, and a failure on one device fails only that call.
 * The same device ordinal may be listed more than once (two contexts on one GPU; used by the tests). */
typedef struct fbgpu_node fbgpu_node;
int fbgpu_node_init(const int32_t *device_ordinals, int32_t n_devices, uint64_t shard_block, fbgpu_node **out);
void fbgpu_node_shutdown(fbgpu_node *node);
int32_t fbgpu_node_devices(const fbgpu_node *node);
int32_t fbgpu_node_owner(const fbgpu_node *node, uint64_t shard);      /* device slot that holds the shard */
fbgpu_ctx *fbgpu_node_ctx(fbgpu_node *node, int32_t slot);             /* the slot's context (stats, counters); owned by the node */
int fbgpu_node_load_fragment(fbgpu_node *node, uint32_t index, uint32_t field, uint32_t view, uint64_t shard,
                             const uint8_t *roaring, uint64_t nbytes);
int fbgpu_node_load_fragments(fbgpu_node *node, uint32_t index, uint32_t field, uint32_t view,
                              const uint64_t *shards, int64_t n, const uint8_t *buf, const uint64_t *offsets);
int fbgpu_node_load_rbf_dir(fbgpu_node *node, uint32_t index, uint64_t shard, const char *dir, const char *const *names,
                            const uint32_t *fields, const uint32_t *views, int32_t n_names, int32_t *out_loaded);
int fbgpu_node_drop_fragment(fbgpu_node *node, uint32_t index, uint32_t field, uint32_t view, uint64_t shard);
int fbgpu_node_apply_containers(fbgpu_node *node, uint32_t index, uint32_t field, uint32_t view, uint64_t shard,
                                const uint8_t *roaring, uint64_t nbytes, const uint64_t *removed_keys, int64_t n_removed);
int fbgpu_node_commit(fbgpu_node *node);
int fbgpu_node_get_stats(fbgpu_node *node, fbgpu_stats *out);           /* summed over the devices */
/* same contracts as the fbgpu_* calls of the same name, over all devices */
int fbgpu_node_count(fbgpu_node *node, uint32_t index, const fbgpu_op *ops, int32_t n_ops,
                     const uint64_t *shards, int64_t n_shards, uint64_t *out_total, uint64_t *out_per_shard);
int fbgpu_node_any(fbgpu_node *node, uint32_t index, const fbgpu_op *ops, int32_t n_ops,
                   const uint64_t *shards, int64_t n_shards, int32_t *out_any);
int fbgpu_node_row(fbgpu_node *node, uint32_t index, const fbgpu_op *ops, int32_t n_ops,
                   const uint64_t *shards, int64_t n_shards, uint8_t *out_buf, uint64_t out_cap, uint64_t *out_len, uint64_t *out_count);
int fbgpu_node_count_pairs(fbgpu_node *node, uint32_t index, uint32_t field_a, uint32_t view_a, const uint64_t *rows_a,
                           uint32_t field_b, uint32_t view_b, const uint64_t *rows_b, int32_t n_pairs,
                           const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
int fbgpu_node_row_counts(fbgpu_node *node, uint32_t index, uint32_t field, uint32_t view, const uint64_t *row_ids, int32_t n_rows,
                          const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
int fbgpu_node_row_counts_views(fbgpu_node *node, uint32_t index, uint32_t field, const uint32_t *views, int32_t n_views,
                                const uint64_t *row_ids, int32_t n_rows, const fbgpu_op *filter, int32_t n_filter_ops,
                                const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
/* both forms; all rows: each device's list merged by row id with the totals summed, then sorted (a shard lives on one device) */
int fbgpu_node_topn_cutoffs(fbgpu_node *node, uint32_t index, uint32_t field, uint32_t view,
                            const uint64_t *row_ids, int32_t n_rows, const fbgpu_op *src, int32_t n_src_ops,
                            uint64_t min_threshold, uint32_t tanimoto_threshold, const uint64_t *shards, int64_t n_shards,
                            uint64_t *out_row_ids, uint64_t *out_counts, int32_t cap, int32_t *out_n);
int fbgpu_node_groupby_views(fbgpu_node *node, uint32_t index, const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views,
                             int32_t n_fields, const uint64_t *row_ids_flat, const int32_t *n_rows,
                             const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
int fbgpu_node_groupby(fbgpu_node *node, uint32_t index, const uint32_t *fields, const uint32_t *views, int32_t n_fields,
                       const uint64_t *row_ids_flat, const int32_t *n_rows, const fbgpu_op *filter, int32_t n_filter_ops,
                       const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
int fbgpu_node_groupby_values(fbgpu_node *node, uint32_t index, const uint32_t *fields, const uint32_t *views, int32_t n_fields,
                              const uint64_t *row_ids_flat, const int32_t *n_rows, uint32_t vfield, uint32_t vview, int32_t bit_depth,
                              const int64_t *values, int32_t n_values, const fbgpu_op *filter, int32_t n_filter_ops,
                              const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
int fbgpu_node_groupby_mixed(fbgpu_node *node, uint32_t index,
                             const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                             const uint64_t *row_ids_flat, const int32_t *n_rows,
                             const uint32_t *vfields, const uint32_t *vviews, const int32_t *bit_depths, int32_t n_ints,
                             const int64_t *values_flat, const int32_t *n_values,
                             const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards, uint64_t *out_counts);
int fbgpu_node_groupby_sum(fbgpu_node *node, uint32_t index,
                           const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                           const uint64_t *row_ids_flat, const int32_t *n_rows,
                           const uint32_t *vfields, const uint32_t *vviews, const int32_t *bit_depths, int32_t n_ints,
                           const int64_t *values_flat, const int32_t *n_values, uint32_t afield, uint32_t aview, int32_t a_depth,
                           const fbgpu_op *filter, int32_t n_filter_ops, const uint64_t *shards, int64_t n_shards,
                           uint64_t *out_counts, int64_t *out_sums);
int fbgpu_node_bsi_sum(fbgpu_node *node, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                       const uint64_t *shards, int64_t n_shards, int64_t *out_sum, uint64_t *out_count);
int fbgpu_node_bsi_minmax(fbgpu_node *node, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                          const uint64_t *shards, int64_t n_shards, int32_t want_max, int64_t *out_val, uint64_t *out_count);
int fbgpu_node_bsi_sort(fbgpu_node *node, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                        const uint64_t *shards, int64_t n_shards, int32_t desc, uint64_t offset, int64_t limit,
                        uint64_t *out_cols, int64_t *out_vals, uint64_t cap, uint64_t *out_n, uint64_t *out_total);
int fbgpu_node_bsi_distinct(fbgpu_node *node, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint32_t field, uint32_t view, int32_t bit_depth,
                            const uint64_t *shards, int64_t n_shards, int64_t *out_vals, uint64_t cap, uint64_t *out_n, uint64_t *out_total);
/* Every device lists its own shards' cells with the same start and limit; the lists merge by cell, counts summed, and the
 * window is cut after the merge (exact: a cell among the node's first K non-empty cells is among the first K of every device
 * where it is non-empty). */
int fbgpu_node_groupby_sparse(fbgpu_node *node, uint32_t index,
                              const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                              const uint64_t *row_ids_flat, const int32_t *n_rows, const fbgpu_op *filter, int32_t n_filter_ops,
                              const uint64_t *shards, int64_t n_shards, uint64_t start, int64_t limit,
                              uint64_t *out_cells, uint64_t *out_counts, uint64_t cap, uint64_t *out_n);
/* The same for fbgpu_groupby_sparse_sum: the lists merge by cell with counts and sums added (the sums wrap), and the window is
 * cut after the merge; exact for the same reason, since a cell is listed on a device exactly when its count there is non-zero. */
int fbgpu_node_groupby_sparse_sum(fbgpu_node *node, uint32_t index,
                                  const uint32_t *fields, const uint32_t *views_flat, const int32_t *n_views, int32_t n_fields,
                                  const uint64_t *row_ids_flat, const int32_t *n_rows,
                                  uint32_t afield, uint32_t aview, int32_t a_depth,
                                  const fbgpu_op *filter, int32_t n_filter_ops,
                                  const uint64_t *shards, int64_t n_shards, uint64_t start, int64_t limit,
                                  uint64_t *out_cells, uint64_t *out_counts, int64_t *out_sums, uint64_t cap, uint64_t *out_n);

/* Inspection (any context): the stack-machine program the library would run for `ops` -- records of 16 bytes {u8 op, u8 pad[3],
 * u32 view slot, u64 row} (csrc/fbgpu_types.h DevOp); *out_depth = operand stack depth.  With index == 0xffffffff,
 * fbgpu_debug_container() takes such a view slot in `field`. */
int fbgpu_debug_compile(fbgpu_ctx *ctx, uint32_t index, const fbgpu_op *ops, int32_t n_ops, uint8_t *out, int32_t cap_ops,
                        int32_t *out_n, int32_t *out_depth);

/* ---- instrumentation (the counters the reference keeps under the roaringstats tag, statsHit()) ---- */
typedef struct {
    uint64_t kernel_launches;   /* kernels of this library launched since init       */
    uint64_t queries;
    float last_query_gpu_ms;    /* CUDA-event time of the last query's kernels        */
    uint32_t pair_kernel_queries; /* Count(Intersect(Row, Row)) queries answered by the fused pair_count_kernel (low 32 bits) */
    uint64_t last_algo_bytes;   /* algorithmic bytes of the last query (SURVEY §8d)   */
    uint64_t groupby_units;     /* (shard, slot) units of GroupBy queries so far ...                          */
    uint64_t groupby_fallback_units; /* ... and how many of them the warp-per-unit kernel handed to the CTA kernel */
} fbgpu_counters;
int fbgpu_get_counters(fbgpu_ctx *ctx, fbgpu_counters *out);
/* algorithmic-bytes accounting (SURVEY §8d): roaring payload bytes and container count of the given rows (NULL = all
 * rows) of a field over the shards, from the host-side directory */
int fbgpu_rows_payload_bytes(fbgpu_ctx *ctx, uint32_t index, uint32_t field, uint32_t view, const uint64_t *row_ids, int32_t n_rows,
                             const uint64_t *shards, int64_t n_shards, uint64_t *out_payload, uint64_t *out_containers);
/* the CUDA stream queries of the calling thread run on (cudaStream_t), for external event timing */
void *fbgpu_stream(fbgpu_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif
