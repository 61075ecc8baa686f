/* rxgpu.h -- C ABI of librxgpu.so: the H100 (sm_90a) replacement for Reindexer's float_vector KNN hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  Every entry point names the reference interface it replaces
 * (paths relative to /root/reference/cpp_src).  Plain C: opaque handles, pointers and sizes only, no exceptions,
 * no torch types.  The C++ adapter reindexer_b200/host/gpu_bruteforce.h wraps these into the `Map` duck-type of
 * HnswIndexBase<Map> (core/index/float_vector/hnsw_index.h:13-57); INTEGRATION.md shows the 3-line patch.
 *
 * Conventions
 *  - return value: 0 = ok, otherwise a reindexer ErrorCode-compatible value (core/type_consts.h:136-181);
 *    rxgpu_last_error() returns the thread-local message (texts match the reference's where its tests match on them).
 *  - distances use the map-space sign convention of hnswlib::DistCalculator (hnswlib/hnswlib.h:147-165,192-197):
 *    L2 -> +L2^2, InnerProduct -> -IP, Cosine -> -IP(q^, v)/||v||; smaller is better.  Queries for Cosine must be
 *    pre-normalised by the caller (HnswIndexBase::search does it, core/index/float_vector/hnsw_index.cc:166-171) --
 *    rxgpu_select_knn() below does that step too.
 *  - labels are FloatVectorId::AsNumber() = rowId << 32 | arrayIdx (core/index/float_vector/float_vector_id.h:11).
 *  - threading: searches are re-entrant and may run concurrently from many host threads ("Read-only concurrency
 *    expected", hnswlib/hnswalg.h:1977); mutators are called by one thread at a time and never concurrently with
 *    searches on the same handle (the namespace lock guarantees that in the reference).  An HNSW streaming session
 *    is advanced by one thread at a time, though not always the same one; different sessions may run concurrently.
 *  - there is NO CPU fallback: every compute entry point fails with errSystem when no CUDA device is usable.
 */
#ifndef RXGPU_H
#define RXGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RXGPU_ABI_VERSION 4 /* 4: + rxgpu_comm_create_local, rxgpu_sharded_ft_select; filter variants 14..17; k <= 127 on the filter path */

/* subset of reindexer::ErrorCode (core/type_consts.h:136-181) that this library produces */
enum { RXGPU_OK = 0, RXGPU_ERR_PARAMS = 3, RXGPU_ERR_LOGIC = 4, RXGPU_ERR_NOT_FOUND = 13, RXGPU_ERR_SYSTEM = 37 };

/* reindexer::VectorMetric {L2, InnerProduct, Cosine} (core/enums.h:101) */
typedef enum { RXGPU_L2 = 0, RXGPU_IP = 1, RXGPU_COS = 2 } rxgpu_metric;

/* index creation flags */
enum {
	RXGPU_FLAG_HOST_MIRROR = 1u /* keep a host copy of the rows so rxgpu_index_get() returns a stable pointer
								   (BruteforceSearch::FloatPtrByExternalLabel, hnswlib/bruteforce.cc:36-42) */
};

typedef struct rxgpu_index rxgpu_index; /* one hnswlib::BruteforceSearch replacement = one shard on one GPU */

const char* rxgpu_last_error(void);
int rxgpu_abi_version(void);
/* number of usable CUDA devices (0 when there is no driver / GPU); never fails */
int rxgpu_device_count(void);

/* ---------------------------------------------------------------- lifetime / maintenance
 * BruteforceSearch(metric, dim, maxElements)                 hnswlib/bruteforce.cc:11-18 */
int rxgpu_index_create(rxgpu_index** out, rxgpu_metric metric, uint32_t dim, uint64_t capacity, int device, uint32_t flags);
/* BruteforceSearch(const BruteforceSearch&, newMaxElements)  hnswlib/bruteforce.cc:20-34 (deep copy; COW namespace clone) */
int rxgpu_index_clone(rxgpu_index** out, const rxgpu_index* src, uint64_t new_capacity);
void rxgpu_index_destroy(rxgpu_index*);
/* ResizeIndex                                                 hnswlib/bruteforce.cc:88-101 */
int rxgpu_index_resize(rxgpu_index*, uint64_t new_capacity);
/* AddPointNoLock (upsert by label)                            hnswlib/bruteforce.cc:44-64 */
int rxgpu_index_upsert(rxgpu_index*, uint64_t label, const float* vec /* dim floats, host */);
int rxgpu_index_upsert_batch(rxgpu_index*, uint64_t n, const uint64_t* labels, const float* vecs /* n x dim row-major, host */);
/* RemovePoint (swap-with-last compaction)                     hnswlib/bruteforce.cc:70-86 */
int rxgpu_index_remove(rxgpu_index*, uint64_t label);
/* FloatPtrByExternalLabel                                     hnswlib/bruteforce.cc:36-42
 * with RXGPU_FLAG_HOST_MIRROR the pointer stays valid until the row is modified; without it the row is fetched into a
 * thread-local buffer that the next rxgpu_index_get() on the same thread overwrites. */
int rxgpu_index_get(const rxgpu_index*, uint64_t label, const float** host_row);
uint64_t rxgpu_index_size(const rxgpu_index*);         /* CurrentElementCount() */
uint64_t rxgpu_index_capacity(const rxgpu_index*);     /* MaxElements() */
uint64_t rxgpu_index_element_size(const rxgpu_index*); /* ElementSize() = dim*4 + 8, asserted by the reference's memstat test */
uint64_t rxgpu_index_device_bytes(const rxgpu_index*); /* HBM held by this shard */
uint32_t rxgpu_index_dim(const rxgpu_index*);
int rxgpu_index_metric(const rxgpu_index*);
int rxgpu_index_device(const rxgpu_index*);

/* ---------------------------------------------------------------- search
 * BruteforceSearch::SearchKnn, batched                        hnswlib/bruteforce.cc:103-127
 * nq independent queries (the reference API is one query per call; nq > 1 is our extension, results identical to nq
 * calls).  Per query: rows sorted best->worst exactly as HnswIndexBase::select drains the reference's max-heap
 * (hnsw_index.cc:258-276), including the reference's tie rule (which of several bit-equal distances survive depends on
 * insertion order and label, SURVEY.md §8a rule 2).  out_count[q] = min(k, size).
 * The exact scan holds one query, zero padded to a multiple of 128 floats, and eight warp lists of min(k + 1, 256) + 32 keys in at
 * most 100 KB of shared memory: a search whose dimension and k exceed that fails with RXGPU_ERR_PARAMS.  At k = 10 the largest
 * dimension served is 24832; a larger k lowers it.  The tensor-core filter serves dimensions up to 2048 only. */
int rxgpu_search_knn(const rxgpu_index*, uint32_t nq, const float* queries /* nq x dim, host */, uint32_t k,
					 float* out_dist /* nq x k */, uint64_t* out_label /* nq x k */, uint32_t* out_count /* nq */);
/* BruteforceSearch::SearchRange (strict dist < radius)        hnswlib/bruteforce.cc:129-143
 * writes the best min(*out_n, max_out) results best-first; *out_n = total number of matches (may exceed max_out). */
int rxgpu_search_range(const rxgpu_index*, const float* query, float radius, uint64_t max_out, float* out_dist, uint64_t* out_label,
					   uint64_t* out_n);
/* BruteforceSearch::SearchRange for nq queries at once (our extension; the reference takes one query per call).
 * radius[q] is in map space, exactly as for rxgpu_search_range.  Per query q the result is identical to
 * rxgpu_search_range(queries + q*dim, radius[q], max_out, ...): out_n[q] = total matches, and the best
 * min(out_n[q], max_out) matches go best-first into row q of out_dist / out_label (nq x max_out).
 * A batch of >= 64 queries on >= 100k rows runs through the tensor-core candidate filter (rxgpu_set_tensor_core_filter), with up to
 * max(4096, 2 * min(max_out, 131072)) candidates per query; a query with more is answered by the exact scan (tc_fallbacks).
 * Does not change the result that rxgpu_last_range_results returns. */
int rxgpu_search_range_batch(const rxgpu_index*, uint32_t nq, const float* queries /* nq x dim, host */,
							 const float* radius /* nq */, uint64_t max_out,
							 float* out_dist, uint64_t* out_label, uint64_t* out_n /* nq */);

/* The result of this thread's last rxgpu_search_range stays retained in the library: entries [offset, offset + n) of it (best first),
 * so a caller that sized its buffers too small fetches the rest WITHOUT a second scan of the rows. */
int rxgpu_last_range_results(uint64_t offset, uint64_t n, float* out_dist, uint64_t* out_label);

/* Same scan with queries and outputs resident in HBM (device pointers), enqueued on `stream` (a cudaStream_t; NULL =
 * the library's own stream).  Used by the benchmark's device-resident leg and by the multi-GPU shard merge.
 * Outputs hold the top-k1 rows per query under the total order (distance, internal row index): out_idx is the shard-local
 * internal index (insertion order with swap-deletes, as in the reference).  No tie replay is applied here. */
int rxgpu_search_knn_device(const rxgpu_index*, uint32_t nq, const float* d_queries, uint32_t k1, float* d_out_dist,
							uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count, void* stream);
/* rows with dist <= dstar (a float compare: -0 == +0) in internal order: the first k of them (device in/out, one query); feeds the
 * tie replay.  *d_out_count = min(k, number of such rows); d_out_* hold k entries, of which the first *d_out_count are written. */
int rxgpu_search_tie_rows_device(const rxgpu_index*, const float* d_query, float dstar, uint32_t k, float* d_out_dist,
								 uint32_t* d_out_idx, uint64_t* d_out_label, uint32_t* d_out_count, void* stream);

/* ---------------------------------------------------------------- shard merge (multi-GPU row of SURVEY.md §8e)
 * Host-side, deterministic.  Inputs: nshards lists per query, each the output of rxgpu_search_knn_device copied to the host
 * (k1 = k + 1 entries so that a tie at the k-th place is visible), shard s holding global rows [base[s], base[s+1]).
 * Output: global top-k under (distance, global row index) and need_tie[q] != 0 where the reference's tie rule must be
 * replayed with rxgpu_tie_replay(). */
int rxgpu_merge_shards(uint32_t nshards, uint32_t nq, uint32_t k, uint32_t k1, const float* dist /* nshards x nq x k1 */,
					   const uint32_t* idx, const uint64_t* label, const uint32_t* count /* nshards x nq */,
					   const uint64_t* shard_base /* nshards */, float* out_dist /* nq x k */, uint64_t* out_gidx,
					   uint64_t* out_label, uint32_t* out_count, uint8_t* need_tie /* nq */);
/* The reference's heap tie rule in closed form (SURVEY.md §8a rule 2; derivation in DESIGN.md):
 *  lower   = the m < k rows with dist < dstar (global index + label), from the merged top-k
 *  first   = the first min(k, .) rows in global internal order with dist <= dstar (from rxgpu_search_tie_rows_device,
 *            merged over shards by global index)
 * writes the k survivors best-first into out_*. */
int rxgpu_tie_replay(uint32_t k, float dstar, uint32_t n_lower, const float* lower_dist, const uint64_t* lower_gidx,
					 const uint64_t* lower_label, uint32_t n_first, const float* first_dist, const uint64_t* first_gidx,
					 const uint64_t* first_label, float* out_dist, uint64_t* out_label, uint32_t* out_count);

/* ---------------------------------------------------------------- multi-GPU: one shard per GPU / rank, NCCL exchange, device merge
 * The sharded equivalent of BruteforceSearch::SearchKnn over the concatenation of all shards (shard r holds the global internal rows
 * [base_r, base_r + size_r), rows are appended shard by shard): ONE call per rank does the local fused scan + top-(k+1), one
 * ncclAllGather of the per-shard lists (NVLink / NVSwitch), a device-side k-way merge under (distance, global row), and -- only when
 * bit-equal distances straddle the k-th place -- the reference's heap tie rule replayed globally from the filter's candidate lists
 * (no second pass over any shard) with a second, tiny all-gather.  Every rank gets the same answer, identical to what the reference
 * returns for one index holding all rows.  NCCL is loaded with dlopen("libnccl.so.2") at the first rxgpu_comm_* call.
 * Bootstrap: rank 0 calls rxgpu_comm_unique_id and ships the 128 bytes to the other ranks by any channel (Reindexer's own RPC; the
 * tests use torch.distributed), then every rank calls rxgpu_comm_create.  nranks == 1 needs no id and no NCCL. */
#define RXGPU_COMM_ID_BYTES 128
typedef struct rxgpu_comm rxgpu_comm;
int rxgpu_comm_unique_id(void* out_id /* RXGPU_COMM_ID_BYTES */);
int rxgpu_comm_create(rxgpu_comm** out, int nranks, int rank, const void* id /* RXGPU_COMM_ID_BYTES, or NULL when nranks == 1 */, int device);
/* the ranks of ONE process (a reindexer process that drives several GPUs: one host thread per rank; the devices may repeat, which is
 * how a one-GPU box exercises the cross-shard paths): out[0..nranks) receive the communicators, rank r on devices[r] (NULL = all on
 * device 0).  Their exchanges go through host memory behind a rendezvous; every rank must make the same collective calls, each from its
 * own thread.  Serves rxgpu_sharded_search_knn, rxgpu_sharded_search_range_batch, rxgpu_sharded_ft_select, rxgpu_sharded_ivf_train,
 * rxgpu_sharded_ivf_search_knn and rxgpu_sharded_ivf_search_range_batch. */
int rxgpu_comm_create_local(rxgpu_comm** out, int nranks, const int* devices);
void rxgpu_comm_destroy(rxgpu_comm*);
int rxgpu_comm_rank(const rxgpu_comm*);
int rxgpu_comm_size(const rxgpu_comm*);
/* collective: every rank calls it with its own shard and the SAME queries / k.  queries: nq x dim floats, host pointer
 * (queries_on_device == 0) or device pointer on the shard's GPU (!= 0).  Outputs: host buffers nq x k, best first, reference tie rule
 * applied globally; out_count[q] = min(k, total rows).  k must be at most 65535 even when all shards together hold fewer rows (a rank
 * does not know the others' sizes before it scans; rxgpu_search_knn clamps k to its size first): a larger k fails with
 * RXGPU_ERR_PARAMS. */
int rxgpu_sharded_search_knn(rxgpu_comm*, const rxgpu_index* shard, uint32_t nq, const float* queries, int queries_on_device, uint32_t k,
							 float* out_dist, uint64_t* out_label, uint32_t* out_count);
/* collective: every rank calls it with its own shard and the SAME queries / radius / max_out.  Per query q the result on EVERY rank is
 * identical to rxgpu_search_range_batch on one index holding the rows of all shards: out_n[q] = total matches over all shards, and the
 * best min(out_n[q], max_out) matches, best first in the order of hitLessByLabel (distance, then label), go into row q of
 * out_dist / out_label (nq x max_out, host); the rest of a row may be overwritten.  queries: host (queries_on_device == 0) or device
 * pointer on the shard's GPU; radius: host, map space.  Labels must be unique across the shards (they are the rows of one namespace).
 * Each shard runs rxgpu_search_range_batch's local part (filter or exact scan, its own choice); the ranks then all-reduce the totals,
 * all-gather up to min(matches, max_out) best matches per query and shard, and merge them on the device (DESIGN.md §7). */
int rxgpu_sharded_search_range_batch(rxgpu_comm*, const rxgpu_index* shard, uint32_t nq, const float* queries, int queries_on_device,
									 const float* radius /* nq */, uint64_t max_out, float* out_dist, uint64_t* out_label, uint64_t* out_n);
/* the device-side merge alone: d_payloads = nshards contributions of rxgpu_shard_payload_bytes(nq, k1) bytes each, laid out as
 * [dist f32 nq*k1][idx u32 nq*k1][label u64 nq*k1][count u32 nq][shard size u64] (sections 16-byte aligned) -- what
 * rxgpu_search_knn_device writes; outputs (device) as rxgpu_merge_shards, ties NOT yet ordered by label. */
uint64_t rxgpu_shard_payload_bytes(uint32_t nq, uint32_t k1);
int rxgpu_merge_shards_device(uint32_t nshards, uint32_t nq, uint32_t k, uint32_t k1, const void* d_payloads, float* d_out_dist,
							  uint64_t* d_out_gidx, uint64_t* d_out_label, uint32_t* d_out_count, uint8_t* d_need_tie, void* stream);

/* ---------------------------------------------------------------- FloatVectorIndex::Select equivalent
 * HnswIndexBase<BruteforceSearch>::search + select/selectRaw   core/index/float_vector/hnsw_index.cc:160-191, 206-229, 232-288
 * query normalisation for Cosine (tools/normalize.h:16-22), k and/or radius, worst->best drain, sign flip for IP/Cosine,
 * ascending row ids inside runs of equal rank when need_sort (KnnCtx::NeedSort), array-field dedup by rowId
 * (float_vector_index.h:141-160) and removeOverK (:194-203). */
typedef struct {
	uint32_t k;           /* 0 = not set */
	int has_radius;       /* params.Radius() or the index-level radius */
	float radius;         /* user-space: squared distance for L2, similarity for IP / Cosine */
	int need_sort;        /* KnnCtx::NeedSort() */
	int is_array;         /* index over an array field */
	int raw;              /* selectRaw(): no tie sort */
} rxgpu_select_params;
int rxgpu_select_knn(const rxgpu_index*, const float* query /* dim floats, NOT normalised */, const rxgpu_select_params*,
					 uint64_t max_out, int32_t* out_row_ids, float* out_ranks, uint64_t* out_n);
/* the post-processing step alone, on the host (no device involved): `dist` / `label` = a map's answer best-first in map space (what
 * SearchKnn / SearchRange return after the worst->best drain); writes at most n rows.  Used by adapters that get their hits elsewhere
 * (a sharded search, an HNSW or IVF map) and pinned against the reference's own select code by tests/test_select_pin.py. */
int rxgpu_select_postprocess(int metric, const rxgpu_select_params*, uint64_t n, const float* dist, const uint64_t* label, int32_t* out_row_ids,
							 float* out_ranks, uint64_t* out_n);

/* ---------------------------------------------------------------- HNSW search on a reference-built graph
 * hnswlib::HierarchicalNSWImpl<float>::SearchKnn                core/index/float_vector/hnswlib/hnswalg.h:1978-2012
 *   = getLayer0EntryPoint (:799-827) + searchBaseLayerST<bareBone> (:829-975) + trim to k + internal id -> label.
 * The graph is built by the reference's own CPU code (insert stays on the CPU, SURVEY.md §8a a9) and imported here: internal id i
 * of the graph must be row i of this index (same insertion order, no deleted nodes).  Layout of the arrays = what
 * hnswalg.h:221-228 / :1034-1040 store per element, de-interleaved:
 *   level0        n x (1 + maxM0) u32   [count | neighbour ids ...]           (get_linklist0)
 *   levels        n i32                 element_levels_
 *   upper_offsets (n + 1) i64           slot of the element's level-1 list; levels 1..L are consecutive slots
 *   upper         slots x (1 + M) u32   [count | neighbour ids ...]           (get_linklist(id, level)) */
typedef struct {
	uint32_t n;
	uint32_t M;
	uint32_t maxM0;
	int32_t maxlevel;
	uint32_t enterpoint;
	uint64_t upper_slots;
	const uint32_t* level0;
	const int32_t* levels;
	const int64_t* upper_offsets;
	const uint32_t* upper;
} rxgpu_hnsw_graph;
int rxgpu_hnsw_import(rxgpu_index*, const rxgpu_hnsw_graph* graph);
/* nq independent searches, one warp each.  ef == 0 -> k*3/2 like hnswalg.h:1995.  Queries pre-normalised for Cosine.
 * Results best-first in map space, ties by label; out_count[q] <= min(k, ef, n).  stats (may be NULL): per query
 * [distance computations, hops] -- the reference's metric_distance_computations / metric_hops (hnswalg.h:250-251). */
int rxgpu_hnsw_search_knn(const rxgpu_index*, uint32_t nq, const float* queries /* host */, uint32_t k, uint32_t ef, float* out_dist,
						  uint64_t* out_label, uint32_t* out_count, uint32_t* stats /* nq x 2 or NULL */);
int rxgpu_hnsw_search_knn_device(const rxgpu_index*, uint32_t nq, const float* d_queries, uint32_t k, uint32_t ef, float* d_out_dist,
								 uint32_t* d_out_idx, uint32_t* d_out_count, uint32_t* d_stats /* nq x 2 or NULL */, void* stream);

/* Restores a graph from the reference's HNSW index cache without building a host graph (SURVEY f4).  The byte stream is what
 * HierarchicalNSWImpl::SaveIndex writes (hnswalg.h:1213-1263) and the loader constructor reads (:297-403): header (max elements, count,
 * max level, enter point, M, efConstruction), per element the level-0 list + either the primary key (alive) or the vector (deleted),
 * then per element the blob of its upper-level lists.  Tokens are pulled through callbacks that mirror hnswlib::IReader
 * (hnswlib.h; implemented by HnswIndexBase's Reader over the storage blob and the namespace's primary keys, hnsw_index.cc:455-483).
 * The index must be empty with capacity >= the element count; rows, labels (tombstones get a label of their own), lists and
 * tombstone bits are uploaded as they are decoded.  get_vstring returns non-zero on failure; the views stay valid until the next call. */
typedef struct {
	void* ctx;
	uint64_t (*get_var_uint)(void* ctx);
	int64_t (*get_var_int)(void* ctx);
	int (*get_vstring)(void* ctx, const char** data, uint64_t* len);
	uint64_t (*read_pk_encoded_data)(void* ctx, float* dest /* dim floats */); /* IReader::ReadPkEncodedData: returns the label */
} rxgpu_hnsw_cache_reader;
typedef struct {
	uint64_t max_elements, count;
	int32_t maxlevel;
	uint32_t enterpoint, M, ef_construction, deleted;
} rxgpu_hnsw_cache_info;
int rxgpu_hnsw_load_index_cache(rxgpu_index*, const rxgpu_hnsw_cache_reader* reader, rxgpu_hnsw_cache_info* info /* or NULL */);
/* Incremental maintenance of the imported graph after the reference's inserter added a point (HierarchicalNSWImpl::addPoint,
 * hnswalg.h:1695-1852): the caller passes the nodes whose lists changed -- the new node (with its vector and label; a tombstoned slot
 * that was reused for another vector counts as new) and the neighbours it was linked to -- and the graph's current top level and
 * enter point.  The device copy is patched in place: O(M) small copies per upsert instead of a re-import.  New nodes must arrive in
 * internal-id order; capacity is what the index had at import (rxgpu_index_resize + re-import beyond it: errLogic). */
typedef struct {
	uint32_t node;          /* internal id */
	int32_t level;          /* element_levels_[node] */
	const uint32_t* level0; /* 1 + maxM0: [count | neighbour ids] */
	const uint32_t* upper;  /* level x (1 + M), or NULL when level == 0 */
	const float* vec;       /* dim floats for a new / reused node, NULL for a node whose lists only were rewritten */
	uint64_t label;         /* with vec */
	int deleted;            /* IsMarkedDeleted(node) */
} rxgpu_hnsw_node_update;
int rxgpu_hnsw_update(rxgpu_index*, int32_t maxlevel, uint32_t enterpoint, uint32_t nupdates, const rxgpu_hnsw_node_update* updates);
uint64_t rxgpu_hnsw_update_count(const rxgpu_index*); /* nodes patched in place since the import */
/* HierarchicalNSWImpl::MarkDelete (hnswalg.h:1303-1335): the row stays in the graph as a tombstone -- searches traverse it but never
 * return it (searchBaseLayerST<bare_bone = false>, :829-975).  Errors: label unknown (errNotFound), already deleted (errLogic).
 * A search that meets more than 4096 deleted nodes waiting for expansion at once fails with errLogic (rebuild the graph). */
int rxgpu_hnsw_mark_deleted(rxgpu_index*, uint64_t label);
uint64_t rxgpu_hnsw_deleted_count(const rxgpu_index*); /* DeletedCountUnsafe */
/* ---------------------------------------------------------------- HNSW graph construction on the device
 * Replaces HierarchicalNSWImpl::addPoint (hnswalg.h:1695-1852) as the transaction path reaches it through AddPointConcurrent: rows
 * [first, n) of the index (n = rxgpu_index_size) are inserted into the graph over rows [0, first) -- none when first == 0, else the graph
 * of rxgpu_hnsw_import, rxgpu_hnsw_load_index_cache or an earlier build -- by a deterministic batched insertion (DESIGN.md §3.8):
 * the batches of rxgpu_hnsw_build_plan; every row of a batch does the greedy descent, searchBaseLayer with ef = efConstruction and
 * getNeighborsByHeuristic2 with M against the graph as the batch began; then the selected neighbours receive their reverse links, a
 * list that overflows Mcurmax being pruned once per batch with the heuristic.  Equal distances are ordered by row id.
 * levels: n - first levels, or NULL to draw them as getRandomLevel does (hnswalg.h:625-635): std::default_random_engine seeded with
 * `seed` (the adapter's 100), one draw per row in row order -- with first == 0 these are the reference's element_levels_.
 * M in [2, 32], efConstruction in [4, 1024] and a dimension the search kernel serves at that ef (errParams otherwise, and for first
 * other than the graph's node count, a graph of another M or negative levels); errLogic when the graph has tombstones, or when a
 * row it covers was rewritten or moved (an upsert of an existing label, a remove) since it was imported, built or patched; errSystem
 * when the workspace does not fit.  On any error the index and its graph are unchanged.  The graph left behind is searched by every
 * rxgpu_hnsw_* call without an import. */
typedef struct {
	uint64_t batches, rows;
	uint64_t distances;      /* distance evaluations (the reference's metric_distance_computations, summed over the inserts) */
	uint64_t reverse_links;  /* links written to the lists of the selected neighbours */
	uint64_t lists_pruned;   /* neighbour lists pruned with the heuristic (one per overflowing list and batch) */
	float search_select_ms;  /* CUDA-event times: the descent, searches and neighbour selection of every row */
	float sort_ms;           /* the sort of the reverse links */
	float link_ms;           /* appending and pruning the lists that receive them */
} rxgpu_hnsw_build_stats;
int rxgpu_hnsw_build(rxgpu_index*, uint32_t M, uint32_t ef_construction, uint64_t first, const int32_t* levels /* n - first or NULL */,
					 uint64_t seed, rxgpu_hnsw_build_stats* stats /* or NULL */);
/* The batches of rxgpu_hnsw_build, on the host: rows [first, n) onto a graph whose top level is maxlevel (-1 exactly when first == 0).
 * out_ends[b] = the end of batch b (at most n - first of them), *out_nbatches = their number; out_levels (n - first, or NULL) = the
 * levels used (drawn when levels is NULL, as rxgpu_hnsw_build draws them). */
int rxgpu_hnsw_build_plan(uint32_t M, uint64_t first, uint64_t n, int32_t maxlevel, const int32_t* levels, uint64_t seed,
						  int32_t* out_levels, uint64_t* out_ends, uint64_t* out_nbatches);
/* Reads the device graph back in the layout of rxgpu_hnsw_graph for nodes[0, nnodes) (NULL: nodes 0 .. nnodes-1).  level0:
 * nnodes x (1 + maxM0); levels: nnodes; upper_offsets: nnodes + 1 slots into `upper`, which receives the nodes' upper-level lists in
 * order (upper_offsets[nnodes] x (1 + M)).  Every output may be NULL (ask for upper_offsets first to size `upper`); info (or NULL)
 * receives n, M, maxM0, maxlevel, enterpoint and upper_slots with NULL arrays.  With nodes == NULL and nnodes == n the arrays are
 * what rxgpu_hnsw_import takes. */
int rxgpu_hnsw_export(const rxgpu_index*, uint64_t nnodes, const uint32_t* nodes, uint32_t* level0, int32_t* levels, int64_t* upper_offsets,
					  uint32_t* upper, rxgpu_hnsw_graph* info);
/* labels of n shard-local internal indices (device pointers; enqueued on `stream`): the HNSW device search returns indices, the
 * multi-GPU merge needs labels */
int rxgpu_gather_labels_device(const rxgpu_index*, uint64_t n, const uint32_t* d_idx, uint64_t* d_out_label, void* stream);
/* HierarchicalNSWImpl::SearchRange                              hnswlib/hnswalg.h:2015-2070
 * The ef-search result seeds a breadth-first expansion over level-0 neighbours with dist < radius (strict); the result is that
 * closure (independent of traversal order).  Writes the best min(*out_n, max_out) results best-first (ties by label);
 * *out_n = total number of matches.  Query pre-normalised for Cosine, radius in map space (IP / Cosine: negated by the caller,
 * hnsw_index.cc:185).  ef == 0 is treated as 1. */
int rxgpu_hnsw_search_range(const rxgpu_index*, const float* query /* host */, float radius, uint32_t ef, uint64_t max_out,
							float* out_dist, uint64_t* out_label, uint64_t* out_n);
/* HierarchicalNSWImpl::SearchRange for nq queries at once (our extension; the reference takes one query per call).
 * Per query q the result is identical to rxgpu_hnsw_search_range(queries + q*dim, radius[q], ef, max_out, ...):
 * out_n[q] = total matches, the best min(out_n[q], max_out) go best-first into row q of out_dist / out_label (nq x max_out).
 * One ef-search for the batch seeds the closures; one launch per BFS level expands the closures of up to (SMs x 32) queries.
 * A query keeps min(n, max(4096, 2 * min(max_out, 131072))) matches on the device; one with more is answered again with room for
 * the whole graph (same answer).  A NaN or -inf radius matches nothing, +inf floods the query's reachable component.
 * rxgpu_last_search_stats: launches = all kernel launches, passes = BFS levels run, tc_fallbacks = queries answered again. */
int rxgpu_hnsw_search_range_batch(const rxgpu_index*, uint32_t nq, const float* queries /* nq x dim, host */,
								  const float* radius /* nq, map space */, uint32_t ef, uint64_t max_out,
								  float* out_dist, uint64_t* out_label, uint64_t* out_n /* nq */);

/* Streaming (resumable) search: HierarchicalNSWImpl::BeginStreamingSearch / ContinueStreamingSearch   hnswlib/hnswalg.h:1864-1975
 * (the KNN iterator of filtered queries pulls batches until enough rows pass the other conditions,
 * core/nsselecter/knn_streaming_index_iterator.cc).  The session state -- visited set, candidate set, top candidates, extras, lower
 * bound -- stays in HBM between calls; a call expands nodes in (distance, id) order until the reference's stop rule holds and returns
 * the next `batch_size` closest expanded nodes, best first (ties by label).  ef == 0 -> 100 (kDefaultStreamingEf); ef, batch <= 1024.
 * Query pre-normalised for Cosine.  The session must end before the index changes or is destroyed. */
typedef struct rxgpu_hnsw_stream rxgpu_hnsw_stream;
int rxgpu_hnsw_stream_begin(const rxgpu_index*, const float* query /* host */, uint32_t ef, rxgpu_hnsw_stream** out);
int rxgpu_hnsw_stream_next(rxgpu_hnsw_stream*, uint32_t batch_size, float* out_dist, uint64_t* out_label, uint32_t* out_count, int* exhausted);
void rxgpu_hnsw_stream_end(rxgpu_hnsw_stream*);

/* ---------------------------------------------------------------- SQ8 scalar quantisation (the quantised HNSW map of the reference)
 * HierarchicalNSWImpl<uint8_t> keeps every vector as dim uint8 codes plus ONE additive corrective offset
 * (scalar_quantization/quantizer.h:93-125; hnswlib/hnswlib.h:255) and measures
 *     dist(a, b) = alpha_2 * int_dist(code_a, code_b) + offset_a + offset_b        (hnswlib.h:192-197; IP / Cosine: negated;
 *                  Cosine: times the row's norm coefficient and the query's 1 / ||q||, hnswalg.h:801,1854-1863)
 * with int_dist = sum (a - b)^2 or sum a * b over the codes (tools/distances/l2_dist.cc:169, ip_dist.cc:163 -- exact integers).
 * rxgpu_sq8_attach puts codes + offsets next to the fp32 rows in HBM: imported from the reference (codes != NULL: [size][dim] bytes and
 * [size] floats, by internal id = row) or produced on the device from the rows with the reference's arithmetic (codes == NULL).
 * Distances computed from them are bit-identical to the reference's: the integer part is exact, the float epilogue repeats its order. */
typedef struct { /* hnswlib::QuantizingParams (scalar_quantization/quantization_params.h:47-106) */
	float min_q, max_q, alpha, alpha_2, delta;
} rxgpu_sq8_params;
int rxgpu_sq8_attach(rxgpu_index*, const rxgpu_sq8_params*, const uint8_t* codes, const float* offsets);
int rxgpu_sq8_export(const rxgpu_index*, uint8_t* codes /* size x dim */, float* offsets /* size */);
/* the query as HierarchicalNSWImpl<uint8_t>::search prepares it (prepareData, hnswalg.h:510-535): codes[dim] + its corrective offset.
 * query: pre-normalised for Cosine, query_norm = ||q|| then (ignored otherwise).  Host only. */
int rxgpu_sq8_prepare_query(const rxgpu_index*, const float* query, float query_norm, uint8_t* codes, float* offset);
/* exact top-k under the quantised metric: a dp4a scan of all codes with the fused top-k (the ground truth of the quantised HNSW
 * search; 4x fewer HBM bytes than the fp32 scan).  query_norms: nq values of ||q|| for Cosine, NULL otherwise.  k <= 256. */
int rxgpu_sq8_search_knn(const rxgpu_index*, uint32_t nq, const float* queries /* host, pre-normalised for Cosine */, const float* query_norms,
						 uint32_t k, float* out_dist, uint64_t* out_label, uint32_t* out_count);
/* HierarchicalNSWImpl<uint8_t>::SearchKnn on the imported graph: the HNSW kernel gathers codes instead of fp32 rows */
int rxgpu_hnsw_search_knn_sq8(const rxgpu_index*, uint32_t nq, const float* queries /* host */, const float* query_norms, uint32_t k, uint32_t ef,
							  float* out_dist, uint64_t* out_label, uint32_t* out_count, uint32_t* stats /* nq x 2 or NULL */);

/* ---------------------------------------------------------------- IVF index (faiss::IndexIVFFlat as reindexer::IvfIndex drives it)
 * Replaces the search side of IvfIndex: map_->search(1, key, k, dists, ids, &IVFSearchParameters{nprobe})
 *   core/index/float_vector/ivf_index.cc:150-204 (callers), vendor_subdirs/faiss/IndexIVF.cpp (search_preassigned), IndexIVFFlat.cpp
 *   (the flat list scanner).  Training (k-means) and list assignment run either on the device (rxgpu_ivf_train / _assign below) or in
 * the reference's FAISS on the CPU; in the second case the adapter fills
 * the device index with the rows GROUPED BY LIST (list 0's vectors first, then list 1's, ...; label = the FAISS id) and hands
 * over the centroids and list sizes.  A search = coarse quantiser (distance to every centroid, nprobe nearest) + a scan of the
 * probed lists with the exact-scan kernel (fused top-k per list) + one merge.  Cosine: queries pre-normalised, rows and centroids
 * carry their norm coefficients like the reference's patched FAISS (IndexFlatCosine, IndexIVFFlat(..., is_cosine)).
 * Results best-first in map space (L2: squared distance; IP / Cosine: -inner product / -cos), bit-equal distances ordered by label;
 * out_count[q] = min(k, rows in the probed lists).  k <= 256, nprobe <= 1024, at most 131072 centroids (the reference's bound;
 * 131073 and more: errParams), dim <= 51200 (the coarse pass stages a query in shared memory). */
int rxgpu_ivf_import(rxgpu_index*, uint32_t nlist, const float* centroids /* nlist x dim, host */, const uint64_t* list_sizes /* nlist */);
int rxgpu_ivf_search_knn(const rxgpu_index*, uint32_t nq, const float* queries /* host */, uint32_t k, uint32_t nprobe, float* out_dist,
						 uint64_t* out_label, uint32_t* out_count);
/* The same search at any k in [1, 65535] and any nprobe (clamped to [1, nlist]): the best min(k, probed rows) rows per query, cut at
 * the k-th place by (distance, internal row) and then ordered by (distance, label), as rxgpu_ivf_search_knn orders them.  k <= 256 with
 * nprobe <= 1024 runs rxgpu_ivf_search_knn itself (same bits); otherwise one distance pass writes every probed row's key to a device
 * workspace and an exact radix select keeps the k best per query (DESIGN.md §3.5).  Same errors as rxgpu_ivf_search_knn; k = 0 or
 * k > 65535: RXGPU_ERR_PARAMS; device memory exhausted: RXGPU_ERR_SYSTEM.  Entries past out_count[q] are not written. */
int rxgpu_ivf_search_knn_large_k(const rxgpu_index*, uint32_t nq, const float* queries /* host */, uint32_t k, uint32_t nprobe,
								 float* out_dist, uint64_t* out_label, uint32_t* out_count);
/* map_->range_search(1, key, radius, &result, &params) (ivf_index.cc:205-300): every row of the nprobe probed lists with
 * dist < radius in map space (strict; IP / Cosine radius negated by the caller), best first; *out_n = total number of matches. */
int rxgpu_ivf_search_range(const rxgpu_index*, const float* query /* host */, float radius, uint32_t nprobe, uint64_t max_out,
						   float* out_dist, uint64_t* out_label, uint64_t* out_n);
/* A batch of IVF range searches.  radius[q] is in map space, exactly as for rxgpu_ivf_search_range.  Per query q the result is identical
 * to rxgpu_ivf_search_range(queries + q*dim, radius[q], nprobe, max_out, ...): out_n[q] = total matches, and the best
 * min(out_n[q], max_out) matches, best first in the order of hitLessByLabel (distance, then label), go into row q of
 * out_dist / out_label (nq x max_out); the rest of a row is not written.  A NaN or -inf radius matches nothing, +inf every probed row.
 * One coarse pass and one key pass over the probed lists serve the batch; each query's matches are counted, kept and sorted on the
 * device (DESIGN.md §3.5), and no query is answered twice.  Same errors as rxgpu_ivf_search_range; device memory exhausted:
 * RXGPU_ERR_SYSTEM.  rxgpu_last_search_stats: launches = all kernel launches, passes = 1, tc_fallbacks = 0. */
int rxgpu_ivf_search_range_batch(const rxgpu_index*, uint32_t nq, const float* queries /* nq x dim, host */,
								 const float* radius /* nq, map space */, uint32_t nprobe, uint64_t max_out,
								 float* out_dist, uint64_t* out_label, uint64_t* out_n /* nq */);

/* Mutable lists -- what IvfIndex::upsert / del do once the index is trained (ivf_index.cc:87-132: map_->add_with_ids(1, vec, &id),
 * map_->remove_ids(IDSelectorArray{1, &id})): rxgpu_ivf_create attaches EMPTY lists to an empty index (the rows then live in the lists:
 * every list owns a region of one row slab with slack, a full list moves to the end of the slab with 1.5x room, dead space is
 * compacted when it exceeds the live rows); rxgpu_ivf_add appends rows to the lists the caller's coarse quantiser chose
 * (list_nos[i] = faiss' lo_listno of the id after the CPU add, so both sides agree on the assignment bit for bit); rxgpu_ivf_remove is
 * the inverted lists' swap-remove.  An upsert costs one row copy, never a re-import.  Searches see every completed call. */
int rxgpu_ivf_create(rxgpu_index*, uint32_t nlist, const float* centroids /* nlist x dim, host */);
int rxgpu_ivf_add(rxgpu_index*, uint64_t n, const uint32_t* list_nos, const uint64_t* labels, const float* vecs /* n x dim, host */);
int rxgpu_ivf_remove(rxgpu_index*, uint64_t label); /* errNotFound when the id is in no list */
uint64_t rxgpu_ivf_size(const rxgpu_index*);
int rxgpu_ivf_list_stats(const rxgpu_index*, uint64_t* slab_rows, uint64_t* dead_rows, uint64_t* relocations, uint64_t* compactions);

/* Training on the device -- what IvfIndex::trainIdx runs on the CPU (idx.train(n, x, norms): IndexIVFFlat::train -> Level1Quantizer::
 * train_q1 -> faiss::Clustering::train, nredo 1, unweighted, spherical for IP and Cosine) and the list assignment of add_with_ids
 * (quantizer->assign).  The sample and the initial centroids come from the same std::mt19937 draws as FAISS's (rxgpu_kmeans_plan); an
 * iteration assigns every point to its nearest centroid under (distance, centroid id) with the coarse pass's exact arithmetic, sums
 * each centroid's members in ascending point order in fp32 and scales by 1 / count, splits empty clusters as split_clusters does,
 * then renormalises (spherical: fp64 norm, one rounding).  Given the same assignments the centroids are FAISS's bit for bit for L2
 * (DESIGN.md §3.7).  Cosine input is normalised first: each vector times norm_coefs[i] when given, else as rxgpu_select_knn normalises
 * a query. */
typedef struct {
	int32_t niter;                   /* Lloyd iterations, >= 0 (IndexIVF: 10) */
	int32_t seed;                    /* >= 0 (1234); FAISS turns a negative seed into a clock-based one: errParams here */
	int32_t max_points_per_centroid; /* >= 1 (256): more than nlist x this points are subsampled */
} rxgpu_ivf_train_params;
typedef struct { /* per iteration, as faiss::ClusteringIterationStats */
	double obj;          /* fp64 sum of the points' exact distances in FAISS's convention (L2: squared distance, IP / Cosine: similarity) */
	int32_t nsplit;      /* empty clusters split */
	float assign_ms;     /* the assignment kernel (CUDA events) */
	float update_ms;     /* the update's device work: key split, sort, sums, splits and renormalisation (CUDA events) */
	float host_ms;       /* the update's host work between them: keys back, objective, histogram, split choices, offsets out */
} rxgpu_ivf_train_stats;
/* Trains nlist centroids on n host vectors and leaves the index as rxgpu_ivf_create(nlist, centroids) would: empty lists, centroids
 * resident.  out_centroids: nlist x dim or NULL; stats: niter entries or NULL (n == nlist after sampling copies the points, as FAISS's
 * corner case does, and reports zeros); params NULL: IndexIVF's defaults.  The index must be empty with no IVF attached (errLogic).
 * errParams: NaN or Inf in the input, n < nlist, nlist outside [1, 131072], dim beyond the coarse pass's bound, bad params.  Device
 * memory short for the training set: errSystem.  On any error the index is unchanged. */
int rxgpu_ivf_train(rxgpu_index*, uint32_t nlist, uint64_t n, const float* vecs /* n x dim, host */,
					const float* norm_coefs /* Cosine: n or NULL */, const rxgpu_ivf_train_params* params, float* out_centroids,
					rxgpu_ivf_train_stats* stats);
/* quantizer->assign as IndexIVF::add_with_ids calls it (same Cosine handling as rxgpu_ivf_train): the nearest centroid of every vector
 * under (distance, centroid id), exactly the centroid rxgpu_ivf_search_* probes first at nprobe = 1.  out_dist: its distance in map
 * space, or NULL.  Needs IVF lists (imported or created) and the index unchanged since, like the searches. */
/* Concurrency: rxgpu_ivf_assign only reads the centroids, which no call changes while the lists exist, so it may run beside searches
 * and adds; rxgpu_ivf_add_assign is a mutation like rxgpu_ivf_add (one at a time per index, as the reference's write lock keeps them). */
int rxgpu_ivf_assign(const rxgpu_index*, uint64_t n, const float* vecs /* n x dim, host */, const float* norm_coefs, uint32_t* out_list_nos,
					 float* out_dist);
/* rxgpu_ivf_assign followed by rxgpu_ivf_add with those lists, all or nothing; out_list_nos (n or NULL) receives the lists, for
 * IndexIVF::add_core on the CPU side. */
int rxgpu_ivf_add_assign(rxgpu_index*, uint64_t n, const uint64_t* labels, const float* vecs /* n x dim, host */, const float* norm_coefs,
						 uint32_t* out_list_nos);
/* Host only: the sample rxgpu_ivf_train takes (subsample_training_set with rand_perm(n, seed): the first nlist x max_points_per_centroid
 * entries when n exceeds that, else 0 .. n-1; out_sample holds min(n, nlist x max_points_per_centroid) rows or is NULL) and the input row
 * each initial centroid copies (out_init, nlist entries: sample[perm[c]] with perm = rand_perm(sample size, seed + 1), or c when the
 * sample size equals nlist). */
int rxgpu_kmeans_plan(uint64_t n, uint32_t nlist, int32_t seed, int32_t max_points_per_centroid, int32_t* out_sample, int32_t* out_init);

/* ---------------------------------------------------------------- multi-GPU IVF: one shard per GPU / rank over the same centroids
 * Shard r holds a row range of the namespace in its own index, with IVF lists over the SAME centroids on every rank: the ranks train once
 * (rxgpu_sharded_ivf_train), each fills its lists with rxgpu_ivf_add_assign (a row's list is a function of the centroids alone, so it is
 * the list a single index would give it), and the searches below answer from all shards.  All three are collectives over an
 * rxgpu_comm (NCCL, or rxgpu_comm_create_local's threads): every rank calls them with the same arguments except its own rows / shard.
 * The exchanges and their sizes are in DESIGN.md §7.
 *
 * rxgpu_sharded_ivf_train: every rank leaves its index exactly as rxgpu_ivf_train leaves an index trained on the concatenation of all
 * ranks' rows in rank order -- the same centroids and per-iteration obj / nsplit, bit for bit, on every rank.  The ranks all-gather their
 * row counts and parameters; each prepares the sample entries it owns (rxgpu_kmeans_plan over the global rows, Cosine normalised as
 * rxgpu_ivf_train does), one all-gather assembles the whole sample in plan order on every rank (each rank keeps it all, as one GPU
 * does), each iteration assigns an even slice of the sample per rank and all-gathers the keys, and every rank runs the same update.
 * stats[i].assign_ms is this rank's slice; obj and nsplit are global.  When the sample is exactly nlist rows, the centroids are the first
 * nlist rows of the concatenation, as rxgpu_ivf_train (and FAISS) take them.  Errors are agreed: ranks that disagree on nlist, dim,
 * metric or the parameters all return errParams; an error of one rank's own (its index not empty, a shard on another device than its
 * communicator, NaN or Inf in its rows, device memory short for the training -- counted for every rank that shares its device) reaches
 * every rank before the sample moves, and all return that code.  The other errors are rxgpu_ivf_train's, on the whole input.  On any
 * of these every index is unchanged.  Not agreed, as in any collective: a null communicator or index, and a failure inside an exchange
 * or of an allocation after the agreement (memory taken by something else meanwhile) -- that rank returns errSystem and its peers wait. */
int rxgpu_sharded_ivf_train(rxgpu_comm*, rxgpu_index* shard, uint32_t nlist, uint64_t n_local, const float* vecs_local /* n_local x dim, host */,
							const float* norm_coefs_local /* Cosine: n_local or NULL */, const rxgpu_ivf_train_params* params,
							float* out_centroids /* nlist x dim or NULL */, rxgpu_ivf_train_stats* stats /* niter or NULL */);
/* The sharded rxgpu_ivf_search_knn_large_k: any k in [1, 65535], any nprobe.  Each rank runs the coarse pass and its own best k under
 * (distance, local row), one all-gather ships the lists, a device merge keeps the k best under (distance, global row) with the shards'
 * rows laid end to end in rank order, and the survivors are ordered by (distance, label).  On every rank the answer has the labels,
 * order and distance bits of rxgpu_ivf_search_knn_large_k on one index holding all rows in the same lists whenever the k-th place is
 * not tied; when it is, the tied rows of the lower rank (then the lower local row) are kept.  With one rank it is that call's answer,
 * bit for bit.  queries: nq x dim, host (queries_on_device == 0) or device pointer on the shard's GPU.  out_*: host, nq x k;
 * out_count[q] = min(k, probed rows over all shards).  Every rank's payload carries a fingerprint of its centroids, nlist, nprobe, k,
 * dim and metric: if they differ, every rank returns errLogic; an error in one rank's local IVF search (no lists, lists stale, device
 * memory short for it) reaches every rank the same way.  Not agreed, as in any collective -- that rank returns alone and its peers wait
 * in the all-gather: an argument error (null pointer, a shard on another device than its communicator, k outside [1, 65535]; every
 * rank passes the same k, so that one is all ranks' error) and a failure to allocate the exchange buffers, 16·nq·k bytes to send and
 * R times that to receive per rank (1.07 GB and 8.6 GB at nq = 1024, k = 65535, 8 ranks). */
int rxgpu_sharded_ivf_search_knn(rxgpu_comm*, const rxgpu_index* shard, uint32_t nq, const float* queries, int queries_on_device, uint32_t k,
								 uint32_t nprobe, float* out_dist, uint64_t* out_label, uint32_t* out_count);
/* The sharded rxgpu_ivf_search_range_batch: per query q the result on every rank is that call's on one index holding all rows in the
 * same lists, bit for bit -- out_n[q] = total matches, the best min(out_n[q], max_out) in the order of hitLessByLabel in row q of
 * out_dist / out_label (host, nq x max_out; the rest of a row may be overwritten), NaN / -inf radii match nothing, +inf every probed
 * row.  Labels must be unique across the shards.  Each rank runs the local range batch; the ranks then all-reduce the status, the
 * width and the words every rank must agree on (the same check as the KNN call's), all-reduce the totals, all-gather the best
 * min(matches, max_out) per query and shard, and merge them on the device -- the exchange of rxgpu_sharded_search_range_batch.  An
 * error in one rank's local range batch reaches every rank through the first all-reduce; argument errors and a failure inside an
 * exchange return on that rank alone, as in rxgpu_sharded_ivf_search_knn. */
int rxgpu_sharded_ivf_search_range_batch(rxgpu_comm*, const rxgpu_index* shard, uint32_t nq, const float* queries, int queries_on_device,
										 const float* radius /* nq, map space */, uint32_t nprobe, uint64_t max_out, float* out_dist,
										 uint64_t* out_label, uint64_t* out_n);

/* ---------------------------------------------------------------- ft_fast full-text merge (BM25 scoring over posting lists)
 * Replaces ft::Merger<IdCont, ft::MergeData, OffsetT>::Merge<Bm25Rx|Bm25Classic|TermCount>  core/ft/ft_fast/mergerimpl.h:466-566
 * -- the seam is Selector<IdCont>::mergeResults (ft_fast/selecterimpl.h:609-627) -- for query parts that are plain terms
 * (each with its variant subterms); phrases and multi-word synonyms stay on the reference's CPU path (returns errParams).
 * Inputs mirror what the reference hands the merger: posting lists = IdRelVec contents (ft/idrelset.h:62-130) de-interleaved,
 * document statistics = the DocsStatsGetter duck-type (index/indextext/indextext.h:245-258), FTConfig members the merger reads
 * (ft/config/ftconfig.h:118-236), query parts = TermResults/SubtermResults + FtDslOpts (ft_fast/querymergedata.h, ft/ftdsl.h:13-30).
 * Output = ft::MergeData (ft_fast/phrasemerger.h:57-78), bit-identical to the reference: same docs, same order for
 * RankAndID / IDOnly, same uint8 ranks, same field; rxgpu_ft_merge_query_areas adds the highlight areas of
 * ft::MergeDataAreas<Area> for queries without phrases. */
typedef struct {
	uint32_t ndocs;
	const uint32_t* doc_ids;   /* ascending vdoc ids, >= 1 (vdoc 0 is the reference's dummy, mergerimpl.h:122) */
	const uint32_t* pos_begin; /* ndocs + 1 offsets into positions */
	const uint32_t* positions; /* PosType: pos | field << 24, ascending within a doc (arrayIdx 0) */
} rxgpu_ft_postings;
typedef struct { /* FTFieldConfig */
	double bm25_boost, bm25_weight, term_len_boost, term_len_weight, position_boost, position_weight;
} rxgpu_ft_field_config;
typedef struct { /* FTConfig members read by the merger */
	uint32_t merge_limit;
	int32_t min_rank;
	double bm25_k1, bm25_b;
	int32_t bm25_type; /* 0 rx (default), 1 classic, 2 wordCount */
	double distance_boost, distance_weight, full_match_boost;
	uint32_t nfields;
	const rxgpu_ft_field_config* fields;
	double summation_ranks_by_fields_ratio; /* FTConfig::summationRanksByFieldsRatio (ftconfig.h:210): 0 = off (the default) */
} rxgpu_ft_config;
typedef struct { /* one TermResults */
	int32_t op; /* OpType: 1 = OpOr, 2 = OpAnd, 3 = OpNot */
	float boost;
	float term_len_boost;
	const float* field_boosts; /* nfields */
	uint32_t nsubterms;
	const uint32_t* postings; /* ids returned by rxgpu_ft_add_postings */
	const float* procs;
	const uint8_t* need_sum_rank; /* nfields flags FtDslFieldOpts::needSumRank (ftdsl.h:15), or NULL = all false; at most 16 set */
	const uint8_t* suppressed;    /* nsubterms flags SubtermResults::Suppressed (querymergedata.h:32; set on the subterms of multi-word
	                               * synonyms that repeat a word of the query, :221-241), or NULL = none */
	uint32_t nsynonyms;           /* PhraseOrTerm::SynonymsIds (querymergedata.h:160): indexes into rxgpu_ft_query::synonyms; query parts only */
	const uint32_t* synonym_ids;
	int32_t phrase_num;           /* FtDslOpts::phraseNum (ftdsl.h): 0 = a plain term; consecutive terms with the same non-zero number
	                               * form ONE query part, a phrase (PhraseResults, querymergedata.h:103-139; merged by PhraseMerger,
	                               * phrasemerger.h:285-399, then Merger::mergePhrase, mergerimpl.h:41-90).  The phrase's op is its first
	                               * term's; subterms of phrase terms keep the caller's order (the reference merges phrases before it sorts) */
	int32_t distance;             /* FtDslOpts::distance: how far after the previous term of the phrase this one may stand (terms 2..) */
} rxgpu_ft_term;
typedef struct { /* ft::Synonym (querymergedata.h:168-188): the terms of one multi-word substitution */
	uint32_t nterms;
	const rxgpu_ft_term* terms;
} rxgpu_ft_synonym;
typedef struct { /* ft::QueryMergeData (querymergedata.h:191-242) */
	uint32_t nterms;
	const rxgpu_ft_term* terms; /* queryParts */
	uint32_t nsynonyms;
	const rxgpu_ft_synonym* synonyms;
} rxgpu_ft_query;
typedef struct { /* ft::MergeInfo */
	int32_t id;
	float proc;
	uint8_t field;
	uint8_t normalized_proc;
} rxgpu_ft_merge_info;
typedef struct rxgpu_ft_index rxgpu_ft_index;

/* document statistics of the index: words_in_field[total_docs][nfields] (NumWordsInField), avg_words[nfields] (AvgWordsCount),
 * removed[total_docs] or NULL (DocRemoved).  total_docs counts the dummy vdoc 0 like the reference's vdocs_.size(). */
int rxgpu_ft_create(rxgpu_ft_index** out, uint32_t total_docs, uint32_t nfields, const uint32_t* words_in_field, const float* avg_words,
					const uint8_t* removed, int device);
void rxgpu_ft_destroy(rxgpu_ft_index*);
int rxgpu_ft_add_postings(rxgpu_ft_index*, const rxgpu_ft_postings* list, uint32_t* out_id); /* uploads one word's postings to HBM */
/* The same from the reference's packed container: `data` = PackedIdRelVec::data_ (core/ft/idrelset.h:154-281, records written by
 * IdRelType::packWithoutArrayIdxs, idrelset.cc:139-183), `count` = its size().  Decoded once on the host (the varint-delta stream has
 * no skip pointers) and uploaded as SoA.  Lists that contain array indexes (arrayFoundPos_ set) are not supported (errParams). */
int rxgpu_ft_add_postings_packed(rxgpu_ft_index*, const uint8_t* data, uint64_t len, uint32_t count, uint32_t* out_id);
/* A whole commit's worth of packed lists in one call: the raw varint streams travel to the device (about 2.5x fewer bytes than the
 * SoA) and are decoded THERE -- one thread per list, two passes (validate + count, then write) into three slabs shared by the batch
 * (IdRelType::unpackWithoutArrayIdxs, idrelset.cc:185-235; iterator state chain idrelset.h:172-211).  A list longer than 256 KiB would
 * hold the batch back behind one thread and goes through the host decoder instead.  All or nothing: on error no list of the batch
 * stays.  out_ids[i] = id of list i. */
int rxgpu_ft_add_postings_packed_batch(rxgpu_ft_index*, uint32_t nlists, const uint8_t* const* data, const uint64_t* lens,
									   const uint32_t* counts, uint32_t* out_ids);
/* The decoder alone (no device involved): fills doc_ids[count], pos_begin[count + 1] and at most max_positions positions; *npos =
 * number of positions in the list (call with max_positions = 0 to size the buffer). */
int rxgpu_ft_decode_packed(const uint8_t* data, uint64_t len, uint32_t count, uint32_t* doc_ids, uint32_t* pos_begin,
						   uint32_t* positions, uint64_t max_positions, uint64_t* npos);
/* excluded: u8[total_docs] (FtMergeStatuses::Statuses docsExcluded) or NULL; rank_sort_type: reindexer::RankSortType.
 * Writes min(*out_n, max_out) entries; *out_n = number of merged documents. */
int rxgpu_ft_merge(rxgpu_ft_index*, const rxgpu_ft_config* cfg, uint32_t nterms, const rxgpu_ft_term* terms, const uint8_t* excluded,
				   int rank_sort_type, uint64_t max_out, rxgpu_ft_merge_info* out, uint64_t* out_n);
/* The same with multi-word synonyms (Merger::Merge, mergerimpl.h:510-560): a synonym's terms are merged after the query parts; a
 * document that entered the result through synonyms stays only if it holds every term of one of them; an AND part is also satisfied by
 * a document that holds all terms of one of its synonyms (buildRestrictingBitmask, :352-363). */
int rxgpu_ft_merge_query(rxgpu_ft_index*, const rxgpu_ft_config* cfg, const rxgpu_ft_query* query, const uint8_t* excluded, int rank_sort_type,
						 uint64_t max_out, rxgpu_ft_merge_info* out, uint64_t* out_n);
/* The same merge with highlight areas: ft::Merger<IdCont, ft::MergeDataAreas<Area>, OffsetT> (ft_fast/merger.h:196-205,
 * core/ft/areaholder.h), what IndexText asks for when the query's context is kFtArea (highlight() / snippet()).  `out` is
 * bit-identical to rxgpu_ft_merge_query's.  For returned entry i and field f its committed areas (AreasInDocument::GetAreas(f), ordered
 * by start) are out_areas[out_area_begin[i * nfields + f] .. out_area_begin[i * nfields + f + 1]); out_area_begin holds
 * min(*out_n, max_out) * nfields + 1 offsets, out_areas has room for max_out * nfields * max_areas_in_doc entries.  out_raw_count (max_out
 * entries, or NULL) = GetAreasCount() before the commit.  max_areas_in_doc = FTConfig::maxAreasInDoc, in [1, 64]; outside that range,
 * or for a query with a phrase, the call returns errParams and changes nothing. */
typedef struct {
	uint32_t start, end; /* Area(start, end, arrayIdx = 0) */
} rxgpu_ft_area;
int rxgpu_ft_merge_query_areas(rxgpu_ft_index*, const rxgpu_ft_config* cfg, const rxgpu_ft_query* query, const uint8_t* excluded,
							   int rank_sort_type, int32_t max_areas_in_doc, uint64_t max_out, rxgpu_ft_merge_info* out,
							   uint32_t* out_area_begin, rxgpu_ft_area* out_areas, uint32_t* out_raw_count, uint64_t* out_n);
/* IndexText::afterSelect + sortAfterSelect on top of the merge, without leaving the device (core/index/indextext/indextext.cc:480-611;
 * Merger::postProcessResults, ft_fast/merger.h:111-155): ranks below min_rank are dropped, the rest is normalised to uint8 by the
 * global maximum, every merged vdoc expands to its row ids, rows whose external status is 0 are skipped (FtUseExternStatuses::Yes),
 * and the rows come back ordered by (rank descending, row id ascending) for RankSortType::RankAndID (1) or by row id for IDOnly (3) --
 * the deterministic "integer top-k, ties by id".  Only the first `limit` rows are copied to the host; *out_n = number of rows that
 * qualify.  rxgpu_ft_set_rows uploads vdocs_[vdoc].RowIds() as CSR (row_begin[total_docs + 1], row_ids) once per commit; without it
 * (or with NULL) vdoc i is row i. */
int rxgpu_ft_set_rows(rxgpu_ft_index*, const uint32_t* row_begin, const int32_t* row_ids);
int rxgpu_ft_select(rxgpu_ft_index*, const rxgpu_ft_config* cfg, uint32_t nterms, const rxgpu_ft_term* terms, const uint8_t* excluded,
					const uint8_t* row_status /* u8 per row id, or NULL */, int rank_sort_type, uint64_t limit, int32_t* out_row_ids,
					float* out_ranks /* RankT = the uint8 rank as float */, uint64_t* out_n);
int rxgpu_ft_select_query(rxgpu_ft_index*, const rxgpu_ft_config* cfg, const rxgpu_ft_query* query, const uint8_t* excluded,
						  const uint8_t* row_status, int rank_sort_type, uint64_t limit, int32_t* out_row_ids, float* out_ranks, uint64_t* out_n);
/* ---------------------------------------------------------------- ft_fast merge over docid-range shards (SURVEY 8e)
 * Shard r of the communicator holds the documents [doc_base_r, doc_base_r + total_docs_r) of the namespace under LOCAL ids, the posting
 * lists restricted to them (the same list ids on every shard; a list may be empty on a shard) and the namespace-wide average field
 * lengths.  One collective call per rank = rxgpu_ft_select over the whole namespace: BM25's document and posting counts, the
 * restricting mask's popcount, the 65 536-bin preselect histogram, the ordered cut at the threshold score (lower shards first) and the
 * largest rank (uint8 normalisation) are exchanged between the shards (five exchanges of a few bytes to 512 KB), every rank's first
 * `limit` rows are gathered and merged, and EVERY rank returns the same rows the unsharded call returns.  Row ids: doc_base + local id,
 * or the shard's rxgpu_ft_set_rows table (global row ids).  Not served: phrases, multi-word synonyms (their slot order is global). */
int rxgpu_sharded_ft_select(rxgpu_comm*, rxgpu_ft_index* shard, uint32_t doc_base, const rxgpu_ft_config* cfg, uint32_t nterms,
							const rxgpu_ft_term* terms, const uint8_t* excluded, const uint8_t* row_status, int rank_sort_type, uint64_t limit,
							int32_t* out_row_ids, float* out_ranks, uint64_t* out_n);
/* statistics of the last merge on this thread */
typedef struct {
	uint32_t launches;
	uint32_t preselected;       /* 1 when preselectMostRelevantDocs ran */
	uint64_t postings_scanned;  /* postings streamed over all passes */
	uint64_t algorithmic_bytes; /* SURVEY.md §8d model: bytes the passes must touch */
	float device_ms;            /* CUDA-event time of the device part */
} rxgpu_ft_stats;
void rxgpu_ft_last_stats(rxgpu_ft_stats* out);

/* ---------------------------------------------------------------- benchmark / test support (not part of the reference surface)
 * Appends n rows generated on the device: element (row r, col c) = synth(seed, (first_row + r) * dim + c), label =
 * (first_row + r) << 32.  The generator is defined in csrc/synth.cuh and mirrored bit-for-bit by oracle/knn_port.c. */
int rxgpu_index_append_synth(rxgpu_index*, uint64_t seed, uint64_t first_row, uint64_t n);
/* fills a device buffer with synth(seed, first_index + i) */
int rxgpu_synth_fill_device(float* d_out, uint64_t seed, uint64_t first_index, uint64_t count, int device, void* stream);
/* tuning knobs, mainly for benchmarks: queries per DB pass (0 = auto) */
int rxgpu_set_query_tile(rxgpu_index*, uint32_t qt);
/* statistics of the last search on this thread: kernel launches, DB passes */
typedef struct {
	uint32_t launches;
	uint32_t passes;
	uint32_t query_tile;
	uint32_t tie_replays;       /* queries whose k-th place was a bit-equal tie: the reference's heap rule was replayed */
	uint32_t tie_from_lists;    /* ... of which answered from the filter's candidate lists (no second pass over the rows) */
	uint64_t algorithmic_bytes; /* SURVEY.md §8d definition: passes x (N*D*4 [+N*4 for Cosine] + QT*D*4 + QT*k*12) */
	uint32_t scan_launches;     /* with rxgpu_set_profile(1): launches of the dominant kernel timed ... */
	float scan_kernel_ms;       /* ... and their summed device time (CUDA events on the launching stream) */
	uint32_t tc_used;           /* 1 when the tensor-core filter + exact re-rank path answered the batch */
	uint32_t tc_fallbacks;      /* queries whose candidate list overflowed and were answered by the exact scan
	                               (rxgpu_hnsw_search_range_batch: whose result region overflowed and were answered again) */
	uint64_t tc_candidates;     /* rows re-ranked exactly */
	uint32_t tc_cluster;        /* CTAs per cluster in the filter kernel (row tiles are TMA-multicast inside a cluster) */
	uint32_t tc_kernel;         /* 1 = knn_tc_filter (wgmma, queries in shared memory); 2..5 = its diagnostic instantiations (rxgpu_tc_diag) */
} rxgpu_search_stats;
void rxgpu_last_search_stats(rxgpu_search_stats* out);
/* large query batches: int8 tensor-core filter (exact integer dot products of per-row scaled codes, certified by per-row
 * residual norms) + exact fp32 re-rank (results identical to the exact scan).
 * mode 0 = automatic (batches >= 64 queries on >= 100k rows, k <= 1023), 1 = whenever possible, 2 = never;
 * 3 / 4 / 5 = as 1 with single CTAs / clusters of up to two / clusters of up to four CTAs sharing every row tile (TMA multicast);
 * 0 and 1 take clusters of up to two on indexes of >= 2^23 rows and single CTAs below; all give the same bits. */
int rxgpu_set_tensor_core_filter(rxgpu_index*, int mode);
/* process-wide switch: bracket every scan-kernel launch with CUDA events (used by bench.py for the roofline figure) */
int rxgpu_set_profile(int on);
/* process-wide, diagnostics only (bench_tc_phases.py): every tensor-core filter launch takes the diagnostic instantiation `mode`
 * (1 = per-phase clock stamps, 2 = rare path compiled out, 3 = producers not fetching, 4 = block test and rare path compiled out;
 * 0 = the production kernel again) and adds its counters to the zeroed device buffer d_counters (knn_tc.cuh: kTcDiag*).  Modes 2
 * to 4 return meaningless results; only query
 * blocks of 128 are served, in the cluster shape the index's rxgpu_set_tensor_core_filter mode picks.  A mode other than 0 is refused (RXGPU_ERR_LOGIC) unless the environment has
 * RXGPU_TC_DIAG=1, and a search a diagnostic instantiation answered reports tc_kernel = 1 + mode in its statistics. */
int rxgpu_tc_diag(int mode, void* d_counters);
/* tests only: the int8 filter's certificate, read back.  Brings the index's int8 shadow up to date (as a large-batch search would;
 * nothing else changes) and writes, for nq queries with thresholds tau[nq] (map space, as a range radius) tested in query blocks of
 * query_block (32, 64, 96 or 128) queries, what the filter's consumers and bookkeepers compute (knn_tc.cuh):
 *   out_shape[2]                 the shadow's slots S and its 64-slot blocks B (whole 128-slot tiles)
 *   slot_row[S]                  the row of every slot (0xFFFFFFFF: dead)        rowc[S][4]  (s_v, r_v, n_v, c_v)
 *   blockc[B][8]                 tc_block_consts' record of every block
 *   row_codes[S][dim]            the int8 codes of every slot, un-swizzled       query_codes[nq][dim], qc[nq][4]: tc_prepare_queries
 *   kab[nq / query_block][2]     (ka, kb) of every query block
 *   block_thr[nq][B]             tc_block_threshold of every (query, block)
 *   row_bound[nq][S][2]          (d~, err) of tc_row_bound with x = float(I), I = the int32 dot product of the codes
 * Call it once with every array null to learn S and B.  Any output but out_shape may be null. */
int rxgpu_tc_audit(const rxgpu_index*, uint32_t nq, const float* queries, const float* tau, uint32_t query_block, uint32_t* out_shape,
                   uint32_t* slot_row, float* rowc, float* blockc, signed char* row_codes, signed char* query_codes, float* qc, float* kab,
                   int32_t* block_thr, float* row_bound);

#ifdef __cplusplus
}
#endif
#endif /* RXGPU_H */
