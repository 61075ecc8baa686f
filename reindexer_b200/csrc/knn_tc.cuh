// Tensor-core candidate filter for large query batches (sm_90a: TMA + wgmma + mbarrier, thread-block clusters), exact results.
//
// knn_scan_warp is HBM-bound only while <= ~16 queries share a pass; a batch of 1024 queries is FMA-bound there.  This kernel
// computes APPROXIMATE scores for a block of NQ queries against every row with int8 operands on the tensor cores and keeps, per
// query, only the rows that can still be among the k best under a CERTIFIED error bound; the survivors under the final threshold
// (~65 of ~420 candidates per query at config 1) are then re-ranked with the exact fp32 routine of knn_scan_warp, so the final
// result is identical to the exact scan.
//
// Quantisation (tc_quantize, the same for rows and queries; fp32 vector v of dimension D):
//   scale     s_v = max|v_i| / 127 (fp32; 0 for an all-zero row)      codes  c_v = round(v / s_v), clamped to +-127
//   residual  rho_v = v - s_v c_v                                       r_v >= ||rho_v||, n_v >= ||v||  (fp64 sums, rounded up to fp32)
// The dot product of the codes I = c_q.c_v is EXACT in the s32 wgmma accumulator (|I| <= 2048 * 127^2 < 2^31 for every dimension the
// filter accepts), and with p = s_q s_v I
//   q.v = p + s_q c_q.rho_v + rho_q.v    =>   |q.v - p| <= (n_q + r_q) r_v + r_q n_v
// The exact scan's own fp32 sum differs from q.v by at most D 2^-23 n_q n_v; 16 more units of 2^-23 n_q n_v and a relative 2^-8
// cover the rearranged fp32 arithmetic of the test below, so
//   e(q, v) = (1 + 2^-8) ((n_q + r_q) r_v + (r_q + (D + 16) 2^-23 n_q) n_v)
//   IP      d~ = -p,                  lb/ub = d~ -+ e
//   Cosine  d~ = -p c_v,              lb/ub = d~ -+ e c_v              (c_v = the exact scan's own norm coefficient)
//   L2      d~ = n_q^2 + n_v^2 - 2p,  lb/ub = d~ -+ (2e + eps (n_q^2 + n_v^2)),  eps = kTcL2Eps + (D + 1) 2^-23 (the exact scan's sum
//                                                                                  of squares and the rounding of d~ itself)
// For sigma = 0.25 rows at 768 dims r_v / n_v is about 0.7 %, so e is about 0.015 n_q n_v.
// These relative bounds assume no fp32 underflow.  Below FLT_MIN every rounding of the exact scan's sum and of s_q s_v is absolute,
// up to D 2^-149 in all, which the relative terms cover only while n_q n_v (L2: n_q^2 + n_v^2) stays above about D 2^-142.  A pair
// below kTcTinyNorm2 = 2^-96 therefore gets err = +inf (tc_row_bound: never rejected by its own bound), and the block test passes
// every pair of a query or a row with 0 < n < kTcTinyNorm = 2^-48 (tc_prepare_queries: 1 / k_q = +inf; tc_block_consts: flag 1), so
// that every such pair reaches the exact re-rank.  Rows and queries that small only arise from subnormal-scale data.
//   threshold     tau_q = the largest entry of the query's BOUND LIST: k1 EXACT distances (the exact scan's own arithmetic,
//                 row_dists_warp) of k1 distinct rows (one small list per query in HBM, updated under a per-query lock -- only
//                 O(k log n) successful inserts per query over a whole pass); a row is a candidate iff lb <= tau_q.  The seed
//                 (tc_seed_slices, tc_seed_merge) fills the list with the exact k1 best of the first kTcInitRows rows; a
//                 bookkeeper computes the exact distance d of a candidate row beyond them whose midpoint d~ is below the threshold
//                 and inserts d when it is below it too.
//                 Every list entry is the exact distance of a distinct row (every tile is visited once per query, seed rows are
//                 never inserted again), so tau_q is at or above the final k1-th best exact distance at every moment: every row of
//                 the true top k1 has lb <= d <= tau_q and stays a candidate, and so does every row at or below the k-th distance
//                 (the tie replay from the lists).  Which rows get rescored only decides how fast tau_q tightens, never whether
//                 it is valid.  tau only decreases.  The re-rank gathers only the candidates with lb <= the final tau_q: one with
//                 lb > tau_q has d >= lb > tau_q >= the k1-th best exact distance, so it is neither among the k1 best nor at or
//                 below the k-th distance (the tie replay still reads the full lists).
//   range search  tau_q = the query's radius, seeded by the host and never tightened (init_rows = UINT32_MAX: no row reaches the
//                 bound list, so ub_list, ub_lock and k1 are never read).  A row matches iff its exact distance d < radius, and every
//                 such row has lb <= d < tau_q, so it is a candidate; the exact re-rank (knn_rerank's range mode) then keeps the
//                 candidates with d < radius, computed with the exact scan's arithmetic -- the same set and the same distance bits as
//                 the exact range scan.  Certification needs no upper bound here, only that lb never exceeds d.
//
// Launch shape: one grid covers G query groups (a group = one query block of NQ queries per CTA of a cluster) with W tile walkers
// each, G x W <= the clusters resident at once (config 1, clusters of two: 4 groups x 16 walkers x 2 = 128 CTAs, one launch per
// batch).  Walker w visits the 128-row tiles w, w + W, w + 2W, ..., so every tile is visited once per query, and the G clusters of
// one walker request the same tiles at about the same time: the first read misses to HBM, the others hit L2, and nothing makes one
// cluster wait for another.
//
// Roles (512 threads = four warpgroups, 1 CTA per SM, persistent over 128-row tiles; every thread gets 128 registers, which the
// consumers' int32 accumulators and block test fit; ptxas ignores a setmaxnreg split of 80 for warpgroup 0 and 144 for the
// consumers "to maintain minimum register requirements", so the register file stays evenly split):
//   warp 0       producer: loads the query block (NQ x dim int8 codes) once by TMA, then streams the walker's 64-row shadow blocks
//                in BLOCK ORDER (below), one K chunk (64 rows x 128 codes = 8 KB) per stage, through ONE RING of up to kTcStages
//                stages shared by all consumers.  The shadow is stored TILED and PRE-SWIZZLED in HBM ([64-row block][K chunk]
//                [64 x 128 B in the SWIZZLE_128B pattern]) so a stage is one contiguous 8 KB cp.async.bulk copy (row-major fp32
//                stays the source of truth; the shadow is private, derived).  In a cluster of C = 2 or 4 CTAs, which own C
//                consecutive query blocks, each CTA fetches 1/C of every stage and multicasts it to all C, so the cluster reads
//                each row byte from L2 once instead of C times.
//   warps 1-3    bookkeepers: warp 1 + w serves the candidate queue of consumer warpgroup w (below): the row's own bound, the
//                append to the per-query candidate lists in HBM, the bound list and tau, off the MMA path.
//   warpgroups 1-3   consumers: a walker's 64-row blocks form one sequence i = 0, 1, 2, ..., block i being half i % 2 of the tile
//                walker + (i / 2) W, and consumer warpgroup i % 3 owns block i.  It multiplies the block with the whole query block
//                (wgmma.m64nNQk32.s32.s8.s8, both operands from shared memory, exact int32 accumulators in registers), releases each
//                stage as soon as its MMAs retired, then tests its 64 x NQ scores against tau and hands every hit to its bookkeeper
//                through a queue in shared memory.  The warpgroups take turns issuing their blocks' MMAs in block order, so each
//                warpgroup's epilogue (drain, test, append) overlaps the two other warpgroups' MMAs.
#pragma once
#include <cuda.h>

#include <type_traits>

#include "common.cuh"
#include "knn_scan.cuh"

namespace rxgpu {

constexpr int kTcThreads = 512;
constexpr int kTcConsumers = 3;      // consumer warpgroups, each with its own bookkeeper warp, queue and (thr, P, R) copies
constexpr int kTcTileRows = 128;     // two 64-row blocks (wgmma M = 64)
constexpr int kTcChunkK = 128;       // int8 codes per 128-byte swizzle row
constexpr int kTcStages = 12;        // ring stages (tc_ring_stages takes fewer only where 12 leave no room for the queues)
constexpr int kTcStagesMin = 8;
constexpr int kTcBlockBytes = 64 * kTcChunkK;               // 8 KB: one 64-row shadow block of one K chunk = one stage
constexpr uint32_t kTcMaxNq = 128;   // queries per CTA (wgmma N <= 128 keeps the accumulators at <= 64 registers per thread)
constexpr uint32_t kTcMaxK1 = 128;  // k + 1 <= 128: the bound list is scanned linearly under the per-query lock (larger k: staged)
constexpr float kTcL2Eps = 1e-5f;

struct TcArgs {
	const unsigned char* shadow;  // int8 codes by SLOT, [64-slot block][K chunk][64 slots x 128 B, SWIZZLE_128B pattern pre-applied]
	const float4* rowc;        // [slots padded to whole tiles] (s_v, r_v, n_v, c_v) of the slot's row: scale, residual norm, norm,
								// Cosine coefficient (1 for IP / L2); zero for dead slots and beyond n
	const uint32_t* slot_row;  // [slots] the row a slot holds (kTcDeadSlot: none)
	const float4* blockc;      // [64-slot blocks][2] the block test's row factors of every block (tc_block_consts)
	const float4* qc;          // [nq_total] (s_q, r_q, n_q, 1 / max(s_q, tiny)) of tc_prepare_queries
	unsigned int* tau;         // [nq_total] ordered-uint of the current threshold (map space), shared by all CTAs
	float* ub_list;            // [nq_total][kTcMaxK1] the bound list: the k1 smallest exact distances of the rows inserted by any CTA
							   // (guarded by ub_lock)
	unsigned int* ub_lock;     // [nq_total]
	uint32_t init_rows;        // ROWS [0, init_rows) are already represented in ub_list by the seed (never insert them twice)
	const float* rows;         // fp32 rows [n][pitch] and the Cosine norm coefficients (nullptr otherwise): the bookkeepers' exact
	const float* norm_coefs;   // distances of the rows they insert into the bound list
	const float* qf;           // [nq_total][kchunks * 128] fp32 queries, zero padded (tc_prepare_queries)
	uint32_t pitch;
	uint32_t* cand_rows;       // [nq_total][cand_cap]
	float* cand_lb;            // [nq_total][cand_cap] the lower bound d~ - err of every listed row (KNN with a bound list; else nullptr)
	unsigned int* cand_count;  // [nq_total]
	uint32_t cand_cap;
	uint32_t n;                // slots: a prefix of the shadow's slots (all of them, or a stage's prefix)
	uint32_t dim;
	uint32_t kchunks;          // padded dim / 128
	uint32_t nq_total;         // queries in the whole batch
	uint32_t q0;               // first query of this launch
	uint32_t groups;           // G: query groups of this launch (a group = one query block per CTA of a cluster)
	uint32_t k1;
	int metric;                // kL2 / kIP / kCos
	uint32_t queue_slots;      // records per candidate queue (tc_queue_slots; a power of two)
	uint32_t stages;           // stages of the ring (tc_ring_stages)
	unsigned long long* diag;  // diagnostic instantiations only (kDiag != 0): the counters of tc_diag_* below; unused otherwise
};

// Diagnostic instantiations of knn_tc_filter (template flag kDiag, 0 in every search; bench_tc_phases.py selects one through
// rxgpu_tc_diag).  kTcDiagStamps stamps every phase of every tile with clock64(); the three ablations bound what the epilogue and the
// row stream cost: kTcDiagNoRare compiles the rare path out (the block test stays, hits are only counted, tau never tightens),
// kTcDiagNoFetch lets the producer cycle the barriers without fetching (the consumers multiply zeroed stages), and kTcDiagNoTest
// compiles the block test and the rare path out (ring, MMAs, turns, drain and both bar.syncs stay; the accumulators only feed an XOR sink
// so the MMAs are kept).  Their candidate lists are meaningless; only the time and the counters are read.
constexpr int kTcDiagStamps = 1;
constexpr int kTcDiagNoRare = 2;
constexpr int kTcDiagNoFetch = 3;
constexpr int kTcDiagNoTest = 4;
// a.diag layout: [gridDim.x][kTcDiagSlots] per-CTA counters, then [kTcDiagWalk] hits per walk position (position i = the walker's
// i-th tile, summed over all CTAs), then [gridDim.x][kTcDiagWalk / kTcDiagMarkEvery] %globaltimer marks taken when a CTA starts the
// walk positions 0, kTcDiagMarkEvery, 2 kTcDiagMarkEvery, ...
constexpr uint32_t kTcDiagSlots = 64;
constexpr uint32_t kTcDiagWalk = 8192;
constexpr uint32_t kTcDiagMarkEvery = 64;
// per-CTA counters: consumer warpgroup w at w * kTcDgPerWg + (one of the phases below, in clock64 cycles summed over its four warps;
// blocks, hits and queue waits are counts), the producer at kTcDgEmpty (cycles waiting on `empty`) and kTcDgProd (total)
enum : uint32_t {
	kTcDgFull,     // waiting on full[stage]
	kTcDgMma,      // the rest of the K loop: tau refresh, block constants, MMA issue, wgmma_wait<1>, stage release, handing the turn over
	kTcDgDrain,    // wgmma_wait<0>, the last release and the block thresholds
	kTcDgBar1,     // the first bar.sync
	kTcDgTest,     // the block test: the branch-free loop that builds the hit mask
	kTcDgAppend,   // the vote on the hit masks and the enqueues of the hits (their waits on a full queue included)
	kTcDgTurn,     // waiting for the warpgroup's turn to issue its MMAs (kTcDiagNoTest: the XOR of its accumulators instead, the sink
				   // that keeps its MMAs)
	kTcDgBar2,     // the second bar.sync
	kTcDgTile,     // the whole tile
	kTcDgBlocks,   // 64-row blocks walked (count, per warp)
	kTcDgHits,     // (query, row) pairs that passed the block test (count)
	kTcDgQueueWait,  // enqueues that found the candidate queue full (count)
	kTcDgPerWg,
	kTcDgEmpty = kTcConsumers * kTcDgPerWg,
	kTcDgProd = kTcDgEmpty + 1,
	kTcDgRescored = kTcDgProd + 1,  // bookkeepers (all three warps summed): rows whose exact distance they computed (count), ...
	kTcDgInserts,                   // ... bound-list inserts attempted under the lock (count), ...
	kTcDgRescoreCycles,             // ... and clock64 cycles spent computing those distances (stamped instantiation only)
	kTcDgGathered,                  // CTA 0's slot only: rows knn_rerank gathered after the filter (count)
};
static_assert(kTcDgGathered < kTcDiagSlots, "diagnostic counters fit their slots");

// shared memory: query block, the stage ring, barriers, per-query constants, then per consumer warpgroup thresholds and block thresholds
__host__ __device__ inline size_t tc_smem_bytes(uint32_t nq_block, uint32_t kchunks, uint32_t stages = kTcStages) {
	return 1024 /*align slack*/ + size_t(nq_block) * kchunks * 128 + size_t(stages) * kTcBlockBytes + 256 /*barriers*/ +
		   size_t(nq_block) * (16 /*qc*/ + kTcConsumers * (4 + 4) /*thr, block threshold per warpgroup*/) + 64;
}

// ---- PTX wrappers -------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"WAIT_%=:\n"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
		"@p bra DONE_%=;\n"
		"bra WAIT_%=;\n"
		"DONE_%=:\n"
		"}\n" ::"r"(smem_u32(bar)),
		"r"(parity)
		: "memory");
}
// arrive on the barrier at the same shared-memory offset in CTA `cta` of the cluster (the CTA itself included).  The default
// (CTA-scope) semantics: a consumer signals with it that its wgmma reads of a stage retired, and nothing it wrote has to become
// visible to the peer.  A cluster-scope release made every arrival wait for this thread's outstanding memory operations
// (DESIGN 3.2: 3.7x / 6.7x slower launches in clusters of two / four, the MMA-only floor included).
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
	uint32_t remote;
	asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
	asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int32_t x, int32_t y) {
	asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
					 smem_u32(dst)),
				 "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y)
				 : "memory");
}
// 1-D bulk copies (TMA engine, no tensor map): the shadow is stored pre-swizzled, so a stage is a verbatim contiguous copy
__device__ __forceinline__ void bulk_load(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
				 "r"(bytes), "r"(smem_u32(bar))
				 : "memory");
}
__device__ __forceinline__ void bulk_load_mc(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint16_t mask) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
					 smem_u32(dst)),
				 "l"(src), "r"(bytes), "r"(smem_u32(bar)), "h"(mask)
				 : "memory");
}
// true in exactly one lane of a converged warp (elect.sync): the single-thread TMA instructions are issued under this predicate
// from warp-uniform code, so their operands stay in uniform registers
__device__ __forceinline__ bool elect_one_sync() {
	uint32_t p;
	asm volatile(
		"{\n"
		".reg .pred P;\n"
		"elect.sync _|P, 0xffffffff;\n"
		"selp.u32 %0, 1, 0, P;\n"
		"}\n"
		: "=r"(p));
	return p != 0;
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
	uint32_t r;
	asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
	return r;
}
__device__ __forceinline__ void cluster_sync_all() {
	asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
	asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// wgmma shared-memory matrix descriptor, K-major, SWIZZLE_128B: 8-row groups are 1024 B apart (SBO), one swizzle atom along K
// (LBO unused); the K step of 32 int8 inside the atom advances the start address by 32 bytes
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
	uint64_t d = 0;
	d |= uint64_t((smem_addr & 0x3FFFFu) >> 4);  // start address, bits [0,14)
	d |= uint64_t(1) << 16;                      // leading byte offset (unused for swizzled K-major)
	d |= uint64_t(1024 >> 4) << 32;              // stride byte offset, bits [32,46)
	d |= uint64_t(1) << 62;                      // layout type: SWIZZLE_128B
	return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
	asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// D[64 rows x N queries] (+)= A[64 x 32] (smem) x B[N x 32]^T (smem), s8 in, exact s32 accumulate; d = the thread's N / 2 accumulators
__device__ __forceinline__ void wgmma_m64n32k32(int (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, %18, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
		"{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, "
		"%16, %17, p;\n"
		"}\n"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]),
		  "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
		: "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n64k32(int (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, %34, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n64k32.s32.s8.s8 "
		"{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
		"%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
		"%32, %33, p;\n"
		"}\n"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]),
		  "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
		  "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
		: "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n96k32(int (&d)[48], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, %50, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n96k32.s32.s8.s8 "
		"{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
		"%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
		"%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, "
		"%48, %49, p;\n"
		"}\n"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]),
		  "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
		  "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]),
		  "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47])
		: "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n128k32(int (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, %66, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
		"{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
		"%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
		"%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
		"%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
		"%64, %65, p;\n"
		"}\n"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]),
		  "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]),
		  "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]),
		  "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]),
		  "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]),
		  "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
		: "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <int N>
__device__ __forceinline__ void wgmma_s8(int (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	if constexpr (N == 32) {
		wgmma_m64n32k32(d, adesc, bdesc, accumulate);
	} else if constexpr (N == 64) {
		wgmma_m64n64k32(d, adesc, bdesc, accumulate);
	} else if constexpr (N == 96) {
		wgmma_m64n96k32(d, adesc, bdesc, accumulate);
	} else {
		static_assert(N == 128, "query block of 32, 64, 96 or 128");
		wgmma_m64n128k32(d, adesc, bdesc, accumulate);
	}
}

// The candidate test lb <= tau.  The block bound e <= n_q M_v, with
//   M_v = c_v (a* r_v + b* n_v),   a* >= (1 + 2^-8) (n_q + r_q) / n_q,   b* >= (1 + 2^-8) (r_q + (D + 16) 2^-23 n_q) / n_q
// (a*, b*: the largest over the CTA's query block, computed once per launch), makes the per-row and the per-query factors separate;
// dividing the test by k_q = s_q (1 for an all-zero query, whose codes are zero) gives, with x = I and S_v = s_v c_v,
//   IP, Cosine  x S_v + P M_v + R >= 0               P = n_q / k_q   R = tau / k_q
//   L2          x S_v + P M_v - Z W_v + R >= 0       Z = 1 / k_q     R = (tau - (1 - eps) n_q^2) / (2 k_q)    W_v = (1 - eps) n_v^2 / 2
// For S_v > 0 this is x >= T(q, v) = -R u_v - P (a* rho_v + b* nu_v) + Z w_v with u_v = 1 / S_v, rho_v = r_v / s_v, nu_v = n_v / s_v
// (c_v cancels) and w_v = W_v / S_v (0 for IP and Cosine); P, a*, b*, Z >= 0.  The shadow stores the rows SORTED so that the 64 rows
// of a slot block have nearly equal factors (ensureShadow: by S_v descending; L2 first by coarse buckets of n_v^2), and tc_block_consts
// keeps per block u_lo <= u_v <= u_hi, rho_hi >= rho_v, nu_hi >= nu_v, w_lo <= w_v <= w_hi over its live rows, each rounded outwards
// from fp64 with directed rounding, so with real arithmetic
//   T_B(q) = min(-R u_lo, -R u_hi) - P (a* rho_hi + b* nu_hi) + Z w_lo  <=  T(q, v)   for every live row v of the block.
// The consumer evaluates T_B once per (query, block) in fp32: about ten roundings, each at most 2^-24 of
//   mag = |R| u_hi + P (a* rho_hi + b* nu_hi) + Z w_hi,
// so the computed value is within 2^-20 mag of T_B; it subtracts slack = 2^-18 mag + 1, rounds down to an int and clamps to
// [-2^30, 2^30] (|I| < 2^25 at every accepted dim; +inf only when tau = -inf or a positive term overflows while the others stay
// finite, so the true T_B is far above 2^25 too).  A score then passes when I >= that integer: one integer compare, no conversion.
// Blocks holding a live row with S_v <= 0 (an all-zero row, a zero-norm Cosine row) or any non-finite factor pass every pair
// (threshold -2^30), and so does a NaN threshold, as "not below zero" lets NaN through in the exact form; a block with no live slot
// passes none.  The bookkeeper then decides every hit with the row's own bound e(q, v), exactly as before.
__host__ __device__ __forceinline__ float tc_l2eps(uint32_t dim) { return kTcL2Eps + float(dim + 1) * 0x1p-23f; }
constexpr uint32_t kTcDeadSlot = 0xFFFFFFFFu;
constexpr int kTcPassAll = -(1 << 30), kTcPassNone = 1 << 30;
// tc_block_consts' record of one 64-slot block: (u_lo, u_hi, rho_hi, nu_hi), (w_lo, w_hi, flag, 0); flag 1 = every pair passes,
// -1 = no live slot (no pair passes), 0 = T_B applies
__device__ __forceinline__ int tc_block_threshold(float R, float P, float Z, float ka, float kb, float4 b0, float4 b1) {
	if (b1.z != 0.f) {
		return b1.z > 0.f ? kTcPassAll : kTcPassNone;
	}
	const float m = P * fmaf(ka, b0.z, kb * b0.w);
	const float t = fminf(-R * b0.x, -R * b0.y) - m + Z * b1.x;
	if (t == INFINITY) {  // tau = -inf (a query that admits nothing), or a positive term beyond fp32 with the others finite
		return kTcPassNone;
	}
	const float mag = fmaf(fabsf(R), b0.y, fmaf(Z, b1.y, m));
	const float f = t - fmaf(mag, 0x1p-18f, 1.f);
	if (!(f >= -0x1p30f)) {  // NaN included
		return kTcPassAll;
	}
	return f > 0x1p30f ? kTcPassNone : int(floorf(f));
}
// (a*, b*) of a query block: every thread folds the queries it holds into s_ab[2] (zeroed first) with tc_block_ab_add, and after a
// barrier tc_block_ab_k turns the maxima into the (ka, kb) tc_block_threshold takes.  The filter and rxgpu_tc_audit both call these.
__device__ __forceinline__ void tc_block_ab_add(float* s_ab, float4 qc, float delta) {  // qc = (s_q, r_q, n_q, 1 / k_q)
	if (qc.z > 0.f) {  // non-negative floats order like their bit patterns
		atomicMax(reinterpret_cast<unsigned int*>(&s_ab[0]), __float_as_uint((qc.z + qc.y) / qc.z));
		atomicMax(reinterpret_cast<unsigned int*>(&s_ab[1]), __float_as_uint(qc.y / qc.z + delta));
	}
}
__device__ __forceinline__ float2 tc_block_ab_k(const float* s_ab) {  // 2^-8 of e, and 2^-8 for the rounding of M_v
	return make_float2((1.f + 0x1p-7f) * s_ab[0], (1.f + 0x1p-7f) * s_ab[1]);
}
__device__ __forceinline__ float2 tc_make_pr(int metric, float tau, float4 qc, float l2eps) {  // qc = (s_q, r_q, n_q, 1 / k_q)
	const float p = qc.z * qc.w;
	if (metric != kL2) {
		return make_float2(p, tau * qc.w);
	}
	return make_float2(p, 0.5f * (tau - (1.f - l2eps) * qc.z * qc.z) * qc.w);
}

// ---- the candidate queue: consumers -> bookkeepers --------------------------------------------------------------------------------
// A (query, row) pair that passes the block test is a hit.  The consumer warpgroup that found it only enqueues it: one shared-memory
// atomicAdd takes a ticket, a 16-byte record (query in the block, slot, x = float(I), ticket + 1) goes into the warpgroup's ring of
// `slots` records, the last word stored with release semantics.  Its BOOKKEEPER warp (warp 1 + w for consumer warpgroup w; idle
// otherwise) takes the records in ticket order, up to 32 at a time, frees their slots, and runs the rare path off
// the MMA path: the slot's row, its own bound, the candidate append, the bound list and tau.  A full ring makes the consumer wait until the
// bookkeeper frees a slot; no hit is ever dropped.
struct TcQueue {
	uint32_t tail;        // tickets taken by the consumers
	uint32_t head;        // tickets whose records the bookkeeper has read (their slots are free again)
	uint32_t done;        // consumer warps that finished their walk
	uint32_t full_waits;  // diagnostic instantiations: enqueues that found the ring full
};
constexpr uint32_t kTcQueueMax = 512;  // records per consumer warpgroup at most (3 x 8 KB), ...
constexpr uint32_t kTcQueueMin = 128;  // ... and at least, at every shape tcQueryBlock picks
__host__ __device__ inline size_t tc_queue_bytes(uint32_t slots) {
	return kTcConsumers * sizeof(TcQueue) + size_t(kTcConsumers) * slots * 16;
}
// stages of the ring: kTcStages, or the most below it that leave kTcQueueMin records per queue (1153 to 1280 dims at a query block
// of 96 are the only shapes of tcQueryBlock that need fewer: 11); 0 when even kTcStagesMin stages leave too little
inline uint32_t tc_ring_stages(uint32_t nq_block, uint32_t kchunks, size_t limit) {
	for (uint32_t s = kTcStages; s >= uint32_t(kTcStagesMin); --s) {
		if (tc_smem_bytes(nq_block, kchunks, s) + tc_queue_bytes(kTcQueueMin) <= limit) {
			return s;
		}
	}
	return 0;
}
// records per queue: the largest power of two in [kTcQueueMin, kTcQueueMax] whose queues fit beside the layout tc_smem_bytes counts
// (0: none fits)
inline uint32_t tc_queue_slots(uint32_t nq_block, uint32_t kchunks, uint32_t stages, size_t limit) {
	for (uint32_t s = kTcQueueMax; s >= kTcQueueMin; s /= 2) {
		if (tc_smem_bytes(nq_block, kchunks, stages) + tc_queue_bytes(s) <= limit) {
			return s;
		}
	}
	return 0;
}

__device__ __forceinline__ uint32_t ld_acquire_shared(const uint32_t* p) {
	uint32_t v;
	asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
	return v;
}
__device__ __forceinline__ void st_release_shared(uint32_t* p, uint32_t v) {
	asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}

// consumer side: returns whether the ring was full (the caller waited)
__device__ __forceinline__ bool tc_enqueue(TcQueue* qu, uint4* rec, uint32_t slots, uint32_t q, uint32_t slot, float x) {
	const uint32_t t = atomicAdd(&qu->tail, 1u);
	bool waited = false;
	while (t - ld_acquire_shared(&qu->head) >= slots) {  // the bookkeeper has not read the record this slot held yet
		waited = true;
		__nanosleep(64);
	}
	uint4* r = rec + (t & (slots - 1));
	r->x = q;
	r->y = slot;
	r->z = __float_as_uint(x);
	st_release_shared(&r->w, t + 1);
	return waited;
}

// the hits of one accumulator quad (h = bits 0..3 for (slot0, q), (slot0, q + 1), (slot1, q), (slot1, q + 1)), out of line: inlined at
// each of the kNq / 8 quads of the unrolled append loop it only spreads the consumer loop over more instruction cache
__device__ __noinline__ bool tc_enqueue_quad(TcQueue* qu, uint4* rec, uint32_t slots, uint32_t h, uint32_t q, uint32_t slot0, uint32_t slot1,
											 float x0, float x1, float x2, float x3) {
	bool waited = false;
	if (h & 1u) waited |= tc_enqueue(qu, rec, slots, q, slot0, x0);
	if (h & 2u) waited |= tc_enqueue(qu, rec, slots, q + 1, slot0, x1);
	if (h & 4u) waited |= tc_enqueue(qu, rec, slots, q, slot1, x2);
	if (h & 8u) waited |= tc_enqueue(qu, rec, slots, q + 1, slot1, x3);
	return waited;
}

// The row's own bound: d~ and its certified error (header comment), from x = float(I) and the query's and the row's constants.  A
// pair below kTcTinyNorm2 (header comment) gets an infinite error: its own bound never rejects it.
constexpr float kTcTinyNorm = 0x1p-48f, kTcTinyNorm2 = 0x1p-96f;
__device__ __forceinline__ float2 tc_row_bound(const TcArgs& a, float x, float4 qc, float4 rc) {
	const float p = qc.x * rc.x * x;
	const float e = (1.f + 0x1p-8f) * fmaf(qc.z + qc.y, rc.y, (qc.y + float(a.dim + 16) * 0x1p-23f * qc.z) * rc.z);
	if (a.metric == kL2) {
		const float nn = qc.z * qc.z + rc.z * rc.z;
		return make_float2(fmaf(-2.f, p, fmaf(qc.z, qc.z, rc.z * rc.z)), nn < kTcTinyNorm2 ? INFINITY : 2.f * e + tc_l2eps(a.dim) * nn);
	}
	const float err = qc.z * rc.z < kTcTinyNorm2 ? INFINITY : e;
	if (a.metric == kCos) {
		return make_float2(-p * rc.w, err * rc.w);
	}
	return make_float2(-p, err);
}

// Exact distance d of a row below the query's threshold: insert it into the query's global bound list (under the per-query lock;
// other CTAs contend) and tighten the global tau.  Returns the list's largest entry afterwards, the query's new threshold.
__device__ __noinline__ float tc_bound_insert(const TcArgs& a, uint32_t q, float ub) {
	while (atomicCAS(&a.ub_lock[q], 0u, 1u) != 0u) {
	}
	__threadfence();
	volatile float* list = a.ub_list + size_t(q) * kTcMaxK1;
	uint32_t mi = 0;
	float mx = list[0];
	for (uint32_t x = 1; x < a.k1; ++x) {
		const float y = list[x];
		if (y > mx) {
			mx = y;
			mi = x;
		}
	}
	float tightened = mx;
	if (ub < mx) {
		list[mi] = ub;
		float nmx = list[0];
		for (uint32_t x = 1; x < a.k1; ++x) {
			nmx = fmaxf(nmx, list[x]);
		}
		atomicMin(&a.tau[q], float_ord(nmx));
		tightened = nmx;
	}
	__threadfence();
	atomicExch(&a.ub_lock[q], 0u);
	return tightened;
}

// The exact distances of the rows flagged in `todo` (one row per lane: row, query ql of the CTA's block), kTcRescoreRows rows in
// flight per pass of the warp; lane l gets its own row's distance.
constexpr int kTcRescoreRows = 4;
template <bool kIsL2>
__device__ __noinline__ float tc_rescore(const TcArgs& a, unsigned todo, uint32_t row, uint32_t ql, uint32_t q0, int lane) {
	const uint32_t nch = a.kchunks, pitch4 = a.pitch >> 2;
	const float4* rows4 = reinterpret_cast<const float4*>(a.rows);
	float mine = 0.f;
	while (todo) {
		uint32_t rr[kTcRescoreRows];
		const float4* qp[kTcRescoreRows][1];
		int who[kTcRescoreRows];
#pragma unroll
		for (int i = 0; i < kTcRescoreRows; ++i) {
			who[i] = todo ? __ffs(todo) - 1 : who[0];  // a short last pass repeats its first row
			todo &= todo - 1u;
			rr[i] = __shfl_sync(0xffffffffu, row, who[i]);
			qp[i][0] = reinterpret_cast<const float4*>(a.qf) + size_t(q0 + __shfl_sync(0xffffffffu, ql, who[i])) * nch * 32u;
		}
		float d[kTcRescoreRows][1];
		row_dists_warp<kIsL2, kTcRescoreRows, 1>(rows4, pitch4, nch, rr, qp, a.norm_coefs, lane, d);
#pragma unroll
		for (int i = 0; i < kTcRescoreRows; ++i) {
			mine = lane == who[i] ? d[i][0] : mine;
		}
	}
	return mine;
}

// Bookkeeper warp of one consumer warpgroup's queue, until every consumer warp is done and the ring is empty.  A hit's slot is mapped
// to its row (a dead slot is dropped); the row is appended
// when its own lower bound d~ - err passes the tightest threshold the CTA knows for the query (NaN: appended); the appends of one
// batch go to the candidate lists with one global atomicAdd per distinct query.  When the row's midpoint d~ beats that threshold
// (and the seed does not hold the row already) the warp computes the row's EXACT distance d with the exact scan's arithmetic; a d
// below the threshold goes into the bound list, and the threshold that comes back is published to the threshold of EVERY consumer
// warpgroup, which turns it into its next block thresholds.  A consumer may read a looser threshold meanwhile (a concurrent store of another writer may even replace a tighter one):
// every threshold ever published is a valid upper bound of the query's final k1-th distance, so the test stays certified.
template <int kNq>
__device__ __forceinline__ float tc_min_thr(const float* s_thr, uint32_t ql) {  // the tightest threshold of the consumer warpgroups
	float t = s_thr[ql];
#pragma unroll
	for (int w = 1; w < kTcConsumers; ++w) {
		t = fminf(t, s_thr[w * kNq + ql]);
	}
	return t;
}
template <int kNq, int kDiag>
__device__ __forceinline__ void tc_bookkeeper(const TcArgs& a, TcQueue* qu, const uint4* rec, uint32_t slots, uint32_t q0, const float4* s_qc,
											  float* s_thr, int lane, unsigned long long* dg) {
	[[maybe_unused]] unsigned long long n_rescored = 0, n_inserts = 0;
	[[maybe_unused]] long long rescore_cycles = 0;
	uint32_t head = 0;
	for (;;) {
		const bool fin = ld_acquire_shared(&qu->done) == 4;  // read before the tail: after it, the tail is final
		const uint32_t n = __shfl_sync(0xffffffffu, min(ld_acquire_shared(&qu->tail) - head, 32u), 0);
		if (n == 0) {
			if (__shfl_sync(0xffffffffu, fin, 0)) {
				break;
			}
			__nanosleep(256);
			continue;
		}
		bool active = uint32_t(lane) < n;
		uint32_t ql = 0, slot = 0;
		float x = 0.f;
		if (active) {
			const uint32_t t = head + lane;
			const uint4* r = rec + (t & (slots - 1));
			while (ld_acquire_shared(&r->w) != t + 1) {  // the consumer holding ticket t has not stored its record yet
			}
			ql = r->x;
			slot = r->y;
			x = __uint_as_float(r->z);
		}
		__syncwarp();
		head += n;
		if (lane == 0) {
			st_release_shared(&qu->head, head);  // the records are read: their slots go back to the consumers
		}
		const uint32_t row = active ? a.slot_row[slot] : kTcDeadSlot;
		active = active && row != kTcDeadSlot;
		float d = 0.f, err = 0.f, tau = 0.f;
		if (active) {
			const float4 qc = s_qc[ql], rc = a.rowc[slot];
			const float2 de = tc_row_bound(a, x, qc, rc);
			d = de.x;
			err = de.y;
			tau = tc_min_thr<kNq>(s_thr, ql);
		}
		const bool append = active && !(d - err > tau);
		const unsigned peers = __match_any_sync(0xffffffffu, append ? ql : ~0u);
		const int leader = __ffs(peers) - 1;
		unsigned base = 0;
		if (append && lane == leader) {
			base = atomicAdd(&a.cand_count[q0 + ql], unsigned(__popc(peers)));
		}
		base = __shfl_sync(0xffffffffu, base, leader);
		if (append) {
			const unsigned pos = base + __popc(peers & ((1u << lane) - 1u));
			if (pos < a.cand_cap) {
				a.cand_rows[size_t(q0 + ql) * a.cand_cap + pos] = row;
				if (a.cand_lb != nullptr) {
					a.cand_lb[size_t(q0 + ql) * a.cand_cap + pos] = d - err;
				}
			}
		}
		// the midpoint rather than the upper bound d + err: tau then follows the k1-th best exact distance instead of trailing it by
		// about err (DESIGN 3.2: 490 against 780 candidates per query at config 1, and the faster step)
		const bool rescore = append && row >= a.init_rows && d < tau;  // NaN: never
		const unsigned todo = __ballot_sync(0xffffffffu, rescore);
		if (todo) {
			[[maybe_unused]] const long long c0 = kDiag == kTcDiagStamps ? clock64() : 0ll;
			const float dx = a.metric == kL2 ? tc_rescore<true>(a, todo, row, ql, q0, lane) : tc_rescore<false>(a, todo, row, ql, q0, lane);
			if constexpr (kDiag != 0) {
				n_rescored += __popc(todo);
				if constexpr (kDiag == kTcDiagStamps) {
					rescore_cycles += clock64() - c0;
				}
			}
			if (rescore && dx < tc_min_thr<kNq>(s_thr, ql)) {  // the threshold may have dropped while the batch was rescored
				if constexpr (kDiag != 0) {
					++n_inserts;
				}
				const float nt = tc_bound_insert(a, q0 + ql, dx);
				for (uint32_t w = 0; w < kTcConsumers; ++w) {
					if (nt < s_thr[w * kNq + ql]) {
						s_thr[w * kNq + ql] = nt;
					}
				}
			}
		}
		__syncwarp();
	}
	if constexpr (kDiag != 0) {
		const unsigned long long ins = __reduce_add_sync(0xffffffffu, uint32_t(n_inserts));
		if (lane == 0) {
			atomicAdd(&dg[kTcDgRescored], n_rescored);
			atomicAdd(&dg[kTcDgInserts], ins);
			atomicAdd(&dg[kTcDgRescoreCycles], (unsigned long long)rescore_cycles);
		}
	}
}

// ---- the filter kernel -----------------------------------------------------------------------------------------------------------
// kNq = queries per CTA (wgmma N); kCluster = CTAs that walk the same row tiles with DIFFERENT query blocks, sharing every stage
// through TMA multicast.
template <int kNq, int kCluster, int kDiag = 0>
__global__ void __launch_bounds__(kTcThreads, 1)
	knn_tc_filter(const __grid_constant__ CUtensorMap map_queries, const __grid_constant__ TcArgs a) {
	static_assert(kNq % 32 == 0 && kNq <= int(kTcMaxNq), "query block");
	static_assert(kCluster == 1 || kCluster == 2 || kCluster == 4, "a stage is split in 1, 2 or 4 equal copies");
	constexpr bool kStamp = kDiag == kTcDiagStamps;
	auto clk = [] {  // 0 outside the stamped instantiation, where every stamp and sum below folds away
		if constexpr (kStamp) {
			return clock64();
		} else {
			return 0ll;
		}
	};
	unsigned long long* dg = kDiag ? a.diag + size_t(blockIdx.x) * kTcDiagSlots : nullptr;
	extern __shared__ unsigned char smem_raw[];
	unsigned char* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // offset arithmetic keeps the shared window
	constexpr uint32_t kQchunkBytes = kNq * 128;                       // one K-chunk of the query block: kNq rows x 128 B
	unsigned char* s_q = base;                                         // [kchunks][kNq][128 B], swizzled by TMA
	unsigned char* s_rows = s_q + size_t(a.kchunks) * kQchunkBytes;    // [stages][64][128 B]   (1024-aligned: kNq % 8 == 0)
	const uint32_t nstages = a.stages;
	uint64_t* bars = reinterpret_cast<uint64_t*>(s_rows + size_t(nstages) * kTcBlockBytes);
	uint64_t* full_bar = bars;                       // [stages] TMA -> MMA
	uint64_t* empty_bar = bars + kTcStages;          // [stages] MMA (the consumer warps of the stage's block in every CTA of the cluster) -> TMA
	uint64_t* q_bar = bars + 2 * kTcStages;          // queries resident
	float* s_ab = reinterpret_cast<float*>(q_bar + 1);                 // (a*, b*) of the block bound
	float4* s_qc = reinterpret_cast<float4*>(bars + 32);               // [kNq] (s_q, r_q, n_q, 1 / k_q)
	float* s_thr = reinterpret_cast<float*>(s_qc + kNq);               // [3][kNq] current tau (map space), per consumer warpgroup
	int* s_tb = reinterpret_cast<int*>(s_thr + kTcConsumers * kNq);    // [3][kNq] the block thresholds of each warpgroup's current block
	TcQueue* s_queue = reinterpret_cast<TcQueue*>(s_tb + kTcConsumers * kNq);  // [3] candidate queue of each consumer warpgroup
	uint4* s_rec = reinterpret_cast<uint4*>(s_queue + kTcConsumers);  // [3][queue_slots] their records (beyond tc_smem_bytes)
	static_assert(2 * kTcStages + 2 <= 32, "barriers and (a*, b*) fit in front of the per-query constants");

	const int warp = __shfl_sync(0xffffffffu, int(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;  // provably warp-uniform
	const uint32_t ntiles = (a.n + kTcTileRows - 1) / kTcTileRows;
	const uint32_t crank = kCluster > 1 ? cluster_ctarank() : 0u;
	// launch shape (header comment): cluster cid serves query group cid % G as walker cid / G of W = ncl / G
	const uint32_t cid = blockIdx.x / kCluster, ncl = gridDim.x / kCluster;
	const uint32_t walker = cid / a.groups, walkers = ncl / a.groups;
	const uint32_t q0 = a.q0 + ((cid % a.groups) * kCluster + crank) * kNq;
	const uint32_t nq_valid = q0 < a.nq_total ? min(uint32_t(kNq), a.nq_total - q0) : 0u;
	const float l2eps = tc_l2eps(a.dim);

	if (threadIdx.x == 0) {
		for (uint32_t s = 0; s < nstages; ++s) {
			mbar_init(&full_bar[s], 1);
			mbar_init(&empty_bar[s], 4 * kCluster);  // the four warps of the warpgroup that owns the stage's block, in every CTA that reads it
		}
		mbar_init(q_bar, 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		s_ab[0] = s_ab[1] = 0.f;
		for (int w = 0; w < kTcConsumers; ++w) {
			s_queue[w] = TcQueue{0u, 0u, 0u, 0u};
		}
	}
	for (uint32_t i = threadIdx.x; i < kTcConsumers * a.queue_slots; i += blockDim.x) {
		s_rec[i].w = 0u;  // no ticket yet (a record of ticket t carries t + 1)
	}
	if constexpr (kDiag == kTcDiagNoFetch) {  // the stages the consumers multiply without a fetch hold zero codes
		for (uint32_t i = threadIdx.x; i < nstages * kTcBlockBytes / 16; i += blockDim.x) {
			reinterpret_cast<uint4*>(s_rows)[i] = make_uint4(0u, 0u, 0u, 0u);
		}
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
	}
	__syncthreads();
	const float delta = float(a.dim + 16) * 0x1p-23f;
	for (uint32_t i = threadIdx.x; i < kNq; i += blockDim.x) {
		const bool valid = i < nq_valid;
		const float thr = valid ? ord_float(a.tau[q0 + i]) : -INFINITY;
		const float4 qc = valid ? a.qc[q0 + i] : make_float4(0.f, 0.f, 0.f, 0.f);
		tc_block_ab_add(s_ab, qc, delta);
		s_qc[i] = qc;
		for (int w = 0; w < kTcConsumers; ++w) {
			s_thr[w * kNq + i] = thr;
			s_tb[w * kNq + i] = kTcPassNone;  // padding queries never match; valid ones are set before every block test
		}
	}
	__syncthreads();
	if constexpr (kCluster > 1) {
		cluster_sync_all();  // the peers' barriers exist before anything of ours can signal them
	}
	// the walker's 64-row blocks i = 0, 1, ..., nblocks - 1: block i is half i % 2 of the tile walker + (i / 2) walkers, shadow block
	// 2 (walker + (i / 2) walkers) + i % 2; its K chunk kc is the (i kchunks + kc)-th stage the producer fills
	const uint32_t nblocks = walker < ntiles ? 2 * ((ntiles - walker + walkers - 1) / walkers) : 0u;

	if (warp == 0) {
		// ===== TMA producer: the whole warp walks the loop, one elected lane issues (operands stay in uniform registers)
		if (elect_one_sync()) {
			mbar_expect_tx(q_bar, a.kchunks * kQchunkBytes);
			for (uint32_t kc = 0; kc < a.kchunks; ++kc) {
				tma_load_2d(s_q + size_t(kc) * kQchunkBytes, &map_queries, q_bar, int32_t(kc * kTcChunkK), int32_t(q0));
			}
		}
		__syncwarp();
		uint64_t* full = full_bar;
		uint64_t* empty = empty_bar;
		unsigned char* ring_smem = s_rows;
		uint32_t stage = 0, phase = 0;
		[[maybe_unused]] long long t_empty = 0;
		[[maybe_unused]] const long long t_start = clk();
		for (uint32_t i = 0; i < nblocks; ++i) {
			// the walker's block i, its K chunks 8 KB apart in HBM
			const unsigned char* src = a.shadow + size_t(2 * (walker + (i >> 1) * walkers) + (i & 1u)) * a.kchunks * kTcBlockBytes;
			for (uint32_t kc = 0; kc < a.kchunks; ++kc) {
				[[maybe_unused]] const long long c0 = clk();
				mbar_wait(&empty[stage], phase ^ 1);
				if constexpr (kStamp) {
					t_empty += clk() - c0;
				}
				unsigned char* dst = ring_smem + size_t(stage) * kTcBlockBytes;
				if constexpr (kDiag == kTcDiagNoFetch) {
					if (elect_one_sync()) {
						mbar_arrive(&full[stage]);
					}
				} else if (elect_one_sync()) {
					mbar_expect_tx(&full[stage], kTcBlockBytes);
					if constexpr (kCluster == 1) {
						bulk_load(dst, src + size_t(kc) * kTcBlockBytes, kTcBlockBytes, &full[stage]);
					} else {  // my 1/C of the stage, delivered to every CTA of the cluster
						constexpr uint32_t kPart = kTcBlockBytes / kCluster;
						bulk_load_mc(dst + crank * kPart, src + size_t(kc) * kTcBlockBytes + crank * kPart, kPart, &full[stage],
									 uint16_t((1u << kCluster) - 1u));
					}
				}
				__syncwarp();
				if (++stage == nstages) {
					stage = 0;
					phase ^= 1;
				}
			}
		}
		if constexpr (kStamp) {
			if (lane == 0) {
				atomicAdd(&dg[kTcDgEmpty], (unsigned long long)t_empty);
				atomicAdd(&dg[kTcDgProd], (unsigned long long)(clk() - t_start));
			}
		}
	} else if (warp < 4) {
		// ===== bookkeeper of consumer warpgroup warp - 1 =====
		const uint32_t wg = uint32_t(warp) - 1;
		tc_bookkeeper<kNq, kDiag>(a, s_queue + wg, s_rec + wg * a.queue_slots, a.queue_slots, q0, s_qc, s_thr, lane, dg);
	} else {
		// ===== consumer warpgroup wg: the walker's blocks i = wg, wg + 3, wg + 6, ... =====
		const uint32_t wg = uint32_t(warp) / 4 - 1, wtid = threadIdx.x - 128 * (wg + 1);
		float* thr = s_thr + wg * kNq;
		int* tb = s_tb + wg * kNq;
		TcQueue* qu = s_queue + wg;
		uint4* rec = s_rec + wg * a.queue_slots;
		const uint32_t slots = a.queue_slots;
		uint64_t* full = full_bar;
		uint64_t* empty = empty_bar;
		const unsigned char* ring_smem = s_rows;
		// accumulator fragment of wgmma.m64nN: d[4j + {0,1}] = (row r0, query 8j + 2c + {0,1}), d[4j + {2,3}] = the same for row r0 + 8
		const uint32_t r0 = (wtid >> 5) * 16 + (lane >> 2), c2 = 2 * (lane & 3);
		const uint32_t my_q = wtid;  // the query whose threshold this thread refreshes from the global list and turns into block thresholds
		unsigned int tau_ahead = my_q < nq_valid ? a.tau[q0 + my_q] : 0u;
		const bool l2 = a.metric == kL2;
		const float2 kab = tc_block_ab_k(s_ab);
		const float ka = kab.x, kb = kab.y;
		auto release = [&](uint32_t st) {  // this warp is done with stage st in every CTA that reads it: lane c signals CTA c
			if constexpr (kCluster == 1) {
				if (lane == 0) {
					mbar_arrive(&empty[st]);
				}
			} else if (lane < kCluster) {
				mbar_arrive_cluster(&empty[st], uint32_t(lane));
			}
		};
		mbar_wait(q_bar, 0);
		[[maybe_unused]] long long dt[kTcDgPerWg] = {};  // kStamp: this warp's cycles per phase (kTcDg*)
		[[maybe_unused]] unsigned long long nhits = 0;
		[[maybe_unused]] uint32_t sink = 0;  // kTcDiagNoTest
		for (uint32_t blk = wg; blk < nblocks; blk += kTcConsumers) {
			const uint32_t t = walker + (blk >> 1) * walkers, half = blk & 1u;
			[[maybe_unused]] const uint32_t walk = blk >> 1;
			[[maybe_unused]] long long s0 = clk(), s1, s2, s3, s4, s5;
			if constexpr (kStamp) {
				if (half == 0 && wtid == 0 && walk % kTcDiagMarkEvery == 0 && walk < kTcDiagWalk) {
					unsigned long long now;
					asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
					a.diag[size_t(gridDim.x) * kTcDiagSlots + kTcDiagWalk + size_t(blockIdx.x) * (kTcDiagWalk / kTcDiagMarkEvery) +
						   walk / kTcDiagMarkEvery] = now;
				}
			}
			// refresh tau from the other CTAs: the global load was issued during the PREVIOUS block, so its latency is hidden
			if (my_q < nq_valid) {
				const float tn = ord_float(tau_ahead);
				if (tn < thr[my_q]) {
					thr[my_q] = tn;
				}
				tau_ahead = a.tau[q0 + my_q];
			}
			const uint32_t sb = 2 * t + half, slot0 = sb * 64 + r0, slot1 = slot0 + 8;
			// the block's row factors (slots are padded to whole tiles), consumed after the MMAs by the threads that own a query
			float4 bc0 = {}, bc1 = {};
			if (my_q < nq_valid) {
				bc0 = a.blockc[2 * sb];
				bc1 = a.blockc[2 * sb + 1];
			}
			int acc[kNq / 2];
#pragma unroll
			for (int i = 0; i < kNq / 2; ++i) {
				acc[i] = 0;
			}
			// Warpgroup turns: the three consumer warpgroups issue their blocks' MMAs in block order, so each one's drain, test and
			// append run under the two others' MMAs instead of all of them testing at once while the tensor pipe idles.  The owner of
			// block blk waits on named barrier 4 + blk % 3 (its own), except for block 0; the owner of block blk - 1 arrives on it
			// once it has issued that block's last chunk, and only if block blk exists, so every wait has exactly one arrival and no
			// arrival is left pending at exit, whatever the walker's block count (0, 1, 2 or any residue mod 3).  A barrier never
			// holds two pending arrivals: the arrival for block j needs block j - 1 issued, which needs block j - 1's wait completed,
			// which needs block j - 2 issued and so block j - 3's wait completed -- the previous use of the same barrier.  No
			// deadlock: the producer fills the ring strictly in block order and a consumer consumes in the same order, so by induction
			// over the global chunk index g = blk kchunks + kc every chunk below g is issued; the stage chunk g needs was then released
			// (chunk g - stages is released when chunk g - stages + 1 of the same block is issued, or by the drain of a block's last
			// chunk, which waits on nothing), so chunk g arrives, and its owner's turn came with the last chunk of block blk - 1.  The
			// producer and the bookkeepers never wait on a turn.  In a cluster of C CTAs all of them walk the same blocks in the same
			// order with the same owners, the turns and the bookkeepers stay per CTA, and the induction runs over the chunks of all C:
			// if every chunk below g is issued in every CTA, then chunk g - stages was released in every CTA (its owner releases it
			// in all C CTAs -- lane c of each of its four warps arrives on `empty` of CTA c, 4 C arrivals per phase -- once its own
			// MMAs on it retired), so every producer's wait on that stage's `empty` completes and each issues its 1/C of chunk g into
			// all C CTAs; `full` of chunk g then completes in every CTA (one local expect_tx arrival, C parts of complete_tx, some of
			// which may land before the expect_tx: the transaction count may go transiently negative), and each owner's turn came
			// as in one CTA.  A peer that is ahead waits only on barriers our side will arrive on; no CTA leaves before the exit
			// cluster sync, so no multicast or remote arrival targets a CTA that has exited.
			const uint32_t g0 = blk * a.kchunks;
			uint32_t stage = g0 % nstages, phase = (g0 / nstages) & 1u;
			[[maybe_unused]] const long long c_turn = clk();
			if (blk != 0) {
				asm volatile("bar.sync %0, 256;" ::"r"(4 + wg) : "memory");
			}
			if constexpr (kStamp) {
				dt[kTcDgTurn] += clk() - c_turn;
			}
			uint32_t prev = 0;
			for (uint32_t kc = 0; kc < a.kchunks; ++kc) {
				[[maybe_unused]] const long long c0 = clk();
				mbar_wait(&full[stage], phase);
				if constexpr (kStamp) {
					dt[kTcDgFull] += clk() - c0;
				}
				const uint32_t a_addr = smem_u32(ring_smem + size_t(stage) * kTcBlockBytes);
				const uint32_t b_addr = smem_u32(s_q + size_t(kc) * kQchunkBytes);
				wgmma_fence();
#pragma unroll
				for (uint32_t k = 0; k < kTcChunkK / 32; ++k) {  // K = 32 int8 = 32 bytes inside the 128-byte swizzle row
					wgmma_s8<kNq>(acc, wgmma_desc_sw128(a_addr + k * 32), wgmma_desc_sw128(b_addr + k * 32), (kc | k) != 0);
				}
				wgmma_commit();
				if (kc > 0) {  // the previous chunk's MMAs have retired: its stage goes back to the producer
					wgmma_wait<1>();
					release(prev);
				}
				prev = stage;
				if (++stage == nstages) {
					stage = 0;
					phase ^= 1;
				}
			}
			// hand the turn to the owner of block blk + 1 once the last chunk is issued, before it retires (if that block exists)
			if (blk + 1 < nblocks) {
				asm volatile("bar.arrive %0, 256;" ::"r"(4 + (wg + 1) % kTcConsumers) : "memory");
			}
			s1 = clk();
			wgmma_wait<0>();
			release(prev);
			// this block's threshold of query my_q (header of tc_block_threshold), from the tightest tau this warpgroup knows now
			if (my_q < nq_valid) {
				const float4 qc = s_qc[my_q];
				const float2 pr = tc_make_pr(a.metric, thr[my_q], qc, l2eps);
				tb[my_q] = tc_block_threshold(pr.y, pr.x, l2 ? qc.w : 0.f, ka, kb, bc0, bc1);
			}
			s2 = clk();
			asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");  // the block thresholds of all queries are visible
			s3 = clk();
			// The block test: the predicate of every accumulator into the hit mask, bit i for acc[i] (quad j: bits 4j + {0, 1, 2, 3} =
			// (slot0, q), (slot0, q + 1), (slot1, q), (slot1, q + 1)): one integer compare per score against the (query, block)
			// threshold.  No call and no branch in the loop; the slots beyond n are masked out of every quad at once after it, and the
			// hits, about one per block, are appended after that.
			const uint32_t ok = (slot0 < a.n ? 0x33333333u : 0u) | (slot1 < a.n ? 0xCCCCCCCCu : 0u);
			constexpr int kMaskWords = (kNq / 2 + 31) / 32;
			uint32_t hm[kMaskWords] = {};
			if constexpr (kDiag == kTcDiagNoTest) {
#pragma unroll
				for (int i = 0; i < kNq / 2; ++i) {
					sink ^= uint32_t(acc[i]);
				}
			} else {
#pragma unroll
				for (int j = 0; j < kNq / 8; ++j) {
					const int2 t2 = *reinterpret_cast<const int2*>(&tb[8 * j + c2]);  // thresholds of queries q and q + 1
					const bool h0 = acc[4 * j] >= t2.x, h1 = acc[4 * j + 1] >= t2.y;
					const bool h2 = acc[4 * j + 2] >= t2.x, h3 = acc[4 * j + 3] >= t2.y;
					hm[4 * j / 32] |= (uint32_t(h0) | uint32_t(h1) << 1 | uint32_t(h2) << 2 | uint32_t(h3) << 3) << (4 * j % 32);
				}
			}
#pragma unroll
			for (int w = 0; w < kMaskWords; ++w) {
				hm[w] &= ok;
			}
			s4 = clk();
			// the append (rare path): one vote per warp, then the lanes with hits hand them to the bookkeeper quad by quad, x = float(I)
			// taken again from the accumulator
			[[maybe_unused]] uint32_t nh = 0;
#pragma unroll
			for (int w = 0; w < kMaskWords; ++w) {
				nh += __popc(hm[w]);
			}
			if constexpr (kDiag != 0) {
				nhits += nh;
			}
			if constexpr (kDiag != kTcDiagNoRare && kDiag != kTcDiagNoTest) {
				if (__any_sync(0xffffffffu, nh != 0)) {
#pragma unroll
					for (int j = 0; j < kNq / 8; ++j) {
						const uint32_t h = hm[4 * j / 32] >> (4 * j % 32) & 15u;
						if (h) {
							const bool waited = tc_enqueue_quad(qu, rec, slots, h, 8 * j + c2, slot0, slot1, float(acc[4 * j]), float(acc[4 * j + 1]),
																float(acc[4 * j + 2]), float(acc[4 * j + 3]));
							if constexpr (kStamp) {
								if (waited) {
									atomicAdd(&qu->full_waits, 1u);
								}
							}
						}
					}
				}
			}
			__syncwarp();  // the rare path diverges (per-lane queue waits): reconverge before the .aligned wgmma of the next block
			s5 = clk();
			asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");  // nobody still reads tb when the next block's thresholds are written
			if constexpr (kStamp) {
				const long long s6 = clk();
				dt[kTcDgMma] += s1 - s0;
				dt[kTcDgDrain] += s2 - s1;
				dt[kTcDgBar1] += s3 - s2;
				dt[kTcDgTest] += s4 - s3;
				dt[kTcDgAppend] += s5 - s4;
				dt[kTcDgBar2] += s6 - s5;
				dt[kTcDgTile] += s6 - s0;
				dt[kTcDgBlocks] += 1;
				const uint32_t h = __reduce_add_sync(0xffffffffu, nh);
				if (lane == 0 && h && walk < kTcDiagWalk) {
					atomicAdd(&a.diag[size_t(gridDim.x) * kTcDiagSlots + walk], (unsigned long long)h);
				}
			}
		}
		__syncwarp();
		if (lane == 0) {  // this warp's tickets are all taken: once all four warps are done, the bookkeeper drains and leaves
			__threadfence_block();
			atomicAdd(&qu->done, 1u);
		}
		if constexpr (kDiag != 0) {
			const uint32_t h = __reduce_add_sync(0xffffffffu, uint32_t(nhits));
			const uint32_t x = __reduce_xor_sync(0xffffffffu, sink);
			if (lane == 0) {
				atomicAdd(&dg[wg * kTcDgPerWg + kTcDgHits], (unsigned long long)h);
				if constexpr (kDiag == kTcDiagNoTest) {
					atomicXor(&dg[wg * kTcDgPerWg + kTcDgTurn], (unsigned long long)x);
				}
				if constexpr (kStamp) {
					dt[kTcDgMma] -= dt[kTcDgFull] + dt[kTcDgTurn];  // the K loop's waits are counted on their own
					for (uint32_t i = 0; i < kTcDgPerWg; ++i) {
						if (i != kTcDgHits) {
							atomicAdd(&dg[wg * kTcDgPerWg + i], (unsigned long long)dt[i]);
						}
					}
				}
			}
		}
	}
	__syncthreads();  // every bookkeeper has drained its queue
	if constexpr (kStamp) {
		if (threadIdx.x < kTcConsumers) {
			dg[threadIdx.x * kTcDgPerWg + kTcDgQueueWait] = s_queue[threadIdx.x].full_waits;
		}
	}
	if constexpr (kCluster > 1) {
		cluster_sync_all();  // nobody leaves while a peer may still multicast into this CTA or signal its barriers
	}
}

// ---- exact re-rank of the candidates ----------------------------------------------------------------------------------------------
// One CTA per query: its 8 warps stream the candidate rows of that query (gathered 128-bit coalesced loads), compute the exact fp32
// distance with the SAME per-row arithmetic sequence as knn_scan_warp (so distances are bit-identical to the exact scan), keep the
// best k1 keys per warp, merge in the CTA and write one ascending list [k1] per query.
template <bool kIsL2>
__global__ void __launch_bounds__(kScanThreads) knn_rerank(const float* rows, uint32_t pitch, uint32_t dim, const float* norm_coefs,
															const float* queries, const uint32_t* cand_rows, const unsigned int* cand_count,
															uint32_t cand_cap, uint32_t k1, uint64_t* lists /* [gridDim.x][k1] */,
															const uint32_t* qsel = nullptr, const float* tie_bound = nullptr,
															const float* radius = nullptr, uint64_t* range_keys = nullptr,
															unsigned int* range_count = nullptr, const float* cand_lb = nullptr,
															const unsigned int* tau = nullptr, unsigned long long* gathered = nullptr) {
	// qsel: CTA b serves query qsel[b] (default: query b).  tie_bound != nullptr = tie mode (kModeTieRows): among the candidates
	// with dist <= tie_bound[b], the first k1 in internal row order (key = row << 32 | ord(dist)) -- every row at or below the k-th
	// distance is a candidate, so this replaces a second scan of the whole shard when the reference's tie rule must be replayed.
	// radius != nullptr = range mode: every candidate with dist < radius[q] (strict, as the exact range scan) is appended, unordered,
	// as make_key(dist, row) to range_keys[q][cand_cap] and counted in range_count[q]; lists and k1 are not used.  The matches are a
	// subset of the query's candidates, so they never exceed cand_cap.
	// cand_lb != nullptr (top-k mode after a filter with a bound list): candidate i is gathered only when cand_lb[q][i] <= the final
	// threshold ord_float(tau[q]) (NaN: gathered).  Its exact distance is at or above its lower bound, and the final threshold is at
	// or above the k1-th best distance, so a skipped row can be neither among the k1 best nor at the k-th distance.  Each chunk of
	// kScanThreads candidates is compacted in shared memory first, so the warps share only the rows they gather.  gathered != nullptr:
	// the rows gathered are added to it (diagnostics).
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t q = qsel ? qsel[blockIdx.x] : blockIdx.x;
	const bool tie = tie_bound != nullptr;
	const bool range = radius != nullptr;
	const float rad = range ? radius[q] : 0.f;
	const float bound = tie ? tie_bound[blockIdx.x] : 0.f;
	const uint32_t nch = (dim + 127u) / 128u, dp4 = nch * 32u, pitch4 = pitch >> 2;
	const uint32_t m = k1 + kCandBuf;
	float4* sq4 = reinterpret_cast<float4*>(smem_raw);  // the query, zero padded to nch * 128 floats (as tc_prepare_queries' qf)
	uint64_t* skeys = reinterpret_cast<uint64_t*>(smem_raw + size_t(dp4) * 16);  // [8 warps][m]
	{
		float* sq = reinterpret_cast<float*>(sq4);
		for (uint32_t i = threadIdx.x; i < dp4 * 4; i += blockDim.x) {
			sq[i] = i < dim ? queries[size_t(q) * dim + i] : 0.f;
		}
		for (uint32_t i = threadIdx.x; i < kScanWarps * m; i += blockDim.x) {
			skeys[i] = kKeyNone;
		}
	}
	__syncthreads();
	uint64_t* wkeys = skeys + size_t(warp) * m;
	uint64_t thr = kKeyNone;
	uint32_t cnt = 0;
	const uint32_t ncand = min(cand_count[q], cand_cap);
	const float4* rows4 = reinterpret_cast<const float4*>(rows);
	const uint32_t* my = cand_rows + size_t(q) * cand_cap;
	const float* my_lb = cand_lb ? cand_lb + size_t(q) * cand_cap : nullptr;
	const float tau_q = cand_lb ? ord_float(tau[q]) : 0.f;
	__shared__ uint32_t s_rows[kScanThreads];
	__shared__ uint32_t s_warp_n[kScanWarps];
	for (uint32_t c0 = 0; c0 < ncand; c0 += kScanThreads) {
		const uint32_t i = c0 + threadIdx.x;
		const bool keep = i < ncand && !(my_lb != nullptr && my_lb[i] > tau_q);
		const unsigned ballot = __ballot_sync(0xffffffffu, keep);
		if (lane == 0) {
			s_warp_n[warp] = __popc(ballot);
		}
		__syncthreads();
		uint32_t base = 0, nkeep = 0;
#pragma unroll
		for (int w = 0; w < kScanWarps; ++w) {
			base += w < warp ? s_warp_n[w] : 0u;
			nkeep += s_warp_n[w];
		}
		if (keep) {
			s_rows[base + __popc(ballot & ((1u << lane) - 1u))] = my[i];
		}
		if (gathered != nullptr && threadIdx.x == 0) {
			atomicAdd(gathered, (unsigned long long)nkeep);
		}
		__syncthreads();
		for (uint32_t j = warp; j < nkeep; j += kScanWarps) {
			const uint32_t row = s_rows[j];
			const float dist = row_dist_warp<kIsL2>(rows4, pitch4, nch, row, sq4, norm_coefs, lane);
			if (range) {
				if (lane == 0 && dist < rad) {
					range_keys[size_t(q) * cand_cap + atomicAdd(&range_count[q], 1u)] = make_key(dist, row);
				}
				continue;
			}
			const uint64_t key = !tie ? make_key(dist, row) : (dist <= bound ? ((uint64_t(row) << 32) | float_ord(dist)) : kKeyNone);
			if (key < thr) {  // warp-uniform
				if (lane == 0) {
					wkeys[k1 + cnt] = key;
				}
				++cnt;
				__syncwarp();
				if (cnt == kCandBuf) {
					warp_select(wkeys, k1 + cnt, k1, lane);
					thr = wkeys[k1 - 1];
					cnt = 0;
				}
			}
		}
		__syncthreads();  // s_rows and s_warp_n are refilled by the next chunk
	}
	if (range) {
		return;
	}
	if (cnt) {
		warp_select(wkeys, k1 + cnt, k1, lane);
	}
	__syncthreads();
	if (warp == 0) {  // CTA merge: strictly increasing selection over the 8 warp lists (keys are unique)
		uint64_t last = 0;
		bool first = true;
		for (uint32_t r = 0; r < k1; ++r) {
			uint64_t best = kKeyNone;
			for (uint32_t i = lane; i < kScanWarps * k1; i += 32) {
				const uint32_t w = i / k1, j = i - w * k1;
				const uint64_t kx = skeys[size_t(w) * m + j];
				if ((first || kx > last) && kx < best) {
					best = kx;
				}
			}
#pragma unroll
			for (int off = 16; off > 0; off >>= 1) {
				const uint64_t ok = __shfl_xor_sync(0xffffffffu, best, off);
				best = ok < best ? ok : best;
			}
			if (lane == 0) {
				lists[size_t(blockIdx.x) * k1 + r] = best;
			}
			last = best;
			first = false;
		}
	}
}

// ---- staged exact thresholds (k1 > kTcMaxK1) ---------------------------------------------------------------------------------------
// Any k1 rows give a valid threshold: their k1-th best exact distance is at least the k1-th best over all rows.  The seed is the exact
// top-k1 over a short prefix of the rows; stage s then runs the filter with that fixed threshold over a prefix of the shadow's SLOTS
// r times longer than the last (slots are sorted, so a prefix holds other rows than the seed: it does not matter), re-ranks the
// candidates with knn_rerank's range mode (radius = the next float above tau: it keeps exactly dist <= tau) and takes the k1-th best
// survivor as the next threshold, or keeps the threshold when fewer than k1 survive.  Every threshold kept is thus its predecessor or
// the k1-th best exact distance of some k1 distinct rows, so it stays valid.  The last stage covers every slot, so every row; its k1
// best survivors are the exact answer.
constexpr uint32_t kTcStagedMaxK1 = 1024;  // k + 1 <= 1024: the staged path's limit
constexpr int kSelThreads = 512;
constexpr uint32_t kSelSort = 4096;        // keys sorted in shared memory by knn_select_topk

// per-query stage status: 0 = the filter decides the query, 1 = it falls back to the exact scan (and admits nothing in later stages)
__global__ void knn_seed_tau(const float* seed_dist, const uint32_t* seed_count, uint32_t k1, uint32_t nq, unsigned int* tau, float* radius,
							 unsigned int* status) {
	const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
	if (q >= nq) {
		return;
	}
	// a non-finite k1-th distance of the prefix (rows of infinite or NaN distance) would admit every row: the exact scan answers
	const float t = seed_count[q] >= k1 ? seed_dist[size_t(q) * k1 + k1 - 1] : NAN;
	const bool ok = isfinite(t);
	tau[q] = float_ord(ok ? t : -INFINITY);
	radius[q] = ok ? nextafterf(t, INFINITY) : -INFINITY;
	status[q] = ok ? 0u : 1u;
}

struct SelectArgs {
	const uint64_t* keys;          // [nq][cap] unordered make_key(dist, row) of knn_rerank's range mode
	const unsigned int* nkeys;     // [nq] keys per region
	const unsigned int* cand_count;  // [nq] the filter's candidate counts (> cap: the list overflowed)
	const uint32_t* qsel;          // CTA b serves query qsel[b], or nullptr (CTA b serves query b)
	const uint64_t* labels;
	uint32_t cap;
	uint32_t k1;
	int mode;                      // kModeTopK: the k1 smallest (dist, row); kModeTieRows: the k1 first rows in internal order
	int last;                      // kModeTopK: the last stage writes the results and decides the fallbacks
	unsigned int* tau;             // kModeTopK: [nq] the next stage's threshold (ordered uint) and radius
	float* radius;
	unsigned int* status;          // kModeTopK: [nq] knn_seed_tau's status
	unsigned long long* reranked;  // kModeTopK: += the candidates re-ranked
	float* out_dist;               // [CTA][k1] (kModeTopK: written by the last stage)
	uint32_t* out_idx;
	uint64_t* out_label;           // may be null
	uint32_t* out_count;
	bool neg_zero;                 // key_dist: zero distances come out as -0 (inner product, cosine)
};

// One CTA per query: the k1 smallest of the query's unordered key region, ascending, in time linear in the region.  A radix select on
// 8-bit digits from the top narrows the keys at or below the k1-th to at most kSelSort (keys are unique, so the last digit always
// does), a bitonic sort in shared memory orders them.  Tie mode selects on row-major keys (row << 32 | ord(dist)).
__global__ void __launch_bounds__(kSelThreads) knn_select_topk(const SelectArgs a) {
	__shared__ uint64_t s_keys[kSelSort];
	__shared__ uint32_t s_hist[256];
	__shared__ uint64_t s_prefix, s_bound;
	__shared__ uint32_t s_below, s_n;
	const uint32_t b = blockIdx.x, q = a.qsel ? a.qsel[b] : b;
	const bool tie = a.mode == kModeTieRows;
	const int lane = threadIdx.x & 31;
	if (!tie) {
		if (threadIdx.x == 0) {
			atomicAdd(a.reranked, (unsigned long long)min(a.cand_count[q], a.cap));
		}
		if (a.status[q]) {  // settled as a fallback: admits nothing from now on
			if (threadIdx.x == 0) {
				a.tau[q] = float_ord(-INFINITY);
				a.radius[q] = -INFINITY;
			}
			return;
		}
	}
	const uint32_t n = min(a.nkeys[q], a.cap);
	const uint64_t* src = a.keys + size_t(q) * a.cap;
	auto load = [&](uint32_t i) {
		const uint64_t k = src[i];
		return tie ? (k << 32) | (k >> 32) : k;
	};
	// whole warps walk the region (the histogram aggregates equal digits of a warp with one shared atomic)
	const uint32_t span = (n + kSelThreads - 1) / kSelThreads * kSelThreads;
	if (threadIdx.x == 0) {
		s_bound = kKeyNone;
		s_prefix = 0;
		s_below = 0;
		s_n = 0;
	}
	__syncthreads();
	if (n > kSelSort) {
		for (int sh = 56; sh >= 0; sh -= 8) {
			const uint64_t hi = sh == 56 ? 0ull : ~0ull << (sh + 8);  // the digits already fixed
			const uint64_t prefix = s_prefix;
			for (uint32_t i = threadIdx.x; i < 256; i += kSelThreads) {
				s_hist[i] = 0;
			}
			__syncthreads();
			for (uint32_t i = threadIdx.x; i < span; i += kSelThreads) {
				const uint64_t k = i < n ? load(i) : 0ull;
				const bool in = i < n && (k & hi) == prefix;
				const uint32_t d = in ? uint32_t(k >> sh) & 0xFFu : 0x100u;
				const unsigned peers = __match_any_sync(0xffffffffu, d);
				if (in && lane == __ffs(peers) - 1) {
					atomicAdd(&s_hist[d], uint32_t(__popc(peers)));
				}
			}
			__syncthreads();
			if (threadIdx.x == 0) {  // the digit of the k1-th key: below + (keys of smaller digits) < k1 <= ... + (keys of this digit)
				const uint32_t need = a.k1 - s_below;
				uint32_t cum = 0, d = 0;
				while (cum + s_hist[d] < need) {
					cum += s_hist[d++];
				}
				s_prefix = prefix | (uint64_t(d) << sh);
				s_below += cum;
				if (s_below + s_hist[d] <= kSelSort) {
					s_bound = s_prefix | ((1ull << sh) - 1ull);
				}
			}
			__syncthreads();
			if (s_bound != kKeyNone) {
				break;
			}
		}
	}
	const uint64_t bound = s_bound;
	for (uint32_t i = threadIdx.x; i < span; i += kSelThreads) {  // gather the keys at or below the bound
		const uint64_t k = i < n ? load(i) : kKeyNone;
		const bool take = i < n && k <= bound;
		const unsigned m = __ballot_sync(0xffffffffu, take);
		uint32_t base = 0;
		if (lane == 0 && m) {
			base = atomicAdd(&s_n, uint32_t(__popc(m)));
		}
		base = __shfl_sync(0xffffffffu, base, 0);
		if (take) {
			s_keys[base + __popc(m & ((1u << lane) - 1u))] = k;
		}
	}
	__syncthreads();
	const uint32_t cnt = s_n;
	uint32_t p2 = 1;
	while (p2 < cnt) {
		p2 <<= 1;
	}
	for (uint32_t i = cnt + threadIdx.x; i < p2; i += kSelThreads) {
		s_keys[i] = kKeyNone;
	}
	__syncthreads();
	for (uint32_t size = 2; size <= p2; size <<= 1) {  // bitonic sort, ascending
		for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
			for (uint32_t t = threadIdx.x; t < p2 / 2; t += kSelThreads) {
				const uint32_t i = 2 * t - (t & (stride - 1)), j = i + stride;
				const bool up = (i & size) == 0;
				const uint64_t x = s_keys[i], y = s_keys[j];
				if ((x > y) == up) {
					s_keys[i] = y;
					s_keys[j] = x;
				}
			}
			__syncthreads();
		}
	}
	const uint32_t m = min(cnt, a.k1);
	if (!tie) {
		// fewer than k1 survivors (an overflowed list of an earlier stage): the threshold stays, it is still valid
		if (!a.last) {
			if (threadIdx.x == 0 && m == a.k1) {
				const float t = ord_float(uint32_t(s_keys[m - 1] >> 32));
				a.tau[q] = float_ord(t);
				a.radius[q] = nextafterf(t, INFINITY);
			}
			return;
		}
		if (m < a.k1 || a.cand_count[q] > a.cap) {
			if (threadIdx.x == 0) {
				a.status[q] = 1u;
			}
			return;
		}
	}
	const size_t ob = size_t(b) * a.k1;
	for (uint32_t r = threadIdx.x; r < m; r += kSelThreads) {
		const uint64_t k = s_keys[r];
		const uint32_t idx = tie ? uint32_t(k >> 32) : uint32_t(k);
		a.out_dist[ob + r] = key_dist(tie ? uint32_t(k) : uint32_t(k >> 32), a.neg_zero);
		a.out_idx[ob + r] = idx;
		if (a.out_label) {
			a.out_label[ob + r] = a.labels[idx];
		}
	}
	if (threadIdx.x == 0) {
		a.out_count[b] = m;
	}
}

// ---- helpers: int8 shadow, query codes, threshold init ------------------------------------------------------------------------------
// The quantiser of the header comment, one warp per vector p[0, dim): calls put(c, code4) for every group of four codes c .. c + 3 of
// [0, padded) (zero beyond dim) and returns (s, r, n) -- r and n rounded up from fp64 sums, so they bound ||rho|| and ||v||.
template <typename Put>
__device__ __forceinline__ float3 tc_quantize(const float* p, uint32_t dim, uint32_t padded, int lane, Put put) {
	float mx = 0.f;
	double ss = 0.0;
	for (uint32_t c = lane; c < dim; c += 32) {
		const float v = p[c];
		mx = fmaxf(mx, fabsf(v));
		ss = fma(double(v), double(v), ss);
	}
	for (int off = 16; off > 0; off >>= 1) {
		mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
		ss += __shfl_xor_sync(0xffffffffu, ss, off);
	}
	const float s = mx / 127.f;  // 0 for an all-zero vector (and for one whose largest entry is below 127 denormal steps)
	double rr = 0.0;
	for (uint32_t c = 4 * lane; c < padded; c += 128) {
		uint32_t code4 = 0;
#pragma unroll
		for (uint32_t i = 0; i < 4; ++i) {
			const float v = c + i < dim ? p[c + i] : 0.f;
			const float code = s > 0.f ? fminf(fmaxf(rintf(v / s), -127.f), 127.f) : 0.f;
			const double rho = double(v) - double(s) * double(code);  // exact: s * code has 32 significant bits
			rr = fma(rho, rho, rr);
			code4 |= (uint32_t(int(code)) & 0xFFu) << (8 * i);
		}
		put(c, code4);
	}
	for (int off = 16; off > 0; off >>= 1) {
		rr += __shfl_xor_sync(0xffffffffu, rr, off);
	}
	// the fp64 sums are within dim * 2^-53 of the true ones: a relative 2^-40 and rounding up keep r and n upper bounds
	return make_float3(s, __double2float_ru(sqrt(rr) * (1.0 + 0x1p-40)), __double2float_ru(sqrt(ss) * (1.0 + 0x1p-40)));
}

// rows fp32 [n][pitch] -> int8 shadow + per-row constants (s_v, r_v, n_v, c_v), c_v = the Cosine norm coefficient (1 otherwise),
// row v into slot row_slot[v].  Shadow layout: [64-slot block][K chunk of 128][64 slots x 128 bytes], and inside every 8 KB block the
// 16-byte units of slot r are XOR-permuted with (r % 8) -- the SWIZZLE_128B pattern wgmma expects in shared memory -- so that a plain
// contiguous cp.async.bulk brings a ready-to-multiply operand tile.
__global__ void tc_convert_rows(const float* rows, uint32_t pitch, uint32_t dim, uint32_t row_begin, uint32_t row_end, const uint32_t* row_slot,
								unsigned char* shadow, uint32_t kchunks, const float* norm_coefs, float4* rowc) {
	const uint32_t row = row_begin + (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	const int lane = threadIdx.x & 31;
	if (row >= row_end) {
		return;
	}
	const uint32_t slot = row_slot[row], blk = slot / 64u, r = slot % 64u;
	const float3 srn = tc_quantize(rows + size_t(row) * pitch, dim, kchunks * kTcChunkK, lane, [&](uint32_t c, uint32_t code4) {
		const uint32_t kc = c / kTcChunkK, cc = c % kTcChunkK;
		const uint32_t unit = (cc >> 4) ^ (r & 7u);  // 16-byte unit = 16 codes
		*reinterpret_cast<uint32_t*>(shadow + (size_t(blk) * kchunks + kc) * kTcBlockBytes + r * 128u + unit * 16u + (cc & 15u)) = code4;
	});
	if (lane == 0) {
		rowc[slot] = make_float4(srn.x, srn.y, srn.z, norm_coefs ? norm_coefs[row] : 1.f);
	}
}

// The sort key of the shadow's slot order (ensureShadow), one warp per row: S_v = s_v c_v descending (s_v as tc_quantize computes it),
// for L2 after a coarse bucket of n_v^2 (its top 10 mantissa bits), so that the rows of a 64-slot block have nearly equal u_v and w_v
// (tc_block_threshold).  The value is the row itself: a stable radix sort then breaks ties by the row.
__global__ void tc_sort_keys(const float* rows, uint32_t pitch, uint32_t dim, uint32_t n, const float* norm_coefs, int metric, uint64_t* keys,
							 uint32_t* vals) {
	const uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	const int lane = threadIdx.x & 31;
	if (row >= n) {
		return;
	}
	const float* p = rows + size_t(row) * pitch;
	float mx = 0.f, ss = 0.f;
	for (uint32_t c = lane; c < dim; c += 32) {
		const float v = p[c];
		mx = fmaxf(mx, fabsf(v));
		ss = fmaf(v, v, ss);
	}
	for (int off = 16; off > 0; off >>= 1) {
		mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
		ss += __shfl_xor_sync(0xffffffffu, ss, off);
	}
	if (lane == 0) {
		const float S = (mx / 127.f) * (norm_coefs ? norm_coefs[row] : 1.f);
		const uint64_t bucket = metric == kL2 ? float_ord(ss) >> 13 : 0u;
		keys[row] = bucket << 32 | ~float_ord(S);
		vals[row] = row;
	}
}

// slot_row[0, n) holds the rows in slot order: the inverse map
__global__ void tc_invert_slots(const uint32_t* slot_row, uint32_t n, uint32_t* row_slot) {
	const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s < n) {
		row_slot[slot_row[s]] = s;
	}
}

// Incremental shadow updates: rows [row_begin, row_end) appended to slots slot_begin, slot_begin + 1, ... (assign), or gone (kill:
// their slots become dead, all-zero constants)
__global__ void tc_assign_slots(uint32_t row_begin, uint32_t row_end, uint32_t slot_begin, uint32_t* slot_row, uint32_t* row_slot) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (row_begin + i < row_end) {
		slot_row[slot_begin + i] = row_begin + i;
		row_slot[row_begin + i] = slot_begin + i;
	}
}
__global__ void tc_kill_rows(uint32_t row_begin, uint32_t row_end, const uint32_t* row_slot, uint32_t* slot_row, float4* rowc) {
	const uint32_t row = row_begin + blockIdx.x * blockDim.x + threadIdx.x;
	if (row < row_end) {
		const uint32_t slot = row_slot[row];
		slot_row[slot] = kTcDeadSlot;
		rowc[slot] = make_float4(0.f, 0.f, 0.f, 0.f);
	}
}

// The block test's factors of every 64-slot block over its live slots (tc_block_threshold), one warp per block, two slots per lane:
// fp64 quotients with directed rounding, so u_lo, w_lo are at or below and u_hi, rho_hi, nu_hi, w_hi at or above every live row's.
// one_minus_eps = 1 - tc_l2eps(dim) for L2 (w = 0 otherwise), the same fp32 value the consumers' R uses.
__global__ void tc_block_consts(const float4* rowc, const uint32_t* slot_row, uint32_t nslots, uint32_t nblocks, float one_minus_eps,
								int metric, float4* blockc) {
	const uint32_t blk = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	const int lane = threadIdx.x & 31;
	if (blk >= nblocks) {
		return;
	}
	float u_lo = INFINITY, u_hi = 0.f, rho_hi = 0.f, nu_hi = 0.f, w_lo = INFINITY, w_hi = 0.f;
	bool live = false, pass_all = false;
	for (uint32_t i = 0; i < 2; ++i) {
		const uint32_t slot = blk * 64 + 2 * lane + i;
		if (slot >= nslots || slot_row[slot] == kTcDeadSlot) {
			continue;
		}
		live = true;
		const float4 rc = rowc[slot];  // (s, r, n, c)
		const double S = double(rc.x) * double(rc.w);  // exact: 24 x 24 significant bits
		if (!(S > 0.0) || !isfinite(S) || !isfinite(rc.y) || !isfinite(rc.z) || rc.z < kTcTinyNorm) {  // NaN included
			pass_all = true;
			continue;
		}
		const float u0 = __double2float_rd(__ddiv_rd(1.0, S)), u1 = __double2float_ru(__ddiv_ru(1.0, S));
		const float rho = __double2float_ru(__ddiv_ru(double(rc.y), double(rc.x)));
		const float nu = __double2float_ru(__ddiv_ru(double(rc.z), double(rc.x)));
		float w0 = 0.f, w1 = 0.f;
		if (metric == kL2) {  // w = (1 - eps) n^2 / (2 S)
			const double nn = double(rc.z) * double(rc.z);  // exact
			w0 = __double2float_rd(__ddiv_rd(__dmul_rd(nn, double(one_minus_eps)), 2.0 * S));
			w1 = __double2float_ru(__ddiv_ru(__dmul_ru(nn, double(one_minus_eps)), 2.0 * S));
		}
		if (!isfinite(u1) || !isfinite(rho) || !isfinite(nu) || !isfinite(w1) || u0 == 0.f) {
			pass_all = true;
			continue;
		}
		u_lo = fminf(u_lo, u0);
		u_hi = fmaxf(u_hi, u1);
		rho_hi = fmaxf(rho_hi, rho);
		nu_hi = fmaxf(nu_hi, nu);
		w_lo = fminf(w_lo, w0);
		w_hi = fmaxf(w_hi, w1);
	}
	for (int off = 16; off > 0; off >>= 1) {
		u_lo = fminf(u_lo, __shfl_xor_sync(0xffffffffu, u_lo, off));
		u_hi = fmaxf(u_hi, __shfl_xor_sync(0xffffffffu, u_hi, off));
		rho_hi = fmaxf(rho_hi, __shfl_xor_sync(0xffffffffu, rho_hi, off));
		nu_hi = fmaxf(nu_hi, __shfl_xor_sync(0xffffffffu, nu_hi, off));
		w_lo = fminf(w_lo, __shfl_xor_sync(0xffffffffu, w_lo, off));
		w_hi = fmaxf(w_hi, __shfl_xor_sync(0xffffffffu, w_hi, off));
	}
	live = __any_sync(0xffffffffu, live);
	pass_all = __any_sync(0xffffffffu, pass_all);
	if (lane == 0) {
		const float flag = pass_all ? 1.f : live ? 0.f : -1.f;
		blockc[2 * blk] = flag == 0.f ? make_float4(u_lo, u_hi, rho_hi, nu_hi) : make_float4(0.f, 0.f, 0.f, 0.f);
		blockc[2 * blk + 1] = flag == 0.f ? make_float4(w_lo, w_hi, flag, 0.f) : make_float4(0.f, 0.f, flag, 0.f);
	}
}

// The seed: ub_list[q] = the k1 best EXACT distances among the first `nrows` (<= kTcInitRows) rows, ascending, -inf beyond k1, and
// tau[q] = the k1-th of them (+inf while fewer than k1 rows exist), computed with row_dists_warp, the exact scan's own arithmetic, so
// every list entry is a row's exact-scan distance (knn_tc.cuh header).  Two kernels:
//   tc_seed_slices  CTA (t, s) computes the distances of query tile t (kTcSeedQ queries of tc_prepare_queries' zero-padded fp32 copy,
//                   staged in shared memory) to the kTcSeedSlice rows of slice s, so a row comes from L2 once per kTcSeedQ queries (a
//                   warp keeps four rows, 128-bit loads, in flight), then keeps each query's k1 smallest of the slice, ascending
//                   (k1 rounds of a warp-wide argmin; ties to the lower row), in part[q][s][0, k1) (+inf where the slice has fewer).
//   tc_seed_merge   one warp per query merges the kTcSeedSlices sorted lists (ties to the lower slice, so to the lower row).
// NaN distances are never picked (they sort as +inf).  Padding queries (q >= nq) are left untouched.
constexpr int kTcSeedQ = 16;
constexpr uint32_t kTcInitRows = 4096;  // DESIGN 3.2: 4096 against 1024 and 2048 at config 1 (fewer early hits and full queues)
constexpr uint32_t kTcSeedSlice = 512;
constexpr uint32_t kTcSeedSlices = kTcInitRows / kTcSeedSlice;
__host__ __device__ inline size_t tc_seed_smem_bytes(uint32_t kchunks) {
	return size_t(kTcSeedQ) * (size_t(kchunks) * 128 + kTcSeedSlice) * sizeof(float);
}
__global__ void __launch_bounds__(256) tc_seed_slices(const float* rows, uint32_t pitch, uint32_t kchunks, const float* norm_coefs,
													  uint32_t nrows, const float* qf, uint32_t nq, uint32_t k1, int metric,
													  float* part /* [nq][kTcSeedSlices][kTcMaxK1] */) {
	extern __shared__ __align__(16) float s_seed[];  // queries [kTcSeedQ][kchunks * 128], then distances [kTcSeedQ][kTcSeedSlice]
	const uint32_t q0 = blockIdx.x * kTcSeedQ, slice = blockIdx.y, row0 = slice * kTcSeedSlice;
	const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t qlen4 = kchunks * 32u;
	float4* sq4 = reinterpret_cast<float4*>(s_seed);
	float* s_d = s_seed + size_t(kTcSeedQ) * qlen4 * 4;
	for (uint32_t i = threadIdx.x; i < kTcSeedQ * qlen4; i += blockDim.x) {  // padding queries of the last tile copy query q0
		const uint32_t qi = i / qlen4, q = q0 + qi < nq ? q0 + qi : q0;
		sq4[i] = reinterpret_cast<const float4*>(qf)[size_t(q) * qlen4 + (i - qi * qlen4)];
	}
	__syncthreads();
	const float4* rows4 = reinterpret_cast<const float4*>(rows);
	constexpr uint32_t kRows = 4;  // rows in flight per warp
	for (uint32_t r0 = warp * kRows; r0 < kTcSeedSlice; r0 += 8 * kRows) {
		float dist[kRows][kTcSeedQ];
		if (row0 + r0 < nrows) {
			uint32_t rr[kRows];
			const float4* qp[kRows][kTcSeedQ];
#pragma unroll
			for (uint32_t x = 0; x < kRows; ++x) {
				rr[x] = min(row0 + r0 + x, nrows - 1);
#pragma unroll
				for (int qi = 0; qi < kTcSeedQ; ++qi) {
					qp[x][qi] = sq4 + qi * qlen4;
				}
			}
			if (metric == kL2) {
				row_dists_warp<true, kRows, kTcSeedQ>(rows4, pitch / 4, kchunks, rr, qp, nullptr, lane, dist);
			} else {
				row_dists_warp<false, kRows, kTcSeedQ>(rows4, pitch / 4, kchunks, rr, qp, norm_coefs, lane, dist);
			}
		}
#pragma unroll
		for (uint32_t x = 0; x < kRows; ++x) {
#pragma unroll
			for (int qi = 0; qi < kTcSeedQ; ++qi) {
				if (lane == uint32_t(qi)) {
					const uint32_t r = r0 + x;
					s_d[qi * kTcSeedSlice + r] = row0 + r < nrows ? dist[x][qi] : INFINITY;
				}
			}
		}
	}
	__syncthreads();
	for (uint32_t qi = warp; qi < kTcSeedQ; qi += 8) {  // the k1 smallest of the slice (rows < nrows sort first, the rest are +inf)
		const uint32_t q = q0 + qi;
		if (q >= nq) {
			break;
		}
		float* d = s_d + qi * kTcSeedSlice;
		float* out = part + (size_t(q) * kTcSeedSlices + slice) * kTcMaxK1;
		for (uint32_t round = 0; round < k1; ++round) {
			float best = INFINITY;
			uint32_t at = lane;
			for (uint32_t j = lane; j < kTcSeedSlice; j += 32) {
				const float y = d[j];
				if (y < best) {
					best = y;
					at = j;
				}
			}
			for (int off = 16; off > 0; off >>= 1) {
				const float ob = __shfl_xor_sync(0xffffffffu, best, off);
				const uint32_t oa = __shfl_xor_sync(0xffffffffu, at, off);
				if (ob < best || (ob == best && oa < at)) {
					best = ob;
					at = oa;
				}
			}
			if (lane == 0) {
				d[at] = INFINITY;
				out[round] = best;
			}
			__syncwarp();
		}
	}
}
__global__ void __launch_bounds__(256) tc_seed_merge(const float* part, uint32_t nq, uint32_t k1, unsigned int* tau, float* ub_list,
													 unsigned int* ub_lock) {
	static_assert(kTcSeedSlices <= 32, "one lane per slice");
	const uint32_t lane = threadIdx.x & 31, q = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	if (q >= nq) {
		return;
	}
	const float* mine = part + (size_t(q) * kTcSeedSlices + lane) * kTcMaxK1;
	uint32_t head = 0;
	float last = INFINITY;
	for (uint32_t round = 0; round < kTcMaxK1; ++round) {
		float best = INFINITY;
		if (round < k1) {
			const float h = lane < kTcSeedSlices && head < k1 ? mine[head] : INFINITY;
			best = h;
			uint32_t at = lane;
			for (int off = 16; off > 0; off >>= 1) {
				const float ob = __shfl_xor_sync(0xffffffffu, best, off);
				const uint32_t oa = __shfl_xor_sync(0xffffffffu, at, off);
				if (ob < best || (ob == best && oa < at)) {
					best = ob;
					at = oa;
				}
			}
			head += lane == at ? 1u : 0u;
			last = best;
		}
		if (lane == 0) {
			ub_list[size_t(q) * kTcMaxK1 + round] = round < k1 ? best : -INFINITY;
		}
	}
	if (lane == 0) {
		tau[q] = float_ord(last);  // +inf while fewer than k1 rows exist
		ub_lock[q] = 0;
	}
}

// queries fp32 [nq][dim] -> int8 codes [nq_pad][pitch] (zero padded) + (s_q, r_q, n_q, 1 / k_q), k_q = s_q (1 when s_q = 0), and the
// fp32 queries zero padded to the same pitch, qf [nq_pad][pitch] (the exact distances of the seed and the filter's bookkeepers)
__global__ void tc_prepare_queries(const float* queries, uint32_t nq, uint32_t nq_pad, uint32_t dim, uint32_t pitch, unsigned char* codes,
								   float4* qc, float* qf) {
	const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	const int lane = threadIdx.x & 31;
	if (q >= nq_pad) {
		return;
	}
	for (uint32_t c = lane; c < pitch; c += 32) {
		qf[size_t(q) * pitch + c] = q < nq && c < dim ? queries[size_t(q) * dim + c] : 0.f;
	}
	unsigned char* out = codes + size_t(q) * pitch;
	const float3 srn = tc_quantize(queries + size_t(q) * dim, q < nq ? dim : 0u, pitch, lane,
								   [&](uint32_t c, uint32_t code4) { *reinterpret_cast<uint32_t*>(out + c) = code4; });
	if (lane == 0 && q < nq) {
		// 1 / k_q = +inf for a tiny but non-zero query: its block thresholds all pass (header comment: fp32 underflow)
		qc[q] = make_float4(srn.x, srn.y, srn.z, srn.z > 0.f && srn.z < kTcTinyNorm ? INFINITY : srn.x > 0.f ? 1.f / srn.x : 1.f);
	}
}

// ---- the certificate's audit (rxgpu_tc_audit) ------------------------------------------------------------------------------------
// One CTA per query block of nqb queries: its (ka, kb) as the filter's consumers compute them, then thr[q][b] = the integer threshold of
// query q against shadow block b, from the query's threshold tau[q] (map space) exactly as a consumer turns it into its block test.
__global__ void tc_audit_thresholds(const float4* qc, const float* tau, uint32_t nq, uint32_t nqb, uint32_t dim, int metric,
									const float4* blockc, uint32_t nblocks, float2* kab, int* thr) {
	__shared__ float s_ab[2];
	const uint32_t q0 = blockIdx.x * nqb, nv = min(nqb, nq - q0);
	if (threadIdx.x == 0) {
		s_ab[0] = s_ab[1] = 0.f;
	}
	__syncthreads();
	const float delta = float(dim + 16) * 0x1p-23f;
	for (uint32_t i = threadIdx.x; i < nv; i += blockDim.x) {
		tc_block_ab_add(s_ab, qc[q0 + i], delta);
	}
	__syncthreads();
	const float2 k = tc_block_ab_k(s_ab);
	if (threadIdx.x == 0) {
		kab[blockIdx.x] = k;
	}
	const float l2eps = tc_l2eps(dim);
	for (uint32_t i = threadIdx.x; i < nv * nblocks; i += blockDim.x) {
		const uint32_t q = q0 + i / nblocks, b = i % nblocks;
		const float4 c = qc[q];
		const float2 pr = tc_make_pr(metric, tau[q], c, l2eps);
		thr[size_t(q) * nblocks + b] = tc_block_threshold(pr.y, pr.x, metric == kL2 ? c.w : 0.f, k.x, k.y, blockc[2 * b], blockc[2 * b + 1]);
	}
}

// bound[q][slot] = (d~, err) of tc_row_bound with x = float(I), I = the plain int32 dot product of the query's and the slot's codes
// (row codes un-swizzled to [slots][pitch], query codes [nq][pitch], both zero beyond dim)
__global__ void tc_audit_bounds(const signed char* qcodes, const float4* qc, const signed char* rcodes, const float4* rowc, uint32_t pitch,
								uint32_t nslots, uint32_t dim, int metric, float2* bound) {
	const uint32_t slot = blockIdx.x * blockDim.x + threadIdx.x, q = blockIdx.y;
	if (slot >= nslots) {
		return;
	}
	const char4* a = reinterpret_cast<const char4*>(qcodes + size_t(q) * pitch);
	const char4* b = reinterpret_cast<const char4*>(rcodes + size_t(slot) * pitch);
	int I = 0;
	for (uint32_t i = 0; i < pitch / 4; ++i) {
		const char4 x = a[i], y = b[i];
		I += int(x.x) * int(y.x) + int(x.y) * int(y.y) + int(x.z) * int(y.z) + int(x.w) * int(y.w);
	}
	TcArgs args{};
	args.dim = dim;
	args.metric = metric;
	bound[size_t(q) * nslots + slot] = tc_row_bound(args, float(I), qc[q], rowc[slot]);
}

}  // namespace rxgpu
