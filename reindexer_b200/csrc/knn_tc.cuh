// Tensor-core candidate filter for large query batches (sm_90a: TMA + wgmma + mbarrier, thread-block clusters), exact results.
//
// knn_scan_warp is HBM-bound only while <= ~16 queries share a pass; a batch of 1024 queries is FMA-bound there.  This kernel
// computes APPROXIMATE scores for a block of NQ queries against every row with bf16 operands on the tensor cores and keeps, per
// query, only the rows that can still be among the k best under a CERTIFIED error bound; the survivors (a few hundred per query)
// are then re-ranked with the exact fp32 routine of knn_scan_warp, so the final result is identical to the exact scan.
//
//   error bound   |q~.v~ - q.v| <= c * ||q|| * ||v||,  c = 2^-8 + 2^-18 (two bf16 roundings, unit roundoff 2^-9 each)
//                                                        + dim * 2^-23 (fp32 accumulation in the MMA); c = 0.0042 leaves 5% slack
//                                                        at 768 dims and 1% at 2048 dims, the largest dimension the filter accepts
//   lower bound   lb = d~ - e, upper bound ub = d~ + e in map space (smaller is better)
//   threshold     tau_q = k1-th smallest ub over all DISTINCT rows seen so far by any CTA (one small list per query in HBM,
//                 updated under a per-query lock -- only O(k log n) successful inserts per query over a whole pass) => a valid
//                 upper bound of the final k1-th best TRUE distance; a row is a candidate iff lb <= tau_q.  tau starts from an
//                 exact scan of the first rows (tc_init_tau) and only decreases.
//
// Launch shape: one grid covers G query groups (a group = one query block of NQ queries per CTA of a cluster) with W tile walkers
// each, G x W <= the clusters resident at once (config 1: 11 blocks x 12 walkers = 132 CTAs, one launch per batch).  Walker w visits
// the 128-row tiles w, w + W, w + 2W, ..., so every tile is visited once per query, and the G CTAs of one walker request the same
// tiles at about the same time: the first read misses to HBM, the others hit L2, and nothing makes one CTA wait for another.
//
// Roles (384 threads = three warpgroups, 1 CTA per SM, persistent over 128-row tiles):
//   warp 0       producer: the query block (NQ x dim bf16) once by TMA, then the bf16 shadow rows, 128 rows x 64 K (16 KB) per stage
//                through a 4-stage mbarrier ring.  The shadow is stored TILED and PRE-SWIZZLED in HBM ([tile of 64 rows][K chunk]
//                [64 x 128 B in the SWIZZLE_128B pattern]) so a stage is two contiguous 8 KB cp.async.bulk copies (row-major fp32
//                stays the source of truth; the shadow is private, derived).  In a cluster of two CTAs (optional; single CTAs are
//                faster on the H100) each CTA fetches half of every stage and multicasts it to both, which own consecutive query blocks.
//   warpgroups 1, 2   consumers: warpgroup w multiplies rows [64 w, 64 w + 64) of every tile with the whole query block
//                (wgmma.m64nNQk16, both operands from shared memory, fp32 accumulators in registers), releases each stage as soon
//                as its MMAs retired, then applies the metric to its 64 x NQ scores, tests them against tau, appends candidates to
//                per-query lists in HBM and tightens tau.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "knn_scan.cuh"

namespace rxgpu {

constexpr int kTcThreads = 384;
constexpr int kTcTileRows = 128;     // two wgmma M = 64 halves, one per consumer warpgroup
constexpr int kTcChunkK = 64;        // bf16 elements per 128-byte swizzle row
constexpr int kTcStages = 4;
constexpr int kTcBlockBytes = 64 * kTcChunkK * 2;           // 8 KB: one 64-row shadow block of one K chunk
constexpr int kTcStageBytes = 2 * kTcBlockBytes;            // 16 KB
constexpr uint32_t kTcMaxNq = 128;   // queries per CTA (wgmma N <= 128 keeps the accumulators at <= 64 registers per thread)
constexpr uint32_t kTcMaxK1 = 128;  // k + 1 <= 128: the bound list is scanned linearly under the per-query lock and ~25-35 (k + 1) candidates
                                    // per query must fit the 4096-entry lists (k = 10: 330; k = 63: 1600; an overflowing query takes the exact scan)
constexpr float kTcErrCoef = 0.0042f;  // see header comment

struct TcArgs {
	const unsigned char* shadow;  // bf16 shadow, [tile of 64 rows][K chunk][64 rows x 128 B, SWIZZLE_128B pattern pre-applied]
	const float2* vw;          // tc_make_vw: [rows padded to whole tiles] (max(||v||, tiny), w)
	const float* qnorm;        // [nq_total] ||q||_2
	unsigned int* tau;         // [nq_total] ordered-uint of the current threshold (map space), shared by all CTAs
	float* ub_list;            // [nq_total][kTcMaxK1] the k1 smallest upper bounds over ALL rows seen by any CTA (guarded by ub_lock)
	unsigned int* ub_lock;     // [nq_total]
	uint32_t init_rows;        // rows [0, init_rows) are already represented in ub_list by tc_init_tau (never insert them twice)
	uint32_t* cand_rows;       // [nq_total][cand_cap]
	unsigned int* cand_count;  // [nq_total]
	uint32_t cand_cap;
	uint32_t n;                // rows
	uint32_t kchunks;          // padded dim / 64
	uint32_t nq_total;         // queries in the whole batch
	uint32_t q0;               // first query of this launch
	uint32_t groups;           // G: query groups of this launch (a group = one query block per CTA of a cluster)
	uint32_t k1;
	int metric;                // kL2 / kIP / kCos
};

// shared memory: query block, stage ring, barriers, then per consumer warpgroup the (P, R) pairs and thresholds of the block
__host__ __device__ inline size_t tc_smem_bytes(uint32_t nq_block, uint32_t kchunks) {
	return 1024 /*align slack*/ + size_t(nq_block) * kchunks * 128 + size_t(kTcStages) * kTcStageBytes + 256 /*barriers*/ +
		   size_t(nq_block) * (4 /*qe*/ + 2 * (4 + 8) /*thr, pr per warpgroup*/) + 64;
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
// arrive on the barrier at the same shared-memory offset in CTA `cta` of the cluster (the CTA itself included)
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
	uint32_t remote;
	asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
	asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
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
// (LBO unused); the K step of 16 bf16 inside the atom advances the start address by 32 bytes
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
// D[64 rows x N queries] (+)= A[64 x 16] (smem) x B[N x 16]^T (smem), bf16 in, fp32 accumulate; d = the thread's N / 2 accumulators
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, %18, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
		"{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, "
		"%16, %17, p, 1, 1, 0, 0;\n"
		"}\n"
		: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
		  "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
		: "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, %34, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
		"{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
		"%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, "
		"%32, %33, p, 1, 1, 0, 0;\n"
		"}\n"
		: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
		  "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
		  "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
		: "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n96k16(float (&d)[48], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, %50, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 "
		"{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
		"%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
		"%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47}, "
		"%48, %49, p, 1, 1, 0, 0;\n"
		"}\n"
		: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
		  "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
		  "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
		  "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
		: "l"(adesc), "l"(bdesc), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"setp.ne.b32 p, %66, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
		"{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
		"%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,"
		"%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,"
		"%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, "
		"%64, %65, p, 1, 1, 0, 0;\n"
		"}\n"
		: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
		  "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
		  "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]),
		  "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
		  "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]),
		  "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
		: "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	if constexpr (N == 32) {
		wgmma_m64n32k16(d, adesc, bdesc, accumulate);
	} else if constexpr (N == 64) {
		wgmma_m64n64k16(d, adesc, bdesc, accumulate);
	} else if constexpr (N == 96) {
		wgmma_m64n96k16(d, adesc, bdesc, accumulate);
	} else {
		static_assert(N == 128, "query block of 32, 64, 96 or 128");
		wgmma_m64n128k16(d, adesc, bdesc, accumulate);
	}
}

// The candidate test  lb = d~ - e <= tau  rewritten as ONE fused multiply-add and one compare on the raw accumulator s = q~.v~:
//   IP      d = -s,               e = qe*vn            <=>  s >= -tau - qe*vn                       P = -qe        R = -tau      w = 0
//   Cosine  d = -s/vn,            e = qe               <=>  s >= (-tau - qe) * vn                   P = -tau - qe  R = 0         w = 0
//   L2      d = qn2 + vn2 - 2s,   e = 2qe*vn + eps*(qn2+vn2)
//                                                      <=>  s - (1-eps)/2*vn2 >= -qe*vn + ((1-eps)*qn2 - tau)/2   (w = (1-eps)/2*vn2 per row)
// The error coefficient carries 5% slack, which also covers the one-ulp differences of these rearrangements.
constexpr float kTcL2Eps = 1e-5f;
__device__ __forceinline__ float2 tc_make_pr(int metric, float tau, float qe) {
	if (metric == kIP) {
		return make_float2(-qe, -tau);
	}
	if (metric == kCos) {
		return make_float2(-tau - qe, 0.f);
	}
	const float qn = qe * (1.f / kTcErrCoef);
	return make_float2(-qe, 0.5f * ((1.f - kTcL2Eps) * qn * qn - tau));
}

// The rare path of the epilogue: row `row` passed the test for query `q` (raw accumulator s, row norm vn, qe = c * ||q||).  Appends
// the candidate, and when its upper bound beats the query's current threshold, inserts it into the query's global bound list (under
// the per-query lock; other CTAs contend) and tightens the global tau.  Returns the new threshold (+inf when it did not change).
// Kept out of line: it runs for a few hundred of 10M rows per query, and inlining it at every accumulator only costs instruction cache.
__device__ __noinline__ float tc_candidate(const TcArgs& a, uint32_t q, uint32_t row, float s, float vn, float qe, float tau) {
	float d, e;
	if (a.metric == kL2) {
		const float qn = qe * (1.f / kTcErrCoef);
		d = fmaf(-2.f, s, fmaf(qn, qn, vn * vn));
		e = 2.f * qe * vn + kTcL2Eps * (qn * qn + vn * vn);
	} else if (a.metric == kCos) {
		const float vinv = 1.f / vn;  // within 1e-5 of the stored coefficient (normalize.cc shortcut), inside the slack
		d = -s * vinv;
		e = qe * 1.0001f;
	} else {
		d = -s;
		e = qe * vn;
	}
	const unsigned pos = atomicAdd(&a.cand_count[q], 1u);
	if (pos < a.cand_cap) {
		a.cand_rows[size_t(q) * a.cand_cap + pos] = row;
	}
	const float ub = d + e;
	float tightened = INFINITY;
	if (ub < tau && row >= a.init_rows) {
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
		if (ub < mx) {
			list[mi] = ub;
			float nmx = list[0];
			for (uint32_t x = 1; x < a.k1; ++x) {
				nmx = fmaxf(nmx, list[x]);
			}
			atomicMin(&a.tau[q], float_ord(nmx));
			tightened = nmx;
		} else {
			tightened = mx;
		}
		__threadfence();
		atomicExch(&a.ub_lock[q], 0u);
	}
	return tightened;
}

// ---- the filter kernel -----------------------------------------------------------------------------------------------------------
// kNq = queries per CTA (wgmma N); kCluster = CTAs that walk the same row tiles with DIFFERENT query blocks, sharing every stage
// through TMA multicast.
template <int kNq, int kCluster>
__global__ void __launch_bounds__(kTcThreads, 1)
	knn_tc_filter(const __grid_constant__ CUtensorMap map_queries, const __grid_constant__ TcArgs a) {
	static_assert(kNq % 32 == 0 && kNq <= int(kTcMaxNq), "query block");
	static_assert(kCluster == 1 || kCluster == 2, "a stage is split in 1 or 2 equal copies");
	extern __shared__ unsigned char smem_raw[];
	unsigned char* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // offset arithmetic keeps the shared window
	constexpr uint32_t kQchunkBytes = kNq * 128;                       // one K-chunk of the query block: kNq rows x 128 B
	unsigned char* s_q = base;                                         // [kchunks][kNq][128 B], swizzled by TMA
	unsigned char* s_rows = s_q + size_t(a.kchunks) * kQchunkBytes;    // [stages][2 blocks][64][128 B]   (1024-aligned: kNq % 8 == 0)
	uint64_t* bars = reinterpret_cast<uint64_t*>(s_rows + size_t(kTcStages) * kTcStageBytes);
	uint64_t* full_bar = bars;                   // [stages] TMA -> MMA
	uint64_t* empty_bar = bars + kTcStages;      // [stages] MMA (every consumer warp of every CTA of the cluster) -> TMA
	uint64_t* q_bar = bars + 2 * kTcStages;      // queries resident
	float* s_qe = reinterpret_cast<float*>(bars + 32);                 // [kNq] c * ||q||
	float* s_thr = s_qe + kNq;                                         // [2][kNq] current tau (map space), per consumer warpgroup
	float2* s_pr = reinterpret_cast<float2*>(s_thr + 2 * kNq);         // [2][kNq] (P, R): candidate iff s - w_row >= fma(P, ||v||, R)

	const int warp = __shfl_sync(0xffffffffu, int(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;  // provably warp-uniform
	const uint32_t ntiles = (a.n + kTcTileRows - 1) / kTcTileRows;
	const uint32_t crank = kCluster > 1 ? cluster_ctarank() : 0u;
	// launch shape (header comment): cluster cid serves query group cid % G as walker cid / G of W = ncl / G
	const uint32_t cid = blockIdx.x / kCluster, ncl = gridDim.x / kCluster;
	const uint32_t walker = cid / a.groups, walkers = ncl / a.groups;
	const uint32_t q0 = a.q0 + ((cid % a.groups) * kCluster + crank) * kNq;
	const uint32_t nq_valid = q0 < a.nq_total ? min(uint32_t(kNq), a.nq_total - q0) : 0u;

	if (threadIdx.x == 0) {
		for (int s = 0; s < kTcStages; ++s) {
			mbar_init(&full_bar[s], 1);
			mbar_init(&empty_bar[s], 8 * kCluster);  // the eight consumer warps of every CTA that reads the stage's bytes
		}
		mbar_init(q_bar, 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	for (uint32_t i = threadIdx.x; i < kNq; i += blockDim.x) {
		const bool valid = i < nq_valid;
		const float thr = valid ? ord_float(a.tau[q0 + i]) : -INFINITY;
		s_qe[i] = valid ? kTcErrCoef * a.qnorm[q0 + i] : 0.f;
		const float2 pr = valid ? tc_make_pr(a.metric, thr, s_qe[i]) : make_float2(0.f, INFINITY);  // padding queries never match
		s_thr[i] = s_thr[kNq + i] = thr;
		s_pr[i] = s_pr[kNq + i] = pr;
	}
	__syncthreads();
	if constexpr (kCluster > 1) {
		cluster_sync_all();  // the peers' barriers exist before anything of ours can signal them
	}

	if (warp == 0) {
		// ===== TMA producer: the whole warp walks the loop, one elected lane issues (operands stay in uniform registers) =====
		if (elect_one_sync()) {
			mbar_expect_tx(q_bar, a.kchunks * kQchunkBytes);
			for (uint32_t kc = 0; kc < a.kchunks; ++kc) {
				tma_load_2d(s_q + size_t(kc) * kQchunkBytes, &map_queries, q_bar, int32_t(kc * kTcChunkK), int32_t(q0));
			}
		}
		__syncwarp();
		uint32_t stage = 0, phase = 0;
		for (uint32_t t = walker; t < ntiles; t += walkers) {
			for (uint32_t kc = 0; kc < a.kchunks; ++kc) {
				mbar_wait(&empty_bar[stage], phase ^ 1);
				// a 128-row stage = the 64-row shadow blocks 2t and 2t+1 of this K chunk, 8 KB each, kchunks * 8 KB apart in HBM
				const unsigned char* src = a.shadow + (size_t(2 * t) * a.kchunks + kc) * kTcBlockBytes;
				unsigned char* dst = s_rows + size_t(stage) * kTcStageBytes;
				if (elect_one_sync()) {
					mbar_expect_tx(&full_bar[stage], kTcStageBytes);
					if constexpr (kCluster == 1) {
						bulk_load(dst, src, kTcBlockBytes, &full_bar[stage]);
						bulk_load(dst + kTcBlockBytes, src + size_t(a.kchunks) * kTcBlockBytes, kTcBlockBytes, &full_bar[stage]);
					} else {  // my 1/C of the stage, delivered to every CTA of the cluster
						constexpr uint32_t kPart = kTcStageBytes / kCluster;
						const uint32_t blk = crank * kPart / kTcBlockBytes, off = crank * kPart % kTcBlockBytes;
						bulk_load_mc(dst + blk * kTcBlockBytes + off, src + size_t(blk) * a.kchunks * kTcBlockBytes + off, kPart, &full_bar[stage],
									 uint16_t((1u << kCluster) - 1u));
					}
				}
				__syncwarp();
				if (++stage == kTcStages) {
					stage = 0;
					phase ^= 1;
				}
			}
		}
	} else if (warp >= 4) {
		// ===== consumer warpgroup wg: rows [64 wg, 64 wg + 64) of every tile =====
		const uint32_t wg = uint32_t(warp) / 4 - 1, wtid = threadIdx.x - 128 * (wg + 1);
		float* thr = s_thr + wg * kNq;
		float2* pr = s_pr + wg * kNq;
		// accumulator fragment of wgmma.m64nN: d[4j + {0,1}] = (row r0, query 8j + 2c + {0,1}), d[4j + {2,3}] = the same for row r0 + 8
		const uint32_t r0 = (wtid >> 5) * 16 + (lane >> 2), c2 = 2 * (lane & 3);
		const uint32_t my_q = wtid;  // the query whose threshold this thread refreshes from the global list
		unsigned int tau_ahead = my_q < nq_valid ? a.tau[q0 + my_q] : 0u;
		auto release = [&](uint32_t st) {  // this warp is done with stage st in every CTA that reads it
			if constexpr (kCluster == 1) {
				mbar_arrive(&empty_bar[st]);
			} else {
				for (uint32_t c = 0; c < uint32_t(kCluster); ++c) {
					mbar_arrive_cluster(&empty_bar[st], c);
				}
			}
		};
		mbar_wait(q_bar, 0);
		uint32_t stage = 0, phase = 0;
		for (uint32_t t = walker; t < ntiles; t += walkers) {
			// refresh tau from the other CTAs: the global load was issued during the PREVIOUS tile, so its latency is hidden
			if (my_q < nq_valid) {
				const float tn = ord_float(tau_ahead);
				if (tn < thr[my_q]) {
					thr[my_q] = tn;
					pr[my_q] = tc_make_pr(a.metric, tn, s_qe[my_q]);
				}
				tau_ahead = a.tau[q0 + my_q];
			}
			const uint32_t row0 = t * kTcTileRows + wg * 64 + r0, row1 = row0 + 8;
			const float2 vw0 = a.vw[row0], vw1 = a.vw[row1];  // rows are padded to whole tiles; consumed after the MMAs
			float acc[kNq / 2];
#pragma unroll
			for (int i = 0; i < kNq / 2; ++i) {
				acc[i] = 0.f;
			}
			uint32_t prev = 0;
			for (uint32_t kc = 0; kc < a.kchunks; ++kc) {
				mbar_wait(&full_bar[stage], phase);
				const uint32_t a_addr = smem_u32(s_rows + size_t(stage) * kTcStageBytes + wg * kTcBlockBytes);
				const uint32_t b_addr = smem_u32(s_q + size_t(kc) * kQchunkBytes);
				wgmma_fence();
#pragma unroll
				for (uint32_t k = 0; k < kTcChunkK / 16; ++k) {  // K = 16 bf16 = 32 bytes inside the 128-byte swizzle row
					wgmma_bf16<kNq>(acc, wgmma_desc_sw128(a_addr + k * 32), wgmma_desc_sw128(b_addr + k * 32), (kc | k) != 0);
				}
				wgmma_commit();
				if (kc > 0) {  // the previous chunk's MMAs have retired: its stage goes back to the producers
					wgmma_wait<1>();
					if (lane == 0) {
						release(prev);
					}
				}
				prev = stage;
				if (++stage == kTcStages) {
					stage = 0;
					phase ^= 1;
				}
			}
			wgmma_wait<0>();
			if (lane == 0) {
				release(prev);
			}
			asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");  // the refreshed (P, R) of all queries are visible
			// a tightened threshold takes effect at once for the rest of the tile: other threads of the warpgroup may store a looser one
			// for the same query concurrently, which is still a valid upper bound (each store is a single aligned store)
			auto tighten = [&](uint32_t qq, float nt) {
				if (nt < thr[qq]) {
					thr[qq] = nt;
					pr[qq] = tc_make_pr(a.metric, nt, s_qe[qq]);
				}
			};
			// hot path: one broadcast LDS.128 per two queries, one FFMA and one compare per score
			const bool ok0 = row0 < a.n, ok1 = row1 < a.n;
#pragma unroll
			for (int j = 0; j < kNq / 8; ++j) {
				const uint32_t q = 8 * j + c2;
				const float4 p2 = *reinterpret_cast<const float4*>(&pr[q]);  // (P, R) of queries q and q + 1
				const bool h0 = ok0 && acc[4 * j] - vw0.y >= fmaf(p2.x, vw0.x, p2.y);
				const bool h1 = ok0 && acc[4 * j + 1] - vw0.y >= fmaf(p2.z, vw0.x, p2.w);
				const bool h2 = ok1 && acc[4 * j + 2] - vw1.y >= fmaf(p2.x, vw1.x, p2.y);
				const bool h3 = ok1 && acc[4 * j + 3] - vw1.y >= fmaf(p2.z, vw1.x, p2.w);
				if (h0 | h1 | h2 | h3) {  // rare path: exact bounds, candidate append, threshold tightening
					if (h0) tighten(q, tc_candidate(a, q0 + q, row0, acc[4 * j], vw0.x, s_qe[q], thr[q]));
					if (h1) tighten(q + 1, tc_candidate(a, q0 + q + 1, row0, acc[4 * j + 1], vw0.x, s_qe[q + 1], thr[q + 1]));
					if (h2) tighten(q, tc_candidate(a, q0 + q, row1, acc[4 * j + 2], vw1.x, s_qe[q], thr[q]));
					if (h3) tighten(q + 1, tc_candidate(a, q0 + q + 1, row1, acc[4 * j + 3], vw1.x, s_qe[q + 1], thr[q + 1]));
				}
			}
			__syncwarp();  // the rare path diverges (per-lane lock loops): reconverge before the .aligned wgmma of the next tile
			asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");  // nobody still reads (P, R) when the next refresh writes them
		}
	}
	__syncthreads();
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
															const uint32_t* qsel = nullptr, const float* tie_bound = nullptr) {
	// qsel: CTA b serves query qsel[b] (default: query b).  tie_bound != nullptr = tie mode (kModeTieRows): among the candidates
	// with dist <= tie_bound[b], the first k1 in internal row order (key = row << 32 | ord(dist)) -- every row at or below the k-th
	// distance is a candidate, so this replaces a second scan of the whole shard when the reference's tie rule must be replayed.
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t q = qsel ? qsel[blockIdx.x] : blockIdx.x;
	const bool tie = tie_bound != nullptr;
	const float bound = tie ? tie_bound[blockIdx.x] : 0.f;
	const uint32_t nch = (dim + 127u) / 128u, dp4 = nch * 32u, pitch4 = pitch >> 2;
	const uint32_t m = k1 + kCandBuf;
	float4* sq4 = reinterpret_cast<float4*>(smem_raw);
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
	for (uint32_t i = warp; i < ncand; i += kScanWarps) {
		const uint32_t row = my[i];
		float s = 0.f;
		for (uint32_t c = 0; c < nch; ++c) {
			const uint32_t f4 = c * 32u + lane;
			const float4 db = f4 < pitch4 ? ldg_stream(rows4 + size_t(row) * pitch4 + f4) : make_float4(0.f, 0.f, 0.f, 0.f);
			const float4 qv = sq4[f4];
			if constexpr (kIsL2) {
				float d;
				d = qv.x - db.x;
				s = fmaf(d, d, s);
				d = qv.y - db.y;
				s = fmaf(d, d, s);
				d = qv.z - db.z;
				s = fmaf(d, d, s);
				d = qv.w - db.w;
				s = fmaf(d, d, s);
			} else {
				s = fmaf(qv.x, db.x, s);
				s = fmaf(qv.y, db.y, s);
				s = fmaf(qv.z, db.z, s);
				s = fmaf(qv.w, db.w, s);
			}
		}
#pragma unroll
		for (int off = 16; off > 0; off >>= 1) {
			s += __shfl_xor_sync(0xffffffffu, s, off);
		}
		float dist = kIsL2 ? s : -s;
		if (!kIsL2 && norm_coefs != nullptr) {
			dist *= norm_coefs[row];
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

// per-row constants of the filter epilogue, one float2 per row: (max(||v||, tiny), w) with w = the row's share of the L2 expansion
// (0 for IP / Cosine); rows beyond n are zero.  A 64-row tile's pairs are one contiguous 512-byte block (one cp.async.bulk).
__global__ void tc_make_vw(const float* vnorm, uint32_t n, uint32_t padded, int metric, float2* vw) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < padded) {
		const float vn = i < n ? vnorm[i] : 0.f;
		vw[i] = make_float2(fmaxf(vn, 1e-30f), metric == kL2 ? 0.5f * (1.f - kTcL2Eps) * vn * vn : 0.f);
	}
}

// ---- helpers: bf16 shadow, norms, query preparation, threshold init ---------------------------------------------------------------
// rows fp32 [n][pitch] -> bf16 shadow + ||row||_2.  Shadow layout: [tile of 64 rows][K chunk of 64][64 rows x 128 bytes], and inside
// every 8 KB block the 16-byte units of row r are XOR-permuted with (r % 8) -- the SWIZZLE_128B pattern wgmma expects in
// shared memory -- so that a plain contiguous cp.async.bulk brings a ready-to-multiply operand tile.
__global__ void tc_convert_rows(const float* rows, uint32_t pitch, uint32_t dim, uint32_t row_begin, uint32_t row_end, __nv_bfloat16* shadow,
								uint32_t kchunks, float* vnorm) {
	const uint32_t row = row_begin + (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	const int lane = threadIdx.x & 31;
	if (row >= row_end) {
		return;
	}
	const float* p = rows + size_t(row) * pitch;
	const uint32_t tile = row / 64u, r = row % 64u;
	float s = 0.f;
	for (uint32_t c = lane; c < kchunks * kTcChunkK; c += 32) {
		const float v = c < dim ? p[c] : 0.f;
		s = fmaf(v, v, s);
		const uint32_t kc = c / kTcChunkK, cc = c % kTcChunkK;
		const uint32_t unit = (cc >> 3) ^ (r & 7u);  // 16-byte unit = 8 bf16
		shadow[(size_t(tile) * kchunks + kc) * 4096u + r * 64u + unit * 8u + (cc & 7u)] = __float2bfloat16_rn(v);
	}
	for (int off = 16; off > 0; off >>= 1) {
		s += __shfl_xor_sync(0xffffffffu, s, off);
	}
	if (lane == 0 && vnorm) {
		vnorm[row] = sqrtf(s);
	}
}

// tau_init[q] = upper bound of the k1-th best distance among the first `nrows` (<= 1024) rows, fp32 dot products.  Any upper bound is
// valid; a small relative slack covers the difference to the arithmetic order of knn_scan_warp.  One block serves kTcInitQ queries
// (staged in shared memory, zero padded to the row pitch) so the rows come from L2 once per kTcInitQ queries; a warp keeps four rows
// (128-bit loads) in flight; the k1 smallest distances of a query are then picked by one warp (k1 rounds of a warp-wide argmin).
constexpr int kTcInitQ = 4;
constexpr uint32_t kTcInitRows = 1024;
__host__ __device__ inline size_t tc_init_smem_bytes(uint32_t pitch) { return size_t(kTcInitQ) * (pitch + kTcInitRows) * sizeof(float); }
__global__ void __launch_bounds__(256) tc_init_tau(const float* rows, uint32_t pitch, uint32_t dim, const float* norm_coefs, uint32_t nrows,
												   const float* queries, uint32_t nq, uint32_t k1, int metric, unsigned int* tau, float* ub_list,
												   unsigned int* ub_lock) {
	extern __shared__ __align__(16) float s_init[];
	float* s_q = s_init;                     // [kTcInitQ][pitch]
	float* s_d = s_init + kTcInitQ * pitch;  // [kTcInitQ][kTcInitRows]
	const uint32_t q0 = blockIdx.x * kTcInitQ;
	const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (uint32_t i = threadIdx.x; i < kTcInitQ * pitch; i += blockDim.x) {
		const uint32_t qi = i / pitch, c = i % pitch;
		s_q[i] = (q0 + qi < nq && c < dim) ? queries[size_t(q0 + qi) * dim + c] : 0.f;
	}
	__syncthreads();
	const uint32_t pitch4 = pitch / 4;
	constexpr uint32_t kRows = 4;  // rows in flight per warp
	for (uint32_t r0 = warp * kRows; r0 < kTcInitRows; r0 += 8 * kRows) {
		float acc[kRows][kTcInitQ];
#pragma unroll
		for (uint32_t x = 0; x < kRows; ++x) {
#pragma unroll
			for (int qi = 0; qi < kTcInitQ; ++qi) {
				acc[x][qi] = 0.f;
			}
		}
		if (r0 < nrows) {
			const float4* p4[kRows];
#pragma unroll
			for (uint32_t x = 0; x < kRows; ++x) {
				p4[x] = reinterpret_cast<const float4*>(rows + size_t(min(r0 + x, nrows - 1)) * pitch);
			}
#pragma unroll 3
			for (uint32_t c = lane; c < pitch4; c += 32) {
				float4 v[kRows];
#pragma unroll
				for (uint32_t x = 0; x < kRows; ++x) {
					v[x] = __ldg(p4[x] + c);
				}
#pragma unroll
				for (int qi = 0; qi < kTcInitQ; ++qi) {
					const float4 qq = reinterpret_cast<const float4*>(s_q + qi * pitch)[c];
#pragma unroll
					for (uint32_t x = 0; x < kRows; ++x) {
						if (metric == kL2) {
							const float a0 = qq.x - v[x].x, a1 = qq.y - v[x].y, a2 = qq.z - v[x].z, a3 = qq.w - v[x].w;
							acc[x][qi] = fmaf(a0, a0, fmaf(a1, a1, fmaf(a2, a2, fmaf(a3, a3, acc[x][qi]))));
						} else {
							acc[x][qi] = fmaf(qq.x, v[x].x, fmaf(qq.y, v[x].y, fmaf(qq.z, v[x].z, fmaf(qq.w, v[x].w, acc[x][qi]))));
						}
					}
				}
			}
		}
#pragma unroll
		for (uint32_t x = 0; x < kRows; ++x) {
#pragma unroll
			for (int qi = 0; qi < kTcInitQ; ++qi) {
				float s = acc[x][qi];
				for (int off = 16; off > 0; off >>= 1) {
					s += __shfl_xor_sync(0xffffffffu, s, off);
				}
				if (lane == uint32_t(qi)) {
					const uint32_t r = r0 + x;
					float d = INFINITY;
					if (r < nrows) {
						d = metric == kL2 ? s : -s;
						if (metric == kCos) {
							d *= norm_coefs[r];
						}
						d += 1e-4f * fabsf(d) + 1e-6f;
					}
					s_d[qi * kTcInitRows + r] = d;
				}
			}
		}
	}
	__syncthreads();
	if (warp < kTcInitQ && q0 + warp < nq) {  // warp w: the k1 smallest of query q0 + w (rows < nrows sort first, the rest are +inf)
		const uint32_t q = q0 + warp;
		float* d = s_d + warp * kTcInitRows;
		float last = INFINITY;
		for (uint32_t round = 0; round < kTcMaxK1; ++round) {
			float best = INFINITY;
			uint32_t at = lane;
			if (round < k1) {
				for (uint32_t j = lane; j < kTcInitRows; j += 32) {
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
				}
				__syncwarp();
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
}

// queries fp32 [nq][dim] -> bf16 [nq_pad][pitch_bf] (zero padded) + ||q||
__global__ void tc_prepare_queries(const float* queries, uint32_t nq, uint32_t nq_pad, uint32_t dim, uint32_t pitch_bf, __nv_bfloat16* out,
								   float* qnorm) {
	const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	const int lane = threadIdx.x & 31;
	if (q >= nq_pad) {
		return;
	}
	float s = 0.f;
	for (uint32_t c = lane; c < pitch_bf; c += 32) {
		const float v = (q < nq && c < dim) ? queries[size_t(q) * dim + c] : 0.f;
		s = fmaf(v, v, s);
		out[size_t(q) * pitch_bf + c] = __float2bfloat16_rn(v);
	}
	for (int off = 16; off > 0; off >>= 1) {
		s += __shfl_xor_sync(0xffffffffu, s, off);
	}
	if (lane == 0 && q < nq) {
		qnorm[q] = sqrtf(s);
	}
}

}  // namespace rxgpu
