// SQ8 scalar quantisation of the float_vector rows (SURVEY.md 8f-2): the reference quantises an HNSW map to uint8 codes with one
// additive corrective offset per vector (cpp_src/core/index/float_vector/scalar_quantization/quantizer.h:93-125) and compares codes with
// integer kernels (tools/distances/l2_dist.cc:169, ip_dist.cc:163): dist = alpha_2 * int_dist(code_a, code_b) + offset_a + offset_b
// (hnswlib/hnswlib.h:192-197; IP / Cosine negated, Cosine scaled by the row's norm coefficient and the query's).
// Here: the codes + offsets live in HBM next to the fp32 rows (4x fewer bytes per distance), either imported from the reference's
// HierarchicalNSWImpl<uint8_t> or produced on the device with the reference's arithmetic; a dp4a scan with the fused top-k of the
// fp32 scan gives the exact answer under the quantised metric (the ground truth of the quantised HNSW search, hnsw.cu).
// The integer part is exact; the float epilogue repeats the reference's operation order, so distances are bit-identical.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include "../../include/rxgpu.h"
#include "../host/knn_select.h"
#include "internal.h"
#include "common.cuh"
#include "sq8.cuh"

using namespace rxgpu;

namespace rxgpu {
void sq8Release(rxgpu_sq8_device* p) { delete p; }
}  // namespace rxgpu

namespace {

constexpr int kSqThreads = 256;
constexpr int kSqWarps = kSqThreads / 32;
constexpr uint32_t kSqMaxK1 = 256;
constexpr int kSqBuf = 32;

// Quantizer::quantize (quantizer.h:93-125), one thread per row: the corrective offset is a SEQUENTIAL float sum over the elements, so
// the element order (and every rounding) is the reference's.  No FMA contraction: the reference is built for SSE4.2 (no FMA unit).
__global__ void sq8_quantize_rows(const float* rows, uint32_t pitch, uint32_t dim, uint32_t n, float minQ, float alpha, float delta, int is_l2,
								  uint8_t* codes, uint32_t code_pitch, float* corr) {
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n) {
		return;
	}
	const float* p = rows + size_t(r) * pitch;
	uint8_t* c = codes + size_t(r) * code_pitch;
	float res = 0.f, shift = 0.f;
	for (uint32_t i = 0; i < dim; ++i) {
		const float val = p[i];
		const float qf = fminf(fmaxf(__fdiv_rn(__fsub_rn(val, minQ), alpha), 0.f), 255.f);  // float2uint8t: std::clamp(.., 0.f, kSq8Range)
		const uint8_t u = uint8_t(qf);                                                          // float -> uint8_t truncates
		const float uf = float(u);
		const float err = __fsub_rn(val, __fadd_rn(__fmul_rn(alpha, uf), minQ));  // val - uint8t2float(uint8)
		if (is_l2) {
			res = __fadd_rn(res, __fmul_rn(__fadd_rn(__fmul_rn(__fmul_rn(2.f, alpha), uf), err), err));  // (2 * alpha * uint8 + err) * err
			shift = __fsub_rn(shift, __fmul_rn(__fmul_rn(__fmul_rn(2.f, alpha), err), uf));           // -= 2.f * alpha * err * uint8
		} else {
			res = __fadd_rn(res, __fadd_rn(__fmul_rn(alpha, uf), err));    // += alpha * uint8 + err
			shift = __fadd_rn(shift, __fmul_rn(__fmul_rn(alpha, err), uf));  // += alpha * err * uint8
		}
		c[i] = u;
	}
	for (uint32_t i = dim; i < code_pitch; ++i) {
		c[i] = 0;
	}
	if (!is_l2) {
		res = __fmul_rn(res, minQ);
		res = __fadd_rn(res, delta);
	}
	corr[r] = __fadd_rn(res, shift);
}

struct SqScanArgs {
	const uint8_t* codes;
	const float* corr;
	const float* norm_coefs;  // Cosine: 1/||row||, else null
	const uint8_t* qcodes;    // [nq][code_pitch]
	const float* qcorr;       // [nq]
	const float* qcoef;       // [nq] query norm coefficient (1 unless Cosine)
	uint64_t* lists;          // out: [grid][QT][k1]
	uint32_t code_pitch, n, nq, k1;
	float alpha2;
	int is_l2;
};

// A warp handles 2 rows per step (16 lanes each, uint4 = 16 codes per load); QT queries share the pass.  Integer sums are exact, so
// the reduction order is free; lane (r * QT + qi) ends up owning the distance of (row r, query qi) and feeds the same per-warp
// sorted-list + candidate-buffer top-k as knn_scan_warp (key = ord(dist) << 32 | row).
template <int QT>
__global__ void __launch_bounds__(kSqThreads, 2) sq8_scan_kernel(const SqScanArgs a) {
	extern __shared__ __align__(16) unsigned char smem_raw[];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint32_t nch = a.code_pitch / 16;
	const uint32_t m = a.k1 + kSqBuf;
	uint4* sq = reinterpret_cast<uint4*>(smem_raw);  // [QT][nch]
	uint64_t* skeys = reinterpret_cast<uint64_t*>(smem_raw + size_t(QT) * a.code_pitch);
	uint64_t* sthr = skeys + size_t(kSqWarps) * QT * m;
	uint32_t* scnt = reinterpret_cast<uint32_t*>(sthr + kSqWarps * QT);
	for (uint32_t i = threadIdx.x; i < QT * nch; i += blockDim.x) {
		const uint32_t qi = i / nch;
		sq[i] = qi < a.nq ? reinterpret_cast<const uint4*>(a.qcodes + size_t(qi) * a.code_pitch)[i - qi * nch] : make_uint4(0, 0, 0, 0);
	}
	for (uint32_t i = threadIdx.x; i < kSqWarps * QT * m; i += blockDim.x) {
		skeys[i] = kKeyNone;
	}
	if (threadIdx.x < kSqWarps * QT) {
		sthr[threadIdx.x] = kKeyNone;
		scnt[threadIdx.x] = 0;
	}
	__syncthreads();
	uint64_t* wkeys = skeys + size_t(warp) * QT * m;
	uint64_t* wthr = sthr + warp * QT;
	uint32_t* wcnt = scnt + warp * QT;
	const int half = lane >> 4, hl = lane & 15;
	const int my_r = lane / QT, my_q = lane % QT;  // result owner: lanes [0, 2 * QT)
	const float my_qcorr = uint32_t(my_q) < a.nq ? a.qcorr[my_q] : 0.f;
	const float my_qcoef = uint32_t(my_q) < a.nq ? a.qcoef[my_q] : 1.f;
	const uint32_t ngroups = (a.n + 1) / 2;
	for (uint32_t g = blockIdx.x * kSqWarps + warp; g < ngroups; g += gridDim.x * kSqWarps) {
		const uint32_t row = g * 2 + half;
		unsigned acc[QT];
#pragma unroll
		for (int qi = 0; qi < QT; ++qi) {
			acc[qi] = 0;
		}
		if (row < a.n) {
			const uint4* rp = reinterpret_cast<const uint4*>(a.codes + size_t(row) * a.code_pitch);
			for (uint32_t c = hl; c < nch; c += 16) {
				uint4 v;
				asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(rp + c));
#pragma unroll
				for (int qi = 0; qi < QT; ++qi) {
					const uint4 q = sq[qi * nch + c];
					if (a.is_l2) {  // sum (a - b)^2: |a - b| per byte, then a 4-way dot product with itself
						unsigned d;
						d = __vabsdiffu4(v.x, q.x);
						acc[qi] = __dp4a(d, d, acc[qi]);
						d = __vabsdiffu4(v.y, q.y);
						acc[qi] = __dp4a(d, d, acc[qi]);
						d = __vabsdiffu4(v.z, q.z);
						acc[qi] = __dp4a(d, d, acc[qi]);
						d = __vabsdiffu4(v.w, q.w);
						acc[qi] = __dp4a(d, d, acc[qi]);
					} else {
						acc[qi] = __dp4a(v.x, q.x, acc[qi]);
						acc[qi] = __dp4a(v.y, q.y, acc[qi]);
						acc[qi] = __dp4a(v.z, q.z, acc[qi]);
						acc[qi] = __dp4a(v.w, q.w, acc[qi]);
					}
				}
			}
		}
		unsigned mine = 0;
#pragma unroll
		for (int qi = 0; qi < QT; ++qi) {
			unsigned v = acc[qi];
#pragma unroll
			for (int off = 8; off > 0; off >>= 1) {
				v += __shfl_xor_sync(0xffffffffu, v, off);
			}
			// lanes 0..15 hold row 0's sum, lanes 16..31 row 1's: hand them to the owner lanes r * QT + qi
			const unsigned r0 = __shfl_sync(0xffffffffu, v, 0), r1 = __shfl_sync(0xffffffffu, v, 16);
			if (lane == qi) {
				mine = r0;
			}
			if (lane == QT + qi) {
				mine = r1;
			}
		}
		const uint32_t orow = g * 2 + my_r;
		const bool valid = lane < 2 * QT && orow < a.n && uint32_t(my_q) < a.nq;
		float dist = 0.f;
		if (valid) {  // DistCalculator<uint8_t>::l2 / ::ip (hnswlib.h:192-197), then the Cosine coefficients (:147-165, hnswalg.h:801)
			dist = __fadd_rn(__fadd_rn(__fmul_rn(a.alpha2, __uint2float_rn(mine)), my_qcorr), a.corr[orow]);
			if (!a.is_l2) {
				dist = -dist;
			}
			if (a.norm_coefs) {
				dist = __fmul_rn(dist, a.norm_coefs[orow]);
			}
			dist = __fmul_rn(my_qcoef, dist);
		}
		const uint64_t key = make_key(dist, orow);
		const bool cand = valid && key < wthr[my_q];
		const unsigned cm = __ballot_sync(0xffffffffu, cand);
		if (cm) {
			const unsigned qpattern = 1u | (1u << QT);
			const unsigned mineq = cm & (qpattern << my_q);
			if (cand) {
				const uint32_t pos = wcnt[my_q] + __popc(mineq & ((1u << lane) - 1u));
				wkeys[my_q * m + a.k1 + pos] = key;
			}
			__syncwarp();
			if (lane < QT) {
				wcnt[lane] += __popc(cm & (qpattern << lane));
			}
			__syncwarp();
#pragma unroll
			for (int qi = 0; qi < QT; ++qi) {
				const uint32_t c = wcnt[qi];
				if (c > uint32_t(kSqBuf - 2)) {
					warp_select_keys(wkeys + qi * m, a.k1 + c, a.k1, lane);
					if (lane == 0) {
						wthr[qi] = wkeys[qi * m + a.k1 - 1];
						wcnt[qi] = 0;
					}
					__syncwarp();
				}
			}
		}
	}
#pragma unroll
	for (int qi = 0; qi < QT; ++qi) {
		const uint32_t c = wcnt[qi];
		if (c) {
			warp_select_keys(wkeys + qi * m, a.k1 + c, a.k1, lane);
		}
	}
	__syncthreads();
	for (int qi = warp; qi < QT; qi += kSqWarps) {  // CTA merge of the 8 warp lists of query qi: strictly increasing selection
		if (uint32_t(qi) >= a.nq) {
			continue;
		}
		uint64_t* out = a.lists + (size_t(blockIdx.x) * QT + qi) * a.k1;
		uint64_t last = 0;
		bool first = true;
		for (uint32_t r = 0; r < a.k1; ++r) {
			uint64_t best = kKeyNone;
			for (uint32_t i = lane; i < kSqWarps * a.k1; i += 32) {
				const uint32_t w = i / a.k1, j = i - w * a.k1;
				const uint64_t kx = skeys[(size_t(w) * QT + qi) * m + j];
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
				out[r] = best;
			}
			last = best;
			first = false;
		}
	}
}

// final merge of the per-CTA lists of one query: one warp, repeated minimum (grid <= 2 x SMs lists of k1 keys)
__global__ void sq8_merge_kernel(const uint64_t* lists, uint32_t nlists, uint32_t qt, uint32_t k1, uint32_t q_offset, const uint64_t* labels,
								 float* out_dist, uint64_t* out_label, uint32_t* out_idx, uint32_t* out_count) {
	const uint32_t qi = blockIdx.x;
	const int lane = threadIdx.x;
	uint64_t last = 0;
	bool first = true;
	uint32_t count = 0;
	for (uint32_t r = 0; r < k1; ++r) {
		uint64_t best = kKeyNone;
		for (uint32_t i = lane; i < nlists * k1; i += 32) {
			const uint32_t l = i / k1, j = i - l * k1;
			const uint64_t kx = lists[(size_t(l) * qt + qi) * k1 + j];
			if ((first || kx > last) && kx < best) {
				best = kx;
			}
		}
#pragma unroll
		for (int off = 16; off > 0; off >>= 1) {
			const uint64_t ok = __shfl_xor_sync(0xffffffffu, best, off);
			best = ok < best ? ok : best;
		}
		if (best == kKeyNone) {
			break;
		}
		if (lane == 0) {
			const uint32_t row = uint32_t(best);
			out_dist[size_t(q_offset + qi) * k1 + r] = ord_float(uint32_t(best >> 32));
			out_idx[size_t(q_offset + qi) * k1 + r] = row;
			out_label[size_t(q_offset + qi) * k1 + r] = labels[row];
		}
		last = best;
		first = false;
		++count;
	}
	if (lane == 0) {
		out_count[q_offset + qi] = count;
	}
}

size_t sqScanSmem(int qt, uint32_t code_pitch, uint32_t k1) {
	return size_t(qt) * code_pitch + size_t(kSqWarps) * qt * (k1 + kSqBuf) * 8 + size_t(kSqWarps) * qt * 8 + size_t(kSqWarps) * qt * 4 + 16;
}

}  // namespace

namespace rxgpu {
// Quantizer::quantize on one vector (the query: prepareData, hnswalg.h:510-535 multiplies it by `scale` = ||q|| for Cosine first)
float sq8QuantizeHost(const rxgpu_sq8_device* s, int metric, uint32_t dim, const float* v, float scale, uint8_t* codes) {
	const float minQ = s->params.min_q, alpha = s->params.alpha;
	float res = 0.f, shift = 0.f;
	const bool isL2 = metric == RXGPU_L2;
	for (uint32_t i = 0; i < dim; ++i) {
		const volatile float val = scale * v[i];  // volatile: every operation below rounds to float exactly like the reference's build
		const float qf = std::min(std::max((val - minQ) / alpha, 0.f), 255.f);
		const uint8_t u = uint8_t(qf);
		const volatile float back = alpha * float(u);
		const volatile float err = val - (back + minQ);
		if (isL2) {
			const volatile float t0 = (2 * alpha) * float(u);
			const volatile float t1 = (t0 + err) * err;
			res = res + t1;
			const volatile float t2 = (2.f * alpha) * err;
			const volatile float t3 = t2 * float(u);
			shift = shift - t3;
		} else {
			const volatile float t1 = back + err;
			res = res + t1;
			const volatile float t2 = alpha * err;
			const volatile float t3 = t2 * float(u);
			shift = shift + t3;
		}
		codes[i] = u;
	}
	if (!isL2) {
		res = res * minQ;
		res = res + s->params.delta;
	}
	return res + shift;
}
}  // namespace rxgpu

extern "C" {

int rxgpu_sq8_attach(rxgpu_index* ix, const rxgpu_sq8_params* p, const uint8_t* codes, const float* offsets) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (!p || (codes && !offsets) || !(p->alpha > 0.f)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: bad SQ8 parameters");
	}
	auto s = std::make_unique<rxgpu_sq8_device>();
	s->params = *p;
	s->code_pitch = (ix->dim + 15u) & ~15u;
	s->n = ix->size;
	const size_t n = std::max<size_t>(ix->size, 1);
	RX_CUDA(s->codes.ensure(n * s->code_pitch));
	RX_CUDA(s->corr.ensure(n));
	if (codes) {  // the reference's own codes and offsets (HierarchicalNSWImpl<uint8_t>, by internal id = row)
		// on the index's stream, which the scans use: a legacy-stream copy would not be ordered before them
		RX_CUDA(cudaMemsetAsync(s->codes.p, 0, n * s->code_pitch, ix->stream));
		RX_CUDA(cudaMemcpy2DAsync(s->codes.p, s->code_pitch, codes, ix->dim, ix->dim, ix->size, cudaMemcpyHostToDevice, ix->stream));
		RX_CUDA(cudaMemcpyAsync(s->corr.p, offsets, size_t(ix->size) * 4, cudaMemcpyHostToDevice, ix->stream));
		RX_CUDA(cudaStreamSynchronize(ix->stream));
	} else if (ix->size) {
		sq8_quantize_rows<<<unsigned((ix->size + 127) / 128), 128, 0, ix->stream>>>(ix->d_rows, ix->pitch, ix->dim, uint32_t(ix->size), p->min_q, p->alpha,
																					 p->delta, ix->metric == RXGPU_L2, s->codes.p, s->code_pitch, s->corr.p);
		RX_CUDA(cudaGetLastError());
		RX_CUDA(cudaStreamSynchronize(ix->stream));
	}
	s->index_version = ix->version;
	if (ix->sq8) {
		sq8Release(ix->sq8);
	}
	ix->sq8 = s.release();
	return 0;
}

int rxgpu_sq8_export(const rxgpu_index* ix, uint8_t* codes, float* offsets) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	const rxgpu_sq8_device* s = ix->sq8;
	if (!s || !codes || !offsets) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no SQ8 codes attached to this index");
	}
	RX_CUDA(cudaMemcpy2D(codes, ix->dim, s->codes.p, s->code_pitch, ix->dim, s->n, cudaMemcpyDeviceToHost));
	RX_CUDA(cudaMemcpy(offsets, s->corr.p, size_t(s->n) * 4, cudaMemcpyDeviceToHost));
	return 0;
}

int rxgpu_sq8_prepare_query(const rxgpu_index* ix, const float* query, float query_norm, uint8_t* codes, float* offset) {
	if (!ix || !query || !codes || !offset) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (!ix->sq8) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no SQ8 codes attached to this index");
	}
	// queryNormCoef = 1 / ||q|| for Cosine (hnswalg.h:1854-1863); prepareData restores the length: val = (1 / normCoef) * q^[i]
	const float scale = ix->metric == RXGPU_COS ? 1.f / (1.f / query_norm) : 1.f;
	*offset = sq8QuantizeHost(ix->sq8, ix->metric, ix->dim, query, scale, codes);
	return 0;
}

int rxgpu_sq8_search_knn(const rxgpu_index* ix, uint32_t nq, const float* queries, const float* query_norms, uint32_t k, float* out_dist,
						 uint64_t* out_label, uint32_t* out_count) {
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	g_stats = rxgpu_search_stats{};
	if (nq == 0) {
		return 0;
	}
	if (!queries || !out_count || (k && (!out_dist || !out_label))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	rxgpu_sq8_device* s = ix->sq8;
	if (!s) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: no SQ8 codes attached to this index");
	}
	if (s->index_version != ix->version) {
		return fail(RXGPU_ERR_LOGIC, "rxgpu: the index changed after the SQ8 codes were attached");
	}
	if (ix->metric == RXGPU_COS && !query_norms) {
		return fail(RXGPU_ERR_PARAMS, "Norm is required for Cosine-metric during corrective offsets calculation in quantized graph");  // hnswalg.h:1857
	}
	const uint32_t kEff = uint32_t(std::min<uint64_t>(k, ix->size));
	if (kEff == 0) {
		std::memset(out_count, 0, size_t(nq) * 4);
		return 0;
	}
	if (kEff > kSqMaxK1) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: SQ8 brute-force search needs k <= 256");
	}
	try {
		std::lock_guard<std::mutex> lck(s->mtx);
		cudaStream_t st = ix->stream;
		const uint32_t cp = s->code_pitch;
		std::vector<uint8_t> hq(size_t(nq) * cp, 0);
		std::vector<float> hcorr(nq), hcoef(nq, 1.f);
		for (uint32_t q = 0; q < nq; ++q) {
			const float norm = query_norms ? query_norms[q] : 1.f;
			const float coef = ix->metric == RXGPU_COS ? 1.f / norm : 1.f;
			hcoef[q] = coef;
			hcorr[q] = sq8QuantizeHost(s, ix->metric, ix->dim, queries + size_t(q) * ix->dim, ix->metric == RXGPU_COS ? 1.f / coef : 1.f,
									   hq.data() + size_t(q) * cp);
		}
		RX_CUDA(s->d_q.ensure(hq.size()));
		RX_CUDA(s->d_qcorr.ensure(nq));
		RX_CUDA(s->d_qcoef.ensure(nq));
		RX_CUDA(cudaMemcpyAsync(s->d_q.p, hq.data(), hq.size(), cudaMemcpyHostToDevice, st));
		RX_CUDA(cudaMemcpyAsync(s->d_qcorr.p, hcorr.data(), size_t(nq) * 4, cudaMemcpyHostToDevice, st));
		RX_CUDA(cudaMemcpyAsync(s->d_qcoef.p, hcoef.data(), size_t(nq) * 4, cudaMemcpyHostToDevice, st));
		// the widest query tile the batch fills whose staged codes and key lists fit the budget: at k = 256, qt = 4 holds up to 7056
		// dims, qt = 2 up to 32656 and qt = 1 every dimension the index accepts, so the refusal below is only a guard
		int qt = nq >= 4 ? 4 : (nq >= 2 ? 2 : 1);
		while (qt > 1 && sqScanSmem(qt, cp, kEff) > 100 * 1024) {
			qt /= 2;
		}
		const unsigned grid = unsigned(std::min<uint64_t>(uint64_t(ix->sm_count) * 2, std::max<uint64_t>(1, (ix->size + 2 * kSqWarps - 1) / (2 * kSqWarps))));
		const size_t smem = sqScanSmem(qt, cp, kEff);
		if (smem > 100 * 1024) {
			return fail(RXGPU_ERR_PARAMS, "rxgpu: dimension/k combination exceeds the shared-memory budget of the SQ8 scan");
		}
		RX_CUDA(s->d_lists.ensure(size_t(grid) * qt * kEff));
		RX_CUDA(s->d_dist.ensure(size_t(nq) * kEff));
		RX_CUDA(s->d_idx.ensure(size_t(nq) * kEff));
		RX_CUDA(s->d_label.ensure(size_t(nq) * kEff));
		RX_CUDA(s->d_count.ensure(nq));
		RX_CUDA(raiseSmemCeilingOnce(sq8_scan_kernel<1>, ix->device, 100 * 1024));
		RX_CUDA(raiseSmemCeilingOnce(sq8_scan_kernel<2>, ix->device, 100 * 1024));
		RX_CUDA(raiseSmemCeilingOnce(sq8_scan_kernel<4>, ix->device, 100 * 1024));
		for (uint32_t q0 = 0; q0 < nq; q0 += qt) {
			SqScanArgs a{};
			a.codes = s->codes.p;
			a.corr = s->corr.p;
			a.norm_coefs = ix->metric == RXGPU_COS ? ix->d_norms : nullptr;
			a.qcodes = s->d_q.p + size_t(q0) * cp;
			a.qcorr = s->d_qcorr.p + q0;
			a.qcoef = s->d_qcoef.p + q0;
			a.lists = s->d_lists.p;
			a.code_pitch = cp;
			a.n = uint32_t(ix->size);
			a.nq = std::min<uint32_t>(qt, nq - q0);
			a.k1 = kEff;
			a.alpha2 = s->params.alpha_2;
			a.is_l2 = ix->metric == RXGPU_L2;
			if (qt == 4) {
				sq8_scan_kernel<4><<<grid, kSqThreads, smem, st>>>(a);
			} else if (qt == 2) {
				sq8_scan_kernel<2><<<grid, kSqThreads, smem, st>>>(a);
			} else {
				sq8_scan_kernel<1><<<grid, kSqThreads, smem, st>>>(a);
			}
			sq8_merge_kernel<<<a.nq, 32, 0, st>>>(s->d_lists.p, grid, qt, kEff, q0, ix->d_labels, s->d_dist.p, s->d_label.p, s->d_idx.p, s->d_count.p);
			RX_CUDA(cudaGetLastError());
			g_stats.launches += 2;
			g_stats.passes += 1;
		}
		std::vector<float> hd(size_t(nq) * kEff);
		std::vector<uint64_t> hl(size_t(nq) * kEff);
		std::vector<uint32_t> hc(nq);
		RX_CUDA(cudaMemcpyAsync(hd.data(), s->d_dist.p, hd.size() * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(hl.data(), s->d_label.p, hl.size() * 8, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaMemcpyAsync(hc.data(), s->d_count.p, size_t(nq) * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		std::vector<Hit> hits;
		for (uint32_t q = 0; q < nq; ++q) {
			hits.clear();
			for (uint32_t j = 0; j < std::min(hc[q], kEff); ++j) {
				hits.push_back(Hit{hd[size_t(q) * kEff + j], 0, hl[size_t(q) * kEff + j]});
			}
			orderTiesByLabel(hits);  // the result queue's comparator (std::less<pair<float, label>>)
			for (size_t j = 0; j < hits.size(); ++j) {
				out_dist[size_t(q) * k + j] = hits[j].dist;
				out_label[size_t(q) * k + j] = hits[j].label;
			}
			out_count[q] = uint32_t(hits.size());
		}
		g_stats.query_tile = uint32_t(qt);
		g_stats.algorithmic_bytes = uint64_t((nq + qt - 1) / qt) * (uint64_t(ix->size) * (cp + 4) + (ix->metric == RXGPU_COS ? uint64_t(ix->size) * 4 : 0));
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

}  // extern "C"
