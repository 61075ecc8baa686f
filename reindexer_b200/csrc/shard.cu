// Multi-GPU brute-force KNN behind the C ABI (SURVEY.md 8e): the namespace is sharded by internal-row range, one shard per GPU / rank.
// One call = local fused scan + top-(k+1) on this rank's shard, ONE ncclAllGather of the per-shard lists over NVLink / NVSwitch, a
// device-side k-way merge under the reference's comparator, and -- only when bit-equal distances straddle the k-th place -- the
// reference's heap tie rule (bruteforce.cc:103-127) replayed globally from the filter's per-query candidate lists (every row at or
// below the k-th distance is in them, so no shard is scanned a second time) with a second, tiny all-gather.
// Range batches: each shard answers its part with rxgpu_search_range_batch's core, two all-reduces agree on the totals and on a payload
// width, one all-gather ships every shard's best min(matches, max_out) per query, and a warp per query merges them under hitLessByLabel.
// IVF (rxgpu_sharded_ivf_search_knn / _range_batch): each shard's part of the IVF search (ivf.cu), then the same merge and range exchange,
// with the words every rank must agree on (centroid fingerprint, nlist, nprobe, ...) and its status carried through the first exchange.
// The exchanges go through commAllGather / commAllReduce: NCCL between processes, a host rendezvous between the threads of one process.
// NCCL is resolved with dlopen at the first rxgpu_comm_* call: librxgpu.so itself keeps loading on a box without NCCL or a GPU.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <condition_variable>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/rxgpu.h"
#include "../host/knn_select.h"
#include "internal.h"
#include "common.cuh"

using namespace rxgpu;

namespace {

struct NcclApi {
	ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
	ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
	ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
	ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
	const char* (*GetErrorString)(ncclResult_t) = nullptr;
	bool ok = false;
};
const NcclApi& nccl() {
	static NcclApi api = [] {
		NcclApi a;
		void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
		if (!h) {
			h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
		}
		if (!h) {
			return a;
		}
		a.GetUniqueId = reinterpret_cast<decltype(a.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
		a.CommInitRank = reinterpret_cast<decltype(a.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
		a.CommDestroy = reinterpret_cast<decltype(a.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
		a.AllGather = reinterpret_cast<decltype(a.AllGather)>(dlsym(h, "ncclAllGather"));
		a.AllReduce = reinterpret_cast<decltype(a.AllReduce)>(dlsym(h, "ncclAllReduce"));
		a.GetErrorString = reinterpret_cast<decltype(a.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
		a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.AllGather && a.AllReduce && a.GetErrorString;
		return a;
	}();
	return api;
}
#define RX_NCCL(expr)                                                                                               \
	do {                                                                                                            \
		ncclResult_t r_ = (expr);                                                                                   \
		if (r_ != ncclSuccess) {                                                                                    \
			return fail(RXGPU_ERR_SYSTEM, std::string("NCCL error: ") + nccl().GetErrorString(r_) + " at " #expr); \
		}                                                                                                           \
	} while (0)

// Layout of one rank's contribution to the exchange (all sections 16-byte aligned):
//   [dist f32 nq*k1][idx u32 nq*k1][label u64 nq*k1][count u32 nq][size u64, pad] -- the IVF search's header (IvfHeader) in place of
// [size u64, pad]
struct PayloadLayout {
	size_t off_dist, off_idx, off_label, off_count, off_size, bytes;
	PayloadLayout(uint32_t nq, uint32_t k1, size_t header = 16) {
		auto up = [](size_t x) { return (x + 15) & ~size_t(15); };
		const size_t n = size_t(nq) * k1;
		off_dist = 0;
		off_idx = up(off_dist + n * 4);
		off_label = up(off_idx + n * 4);
		off_count = up(off_label + n * 8);
		off_size = up(off_count + size_t(nq) * 4);
		bytes = up(off_size + header);
	}
};

// One warp per query: lane s walks shard s's list (already ascending under (dist, internal row)); k rounds of a warp-wide minimum
// under (dist, global row) give the global top-k; one more round looks at the (k+1)-th candidate to flag a straddling tie.
// Map-space distances compare as floats (-0 == +0, like the reference's float compare and the host merge).
__global__ void shard_merge_kernel(const unsigned char* all, uint32_t nshards, uint32_t nq, uint32_t k, uint32_t k1, PayloadLayout lay,
								   float* out_dist, uint64_t* out_gidx, uint64_t* out_label, uint32_t* out_count, uint8_t* need_tie) {
	const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	const int lane = threadIdx.x & 31;
	if (q >= nq) {
		return;
	}
	// shard bases = prefix sums of the shard sizes (rows are appended shard by shard)
	uint64_t base = 0;
	for (uint32_t s = 0; s < nshards && s < uint32_t(lane); ++s) {
		base += *reinterpret_cast<const uint64_t*>(all + size_t(s) * lay.bytes + lay.off_size);
	}
	const unsigned char* mine = all + size_t(lane) * lay.bytes;
	const bool have = uint32_t(lane) < nshards;
	const uint32_t cnt = have ? min(reinterpret_cast<const uint32_t*>(mine + lay.off_count)[q], k1) : 0u;
	const float* d = reinterpret_cast<const float*>(mine + lay.off_dist) + size_t(q) * k1;
	const uint32_t* ix = reinterpret_cast<const uint32_t*>(mine + lay.off_idx) + size_t(q) * k1;
	const uint64_t* lb = reinterpret_cast<const uint64_t*>(mine + lay.off_label) + size_t(q) * k1;
	uint32_t head = 0, n = 0;
	float last = 0.f;
	bool tie = false;
	for (uint32_t r = 0; r <= k; ++r) {
		float hd = head < cnt ? d[head] : INFINITY;
		uint64_t hg = head < cnt ? base + ix[head] : ~0ull;
		bool valid = head < cnt;
		int owner = lane;
#pragma unroll
		for (int off = 16; off > 0; off >>= 1) {
			const float od = __shfl_xor_sync(0xffffffffu, hd, off);
			const uint64_t og = __shfl_xor_sync(0xffffffffu, hg, off);
			const bool ov = __shfl_xor_sync(0xffffffffu, valid, off);
			const int oo = __shfl_xor_sync(0xffffffffu, owner, off);
			const bool better = ov && (!valid || od < hd || (!(hd < od) && og < hg));
			if (better) {
				hd = od;
				hg = og;
				valid = ov;
				owner = oo;
			}
		}
		if (!valid) {
			break;
		}
		if (r == k) {
			tie = !(last < hd);  // the k-th and the (k+1)-th distance are bit-equal (as floats): the reference's tie rule decides
			break;
		}
		if (lane == owner) {
			out_dist[size_t(q) * k + r] = d[head];
			out_gidx[size_t(q) * k + r] = hg;
			out_label[size_t(q) * k + r] = lb[head];
			++head;
		}
		last = hd;
		++n;
	}
	if (lane == 0) {
		out_count[q] = n;
		need_tie[q] = tie ? 1 : 0;
	}
}

// Layout of one rank's contribution to the range exchange (all sections 16-byte aligned), w entries per query:
//   [dist f32 nq*w][label u64 nq*w][kept u32 nq]
struct RangeLayout {
	size_t off_dist, off_label, off_kept, bytes;
	RangeLayout(uint32_t nq, uint32_t w) {
		auto up = [](size_t x) { return (x + 15) & ~size_t(15); };
		const size_t n = size_t(nq) * w;
		off_dist = 0;
		off_label = up(n * 4);
		off_kept = up(off_label + n * 8);
		bytes = up(off_kept + size_t(nq) * 4);
	}
};

// The header of a sharded IVF KNN payload: the shard's size first, as the merge reads it, then what every rank must agree on, and the
// status of its local part
struct IvfHeader {
	uint64_t size, fingerprint;
	uint32_t nlist, nprobe, k, dim, metric;
	int32_t status;
};

// One rank's part of a sharded range batch: per query its matches in total and the best min(total, max_out) of them, best first under
// hitLessByLabel, at dist / label [first, first + kept)
struct RangeLocal {
	std::vector<uint64_t> n;
	std::vector<uint32_t> kept;
	std::vector<size_t> first;
	std::vector<float> dist;
	std::vector<uint64_t> label;
	explicit RangeLocal(uint32_t nq) : n(nq, 0), kept(nq, 0), first(nq, 0) {}
};

// One warp per query: lane s walks shard s's matches, already best first under hitLessByLabel.  Each round writes the warp-wide minimum
// under that same comparator -- a float compare of the distances (-0 == +0), then the label, which is unique across the shards -- and the
// owning lane advances, until `width` entries are out or every list is drained.  Row q of the output holds `width` entries; the ones
// after the answer are zeroed.
__global__ void range_merge_kernel(const unsigned char* all, uint32_t nshards, uint32_t nq, uint32_t w, RangeLayout lay, uint32_t width,
								   float* out_dist, uint64_t* out_label) {
	const uint32_t q = (blockIdx.x * blockDim.x + threadIdx.x) / 32;
	const int lane = threadIdx.x & 31;
	if (q >= nq) {
		return;
	}
	const unsigned char* mine = all + size_t(lane) * lay.bytes;
	const bool have = uint32_t(lane) < nshards;
	const uint32_t cnt = have ? min(reinterpret_cast<const uint32_t*>(mine + lay.off_kept)[q], w) : 0u;
	const float* d = reinterpret_cast<const float*>(mine + lay.off_dist) + size_t(q) * w;
	const uint64_t* lb = reinterpret_cast<const uint64_t*>(mine + lay.off_label) + size_t(q) * w;
	float* od_row = out_dist + size_t(q) * width;
	uint64_t* ol_row = out_label + size_t(q) * width;
	uint32_t head = 0, r = 0;
	for (; r < width; ++r) {
		bool valid = head < cnt;
		float hd = valid ? d[head] : INFINITY;
		uint64_t hl = valid ? lb[head] : ~0ull;
		int owner = lane;
#pragma unroll
		for (int off = 16; off > 0; off >>= 1) {
			const float od = __shfl_xor_sync(0xffffffffu, hd, off);
			const uint64_t ol = __shfl_xor_sync(0xffffffffu, hl, off);
			const bool ov = __shfl_xor_sync(0xffffffffu, valid, off);
			const int oo = __shfl_xor_sync(0xffffffffu, owner, off);
			const bool better = ov && (!valid || od < hd || (!(hd < od) && ol < hl));
			if (better) {
				hd = od;
				hl = ol;
				valid = ov;
				owner = oo;
			}
		}
		if (!valid) {
			break;
		}
		if (lane == owner) {
			od_row[r] = hd;  // the winner's own bits: -0 stays -0
			ol_row[r] = hl;
			++head;
		}
	}
	for (uint32_t j = r + uint32_t(lane); j < width; j += 32) {
		od_row[j] = 0.f;
		ol_row[j] = 0;
	}
}

}  // namespace

// Ranks that live in ONE process (one host thread per rank; the GPUs may differ or be the same): the exchange goes through pinned host
// memory behind a rendezvous instead of NCCL, which refuses two ranks on one device.  This is what a single reindexer process driving
// several GPUs uses, and what lets a one-GPU box exercise every cross-shard code path.
struct LocalGroup {
	int n = 0;
	std::mutex m;
	std::condition_variable cv;
	int arrived = 0;
	uint64_t generation = 0;
	std::vector<std::vector<unsigned char>> contrib;  // per rank
	std::vector<unsigned char> result;
	template <class F>
	void rendezvous(F&& leader_work) {  // the last rank to arrive runs leader_work, then everybody leaves
		std::unique_lock<std::mutex> lck(m);
		if (++arrived == n) {
			leader_work();
			arrived = 0;
			++generation;
			cv.notify_all();
		} else {
			const uint64_t g = generation;
			cv.wait(lck, [&] { return generation != g; });
		}
	}
};

struct rxgpu_comm {
	ncclComm_t comm = nullptr;
	std::shared_ptr<LocalGroup> local;  // set: the ranks of this communicator are threads of this process
	int nranks = 1, rank = 0, device = 0;
	cudaStream_t stream = nullptr;
	std::mutex mtx;  // one collective call at a time per communicator
	DevBuf<float> d_queries;
	DevBuf<unsigned char> d_send, d_recv;
	DevBuf<float> d_m_dist;
	DevBuf<uint64_t> d_m_gidx, d_m_label;
	DevBuf<uint32_t> d_m_count;
	DevBuf<uint8_t> d_m_tie;
	PinBuf<float> h_m_dist;
	PinBuf<uint64_t> h_m_gidx, h_m_label;
	PinBuf<uint32_t> h_m_count;
	PinBuf<uint8_t> h_m_tie;
	PinBuf<unsigned char> h_tie_recv;
	PinBuf<uint64_t> h_size;
	DevBuf<uint64_t> d_r_n;  // range batch: the per-query totals
	DevBuf<uint32_t> d_r_words;  // range batch: the agreed width (and the IVF search's status and words every rank must hold)
	PinBuf<uint64_t> h_r_n;
	PinBuf<unsigned char> h_r_send;  // this rank's range payload, staged for the copy to the device
	~rxgpu_comm() {
		cudaSetDevice(device);
		if (comm && nccl().ok) {
			nccl().CommDestroy(comm);
		}
		if (stream) {
			cudaStreamDestroy(stream);
		}
	}
};

// ---- collectives for the other translation units (declared in internal.h): in place on device buffers, on the caller's stream ------
namespace rxgpu {
int commRank(const rxgpu_comm* c) { return c ? c->rank : 0; }
int commSize(const rxgpu_comm* c) { return c ? c->nranks : 1; }
int commDevice(const rxgpu_comm* c) { return c ? c->device : 0; }
std::mutex& commMutex(rxgpu_comm* c) { return c->mtx; }

int commAllReduce(rxgpu_comm* c, void* d_buf, size_t count, CommOp op, cudaStream_t st) {
	if (!c || c->nranks == 1 || count == 0) {
		return 0;
	}
	const size_t esz = op == CommOp::SumU64 ? 8 : 4;
	if (c->local) {
		LocalGroup& g = *c->local;
		std::vector<unsigned char>& mine = g.contrib[size_t(c->rank)];
		mine.resize(count * esz);
		RX_CUDA(cudaMemcpyAsync(mine.data(), d_buf, count * esz, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		g.rendezvous([&] {
			g.result = g.contrib[0];
			for (int r = 1; r < g.n; ++r) {
				for (size_t i = 0; i < count; ++i) {
					if (op == CommOp::SumU64) {
						reinterpret_cast<unsigned long long*>(g.result.data())[i] += reinterpret_cast<const unsigned long long*>(g.contrib[size_t(r)].data())[i];
					} else if (op == CommOp::SumU32) {
						reinterpret_cast<uint32_t*>(g.result.data())[i] += reinterpret_cast<const uint32_t*>(g.contrib[size_t(r)].data())[i];
					} else {
						uint32_t& a = reinterpret_cast<uint32_t*>(g.result.data())[i];
						a = std::max(a, reinterpret_cast<const uint32_t*>(g.contrib[size_t(r)].data())[i]);
					}
				}
			}
		});
		RX_CUDA(cudaMemcpyAsync(d_buf, g.result.data(), count * esz, cudaMemcpyHostToDevice, st));
		RX_CUDA(cudaStreamSynchronize(st));
		g.rendezvous([] {});  // nobody starts the next exchange (which rewrites `result`) before everybody has copied this one
		return 0;
	}
	const ncclDataType_t ty = op == CommOp::SumU64 ? ncclUint64 : ncclUint32;
	RX_NCCL(nccl().AllReduce(d_buf, d_buf, count, ty, op == CommOp::MaxU32 ? ncclMax : ncclSum, c->comm, st));
	return 0;
}

int commAllGather(rxgpu_comm* c, const void* d_send, void* d_recv, size_t bytes, cudaStream_t st) {
	if (bytes == 0) {
		return 0;
	}
	if (!c || c->nranks == 1) {
		RX_CUDA(cudaMemcpyAsync(d_recv, d_send, bytes, cudaMemcpyDeviceToDevice, st));
		return 0;
	}
	if (c->local) {
		LocalGroup& g = *c->local;
		std::vector<unsigned char>& mine = g.contrib[size_t(c->rank)];
		mine.resize(bytes);
		RX_CUDA(cudaMemcpyAsync(mine.data(), d_send, bytes, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		g.rendezvous([&] {
			g.result.resize(bytes * size_t(g.n));
			for (int r = 0; r < g.n; ++r) {
				std::memcpy(g.result.data() + bytes * size_t(r), g.contrib[size_t(r)].data(), bytes);
			}
		});
		RX_CUDA(cudaMemcpyAsync(d_recv, g.result.data(), bytes * size_t(g.n), cudaMemcpyHostToDevice, st));
		RX_CUDA(cudaStreamSynchronize(st));
		g.rendezvous([] {});
		return 0;
	}
	RX_NCCL(nccl().AllGather(d_send, d_recv, bytes, ncclChar, c->comm, st));
	return 0;
}
}  // namespace rxgpu

namespace {
// The device merge of the R payloads gathered in c->d_recv (layout `lay`, k1 >= k entries per query): the k best under (distance, global
// row), then on the host the runs of bit-equal distances ordered by label, into out_* (host, nq x k); the merged rows stay in c->h_m_*.
// With tieQ, the queries whose k-th and (k+1)-th distances are bit-equal go to tieQ, with that distance to tieD.
int mergePayloads(rxgpu_comm* c, uint32_t nq, uint32_t k, uint32_t k1, const PayloadLayout& lay, cudaStream_t st, float* out_dist,
				  uint64_t* out_label, uint32_t* out_count, std::vector<uint32_t>* tieQ, std::vector<float>* tieD) {
	const size_t on = size_t(nq) * k;
	RX_CUDA(c->d_m_dist.ensure(on));
	RX_CUDA(c->d_m_gidx.ensure(on));
	RX_CUDA(c->d_m_label.ensure(on));
	RX_CUDA(c->d_m_count.ensure(nq));
	RX_CUDA(c->d_m_tie.ensure(nq));
	RX_CUDA(c->h_m_dist.ensure(on));
	RX_CUDA(c->h_m_gidx.ensure(on));
	RX_CUDA(c->h_m_label.ensure(on));
	RX_CUDA(c->h_m_count.ensure(nq));
	RX_CUDA(c->h_m_tie.ensure(nq));
	const unsigned blocks = unsigned((uint64_t(nq) * 32 + 255) / 256);
	shard_merge_kernel<<<blocks, 256, 0, st>>>(c->d_recv.p, uint32_t(c->nranks), nq, k, k1, lay, c->d_m_dist.p, c->d_m_gidx.p, c->d_m_label.p,
											   c->d_m_count.p, c->d_m_tie.p);
	RX_CUDA(cudaGetLastError());
	RX_CUDA(cudaMemcpyAsync(c->h_m_dist.p, c->d_m_dist.p, on * 4, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaMemcpyAsync(c->h_m_gidx.p, c->d_m_gidx.p, on * 8, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaMemcpyAsync(c->h_m_label.p, c->d_m_label.p, on * 8, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaMemcpyAsync(c->h_m_count.p, c->d_m_count.p, size_t(nq) * 4, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaMemcpyAsync(c->h_m_tie.p, c->d_m_tie.p, nq, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaStreamSynchronize(st));
	collectProfile();
	// runs of bit-equal distances ordered by label (the drain order of the reference's heap, and the order of rxgpu_ivf_search_knn)
	std::vector<Hit> top;
	for (uint32_t q = 0; q < nq; ++q) {
		const uint32_t n = c->h_m_count.p[q];
		top.resize(n);
		bool anyEqual = false;
		for (uint32_t j = 0; j < n; ++j) {
			top[j] = Hit{c->h_m_dist.p[size_t(q) * k + j], c->h_m_gidx.p[size_t(q) * k + j], c->h_m_label.p[size_t(q) * k + j]};
			anyEqual |= j && !(top[j - 1].dist < top[j].dist);
		}
		if (anyEqual) {
			orderTiesByLabel(top);
		}
		for (uint32_t j = 0; j < n; ++j) {
			out_dist[size_t(q) * k + j] = top[j].dist;
			out_label[size_t(q) * k + j] = top[j].label;
		}
		out_count[q] = n;
		if (tieQ && c->h_m_tie.p[q] && n == k) {
			tieQ->push_back(q);
			tieD->push_back(c->h_m_dist.p[size_t(q) * k + k - 1]);
		}
	}
	return 0;
}

// The exchange of the sharded range batches after each rank's local part `loc`: one MaxU32 all-reduce of the width every rank sends --
// and, when `agree` is given, of this rank's status and of every word of `agree` beside its complement, so that the ranks learn at once
// whether any failed (that code, on every rank) or differ in a word (errLogic) -- then the SumU64 all-reduce of the totals, one
// all-gather of min(matches, max_out) per query and shard, and range_merge_kernel.  The totals go to out_n, the merged rows to
// out_dist / out_label (host, nq x max_out).
int rangeExchange(rxgpu_comm* c, uint32_t nq, uint64_t max_out, const RangeLocal& loc, int status, const std::string& why,
				  const std::vector<uint32_t>* agree, cudaStream_t st, float* out_dist, uint64_t* out_label, uint64_t* out_n) {
	const uint32_t R = uint32_t(c->nranks);
	uint32_t W = *std::max_element(loc.kept.begin(), loc.kept.end());
	if (max_out || agree) {
		std::vector<uint32_t> words{W, uint32_t(status)};
		if (agree) {
			for (const uint32_t a : *agree) {
				words.push_back(a);
				words.push_back(~a);
			}
		}
		RX_CUDA(c->d_r_words.ensure(words.size()));
		RX_CUDA(cudaMemcpyAsync(c->d_r_words.p, words.data(), words.size() * 4, cudaMemcpyHostToDevice, st));
		if (int rc = commAllReduce(c, c->d_r_words.p, words.size(), CommOp::MaxU32, st)) {
			return rc;
		}
		RX_CUDA(cudaMemcpyAsync(words.data(), c->d_r_words.p, words.size() * 4, cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		if (words[1]) {
			return fail(int(words[1]), uint32_t(status) == words[1] ? why : "rxgpu: the sharded search failed on another rank");
		}
		for (size_t i = 2; i < words.size(); i += 2) {
			if (words[i] != ~words[i + 1]) {  // max(a) == ~max(~a) = min(a) only when every rank holds the same word
				return fail(RXGPU_ERR_LOGIC, "rxgpu: the shards of a sharded IVF search differ in their centroids, nlist, nprobe, dim or metric");
			}
		}
		W = words[0];
	}
	RX_CUDA(c->h_r_n.ensure(nq));
	RX_CUDA(c->d_r_n.ensure(nq));
	RX_CUDA(cudaMemcpyAsync(c->d_r_n.p, loc.n.data(), size_t(nq) * 8, cudaMemcpyHostToDevice, st));
	if (int rc = commAllReduce(c, c->d_r_n.p, nq, CommOp::SumU64, st)) {
		return rc;
	}
	RX_CUDA(cudaMemcpyAsync(c->h_r_n.p, c->d_r_n.p, size_t(nq) * 8, cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaStreamSynchronize(st));
	std::memcpy(out_n, c->h_r_n.p, size_t(nq) * 8);
	if (max_out == 0 || W == 0) {  // nothing to return, or no match on any shard
		return 0;
	}
	// one all-gather of the padded payloads, the device merge, and only the merged rows cross to the host
	const RangeLayout lay(nq, W);
	RX_CUDA(c->h_r_send.ensure(lay.bytes));
	float* h_dist = reinterpret_cast<float*>(c->h_r_send.p + lay.off_dist);
	uint64_t* h_label = reinterpret_cast<uint64_t*>(c->h_r_send.p + lay.off_label);
	for (uint32_t q = 0; q < nq; ++q) {
		std::memcpy(h_dist + size_t(q) * W, loc.dist.data() + loc.first[q], size_t(loc.kept[q]) * 4);
		std::memcpy(h_label + size_t(q) * W, loc.label.data() + loc.first[q], size_t(loc.kept[q]) * 8);
	}
	std::memcpy(c->h_r_send.p + lay.off_kept, loc.kept.data(), size_t(nq) * 4);
	RX_CUDA(c->d_send.ensure(lay.bytes));
	RX_CUDA(c->d_recv.ensure(lay.bytes * R));
	unsigned char* snd = R > 1 ? c->d_send.p : c->d_recv.p;  // a single shard merges its own payload in place
	RX_CUDA(cudaMemcpyAsync(snd, c->h_r_send.p, lay.bytes, cudaMemcpyHostToDevice, st));
	if (R > 1) {
		if (int rc = commAllGather(c, c->d_send.p, c->d_recv.p, lay.bytes, st)) {
			return rc;
		}
	}
	const uint32_t width = uint32_t(std::min<uint64_t>(max_out, uint64_t(R) * W));
	const size_t on = size_t(nq) * width;
	RX_CUDA(c->d_m_dist.ensure(on));
	RX_CUDA(c->d_m_label.ensure(on));
	const unsigned blocks = unsigned((uint64_t(nq) * 32 + 255) / 256);
	range_merge_kernel<<<blocks, 256, 0, st>>>(c->d_recv.p, R, nq, W, lay, width, c->d_m_dist.p, c->d_m_label.p);
	RX_CUDA(cudaGetLastError());
	g_stats.launches += 1;
	RX_CUDA(cudaMemcpy2DAsync(out_dist, size_t(max_out) * 4, c->d_m_dist.p, size_t(width) * 4, size_t(width) * 4, nq,
							  cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaMemcpy2DAsync(out_label, size_t(max_out) * 8, c->d_m_label.p, size_t(width) * 8, size_t(width) * 8, nq,
							  cudaMemcpyDeviceToHost, st));
	RX_CUDA(cudaStreamSynchronize(st));
	return 0;
}
}  // namespace

extern "C" {

int rxgpu_comm_unique_id(void* out128) {
	if (!out128) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	if (!nccl().ok) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: libnccl.so.2 could not be loaded (multi-GPU sharding needs NCCL)");
	}
	static_assert(sizeof(ncclUniqueId) == RXGPU_COMM_ID_BYTES, "unique id size");
	ncclUniqueId id;
	RX_NCCL(nccl().GetUniqueId(&id));
	std::memcpy(out128, &id, sizeof(id));
	return 0;
}

int rxgpu_comm_create(rxgpu_comm** out, int nranks, int rank, const void* id128, int device) {
	if (!out || nranks < 1 || rank < 0 || rank >= nranks || (nranks > 1 && !id128)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: bad communicator arguments");
	}
	*out = nullptr;
	if (nranks > 32) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: at most 32 shards per communicator (one warp lane per shard in the merge)");
	}
	if (rxgpu_device_count() <= device || device < 0) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: no usable CUDA device (this library has no CPU fallback)");
	}
	RX_CUDA(cudaSetDevice(device));
	auto c = std::make_unique<rxgpu_comm>();
	c->nranks = nranks;
	c->rank = rank;
	c->device = device;
	RX_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
	if (nranks > 1) {
		if (!nccl().ok) {
			return fail(RXGPU_ERR_SYSTEM, "rxgpu: libnccl.so.2 could not be loaded (multi-GPU sharding needs NCCL)");
		}
		ncclUniqueId id;
		std::memcpy(&id, id128, sizeof(id));
		RX_NCCL(nccl().CommInitRank(&c->comm, nranks, id, rank));
	}
	*out = c.release();
	return 0;
}

int rxgpu_comm_create_local(rxgpu_comm** out, int nranks, const int* devices) {
	if (!out || nranks < 1 || nranks > 32) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: bad communicator arguments (1..32 ranks)");
	}
	for (int r = 0; r < nranks; ++r) {
		out[r] = nullptr;
	}
	auto group = std::make_shared<LocalGroup>();
	group->n = nranks;
	group->contrib.resize(size_t(nranks));
	std::vector<std::unique_ptr<rxgpu_comm>> made;
	for (int r = 0; r < nranks; ++r) {
		const int device = devices ? devices[r] : 0;
		if (rxgpu_device_count() <= device || device < 0) {
			return fail(RXGPU_ERR_SYSTEM, "rxgpu: no usable CUDA device (this library has no CPU fallback)");
		}
		RX_CUDA(cudaSetDevice(device));
		auto c = std::make_unique<rxgpu_comm>();
		c->nranks = nranks;
		c->rank = r;
		c->device = device;
		c->local = group;
		RX_CUDA(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
		made.push_back(std::move(c));
	}
	for (int r = 0; r < nranks; ++r) {
		out[r] = made[size_t(r)].release();
	}
	return 0;
}

void rxgpu_comm_destroy(rxgpu_comm* c) { delete c; }
int rxgpu_comm_rank(const rxgpu_comm* c) { return c ? c->rank : -1; }
int rxgpu_comm_size(const rxgpu_comm* c) { return c ? c->nranks : 0; }

int rxgpu_merge_shards_device(uint32_t nshards, uint32_t nq, uint32_t k, uint32_t k1, const void* d_payloads, float* d_out_dist,
							  uint64_t* d_out_gidx, uint64_t* d_out_label, uint32_t* d_out_count, uint8_t* d_need_tie, void* stream) {
	if (nshards == 0 || nshards > 32 || k == 0 || k1 < k) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: bad shard merge arguments");
	}
	if (nq == 0) {
		return 0;
	}
	const PayloadLayout lay(nq, k1);
	const unsigned blocks = unsigned((uint64_t(nq) * 32 + 255) / 256);
	shard_merge_kernel<<<blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(static_cast<const unsigned char*>(d_payloads), nshards, nq, k, k1, lay,
																			 d_out_dist, d_out_gidx, d_out_label, d_out_count, d_need_tie);
	RX_CUDA(cudaGetLastError());
	return 0;
}

uint64_t rxgpu_shard_payload_bytes(uint32_t nq, uint32_t k1) { return PayloadLayout(nq, k1).bytes; }

int rxgpu_sharded_search_knn(rxgpu_comm* c, const rxgpu_index* ix, uint32_t nq, const float* queries, int queries_on_device, uint32_t k,
							 float* out_dist, uint64_t* out_label, uint32_t* out_count) {
	if (!c) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null communicator");
	}
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (ix->device != c->device) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: the shard lives on another device than its communicator");
	}
	if (nq && (!queries || !out_count || (k && (!out_dist || !out_label)))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	g_stats = rxgpu_search_stats{};
	if (nq == 0) {
		return 0;
	}
	if (k == 0) {
		std::memset(out_count, 0, size_t(nq) * 4);
		return 0;
	}
	const uint32_t k1 = k + 1;  // the same on every rank (shard sizes differ): one extra row exposes a tie at the k-th place
	if (k1 > 65536u) {  // kMaxSearchK1 of the scan
		return fail(RXGPU_ERR_PARAMS, "rxgpu: k must be in [1, 65535]");
	}
	std::lock_guard<std::mutex> lck(c->mtx);
	try {
		cudaStream_t st = c->stream;
		WsLease lease(ix);
		lease.st = st;
		Workspace& ws = *lease.ws;
		const PayloadLayout lay(nq, k1);
		const uint32_t R = uint32_t(c->nranks);
		const float* d_q = queries;
		if (!queries_on_device) {
			RX_CUDA(c->d_queries.ensure(size_t(nq) * ix->dim));
			RX_CUDA(cudaMemcpyAsync(c->d_queries.p, queries, size_t(nq) * ix->dim * 4, cudaMemcpyHostToDevice, st));
			d_q = c->d_queries.p;
		}
		RX_CUDA(c->d_send.ensure(lay.bytes));
		RX_CUDA(c->d_recv.ensure(lay.bytes * R));
		RX_CUDA(c->h_size.ensure(2));
		unsigned char* snd = R > 1 ? c->d_send.p : c->d_recv.p;  // a single shard merges its own payload in place
		float* s_dist = reinterpret_cast<float*>(snd + lay.off_dist);
		uint32_t* s_idx = reinterpret_cast<uint32_t*>(snd + lay.off_idx);
		uint64_t* s_label = reinterpret_cast<uint64_t*>(snd + lay.off_label);
		uint32_t* s_count = reinterpret_cast<uint32_t*>(snd + lay.off_count);
		c->h_size.p[0] = ix->size;
		c->h_size.p[1] = 0;
		RX_CUDA(cudaMemcpyAsync(snd + lay.off_size, c->h_size.p, 16, cudaMemcpyHostToDevice, st));
		// ---- 1. this shard's top-(k+1) under (dist, internal row), straight into the send buffer
		if (ix->size == 0) {
			RX_CUDA(cudaMemsetAsync(s_count, 0, size_t(nq) * 4, st));
			ws.tc_lists_valid = false;
		} else if (int rc = scanTopK(ix, ws, st, d_q, nq, k1, kModeTopK, 0.f, s_dist, s_idx, s_label, s_count)) {
			return rc;
		}
		const rxgpu_search_stats scanStats = g_stats;  // what the roofline figure describes: the shard scan, not the rare tie pass
		// ---- 2. one all-gather, 3. device merge, 4. bit-equal distances ordered by label
		if (R > 1) {
			if (int rc = commAllGather(c, c->d_send.p, c->d_recv.p, lay.bytes, st)) {
				return rc;
			}
		}
		std::vector<uint32_t> tieQ;
		std::vector<float> tieD;
		if (int rc = mergePayloads(c, nq, k, k1, lay, st, out_dist, out_label, out_count, &tieQ, &tieD)) {
			return rc;
		}
		// ---- 5. rare: a tie straddles the global k-th place of some queries (the same set on every rank) -> replay the reference's rule
		if (!tieQ.empty()) {
			const uint32_t nt = uint32_t(tieQ.size());
			const PayloadLayout tlay(nt, k);
			RX_CUDA(c->d_send.ensure(tlay.bytes));
			RX_CUDA(c->d_recv.ensure(tlay.bytes * R));
			unsigned char* tsnd = R > 1 ? c->d_send.p : c->d_recv.p;
			RX_CUDA(cudaMemcpyAsync(tsnd + tlay.off_size, c->h_size.p, 16, cudaMemcpyHostToDevice, st));
			if (ix->size == 0) {
				RX_CUDA(cudaMemsetAsync(tsnd + tlay.off_count, 0, size_t(nt) * 4, st));
			} else if (int rc = tieRowsAfterScan(ix, ws, st, d_q, nt, tieQ.data(), tieD.data(), k, reinterpret_cast<float*>(tsnd + tlay.off_dist),
												 reinterpret_cast<uint32_t*>(tsnd + tlay.off_idx), reinterpret_cast<uint64_t*>(tsnd + tlay.off_label),
												 reinterpret_cast<uint32_t*>(tsnd + tlay.off_count))) {
				return rc;
			}
			if (R > 1) {
				if (int rc = commAllGather(c, c->d_send.p, c->d_recv.p, tlay.bytes, st)) {
					return rc;
				}
			}
			RX_CUDA(c->h_tie_recv.ensure(tlay.bytes * R));
			RX_CUDA(cudaMemcpyAsync(c->h_tie_recv.p, c->d_recv.p, tlay.bytes * R, cudaMemcpyDeviceToHost, st));
			RX_CUDA(cudaStreamSynchronize(st));
			std::vector<uint64_t> base(R, 0);
			for (uint32_t s = 1; s < R; ++s) {
				base[s] = base[s - 1] + *reinterpret_cast<const uint64_t*>(c->h_tie_recv.p + size_t(s - 1) * tlay.bytes + tlay.off_size);
			}
			std::vector<Hit> lower, first;
			for (uint32_t t = 0; t < nt; ++t) {
				const uint32_t q = tieQ[t];
				const float dstar = tieD[t];
				lower.clear();
				first.clear();
				for (uint32_t j = 0; j < k && c->h_m_dist.p[size_t(q) * k + j] < dstar; ++j) {
					lower.push_back(Hit{c->h_m_dist.p[size_t(q) * k + j], c->h_m_gidx.p[size_t(q) * k + j], c->h_m_label.p[size_t(q) * k + j]});
				}
				for (uint32_t s = 0; s < R; ++s) {  // shards in rank order = global internal order; each list is already in internal order
					const unsigned char* p = c->h_tie_recv.p + size_t(s) * tlay.bytes;
					const uint32_t cnt = std::min(reinterpret_cast<const uint32_t*>(p + tlay.off_count)[t], k);
					for (uint32_t j = 0; j < cnt && first.size() < k; ++j) {
						first.push_back(Hit{reinterpret_cast<const float*>(p + tlay.off_dist)[size_t(t) * k + j],
											base[s] + reinterpret_cast<const uint32_t*>(p + tlay.off_idx)[size_t(t) * k + j],
											reinterpret_cast<const uint64_t*>(p + tlay.off_label)[size_t(t) * k + j]});
					}
				}
				const std::vector<Hit> res = tieReplay(k, dstar, lower, first);
				for (size_t j = 0; j < res.size(); ++j) {
					out_dist[size_t(q) * k + j] = res[j].dist;
					out_label[size_t(q) * k + j] = res[j].label;
				}
				out_count[q] = uint32_t(res.size());
			}
		}
		// report the shard scan's figures (kernel, tile, launches timed) plus what the tie pass added
		const rxgpu_search_stats after = g_stats;
		g_stats.query_tile = scanStats.query_tile;
		g_stats.tc_used = scanStats.tc_used;
		g_stats.tc_cluster = scanStats.tc_cluster;
		g_stats.tc_kernel = scanStats.tc_kernel;
		g_stats.tc_candidates = scanStats.tc_candidates;
		g_stats.tc_fallbacks = scanStats.tc_fallbacks;
		g_stats.launches = after.launches + 1;
		g_stats.tie_replays = uint32_t(tieQ.size());
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_sharded_search_range_batch(rxgpu_comm* c, const rxgpu_index* ix, uint32_t nq, const float* queries, int queries_on_device,
									 const float* radius, uint64_t max_out, float* out_dist, uint64_t* out_label, uint64_t* out_n) {
	if (!c) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null communicator");
	}
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (ix->device != c->device) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: the shard lives on another device than its communicator");
	}
	if (nq && (!queries || !radius || !out_n || (max_out && (!out_dist || !out_label)))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	g_stats = rxgpu_search_stats{};
	if (nq == 0) {
		return 0;
	}
	std::lock_guard<std::mutex> lck(c->mtx);
	try {
		cudaStream_t st = c->stream;
		// ---- 1. this shard's matches; the best min(n, max_out) of every query are kept, best first (a global top-max_out never needs more)
		RangeLocal loc(nq);
		if (ix->size != 0) {
			const float* d_q = queries;
			if (!queries_on_device) {
				RX_CUDA(c->d_queries.ensure(size_t(nq) * ix->dim));
				RX_CUDA(cudaMemcpyAsync(c->d_queries.p, queries, size_t(nq) * ix->dim * 4, cudaMemcpyHostToDevice, st));
				d_q = c->d_queries.p;
			}
			WsLease lease(ix);
			lease.st = st;
			const RangeEmit emit = [&](uint32_t q, const std::vector<Hit>& hits) {
				loc.n[q] = hits.size();
				loc.kept[q] = uint32_t(std::min<uint64_t>(hits.size(), max_out));
				loc.first[q] = loc.dist.size();
				for (uint32_t i = 0; i < loc.kept[q]; ++i) {
					loc.dist.push_back(hits[i].dist);
					loc.label.push_back(hits[i].label);
				}
			};
			if (int rc = rangeBatch(ix, *lease.ws, st, d_q, nq, radius, max_out, emit)) {
				return rc;
			}
		}
		// ---- 2. the width every rank sends and the totals over all shards, 3. one all-gather, 4. device merge
		return rangeExchange(c, nq, max_out, loc, 0, std::string(), nullptr, st, out_dist, out_label, out_n);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

int rxgpu_sharded_ivf_search_knn(rxgpu_comm* c, const rxgpu_index* ix, uint32_t nq, const float* queries, int queries_on_device, uint32_t k,
								 uint32_t nprobe, float* out_dist, uint64_t* out_label, uint32_t* out_count) {
	(void)queries_on_device;  // the coarse pass stages host and device queries alike
	if (!c) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null communicator");
	}
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (ix->device != c->device) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: the shard lives on another device than its communicator");
	}
	if (nq && (!queries || !out_count || !out_dist || !out_label)) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	g_stats = rxgpu_search_stats{};
	if (nq == 0) {
		return 0;
	}
	if (k == 0 || k > 65535u) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: IVF search needs k in [1, 65535]");
	}
	std::lock_guard<std::mutex> lck(c->mtx);
	try {
		cudaStream_t st = c->stream;
		const PayloadLayout lay(nq, k, sizeof(IvfHeader));
		const uint32_t R = uint32_t(c->nranks);
		RX_CUDA(c->d_send.ensure(lay.bytes));
		RX_CUDA(c->d_recv.ensure(lay.bytes * R));
		unsigned char* snd = R > 1 ? c->d_send.p : c->d_recv.p;  // a single shard merges its own payload in place
		// ---- 1. this shard's best k under (distance, local row), straight into the send buffer (on the index's stream, done on return)
		IvfShardView v{};
		const int status = ivfShardKnn(ix, nq, queries, k, nprobe, k, reinterpret_cast<float*>(snd + lay.off_dist),
									   reinterpret_cast<uint32_t*>(snd + lay.off_idx), reinterpret_cast<uint64_t*>(snd + lay.off_label),
									   reinterpret_cast<uint32_t*>(snd + lay.off_count), v);
		const std::string why = status ? g_err : std::string();
		const IvfHeader mine{v.rows, v.fingerprint, v.nlist, v.nprobe, k, ix->dim, uint32_t(ix->metric), status};
		RX_CUDA(cudaMemcpyAsync(snd + lay.off_size, &mine, sizeof(mine), cudaMemcpyHostToDevice, st));
		// ---- 2. one all-gather; every rank reads every header, so all return the same error or none
		if (R > 1) {
			if (int rc = commAllGather(c, c->d_send.p, c->d_recv.p, lay.bytes, st)) {
				return rc;
			}
		}
		std::vector<IvfHeader> hdr(R);
		RX_CUDA(cudaMemcpy2DAsync(hdr.data(), sizeof(IvfHeader), c->d_recv.p + lay.off_size, lay.bytes, sizeof(IvfHeader), R,
								  cudaMemcpyDeviceToHost, st));
		RX_CUDA(cudaStreamSynchronize(st));
		for (uint32_t r = 0; r < R; ++r) {
			if (hdr[r].status) {
				return fail(hdr[r].status, r == uint32_t(c->rank) ? why : "rxgpu: the sharded IVF search failed on rank " + std::to_string(r));
			}
		}
		for (uint32_t r = 1; r < R; ++r) {
			const IvfHeader& a = hdr[0];
			const IvfHeader& b = hdr[r];
			if (a.fingerprint != b.fingerprint || a.nlist != b.nlist || a.nprobe != b.nprobe || a.k != b.k || a.dim != b.dim || a.metric != b.metric) {
				return fail(RXGPU_ERR_LOGIC, "rxgpu: the shards of a sharded IVF search differ in their centroids, nlist, nprobe, k, dim or metric");
			}
		}
		// ---- 3. device merge under (distance, global row), 4. the k survivors by (distance, label)
		if (int rc = mergePayloads(c, nq, k, k, lay, st, out_dist, out_label, out_count, nullptr, nullptr)) {
			return rc;
		}
		g_stats.launches += 1;
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
	return 0;
}

int rxgpu_sharded_ivf_search_range_batch(rxgpu_comm* c, const rxgpu_index* ix, uint32_t nq, const float* queries, int queries_on_device,
										 const float* radius, uint32_t nprobe, uint64_t max_out, float* out_dist, uint64_t* out_label,
										 uint64_t* out_n) {
	(void)queries_on_device;  // the coarse pass stages host and device queries alike
	if (!c) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null communicator");
	}
	if (int rc = checkIndex(ix)) {
		return rc;
	}
	if (ix->device != c->device) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: the shard lives on another device than its communicator");
	}
	if (nq && (!queries || !radius || !out_n || (max_out && (!out_dist || !out_label)))) {
		return fail(RXGPU_ERR_PARAMS, "rxgpu: null argument");
	}
	g_stats = rxgpu_search_stats{};
	if (nq == 0) {
		return 0;
	}
	std::lock_guard<std::mutex> lck(c->mtx);
	try {
		// ---- 1. this shard's matches (the core of rxgpu_ivf_search_range_batch), the best min(n, max_out) of every query kept
		RangeLocal loc(nq);
		IvfShardView v{};
		const IvfRangeEmit emit = [&](uint32_t q, uint64_t n, const float* dist, const uint64_t* label, uint64_t m) {
			loc.n[q] = n;
			loc.kept[q] = uint32_t(m);
			loc.first[q] = loc.dist.size();
			loc.dist.insert(loc.dist.end(), dist, dist + m);
			loc.label.insert(loc.label.end(), label, label + m);
		};
		const int status = ivfShardRange(ix, nq, queries, radius, nprobe, max_out, emit, v);
		const std::string why = status ? g_err : std::string();
		const std::vector<uint32_t> agree{uint32_t(v.fingerprint), uint32_t(v.fingerprint >> 32), v.nlist, v.nprobe, ix->dim, uint32_t(ix->metric)};
		// ---- 2. the status, the agreed words and the width; the totals, 3. one all-gather, 4. device merge
		return rangeExchange(c, nq, max_out, loc, status, why, &agree, c->stream, out_dist, out_label, out_n);
	} catch (const std::bad_alloc&) {
		return fail(RXGPU_ERR_SYSTEM, "rxgpu: out of host memory");
	}
}

}  // extern "C"
