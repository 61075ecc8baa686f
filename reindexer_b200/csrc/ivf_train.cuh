// k-means on the device (rxgpu_ivf_train, ivf_train.cu): the kernels of one Lloyd iteration after the assignment, which is the coarse
// pass's own kernel in argmin mode (ivf_coarse.cuh: ivf_coarse_dist_kernel<..., kArgmin = true>).  faiss::Clustering::train restated:
//   kmeans_split_keys_kernel -- the assignment keys into (centroid, point) pairs for the stable radix sort by centroid
//   kmeans_update_kernel     -- compute_centroids (Clustering.cpp:153-235): one thread per (centroid, coordinate) sums the centroid's
//                               members in ascending point order in fp32 starting from 0, then multiplies by 1 / count in fp32 (count
//                               as FAISS's float histogram holds it); an empty centroid is 0
//   kmeans_split_kernel      -- split_clusters (:247-294) given the host's choices: copy, then the symmetric perturbation x (1 +- 2^-10)
//                               taken in double and rounded once, as FAISS's `float *= double` does; pairs applied in order
//   kmeans_renorm_kernel     -- fvec_renorm_L2 for spherical k-means: fp64 norm, each coordinate divided by it and rounded once
//   kmeans_gather_rows_kernel -- the sharded training's row moves: the all-gathered sample into plan order, initial centroids from it
#pragma once
#include "common.cuh"

namespace rxgpu {

__global__ void kmeans_split_keys_kernel(const uint64_t* keys, uint32_t n, uint32_t* assign, uint32_t* point) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) {
		assign[i] = uint32_t(keys[i]);
		point[i] = i;
	}
}

// grid (nlist, ceil(dim / 128)), 128 threads: members of centroid c are point[off[c] .. off[c + 1]) of x [n][dim], ascending
__global__ void __launch_bounds__(128) kmeans_update_kernel(const float* x, uint32_t dim, const uint32_t* point, const uint32_t* off,
															 float* centroids, uint32_t pitch) {
	const uint32_t c = blockIdx.x, j = blockIdx.y * 128u + threadIdx.x;
	if (j >= dim) {
		return;
	}
	const uint32_t b = off[c], e = off[c + 1];
	float s = 0.f;
	uint32_t m = b;
	for (; m + 4 <= e; m += 4) {  // four loads in flight, added in order
		const float v0 = x[size_t(point[m]) * dim + j], v1 = x[size_t(point[m + 1]) * dim + j];
		const float v2 = x[size_t(point[m + 2]) * dim + j], v3 = x[size_t(point[m + 3]) * dim + j];
		s = __fadd_rn(s, v0);
		s = __fadd_rn(s, v1);
		s = __fadd_rn(s, v2);
		s = __fadd_rn(s, v3);
	}
	for (; m < e; ++m) {
		s = __fadd_rn(s, x[size_t(point[m]) * dim + j]);
	}
	if (e > b) {
		// FAISS counts in a float (hassign[ci] += 1.0), which stops growing at 2^24
		const float h = float(min(e - b, 1u << 24));
		s = __fmul_rn(s, __fdiv_rn(1.f, h));
	}
	centroids[size_t(c) * pitch + j] = s;
}

// one thread per coordinate: splits (ci, cj) in FAISS's order -- a later split may copy an earlier one's result, coordinate by coordinate
__global__ void kmeans_split_kernel(const uint2* splits, uint32_t nsplit, uint32_t dim, float* centroids, uint32_t pitch) {
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= dim) {
		return;
	}
	const double up = 1.0 + 1.0 / 1024.0, down = 1.0 - 1.0 / 1024.0;
	for (uint32_t s = 0; s < nsplit; ++s) {
		float* ci = centroids + size_t(splits[s].x) * pitch;
		float* cj = centroids + size_t(splits[s].y) * pitch;
		const double v = double(cj[j]);
		ci[j] = __double2float_rn(__dmul_rn(v, (j & 1) ? down : up));
		cj[j] = __double2float_rn(__dmul_rn(v, (j & 1) ? up : down));
	}
}

// one warp per centroid
__global__ void kmeans_renorm_kernel(float* centroids, uint32_t pitch, uint32_t dim, uint32_t nlist) {
	const uint32_t c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
	const int lane = threadIdx.x & 31;
	if (c >= nlist) {
		return;
	}
	float* row = centroids + size_t(c) * pitch;
	double s = 0.0;
	for (uint32_t j = lane; j < dim; j += 32) {
		s = __fma_rn(double(row[j]), double(row[j]), s);
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		s += __shfl_xor_sync(0xffffffffu, s, o);
	}
	if (s > 0.0) {
		const double nr = sqrt(s);
		for (uint32_t j = lane; j < dim; j += 32) {
			row[j] = __double2float_rn(__ddiv_rn(double(row[j]), nr));
		}
	}
}

// one CTA per output row: dst[i] (pitch dstPitch) = src[from[i]] (pitch dim), coordinates copied as they are
__global__ void kmeans_gather_rows_kernel(const float* src, uint32_t dim, const uint64_t* from, float* dst, uint32_t dstPitch) {
	const float* s = src + from[blockIdx.x] * dim;
	float* d = dst + size_t(blockIdx.x) * dstPitch;
	for (uint32_t j = threadIdx.x; j < dim; j += blockDim.x) {
		d[j] = s[j];
	}
}

}  // namespace rxgpu
