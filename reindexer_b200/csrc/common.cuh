// Shared device/host helpers for librxgpu (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace rxgpu {

// ---------------------------------------------------------------------------------------------------------------------
// Synthetic data generator (benchmark / test support).  Mirrored bit-for-bit by oracle/knn_port.c:port_synth_value and
// oracle/oracle.py:synth -- sum of four 16-bit uniforms (exact integer arithmetic) times one fp32 constant, sigma = 0.25
// like the reference's own test generator N(0, 0.25) (cpp_src/gtests/tools.h:120-129).
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
	z += 0x9E3779B97F4A7C15ull;
	z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
	z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
	return z ^ (z >> 31);
}
__host__ __device__ __forceinline__ float synth_value(uint64_t seed, uint64_t index) {
	const uint64_t h = mix64(seed ^ (index * 0xD1342543DE82EF95ull));
	const int32_t s = int32_t(h & 0xFFFF) + int32_t((h >> 16) & 0xFFFF) + int32_t((h >> 32) & 0xFFFF) + int32_t(h >> 48);
	return float(s - 131070) * 6.6072488e-06f;
}

// ---------------------------------------------------------------------------------------------------------------------
// Result keys.  A candidate is one u64 so that "better" is a single unsigned compare:
//   scan mode : key = ord(dist) << 32 | internal_row   -> total order (distance, internal row index)
//   tie  mode : key = internal_row << 32 | ord(dist)   -> internal order among rows with dist <= dstar
// ord() is the usual order-preserving float -> u32 map; -0.0 is canonicalised to +0.0 first so that it ties with +0.0 the
// way the reference's float compare does.
constexpr uint64_t kKeyNone = ~0ull;

__host__ __device__ __forceinline__ uint32_t float_ord(float f) {
	f += 0.0f;
#ifdef __CUDA_ARCH__
	uint32_t u = __float_as_uint(f);
#else
	union {
		float f;
		uint32_t u;
	} c{f};
	uint32_t u = c.u;
#endif
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float ord_float(uint32_t o) {
	const uint32_t u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
#ifdef __CUDA_ARCH__
	return __uint_as_float(u);
#else
	union {
		uint32_t u;
		float f;
	} c{u};
	return c.f;
#endif
}
__host__ __device__ __forceinline__ uint64_t make_key(float dist, uint32_t row) { return (uint64_t(float_ord(dist)) << 32) | row; }
// the distance of a key.  Keys hold a zero distance as +0, but the exact arithmetic gives -(+0) = -0 for an inner-product or cosine row
// whose dot product is zero -- as the reference's DistCalculator::ip does -- and +0 for L2: neg_zero (metric != L2) restores the sign
__host__ __device__ __forceinline__ float key_dist(uint32_t o, bool neg_zero) {
	const float f = ord_float(o);
	return neg_zero && f == 0.f ? -0.f : f;
}

enum Metric : int { kL2 = 0, kIP = 1, kCos = 2 };
enum ScanMode : int { kModeTopK = 0, kModeTieRows = 1 };

}  // namespace rxgpu
