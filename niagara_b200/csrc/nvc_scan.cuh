// nvc_scan.cuh — the scan and search primitives of the load-time kernels (scene-cache codecs, mesh cookers, OBJ loader).
//   warp_inclusive / warp_exclusive   one warp
//   block_exclusive / block_sum       one CTA, one value per thread
//   scan_tiles                        one CTA over n values, THREADS at a time, with a running carry between tiles
//   offsets_kernel                    one CTA per row: 32-bit sizes into 64-bit offsets, the total at offsets[n]
//   reduce_kernel / apply_kernel      the device-wide scan, with offsets_kernel between them (launch_scan in
//                                     nvc_kernels.cu): per-block sums of kScanItems values, their offsets, then each block
//                                     scanned from its offset; out[n] = the total
//   last_at_most                      binary search over a non-decreasing key
// Every scan is exclusive and sums 32-bit values within a CTA.  An operation is applied as op(earlier, later), so it need
// not be commutative, and 0 must be its identity (vcodec::combine's channels are abelian groups with identity 0).  Nothing
// waits on another CTA, so the kernels run as they are under the SIMT emulation (tests/cuda_emu) too.
#pragma once

#include "nvc_internal.h"

namespace nvc
{
namespace scan
{

constexpr uint32_t kFull = 0xffffffffu;
constexpr uint32_t kOffsetsThreads = 1024; // the CTA of offsets_kernel
constexpr uint32_t kThreads = 256;         // the CTAs of reduce_kernel and apply_kernel
constexpr uint32_t kPerThread = kScanItems / kThreads;

struct Plus
{
	template <typename A, typename B>
	__device__ __forceinline__ A operator()(A a, B b) const
	{
		return a + b;
	}
};

template <typename Op = Plus>
__device__ __forceinline__ uint32_t warp_inclusive(uint32_t v, uint32_t lane, Op op = {})
{
	for (uint32_t d = 1; d < 32; d <<= 1)
	{
		const uint32_t y = __shfl_up_sync(kFull, v, d);
		if (lane >= d)
			v = op(y, v);
	}
	return v;
}

template <typename Op = Plus>
__device__ __forceinline__ uint32_t warp_exclusive(uint32_t v, uint32_t lane, Op op = {})
{
	const uint32_t before = __shfl_up_sync(kFull, warp_inclusive(v, lane, op), 1);
	return lane ? before : 0u;
}

// the exclusive scan of v over a CTA of THREADS threads, and the CTA's total; s_warp holds THREADS / 32 words and may be
// reused as soon as this returns
template <uint32_t THREADS, typename Op = Plus>
__device__ __forceinline__ uint32_t block_exclusive(uint32_t v, uint32_t* s_warp, uint32_t& total, Op op = {})
{
	constexpr uint32_t W = THREADS / 32;
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	const uint32_t incl = warp_inclusive(v, lane, op);
	if (lane == 31)
		s_warp[warp] = incl;
	__syncthreads();
	if (warp == 0)
	{
		const uint32_t w = warp_inclusive(lane < W ? s_warp[lane] : 0u, lane, op);
		if (lane < W)
			s_warp[lane] = w;
	}
	__syncthreads();
	uint32_t before = __shfl_up_sync(kFull, incl, 1);
	if (lane == 0)
		before = 0;
	if (warp)
		before = op(s_warp[warp - 1], before);
	total = s_warp[W - 1];
	__syncthreads();
	return before;
}

// the sum of v over a CTA of THREADS threads, in thread 0; s_warp holds THREADS / 32 words
template <uint32_t THREADS>
__device__ __forceinline__ uint32_t block_sum(uint32_t v, uint32_t* s_warp)
{
	for (uint32_t d = 16; d > 0; d >>= 1)
		v += __shfl_down_sync(kFull, v, d);
	if ((threadIdx.x & 31u) == 0)
		s_warp[threadIdx.x >> 5] = v;
	__syncthreads();
	uint32_t total = 0;
	if (threadIdx.x == 0)
		for (uint32_t w = 0; w < THREADS / 32; ++w)
			total += s_warp[w];
	return total;
}

// One CTA of THREADS threads over value(i), i < n, one tile of THREADS values at a time: emit(i, op(running, the tile's
// values before i)), then running = op(running, the tile's total).  Returns the last running value.  Each tile sums in 32
// bits; `running` keeps the caller's width.
template <uint32_t THREADS, typename Carry, typename Value, typename Emit, typename Op = Plus>
__device__ __forceinline__ Carry scan_tiles(uint32_t n, Carry running, uint32_t* s_warp, const Value& value, const Emit& emit, Op op = {})
{
	for (uint32_t base = 0; base < n; base += THREADS)
	{
		const uint32_t i = base + threadIdx.x;
		uint32_t total;
		const uint32_t before = block_exclusive<THREADS>(i < n ? value(i) : 0u, s_warp, total, op);
		if (i < n)
			emit(i, op(running, before));
		running = op(running, total);
	}
	return running;
}

// One CTA per row: offsets[i] = the sum of sizes[0, i) and offsets[n] = the total, in 64 bits; row r reads sizes + r n and
// writes offsets + r (n + 1).  The sizes of one tile of kOffsetsThreads add up to less than 2^32 (each is a block's or an
// item's bytes or count).
__global__ void __launch_bounds__(kOffsetsThreads) offsets_kernel(const uint32_t* sizes, uint32_t n, unsigned long long* offsets)
{
	__shared__ uint32_t s_warp[kOffsetsThreads / 32];
	sizes += size_t(blockIdx.x) * n;
	offsets += size_t(blockIdx.x) * (size_t(n) + 1);
	const unsigned long long total = scan_tiles<kOffsetsThreads>(
	    n, 0ull, s_warp, [&](uint32_t i) { return sizes[i]; }, [&](uint32_t i, unsigned long long v) { offsets[i] = v; });
	if (threadIdx.x == 0)
		offsets[n] = total;
}

// ---- the device-wide scan of row blockIdx.y of `in` (n values per row), in blocks of kScanItems ----------------------------

// block_sums[row][block] = the block's sum
template <typename In>
__global__ void __launch_bounds__(kThreads) reduce_kernel(const In* in, uint64_t n, uint32_t* block_sums)
{
	__shared__ uint32_t s_warp[kThreads / 32];
	in += blockIdx.y * n;
	const uint64_t first = uint64_t(blockIdx.x) * kScanItems + uint64_t(threadIdx.x) * kPerThread;
	uint32_t sum = 0;
	for (uint32_t k = 0; k < kPerThread; ++k)
		sum += first + k < n ? in[first + k] : 0u;
	const uint32_t total = block_sum<kThreads>(sum, s_warp);
	if (threadIdx.x == 0)
		block_sums[uint64_t(blockIdx.y) * gridDim.x + blockIdx.x] = total;
}

// out[row][i] = the block's offset + the values before i in its block; out[row][n] = the row's total
template <typename In, typename Out>
__global__ void __launch_bounds__(kThreads) apply_kernel(const In* in, uint64_t n, const unsigned long long* offsets, Out* out)
{
	__shared__ uint32_t s_warp[kThreads / 32];
	in += blockIdx.y * n;
	offsets += blockIdx.y * (uint64_t(gridDim.x) + 1);
	out += blockIdx.y * (n + 1);
	const uint64_t first = uint64_t(blockIdx.x) * kScanItems + uint64_t(threadIdx.x) * kPerThread;
	In v[kPerThread];
	uint32_t sum = 0;
	for (uint32_t k = 0; k < kPerThread; ++k)
	{
		v[k] = first + k < n ? in[first + k] : In(0);
		sum += v[k];
	}
	uint32_t total;
	Out before = Out(offsets[blockIdx.x]) + block_exclusive<kThreads>(sum, s_warp, total);
	for (uint32_t k = 0; k < kPerThread; ++k)
		if (first + k < n)
		{
			out[first + k] = before;
			before += v[k];
		}
	if (blockIdx.x == 0 && threadIdx.x == 0)
		out[n] = Out(offsets[gridDim.x]);
}

// the last i in [0, n) with key(i) <= x, for a non-decreasing key with key(0) <= x; 0 when n <= 1
template <typename X, typename Key>
__device__ __forceinline__ uint32_t last_at_most(uint32_t n, X x, const Key& key)
{
	uint32_t lo = 0, hi = n;
	while (hi - lo > 1)
	{
		const uint32_t mid = (lo + hi) >> 1;
		if (key(mid) <= x)
			lo = mid;
		else
			hi = mid;
	}
	return lo;
}

} // namespace scan
} // namespace nvc
