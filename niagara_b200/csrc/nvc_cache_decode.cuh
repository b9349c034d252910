// nvc_cache_decode.cuh — device decoders of a compressed scene cache's vertex and meshlet streams, for
// nvc_scene_cache_read_device (nvc_scene_cache_device.cpp).  Their outputs equal the host decoders'
// (nvc_meshopt_decode.cpp, nvc_scene_cache.cpp) byte for byte; the formats are in nvc_meshopt_format.h.
//
// Vertex codec (VERTICES, stride 16; MESHLETVTX0, stride 8).  The host walk (walk_vertex_stream) has already checked the
// whole stream and found every block's and every byte plane's start, so nothing here can fail.  Three launches:
//   blocks   one warp per block of 256 vertices: stage the block's bytes in shared memory; one lane per plane finds its
//            groups' offsets from the selectors and the escape counts (nvc_meshopt_format.h); one lane per (plane, group)
//            unpacks; then per 4-byte column a warp scan of the delta terms with the previous vertex taken as 0.  The
//            block's words go out coalesced; its last vertex's words are the block's totals.
//   carry    one CTA per column: exclusive scan of the block totals from the baseline vertex (the column's channel fixes
//            the combination for the whole stream, and each is an abelian group, so the scan is exact).
//   apply    every output word combined with its block's carry.
// Meshlet codec (MESHLETDATA).  Each block is a serial chain (triangle history, unseen counter, explicit-byte cursor), so
// one lane decodes one meshlet.  A warp takes the 32 meshlets after one checkpoint of the host's index: their blocks are
// adjacent in the stream and are staged in shared memory as one coalesced span when it fits (the reference's 64 / 96
// meshlets take about 5 KB), else read where they lie.  Each lane runs the host reader's block decoder
// (mcodec::decode_block), bounded by the block's own extent from the size chain; a malformed block raises a flag
// (NVC_ERROR_CORRUPT).  Outputs are whole words: the host index admits only caches whose meshlets' word ranges do not
// overlap, so a meshlet owns its words, and the zero bytes a word holds past the meshlet's last reference or triangle
// are what the host's zero fill leaves there.
#pragma once

#include "nvc_internal.h"
#include "nvc_meshopt_format.h"
#include "nvc_scan.cuh"

namespace nvc
{
namespace cache
{

constexpr uint32_t kVertexBlock = 256; // vcodec::block_vertices of strides 8 and 16
constexpr uint32_t kVertexWarps = 4;
constexpr uint32_t kCarryThreads = 1024;
constexpr uint32_t kApplyThreads = 256;
constexpr uint32_t kMeshletWarps = 4;
constexpr uint32_t kMeshletStageWords = 2048; // 8 KB per warp

// Shared memory of one warp of the block kernel.  span: the most bytes one block of stride S can span (its control bytes,
// then per plane the selector header and 16 groups of at most 24 bytes: 4-bit fields that are all escaped).  words: that
// span staged from a word boundary; later the block's decoded words, padded by one word per 8 vertices so that the lanes'
// stores (8 consecutive vertices each) fall into distinct banks.
template <uint32_t S>
struct VertexStage
{
	static constexpr uint32_t span = S / 4 + S * (4 + 16 * 24);
	static constexpr uint32_t staged = (span + 3 + 3) / 4, decoded = kVertexBlock * S / 4 + 32;
	static constexpr uint32_t words = staged > decoded ? staged : decoded;
};

// v[k] by selects: a dynamic index into a kernel parameter array would copy the array to the stack
__device__ __forceinline__ uint32_t column_value(const uint32_t (&v)[4], uint32_t k)
{
	return k == 0 ? v[0] : k == 1 ? v[1] : k == 2 ? v[2] : v[3];
}

// vcodec::combine of one column's channel, as a scan operation
struct Combine
{
	uint32_t channel;
	__device__ __forceinline__ uint32_t operator()(uint32_t x, uint32_t y) const { return vcodec::combine(x, y, channel); }
};

__device__ __forceinline__ uint32_t padded_word(uint32_t vertex, uint32_t column, uint32_t columns)
{
	return vertex * columns + column + vertex / 8u;
}

template <uint32_t S>
__global__ void __launch_bounds__(kVertexWarps * 32) decode_vertex_blocks_kernel(const VertexDecodeArgs a)
{
	constexpr uint32_t C = S / 4;
	__shared__ uint32_t s_stage[kVertexWarps][VertexStage<S>::words];
	__shared__ __align__(8) uint8_t s_planes[kVertexWarps][S * kVertexBlock];
	__shared__ uint16_t s_group[kVertexWarps][S * 16];
	__shared__ uint16_t s_plane[kVertexWarps][S];
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	const uint32_t b = blockIdx.x * kVertexWarps + warp;
	if (b >= a.blocks)
		return; // whole warps
	const uint32_t first = b * kVertexBlock;
	const uint32_t n = min(a.vertex_count - first, kVertexBlock), groups = (n + 15u) / 16u;
	uint32_t* stage = s_stage[warp];
	uint8_t* planes = s_planes[warp];
	uint16_t* group = s_group[warp];

	const uint32_t start = a.block_start[b], end = a.block_start[b + 1];
	const uint32_t* src = reinterpret_cast<const uint32_t*>(a.stream) + start / 4u;
	const uint32_t words = end / 4u + ((end & 3u) != 0) - start / 4u; // no wrap for offsets near 2^32
	for (uint32_t i = lane; i < words; i += 32)
		stage[i] = __ldg(src + i);
	__syncwarp();
	const uint8_t* block = reinterpret_cast<const uint8_t*>(stage) + (start & 3u);

	// each plane's control (v1: 2 bits per plane in the block's leading bytes) and its groups' offsets in the block
	if (lane < S)
	{
		const uint32_t p0 = a.plane_offset[size_t(b) * S + lane];
		s_plane[warp][lane] = uint16_t(p0);
		const int control = a.version ? int((block[lane / 4] >> ((lane % 4) * 2)) & 3u) : 0;
		if (control < 2)
		{
			uint32_t at = p0 + vcodec::selector_bytes(groups);
			for (uint32_t g = 0; g < groups; ++g)
			{
				group[lane * 16 + g] = uint16_t(at);
				at += vcodec::group_bytes(block + at, vcodec::group_width(a.version, control, (block[p0 + g / 4] >> ((g % 4) * 2)) & 3u));
			}
		}
	}
	__syncwarp();

	// unpack: one lane per (plane, group of 16 values)
	for (uint32_t item = lane; item < S * 16; item += 32)
	{
		const uint32_t q = item >> 4, g = item & 15u;
		if (g >= groups)
			continue;
		const uint32_t p0 = s_plane[warp][q];
		const int control = a.version ? int((block[q / 4] >> ((q % 4) * 2)) & 3u) : 0;
		uint8_t* out = planes + q * kVertexBlock + g * 16;
		if (control == 3)
			for (uint32_t i = 0; i < 16; ++i)
				out[i] = g * 16 + i < n ? block[p0 + g * 16 + i] : 0;
		else if (control == 2)
			for (uint32_t i = 0; i < 16; ++i)
				out[i] = 0;
		else
		{
			const int width = vcodec::group_width(a.version, control, (block[p0 + g / 4] >> ((g % 4) * 2)) & 3u);
			const uint8_t* bytes = block + group[q * 16 + g];
			if (width == 0 || width == 8)
				for (uint32_t i = 0; i < 16; ++i)
					out[i] = width ? bytes[i] : 0;
			else
				vcodec::unpack_group(bytes, width, out);
		}
	}
	__syncwarp();

	// deltas per column, the previous vertex taken as 0: lane l owns vertices 8 l .. 8 l + 7 (the staged bytes are dead now)
	uint32_t* decoded = stage;
	for (uint32_t k = 0; k < C; ++k)
	{
		const uint32_t channel = column_value(a.channel, k);
		uint2 pl[4];
		for (uint32_t j = 0; j < 4; ++j)
			pl[j] = *reinterpret_cast<const uint2*>(planes + (4 * k + j) * kVertexBlock + lane * 8);
		uint32_t v[8], acc = 0;
		for (uint32_t t = 0; t < 8; ++t)
		{
			const uint32_t sh = (t & 3u) * 8u;
			uint32_t bytes4 = 0;
			for (uint32_t j = 0; j < 4; ++j)
				bytes4 |= (((t < 4 ? pl[j].x : pl[j].y) >> sh) & 255u) << (8 * j);
			acc = vcodec::combine(acc, vcodec::delta_term(bytes4, channel), channel);
			v[t] = acc;
		}
		const uint32_t before = scan::warp_exclusive(acc, lane, Combine{ channel });
		for (uint32_t t = 0; t < 8; ++t)
		{
			const uint32_t i = lane * 8 + t;
			const uint32_t value = vcodec::combine(before, v[t], channel);
			decoded[padded_word(i, k, C)] = value;
			if (i == n - 1)
				a.carry[size_t(b) * C + k] = value;
		}
	}
	__syncwarp();
	uint32_t* dst = a.out + size_t(first) * C;
	for (uint32_t w = lane; w < n * C; w += 32)
		dst[w] = decoded[w + (w / C) / 8u];
}

// carry[b][k] = baseline[k] combined with the totals of blocks 0 .. b-1 (in place)
template <uint32_t C>
__global__ void __launch_bounds__(kCarryThreads) decode_vertex_carry_kernel(const VertexDecodeArgs a)
{
	__shared__ uint32_t s_warp[kCarryThreads / 32];
	const uint32_t k = blockIdx.x, channel = column_value(a.channel, k);
	uint32_t* carry = a.carry + k;
	scan::scan_tiles<kCarryThreads>(
	    a.blocks, column_value(a.baseline, k), s_warp, [&](uint32_t b) { return carry[size_t(b) * C]; }, [&](uint32_t b, uint32_t v) { carry[size_t(b) * C] = v; },
	    Combine{ channel });
}

template <uint32_t C>
__global__ void __launch_bounds__(kApplyThreads) decode_vertex_apply_kernel(const VertexDecodeArgs a)
{
	const size_t words = size_t(a.vertex_count) * C;
	const size_t step = size_t(gridDim.x) * kApplyThreads; // a multiple of C: a thread keeps its column
	const size_t w0 = size_t(blockIdx.x) * kApplyThreads + threadIdx.x;
	const uint32_t k = uint32_t(w0 % C), channel = column_value(a.channel, k);
	for (size_t w = w0; w < words; w += step)
		a.out[w] = vcodec::combine(a.carry[w / C / kVertexBlock * C + k], a.out[w], channel);
}

// Where mcodec::decode_block puts a meshlet's outputs on the device: whole words from `out` on, the references one per
// word or, with shortRefs, two per word, then the triangles' index bytes.  `word` holds the `filled` bytes decoded since
// the last store.
struct MeshletWordWriter
{
	uint32_t* out;
	bool short_refs;
	uint32_t word = 0, filled = 0;
	__device__ __forceinline__ void put(uint32_t value, uint32_t bytes)
	{
		word |= value << (8 * filled);
		filled += bytes;
		if (filled == 4)
			flush();
	}
	__device__ __forceinline__ void reference(uint32_t, uint32_t value)
	{
		if (short_refs)
			put(value & 0xffffu, 2);
		else
			*out++ = value;
	}
	__device__ __forceinline__ void triangle(uint32_t, uint32_t a, uint32_t b, uint32_t c)
	{
		put(a, 1);
		put(b, 1);
		put(c, 1);
	}
	__device__ __forceinline__ void flush()
	{
		if (filled)
			*out++ = word;
		word = 0;
		filled = 0;
	}
};

__global__ void __launch_bounds__(kMeshletWarps * 32) decode_meshlets_kernel(const MeshletDecodeArgs a)
{
	__shared__ uint32_t s_stage[kMeshletWarps][kMeshletStageWords];
	__shared__ uint32_t s_at[kMeshletWarps][32];
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	const uint32_t g = blockIdx.x * kMeshletWarps + warp, first = g * 32u;
	if (first >= a.meshlet_count)
		return; // whole warps
	const uint32_t m = min(a.meshlet_count - first, 32u);
	const uint32_t start = a.checkpoints[g], end = a.checkpoints[g + 1];
	const uint32_t words = end / 4u + ((end & 3u) != 0) - start / 4u; // no wrap for offsets near 2^32
	const uint8_t* span = a.stream + start;
	if (words <= kMeshletStageWords)
	{
		const uint32_t* src = reinterpret_cast<const uint32_t*>(a.stream) + start / 4u;
		for (uint32_t i = lane; i < words; i += 32)
			s_stage[warp][i] = __ldg(src + i);
		span = reinterpret_cast<const uint8_t*>(s_stage[warp]) + (start & 3u);
	}
	__syncwarp();
	// the size chain of the group (the host walk checked that it adds up to the section's size)
	if (lane == 0)
		for (uint32_t i = 0, at = 0; i < m; ++i)
		{
			s_at[warp][i] = at;
			at += 2u + (uint32_t(span[at]) | (uint32_t(span[at + 1]) << 8));
		}
	__syncwarp();
	if (lane >= m)
		return;
	const uint32_t at = s_at[warp][lane];
	const uint32_t size = uint32_t(span[at]) | (uint32_t(span[at + 1]) << 8);
	const uint2 r = __ldg(reinterpret_cast<const uint2*>(a.records) + first + lane);
	MeshletWordWriter out = { a.out + r.x, ((r.y >> 16) & 1u) != 0 };
	if (!mcodec::decode_block(span + at + 2, size, r.y & 255u, (r.y >> 8) & 255u, out))
		atomicOr(a.corrupt, 1u);
}

// Index codec (INDICES).  The decoder's state is small: a 16-slot vertex ring, two 16-slot edge rings pushed together,
// `next` and `last`.  A chunk of kIndexChunk triangles changes it by a substitution that does not depend on the entry
// state: each exit slot, and the exit `next` and `last`, is a constant, entry next + k, entry last + k, or one named entry
// slot (icodec::decode_triangle copies values between slots and only ever adds to `next` and `last`), and each ring's
// head advances by a count the codes fix.  Substitutions compose associatively, so:
//   symbolic  one thread per chunk runs the decoder's step from a symbolic entry state (slot j holds "entry slot j",
//             next "entry next + 0", ...) and stores the chunk's substitution.  The host walk (walk_index_stream) has
//             found where each chunk's data bytes start and checked the whole stream, so nothing here can fail.
//   scan      an exclusive scan of the substitutions from the decoder's initial state (every slot 0xffffffff, next = last
//             = 0), in three launches: one warp per run of kIndexRun chunks composes their total; one warp scans the run
//             totals; one warp per run scans its chunks from the run's entry state.  A warp holds a substitution as
//             kIndexEntries words over its lanes and composes with shuffles.  The result is each chunk's entry state.
//   concrete  one thread per chunk decodes it again from its true entry state; a warp stages kIndexBatch triangles per
//             lane in shared memory and stores each lane's run of indices as one coalesced span.
// Rings are kept as the host decoder keeps them, physical slots and a head, including the slot a FIFO hit writes without
// advancing; a substitution's slots are named relative to the heads at its entry.  The exact serial decoder's state is
// reproduced at every chunk's entry.  Symbolic values are uint2 { tag, k }: tag < 48 names an entry slot (vertex ring 0 ..
// 15, edge ring a 16 .. 31, edge ring b 32 .. 47), kTagNext / kTagLast entry next / last + k, kTagConst the constant k.
// Word kIndexEntries - 1 of a substitution holds its head advances { vertex, edge }.
constexpr uint32_t kIndexThreads = 64;
constexpr uint32_t kIndexBatch = 8;                         // triangles a lane stages between coalesced stores
constexpr uint32_t kIndexStageStride = kIndexBatch * 3 + 1; // words per lane, odd: the lanes' staging stores miss each other's banks
constexpr uint32_t kIndexScanWarps = 4;
constexpr uint32_t kTagNext = 48, kTagLast = 49, kTagConst = 50;

__device__ __forceinline__ uint32_t index_add(uint32_t v, uint32_t k)
{
	return v + k;
}

__device__ __forceinline__ uint2 index_add(uint2 v, uint32_t k)
{
	return make_uint2(v.x, v.y + k);
}

// The decoder's state for icodec::decode_triangle with its rings in shared memory: slot j of this thread's 48 at
// ring[j * kIndexThreads] (the threads of a warp always touch distinct banks)
template <typename V>
struct SharedIndexState
{
	using Value = V;
	V* ring;
	uint32_t vhead, ehead;
	V next, last;
	__device__ __forceinline__ static V add(V v, uint32_t k) { return index_add(v, k); }
	__device__ __forceinline__ static V zero() { return index_add(V(), 0u) ; }
	__device__ __forceinline__ V vert(uint32_t n) const { return ring[((vhead - n) & 15u) * kIndexThreads]; }
	__device__ __forceinline__ V edge_a(uint32_t n) const { return ring[(16u + ((ehead - n) & 15u)) * kIndexThreads]; }
	__device__ __forceinline__ V edge_b(uint32_t n) const { return ring[(32u + ((ehead - n) & 15u)) * kIndexThreads]; }
	__device__ __forceinline__ void put_vert(V v, bool advance)
	{
		ring[vhead * kIndexThreads] = v;
		vhead = (vhead + (advance ? 1u : 0u)) & 15u;
	}
	__device__ __forceinline__ void put_edge(V a, V b)
	{
		ring[(16u + ehead) * kIndexThreads] = a;
		ring[(32u + ehead) * kIndexThreads] = b;
		ehead = (ehead + 1u) & 15u;
	}
};

template <>
__device__ __forceinline__ uint2 SharedIndexState<uint2>::zero()
{
	return make_uint2(kTagConst, 0u);
}

// a chunk's data bytes, where the host walk found them
struct IndexBytes
{
	const uint8_t* at;
	__device__ __forceinline__ bool next(uint32_t& b)
	{
		b = __ldg(at++);
		return true;
	}
};

// the 16-byte aux table into shared memory, before any thread returns
__device__ __forceinline__ void load_index_aux(const IndexDecodeArgs& a, uint8_t* s_aux)
{
	if (threadIdx.x < 16)
		s_aux[threadIdx.x] = __ldg(a.stream + a.aux_offset + threadIdx.x);
	__syncthreads();
}

template <typename V>
// triangles first .. first + count - 1 of chunk c; stage (when not null) receives their corners from stage[0] on
__device__ __forceinline__ void decode_index_chunk(SharedIndexState<V>& s, const IndexDecodeArgs& a, const uint8_t* aux, uint32_t c, uint32_t first, uint32_t count,
    IndexBytes& data, V* stage)
{
	for (uint32_t t = first; t < first + count; ++t)
	{
		V corner[3];
		icodec::decode_triangle(s, __ldg(a.stream + 1 + size_t(c) * kIndexChunk + t), aux, a.direct_slots, data, corner);
		if (stage)
			for (uint32_t j = 0; j < 3; ++j)
				stage[(t - first) * 3 + j] = corner[j];
	}
}

__global__ void __launch_bounds__(kIndexThreads) decode_index_symbolic_kernel(const IndexDecodeArgs a)
{
	__shared__ uint2 s_ring[48 * kIndexThreads];
	__shared__ uint8_t s_aux[16];
	load_index_aux(a, s_aux);
	const uint32_t c = blockIdx.x * kIndexThreads + threadIdx.x;
	if (c >= a.chunks)
		return;
	SharedIndexState<uint2> s = { s_ring + threadIdx.x, 0u, 0u, make_uint2(kTagNext, 0u), make_uint2(kTagLast, 0u) };
	for (uint32_t j = 0; j < 48; ++j)
		s.ring[j * kIndexThreads] = make_uint2(j, 0u);
	IndexBytes data = { a.stream + a.chunk_data[c] };
	decode_index_chunk<uint2>(s, a, s_aux, c, 0, min(kIndexChunk, a.triangles - c * kIndexChunk), data, nullptr);
	for (uint32_t j = 0; j < 48; ++j)
		a.sub[size_t(j) * a.chunks + c] = s.ring[j * kIndexThreads];
	a.sub[size_t(48) * a.chunks + c] = s.next;
	a.sub[size_t(49) * a.chunks + c] = s.last;
	a.sub[size_t(50) * a.chunks + c] = make_uint2(s.vhead, s.ehead);
}

__device__ __forceinline__ uint2 shfl2(uint2 v, uint32_t src)
{
	return make_uint2(__shfl_sync(0xffffffffu, v.x, src), __shfl_sync(0xffffffffu, v.y, src));
}

// A substitution held by a warp: entry `lane` in lo, entry 32 + lane in hi (lanes 0 .. 17), the head advances in heads
struct IndexSub
{
	uint2 lo, hi, heads;
};

__device__ __forceinline__ IndexSub load_index_sub(const uint2* buf, size_t n, size_t i)
{
	const uint32_t lane = threadIdx.x & 31u;
	IndexSub s;
	s.lo = buf[lane * n + i];
	s.hi = lane < 18 ? buf[(32 + lane) * n + i] : make_uint2(kTagConst, 0u);
	// lane 0 alone reads and writes the heads word, so that a warp that overwrites substitutions with entry states in
	// place never reads a word another lane has written
	const uint2 h = lane == 0 ? buf[size_t(kIndexEntries - 1) * n + i] : make_uint2(0u, 0u);
	s.heads = shfl2(h, 0);
	return s;
}

__device__ __forceinline__ void store_index_sub(uint2* buf, size_t n, size_t i, const IndexSub& s)
{
	const uint32_t lane = threadIdx.x & 31u;
	buf[lane * n + i] = s.lo;
	if (lane < 18)
		buf[(32 + lane) * n + i] = s.hi;
	if (lane == 0)
		buf[size_t(kIndexEntries - 1) * n + i] = s.heads;
}

// b's value v, whose tags name slots at b's entry = a's exit, in terms of a's entry
__device__ __forceinline__ uint2 resolve_index_value(const IndexSub& a, uint2 v)
{
	const uint32_t src = v.x < 16 ? (a.heads.x + v.x) & 15u : v.x < 48 ? (v.x & 48u) + ((a.heads.y + v.x) & 15u) : v.x;
	const uint2 lo = shfl2(a.lo, src & 31u), hi = shfl2(a.hi, src & 31u);
	const uint2 r = src < 32 ? lo : hi;
	return v.x >= kTagConst ? v : make_uint2(r.x, r.y + v.y);
}

// a then b.  b's exit slot j is a's exit-relative slot j, the slot (j - a's advance) relative to a's entry heads
__device__ __forceinline__ IndexSub compose_index(const IndexSub& a, const IndexSub& b)
{
	const uint32_t lane = threadIdx.x & 31u;
	const uint2 lo = shfl2(b.lo, (lane & 16u) | ((lane - (lane < 16 ? a.heads.x : a.heads.y)) & 15u));
	const uint2 hi = shfl2(b.hi, lane < 16 ? (lane - a.heads.y) & 15u : lane);
	IndexSub r;
	r.lo = resolve_index_value(a, lo);
	r.hi = resolve_index_value(a, hi);
	r.heads = make_uint2((a.heads.x + b.heads.x) & 15u, (a.heads.y + b.heads.y) & 15u);
	return r;
}

// the substitution that changes nothing, and the decoder's initial state as one (every value constant)
__device__ __forceinline__ IndexSub identity_index_sub()
{
	const uint32_t lane = threadIdx.x & 31u;
	return { make_uint2(lane, 0u), make_uint2(32u + lane, 0u), make_uint2(0u, 0u) };
}

__device__ __forceinline__ IndexSub initial_index_state()
{
	const uint32_t lane = threadIdx.x & 31u;
	return { make_uint2(kTagConst, 0xffffffffu), make_uint2(kTagConst, lane < 16 ? 0xffffffffu : 0u), make_uint2(0u, 0u) };
}

// kPrefix false: each run's total into a.run.  kPrefix true: from each run's entry state (a.run), each chunk's entry
// state over its substitution in a.sub.  One warp per run, the next chunk's substitution loaded while one is composed.
template <bool kPrefix>
__global__ void __launch_bounds__(kIndexScanWarps * 32) decode_index_scan_kernel(const IndexDecodeArgs a)
{
	const uint32_t r = blockIdx.x * kIndexScanWarps + (threadIdx.x >> 5);
	if (r >= a.runs)
		return; // whole warps
	const uint32_t first = r * kIndexRun, end = min(first + kIndexRun, a.chunks);
	IndexSub acc = kPrefix ? load_index_sub(a.run, a.runs, r) : identity_index_sub();
	IndexSub b = load_index_sub(a.sub, a.chunks, first);
	for (uint32_t c = first; c < end; ++c)
	{
		const IndexSub next = c + 1 < end ? load_index_sub(a.sub, a.chunks, c + 1) : b;
		if (kPrefix)
			store_index_sub(a.sub, a.chunks, c, acc);
		acc = compose_index(acc, b);
		b = next;
	}
	if (!kPrefix)
		store_index_sub(a.run, a.runs, r, acc);
}

// one warp: the runs' totals in a.run become their entry states
__global__ void __launch_bounds__(32) decode_index_runs_kernel(const IndexDecodeArgs a)
{
	IndexSub acc = initial_index_state();
	IndexSub b = load_index_sub(a.run, a.runs, 0);
	for (uint32_t r = 0; r < a.runs; ++r)
	{
		const IndexSub next = r + 1 < a.runs ? load_index_sub(a.run, a.runs, r + 1) : b;
		store_index_sub(a.run, a.runs, r, acc);
		acc = compose_index(acc, b);
		b = next;
	}
}

__global__ void __launch_bounds__(kIndexThreads) decode_index_concrete_kernel(const IndexDecodeArgs a)
{
	__shared__ uint32_t s_ring[48 * kIndexThreads];
	__shared__ uint32_t s_stage[kIndexThreads / 32][32 * kIndexStageStride];
	__shared__ uint8_t s_aux[16];
	load_index_aux(a, s_aux);
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	const uint32_t warp_first = blockIdx.x * kIndexThreads + warp * 32u, c = warp_first + lane;
	if (warp_first >= a.chunks)
		return; // whole warps
	const bool active = c < a.chunks;
	const uint32_t count = active ? min(kIndexChunk, a.triangles - c * kIndexChunk) : 0u;
	SharedIndexState<uint32_t> s = { s_ring + threadIdx.x, 0u, 0u, 0u, 0u };
	IndexBytes data = { a.stream };
	if (active)
	{
		for (uint32_t j = 0; j < 48; ++j)
			s.ring[j * kIndexThreads] = a.sub[size_t(j) * a.chunks + c].y;
		s.next = a.sub[size_t(48) * a.chunks + c].y;
		s.last = a.sub[size_t(49) * a.chunks + c].y;
		const uint2 heads = a.sub[size_t(50) * a.chunks + c];
		s.vhead = heads.x;
		s.ehead = heads.y;
		data.at = a.stream + a.chunk_data[c];
	}
	uint32_t* stage = s_stage[warp];
	for (uint32_t b = 0; b < kIndexChunk; b += kIndexBatch)
	{
		const uint32_t n = count > b ? min(kIndexBatch, count - b) : 0u;
		decode_index_chunk<uint32_t>(s, a, s_aux, c, b, n, data, stage + lane * kIndexStageStride);
		__syncwarp();
		for (uint32_t l = 0; l < 32; ++l)
		{
			const uint32_t cl = warp_first + l;
			const uint32_t nl = cl < a.chunks ? min(kIndexChunk, a.triangles - cl * kIndexChunk) : 0u;
			const uint32_t words = nl > b ? min(kIndexBatch, nl - b) * 3u : 0u;
			if (lane < words)
				a.out[(size_t(cl) * kIndexChunk + b) * 3 + lane] = stage[l * kIndexStageStride + lane];
		}
		__syncwarp();
	}
}

} // namespace cache
} // namespace nvc
