// nvc_cache_encode.cuh — device encoders of a compressed scene cache's vertex and meshlet streams, for
// nvc_scene_cache_write (nvc_scene_cache_write.cpp).  Their output equals, byte for byte, what saveSceneCache writes with
// meshoptimizer's encoders at the settings it uses (vertex codec v1 at level 2, meshlet codec behind a uint16 size).  The
// formats are in nvc_meshopt_format.h and nvc_meshopt_decode.cpp; this file restates only the encoder's choices.
//
// Vertex codec.  Both per-stream decisions are made from the input alone, so every 256-vertex block is encoded on its own:
//   estimate  per 4-byte column, the delta channel (0: per byte, 1: per 16 bits) whose byte planes need fewer bytes on every
//             third block (blocks 0, 3, 6, ...), each block's deltas taken from the input vertex before it (block 0: from
//             vertex 0), every group of 16 bytes counted at its best of the 1/2/4/8-bit widths; ties keep channel 0.  One
//             thread per (sampled block, group, column); the sums are integers, reduced in any order.
//   blocks    one warp per block, one lane per byte plane.  The block's vertices are staged in shared memory behind the
//             baseline (the input vertex before the block; block 0: vertex 0).  A lane takes its plane's deltas, picks the
//             plane's control (all zero: 2; else the cheaper of the {0,1,2,4} / {1,2,4,8} width tables, unless neither beats
//             `count` literal bytes: 3) and per group of 16 the width (the smallest size, scanning the table's last entry
//             first; an equal size switches to the width the previous group used, never away from literals).  Run twice:
//             the measure pass stores each block's size; after their scan (scan::offsets_kernel) the write pass stores the
//             block where it belongs, control bytes first, then the planes in order.  The write pass also stores the header byte and the
//             tail (zeros up to 24 bytes, vertex 0, the channel bytes).
// Meshlet codec.  One thread per meshlet, measure then write as above; a meshlet's record is its uint16 size, then the block
// mcodec::decode_block reads back: the reference deltas, the explicit triangle bytes, the zero gap, the reference control
// bytes and the triangle codes.  A meshlet whose words lie outside meshletdata or whose counts pass mcodec::kMaxVertices /
// kMaxTriangles is not read; it raises a flag that the host turns into NVC_ERROR_INVALID_ARGUMENT before anything reaches
// the caller's buffer.
#pragma once

#include "nvc_internal.h"
#include "nvc_meshopt_format.h"
#include "nvc_scan.cuh"

namespace nvc
{
namespace cache
{

constexpr uint32_t kEncodeWarps = 4;
constexpr uint32_t kEstimateThreads = 256;
constexpr uint32_t kMeshletEncodeThreads = 128;

// The delta byte of plane q for a vertex whose words are `cur`, after the vertex whose words are `prev` (C words each):
// channel 0 zigzags the byte's difference, channel 1 the difference of the 16-bit half holding it.
template <uint32_t C>
__device__ __forceinline__ uint32_t delta_byte(const uint32_t* cur, const uint32_t* prev, uint32_t q, uint32_t channel)
{
	const uint32_t a = cur[q / 4], b = prev[q / 4];
	if (channel == 0)
	{
		const uint32_t sh = (q & 3u) * 8u, d = ((a >> sh) - (b >> sh)) & 255u;
		return ((d << 1) ^ (0u - (d >> 7))) & 255u;
	}
	const uint32_t sh = (q & 2u) * 8u, d = ((a >> sh) - (b >> sh)) & 0xffffu;
	return ((((d << 1) ^ (0u - (d >> 15))) & 0xffffu) >> ((q & 1u) * 8u)) & 255u;
}

struct Group16
{
	uint32_t w[4]; // byte i of the group at w[i / 4] >> (i % 4 * 8)
	__device__ __forceinline__ uint32_t byte(uint32_t i) const
	{
		const uint32_t x = i < 4 ? w[0] : i < 8 ? w[1] : i < 12 ? w[2] : w[3];
		return (x >> ((i & 3u) * 8u)) & 255u;
	}
};

constexpr uint32_t kNoFit = 0xffffu; // width 0 for a group that is not all zero

// bytes a group of 16 takes at `bits` bits per value: the packed fields plus one escape byte per value >= 2^bits - 1
__device__ __forceinline__ uint32_t group_size(const Group16& g, int bits)
{
	if (bits == 0)
		return (g.w[0] | g.w[1] | g.w[2] | g.w[3]) ? kNoFit : 0u;
	if (bits == 8)
		return 16u;
	const uint32_t sentinel = (1u << bits) - 1u;
	uint32_t n = 2u * uint32_t(bits);
	for (uint32_t i = 0; i < 16; ++i)
		n += g.byte(i) >= sentinel;
	return n;
}

// v1 width tables from the control: 0 -> {0, 1, 2, 4}, 1 -> {1, 2, 4, 8}
__device__ __forceinline__ int table_bits(int control, int k)
{
	return vcodec::group_width(1, control, uint32_t(k));
}

// ---- vertex codec: channel estimate -----------------------------------------------------------------------------------
// items (sample, group, column) with the column fastest; the grid-stride step is a multiple of C, so a thread keeps its column
template <uint32_t S>
__global__ void __launch_bounds__(kEstimateThreads) encode_vertex_estimate_kernel(const VertexEncodeArgs a)
{
	constexpr uint32_t C = S / 4;
	const uint32_t samples = uint32_t((uint64_t(a.vertex_count) + 3u * kVertexBlockEncode - 1u) / (3u * kVertexBlockEncode)); // no wrap near 2^32
	const size_t items = size_t(samples) * 16u * C, step = size_t(gridDim.x) * kEstimateThreads;
	const uint32_t* words = reinterpret_cast<const uint32_t*>(a.vertices);
	uint32_t sum[2] = { 0, 0 };
	for (size_t item = size_t(blockIdx.x) * kEstimateThreads + threadIdx.x; item < items; item += step)
	{
		const uint32_t k = uint32_t(item % C), g = uint32_t(item / C % 16u), s = uint32_t(item / C / 16u);
		const uint32_t first = s * 3u * kVertexBlockEncode, n = min(a.vertex_count - first, kVertexBlockEncode);
		if (g * 16u >= n)
			continue;
		for (uint32_t channel = 0; channel < 2; ++channel)
			for (uint32_t j = 0; j < 4; ++j)
			{
				Group16 grp = { { 0, 0, 0, 0 } };
				for (uint32_t i = 0; i < 16; ++i)
				{
					const uint32_t v = first + g * 16u + i;
					if (v >= first + n)
						break;
					const uint32_t* cur = words + size_t(v) * C;
					const uint32_t* prev = words + size_t(v == first && first == 0 ? 0 : v - 1) * C;
					grp.w[i / 4] |= delta_byte<C>(cur + k, prev + k, j, channel) << ((i & 3u) * 8u);
				}
				uint32_t best = min(min(group_size(grp, 1), group_size(grp, 2)), min(group_size(grp, 4), 16u));
				sum[channel] += best;
			}
	}
	for (uint32_t d = C; d < 32; d <<= 1)
	{
		sum[0] += __shfl_xor_sync(0xffffffffu, sum[0], int(d));
		sum[1] += __shfl_xor_sync(0xffffffffu, sum[1], int(d));
	}
	const uint32_t lane = threadIdx.x & 31u;
	if (lane < C)
	{
		atomicAdd(a.estimate + 2 * lane, (unsigned long long)sum[0]);
		atomicAdd(a.estimate + 2 * lane + 1, (unsigned long long)sum[1]);
	}
}

// ---- vertex codec: blocks -----------------------------------------------------------------------------------------------
template <uint32_t C>
__device__ __forceinline__ uint32_t column_channel(const VertexEncodeArgs& a, uint32_t k)
{
	return a.estimate[2 * k + 1] < a.estimate[2 * k] ? 1u : 0u;
}

template <uint32_t S, bool Write>
__global__ void __launch_bounds__(kEncodeWarps * 32) encode_vertex_blocks_kernel(const VertexEncodeArgs a)
{
	constexpr uint32_t C = S / 4;
	const uint32_t full = 0xffffffffu;
	__shared__ uint32_t s_rows[kEncodeWarps][(kVertexBlockEncode + 1) * C];
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	const uint32_t b = blockIdx.x * kEncodeWarps + warp;
	const uint32_t* words = reinterpret_cast<const uint32_t*>(a.vertices);
	if (Write && blockIdx.x == 0 && threadIdx.x == 0)
	{
		// header byte, and the tail: zeros to the v1 minimum of 24 bytes, vertex 0, the channel bytes
		uint8_t* tail = a.out + 1 + a.offsets[a.blocks];
		a.out[0] = 0xa1;
		const uint32_t pad = S + C < 24u ? 24u - (S + C) : 0u;
		for (uint32_t i = 0; i < pad; ++i)
			tail[i] = 0;
		for (uint32_t i = 0; i < S; ++i)
			tail[pad + i] = uint8_t(words[i / 4] >> ((i & 3u) * 8u));
		for (uint32_t k = 0; k < C; ++k)
			tail[pad + S + k] = uint8_t(column_channel<C>(a, k));
	}
	if (b >= a.blocks)
		return; // whole warps
	const uint32_t first = b * kVertexBlockEncode, n = min(a.vertex_count - first, kVertexBlockEncode), groups = (n + 15u) / 16u;
	uint32_t* rows = s_rows[warp];
	const uint32_t* src = words + (size_t(first) - (first ? 1u : 0u)) * C; // row 0: the baseline
	if (first == 0)
		for (uint32_t w = lane; w < C; w += 32)
			rows[w] = __ldg(words + w);
	for (uint32_t w = lane; w < (n + (first ? 1u : 0u)) * C; w += 32)
		rows[w + (first ? 0u : C)] = __ldg(src + w);
	__syncwarp();

	// this lane's plane: control, per-group widths (2 bits each: at most 16 groups), size
	const uint32_t q = lane, channel = q < S ? column_channel<C>(a, q / 4) : 0u;
	int control = 2;
	uint32_t selectors = 0, size = 0;
	auto group = [&](uint32_t g) {
		Group16 grp = { { 0, 0, 0, 0 } };
		for (uint32_t i = 0; i < 16; ++i)
		{
			const uint32_t v = g * 16u + i;
			if (v >= n)
				break;
			grp.w[i / 4] |= delta_byte<C>(rows + (v + 1) * C, rows + v * C, q, channel) << ((i & 3u) * 8u);
		}
		return grp;
	};
	if (q < S)
	{
		uint32_t est0 = (groups + 3u) / 4u, est1 = est0;
		bool zero = true;
		for (uint32_t g = 0; g < groups; ++g)
		{
			const Group16 grp = group(g);
			const uint32_t s0 = group_size(grp, 0), s124 = min(min(group_size(grp, 1), group_size(grp, 2)), group_size(grp, 4));
			zero = zero && s0 == 0;
			est0 += min(s124, s0);
			est1 += min(s124, 16u);
		}
		control = zero ? 2 : (est0 < n || est1 < n) ? (est0 < est1 ? 0 : 1) : 3;
		if (control == 3)
			size = n;
		else if (control < 2)
		{
			size = (groups + 3u) / 4u;
			int last_bits = -1;
			for (uint32_t g = 0; g < groups; ++g)
			{
				const Group16 grp = group(g);
				int best_k = 3;
				uint32_t best = group_size(grp, table_bits(control, 3));
				for (int k = 0; k < 3; ++k)
				{
					const int bits = table_bits(control, k);
					const uint32_t s = group_size(grp, bits);
					if (s < best || (s == best && bits == last_bits && table_bits(control, best_k) != 8))
					{
						best_k = k;
						best = s;
					}
				}
				selectors |= uint32_t(best_k) << (2 * g);
				size += best;
				last_bits = table_bits(control, best_k);
			}
		}
	}

	// the planes' offsets in the block, after its control bytes
	uint32_t at = scan::warp_inclusive(size, lane);
	const uint32_t total = __shfl_sync(full, at, 31) + C;
	at = at - size + C;
	// the control byte of column `lane`: 2 bits per plane, from lanes 4 lane .. 4 lane + 3
	uint32_t ctrl_byte = 0;
	for (uint32_t j = 0; j < 4; ++j)
		ctrl_byte |= uint32_t(__shfl_sync(full, control, int((4u * lane + j) & 31u))) << (2 * j);
	if (!Write)
	{
		if (lane == 0)
			a.block_bytes[b] = total;
		return;
	}
	uint8_t* out = a.out + 1 + a.offsets[b];
	if (lane < C)
		out[lane] = uint8_t(ctrl_byte);
	if (q >= S || control == 2)
		return;
	uint8_t* p = out + at;
	if (control == 3)
	{
		for (uint32_t v = 0; v < n; ++v)
			p[v] = uint8_t(delta_byte<C>(rows + (v + 1) * C, rows + v * C, q, channel));
		return;
	}
	const uint32_t header = (groups + 3u) / 4u;
	for (uint32_t h = 0; h < header; ++h)
		p[h] = uint8_t(selectors >> (8 * h));
	p += header;
	for (uint32_t g = 0; g < groups; ++g)
	{
		const Group16 grp = group(g);
		const int bits = table_bits(control, int((selectors >> (2 * g)) & 3u));
		if (bits == 0)
			continue;
		if (bits == 8)
		{
			for (uint32_t i = 0; i < 16; ++i)
				p[i] = uint8_t(grp.byte(i));
			p += 16;
			continue;
		}
		// fields: 1-bit least significant first, 2/4-bit most significant first; then the escaped values in order
		const uint32_t sentinel = (1u << bits) - 1u, per_byte = 8u / uint32_t(bits);
		for (uint32_t o = 0; o < 16u / per_byte; ++o)
		{
			uint32_t byte = 0;
			for (uint32_t i = 0; i < per_byte; ++i)
			{
				const uint32_t v = min(grp.byte(o * per_byte + i), sentinel);
				byte |= bits == 1 ? v << i : v << (8u - uint32_t(bits) * (i + 1u));
			}
			*p++ = uint8_t(byte);
		}
		for (uint32_t i = 0; i < 16; ++i)
			if (grp.byte(i) >= sentinel)
				*p++ = uint8_t(grp.byte(i));
	}
}

// ---- meshlet codec --------------------------------------------------------------------------------------------------------
// One meshlet's block, the inverse of mcodec::decode_block (nvc_meshopt_format.h, with the layout); Write = false
// only measures.  `out` is where the block starts.  The fixed-size control bytes and codes sit after the variable-size
// deltas and explicit bytes, so the write pass takes deltas_size / explicit_size from the measure pass.
template <bool Write>
__device__ __forceinline__ void encode_meshlet_block(const uint32_t* words, const NvcMeshlet& m, uint8_t* out, uint32_t& deltas_size, uint32_t& explicit_size)
{
	const uint32_t vertex_count = m.vertexCount, triangle_count = m.triangleCount;
	const uint32_t codes_size = (triangle_count + 1) / 2, ctrl_size = (vertex_count + 3) / 4;
	const uint32_t gap_size = codes_size + ctrl_size < 16 ? 16 - (codes_size + ctrl_size) : 0;
	const uint32_t* refs = words + m.dataOffset;
	uint8_t* const explicit_bytes = out + deltas_size;
	uint8_t* const ctrl = explicit_bytes + explicit_size + gap_size;
	uint8_t* const codes = ctrl + ctrl_size;
	if (Write)
		for (uint32_t i = 0; i < gap_size; ++i)
			explicit_bytes[explicit_size + i] = 0;

	// References, four per control byte.  Each is stored as the zigzag of (reference - previous - 1), previous starting at
	// ~0, in the fewest whole little-endian bytes (none for 0); the 2-bit byte count goes to bits k and k + 4 of the
	// control byte.  Control 0xff reads as four 4-byte values instead, so a group in which one value needs 4 bytes, or
	// in which all four need 3 (which would read as 0xff), is written that way.
	uint32_t cursor = 0, previous = ~0u;
	for (uint32_t group = 0; group * 4 < vertex_count; ++group)
	{
		uint32_t value[4] = { 0, 0, 0, 0 }, width[4];
		uint32_t widest = 0, narrowest = 4;
		for (uint32_t k = 0; k < 4; ++k)
		{
			const uint32_t i = group * 4 + k;
			if (i < vertex_count)
			{
				const uint32_t r = m.shortRefs ? (refs[i / 2] >> (16 * (i & 1u))) & 0xffffu : refs[i];
				const uint32_t delta = r - previous - 1u;
				value[k] = (delta << 1) ^ (0u - (delta >> 31));
				previous = r;
			}
			width[k] = value[k] == 0 ? 0u : value[k] < (1u << 8) ? 1u : value[k] < (1u << 16) ? 2u : value[k] < (1u << 24) ? 3u : 4u;
			widest = max(widest, width[k]);
			narrowest = min(narrowest, width[k]);
		}
		const bool four_bytes = widest == 4 || narrowest == 3;
		uint32_t control = four_bytes ? 0xffu : 0u;
		for (uint32_t k = 0; k < 4; ++k)
		{
			const uint32_t bytes = four_bytes ? 4u : width[k];
			control |= four_bytes ? 0u : ((width[k] & 1u) << k) | ((width[k] >> 1) << (k + 4));
			if (Write)
				for (uint32_t b = 0; b < bytes; ++b)
					out[cursor + b] = uint8_t(value[k] >> (8 * b));
			cursor += bytes;
		}
		if (Write)
			ctrl[group] = uint8_t(control);
	}
	deltas_size = cursor;

	// Triangles, one 4-bit code each.  Codes 0..11 take edge (a, c) (even slot) or (c, b) (odd slot) of the triangle
	// slot / 2 back as the new triangle's first two corners, the newest such edge first, and the low bit says whether the
	// third corner is an explicit byte or the next unseen vertex.  Any other triangle is rotated so that its largest corner
	// comes last (of equal largest corners, the later one), and codes 12 + e say that its first e corners are explicit bytes
	// and the rest continue the unseen run.
	const uint8_t* tris = reinterpret_cast<const uint8_t*>(refs + mcodec::reference_words(vertex_count, m.shortRefs));
	uint32_t h0 = 0, h1 = 0, h2 = 0; // the three previous triangles as coded, a | b << 8 | c << 16, h0 the most recent
	uint32_t unseen = 0, explicit_count = 0, code_pair = 0;
	auto put_explicit = [&](uint32_t v) {
		if (Write)
			explicit_bytes[explicit_count] = uint8_t(v);
		++explicit_count;
	};
	for (uint32_t t = 0; t < triangle_count; ++t)
	{
		const uint32_t tri[3] = { tris[3 * t], tris[3 * t + 1], tris[3 * t + 2] };
		uint32_t slot = 6, first = 0;
		for (uint32_t s = 0; s < 6 && s / 2 < t && slot == 6; ++s)
		{
			const uint32_t from = s < 2 ? h0 : s < 4 ? h1 : h2;
			const uint32_t x = (s & 1) ? from >> 16 : from & 255u, y = (s & 1) ? (from >> 8) & 255u : from >> 16;
			for (uint32_t k = 0; k < 3 && slot == 6; ++k)
				if (tri[k] == x && tri[(k + 1) % 3] == y)
					slot = s, first = k;
		}
		uint32_t code;
		if (slot < 6)
		{
			const uint32_t c = tri[(first + 2) % 3];
			code = 2 * slot + (c == unseen ? 0u : 1u);
			if (c == unseen)
				++unseen;
			else
				put_explicit(c);
		}
		else
		{
			uint32_t top = 0;
			for (uint32_t k = 1; k < 3; ++k)
				top = tri[k] >= tri[top] ? k : top;
			first = (top + 1) % 3;
			const uint32_t a = tri[first], b = tri[(first + 1) % 3], c = tri[(first + 2) % 3];
			const uint32_t explicit_corners = (a == unseen && b == unseen + 1 && c == unseen + 2) ? 0u : (b == unseen && c == unseen + 1) ? 1u : c == unseen ? 2u : 3u;
			code = 12 + explicit_corners;
			for (uint32_t j = 0; j < explicit_corners; ++j)
				put_explicit(j == 0 ? a : j == 1 ? b : c);
			unseen += 3 - explicit_corners;
		}
		h2 = h1;
		h1 = h0;
		h0 = tri[first] | (tri[(first + 1) % 3] << 8) | (tri[(first + 2) % 3] << 16);
		code_pair |= code << ((t & 1u) * 4u);
		if (Write && ((t & 1u) || t + 1 == triangle_count))
			codes[t / 2] = uint8_t(code_pair);
		if (t & 1u)
			code_pair = 0;
	}
	explicit_size = explicit_count;
}

// the meshlet's words lie inside meshletdata and its counts inside the header's limits
__device__ __forceinline__ bool meshlet_encodable(const NvcMeshlet& m, uint32_t meshletdata_count)
{
	return m.vertexCount <= mcodec::kMaxVertices && m.triangleCount <= mcodec::kMaxTriangles &&
	       uint64_t(m.dataOffset) + mcodec::meshlet_words(m.vertexCount, m.triangleCount, m.shortRefs) <= meshletdata_count;
}

__device__ __forceinline__ NvcMeshlet load_meshlet(const NvcMeshlet* p)
{
	const uint32_t* w = reinterpret_cast<const uint32_t*>(p); // 24 bytes, 4-byte aligned
	NvcMeshlet m;
	uint32_t* d = reinterpret_cast<uint32_t*>(&m);
	for (uint32_t i = 0; i < 6; ++i)
		d[i] = __ldg(w + i);
	return m;
}

template <bool Write>
__global__ void __launch_bounds__(kMeshletEncodeThreads) encode_meshlets_kernel(const MeshletEncodeArgs a)
{
	const uint32_t i = blockIdx.x * kMeshletEncodeThreads + threadIdx.x;
	if (i >= a.meshlet_count)
		return;
	const NvcMeshlet m = load_meshlet(a.meshlets + i);
	if (!meshlet_encodable(m, a.meshletdata_count))
	{
		if (!Write)
		{
			a.block_bytes[i] = 0;
			atomicOr(a.invalid, 1u);
		}
		return;
	}
	uint32_t deltas_size = 0, explicit_size = 0;
	encode_meshlet_block<false>(a.meshletdata, m, nullptr, deltas_size, explicit_size);
	const uint32_t codes_size = (m.triangleCount + 1u) / 2u, ctrl_size = (m.vertexCount + 3u) / 4u;
	const uint32_t gap = codes_size + ctrl_size < 16 ? 16 - (codes_size + ctrl_size) : 0;
	const uint32_t size = deltas_size + explicit_size + gap + ctrl_size + codes_size;
	if (!Write)
	{
		a.block_bytes[i] = 2u + size;
		return;
	}
	uint8_t* out = a.out + a.offsets[i];
	out[0] = uint8_t(size);
	out[1] = uint8_t(size >> 8);
	encode_meshlet_block<true>(a.meshletdata, m, out + 2, deltas_size, explicit_size);
}

} // namespace cache
} // namespace nvc
