// nvc_meshopt_format.h — the meshopt codec formats, written once for the host and the device.
//   vertex codec  the block structure (format restated in nvc_meshopt_host.h) and the delta rule, for the host decoder
//                 and the host walk that indexes a stream for the device decoder (nvc_meshopt_host.h), and the device
//                 decoder (nvc_cache_decode.cuh).  Sizes only come from here, so the walk accepts exactly the streams the
//                 host decoder accepts, and the device finds every group where the walk measured it.
//   meshlet codec a meshlet's words and the block decoder, for the host reader (nvc_scene_cache.cpp), the device decoder
//                 (nvc_cache_decode.cuh) and the device encoder (nvc_cache_encode.cuh), which writes what it reads back.
//   index codec   the decoder's FIFO rings, for the host decoder and encoder (nvc_meshopt_host.h, nvc_meshopt_encode.cpp),
//                 and the per-triangle step, for the host decoder, the host walk that cuts a stream into chunks
//                 (nvc_meshopt_host.h) and the device decoder (nvc_cache_decode.cuh).
#pragma once

#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "../../include/niagara_cull.h"

#if defined(__CUDACC__) || defined(NVC_EMU)
#define NVC_CODEC_FN __host__ __device__
#else
#define NVC_CODEC_FN
#endif

namespace nvc
{
namespace vcodec
{

// vertices per block: min(256, (8192 / stride) & ~15)
NVC_CODEC_FN inline uint32_t block_vertices(uint32_t stride)
{
	uint32_t n = (8192u / stride) & ~15u;
	return n < 256u ? n : 256u;
}

// group width in bits from a 2-bit selector: v0 {0, 2, 4, 8}; v1 control 0 {0, 1, 2, 4}, control 1 {1, 2, 4, 8}
NVC_CODEC_FN inline int group_width(int version, int control, uint32_t sel)
{
	if (version == 0)
		return sel == 0 ? 0 : 1 << sel; // 0, 2, 4, 8
	uint32_t i = sel + uint32_t(control); // v1 table {0, 1, 2, 4, 8} from offset control
	return i == 0 ? 0 : 1 << (i - 1);
}

// selector header of a plane of `groups` groups of 16 values: 2 bits per group
NVC_CODEC_FN inline uint32_t selector_bytes(uint32_t groups)
{
	return (groups + 3u) / 4u;
}

NVC_CODEC_FN inline int popcount32(uint32_t v)
{
#if defined(__CUDA_ARCH__)
	return __popc(v);
#else
	return __builtin_popcount(v);
#endif
}

// Bytes one group of 16 values of `width` bits occupies from p: 0 (zeros), 16 (literals), or the packed fields plus one
// escape byte per field that holds the all-ones code, counted on the packed bits without unpacking them.  Fields never
// straddle a byte, so the byte order of the loads does not matter.  Width 1/2/4: p must hold 2 * width readable bytes.
NVC_CODEC_FN inline uint32_t group_bytes(const uint8_t* p, int width)
{
	if (width == 0)
		return 0;
	if (width == 8)
		return 16;
	if (width == 1)
		return 2u + uint32_t(popcount32(uint32_t(p[0]) | (uint32_t(p[1]) << 8)));
	uint32_t x = uint32_t(p[0]) | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24);
	if (width == 2)
		return 4u + uint32_t(popcount32(x & (x >> 1) & 0x55555555u));
	uint32_t y = uint32_t(p[4]) | (uint32_t(p[5]) << 8) | (uint32_t(p[6]) << 16) | (uint32_t(p[7]) << 24);
	x &= x >> 1;
	y &= y >> 1;
	return 8u + uint32_t(popcount32(x & (x >> 2) & 0x11111111u)) + uint32_t(popcount32(y & (y >> 2) & 0x11111111u));
}

// The 16 values of a group of width 1, 2 or 4 that occupies group_bytes(p, width) bytes from p: fields (1-bit: least
// significant bit first, 2/4-bit: most significant first), an all-ones field replaced by the next escape byte, in order.
NVC_CODEC_FN inline void unpack_group(const uint8_t* p, int width, uint8_t* out)
{
	const uint32_t escape = (1u << width) - 1u;
	const uint8_t* e = p + 2 * width;
	for (int i = 0; i < 16; ++i)
	{
		uint32_t v;
		if (width == 4)
			v = (p[i >> 1] >> ((i & 1) ? 0 : 4)) & 15u;
		else if (width == 2)
			v = (p[i >> 2] >> (6 - 2 * (i & 3))) & 3u;
		else
			v = (p[i >> 3] >> (i & 7)) & 1u;
		out[i] = v == escape ? *e++ : uint8_t(v);
	}
}

// Deltas of one 4-byte column by its channel: a vertex's value is the previous one combined with the delta term of its
// four plane bytes.  All three combinations are abelian groups with 0 as identity, so a block can be decoded from 0 and
// the blocks' carries found by a scan.
//   channel & 3 == 0: per byte, zigzag delta, add mod 2^8
//   channel & 3 == 1: per 16 bits, zigzag delta, add mod 2^16
//   channel & 3 == 2: 32-bit xor after rotating left by (32 - (channel >> 4)) & 31
NVC_CODEC_FN inline uint32_t delta_term(uint32_t bytes4, uint32_t channel)
{
	switch (channel & 3u)
	{
	case 0:
		return ((bytes4 >> 1) & 0x7f7f7f7fu) ^ ((bytes4 & 0x01010101u) * 0xffu);
	case 1:
		return ((bytes4 >> 1) & 0x7fff7fffu) ^ ((bytes4 & 0x00010001u) * 0xffffu);
	default:
	{
		uint32_t r = (32u - (channel >> 4)) & 31u;
		return (bytes4 << r) | (bytes4 >> ((32u - r) & 31u));
	}
	}
}

NVC_CODEC_FN inline uint32_t combine(uint32_t a, uint32_t b, uint32_t channel)
{
	switch (channel & 3u)
	{
	case 0:
		return ((a & 0x7f7f7f7fu) + (b & 0x7f7f7f7fu)) ^ ((a ^ b) & 0x80808080u);
	case 1:
		return ((a & 0x7fff7fffu) + (b & 0x7fff7fffu)) ^ ((a ^ b) & 0x80008000u);
	default:
		return a ^ b;
	}
}

} // namespace vcodec

// Meshlet codec (meshoptimizer v1.0 meshletcodec, extern/meshoptimizer/src/meshletcodec.cpp — restated, not copied).  A
// compressed MESHLETDATA section (writeMeshletDataCompressed, scenecache.cpp:84-117) holds, for every Meshlet in order, a
// uint16 byte count and one block that decodes into the words meshletdata[dataOffset ...]: vertexCount references
// (uint16 when shortRefs, else uint32) followed by triangleCount * 3 index bytes.
//
// Block layout, from the END of the block:   [ deltas | extra | gap | ctrl | codes ]
//   codes  (triangleCount + 1) / 2 bytes, one nibble per triangle
//   ctrl   (vertexCount + 3) / 4 bytes, 2 bits per reference (bit k and bit k + 4 of the group's byte)
//   gap    pads codes + ctrl to 16 bytes (decoder over-read room); deltas and extra must end exactly at the gap
// References: per group of four, each value is a 0/1/2/3-byte little-endian zigzag delta to the previous
//   reference plus one (a ctrl byte of 0xff switches the whole group to 4-byte values); the first is relative to -1.
// Triangles: nibble < 12 re-uses one edge of one of the three previous triangles (nibble / 4 = how far back, bit 1 =
//   which edge: (a, c) or (c, b)), bit 0 says whether the third corner is an explicit byte or the next unseen
//   vertex; nibble >= 12 starts a new triangle with nibble - 12 explicit bytes for its (a, b, c) — explicit bytes
//   come first, then consecutive unseen vertices.
namespace mcodec
{

constexpr uint32_t kMaxVertices = 64, kMaxTriangles = 96; // per meshlet, as the reference builds them (the header's meshletMax*)

// words of meshletdata a meshlet's references take (two per word with shortRefs), and all its words with the triangles
NVC_CODEC_FN inline uint32_t reference_words(uint32_t vertex_count, bool short_refs)
{
	return short_refs ? (vertex_count + 1) / 2 : vertex_count;
}

NVC_CODEC_FN inline uint32_t meshlet_words(uint32_t vertex_count, uint32_t triangle_count, bool short_refs)
{
	return reference_words(vertex_count, short_refs) + (triangle_count * 3 + 3) / 4;
}

// One block of `size` bytes holding vertex_count references and triangle_count triangles; false when malformed.  Every
// read stays inside the block.  The outputs go to `out`, in this order, as they are decoded:
//   out.reference(i, value)     each reference, i = 0 .. vertex_count - 1
//   out.flush()                 after the last reference, and after the last triangle (a writer that assembles whole
//                               words stores its partial word there)
//   out.triangle(t, a, b, c)    each triangle, t = 0 .. triangle_count - 1, its corners in the low byte of a, b and c
template <typename Out>
NVC_CODEC_FN inline bool decode_block(const uint8_t* block, uint32_t size, uint32_t vertex_count, uint32_t triangle_count, Out& out)
{
	const uint32_t codes_size = (triangle_count + 1) / 2, ctrl_size = (vertex_count + 3) / 4;
	const uint32_t gap_size = codes_size + ctrl_size < 16 ? 16 - (codes_size + ctrl_size) : 0;
	if (size < codes_size + ctrl_size + gap_size)
		return false;
	const uint8_t* codes = block + size - codes_size;
	const uint8_t* ctrl = codes - ctrl_size;
	const uint32_t limit = size - codes_size - ctrl_size - gap_size; // deltas + extra occupy [0, limit)
	uint32_t cursor = 0;

	uint32_t previous = ~0u;
	for (uint32_t group = 0; group * 4 < vertex_count; ++group)
	{
		const uint32_t control = ctrl[group];
		for (uint32_t k = 0; k < 4; ++k)
		{
			const uint32_t width = control == 0xff ? 4 : (((control >> k) & 1u) | ((control >> (k + 3)) & 2u));
			if (limit - cursor < width)
				return false;
			uint32_t value = 0;
			for (uint32_t i = 0; i < width; ++i)
				value |= uint32_t(block[cursor + i]) << (8 * i);
			cursor += width;
			previous = previous + ((value >> 1) ^ (0u - (value & 1u))) + 1;
			const uint32_t i = group * 4 + k;
			if (i < vertex_count)
				out.reference(i, previous);
		}
	}
	out.flush();

	uint32_t h0 = 0, h1 = 0, h2 = 0; // the three previous triangles, a | b << 8 | c << 16, h0 the most recent
	uint32_t unseen = 0;
	for (uint32_t t = 0; t < triangle_count; ++t)
	{
		const uint32_t code = (codes[t / 2] >> ((t & 1) * 4)) & 15u;
		uint32_t c[3];
		if (code < 12)
		{
			const uint32_t from = code < 4 ? h0 : code < 8 ? h1 : h2;
			c[0] = (code & 2) ? from >> 16 : from & 255u;
			c[1] = (code & 2) ? (from >> 8) & 255u : from >> 16;
			if (code & 1)
			{
				if (cursor >= limit)
					return false;
				c[2] = block[cursor++];
			}
			else
				c[2] = unseen++ & 255u;
		}
		else
			for (uint32_t j = 0; j < 3; ++j)
			{
				if (code > 12 + j)
				{
					if (cursor >= limit)
						return false;
					c[j] = block[cursor++];
				}
				else
					c[j] = unseen++ & 255u;
			}
		out.triangle(t, c[0], c[1], c[2]);
		h2 = h1;
		h1 = h0;
		h0 = c[0] | (c[1] << 8) | (c[2] << 16);
	}
	out.flush();
	return cursor == limit;
}

} // namespace mcodec

namespace icodec
{

// One of the index codec's 16-entry FIFOs (vertices; edges as two rings pushed together), as the decoder keeps it.  The
// encoder keeps the same rings, so that every slot it codes is the one the decoder will read.
struct Ring16
{
	uint32_t slot[16];
	uint32_t head = 0;
	Ring16() { memset(slot, 0xff, sizeof(slot)); }
	// the slot is written even when the head does not advance (a vertex re-read from the FIFO); the next put overwrites it
	// before any lookup can reach it
	void put(uint32_t v, bool advance = true)
	{
		slot[head] = v;
		head = (head + (advance ? 1u : 0u)) & 15u;
	}
	uint32_t back(uint32_t n) const { return slot[(head - n) & 15u]; } // back(1) = most recent
};

NVC_CODEC_FN inline uint32_t unzigzag(uint32_t v)
{
	return (v >> 1) ^ (0u - (v & 1u));
}

// A varint of 7 bits per byte, low group first: it ends at the first byte below 128 or after its fifth byte, whatever
// that byte's top bit.  `data.next(b)` gives the next data byte; false when the data has ended.
template <typename Data>
NVC_CODEC_FN inline bool read_varint(Data& data, uint32_t& value)
{
	value = 0;
	for (int i = 0; i < 5; ++i)
	{
		uint32_t b;
		if (!data.next(b))
			return false;
		value |= (b & 127u) << (7 * i);
		if (b < 128u)
			break;
	}
	return true;
}

// One triangle of the index codec (the format is in nvc_meshopt_host.h), for the host decoder, the host walk that finds
// where each chunk's data starts (nvc_meshopt_host.h) and the device decoder's symbolic and concrete passes
// (nvc_cache_decode.cuh).  The state `s` holds values of type S::Value, concrete indices or not:
//   S::add(v, k), S::zero()         v + k mod 2^32; the value 0 (a reset `next`)
//   s.next, s.last                  the next new vertex, the last explicit index
//   s.vert(n), s.edge_a(n), s.edge_b(n)   ring lookups n back, 1 <= n <= 15 (1 = the most recent push)
//   s.put_vert(v, advance), s.put_edge(a, b)
// A FIFO hit (put_vert(v, false)) writes the head slot without advancing, and the next advancing put overwrites that slot;
// lookups reach at most 15 back in a 16-slot ring, so nothing reads it in between.  The device decoder still tracks that
// write, physical slot by slot, so its chunk entry states are the serial decoder's exactly.
// Data bytes come from `data` (see read_varint).  Returns false, with the triangle unfinished, exactly where
// decode_index_buffer finds the stream corrupt: an aux byte or a varint that runs past the data.
template <typename S, typename Data>
NVC_CODEC_FN inline bool decode_triangle(S& s, uint32_t code, const uint8_t* aux, uint32_t direct_slots, Data& data, typename S::Value (&corner)[3])
{
	if (code < 0xf0u)
	{
		const uint32_t e = (code >> 4) + 1u, sel = code & 15u;
		corner[0] = s.edge_a(e);
		corner[1] = s.edge_b(e);
		if (sel < direct_slots)
		{
			corner[2] = sel == 0 ? s.next : s.vert(sel + 1u);
			if (sel == 0)
				s.next = S::add(s.next, 1u);
			s.put_vert(corner[2], sel == 0);
		}
		else
		{
			uint32_t delta = sel == 13u ? 0xffffffffu : 1u; // 13 -> -1, 14 -> +1
			if (sel == 15u && !read_varint(data, delta))
				return false;
			s.last = S::add(s.last, sel == 15u ? unzigzag(delta) : delta);
			corner[2] = s.last;
			s.put_vert(corner[2], true);
		}
		s.put_edge(corner[2], corner[1]);
		s.put_edge(corner[0], corner[2]);
		return true;
	}
	uint32_t sel_a = 0, x;
	if (code < 0xfeu)
		x = aux[code & 15u];
	else
	{
		if (!data.next(x))
			return false;
		sel_a = code == 0xfeu ? 0u : 15u;
		if (x == 0)
			s.next = S::zero();
	}
	// each corner: the next new vertex (0), an explicit varint (15), else a vertex-ring lookup.  Lookups see the ring as
	// it is before this triangle's pushes; `next` and the varints are consumed in corner order a, b, c.
	const uint32_t sel[3] = { sel_a, x >> 4, x & 15u };
	for (int j = 0; j < 3; ++j)
	{
		if (sel[j] == 0)
		{
			corner[j] = s.next;
			s.next = S::add(s.next, 1u);
		}
		else if (sel[j] == 15u)
		{
			uint32_t delta;
			if (!read_varint(data, delta))
				return false;
			s.last = S::add(s.last, unzigzag(delta));
			corner[j] = s.last;
		}
		else
			corner[j] = s.vert(sel[j]);
	}
	s.put_vert(corner[0], true);
	s.put_vert(corner[1], sel[1] == 0 || sel[1] == 15u);
	s.put_vert(corner[2], sel[2] == 0 || sel[2] == 15u);
	s.put_edge(corner[1], corner[0]);
	s.put_edge(corner[2], corner[1]);
	s.put_edge(corner[0], corner[2]);
	return true;
}

} // namespace icodec

// Where a vertex stream keeps its version, baseline vertex and (v1) channel bytes (channels nullptr for v0)
struct VertexStreamTail
{
	int version;
	const uint8_t* baseline;
	const uint8_t* channels;
};

// the host decoders (decode_vertex_stream, walk_vertex_stream, decode_index_stream, ...) are inline in nvc_meshopt_host.h

// nvc_meshopt_encode.cpp (host): index codec v1 of index_count indices (a multiple of 3) into out[index_stream_bound]
size_t index_stream_bound(size_t index_count);
size_t encode_index_stream(const uint32_t* indices, size_t index_count, uint8_t* out);

// nvc_scene_cache.cpp (host): the per-meshlet stream of a compressed MESHLETDATA section indexed for the device decoder,
// without decoding it.  checkpoints[(meshletCount + kMeshletGroup - 1) / kMeshletGroup + 1]: the offset of every
// kMeshletGroup-th meshlet's size field, then the section's size.  records[meshletCount][2]: dataOffset and
// vertexCount | triangleCount << 8 | shortRefs << 16.  NVC_ERROR_UNSUPPORTED when the meshlets' word ranges are not in
// increasing, non-overlapping order (every cache the reference writes is: appendMeshlet appends), so that each meshlet
// owns whole words of the output, or when the section is 4 GiB or larger; NVC_ERROR_INVALID_ARGUMENT when `info` does not
// describe the file.
constexpr uint32_t kMeshletGroup = 32;

// bytes per element of each section (NvcSceneCacheSectionId order), as the header counts them
constexpr uint32_t kCacheElementSize[NVC_CACHE_SECTION_COUNT] = { 16, 4, 24, 4, 2, 208, 64, 48, 32, 24, 32, 1, 1, 4, 256 };
int index_meshlet_stream(const void* file, size_t file_size, const NvcSceneCacheInfo* info, uint32_t* checkpoints, uint32_t* records);

} // namespace nvc
