// nvc_meshopt_format.h — the block structure of the meshopt vertex codec (format restated in nvc_meshopt_decode.cpp),
// written once for its three users: the host decoder (nvc_meshopt_decode.cpp), the host walk that indexes a stream for
// the device decoder (same file) and the device decoder (nvc_cache_decode.cuh).  Sizes only come from here, so the walk
// accepts exactly the streams the host decoder accepts, and the device finds every group where the walk measured it.
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

} // namespace icodec

// Where a vertex stream keeps its version, baseline vertex and (v1) channel bytes (channels nullptr for v0)
struct VertexStreamTail
{
	int version;
	const uint8_t* baseline;
	const uint8_t* channels;
};

// nvc_meshopt_decode.cpp (host)
int decode_vertex_stream(const uint8_t* stream, size_t stream_size, uint32_t vertex_count, uint32_t stride, uint8_t* out);
int decode_index_stream(const uint8_t* stream, size_t stream_size, uint32_t index_count, uint32_t* out);
int walk_vertex_stream(const uint8_t* stream, size_t stream_size, uint32_t vertex_count, uint32_t stride, uint32_t* block_start, uint16_t* plane_offset,
    VertexStreamTail* tail);

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
