// nvc_scene_cache.cpp — reader of the reference's scene cache (.cache v7), SURVEY §8(f) row N2.  Host only.
// (The vertex / index codec streams are decoded by nvc_meshopt_decode.cpp; loadSceneCache's normalizeIndicesForOMM step,
// scenecache.cpp:344-353, belongs to the ray-tracing feature and is not applied.)
//
// Follows src/scenecache.cpp: SceneHeader (16-55), the section order of saveSceneCache (158-197) and, for the
// per-meshlet compressed stream, the layout written by writeMeshletDataCompressed (84-117): for every Meshlet, in
// order, a uint16 byte count followed by one meshopt "meshlet codec" block (meshoptimizer v1.0 meshletcodec,
// extern/meshoptimizer/src/meshletcodec.cpp) that decodes into the words meshletdata[dataOffset ...]:
// vertexCount references (uint16 when shortRefs, else uint32) followed by triangleCount * 3 index bytes.
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
#include "../../include/niagara_cull.h"
#include "nvc_meshopt_format.h"

#include <string.h>

namespace
{

// one meshlet block -> refs (ref_size 2 or 4 bytes each) and triangles (3 bytes each); false when malformed
bool decodeMeshletBlock(const uint8_t* block, size_t size, uint32_t vertex_count, uint32_t triangle_count, uint32_t ref_size, uint8_t* refs_out, uint8_t* triangles_out)
{
	size_t codes_size = (triangle_count + 1) / 2, ctrl_size = (vertex_count + 3) / 4;
	size_t gap_size = codes_size + ctrl_size < 16 ? 16 - (codes_size + ctrl_size) : 0;
	if (size < codes_size + ctrl_size + gap_size)
		return false;
	const uint8_t* codes = block + size - codes_size;
	const uint8_t* ctrl = codes - ctrl_size;
	const uint8_t* limit = ctrl - gap_size; // deltas + extra occupy [block, limit)
	const uint8_t* cursor = block;

	uint32_t previous = ~0u;
	for (uint32_t group = 0; group * 4 < vertex_count; ++group)
	{
		uint8_t control = ctrl[group];
		for (uint32_t k = 0; k < 4; ++k)
		{
			uint32_t width = control == 0xff ? 4 : (((control >> k) & 1u) | ((control >> (k + 3)) & 2u));
			if (size_t(limit - cursor) < width)
				return false;
			uint32_t value = 0;
			for (uint32_t b = 0; b < width; ++b)
				value |= uint32_t(cursor[b]) << (8 * b);
			cursor += width;
			uint32_t delta = (value >> 1) ^ (0u - (value & 1u));
			previous = previous + delta + 1;
			uint32_t i = group * 4 + k;
			if (i < vertex_count)
			{
				if (ref_size == 2)
				{
					uint16_t r = uint16_t(previous);
					memcpy(refs_out + size_t(i) * 2, &r, 2);
				}
				else
					memcpy(refs_out + size_t(i) * 4, &previous, 4);
			}
		}
	}

	struct Tri
	{
		uint8_t a, b, c;
	};
	Tri history[3] = {}; // [0] = most recent
	uint32_t unseen = 0;
	auto corner = [&](bool explicit_byte, uint8_t& out) -> bool {
		if (explicit_byte)
		{
			if (cursor >= limit)
				return false;
			out = *cursor++;
		}
		else
			out = uint8_t(unseen++);
		return true;
	};
	for (uint32_t i = 0; i < triangle_count; ++i)
	{
		uint32_t code = (codes[i / 2] >> ((i & 1) * 4)) & 0xfu;
		Tri t;
		if (code < 12)
		{
			const Tri& from = history[code / 4];
			if (code & 2)
				t.a = from.c, t.b = from.b;
			else
				t.a = from.a, t.b = from.c;
			if (!corner((code & 1) != 0, t.c))
				return false;
		}
		else if (!corner(code > 12, t.a) || !corner(code > 13, t.b) || !corner(code > 14, t.c))
			return false;
		triangles_out[i * 3 + 0] = t.a;
		triangles_out[i * 3 + 1] = t.b;
		triangles_out[i * 3 + 2] = t.c;
		history[2] = history[1];
		history[1] = history[0];
		history[0] = t;
	}
	return cursor == limit;
}

} // namespace

extern "C" NVC_API int nvc_scene_cache_parse(const void* file, size_t file_size, NvcSceneCacheInfo* out)
{
	if (!file || !out)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (file_size < sizeof(NvcSceneCacheHeader))
		return NVC_ERROR_CORRUPT;
	memset(out, 0, sizeof(*out));
	NvcSceneCacheHeader& h = out->header;
	memcpy(&h, file, sizeof(h));
	if (h.magic != NVC_SCENE_CACHE_MAGIC)
		return NVC_ERROR_CORRUPT;
	if (h.version != NVC_SCENE_CACHE_VERSION)
		return NVC_ERROR_UNSUPPORTED;

	const uint32_t counts[NVC_CACHE_SECTION_COUNT] = { h.vertexCount, h.indexCount, h.meshletCount, h.meshletdataCount, h.meshletvtx0Count, h.meshCount,
		h.materialCount, h.drawCount, h.lightCount, h.animationCount, h.keyframeCount, h.ommArrayDataSize, h.ommIndexDataSize, h.ommDescCount, h.texturePathCount };
	uint64_t offset = sizeof(NvcSceneCacheHeader);
	for (int s = 0; s < NVC_CACHE_SECTION_COUNT; ++s)
	{
		NvcSceneCacheSection& sec = out->sections[s];
		sec.count = counts[s];
		sec.element_size = nvc::kCacheElementSize[s];
		sec.decoded_bytes = uint64_t(sec.count) * sec.element_size;
		sec.stored_bytes = sec.decoded_bytes;
		if (h.compressed)
		{
			// scenecache.cpp:160-179: exactly these four sections go through a meshopt codec
			if (s == NVC_CACHE_VERTICES)
				sec.stored_bytes = h.compressedVertexBytes, sec.compressed = 1;
			else if (s == NVC_CACHE_INDICES)
				sec.stored_bytes = h.compressedIndexBytes, sec.compressed = 1;
			else if (s == NVC_CACHE_MESHLETDATA)
				sec.stored_bytes = h.compressedMeshletDataBytes, sec.compressed = 1;
			else if (s == NVC_CACHE_MESHLETVTX0)
				sec.stored_bytes = h.compressedMeshletVtx0Bytes, sec.compressed = 1;
		}
		sec.offset = offset;
		offset += sec.stored_bytes;
		if (offset > file_size)
			return NVC_ERROR_CORRUPT;
	}
	if (offset != file_size)
		return NVC_ERROR_CORRUPT;

	const NvcSceneCacheSection& md = out->sections[NVC_CACHE_MESHLETDATA];
	const NvcMeshlet* meshlets = reinterpret_cast<const NvcMeshlet*>(static_cast<const uint8_t*>(file) + out->sections[NVC_CACHE_MESHLETS].offset);
	// every meshlet's words must lie inside meshletdata[]
	for (uint32_t i = 0; i < h.meshletCount; ++i)
	{
		NvcMeshlet m;
		memcpy(&m, meshlets + i, sizeof(m));
		uint64_t ref_words = m.shortRefs ? (uint64_t(m.vertexCount) + 1) / 2 : m.vertexCount;
		uint64_t words = ref_words + (uint64_t(m.triangleCount) * 3 + 3) / 4;
		if (uint64_t(m.dataOffset) + words > h.meshletdataCount)
			return NVC_ERROR_CORRUPT;
	}
	if (md.compressed)
	{
		// the uint16 size chain of writeMeshletDataCompressed must add up (scenecache.cpp:108-113)
		const uint8_t* p = static_cast<const uint8_t*>(file) + md.offset;
		uint64_t at = 0;
		for (uint32_t i = 0; i < h.meshletCount; ++i)
		{
			if (at + 2 > md.stored_bytes)
				return NVC_ERROR_CORRUPT;
			uint16_t n;
			memcpy(&n, p + at, 2);
			at += 2 + uint64_t(n);
		}
		if (at != md.stored_bytes)
			return NVC_ERROR_CORRUPT;
	}
	return NVC_OK;
}

extern "C" NVC_API int nvc_scene_cache_read(const void* file, size_t file_size, const NvcSceneCacheInfo* info, int section, void* dst, size_t dst_bytes)
{
	if (!file || !info || section < 0 || section >= NVC_CACHE_SECTION_COUNT || (!dst && dst_bytes))
		return NVC_ERROR_INVALID_ARGUMENT;
	const NvcSceneCacheSection& sec = info->sections[section];
	if (dst_bytes < sec.decoded_bytes || sec.offset + sec.stored_bytes > file_size)
		return NVC_ERROR_INVALID_ARGUMENT;
	const uint8_t* base = static_cast<const uint8_t*>(file);
	if (!sec.compressed)
	{
		if (sec.decoded_bytes)
			memcpy(dst, base + sec.offset, sec.decoded_bytes);
		return NVC_OK;
	}
	if (section == NVC_CACHE_VERTICES) // readVertexCompressed, scenecache.cpp:244-248, Vertex stride
		return nvc::decode_vertex_stream(base + sec.offset, sec.stored_bytes, sec.count, 16, static_cast<uint8_t*>(dst));
	if (section == NVC_CACHE_MESHLETVTX0) // uint16 x 4 per element of the stream (scenecache.cpp:329)
		return sec.count % 4 ? NVC_ERROR_CORRUPT : nvc::decode_vertex_stream(base + sec.offset, sec.stored_bytes, sec.count / 4, 8, static_cast<uint8_t*>(dst));
	if (section == NVC_CACHE_INDICES) // readIndexCompressed, scenecache.cpp:250-254
		return nvc::decode_index_stream(base + sec.offset, sec.stored_bytes, sec.count, static_cast<uint32_t*>(dst));
	if (section != NVC_CACHE_MESHLETDATA)
		return NVC_ERROR_UNSUPPORTED;

	// readMeshletDataCompressed, scenecache.cpp:256-271
	memset(dst, 0, sec.decoded_bytes);
	uint32_t* words = static_cast<uint32_t*>(dst);
	const uint8_t* meshlets = base + info->sections[NVC_CACHE_MESHLETS].offset;
	const uint8_t* p = base + sec.offset;
	uint64_t at = 0;
	for (uint32_t i = 0; i < info->header.meshletCount; ++i)
	{
		NvcMeshlet m;
		memcpy(&m, meshlets + size_t(i) * sizeof(NvcMeshlet), sizeof(m));
		uint16_t n;
		memcpy(&n, p + at, 2);
		at += 2;
		uint32_t ref_words = m.shortRefs ? (uint32_t(m.vertexCount) + 1) / 2 : m.vertexCount;
		uint8_t* refs = reinterpret_cast<uint8_t*>(words + m.dataOffset);
		uint8_t* triangles = reinterpret_cast<uint8_t*>(words + m.dataOffset + ref_words);
		if (!decodeMeshletBlock(p + at, n, m.vertexCount, m.triangleCount, m.shortRefs ? 2u : 4u, refs, triangles))
			return NVC_ERROR_CORRUPT;
		at += n;
	}
	return NVC_OK;
}

namespace nvc
{

int index_meshlet_stream(const void* file, size_t file_size, const NvcSceneCacheInfo* info, uint32_t* checkpoints, uint32_t* records)
{
	const NvcSceneCacheSection& md = info->sections[NVC_CACHE_MESHLETDATA];
	const NvcSceneCacheSection& ms = info->sections[NVC_CACHE_MESHLETS];
	const uint32_t count = info->header.meshletCount;
	if (ms.offset > file_size || uint64_t(count) * sizeof(NvcMeshlet) > file_size - ms.offset || md.offset > file_size || md.stored_bytes > file_size - md.offset)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (md.stored_bytes > 0xffffffffull)
		return NVC_ERROR_UNSUPPORTED; // checkpoints are 32-bit offsets
	const uint8_t* base = static_cast<const uint8_t*>(file);
	const uint8_t* p = base + md.offset;
	uint64_t at = 0, end = 0;
	bool ordered = true;
	for (uint32_t i = 0; i < count; ++i)
	{
		NvcMeshlet m;
		memcpy(&m, base + ms.offset + size_t(i) * sizeof(NvcMeshlet), sizeof(m));
		uint64_t ref_words = m.shortRefs ? (uint64_t(m.vertexCount) + 1) / 2 : m.vertexCount;
		uint64_t words = ref_words + (uint64_t(m.triangleCount) * 3 + 3) / 4;
		// nvc_scene_cache_parse checks both of these: an info they fail does not describe this file
		if (uint64_t(m.dataOffset) + words > md.count || at + 2 > md.stored_bytes)
			return NVC_ERROR_INVALID_ARGUMENT;
		ordered = ordered && m.dataOffset >= end;
		end = m.dataOffset + words;
		if (i % kMeshletGroup == 0)
			checkpoints[i / kMeshletGroup] = uint32_t(at);
		records[2 * size_t(i)] = m.dataOffset;
		records[2 * size_t(i) + 1] = uint32_t(m.vertexCount) | (uint32_t(m.triangleCount) << 8) | (m.shortRefs ? 1u << 16 : 0u);
		uint16_t n;
		memcpy(&n, p + at, 2);
		at += 2 + uint64_t(n);
	}
	if (at != md.stored_bytes)
		return NVC_ERROR_INVALID_ARGUMENT;
	checkpoints[(count + kMeshletGroup - 1) / kMeshletGroup] = uint32_t(at);
	return ordered ? NVC_OK : NVC_ERROR_UNSUPPORTED;
}

} // namespace nvc

extern "C" NVC_API int nvc_decode_vertex_stream(void* dst, uint32_t vertex_count, uint32_t vertex_size, const void* stream, size_t stream_size)
{
	if ((!dst && vertex_count) || !stream)
		return NVC_ERROR_INVALID_ARGUMENT;
	return nvc::decode_vertex_stream(static_cast<const uint8_t*>(stream), stream_size, vertex_count, vertex_size, static_cast<uint8_t*>(dst));
}

extern "C" NVC_API int nvc_decode_index_stream(uint32_t* dst, uint32_t index_count, const void* stream, size_t stream_size)
{
	if ((!dst && index_count) || !stream)
		return NVC_ERROR_INVALID_ARGUMENT;
	return nvc::decode_index_stream(static_cast<const uint8_t*>(stream), stream_size, index_count, dst);
}

extern "C" NVC_API int nvc_decode_meshlet_stream(void* references, uint32_t vertex_count, uint32_t reference_size, uint8_t* triangles, uint32_t triangle_count,
    const void* stream, size_t stream_size)
{
	if (!stream || (reference_size != 2 && reference_size != 4) || vertex_count > 256 || triangle_count > 256 || (!references && vertex_count) || (!triangles && triangle_count))
		return NVC_ERROR_INVALID_ARGUMENT;
	return decodeMeshletBlock(static_cast<const uint8_t*>(stream), stream_size, vertex_count, triangle_count, reference_size, static_cast<uint8_t*>(references), triangles) ? NVC_OK
	                                                                                                                                                                     : NVC_ERROR_CORRUPT;
}
