// nvc_scene_cache.cpp — reader of the reference's scene cache (.cache v7), SURVEY §8(f) row N2.  Host only.
// (The vertex / index codec streams are decoded by nvc_meshopt_host.h; loadSceneCache's normalizeIndicesForOMM step,
// scenecache.cpp:344-353, belongs to the ray-tracing feature and is not applied.)
//
// Follows src/scenecache.cpp: SceneHeader (16-55), the section order of saveSceneCache (158-197) and, for the
// per-meshlet compressed stream, the layout written by writeMeshletDataCompressed (84-117), decoded by the meshlet codec of
// nvc_meshopt_format.h.
#include "../../include/niagara_cull.h"
#include "nvc_meshopt_host.h"

#include <string.h>

namespace
{

// Where mcodec::decode_block puts a meshlet's outputs on the host: only the bytes of each reference (ref_size 2 or 4)
// and of each triangle, so that nothing else in the destination changes
struct MeshletByteWriter
{
	uint8_t* refs;
	uint8_t* triangles;
	uint32_t ref_size;
	void reference(uint32_t i, uint32_t value)
	{
		if (ref_size == 2)
		{
			uint16_t r = uint16_t(value);
			memcpy(refs + size_t(i) * 2, &r, 2);
		}
		else
			memcpy(refs + size_t(i) * 4, &value, 4);
	}
	void triangle(uint32_t t, uint32_t a, uint32_t b, uint32_t c)
	{
		triangles[size_t(t) * 3 + 0] = uint8_t(a);
		triangles[size_t(t) * 3 + 1] = uint8_t(b);
		triangles[size_t(t) * 3 + 2] = uint8_t(c);
	}
	void flush() {}
};

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
		if (uint64_t(m.dataOffset) + nvc::mcodec::meshlet_words(m.vertexCount, m.triangleCount, m.shortRefs) > h.meshletdataCount)
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
		uint32_t* refs = words + m.dataOffset;
		MeshletByteWriter out = { reinterpret_cast<uint8_t*>(refs), reinterpret_cast<uint8_t*>(refs + nvc::mcodec::reference_words(m.vertexCount, m.shortRefs)), m.shortRefs ? 2u : 4u };
		if (!nvc::mcodec::decode_block(p + at, n, m.vertexCount, m.triangleCount, out))
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
		const uint32_t words = mcodec::meshlet_words(m.vertexCount, m.triangleCount, m.shortRefs);
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
	// a block of at most 256 references and 256 triangles spans far less than 4 GiB: a larger stream cannot be one block
	if (stream_size > 0xffffffffull)
		return NVC_ERROR_CORRUPT;
	MeshletByteWriter out = { static_cast<uint8_t*>(references), triangles, reference_size };
	return nvc::mcodec::decode_block(static_cast<const uint8_t*>(stream), uint32_t(stream_size), vertex_count, triangle_count, out) ? NVC_OK : NVC_ERROR_CORRUPT;
}
