// nvc_scene_cache_write.cpp — the scene cache (.cache v7) writer: the file saveSceneCache (src/scenecache.cpp:119-203) writes,
// byte for byte, into a caller's host buffer.  Compressed caches encode VERTICES and MESHLETVTX0 (vertex codec) and MESHLETDATA
// (meshlet codec) with the kernels of nvc_cache_encode.cuh, and INDICES (index codec, one sequential state machine) on the host
// while those run.  Everything is checked, and every stream measured, before the first byte reaches the caller's buffer.
#include "nvc_internal.h"
#include "nvc_meshopt_format.h"

#include <string.h>

#include <memory>
#include <vector>

namespace
{

const uint32_t kTailBytes = 24; // the vertex codec v1's tail: at least 24 bytes, and stride + stride / 4 <= 20 here
const uint32_t kMeshletRecordBound = 2 + 48 + 288 + 16 + 256; // size field, then codes, extra, ctrl and data at 96 / 64

struct Encoded
{
	size_t offset = 0; // in the scratch: where the stream's bytes are
	uint64_t bytes = 0;
};

bool on_device(const NvcSceneCacheWriteDesc* d, int s)
{
	return (d->device_sections >> s) & 1u;
}

uint64_t raw_bytes(const NvcSceneCacheWriteDesc* d, int s)
{
	return uint64_t(d->count[s]) * nvc::kCacheElementSize[s];
}

// vertex codec streams: header byte, blocks of 256 vertices (at most stride / 4 control bytes and per plane 4 selector
// bytes and 16 groups of 16), the tail
uint64_t vertex_stream_bound(uint64_t vertex_count, uint32_t stride)
{
	const uint64_t blocks = (vertex_count + nvc::kVertexBlockEncode - 1) / nvc::kVertexBlockEncode;
	return 1 + blocks * stride * (stride / 4 + 4 + nvc::kVertexBlockEncode) + kTailBytes;
}

uint64_t section_bound(const NvcSceneCacheWriteDesc* d, int s)
{
	if (!d->compressed)
		return raw_bytes(d, s);
	switch (s)
	{
	case NVC_CACHE_VERTICES:
		return vertex_stream_bound(d->count[s], 16);
	case NVC_CACHE_MESHLETVTX0:
		return vertex_stream_bound(d->count[s] / 4, 8);
	case NVC_CACHE_INDICES:
		return nvc::index_stream_bound(d->count[s]);
	case NVC_CACHE_MESHLETDATA:
		return uint64_t(d->count[NVC_CACHE_MESHLETS]) * kMeshletRecordBound;
	default:
		return raw_bytes(d, s);
	}
}

// a compressed section whose stream the kernels produce (it needs a context)
bool device_encoded(const NvcSceneCacheWriteDesc* d, int s)
{
	if (!d->compressed)
		return false;
	if (s == NVC_CACHE_VERTICES || s == NVC_CACHE_MESHLETVTX0)
		return d->count[s] >= (s == NVC_CACHE_VERTICES ? 1u : 4u);
	return s == NVC_CACHE_MESHLETDATA && d->count[NVC_CACHE_MESHLETS] > 0;
}

int check_desc(NvcContext* ctx, const NvcSceneCacheWriteDesc* d)
{
	bool needs_ctx = false;
	for (int s = 0; s < NVC_CACHE_SECTION_COUNT; ++s)
	{
		if (d->count[s] && !d->data[s])
			return NVC_ERROR_INVALID_ARGUMENT;
		if (on_device(d, s) && (reinterpret_cast<uintptr_t>(d->data[s]) & 3u))
			return NVC_ERROR_INVALID_ARGUMENT;
		needs_ctx = needs_ctx || on_device(d, s) || device_encoded(d, s);
	}
	if (d->device_sections >> NVC_CACHE_SECTION_COUNT)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (d->compressed && (d->count[NVC_CACHE_INDICES] % 3 || d->count[NVC_CACHE_MESHLETVTX0] % 4))
		return NVC_ERROR_INVALID_ARGUMENT;
	return needs_ctx && !ctx ? NVC_ERROR_INVALID_ARGUMENT : NVC_OK;
}

// the input of a device encoder: the caller's device pointer, or the host array copied into the scratch at `at`
const void* device_input(const NvcSceneCacheWriteDesc* d, int s, char* scratch, size_t at)
{
	return on_device(d, s) ? d->data[s] : scratch + at;
}

} // namespace

extern "C" NVC_API int nvc_scene_cache_write_bound(const NvcSceneCacheWriteDesc* desc, size_t* bytes)
{
	if (!desc || !bytes)
		return NVC_ERROR_INVALID_ARGUMENT;
	uint64_t total = sizeof(NvcSceneCacheHeader);
	for (int s = 0; s < NVC_CACHE_SECTION_COUNT; ++s)
		total += section_bound(desc, s);
	if (total > uint64_t(SIZE_MAX))
		return NVC_ERROR_UNSUPPORTED;
	*bytes = size_t(total);
	return NVC_OK;
}

extern "C" NVC_API int nvc_scene_cache_write(NvcContext* ctx, void* stream, const NvcSceneCacheWriteDesc* desc, void* file_out, size_t capacity, size_t* file_size)
{
	if (!desc || !file_out || !file_size)
		return NVC_ERROR_INVALID_ARGUMENT;
	const NvcSceneCacheWriteDesc* d = desc;
	int status = check_desc(ctx, d);
	if (status != NVC_OK)
		return status;
	size_t bound = 0;
	status = nvc_scene_cache_write_bound(d, &bound);
	if (status != NVC_OK)
		return status;
	if (capacity < bound)
		return NVC_ERROR_INVALID_ARGUMENT;
	bool uses_device = false;
	for (int s = 0; s < NVC_CACHE_SECTION_COUNT; ++s)
		uses_device = uses_device || on_device(d, s) || device_encoded(d, s);
	if (uses_device)
	{
		if (!nvc::device_is_current(ctx))
			return NVC_ERROR_INVALID_ARGUMENT;
		// the caller's work on `stream` (which produced the device arrays) and the previous user of the scratch finish first
		cudaError_t e = cudaDeviceSynchronize();
		if (e != cudaSuccess)
			return nvc::load_fail(ctx, e, "nvc_scene_cache_write");
	}
	const cudaStream_t cs = static_cast<cudaStream_t>(stream);
	Encoded enc[NVC_CACHE_SECTION_COUNT];
	std::unique_ptr<uint8_t[]> index_stream; // the bound is 17 bytes per triangle: not zero-filled before the encode
	uint32_t invalid = 0;

	if (d->compressed)
	{
		// the scratch: host inputs of the device encoders, their passes' arrays, the encoded streams
		const uint32_t vertex_sections[2] = { NVC_CACHE_VERTICES, NVC_CACHE_MESHLETVTX0 };
		nvc::ScratchPlan plan;
		size_t in_at[NVC_CACHE_SECTION_COUNT] = {};
		bool staged[NVC_CACHE_SECTION_COUNT] = {};
		for (int s : { int(NVC_CACHE_VERTICES), int(NVC_CACHE_MESHLETVTX0), int(NVC_CACHE_MESHLETS), int(NVC_CACHE_MESHLETDATA) })
		{
			const bool input = device_encoded(d, s) || (s == NVC_CACHE_MESHLETS && device_encoded(d, NVC_CACHE_MESHLETDATA));
			staged[s] = input && !on_device(d, s);
			if (staged[s])
				in_at[s] = plan.take(raw_bytes(d, s));
		}
		nvc::VertexEncodeArgs va[2];
		size_t v_est[2] = {}, v_sizes[2] = {}, v_offsets[2] = {};
		for (int i = 0; i < 2; ++i)
		{
			const int s = int(vertex_sections[i]);
			memset(&va[i], 0, sizeof(va[i]));
			if (!device_encoded(d, s))
				continue;
			va[i].vertex_count = s == NVC_CACHE_VERTICES ? d->count[s] : d->count[s] / 4;
			va[i].blocks = uint32_t((uint64_t(va[i].vertex_count) + nvc::kVertexBlockEncode - 1) / nvc::kVertexBlockEncode); // no wrap near 2^32
			v_est[i] = plan.take(sizeof(unsigned long long) * 8);
			v_sizes[i] = plan.take(size_t(va[i].blocks) * 4);
			v_offsets[i] = plan.take((size_t(va[i].blocks) + 1) * 8);
			enc[s].offset = plan.take(section_bound(d, s));
		}
		nvc::MeshletEncodeArgs ma;
		memset(&ma, 0, sizeof(ma));
		size_t m_sizes = 0, m_offsets = 0, m_flag = 0;
		const bool meshlets = device_encoded(d, NVC_CACHE_MESHLETDATA);
		if (meshlets)
		{
			ma.meshlet_count = d->count[NVC_CACHE_MESHLETS];
			ma.meshletdata_count = d->count[NVC_CACHE_MESHLETDATA];
			m_sizes = plan.take(size_t(ma.meshlet_count) * 4);
			m_offsets = plan.take((size_t(ma.meshlet_count) + 1) * 8);
			m_flag = plan.take(4);
			enc[NVC_CACHE_MESHLETDATA].offset = plan.take(section_bound(d, NVC_CACHE_MESHLETDATA));
		}

		cudaError_t e = cudaSuccess;
		char* base = nullptr;
		if (plan.bytes)
		{
			e = nvc::reserve_scratch(ctx, plan.bytes);
			base = static_cast<char*>(ctx->load_scratch);
		}
		auto input = [&](int s) { return nvc::Upload{ base + in_at[s], d->data[s], staged[s] ? size_t(raw_bytes(d, s)) : 0 }; };
		if (e == cudaSuccess && uses_device)
			e = nvc::upload({ input(NVC_CACHE_VERTICES), input(NVC_CACHE_MESHLETVTX0), input(NVC_CACHE_MESHLETS), input(NVC_CACHE_MESHLETDATA) });
		// indices in device memory come down before the kernels are queued, so that the copy does not wait for them
		std::vector<uint32_t> indices;
		const uint32_t* index_src = static_cast<const uint32_t*>(d->data[NVC_CACHE_INDICES]);
		if (e == cudaSuccess && on_device(d, NVC_CACHE_INDICES) && d->count[NVC_CACHE_INDICES])
		{
			indices.resize(d->count[NVC_CACHE_INDICES]);
			e = cudaMemcpy(indices.data(), index_src, indices.size() * 4, cudaMemcpyDeviceToHost);
			index_src = indices.data();
		}
		for (int i = 0; i < 2 && e == cudaSuccess; ++i)
		{
			const int s = int(vertex_sections[i]);
			if (!device_encoded(d, s))
				continue;
			va[i].vertices = static_cast<const uint8_t*>(device_input(d, s, base, in_at[s]));
			va[i].estimate = reinterpret_cast<unsigned long long*>(base + v_est[i]);
			va[i].block_bytes = reinterpret_cast<uint32_t*>(base + v_sizes[i]);
			va[i].offsets = reinterpret_cast<unsigned long long*>(base + v_offsets[i]);
			va[i].out = reinterpret_cast<uint8_t*>(base + enc[s].offset);
			e = nvc::launch_encode_vertices(va[i], s == NVC_CACHE_VERTICES ? 16 : 8, cs);
		}
		if (e == cudaSuccess && meshlets)
		{
			ma.meshlets = static_cast<const NvcMeshlet*>(device_input(d, NVC_CACHE_MESHLETS, base, in_at[NVC_CACHE_MESHLETS]));
			ma.meshletdata = static_cast<const uint32_t*>(device_input(d, NVC_CACHE_MESHLETDATA, base, in_at[NVC_CACHE_MESHLETDATA]));
			ma.block_bytes = reinterpret_cast<uint32_t*>(base + m_sizes);
			ma.offsets = reinterpret_cast<unsigned long long*>(base + m_offsets);
			ma.out = reinterpret_cast<uint8_t*>(base + enc[NVC_CACHE_MESHLETDATA].offset);
			ma.invalid = reinterpret_cast<uint32_t*>(base + m_flag);
			e = nvc::launch_encode_meshlets(ma, cs);
		}
		if (e != cudaSuccess)
			return nvc::load_fail(ctx, e, "nvc_scene_cache_write");

		// the index stream, on the host while the kernels run
		index_stream.reset(new uint8_t[nvc::index_stream_bound(d->count[NVC_CACHE_INDICES])]);
		enc[NVC_CACHE_INDICES].bytes = nvc::encode_index_stream(index_src, d->count[NVC_CACHE_INDICES], index_stream.get());

		if (uses_device)
			e = cudaDeviceSynchronize();
		for (int i = 0; i < 2 && e == cudaSuccess; ++i)
		{
			const int s = int(vertex_sections[i]);
			if (!device_encoded(d, s))
				continue;
			unsigned long long blocks_bytes = 0;
			e = cudaMemcpy(&blocks_bytes, va[i].offsets + va[i].blocks, 8, cudaMemcpyDeviceToHost);
			enc[s].bytes = 1 + blocks_bytes + kTailBytes;
		}
		if (e == cudaSuccess && meshlets)
		{
			unsigned long long section_bytes = 0;
			e = cudaMemcpy(&section_bytes, ma.offsets + ma.meshlet_count, 8, cudaMemcpyDeviceToHost);
			if (e == cudaSuccess)
				e = cudaMemcpy(&invalid, ma.invalid, 4, cudaMemcpyDeviceToHost);
			enc[NVC_CACHE_MESHLETDATA].bytes = section_bytes;
		}
		if (e != cudaSuccess)
			return nvc::load_fail(ctx, e, "nvc_scene_cache_write");
		if (invalid)
		{
			ctx->last_error = "nvc_scene_cache_write: a meshlet's words lie outside meshletdata, or it has more than 64 vertices or 96 triangles";
			return NVC_ERROR_INVALID_ARGUMENT;
		}
		// an empty vertex stream: the header byte and a tail of zeros (no first vertex, every channel 0)
		for (int s : { int(NVC_CACHE_VERTICES), int(NVC_CACHE_MESHLETVTX0) })
			if (!device_encoded(d, s))
				enc[s].bytes = 1 + kTailBytes;
		for (int s : { int(NVC_CACHE_VERTICES), int(NVC_CACHE_INDICES), int(NVC_CACHE_MESHLETDATA), int(NVC_CACHE_MESHLETVTX0) })
			if (enc[s].bytes > 0xffffffffull)
			{
				if (ctx)
					ctx->last_error = "nvc_scene_cache_write: a compressed stream of 4 GiB or more (the header holds 32-bit byte counts)";
				return NVC_ERROR_UNSUPPORTED;
			}
	}

	// nothing can fail from here on but a CUDA copy
	NvcSceneCacheHeader h;
	memset(&h, 0, sizeof(h));
	h.magic = NVC_SCENE_CACHE_MAGIC;
	h.version = NVC_SCENE_CACHE_VERSION;
	h.hashMeta = d->hashMeta;
	h.meshletMaxVertices = nvc::mcodec::kMaxVertices;
	h.meshletMaxTriangles = nvc::mcodec::kMaxTriangles;
	h.clrtMode = uint8_t(d->clrtMode != 0);
	h.compressed = uint8_t(d->compressed != 0);
	if (d->compressed)
	{
		h.compressedVertexBytes = uint32_t(enc[NVC_CACHE_VERTICES].bytes);
		h.compressedIndexBytes = uint32_t(enc[NVC_CACHE_INDICES].bytes);
		h.compressedMeshletDataBytes = uint32_t(enc[NVC_CACHE_MESHLETDATA].bytes);
		h.compressedMeshletVtx0Bytes = uint32_t(enc[NVC_CACHE_MESHLETVTX0].bytes);
	}
	const uint32_t* c = d->count;
	h.vertexCount = c[NVC_CACHE_VERTICES], h.indexCount = c[NVC_CACHE_INDICES], h.meshletCount = c[NVC_CACHE_MESHLETS];
	h.meshletdataCount = c[NVC_CACHE_MESHLETDATA], h.meshletvtx0Count = c[NVC_CACHE_MESHLETVTX0], h.meshCount = c[NVC_CACHE_MESHES];
	h.materialCount = c[NVC_CACHE_MATERIALS], h.drawCount = c[NVC_CACHE_DRAWS], h.texturePathCount = c[NVC_CACHE_TEXTURE_PATHS];
	h.lightCount = c[NVC_CACHE_LIGHTS], h.animationCount = c[NVC_CACHE_ANIMATIONS], h.keyframeCount = c[NVC_CACHE_KEYFRAMES];
	h.ommArrayDataSize = c[NVC_CACHE_OMM_DATA], h.ommIndexDataSize = c[NVC_CACHE_OMM_INDICES], h.ommDescCount = c[NVC_CACHE_OMM_DESCS];
	h.ommStates = d->ommStates;
	h.camera = d->camera;
	memcpy(h.sunDirection, d->sunDirection, sizeof(h.sunDirection));

	uint8_t* out = static_cast<uint8_t*>(file_out);
	memcpy(out, &h, sizeof(h));
	size_t at = sizeof(h);
	cudaError_t e = cudaSuccess;
	const char* base = static_cast<const char*>(ctx ? ctx->load_scratch : nullptr);
	for (int s = 0; s < NVC_CACHE_SECTION_COUNT && e == cudaSuccess; ++s)
	{
		const bool coded = d->compressed && (s == NVC_CACHE_VERTICES || s == NVC_CACHE_INDICES || s == NVC_CACHE_MESHLETDATA || s == NVC_CACHE_MESHLETVTX0);
		if (coded)
		{
			const size_t n = size_t(enc[s].bytes);
			if (s == NVC_CACHE_INDICES)
				memcpy(out + at, index_stream.get(), n);
			else if (device_encoded(d, s))
				e = cudaMemcpy(out + at, base + enc[s].offset, n, cudaMemcpyDeviceToHost);
			else if (n) // an empty vertex stream (an empty MESHLETDATA has no bytes)
			{
				memset(out + at, 0, n);
				out[at] = 0xa1;
			}
			at += n;
			continue;
		}
		const size_t n = size_t(raw_bytes(d, s));
		if (n && on_device(d, s))
			e = cudaMemcpy(out + at, d->data[s], n, cudaMemcpyDeviceToHost);
		else if (n)
			memcpy(out + at, d->data[s], n);
		if (s == NVC_CACHE_TEXTURE_PATHS) // strncpy(record, path, 255) into a zeroed record
			for (size_t r = 0; r < c[s]; ++r)
			{
				uint8_t* rec = out + at + r * 256;
				const size_t len = strnlen(reinterpret_cast<const char*>(rec), 255);
				memset(rec + len, 0, 256 - len);
			}
		at += n;
	}
	if (e != cudaSuccess)
		return nvc::load_fail(ctx, e, "nvc_scene_cache_write");
	*file_size = at;
	return NVC_OK;
}
