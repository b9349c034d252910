// nvc_scene_cache_device.cpp — nvc_scene_cache_read into device memory.  The vertex streams (VERTICES, MESHLETVTX0), the
// per-meshlet stream (MESHLETDATA) and the index stream (INDICES) go up as stored, with an index the host finds by walking
// their sizes only (walk_vertex_stream, index_meshlet_stream, walk_index_stream), and are decoded by the kernels of
// nvc_cache_decode.cuh.  Raw sections are copied up.
#include "nvc_internal.h"
#include "nvc_meshopt_host.h"

#include <string.h>

#include <vector>

namespace
{

// a stored stream staged in whole words: the kernels' word loads cover its last byte and go no further
size_t staged_bytes(uint64_t stored)
{
	return size_t((stored + 3) & ~uint64_t(3));
}

int read_vertices(NvcContext* ctx, cudaStream_t stream, const uint8_t* data, const NvcSceneCacheSection& sec, uint32_t vertex_count, uint32_t stride, void* dst)
{
	const uint32_t blocks = (vertex_count + nvc::vcodec::block_vertices(stride) - 1) / nvc::vcodec::block_vertices(stride);
	std::vector<uint32_t> block_start(size_t(blocks) + 1);
	std::vector<uint16_t> plane_offset(size_t(blocks) * stride);
	nvc::VertexStreamTail tail;
	int status = nvc::walk_vertex_stream(data, sec.stored_bytes, vertex_count, stride, block_start.data(), plane_offset.data(), &tail);
	if (status != NVC_OK)
		return status;

	nvc::ScratchPlan plan; // the staged stream is taken last: a scratch allocated for this call ends where its last word does
	const size_t o_start = plan.take(block_start.size() * 4), o_plane = plan.take(plane_offset.size() * 2);
	const size_t o_carry = plan.take(size_t(blocks) * stride), o_stream = plan.take(staged_bytes(sec.stored_bytes));
	cudaError_t e = nvc::reserve_scratch(ctx, plan.bytes);
	char* base = static_cast<char*>(ctx->load_scratch);
	if (e == cudaSuccess)
		e = nvc::upload({ { base + o_stream, data, sec.stored_bytes }, { base + o_start, block_start.data(), block_start.size() * 4 },
		    { base + o_plane, plane_offset.data(), plane_offset.size() * 2 } });
	if (e != cudaSuccess)
		return nvc::load_fail(ctx, e, "nvc_scene_cache_read_device");

	nvc::VertexDecodeArgs a;
	memset(&a, 0, sizeof(a));
	a.stream = reinterpret_cast<const uint8_t*>(base + o_stream);
	a.block_start = reinterpret_cast<const uint32_t*>(base + o_start);
	a.plane_offset = reinterpret_cast<const uint16_t*>(base + o_plane);
	a.out = static_cast<uint32_t*>(dst);
	a.carry = reinterpret_cast<uint32_t*>(base + o_carry);
	a.vertex_count = vertex_count;
	a.blocks = blocks;
	a.version = uint32_t(tail.version);
	memcpy(a.baseline, tail.baseline, stride);
	for (uint32_t k = 0; k < stride / 4; ++k)
		a.channel[k] = tail.channels ? tail.channels[k] : 0u;
	e = nvc::launch_decode_vertices(a, stride, stream);
	if (e == cudaSuccess)
		e = cudaDeviceSynchronize();
	return e == cudaSuccess ? NVC_OK : nvc::load_fail(ctx, e, "nvc_scene_cache_read_device");
}

int read_meshletdata(NvcContext* ctx, cudaStream_t stream, const void* file, size_t file_size, const NvcSceneCacheInfo* info, void* dst)
{
	const NvcSceneCacheSection& sec = info->sections[NVC_CACHE_MESHLETDATA];
	const uint32_t count = info->header.meshletCount;
	std::vector<uint32_t> checkpoints((count + nvc::kMeshletGroup - 1) / nvc::kMeshletGroup + 1);
	std::vector<uint32_t> records(size_t(count) * 2);
	int status = nvc::index_meshlet_stream(file, file_size, info, checkpoints.data(), records.data());
	if (status != NVC_OK)
		return status;

	nvc::ScratchPlan plan;
	const size_t o_check = plan.take(checkpoints.size() * 4), o_records = plan.take(records.size() * 4), o_flag = plan.take(4);
	const size_t o_stream = plan.take(staged_bytes(sec.stored_bytes));
	cudaError_t e = nvc::reserve_scratch(ctx, plan.bytes);
	char* base = static_cast<char*>(ctx->load_scratch);
	if (e == cudaSuccess)
		e = nvc::upload({ { base + o_stream, static_cast<const uint8_t*>(file) + sec.offset, sec.stored_bytes }, { base + o_check, checkpoints.data(), checkpoints.size() * 4 },
		    { base + o_records, records.data(), records.size() * 4 } });
	// as the host read: bytes no meshlet writes (padding, the unused half of an odd shortRefs word) are 0
	if (e == cudaSuccess && sec.decoded_bytes)
		e = cudaMemsetAsync(dst, 0, sec.decoded_bytes, stream);
	if (e == cudaSuccess)
		e = cudaMemsetAsync(base + o_flag, 0, 4, stream);
	if (e != cudaSuccess)
		return nvc::load_fail(ctx, e, "nvc_scene_cache_read_device");

	nvc::MeshletDecodeArgs a;
	a.stream = reinterpret_cast<const uint8_t*>(base + o_stream);
	a.checkpoints = reinterpret_cast<const uint32_t*>(base + o_check);
	a.records = reinterpret_cast<const uint32_t*>(base + o_records);
	a.out = static_cast<uint32_t*>(dst);
	a.meshlet_count = count;
	a.corrupt = reinterpret_cast<uint32_t*>(base + o_flag);
	e = nvc::launch_decode_meshlets(a, stream);
	if (e == cudaSuccess)
		e = cudaDeviceSynchronize();
	uint32_t corrupt = 0;
	if (e == cudaSuccess)
		e = cudaMemcpy(&corrupt, a.corrupt, 4, cudaMemcpyDeviceToHost);
	if (e != cudaSuccess)
		return nvc::load_fail(ctx, e, "nvc_scene_cache_read_device");
	return corrupt ? NVC_ERROR_CORRUPT : NVC_OK;
}

int read_indices(NvcContext* ctx, cudaStream_t stream, const uint8_t* data, const NvcSceneCacheSection& sec, void* dst)
{
	const uint32_t triangles = sec.count / 3, chunks = (triangles + nvc::kIndexChunk - 1) / nvc::kIndexChunk;
	const uint32_t runs = (chunks + nvc::kIndexRun - 1) / nvc::kIndexRun;
	std::vector<uint64_t> chunk_data(chunks);
	const int version = nvc::walk_index_stream(data, sec.stored_bytes, sec.count, nvc::kIndexChunk, chunk_data.data());
	if (version < 0)
		return version;
	if (chunks == 0)
		return NVC_OK;

	nvc::ScratchPlan plan; // the staged stream is taken last: a scratch allocated for this call ends where its last word does
	const size_t o_data = plan.take(chunk_data.size() * 8), o_sub = plan.take(size_t(chunks) * nvc::kIndexEntries * 8);
	const size_t o_run = plan.take(size_t(runs) * nvc::kIndexEntries * 8), o_stream = plan.take(staged_bytes(sec.stored_bytes));
	cudaError_t e = nvc::reserve_scratch(ctx, plan.bytes);
	char* base = static_cast<char*>(ctx->load_scratch);
	if (e == cudaSuccess)
		e = nvc::upload({ { base + o_stream, data, sec.stored_bytes }, { base + o_data, chunk_data.data(), chunk_data.size() * 8 } });
	if (e != cudaSuccess)
		return nvc::load_fail(ctx, e, "nvc_scene_cache_read_device");

	nvc::IndexDecodeArgs a;
	a.stream = reinterpret_cast<const uint8_t*>(base + o_stream);
	a.chunk_data = reinterpret_cast<const uint64_t*>(base + o_data);
	a.sub = reinterpret_cast<uint2*>(base + o_sub);
	a.run = reinterpret_cast<uint2*>(base + o_run);
	a.out = static_cast<uint32_t*>(dst);
	a.aux_offset = sec.stored_bytes - 16;
	a.triangles = triangles;
	a.chunks = chunks;
	a.runs = runs;
	a.direct_slots = nvc::index_direct_slots(version);
	e = nvc::launch_decode_indices(a, stream);
	if (e == cudaSuccess)
		e = cudaDeviceSynchronize();
	return e == cudaSuccess ? NVC_OK : nvc::load_fail(ctx, e, "nvc_scene_cache_read_device");
}

} // namespace

extern "C" NVC_API int nvc_scene_cache_read_device(NvcContext* ctx, void* stream, const void* file, size_t file_size, const NvcSceneCacheInfo* info, int section, void* dst,
    size_t dst_bytes)
{
	if (!ctx || !file || !info || section < 0 || section >= NVC_CACHE_SECTION_COUNT || (!dst && dst_bytes) || (reinterpret_cast<uintptr_t>(dst) & 3u))
		return NVC_ERROR_INVALID_ARGUMENT;
	const NvcSceneCacheSection& sec = info->sections[section];
	if (dst_bytes < sec.decoded_bytes || sec.offset > file_size || sec.stored_bytes > file_size - sec.offset)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!nvc::device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	const uint8_t* data = static_cast<const uint8_t*>(file) + sec.offset;
	const cudaStream_t s = static_cast<cudaStream_t>(stream);
	// the caller's earlier work on `stream` and the previous user of the scratch finish before the copies below, which are not
	// ordered with `stream` (nvc::upload)
	cudaError_t e = cudaDeviceSynchronize();
	if (e != cudaSuccess)
		return nvc::load_fail(ctx, e, "nvc_scene_cache_read_device");

	if (!sec.compressed)
	{
		if (sec.decoded_bytes > sec.stored_bytes)
			return NVC_ERROR_INVALID_ARGUMENT;
		e = nvc::upload({ { dst, data, sec.decoded_bytes } });
		return e == cudaSuccess ? NVC_OK : nvc::load_fail(ctx, e, "nvc_scene_cache_read_device");
	}
	// the vertex and meshlet kernels and their indexes address the staged stream with 32-bit offsets (the index kernels' chunk
	// offsets are 64-bit: a triangle takes up to 15 data bytes)
	if (section != NVC_CACHE_INDICES && sec.stored_bytes > 0xffffffffull)
		return NVC_ERROR_UNSUPPORTED;
	if (section == NVC_CACHE_VERTICES)
		return read_vertices(ctx, s, data, sec, sec.count, 16, dst);
	if (section == NVC_CACHE_MESHLETVTX0) // uint16 x 4 per element of the stream
		return sec.count % 4 ? NVC_ERROR_CORRUPT : read_vertices(ctx, s, data, sec, sec.count / 4, 8, dst);
	if (section == NVC_CACHE_INDICES)
		return read_indices(ctx, s, data, sec, dst);
	if (section != NVC_CACHE_MESHLETDATA)
		return NVC_ERROR_UNSUPPORTED;
	return read_meshletdata(ctx, s, file, file_size, info, dst);
}
