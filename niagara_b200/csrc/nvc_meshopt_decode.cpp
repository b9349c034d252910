// nvc_meshopt_decode.cpp — the exported entry points of the meshopt decoders that a glTF EXT_ / KHR_meshopt_compression
// buffer view needs beyond the scene cache's (nvc_decode_vertex_stream / _index_stream / _meshlet_stream live with the cache
// reader in nvc_scene_cache.cpp): the index codec into 16- or 32-bit indices, the index-sequence codec and the vertex
// filters.  The decoders themselves are inline in nvc_meshopt_host.h (formats restated there), so that the importer links
// on its own.  Host only.
#include "../../include/niagara_cull.h"
#include "nvc_meshopt_host.h"

extern "C" NVC_API int nvc_decode_index_buffer(void* dst, uint32_t index_count, uint32_t index_size, const void* stream, size_t stream_size)
{
	if ((!dst && index_count) || !stream)
		return NVC_ERROR_INVALID_ARGUMENT;
	return nvc::decode_index_buffer(static_cast<const uint8_t*>(stream), stream_size, index_count, index_size, dst);
}

extern "C" NVC_API int nvc_decode_index_sequence(void* dst, uint32_t index_count, uint32_t index_size, const void* stream, size_t stream_size)
{
	if ((!dst && index_count) || !stream)
		return NVC_ERROR_INVALID_ARGUMENT;
	return nvc::decode_index_sequence(static_cast<const uint8_t*>(stream), stream_size, index_count, index_size, dst);
}

extern "C" NVC_API int nvc_decode_vertex_filter(int filter, void* data, uint32_t count, uint32_t stride)
{
	if ((!data && count) || !nvc::filter_stride_ok(filter, stride))
		return NVC_ERROR_INVALID_ARGUMENT;
	nvc::decode_vertex_filter(filter, static_cast<uint8_t*>(data), count, stride);
	return NVC_OK;
}
