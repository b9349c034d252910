// The reference's encoders on one host thread, as saveSceneCache calls them, for tools/scene_cache_write_bench.py: reads an
// uncompressed cache, encodes VERTICES and MESHLETVTX0 (meshopt_encodeVertexBufferLevel, level 2, version 1), INDICES
// (meshopt_encodeIndexBuffer) and MESHLETDATA (per Meshlet a uint16 size and meshopt_encodeMeshlet's block, references widened
// from uint16 when shortRefs) with the functions of oracle/_ref/libmeshopt_ref.so, and writes the compressed cache those
// streams make.  It also times this library's own host index encoder (nvc::encode_index_stream, the serial part of
// nvc_scene_cache_write) on the same indices, on its own, and checks that its stream equals the reference's.  Built from the
// library's host sources by the bench.
// Usage: scene_cache_ref_encode_timer <libmeshopt_ref.so> <raw.cache> <out.z.cache> <iterations>; prints one JSON line with
// the median milliseconds of each section's encode.
#include "nvc_meshopt_format.h"

#include <memory>

#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <vector>

typedef size_t (*VertexBound)(size_t, size_t);
typedef size_t (*VertexEncode)(unsigned char*, size_t, const void*, size_t, size_t, int, int);
typedef size_t (*IndexBound)(size_t, size_t);
typedef size_t (*IndexEncode)(unsigned char*, size_t, const unsigned int*, size_t);
typedef size_t (*MeshletBound)(size_t, size_t);
typedef size_t (*MeshletEncode)(unsigned char*, size_t, const unsigned int*, size_t, const unsigned char*, size_t);

template <typename F>
static double median_ms(int iterations, F&& f)
{
	std::vector<double> t;
	for (int i = 0; i < iterations; ++i)
	{
		auto t0 = std::chrono::steady_clock::now();
		f();
		t.push_back(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
	}
	std::sort(t.begin(), t.end());
	return t[t.size() / 2];
}

static void* sym(void* lib, const char* name)
{
	void* p = dlsym(lib, name);
	if (!p)
	{
		fprintf(stderr, "%s missing\n", name);
		exit(1);
	}
	return p;
}

int main(int argc, char** argv)
{
	if (argc < 5)
	{
		fprintf(stderr, "usage: %s libmeshopt_ref.so raw.cache out.z.cache iterations\n", argv[0]);
		return 2;
	}
	void* lib = dlopen(argv[1], RTLD_NOW);
	if (!lib)
		return 1;
	VertexBound vbound = (VertexBound)sym(lib, "meshopt_encodeVertexBufferBound");
	VertexEncode vencode = (VertexEncode)sym(lib, "meshopt_encodeVertexBufferLevel");
	IndexBound ibound = (IndexBound)sym(lib, "meshopt_encodeIndexBufferBound");
	IndexEncode iencode = (IndexEncode)sym(lib, "meshopt_encodeIndexBuffer");
	MeshletBound mbound = (MeshletBound)sym(lib, "meshopt_encodeMeshletBound");
	MeshletEncode mencode = (MeshletEncode)sym(lib, "meshopt_encodeMeshlet");
	const int iterations = atoi(argv[4]);

	FILE* f = fopen(argv[2], "rb");
	if (!f)
		return 1;
	fseek(f, 0, SEEK_END);
	std::vector<unsigned char> file(size_t(ftell(f)));
	fseek(f, 0, SEEK_SET);
	if (fread(file.data(), 1, file.size(), f) != file.size())
		return 1;
	fclose(f);
	NvcSceneCacheInfo info;
	if (nvc_scene_cache_parse(file.data(), file.size(), &info) != NVC_OK || info.header.compressed)
		return 1;
	auto section = [&](int s) { return file.data() + info.sections[s].offset; };
	const NvcSceneCacheHeader& h = info.header;

	std::vector<unsigned char> streams[NVC_CACHE_SECTION_COUNT];
	auto vertex = [&](int s, size_t stride, size_t count) {
		std::vector<unsigned char>& out = streams[s];
		out.resize(vbound(count, stride));
		out.resize(vencode(out.data(), out.size(), section(s), count, stride, 2, 1));
	};
	double ms[4];
	ms[0] = median_ms(iterations, [&] { vertex(NVC_CACHE_VERTICES, 16, h.vertexCount); });
	ms[1] = median_ms(iterations, [&] {
		std::vector<unsigned char>& out = streams[NVC_CACHE_INDICES];
		out.resize(ibound(h.indexCount, ~0u));
		out.resize(iencode(out.data(), out.size(), reinterpret_cast<const unsigned int*>(section(NVC_CACHE_INDICES)), h.indexCount));
	});
	ms[2] = median_ms(iterations, [&] {
		std::vector<unsigned char>& out = streams[NVC_CACHE_MESHLETDATA];
		out.clear();
		std::vector<unsigned char> block(mbound(64, 96));
		unsigned int refs[64];
		const NvcMeshlet* meshlets = reinterpret_cast<const NvcMeshlet*>(section(NVC_CACHE_MESHLETS));
		const uint32_t* words = reinterpret_cast<const uint32_t*>(section(NVC_CACHE_MESHLETDATA));
		for (uint32_t i = 0; i < h.meshletCount; ++i)
		{
			const NvcMeshlet& m = meshlets[i];
			const uint32_t* data = words + m.dataOffset;
			const uint32_t vertex_words = m.shortRefs ? (m.vertexCount + 1) / 2 : m.vertexCount;
			const unsigned int* vertices = data;
			if (m.shortRefs)
			{
				for (uint32_t k = 0; k < m.vertexCount; ++k)
					refs[k] = reinterpret_cast<const uint16_t*>(data)[k];
				vertices = refs;
			}
			const size_t n = mencode(block.data(), block.size(), vertices, m.vertexCount, reinterpret_cast<const unsigned char*>(data + vertex_words), m.triangleCount);
			const uint16_t n16 = uint16_t(n);
			out.insert(out.end(), reinterpret_cast<const unsigned char*>(&n16), reinterpret_cast<const unsigned char*>(&n16) + 2);
			out.insert(out.end(), block.data(), block.data() + n);
		}
	});
	ms[3] = median_ms(iterations, [&] { vertex(NVC_CACHE_MESHLETVTX0, 8, h.meshletvtx0Count / 4); });
	std::unique_ptr<uint8_t[]> own(new uint8_t[nvc::index_stream_bound(h.indexCount)]);
	size_t own_size = 0;
	const double own_ms = median_ms(iterations, [&] {
		own_size = nvc::encode_index_stream(reinterpret_cast<const uint32_t*>(section(NVC_CACHE_INDICES)), h.indexCount, own.get());
	});
	const std::vector<unsigned char>& ref_indices = streams[NVC_CACHE_INDICES];
	const bool own_equal = own_size == ref_indices.size() && memcmp(own.get(), ref_indices.data(), own_size) == 0;

	NvcSceneCacheHeader z = h;
	z.compressed = 1;
	z.compressedVertexBytes = uint32_t(streams[NVC_CACHE_VERTICES].size());
	z.compressedIndexBytes = uint32_t(streams[NVC_CACHE_INDICES].size());
	z.compressedMeshletDataBytes = uint32_t(streams[NVC_CACHE_MESHLETDATA].size());
	z.compressedMeshletVtx0Bytes = uint32_t(streams[NVC_CACHE_MESHLETVTX0].size());
	FILE* o = fopen(argv[3], "wb");
	if (!o)
		return 1;
	fwrite(&z, sizeof(z), 1, o);
	for (int s = 0; s < NVC_CACHE_SECTION_COUNT; ++s)
		if (s == NVC_CACHE_VERTICES || s == NVC_CACHE_INDICES || s == NVC_CACHE_MESHLETDATA || s == NVC_CACHE_MESHLETVTX0)
			fwrite(streams[s].data(), 1, streams[s].size(), o);
		else
			fwrite(section(s), 1, info.sections[s].stored_bytes, o);
	fclose(o);
	printf("{\"vertices_ms\": %.3f, \"indices_ms\": %.3f, \"meshletdata_ms\": %.3f, \"meshletvtx0_ms\": %.3f, \"own_index_encode_ms\": %.3f, \"own_index_equal\": %s}\n",
	    ms[0], ms[1], ms[2], ms[3], own_ms, own_equal ? "true" : "false");
	return 0;
}
