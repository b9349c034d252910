// Times the host walks of nvc_scene_cache_read_device on their own: walk_vertex_stream over VERTICES,
// walk_index_stream over INDICES and index_meshlet_stream over MESHLETDATA, the serial part of the device read.  Built
// from the library's host sources by tools/scene_cache_device_bench.py.  Usage: scene_cache_walk_timer <file.cache> <iterations>; prints one JSON line with
// the median milliseconds of each walk.
#include "nvc_meshopt_host.h"

#include <algorithm>
#include <chrono>
#include <stdio.h>
#include <stdlib.h>
#include <vector>

template <typename F>
static double median_ms(int iterations, F&& f)
{
	std::vector<double> t;
	for (int i = 0; i < iterations; ++i)
	{
		auto t0 = std::chrono::steady_clock::now();
		if (f() < 0)
		{
			fprintf(stderr, "walk failed\n");
			exit(1);
		}
		t.push_back(std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count());
	}
	std::sort(t.begin(), t.end());
	return t[t.size() / 2];
}

int main(int argc, char** argv)
{
	if (argc != 3)
		return 2;
	FILE* f = fopen(argv[1], "rb");
	if (!f)
		return 2;
	std::vector<uint8_t> file;
	uint8_t buf[1 << 16];
	for (size_t n; (n = fread(buf, 1, sizeof(buf), f)) > 0;)
		file.insert(file.end(), buf, buf + n);
	fclose(f);
	NvcSceneCacheInfo info;
	if (nvc_scene_cache_parse(file.data(), file.size(), &info) != NVC_OK)
		return 3;
	const int iterations = atoi(argv[2]);
	const NvcSceneCacheSection& v = info.sections[NVC_CACHE_VERTICES];
	const uint32_t blocks = (v.count + 255) / 256;
	std::vector<uint32_t> starts(blocks + 1);
	std::vector<uint16_t> planes(size_t(blocks) * 16);
	nvc::VertexStreamTail tail;
	double vertex_ms = median_ms(iterations, [&] { return nvc::walk_vertex_stream(file.data() + v.offset, v.stored_bytes, v.count, 16, starts.data(), planes.data(), &tail); });
	const uint32_t meshlets = info.header.meshletCount;
	std::vector<uint32_t> checkpoints((meshlets + nvc::kMeshletGroup - 1) / nvc::kMeshletGroup + 1), records(size_t(meshlets) * 2);
	double meshlet_ms = median_ms(iterations, [&] { return nvc::index_meshlet_stream(file.data(), file.size(), &info, checkpoints.data(), records.data()); });
	const NvcSceneCacheSection& x = info.sections[NVC_CACHE_INDICES];
	const uint32_t chunk = 256; // the device decoder's kIndexChunk (nvc_internal.h)
	std::vector<uint64_t> chunk_data((x.count / 3 + chunk - 1) / chunk);
	double index_ms = x.count ? median_ms(iterations, [&] { return nvc::walk_index_stream(file.data() + x.offset, x.stored_bytes, x.count, chunk, chunk_data.data()); }) : 0.0;
	printf("{\"vertices_walk_ms\": %.3f, \"indices_walk_ms\": %.3f, \"meshletdata_walk_ms\": %.3f}\n", vertex_ms, index_ms, meshlet_ms);
	return 0;
}
