// TEST INFRASTRUCTURE (oracle side): the reference's own importer and scene-cache writer run as a CLRT=1 run of the reference
// runs them (niagara.cpp:844): loadMesh / loadScene with clrt = true, so the cooker builds each mesh's lodRT with
// meshopt_buildMeshletsSpatial and fills meshletvtx0 (scene.cpp:52-67,102-103,266-276), and saveSceneCache / loadSceneCache
// with clrtMode = true.  The reference sources are compiled where they lie (see Makefile); nothing is copied.  The fixtures
// of nvc_cook_meshlets_clrt come from here (tests/golden/make_meshlet_clrt_fixtures.py).
//
//   write_cache_clrt <prefix> input.{obj,gltf,glb}...
//     <prefix>.raw.cache   saveSceneCache(..., clrtMode = true, compressed = false)
//     <prefix>.z.cache     saveSceneCache(..., clrtMode = true, compressed = true), read back by the reference's loadSceneCache
//                          with clrtMode = true and checked equal to what was saved (Meshlet[], meshletvtx0, Vertex[], MeshDraw[])
#include "../refscene/scene_arrays.h"

#include <stdio.h>

int main(int argc, char** argv)
{
	if (argc < 3)
	{
		fprintf(stderr, "usage: %s prefix input.{obj,gltf,glb}...\n", argv[0]);
		return 2;
	}

	SceneArrays in;
	in.cam.orientation = quat(1, 0, 0, 0);
	in.cam.fovY = glm::radians(70.f);
	in.cam.znear = 0.1f;
	in.sun = normalize(vec3(1.0f, 1.0f, 1.0f));
	for (int i = 2; i < argc; ++i)
	{
		size_t firstMesh = in.geo.meshes.size();
		const char* ext = strrchr(argv[i], '.');
		bool scene = ext && (strcmp(ext, ".gltf") == 0 || strcmp(ext, ".glb") == 0);
		bool ok = scene ? loadScene(in.geo, in.mats, in.draws, in.lights, in.textures, in.tracks, in.keys, in.cam, in.sun, argv[i], true)
		                : loadMesh(in.geo, argv[i], true);
		if (!ok)
		{
			fprintf(stderr, "failed to load %s\n", argv[i]);
			return 1;
		}
		if (!scene) // a bare mesh: one identity draw per mesh
			for (size_t m = firstMesh; m < in.geo.meshes.size(); ++m)
			{
				MeshDraw draw = {};
				draw.scale = 1.f;
				draw.orientation = quat(1, 0, 0, 0);
				draw.meshIndex = uint32_t(m);
				in.draws.push_back(draw);
			}
	}

	// meshletVisibilityOffset as niagara.cpp:1003-1020 assigns it
	uint32_t meshletVisibilityCount = 0;
	for (MeshDraw& draw : in.draws)
	{
		const Mesh& mesh = in.geo.meshes[draw.meshIndex];
		draw.meshletVisibilityOffset = meshletVisibilityCount;
		uint32_t meshletCount = 0;
		for (uint32_t l = 0; l < mesh.lodCount; ++l)
			meshletCount = std::max(meshletCount, mesh.lods[l].meshletCount);
		meshletVisibilityCount += meshletCount;
	}

	std::string prefix = argv[1];
	const uint64_t hashMeta = 0x0123456789abcdefull;
	if (!saveSceneCache((prefix + ".raw.cache").c_str(), in.geo, in.mats, in.draws, in.lights, in.textures, in.tracks, in.keys, in.cam, in.sun, hashMeta, true, false, false) ||
	    !saveSceneCache((prefix + ".z.cache").c_str(), in.geo, in.mats, in.draws, in.lights, in.textures, in.tracks, in.keys, in.cam, in.sun, hashMeta, true, true, false))
	{
		fprintf(stderr, "saveSceneCache failed\n");
		return 1;
	}

	Geometry g2;
	std::vector<Material> m2;
	std::vector<MeshDraw> d2;
	std::vector<Light> l2;
	std::vector<std::string> t2;
	std::vector<Animation> a2;
	std::vector<Keyframe> k2;
	Camera c2 = {};
	vec3 s2(0.f);
	if (!loadSceneCache((prefix + ".z.cache").c_str(), g2, m2, d2, l2, t2, a2, k2, c2, s2, hashMeta, true, 0))
	{
		fprintf(stderr, "loadSceneCache failed\n");
		return 1;
	}
	const Geometry& g = in.geo;
	if (g2.meshlets.size() != g.meshlets.size() || memcmp(g2.meshlets.data(), g.meshlets.data(), g.meshlets.size() * sizeof(Meshlet)) != 0 ||
	    g2.meshletvtx0 != g.meshletvtx0 || d2.size() != in.draws.size() || memcmp(d2.data(), in.draws.data(), d2.size() * sizeof(MeshDraw)) != 0 ||
	    g2.vertices.size() != g.vertices.size() || memcmp(g2.vertices.data(), g.vertices.data(), g.vertices.size() * sizeof(Vertex)) != 0)
	{
		fprintf(stderr, "round trip mismatch\n");
		return 1;
	}

	printf("%s: meshes %zu meshlets %zu meshletdata %zu meshletvtx0 %zu vertices %zu indices %zu\n", prefix.c_str(), g.meshes.size(), g.meshlets.size(),
	    g.meshletdata.size(), g.meshletvtx0.size(), g.vertices.size(), g.indices.size());
	return 0;
}
