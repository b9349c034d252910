// nvc_meshlets.cuh — meshlet building and packing, SURVEY §8(f) row N4 (the producer of Meshlet[] and meshletdata).
//
// Restates what the reference's cooker does per LOD (src/scene.cpp:90-115 appendMeshlets with clrt off ->
// meshopt_buildMeshlets(max_vertices 64, max_triangles 96, cone_weight 0.25) = meshopt_buildMeshletsFlex with
// min_triangles = max_triangles and split_factor 0, extern/meshoptimizer/src/clusterizer.cpp:40-639,1035-1229; then per
// meshlet meshopt_optimizeMeshletLevel(level 1), meshletutils.cpp:366-553; then the packing of scene.cpp:24-88) with the
// same operations in the same order, so that the meshlets, their vertex and triangle order and every float that decides
// a choice are BIT-IDENTICAL to the reference's.  Arithmetic is spelled through cook::mul/add/... (nvc_cook.cuh).
//
// Work split (kernels in nvc_kernels.cu):
//   build      one warp per (mesh, LOD) job: triangle cones (lanes), adjacency (lane scan + a stable sequential fill),
//              kd-tree (sequential), then the greedy loop.  Each step's candidate scan (meshlet vertices x their live
//              adjacency) is shared by the lanes and reduced with keys (priority, score, scan position), which gives the
//              reference's first-strict-minimum.  Seeds, kd-tree search and the meshlet append are sequential in lane 0.
//   optimize   one thread per meshlet: optimizeMeshletLevel(level 1), then minVertex / shortRefs / word count.
//   scan       one block: LOD meshlet offsets and meshlet data offsets in job order.
//   pack       one thread per meshlet: Meshlet record + meshletdata words, then cook::meshlet_bounds on them.
#pragma once

#include "nvc_cook.cuh"

namespace nvc
{
namespace cook
{

constexpr uint32_t kMaxVertices = 64;  // MESH_MAXVTX (config.h)
constexpr uint32_t kMaxTriangles = 96; // MESH_MAXTRI (config.h)
constexpr float kConeWeight = 0.25f;   // MESHLET_CONE_WEIGHT (config.h)
constexpr uint32_t kMaxSeeds = 256;    // clusterizer.cpp:27-28
constexpr uint32_t kAddSeeds = 4;
constexpr uint32_t kLeafSize = 8;      // kdtreeBuild leaf_size (clusterizer.cpp:1082)
constexpr int kMaxTreeDepth = 50;      // clusterizer.cpp:31
constexpr uint32_t kNone = ~0u;

// One (mesh, LOD) of the call.  Offsets place the job's scratch: triangles, vertices, indices and meshlet slots.
struct CookJob
{
	uint32_t mesh, lod;
	uint32_t index_offset, index_count; // lods[lod], into the call's index buffer (mesh-local indices)
	uint32_t vertex_offset, vertex_count; // the mesh's, into the call's Vertex[]
	uint64_t tri, vtx, idx, slot;
};

// meshopt_buildMeshletsBound(index_count, 64, 96) (clusterizer.cpp:1017-1033)
NVC_HD uint64_t meshlets_bound(uint64_t index_count)
{
	uint64_t by_vertices = (index_count + (kMaxVertices - 2) - 1) / (kMaxVertices - 2);
	uint64_t by_triangles = (index_count / 3 + kMaxTriangles - 1) / kMaxTriangles;
	return by_vertices > by_triangles ? by_vertices : by_triangles;
}

// Words an LOD can need: the references of its meshlets are at most one per index (each meshlet vertex is added by a
// triangle corner), and sum((3 t + 3) / 4) <= index_count / 4 + meshlets.
NVC_HD uint64_t words_bound(uint64_t index_count) { return index_count + (index_count + 3) / 4 + meshlets_bound(index_count); }

// clusterizer.cpp:167-171; the cones array holds 6 floats per triangle in this order
struct Cone
{
	float px, py, pz, nx, ny, nz;
};

// clusterizer.cpp:201-241 for one triangle; returns its area (the caller sums the areas in triangle order)
NVC_HD float triangle_cone(V3 p0, V3 p1, V3 p2, Cone& t)
{
	float p10x = sub(p1.x, p0.x), p10y = sub(p1.y, p0.y), p10z = sub(p1.z, p0.z);
	float p20x = sub(p2.x, p0.x), p20y = sub(p2.y, p0.y), p20z = sub(p2.z, p0.z);
	float nx = sub(mul(p10y, p20z), mul(p10z, p20y));
	float ny = sub(mul(p10z, p20x), mul(p10x, p20z));
	float nz = sub(mul(p10x, p20y), mul(p10y, p20x));
	float area = root(add(add(mul(nx, nx), mul(ny, ny)), mul(nz, nz)));
	float invarea = area == 0.0f ? 0.0f : div(1.0f, area);
	t.px = div(add(add(p0.x, p1.x), p2.x), 3.0f);
	t.py = div(add(add(p0.y, p1.y), p2.y), 3.0f);
	t.pz = div(add(add(p0.z, p1.z), p2.z), 3.0f);
	t.nx = mul(nx, invarea);
	t.ny = mul(ny, invarea);
	t.nz = mul(nz, invarea);
	return area;
}

// clusterizer.cpp:181-199
NVC_HD Cone meshlet_cone(const Cone& acc, uint32_t triangle_count)
{
	Cone r = acc;
	float center_scale = triangle_count == 0 ? 0.0f : div(1.0f, float(triangle_count));
	r.px = mul(r.px, center_scale);
	r.py = mul(r.py, center_scale);
	r.pz = mul(r.pz, center_scale);
	float axis_length = add(add(mul(r.nx, r.nx), mul(r.ny, r.ny)), mul(r.nz, r.nz));
	float axis_scale = axis_length == 0.0f ? 0.0f : div(1.0f, root(axis_length));
	r.nx = mul(r.nx, axis_scale);
	r.ny = mul(r.ny, axis_scale);
	r.nz = mul(r.nz, axis_scale);
	return r;
}

// clusterizer.cpp:173-179 with cone_weight 0.25 (1 - cone_weight = 0.75 exactly)
NVC_HD float meshlet_score(float distance, float spread, float expected_radius)
{
	float cone = sub(1.0f, mul(spread, kConeWeight));
	float cone_clamped = cone < 1e-3f ? 1e-3f : cone;
	return mul(add(1.0f, mul(div(distance, expected_radius), 1.0f - kConeWeight)), cone_clamped);
}

NVC_HD float point_distance(const float* p, float x, float y, float z)
{
	float dx = sub(p[0], x), dy = sub(p[1], y), dz = sub(p[2], z);
	return root(add(add(mul(dx, dx), mul(dy, dy)), mul(dz, dz)));
}

// kd-tree nodes: 3 words each {index or split bits, axis (3 = leaf), children} (clusterizer.cpp:473-485)
NVC_HD void kd_leaf(uint32_t* nodes, uint32_t offset, const uint32_t* idx, uint32_t count)
{
	nodes[3 * offset + 0] = idx[0];
	nodes[3 * offset + 1] = 3;
	nodes[3 * offset + 2] = count;
	for (uint32_t i = 1; i < count; ++i)
	{
		nodes[3 * (offset + i) + 0] = idx[i];
		nodes[3 * (offset + i) + 1] = 3;
		nodes[3 * (offset + i) + 2] = ~0u >> 2;
	}
}

// kdtreeBuild + kdtreePartition (clusterizer.cpp:487-581), with the recursion unrolled: the left subtree follows its node,
// and the pending right subtrees are kept on a stack.  count > 0.
NVC_HD void kd_build(uint32_t* nodes, const float* cones, uint32_t* idx, uint32_t count)
{
	uint32_t stack_parent[kMaxTreeDepth + 2], stack_start[kMaxTreeDepth + 2], stack_count[kMaxTreeDepth + 2];
	int stack_depth[kMaxTreeDepth + 2];
	int sp = 0;
	uint32_t offset = 0, start = 0, n = count;
	int depth = 0;
	for (;;)
	{
		uint32_t* ind = idx + start;
		bool leaf = n <= kLeafSize;
		uint32_t middle = 0;
		int axis = 0;
		float split = 0.0f;
		if (!leaf)
		{
			float mean[3] = { 0.0f, 0.0f, 0.0f }, vars[3] = { 0.0f, 0.0f, 0.0f };
			float runc = 1.0f, runs = 1.0f;
			for (uint32_t i = 0; i < n; ++i, runc = add(runc, 1.0f), runs = div(1.0f, runc))
			{
				const float* point = cones + size_t(ind[i]) * 6u;
				for (int k = 0; k < 3; ++k)
				{
					float delta = sub(point[k], mean[k]);
					mean[k] = add(mean[k], mul(delta, runs));
					vars[k] = add(vars[k], mul(delta, sub(point[k], mean[k])));
				}
			}
			axis = (vars[0] >= vars[1] && vars[0] >= vars[2]) ? 0 : (vars[1] >= vars[2] ? 1 : 2);
			split = mean[axis];
			for (uint32_t i = 0; i < n; ++i)
			{
				float v = cones[size_t(ind[i]) * 6u + axis];
				uint32_t t = ind[middle];
				ind[middle] = ind[i];
				ind[i] = t;
				middle += v < split;
			}
			leaf = middle <= kLeafSize / 2 || middle >= n - kLeafSize / 2 || depth >= kMaxTreeDepth;
		}
		if (!leaf)
		{
			nodes[3 * offset + 0] = float_bits(split);
			nodes[3 * offset + 1] = uint32_t(axis);
			stack_parent[sp] = offset;
			stack_start[sp] = start + middle;
			stack_count[sp] = n - middle;
			stack_depth[sp] = depth + 1;
			++sp;
			offset += 1;
			n = middle;
			depth += 1;
			continue;
		}
		kd_leaf(nodes, offset, ind, n);
		uint32_t next = offset + n;
		if (sp == 0)
			return;
		--sp;
		nodes[3 * stack_parent[sp] + 2] = next - stack_parent[sp] - 1;
		offset = next;
		start = stack_start[sp];
		n = stack_count[sp];
		depth = stack_depth[sp];
	}
}

// kdtreeNearest (clusterizer.cpp:583-639), the recursion unrolled: the second child of every branch is kept on a stack
// with its delta and visited when it is popped and fabsf(delta) <= limit at that time, as after the reference's first call
// returns.  Deactivates emptied leaves and branches as the reference does.
NVC_HD void kd_nearest(uint32_t* nodes, const float* cones, const uint8_t* emitted, const float* position, uint32_t& result, float& limit)
{
	uint32_t stack_node[kMaxTreeDepth + 2];
	float stack_delta[kMaxTreeDepth + 2];
	int sp = 0;
	uint32_t root = 0;
	for (;;)
	{
		uint32_t* node = nodes + 3 * size_t(root);
		bool descend = false;
		if (node[2] != 0)
		{
			if (node[1] == 3)
			{
				bool inactive = true;
				for (uint32_t i = 0; i < node[2]; ++i)
				{
					uint32_t index = nodes[3 * size_t(root + i)];
					if (emitted[index])
						continue;
					inactive = false;
					float distance = point_distance(cones + size_t(index) * 6u, position[0], position[1], position[2]);
					if (distance < limit)
					{
						result = index;
						limit = distance;
					}
				}
				if (inactive)
					node[2] = 0;
			}
			else
			{
				float delta = sub(position[node[1]], bits_float(node[0]));
				uint32_t first = delta <= 0 ? 0 : node[2];
				uint32_t second = first ^ node[2];
				if ((nodes[3 * size_t(root + 1 + first) + 2] | nodes[3 * size_t(root + 1 + second) + 2]) == 0)
					node[2] = 0;
				stack_node[sp] = root + 1 + second;
				stack_delta[sp] = delta;
				++sp;
				root = root + 1 + first;
				descend = true;
			}
		}
		if (descend)
			continue;
		for (;;)
		{
			if (sp == 0)
				return;
			--sp;
			if (fabsf(stack_delta[sp]) <= limit)
			{
				root = stack_node[sp];
				break;
			}
		}
	}
}

// One meshlet in the making (meshopt_Meshlet): offsets into the job's meshlet_vertices / meshlet_triangles
struct Building
{
	uint32_t vertex_offset, triangle_offset, vertex_count, triangle_count;
};

// appendMeshlet (clusterizer.cpp:243-300) with max_vertices 64, max_triangles 96, split false.  `used` entries are
// referenced, not copied: a triangle with a repeated vertex sees its own update, as in the reference.
NVC_HD bool append_triangle(Building& m, uint32_t a, uint32_t b, uint32_t c, int16_t* used, uint4* records, uint32_t meshlet_offset,
    uint32_t* meshlet_vertices, uint8_t* meshlet_triangles)
{
	int16_t& av = used[a];
	int16_t& bv = used[b];
	int16_t& cv = used[c];
	bool result = false;
	int used_extra = (av < 0) + (bv < 0) + (cv < 0);
	if (m.vertex_count + used_extra > kMaxVertices || m.triangle_count >= kMaxTriangles)
	{
		records[meshlet_offset] = make_uint4(m.vertex_offset, m.triangle_offset, m.vertex_count, m.triangle_count);
		for (uint32_t j = 0; j < m.vertex_count; ++j)
			used[meshlet_vertices[m.vertex_offset + j]] = -1;
		m.vertex_offset += m.vertex_count;
		m.triangle_offset += m.triangle_count * 3;
		m.vertex_count = 0;
		m.triangle_count = 0;
		result = true;
	}
	if (av < 0)
	{
		av = int16_t(m.vertex_count);
		meshlet_vertices[m.vertex_offset + m.vertex_count++] = a;
	}
	if (bv < 0)
	{
		bv = int16_t(m.vertex_count);
		meshlet_vertices[m.vertex_offset + m.vertex_count++] = b;
	}
	if (cv < 0)
	{
		cv = int16_t(m.vertex_count);
		meshlet_vertices[m.vertex_offset + m.vertex_count++] = c;
	}
	meshlet_triangles[m.triangle_offset + m.triangle_count * 3 + 0] = uint8_t(av);
	meshlet_triangles[m.triangle_offset + m.triangle_count * 3 + 1] = uint8_t(bv);
	meshlet_triangles[m.triangle_offset + m.triangle_count * 3 + 2] = uint8_t(cv);
	m.triangle_count++;
	return result;
}

// selectSeedTriangle (clusterizer.cpp:447-471)
NVC_HD uint32_t select_seed(const uint32_t* seeds, uint32_t seed_count, const uint32_t* indices, const float* cones, const uint32_t* live,
    const float* corner)
{
	uint32_t best_seed = kNone, best_live = kNone;
	float best_score = FLT_MAX;
	for (uint32_t i = 0; i < seed_count; ++i)
	{
		uint32_t index = seeds[i];
		uint32_t l = live[indices[index * 3 + 0]] + live[indices[index * 3 + 1]] + live[indices[index * 3 + 2]];
		float score = point_distance(cones + size_t(index) * 6u, corner[0], corner[1], corner[2]);
		if (l < best_live || (l == best_live && score < best_score))
		{
			best_seed = index;
			best_live = l;
			best_score = score;
		}
	}
	return best_seed;
}

// meshopt_optimizeMeshletLevel(level 1) (meshletutils.cpp:366-553) on one meshlet, in place
NVC_HD void optimize_meshlet(uint32_t* vertices, uint32_t vertex_count, uint8_t* indices, uint32_t triangle_count)
{
	const int level = 1;
	uint8_t cache[kMaxVertices], valence[kMaxVertices];
	for (uint32_t i = 0; i < vertex_count; ++i)
		cache[i] = valence[i] = 0;
	uint8_t cache_last = 128;
	const uint8_t cache_cutoff = 3;
	for (uint32_t i = 0; i < triangle_count * 3; ++i)
		valence[indices[i]]++;

	for (uint32_t i = 0; i < triangle_count; ++i)
	{
		int next = -1, next_score = -1, edges = 0;
		for (uint32_t j = i; j < triangle_count; ++j)
		{
			uint8_t a = indices[j * 3 + 0], b = indices[j * 3 + 1], c = indices[j * 3 + 2];
			uint8_t ad = uint8_t(cache_last - cache[a]), bd = uint8_t(cache_last - cache[b]), cd = uint8_t(cache_last - cache[c]);
			int match = (ad < cache_cutoff) + (bd < cache_cutoff) + (cd < cache_cutoff);
			int vmin = valence[a] < valence[b] ? valence[a] : valence[b];
			vmin = valence[c] < vmin ? valence[c] : vmin;
			int score = match * 1024 + (1023 - ad - bd - cd);
			score = score * 256 + (255 - vmin);
			next = (score > next_score) ? int(j) : next;
			next_score = (score > next_score) ? score : next_score;
			if (match >= 2 && ++edges >= level)
				break;
		}
		uint8_t a = indices[next * 3 + 0], b = indices[next * 3 + 1], c = indices[next * 3 + 2];
		for (uint32_t k = uint32_t(next) * 3; k > i * 3; --k) // memmove of triangles [i, next) one slot up
			indices[k + 2] = indices[k - 1];
		indices[i * 3 + 0] = a;
		indices[i * 3 + 1] = b;
		indices[i * 3 + 2] = c;
		cache_last++;
		cache[a] = cache_last;
		cache[b] = cache_last;
		cache[c] = cache_last;
		valence[a]--;
		valence[b]--;
		valence[c]--;
	}

	for (uint32_t i = 0; i < vertex_count; ++i)
		cache[i] = 0;
	for (uint32_t i = 0; i < triangle_count; ++i)
	{
		uint8_t a = indices[i * 3 + 0], b = indices[i * 3 + 1], c = indices[i * 3 + 2];
		if (!cache[a] && cache[b] && !cache[c])
		{
			uint8_t t = a;
			a = b, b = c, c = t;
		}
		else if (!cache[a] && !cache[b] && !cache[c])
		{
			bool needab = false, needbc = false, needca = false;
			for (uint32_t j = i + 1; j < triangle_count && j <= i + cache_cutoff; ++j)
			{
				uint8_t oa = indices[j * 3 + 0], ob = indices[j * 3 + 1], oc = indices[j * 3 + 2];
				needab |= (oa == b && ob == a) || (ob == b && oc == a) || (oc == b && oa == a);
				needbc |= (oa == c && ob == b) || (ob == c && oc == b) || (oc == c && oa == b);
				needca |= (oa == a && ob == c) || (ob == a && oc == c) || (oc == a && oa == c);
			}
			if (needab && !needbc)
			{
				uint8_t t = a;
				a = b, b = c, c = t;
			}
			else if ((needab && !needca) || (!needab && needbc && !needca))
			{
				uint8_t t = c;
				c = b, b = a, a = t;
			}
		}
		indices[i * 3 + 0] = a, indices[i * 3 + 1] = b, indices[i * 3 + 2] = c;
		cache[a] = cache[b] = cache[c] = 1;
	}

	uint32_t order[kMaxVertices];
	int16_t remap[kMaxVertices];
	for (uint32_t i = 0; i < vertex_count; ++i)
		remap[i] = -1;
	uint32_t vertex_offset = 0;
	for (uint32_t i = 0; i < triangle_count * 3; ++i)
	{
		int16_t& r = remap[indices[i]];
		if (r < 0)
		{
			r = int16_t(vertex_offset);
			order[vertex_offset] = vertices[indices[i]];
			vertex_offset++;
		}
		indices[i] = uint8_t(r);
	}
	for (uint32_t i = 0; i < vertex_offset; ++i)
		vertices[i] = order[i];
}

// ---- clrt builds: the ray-tracing LOD (scene.cpp:102-103) -----------------------------------------------------------------
// meshopt_buildMeshletsSpatial(max_vertices 64, min_triangles 24, max_triangles 96, fill_weight 0.5), clusterizer.cpp:640-1013,
// 1266-1365, as compiled for x86-64 (SIMD_SSE).  The sort, the box scans, the pivot search and the partitions are warp-parallel
// in the kernel (nvc_kernels.cu); what is sequential there is spelled here.  Since min_triangles != max_triangles, bvhSplit's
// pivot step is always 1.

constexpr uint32_t kSpatialMinTriangles = kMaxTriangles / 4; // MESH_MAXTRI / 4 (scene.cpp:93)
constexpr float kFillWeight = 0.5f;                           // MESHLET_FILL_WEIGHT (config.h)
constexpr float kShadowLodError = 3e-3f;                      // scene.cpp:22, the lodRT threshold
constexpr uint32_t kSpatialLeafSplit = kMaxVertices / 3;      // bvhPackTail's chunk of a vertex-bound run, and bvhSplit's mint

// scene.cpp:266-268, run in every build: the last LOD with error * maxScale < kShadowLodError (0 when none is), with the
// reference's float multiply
NVC_HD uint32_t lod_rt(const NvcMesh& mesh, float max_scale)
{
	uint32_t rt = 0;
	for (uint32_t i = 0; i < mesh.lodCount; ++i)
		if (mesh.lods[i].error * max_scale < kShadowLodError)
			rt = i;
	return rt;
}

// meshopt_buildMeshletsBound(index_count, 64, 24): the meshlet array the reference sizes for every LOD (scene.cpp:98)
NVC_HD uint64_t spatial_meshlets_bound(uint64_t index_count)
{
	uint64_t by_vertices = (index_count + (kMaxVertices - 2) - 1) / (kMaxVertices - 2);
	uint64_t by_triangles = (index_count / 3 + kSpatialMinTriangles - 1) / kSpatialMinTriangles;
	return by_vertices > by_triangles ? by_vertices : by_triangles;
}

// as words_bound, with the spatial meshlet bound
NVC_HD uint64_t spatial_words_bound(uint64_t index_count) { return index_count + (index_count + 3) / 4 + spatial_meshlets_bound(index_count); }

// the SSE boxMerge per component: _mm_min_ps / _mm_max_ps return the second operand (the merged box) on ties and NaN
NVC_HD float box_min(float box, float other) { return box < other ? box : other; }
NVC_HD float box_max(float box, float other) { return box > other ? box : other; }

// bvhPrepare's centroid (min + max) / 2.f with the NaN bits of x86 SSE, the reference's target: a NaN operand comes back
// quieted (the first one when both are NaN) and a NaN made from numbers (inf - inf) is the default NaN 0xffc00000.  The GPU's
// arithmetic returns 0x7fffffff for both.  The radix sort orders NaN centroids by these bits.
NVC_HD float centroid(float mn, float mx)
{
	if (mn != mn)
		return bits_float(float_bits(mn) | 0x00400000u);
	if (mx != mx)
		return bits_float(float_bits(mx) | 0x00400000u);
	float s = add(mn, mx);
	return s != s ? bits_float(0xffc00000u) : div(s, 2.0f);
}

// the SSE boxMerge's area: (sx * sy + sy * sz) + sz * sx
NVC_HD float box_area(const float mn[3], const float mx[3])
{
	float sx = sub(mx[0], mn[0]), sy = sub(mx[1], mn[1]), sz = sub(mx[2], mn[2]);
	return add(add(mul(sx, sy), mul(sy, sz)), mul(sz, sx));
}

// bvhCountVertices (clusterizer.cpp:816-840): unique vertices of order[0..count), out[i] after triangle i when out is given
// (a triangle with a repeated new vertex counts it twice, as in the reference); used[] is left all -1
NVC_HD uint32_t bvh_count_vertices(const uint32_t* order, uint32_t count, int16_t* used, const uint32_t* indices, uint32_t* out)
{
	uint32_t used_vertices = 0;
	for (uint32_t i = 0; i < count; ++i)
	{
		uint32_t index = order[i];
		uint32_t a = indices[index * 3 + 0], b = indices[index * 3 + 1], c = indices[index * 3 + 2];
		used_vertices += (used[a] < 0) + (used[b] < 0) + (used[c] < 0);
		used[a] = used[b] = used[c] = 1;
		if (out)
			out[i] = used_vertices;
	}
	for (uint32_t i = 0; i < count; ++i)
	{
		uint32_t index = order[i];
		used[indices[index * 3 + 0]] = used[indices[index * 3 + 1]] = used[indices[index * 3 + 2]] = -1;
	}
	return used_vertices;
}

NVC_HD void bvh_pack_leaf(uint8_t* boundary, uint32_t count)
{
	boundary[0] = 1;
	for (uint32_t i = 1; i < count; ++i)
		boundary[i] = 0;
}

// bvhPackTail (clusterizer.cpp:851-870)
NVC_HD void bvh_pack_tail(uint8_t* boundary, const uint32_t* order, uint32_t count, int16_t* used, const uint32_t* indices)
{
	for (uint32_t i = 0; i < count;)
	{
		uint32_t chunk = i + kMaxTriangles <= count ? kMaxTriangles : count - i;
		if (bvh_count_vertices(order + i, chunk, used, indices, nullptr) <= kMaxVertices)
		{
			bvh_pack_leaf(boundary + i, chunk);
			i += chunk;
			continue;
		}
		bvh_pack_leaf(boundary + i, kSpatialLeafSplit);
		i += kSpatialLeafSplit;
	}
}

// bvhDivisible (clusterizer.cpp:872-878)
NVC_HD bool bvh_divisible(uint32_t count, uint32_t min, uint32_t max)
{
	return min * 2 <= max ? count >= min : count % min <= (count / min) * (max - min);
}

// One candidate i of bvhPivot (clusterizer.cpp:895-920): false if not admissible; else `sah`, the cost the early
// `cost > bestcost` skip tests, and `full`, the cost with the fill term.  rfill is the left count, as written.
NVC_HD bool pivot_cost(const float* areas, const uint32_t* vertices, uint32_t count, uint32_t i, uint32_t min, bool aligned, uint32_t maxfill,
    float rmaxfill, float& sah, float& full)
{
	uint32_t lsplit = i + 1, rsplit = count - (i + 1);
	if (!bvh_divisible(lsplit, min, kMaxTriangles))
		return false;
	if (aligned && !bvh_divisible(rsplit, min, kMaxTriangles))
		return false;
	float larea = areas[i], rarea = areas[(count - 1 - (i + 1)) + count];
	sah = add(mul(larea, float(int(lsplit))), mul(rarea, float(int(rsplit))));
	uint32_t lfill = vertices ? vertices[i] : lsplit;
	uint32_t rfill = vertices ? vertices[i] : rsplit;
	int lrest = int(mul(float(int(lfill + maxfill - 1)), rmaxfill)) * int(maxfill) - int(lfill);
	int rrest = int(mul(float(int(rfill + maxfill - 1)), rmaxfill)) * int(maxfill) - int(rfill);
	full = add(sah, mul(kFillWeight, add(mul(float(lrest), larea), mul(float(rrest), rarea))));
	return true;
}

// bvhPivot's admissible range: [min - 1, end)
NVC_HD bool pivot_aligned(uint32_t count, uint32_t min) { return count >= min * 2 && bvh_divisible(count, min, kMaxTriangles); }
NVC_HD uint32_t pivot_end(uint32_t count, uint32_t min) { return pivot_aligned(count, min) ? count - min : count - 1; }

// bvhPivot (clusterizer.cpp:880-926) as written, with its early skip: the split after the first strict minimum
NVC_HD uint32_t bvh_pivot(const float* areas, const uint32_t* vertices, uint32_t count, uint32_t min, uint32_t maxfill, float& out_cost)
{
	bool aligned = pivot_aligned(count, min);
	uint32_t end = pivot_end(count, min);
	float rmaxfill = div(1.0f, float(int(maxfill)));
	uint32_t bestsplit = 0;
	float bestcost = FLT_MAX;
	for (uint32_t i = min - 1; i < end; ++i)
	{
		float sah, full;
		if (!pivot_cost(areas, vertices, count, i, min, aligned, maxfill, rmaxfill, sah, full))
			continue;
		if (sah > bestcost)
			continue;
		if (full < bestcost)
		{
			bestcost = full;
			bestsplit = i + 1;
		}
	}
	out_cost = bestcost;
	return bestsplit;
}

// appendMeshlet's flush (clusterizer.cpp:262-275), for the spatial packing loop's `split`
NVC_HD void flush_meshlet(Building& m, int16_t* used, uint4* records, uint32_t meshlet_offset, const uint32_t* meshlet_vertices)
{
	records[meshlet_offset] = make_uint4(m.vertex_offset, m.triangle_offset, m.vertex_count, m.triangle_count);
	for (uint32_t j = 0; j < m.vertex_count; ++j)
		used[meshlet_vertices[m.vertex_offset + j]] = -1;
	m.vertex_offset += m.vertex_count;
	m.triangle_offset += m.triangle_count * 3;
	m.vertex_count = 0;
	m.triangle_count = 0;
}

} // namespace cook
} // namespace nvc
