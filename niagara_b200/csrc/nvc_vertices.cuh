// nvc_vertices.cuh — the first stage of the reference's cooker on the device, SURVEY §8(f) row N4 (nvc_cook_mesh_vertices).
//
// Restates appendMesh's vertex processing (src/scene.cpp:172-184), so that the Vertex[] and LOD 0 index buffer are
// BIT-IDENTICAL to the reference's:
//   meshopt_filterIndexBuffer    extern/meshoptimizer/src/indexgenerator.cpp:331-386,483-498 over the 6 position bytes
//   meshopt_generateVertexRemap  indexgenerator.cpp:252-286,390-401 over all 16 bytes, then the remap of both buffers
//   meshopt_optimizeVertexCache  nvc_lods.cuh's lods::optimize_vertex_cache, unchanged
//   meshopt_optimizeVertexFetch  extern/meshoptimizer/src/vfetchoptimizer.cpp:29-71
// Every step but the vertex cache one is data-parallel over all meshes of a call at once, and no result depends on thread
// order: the hash tables only decide equality, every "first" is an atomicMin, and every rank comes from an exclusive scan
// of flags laid out in the reference's visiting order.
//   filter  The reference's remap ids serve only for equality and for rotating each triangle to its smallest id, so any
//           total order on the 48-bit position works: a triangle with two equal positions is dropped, the others are
//           rotated min-first and inserted into a table keyed by (mesh, rotated positions).  An entry holds a triangle
//           index and keeps the smallest with atomicMin; keys are compared by re-reading the (immutable) inputs, so a
//           collision probes on and no thread waits.  A triangle is kept when it is its entry's minimum; kept triangles
//           are compacted in order with their original indices.
//   remap   first[v] is the smallest filtered position referencing v.  Byte-equal vertices of a mesh share an entry of a
//           second table, which keeps the smallest `first` of its members; each class flags that position, and the scan
//           of the flags ranks the classes in the order of their first reference, which is generateVertexRemap's order.
//   fetch   first use of each vertex over the optimised indices by atomicMin, flags, scan, as above.
// A scan is nvc_scan.cuh's device-wide scan of the flags into `rank`, the total at rank[n].  Nothing spins, so the kernels
// run as they are under the SIMT emulation too.
#pragma once

#include "nvc_lods.cuh"
#include "nvc_scan.cuh"

namespace nvc
{
namespace verts
{

constexpr uint32_t kNone = ~0u;
constexpr uint32_t kThreads = 256;

// the vertex cache optimiser's arrays of a mesh with at most V vertices and N indices (lods::carve's layout for them);
// returns the mesh's words.  base == nullptr: size only
NVC_HD uint64_t carve(uint32_t V, uint32_t N, uint32_t* base, lods::Scratch* s)
{
	const uint64_t T = N / 3;
	uint64_t at = 0;
	auto take = [&](uint64_t words) {
		uint32_t* p = base ? base + at : nullptr;
		at += (words + 3) & ~uint64_t(3);
		return p;
	};
	lods::Scratch w = {};
	w.vcount = take(V);
	w.voff = take(V);
	w.vdata = take(N);
	w.vscore = reinterpret_cast<float*>(take(V));
	w.tscore = reinterpret_cast<float*>(take(T));
	w.emitted = take(T);
	if (s)
		*s = w;
	return at;
}

// claims an empty table bucket: atomicCAS; under the CPU emulation (tests/cuda_emu: one OS thread, no atomicCAS there) the
// same read-modify-write done plainly
__device__ __forceinline__ uint32_t claim(uint32_t* bucket, uint32_t item)
{
#if defined(NVC_EMU)
	const uint32_t held = *bucket;
	if (held == kNone)
		*bucket = item;
	return held;
#else
	return atomicCAS(bucket, kNone, item);
#endif
}

__device__ __forceinline__ uint32_t hash_mix(uint64_t h, uint64_t k)
{
	h = (h ^ k) * 0x9e3779b97f4a7c15ull;
	return uint32_t(h >> 32) ^ uint32_t(h);
}

// the mesh whose range holds a triangle, slot or position (an empty mesh shares its base with the next one)
__device__ __forceinline__ uint32_t job_of_triangle(const VertexArgs& a, uint32_t t)
{
	return scan::last_at_most(a.mesh_count, t, [&](uint32_t m) { return a.jobs[m].tri_base; });
}

__device__ __forceinline__ uint32_t job_of_slot(const VertexArgs& a, uint32_t s)
{
	return scan::last_at_most(a.mesh_count, s, [&](uint32_t m) { return a.jobs[m].slot_base; });
}

__device__ __forceinline__ uint32_t job_of_position(const VertexArgs& a, uint32_t p)
{
	return scan::last_at_most(a.mesh_count, p, [&](uint32_t m) { return a.index_base[m]; });
}

__device__ __forceinline__ uint64_t position_key(const NvcVertex& v)
{
	return uint64_t(v.vx) | uint64_t(v.vy) << 16 | uint64_t(v.vz) << 32;
}

// triangle t's corner keys rotated so that the smallest comes first; false when two corners share a position
__device__ __forceinline__ bool triangle_key(const VertexArgs& a, const VertexJob& job, uint32_t t, uint64_t k[3])
{
	const uint32_t* tri = a.indices + job.index_offset + uint64_t(t - job.tri_base) * 3;
	const NvcVertex* v = a.vertices + job.vertex_offset;
	const uint64_t x = position_key(v[tri[0]]), y = position_key(v[tri[1]]), z = position_key(v[tri[2]]);
	if (x == y || x == z || y == z)
		return false;
	const bool y_least = y < x && y < z, z_least = z < x && z < y;
	k[0] = y_least ? y : z_least ? z : x;
	k[1] = y_least ? z : z_least ? x : y;
	k[2] = y_least ? x : z_least ? y : z;
	return true;
}

// ---- rejection and the filter ----------------------------------------------------------------------------------------------

// a mesh with an index >= its vertexCount is rejected before any of its vertices is read
__global__ void __launch_bounds__(kThreads) verts_reject_kernel(const VertexArgs a)
{
	const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
	if (t >= a.tri_count)
		return;
	const uint32_t m = job_of_triangle(a, t);
	const VertexJob& job = a.jobs[m];
	const uint32_t* tri = a.indices + job.index_offset + uint64_t(t - job.tri_base) * 3;
	if (tri[0] >= job.vertex_count || tri[1] >= job.vertex_count || tri[2] >= job.vertex_count)
		a.rejected[m] = 1;
}

// one thread per triangle: degenerate test, min-first rotation, insertion; tri_entry[t] = its bucket, kNone when dropped
__global__ void __launch_bounds__(kThreads) verts_filter_insert_kernel(const VertexArgs a)
{
	const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
	if (t >= a.tri_count)
		return;
	const uint32_t m = job_of_triangle(a, t);
	const VertexJob& job = a.jobs[m];
	uint64_t k[3];
	if (a.rejected[m] || !triangle_key(a, job, t, k))
	{
		a.tri_entry[t] = kNone;
		return;
	}
	uint32_t bucket = hash_mix(hash_mix(hash_mix(m, k[0]), k[1]), k[2]) & a.tri_mask;
	for (uint32_t probe = 0;; ++probe)
	{
		uint32_t held = a.tri_table[bucket];
		if (held == kNone)
		{
			held = claim(&a.tri_table[bucket], t);
			if (held == kNone)
				break;
		}
		uint64_t hk[3];
		const uint32_t hm = job_of_triangle(a, held);
		if (hm == m && triangle_key(a, a.jobs[hm], held, hk) && hk[0] == k[0] && hk[1] == k[1] && hk[2] == k[2])
		{
			atomicMin(&a.tri_table[bucket], t);
			break;
		}
		bucket = (bucket + probe + 1) & a.tri_mask;
	}
	a.tri_entry[t] = bucket;
}

// kept: the smallest triangle of its entry
__global__ void __launch_bounds__(kThreads) verts_filter_flag_kernel(const VertexArgs a)
{
	const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
	if (t >= a.tri_count)
		return;
	const uint32_t e = a.tri_entry[t];
	a.flags[t] = e != kNone && a.tri_table[e] == t;
}

// kept triangles in order, original mesh-local indices
__global__ void __launch_bounds__(kThreads) verts_filter_compact_kernel(const VertexArgs a)
{
	const uint32_t t = blockIdx.x * kThreads + threadIdx.x;
	if (t >= a.tri_count || !a.flags[t])
		return;
	const VertexJob& job = a.jobs[job_of_triangle(a, t)];
	const uint32_t* tri = a.indices + job.index_offset + uint64_t(t - job.tri_base) * 3;
	uint32_t* dst = a.filtered + uint64_t(a.rank[t]) * 3;
	dst[0] = tri[0];
	dst[1] = tri[1];
	dst[2] = tri[2];
}

// per mesh: its first filtered index; the filtered total is the indices written (totals4[1])
__global__ void __launch_bounds__(kThreads) verts_index_base_kernel(const VertexArgs a)
{
	const uint32_t m = blockIdx.x * kThreads + threadIdx.x;
	if (m >= a.mesh_count)
		return;
	a.index_base[m] = 3 * a.rank[a.jobs[m].tri_base];
	if (m == 0)
		a.totals4[1] = 3 * a.rank[a.tri_count];
	if (a.rejected[m])
		atomicAdd(&a.totals4[2], 1u);
}

// ---- remap -----------------------------------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t slot_of_position(const VertexArgs& a, uint32_t p, uint32_t& m)
{
	m = job_of_position(a, p);
	return a.jobs[m].slot_base + a.filtered[p];
}

// first[slot] = the smallest filtered position referencing the vertex
__global__ void __launch_bounds__(kThreads) verts_first_kernel(const VertexArgs a)
{
	const uint32_t p = blockIdx.x * kThreads + threadIdx.x;
	if (p >= a.totals4[1])
		return;
	uint32_t m;
	atomicMin(&a.first[slot_of_position(a, p, m)], p);
}

__device__ __forceinline__ const NvcVertex& vertex_of_slot(const VertexArgs& a, uint32_t s, uint32_t m)
{
	const VertexJob& job = a.jobs[m];
	return a.vertices[job.vertex_offset + (s - job.slot_base)];
}

__device__ __forceinline__ bool same_bytes(const NvcVertex& x, const NvcVertex& y)
{
	return x.vx == y.vx && x.vy == y.vy && x.vz == y.vz && x.tp == y.tp && x.np == y.np && x.tu == y.tu && x.tv == y.tv;
}

// one thread per referenced vertex: its class's entry (vtx_entry), which keeps the smallest `first` of its members
__global__ void __launch_bounds__(kThreads) verts_class_insert_kernel(const VertexArgs a)
{
	const uint32_t s = blockIdx.x * kThreads + threadIdx.x;
	if (s >= a.slot_count)
		return;
	const uint32_t f = a.first[s];
	if (f == kNone)
		return;
	const uint32_t m = job_of_slot(a, s);
	const NvcVertex v = vertex_of_slot(a, s, m);
	uint32_t w[4];
	memcpy(w, &v, 16);
	uint32_t bucket = hash_mix(hash_mix(hash_mix(hash_mix(m, w[0]), w[1]), w[2]), w[3]) & a.vtx_mask;
	for (uint32_t probe = 0;; ++probe)
	{
		uint32_t held = a.vtx_table[bucket];
		if (held == kNone)
		{
			held = claim(&a.vtx_table[bucket], s);
			if (held == kNone)
				break;
		}
		const uint32_t hm = job_of_slot(a, held);
		if (hm == m && same_bytes(vertex_of_slot(a, held, hm), v))
			break;
		bucket = (bucket + probe + 1) & a.vtx_mask;
	}
	a.vtx_entry[s] = bucket;
	atomicMin(&a.vtx_first[bucket], f);
}

// a class's first reference is the `first` of exactly one member: it flags that position
__global__ void __launch_bounds__(kThreads) verts_class_flag_kernel(const VertexArgs a)
{
	const uint32_t s = blockIdx.x * kThreads + threadIdx.x;
	if (s >= a.slot_count)
		return;
	const uint32_t f = a.first[s];
	if (f != kNone && a.vtx_first[a.vtx_entry[s]] == f)
		a.flags[f] = 1;
}

// per mesh, after the class scan: the output Mesh record; the classes are the vertices written (totals4[0])
__global__ void __launch_bounds__(kThreads) verts_mesh_kernel(const VertexArgs a)
{
	const uint32_t m = blockIdx.x * kThreads + threadIdx.x;
	if (m >= a.mesh_count)
		return;
	const uint32_t n = a.totals4[1];
	const uint32_t ib = a.index_base[m], ie = m + 1 < a.mesh_count ? a.index_base[m + 1] : n;
	const uint32_t vb = a.rank[ib], ve = a.rank[ie];
	a.vertex_base[m] = vb;
	if (m == 0)
		a.totals4[0] = a.rank[n];
	NvcMesh mesh = {};
	mesh.vertexOffset = vb;
	mesh.vertexCount = ve - vb;
	mesh.lodCount = 1;
	mesh.lods[0].indexOffset = ib;
	mesh.lods[0].indexCount = ie - ib;
	a.meshes[m] = mesh;
}

// each class's vertex to its rank (generateVertexRemap + remapVertexBuffer)
__global__ void __launch_bounds__(kThreads) verts_class_scatter_kernel(const VertexArgs a)
{
	const uint32_t s = blockIdx.x * kThreads + threadIdx.x;
	if (s >= a.slot_count)
		return;
	const uint32_t f = a.first[s];
	if (f == kNone || a.vtx_first[a.vtx_entry[s]] != f)
		return;
	a.classes[a.rank[f]] = vertex_of_slot(a, s, job_of_slot(a, s));
}

// each filtered index to its class, mesh-local (remapIndexBuffer)
__global__ void __launch_bounds__(kThreads) verts_remap_kernel(const VertexArgs a)
{
	const uint32_t p = blockIdx.x * kThreads + threadIdx.x;
	if (p >= a.totals4[1])
		return;
	uint32_t m;
	const uint32_t s = slot_of_position(a, p, m);
	a.remapped[p] = a.rank[a.vtx_first[a.vtx_entry[s]]] - a.vertex_base[m];
}

// ---- vertex cache: one single-thread CTA per mesh, longest first; remapped -> lod0_out -------------------------------------
__global__ void __launch_bounds__(1) verts_vcache_kernel(const VertexArgs a)
{
	const uint32_t m = a.order[blockIdx.x];
	const NvcMesh& mesh = a.meshes[m];
	const uint32_t n = mesh.lods[0].indexCount, V = mesh.vertexCount, ib = mesh.lods[0].indexOffset;
	if (n == 0)
		return;
	lods::Scratch w;
	const VertexJob& job = a.jobs[m];
	carve(min(job.vertex_count, job.index_count), job.index_count, a.scratch + job.scratch, &w);
	lods::optimize_vertex_cache(w, a.lod0_out + ib, a.remapped + ib, n, V);
}

// ---- fetch order -----------------------------------------------------------------------------------------------------------

// first_use[class] = the smallest optimised position using it
__global__ void __launch_bounds__(kThreads) verts_fetch_first_kernel(const VertexArgs a)
{
	const uint32_t p = blockIdx.x * kThreads + threadIdx.x;
	if (p >= a.totals4[1])
		return;
	const uint32_t m = job_of_position(a, p);
	atomicMin(&a.first_use[a.vertex_base[m] + a.lod0_out[p]], p);
}

__global__ void __launch_bounds__(kThreads) verts_fetch_flag_kernel(const VertexArgs a)
{
	const uint32_t c = blockIdx.x * kThreads + threadIdx.x;
	if (c >= a.totals4[0])
		return;
	a.flags[a.first_use[c]] = 1;
}

// the vertices in first-use order, the indices rewritten to match (optimizeVertexFetch)
__global__ void __launch_bounds__(kThreads) verts_fetch_scatter_kernel(const VertexArgs a)
{
	const uint32_t c = blockIdx.x * kThreads + threadIdx.x;
	if (c >= a.totals4[0])
		return;
	a.vertices_out[a.rank[a.first_use[c]]] = a.classes[c];
}

__global__ void __launch_bounds__(kThreads) verts_fetch_index_kernel(const VertexArgs a)
{
	const uint32_t p = blockIdx.x * kThreads + threadIdx.x;
	if (p >= a.totals4[1])
		return;
	const uint32_t vb = a.vertex_base[job_of_position(a, p)];
	a.lod0_out[p] = a.rank[a.first_use[vb + a.lod0_out[p]]] - vb;
}

} // namespace verts
} // namespace nvc
