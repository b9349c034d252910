// nvc_lods.cuh — the LOD chain of the reference's cooker on the device, SURVEY §8(f) row N4 (nvc_cook_mesh_lods).
//
// Restates appendMesh's LOD loop (src/scene.cpp:193-268) and the two meshoptimizer calls it makes, only on the path it
// uses, so that the Mesh record and the index buffer are BIT-IDENTICAL to the reference's:
//   meshopt_simplifyWithAttributes  extern/meshoptimizer/src/simplifier.cpp:2344-2626 (meshopt_simplifyEdge) with
//                                   meshopt_SimplifySparse, 3 attributes of weight 1 (the decoded normal), no vertex lock,
//                                   target error 1e-1, no prune, no solve, no permissive mode
//   meshopt_optimizeVertexCache     extern/meshoptimizer/src/vcacheoptimizer.cpp:169-343 with kVertexScoreTable
//   meshopt_simplifyScale           simplifier.cpp:549-603,2938-2948
// Each mesh's chain is one thread's sequential work (LOD k + 1 starts from LOD k), in a CTA of its own; meshes run side by
// side.  Every stage visits its data in the reference's order, so each float sum has the reference's operands in the
// reference's order.  The translation unit is built with -fmad=false (nvcc) / -ffp-contract=off (host), so the plain
// operators below are single IEEE operations with round-to-nearest, like the reference's x86-64 SSE code without FMA.
// NaN payloads reach the outputs only through Mesh::center and lods[].error; those few operations use the x86_* helpers,
// which give the bits x86 SSE gives.  Comparisons with NaN behave alike everywhere, so no other result depends on them.
#pragma once

#include "nvc_meshlets.cuh"

namespace nvc
{
namespace lods
{

constexpr uint32_t kNone = ~0u;
constexpr uint32_t kSortBins = 2048 + 512; // sortEdgeCollapses: 12-bit keys, exponent range [-127, 32)
constexpr float kMaxError = 1e-1f;         // scene.cpp:231

// per mesh: one LOD chain.  index_offset / index_count: LOD 0 in the caller's lod0_indices; scratch: first word of the
// mesh's scratch; capacity: chain_capacity(index_count)
struct LodJob
{
	uint32_t vertex_offset, vertex_count, index_offset, index_count;
	uint64_t scratch;
	uint64_t capacity;
};

// indices appendMesh's loop can emit from a LOD 0 of n indices: LOD l + 1 is kept only when it has fewer than
// size_t(double(c_l) * 0.85) indices, a multiple of 3, and more than 0; at most 8 LODs
NVC_HD uint64_t chain_capacity(uint32_t n)
{
	uint64_t total = 0, c = n;
	for (uint32_t l = 0; l < NVC_MAX_LODS; ++l)
	{
		total += c;
		uint64_t below = uint64_t(double(c) * 0.85);
		if (below == 0)
			break;
		c = (below - 1) / 3 * 3;
		if (c == 0)
			break;
	}
	return total;
}

// hashBuckets2 (simplifier.cpp:165-172)
NVC_HD uint32_t hash_buckets(uint32_t count)
{
	uint32_t buckets = 1;
	while (buckets < count + count / 4)
		buckets *= 2;
	return buckets;
}

struct Quadric
{
	float a00, a11, a22, a10, a20, a21, b0, b1, b2, c, w;
};

struct Grad
{
	float gx, gy, gz, gw;
};

struct Collapse
{
	uint32_t v0, v1;
	uint32_t bits; // bidi while picking, then the error's bits
};

// Scratch of one mesh, carved from 4-byte words.  V = vertexCount, N = LOD 0 indices, U = min(V, N) (the vertices a
// sparse simplification can see), C = chain_capacity(N)
struct Scratch
{
	uint32_t* out;      // C: the chain, LOD after LOD
	uint32_t* cur;      // N: lodIndices
	uint32_t* tmp;      // N: the vertex cache optimiser's input copy
	uint32_t* d2s;      // V: mesh vertex -> sparse vertex, kNone outside a simplification
	uint32_t* vcount;   // V
	uint32_t* voff;     // V
	uint32_t* vdata;    // N
	float* vscore;      // V
	float* tscore;      // N / 3
	uint32_t* emitted;  // N / 3
	uint32_t* sparse;   // U: sparse vertex -> mesh vertex
	uint32_t* adj_off;  // U + 1
	uint32_t* adj_data; // 2 N: (next, prev) per half-edge
	uint32_t* remap;    // U
	uint32_t* wedge;    // U
	uint32_t* table;    // hash_buckets(U)
	uint32_t* kind;     // U
	uint32_t* loop;     // U
	uint32_t* loopback; // U
	float* pos;         // 3 U
	float* attr;        // 3 U
	Quadric* vq;        // U
	Quadric* aq;        // U
	Grad* ag;           // 3 U
	Collapse* col;      // N + 3
	uint32_t* order;    // N + 3
	uint32_t* cremap;   // U
	uint32_t* clocked;  // U
	uint32_t* hist;     // kSortBins
};

// word offsets of Scratch's arrays from the mesh's first word; returns the mesh's words.  base == nullptr: size only
NVC_HD uint64_t carve(uint32_t V, uint32_t N, uint64_t C, uint32_t* base, Scratch* s)
{
	const uint64_t U = V < N ? V : N, T = N / 3;
	uint64_t at = 0;
	auto take = [&](uint64_t words) {
		uint32_t* p = base ? base + at : nullptr;
		at += (words + 3) & ~uint64_t(3); // 16-byte aligned arrays
		return p;
	};
	Scratch w;
	w.out = take(C);
	w.cur = take(N);
	w.tmp = take(N);
	w.d2s = take(V);
	w.vcount = take(V);
	w.voff = take(V);
	w.vdata = take(N);
	w.vscore = reinterpret_cast<float*>(take(V));
	w.tscore = reinterpret_cast<float*>(take(T));
	w.emitted = take(T);
	w.sparse = take(U);
	w.adj_off = take(U + 1);
	w.adj_data = take(2 * uint64_t(N));
	w.remap = take(U);
	w.wedge = take(U);
	w.table = take(hash_buckets(uint32_t(U)));
	w.kind = take(U);
	w.loop = take(U);
	w.loopback = take(U);
	w.pos = reinterpret_cast<float*>(take(3 * U));
	w.attr = reinterpret_cast<float*>(take(3 * U));
	w.vq = reinterpret_cast<Quadric*>(take(11 * U));
	w.aq = reinterpret_cast<Quadric*>(take(11 * U));
	w.ag = reinterpret_cast<Grad*>(take(12 * U));
	w.col = reinterpret_cast<Collapse*>(take(3 * (uint64_t(N) + 3)));
	w.order = take(uint64_t(N) + 3);
	w.cremap = take(U);
	w.clocked = take(U);
	w.hist = take(kSortBins);
	if (s)
		*s = w;
	return at;
}

// ---- x86 SSE NaN bits (the reference's target): a NaN operand comes back quieted, the first one when both are; a NaN
// made from numbers is the default NaN 0xffc00000.  The GPU returns 0x7fffffff for all of these.
NVC_HD float x86_nan(float a, float b, float r)
{
	if (a != a)
		return cook::bits_float(cook::float_bits(a) | 0x00400000u);
	if (b != b)
		return cook::bits_float(cook::float_bits(b) | 0x00400000u);
	return r != r ? cook::bits_float(0xffc00000u) : r;
}
NVC_HD float x86_add(float a, float b) { return x86_nan(a, b, a + b); }
NVC_HD float x86_sub(float a, float b) { return x86_nan(a, b, a - b); }
NVC_HD float x86_mul(float a, float b) { return x86_nan(a, b, a * b); }
NVC_HD float x86_div(float a, float b) { return x86_nan(a, b, a / b); }

// ---- the mesh's vertices, as appendMesh sees them (scene.cpp:193-205)
struct Source
{
	const NvcVertex* v; // vertices + vertexOffset
	__device__ float position(uint32_t i, int k) const
	{
		NvcVertex x = v[i];
		return cook::dequantize_half(k == 0 ? x.vx : (k == 1 ? x.vy : x.vz));
	}
	__device__ float normal(uint32_t i, int k) const { return float((v[i].np >> (10 * k)) & 1023) / 511.f - 1.f; }
};

// rescalePositions' extent (simplifier.cpp:549-581), positions i < count of point(i)
template <typename F>
__device__ inline float extent_of(uint32_t count, const F& point, float minv[3])
{
	float maxv[3] = { -FLT_MAX, -FLT_MAX, -FLT_MAX };
	minv[0] = minv[1] = minv[2] = FLT_MAX;
	for (uint32_t i = 0; i < count; ++i)
		for (int j = 0; j < 3; ++j)
		{
			float vj = point(i, j);
			minv[j] = minv[j] > vj ? vj : minv[j];
			maxv[j] = maxv[j] < vj ? vj : maxv[j];
		}
	float extent = 0.f;
	for (int j = 0; j < 3; ++j)
	{
		float d = x86_sub(maxv[j], minv[j]);
		extent = d < extent ? extent : d;
	}
	return extent;
}

// ---- edge adjacency (simplifier.cpp:52-109), remap == nullptr: none
__device__ inline void update_adjacency(const Scratch& w, const uint32_t* indices, uint32_t index_count, uint32_t vertex_count, const uint32_t* remap)
{
	uint32_t* offsets = w.adj_off + 1;
	for (uint32_t i = 0; i < vertex_count; ++i)
		offsets[i] = 0;
	for (uint32_t i = 0; i < index_count; ++i)
		offsets[remap ? remap[indices[i]] : indices[i]]++;
	uint32_t offset = 0;
	for (uint32_t i = 0; i < vertex_count; ++i)
	{
		uint32_t count = offsets[i];
		offsets[i] = offset;
		offset += count;
	}
	for (uint32_t i = 0; i < index_count; i += 3)
	{
		uint32_t a = indices[i + 0], b = indices[i + 1], c = indices[i + 2];
		if (remap)
		{
			a = remap[a];
			b = remap[b];
			c = remap[c];
		}
		uint32_t* d = w.adj_data;
		d[2 * offsets[a]] = b;
		d[2 * offsets[a] + 1] = c;
		offsets[a]++;
		d[2 * offsets[b]] = c;
		d[2 * offsets[b] + 1] = a;
		offsets[b]++;
		d[2 * offsets[c]] = a;
		d[2 * offsets[c] + 1] = b;
		offsets[c]++;
	}
	w.adj_off[0] = 0;
}

__device__ inline bool has_edge(const Scratch& w, uint32_t a, uint32_t b)
{
	for (uint32_t e = w.adj_off[a]; e < w.adj_off[a + 1]; ++e)
		if (w.adj_data[2 * e] == b)
			return true;
	return false;
}

// kCanCollapse / kHasOpposite (simplifier.cpp:312-331), row k0 in bits 5 * k0 .. 5 * k0 + 4
enum Kind : uint32_t
{
	Manifold,
	Border,
	Seam,
	Complex,
	Locked
};
NVC_HD uint32_t can_collapse(uint32_t k0, uint32_t k1) { return (0x000C525Fu >> (5 * k0 + k1)) & 1u; }
NVC_HD uint32_t has_opposite(uint32_t k0, uint32_t k1) { return (0x0050DCBFu >> (5 * k0 + k1)) & 1u; }

// classifyVertices (simplifier.cpp:364-479) without lock, permissive and lock-border options
__device__ inline void classify(const Scratch& w, uint32_t vertex_count)
{
	uint32_t* openinc = w.loopback;
	uint32_t* openout = w.loop;
	for (uint32_t i = 0; i < vertex_count; ++i)
		openinc[i] = openout[i] = kNone;
	for (uint32_t vertex = 0; vertex < vertex_count; ++vertex)
		for (uint32_t e = w.adj_off[vertex]; e < w.adj_off[vertex + 1]; ++e)
		{
			uint32_t target = w.adj_data[2 * e];
			if (target == vertex)
				openinc[vertex] = openout[vertex] = vertex;
			else if (!has_edge(w, target, vertex))
			{
				openinc[target] = openinc[target] == kNone ? vertex : target;
				openout[vertex] = openout[vertex] == kNone ? target : vertex;
			}
		}
	const uint32_t* remap = w.remap;
	const uint32_t* wedge = w.wedge;
	for (uint32_t i = 0; i < vertex_count; ++i)
	{
		uint32_t k;
		if (remap[i] != i)
			k = w.kind[remap[i]];
		else if (wedge[i] == i)
		{
			uint32_t openi = openinc[i], openo = openout[i];
			if (openi == kNone && openo == kNone)
				k = Manifold;
			else if (openi != kNone && openo != kNone && remap[openi] == remap[openo] && openi != i)
				k = Seam;
			else if (openi != i && openo != i)
				k = Border;
			else
				k = Locked;
		}
		else if (wedge[wedge[i]] == i)
		{
			uint32_t ww = wedge[i];
			uint32_t openiv = openinc[i], openov = openout[i], openiw = openinc[ww], openow = openout[ww];
			if (openiv != kNone && openiv != i && openov != kNone && openov != i && openiw != kNone && openiw != ww && openow != kNone && openow != ww)
				k = remap[openiv] == remap[openow] && remap[openov] == remap[openiw] && remap[openiv] != remap[openov] ? Seam : Locked;
			else
				k = Locked;
		}
		else
			k = Locked;
		w.kind[i] = k;
	}
}

// ---- quadrics (simplifier.cpp:702-1179), each expression in the reference's operand order
__device__ inline void quadric_add(Quadric& Q, const Quadric& R)
{
	Q.a00 += R.a00;
	Q.a11 += R.a11;
	Q.a22 += R.a22;
	Q.a10 += R.a10;
	Q.a20 += R.a20;
	Q.a21 += R.a21;
	Q.b0 += R.b0;
	Q.b1 += R.b1;
	Q.b2 += R.b2;
	Q.c += R.c;
	Q.w += R.w;
}

__device__ inline void grad_add(Grad* G, const Grad* R)
{
	for (int k = 0; k < 3; ++k)
	{
		G[k].gx += R[k].gx;
		G[k].gy += R[k].gy;
		G[k].gz += R[k].gz;
		G[k].gw += R[k].gw;
	}
}

__device__ inline float quadric_eval(const Quadric& Q, const float* v)
{
	float rx = Q.b0, ry = Q.b1, rz = Q.b2;
	rx += Q.a10 * v[1];
	ry += Q.a21 * v[2];
	rz += Q.a20 * v[0];
	rx *= 2;
	ry *= 2;
	rz *= 2;
	rx += Q.a00 * v[0];
	ry += Q.a11 * v[1];
	rz += Q.a22 * v[2];
	float r = Q.c;
	r += rx * v[0];
	r += ry * v[1];
	r += rz * v[2];
	return r;
}

__device__ inline float quadric_error(const Quadric& Q, const float* v)
{
	float r = quadric_eval(Q, v);
	float s = Q.w == 0.f ? 0.f : 1.f / Q.w;
	return fabsf(r) * s;
}

__device__ inline float quadric_error(const Quadric& Q, const Grad* G, const float* v, const float* va)
{
	float r = quadric_eval(Q, v);
	for (int k = 0; k < 3; ++k)
	{
		float a = va[k];
		float g = v[0] * G[k].gx + v[1] * G[k].gy + v[2] * G[k].gz + G[k].gw;
		r += a * (a * Q.w - 2 * g);
	}
	return fabsf(r);
}

__device__ inline float normalize(float* v)
{
	float length = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
	if (length > 0)
	{
		v[0] /= length;
		v[1] /= length;
		v[2] /= length;
	}
	return length;
}

__device__ inline void quadric_from_plane(Quadric& Q, float a, float b, float c, float d, float w)
{
	float aw = a * w, bw = b * w, cw = c * w, dw = d * w;
	Q.a00 = a * aw;
	Q.a11 = b * bw;
	Q.a22 = c * cw;
	Q.a10 = a * bw;
	Q.a20 = a * cw;
	Q.a21 = b * cw;
	Q.b0 = a * dw;
	Q.b1 = b * dw;
	Q.b2 = c * dw;
	Q.c = d * dw;
	Q.w = w;
}

__device__ inline void cross_edges(const float* p0, const float* p1, const float* p2, float* p10, float* p20, float* normal)
{
	for (int k = 0; k < 3; ++k)
	{
		p10[k] = p1[k] - p0[k];
		p20[k] = p2[k] - p0[k];
	}
	normal[0] = p10[1] * p20[2] - p10[2] * p20[1];
	normal[1] = p10[2] * p20[0] - p10[0] * p20[2];
	normal[2] = p10[0] * p20[1] - p10[1] * p20[0];
}

__device__ inline void quadric_from_triangle(Quadric& Q, const float* p0, const float* p1, const float* p2, float weight)
{
	float p10[3], p20[3], normal[3];
	cross_edges(p0, p1, p2, p10, p20, normal);
	float area = normalize(normal);
	float distance = normal[0] * p0[0] + normal[1] * p0[1] + normal[2] * p0[2];
	quadric_from_plane(Q, normal[0], normal[1], normal[2], -distance, sqrtf(area) * weight);
}

__device__ inline void quadric_from_triangle_edge(Quadric& Q, const float* p0, const float* p1, const float* p2, float weight)
{
	float p10[3] = { p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2] };
	float lengthsq = p10[0] * p10[0] + p10[1] * p10[1] + p10[2] * p10[2];
	float length = sqrtf(lengthsq);
	float p20[3] = { p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2] };
	float p20p = p20[0] * p10[0] + p20[1] * p10[1] + p20[2] * p10[2];
	float perp[3] = { p20[0] * lengthsq - p10[0] * p20p, p20[1] * lengthsq - p10[1] * p20p, p20[2] * lengthsq - p10[2] * p20p };
	normalize(perp);
	float distance = perp[0] * p0[0] + perp[1] * p0[1] + perp[2] * p0[2];
	quadric_from_plane(Q, perp[0], perp[1], perp[2], -distance, length * weight);
}

__device__ inline void quadric_from_attributes(Quadric& Q, Grad* G, const float* p0, const float* p1, const float* p2, const float* va0, const float* va1, const float* va2)
{
	float v0[3], v1[3], normal[3];
	cross_edges(p0, p1, p2, v0, v1, normal);
	float area = sqrtf(normal[0] * normal[0] + normal[1] * normal[1] + normal[2] * normal[2]) * 0.5f;
	float w = area;
	float d00 = v0[0] * v0[0] + v0[1] * v0[1] + v0[2] * v0[2];
	float d01 = v0[0] * v1[0] + v0[1] * v1[1] + v0[2] * v1[2];
	float d11 = v1[0] * v1[0] + v1[1] * v1[1] + v1[2] * v1[2];
	float denom = d00 * d11 - d01 * d01;
	float denomr = denom == 0 ? 0.f : 1.f / denom;
	float gx1 = (d11 * v0[0] - d01 * v1[0]) * denomr;
	float gx2 = (d00 * v1[0] - d01 * v0[0]) * denomr;
	float gy1 = (d11 * v0[1] - d01 * v1[1]) * denomr;
	float gy2 = (d00 * v1[1] - d01 * v0[1]) * denomr;
	float gz1 = (d11 * v0[2] - d01 * v1[2]) * denomr;
	float gz2 = (d00 * v1[2] - d01 * v0[2]) * denomr;
	Q = Quadric{ 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0 };
	Q.w = w;
	for (int k = 0; k < 3; ++k)
	{
		float a0 = va0[k], a1 = va1[k], a2 = va2[k];
		float gx = gx1 * (a1 - a0) + gx2 * (a2 - a0);
		float gy = gy1 * (a1 - a0) + gy2 * (a2 - a0);
		float gz = gz1 * (a1 - a0) + gz2 * (a2 - a0);
		float gw = a0 - p0[0] * gx - p0[1] * gy - p0[2] * gz;
		Q.a00 += w * (gx * gx);
		Q.a11 += w * (gy * gy);
		Q.a22 += w * (gz * gz);
		Q.a10 += w * (gy * gx);
		Q.a20 += w * (gz * gx);
		Q.a21 += w * (gz * gy);
		Q.b0 += w * (gx * gw);
		Q.b1 += w * (gy * gw);
		Q.b2 += w * (gz * gw);
		Q.c += w * (gw * gw);
		G[k].gx = w * gx;
		G[k].gy = w * gy;
		G[k].gz = w * gz;
		G[k].gw = w * gw;
	}
}

// hasTriangleFlip (simplifier.cpp:1182-1198): does triangle abc flip when c is replaced with d?
__device__ inline bool has_triangle_flip(const float* a, const float* b, const float* c, const float* d)
{
	float eb[3], ec[3], ed[3];
	for (int k = 0; k < 3; ++k)
	{
		eb[k] = b[k] - a[k];
		ec[k] = c[k] - a[k];
		ed[k] = d[k] - a[k];
	}
	float nbc[3] = { eb[1] * ec[2] - eb[2] * ec[1], eb[2] * ec[0] - eb[0] * ec[2], eb[0] * ec[1] - eb[1] * ec[0] };
	float nbd[3] = { eb[1] * ed[2] - eb[2] * ed[1], eb[2] * ed[0] - eb[0] * ed[2], eb[0] * ed[1] - eb[1] * ed[0] };
	float ndp = nbc[0] * nbd[0] + nbc[1] * nbd[1] + nbc[2] * nbd[2];
	float abc = nbc[0] * nbc[0] + nbc[1] * nbc[1] + nbc[2] * nbc[2];
	float abd = nbd[0] * nbd[0] + nbd[1] * nbd[1] + nbd[2] * nbd[2];
	return ndp <= 0.25f * sqrtf(abc * abd);
}

__device__ inline bool has_triangle_flips(const Scratch& w, uint32_t i0, uint32_t i1)
{
	const float* v0 = w.pos + 3 * i0;
	const float* v1 = w.pos + 3 * i1;
	for (uint32_t e = w.adj_off[i0]; e < w.adj_off[i0 + 1]; ++e)
	{
		uint32_t a = w.cremap[w.adj_data[2 * e]], b = w.cremap[w.adj_data[2 * e + 1]];
		if (a == i1 || b == i1 || a == b)
			continue;
		if (has_triangle_flip(w.pos + 3 * a, w.pos + 3 * b, v0, v1))
			return true;
	}
	return false;
}

__device__ inline uint32_t complex_target(const Scratch& w, uint32_t v, uint32_t target)
{
	uint32_t r = w.remap[target];
	if (w.loop[v] != kNone && w.remap[w.loop[v]] == r)
		return w.loop[v];
	else if (w.loopback[v] != kNone && w.remap[w.loopback[v]] == r)
		return w.loopback[v];
	return target;
}

__device__ inline float attribute_error(const Scratch& w, uint32_t v, uint32_t t)
{
	return quadric_error(w.aq[v], w.ag + 3 * v, w.pos + 3 * t, w.attr + 3 * t);
}

// meshopt_simplifyWithAttributes(indices in place, Sparse, the decoded normals with weights 1, target_error 1e-1) over the
// mesh's vertex_count vertices; returns the result's index count, *out_error its error
__device__ inline uint32_t simplify(const Scratch& w, const Source& src, uint32_t* indices, uint32_t index_count, uint32_t target_index_count, float* out_error)
{
	// buildSparseRemap: sparse vertices in order of first appearance
	uint32_t vc = 0;
	for (uint32_t i = 0; i < index_count; ++i)
	{
		uint32_t index = indices[i], e = w.d2s[index];
		if (e == kNone)
		{
			e = w.d2s[index] = vc;
			w.sparse[vc++] = index;
		}
		indices[i] = e;
	}

	update_adjacency(w, indices, index_count, vc, nullptr);

	// buildPositionRemap: remap[i] = the first vertex whose position is float-equal to i's (-0 == +0; NaN equals nothing)
	const uint32_t table_size = hash_buckets(vc), hashmod = table_size - 1;
	for (uint32_t i = 0; i < table_size; ++i)
		w.table[i] = kNone;
	for (uint32_t i = 0; i < vc; ++i)
	{
		float p[3];
		uint32_t key[3];
		for (int k = 0; k < 3; ++k)
		{
			p[k] = src.position(w.sparse[i], k);
			key[k] = cook::float_bits(p[k]);
			key[k] = key[k] == 0x80000000u ? 0u : key[k];
			key[k] ^= key[k] >> 17;
		}
		uint32_t bucket = ((key[0] * 73856093u) ^ (key[1] * 19349663u) ^ (key[2] * 83492791u)) & hashmod;
		for (uint32_t probe = 0;; ++probe)
		{
			uint32_t item = w.table[bucket];
			if (item == kNone)
			{
				w.table[bucket] = i;
				w.remap[i] = i;
				break;
			}
			uint32_t ri = w.sparse[item];
			if (src.position(ri, 0) == p[0] && src.position(ri, 1) == p[1] && src.position(ri, 2) == p[2])
			{
				w.remap[i] = item;
				break;
			}
			bucket = (bucket + probe + 1) & hashmod;
		}
	}
	for (uint32_t i = 0; i < vc; ++i)
		w.wedge[i] = i;
	for (uint32_t i = 0; i < vc; ++i)
		if (w.remap[i] != i)
		{
			uint32_t r = w.remap[i];
			w.wedge[i] = w.wedge[r];
			w.wedge[r] = i;
		}

	classify(w, vc);

	// rescalePositions / rescaleAttributes over the sparse vertices
	float minv[3];
	float extent = extent_of(vc, [&](uint32_t i, int k) { return src.position(w.sparse[i], k); }, minv);
	float scale = extent == 0 ? 0.f : 1.f / extent;
	for (uint32_t i = 0; i < vc; ++i)
		for (int k = 0; k < 3; ++k)
		{
			w.pos[3 * i + k] = (src.position(w.sparse[i], k) - minv[k]) * scale;
			w.attr[3 * i + k] = src.normal(w.sparse[i], k);
		}

	const Quadric zero = { 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0 };
	for (uint32_t i = 0; i < vc; ++i)
	{
		w.vq[i] = zero;
		w.aq[i] = zero;
		for (int k = 0; k < 3; ++k)
			w.ag[3 * i + k] = Grad{ 0, 0, 0, 0 };
	}

	// fillFaceQuadrics
	for (uint32_t i = 0; i < index_count; i += 3)
	{
		uint32_t i0 = indices[i], i1 = indices[i + 1], i2 = indices[i + 2];
		Quadric Q;
		quadric_from_triangle(Q, w.pos + 3 * i0, w.pos + 3 * i1, w.pos + 3 * i2, 1.f);
		quadric_add(w.vq[w.remap[i0]], Q);
		quadric_add(w.vq[w.remap[i1]], Q);
		quadric_add(w.vq[w.remap[i2]], Q);
	}
	// fillVertexQuadrics: regularisation weight 1e-7
	for (uint32_t i = 0; i < vc; ++i)
	{
		if (w.remap[i] != i)
			continue;
		const float* p = w.pos + 3 * i;
		float wt = w.vq[i].w * 1e-7f;
		Quadric Q;
		Q.a00 = Q.a11 = Q.a22 = wt;
		Q.a10 = Q.a20 = Q.a21 = 0;
		Q.b0 = -p[0] * wt;
		Q.b1 = -p[1] * wt;
		Q.b2 = -p[2] * wt;
		Q.c = (p[0] * p[0] + p[1] * p[1] + p[2] * p[2]) * wt;
		Q.w = wt;
		quadric_add(w.vq[i], Q);
	}
	// fillEdgeQuadrics
	for (uint32_t i = 0; i < index_count; i += 3)
		for (int e = 0; e < 3; ++e)
		{
			uint32_t i0 = indices[i + e], i1 = indices[i + (e + 1) % 3];
			uint32_t k0 = w.kind[i0], k1 = w.kind[i1];
			bool edge0 = k0 == Border || k0 == Seam, edge1 = k1 == Border || k1 == Seam;
			if (!edge0 && !edge1)
				continue;
			if (edge0 && w.loop[i0] != i1)
				continue;
			if (edge1 && w.loopback[i1] != i0)
				continue;
			uint32_t i2 = indices[i + (e + 2) % 3];
			float edge_weight = (k0 == Border || k1 == Border) ? 10.f : 0.5f;
			Quadric Q, QT;
			quadric_from_triangle_edge(Q, w.pos + 3 * i0, w.pos + 3 * i1, w.pos + 3 * i2, edge_weight);
			quadric_from_triangle(QT, w.pos + 3 * i0, w.pos + 3 * i1, w.pos + 3 * i2, edge_weight);
			QT.w = 0;
			quadric_add(Q, QT);
			quadric_add(w.vq[w.remap[i0]], Q);
			quadric_add(w.vq[w.remap[i1]], Q);
		}
	// fillAttributeQuadrics
	for (uint32_t i = 0; i < index_count; i += 3)
	{
		uint32_t i0 = indices[i], i1 = indices[i + 1], i2 = indices[i + 2];
		Quadric QA;
		Grad G[3];
		quadric_from_attributes(QA, G, w.pos + 3 * i0, w.pos + 3 * i1, w.pos + 3 * i2, w.attr + 3 * i0, w.attr + 3 * i1, w.attr + 3 * i2);
		quadric_add(w.aq[i0], QA);
		quadric_add(w.aq[i1], QA);
		quadric_add(w.aq[i2], QA);
		grad_add(w.ag + 3 * i0, G);
		grad_add(w.ag + 3 * i1, G);
		grad_add(w.ag + 3 * i2, G);
	}

	// boundEdgeCollapses
	uint32_t dual_count = 0;
	for (uint32_t i = 0; i < vc; ++i)
		dual_count += (w.kind[i] == Manifold || w.kind[i] == Seam) ? w.adj_off[i + 1] - w.adj_off[i] : 0;
	const uint32_t collapse_capacity = (index_count - dual_count / 2) + 3;

	uint32_t result_count = index_count;
	float result_error = 0;
	const float error_limit = (kMaxError * kMaxError) / (1.f * 1.f);

	while (result_count > target_index_count)
	{
		update_adjacency(w, indices, result_count, vc, w.remap);

		// pickEdgeCollapses
		uint32_t collapse_count = 0;
		for (uint32_t i = 0; i < result_count; i += 3)
		{
			if (collapse_count + 3 > collapse_capacity)
				break;
			for (int e = 0; e < 3; ++e)
			{
				uint32_t i0 = indices[i + e], i1 = indices[i + (e + 1) % 3];
				if (w.remap[i0] == w.remap[i1])
					continue;
				uint32_t k0 = w.kind[i0], k1 = w.kind[i1];
				if (!(can_collapse(k0, k1) | can_collapse(k1, k0)))
					continue;
				if (has_opposite(k0, k1) && w.remap[i1] > w.remap[i0])
					continue;
				if ((k0 == Border || k0 == Seam) && k1 != Manifold && w.loop[i0] != i1)
					continue;
				if ((k1 == Border || k1 == Seam) && k0 != Manifold && w.loopback[i1] != i0)
					continue;
				if (can_collapse(k0, k1) & can_collapse(k1, k0))
					w.col[collapse_count++] = Collapse{ i0, i1, 1 };
				else
				{
					bool forward = can_collapse(k0, k1);
					w.col[collapse_count++] = Collapse{ forward ? i0 : i1, forward ? i1 : i0, 0 };
				}
			}
		}
		if (collapse_count == 0)
			break;

		// rankEdgeCollapses
		for (uint32_t i = 0; i < collapse_count; ++i)
		{
			Collapse& c = w.col[i];
			uint32_t i0 = c.v0, i1 = c.v1;
			bool bidi = c.bits != 0;
			float ei = quadric_error(w.vq[w.remap[i0]], w.pos + 3 * i1);
			float ej = bidi ? quadric_error(w.vq[w.remap[i1]], w.pos + 3 * i0) : FLT_MAX;
			ei += attribute_error(w, i0, i1);
			ej += bidi ? attribute_error(w, i1, i0) : 0;
			if (w.kind[i0] == Seam)
			{
				uint32_t s0 = w.wedge[i0];
				uint32_t s1 = w.loop[i0] == i1 ? w.loopback[s0] : w.loop[s0];
				s1 = s1 != kNone ? s1 : w.wedge[i1];
				ei += attribute_error(w, s0, s1);
				ej += bidi ? attribute_error(w, s1, s0) : 0;
			}
			else
			{
				if (w.kind[i0] == Complex)
					for (uint32_t v = w.wedge[i0]; v != i0; v = w.wedge[v])
						ei += attribute_error(w, v, complex_target(w, v, i1));
				if (w.kind[i1] == Complex && bidi)
					for (uint32_t v = w.wedge[i1]; v != i1; v = w.wedge[v])
						ej += attribute_error(w, v, complex_target(w, v, i0));
			}
			bool rev = bidi & (ej < ei);
			c.v0 = rev ? i1 : i0;
			c.v1 = rev ? i0 : i1;
			c.bits = cook::float_bits(ej < ei ? ej : ei);
		}

		// sortEdgeCollapses: stable counting sort on the top 12 bits below the sign
		for (uint32_t i = 0; i < kSortBins; ++i)
			w.hist[i] = 0;
		for (uint32_t i = 0; i < collapse_count; ++i)
		{
			uint32_t key = (w.col[i].bits << 1) >> 20;
			w.hist[key < kSortBins ? key : kSortBins - 1]++;
		}
		uint32_t sum = 0;
		for (uint32_t i = 0; i < kSortBins; ++i)
		{
			uint32_t count = w.hist[i];
			w.hist[i] = sum;
			sum += count;
		}
		for (uint32_t i = 0; i < collapse_count; ++i)
		{
			uint32_t key = (w.col[i].bits << 1) >> 20;
			w.order[w.hist[key < kSortBins ? key : kSortBins - 1]++] = i;
		}

		// performEdgeCollapses
		const uint32_t triangle_collapse_goal = (result_count - target_index_count) / 3;
		for (uint32_t i = 0; i < vc; ++i)
		{
			w.cremap[i] = i;
			w.clocked[i] = 0;
		}
		uint32_t edge_collapses = 0, triangle_collapses = 0, edge_collapse_goal = triangle_collapse_goal / 2;
		for (uint32_t i = 0; i < collapse_count; ++i)
		{
			const Collapse c = w.col[w.order[i]];
			const float error = cook::bits_float(c.bits);
			if (error > error_limit)
				break;
			if (triangle_collapses >= triangle_collapse_goal)
				break;
			float error_goal = edge_collapse_goal < collapse_count ? 1.5f * cook::bits_float(w.col[w.order[edge_collapse_goal]].bits) : FLT_MAX;
			if (error > error_goal && error > result_error && triangle_collapses > triangle_collapse_goal / 6)
				break;
			uint32_t i0 = c.v0, i1 = c.v1;
			uint32_t r0 = w.remap[i0], r1 = w.remap[i1];
			uint32_t kind = w.kind[i0];
			if (w.clocked[r0] | w.clocked[r1])
				continue;
			if (has_triangle_flips(w, r0, r1))
			{
				edge_collapse_goal++;
				continue;
			}
			if (kind == Complex)
			{
				uint32_t v = i0;
				do
				{
					w.cremap[v] = complex_target(w, v, i1);
					v = w.wedge[v];
				} while (v != i0);
			}
			else if (kind == Seam)
			{
				uint32_t s0 = w.wedge[i0];
				uint32_t s1 = w.loop[i0] == i1 ? w.loopback[s0] : w.loop[s0];
				s1 = s1 != kNone ? s1 : w.wedge[i1];
				w.cremap[i0] = i1;
				w.cremap[s0] = s1;
			}
			else
				w.cremap[i0] = i1;
			w.clocked[r0] = 1;
			w.clocked[r1] = 1;
			triangle_collapses += kind == Border ? 1 : 2;
			edge_collapses++;
			result_error = result_error < error ? error : result_error;
		}
		if (edge_collapses == 0)
			break;

		// updateQuadrics, sources in ascending index (vertex_error is only read by prune, which this path does not run)
		for (uint32_t i0 = 0; i0 < vc; ++i0)
		{
			uint32_t i1 = w.cremap[i0];
			if (i1 == i0)
				continue;
			uint32_t r0 = w.remap[i0], r1 = w.remap[i1];
			if (i0 == r0)
				quadric_add(w.vq[r1], w.vq[r0]);
			quadric_add(w.aq[i1], w.aq[i0]);
			grad_add(w.ag + 3 * i1, w.ag + 3 * i0);
		}

		// remapEdgeLoops, in place in ascending index as the reference does
		for (int side = 0; side < 2; ++side)
		{
			uint32_t* loop = side == 0 ? w.loop : w.loopback;
			for (uint32_t i = 0; i < vc; ++i)
				if (loop[i] != kNone)
				{
					uint32_t l = loop[i], r = w.cremap[l];
					loop[i] = i == r ? (loop[l] != kNone ? w.cremap[loop[l]] : kNone) : r;
				}
		}

		// remapIndexBuffer
		uint32_t write = 0;
		for (uint32_t i = 0; i < result_count; i += 3)
		{
			uint32_t v0 = w.cremap[indices[i]], v1 = w.cremap[indices[i + 1]], v2 = w.cremap[indices[i + 2]];
			uint32_t r0 = w.remap[v0], r1 = w.remap[v1], r2 = w.remap[v2];
			if (r0 != r1 && r0 != r2 && r1 != r2)
			{
				indices[write + 0] = v0;
				indices[write + 1] = v1;
				indices[write + 2] = v2;
				write += 3;
			}
		}
		result_count = write;
	}

	for (uint32_t i = 0; i < result_count; ++i)
		indices[i] = w.sparse[indices[i]];
	for (uint32_t i = 0; i < vc; ++i)
		w.d2s[w.sparse[i]] = kNone;
	*out_error = sqrtf(result_error) * 1.f;
	return result_count;
}

// ---- meshopt_optimizeVertexCache (vcacheoptimizer.cpp:169-343, kVertexScoreTable, cache size 16): tmp -> dst
__device__ inline float vertex_score(int cache_position, uint32_t live_triangles)
{
	const float cache[17] = { 0.f, 0.779f, 0.791f, 0.789f, 0.981f, 0.843f, 0.726f, 0.847f, 0.882f, 0.867f, 0.799f, 0.642f, 0.613f, 0.600f, 0.568f, 0.372f, 0.234f };
	const float live[9] = { 0.f, 0.995f, 0.713f, 0.450f, 0.404f, 0.059f, 0.005f, 0.147f, 0.006f };
	return cache[1 + cache_position] + live[live_triangles < 8 ? live_triangles : 8];
}

__device__ inline void optimize_vertex_cache(const Scratch& w, uint32_t* dst, const uint32_t* indices, uint32_t index_count, uint32_t vertex_count)
{
	if (index_count == 0 || vertex_count == 0)
		return;
	const uint32_t face_count = index_count / 3, cache_size = 16;
	uint32_t* counts = w.vcount;
	for (uint32_t i = 0; i < vertex_count; ++i)
		counts[i] = 0;
	for (uint32_t i = 0; i < index_count; ++i)
		counts[indices[i]]++;
	uint32_t offset = 0;
	for (uint32_t i = 0; i < vertex_count; ++i)
	{
		w.voff[i] = offset;
		offset += counts[i];
	}
	for (uint32_t i = 0; i < face_count; ++i)
		for (int k = 0; k < 3; ++k)
			w.vdata[w.voff[indices[i * 3 + k]]++] = i;
	for (uint32_t i = 0; i < vertex_count; ++i)
		w.voff[i] -= counts[i];

	for (uint32_t i = 0; i < face_count; ++i)
		w.emitted[i] = 0;
	for (uint32_t i = 0; i < vertex_count; ++i)
		w.vscore[i] = vertex_score(-1, counts[i]);
	for (uint32_t i = 0; i < face_count; ++i)
		w.tscore[i] = w.vscore[indices[i * 3]] + w.vscore[indices[i * 3 + 1]] + w.vscore[indices[i * 3 + 2]];

	uint32_t holder[2 * (16 + 4)];
	uint32_t* cache = holder;
	uint32_t* cache_new = holder + 16 + 4;
	uint32_t cache_count = 0;
	uint32_t current = 0, input_cursor = 1, output = 0;
	while (current != kNone)
	{
		uint32_t a = indices[current * 3], b = indices[current * 3 + 1], c = indices[current * 3 + 2];
		dst[output * 3] = a;
		dst[output * 3 + 1] = b;
		dst[output * 3 + 2] = c;
		output++;
		w.emitted[current] = 1;
		w.tscore[current] = 0;

		uint32_t cache_write = 0;
		cache_new[cache_write++] = a;
		cache_new[cache_write++] = b;
		cache_new[cache_write++] = c;
		for (uint32_t i = 0; i < cache_count; ++i)
		{
			uint32_t index = cache[i];
			cache_new[cache_write] = index;
			cache_write += (index != a) & (index != b) & (index != c);
		}
		uint32_t* t = cache;
		cache = cache_new;
		cache_new = t;
		cache_count = cache_write > cache_size ? cache_size : cache_write;

		for (int k = 0; k < 3; ++k)
		{
			uint32_t index = indices[current * 3 + k];
			uint32_t* neighbors = w.vdata + w.voff[index];
			uint32_t size = counts[index];
			for (uint32_t i = 0; i < size; ++i)
				if (neighbors[i] == current)
				{
					neighbors[i] = neighbors[size - 1];
					counts[index]--;
					break;
				}
		}

		uint32_t best_triangle = kNone;
		float best_score = 0;
		for (uint32_t i = 0; i < cache_write; ++i)
		{
			uint32_t index = cache[i];
			if (counts[index] == 0)
				continue;
			float score = vertex_score(i >= cache_size ? -1 : int(i), counts[index]);
			float score_diff = score - w.vscore[index];
			w.vscore[index] = score;
			const uint32_t* neighbors = w.vdata + w.voff[index];
			for (uint32_t n = 0; n < counts[index]; ++n)
			{
				uint32_t tri = neighbors[n];
				float tri_score = w.tscore[tri] + score_diff;
				best_triangle = best_score < tri_score ? tri : best_triangle;
				best_score = best_score < tri_score ? tri_score : best_score;
				w.tscore[tri] = tri_score;
			}
		}
		current = best_triangle;
		if (current == kNone)
		{
			while (input_cursor < face_count && w.emitted[input_cursor])
				++input_cursor;
			current = input_cursor < face_count ? input_cursor : kNone;
		}
	}
}

// appendMesh (scene.cpp:193-268) for one mesh: the Mesh record with chain-relative index offsets, the chain in w.out;
// returns the chain's index count.  A LOD 0 index >= vertexCount rejects the mesh before any vertex is read.
__device__ inline uint64_t cook_chain(const LodJob& job, const NvcVertex* vertices, const uint32_t* lod0, float max_scale, uint32_t* scratch, NvcMesh& mesh, bool& rejected)
{
	mesh = NvcMesh{};
	mesh.vertexOffset = job.vertex_offset;
	mesh.vertexCount = job.vertex_count;
	const uint32_t V = job.vertex_count, N = job.index_count;
	rejected = false;
	for (uint32_t i = 0; i < N; ++i)
		if (lod0[i] >= V)
		{
			rejected = true;
			return 0;
		}
	Scratch w;
	carve(V, N, job.capacity, scratch + job.scratch, &w);
	const Source src = { vertices + job.vertex_offset };

	// center: sequential float sum / float(count); radius: max of glm::distance(center, p) = length(p - center)
	float center[3] = { 0.f, 0.f, 0.f };
	for (uint32_t i = 0; i < V; ++i)
		for (int k = 0; k < 3; ++k)
			center[k] = x86_add(center[k], src.position(i, k));
	for (int k = 0; k < 3; ++k)
		center[k] = x86_div(center[k], float(V));
	float radius = 0;
	for (uint32_t i = 0; i < V; ++i)
	{
		float d[3];
		for (int k = 0; k < 3; ++k)
			d[k] = src.position(i, k) - center[k];
		float dist = sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
		radius = radius < dist ? dist : radius;
	}
	for (int k = 0; k < 3; ++k)
		mesh.center[k] = center[k];
	mesh.radius = radius;

	float minv[3];
	const float lod_scale = extent_of(V, [&](uint32_t i, int k) { return src.position(i, k); }, minv);

	for (uint32_t i = 0; i < V; ++i)
		w.d2s[i] = kNone;
	for (uint32_t i = 0; i < N; ++i)
		w.cur[i] = lod0[i];
	uint32_t n = N;
	uint64_t total = 0;
	float lod_error = 0.f;
	while (mesh.lodCount < NVC_MAX_LODS)
	{
		NvcMeshLod& lod = mesh.lods[mesh.lodCount++];
		lod.indexOffset = uint32_t(total);
		lod.indexCount = n;
		for (uint32_t i = 0; i < n; ++i)
			w.out[total + i] = w.cur[i];
		total += n;
		lod.error = x86_mul(lod_error, lod_scale);
		if (mesh.lodCount == NVC_MAX_LODS)
			break;
		const uint32_t target = uint32_t(uint64_t(double(n) * 0.6) / 3 * 3);
		float next_error = 0.f;
		const uint32_t next = simplify(w, src, w.cur, n, target, &next_error);
		if (next == n || next == 0)
			break;
		if (next >= uint64_t(double(n) * 0.85))
			break;
		n = next;
		lod_error = lod_error * 1.5f < next_error ? next_error : lod_error * 1.5f;
		for (uint32_t i = 0; i < n; ++i)
			w.tmp[i] = w.cur[i];
		optimize_vertex_cache(w, w.cur, w.tmp, n, V);
	}
	mesh.lodRT = cook::lod_rt(mesh, max_scale);
	return total;
}

} // namespace lods
} // namespace nvc
