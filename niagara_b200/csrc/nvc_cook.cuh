// nvc_cook.cuh — meshlet bounds + normal cone, SURVEY §8(f) row N4 (the producer of the Meshlet[] cull fields).
//
// Restates what the reference's cooker computes per meshlet (src/scene.cpp:24-83 appendMeshlet ->
// meshopt_computeMeshletBounds, extern/meshoptimizer/src/meshletutils.cpp:22-131,133-272,314-339, and the
// quantisation helpers of extern/meshoptimizer/src/quantization.cpp:14-37,60-78 / meshoptimizer.h:1133-1143) with the
// same operations in the same order, so that the result is BIT-IDENTICAL to the Meshlet[] the reference writes:
//   positions      = dequantizeHalf(Vertex.vx/vy/vz) of vertex baseVertex + ref[k]       (scene.cpp:193-198)
//   triangle plane = normalised cross product of (p1 - p0, p2 - p0), degenerate triangles dropped
//   bounding sphere (Ritter seeded by the extremal pair over 7 axes, then one growing pass) over the corners
//   cone axis      = centre of the bounding sphere (3 axes) of the unit normals, normalised; mindp = min dot
//   outputs        center/radius -> quantizeHalf, axis -> snorm8, cutoff -> snorm8 rounded up by the axis error
// The arithmetic is spelled through cook::mul/add/... which are __f*_rn intrinsics on the device (the TU is built
// -fmad=false as well) and plain operators on the host (tests compile this header with g++ -ffp-contract=off to
// check the algorithm against the reference's output before any GPU time is spent; the product only ships the kernel).
// Normals are recomputed on every pass instead of being stored (no per-thread arrays); identical inputs give
// identical bits, so this does not change the result.
#pragma once

#include "../../include/niagara_cull.h"

#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define NVC_HD __host__ __device__ __forceinline__
#else
#define NVC_HD inline
#endif

namespace nvc
{
namespace cook
{

#if defined(__CUDA_ARCH__)
NVC_HD float mul(float a, float b) { return __fmul_rn(a, b); }
NVC_HD float add(float a, float b) { return __fadd_rn(a, b); }
NVC_HD float sub(float a, float b) { return __fsub_rn(a, b); }
NVC_HD float div(float a, float b) { return __fdiv_rn(a, b); }
NVC_HD float root(float a) { return __fsqrt_rn(a); }
NVC_HD uint32_t float_bits(float f) { return __float_as_uint(f); }
NVC_HD float bits_float(uint32_t u) { return __uint_as_float(u); }
#else
NVC_HD float mul(float a, float b) { return a * b; }
NVC_HD float add(float a, float b) { return a + b; }
NVC_HD float sub(float a, float b) { return a - b; }
NVC_HD float div(float a, float b) { return a / b; }
NVC_HD float root(float a) { return sqrtf(a); }
NVC_HD uint32_t float_bits(float f)
{
	uint32_t u;
	memcpy(&u, &f, 4);
	return u;
}
NVC_HD float bits_float(uint32_t u)
{
	float f;
	memcpy(&f, &u, 4);
	return f;
}
#endif

struct V3
{
	float x, y, z;
};

// quantization.cpp:60-78: fp16 denormals flush to zero, inf/NaN keep their payload
NVC_HD float dequantize_half(uint16_t h)
{
	uint32_t s = uint32_t(h & 0x8000u) << 16;
	int32_t em = h & 0x7fff;
	int32_t r = (em + (112 << 10)) << 13;
	r = em < (1 << 10) ? 0 : r;
	r += em >= (31 << 10) ? (112 << 23) : 0;
	return bits_float(s | uint32_t(r));
}

// quantization.cpp:14-37: round half up in magnitude, flush below 2^-14, saturate to inf, any NaN -> 0x7e00
NVC_HD uint16_t quantize_half(float v)
{
	uint32_t ui = float_bits(v);
	int32_t s = int32_t((ui >> 16) & 0x8000u);
	int32_t em = int32_t(ui & 0x7fffffffu);
	int32_t h = (em - (112 << 23) + (1 << 12)) >> 13;
	h = em < (113 << 23) ? 0 : h;
	h = em >= (143 << 23) ? 0x7c00 : h;
	h = em > (255 << 23) ? 0x7e00 : h;
	return uint16_t(s | h);
}

// meshoptimizer.h:1133-1143: N-bit snorm, N = 8 for cone axes and 10 for OBJ normals
NVC_HD int quantize_snorm(float v, int N)
{
	const float scale = float((1 << (N - 1)) - 1);
	float round = v >= 0 ? 0.5f : -0.5f;
	v = v >= -1 ? v : -1;
	v = v <= +1 ? v : +1;
	return int(add(mul(v, scale), round));
}

NVC_HD float dot3(const float* a, const V3& p) { return add(add(mul(a[0], p.x), mul(a[1], p.y)), mul(a[2], p.z)); }

NVC_HD float distance2(const V3& a, const V3& b)
{
	float dx = sub(a.x, b.x), dy = sub(a.y, b.y), dz = sub(a.z, b.z);
	return add(add(mul(dx, dx), mul(dy, dy)), mul(dz, dz));
}

// meshletutils.cpp:22-131 with every radius = 0 (the `radii` argument is &rzero with stride 0 at both call sites).
// Points: point(i) for i < count.  `first` is the point the extremal slots start at (the reference initialises them
// to index 0 of the underlying array; they are overwritten by the first finite point, so only count == 0 or NaN
// input could tell the difference).
template <typename PointFn>
NVC_HD void bounding_sphere(const PointFn& point, uint32_t count, int axis_count, float result[4])
{
	const float axes[7][3] = {
		{ 1, 0, 0 }, { 0, 1, 0 }, { 0, 0, 1 },
		{ 0.57735026f, 0.57735026f, 0.57735026f }, { -0.57735026f, 0.57735026f, 0.57735026f },
		{ 0.57735026f, -0.57735026f, 0.57735026f }, { 0.57735026f, 0.57735026f, -0.57735026f },
	};

	uint32_t pmin[7], pmax[7];
	float tmin[7], tmax[7];
	for (int axis = 0; axis < axis_count; ++axis)
	{
		pmin[axis] = pmax[axis] = 0;
		tmin[axis] = FLT_MAX;
		tmax[axis] = -FLT_MAX;
	}
	for (uint32_t i = 0; i < count; ++i)
	{
		V3 p = point(i);
		for (int axis = 0; axis < axis_count; ++axis)
		{
			float tp = dot3(axes[axis], p);
			float tpmin = sub(tp, 0.0f), tpmax = add(tp, 0.0f);
			pmin[axis] = tpmin < tmin[axis] ? i : pmin[axis];
			pmax[axis] = tpmax > tmax[axis] ? i : pmax[axis];
			tmin[axis] = tpmin < tmin[axis] ? tpmin : tmin[axis];
			tmax[axis] = tpmax > tmax[axis] ? tpmax : tmax[axis];
		}
	}

	int paxis = 0;
	float paxisdr = 0;
	for (int axis = 0; axis < axis_count; ++axis)
	{
		float dr = add(add(root(distance2(point(pmax[axis]), point(pmin[axis]))), 0.0f), 0.0f);
		if (dr > paxisdr)
		{
			paxisdr = dr;
			paxis = axis;
		}
	}

	V3 p1 = point(pmin[paxis]), p2 = point(pmax[paxis]);
	float paxisd = root(distance2(p2, p1));
	float paxisk = paxisd > 0 ? div(sub(add(paxisd, 0.0f), 0.0f), mul(2.0f, paxisd)) : 0.0f;
	V3 center = { add(p1.x, mul(sub(p2.x, p1.x), paxisk)), add(p1.y, mul(sub(p2.y, p1.y), paxisk)), add(p1.z, mul(sub(p2.z, p1.z), paxisk)) };
	float radius = div(paxisdr, 2.0f);

	for (uint32_t i = 0; i < count; ++i)
	{
		V3 p = point(i);
		float d = root(distance2(p, center));
		if (add(d, 0.0f) > radius)
		{
			float k = d > 0 ? div(sub(add(d, 0.0f), radius), mul(2.0f, d)) : 0.0f;
			center.x = add(center.x, mul(k, sub(p.x, center.x)));
			center.y = add(center.y, mul(k, sub(p.y, center.y)));
			center.z = add(center.z, mul(k, sub(p.z, center.z)));
			radius = div(add(add(radius, d), 0.0f), 2.0f);
		}
	}
	result[0] = center.x;
	result[1] = center.y;
	result[2] = center.z;
	result[3] = radius;
}

// One meshlet: reads vertexCount / triangleCount / shortRefs / dataOffset / baseVertex, returns the four cull fields.
struct MeshletView
{
	const NvcVertex* vertices;
	const uint32_t* data; // meshletdata + dataOffset
	uint32_t baseVertex, vertexCount, triangleCount, shortRefs;

	NVC_HD uint32_t ref(uint32_t k) const
	{
		if (shortRefs)
			return (data[k >> 1] >> ((k & 1u) * 16u)) & 0xffffu;
		return data[k];
	}
	NVC_HD V3 position(uint32_t k) const
	{
		const NvcVertex& v = vertices[size_t(baseVertex) + ref(k)];
		return V3{ dequantize_half(v.vx), dequantize_half(v.vy), dequantize_half(v.vz) };
	}
	NVC_HD uint32_t corner(uint32_t t, uint32_t c) const
	{
		uint32_t words = shortRefs ? (vertexCount + 1u) / 2u : vertexCount;
		uint32_t byte = t * 3u + c;
		return (data[words + (byte >> 2)] >> ((byte & 3u) * 8u)) & 0xffu;
	}
	// meshletutils.cpp:140-172: unit normal of triangle t; false when the triangle is degenerate (area == 0)
	NVC_HD bool normal(uint32_t t, float n[4]) const
	{
		V3 p0 = position(corner(t, 0)), p1 = position(corner(t, 1)), p2 = position(corner(t, 2));
		float ax = sub(p1.x, p0.x), ay = sub(p1.y, p0.y), az = sub(p1.z, p0.z);
		float bx = sub(p2.x, p0.x), by = sub(p2.y, p0.y), bz = sub(p2.z, p0.z);
		float nx = sub(mul(ay, bz), mul(az, by));
		float ny = sub(mul(az, bx), mul(ax, bz));
		float nz = sub(mul(ax, by), mul(ay, bx));
		float area = root(add(add(mul(nx, nx), mul(ny, ny)), mul(nz, nz)));
		if (area == 0.0f)
			return false;
		nx = div(nx, area);
		ny = div(ny, area);
		nz = div(nz, area);
		n[0] = nx;
		n[1] = ny;
		n[2] = nz;
		n[3] = -add(add(mul(nx, p0.x), mul(ny, p0.y)), mul(nz, p0.z));
		return true;
	}
};

struct NormalPoints // the i-th NON-degenerate triangle's normal, as a point
{
	const MeshletView* m;
	bool dense; // no degenerate triangle: the i-th point is triangle i
	NVC_HD V3 operator()(uint32_t i) const
	{
		float n[4] = { 0, 0, 0, 0 };
		if (dense)
			m->normal(i, n);
		else
		{
			uint32_t seen = 0;
			for (uint32_t t = 0; t < m->triangleCount; ++t)
				if (m->normal(t, n))
				{
					if (seen == i)
						break;
					++seen;
				}
		}
		return V3{ n[0], n[1], n[2] };
	}
};

struct CornerPoints
{
	const MeshletView* m;
	NVC_HD V3 operator()(uint32_t i) const { return m->position(i); }
};

// writes center[3], radius (fp16 bits), cone_axis[3], cone_cutoff of *out; every other field is left alone
NVC_HD void meshlet_bounds(const MeshletView& m, NvcMeshlet* out)
{
	uint16_t center_h[3] = { 0, 0, 0 }, radius_h = 0;
	int8_t axis_s8[3] = { 0, 0, 0 }, cutoff_s8 = 0;

	// meshletutils.cpp:324-336: corners = references [0, highest index used by a triangle]
	uint32_t corner_count = 0, triangles = 0;
	float n[4];
	for (uint32_t t = 0; t < m.triangleCount; ++t)
	{
		for (uint32_t c = 0; c < 3; ++c)
		{
			uint32_t k = m.corner(t, c);
			corner_count = k >= corner_count ? k + 1 : corner_count;
		}
		triangles += m.normal(t, n) ? 1u : 0u;
	}

	if (triangles != 0) // :179-181 degenerate cluster: everything stays 0
	{
		float psphere[4], nsphere[4];
		bounding_sphere(CornerPoints{ &m }, corner_count, 7, psphere);
		bounding_sphere(NormalPoints{ &m, triangles == m.triangleCount }, triangles, 3, nsphere);

		float axis[3] = { nsphere[0], nsphere[1], nsphere[2] };
		float axislength = root(add(add(mul(axis[0], axis[0]), mul(axis[1], axis[1])), mul(axis[2], axis[2])));
		float invaxislength = axislength == 0.0f ? 0.0f : div(1.0f, axislength);
		axis[0] = mul(axis[0], invaxislength);
		axis[1] = mul(axis[1], invaxislength);
		axis[2] = mul(axis[2], invaxislength);

		float mindp = 1.0f;
		for (uint32_t t = 0; t < m.triangleCount; ++t)
			if (m.normal(t, n))
			{
				float dp = add(add(mul(n[0], axis[0]), mul(n[1], axis[1])), mul(n[2], axis[2]));
				mindp = dp < mindp ? dp : mindp;
			}

		center_h[0] = quantize_half(psphere[0]);
		center_h[1] = quantize_half(psphere[1]);
		center_h[2] = quantize_half(psphere[2]);
		radius_h = quantize_half(psphere[3]);

		if (mindp <= 0.1f) // :222-227 cone wider than ~168 degrees: never culls
			cutoff_s8 = 127;
		else
		{
			float cutoff = root(sub(1.0f, mul(mindp, mindp))); // :256
			float err = cutoff;
			for (int i = 0; i < 3; ++i)
			{
				int q = quantize_snorm(axis[i], 8);
				axis_s8[i] = int8_t(q);
				err = add(err, fabsf(sub(div(float(int(axis_s8[i])), 127.0f), axis[i]))); // :264-269, summed left to right
			}
			int c = int(add(mul(127.0f, err), 1.0f)); // :269 round up
			cutoff_s8 = c > 127 ? int8_t(127) : int8_t(c);
		}
	}

	memcpy(out->center, center_h, sizeof(center_h));
	memcpy(&out->radius, &radius_h, sizeof(radius_h));
	out->cone_axis[0] = axis_s8[0];
	out->cone_axis[1] = axis_s8[1];
	out->cone_axis[2] = axis_s8[2];
	out->cone_cutoff = cutoff_s8;
}

} // namespace cook
} // namespace nvc
