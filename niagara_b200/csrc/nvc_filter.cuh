// nvc_filter.cuh — conservative FILTER for the per-meshlet visibility test of clustercull.comp.glsl:72-124.
//
// The contract of the cluster pass is bit-exact DECISIONS (visible / not visible per meshlet), not bit-exact
// intermediates.  The exact restatement (nvc_math.cuh, strict IEEE, no contraction) costs ~500 instructions per
// meshlet and makes the pass issue-bound (DESIGN.md §5).  This header evaluates the same test with fused
// multiply-adds, MUFU reciprocals / square roots and per-COMMAND precomputed transforms, and attaches to every
// comparison a margin that bounds  |value computed here - value the exact path computes|.  A decision is taken here
// only when every comparison on its path clears its margin; everything else ("undecided") is handed to the exact
// path by the caller (a per-warp queue drained on full warps).  Wrong decisions are therefore impossible as long as the
// margins below are upper bounds; undecided items only cost time.
//
// Notation: u = 2^-24 (round-to-nearest unit roundoff).  "exact path" = nvc_math.cuh / oracle.cpp / the GLSL.
//
// ---- error model -------------------------------------------------------------------------------------------------
// (1) view-space centre.  Exact path: rotate_quat (math.h:46-49) -> *scale + position -> view * vec4 (14 roundings
//     deep).  Here: c = M*lc + T with M = scale * V3 * R(q), T = V3*t + tv built once per task command (build_record).
//     With q2 = |q|^2 <= 1.01 (checked per command; R(q) = (1-q2) I + q2 R(q/|q|), so |R(q)|_2 <= 1.02), Vr = max row
//     abs sum of V3 <= 2 (checked per launch), n = |lc|_2 <= l1 = |lc|_1, standard forward analysis gives
//        exact path:  |c_e - c*|_inf <= 25.6 Vr u s n + 5 u Tm        Tm_i = sum_j |V_ij||t_j| + |V_i3|
//        this path :  |c_a - c*|_inf <= 12.4 Vr u s l1 + 6 u Tm
//     so with  Em = 42 u s max(Vr,1),  Et = 12 u Tm + 4 u znear + 2^-100,  E = Em (l1 + |r_local|) + Et :
//        |c_e - c_a|_inf <= E,   u |c_i| <= E/12,   u r <= E/42        (r = r_local * s is computed identically)
// (2) frustum (clustercull.comp.glsl:104-108): both sides evaluate  c.z f1 - |c.x| f0 + r  etc. within
//     (|f0|+|f1|) 1.34 E of each other  ->  margin mF = 1.5 max(|f0|+|f1|, |f2|+|f3|, 1) E.  The far plane uses
//     zfar (1 -+ 2^-20) on the two sides so that no term proportional to u zfar enters E.
// (3) cone (math.h:41-44), compared after scaling by 127 s: |dot difference| <= 180 u |c|_1 + 6.2 E <= 51 E,
//     |rhs difference| <= 8 E  ->  margin 64 E (x 127 s, kept per command as kC).
// (4) projectSphere (math.h:2-22).  Here X+- = (cx cz +- r vx) / (cz^2 - r^2), algebraically equal to the reference's
//     (vx cx -+ cz r) / (vx cz +- cx r) but with ONE shared reciprocal.  With D = cz - r > 0 (guaranteed by the
//     "sphere clears the near plane" test), relE = E / D, g = 1 + r / D  and the validity cone (per axis)
//     |cx| + r sqrt(1+G^2) <= G cz, G = 1 / hP  (the sphere lies inside the wedge |x| <= G z, which bounds |X| hP <= 1):
//        |uv_e - uv_a| <= Kuv g relE,   Kuv = 1.1 sqrt2 (hP + 1/hP) + 0.62 (1 + hP) + 0.25 hP + 2.2   (max over axes)
//     (sensitivity of tan(theta +- phi) to the centre, the exact path's own rounding of its cancellation-prone
//     formula, and this path's rounding; derivation in DESIGN.md §5a).
// (5) mip selection (math.h:24-39): m = max(size) * pyramid size differs by <= dm = gr (Km1 + Km2 m), gr = g relE;
//     undecided when m is within dm of a power of two.  "fits" test at the finer level: px and the sum differ by
//     <= ef = 2^(1-L) (pmax Kuv gr + dm); undecided when fract(px) is within ef of 0 / 1 or the sum within ef of 2.
// (6) footprint (resources.cpp:294-325 MIN sampler): x = u w - 0.5 differs by <= efp = w Kuv gr; undecided when
//     fract(x) is within efp of 0 / 1 (this includes the fract == 0 special case of the sampler).  Decided items read
//     exactly the texels the exact path reads, so `depth` is the same float.
// (7) depthSphere = znear / (cz - r) differs by <= 1.7 relE depthSphere -> margin 2 relE depthSphere.
// (8) rcp.approx.ftz / sqrt.approx.ftz are within a relative 2^-22 of the true value only where argument and result are
//     normal: a subnormal argument is read as 0 and a subnormal result written as 0 (100 % error), and below ~2^-126 the
//     other products round with an absolute, not relative, error of 2^-150 that (1)-(7) do not budget.  The root of the
//     cone test and the shared reciprocal of (4) therefore decide only when their argument lies in [2^-110, 2^110]:
//     |c|^2 >= 2^-110 for the cone; c.z^2 - r^2 in [2^-110, 2^110] for the occlusion stage (then c.x^2 + c.z^2 - r^2 is
//     normal too, and c.z - r >= znear > 1e-30 is required anyway).  Inside that range every subnormal rounding is below
//     2^-40 relative to what it perturbs; the rest of the cone and the frustum are covered by the 2^-100 floor of E.
// Non-finite or out-of-range inputs never produce a decision: every "sure" predicate is a strict comparison that is
// false for NaN, commands with unusual transforms are flagged exact-only in build_record, and integer conversions are
// clamped first.  tests/filter_harness.cpp checks 10^8+ random / hostile items against the exact path with the MUFU
// results perturbed by +-2 ulp and flushed as the device flushes them, and checks the margins against a float64
// evaluation; tests/test_filter_approx.py compares both instructions on the H100 with float64 over all 2^32 inputs.
#pragma once

#include "nvc_internal.h"
#include "nvc_math.cuh"

#include <math.h>
#include <string.h>

namespace nvc
{

#if defined(NVC_EMU)
// CPU stand-ins with the special-value rules of the .ftz instructions: a subnormal argument is read as a zero of its sign, a
// subnormal result is written as one, NaN results are the canonical 0x7fffffff, sqrt(-0) = -0 and sqrt(x < 0) = NaN.
// NVF_PERTURB (tests) scales every normal result by 1 +- 2^-22 pseudo-randomly (the relative error budget of both instructions).
#ifdef NVF_PERTURB
extern thread_local uint32_t nvf_perturb_state;
__device__ __forceinline__ float nvf_jitter(float v)
{
	nvf_perturb_state = nvf_perturb_state * 1664525u + 1013904223u;
	uint32_t k = nvf_perturb_state >> 29; // 0..7
	const float f[8] = { 1.0f, 1.0f + 2.4e-7f, 1.0f - 2.4e-7f, 1.0f + 1.2e-7f, 1.0f - 1.2e-7f, 1.0f, 1.0f + 2.4e-7f, 1.0f - 2.4e-7f };
	return v * f[k];
}
#else
__device__ __forceinline__ float nvf_jitter(float v) { return v; }
#endif
__device__ __forceinline__ float nvf_ftz(float x)
{
	return (__float_as_uint(x) & 0x7f800000u) == 0u ? __uint_as_float(__float_as_uint(x) & 0x80000000u) : x;
}
__device__ __forceinline__ float nvf_result(float v)
{
	const uint32_t e = __float_as_uint(v) & 0x7f800000u;
	if (v != v)
		return __uint_as_float(0x7fffffffu);
	if (e == 0u)
		return nvf_ftz(v);
	return e == 0x7f800000u ? v : nvf_jitter(v);
}
__device__ __forceinline__ float nvf_rcp(float x) { return nvf_result(1.0f / nvf_ftz(x)); }
__device__ __forceinline__ float nvf_sqrt(float x) { return nvf_result(sqrtf(nvf_ftz(x))); }
#else
__device__ __forceinline__ float nvf_rcp(float x)
{
	float r;
	asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
	return r;
}
__device__ __forceinline__ float nvf_sqrt(float x)
{
	float r;
	asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
	return r;
}
#endif

__device__ __forceinline__ float nvf_fma(float a, float b, float c) { return __fmaf_rn(a, b, c); }

// Error model (8): the range of arguments of nvf_rcp / nvf_sqrt in which a decision may be taken
constexpr float kNvfMinArg = 7.7037198e-34f; // 2^-110
constexpr float kNvfMaxArg = 1.2980742e33f;  // 2^110

// Host side: the per-launch constants from the pass's CullData and pyramid (called by nvc_clustercull, nvc_api.cu).
// Anything unusual (non-finite view, huge row sums, non-positive projection scale, non power-of-two pyramid) switches
// the filter, or only its occlusion stage, off — the exact path then does that work.
inline FilterConsts make_filter_consts(const NvcCullData& cd, const HiZDesc& hiz, bool need_hiz)
{
	FilterConsts fc;
	memset(&fc, 0, sizeof(fc));
	const double u = 5.9604644775390625e-8;
	auto bits = [](float f) { uint32_t b; memcpy(&b, &f, 4); return b; };
	auto finite = [](double v) { return v == v && v - v == 0.0; };
	bool ok = true;
	double vr = 0;
	for (int i = 0; i < 3; ++i)
	{
		double row = fabs(double(cd.view[i])) + fabs(double(cd.view[4 + i])) + fabs(double(cd.view[8 + i]));
		ok = ok && finite(row) && finite(cd.view[12 + i]);
		vr = row > vr ? row : vr;
	}
	ok = ok && vr <= 2.0;
	for (int i = 0; i < 4; ++i)
		ok = ok && finite(cd.frustum[i]) && fabs(double(cd.frustum[i])) <= 4.0;
	ok = ok && finite(cd.znear) && cd.znear > 1e-30f && cd.znear < 1e15f && cd.zfar == cd.zfar && cd.zfar > 0.f;
	const double f01 = fabs(double(cd.frustum[0])) + fabs(double(cd.frustum[1])), f23 = fabs(double(cd.frustum[2])) + fabs(double(cd.frustum[3]));
	double fk = f01 > f23 ? f01 : f23;
	fk = fk > 1.0 ? fk : 1.0;
	fc.vrE = float(vr > 1.0 ? vr : 1.0) * 1.000001f;
	fc.fr.x = float(1.5 * fk);
	fc.fr.y = cd.zfar * (1.f - 9.5367431640625e-7f);
	fc.fr.z = cd.zfar * (1.f + 9.5367431640625e-7f);
	fc.fr.w = float(4.0 * u * double(cd.znear));
	fc.enabled = ok ? 1u : 0u;

	// occlusion stage
	bool occ = ok && need_hiz && finite(cd.P00) && finite(cd.P11) && cd.P00 > 9.765625e-4f && cd.P11 > 9.765625e-4f && cd.P00 < 1024.f && cd.P11 < 1024.f;
	occ = occ && finite(cd.pyramidWidth) && finite(cd.pyramidHeight) && cd.pyramidWidth >= 1.f && cd.pyramidHeight >= 1.f && cd.pyramidWidth <= 65536.f && cd.pyramidHeight <= 65536.f;
	occ = occ && hiz.levels >= 1 && hiz.levels <= NVC_MAX_HIZ_LEVELS && hiz.width >= 1 && hiz.height >= 1 && (hiz.width & (hiz.width - 1)) == 0 && (hiz.height & (hiz.height - 1)) == 0 && hiz.width <= 65536 && hiz.height <= 65536;
	if (occ)
	{
		const double hpx = 0.5 * double(cd.P00), hpy = 0.5 * double(cd.P11);
		fc.pr.x = float(hpx);
		fc.pr.y = float(-hpy);
		fc.cg.x = float(1.0 / hpx);
		fc.cg.y = float(sqrt(1.0 + 1.0 / (hpx * hpx)) * 1.000001);
		fc.cg.z = float(1.0 / hpy);
		fc.cg.w = float(sqrt(1.0 + 1.0 / (hpy * hpy)) * 1.000001);
		fc.pr.z = float(2.0 * hpx * double(cd.pyramidWidth));
		fc.pr.w = float(2.0 * hpy * double(cd.pyramidHeight));
		auto kuv = [](double hp) { return 1.1 * 1.41421356237 * (hp + 1.0 / hp) + 0.62 * (1.0 + hp) + 0.25 * hp + 2.2; };
		const double Kuv = kuv(hpx) > kuv(hpy) ? kuv(hpx) : kuv(hpy);
		const double pmax = double(cd.pyramidWidth > cd.pyramidHeight ? cd.pyramidWidth : cd.pyramidHeight);
		const double hpmax = hpx > hpy ? hpx : hpy, gmax = 1.0 / (hpx < hpy ? hpx : hpy);
		fc.Kuv = float(Kuv);
		fc.mk.z = float(pmax * Kuv * 1.05);
		fc.mk.x = float(pmax * (1.24 * (1.0 + hpmax) + 0.6) * 1.1);
		fc.mk.y = float((5.0 + gmax) * 1.1);
		fc.mk.w = float(2.0 * Kuv * 1.05);
		const float top = float(1u << (hiz.levels - 1));
		fc.lv.y = bits(top);
		fc.lv.x = bits(top * 2.f);
		fc.lv.z = bits(float(hiz.width));
		fc.lv.w = bits(float(hiz.height));
	}
	fc.occ_ok = occ ? 1u : 0u;
	return fc;
}

// What the filter needs per task command: 20 words in shared memory, read by every item of the command.
struct alignas(16) CmdRecord
{
	float4 row0, row1, row2; // (M_i0, M_i1, M_i2, T_i)
	float4 aux;              // s, Em, Et, flags as bits (bit 0 lateDrawVisibility, bit 1 exact-only)
	uint4 ids;               // taskOffset, meshletVisibilityOffset, the command's 64 visibility bits (lo, hi; 0 when the pass does not track them)
};
static_assert(sizeof(CmdRecord) == 80, "five 16-byte shared-memory loads");

constexpr uint32_t kRecLate = 1u, kRecExactOnly = 2u;

// Built once per task command by the lane that owns it.  view = CullData.view (column-major).
__device__ __forceinline__ void build_record(const FilterConsts& fc, const float* __restrict__ view, float4 d0, float4 d1, uint32_t taskOffset, uint32_t mvo, uint32_t bits_lo,
    uint32_t bits_hi, uint32_t lateVis, CmdRecord& rec)
{
	const float x = d1.x, y = d1.y, z = d1.z, w = d1.w, s = d0.w;
	const float xx = x * x, yy = y * y, zz = z * z, ww = w * w;
	const float xy = x * y, xz = x * z, yz = y * z, wx = w * x, wy = w * y, wz = w * z;
	// R(q): the linear map of math.h:46-49 (valid for any q, unit or not)
	const float r00 = nvf_fma(-2.f, yy + zz, 1.f), r01 = 2.f * (xy - wz), r02 = 2.f * (xz + wy);
	const float r10 = 2.f * (xy + wz), r11 = nvf_fma(-2.f, xx + zz, 1.f), r12 = 2.f * (yz - wx);
	const float r20 = 2.f * (xz - wy), r21 = 2.f * (yz + wx), r22 = nvf_fma(-2.f, xx + yy, 1.f);
	float tmax = 0.f, msum = 0.f;
	float4 rows[3];
#pragma unroll
	for (int i = 0; i < 3; ++i)
	{
		const float v0 = view[i], v1 = view[4 + i], v2 = view[8 + i], v3 = view[12 + i];
		float4 r;
		r.x = s * nvf_fma(v0, r00, nvf_fma(v1, r10, v2 * r20));
		r.y = s * nvf_fma(v0, r01, nvf_fma(v1, r11, v2 * r21));
		r.z = s * nvf_fma(v0, r02, nvf_fma(v1, r12, v2 * r22));
		r.w = nvf_fma(v0, d0.x, nvf_fma(v1, d0.y, nvf_fma(v2, d0.z, v3)));
		const float tm = nvf_fma(fabsf(v0), fabsf(d0.x), nvf_fma(fabsf(v1), fabsf(d0.y), nvf_fma(fabsf(v2), fabsf(d0.z), fabsf(v3))));
		tmax = fmaxf(tmax, tm);
		msum += fabsf(r.x) + fabsf(r.y) + fabsf(r.z) + fabsf(r.w) + tm;
		rows[i] = r;
	}
	const float q2 = (xx + yy) + (zz + ww);
	// sane = finite, moderate magnitudes (products of two centre-sized values stay far from overflow), near-unit quaternion
	const bool sane = q2 <= 1.01f && s > 9.094947e-13f /* 2^-40 */ && s < 1.0995116e12f /* 2^40 */ && msum < 1.0995116e12f;
	const float u = 5.9604645e-8f; // 2^-24
	rec.row0 = rows[0];
	rec.row1 = rows[1];
	rec.row2 = rows[2];
	rec.aux.x = s;
	rec.aux.y = 42.f * u * s * fc.vrE;
	rec.aux.z = nvf_fma(12.f * u, tmax, fc.fr.w) + 7.8886091e-31f /* 2^-100 */;
	rec.aux.w = __uint_as_float((lateVis == 1u ? kRecLate : 0u) | (sane ? 0u : kRecExactOnly));
	rec.ids = make_uint4(taskOffset, mvo, bits_lo, bits_hi);
}

// Result of the filter for one meshlet
#ifdef NVF_DEBUG
struct FilterDebug
{
	float c[3], r, E, aabb[4], gr, m, dm, ef, efp, dS, depth;
	int level, stage; // stage: bit0 frustum/cone undecided, bit1 ok-test, bit2 domain, bit3 level, bit4 fits, bit5 footprint, bit6 depth
};
extern thread_local FilterDebug* nvf_debug;
#endif

struct FilterResult
{
	bool decided; // false: the caller must run the exact path
	bool visible; // the GLSL's `visible` after all tests (meaningful when decided)
};

// The occlusion stage of the filter (drawcull.comp.glsl:88-103 == clustercull.comp.glsl:112-123) for a view-space sphere whose
// centre is known to within E per component of the exact path's (E must also satisfy u |c_i| <= E / 12 and u r <= E / 42; with an
// EXACT centre, E = 12 u max|c_i| + 42 u |r| does).  mF: margin of the near-plane test.  Outputs: occ_vis / occ_hid = the exact
// path surely returns visible / occluded; neither = undecided.
template <bool FP>
__device__ __forceinline__ void filter_occlusion(const FilterConsts& fc, const NvcCullData& cd, const HiZDesc& hiz, float cx, float cy, float cz, float r, float E, float mF, bool& occ_vis,
    bool& occ_hid
#ifdef NVF_DEBUG
    ,
    FilterDebug* dbg
#endif
)
{
	const float bn = cz - cd.znear;
	const float tn = bn - r; // ok = !(cz < r + znear)
	const bool sure_ok = tn > mF, sure_not_ok = tn < -mF;
	const float D = cz - r, Sz = cz + r;
	const float czr2 = D * Sz;
	const float iD = nvf_rcp(D), icz = nvf_rcp(czr2);
	const float relE = E * iD;
	const float g = nvf_fma(r, iD, 1.f);
	const float gr = g * relE;
	// domain of the error analysis: radius >= 0, sphere inside the validity cone, small relative uncertainty, c.z^2 - r^2 far
	// from the range where the approximate reciprocal / roots flush (then so is c.x^2 + c.z^2 - r^2 >= c.z^2 - r^2)
	const float cone_x = nvf_fma(-fc.cg.x, cz, nvf_fma(r, fc.cg.y, fabsf(cx))), cone_y = nvf_fma(-fc.cg.z, cz, nvf_fma(r, fc.cg.w, fabsf(cy)));
	const bool dom_ok = r >= 0.f && cone_x <= 0.f && cone_y <= 0.f && gr < 9.765625e-4f /* 2^-10 */ && czr2 >= kNvfMinArg && czr2 <= kNvfMaxArg; // (fc.occ_ok is checked by the host: nvc_clustercull)

	const float vx = nvf_sqrt(nvf_fma(cx, cx, czr2)), vy = nvf_sqrt(nvf_fma(cy, cy, czr2));
	const float cxz = cx * cz, cyz = cy * cz, rvx = r * vx, rvy = r * vy;
	const float kx = icz * fc.pr.x, ky = icz * fc.pr.y;
	const float aabb_x = nvf_fma(cxz - rvx, kx, 0.5f), aabb_z = nvf_fma(cxz + rvx, kx, 0.5f);
	const float aabb_y = nvf_fma(cyz + rvy, ky, 0.5f), aabb_w = nvf_fma(cyz - rvy, ky, 0.5f);

	// mip level: L = ceil(log2 m) clamped to [1, levels], as the exponent field Lb of 2^L
	const float Sx = rvx * (icz * fc.pr.z), Sy = rvy * (icz * fc.pr.w);
	const float m = fmaxf(Sx, Sy);
	uint32_t Lb = (__float_as_uint(m) + 0x007fffffu) & 0x7f800000u;
	Lb = min(max(Lb, 0x40000000u), fc.lv.x);
	const float P = __uint_as_float(Lb);
	const float dm = gr * nvf_fma(m, fc.mk.y, fc.mk.x);
	const bool lev_ok = (P - m) > dm && fabsf(nvf_fma(-0.5f, P, m)) > dm;

	// does the box fit 2x2 texels of the next finer mip?  scale = 2^(1-L)
	const float scale = __uint_as_float(0x7f800000u - Lb);
	const float px = (aabb_x * cd.pyramidWidth) * scale, py = (aabb_y * cd.pyramidHeight) * scale;
	const float fx = px - floorf(px), fy = py - floorf(py);
	const float dfx = nvf_fma(Sx, scale, fx) - 2.f, dfy = nvf_fma(Sy, scale, fy) - 2.f;
	const float ef = scale * nvf_fma(gr, fc.mk.z, dm);
	const float hf = 0.5f - ef;
	const float dmax = fmaxf(dfx, dfy);
	const bool fits = dmax < -ef;
	const bool fit_ok = fabsf(fx - 0.5f) < hf && fabsf(fy - 0.5f) < hf && (fits || dmax > ef);

	// final level (exponent field) and its size
	const uint32_t LbF = min(Lb - (fits ? 0x00800000u : 0u), fc.lv.y);
	const uint32_t level = (LbF >> 23) - 127u;
	const float wf = fmaxf(__uint_as_float(fc.lv.z + 0x3f800000u - LbF), 1.f), hf2 = fmaxf(__uint_as_float(fc.lv.w + 0x3f800000u - LbF), 1.f);
	const float whx = 0.5f * wf, why = 0.5f * hf2;
	const float x = nvf_fma(aabb_x + aabb_z, whx, -0.5f), y = nvf_fma(aabb_y + aabb_w, why, -0.5f);
	const float flx = floorf(x), fly = floorf(y);
	const float efp = (fmaxf(whx, why) * gr) * fc.mk.w;
	const float hfp = 0.5f - efp;
	const bool fp_ok = fabsf((x - flx) - 0.5f) < hfp && fabsf((y - fly) - 0.5f) < hfp;
	const bool robust = sure_ok && dom_ok && lev_ok && fit_ok && fp_ok;

	const float wmax = wf - 1.f, hmax = hf2 - 1.f;
	const uint32_t wi = max(1u, hiz.width >> level);
	float depth;
	if (FP && level >= hiz.fp_first)
	{
		// fract != 0 on both axes here, so all four texels of the footprint count: one load from the footprint image
		const uint32_t ix = (uint32_t)(fminf(fmaxf(flx, -1.f), wmax) + 1.f), iy = (uint32_t)(fminf(fmaxf(fly, -1.f), hmax) + 1.f);
		depth = __ldg(hiz.fp + (hiz.fp_offset[level] + iy * fp_pitch(wi) + ix));
	}
	else
	{
		const uint32_t x0 = (uint32_t)fminf(fmaxf(flx, 0.f), wmax), x1 = (uint32_t)fminf(fmaxf(flx + 1.f, 0.f), wmax);
		const uint32_t y0 = (uint32_t)fminf(fmaxf(fly, 0.f), hmax), y1 = (uint32_t)fminf(fmaxf(fly + 1.f, 0.f), hmax);
		const uint32_t base = hiz.level_offset[level];
		const uint32_t r0 = base + y0 * wi, r1 = base + y1 * wi;
		// clamped indices are always inside the level: the four loads are unconditional and in flight together
		const float t00 = __ldg(hiz.texels + (r0 + x0)), t01 = __ldg(hiz.texels + (r0 + x1));
		const float t10 = __ldg(hiz.texels + (r1 + x0)), t11 = __ldg(hiz.texels + (r1 + x1));
		depth = fminf(fminf(t00, t01), fminf(t10, t11)); // fract != 0 on both axes here: all four texels count
	}

	const float dS = cd.znear * iD;
	const float dd = dS - depth;
	const float md = dS * (2.f * relE);
	occ_vis = sure_not_ok || (robust && dd > md);
	occ_hid = robust && dd < -md;

#ifdef NVF_DEBUG
	if (dbg)
	{
		FilterDebug& d = *dbg;
		d.aabb[0] = aabb_x, d.aabb[1] = aabb_y, d.aabb[2] = aabb_z, d.aabb[3] = aabb_w;
		d.gr = gr, d.m = m, d.dm = dm, d.ef = ef, d.efp = efp, d.dS = dS, d.depth = depth, d.level = int(level);
		d.stage = (!(sure_ok || sure_not_ok) ? 2 : 0) | (!dom_ok ? 4 : 0) | (!lev_ok ? 8 : 0) | (!fit_ok ? 16 : 0) | (!fp_ok ? 32 : 0) | (!(dd > md || dd < -md) ? 64 : 0);
	}
#endif
}

// One meshlet through the filter.  `b0`, `b1`: first 12 bytes of the Meshlet (center/radius halves, cone s8 x 4).
// LATE && occlusion: the Hi-Z stage runs; `backface`: clusterBackfaceEnabled != 0.
template <bool LATE, bool FP>
__device__ __forceinline__ FilterResult filter_meshlet(const FilterConsts& fc, const NvcCullData& cd, const HiZDesc& hiz, const float4 row0, const float4 row1, const float4 row2,
    const float4 aux, uint2 b0, uint32_t b1, bool backface, bool occlusion)
{
	FilterResult res;
	const float lx = half_bits_to_float(b0.x & 0xffffu), ly = half_bits_to_float(b0.x >> 16), lz = half_bits_to_float(b0.y & 0xffffu), rl = half_bits_to_float(b0.y >> 16);
	const float cx = nvf_fma(row0.x, lx, nvf_fma(row0.y, ly, nvf_fma(row0.z, lz, row0.w)));
	const float cy = nvf_fma(row1.x, lx, nvf_fma(row1.y, ly, nvf_fma(row1.z, lz, row1.w)));
	const float cz = nvf_fma(row2.x, lx, nvf_fma(row2.y, ly, nvf_fma(row2.z, lz, row2.w)));
	const float r = __fmul_rn(rl, aux.x); // identical to the exact path's radius
	const float l1 = (fabsf(lx) + fabsf(ly)) + (fabsf(lz) + fabsf(rl));
	const float E = nvf_fma(aux.y, l1, aux.z); // inf / NaN when any meshlet field is not finite: nothing below is "sure" then

	// ---- frustum: every test has the form  b > -r --------------------------------------------------------------
	const float mF = fc.fr.x * E;
	const float bx = nvf_fma(-fabsf(cx), cd.frustum[0], cz * cd.frustum[1]);
	const float by = nvf_fma(-fabsf(cy), cd.frustum[2], cz * cd.frustum[3]);
	const float bn = cz - cd.znear;
	const float m3 = fminf(fminf(bx, by), bn); // operands are finite (sane record, finite meshlet) or E is not
	const float rp = mF - r, rm = -mF - r;
	bool pass = fminf(m3, fc.fr.y - cz) > rp;
	bool fail = m3 < rm || (fc.fr.z - cz) < rm;

	// ---- cone, scaled by 127 s -------------------------------------------------------------------------------------
	if (backface)
	{
		const float ax = (float)(int8_t)(b1 & 0xffu), ay = (float)(int8_t)((b1 >> 8) & 0xffu), az = (float)(int8_t)((b1 >> 16) & 0xffu), ac = (float)(int8_t)(b1 >> 24);
		const float Ax = nvf_fma(row0.x, ax, nvf_fma(row0.y, ay, row0.z * az));
		const float Ay = nvf_fma(row1.x, ax, nvf_fma(row1.y, ay, row1.z * az));
		const float Az = nvf_fma(row2.x, ax, nvf_fma(row2.y, ay, row2.z * az));
		const float dotv = nvf_fma(cx, Ax, nvf_fma(cy, Ay, cz * Az));
		const float lsq = nvf_fma(cx, cx, nvf_fma(cy, cy, cz * cz));
		const float len = nvf_sqrt(lsq);
		const float rhs = aux.x * nvf_fma(ac, len, 127.f * r);
		const float tc = rhs - dotv; // > 0: not back-facing
		const float mC = (8300.f * aux.x) * E; // 64 E x 127 s (+2 %)
		const bool cone_dom = lsq >= kNvfMinArg; // the root is not flushed, and the squares' subnormal rounding is negligible
		pass = pass && tc > mC && cone_dom;
		fail = fail || (tc < -mC && cone_dom);
	}

	if (!LATE || !occlusion)
	{
		res.decided = pass || fail;
		res.visible = pass;
		return res;
	}

	// ---- occlusion ----
	bool occ_vis, occ_hid;
#ifdef NVF_DEBUG
	filter_occlusion<FP>(fc, cd, hiz, cx, cy, cz, r, E, mF, occ_vis, occ_hid, nvf_debug);
#else
	filter_occlusion<FP>(fc, cd, hiz, cx, cy, cz, r, E, mF, occ_vis, occ_hid);
#endif

	res.decided = fail || occ_hid || (pass && occ_vis);
	res.visible = pass && occ_vis && !fail && !occ_hid;
#ifdef NVF_DEBUG
	if (nvf_debug)
	{
		FilterDebug& d = *nvf_debug;
		d.c[0] = cx, d.c[1] = cy, d.c[2] = cz, d.r = r, d.E = E;
		d.stage |= !(pass || fail) ? 1 : 0;
	}
#endif
	return res;
}

} // namespace nvc
