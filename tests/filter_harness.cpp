// TEST INFRASTRUCTURE — large-scale check of the conservative meshlet filter (niagara_b200/csrc/nvc_filter.cuh) against
// the exact per-meshlet test (nvc_math.cuh, the same functions the exact kernel path and the oracle restate).
// Built by tests/test_filter.py with g++ against tests/cuda_emu/include (NVC_EMU, NVF_PERTURB, NVF_DEBUG):
//   * every DECIDED item must agree with the exact decision (a single mismatch fails the run);
//   * the approximate reciprocals / roots are perturbed by up to +-2 ulp (the hardware's MUFU error budget);
//   * the margins are compared with what they bound: |c_exact - c_filter| / E and |aabb_exact - aabb_filter| / (Kuv g relE),
//     the largest ratio seen is reported (must stay < 1; the analysis says ~0.1-0.3 typically);
//   * the share of undecided items is reported per scenario and per stage.
// Usage: filter_harness <scenario> <items> <seed> [threads]
#include "cuda_runtime.h"

#include <stdio.h>

#include <atomic>
#include <random>
#include <thread>
#include <vector>

#include "nvc_filter.cuh"

namespace nvc
{
thread_local uint32_t nvf_perturb_state = 12345u;
thread_local FilterDebug* nvf_debug = nullptr;
} // namespace nvc

extern "C" void nvc_host_cull_data(const NvcCamera* camera, uint32_t screen_width, uint32_t screen_height, uint32_t draw_count, const NvcCullOptions* options, NvcCullData* out, float* out_projection16);
extern "C" int nvc_hiz_layout(uint32_t depth_width, uint32_t depth_height, NvcHiZ* out);

using namespace nvc;

struct HiZLoadHost
{
	const float* texels;
	uint32_t offset;
	float operator()(uint32_t idx) const { return texels[offset + idx]; }
};

// clustercull.comp.glsl:72-124 for one meshlet, strict IEEE (the per-lane body of meshlet_compute in nvc_kernels.cu)
static bool exact_visible(const NvcCullData& cd, const HiZDesc& hiz, float4 d0, float4 d1, uint2 b0, uint32_t b1, bool late, float* out_center, float* out_aabb, bool* out_ok)
{
	f3 lc = { half_bits_to_float(b0.x & 0xffffu), half_bits_to_float(b0.x >> 16), half_bits_to_float(b0.y & 0xffffu) };
	f3 rc = rotate_quat(lc, d1);
	f3 center = { __fadd_rn(__fmul_rn(rc.x, d0.w), d0.x), __fadd_rn(__fmul_rn(rc.y, d0.w), d0.y), __fadd_rn(__fmul_rn(rc.z, d0.w), d0.z) };
	center = transform_point(cd.view, center);
	float radius = __fmul_rn(half_bits_to_float(b0.y >> 16), d0.w);
	out_center[0] = center.x, out_center[1] = center.y, out_center[2] = center.z;
	bool alive = frustum_visible(cd, center, radius);
	if (cd.clusterBackfaceEnabled != 0)
	{
		f3 la = { s8_div127(int(int8_t(b1 & 0xffu))), s8_div127(int(int8_t((b1 >> 8) & 0xffu))), s8_div127(int(int8_t((b1 >> 16) & 0xffu))) };
		f3 axis = transform_vector(cd.view, rotate_quat(la, d1));
		float cutoff = s8_div127(int(int8_t(b1 >> 24)));
		bool backface = dot3(center, axis) >= __fadd_rn(__fmul_rn(cutoff, length3(center)), radius);
		alive = alive && !backface;
	}
	*out_ok = false;
	if (late && cd.clusterOcclusionEnabled == 1)
	{
		float4 aabb;
		bool ok = project_sphere(center, radius, cd.znear, cd.P00, cd.P11, aabb);
		out_aabb[0] = aabb.x, out_aabb[1] = aabb.y, out_aabb[2] = aabb.z, out_aabb[3] = aabb.w;
		*out_ok = ok;
		int level = occlusion_mip(aabb, cd.pyramidWidth, cd.pyramidHeight, int(hiz.levels) - 1);
		uint32_t w = max(1u, hiz.width >> level), h = max(1u, hiz.height >> level);
		float u = __fmul_rn(__fadd_rn(aabb.x, aabb.z), 0.5f);
		float v = __fmul_rn(__fadd_rn(aabb.y, aabb.w), 0.5f);
		HiZLoadHost load = { hiz.texels, hiz.level_offset[level] };
		float depth = sample_min(load, w, h, u, v);
		float depthSphere = __fdiv_rn(cd.znear, __fsub_rn(center.z, radius));
		bool occ = !ok || depthSphere > depth;
		alive = alive && occ;
	}
	return alive;
}

struct Stats
{
	uint64_t items = 0, undecided = 0, wrong = 0, visible = 0, exact_only = 0;
	uint64_t xc_items = 0, xc_undecided = 0, xc_wrong = 0; // occlusion stage alone on the EXACT centre (the drawcull use)
	uint64_t stage[7] = { 0, 0, 0, 0, 0, 0, 0 };
	double max_c_ratio = 0, max_uv_ratio = 0;
};

struct Scenario
{
	const char* name;
	int kind; // 0 C4-like, 1 big local coordinates (bistro-like), 2 hostile bits, 3 near the camera, 4 random camera + big world offsets,
	          // 5 subnormal: znear, scale and view-space magnitudes where |c|^2, c.x^2 + c.z^2 - r^2 and c.z^2 - r^2 straddle [2^-149, 2^-126)
};

static uint16_t to_half(float f)
{
	// round-to-nearest-even float -> half (finite inputs in half range)
	uint32_t b;
	memcpy(&b, &f, 4);
	uint32_t sign = (b >> 16) & 0x8000u;
	int32_t e = int32_t((b >> 23) & 0xff) - 127 + 15;
	uint32_t m = b & 0x7fffffu;
	if (e <= 0)
	{
		if (e < -10)
			return uint16_t(sign);
		m |= 0x800000u;
		uint32_t shift = uint32_t(14 - e);
		uint32_t r = m >> shift;
		uint32_t rem = m & ((1u << shift) - 1u), half = 1u << (shift - 1);
		if (rem > half || (rem == half && (r & 1u)))
			++r;
		return uint16_t(sign | r);
	}
	if (e >= 31)
		return uint16_t(sign | 0x7c00u);
	uint32_t r = (uint32_t(e) << 10) | (m >> 13);
	uint32_t rem = m & 0x1fffu;
	if (rem > 0x1000u || (rem == 0x1000u && (r & 1u)))
		++r;
	return uint16_t(sign | r);
}

static void run(const Scenario& sc, uint64_t items, uint32_t seed, Stats& st)
{
	std::mt19937_64 rng(seed);
	std::uniform_real_distribution<double> U(0.0, 1.0);
	auto uni = [&](double a, double b) { return a + (b - a) * U(rng); };
	nvf_perturb_state = seed * 2654435761u + 1u;
	FilterDebug dbg;
	nvf_debug = &dbg;

	uint64_t done = 0;
	while (done < items)
	{
		// ---- one "frame": camera, screen, pyramid ----
		const uint32_t sizes[5][2] = { { 4096, 4096 }, { 1920, 1080 }, { 1024, 768 }, { 3840, 2160 }, { 512, 2048 } };
		const uint32_t* sz = sizes[rng() % 5];
		NvcCamera cam;
		memset(&cam, 0, sizeof(cam));
		cam.orientation[3] = 1.f;
		cam.fovY = float(uni(0.5, 1.6));
		cam.znear = float(sc.kind == 5 ? pow(10.0, uni(-29.9, -18.0)) : sc.kind == 3 ? uni(0.01, 0.5) : uni(0.05, 1.0));
		double world = 0;
		if (sc.kind == 4 || sc.kind == 5 || (rng() & 3) == 0)
		{
			// random orientation; kind 4 also moves the whole scene far from the origin, kind 5 keeps the camera within a few znear of it
			double q[4] = { uni(-1, 1), uni(-1, 1), uni(-1, 1), uni(-1, 1) };
			double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
			for (int i = 0; i < 4; ++i)
				cam.orientation[i] = float(q[i] / n);
			world = sc.kind == 4 ? uni(0, 3000) : sc.kind == 5 ? 4.0 * cam.znear : uni(0, 50);
			for (int i = 0; i < 3; ++i)
				cam.position[i] = float(uni(-world, world));
		}
		NvcCullOptions opt = { float(uni(100, 1000)), 1, 1, 1, 1, 1, 0 };
		NvcCullData cd;
		nvc_host_cull_data(&cam, sz[0], sz[1], 1000, &opt, &cd, nullptr);
		cd.clusterBackfaceEnabled = (rng() & 7) ? 1 : 0;
		NvcHiZ hz;
		nvc_hiz_layout(sz[0], sz[1], &hz);
		std::vector<float> texels(hz.total_texels);
		{
			// blocky random depth: a few planes per 16x16 block of each level (values znear / z), some zeros (sky)
			for (uint32_t l = 0; l < hz.levels; ++l)
			{
				uint32_t w = std::max(1u, hz.width >> l), h = std::max(1u, hz.height >> l);
				float* t = texels.data() + hz.level_offset[l];
				uint32_t bw = (w + 15) / 16;
				std::vector<float> planes(size_t(bw) * ((h + 15) / 16));
				for (auto& p : planes)
					p = (rng() & 3) == 0 ? 0.f : float(sc.kind == 5 ? cd.znear / pow(2.0, uni(-78.0, -55.0)) : cd.znear / uni(2.0, 400.0));
				for (uint32_t y = 0; y < h; ++y)
					for (uint32_t x = 0; x < w; ++x)
						t[size_t(y) * w + x] = planes[(y / 16) * bw + x / 16];
			}
		}
		HiZDesc hiz;
		memset(&hiz, 0, sizeof(hiz));
		hiz.texels = texels.data();
		hiz.width = hz.width, hiz.height = hz.height, hiz.levels = hz.levels;
		memcpy(hiz.level_offset, hz.level_offset, sizeof(hiz.level_offset));
		hiz.stage_level = hz.levels;
		// footprint image (what footprint_kernel builds)
		std::vector<float> fp;
		{
			uint32_t total = 0;
			for (uint32_t l = 0; l < hz.levels; ++l)
			{
				uint32_t w = std::max(1u, hz.width >> l), h = std::max(1u, hz.height >> l);
				hiz.fp_offset[l] = total;
				total += fp_pitch(w) * (h + 1);
			}
			fp.resize(total);
			for (uint32_t l = 0; l < hz.levels; ++l)
			{
				uint32_t w = std::max(1u, hz.width >> l), h = std::max(1u, hz.height >> l);
				const float* t = texels.data() + hz.level_offset[l];
				for (uint32_t iy = 0; iy <= h; ++iy)
					for (uint32_t ix = 0; ix <= w; ++ix)
					{
						uint32_t x0 = ix ? ix - 1 : 0, x1 = std::min(ix, w - 1), y0 = iy ? iy - 1 : 0, y1 = std::min(iy, h - 1);
						fp[hiz.fp_offset[l] + iy * fp_pitch(w) + ix] = fminf(fminf(t[y0 * w + x0], t[y0 * w + x1]), fminf(t[y1 * w + x0], t[y1 * w + x1]));
					}
			}
			hiz.fp = fp.data();
			hiz.fp_first = uint32_t((done / 2000000) % 3); // the kernels take the four-texel path below this mip
		}
		FilterConsts fc = make_filter_consts(cd, hiz, true);

		// view-space -> world: world = R_cam * (vx, vy, -vz) + pos  (view = inverse camera transform with z flipped)
		const float* V = cd.view;
		auto to_world = [&](double vx, double vy, double vz, float* out) {
			// solve V3 * w + tv = v  with V3 orthonormal: w = V3^T (v - tv)
			double v[3] = { vx - V[12], vy - V[13], vz - V[14] };
			for (int j = 0; j < 3; ++j)
				out[j] = float(V[4 * j + 0] * v[0] + V[4 * j + 1] * v[1] + V[4 * j + 2] * v[2]);
		};

		// one wrong decision as a reproducible item (float fields as bit patterns) on stderr: camera, screen, draw, meshlet
		auto print_case = [&](const char* check, float4 d0, float4 d1, uint2 b0, uint32_t b1, bool exact, bool got) {
			auto fb = [](float f) { return __float_as_uint(f); };
			fprintf(stderr,
			    "CASE {\"scenario\": \"%s\", \"check\": \"%s\", \"camera\": [%u, %u, %u, %u, %u, %u, %u, %u, %u], \"screen\": [%u, %u], \"draw_distance\": %u, \"backface\": %d, "
			    "\"draw\": [%u, %u, %u, %u, %u, %u, %u, %u], \"meshlet\": [%u, %u, %u], \"exact\": %d, \"filter\": %d}\n",
			    sc.name, check, fb(cam.position[0]), fb(cam.position[1]), fb(cam.position[2]), fb(cam.orientation[0]), fb(cam.orientation[1]), fb(cam.orientation[2]), fb(cam.orientation[3]), fb(cam.fovY),
			    fb(cam.znear), sz[0], sz[1], fb(opt.draw_distance), int(cd.clusterBackfaceEnabled), fb(d0.x), fb(d0.y), fb(d0.z), fb(d0.w), fb(d1.x), fb(d1.y), fb(d1.z), fb(d1.w), b0.x, b0.y, b1,
			    int(exact), int(got));
		};
		const uint64_t frame_items = std::min<uint64_t>(items - done, 2000000);
		const uint32_t per_draw = sc.kind == 2 ? 1 : 10;
		const double ty = tan(cam.fovY * 0.5), tx = ty * double(sz[0]) / double(sz[1]);
		for (uint64_t i = 0; i < frame_items;)
		{
			// ---- one draw ----
			float4 d0, d1;
			double sscale, rho = 0;
			if (sc.kind == 5)
			{
				// view-space distance rho in [2^-77, 2^-50]: |c|^2 from below 2^-149 to above the filter's 2^-110 (nvc_filter.cuh (8)),
				// mostly inside the frustum, some beside or behind the eye
				rho = pow(2.0, uni(-77.0, -50.0));
				double v[3] = { uni(-1, 1) * tx * 1.15, uni(-1, 1) * ty * 1.15, (rng() & 7) ? 1.0 : uni(-1, 1) };
				const double vn = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
				float pos[3];
				to_world(rho * v[0] / vn, rho * v[1] / vn, rho * v[2] / vn, pos);
				sscale = pow(2.0, uni(-39.99, -30.0));
				double q[4] = { uni(-1, 1), uni(-1, 1), uni(-1, 1), uni(-1, 1) };
				const double qn = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
				d1 = make_float4(float(q[0] / qn), float(q[1] / qn), float(q[2] / qn), float(q[3] / qn));
				d0 = make_float4(pos[0], pos[1], pos[2], float(sscale));
			}
			else if (sc.kind == 2)
			{
				// hostile: arbitrary bit patterns in a third of the cases, wild magnitudes otherwise
				auto wild = [&]() -> float {
					uint32_t r = uint32_t(rng());
					if ((r & 3) == 0)
					{
						float f;
						uint32_t b = uint32_t(rng());
						memcpy(&f, &b, 4);
						return f;
					}
					return float(uni(-1, 1) * pow(10.0, uni(-6, 6)));
				};
				d0 = make_float4(wild(), wild(), wild(), wild());
				d1 = make_float4(wild(), wild(), wild(), wild());
				if (rng() & 1)
				{
					double n = sqrt(double(d1.x) * d1.x + double(d1.y) * d1.y + double(d1.z) * d1.z + double(d1.w) * d1.w);
					if (n > 0 && n < 1e30)
						d1 = make_float4(float(d1.x / n), float(d1.y / n), float(d1.z / n), float(d1.w / n));
				}
				sscale = d0.w;
			}
			else
			{
				double z = sc.kind == 3 ? uni(0.0, 6.0) : pow(uni(pow(4.0, 3), pow(double(opt.draw_distance) * 1.1, 3)), 1.0 / 3.0);
				double fill = 1.15; // some draws straddle / leave the frustum
				double vx = uni(-1, 1) * tx * z * fill, vy = uni(-1, 1) * ty * z * fill;
				float pos[3];
				to_world(vx, vy, z, pos);
				sscale = sc.kind == 1 ? uni(0.5, 1.5) : uni(2.0, 4.0);
				double ax[3] = { uni(-1, 1), uni(-1, 1), uni(-1, 1) };
				double an = sqrt(ax[0] * ax[0] + ax[1] * ax[1] + ax[2] * ax[2]) + 1e-9;
				double ang = uni(0, 3.14159);
				double sn = sin(ang * 0.5) / an;
				d1 = make_float4(float(ax[0] * sn), float(ax[1] * sn), float(ax[2] * sn), float(cos(ang * 0.5)));
				d0 = make_float4(pos[0], pos[1], pos[2], float(sscale));
			}
			CmdRecord rec;
			build_record(fc, cd.view, d0, d1, 0, 0, 0, 0, 0, rec);
			const bool exact_only = (__float_as_uint(rec.aux.w) & kRecExactOnly) != 0 || fc.enabled == 0 || fc.occ_ok == 0; // (the host launches the exact kernel then)

			for (uint32_t k = 0; k < per_draw && i < frame_items; ++k, ++i)
			{
				uint2 b0;
				uint32_t b1;
				if (sc.kind == 2)
				{
					b0.x = uint32_t(rng()), b0.y = uint32_t(rng()), b1 = uint32_t(rng());
					if (rng() & 1)
						b0.y = (b0.y & 0xffffu) | (uint32_t(to_half(float(uni(0, 2)))) << 16);
				}
				else
				{
					double ext = sc.kind == 1 ? 60.0 : 0.5;
					float c[3] = { float(uni(-ext, ext)), float(uni(-ext, ext)), float(uni(-ext, ext)) };
					double rr = sc.kind == 1 ? uni(0.05, 3.0) : 0.02 + 0.43 * pow(U(rng), 4.0);
					if ((rng() & 63) == 0)
						rr = 0.0;
					if (sc.kind == 5)
					{
						// local offsets of the order of rho (often 0); radius 0, an fp16 subnormal, a small normal or of the order of rho
						const double lr = rho / sscale;
						for (int j = 0; j < 3; ++j)
							c[j] = (rng() & 1) ? 0.f : float(uni(-2, 2) * lr);
						const uint32_t rk = uint32_t(rng() & 3);
						rr = rk == 0 ? 0.0 : rk == 1 ? pow(2.0, uni(-24.0, -14.0)) : rk == 2 ? pow(2.0, uni(-14.0, -6.0)) : lr * pow(2.0, uni(-8.0, 0.5));
					}
					b0.x = to_half(c[0]) | (uint32_t(to_half(c[1])) << 16);
					b0.y = to_half(c[2]) | (uint32_t(to_half(float(rr))) << 16);
					double a[3] = { uni(-1, 1), uni(-1, 1), uni(-1, 1) };
					double an = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]) + 1e-9;
					int cut = sc.kind == 5 ? int(int8_t(uint8_t(rng()))) : (rng() % 16 == 0) ? 127 : int(rng() % 112) + 16;
					b1 = uint32_t(uint8_t(int8_t(lrint(a[0] / an * 127)))) | (uint32_t(uint8_t(int8_t(lrint(a[1] / an * 127)))) << 8) | (uint32_t(uint8_t(int8_t(lrint(a[2] / an * 127)))) << 16) |
					     (uint32_t(uint8_t(int8_t(cut))) << 24);
				}

				float ce[3], ae[4] = { 0, 0, 0, 0 };
				bool ok_e;
				const bool late = true;
				const bool ve = exact_visible(cd, hiz, d0, d1, b0, b1, late, ce, ae, &ok_e);
				++st.items;
				st.visible += ve ? 1 : 0;
				if (exact_only)
				{
					++st.exact_only;
					++st.undecided;
					continue;
				}
				FilterResult fr = filter_meshlet<true, false>(fc, cd, hiz, rec.row0, rec.row1, rec.row2, rec.aux, b0, b1, cd.clusterBackfaceEnabled != 0, cd.clusterOcclusionEnabled == 1);
				{
					// the footprint-image variant must give the same answer
					FilterDebug keep = dbg;
					FilterResult fq = filter_meshlet<true, true>(fc, cd, hiz, rec.row0, rec.row1, rec.row2, rec.aux, b0, b1, cd.clusterBackfaceEnabled != 0, cd.clusterOcclusionEnabled == 1);
					if (fq.decided && fq.visible != ve) // (the jitter differs between the two calls, so `decided` may differ)
					{
						if (++st.wrong < 5)
							print_case("footprint", d0, d1, b0, b1, ve, fq.visible);
					}
					dbg = keep;
				}
				if (!fr.decided)
				{
					++st.undecided;
					for (int s = 0; s < 7; ++s)
						if (dbg.stage & (1 << s))
						{
							++st.stage[s]; // first failing stage only
							break;
						}
				}
				else if (fr.visible != ve)
				{
					++st.wrong;
					if (st.wrong < 5)
					{
						fprintf(stderr, "MISMATCH %s: exact %d filter %d  c=(%g %g %g) r=%g E=%g aabb_e=(%g %g %g %g) aabb_a=(%g %g %g %g) level %d stage %d\n", sc.name, int(ve), int(fr.visible), dbg.c[0], dbg.c[1],
						    dbg.c[2], dbg.r, dbg.E, ae[0], ae[1], ae[2], ae[3], dbg.aabb[0], dbg.aabb[1], dbg.aabb[2], dbg.aabb[3], dbg.level, dbg.stage);
						print_case("filter", d0, d1, b0, b1, ve, fr.visible);
					}
				}
				// ---- the drawcull use of the occlusion stage: exact centre, rounding-only error scale ----
				if (ce[0] == ce[0] && ce[1] == ce[1] && ce[2] == ce[2])
				{
					const float rr = __fmul_rn(half_bits_to_float(b0.y >> 16), d0.w);
					const float E2 = 12.f * 5.9604645e-8f * fmaxf(fmaxf(fabsf(ce[0]), fabsf(ce[1])), fabsf(ce[2])) + 42.f * 5.9604645e-8f * fabsf(rr) + 7.8886091e-31f;
					bool ov, oh;
					FilterDebug keep = dbg;
					filter_occlusion<false>(fc, cd, hiz, ce[0], ce[1], ce[2], rr, E2, fc.fr.x * E2, ov, oh, nullptr);
					dbg = keep;
					// the exact occlusion verdict for this sphere (independent of the frustum / cone outcome)
					f3 c3 = { ce[0], ce[1], ce[2] };
					float4 aabb;
					bool ok2 = project_sphere(c3, rr, cd.znear, cd.P00, cd.P11, aabb);
					int level = occlusion_mip(aabb, cd.pyramidWidth, cd.pyramidHeight, int(hiz.levels) - 1);
					uint32_t w = max(1u, hiz.width >> level), h = max(1u, hiz.height >> level);
					HiZLoadHost load = { hiz.texels, hiz.level_offset[level] };
					float depth = sample_min(load, w, h, __fmul_rn(__fadd_rn(aabb.x, aabb.z), 0.5f), __fmul_rn(__fadd_rn(aabb.y, aabb.w), 0.5f));
					bool occ_exact = !ok2 || __fdiv_rn(cd.znear, __fsub_rn(ce[2], rr)) > depth;
					++st.xc_items;
					if (!(ov || oh))
						++st.xc_undecided;
					else if (ov != occ_exact || (oh && occ_exact))
					{
						if (++st.xc_wrong < 5)
							print_case("exact_centre", d0, d1, b0, b1, occ_exact, ov);
					}
				}
				// margins vs what they bound (only where the filter's domain conditions hold)
				if (dbg.E == dbg.E && dbg.E < 1e30f && dbg.E > 0)
				{
					for (int j = 0; j < 3; ++j)
					{
						double ratio = fabs(double(ce[j]) - double(dbg.c[j])) / double(dbg.E);
						if (ratio > st.max_c_ratio)
							st.max_c_ratio = ratio;
					}
					if (ok_e && !(dbg.stage & 6) && dbg.gr > 0)
						for (int j = 0; j < 4; ++j)
						{
							double ratio = fabs(double(ae[j]) - double(dbg.aabb[j])) / (double(fc.Kuv) * double(dbg.gr));
							if (ratio > st.max_uv_ratio)
								st.max_uv_ratio = ratio;
						}
				}
			}
		}
		done += frame_items;
	}
	nvf_debug = nullptr;
}

int main(int argc, char** argv)
{
	const Scenario scenarios[] = { { "c4", 0 }, { "biglocal", 1 }, { "hostile", 2 }, { "near", 3 }, { "farworld", 4 }, { "subnormal", 5 } };
	if (argc < 4)
	{
		fprintf(stderr, "usage: %s <scenario|all> <items> <seed> [threads]\n", argv[0]);
		return 2;
	}
	const uint64_t items = strtoull(argv[2], nullptr, 10);
	const uint32_t seed = uint32_t(strtoul(argv[3], nullptr, 10));
	const int threads = argc > 4 ? atoi(argv[4]) : int(std::thread::hardware_concurrency());
	int rc = 0;
	for (const Scenario& sc : scenarios)
	{
		if (strcmp(argv[1], "all") != 0 && strcmp(argv[1], sc.name) != 0)
			continue;
		std::vector<Stats> stats(threads);
		std::vector<std::thread> pool;
		for (int t = 0; t < threads; ++t)
			pool.emplace_back([&, t]() { run(sc, items / threads, seed * 1000u + uint32_t(t), stats[t]); });
		for (auto& th : pool)
			th.join();
		Stats s;
		for (const Stats& t : stats)
		{
			s.items += t.items, s.undecided += t.undecided, s.wrong += t.wrong, s.visible += t.visible, s.exact_only += t.exact_only;
			s.xc_items += t.xc_items, s.xc_undecided += t.xc_undecided, s.xc_wrong += t.xc_wrong;
			for (int k = 0; k < 7; ++k)
				s.stage[k] += t.stage[k];
			s.max_c_ratio = std::max(s.max_c_ratio, t.max_c_ratio);
			s.max_uv_ratio = std::max(s.max_uv_ratio, t.max_uv_ratio);
		}
		printf("{\"scenario\": \"%s\", \"items\": %llu, \"wrong\": %llu, \"undecided\": %.6f, \"exact_only\": %.6f, \"visible\": %.4f, \"undecided_by_stage\": {\"frustum_cone\": %.6f, \"near_plane\": %.6f, \"domain\": %.6f, "
		       "\"level\": %.6f, \"fits\": %.6f, \"footprint\": %.6f, \"depth\": %.6f}, \"max_center_err_over_E\": %.4f, \"max_uv_err_over_margin\": %.4f, \"exact_centre_occlusion\": {\"items\": %llu, \"wrong\": %llu, \"undecided\": %.6f}}\n",
		    sc.name, (unsigned long long)s.items, (unsigned long long)s.wrong, double(s.undecided) / double(s.items), double(s.exact_only) / double(s.items), double(s.visible) / double(s.items),
		    double(s.stage[0]) / double(s.items), double(s.stage[1]) / double(s.items), double(s.stage[2]) / double(s.items), double(s.stage[3]) / double(s.items), double(s.stage[4]) / double(s.items),
		    double(s.stage[5]) / double(s.items), double(s.stage[6]) / double(s.items), s.max_c_ratio, s.max_uv_ratio, (unsigned long long)s.xc_items, (unsigned long long)s.xc_wrong,
		    s.xc_items ? double(s.xc_undecided) / double(s.xc_items) : 0.0);
		if (s.wrong || s.xc_wrong || s.max_c_ratio >= 1.0 || s.max_uv_ratio >= 1.0)
			rc = 1;
	}
	return rc;
}
