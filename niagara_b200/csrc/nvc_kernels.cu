// nvc_kernels.cu — sm_90a kernels of the visibility path.
//
//   drawcull_kernel<LATE,TASK>   drawcull.comp.glsl:54-156  (+ tasksubmit.comp.glsl:27-47 as last-block epilogue)
//   clustercull_kernel<LATE>     clustercull.comp.glsl:56-149 (+ clustersubmit.comp.glsl:25-45 as last-block epilogue)
//   taskcull_kernel<LATE>        meshlet.task.glsl:53-149
//   pyramid_kernel<EXACT>        depthreduce.comp.glsl:14-22 x all mips (niagara.cpp:1703-1733) in one launch
//
// Everything here is HBM/L2/ALU work on plain CUDA cores — there is no dense contraction, so no tensor cores.
// Compiled with -fmad=false; see nvc_math.cuh for the arithmetic contract.
#include "nvc_internal.h"
#include "nvc_math.cuh"
#include "nvc_cook.cuh"
#include "nvc_meshlets.cuh"
#include "nvc_lods.cuh"
#include "nvc_tma.cuh"
#include "nvc_filter.cuh"
#include "nvc_cache_decode.cuh"
#include "nvc_cache_encode.cuh"
#include "nvc_vertices.cuh"
#include "nvc_obj.cuh"
#include "nvc_scan.cuh"

#include <cuda_runtime.h>
#include <string.h>

#include <type_traits>

namespace nvc
{

// ------------------------------------------------------------------------------------------------------
// small helpers
// ------------------------------------------------------------------------------------------------------

__device__ __forceinline__ uint32_t lane_id()
{
	return threadIdx.x & 31u;
}

__device__ __forceinline__ uint32_t lanemask_lt()
{
	uint32_t m;
	asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
	return m;
}

__device__ __forceinline__ uint32_t lanemask_le()
{
	uint32_t m;
	asm("mov.u32 %0, %%lanemask_le;" : "=r"(m));
	return m;
}

// streaming 128-bit read-only load (each MeshDraw byte is touched once per pass)
__device__ __forceinline__ float4 ldg_f4(const void* p)
{
	return __ldg(reinterpret_cast<const float4*>(p));
}

__device__ __forceinline__ uint4 ldg_u4(const void* p)
{
	return __ldg(reinterpret_cast<const uint4*>(p));
}

// Read-once streams (meshlet bounds, task commands): read-only path with an L2 evict-first policy, so that the hundreds of MB a pass
// streams through do not push the depth pyramid / footprint image (read at random, many times) out of L2.
#if !defined(NVC_EMU)
__device__ __forceinline__ uint64_t stream_policy()
{
	uint64_t pol;
	asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
	return pol;
}
__device__ __forceinline__ uint2 ldg_stream_u2(const void* p, uint64_t pol)
{
	uint2 v;
	asm("ld.global.nc.L2::cache_hint.v2.u32 {%0,%1}, [%2], %3;" : "=r"(v.x), "=r"(v.y) : "l"(p), "l"(pol));
	return v;
}
__device__ __forceinline__ uint32_t ldg_stream_u32(const void* p, uint64_t pol)
{
	uint32_t v;
	asm("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
	return v;
}
__device__ __forceinline__ float4 ldg_stream_f4(const void* p, uint64_t pol)
{
	float4 v;
	asm("ld.global.nc.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
	return v;
}
#else
__device__ __forceinline__ uint64_t stream_policy() { return 0; }
__device__ __forceinline__ uint2 ldg_stream_u2(const void* p, uint64_t) { return __ldg(reinterpret_cast<const uint2*>(p)); }
__device__ __forceinline__ uint32_t ldg_stream_u32(const void* p, uint64_t) { return __ldg(reinterpret_cast<const uint32_t*>(p)); }
__device__ __forceinline__ float4 ldg_stream_f4(const void* p, uint64_t) { return __ldg(reinterpret_cast<const float4*>(p)); }
#endif

// The numeric per-pass constants the per-item math reads.  They stay in the kernel-parameter constant bank: ptxas
// re-materialises them as uniform loads (LDCU) inside the persistent loop; pinning them in registers was tried and is
// not expressible at the PTX level (ptxas sees through register copies), see DESIGN.md "things that did not help".
typedef NvcCullData ClusterConsts;


struct HiZLoad
{
	const float* texels; // uniform base; the level offset is folded into the 32-bit index
	uint32_t offset;
	__device__ __forceinline__ float operator()(uint32_t idx) const { return __ldg(texels + (offset + idx)); }
};

// Loads from the shared-memory copy of the coarse mips (staged by TMA at kernel start); offset is relative to it
struct HiZLoadShared
{
	const float* staged;
	uint32_t offset;
	__device__ __forceinline__ float operator()(uint32_t idx) const { return staged[offset + idx]; }
};

// drawcull.comp.glsl:88-103 == clustercull.comp.glsl:112-123.  Straight-line: every lane computes, the
// "sphere crosses the near plane -> stays visible" case is a select at the end.
// STAGED: when every live lane of the warp samples a mip that was staged into shared memory the four texel fetches
// are shared-memory loads; otherwise the warp takes the global (L1/L2) path.  The choice is warp-uniform, so the
// common fine-mip case pays one vote and no per-load select.
template <bool STAGED, typename CD>
__device__ __forceinline__ bool occlusion_visible(const CD& cd, const HiZDesc& hiz, const float* staged, bool alive, f3 center, float radius)
{
	float4 aabb;
	bool ok = project_sphere(center, radius, cd.znear, cd.P00, cd.P11, aabb);
	int level = occlusion_mip(aabb, cd.pyramidWidth, cd.pyramidHeight, int(hiz.levels) - 1);
	if (STAGED && !alive)
		level = int(hiz.levels) - 1; // dead lanes compute on garbage: keep their (ignored) fetch inside the staged range
	uint32_t w = max(1u, hiz.width >> level), h = max(1u, hiz.height >> level);
	float u = __fmul_rn(__fadd_rn(aabb.x, aabb.z), 0.5f);
	float v = __fmul_rn(__fadd_rn(aabb.y, aabb.w), 0.5f);
	float depth;
	if (STAGED && __all_sync(0xffffffffu, uint32_t(level) >= hiz.stage_level))
	{
		HiZLoadShared load = { staged, hiz.level_offset[level] - hiz.level_offset[hiz.stage_level] };
		depth = sample_min(load, w, h, u, v);
	}
	else
	{
		HiZLoad load = { hiz.texels, hiz.level_offset[level] };
		depth = sample_min(load, w, h, u, v);
	}
	float depthSphere = __fdiv_rn(cd.znear, __fsub_rn(center.z, radius));
	return !ok || depthSphere > depth;
}

// Stages the coarse tail of the pyramid (mips >= stage_level, contiguous in the packed layout) into shared memory:
// one elected thread arms an mbarrier and issues ONE cp.async.bulk (TMA, UBLKCP); the <= 3 texels that do not fill a
// 16-byte unit are copied by hand.  Every thread must call hiz_stage_wait() before reading `staged`.
__device__ __forceinline__ void hiz_stage_begin(const HiZDesc& hiz, float* staged, uint64_t* bar)
{
	const uint32_t bulk_texels = hiz.stage_texels & ~3u;
	if (threadIdx.x == 0)
		mbar_init(bar, 1);
	__syncthreads();
	const float* src = hiz.texels + hiz.level_offset[hiz.stage_level];
	if (threadIdx.x == 0)
	{
		mbar_arrive_expect_tx(bar, bulk_texels * 4u);
		bulk_copy_g2s(staged, src, bulk_texels * 4u, bar);
	}
	if (threadIdx.x < hiz.stage_texels - bulk_texels)
		staged[bulk_texels + threadIdx.x] = __ldg(src + bulk_texels + threadIdx.x);
	__syncthreads();
}

__device__ __forceinline__ void hiz_stage_wait(uint64_t* bar)
{
	mbar_wait(bar, 0);
}

// ------------------------------------------------------------------------------------------------------
// drawcull
// ------------------------------------------------------------------------------------------------------

constexpr int kDrawBlock = 256;
// Draws per thread.  The idea of DPT > 1: all DPT x 3 draw loads are in flight together and the fixed part of a CTA (dependent
// mesh-head load, the block's atomicAdd round trip, completion ticket, turnover) is paid once per DPT x 256 draws.  The registers
// and the longer tail of DPT > 1 cost more than the amortisation wins, so the kernel runs one draw per thread.  Its per-draw
// state stays in length-kDPT arrays walked by the phase loops: written as scalars, the compiler merges the branches of the
// mesh-head loads and of the sphere tests, which changes the generated code of every instantiation.
constexpr int kDPT = 1;
constexpr uint32_t kDrawQueue = 128; // undecided draws per block that go through the shared queue (more: evaluated in place)
constexpr uint32_t kDrawStage = 512; // commands staged per block before the coalesced write-out (static shared memory <= 48 KB)

template <bool LATE, bool TASK>
__global__ void __launch_bounds__(kDrawBlock) drawcull_kernel(const DrawCullParams p)
{
	__shared__ uint32_t s_warp_total[kDrawBlock / 32];
	__shared__ uint32_t s_block_base, s_block_total;
	__shared__ uint32_t s_is_last;
	__shared__ uint32_t s_stage[kDrawStage * (TASK ? 5 : 6)];
	// late pass, filtered occlusion: draws the filter could not decide, re-evaluated exactly by the first threads of the block
	__shared__ float4 s_qsphere[LATE ? kDrawQueue : 1];
	__shared__ uint8_t s_qresult[LATE ? kDrawQueue : 1];
	__shared__ uint32_t s_qcount;

	const NvcCullData& cd = p.cull;
	const uint32_t tid = threadIdx.x;
	const uint32_t lane = tid & 31u, warp = tid >> 5;
	const bool packed = p.mesh_heads != nullptr;
	if (LATE && tid == 0)
		s_qcount = 0;
	if (LATE)
		__syncthreads();

	// per-draw state of this thread's kDPT draws (draw k of the thread: block base + k * 256 + tid, so that every load
	// instruction of a warp still covers 32 consecutive MeshDraws)
	uint32_t di[kDPT];
	float4 d0[kDPT], d1[kDPT];
	uint4 d2[kDPT];
	bool reached[kDPT];
	uint32_t dv[kDPT];
	bool emit[kDPT];
	uint32_t units[kDPT]; // commands this draw appends: taskGroups (TASK) or 1
	uint32_t lodIndex[kDPT], meshletOffset[kDPT], meshletCount[kDPT];

	// ---- phase 1: all MeshDraw loads ----
#pragma unroll
	for (int k = 0; k < kDPT; ++k)
	{
		di[k] = (blockIdx.x * kDPT + k) * kDrawBlock + tid;
		d0[k] = make_float4(0.f, 0.f, 0.f, 0.f);
		d1[k] = make_float4(0.f, 0.f, 0.f, 1.f);
		d2[k] = make_uint4(0u, 0u, 0u, 0u);
		reached[k] = false;
		if (di[k] < cd.drawCount)
		{
			const char* dp = reinterpret_cast<const char*>(p.draws + di[k]);
			d0[k] = ldg_f4(dp);      // position.xyz, scale
			d1[k] = ldg_f4(dp + 16); // orientation
			d2[k] = ldg_u4(dp + 32); // meshIndex, meshletVisibilityOffset, postPass, materialIndex
			reached[k] = d2[k].z == cd.postPass; // :63
		}
	}
	// ---- phase 2: draw visibility ----
#pragma unroll
	for (int k = 0; k < kDPT; ++k)
	{
		dv[k] = 0;
		if (reached[k])
		{
			dv[k] = p.draw_visibility[di[k]];
			if (!LATE && dv[k] == 0) // :67
				reached[k] = false;
		}
	}
	// ---- phase 3: mesh heads (dependent on meshIndex) ----
	float4 m0[kDPT];
	uint4 h1[kDPT];
#pragma unroll
	for (int k = 0; k < kDPT; ++k)
	{
		m0[k] = make_float4(0.f, 0.f, 0.f, 0.f);
		h1[k] = make_uint4(0u, 0u, 0u, 0u);
		if (reached[k])
		{
			const char* mp = reinterpret_cast<const char*>(p.meshes + d2[k].x);
			// packed: one 32-byte sector holds center, radius, lodCount and the LOD-0 meshlet range
			const char* hp = packed ? reinterpret_cast<const char*>(p.mesh_heads + d2[k].x) : mp;
			m0[k] = ldg_f4(hp); // center.xyz, radius
			if (packed)
				h1[k] = ldg_u4(hp + 16); // lodCount, lod0.meshletOffset, lod0.meshletCount, vertexOffset
		}
	}
	// ---- phase 4a: view-space sphere, frustum, occlusion ----
	f3 centers[kDPT];
	float radii[kDPT];
	bool vis[kDPT];
	int qslot[kDPT];
	const bool filtered = LATE && p.use_filter != 0u && cd.occlusionEnabled == 1;
#pragma unroll
	for (int k = 0; k < kDPT; ++k)
	{
		vis[k] = false;
		qslot[k] = -1;
		centers[k] = { 0.f, 0.f, 0.f };
		radii[k] = 0.f;
		if (reached[k])
		{
			f3 mc = { m0[k].x, m0[k].y, m0[k].z };
			f3 rc = rotate_quat(mc, d1[k]);
			f3 center = { __fadd_rn(__fmul_rn(rc.x, d0[k].w), d0[k].x), __fadd_rn(__fmul_rn(rc.y, d0[k].w), d0[k].y), __fadd_rn(__fmul_rn(rc.z, d0[k].w), d0[k].z) };
			center = transform_point(cd.view, center);
			float radius = __fmul_rn(m0[k].w, d0[k].w);
			centers[k] = center;
			radii[k] = radius;

			bool visible = frustum_visible(cd, center, radius);
			visible = visible || cd.cullingEnabled == 0; // :85

			if (LATE && visible && cd.occlusionEnabled == 1) // :87
			{
				if (filtered)
				{
					// conservative filter on the EXACT centre (nvc_filter.cuh): E covers only rounding
					const float u = 5.9604645e-8f;
					const float E = nvf_fma(12.f * u, fmaxf(fmaxf(fabsf(center.x), fabsf(center.y)), fabsf(center.z)), nvf_fma(42.f * u, fabsf(radius), 7.8886091e-31f));
					bool occ_vis, occ_hid;
					if (p.hiz.fp)
						filter_occlusion<true>(p.filter, cd, p.hiz, center.x, center.y, center.z, radius, E, p.filter.fr.x * E, occ_vis, occ_hid);
					else
						filter_occlusion<false>(p.filter, cd, p.hiz, center.x, center.y, center.z, radius, E, p.filter.fr.x * E, occ_vis, occ_hid);
					if (occ_vis || occ_hid)
						visible = occ_vis;
					else
					{
						const uint32_t slot = atomicAdd(&s_qcount, 1u);
						if (slot < kDrawQueue)
						{
							s_qsphere[slot] = make_float4(center.x, center.y, center.z, radius);
							qslot[k] = int(slot);
						}
						else
							visible = occlusion_visible<false>(cd, p.hiz, nullptr, true, center, radius); // queue full: in place
					}
				}
				else
					visible = occlusion_visible<false>(cd, p.hiz, nullptr, true, center, radius);
			}
			vis[k] = visible;
		}
	}
	if (LATE && filtered)
	{
		// the undecided draws of the block, exactly, on its first threads (whole warps instead of scattered lanes)
		__syncthreads();
		const uint32_t nq = min(s_qcount, kDrawQueue);
		if (tid < nq)
		{
			const float4 sp = s_qsphere[tid];
			f3 c = { sp.x, sp.y, sp.z };
			s_qresult[tid] = occlusion_visible<false>(cd, p.hiz, nullptr, true, c, sp.w) ? 1 : 0;
		}
		__syncthreads();
#pragma unroll
		for (int k = 0; k < kDPT; ++k)
			if (qslot[k] >= 0)
				vis[k] = s_qresult[qslot[k]] != 0;
	}

	// ---- phase 4b: LOD selection and the command counts ----
	uint32_t thread_units = 0;
#pragma unroll
	for (int k = 0; k < kDPT; ++k)
	{
		emit[k] = false;
		units[k] = 0;
		lodIndex[k] = 0;
		meshletOffset[k] = 0;
		meshletCount[k] = 0;
		if (reached[k])
		{
			const uint32_t meshIndex = d2[k].x;
			const char* mp = reinterpret_cast<const char*>(p.meshes + meshIndex);
			const f3 center = centers[k];
			const float radius = radii[k];
			const bool visible = vis[k];

			// :108  (TASK_CULL == 1, config.h:8)
			if (visible && (!LATE || cd.clusterOcclusionEnabled == 1 || dv[k] == 0 || cd.postPass != 0))
			{
				uint32_t lodCount = 0;
				if (cd.lodEnabled == 1)
					lodCount = min(packed ? h1[k].x : __ldg(reinterpret_cast<const uint32_t*>(mp + 32)), NVC_MAX_LODS);
				if (lodCount > 1) // :112-120 (with a single LOD the loop below is empty and lodIndex stays 0: the distance is not needed)
				{
					float d = __fsub_rn(length3(center), radius);
					float distance = d > 0.f ? d : 0.f;
					float threshold = __fdiv_rn(__fmul_rn(distance, cd.lodTarget), d0[k].w);
					const float* errors = packed ? p.mesh_errors + size_t(meshIndex) * NVC_MAX_LODS : nullptr;
					for (uint32_t i = 1; i < lodCount; ++i)
					{
						float err = packed ? __ldg(errors + i) : __ldg(reinterpret_cast<const float*>(mp + 48 + i * 20 + 16));
						if (err < threshold)
							lodIndex[k] = i;
					}
				}
				emit[k] = true;
				if (TASK)
				{
					meshletCount[k] = (packed && lodIndex[k] == 0) ? h1[k].z : __ldg(reinterpret_cast<const uint32_t*>(mp + 48 + lodIndex[k] * 20 + 12));
					meshletOffset[k] = (packed && lodIndex[k] == 0) ? h1[k].y : __ldg(reinterpret_cast<const uint32_t*>(mp + 48 + lodIndex[k] * 20 + 8));
					units[k] = (meshletCount[k] + NVC_TASK_WGSIZE - 1) / NVC_TASK_WGSIZE; // :122
				}
				else
					units[k] = 1;
			}

			if (LATE)
				p.draw_visibility[di[k]] = visible ? 1u : 0u; // :154-155
		}
		thread_units += units[k];
	}

	// ---- block-wide exclusive scan of the threads' command counts, ONE global atomicAdd per block (the GLSL: one per thread) ----
	uint32_t incl = thread_units;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1)
	{
		uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
		if (lane >= uint32_t(o))
			incl += n;
	}
	if (lane == 31)
		s_warp_total[warp] = incl;
	__syncthreads();
	if (warp == 0)
	{
		uint32_t t = lane < kDrawBlock / 32 ? s_warp_total[lane] : 0;
		uint32_t ti = t;
#pragma unroll
		for (int o = 1; o < kDrawBlock / 32; o <<= 1)
		{
			uint32_t n = __shfl_up_sync(0xffffffffu, ti, o);
			if (lane >= uint32_t(o))
				ti += n;
		}
		if (lane < kDrawBlock / 32)
			s_warp_total[lane] = ti - t; // exclusive warp offsets
		uint32_t total = __shfl_sync(0xffffffffu, ti, kDrawBlock / 32 - 1);
		if (lane == 0)
		{
			s_block_total = total;
			s_block_base = total ? atomicAdd(&p.scratch->draw_counter, total) : 0u;
		}
	}
	__syncthreads();

	// ---- command write-out.  The block's commands are contiguous in dcb, so they are staged in shared memory and
	// copied out with fully coalesced 4-byte stores (the GLSL stores 5-6 scattered words per thread).  Blocks that
	// exceed the staging capacity or run into TASK_WGLIMIT take the direct per-thread path. ----
	constexpr uint32_t kWords = TASK ? 5u : 6u;
	const uint32_t block_total = s_block_total;
	uint32_t local = s_warp_total[warp] + (incl - thread_units);
	const bool staged = block_total <= kDrawStage && (!TASK || uint64_t(s_block_base) + block_total <= p.task_wglimit);
#pragma unroll
	for (int k = 0; k < kDPT; ++k)
	{
		if (emit[k])
		{
			const uint32_t dci = s_block_base + local;
			const char* mp = reinterpret_cast<const char*>(p.meshes + d2[k].x);
			const uint32_t* lp = reinterpret_cast<const uint32_t*>(mp + 48 + lodIndex[k] * 20);
			if (TASK)
			{
				// :129 drop on overflow; the counter has already advanced
				if (staged || uint64_t(dci) + units[k] <= p.task_wglimit)
				{
					uint32_t* out = staged ? s_stage + local * 5u : reinterpret_cast<uint32_t*>(static_cast<NvcMeshTaskCommand*>(p.commands) + dci);
					uint32_t* mc = (!staged && p.mc_commands) ? p.mc_commands + size_t(dci) * 5u : nullptr; // (staged blocks mirror in the copy-out loop)
					for (uint32_t i = 0; i < units[k]; ++i, out += 5)
					{
						out[0] = di[k];                                                             // drawId
						out[1] = meshletOffset[k] + i * NVC_TASK_WGSIZE;                            // taskOffset
						out[2] = min(NVC_TASK_WGSIZE, meshletCount[k] - i * NVC_TASK_WGSIZE);       // taskCount
						out[3] = dv[k];                                                             // lateDrawVisibility
						out[4] = d2[k].y + i * NVC_TASK_WGSIZE;                                     // meshletVisibilityOffset
						if (mc)
						{
							for (int wd = 0; wd < 5; ++wd)
								mc[wd] = out[wd];
							mc += 5;
						}
					}
				}
			}
			else
			{
				uint32_t* out = staged ? s_stage + local * 6u : reinterpret_cast<uint32_t*>(static_cast<NvcMeshDrawCommand*>(p.commands) + dci);
				out[0] = di[k];                                                    // drawId
				out[1] = __ldg(lp + 1);                                            // indexCount
				out[2] = 1;                                                        // instanceCount
				out[3] = __ldg(lp + 0);                                            // firstIndex
				out[4] = __ldg(reinterpret_cast<const uint32_t*>(mp + 16));        // vertexOffset
				out[5] = 0;                                                        // firstInstance
			}
		}
		local += units[k];
	}
	if (staged && block_total)
	{
		__syncthreads();
		uint32_t* out = reinterpret_cast<uint32_t*>(p.commands) + size_t(s_block_base) * kWords;
		for (uint32_t i = tid; i < block_total * kWords; i += kDrawBlock)
			out[i] = s_stage[i];
		if (TASK && p.mc_commands)
		{
			// fused all-gather: the same coalesced stream goes once more through the NVSwitch multicast mapping, which
			// replicates it into this rank's slot of EVERY rank's gathered buffer (one store per word instead of N unicast copies)
			uint32_t* mc = p.mc_commands + size_t(s_block_base) * kWords;
			for (uint32_t i = tid; i < block_total * kWords; i += kDrawBlock)
				mc[i] = s_stage[i];
		}
	}

	// ---- last-block epilogue: tasksubmit.comp.glsl:27-47 (TASK) / publish the count (draw path) ----
	__threadfence();
	__syncthreads();
	if (tid == 0)
		s_is_last = atomicAdd(&p.scratch->draw_done, 1u) == gridDim.x - 1;
	__syncthreads();
	if (!s_is_last)
		return;
	__threadfence();

	uint32_t commandCount = *reinterpret_cast<volatile uint32_t*>(&p.scratch->draw_counter);
	if (TASK)
	{
		uint32_t count = min(commandCount, p.task_wglimit);
		if (tid == 0)
		{
			p.command_count4[0] = commandCount;
			p.command_count4[1] = min((count + 63) / 64, NVC_MAX_DISPATCH_GROUPS);
			p.command_count4[2] = 64;
			p.command_count4[3] = 1;
		}
		uint32_t boundary = (count + 63) & ~63u;
		if (tid < 64 && count + tid < boundary)
		{
			NvcMeshTaskCommand* out = static_cast<NvcMeshTaskCommand*>(p.commands) + count + tid;
			out->drawId = 0;
			out->taskOffset = 0;
			out->taskCount = 0;
			out->lateDrawVisibility = 0;
			out->meshletVisibilityOffset = 0;
			if (p.mc_commands)
			{
				uint32_t* mc = p.mc_commands + size_t(count + tid) * 5u;
				for (int wd = 0; wd < 5; ++wd)
					mc[wd] = 0u;
			}
		}
	}
	else if (tid == 0)
	{
		p.command_count4[0] = commandCount;
		p.command_count4[1] = 0;
		p.command_count4[2] = 0;
		p.command_count4[3] = 0;
	}
	__syncthreads();
	if (tid == 0)
	{
		// leave the scratch counters zeroed for the next pass: replaces vkCmdFillBuffer(dccb, 0, 4, 0) niagara.cpp:1541
		p.scratch->draw_counter = 0;
		p.scratch->draw_done = 0;
	}
}

// ------------------------------------------------------------------------------------------------------
// per-meshlet test shared by clustercull / taskcull
// ------------------------------------------------------------------------------------------------------

// position of the r-th (0-based) set bit of the 64-bit mask {hi, lo}; r < popc(mask)
__device__ __forceinline__ uint32_t select_bit64(uint32_t lo, uint32_t hi, uint32_t r)
{
	uint32_t c = __popc(lo);
	bool upper = r >= c;
	uint32_t w = upper ? hi : lo;
	r = upper ? r - c : r;
	uint32_t pos = upper ? 32u : 0u;
	uint32_t t;
	t = __popc(w & 0xffffu);
	if (r >= t)
	{
		r -= t;
		pos += 16;
		w >>= 16;
	}
	t = __popc(w & 0xffu);
	if (r >= t)
	{
		r -= t;
		pos += 8;
		w >>= 8;
	}
	t = __popc(w & 0xfu);
	if (r >= t)
	{
		r -= t;
		pos += 4;
		w >>= 4;
	}
	t = __popc(w & 0x3u);
	if (r >= t)
	{
		r -= t;
		pos += 2;
		w >>= 2;
	}
	pos += (r >= (w & 1u)) ? 1u : 0u;
	return pos;
}

// One lane's work item inside a chunk and the raw data its test needs.
struct ItemRef
{
	uint32_t drawId, lateVis, mi, mvi, code; // code = commandId | (mgi << 24), the value appended on success
	bool active;
	bool alive_known; // early pass, item list built from the set visibility bits: the bit test is already decided
};

struct ItemData
{
	float4 d0, d1;  // MeshDraw: position.xyz + scale, orientation
	uint2 b0;       // Meshlet: center[3], radius (4 x binary16)
	uint32_t b1;    // Meshlet: cone_axis[3], cone_cutoff (4 x s8)
	uint32_t word;  // visibility word of this lane's bit (when the pass tracks bits)
	bool have_geom; // d0/d1/b0/b1 were loaded
};

// The 12 bytes of meshlet `mi` that every cluster test reads: b0 = center[3], radius (4 x binary16), b1 = cone_axis[3],
// cone_cutoff (4 x s8).  From the prepared view (nvc_prepare_meshlets: 8 + 4 bytes at dense strides, so a warp's loads are
// fully coalesced) when the pass reads the prepared Meshlet[], else from the first 12 bytes of the 24-byte record: the host
// sets the bases and strides (ClusterParams), the same two multiply-adds serve both.  STREAM: L2 evict-first loads (policy
// `pol`), else plain read-only loads.
template <bool STREAM>
__device__ __forceinline__ void load_meshlet_cull(const ClusterParams& p, uint32_t mi, uint64_t pol, uint2& b0, uint32_t& b1)
{
	const char* sp = p.ml_sphere + size_t(mi) * p.ml_sphere_stride;
	const char* cp = p.ml_cone + size_t(mi) * p.ml_cone_stride;
	if (STREAM)
	{
		b0 = ldg_stream_u2(sp, pol);
		b1 = ldg_stream_u32(cp, pol);
	}
	else
	{
		b0 = __ldg(reinterpret_cast<const uint2*>(sp));
		b1 = __ldg(reinterpret_cast<const uint32_t*>(cp));
	}
}

__device__ __forceinline__ void load_geometry(const ClusterParams& p, const ItemRef& r, ItemData& d)
{
	const char* dp = reinterpret_cast<const char*>(p.draws + r.drawId);
	d.d0 = ldg_f4(dp);
	d.d1 = ldg_f4(dp + 16);
	load_meshlet_cull<false>(p, r.mi, 0, d.b0, d.b1);
}

// Issues the loads of one chunk.  LATE: everything an active lane needs (bit word + geometry).  EARLY: only the bit
// word when the pass tracks bits (the geometry of meshlets that were invisible last frame is never touched), else
// the geometry.
template <bool LATE>
__device__ __forceinline__ void meshlet_fetch(const ClusterParams& p, const ItemRef& r, ItemData& d)
{
	const NvcCullData& cd = p.cull;
	const bool track = cd.clusterOcclusionEnabled == 1 && cd.postPass == 0; // :86
	d.d0 = make_float4(0.f, 0.f, 0.f, 1.f);
	d.d1 = make_float4(0.f, 0.f, 0.f, 1.f);
	d.b0 = make_uint2(0u, 0u);
	d.b1 = 0;
	d.word = 0;
	d.have_geom = false;
	if (r.active && !LATE && r.alive_known)
	{
		d.word = 0xffffffffu; // the item exists because its bit is set
		load_geometry(p, r, d);
		d.have_geom = true;
	}
	else if (r.active)
	{
		if (track) // early: read-only this pass.  late: only this lane's own bit matters and nobody else changes it.
			d.word = LATE ? __ldcg(p.meshlet_visibility + (r.mvi >> 5)) : __ldg(p.meshlet_visibility + (r.mvi >> 5));
		if (LATE || !track)
		{
			load_geometry(p, r, d);
			d.have_geom = true;
		}
	}
}

// clustercull.comp.glsl:72-124 for one 32-lane chunk.  Only warp-uniform branches: the GLSL's `visible && ...` chain
// (a pure conjunction, free of side effects) is evaluated straight through, and the expensive occlusion stage runs
// only when some lane is still alive.
//   visible  the GLSL's `visible` after all tests
//   skip     clustercull.comp.glsl:97-98
//   oldbit   the lane's previous visibility bit (meaningful when clusterOcclusionEnabled == 1 && postPass == 0)
template <bool LATE, bool STAGED>
__device__ __forceinline__ void meshlet_compute(const ClusterParams& p, const ClusterConsts& cc, const float* staged, const ItemRef& r, ItemData& d, bool& visible, bool& skip, bool& oldbit)
{
	const NvcCullData& cd = p.cull;
	bool alive = r.active;
	skip = false;
	oldbit = false;

	if (cd.clusterOcclusionEnabled == 1 && cd.postPass == 0) // :86
	{
		bool bit = (d.word >> (r.mvi & 31u)) & 1u;
		oldbit = bit;
		if (!LATE)
			alive = alive && bit; // :91-92
		else
			skip = r.lateVis == 1 && bit; // :97-98
	}
	visible = false;
	if (!LATE)
	{
		if (!__any_sync(0xffffffffu, alive))
			return; // nothing in this chunk was visible last frame
		if (alive && !d.have_geom)
			load_geometry(p, r, d);
	}

	f3 lc = { half_bits_to_float(d.b0.x & 0xffffu), half_bits_to_float(d.b0.x >> 16), half_bits_to_float(d.b0.y & 0xffffu) };
	f3 rc = rotate_quat(lc, d.d1);
	f3 center = { __fadd_rn(__fmul_rn(rc.x, d.d0.w), d.d0.x), __fadd_rn(__fmul_rn(rc.y, d.d0.w), d.d0.y), __fadd_rn(__fmul_rn(rc.z, d.d0.w), d.d0.z) };
	center = transform_point(cc.view, center);
	float radius = __fmul_rn(half_bits_to_float(d.b0.y >> 16), d.d0.w);

	alive = alive && frustum_visible(cc, center, radius); // :104-108

	if (cd.clusterBackfaceEnabled != 0) // :102
	{
		f3 la = { s8_div127(int(int8_t(d.b1 & 0xffu))), s8_div127(int(int8_t((d.b1 >> 8) & 0xffu))), s8_div127(int(int8_t((d.b1 >> 16) & 0xffu))) };
		f3 axis = transform_vector(cc.view, rotate_quat(la, d.d1));
		float cutoff = s8_div127(int(int8_t(d.b1 >> 24)));
		// math.h:41-44 with camera_position = 0
		bool backface = dot3(center, axis) >= __fadd_rn(__fmul_rn(cutoff, length3(center)), radius);
		alive = alive && !backface;
	}

	if (LATE && cd.clusterOcclusionEnabled == 1 && __any_sync(0xffffffffu, alive)) // :110
		alive = occlusion_visible<STAGED>(cc, p.hiz, staged, alive, center, radius) && alive;

	visible = alive;
}

// clustercull.comp.glsl:126-131 for one 32-item chunk: lanes with consecutive bit indices inside one word form a run;
// the run's head lane applies the whole run with at most two atomics (the GLSL issues one atomic per lane).
__device__ __forceinline__ void update_visibility_bits(uint32_t* mvb, bool active, bool visible, uint32_t mvi)
{
	const uint32_t lane = lane_id();
	uint32_t prev_mvi = __shfl_up_sync(0xffffffffu, mvi, 1);
	uint32_t act = __ballot_sync(0xffffffffu, active);
	bool prev_active = lane > 0 && ((act >> (lane - 1)) & 1u);
	bool head = active && (!prev_active || mvi != prev_mvi + 1 || (mvi & 31u) == 0);
	uint32_t heads = __ballot_sync(0xffffffffu, head);
	uint32_t vis = __ballot_sync(0xffffffffu, active && visible);
	if (!head)
		return;

	// run = [lane, next head or first inactive lane)
	uint32_t stop = (heads | ~act) & ~lanemask_le();
	uint32_t end = stop ? uint32_t(__ffs(int(stop)) - 1) : 32u;
	uint32_t len = end - lane; // 1..32
	uint32_t runmask = len >= 32 ? 0xffffffffu : ((1u << len) - 1u);
	uint32_t shift = mvi & 31u;
	uint32_t all = runmask << shift; // the run never crosses a word boundary ((mvi & 31) == 0 starts a new run)
	uint32_t set = ((vis >> lane) & runmask) << shift;
	uint32_t* word = mvb + (mvi >> 5);
	if (all == 0xffffffffu)
		*word = set; // all 32 bits of the word belong to this run: no other thread touches it this pass
	else
	{
		if (set)
			atomicOr(word, set);
		uint32_t clr = all & ~set;
		if (clr)
			atomicAnd(word, ~clr);
	}
}

// ------------------------------------------------------------------------------------------------------
// clustercull
// ------------------------------------------------------------------------------------------------------

constexpr int kClusterBlock = 256;
constexpr int kClusterWarps = kClusterBlock / 32;
constexpr int kStage = 256; // staged cluster indices per warp before one global atomicAdd + coalesced write-out
// Software prefetch of the next chunk's loads is not used (its extra registers cost occupancy); registers are capped at 40
// so that 6 CTAs (48 warps) are resident per SM.
constexpr int kClusterMinBlocks = 6;

__device__ __forceinline__ void flush_stage(const ClusterParams& p, uint32_t* stage, uint32_t& nst)
{
	const uint32_t lane = lane_id();
	__syncwarp();
	uint32_t base = 0;
	if (lane == 0)
		base = atomicAdd(&p.scratch->cluster_counter, nst); // :135, aggregated
	base = __shfl_sync(0xffffffffu, base, 0);
	for (uint32_t i = lane; i < nst; i += 32)
	{
		uint32_t index = base + i;
		if (index < p.cluster_limit) // :137
			p.cluster_indices[index] = stage[i];
	}
	__syncwarp();
	nst = 0;
}

// clustersubmit.comp.glsl:25-45 as the epilogue of a cluster pass; every thread of the 256-thread block calls it at the end.
// The CTA that takes the last ticket on cluster_done publishes the cluster count, pads cib with ~0u up to the next multiple
// of 256 (blockDim == 256 == clustersubmit's local_size_x), and zeroes the pass's scratch counters for the next pass.
// TASKOUT: the survivors went to the task payloads, so there is no cluster list to publish or pad.
template <bool TASKOUT>
__device__ __forceinline__ void clustersubmit_epilogue(const ClusterParams& p, uint32_t& s_is_last)
{
	const uint32_t tid = threadIdx.x;
	__threadfence();
	__syncthreads();
	if (tid == 0)
		s_is_last = atomicAdd(&p.scratch->cluster_done, 1u) == gridDim.x - 1;
	__syncthreads();
	if (!s_is_last)
		return;
	__threadfence();

	if (!TASKOUT)
	{
		const uint32_t clusterCount = *reinterpret_cast<volatile uint32_t*>(&p.scratch->cluster_counter);
		const uint32_t count = min(clusterCount, p.cluster_limit);
		if (tid == 0)
		{
			p.cluster_count4[0] = clusterCount;
			p.cluster_count4[1] = NVC_CLUSTER_TILE;
			p.cluster_count4[2] = min((count + 255) / 256, NVC_MAX_DISPATCH_GROUPS);
			p.cluster_count4[3] = 256 / NVC_CLUSTER_TILE;
		}
		const uint32_t boundary = (count + 255) & ~255u;
		if (count + tid < boundary)
			p.cluster_indices[count + tid] = ~0u;
	}
	__syncthreads();
	if (tid == 0)
	{
		p.scratch->cluster_counter = 0; // replaces vkCmdFillBuffer(ccb, 0, 4, 0) niagara.cpp:1586
		p.scratch->cluster_done = 0;
		p.scratch->cluster_batch = 0;
	}
}

template <bool LATE, bool STAGED>
__global__ void __launch_bounds__(kClusterBlock, kClusterMinBlocks) clustercull_kernel(const ClusterParams p)
{
	__shared__ uint32_t s_stage[kClusterWarps][kStage];
	__shared__ uint32_t s_is_last;
	__shared__ __align__(8) uint64_t s_hiz_bar;
	extern __shared__ __align__(16) float s_hiz[]; // coarse Hi-Z mips (STAGED only)

	if (STAGED)
		hiz_stage_begin(p.hiz, s_hiz, &s_hiz_bar); // the copy overlaps the first batch's command / geometry loads
	bool hiz_ready = !STAGED;

	const NvcCullData& cd = p.cull;
	const ClusterConsts& cc = cd;
	const uint32_t tid = threadIdx.x;
	const uint32_t lane = tid & 31u, warp = tid >> 5;
	uint32_t* stage = s_stage[warp];
	uint32_t nst = 0;

	// the reference dispatches (X,64,1) groups from dccb+4 (niagara.cpp:1599): commandId < X * 64
	const uint32_t ncmd = p.command_count4[1] * 64u;
	const uint32_t nbatch = (ncmd + 31u) / 32u;
	const bool track_late = LATE && cd.clusterOcclusionEnabled == 1;
	const bool bits_known = cd.postPass == 0; // meshlet_test read the previous bit (clustercull.comp.glsl:86)

	for (;;)
	{
		// dynamic batch of 32 consecutive task commands per warp
		uint32_t batch = 0;
		if (lane == 0)
			batch = atomicAdd(&p.scratch->cluster_batch, 1u);
		batch = __shfl_sync(0xffffffffu, batch, 0);
		if (batch >= nbatch)
			break;

		const uint32_t cid = batch * 32u + lane;
		uint32_t c_draw = 0, c_task = 0, c_count = 0, c_late = 0, c_mvo = 0;
		if (cid < ncmd)
		{
			const uint32_t* cp = reinterpret_cast<const uint32_t*>(p.task_commands + cid);
			c_draw = __ldg(cp + 0);
			c_task = __ldg(cp + 1);
			c_count = min(__ldg(cp + 2), NVC_TASK_WGSIZE); // valid = mgi < taskCount with mgi < 64
			c_late = __ldg(cp + 3);
			c_mvo = __ldg(cp + 4);
		}

		// Early pass with visibility tracking: only meshlets whose bit is set can survive (clustercull.comp.glsl:91-92), and
		// the bits are known up front — so flatten the SET BITS of every command's 64-bit visibility window instead of
		// all its lanes.  Meshlets that were invisible last frame then cost nothing (no geometry fetch, no arithmetic).
		const bool alive_flatten = !LATE && cd.clusterOcclusionEnabled == 1 && cd.postPass == 0;
		uint32_t amask_lo = 0, amask_hi = 0;
		uint32_t eff_count = c_count;
		if (alive_flatten)
		{
			if (c_count)
			{
				const uint32_t sh = c_mvo & 31u;
				const uint32_t nwords = (sh + c_count + 31u) >> 5; // 1..3 words hold the command's bits
				const uint32_t* wp = p.meshlet_visibility + (c_mvo >> 5);
				uint32_t w0 = __ldg(wp), w1 = nwords > 1 ? __ldg(wp + 1) : 0u, w2 = nwords > 2 ? __ldg(wp + 2) : 0u;
				amask_lo = __funnelshift_r(w0, w1, sh);
				amask_hi = __funnelshift_r(w1, w2, sh);
				// keep the command's own `count` bits
				amask_lo &= c_count >= 32 ? 0xffffffffu : ((1u << c_count) - 1u);
				amask_hi &= c_count >= 64 ? 0xffffffffu : (c_count > 32 ? ((1u << (c_count - 32)) - 1u) : 0u);
			}
			eff_count = __popc(amask_lo) + __popc(amask_hi);
		}

		// flatten (command, item) pairs: inclusive scan of the per-command item count over the batch
		uint32_t incl = eff_count;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1)
		{
			uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= uint32_t(o))
				incl += n;
		}
		const uint32_t excl = incl - eff_count;
		const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
		const uint32_t nz = __ballot_sync(0xffffffffu, eff_count != 0);
		const bool nz_prefix = (nz & (nz + 1u)) == 0; // non-empty commands form a prefix (always, except stale slots)
		// all 32 commands carry the same meshlet count (instanced meshes at one LOD, the synthetic scenes): then
		// command = item / count, one multiply-high with a per-batch reciprocal (exact: item < 2^11, count <= 64)
		const uint32_t count0 = __shfl_sync(0xffffffffu, eff_count, 0);
		const bool uniform = count0 >= 2 && __all_sync(0xffffffffu, eff_count == count0); // (count 1: the reciprocal would not fit)
		const uint32_t recip = uniform ? 0xffffffffu / count0 + 1u : 0u; // ceil(2^32 / count0)

		// item -> command mapping of the chunk starting at `base` (executed by all lanes)
		auto map_chunk = [&](uint32_t base) -> ItemRef {
			const uint32_t item = base + lane;
			uint32_t j;
			if (uniform)
				j = __umulhi(item, recip);
			else if (nz_prefix)
			{
				// head bits: commands that START inside this chunk (bit 0 excluded: that command is `first`)
				uint32_t rel = excl - base;
				uint32_t hbit = (eff_count != 0 && rel >= 1 && rel < 32) ? (1u << rel) : 0u;
				uint32_t heads = __reduce_or_sync(0xffffffffu, hbit);
				uint32_t first = __popc(__ballot_sync(0xffffffffu, eff_count != 0 && incl <= base));
				j = first + __popc(heads & lanemask_le());
			}
			else
			{
				// generic: binary search for the smallest j with incl[j] > item
				j = 0;
#pragma unroll
				for (int s = 16; s >= 1; s >>= 1)
				{
					uint32_t v = __shfl_sync(0xffffffffu, incl, (j + s - 1) & 31u);
					if (v <= item)
						j += s;
				}
			}
			j &= 31u;
			ItemRef r;
			r.active = item < total;
			r.drawId = __shfl_sync(0xffffffffu, c_draw, j);
			r.lateVis = __shfl_sync(0xffffffffu, c_late, j);
			uint32_t mgi = item - __shfl_sync(0xffffffffu, excl, j); // rank of the item inside its command
			if (alive_flatten)
			{
				// the rank-th SET bit of the command's visibility window is the meshlet's lane index
				const uint32_t mlo = __shfl_sync(0xffffffffu, amask_lo, j), mhi = __shfl_sync(0xffffffffu, amask_hi, j);
				mgi = r.active ? select_bit64(mlo, mhi, mgi) : 0u;
			}
			r.mi = __shfl_sync(0xffffffffu, c_task, j) + mgi;
			r.mvi = __shfl_sync(0xffffffffu, c_mvo, j) + mgi;
			r.alive_known = alive_flatten;
			r.code = (batch * 32u + j) | (mgi << 24); // :138
			return r;
		};

		// one chunk's bookkeeping after its verdicts are known: visibility bits (late) and compaction
		auto commit_chunk = [&](const ItemRef& r, bool visible, bool skip, bool oldbit) {
			// :126-131 — the GLSL rewrites every valid lane's bit; bits that already hold the new value need no
			// traffic, so the whole chunk skips the update when no lane changes state (the steady-state case)
			if (track_late && __any_sync(0xffffffffu, r.active && (!bits_known || oldbit != visible)))
				update_visibility_bits(p.meshlet_visibility, r.active, visible, r.mvi);

			const bool out = visible && !skip; // :133
			const uint32_t omask = __ballot_sync(0xffffffffu, out);
			const uint32_t n = __popc(omask);
			if (n)
			{
				if (nst + n > kStage)
					flush_stage(p, stage, nst);
				if (out)
					stage[nst + __popc(omask & lanemask_lt())] = r.code;
				nst += n;
			}
		};

		ItemRef cur = map_chunk(0);
		ItemData cur_data;
		if (total)
			meshlet_fetch<LATE>(p, cur, cur_data);

		for (uint32_t base = 0; base < total; base += 32)
		{
			if (!hiz_ready)
			{
				hiz_stage_wait(&s_hiz_bar);
				hiz_ready = true;
			}
			bool skip, oldbit, visible;
			meshlet_compute<LATE, STAGED>(p, cc, s_hiz, cur, cur_data, visible, skip, oldbit);
			commit_chunk(cur, visible, skip, oldbit);
			if (base + 32 < total)
			{
				cur = map_chunk(base + 32);
				meshlet_fetch<LATE>(p, cur, cur_data);
			}
		}
	}
	if (nst)
		flush_stage(p, stage, nst);
	if (!hiz_ready)
		hiz_stage_wait(&s_hiz_bar); // never leave the CTA while the bulk copy may still be writing its shared memory

	clustersubmit_epilogue<false>(p, s_is_last);
}

// ------------------------------------------------------------------------------------------------------
// clustercull, filtered: the default cluster pass.
//
// Same contract and the same outputs as clustercull_kernel, ~2x fewer instructions per meshlet:
//   * the lane that owns a task command builds, ONCE per command, the command's view-space transform
//     (M = scale * view3 * R(orientation), T = view * position) and the error scales of the filter into a shared-memory
//     record (CmdRecord, 80 bytes); every meshlet of the command then needs 9 fused multiply-adds for its centre
//     instead of the exact path's 54 unfused operations, and no shuffles / draw loads per item;
//   * each meshlet goes through filter_meshlet (nvc_filter.cuh): fused arithmetic, MUFU reciprocals / roots, and a
//     margin on every comparison.  Decided meshlets are committed at once;
//   * undecided meshlets (a few per cent: a screen-space coordinate within its error bound of a texel / mip boundary,
//     unusual transforms, non-finite data) are appended to a per-warp queue and re-evaluated by the EXACT
//     meshlet_compute on full warps, 32 at a time — so the result is bit-identical to the exact kernel's.
// ------------------------------------------------------------------------------------------------------

// resident CTAs per SM of the late and of the EARLY filtered kernel (no occlusion stage: fewer live registers; its shared-memory
// block is sized below)
constexpr int kFilterMinBlocks = 4;
constexpr int kFilterMinBlocksEarly = 4;
constexpr int kFFlush = 128;           // cluster indices written out per flush: ONE atomicAdd + four coalesced 128-byte stores per warp
constexpr int kFStage = kFFlush + 32;  // staged cluster indices per warp (a chunk appends <= 32 before the next flush)
constexpr int kFQueue = 64;            // undecided items per warp (drained 32 at a time)
// early pass: (command lane, meshlet lane) of every flattened item of one (sub-)batch; batches with more set bits are
// processed as four sub-batches of 8 commands (<= 512 items)
constexpr uint32_t kFItems = 896;
static_assert(kFItems >= 8u * 64u, "a sub-batch of 8 commands (<= 64 meshlets each) must fit the item table");

// One block of shared memory per warp: every field sits at a compile-time offset from the warp's base address.
template <bool LATE>
struct alignas(16) FilterWarpShared
{
	CmdRecord rec[32];
	uint4 queue[kFQueue];
	uint32_t stage[kFStage];
	uint16_t items[LATE ? 8 : kFItems];
};
static_assert(sizeof(FilterWarpShared<false>) * (256 / 32) + 16 <= 48 * 1024, "static shared memory");

// TRACK: clusterOcclusionEnabled == 1 && postPass == 0 (the main passes of a frame) as a compile-time fact; the generic
// instantiation reads the flags at run time.
// TASKOUT: meshlet.task.glsl's submission mode — survivors go to their command's payload (slot from an atomic counter per
// command, aggregated per warp; the reference's order inside a payload is unspecified too: atomicAdd(sharedCount), :137)
// and the count to emit_counts[command] instead of cib / ccb.
// BF: clusterBackfaceEnabled as a compile-time fact (0 / 1; -1 = read at run time).  With it the cone arithmetic is
// scheduled between the Hi-Z load and its use instead of behind a branch.
template <bool LATE, bool FP, bool TRACK, bool TASKOUT, int BF>
__global__ void __launch_bounds__(kClusterBlock, LATE ? kFilterMinBlocks : kFilterMinBlocksEarly) clustercull_filter_kernel(const ClusterParams p)
{
	__shared__ FilterWarpShared<LATE> sh_all[kClusterWarps];
	__shared__ uint32_t s_is_last;

	const NvcCullData& cd = p.cull;
	const ClusterConsts& cc = cd;
	const FilterConsts& fc = p.filter;
	const uint32_t tid = threadIdx.x;
	const uint32_t lane = tid & 31u, warp = tid >> 5;
	FilterWarpShared<LATE>& sh = sh_all[warp];
	uint32_t* const stage = sh.stage;
	uint4* const queue = sh.queue;
	CmdRecord* const recs = sh.rec;
	uint32_t nst = 0, nq = 0;
	uint32_t stat_items = 0, stat_undecided = 0; // per warp (uniform)
	const uint64_t spol = stream_policy();

	const uint32_t ncmd = p.command_count4[1] * 64u; // niagara.cpp:1599: commandId < X * 64
	const uint32_t nbatch = (ncmd + 31u) / 32u;
	const bool track = TRACK || (cd.clusterOcclusionEnabled == 1 && cd.postPass == 0); // clustercull.comp.glsl:86
	const bool track_late = LATE && (TRACK || cd.clusterOcclusionEnabled == 1);
	const bool bits_known = TRACK || cd.postPass == 0;
	const bool backface = BF >= 0 ? BF != 0 : cd.clusterBackfaceEnabled != 0;
	const bool occlusion = LATE && (TRACK || cd.clusterOcclusionEnabled == 1);

	// cluster indices (:133-139): staged per warp, written out 128 at a time
	auto flush_full = [&]() {
		__syncwarp();
		uint32_t base = 0;
		if (lane == 0)
			base = atomicAdd(&p.scratch->cluster_counter, uint32_t(kFFlush)); // :135, aggregated
		base = __shfl_sync(0xffffffffu, base, 0) + lane;
#pragma unroll
		for (int k = 0; k < kFFlush / 32; ++k)
		{
			const uint32_t v = stage[k * 32 + lane];
			if (base + k * 32 < p.cluster_limit) // :137
				p.cluster_indices[base + k * 32] = v;
		}
		const uint32_t rest = nst - uint32_t(kFFlush); // < 32
		const uint32_t t = stage[kFFlush + lane];
		__syncwarp();
		if (lane < rest)
			stage[lane] = t;
		nst = rest;
		__syncwarp();
	};

	// bookkeeping of one group of <= 32 verdicts: visibility bits (late, :126-131) and compaction (:133-139)
	auto commit = [&](bool active, bool visible, bool skip, bool oldbit, uint32_t mvi, uint32_t code) {
		if (track_late && __any_sync(0xffffffffu, active && (!bits_known || oldbit != visible)))
			update_visibility_bits(p.meshlet_visibility, active, visible, mvi);
		const bool out = active && visible && !skip;
		const uint32_t omask = __ballot_sync(0xffffffffu, out);
		const uint32_t n = __popc(omask);
		if (TASKOUT)
		{
			if (n) // warp-uniform: every lane takes part in the collectives, only emitting lanes touch memory
			{
				// lanes of one command share ONE atomic: leader = lowest emitting lane of the command's group
				const uint32_t cmd = code & 0xffffffu;
				const uint32_t group = __match_any_sync(0xffffffffu, out ? cmd : 0xffffffffu) & omask;
				const uint32_t leader = group ? uint32_t(__ffs(int(group)) - 1) : 0u;
				uint32_t base = 0;
				if (out && lane_id() == leader)
					base = atomicAdd(p.emit_counts + cmd, uint32_t(__popc(group)));
				base = __shfl_sync(0xffffffffu, base, int(leader));
				if (out)
					p.payloads[cmd].clusterIndices[base + __popc(group & lanemask_lt())] = code; // :137-139
			}
		}
		else if (n)
		{
			if (out)
				stage[nst + __popc(omask & lanemask_lt())] = code;
			nst += n;
			if (nst >= uint32_t(kFFlush))
				flush_full();
		}
	};

	// the exact path for up to 32 queued items (all lanes execute; lanes >= n are inactive)
	auto drain = [&](uint32_t n) {
		__syncwarp();
		const uint4 q = queue[lane < n ? lane : 0u];
		ItemRef r;
		r.active = lane < n;
		r.drawId = r.active ? __ldg(&p.task_commands[q.w & 0xffffffu].drawId) : 0u; // the exact path needs the draw: re-read the command (rare)
		r.mi = q.y;
		r.mvi = q.z;
		r.code = q.w & 0x7fffffffu;
		r.lateVis = q.w >> 31;
		r.alive_known = !LATE && track; // early + tracking: only meshlets whose bit is set are queued
		ItemData d;
		meshlet_fetch<LATE>(p, r, d);
		bool visible, skip, oldbit;
		meshlet_compute<LATE, false>(p, cc, nullptr, r, d, visible, skip, oldbit);
		commit(r.active, visible, skip, oldbit, r.mvi, r.code);
		// move the rest of the queue down
		__syncwarp();
		const uint32_t rest = nq - n;
		uint4 t0 = make_uint4(0u, 0u, 0u, 0u);
		if (lane < rest)
			t0 = queue[n + lane];
		__syncwarp();
		if (lane < rest)
			queue[lane] = t0;
		nq = rest;
		__syncwarp();
	};

	for (;;)
	{
		uint32_t batch = 0;
		if (lane == 0)
			batch = atomicAdd(&p.scratch->cluster_batch, 1u);
		batch = __shfl_sync(0xffffffffu, batch, 0);
		if (batch >= nbatch)
			break;

		// ---- per command: load, visibility window, transform record ----
		const uint32_t cid = batch * 32u + lane;
		uint32_t c_count = 0;
		// early pass with tracking: flatten only the SET visibility bits of every command (see clustercull_kernel)
		const bool alive_flatten = !LATE && track;
		uint32_t amask_lo = 0, amask_hi = 0;
		__syncwarp(); // the previous batch's readers of `recs` are done
		if (cid < ncmd)
		{
			const uint32_t* cp = reinterpret_cast<const uint32_t*>(p.task_commands + cid);
			const uint32_t c_draw = ldg_stream_u32(cp + 0, spol), c_task = ldg_stream_u32(cp + 1, spol);
			c_count = min(ldg_stream_u32(cp + 2, spol), NVC_TASK_WGSIZE); // valid = mgi < taskCount with mgi < 64
			const uint32_t c_late = ldg_stream_u32(cp + 3, spol), c_mvo = ldg_stream_u32(cp + 4, spol);
			if (TASKOUT)
				p.emit_counts[cid] = 0u; // sharedCount = 0 (:71); ordered before this warp's atomics by the __syncwarp below
			if (c_count)
			{
				if (track)
				{
					// the command's 64-bit window of visibility bits, read ONCE per command: bit mgi belongs to meshlet mgi.  Late
					// pass: other warps flip NEIGHBOUR bits of these words concurrently; a lane only ever looks at its own bit,
					// which nobody else touches during the pass (L2 load: lines of an earlier launch are never stale there).
					const uint32_t sft = c_mvo & 31u;
					const uint32_t nwords = (sft + c_count + 31u) >> 5; // 1..3 words hold the command's bits
					const uint32_t* wp = p.meshlet_visibility + (c_mvo >> 5);
					uint32_t w0 = __ldcg(wp), w1 = nwords > 1 ? __ldcg(wp + 1) : 0u, w2 = nwords > 2 ? __ldcg(wp + 2) : 0u;
					amask_lo = __funnelshift_r(w0, w1, sft);
					amask_hi = __funnelshift_r(w1, w2, sft);
					amask_lo &= c_count >= 32 ? 0xffffffffu : ((1u << c_count) - 1u);
					amask_hi &= c_count >= 64 ? 0xffffffffu : (c_count > 32 ? ((1u << (c_count - 32)) - 1u) : 0u);
				}
				const char* dp = reinterpret_cast<const char*>(p.draws + c_draw);
				const float4 d0 = ldg_f4(dp), d1 = ldg_f4(dp + 16);
				build_record(fc, cd.view, d0, d1, c_task, c_mvo, amask_lo, amask_hi, c_late, recs[lane]);
			}
		}
		const uint32_t eff_count = alive_flatten ? uint32_t(__popc(amask_lo) + __popc(amask_hi)) : c_count;

		uint32_t incl = eff_count;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1)
		{
			uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= uint32_t(o))
				incl += n;
		}
		const uint32_t excl = incl - eff_count;
		const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
		stat_items += total;

		// ---- one run of flattened items [0, run_total): chunks of 32, software pipelined ----
		// TABLE: item -> (command lane, meshlet lane) comes from sh.items (early pass, set bits only); otherwise it is derived
		// from the scan (`run_excl`: exclusive offsets of this run's commands): multiply-high for uniform batches, head-bit
		// popcount when the non-empty commands form a prefix, binary search over the scan else.
		auto run = [&](auto table_tag, uint32_t run_total, uint32_t run_excl, uint32_t run_incl) {
			constexpr bool TABLE = decltype(table_tag)::value;
			uint32_t count0 = 0, recip = 0;
			bool uniform = false, nz_prefix = false;
			if (!TABLE)
			{
				const uint32_t nz = __ballot_sync(0xffffffffu, eff_count != 0);
				nz_prefix = (nz & (nz + 1u)) == 0;
				count0 = __shfl_sync(0xffffffffu, eff_count, 0);
				uniform = count0 >= 2 && __all_sync(0xffffffffu, eff_count == count0);
				recip = uniform ? 0xffffffffu / count0 + 1u : 0u;
			}

			// item -> (j, mgi) and the meshlet's loads for the chunk starting at `b`.  Software pipeline: the loads of chunks k+1
			// and k+2 are issued before chunk k is evaluated, so their DRAM latency overlaps its arithmetic.
			// Carried state: one packed word (j | mgi << 8 | old visibility bit << 30 | active << 31) + the 12 loaded bytes.
			auto fetch = [&](uint32_t b, uint32_t& jm, uint2& b0, uint32_t& b1) {
				const uint32_t item = b + lane;
				const bool active = item < run_total;
				uint32_t j, mgi;
				if (TABLE)
				{
					const uint32_t e = active ? uint32_t(sh.items[item]) : 0u;
					j = e >> 6;
					mgi = e & 63u;
				}
				else
				{
					if (uniform)
						j = __umulhi(item, recip);
					else if (nz_prefix)
					{
						uint32_t rel = run_excl - b;
						uint32_t hbit = (eff_count != 0 && rel >= 1 && rel < 32) ? (1u << rel) : 0u;
						uint32_t heads = __reduce_or_sync(0xffffffffu, hbit);
						uint32_t first = __popc(__ballot_sync(0xffffffffu, eff_count != 0 && run_incl <= b));
						j = first + __popc(heads & lanemask_le());
					}
					else
					{
						j = 0;
#pragma unroll
						for (int s = 16; s >= 1; s >>= 1)
						{
							uint32_t v = __shfl_sync(0xffffffffu, run_incl, (j + s - 1) & 31u);
							if (v <= item)
								j += s;
						}
					}
					j &= 31u;
					mgi = uniform ? item - j * count0 : item - __shfl_sync(0xffffffffu, run_excl, j);
					if (!active)
						j = 0u, mgi = 0u;
					mgi &= 63u;
				}
				const uint4 ids = recs[j].ids;
				uint32_t bit = 0u;
				if (TABLE)
					bit = 1u; // only set bits are listed
				else if (track)
					bit = ((mgi & 32u ? ids.w : ids.z) >> (mgi & 31u)) & 1u;
				jm = j | (mgi << 8) | (bit << 30) | (active ? 0x80000000u : 0u);
				b0 = make_uint2(0u, 0u);
				b1 = 0u;
				if (active)
					load_meshlet_cull<true>(p, ids.x + mgi, spol, b0, b1);
			};

			// Prefetch distance 2 chunks: two chunks (2 x 384 bytes per warp from the meshlet cull view, 2 x 768 from the 24-byte
			// records) in flight.  With one, a chunk's arithmetic (~0.6 us at 8 warps per scheduler) is shorter than the DRAM
			// latency under load; with none, the whole latency is exposed.  n_*: chunk k+1, m_*: chunk k+2.
			uint32_t n_jm = 0, n_b1 = 0, m_jm = 0, m_b1 = 0;
			uint2 n_b0 = make_uint2(0u, 0u), m_b0 = make_uint2(0u, 0u);
			if (run_total)
				fetch(0u, n_jm, n_b0, n_b1);
			if (run_total > 32u)
				fetch(32u, m_jm, m_b0, m_b1);
			for (uint32_t base = 0; base < run_total; base += 32)
			{
				const uint32_t jm = n_jm, b1 = n_b1;
				const uint2 b0 = n_b0;
				n_jm = m_jm, n_b0 = m_b0, n_b1 = m_b1;
				if (base + 64u < run_total)
					fetch(base + 64u, m_jm, m_b0, m_b1);
				const bool active = (jm >> 31) != 0u;
				const uint32_t j = jm & 31u;

				// ---- the command's record, the meshlet's visibility bit ----
				const CmdRecord& rec = recs[j];
				const float4 row0 = rec.row0, row1 = rec.row1, row2 = rec.row2, aux = rec.aux;
				const uint32_t flags = __float_as_uint(aux.w);
				const bool bit = (jm & 0x40000000u) != 0u; // (false when the pass does not track bits)
				const bool oldbit = bit;
				const bool alive = (!LATE && track) ? (active && bit) : active; // :91-92
				const bool skip = LATE && track && (flags & kRecLate) != 0u && bit; // :97-98

				const FilterResult fr = filter_meshlet<LATE, FP>(fc, cd, p.hiz, row0, row1, row2, aux, b0, b1, backface, occlusion);
				const bool undecided = alive && (!fr.decided || (flags & kRecExactOnly) != 0u);
				const bool visible = alive && fr.visible;

				// ---- nothing undecided, no visibility bit changes, nothing to append (the steady-state chunk of the late pass) ----
				const bool work = active && !undecided && ((visible && !skip) || (track_late && (!bits_known || oldbit != visible)));
				const uint32_t umask = __ballot_sync(0xffffffffu, undecided);
				const bool any_work = __any_sync(0xffffffffu, work);
				if (!(umask | uint32_t(any_work)))
					continue;

				const uint32_t mgi = (jm >> 8) & 63u;
				const uint32_t code = (batch * 32u + j) | (mgi << 24); // :138
				const uint32_t mvi = rec.ids.y + mgi;
				// ---- undecided lanes -> queue (exact path on full warps) ----
				if (umask)
				{
					if (undecided)
						queue[nq + __popc(umask & lanemask_lt())] = make_uint4(0u, rec.ids.x + mgi, mvi, code | ((flags & kRecLate) << 31));
					nq += __popc(umask);
					stat_undecided += __popc(umask);
				}
				if (any_work)
					commit(active && !undecided, visible, skip, oldbit, mvi, code);
				if (nq >= 32u)
					drain(32u);
			}
		};

		if (alive_flatten)
		{
			// every command lane lists the positions of its set bits ONCE per (sub-)batch; items then read one 16-bit entry
			// (command lane << 6 | meshlet lane) instead of searching the scan and selecting the rank-th set bit of the window
			const uint32_t span = total <= kFItems ? 32u : 8u;
			for (uint32_t lo = 0; lo < 32u; lo += span)
			{
				const uint32_t sub_base = __shfl_sync(0xffffffffu, excl, int(lo));
				const uint32_t sub_end = lo + span < 32u ? __shfl_sync(0xffffffffu, excl, int((lo + span) & 31u)) : total;
				if (sub_end == sub_base)
					continue;
				if (lane >= lo && lane < lo + span)
				{
					uint16_t* tbl = sh.items + (excl - sub_base);
					const uint32_t tag = lane << 6;
					for (uint32_t m = amask_lo; m; m &= m - 1u)
						*tbl++ = uint16_t(tag | uint32_t(__ffs(int(m)) - 1));
					for (uint32_t m = amask_hi; m; m &= m - 1u)
						*tbl++ = uint16_t(tag | uint32_t(32 + __ffs(int(m)) - 1));
				}
				__syncwarp(); // records and the item table visible to the whole warp
				run(std::true_type(), sub_end - sub_base, 0u, 0u);
				__syncwarp(); // the table's readers are done
			}
		}
		else
		{
			__syncwarp(); // records visible to the whole warp
			run(std::false_type(), total, excl, incl);
		}
	}
	while (nq)
		drain(min(nq, 32u));
	if (nst)
		flush_stage(p, stage, nst);
	if (lane == 0 && stat_items)
	{
		atomicAdd(&p.scratch->filter_items, (unsigned long long)stat_items);
		if (stat_undecided)
			atomicAdd(&p.scratch->filter_undecided, (unsigned long long)stat_undecided);
	}

	clustersubmit_epilogue<TASKOUT>(p, s_is_last);
}

// ------------------------------------------------------------------------------------------------------
// taskcull: meshlet.task.glsl:53-149 — one warp per command (two 32-lane halves), payload compaction per command
// ------------------------------------------------------------------------------------------------------

template <bool LATE>
__global__ void __launch_bounds__(kClusterBlock) taskcull_kernel(const ClusterParams p, NvcMeshTaskPayload* payloads, uint32_t* emit_counts)
{
	const NvcCullData& cd = p.cull;
	const ClusterConsts& cc = cd;
	const uint32_t lane = lane_id();
	const uint32_t ncmd = p.command_count4[1] * 64u;
	const uint32_t warps_total = gridDim.x * kClusterWarps;
	const bool track_late = LATE && cd.clusterOcclusionEnabled == 1;

	for (uint32_t cid = blockIdx.x * kClusterWarps + (threadIdx.x >> 5); cid < ncmd; cid += warps_total)
	{
		const uint32_t* cp = reinterpret_cast<const uint32_t*>(p.task_commands + cid);
		const uint32_t c_draw = __ldg(cp + 0), c_task = __ldg(cp + 1), c_count = min(__ldg(cp + 2), NVC_TASK_WGSIZE);
		const uint32_t c_late = __ldg(cp + 3), c_mvo = __ldg(cp + 4);

		uint32_t sharedCount = 0; // :71
#pragma unroll 1
		for (uint32_t half = 0; half < 2; ++half)
		{
			const uint32_t mgi = half * 32 + lane;
			const bool active = mgi < c_count;
			if (!__any_sync(0xffffffffu, active))
				break;
			bool skip, visible, oldbit;
			ItemRef r;
			r.active = active;
			r.drawId = c_draw;
			r.lateVis = c_late;
			r.mi = c_task + mgi;
			r.mvi = c_mvo + mgi;
			r.code = cid | (mgi << 24);
			r.alive_known = false;
			ItemData d;
			meshlet_fetch<LATE>(p, r, d);
			meshlet_compute<LATE, false>(p, cc, nullptr, r, d, visible, skip, oldbit);
			if (track_late && __any_sync(0xffffffffu, active && (cd.postPass != 0 || oldbit != visible)))
				update_visibility_bits(p.meshlet_visibility, active, visible, c_mvo + mgi);
			const bool out = visible && !skip;
			const uint32_t omask = __ballot_sync(0xffffffffu, out);
			if (out)
				payloads[cid].clusterIndices[sharedCount + __popc(omask & lanemask_lt())] = cid | (mgi << 24); // :137-139
			sharedCount += __popc(omask);
		}
		if (lane == 0)
			emit_counts[cid] = sharedCount; // EmitMeshTasksEXT(sharedCount, 1, 1)  :143
	}
}

// ------------------------------------------------------------------------------------------------------
// TASK_CULL = 0 (nvc_set_task_cull(ctx, 0)): the cluster and task passes without meshlet tests.  Only the task commands are
// read; draws, meshlets, meshlet visibility and the Hi-Z are not touched.
// ------------------------------------------------------------------------------------------------------

constexpr uint32_t kPassBlock = 256; // task commands per tile (one thread each)

// clustercull.comp.glsl:140-147 + clustersubmit.comp.glsl:25-45: every lane mgi < taskCount of command c < command_count4[1] * 64
// appends c | (mgi << 24) (mgi < 64: the workgroup has 64 lanes).  Per tile of 256 commands: one thread loads a command's
// taskCount, a block-wide scan gives each command its offset, ONE atomicAdd on the cluster counter reserves the tile's contiguous
// range, and each warp writes whole commands with consecutive stores.  The counter counts past cluster_limit; stores at or above
// it are dropped.  The last CTA runs the clustersubmit epilogue and leaves the scratch counters zeroed.
__global__ void __launch_bounds__(kPassBlock) clustercull_passthrough_kernel(const ClusterParams p)
{
	__shared__ uint32_t s_count[kPassBlock], s_offset[kPassBlock];
	__shared__ uint32_t s_warp_total[kPassBlock / 32];
	__shared__ uint32_t s_base, s_is_last;

	const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
	const uint32_t ncmd = p.command_count4[1] * 64u;
	for (uint32_t tile = blockIdx.x * kPassBlock; tile < ncmd; tile += gridDim.x * kPassBlock)
	{
		const uint32_t cid = tile + tid;
		const uint32_t count = cid < ncmd ? min(__ldg(reinterpret_cast<const uint32_t*>(p.task_commands + cid) + 2), NVC_TASK_WGSIZE) : 0u;
		uint32_t incl = count;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1)
		{
			const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= uint32_t(o))
				incl += n;
		}
		if (lane == 31)
			s_warp_total[warp] = incl;
		__syncthreads();
		if (warp == 0)
		{
			const uint32_t t = lane < kPassBlock / 32 ? s_warp_total[lane] : 0u;
			uint32_t ti = t;
#pragma unroll
			for (int o = 1; o < int(kPassBlock / 32); o <<= 1)
			{
				const uint32_t n = __shfl_up_sync(0xffffffffu, ti, o);
				if (lane >= uint32_t(o))
					ti += n;
			}
			if (lane < kPassBlock / 32)
				s_warp_total[lane] = ti - t; // exclusive warp offsets
			const uint32_t total = __shfl_sync(0xffffffffu, ti, kPassBlock / 32 - 1);
			if (lane == 0)
				s_base = total ? atomicAdd(&p.scratch->cluster_counter, total) : 0u; // :143, aggregated
		}
		__syncthreads();
		s_count[tid] = count;
		s_offset[tid] = s_warp_total[warp] + incl - count;
		__syncthreads();
		const uint32_t base = s_base;
		for (uint32_t c = warp; c < kPassBlock; c += kPassBlock / 32)
		{
			const uint32_t n = s_count[c], first = base + s_offset[c];
			for (uint32_t mgi = lane; mgi < n; mgi += 32)
				if (first + mgi < p.cluster_limit) // :145
					p.cluster_indices[first + mgi] = (tile + c) | (mgi << 24);
		}
		__syncthreads(); // s_count / s_offset / s_warp_total are reused by the next tile
	}

	clustersubmit_epilogue<false>(p, s_is_last);
}

// meshlet.task.glsl:144-148: for every command c < command_count4[1] * 64, all 64 lanes write payload.clusterIndices[lane] =
// c | (lane << 24), taskCount or not, and the shader emits taskCount mesh workgroups, as read (not clamped to 64).  A pure
// streaming write: 16 bytes of payload per thread step (4 bytes when payloads is not 16-byte aligned), emit_counts[c] from the
// command's taskCount.
__global__ void __launch_bounds__(kPassBlock) taskcull_passthrough_kernel(const NvcMeshTaskCommand* __restrict__ task_commands, const uint32_t* __restrict__ command_count4,
    NvcMeshTaskPayload* __restrict__ payloads, uint32_t* __restrict__ emit_counts)
{
	const uint32_t ncmd = __ldg(command_count4 + 1) * 64u;
	const uint32_t stride = gridDim.x * kPassBlock;
	const uint32_t first = blockIdx.x * kPassBlock + threadIdx.x;
	for (uint32_t c = first; c < ncmd; c += stride)
		emit_counts[c] = __ldg(reinterpret_cast<const uint32_t*>(task_commands + c) + 2);
	uint32_t* const words = reinterpret_cast<uint32_t*>(payloads);
	if ((reinterpret_cast<uintptr_t>(payloads) & 15u) == 0)
	{
		const uint32_t nvec = ncmd * (NVC_TASK_WGSIZE / 4);
		for (uint32_t v = first; v < nvec; v += stride)
		{
			const uint32_t c = v / (NVC_TASK_WGSIZE / 4), lane = (v % (NVC_TASK_WGSIZE / 4)) * 4u;
			reinterpret_cast<uint4*>(words)[v] = make_uint4(c | (lane << 24), c | ((lane + 1u) << 24), c | ((lane + 2u) << 24), c | ((lane + 3u) << 24));
		}
	}
	else
	{
		const uint32_t nword = ncmd * NVC_TASK_WGSIZE;
		for (uint32_t w = first; w < nword; w += stride)
			words[w] = (w / NVC_TASK_WGSIZE) | ((w % NVC_TASK_WGSIZE) << 24);
	}
}

// ------------------------------------------------------------------------------------------------------
// depth pyramid: all mips in ONE launch.
// Each CTA owns a 64x64 tile of mip 0 (128x128 depth texels when the ratio is exactly 2:1), reduces it through
// mips 0..6 in shared memory, writing every level; the last CTA to finish (global ticket) reduces the remaining
// small mips.  min() is exact and order independent, so the result is bit-identical to the reference's
// level-by-level dispatch chain (niagara.cpp:1713-1728).
// ------------------------------------------------------------------------------------------------------

constexpr int kPyrBlock = 256;
constexpr int kPyrTile = 64; // mip-0 texels per CTA edge
constexpr int kPyrTileLevels = 7; // 64 -> 1

struct DepthLoad
{
	const float* base;
	__device__ __forceinline__ float operator()(uint32_t idx) const { return __ldg(base + idx); }
};

// dst(x, y) = min of src[2x..2x+1][2y..2y+1] clamped to the source extent (exact 2:1 MIN-sampler footprint)
__device__ __forceinline__ float reduce2x2(const float* src, uint32_t sw, uint32_t sh, uint32_t spitch, uint32_t x, uint32_t y)
{
	uint32_t x0 = min(2 * x, sw - 1), x1 = min(2 * x + 1, sw - 1);
	uint32_t y0 = min(2 * y, sh - 1), y1 = min(2 * y + 1, sh - 1);
	return fminf(fminf(src[y0 * spitch + x0], src[y0 * spitch + x1]), fminf(src[y1 * spitch + x0], src[y1 * spitch + x1]));
}

// 7 resident CTAs per SM = 1036 slots: the 1024 tiles of a 2048^2 pyramid (4096^2 depth target) run as ONE wave
constexpr int kPyrMinBlocks = 7;

template <bool EXACT>
__global__ void __launch_bounds__(kPyrBlock, kPyrMinBlocks) pyramid_kernel(const PyramidParams p)
{
	__shared__ float s_a[kPyrTile * kPyrTile];             // level 0 tile, later levels 2, 4, 6
	__shared__ float s_b[(kPyrTile / 2) * (kPyrTile / 2)]; // levels 1, 3, 5
	__shared__ uint32_t s_is_last;

	const HiZDesc& hz = p.hiz;
	const uint32_t tid = threadIdx.x;
	const uint32_t tile_x = blockIdx.x * kPyrTile, tile_y = blockIdx.y * kPyrTile;

	// ---- mip 0 from the depth target: depthreduce.comp.glsl:19 with imageSize = (hz.width, hz.height) ----
	const bool full_tile = tile_x + kPyrTile <= hz.width && tile_y + kPyrTile <= hz.height;
	uint32_t first_smem_level = 1; // first mip still to be produced from the shared-memory tile
	if (EXACT && full_tile && p.vector_ok && hz.levels > 3)
	{
		// Streaming fast path.  Warp w owns mip-0 rows 8w..8w+7 of the tile, lane l owns mip-0 columns 2l, 2l+1: the
		// 128 x 128 depth texels of the tile arrive as 16 independent 16-byte loads per thread (all issued before the
		// first use, 64 KB in flight per CTA).  Mips 0-3 are then reduced in registers: vertically inside the thread,
		// horizontally with xor-shuffles ("wave recursion"), no shared memory and no barrier until mip 4.
		const uint32_t warp = tid >> 5, lane = tid & 31u;
		const uint32_t row0 = tile_y + 8 * warp;
		const float* src_row = p.depth + size_t(2 * row0) * p.depth_width + 2 * tile_x + 4 * lane;
		float4 a[8], b[8];
#pragma unroll
		for (int j = 0; j < 8; ++j)
		{
			a[j] = __ldcs(reinterpret_cast<const float4*>(src_row + size_t(2 * j) * p.depth_width));
			b[j] = __ldcs(reinterpret_cast<const float4*>(src_row + size_t(2 * j + 1) * p.depth_width));
		}
		float2 v0[8];
		{
			float* dst = hz.texels + hz.level_offset[0] + size_t(row0) * hz.width + tile_x + 2 * lane;
#pragma unroll
			for (int j = 0; j < 8; ++j)
			{
				v0[j].x = fminf(fminf(a[j].x, a[j].y), fminf(b[j].x, b[j].y));
				v0[j].y = fminf(fminf(a[j].z, a[j].w), fminf(b[j].z, b[j].w));
				*reinterpret_cast<float2*>(dst + size_t(j) * hz.width) = v0[j];
			}
		}
		float v1[4]; // mip 1: rows 4w..4w+3 of the tile, column l
		{
			const uint32_t w1 = hz.width >> 1;
			float* dst = hz.texels + hz.level_offset[1] + size_t((tile_y >> 1) + 4 * warp) * w1 + (tile_x >> 1) + lane;
#pragma unroll
			for (int j = 0; j < 4; ++j)
			{
				v1[j] = fminf(fminf(v0[2 * j].x, v0[2 * j].y), fminf(v0[2 * j + 1].x, v0[2 * j + 1].y));
				dst[size_t(j) * w1] = v1[j];
			}
		}
		float v2[2]; // mip 2: rows 2w..2w+1, column l/2 (valid in even lanes)
		{
			const uint32_t w2 = hz.width >> 2;
			float* dst = hz.texels + hz.level_offset[2] + size_t((tile_y >> 2) + 2 * warp) * w2 + (tile_x >> 2) + (lane >> 1);
#pragma unroll
			for (int j = 0; j < 2; ++j)
			{
				float m = fminf(v1[2 * j], v1[2 * j + 1]);
				v2[j] = fminf(m, __shfl_xor_sync(0xffffffffu, m, 1));
				if ((lane & 1u) == 0)
					dst[size_t(j) * w2] = v2[j];
			}
		}
		{
			// mip 3: row w, column l/4 (valid in lanes that are multiples of 4)
			const uint32_t w3 = hz.width >> 3;
			float m = fminf(v2[0], v2[1]);
			m = fminf(m, __shfl_xor_sync(0xffffffffu, m, 2));
			if ((lane & 3u) == 0)
			{
				hz.texels[hz.level_offset[3] + size_t((tile_y >> 3) + warp) * w3 + (tile_x >> 3) + (lane >> 2)] = m;
				s_b[warp * 8 + (lane >> 2)] = m; // 8 x 8 tile of mip 3 for the remaining levels
			}
		}
		first_smem_level = 4;
	}
	else
	{
		const uint32_t lw = hz.width, lh = hz.height;
		float* dst = hz.texels + hz.level_offset[0];
		for (uint32_t i = tid; i < kPyrTile * kPyrTile; i += kPyrBlock)
		{
			uint32_t lx = i % kPyrTile, ly = i / kPyrTile;
			uint32_t x = tile_x + lx, y = tile_y + ly;
			float v = 0.f;
			if (x < lw && y < lh)
			{
				if (EXACT)
				{
					// depth is exactly (2*lw) x (2*lh): footprint is the 2x2 block
					const float* r0 = p.depth + size_t(2 * y) * p.depth_width + 2 * x;
					const float* r1 = r0 + p.depth_width;
					v = fminf(fminf(__ldg(r0), __ldg(r0 + 1)), fminf(__ldg(r1), __ldg(r1 + 1)));
				}
				else
				{
					float u = __fdiv_rn(__fadd_rn(float(x), 0.5f), float(lw));
					float w = __fdiv_rn(__fadd_rn(float(y), 0.5f), float(lh));
					DepthLoad load = { p.depth };
					v = sample_min(load, p.depth_width, p.depth_height, u, w);
				}
				dst[size_t(y) * lw + x] = v;
			}
			s_a[i] = v;
		}
	}
	__syncthreads();

	// ---- remaining mips (up to 6) of this tile in shared memory ----
	float* src = first_smem_level == 4 ? s_b : s_a;
	float* out = first_smem_level == 4 ? s_a : s_b;
	uint32_t src_pitch = kPyrTile >> (first_smem_level - 1);
	for (uint32_t l = first_smem_level; l < kPyrTileLevels && l < hz.levels; ++l)
	{
		const uint32_t lw = max(1u, hz.width >> l), lh = max(1u, hz.height >> l);
		const uint32_t pw = max(1u, hz.width >> (l - 1)), ph = max(1u, hz.height >> (l - 1)); // previous level size
		const uint32_t edge = kPyrTile >> l;                                                       // tile edge at this level
		const uint32_t ox = tile_x >> l, oy = tile_y >> l;                                         // tile origin at this level
		const uint32_t pox = tile_x >> (l - 1), poy = tile_y >> (l - 1);
		// valid extent of the previous level inside this tile
		const uint32_t sw = min(kPyrTile >> (l - 1), pw > pox ? pw - pox : 0u), sh = min(kPyrTile >> (l - 1), ph > poy ? ph - poy : 0u);
		float* dst = hz.texels + hz.level_offset[l];
		for (uint32_t i = tid; i < edge * edge; i += kPyrBlock)
		{
			uint32_t lx = i % edge, ly = i / edge;
			uint32_t x = ox + lx, y = oy + ly;
			float v = 0.f;
			if (x < lw && y < lh && sw && sh)
			{
				v = reduce2x2(src, sw, sh, src_pitch, lx, ly);
				dst[size_t(y) * lw + x] = v;
			}
			out[ly * edge + lx] = v;
		}
		__syncthreads();
		float* t = src;
		src = out;
		out = t;
		src_pitch = edge;
	}

	if (hz.levels <= kPyrTileLevels && gridDim.x * gridDim.y == 1)
		return; // single tile covered every level

	// ---- remaining mips by the last CTA to finish ----
	__threadfence();
	__syncthreads();
	if (tid == 0)
		s_is_last = atomicAdd(&p.scratch->pyramid_done, 1u) == gridDim.x * gridDim.y - 1;
	__syncthreads();
	if (!s_is_last)
		return;
	__threadfence();

	// The tiles completed mips 0 .. kPyrTileLevels-1 (tiles whose extent degenerates on non-square pyramids still wrote
	// every texel of those levels).  Reduce the rest here: from global memory while a level is too large for the
	// 16 KB tile buffer, then entirely in shared memory (one global read phase instead of one per level).
	uint32_t l = kPyrTileLevels;
	for (; l < hz.levels; ++l)
	{
		const uint32_t pw = max(1u, hz.width >> (l - 1)), ph = max(1u, hz.height >> (l - 1));
		const uint32_t lw = max(1u, hz.width >> l), lh = max(1u, hz.height >> l);
		if (pw * ph <= kPyrTile * kPyrTile && lw * lh <= (kPyrTile / 2) * (kPyrTile / 2))
			break; // this level fits s_a and the next one fits s_b: finish in shared memory
		const float* prev = hz.texels + hz.level_offset[l - 1];
		float* dst = hz.texels + hz.level_offset[l];
		for (uint32_t i = tid; i < lw * lh; i += kPyrBlock)
		{
			uint32_t x = i % lw, y = i / lw;
			uint32_t x0 = min(2 * x, pw - 1), x1 = min(2 * x + 1, pw - 1);
			uint32_t y0 = min(2 * y, ph - 1), y1 = min(2 * y + 1, ph - 1);
			// written by other CTAs / earlier iterations of this loop: bypass L1
			float v = fminf(fminf(__ldcg(prev + y0 * pw + x0), __ldcg(prev + y0 * pw + x1)), fminf(__ldcg(prev + y1 * pw + x0), __ldcg(prev + y1 * pw + x1)));
			dst[i] = v;
		}
		__threadfence_block();
		__syncthreads();
	}
	if (l < hz.levels)
	{
		uint32_t pw = max(1u, hz.width >> (l - 1)), ph = max(1u, hz.height >> (l - 1));
		const float* prev = hz.texels + hz.level_offset[l - 1];
		float* cur = s_a;
		float* nxt = s_b;
		for (uint32_t i = tid; i < pw * ph; i += kPyrBlock)
			cur[i] = __ldcg(prev + i); // written by other CTAs: bypass L1
		__syncthreads();
		for (; l < hz.levels; ++l)
		{
			const uint32_t lw = max(1u, hz.width >> l), lh = max(1u, hz.height >> l);
			float* dst = hz.texels + hz.level_offset[l];
			for (uint32_t i = tid; i < lw * lh; i += kPyrBlock)
			{
				float v = reduce2x2(cur, pw, ph, pw, i % lw, i / lw);
				dst[i] = v;
				nxt[i] = v; // fits: the first step writes <= 1024 texels into s_b, every later level at most halves
			}
			__syncthreads();
			float* t = cur;
			cur = nxt;
			nxt = t;
			pw = lw;
			ph = lh;
		}
	}
	if (tid == 0)
		p.scratch->pyramid_done = 0;
}

// ------------------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------------------

// meshlet.mesh.glsl:89-105 — what every mesh workgroup of vkCmdDrawMeshTasksIndirectEXT(ccb, 4) reads before it starts
// emitting vertices: slot -> cluster index -> task command -> meshlet.
__global__ void __launch_bounds__(256) decode_clusters_kernel(const uint32_t* __restrict__ cluster_indices, const uint32_t* __restrict__ cluster_count4,
    const NvcMeshTaskCommand* __restrict__ task_commands, const NvcMeshlet* __restrict__ meshlets, NvcClusterRecord* __restrict__ records, uint32_t* __restrict__ stats4)
{
	// dispatch (X, Y, Z) = (16, Y, 16): workgroup (x, y, z) reads clusterIndices[x + y * 256 + z * CLUSTER_TILE]
	const uint32_t gx = cluster_count4[1], gy = cluster_count4[2], gz = cluster_count4[3];
	const uint32_t slots = gx * gy * gz;
	uint32_t decoded = 0, skipped = 0, invalid = 0, triangles = 0;
	for (uint32_t w = blockIdx.x * blockDim.x + threadIdx.x; w < slots; w += gridDim.x * blockDim.x)
	{
		// enumerate workgroups x fastest, then z, then y so that slot = x + z * 16 + y * 256 is also w for (16, Y, 16)
		uint32_t x = w % gx, z = (w / gx) % gz, y = w / (gx * gz);
		uint32_t slot = x + y * 256u + z * NVC_CLUSTER_TILE;
		uint32_t ci = cluster_indices[slot];
		NvcClusterRecord r = { ~0u, ~0u, ~0u, ~0u };
		if (ci == ~0u)
			skipped++; // SetMeshOutputsEXT(0, 0)  :96-100
		else
		{
			const uint32_t* cp = reinterpret_cast<const uint32_t*>(task_commands + (ci & 0xffffffu)); // :102
			uint32_t lane = ci >> 24;
			uint32_t mi = cp[1] + lane; // :103
			if (lane >= cp[2])
				invalid++;
			r.drawId = cp[0];
			r.meshletIndex = mi;
			r.vertexCount = meshlets[mi].vertexCount;     // :107
			r.triangleCount = meshlets[mi].triangleCount; // :108
			decoded++;
			triangles += r.triangleCount;
		}
		if (records)
			records[slot] = r;
	}
	// warp-aggregate the four statistics, one atomic per warp and counter
#pragma unroll
	for (int o = 16; o >= 1; o >>= 1)
	{
		decoded += __shfl_xor_sync(0xffffffffu, decoded, o);
		skipped += __shfl_xor_sync(0xffffffffu, skipped, o);
		invalid += __shfl_xor_sync(0xffffffffu, invalid, o);
		triangles += __shfl_xor_sync(0xffffffffu, triangles, o);
	}
	if ((threadIdx.x & 31u) == 0)
	{
		if (decoded)
			atomicAdd(stats4 + 0, decoded);
		if (skipped)
			atomicAdd(stats4 + 1, skipped);
		if (invalid)
			atomicAdd(stats4 + 2, invalid);
		if (triangles)
			atomicAdd(stats4 + 3, triangles);
	}
}

cudaError_t launch_decode_clusters(const uint32_t* cluster_indices, const uint32_t* cluster_count4, const NvcMeshTaskCommand* task_commands, const NvcMeshlet* meshlets,
    NvcClusterRecord* records, uint32_t* stats4, uint32_t blocks, cudaStream_t stream)
{
	cudaError_t e = cudaMemsetAsync(stats4, 0, 16, stream);
	if (e != cudaSuccess)
		return e;
	decode_clusters_kernel<<<blocks, 256, 0, stream>>>(cluster_indices, cluster_count4, task_commands, meshlets, records, stats4);
	return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------
// Depth-only consumers of the cull output: what the reference's mesh / vertex stage + rasteriser do to the depth target between the
// cull passes (niagara.cpp:1576-1701, fixed-function raster, depth test GREATER on the reverse-Z buffer), in its three submission
// modes:
//   cluster submit  vkCmdDrawMeshTasksIndirectEXT(ccb, 4) -> meshlet.mesh.glsl:89-206 over cib       raster_clusters_kernel<false, *>
//   task shading    vkCmdDrawMeshTasksIndirectEXT(dccb, 4) -> meshlet.task EmitMeshTasksEXT(n) ->
//                   meshlet.mesh.glsl (TASK = true) over the task payloads                            raster_clusters_kernel<true, *>
//   (second parameter: the mesh shader's per-triangle cull stage, MESH_CULL = 1, nvc_set_mesh_cull)
//   indexed draws   vkCmdDrawIndexedIndirectCount(dcb + 4, dccb, 0, maxDrawCount, 24) -> mesh.vert    raster_indexed_kernel
// Cluster modes: one warp per cluster; the lanes transform the <= 64 vertices exactly as the mesh shader does (strict IEEE, GLSL
// operation order) into shared memory, then each lane rasterises its share of the <= 96 triangles.  Indexed mode: one warp per
// 1/32 of a command's triangles, each lane transforms the three corners of its triangles (mesh.vert's arithmetic is the mesh shader's).  Every triangle
// is sampled with the rule of the test rasteriser (oracle/refshader/driver.cpp rasterTriangle: pixel centres, edge functions and
// depth interpolation in binary64, back faces / w <= 0 dropped) and merged with atomicMax — max is order independent, so the image
// is bit-identical to the sequential CPU rasteriser's.
// This is what lets the two-phase path run on PRODUCED depth on the device (BASELINE configs[2]).
// ------------------------------------------------------------------------------------------------------
constexpr int kRasterWarps = 4;

__device__ __forceinline__ float4 mat4_mul_vec4(const float* __restrict__ m, float x, float y, float z, float w)
{
	// GLSL mat4 * vec4, column-major: ((col0 * x + col1 * y) + col2 * z) + col3 * w, every operation rounded
	float4 r;
	r.x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[0], x), __fmul_rn(m[4], y)), __fmul_rn(m[8], z)), __fmul_rn(m[12], w));
	r.y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[1], x), __fmul_rn(m[5], y)), __fmul_rn(m[9], z)), __fmul_rn(m[13], w));
	r.z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[2], x), __fmul_rn(m[6], y)), __fmul_rn(m[10], z)), __fmul_rn(m[14], w));
	r.w = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(m[3], x), __fmul_rn(m[7], y)), __fmul_rn(m[11], z)), __fmul_rn(m[15], w));
	return r;
}

// Clip position of vertices[vi] under the draw (d0 = position.xyz, scale; d1 = orientation): meshlet.mesh.glsl:127-140 ==
// mesh.vert.glsl:44-57, rotateQuat(position) * scale + position, then projection * (view * vec4(wpos, 1)).
__device__ __forceinline__ float4 transform_vertex(const NvcVertex* vertices, uint32_t vi, float4 d0, float4 d1, const float* view, const float* projection)
{
	const uint2 vv = __ldg(reinterpret_cast<const uint2*>(vertices + vi)); // vx, vy | vz, tp
	f3 pos = { half_bits_to_float(vv.x & 0xffffu), half_bits_to_float(vv.x >> 16), half_bits_to_float(vv.y & 0xffffu) };
	f3 r = rotate_quat(pos, d1);
	const float wx = __fadd_rn(__fmul_rn(r.x, d0.w), d0.x), wy = __fadd_rn(__fmul_rn(r.y, d0.w), d0.y), wz = __fadd_rn(__fmul_rn(r.z, d0.w), d0.z);
	const float4 v = mat4_mul_vec4(view, wx, wy, wz, 1.0f);
	return mat4_mul_vec4(projection, v.x, v.y, v.z, v.w);
}

// One triangle given as three clip-space corners, sampled into depth[height][width] with max (driver.cpp rasterTriangle).
// tris counts triangles that reach sampling, writes the depth updates issued.
__device__ __forceinline__ void raster_triangle(const float4 (&pc)[3], float* depth, uint32_t width, uint32_t height, double fw, double fh, uint32_t& tris, uint32_t& writes)
{
	double sx[3], sy[3], sz[3];
	bool front = true;
#pragma unroll
	for (int c = 0; c < 3; ++c)
	{
		front = front && pc[c].w > 0.0f;
		const float fx = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(pc[c].x, pc[c].w), 0.5f), 0.5f), float(width));
		const float fy = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(pc[c].y, pc[c].w), 0.5f), 0.5f), float(height));
		sx[c] = double(fx);
		sy[c] = double(fy);
		sz[c] = double(__fdiv_rn(pc[c].z, pc[c].w));
	}
	if (!front)
		return;
	const double ebx = __dsub_rn(sx[1], sx[0]), eby = __dsub_rn(sy[1], sy[0]), ecx = __dsub_rn(sx[2], sx[0]), ecy = __dsub_rn(sy[2], sy[0]);
	const double area = __dsub_rn(__dmul_rn(ebx, ecy), __dmul_rn(eby, ecx));
	if (!(area > 0.0))
		return; // back facing or zero area
	// flipped viewport: rows count from the top; swapping two corners keeps the edge functions positive inside
#pragma unroll
	for (int c = 0; c < 3; ++c)
		sy[c] = __dsub_rn(fh, sy[c]);
	{
		double tx = sx[1], ty = sy[1], tz = sz[1];
		sx[1] = sx[2], sy[1] = sy[2], sz[1] = sz[2];
		sx[2] = tx, sy[2] = ty, sz[2] = tz;
	}
	const double minx = fmin(sx[0], fmin(sx[1], sx[2])), maxx = fmax(sx[0], fmax(sx[1], sx[2]));
	const double miny = fmin(sy[0], fmin(sy[1], sy[2])), maxy = fmax(sy[0], fmax(sy[1], sy[2]));
	if (!(maxx >= 0.0 && maxy >= 0.0 && minx <= fw && miny <= fh))
		return;
	const int x0 = int(fmax(0.0, floor(__dsub_rn(minx, 0.5)))), x1 = int(fmin(__dsub_rn(fw, 1.0), ceil(__dsub_rn(maxx, 0.5))));
	const int y0 = int(fmax(0.0, floor(__dsub_rn(miny, 0.5)))), y1 = int(fmin(__dsub_rn(fh, 1.0), ceil(__dsub_rn(maxy, 0.5))));
	++tris;
	for (int yy = y0; yy <= y1; ++yy)
		for (int xx = x0; xx <= x1; ++xx)
		{
			const double px = __dadd_rn(double(xx), 0.5), py = __dadd_rn(double(yy), 0.5);
			const double w0 = __dsub_rn(__dmul_rn(__dsub_rn(sx[1], px), __dsub_rn(sy[2], py)), __dmul_rn(__dsub_rn(sy[1], py), __dsub_rn(sx[2], px)));
			const double w1 = __dsub_rn(__dmul_rn(__dsub_rn(sx[2], px), __dsub_rn(sy[0], py)), __dmul_rn(__dsub_rn(sy[2], py), __dsub_rn(sx[0], px)));
			const double w2 = __dsub_rn(__dmul_rn(__dsub_rn(sx[0], px), __dsub_rn(sy[1], py)), __dmul_rn(__dsub_rn(sy[0], py), __dsub_rn(sx[1], px)));
			if (w0 < 0.0 || w1 < 0.0 || w2 < 0.0)
				continue;
			const double num = __dadd_rn(__dadd_rn(__dmul_rn(w0, sz[0]), __dmul_rn(w1, sz[1])), __dmul_rn(w2, sz[2]));
			const double den = __dadd_rn(__dadd_rn(w0, w1), w2);
			const float zf = float(__ddiv_rn(num, den));
			// depth test GREATER on a buffer cleared to 0: only positive, ordered values can win; for those the float
			// order is the order of their bit patterns
			if (zf > 0.0f)
			{
				atomicMax(reinterpret_cast<int*>(depth) + size_t(yy) * width + xx, __float_as_int(zf));
				++writes;
			}
		}
}

// The per-triangle cull stage of meshlet.mesh.glsl:175-195 (compiled in with MESH_CULL = 1): true when the mesh shader marks the
// triangle gl_CullPrimitiveEXT.  p = (clip.xy / clip.w * 0.5 + 0.5) * screen is the float fx / fy of raster_triangle (meshlet.mesh.glsl:150
// keeps it in vertexClip); back faces and zero area: eb.x * ec.y <= eb.y * ec.x with two rounded products; small primitives: the
// bounding box rounds to one column or one row, sbprec = 1/256, `round` = roundf (halfway away from zero, the rule the host shim
// uses); all of it only when every corner has w > 0.  min / max are IEEE minNum / maxNum (a NaN corner drops out of the box, as in the
// shim); every comparison with a NaN operand is false, so a NaN w is never culled and reaches raster_triangle, which drops it.
__device__ __forceinline__ bool mesh_cull_triangle(const float4 (&pc)[3], float sw, float sh)
{
	float px[3], py[3];
#pragma unroll
	for (int c = 0; c < 3; ++c)
	{
		px[c] = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(pc[c].x, pc[c].w), 0.5f), 0.5f), sw);
		py[c] = __fmul_rn(__fadd_rn(__fmul_rn(__fdiv_rn(pc[c].y, pc[c].w), 0.5f), 0.5f), sh);
	}
	const float ebx = __fsub_rn(px[1], px[0]), eby = __fsub_rn(py[1], py[0]), ecx = __fsub_rn(px[2], px[0]), ecy = __fsub_rn(py[2], py[0]);
	bool culled = __fmul_rn(ebx, ecy) <= __fmul_rn(eby, ecx);
	const float bminx = fminf(px[0], fminf(px[1], px[2])), bmaxx = fmaxf(px[0], fmaxf(px[1], px[2]));
	const float bminy = fminf(py[0], fminf(py[1], py[2])), bmaxy = fmaxf(py[0], fmaxf(py[1], py[2]));
	const float sbprec = 1.0f / 256.0f;
	culled = culled || roundf(__fsub_rn(bminx, sbprec)) == roundf(bmaxx) || roundf(bminy) == roundf(__fadd_rn(bmaxy, sbprec));
	return culled && pc[0].w > 0.0f && pc[1].w > 0.0f && pc[2].w > 0.0f;
}

// warp-reduces the four per-lane counters and adds them to stats4 (nullptr: not wanted)
__device__ __forceinline__ void flush_stats4(uint32_t* stats4, uint32_t s0, uint32_t s1, uint32_t s2, uint32_t s3)
{
	if (!stats4)
		return;
#pragma unroll
	for (int o = 16; o >= 1; o >>= 1)
	{
		s0 += __shfl_xor_sync(0xffffffffu, s0, o);
		s1 += __shfl_xor_sync(0xffffffffu, s1, o);
		s2 += __shfl_xor_sync(0xffffffffu, s2, o);
		s3 += __shfl_xor_sync(0xffffffffu, s3, o);
	}
	if (lane_id() == 0)
	{
		if (s0)
			atomicAdd(stats4 + 0, s0);
		if (s1)
			atomicAdd(stats4 + 1, s1);
		if (s2)
			atomicAdd(stats4 + 2, s2);
		if (s3)
			atomicAdd(stats4 + 3, s3);
	}
}

struct RasterParams
{
	float projection[16];
	float view[16];
	const uint32_t* cluster_indices; // cluster submit: cib
	const uint32_t* cluster_count4;  // cluster submit: ccb
	const NvcMeshTaskPayload* payloads; // task shading: payloads[c], emit_counts[c] for c < command_count4[1] * 64
	const uint32_t* emit_counts;
	const uint32_t* command_count4; // task shading / indexed draws: dccb
	const NvcMeshTaskCommand* task_commands;
	const NvcMeshDrawCommand* draw_commands; // indexed draws: dcb, indices[index_count]
	const uint32_t* indices;
	uint32_t index_count, max_draw_count;
	const NvcMeshDraw* draws;
	const NvcMeshlet* meshlets;
	const uint32_t* meshletdata;
	uint32_t meshletdata_words;
	const NvcVertex* vertices;
	uint32_t vertex_count;
	float* depth;
	uint32_t width, height;
	// clusters / commands drawn, triangles rasterised, clusters / commands rejected (data out of range), cluster modes: depth
	// updates issued, indexed draws: triangles rejected (vertex index out of range)
	uint32_t* stats4;
	// MeshCull instantiations: triangles tested and culled by the mesh-cull stage, added to these two context-owned counters
	unsigned long long* mesh_cull2;
};

// Task = false: work item w is slot x + y * 256 + z * 16 of the (16, Y, 16) dispatch in ccb, reading cib (meshlet.mesh.glsl:94).
// Task = true: work item w is mesh workgroup i = w % 64 of task command c = w / 64 of the (X, 64, 1) dispatch in dccb; it exists when
// i < min(emit_counts[c], 64) and reads payloads[c].clusterIndices[i].  Everything after the cluster index is the same code.
// MeshCull = true: a triangle that passes the index checks is first given the mesh-cull decision (mesh_cull_triangle) and only
// sampled when not culled; tested / culled triangles are added to p.mesh_cull2.
template <bool Task, bool MeshCull>
__global__ void __launch_bounds__(kRasterWarps * 32) raster_clusters_kernel(const RasterParams p)
{
	__shared__ float4 s_clip[kRasterWarps][64];
	const uint32_t lane = lane_id(), warp = threadIdx.x >> 5;
	uint32_t gx = 0, gz = 0, items;
	if (Task)
		items = min(p.command_count4[1], NVC_MAX_DISPATCH_GROUPS) * NVC_TASK_WGSIZE * NVC_TASK_WGSIZE;
	else
	{
		gx = p.cluster_count4[1];
		gz = p.cluster_count4[3];
		items = gx * p.cluster_count4[2] * gz;
	}
	float4* clip = s_clip[warp];
	uint32_t drawn = 0, tris = 0, rejected = 0, writes = 0, tested = 0, culled = 0;
	const double fw = double(p.width), fh = double(p.height);

	for (uint32_t w = blockIdx.x * kRasterWarps + warp; w < items; w += gridDim.x * kRasterWarps)
	{
		uint32_t ci;
		if (Task)
		{
			const uint32_t c = w / NVC_TASK_WGSIZE, i = w % NVC_TASK_WGSIZE;
			if (i >= min(__ldg(p.emit_counts + c), NVC_TASK_WGSIZE))
				continue; // EmitMeshTasksEXT(n) launched no such workgroup
			ci = __ldg(p.payloads[c].clusterIndices + i);
		}
		else
		{
			const uint32_t x = w % gx, z = (w / gx) % gz, y = w / (gx * gz);
			const uint32_t slot = x + y * 256u + z * NVC_CLUSTER_TILE; // meshlet.mesh.glsl:94
			ci = __ldg(p.cluster_indices + slot);
		}
		if (ci == ~0u)
			continue; // SetMeshOutputsEXT(0, 0)
		const uint32_t* cp = reinterpret_cast<const uint32_t*>(p.task_commands + (ci & 0xffffffu));
		const uint32_t drawId = __ldg(cp + 0), mi = __ldg(cp + 1) + (ci >> 24);
		const NvcMeshlet& ml = p.meshlets[mi];
		const uint32_t vertexCount = ml.vertexCount, triangleCount = ml.triangleCount;
		const uint32_t dataOffset = ml.dataOffset, baseVertex = ml.baseVertex;
		const bool shortRefs = ml.shortRefs == 1;
		const uint32_t indexOffset = dataOffset + mcodec::reference_words(vertexCount, shortRefs);
		// the meshlet's references / triangle bytes must lie inside meshletdata (robustBufferAccess in the reference; here: skip)
		const uint64_t end_words = uint64_t(indexOffset) + (uint64_t(triangleCount) * 3 + 3) / 4;
		if (vertexCount > mcodec::kMaxVertices || triangleCount > mcodec::kMaxTriangles || end_words > p.meshletdata_words)
		{
			rejected += lane == 0;
			continue;
		}
		const char* dp = reinterpret_cast<const char*>(p.draws + drawId);
		const float4 d0 = ldg_f4(dp), d1 = ldg_f4(dp + 16);

		// ---- vertices: meshlet.mesh.glsl:126-147 ----
		bool bad = false;
		for (uint32_t i = lane; i < vertexCount; i += 32)
		{
			uint32_t ref = shortRefs ? uint32_t(reinterpret_cast<const uint16_t*>(p.meshletdata)[size_t(dataOffset) * 2 + i]) : __ldg(p.meshletdata + dataOffset + i);
			uint32_t vi = ref + baseVertex;
			if (vi >= p.vertex_count)
			{
				bad = true;
				break;
			}
			clip[i] = transform_vertex(p.vertices, vi, d0, d1, p.view, p.projection);
		}
		if (__any_sync(0xffffffffu, bad))
		{
			rejected += lane == 0;
			__syncwarp();
			continue;
		}
		__syncwarp();
		drawn += lane == 0;

		// ---- triangles ----
		const uint8_t* tri8 = reinterpret_cast<const uint8_t*>(p.meshletdata) + size_t(indexOffset) * 4;
		for (uint32_t t = lane; t < triangleCount; t += 32)
		{
			const uint32_t ia = tri8[t * 3 + 0], ib = tri8[t * 3 + 1], ic = tri8[t * 3 + 2];
			if (ia >= vertexCount || ib >= vertexCount || ic >= vertexCount)
				continue;
			const float4 pc[3] = { clip[ia], clip[ib], clip[ic] };
			if (MeshCull)
			{
				++tested;
				if (mesh_cull_triangle(pc, float(p.width), float(p.height)))
				{
					++culled;
					continue; // gl_CullPrimitiveEXT
				}
			}
			raster_triangle(pc, p.depth, p.width, p.height, fw, fh, tris, writes);
		}
		__syncwarp(); // the next cluster reuses clip[]
	}
	flush_stats4(p.stats4, drawn, tris, rejected, writes);
	if (MeshCull)
	{
#pragma unroll
		for (int o = 16; o >= 1; o >>= 1)
		{
			tested += __shfl_xor_sync(0xffffffffu, tested, o);
			culled += __shfl_xor_sync(0xffffffffu, culled, o);
		}
		if (lane == 0 && tested)
		{
			atomicAdd(p.mesh_cull2 + 0, (unsigned long long)tested);
			atomicAdd(p.mesh_cull2 + 1, (unsigned long long)culled);
		}
	}
}

// Commands i < min(command_count4[0], max_draw_count) of dcb, each split into kIndexedSlices equal runs of its indexCount / 3
// triangles; one warp per (command, run) (grid-stride), the lanes striding over the run.  Corner k of triangle t is vertex
// indices[firstIndex + 3t + k] + vertexOffset (uint32 wrap) under draws[drawId] (gl_DrawIDARB only selects the command).
// mesh.vert ignores gl_InstanceIndex and max is idempotent, so a command with instanceCount >= 1 is drawn once and one with
// instanceCount == 0 draws nothing.
// One warp per whole command was 8x slower than cluster submit on the C3 stand-in (H100, 23 ms against 2.9 ms for the early
// pass): a close LOD-0 kitten (28 944 triangles) kept a single warp busy for the whole pass.
constexpr uint32_t kIndexedSlices = 32;

__global__ void __launch_bounds__(kRasterWarps * 32) raster_indexed_kernel(const RasterParams p)
{
	const uint32_t lane = lane_id(), warp = threadIdx.x >> 5;
	const uint64_t items = uint64_t(min(p.command_count4[0], p.max_draw_count)) * kIndexedSlices;
	uint32_t drawn = 0, tris = 0, rejected = 0, bad_tris = 0, writes = 0;
	const double fw = double(p.width), fh = double(p.height);

	for (uint64_t w = blockIdx.x * kRasterWarps + warp; w < items; w += gridDim.x * kRasterWarps)
	{
		const uint32_t slice = uint32_t(w % kIndexedSlices);
		const uint32_t* cp = reinterpret_cast<const uint32_t*>(p.draw_commands + w / kIndexedSlices);
		const uint32_t drawId = __ldg(cp + 0), indexCount = __ldg(cp + 1), instanceCount = __ldg(cp + 2);
		const uint32_t firstIndex = __ldg(cp + 3), vertexOffset = __ldg(cp + 4);
		if (instanceCount == 0)
			continue;
		if (uint64_t(firstIndex) + indexCount > p.index_count)
		{
			rejected += lane == 0 && slice == 0;
			continue;
		}
		drawn += lane == 0 && slice == 0;
		const uint32_t triangles = indexCount / 3; // trailing indices that make no whole triangle are not drawn
		const uint32_t run = (triangles + kIndexedSlices - 1) / kIndexedSlices;
		const uint32_t t_end = min(triangles, slice * run + run);
		if (slice * run >= t_end)
			continue;
		const char* dp = reinterpret_cast<const char*>(p.draws + drawId);
		const float4 d0 = ldg_f4(dp), d1 = ldg_f4(dp + 16);
		const uint32_t* idx = p.indices + firstIndex;
		for (uint32_t t = slice * run + lane; t < t_end; t += 32)
		{
			const uint32_t va = __ldg(idx + size_t(t) * 3 + 0) + vertexOffset, vb = __ldg(idx + size_t(t) * 3 + 1) + vertexOffset, vc = __ldg(idx + size_t(t) * 3 + 2) + vertexOffset;
			if (va >= p.vertex_count || vb >= p.vertex_count || vc >= p.vertex_count)
			{
				++bad_tris;
				continue;
			}
			const float4 pc[3] = { transform_vertex(p.vertices, va, d0, d1, p.view, p.projection), transform_vertex(p.vertices, vb, d0, d1, p.view, p.projection),
				transform_vertex(p.vertices, vc, d0, d1, p.view, p.projection) };
			raster_triangle(pc, p.depth, p.width, p.height, fw, fh, tris, writes);
		}
	}
	flush_stats4(p.stats4, drawn, tris, rejected, bad_tris);
}

namespace
{

RasterParams raster_params(const float* projection16, const NvcCullData& pass, const NvcMeshDraw* draws, const NvcVertex* vertices, uint32_t vertex_count, float* depth, uint32_t width,
    uint32_t height, uint32_t* stats4)
{
	RasterParams p;
	memset(&p, 0, sizeof(p));
	memcpy(p.projection, projection16, sizeof(p.projection));
	memcpy(p.view, pass.view, sizeof(p.view));
	p.draws = draws;
	p.vertices = vertices;
	p.vertex_count = vertex_count;
	p.depth = depth;
	p.width = width;
	p.height = height;
	p.stats4 = stats4;
	return p;
}

cudaError_t launch_raster(void (*kernel)(RasterParams), const RasterParams& p, uint32_t blocks, cudaStream_t stream)
{
	if (p.stats4)
	{
		cudaError_t e = cudaMemsetAsync(p.stats4, 0, 16, stream);
		if (e != cudaSuccess)
			return e;
	}
	kernel<<<blocks, kRasterWarps * 32, 0, stream>>>(p);
	return cudaGetLastError();
}

} // namespace

cudaError_t launch_raster_depth(const float* projection16, const NvcCullData& pass, const uint32_t* cluster_indices, const uint32_t* cluster_count4, const NvcMeshTaskCommand* task_commands,
    const NvcMeshDraw* draws, const NvcMeshlet* meshlets, const uint32_t* meshletdata, uint32_t meshletdata_words, const NvcVertex* vertices, uint32_t vertex_count, float* depth, uint32_t width,
    uint32_t height, uint32_t* stats4, unsigned long long* mesh_cull2, uint32_t blocks, cudaStream_t stream)
{
	RasterParams p = raster_params(projection16, pass, draws, vertices, vertex_count, depth, width, height, stats4);
	p.cluster_indices = cluster_indices;
	p.cluster_count4 = cluster_count4;
	p.task_commands = task_commands;
	p.meshlets = meshlets;
	p.meshletdata = meshletdata;
	p.meshletdata_words = meshletdata_words;
	p.mesh_cull2 = mesh_cull2;
	return launch_raster(mesh_cull2 ? raster_clusters_kernel<false, true> : raster_clusters_kernel<false, false>, p, blocks, stream);
}

cudaError_t launch_raster_depth_tasks(const float* projection16, const NvcCullData& pass, const NvcMeshTaskPayload* payloads, const uint32_t* emit_counts, const uint32_t* command_count4,
    const NvcMeshTaskCommand* task_commands, const NvcMeshDraw* draws, const NvcMeshlet* meshlets, const uint32_t* meshletdata, uint32_t meshletdata_words, const NvcVertex* vertices,
    uint32_t vertex_count, float* depth, uint32_t width, uint32_t height, uint32_t* stats4, unsigned long long* mesh_cull2, uint32_t blocks, cudaStream_t stream)
{
	RasterParams p = raster_params(projection16, pass, draws, vertices, vertex_count, depth, width, height, stats4);
	p.payloads = payloads;
	p.emit_counts = emit_counts;
	p.command_count4 = command_count4;
	p.task_commands = task_commands;
	p.meshlets = meshlets;
	p.meshletdata = meshletdata;
	p.meshletdata_words = meshletdata_words;
	p.mesh_cull2 = mesh_cull2;
	return launch_raster(mesh_cull2 ? raster_clusters_kernel<true, true> : raster_clusters_kernel<true, false>, p, blocks, stream);
}

cudaError_t launch_raster_depth_indexed(const float* projection16, const NvcCullData& pass, const NvcMeshDrawCommand* draw_commands, const uint32_t* command_count4, uint32_t max_draw_count,
    const NvcMeshDraw* draws, const uint32_t* indices, uint32_t index_count, const NvcVertex* vertices, uint32_t vertex_count, float* depth, uint32_t width, uint32_t height, uint32_t* stats4,
    uint32_t blocks, cudaStream_t stream)
{
	RasterParams p = raster_params(projection16, pass, draws, vertices, vertex_count, depth, width, height, stats4);
	p.draw_commands = draw_commands;
	p.command_count4 = command_count4;
	p.max_draw_count = max_draw_count;
	p.indices = indices;
	p.index_count = index_count;
	return launch_raster(raster_indexed_kernel, p, blocks, stream);
}

// N4: meshlet bounds + normal cone, one thread per meshlet (csrc/nvc_cook.cuh).  A meshlet whose data or vertices would
// fall outside the given arrays is left untouched and counted in *rejected.
__global__ void __launch_bounds__(128) cook_meshlet_bounds_kernel(const NvcVertex* __restrict__ vertices, uint32_t vertex_count, const uint32_t* __restrict__ meshletdata,
    uint32_t meshletdata_words, NvcMeshlet* __restrict__ meshlets, uint32_t meshlet_count, uint32_t* __restrict__ rejected)
{
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= meshlet_count)
		return;
	NvcMeshlet m = meshlets[i];
	cook::MeshletView view;
	view.vertices = vertices;
	view.data = meshletdata + m.dataOffset;
	view.baseVertex = m.baseVertex;
	view.vertexCount = m.vertexCount;
	view.triangleCount = m.triangleCount;
	view.shortRefs = m.shortRefs;
	uint32_t ref_words = m.shortRefs ? (uint32_t(m.vertexCount) + 1u) / 2u : m.vertexCount;
	uint64_t words = uint64_t(ref_words) + (uint64_t(m.triangleCount) * 3u + 3u) / 4u;
	bool ok = uint64_t(m.dataOffset) + words <= meshletdata_words;
	if (ok)
	{
		for (uint32_t k = 0; k < m.vertexCount; ++k)
			ok = ok && uint64_t(m.baseVertex) + view.ref(k) < vertex_count;
		for (uint32_t t = 0; t < m.triangleCount; ++t)
			for (uint32_t c = 0; c < 3; ++c)
				ok = ok && view.corner(t, c) < m.vertexCount;
	}
	if (!ok)
	{
		if (rejected)
			atomicAdd(rejected, 1u);
		return;
	}
	cook::meshlet_bounds(view, &m);
	// center[3] + radius + cone_axis[3] + cone_cutoff = the first 12 bytes of the Meshlet
	uint32_t w[3];
	memcpy(w, &m, 12);
	uint32_t* dst = reinterpret_cast<uint32_t*>(meshlets + i);
	dst[0] = w[0];
	dst[1] = w[1];
	dst[2] = w[2];
}

cudaError_t launch_cook_meshlet_bounds(const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* meshletdata, uint32_t meshletdata_words, NvcMeshlet* meshlets,
    uint32_t meshlet_count, uint32_t* rejected, cudaStream_t stream)
{
	if (rejected)
	{
		cudaError_t e = cudaMemsetAsync(rejected, 0, 4, stream);
		if (e != cudaSuccess)
			return e;
	}
	if (meshlet_count == 0)
		return cudaSuccess;
	cook_meshlet_bounds_kernel<<<(meshlet_count + 127u) / 128u, 128, 0, stream>>>(vertices, vertex_count, meshletdata, meshletdata_words, meshlets, meshlet_count, rejected);
	return cudaGetLastError();
}

// N4: meshlet building and packing (csrc/nvc_meshlets.cuh)
namespace
{

constexpr uint32_t kCookWarps = 4;        // jobs per block of the build kernel
constexpr uint32_t kCookScanThreads = 256; // the one block of the scan kernel

// Orders scores as floats do, with -0 == +0 and NaN above everything
__device__ __forceinline__ uint32_t cook_score_key(float s)
{
	if (s != s)
		return 0xffffffffu;
	uint32_t u = cook::float_bits(s == 0.0f ? 0.0f : s);
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// getNeighborTriangle (clusterizer.cpp:302-362) for the whole warp.  Candidate k is the k-th (meshlet vertex, live
// neighbour) pair in the reference's loop order; lanes take k = lane, lane + 32, ...  The reference keeps the best
// (priority, score) on a strict '<', i.e. among the lowest priority the first candidate of the least score -- unless the
// first candidate of that priority scores NaN, which no later candidate then replaces.  So two minima are reduced:
// (priority, k) and (priority, score, k).
__device__ uint32_t cook_neighbor(uint32_t lane, const cook::Building& m, const cook::Cone& mc, const uint32_t* mlv, const uint32_t* indices, const uint32_t* counts,
    const uint32_t* offsets, const uint32_t* data, const float* cones, const int16_t* used, float expected_radius, uint32_t* s_prefix, uint32_t* s_mv)
{
	const uint32_t full = 0xffffffffu;
	uint32_t v0 = 0, v1 = 0, c0 = 0, c1 = 0;
	if (lane < m.vertex_count)
	{
		v0 = mlv[m.vertex_offset + lane];
		c0 = counts[v0];
	}
	if (lane + 32 < m.vertex_count)
	{
		v1 = mlv[m.vertex_offset + lane + 32];
		c1 = counts[v1];
	}
	uint32_t p0 = scan::warp_inclusive(c0, lane);
	uint32_t p1 = scan::warp_inclusive(c1, lane) + __shfl_sync(full, p0, 31);
	if (lane == 0)
		s_prefix[0] = 0;
	s_prefix[lane + 1] = p0;
	s_prefix[lane + 33] = p1;
	s_mv[lane] = v0;
	s_mv[lane + 32] = v1;
	__syncwarp();
	const uint32_t total = s_prefix[m.vertex_count];

	uint32_t fp = 5, fk = 0, fs = 0, ft = cook::kNone; // first candidate of the least priority, its score bits
	uint32_t bp = 5, bs = 0, bk = 0, bt = cook::kNone; // least (priority, score, k)
	for (uint32_t k = lane; k < total; k += 32)
	{
		const uint32_t lo = scan::last_at_most(m.vertex_count, k, [&](uint32_t i) { return s_prefix[i]; });
		uint32_t tri = data[offsets[s_mv[lo]] + (k - s_prefix[lo])];
		uint32_t a = indices[tri * 3 + 0], b = indices[tri * 3 + 1], c = indices[tri * 3 + 2];
		uint32_t extra = (used[a] < 0) + (used[b] < 0) + (used[c] < 0);
		uint32_t priority;
		if (extra == 0)
			priority = 0;
		else if (counts[a] == 1 || counts[b] == 1 || counts[c] == 1)
			priority = 1;
		else if ((counts[a] == 2) + (counts[b] == 2) + (counts[c] == 2) >= 2)
			priority = 1 + extra;
		else
			priority = 2 + extra;
		if (priority > bp)
			continue;
		const float* tc = cones + size_t(tri) * 6u;
		float distance = cook::point_distance(tc, mc.px, mc.py, mc.pz);
		float spread = cook::add(cook::add(cook::mul(tc[3], mc.nx), cook::mul(tc[4], mc.ny)), cook::mul(tc[5], mc.nz));
		float score = cook::meshlet_score(distance, spread, expected_radius);
		uint32_t key = cook_score_key(score);
		if (priority < fp) // k increases within a lane: the first of a priority is the first seen
		{
			fp = priority;
			fk = k;
			fs = cook::float_bits(score);
			ft = tri;
		}
		if (priority < bp || (priority == bp && key < bs))
		{
			bp = priority;
			bs = key;
			bk = k;
			bt = tri;
		}
	}
	for (int d = 16; d > 0; d >>= 1)
	{
		uint32_t op = __shfl_xor_sync(full, fp, d), ok = __shfl_xor_sync(full, fk, d), os = __shfl_xor_sync(full, fs, d), ot = __shfl_xor_sync(full, ft, d);
		if (op < fp || (op == fp && ok < fk))
			fp = op, fk = ok, fs = os, ft = ot;
		uint32_t bp2 = __shfl_xor_sync(full, bp, d), bs2 = __shfl_xor_sync(full, bs, d), bk2 = __shfl_xor_sync(full, bk, d), bt2 = __shfl_xor_sync(full, bt, d);
		if (bp2 < bp || (bp2 == bp && (bs2 < bs || (bs2 == bs && bk2 < bk))))
			bp = bp2, bs = bs2, bk = bk2, bt = bt2;
	}
	__syncwarp(); // s_prefix / s_mv are rewritten by the next call
	if (fp == 5)
		return cook::kNone;
	float first = cook::bits_float(fs);
	return first != first ? ft : bt;
}

// One warp per (mesh, LOD) job: meshopt_buildMeshletsFlex (clusterizer.cpp:1035-1224) with the parameters of
// meshopt_buildMeshlets(64, 96, 0.25).  Jobs are taken in a.order (largest first); results are placed by job index.
__global__ void __launch_bounds__(kCookWarps * 32) cook_build_kernel(const CookArgs a)
{
	__shared__ uint32_t s_seeds[kCookWarps][cook::kMaxSeeds];
	__shared__ uint32_t s_prefix[kCookWarps][2 * 32 + 1];
	__shared__ uint32_t s_mv[kCookWarps][cook::kMaxVertices];
	__shared__ uint32_t s_bn[kCookWarps][cook::kMaxVertices];
	__shared__ uint32_t s_bl[kCookWarps][cook::kMaxVertices];
	__shared__ float s_bs[kCookWarps][cook::kMaxVertices];
	const uint32_t full = 0xffffffffu;
	const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
	const uint32_t w = blockIdx.x * kCookWarps + warp;
	if (w >= a.job_count)
		return;
	const uint32_t j = a.order[w];
	const cook::CookJob job = a.jobs[j];
	const uint32_t* indices = a.indices + job.index_offset;
	const uint32_t index_count = job.index_count, faces = index_count / 3, vertex_count = job.vertex_count;

	// an index outside the mesh: the LOD gets no meshlets (the reference asserts)
	bool bad = false;
	for (uint32_t i = lane; i < index_count; i += 32)
		bad = bad || indices[i] >= vertex_count;
	if (__any_sync(full, bad) || faces == 0)
	{
		if (lane == 0)
		{
			a.job_meshlets[j] = 0;
			if (faces != 0)
				atomicAdd(a.totals4 + 2, 1u);
		}
		return;
	}

	float* cones = a.cones + job.tri * 6u;
	uint32_t* counts = a.adj_counts + job.vtx;
	uint32_t* offsets = a.adj_offsets + job.vtx;
	uint32_t* data = a.adj_data + job.idx;
	int16_t* used = a.used + job.vtx;
	uint8_t* emitted = a.emitted + job.tri;
	uint32_t* nodes = a.kd_nodes + job.tri * 6u;
	uint32_t* kdi = a.kd_index + job.tri;
	uint32_t* mlv = a.ml_vertices + job.idx;
	uint8_t* mlt = a.ml_triangles + job.idx;
	uint4* records = a.ml_records + job.slot;
	float* areas = reinterpret_cast<float*>(mlv); // free until the greedy loop
	const NvcVertex* verts = a.vertices + job.vertex_offset;

	// computeTriangleCones (clusterizer.cpp:201-241), areas summed below in triangle order
	for (uint32_t t = lane; t < faces; t += 32)
	{
		cook::V3 p[3];
		for (int k = 0; k < 3; ++k)
		{
			const NvcVertex& v = verts[indices[t * 3 + k]];
			p[k] = cook::V3{ cook::dequantize_half(v.vx), cook::dequantize_half(v.vy), cook::dequantize_half(v.vz) };
		}
		cook::Cone c;
		areas[t] = cook::triangle_cone(p[0], p[1], p[2], c);
		float* dst = cones + size_t(t) * 6u;
		dst[0] = c.px, dst[1] = c.py, dst[2] = c.pz, dst[3] = c.nx, dst[4] = c.ny, dst[5] = c.nz;
		emitted[t] = 0;
		kdi[t] = t;
	}
	for (uint32_t v = lane; v < vertex_count; v += 32)
	{
		counts[v] = 0;
		used[v] = -1;
	}
	__syncwarp();
	// buildTriangleAdjacency (clusterizer.cpp:40-86): counts, offsets, then a sequential (stable) fill
	for (uint32_t i = lane; i < index_count; i += 32)
		atomicAdd(counts + indices[i], 1u);
	__syncwarp();
	uint32_t carry = 0;
	for (uint32_t base = 0; base < vertex_count; base += 32)
	{
		uint32_t v = base + lane;
		uint32_t c = v < vertex_count ? counts[v] : 0u;
		uint32_t incl = scan::warp_inclusive(c, lane);
		if (v < vertex_count)
			offsets[v] = carry + incl - c;
		carry += __shfl_sync(full, incl, 31);
	}
	__syncwarp();

	float expected_radius = 0.0f, corner[3] = { FLT_MAX, FLT_MAX, FLT_MAX };
	uint32_t initial_seed = cook::kNone;
	if (lane == 0)
	{
		for (uint32_t t = 0; t < faces; ++t)
		{
			data[offsets[indices[t * 3 + 0]]++] = t;
			data[offsets[indices[t * 3 + 1]]++] = t;
			data[offsets[indices[t * 3 + 2]]++] = t;
		}
		float mesh_area = 0.0f;
		for (uint32_t t = 0; t < faces; ++t)
			mesh_area = cook::add(mesh_area, areas[t]);
		float triangle_area_avg = cook::mul(cook::div(mesh_area, float(faces)), 0.5f);
		expected_radius = cook::mul(cook::root(cook::mul(triangle_area_avg, float(cook::kMaxTriangles))), 0.5f);
		cook::kd_build(nodes, cones, kdi, faces);
		for (uint32_t t = 0; t < faces; ++t)
		{
			const float* c = cones + size_t(t) * 6u;
			corner[0] = corner[0] > c[0] ? c[0] : corner[0];
			corner[1] = corner[1] > c[1] ? c[1] : corner[1];
			corner[2] = corner[2] > c[2] ? c[2] : corner[2];
		}
		float initial_score = FLT_MAX;
		for (uint32_t t = 0; t < faces; ++t)
		{
			float score = cook::point_distance(cones + size_t(t) * 6u, corner[0], corner[1], corner[2]);
			if (initial_seed == cook::kNone || score < initial_score)
			{
				initial_seed = t;
				initial_score = score;
			}
		}
	}
	__syncwarp();
	for (uint32_t v = lane; v < vertex_count; v += 32)
		offsets[v] -= counts[v];
	expected_radius = __shfl_sync(full, expected_radius, 0);
	corner[0] = __shfl_sync(full, corner[0], 0);
	corner[1] = __shfl_sync(full, corner[1], 0);
	corner[2] = __shfl_sync(full, corner[2], 0);
	initial_seed = __shfl_sync(full, initial_seed, 0);
	__syncwarp();

	uint32_t* seeds = s_seeds[warp];
	uint32_t seed_count = 0, meshlet_offset = 0;
	cook::Building m = { 0, 0, 0, 0 };
	cook::Cone acc = { 0, 0, 0, 0, 0, 0 };
	for (;;)
	{
		cook::Cone mc = cook::meshlet_cone(acc, m.triangle_count);
		uint32_t best = cook::kNone;
		if (meshlet_offset == 0 && m.triangle_count == 0)
			best = initial_seed;
		else
			best = cook_neighbor(lane, m, mc, mlv, indices, counts, offsets, data, cones, used, expected_radius, s_prefix[warp], s_mv[warp]);
		if (best == cook::kNone)
		{
			if (lane == 0)
			{
				float position[3] = { mc.px, mc.py, mc.pz };
				float distance = FLT_MAX;
				cook::kd_nearest(nodes, cones, emitted, position, best, distance);
			}
			best = __shfl_sync(full, best, 0);
		}
		if (best == cook::kNone)
			break;

		int best_extra = (used[indices[best * 3 + 0]] < 0) + (used[indices[best * 3 + 1]] < 0) + (used[indices[best * 3 + 2]] < 0);
		if (m.vertex_count + best_extra > cook::kMaxVertices || m.triangle_count >= cook::kMaxTriangles)
		{
			// appendSeedTriangles (clusterizer.cpp:364-430): each meshlet vertex's least-live neighbour, by lanes
			for (uint32_t i = lane; i < m.vertex_count; i += 32)
			{
				uint32_t v = mlv[m.vertex_offset + i];
				const uint32_t* nb = data + offsets[v];
				uint32_t n = counts[v], bn = cook::kNone, bl = cook::kNone;
				for (uint32_t q = 0; q < n; ++q)
				{
					uint32_t tri = nb[q];
					uint32_t live = counts[indices[tri * 3 + 0]] + counts[indices[tri * 3 + 1]] + counts[indices[tri * 3 + 2]];
					if (live < bl)
					{
						bn = tri;
						bl = live;
					}
				}
				s_bn[warp][i] = bn;
				s_bl[warp][i] = bl;
				s_bs[warp][i] = bn == cook::kNone ? 0.0f : cook::point_distance(cones + size_t(bn) * 6u, corner[0], corner[1], corner[2]);
			}
			__syncwarp();
			if (lane == 0)
			{
				// pruneSeedTriangles (:432-445) and the cap of :1164
				uint32_t kept = 0;
				for (uint32_t i = 0; i < seed_count; ++i)
				{
					uint32_t index = seeds[i];
					seeds[kept] = index;
					kept += emitted[index] == 0;
				}
				seed_count = kept + cook::kAddSeeds <= cook::kMaxSeeds ? kept : cook::kMaxSeeds - cook::kAddSeeds;
				uint32_t best_seeds[cook::kAddSeeds], best_live[cook::kAddSeeds];
				float best_score[cook::kAddSeeds];
				for (uint32_t i = 0; i < cook::kAddSeeds; ++i)
				{
					best_seeds[i] = cook::kNone;
					best_live[i] = cook::kNone;
					best_score[i] = FLT_MAX;
				}
				for (uint32_t i = 0; i < m.vertex_count; ++i)
				{
					uint32_t bn = s_bn[warp][i], bl = s_bl[warp][i];
					float bs = s_bs[warp][i];
					if (bn == cook::kNone)
						continue;
					for (uint32_t q = 0; q < cook::kAddSeeds; ++q)
						if (bl < best_live[q] || (bl == best_live[q] && bs <= best_score[q]))
						{
							best_seeds[q] = bn;
							best_live[q] = bl;
							best_score[q] = bs;
							break;
						}
				}
				for (uint32_t i = 0; i < cook::kAddSeeds; ++i)
					if (best_seeds[i] != cook::kNone)
						seeds[seed_count++] = best_seeds[i];
				uint32_t best_seed = cook::select_seed(seeds, seed_count, indices, cones, counts, corner);
				best = best_seed != cook::kNone ? best_seed : best;
			}
			best = __shfl_sync(full, best, 0);
			seed_count = __shfl_sync(full, seed_count, 0);
		}

		uint32_t flushed = 0;
		if (lane == 0)
			flushed = cook::append_triangle(m, indices[best * 3 + 0], indices[best * 3 + 1], indices[best * 3 + 2], used, records, meshlet_offset, mlv, mlt) ? 1u : 0u;
		flushed = __shfl_sync(full, flushed, 0);
		m.vertex_offset = __shfl_sync(full, m.vertex_offset, 0);
		m.triangle_offset = __shfl_sync(full, m.triangle_offset, 0);
		m.vertex_count = __shfl_sync(full, m.vertex_count, 0);
		m.triangle_count = __shfl_sync(full, m.triangle_count, 0);
		if (flushed)
		{
			meshlet_offset++;
			acc = cook::Cone{ 0, 0, 0, 0, 0, 0 };
		}
		__syncwarp();

		// swap-with-last removal of `best` from its vertices' lists (:1186-1204), one vertex after the other
		for (int k = 0; k < 3; ++k)
		{
			uint32_t v = indices[best * 3 + k];
			uint32_t* nb = data + offsets[v];
			uint32_t n = counts[v];
			for (uint32_t base = 0; base < n; base += 32)
			{
				uint32_t i = base + lane;
				uint32_t hit = __ballot_sync(full, i < n && nb[i] == best);
				if (hit)
				{
					if (lane == uint32_t(__ffs(int(hit)) - 1))
					{
						nb[i] = nb[n - 1];
						counts[v] = n - 1;
					}
					break;
				}
			}
			__syncwarp();
		}

		const float* bc = cones + size_t(best) * 6u;
		acc.px = cook::add(acc.px, bc[0]);
		acc.py = cook::add(acc.py, bc[1]);
		acc.pz = cook::add(acc.pz, bc[2]);
		acc.nx = cook::add(acc.nx, bc[3]);
		acc.ny = cook::add(acc.ny, bc[4]);
		acc.nz = cook::add(acc.nz, bc[5]);
		if (lane == 0)
			emitted[best] = 1;
		__syncwarp();
	}
	if (lane == 0)
	{
		if (m.triangle_count)
			records[meshlet_offset++] = make_uint4(m.vertex_offset, m.triangle_offset, m.vertex_count, m.triangle_count);
		a.job_meshlets[j] = meshlet_offset;
	}
}

// One thread per meshlet: meshopt_optimizeMeshletLevel(level 1), then what appendMeshlet (scene.cpp:26-47) derives from
// the meshlet's vertices: minVertex, shortRefs and the words it takes.
__global__ void __launch_bounds__(128) cook_optimize_kernel(const CookArgs a)
{
	uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s >= a.slot_count)
		return;
	uint32_t j = scan::last_at_most(a.job_count, s, [&](uint32_t i) { return a.jobs[i].slot; });
	const cook::CookJob& job = a.jobs[j];
	if (s - job.slot >= a.job_meshlets[j])
	{
		a.slot_words[s] = 0;
		return;
	}
	uint4 r = a.ml_records[s];
	uint32_t* mv = a.ml_vertices + job.idx + r.x;
	cook::optimize_meshlet(mv, r.z, a.ml_triangles + job.idx + r.y, r.w);
	uint32_t lo = ~0u, hi = 0;
	for (uint32_t i = 0; i < r.z; ++i)
	{
		lo = mv[i] < lo ? mv[i] : lo;
		hi = mv[i] > hi ? mv[i] : hi;
	}
	bool short_refs = hi - lo < (1u << 16);
	a.slot_min[s] = lo;
	a.slot_words[s] = (short_refs ? (r.z + 1u) / 2u : r.z) + (r.w * 3u + 3u) / 4u;
}

// One block: LOD meshlet offsets (scene.cpp:274-275) and meshlet data offsets, both in job order; the totals and the
// overflow flag.
__global__ void __launch_bounds__(kCookScanThreads) cook_scan_kernel(const CookArgs a)
{
	__shared__ uint32_t s_warp[kCookScanThreads / 32];
	const uint64_t meshlets = scan::scan_tiles<kCookScanThreads>(
	    a.job_count, uint64_t(0), s_warp, [&](uint32_t j) { return a.job_meshlets[j]; },
	    [&](uint32_t j, uint64_t first) {
		    a.job_first[j] = uint32_t(first);
		    NvcMeshLod& lod = a.meshes[a.jobs[j].mesh].lods[a.jobs[j].lod];
		    lod.meshletOffset = uint32_t(first);
		    lod.meshletCount = a.job_meshlets[j];
	    });
	const uint64_t words = scan::scan_tiles<kCookScanThreads>(
	    a.slot_count, uint64_t(0), s_warp, [&](uint32_t s) { return a.slot_words[s]; }, [&](uint32_t s, uint64_t first) { a.slot_data[s] = uint32_t(first); });
	if (threadIdx.x == 0)
	{
		a.totals4[0] = meshlets > 0xffffffffull ? 0xffffffffu : uint32_t(meshlets);
		a.totals4[1] = words > 0xffffffffull ? 0xffffffffu : uint32_t(words);
		a.totals4[3] = (meshlets > a.meshlet_capacity || words > a.meshletdata_capacity) ? 1u : 0u;
	}
}

// One thread per meshlet: the Meshlet record and its meshletdata words (scene.cpp:26-80), then the bounds of
// meshopt_computeMeshletBounds from the words just written (cook::meshlet_bounds).  Nothing is written on overflow.
__global__ void __launch_bounds__(128) cook_pack_kernel(const CookArgs a)
{
	uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s >= a.slot_count || a.totals4[3])
		return;
	uint32_t j = scan::last_at_most(a.job_count, s, [&](uint32_t i) { return a.jobs[i].slot; });
	const cook::CookJob& job = a.jobs[j];
	uint32_t local = s - uint32_t(job.slot);
	if (local >= a.job_meshlets[j])
		return;
	uint4 r = a.ml_records[s];
	const uint32_t* mv = a.ml_vertices + job.idx + r.x;
	const uint8_t* mt = a.ml_triangles + job.idx + r.y;
	uint32_t lo = a.slot_min[s];
	uint32_t hi = 0;
	for (uint32_t i = 0; i < r.z; ++i)
		hi = mv[i] > hi ? mv[i] : hi;
	bool short_refs = hi - lo < (1u << 16);
	uint32_t* dst = a.meshletdata + a.slot_data[s];
	const uint32_t ref_words = mcodec::reference_words(r.z, short_refs);
	for (uint32_t k = 0; k < ref_words; ++k)
	{
		if (short_refs)
			dst[k] = (mv[2 * k] - lo) | (2 * k + 1 < r.z ? (mv[2 * k + 1] - lo) << 16 : 0u);
		else
			dst[k] = mv[k] - lo;
	}
	uint32_t tri_bytes = r.w * 3u;
	for (uint32_t wi = 0; wi < (tri_bytes + 3u) / 4u; ++wi)
	{
		uint32_t word = 0;
		for (uint32_t q = 0; q < 4; ++q)
			word |= (4 * wi + q < tri_bytes ? uint32_t(mt[4 * wi + q]) : 0u) << (8 * q);
		dst[ref_words + wi] = word;
	}
	NvcMeshlet m;
	memset(&m, 0, sizeof(m));
	m.dataOffset = a.slot_data[s];
	m.baseVertex = job.vertex_offset + lo;
	m.vertexCount = uint8_t(r.z);
	m.triangleCount = uint8_t(r.w);
	m.shortRefs = short_refs ? 1 : 0;
	cook::MeshletView view;
	view.vertices = a.vertices;
	view.data = dst;
	view.baseVertex = m.baseVertex;
	view.vertexCount = m.vertexCount;
	view.triangleCount = m.triangleCount;
	view.shortRefs = m.shortRefs;
	cook::meshlet_bounds(view, &m);
	a.meshlets[a.job_first[j] + local] = m;
}

// ---- clrt builds: meshopt_buildMeshletsSpatial for each mesh's lodRT (nvc_meshlets.cuh) ------------------------------------

constexpr uint32_t kSpatialWarps = 4;          // jobs per block of the spatial build kernel
constexpr uint32_t kSpatialStack = 64;         // pending bvhSplit nodes: at most depth + 2 <= kMaxTreeDepth + 2
constexpr uint32_t kRadixBuckets = 1024;       // the reference's 10-bit digits

// One LSD pass of the reference's radix sort (clusterizer.cpp:737-748): dst = src stably ordered by bits
// [shift, shift + 10) of radixFloat(key).  hist is the warp's 1024 buckets.
__device__ void spatial_radix_pass(uint32_t lane, uint32_t* dst, const uint32_t* src, const uint32_t* keys, uint32_t n, uint32_t shift, uint32_t* hist)
{
	const uint32_t full = 0xffffffffu;
	for (uint32_t b = lane; b < kRadixBuckets; b += 32)
		hist[b] = 0;
	__syncwarp();
	for (uint32_t i = lane; i < n; i += 32)
	{
		uint32_t u = keys[i];
		atomicAdd(hist + (((u ^ ((uint32_t(int(u) >> 31)) | 0x80000000u)) >> shift) & 1023u), 1u);
	}
	__syncwarp();
	// exclusive prefix: lane owns buckets [32 lane, 32 lane + 32)
	uint32_t sum = 0;
	for (uint32_t q = 0; q < 32; ++q)
		sum += hist[lane * 32 + q];
	uint32_t run = scan::warp_inclusive(sum, lane) - sum;
	for (uint32_t q = 0; q < 32; ++q)
	{
		uint32_t c = hist[lane * 32 + q];
		hist[lane * 32 + q] = run;
		run += c;
	}
	__syncwarp();
	// stable scatter, 32 elements at a time: rank among the earlier lanes of the same digit
	for (uint32_t base = 0; base < n; base += 32)
	{
		uint32_t i = base + lane;
		bool valid = i < n;
		uint32_t v = valid ? src[i] : 0u, d = kRadixBuckets + lane;
		if (valid)
		{
			uint32_t u = keys[v];
			d = ((u ^ ((uint32_t(int(u) >> 31)) | 0x80000000u)) >> shift) & 1023u;
		}
		uint32_t peers = __match_any_sync(full, d);
		uint32_t rank = __popc(peers & ((1u << lane) - 1u));
		if (valid)
			dst[hist[d] + rank] = v;
		__syncwarp();
		if (valid && (peers >> lane) == 1u) // the group's last lane moves the bucket on
			hist[d] += __popc(peers);
		__syncwarp();
	}
}

// Inclusive running boxMerge component over the warp's 32 elements after `carry`.  box op NaN = NaN and NaN op x = x, so a
// NaN element restarts the fold: the scan combines (value, restarted) pairs, which is associative.
template <bool kMax>
__device__ __forceinline__ float spatial_box_scan(float v, float carry, uint32_t lane)
{
	const uint32_t full = 0xffffffffu;
	uint32_t r = v != v;
	for (uint32_t d = 1; d < 32; d <<= 1)
	{
		float pv = __shfl_up_sync(full, v, d);
		uint32_t pr = __shfl_up_sync(full, r, d);
		if (lane >= d)
		{
			if (!r)
				v = kMax ? cook::box_max(pv, v) : cook::box_min(pv, v);
			r |= pr;
		}
	}
	if (!r)
		v = kMax ? cook::box_max(carry, v) : cook::box_min(carry, v);
	return v;
}

// bvhComputeArea (clusterizer.cpp:866-878): areas[i] = area of boxes order[0..i], areas[count + i] = of order[count-1-i..]
__device__ void spatial_areas(uint32_t lane, float* areas, const float* boxes, const uint32_t* order, uint32_t count)
{
	const uint32_t full = 0xffffffffu;
	float lc[6] = { FLT_MAX, FLT_MAX, FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX };
	float rc[6] = { FLT_MAX, FLT_MAX, FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX };
	for (uint32_t base = 0; base < count; base += 32)
	{
		uint32_t i = base + lane;
		bool valid = i < count;
		uint32_t last = (count - base < 32 ? count - base : 32) - 1;
		const float* lb = boxes + size_t(order[valid ? i : count - 1]) * 6u;
		const float* rb = boxes + size_t(order[valid ? count - 1 - i : 0]) * 6u;
		float l[6], r[6];
		for (int k = 0; k < 3; ++k)
		{
			l[k] = spatial_box_scan<false>(lb[k], lc[k], lane);
			l[k + 3] = spatial_box_scan<true>(lb[k + 3], lc[k + 3], lane);
			r[k] = spatial_box_scan<false>(rb[k], rc[k], lane);
			r[k + 3] = spatial_box_scan<true>(rb[k + 3], rc[k + 3], lane);
		}
		if (valid)
		{
			areas[i] = cook::box_area(l, l + 3);
			areas[i + count] = cook::box_area(r, r + 3);
		}
		for (int k = 0; k < 6; ++k)
		{
			lc[k] = __shfl_sync(full, l[k], last);
			rc[k] = __shfl_sync(full, r[k], last);
		}
	}
}

// bvhPivot by lanes.  bvhPivot keeps the first strict minimum of the full cost but skips candidates whose SAH part alone
// exceeds the best so far.  A skipped candidate with full >= sah (the fill term >= 0) or full = NaN could not have won,
// so where no candidate has full < sah the result is the first strict minimum of the full cost below FLT_MAX, reduced
// over lanes by (cost, i).  Otherwise lane 0 runs the reference's loop as written.  The fill term is negative only when the
// float round-up int(float(fill + maxfill - 1) * (1.f / maxfill)) truncates low, which it does not for any fill below 2^25 with
// maxfill 64 or 96 (checked exhaustively in float32), so the fallback only guards LODs of 2^25 triangles and more.
__device__ uint32_t spatial_pivot(uint32_t lane, const float* areas, const uint32_t* vertices, uint32_t count, uint32_t min, uint32_t maxfill, float& out_cost)
{
	const uint32_t full_mask = 0xffffffffu;
	bool aligned = cook::pivot_aligned(count, min);
	uint32_t end = cook::pivot_end(count, min);
	float rmaxfill = cook::div(1.0f, float(int(maxfill)));
	uint32_t bkey = 0xffffffffu, bi = 0xffffffffu, bbits = 0;
	bool skip_matters = false;
	for (uint32_t i = min - 1 + lane; i < end; i += 32)
	{
		float sah, full;
		if (!cook::pivot_cost(areas, vertices, count, i, min, aligned, maxfill, rmaxfill, sah, full))
			continue;
		skip_matters = skip_matters || full < sah;
		if (!(full < FLT_MAX))
			continue;
		uint32_t key = cook_score_key(full);
		if (key < bkey) // i increases within a lane: the first of equal costs is kept
		{
			bkey = key;
			bi = i;
			bbits = cook::float_bits(full);
		}
	}
	for (int d = 16; d > 0; d >>= 1)
	{
		uint32_t ok = __shfl_xor_sync(full_mask, bkey, d), oi = __shfl_xor_sync(full_mask, bi, d), ob = __shfl_xor_sync(full_mask, bbits, d);
		if (ok < bkey || (ok == bkey && oi < bi))
			bkey = ok, bi = oi, bbits = ob;
	}
	if (__any_sync(full_mask, skip_matters))
	{
		uint32_t split = 0;
		float cost = FLT_MAX;
		if (lane == 0)
			split = cook::bvh_pivot(areas, vertices, count, min, maxfill, cost);
		out_cost = __shfl_sync(full_mask, cost, 0);
		return __shfl_sync(full_mask, split, 0);
	}
	out_cost = bi == 0xffffffffu ? FLT_MAX : cook::bits_float(bbits);
	return bi == 0xffffffffu ? 0u : bi + 1;
}

// One warp per ray-tracing job: meshopt_buildMeshletsSpatial (clusterizer.cpp:1266-1365) with the parameters of
// scene.cpp:103.  Fills the same per-job outputs as cook_build_kernel (records in the job's slots, ml_vertices,
// ml_triangles, job_meshlets); the optimize, scan and pack kernels then treat both kinds of job alike.  Scratch of the job
// (sized for the greedy builder): cones = boxes (6 floats per triangle), kd_nodes = the three axis orders then the sort
// keys / areas, kd_index = sort and partition temp, emitted = sides, adj_data = boundary bytes.  bvhSplit's recursion
// is a depth-first stack of (start, count, depth); each node's work is spread over the lanes.
__global__ void __launch_bounds__(kSpatialWarps * 32) cook_spatial_kernel(const CookClrtArgs c)
{
	__shared__ uint32_t s_hist[kSpatialWarps][kRadixBuckets];
	const CookArgs& a = c.base;
	const uint32_t full = 0xffffffffu;
	const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
	const uint32_t w = blockIdx.x * kSpatialWarps + warp;
	if (w >= c.rt_count)
		return;
	const uint32_t j = a.order[c.greedy_count + w];
	const cook::CookJob job = a.jobs[j];
	const uint32_t* indices = a.indices + job.index_offset;
	const uint32_t index_count = job.index_count, n = index_count / 3, vertex_count = job.vertex_count;

	bool bad = false;
	for (uint32_t i = lane; i < index_count; i += 32)
		bad = bad || indices[i] >= vertex_count;
	if (__any_sync(full, bad) || n == 0)
	{
		if (lane == 0)
		{
			a.job_meshlets[j] = 0;
			if (n != 0)
				atomicAdd(a.totals4 + 2, 1u);
		}
		return;
	}

	float* boxes = a.cones + job.tri * 6u;
	uint32_t* axes = a.kd_nodes + job.tri * 6u;
	uint32_t* keys = axes + 3u * n;
	float* areas = reinterpret_cast<float*>(keys);
	uint32_t* temp = a.kd_index + job.tri;
	uint8_t* sides = a.emitted + job.tri;
	uint8_t* boundary = reinterpret_cast<uint8_t*>(a.adj_data + job.idx);
	int16_t* used = a.used + job.vtx;
	uint32_t* mlv = a.ml_vertices + job.idx;
	uint8_t* mlt = a.ml_triangles + job.idx;
	uint4* records = a.ml_records + job.slot;
	const NvcVertex* verts = a.vertices + job.vertex_offset;

	// bvhPrepare (clusterizer.cpp:750-775)
	for (uint32_t t = lane; t < n; t += 32)
	{
		float p[3][3];
		for (int q = 0; q < 3; ++q)
		{
			const NvcVertex& v = verts[indices[t * 3 + q]];
			p[q][0] = cook::dequantize_half(v.vx);
			p[q][1] = cook::dequantize_half(v.vy);
			p[q][2] = cook::dequantize_half(v.vz);
		}
		for (int k = 0; k < 3; ++k)
		{
			float mn = p[0][k] < p[1][k] ? p[0][k] : p[1][k];
			mn = p[2][k] < mn ? p[2][k] : mn;
			float mx = p[0][k] > p[1][k] ? p[0][k] : p[1][k];
			mx = p[2][k] > mx ? p[2][k] : mx;
			boxes[size_t(t) * 6u + k] = mn;
			boxes[size_t(t) * 6u + 3 + k] = mx;
			keys[k * n + t] = cook::float_bits(cook::centroid(mn, mx));
		}
	}
	for (uint32_t v = lane; v < vertex_count; v += 32)
		used[v] = -1;
	__syncwarp();

	// the three radix sorts (clusterizer.cpp:1300-1314), from identity order
	for (int k = 0; k < 3; ++k)
	{
		uint32_t* order = axes + k * n;
		for (uint32_t i = lane; i < n; i += 32)
			temp[i] = i;
		__syncwarp();
		spatial_radix_pass(lane, order, temp, keys + k * n, n, 2, s_hist[warp]);
		spatial_radix_pass(lane, temp, order, keys + k * n, n, 12, s_hist[warp]);
		spatial_radix_pass(lane, order, temp, keys + k * n, n, 22, s_hist[warp]);
	}
	__syncwarp();

	// bvhSplit (clusterizer.cpp:942-1012)
	uint32_t st_start[kSpatialStack], st_count[kSpatialStack];
	int st_depth[kSpatialStack];
	int sp = 0;
	st_start[0] = 0, st_count[0] = n, st_depth[0] = 0, sp = 1;
	while (sp > 0)
	{
		--sp;
		const uint32_t start = st_start[sp], count = st_count[sp];
		const int depth = st_depth[sp];
		uint8_t* bnd = boundary + start;
		if (count <= cook::kMaxTriangles)
		{
			uint32_t nv = 0;
			if (lane == 0)
				nv = cook::bvh_count_vertices(axes + start, count, used, indices, nullptr);
			nv = __shfl_sync(full, nv, 0);
			if (nv <= cook::kMaxVertices)
			{
				for (uint32_t i = lane; i < count; i += 32)
					bnd[i] = i == 0;
				__syncwarp();
				continue;
			}
		}
		// a node of <= 96 triangles that did not pack is vertex bound
		const uint32_t mint = count <= cook::kMaxTriangles ? cook::kSpatialLeafSplit : cook::kSpatialMinTriangles;
		const uint32_t maxfill = count <= cook::kMaxTriangles ? cook::kMaxVertices : cook::kMaxTriangles;
		int bestk = -1;
		uint32_t bestsplit = 0;
		float bestcost = FLT_MAX;
		for (int k = 0; k < 3; ++k)
		{
			const uint32_t* order = axes + k * n + start;
			spatial_areas(lane, areas, boxes, order, count);
			uint32_t* vertices = nullptr;
			if (count <= cook::kMaxTriangles)
			{
				vertices = reinterpret_cast<uint32_t*>(areas + 2 * count);
				if (lane == 0)
					cook::bvh_count_vertices(order, count, used, indices, vertices);
			}
			__syncwarp();
			float axiscost = FLT_MAX;
			uint32_t axissplit = spatial_pivot(lane, areas, vertices, count, mint, maxfill, axiscost);
			if (axissplit && axiscost < bestcost)
			{
				bestk = k;
				bestcost = axiscost;
				bestsplit = axissplit;
			}
			__syncwarp();
		}
		if (bestk < 0 || depth >= cook::kMaxTreeDepth)
		{
			if (lane == 0)
				cook::bvh_pack_tail(bnd, axes + start, count, used, indices);
			__syncwarp();
			continue;
		}
		const uint32_t* best = axes + bestk * n + start;
		for (uint32_t i = lane; i < count; i += 32)
			sides[best[i]] = i >= bestsplit;
		__syncwarp();
		// bvhPartition of the two other axes (clusterizer.cpp:928-940), stable, 32 elements at a time
		for (int k = 0; k < 3; ++k)
		{
			if (k == bestk)
				continue;
			uint32_t* axis = axes + k * n + start;
			for (uint32_t i = lane; i < count; i += 32)
				temp[i] = axis[i];
			__syncwarp();
			uint32_t l = 0, r = bestsplit;
			for (uint32_t base = 0; base < count; base += 32)
			{
				uint32_t i = base + lane;
				bool valid = i < count;
				uint32_t v = valid ? temp[i] : 0u;
				bool side = valid && sides[v];
				uint32_t lm = __ballot_sync(full, valid && !side), rm = __ballot_sync(full, side);
				uint32_t below = (1u << lane) - 1u;
				if (valid)
					axis[side ? r + __popc(rm & below) : l + __popc(lm & below)] = v;
				l += __popc(lm);
				r += __popc(rm);
			}
			__syncwarp();
		}
		st_start[sp] = start + bestsplit, st_count[sp] = count - bestsplit, st_depth[sp] = depth + 1, ++sp;
		st_start[sp] = start, st_count[sp] = bestsplit, st_depth[sp] = depth + 1, ++sp;
	}

	// the packing loop (clusterizer.cpp:1326-1358), sequential: boundaries, the over-bound rule and appendMeshlet's own splits
	uint32_t marks = 0;
	for (uint32_t i = lane; i < n; i += 32)
		marks += boundary[i];
	const uint32_t meshlet_count = __shfl_sync(full, scan::warp_inclusive(marks, lane), 31);
	if (lane == 0)
	{
		const uint64_t meshlet_bound = cook::spatial_meshlets_bound(index_count);
		cook::Building m = { 0, 0, 0, 0 };
		uint64_t meshlet_offset = 0, meshlet_pending = meshlet_count;
		bool over = false;
		for (uint32_t i = 0; i < n; ++i)
		{
			bool split = i > 0 && boundary[i] == 1;
			if (split && meshlet_count > meshlet_bound && meshlet_offset + meshlet_pending >= meshlet_bound)
				split = false;
			// the reference asserts meshlet_offset <= meshlet_bound; the job's slots end there
			if (meshlet_offset >= meshlet_bound)
			{
				over = true;
				break;
			}
			// appendMeshlet(..., split): a split flushes first, and the emptied meshlet then takes the triangle without a flush
			uint32_t index = axes[i];
			if (split)
				cook::flush_meshlet(m, used, records, uint32_t(meshlet_offset), mlv);
			bool flushed = cook::append_triangle(m, indices[index * 3 + 0], indices[index * 3 + 1], indices[index * 3 + 2], used, records, uint32_t(meshlet_offset), mlv, mlt);
			meshlet_offset += (split || flushed) ? 1u : 0u;
			meshlet_pending -= boundary[i];
		}
		if (!over && m.triangle_count)
		{
			if (meshlet_offset >= meshlet_bound)
				over = true;
			else
				records[meshlet_offset++] = make_uint4(m.vertex_offset, m.triangle_offset, m.vertex_count, m.triangle_count);
		}
		a.job_meshlets[j] = over ? 0u : uint32_t(meshlet_offset);
		if (over)
			atomicAdd(a.totals4 + 2, 1u);
	}
}

// meshletvtx0 offsets (scene.cpp:52-67): 4 elements per vertex of every meshlet of a ray-tracing job, in slot order (= job,
// then meshlet order); totals8[4] and the overflow flag.  Runs after cook_scan_kernel, before the pack kernels.
__global__ void __launch_bounds__(kCookScanThreads) cook_vtx0_scan_kernel(const CookClrtArgs c)
{
	__shared__ uint32_t s_warp[kCookScanThreads / 32];
	const CookArgs& a = c.base;
	auto elements = [&](uint32_t s) {
		const uint32_t j = scan::last_at_most(a.job_count, s, [&](uint32_t i) { return a.jobs[i].slot; });
		return c.job_rt[j] && s - uint32_t(a.jobs[j].slot) < a.job_meshlets[j] ? 4u * a.ml_records[s].z : 0u;
	};
	const uint64_t carry = scan::scan_tiles<kCookScanThreads>(a.slot_count, uint64_t(0), s_warp, elements, [&](uint32_t s, uint64_t first) { c.slot_vtx0[s] = uint32_t(first); });
	if (threadIdx.x == 0)
	{
		a.totals4[4] = carry > 0xffffffffull ? 0xffffffffu : uint32_t(carry);
		if (carry > c.meshletvtx0_capacity)
			a.totals4[3] = 1u;
	}
}

// One thread per ray-tracing meshlet: quantizeHalf of its positions (the dequantized fp16 of Vertex, so NaN becomes
// 0x7e00 and denormals flush to 0) in the optimized vertex order, then 0.  Nothing is written on overflow.
__global__ void __launch_bounds__(128) cook_vtx0_pack_kernel(const CookClrtArgs c)
{
	const CookArgs& a = c.base;
	uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s >= a.slot_count || a.totals4[3])
		return;
	uint32_t j = scan::last_at_most(a.job_count, s, [&](uint32_t i) { return a.jobs[i].slot; });
	const cook::CookJob& job = a.jobs[j];
	if (!c.job_rt[j] || s - uint32_t(job.slot) >= a.job_meshlets[j])
		return;
	uint4 r = a.ml_records[s];
	const uint32_t* mv = a.ml_vertices + job.idx + r.x;
	uint16_t* dst = c.meshletvtx0 + c.slot_vtx0[s];
	for (uint32_t i = 0; i < r.z; ++i)
	{
		const NvcVertex& v = a.vertices[job.vertex_offset + mv[i]];
		dst[4 * i + 0] = cook::quantize_half(cook::dequantize_half(v.vx));
		dst[4 * i + 1] = cook::quantize_half(cook::dequantize_half(v.vy));
		dst[4 * i + 2] = cook::quantize_half(cook::dequantize_half(v.vz));
		dst[4 * i + 3] = 0;
	}
}

} // namespace

cudaError_t launch_cook_meshlets_clrt(const CookClrtArgs& c, cudaStream_t stream)
{
	const CookArgs& a = c.base;
	cudaError_t e = cudaMemsetAsync(a.totals4, 0, 32, stream);
	if (e != cudaSuccess)
		return e;
	if (c.greedy_count)
	{
		CookArgs g = a;
		g.job_count = c.greedy_count; // the build kernel takes order[0, job_count)
		cook_build_kernel<<<(c.greedy_count + kCookWarps - 1) / kCookWarps, kCookWarps * 32, 0, stream>>>(g);
	}
	if (c.rt_count)
		cook_spatial_kernel<<<(c.rt_count + kSpatialWarps - 1) / kSpatialWarps, kSpatialWarps * 32, 0, stream>>>(c);
	if (a.slot_count)
		cook_optimize_kernel<<<(a.slot_count + 127u) / 128u, 128, 0, stream>>>(a);
	cook_scan_kernel<<<1, kCookScanThreads, 0, stream>>>(a);
	cook_vtx0_scan_kernel<<<1, kCookScanThreads, 0, stream>>>(c);
	if (a.slot_count)
	{
		cook_pack_kernel<<<(a.slot_count + 127u) / 128u, 128, 0, stream>>>(a);
		cook_vtx0_pack_kernel<<<(a.slot_count + 127u) / 128u, 128, 0, stream>>>(c);
	}
	return cudaGetLastError();
}

cudaError_t launch_cook_meshlets(const CookArgs& a, cudaStream_t stream)
{
	cudaError_t e = cudaMemsetAsync(a.totals4, 0, 16, stream);
	if (e != cudaSuccess)
		return e;
	if (a.job_count)
		cook_build_kernel<<<(a.job_count + kCookWarps - 1) / kCookWarps, kCookWarps * 32, 0, stream>>>(a);
	if (a.slot_count)
		cook_optimize_kernel<<<(a.slot_count + 127u) / 128u, 128, 0, stream>>>(a);
	cook_scan_kernel<<<1, kCookScanThreads, 0, stream>>>(a);
	if (a.slot_count)
		cook_pack_kernel<<<(a.slot_count + 127u) / 128u, 128, 0, stream>>>(a);
	return cudaGetLastError();
}

// ---- nvc_cook_mesh_lods: appendMesh's LOD chain (nvc_lods.cuh) ------------------------------------------------------------
// One single-thread CTA per mesh, largest LOD 0 first: the chain's stages are sequential (each LOD starts from the last one).
// Writes the Mesh record with chain-relative index offsets and the chain into the mesh's scratch.
__global__ void __launch_bounds__(1) lods_chain_kernel(const LodArgs a)
{
	const uint32_t m = a.order[blockIdx.x];
	NvcMesh mesh;
	bool rejected;
	a.chain[m] = lods::cook_chain(a.jobs[m], a.vertices, a.lod0_indices + a.jobs[m].index_offset, a.max_scale[m], a.scratch, mesh, rejected);
	a.rejected[m] = rejected;
	a.meshes[m] = mesh;
}

// Places the chains in mesh order (the reference's ib layout): offsets, totals, overflow flag.  One thread; a mesh is a
// few additions.
__global__ void __launch_bounds__(1) lods_scan_kernel(const LodArgs a)
{
	uint64_t base = 0;
	uint32_t rejected = 0;
	for (uint32_t m = 0; m < a.mesh_count; ++m)
	{
		a.base[m] = base;
		rejected += a.rejected[m];
		NvcMesh& mesh = a.meshes[m];
		for (uint32_t l = 0; l < mesh.lodCount; ++l)
			mesh.lods[l].indexOffset = uint32_t(base + mesh.lods[l].indexOffset);
		base += a.chain[m];
	}
	a.totals4[0] = base > 0xffffffffull ? 0xffffffffu : uint32_t(base);
	a.totals4[1] = rejected;
	a.totals4[2] = base > a.index_capacity;
	a.totals4[3] = 0;
}

// Copies each chain to its place, one CTA per mesh; nothing when the chains overflow the capacity
__global__ void __launch_bounds__(256) lods_copy_kernel(const LodArgs a)
{
	if (a.totals4[2])
		return;
	const uint32_t m = blockIdx.x;
	const uint32_t* src = a.scratch + a.jobs[m].scratch;
	uint32_t* dst = a.indices + a.base[m];
	for (uint64_t i = threadIdx.x; i < a.chain[m]; i += blockDim.x)
		dst[i] = src[i];
}

cudaError_t launch_cook_mesh_lods(const LodArgs& a, cudaStream_t stream)
{
	if (a.mesh_count)
		lods_chain_kernel<<<a.mesh_count, 1, 0, stream>>>(a);
	lods_scan_kernel<<<1, 1, 0, stream>>>(a);
	if (a.mesh_count)
		lods_copy_kernel<<<a.mesh_count, 256, 0, stream>>>(a);
	return cudaGetLastError();
}

// ---- the device-wide scan (nvc_scan.cuh) ----------------------------------------------------------------------------------
// The exclusive scans of `rows` rows of n values each: row r of `out` is n + 1 long and ends with the row's total.
// block_sums and block_offsets hold rows x ceil(n / scan::kScanItems) and rows x (that + 1) words.
template <typename In, typename Out>
static cudaError_t launch_scan(const In* in, uint64_t n, uint32_t rows, uint32_t* block_sums, unsigned long long* block_offsets, Out* out, cudaStream_t stream)
{
	using namespace scan;
	if (n == 0)
		return cudaMemsetAsync(out, 0, rows * sizeof(Out), stream); // the totals
	const uint32_t blocks = uint32_t((n + scan::kScanItems - 1) / scan::kScanItems);
	reduce_kernel<In><<<dim3(blocks, rows), scan::kThreads, 0, stream>>>(in, n, block_sums);
	offsets_kernel<<<rows, scan::kOffsetsThreads, 0, stream>>>(block_sums, blocks, block_offsets);
	apply_kernel<In, Out><<<dim3(blocks, rows), scan::kThreads, 0, stream>>>(in, n, block_offsets, out);
	return cudaSuccess;
}

// ---- nvc_cook_mesh_vertices: appendMesh's vertex processing (nvc_vertices.cuh) ---------------------------------------------
uint64_t vertex_cache_words(uint32_t vertices, uint32_t indices)
{
	return verts::carve(vertices, indices, nullptr, nullptr);
}

cudaError_t launch_cook_mesh_vertices(const VertexArgs& a, cudaStream_t stream)
{
	using namespace verts;
	const uint32_t T = a.tri_count, N = a.position_count, S = a.slot_count, M = a.mesh_count;
	auto grid = [](uint32_t n) { return (n + verts::kThreads - 1) / verts::kThreads; };
	cudaError_t e = cudaSuccess;
	auto fill = [&](void* p, int value, size_t bytes) {
		if (e == cudaSuccess && bytes)
			e = cudaMemsetAsync(p, value, bytes, stream);
	};
	auto scan_flags = [&](uint32_t n) {
		if (e == cudaSuccess)
			e = launch_scan(a.flags, n, 1, a.block_sums, a.offsets, a.rank, stream);
	};
	fill(a.totals4, 0, 16);
	fill(a.rejected, 0, M);
	fill(a.tri_table, 0xff, (size_t(a.tri_mask) + 1) * 4);
	fill(a.vtx_table, 0xff, (size_t(a.vtx_mask) + 1) * 4);
	fill(a.vtx_first, 0xff, (size_t(a.vtx_mask) + 1) * 4);
	fill(a.first, 0xff, size_t(S) * 4);
	fill(a.first_use, 0xff, size_t(S) * 4);
	if (e != cudaSuccess)
		return e;
	// filter: rejection, then one thread per triangle, then the kept triangles compacted
	if (T)
	{
		verts_reject_kernel<<<grid(T), verts::kThreads, 0, stream>>>(a);
		verts_filter_insert_kernel<<<grid(T), verts::kThreads, 0, stream>>>(a);
		verts_filter_flag_kernel<<<grid(T), verts::kThreads, 0, stream>>>(a);
	}
	scan_flags(T);
	if (T)
		verts_filter_compact_kernel<<<grid(T), verts::kThreads, 0, stream>>>(a);
	if (M)
		verts_index_base_kernel<<<grid(M), verts::kThreads, 0, stream>>>(a);
	// remap: first references, classes, their ranks over the filtered positions
	fill(a.flags, 0, N);
	if (N)
		verts_first_kernel<<<grid(N), verts::kThreads, 0, stream>>>(a);
	if (S)
	{
		verts_class_insert_kernel<<<grid(S), verts::kThreads, 0, stream>>>(a);
		verts_class_flag_kernel<<<grid(S), verts::kThreads, 0, stream>>>(a);
	}
	scan_flags(N);
	if (M)
		verts_mesh_kernel<<<grid(M), verts::kThreads, 0, stream>>>(a);
	if (S)
		verts_class_scatter_kernel<<<grid(S), verts::kThreads, 0, stream>>>(a);
	if (N)
		verts_remap_kernel<<<grid(N), verts::kThreads, 0, stream>>>(a);
	// vertex cache, one mesh per single-thread CTA
	if (M)
		verts_vcache_kernel<<<M, 1, 0, stream>>>(a);
	// fetch order
	fill(a.flags, 0, N);
	if (e != cudaSuccess)
		return e;
	if (N)
		verts_fetch_first_kernel<<<grid(N), verts::kThreads, 0, stream>>>(a);
	if (S)
		verts_fetch_flag_kernel<<<grid(S), verts::kThreads, 0, stream>>>(a);
	scan_flags(N);
	if (S)
		verts_fetch_scatter_kernel<<<grid(S), verts::kThreads, 0, stream>>>(a);
	if (N)
		verts_fetch_index_kernel<<<grid(N), verts::kThreads, 0, stream>>>(a);
	return e != cudaSuccess ? e : cudaGetLastError();
}

// ---- nvc_obj_load: loadObj over fast_obj (nvc_obj.cuh) -----------------------------------------------------------------------
static uint32_t obj_grid(uint64_t n)
{
	return uint32_t((n + obj::kThreads - 1) / obj::kThreads);
}

cudaError_t launch_obj_lines(const ObjArgs& a, cudaStream_t stream)
{
	using namespace obj;
	if (a.tile_count)
		obj_tile_count_kernel<<<a.tile_count, obj::kThreads, 0, stream>>>(a);
	void (*offsets)(const uint32_t*, uint32_t, unsigned long long*) = scan::offsets_kernel;
	offsets<<<1, scan::kOffsetsThreads, 0, stream>>>(a.tile_lines, a.tile_count, a.tile_offsets);
	return cudaGetLastError();
}

cudaError_t launch_obj_count(const ObjArgs& a, cudaStream_t stream)
{
	using namespace obj;
	cudaError_t e = cudaMemsetAsync(a.state, 0xff, size_t(a.file_count) * sizeof(FileState), stream);
	if (e != cudaSuccess)
		return e;
	if (a.tile_count)
	{
		obj_line_end_kernel<<<a.tile_count, obj::kThreads, 0, stream>>>(a);
		obj_cut_kernel<<<obj_grid(a.tile_count), obj::kThreads, 0, stream>>>(a);
	}
	obj_file_kernel<<<obj_grid(a.file_count), obj::kThreads, 0, stream>>>(a);
	obj_classify_kernel<<<obj_grid(a.line_slots), obj::kThreads, 0, stream>>>(a);
	e = launch_scan(a.counts, a.line_slots, kFields, a.block_sums, a.block_offsets, a.prefix, stream);
	if (e != cudaSuccess)
		return e;
	obj_info_kernel<<<obj_grid(a.file_count), obj::kThreads, 0, stream>>>(a);
	return cudaGetLastError();
}

cudaError_t launch_obj_parse(const ObjArgs& a, cudaStream_t stream)
{
	using namespace obj;
	obj_dummy_kernel<<<obj_grid(a.file_count), obj::kThreads, 0, stream>>>(a);
	obj_parse_kernel<<<obj_grid(a.line_slots), obj::kThreads, 0, stream>>>(a);
	if (a.face_count)
		obj_check_kernel<<<obj_grid(a.face_count), obj::kThreads, 0, stream>>>(a);
	return cudaGetLastError();
}

cudaError_t launch_obj_expand(const ObjArgs& a, cudaStream_t stream)
{
	using namespace obj;
	if (a.corner_count)
		obj_expand_kernel<<<obj_grid(a.corner_count), obj::kThreads, 0, stream>>>(a);
	return cudaGetLastError();
}

// N3: draws[update_indices[i]] = update_values[i]; one thread per 16-byte third of a 48-byte MeshDraw
__global__ void update_draws_kernel(NvcMeshDraw* __restrict__ draws, uint32_t draw_count, const uint32_t* __restrict__ update_indices,
    const NvcMeshDraw* __restrict__ update_values, uint32_t count)
{
	uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	uint32_t i = t / 3u, part = t - i * 3u;
	if (i >= count)
		return;
	uint32_t di = __ldg(update_indices + i);
	if (di >= draw_count)
		return;
	reinterpret_cast<uint4*>(draws)[size_t(di) * 3u + part] = __ldg(reinterpret_cast<const uint4*>(update_values) + size_t(i) * 3u + part);
}

cudaError_t launch_update_draws(NvcMeshDraw* draws, uint32_t draw_count, const uint32_t* update_indices, const NvcMeshDraw* update_values, uint32_t count, cudaStream_t stream)
{
	if (count == 0)
		return cudaSuccess;
	uint64_t threads = uint64_t(count) * 3u;
	update_draws_kernel<<<uint32_t((threads + 255u) / 256u), 256, 0, stream>>>(draws, draw_count, update_indices, update_values, count);
	return cudaGetLastError();
}

// Diagnostics: the filter's approximate reciprocal (op 0) or square root (op 1) of every input bit pattern
__global__ void filter_approx_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, uint64_t n, int op)
{
	const uint64_t i = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
	if (i >= n)
		return;
	const float x = __uint_as_float(__ldg(in + i));
	out[i] = __float_as_uint(op == 0 ? nvf_rcp(x) : nvf_sqrt(x));
}

cudaError_t launch_filter_approx(const uint32_t* in, uint32_t* out, uint64_t n, int op, cudaStream_t stream)
{
	if (n == 0)
		return cudaSuccess;
	filter_approx_kernel<<<uint32_t((n + 255u) / 256u), 256, 0, stream>>>(in, out, n, op);
	return cudaGetLastError();
}

__global__ void pack_meshes_kernel(const NvcMesh* __restrict__ meshes, uint32_t count, MeshCullHead* __restrict__ heads, float* __restrict__ errors)
{
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count)
		return;
	const NvcMesh& m = meshes[i];
	MeshCullHead h;
	h.center[0] = m.center[0], h.center[1] = m.center[1], h.center[2] = m.center[2];
	h.radius = m.radius;
	h.lodCount = m.lodCount;
	h.lod0MeshletOffset = m.lods[0].meshletOffset;
	h.lod0MeshletCount = m.lods[0].meshletCount;
	h.vertexOffset = m.vertexOffset;
	heads[i] = h;
	for (uint32_t l = 0; l < NVC_MAX_LODS; ++l)
		errors[size_t(i) * NVC_MAX_LODS + l] = m.lods[l].error;
}

cudaError_t launch_pack_meshes(const NvcMesh* meshes, uint32_t count, MeshCullHead* heads, float* errors, cudaStream_t stream)
{
	if (count == 0)
		return cudaSuccess;
	pack_meshes_kernel<<<(count + 255) / 256, 256, 0, stream>>>(meshes, count, heads, errors);
	return cudaGetLastError();
}

// the meshlet cull view (nvc_prepare_meshlets): bytes 0-7 and 8-11 of every 24-byte record, copied unchanged
__global__ void pack_meshlets_kernel(const NvcMeshlet* __restrict__ meshlets, uint32_t count, uint2* __restrict__ sphere, uint32_t* __restrict__ cone)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= count)
		return;
	const char* mp = reinterpret_cast<const char*>(meshlets + i);
	sphere[i] = *reinterpret_cast<const uint2*>(mp);
	cone[i] = *reinterpret_cast<const uint32_t*>(mp + 8);
}

cudaError_t launch_pack_meshlets(const NvcMeshlet* meshlets, uint32_t count, uint2* sphere, uint32_t* cone, cudaStream_t stream)
{
	if (count == 0)
		return cudaSuccess;
	pack_meshlets_kernel<<<(count + 255) / 256, 256, 0, stream>>>(meshlets, count, sphere, cone);
	return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------------
// footprint image: F_l(i, j) = min over the clamped 2 x 2 footprint (i, i+1) x (j, j+1) of mip l, i in [-1, w-1]
// (see HiZDesc).  With it a sampler access whose four texels all count (fract != 0 on both axes — the only case the
// filter decides) is ONE load instead of four scattered ones.
// A CTA owns kFpRows consecutive rows of one level's image and walks them in x: per column it reads the two texels of
// kFpRows + 1 pyramid rows (written by the previous launch, served by L2 / L1), takes the horizontal minima once and
// combines vertically adjacent ones — 10 loads and ~50 instructions for 4 entries.  (The first version, one thread
// per entry with a level search and an integer division, was instruction bound.)
// ------------------------------------------------------------------------------------------------------
constexpr uint32_t kFpRows = 4;

__host__ __device__ __forceinline__ uint32_t footprint_row_groups(uint32_t h)
{
	return (h + 1u + kFpRows - 1u) / kFpRows;
}

// A CTA owns kFpRows consecutive rows of one level's image; a thread produces 4 x kFpRows entries: per pyramid row one
// 16-byte load (texels ix0 .. ix0+3) and one 4-byte load (texel ix0-1), the four horizontal minima, then the vertical
// combination of adjacent rows and one 16-byte store per image row — 10 loads and ~70 instructions for 16 entries.
// (Versions before: one thread per entry with a level search and an integer division; one thread per column with two scalar
// loads per row.  Both were instruction bound.)
__global__ void __launch_bounds__(256) footprint_kernel(const HiZDesc hz, float* __restrict__ fp, uint32_t total)
{
	(void)total;
	// block -> (level, row group): uniform walk over <= 16 levels
	uint32_t l = hz.fp_first, rg = blockIdx.x;
	for (;;)
	{
		const uint32_t n = footprint_row_groups(max(1u, hz.height >> l));
		if (rg < n || l + 1u >= hz.levels)
			break;
		rg -= n;
		++l;
	}
	const uint32_t w = max(1u, hz.width >> l), h = max(1u, hz.height >> l);
	const uint32_t pitch = fp_pitch(w);
	const uint32_t iy0 = rg * kFpRows;
	if (iy0 > h)
		return;
	const float* __restrict__ t = hz.texels + hz.level_offset[l];
	float* __restrict__ out = fp + hz.fp_offset[l] + iy0 * pitch;
	// pyramid rows clamp(iy0 - 1 + k, 0, h - 1), k = 0..kFpRows
	uint32_t rowoff[kFpRows + 1];
#pragma unroll
	for (uint32_t k = 0; k <= kFpRows; ++k)
	{
		const uint32_t iy = iy0 + k; // row iy - 1, clamped
		rowoff[k] = min(iy ? iy - 1u : 0u, h - 1u) * w;
	}
	// rows of the level start 16-byte aligned when w is a multiple of 4 and the level's base is (packed power-of-two pyramids)
	const bool vec = (w & 3u) == 0 && ((reinterpret_cast<uintptr_t>(t) | reinterpret_cast<uintptr_t>(fp)) & 15u) == 0 && (hz.fp_offset[l] & 3u) == 0;
	if (vec)
	{
		for (uint32_t ix0 = threadIdx.x * 4u; ix0 < pitch; ix0 += 1024u)
		{
			// entries ix0 .. ix0+3 use texels ix0-1 .. ix0+3 (clamped to [0, w-1]); ix0 == w: only entry w exists (texel w-1 twice)
			float4 m[kFpRows + 1];
#pragma unroll
			for (uint32_t k = 0; k <= kFpRows; ++k)
			{
				const float* row = t + rowoff[k];
				const float left = __ldg(row + (ix0 ? ix0 - 1u : 0u));
				float4 b = make_float4(left, left, left, left);
				if (ix0 < w)
					b = __ldg(reinterpret_cast<const float4*>(row + ix0));
				m[k] = make_float4(fminf(left, b.x), fminf(b.x, b.y), fminf(b.y, b.z), fminf(b.z, b.w));
			}
#pragma unroll
			for (uint32_t k = 0; k < kFpRows; ++k)
				if (iy0 + k <= h)
					*reinterpret_cast<float4*>(out + k * pitch + ix0) = make_float4(fminf(m[k].x, m[k + 1].x), fminf(m[k].y, m[k + 1].y), fminf(m[k].z, m[k + 1].z), fminf(m[k].w, m[k + 1].w));
		}
		return;
	}
	for (uint32_t ix = threadIdx.x; ix <= w; ix += 256u)
	{
		const uint32_t x0 = ix ? ix - 1u : 0u, x1 = min(ix, w - 1u);
		float m[kFpRows + 1];
#pragma unroll
		for (uint32_t k = 0; k <= kFpRows; ++k)
			m[k] = fminf(__ldg(t + rowoff[k] + x0), __ldg(t + rowoff[k] + x1));
#pragma unroll
		for (uint32_t k = 0; k < kFpRows; ++k)
			if (iy0 + k <= h)
				out[k * pitch + ix] = fminf(m[k], m[k + 1]);
	}
}

cudaError_t launch_footprint(const HiZDesc& hiz, float* fp, uint32_t total, cudaStream_t stream)
{
	if (total == 0)
		return cudaSuccess;
	uint32_t blocks = 0;
	for (uint32_t l = hiz.fp_first; l < hiz.levels; ++l)
		blocks += footprint_row_groups(hiz.height >> l ? hiz.height >> l : 1u);
	footprint_kernel<<<blocks, 256, 0, stream>>>(hiz, fp, total);
	return cudaGetLastError();
}

cudaError_t launch_drawcull(const DrawCullParams& p, bool late, bool task, cudaStream_t stream)
{
	uint32_t blocks = (p.cull.drawCount + kDrawBlock * kDPT - 1) / (kDrawBlock * kDPT);
	if (blocks == 0)
		blocks = 1;
	void (*kernel)(DrawCullParams) = late ? (task ? drawcull_kernel<true, true> : drawcull_kernel<true, false>) : (task ? drawcull_kernel<false, true> : drawcull_kernel<false, false>);
	kernel<<<blocks, kDrawBlock, 0, stream>>>(p);
	return cudaGetLastError();
}

uint32_t hiz_stage_bytes(const HiZDesc& hiz)
{
	return hiz.stage_level < hiz.levels ? ((hiz.stage_texels * 4u + 15u) & ~15u) : 0u;
}

// the main passes of a frame (TRACK) are specialised on the backface flag too; everything else reads its flags at run time
template <bool LATE, bool FP, bool TASKOUT>
static void (*pick_filter_kernel(bool track, bool bf))(ClusterParams)
{
	if (!track)
		return clustercull_filter_kernel<LATE, FP, false, TASKOUT, -1>;
	return bf ? clustercull_filter_kernel<LATE, FP, true, TASKOUT, 1> : clustercull_filter_kernel<LATE, FP, true, TASKOUT, 0>;
}

cudaError_t launch_clustercull(const ClusterParams& p, bool late, uint32_t blocks, cudaStream_t stream)
{
	if (p.use_filter)
	{
		const bool track = p.cull.clusterOcclusionEnabled == 1 && p.cull.postPass == 0;
		const bool taskout = p.payloads != nullptr;
		const bool bf = p.cull.clusterBackfaceEnabled != 0;
		void (*kernel)(ClusterParams);
		if (taskout)
			kernel = late ? (p.hiz.fp ? pick_filter_kernel<true, true, true>(track, bf) : pick_filter_kernel<true, false, true>(track, bf)) : pick_filter_kernel<false, false, true>(track, bf);
		else
			kernel = late ? (p.hiz.fp ? pick_filter_kernel<true, true, false>(track, bf) : pick_filter_kernel<true, false, false>(track, bf)) : pick_filter_kernel<false, false, false>(track, bf);
		kernel<<<blocks, kClusterBlock, 0, stream>>>(p);
		return cudaGetLastError();
	}
	const uint32_t stage_bytes = late ? hiz_stage_bytes(p.hiz) : 0u;
	void (*kernel)(ClusterParams) = late ? (stage_bytes ? clustercull_kernel<true, true> : clustercull_kernel<true, false>) : clustercull_kernel<false, false>;
	kernel<<<blocks, kClusterBlock, stage_bytes, stream>>>(p);
	return cudaGetLastError();
}

cudaError_t launch_taskcull(const ClusterParams& p, bool late, NvcMeshTaskPayload* payloads, uint32_t* emit_counts, uint32_t blocks, cudaStream_t stream)
{
	if (p.use_filter)
	{
		ClusterParams q = p; // filtered kernel in task-shading output mode (flattened items, per-command records)
		q.payloads = payloads;
		q.emit_counts = emit_counts;
		return launch_clustercull(q, late, blocks, stream);
	}
	void (*kernel)(ClusterParams, NvcMeshTaskPayload*, uint32_t*) = late ? taskcull_kernel<true> : taskcull_kernel<false>;
	kernel<<<blocks, kClusterBlock, 0, stream>>>(p, payloads, emit_counts);
	return cudaGetLastError();
}

cudaError_t launch_clustercull_passthrough(const ClusterParams& p, uint32_t blocks, cudaStream_t stream)
{
	clustercull_passthrough_kernel<<<blocks, kPassBlock, 0, stream>>>(p);
	return cudaGetLastError();
}

cudaError_t launch_taskcull_passthrough(const NvcMeshTaskCommand* task_commands, const uint32_t* command_count4, NvcMeshTaskPayload* payloads, uint32_t* emit_counts, uint32_t blocks,
    cudaStream_t stream)
{
	taskcull_passthrough_kernel<<<blocks, kPassBlock, 0, stream>>>(task_commands, command_count4, payloads, emit_counts);
	return cudaGetLastError();
}

cudaError_t launch_pyramid(const PyramidParams& p, cudaStream_t stream)
{
	dim3 grid((p.hiz.width + kPyrTile - 1) / kPyrTile, (p.hiz.height + kPyrTile - 1) / kPyrTile);
	bool exact = p.depth_width == 2 * p.hiz.width && p.depth_height == 2 * p.hiz.height;
	PyramidParams q = p;
	// 16-byte loads of the depth rows / 8-byte stores of mip 0 need aligned bases (row pitches are multiples of 4 / 2
	// texels whenever a full 64-texel tile exists)
	q.vector_ok = (reinterpret_cast<uintptr_t>(p.depth) & 15u) == 0 && (reinterpret_cast<uintptr_t>(p.hiz.texels) & 7u) == 0 && (p.depth_width & 3u) == 0;
	void (*kernel)(PyramidParams) = exact ? pyramid_kernel<true> : pyramid_kernel<false>;
	kernel<<<grid, kPyrBlock, 0, stream>>>(q);
	return cudaGetLastError();
}

cudaError_t clustercull_occupancy(int* blocks_per_sm_early, int* blocks_per_sm_late, int* blocks_per_sm_late_staged, uint32_t stage_bytes)
{
	cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm_early, clustercull_kernel<false, false>, kClusterBlock, 0);
	if (e == cudaSuccess)
		e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm_late, clustercull_kernel<true, false>, kClusterBlock, 0);
	if (e == cudaSuccess)
		e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm_late_staged, clustercull_kernel<true, true>, kClusterBlock, stage_bytes);
	return e;
}

cudaError_t clustercull_filter_occupancy(int* blocks_per_sm_early, int* blocks_per_sm_late)
{
	cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm_early, clustercull_filter_kernel<false, false, true, false, 1>, kClusterBlock, 0);
	if (e == cudaSuccess)
		e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm_late, clustercull_filter_kernel<true, true, true, false, 1>, kClusterBlock, 0);
	return e;
}

// nvc_scene_cache_read_device: the vertex codec's three passes (nvc_cache_decode.cuh)
cudaError_t launch_decode_vertices(const VertexDecodeArgs& a, uint32_t stride, cudaStream_t stream)
{
	if (a.blocks == 0)
		return cudaSuccess;
	const size_t words = size_t(a.vertex_count) * (stride / 4);
	const uint32_t apply_blocks = uint32_t(min(size_t(4096), (words + cache::kApplyThreads - 1) / cache::kApplyThreads));
	const uint32_t grid = (a.blocks + cache::kVertexWarps - 1) / cache::kVertexWarps;
	void (*blocks)(VertexDecodeArgs) = stride == 16 ? cache::decode_vertex_blocks_kernel<16> : cache::decode_vertex_blocks_kernel<8>;
	void (*carry)(VertexDecodeArgs) = stride == 16 ? cache::decode_vertex_carry_kernel<4> : cache::decode_vertex_carry_kernel<2>;
	void (*apply)(VertexDecodeArgs) = stride == 16 ? cache::decode_vertex_apply_kernel<4> : cache::decode_vertex_apply_kernel<2>;
	blocks<<<grid, cache::kVertexWarps * 32, 0, stream>>>(a);
	carry<<<stride / 4, cache::kCarryThreads, 0, stream>>>(a);
	apply<<<apply_blocks, cache::kApplyThreads, 0, stream>>>(a);
	return cudaGetLastError();
}

cudaError_t launch_decode_meshlets(const MeshletDecodeArgs& a, cudaStream_t stream)
{
	if (a.meshlet_count == 0)
		return cudaSuccess;
	const uint32_t groups = (a.meshlet_count + 31) / 32;
	void (*kernel)(MeshletDecodeArgs) = cache::decode_meshlets_kernel;
	kernel<<<(groups + cache::kMeshletWarps - 1) / cache::kMeshletWarps, cache::kMeshletWarps * 32, 0, stream>>>(a);
	return cudaGetLastError();
}

// nvc_scene_cache_read_device: the index codec's symbolic pass, three-launch scan and concrete pass (nvc_cache_decode.cuh)
cudaError_t launch_decode_indices(const IndexDecodeArgs& a, cudaStream_t stream)
{
	if (a.chunks == 0)
		return cudaSuccess;
	const uint32_t grid = (a.chunks + cache::kIndexThreads - 1) / cache::kIndexThreads;
	const uint32_t scan_grid = (a.runs + cache::kIndexScanWarps - 1) / cache::kIndexScanWarps;
	void (*symbolic)(IndexDecodeArgs) = cache::decode_index_symbolic_kernel;
	void (*totals)(IndexDecodeArgs) = cache::decode_index_scan_kernel<false>;
	void (*runs)(IndexDecodeArgs) = cache::decode_index_runs_kernel;
	void (*prefix)(IndexDecodeArgs) = cache::decode_index_scan_kernel<true>;
	void (*concrete)(IndexDecodeArgs) = cache::decode_index_concrete_kernel;
	symbolic<<<grid, cache::kIndexThreads, 0, stream>>>(a);
	totals<<<scan_grid, cache::kIndexScanWarps * 32, 0, stream>>>(a);
	runs<<<1, 32, 0, stream>>>(a);
	prefix<<<scan_grid, cache::kIndexScanWarps * 32, 0, stream>>>(a);
	concrete<<<grid, cache::kIndexThreads, 0, stream>>>(a);
	return cudaGetLastError();
}

// nvc_scene_cache_write: the vertex codec's estimate, measure, scan and write passes (nvc_cache_encode.cuh)
cudaError_t launch_encode_vertices(const VertexEncodeArgs& a, uint32_t stride, cudaStream_t stream)
{
	cudaError_t e = cudaMemsetAsync(a.estimate, 0, sizeof(unsigned long long) * 2 * (stride / 4), stream);
	if (e != cudaSuccess)
		return e;
	const uint32_t grid = (a.blocks + cache::kEncodeWarps - 1) / cache::kEncodeWarps;
	const size_t items = (size_t(a.vertex_count) + 3 * kVertexBlockEncode - 1) / (3 * kVertexBlockEncode) * 16 * (stride / 4);
	const uint32_t estimate_blocks = uint32_t(min(size_t(4096), (items + cache::kEstimateThreads - 1) / cache::kEstimateThreads));
	void (*estimate)(VertexEncodeArgs) = stride == 16 ? cache::encode_vertex_estimate_kernel<16> : cache::encode_vertex_estimate_kernel<8>;
	void (*measure)(VertexEncodeArgs) = stride == 16 ? cache::encode_vertex_blocks_kernel<16, false> : cache::encode_vertex_blocks_kernel<8, false>;
	void (*write)(VertexEncodeArgs) = stride == 16 ? cache::encode_vertex_blocks_kernel<16, true> : cache::encode_vertex_blocks_kernel<8, true>;
	void (*offsets)(const uint32_t*, uint32_t, unsigned long long*) = scan::offsets_kernel;
	if (a.vertex_count > 1) // one vertex keeps channel 0 everywhere
		estimate<<<estimate_blocks, cache::kEstimateThreads, 0, stream>>>(a);
	measure<<<grid, cache::kEncodeWarps * 32, 0, stream>>>(a);
	offsets<<<1, scan::kOffsetsThreads, 0, stream>>>(a.block_bytes, a.blocks, a.offsets);
	write<<<grid, cache::kEncodeWarps * 32, 0, stream>>>(a);
	return cudaGetLastError();
}

cudaError_t launch_encode_meshlets(const MeshletEncodeArgs& a, cudaStream_t stream)
{
	cudaError_t e = cudaMemsetAsync(a.invalid, 0, 4, stream);
	if (e != cudaSuccess)
		return e;
	const uint32_t grid = (a.meshlet_count + cache::kMeshletEncodeThreads - 1) / cache::kMeshletEncodeThreads;
	void (*measure)(MeshletEncodeArgs) = cache::encode_meshlets_kernel<false>;
	void (*write)(MeshletEncodeArgs) = cache::encode_meshlets_kernel<true>;
	void (*offsets)(const uint32_t*, uint32_t, unsigned long long*) = scan::offsets_kernel;
	if (a.meshlet_count)
		measure<<<grid, cache::kMeshletEncodeThreads, 0, stream>>>(a);
	offsets<<<1, scan::kOffsetsThreads, 0, stream>>>(a.block_bytes, a.meshlet_count, a.offsets);
	if (a.meshlet_count)
		write<<<grid, cache::kMeshletEncodeThreads, 0, stream>>>(a);
	return cudaGetLastError();
}

} // namespace nvc
