// nvc_api.cu — the C ABI declared in include/niagara_cull.h (context, argument validation, launches).
#include "nvc_internal.h"
#include "nvc_filter.cuh"
#include "nvc_meshlets.cuh"
#include "nvc_lods.cuh"

#include <algorithm>
#include <numeric>
#include <vector>

#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace
{

// Coarse Hi-Z mips staged per CTA (TMA): static + dynamic shared memory of clustercull_kernel<true, true> must stay under the
// 48 KB a kernel gets without opting in; its static part is 8.2 KB (s_stage[8][256] + barriers), so 39 KB = 9984 texels.
constexpr uint32_t kMaxStageTexels = 9984;

using nvc::cuda_fail;
using nvc::device_is_current;

// Picks the coarse tail of the pyramid that is staged into shared memory by TMA: the largest set of top mips whose
// texels fit the budget, whose start is 16-byte aligned in the packed allocation and that holds at least one 16-byte unit.
void choose_stage(nvc::HiZDesc& hz, uint32_t total_texels, uint32_t budget_texels)
{
	hz.stage_level = hz.levels;
	hz.stage_texels = 0;
	if (budget_texels == 0)
		return;
	for (uint32_t l = 0; l < hz.levels; ++l)
	{
		uint32_t tail = total_texels - hz.level_offset[l];
		uintptr_t addr = reinterpret_cast<uintptr_t>(hz.texels + hz.level_offset[l]);
		if (tail <= budget_texels && tail >= 4 && (addr & 15u) == 0)
		{
			hz.stage_level = l;
			hz.stage_texels = tail;
			return;
		}
	}
}

} // namespace

namespace nvc
{
void choose_stage_public(HiZDesc& hz, uint32_t total_texels, uint32_t budget_texels)
{
	choose_stage(hz, total_texels, budget_texels);
}
} // namespace nvc

namespace
{

// Lifetime calls (destroy / prepare / staging) work on the context's device and put the caller's device back afterwards.
struct DeviceGuard
{
	int previous = -1;
	explicit DeviceGuard(int device)
	{
		if (cudaGetDevice(&previous) != cudaSuccess)
			previous = -1;
		if (previous != device)
			cudaSetDevice(device);
		else
			previous = -1; // nothing to restore
	}
	~DeviceGuard()
	{
		if (previous >= 0)
			cudaSetDevice(previous);
	}
};

bool fill_hiz(const NvcHiZ* in, nvc::HiZDesc& out)
{
	memset(&out, 0, sizeof(out));
	if (!in)
		return false;
	if (!in->texels || in->levels == 0 || in->levels > NVC_MAX_HIZ_LEVELS || in->width == 0 || in->height == 0)
		return false;
	out.texels = in->texels;
	out.width = in->width;
	out.height = in->height;
	out.levels = in->levels;
	memcpy(out.level_offset, in->level_offset, sizeof(out.level_offset));
	out.stage_level = in->levels; // staging is opted into per pass
	out.stage_texels = 0;
	return true;
}

// Attaches the context's footprint image when it was built (nvc_depth_pyramid) for exactly this pyramid.
void attach_footprints(const NvcContext* ctx, const NvcHiZ* in, nvc::HiZDesc& out)
{
	out.fp = nullptr;
	if (!ctx->hiz_fp || !ctx->hiz_fp_valid || !in || ctx->hiz_fp_key != in->texels || ctx->hiz_fp_width != in->width || ctx->hiz_fp_height != in->height || ctx->hiz_fp_levels != in->levels)
		return;
	out.fp = ctx->hiz_fp;
	out.fp_first = ctx->hiz_fp_first;
	memcpy(out.fp_offset, ctx->hiz_fp_offset, sizeof(out.fp_offset));
}

} // namespace

extern "C"
{

NVC_API const char* nvc_version(void)
{
	return "niagara_b200 0.1 (sm_90a)";
}

NVC_API const char* nvc_status_string(int status)
{
	switch (status)
	{
	case NVC_OK:
		return "ok";
	case NVC_ERROR_INVALID_ARGUMENT:
		return "invalid argument";
	case NVC_ERROR_CUDA:
		return "CUDA error";
	case NVC_ERROR_NO_DEVICE:
		return "no CUDA device";
	case NVC_ERROR_OUT_OF_MEMORY:
		return "out of memory";
	case NVC_ERROR_NCCL:
		return "NCCL error";
	case NVC_ERROR_UNSUPPORTED:
		return "unsupported input";
	case NVC_ERROR_CORRUPT:
		return "corrupt scene cache";
	default:
		return "unknown status";
	}
}

NVC_API const char* nvc_last_error(const NvcContext* ctx)
{
	return ctx ? ctx->last_error.c_str() : "";
}

NVC_API int nvc_create(int device, const NvcLimits* limits, NvcContext** out_ctx)
{
	if (!out_ctx)
		return NVC_ERROR_INVALID_ARGUMENT;
	*out_ctx = nullptr;

	int count = 0;
	if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0)
		return NVC_ERROR_NO_DEVICE; // no CPU fallback: the product path needs a GPU
	if (device < 0 || device >= count)
		return NVC_ERROR_INVALID_ARGUMENT;

	NvcContext* ctx = new NvcContext();
	ctx->device = device;
	if (limits)
	{
		if (limits->task_wglimit == 0 || limits->cluster_limit == 0 || limits->cluster_limit > (1u << 24) || limits->task_wglimit > (1u << 24))
		{
			delete ctx;
			return NVC_ERROR_INVALID_ARGUMENT; // cluster index packs a 24-bit command id
		}
		ctx->limits = *limits;
	}

	cudaError_t e = cudaSetDevice(device);
	if (e == cudaSuccess)
		e = cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device);
	if (e == cudaSuccess)
		e = cudaMalloc(&ctx->scratch, sizeof(nvc::Scratch));
	if (e == cudaSuccess)
		e = cudaMemset(ctx->scratch, 0, sizeof(nvc::Scratch));
	if (e == cudaSuccess)
	{
		if (const char* env = getenv("NVC_HIZ_STAGE_TEXELS"))
			ctx->hiz_stage_budget = uint32_t(strtoul(env, nullptr, 10));
		if (ctx->hiz_stage_budget > kMaxStageTexels)
			ctx->hiz_stage_budget = kMaxStageTexels;
		e = nvc::clustercull_occupancy(&ctx->cluster_blocks_early, &ctx->cluster_blocks_late, &ctx->cluster_blocks_late_staged, ctx->hiz_stage_budget * 4u);
	}
	if (e == cudaSuccess)
		e = nvc::clustercull_filter_occupancy(&ctx->cluster_filter_blocks_early, &ctx->cluster_filter_blocks_late);
	if (const char* env = getenv("NVC_CLUSTER_FILTER"))
		ctx->cluster_filter = atoi(env) != 0;
	if (const char* env = getenv("NVC_DRAW_FILTER"))
		ctx->draw_filter = atoi(env) != 0;
	if (e == cudaSuccess)
		e = cudaDeviceSynchronize();
	if (e != cudaSuccess)
	{
		fprintf(stderr, "nvc_create: %s\n", cudaGetErrorString(e));
		if (ctx->scratch)
			cudaFree(ctx->scratch);
		delete ctx;
		return e == cudaErrorMemoryAllocation ? NVC_ERROR_OUT_OF_MEMORY : NVC_ERROR_CUDA;
	}
	if (ctx->cluster_blocks_early < 1)
		ctx->cluster_blocks_early = 1;
	if (ctx->cluster_blocks_late < 1)
		ctx->cluster_blocks_late = 1;
	if (ctx->cluster_blocks_late_staged < 1)
		ctx->cluster_blocks_late_staged = 1;
	if (ctx->cluster_filter_blocks_early < 1)
		ctx->cluster_filter_blocks_early = 1;
	if (ctx->cluster_filter_blocks_late < 1)
		ctx->cluster_filter_blocks_late = 1;

	*out_ctx = ctx;
	return NVC_OK;
}

NVC_API void nvc_destroy(NvcContext* ctx)
{
	if (!ctx)
		return;
	DeviceGuard guard(ctx->device);
	nvc::gather_destroy(ctx);
	nvc::nccl_destroy(ctx);
	if (ctx->scratch)
		cudaFree(ctx->scratch);
	if (ctx->mesh_heads)
		cudaFree(ctx->mesh_heads);
	if (ctx->mesh_errors)
		cudaFree(ctx->mesh_errors);
	if (ctx->meshlet_sphere)
		cudaFree(ctx->meshlet_sphere);
	if (ctx->meshlet_cone)
		cudaFree(ctx->meshlet_cone);
	if (ctx->hiz_fp)
		cudaFree(ctx->hiz_fp);
	if (ctx->load_scratch)
		cudaFree(ctx->load_scratch);
	delete ctx;
}

NVC_API int nvc_prepare_meshes(NvcContext* ctx, void* stream, const NvcMesh* meshes, uint32_t mesh_count)
{
	if (!ctx)
		return NVC_ERROR_INVALID_ARGUMENT;
	DeviceGuard guard(ctx->device);
	if (ctx->mesh_heads)
	{
		cudaDeviceSynchronize();
		cudaFree(ctx->mesh_heads);
		cudaFree(ctx->mesh_errors);
		ctx->mesh_heads = nullptr;
		ctx->mesh_errors = nullptr;
		ctx->prepared_meshes = nullptr;
		ctx->prepared_mesh_count = 0;
	}
	if (!meshes || mesh_count == 0)
		return NVC_OK; // un-prepare
	cudaError_t e = cudaMalloc(&ctx->mesh_heads, size_t(mesh_count) * sizeof(nvc::MeshCullHead));
	if (e == cudaSuccess)
		e = cudaMalloc(&ctx->mesh_errors, size_t(mesh_count) * NVC_MAX_LODS * sizeof(float));
	if (e == cudaSuccess)
		e = nvc::launch_pack_meshes(meshes, mesh_count, static_cast<nvc::MeshCullHead*>(ctx->mesh_heads), ctx->mesh_errors, static_cast<cudaStream_t>(stream));
	if (e != cudaSuccess)
	{
		cudaFree(ctx->mesh_heads);
		cudaFree(ctx->mesh_errors);
		ctx->mesh_heads = nullptr;
		ctx->mesh_errors = nullptr;
		return e == cudaErrorMemoryAllocation ? NVC_ERROR_OUT_OF_MEMORY : cuda_fail(ctx, e, "nvc_prepare_meshes");
	}
	ctx->prepared_meshes = meshes;
	ctx->prepared_mesh_count = mesh_count;
	return NVC_OK;
}

NVC_API int nvc_prepare_meshlets(NvcContext* ctx, void* stream, const NvcMeshlet* meshlets, uint32_t meshlet_count)
{
	if (!ctx)
		return NVC_ERROR_INVALID_ARGUMENT;
	DeviceGuard guard(ctx->device);
	if (ctx->meshlet_sphere)
	{
		cudaDeviceSynchronize();
		cudaFree(ctx->meshlet_sphere);
		cudaFree(ctx->meshlet_cone);
		ctx->meshlet_sphere = nullptr;
		ctx->meshlet_cone = nullptr;
		ctx->prepared_meshlets = nullptr;
	}
	if (!meshlets || meshlet_count == 0)
		return NVC_OK; // un-prepare
	cudaError_t e = cudaMalloc(&ctx->meshlet_sphere, size_t(meshlet_count) * sizeof(uint2));
	if (e == cudaSuccess)
		e = cudaMalloc(&ctx->meshlet_cone, size_t(meshlet_count) * sizeof(uint32_t));
	if (e == cudaSuccess)
		e = nvc::launch_pack_meshlets(meshlets, meshlet_count, ctx->meshlet_sphere, ctx->meshlet_cone, static_cast<cudaStream_t>(stream));
	if (e != cudaSuccess)
	{
		cudaFree(ctx->meshlet_sphere);
		cudaFree(ctx->meshlet_cone);
		ctx->meshlet_sphere = nullptr;
		ctx->meshlet_cone = nullptr;
		return e == cudaErrorMemoryAllocation ? NVC_ERROR_OUT_OF_MEMORY : cuda_fail(ctx, e, "nvc_prepare_meshlets");
	}
	ctx->prepared_meshlets = meshlets;
	return NVC_OK;
}

NVC_API int nvc_set_hiz_staging(NvcContext* ctx, uint32_t texels)
{
	if (!ctx)
		return NVC_ERROR_INVALID_ARGUMENT;
	DeviceGuard guard(ctx->device);
	ctx->hiz_stage_budget = texels > kMaxStageTexels ? kMaxStageTexels : texels;
	int early = 0, late = 0;
	cudaError_t e = nvc::clustercull_occupancy(&early, &late, &ctx->cluster_blocks_late_staged, ctx->hiz_stage_budget * 4u);
	if (e != cudaSuccess)
		return cuda_fail(ctx, e, "nvc_set_hiz_staging");
	if (ctx->cluster_blocks_late_staged < 1)
		ctx->cluster_blocks_late_staged = 1;
	return NVC_OK;
}

NVC_API int nvc_set_cluster_filter(NvcContext* ctx, int enabled)
{
	if (!ctx)
		return NVC_ERROR_INVALID_ARGUMENT;
	ctx->cluster_filter = enabled != 0;
	return NVC_OK;
}

NVC_API int nvc_filter_stats(NvcContext* ctx, uint64_t* out_items_undecided2, int reset)
{
	if (!ctx)
		return NVC_ERROR_INVALID_ARGUMENT;
	DeviceGuard guard(ctx->device);
	cudaError_t e = cudaDeviceSynchronize();
	unsigned long long v[2] = { 0, 0 };
	if (e == cudaSuccess)
		e = cudaMemcpy(v, &ctx->scratch->filter_items, sizeof(v), cudaMemcpyDeviceToHost);
	if (e == cudaSuccess && reset)
		e = cudaMemset(&ctx->scratch->filter_items, 0, sizeof(v));
	if (e != cudaSuccess)
		return cuda_fail(ctx, e, "nvc_filter_stats");
	if (out_items_undecided2)
	{
		out_items_undecided2[0] = v[0];
		out_items_undecided2[1] = v[1];
	}
	return NVC_OK;
}

NVC_API int nvc_filter_approx(NvcContext* ctx, void* stream, int op, const uint32_t* in, uint32_t* out, uint64_t n)
{
	if (!ctx || (op != 0 && op != 1) || (n && (!in || !out)) || n > (uint64_t(INT32_MAX) << 8)) // one 256-thread block per 256 inputs
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	cudaError_t e = nvc::launch_filter_approx(in, out, n, op, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_filter_approx");
}

NVC_API int nvc_drawcull(NvcContext* ctx, void* stream, const NvcCullData* cull, int late, int task,
    const NvcMeshDraw* draws, const NvcMesh* meshes, uint32_t* draw_visibility,
    void* commands, uint32_t* command_count4, const NvcHiZ* hiz)
{
	if (!ctx || !cull || !commands || !command_count4)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (cull->drawCount && (!draws || !meshes || !draw_visibility))
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;

	nvc::DrawCullParams p;
	memset(&p, 0, sizeof(p));
	p.cull = *cull;
	// TASK_CULL = 0: drawcull.comp.glsl:104 loses its (clusterOcclusionEnabled == 1 && TASK_CULL == 1) term; the kernel reads the
	// field only there
	if (!ctx->task_cull)
		p.cull.clusterOcclusionEnabled = 0;
	p.draws = draws;
	p.meshes = meshes;
	if (ctx->mesh_heads && ctx->prepared_meshes == meshes)
	{
		p.mesh_heads = static_cast<const nvc::MeshCullHead*>(ctx->mesh_heads);
		p.mesh_errors = ctx->mesh_errors;
	}
	p.draw_visibility = draw_visibility;
	p.commands = commands;
	p.command_count4 = command_count4;
	p.scratch = ctx->scratch;
	p.task_wglimit = ctx->limits.task_wglimit;
	if (late && task && ctx->gather)
		p.mc_commands = nvc::gather_fused_target(ctx); // armed by nvc_gather_fuse_next_drawcull, else nullptr
	bool need_hiz = late && cull->occlusionEnabled == 1;
	if (!fill_hiz(hiz, p.hiz) && need_hiz)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (need_hiz && ctx->cluster_filter && ctx->draw_filter)
	{
		// the occlusion stage as a conservative filter (same switch and the same validity domain as the cluster pass)
		attach_footprints(ctx, hiz, p.hiz);
		p.filter = nvc::make_filter_consts(p.cull, p.hiz, true);
		p.use_filter = (p.filter.enabled && p.filter.occ_ok) ? 1u : 0u;
	}

	cudaError_t e = nvc::launch_drawcull(p, late != 0, task != 0, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_drawcull");
}

static int fill_cluster_params(NvcContext* ctx, const NvcCullData* cull, int late, const NvcMeshTaskCommand* task_commands,
    const uint32_t* command_count4, const NvcMeshDraw* draws, const NvcMeshlet* meshlets, uint32_t* meshlet_visibility,
    const NvcHiZ* hiz, nvc::ClusterParams& p)
{
	if (!ctx || !cull || !task_commands || !command_count4 || !draws || !meshlets)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (cull->clusterOcclusionEnabled == 1 && !meshlet_visibility)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	memset(&p, 0, sizeof(p));
	p.cull = *cull;
	p.task_commands = task_commands;
	p.command_count4 = command_count4;
	p.draws = draws;
	p.meshlets = meshlets;
	if (ctx->meshlet_sphere && ctx->prepared_meshlets == meshlets)
	{
		p.ml_sphere = reinterpret_cast<const char*>(ctx->meshlet_sphere);
		p.ml_cone = reinterpret_cast<const char*>(ctx->meshlet_cone);
		p.ml_sphere_stride = sizeof(uint2);
		p.ml_cone_stride = sizeof(uint32_t);
	}
	else
	{
		p.ml_sphere = reinterpret_cast<const char*>(meshlets);
		p.ml_cone = reinterpret_cast<const char*>(meshlets) + 8;
		p.ml_sphere_stride = p.ml_cone_stride = sizeof(NvcMeshlet);
	}
	p.meshlet_visibility = meshlet_visibility;
	p.scratch = ctx->scratch;
	p.cluster_limit = ctx->limits.cluster_limit;
	bool need_hiz = late && cull->clusterOcclusionEnabled == 1;
	if (!fill_hiz(hiz, p.hiz) && need_hiz)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (need_hiz)
		attach_footprints(ctx, hiz, p.hiz);
	return NVC_OK;
}

NVC_API int nvc_clustercull(NvcContext* ctx, void* stream, const NvcCullData* cull, int late,
    const NvcMeshTaskCommand* task_commands, const uint32_t* command_count4,
    const NvcMeshDraw* draws, const NvcMeshlet* meshlets, uint32_t* meshlet_visibility,
    uint32_t* cluster_indices, uint32_t* cluster_count4, const NvcHiZ* hiz)
{
	if (!cluster_indices || !cluster_count4)
		return NVC_ERROR_INVALID_ARGUMENT;
	nvc::ClusterParams p;
	int s = fill_cluster_params(ctx, cull, late, task_commands, command_count4, draws, meshlets, meshlet_visibility, hiz, p);
	if (s != NVC_OK)
		return s;
	p.cluster_indices = cluster_indices;
	p.cluster_count4 = cluster_count4;
	if (!ctx->task_cull)
	{
		cudaError_t e = nvc::launch_clustercull_passthrough(p, uint32_t(ctx->sm_count) * 8u, static_cast<cudaStream_t>(stream));
		return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_clustercull");
	}

	bool staged = false;
	if (late && cull->clusterOcclusionEnabled == 1 && hiz)
	{
		nvc::choose_stage_public(p.hiz, hiz->total_texels, ctx->hiz_stage_budget);
		staged = p.hiz.stage_level < p.hiz.levels;
	}
	uint32_t blocks = uint32_t(ctx->sm_count) * uint32_t(late ? (staged ? ctx->cluster_blocks_late_staged : ctx->cluster_blocks_late) : ctx->cluster_blocks_early);
	// default: the filtered kernel (conservative filter + exact fallback, same results); TMA-staged Hi-Z and
	// nvc_set_cluster_filter(ctx, 0) select the exact kernel
	if (ctx->cluster_filter && !staged)
	{
		const bool need_occlusion = late && cull->clusterOcclusionEnabled == 1;
		p.filter = nvc::make_filter_consts(p.cull, p.hiz, need_occlusion);
		// unusual view / projection / pyramid shapes are outside the filter's error analysis: the exact kernel takes the pass
		if (p.filter.enabled && (!need_occlusion || p.filter.occ_ok))
		{
			p.use_filter = 1;
			blocks = uint32_t(ctx->sm_count) * uint32_t(late ? ctx->cluster_filter_blocks_late : ctx->cluster_filter_blocks_early);
		}
	}
	// multi-GPU: the persistent grid would otherwise own every register of every SM for the whole pass, and the exchange's
	// one-block helper kernels (acknowledgement wait, flag raise) could not start before it ends — leave two CTA slots free
	if (ctx->gather)
	{
		const uint32_t reserve = nvc::gather_reserved_blocks(ctx);
		if (blocks > 4 * reserve)
			blocks -= reserve;
	}
	cudaError_t e = nvc::launch_clustercull(p, late != 0, blocks, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_clustercull");
}

NVC_API int nvc_taskcull(NvcContext* ctx, void* stream, const NvcCullData* cull, int late,
    const NvcMeshTaskCommand* task_commands, const uint32_t* command_count4,
    const NvcMeshDraw* draws, const NvcMeshlet* meshlets, uint32_t* meshlet_visibility,
    NvcMeshTaskPayload* payloads, uint32_t* emit_counts, const NvcHiZ* hiz)
{
	if (!payloads || !emit_counts)
		return NVC_ERROR_INVALID_ARGUMENT;
	nvc::ClusterParams p;
	int s = fill_cluster_params(ctx, cull, late, task_commands, command_count4, draws, meshlets, meshlet_visibility, hiz, p);
	if (s != NVC_OK)
		return s;
	if (!ctx->task_cull)
	{
		cudaError_t e = nvc::launch_taskcull_passthrough(task_commands, command_count4, payloads, emit_counts, uint32_t(ctx->sm_count) * 8u, static_cast<cudaStream_t>(stream));
		return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_taskcull");
	}
	uint32_t blocks = uint32_t(ctx->sm_count) * 4u;
	if (ctx->cluster_filter)
	{
		const bool need_occlusion = late && cull->clusterOcclusionEnabled == 1;
		p.filter = nvc::make_filter_consts(p.cull, p.hiz, need_occlusion);
		if (p.filter.enabled && (!need_occlusion || p.filter.occ_ok))
		{
			p.use_filter = 1;
			blocks = uint32_t(ctx->sm_count) * uint32_t(late ? ctx->cluster_filter_blocks_late : ctx->cluster_filter_blocks_early);
		}
	}
	cudaError_t e = nvc::launch_taskcull(p, late != 0, payloads, emit_counts, blocks, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_taskcull");
}

NVC_API int nvc_decode_clusters(NvcContext* ctx, void* stream, const uint32_t* cluster_indices, const uint32_t* cluster_count4,
    const NvcMeshTaskCommand* task_commands, const NvcMeshlet* meshlets, NvcClusterRecord* records, uint32_t* stats4)
{
	if (!ctx || !cluster_indices || !cluster_count4 || !task_commands || !meshlets || !stats4)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	cudaError_t e = nvc::launch_decode_clusters(cluster_indices, cluster_count4, task_commands, meshlets, records, stats4, uint32_t(ctx->sm_count) * 8u, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_decode_clusters");
}

NVC_API int nvc_set_task_cull(NvcContext* ctx, int enabled)
{
	if (!ctx)
		return NVC_ERROR_INVALID_ARGUMENT;
	ctx->task_cull = enabled != 0;
	return NVC_OK;
}

// the mesh-cull counters when the stage is on (read when the call is enqueued), nullptr when it is off
static unsigned long long* mesh_cull_counters(NvcContext* ctx)
{
	return ctx->mesh_cull ? &ctx->scratch->mesh_cull_tested : nullptr;
}

NVC_API int nvc_set_mesh_cull(NvcContext* ctx, int enabled)
{
	if (!ctx)
		return NVC_ERROR_INVALID_ARGUMENT;
	ctx->mesh_cull = enabled != 0;
	return NVC_OK;
}

NVC_API int nvc_mesh_cull_stats(NvcContext* ctx, uint64_t* out_tested_culled2, int reset)
{
	if (!ctx)
		return NVC_ERROR_INVALID_ARGUMENT;
	DeviceGuard guard(ctx->device);
	cudaError_t e = cudaDeviceSynchronize();
	unsigned long long v[2] = { 0, 0 };
	if (e == cudaSuccess)
		e = cudaMemcpy(v, &ctx->scratch->mesh_cull_tested, sizeof(v), cudaMemcpyDeviceToHost);
	if (e == cudaSuccess && reset)
		e = cudaMemset(&ctx->scratch->mesh_cull_tested, 0, sizeof(v));
	if (e != cudaSuccess)
		return cuda_fail(ctx, e, "nvc_mesh_cull_stats");
	if (out_tested_culled2)
	{
		out_tested_culled2[0] = v[0];
		out_tested_culled2[1] = v[1];
	}
	return NVC_OK;
}

NVC_API int nvc_raster_depth(NvcContext* ctx, void* stream, const float* projection16, const NvcCullData* pass, const uint32_t* cluster_indices, const uint32_t* cluster_count4,
    const NvcMeshTaskCommand* task_commands, const NvcMeshDraw* draws, const NvcMeshlet* meshlets, const uint32_t* meshletdata, uint32_t meshletdata_words, const NvcVertex* vertices,
    uint32_t vertex_count, float* depth, uint32_t width, uint32_t height, uint32_t* stats4)
{
	if (!ctx || !projection16 || !pass || !cluster_indices || !cluster_count4 || !task_commands || !draws || !meshlets || !meshletdata || !vertices || !depth || width == 0 || height == 0)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (uint64_t(width) * height >= (1ull << 31))
		return NVC_ERROR_UNSUPPORTED;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	cudaError_t e = nvc::launch_raster_depth(projection16, *pass, cluster_indices, cluster_count4, task_commands, draws, meshlets, meshletdata, meshletdata_words, vertices, vertex_count, depth,
	    width, height, stats4, mesh_cull_counters(ctx), uint32_t(ctx->sm_count) * 16u, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_raster_depth");
}

NVC_API int nvc_raster_depth_tasks(NvcContext* ctx, void* stream, const float* projection16, const NvcCullData* pass, const NvcMeshTaskPayload* payloads, const uint32_t* emit_counts,
    const uint32_t* command_count4, const NvcMeshTaskCommand* task_commands, const NvcMeshDraw* draws, const NvcMeshlet* meshlets, const uint32_t* meshletdata, uint32_t meshletdata_words,
    const NvcVertex* vertices, uint32_t vertex_count, float* depth, uint32_t width, uint32_t height, uint32_t* stats4)
{
	if (!ctx || !projection16 || !pass || !payloads || !emit_counts || !command_count4 || !task_commands || !draws || !meshlets || !meshletdata || !vertices || !depth || width == 0 || height == 0)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (uint64_t(width) * height >= (1ull << 31))
		return NVC_ERROR_UNSUPPORTED;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	cudaError_t e = nvc::launch_raster_depth_tasks(projection16, *pass, payloads, emit_counts, command_count4, task_commands, draws, meshlets, meshletdata, meshletdata_words, vertices, vertex_count,
	    depth, width, height, stats4, mesh_cull_counters(ctx), uint32_t(ctx->sm_count) * 16u, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_raster_depth_tasks");
}

NVC_API int nvc_raster_depth_indexed(NvcContext* ctx, void* stream, const float* projection16, const NvcCullData* pass, const NvcMeshDrawCommand* draw_commands, const uint32_t* command_count4,
    uint32_t max_draw_count, const NvcMeshDraw* draws, const uint32_t* indices, uint32_t index_count, const NvcVertex* vertices, uint32_t vertex_count, float* depth, uint32_t width, uint32_t height,
    uint32_t* stats4)
{
	if (!ctx || !projection16 || !pass || !draw_commands || !command_count4 || !draws || !indices || !vertices || !depth || width == 0 || height == 0)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (uint64_t(width) * height >= (1ull << 31))
		return NVC_ERROR_UNSUPPORTED;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	cudaError_t e = nvc::launch_raster_depth_indexed(projection16, *pass, draw_commands, command_count4, max_draw_count, draws, indices, index_count, vertices, vertex_count, depth, width, height,
	    stats4, uint32_t(ctx->sm_count) * 16u, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_raster_depth_indexed");
}

NVC_API int nvc_depth_pyramid(NvcContext* ctx, void* stream, const float* depth,
    uint32_t depth_width, uint32_t depth_height, const NvcHiZ* hiz)
{
	if (!ctx || !depth || !hiz || depth_width == 0 || depth_height == 0)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	nvc::PyramidParams p;
	memset(&p, 0, sizeof(p));
	if (!fill_hiz(hiz, p.hiz))
		return NVC_ERROR_INVALID_ARGUMENT;
	// the pyramid must be the one the reference would allocate for this depth target (niagara.cpp:1339-1342)
	if (hiz->width != nvc_previous_pow2(depth_width) || hiz->height != nvc_previous_pow2(depth_height) ||
	    hiz->levels != nvc_image_mip_levels(hiz->width, hiz->height))
		return NVC_ERROR_INVALID_ARGUMENT;
	p.depth = depth;
	p.depth_width = depth_width;
	p.depth_height = depth_height;
	p.scratch = ctx->scratch;
	cudaError_t e = nvc::launch_pyramid(p, static_cast<cudaStream_t>(stream));
	if (e == cudaSuccess && ctx->hiz_fp && ctx->hiz_fp_key == hiz->texels && ctx->hiz_fp_width == hiz->width && ctx->hiz_fp_height == hiz->height && ctx->hiz_fp_levels == hiz->levels)
	{
		// derived footprint image of the pyramid just built (nvc_prepare_hiz), one more launch on the same stream
		memcpy(p.hiz.fp_offset, ctx->hiz_fp_offset, sizeof(p.hiz.fp_offset));
		p.hiz.fp_first = ctx->hiz_fp_first;
		e = nvc::launch_footprint(p.hiz, ctx->hiz_fp, ctx->hiz_fp_total, static_cast<cudaStream_t>(stream));
		ctx->hiz_fp_valid = e == cudaSuccess;
	}
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_depth_pyramid");
}

NVC_API int nvc_prepare_hiz(NvcContext* ctx, const NvcHiZ* hiz)
{
	if (!ctx)
		return NVC_ERROR_INVALID_ARGUMENT;
	DeviceGuard guard(ctx->device);
	if (ctx->hiz_fp)
	{
		cudaDeviceSynchronize();
		cudaFree(ctx->hiz_fp);
		ctx->hiz_fp = nullptr;
	}
	ctx->hiz_fp_key = nullptr;
	ctx->hiz_fp_valid = false;
	ctx->hiz_fp_total = 0;
	if (!hiz)
		return NVC_OK; // un-prepare
	if (!hiz->texels || hiz->levels == 0 || hiz->levels > NVC_MAX_HIZ_LEVELS || hiz->width == 0 || hiz->height == 0 || hiz->width > 65536 || hiz->height > 65536)
		return NVC_ERROR_INVALID_ARGUMENT;
	uint64_t total = 0;
	if (const char* env = getenv("NVC_FP_FIRST_LEVEL"))
		ctx->hiz_fp_first = uint32_t(strtoul(env, nullptr, 10));
	if (ctx->hiz_fp_first >= hiz->levels)
		ctx->hiz_fp_first = hiz->levels - 1; // at least the coarsest mip has an image
	for (uint32_t l = 0; l < hiz->levels; ++l)
	{
		uint32_t w = hiz->width >> l, h = hiz->height >> l;
		w = w ? w : 1;
		h = h ? h : 1;
		ctx->hiz_fp_offset[l] = uint32_t(total);
		if (l >= ctx->hiz_fp_first)
			total += uint64_t(nvc::fp_pitch(w)) * (h + 1);
	}
	if (total >= (1ull << 31))
		return NVC_ERROR_UNSUPPORTED;
	cudaError_t e = cudaMalloc(&ctx->hiz_fp, size_t(total) * sizeof(float));
	if (e != cudaSuccess)
	{
		ctx->hiz_fp = nullptr;
		return e == cudaErrorMemoryAllocation ? NVC_ERROR_OUT_OF_MEMORY : cuda_fail(ctx, e, "nvc_prepare_hiz");
	}
	ctx->hiz_fp_key = hiz->texels;
	ctx->hiz_fp_width = hiz->width;
	ctx->hiz_fp_height = hiz->height;
	ctx->hiz_fp_levels = hiz->levels;
	ctx->hiz_fp_total = uint32_t(total);
	return NVC_OK;
}

NVC_API int nvc_hiz_footprints(NvcContext* ctx, const float** image_out, uint32_t* first_level_out, uint32_t* offset_out, uint32_t* total_out)
{
	if (!ctx || !image_out)
		return NVC_ERROR_INVALID_ARGUMENT;
	const bool have = ctx->hiz_fp && ctx->hiz_fp_valid;
	*image_out = have ? ctx->hiz_fp : nullptr;
	if (first_level_out)
		*first_level_out = ctx->hiz_fp_first;
	if (offset_out)
		memcpy(offset_out, ctx->hiz_fp_offset, sizeof(ctx->hiz_fp_offset));
	if (total_out)
		*total_out = have ? ctx->hiz_fp_total : 0u;
	return NVC_OK;
}

NVC_API int nvc_update_draws(NvcContext* ctx, void* stream, NvcMeshDraw* draws, uint32_t draw_count, const uint32_t* update_indices,
    const NvcMeshDraw* update_values, uint32_t count)
{
	if (!ctx || !draws || (count && (!update_indices || !update_values)))
		return NVC_ERROR_INVALID_ARGUMENT;
	if ((reinterpret_cast<uintptr_t>(draws) | reinterpret_cast<uintptr_t>(update_values)) & 15u)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	cudaError_t e = nvc::launch_update_draws(draws, draw_count, update_indices, update_values, count, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_update_draws");
}

NVC_API int nvc_cook_meshlet_bounds(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* meshletdata,
    uint32_t meshletdata_words, NvcMeshlet* meshlets, uint32_t meshlet_count, uint32_t* rejected)
{
	if (!ctx || (meshlet_count && (!vertices || !meshletdata || !meshlets)))
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	cudaError_t e = nvc::launch_cook_meshlet_bounds(vertices, vertex_count, meshletdata, meshletdata_words, meshlets, meshlet_count, rejected, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_cook_meshlet_bounds");
}

} // extern "C"

namespace
{

// Sorts the job indices in [first, last) longest job (most indices) first, ties in index order: the cook kernels take jobs
// in this order, so the longest sequential jobs start first.  Outputs are placed by job index, so the order does not
// change them.
template <typename It, typename Job>
static void longest_first(It first, It last, const std::vector<Job>& jobs)
{
	std::stable_sort(first, last, [&](uint32_t x, uint32_t y) { return jobs[x].index_count > jobs[y].index_count; });
}

// The meshlet cooker's walk over meshes x LODs, in mesh then LOD order: per LOD its job (the scratch ranges of
// nvc_cook_meshlets laid out in that order) and whether it is the mesh's lodRT, and the sums of the per-LOD bounds.  The
// capacity queries return the sums and the cook plans its call with the jobs, so that a capacity is what the call plans.
struct CookPlan
{
	std::vector<nvc::cook::CookJob> jobs;
	std::vector<uint32_t> job_rt;  // per job: 1 for the mesh's lodRT
	std::vector<uint32_t> mesh_rt; // per mesh: its lodRT (clrt), NVC_MAX_LODS otherwise
	uint64_t tri = 0, vtx = 0, idx = 0;
	uint64_t slots = 0, words = 0, vtx0 = 0; // meshlet slots (= the meshlet bound), meshletdata words, meshletvtx0 elements
	bool in_range = true; // every vertex range and LOD index range inside the call's buffers, index counts multiples of 3
};

// false: a mesh has more than NVC_MAX_LODS LODs.  Without clrt no LOD is a lodRT (greedy bounds throughout).
bool plan_cook(const NvcMesh* meshes, uint32_t mesh_count, bool clrt, const float* max_scale, uint64_t vertex_count, uint64_t index_count, CookPlan& plan)
{
	for (uint32_t i = 0; i < mesh_count; ++i)
	{
		const NvcMesh& mesh = meshes[i];
		if (mesh.lodCount > NVC_MAX_LODS)
			return false;
		plan.in_range = plan.in_range && uint64_t(mesh.vertexOffset) + mesh.vertexCount <= vertex_count;
		const uint32_t rt = clrt ? nvc::cook::lod_rt(mesh, max_scale ? max_scale[i] : 1.0f) : NVC_MAX_LODS;
		plan.mesh_rt.push_back(rt);
		for (uint32_t l = 0; l < mesh.lodCount; ++l)
		{
			const NvcMeshLod& lod = mesh.lods[l];
			const uint32_t n = lod.indexCount;
			plan.in_range = plan.in_range && n % 3 == 0 && uint64_t(lod.indexOffset) + n <= index_count;
			plan.jobs.push_back({ i, l, lod.indexOffset, n, mesh.vertexOffset, mesh.vertexCount, plan.tri, plan.vtx, plan.idx, plan.slots });
			plan.job_rt.push_back(l == rt);
			plan.tri += n / 3;
			plan.vtx += mesh.vertexCount;
			plan.idx += n;
			plan.slots += l == rt ? nvc::cook::spatial_meshlets_bound(n) : nvc::cook::meshlets_bound(n);
			plan.words += l == rt ? nvc::cook::spatial_words_bound(n) : nvc::cook::words_bound(n);
			plan.vtx0 += l == rt ? 4ull * n : 0ull;
		}
	}
	return true;
}

uint32_t saturate32(uint64_t v)
{
	return v > 0xffffffffull ? 0xffffffffu : uint32_t(v);
}

} // namespace

NVC_API int nvc_cook_meshlets_capacity(const NvcMesh* host_meshes, uint32_t mesh_count, uint32_t* meshlets_out, uint64_t* words_out)
{
	if ((mesh_count && !host_meshes) || !meshlets_out || !words_out)
		return NVC_ERROR_INVALID_ARGUMENT;
	CookPlan plan; // the capacity does not depend on the ranges
	if (!plan_cook(host_meshes, mesh_count, false, nullptr, 0, 0, plan))
		return NVC_ERROR_INVALID_ARGUMENT;
	*meshlets_out = saturate32(plan.slots);
	*words_out = plan.words;
	return NVC_OK;
}

// nvc_cook_meshlets and, with clrt, nvc_cook_meshlets_clrt (whose meshletvtx0 arguments are unused otherwise)
static int cook_meshlets(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* indices, uint32_t index_count,
    const NvcMesh* host_meshes, NvcMesh* meshes, uint32_t mesh_count, NvcMeshlet* meshlets, uint32_t meshlet_capacity, uint32_t* meshletdata,
    uint32_t meshletdata_capacity, uint32_t* totals4, bool clrt, const float* max_scale, uint16_t* meshletvtx0, uint32_t meshletvtx0_capacity, const char* what)
{
	if (!ctx || !totals4 || (mesh_count && (!host_meshes || !meshes)) || (meshlet_capacity && !meshlets) || (meshletdata_capacity && !meshletdata))
		return NVC_ERROR_INVALID_ARGUMENT;
	if (clrt && meshletvtx0_capacity && !meshletvtx0)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;

	CookPlan plan;
	if (!plan_cook(host_meshes, mesh_count, clrt, max_scale, vertex_count, index_count, plan) || !plan.in_range)
		return NVC_ERROR_INVALID_ARGUMENT;
	if ((plan.idx && !indices) || (plan.jobs.size() && !vertices))
		return NVC_ERROR_INVALID_ARGUMENT;
	if (plan.slots > 0xffffffffull)
		return NVC_ERROR_INVALID_ARGUMENT; // meshlet slots are counted in 32 bits
	const std::vector<nvc::cook::CookJob>& jobs = plan.jobs;
	const uint32_t job_count = uint32_t(jobs.size());
	const uint64_t tri = plan.tri, vtx = plan.vtx, idx = plan.idx, slot = plan.slots;
	// clrt: Mesh[] as uploaded, with lodRT set
	std::vector<NvcMesh> rt_meshes;
	if (clrt)
		for (uint32_t i = 0; i < mesh_count; ++i)
		{
			rt_meshes.push_back(host_meshes[i]);
			rt_meshes[i].lodRT = plan.mesh_rt[i];
		}
	// clrt: the greedy jobs, then the ray-tracing jobs, each longest first
	std::vector<uint32_t> order(job_count);
	std::iota(order.begin(), order.end(), 0u);
	auto rt_end = std::stable_partition(order.begin(), order.end(), [&](uint32_t x) { return !plan.job_rt[x]; });
	longest_first(order.begin(), rt_end, jobs);
	longest_first(rt_end, order.end(), jobs);
	const uint32_t greedy_count = uint32_t(rt_end - order.begin());

	nvc::ScratchPlan sp;
	const size_t o_jobs = sp.take(job_count * sizeof(nvc::cook::CookJob)), o_order = sp.take(job_count * 4ull);
	const size_t o_cones = sp.take(tri * 24u), o_counts = sp.take(vtx * 4u), o_offsets = sp.take(vtx * 4u), o_used = sp.take(vtx * 2u);
	const size_t o_data = sp.take(idx * 4u), o_mlv = sp.take(idx * 4u), o_mlt = sp.take(idx), o_emitted = sp.take(tri);
	const size_t o_nodes = sp.take(tri * 24u), o_kdi = sp.take(tri * 4u), o_records = sp.take(slot * 16u);
	const size_t o_words = sp.take(slot * 4u), o_min = sp.take(slot * 4u), o_sdata = sp.take(slot * 4u);
	const size_t o_jm = sp.take(job_count * 4ull), o_jf = sp.take(job_count * 4ull);
	const size_t o_rt = clrt ? sp.take(job_count * 4ull) : 0, o_svtx = clrt ? sp.take(slot * 4u) : 0;

	// the previous user of the scratch finishes first
	cudaError_t e = cudaDeviceSynchronize();
	if (e != cudaSuccess)
		return cuda_fail(ctx, e, what);
	e = nvc::reserve_scratch(ctx, sp.bytes);
	if (e != cudaSuccess)
		return nvc::load_fail(ctx, e, what);
	char* base = static_cast<char*>(ctx->load_scratch);
	e = nvc::upload({ { base + o_jobs, jobs.data(), job_count * sizeof(nvc::cook::CookJob) }, { base + o_order, order.data(), job_count * 4ull },
	    { base + o_rt, plan.job_rt.data(), clrt ? job_count * 4ull : 0 }, { meshes, clrt ? rt_meshes.data() : host_meshes, size_t(mesh_count) * sizeof(NvcMesh) } });
	if (e != cudaSuccess)
		return cuda_fail(ctx, e, what);

	nvc::CookArgs a;
	a.vertices = vertices;
	a.indices = indices;
	a.jobs = reinterpret_cast<const nvc::cook::CookJob*>(base + o_jobs);
	a.order = reinterpret_cast<const uint32_t*>(base + o_order);
	a.job_count = job_count;
	a.slot_count = uint32_t(slot);
	a.cones = reinterpret_cast<float*>(base + o_cones);
	a.adj_counts = reinterpret_cast<uint32_t*>(base + o_counts);
	a.adj_offsets = reinterpret_cast<uint32_t*>(base + o_offsets);
	a.adj_data = reinterpret_cast<uint32_t*>(base + o_data);
	a.used = reinterpret_cast<int16_t*>(base + o_used);
	a.emitted = reinterpret_cast<uint8_t*>(base + o_emitted);
	a.kd_nodes = reinterpret_cast<uint32_t*>(base + o_nodes);
	a.kd_index = reinterpret_cast<uint32_t*>(base + o_kdi);
	a.ml_vertices = reinterpret_cast<uint32_t*>(base + o_mlv);
	a.ml_triangles = reinterpret_cast<uint8_t*>(base + o_mlt);
	a.ml_records = reinterpret_cast<uint4*>(base + o_records);
	a.job_meshlets = reinterpret_cast<uint32_t*>(base + o_jm);
	a.job_first = reinterpret_cast<uint32_t*>(base + o_jf);
	a.slot_words = reinterpret_cast<uint32_t*>(base + o_words);
	a.slot_min = reinterpret_cast<uint32_t*>(base + o_min);
	a.slot_data = reinterpret_cast<uint32_t*>(base + o_sdata);
	a.meshes = meshes;
	a.meshlets = meshlets;
	a.meshlet_capacity = meshlet_capacity;
	a.meshletdata = meshletdata;
	a.meshletdata_capacity = meshletdata_capacity;
	a.totals4 = totals4;
	if (clrt)
	{
		nvc::CookClrtArgs c;
		c.base = a;
		c.greedy_count = greedy_count;
		c.rt_count = job_count - greedy_count;
		c.job_rt = reinterpret_cast<const uint32_t*>(base + o_rt);
		c.slot_vtx0 = reinterpret_cast<uint32_t*>(base + o_svtx);
		c.meshletvtx0 = meshletvtx0;
		c.meshletvtx0_capacity = meshletvtx0_capacity;
		e = nvc::launch_cook_meshlets_clrt(c, static_cast<cudaStream_t>(stream));
	}
	else
		e = nvc::launch_cook_meshlets(a, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, what);
}

NVC_API int nvc_cook_meshlets(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* indices, uint32_t index_count,
    const NvcMesh* host_meshes, NvcMesh* meshes, uint32_t mesh_count, NvcMeshlet* meshlets, uint32_t meshlet_capacity, uint32_t* meshletdata,
    uint32_t meshletdata_capacity, uint32_t* totals4)
{
	return cook_meshlets(ctx, stream, vertices, vertex_count, indices, index_count, host_meshes, meshes, mesh_count, meshlets, meshlet_capacity, meshletdata,
	    meshletdata_capacity, totals4, false, nullptr, nullptr, 0, "nvc_cook_meshlets");
}

NVC_API int nvc_cook_meshlets_clrt_capacity(const NvcMesh* host_meshes, const float* max_scale, uint32_t mesh_count, uint32_t* meshlets_out, uint64_t* words_out,
    uint64_t* vtx0_out)
{
	if ((mesh_count && !host_meshes) || !meshlets_out || !words_out || !vtx0_out)
		return NVC_ERROR_INVALID_ARGUMENT;
	CookPlan plan;
	if (!plan_cook(host_meshes, mesh_count, true, max_scale, 0, 0, plan))
		return NVC_ERROR_INVALID_ARGUMENT;
	*meshlets_out = saturate32(plan.slots);
	*words_out = plan.words;
	*vtx0_out = plan.vtx0;
	return NVC_OK;
}

NVC_API int nvc_cook_meshlets_clrt(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* indices, uint32_t index_count,
    const NvcMesh* host_meshes, const float* max_scale, NvcMesh* meshes, uint32_t mesh_count, NvcMeshlet* meshlets, uint32_t meshlet_capacity,
    uint32_t* meshletdata, uint32_t meshletdata_capacity, uint16_t* meshletvtx0, uint32_t meshletvtx0_capacity, uint32_t* totals8)
{
	return cook_meshlets(ctx, stream, vertices, vertex_count, indices, index_count, host_meshes, meshes, mesh_count, meshlets, meshlet_capacity, meshletdata,
	    meshletdata_capacity, totals8, true, max_scale, meshletvtx0, meshletvtx0_capacity, "nvc_cook_meshlets_clrt");
}

namespace
{

// The LOD cooker's walk over the meshes: per mesh its job, with its own scratch words (nvc_lods.cuh carve), and the sums of
// the chain capacities and scratch words.  The capacity query returns the first sum; nvc_cook_mesh_lods plans its call with
// the jobs.
struct LodPlan
{
	std::vector<nvc::lods::LodJob> jobs;
	uint64_t indices = 0, words = 0;
	bool in_range = true; // every LOD 0 and vertex range inside the call's buffers, LOD 0 index counts multiples of 3
};

LodPlan plan_lods(const NvcMesh* meshes, uint32_t mesh_count, uint64_t vertex_count, uint64_t lod0_index_count)
{
	LodPlan plan;
	plan.jobs.resize(mesh_count);
	for (uint32_t i = 0; i < mesh_count; ++i)
	{
		const NvcMesh& mesh = meshes[i];
		nvc::lods::LodJob& job = plan.jobs[i];
		job.vertex_offset = mesh.vertexOffset;
		job.vertex_count = mesh.vertexCount;
		job.index_offset = mesh.lods[0].indexOffset;
		job.index_count = mesh.lods[0].indexCount;
		job.scratch = plan.words;
		job.capacity = nvc::lods::chain_capacity(job.index_count);
		plan.words += nvc::lods::carve(job.vertex_count, job.index_count, job.capacity, nullptr, nullptr);
		plan.indices += job.capacity;
		plan.in_range = plan.in_range && job.index_count % 3 == 0 && uint64_t(job.index_offset) + job.index_count <= lod0_index_count &&
		                uint64_t(job.vertex_offset) + job.vertex_count <= vertex_count;
	}
	return plan;
}

} // namespace

NVC_API int nvc_cook_mesh_lods_capacity(const NvcMesh* host_meshes, uint32_t mesh_count, uint32_t* indices_out)
{
	if ((mesh_count && !host_meshes) || !indices_out)
		return NVC_ERROR_INVALID_ARGUMENT;
	*indices_out = saturate32(plan_lods(host_meshes, mesh_count, 0, 0).indices); // the capacity does not depend on the ranges
	return NVC_OK;
}

NVC_API int nvc_cook_mesh_lods(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* lod0_indices,
    uint32_t lod0_index_count, const NvcMesh* host_meshes, const float* max_scale, uint32_t mesh_count, NvcMesh* meshes, uint32_t* indices,
    uint32_t index_capacity, uint32_t* totals4)
{
	if (!ctx || !totals4 || (mesh_count && (!host_meshes || !meshes)) || (index_capacity && !indices))
		return NVC_ERROR_INVALID_ARGUMENT;
	if ((vertex_count && !vertices) || (lod0_index_count && !lod0_indices))
		return NVC_ERROR_INVALID_ARGUMENT;
	const LodPlan plan = plan_lods(host_meshes, mesh_count, vertex_count, lod0_index_count);
	if (!plan.in_range)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;

	const std::vector<nvc::lods::LodJob>& jobs = plan.jobs;
	std::vector<float> scales(mesh_count, 1.0f);
	if (max_scale)
		scales.assign(max_scale, max_scale + mesh_count);
	std::vector<uint32_t> order(mesh_count);
	std::iota(order.begin(), order.end(), 0u);
	longest_first(order.begin(), order.end(), jobs);

	const size_t n = mesh_count;
	nvc::ScratchPlan sp;
	const size_t o_jobs = sp.take(n * sizeof(nvc::lods::LodJob)), o_order = sp.take(n * 4), o_scale = sp.take(n * 4);
	const size_t o_chain = sp.take(n * 8), o_base = sp.take(n * 8), o_rejected = sp.take(n), o_words = sp.take(plan.words * 4);

	// the previous user of the scratch finishes first
	cudaError_t e = cudaDeviceSynchronize();
	if (e != cudaSuccess)
		return cuda_fail(ctx, e, "nvc_cook_mesh_lods");
	e = nvc::reserve_scratch(ctx, sp.bytes);
	if (e != cudaSuccess)
		return nvc::load_fail(ctx, e, "nvc_cook_mesh_lods");
	char* base = static_cast<char*>(ctx->load_scratch);
	e = nvc::upload({ { base + o_jobs, jobs.data(), n * sizeof(nvc::lods::LodJob) }, { base + o_order, order.data(), n * 4 }, { base + o_scale, scales.data(), n * 4 } });
	if (e != cudaSuccess)
		return cuda_fail(ctx, e, "nvc_cook_mesh_lods");

	nvc::LodArgs a;
	a.vertices = vertices;
	a.lod0_indices = lod0_indices;
	a.jobs = reinterpret_cast<const nvc::lods::LodJob*>(base + o_jobs);
	a.order = reinterpret_cast<const uint32_t*>(base + o_order);
	a.max_scale = reinterpret_cast<const float*>(base + o_scale);
	a.mesh_count = mesh_count;
	a.scratch = reinterpret_cast<uint32_t*>(base + o_words);
	a.chain = reinterpret_cast<uint64_t*>(base + o_chain);
	a.rejected = reinterpret_cast<uint8_t*>(base + o_rejected);
	a.base = reinterpret_cast<uint64_t*>(base + o_base);
	a.meshes = meshes;
	a.indices = indices;
	a.index_capacity = index_capacity;
	a.totals4 = totals4;
	e = nvc::launch_cook_mesh_lods(a, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_cook_mesh_lods");
}

namespace
{

// The vertex cooker's walk over the meshes: per mesh its job (its first triangle and vertex slot, its vertex cache scratch
// words), and the call's triangles, index positions, vertex slots and scratch words.
struct VertexPlan
{
	std::vector<nvc::verts::VertexJob> jobs;
	uint64_t triangles = 0, positions = 0, slots = 0, words = 0;
	bool in_range = true; // every index and vertex range inside the call's buffers, index counts multiples of 3
};

VertexPlan plan_vertices(const NvcMesh* meshes, uint32_t mesh_count, uint64_t vertex_count, uint64_t index_count)
{
	VertexPlan plan;
	plan.jobs.resize(mesh_count);
	for (uint32_t i = 0; i < mesh_count; ++i)
	{
		const NvcMesh& mesh = meshes[i];
		nvc::verts::VertexJob& job = plan.jobs[i];
		job.vertex_offset = mesh.vertexOffset;
		job.vertex_count = mesh.vertexCount;
		job.index_offset = mesh.lods[0].indexOffset;
		job.index_count = mesh.lods[0].indexCount;
		job.tri_base = uint32_t(plan.triangles);
		job.slot_base = uint32_t(plan.slots);
		job.scratch = plan.words;
		plan.words += nvc::vertex_cache_words(std::min(job.vertex_count, job.index_count), job.index_count);
		plan.triangles += job.index_count / 3;
		plan.positions += job.index_count;
		plan.slots += job.vertex_count;
		plan.in_range = plan.in_range && job.index_count % 3 == 0 && uint64_t(job.index_offset) + job.index_count <= index_count &&
		                uint64_t(job.vertex_offset) + job.vertex_count <= vertex_count;
	}
	return plan;
}

} // namespace

NVC_API int nvc_cook_mesh_vertices(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* indices,
    uint32_t index_count, const NvcMesh* host_meshes, uint32_t mesh_count, NvcMesh* meshes, NvcVertex* vertices_out, uint32_t vertex_capacity,
    uint32_t* lod0_out, uint32_t index_capacity, uint32_t* totals4)
{
	if (!ctx || !totals4 || (mesh_count && (!host_meshes || !meshes)))
		return NVC_ERROR_INVALID_ARGUMENT;
	if ((vertex_count && !vertices) || (index_count && !indices) || (vertex_capacity && !vertices_out) || (index_capacity && !lod0_out))
		return NVC_ERROR_INVALID_ARGUMENT;
	const VertexPlan plan = plan_vertices(host_meshes, mesh_count, vertex_count, index_count);
	// neither output outgrows its input, counted per mesh (meshes may share ranges)
	if (!plan.in_range || vertex_capacity < std::max<uint64_t>(vertex_count, plan.slots) || index_capacity < std::max<uint64_t>(index_count, plan.positions))
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	if (plan.slots > (1u << 30))
		return NVC_ERROR_OUT_OF_MEMORY; // the class table would need 2^32 buckets

	const std::vector<nvc::verts::VertexJob>& jobs = plan.jobs;
	std::vector<uint32_t> order(mesh_count);
	std::iota(order.begin(), order.end(), 0u);
	longest_first(order.begin(), order.end(), jobs);

	const size_t M = mesh_count, T = plan.triangles, N = plan.positions, S = plan.slots;
	const size_t tri_buckets = nvc::lods::hash_buckets(uint32_t(T)), vtx_buckets = nvc::lods::hash_buckets(uint32_t(S));
	const size_t blocks = (N + nvc::scan::kScanItems - 1) / nvc::scan::kScanItems;
	nvc::ScratchPlan sp;
	const size_t o_jobs = sp.take(M * sizeof(nvc::verts::VertexJob)), o_order = sp.take(M * 4), o_rejected = sp.take(M);
	const size_t o_ibase = sp.take(M * 4), o_vbase = sp.take(M * 4);
	const size_t o_tri_table = sp.take(tri_buckets * 4), o_tri_entry = sp.take(T * 4);
	const size_t o_flags = sp.take(N), o_rank = sp.take((N + 1) * 4), o_sums = sp.take(blocks * 4), o_offsets = sp.take((blocks + 1) * 8);
	const size_t o_filtered = sp.take(N * 4), o_remapped = sp.take(N * 4);
	const size_t o_first = sp.take(S * 4), o_vtx_table = sp.take(vtx_buckets * 4), o_vtx_first = sp.take(vtx_buckets * 4);
	const size_t o_vtx_entry = sp.take(S * 4), o_classes = sp.take(S * 16), o_first_use = sp.take(S * 4), o_words = sp.take(plan.words * 4);

	// the previous user of the scratch finishes first
	cudaError_t e = cudaDeviceSynchronize();
	if (e != cudaSuccess)
		return cuda_fail(ctx, e, "nvc_cook_mesh_vertices");
	e = nvc::reserve_scratch(ctx, sp.bytes);
	if (e != cudaSuccess)
		return nvc::load_fail(ctx, e, "nvc_cook_mesh_vertices");
	char* base = static_cast<char*>(ctx->load_scratch);
	e = nvc::upload({ { base + o_jobs, jobs.data(), M * sizeof(nvc::verts::VertexJob) }, { base + o_order, order.data(), M * 4 } });
	if (e != cudaSuccess)
		return cuda_fail(ctx, e, "nvc_cook_mesh_vertices");

	nvc::VertexArgs a;
	a.vertices = vertices;
	a.indices = indices;
	a.jobs = reinterpret_cast<const nvc::verts::VertexJob*>(base + o_jobs);
	a.order = reinterpret_cast<const uint32_t*>(base + o_order);
	a.mesh_count = mesh_count;
	a.tri_count = uint32_t(T);
	a.position_count = uint32_t(N);
	a.slot_count = uint32_t(S);
	a.rejected = reinterpret_cast<uint8_t*>(base + o_rejected);
	a.tri_table = reinterpret_cast<uint32_t*>(base + o_tri_table);
	a.tri_mask = uint32_t(tri_buckets - 1);
	a.tri_entry = reinterpret_cast<uint32_t*>(base + o_tri_entry);
	a.flags = reinterpret_cast<uint8_t*>(base + o_flags);
	a.rank = reinterpret_cast<uint32_t*>(base + o_rank);
	a.block_sums = reinterpret_cast<uint32_t*>(base + o_sums);
	a.offsets = reinterpret_cast<unsigned long long*>(base + o_offsets);
	a.filtered = reinterpret_cast<uint32_t*>(base + o_filtered);
	a.index_base = reinterpret_cast<uint32_t*>(base + o_ibase);
	a.vertex_base = reinterpret_cast<uint32_t*>(base + o_vbase);
	a.first = reinterpret_cast<uint32_t*>(base + o_first);
	a.vtx_table = reinterpret_cast<uint32_t*>(base + o_vtx_table);
	a.vtx_first = reinterpret_cast<uint32_t*>(base + o_vtx_first);
	a.vtx_mask = uint32_t(vtx_buckets - 1);
	a.vtx_entry = reinterpret_cast<uint32_t*>(base + o_vtx_entry);
	a.classes = reinterpret_cast<NvcVertex*>(base + o_classes);
	a.remapped = reinterpret_cast<uint32_t*>(base + o_remapped);
	a.first_use = reinterpret_cast<uint32_t*>(base + o_first_use);
	a.scratch = reinterpret_cast<uint32_t*>(base + o_words);
	a.meshes = meshes;
	a.vertices_out = vertices_out;
	a.lod0_out = lod0_out;
	a.totals4 = totals4;
	e = nvc::launch_cook_mesh_vertices(a, static_cast<cudaStream_t>(stream));
	return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_cook_mesh_vertices");
}

namespace
{

// nvc_obj_load's scratch, in three parts, each planned once the counts it needs are known: the files and their line index;
// the per-line arrays (L line slots); the parsed arrays (the call's v / vt / vn lines, index records and faces).
struct ObjLayout
{
	size_t files, text, tile_lines, tile_offsets, part1;
	size_t state, line_end, counts, block_sums, block_offsets, prefix, infos, part2;
	size_t positions, texcoords, normals, records, faces, part3;
};

ObjLayout plan_obj(uint32_t file_count, uint64_t text_bytes, uint32_t tiles, uint64_t lines, const uint64_t* totals)
{
	using namespace nvc::obj;
	const uint64_t F = file_count, blocks = (lines + nvc::scan::kScanItems - 1) / nvc::scan::kScanItems;
	ObjLayout o;
	nvc::ScratchPlan sp;
	o.files = sp.take((F + 1) * sizeof(File));
	o.text = sp.take(text_bytes);
	o.tile_lines = sp.take(size_t(tiles) * 4);
	o.tile_offsets = sp.take((size_t(tiles) + 1) * 8);
	o.part1 = sp.bytes;
	o.state = sp.take(F * sizeof(FileState));
	o.line_end = sp.take(lines * 4);
	o.counts = sp.take(kFields * lines * 4);
	o.block_sums = sp.take(kFields * blocks * 4);
	o.block_offsets = sp.take(kFields * (blocks + 1) * 8);
	o.prefix = sp.take(kFields * (lines + 1) * 8);
	o.infos = sp.take(F * sizeof(NvcObjInfo));
	o.part2 = sp.bytes;
	o.positions = sp.take((totals[kPositions] + F) * 12);
	o.texcoords = sp.take((totals[kTexcoords] + F) * 8);
	o.normals = sp.take((totals[kNormals] + F) * 12);
	o.records = sp.take(totals[kRecords] * sizeof(Record));
	o.faces = sp.take(totals[kFaces] * sizeof(Face));
	o.part3 = sp.bytes;
	return o;
}

// fast_obj's arrays hold 32-bit sizes, and growing one rounds its capacity up to 16 elements
bool obj_arrays_fit(const NvcObjInfo& info)
{
	const uint64_t limit = 0xffffffffull - 15;
	return 3 * (uint64_t(info.position_count) + 1) <= limit && 2 * (uint64_t(info.texcoord_count) + 1) <= limit &&
	       3 * (uint64_t(info.normal_count) + 1) <= limit && info.index_count <= limit;
}

} // namespace

NVC_API int nvc_obj_load(NvcContext* ctx, void* stream, const NvcObjFile* files, uint32_t file_count, NvcVertex* vertices, uint64_t vertex_capacity,
    NvcObjInfo* infos)
{
	using namespace nvc::obj;
	if (!ctx || (file_count && (!files || !infos)) || (reinterpret_cast<uintptr_t>(vertices) & 15))
		return NVC_ERROR_INVALID_ARGUMENT;
	uint64_t size_sum = 0;
	for (uint32_t f = 0; f < file_count; ++f)
	{
		if (files[f].size && !files[f].data)
			return NVC_ERROR_INVALID_ARGUMENT;
		size_sum += std::min<uint64_t>(files[f].size, 1ull << 40);
	}
	if (!device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	if (file_count == 0)
		return NVC_OK;
	if (size_sum > 0xffffffffull)
		return NVC_ERROR_UNSUPPORTED; // line ends, index records and window starts are 32-bit

	std::vector<File> jobs(file_count + 1);
	uint64_t text_bytes = 0, tiles = 0;
	for (uint32_t f = 0; f < file_count; ++f)
	{
		jobs[f].data = text_bytes;
		jobs[f].size = uint32_t(files[f].size);
		jobs[f].tile_base = uint32_t(tiles);
		text_bytes += (files[f].size + 15) & ~15ull;
		tiles += (files[f].size + kTileBytes - 1) / kTileBytes;
	}
	jobs[file_count] = File{ text_bytes, 0, uint32_t(tiles) };

	const cudaStream_t s = static_cast<cudaStream_t>(stream);
	uint64_t lines = 0, totals[kFields] = {};
	std::vector<NvcObjInfo> info(file_count);
	std::vector<FileState> state(file_count);
	// a part that does not fit the scratch grows it, and the call starts over from the upload (at most twice)
	for (;;)
	{
		ObjLayout o = plan_obj(file_count, text_bytes, uint32_t(tiles), lines, totals);
		// the previous user of the scratch finishes first
		cudaError_t e = cudaDeviceSynchronize();
		if (e == cudaSuccess)
			e = nvc::reserve_scratch(ctx, o.part3); // the parts not planned yet are empty
		if (e != cudaSuccess)
			return nvc::load_fail(ctx, e, "nvc_obj_load");
		char* base = static_cast<char*>(ctx->load_scratch);
		nvc::ObjArgs a = {};
		a.text = reinterpret_cast<const uint8_t*>(base + o.text);
		a.files = reinterpret_cast<const File*>(base + o.files);
		a.file_count = file_count;
		a.tile_count = uint32_t(tiles);
		a.tile_lines = reinterpret_cast<uint32_t*>(base + o.tile_lines);
		a.tile_offsets = reinterpret_cast<unsigned long long*>(base + o.tile_offsets);
		e = cudaMemcpy(base + o.files, jobs.data(), jobs.size() * sizeof(File), cudaMemcpyHostToDevice);
		for (uint32_t f = 0; f < file_count && e == cudaSuccess; ++f)
			if (files[f].size)
				e = cudaMemcpy(base + o.text + jobs[f].data, files[f].data, files[f].size, cudaMemcpyHostToDevice);
		// a copy from pageable memory is not ordered with a non-blocking stream
		if (e == cudaSuccess)
			e = cudaDeviceSynchronize();
		if (e == cudaSuccess)
			e = nvc::launch_obj_lines(a, s);
		unsigned long long newlines = 0;
		if (e == cudaSuccess)
			e = cudaDeviceSynchronize();
		if (e == cudaSuccess)
			e = cudaMemcpy(&newlines, a.tile_offsets + tiles, 8, cudaMemcpyDeviceToHost);
		if (e != cudaSuccess)
			return cuda_fail(ctx, e, "nvc_obj_load");

		// part 2: one line slot per '\n', and one per file for a last line without one
		if (newlines + file_count > 0xffffffffull)
			return NVC_ERROR_UNSUPPORTED;
		lines = newlines + file_count;
		o = plan_obj(file_count, text_bytes, uint32_t(tiles), lines, totals);
		if (o.part2 > ctx->load_scratch_bytes)
			continue;
		a.line_slots = uint32_t(lines);
		a.line_end = reinterpret_cast<uint32_t*>(base + o.line_end);
		a.state = reinterpret_cast<FileState*>(base + o.state);
		a.counts = reinterpret_cast<uint32_t*>(base + o.counts);
		a.block_sums = reinterpret_cast<uint32_t*>(base + o.block_sums);
		a.block_offsets = reinterpret_cast<unsigned long long*>(base + o.block_offsets);
		a.prefix = reinterpret_cast<unsigned long long*>(base + o.prefix);
		a.infos = reinterpret_cast<NvcObjInfo*>(base + o.infos);
		e = nvc::launch_obj_count(a, s);
		if (e == cudaSuccess)
			e = cudaDeviceSynchronize();
		uint64_t now[kFields];
		for (uint32_t k = 0; k < kFields && e == cudaSuccess; ++k)
			e = cudaMemcpy(&now[k], a.prefix + uint64_t(k) * (lines + 1) + lines, 8, cudaMemcpyDeviceToHost);
		if (e == cudaSuccess)
			e = cudaMemcpy(info.data(), a.infos, file_count * sizeof(NvcObjInfo), cudaMemcpyDeviceToHost);
		if (e == cudaSuccess)
			e = cudaMemcpy(state.data(), a.state, file_count * sizeof(FileState), cudaMemcpyDeviceToHost);
		if (e != cudaSuccess)
			return cuda_fail(ctx, e, "nvc_obj_load");
		memcpy(infos, info.data(), file_count * sizeof(NvcObjInfo));
		bool fits = now[kCorners] <= 0xffffffffull;
		for (uint32_t f = 0; f < file_count; ++f)
			fits = fits && obj_arrays_fit(info[f]);
		if (!fits)
			return NVC_ERROR_UNSUPPORTED;
		for (uint32_t f = 0; f < file_count; ++f)
			if (state[f].flags & kBadFace)
				return NVC_ERROR_CORRUPT;

		// part 3: the parsed arrays
		memcpy(totals, now, sizeof(now));
		o = plan_obj(file_count, text_bytes, uint32_t(tiles), lines, totals);
		if (o.part3 > ctx->load_scratch_bytes)
			continue;
		a.positions = reinterpret_cast<float*>(base + o.positions);
		a.texcoords = reinterpret_cast<float*>(base + o.texcoords);
		a.normals = reinterpret_cast<float*>(base + o.normals);
		a.records = reinterpret_cast<Record*>(base + o.records);
		a.faces = reinterpret_cast<Face*>(base + o.faces);
		a.face_count = uint32_t(totals[kFaces]);
		a.corner_count = totals[kCorners];
		e = nvc::launch_obj_parse(a, s);
		if (e == cudaSuccess)
			e = cudaDeviceSynchronize();
		if (e == cudaSuccess)
			e = cudaMemcpy(state.data(), a.state, file_count * sizeof(FileState), cudaMemcpyDeviceToHost);
		if (e != cudaSuccess)
			return cuda_fail(ctx, e, "nvc_obj_load");
		for (uint32_t f = 0; f < file_count; ++f)
			if (state[f].flags & kBadIndex)
				return NVC_ERROR_CORRUPT;
		if (!vertices)
			return NVC_OK;
		if (vertex_capacity < a.corner_count)
			return NVC_ERROR_INVALID_ARGUMENT;
		a.vertices = vertices;
		e = nvc::launch_obj_expand(a, s);
		return e == cudaSuccess ? NVC_OK : cuda_fail(ctx, e, "nvc_obj_load");
	}
}
