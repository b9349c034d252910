// nvc_nccl.cpp — exchange of the per-rank visible slabs over NVLink with NCCL (new in this implementation: the
// reference is single-GPU, SURVEY.md §2.3).  libnccl is bound at run time with dlopen so that the library has
// no link-time NCCL dependency and, inside a PyTorch process, shares the libnccl.so.2 torch already loaded.
#include "nvc_internal.h"

#include <dlfcn.h>
#include <nccl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

namespace
{

struct NcclApi
{
	void* handle = nullptr;
	ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
	ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
	ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
	ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
	ncclResult_t (*GroupStart)() = nullptr;
	ncclResult_t (*GroupEnd)() = nullptr;
	const char* (*GetErrorString)(ncclResult_t) = nullptr;
	bool ok = false;
};

NcclApi& api()
{
	static NcclApi a;
	static bool tried = false;
	if (tried)
		return a;
	tried = true;
	const char* names[] = { getenv("NVC_NCCL_LIB"), "libnccl.so.2", "libnccl.so" };
	for (const char* n : names)
	{
		if (!n || !*n)
			continue;
		// RTLD_NOLOAD first: reuse the copy PyTorch (or the host app) has already mapped
		a.handle = dlopen(n, RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
		if (!a.handle)
			a.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
		if (a.handle)
			break;
	}
	if (!a.handle)
		return a;
#define NVC_SYM(field, name) a.field = reinterpret_cast<decltype(a.field)>(dlsym(a.handle, name))
	NVC_SYM(GetUniqueId, "ncclGetUniqueId");
	NVC_SYM(CommInitRank, "ncclCommInitRank");
	NVC_SYM(CommDestroy, "ncclCommDestroy");
	NVC_SYM(AllGather, "ncclAllGather");
	NVC_SYM(GroupStart, "ncclGroupStart");
	NVC_SYM(GroupEnd, "ncclGroupEnd");
	NVC_SYM(GetErrorString, "ncclGetErrorString");
#undef NVC_SYM
	a.ok = a.GetUniqueId && a.CommInitRank && a.CommDestroy && a.AllGather && a.GroupStart && a.GroupEnd && a.GetErrorString;
	return a;
}

int nccl_fail(NvcContext* ctx, ncclResult_t r, const char* what)
{
	if (ctx)
		ctx->last_error = std::string(what) + ": " + (api().GetErrorString ? api().GetErrorString(r) : "nccl error");
	return NVC_ERROR_NCCL;
}

} // namespace

namespace nvc
{

void nccl_destroy(NvcContext* ctx)
{
	if (ctx && ctx->nccl_comm && api().ok)
		api().CommDestroy(static_cast<ncclComm_t>(ctx->nccl_comm));
	if (ctx)
		ctx->nccl_comm = nullptr;
}

} // namespace nvc

extern "C"
{

static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");

NVC_API int nvc_nccl_unique_id(void* out_unique_id128)
{
	if (!out_unique_id128)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!api().ok)
		return NVC_ERROR_NCCL;
	ncclUniqueId id;
	ncclResult_t r = api().GetUniqueId(&id);
	if (r != ncclSuccess)
		return NVC_ERROR_NCCL;
	memcpy(out_unique_id128, &id, sizeof(id));
	return NVC_OK;
}

NVC_API int nvc_nccl_init(NvcContext* ctx, const void* unique_id128, int rank, int world_size)
{
	if (!ctx || !unique_id128 || world_size < 1 || rank < 0 || rank >= world_size)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!api().ok)
	{
		ctx->last_error = "libnccl.so.2 could not be loaded";
		return NVC_ERROR_NCCL;
	}
	cudaSetDevice(ctx->device);
	nvc::nccl_destroy(ctx);
	ncclUniqueId id;
	memcpy(&id, unique_id128, sizeof(id));
	ncclComm_t comm = nullptr;
	ncclResult_t r = api().CommInitRank(&comm, world_size, id, rank);
	if (r != ncclSuccess)
		return nccl_fail(ctx, r, "ncclCommInitRank");
	ctx->nccl_comm = comm;
	ctx->nccl_rank = rank;
	ctx->nccl_world = world_size;
	return NVC_OK;
}

NVC_API int nvc_allgather_visible(NvcContext* ctx, void* stream, const void* local_slab, size_t slab_bytes,
    const uint32_t* local_count4, void* gathered_slabs, uint32_t* gathered_count4)
{
	if (!ctx || !local_count4 || !gathered_count4 || (slab_bytes && (!local_slab || !gathered_slabs)))
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!ctx->nccl_comm)
	{
		ctx->last_error = "nvc_nccl_init has not been called";
		return NVC_ERROR_NCCL;
	}
	if (!nvc::device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	ncclComm_t comm = static_cast<ncclComm_t>(ctx->nccl_comm);
	cudaStream_t s = static_cast<cudaStream_t>(stream);
	// one fused group: the 16-byte counter blocks and the fixed-capacity slabs
	ncclResult_t r = api().GroupStart();
	if (r == ncclSuccess)
		r = api().AllGather(local_count4, gathered_count4, 16, ncclUint8, comm, s);
	if (r == ncclSuccess && slab_bytes)
		r = api().AllGather(local_slab, gathered_slabs, slab_bytes, ncclUint8, comm, s);
	ncclResult_t e = api().GroupEnd();
	if (r == ncclSuccess)
		r = e;
	return r == ncclSuccess ? NVC_OK : nccl_fail(ctx, r, "ncclAllGather");
}

} // extern "C"
