// nvc_peer.cu — all-gather of the per-rank visible command slabs over NVLink WITHOUT SMs: every rank pushes its slab
// and counters into every peer's gathered buffer with copy-engine peer copies (cudaMemcpyAsync on CUDA-IPC mapped
// memory, fanned out over a few side streams so several copy engines run at once), then raises a per-sender flag in
// the peer's memory; the receiver's stream blocks in a tiny spin kernel until all flags carry the current frame tag.
// Unlike an NCCL all-gather this needs no SMs, so it overlaps the (persistent, SM-filling) late cluster pass.
// One process per GPU; the IPC tickets are exchanged by the caller (any transport).
//
// Flow control (no barrier anywhere): the receive buffers are DOUBLE-BUFFERED by the parity of the frame tag, and every
// receiver acknowledges to every sender which frame it has finished with:
//   push(T)  waits (device side, on a side stream) until every peer has acknowledged frame T-2 — the previous user of the
//            parity-T&1 buffers — then copies into the peers' parity-T&1 slots and raises flag = T;
//   wait(T)  first tells every peer "I am done with frame T-1" (everything enqueued on `stream` before this call has read
//            it), then blocks `stream` until all flags carry T.  The gathered data of frame T stay valid until this rank
//            calls wait(T+1).
// A fast rank can therefore run at most one frame ahead of the slowest consumer of its data; nothing is overwritten
// while it may still be read.
#include "nvc_internal.h"

#include <stdlib.h>
#include <string.h>

namespace
{

constexpr int kMaxWorld = 64;
constexpr int kSideStreams = 8; // one per peer at 8 GPUs: independent copy engines

struct Ticket // what a rank publishes: IPC handles of its receive buffers (counts, flags and acks share one allocation)
{
	cudaIpcMemHandle_t slabs, counts, flags;
};
static_assert(sizeof(Ticket) == 192, "ticket is 3 x 64 bytes");

// layout of the small `flags` allocation (uint32 words): [0, kMaxWorld) data flags, [kMaxWorld, 2 kMaxWorld) acks
constexpr int kAckBase = 64;

// Every kernel of the protocol adds *epoch (a device word, 0 unless nvc_gather_graph_advance is used) to the tag it was launched
// with: a captured CUDA graph holds its tags as launch arguments, and each replay must speak of later frames than the one before.
__global__ void raise_flags_kernel(uint32_t* const* peer_flags, int world, int rank, uint32_t tag, const uint32_t* epoch)
{
	int p = threadIdx.x;
	if (p < world)
	{
		tag += *epoch;
		__threadfence_system();
		*reinterpret_cast<volatile uint32_t*>(peer_flags[p] + rank) = tag; // P2P store over NVLink (or local)
	}
}

// SM variant of the push: a few CTAs stream the VALID part of the local slab (count x 20 bytes, known only on the
// device) to every rank's slot with 16-byte peer stores.  Launched on a high-priority stream right before the late
// cluster pass so that its CTAs are placed first; the persistent cluster kernel fills the remaining slots.
__global__ void __launch_bounds__(256) push_kernel(const uint4* __restrict__ local_slab, const uint32_t* __restrict__ local_count4, uint8_t* const* peer_slabs,
    uint32_t* const* peer_counts, size_t slab_bytes, int world, int rank, uint32_t parity)
{
	const size_t slot = size_t(parity) * world + rank;
	const uint32_t count = local_count4[0];
	size_t bytes = size_t(count) * sizeof(NvcMeshTaskCommand);
	bytes = bytes < slab_bytes ? bytes : slab_bytes;
	const size_t n16 = (bytes + 15) / 16; // slab_bytes is a multiple of 64 commands = 1280 bytes, so rounding up stays inside
	const size_t stride = size_t(gridDim.x) * blockDim.x;
	for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n16; i += stride)
	{
		uint4 v = __ldg(local_slab + i);
		for (int k = 0; k < world; ++k)
		{
			int p = (rank + k) % world;
			reinterpret_cast<uint4*>(peer_slabs[p] + slot * slab_bytes)[i] = v;
		}
	}
	if (blockIdx.x == 0 && threadIdx.x < uint32_t(world))
	{
		uint4 c = *reinterpret_cast<const uint4*>(local_count4);
		*reinterpret_cast<uint4*>(peer_counts[threadIdx.x] + 4 * slot) = c;
	}
	__threadfence_system();
}

// tells every peer that this rank is done with frame `tag`: acks[rank] = tag in the peer's memory
__global__ void raise_acks_kernel(uint32_t* const* peer_flags, int world, int rank, uint32_t tag, const uint32_t* epoch)
{
	int p = threadIdx.x;
	if (p < world)
	{
		tag += *epoch;
		__threadfence_system();
		*reinterpret_cast<volatile uint32_t*>(peer_flags[p] + kAckBase + rank) = tag;
	}
}

// Multicast variant of the push: every 16-byte unit of the VALID part of the slab is stored ONCE, through the NVSwitch
// multicast alias of this rank's slot — the switch replicates it into every rank's gathered buffer (egress 1x instead
// of world x).  Same launch shape and placement as push_kernel.
__global__ void __launch_bounds__(256) mc_push_kernel(const uint4* __restrict__ local_slab, const uint32_t* __restrict__ local_count4, uint8_t* mc_slabs, uint32_t* mc_counts,
    size_t slab_bytes, int world, int rank, uint32_t parity, int with_slab)
{
	const size_t slot = size_t(parity) * world + rank;
	if (with_slab)
	{
		const uint32_t count = local_count4[0];
		size_t bytes = (size_t(count) + 63) / 64 * 64 * sizeof(NvcMeshTaskCommand); // the zero-padded group the consumer dispatches over
		bytes = bytes < slab_bytes ? bytes : slab_bytes;
		const size_t n16 = bytes / 16; // 64 commands = 1280 bytes: a multiple of 16
		const size_t stride = size_t(gridDim.x) * blockDim.x;
		uint4* dst = reinterpret_cast<uint4*>(mc_slabs + slot * slab_bytes);
		for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n16; i += stride)
			dst[i] = __ldg(local_slab + i);
	}
	if (blockIdx.x == 0 && threadIdx.x == 0)
		*reinterpret_cast<uint4*>(mc_counts + 4 * slot) = *reinterpret_cast<const uint4*>(local_count4);
	__threadfence_system();
}

// A peer that never answers (a crashed process, ranks that disagree about the frame they are in) must not hang this GPU for ever:
// after ~20 s (SM cycles) a wait gives up and marks the exchange DEAD (word 1 of `epoch`); every later wait returns at once and
// nvc_gather_status reports it.  The gathered data are then undefined; the caller decides what to do.
constexpr long long kSpinLimitCycles = 40000000000ll;

__global__ void wait_flags_kernel(const uint32_t* flags, int world, uint32_t tag, uint32_t* epoch)
{
	int q = threadIdx.x;
	if (q < world)
	{
		tag += epoch[0];
		volatile uint32_t* dead = epoch + 1;
		const long long t0 = clock64();
		// tags increase monotonically; signed distance handles wrap-around
		while (int32_t(*reinterpret_cast<const volatile uint32_t*>(flags + q) - tag) < 0)
		{
			if (*dead != 0u || clock64() - t0 > kSpinLimitCycles)
			{
				*dead = 1u;
				break;
			}
			__nanosleep(200);
		}
		__threadfence_system();
	}
}

__global__ void advance_epoch_kernel(uint32_t* epoch, uint32_t frames)
{
	*epoch += frames;
}

} // namespace

struct NvcGather
{
	int world = 1, rank = 0;
	size_t slab_bytes = 0;
	uint8_t* slabs = nullptr;   // [2][world][slab_bytes] receive buffers of this rank, indexed by tag parity
	uint32_t* counts = nullptr; // [2][world][4]
	uint32_t* flags = nullptr;  // [kMaxWorld] data flags + [kMaxWorld] acks
	uint8_t* peer_slabs[kMaxWorld] = {};
	uint32_t* peer_counts[kMaxWorld] = {};
	uint32_t* peer_flags[kMaxWorld] = {};
	uint32_t** d_peer_flags = nullptr; // device copy of peer_flags
	uint8_t** d_peer_slabs = nullptr;
	uint32_t** d_peer_counts = nullptr;
	cudaStream_t hi = nullptr; // high-priority stream of the SM push
	int mode = 0;              // 0 = copy engines, 1 = SM unicast push kernel, 2 = SM multicast push kernel, 3 = fused into drawcull
	bool attached = false;     // buffers live in a caller-owned symmetric region (nvc_gather_attach): never freed / closed here
	uint8_t* mc_slabs = nullptr;   // NVSwitch multicast aliases of the region (stores land in every rank's copy), or null
	uint32_t* mc_counts = nullptr;
	uint32_t fused_tag = 0;    // tag armed by nvc_gather_fuse_next_drawcull (0 = none)
	bool fused_consumed = false; // the armed late drawcull has been launched
	cudaStream_t side[kSideStreams] = {};
	cudaEvent_t fork = nullptr, join[kSideStreams] = {};
	uint32_t* count_stage = nullptr; // [2][4] snapshot of the local counters, by tag parity; word 8: the graph epoch (see advance_epoch_kernel), word 9: the "exchange dead" mark
	cudaEvent_t acked = nullptr;
	uint32_t tag = 0, acked_tag = 0;
	bool connected = false;
};

namespace nvc
{

// CTA slots the persistent cluster grid leaves free so that the exchange's kernels can run beside it: the one-block
// helpers (acknowledgement wait, flag raise) always; the 16-CTA push kernels of the SM / multicast transports too.
uint32_t gather_reserved_blocks(NvcContext* ctx)
{
	NvcGather* g = static_cast<NvcGather*>(ctx->gather);
	if (!g || !g->connected)
		return 0;
	return (g->mode == 1 || g->mode == 2) ? 18u : 2u;
}

uint32_t* gather_fused_target(NvcContext* ctx)
{
	NvcGather* g = static_cast<NvcGather*>(ctx->gather);
	if (!g || !g->connected || g->mode != 3 || !g->mc_slabs || g->fused_tag == 0 || g->fused_consumed)
		return nullptr;
	g->fused_consumed = true;
	const size_t slot = size_t(g->fused_tag & 1u) * size_t(g->world) + size_t(g->rank);
	return reinterpret_cast<uint32_t*>(g->mc_slabs + slot * g->slab_bytes);
}

void gather_destroy(NvcContext* ctx)
{
	NvcGather* g = static_cast<NvcGather*>(ctx->gather);
	if (!g)
		return;
	cudaSetDevice(ctx->device);
	cudaDeviceSynchronize();
	for (int p = 0; p < g->world; ++p)
		if (p != g->rank && g->connected && !g->attached)
		{
			if (g->peer_slabs[p])
				cudaIpcCloseMemHandle(g->peer_slabs[p]);
			if (g->peer_counts[p])
				cudaIpcCloseMemHandle(g->peer_counts[p]);
			if (g->peer_flags[p])
				cudaIpcCloseMemHandle(g->peer_flags[p]);
		}
	for (int i = 0; i < kSideStreams; ++i)
	{
		if (g->side[i])
			cudaStreamDestroy(g->side[i]);
		if (g->join[i])
			cudaEventDestroy(g->join[i]);
	}
	if (g->fork)
		cudaEventDestroy(g->fork);
	if (g->acked)
		cudaEventDestroy(g->acked);
	cudaFree(g->count_stage);
	if (!g->attached)
	{
		cudaFree(g->slabs);
		cudaFree(g->counts);
		cudaFree(g->flags);
	}
	cudaFree(g->d_peer_flags);
	cudaFree(g->d_peer_slabs);
	cudaFree(g->d_peer_counts);
	if (g->hi)
		cudaStreamDestroy(g->hi);
	delete g;
	ctx->gather = nullptr;
}

} // namespace nvc

extern "C"
{

NVC_API int nvc_gather_create(NvcContext* ctx, size_t slab_bytes, int rank, int world, void* ticket192_out)
{
	// slabs are moved in 16-byte units (and hold whole 64-command groups in the reference's sizing)
	if (!ctx || !ticket192_out || world < 1 || world > kMaxWorld || rank < 0 || rank >= world || slab_bytes == 0 || slab_bytes % 16 != 0)
		return NVC_ERROR_INVALID_ARGUMENT;
	int previous_device = -1;
	cudaGetDevice(&previous_device);
	cudaSetDevice(ctx->device);
	struct Restore
	{
		int d;
		~Restore()
		{
			if (d >= 0)
				cudaSetDevice(d);
		}
	} restore{ previous_device };
	nvc::gather_destroy(ctx);
	NvcGather* g = new NvcGather();
	g->world = world;
	g->rank = rank;
	g->slab_bytes = slab_bytes;
	cudaError_t e = cudaMalloc(&g->slabs, 2 * slab_bytes * world);
	if (e == cudaSuccess)
		e = cudaMalloc(&g->counts, 2 * sizeof(uint32_t) * 4 * world);
	if (e == cudaSuccess)
		e = cudaMalloc(&g->flags, sizeof(uint32_t) * 2 * kMaxWorld);
	if (e == cudaSuccess)
		e = cudaMalloc(&g->d_peer_flags, sizeof(uint32_t*) * kMaxWorld);
	if (e == cudaSuccess)
		e = cudaMalloc(&g->d_peer_slabs, sizeof(uint8_t*) * kMaxWorld);
	if (e == cudaSuccess)
		e = cudaMalloc(&g->d_peer_counts, sizeof(uint32_t*) * kMaxWorld);
	if (e == cudaSuccess)
	{
		int lo = 0, hi = 0;
		cudaDeviceGetStreamPriorityRange(&lo, &hi);
		e = cudaStreamCreateWithPriority(&g->hi, cudaStreamNonBlocking, hi);
	}
	if (const char* env = getenv("NVC_GATHER_MODE"))
		g->mode = (strcmp(env, "sm") == 0) ? 1 : 0;
	if (e == cudaSuccess)
		e = cudaMemset(g->counts, 0, 2 * sizeof(uint32_t) * 4 * world);
	if (e == cudaSuccess)
		e = cudaMemset(g->flags, 0, sizeof(uint32_t) * 2 * kMaxWorld);
	for (int i = 0; i < kSideStreams && e == cudaSuccess; ++i)
	{
		e = cudaStreamCreateWithFlags(&g->side[i], cudaStreamNonBlocking);
		if (e == cudaSuccess)
			e = cudaEventCreateWithFlags(&g->join[i], cudaEventDisableTiming);
	}
	if (e == cudaSuccess)
		e = cudaEventCreateWithFlags(&g->fork, cudaEventDisableTiming);
	if (e == cudaSuccess)
		e = cudaEventCreateWithFlags(&g->acked, cudaEventDisableTiming);
	if (e == cudaSuccess)
		e = cudaMalloc(&g->count_stage, 48);
	if (e == cudaSuccess)
		e = cudaMemset(g->count_stage, 0, 48);
	Ticket t;
	memset(&t, 0, sizeof(t));
	if (e == cudaSuccess)
		e = cudaIpcGetMemHandle(&t.slabs, g->slabs);
	if (e == cudaSuccess)
		e = cudaIpcGetMemHandle(&t.counts, g->counts);
	if (e == cudaSuccess)
		e = cudaIpcGetMemHandle(&t.flags, g->flags);
	if (e == cudaSuccess)
		e = cudaDeviceSynchronize();
	ctx->gather = g;
	if (e != cudaSuccess)
	{
		ctx->last_error = std::string("nvc_gather_create: ") + cudaGetErrorString(e);
		nvc::gather_destroy(ctx);
		return e == cudaErrorMemoryAllocation ? NVC_ERROR_OUT_OF_MEMORY : NVC_ERROR_CUDA;
	}
	memcpy(ticket192_out, &t, sizeof(t));
	return NVC_OK;
}

NVC_API int nvc_gather_connect(NvcContext* ctx, const void* all_tickets /* world x 192 bytes, rank order */)
{
	NvcGather* g = ctx ? static_cast<NvcGather*>(ctx->gather) : nullptr;
	if (!g || !all_tickets)
		return NVC_ERROR_INVALID_ARGUMENT;
	int previous_device = -1;
	cudaGetDevice(&previous_device);
	cudaSetDevice(ctx->device);
	struct Restore
	{
		int d;
		~Restore()
		{
			if (d >= 0)
				cudaSetDevice(d);
		}
	} restore{ previous_device };
	const Ticket* tickets = static_cast<const Ticket*>(all_tickets);
	cudaError_t e = cudaSuccess;
	for (int p = 0; p < g->world && e == cudaSuccess; ++p)
	{
		if (p == g->rank)
		{
			g->peer_slabs[p] = g->slabs;
			g->peer_counts[p] = g->counts;
			g->peer_flags[p] = g->flags;
			continue;
		}
		e = cudaIpcOpenMemHandle(reinterpret_cast<void**>(&g->peer_slabs[p]), tickets[p].slabs, cudaIpcMemLazyEnablePeerAccess);
		if (e == cudaSuccess)
			e = cudaIpcOpenMemHandle(reinterpret_cast<void**>(&g->peer_counts[p]), tickets[p].counts, cudaIpcMemLazyEnablePeerAccess);
		if (e == cudaSuccess)
			e = cudaIpcOpenMemHandle(reinterpret_cast<void**>(&g->peer_flags[p]), tickets[p].flags, cudaIpcMemLazyEnablePeerAccess);
	}
	if (e == cudaSuccess)
		e = cudaMemcpy(g->d_peer_flags, g->peer_flags, sizeof(uint32_t*) * g->world, cudaMemcpyHostToDevice);
	if (e == cudaSuccess)
		e = cudaMemcpy(g->d_peer_slabs, g->peer_slabs, sizeof(uint8_t*) * g->world, cudaMemcpyHostToDevice);
	if (e == cudaSuccess)
		e = cudaMemcpy(g->d_peer_counts, g->peer_counts, sizeof(uint32_t*) * g->world, cudaMemcpyHostToDevice);
	if (e != cudaSuccess)
	{
		ctx->last_error = std::string("nvc_gather_connect: ") + cudaGetErrorString(e);
		// close whatever was opened: a half-connected gather is not usable and must not leak the mappings
		for (int p = 0; p < g->world; ++p)
			if (p != g->rank)
			{
				if (g->peer_slabs[p])
					cudaIpcCloseMemHandle(g->peer_slabs[p]);
				if (g->peer_counts[p])
					cudaIpcCloseMemHandle(g->peer_counts[p]);
				if (g->peer_flags[p])
					cudaIpcCloseMemHandle(g->peer_flags[p]);
				g->peer_slabs[p] = nullptr;
				g->peer_counts[p] = nullptr;
				g->peer_flags[p] = nullptr;
			}
		return NVC_ERROR_CUDA;
	}
	g->connected = true;
	return NVC_OK;
}

// Enqueues (after everything already on `stream`): push of local_slab / local_count4 into slot `rank` of every rank's
// gathered buffers (parity of the new frame tag) over the side streams, then the flag raise.  Returns immediately;
// `stream` itself is not blocked by the copies (call nvc_gather_wait on the stream that consumes the gathered data).
// local_count4 is snapshotted on `stream` right here; local_slab must stay unchanged until nvc_gather_wait.
NVC_API int nvc_gather_push(NvcContext* ctx, void* stream, const void* local_slab, const uint32_t* local_count4)
{
	NvcGather* g = ctx ? static_cast<NvcGather*>(ctx->gather) : nullptr;
	if (!g || !g->connected || !local_slab || !local_count4)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!nvc::device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	cudaStream_t s = static_cast<cudaStream_t>(stream);
	// fused mode: the tag was taken (and the peers' acknowledgements awaited) by nvc_gather_fuse_next_drawcull, and the slab
	// has already travelled inside the late drawcull — only the counters and the flags are left
	const bool fused = g->mode == 3 && g->fused_tag != 0 && g->fused_consumed;
	if (g->mode == 3 && !fused)
	{
		ctx->last_error = "nvc_gather_push in fused mode needs nvc_gather_fuse_next_drawcull + the late nvc_drawcull before it";
		return NVC_ERROR_INVALID_ARGUMENT;
	}
	if (!fused)
		g->tag += 1;
	g->fused_tag = 0;
	g->fused_consumed = false;
	const uint32_t tag = g->tag;
	const size_t parity = tag & 1u;
	const size_t slot = parity * size_t(g->world) + size_t(g->rank); // this rank's slot in every receiver's buffers
	uint32_t* count_stage = g->count_stage + 4 * parity;
	// the counters are snapshotted in stream order: later passes on `stream` may rewrite local_count4 at once
	cudaError_t e = cudaMemcpyAsync(count_stage, local_count4, 16, cudaMemcpyDeviceToDevice, s);
	if (e == cudaSuccess)
		e = cudaEventRecord(g->fork, s);
	cudaStream_t lead = g->mode >= 1 ? g->hi : g->side[0];
	if (e == cudaSuccess)
		e = cudaStreamWaitEvent(lead, g->fork, 0);
	if (e == cudaSuccess && tag >= 3 && !fused)
	{
		// the parity buffers were last used by frame tag-2: every peer must have acknowledged it
		wait_flags_kernel<<<1, kMaxWorld, 0, lead>>>(g->flags + kAckBase, g->world, tag - 2, g->count_stage + 8);
		e = cudaGetLastError();
	}
	if (g->mode >= 1 && e == cudaSuccess)
	{
		// SM push: one kernel on the high-priority stream, then the flag raise behind it
		if (g->mode == 1)
			push_kernel<<<16, 256, 0, g->hi>>>(static_cast<const uint4*>(local_slab), count_stage, g->d_peer_slabs, g->d_peer_counts, g->slab_bytes, g->world, g->rank, uint32_t(parity));
		else
			mc_push_kernel<<<fused ? 1 : 16, 256, 0, g->hi>>>(static_cast<const uint4*>(local_slab), count_stage, g->mc_slabs, g->mc_counts, g->slab_bytes, g->world, g->rank, uint32_t(parity), fused ? 0 : 1);
		e = cudaGetLastError();
		if (e == cudaSuccess)
		{
			raise_flags_kernel<<<1, kMaxWorld, 0, g->hi>>>(g->d_peer_flags, g->world, g->rank, tag, g->count_stage + 8);
			e = cudaGetLastError();
		}
		if (e == cudaSuccess)
			e = cudaEventRecord(g->join[0], g->hi);
		if (e != cudaSuccess)
		{
			ctx->last_error = std::string("nvc_gather_push: ") + cudaGetErrorString(e);
			return NVC_ERROR_CUDA;
		}
		return NVC_OK;
	}
	if (e == cudaSuccess)
		e = cudaEventRecord(g->acked, g->side[0]);
	for (int i = 1; i < kSideStreams && e == cudaSuccess; ++i)
		e = cudaStreamWaitEvent(g->side[i], g->acked, 0);
	for (int k = 0; k < g->world && e == cudaSuccess; ++k)
	{
		int p = (g->rank + k) % g->world; // stagger the targets so that ranks do not all hit the same peer first
		cudaStream_t ss = g->side[k % kSideStreams];
		e = cudaMemcpyAsync(g->peer_slabs[p] + slot * g->slab_bytes, local_slab, g->slab_bytes, cudaMemcpyDeviceToDevice, ss);
		if (e == cudaSuccess)
			e = cudaMemcpyAsync(g->peer_counts[p] + 4 * slot, count_stage, 16, cudaMemcpyDeviceToDevice, ss);
	}
	// flags go out once every copy of this rank has completed: join the side streams on side[0], raise there
	for (int i = 1; i < kSideStreams && e == cudaSuccess; ++i)
	{
		e = cudaEventRecord(g->join[i], g->side[i]);
		if (e == cudaSuccess)
			e = cudaStreamWaitEvent(g->side[0], g->join[i], 0);
	}
	if (e == cudaSuccess)
	{
		raise_flags_kernel<<<1, kMaxWorld, 0, g->side[0]>>>(g->d_peer_flags, g->world, g->rank, tag, g->count_stage + 8);
		e = cudaGetLastError();
	}
	if (e == cudaSuccess)
		e = cudaEventRecord(g->join[0], g->side[0]);
	if (e != cudaSuccess)
	{
		ctx->last_error = std::string("nvc_gather_push: ") + cudaGetErrorString(e);
		return NVC_ERROR_CUDA;
	}
	return NVC_OK;
}

// For the latest push (frame tag T): acknowledges frame T-1 to every peer (all work enqueued on `stream` so far has
// read it), then blocks `stream` (device side) until every rank's slab of frame T has landed in this rank's gathered
// buffers and this rank's own outgoing copies are done (so the local slab may be overwritten by the next pass).
// The gathered buffers of frame T (nvc_gather_buffers) stay valid until the next nvc_gather_wait.
NVC_API int nvc_gather_wait(NvcContext* ctx, void* stream)
{
	NvcGather* g = ctx ? static_cast<NvcGather*>(ctx->gather) : nullptr;
	if (!g || !g->connected)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!nvc::device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	cudaStream_t s = static_cast<cudaStream_t>(stream);
	cudaError_t e = cudaSuccess;
	if (g->tag >= 2 && g->acked_tag != g->tag - 1)
	{
		raise_acks_kernel<<<1, kMaxWorld, 0, s>>>(g->d_peer_flags, g->world, g->rank, g->tag - 1, g->count_stage + 8);
		e = cudaGetLastError();
		g->acked_tag = g->tag - 1;
	}
	if (e == cudaSuccess)
		e = cudaStreamWaitEvent(s, g->join[0], 0);
	if (e == cudaSuccess)
	{
		wait_flags_kernel<<<1, kMaxWorld, 0, s>>>(g->flags, g->world, g->tag, g->count_stage + 8);
		e = cudaGetLastError();
	}
	if (e != cudaSuccess)
	{
		ctx->last_error = std::string("nvc_gather_wait: ") + cudaGetErrorString(e);
		return NVC_ERROR_CUDA;
	}
	return NVC_OK;
}

NVC_API int nvc_gather_set_mode(NvcContext* ctx, int mode)
{
	NvcGather* g = ctx ? static_cast<NvcGather*>(ctx->gather) : nullptr;
	if (!g || mode < 0 || mode > 3)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (mode >= 2 && !g->mc_slabs)
	{
		ctx->last_error = "multicast transports need nvc_gather_attach with a multicast mapping";
		return NVC_ERROR_UNSUPPORTED;
	}
	if (mode == 0 && g->attached)
	{
		ctx->last_error = "the copy-engine transport needs nvc_gather_create / nvc_gather_connect buffers";
		return NVC_ERROR_UNSUPPORTED;
	}
	g->mode = mode;
	g->fused_tag = 0;
	g->fused_consumed = false;
	return NVC_OK;
}

// ---- symmetric-memory attachment: NVSwitch multicast ------------------------------------------------------------------------
// Layout of the region every rank allocates (identically) with a symmetric allocator:
//   [2][world][slab_bytes] slabs | [2][world][4] u32 counters | [2 x 64] u32 flags + acknowledgements
static size_t region_counts_offset(size_t slab_bytes, int world) { return 2 * slab_bytes * size_t(world); }
static size_t region_flags_offset(size_t slab_bytes, int world) { return region_counts_offset(slab_bytes, world) + 2 * 16 * size_t(world); }

NVC_API size_t nvc_gather_region_bytes(size_t slab_bytes, int world_size)
{
	if (world_size < 1 || world_size > kMaxWorld || slab_bytes == 0 || slab_bytes % 16 != 0)
		return 0;
	return region_flags_offset(slab_bytes, world_size) + sizeof(uint32_t) * 2 * kMaxWorld;
}

NVC_API int nvc_gather_attach(NvcContext* ctx, size_t slab_bytes, int rank, int world, void* const* peer_regions, void* multicast_region)
{
	if (!ctx || !peer_regions || world < 1 || world > kMaxWorld || rank < 0 || rank >= world || nvc_gather_region_bytes(slab_bytes, world) == 0)
		return NVC_ERROR_INVALID_ARGUMENT;
	for (int p = 0; p < world; ++p)
		if (!peer_regions[p] || (reinterpret_cast<uintptr_t>(peer_regions[p]) & 15u))
			return NVC_ERROR_INVALID_ARGUMENT;
	if (!nvc::device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	nvc::gather_destroy(ctx);
	NvcGather* g = new NvcGather();
	g->world = world;
	g->rank = rank;
	g->slab_bytes = slab_bytes;
	g->attached = true;
	const size_t co = region_counts_offset(slab_bytes, world), fo = region_flags_offset(slab_bytes, world);
	for (int p = 0; p < world; ++p)
	{
		uint8_t* base = static_cast<uint8_t*>(peer_regions[p]);
		g->peer_slabs[p] = base;
		g->peer_counts[p] = reinterpret_cast<uint32_t*>(base + co);
		g->peer_flags[p] = reinterpret_cast<uint32_t*>(base + fo);
	}
	g->slabs = g->peer_slabs[rank];
	g->counts = g->peer_counts[rank];
	g->flags = g->peer_flags[rank];
	if (multicast_region)
	{
		g->mc_slabs = static_cast<uint8_t*>(multicast_region);
		g->mc_counts = reinterpret_cast<uint32_t*>(g->mc_slabs + co);
	}
	cudaError_t e = cudaMalloc(&g->d_peer_flags, sizeof(uint32_t*) * kMaxWorld);
	if (e == cudaSuccess)
		e = cudaMalloc(&g->d_peer_slabs, sizeof(uint8_t*) * kMaxWorld);
	if (e == cudaSuccess)
		e = cudaMalloc(&g->d_peer_counts, sizeof(uint32_t*) * kMaxWorld);
	if (e == cudaSuccess)
		e = cudaMalloc(&g->count_stage, 48);
	if (e == cudaSuccess)
		e = cudaMemset(g->count_stage, 0, 48);
	if (e == cudaSuccess)
	{
		int lo = 0, hi = 0;
		cudaDeviceGetStreamPriorityRange(&lo, &hi);
		e = cudaStreamCreateWithPriority(&g->hi, cudaStreamNonBlocking, hi);
	}
	for (int i = 0; i < kSideStreams && e == cudaSuccess; ++i)
	{
		e = cudaStreamCreateWithFlags(&g->side[i], cudaStreamNonBlocking);
		if (e == cudaSuccess)
			e = cudaEventCreateWithFlags(&g->join[i], cudaEventDisableTiming);
	}
	if (e == cudaSuccess)
		e = cudaEventCreateWithFlags(&g->fork, cudaEventDisableTiming);
	if (e == cudaSuccess)
		e = cudaEventCreateWithFlags(&g->acked, cudaEventDisableTiming);
	// this rank clears ITS OWN counters / flags / acknowledgements; the caller barriers before the first push
	if (e == cudaSuccess)
		e = cudaMemset(g->counts, 0, 2 * 16 * size_t(world));
	if (e == cudaSuccess)
		e = cudaMemset(g->flags, 0, sizeof(uint32_t) * 2 * kMaxWorld);
	if (e == cudaSuccess)
		e = cudaMemcpy(g->d_peer_flags, g->peer_flags, sizeof(uint32_t*) * world, cudaMemcpyHostToDevice);
	if (e == cudaSuccess)
		e = cudaMemcpy(g->d_peer_slabs, g->peer_slabs, sizeof(uint8_t*) * world, cudaMemcpyHostToDevice);
	if (e == cudaSuccess)
		e = cudaMemcpy(g->d_peer_counts, g->peer_counts, sizeof(uint32_t*) * world, cudaMemcpyHostToDevice);
	if (e == cudaSuccess)
		e = cudaDeviceSynchronize();
	ctx->gather = g;
	if (e != cudaSuccess)
	{
		ctx->last_error = std::string("nvc_gather_attach: ") + cudaGetErrorString(e);
		nvc::gather_destroy(ctx);
		return e == cudaErrorMemoryAllocation ? NVC_ERROR_OUT_OF_MEMORY : NVC_ERROR_CUDA;
	}
	g->connected = true;
	g->mode = g->mc_slabs ? 2 : 1; // multicast push when the mapping exists, unicast SM push otherwise
	return NVC_OK;
}

// Fused all-gather: takes the next frame tag, blocks `stream` until every peer has acknowledged the previous user of that
// parity's buffers, and arms the NEXT late task-mode nvc_drawcull of this context: that launch stores its commands to the
// local buffer AND through the multicast mapping into every rank's gathered slab.  Follow with nvc_gather_push (sends the
// counters and raises the flags only) and nvc_gather_wait as usual.
NVC_API int nvc_gather_fuse_next_drawcull(NvcContext* ctx, void* stream)
{
	NvcGather* g = ctx ? static_cast<NvcGather*>(ctx->gather) : nullptr;
	if (!g || !g->connected || g->mode != 3 || !g->mc_slabs)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!nvc::device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	if (g->fused_tag != 0)
	{
		ctx->last_error = "nvc_gather_fuse_next_drawcull: the previous armed frame has not been pushed";
		return NVC_ERROR_INVALID_ARGUMENT;
	}
	g->tag += 1;
	g->fused_tag = g->tag;
	g->fused_consumed = false;
	if (g->tag >= 3)
	{
		wait_flags_kernel<<<1, kMaxWorld, 0, static_cast<cudaStream_t>(stream)>>>(g->flags + kAckBase, g->world, g->tag - 2, g->count_stage + 8);
		cudaError_t e = cudaGetLastError();
		if (e != cudaSuccess)
		{
			ctx->last_error = std::string("nvc_gather_fuse_next_drawcull: ") + cudaGetErrorString(e);
			return NVC_ERROR_CUDA;
		}
	}
	return NVC_OK;
}

// CUDA-graph replay of frames that contain the exchange.  The calls above bake the frame tags they took at capture time into the
// graph; enqueue this as the LAST operation of the captured sequence with `frames` = the number of nvc_gather_push calls captured
// (even: the receive buffers alternate by tag parity and their addresses are baked too).  Every replay then advances all tags of
// the next replay by `frames`.  Each captured push needs its nvc_gather_wait inside the same capture, and all ranks must replay
// the same graphs the same number of times.
NVC_API int nvc_gather_graph_advance(NvcContext* ctx, void* stream, uint32_t frames)
{
	NvcGather* g = ctx ? static_cast<NvcGather*>(ctx->gather) : nullptr;
	if (!g || !g->connected || frames == 0 || (frames & 1u))
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!nvc::device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	advance_epoch_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(g->count_stage + 8, frames);
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess)
	{
		ctx->last_error = std::string("nvc_gather_graph_advance: ") + cudaGetErrorString(e);
		return NVC_ERROR_CUDA;
	}
	return NVC_OK;
}

// 1 in *timed_out when a wait of this context has given up (see wait_flags_kernel); synchronises the device.
NVC_API int nvc_gather_status(NvcContext* ctx, int* timed_out)
{
	NvcGather* g = ctx ? static_cast<NvcGather*>(ctx->gather) : nullptr;
	if (!g || !timed_out)
		return NVC_ERROR_INVALID_ARGUMENT;
	if (!nvc::device_is_current(ctx))
		return NVC_ERROR_INVALID_ARGUMENT;
	uint32_t v = 0;
	cudaError_t e = cudaMemcpy(&v, g->count_stage + 9, sizeof(v), cudaMemcpyDeviceToHost);
	if (e != cudaSuccess)
	{
		ctx->last_error = std::string("nvc_gather_status: ") + cudaGetErrorString(e);
		return NVC_ERROR_CUDA;
	}
	*timed_out = v != 0u;
	return NVC_OK;
}

NVC_API int nvc_gather_buffers(NvcContext* ctx, void** gathered_slabs, uint32_t** gathered_count4)
{
	NvcGather* g = ctx ? static_cast<NvcGather*>(ctx->gather) : nullptr;
	if (!g)
		return NVC_ERROR_INVALID_ARGUMENT;
	// the buffers of the latest frame (parity of its tag); valid between nvc_gather_wait and the next nvc_gather_wait
	const size_t parity = g->tag & 1u;
	if (gathered_slabs)
		*gathered_slabs = g->slabs + parity * size_t(g->world) * g->slab_bytes;
	if (gathered_count4)
		*gathered_count4 = g->counts + parity * size_t(g->world) * 4;
	return NVC_OK;
}

} // extern "C"
