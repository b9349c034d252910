/*
 * niagara_cull.h — C ABI of the H100-native visibility path for zeux/niagara.
 *
 * This library replaces the Vulkan compute dispatches of niagara's GPU-driven visibility path
 * (reference call sites, all in src/niagara.cpp):
 *
 *   cull lambda      niagara.cpp:1530-1574   drawcull.comp (+ tasksubmit.comp)    -> nvc_drawcull
 *   render lambda    niagara.cpp:1582-1610   clustercull.comp + clustersubmit.comp -> nvc_clustercull
 *   pyramid lambda   niagara.cpp:1703-1733   depthreduce.comp, one dispatch / mip  -> nvc_depth_pyramid
 *   task-shader path niagara.cpp:1666-1679   meshlet.task.glsl (payload variant)   -> nvc_taskcull
 *
 * with hand-written sm_90a CUDA kernels.  The buffer contract (struct layouts, counters, padding,
 * overflow behaviour) is the reference's, bit for bit, so the outputs can be consumed by the existing
 * indirect-draw path (vkCmdDrawIndexedIndirectCount / vkCmdDrawMeshTasksIndirectEXT) unchanged.
 *
 * Conventions
 *   - plain C, no CUDA or torch types in signatures: streams are passed as void* (a cudaStream_t),
 *     device buffers as plain pointers to the structs below.
 *   - every pass call only ENQUEUES work on `stream`; no allocation, no synchronisation, safe to capture
 *     into a CUDA graph.  A context is not re-entrant (the reference's frame loop is single threaded): its passes
 *     share device-side ticket counters, so the passes of ONE context must be ordered — same stream, or streams
 *     ordered by events; use one context per concurrently running frame.  The context's device must be the calling
 *     thread's current CUDA device for pass calls (else NVC_ERROR_INVALID_ARGUMENT); nvc_create makes `device` current
 *     and leaves it so, the other lifetime calls restore the caller's device.
 *   - return value: 0 = NVC_OK, negative = NvcStatus error.  Capacity overflow (TASK_WGLIMIT /
 *     CLUSTER_LIMIT) is NOT an error: it is the reference's defined drop-and-clamp behaviour.
 *   - all struct layouts below are asserted (size/offset) against src/shaders/mesh.h + src/scene.h.
 */
#ifndef NIAGARA_CULL_H
#define NIAGARA_CULL_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#define NVC_API __declspec(dllexport)
#else
#define NVC_API __attribute__((visibility("default")))
#endif

/* ---- limits: src/config.h:1-28 ------------------------------------------------------------ */
#define NVC_TASK_WGSIZE 64u           /* config.h:2  meshlets per task command / cluster-cull group  */
#define NVC_TASK_WGLIMIT (1u << 22)   /* config.h:25 max task commands                               */
#define NVC_CLUSTER_LIMIT (1u << 24)  /* config.h:28 max visible cluster indices                     */
#define NVC_CLUSTER_TILE 16u          /* config.h:22 X dimension of the 16 x Y x 16 mesh dispatch    */
#define NVC_MAX_DISPATCH_GROUPS 65535u /* tasksubmit.comp.glsl:36, clustersubmit.comp.glsl:37       */
#define NVC_MAX_LODS 8u               /* mesh.h:77   Mesh::lods[8]                                   */
#define NVC_MAX_HIZ_LEVELS 16u        /* sampler maxLod 16 (resources.cpp:306)                       */

/* ---- data layouts: src/shaders/mesh.h:11-123 == src/scene.h:10-93 == src/niagara.cpp:227-260 ---- */

/* mesh.h:11-24 / scene.h:10-23 — 24 B, 8-byte aligned.  Cull reads bytes 0..11 only. */
typedef struct NvcMeshlet
{
	uint16_t center[3]; /* IEEE binary16 */
	uint16_t radius;    /* IEEE binary16 */
	int8_t cone_axis[3];
	int8_t cone_cutoff;
	uint32_t dataOffset;
	uint32_t baseVertex;
	uint8_t vertexCount;
	uint8_t triangleCount;
	uint8_t shortRefs;
	uint8_t padding;
} NvcMeshlet;

/* mesh.h:53-60 / scene.h:68-75 — 20 B */
typedef struct NvcMeshLod
{
	uint32_t indexOffset;
	uint32_t indexCount;
	uint32_t meshletOffset;
	uint32_t meshletCount;
	float error;
} NvcMeshLod;

/* mesh.h:62-78 / scene.h:77-93 — 208 B, 16-byte aligned */
typedef struct NvcMesh
{
	float center[3];
	float radius;
	uint32_t vertexOffset;
	uint32_t vertexCount;
	uint32_t ommIndexData;
	uint32_t ommIndexBase;
	uint32_t lodCount;
	uint32_t lodRT;
	uint32_t padding[2];
	NvcMeshLod lods[NVC_MAX_LODS];
} NvcMesh;

/* mesh.h:92-102 / scene.h:39-49 — 48 B, 16-byte aligned; orientation stored x,y,z,w */
typedef struct NvcMeshDraw
{
	float position[3];
	float scale;
	float orientation[4];
	uint32_t meshIndex;
	uint32_t meshletVisibilityOffset;
	uint32_t postPass;
	uint32_t materialIndex;
} NvcMeshDraw;

/* mesh.h:104-114 / niagara.cpp:227-231 — 24 B: drawId + VkDrawIndexedIndirectCommand */
typedef struct NvcMeshDrawCommand
{
	uint32_t drawId;
	uint32_t indexCount;
	uint32_t instanceCount;
	uint32_t firstIndex;
	uint32_t vertexOffset;
	uint32_t firstInstance;
} NvcMeshDrawCommand;

/* mesh.h:116-123 / niagara.cpp:233-240 — 20 B */
typedef struct NvcMeshTaskCommand
{
	uint32_t drawId;
	uint32_t taskOffset;
	uint32_t taskCount;
	uint32_t lateDrawVisibility;
	uint32_t meshletVisibilityOffset;
} NvcMeshTaskCommand;

/* mesh.h:26-44 / niagara.cpp:242-260 — 144 B (alignas 16), passed verbatim (the reference's push constants) */
typedef struct NvcCullData
{
	float view[16]; /* column-major mat4 */
	float P00, P11, znear, zfar;
	float frustum[4];
	float lodTarget;
	float pyramidWidth, pyramidHeight;
	uint32_t drawCount;
	int32_t cullingEnabled;
	int32_t lodEnabled;
	int32_t occlusionEnabled;
	int32_t clusterOcclusionEnabled;
	int32_t clusterBackfaceEnabled;
	uint32_t postPass;
	uint32_t pad_[2];
} NvcCullData;

/* mesh.h:125-128 — task-shader payload (meshlet.task.glsl:47) */
typedef struct NvcMeshTaskPayload
{
	uint32_t clusterIndices[NVC_TASK_WGSIZE];
} NvcMeshTaskPayload;

/* Depth pyramid ("depthPyramid" image, niagara.cpp:1339-1350): R32F, width x height = previousPow2 of the
 * depth target, full mip chain.  In place of a VkImage: one linear device allocation, level l stored
 * row-major and tightly packed at texels + level_offset[l], size max(1,width>>l) x max(1,height>>l). */
typedef struct NvcHiZ
{
	float* texels; /* device pointer */
	uint32_t width, height, levels;
	uint32_t level_offset[NVC_MAX_HIZ_LEVELS]; /* in texels */
	uint32_t total_texels;
} NvcHiZ;

typedef struct NvcLimits
{
	uint32_t task_wglimit;  /* default NVC_TASK_WGLIMIT  */
	uint32_t cluster_limit; /* default NVC_CLUSTER_LIMIT */
} NvcLimits;

typedef enum NvcStatus
{
	NVC_OK = 0,
	NVC_ERROR_INVALID_ARGUMENT = -1,
	NVC_ERROR_CUDA = -2,
	NVC_ERROR_NO_DEVICE = -3,
	NVC_ERROR_OUT_OF_MEMORY = -4,
	NVC_ERROR_NCCL = -5,
	NVC_ERROR_UNSUPPORTED = -6, /* valid input this build has no decoder for (see nvc_scene_cache_read) */
	NVC_ERROR_CORRUPT = -7      /* a scene cache whose sections do not add up */
} NvcStatus;

typedef struct NvcContext NvcContext;

/* ---- lifetime -------------------------------------------------------------------------------- */

/* Replaces pipeline/program creation for the cull path (niagara.cpp:652-762).  `limits` may be NULL. */
NVC_API int nvc_create(int device, const NvcLimits* limits, NvcContext** out_ctx);
NVC_API void nvc_destroy(NvcContext* ctx);
NVC_API const char* nvc_status_string(int status);
/* last CUDA error text recorded by this context (for NVC_ERROR_CUDA) */
NVC_API const char* nvc_last_error(const NvcContext* ctx);
NVC_API const char* nvc_version(void);

/* Optional, once per geometry upload (where the reference uploads `mb`, niagara.cpp:1040-1046): builds a context-owned,
 * read-only cull view of Mesh[] — a 32-byte head per mesh {center, radius, lodCount, lods[0].meshletOffset/Count,
 * vertexOffset} plus the 8 LOD errors — so that nvc_drawcull touches ONE 32-byte sector per draw for single-LOD / LOD-0
 * task draws instead of the 3-4 sectors the 208-byte AoS record spreads those fields over.  Used automatically by
 * nvc_drawcull calls that pass the same `meshes` pointer; results are identical.  The Mesh[] contents must not change
 * afterwards (call again after re-uploading; meshes = NULL releases the view). */
NVC_API int nvc_prepare_meshes(NvcContext* ctx, void* stream, const NvcMesh* meshes, uint32_t mesh_count);

/* Optional, once per geometry upload (where the reference uploads `mlb`, niagara.cpp:1055, next to nvc_prepare_meshes):
 * builds a context-owned, read-only cull view of Meshlet[] — exact copies of the 12 bytes the cluster tests read, as two dense
 * arrays: bytes 0-7 of every record (center[3], radius) and bytes 8-11 (cone_axis[3], cone_cutoff).  nvc_clustercull and
 * nvc_taskcull calls that pass the same `meshlets` pointer then read 12 bytes per meshlet as two coalesced streams instead of
 * the 24-byte records; any other pointer reads the records.  Results are identical.  The Meshlet[] contents must not change
 * afterwards (call again after re-uploading; meshlets = NULL releases the view).  Allocates / frees: call outside stream
 * capture. */
NVC_API int nvc_prepare_meshlets(NvcContext* ctx, void* stream, const NvcMeshlet* meshlets, uint32_t meshlet_count);

/* Tuning: stage the coarse tail of the depth pyramid (top mips, at most `texels` texels, capped at 11264 = 44 KB) into
 * shared memory once per CTA of the late cluster pass with one TMA bulk copy (cp.async.bulk, SASS UBLKCP); lookups
 * whose whole warp samples a staged mip then read shared memory.  0 (default) disables it: on the measured workloads
 * the shared-memory carve-out costs more L1 hit rate on the fine mips than the staged mips save (DESIGN.md §5).
 * Results are identical either way.  Also settable with the environment variable NVC_HIZ_STAGE_TEXELS. */
NVC_API int nvc_set_hiz_staging(NvcContext* ctx, uint32_t texels);

/* Derived, optional, results identical (like nvc_prepare_meshes): allocates a context-owned FOOTPRINT IMAGE for this pyramid
 * (same texel count + one row / column per mip).  nvc_depth_pyramid then also writes, for every mip and every 2 x 2 sampler
 * footprint, the minimum of its four (edge-clamped) texels; the late cluster pass reads ONE value per meshlet instead of four
 * scattered texels.  The image is valid only for pyramids written by nvc_depth_pyramid: a caller that stores texels itself must
 * not prepare (or must pass NULL here to release).  Allocates / frees: call outside stream capture.  hiz == NULL releases. */
NVC_API int nvc_prepare_hiz(NvcContext* ctx, const NvcHiZ* hiz);
/* Diagnostics / tests: the device pointer of the footprint image, its first mip (mips below it have no image), the entry offset of
 * every mip (offset_out[NVC_MAX_HIZ_LEVELS], floats) and the total entry count.  Mip l of width w, height h: rows of pitch
 * (w + 4) & ~3 entries, entry (i + 1, j + 1) = min of texels (i..i+1, j..j+1) clamped to the mip, i in [-1, w-1], j in [-1, h-1].
 * Valid after the nvc_depth_pyramid call that wrote it; *image_out = NULL when no image is prepared. */
NVC_API int nvc_hiz_footprints(NvcContext* ctx, const float** image_out, uint32_t* first_level_out, uint32_t* offset_out, uint32_t* total_out);

/* The cluster pass runs by default as a conservative FILTER (fused arithmetic with an error margin on every comparison,
 * per-command transforms) whose undecided meshlets are re-evaluated by the exact strict-IEEE path: results are identical,
 * the pass is ~2x faster.  enabled = 0 selects the exact kernel for every meshlet (A/B measurements, debugging). */
NVC_API int nvc_set_cluster_filter(NvcContext* ctx, int enabled);
/* Diagnostics (synchronises the device): out[0] = meshlets the filtered cluster passes evaluated, out[1] = how many of them
 * were undecided and took the exact path, both cumulative since the last call with reset != 0. */
NVC_API int nvc_filter_stats(NvcContext* ctx, uint64_t* out_items_undecided2, int reset);
/* Diagnostics / tests: enqueues on `stream` the filter's approximate reciprocal (op 0) or square root (op 1) of n float bit
 * patterns: out[i] = bits of op(float bits in[i]), as the filtered cluster pass computes them (device arrays of n uint32). */
NVC_API int nvc_filter_approx(NvcContext* ctx, void* stream, int op, const uint32_t* in, uint32_t* out, uint64_t n);

/* ---- pyramid layout (host only): niagara.cpp:439-447 previousPow2, resources.cpp:280-292 getImageMipLevels,
 *      niagara.cpp:1339-1342 ------------------------------------------------------------------------- */
NVC_API uint32_t nvc_previous_pow2(uint32_t v);
NVC_API uint32_t nvc_image_mip_levels(uint32_t width, uint32_t height);
/* Fills width/height/levels/level_offset/total_texels for a depth target of depth_width x depth_height;
 * leaves `texels` NULL (caller allocates total_texels * 4 bytes on the device). */
NVC_API int nvc_hiz_layout(uint32_t depth_width, uint32_t depth_height, NvcHiZ* out);

/* ---- passes ---------------------------------------------------------------------------------- */

/* drawcull.comp.glsl:54-156 for all four (LATE, TASK) specialisations; when task != 0 the
 * tasksubmit.comp.glsl:27-47 epilogue (group counts + zero padding to x64) is fused into the same launch.
 *   draws            MeshDraw[cull->drawCount]                      (db)
 *   meshes           Mesh[]                                         (mb)
 *   draw_visibility  uint32[drawCount], read; written when late     (dvb)
 *   commands         task ? MeshTaskCommand[task_wglimit] : MeshDrawCommand[drawCount]   (dcb)
 *   command_count4   uint32[4] {commandCount, groupCountX, groupCountY, groupCountZ}      (dccb)
 *                    fully written by the call (the host-side vkCmdFillBuffer reset of niagara.cpp:1541 is
 *                    folded in); for task == 0 only [0] is meaningful, [1..3] are set to 0.
 *   hiz              depth pyramid; required when late && cull->occlusionEnabled == 1, else may be NULL */
NVC_API int nvc_drawcull(NvcContext* ctx, void* stream, const NvcCullData* cull, int late, int task,
    const NvcMeshDraw* draws, const NvcMesh* meshes, uint32_t* draw_visibility,
    void* commands, uint32_t* command_count4, const NvcHiZ* hiz);

/* clustercull.comp.glsl:56-149 (LATE = 0/1) with the clustersubmit.comp.glsl:25-45 epilogue fused.
 * Processes commandId < command_count4[1] * 64 exactly as the reference's indirect dispatch (X,64,1) does.
 *   task_commands       MeshTaskCommand[] written by nvc_drawcull(task=1)   (dcb)
 *   command_count4      uint32[4] written by nvc_drawcull(task=1)           (dccb)
 *   meshlets            Meshlet[]                                            (mlb)
 *   meshlet_visibility  bit array, read; atomically updated when late        (mvb)
 *   cluster_indices     uint32[cluster_limit rounded up to 256]              (cib)
 *   cluster_count4      uint32[4] {clusterCount, 16, Y, 16}, fully written   (ccb) */
NVC_API int nvc_clustercull(NvcContext* ctx, void* stream, const NvcCullData* cull, int late,
    const NvcMeshTaskCommand* task_commands, const uint32_t* command_count4,
    const NvcMeshDraw* draws, const NvcMeshlet* meshlets, uint32_t* meshlet_visibility,
    uint32_t* cluster_indices, uint32_t* cluster_count4, const NvcHiZ* hiz);

/* meshlet.task.glsl:53-149 (task-shader submission mode, niagara.cpp:1666-1679): same per-meshlet test as
 * nvc_clustercull, but the survivors of command c are compacted into payloads[c].clusterIndices[0..n) and
 * n is written to emit_counts[c] (the EmitMeshTasksEXT(n,1,1) argument).  Order inside a payload is
 * ascending lane (the reference's shared-memory atomic makes it arbitrary). */
NVC_API int nvc_taskcull(NvcContext* ctx, void* stream, const NvcCullData* cull, int late,
    const NvcMeshTaskCommand* task_commands, const uint32_t* command_count4,
    const NvcMeshDraw* draws, const NvcMeshlet* meshlets, uint32_t* meshlet_visibility,
    NvcMeshTaskPayload* payloads, uint32_t* emit_counts, const NvcHiZ* hiz);

/* Consumer-side walk of the cluster pass output (SURVEY §8(f) N1), exactly as meshlet.mesh.glsl:89-105 decodes it under
 * vkCmdDrawMeshTasksIndirectEXT(ccb, 4): one slot per mesh workgroup, slot = x + y * 256 + z * 16 for the dispatch
 * (16, Y, 16) stored in cluster_count4[1..3]; ci == ~0 -> skipped; command = taskCommands[ci & 0xffffff];
 * mi = command.taskOffset + (ci >> 24).  Writes per slot {drawId, mi, vertexCount, triangleCount} (all ~0 for skipped
 * slots) and stats[4] = {decoded slots, skipped slots, invalid slots (lane >= taskCount), triangles}.  Used to prove the
 * output is a drop-in for the reference's consumers; not part of the per-frame path.  records may be NULL (stats only). */
typedef struct NvcClusterRecord
{
	uint32_t drawId, meshletIndex, vertexCount, triangleCount;
} NvcClusterRecord;
NVC_API int nvc_decode_clusters(NvcContext* ctx, void* stream, const uint32_t* cluster_indices, const uint32_t* cluster_count4,
    const NvcMeshTaskCommand* task_commands, const NvcMeshlet* meshlets, NvcClusterRecord* records, uint32_t* stats4);

/* depthreduce.comp.glsl:14-22 + the per-mip loop of niagara.cpp:1703-1733, as ONE launch.
 *   depth  float[depth_height][depth_width], reverse-Z (the D32 depthTarget)
 *   hiz    layout from nvc_hiz_layout(depth_width, depth_height) with `texels` set */
NVC_API int nvc_depth_pyramid(NvcContext* ctx, void* stream, const float* depth,
    uint32_t depth_width, uint32_t depth_height, const NvcHiZ* hiz);

/* ---- host-side helpers mirroring the reference's host code (pure CPU, no context needed) ---------- */

/* niagara.cpp:449-481 PCG32 + rand01/rand32 and the random scene of niagara.cpp:969-998.
 * Fills draws[draw_count] exactly as the reference does (rng state = 0x42, inc = PCG32 default). */
NVC_API void nvc_host_random_draws(NvcMeshDraw* draws, uint32_t draw_count, uint32_t mesh_count, float scene_radius);

/* niagara.cpp:1002-1020: meshletVisibilityOffset = exclusive prefix sum over draws of max-over-LODs
 * meshletCount; returns the total bit count; *post_pass_mask gets OR(1 << postPass) (may be NULL). */
NVC_API uint32_t nvc_host_visibility_offsets(NvcMeshDraw* draws, uint32_t draw_count, const NvcMesh* meshes, uint32_t* post_pass_mask);

typedef struct NvcCamera
{
	float position[3];
	float orientation[4]; /* x,y,z,w */
	float fovY;
	float znear;
} NvcCamera;

typedef struct NvcCullOptions
{
	float draw_distance; /* zfar, niagara.cpp:1000 (200) */
	int32_t culling, lod, occlusion, cluster_occlusion, mesh_shading; /* runtime toggles niagara.cpp:31-44 */
	int32_t debug_lod_step;
} NvcCullOptions;

/* niagara.cpp:424-432 + 1487-1516: view, infinite reverse-Z projection, frustum planes, lodTarget, pyramid size.
 * Leaves clusterBackfaceEnabled = 0 and postPass = 0 exactly like `cullData` at niagara.cpp:1499-1516;
 * the per-pass copies (niagara.cpp:1547-1550, 1595-1596) are the caller's job, see nvc_host_pass_data. */
NVC_API void nvc_host_cull_data(const NvcCamera* camera, uint32_t screen_width, uint32_t screen_height,
    uint32_t draw_count, const NvcCullOptions* options, NvcCullData* out, float* out_projection16 /* may be NULL */);

/* passData of the cull lambda (niagara.cpp:1547-1550): clusterBackfaceEnabled = (postPass == 0), postPass set. */
NVC_API void nvc_host_pass_data(const NvcCullData* frame, int for_drawcull, uint32_t post_pass, NvcCullData* out);

/* ---- multi-GPU: exchange of the per-rank visible slabs (new in this implementation; the reference is single-GPU) */

/* Bootstraps an NCCL communicator owned by the context.  unique_id is the 128-byte ncclUniqueId produced by
 * nvc_nccl_unique_id on rank 0 and distributed by the caller (e.g. torch.distributed broadcast). */
NVC_API int nvc_nccl_unique_id(void* out_unique_id128);
NVC_API int nvc_nccl_init(NvcContext* ctx, const void* unique_id128, int rank, int world_size);
/* Gathers every rank's {count, slab[0..slab_capacity)} into gathered_counts[world] and
 * gathered[world][slab_capacity] on every rank (one ncclAllGather each), after globalising nothing: ids inside
 * the slabs are rank-local; rank r's base draw id is the caller's partition offset. */
NVC_API int nvc_allgather_visible(NvcContext* ctx, void* stream, const void* local_slab, size_t slab_bytes,
    const uint32_t* local_count4, void* gathered_slabs, uint32_t* gathered_count4);

/* Copy-engine variant of the same exchange (no SMs, so it overlaps the SM-filling late cluster pass): every rank
 * PUSHES its slab + counters into slot `rank` of every rank's gathered buffers with peer cudaMemcpyAsync over CUDA-IPC
 * mappings, then raises a flag in the peer's memory; nvc_gather_wait blocks a stream (device side) until all ranks'
 * data of the latest push has landed.  One process per GPU.
 *   nvc_gather_create   allocates this rank's receive buffers (double-buffered by frame parity), returns a 192-byte IPC ticket
 *   nvc_gather_connect  all ranks' tickets (world x 192 bytes, rank order, exchanged by the caller)
 *   nvc_gather_push     enqueue after the pass that produced local_slab / local_count4 on `stream`; the counters are
 *                       snapshotted in stream order, the slab must stay unchanged until nvc_gather_wait
 *   nvc_gather_wait     enqueue on the stream that consumes the gathered data (or reuses local_slab); every push must be
 *                       followed by its wait before the second-next push
 *   nvc_gather_buffers  this rank's gathered slabs [world][slab_bytes] and counters [world][4] of the latest frame, valid from
 *                       its nvc_gather_wait until the next nvc_gather_wait
 * No barrier is needed between frames: receivers acknowledge to senders which frame they are done with, and a sender reuses a
 * parity buffer only after every peer has acknowledged its previous user (a fast rank runs at most one frame ahead). */
NVC_API int nvc_gather_create(NvcContext* ctx, size_t slab_bytes, int rank, int world_size, void* ticket192_out);
NVC_API int nvc_gather_connect(NvcContext* ctx, const void* all_tickets);
NVC_API int nvc_gather_push(NvcContext* ctx, void* stream, const void* local_slab, const uint32_t* local_count4);
NVC_API int nvc_gather_wait(NvcContext* ctx, void* stream);
NVC_API int nvc_gather_buffers(NvcContext* ctx, void** gathered_slabs, uint32_t** gathered_count4);
/* CUDA-graph replay of frames that contain the exchange: the calls above bake their frame tags (and the parity-selected buffer
 * addresses) into a captured graph.  Enqueue this as the LAST operation of the captured sequence with `frames` = the number of
 * nvc_gather_push calls captured (must be even); every replay then shifts the tags of the next one by `frames`.  Each captured push
 * needs its nvc_gather_wait inside the same capture; all ranks replay the same graphs the same number of times. */
NVC_API int nvc_gather_graph_advance(NvcContext* ctx, void* stream, uint32_t frames);
/* The device-side waits of the protocol give up after ~20 s (a peer that crashed or disagrees about the frame) instead of hanging the
 * GPU; *timed_out = 1 from then on (the gathered data are undefined, later waits return at once).  Synchronises the device. */
NVC_API int nvc_gather_status(NvcContext* ctx, int* timed_out);
/* transport of nvc_gather_push: 0 = copy engines (default), 2 / 3 = NVSwitch multicast (below), 1 = a 32-CTA kernel on a high-priority stream that writes only
 * the valid count x 20 bytes with 16-byte peer stores (also selectable with NVC_GATHER_MODE=sm) */
NVC_API int nvc_gather_set_mode(NvcContext* ctx, int mode);

/* NVSwitch MULTICAST transports (modes 2 and 3).  Every rank allocates ONE region of nvc_gather_region_bytes() with a symmetric
 * allocator that also yields a multicast mapping of it (CUDA VMM: cuMemCreate + cuMulticastCreate / AddDevice / BindMem, handles
 * exchanged between the processes; or torch.distributed._symmetric_memory, as bench.py does) and attaches it:
 *   peer_regions[p]    this process's mapping of rank p's region (p == rank: its own)
 *   multicast_region   the multicast alias (a store through it lands in EVERY rank's region), or NULL: unicast SM push only
 * The caller barriers once after every rank has attached.  mode 2: nvc_gather_push launches a kernel that stores the valid part
 * of the slab ONCE through the multicast mapping (egress 1x instead of world x).  mode 3 (fused compute + collective):
 *   nvc_gather_fuse_next_drawcull(ctx, stream);   // takes the frame tag, waits for the peers' acknowledgements on `stream`
 *   nvc_drawcull(ctx, stream, ..., late = 1, task = 1, ...);   // its command write-out also goes through the multicast mapping
 *   nvc_gather_push(ctx, stream, dcb, dccb);      // counters + flags only
 *   ...late cluster pass...;  nvc_gather_wait(ctx, stream); */
NVC_API size_t nvc_gather_region_bytes(size_t slab_bytes, int world_size);
NVC_API int nvc_gather_attach(NvcContext* ctx, size_t slab_bytes, int rank, int world_size, void* const* peer_regions, void* multicast_region);
NVC_API int nvc_gather_fuse_next_drawcull(NvcContext* ctx, void* stream);

/* ---- widening N2 (SURVEY 8(f)): scene cache (.cache v7) reader — the on-disk format that feeds the path ----------------
 * Replaces loadSceneCache (src/scenecache.cpp:273-370) for the arrays the visibility path consumes.  Host-only, no
 * CUDA calls: the caller maps the file, parses it once and copies Meshlet[] / Mesh[] / MeshDraw[] / Animation[] /
 * Keyframe[] straight from the mapping to the device (they are stored raw, scenecache.cpp:170,181-186).  The
 * meshopt-compressed sections are located by the header's byte counts and decoded by nvc_scene_cache_read: the
 * per-meshlet stream ("meshlet codec", scenecache.cpp:84-117,256-271), the vertex codec (vertices and RT positions) and
 * the index codec.  Every stream is bounds-checked (NVC_ERROR_CORRUPT), nothing is written outside dst. */

#define NVC_SCENE_CACHE_MAGIC 0x434E4353u /* 'SCNC', scenecache.cpp:12 */
#define NVC_SCENE_CACHE_VERSION 7u        /* scenecache.cpp:13 */

/* scenecache.cpp:16-55 — 160 bytes */
typedef struct NvcSceneCacheHeader
{
	uint32_t magic, version;
	uint64_t hashMeta;
	uint32_t meshletMaxVertices, meshletMaxTriangles;
	uint8_t clrtMode, compressed, pad0_[2];
	uint32_t compressedVertexBytes, compressedIndexBytes, compressedMeshletDataBytes, compressedMeshletVtx0Bytes;
	uint32_t vertexCount, indexCount, meshletCount, meshletdataCount, meshletvtx0Count, meshCount;
	uint32_t materialCount, drawCount, texturePathCount, lightCount, animationCount, keyframeCount;
	uint32_t ommArrayDataSize, ommIndexDataSize, ommDescCount, ommStates;
	NvcCamera camera;
	float sunDirection[3];
	uint32_t pad1_;
} NvcSceneCacheHeader;

/* sections in file order (saveSceneCache, scenecache.cpp:158-197) */
typedef enum NvcSceneCacheSectionId
{
	NVC_CACHE_VERTICES = 0, /* Vertex 16 B, vertex codec when compressed */
	NVC_CACHE_INDICES,      /* uint32, index codec when compressed */
	NVC_CACHE_MESHLETS,     /* Meshlet 24 B, always raw */
	NVC_CACHE_MESHLETDATA,  /* uint32 words, meshlet codec when compressed */
	NVC_CACHE_MESHLETVTX0,  /* uint16, vertex codec (stride 8) when compressed */
	NVC_CACHE_MESHES,       /* Mesh 208 B */
	NVC_CACHE_MATERIALS,    /* Material 64 B */
	NVC_CACHE_DRAWS,        /* MeshDraw 48 B */
	NVC_CACHE_LIGHTS,       /* Light 32 B */
	NVC_CACHE_ANIMATIONS,   /* Animation 24 B */
	NVC_CACHE_KEYFRAMES,    /* Keyframe 32 B */
	NVC_CACHE_OMM_DATA,     /* bytes */
	NVC_CACHE_OMM_INDICES,  /* bytes */
	NVC_CACHE_OMM_DESCS,    /* uint32 */
	NVC_CACHE_TEXTURE_PATHS, /* char[256] each */
	NVC_CACHE_SECTION_COUNT
} NvcSceneCacheSectionId;

typedef struct NvcSceneCacheSection
{
	uint64_t offset;        /* from the start of the file */
	uint64_t stored_bytes;  /* bytes occupied in the file */
	uint64_t decoded_bytes; /* count * element_size */
	uint32_t count, element_size;
	uint32_t compressed;    /* 1: stored_bytes is a meshopt stream, not the array */
	uint32_t pad_;
} NvcSceneCacheSection;

typedef struct NvcSceneCacheInfo
{
	NvcSceneCacheHeader header;
	NvcSceneCacheSection sections[NVC_CACHE_SECTION_COUNT];
} NvcSceneCacheInfo;

/* nvc_scene_cache_read into DEVICE memory: dst is a device pointer, 4-byte aligned, with room for
 * info->sections[section].decoded_bytes.  Raw sections are copied up.  VERTICES, MESHLETVTX0 (vertex codec), INDICES (index
 * codec) and MESHLETDATA (meshlet codec) go up compressed, with an index the host finds by walking their sizes, and are
 * decoded by kernels; no host copy of the decoded section is made.  INDICES is cut into chunks of 256 triangles: each
 * chunk's effect on the decoder's FIFO state is found on its own, the effects are combined by a scan, and every chunk is
 * then decoded from its exact entry state.  Result byte for byte and status equal to nvc_scene_cache_read + a copy, except that a cache whose
 * meshlet word ranges are not in increasing, non-overlapping order is refused with NVC_ERROR_UNSUPPORTED before anything
 * is written (every cache the reference writes is in that order: appendMeshlet appends), and a compressed VERTICES,
 * MESHLETVTX0 or MESHLETDATA stream of 4 GiB or more is refused likewise (its index holds 32-bit offsets).  On NVC_ERROR_CORRUPT the
 * contents of dst are unspecified, as on the host.  A corrupt vertex or index stream is found by the host walk, before any
 * launch, and dst is not written.
 * Runs on `stream` and synchronises the device (it reads back a corruption flag), so it belongs at load time, outside
 * stream capture.  The staged stream and its index live in scratch the context owns, grown as needed. */
NVC_API int nvc_scene_cache_read_device(NvcContext* ctx, void* stream, const void* file, size_t file_size, const NvcSceneCacheInfo* info, int section,
    void* dst, size_t dst_bytes);

/* What nvc_scene_cache_write stores: the header fields the caller chooses, and per section (NvcSceneCacheSectionId) a pointer
 * and an element count in the reader's units (NvcSceneCacheSection.count: MESHLETVTX0 in uint16 elements, OMM data and
 * indices in bytes, texture paths in 256-byte records).  Bit s of device_sections says that data[s] is device memory of the
 * context's device (4-byte aligned); any section may be, and each other pointer is host memory.  A section with count 0 may
 * have a NULL pointer. */
typedef struct NvcSceneCacheWriteDesc
{
	uint64_t hashMeta;
	uint32_t clrtMode, compressed, ommStates;
	uint32_t device_sections;
	NvcCamera camera;
	float sunDirection[3];
	const void* data[NVC_CACHE_SECTION_COUNT];
	uint32_t count[NVC_CACHE_SECTION_COUNT];
} NvcSceneCacheWriteDesc;

/* Host: a size of the file nvc_scene_cache_write makes from `desc` that always suffices (the codecs' worst cases). */
NVC_API int nvc_scene_cache_write_bound(const NvcSceneCacheWriteDesc* desc, size_t* bytes);
/* The file saveSceneCache (src/scenecache.cpp:119-203) writes for these arrays, byte for byte, into the HOST buffer file_out
 * (capacity >= nvc_scene_cache_write_bound); *file_size = its length.  The caller writes the file.
 *   header      zero padding, meshletMaxVertices 64 / meshletMaxTriangles 96, the compressed byte counts when compressed
 *   compressed  VERTICES and MESHLETVTX0 by the vertex codec v1 at level 2 (strides 16 and 8; an empty stream is 25 bytes),
 *               INDICES by the index codec v1, MESHLETDATA as one uint16 size and one meshlet codec block per Meshlet, the
 *               block encoding its vertexCount references (widened from uint16 when shortRefs) and triangleCount * 3 bytes
 *   other       copied; texture paths as strncpy(record, path, 255) into a zeroed record
 * The vertex and meshlet streams are encoded by kernels on `stream` (inputs in host memory are copied up first), the index
 * stream on the host while they run (indices in device memory are copied down first).  Uncompressed writes run no kernel,
 * and ctx may be NULL when no section is in device memory and nothing is encoded on the device.  Refused before
 * anything is written to file_out:
 *   NVC_ERROR_INVALID_ARGUMENT  a capacity below the bound; a device pointer, or compressed vertex / meshlet data, without
 *                               a context; a misaligned device pointer; compressed with an index count that is not a
 *                               multiple of 3 or a MESHLETVTX0 count that is not a multiple of 4; a meshlet whose words lie
 *                               outside meshletdata or whose counts pass 64 vertices / 96 triangles (found on the device)
 *   NVC_ERROR_UNSUPPORTED       a compressed stream of 4 GiB or more (the header's byte counts are 32-bit)
 * Scratch is context-owned and grows as needed; the call synchronises the device, so it belongs at load time, outside
 * stream capture. */
NVC_API int nvc_scene_cache_write(NvcContext* ctx, void* stream, const NvcSceneCacheWriteDesc* desc, void* file_out, size_t capacity, size_t* file_size);

/* The three meshopt stream decoders on their own (the same streams appear in glTF EXT_meshopt_compression buffers):
 *   vertex codec v0 / v1   -> dst[vertex_count * vertex_size], vertex_size a multiple of 4, <= 256
 *   index codec v0 / v1    -> dst[index_count] uint32, index_count a multiple of 3 (triangles come back rotated)
 *   meshlet codec          -> vertex references (reference_size 2 or 4 bytes each) and triangle_count * 3 index bytes
 * Return NVC_OK, NVC_ERROR_CORRUPT (malformed stream; nothing is written outside the destinations),
 * NVC_ERROR_UNSUPPORTED (a newer codec version) or NVC_ERROR_INVALID_ARGUMENT. */
NVC_API int nvc_decode_vertex_stream(void* dst, uint32_t vertex_count, uint32_t vertex_size, const void* stream, size_t stream_size);
NVC_API int nvc_decode_index_stream(uint32_t* dst, uint32_t index_count, const void* stream, size_t stream_size);
NVC_API int nvc_decode_meshlet_stream(void* references, uint32_t vertex_count, uint32_t reference_size, uint8_t* triangles,
    uint32_t triangle_count, const void* stream, size_t stream_size);

/* The rest of the family a glTF EXT_ / KHR_meshopt_compression buffer view can hold (meshoptimizer's decodeIndexBuffer,
 * decodeIndexSequence and decodeFilter*):
 *   index codec            -> dst[index_count] of index_size 2 or 4 bytes, index_count a multiple of 3; 2-byte indices keep
 *                             the low 16 bits (nvc_decode_index_buffer(dst, n, 4, ...) == nvc_decode_index_stream)
 *   index-sequence codec   -> dst[index_count] of index_size 2 or 4 bytes (header 0xd0 | version, versions 0 and 1)
 * Same returns as the stream decoders above.
 *   vertex filter          in place over count elements of `stride` bytes: OCTAHEDRAL (stride 4 or 8), QUATERNION (8),
 *                          EXPONENTIAL (any multiple of 4 up to 256), COLOR (4 or 8); NONE leaves the data as it is.
 *                          NVC_ERROR_INVALID_ARGUMENT for a stride the glTF extension does not allow with the filter.
 * The filters compute what the reference's SSE2 build computes, operation for operation: float -> int conversions round to
 * nearest even, and the 8-bit OCTAHEDRAL and COLOR filters use the x86 rsqrtps / rcpps approximations, whose bits the CPU
 * defines — on x86 the result is bit-identical to the reference's decoder run on the same host (elsewhere those two use the
 * exact reciprocal square root / reciprocal). */
typedef enum NvcMeshoptFilter
{
	NVC_MESHOPT_FILTER_NONE = 0,
	NVC_MESHOPT_FILTER_OCTAHEDRAL = 1,
	NVC_MESHOPT_FILTER_QUATERNION = 2,
	NVC_MESHOPT_FILTER_EXPONENTIAL = 3,
	NVC_MESHOPT_FILTER_COLOR = 4
} NvcMeshoptFilter;
NVC_API int nvc_decode_index_buffer(void* dst, uint32_t index_count, uint32_t index_size, const void* stream, size_t stream_size);
NVC_API int nvc_decode_index_sequence(void* dst, uint32_t index_count, uint32_t index_size, const void* stream, size_t stream_size);
NVC_API int nvc_decode_vertex_filter(int filter, void* data, uint32_t count, uint32_t stride);

/* scene.h:141-161 */
typedef struct NvcKeyframe
{
	float translation[3];
	float scale;
	float rotation[4]; /* x,y,z,w */
} NvcKeyframe;

typedef struct NvcAnimation
{
	int32_t drawIndex, lightIndex;
	float startTime, period;
	uint32_t keyframeOffset, keyframeCount;
} NvcAnimation;

/* Validates magic / version / that every section lies inside the file (and, when compressed, that the per-meshlet
 * stream's size chain adds up to compressedMeshletDataBytes), fills the section table.  The caller decides about
 * hashMeta / meshlet limits / clrtMode / ommStates (loadSceneCache's other rejections, scenecache.cpp:283-290). */
NVC_API int nvc_scene_cache_parse(const void* file, size_t file_size, NvcSceneCacheInfo* out);
/* Copies (raw sections) or decodes (compressed sections) one section into dst[decoded_bytes]. */
NVC_API int nvc_scene_cache_read(const void* file, size_t file_size, const NvcSceneCacheInfo* info, int section,
    void* dst, size_t dst_bytes);

/* ---- widening N3: animated MeshDraw updates (niagara.cpp:1362-1411, the frame loop's keyframe evaluation) --------------
 * Host: evaluates every animation with drawIndex >= 0 at animation_time exactly as the reference does (double index
 * arithmetic, glm::mix for position / scale, glm::slerp for orientation), writes the new values into draws[] (the
 * reference's `draws[animation.drawIndex]`) and appends {index, MeshDraw} to the packed update list.  Returns the
 * number of updates written (<= max_updates), or a negative NvcStatus. */
NVC_API int nvc_host_animate(const NvcAnimation* animations, uint32_t animation_count, const NvcKeyframe* keyframes,
    uint32_t keyframe_count, double animation_time, NvcMeshDraw* draws, uint32_t draw_count,
    uint32_t* update_indices, NvcMeshDraw* update_values, uint32_t max_updates);
/* Device: draws[update_indices[i]] = update_values[i] for i < count (the reference memcpy's into its host-visible
 * `db`, niagara.cpp:1394-1395; here the packed list is one H2D copy and one scatter launch).  Indices >= draw_count
 * are ignored; indices must be unique (the importer gives every animation its own draw, scene.cpp:777) — with
 * duplicates one of the values lands, unspecified which. */
NVC_API int nvc_update_draws(NvcContext* ctx, void* stream, NvcMeshDraw* draws, uint32_t draw_count,
    const uint32_t* update_indices, const NvcMeshDraw* update_values, uint32_t count);

/* ---- widening N4: meshlet bounds + normal cones on the GPU (the producer of Meshlet[]'s cull fields) --------------------
 * scene.h:51-57 / mesh.h:3-9 — 16 B */
typedef struct NvcVertex
{
	uint16_t vx, vy, vz; /* fp16 position */
	uint16_t tp;
	uint32_t np;
	uint16_t tu, tv;
} NvcVertex;

/* ---- N3: glTF 2.0 scene import for the visibility path (loadScene, src/scene.cpp:473-853) -----------------------------------------
 * MeshDraw[] (world transform of every mesh node decomposed as scene.cpp:295-340 does, meshIndex = first_mesh_index + running index of
 * the indexed triangle primitives, materialIndex = material_offset + material, postPass 1 for non-opaque / 2 for transmissive materials),
 * Animation[] + Keyframe[] (LINEAR TRS samplers baked per key through the node hierarchy, scene.cpp:713-830), camera, sun direction,
 * and per primitive the quantised Vertex[] / index arrays of loadVertices (scene.cpp:342-405) — bit-identical to what the reference's
 * importer produces from the same file.  Host only; .gltf (data: URIs or external buffers under base_dir) and .glb.  Sparse accessors:
 * NVC_ERROR_UNSUPPORTED.  Malformed files: NVC_ERROR_CORRUPT, never read outside the buffers.
 * Meshopt compression (EXT_meshopt_compression / KHR_meshopt_compression, what gltfpack -c / -cc / -cz writes): every compressed
 * buffer view is validated as cgltf_validate does and decoded at import, used by a primitive or not (the reference's
 * decompressMeshopt, scene.cpp:405-470); the decoded bytes are what accessors and animation samplers read.  A buffer without data
 * is accepted when it is a meshopt fallback buffer ("fallback": true); an uncompressed view into one is NVC_ERROR_CORRUPT.  A
 * view that breaks a validation rule is NVC_ERROR_CORRUPT; a stream that does not decode returns the decoder's status
 * (NVC_ERROR_CORRUPT, or NVC_ERROR_UNSUPPORTED for a newer codec version); NVC_ERROR_OUT_OF_MEMORY when a decoded view cannot be
 * allocated.  Filters follow nvc_decode_vertex_filter (bit-identical
 * to the reference on an x86 host). */
typedef struct NvcGltfScene NvcGltfScene;
typedef struct NvcGltfInfo
{
	uint32_t node_count, mesh_count, primitive_count, draw_count, animation_count, keyframe_count, material_count, point_light_count;
	uint32_t has_camera, has_sun;
	NvcCamera camera;        /* position, orientation, fovY of the (last) camera node; znear stays 0: the application sets it */
	float sun_direction[3];  /* local +Z of the (last) directional light node */
} NvcGltfInfo;
NVC_API int nvc_gltf_import(const void* file, size_t file_size, const char* base_dir, uint32_t first_mesh_index, uint32_t material_offset, NvcGltfScene** out_scene);
NVC_API void nvc_gltf_free(NvcGltfScene* scene);
NVC_API int nvc_gltf_info(const NvcGltfScene* scene, NvcGltfInfo* out);
/* any output may be NULL; sizes from nvc_gltf_info; mesh_scale[primitive_count] = the scale appendMesh receives (scene.cpp:503-519) */
NVC_API int nvc_gltf_scene_arrays(const NvcGltfScene* scene, NvcMeshDraw* draws, NvcAnimation* animations, NvcKeyframe* keyframes, float* mesh_scale);
NVC_API int nvc_gltf_primitive_size(const NvcGltfScene* scene, uint32_t primitive, uint32_t* vertex_count, uint32_t* index_count);
NVC_API int nvc_gltf_primitive_data(const NvcGltfScene* scene, uint32_t primitive, NvcVertex* vertices, uint32_t* indices);

/* Depth-only consumer of cib / ccb / dcb on the device (new; stands in for what the reference's mesh stage and fixed-function
 * rasteriser do to depthTarget between the cull passes, niagara.cpp:1576-1701 with meshlet.mesh.glsl:89-206): every cluster slot of
 * the (16, Y, 16) dispatch is decoded like the mesh shader does, its vertices are transformed with the shader's arithmetic
 * (strict IEEE, GLSL operation order) by `projection16 * (pass->view * vec4(world, 1))`, and its front-facing triangles are sampled at
 * pixel centres into `depth` (float, width x height, reverse Z, test GREATER: depth = max).  The caller clears `depth` to 0 before
 * the early pass; the late pass adds to it.  Meshlets whose references fall outside meshletdata / vertices are skipped and counted.
 * stats4 (may be NULL): clusters drawn, triangles sampled, clusters rejected, depth updates issued.  The image is deterministic
 * (max is order independent) and equals the sequential test rasteriser's (oracle/refshader) bit for bit. */
NVC_API int nvc_raster_depth(NvcContext* ctx, void* stream, const float* projection16, const NvcCullData* pass,
    const uint32_t* cluster_indices, const uint32_t* cluster_count4, const NvcMeshTaskCommand* task_commands,
    const NvcMeshDraw* draws, const NvcMeshlet* meshlets, const uint32_t* meshletdata, uint32_t meshletdata_words,
    const NvcVertex* vertices, uint32_t vertex_count, float* depth, uint32_t width, uint32_t height, uint32_t* stats4);

/* The same depth producer in the task-shading submission mode (niagara.cpp:1666-1679: vkCmdDrawMeshTasksIndirectEXT(dccb, 4) ->
 * meshlet.task.glsl EmitMeshTasksEXT(n, 1, 1) -> meshlet.mesh.glsl:94-103 with TASK = true): every command c < command_count4[1] * 64 of
 * the (X, 64, 1) dispatch nvc_taskcull processed (padding commands included, X clamped to NVC_MAX_DISPATCH_GROUPS) launches
 * n = min(emit_counts[c], 64) mesh workgroups (the clamp of the test driver's rs_mesh_payloads); workgroup i < n decodes
 * ci = payloads[c].clusterIndices[i] exactly like nvc_raster_depth decodes a cib entry (~0 draws nothing, command = task_commands[ci & 0xffffff],
 * meshlet = command.taskOffset + (ci >> 24)) and draws it with the same arithmetic, sampling and rejection rules.  payloads / emit_counts
 * as written by nvc_taskcull.  stats4 (may be NULL, zeroed by the call): clusters drawn, triangles sampled, clusters rejected, depth
 * updates issued.  Same bits as nvc_raster_depth over a cib holding the same cluster indices. */
NVC_API int nvc_raster_depth_tasks(NvcContext* ctx, void* stream, const float* projection16, const NvcCullData* pass,
    const NvcMeshTaskPayload* payloads, const uint32_t* emit_counts, const uint32_t* command_count4,
    const NvcMeshTaskCommand* task_commands, const NvcMeshDraw* draws, const NvcMeshlet* meshlets,
    const uint32_t* meshletdata, uint32_t meshletdata_words, const NvcVertex* vertices, uint32_t vertex_count,
    float* depth, uint32_t width, uint32_t height, uint32_t* stats4);

/* The same depth producer in the indexed-draw submission mode (mesh shading off, niagara.cpp:1680-1694:
 * vkCmdDrawIndexedIndirectCount(dcb + 4, dccb, 0, maxDrawCount, 24) with mesh.vert.glsl:39-57): commands i < min(command_count4[0],
 * max_draw_count) of draw_commands (written by nvc_drawcull(task = 0)); command i draws indexCount / 3 triangles from firstIndex
 * (trailing indices that make no whole triangle are ignored); corner k of triangle t is vertex indices[firstIndex + 3t + k] + vertexOffset
 * (uint32 wrap), transformed with draws[command.drawId] by mesh.vert's arithmetic (gl_DrawIDARB only selects the command).
 * instanceCount == 0 draws nothing; instanceCount > 1 is drawn once (mesh.vert ignores gl_InstanceIndex and max is idempotent, so the
 * image is the same).  A command whose [firstIndex, firstIndex + indexCount) is not inside indices[0, index_count) is skipped whole and
 * counted; a triangle with a vertex >= vertex_count is skipped and counted; nothing is read outside the given arrays.  stats4 (may be
 * NULL, zeroed by the call): commands drawn, triangles sampled, commands rejected, triangles rejected.  The image equals the test
 * rasteriser's (oracle/refshader rs_draw_indexed) bit for bit. */
NVC_API int nvc_raster_depth_indexed(NvcContext* ctx, void* stream, const float* projection16, const NvcCullData* pass,
    const NvcMeshDrawCommand* draw_commands, const uint32_t* command_count4, uint32_t max_draw_count,
    const NvcMeshDraw* draws, const uint32_t* indices, uint32_t index_count, const NvcVertex* vertices, uint32_t vertex_count,
    float* depth, uint32_t width, uint32_t height, uint32_t* stats4);

/* meshlet.mesh.glsl with MESH_CULL = 1 (config.h:11; the reference default is 0): nvc_raster_depth and nvc_raster_depth_tasks
 * enqueued after this call drop the triangles the mesh shader marks gl_CullPrimitiveEXT (meshlet.mesh.glsl:175-195: back-facing and
 * zero-area triangles, and triangles whose screen bounding box rounds to a single column or row, when all three corners have w > 0;
 * `round` is half away from zero).  A culled triangle is not sampled, so stats4[1] (triangles sampled) gets smaller; the other
 * statistics keep their meaning.  nvc_raster_depth_indexed is not affected (mesh.vert has no such stage).  Default 0.  The setting
 * is read when a call is enqueued: a captured graph keeps the value that was current at capture time. */
NVC_API int nvc_set_mesh_cull(NvcContext* ctx, int enabled);
/* Diagnostics (synchronises the device): out[0] = triangles the mesh-cull stage tested, out[1] = how many it culled, both
 * cumulative since the last call with reset != 0. */
NVC_API int nvc_mesh_cull_stats(NvcContext* ctx, uint64_t* out_tested_culled2, int reset);

/* The reference's TASK_CULL switch (config.h:8, "meshlet frustum, occlusion and backface culling in the task shader"; the
 * reference default and the default here are 1).  With enabled = 0, calls enqueued after this one behave as a TASK_CULL 0 build:
 *   nvc_drawcull     the late pass emits only draws that were not visible last frame, plus post-pass draws
 *                    (drawcull.comp.glsl:104 without its clusterOcclusionEnabled term), in both task and draw modes;
 *   nvc_clustercull  every lane mgi < min(taskCount, 64) of every command c < command_count4[1] * 64 appends c | (mgi << 24)
 *                    (clustercull.comp.glsl:140-147), with the usual cluster_limit overflow rule and the clustersubmit epilogue;
 *   nvc_taskcull     payloads[c].clusterIndices[i] = c | (i << 24) for all 64 entries and emit_counts[c] = taskCount as stored,
 *                    not clamped to 64 (meshlet.task.glsl:144-148), padding commands included.
 * The cluster and task passes then test no meshlet: they read only task_commands and command_count4; draws, meshlets, the Hi-Z
 * and meshlet_visibility are not read, and meshlet_visibility is not written.  Argument validation is unchanged, so callers pass
 * the same buffers either way.  Turning the switch back on mid-sequence makes the cluster passes read visibility bits nobody
 * maintained while it was off (the reference has no runtime switch, so no reference behaviour covers that).  The setting is read
 * when a call is enqueued: a captured graph keeps the value that was current at capture time.  The multi-GPU exchange
 * (nvc_gather_*) is not covered with the switch off. */
NVC_API int nvc_set_task_cull(NvcContext* ctx, int enabled);

/* Recomputes center / radius / cone_axis / cone_cutoff of meshlets[0..meshlet_count) from geometry, bit-identical to
 * what the reference's cooker stores (scene.cpp:69-80 appendMeshlet -> meshopt_computeMeshletBounds,
 * meshletutils.cpp:133-272,314-339): one thread per meshlet reads its references and triangles from
 * meshletdata[dataOffset...] (layout of scene.cpp:36-50, triangle order as cooked — NOT as re-read from a compressed
 * cache, whose codec rotates triangles) and the fp16 positions of vertices[baseVertex + ref].  The other Meshlet
 * fields are inputs and stay untouched.  For streamed / re-skinned geometry whose bounds must follow the vertices.
 * A meshlet whose words, references or triangle indices fall outside the given arrays is left untouched and counted
 * in *rejected (device uint32, zeroed by the call; may be NULL). */
NVC_API int nvc_cook_meshlet_bounds(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count,
    const uint32_t* meshletdata, uint32_t meshletdata_words, NvcMeshlet* meshlets, uint32_t meshlet_count, uint32_t* rejected);

/* Builds and packs the meshlets of every LOD of a whole Mesh[] on the device, bit-identical to what the reference's cooker
 * stores (scene.cpp:270-276 appendMesh -> appendMeshlets with clrt off: meshopt_buildMeshlets(64 vertices, 96 triangles, cone
 * weight 0.25), meshopt_optimizeMeshletLevel(level 1) per meshlet, then appendMeshlet's packing and bounds):
 *   vertices / vertex_count   device: the scene's Vertex[] (vb); positions are the fp16 vx, vy, vz
 *   indices / index_count     device: the mesh-local indices of every LOD (ib)
 *   host_meshes / mesh_count  host: vertexOffset, vertexCount, lodCount and lods[].indexOffset / indexCount are read
 *   meshes                    device out: host_meshes with lods[l].meshletOffset / meshletCount set for l < lodCount
 *   meshlets, meshletdata     device out: Meshlet[] and meshletdata, meshlets of mesh 0 LOD 0 first; may be NULL with capacity 0
 *   totals4                   device out: meshlets needed, words needed (saturated at 2^32 - 1), LODs rejected, overflow flag
 * The bytes of a meshlet's last triangle word past triangleCount * 3 are 0 (the reference leaves whatever its scratch buffer
 * held there; nothing reads them).  A LOD with an index >= its mesh's vertexCount is rejected: it gets meshletCount 0, is
 * counted in totals4[2], and none of its vertices is read.  When the meshlets or words needed exceed meshlet_capacity or
 * meshletdata_capacity, totals4[3] is 1 and neither array is written (meshes is); nvc_cook_meshlets_capacity gives sizes
 * that always suffice.  NVC_ERROR_INVALID_ARGUMENT: lodCount > 8, an indexCount not a multiple of 3, or a LOD index range or
 * mesh vertex range outside indices / vertices.  Scratch is context-owned and grows as needed, and the call synchronises the
 * device before it enqueues its kernels on `stream`: call it at load time, outside stream capture.  The cooker of clrt
 * builds (a ray-tracing LOD of spatial meshlets, meshletvtx0) is nvc_cook_meshlets_clrt below; the LOD chain that makes the
 * index ranges is nvc_cook_mesh_lods.  Not covered: appending to existing Meshlet[] / meshletdata. */
NVC_API int nvc_cook_meshlets(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* indices,
    uint32_t index_count, const NvcMesh* host_meshes, NvcMesh* meshes, uint32_t mesh_count, NvcMeshlet* meshlets, uint32_t meshlet_capacity,
    uint32_t* meshletdata, uint32_t meshletdata_capacity, uint32_t* totals4);
/* Host: capacities nvc_cook_meshlets never exceeds for these meshes: per LOD meshopt_buildMeshletsBound(indexCount, 64, 96)
 * meshlets and indexCount + ceil(indexCount / 4) + that bound words.  NVC_ERROR_INVALID_ARGUMENT when a lodCount > 8. */
NVC_API int nvc_cook_meshlets_capacity(const NvcMesh* host_meshes, uint32_t mesh_count, uint32_t* meshlets_out, uint64_t* words_out);

/* nvc_cook_meshlets as the reference's cooker runs in a clrt build (CLRT=1, niagara.cpp:844; scene.cpp:266-276, 52-67, 102-103),
 * bit-identical to the Mesh[], Meshlet[], meshletdata and meshletvtx0 it stores:
 *   max_scale    host, per mesh, the maxScale appendMesh receives: 1.0 for loadMesh, meshScale[i] for glTF (the mesh_scale
 *                output of nvc_gltf_scene_arrays); NULL = 1.0 for every mesh
 *   meshes       as nvc_cook_meshlets, and lodRT = the last LOD with lods[i].error * max_scale < 3e-3 (float multiply; 0 when
 *                none is; NaN and inf fail the test); the input's lodRT is ignored
 *   LOD lodRT    meshopt_buildMeshletsSpatial(64 vertices, min 24, max 96 triangles, fill weight 0.5) instead of the greedy
 *                builder, then the same optimisation, packing and bounds; every other LOD exactly as nvc_cook_meshlets
 *   meshletvtx0  device out: for each meshlet of each mesh's lodRT, in Meshlet[] order, per vertex (optimised order)
 *                quantizeHalf(dequantizeHalf(v)) of x, y, z, then 0 (NaN becomes 0x7e00, fp16 denormals flush to 0);
 *                may be NULL with capacity 0 (uint16 elements)
 *   totals8      device out: meshlets needed, words needed, LODs rejected, overflow flag, meshletvtx0 elements needed
 *                (counts saturated at 2^32 - 1), then three zeros
 * A rejected lodRT (an index >= vertexCount) gets meshletCount 0 and contributes no meshletvtx0.  When any of the three
 * capacities is exceeded, totals8[3] is 1 and none of the three arrays is written (meshes is).  Argument validation is
 * nvc_cook_meshlets', plus meshletvtx0_capacity != 0 with meshletvtx0 NULL.  Scratch and synchronisation as nvc_cook_meshlets. */
NVC_API int nvc_cook_meshlets_clrt(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* indices,
    uint32_t index_count, const NvcMesh* host_meshes, const float* max_scale, NvcMesh* meshes, uint32_t mesh_count, NvcMeshlet* meshlets,
    uint32_t meshlet_capacity, uint32_t* meshletdata, uint32_t meshletdata_capacity, uint16_t* meshletvtx0, uint32_t meshletvtx0_capacity,
    uint32_t* totals8);
/* Host: capacities nvc_cook_meshlets_clrt never exceeds: nvc_cook_meshlets_capacity's per LOD, except that each mesh's lodRT
 * takes meshopt_buildMeshletsBound(indexCount, 64, 24) meshlets (the array the reference sizes, scene.cpp:98), the matching
 * words, and 4 * indexCount meshletvtx0 elements.  NVC_ERROR_INVALID_ARGUMENT when a lodCount > 8. */
NVC_API int nvc_cook_meshlets_clrt_capacity(const NvcMesh* host_meshes, const float* max_scale, uint32_t mesh_count, uint32_t* meshlets_out,
    uint64_t* words_out, uint64_t* vtx0_out);

/* Builds every mesh's LOD chain on the device, bit-identical to the Mesh[] (meshlet fields aside) and index buffer the reference's
 * cooker stores (scene.cpp:193-268 appendMesh: meshopt_simplifyWithAttributes with meshopt_SimplifySparse, the decoded normals
 * as 3 attributes of weight 1 and target error 1e-1, down to 60% of the last LOD's indices, then meshopt_optimizeVertexCache):
 *   vertices / vertex_count         device: the processed Vertex[] (vb); positions are the fp16 vx, vy, vz, normals np
 *   lod0_indices / lod0_index_count device: mesh-local LOD 0 indices
 *   host_meshes / mesh_count        host: vertexOffset, vertexCount and lods[0].indexOffset / indexCount (into lod0_indices) are read
 *   max_scale                       host, per mesh, as nvc_cook_meshlets_clrt takes it; NULL = 1.0 for every mesh
 *   meshes                          device out: center / radius (float sum of the dequantised positions over float(vertexCount),
 *                                   then the largest distance), vertexOffset / vertexCount copied, lodCount, lods[l].indexOffset
 *                                   (into indices) / indexCount / error, lodRT (the last LOD with error * max_scale < 3e-3, in
 *                                   every build); every other field 0, meshletOffset / meshletCount included
 *   indices / index_capacity        device out: the chains, meshes in order and each mesh's LODs in order (the reference's ib)
 *   totals4                         device out: indices needed (saturated at 2^32 - 1), meshes rejected, overflow flag, 0
 * A LOD after LOD l is kept when the simplifier returns fewer than 85% of its indices and more than 0; at most 8 LODs.  A mesh
 * with a LOD 0 index >= its vertexCount is rejected: it gets lodCount 0, contributes no indices, none of its vertices is read,
 * and it is counted in totals4[1].  When the indices needed exceed index_capacity, totals4[2] is 1 and indices is not written
 * (meshes is); nvc_cook_mesh_lods_capacity gives a size that always suffices.  NVC_ERROR_INVALID_ARGUMENT: a LOD 0 indexCount
 * not a multiple of 3, or a LOD 0 index range or mesh vertex range outside lod0_indices / vertices; nothing is written then.
 * Each mesh's chain runs as one sequential CTA, meshes side by side.  Scratch is context-owned (per mesh about 20 words per
 * LOD 0 index and 60 per vertex) and grows as needed, and the call synchronises the device before it enqueues its kernels on
 * `stream`: call it at load time, outside stream capture. */
NVC_API int nvc_cook_mesh_lods(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* lod0_indices,
    uint32_t lod0_index_count, const NvcMesh* host_meshes, const float* max_scale, uint32_t mesh_count, NvcMesh* meshes, uint32_t* indices,
    uint32_t index_capacity, uint32_t* totals4);
/* Host: the indices nvc_cook_mesh_lods can ever emit for these meshes (saturated at 2^32 - 1): per mesh, the sum over at most 8
 * LODs of c0 = lods[0].indexCount and c(l+1) = the largest multiple of 3 below size_t(double(c(l)) * 0.85). */
NVC_API int nvc_cook_mesh_lods_capacity(const NvcMesh* host_meshes, uint32_t mesh_count, uint32_t* indices_out);

/* Turns what an importer produces into the processed Vertex[] and LOD 0 that nvc_cook_mesh_lods takes, bit-identical to the
 * reference's cooker (scene.cpp:172-184 appendMesh: meshopt_filterIndexBuffer over the 6 position bytes,
 * meshopt_generateVertexRemap over all 16 bytes and the remap of both buffers, meshopt_optimizeVertexCache,
 * meshopt_optimizeVertexFetch):
 *   vertices / vertex_count   device: Vertex[] as loadObj / loadVertices leave it (nvc_gltf_primitive_data's vertices)
 *   indices / index_count     device: mesh-local indices
 *   host_meshes / mesh_count  host: vertexOffset, vertexCount and lods[0].indexOffset / indexCount are read
 *   meshes                    device out: vertexOffset / vertexCount of the mesh's vertices in vertices_out, lods[0] its range
 *                             in lod0_out, lodCount 1, every other field 0; after a download, nvc_cook_mesh_lods' host_meshes
 *   vertices_out              device out: the processed Vertex[], meshes in order; vertex_capacity >= vertex_count and >= the
 *                             sum of the meshes' vertexCount
 *   lod0_out                  device out: the mesh-local LOD 0 indices, meshes in order; index_capacity >= index_count and >=
 *                             the sum of the meshes' lods[0].indexCount
 *   totals4                   device out: vertices written, indices written, meshes rejected, 0
 * A triangle is dropped when two corners have the same position bytes (so +-0 and NaN payloads stay distinct), or when an
 * earlier kept triangle of the mesh is the same cyclic sequence of positions (a reversed triangle is not); kept triangles
 * keep their order.  Vertices no kept triangle references are dropped.  A mesh with an index >= its vertexCount is
 * rejected: it gets vertexCount 0 and an empty LOD 0, none of its vertices is read, and it is counted in totals4[2]; a mesh
 * whose triangles are all dropped gets the same record.  NVC_ERROR_INVALID_ARGUMENT: an indexCount not a multiple of 3, an
 * index or vertex range outside indices / vertices, or a capacity below the above; nothing is written then.
 * NVC_ERROR_OUT_OF_MEMORY beyond 2^30 mesh vertices in one call.  Every step but the vertex cache optimisation (one
 * sequential CTA per mesh) is data-parallel over all meshes.  Scratch is context-owned (about 24 bytes per index and 56 per
 * vertex) and grows as needed, and the call synchronises the device before it enqueues its kernels on `stream`: call it at
 * load time, outside stream capture. */
NVC_API int nvc_cook_mesh_vertices(NvcContext* ctx, void* stream, const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* indices,
    uint32_t index_count, const NvcMesh* host_meshes, uint32_t mesh_count, NvcMesh* meshes, NvcVertex* vertices_out, uint32_t vertex_capacity,
    uint32_t* lod0_out, uint32_t index_capacity, uint32_t* totals4);

/* ---- OBJ import (loadMesh's loadObj, src/scene.cpp:117-168, over extern/fast_obj) --------------------------------------------- */
typedef struct NvcObjFile
{
	const void* data; /* host: the file's bytes, as read from disk */
	uint64_t size;
} NvcObjFile;

typedef struct NvcObjInfo
{
	uint64_t bytes_parsed;                                  /* where fast_obj's reader stops (the 64 KiB rule below) */
	uint32_t position_count, texcoord_count, normal_count; /* v / vt / vn lines; the dummy element 0 is not counted */
	uint32_t face_count;                                    /* faces pushed */
	uint64_t index_count;                                   /* index records pushed, orphans included */
	uint64_t corner_offset, corner_count;                   /* the file's range of `vertices`: the sum of 3 * (face_vertices - 2) */
} NvcObjInfo;

/* Loads OBJ files on the device: `vertices` gets, file after file, the Vertex[] the reference's loadObj returns for each, bit
 * for bit (one 16-byte record per triangle corner: fp16 position, tp 0, three 10-bit snorm normal fields + 511, fp16 texcoord).
 *   files / file_count   host: each file's bytes; they are uploaded into context-owned scratch
 *   vertices             device out (16-byte aligned), or NULL to query: then only `infos` is written
 *   vertex_capacity      records `vertices` holds; below the call's corners: NVC_ERROR_INVALID_ARGUMENT, `infos` still filled
 *   infos                host out, file_count entries
 * loadMesh gives appendMesh the identity indices, so file f is nvc_cook_mesh_vertices' mesh with vertexOffset = corner_offset,
 * vertexCount = corner_count and lods[0] = { corner_offset, corner_count } over the indices 0..n-1.
 * The file is parsed as fast_obj parses it: read in 64 KiB blocks of whole lines, a full block without '\n' ends the parse (a
 * line of more than 64 KiB truncates the file there), a final line without '\n' is parsed.  `v` pushes 3 numbers, `vt` 2,
 * `vn` 3, missing ones 0; `f` pushes one index record per `v`, `v/t`, `v//n` or `v/t/n`, negative indices relative to the
 * counts at that line, and a vertex index of 0 (or anything that is not a number) ends the line without a face, the records
 * before it staying in the index stream, which loadObj walks by the running sum of the face sizes.  Every other line is
 * ignored; `mtllib` is not followed (materials cannot change loadObj's output, and there is no base path for file bytes).  A
 * number is accumulated as fast_obj does in binary64; a NaN it produces is 0xffc00000, as on x86, the reference's platform.
 * Refusals, decided before anything is written to `vertices`:
 *   NVC_ERROR_CORRUPT       a face of fewer than 3 vertices, or a corner loadObj reads with a position, texcoord or normal
 *                           index past the file's final count (the reference crashes or reads out of bounds on these);
 *                           `infos` is filled, with such faces counted as 0 corners
 *   NVC_ERROR_UNSUPPORTED   4 GiB or more of files in one call, 2^32 or more corners in one call, or a file whose arrays
 *                           would overflow fast_obj's 32-bit sizes; `infos` is filled when the files were parsed
 *   NVC_ERROR_INVALID_ARGUMENT  a NULL context or infos, a NULL file with bytes, a misaligned `vertices`, or the capacity above
 * Index values of 10 or more digits wrap modulo 2^32, as the reference's x86 build does.  Scratch is context-owned (about
 * 90 bytes per line, 12 per index record and 24 per face, plus the files); the call synchronises the device before it touches it, after
 * the upload and before it reads back the counts and flags, and enqueues its kernels on `stream`: call it at load time,
 * outside stream capture. */
NVC_API int nvc_obj_load(NvcContext* ctx, void* stream, const NvcObjFile* files, uint32_t file_count, NvcVertex* vertices, uint64_t vertex_capacity,
    NvcObjInfo* infos);

#ifdef __cplusplus
} /* extern "C" */

static_assert(sizeof(NvcVertex) == 16, "Vertex must match src/scene.h:51-57");
static_assert(sizeof(NvcMeshlet) == 24, "Meshlet must match src/shaders/mesh.h:11-24");
static_assert(sizeof(NvcMeshLod) == 20, "MeshLod must match src/shaders/mesh.h:53-60");
static_assert(sizeof(NvcMesh) == 208, "Mesh must match src/shaders/mesh.h:62-78");
static_assert(sizeof(NvcMeshDraw) == 48, "MeshDraw must match src/shaders/mesh.h:92-102");
static_assert(sizeof(NvcMeshDrawCommand) == 24, "MeshDrawCommand must match src/shaders/mesh.h:104-114");
static_assert(sizeof(NvcMeshTaskCommand) == 20, "MeshTaskCommand must match src/shaders/mesh.h:116-123");
static_assert(sizeof(NvcCullData) == 144, "CullData must match src/niagara.cpp:242-260 (alignas 16)");
static_assert(offsetof(NvcMesh, lods) == 48, "Mesh::lods offset");
static_assert(offsetof(NvcMesh, lodCount) == 32, "Mesh::lodCount offset");
static_assert(offsetof(NvcMeshDraw, meshIndex) == 32, "MeshDraw::meshIndex offset");
static_assert(offsetof(NvcMeshlet, cone_axis) == 8, "Meshlet::cone_axis offset");
static_assert(offsetof(NvcMeshlet, dataOffset) == 12, "Meshlet::dataOffset offset");
static_assert(offsetof(NvcCullData, P00) == 64, "CullData::P00 offset");
static_assert(offsetof(NvcCullData, frustum) == 80, "CullData::frustum offset");
static_assert(offsetof(NvcCullData, lodTarget) == 96, "CullData::lodTarget offset");
static_assert(offsetof(NvcCullData, drawCount) == 108, "CullData::drawCount offset");
static_assert(offsetof(NvcCullData, clusterBackfaceEnabled) == 128, "CullData::clusterBackfaceEnabled offset");
static_assert(offsetof(NvcCullData, postPass) == 132, "CullData::postPass offset");
static_assert(sizeof(NvcSceneCacheHeader) == 160, "SceneHeader must match src/scenecache.cpp:16-55");
static_assert(offsetof(NvcSceneCacheHeader, compressedVertexBytes) == 28 && offsetof(NvcSceneCacheHeader, vertexCount) == 44, "SceneHeader offsets");
static_assert(offsetof(NvcSceneCacheHeader, camera) == 108 && offsetof(NvcSceneCacheHeader, sunDirection) == 144, "SceneHeader offsets");
static_assert(sizeof(NvcKeyframe) == 32 && sizeof(NvcAnimation) == 24, "Keyframe / Animation must match src/scene.h:141-161");
#endif

#endif /* NIAGARA_CULL_H */
