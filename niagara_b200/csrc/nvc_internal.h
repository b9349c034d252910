// nvc_internal.h — types shared between the C ABI (nvc_api.cu) and the kernels (nvc_kernels.cu).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <initializer_list>
#include <string>

#include "../../include/niagara_cull.h"

namespace nvc
{
struct Scratch;
}

struct NvcContext
{
	int device = 0;
	int sm_count = 0;
	int cluster_blocks_early = 0, cluster_blocks_late = 0, cluster_blocks_late_staged = 0;
	int cluster_filter_blocks_early = 0, cluster_filter_blocks_late = 0;
	bool draw_filter = false;   // env NVC_DRAW_FILTER=1: filtered occlusion stage of the late drawcull (off by default: the pass is not issue bound)
	bool cluster_filter = true; // nvc_set_cluster_filter / env NVC_CLUSTER_FILTER: filtered cluster kernel (default) or the exact one
	bool mesh_cull = false;     // nvc_set_mesh_cull: the mesh shader's per-triangle cull stage (MESH_CULL) in the cluster-mode depth producers
	bool task_cull = true;      // nvc_set_task_cull: meshlet culling in the cluster / task passes (TASK_CULL); off = pass-through
	uint32_t hiz_stage_budget = 0; // texels (24 KB) of coarse Hi-Z mips staged per CTA; 0 = off (env NVC_HIZ_STAGE_TEXELS)
	NvcLimits limits = { NVC_TASK_WGLIMIT, NVC_CLUSTER_LIMIT };
	nvc::Scratch* scratch = nullptr;
	std::string last_error;
	void* nccl_comm = nullptr; // ncclComm_t, owned (nvc_nccl.cpp)
	void* gather = nullptr;    // NvcGather, owned (nvc_peer.cu)
	// derived mesh cull view (nvc_prepare_meshes)
	const void* prepared_meshes = nullptr;
	uint32_t prepared_mesh_count = 0;
	void* mesh_heads = nullptr;
	float* mesh_errors = nullptr;
	// derived meshlet cull view (nvc_prepare_meshlets): bytes 0-7 and 8-11 of every Meshlet record
	const void* prepared_meshlets = nullptr;
	uint2* meshlet_sphere = nullptr;
	uint32_t* meshlet_cone = nullptr;
	int nccl_rank = 0, nccl_world = 1;
	// footprint image of one pyramid (nvc_prepare_hiz): keyed by the pyramid's texel pointer and shape
	float* hiz_fp = nullptr;
	const float* hiz_fp_key = nullptr;
	uint32_t hiz_fp_width = 0, hiz_fp_height = 0, hiz_fp_levels = 0, hiz_fp_total = 0;
	uint32_t hiz_fp_first = 0; // first mip with a footprint image (env NVC_FP_FIRST_LEVEL)
	uint32_t hiz_fp_offset[NVC_MAX_HIZ_LEVELS] = {};
	bool hiz_fp_valid = false; // set by nvc_depth_pyramid, cleared by nvc_prepare_hiz
	// the load-time calls' scratch, grown as needed (nvc::reserve_scratch): the cookers' job tables and per-job arrays, the
	// staged streams of nvc_scene_cache_read_device, the inputs and encoded streams of nvc_scene_cache_write.  Each of these
	// calls synchronises the device before it touches it, so one call's use has ended when the next one's begins.
	void* load_scratch = nullptr;
	size_t load_scratch_bytes = 0;
};

namespace nvc
{
void nccl_destroy(NvcContext* ctx);   // nvc_nccl.cpp
void gather_destroy(NvcContext* ctx); // nvc_peer.cu
uint32_t* gather_fused_target(NvcContext* ctx);
uint32_t gather_reserved_blocks(NvcContext* ctx); // nvc_peer.cu: CTA slots the persistent cluster grid leaves to the exchange's kernels // nvc_peer.cu: multicast destination of the armed late drawcull, or nullptr (disarms)

// Calls that work on the caller's stream need the context's device to be current (the reference drives one VkDevice from
// one thread; nothing here switches devices behind the caller's back).
inline bool device_is_current(NvcContext* ctx)
{
	int current = -1;
	if (cudaGetDevice(&current) != cudaSuccess || current != ctx->device)
	{
		ctx->last_error = "the context's CUDA device is not the calling thread's current device";
		return false;
	}
	return true;
}

// A failed CUDA step of the call `what`, named with the error in nvc_last_error: NVC_ERROR_CUDA
inline int cuda_fail(NvcContext* ctx, cudaError_t e, const char* what)
{
	if (ctx)
		ctx->last_error = std::string(what) + ": " + cudaGetErrorString(e);
	return NVC_ERROR_CUDA;
}
// as cuda_fail, but a failed allocation is NVC_ERROR_OUT_OF_MEMORY: the scene-cache calls' steps, and the cookers' growth of
// the load-time scratch
inline int load_fail(NvcContext* ctx, cudaError_t e, const char* what)
{
	cuda_fail(ctx, e, what);
	return e == cudaErrorMemoryAllocation ? NVC_ERROR_OUT_OF_MEMORY : NVC_ERROR_CUDA;
}

// Device-side counters owned by the context.  Each pass's last-block epilogue leaves them zeroed, which replaces
// the reference's vkCmdFillBuffer resets (niagara.cpp:1541,1586) and keeps every pass a single launch.
// Hot atomics live on separate 128-byte lines.
struct alignas(128) Scratch
{
	uint32_t draw_counter;
	uint32_t pad0[31];
	uint32_t draw_done;
	uint32_t pad1[31];
	uint32_t cluster_counter;
	uint32_t pad2[31];
	uint32_t cluster_done;
	uint32_t pad3[31];
	uint32_t cluster_batch;
	uint32_t pad4[31];
	uint32_t pyramid_done;
	uint32_t pad5[31];
	// filtered cluster pass, cumulative since the last nvc_filter_stats(reset): meshlets evaluated, meshlets that took the exact path
	unsigned long long filter_items, filter_undecided;
	uint32_t pad6[28];
	// mesh-cull stage of the depth producers (nvc_set_mesh_cull), cumulative since the last nvc_mesh_cull_stats(reset): triangles
	// tested, triangles culled
	unsigned long long mesh_cull_tested, mesh_cull_culled;
	uint32_t pad7[28];
};

// row pitch of a footprint-image level of width w (w + 1 entries per row, padded so that every row starts 16-byte aligned)
#if defined(__CUDACC__)
__host__ __device__
#endif
inline uint32_t fp_pitch(uint32_t w)
{
	return (w + 4u) & ~3u;
}

struct HiZDesc
{
	float* texels;
	uint32_t width, height, levels;
	uint32_t level_offset[NVC_MAX_HIZ_LEVELS];
	// mips >= stage_level (the coarse tail of the packed pyramid, stage_texels texels) are staged into shared memory
	// once per CTA with one TMA bulk copy; stage_level == levels disables staging
	uint32_t stage_level, stage_texels;
	// Footprint image (nvc_prepare_hiz; built by nvc_depth_pyramid): for every mip, F(i, j) = min of the 2 x 2 texel
	// footprint whose lower corner is (i, j), i in [-1, w-1], j in [-1, h-1], indices clamped to the level — what the
	// MIN-reduction sampler returns for any coordinate whose bilinear footprint starts there (resources.cpp:294-325).
	// Level l: fp + fp_offset[l], pitch w + 1, entry (i + 1, j + 1).  fp == nullptr: not available.
	// Level l: fp + fp_offset[l], row pitch fp_pitch(w) (a multiple of four entries: rows are 16-byte aligned), entry (i + 1, j + 1).
	// Only mips >= fp_first have an image (the finest mips hold 15/16 of the texels and are sampled by sub-8-pixel spheres only;
	// lookups into them take the four texel loads).
	const float* fp;
	uint32_t fp_offset[NVC_MAX_HIZ_LEVELS];
	uint32_t fp_first;
};

// Derived, read-only cull view of the reference's 208-byte Mesh records, built once per geometry upload by
// nvc_prepare_meshes: one 32-byte head per mesh (everything a single-LOD / LOD-0 task draw needs = ONE sector instead
// of the 3-4 sectors the AoS struct spreads it over) and the 8 LOD errors as a second 32-byte record.
struct MeshCullHead
{
	float center[3];
	float radius;
	uint32_t lodCount;
	uint32_t lod0MeshletOffset;
	uint32_t lod0MeshletCount;
	uint32_t vertexOffset;
};
static_assert(sizeof(MeshCullHead) == 32, "one sector");

// Per-launch constants of the conservative meshlet filter (nvc_filter.cuh; host-computed by make_filter_consts).
// Grouped in 16-byte vectors in the order the kernel consumes them, so that each group is ONE uniform load per chunk.
struct FilterConsts
{
	float4 fr;        // mFk (frustum margin = mFk * E), zfarLo, zfarHi (zfar (1 -+ 2^-20)), zn4u (4 u znear, enters Et)
	float4 pr;        // hPx, hPyn (0.5 P00, -0.5 P11), sxk, syk (size.x * pyramidWidth = r vx icz sxk, sxk = 2 hPx pw; same for y)
	float4 cg;        // kGx, kGrx, kGy, kGry: validity cone per axis |cx| + r kGrx <= kGx cz (kGx = 1 / hPx, kGrx = sqrt(1 + kGx^2))
	float4 mk;        // Km1, Km2 (dm = gr (Km1 + Km2 m)), KuvP (max(pw, ph) Kuv 1.05), Kfp (footprint margin = Kfp whf gr)
	uint4 lv;         // float bits of 2^levels, 2^(levels-1), (float)hiz.width, (float)hiz.height
	float vrE;        // max(max row abs sum of V3, 1)
	float Kuv;        // uv error = Kuv g relE (informational; folded into KuvP / Kfp)
	uint32_t enabled; // 0: every item is undecided (unusual view / projection: the exact path does everything)
	uint32_t occ_ok;  // 0: the occlusion stage is never decided here (non power-of-two pyramid, ...)
};

struct DrawCullParams
{
	NvcCullData cull;
	const NvcMeshDraw* draws;
	const NvcMesh* meshes;
	const MeshCullHead* mesh_heads; // may be null: read everything from `meshes`
	const float* mesh_errors;       // [mesh][8], valid when mesh_heads != null
	uint32_t* draw_visibility;
	void* commands;
	uint32_t* command_count4;
	Scratch* scratch;
	HiZDesc hiz;
	uint32_t task_wglimit;
	// multi-GPU, fused all-gather (nvc_gather_fuse_next_drawcull): NVSwitch multicast alias of THIS rank's slot in every
	// rank's gathered slab buffer; every command the pass writes to `commands` is also stored there (replicated by the
	// switch to all ranks), so the exchange happens inside the producing kernel.  nullptr: not fused.
	uint32_t* mc_commands;
	// late pass: the occlusion stage runs as a conservative filter on the exact centre; undecided draws take the exact path
	FilterConsts filter;
	uint32_t use_filter;
};

struct ClusterParams
{
	NvcCullData cull;
	const NvcMeshTaskCommand* task_commands;
	const uint32_t* command_count4;
	const NvcMeshDraw* draws;
	const NvcMeshlet* meshlets;
	// Where the 12 bytes the cluster tests read live for meshlet i: bytes 0-7 (center[3], radius as binary16) at
	// ml_sphere + i * ml_sphere_stride, bytes 8-11 (cone_axis[3], cone_cutoff as s8) at ml_cone + i * ml_cone_stride.
	// Either the prepared view of `meshlets` (nvc_prepare_meshlets: strides 8 and 4) or the records themselves (stride 24),
	// resolved on the host so that the kernels' address arithmetic has no branch.
	const char* ml_sphere;
	const char* ml_cone;
	uint32_t ml_sphere_stride, ml_cone_stride;
	uint32_t* meshlet_visibility;
	uint32_t* cluster_indices;
	uint32_t* cluster_count4;
	Scratch* scratch;
	HiZDesc hiz;
	uint32_t cluster_limit;
	// task-shading submission mode (meshlet.task.glsl): per-command payloads + emit counts instead of cib / ccb
	NvcMeshTaskPayload* payloads;
	uint32_t* emit_counts;
	FilterConsts filter; // valid when use_filter
	uint32_t use_filter; // 1: clustercull_filter_kernel (conservative filter + exact fallback), 0: the exact kernel
};

struct PyramidParams
{
	const float* depth;
	uint32_t depth_width, depth_height;
	HiZDesc hiz;
	Scratch* scratch;
	uint32_t vector_ok; // set by launch_pyramid: bases aligned for 16-byte loads
};

cudaError_t launch_drawcull(const DrawCullParams& p, bool late, bool task, cudaStream_t stream);
cudaError_t launch_clustercull(const ClusterParams& p, bool late, uint32_t blocks, cudaStream_t stream);
cudaError_t launch_taskcull(const ClusterParams& p, bool late, NvcMeshTaskPayload* payloads, uint32_t* emit_counts, uint32_t blocks, cudaStream_t stream);
// TASK_CULL = 0: the cluster / task passes without meshlet tests (read only the task commands and their count)
cudaError_t launch_clustercull_passthrough(const ClusterParams& p, uint32_t blocks, cudaStream_t stream);
cudaError_t launch_taskcull_passthrough(const NvcMeshTaskCommand* task_commands, const uint32_t* command_count4, NvcMeshTaskPayload* payloads, uint32_t* emit_counts, uint32_t blocks,
    cudaStream_t stream);
cudaError_t launch_pyramid(const PyramidParams& p, cudaStream_t stream);
cudaError_t launch_footprint(const HiZDesc& hiz, float* fp, uint32_t total, cudaStream_t stream);
cudaError_t launch_decode_clusters(const uint32_t* cluster_indices, const uint32_t* cluster_count4, const NvcMeshTaskCommand* task_commands, const NvcMeshlet* meshlets, NvcClusterRecord* records, uint32_t* stats4, uint32_t blocks, cudaStream_t stream);
cudaError_t launch_raster_depth(const float* projection16, const NvcCullData& pass, const uint32_t* cluster_indices, const uint32_t* cluster_count4, const NvcMeshTaskCommand* task_commands,
    const NvcMeshDraw* draws, const NvcMeshlet* meshlets, const uint32_t* meshletdata, uint32_t meshletdata_words, const NvcVertex* vertices, uint32_t vertex_count, float* depth, uint32_t width,
    uint32_t height, uint32_t* stats4, unsigned long long* mesh_cull2, uint32_t blocks, cudaStream_t stream);
cudaError_t launch_raster_depth_tasks(const float* projection16, const NvcCullData& pass, const NvcMeshTaskPayload* payloads, const uint32_t* emit_counts, const uint32_t* command_count4,
    const NvcMeshTaskCommand* task_commands, const NvcMeshDraw* draws, const NvcMeshlet* meshlets, const uint32_t* meshletdata, uint32_t meshletdata_words, const NvcVertex* vertices,
    uint32_t vertex_count, float* depth, uint32_t width, uint32_t height, uint32_t* stats4, unsigned long long* mesh_cull2, uint32_t blocks, cudaStream_t stream);
cudaError_t launch_raster_depth_indexed(const float* projection16, const NvcCullData& pass, const NvcMeshDrawCommand* draw_commands, const uint32_t* command_count4, uint32_t max_draw_count,
    const NvcMeshDraw* draws, const uint32_t* indices, uint32_t index_count, const NvcVertex* vertices, uint32_t vertex_count, float* depth, uint32_t width, uint32_t height, uint32_t* stats4,
    uint32_t blocks, cudaStream_t stream);
cudaError_t launch_cook_meshlet_bounds(const NvcVertex* vertices, uint32_t vertex_count, const uint32_t* meshletdata, uint32_t meshletdata_words, NvcMeshlet* meshlets, uint32_t meshlet_count, uint32_t* rejected, cudaStream_t stream);
namespace cook
{
struct CookJob;
}

// nvc_cook_meshlets: the jobs (one per mesh LOD, in mesh then LOD order), the order the build kernel takes them in, and the
// scratch the host planned for them (nvc_meshlets.cuh).  Every pointer is device memory.
struct CookArgs
{
	const NvcVertex* vertices;
	const uint32_t* indices;
	const cook::CookJob* jobs;
	const uint32_t* order; // job indices, largest first
	uint32_t job_count;
	uint32_t slot_count; // meshlet slots of all jobs (sum of their bounds)
	float* cones;        // 6 per triangle
	uint32_t* adj_counts; // per vertex: live triangles
	uint32_t* adj_offsets;
	uint32_t* adj_data;   // per index
	int16_t* used;        // per vertex
	uint8_t* emitted;     // per triangle
	uint32_t* kd_nodes;   // 2 nodes of 3 words per triangle
	uint32_t* kd_index;   // per triangle
	uint32_t* ml_vertices; // per index; also the triangle areas before the greedy loop
	uint8_t* ml_triangles; // per index
	uint4* ml_records;     // per slot: vertex offset, triangle offset, vertex count, triangle count
	uint32_t* job_meshlets; // per job: meshlets built
	uint32_t* job_first;    // per job: first output meshlet
	uint32_t* slot_words;   // per slot: meshletdata words (0 for an unused slot)
	uint32_t* slot_min;     // per slot: minVertex
	uint32_t* slot_data;    // per slot: dataOffset
	NvcMesh* meshes;
	NvcMeshlet* meshlets;
	uint32_t meshlet_capacity;
	uint32_t* meshletdata;
	uint32_t meshletdata_capacity;
	uint32_t* totals4;
};
cudaError_t launch_cook_meshlets(const CookArgs& a, cudaStream_t stream);
// nvc_cook_meshlets_clrt: `base` as above, with base.order = the greedy jobs (largest first) followed by the ray-tracing
// jobs (largest first), base.totals4 = totals8
struct CookClrtArgs
{
	CookArgs base;
	uint32_t greedy_count;  // base.order[0, greedy_count): meshopt_buildMeshlets jobs
	uint32_t rt_count;      // base.order[greedy_count, + rt_count): meshopt_buildMeshletsSpatial jobs
	const uint32_t* job_rt; // per job: 1 for the mesh's lodRT
	uint32_t* slot_vtx0;    // per slot: first meshletvtx0 element
	uint16_t* meshletvtx0;
	uint32_t meshletvtx0_capacity;
};
cudaError_t launch_cook_meshlets_clrt(const CookClrtArgs& c, cudaStream_t stream);
namespace lods
{
struct LodJob;
}
// nvc_cook_mesh_lods (nvc_lods.cuh): one job per mesh, in mesh order, and the order the chain kernel takes them in.  Every
// pointer is device memory.
struct LodArgs
{
	const NvcVertex* vertices;
	const uint32_t* lod0_indices;
	const lods::LodJob* jobs;
	const uint32_t* order;    // mesh indices, largest LOD 0 first
	const float* max_scale;   // per mesh
	uint32_t mesh_count;
	uint32_t* scratch;        // the jobs' scratch words
	uint64_t* chain;          // per mesh: indices of its chain
	uint8_t* rejected;        // per mesh
	uint64_t* base;           // per mesh: first output index
	NvcMesh* meshes;
	uint32_t* indices;
	uint32_t index_capacity;
	uint32_t* totals4;
};
cudaError_t launch_cook_mesh_lods(const LodArgs& a, cudaStream_t stream);
namespace scan
{
constexpr uint32_t kScanItems = 2048; // values per block of nvc_scan.cuh's device-wide scan
}
namespace verts
{
// per mesh: its input ranges, its first triangle and first vertex slot among the call's, and its vertex cache scratch
struct VertexJob
{
	uint32_t vertex_offset, vertex_count, index_offset, index_count;
	uint32_t tri_base, slot_base;
	uint64_t scratch;
};
}
// nvc_cook_mesh_vertices (nvc_vertices.cuh): one job per mesh, in mesh order.  T = the call's triangles, N = 3 T its index
// positions, S = the sum of the meshes' vertexCount (one slot per mesh vertex).  Every pointer is device memory.
struct VertexArgs
{
	const NvcVertex* vertices;
	const uint32_t* indices;
	const verts::VertexJob* jobs;
	const uint32_t* order; // mesh indices, longest LOD 0 first
	uint32_t mesh_count;
	uint32_t tri_count, position_count, slot_count; // T, N, S
	uint8_t* rejected;             // per mesh
	uint32_t* tri_table;           // hash_buckets(T): a triangle of each (mesh, rotated positions), the smallest
	uint32_t tri_mask;
	uint32_t* tri_entry;           // T: the triangle's bucket, or ~0 when it is dropped before the table
	uint8_t* flags;                // N
	uint32_t* rank;                // N + 1: the last scan's result, its total last
	uint32_t* block_sums;          // ceil(N / scan::kScanItems)
	unsigned long long* offsets;   // that + 1
	uint32_t* filtered;            // N: the kept triangles' indices, mesh-local
	uint32_t* index_base;          // per mesh: its first filtered (= output) index
	uint32_t* vertex_base;         // per mesh: its first class (= output vertex)
	uint32_t* first;               // S: the first filtered position referencing the slot, ~0 when none
	uint32_t* vtx_table;           // hash_buckets(S): a slot of each (mesh, 16 vertex bytes)
	uint32_t* vtx_first;           // hash_buckets(S): the smallest `first` of the entry's class
	uint32_t vtx_mask;
	uint32_t* vtx_entry;           // S: the slot's bucket
	NvcVertex* classes;            // S: the class vertices, in class order
	uint32_t* remapped;            // N: the filtered indices remapped to classes
	uint32_t* first_use;           // S: per class, its first position in the optimised indices
	uint32_t* scratch;             // the jobs' vertex cache words
	NvcMesh* meshes;
	NvcVertex* vertices_out;
	uint32_t* lod0_out;
	uint32_t* totals4;
};
cudaError_t launch_cook_mesh_vertices(const VertexArgs& a, cudaStream_t stream);
// the vertex cache scratch words of a mesh with at most `vertices` vertices and `indices` indices
uint64_t vertex_cache_words(uint32_t vertices, uint32_t indices);
namespace obj
{
constexpr uint32_t kTileBytes = 4096;   // bytes per line-index tile: 256 threads x 16
constexpr uint32_t kBlockBytes = 65536; // fast_obj's read block
constexpr uint32_t kTilesPerBlock = kBlockBytes / kTileBytes;
// the per-line counts, scanned into per-line prefixes over the call's lines
enum Field : uint32_t
{
	kPositions,
	kTexcoords,
	kNormals,
	kRecords,     // index records pushed, orphans included
	kFaces,       // faces pushed
	kFaceIndices, // a face's vertex count, 0 for other lines: the running sum locates loadObj's windows
	kCorners,     // 3 * (vertices - 2) for a face of 3 or more vertices
	kFields
};
constexpr uint32_t kBadFace = 1;  // a face of fewer than 3 vertices
constexpr uint32_t kBadIndex = 2; // a corner loadObj reads has an index past the file's final count
// per file, host-built, plus a sentinel whose tile_base is the call's tile count
struct File
{
	uint64_t data;      // its first byte in ObjArgs::text (16-byte aligned)
	uint32_t size;
	uint32_t tile_base; // its first tile among the call's
};
// per file, device-computed
struct FileState
{
	uint32_t cut;        // the first full 64 KiB block without '\n' (the reader stops there), ~0 when none
	uint32_t first_line; // its first line slot: the '\n' bytes of the files before it + its index
	uint32_t line_count; // the lines the reader parses
	uint32_t flags;      // kBadFace | kBadIndex
	uint32_t positions, texcoords, normals; // final counts (v, vt and vn lines parsed)
	uint32_t pad;
	uint64_t position_base, texcoord_base, normal_base; // its element 0 (the dummy) in the call's arrays
};
struct Record
{
	uint32_t p, t, n; // resolved as fast_obj resolves them, file-local
};
struct Face
{
	uint32_t window; // its first index record: the file's first record + the face vertices of the file's earlier faces
	uint32_t count;
	uint32_t file, pad;
	uint64_t corner; // its first output record
};
}
// nvc_obj_load (nvc_obj.cuh).  L = the call's line slots: its '\n' bytes plus one per file (a final line without '\n').
// Every pointer is device memory.
struct ObjArgs
{
	const uint8_t* text;
	const obj::File* files; // file_count + 1
	uint32_t file_count, tile_count;
	uint32_t* tile_lines;                 // per tile: its '\n' bytes
	unsigned long long* tile_offsets;     // tile_count + 1: their exclusive scan
	uint32_t line_slots;                  // L
	uint32_t* line_end;                   // L: the line's '\n' (or the file's end), file-relative
	obj::FileState* state;                // file_count
	uint32_t* counts;                     // kFields x L
	uint32_t* block_sums;                 // kFields x ceil(L / scan::kScanItems)
	unsigned long long* block_offsets;    // kFields x (ceil(L / scan::kScanItems) + 1)
	unsigned long long* prefix;           // kFields x (L + 1): exclusive scans of `counts`, the totals last
	float* positions;                     // 3 per element, each file's dummy first
	float* texcoords;                     // 2 per element
	float* normals;                       // 3 per element
	obj::Record* records;                 // the index stream
	obj::Face* faces;                     // the face list
	uint32_t face_count;
	uint64_t corner_count;
	NvcObjInfo* infos;                    // file_count
	NvcVertex* vertices;
};
// line index: the tiles' '\n' counts and their scan
cudaError_t launch_obj_lines(const ObjArgs& a, cudaStream_t stream);
// line ends, the reader's cut, per-line counts and their scans, per-file infos
cudaError_t launch_obj_count(const ObjArgs& a, cudaStream_t stream);
// numbers, index records, faces, the range check
cudaError_t launch_obj_parse(const ObjArgs& a, cudaStream_t stream);
// the Vertex[] records
cudaError_t launch_obj_expand(const ObjArgs& a, cudaStream_t stream);
// nvc_scene_cache_read_device (nvc_cache_decode.cuh).  Every pointer is device memory; `stream` is the section as stored,
// padded so that word loads that cover its last byte stay inside the allocation.
struct VertexDecodeArgs
{
	const uint8_t* stream;
	const uint32_t* block_start;  // [blocks + 1] (walk_vertex_stream)
	const uint16_t* plane_offset; // [blocks][stride]
	uint32_t* out;                // vertex_count * stride / 4 words
	uint32_t* carry;              // [blocks][stride / 4]: block totals, then carries
	uint32_t vertex_count, blocks, version;
	uint32_t baseline[4]; // per 4-byte column: the baseline vertex of the stream's tail
	uint32_t channel[4];  // per column: the channel byte of a v1 tail, 0 for v0
};
cudaError_t launch_decode_vertices(const VertexDecodeArgs& a, uint32_t stride, cudaStream_t stream);
struct MeshletDecodeArgs
{
	const uint8_t* stream;
	const uint32_t* checkpoints; // [groups of 32 meshlets + 1]: offset of the group's first size field (index_meshlet_stream)
	const uint32_t* records;     // [meshlets][2]: dataOffset, vertexCount | triangleCount << 8 | shortRefs << 16
	uint32_t* out;               // meshletdata words, zeroed
	uint32_t meshlet_count;
	uint32_t* corrupt; // set to 1 by a malformed block
};
cudaError_t launch_decode_meshlets(const MeshletDecodeArgs& a, cudaStream_t stream);
constexpr uint32_t kIndexChunk = 256;   // triangles per chunk of the index decoder
constexpr uint32_t kIndexRun = 256;     // chunks per run of its combine step
constexpr uint32_t kIndexEntries = 51;  // uint2 words of a chunk's state substitution (nvc_cache_decode.cuh)
struct IndexDecodeArgs
{
	const uint8_t* stream;      // the section as stored
	const uint64_t* chunk_data; // [chunks]: offset of each chunk's first data byte in `stream` (walk_index_stream)
	uint2* sub;                 // [kIndexEntries][chunks]: each chunk's substitution, then its entry state
	uint2* run;                 // [kIndexEntries][runs]: each run's substitution, then its entry state
	uint32_t* out;              // triangles * 3 indices
	uint64_t aux_offset;        // of the 16-byte aux table in `stream`
	uint32_t triangles, chunks, runs, direct_slots;
};
cudaError_t launch_decode_indices(const IndexDecodeArgs& a, cudaStream_t stream);
// Sub-allocations of the context's load-time scratch, each 256-byte aligned; `bytes` ends where the last one does
struct ScratchPlan
{
	size_t bytes = 0;
	size_t take(size_t n)
	{
		size_t at = (bytes + 255) & ~size_t(255);
		bytes = at + n;
		return at;
	}
};
// grows the context's load-time scratch to `bytes`; its previous user has finished (the caller synchronised the device)
inline cudaError_t reserve_scratch(NvcContext* ctx, size_t bytes)
{
	if (bytes <= ctx->load_scratch_bytes)
		return cudaSuccess;
	cudaFree(ctx->load_scratch);
	ctx->load_scratch = nullptr;
	ctx->load_scratch_bytes = 0;
	cudaError_t e = cudaMalloc(&ctx->load_scratch, bytes);
	if (e == cudaSuccess)
		ctx->load_scratch_bytes = bytes;
	return e;
}
// One host-to-device copy of a load-time call; a copy of 0 bytes is skipped.
struct Upload
{
	void* dst;
	const void* src;
	size_t bytes;
};
// A copy from pageable host memory may return before its DMA has landed, and it is not ordered with a non-blocking stream:
// the copies are followed by a device synchronise, before a kernel reads them or the call returns.
inline cudaError_t upload(std::initializer_list<Upload> copies)
{
	for (const Upload& c : copies)
		if (c.bytes)
		{
			cudaError_t e = cudaMemcpy(c.dst, c.src, c.bytes, cudaMemcpyHostToDevice);
			if (e != cudaSuccess)
				return e;
		}
	return cudaDeviceSynchronize();
}
// nvc_scene_cache_write (nvc_cache_encode.cuh).  Every pointer is device memory.
constexpr uint32_t kVertexBlockEncode = 256; // vcodec::block_vertices of strides 8 and 16
struct VertexEncodeArgs
{
	const uint8_t* vertices;       // vertex_count * stride bytes, 4-byte aligned
	uint32_t vertex_count, blocks; // blocks of kVertexBlockEncode vertices
	unsigned long long* estimate;  // [stride / 4][2]: per column the channel estimate's byte counts of channels 0 and 1
	uint32_t* block_bytes;         // [blocks]: each block's size (measure pass)
	unsigned long long* offsets;   // [blocks + 1]: their exclusive scan, then the total
	uint8_t* out;                  // the stream: header byte, blocks, tail
};
// estimate, measure, scan, write; the stream takes 1 + offsets[blocks] + 24 bytes.  vertex_count > 0.
cudaError_t launch_encode_vertices(const VertexEncodeArgs& a, uint32_t stride, cudaStream_t stream);
struct MeshletEncodeArgs
{
	const NvcMeshlet* meshlets;
	const uint32_t* meshletdata;
	uint32_t meshlet_count, meshletdata_count;
	uint32_t* block_bytes;       // [meshlets]: 2 + each meshlet's block size (measure pass)
	unsigned long long* offsets; // [meshlets + 1]: their exclusive scan, then the section's size
	uint8_t* out;                // the MESHLETDATA section
	uint32_t* invalid;           // zeroed; set to 1 by a meshlet outside meshletdata or past 64 vertices / 96 triangles
};
// measure, scan, write (the write pass skips the meshlets the measure pass flagged)
cudaError_t launch_encode_meshlets(const MeshletEncodeArgs& a, cudaStream_t stream);
cudaError_t launch_update_draws(NvcMeshDraw* draws, uint32_t draw_count, const uint32_t* update_indices, const NvcMeshDraw* update_values, uint32_t count, cudaStream_t stream);
cudaError_t launch_filter_approx(const uint32_t* in, uint32_t* out, uint64_t n, int op, cudaStream_t stream);
cudaError_t launch_pack_meshes(const NvcMesh* meshes, uint32_t count, MeshCullHead* heads, float* errors, cudaStream_t stream);
cudaError_t launch_pack_meshlets(const NvcMeshlet* meshlets, uint32_t count, uint2* sphere, uint32_t* cone, cudaStream_t stream);
cudaError_t clustercull_occupancy(int* blocks_per_sm_early, int* blocks_per_sm_late, int* blocks_per_sm_late_staged, uint32_t stage_bytes);
cudaError_t clustercull_filter_occupancy(int* blocks_per_sm_early, int* blocks_per_sm_late);
uint32_t hiz_stage_bytes(const HiZDesc& hiz);
void choose_stage_public(HiZDesc& hz, uint32_t total_texels, uint32_t budget_texels);

} // namespace nvc
