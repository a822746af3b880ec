/* include/tinybvh_b200.h - the drop-in boundary: a C-ABI over the H100 (sm_90a) engine.
 *
 * Plain pointers and sizes only; no torch / C++ types.  Each entry point names the reference interface it
 * replaces (file:line under the jbikker/tinybvh checkout, v1.6.7).  The C++ shim that keeps tinybvh's class
 * and method names on top of this ABI is include/tinybvh_b200.hpp; the reference-side binding a maintainer
 * would add is shown in INTEGRATION.md.
 *
 * Conventions
 *  - every function returns TBVH_OK (0) or a negative TBVH_E_* code; tbvh_last_error() gives the message
 *    (the reference has no error codes: BVH_FATAL_ERROR prints and exit(1)s, tiny_bvh.h:1617-1620 - the
 *    shim maps non-zero to that behaviour).
 *  - there is NO CPU fallback: without a CUDA device every call that touches data fails with TBVH_E_CUDA.
 *  - `space` says where a caller pointer lives: TBVH_HOST or TBVH_DEVICE (device pointers are plain
 *    CUdeviceptr values of the context's device, e.g. torch tensor data_ptr()).
 *  - device-space INPUTS (vertices, indices, node arrays passed with TBVH_DEVICE) are read on the engine's own stream: the caller
 *    makes sure the work that produces them has completed (synchronise the producing stream) before the call.  The *_device
 *    traversal calls are the exception: they run on the stream the caller passes.
 *  - host batch calls (tbvh_intersect / _packed / tbvh_occluded) may be issued from several threads on one handle, as the
 *    reference's const Intersect / IsOccluded are (tiny_bvh_speedtest.cpp:392-401); they are serialised per context.  Builds,
 *    uploads, conversions and refits are exclusive, like the reference's Build.
 *  - ray records are the reference's `Ray` (tiny_bvh.h:688-709): O at byte 0, D at 16, rD at 32, hit
 *    (t,u,v,prim) at 48..63; `stride` is 128 for the host struct, 64 for the packed GPU record
 *    (traverse.cl:11-17).  hit.t on entry is the ray's maximum distance.
 */
#ifndef TINYBVH_B200_H
#define TINYBVH_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TBVH_OK 0
#define TBVH_E_CUDA -1      /* CUDA runtime / driver error, or no device */
#define TBVH_E_ARG -2       /* invalid argument */
#define TBVH_E_STATE -3     /* handle does not hold the requested layout */
#define TBVH_E_LIMIT -4     /* tree exceeds a device limit (e.g. depth > traversal stack) */
#define TBVH_E_UNSUPPORTED -5

#define TBVH_HOST 0
#define TBVH_DEVICE 1

/* layouts a handle can hold (values follow BVHBase::BVHType, tiny_bvh.h:773-793) */
#define TBVH_LAYOUT_BVH 1      /* Wald 32-byte nodes, BVH::BVHNode tiny_bvh.h:861-869 */
#define TBVH_LAYOUT_BVH_GPU 5  /* Aila-Laine 64-byte nodes, BVH_GPU::BVHNode tiny_bvh.h:1095-1105 */
#define TBVH_LAYOUT_CWBVH 10   /* 80-byte compressed wide nodes + 48-byte triangles, tiny_bvh.h:1356-1359 */

typedef struct tbvh_ctx_t* tbvh_ctx;   /* one per CUDA device */
typedef struct tbvh_bvh_t* tbvh_bvh;   /* one acceleration structure (any subset of the layouts) */
typedef struct tbvh_group_t* tbvh_group; /* several devices of one process: BVH replicas + index-sharded ray batches */

typedef struct tbvh_info
{
	uint32_t prim_count;     /* BVHBase::triCount */
	uint32_t idx_count;      /* BVHBase::idxCount */
	uint32_t used_nodes;     /* BVH::usedNodes (32-byte nodes, node 1 unused) */
	uint32_t used_nodes_gpu; /* BVH_GPU::usedNodes (64-byte nodes) */
	uint32_t used_blocks;    /* BVH8_CWBVH::usedBlocks (16-byte blocks; nodes = used_blocks/5) */
	uint32_t cwbvh_tri_count;/* BVH8_CWBVH triangle records (48 bytes each) */
	uint32_t max_depth;      /* depth of the BVH2 (root = 0) */
	uint32_t layouts;        /* bit (1<<TBVH_LAYOUT_*) per resident layout */
	float aabb_min[3], aabb_max[3]; /* BVHBase::aabbMin / aabbMax */
	double build_ms;         /* device time of the last tbvh_build on this handle */
} tbvh_info;

/* ---- context ---------------------------------------------------------------------------------------- */
int tbvh_ctx_create( int device, tbvh_ctx* out );
int tbvh_ctx_destroy( tbvh_ctx ctx );
const char* tbvh_last_error( void );
int tbvh_device_count( void );
/* host topology of a device: the NUMA node it hangs off (-1 when the system does not say), and a call that restricts the calling
 * thread (and the threads it creates afterwards) to that node's CPUs - ray buffers first-touched or page-locked from such a thread
 * are read by the device's DMA engine from local memory instead of across the socket interconnect. */
int tbvh_device_numa_node( int device );
int tbvh_bind_thread_to_device( int device );
/* tuning knobs (no reference counterpart; defaults are the measured best): "trace_variant" 0 = generic BVH2 kernel,
 * 3 = octant-switch, 4 = persistent warps; "small_t" builder switch point (8..256); "d2h_mode" / "h2d_split" / "host_path"
 * select how the host-buffer path moves ray records and hits across PCIe ("host_path" 0 = copy engine 2D copies, the default;
 * 1 = gather kernel over the pinned mapping; "d2h_mode" 0 = 2D copy of the 16-byte hits into the records, 1 = bytes 0..63 of every record return (full cache lines), 2 = packed copy + host
 * threads scatter, 3 = scatter kernel over
 * the pinned mapping; "h2d_split" 1..4 inbound streams per chunk; "chunk_rays" rays per pipeline chunk, default 524288).
 * Environment variables TBVH_<KEY> set the defaults at context creation.  BuildHQ: "hq_small" (fragments below which a subtree goes to the warp kernel, default 16),
 * "hq_cluster" (largest thread-block cluster per node, 1..16).  "inst_idx_bits": the host program's INST_IDX_BITS (see
 * tbvh_build_tlas). */
int tbvh_set_option( tbvh_ctx ctx, const char* key, int value );
/* pinned host memory for ray buffers (replaces tinybvh::malloc64 / BVHContext::malloc for rays, tiny_bvh.h:261-292, 763-768).
 * The pages are taken from the NUMA node of the current CUDA device (tbvh_host_alloc) or of `device` (_near); buffers of 8 MiB and more
 * are anonymous memory advised into transparent huge pages and then page-locked (TBVH_HOST_HUGE=0 switches that off): with an IOMMU
 * translating the DMA engine's addresses, 2 MiB pages are worth 5-9 % on the host-buffer path. */
int tbvh_host_alloc( size_t bytes, void** out );
int tbvh_host_alloc_near( int device, size_t bytes, void** out );
int tbvh_host_alloc_node( int numa_node, size_t bytes, void** out );
int tbvh_host_free( void* p );
int tbvh_host_register( void* p, size_t bytes );
int tbvh_host_unregister( void* p );

/* ---- acceleration structure --------------------------------------------------------------------------- */
int tbvh_bvh_create( tbvh_ctx ctx, tbvh_bvh* out );
int tbvh_bvh_destroy( tbvh_bvh bvh );
int tbvh_bvh_info( tbvh_bvh bvh, tbvh_info* out );

/* BVH::Build( const bvhvec4*, primCount ) tiny_bvh.h:2124 / Build( bvhvec4slice ) :2131 - binned SAH on the GPU.
 * verts: prim_count*3 vertices, `stride` bytes apart (16 for bvhvec4), xyz used.  The engine copies them
 * (the reference keeps a pointer: "we're not copying this data").  c_trav / c_int = BVHBase::c_trav, c_int. */
int tbvh_build( tbvh_bvh bvh, const void* verts, uint32_t stride, uint32_t prim_count, int space, float c_trav, float c_int );

/* The same builder with the decisions of BVH::BuildAVX (tiny_bvh.h:6400-6671) - the builder BuildDefault (:1817-1832) picks
 * on x86, i.e. what BVH_GPU::Build, BVH8_CWBVH::Build and BVH8_CPU::Build construct their trees with.  It differs from
 * BVH::Build in bin rounding, the partition's bin function, minDim and the plane tie-break order; the trees are
 * "nearly identical" (:6352) but not byte-identical, so both flavours exist. */
#define TBVH_BUILD_REFERENCE 0   /* BVH::Build */
#define TBVH_BUILD_AVX 1         /* BVH::BuildAVX / BuildDefault */
/* BVH::BuildHQ (tiny_bvh.h:2623-3040): SBVH - object split vs. spatial split with clipping (ClipFrag :8614, SplitFrag :8731)
 * and unsplitting, followed by Compact() (:3733).  idx_count becomes prim_count + prim_count/2 as in the reference (the
 * leaves reference the first sum(triCount) entries; the rest is zero), used_nodes up to 3 * prim_count. */
#define TBVH_BUILD_HQ 2          /* BVH::BuildHQ */
/* Not a reference builder: parallel locally-ordered clustering (Meister & Bittner 2018), a bottom-up build for meshes rebuilt every
 * few frames (skinned, deforming, breaking).  Triangles are put in Morton order (21 bits per axis of the box centroid in the root
 * box), neighbouring clusters within 16 places that are each other's cheapest union merge until one remains, and subtrees of at most
 * 4 triangles whose SAH leaf cost (c_int) is not above their interior cost (c_trav) become one leaf.  DESIGN.md §4.8 states every
 * rule; the tree is the same alone or in any batch (not promised for vertices with a NaN coordinate).  The nodes are numbered as BVH::ConvertFrom( BVH_Verbose ) numbers them (DFS
 * preorder, node 1 unused) and every box is the one BVH::Refit computes, so the handle is what tbvh_upload_bvh of the same arrays
 * leaves, plus refittable, kept indices and build_ms; idx_count = prim_count.  Its SAHCost is close to, but not, that of
 * BVH::Build's tree.  Refusals, limits and failures are those of TBVH_BUILD_REFERENCE.  Device scratch: about 330 bytes per
 * triangle during the build. */
#define TBVH_BUILD_PLOC 3        /* parallel locally-ordered clustering */
int tbvh_build_flavour( tbvh_bvh bvh, const void* verts, uint32_t stride, uint32_t prim_count, int space, float c_trav, float c_int, int flavour );

/* Indexed geometry: BVH::Build / BuildAVX / BuildHQ( const bvhvec4* vertices, const uint32_t* indices, primCount ) and their
 * bvhvec4slice forms (tiny_bvh.h:889-900; PrepareBuild reads verts[vertIdx[3 i + k]], :2290-2297).  verts: vert_count
 * vertices `stride` bytes apart; indices: 3 * prim_count entries.  primIdx numbers triangles exactly as the reference does
 * (triangle i = indices[3 i .. 3 i + 2]); an index >= vert_count is TBVH_E_ARG (the reference reads out of bounds).
 * tbvh_build, tbvh_build_flavour and tbvh_build_indexed are one-mesh calls of tbvh_build_batch / tbvh_build_batch_hq below, with their
 * refusals, codes and limits.  Every refusal comes before the handle is touched, so a refused build leaves the handle and a TLAS over
 * it as they were: TBVH_E_ARG for a NULL handle or verts, an unknown flavour or space, prim_count 0, a bad stride, NULL indices,
 * vert_count 0, or an index >= vert_count (host indices are checked on the CPU before anything is read on the device); TBVH_E_LIMIT
 * for more than TBVH_BATCH_MAX_PRIMS triangles, before any vertex is read.  The new vertices are staged before the old arrays are
 * released, so a rebuild of a handle briefly holds both (48 bytes per triangle on top of the old tree).  A failure after the device
 * work started leaves the handle empty. */
int tbvh_build_indexed( tbvh_bvh bvh, const void* verts, uint32_t stride, uint32_t vert_count, const uint32_t* indices, uint32_t prim_count, int space,
	float c_trav, float c_int, int flavour );

/* Many meshes in one call: a binned-SAH tree per mesh, as the reference's scene code builds one BLAS per mesh (tiny_scene.h,
 * tmpl8/game.cpp).  bvhs[i] receives the tree of meshes[i] and ends up exactly as tbvh_build_flavour (or, with indices,
 * tbvh_build_indexed) of that mesh alone would leave it: nodes, primIdx and leaf triangles byte for byte, the same info (build_ms is
 * the device time of the whole batch), layout TBVH_LAYOUT_BVH, refittable, and a TLAS built over its old arrays is stale.  The
 * trees are built together by the same kernels, so the fixed cost of a build (allocations, launches, host round trips) is paid once
 * per batch instead of once per mesh; the order of `meshes` changes no tree.  All meshes are in one `space`; device-space inputs
 * follow the rule above.
 *  flavour: TBVH_BUILD_REFERENCE, TBVH_BUILD_AVX or TBVH_BUILD_PLOC; TBVH_BUILD_HQ is TBVH_E_UNSUPPORTED (SBVH batches: tbvh_build_batch_hq below).
 *  Refusals come before any handle is touched, so every handle keeps its previous tree: TBVH_E_ARG for count 0, a NULL or repeated
 *  handle, handles of different contexts, prim_count 0, a bad stride, or any index >= vert_count; TBVH_E_LIMIT when the meshes
 *  hold more than TBVH_BATCH_MAX_PRIMS triangles together (positions of one shared index space must fit the builder's 32-bit
 *  encodings).  A failure after the device work started leaves every handle of the batch empty, as a failed build does. */
typedef struct tbvh_mesh
{
	const void* verts;          /* as for tbvh_build (flat: 3 * prim_count vertices) or tbvh_build_indexed (vert_count vertices) */
	uint32_t stride;            /* bytes between vertices, a multiple of 4, at least 12 */
	uint32_t vert_count;        /* used with indices only */
	const uint32_t* indices;    /* NULL: flat triangle soup; else 3 * prim_count vertex indices, in the same space as verts */
	uint32_t prim_count;
} tbvh_mesh;
#define TBVH_BATCH_MAX_PRIMS (1u << 30)
int tbvh_build_batch( tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, float c_trav, float c_int, int flavour );

/* Many meshes in one SBVH build: BVH::BuildHQ (tiny_bvh.h:2623) per mesh, as a static scene builds its BLASes for the best traversal
 * quality.  bvhs[i] ends up exactly as tbvh_build_flavour( .., TBVH_BUILD_HQ ) (or, with indices, tbvh_build_indexed) of meshes[i]
 * alone would leave it: nodes, the whole primIdx (idx_count = prim_count + prim_count / 2, zeros past the leaf entries) and leaf
 * triangles byte for byte, the same info (build_ms is the device time of the whole batch), layout TBVH_LAYOUT_BVH, not refittable,
 * and a TLAS built over its old arrays is stale.  The order of `meshes` and their neighbours change no tree.  Launches and host
 * synchronisations grow with the deepest tree's level count, not with count.
 *  Refusals are those of tbvh_build_batch, with the same codes, and come before any handle or vertex is touched; besides, TBVH_E_LIMIT
 *  when the batch's temporary node space, 3 * (total prim_count) + 2 nodes, exceeds TBVH_BATCH_HQ_MAX_NODES (node and position
 *  numbers of the shared spaces are 32-bit).  A failure after the device work started leaves every handle of the batch empty. */
#define TBVH_BATCH_HQ_MAX_NODES 0xffffffffu
int tbvh_build_batch_hq( tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, float c_trav, float c_int );

/* TLAS: BVH::Build( BLASInstance* instances, instCount, BVHBase** blasses, blasCount ) tiny_bvh.h:2221, traversed by
 * BVH::IntersectTLAS (:3306) / IsOccludedTLAS (:3455) whenever tbvh_intersect / tbvh_occluded (or the _device forms) are
 * called on the handle.  instances: inst_count records of the reference's 192-byte BLASInstance (:1443), inst_stride bytes
 * apart, ALREADY Update()d (invTransform and world box filled in: the reference's own "blasses == 0" mode, :2245);
 * blasses: handles holding a BVH-layout triangle tree in the same context - they must outlive the TLAS ("both must be kept
 * alive").  INST_IDX_BITS == 32 (the library default): a hit stores the instance number in hit.inst, byte 44 of the Ray
 * record, so closest hits are always returned in place (tbvh_intersect_packed / a separate d_hits array: TBVH_E_UNSUPPORTED).
 * A host program compiled with another INST_IDX_BITS (4..31) sets tbvh_set_option( ctx, "inst_idx_bits", bits ): hits then
 * carry the instance in the top bits of hit.prim (prim = triIdx + (inst << (32 - bits)), :8527) and byte 44 is left alone.
 * The `layout` argument of the traversal calls on a TLAS names the layout the BLASses are walked in: TBVH_LAYOUT_BVH (what the
 * reference's CPU IntersectTLAS does, :3341), or TBVH_LAYOUT_CWBVH - the arrangement of the reference's GPU path (traverse_tlas.cl:13-107:
 * BVH2 TLAS, per-instance ray transform, CWBVH BLASses, a BLAS hit kept when it is closer, the instance attached), semantics of
 * BVH8_CWBVH::Intersect (:7046) per BLAS.  A BLAS may hold either layout or both (CWBVH: tbvh_convert / tbvh_upload_cwbvh BEFORE
 * tbvh_build_tlas - the TLAS records the arrays each BLAS holds at that moment); walking a layout some BLAS did not hold is
 * TBVH_E_STATE, and so is walking a TLAS after one of its BLASses was rebuilt, re-converted, re-uploaded or destroyed.
 * The two-level kernel walks a BVH-layout BLAS with a 64-entry stack: a BLAS whose BVH2 has depth 64 or more is refused
 * (TBVH_E_LIMIT) unless it also holds its CWBVH; then the TLAS is built, walks in TBVH_LAYOUT_CWBVH run, and walks in
 * TBVH_LAYOUT_BVH are refused with TBVH_E_LIMIT.
 * Refusals (TBVH_E_ARG for bad arguments, a NULL BLAS or one from another context, or an instance naming a BLAS past blas_count;
 * TBVH_E_STATE / TBVH_E_LIMIT for the BLAS states above) come before the handle is touched: a refused call leaves the handle, and
 * any TLAS it held, as they were.  Any later failure - a TLAS deeper than the 64-entry stack of IntersectTLAS (TBVH_E_LIMIT), or a
 * CUDA error - leaves the handle empty, as a failed build does. */
/* BVH::SAHCost( 0 ) tiny_bvh.h:1889-1897: the tree's SAH cost, host recursion over the (downloaded) 32-byte node array in the
 * reference's own order and rounding - the number the speedtest prints after every build.  _nodes works on a host array. */
int tbvh_sah_cost( tbvh_bvh bvh, float c_trav, float c_int, float* out );
int tbvh_sah_cost_nodes( const void* nodes32, uint32_t used_nodes, float c_trav, float c_int, float* out );

/* Lower the SAH cost of a resident tree on the device: rounds of parallel subtree reinsertion (Meister & Bittner 2018).  The
 * reference's optimiser, BVH::Optimize tiny_bvh.h:3043 over BVH_Verbose::Optimize :4338, reinserts one subtree at a time; this is
 * a different algorithm and its tree is NOT the reference's.  Each round every node searches the round's tree for its cheapest
 * place, the non-conflicting moves are applied together and interior boxes refolded; the round is kept when SAHCost( c_trav,
 * c_int ) falls strictly and the depth stays <= max( max_depth, 63 ), else it is retried with the better half of its moves, down
 * to one; the call ends after max_rounds kept rounds or at the first round nothing is kept.  Rules: DESIGN.md §4.7.
 *  Input: any handle holding a BVH-layout tree: builds of every flavour, indexed or flat, batch builds, and tbvh_upload_bvh trees
 *  whose node slots but node 1 all belong to the tree (as every builder leaves them).  A tbvh_upload_bvh_gpu upload holds no
 *  BVH-layout tree (tbvh_sah_cost and tbvh_refit refuse it too).  Leaves keep firstTri, triCount and their box bits; primIdx,
 *  idx_count and prim_count stay as they are; only the interior structure moves.
 *  Output: the handle ends up as tbvh_upload_bvh( .., TBVH_DEVICE ) of the new nodes would leave it (traversal arrays, root,
 *  max_depth, stack choice, aabb_min / aabb_max), keeping its primIdx, vertices, kept indices and refittability.  The nodes are
 *  numbered as BVH::ConvertFrom( BVH_Verbose ) numbers a tree: DFS preorder, the k-th interior node's children at 2 + 2k and
 *  3 + 2k, interior boxes the fold of their children; used_nodes = 2 + 2 x interior nodes.  BVH_GPU and CWBVH are dropped (as
 *  tbvh_refit drops them), the generation is renewed (a TLAS over the handle is stale), device views end; info.build_ms is the
 *  device time of the call.  When no round is kept (always for a tree of one or two leaves) the handle is left exactly as it was.
 *  *rounds: rounds kept (<= max_rounds); *sah: the final SAHCost, bit for bit tbvh_sah_cost of the result; either may be NULL.
 *  Refusals come before anything is touched: TBVH_E_ARG for a NULL handle, max_rounds 0, or c_trav / c_int not finite and > 0;
 *  TBVH_E_STATE for a TLAS, a handle without a BVH-layout tree (an empty handle, a tbvh_upload_bvh_gpu or CWBVH-only upload), or a
 *  tbvh_upload_bvh tree with slots outside it (a slot other than node 1 unreached, or node 1, a slot past used_nodes or one slot
 *  twice reached from the root); TBVH_E_LIMIT for a tree deeper than 255 (the search's stack).
 *  A failure after the device work began leaves the handle empty, as a failed build does. */
int tbvh_optimize( tbvh_bvh bvh, uint32_t max_rounds, float c_trav, float c_int, uint32_t* rounds, float* sah );

/* BLASInstance::Update( BVHBase* blas ) tiny_bvh.h:8386 on one 192-byte record: invTransform = inverse of transform
 * (InvertTransform :8402), aabbMin / aabbMax = box of the eight transformed corners of the BLAS's root box.  Host arithmetic in
 * the reference build's own operation order: the record comes out bit-identical to the reference's.  _box takes the root box
 * directly (no device needed). */
int tbvh_instance_update( void* instance, tbvh_bvh blas );
int tbvh_instance_update_box( void* instance, const float* blas_aabb_min, const float* blas_aabb_max );
int tbvh_build_tlas( tbvh_bvh tlas, const void* instances, uint32_t inst_stride, uint32_t inst_count, const tbvh_bvh* blasses, uint32_t blas_count,
	float c_trav, float c_int );

/* BVH::Build( BLASInstance*, instCount, BVHBase**, blasCount ) tiny_bvh.h:2221 with blasses != 0, the call an animated scene makes every
 * frame after it refitted its BLASes and wrote the new transforms (tiny_bvh_anim.cpp, tmpl8/game.cpp): every instance is Update()d
 * (:2245-2250, :8386) and the TLAS is built over the new boxes.  Update runs on the device, one kernel for the whole list, and that
 * kernel also fills the tables the two-level walk and the builder read: no host loop touches the records.
 *  instances: inst_count records of the 192-byte BLASInstance, inst_stride bytes apart, in `space`.  Read: transform (byte 0), blasIdx
 *  (140), mask (156).  Written back in place as Update does: invTransform (64), aabbMin (128), aabbMax (144); no other byte changes.
 *  TBVH_DEVICE: the pointer and the stride are multiples of 16 and the records follow the rule for device-space inputs above.
 *  TBVH_HOST: the stride is a multiple of 4 and at least 160; the records go through the device in one strided copy each way.
 *  The root box of instance i is that of blasses[blasIdx] as tbvh_bvh_info reports it - what tbvh_instance_update uses, and what
 *  tbvh_refit_batch has just brought up to date.
 * The result is exactly what tbvh_instance_update on every record followed by tbvh_build_tlas leaves: the same record bytes, TLAS
 * nodes, primIdx and info (build_ms includes the update kernel), the same rules for the layouts of the BLASses, the same staleness.
 * (Where the arithmetic itself generates a NaN - a determinant that overflows - both give a NaN; its sign and payload are the processor's.)
 * Refusals: those of tbvh_build_tlas with the same codes, TBVH_E_STATE for a BLAS without a BVH-layout tree (its root box is not
 * known: tbvh_instance_update's refusal), TBVH_E_ARG for an unknown space, a bad stride or a misaligned device pointer.  Whatever host
 * state decides - handles, counts, stride, the state and limits of the BLASses, and for host records blasIdx < blas_count - is checked
 * before the handle is touched: a refused call leaves a walkable TLAS walkable and the records as they were.  In device records
 * blasIdx is checked by the kernel, which never dereferences an index past the list: TBVH_E_ARG, the handle left empty as after a
 * failed build, the records unspecified.  Every other failure leaves the handle empty too, as for tbvh_build_tlas.
 * A handle that already is a TLAS over the same inst_count and blas_count keeps its instance boxes, instance and BLAS tables and the
 * staging of host records; what a frame still allocates is the builder's own (the node and primIdx arrays and its scratch). */
int tbvh_build_tlas_update( tbvh_bvh tlas, void* instances, uint32_t inst_stride, uint32_t inst_count, int space, const tbvh_bvh* blasses,
	uint32_t blas_count, float c_trav, float c_int );

/* BVH::Refit (tiny_bvh.h:3055-3093): the triangles moved, the topology stays - leaf boxes from the new vertices, interior
 * boxes bottom-up.  verts as for tbvh_build, same prim_count.  Derived layouts on the handle are dropped; tbvh_convert again.
 * tbvh_refit and tbvh_refit_layouts are one-mesh calls of tbvh_refit_batch below (keep_layouts 0 and 1), with its refusals, codes and
 * limit, all before the handle is touched: TBVH_E_ARG for a NULL handle or verts, an unknown space, another prim_count or a bad
 * stride; TBVH_E_STATE for an SBVH (the reference's fatal "refitting an SBVH"), a TLAS, or when no BVH-layout tree is resident;
 * TBVH_E_LIMIT past TBVH_REFIT_BATCH_MAX_NODES. */
int tbvh_refit( tbvh_bvh bvh, const void* verts, uint32_t stride, uint32_t prim_count, int space );

/* Refit that keeps the derived layouts: tbvh_refit's BVH::Refit, then every layout the handle holds brought up to date in place
 * instead of dropped, with the same arguments.
 *  - BVH_GPU: BVH_GPU::ConvertFrom (tiny_bvh.h:4612) of the refitted tree, byte for byte (the conversion is a pure relayout).
 *  - CWBVH: the 8-wide collapse of the last tbvh_convert is kept - which BVH2 nodes are the children of each wide node, in
 *    adoption order.  The boxes come from the refitted BVH2 after SplitLeafs(3) (chain leaves keep their refitted parent leaf's
 *    box); BVH8_CWBVH::ConvertFrom's greedy slot assignment, stack-order addresses and quantised encode (:5884) run on that, and
 *    bvh8Tris is taken from the new vertices.  The wide-node count and depth stay; slot assignment and node addresses may change.
 *    Every frame uses the collapse of the conversion, not that of the previous frame, so a long animation keeps the tree quality
 *    of its first frame: call tbvh_convert again to collapse anew.
 *  - info.build_ms is the device time of the call, aabb_min / aabb_max the new root box.
 * Refusals leave the handle unmodified: TBVH_E_STATE for an SBVH, a TLAS, no BVH-layout tree, or a CWBVH that tbvh_convert did not
 * produce from the resident tree (tbvh_upload_cwbvh, a group replica); TBVH_E_ARG for another prim_count, a bad stride or an
 * unknown space; TBVH_E_LIMIT as for tbvh_refit.
 * As after every refit, a TLAS over this BLAS is stale (its instance boxes are) until tbvh_build_tlas runs again, and group
 * replicas keep the old boxes until tbvh_group_replicate runs again. */
int tbvh_refit_layouts( tbvh_bvh bvh, const void* verts, uint32_t stride, uint32_t prim_count, int space );

/* Many trees refitted in one call, as an animated scene refits its BLASes every frame (tiny_bvh_anim.cpp, tmpl8/game.cpp).
 * meshes[i] holds the new vertices of bvhs[i] as for tbvh_refit: verts, stride, prim_count; indices must be NULL and vert_count 0
 * (a refit takes the flat slice).  All meshes are in one `space`; device-space inputs follow the rule above.
 *  keep_layouts = 0: each bvhs[i] ends up exactly as tbvh_refit of it alone leaves it (BVH_GPU and CWBVH dropped; its generation
 *  renewed, so a TLAS over it is stale, only where a CWBVH was dropped).
 *  keep_layouts = 1: each ends up exactly as tbvh_refit_layouts of it alone leaves it: every BVH_GPU and kept CWBVH brought up to
 *  date in place, the rD limit of each CWBVH recomputed for its own tree, the new root box in its info, and a TLAS over any of them
 *  stale.  The handles of one batch may hold different subsets of BVH_GPU and CWBVH.
 * The trees are refitted together by the same kernels, so the fixed cost of a refit (launches, allocations, host round trips) is paid
 * once per batch instead of once per tree: launches grow with the deepest kept wide tree's level count, not with `count`, and a call
 * synchronises the host once.  info.build_ms is the device time of the whole batch; the order of `bvhs` and the other trees of the
 * batch change no tree.
 *  Refusals come before any handle or vertex array is touched, so every handle keeps its trees and its generation: TBVH_E_ARG for count
 *  0, a NULL or repeated handle, handles of different contexts, non-NULL indices or a vert_count, an unknown space, or a keep_layouts
 *  other than 0 or 1; then per handle, in order, tbvh_refit's / tbvh_refit_layouts' own refusals (TBVH_E_STATE for no BVH-layout
 *  tree, an SBVH, a TLAS, or with keep_layouts a CWBVH that tbvh_convert did not produce; TBVH_E_ARG for another prim_count or a bad
 *  stride); TBVH_E_LIMIT when the BVH2 nodes, primitive references, or (with keep_layouts) kept split-tree or wide nodes of the batch
 *  add up to more than TBVH_REFIT_BATCH_MAX_NODES (node indices of the shared index spaces are 32-bit).  A failure after the device
 *  work started leaves every handle of the batch with its BVH-layout tree, whose boxes are unspecified, and without BVH_GPU or CWBVH. */
#define TBVH_REFIT_BATCH_MAX_NODES (1u << 31)
int tbvh_refit_batch( tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, int keep_layouts );

/* Refit of indexed meshes: BVH::Refit (tiny_bvh.h:3055-3093) of a tree built with vertIdx set reads the moved vertices through the
 * indices (BVHBase::vertIdx, :806-807), so the caller moves vert_count vertices, not 3 * prim_count.  A refittable indexed build -
 * tbvh_build_indexed with TBVH_BUILD_REFERENCE or TBVH_BUILD_AVX, or a mesh with indices of tbvh_build_batch - keeps a device copy of
 * its indices and its vert_count on the handle for this call: 12 bytes of device memory per triangle.  SBVH builds and flat builds keep
 * none.  Every build, tbvh_upload_bvh / tbvh_upload_bvh_gpu and TLAS build on the handle, and a failed batch build, drop them; refits
 * and conversions leave them.  Group replicas do not carry them.
 *  meshes[i].vert_count > 0: verts holds the new positions of the vert_count vertices bvhs[i] was built from (the build's vert_count),
 *  `stride` bytes apart; indices must be NULL (the kept ones are used); prim_count and stride as for tbvh_refit.
 *  meshes[i].vert_count == 0: a flat slice, as for tbvh_refit_batch; the flat and indexed meshes of a scene refit in one call.
 * Each handle ends up exactly as tbvh_refit (keep_layouts = 0) or tbvh_refit_layouts (keep_layouts = 1) of the flat slice
 * verts[indices[j]], j < 3 * prim_count, at the same stride leaves it: BVH2 nodes, primIdx, BVH_GPU, bvh8Data / bvh8Tris, leaf
 * triangles, info, traversal limits, generation and the staleness of a TLAS over it.  As in tbvh_refit, below stride 16 the w lanes are
 * not replaced.  The vertex rows of the indexed meshes are staged at a 16-byte pitch on the device (host and device space alike) and
 * one kernel writes every indexed handle's vertices through its indices; then the refit runs as in tbvh_refit_batch, with one host
 * synchronisation.  count = 1 refits a single handle.
 *  Refusals come before any handle or vertex array is touched: those of tbvh_refit_batch with the same codes, except that a mesh may
 *  carry a vert_count; besides, TBVH_E_ARG for non-NULL indices or a vert_count other than the build's, TBVH_E_STATE for a vert_count on
 *  a handle that keeps no indices, and TBVH_E_LIMIT also when the indexed meshes hold more than TBVH_REFIT_BATCH_MAX_NODES indices. */
int tbvh_refit_batch_indexed( tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, int keep_layouts );

/* consume a tree built elsewhere, in the reference's own layouts (the public members bvhNode / primIdx /
 * verts of tiny_bvh.h:952-964, BVH_GPU::bvhNode :1124, BVH8_CWBVH::bvh8Data / bvh8Tris :1356-1357) */
int tbvh_upload_bvh( tbvh_bvh bvh, const void* nodes32, uint32_t used_nodes, const uint32_t* prim_idx, uint32_t idx_count,
	const void* verts, uint32_t stride, uint32_t prim_count, int space );
int tbvh_upload_bvh_gpu( tbvh_bvh bvh, const void* nodes64, uint32_t used_nodes, const uint32_t* prim_idx, uint32_t idx_count,
	const void* verts, uint32_t stride, uint32_t prim_count, int space );
int tbvh_upload_cwbvh( tbvh_bvh bvh, const void* bvh8_data, uint32_t used_blocks, const void* bvh8_tris, uint32_t tri_count, int space );

/* layout conversion on the device: BVH_GPU::ConvertFrom tiny_bvh.h:4612; BVH8_CWBVH::Build's chain
 * Compact :3733 + SplitLeafs(3) :1988 + MBVH<8>::ConvertFrom :4975 + BVH8_CWBVH::ConvertFrom :5884.  A handle without a
 * BVH-layout tree is TBVH_E_STATE whatever the target; another target than the two is TBVH_E_UNSUPPORTED.  To CWBVH the call is a
 * one-handle tbvh_convert_batch below, with its refusals, codes and limit, all before the handle is touched: TBVH_E_STATE for a TLAS
 * (its leaves are instances, not triangles); TBVH_E_LIMIT when the split tree could hold more than TBVH_CONVERT_BATCH_MAX_NODES
 * nodes.  A conversion to CWBVH that fails on the device leaves the handle without a CWBVH. */
int tbvh_convert( tbvh_bvh bvh, int to_layout );

/* Many trees converted to CWBVH in one call, as a scene converts every BLAS before a TLAS walks them in TBVH_LAYOUT_CWBVH.
 * Afterwards each bvhs[i] holds exactly what tbvh_convert( bvhs[i], TBVH_LAYOUT_CWBVH ) would leave: bvh8Data and bvh8Tris byte
 * for byte, the same info (build_ms untouched), layout bits and traversal limits, a renewed generation where it held a CWBVH before
 * (a TLAS over the old arrays is stale), and on a refittable tree the collapse tbvh_refit_layouts reuses.  The trees are converted
 * together by the same kernels, so the fixed cost of a conversion (allocations, launches, host round trips) is paid once per batch
 * instead of once per tree; the order of `bvhs` and the other trees of the batch change no tree.  Any BVH_GPU layout stays.
 *  to_layout: TBVH_LAYOUT_CWBVH; any other is TBVH_E_UNSUPPORTED (BVH_GPU::ConvertFrom is a relayout without a fixed cost worth
 *  batching: tbvh_convert per handle).
 *  Refusals come before any handle is touched, so every handle keeps its arrays and its generation: TBVH_E_ARG for count 0, a NULL
 *  or repeated handle, or handles of different contexts; TBVH_E_STATE for a handle without a BVH-layout tree, or a TLAS (its leaves
 *  are instances, not triangles); TBVH_E_LIMIT when the split trees together could hold more than TBVH_CONVERT_BATCH_MAX_NODES
 *  nodes, counted as the sum of max( used_nodes, 2 ) + 2 * ceil( idx_count / 3 ) (node indices of the shared index space are 32-bit).  A
 *  failure after the device work started leaves every handle of the batch with its BVH-layout tree and any other layout it had,
 *  and without a CWBVH. */
#define TBVH_CONVERT_BATCH_MAX_NODES (1u << 31)
int tbvh_convert_batch( tbvh_bvh* bvhs, uint32_t count, int to_layout );

/* read a layout back in the reference's format so SAHCost / Save / ConvertFrom / the CPU traversals can use a
 * GPU-built tree.  Buffers are sized from tbvh_bvh_info. */
int tbvh_download_bvh( tbvh_bvh bvh, void* nodes32, uint32_t* prim_idx, int space );
int tbvh_download_bvh_gpu( tbvh_bvh bvh, void* nodes64, int space );
int tbvh_download_cwbvh( tbvh_bvh bvh, void* bvh8_data, void* bvh8_tris, int space );

/* ---- traversal ------------------------------------------------------------------------------------------ */
/* BVH::Intersect( Ray& ) tiny_bvh.h:3222 / BVH_GPU::Intersect :4657 / BVH8_CWBVH::Intersect :7046 and the OpenCL
 * batch kernels batch_ailalaine (traverse_bvh2.cl:209) / batch_cwbvh (traverse_cwbvh.cl:554) for a whole batch:
 * host records, in place - copies bytes 0..63 in, writes t,u,v,prim back to bytes 48..63 of every record. */
int tbvh_intersect( tbvh_bvh bvh, int layout, void* rays, uint32_t stride, uint64_t n );
/* same traversal, hits delivered as a packed array of 16-byte (t,u,v,prim) records instead of being scattered into the
 * 128-byte ray records: the return trip becomes one contiguous copy per chunk (the in-place form pays a strided
 * 16-byte-row copy; see DESIGN.md 4.5).  `rays` is not modified. */
int tbvh_intersect_packed( tbvh_bvh bvh, int layout, const void* rays, uint32_t stride, uint64_t n, void* hits );
/* BVH::IsOccluded( const Ray& ) tiny_bvh.h:3382 / isoccluded_cwbvh (traverse_cwbvh.cl:343) for a batch:
 * bits[i>>5] bit (i&31) = occluded; (n+31)/32 words are written. */
int tbvh_occluded( tbvh_bvh bvh, int layout, const void* rays, uint32_t stride, uint64_t n, uint32_t* bits );

/* the same with everything already resident in HBM, asynchronous on `stream` (a cudaStream_t, 0 = default).
 * hits == NULL writes t,u,v,prim into bytes 48..63 of each record; otherwise 16-byte records to hits[]. */
int tbvh_intersect_device( tbvh_bvh bvh, int layout, void* d_rays, uint32_t stride, void* d_hits, uint64_t n, void* stream );
int tbvh_occluded_device( tbvh_bvh bvh, int layout, const void* d_rays, uint32_t stride, uint32_t* d_bits, uint64_t n, void* stream );

/* ---- proximity queries ---------------------------------------------------------------------------------- */
/* Nearest surface point and sphere overlap of query points over the BVH-layout tree of `bvh` (the arrays the BVH2 walk reads): builds of
 * every flavour, flat, indexed and batched; BVH_GPU and CWBVH objects built or converted by the library; tbvh_upload_bvh /
 * tbvh_upload_bvh_gpu trees; refitted and optimised trees; group replicas.  The engine's own definition (DESIGN.md 4.9), not bit for
 * bit the reference's BVH::IntersectSphere (tiny_bvh.h:3140-3200), whose separating-axis test may decide otherwise where a sphere only
 * touches a triangle: a reference (leaf, triangle) is worth d2 = max( |p - closest point|^2, P ), P the squared distance bound of the
 * boxes on its leaf's path, and results are the smallest ( d2, prim ), whatever the tree's visiting order.
 *  tbvh_closest_point  queries: n float4 { x, y, z, r_max } (r_max = INFINITY: unbounded); results: n 16-byte records { d, u, v, prim }:
 *                      d = the distance to the nearest triangle within r_max, its closest point v0 + u (v1 - v0) + v (v2 - v0) (the
 *                      u, v of a Moeller-Trumbore hit; u, v >= 0, u + v <= 1); nothing within r_max, a NaN coordinate or an r_max
 *                      not >= 0: { r_max, 0, 0, 0xffffffff }.
 *  tbvh_sphere_overlap queries: n float4 { x, y, z, r }; bits[i>>5] bit (i&31) = some triangle lies within r of the centre, exactly
 *                      when tbvh_closest_point with r_max = r finds one; (n+31)/32 words are written, bits past n are 0.
 * TBVH_DEVICE: asynchronous on `stream` (a cudaStream_t, 0 = default), pointers 16-byte aligned.  TBVH_HOST: staged through the
 * device and complete on return (`stream` unused).  n = 0 does nothing.  Refusals, before any launch: TBVH_E_ARG for NULL arguments,
 * an unknown space, a misaligned device pointer or a batch too large for one launch; TBVH_E_STATE for a handle without a BVH-layout
 * tree (empty, or a CWBVH-only upload); TBVH_E_UNSUPPORTED for a TLAS; TBVH_E_LIMIT for a tree deeper than 255. */
int tbvh_closest_point( tbvh_bvh bvh, const void* queries, void* results, uint64_t n, int space, void* stream );
int tbvh_sphere_overlap( tbvh_bvh bvh, const void* queries, uint32_t* bits, uint64_t n, int space, void* stream );

/* ---- signed distances ----------------------------------------------------------------------------------- */
/* Signed distance of query points to the triangles of `bvh` (DESIGN.md 4.10): the closest-point query above, signed by the angle-weighted
 * pseudonormal (Baerentzen & Aanaes 2005) of the feature - face, edge or vertex - the closest point lies on.  Topology comes from
 * positions, not indices: corners whose x, y and z are equal as values (-0 equals +0) are one vertex, a corner with a NaN coordinate welds
 * to nothing, so a flat soup, an indexed build and its V[I] soup get the same pseudonormals.
 * The sign is meaningful only on closed, consistently oriented, manifold surfaces whose normals by the right-hand rule on (v0, v1, v2)
 * point outward: then sd < 0 exactly inside.  Boundary and non-manifold edges get the same sums, and no claim is made about the sign there.
 *  tbvh_signed_distance_prepare  builds the handle's pseudonormal table on the engine stream (7 x 16 bytes per triangle) and returns when
 *                      it is complete.  The table is tied to the tree and vertices it was made from: any later build, upload of a
 *                      BVH or BVH_GPU, tbvh_optimize that changes the tree, or refit makes it stale, and it must be prepared again.
 *                      A conversion (tbvh_convert, tbvh_convert_batch) or a CWBVH upload changes neither and keeps it.  Refusals:
 *                      TBVH_E_ARG for NULL; TBVH_E_UNSUPPORTED for a TLAS; TBVH_E_STATE without a BVH-layout tree; TBVH_E_LIMIT above
 *                      2^30 triangles.  A failure after the device work began leaves the tree untouched and no table.
 *  tbvh_signed_distance  queries: n float4 { x, y, z, r_max } as tbvh_closest_point; results: n 16-byte records { sd, u, v, prim }:
 *                      u, v and prim are tbvh_closest_point's, |sd| is its d, and sd < 0 exactly when ( p - c ) . N < 0, c the
 *                      closest point and N the feature's pseudonormal (a point on the surface gives +0).  A miss, a NaN coordinate
 *                      or an r_max not >= 0 gives the closest-point miss record { r_max, 0, 0, 0xffffffff }: there the sign is unknown.
 *                      Space, stream and refusals as tbvh_closest_point, in the same order; after them TBVH_E_STATE when no table was
 *                      prepared or the table is stale.  Every refusal comes before any launch. */
int tbvh_signed_distance_prepare( tbvh_bvh bvh );
int tbvh_signed_distance( tbvh_bvh bvh, const void* queries, void* results, uint64_t n, int space, void* stream );

/* ---- generalized winding numbers ------------------------------------------------------------------------ */
/* The generalized winding number w(q) of the triangles `bvh` references (DESIGN.md 4.11; Jacobson et al. 2013, Barill et al. 2018): 1
 * inside and 0 outside a closed mesh whose normals by the right-hand rule on (v0, v1, v2) point outward, 2 where two such solids overlap,
 * and a smooth value across holes, so "w > 0.5" is an inside test for open, self-intersecting and non-manifold meshes too.  No topology
 * is needed.  Each triangle counts once: a triangle an SBVH references from several leaves belongs to its first reached reference.
 * Subtrees far from the query (|p - q| > beta r, p and r the centre and half diagonal of the box of their triangles) contribute a
 * second-order expansion; the others are summed exactly.  beta = +inf gives the exact sum.
 * For an inside/outside sign on an open mesh: |d| from tbvh_closest_point, negative where the winding number is > 0.5.
 *  tbvh_winding_number_prepare  builds the handle's table on the engine stream (64 bytes per node slot plus 4 bytes per primitive
 *                      reference) and returns when it is complete.  Stale after the same calls as the signed-distance table.
 *                      Refusals: TBVH_E_ARG for NULL; TBVH_E_UNSUPPORTED for a TLAS; TBVH_E_STATE without a BVH-layout tree, or for a
 *                      tree that reaches a node on two paths (a DAG); TBVH_E_LIMIT for a tree deeper than 255.  A refused prepare
 *                      leaves the tree untouched and no table.
 *  tbvh_winding_number  queries: n float4 { x, y, z, ignored } (16-byte aligned); results: n floats (4-byte aligned).  A NaN coordinate
 *                      gives NaN.  beta must be > 1 (+inf allowed).  Space and stream as tbvh_closest_point.  Refusals, before any
 *                      launch, in this order: TBVH_E_ARG (NULL, space, alignment, beta not > 1, NaN included), TBVH_E_UNSUPPORTED for a
 *                      TLAS, TBVH_E_STATE / TBVH_E_LIMIT as tbvh_closest_point, then TBVH_E_STATE when no table was prepared or it is
 *                      stale. */
int tbvh_winding_number_prepare( tbvh_bvh bvh );
int tbvh_winding_number( tbvh_bvh bvh, const void* queries, float* results, uint64_t n, float beta, int space, void* stream );

/* ---- intersecting triangle pairs ------------------------------------------------------------------------ */
/* Which triangles of mesh a cross which triangles of mesh b, and (b == a) which triangles of one mesh cross each other (DESIGN.md 4.12).
 * Both handles hold a BVH-layout tree as for tbvh_closest_point; their vertices are taken as they are, in one space (no transforms).
 * The pair test tt_overlap( T, U ) is on closed triangles, so touching counts, and uses orientation predicates only (after Guigue &
 * Devillers 2003), in fp32 in a fixed order: the triangle whose nine coordinates are lexicographically smaller as ordered keys is T,
 * T's v0 is subtracted from all six corners and the differences are scaled by the power of two of their largest magnitude.  So the test
 * is symmetric bit for bit, scaling both meshes by 2^k (k in [-40, 40]) gives the same pairs, and on integer coordinates in [-16, 16]
 * every predicate is exact.  A triangle of zero scaled normal (zero area) or with a NaN or infinite coordinate is never reported.
 * Triangles are the input corners of each handle (the vertices it was built, uploaded or refitted with).
 *  two meshes: the pairs (i, j), i a triangle of a and j of b, such that some reference of j in b's tree is reached (every box on its
 *              path but the root's overlaps the box of triangle i: closed boxes compared in fp32) and tt_overlap holds.  With boxes that
 *              hold their triangles, as every builder's, that is every intersecting pair.
 *  b == a:     the pairs i < j of one mesh.  Corners at equal positions (as values: -0 equals +0, NaN equals nothing) are shared, and a
 *              pair sharing none is reported by tt_overlap; sharing one, when the edge opposite the shared corner in either triangle
 *              meets the other triangle; sharing two (an edge), only when both lie in one plane with their third corners on the same side
 *              of the shared edge (a face folded onto its neighbour); sharing three (a duplicate face), always.
 *  tbvh_mesh_overlap_pairs  pairs: capacity pairs of two uint32 { i, j } (8-byte aligned in device space; NULL allowed when capacity
 *              is 0), sorted by (i, j) without repeats (a triangle an SBVH references from several leaves, or a leaf a DAG reaches twice,
 *              still gives one pair).  *count (a host word) = the number of pairs, even when it exceeds capacity: the first
 *              min( count, capacity ) are written and a caller can call again with a larger buffer.  Synchronous: its scratch is sized
 *              from a counting pass; in TBVH_DEVICE its device work is ordered after `stream`'s work so far, in TBVH_HOST `stream` is
 *              unused.  After the counting pass, TBVH_E_LIMIT when the raw pairs (repeats included) exceed 2^31: *count is then that
 *              raw total, and no pair is written.
 *  tbvh_mesh_overlap_bits   bits: (n + 31) / 32 words (4-byte aligned in device space), n the triangles of a; bit (i & 31) of word
 *              i >> 5 = triangle i of a is a member of some pair (b == a: either member, so every j != i is tested); bits past n are 0.
 *              TBVH_DEVICE: one launch, asynchronous on `stream`.  TBVH_HOST: complete on return (`stream` unused).
 * Refusals, before any launch, leaving the outputs untouched, in this order: TBVH_E_ARG for NULL arguments, an unknown space, a
 * misaligned device output or handles of different contexts; TBVH_E_UNSUPPORTED for a TLAS on either side; TBVH_E_STATE when either
 * handle holds no BVH-layout tree (empty, or a CWBVH-only upload); TBVH_E_LIMIT when b's tree is deeper than 255. */
int tbvh_mesh_overlap_pairs( tbvh_bvh a, tbvh_bvh b, uint32_t* pairs, uint64_t capacity, uint64_t* count, int space, void* stream );
int tbvh_mesh_overlap_bits( tbvh_bvh a, tbvh_bvh b, uint32_t* bits, int space, void* stream );

/* ---- distances between meshes --------------------------------------------------------------------------- */
/* How far each triangle of mesh a lies from mesh b, and which pairs lie within a distance (DESIGN.md 4.13): contact candidates within a
 * margin, clearance between bodies, and (b == a) thin walls and near-touching sheets of one mesh.  Handles, trees and vertices as for
 * tbvh_mesh_overlap_pairs (a BVH-layout tree on each, vertices in one space, the input corners of each handle).
 * The pair distance tt_dist2( T, U ) is the engine's own, fp32 in a fixed order: a pair with a NaN or infinite coordinate is skipped (never
 * a candidate, not even at r = +inf); a pair that tt_overlap reports (tbvh_mesh_overlap_pairs' test) is at 0; otherwise it is the least of
 * six vertex-triangle distances (the per-triangle function of tbvh_closest_point) and the nine edge-edge distances at interior solutions,
 * on the canonical pair moved to T's v0 and scaled by a power of two.  So it is symmetric bit for bit, and scaling both meshes by 2^k
 * (k in [-40, 40]) scales every distance by exactly 2^k.  A zero-area triangle is never at 0 unless a vertex or edge candidate is.
 * The value of a reference (leaf, j) of b's tree for triangle i of a is max( tt_dist2, LBtri, P ): LBtri the squared gap of the two
 * triangles' boxes, P the largest squared gap between i's box and a box on the path to the leaf (the root's excepted; the least over
 * several paths).  Where boxes hold their triangles that is tt_dist2 up to rounding.
 *  b == a:  the self query: pairs i != j that share no corner (corners equal as values: -0 equals +0, NaN equals nothing).  Neighbours
 *           are at distance 0 by construction; a face folded onto its neighbour is tbvh_mesh_overlap_pairs' to find.
 *  tbvh_mesh_distance        results: n 8-byte records { float d, uint32 j } (8-byte aligned in device space), n the triangles of a: the
 *           smallest ( value, j ) with value <= r_max^2, d = sqrt( value ); { r_max, 0xffffffff } when nothing is found or triangle i has
 *           a non-finite coordinate.  r_max = +INFINITY: unbounded.  The separation of the meshes is the least d.  TBVH_DEVICE: one
 *           launch, asynchronous on `stream`.  TBVH_HOST: complete on return (`stream` unused).
 *  tbvh_mesh_distance_pairs  pairs: every (i, j) with some reference of j reached at value <= r^2 (r = 0: touching and crossing pairs;
 *           b == a: i < j only), as tbvh_mesh_overlap_pairs returns them: capacity pairs of two uint32, sorted without repeats, *count
 *           the exact number even above capacity, synchronous, ordered after `stream` in TBVH_DEVICE, TBVH_E_LIMIT above 2^31 raw pairs.
 * Refusals, before any launch, leaving the outputs untouched, in this order: TBVH_E_ARG for r_max / r NaN or negative, then
 * tbvh_mesh_overlap_pairs' refusals in their order (TBVH_E_ARG, TBVH_E_UNSUPPORTED, TBVH_E_STATE, TBVH_E_LIMIT). */
int tbvh_mesh_distance( tbvh_bvh a, tbvh_bvh b, float r_max, void* results, int space, void* stream );
int tbvh_mesh_distance_pairs( tbvh_bvh a, tbvh_bvh b, float r, uint32_t* pairs, uint64_t capacity, uint64_t* count, int space, void* stream );

/* Traversal from the caller's own kernels (include/tinybvh_b200_device.cuh): the traversal functions of the reference's GPU code
 * (traverse_cwbvh / isoccluded_cwbvh, traverse_ailalaine, traverse_tlas / isoccluded_tlas, SURVEY.md 2.3) as device functions over a
 * view of a resident tree.  A view holds what the matching tbvh_intersect_device / tbvh_occluded_device launch passes its kernel:
 * plain device pointers, the root, and the walk's limits.  It is passed to a kernel by value (64 bytes).
 *  tbvh_device_view  the view of `bvh` for `layout`, which means what it means in tbvh_intersect_device: TBVH_LAYOUT_BVH or
 *                    TBVH_LAYOUT_BVH_GPU -> kind TBVH_VIEW_BVH (the BVH2 walk), TBVH_LAYOUT_CWBVH -> TBVH_VIEW_CWBVH; on a TLAS the
 *                    layout its BLASses are walked in -> TBVH_VIEW_TLAS_BVH / TBVH_VIEW_TLAS_CWBVH.
 *  Refusals are exactly those of tbvh_intersect_device / tbvh_occluded_device for the same handle and layout (n > 0), with the same
 *  codes: TBVH_E_STATE when the layout is not resident or a TLAS is stale; TBVH_E_LIMIT for a BVH2 of depth 256 or more, a CWBVH
 *  that can leave more than CW_STACK node groups pending, or a TLAS walked in TBVH_LAYOUT_BVH over a BLAS too deep for it;
 *  TBVH_E_ARG for a wide tree whose links form a cycle, an unknown layout, or NULL arguments.  A refused call leaves *out of kind 0,
 *  which every device function ignores.
 *  Taking a view is host work only: no launch, no copy, no synchronisation.
 *  Lifetime: a view is valid as long as the batch call on the same handle would walk the same arrays.  A rebuild, an upload, a
 *  (re)conversion, a tbvh_refit or refit batch that drops layouts, and tbvh_bvh_destroy end it; so does, for a TLAS, anything that
 *  makes the TLAS stale (a BLAS rebuilt, re-uploaded, re-converted, refitted or destroyed), any rebuild of the TLAS itself, and
 *  tbvh_set_option( inst_idx_bits ), whose value a TLAS view holds (inst_shift) where the batch call reads it at each launch.  Take
 *  a new view per frame: a stale view is a dangling pointer, which no device function can detect. */
#define TBVH_VIEW_BVH 1          /* tbvh::intersect_bvh / isoccluded_bvh */
#define TBVH_VIEW_CWBVH 10       /* tbvh::intersect_cwbvh / isoccluded_cwbvh */
#define TBVH_VIEW_TLAS_BVH 101   /* tbvh::intersect_tlas< TBVH_LAYOUT_BVH > / isoccluded_tlas< TBVH_LAYOUT_BVH > */
#define TBVH_VIEW_TLAS_CWBVH 110 /* tbvh::intersect_tlas< TBVH_LAYOUT_CWBVH > / isoccluded_tlas< TBVH_LAYOUT_CWBVH > */
typedef struct tbvh_view
{
	int32_t kind;                  /* TBVH_VIEW_*, 0 = no tree */
	uint32_t root_ref, root_count; /* BVH2, TLAS: the root as a child record (count 0: child-pair index, else leaf range) */
	uint32_t stack;                /* BVH2: traversal stack entries, 64 for a tree of depth below 64, else 256 */
	const void* nodes;             /* BVH2: child-pair nodes; CWBVH: traversal nodes; TLAS: the TLAS's child-pair nodes */
	const void* tris;              /* BVH2: leaf-ordered triangle records; CWBVH: bvh8Tris */
	const void* prim_idx;          /* TLAS: primIdx (instance numbers) */
	const void* inst;              /* TLAS: instance table (inverse transform, BLAS number, mask) */
	const void* blas;              /* TLAS: BLAS table (each BLAS's traversal arrays) */
	float cw_rd_limit;             /* CWBVH: rays with |rD| up to this (and |O| <= 2^126) may take the integer-ordered slab test */
	uint32_t inst_shift;           /* TLAS: 32 - INST_IDX_BITS (tbvh_set_option inst_idx_bits), 0 = the instance goes to hit.inst */
} tbvh_view;
int tbvh_device_view( tbvh_bvh bvh, int layout, tbvh_view* out );

/* counters of the last device traversal on this handle when statistics are enabled (debug aid; the reference
 * returns the per-ray cost from Intersect, tiny_bvh.h:3303): steps = nodes visited, tris = triangle tests. */
int tbvh_set_stats( tbvh_bvh bvh, int enable );
int tbvh_get_stats( tbvh_bvh bvh, uint64_t* steps, uint64_t* tris );
/* the same plus the CWBVH kernels' child-pair steps: out = { node visits, triangle tests, pair steps, 0 } */
int tbvh_get_stats_ex( tbvh_bvh bvh, uint64_t out[4] );
/* rays[0..n) of a host buffer -> packed 64-byte device records (bytes 0..63 of each record; the speedtest's upload,
 * tiny_bvh_speedtest.cpp:1110-1115), asynchronous on `stream` */
int tbvh_copy_rays_to_device( const void* rays, uint32_t stride, uint64_t n, void* d_rays, void* stream );
/* device memory / synchronisation for host programs that do not link the CUDA runtime themselves (the role tinyocl::Buffer plays
 * in the reference's GPU section, tiny_bvh_speedtest.cpp:1100-1115): cudaMalloc / cudaFree / cudaDeviceSynchronize / a blocking
 * device-to-host copy on the context's device */
int tbvh_device_alloc( tbvh_ctx ctx, size_t bytes, void** out );
int tbvh_device_free( tbvh_ctx ctx, void* p );
int tbvh_device_sync( tbvh_ctx ctx );
int tbvh_copy_from_device( void* host, const void* d_src, size_t bytes );

/* ---- several GPUs in one process (SURVEY.md 8(e): rays shard by index, the BVH is replicated once, no traffic between devices
 * during traversal).  The reference has no counterpart: its GPU path drives one OpenCL device (tiny_bvh_speedtest.cpp:1092-1241).
 *  tbvh_group_create     devices[count] (NULL / 0 = all devices), one engine context each, peer access enabled where possible
 *  tbvh_group_replicate  copy the traversal arrays of a built / uploaded / converted BVH to every device of the group (peer copies
 *                        over NVLink); ms_out = device time of the copies.  Call again after the source changed.  A plain BVH's
 *                        replicas are released and made again on every call.
 *                        A TLAS (an instanced scene): every device whose context is not the source's gets one replica BLAS per
 *                        distinct BLAS handle the TLAS links to, holding only what the two-level walk reads in the layouts the
 *                        source can be walked in (the BVH2 pair array and leaf triangles, the CWBVH traversal nodes and bvh8Tris),
 *                        and one replica TLAS (nodes, primIdx, instances; its BLAS table made over the replica BLASes).  The
 *                        replica TLAS refuses exactly what the source refuses, with the same codes.  Called once per frame, after
 *                        the refits and tbvh_build_tlas_update, it refreshes in place: BLASes whose handle and generation did not
 *                        change are not copied, changed ones of unchanged sizes are copied into their arrays, unlinked ones are
 *                        released, and every byte bound for one device goes in one copy launch (one cudaMemcpyPeerAsync per array
 *                        where that device cannot read the source's).  Refused before any replica is touched: a stale source TLAS,
 *                        a TLAS whose BLASes share no walkable layout, and a group context whose inst_idx_bits differs from the
 *                        source context's (TBVH_E_STATE).  A failure after the copies began releases every replica.  A plain BVH
 *                        replicated after a TLAS releases the scene's replicas, and the other way round.
 *  tbvh_group_replica    replica i: the source itself where its context is device i's, else the group's copy (for a TLAS, the
 *                        replica TLAS).  It and tbvh_device_view of it stay valid until the next tbvh_group_replicate or
 *                        tbvh_group_destroy; a view of replica i reads device i's own arrays.
 *  tbvh_group_intersect / _occluded  tbvh_intersect / tbvh_occluded on a HOST batch, rays [first, first+count) of
 *                        tbvh_shard_range( n, g, size ) going to device g from a worker thread bound to that device's NUMA node
 *  tbvh_group_host_alloc page-locked buffer of n records whose index ranges live on the NUMA node of the device that reads them
 *  tbvh_shard_range      the partition itself: contiguous, boundaries on multiples of 32 rays (occlusion words are never shared) */
int tbvh_group_create( const int* devices, int count, tbvh_group* out );
int tbvh_group_destroy( tbvh_group group );
int tbvh_group_size( tbvh_group group );
tbvh_ctx tbvh_group_ctx( tbvh_group group, int i );
tbvh_bvh tbvh_group_replica( tbvh_group group, int i );
int tbvh_group_replicate( tbvh_group group, tbvh_bvh src, double* ms_out );
int tbvh_group_intersect( tbvh_group group, int layout, void* rays, uint32_t stride, uint64_t n );
int tbvh_group_occluded( tbvh_group group, int layout, const void* rays, uint32_t stride, uint64_t n, uint32_t* bits );
int tbvh_group_host_alloc( tbvh_group group, uint32_t stride, uint64_t n, void** out );
int tbvh_group_host_free( tbvh_group group, void* p );
void tbvh_shard_range( uint64_t n, uint32_t part, uint32_t parts, uint64_t* first, uint64_t* count );

/* number of kernels this library has launched since load (bench.py reports it as gpu_launches) */
uint64_t tbvh_launch_count( void );

#ifdef __cplusplus
}
#endif
#endif
