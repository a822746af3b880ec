// tinybvh_b200/csrc/common.cuh - shared device/host definitions of the sm_90a engine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <mutex>
#include <vector>
#include <atomic>
#include "../../include/tinybvh_b200.h"

#define BVH_FAR 1e30f
#define TBVH_STACK 64          // traversal stack entries per ray of the default BVH2 kernels; deeper trees run the TBVH_STACK_DEEP instances
#define TBVH_STACK_DEEP 256    // the reference's own closest-hit stack (tiny_bvh.h:3249; any-hit uses 64, :3409)

// ---- error plumbing -------------------------------------------------------------------------------------
void tbvh_set_error( const char* fmt, ... );
extern unsigned long long g_tbvh_launches;
#define CUDA_TRY( x ) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { tbvh_set_error( "%s:%d %s -> %s", __FILE__, __LINE__, #x, cudaGetErrorString( e_ ) ); return TBVH_E_CUDA; } } while (0)
#define LAUNCHED() do { g_tbvh_launches++; cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) { tbvh_set_error( "%s:%d launch -> %s", __FILE__, __LINE__, cudaGetErrorString( e_ ) ); return TBVH_E_CUDA; } } while (0)
#define ARG_CHECK( c, msg ) do { if (!(c)) { tbvh_set_error( "%s: %s", __func__, msg ); return TBVH_E_ARG; } } while (0)
#define TRY( x ) do { int r_ = (x); if (r_ != TBVH_OK) return r_; } while (0)

// ---- handles ----------------------------------------------------------------------------------------------
// one stage buffer set of the host-buffer pipeline (api.cu "host path")
struct HostSlot
{
	void* d_rays = 0;                // chunk of 64-byte device records
	void* d_hits = 0;                // packed 16-byte hits of the chunk
	void* d_bits = 0;                // occlusion words of the chunk
	void* h_hits = 0;                // page-locked staging for the chunk's packed hits (d2h_mode 2: scattered into the records by host threads)
	cudaEvent_t in_done = 0, run_done = 0, out_done = 0;
};
#define TBVH_SLOTS 4

struct tbvh_ctx_t
{
	int device = 0;
	int sm_count = 132;
	int numa_node = -1;              // host NUMA node the device hangs off (-1 = unknown)
	cudaStream_t stream = 0;         // engine stream (builds, uploads, conversions)
	// host-buffer pipeline: inbound copies, traversal and outbound copies each own a stream, so chunk k+1 flows in while chunk k
	// is traced and the hits of chunk k-1 flow out; the slots are handed round-robin and recycled through events
	std::mutex host_mutex;           // host batch calls on one context are serialised (SURVEY 8(b): thread-safe per handle)
	cudaStream_t s_in = 0, s_run = 0, s_out = 0;
	cudaStream_t s_in_part[3] = { 0, 0, 0 }; // extra inbound streams when h2d_split > 1
	cudaEvent_t ev_part[TBVH_SLOTS][3] = {};
	cudaEvent_t ev_fork = 0;
	HostSlot slot[TBVH_SLOTS];
	size_t chunk_rays = 1u << 19;    // rays per chunk (32 MiB of device records)
	size_t slot_rays = 0;            // capacity the slots were allocated for
	size_t slot_rec = 0;             // bytes per staged ray record the slots were allocated for (64, or 128 under host_path 2)
	int host_path = 0;               // inbound: 0 = copy engine (cudaMemcpy2DAsync of 64-byte rows), 1 = gather kernel through the pinned mapping, 2 = whole 128-byte records in one contiguous copy
	int h2d_split = 1;               // inbound 2D copy of a chunk split over this many streams (copy engines)
	int d2h_mode = 1;                // in-place hits: 1 = bytes 0..63 of every record return (full cache lines, the default), 0 = 2D copy of 16-byte rows,
	                                 // 2 = packed copy + host threads scatter, 3 = scatter kernel through the pinned mapping
	int scatter_threads = 8;         // d2h_mode 2: host threads (bound to the device's NUMA node) that write the hits into the records
	struct HostPool* pool = 0;
	int trace_variant = 3;           // BVH2 traversal kernel: 0 generic, 3 octant switch, 4 persistent warps (see trace_bvh2.cu)
	int small_mode = 0;              // warp-subtree kernel: bit 0 = fragments staged in shared memory, bit 1 = aggregated bin updates
	int inst_idx_bits = 32;          // the host program's INST_IDX_BITS (tiny_bvh.h:118): 32 = TLAS hits store hit.inst, 4..31 = top bits of hit.prim
	int hq_small = 16;               // BuildHQ: nodes of at most this many fragments go to the warp-per-subtree kernel (<= 256)
	int hq_cluster = 16;             // BuildHQ: largest thread-block cluster a node of the level phase may get (1..16)
	int small_t = 128;               // builder: subtrees of at most this many primitives go to the warp kernel (<= 256)
	int build_ctas = 0;              // persistent large phase: CTAs per SM (0 = by scene size)
	int build_mode = 0;              // BVH::Build large phase: 0 = one persistent cooperative launch (k_large_phase), 1 = one launch per stage and level
	// ring of 8-byte device counters for kernels that pull work from a counter (one per launch, so launches on different
	// streams never share one)
	unsigned long long* d_counters = 0;
	std::atomic<uint32_t> counter_next{ 0 };
	// refits (convert_cwbvh.cu refit_trees): tables and scratch of one call, kept and grown, so a steady-state frame allocates nothing
	std::mutex refit_mutex;
	void* refit_dev = 0; size_t refit_dev_bytes = 0;   // device: tables, arrival counters, parents, BVH_GPU workspace, results
	void* refit_host = 0; size_t refit_host_bytes = 0; // page-locked: the tables on their way in, the results on their way out
	cudaEvent_t refit_e0 = 0, refit_e1 = 0;
};
#define TBVH_COUNTERS 256

uint32_t tbvh_next_generation(); // process-wide: a value no handle has carried before (a recycled handle address cannot revalidate a stale TLAS)
struct BlasLink { tbvh_bvh blas; uint32_t generation; }; // host side: what a TLAS was built over

struct tbvh_bvh_t
{
	tbvh_ctx ctx = 0;
	tbvh_info info = {};
	// geometry (engine-owned copy, float4 per vertex)
	float4* d_verts = 0;
	// LAYOUT_BVH: reference node array; children of an interior node are the 64-byte pair at nodes[leftFirst]
	float4* d_nodes = 0;       // 2 float4 per node
	uint32_t* d_prim_idx = 0;
	// traversal view of the BVH2: d_trav aliases d_nodes (LAYOUT_BVH) or is the pair array derived from a BVH_GPU upload
	float4* d_trav = 0;
	uint32_t root_ref = 0, root_count = 0; // the root as a child record: count==0 -> pair index, else leaf range
	// leaf-ordered triangle records for BVH2 traversal: 3 float4 per prim reference
	//   [0] = (v0.xyz, as_float(primIdx))  [1] = e1 = v1-v0  [2] = e2 = v2-v0
	float4* d_leaf_tris = 0;
	uint32_t leaf_tris_count = 0; // records d_leaf_tris was allocated for
	// LAYOUT_BVH_GPU mirror (only materialised on upload / convert / download)
	float4* d_nodes_gpu = 0;   // 4 float4 per node
	// LAYOUT_CWBVH
	float4* d_cw_nodes = 0;    // 5 float4 per node
	float4* d_cw_tris = 0;     // 3 float4 per triangle
	float4* d_cw_trav = 0;     // traversal nodes derived from d_cw_nodes (trace_cwbvh.cu cw_make_trav): 10 float4 per node
	uint32_t cw_pending = 0;   // most node groups a walk of the wide tree can leave pending (trace_cwbvh.cu k_cw_pending)
	float cw_rd_limit = -1.0f; // rays with |rD| up to this (and |O| <= 2^126) take the integer-ordered slab test (cw_walk.cuh cw_ray_fits); < 0: none
	uint32_t generation = 0;   // renewed (tbvh_next_generation) whenever the arrays a TLAS may point at are replaced (build, upload, refit, convert)
	// TLAS (BVH::Build( BLASInstance*, instCount, BVHBase**, blasCount ) :2221): nodes / primIdx over instance boxes + device tables
	float4* d_aabbs = 0;       // instance boxes the TLAS was built over (2 float4 per instance)
	void* d_inst = 0;          // TlasInst records (inverse transform, BLAS number, mask)
	void* d_blas = 0;          // BlasRef records (traversal arrays of every BLAS); tbvh_build_tlas_update: then each BLAS's root box and a flag word
	void* d_inst_stage = 0;    // tbvh_build_tlas_update with host records: bytes 0..159 of every record on their way through the device
	size_t blas_table_bytes = 0; // bytes of d_blas when tbvh_build_tlas_update made it (0: tbvh_build_tlas's, BlasRef records only)
	uint32_t inst_count = 0, blas_count = 0;
	uint32_t tlas_blas_layouts = 0; // TLAS only: layouts EVERY BLAS held at build time (bit TBVH_LAYOUT_BVH / TBVH_LAYOUT_CWBVH)
	uint32_t tlas_deep_blas = 0, tlas_deep_depth = 0; // TLAS only: 1 + the first BLAS whose BVH2 is too deep for the two-level walk (0: none), and its depth
	std::vector<BlasLink> links; // TLAS only: the BLAS handles it points into, with the generation they had at build time
	bool refittable = true;    // BVHBase::refittable (:811): false after BuildHQ ("can't refit an SBVH", :3027)
	struct CwKeep* cw_keep = 0; // refittable trees: the 8-wide collapse of the last tbvh_convert to CWBVH (convert_cwbvh.cu), for tbvh_refit_layouts
	// statistics
	int stats = 0;
	unsigned long long* d_stats = 0; // [0]=steps [1]=tris, accumulated over every launch of one API call
};

// ---- device math in the oracle's exact operation order (oracle/tbvh_oracle.c header lists the pairing) ----
// Every fused pair is spelled __fmaf_rn, every unfused product / sum an _rn intrinsic, so nvcc's own
// contraction (-fmad) cannot change the rounding.

// MOLLER_TRUMBORE_TEST tiny_bvh.h:1644-1656 with e1,e2 precomputed (identical bits: v1-v0 is exact-rounded once).
// Returns true when the triangle is accepted for [0, tmax] ([0, tmax) with below_tmax); writes t,u,v.
__device__ __forceinline__ bool mt_test( const float ox, const float oy, const float oz, const float dx, const float dy, const float dz,
	const float4 v0, const float4 e1, const float4 e2, const float tmax, float& t, float& u, float& v, const bool below_tmax = false )
{
	const float hx = __fmaf_rn( dy, e2.z, -__fmul_rn( dz, e2.y ) );
	const float hy = __fmaf_rn( dz, e2.x, -__fmul_rn( dx, e2.z ) );
	const float hz = __fmaf_rn( dx, e2.y, -__fmul_rn( dy, e2.x ) );
	const float a = __fmaf_rn( e1.z, hz, __fmaf_rn( e1.x, hx, __fmul_rn( e1.y, hy ) ) );
	if (fabsf( a ) < 0.000001f) return false;
	const float f = __fdiv_rn( 1.0f, a );
	const float sx = __fsub_rn( ox, v0.x ), sy = __fsub_rn( oy, v0.y ), sz = __fsub_rn( oz, v0.z );
	u = __fmul_rn( f, __fmaf_rn( hz, sz, __fmaf_rn( hx, sx, __fmul_rn( hy, sy ) ) ) );
	const float qx = __fmaf_rn( -e1.y, sz, __fmul_rn( e1.z, sy ) );
	const float qy = __fmaf_rn( -e1.z, sx, __fmul_rn( e1.x, sz ) );
	const float qz = __fmaf_rn( -e1.x, sy, __fmul_rn( e1.y, sx ) );
	v = __fmul_rn( f, __fmaf_rn( dz, qz, __fmaf_rn( dy, qy, __fmul_rn( dx, qx ) ) ) );
	if (u < 0 || v < 0 || __fadd_rn( u, v ) > 1) return false;
	t = __fmul_rn( f, __fmaf_rn( e2.z, qz, __fmaf_rn( e2.x, qx, __fmul_rn( e2.y, qy ) ) ) );
	return !(t < 0 || (below_tmax ? t >= tmax : t > tmax));
}

// ray record i of a traversal batch: O | mask, D, rD | inst, hit (t, u, v, prim) - four 16-byte loads
__device__ __forceinline__ void load_ray( const char* rays, const uint64_t i, const uint32_t stride, float4& ro4, float4& rd4, float4& rr4, float4& rh4 )
{
	const float4* rp = (const float4*)(rays + i * stride);
	ro4 = rp[0], rd4 = rp[1], rr4 = rp[2], rh4 = rp[3];
}

// any-hit result of a one-ray-per-thread kernel: one ballot word per warp.  blockDim is a multiple of 32 and i is the global thread
// index, so lane l of a warp holds ray 32*w + l; every lane of the warp must call it.
__device__ __forceinline__ void store_occlusion_word( uint32_t* bits, const uint64_t i, const uint64_t n, const bool occluded )
{
	const uint32_t m = __ballot_sync( 0xffffffffu, occluded );
	if ((threadIdx.x & 31) == 0 && (i & ~31ull) < n) bits[i >> 5] = m;
}

// order-preserving float <-> uint key for atomicMin/Max on floats
__device__ __forceinline__ uint32_t f2key( float f ) { uint32_t u = __float_as_uint( f ); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ float key2f( uint32_t k ) { return __uint_as_float( (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k ); }

// Signed zeros.  The reference folds bounds with tinybvh_min / tinybvh_max (tiny_bvh.h:445-446), a < b ? a : b and a > b ? a : b:
// on a tie the second operand wins, so of several zero bounds the one folded LAST gives the result its sign.  The key reductions
// above find the value in any order (key(-0) = 0x7fffffff sits just below key(+0) = 0x80000000); where that value is a zero, the
// builders take the sign from a position word, ((fold position + 1) << 1) | sign bit, reduced with a max.
__device__ __forceinline__ float ref_min( const float a, const float b ) { return a < b ? a : b; }
__device__ __forceinline__ float ref_max( const float a, const float b ) { return a > b ? a : b; }
__device__ __forceinline__ bool zero_key( const uint32_t k ) { return k == 0x7fffffffu || k == 0x80000000u; }
__device__ __forceinline__ uint32_t zpos_word( const uint32_t pos, const float f ) { return ((pos + 1u) << 1) | (__float_as_uint( f ) >> 31); }
// the key of a zero bound whose sign a position word decided (0: no word, keep the key)
__device__ __forceinline__ uint32_t zero_resolve( const uint32_t key, const uint32_t zw ) { return (zw && zero_key( key )) ? ((zw & 1u) ? 0x7fffffffu : 0x80000000u) : key; }

// leaf-ordered triangle record p of a BVH2 (tbvh_bvh_t::d_leaf_tris) for primitive pi: 3 x 16 B gathered vertex reads, 3 x 16 B writes.
// e1 = v1 - v0, e2 = v2 - v0 exactly as IntersectTri computes them per test (tiny_bvh.h:8510)
__device__ __forceinline__ void leaf_tri_record( const float4* __restrict__ verts, const uint32_t pi, float4* __restrict__ out, const uint32_t p )
{
	const float4 v0 = __ldg( verts + (size_t)pi * 3 ), v1 = __ldg( verts + (size_t)pi * 3 + 1 ), v2 = __ldg( verts + (size_t)pi * 3 + 2 );
	out[(size_t)p * 3] = make_float4( v0.x, v0.y, v0.z, __uint_as_float( pi ) );
	out[(size_t)p * 3 + 1] = make_float4( __fsub_rn( v1.x, v0.x ), __fsub_rn( v1.y, v0.y ), __fsub_rn( v1.z, v0.z ), 0.0f );
	out[(size_t)p * 3 + 2] = make_float4( __fsub_rn( v2.x, v0.x ), __fsub_rn( v2.y, v0.y ), __fsub_rn( v2.z, v0.z ), 0.0f );
}

// ---- DFS preorder of a BVH2 in the reference's layout (node 1 unused, children paired at leftFirst), whatever its numbering and
// whatever the order of its leaf ranges in primIdx.  Used by BuildHQ's Compact() (build_hq.cu) and BVH_GPU::ConvertFrom (convert.cu).
// parent[]: the parent of every reachable node, 0xffffffff for the root.
// Bottom-up from leaf x carrying weight w: sub_int[] = interior nodes per subtree, sub_w[] = summed leaf weights per subtree.  The
// second arrival at a parent (arrive[] zeroed beforehand) sums both children and carries on, as refit.cu climbs.
__device__ __forceinline__ void dfs_sizes_up( const float4* nodes, const uint32_t* parent, uint32_t* arrive, uint32_t* sub_int, uint32_t* sub_w,
	uint32_t x, const uint32_t w )
{
	sub_int[x] = 0, sub_w[x] = w;
	for (;;)
	{
		const uint32_t p = parent[x];
		if (p == 0xffffffffu) break;
		__threadfence();
		if (atomicAdd( &arrive[p], 1u ) == 0) break;
		__threadfence();
		const uint32_t lc = __float_as_uint( nodes[(size_t)p * 2].w );
		const volatile uint32_t* si = sub_int; const volatile uint32_t* sw = sub_w;
		sub_int[p] = si[lc] + si[lc + 1] + 1, sub_w[p] = sw[lc] + sw[lc + 1];
		x = p;
	}
}
// Top-down by walking x's path to the root: K = interior nodes before x in DFS preorder, O = leaf weights before x, Kp = the part of
// K that x's own step added (K of x's parent is K - Kp).  With every leaf weighing 1, x's preorder index is K + O.
__device__ __forceinline__ void dfs_rank( const float4* nodes, const uint32_t* parent, const uint32_t* sub_int, const uint32_t* sub_w,
	const uint32_t x, uint32_t& K, uint32_t& O, uint32_t& Kp )
{
	K = 0, O = 0, Kp = 0;
	for (uint32_t c = x; c != 0;)
	{
		const uint32_t p = parent[c], lc = __float_as_uint( nodes[(size_t)p * 2].w );
		uint32_t add = 1;
		if (c == lc + 1) add += sub_int[lc], O += sub_w[lc];
		if (c == x) Kp = add;
		K += add, c = p;
	}
}

// ---- batch tables: the entry of T[0 .. K) whose index range holds g (T[k].*F rises strictly: every entry owns an index)
template <class E, uint32_t E::*F> __device__ __forceinline__ uint32_t batch_entry( const E* __restrict__ T, const uint32_t K, const uint32_t g )
{
	uint32_t lo = 0, hi = K;
	while (hi - lo > 1) { const uint32_t m = (lo + hi) >> 1; if (T[m].*F <= g) lo = m; else hi = m; }
	return lo;
}

// one tree of a refit (refit.cu, convert.cu): BVH::Refit over the batch's node space, the BVH2 traversal records over its primitive
// reference space.  A single tree passes its entry as a kernel parameter instead of a table.
struct RfTree
{
	float4* nodes;
	const uint32_t* prim_idx;
	const float4* verts;
	float4* leaf_tris;
	uint32_t* parent;             // the tree's parents by local node number: kept in its CwKeep, or scratch of the call
	uint32_t nbase, used;         // first node in the batch's node space, BVH2 nodes
	uint32_t pbase, idx_count;    // first primitive reference in the batch's reference space, references
	uint32_t fill;                // parent is filled by this call
};
// one tree of a BVH_GPU::ConvertFrom pass (convert.cu): its BVH2, its output, and its first node in the pass's node space
struct GpuTree { const float4* nodes; float4* out; uint32_t nbase, used; };
// one wide tree of a traversal-node pass (trace_cwbvh.cu): its bvh8Data (src), its traversal nodes (dst), where its results go
// (res[0]: range, res[1]: pending bound) and its first node in the pass's node index space (wbase)
struct CwTrav { const uint4* src; uint4* dst; uint32_t* res; uint32_t wbase, count; };

// ---- internal entry points (one per .cu) -------------------------------------------------------------------
// d_stats: NULL, or two counters the launch ADDS its node visits / triangle tests to (the caller zeroes them once per API call)
int bvh2_trace_launch( tbvh_bvh b, const void* d_rays, uint32_t stride, void* d_hits, uint32_t hit_stride, uint32_t* d_bits, uint64_t n, bool anyhit, cudaStream_t s, unsigned long long* d_stats );
int cwbvh_trace_launch( tbvh_bvh b, const void* d_rays, uint32_t stride, void* d_hits, uint32_t hit_stride, uint32_t* d_bits, uint64_t n, bool anyhit, cudaStream_t s, unsigned long long* d_stats );
// traversal nodes, cw_rd_limit and cw_pending of the CWBVH of each of bs[0 .. K), in one pass (trace_cwbvh.cu); synchronises s
int cw_make_trav( const tbvh_bvh* bs, uint32_t K, cudaStream_t s );
// cw_make_trav's node expansion of the W nodes of K trees (table d_T; K = 1: `one`) into their d_cw_trav; parent: NULL (a refit)
// or where the pending pass finds the parents
int cw_expand( const CwTrav* d_T, uint32_t K, const CwTrav& one, uint32_t W, uint32_t* parent, cudaStream_t s );
float cw_rd_limit_for( uint32_t range );                               // cw_rd_limit of a tree whose expansion found `range`
unsigned long long* ctx_next_counter( tbvh_ctx c ); // a zero-on-use 8-byte device counter from the context's ring (persistent-warp ray fetch)
// binned-SAH builds of `trees` handles of one context at once (build_sah.cu); a single build is trees = 1
int build_sah_launch( const tbvh_bvh* bs, uint32_t trees, float c_trav, float c_int, int flavour );
int build_hq_launch( tbvh_bvh b, float c_trav, float c_int );
// BVH::Refit of K trees over one node space of `nodes` nodes; arrive: `nodes` zeroed words; fill: some tree's parents are filled.
// K = 1 runs the single-tree instances with `one`.
int refit_enqueue( const RfTree* d_T, uint32_t K, const RfTree& one, uint32_t nodes, uint32_t* arrive, bool fill, cudaStream_t s );
int refit_roots( const RfTree* d_T, uint32_t K, uint32_t* out, cudaStream_t s ); // each tree's root node (8 words) to out[8 t ..]
// the leaf-ordered triangle records of K trees over one space of `refs` primitive references (convert.cu); K = 1 as above
int leaf_tris_enqueue( const RfTree* d_T, uint32_t K, const RfTree& one, uint32_t refs, cudaStream_t s );
int leaf_tris_alloc( tbvh_bvh b ); // d_leaf_tris sized to idx_count (kept when it is: a TLAS holding its address stays valid)
// Refit of K handles of one context (tbvh_refit, tbvh_refit_layouts, tbvh_refit_batch): d_verts already hold the new positions.
// keep_layouts: BVH_GPU and CWBVH brought up to date in place, the generation renewed; else both dropped.  One host synchronisation.
// On failure every handle holds its BVH-layout tree (boxes unspecified) and neither BVH_GPU nor CWBVH.
int refit_trees( const tbvh_bvh* bs, uint32_t K, bool keep_layouts, cudaStream_t s );
void cw_keep_sizes( tbvh_bvh b, uint32_t* total, uint32_t* wide_count ); // split-tree and wide nodes of the kept collapse (0: none)
// BVH_GPU::ConvertFrom of K trees over one node space of n nodes into their `out` arrays; w: 4 n words of workspace (zeroed here)
int bvh_gpu_enqueue( const GpuTree* d_T, uint32_t K, const GpuTree& one, uint32_t n, uint32_t* w, cudaStream_t s );
int tlas_trace_launch( tbvh_bvh b, int layout, const void* d_rays, uint32_t stride, uint32_t* d_bits, uint64_t n, bool anyhit, cudaStream_t s );
struct TlasInst { float inv[16]; uint32_t blasIdx, mask, pad0, pad1; };                                  // 80 bytes
struct BlasRef { const float4* trav; const float4* tris; uint32_t root_ref, root_count; float cw_rd_limit; uint32_t pad1; const float4* cw_nodes; const float4* cw_tris; }; // 48 bytes: BVH-layout arrays, CWBVH traversal nodes + bvh8Tris (0 when absent) and their rD limit
// BLASInstance::Update of n records `stride` bytes apart (instance_update.cu): invTransform and world box into the records, the TlasInst
// entries and the builder's boxes in one pass; *d_bad_blas is set when a record names a BLAS past blas_count
int instance_update_launch( void* d_records, uint32_t stride, uint32_t n, const float4* d_blas_box, uint32_t blas_count, void* d_tlas_inst, float4* d_aabbs,
	uint32_t* d_bad_blas, cudaStream_t s );
int make_leaf_tris( tbvh_bvh b, cudaStream_t s );
int bvh_gpu_to_bvh( tbvh_bvh b, uint32_t used_nodes_gpu, cudaStream_t s );
int bvh_to_bvh_gpu( tbvh_bvh b, cudaStream_t s ); // sets the BVH_GPU bit on success; on failure the handle holds no BVH_GPU
void drop_bvh_gpu( tbvh_bvh b );                  // the BVH_GPU array, its bit and used_nodes_gpu (no TLAS points at it: the generation stays)
// BVH8_CWBVH::Build's conversion chain for K handles of one context at once (convert_cwbvh.cu); tbvh_convert is K = 1
int bvh_to_cwbvh( const tbvh_bvh* bs, uint32_t K, cudaStream_t s );
// the CWBVH arrays, the kept collapse, the bit, the counts and the traversal limits; a TLAS over the arrays becomes stale
void drop_cwbvh( tbvh_bvh b );
// exclusive scan of in[0..n) into out[0..n] (out[n] = total); tile_sum needs n/2048 + 2 words (build_sah.cu)
int exclusive_scan( const uint32_t* in, uint32_t* out, uint32_t* tile_sum, uint32_t n, cudaStream_t s );
