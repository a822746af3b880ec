// tinybvh_b200/csrc/common.cuh - shared device/host definitions of the sm_90a engine.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <mutex>
#include <vector>
#include <atomic>
#include "../../include/tinybvh_b200.h"
#include "../../include/tinybvh_b200_device/base.cuh" // BVH_FAR, the stack sizes, mt_test, ref_min / ref_max, load_ray, TlasInst / BlasRef

using tbvh::mt_test;
using tbvh::ref_min;
using tbvh::ref_max;
using tbvh::load_ray;
using tbvh::TlasInst;
using tbvh::BlasRef;

// ---- error plumbing -------------------------------------------------------------------------------------
void tbvh_set_error( const char* fmt, ... );
extern unsigned long long g_tbvh_launches;
#define CUDA_TRY( x ) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { tbvh_set_error( "%s:%d %s -> %s", __FILE__, __LINE__, #x, cudaGetErrorString( e_ ) ); return TBVH_E_CUDA; } } while (0)
#define LAUNCHED() do { g_tbvh_launches++; cudaError_t e_ = cudaGetLastError(); if (e_ != cudaSuccess) { tbvh_set_error( "%s:%d launch -> %s", __FILE__, __LINE__, cudaGetErrorString( e_ ) ); return TBVH_E_CUDA; } } while (0)
#define ARG_CHECK( c, msg ) do { if (!(c)) { tbvh_set_error( "%s: %s", __func__, msg ); return TBVH_E_ARG; } } while (0)
#define TRY( x ) do { int r_ = (x); if (r_ != TBVH_OK) return r_; } while (0)

// ---- the scratch of one host call on stream s: its device allocations (one cudaMalloc each), its page-locked words and its two timing
// events.  The destructor drains s and then frees them all, on every return path.  Buffers that outlive the call are not scratch.
struct Scratch
{
	cudaStream_t s;
	cudaEvent_t e0 = 0, e1 = 0;
	std::vector<void*> dev, pinned;
	explicit Scratch( cudaStream_t stream ) : s( stream ) {}
	Scratch( const Scratch& ) = delete;
	Scratch& operator=( const Scratch& ) = delete;
	~Scratch()
	{
		cudaStreamSynchronize( s );
		for (void* p : dev) cudaFree( p );
		for (void* p : pinned) cudaFreeHost( p );
		if (e0) cudaEventDestroy( e0 );
		if (e1) cudaEventDestroy( e1 );
	}
	template <class T> int alloc( T*& p, size_t bytes ) { void* q = 0; CUDA_TRY( cudaMalloc( &q, bytes ) ); dev.push_back( q ); p = (T*)q; return TBVH_OK; }
	template <class T> int alloc_host( T*& p, size_t bytes ) { void* q = 0; CUDA_TRY( cudaMallocHost( &q, bytes ) ); pinned.push_back( q ); p = (T*)q; return TBVH_OK; }
	int events() { CUDA_TRY( cudaEventCreate( &e0 ) ); CUDA_TRY( cudaEventCreate( &e1 ) ); return TBVH_OK; }
};

// ---- the owner of one allocation that outlives a call: one cudaMalloc (HOST: one page-locked block), freed when the owner is reset,
// reassigned or destroyed.  It frees on the current device: whoever releases it sets the device first, and drains any stream whose
// queued work may still read it.  bytes: the size of the block (reserve keeps it while a request fits).
template <bool HOST> struct Owned
{
	void* p = 0;
	size_t bytes = 0;
	Owned() = default;
	Owned( Owned&& o ) noexcept : p( o.p ), bytes( o.bytes ) { o.p = 0, o.bytes = 0; }
	Owned& operator=( Owned&& o ) noexcept { if (this != &o) { reset(); p = o.p, bytes = o.bytes, o.p = 0, o.bytes = 0; } return *this; }
	~Owned() { reset(); }
	void reset() { if (p) { if (HOST) cudaFreeHost( p ); else cudaFree( p ); } p = 0, bytes = 0; }
	int alloc( size_t n )
	{
		reset();
		void* q = 0;
		CUDA_TRY( HOST ? cudaMallocHost( &q, n ) : cudaMalloc( &q, n ) );
		p = q, bytes = n;
		return TBVH_OK;
	}
	int reserve( size_t n ) { return n <= bytes ? TBVH_OK : alloc( n + n / 4 ); } // grown with a quarter of headroom, so a steady state allocates nothing
	void adopt( void* q, size_t n ) { reset(); p = q, bytes = n; }              // a block allocated elsewhere (HOST: cudaHostAlloc on a NUMA node)
};
typedef Owned<false> DevMem;
typedef Owned<true> HostMem;
template <class T> struct DevArray : DevMem { T* get() const { return (T*)p; } operator T*() const { return get(); } };

// ---- a CUB radix sort on s (build_ploc.cu, signed_distance.cu).  Its kernel launches are counted exactly (g_tbvh_launches): the same call is first captured into a graph
// that is never launched, and its kernel nodes are counted; then it is enqueued.
template <class Sort> int sort_enqueue( cudaStream_t s, Sort sort )
{
	cudaGraph_t g = 0;
	CUDA_TRY( cudaStreamBeginCapture( s, cudaStreamCaptureModeRelaxed ) );
	const cudaError_t e = sort(), e2 = cudaStreamEndCapture( s, &g );
	size_t count = 0, kernels = 0;
	if (e == cudaSuccess && e2 == cudaSuccess && cudaGraphGetNodes( g, 0, &count ) == cudaSuccess)
	{
		std::vector<cudaGraphNode_t> nodes( count );
		cudaGraphGetNodes( g, nodes.data(), &count );
		for (cudaGraphNode_t x : nodes) { cudaGraphNodeType t; if (cudaGraphNodeGetType( x, &t ) == cudaSuccess && t == cudaGraphNodeTypeKernel) kernels++; }
	}
	if (g) cudaGraphDestroy( g );
	CUDA_TRY( e );
	CUDA_TRY( e2 );
	CUDA_TRY( sort() );
	g_tbvh_launches += kernels;
	return TBVH_OK;
}

// ---- handles ----------------------------------------------------------------------------------------------
// one stage buffer set of the host-buffer pipeline (api.cu "host path")
struct HostSlot
{
	DevArray<char> d_rays;           // chunk of 64-byte device records
	DevArray<float4> d_hits;         // packed 16-byte hits of the chunk
	DevArray<uint32_t> d_bits;       // occlusion words of the chunk
	HostMem h_hits;                  // page-locked staging for the chunk's packed hits (d2h_mode 2: scattered into the records by host threads)
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
	DevArray<unsigned long long> d_counters;
	std::atomic<uint32_t> counter_next{ 0 };
	// refits (convert_cwbvh.cu refit_trees): tables and scratch of one call, kept and grown, so a steady-state frame allocates nothing
	std::mutex refit_mutex;
	DevArray<char> refit_dev;        // device: tables, arrival counters, parents, BVH_GPU workspace, results
	HostMem refit_host;              // page-locked: the tables on their way in, the results on their way out
	cudaEvent_t refit_e0 = 0, refit_e1 = 0;
	// indexed refits (api.cu tbvh_refit_batch_indexed): the new vertices of the call's indexed meshes at a 16-byte pitch and the gather
	// table, kept and grown; the mutex is held for the whole call (the refit inside it takes refit_mutex)
	std::mutex ix_mutex;
	DevArray<char> ix_dev;
};
#define TBVH_COUNTERS 256

uint32_t tbvh_next_generation(); // process-wide: a value no handle has carried before (a recycled handle address cannot revalidate a stale TLAS)
struct BlasLink { tbvh_bvh blas; uint32_t generation; }; // host side: what a TLAS was built over

struct tbvh_bvh_t
{
	tbvh_ctx ctx = 0;
	tbvh_info info = {};
	// geometry (engine-owned copy, float4 per vertex)
	DevArray<float4> d_verts;
	// indexed, refittable builds: the 3 * prim_count vertex indices and the vertex count (BVHBase::vertIdx, tiny_bvh.h:806-807), through
	// which tbvh_refit_batch_indexed writes d_verts from the new positions.  Dropped with the tree (free_layouts); 0 otherwise.
	DevArray<uint32_t> d_vert_idx;
	uint32_t vert_count = 0;
	// LAYOUT_BVH: reference node array; children of an interior node are the 64-byte pair at nodes[leftFirst]
	DevArray<float4> d_nodes;  // 2 float4 per node
	DevArray<uint32_t> d_prim_idx;
	// the child-pair array derived from a BVH_GPU upload (convert.cu bvh_gpu_to_bvh); empty otherwise
	DevArray<float4> d_pairs;
	// traversal view of the BVH2: the pair array of a BVH_GPU upload, else d_nodes (LAYOUT_BVH)
	float4* trav() const { return d_pairs.p ? d_pairs : d_nodes; }
	uint32_t root_ref = 0, root_count = 0; // the root as a child record: count==0 -> pair index, else leaf range
	// leaf-ordered triangle records for BVH2 traversal: 3 float4 per prim reference
	//   [0] = (v0.xyz, as_float(primIdx))  [1] = e1 = v1-v0  [2] = e2 = v2-v0
	DevArray<float4> d_leaf_tris;
	uint32_t leaf_tris_count = 0; // records d_leaf_tris was allocated for
	// LAYOUT_BVH_GPU mirror (only materialised on upload / convert / download)
	DevArray<float4> d_nodes_gpu; // 4 float4 per node
	// LAYOUT_CWBVH
	DevArray<float4> d_cw_nodes;  // 5 float4 per node
	DevArray<float4> d_cw_tris;   // 3 float4 per triangle
	DevArray<float4> d_cw_trav;   // traversal nodes derived from d_cw_nodes (trace_cwbvh.cu cw_make_trav): 10 float4 per node
	uint32_t cw_pending = 0;   // most node groups a walk of the wide tree can leave pending (trace_cwbvh.cu k_cw_pending)
	float cw_rd_limit = -1.0f; // rays with |rD| up to this (and |O| <= 2^126) take the integer-ordered slab test (cw_walk.cuh cw_ray_fits); < 0: none
	uint32_t generation = 0;   // renewed (tbvh_next_generation) whenever the arrays a TLAS may point at are replaced (build, upload, refit, convert)
	uint32_t revision = 0;     // counts refits: a refit that drops no layout rewrites the BVH2 arrays in place under the same generation, and a
	                           // group's scene replicas (multi.cu) must notice that too
	uint32_t tree_stamp = 0;   // renewed (tbvh_next_generation) whenever the BVH2 or its vertices are replaced (build, upload, changing optimize);
	                           // unlike the generation, not by a conversion, which leaves both as they were
	// TLAS (BVH::Build( BLASInstance*, instCount, BVHBase**, blasCount ) :2221): nodes / primIdx over instance boxes + device tables
	DevArray<float4> d_aabbs;  // instance boxes the TLAS was built over (2 float4 per instance)
	DevArray<TlasInst> d_inst; // TlasInst records (inverse transform, BLAS number, mask)
	DevArray<char> d_blas;     // BlasRef records (traversal arrays of every BLAS); tbvh_build_tlas_update: then each BLAS's root box and a flag word
	DevArray<char> d_inst_stage; // tbvh_build_tlas_update with host records: bytes 0..159 of every record on their way through the device
	size_t blas_table_bytes = 0; // bytes of d_blas when tbvh_build_tlas_update made it (0: tbvh_build_tlas's, BlasRef records only)
	uint32_t inst_count = 0, blas_count = 0;
	uint32_t tlas_blas_layouts = 0; // TLAS only: layouts EVERY BLAS held at build time (bit TBVH_LAYOUT_BVH / TBVH_LAYOUT_CWBVH)
	uint32_t tlas_deep_blas = 0, tlas_deep_depth = 0; // TLAS only: 1 + the first BLAS whose BVH2 is too deep for the two-level walk (0: none), and its depth
	std::vector<BlasLink> links; // TLAS only: the BLAS handles it points into, with the generation they had at build time
	bool refittable = true;    // BVHBase::refittable (:811): false after BuildHQ ("can't refit an SBVH", :3027)
	bool stray_slots = false;  // tbvh_upload_bvh: a slot other than node 1 is outside the tree, or the tree reaches node 1 or a slot past
	                           // used_nodes, or reaches a slot twice (builders never leave such a tree; tbvh_optimize refuses it)
	// signed-distance table (signed_distance.cu): 7 float4 per primitive, valid while the handle's tree_stamp and revision equal the
	// stamp taken by tbvh_signed_distance_prepare (every build, upload, changing optimisation and refit changes one of them)
	DevArray<float4> d_sdf;
	uint32_t sdf_tree_stamp = 0, sdf_revision = 0;
	// winding-number table (winding_number.cu): 4 float4 per slot of trav() plus the root's, and per primitive reference the prim it
	// owns (0xffffffff: none); stamped and made stale exactly as d_sdf
	DevArray<float4> d_wn;
	DevArray<uint32_t> d_wn_own;
	uint32_t wn_tree_stamp = 0, wn_revision = 0;
	struct CwKeep* cw_keep = 0; // refittable trees: the 8-wide collapse of the last tbvh_convert to CWBVH (convert_cwbvh.cu), for tbvh_refit_layouts
	// statistics
	int stats = 0;
	DevArray<unsigned long long> d_stats; // [0]=steps [1]=tris, accumulated over every launch of one API call
};

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

// Signed zeros.  The reference folds bounds with tinybvh_min / tinybvh_max (ref_min / ref_max): on a tie the second operand wins,
// so of several zero bounds the one folded LAST gives the result its sign.  The key reductions above find the value in any order
// (key(-0) = 0x7fffffff sits just below key(+0) = 0x80000000); where that value is a zero, the builders take the sign from a
// position word, ((fold position + 1) << 1) | sign bit, reduced with a max.
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
// The walk ends at node 0 or at a node whose parent is 0xffffffff, and returns that root: the trees of a BuildHQ batch share one
// node space, tree t rooted at node 2t.
__device__ __forceinline__ uint32_t dfs_rank( const float4* nodes, const uint32_t* parent, const uint32_t* sub_int, const uint32_t* sub_w,
	const uint32_t x, uint32_t& K, uint32_t& O, uint32_t& Kp )
{
	K = 0, O = 0, Kp = 0;
	uint32_t c = x;
	for (uint32_t p; c != 0 && (p = parent[c]) != 0xffffffffu; c = p)
	{
		const uint32_t lc = __float_as_uint( nodes[(size_t)p * 2].w );
		uint32_t add = 1;
		if (c == lc + 1) add += sub_int[lc], O += sub_w[lc];
		if (c == x) Kp = add;
		K += add;
	}
	return c;
}

// ---- batch tables: the entry of T[0 .. K) whose index range holds g (T[k].*F rises strictly: every entry owns an index)
template <class E, uint32_t E::*F> __device__ __forceinline__ uint32_t batch_entry( const E* __restrict__ T, const uint32_t K, const uint32_t g )
{
	uint32_t lo = 0, hi = K;
	while (hi - lo > 1) { const uint32_t m = (lo + hi) >> 1; if (T[m].*F <= g) lo = m; else hi = m; }
	return lo;
}

// one tree of a refit (refit.cu, convert.cu): BVH::Refit over the batch's node space, the BVH2 traversal records over its primitive
// reference space.  A single tree is a one-entry table.
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
// cw_make_trav's node expansion of the W nodes of K trees (table d_T) into their d_cw_trav; parent: NULL (a refit) or where the
// pending pass finds the parents
int cw_expand( const CwTrav* d_T, uint32_t K, uint32_t W, uint32_t* parent, cudaStream_t s );
float cw_rd_limit_for( uint32_t range );                               // cw_rd_limit of a tree whose expansion found `range`
unsigned long long* ctx_next_counter( tbvh_ctx c ); // a zero-on-use 8-byte device counter from the context's ring (persistent-warp ray fetch)
// A tree a builder has written into a handle's d_nodes / d_prim_idx: the root node's 8 words (aabbMin, leftFirst, aabbMax, triCount)
// and the counts.  install_tree (api.cu) makes the handle hold it.
struct BuiltTree { uint32_t root[8]; uint32_t used_nodes, idx_count, max_depth; };
// The builders of `trees` handles of one context at once; a single build is trees = 1.  Each handle holds its primitives (d_verts, or
// d_aabbs for a TLAS, which is built alone) and info.prim_count.  The builder allocates the handle's d_nodes, d_prim_idx and (but for a
// TLAS) d_leaf_tris; on success out[t] describes tree t and *ms is the call's build time.  On failure the caller empties the handles.
// binned SAH (build_sah.cu)
int build_sah_launch( const tbvh_bvh* bs, uint32_t trees, float c_trav, float c_int, int flavour, BuiltTree* out, float* ms );
// the fragment pass of the binned builder (k_fragments) for the PLOC builder, on sc.s: every triangle's box into frag_min / frag_max at
// its position of the batch's index space (tree t from d_base[t] on), every tree's root box as six ordered keys (min xyz, max xyz) at
// (*keys)[key_stride * t ..]; its allocations are sc's
int fragments_launch( const tbvh_bvh* bs, uint32_t trees, const uint32_t* d_base, uint32_t n, float4* frag_min, float4* frag_max,
	const uint32_t** keys, uint32_t* key_stride, Scratch& sc );
// PLOC (TBVH_BUILD_PLOC, build_ploc.cu)
int build_ploc_launch( const tbvh_bvh* bs, uint32_t trees, float c_trav, float c_int, BuiltTree* out, float* ms );
// SBVH (BuildHQ, build_hq.cu)
int build_hq_launch( const tbvh_bvh* bs, uint32_t trees, float c_trav, float c_int, BuiltTree* out, float* ms );
// BVH::Refit of K trees over one node space of `nodes` nodes; arrive: `nodes` zeroed words; fill: some tree's parents are filled
int refit_enqueue( const RfTree* d_T, uint32_t K, uint32_t nodes, uint32_t* arrive, bool fill, cudaStream_t s );
int refit_roots( const RfTree* d_T, uint32_t K, uint32_t* out, cudaStream_t s ); // each tree's root node (8 words) to out[8 t ..]
// the leaf-ordered triangle records of K trees over one space of `refs` primitive references (convert.cu)
int leaf_tris_enqueue( const RfTree* d_T, uint32_t K, uint32_t refs, cudaStream_t s );
int leaf_tris_alloc( tbvh_bvh b ); // d_leaf_tris sized to idx_count (kept when it is: a TLAS holding its address stays valid)
// Refit of K handles of one context (tbvh_refit, tbvh_refit_layouts, tbvh_refit_batch): d_verts already hold the new positions.
// keep_layouts: BVH_GPU and CWBVH brought up to date in place, the generation renewed; else both dropped.  One host synchronisation.
// On failure every handle holds its BVH-layout tree (boxes unspecified) and neither BVH_GPU nor CWBVH.
int refit_trees( const tbvh_bvh* bs, uint32_t K, bool keep_layouts, cudaStream_t s );
void cw_keep_sizes( tbvh_bvh b, uint32_t* total, uint32_t* wide_count ); // split-tree and wide nodes of the kept collapse (0: none)
// BVH_GPU::ConvertFrom of K trees over one node space of n nodes into their `out` arrays; w: 4 n words of workspace (zeroed here)
int bvh_gpu_enqueue( const GpuTree* d_T, uint32_t K, uint32_t n, uint32_t* w, cudaStream_t s );
int tlas_trace_launch( tbvh_bvh b, int layout, const void* d_rays, uint32_t stride, uint32_t* d_bits, uint64_t n, bool anyhit, cudaStream_t s );
// the refusals of a launch of n rays before any work (n = 0 refuses only what precedes the launches' own `n == 0` exit); the device
// views (api.cu tbvh_device_view) make the same checks for n > 0
int bvh2_trace_check( tbvh_bvh b, uint64_t n );
int cwbvh_trace_check( tbvh_bvh b, uint64_t n );
int tlas_trace_check( tbvh_bvh b, int layout );
uint32_t tlas_inst_shift( tbvh_bvh b ); // 32 - INST_IDX_BITS of the context's inst_idx_bits, 0 for 32 (hit.inst)
// the BLAS list of a TLAS build (api.cu): the device record of every BLAS, the layouts all of them hold, and the first BLAS too deep for
// the two-level kernel's BVH-layout walk (1 + its number; 0: none).  Reads host state only and touches no handle.
struct TlasBlasTable { std::vector<BlasRef> refs; uint32_t layouts, deep_blas, deep_depth; };
int tlas_blas_table( const tbvh_bvh t, const tbvh_bvh* blasses, const uint32_t blas_count, TlasBlasTable& T );
int tlas_stale_check( tbvh_bvh t ); // TBVH_E_STATE once a BLAS the TLAS was built over has been rebuilt, re-uploaded or destroyed
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
// tbvh_optimize's rounds over b's BVH-layout tree (optimize.cu).  Writes nothing when *rounds ends 0; else out is a new allocation
// holding the renumbered tree (*used nodes, depth *depth), *sah its SAHCost and *ms the device time of the call.
int optimize_tree( tbvh_bvh b, uint32_t max_rounds, float c_trav, float c_int, DevArray<float4>& out, uint32_t* used, uint32_t* depth, uint32_t* rounds, float* sah, float* ms );
// exclusive scan of in[0..n) into out[0..n] (out[n] = total); tile_sum needs n/2048 + 2 words (build_sah.cu)
int exclusive_scan( const uint32_t* in, uint32_t* out, uint32_t* tile_sum, uint32_t n, cudaStream_t s );
// batched proximity queries (closest_point.cu): the argument checks, the staging of TBVH_HOST batches and the launch of one kind
// PROX_WINDING: 4-byte results and the expansion's beta (unused by the other kinds)
enum { PROX_CLOSEST = 0, PROX_ANY = 1, PROX_SIGNED = 2, PROX_WINDING = 3 };
int proximity_query( const char* fn, tbvh_bvh b, const void* queries, void* out, uint64_t n, int space, void* stream, int kind, float beta = 0.0f );
// signed distances (signed_distance.cu): TBVH_E_STATE without a table prepared for the handle's current tree and vertices; the launch
// of n > 0 device-space queries after proximity_query's checks
int sd_table_check( tbvh_bvh b );
int sd_launch( tbvh_bvh b, const float4* d_queries, float4* d_results, uint64_t n, cudaStream_t s );
// winding numbers (winding_number.cu): the same pair for the winding-number table
int wn_table_check( tbvh_bvh b );
int wn_launch( tbvh_bvh b, const float4* d_queries, float* d_results, uint64_t n, float beta, cudaStream_t s );
