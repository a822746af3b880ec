// oracle/ref_wrap.cpp - C-ABI wrapper around the UNMODIFIED reference (tiny_bvh.h), compiled from where
// it lies under /root/reference into oracle/_ref/libtinybvh_ref.so (recipe: oracle/Makefile).
//
// TEST INFRASTRUCTURE ONLY.  Nothing under tinybvh_b200/ (the product) may load this library; it is
// used by tests/, by __graft_entry__.smoke() and by bench.py's cpu_baseline / --impl reference arms
// as the checker / the CPU baseline.  No reference source is copied here: this file only *includes*
// the reference header and calls its public API.
//
// What is exposed (all cited lines are /root/reference/tiny_bvh.h):
//   ref_bvh_build        -> BVH::Build  (:2124, scalar binned SAH "reference builder"), BuildAVX (:6351), BuildHQ (:2623)
//   ref_bvh_optimize     -> BVH::Build (:2124) followed by BVH::Optimize (:3043, BVH_Verbose::Optimize :4338)
//   ref_bvh_intersect    -> BVH::Intersect (:3222)      ref_bvh_occluded -> BVH::IsOccluded (:3382)
//   ref_bvhgpu_*         -> BVH_GPU::ConvertFrom (:4612), BVH_GPU::Intersect (:4657)
//   ref_cwbvh_*          -> BVH8_CWBVH::Build/BuildHQ (:5822-5866), ConvertFrom (:5884), CPU Intersect (:7046)
//   ref_bvh8cpu_*        -> BVH8_CPU::Build/BuildHQ, Intersect (:7210), IsOccluded  (the CPU *performance* baseline)
#define TINYBVH_IMPLEMENTATION
#include "tiny_bvh.h"
#include <atomic>
#include <thread>
#include <vector>
#include <cstring>
#include <cstdio>

using namespace tinybvh;

static_assert( sizeof( Ray ) == 128, "host Ray record is 128 bytes" );
static_assert( offsetof( Ray, hit ) + offsetof( Intersection, t ) == 48, "hit.t at byte 48" );
static_assert( offsetof( Ray, hit ) + offsetof( Intersection, prim ) == 60, "hit.prim at byte 60" );
static_assert( sizeof( BVH::BVHNode ) == 32 && sizeof( BVH_GPU::BVHNode ) == 64, "node sizes" );

// ---- generic multi-threaded driver: 10,000-ray batches off an atomic counter (tiny_bvh_speedtest.cpp:387-401)
template <class F> static void parallel_rays( uint64_t n, int threads, F f )
{
	if (threads <= 0) threads = (int)std::thread::hardware_concurrency();
	if (threads <= 1 || n < 20000) { f( 0, n ); return; }
	const uint64_t B = 10000, batches = (n + B - 1) / B;
	std::atomic<uint64_t> next( 0 );
	std::vector<std::thread> pool;
	for (int t = 0; t < threads; t++) pool.emplace_back( [&]() {
		for (;;) { uint64_t b = next.fetch_add( 1 ); if (b >= batches) break; uint64_t s = b * B, e = s + B > n ? n : s + B; f( s, e ); }
	} );
	for (auto& t : pool) t.join();
}

extern "C" {

int ref_hardware_threads() { return (int)std::thread::hardware_concurrency(); }
int ref_sizeof_ray() { return (int)sizeof( Ray ); }

// ---------------------------------------------------------------- BVH (Wald 32-byte nodes)
// mode: 0 = BVH::Build (scalar reference builder), 1 = BuildAVX, 2 = BuildHQ (SBVH).
// threaded: 0 -> deterministic single-thread node numbering (children of the k-th split interior node in DFS
// preorder get indices 2+2k, 3+2k: tiny_bvh.h:2426-2443), 1 -> library default (std::thread fan-out, :2433).
void* ref_bvh_build( const float* verts, uint32_t primCount, int mode, int threaded )
{
	BVH* b = new BVH();
	b->threadedBuild = threaded != 0;
	const bvhvec4* v = (const bvhvec4*)verts;
	if (mode == 0) b->Build( v, primCount );
	else if (mode == 1) b->BuildAVX( v, primCount );
	else b->BuildHQ( v, primCount );
	return b;
}
// non-default SAH constants (BVHBase::c_trav / c_int, :819-820)
void* ref_bvh_build_costs( const float* verts, uint32_t primCount, int mode, int threaded, float c_trav, float c_int )
{
	BVH* b = new BVH();
	b->threadedBuild = threaded != 0, b->c_trav = c_trav, b->c_int = c_int;
	const bvhvec4* v = (const bvhvec4*)verts;
	if (mode == 0) b->Build( v, primCount ); else if (mode == 1) b->BuildAVX( v, primCount ); else b->BuildHQ( v, primCount );
	return b;
}
// the ( vertices, indices, primCount ) overloads (:2139, :6410, :2641): verts holds vertCount vertices, indices 3 * primCount entries
void* ref_bvh_build_indexed( const float* verts, uint32_t vertCount, const uint32_t* indices, uint32_t primCount, int mode, int threaded )
{
	BVH* b = new BVH();
	b->threadedBuild = threaded != 0;
	const bvhvec4slice v( (const bvhvec4*)verts, vertCount, sizeof( bvhvec4 ) );
	if (mode == 0) b->Build( v, indices, primCount );
	else if (mode == 1) b->BuildAVX( v, indices, primCount );
	else b->BuildHQ( v, indices, primCount );
	return b;
}
void ref_bvh_destroy( void* h ) { delete (BVH*)h; }
uint32_t ref_bvh_used_nodes( void* h ) { return ((BVH*)h)->usedNodes; }
uint32_t ref_bvh_idx_count( void* h ) { return ((BVH*)h)->idxCount; }
uint32_t ref_bvh_tri_count( void* h ) { return ((BVH*)h)->triCount; }
const void* ref_bvh_nodes( void* h ) { return ((BVH*)h)->bvhNode; }
const uint32_t* ref_bvh_prim_idx( void* h ) { return ((BVH*)h)->primIdx; }
float ref_bvh_sah_cost( void* h ) { return ((BVH*)h)->SAHCost(); }
void ref_bvh_compact( void* h ) { ((BVH*)h)->Compact(); }
void ref_bvh_refit( void* h ) { ((BVH*)h)->Refit(); } // the caller has already moved the vertices in the array the BVH points at
void ref_bvh_split_leafs( void* h, uint32_t maxPrims ) { ((BVH*)h)->SplitLeafs( maxPrims ); }
// BVH::Build, then the reference's own reinsertion optimiser: the tree the shim's BVH::Optimize uploads (subtrees moved, every leaf
// keeps its firstTri, so the leaf ranges are no longer in DFS order)
void* ref_bvh_optimize( const float* verts, uint32_t primCount, uint32_t iterations, int extreme, int stochastic )
{
	BVH* b = new BVH();
	b->threadedBuild = false;
	b->Build( (const bvhvec4*)verts, primCount );
	b->Optimize( iterations, extreme != 0, stochastic != 0 );
	return b;
}
// wrap externally produced arrays (e.g. a GPU-built tree) so the reference can traverse / score them.
void* ref_bvh_from_arrays( const void* nodes, uint32_t usedNodes, const uint32_t* primIdx, uint32_t idxCount, const float* verts, uint32_t primCount )
{
	BVH* b = new BVH();
	b->bvhNode = (BVH::BVHNode*)b->AlignedAlloc( (size_t)usedNodes * 32 );
	memcpy( b->bvhNode, nodes, (size_t)usedNodes * 32 );
	b->primIdx = (uint32_t*)b->AlignedAlloc( (size_t)idxCount * 4 );
	memcpy( b->primIdx, primIdx, (size_t)idxCount * 4 );
	b->verts = bvhvec4slice( (const bvhvec4*)verts, primCount * 3, sizeof( bvhvec4 ) );
	b->usedNodes = b->allocatedNodes = usedNodes, b->idxCount = idxCount, b->triCount = primCount;
	b->aabbMin = b->bvhNode[0].aabbMin, b->aabbMax = b->bvhNode[0].aabbMax;
	return b;
}
void ref_bvh_intersect( void* h, void* rays, uint64_t n, int threads )
{
	const BVH* b = (BVH*)h; Ray* r = (Ray*)rays;
	parallel_rays( n, threads, [=]( uint64_t s, uint64_t e ) { for (uint64_t i = s; i < e; i++) b->Intersect( r[i] ); } );
}
// the sum of the values BVH::Intersect returns - (int32_t)( c_trav * nodes visited + c_int * triangles tested ) per ray (:3303), which
// the speedtest accumulates into rayCost (tiny_bvh_speedtest.cpp:197-214)
uint64_t ref_bvh_intersect_cost( void* h, void* rays, uint64_t n, int threads )
{
	const BVH* b = (BVH*)h; Ray* r = (Ray*)rays;
	std::atomic<uint64_t> total( 0 );
	std::atomic<uint64_t>* tp = &total;
	parallel_rays( n, threads, [=]( uint64_t s, uint64_t e ) { uint64_t c = 0; for (uint64_t i = s; i < e; i++) c += (uint64_t)b->Intersect( r[i] ); *tp += c; } );
	return total.load();
}
// bits: one bit per ray, bit (i&31) of word i>>5; caller zero-initialises.  Batches are 10,000 rays, not
// word-aligned, so occlusion is first written as bytes and packed afterwards.
void ref_bvh_occluded( void* h, const void* rays, uint64_t n, uint32_t* bits, int threads )
{
	const BVH* b = (BVH*)h; const Ray* r = (const Ray*)rays;
	std::vector<uint8_t> occ( n );
	uint8_t* o = occ.data();
	parallel_rays( n, threads, [=]( uint64_t s, uint64_t e ) { for (uint64_t i = s; i < e; i++) o[i] = b->IsOccluded( r[i] ) ? 1 : 0; } );
	for (uint64_t i = 0; i < n; i++) if (o[i]) bits[i >> 5] |= 1u << (i & 31);
}

// SBVH helpers, exposed so the restatement's clip_frag / split_frag can be pinned function by function
int ref_clip_frag( void* h, const void* orig, void* out, const float* bmin, const float* bmax, const float* minDim, uint32_t axis )
{
	const BVH* b = (BVH*)h;
	return b->ClipFrag( *(const BVHBase::Fragment*)orig, *(BVHBase::Fragment*)out, bvhvec3( bmin[0], bmin[1], bmin[2] ), bvhvec3( bmax[0], bmax[1], bmax[2] ),
		bvhvec3( minDim[0], minDim[1], minDim[2] ), axis ) ? 1 : 0;
}
void ref_split_frag( void* h, const void* orig, void* left, void* right, const float* minDim, uint32_t axis, float pos, int* lok, int* rok )
{
	const BVH* b = (BVH*)h;
	bool l = false, r = false;
	const bvhvec3 md( minDim[0], minDim[1], minDim[2] );
	b->SplitFrag( *(const BVHBase::Fragment*)orig, *(BVHBase::Fragment*)left, *(BVHBase::Fragment*)right, md, axis, pos, l, r );
	*lok = l, *rok = r;
}

// ---------------------------------------------------------------- TLAS over BVH-layout BLASses
// BVH::Build( BLASInstance*, instCount, BVHBase**, blasCount ) :2221 + IntersectTLAS :3306 / IsOccludedTLAS :3455.
// instances: instCount records of the reference's 192-byte BLASInstance (:1443) with transform / blasIdx / mask filled in;
// Update() (:8386) writes invTransform and the world-space box into them, as the reference's own Build does.
static_assert( sizeof( BLASInstance ) == 192, "BLASInstance is 192 bytes" );
struct RefTLAS { BVH tlas; std::vector<BVHBase*> blas; };
void* ref_tlas_build( void* instances, uint32_t instCount, void** blasHandles, uint32_t blasCount )
{
	RefTLAS* t = new RefTLAS();
	for (uint32_t i = 0; i < blasCount; i++) t->blas.push_back( (BVH*)blasHandles[i] );
	t->tlas.threadedBuild = false;
	t->tlas.Build( (BLASInstance*)instances, instCount, t->blas.data(), blasCount );
	return t;
}
// BLASInstance::Update (:8386) on one 192-byte record, for a BLAS whose root box is [bmin, bmax]
void ref_instance_update( void* instance, const float* bmin, const float* bmax )
{
	BVH blas;
	blas.aabbMin = bvhvec3( bmin[0], bmin[1], bmin[2] ), blas.aabbMax = bvhvec3( bmax[0], bmax[1], bmax[2] );
	((BLASInstance*)instance)->Update( &blas );
}
void ref_tlas_destroy( void* h ) { delete (RefTLAS*)h; }
void* ref_tlas_bvh( void* h ) { return &((RefTLAS*)h)->tlas; }
int ref_sizeof_blas_instance() { return (int)sizeof( BLASInstance ); }
int ref_inst_idx_bits() { return INST_IDX_BITS; }
int ref_offsetof_hit_inst() {
#if INST_IDX_BITS == 32
	return (int)(offsetof( Ray, hit ) + offsetof( Intersection, inst ));
#else
	return -1;
#endif
}

// ---------------------------------------------------------------- BVH_GPU (Aila-Laine 64-byte nodes)
void* ref_bvhgpu_from_bvh( void* bvh, int compact )
{
	BVH_GPU* g = new BVH_GPU();
	g->ConvertFrom( *(BVH*)bvh, compact != 0 );
	return g;
}
void ref_bvhgpu_destroy( void* h ) { delete (BVH_GPU*)h; }
uint32_t ref_bvhgpu_used_nodes( void* h ) { return ((BVH_GPU*)h)->usedNodes; }
const void* ref_bvhgpu_nodes( void* h ) { return ((BVH_GPU*)h)->bvhNode; }
void ref_bvhgpu_intersect( void* h, void* rays, uint64_t n, int threads )
{
	const BVH_GPU* b = (BVH_GPU*)h; Ray* r = (Ray*)rays;
	parallel_rays( n, threads, [=]( uint64_t s, uint64_t e ) { for (uint64_t i = s; i < e; i++) b->Intersect( r[i] ); } );
}

// ---------------------------------------------------------------- BVH8_CWBVH
// mode 0: BVH8_CWBVH::Build (BuildDefault = BuildAVX on x86), 1: BuildHQ,
// mode 2: conversion chain of BVH8_CWBVH::Build (:5827-5834) applied to the *scalar* BVH::Build tree.
void* ref_cwbvh_build( const float* verts, uint32_t primCount, int mode, int threaded )
{
	BVH8_CWBVH* c = new BVH8_CWBVH();
	const bvhvec4* v = (const bvhvec4*)verts;
	if (mode == 0) c->Build( v, primCount );
	else if (mode == 1) c->BuildHQ( v, primCount );
	else
	{
		c->bvh8.bvh.context = c->bvh8.context = c->context;
		c->bvh8.bvh.threadedBuild = threaded != 0;
		c->bvh8.bvh.Build( v, primCount );
		c->bvh8.bvh.Compact();
		c->bvh8.bvh.SplitLeafs( 3 );
		c->bvh8.ConvertFrom( c->bvh8.bvh, false );
		c->ConvertFrom( c->bvh8, true );
	}
	return c;
}
void ref_cwbvh_destroy( void* h ) { delete (BVH8_CWBVH*)h; }
uint32_t ref_cwbvh_used_blocks( void* h ) { return ((BVH8_CWBVH*)h)->usedBlocks; }
uint32_t ref_cwbvh_idx_count( void* h ) { return ((BVH8_CWBVH*)h)->idxCount; }
uint32_t ref_cwbvh_tri_count( void* h ) { return ((BVH8_CWBVH*)h)->triCount; }
const void* ref_cwbvh_nodes( void* h ) { return ((BVH8_CWBVH*)h)->bvh8Data; }
const void* ref_cwbvh_tris( void* h ) { return ((BVH8_CWBVH*)h)->bvh8Tris; }
// the BVH2 the CWBVH was collapsed from (after Compact + SplitLeafs), for conversion parity tests
void* ref_cwbvh_source_bvh( void* h ) { return &((BVH8_CWBVH*)h)->bvh8.bvh; }
void ref_cwbvh_intersect( void* h, void* rays, uint64_t n, int threads )
{
	const BVH8_CWBVH* b = (BVH8_CWBVH*)h; Ray* r = (Ray*)rays;
	parallel_rays( n, threads, [=]( uint64_t s, uint64_t e ) { for (uint64_t i = s; i < e; i++) b->Intersect( r[i] ); } );
}

// ---------------------------------------------------------------- BVH8_CPU (AVX2) - performance baseline only
void* ref_bvh8cpu_build( const float* verts, uint32_t primCount, int hq )
{
	BVH8_CPU* c = new BVH8_CPU();
	const bvhvec4* v = (const bvhvec4*)verts;
	if (hq) c->BuildHQ( v, primCount ); else c->Build( v, primCount );
	return c;
}
void ref_bvh8cpu_destroy( void* h ) { delete (BVH8_CPU*)h; }
void ref_bvh8cpu_intersect( void* h, void* rays, uint64_t n, int threads )
{
	const BVH8_CPU* b = (BVH8_CPU*)h; Ray* r = (Ray*)rays;
	parallel_rays( n, threads, [=]( uint64_t s, uint64_t e ) { for (uint64_t i = s; i < e; i++) b->Intersect( r[i] ); } );
}
void ref_bvh8cpu_occluded( void* h, const void* rays, uint64_t n, uint32_t* bits, int threads )
{
	const BVH8_CPU* b = (BVH8_CPU*)h; const Ray* r = (const Ray*)rays;
	std::vector<uint8_t> occ( n );
	uint8_t* o = occ.data();
	parallel_rays( n, threads, [=]( uint64_t s, uint64_t e ) { for (uint64_t i = s; i < e; i++) o[i] = b->IsOccluded( r[i] ) ? 1 : 0; } );
	for (uint64_t i = 0; i < n; i++) if (o[i]) bits[i >> 5] |= 1u << (i & 31);
}

} // extern "C"
