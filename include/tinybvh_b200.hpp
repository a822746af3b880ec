// include/tinybvh_b200.hpp - header-only C++ shim that keeps tinybvh's class / method names over the C-ABI
// (include/tinybvh_b200.h -> libtinybvh_b200.so).  Host code that today calls
//     tinybvh::BVH::Build( tris, N )            tiny_bvh.h:2124      tinybvh::BVH::Intersect( ray )    :3222
//     tinybvh::BVH::IsOccluded( ray )           :3382                tinybvh::BVH_GPU::ConvertFrom     :4612
//     tinybvh::BVH8_CWBVH::Build / ConvertFrom  :5822 / :5884
// switches namespaces (tinybvh -> tinybvh_b200) and, for throughput, calls the batch overloads
//     Intersect( Ray* rays, n )   /   IsOccluded( const Ray* rays, n, uint32_t* bits )
// instead of per-ray loops (the reference has no batch entry point; its GPU "batch" is an OpenCL kernel launch,
// tiny_bvh_speedtest.cpp:1092-1241).  The shim does not include tiny_bvh.h: vertex and ray arguments are templates
// over any 16-byte-stride vertex type and any 64-/128-byte ray record with the reference's field offsets, so
// tinybvh::bvhvec4 / tinybvh::Ray work unchanged.  Error behaviour is the reference's: message on stderr, exit(1)
// (BVH_FATAL_ERROR, tiny_bvh.h:1617-1620).  There is no CPU fallback.
#pragma once
#include "tinybvh_b200.h"
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <array>
#include <vector>

namespace tinybvh_b200 {

#define TBVH_FATAL_IF( rc, where ) do { if ((rc) != TBVH_OK) { fprintf( stderr, "Fatal error in tinybvh_b200 %s: %s\n", where, tbvh_last_error() ); exit( 1 ); } } while (0)

// Layout-compatible stand-in for tinybvh::Ray (tiny_bvh.h:688-709) for programs that do not include the reference.
struct alignas( 64 ) Ray
{
	float O[3]; uint32_t mask = 0xFFFF;
	float D[3]; uint32_t instIdx = 0;
	float rD[3]; uint32_t pad = 0;
	float t = 1e30f, u = 0, v = 0; uint32_t prim = 0; // Intersection hit
	unsigned char aux[64];
	Ray() = default;
	Ray( const float* origin, const float* direction, float tmax = 1e30f )
	{
		memset( this, 0, sizeof( Ray ) );
		const float l = sqrtf( direction[0] * direction[0] + direction[1] * direction[1] + direction[2] * direction[2] ), rl = l == 0 ? 0 : 1.0f / l;
		for (int a = 0; a < 3; a++)
		{
			O[a] = origin[a], D[a] = direction[a] * rl;
			rD[a] = (D[a] > 1e-12f || D[a] < -1e-12f) ? 1.0f / D[a] : (D[a] >= 0 ? 1e30f : -1e30f); // tinybvh_safercp :442
		}
		t = tmax, mask = 0xFFFF;
	}
};
static_assert( sizeof( Ray ) == 128, "host ray record is 128 bytes" );

inline tbvh_ctx context( int device = -1 )
{
	// one context per device; device from TINYBVH_B200_DEVICE (the reference API has no place for a device index)
	static tbvh_ctx ctx[16] = {};
	if (device < 0) { const char* e = getenv( "TINYBVH_B200_DEVICE" ); device = e ? atoi( e ) : 0; }
	if (device < 0 || device >= 16) device = 0;
	if (!ctx[device]) TBVH_FATAL_IF( tbvh_ctx_create( device, &ctx[device] ), "context()" );
	return ctx[device];
}

// pinned allocation for ray batches (replaces tinybvh::malloc64 for buffers that cross PCIe)
inline void* malloc_pinned( size_t bytes ) { void* p = 0; TBVH_FATAL_IF( tbvh_host_alloc( bytes, &p ), "malloc_pinned" ); return p; }
inline void free_pinned( void* p ) { tbvh_host_free( p ); }

// Many meshes in one call (tbvh_build_batch): objs[i] ends up as if its own Build( vertices[i], primCounts[i] ) had run - the tree,
// Refit and Optimize working from the caller's arrays, the public counters.  flavour: TBVH_BUILD_REFERENCE (BVH::Build),
// TBVH_BUILD_AVX or TBVH_BUILD_PLOC (BuildPLOC, not in the reference); by default the builder the class's own Build uses.  TBVH_BUILD_HQ: each object as its own BuildHQ( vertices[i],
// primCounts[i] ) leaves it (tbvh_build_batch_hq).  BVH_GPU / BVH8_CWBVH objects are converted afterwards.
template <class T, class Vec4> void BuildBatch( T* const* objs, const Vec4* const* vertices, const uint32_t* primCounts, uint32_t count, int flavour = -1 );
// Many refits in one call (tbvh_refit_batch), as an animated scene refits its BLASes every frame: every object refitted from the vertex
// array it was built from, exactly as its own Refit() would leave it - the tree and the public counters.
class BVH;
void RefitBatch( BVH* const* objs, uint32_t count );

class BVHBase
{
public:
	float c_trav = 1, c_int = 1;   // BVHBase::c_trav / c_int (tiny_bvh.h:819-820)
	uint32_t usedNodes = 0, triCount = 0, idxCount = 0;
	float aabbMin[3] = { 0, 0, 0 }, aabbMax[3] = { 0, 0, 0 };
	double buildMs = 0;            // device time of the last Build
	tbvh_bvh handle() const { return h; }
	int Layout() const { return layout; }  // TBVH_LAYOUT_*: the layout Intersect / IsOccluded walk (BVHBase::layout, tiny_bvh.h:795-805)
	tbvh_info Info() const { tbvh_info i; TBVH_FATAL_IF( tbvh_bvh_info( h, &i ), "Info" ); return i; }
	// tbvh_optimize: rounds of parallel subtree reinsertion on the device that lower the resident tree's SAH cost - indexed and
	// device-resident builds included.  Not the reference's BVH::Optimize (tiny_bvh.h:3043), which BVH::Optimize below still runs
	// on the host.  A BVH_GPU or BVH8_CWBVH converts the optimised tree again, as its Build does.  Returns the rounds kept.
	uint32_t OptimizeOnDevice( const uint32_t maxRounds = 8 )
	{
		uint32_t rounds = 0;
		TBVH_FATAL_IF( tbvh_optimize( h, maxRounds, c_trav, c_int, &rounds, 0 ), "OptimizeOnDevice" );
		if (rounds && layout != TBVH_LAYOUT_BVH) TBVH_FATAL_IF( tbvh_convert( h, layout ), "OptimizeOnDevice" );
		sync_info();
		return rounds;
	}
	// batch traversal: the calls the patched harness makes instead of its per-ray loops
	// Return value: 0, or - with collectCost set - the sum over the batch of what the reference's per-ray Intersect returns,
	// (int32_t)( c_trav * nodes visited + c_int * triangles tested ) (tiny_bvh.h:3303; the speedtest adds these up into rayCost,
	// tiny_bvh_speedtest.cpp:197-214).  Exact for integral c_trav / c_int (the defaults); the counting kernels are slower.
	bool collectCost = false;
	template <class RayT> int64_t Intersect( RayT* rays, uint64_t n ) const
	{
		static_assert( sizeof( RayT ) == 64 || sizeof( RayT ) == 128, "ray record must be the 64- or 128-byte layout" );
		if (collectCost) TBVH_FATAL_IF( tbvh_set_stats( h, 1 ), "Intersect" );
		TBVH_FATAL_IF( tbvh_intersect( h, layout, rays, (uint32_t)sizeof( RayT ), n ), "Intersect" );
		if (!collectCost) return 0;
		uint64_t steps = 0, tris = 0;
		TBVH_FATAL_IF( tbvh_get_stats( h, &steps, &tris ), "Intersect" );
		TBVH_FATAL_IF( tbvh_set_stats( h, 0 ), "Intersect" );
		return (int64_t)(c_trav * (double)steps + c_int * (double)tris);
	}
	// batch traversal with packed results: hits[i] = { t, u, v, prim } (16 bytes), rays untouched - the fast return path
	template <class RayT> void Intersect( const RayT* rays, uint64_t n, void* hits16 ) const
	{
		TBVH_FATAL_IF( tbvh_intersect_packed( h, layout, rays, (uint32_t)sizeof( RayT ), n, hits16 ), "Intersect (packed)" );
	}
	template <class RayT> void IsOccluded( const RayT* rays, uint64_t n, uint32_t* bits ) const
	{
		TBVH_FATAL_IF( tbvh_occluded( h, layout, rays, (uint32_t)sizeof( RayT ), n, bits ), "IsOccluded" );
	}
	// device-resident batches (the reference's GPU section keeps its rays in a tinyocl::Buffer and times the kernel alone,
	// tiny_bvh_speedtest.cpp:1110-1135): 64-byte records made by UploadRays, hits written in place, asynchronous until Sync()
	template <class RayT> void* UploadRays( const RayT* rays, uint64_t n ) const
	{
		void* d = 0;
		TBVH_FATAL_IF( tbvh_device_alloc( context(), n * 64, &d ), "UploadRays" );
		TBVH_FATAL_IF( tbvh_copy_rays_to_device( rays, (uint32_t)sizeof( RayT ), n, d, 0 ), "UploadRays" );
		Sync();
		return d;
	}
	// the view a kernel of the caller's passes to tbvh::intersect_* / isoccluded_* (include/tinybvh_b200_device.cuh); take a new one per frame
	tbvh_view DeviceView() const { tbvh_view v; TBVH_FATAL_IF( tbvh_device_view( h, layout, &v ), "DeviceView" ); return v; }
	void IntersectDevice( void* d_rays64, uint64_t n ) const { TBVH_FATAL_IF( tbvh_intersect_device( h, layout, d_rays64, 64, 0, n, 0 ), "IntersectDevice" ); }
	void IsOccludedDevice( const void* d_rays64, uint64_t n, uint32_t* d_bits ) const { TBVH_FATAL_IF( tbvh_occluded_device( h, layout, d_rays64, 64, d_bits, n, 0 ), "IsOccludedDevice" ); }
	// t,u,v,prim of n device records back into host Ray records
	template <class RayT> void DownloadHits( RayT* rays, const void* d_rays64, uint64_t n ) const
	{
		char* tmp = (char*)malloc( n * 64 );
		TBVH_FATAL_IF( tbvh_copy_from_device( tmp, d_rays64, n * 64 ), "DownloadHits" );
		for (uint64_t i = 0; i < n; i++) memcpy( (char*)&rays[i] + 48, tmp + i * 64 + 48, 16 );
		free( tmp );
	}
	void FreeDevice( void* d ) const { tbvh_device_free( context(), d ); }
	void Sync() const { TBVH_FATAL_IF( tbvh_device_sync( context() ), "Sync" ); }
	// per-ray forms with the reference's signatures (correct, but one PCIe round trip each: use the batch forms)
	template <class RayT> int32_t Intersect( RayT& ray ) const { return (int32_t)Intersect( &ray, 1 ); }
	template <class RayT> bool IsOccluded( const RayT& ray ) const { uint32_t b = 0; IsOccluded( &ray, 1, &b ); return b & 1; }
	// multi-hit rays over the BVH-layout tree (tbvh_intersect_all): hits16 + i * k * 16 holds ray i's k nearest distinct hits { t, u, v,
	// prim }, nearest first, slots past the count { tmax, 0, 0, 0xffffffff }; counts[i] = the triangles it crosses, saturated at k + 1
	template <class RayT> void IntersectAll( const RayT* rays, uint64_t n, uint32_t k, void* hits16, uint32_t* counts ) const
	{
		static_assert( sizeof( RayT ) == 64 || sizeof( RayT ) == 128, "ray record must be the 64- or 128-byte layout" );
		TBVH_FATAL_IF( tbvh_intersect_all( h, rays, (uint32_t)sizeof( RayT ), n, k, hits16, counts, TBVH_HOST, 0 ), "IntersectAll" );
	}
	// the same over a TLAS (tbvh_intersect_all_tlas): hits16 as above with prim the BLAS's own triangle, insts + i * k the k instances
	// (0xffffffff past the count)
	template <class RayT> void IntersectAll( const RayT* rays, uint64_t n, uint32_t k, void* hits16, uint32_t* insts, uint32_t* counts ) const
	{
		static_assert( sizeof( RayT ) == 64 || sizeof( RayT ) == 128, "ray record must be the 64- or 128-byte layout" );
		TBVH_FATAL_IF( tbvh_intersect_all_tlas( h, rays, (uint32_t)sizeof( RayT ), n, k, hits16, insts, counts, TBVH_HOST, 0 ), "IntersectAll (TLAS)" );
	}
	// proximity queries over the BVH-layout tree (tbvh_closest_point / tbvh_sphere_overlap), host batches of 16-byte { x, y, z, r }
	// records (bvhvec4 or any float4-like type).  ClosestPoint: results16[i] = { d, u, v, prim } of the nearest triangle within r, the
	// point v0 + u (v1 - v0) + v (v2 - v0); { r, 0, 0, 0xffffffff } when none.  IntersectSphere: bit i of bits = some triangle lies within r.
	template <class Vec4> void ClosestPoint( const Vec4* q, uint64_t n, void* results16 ) const
	{
		static_assert( sizeof( Vec4 ) == 16, "queries are 16-byte { x, y, z, r } records" );
		TBVH_FATAL_IF( tbvh_closest_point( h, q, results16, n, TBVH_HOST, 0 ), "ClosestPoint" );
	}
	template <class Vec4> void IntersectSphere( const Vec4* q, uint64_t n, uint32_t* bits ) const
	{
		static_assert( sizeof( Vec4 ) == 16, "queries are 16-byte { x, y, z, r } records" );
		TBVH_FATAL_IF( tbvh_sphere_overlap( h, q, bits, n, TBVH_HOST, 0 ), "IntersectSphere" );
	}
	// sphere casts (tbvh_sphere_cast / tbvh_sphere_cast_occluded), host batches of 32-byte { cx, cy, cz, r, dx, dy, dz, tmax } records: the
	// sphere's centre moves along c + t D, t in [0, tmax].  SphereCast: results16[i] = { t, u, v, prim } of the first triangle it touches,
	// at the point v0 + u (v1 - v0) + v (v2 - v0); { tmax, 0, 0, 0xffffffff } when none.  SphereCastOccluded: bit i of bits = it touches one.
	template <class Query> void SphereCast( const Query* q, uint64_t n, void* results16 ) const
	{
		static_assert( sizeof( Query ) == 32, "queries are 32-byte { cx, cy, cz, r, dx, dy, dz, tmax } records" );
		TBVH_FATAL_IF( tbvh_sphere_cast( h, q, results16, n, TBVH_HOST, 0 ), "SphereCast" );
	}
	template <class Query> void SphereCastOccluded( const Query* q, uint64_t n, uint32_t* bits ) const
	{
		static_assert( sizeof( Query ) == 32, "queries are 32-byte { cx, cy, cz, r, dx, dy, dz, tmax } records" );
		TBVH_FATAL_IF( tbvh_sphere_cast_occluded( h, q, bits, n, TBVH_HOST, 0 ), "SphereCastOccluded" );
	}
	// signed distances (tbvh_signed_distance_prepare / tbvh_signed_distance): PrepareSignedDistance builds the pseudonormal table once per
	// tree and vertex set (again after any rebuild or refit); SignedDistance: results16[i] = { sd, u, v, prim }, ClosestPoint's record with
	// the distance negative inside a closed, outward-oriented mesh.
	void PrepareSignedDistance() { TBVH_FATAL_IF( tbvh_signed_distance_prepare( h ), "PrepareSignedDistance" ); }
	template <class Vec4> void SignedDistance( const Vec4* q, uint64_t n, void* results16 ) const
	{
		static_assert( sizeof( Vec4 ) == 16, "queries are 16-byte { x, y, z, r } records" );
		TBVH_FATAL_IF( tbvh_signed_distance( h, q, results16, n, TBVH_HOST, 0 ), "SignedDistance" );
	}
	// generalized winding numbers (tbvh_winding_number_prepare / tbvh_winding_number): PrepareWindingNumber builds the moment table once
	// per tree and vertex set (again after any rebuild or refit); WindingNumber: w[i] = the winding number at q[i] (its w ignored), 1 inside
	// and 0 outside a closed, outward-oriented mesh, also meaningful on open and self-intersecting ones; beta = INFINITY: the exact sum.
	void PrepareWindingNumber() { TBVH_FATAL_IF( tbvh_winding_number_prepare( h ), "PrepareWindingNumber" ); }
	template <class Vec4> void WindingNumber( const Vec4* q, uint64_t n, float* w, float beta = 2.0f ) const
	{
		static_assert( sizeof( Vec4 ) == 16, "queries are 16-byte { x, y, z, ignored } records" );
		TBVH_FATAL_IF( tbvh_winding_number( h, q, w, n, beta, TBVH_HOST, 0 ), "WindingNumber" );
	}
	// intersecting triangle pairs (tbvh_mesh_overlap_pairs / tbvh_mesh_overlap_bits, DESIGN.md 4.12), both meshes' vertices in one space.
	// OverlapPairs: every (i, j), i a triangle of this mesh and j of other, that intersect, sorted by (i, j); SelfIntersections: the pairs
	// i < j of this mesh that intersect, apart from neighbours that only share corners or an edge; OverlapBits( other, bits ): bit i of
	// (triCount + 31) / 32 words = triangle i intersects some triangle of other (other = *this: some other triangle of this mesh).
	void OverlapPairs( const BVHBase& other, std::vector<std::array<uint32_t, 2>>& pairs ) const
	{
		uint64_t count = 0;
		pairs.resize( Info().prim_count );
		TBVH_FATAL_IF( tbvh_mesh_overlap_pairs( h, other.h, pairs.empty() ? 0 : pairs[0].data(), pairs.size(), &count, TBVH_HOST, 0 ), "OverlapPairs" );
		if (count > pairs.size())
		{
			pairs.resize( count );
			TBVH_FATAL_IF( tbvh_mesh_overlap_pairs( h, other.h, pairs[0].data(), pairs.size(), &count, TBVH_HOST, 0 ), "OverlapPairs" );
		}
		pairs.resize( count );
	}
	void SelfIntersections( std::vector<std::array<uint32_t, 2>>& pairs ) const { OverlapPairs( *this, pairs ); }
	void OverlapBits( const BVHBase& other, uint32_t* bits ) const { TBVH_FATAL_IF( tbvh_mesh_overlap_bits( h, other.h, bits, TBVH_HOST, 0 ), "OverlapBits" ); }
	// distances between meshes (tbvh_mesh_distance / tbvh_mesh_distance_pairs, DESIGN.md 4.13), both meshes' vertices in one space.
	// NearestTriangles: results8[i] = { float d, uint32 j } of the nearest triangle j of other within r_max of triangle i (r_max = INFINITY:
	// unbounded), { r_max, 0xffffffff } when none; other = *this: the nearest triangle sharing no corner.  DistancePairs: every (i, j) within
	// distance r, sorted by (i, j) (other = *this: i < j, sharing no corner).
	void NearestTriangles( const BVHBase& other, const float r_max, void* results8 ) const
	{
		TBVH_FATAL_IF( tbvh_mesh_distance( h, other.h, r_max, results8, TBVH_HOST, 0 ), "NearestTriangles" );
	}
	void DistancePairs( const BVHBase& other, const float r, std::vector<std::array<uint32_t, 2>>& pairs ) const
	{
		uint64_t count = 0;
		pairs.resize( Info().prim_count );
		TBVH_FATAL_IF( tbvh_mesh_distance_pairs( h, other.h, r, pairs.empty() ? 0 : pairs[0].data(), pairs.size(), &count, TBVH_HOST, 0 ), "DistancePairs" );
		if (count > pairs.size())
		{
			pairs.resize( count );
			TBVH_FATAL_IF( tbvh_mesh_distance_pairs( h, other.h, r, pairs[0].data(), pairs.size(), &count, TBVH_HOST, 0 ), "DistancePairs" );
		}
		pairs.resize( count );
	}
	// times of impact between moving meshes (tbvh_mesh_toi / tbvh_mesh_toi_pairs, DESIGN.md 4.15): every vertex moves linearly from the
	// handle's vertices to the host end frames `end` / `other_end` (16-byte rows, the same triangles; other = *this: pass end twice).
	// TimeOfImpact: results16[i] = { float t, float d, uint32 j, uint32 iters } of the first triangle j of other within eta + xi of triangle i
	// during the step, { inf, inf, 0xffffffff, 0 } when none.  ImpactPairs: every (i, j) in contact within the step, sorted by (i, j), and
	// each pair's contact time.
	template <class Vec4> void TimeOfImpact( const Vec4* end, const BVHBase& other, const Vec4* other_end, const float eta, const float xi,
		const uint32_t max_iters, void* results16 ) const
	{
		TBVH_FATAL_IF( tbvh_mesh_toi( h, end, sizeof( Vec4 ), other.h, other_end, sizeof( Vec4 ), eta, xi, max_iters, results16, TBVH_HOST, 0 ), "TimeOfImpact" );
	}
	template <class Vec4> void ImpactPairs( const Vec4* end, const BVHBase& other, const Vec4* other_end, const float eta, const float xi,
		const uint32_t max_iters, std::vector<std::array<uint32_t, 2>>& pairs, std::vector<float>& times ) const
	{
		uint64_t count = 0;
		pairs.resize( Info().prim_count ), times.resize( pairs.size() );
		TBVH_FATAL_IF( tbvh_mesh_toi_pairs( h, end, sizeof( Vec4 ), other.h, other_end, sizeof( Vec4 ), eta, xi, max_iters, pairs.empty() ? 0 : pairs[0].data(),
			times.empty() ? 0 : times.data(), pairs.size(), &count, TBVH_HOST, 0 ), "ImpactPairs" );
		if (count > pairs.size())
		{
			pairs.resize( count ), times.resize( count );
			TBVH_FATAL_IF( tbvh_mesh_toi_pairs( h, end, sizeof( Vec4 ), other.h, other_end, sizeof( Vec4 ), eta, xi, max_iters, pairs[0].data(), times.data(),
				pairs.size(), &count, TBVH_HOST, 0 ), "ImpactPairs" );
		}
		pairs.resize( count ), times.resize( count );
	}
	// BVH::IntersectSphere( pos, r ) tiny_bvh.h:3140 with its signature, one query (a PCIe round trip: batch where you can).  It answers
	// under this library's definition (DESIGN.md 4.9: some triangle within r by exact closest-point distance), not the reference's
	// separating-axis test, which may decide otherwise where the sphere only touches a triangle.
	template <class Vec3> bool IntersectSphere( const Vec3& pos, const float r ) const
	{
		const float q[4] = { pos.x, pos.y, pos.z, r };
		uint32_t bits = 0;
		TBVH_FATAL_IF( tbvh_sphere_overlap( h, q, &bits, 1, TBVH_HOST, 0 ), "IntersectSphere" );
		return bits & 1;
	}
protected:
	BVHBase( int l ) : layout( l ) { TBVH_FATAL_IF( tbvh_bvh_create( context(), &h ), "BVHBase" ); }
	~BVHBase() { if (own) tbvh_bvh_destroy( h ); }
	BVHBase( const BVHBase& ) = delete;
	BVHBase& operator=( const BVHBase& ) = delete;
	void sync_info()
	{
		const tbvh_info i = Info();
		usedNodes = layout == TBVH_LAYOUT_BVH_GPU ? i.used_nodes_gpu : i.used_nodes, triCount = i.prim_count, idxCount = i.idx_count, buildMs = i.build_ms;
		memcpy( aabbMin, i.aabb_min, 12 ), memcpy( aabbMax, i.aabb_max, 12 );
	}
	// the ( vertices, indices, primCount ) overloads (tiny_bvh.h:889-900, 1111-1117, 1145-1150): the reference takes no vertex
	// count there, so it is derived from the largest index; returns that count
	template <class Vec4> uint32_t build_indexed( const Vec4* vertices, const uint32_t* indices, const uint32_t primCount, const int flavour, const char* what )
	{
		uint32_t vmax = 0;
		for (size_t i = 0; i < (size_t)primCount * 3; i++) vmax = indices[i] > vmax ? indices[i] : vmax;
		TBVH_FATAL_IF( tbvh_build_indexed( h, vertices, (uint32_t)sizeof( Vec4 ), vmax + 1, indices, primCount, TBVH_HOST, c_trav, c_int, flavour ), what );
		return vmax + 1;
	}
	static void batch_convert( tbvh_bvh*, uint32_t ) {} // BuildBatch: layouts converted for the whole batch at once (BVH8_CWBVH)
	void adopt( const BVHBase& o ) { if (own) tbvh_bvh_destroy( h ); h = o.h, own = false; } // "both must be kept alive" (README.md:99)
	tbvh_bvh h = 0;
	int layout;
	bool own = true;
	friend class BVH_GPU;
	friend class BVH8_CWBVH;
	template <class T, class Vec4> friend void BuildBatch( T* const*, const Vec4* const*, const uint32_t*, uint32_t, int );
};

class BVH : public BVHBase
{
public:
	static constexpr int defaultFlavour = TBVH_BUILD_REFERENCE; // BVH::Build
	BVH() : BVHBase( TBVH_LAYOUT_BVH ) {}
	// BVH::Build( const bvhvec4* vertices, uint32_t primCount ) tiny_bvh.h:2124 - binned SAH on the GPU
	template <class Vec4> void Build( const Vec4* vertices, const uint32_t primCount )
	{
		TBVH_FATAL_IF( tbvh_build( h, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST, c_trav, c_int ), "BVH::Build" );
		remember( vertices, (uint32_t)sizeof( Vec4 ), 0, primCount ), sync_info();
	}
	// BVH::BuildAVX( const bvhvec4*, uint32_t ) tiny_bvh.h:6400 - the flavour BuildDefault picks on x86
	template <class Vec4> void BuildAVX( const Vec4* vertices, const uint32_t primCount )
	{
		TBVH_FATAL_IF( tbvh_build_flavour( h, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST, c_trav, c_int, TBVH_BUILD_AVX ), "BVH::BuildAVX" );
		remember( vertices, (uint32_t)sizeof( Vec4 ), 0, primCount ), sync_info();
	}
	// BVH::Refit( nodeIdx = 0 ) tiny_bvh.h:3055 - the caller moved the vertices in the array it built from; like the reference the
	// shim kept the pointer (BVHBase::verts, "we're not copying this data" :2055), the engine receives the new positions.  Indexed
	// geometry: the vertex array itself, read on the device through the indices the engine kept from the build (vertIdx, :806-807)
	void Refit( const uint32_t = 0 )
	{
		const tbvh_mesh m = refit_mesh( "BVH::Refit" );
		tbvh_bvh hb = h;
		TBVH_FATAL_IF( m.vert_count ? tbvh_refit_batch_indexed( &hb, &m, 1, TBVH_HOST, 0 ) : tbvh_refit( h, m.verts, m.stride, m.prim_count, TBVH_HOST ), "BVH::Refit" );
		sync_info();
	}
	// BVH::BuildHQ( const bvhvec4*, uint32_t ) tiny_bvh.h:2623 - SBVH (spatial splits), ends with Compact()
	template <class Vec4> void BuildHQ( const Vec4* vertices, const uint32_t primCount )
	{
		TBVH_FATAL_IF( tbvh_build_flavour( h, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST, c_trav, c_int, TBVH_BUILD_HQ ), "BVH::BuildHQ" );
		remember( vertices, (uint32_t)sizeof( Vec4 ), 0, primCount ), sync_info();
	}
	// TLAS: BVH::Build( BLASInstance* instances, instCount, BVHBase** blasses, blasCount ) tiny_bvh.h:2221.  Inst is the
	// reference's 192-byte tinybvh::BLASInstance.  As in the reference (:2245-2250) every instance is Update()d first - inverse
	// transform and world box, computed on the host bit-identically to BLASInstance::Update (:8386) - and written back.
	// Intersect / IsOccluded on the TLAS are then IntersectTLAS / IsOccludedTLAS; a hit carries hit.inst (INST_IDX_BITS == 32).
	// When EVERY BLAS is a BVH8_CWBVH object the BLASses are walked in that layout (the arrangement of the reference's GPU path,
	// traverse_tlas.cl:60-67 "GPU_STATIC"); otherwise in the BVH layout, which every BLAS built by this shim holds as well.
	template <class Inst> void Build( Inst* instances, const uint32_t instCount, BVHBase** blasses, const uint32_t blasCount )
	{
		static_assert( sizeof( Inst ) == 192, "tinybvh::BLASInstance is 192 bytes (tiny_bvh.h:1443)" );
#ifdef INST_IDX_BITS
		TBVH_FATAL_IF( tbvh_set_option( context(), "inst_idx_bits", INST_IDX_BITS ), "inst_idx_bits" ); // where a hit stores its instance (:114-119)
#endif
		tbvh_bvh* hs = (tbvh_bvh*)malloc( sizeof( tbvh_bvh ) * (blasCount ? blasCount : 1) );
		bool allWide = blasCount > 0;
		for (uint32_t k = 0; k < blasCount; k++) hs[k] = blasses[k]->handle(), allWide = allWide && blasses[k]->Layout() == TBVH_LAYOUT_CWBVH;
		layout = allWide ? TBVH_LAYOUT_CWBVH : TBVH_LAYOUT_BVH;
		for (uint32_t i = 0; i < instCount; i++) // instList[i].Update( blas ) :2247-2249, bit-identical to the reference's
		{
			uint32_t blasIdx;
			memcpy( &blasIdx, (const char*)&instances[i] + 140, 4 );
			TBVH_FATAL_IF( blasIdx >= blasCount || tbvh_instance_update( &instances[i], hs[blasIdx] ), "BLASInstance::Update" );
		}
		const int rc = tbvh_build_tlas( h, instances, (uint32_t)sizeof( Inst ), instCount, hs, blasCount, c_trav, c_int );
		free( hs );
		TBVH_FATAL_IF( rc, "BVH::Build( BLASInstance*, .. )" );
		sync_info();
	}
	// The same Build( BLASInstance*, .. ) for the frame of an animation - RefitBatch( .. ); tlas.BuildUpdated( inst, n, blas, m ); -
	// through tbvh_build_tlas_update: Update() runs on the device for the whole list and the records come back as above, bit for bit;
	// rebuilding a TLAS of the same instance and BLAS counts reuses its device tables.
	template <class Inst> void BuildUpdated( Inst* instances, const uint32_t instCount, BVHBase** blasses, const uint32_t blasCount )
	{
		static_assert( sizeof( Inst ) == 192, "tinybvh::BLASInstance is 192 bytes (tiny_bvh.h:1443)" );
#ifdef INST_IDX_BITS
		TBVH_FATAL_IF( tbvh_set_option( context(), "inst_idx_bits", INST_IDX_BITS ), "inst_idx_bits" );
#endif
		tbvh_bvh* hs = (tbvh_bvh*)malloc( sizeof( tbvh_bvh ) * (blasCount ? blasCount : 1) );
		bool allWide = blasCount > 0;
		for (uint32_t k = 0; k < blasCount; k++) hs[k] = blasses[k]->handle(), allWide = allWide && blasses[k]->Layout() == TBVH_LAYOUT_CWBVH;
		layout = allWide ? TBVH_LAYOUT_CWBVH : TBVH_LAYOUT_BVH;
		const int rc = tbvh_build_tlas_update( h, instances, (uint32_t)sizeof( Inst ), instCount, TBVH_HOST, hs, blasCount, c_trav, c_int );
		free( hs );
		TBVH_FATAL_IF( rc, "BVH::BuildUpdated( BLASInstance*, .. )" );
		sync_info();
	}
	// indexed geometry: BVH::Build / BuildAVX / BuildHQ( vertices, indices, primCount ) tiny_bvh.h:889-900
	template <class Vec4> void Build( const Vec4* vertices, const uint32_t* indices, const uint32_t primCount ) { const uint32_t n = build_indexed( vertices, indices, primCount, TBVH_BUILD_REFERENCE, "BVH::Build" ); remember( vertices, (uint32_t)sizeof( Vec4 ), indices, primCount, n ), sync_info(); }
	template <class Vec4> void BuildAVX( const Vec4* vertices, const uint32_t* indices, const uint32_t primCount ) { const uint32_t n = build_indexed( vertices, indices, primCount, TBVH_BUILD_AVX, "BVH::BuildAVX" ); remember( vertices, (uint32_t)sizeof( Vec4 ), indices, primCount, n ), sync_info(); }
	template <class Vec4> void BuildHQ( const Vec4* vertices, const uint32_t* indices, const uint32_t primCount ) { build_indexed( vertices, indices, primCount, TBVH_BUILD_HQ, "BVH::BuildHQ" ); sync_info(); }
	// not in the reference: the PLOC build (TBVH_BUILD_PLOC), a refittable tree for meshes rebuilt every few frames
	template <class Vec4> void BuildPLOC( const Vec4* vertices, const uint32_t primCount )
	{
		TBVH_FATAL_IF( tbvh_build_flavour( h, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST, c_trav, c_int, TBVH_BUILD_PLOC ), "BVH::BuildPLOC" );
		remember( vertices, (uint32_t)sizeof( Vec4 ), 0, primCount ), sync_info();
	}
	template <class Vec4> void BuildPLOC( const Vec4* vertices, const uint32_t* indices, const uint32_t primCount ) { const uint32_t n = build_indexed( vertices, indices, primCount, TBVH_BUILD_PLOC, "BVH::BuildPLOC" ); remember( vertices, (uint32_t)sizeof( Vec4 ), indices, primCount, n ), sync_info(); }
	// BVH::SAHCost( nodeIdx = 0 ) tiny_bvh.h:1889 - the reference's value, bit for bit
	float SAHCost( const uint32_t = 0 ) const { float c = 0; TBVH_FATAL_IF( tbvh_sah_cost( h, c_trav, c_int, &c ), "BVH::SAHCost" ); return c; }
	// consume / produce the reference's public arrays (bvhNode, primIdx: tiny_bvh.h:952-964)
	template <class Vec4> void Upload( const void* bvhNode, uint32_t used, const uint32_t* primIdx, uint32_t idxCnt, const Vec4* vertices, uint32_t primCount )
	{
		TBVH_FATAL_IF( tbvh_upload_bvh( h, bvhNode, used, primIdx, idxCnt, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST ), "BVH::Upload" );
		sync_info();
	}
	void Download( void* bvhNode, uint32_t* primIdx ) const { TBVH_FATAL_IF( tbvh_download_bvh( h, bvhNode, primIdx, TBVH_HOST ), "BVH::Download" ); }
#ifdef TINY_BVH_H_
	// BVH::Save / BVH::Load (tiny_bvh.h:1747-1799).  The reference's file is a version word, the triangle count, the C++ object
	// itself and the node / primIdx arrays, so the format is whatever the tiny_bvh.h the host program was compiled with says it is:
	// with that header included before this one, a GPU-built tree is handed to a tinybvh::BVH object and written / read by the
	// reference's own code - files are interchangeable with the reference's in both directions.
	// the arrays and counters of a tree in the reference's BVH layout -> a tinybvh::BVH object (no device involved: usable on its own)
	static void FillReference( tinybvh::BVH& out, const tbvh_info& i, const void* nodes32, const uint32_t* primIdx, const float c_trav, const float c_int,
		const void* vertsPtr, const uint32_t vertsPrims, const uint32_t vertsStride )
	{
		out.AlignedFree( out.bvhNode ), out.AlignedFree( out.primIdx );
		out.bvhNode = (tinybvh::BVH::BVHNode*)out.AlignedAlloc( (size_t)i.used_nodes * 32 );
		out.primIdx = (uint32_t*)out.AlignedAlloc( (size_t)i.idx_count * 4 );
		memcpy( out.bvhNode, nodes32, (size_t)i.used_nodes * 32 ), memcpy( out.primIdx, primIdx, (size_t)i.idx_count * 4 );
		out.allocatedNodes = out.usedNodes = i.used_nodes, out.triCount = i.prim_count, out.idxCount = i.idx_count;
		out.aabbMin = tinybvh::bvhvec3( i.aabb_min[0], i.aabb_min[1], i.aabb_min[2] ), out.aabbMax = tinybvh::bvhvec3( i.aabb_max[0], i.aabb_max[1], i.aabb_max[2] );
		out.c_trav = c_trav, out.c_int = c_int, out.may_have_holes = false, out.rebuildable = false; // no fragments on the host: not rebuildable
		out.refittable = i.idx_count == i.prim_count; // an SBVH cannot be refitted (:3027)
		if (vertsPtr) out.verts = tinybvh::bvhvec4slice{ (const tinybvh::bvhvec4*)vertsPtr, vertsPrims * 3, vertsStride };
	}
	void ToReference( tinybvh::BVH& out ) const // a CPU-side tinybvh::BVH holding the GPU-built tree (SAHCost, Save, ConvertFrom, Intersect ...)
	{
		const tbvh_info i = Info();
		void* nodes = malloc( (size_t)i.used_nodes * 32 );
		uint32_t* idx = (uint32_t*)malloc( (size_t)i.idx_count * 4 + 4 );
		Download( nodes, idx );
		FillReference( out, i, nodes, idx, c_trav, c_int, vertsPtr, vertsPrims, vertsStride );
		free( nodes ), free( idx );
	}
	// BVH::Optimize( iterations, extreme, stochastic ) tiny_bvh.h:3043 - the insertion-based optimiser (BVH_Verbose::Optimize :4338) is
	// sequential host code in the reference and stays exactly that: the GPU-built tree is handed to a tinybvh::BVH, the reference's own
	// Optimize runs on it, and the result is uploaded (derived layouts are dropped: ConvertFrom again, as in the reference).
	void Optimize( const uint32_t iterations = 25, bool extreme = false, bool stochastic = false )
	{
		if (!vertsPtr || vertIdx) { fprintf( stderr, "Fatal error in tinybvh_b200 BVH::Optimize: needs a tree built from a (non-indexed) host vertex array.\n" ); exit( 1 ); }
		tinybvh::BVH tmp;
		ToReference( tmp );
		tmp.Optimize( iterations, extreme, stochastic );
		TBVH_FATAL_IF( tbvh_upload_bvh( h, tmp.bvhNode, tmp.usedNodes, tmp.primIdx, tmp.idxCount, vertsPtr, vertsStride, vertsPrims, TBVH_HOST ), "BVH::Optimize" );
		sync_info();
	}
	void Save( const char* fileName ) const { tinybvh::BVH tmp; ToReference( tmp ); tmp.Save( fileName ); }
	template <class Vec4> bool Load( const char* fileName, const Vec4* vertices, const uint32_t primCount )
	{
		tinybvh::BVH tmp;
		if (!tmp.Load( fileName, (const tinybvh::bvhvec4*)vertices, primCount )) return false;
		Upload( tmp.bvhNode, tmp.usedNodes, tmp.primIdx, tmp.idxCount, vertices, primCount );
		remember( vertices, (uint32_t)sizeof( Vec4 ), 0, primCount );
		return true;
	}
#endif
private:
	template <class T, class Vec4> friend void BuildBatch( T* const*, const Vec4* const*, const uint32_t*, uint32_t, int );
	friend void RefitBatch( BVH* const*, uint32_t );
	void batch_built( const void* v, uint32_t stride, uint32_t prims ) { remember( v, stride, 0, prims ), sync_info(); }
	// the mesh a refit hands the engine (tbvh_refit_batch_indexed): the caller's array the object was built from - a flat triangle
	// soup, or the vertices of indexed geometry with their count, which the engine reads through the indices it kept
	tbvh_mesh refit_mesh( const char* what ) const
	{
		if (!vertsPtr) { fprintf( stderr, "Fatal error in tinybvh_b200 %s: nothing was built from a host vertex array.\n", what ); exit( 1 ); }
		tbvh_mesh m = {};
		m.verts = vertsPtr, m.stride = vertsStride, m.vert_count = vertIdx ? vertsCount : 0, m.prim_count = vertsPrims;
		return m;
	}
	void remember( const void* v, uint32_t stride, const uint32_t* idx, uint32_t prims, uint32_t nverts = 0 ) { vertsPtr = v, vertsStride = stride, vertIdx = idx, vertsPrims = prims, vertsCount = nverts; }
	const void* vertsPtr = 0; const uint32_t* vertIdx = 0; // BVHBase::verts / vertIdx (:806-807): pointers to the caller's arrays, for Refit
	uint32_t vertsStride = 16, vertsPrims = 0, vertsCount = 0; // vertsCount: vertices of an indexed build (the largest index + 1)
};

class BVH_GPU : public BVHBase
{
public:
	static constexpr int defaultFlavour = TBVH_BUILD_AVX; // BuildDefault on x86 (tiny_bvh.h:1817-1832)
	BVH_GPU() : BVHBase( TBVH_LAYOUT_BVH_GPU ) {}
	template <class Vec4> void Build( const Vec4* vertices, const uint32_t primCount )
	{
		// BVH_GPU::Build -> bvh.BuildDefault = BuildAVX on x86 (tiny_bvh.h:1817-1832)
		TBVH_FATAL_IF( tbvh_build_flavour( h, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST, c_trav, c_int, TBVH_BUILD_AVX ), "BVH_GPU::Build" );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_BVH_GPU ), "BVH_GPU::Build" );
		sync_info();
	}
	template <class Vec4> void Build( const Vec4* vertices, const uint32_t* indices, const uint32_t primCount ) // :4560
	{
		build_indexed( vertices, indices, primCount, TBVH_BUILD_AVX, "BVH_GPU::Build" );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_BVH_GPU ), "BVH_GPU::Build" );
		sync_info();
	}
	template <class Vec4> void BuildHQ( const Vec4* vertices, const uint32_t* indices, const uint32_t primCount ) // :4594
	{
		build_indexed( vertices, indices, primCount, TBVH_BUILD_HQ, "BVH_GPU::BuildHQ" );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_BVH_GPU ), "BVH_GPU::BuildHQ" );
		sync_info();
	}
	// not in the reference: the PLOC build (TBVH_BUILD_PLOC), then the conversion
	template <class Vec4> void BuildPLOC( const Vec4* vertices, const uint32_t primCount )
	{
		TBVH_FATAL_IF( tbvh_build_flavour( h, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST, c_trav, c_int, TBVH_BUILD_PLOC ), "BVH_GPU::BuildPLOC" );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_BVH_GPU ), "BVH_GPU::BuildPLOC" );
		sync_info();
	}
	// BVH_GPU::BuildHQ tiny_bvh.h:4588: bvh.BuildHQ, then ConvertFrom
	template <class Vec4> void BuildHQ( const Vec4* vertices, const uint32_t primCount )
	{
		TBVH_FATAL_IF( tbvh_build_flavour( h, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST, c_trav, c_int, TBVH_BUILD_HQ ), "BVH_GPU::BuildHQ" );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_BVH_GPU ), "BVH_GPU::BuildHQ" );
		sync_info();
	}
	// BVH_GPU::ConvertFrom( const BVH& ) tiny_bvh.h:4612 - shares the source's device data, like the reference
	void ConvertFrom( const BVH& original )
	{
		adopt( original );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_BVH_GPU ), "BVH_GPU::ConvertFrom" );
		sync_info();
	}
	void Download( void* bvhNode ) const { TBVH_FATAL_IF( tbvh_download_bvh_gpu( h, bvhNode, TBVH_HOST ), "BVH_GPU::Download" ); }
private:
	template <class T, class Vec4> friend void BuildBatch( T* const*, const Vec4* const*, const uint32_t*, uint32_t, int );
	void batch_built( const void*, uint32_t, uint32_t ) { TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_BVH_GPU ), "BuildBatch" ); sync_info(); }
};

class BVH8_CWBVH : public BVHBase
{
public:
	static constexpr int defaultFlavour = TBVH_BUILD_AVX; // BuildDefault on x86 (tiny_bvh.h:5830)
	BVH8_CWBVH() : BVHBase( TBVH_LAYOUT_CWBVH ) {}
	uint32_t usedBlocks = 0;
	template <class Vec4> void Build( const Vec4* vertices, const uint32_t primCount )
	{
		// BVH8_CWBVH::Build -> bvh8.bvh.BuildDefault = BuildAVX on x86 (tiny_bvh.h:5830)
		TBVH_FATAL_IF( tbvh_build_flavour( h, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST, c_trav, c_int, TBVH_BUILD_AVX ), "BVH8_CWBVH::Build" );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_CWBVH ), "BVH8_CWBVH::Build" );
		sync_info(), usedBlocks = Info().used_blocks;
	}
	template <class Vec4> void Build( const Vec4* vertices, const uint32_t* indices, const uint32_t primCount ) // :5836
	{
		build_indexed( vertices, indices, primCount, TBVH_BUILD_AVX, "BVH8_CWBVH::Build" );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_CWBVH ), "BVH8_CWBVH::Build" );
		sync_info(), usedBlocks = Info().used_blocks;
	}
	// not in the reference: the PLOC build (TBVH_BUILD_PLOC), then the conversion
	template <class Vec4> void BuildPLOC( const Vec4* vertices, const uint32_t primCount )
	{
		TBVH_FATAL_IF( tbvh_build_flavour( h, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST, c_trav, c_int, TBVH_BUILD_PLOC ), "BVH8_CWBVH::BuildPLOC" );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_CWBVH ), "BVH8_CWBVH::BuildPLOC" );
		sync_info(), usedBlocks = Info().used_blocks;
	}
	// BVH8_CWBVH::BuildHQ tiny_bvh.h:5859: bvh.BuildHQ, SplitLeafs(3), MBVH<8> collapse, CWBVH encode
	template <class Vec4> void BuildHQ( const Vec4* vertices, const uint32_t primCount )
	{
		TBVH_FATAL_IF( tbvh_build_flavour( h, vertices, (uint32_t)sizeof( Vec4 ), primCount, TBVH_HOST, c_trav, c_int, TBVH_BUILD_HQ ), "BVH8_CWBVH::BuildHQ" );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_CWBVH ), "BVH8_CWBVH::BuildHQ" );
		sync_info(), usedBlocks = Info().used_blocks;
	}
	void ConvertFrom( const BVH& original )
	{
		adopt( original );
		TBVH_FATAL_IF( tbvh_convert( h, TBVH_LAYOUT_CWBVH ), "BVH8_CWBVH::ConvertFrom" );
		sync_info(), usedBlocks = Info().used_blocks;
	}
	// consume CPU-built data: bvh8Data / bvh8Tris / usedBlocks / idxCount (tiny_bvh.h:1356-1359), as the speedtest
	// uploads them today (tiny_bvh_speedtest.cpp:1200-1208)
	void Upload( const void* bvh8Data, uint32_t blocks, const void* bvh8Tris, uint32_t triRecords )
	{
		TBVH_FATAL_IF( tbvh_upload_cwbvh( h, bvh8Data, blocks, bvh8Tris, triRecords, TBVH_HOST ), "BVH8_CWBVH::Upload" );
		usedBlocks = blocks, idxCount = triRecords;
	}
	void Download( void* bvh8Data, void* bvh8Tris ) const { TBVH_FATAL_IF( tbvh_download_cwbvh( h, bvh8Data, bvh8Tris, TBVH_HOST ), "BVH8_CWBVH::Download" ); }
#ifdef TINY_BVH_H_
	// BVH8_CWBVH::Save / Load (tiny_bvh.h:5786-5820), through the reference's own code (see BVH::Save above): caches written here
	// load in tools built on the reference (tmpl8/game.cpp:78-81) and the other way round.
	void ToReference( tinybvh::BVH8_CWBVH& out ) const
	{
		const tbvh_info i = Info();
		out.AlignedFree( out.bvh8Data ), out.AlignedFree( out.bvh8Tris );
		out.bvh8Data = (tinybvh::bvhvec4*)out.AlignedAlloc( (size_t)i.used_blocks * 16 );
		out.bvh8Tris = (tinybvh::bvhvec4*)out.AlignedAlloc( (size_t)i.cwbvh_tri_count * 4 * 16 ); // the reference sizes it 4 blocks per triangle (:5895)
		memset( out.bvh8Tris, 0, (size_t)i.cwbvh_tri_count * 4 * 16 );
		Download( out.bvh8Data, out.bvh8Tris );
		out.allocatedBlocks = out.usedBlocks = i.used_blocks;
		out.triCount = i.prim_count, out.idxCount = i.cwbvh_tri_count, out.usedNodes = i.used_blocks / 5;
		out.bvh8.triCount = i.prim_count, out.bvh8.idxCount = i.cwbvh_tri_count; // Save sizes the triangle block from bvh8.idxCount (:5796)
		out.aabbMin = tinybvh::bvhvec3( i.aabb_min[0], i.aabb_min[1], i.aabb_min[2] ), out.aabbMax = tinybvh::bvhvec3( i.aabb_max[0], i.aabb_max[1], i.aabb_max[2] );
		out.c_trav = c_trav, out.c_int = c_int, out.rebuildable = false, out.refittable = false;
	}
	void Save( const char* fileName ) const { tinybvh::BVH8_CWBVH tmp; ToReference( tmp ); tmp.Save( fileName ); }
	bool Load( const char* fileName, const uint32_t expectedTris )
	{
		tinybvh::BVH8_CWBVH tmp;
		if (!tmp.Load( fileName, expectedTris )) return false;
		Upload( tmp.bvh8Data, tmp.usedBlocks, tmp.bvh8Tris, tmp.idxCount );
		triCount = tmp.triCount;
		return true;
	}
#endif
private:
	template <class T, class Vec4> friend void BuildBatch( T* const*, const Vec4* const*, const uint32_t*, uint32_t, int );
	static void batch_convert( tbvh_bvh* hs, uint32_t count ) { TBVH_FATAL_IF( tbvh_convert_batch( hs, count, TBVH_LAYOUT_CWBVH ), "BuildBatch" ); }
	void batch_built( const void*, uint32_t, uint32_t ) { sync_info(), usedBlocks = Info().used_blocks; }
};

template <class T, class Vec4> void BuildBatch( T* const* objs, const Vec4* const* vertices, const uint32_t* primCounts, uint32_t count, int flavour )
{
	tbvh_bvh* hs = (tbvh_bvh*)malloc( sizeof( tbvh_bvh ) * (count ? count : 1) );
	tbvh_mesh* ms = (tbvh_mesh*)calloc( count ? count : 1, sizeof( tbvh_mesh ) );
	for (uint32_t k = 0; k < count; k++)
	{
		hs[k] = objs[k] ? objs[k]->handle() : 0;
		ms[k].verts = vertices[k], ms[k].stride = (uint32_t)sizeof( Vec4 ), ms[k].prim_count = primCounts[k];
	}
	const float ct = count && objs[0] ? objs[0]->c_trav : 1.0f, ci = count && objs[0] ? objs[0]->c_int : 1.0f;
	const int rc = flavour == TBVH_BUILD_HQ ? tbvh_build_batch_hq( hs, ms, count, TBVH_HOST, ct, ci )
		: tbvh_build_batch( hs, ms, count, TBVH_HOST, ct, ci, flavour < 0 ? T::defaultFlavour : flavour );
	free( ms );
	if (rc != TBVH_OK) free( hs );
	TBVH_FATAL_IF( rc, "BuildBatch" );
	T::batch_convert( hs, count );
	free( hs );
	for (uint32_t k = 0; k < count; k++) objs[k]->batch_built( vertices[k], (uint32_t)sizeof( Vec4 ), primCounts[k] );
}

inline void RefitBatch( BVH* const* objs, uint32_t count )
{
	tbvh_bvh* hs = (tbvh_bvh*)malloc( sizeof( tbvh_bvh ) * (count ? count : 1) );
	tbvh_mesh* ms = (tbvh_mesh*)calloc( count ? count : 1, sizeof( tbvh_mesh ) );
	for (uint32_t k = 0; k < count; k++)
	{
		hs[k] = objs[k] ? objs[k]->handle() : 0;
		if (objs[k]) ms[k] = objs[k]->refit_mesh( "RefitBatch" );
	}
	const int rc = tbvh_refit_batch_indexed( hs, ms, count, TBVH_HOST, 0 );
	free( ms ), free( hs );
	TBVH_FATAL_IF( rc, "RefitBatch" );
	for (uint32_t k = 0; k < count; k++) objs[k]->sync_info();
}

} // namespace tinybvh_b200

// A program that does NOT include tiny_bvh.h can keep writing tinybvh::BVH, tinybvh::BVH8_CWBVH, tinybvh::Ray ...:
//     #define TINYBVH_B200_AS_TINYBVH
//     #include "tinybvh_b200.hpp"
// (next to the real header the two namespaces live side by side, as in harness/speedtest_b200.patch)
#ifdef TINYBVH_B200_AS_TINYBVH
namespace tinybvh = tinybvh_b200;
#endif
