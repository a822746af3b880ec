// tinybvh_b200/csrc/tri_pair.cuh - the triangle-pair test tt_overlap of DESIGN.md 4.12 (mo_test: orientation predicates only, fp32 in a
// fixed order), the closed box test of a triangle's box against a node box, the pair distance tt_dist2 and box-box bound of 4.13, and the
// pairs pipeline shared by tbvh_mesh_overlap_pairs (mesh_overlap.cu), tbvh_mesh_distance_pairs (mesh_distance.cu) and
// tbvh_mesh_toi_pairs (mesh_toi.cu).  tests/tritri_oracle.c and tests/meshdist_oracle.c restate the pair functions on the host.
#pragma once
#include "common.cuh"
#include "../../include/tinybvh_b200_device/closest_walk.cuh"
#include <functional>

#define MO_MAX_KEYS (1ull << 31) // raw pairs a pairs call sorts at most (16 GiB of keys and their sort buffer)

namespace
{
using tbvh::cp_dot;
using tbvh::cp_cross;

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 v3sub( const V3& a, const V3& b ) { return V3{ __fsub_rn( a.x, b.x ), __fsub_rn( a.y, b.y ), __fsub_rn( a.z, b.z ) }; }
__device__ __forceinline__ V3 v3cross( const V3& a, const V3& b ) { V3 r; cp_cross( a.x, a.y, a.z, b.x, b.y, b.z, r.x, r.y, r.z ); return r; }
__device__ __forceinline__ float v3dot( const V3& a, const V3& b ) { return cp_dot( a.x, a.y, a.z, b.x, b.y, b.z ); }
__device__ __forceinline__ float v3c( const V3& a, const int k ) { return k == 0 ? a.x : k == 1 ? a.y : a.z; }
// ( x - o ) . n: the side of x against the plane through o with normal n
__device__ __forceinline__ float mo_side( const V3& x, const V3& o, const V3& n ) { return v3dot( v3sub( x, o ), n ); }
// [b - a, c - a, d - a]
__device__ __forceinline__ float mo_orient3d( const V3& a, const V3& b, const V3& c, const V3& d ) { return mo_side( d, a, v3cross( v3sub( b, a ), v3sub( c, a ) ) ); }
// ( b - a ) x ( c - a ) on the axes (i, j)
__device__ __forceinline__ float mo_orient2d( const V3& a, const V3& b, const V3& c, const int i, const int j )
{
	return __fsub_rn( __fmul_rn( __fsub_rn( v3c( b, i ), v3c( a, i ) ), __fsub_rn( v3c( c, j ), v3c( a, j ) ) ),
		__fmul_rn( __fsub_rn( v3c( b, j ), v3c( a, j ) ), __fsub_rn( v3c( c, i ), v3c( a, i ) ) ) );
}
// the projection that drops the axis of n's largest component (x when |nx| > |nz| and |nx| >= |ny|, else y when |ny| > |nz| and
// |ny| >= |nx|, else z)
__device__ __forceinline__ void mo_axes( const V3& n, int& i, int& j )
{
	const float ax = fabsf( n.x ), ay = fabsf( n.y ), az = fabsf( n.z );
	if (ax > az && ax >= ay) i = 1, j = 2;
	else if (ay > az && ay >= ax) i = 2, j = 0;
	else i = 0, j = 1;
}
__device__ __forceinline__ bool mo_same3( const float a, const float b, const float c ) { return (a > 0.0f && b > 0.0f && c > 0.0f) || (a < 0.0f && b < 0.0f && c < 0.0f); }
__device__ __forceinline__ bool mo_opp( const float s, const float x ) { return s > 0.0f ? x < 0.0f : s < 0.0f ? x > 0.0f : false; }
// the line through edge (a, b) of a triangle whose third corner is c has the points y[0 .. K) strictly on its far side
template <int K> __device__ __forceinline__ bool mo_sep2( const V3& a, const V3& b, const V3& c, const V3* y, const int i, const int j )
{
	const float s = mo_orient2d( a, b, c, i, j );
	#pragma unroll
	for (int t = 0; t < K; t++) if (!mo_opp( s, mo_orient2d( a, b, y[t], i, j ) )) return false;
	return true;
}
// the closed segment (a, b) meets the closed triangle X; sa / sb: the sides of a and b against X's plane, n: X's normal
__device__ __forceinline__ bool mo_seg_tri( const V3& a, const V3& b, const float sa, const float sb, const V3* X, const V3& n )
{
	if ((sa > 0.0f && sb > 0.0f) || (sa < 0.0f && sb < 0.0f)) return false;
	if (sa == 0.0f && sb == 0.0f)
	{
		int i, j;
		mo_axes( n, i, j );
		const V3 ab[2] = { a, b };
		#pragma unroll
		for (int e = 0; e < 3; e++) if (mo_sep2<2>( X[e], X[(e + 1) % 3], X[(e + 2) % 3], ab, i, j )) return false;
		return !mo_same3( mo_orient2d( a, b, X[0], i, j ), mo_orient2d( a, b, X[1], i, j ), mo_orient2d( a, b, X[2], i, j ) );
	}
	if (sa == 0.0f || sb == 0.0f)
	{
		// one end on the plane: the segment meets it there only, so that point against X in the projection
		int i, j;
		mo_axes( n, i, j );
		const V3 p[1] = { sa == 0.0f ? a : b };
		#pragma unroll
		for (int e = 0; e < 3; e++) if (mo_sep2<1>( X[e], X[(e + 1) % 3], X[(e + 2) % 3], p, i, j )) return false;
		return true;
	}
	const float o1 = mo_orient3d( a, b, X[0], X[1] ), o2 = mo_orient3d( a, b, X[1], X[2] ), o3 = mo_orient3d( a, b, X[2], X[0] );
	return (o1 >= 0.0f && o2 >= 0.0f && o3 >= 0.0f) || (o1 <= 0.0f && o2 <= 0.0f && o3 <= 0.0f);
}
__device__ __forceinline__ bool mo_finite( const float f ) { return fabsf( f ) <= 3.402823466e38f; }
__device__ __forceinline__ bool mo_eq( const V3& a, const V3& b ) { return a.x == b.x && a.y == b.y && a.z == b.z; }
// a corner read as x + 0: -0 becomes +0 and every other value keeps its bits
__device__ __forceinline__ V3 mo_pos( const V3& a ) { return V3{ __fadd_rn( a.x, 0.0f ), __fadd_rn( a.y, 0.0f ), __fadd_rn( a.z, 0.0f ) }; }

// The pair test of triangles a and b (three corners each), DESIGN.md 4.12; SELF applies the self rules of shared corners.  The corners are
// read as x + 0, so the canonical order and every step after it are those of the +0 twin: the result does not depend on the sign of zero.
template <bool SELF> __device__ __forceinline__ bool mo_test( const V3* a_in, const V3* b_in )
{
	const V3 a[3] = { mo_pos( a_in[0] ), mo_pos( a_in[1] ), mo_pos( a_in[2] ) }, b[3] = { mo_pos( b_in[0] ), mo_pos( b_in[1] ), mo_pos( b_in[2] ) };
	#pragma unroll
	for (int c = 0; c < 3; c++)
		if (!(mo_finite( a[c].x ) && mo_finite( a[c].y ) && mo_finite( a[c].z ) && mo_finite( b[c].x ) && mo_finite( b[c].y ) && mo_finite( b[c].z ))) return false;
	// the closed boxes of the input corners
	#pragma unroll
	for (int k = 0; k < 3; k++)
		if (fmaxf( fmaxf( v3c( a[0], k ), v3c( a[1], k ) ), v3c( a[2], k ) ) < fminf( fminf( v3c( b[0], k ), v3c( b[1], k ) ), v3c( b[2], k ) ) ||
			fmaxf( fmaxf( v3c( b[0], k ), v3c( b[1], k ) ), v3c( b[2], k ) ) < fminf( fminf( v3c( a[0], k ), v3c( a[1], k ) ), v3c( a[2], k ) )) return false;
	// canonical order: the triangle whose nine ordered keys are lexicographically smaller is T
	bool swap = false, done = false;
	#pragma unroll
	for (int k = 0; k < 9; k++)
	{
		const uint32_t ka = f2key( v3c( a[k / 3], k % 3 ) ), kb = f2key( v3c( b[k / 3], k % 3 ) );
		if (!done && ka != kb) swap = kb < ka, done = true;
	}
	const V3* rt = swap ? b : a, * ru = swap ? a : b;
	// T's v0 subtracted from all six corners, then the power of two of their largest magnitude
	V3 T[3], U[3];
	float m = 0.0f;
	#pragma unroll
	for (int c = 0; c < 3; c++)
	{
		T[c] = v3sub( rt[c], rt[0] );
		m = fmaxf( m, fabsf( T[c].x ) ), m = fmaxf( m, fabsf( T[c].y ) ), m = fmaxf( m, fabsf( T[c].z ) );
	}
	#pragma unroll
	for (int c = 0; c < 3; c++)
	{
		U[c] = v3sub( ru[c], rt[0] );
		m = fmaxf( m, fabsf( U[c].x ) ), m = fmaxf( m, fabsf( U[c].y ) ), m = fmaxf( m, fabsf( U[c].z ) );
	}
	float inv;
	const float s = tbvh::cp_pow2( m, inv );
	#pragma unroll
	for (int c = 0; c < 3; c++)
	{
		T[c] = V3{ __fmul_rn( T[c].x, s ), __fmul_rn( T[c].y, s ), __fmul_rn( T[c].z, s ) };
		U[c] = V3{ __fmul_rn( U[c].x, s ), __fmul_rn( U[c].y, s ), __fmul_rn( U[c].z, s ) };
	}
	const V3 nT = v3cross( v3sub( T[1], T[0] ), v3sub( T[2], T[0] ) ), nU = v3cross( v3sub( U[1], U[0] ), v3sub( U[2], U[0] ) );
	if ((nT.x == 0.0f && nT.y == 0.0f && nT.z == 0.0f) || (nU.x == 0.0f && nU.y == 0.0f && nU.z == 0.0f)) return false;
	float dU[3], dT[3];
	#pragma unroll
	for (int c = 0; c < 3; c++) dU[c] = mo_side( U[c], T[0], nT ), dT[c] = mo_side( T[c], U[0], nU );
	if (SELF)
	{
		// shared corners: equal positions as values (-0 equals +0, NaN equals nothing)
		int shared = 0, ta = 0, ub = 0, tm = 0, um = 0;
		#pragma unroll
		for (int x = 0; x < 3; x++)
		{
			bool found = false;
			#pragma unroll
			for (int y = 0; y < 3; y++)
				if (!found && mo_eq( rt[x], ru[y] ))
				{
					found = true, shared++, ta = x, ub = y;
					tm |= 1 << x, um |= 1 << y;
				}
		}
		if (shared == 3) return true;
		if (shared == 1)
			return mo_seg_tri( T[(ta + 1) % 3], T[(ta + 2) % 3], dT[(ta + 1) % 3], dT[(ta + 2) % 3], U, nU ) ||
				mo_seg_tri( U[(ub + 1) % 3], U[(ub + 2) % 3], dU[(ub + 1) % 3], dU[(ub + 2) % 3], T, nT );
		if (shared == 2)
		{
			#pragma unroll
			for (int c = 0; c < 3; c++) if (dU[c] != 0.0f || dT[c] != 0.0f) return false;
			const int t3 = (tm & 1) == 0 ? 0 : (tm & 2) == 0 ? 1 : 2, u3 = (um & 1) == 0 ? 0 : (um & 2) == 0 ? 1 : 2;
			int i, j;
			mo_axes( nT, i, j );
			const float s1 = mo_orient2d( T[(t3 + 1) % 3], T[(t3 + 2) % 3], T[t3], i, j ), s2 = mo_orient2d( T[(t3 + 1) % 3], T[(t3 + 2) % 3], U[u3], i, j );
			return (s1 > 0.0f && s2 > 0.0f) || (s1 < 0.0f && s2 < 0.0f);
		}
	}
	if (mo_same3( dU[0], dU[1], dU[2] ) || mo_same3( dT[0], dT[1], dT[2] )) return false;
	if (dU[0] == 0.0f && dU[1] == 0.0f && dU[2] == 0.0f)
	{
		// coplanar: separated exactly when the line of some edge of either triangle has the other strictly on its far side
		int i, j;
		mo_axes( nT, i, j );
		#pragma unroll
		for (int e = 0; e < 3; e++)
			if (mo_sep2<3>( T[e], T[(e + 1) % 3], T[(e + 2) % 3], U, i, j ) || mo_sep2<3>( U[e], U[(e + 1) % 3], U[(e + 2) % 3], T, i, j )) return false;
		return true;
	}
	// two closed triangles not in one plane meet exactly when an edge of one meets the other
	#pragma unroll
	for (int e = 0; e < 3; e++)
	{
		if (mo_seg_tri( T[e], T[(e + 1) % 3], dT[e], dT[(e + 1) % 3], U, nU )) return true;
		if (mo_seg_tri( U[e], U[(e + 1) % 3], dU[e], dU[(e + 1) % 3], T, nT )) return true;
	}
	return false;
}

__device__ __forceinline__ V3 mo_corner( const float4* __restrict__ v, const size_t k ) { const float4 c = __ldg( v + k ); return V3{ c.x, c.y, c.z }; }
// the closed box test in fp32 (a NaN bound fails it)
__device__ __forceinline__ bool mo_box( const V3& mn, const V3& mx, const float4& bmin, const float4& bmax )
{
	return bmin.x <= mx.x && mn.x <= bmax.x && bmin.y <= mx.y && mn.y <= bmax.y && bmin.z <= mx.z && mn.z <= bmax.z;
}

// ---- the pair distance of DESIGN.md 4.13 (mesh_distance.cu, mesh_toi.cu)
__device__ __forceinline__ float4 md_f4( const V3& a ) { return make_float4( a.x, a.y, a.z, 0.0f ); }

// the squared distance between a point and the triangle (v0, v1, v2): the 4.9 per-triangle function on (v0, v1 - v0, v2 - v0)
__device__ __forceinline__ float md_point( const V3& p, const V3& v0, const V3& v1, const V3& v2 )
{
	float u, v;
	return tbvh::cp_triangle( p.x, p.y, p.z, md_f4( v0 ), md_f4( v3sub( v1, v0 ) ), md_f4( v3sub( v2, v0 ) ), u, v );
}

// the edge-edge candidate of (p, p + d1) and (q, q + d2): |r + s d1 - t d2|^2, r = p - q, at the unclamped solution s = ((q - p) x d2) . n /
// |n|^2, t = ((q - p) x d1) . n / |n|^2, n = d1 x d2, when |n|^2 > 0 and s, t lie in [0, 1]; +inf (no candidate) otherwise.  The cross
// products keep s and t accurate on nearly parallel edges, where Ericson's a e - b b loses its digits.
__device__ __forceinline__ float md_edges( const V3& p, const V3& p1, const V3& q, const V3& q1 )
{
	const V3 d1 = v3sub( p1, p ), d2 = v3sub( q1, q ), r = v3sub( p, q ), w = v3sub( q, p );
	const V3 n = v3cross( d1, d2 );
	const float nn = v3dot( n, n );
	if (!(nn > 0.0f)) return __int_as_float( 0x7f800000 );
	const float s = __fdiv_rn( v3dot( v3cross( w, d2 ), n ), nn ), t = __fdiv_rn( v3dot( v3cross( w, d1 ), n ), nn );
	if (!(s >= 0.0f && s <= 1.0f && t >= 0.0f && t <= 1.0f)) return __int_as_float( 0x7f800000 );
	const V3 x{ __fsub_rn( __fmaf_rn( s, d1.x, r.x ), __fmul_rn( t, d2.x ) ), __fsub_rn( __fmaf_rn( s, d1.y, r.y ), __fmul_rn( t, d2.y ) ),
		__fsub_rn( __fmaf_rn( s, d1.z, r.z ), __fmul_rn( t, d2.z ) ) };
	return v3dot( x, x );
}

// the squared distance from p to the segment (q, q + d), d = q1 - q: the projection parameter clamped to [0, 1] (0 / 0 gives q)
__device__ __forceinline__ float md_seg( const V3& p, const V3& q, const V3& q1 )
{
	const V3 d = v3sub( q1, q ), r = v3sub( p, q );
	const float t = tbvh::cp_edge( v3dot( r, d ), v3dot( d, d ) );
	const V3 w{ __fsub_rn( r.x, __fmul_rn( t, d.x ) ), __fsub_rn( r.y, __fmul_rn( t, d.y ) ), __fsub_rn( r.z, __fmul_rn( t, d.z ) ) };
	return v3dot( w, w );
}

__device__ __forceinline__ bool md_finite3( const V3* a ) { return mo_finite( a[0].x ) && mo_finite( a[0].y ) && mo_finite( a[0].z ) &&
	mo_finite( a[1].x ) && mo_finite( a[1].y ) && mo_finite( a[1].z ) && mo_finite( a[2].x ) && mo_finite( a[2].y ) && mo_finite( a[2].z ); }

// tt_dist2( a, b ), DESIGN.md 4.13, of two finite triangles: 0 when tt_overlap holds, else the least of six vertex-triangle, nine
// edge-edge and eighteen vertex-edge candidates on the canonical, scaled corners, scaled back; the corners read as x + 0 as in mo_test
__device__ __forceinline__ float tt_dist2( const V3* a_in, const V3* b_in )
{
	const V3 a[3] = { mo_pos( a_in[0] ), mo_pos( a_in[1] ), mo_pos( a_in[2] ) }, b[3] = { mo_pos( b_in[0] ), mo_pos( b_in[1] ), mo_pos( b_in[2] ) };
	if (mo_test<false>( a, b )) return 0.0f;
	bool swap = false, done = false;
	#pragma unroll
	for (int k = 0; k < 9; k++)
	{
		const uint32_t ka = f2key( v3c( a[k / 3], k % 3 ) ), kb = f2key( v3c( b[k / 3], k % 3 ) );
		if (!done && ka != kb) swap = kb < ka, done = true;
	}
	const V3* rt = swap ? b : a, * ru = swap ? a : b;
	V3 T[3], U[3];
	float m = 0.0f;
	#pragma unroll
	for (int c = 0; c < 3; c++)
	{
		T[c] = v3sub( rt[c], rt[0] );
		m = fmaxf( m, fabsf( T[c].x ) ), m = fmaxf( m, fabsf( T[c].y ) ), m = fmaxf( m, fabsf( T[c].z ) );
	}
	#pragma unroll
	for (int c = 0; c < 3; c++)
	{
		U[c] = v3sub( ru[c], rt[0] );
		m = fmaxf( m, fabsf( U[c].x ) ), m = fmaxf( m, fabsf( U[c].y ) ), m = fmaxf( m, fabsf( U[c].z ) );
	}
	float inv;
	const float s = tbvh::cp_pow2( m, inv );
	#pragma unroll
	for (int c = 0; c < 3; c++)
	{
		T[c] = V3{ __fmul_rn( T[c].x, s ), __fmul_rn( T[c].y, s ), __fmul_rn( T[c].z, s ) };
		U[c] = V3{ __fmul_rn( U[c].x, s ), __fmul_rn( U[c].y, s ), __fmul_rn( U[c].z, s ) };
	}
	// U's corners against T, then T's against U, then the edges (T's edge k from corner k to k + 1) against U's
	float d = md_point( U[0], T[0], T[1], T[2] );
	d = fminf( d, md_point( U[1], T[0], T[1], T[2] ) );
	d = fminf( d, md_point( U[2], T[0], T[1], T[2] ) );
	d = fminf( d, md_point( T[0], U[0], U[1], U[2] ) );
	d = fminf( d, md_point( T[1], U[0], U[1], U[2] ) );
	d = fminf( d, md_point( T[2], U[0], U[1], U[2] ) );
	#pragma unroll
	for (int k = 0; k < 3; k++)
		#pragma unroll
		for (int l = 0; l < 3; l++) d = fminf( d, md_edges( T[k], T[(k + 1) % 3], U[l], U[(l + 1) % 3] ) );
	// every corner against every edge of the other: exact where the per-triangle function's regions misplace the point (an edge of zero
	// length), and the endpoint cases of the edge pairs
	#pragma unroll
	for (int k = 0; k < 3; k++)
		#pragma unroll
		for (int l = 0; l < 3; l++) d = fminf( fminf( d, md_seg( U[k], T[l], T[(l + 1) % 3] ) ), md_seg( T[k], U[l], U[(l + 1) % 3] ) );
	return __fmul_rn( __fmul_rn( d, inv ), inv );
}

// the box-box bound of the box [mn, mx] against [bmin, bmax]: per axis g = max( bmin - mx, mn - bmax, 0 ), then fma( gz, gz, fma( gy, gy,
// gx gx ) ); every step is monotone in both boxes
__device__ __forceinline__ float md_box_bound( const V3& mn, const V3& mx, const float bminx, const float bminy, const float bminz,
	const float bmaxx, const float bmaxy, const float bmaxz )
{
	const float gx = fmaxf( fmaxf( __fsub_rn( bminx, mx.x ), __fsub_rn( mn.x, bmaxx ) ), 0.0f );
	const float gy = fmaxf( fmaxf( __fsub_rn( bminy, mx.y ), __fsub_rn( mn.y, bmaxy ) ), 0.0f );
	const float gz = fmaxf( fmaxf( __fsub_rn( bminz, mx.z ), __fsub_rn( mn.z, bmaxz ) ), 0.0f );
	return __fmaf_rn( gz, gz, __fmaf_rn( gy, gy, __fmul_rn( gx, gx ) ) );
}
__device__ __forceinline__ float md_node_bound( const V3& mn, const V3& mx, const float4& bmin, const float4& bmax )
{
	return md_box_bound( mn, mx, bmin.x, bmin.y, bmin.z, bmax.x, bmax.y, bmax.z );
}
} // namespace

// Every refusal of a two-mesh query before any launch, in the documented order (DESIGN.md 4.12): TBVH_E_ARG (NULL arguments, unknown
// space, out misaligned to `align` in device space, handles of different contexts), TBVH_E_UNSUPPORTED (a TLAS), TBVH_E_STATE (no
// BVH-layout tree), TBVH_E_LIMIT (b's tree deeper than the deep stack).
int mo_check( const char* fn, tbvh_bvh a, tbvh_bvh b, const void* out, bool out_needed, uint64_t* count, bool need_count, int space, uintptr_t align );

// The pairs pipeline of one query of a against b, on the engine stream behind `stream`'s work so far in device space: launch( fill = false,
// counts ) writes the raw pairs per triangle of a, an exclusive scan, one host synchronisation for the raw total, launch( fill = true,
// offsets, keys ) writes the keys (i << 32) | j at the scanned offsets, a radix sort, DeviceSelect::Unique, and the first
// min( unique, capacity ) pairs out; *count = the unique pairs.  TBVH_E_LIMIT above MO_MAX_KEYS raw keys (*count = that raw total).
// The caller has run every refusal.  fn: the C-ABI name for error messages.
typedef std::function<int( bool fill, uint64_t* counts, const uint64_t* offsets, uint64_t* keys, cudaStream_t s )> PairsLaunch;
int mesh_pairs_run( const char* fn, tbvh_bvh a, uint32_t* pairs, uint64_t capacity, uint64_t* count, int space, void* stream, const PairsLaunch& launch );
