// tinybvh_b200/csrc/mesh_overlap.cu - intersecting triangle pairs between two meshes and within one mesh (tbvh_mesh_overlap_pairs /
// tbvh_mesh_overlap_bits): one walk of B's BVH2 per triangle of A with the closed box test, and a pair test of orientation predicates
// only.  DESIGN.md 4.12 states the rules; tests/tritri_oracle.c restates them on the host in the same fp32 operation order.
//
// Pairs, on one stream: k_mesh_overlap<COUNT> (pairs per triangle of A), an exclusive scan, one host synchronisation for the raw total,
// k_mesh_overlap<FILL> ((i << 32) | j keys at the scanned offsets), a radix sort, DeviceSelect::Unique, and k_overlap_out, which writes
// the first min( unique, capacity ) pairs.  Bits: k_mesh_overlap<BITS>, one launch.
#include "common.cuh"
#include "../../include/tinybvh_b200_device/closest_walk.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <algorithm>

#define MO_MAX_KEYS (1ull << 31) // raw pairs a pairs call sorts at most (16 GiB of keys and their sort buffer)

namespace
{
using tbvh::cp_dot;
using tbvh::cp_cross;

enum { MO_COUNT = 0, MO_FILL = 1, MO_BITS = 2 };

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

// The pair test of triangles a and b (three corners each), DESIGN.md 4.12; SELF applies the self rules of shared corners.
template <bool SELF> __device__ __forceinline__ bool mo_test( const V3* a, const V3* b )
{
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
} // namespace

// One thread per triangle i of A in 128-thread CTAs: the box of its corners against B's child-pair nodes (the root's box untested), and
// every reference of every reached leaf through the pair test; SELF: B is A and the pairs passes keep j > i, the bits pass j != i.
// COUNT: counts[i] = the pairs found (a reference reached on several paths counts once per path); FILL: their keys (i << 32) | j from
// offsets[i] on, in the same order; BITS: one bit per triangle (store_occlusion_word), the walk ends at the first pair.  STACKN as
// k_closest_point.
template <int MODE, bool SELF, int STACKN>
__global__ void __launch_bounds__( 128 ) k_mesh_overlap( const float4* __restrict__ nodes, const float4* __restrict__ tris, const float4* __restrict__ vb,
	const float4* __restrict__ va, const uint64_t n, const uint32_t root_ref, const uint32_t root_count, uint64_t* __restrict__ counts,
	const uint64_t* __restrict__ offsets, uint64_t* __restrict__ keys, uint32_t* __restrict__ bits )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	bool hit = false;
	if (i < n)
	{
		V3 t[3];
		#pragma unroll
		for (int c = 0; c < 3; c++) t[c] = mo_corner( va, i * 3 + c );
		const V3 mn{ fminf( fminf( t[0].x, t[1].x ), t[2].x ), fminf( fminf( t[0].y, t[1].y ), t[2].y ), fminf( fminf( t[0].z, t[1].z ), t[2].z ) };
		const V3 mx{ fmaxf( fmaxf( t[0].x, t[1].x ), t[2].x ), fmaxf( fmaxf( t[0].y, t[1].y ), t[2].y ), fmaxf( fmaxf( t[0].z, t[1].z ), t[2].z ) };
		uint2 stack[STACKN];
		int sp = 0;
		uint32_t ref = root_ref, cnt = root_count;
		uint64_t found = 0, o = MODE == MO_FILL ? offsets[i] : 0;
		while (true)
		{
			if (cnt == 0)
			{
				const float4* q = nodes + (size_t)ref * 2;
				const float4 a0 = __ldg( q ), a1 = __ldg( q + 1 ), b0 = __ldg( q + 2 ), b1 = __ldg( q + 3 );
				const bool ha = mo_box( mn, mx, a0, a1 ), hb = mo_box( mn, mx, b0, b1 );
				const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w ), refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
				if (ha && hb) { stack[sp++] = make_uint2( refb, cntb ); ref = refa, cnt = cnta; continue; }
				if (ha) { ref = refa, cnt = cnta; continue; }
				if (hb) { ref = refb, cnt = cntb; continue; }
			}
			else
			{
				for (uint32_t k = 0; k < cnt && !hit; k++)
				{
					const uint32_t j = __float_as_uint( __ldg( &tris[(size_t)(ref + k) * 3].w ) );
					if (SELF && (MODE == MO_BITS ? j == i : j <= i)) continue;
					const V3 u[3] = { mo_corner( vb, (size_t)j * 3 ), mo_corner( vb, (size_t)j * 3 + 1 ), mo_corner( vb, (size_t)j * 3 + 2 ) };
					if (!mo_test<SELF>( t, u )) continue;
					if (MODE == MO_BITS) hit = true;
					else if (MODE == MO_FILL) keys[o++] = (i << 32) | j;
					else found++;
				}
				if (hit) break;
			}
			if (sp == 0) break;
			const uint2 e = stack[--sp];
			ref = e.x, cnt = e.y;
		}
		if (MODE == MO_COUNT) counts[i] = found;
	}
	if (MODE == MO_BITS) store_occlusion_word( bits, i, n, hit );
}

// keys (i << 32) | j -> pairs [i, j] for the first min( *num, cap ) keys
__global__ void k_overlap_out( const uint64_t* __restrict__ keys, const int64_t* __restrict__ num, const uint64_t cap, uint32_t* __restrict__ pairs )
{
	const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= cap || k >= (uint64_t)*num) return;
	const uint64_t x = keys[k];
	pairs[k * 2] = (uint32_t)(x >> 32), pairs[k * 2 + 1] = (uint32_t)x;
}

static int mo_launch( int mode, tbvh_bvh a, tbvh_bvh b, uint64_t* counts, const uint64_t* offsets, uint64_t* keys, uint32_t* bits, cudaStream_t s )
{
	const uint64_t n = a->info.prim_count;
	const uint32_t grid = (uint32_t)((n + 127) / 128);
	const bool self = a == b, deep = b->info.max_depth + 1 > TBVH_STACK;
	#define MO_ARGS <<<grid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, b->d_verts, a->d_verts, n, b->root_ref, b->root_count, counts, offsets, keys, bits )
	#define MO_MODE( M, D ) do { if (self) k_mesh_overlap<M, true, D> MO_ARGS; else k_mesh_overlap<M, false, D> MO_ARGS; } while (0)
	#define MO_DEPTH( D ) do { if (mode == MO_COUNT) MO_MODE( MO_COUNT, D ); else if (mode == MO_FILL) MO_MODE( MO_FILL, D ); else MO_MODE( MO_BITS, D ); } while (0)
	if (deep) MO_DEPTH( TBVH_STACK_DEEP ); else MO_DEPTH( TBVH_STACK );
	#undef MO_DEPTH
	#undef MO_MODE
	#undef MO_ARGS
	LAUNCHED();
	return TBVH_OK;
}

// every refusal before any launch, in the documented order; align: the device alignment of out
static int mo_check( const char* fn, tbvh_bvh a, tbvh_bvh b, const void* out, bool out_needed, uint64_t* count, bool need_count, int space, uintptr_t align )
{
	if (!a || !b || (out_needed && !out) || (need_count && !count)) { tbvh_set_error( "%s: NULL argument", fn ); return TBVH_E_ARG; }
	if (space != TBVH_HOST && space != TBVH_DEVICE) { tbvh_set_error( "%s: unknown space %d", fn, space ); return TBVH_E_ARG; }
	if (space == TBVH_DEVICE && ((uintptr_t)out & (align - 1))) { tbvh_set_error( "%s: the device output must be %u-byte aligned", fn, (unsigned)align ); return TBVH_E_ARG; }
	if (a->ctx != b->ctx) { tbvh_set_error( "%s: the two handles belong to different contexts", fn ); return TBVH_E_ARG; }
	if (a->d_inst || b->d_inst) { tbvh_set_error( "%s: overlap queries on a TLAS are not supported", fn ); return TBVH_E_UNSUPPORTED; }
	for (tbvh_bvh h : { a, b })
		if (!h->trav() || !h->d_leaf_tris || !h->d_verts) { tbvh_set_error( "%s: no BVH-layout tree on a handle", fn ); return TBVH_E_STATE; }
	if (b->info.max_depth + 1 > TBVH_STACK_DEEP) { tbvh_set_error( "%s: BVH depth %u exceeds the %d-entry traversal stack", fn, b->info.max_depth, TBVH_STACK_DEEP ); return TBVH_E_LIMIT; }
	return TBVH_OK;
}

extern "C" {

int tbvh_mesh_overlap_pairs( tbvh_bvh a, tbvh_bvh b, uint32_t* pairs, uint64_t capacity, uint64_t* count, int space, void* stream )
{
	TRY( mo_check( __func__, a, b, pairs, capacity > 0, count, true, space, 8 ) );
	CUDA_TRY( cudaSetDevice( a->ctx->device ) );
	const uint64_t n = a->info.prim_count;
	if (n == 0) { *count = 0; return TBVH_OK; }
	// the pipeline runs on the engine stream (CUB's launches are counted by capture, which the legacy default stream does not allow),
	// behind everything queued on the caller's stream so far
	Scratch sc( a->ctx->stream );
	const cudaStream_t s = sc.s;
	if (space == TBVH_DEVICE)
	{
		TRY( sc.events() );
		CUDA_TRY( cudaEventRecord( sc.e0, (cudaStream_t)stream ) );
		CUDA_TRY( cudaStreamWaitEvent( s, sc.e0, 0 ) );
	}
	uint64_t* cnt = 0, * off = 0, * h = 0;
	TRY( sc.alloc( cnt, (n + 1) * 8 ) );
	TRY( sc.alloc( off, (n + 1) * 8 ) );
	TRY( sc.alloc_host( h, 16 ) );
	size_t tb = 0;
	CUDA_TRY( cub::DeviceScan::ExclusiveSum( (void*)0, tb, cnt, off, (int64_t)(n + 1), s ) );
	void* temp = 0;
	TRY( sc.alloc( temp, std::max( tb, (size_t)16 ) ) );
	CUDA_TRY( cudaMemsetAsync( cnt + n, 0, 8, s ) );
	TRY( mo_launch( MO_COUNT, a, b, cnt, 0, 0, 0, s ) );
	TRY( sort_enqueue( s, [&]() { return cub::DeviceScan::ExclusiveSum( temp, tb, cnt, off, (int64_t)(n + 1), s ); } ) );
	CUDA_TRY( cudaMemcpyAsync( h, off + n, 8, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	const uint64_t raw = h[0];
	if (raw > MO_MAX_KEYS)
	{
		*count = raw;
		tbvh_set_error( "%s: %llu raw pairs exceed the %llu a call sorts", __func__, (unsigned long long)raw, MO_MAX_KEYS );
		return TBVH_E_LIMIT;
	}
	if (raw == 0) { *count = 0; return TBVH_OK; }
	uint64_t* keys[2] = {};
	int64_t* num = 0;
	uint32_t* out = pairs;
	const uint64_t m = std::min( raw, capacity );
	TRY( sc.alloc( keys[0], raw * 8 ) );
	TRY( sc.alloc( keys[1], raw * 8 ) );
	TRY( sc.alloc( num, 8 ) );
	if (space == TBVH_HOST && m) TRY( sc.alloc( out, m * 8 ) );
	// the sort needs the bits of i and all 32 of j
	int end_bit = 32;
	while (end_bit < 64 && (n - 1) >> (end_bit - 32)) end_bit++;
	size_t tb2 = 0, tb3 = 0;
	CUDA_TRY( cub::DeviceRadixSort::SortKeys( (void*)0, tb2, keys[0], keys[1], (int64_t)raw, 0, end_bit, s ) );
	CUDA_TRY( cub::DeviceSelect::Unique( (void*)0, tb3, keys[1], keys[0], num, (int64_t)raw, s ) );
	void* temp2 = 0;
	TRY( sc.alloc( temp2, std::max( tb2, tb3 ) ) );
	tb2 = tb3 = std::max( tb2, tb3 );
	TRY( mo_launch( MO_FILL, a, b, 0, off, keys[0], 0, s ) );
	TRY( sort_enqueue( s, [&]() { return cub::DeviceRadixSort::SortKeys( temp2, tb2, keys[0], keys[1], (int64_t)raw, 0, end_bit, s ); } ) );
	TRY( sort_enqueue( s, [&]() { return cub::DeviceSelect::Unique( temp2, tb3, keys[1], keys[0], num, (int64_t)raw, s ); } ) );
	if (m)
	{
		k_overlap_out<<<(uint32_t)((m + 255) / 256), 256, 0, s>>>( keys[0], num, m, out );
		LAUNCHED();
	}
	CUDA_TRY( cudaMemcpyAsync( h + 1, num, 8, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	const uint64_t unique = h[1], w = std::min( unique, capacity );
	if (space == TBVH_HOST && w)
	{
		CUDA_TRY( cudaMemcpyAsync( pairs, out, w * 8, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
	}
	*count = unique;
	return TBVH_OK;
}

int tbvh_mesh_overlap_bits( tbvh_bvh a, tbvh_bvh b, uint32_t* bits, int space, void* stream )
{
	TRY( mo_check( __func__, a, b, bits, true, 0, false, space, 4 ) );
	CUDA_TRY( cudaSetDevice( a->ctx->device ) );
	const uint64_t n = a->info.prim_count;
	if (n == 0) return TBVH_OK;
	if (space == TBVH_DEVICE) return mo_launch( MO_BITS, a, b, 0, 0, 0, bits, (cudaStream_t)stream );
	const size_t bytes = ((n + 31) / 32) * 4;
	Scratch sc( a->ctx->stream );
	uint32_t* d_bits = 0;
	TRY( sc.alloc( d_bits, bytes ) );
	TRY( mo_launch( MO_BITS, a, b, 0, 0, 0, d_bits, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( bits, d_bits, bytes, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaStreamSynchronize( sc.s ) );
	return TBVH_OK;
}

} // extern "C"
