// tinybvh_b200/csrc/mesh_distance.cu - distances between meshes (tbvh_mesh_distance / tbvh_mesh_distance_pairs): the nearest triangle of
// mesh B for every triangle of mesh A, and every pair within a distance, over B's BVH2 with the path bound of the proximity walk and the
// triangle-triangle distance tt_dist2.  DESIGN.md 4.13 states the rules; tests/meshdist_oracle.c restates them on the host in the same fp32
// operation order.
//
// Nearest: k_mesh_distance<NEAREST>, one launch.  Pairs: k_mesh_distance<COUNT>, k_mesh_distance<FILL> and the pipeline of
// tbvh_mesh_overlap_pairs (mesh_pairs_run).
#include "tri_pair.cuh"

namespace
{
enum { MD_NEAREST = 0, MD_COUNT = 1, MD_FILL = 2 };

struct MdRec { float d; uint32_t j; }; // the 8-byte result record of one triangle of A

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

// One thread per triangle i of A in 128-thread CTAs; B's BVH2 walked as cp_walk walks it, with the box-box bound of i's box against each
// node box as the path bound and the value of a reference (leaf, j) = max( tt_dist2, LBtri, P( leaf ) ) (DESIGN.md 4.13).  SELF: B is A,
// j != i and the two share no corner (values equal as the weld rule), and the pairs passes keep j > i.  NEAREST: best starts at r2 and
// falls to the smallest ( value, j ); results[i] = { sqrt( best ), j }, or { r_max, 0xffffffff } when nothing is found or i is not finite.
// COUNT / FILL: best stays r2 and every reference with value <= r2 is counted / written as (i << 32) | j from offsets[i] on, in the same
// order.  STACKN as k_closest_point.
template <int MODE, bool SELF, int STACKN>
__global__ void __launch_bounds__( 128 ) k_mesh_distance( const float4* __restrict__ nodes, const float4* __restrict__ tris, const float4* __restrict__ vb,
	const float4* __restrict__ va, const uint64_t n, const uint32_t root_ref, const uint32_t root_count, const float r_max, MdRec* __restrict__ results,
	uint64_t* __restrict__ counts, const uint64_t* __restrict__ offsets, uint64_t* __restrict__ keys )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	V3 t[3];
	#pragma unroll
	for (int c = 0; c < 3; c++) t[c] = mo_corner( va, i * 3 + c );
	const float r2 = __fmul_rn( r_max, r_max );
	float best = r2;
	uint32_t bj = tbvh::CP_NO_PRIM;
	uint64_t found = 0, o = MODE == MD_FILL ? offsets[i] : 0;
	if (md_finite3( t ))
	{
		const V3 mn{ fminf( fminf( t[0].x, t[1].x ), t[2].x ), fminf( fminf( t[0].y, t[1].y ), t[2].y ), fminf( fminf( t[0].z, t[1].z ), t[2].z ) };
		const V3 mx{ fmaxf( fmaxf( t[0].x, t[1].x ), t[2].x ), fmaxf( fmaxf( t[0].y, t[1].y ), t[2].y ), fmaxf( fmaxf( t[0].z, t[1].z ), t[2].z ) };
		tbvh::CpEntry stack[STACKN];
		int sp = 0;
		uint32_t ref = root_ref, cnt = root_count;
		float P = 0.0f;
		while (true)
		{
			if (cnt == 0)
			{
				const float4* q = nodes + (size_t)ref * 2;
				const float4 a0 = __ldg( q ), a1 = __ldg( q + 1 ), b0 = __ldg( q + 2 ), b1 = __ldg( q + 3 );
				const float Pa = fmaxf( md_node_bound( mn, mx, a0, a1 ), P ), Pb = fmaxf( md_node_bound( mn, mx, b0, b1 ), P );
				const bool ha = !(Pa > best), hb = !(Pb > best);
				const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w ), refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
				if (ha && hb)
				{
					const bool swp = Pb < Pa; // nearer child first, the left one on ties
					ref = swp ? refb : refa, cnt = swp ? cntb : cnta, P = swp ? Pb : Pa;
					stack[sp++] = swp ? tbvh::CpEntry{ refa, cnta, Pa } : tbvh::CpEntry{ refb, cntb, Pb };
					continue;
				}
				if (ha) { ref = refa, cnt = cnta, P = Pa; continue; }
				if (hb) { ref = refb, cnt = cntb, P = Pb; continue; }
			}
			else
			{
				for (uint32_t k = 0; k < cnt; k++)
				{
					const uint32_t j = __float_as_uint( __ldg( &tris[(size_t)(ref + k) * 3].w ) );
					if (SELF && (MODE == MD_NEAREST ? j == i : j <= i)) continue;
					const V3 u[3] = { mo_corner( vb, (size_t)j * 3 ), mo_corner( vb, (size_t)j * 3 + 1 ), mo_corner( vb, (size_t)j * 3 + 2 ) };
					// the box-box bound of the two triangles first: a reference it puts above best is skipped without the pair distance
					const float lb = fmaxf( md_box_bound( mn, mx, fminf( fminf( u[0].x, u[1].x ), u[2].x ), fminf( fminf( u[0].y, u[1].y ), u[2].y ),
						fminf( fminf( u[0].z, u[1].z ), u[2].z ), fmaxf( fmaxf( u[0].x, u[1].x ), u[2].x ), fmaxf( fmaxf( u[0].y, u[1].y ), u[2].y ),
						fmaxf( fmaxf( u[0].z, u[1].z ), u[2].z ) ), P );
					if (lb > best || !md_finite3( u )) continue;
					if (SELF)
					{
						bool shared = false;
						#pragma unroll
						for (int x = 0; x < 3; x++)
							#pragma unroll
							for (int y = 0; y < 3; y++) shared |= mo_eq( t[x], u[y] );
						if (shared) continue;
					}
					const float v = fmaxf( tt_dist2( t, u ), lb );
					if (MODE == MD_NEAREST) { if (v < best || (v == best && j < bj)) best = v, bj = j; }
					else if (v <= best)
					{
						if (MODE == MD_FILL) keys[o++] = (i << 32) | j;
						else found++;
					}
				}
			}
			// pop, pruning again against the current best
			bool popped = false;
			while (sp > 0)
			{
				const tbvh::CpEntry e = stack[--sp];
				if (!(e.P > best)) { ref = e.ref, cnt = e.cnt, P = e.P, popped = true; break; }
			}
			if (!popped) break;
		}
	}
	if (MODE == MD_COUNT) counts[i] = found;
	if (MODE == MD_NEAREST) results[i] = bj == tbvh::CP_NO_PRIM ? MdRec{ r_max, bj } : MdRec{ __fsqrt_rn( best ), bj };
}

static int md_launch( int mode, tbvh_bvh a, tbvh_bvh b, float r, MdRec* results, uint64_t* counts, const uint64_t* offsets, uint64_t* keys, cudaStream_t s )
{
	const uint64_t n = a->info.prim_count;
	const uint32_t grid = (uint32_t)((n + 127) / 128);
	const bool self = a == b, deep = b->info.max_depth + 1 > TBVH_STACK;
	#define MD_ARGS <<<grid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, b->d_verts, a->d_verts, n, b->root_ref, b->root_count, r, results, counts, offsets, keys )
	#define MD_MODE( M, D ) do { if (self) k_mesh_distance<M, true, D> MD_ARGS; else k_mesh_distance<M, false, D> MD_ARGS; } while (0)
	#define MD_DEPTH( D ) do { if (mode == MD_NEAREST) MD_MODE( MD_NEAREST, D ); else if (mode == MD_COUNT) MD_MODE( MD_COUNT, D ); else MD_MODE( MD_FILL, D ); } while (0)
	if (deep) MD_DEPTH( TBVH_STACK_DEEP ); else MD_DEPTH( TBVH_STACK );
	#undef MD_DEPTH
	#undef MD_MODE
	#undef MD_ARGS
	LAUNCHED();
	return TBVH_OK;
}

// the distance argument: r >= 0, +inf allowed (NaN and negative refused)
static int md_check_r( const char* fn, const float r )
{
	if (!(r >= 0.0f)) { tbvh_set_error( "%s: the distance must be >= 0 (+inf allowed), not %g", fn, (double)r ); return TBVH_E_ARG; }
	return TBVH_OK;
}

extern "C" {

int tbvh_mesh_distance( tbvh_bvh a, tbvh_bvh b, float r_max, void* results, int space, void* stream )
{
	TRY( md_check_r( __func__, r_max ) );
	TRY( mo_check( __func__, a, b, results, true, 0, false, space, 8 ) );
	CUDA_TRY( cudaSetDevice( a->ctx->device ) );
	const uint64_t n = a->info.prim_count;
	if (n == 0) return TBVH_OK;
	if (space == TBVH_DEVICE) return md_launch( MD_NEAREST, a, b, r_max, (MdRec*)results, 0, 0, 0, (cudaStream_t)stream );
	Scratch sc( a->ctx->stream );
	MdRec* d_out = 0;
	TRY( sc.alloc( d_out, n * 8 ) );
	TRY( md_launch( MD_NEAREST, a, b, r_max, d_out, 0, 0, 0, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( results, d_out, n * 8, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaStreamSynchronize( sc.s ) );
	return TBVH_OK;
}

int tbvh_mesh_distance_pairs( tbvh_bvh a, tbvh_bvh b, float r, uint32_t* pairs, uint64_t capacity, uint64_t* count, int space, void* stream )
{
	TRY( md_check_r( __func__, r ) );
	TRY( mo_check( __func__, a, b, pairs, capacity > 0, count, true, space, 8 ) );
	return mesh_pairs_run( __func__, a, pairs, capacity, count, space, stream,
		[&]( bool fill, uint64_t* counts, const uint64_t* offsets, uint64_t* keys, cudaStream_t s ) { return md_launch( fill ? MD_FILL : MD_COUNT, a, b, r, 0, counts, offsets, keys, s ); } );
}

} // extern "C"
