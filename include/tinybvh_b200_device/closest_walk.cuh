// include/tinybvh_b200_device/closest_walk.cuh - the proximity walk over the BVH2: nearest surface point and sphere overlap of a query
// point.  Shared by the library's kernel (closest_point.cu: k_closest_point) and the device functions of include/tinybvh_b200_device.cuh.
//
// Semantics are the engine's own (DESIGN.md 4.9), restated on the host by tests/closest_oracle.c in the same fp32 operation order:
//  * per triangle: Ericson's ClosestPtPointTriangle (Real-Time Collision Detection 5.1.5) on a = v0, ab = e1, ac = e2 of the leaf record,
//    as barycentric weights (u, v) of e1, e2; every fused pair is __fmaf_rn, every other operation an _rn intrinsic;
//  * per node: the box lower bound LB = |max( bmin - p, p - bmax, 0 )|^2 and the path bound P( child ) = fmaxf( LB( child ), P( parent ) ),
//    P( root ) = 0, so P never decreases down a path whether or not child boxes lie inside their parents; a leaf that an uploaded tree
//    reaches on several paths is walked once per path, so its references are worth their least value over those paths;
//  * a reference (leaf, triangle) is worth d2 = fmaxf( d2_raw, P( leaf ) ); the result is the smallest ( d2, prim ) with d2 <= r_max^2,
//    independent of the visiting order, so a node with P > best is pruned exactly.
#pragma once
#include "base.cuh"

namespace tbvh
{

constexpr uint32_t CP_NO_PRIM = 0xffffffffu; // the prim of a miss record

__device__ __forceinline__ float cp_dot( const float ax, const float ay, const float az, const float bx, const float by, const float bz )
{
	return __fmaf_rn( az, bz, __fmaf_rn( ay, by, __fmul_rn( ax, bx ) ) );
}
// x clamped to [0, 1]; NaN and -0 give +0 (selects, not fminf / fmaxf, so that no zero sign depends on the instruction)
__device__ __forceinline__ float cp_unit( const float x ) { const float y = x > 0.0f ? x : 0.0f; return y < 1.0f ? y : 1.0f; }
// the edge parameter num / den clamped to [0, 1]; 0 / 0 (a zero-length edge) gives 0, its start point
__device__ __forceinline__ float cp_edge( const float num, const float den ) { return cp_unit( __fdiv_rn( num, den ) ); }
// a x b, each component one difference of two rounded products
__device__ __forceinline__ void cp_cross( const float ax, const float ay, const float az, const float bx, const float by, const float bz, float& x, float& y, float& z )
{
	x = __fsub_rn( __fmul_rn( ay, bz ), __fmul_rn( az, by ) );
	y = __fsub_rn( __fmul_rn( az, bx ), __fmul_rn( ax, bz ) );
	z = __fsub_rn( __fmul_rn( ax, by ), __fmul_rn( ay, bx ) );
}
// |ap - (u e1 + v e2)|^2
__device__ __forceinline__ float cp_dist2( const float apx, const float apy, const float apz, const float4& e1, const float4& e2, const float u, const float v )
{
	const float dx = __fsub_rn( apx, __fmaf_rn( v, e2.x, __fmul_rn( u, e1.x ) ) );
	const float dy = __fsub_rn( apy, __fmaf_rn( v, e2.y, __fmul_rn( u, e1.y ) ) );
	const float dz = __fsub_rn( apz, __fmaf_rn( v, e2.z, __fmul_rn( u, e1.z ) ) );
	return __fmaf_rn( dz, dz, __fmaf_rn( dy, dy, __fmul_rn( dx, dx ) ) );
}

// The feature of the triangle a closest point lies on (DESIGN.md 4.10), decided by the branch and the clamp of cp_triangle_feature that
// produced (u, v), never by comparing floats afterwards: the face, a vertex (v0, v1, v2) or an edge (AB = v0v1, AC = v0v2, BC = v1v2).
// The values index a signed-distance table record (signed_distance.cu): face normal, three vertex and three edge pseudonormals.
enum CpFeature : uint32_t { CP_FACE = 0, CP_V0 = 1, CP_V1 = 2, CP_V2 = 3, CP_AB = 4, CP_AC = 5, CP_BC = 6 };
// an edge from vertex a to vertex b at the clamped parameter t: its end vertex where t is exactly 0 or 1, else the edge
__device__ __forceinline__ uint32_t cp_edge_feature( const float t, const uint32_t a, const uint32_t b, const uint32_t e ) { return t == 0.0f ? a : t == 1.0f ? b : e; }

// The power of two that brings m (a largest magnitude, >= 0) into [1, 2): 2^-e for m in [2^e, 2^(e+1)), e clamped to [-126, 126] so that
// both it and its inverse (*inv = 2^e) are normal; 1 when m is 0 or not finite.  Multiplying by it is exact wherever nothing over- or
// underflows, so a quantity of degree k in lengths comes out scaled by exactly its k-th power.
__device__ __forceinline__ float cp_pow2( const float m, float& inv )
{
	const uint32_t f = __float_as_uint( m ) >> 23;
	if (!(m > 0.0f) || f == 255u) { inv = 1.0f; return 1.0f; }
	const uint32_t c = f < 1u ? 1u : f > 253u ? 253u : f;
	inv = __uint_as_float( c << 23 );
	return __uint_as_float( (254u - c) << 23 );
}

// ClosestPtPointTriangle of p against the leaf record (v0 | prim, e1, e2): the closest point is v0 + u e1 + v e2, u, v >= 0, u + v <= 1.
// Returns d2_raw; f: the feature of the closest point.  Regions in Ericson's order: A, B, AB, C, AC, BC, face; the face region takes the
// nearest of its face point (when the triangle's normal is not 0) and the three clamped edge points, ties to the face, then AB, AC, BC.
// A face point clamped onto an edge gives that edge (uf == 0: AC, vf == 0: AB, vf limited by 1 - uf: BC), two clamps their vertex.
// ap, e1 and e2 are first scaled by the power of two of their largest component (cp_pow2): the region products (vc, vb, va) and |n|^2
// are of degree 4 in lengths and would over- or underflow from about 2^32 and below 2^-31; d2_raw is scaled back at the end.
__device__ __forceinline__ float cp_triangle_feature( const float px, const float py, const float pz, const float4& v0, const float4& e1r, const float4& e2r,
	float& u, float& v, uint32_t& f )
{
	const float rx = __fsub_rn( px, v0.x ), ry = __fsub_rn( py, v0.y ), rz = __fsub_rn( pz, v0.z );
	const float m = fmaxf( fmaxf( fmaxf( fmaxf( fabsf( rx ), fabsf( ry ) ), fmaxf( fabsf( rz ), fabsf( e1r.x ) ) ), fmaxf( fmaxf( fabsf( e1r.y ), fabsf( e1r.z ) ),
		fmaxf( fabsf( e2r.x ), fabsf( e2r.y ) ) ) ), fabsf( e2r.z ) );
	float inv;
	const float s = cp_pow2( m, inv );
	const float apx = __fmul_rn( rx, s ), apy = __fmul_rn( ry, s ), apz = __fmul_rn( rz, s );
	const float4 e1 = make_float4( __fmul_rn( e1r.x, s ), __fmul_rn( e1r.y, s ), __fmul_rn( e1r.z, s ), 0.0f );
	const float4 e2 = make_float4( __fmul_rn( e2r.x, s ), __fmul_rn( e2r.y, s ), __fmul_rn( e2r.z, s ), 0.0f );
	const float d1 = cp_dot( e1.x, e1.y, e1.z, apx, apy, apz ), d2 = cp_dot( e2.x, e2.y, e2.z, apx, apy, apz );
	if (d1 <= 0.0f && d2 <= 0.0f) u = 0.0f, v = 0.0f, f = CP_V0;                                 // A
	else
	{
		const float bpx = __fsub_rn( apx, e1.x ), bpy = __fsub_rn( apy, e1.y ), bpz = __fsub_rn( apz, e1.z );
		const float d3 = cp_dot( e1.x, e1.y, e1.z, bpx, bpy, bpz ), d4 = cp_dot( e2.x, e2.y, e2.z, bpx, bpy, bpz );
		const float cpx = __fsub_rn( apx, e2.x ), cpy = __fsub_rn( apy, e2.y ), cpz = __fsub_rn( apz, e2.z );
		const float d5 = cp_dot( e1.x, e1.y, e1.z, cpx, cpy, cpz ), d6 = cp_dot( e2.x, e2.y, e2.z, cpx, cpy, cpz );
		const float vc = __fsub_rn( __fmul_rn( d1, d4 ), __fmul_rn( d3, d2 ) );
		const float vb = __fsub_rn( __fmul_rn( d5, d2 ), __fmul_rn( d1, d6 ) );
		const float va = __fsub_rn( __fmul_rn( d3, d6 ), __fmul_rn( d5, d4 ) );
		const float x = __fsub_rn( d4, d3 ), y = __fsub_rn( d5, d6 );
		if (d3 >= 0.0f && d4 <= d3) u = 1.0f, v = 0.0f, f = CP_V1;                                 // B
		else if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f)                                            // AB
			u = cp_edge( d1, __fsub_rn( d1, d3 ) ), v = 0.0f, f = cp_edge_feature( u, CP_V0, CP_V1, CP_AB );
		else if (d6 >= 0.0f && d5 <= d6) u = 0.0f, v = 1.0f, f = CP_V2;                            // C
		else if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f)                                            // AC
			u = 0.0f, v = cp_edge( d2, __fsub_rn( d2, d6 ) ), f = cp_edge_feature( v, CP_V0, CP_V2, CP_AC );
		else if (va <= 0.0f && x >= 0.0f && y >= 0.0f)                                              // BC
		{
			const float w = cp_edge( x, __fadd_rn( x, y ) );
			u = __fsub_rn( 1.0f, w ), v = w, f = cp_edge_feature( w, CP_V1, CP_V2, CP_BC );
		}
		else
		{
			// face: the clamped edge points - AB at d1 / |ab|^2, AC at d2 / |ac|^2, BC at (bp . bc) / |bc|^2 from b - and, when n = e1 x e2
			// is not 0, the face point u = ((ap x e2) . n) / |n|^2, v = ((e1 x ap) . n) / |n|^2; the nearest, ties to the face, then AB, AC,
			// BC.  The cross products keep the face weights accurate where Ericson's va / vb / vc (differences of products of dot products)
			// lose their digits, and on a sliver, whose face weights no formula keeps, the edges bound the error by the sliver's width.
			const float bcx = __fsub_rn( e2.x, e1.x ), bcy = __fsub_rn( e2.y, e1.y ), bcz = __fsub_rn( e2.z, e1.z );
			const float tab = cp_edge( d1, cp_dot( e1.x, e1.y, e1.z, e1.x, e1.y, e1.z ) );
			const float tac = cp_edge( d2, cp_dot( e2.x, e2.y, e2.z, e2.x, e2.y, e2.z ) );
			const float tbc = cp_edge( cp_dot( bcx, bcy, bcz, bpx, bpy, bpz ), cp_dot( bcx, bcy, bcz, bcx, bcy, bcz ) );
			float nx, ny, nz, ax, ay, az, bx, by, bz;
			cp_cross( e1.x, e1.y, e1.z, e2.x, e2.y, e2.z, nx, ny, nz );
			const float nn = cp_dot( nx, ny, nz, nx, ny, nz );
			const float dab = cp_dist2( apx, apy, apz, e1, e2, tab, 0.0f );
			float dm = dab;
			u = tab, v = 0.0f, f = cp_edge_feature( tab, CP_V0, CP_V1, CP_AB );
			if (nn > 0.0f)
			{
				cp_cross( apx, apy, apz, e2.x, e2.y, e2.z, ax, ay, az );
				cp_cross( e1.x, e1.y, e1.z, apx, apy, apz, bx, by, bz );
				const float inv = __fdiv_rn( 1.0f, nn );
				const float uf = cp_unit( __fmul_rn( cp_dot( ax, ay, az, nx, ny, nz ), inv ) );
				const float vmax = __fsub_rn( 1.0f, uf ), w = cp_unit( __fmul_rn( cp_dot( bx, by, bz, nx, ny, nz ), inv ) );
				const float vf = w < vmax ? w : vmax, df = cp_dist2( apx, apy, apz, e1, e2, uf, vf );
				if (df <= dab)
				{
					const bool cu = uf == 0.0f, cv = vf == 0.0f, cl = !(w < vmax);
					u = uf, v = vf, dm = df;
					f = cu ? (cv ? CP_V0 : cl ? CP_V2 : CP_AC) : cv ? (cl ? CP_V1 : CP_AB) : cl ? CP_BC : CP_FACE;
				}
			}
			const float dac = cp_dist2( apx, apy, apz, e1, e2, 0.0f, tac );
			if (dac < dm) u = 0.0f, v = tac, dm = dac, f = cp_edge_feature( tac, CP_V0, CP_V2, CP_AC );
			const float ubc = __fsub_rn( 1.0f, tbc ), dbc = cp_dist2( apx, apy, apz, e1, e2, ubc, tbc );
			if (dbc < dm) u = ubc, v = tbc, f = cp_edge_feature( tbc, CP_V1, CP_V2, CP_BC );
		}
	}
	return __fmul_rn( __fmul_rn( cp_dist2( apx, apy, apz, e1, e2, u, v ), inv ), inv );
}
// the form the walk calls: no feature
__device__ __forceinline__ float cp_triangle( const float px, const float py, const float pz, const float4& v0, const float4& e1, const float4& e2,
	float& u, float& v )
{
	uint32_t f;
	return cp_triangle_feature( px, py, pz, v0, e1, e2, u, v, f );
}

// squared distance from p to the box [bmin, bmax] (0 inside): each operation is monotone in the box and in the distance
__device__ __forceinline__ float cp_box_bound( const float px, const float py, const float pz, const float4& bmin, const float4& bmax )
{
	const float gx = fmaxf( fmaxf( __fsub_rn( bmin.x, px ), __fsub_rn( px, bmax.x ) ), 0.0f );
	const float gy = fmaxf( fmaxf( __fsub_rn( bmin.y, py ), __fsub_rn( py, bmax.y ) ), 0.0f );
	const float gz = fmaxf( fmaxf( __fsub_rn( bmin.z, pz ), __fsub_rn( pz, bmax.z ) ), 0.0f );
	return __fmaf_rn( gz, gz, __fmaf_rn( gy, gy, __fmul_rn( gx, gx ) ) );
}

// a pending subtree: the child record (ref, cnt) and its path bound
struct CpEntry { uint32_t ref, cnt; float P; };

// One query's walk from (ref, cnt) = the root with a caller-supplied stack deep enough for the tree (bvh2_walk's sizes).
// Closest (ANY = false): best / bprim / bu / bv enter as (r_max^2, CP_NO_PRIM, 0, 0) and leave as the smallest ( d2, prim ).
// ANY: returns true at the first reference with d2 <= best; best is not lowered.
template <bool ANY> __device__ __forceinline__ bool cp_walk( const float4* __restrict__ nodes, const float4* __restrict__ tris, uint32_t ref, uint32_t cnt,
	const float px, const float py, const float pz, float& best, uint32_t& bprim, float& bu, float& bv, CpEntry* stack )
{
	int sp = 0;
	float P = 0.0f;
	while (true)
	{
		if (cnt == 0)
		{
			const float4* q = nodes + (size_t)ref * 2;
			const float4 a0 = __ldg( q ), a1 = __ldg( q + 1 ), b0 = __ldg( q + 2 ), b1 = __ldg( q + 3 );
			const float Pa = fmaxf( cp_box_bound( px, py, pz, a0, a1 ), P ), Pb = fmaxf( cp_box_bound( px, py, pz, b0, b1 ), P );
			const bool va = !(Pa > best), vb = !(Pb > best); // strict: a subtree at exactly `best` may still hold a smaller prim
			const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w ), refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
			if (va && vb)
			{
				const bool swp = Pb < Pa; // nearer child first, the left one on ties
				ref = swp ? refb : refa, cnt = swp ? cntb : cnta, P = swp ? Pb : Pa;
				stack[sp++] = swp ? CpEntry{ refa, cnta, Pa } : CpEntry{ refb, cntb, Pb };
				continue;
			}
			if (va) { ref = refa, cnt = cnta, P = Pa; continue; }
			if (vb) { ref = refb, cnt = cntb, P = Pb; continue; }
		}
		else
		{
			const float4* tp = tris + (size_t)ref * 3;
			for (uint32_t k = 0; k < cnt; k++, tp += 3)
			{
				const float4 v0 = __ldg( tp ), e1 = __ldg( tp + 1 ), e2 = __ldg( tp + 2 );
				float u, v;
				const float d2 = fmaxf( cp_triangle( px, py, pz, v0, e1, e2, u, v ), P );
				const uint32_t prim = __float_as_uint( v0.w );
				if (ANY) { if (d2 <= best) return true; }
				else if (d2 < best || (d2 == best && prim < bprim)) best = d2, bprim = prim, bu = u, bv = v;
			}
		}
		// pop, pruning again against the current best
		while (true)
		{
			if (sp == 0) return false;
			const CpEntry e = stack[--sp];
			if (!(e.P > best)) { ref = e.ref, cnt = e.cnt, P = e.P; break; }
		}
	}
}

// whether a query takes a walk: no NaN coordinate, r >= 0
__device__ __forceinline__ bool cp_query_ok( const float4& q ) { return q.x == q.x && q.y == q.y && q.z == q.z && q.w >= 0.0f; }

// the result record of one closest-point query: { d, u, v, prim }, or { r_max, 0, 0, CP_NO_PRIM } when nothing lies within r_max
template <int STACKN> __device__ __forceinline__ float4 cp_closest( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	const uint32_t root_ref, const uint32_t root_count, const float4& q )
{
	if (!cp_query_ok( q )) return make_float4( q.w, 0.0f, 0.0f, __uint_as_float( CP_NO_PRIM ) );
	float best = __fmul_rn( q.w, q.w ), bu = 0.0f, bv = 0.0f;
	uint32_t bprim = CP_NO_PRIM;
	CpEntry stack[STACKN];
	cp_walk<false>( nodes, tris, root_ref, root_count, q.x, q.y, q.z, best, bprim, bu, bv, stack );
	if (bprim == CP_NO_PRIM) return make_float4( q.w, 0.0f, 0.0f, __uint_as_float( CP_NO_PRIM ) );
	return make_float4( __fsqrt_rn( best ), bu, bv, __uint_as_float( bprim ) );
}

// the sphere-overlap bit of one query { x, y, z, r }: some reference has d2 <= r^2
template <int STACKN> __device__ __forceinline__ bool cp_overlaps( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	const uint32_t root_ref, const uint32_t root_count, const float4& q )
{
	if (!cp_query_ok( q )) return false;
	float best = __fmul_rn( q.w, q.w ), bu = 0.0f, bv = 0.0f;
	uint32_t bprim = CP_NO_PRIM;
	CpEntry stack[STACKN];
	return cp_walk<true>( nodes, tris, root_ref, root_count, q.x, q.y, q.z, best, bprim, bu, bv, stack );
}

} // namespace tbvh
