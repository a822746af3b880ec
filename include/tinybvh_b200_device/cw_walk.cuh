// include/tinybvh_b200_device/cw_walk.cuh - the CWBVH walk of every traversal that reads the wide layout (trace_cwbvh.cu: k_trace_wide;
// trace_tlas.cu: the CWBVH BLASses of the two-level kernel; the device functions of include/tinybvh_b200_device.cuh): the node step
// (node_hits: one 160-byte traversal node, layout in trace_cwbvh.cu cw_make_trav, against one ray -> the node's hit word) and the
// walk from the root (cw_trace).  Semantics: BVH8_CWBVH::Intersect, tiny_bvh.h:7046-7154.
#pragma once
#include "base.cuh"
#include <cuda_fp16.h>

#define CW_STACK 128            // node groups a ray can have pending: one per ancestor with inner siblings left (the reference's own limit, tiny_bvh.h:7048)
#define CW_NODE_F4 10           // float4 per traversal node
// Quantised planes in the traversal nodes: 0 = half pairs (widened by two HADD2.F32), 1 = bfloat16 pairs (0..255 is exact in 8
// significant bits; widening is one IMAD shift for the low half and one mask for the high half).  The library builds its traversal
// nodes as half pairs, so a caller's kernel must decode them the same way: the value is fixed here, not a build option.
#if defined( CW_PLANES_BF16 ) && CW_PLANES_BF16 != 0
#error "CW_PLANES_BF16: the library's traversal nodes hold half pairs (0)"
#endif
#undef CW_PLANES_BF16
#define CW_PLANES_BF16 0

namespace tbvh
{

__device__ __forceinline__ float2 widen( const uint32_t h2 )
{
#if CW_PLANES_BF16
	return make_float2( __uint_as_float( h2 * 65536u ), __uint_as_float( h2 & 0xffff0000u ) );
#else
	return __half22float2( *(const __half2*)&h2 );
#endif
}

// the same plane of two children: two fused multiply-adds, round to nearest (sm_90 has no packed fp32 FMA)
__device__ __forceinline__ float2 fma2( const float2 a, const float2 b, const float2 c )
{
	return make_float2( __fmaf_rn( a.x, b.x, c.x ), __fmaf_rn( a.y, b.y, c.y ) );
}

// The float slab test must use tinybvh_max / tinybvh_min (base.cuh ref_max / ref_min): a NaN plane (0 * inf where 2^e * rD
// overflows) in the second operand is returned, where fmaxf / fminf would drop it and keep the other side

// one pair of children against one ray: `near` / `far` words already chosen by the ray's signs.  IORD: the slab test on the bit
// patterns of the plane values as signed integers (cw_ray_fits states when that gives the float test's result)
template <bool IORD> __device__ __forceinline__ uint32_t pair_hits( const uint32_t wnx, const uint32_t wny, const uint32_t wnz, const uint32_t wfx, const uint32_t wfy, const uint32_t wfz,
	const uint32_t bits_a, const uint32_t bits_b, const float2 ax, const float2 ay, const float2 az, const float2 bx, const float2 by, const float2 bz, const float t )
{
	const float2 tnx = fma2( widen( wnx ), ax, bx ), tny = fma2( widen( wny ), ay, by ), tnz = fma2( widen( wnz ), az, bz );
	const float2 tfx = fma2( widen( wfx ), ax, bx ), tfy = fma2( widen( wfy ), ay, by ), tfz = fma2( widen( wfz ), az, bz );
	if (IORD)
	{
		// max( tn, +0 ) and min( tf ) in two three-input integer instructions each; `!( in > t )` lets a NaN t pass as fminf ignores it
		const int in_a = __vimax3_s32_relu( __float_as_int( tnx.x ), __float_as_int( tny.x ), __float_as_int( tnz.x ) );
		const int in_b = __vimax3_s32_relu( __float_as_int( tnx.y ), __float_as_int( tny.y ), __float_as_int( tnz.y ) );
		const int out_a = __vimin3_s32( __float_as_int( tfx.x ), __float_as_int( tfy.x ), __float_as_int( tfz.x ) );
		const int out_b = __vimin3_s32( __float_as_int( tfx.y ), __float_as_int( tfy.y ), __float_as_int( tfz.y ) );
		return (in_a <= out_a && !(__int_as_float( in_a ) > t) ? bits_a : 0u) | (in_b <= out_b && !(__int_as_float( in_b ) > t) ? bits_b : 0u);
	}
	// (a NaN t still passes, through fminf, as in the integer form)
	const float in_a = ref_max( ref_max( ref_max( tnx.x, tny.x ), tnz.x ), 0.0f ), out_a = fminf( ref_min( ref_min( tfx.x, tfy.x ), tfz.x ), t );
	const float in_b = ref_max( ref_max( ref_max( tnx.y, tny.y ), tnz.y ), 0.0f ), out_b = fminf( ref_min( ref_min( tfx.y, tfy.y ), tfz.y ), t );
	return (in_a <= out_a ? bits_a : 0u) | (in_b <= out_b ? bits_b : 0u);
}

// bits 24..31 of `w` hold inner-child hits by slot; move slot s to position s ^ o (o = 7 - octant)
__device__ __forceinline__ uint32_t slots_to_order( const uint32_t w, const uint32_t o )
{
	uint32_t top = w >> 24;
	if (o & 1u) top = ((top & 0x55u) << 1) | ((top >> 1) & 0x55u);
	if (o & 2u) top = ((top & 0x33u) << 2) | ((top >> 2) & 0x33u);
	if (o & 4u) top = ((top & 0x0fu) << 4) | (top >> 4);
	return top << 24;
}

// The integer-ordered slab test (pair_hits<true>) gives the float test's result when no plane value is NaN and no far plane is -0:
// the bit patterns of non-negative floats order as signed integers do, every negative float sorts below every non-negative one
// (so it still fails `in <= out` against in >= +0, as in float), and the RELU's 0 is +0.  -0 is excluded by adding +0 to
// ( p - O ) * rD (node_hits), which changes no comparison: fma( q, a, b ) is then -0 for no q.  NaN is excluded per ray and tree:
// a plane value fma( q, 2^e * rD, ( p - O ) * rD ) with q in 0..255 is not NaN when 2^e * rD is finite and ( p - O ) * rD is not
// NaN, which holds when |rD| <= rd_limit = 2^( 127 - largest e ) and |O|, |p| <= 2^126.  cw_make_trav finds the largest e and
// |p| of the tree and sets rd_limit < 0 (no ray fits) for a tree that has e = -128 (2^e is stored as -inf, :7072-7074) or
// |p| > 2^126.  A NaN running t is not excluded: `!( in > t )` passes it, as fminf( out, NaN ) ignores it.
#define CW_ORIGIN_LIMIT 8.5070592e37f // 2^126
__device__ __forceinline__ bool cw_ray_fits( const float ox, const float oy, const float oz, const float rdx, const float rdy, const float rdz, const float rd_limit )
{
	return fabsf( rdx ) <= rd_limit && fabsf( rdy ) <= rd_limit && fabsf( rdz ) <= rd_limit && // NaN fails every comparison
		fabsf( ox ) <= CW_ORIGIN_LIMIT && fabsf( oy ) <= CW_ORIGIN_LIMIT && fabsf( oz ) <= CW_ORIGIN_LIMIT;
}

// One traversal node against one ray -> the node's hit word in traversal order (inner children in bits 24..31 by s ^ o, triangles
// in bits 0..23).  h0 / h1: the node's header, already loaded.  OCT < 0: the ray's own signs (per lane); OCT = 0..7: every ray of
// the warp has negative x / y / z direction components as bits 2 / 1 / 0 of OCT say - plane choice and bit order are then
// compile-time.  IORD: the integer-ordered slab test, for rays that pass cw_ray_fits.
template <int OCT, bool IORD> __device__ __forceinline__ uint32_t node_hits( const float4* __restrict__ np, const float4 h0, const float4 h1,
	const float ox, const float oy, const float oz, const float rdx, const float rdy, const float rdz, const bool negx, const bool negy, const bool negz, const uint32_t o, const float t )
{
	// scale = 2^e as a float bit pattern, ( e + 127 ) << 23 (:7072-7074), stored by cw_make_trav as top halves
	const uint32_t sxy = __float_as_uint( h0.w ), szm = __float_as_uint( h1.z );
	const float scx = __uint_as_float( sxy << 16 ), scy = __uint_as_float( sxy & 0xffff0000u ), scz = __uint_as_float( szm << 16 );
	const float ax1 = __fmul_rn( scx, rdx ), ay1 = __fmul_rn( scy, rdy ), az1 = __fmul_rn( scz, rdz );
	// + 0: -0 becomes +0 (see cw_ray_fits)
	const float bx1 = __fadd_rn( __fmul_rn( -__fsub_rn( ox, h0.x ), rdx ), 0.0f ), by1 = __fadd_rn( __fmul_rn( -__fsub_rn( oy, h0.y ), rdy ), 0.0f );
	const float bz1 = __fadd_rn( __fmul_rn( -__fsub_rn( oz, h0.z ), rdz ), 0.0f );
	const bool nx = OCT < 0 ? negx : (OCT & 4) != 0, ny = OCT < 0 ? negy : (OCT & 2) != 0, nz = OCT < 0 ? negz : (OCT & 1) != 0;
	const float2 ax = make_float2( ax1, ax1 ), ay = make_float2( ay1, ay1 ), az = make_float2( az1, az1 );
	const float2 bx = make_float2( bx1, bx1 ), by = make_float2( by1, by1 ), bz = make_float2( bz1, bz1 );
	// All four pair records, unconditionally: a node visited on the way to a hit is almost always full (3.83 of 4 pair steps per visited
	// node on Bistro camera rays), the records behind the node's pair count are zero (no bits, so whatever their planes say contributes
	// nothing), and without the four branch regions the eight loads leave together.
	float4 A[4], B[4];
	#pragma unroll
	for (int j = 0; j < 4; j++) A[j] = __ldg( np + 2 + 2 * j ), B[j] = __ldg( np + 3 + 2 * j );
	uint32_t got = 0;
	#pragma unroll
	for (int j = 0; j < 4; j++)
	{
		const uint32_t lx = __float_as_uint( A[j].x ), ly = __float_as_uint( A[j].y ), lz = __float_as_uint( A[j].z );
		const uint32_t hx = __float_as_uint( A[j].w ), hy = __float_as_uint( B[j].x ), hz = __float_as_uint( B[j].y );
		got |= pair_hits<IORD>( nx ? hx : lx, ny ? hy : ly, nz ? hz : lz, nx ? lx : hx, ny ? ly : hy, nz ? lz : hz,
			__float_as_uint( B[j].z ), __float_as_uint( B[j].w ), ax, ay, az, bx, by, bz, t );
	}
	return slots_to_order( got, OCT < 0 ? o : (uint32_t)(7 - OCT) ) | (got & 0x00ffffffu);
}

// One ray's walk from the root with one instance of the node step (OCT, IORD: node_hits), `pending` holding CW_STACK groups.
// Returns true on an any-hit; closest hits update t / hu / hv / hprim.  STATS: node steps, triangle tests and pair steps are added
// to stats[0..2].
// Any-hit is BVH8_CWBVH::IsOccluded, FALLBACK_SHADOW_QUERY (tiny_bvh.h:312): Intersect, then hit.t < tmax - a triangle exactly at
// tmax does not occlude (boxes are still culled at tmax).  An any-hit walk never lowers t, so that is mt_test's below_tmax.
// LT_T: an any-hit triangle must also compare below t, as the two-level walk keeps a BLAS result (`blasHit.x < hit.x`): there a NaN
// distance (Moeller-Trumbore overflowing) or a NaN t does not occlude, where below_tmax alone (`!( tt >= t )`) lets it.
template <bool ANYHIT, bool STATS, int OCT, bool IORD, bool LT_T = false> __device__ __forceinline__ bool cw_trace( const float4* __restrict__ nodes,
	const float4* __restrict__ tris, const float ox, const float oy, const float oz, const float dx, const float dy, const float dz,
	const float rdx, const float rdy, const float rdz, const uint32_t o, const bool negx, const bool negy, const bool negz,
	float& t, float& hu, float& hv, uint32_t& hprim, uint2* pending, unsigned long long* __restrict__ stats )
{
	int depth = 0;
	uint32_t base = 0, word = 0x80000000u; // the root as a one-child group: bit 31, no siblings
	unsigned long long nsteps = 0, ntris = 0, npairs = 0;
	bool occluded = false;
	while (true)
	{
		// ---- enter the pending inner child with the highest bit
		const uint32_t bit = 31u - __clz( word );
		const uint32_t rest = word & ~(1u << bit);
		if (rest > 0x00ffffffu) pending[depth++] = make_uint2( base, rest );
		const uint32_t slot = (bit - 24u) ^ (OCT < 0 ? o : (uint32_t)(7 - OCT));
		const uint32_t nidx = base + __popc( word & ~(0xffffffffu << slot) );
		const float4* np = nodes + (size_t)nidx * CW_NODE_F4;
		const float4 h0 = __ldg( np ), h1 = __ldg( np + 1 );
		const uint32_t szm = __float_as_uint( h1.z );
		if (STATS) nsteps++, npairs += szm >> 24;
		const uint32_t got = node_hits<OCT, IORD>( np, h0, h1, ox, oy, oz, rdx, rdy, rdz, negx, negy, negz, o, t );
		base = __float_as_uint( h1.x );
		word = (got & 0xff000000u) | ((szm >> 16) & 255u);
		// ---- triangles of the leaf children that were hit, highest bit first (:7132-7142)
		uint32_t tmask = got & 0x00ffffffu;
		const float4* tbase = tris + __float_as_uint( h1.y );
		while (tmask)
		{
			const uint32_t k = 31u - __clz( tmask );
			tmask &= ~(1u << k);
			const float4* tp = tbase + k * 3;
			const float4 e2 = __ldg( tp ), e1 = __ldg( tp + 1 ), v0 = __ldg( tp + 2 );
			if (STATS) ntris++;
			float tt, u, v;
			if (mt_test( ox, oy, oz, dx, dy, dz, v0, e1, e2, t, tt, u, v, ANYHIT && !LT_T ) && (!(ANYHIT && LT_T) || tt < t))
			{
				if (ANYHIT) { occluded = true; break; }
				t = tt, hu = u, hv = v, hprim = __float_as_uint( v0.w );
			}
		}
		if (ANYHIT && occluded) break;
		if (word > 0x00ffffffu) continue;
		if (depth == 0) break;
		const uint2 e = pending[--depth];
		base = e.x, word = e.y;
	}
	if (STATS) { atomicAdd( &stats[0], nsteps ); atomicAdd( &stats[1], ntris ); atomicAdd( &stats[2], npairs ); }
	return occluded;
}

} // namespace tbvh
