// include/tinybvh_b200_device/bvh2_walk.cuh - the BVH2 walk of every traversal that reads the BVH layout: the library's kernels
// (trace_bvh2.cu: k_trace_bvh2, k_trace_bvh2_persist; trace_tlas.cu: the TLAS itself and its BVH-layout BLASses) and the device
// functions of include/tinybvh_b200_device.cuh.
//
// Semantics are the oracle's, bit for bit (SURVEY.md Appendix A): stored rD, slab term fma(bound, rD, -(O*rD)),
// tmin = max(tx1,ty1,tz1,0), tmax = min(tx2,ty2,tz2,hit.t), hit iff tmax >= tmin, nearer child first with the LEFT
// child on ties, leaf triangles in primIdx order, Moeller-Trumbore accepted on t in [0, hit.t] (later equal-t hits win).
//
// Device layout (DESIGN.md "BVH2 in HBM"): the two children of an interior node are one 64-byte, 64-aligned record
// (the reference's sibling pair nodes[leftFirst], nodes[leftFirst+1]) fetched as 4 x LDG.128; a child is
// {min.xyz, ref, max.xyz, count}: count == 0 -> interior, ref = index of its own pair; count > 0 -> leaf, ref = first
// record in the leaf-ordered triangle array (3 x float4 per triangle: v0|primIdx, e1, e2), so a leaf costs no node
// fetch and no primIdx indirection.
#pragma once
#include "base.cuh"
#include <type_traits>

namespace tbvh
{

// One interior step at the child pair `ref`: SLAB_TEST_TWO_NODES (tiny_bvh.h:3202-3220) of both children (near plane = min when
// D >= 0 else max), then the nearer hit child becomes (ref, cnt) and the other one is pushed.  Returns false when neither child is
// hit.  `uni` (every ray of the warp lies in this ray's direction octant, the normal case for camera and shadow rays): the slab
// test runs through the instance compiled for that octant, picked by a warp-uniform switch, which removes its 12 selects; otherwise
// it selects per lane by posX / posY / posZ.  Same arithmetic, same order, same results either way.  min / max are fminf / fmaxf
// (FMNMX), which drop a NaN plane the reference may keep (DESIGN.md 4.1).
__device__ __forceinline__ bool bvh2_pair_step( const float4* __restrict__ nodes, uint32_t& ref, uint32_t& cnt, uint2* stack, int& sp,
	const bool posX, const bool posY, const bool posZ, const bool uni, const float rdx, const float rdy, const float rdz,
	const float nrox, const float nroy, const float nroz, const float tmax )
{
	const float4* p = nodes + (size_t)ref * 2;
	const float4 a0 = __ldg( p ), a1 = __ldg( p + 1 ), b0 = __ldg( p + 2 ), b1 = __ldg( p + 3 );
	float tmina, tminb, tmaxa, tmaxb;
	// OCT = 0..7: D >= 0 in x / y / z as bits 2 / 1 / 0 of OCT say, compile-time; OCT < 0: the lane's own signs
	const auto slab = [&]( auto O )
	{
		constexpr int OCT = decltype( O )::value;
		const bool PX = OCT < 0 ? posX : (OCT & 4) != 0, PY = OCT < 0 ? posY : (OCT & 2) != 0, PZ = OCT < 0 ? posZ : (OCT & 1) != 0;
		const float tx1a = __fmaf_rn( PX ? a0.x : a1.x, rdx, nrox ), tx2a = __fmaf_rn( PX ? a1.x : a0.x, rdx, nrox );
		const float ty1a = __fmaf_rn( PY ? a0.y : a1.y, rdy, nroy ), ty2a = __fmaf_rn( PY ? a1.y : a0.y, rdy, nroy );
		const float tz1a = __fmaf_rn( PZ ? a0.z : a1.z, rdz, nroz ), tz2a = __fmaf_rn( PZ ? a1.z : a0.z, rdz, nroz );
		const float tx1b = __fmaf_rn( PX ? b0.x : b1.x, rdx, nrox ), tx2b = __fmaf_rn( PX ? b1.x : b0.x, rdx, nrox );
		const float ty1b = __fmaf_rn( PY ? b0.y : b1.y, rdy, nroy ), ty2b = __fmaf_rn( PY ? b1.y : b0.y, rdy, nroy );
		const float tz1b = __fmaf_rn( PZ ? b0.z : b1.z, rdz, nroz ), tz2b = __fmaf_rn( PZ ? b1.z : b0.z, rdz, nroz );
		tmina = fmaxf( fmaxf( tx1a, ty1a ), fmaxf( tz1a, 0.0f ) ), tminb = fmaxf( fmaxf( tx1b, ty1b ), fmaxf( tz1b, 0.0f ) );
		tmaxa = fminf( fminf( tx2a, ty2a ), fminf( tz2a, tmax ) ), tmaxb = fminf( fminf( tx2b, ty2b ), fminf( tz2b, tmax ) );
	};
	using std::integral_constant;
	if (uni)
	{
		switch ((posX ? 4u : 0u) | (posY ? 2u : 0u) | (posZ ? 1u : 0u))
		{
		case 0: slab( integral_constant<int, 0>() ); break;
		case 1: slab( integral_constant<int, 1>() ); break;
		case 2: slab( integral_constant<int, 2>() ); break;
		case 3: slab( integral_constant<int, 3>() ); break;
		case 4: slab( integral_constant<int, 4>() ); break;
		case 5: slab( integral_constant<int, 5>() ); break;
		case 6: slab( integral_constant<int, 6>() ); break;
		default: slab( integral_constant<int, 7>() ); break;
		}
	}
	else slab( integral_constant<int, -1>() );
	const bool hita = tmaxa >= tmina, hitb = tmaxb >= tminb;
	const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w );
	const uint32_t refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
	if (hita && hitb)
	{
		// swap only on dist1 > dist2: ties visit the left child first (:3292)
		const bool swp = tmina > tminb;
		ref = swp ? refb : refa, cnt = swp ? cntb : cnta;
		stack[sp++] = swp ? make_uint2( refa, cnta ) : make_uint2( refb, cntb );
		return true;
	}
	// separate exits, not one `return hita || hitb`: nvcc 12.9 if-converts the latter into selects, which changes the descent
	// k_trace_bvh2 compiles to; with separate exits it compiles as a branch per case, as the callers' `continue` expects
	if (hita) { ref = refa, cnt = cnta; return true; }
	if (hitb) { ref = refb, cnt = cntb; return true; }
	return false;
}

// One leaf: cnt triangles starting at record ref, in primIdx order (:3281-3285).  Any-hit: returns true on the first accepted
// triangle.  Closest hit: every accepted triangle updates tmax / hu / hv / hprim; returns whether one was accepted.  STATS: each
// triangle test adds one to *ntris.
template <bool ANYHIT, bool STATS> __device__ __forceinline__ bool bvh2_leaf( const float4* __restrict__ tris, const uint32_t ref, const uint32_t cnt,
	const float ox, const float oy, const float oz, const float dx, const float dy, const float dz,
	float& tmax, float& hu, float& hv, uint32_t& hprim, unsigned long long* ntris )
{
	bool hit = false;
	const float4* tp = tris + (size_t)ref * 3;
	for (uint32_t k = 0; k < cnt; k++, tp += 3)
	{
		const float4 v0 = __ldg( tp ), e1 = __ldg( tp + 1 ), e2 = __ldg( tp + 2 );
		float t, u, v;
		if (STATS) (*ntris)++;
		if (mt_test( ox, oy, oz, dx, dy, dz, v0, e1, e2, tmax, t, u, v ))
		{
			if (ANYHIT) return true;
			tmax = t, hu = u, hv = v, hprim = __float_as_uint( v0.w ), hit = true;
		}
	}
	return hit;
}

// One ray's walk from (ref, cnt) = the root, with a caller-supplied stack deep enough for the tree.  Returns what bvh2_leaf returns,
// over the whole walk.  `uni`: as bvh2_pair_step, decided per warp by the caller.  STATS: node steps and triangle tests are added
// to stats[0] / stats[1].
template <bool ANYHIT, bool STATS> __device__ __forceinline__ bool bvh2_walk( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	uint32_t ref, uint32_t cnt, const float ox, const float oy, const float oz, const float dx, const float dy, const float dz,
	const float rdx, const float rdy, const float rdz, const bool uni, float& tmax, float& hu, float& hv, uint32_t& hprim, uint2* stack,
	unsigned long long* __restrict__ stats )
{
	const bool posX = dx >= 0, posY = dy >= 0, posZ = dz >= 0;
	// -(O*rD), rounded product as the oracle's `rox` (:3252-3254)
	const float nrox = -__fmul_rn( ox, rdx ), nroy = -__fmul_rn( oy, rdy ), nroz = -__fmul_rn( oz, rdz );
	int sp = 0;
	unsigned long long nsteps = 0, ntris = 0;
	bool hit = false;
	while (true)
	{
		if (STATS) nsteps++;
		if (cnt == 0)
		{
			if (bvh2_pair_step( nodes, ref, cnt, stack, sp, posX, posY, posZ, uni, rdx, rdy, rdz, nrox, nroy, nroz, tmax )) continue;
		}
		else if (bvh2_leaf<ANYHIT, STATS>( tris, ref, cnt, ox, oy, oz, dx, dy, dz, tmax, hu, hv, hprim, &ntris ))
		{
			hit = true;
			if (ANYHIT) break;
		}
		if (sp == 0) break;
		const uint2 e = stack[--sp];
		ref = e.x, cnt = e.y;
	}
	if (STATS) { atomicAdd( &stats[0], nsteps ); atomicAdd( &stats[1], ntris ); }
	return hit;
}

} // namespace tbvh
