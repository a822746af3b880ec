// include/tinybvh_b200_device.cuh - ray traversal from the caller's own CUDA kernels (sm_90a).
//
// The reference's GPU code traces from inside the application's kernels: traverse_cwbvh / isoccluded_cwbvh, traverse_ailalaine and
// traverse_tlas / isoccluded_tlas are device functions that wavefront.cl's Extend / Connect call.  This header gives the same shape
// over the engine's resident trees: take a view on the host (tbvh_device_view, include/tinybvh_b200.h), pass it to a kernel by value,
// and call
//
//     tbvh::intersect_bvh( view, ray )             tbvh::isoccluded_bvh( view, ray )              BVH / BVH_GPU layout
//     tbvh::intersect_cwbvh( view, ray )           tbvh::isoccluded_cwbvh( view, ray )            BVH8_CWBVH
//     tbvh::intersect_tlas<LAYOUT>( view, ray )    tbvh::isoccluded_tlas<LAYOUT>( view, ray )     TLAS, BLASses walked in LAYOUT
//
// The ray is the 64-byte device record in registers (tbvh::Ray: O | mask, D | instIdx, rD | hit.inst, t u v prim).  intersect_*
// updates ray.hit - and for a TLAS with INST_IDX_BITS 32 the hit.inst word, byte 44 - exactly as tbvh_intersect_device writes those
// bytes of the same record; isoccluded_* returns the bit tbvh_occluded_device writes.  Both run the library's own walks (this
// header's code is what its batch kernels run), so results agree bit for bit.
//
//  * Any subset of a warp's lanes may call, from loops and branches, with different views or layouts in different lanes.  The walks
//    pick a warp-uniform fast path (a direction octant compiled in, the integer-ordered CWBVH slab test) by votes over the lanes
//    that call together (__activemask()); every instance gives each ray the same result, so a lane's result never depends on which
//    other lanes take part.
//  * A function given a view of another kind returns without touching the ray (isoccluded_*: false).  It checks view.kind only;
//    a view is valid as long as include/tinybvh_b200.h says, and a stale view is a dangling pointer.
//  * Stacks are the batch kernels': 64 entries for BVH2 trees of depth below 64, 256 above (chosen per view), CW_STACK node groups
//    for a CWBVH, TLAS_STACK plus the BLAS stack for a TLAS - local memory per calling thread.  No statistics are collected.
//
// Compile with nvcc for sm_90a and -I <this directory>; nothing else is needed (no library link for the device code).
#pragma once
#include "tinybvh_b200.h"
#include "tinybvh_b200_device/base.cuh"
#include "tinybvh_b200_device/bvh2_walk.cuh"
#include "tinybvh_b200_device/cw_walk.cuh"

namespace tbvh
{

// ---- the per-ray bodies of the library's traversal kernels -------------------------------------------------------------------
// Each walks one ray record held in registers (its rows O | mask, D, rD | inst, hit) and writes what the kernel stores: closest hits
// through hit_out (and inst_out), any-hit as the result.  The kernels load the record, take their warp votes (uni, iord) over the whole
// warp and call the body with hit_out pointing into the hit buffer; the device functions below point it at the ray itself.  The
// interfaces follow the kernels' own variables, so that each kernel compiles to the code it had when the walk was written out in it.

// k_trace_bvh2: BVH::Intersect / IsOccluded from the root (root_ref, root_count) with a STACKN-entry stack.  `uni`: every ray of the
// voting lanes lies in this ray's direction octant (bvh2_pair_step).  Closest hit: *hit_out = (t, u, v, prim).
template <bool ANYHIT, bool STATS> __device__ __forceinline__ bool bvh2_trace( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	const uint32_t root_ref, const uint32_t root_count, const float4& O, const float4& D, const float4& rD, const float4& hit, float4* hit_out,
	const bool uni, uint2* stack, unsigned long long* __restrict__ stats )
{
	float tmax = hit.x, hu = hit.y, hv = hit.z;
	uint32_t hprim = __float_as_uint( hit.w );
	const bool occluded = bvh2_walk<ANYHIT, STATS>( nodes, tris, root_ref, root_count, O.x, O.y, O.z, D.x, D.y, D.z,
		rD.x, rD.y, rD.z, uni, tmax, hu, hv, hprim, stack, stats );
	if (!ANYHIT) *hit_out = make_float4( tmax, hu, hv, __uint_as_float( hprim ) );
	return occluded;
}

// The signs a CWBVH walk of a ray runs on: o = octinv of tiny_bvh.h:7053 (signs of D, visiting order), neg* and oct = the signs of rD
// (plane swizzle, :7082)
struct CwSigns { uint32_t o, oct; bool negx, negy, negz; };
__device__ __forceinline__ CwSigns cw_signs( const float4& D, const float4& rD )
{
	CwSigns g;
	g.o = 7u - ((D.x < 0 ? 4u : 0u) | (D.y < 0 ? 2u : 0u) | (D.z < 0 ? 1u : 0u));
	g.negx = rD.x < 0, g.negy = rD.y < 0, g.negz = rD.z < 0;
	g.oct = (g.negx ? 4u : 0u) | (g.negy ? 2u : 0u) | (g.negz ? 1u : 0u);
	return g;
}

// k_trace_wide: BVH8_CWBVH::Intersect / IsOccluded.  `uni_iord`: every ray of the voting lanes has this ray's octant, in the signs of rD
// (plane choice) and of D (visiting order) alike, and passes cw_ray_fits( .., rd_limit ); `iord`: every one passes cw_ray_fits.  Closest
// hit: *hit_out = (t, u, v, prim), with the ray's own u, v, prim kept when t is not below BVH_FAR.  o, oct, neg*: cw_signs( D, rD ).
// `pending`: CW_STACK node groups.
template <bool ANYHIT, bool STATS> __device__ __forceinline__ bool cw_trace_ray( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	const float ox, const float oy, const float oz, const float dx, const float dy, const float dz, const float rdx, const float rdy, const float rdz,
	const float4& hit, float4* hit_out, const uint32_t o, const uint32_t oct, const bool negx, const bool negy, const bool negz, const bool uni_iord,
	const bool iord, uint2* pending, unsigned long long* __restrict__ stats )
{
	bool occluded;
	float t = hit.x, hu = hit.y, hv = hit.z;
	uint32_t hprim = __float_as_uint( hit.w );
	#define TBVH_CW_TRACE_( O, I ) occluded = cw_trace<ANYHIT, STATS, O, I>( nodes, tris, ox, oy, oz, dx, dy, dz, rdx, rdy, rdz, o, negx, negy, negz, t, hu, hv, hprim, pending, stats )
	if (uni_iord)
	{
		switch (oct)
		{
		case 0: TBVH_CW_TRACE_( 0, true ); break;
		case 1: TBVH_CW_TRACE_( 1, true ); break;
		case 2: TBVH_CW_TRACE_( 2, true ); break;
		case 3: TBVH_CW_TRACE_( 3, true ); break;
		case 4: TBVH_CW_TRACE_( 4, true ); break;
		case 5: TBVH_CW_TRACE_( 5, true ); break;
		case 6: TBVH_CW_TRACE_( 6, true ); break;
		default: TBVH_CW_TRACE_( 7, true ); break;
		}
	}
	else if (iord) TBVH_CW_TRACE_( -1, true );
	else TBVH_CW_TRACE_( -1, false );
	#undef TBVH_CW_TRACE_
	if (!ANYHIT)
	{
		// the reference stores t, but u, v and prim only when t < BVH_FAR (end of :7046-7154): a NaN or infinite distance (Moeller-Trumbore
		// overflowing on huge coordinates) leaves the ray's own u, v, prim
		if (!(t < BVH_FAR)) hu = hit.y, hv = hit.z, hprim = __float_as_uint( hit.w );
		*hit_out = make_float4( t, hu, hv, __uint_as_float( hprim ) );
	}
	return occluded;
}

// k_trace_tlas: BVH::IntersectTLAS / IsOccludedTLAS (tiny_bvh.h:3306-3380, :3455-3519).  The TLAS is walked like any BVH2 (bvh2_pair_step:
// stored rD, near child first, left on ties); per instance of a TLAS leaf, in primIdx order: skip unless inst.mask & ray.mask (:3326);
// O' = transform_point( O, invTransform ), D' = transform_vector( D, invTransform ) in the reference build's operation order (:513-527
// compile to  fma( Tz, z, fma( Tx, x, Ty*y ) ) + Tw  per row, the point divided by w only when w != 1); rD' = safercp( D' ); then the
// BLAS is walked with the running hit distance, and a hit records the instance.  CW: the BLASses are walked in their BVH8_CWBVH layout
// (traverse_tlas.cl) by cw_trace's per-lane form, since transformed rays of one warp share no octant.  Closest hit: (t, u, v,
// prim) to hit_out and, when inst_shift is 0 (INST_IDX_BITS 32), hit.inst to inst_out (both may alias the inputs); otherwise the instance goes into the top bits of prim.
template <bool ANYHIT, bool CW> __device__ __forceinline__ bool tlas_trace( const float4* __restrict__ nodes, const uint32_t* __restrict__ prim_idx,
	const TlasInst* __restrict__ inst, const BlasRef* __restrict__ blas, const uint32_t root_ref, const uint32_t root_count,
	const uint32_t inst_shift /* 32 - INST_IDX_BITS; 0 = separate hit.inst field */, const float4& O, const float4& D, const float4& rD, const float4& hit,
	float& inst_out, float4& hit_out, uint2* stack, uint2* bstack )
{
	const float ox = O.x, oy = O.y, oz = O.z, dx = D.x, dy = D.y, dz = D.z, rdx = rD.x, rdy = rD.y, rdz = rD.z;
	const uint32_t rmask = __float_as_uint( O.w );
	const bool px = dx >= 0, py = dy >= 0, pz = dz >= 0;
	const float nrox = -__fmul_rn( ox, rdx ), nroy = -__fmul_rn( oy, rdy ), nroz = -__fmul_rn( oz, rdz );
	float tmax = hit.x, hu = hit.y, hv = hit.z;
	uint32_t hprim = __float_as_uint( hit.w ), hinst = __float_as_uint( rD.w ); // hit.inst sits in the w lane of the rD row (byte 44)
	int sp = 0;
	uint32_t ref = root_ref, cnt = root_count;
	bool occluded = false;
	while (true)
	{
		if (cnt == 0)
		{
			if (bvh2_pair_step( nodes, ref, cnt, stack, sp, px, py, pz, false, rdx, rdy, rdz, nrox, nroy, nroz, tmax )) continue;
		}
		else
		{
			for (uint32_t k = 0; k < cnt; k++)
			{
				const uint32_t instIdx = __ldg( prim_idx + ref + k );
				const float4* ip = (const float4*)(inst + instIdx);
				const float4 r0 = __ldg( ip ), r1 = __ldg( ip + 1 ), r2 = __ldg( ip + 2 ), r3 = __ldg( ip + 3 ), meta = __ldg( ip + 4 );
				if (!(__float_as_uint( meta.y ) & rmask)) continue;
				// tinybvh_transform_point / _vector (:513-527) in the reference build's pairing
				float tox = __fadd_rn( __fmaf_rn( r0.z, oz, __fmaf_rn( r0.x, ox, __fmul_rn( r0.y, oy ) ) ), r0.w );
				float toy = __fadd_rn( __fmaf_rn( r1.z, oz, __fmaf_rn( r1.x, ox, __fmul_rn( r1.y, oy ) ) ), r1.w );
				float toz = __fadd_rn( __fmaf_rn( r2.z, oz, __fmaf_rn( r2.x, ox, __fmul_rn( r2.y, oy ) ) ), r2.w );
				const float w = __fadd_rn( __fmaf_rn( oz, r3.z, __fmaf_rn( ox, r3.x, __fmul_rn( oy, r3.y ) ) ), r3.w );
				if (!(w == 1.0f)) { const float rw = __fdiv_rn( 1.0f, w ); tox = __fmul_rn( tox, rw ), toy = __fmul_rn( toy, rw ), toz = __fmul_rn( toz, rw ); }
				const float tdx = __fmaf_rn( r0.z, dz, __fmaf_rn( r0.x, dx, __fmul_rn( r0.y, dy ) ) );
				const float tdy = __fmaf_rn( r1.z, dz, __fmaf_rn( r1.x, dx, __fmul_rn( r1.y, dy ) ) );
				const float tdz = __fmaf_rn( r2.z, dz, __fmaf_rn( r2.x, dx, __fmul_rn( r2.y, dy ) ) );
				const BlasRef B = blas[__float_as_uint( meta.x )];
				const float trdx = safercp( tdx ), trdy = safercp( tdy ), trdz = safercp( tdz );
				bool hit; // any-hit: the ray is occluded; closest hit: the BLAS gave a nearer hit
				if (!CW) hit = bvh2_walk<ANYHIT, false>( B.trav, B.tris, B.root_ref, B.root_count, tox, toy, toz, tdx, tdy, tdz, trdx, trdy, trdz, false, tmax, hu, hv, hprim, bstack, nullptr );
				else
				{
					// BVH8_CWBVH::Intersect from the running distance t_in, kept only when it ends below it (`blasHit.x < hit.x`): a triangle
					// met at exactly t_in changes nothing.  Any-hit never lowers t, so LT_T tests each triangle against t_in itself.
					const uint32_t o = 7u - ((tdx < 0 ? 4u : 0u) | (tdy < 0 ? 2u : 0u) | (tdz < 0 ? 1u : 0u)); // octinv (:7053, signs of D)
					const float t_in = tmax;
					float t = tmax, lu = 0, lv = 0;
					uint32_t lprim = 0;
					if (cw_ray_fits( tox, toy, toz, trdx, trdy, trdz, B.cw_rd_limit ))
						hit = cw_trace<ANYHIT, false, -1, true, true>( B.cw_nodes, B.cw_tris, tox, toy, toz, tdx, tdy, tdz, trdx, trdy, trdz, o, trdx < 0, trdy < 0, trdz < 0, t, lu, lv, lprim, bstack, nullptr );
					else hit = cw_trace<ANYHIT, false, -1, false, true>( B.cw_nodes, B.cw_tris, tox, toy, toz, tdx, tdy, tdz, trdx, trdy, trdz, o, trdx < 0, trdy < 0, trdz < 0, t, lu, lv, lprim, bstack, nullptr );
					if (!ANYHIT && t < t_in) tmax = t, hu = lu, hv = lv, hprim = lprim, hit = true;
				}
				if (ANYHIT && hit)
				{
					occluded = true;
					break;
				}
				if (hit)
				{
					hinst = instIdx; // hit.inst = ray.instIdx (IntersectTri :8525)
					if (inst_shift) hprim += instIdx << inst_shift; // INST_IDX_BITS != 32: hit.prim = triIdx + ( instIdx << INST_IDX_SHFT ) (:8527)
				}
			}
			if (ANYHIT && occluded) break;
		}
		if (sp == 0) break;
		const uint2 e = stack[--sp];
		ref = e.x, cnt = e.y;
	}
	if (!ANYHIT)
	{
		if (inst_shift == 0) inst_out = __uint_as_float( hinst ); // INST_IDX_BITS == 32: hit.inst (:664)
		hit_out = make_float4( tmax, hu, hv, __uint_as_float( hprim ) );
	}
	return occluded;
}

// ---- device functions over a view -------------------------------------------------------------------------------------------

// the warp vote of the fast paths, over the lanes that call together: true when every one of them passes `key` equal to the first
// one's and `ok`
__device__ __forceinline__ bool lanes_agree( const uint32_t key, const bool ok )
{
	const uint32_t m = __activemask();
	const uint32_t key0 = __shfl_sync( m, key, __ffs( m ) - 1 );
	return __all_sync( m, ok && key == key0 );
}

template <bool ANYHIT> __device__ __forceinline__ bool bvh2_view_trace( const tbvh_view& v, Ray& r )
{
	const uint32_t oct = (r.D.x >= 0 ? 4u : 0u) | (r.D.y >= 0 ? 2u : 0u) | (r.D.z >= 0 ? 1u : 0u);
	const bool uni = lanes_agree( oct, true );
	const float4* nodes = (const float4*)v.nodes, * tris = (const float4*)v.tris;
	if (v.stack > TBVH_STACK)
	{
		uint2 stack[TBVH_STACK_DEEP];
		return bvh2_trace<ANYHIT, false>( nodes, tris, v.root_ref, v.root_count, r.O, r.D, r.rD, r.hit, &r.hit, uni, stack, nullptr );
	}
	uint2 stack[TBVH_STACK];
	return bvh2_trace<ANYHIT, false>( nodes, tris, v.root_ref, v.root_count, r.O, r.D, r.rD, r.hit, &r.hit, uni, stack, nullptr );
}

template <bool ANYHIT> __device__ __forceinline__ bool cw_view_trace( const tbvh_view& v, Ray& r )
{
	const CwSigns g = cw_signs( r.D, r.rD );
	const bool uni = lanes_agree( g.oct, g.o == 7u - g.oct );
	const bool iord = lanes_agree( 0u, cw_ray_fits( r.O.x, r.O.y, r.O.z, r.rD.x, r.rD.y, r.rD.z, v.cw_rd_limit ) );
	uint2 pending[CW_STACK];
	return cw_trace_ray<ANYHIT, false>( (const float4*)v.nodes, (const float4*)v.tris, r.O.x, r.O.y, r.O.z, r.D.x, r.D.y, r.D.z, r.rD.x, r.rD.y, r.rD.z,
		r.hit, &r.hit, g.o, g.oct, g.negx, g.negy, g.negz, uni && iord, iord, pending, nullptr );
}

template <int BLAS_LAYOUT> __device__ __forceinline__ constexpr int32_t tlas_view_kind()
{
	static_assert( BLAS_LAYOUT == TBVH_LAYOUT_BVH || BLAS_LAYOUT == TBVH_LAYOUT_CWBVH, "a TLAS walks its BLASses in TBVH_LAYOUT_BVH or TBVH_LAYOUT_CWBVH" );
	return BLAS_LAYOUT == TBVH_LAYOUT_CWBVH ? TBVH_VIEW_TLAS_CWBVH : TBVH_VIEW_TLAS_BVH;
}

template <bool ANYHIT, int BLAS_LAYOUT> __device__ __forceinline__ bool tlas_view_trace( const tbvh_view& v, Ray& r )
{
	uint2 stack[TLAS_STACK], bstack[BLAS_LAYOUT == TBVH_LAYOUT_CWBVH ? CW_STACK : TBVH_STACK];
	return tlas_trace<ANYHIT, BLAS_LAYOUT == TBVH_LAYOUT_CWBVH>( (const float4*)v.nodes, (const uint32_t*)v.prim_idx, (const TlasInst*)v.inst,
		(const BlasRef*)v.blas, v.root_ref, v.root_count, v.inst_shift, r.O, r.D, r.rD, r.hit, r.rD.w, r.hit, stack, bstack );
}

// BVH::Intersect / BVH_GPU::Intersect (tiny_bvh.h:3222, :4657) of one ray: a view of kind TBVH_VIEW_BVH
__device__ __forceinline__ void intersect_bvh( const tbvh_view& v, Ray& r )
{
	if (v.kind == TBVH_VIEW_BVH) bvh2_view_trace<false>( v, r );
}
// BVH::IsOccluded (:3382): any hit in [0, r.hit.t]
__device__ __forceinline__ bool isoccluded_bvh( const tbvh_view& v, const Ray& r )
{
	if (v.kind != TBVH_VIEW_BVH) return false;
	Ray c = r;
	return bvh2_view_trace<true>( v, c );
}

// BVH8_CWBVH::Intersect (:7046-7154): a view of kind TBVH_VIEW_CWBVH
__device__ __forceinline__ void intersect_cwbvh( const tbvh_view& v, Ray& r )
{
	if (v.kind == TBVH_VIEW_CWBVH) cw_view_trace<false>( v, r );
}
// BVH8_CWBVH::IsOccluded with FALLBACK_SHADOW_QUERY (:312): a hit with t < r.hit.t
__device__ __forceinline__ bool isoccluded_cwbvh( const tbvh_view& v, const Ray& r )
{
	if (v.kind != TBVH_VIEW_CWBVH) return false;
	Ray c = r;
	return cw_view_trace<true>( v, c );
}

// BVH::IntersectTLAS (:3306) with the BLASses walked in BLAS_LAYOUT (TBVH_LAYOUT_BVH, or TBVH_LAYOUT_CWBVH as traverse_tlas.cl does):
// a view taken for that layout, kind TBVH_VIEW_TLAS_BVH / TBVH_VIEW_TLAS_CWBVH
template <int BLAS_LAYOUT> __device__ __forceinline__ void intersect_tlas( const tbvh_view& v, Ray& r )
{
	if (v.kind == tlas_view_kind<BLAS_LAYOUT>()) tlas_view_trace<false, BLAS_LAYOUT>( v, r );
}
// BVH::IsOccludedTLAS (:3455)
template <int BLAS_LAYOUT> __device__ __forceinline__ bool isoccluded_tlas( const tbvh_view& v, const Ray& r )
{
	if (v.kind != tlas_view_kind<BLAS_LAYOUT>()) return false;
	Ray c = r;
	return tlas_view_trace<true, BLAS_LAYOUT>( v, c );
}

} // namespace tbvh
