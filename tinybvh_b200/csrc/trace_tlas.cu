// tinybvh_b200/csrc/trace_tlas.cu - two-level traversal: a TLAS over instances of BVH-layout BLASses, for sm_90a.
//
// Replaces BVH::IntersectTLAS<posX,posY,posZ> (tiny_bvh.h:3306-3380) and BVH::IsOccludedTLAS (:3455-3519) with
// INST_IDX_BITS == 32 (the library default: the instance number travels in hit.inst, byte 44 of the Ray record).
// The TLAS is walked like any BVH2 (bvh2_pair_step of bvh2_walk.cuh: stored rD, near child first, left on ties); per instance of a
// TLAS leaf, in primIdx order: skip unless inst.mask & ray.mask (:3326); O' = transform_point( O, invTransform ), D' = transform_vector(
// D, invTransform ) in the reference build's operation order (:513-527 compile to  fma( Tz, z, fma( Tx, x, Ty*y ) ) + Tw  per
// row, the point divided by w only when w != 1); rD' = safercp( D' ) (:442); then the BLAS is walked by k_trace_bvh2's own walk
// (bvh2_walk) with the running hit distance, and a hit records the instance.  Results are bit-identical to the
// oracle's (tests/test_tlas_gpu.py): t, u, v, prim, inst, occlusion bits.
//
// CW = true: the BLASses are walked in their BVH8_CWBVH layout instead - the arrangement of the reference's GPU path (traverse_tlas.cl:
// BVH2 TLAS, per-instance transform, CWBVH per BLAS, the hit kept when it is closer, the instance attached to it).  The reference's CPU
// IntersectTLAS refuses LAYOUT_CWBVH BLASses (:3339), so the oracle here is the composition of its two pinned pieces (oracle/tbvh_oracle.h,
// orc_intersect_tlas_cw): this file's TLAS walk and transform with BVH8_CWBVH::Intersect (:7046-7154) as the BLAS step - k_trace_wide's
// own walk (cw_trace of cw_walk.cuh) in its per-lane form, since transformed rays of one warp share no octant.
#include "bvh2_walk.cuh"
#include "cw_walk.cuh"

#define TLAS_STACK 64   // the reference's IntersectTLAS stack (:3308)

namespace
{
__device__ __forceinline__ float safercp( const float x ) { return (x > 1e-12f || x < -1e-12f) ? __fdiv_rn( 1.0f, x ) : (x >= 0 ? BVH_FAR : -BVH_FAR); }

template <bool ANYHIT, bool CW> __global__ void __launch_bounds__( 128 ) k_trace_tlas( const float4* __restrict__ nodes, const uint32_t* __restrict__ prim_idx,
	const TlasInst* __restrict__ inst, const BlasRef* __restrict__ blas, char* rays, const uint32_t stride, uint32_t* __restrict__ bits, const uint64_t n,
	const uint32_t root_ref, const uint32_t root_count, const uint32_t inst_shift /* 32 - INST_IDX_BITS; 0 = separate hit.inst field */ )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	bool occluded = false;
	if (i < n)
	{
		float4 ro4, rd4, rr4, rh4;
		load_ray( rays, i, stride, ro4, rd4, rr4, rh4 );
		const float ox = ro4.x, oy = ro4.y, oz = ro4.z, dx = rd4.x, dy = rd4.y, dz = rd4.z, rdx = rr4.x, rdy = rr4.y, rdz = rr4.z;
		const uint32_t rmask = __float_as_uint( ro4.w );
		const bool px = dx >= 0, py = dy >= 0, pz = dz >= 0;
		const float nrox = -__fmul_rn( ox, rdx ), nroy = -__fmul_rn( oy, rdy ), nroz = -__fmul_rn( oz, rdz );
		float tmax = rh4.x, hu = rh4.y, hv = rh4.z;
		uint32_t hprim = __float_as_uint( rh4.w ), hinst = __float_as_uint( rr4.w ); // hit.inst sits in the w lane of the rD row (byte 44)
		uint2 stack[TLAS_STACK], bstack[CW ? CW_STACK : TBVH_STACK];
		int sp = 0;
		uint32_t ref = root_ref, cnt = root_count;
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
			char* rec = rays + i * stride;
			if (inst_shift == 0) *(uint32_t*)(rec + 44) = hinst; // INST_IDX_BITS == 32: hit.inst (:664)
			*(float4*)(rec + 48) = make_float4( tmax, hu, hv, __uint_as_float( hprim ) );
		}
	}
	if (ANYHIT) store_occlusion_word( bits, i, n, occluded );
}
} // namespace

int tlas_trace_launch( tbvh_bvh b, int layout, const void* d_rays, uint32_t stride, uint32_t* d_bits, uint64_t n, bool anyhit, cudaStream_t s )
{
	if (!b->d_inst || !b->d_blas || !b->d_nodes) { tbvh_set_error( "TLAS not resident" ); return TBVH_E_STATE; }
	const bool cw = layout == TBVH_LAYOUT_CWBVH;
	if (!cw && layout != TBVH_LAYOUT_BVH && layout != TBVH_LAYOUT_BVH_GPU) { tbvh_set_error( "unknown layout %d", layout ); return TBVH_E_ARG; }
	if (cw && !(b->tlas_blas_layouts & (1u << TBVH_LAYOUT_CWBVH)))
	{ tbvh_set_error( "TLAS: not every BLAS held its CWBVH layout when the TLAS was built (tbvh_convert the BLASses, then tbvh_build_tlas)" ); return TBVH_E_STATE; }
	if (!cw && !(b->tlas_blas_layouts & (1u << TBVH_LAYOUT_BVH)))
	{ tbvh_set_error( "TLAS: not every BLAS holds a BVH-layout tree; walk it with TBVH_LAYOUT_CWBVH" ); return TBVH_E_STATE; }
	if (n == 0) return TBVH_OK;
	const uint64_t grid = (n + 127) / 128;
	if (grid > 0x7fffffffull) { tbvh_set_error( "ray batch too large for one launch" ); return TBVH_E_ARG; }
	const int bits_opt = b->ctx->inst_idx_bits;
	const uint32_t shift = bits_opt >= 4 && bits_opt < 32 ? (uint32_t)(32 - bits_opt) : 0u;
	#define LAUNCH( A, C ) k_trace_tlas<A, C><<<(uint32_t)grid, 128, 0, s>>>( b->d_nodes, b->d_prim_idx, (const TlasInst*)b->d_inst, (const BlasRef*)b->d_blas, \
		(char*)d_rays, stride, d_bits, n, b->root_ref, b->root_count, shift )
	if (anyhit) { if (cw) LAUNCH( true, true ); else LAUNCH( true, false ); }
	else { if (cw) LAUNCH( false, true ); else LAUNCH( false, false ); }
	#undef LAUNCH
	LAUNCHED();
	return TBVH_OK;
}
