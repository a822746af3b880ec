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
#include "common.cuh"
#include "../../include/tinybvh_b200_device.cuh"

namespace
{
// the per-ray body is tbvh::tlas_trace (include/tinybvh_b200_device.cuh), which the device functions callers' kernels use run too
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
		uint2 stack[TLAS_STACK], bstack[CW ? CW_STACK : TBVH_STACK];
		occluded = tbvh::tlas_trace<ANYHIT, CW>( nodes, prim_idx, inst, blas, root_ref, root_count, inst_shift, ro4, rd4, rr4, rh4, rr4.w, rh4, stack, bstack );
		if (!ANYHIT)
		{
			char* rec = rays + i * stride;
			if (inst_shift == 0) *(uint32_t*)(rec + 44) = __float_as_uint( rr4.w ); // INST_IDX_BITS == 32: hit.inst (:664)
			*(float4*)(rec + 48) = rh4;
		}
	}
	if (ANYHIT) store_occlusion_word( bits, i, n, occluded );
}
} // namespace

int tlas_trace_check( tbvh_bvh b, int layout )
{
	if (!b->d_inst || !b->d_blas || !b->d_nodes) { tbvh_set_error( "TLAS not resident" ); return TBVH_E_STATE; }
	const bool cw = layout == TBVH_LAYOUT_CWBVH;
	if (!cw && layout != TBVH_LAYOUT_BVH && layout != TBVH_LAYOUT_BVH_GPU) { tbvh_set_error( "unknown layout %d", layout ); return TBVH_E_ARG; }
	if (cw && !(b->tlas_blas_layouts & (1u << TBVH_LAYOUT_CWBVH)))
	{ tbvh_set_error( "TLAS: not every BLAS held its CWBVH layout when the TLAS was built (tbvh_convert the BLASses, then tbvh_build_tlas)" ); return TBVH_E_STATE; }
	if (!cw && !(b->tlas_blas_layouts & (1u << TBVH_LAYOUT_BVH)))
	{ tbvh_set_error( "TLAS: not every BLAS holds a BVH-layout tree; walk it with TBVH_LAYOUT_CWBVH" ); return TBVH_E_STATE; }
	return TBVH_OK;
}

uint32_t tlas_inst_shift( tbvh_bvh b )
{
	const int bits_opt = b->ctx->inst_idx_bits;
	return bits_opt >= 4 && bits_opt < 32 ? (uint32_t)(32 - bits_opt) : 0u;
}

int tlas_trace_launch( tbvh_bvh b, int layout, const void* d_rays, uint32_t stride, uint32_t* d_bits, uint64_t n, bool anyhit, cudaStream_t s )
{
	TRY( tlas_trace_check( b, layout ) );
	const bool cw = layout == TBVH_LAYOUT_CWBVH;
	if (n == 0) return TBVH_OK;
	const uint64_t grid = (n + 127) / 128;
	if (grid > 0x7fffffffull) { tbvh_set_error( "ray batch too large for one launch" ); return TBVH_E_ARG; }
	const uint32_t shift = tlas_inst_shift( b );
	#define LAUNCH( A, C ) k_trace_tlas<A, C><<<(uint32_t)grid, 128, 0, s>>>( b->d_nodes, b->d_prim_idx, b->d_inst, (const BlasRef*)b->d_blas.p, \
		(char*)d_rays, stride, d_bits, n, b->root_ref, b->root_count, shift )
	if (anyhit) { if (cw) LAUNCH( true, true ); else LAUNCH( true, false ); }
	else { if (cw) LAUNCH( false, true ); else LAUNCH( false, false ); }
	#undef LAUNCH
	LAUNCHED();
	return TBVH_OK;
}
