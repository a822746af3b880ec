// tinybvh_b200/csrc/trace_tlas.cu - two-level traversal: a TLAS over instances of BVH-layout BLASses, for sm_90a.
//
// Replaces BVH::IntersectTLAS<posX,posY,posZ> (tiny_bvh.h:3306-3380) and BVH::IsOccludedTLAS (:3455-3519) with
// INST_IDX_BITS == 32 (the library default: the instance number travels in hit.inst, byte 44 of the Ray record).
// The TLAS is walked like any BVH2 (stored rD, near child first, left on ties); per instance of a TLAS leaf, in primIdx
// order: skip unless inst.mask & ray.mask (:3326); O' = transform_point( O, invTransform ), D' = transform_vector( D,
// invTransform ) in the reference build's operation order (:513-527 compile to  fma( Tz, z, fma( Tx, x, Ty*y ) ) + Tw  per
// row, the point divided by w only when w != 1); rD' = safercp( D' ) (:442); then the BLAS is walked exactly as
// k_trace_bvh2 walks it, with the running hit distance, and a hit records the instance.  Results are bit-identical to the
// oracle's (tests/test_tlas_gpu.py): t, u, v, prim, inst, occlusion bits.
//
// CW = true: the BLASses are walked in their BVH8_CWBVH layout instead - the arrangement of the reference's GPU path (traverse_tlas.cl:
// BVH2 TLAS, per-instance transform, CWBVH per BLAS, the hit kept when it is closer, the instance attached to it).  The reference's CPU
// IntersectTLAS refuses LAYOUT_CWBVH BLASses (:3339), so the oracle here is the composition of its two pinned pieces (oracle/tbvh_oracle.h,
// orc_intersect_tlas_cw): this file's TLAS walk and transform with BVH8_CWBVH::Intersect (:7046-7154) as the BLAS step - the per-lane form
// of the node step in cw_walk.cuh, since transformed rays of one warp share no octant.
#include "cw_walk.cuh"

#define TLAS_STACK 64   // the reference's IntersectTLAS stack (:3308)

namespace
{
__device__ __forceinline__ float safercp( const float x ) { return (x > 1e-12f || x < -1e-12f) ? __fdiv_rn( 1.0f, x ) : (x >= 0 ? BVH_FAR : -BVH_FAR); }

// SLAB_TEST_TWO_NODES (:3202-3220) for one child box
__device__ __forceinline__ bool slab( const float4 c0, const float4 c1, const bool px, const bool py, const bool pz, const float rdx, const float rdy, const float rdz,
	const float nrox, const float nroy, const float nroz, const float tmax, float& tmin )
{
	const float tx1 = __fmaf_rn( px ? c0.x : c1.x, rdx, nrox ), tx2 = __fmaf_rn( px ? c1.x : c0.x, rdx, nrox );
	const float ty1 = __fmaf_rn( py ? c0.y : c1.y, rdy, nroy ), ty2 = __fmaf_rn( py ? c1.y : c0.y, rdy, nroy );
	const float tz1 = __fmaf_rn( pz ? c0.z : c1.z, rdz, nroz ), tz2 = __fmaf_rn( pz ? c1.z : c0.z, rdz, nroz );
	tmin = fmaxf( fmaxf( tx1, ty1 ), fmaxf( tz1, 0.0f ) );
	return fminf( fminf( tx2, ty2 ), fminf( tz2, tmax ) ) >= tmin;
}

// one BLAS, walked as k_trace_bvh2 does (trace_bvh2.cu): returns true on an any-hit; closest hits update tmax / hu / hv / hprim
template <bool ANYHIT> __device__ bool trace_blas( const BlasRef B, const float ox, const float oy, const float oz, const float dx, const float dy, const float dz,
	const float rdx, const float rdy, const float rdz, float& tmax, float& hu, float& hv, uint32_t& hprim, bool& hit, uint2* stack )
{
	const bool px = dx >= 0, py = dy >= 0, pz = dz >= 0;
	const float nrox = -__fmul_rn( ox, rdx ), nroy = -__fmul_rn( oy, rdy ), nroz = -__fmul_rn( oz, rdz );
	int sp = 0;
	uint32_t ref = B.root_ref, cnt = B.root_count;
	while (true)
	{
		if (cnt == 0)
		{
			const float4* p = B.trav + (size_t)ref * 2;
			const float4 a0 = __ldg( p ), a1 = __ldg( p + 1 ), b0 = __ldg( p + 2 ), b1 = __ldg( p + 3 );
			float tmina, tminb;
			const bool hita = slab( a0, a1, px, py, pz, rdx, rdy, rdz, nrox, nroy, nroz, tmax, tmina );
			const bool hitb = slab( b0, b1, px, py, pz, rdx, rdy, rdz, nrox, nroy, nroz, tmax, tminb );
			const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w ), refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
			if (hita && hitb)
			{
				const bool swp = tmina > tminb;
				ref = swp ? refb : refa, cnt = swp ? cntb : cnta;
				stack[sp++] = swp ? make_uint2( refa, cnta ) : make_uint2( refb, cntb );
				continue;
			}
			if (hita) { ref = refa, cnt = cnta; continue; }
			if (hitb) { ref = refb, cnt = cntb; continue; }
		}
		else
		{
			const float4* tp = B.tris + (size_t)ref * 3;
			for (uint32_t k = 0; k < cnt; k++, tp += 3)
			{
				const float4 v0 = __ldg( tp ), e1 = __ldg( tp + 1 ), e2 = __ldg( tp + 2 );
				float t, u, v;
				if (mt_test( ox, oy, oz, dx, dy, dz, v0, e1, e2, tmax, t, u, v ))
				{
					if (ANYHIT) return true;
					tmax = t, hu = u, hv = v, hprim = __float_as_uint( v0.w ), hit = true;
				}
			}
		}
		if (sp == 0) break;
		const uint2 e = stack[--sp];
		ref = e.x, cnt = e.y;
	}
	return false;
}

// one BLAS in its CWBVH layout, walked as k_trace_wide walks it (trace_cwbvh.cu) in the per-lane form; IORD as node_hits.  BVH8_CWBVH::Intersect starts from
// the running hit distance and the two-level walk keeps its result only when it ends BELOW that distance (`blasHit.x < hit.x`): a
// triangle met at exactly the running distance changes nothing.
template <bool ANYHIT, bool IORD> __device__ bool trace_blas_cw( const float4* __restrict__ nodes, const float4* __restrict__ tris, const float ox, const float oy, const float oz,
	const float dx, const float dy, const float dz, const float rdx, const float rdy, const float rdz, float& tmax, float& hu, float& hv, uint32_t& hprim, bool& hit, uint2* pending )
{
	const uint32_t o = 7u - ((dx < 0 ? 4u : 0u) | (dy < 0 ? 2u : 0u) | (dz < 0 ? 1u : 0u)); // octinv (:7053, signs of D)
	const bool negx = rdx < 0, negy = rdy < 0, negz = rdz < 0;                                // plane choice (:7082, signs of rD)
	const float t_in = tmax;
	float t = tmax, lu = 0, lv = 0;
	uint32_t lprim = 0;
	int depth = 0;
	uint32_t base = 0, word = 0x80000000u;
	while (true)
	{
		const uint32_t bit = 31u - __clz( word );
		const uint32_t rest = word & ~(1u << bit);
		if (rest > 0x00ffffffu) pending[depth++] = make_uint2( base, rest );
		const uint32_t slot = (bit - 24u) ^ o;
		const uint32_t nidx = base + __popc( word & ~(0xffffffffu << slot) );
		const float4* np = nodes + (size_t)nidx * CW_NODE_F4;
		const float4 h0 = __ldg( np ), h1 = __ldg( np + 1 );
		const uint32_t szm = __float_as_uint( h1.z );
		const uint32_t got = node_hits<-1, IORD>( np, h0, h1, ox, oy, oz, rdx, rdy, rdz, negx, negy, negz, o, t );
		base = __float_as_uint( h1.x );
		word = (got & 0xff000000u) | ((szm >> 16) & 255u);
		uint32_t tmask = got & 0x00ffffffu;
		const float4* tbase = tris + __float_as_uint( h1.y );
		while (tmask)
		{
			const uint32_t k = 31u - __clz( tmask );
			tmask &= ~(1u << k);
			const float4* tp = tbase + k * 3;
			const float4 e2 = __ldg( tp ), e1 = __ldg( tp + 1 ), v0 = __ldg( tp + 2 );
			float tt, u, v;
			if (mt_test( ox, oy, oz, dx, dy, dz, v0, e1, e2, t, tt, u, v ))
			{
				if (ANYHIT) { if (tt < t_in) return true; }
				else t = tt, lu = u, lv = v, lprim = __float_as_uint( v0.w );
			}
		}
		if (word > 0x00ffffffu) continue;
		if (depth == 0) break;
		const uint2 e = pending[--depth];
		base = e.x, word = e.y;
	}
	if (!ANYHIT && t < t_in) tmax = t, hu = lu, hv = lv, hprim = lprim, hit = true;
	return false;
}

template <bool ANYHIT, bool CW> __global__ void __launch_bounds__( 128 ) k_trace_tlas( const float4* __restrict__ nodes, const uint32_t* __restrict__ prim_idx,
	const TlasInst* __restrict__ inst, const BlasRef* __restrict__ blas, char* rays, const uint32_t stride, uint32_t* __restrict__ bits, const uint64_t n,
	const uint32_t root_ref, const uint32_t root_count, const uint32_t inst_shift /* 32 - INST_IDX_BITS; 0 = separate hit.inst field */ )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	bool occluded = false;
	if (i < n)
	{
		const float4* rp = (const float4*)(rays + i * stride);
		const float4 ro4 = rp[0], rd4 = rp[1], rr4 = rp[2], rh4 = rp[3];
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
				const float4* p = nodes + (size_t)ref * 2;
				const float4 a0 = __ldg( p ), a1 = __ldg( p + 1 ), b0 = __ldg( p + 2 ), b1 = __ldg( p + 3 );
				float tmina, tminb;
				const bool hita = slab( a0, a1, px, py, pz, rdx, rdy, rdz, nrox, nroy, nroz, tmax, tmina );
				const bool hitb = slab( b0, b1, px, py, pz, rdx, rdy, rdz, nrox, nroy, nroz, tmax, tminb );
				const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w ), refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
				if (hita && hitb)
				{
					const bool swp = tmina > tminb;
					ref = swp ? refb : refa, cnt = swp ? cntb : cnta;
					stack[sp++] = swp ? make_uint2( refa, cnta ) : make_uint2( refb, cntb );
					continue;
				}
				if (hita) { ref = refa, cnt = cnta; continue; }
				if (hitb) { ref = refb, cnt = cntb; continue; }
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
					bool hit = false;
					const BlasRef B = blas[__float_as_uint( meta.x )];
					const float trdx = safercp( tdx ), trdy = safercp( tdy ), trdz = safercp( tdz );
					bool occ;
					if (!CW) occ = trace_blas<ANYHIT>( B, tox, toy, toz, tdx, tdy, tdz, trdx, trdy, trdz, tmax, hu, hv, hprim, hit, bstack );
					else if (cw_ray_fits( tox, toy, toz, trdx, trdy, trdz, B.cw_rd_limit ))
						occ = trace_blas_cw<ANYHIT, true>( B.cw_nodes, B.cw_tris, tox, toy, toz, tdx, tdy, tdz, trdx, trdy, trdz, tmax, hu, hv, hprim, hit, bstack );
					else occ = trace_blas_cw<ANYHIT, false>( B.cw_nodes, B.cw_tris, tox, toy, toz, tdx, tdy, tdz, trdx, trdy, trdz, tmax, hu, hv, hprim, hit, bstack );
					if (occ)
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
	if (ANYHIT)
	{
		const uint32_t m = __ballot_sync( 0xffffffffu, occluded );
		if ((threadIdx.x & 31) == 0 && (i & ~31ull) < n) bits[i >> 5] = m;
	}
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
