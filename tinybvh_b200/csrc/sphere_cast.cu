// tinybvh_b200/csrc/sphere_cast.cu - batched sphere casts over the BVH2: the first contact of a sphere moving along a line
// (tbvh_sphere_cast) and whether it touches anything on the way (tbvh_sphere_cast_occluded).  The walk is
// include/tinybvh_b200_device/sweep_walk.cuh, shared with the device functions callers' kernels use; DESIGN.md 4.16 states the rules.
// Argument checks and the staging of TBVH_HOST batches are proximity_query's (closest_point.cu).
#include "common.cuh"
#include "../../include/tinybvh_b200_device/sweep_walk.cuh"

// One query per thread in 128-thread CTAs, its two rows { c, r }, { D, tmax } loaded as two float4.  STACKN: TBVH_STACK for trees of depth
// below 64, TBVH_STACK_DEEP up to 255, as the ray walk.  ANY: one bit per query (store_occlusion_word), else one 16-byte record
// { t, u, v, prim }.  The minimum of 4 CTAs per SM (up to 128 registers) is a hint that keeps ptxas from fitting the bit instance into 63
// registers with a spill.
template <bool ANY, int STACKN>
__global__ void __launch_bounds__( 128, 4 ) k_sphere_cast( const float4* __restrict__ nodes, const float4* __restrict__ tris, const float4* __restrict__ queries,
	float4* __restrict__ results, uint32_t* __restrict__ bits, const uint64_t n, const uint32_t root_ref, const uint32_t root_count )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	bool hit = false;
	if (i < n)
	{
		const float4 q0 = __ldg( queries + 2 * i ), q1 = __ldg( queries + 2 * i + 1 );
		if (ANY) hit = tbvh::sc_blocked<STACKN>( nodes, tris, root_ref, root_count, q0, q1 );
		else results[i] = tbvh::sc_cast<STACKN>( nodes, tris, root_ref, root_count, q0, q1 );
	}
	if (ANY) store_occlusion_word( bits, i, n, hit );
}

int sc_launch( tbvh_bvh b, const float4* d_queries, float4* d_results, uint32_t* d_bits, uint64_t n, cudaStream_t s )
{
	const bool any = d_bits != 0, deep = b->info.max_depth + 1 > TBVH_STACK;
	const uint32_t grid = (uint32_t)((n + 127) / 128);
	#define LAUNCH( A, D ) k_sphere_cast<A, D><<<grid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, d_queries, d_results, d_bits, n, b->root_ref, b->root_count )
	if (deep) { if (any) LAUNCH( true, TBVH_STACK_DEEP ); else LAUNCH( false, TBVH_STACK_DEEP ); }
	else { if (any) LAUNCH( true, TBVH_STACK ); else LAUNCH( false, TBVH_STACK ); }
	#undef LAUNCH
	LAUNCHED();
	return TBVH_OK;
}

extern "C" {

int tbvh_sphere_cast( tbvh_bvh b, const void* queries, void* results, uint64_t n, int space, void* stream )
{
	return proximity_query( __func__, b, queries, results, n, space, stream, PROX_SWEEP );
}

int tbvh_sphere_cast_occluded( tbvh_bvh b, const void* queries, uint32_t* bits, uint64_t n, int space, void* stream )
{
	return proximity_query( __func__, b, queries, bits, n, space, stream, PROX_SWEEP_ANY );
}

} // extern "C"
