// tinybvh_b200/csrc/closest_point.cu - batched proximity queries over the BVH2: nearest surface point (tbvh_closest_point) and sphere
// overlap (tbvh_sphere_overlap, the batched BVH::IntersectSphere, tiny_bvh.h:3140-3200, under the engine's own definition).  The walk is
// include/tinybvh_b200_device/closest_walk.cuh, shared with the device functions callers' kernels use; DESIGN.md 4.9 states the rules.
#include "common.cuh"
#include "../../include/tinybvh_b200_device/closest_walk.cuh"

// One query per thread in 128-thread CTAs.  STACKN: TBVH_STACK for trees of depth below 64, TBVH_STACK_DEEP up to 255, as the ray walk.
// ANY: one bit per query (store_occlusion_word), else one 16-byte record { d, u, v, prim }.
template <bool ANY, int STACKN>
__global__ void __launch_bounds__( 128 ) k_closest_point( const float4* __restrict__ nodes, const float4* __restrict__ tris, const float4* __restrict__ queries,
	float4* __restrict__ results, uint32_t* __restrict__ bits, const uint64_t n, const uint32_t root_ref, const uint32_t root_count )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	bool hit = false;
	if (i < n)
	{
		const float4 q = __ldg( queries + i );
		if (ANY) hit = tbvh::cp_overlaps<STACKN>( nodes, tris, root_ref, root_count, q );
		else results[i] = tbvh::cp_closest<STACKN>( nodes, tris, root_ref, root_count, q );
	}
	if (ANY) store_occlusion_word( bits, i, n, hit );
}

// the refusals of a query batch before any work: TLAS, no BVH2, depth, launch size
static int closest_check( tbvh_bvh b, uint64_t n )
{
	if (b->d_inst) { tbvh_set_error( "proximity queries on a TLAS are not supported (distances do not survive non-rigid instance transforms)" ); return TBVH_E_UNSUPPORTED; }
	TRY( bvh2_trace_check( b, n ) );
	if ((n + 127) / 128 > 0x7fffffffull) { tbvh_set_error( "query batch too large for one launch" ); return TBVH_E_ARG; }
	return TBVH_OK;
}

// n > 0 queries after closest_check
static int closest_launch( tbvh_bvh b, const float4* d_queries, float4* d_results, uint32_t* d_bits, uint64_t n, cudaStream_t s )
{
	const bool any = d_bits != 0, deep = b->info.max_depth + 1 > TBVH_STACK;
	const uint32_t grid = (uint32_t)((n + 127) / 128);
	#define LAUNCH( A, D ) k_closest_point<A, D><<<grid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, d_queries, d_results, d_bits, n, b->root_ref, b->root_count )
	if (deep) { if (any) LAUNCH( true, TBVH_STACK_DEEP ); else LAUNCH( false, TBVH_STACK_DEEP ); }
	else { if (any) LAUNCH( true, TBVH_STACK ); else LAUNCH( false, TBVH_STACK ); }
	#undef LAUNCH
	LAUNCHED();
	return TBVH_OK;
}

// tbvh_closest_point / tbvh_sphere_overlap / tbvh_signed_distance / tbvh_winding_number / tbvh_sphere_cast(_occluded): every refusal
// before any launch; TBVH_HOST stages through the call's scratch
int proximity_query( const char* fn, tbvh_bvh b, const void* queries, void* out, uint64_t n, int space, void* stream, int kind, float beta )
{
	const bool any = kind == PROX_ANY || kind == PROX_SWEEP_ANY, wn = kind == PROX_WINDING, sweep = kind == PROX_SWEEP || kind == PROX_SWEEP_ANY;
	const size_t q_bytes = sweep ? 32 : 16;
	if (!b || !queries || !out) { tbvh_set_error( "%s: NULL argument", fn ); return TBVH_E_ARG; }
	if (space != TBVH_HOST && space != TBVH_DEVICE) { tbvh_set_error( "%s: unknown space %d", fn, space ); return TBVH_E_ARG; }
	if (space == TBVH_DEVICE && (((uintptr_t)queries & 15) || ((uintptr_t)out & (wn ? 3 : 15))))
	{ tbvh_set_error( wn ? "%s: device queries must be 16-byte and results 4-byte aligned" : "%s: device pointers must be 16-byte aligned", fn ); return TBVH_E_ARG; }
	if (wn && !(beta > 1.0f)) { tbvh_set_error( "%s: beta must be > 1 (the expansion needs the query outside the ball)", fn ); return TBVH_E_ARG; }
	TRY( closest_check( b, n ) );
	if (kind == PROX_SIGNED) TRY( sd_table_check( b ) );
	if (wn) TRY( wn_table_check( b ) );
	if (n == 0) return TBVH_OK;
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	auto launch = [&]( const float4* q, void* o, cudaStream_t s )
	{
		if (wn) return wn_launch( b, q, (float*)o, n, beta, s );
		if (sweep) return sc_launch( b, q, any ? 0 : (float4*)o, any ? (uint32_t*)o : 0, n, s );
		return kind == PROX_SIGNED ? sd_launch( b, q, (float4*)o, n, s ) : closest_launch( b, q, any ? 0 : (float4*)o, any ? (uint32_t*)o : 0, n, s );
	};
	if (space == TBVH_DEVICE) return launch( (const float4*)queries, out, (cudaStream_t)stream );
	const size_t out_bytes = any ? ((n + 31) / 32) * 4 : wn ? n * 4 : n * 16;
	Scratch sc( b->ctx->stream );
	float4* d_q = 0;
	char* d_out = 0;
	TRY( sc.alloc( d_q, n * q_bytes ) );
	TRY( sc.alloc( d_out, out_bytes ) );
	CUDA_TRY( cudaMemcpyAsync( d_q, queries, n * q_bytes, cudaMemcpyHostToDevice, sc.s ) );
	TRY( launch( d_q, d_out, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( out, d_out, out_bytes, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaStreamSynchronize( sc.s ) );
	return TBVH_OK;
}

extern "C" {

int tbvh_closest_point( tbvh_bvh b, const void* queries, void* results, uint64_t n, int space, void* stream )
{
	return proximity_query( __func__, b, queries, results, n, space, stream, PROX_CLOSEST );
}

int tbvh_sphere_overlap( tbvh_bvh b, const void* queries, uint32_t* bits, uint64_t n, int space, void* stream )
{
	return proximity_query( __func__, b, queries, bits, n, space, stream, PROX_ANY );
}

} // extern "C"
