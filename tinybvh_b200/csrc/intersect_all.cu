// tinybvh_b200/csrc/intersect_all.cu - multi-hit ray queries over the BVH2 (tbvh_intersect_all) and over a TLAS of BVH-layout BLASses
// (tbvh_intersect_all_tlas): the k nearest distinct triangles (instance hits) each ray crosses, nearest first, and how many it crosses
// (saturated at k + 1).  The walks are include/tinybvh_b200_device/all_hits_walk.cuh, shared with the device functions callers' kernels
// use; DESIGN.md 4.14 states the rules.
#include "common.cuh"
#include "../../include/tinybvh_b200_device/all_hits_walk.cuh"

// One ray per thread in 128-thread CTAs.  CAP / REG: the buffer of k + 1 <= CAP entries, in registers (k <= TBVH_INTERSECT_ALL_REG_K) or
// local memory (up to TBVH_INTERSECT_ALL_MAX_K).  STACKN: TBVH_STACK for trees of depth below 64, TBVH_STACK_DEEP up to 255, as the ray walk.
// Row i of hits is the k records at hits + i * k; counts[i] the count.
template <int CAP, bool REG, int STACKN>
__global__ void __launch_bounds__( 128 ) k_intersect_all( const float4* __restrict__ nodes, const float4* __restrict__ tris, const char* __restrict__ rays,
	const uint32_t stride, const uint32_t k, float4* __restrict__ hits, uint32_t* __restrict__ counts, const uint64_t n, const uint32_t root_ref,
	const uint32_t root_count )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	float4 ro4, rd4, rr4, rh4;
	tbvh::load_ray( rays, i, stride, ro4, rd4, rr4, rh4 );
	tbvh::CpEntry stack[STACKN];
	counts[i] = tbvh::ah_walk<CAP, REG>( nodes, tris, root_ref, root_count, ro4, rd4, rr4, rh4.x, k, hits + i * k, stack );
}

// n > 0 rays after the refusals
static int intersect_all_launch( tbvh_bvh b, const char* d_rays, uint32_t stride, uint32_t k, float4* d_hits, uint32_t* d_counts, uint64_t n, cudaStream_t s )
{
	const bool deep = b->info.max_depth + 1 > TBVH_STACK, reg = k <= TBVH_INTERSECT_ALL_REG_K;
	const uint32_t grid = (uint32_t)((n + 127) / 128);
	#define LAUNCH( C, R, D ) k_intersect_all<C, R, D><<<grid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, d_rays, stride, k, d_hits, d_counts, n, b->root_ref, b->root_count )
	constexpr int CREG = TBVH_INTERSECT_ALL_REG_K + 1, CMAX = TBVH_INTERSECT_ALL_MAX_K + 1;
	if (deep) { if (reg) LAUNCH( CREG, true, TBVH_STACK_DEEP ); else LAUNCH( CMAX, false, TBVH_STACK_DEEP ); }
	else { if (reg) LAUNCH( CREG, true, TBVH_STACK ); else LAUNCH( CMAX, false, TBVH_STACK ); }
	#undef LAUNCH
	LAUNCHED();
	return TBVH_OK;
}

// One ray per thread in 128-thread CTAs over a TLAS: CAP / REG as k_intersect_all; the TLAS stack has TLAS_STACK entries and the BLAS stack
// TBVH_STACK, the two-level walks' limits (a TLAS whose BLASses are deeper is refused before the launch).  Row i of insts is the k instances
// at insts + i * k.
template <int CAP, bool REG>
__global__ void __launch_bounds__( 128 ) k_intersect_all_tlas( const float4* __restrict__ nodes, const uint32_t* __restrict__ prim_idx,
	const tbvh::TlasInst* __restrict__ inst, const tbvh::BlasRef* __restrict__ blas, const char* __restrict__ rays, const uint32_t stride, const uint32_t k,
	float4* __restrict__ hits, uint32_t* __restrict__ insts, uint32_t* __restrict__ counts, const uint64_t n, const uint32_t root_ref, const uint32_t root_count )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	float4 ro4, rd4, rr4, rh4;
	tbvh::load_ray( rays, i, stride, ro4, rd4, rr4, rh4 );
	tbvh::CpEntry stack[TLAS_STACK], bstack[TBVH_STACK];
	counts[i] = tbvh::ah_walk_tlas<CAP, REG>( nodes, prim_idx, inst, blas, root_ref, root_count, ro4, rd4, rr4, rh4.x, k, hits + i * k, insts + i * k,
		stack, bstack );
}

static int intersect_all_tlas_launch( tbvh_bvh b, const char* d_rays, uint32_t stride, uint32_t k, float4* d_hits, uint32_t* d_insts, uint32_t* d_counts,
	uint64_t n, cudaStream_t s )
{
	const uint32_t grid = (uint32_t)((n + 127) / 128);
	#define LAUNCH( C, R ) k_intersect_all_tlas<C, R><<<grid, 128, 0, s>>>( b->d_nodes, b->d_prim_idx, b->d_inst, (const BlasRef*)b->d_blas.p, d_rays, stride, k, \
		d_hits, d_insts, d_counts, n, b->root_ref, b->root_count )
	if (k <= TBVH_INTERSECT_ALL_REG_K) LAUNCH( TBVH_INTERSECT_ALL_REG_K + 1, true );
	else LAUNCH( TBVH_INTERSECT_ALL_MAX_K + 1, false );
	#undef LAUNCH
	LAUNCHED();
	return TBVH_OK;
}

// the argument refusals both calls share (TBVH_E_ARG); insts: NULL for tbvh_intersect_all
static int intersect_all_args( const char* fn, tbvh_bvh b, const void* rays, uint32_t stride, uint64_t n, uint32_t k, const void* hits, const uint32_t* insts,
	const uint32_t* counts, int space, bool tlas )
{
	if (!b || !rays || !hits || !counts || (tlas && !insts)) { tbvh_set_error( "%s: NULL argument", fn ); return TBVH_E_ARG; }
	if (space != TBVH_HOST && space != TBVH_DEVICE) { tbvh_set_error( "%s: unknown space %d", fn, space ); return TBVH_E_ARG; }
	if (stride < 64 || (stride & 15)) { tbvh_set_error( "%s: ray stride %u is not a multiple of 16 of at least 64", fn, stride ); return TBVH_E_ARG; }
	if (space == TBVH_DEVICE && (((uintptr_t)rays & 15) || ((uintptr_t)hits & 15) || ((uintptr_t)counts & 3) || ((uintptr_t)insts & 3)))
	{ tbvh_set_error( "%s: device rays and hits must be 16-byte and counts%s 4-byte aligned", fn, tlas ? " and insts" : "" ); return TBVH_E_ARG; }
	if (k < 1 || k > TBVH_INTERSECT_ALL_MAX_K) { tbvh_set_error( "%s: k = %u outside 1..%d", fn, k, TBVH_INTERSECT_ALL_MAX_K ); return TBVH_E_ARG; }
	if ((n + 127) / 128 > 0x7fffffffull) { tbvh_set_error( "%s: ray batch too large for one launch", fn ); return TBVH_E_ARG; }
	return TBVH_OK;
}

extern "C" {

int tbvh_intersect_all( tbvh_bvh b, const void* rays, uint32_t stride, uint64_t n, uint32_t k, void* hits, uint32_t* counts, int space, void* stream )
{
	const char* fn = __func__;
	TRY( intersect_all_args( fn, b, rays, stride, n, k, hits, nullptr, counts, space, false ) );
	if (b->d_inst) { tbvh_set_error( "%s: a TLAS takes tbvh_intersect_all_tlas", fn ); return TBVH_E_UNSUPPORTED; }
	TRY( bvh2_trace_check( b, n ) );
	if (n == 0) return TBVH_OK;
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	if (space == TBVH_DEVICE) return intersect_all_launch( b, (const char*)rays, stride, k, (float4*)hits, counts, n, (cudaStream_t)stream );
	Scratch sc( b->ctx->stream );
	char* d_rays = 0;
	float4* d_hits = 0;
	uint32_t* d_counts = 0;
	TRY( sc.alloc( d_rays, n * stride ) );
	TRY( sc.alloc( d_hits, n * k * 16 ) );
	TRY( sc.alloc( d_counts, n * 4 ) );
	CUDA_TRY( cudaMemcpyAsync( d_rays, rays, n * stride, cudaMemcpyHostToDevice, sc.s ) );
	TRY( intersect_all_launch( b, d_rays, stride, k, d_hits, d_counts, n, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( hits, d_hits, n * k * 16, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( counts, d_counts, n * 4, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaStreamSynchronize( sc.s ) );
	return TBVH_OK;
}

int tbvh_intersect_all_tlas( tbvh_bvh b, const void* rays, uint32_t stride, uint64_t n, uint32_t k, void* hits, uint32_t* insts, uint32_t* counts, int space,
	void* stream )
{
	const char* fn = __func__;
	TRY( intersect_all_args( fn, b, rays, stride, n, k, hits, insts, counts, space, true ) );
	if (!b->d_inst) { tbvh_set_error( "%s: the handle holds no TLAS (a single BVH takes tbvh_intersect_all)", fn ); return TBVH_E_UNSUPPORTED; }
	// what tbvh_intersect_device( b, TBVH_LAYOUT_BVH, .. ) refuses: too deep a BLAS, a BLAS without its BVH-layout tree, a stale TLAS
	TRY( tlas_check( b, TBVH_LAYOUT_BVH ) );
	TRY( tlas_trace_check( b, TBVH_LAYOUT_BVH ) );
	if (n == 0) return TBVH_OK;
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	if (space == TBVH_DEVICE) return intersect_all_tlas_launch( b, (const char*)rays, stride, k, (float4*)hits, insts, counts, n, (cudaStream_t)stream );
	Scratch sc( b->ctx->stream );
	char* d_rays = 0;
	float4* d_hits = 0;
	uint32_t* d_insts = 0, * d_counts = 0;
	TRY( sc.alloc( d_rays, n * stride ) );
	TRY( sc.alloc( d_hits, n * k * 16 ) );
	TRY( sc.alloc( d_insts, n * k * 4 ) );
	TRY( sc.alloc( d_counts, n * 4 ) );
	CUDA_TRY( cudaMemcpyAsync( d_rays, rays, n * stride, cudaMemcpyHostToDevice, sc.s ) );
	TRY( intersect_all_tlas_launch( b, d_rays, stride, k, d_hits, d_insts, d_counts, n, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( hits, d_hits, n * k * 16, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( insts, d_insts, n * k * 4, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( counts, d_counts, n * 4, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaStreamSynchronize( sc.s ) );
	return TBVH_OK;
}

} // extern "C"
