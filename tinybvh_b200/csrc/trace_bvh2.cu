// tinybvh_b200/csrc/trace_bvh2.cu - BVH2 closest-hit / any-hit traversal for sm_90a.
//
// Replaces BVH::Intersect<posX,posY,posZ> (tiny_bvh.h:3247-3304), BVH::IsOccluded<...> (:3407-3453) and the OpenCL
// kernels traverse_ailalaine / isoccluded_ailalaine (traverse_bvh2.cl:80,147) for whole ray batches.  The walk itself - node
// layout, slab test, descent order, leaf loop - is include/tinybvh_b200_device/bvh2_walk.cuh, and the per-ray body is
// tbvh::bvh2_trace, shared with the two-level kernel (trace_tlas.cu) and the device functions callers' kernels use.
#include "common.cuh"
#include "../../include/tinybvh_b200_device.cuh"
#include <stdlib.h>

// 128 threads with at least 10 resident CTAs per SM (40 warps / SM without spills; 12 and 16 were measured slower).
// OCTSW = 1: warps whose rays all lie in one direction octant take the octant-specialised slab tests (bvh2_pair_step).
// STACKN = traversal stack entries: TBVH_STACK (64) for trees of depth < 64, TBVH_STACK_DEEP (256, the reference's own stack, :3249) above.
template <bool ANYHIT, bool STATS, int OCTSW, int STACKN>
__global__ void __launch_bounds__( 128, 10 ) k_trace_bvh2( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	const char* rays, const uint32_t stride, char* hits, const uint32_t hit_stride, // may alias (in-place hits): plain loads
	uint32_t* __restrict__ bits, const uint64_t n, const uint32_t root_ref, const uint32_t root_count,
	unsigned long long* __restrict__ stats )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	bool occluded = false;
	const bool valid = i < n;
	float4 ro4 = make_float4( 0, 0, 0, 0 ), rd4 = ro4, rr4 = ro4, rh4 = ro4;
	if (valid) load_ray( rays, i, stride, ro4, rd4, rr4, rh4 );
	const uint32_t oct = (rd4.x >= 0 ? 4u : 0u) | (rd4.y >= 0 ? 2u : 0u) | (rd4.z >= 0 ? 1u : 0u);
	bool uni = false;
	if (OCTSW)
	{
		const uint32_t vm = __ballot_sync( 0xffffffffu, valid );
		const uint32_t oct0 = __shfl_sync( 0xffffffffu, oct, vm ? __ffs( vm ) - 1 : 0 );
		uni = __all_sync( 0xffffffffu, !valid || oct == oct0 );
	}
	if (valid)
	{
		uint2 stack[STACKN];
		occluded = tbvh::bvh2_trace<ANYHIT, STATS>( nodes, tris, root_ref, root_count, ro4, rd4, rr4, rh4, (float4*)(hits + i * hit_stride), uni, stack, stats );
	}
	if (ANYHIT) store_occlusion_word( bits, i, n, occluded );
}

// Persistent-warp variant for incoherent ray sets (diffuse bounces): resident warps pull rays from a global counter and
// refill the lanes whose ray has terminated once at least REFILL_MIN lanes are idle, so a few long rays no longer hold 31
// idle lanes hostage (the persistent-thread ray fetch of wavefront.cl:93-115, at lane granularity).  Each ray is still
// traversed exactly as in k_trace_bvh2 - same order, same arithmetic - only the lane it runs on differs.
#define PERSIST_ROUND 12     // traversal steps between two refill votes
#define REFILL_MIN 6         // idle lanes needed before the warp pays for a refill
template <bool ANYHIT>
__global__ void __launch_bounds__( 128, 10 ) k_trace_bvh2_persist( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	const char* rays, const uint32_t stride, char* hits, const uint32_t hit_stride, uint32_t* bits, const uint64_t n,
	const uint32_t root_ref, const uint32_t root_count, unsigned long long* next )
{
	const uint32_t lane = threadIdx.x & 31;
	bool active = false, more = true;
	uint64_t idx = 0;
	float ox = 0, oy = 0, oz = 0, dx = 0, dy = 0, dz = 0, rdx = 0, rdy = 0, rdz = 0, nrox = 0, nroy = 0, nroz = 0;
	float tmax = 0, hu = 0, hv = 0;
	uint32_t hprim = 0, ref = 0, cnt = 0;
	bool posX = true, posY = true, posZ = true;
	uint2 stack[TBVH_STACK];
	int sp = 0;
	while (true)
	{
		const uint32_t idle = __ballot_sync( 0xffffffffu, !active );
		if (more && (idle == 0xffffffffu || __popc( idle ) >= REFILL_MIN))
		{
			unsigned long long base = 0;
			if (lane == 0) base = atomicAdd( next, (unsigned long long)__popc( idle ) );
			base = __shfl_sync( 0xffffffffu, base, 0 );
			if (base >= n) more = false; // warp-uniform: the pool is dry
			if (!active)
			{
				idx = base + __popc( idle & ((1u << lane) - 1u) );
				if (idx < n)
				{
					float4 ro4, rd4, rr4, rh4;
					load_ray( rays, idx, stride, ro4, rd4, rr4, rh4 );
					ox = ro4.x, oy = ro4.y, oz = ro4.z, dx = rd4.x, dy = rd4.y, dz = rd4.z, rdx = rr4.x, rdy = rr4.y, rdz = rr4.z;
					nrox = -__fmul_rn( ox, rdx ), nroy = -__fmul_rn( oy, rdy ), nroz = -__fmul_rn( oz, rdz );
					posX = dx >= 0, posY = dy >= 0, posZ = dz >= 0;
					tmax = rh4.x, hu = rh4.y, hv = rh4.z, hprim = __float_as_uint( rh4.w );
					ref = root_ref, cnt = root_count, sp = 0, active = true;
				}
			}
		}
		if (!__any_sync( 0xffffffffu, active )) break;
		if (active)
		{
			bool done = false, occluded = false;
			for (int it = 0; it < PERSIST_ROUND; it++)
			{
				if (cnt == 0)
				{
					if (tbvh::bvh2_pair_step( nodes, ref, cnt, stack, sp, posX, posY, posZ, false, rdx, rdy, rdz, nrox, nroy, nroz, tmax )) continue;
				}
				else if (tbvh::bvh2_leaf<ANYHIT, false>( tris, ref, cnt, ox, oy, oz, dx, dy, dz, tmax, hu, hv, hprim, nullptr ) && ANYHIT) { occluded = done = true; break; }
				if (sp == 0) { done = true; break; }
				const uint2 e = stack[--sp];
				ref = e.x, cnt = e.y;
			}
			if (done)
			{
				if (!ANYHIT) *(float4*)(hits + idx * hit_stride) = make_float4( tmax, hu, hv, __uint_as_float( hprim ) );
				else if (occluded) atomicOr( bits + (idx >> 5), 1u << (uint32_t)(idx & 31) );
				active = false;
			}
		}
	}
}

unsigned long long* ctx_next_counter( tbvh_ctx c ) { return c->d_counters + (c->counter_next.fetch_add( 1 ) % TBVH_COUNTERS); }

int bvh2_trace_check( tbvh_bvh b, uint64_t n )
{
	if (!b->trav() || !b->d_leaf_tris) { tbvh_set_error( "BVH2 layout not resident" ); return TBVH_E_STATE; }
	if (n == 0) return TBVH_OK;
	if (b->info.max_depth + 1 > TBVH_STACK_DEEP) { tbvh_set_error( "BVH depth %u exceeds the %d-entry traversal stack (the reference's own, tiny_bvh.h:3249)", b->info.max_depth, TBVH_STACK_DEEP ); return TBVH_E_LIMIT; }
	return TBVH_OK;
}

int bvh2_trace_launch( tbvh_bvh b, const void* d_rays, uint32_t stride, void* d_hits, uint32_t hit_stride, uint32_t* d_bits,
	uint64_t n, bool anyhit, cudaStream_t s, unsigned long long* d_stats )
{
	TRY( bvh2_trace_check( b, n ) );
	if (n == 0) return TBVH_OK;
	const bool deep = b->info.max_depth + 1 > TBVH_STACK;
	const uint32_t root_ref = b->root_ref, root_count = b->root_count;
	const uint32_t block = 128;
	const uint64_t grid = (n + block - 1) / block;
	if (grid > 0x7fffffffull) { tbvh_set_error( "ray batch too large for one launch" ); return TBVH_E_ARG; }
	const int variant = b->ctx->trace_variant;
	#define LAUNCH( A, S, O, D ) k_trace_bvh2<A, S, O, D><<<(uint32_t)grid, block, 0, s>>>( b->trav(), b->d_leaf_tris, (const char*)d_rays, stride, \
		(char*)d_hits, hit_stride, d_bits, n, root_ref, root_count, d_stats )
	if (deep)
	{
		// depth 64..255: the same kernel with the reference's 256-entry stack (2 KiB of local memory per ray)
		if (d_stats) { if (anyhit) LAUNCH( true, true, 0, TBVH_STACK_DEEP ); else LAUNCH( false, true, 0, TBVH_STACK_DEEP ); }
		else { if (anyhit) LAUNCH( true, false, 1, TBVH_STACK_DEEP ); else LAUNCH( false, false, 1, TBVH_STACK_DEEP ); }
		LAUNCHED();
		return TBVH_OK;
	}
	if (variant == 4 && !d_stats)
	{
		// persistent warps: one resident wave (10 CTAs of 128 threads per SM), rays pulled from a counter that belongs to this launch
		unsigned long long* next = ctx_next_counter( b->ctx );
		CUDA_TRY( cudaMemsetAsync( next, 0, 8, s ) );
		if (anyhit) CUDA_TRY( cudaMemsetAsync( d_bits, 0, ((n + 31) / 32) * 4, s ) );
		const uint32_t pgrid = (uint32_t)b->ctx->sm_count * 10u;
		if (anyhit) k_trace_bvh2_persist<true><<<pgrid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, (const char*)d_rays, stride, (char*)d_hits, hit_stride, d_bits, n, root_ref, root_count, next );
		else k_trace_bvh2_persist<false><<<pgrid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, (const char*)d_rays, stride, (char*)d_hits, hit_stride, d_bits, n, root_ref, root_count, next );
		LAUNCHED();
		return TBVH_OK;
	}
	if (d_stats) { if (anyhit) LAUNCH( true, true, 0, TBVH_STACK ); else LAUNCH( false, true, 0, TBVH_STACK ); }
	else if (variant == 3) { if (anyhit) LAUNCH( true, false, 1, TBVH_STACK ); else LAUNCH( false, false, 1, TBVH_STACK ); }
	else { if (anyhit) LAUNCH( true, false, 0, TBVH_STACK ); else LAUNCH( false, false, 0, TBVH_STACK ); }
	#undef LAUNCH
	LAUNCHED();
	return TBVH_OK;
}
