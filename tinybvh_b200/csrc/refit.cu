// tinybvh_b200/csrc/refit.cu - BVH::Refit (tiny_bvh.h:3055-3093) on sm_90a: new vertex positions, same topology.
//
// The reference walks the node array backwards (children sit behind their parent): a leaf takes the box of its triangles'
// current vertices, an interior node the union of its two children.  Here: one thread per leaf computes the leaf box in the
// reference's own operation order (min( min( v0, box ), min( v1, v2 ) ) per triangle, :3075-3079), then climbs; at every
// interior node the second arrival (atomic counter) unions the two finished children and carries on, so every node is
// written exactly once and only after both of its children.  Boxes are min / max of inputs, so the result is the
// reference's byte for byte.  Node 1 stays untouched, as in the reference (`if (i != 1)`).
#include "common.cuh"

namespace
{
__device__ __forceinline__ float tmin( const float a, const float b ) { return a < b ? a : b; }   // tinybvh_min :432
__device__ __forceinline__ float tmax( const float a, const float b ) { return a > b ? a : b; }   // tinybvh_max :433

__global__ void k_refit_parents( const float4* __restrict__ nodes, uint32_t* __restrict__ parent, const uint32_t used )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= used || i == 1) return;
	if (i == 0) parent[0] = 0xffffffffu;
	const float4 a = nodes[(size_t)i * 2], b = nodes[(size_t)i * 2 + 1];
	if (__float_as_uint( b.w ) == 0) { const uint32_t l = __float_as_uint( a.w ); parent[l] = parent[l + 1] = i; }
}

__global__ void k_refit( float4* nodes, const uint32_t* __restrict__ prim_idx, const float4* __restrict__ verts, const uint32_t* __restrict__ parent,
	uint32_t* arrive, const uint32_t used )
{
	uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= used || x == 1) return;
	const float4 a = nodes[(size_t)x * 2], b = nodes[(size_t)x * 2 + 1];
	const uint32_t first = __float_as_uint( a.w ), count = __float_as_uint( b.w );
	if (count == 0) return; // interior nodes are written by whichever child arrives second
	float mn[3] = { BVH_FAR, BVH_FAR, BVH_FAR }, mx[3] = { -BVH_FAR, -BVH_FAR, -BVH_FAR };
	for (uint32_t j = 0; j < count; j++)
	{
		const size_t v = (size_t)prim_idx[first + j] * 3;
		const float4 v0 = verts[v], v1 = verts[v + 1], v2 = verts[v + 2];
		mn[0] = tmin( tmin( v0.x, mn[0] ), tmin( v1.x, v2.x ) ), mx[0] = tmax( tmax( v0.x, mx[0] ), tmax( v1.x, v2.x ) );
		mn[1] = tmin( tmin( v0.y, mn[1] ), tmin( v1.y, v2.y ) ), mx[1] = tmax( tmax( v0.y, mx[1] ), tmax( v1.y, v2.y ) );
		mn[2] = tmin( tmin( v0.z, mn[2] ), tmin( v1.z, v2.z ) ), mx[2] = tmax( tmax( v0.z, mx[2] ), tmax( v1.z, v2.z ) );
	}
	nodes[(size_t)x * 2] = make_float4( mn[0], mn[1], mn[2], a.w ), nodes[(size_t)x * 2 + 1] = make_float4( mx[0], mx[1], mx[2], b.w );
	for (;;)
	{
		const uint32_t p = parent[x];
		if (p == 0xffffffffu) break;
		__threadfence();
		if (atomicAdd( &arrive[p], 1u ) == 0) break;
		__threadfence();
		// children were written by other threads: read them past L1 (ld.global.cg)
		const float4 pa = __ldcg( nodes + (size_t)p * 2 ), pb = __ldcg( nodes + (size_t)p * 2 + 1 );
		const uint32_t l = __float_as_uint( pa.w );
		const float4 l0 = __ldcg( nodes + (size_t)l * 2 ), l1 = __ldcg( nodes + (size_t)l * 2 + 1 ), r0 = __ldcg( nodes + (size_t)l * 2 + 2 ), r1 = __ldcg( nodes + (size_t)l * 2 + 3 );
		nodes[(size_t)p * 2] = make_float4( tmin( l0.x, r0.x ), tmin( l0.y, r0.y ), tmin( l0.z, r0.z ), pa.w );
		nodes[(size_t)p * 2 + 1] = make_float4( tmax( l1.x, r1.x ), tmax( l1.y, r1.y ), tmax( l1.z, r1.z ), pb.w );
		x = p;
	}
}
} // namespace

// enqueue BVH::Refit on s (d_verts already holds the new positions).  parent / arrive: `used` words each; parent depends on the
// topology only, so it is filled only when fill_parent (a caller may keep it between refits)
int refit_enqueue( tbvh_bvh b, cudaStream_t s, uint32_t* parent, uint32_t* arrive, bool fill_parent )
{
	const uint32_t used = b->info.used_nodes;
	CUDA_TRY( cudaMemsetAsync( arrive, 0, (size_t)used * 4, s ) );
	if (fill_parent) { k_refit_parents<<<(used + 255) / 256, 256, 0, s>>>( b->d_nodes, parent, used ); LAUNCHED(); }
	k_refit<<<(used + 255) / 256, 256, 0, s>>>( b->d_nodes, b->d_prim_idx, b->d_verts, parent, arrive, used ); LAUNCHED();
	return TBVH_OK;
}

// d_verts already holds the new positions
int refit_launch( tbvh_bvh b, cudaStream_t s )
{
	const uint32_t used = b->info.used_nodes;
	uint32_t* d_parent = 0; uint32_t* d_arrive = 0;
	cudaEvent_t e0 = 0, e1 = 0;
	auto body = [&]() -> int
	{
		CUDA_TRY( cudaMalloc( &d_parent, (size_t)used * 4 ) );
		CUDA_TRY( cudaMalloc( &d_arrive, (size_t)used * 4 ) );
		CUDA_TRY( cudaEventCreate( &e0 ) ); CUDA_TRY( cudaEventCreate( &e1 ) );
		CUDA_TRY( cudaEventRecord( e0, s ) );
		{ const int r = refit_enqueue( b, s, d_parent, d_arrive, true ); if (r != TBVH_OK) return r; }
		CUDA_TRY( cudaEventRecord( e1, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		float ms = 0;
		CUDA_TRY( cudaEventElapsedTime( &ms, e0, e1 ) );
		b->info.build_ms = ms;
		uint32_t rootw[8];
		CUDA_TRY( cudaMemcpy( rootw, b->d_nodes, 32, cudaMemcpyDeviceToHost ) );
		memcpy( b->info.aabb_min, rootw, 12 ), memcpy( b->info.aabb_max, rootw + 4, 12 );
		return TBVH_OK;
	};
	const int rc = body();
	cudaStreamSynchronize( s );
	if (d_parent) cudaFree( d_parent );
	if (d_arrive) cudaFree( d_arrive );
	if (e0) cudaEventDestroy( e0 );
	if (e1) cudaEventDestroy( e1 );
	return rc;
}
