// tinybvh_b200/csrc/refit.cu - BVH::Refit (tiny_bvh.h:3055-3093) on sm_90a: new vertex positions, same topology.
//
// The reference walks the node array backwards (children sit behind their parent): a leaf takes the box of its triangles'
// current vertices, an interior node the union of its two children.  Here: one thread per leaf computes the leaf box in the
// reference's own operation order (min( min( v0, box ), min( v1, v2 ) ) per triangle, :3075-3079), then climbs; at every
// interior node the second arrival (atomic counter) unions the two finished children and carries on, so every node is
// written exactly once and only after both of its children.  Boxes are min / max of inputs, so the result is the
// reference's byte for byte.  Node 1 stays untouched, as in the reference (`if (i != 1)`).
//
// Batches (tbvh_refit_batch; a single refit is K = 1): the K trees share one node index space, tree t owning nodes nbase .. nbase +
// used of it, so one launch and one arrival-counter memset cover them all.  A thread finds its tree in a table (RfTree) and works
// on the tree's own arrays with local node numbers; node 1 is skipped per tree.  A single tree is a one-entry table.
// The driver (refit_trees) is in convert_cwbvh.cu, next to the re-encode of the kept CWBVH collapse.
#include "common.cuh"

namespace
{
__device__ __forceinline__ float tmin( const float a, const float b ) { return a < b ? a : b; }   // tinybvh_min :432
__device__ __forceinline__ float tmax( const float a, const float b ) { return a > b ? a : b; }   // tinybvh_max :433

__global__ void k_refit_parents( const RfTree* __restrict__ T, const uint32_t K, const uint32_t n )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n) return;
	const RfTree& tr = T[batch_entry<RfTree, &RfTree::nbase>( T, K, g )];
	const uint32_t i = g - tr.nbase;
	if (!tr.fill || i == 1) return;
	const float4* __restrict__ nodes = tr.nodes;
	uint32_t* __restrict__ parent = tr.parent;
	if (i == 0) parent[0] = 0xffffffffu;
	const float4 a = nodes[(size_t)i * 2], b = nodes[(size_t)i * 2 + 1];
	if (__float_as_uint( b.w ) == 0) { const uint32_t l = __float_as_uint( a.w ); parent[l] = parent[l + 1] = i; }
}

// leaf x of one tree: its box, then the climb (arrive: the tree's counters)
__device__ __forceinline__ void refit_leaf( float4* nodes, const uint32_t* __restrict__ prim_idx, const float4* __restrict__ verts, const uint32_t* __restrict__ parent,
	uint32_t* arrive, uint32_t x )
{
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

// node g of the batch's node space, in the tree that owns it; arrive: the batch's counters, tree t's from nbase on
__global__ void k_refit( const RfTree* __restrict__ T, const uint32_t K, uint32_t* arrive, const uint32_t n )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n) return;
	const RfTree& tr = T[batch_entry<RfTree, &RfTree::nbase>( T, K, g )];
	const uint32_t x = g - tr.nbase;
	if (x != 1) refit_leaf( tr.nodes, tr.prim_idx, tr.verts, tr.parent, arrive + tr.nbase, x );
}

// the root node of every tree (its box is the handle's aabb), read back with the call's other results
__global__ void k_refit_roots( const RfTree* __restrict__ T, const uint32_t K, uint4* __restrict__ out )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= K) return;
	const uint4* r = (const uint4*)T[t].nodes;
	out[(size_t)t * 2] = r[0], out[(size_t)t * 2 + 1] = r[1];
}
} // namespace

int refit_enqueue( const RfTree* d_T, const uint32_t K, const uint32_t n, uint32_t* arrive, const bool fill, cudaStream_t s )
{
	const uint32_t g = (n + 255) / 256;
	if (fill) { k_refit_parents<<<g, 256, 0, s>>>( d_T, K, n ); LAUNCHED(); }
	k_refit<<<g, 256, 0, s>>>( d_T, K, arrive, n ); LAUNCHED();
	return TBVH_OK;
}

int refit_roots( const RfTree* d_T, const uint32_t K, uint32_t* out, cudaStream_t s )
{
	k_refit_roots<<<(K + 127) / 128, 128, 0, s>>>( d_T, K, (uint4*)out ); LAUNCHED();
	return TBVH_OK;
}
