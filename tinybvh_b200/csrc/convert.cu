// tinybvh_b200/csrc/convert.cu - layout transforms on the device.
//   make_leaf_tris   : primIdx + verts -> leaf-ordered (v0|primIdx, e1, e2) records for BVH2 traversal
//   bvh_gpu_to_bvh   : BVH_GPU (Aila-Laine 64-byte, tiny_bvh.h:1095-1105) -> child-pair traversal array
//   bvh_to_bvh_gpu   : BVH_GPU::ConvertFrom (tiny_bvh.h:4612-4655)
//   bvh_to_cwbvh     : BVH8_CWBVH::Build's conversion chain (tiny_bvh.h:5827-5834)
#include "common.cuh"

// TLAS staleness (api.cu tlas_check): every change of the arrays a TLAS may point at gives the handle a generation no handle has had before
uint32_t tbvh_next_generation()
{
	static std::atomic<uint32_t> counter{ 0 };
	return ++counter;
}

// one thread per primitive reference: 4 B index read + the record (common.cuh leaf_tri_record)
__global__ void k_make_leaf_tris( const float4* __restrict__ verts, const uint32_t* __restrict__ prim_idx, float4* __restrict__ out, const uint32_t idx_count )
{
	const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= idx_count) return;
	leaf_tri_record( verts, __ldg( prim_idx + p ), out, p );
}

int make_leaf_tris( tbvh_bvh b, cudaStream_t s )
{
	const uint32_t n = b->info.idx_count;
	// a refit keeps the array (same idx_count): a TLAS holding its address stays valid
	if (b->d_leaf_tris && b->leaf_tris_count != n) { cudaFree( b->d_leaf_tris ); b->d_leaf_tris = 0; }
	if (!b->d_leaf_tris) { CUDA_TRY( cudaMalloc( &b->d_leaf_tris, (size_t)n * 48 ) ); b->leaf_tris_count = n; b->generation = tbvh_next_generation(); }
	k_make_leaf_tris<<<(n + 255) / 256, 256, 0, s>>>( b->d_verts, b->d_prim_idx, b->d_leaf_tris, n );
	LAUNCHED();
	return TBVH_OK;
}

// one thread per Aila-Laine node i; an interior node writes its children as the pair at slots 2i, 2i+1:
//   {lmin, ref(L), lmax, cnt(L)}, {rmin, ref(R), rmax, cnt(R)},  ref(c) = leaf ? firstTri : 2*c,  cnt(c) = triCount(c)
__global__ void k_bvh_gpu_to_pairs( const float4* __restrict__ g, float4* __restrict__ pairs, const uint32_t used )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= used) return;
	const float4 n0 = g[(size_t)i * 4], n1 = g[(size_t)i * 4 + 1], n2 = g[(size_t)i * 4 + 2], n3 = g[(size_t)i * 4 + 3];
	float4 o0 = make_float4( 0, 0, 0, 0 ), o1 = o0, o2 = o0, o3 = o0;
	if (__float_as_uint( n2.w ) == 0) // interior
	{
		const uint32_t L = __float_as_uint( n0.w ), R = __float_as_uint( n1.w );
		const uint32_t lc = __float_as_uint( g[(size_t)L * 4 + 2].w ), rc = __float_as_uint( g[(size_t)R * 4 + 2].w );
		const uint32_t lr = lc ? __float_as_uint( g[(size_t)L * 4 + 3].w ) : 2 * L, rr = rc ? __float_as_uint( g[(size_t)R * 4 + 3].w ) : 2 * R;
		o0 = make_float4( n0.x, n0.y, n0.z, __uint_as_float( lr ) ), o1 = make_float4( n1.x, n1.y, n1.z, __uint_as_float( lc ) );
		o2 = make_float4( n2.x, n2.y, n2.z, __uint_as_float( rr ) ), o3 = make_float4( n3.x, n3.y, n3.z, __uint_as_float( rc ) );
	}
	pairs[(size_t)i * 4] = o0, pairs[(size_t)i * 4 + 1] = o1, pairs[(size_t)i * 4 + 2] = o2, pairs[(size_t)i * 4 + 3] = o3;
}

int bvh_gpu_to_bvh( tbvh_bvh b, uint32_t used, cudaStream_t s )
{
	float4* pairs = 0;
	CUDA_TRY( cudaMalloc( &pairs, (size_t)used * 64 ) );
	k_bvh_gpu_to_pairs<<<(used + 255) / 256, 256, 0, s>>>( b->d_nodes_gpu, pairs, used );
	LAUNCHED();
	b->d_trav = pairs;
	return TBVH_OK;
}

// ---- BVH -> BVH_GPU (BVH_GPU::ConvertFrom, tiny_bvh.h:4612-4655) --------------------------------------------------
// The reference re-lays the tree out in DFS preorder (node, left subtree, right subtree) with an explicit stack.  Here the preorder
// index of every node comes from subtree sizes (dfs_sizes_up / dfs_rank in common.cuh, shared with BuildHQ's Compact):
//     pre(left) = pre(p) + 1,   pre(right) = pre(p) + 1 + size(left)
// so it depends on the tree's shape alone: neither on the node numbering nor on the order of the leaf ranges in primIdx (a tree
// after BVH::Optimize, or uploaded from elsewhere, has its leaf ranges out of DFS order).
__global__ void k_gpu_parents( const float4* __restrict__ nodes, uint32_t* __restrict__ parent, const uint32_t used )
{
	const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= used || x == 1) return;
	if (x == 0) parent[0] = 0xffffffffu;
	if (__float_as_uint( nodes[(size_t)x * 2 + 1].w ) != 0) return;
	const uint32_t c = __float_as_uint( nodes[(size_t)x * 2].w );
	parent[c] = x, parent[c + 1] = x;
}

// bottom-up from every leaf: interior nodes and leaves per subtree (every leaf weighs 1)
__global__ void k_gpu_sizes( const float4* __restrict__ nodes, const uint32_t* __restrict__ parent, uint32_t* arrive, uint32_t* sub_int, uint32_t* sub_leaves,
	const uint32_t used )
{
	const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= used || x == 1) return;
	if (__float_as_uint( nodes[(size_t)x * 2 + 1].w ) == 0) return; // leaves only
	dfs_sizes_up( nodes, parent, arrive, sub_int, sub_leaves, x, 1u );
}

// one thread per node: its preorder index from its path to the root; an interior node's left child follows it, its right child
// follows the left subtree (sub_int + sub_leaves nodes)
__global__ void k_gpu_emit( const float4* __restrict__ nodes, const uint32_t* __restrict__ parent, const uint32_t* __restrict__ sub_int,
	const uint32_t* __restrict__ sub_leaves, float4* __restrict__ out, const uint32_t used )
{
	const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= used || x == 1) return;
	const float4 a = nodes[(size_t)x * 2], b = nodes[(size_t)x * 2 + 1];
	uint32_t K, L, Kp;
	dfs_rank( nodes, parent, sub_int, sub_leaves, x, K, L, Kp );
	const uint32_t idx = K + L, cnt = __float_as_uint( b.w );
	const float4 z = make_float4( 0, 0, 0, 0 );
	if (cnt)
	{
		out[(size_t)idx * 4] = z, out[(size_t)idx * 4 + 1] = z;
		out[(size_t)idx * 4 + 2] = make_float4( 0, 0, 0, __uint_as_float( cnt ) ), out[(size_t)idx * 4 + 3] = make_float4( 0, 0, 0, a.w );
		return;
	}
	const uint32_t c = __float_as_uint( a.w );
	const float4 l0 = nodes[(size_t)c * 2], l1 = nodes[(size_t)c * 2 + 1], r0 = nodes[(size_t)c * 2 + 2], r1 = nodes[(size_t)c * 2 + 3];
	const uint32_t ridx = idx + 1 + sub_int[c] + sub_leaves[c];
	out[(size_t)idx * 4] = make_float4( l0.x, l0.y, l0.z, __uint_as_float( idx + 1 ) );
	out[(size_t)idx * 4 + 1] = make_float4( l1.x, l1.y, l1.z, __uint_as_float( ridx ) );
	out[(size_t)idx * 4 + 2] = make_float4( r0.x, r0.y, r0.z, __uint_as_float( 0u ) );
	out[(size_t)idx * 4 + 3] = make_float4( r1.x, r1.y, r1.z, __uint_as_float( 0u ) );
}

void drop_bvh_gpu( tbvh_bvh b )
{
	if (b->d_nodes_gpu) cudaFree( b->d_nodes_gpu );
	b->d_nodes_gpu = 0;
	b->info.layouts &= ~(1u << TBVH_LAYOUT_BVH_GPU), b->info.used_nodes_gpu = 0;
}

int bvh_to_bvh_gpu( tbvh_bvh b, cudaStream_t s )
{
	const uint32_t used = b->info.used_nodes;
	drop_bvh_gpu( b );
	uint32_t* w = 0; // workspace: parent, arrive, sub_int, sub_leaves [used]
	const size_t words = (size_t)used * 4;
	auto body = [&]() -> int
	{
		CUDA_TRY( cudaMalloc( &b->d_nodes_gpu, (size_t)used * 64 ) );
		CUDA_TRY( cudaMalloc( &w, words * 4 ) );
		uint32_t* parent = w, * arrive = w + used, * sub_int = arrive + used, * sub_leaves = sub_int + used;
		CUDA_TRY( cudaMemsetAsync( w, 0, words * 4, s ) );
		const uint32_t g = (used + 255) / 256;
		k_gpu_parents<<<g, 256, 0, s>>>( b->d_nodes, parent, used ); LAUNCHED();
		k_gpu_sizes<<<g, 256, 0, s>>>( b->d_nodes, parent, arrive, sub_int, sub_leaves, used ); LAUNCHED();
		k_gpu_emit<<<g, 256, 0, s>>>( b->d_nodes, parent, sub_int, sub_leaves, b->d_nodes_gpu, used ); LAUNCHED();
		CUDA_TRY( cudaStreamSynchronize( s ) );
		return TBVH_OK;
	};
	const int rc = body();
	cudaStreamSynchronize( s );
	cudaFree( w );
	if (rc != TBVH_OK) drop_bvh_gpu( b );
	else b->info.used_nodes_gpu = used - 1, b->info.layouts |= 1u << TBVH_LAYOUT_BVH_GPU; // node 1 of the Wald layout is unused
	return rc;
}

// bvh_to_cwbvh lives in convert_cwbvh.cu
