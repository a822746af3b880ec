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

// one thread per primitive reference: 4 B index read + the record (common.cuh leaf_tri_record).  Reference g of the batch's
// reference space, in the tree that owns it (RfTree::pbase)
__global__ void k_make_leaf_tris( const RfTree* __restrict__ T, const uint32_t K, const uint32_t n )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n) return;
	const RfTree& tr = T[batch_entry<RfTree, &RfTree::pbase>( T, K, g )];
	const uint32_t p = g - tr.pbase;
	leaf_tri_record( tr.verts, __ldg( tr.prim_idx + p ), tr.leaf_tris, p );
}

int leaf_tris_enqueue( const RfTree* d_T, const uint32_t K, const uint32_t n, cudaStream_t s )
{
	k_make_leaf_tris<<<(n + 255) / 256, 256, 0, s>>>( d_T, K, n );
	LAUNCHED();
	return TBVH_OK;
}

int leaf_tris_alloc( tbvh_bvh b )
{
	const uint32_t n = b->info.idx_count;
	// a refit keeps the array (same idx_count): a TLAS holding its address stays valid
	if (b->d_leaf_tris && b->leaf_tris_count == n) return TBVH_OK;
	TRY( b->d_leaf_tris.alloc( (size_t)n * 48 ) );
	b->leaf_tris_count = n, b->generation = tbvh_next_generation();
	return TBVH_OK;
}

int make_leaf_tris( tbvh_bvh b, cudaStream_t s )
{
	TRY( leaf_tris_alloc( b ) );
	// the tree as a one-entry table; an upload synchronises right after, so the table lives for the call only
	RfTree entry = {};
	entry.prim_idx = b->d_prim_idx, entry.verts = b->d_verts, entry.leaf_tris = b->d_leaf_tris;
	Scratch sc( s );
	RfTree* d_T = 0;
	TRY( sc.alloc( d_T, sizeof( RfTree ) ) );
	CUDA_TRY( cudaMemcpyAsync( d_T, &entry, sizeof( RfTree ), cudaMemcpyHostToDevice, s ) );
	TRY( leaf_tris_enqueue( d_T, 1, b->info.idx_count, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
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
	TRY( b->d_pairs.alloc( (size_t)used * 64 ) );
	k_bvh_gpu_to_pairs<<<(used + 255) / 256, 256, 0, s>>>( b->d_nodes_gpu, b->d_pairs, used );
	LAUNCHED();
	return TBVH_OK;
}

// ---- BVH -> BVH_GPU (BVH_GPU::ConvertFrom, tiny_bvh.h:4612-4655) --------------------------------------------------
// The reference re-lays the tree out in DFS preorder (node, left subtree, right subtree) with an explicit stack.  Here the preorder
// index of every node comes from subtree sizes (dfs_sizes_up / dfs_rank in common.cuh, shared with BuildHQ's Compact):
//     pre(left) = pre(p) + 1,   pre(right) = pre(p) + 1 + size(left)
// so it depends on the tree's shape alone: neither on the node numbering nor on the order of the leaf ranges in primIdx (a tree
// after BVH::Optimize, or uploaded from elsewhere, has its leaf ranges out of DFS order).
// Node g of the pass's node space, in the tree that owns it (GpuTree::nbase); the workspace arrays are the pass's, tree t's from nbase
// on, and hold local node numbers.
__global__ void k_gpu_parents( const GpuTree* __restrict__ T, const uint32_t K, uint32_t* __restrict__ parent, const uint32_t n )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n) return;
	const GpuTree& tr = T[batch_entry<GpuTree, &GpuTree::nbase>( T, K, g )];
	const uint32_t x = g - tr.nbase;
	if (x == 1) return;
	const float4* __restrict__ nodes = tr.nodes;
	parent += tr.nbase;
	if (x == 0) parent[0] = 0xffffffffu;
	if (__float_as_uint( nodes[(size_t)x * 2 + 1].w ) != 0) return;
	const uint32_t c = __float_as_uint( nodes[(size_t)x * 2].w );
	parent[c] = x, parent[c + 1] = x;
}

// bottom-up from every leaf: interior nodes and leaves per subtree (every leaf weighs 1)
__global__ void k_gpu_sizes( const GpuTree* __restrict__ T, const uint32_t K, const uint32_t* __restrict__ parent, uint32_t* arrive, uint32_t* sub_int,
	uint32_t* sub_leaves, const uint32_t n )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n) return;
	const GpuTree& tr = T[batch_entry<GpuTree, &GpuTree::nbase>( T, K, g )];
	const uint32_t x = g - tr.nbase;
	if (x == 1) return;
	const float4* __restrict__ nodes = tr.nodes;
	if (__float_as_uint( nodes[(size_t)x * 2 + 1].w ) == 0) return; // leaves only
	parent += tr.nbase, arrive += tr.nbase, sub_int += tr.nbase, sub_leaves += tr.nbase;
	dfs_sizes_up( nodes, parent, arrive, sub_int, sub_leaves, x, 1u );
}

// one thread per node: its preorder index from its path to the root; an interior node's left child follows it, its right child
// follows the left subtree (sub_int + sub_leaves nodes)
__global__ void k_gpu_emit( const GpuTree* __restrict__ T, const uint32_t K, const uint32_t* __restrict__ parent, const uint32_t* __restrict__ sub_int,
	const uint32_t* __restrict__ sub_leaves, const uint32_t n )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n) return;
	const GpuTree& tr = T[batch_entry<GpuTree, &GpuTree::nbase>( T, K, g )];
	const uint32_t x = g - tr.nbase;
	if (x == 1) return;
	const float4* __restrict__ nodes = tr.nodes;
	float4* __restrict__ out = tr.out;
	parent += tr.nbase, sub_int += tr.nbase, sub_leaves += tr.nbase;
	const float4 a = nodes[(size_t)x * 2], b = nodes[(size_t)x * 2 + 1];
	uint32_t Kx, L, Kp;
	dfs_rank( nodes, parent, sub_int, sub_leaves, x, Kx, L, Kp );
	const uint32_t idx = Kx + L, cnt = __float_as_uint( b.w );
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

int bvh_gpu_enqueue( const GpuTree* d_T, const uint32_t K, const uint32_t n, uint32_t* w, cudaStream_t s )
{
	uint32_t* parent = w, * arrive = w + n, * sub_int = arrive + n, * sub_leaves = sub_int + n;
	CUDA_TRY( cudaMemsetAsync( w, 0, (size_t)n * 16, s ) );
	const uint32_t g = (n + 255) / 256;
	k_gpu_parents<<<g, 256, 0, s>>>( d_T, K, parent, n ); LAUNCHED();
	k_gpu_sizes<<<g, 256, 0, s>>>( d_T, K, parent, arrive, sub_int, sub_leaves, n ); LAUNCHED();
	k_gpu_emit<<<g, 256, 0, s>>>( d_T, K, parent, sub_int, sub_leaves, n ); LAUNCHED();
	return TBVH_OK;
}

void drop_bvh_gpu( tbvh_bvh b )
{
	b->d_nodes_gpu.reset();
	b->info.layouts &= ~(1u << TBVH_LAYOUT_BVH_GPU), b->info.used_nodes_gpu = 0;
}

int bvh_to_bvh_gpu( tbvh_bvh b, cudaStream_t s )
{
	const uint32_t used = b->info.used_nodes;
	drop_bvh_gpu( b );
	const size_t words = (size_t)used * 4;
	auto body = [&]() -> int
	{
		GpuTree entry;
		Scratch sc( s );
		TRY( b->d_nodes_gpu.alloc( (size_t)used * 64 ) );
		uint32_t* w = 0; // workspace: parent, arrive, sub_int, sub_leaves [used], then the tree as a one-entry table
		TRY( sc.alloc( w, words * 4 + sizeof( GpuTree ) ) );
		entry = GpuTree{ b->d_nodes, b->d_nodes_gpu, 0, used };
		GpuTree* const d_T = (GpuTree*)(w + words);
		CUDA_TRY( cudaMemcpyAsync( d_T, &entry, sizeof( GpuTree ), cudaMemcpyHostToDevice, s ) );
		TRY( bvh_gpu_enqueue( d_T, 1, used, w, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		return TBVH_OK;
	};
	const int rc = body(); // the stream is drained and the workspace freed before a failure drops the BVH_GPU array
	if (rc != TBVH_OK) drop_bvh_gpu( b );
	else b->info.used_nodes_gpu = used - 1, b->info.layouts |= 1u << TBVH_LAYOUT_BVH_GPU; // node 1 of the Wald layout is unused
	return rc;
}

// bvh_to_cwbvh lives in convert_cwbvh.cu
