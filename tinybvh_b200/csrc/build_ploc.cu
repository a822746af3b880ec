// tinybvh_b200/csrc/build_ploc.cu - TBVH_BUILD_PLOC: BVH construction by parallel locally-ordered clustering on sm_90a
// (Meister & Bittner 2018, "Parallel Locally-Ordered Clustering for Bounding Volume Hierarchy Construction").
//
// The reference has no such builder: the tree is held byte for byte to tests/ploc_oracle.c, which restates the rules of DESIGN.md
// §4.8 sequentially.  Steps, for a batch of K trees in one index space (tree t owns positions tree_base[t] .. tree_base[t+1]):
//   fragments    k_fragments of build_sah.cu (fragments_launch): triangle boxes and each tree's root box as ordered keys
//   Morton       k_morton: 21 bits per axis of the box centroid normalised to the tree's root box; CUB radix sort by code, then
//                (batches) a stable sort by tree, so the order is (tree, code, triangle)
//   clustering   iterations of k_nn (nearest neighbour within +-PLOC_R in the tree's segment), k_flags + exclusive_scan (survivors)
//                and k_compact (mutual pairs merge into a new node record, segments compacted in order).  Iterations are enqueued in
//                groups of PLOC_GROUP; every kernel reads the live count from the device, so iterations past the end cost launches
//                and no work.  One host synchronisation per group.
//   collapse     k_cost: one bottom-up climb with arrival counters; a node becomes one leaf when its leaf cost is not higher than
//                its interior cost and it holds at most PLOC_MAX_LEAF triangles
//   output       k_sizes / k_renumber: dfs_sizes_up / dfs_rank give BVH::ConvertFrom( BVH_Verbose )'s DFS numbering and the
//                primIdx offsets; then refit_enqueue writes every box as BVH::Refit does and leaf_tris_enqueue the traversal records.
// The node records of the temporary tree sit in the reference's layout: tree t's root in slot 2t (2t + 1 unused), and every merge
// owns a slot pair holding its two children, so the numbering helpers of common.cuh walk it as they walk a builder's tree.
#include "common.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>
#include <vector>

#define PLOC_R 16          // search radius (tests/ploc_oracle.c PLOC_R)
#define PLOC_MAX_LEAF 4    // most triangles of a collapsed leaf (tests/ploc_oracle.c PLOC_MAX_LEAF)
#define PLOC_GROUP 8       // clustering iterations enqueued between two reads of the live count

namespace
{
constexpr uint32_t NONE = 0xffffffffu;

__device__ __forceinline__ float tmin( const float a, const float b ) { return a < b ? a : b; }   // tinybvh_min :432
__device__ __forceinline__ float tmax( const float a, const float b ) { return a > b ? a : b; }   // tinybvh_max :433
__device__ __forceinline__ uint32_t first( const float4* r, const uint32_t s ) { return __float_as_uint( r[(size_t)s * 2].w ); }
__device__ __forceinline__ uint32_t count( const float4* r, const uint32_t s ) { return __float_as_uint( r[(size_t)s * 2 + 1].w ); }

// oracle half_area of a record's box
__device__ __forceinline__ float rec_area( const float4 a, const float4 b )
{
	const float ex = __fsub_rn( b.x, a.x ), ey = __fsub_rn( b.y, a.y ), ez = __fsub_rn( b.z, a.z );
	return __fmaf_rn( ez, ex, __fmaf_rn( ey, ex, __fmul_rn( ey, ez ) ) );
}
// ordered key of an area, NaN above +inf
__device__ __forceinline__ uint32_t area_key( const float f ) { return f != f ? 0xffffffffu : f2key( f ); }
__device__ __forceinline__ uint32_t quant( const float c, const float mn, const float ext )
{
	if (!(ext > 0.0f) || !(ext <= 3.40282347e38f)) return 0;
	const float f = __fmul_rn( __fdiv_rn( __fsub_rn( c, mn ), ext ), 2097152.0f );
	if (!(f > 0.0f)) return 0;
	if (f >= 2097151.0f) return 2097151u;
	return __float2uint_rz( f );
}
__device__ __forceinline__ uint64_t spread21( const uint32_t v )
{
	uint64_t x = v & 0x1fffffu;
	x = (x | x << 32) & 0x1f00000000ffffull;
	x = (x | x << 16) & 0x1f0000ff0000ffull;
	x = (x | x << 8) & 0x100f00f00f00f00full;
	x = (x | x << 4) & 0x10c30c30c30c30c3ull;
	x = (x | x << 2) & 0x1249249249249249ull;
	return x;
}
// the entry of T[0 .. K) with T[k] <= g < T[k + 1] (T rises strictly)
__device__ __forceinline__ uint32_t seg_of( const uint32_t* __restrict__ T, const uint32_t K, const uint32_t g )
{
	uint32_t lo = 0, hi = K;
	while (hi - lo > 1) { const uint32_t m = (lo + hi) >> 1; if (T[m] <= g) lo = m; else hi = m; }
	return lo;
}

__global__ void __launch_bounds__( 256 ) k_morton( const float4* __restrict__ fmin_, const float4* __restrict__ fmax_, const uint32_t* __restrict__ base,
	const uint32_t trees, const uint32_t* __restrict__ keys, const uint32_t key_stride, const uint32_t n, uint64_t* __restrict__ code, uint32_t* __restrict__ val )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint32_t* k = keys + (size_t)key_stride * seg_of( base, trees, i );
	const float4 lo = fmin_[i], hi = fmax_[i];
	const float bl[3] = { lo.x, lo.y, lo.z }, bh[3] = { hi.x, hi.y, hi.z };
	uint64_t c = 0;
#pragma unroll
	for (int a = 0; a < 3; a++)
	{
		const float rmn = key2f( k[a] ), rmx = key2f( k[3 + a] );
		c |= spread21( quant( __fmul_rn( __fadd_rn( bl[a], bh[a] ), 0.5f ), rmn, __fsub_rn( rmx, rmn ) ) ) << (2 - a);
	}
	code[i] = c, val[i] = i;
}
__global__ void __launch_bounds__( 256 ) k_tree_keys( const uint32_t* __restrict__ val, const uint32_t* __restrict__ base, const uint32_t trees, const uint32_t n, uint32_t* __restrict__ tkey )
{
	const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p < n) tkey[p] = seg_of( base, trees, val[p] );
}
// the leaf record of every sorted position and the first segments
__global__ void __launch_bounds__( 256 ) k_init_clusters( const uint32_t* __restrict__ val, const float4* __restrict__ fmin_, const float4* __restrict__ fmax_, const uint32_t n,
	float4* __restrict__ cl, const uint32_t* __restrict__ base, uint32_t* __restrict__ seg, const uint32_t trees )
{
	const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p <= trees) seg[p] = base[p];
	if (p >= n) return;
	const uint32_t g = val[p];
	const float4 lo = fmin_[g], hi = fmax_[g];
	cl[(size_t)p * 2] = make_float4( lo.x, lo.y, lo.z, __uint_as_float( p ) ), cl[(size_t)p * 2 + 1] = make_float4( hi.x, hi.y, hi.z, __uint_as_float( 1u ) );
}

// every live cluster's nearest neighbour in its tree's segment: least area key, then least distance, then the local pair partner
// (i ^ 1), then the lower index; the union folds the lower position first
__global__ void __launch_bounds__( 256 ) k_nn( const float4* __restrict__ cl, const uint32_t* __restrict__ seg, const uint32_t trees, uint32_t* __restrict__ nn )
{
	const uint32_t M = seg[trees];
	for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < M; p += gridDim.x * blockDim.x)
	{
		const uint32_t t = seg_of( seg, trees, p ), s = seg[t], m = seg[t + 1] - s, i = p - s;
		if (m == 1) { nn[p] = p; continue; }
		const uint32_t lo = i > PLOC_R ? i - PLOC_R : 0, hi = i + PLOC_R < m - 1 ? i + PLOC_R : m - 1;
		const float4 a = cl[(size_t)p * 2], b = cl[(size_t)p * 2 + 1];
		uint32_t best = NONE, bk = 0, bd = 0, bp = 0;
		for (uint32_t j = lo; j <= hi; j++) if (j != i)
		{
			const float4 c = cl[(size_t)(s + j) * 2], d = cl[(size_t)(s + j) * 2 + 1];
			const bool below = j < i;
			const float4 mn = below ? make_float4( tmin( c.x, a.x ), tmin( c.y, a.y ), tmin( c.z, a.z ), 0 ) : make_float4( tmin( a.x, c.x ), tmin( a.y, c.y ), tmin( a.z, c.z ), 0 );
			const float4 mx = below ? make_float4( tmax( d.x, b.x ), tmax( d.y, b.y ), tmax( d.z, b.z ), 0 ) : make_float4( tmax( b.x, d.x ), tmax( b.y, d.y ), tmax( b.z, d.z ), 0 );
			const uint32_t k = area_key( rec_area( mn, mx ) ), dist = below ? i - j : j - i, par = j == (i ^ 1u) ? 0 : 1;
			if (best == NONE || k < bk || (k == bk && (dist < bd || (dist == bd && par < bp)))) best = j, bk = k, bd = dist, bp = par;
		}
		nn[p] = s + best;
	}
}
// survivors: every cluster but the upper one of a mutual pair; 0 from the live count up to `bound`
__global__ void __launch_bounds__( 256 ) k_flags( const uint32_t* __restrict__ seg, const uint32_t trees, const uint32_t* __restrict__ nn, uint32_t* __restrict__ flags, const uint32_t bound )
{
	const uint32_t M = seg[trees];
	for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < bound; p += gridDim.x * blockDim.x)
	{
		uint32_t f = 0;
		if (p < M) { const uint32_t j = nn[p]; f = !(j < p && nn[j] == p); }
		flags[p] = f;
	}
}
__device__ __forceinline__ void set_parents( const float4 b, const float4 a, uint32_t* parent, const uint32_t slot )
{
	if (__float_as_uint( b.w ) == 0) { const uint32_t l = __float_as_uint( a.w ); parent[l] = parent[l + 1] = slot; }
}
// mutual pairs merge (lower position: left child), survivors move to their compacted place, segment starts follow
__global__ void __launch_bounds__( 256 ) k_compact( const float4* __restrict__ cl, float4* __restrict__ nx, const uint32_t* __restrict__ seg, uint32_t* __restrict__ seg_nx,
	const uint32_t trees, const uint32_t* __restrict__ nn, const uint32_t* __restrict__ scan, float4* __restrict__ pool, uint32_t* __restrict__ parent, uint32_t* pairs )
{
	const uint32_t M = seg[trees], g0 = blockIdx.x * blockDim.x + threadIdx.x, stride = gridDim.x * blockDim.x;
	for (uint32_t t = g0; t <= trees; t += stride) seg_nx[t] = scan[seg[t]];
	for (uint32_t p = g0; p < M; p += stride)
	{
		const uint32_t j = nn[p];
		float4 a = cl[(size_t)p * 2], b = cl[(size_t)p * 2 + 1];
		if (j != p && nn[j] == p)
		{
			if (j < p) continue;
			const float4 c = cl[(size_t)j * 2], d = cl[(size_t)j * 2 + 1];
			const uint32_t P = trees + atomicAdd( pairs, 1u );
			pool[(size_t)P * 4] = a, pool[(size_t)P * 4 + 1] = b, pool[(size_t)P * 4 + 2] = c, pool[(size_t)P * 4 + 3] = d;
			set_parents( b, a, parent, 2 * P ), set_parents( d, c, parent, 2 * P + 1 );
			a = make_float4( tmin( a.x, c.x ), tmin( a.y, c.y ), tmin( a.z, c.z ), __uint_as_float( 2 * P ) );
			b = make_float4( tmax( b.x, d.x ), tmax( b.y, d.y ), tmax( b.z, d.z ), __uint_as_float( 0u ) );
		}
		const uint32_t q = scan[p];
		nx[(size_t)q * 2] = a, nx[(size_t)q * 2 + 1] = b;
	}
}
// every tree's last cluster becomes its root, slot 2t
__global__ void k_roots( const float4* __restrict__ cl, const uint32_t trees, float4* __restrict__ pool, uint32_t* __restrict__ parent )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= trees) return;
	const float4 a = cl[(size_t)t * 2], b = cl[(size_t)t * 2 + 1];
	pool[(size_t)t * 4] = a, pool[(size_t)t * 4 + 1] = b, pool[(size_t)t * 4 + 2] = pool[(size_t)t * 4 + 3] = make_float4( 0, 0, 0, 0 );
	parent[2 * t] = parent[2 * t + 1] = NONE;
	set_parents( b, a, parent, 2 * t );
}

// collapse: from every leaf record up, the second arrival at a node decides it (sah_rec's leaf and interior costs)
__global__ void __launch_bounds__( 256 ) k_cost( const float4* __restrict__ pool, const uint32_t* __restrict__ parent, uint32_t* arrive, uint32_t* cnt, float* cost,
	uint32_t* coll, const uint32_t slots, const float c_trav, const float c_int )
{
	uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= slots || count( pool, x ) != 1) return;
	cnt[x] = 1, coll[x] = 0, cost[x] = __fmul_rn( __fmul_rn( c_int, rec_area( pool[(size_t)x * 2], pool[(size_t)x * 2 + 1] ) ), 1.0f );
	for (;;)
	{
		const uint32_t p = parent[x];
		if (p == NONE) break;
		__threadfence();
		if (atomicAdd( &arrive[p], 1u ) == 0) break;
		__threadfence();
		const volatile uint32_t* vc = cnt; const volatile float* vf = cost;
		const uint32_t l = first( pool, p ), N = vc[l] + vc[l + 1];
		const float A = rec_area( pool[(size_t)p * 2], pool[(size_t)p * 2 + 1] );
		const float leafc = __fmul_rn( __fmul_rn( c_int, A ), (float)N ), intc = __fadd_rn( __fadd_rn( __fmul_rn( c_trav, A ), vf[l] ), vf[l + 1] );
		const bool col = N <= PLOC_MAX_LEAF && leafc <= intc;
		cnt[p] = N, cost[p] = col ? leafc : intc, coll[p] = col;
		x = p;
	}
}
// a slot of the output tree: a used slot with no collapsed ancestor (collapses hold at most PLOC_MAX_LEAF triangles, so the walk up
// stops at the first ancestor with more)
__device__ __forceinline__ bool kept( const uint32_t* __restrict__ parent, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ coll, const uint32_t trees, const uint32_t s )
{
	if (s < 2 * trees && (s & 1)) return false;
	for (uint32_t x = parent[s]; x != NONE && cnt[x] <= PLOC_MAX_LEAF; x = parent[x]) if (coll[x]) return false;
	return true;
}
__device__ __forceinline__ bool is_leaf( const float4* pool, const uint32_t* coll, const uint32_t s ) { return count( pool, s ) == 1 || coll[s]; }

__global__ void __launch_bounds__( 256 ) k_sizes( const float4* __restrict__ pool, const uint32_t* __restrict__ parent, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ coll,
	uint32_t* arrive, uint32_t* sub_int, uint32_t* sub_w, const uint32_t slots, const uint32_t trees )
{
	const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s >= slots || !is_leaf( pool, coll, s ) || !kept( parent, cnt, coll, trees, s )) return;
	dfs_sizes_up( pool, parent, arrive, sub_int, sub_w, s, cnt[s] );
}

struct PlocOut { float4* nodes; uint32_t* prim_idx; uint32_t base; };

__global__ void __launch_bounds__( 256 ) k_renumber( const float4* __restrict__ pool, const uint32_t* __restrict__ parent, const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ coll,
	const uint32_t* __restrict__ sub_int, const uint32_t* __restrict__ sub_w, const uint32_t* __restrict__ val, const PlocOut* __restrict__ io, uint32_t* depth,
	const uint32_t slots, const uint32_t trees )
{
	const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
	if (s >= slots || !kept( parent, cnt, coll, trees, s )) return;
	uint32_t K, O, Kp;
	const uint32_t root = dfs_rank( pool, parent, sub_int, sub_w, s, K, O, Kp );
	const PlocOut o = io[root >> 1];
	uint32_t at = 0;
	if (s != root) { const uint32_t p = parent[s]; at = 2 + 2 * (K - Kp) + (s == first( pool, p ) + 1 ? 1 : 0); }
	float4 a = pool[(size_t)s * 2], b = pool[(size_t)s * 2 + 1];
	if (is_leaf( pool, coll, s ))
	{
		a.w = __uint_as_float( O ), b.w = __uint_as_float( cnt[s] );
		// the subtree's triangles in DFS order, left first
		uint32_t st[PLOC_MAX_LEAF], sp = 0, w = O;
		st[sp++] = s;
		while (sp)
		{
			const uint32_t x = st[--sp];
			if (count( pool, x ) == 1) { o.prim_idx[w++] = val[first( pool, x )] - o.base; continue; }
			const uint32_t l = first( pool, x );
			st[sp++] = l + 1, st[sp++] = l;
		}
		uint32_t d = 0;
		for (uint32_t x = s; x != root; x = parent[x]) d++;
		atomicMax( &depth[root >> 1], d );
	}
	else a.w = __uint_as_float( 2 + 2 * K ), b.w = __uint_as_float( 0u );
	o.nodes[(size_t)at * 2] = a, o.nodes[(size_t)at * 2 + 1] = b;
	if (s == root) o.nodes[2] = o.nodes[3] = make_float4( 0, 0, 0, 0 ); // node 1, unused (:2285)
}
} // namespace

// A CUB radix sort on s.  Its kernel launches are counted exactly (g_tbvh_launches): the same call is first captured into a graph
// that is never launched, and its kernel nodes are counted; then it is enqueued.
template <class Sort> static int sort_enqueue( cudaStream_t s, Sort sort )
{
	cudaGraph_t g = 0;
	CUDA_TRY( cudaStreamBeginCapture( s, cudaStreamCaptureModeRelaxed ) );
	const cudaError_t e = sort(), e2 = cudaStreamEndCapture( s, &g );
	size_t count = 0, kernels = 0;
	if (e == cudaSuccess && e2 == cudaSuccess && cudaGraphGetNodes( g, 0, &count ) == cudaSuccess)
	{
		std::vector<cudaGraphNode_t> nodes( count );
		cudaGraphGetNodes( g, nodes.data(), &count );
		for (cudaGraphNode_t x : nodes) { cudaGraphNodeType t; if (cudaGraphNodeGetType( x, &t ) == cudaSuccess && t == cudaGraphNodeTypeKernel) kernels++; }
	}
	if (g) cudaGraphDestroy( g );
	CUDA_TRY( e );
	CUDA_TRY( e2 );
	CUDA_TRY( sort() );
	g_tbvh_launches += kernels;
	return TBVH_OK;
}

int build_ploc_launch( const tbvh_bvh* bs, const uint32_t trees, const float c_trav, const float c_int, BuiltTree* out, float* ms )
{
	const tbvh_ctx ctx = bs[0]->ctx;
	cudaStream_t s = ctx->stream;
	std::vector<uint32_t> base( (size_t)trees + 1, 0 );
	for (uint32_t t = 0; t < trees; t++) base[t + 1] = base[t] + bs[t]->info.prim_count;
	const uint32_t n = base[trees], slots = 2 * n;
	for (uint32_t t = 0; t < trees; t++)
	{
		const tbvh_bvh b = bs[t];
		const size_t nt = b->info.prim_count;
		TRY( b->d_nodes.alloc( (2 * nt + 2) * 32 ) );
		TRY( b->d_prim_idx.alloc( nt * 4 ) );
		TRY( b->d_leaf_tris.alloc( nt * 48 ) );
		b->leaf_tris_count = (uint32_t)nt;
	}
	Scratch sc( s );
	uint32_t* h_res = 0;
	uint32_t* d_base = 0, * seg[2] = {}, * nn = 0, * flags = 0, * scan = 0, * tile = 0, * pairs = 0, * parent = 0, * arrive = 0, * cnt = 0, * coll = 0, * sub_int = 0, * sub_w = 0, * depth = 0;
	uint32_t* val[2] = {}, * tkey[2] = {};
	uint64_t* code[2] = {};
	float4* fmin_ = 0, * fmax_ = 0, * cl[2] = {}, * pool = 0;
	float* cost = 0;
	PlocOut* d_io = 0;
	TRY( sc.alloc( d_base, base.size() * 4 ) );
	TRY( sc.alloc( fmin_, (size_t)n * 16 ) ); TRY( sc.alloc( fmax_, (size_t)n * 16 ) );
	for (int k = 0; k < 2; k++) { TRY( sc.alloc( code[k], (size_t)n * 8 ) ); TRY( sc.alloc( val[k], (size_t)n * 4 ) ); TRY( sc.alloc( cl[k], (size_t)n * 32 ) ); TRY( sc.alloc( seg[k], ((size_t)trees + 1) * 4 ) ); }
	if (trees > 1) for (int k = 0; k < 2; k++) TRY( sc.alloc( tkey[k], (size_t)n * 4 ) );
	TRY( sc.alloc( nn, (size_t)n * 4 ) ); TRY( sc.alloc( flags, ((size_t)n + 1) * 4 ) ); TRY( sc.alloc( scan, ((size_t)n + 1) * 4 ) ); TRY( sc.alloc( tile, ((size_t)n / 2048 + 2) * 4 ) );
	TRY( sc.alloc( pairs, 4 ) ); TRY( sc.alloc( pool, (size_t)slots * 32 ) ); TRY( sc.alloc( parent, (size_t)slots * 4 ) ); TRY( sc.alloc( arrive, (size_t)slots * 4 ) );
	TRY( sc.alloc( cnt, (size_t)slots * 4 ) ); TRY( sc.alloc( coll, (size_t)slots * 4 ) ); TRY( sc.alloc( cost, (size_t)slots * 4 ) );
	TRY( sc.alloc( sub_int, (size_t)slots * 4 ) ); TRY( sc.alloc( sub_w, (size_t)slots * 4 ) ); TRY( sc.alloc( depth, (size_t)trees * 4 ) ); TRY( sc.alloc( d_io, (size_t)trees * sizeof( PlocOut ) ) );
	TRY( sc.alloc_host( h_res, ((size_t)trees * 2 + 2) * 4 ) );
	TRY( sc.events() );
	std::vector<PlocOut> io( trees );
	for (uint32_t t = 0; t < trees; t++) io[t] = PlocOut{ bs[t]->d_nodes, bs[t]->d_prim_idx, base[t] };
	CUDA_TRY( cudaEventRecord( sc.e0, s ) );
	CUDA_TRY( cudaMemcpyAsync( d_base, base.data(), base.size() * 4, cudaMemcpyHostToDevice, s ) );
	CUDA_TRY( cudaMemcpyAsync( d_io, io.data(), io.size() * sizeof( PlocOut ), cudaMemcpyHostToDevice, s ) );
	// fragments and Morton order
	const uint32_t* keys = 0;
	uint32_t key_stride = 0;
	TRY( fragments_launch( bs, trees, d_base, n, fmin_, fmax_, &keys, &key_stride, sc ) );
	const uint32_t g = (n + 255) / 256;
	k_morton<<<g, 256, 0, s>>>( fmin_, fmax_, d_base, trees, keys, key_stride, n, code[0], val[0] ); LAUNCHED();
	size_t tb = 0, tb2 = 0;
	CUDA_TRY( cub::DeviceRadixSort::SortPairs( (void*)0, tb, code[0], code[1], val[0], val[1], (int)n, 0, 63, s ) );
	int tree_bits = 0;
	while (tree_bits < 32 && (1ull << tree_bits) < trees) tree_bits++;
	if (trees > 1) CUDA_TRY( cub::DeviceRadixSort::SortPairs( (void*)0, tb2, tkey[0], tkey[1], val[1], val[0], (int)n, 0, tree_bits, s ) );
	void* temp = 0;
	TRY( sc.alloc( temp, std::max( tb, tb2 ) ) );
	TRY( sort_enqueue( s, [&]() { return cub::DeviceRadixSort::SortPairs( temp, tb, code[0], code[1], val[0], val[1], (int)n, 0, 63, s ); } ) );
	const uint32_t* order = val[1];
	if (trees > 1)
	{
		k_tree_keys<<<g, 256, 0, s>>>( val[1], d_base, trees, n, tkey[0] ); LAUNCHED();
		tb2 = std::max( tb, tb2 );
		TRY( sort_enqueue( s, [&]() { return cub::DeviceRadixSort::SortPairs( temp, tb2, tkey[0], tkey[1], val[1], val[0], (int)n, 0, tree_bits, s ); } ) );
		order = val[0];
	}
	k_init_clusters<<<(std::max( n, trees + 1 ) + 255) / 256, 256, 0, s>>>( order, fmin_, fmax_, n, cl[0], d_base, seg[0], trees ); LAUNCHED();
	CUDA_TRY( cudaMemsetAsync( pairs, 0, 4, s ) );
	// clustering, PLOC_GROUP iterations per host round trip
	uint32_t live = n, par = 0;
	while (live > trees)
	{
		const uint32_t bound = live, grid = std::min( (bound + 255) / 256, (uint32_t)ctx->sm_count * 8 );
		for (int it = 0; it < PLOC_GROUP; it++, par ^= 1)
		{
			k_nn<<<grid, 256, 0, s>>>( cl[par], seg[par], trees, nn ); LAUNCHED();
			k_flags<<<grid, 256, 0, s>>>( seg[par], trees, nn, flags, bound ); LAUNCHED();
			TRY( exclusive_scan( flags, scan, tile, bound, s ) );
			k_compact<<<grid, 256, 0, s>>>( cl[par], cl[par ^ 1], seg[par], seg[par ^ 1], trees, nn, scan, pool, parent, pairs ); LAUNCHED();
		}
		CUDA_TRY( cudaMemcpyAsync( h_res, seg[par] + trees, 4, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		// every iteration over a tree of two or more clusters merges a pair
		if (h_res[0] >= live) { tbvh_set_error( "build (PLOC): the clustering stopped merging" ); return TBVH_E_LIMIT; }
		live = h_res[0];
	}
	k_roots<<<(trees + 127) / 128, 128, 0, s>>>( cl[par], trees, pool, parent ); LAUNCHED();
	// collapse, numbering, primIdx
	const uint32_t gs = (slots + 255) / 256;
	CUDA_TRY( cudaMemsetAsync( arrive, 0, (size_t)slots * 4, s ) );
	k_cost<<<gs, 256, 0, s>>>( pool, parent, arrive, cnt, cost, coll, slots, c_trav, c_int ); LAUNCHED();
	CUDA_TRY( cudaMemsetAsync( arrive, 0, (size_t)slots * 4, s ) );
	k_sizes<<<gs, 256, 0, s>>>( pool, parent, cnt, coll, arrive, sub_int, sub_w, slots, trees ); LAUNCHED();
	CUDA_TRY( cudaMemsetAsync( depth, 0, (size_t)trees * 4, s ) );
	k_renumber<<<gs, 256, 0, s>>>( pool, parent, cnt, coll, sub_int, sub_w, order, d_io, depth, slots, trees ); LAUNCHED();
	CUDA_TRY( cudaMemcpy2DAsync( h_res, 4, sub_int, 8, 4, trees, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaMemcpyAsync( h_res + trees, depth, (size_t)trees * 4, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	// boxes as BVH::Refit computes them, and the traversal records
	std::vector<RfTree> T( trees );
	uint32_t nodes_total = 0;
	for (uint32_t t = 0; t < trees; t++)
	{
		const tbvh_bvh b = bs[t];
		const uint32_t used = 2 + 2 * h_res[t];
		T[t] = RfTree{ b->d_nodes, b->d_prim_idx, b->d_verts, b->d_leaf_tris, parent + nodes_total, nodes_total, used, base[t], b->info.prim_count, 1 };
		out[t].used_nodes = used, out[t].idx_count = b->info.prim_count, out[t].max_depth = h_res[trees + t];
		nodes_total += used;
	}
	RfTree* d_T = 0;
	uint32_t* roots = 0;
	TRY( sc.alloc( d_T, (size_t)trees * sizeof( RfTree ) ) ); TRY( sc.alloc( roots, (size_t)trees * 32 ) );
	CUDA_TRY( cudaMemcpyAsync( d_T, T.data(), T.size() * sizeof( RfTree ), cudaMemcpyHostToDevice, s ) );
	CUDA_TRY( cudaMemsetAsync( arrive, 0, (size_t)nodes_total * 4, s ) );
	TRY( refit_enqueue( d_T, trees, nodes_total, arrive, true, s ) );
	TRY( leaf_tris_enqueue( d_T, trees, n, s ) );
	CUDA_TRY( cudaEventRecord( sc.e1, s ) );
	TRY( refit_roots( d_T, trees, roots, s ) );
	std::vector<uint32_t> rootw( (size_t)trees * 8 );
	CUDA_TRY( cudaMemcpyAsync( rootw.data(), roots, rootw.size() * 4, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	CUDA_TRY( cudaEventElapsedTime( ms, sc.e0, sc.e1 ) );
	for (uint32_t t = 0; t < trees; t++) memcpy( out[t].root, rootw.data() + (size_t)t * 8, 32 );
	return TBVH_OK;
}
