// tinybvh_b200/csrc/optimize.cu - tbvh_optimize on sm_90a: rounds of parallel subtree reinsertion that lower a resident tree's SAH cost.
//
// The reference's optimiser (BVH::Optimize :3043 over BVH_Verbose::Optimize :4338) reinserts one subtree at a time.  This is the
// parallel form (Meister & Bittner 2018): in each round every node searches the round's tree for the place where it would cost
// least, the moves whose node sets do not overlap are applied together, and the round is kept only if SAHCost falls.  The rules are
// DESIGN.md §4.7; tests/optimize_oracle.c restates them on the host and the result must equal it byte for byte, so every float
// operation that decides a move or the acceptance is written with explicit rounding (no contraction).
//
// The tree stays in the reference's node layout (children paired at leftFirst, node 1 unused) in a scratch copy: a move copies four
// node records between the slots it owns, so a node is named by its slot.  One round is eight launches and one host synchronisation
// (moves, cost, depth); a rejected round retries with the better half of its moves.  At the end the tree is renumbered to
// BVH::ConvertFrom( BVH_Verbose )'s DFS order with dfs_sizes_up / dfs_rank (common.cuh).
#include "common.cuh"
#include <algorithm>

namespace
{
constexpr uint32_t NONE = 0xffffffffu;
constexpr uint32_t OPT_VISITS = 2048;   // stack pops per search (tests/optimize_oracle.c OPT_VISITS)
constexpr uint32_t OPT_STACK = 258;     // the search's stack: depth <= 255 during the rounds, one pending sibling per level + 2

struct Box { float mn[3], mx[3]; };
struct OptRes { uint32_t moves, height, interior, pad; float sah, pad2[3]; };

__device__ __forceinline__ float tmin( const float a, const float b ) { return a < b ? a : b; }   // tinybvh_min :432
__device__ __forceinline__ float tmax( const float a, const float b ) { return a > b ? a : b; }   // tinybvh_max :433
// BVHBase::SA :8477 in tbvh_sah_cost's pairing
__device__ __forceinline__ float box_sa( const Box& b )
{
	const float ex = __fsub_rn( b.mx[0], b.mn[0] ), ey = __fsub_rn( b.mx[1], b.mn[1] ), ez = __fsub_rn( b.mx[2], b.mn[2] );
	return fmaf( ez, ex, fmaf( ey, ex, __fmul_rn( ey, ez ) ) );
}
__device__ __forceinline__ Box fold( const Box& a, const Box& b )
{
	Box r;
#pragma unroll
	for (int k = 0; k < 3; k++) r.mn[k] = tmin( a.mn[k], b.mn[k] ), r.mx[k] = tmax( a.mx[k], b.mx[k] );
	return r;
}
__device__ __forceinline__ Box node_box( const float4* nd, const uint32_t i )
{
	const float4 a = __ldcg( nd + (size_t)i * 2 ), b = __ldcg( nd + (size_t)i * 2 + 1 );
	return Box{ { a.x, a.y, a.z }, { b.x, b.y, b.z } };
}
__device__ __forceinline__ uint32_t first( const float4* nd, const uint32_t i ) { return __float_as_uint( __ldcg( nd + (size_t)i * 2 ).w ); }
__device__ __forceinline__ uint32_t count( const float4* nd, const uint32_t i ) { return __float_as_uint( __ldcg( nd + (size_t)i * 2 + 1 ).w ); }
// N's sibling: the other slot of its parent's child pair
__device__ __forceinline__ uint32_t sibling( const float4* nd, const uint32_t P, const uint32_t N ) { return first( nd, P ) == N ? N + 1 : N - 1; }

// every slot's parent (NONE for the root); every slot but 1 is in the tree
__global__ void k_opt_parents( const float4* __restrict__ nd, uint32_t* __restrict__ parent, const uint32_t n )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n || i == 1) return;
	if (i == 0) parent[0] = NONE;
	if (count( nd, i ) == 0) { const uint32_t l = first( nd, i ); parent[l] = parent[l + 1] = i; }
}

// refold + SAH + height in one climb from every leaf, as refit.cu climbs (the second arrival at a node folds its two finished
// children); leaf boxes are kept (an SBVH's are clipped).  cost: sah_rec's value per node in its operation order (api.cu); the
// thread that finishes the root writes SAHCost and the depth to res.
__global__ void k_opt_climb( float4* nd, const uint32_t* __restrict__ parent, uint32_t* arrive, float* area, float* cost, uint32_t* height,
	const float c_trav, const float c_int, OptRes* res, const uint32_t n )
{
	uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= n || x == 1) return;
	const uint32_t cnt = count( nd, x );
	if (cnt == 0) return;
	const float a = box_sa( node_box( nd, x ) );
	area[x] = a, cost[x] = __fmul_rn( __fmul_rn( c_int, a ), __uint2float_rn( cnt ) ), height[x] = 0;
	float sa = a;
	for (;;)
	{
		const uint32_t p = parent[x];
		if (p == NONE) break;
		__threadfence();
		if (atomicAdd( &arrive[p], 1u ) == 0) break;
		__threadfence();
		const uint32_t l = first( nd, p );
		const Box b = fold( node_box( nd, l ), node_box( nd, l + 1 ) );
		const float4 pa = nd[(size_t)p * 2], pb = nd[(size_t)p * 2 + 1];
		nd[(size_t)p * 2] = make_float4( b.mn[0], b.mn[1], b.mn[2], pa.w ), nd[(size_t)p * 2 + 1] = make_float4( b.mx[0], b.mx[1], b.mx[2], pb.w );
		const volatile float* vc = cost; const volatile uint32_t* vh = height;
		sa = box_sa( b );
		area[p] = sa, cost[p] = __fadd_rn( __fadd_rn( __fmul_rn( c_trav, sa ), vc[l] ), vc[l + 1] ), height[p] = 1 + max( vh[l], vh[l + 1] );
		x = p;
	}
	if (x == 0) // the root's climb (a leaf root never reaches this kernel)
	{
		const volatile float* vc = cost; const volatile uint32_t* vh = height;
		res->sah = __fdiv_rn( vc[0], sa ), res->height = vh[0]; // the root divides by its own area (:1896)
	}
}

__global__ void k_opt_depth( const uint32_t* __restrict__ parent, uint32_t* __restrict__ depth, const uint32_t n )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n || i == 1) return;
	uint32_t d = 0;
	for (uint32_t q = parent[i]; q != NONE; q = parent[q]) d++;
	depth[i] = d;
}

// step 2: node N's best target X (NONE: no place beats its own), branch-and-bound from the root, left child first
__global__ void __launch_bounds__( 128 ) k_opt_search( const float4* __restrict__ nd, const uint32_t* __restrict__ parent, const uint32_t* __restrict__ depth,
	const uint32_t* __restrict__ height, const float* __restrict__ area, uint32_t* __restrict__ cand, const uint32_t L, const uint32_t n )
{
	const uint32_t N = blockIdx.x * blockDim.x + threadIdx.x;
	if (N >= n) return;
	if (N < 2) { cand[N] = NONE; return; }
	const uint32_t P = parent[N], S = sibling( nd, P, N );
	const Box bN = node_box( nd, N );
	const float aN = area[N];
	const uint32_t hN = height[N];
	float best = area[P]; // the induced cost of N's own place: A( S u N ), and no ancestor grows
	uint32_t bestX = NONE, sp = 0, visits = 0;
	uint32_t st[OPT_STACK];
	float sc[OPT_STACK];
	st[sp] = 0, sc[sp++] = 0.0f;
	while (sp > 0 && visits < OPT_VISITS)
	{
		visits++;
		const uint32_t x = st[--sp];
		const float ci = sc[sp];
		if (x == N) continue;
		if (!(__fadd_rn( ci, aN ) < best)) continue;
		const float aU = box_sa( fold( node_box( nd, x ), bN ) );
		if (x != P && x != S && depth[x] + 1 + hN <= L)
		{
			const float c = __fadd_rn( ci, aU );
			if (c < best) best = c, bestX = x;
		}
		if (count( nd, x ) == 0)
		{
			const float ci2 = __fadd_rn( ci, __fsub_rn( aU, area[x] ) );
			const uint32_t l = first( nd, x );
			st[sp] = l + 1, sc[sp++] = ci2;
			st[sp] = l, sc[sp++] = ci2;
		}
	}
	cand[N] = bestX;
}

// the six nodes whose links a move N -> next to X changes: N, P, S, G, X and X's parent (NONE where absent)
__device__ __forceinline__ void move_nodes( const float4* nd, const uint32_t* parent, const uint32_t N, const uint32_t X, uint32_t v[6] )
{
	const uint32_t P = parent[N];
	v[0] = N, v[1] = P, v[2] = sibling( nd, P, N ), v[3] = parent[P], v[4] = X, v[5] = parent[X];
}

// step 3: c_trav x the area the move saves on the round's tree (tests/optimize_oracle.c area_saved, line for line); a finite gain
// > 0 makes the move a candidate with key (gain bits, N), claimed on its six nodes with atomicMax
__global__ void k_opt_gain( const float4* __restrict__ nd, const uint32_t* __restrict__ par, const uint32_t* __restrict__ dep, const float* __restrict__ area,
	const uint32_t* __restrict__ cand, unsigned long long* __restrict__ key, unsigned long long* lock, const float c_trav, const uint32_t n )
{
	const uint32_t N = blockIdx.x * blockDim.x + threadIdx.x;
	if (N >= n) return;
	key[N] = 0;
	const uint32_t X = cand[N];
	if (N < 2 || X == NONE) return;
	const uint32_t P = par[N], S = sibling( nd, P, N ), G = par[P], PX = par[X];
	int dM = -1; // M: the deepest common ancestor of X's parent and G (X the root: above it)
	if (G != NONE && PX != NONE)
	{
		uint32_t a = PX, b = G;
		while (dep[a] > dep[b]) a = par[a];
		while (dep[b] > dep[a]) b = par[b];
		while (a != b) a = par[a], b = par[b];
		dM = (int)dep[a];
	}
	float s = 0.0f;
	uint32_t J = NONE; // the node of G's path just below M, and its box without N
	Box bJ = node_box( nd, 0 );
	if (G != NONE) // climb 1: the removal
	{
		uint32_t q = G, came = P;
		Box cb = node_box( nd, S );
		while (q != NONE && (int)dep[q] > dM)
		{
			const uint32_t l = first( nd, q );
			const Box nb = fold( l == came ? cb : node_box( nd, l ), l + 1 == came ? cb : node_box( nd, l + 1 ) );
			s = __fadd_rn( s, __fsub_rn( area[q], box_sa( nb ) ) );
			if ((int)dep[q] == dM + 1) J = q, bJ = nb;
			came = q, cb = nb, q = par[q];
		}
	}
	Box cb = fold( X == J ? bJ : node_box( nd, X ), node_box( nd, N ) );
	s = __fadd_rn( s, __fsub_rn( area[P], box_sa( cb ) ) );
	uint32_t came = X;
	for (uint32_t q = PX; q != NONE; q = q == S ? G : par[q]) // climb 2: the insertion
	{
		uint32_t l = first( nd, q ), r = l + 1;
		if (l == P) l = S;
		if (r == P) r = S;
		const Box lb = l == came ? cb : l == J ? bJ : node_box( nd, l ), rb = r == came ? cb : r == J ? bJ : node_box( nd, r );
		const Box nb = fold( lb, rb );
		s = __fadd_rn( s, __fsub_rn( area[q], box_sa( nb ) ) );
		came = q, cb = nb;
	}
	const float g = __fmul_rn( c_trav, s );
	if (!(g > 0.0f && g <= 3.40282347e38f)) return;
	const unsigned long long k = ((unsigned long long)__float_as_uint( g ) << 32) | N;
	key[N] = k;
	uint32_t v[6];
	move_nodes( nd, par, N, X, v );
	for (int j = 0; j < 6; j++) if (v[j] != NONE) atomicMax( lock + v[j], k );
}

// step 4a: a candidate wins when it holds all six of its claims
__global__ void k_opt_claim( const float4* __restrict__ nd, const uint32_t* __restrict__ par, const uint32_t* __restrict__ cand, const unsigned long long* __restrict__ key,
	const unsigned long long* __restrict__ lock, uint32_t* __restrict__ won, const uint32_t n )
{
	const uint32_t N = blockIdx.x * blockDim.x + threadIdx.x;
	if (N >= n) return;
	const unsigned long long k = key[N];
	uint32_t w = 0;
	if (k)
	{
		uint32_t v[6];
		move_nodes( nd, par, N, cand[N], v );
		w = 1;
		for (int j = 0; j < 6; j++) if (v[j] != NONE && lock[v[j]] != k) w = 0;
	}
	won[N] = w;
}

// step 4b: a winner is dropped when another winner's N lies on the path from its X to the root; the others are listed
__global__ void k_opt_cross( const uint32_t* __restrict__ par, const uint32_t* __restrict__ cand, const uint32_t* __restrict__ won, uint32_t* __restrict__ list,
	OptRes* res, const uint32_t n )
{
	const uint32_t N = blockIdx.x * blockDim.x + threadIdx.x;
	if (N >= n || !won[N]) return;
	for (uint32_t y = cand[N]; y != NONE; y = par[y]) if (y != N && won[y]) return;
	list[atomicAdd( &res->moves, 1u )] = N;
}

// the keep-th largest key of the listed moves (keys are distinct: they end in N), by one bit at a time from the top
__global__ void k_opt_select( const uint32_t* __restrict__ list, const unsigned long long* __restrict__ key, const uint32_t m, const uint32_t keep,
	unsigned long long* thr )
{
	__shared__ uint32_t total;
	unsigned long long t = 0;
	for (int bit = 63; bit >= 0; bit--)
	{
		const unsigned long long c = t | (1ull << bit);
		if (threadIdx.x == 0) total = 0;
		__syncthreads();
		uint32_t k = 0;
		for (uint32_t i = threadIdx.x; i < m; i += blockDim.x) k += key[list[i]] >= c;
		k = __reduce_add_sync( 0xffffffffu, k );
		if ((threadIdx.x & 31) == 0) atomicAdd( &total, k );
		__syncthreads();
		if (total >= keep) t = c;
		__syncthreads();
	}
	if (threadIdx.x == 0) *thr = t;
}

// step 5: the listed moves with key >= *thr, each on the four slots it owns: S's record into P's slot, P' = (X, N) into X's slot,
// X and N into P's child pair
__global__ void k_opt_apply( float4* nd, const uint32_t* __restrict__ par, const uint32_t* __restrict__ cand, const unsigned long long* __restrict__ key,
	const uint32_t* __restrict__ list, const OptRes* res, const unsigned long long* thr )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= res->moves) return;
	const uint32_t N = list[i];
	if (key[N] < *thr) return;
	const uint32_t X = cand[N], P = par[N], c = first( nd, P ), S = c == N ? N + 1 : N - 1;
	float4* r = nd;
	const float4 s0 = r[(size_t)S * 2], s1 = r[(size_t)S * 2 + 1], x0 = r[(size_t)X * 2], x1 = r[(size_t)X * 2 + 1];
	const float4 n0 = r[(size_t)N * 2], n1 = r[(size_t)N * 2 + 1], p0 = r[(size_t)P * 2], p1 = r[(size_t)P * 2 + 1];
	r[(size_t)P * 2] = s0, r[(size_t)P * 2 + 1] = s1;
	r[(size_t)X * 2] = make_float4( p0.x, p0.y, p0.z, __uint_as_float( c ) ), r[(size_t)X * 2 + 1] = make_float4( p1.x, p1.y, p1.z, 0.0f );
	r[(size_t)c * 2] = x0, r[(size_t)c * 2 + 1] = x1;
	r[(size_t)c * 2 + 2] = n0, r[(size_t)c * 2 + 3] = n1;
}

// write-back: interior nodes per subtree (dfs_sizes_up, every leaf weighing 1), then every slot to its DFS-preorder place
__global__ void k_opt_sizes( const float4* __restrict__ nd, const uint32_t* __restrict__ parent, uint32_t* arrive, uint32_t* sub_int, uint32_t* sub_w, const uint32_t n )
{
	const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= n || x == 1 || count( nd, x ) == 0) return;
	dfs_sizes_up( nd, parent, arrive, sub_int, sub_w, x, 1 );
}
__global__ void k_opt_renumber( const float4* __restrict__ nd, const uint32_t* __restrict__ parent, const uint32_t* __restrict__ sub_int, const uint32_t* __restrict__ sub_w,
	float4* __restrict__ out, OptRes* res, const uint32_t n )
{
	const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= n || x == 1) return;
	uint32_t K, O, Kp;
	dfs_rank( nd, parent, sub_int, sub_w, x, K, O, Kp );
	uint32_t at = 0;
	if (x != 0) { const uint32_t p = parent[x]; at = 2 + 2 * (K - Kp) + (x == first( nd, p ) + 1 ? 1 : 0); }
	float4 a = nd[(size_t)x * 2], b = nd[(size_t)x * 2 + 1];
	if (__float_as_uint( b.w ) == 0) a.w = __uint_as_float( 2 + 2 * K );
	out[(size_t)at * 2] = a, out[(size_t)at * 2 + 1] = b;
	if (x == 0) out[2] = out[3] = make_float4( 0.0f, 0.0f, 0.0f, 0.0f ), res->interior = sub_int[0];
}
} // namespace

// tbvh_optimize's device work (api.cu does the checks and the handle's bookkeeping).  On success with *rounds > 0, *out holds the
// renumbered tree (*used nodes, depth *depth) in a new allocation the caller takes; with *rounds == 0 nothing was written anywhere.
int optimize_tree( tbvh_bvh b, const uint32_t max_rounds, const float c_trav, const float c_int, DevArray<float4>& out, uint32_t* used, uint32_t* depth,
	uint32_t* rounds, float* sah, float* ms )
{
	*rounds = 0;
	const uint32_t n = b->info.used_nodes, L = std::max( b->info.max_depth, 63u );
	cudaStream_t s = b->ctx->stream;
	// scratch: the tree and its saved copy, per slot parent / depth / height / arrival / candidate / won / list words, area and
	// cost floats, key and lock words; then the results and the threshold
	const size_t nb = (size_t)n * 32, w4 = ((size_t)n * 4 + 255) & ~(size_t)255, w8 = ((size_t)n * 8 + 255) & ~(size_t)255;
	const size_t bytes = 2 * nb + 9 * w4 + 2 * w8 + 256;
	Scratch sc( s );
	char* m = 0;
	TRY( sc.alloc( m, bytes ) );
	float4* cur = (float4*)m, * saved = (float4*)(m + nb);
	char* q = m + 2 * nb;
	uint32_t* parent = (uint32_t*)q; q += w4;
	uint32_t* dep = (uint32_t*)q; q += w4;
	uint32_t* height = (uint32_t*)q; q += w4;
	uint32_t* arrive = (uint32_t*)q; q += w4;
	uint32_t* cand = (uint32_t*)q; q += w4;
	uint32_t* won = (uint32_t*)q; q += w4;
	uint32_t* list = (uint32_t*)q; q += w4;
	float* area = (float*)q; q += w4;
	float* cost = (float*)q; q += w4;
	unsigned long long* key = (unsigned long long*)q; q += w8;
	unsigned long long* lock = (unsigned long long*)q; q += w8;
	OptRes* res = (OptRes*)q;
	unsigned long long* thr = (unsigned long long*)(q + sizeof( OptRes ));
	const uint32_t g = (n + 255) / 256;
	OptRes h = {};
	TRY( sc.events() );
	CUDA_TRY( cudaEventRecord( sc.e0, s ) );
	auto settle = [&]() -> int // parents, refold + SAH + depth, and the round's one host synchronisation
	{
		k_opt_parents<<<g, 256, 0, s>>>( cur, parent, n ); LAUNCHED();
		CUDA_TRY( cudaMemsetAsync( arrive, 0, (size_t)n * 4, s ) );
		k_opt_climb<<<g, 256, 0, s>>>( cur, parent, arrive, area, cost, height, c_trav, c_int, res, n ); LAUNCHED();
		CUDA_TRY( cudaMemcpyAsync( &h, res, sizeof( h ), cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		return TBVH_OK;
	};
	CUDA_TRY( cudaMemcpyAsync( cur, b->d_nodes, nb, cudaMemcpyDeviceToDevice, s ) );
	CUDA_TRY( cudaMemsetAsync( res, 0, sizeof( OptRes ) + 8, s ) );
	TRY( settle() );
	float best = h.sah;
	uint32_t accepted = 0, best_depth = h.height;
	bool restored = false;
	while (accepted < max_rounds)
	{
		CUDA_TRY( cudaMemcpyAsync( saved, cur, nb, cudaMemcpyDeviceToDevice, s ) );
		k_opt_depth<<<g, 256, 0, s>>>( parent, dep, n ); LAUNCHED();
		CUDA_TRY( cudaMemsetAsync( lock, 0, (size_t)n * 8, s ) );
		k_opt_search<<<(n + 127) / 128, 128, 0, s>>>( cur, parent, dep, height, area, cand, L, n ); LAUNCHED();
		k_opt_gain<<<g, 256, 0, s>>>( cur, parent, dep, area, cand, key, lock, c_trav, n ); LAUNCHED();
		k_opt_claim<<<g, 256, 0, s>>>( cur, parent, cand, key, lock, won, n ); LAUNCHED();
		CUDA_TRY( cudaMemsetAsync( res, 0, sizeof( OptRes ) + 8, s ) ); // moves and the threshold
		k_opt_cross<<<g, 256, 0, s>>>( parent, cand, won, list, res, n ); LAUNCHED();
		k_opt_apply<<<g, 256, 0, s>>>( cur, parent, cand, key, list, res, thr ); LAUNCHED();
		TRY( settle() );
		const uint32_t moves = h.moves;
		if (moves == 0) break;
		bool ok = false;
		for (uint32_t keep = moves;;)
		{
			if (h.sah < best && h.height <= L) { ok = true; break; }
			CUDA_TRY( cudaMemcpyAsync( cur, saved, nb, cudaMemcpyDeviceToDevice, s ) );
			restored = true;
			if (keep == 1) break;
			keep /= 2;
			k_opt_select<<<1, 1024, 0, s>>>( list, key, moves, keep, thr ); LAUNCHED();
			k_opt_parents<<<g, 256, 0, s>>>( cur, parent, n ); LAUNCHED(); // the round's parents, which the moves are written against
			k_opt_apply<<<g, 256, 0, s>>>( cur, parent, cand, key, list, res, thr ); LAUNCHED();
			TRY( settle() );
			restored = false;
		}
		if (!ok) break;
		best = h.sah, best_depth = h.height, accepted++;
	}
	if (accepted > 0)
	{
		if (restored) { k_opt_parents<<<g, 256, 0, s>>>( cur, parent, n ); LAUNCHED(); }
		CUDA_TRY( cudaMemsetAsync( arrive, 0, (size_t)n * 4, s ) );
		k_opt_sizes<<<g, 256, 0, s>>>( cur, parent, arrive, dep, cand, n ); LAUNCHED();
		DevArray<float4> o;
		TRY( o.alloc( nb ) );
		k_opt_renumber<<<g, 256, 0, s>>>( cur, parent, dep, cand, o, res, n );
		const cudaError_t le = cudaGetLastError();
		g_tbvh_launches++;
		if (le == cudaSuccess) CUDA_TRY( cudaMemcpyAsync( &h, res, sizeof( h ), cudaMemcpyDeviceToHost, s ) );
		if (le != cudaSuccess || cudaStreamSynchronize( s ) != cudaSuccess)
		{
			tbvh_set_error( "tbvh_optimize: write-back -> %s", cudaGetErrorString( le != cudaSuccess ? le : cudaGetLastError() ) );
			return TBVH_E_CUDA;
		}
		out = std::move( o ), *used = 2 + 2 * h.interior, *depth = best_depth;
	}
	CUDA_TRY( cudaEventRecord( sc.e1, s ) );
	CUDA_TRY( cudaEventSynchronize( sc.e1 ) );
	CUDA_TRY( cudaEventElapsedTime( ms, sc.e0, sc.e1 ) );
	*rounds = accepted, *sah = best;
	return TBVH_OK;
}
