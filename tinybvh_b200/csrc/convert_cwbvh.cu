// tinybvh_b200/csrc/convert_cwbvh.cu - BVH2 -> CWBVH on the device.
//
// Replaces the conversion chain of BVH8_CWBVH::Build (tiny_bvh.h:5827-5834):
//     Compact (:3733)  -> identity on a hole-free DFS-ordered tree, skipped (node numbering does not reach the output)
//     SplitLeafs(3) (:1988-2017)               k_split_count / scan / k_split_emit
//     MBVH<8>::ConvertFrom (:4975-5048)        k_collapse, level by level, top-down (a node adopts the uncollapsed
//                                              interior child of largest surface area until it has 8 children)
//     BVH8_CWBVH::ConvertFrom (:5884-6018)     k_assign (greedy 8x8 child->octant-slot assignment), k_sizes (bottom-up
//                                              subtree node / triangle counts), k_addresses (top-down), k_encode
// The reference emits nodes and triangles in the order of a stack-driven walk (children of a node contiguous, the LAST
// interior child processed first).  That order is a pure function of subtree sizes:
//     childBase(c_j) = childBase(X) + k + sum_{j' > j} (size(c_j') - 1)
//     triBase(c_j)   = triBase(X) + 3 * leafTris(X) + sum_{j' > j} 3 * tris(c_j')
// (k = number of interior children of X, c_j its j-th interior child in slot order), so the output is byte-identical to
// the reference's without walking the tree sequentially.  tests/test_convert_gpu.py compares bvh8Data / bvh8Tris bytes.
//
// On a refittable tree the collapse is kept (CwKeep), and tbvh_refit_layouts runs everything after it again over the refitted boxes
// (refit_trees): the result is BVH8_CWBVH::ConvertFrom of an MBVH<8> with the collapse of the conversion and the boxes of the
// refitted tree, which tests/cwbvh_refit_oracle.c restates.
//
// Batches (tbvh_convert_batch; a single conversion is K = 1).  Up to the collapse, K trees share one index space per stage: tree t
// owns BVH2 nodes nbase[t] .. nbase[t+1] of the SplitLeafs scan and split-tree nodes ext_base[t] .. ext_base[t+1] of one `ext`
// array, whose child links are global.  Level 0 of the collapse holds the K roots; a level places every node's interior children by
// a scan over the level in list order, so each level is grouped by tree in batch order and the lists are deterministic.
// Everything after the collapse is one per-tree pipeline, shared with the refit: k_keep makes every tree's collapse tree-local, and
// cw_assign_encode runs over a table of trees (CwTree) and each tree's runs of the levels (CwRun).  A single tree is a one-entry
// table; its forest is already tree-local, so unless it keeps its collapse the table points into the forest and k_keep does not run.
// The fixed costs - allocations, launches and host round trips - grow with the deepest tree's level count, not with K.
#include "common.cuh"
#include <algorithm>
#include <new>
#include <string.h>
#include <vector>

// scratch record of one wide node, indexed by wide node (level order, the order of the level lists)
struct WideNode
{
	uint32_t child[8];      // split-tree node of the child in octant slot s (0 = empty)
	uint32_t wchild[8];     // wide node of an interior child in slot s (0 = leaf or empty: the root is nobody's child)
	uint32_t ichild;        // interior children
	uint32_t leaf_tris;     // triangles in leaf children
	uint32_t size;          // wide nodes in the subtree, including this one
	uint32_t tris;          // triangles in the subtree
	uint32_t addr;          // index of this node in the output (node units)
	uint32_t cbase;         // index of its first interior child
	uint32_t tbase;         // first triangle record of its leaf children (float4 units)
};

// The 8-wide collapse of the last conversion, kept on refittable handles for tbvh_refit_layouts: a refit moves boxes, not
// topology, so everything the collapse decided stays valid and only the box-dependent steps run again.
struct CwKeep
{
	uint32_t used = 0, total = 0, wide_count = 0; // BVH2 nodes, nodes after SplitLeafs(3), wide nodes
	bool leaf_root = false;                       // the wide root wraps a leaf root (MBVH<8>::ConvertFrom :5036)
	std::vector<uint32_t> off;                    // level l holds wide nodes off[l] .. off[l+1]
	// one allocation, at base, holds the four arrays of the collapse
	DevArray<uint32_t> base;                      // used + 1: k_split_count scan, where each split leaf's chain goes
	uint32_t* list = 0;                           // wide_count: split-tree node of every wide node
	uint32_t* adopt = 0;                          // wide_count * 8: its children in ADOPTION order (k_assign breaks ties by it)
	uint32_t* ifirst = 0;                         // wide_count: wide node of its first interior child; the others follow
	// refit scratch: allocated by the first refit, alone or in a batch, and kept until the CWBVH is dropped
	DevArray<float4> ext;                         // total * 2: the split tree with the refitted boxes
	DevArray<WideNode> wide;                      // wide_count
	DevArray<uint32_t> parent;                    // used: BVH::Refit's parents (topology only), filled by the first refit
};

// One tree of a conversion or of a refit that keeps its CWBVH (device table, indexed by tree).  Everything after the collapse works on
// the tree's own arrays with tree-local numbers.
struct CwTree
{
	const float4* nodes;                // BVH2 nodes (d_nodes)
	const uint32_t* prim_idx;           // the tree's own primIdx
	const float4* verts;
	float4* cw_nodes, * cw_tris;        // bvh8Data / bvh8Tris of the handle
	float4* ext;                        // its split tree, from its node 0
	const uint32_t* scan;               // its SplitLeafs scan, from its node 0: node x's chain pairs follow scan[x] - scan[0] others
	uint32_t* list, * adopt, * ifirst;  // its collapse (CwKeep)
	WideNode* wide;
	uint32_t* keep;                     // a conversion's k_keep writes the tree-local collapse here (base | list | adopt | ifirst), else NULL
	uint32_t shift;                     // added to every child link ext stores: the tree's first node in a conversion's forest (ext_base)
	uint32_t nbase, used;               // first BVH2 node in the call's node space, BVH2 nodes
	uint32_t wbase, wide_count;         // first wide node in the call's wide-node space (tree by tree), wide nodes
	uint32_t leaf_root;                 // the wide root wraps a leaf root
};
// a batch level is each tree's run of nodes on that level, in batch order: the call's wide nodes first .. (level order) are the
// tree's nodes lo ..
struct CwRun { uint32_t first, tree, lo, pad; };

// A tree owns at least two split-tree nodes before its chain nodes: a leaf root is wrapped into node 1 (wrap_leaf_root), which an
// uploaded one-node tree does not have
__host__ __device__ __forceinline__ uint32_t cw_seg( const uint32_t used ) { return used < 2 ? 2 : used; }

// BVH::SA (tiny_bvh.h:8477) in the oracle's pairing
__device__ __forceinline__ float node_sa( const float4 mn, const float4 mx )
{
	const float ex = __fsub_rn( mx.x, mn.x ), ey = __fsub_rn( mx.y, mn.y ), ez = __fsub_rn( mx.z, mn.z );
	return __fmaf_rn( ez, ex, __fmaf_rn( ey, ex, __fmul_rn( ez, ey ) ) );
}

// ---- SplitLeafs(3): a leaf with c > 3 primitives becomes a right-leaning chain of ceil(c/3) leaves that all keep the
// original bounds (:1996-2003).  New nodes are appended after the tree's existing ones.
__global__ void k_split_count( const CwTree* __restrict__ T, const uint32_t K, const uint32_t n, uint32_t* __restrict__ extra, const uint32_t max_prims )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n) return;
	const CwTree& tr = T[batch_entry<CwTree, &CwTree::nbase>( T, K, g )];
	const uint32_t x = g - tr.nbase;
	const uint32_t c = x == 1 || x >= tr.used ? 0 : __float_as_uint( tr.nodes[(size_t)x * 2 + 1].w );
	extra[g] = c > max_prims ? 2 * ((c + max_prims - 1) / max_prims - 1) : 0;
}

// first split-tree node of every tree, from the scan of k_split_count: the nodes and chain nodes of the trees before it
__global__ void k_tree_bases( const CwTree* __restrict__ T, const uint32_t K, const uint32_t* __restrict__ base, uint32_t* __restrict__ ext_base )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= K) return;
	const uint32_t nb = T[t].nbase, seg = cw_seg( T[t].used );
	ext_base[t] = nb + base[nb];
	if (t == K - 1) ext_base[K] = nb + seg + base[nb + seg];
}

// BVH2 node x (a, b) as node x of the tree's split tree: a link to its children carries `shift`, and a long leaf's chain goes to the
// pairs from `pair` on
__device__ __forceinline__ void split_emit( float4 a, const float4 b, const uint32_t x, const uint32_t shift, uint32_t pair, float4* __restrict__ ext, const uint32_t max_prims )
{
	const uint32_t c = x == 1 ? 0 : __float_as_uint( b.w ), first = __float_as_uint( a.w );
	uint32_t cur = x;
	if (c <= max_prims)
	{
		if (__float_as_uint( b.w ) == 0) a.w = __uint_as_float( first + shift );
		ext[(size_t)cur * 2] = a, ext[(size_t)cur * 2 + 1] = b;
		return;
	}
	const uint32_t k = (c + max_prims - 1) / max_prims; // leaves in the chain
	for (uint32_t j = 0; j + 1 < k; j++, pair += 2)
	{
		// `cur` becomes interior over (leaf of max_prims, rest)
		ext[(size_t)cur * 2] = make_float4( a.x, a.y, a.z, __uint_as_float( pair + shift ) );
		ext[(size_t)cur * 2 + 1] = make_float4( b.x, b.y, b.z, __uint_as_float( 0u ) );
		ext[(size_t)pair * 2] = make_float4( a.x, a.y, a.z, __uint_as_float( first + j * max_prims ) );
		ext[(size_t)pair * 2 + 1] = make_float4( b.x, b.y, b.z, __uint_as_float( max_prims ) );
		cur = pair + 1;
	}
	ext[(size_t)cur * 2] = make_float4( a.x, a.y, a.z, __uint_as_float( first + (k - 1) * max_prims ) );
	ext[(size_t)cur * 2 + 1] = make_float4( b.x, b.y, b.z, __uint_as_float( c - (k - 1) * max_prims ) );
}

// Every tree's chains follow its own nodes.  A conversion's forest (shift = ext_base, the batch scan from nbase) keeps global child
// links for k_collapse; a refit's kept split tree (shift = 0, CwKeep::base) is local.  Node g of the call's node space, in the tree
// of T that owns it.
__global__ void k_split_emit( const CwTree* __restrict__ T, const uint32_t K, const uint32_t n, const uint32_t max_prims )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n) return;
	const CwTree& tr = T[batch_entry<CwTree, &CwTree::nbase>( T, K, g )];
	const uint32_t x = g - tr.nbase;
	if (x >= tr.used) return; // node 1 of a one-node tree in a conversion: only a leaf-root wrap writes it
	split_emit( tr.nodes[(size_t)x * 2], tr.nodes[(size_t)x * 2 + 1], x, tr.shift, cw_seg( tr.used ) + tr.scan[x] - tr.scan[0], tr.ext, max_prims );
}
static int cw_split_emit( const CwTree* d_T, const uint32_t K, const uint32_t n, cudaStream_t s )
{
	k_split_emit<<<(n + 255) / 256, 256, 0, s>>>( d_T, K, n, 3 );
	LAUNCHED();
	return TBVH_OK;
}

// MBVH<8>::ConvertFrom :5036-5044: a leaf root x is copied to node x + 1 (its tree's unused node 1), and x becomes a one-child
// interior node (wide node w)
__device__ __forceinline__ void wrap_leaf_root( float4* ext, uint32_t* adopt, const uint32_t x, const uint32_t w )
{
	ext[(size_t)(x + 1) * 2] = ext[(size_t)x * 2], ext[(size_t)(x + 1) * 2 + 1] = ext[(size_t)x * 2 + 1];
	ext[(size_t)x * 2 + 1].w = __uint_as_float( 0u );
	adopt[(size_t)w * 8] = x + 1;
	for (int i = 1; i < 8; i++) adopt[(size_t)w * 8 + i] = 0;
}
// the leaf roots of a refit's trees, each into its tree's node 1
__global__ void k_wrap_leaf_roots( const CwTree* __restrict__ T, const uint32_t K )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t < K && T[t].leaf_root) wrap_leaf_root( T[t].ext, T[t].adopt, 0, 0 );
}

// ---- MBVH<8>::ConvertFrom collapse for one level of wide nodes (:5010-5033): wide nodes lo .. lo+num-1 of `list`; their interior
// children are appended to `list` as the next level, each node's contiguously and in adoption order, the nodes in list order.  On
// level 0 (roots = K) a leaf root is wrapped instead.  Where a node's children go is an exclusive scan of the interior-child counts
// over the level: a block scan, then each block looks back over its predecessors' published sums (decoupled look-back).  Blocks
// take their place in the level from a ticket, so every block a block waits for is already running.  look: one zeroed word per
// block of the level; *next_count receives the size of the next level.  groups (a batch only): the first wide node of every run of
// one tree's nodes on the level, as (tree, node), appended in any order at *ngroups.
#define CW_LEVEL_T 256
#define CW_MAX_LEVELS 4096
__global__ void __launch_bounds__( CW_LEVEL_T ) k_collapse( float4* __restrict__ ext, uint32_t* __restrict__ list, uint32_t* __restrict__ wtree, const uint32_t lo,
	const uint32_t num, const uint32_t roots, uint32_t* __restrict__ adopt, uint32_t* __restrict__ ifirst, uint32_t* __restrict__ leaf_root,
	unsigned long long* look, uint32_t* ticket, uint32_t* __restrict__ next_count, uint2* __restrict__ groups, uint32_t* __restrict__ ngroups )
{
	__shared__ uint32_t s_blk, s_excl, s_warp[CW_LEVEL_T / 32];
	if (threadIdx.x == 0) s_blk = atomicAdd( ticket, 1u );
	__syncthreads();
	const uint32_t blk = s_blk, t = blk * CW_LEVEL_T + threadIdx.x, w = lo + t;
	uint32_t c[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
	uint32_t n = 0, ic = 0;
	if (t < num)
	{
		const uint32_t x = list[w];
		if (groups && (t == 0 || wtree[w - 1] != wtree[w])) groups[atomicAdd( ngroups, 1u )] = make_uint2( wtree[w], w );
		if (t < roots && __float_as_uint( ext[(size_t)x * 2 + 1].w ) != 0) wrap_leaf_root( ext, adopt, x, w ), leaf_root[t] = 1;
		else
		{
			n = 2;
			c[0] = __float_as_uint( ext[(size_t)x * 2].w ), c[1] = c[0] + 1;
			while (n < 8)
			{
				int best = -1;
				float bestSA = 0;
				for (uint32_t i = 0; i < n; i++)
				{
					const float4 mn = ext[(size_t)c[i] * 2], mx = ext[(size_t)c[i] * 2 + 1];
					if (__float_as_uint( mx.w ) != 0) continue; // leaf: cannot be adopted
					const float sa = node_sa( mn, mx );
					if (sa > bestSA) best = (int)i, bestSA = sa;
				}
				if (best < 0) break;
				const uint32_t g = __float_as_uint( ext[(size_t)c[best] * 2].w );
				c[best] = g, c[n++] = g + 1;
			}
			for (uint32_t i = 0; i < 8; i++)
			{
				adopt[(size_t)w * 8 + i] = c[i];
				if (i < n && __float_as_uint( ext[(size_t)c[i] * 2 + 1].w ) == 0) ic++;
			}
		}
	}
	const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	uint32_t inc = ic;
	#pragma unroll
	for (uint32_t d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync( 0xffffffffu, inc, d ); if (lane >= d) inc += y; }
	if (lane == 31) s_warp[warp] = inc;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		uint32_t agg = 0;
		for (int i = 0; i < CW_LEVEL_T / 32; i++) { const uint32_t v = s_warp[i]; s_warp[i] = agg, agg += v; }
		// look word: status (1 = this block's sum, 2 = the sum of every block up to and including it) << 32 | value
		uint32_t excl = 0;
		if (blk)
		{
			atomicExch( look + blk, (1ull << 32) | agg );
			for (uint32_t p = blk - 1;; p--)
			{
				unsigned long long v;
				do v = *(volatile unsigned long long*)(look + p); while ((v >> 32) == 0);
				excl += (uint32_t)v;
				if ((v >> 32) == 2) break;
			}
		}
		atomicExch( look + blk, (2ull << 32) | (excl + agg) );
		s_excl = excl;
		if (blk == gridDim.x - 1) *next_count = excl + agg;
	}
	__syncthreads();
	if (t < num)
	{
		uint32_t at = lo + num + s_excl + s_warp[warp] + inc - ic;
		ifirst[w] = at;
		const uint32_t tree = wtree[w];
		for (uint32_t i = 0; i < n; i++) if (__float_as_uint( ext[(size_t)c[i] * 2 + 1].w ) == 0) list[at] = c[i], wtree[at] = tree, at++;
	}
}

// the collapse of a conversion's trees into their keep blocks (every tree of a batch; a single tree when it is refittable), local to
// the tree: the forest numbers wide nodes in level order, so
// wide node i of run r (CwRun) is the tree's node r.lo + i - r.first, split-tree nodes lose ext_base, and the SplitLeafs scan starts
// at 0.  Threads 0 .. W-1 take the wide nodes, W .. W+N-1 the BVH2 nodes.
__global__ void k_keep( const CwTree* __restrict__ T, const uint32_t K, const CwRun* __restrict__ runs, const uint32_t G, const uint32_t W,
	const uint32_t* __restrict__ list, const uint32_t* __restrict__ adopt, const uint32_t* __restrict__ ifirst, const uint32_t* __restrict__ base, const uint32_t N )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < W)
	{
		const CwRun r = runs[batch_entry<CwRun, &CwRun::first>( runs, G, i )];
		const CwTree& tr = T[r.tree];
		const uint32_t x = r.lo + i - r.first;
		uint32_t* kl = tr.keep + tr.used + 1, * ka = kl + tr.wide_count, * ki = ka + (size_t)8 * tr.wide_count;
		kl[x] = list[i] - tr.shift;
		for (int j = 0; j < 8; j++) { const uint32_t a = adopt[(size_t)i * 8 + j]; ka[(size_t)x * 8 + j] = a ? a - tr.shift : 0u; }
		// read only for nodes with interior children, which are the tree's own nodes on the next level
		const uint32_t c = ifirst[i];
		const CwRun rc = c < W ? runs[batch_entry<CwRun, &CwRun::first>( runs, G, c )] : CwRun{};
		ki[x] = c < W && rc.tree == r.tree ? rc.lo + c - rc.first : 0u;
	}
	else if (i - W < N)
	{
		const uint32_t g = i - W;
		const CwTree& tr = T[batch_entry<CwTree, &CwTree::nbase>( T, K, g )];
		const uint32_t x = g - tr.nbase;
		if (x >= tr.used) return;
		const uint32_t b0 = base[tr.nbase];
		tr.keep[x] = base[g] - b0;
		if (x + 1 == tr.used) tr.keep[tr.used] = base[g + 1] - b0;
	}
}

// ---- BVH8_CWBVH::ConvertFrom, greedy child -> slot assignment (:5910-5946) and per-node child statistics, one thread per wide node.
// Wide node g of the call's wide-node space, in the tree of T that owns it.  A tree's own arrays, local numbers: its local node 0 is
// its root.
__global__ void k_assign( const CwTree* __restrict__ T, const uint32_t K, const uint32_t num )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= num) return;
	const CwTree& tr = T[batch_entry<CwTree, &CwTree::wbase>( T, K, g )];
	const uint32_t t = g - tr.wbase;
	const float4* __restrict__ ext = tr.ext;
	const uint32_t* __restrict__ adopt = tr.adopt;
	const uint32_t x = tr.list[t];
	WideNode w = {};
	for (int i = 0; i < 8; i++) w.child[i] = adopt[(size_t)t * 8 + i];
	const float4 lo = ext[(size_t)x * 2], hi = ext[(size_t)x * 2 + 1];
	const float ncx = __fmul_rn( __fadd_rn( lo.x, hi.x ), 0.5f ), ncy = __fmul_rn( __fadd_rn( lo.y, hi.y ), 0.5f ), ncz = __fmul_rn( __fadd_rn( lo.z, hi.z ), 0.5f );
	float dx[8], dy[8], dz[8];
	for (uint32_t i = 0; i < 8; i++)
	{
		dx[i] = dy[i] = dz[i] = 0;
		if (w.child[i] == 0) continue;
		const float4 mn = ext[(size_t)w.child[i] * 2], mx = ext[(size_t)w.child[i] * 2 + 1];
		dx[i] = __fsub_rn( __fmul_rn( __fadd_rn( mn.x, mx.x ), 0.5f ), ncx );
		dy[i] = __fsub_rn( __fmul_rn( __fadd_rn( mn.y, mx.y ), 0.5f ), ncy );
		dz[i] = __fsub_rn( __fmul_rn( __fadd_rn( mn.z, mx.z ), 0.5f ), ncz );
	}
	int assignment[8];
	bool slot_empty[8];
	for (int s = 0; s < 8; s++) slot_empty[s] = true, assignment[s] = -1;
	while (true)
	{
		float minCost = BVH_FAR;
		int ms = -1, mi = -1;
		for (int s = 0; s < 8; s++)
		{
			if (!slot_empty[s]) continue;
			const float sx = (s & 4) ? -1.0f : 1.0f, sy = (s & 2) ? -1.0f : 1.0f, sz = (s & 1) ? -1.0f : 1.0f;
			for (int i = 0; i < 8; i++)
			{
				if (assignment[i] != -1 || w.child[i] == 0) continue; // empty children cost BVH_FAR: never < minCost
				// tinybvh_dot( childCentroid - nodeCentroid, ds ): products with +-1 are exact, sums round as (x + y) + z
				const float cost = __fadd_rn( __fadd_rn( __fmul_rn( dx[i], sx ), __fmul_rn( dy[i], sy ) ), __fmul_rn( dz[i], sz ) );
				if (cost < minCost) minCost = cost, ms = s, mi = i;
			}
		}
		if (ms == -1) break;
		slot_empty[ms] = false, assignment[mi] = ms;
	}
	for (int i = 0; i < 8; i++) if (assignment[i] == -1) for (int s = 0; s < 8; s++) if (slot_empty[s]) { slot_empty[s] = false, assignment[i] = s; break; }
	// interior children in adoption order are the wide nodes ifirst, ifirst + 1, .. (k_collapse)
	const uint32_t adopted[8] = { w.child[0], w.child[1], w.child[2], w.child[3], w.child[4], w.child[5], w.child[6], w.child[7] };
	uint32_t wi = tr.ifirst[t], lt = 0;
	for (int i = 0; i < 8; i++)
	{
		const uint32_t c = adopted[i];
		const int s = assignment[i];
		w.child[s] = c;
		if (c == 0) continue;
		const uint32_t cnt = __float_as_uint( ext[(size_t)c * 2 + 1].w );
		if (cnt == 0) w.wchild[s] = wi++, w.ichild++; else lt += cnt;
	}
	w.leaf_tris = lt, w.size = 1, w.tris = lt;
	if (t == 0) w.cbase = 1; // the root: node 0 of its tree, its children from node 1, its triangles from record 0
	tr.wide[t] = w;
}

// wide node lo + t of the call's level order: of the level's run that holds it, in its tree's own array
__device__ __forceinline__ uint32_t level_node( const CwTree* __restrict__ T, const CwRun* __restrict__ runs, const uint32_t nruns, const uint32_t lo,
	const uint32_t t, WideNode* __restrict__& wide )
{
	const CwRun r = runs[batch_entry<CwRun, &CwRun::first>( runs, nruns, lo + t )];
	wide = T[r.tree].wide;
	return r.lo + lo + t - r.first;
}

// bottom-up: subtree node / triangle counts of wide nodes lo .. lo+num-1 (the next level's are final already)
__global__ void k_sizes( const CwTree* __restrict__ T, const CwRun* __restrict__ runs, const uint32_t nruns, const uint32_t lo, const uint32_t num )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= num) return;
	WideNode* wide;
	const uint32_t x = level_node( T, runs, nruns, lo, t, wide );
	uint32_t size = 1, tris = wide[x].leaf_tris;
	for (int s = 0; s < 8; s++)
	{
		const uint32_t c = wide[x].wchild[s];
		if (c == 0) continue;
		size += wide[c].size, tris += wide[c].tris;
	}
	wide[x].size = size, wide[x].tris = tris;
}

// top-down: output addresses of the children of wide nodes lo .. lo+num-1 (see the header comment)
__global__ void k_addresses( const CwTree* __restrict__ T, const CwRun* __restrict__ runs, const uint32_t nruns, const uint32_t lo, const uint32_t num )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= num) return;
	WideNode* wide;
	const uint32_t x = level_node( T, runs, nruns, lo, t, wide );
	const WideNode w = wide[x];
	uint32_t accS = 0, accT = 0, j = w.ichild;
	for (int s = 7; s >= 0; s--)
	{
		const uint32_t c = w.wchild[s];
		if (c == 0) continue;
		j--;
		wide[c].addr = w.cbase + j;
		wide[c].cbase = w.cbase + w.ichild + accS;
		wide[c].tbase = w.tbase + 3 * w.leaf_tris + accT;
		accS += wide[c].size - 1, accT += 3 * wide[c].tris;
	}
}

// (int8_t)ceilf( log2f( extent / 255.0f ) ) with gcc/x86 conversion semantics (:5948-5950)
__device__ __forceinline__ int quant_exponent( const float extent )
{
	const float q = __fdiv_rn( extent, 255.0f );
	const float l = (float)log2( (double)q ); // correctly rounded single-precision log2
	const int v = __float2int_rz( ceilf( l ) );  // -inf / NaN -> INT_MIN / 0: low byte 0, as cvttss2si + truncation
	return (int)(int8_t)(v & 0xff);
}

// wide node w over split-tree node x: its 80-byte node at w.addr of out_nodes, its leaf children's triangles from w.tbase of out_tris
__device__ __forceinline__ void encode_node( const float4* __restrict__ ext, const uint32_t x, const WideNode& w, const uint32_t* __restrict__ prim_idx,
	const float4* __restrict__ verts, float4* __restrict__ out_nodes, float4* __restrict__ out_tris )
{
	const float4 lo = ext[(size_t)x * 2], hi = ext[(size_t)x * 2 + 1];
	const int ex = quant_exponent( __fsub_rn( hi.x, lo.x ) ), ey = quant_exponent( __fsub_rn( hi.y, lo.y ) ), ez = quant_exponent( __fsub_rn( hi.z, lo.z ) );
	const float sx = ldexpf( 1.0f, ex ), sy = ldexpf( 1.0f, ey ), sz = ldexpf( 1.0f, ez ); // powf( 2, e ), exact
	uint32_t q[12] = { 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0 }; // qlox[8] qloy[8] qloz[8] qhix[8] qhiy[8] qhiz[8] as 12 words
	uint32_t meta[2] = { 0, 0 };
	uint32_t imask = 0, icount = 0, tri_count = 0;
	bool any_leaf = false;
	for (int s = 0; s < 8; s++)
	{
		const uint32_t c = w.child[s];
		if (c == 0) continue;
		const float4 mn = ext[(size_t)c * 2], mx = ext[(size_t)c * 2 + 1];
		const uint32_t b[6] = {
			(uint32_t)(int)floorf( __fdiv_rn( __fsub_rn( mn.x, lo.x ), sx ) ) & 0xffu, (uint32_t)(int)floorf( __fdiv_rn( __fsub_rn( mn.y, lo.y ), sy ) ) & 0xffu,
			(uint32_t)(int)floorf( __fdiv_rn( __fsub_rn( mn.z, lo.z ), sz ) ) & 0xffu, (uint32_t)(int)ceilf( __fdiv_rn( __fsub_rn( mx.x, lo.x ), sx ) ) & 0xffu,
			(uint32_t)(int)ceilf( __fdiv_rn( __fsub_rn( mx.y, lo.y ), sy ) ) & 0xffu, (uint32_t)(int)ceilf( __fdiv_rn( __fsub_rn( mx.z, lo.z ), sz ) ) & 0xffu };
		#pragma unroll
		for (int f = 0; f < 6; f++) q[f * 2 + (s >> 2)] |= b[f] << (8 * (s & 3));
		const uint32_t cnt = __float_as_uint( mx.w );
		uint32_t m;
		if (cnt == 0) m = (1u << 5) | (24u + (uint32_t)s), imask |= 1u << s, icount++;
		else
		{
			m = ((cnt == 1 ? 1u : cnt == 2 ? 3u : 7u) << 5) | tri_count;
			const uint32_t first = __float_as_uint( mn.w );
			for (uint32_t j = 0; j < cnt; j++)
			{
				const uint32_t ti = prim_idx[first + j];
				const float4 v0 = verts[(size_t)ti * 3], v1 = verts[(size_t)ti * 3 + 1], v2 = verts[(size_t)ti * 3 + 2];
				float4* o = out_tris + (size_t)w.tbase + (size_t)(tri_count + j) * 3;
				o[0] = make_float4( __fsub_rn( v2.x, v0.x ), __fsub_rn( v2.y, v0.y ), __fsub_rn( v2.z, v0.z ), __fsub_rn( v2.w, v0.w ) );
				o[1] = make_float4( __fsub_rn( v1.x, v0.x ), __fsub_rn( v1.y, v0.y ), __fsub_rn( v1.z, v0.z ), __fsub_rn( v1.w, v0.w ) );
				o[2] = make_float4( v0.x, v0.y, v0.z, __uint_as_float( ti ) );
			}
			tri_count += cnt, any_leaf = true;
		}
		meta[s >> 2] |= (m & 0xffu) << (8 * (s & 3));
	}
	const uint32_t n0w = ((uint32_t)ex & 0xffu) | (((uint32_t)ey & 0xffu) << 8) | (((uint32_t)ez & 0xffu) << 16) | (imask << 24);
	float4* o = out_nodes + (size_t)w.addr * 5;
	o[0] = make_float4( lo.x, lo.y, lo.z, __uint_as_float( n0w ) );
	o[1] = make_float4( __uint_as_float( icount ? w.cbase : 0u ), __uint_as_float( any_leaf ? w.tbase : 0u ), __uint_as_float( meta[0] ), __uint_as_float( meta[1] ) );
	o[2] = make_float4( __uint_as_float( q[0] ), __uint_as_float( q[1] ), __uint_as_float( q[2] ), __uint_as_float( q[3] ) );
	o[3] = make_float4( __uint_as_float( q[4] ), __uint_as_float( q[5] ), __uint_as_float( q[6] ), __uint_as_float( q[7] ) );
	o[4] = make_float4( __uint_as_float( q[8] ), __uint_as_float( q[9] ), __uint_as_float( q[10] ), __uint_as_float( q[11] ) );
}

// wide node g, as for k_assign
__global__ void k_encode( const CwTree* __restrict__ T, const uint32_t K, const uint32_t num )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= num) return;
	const CwTree& tr = T[batch_entry<CwTree, &CwTree::wbase>( T, K, g )];
	const uint32_t t = g - tr.wbase;
	encode_node( tr.ext, tr.list[t], tr.wide[t], tr.prim_idx, tr.verts, tr.cw_nodes, tr.cw_tris );
}

// The levels of K trees in the call's level order: level l is wide nodes off[l] .. off[l+1], each tree's run of it in batch order,
// runs start[l] .. start[l+1].  tree_off[i]: tree i's own level offsets (CwKeep::off).
struct CwLevels { std::vector<CwRun> runs; std::vector<uint32_t> off, start; };
static CwLevels cw_levels( const std::vector<const std::vector<uint32_t>*>& tree_off )
{
	CwLevels lv;
	size_t levels = 0;
	for (const auto* o : tree_off) levels = std::max( levels, o->size() - 1 );
	lv.off.assign( 1, 0 ), lv.start.assign( 1, 0 );
	for (size_t l = 0; l < levels; l++)
	{
		uint32_t at = lv.off.back();
		for (uint32_t i = 0; i < (uint32_t)tree_off.size(); i++)
		{
			const std::vector<uint32_t>& o = *tree_off[i];
			if (l + 1 < o.size()) lv.runs.push_back( CwRun{ at, i, o[l], 0 } ), at += o[l + 1] - o[l];
		}
		lv.off.push_back( at ), lv.start.push_back( (uint32_t)lv.runs.size() );
	}
	return lv;
}

// slot assignment, subtree sizes (bottom-up), addresses (top-down), encode: everything after the collapse that depends on boxes, for
// the K trees of the table d_T whose levels are lv (runs on the device at d_runs)
static int cw_assign_encode( const CwTree* d_T, const uint32_t K, const CwLevels& lv, const CwRun* d_runs, cudaStream_t s )
{
	const uint32_t levels = (uint32_t)lv.off.size() - 1, W = lv.off[levels];
	k_assign<<<(W + 127) / 128, 128, 0, s>>>( d_T, K, W ); LAUNCHED();
	#define CW_LEVEL( kernel, l ) do { const uint32_t num_ = lv.off[l + 1] - lv.off[l]; \
		kernel<<<(num_ + 127) / 128, 128, 0, s>>>( d_T, d_runs + lv.start[l], lv.start[l + 1] - lv.start[l], lv.off[l], num_ ); LAUNCHED(); } while (0)
	for (int l = (int)levels - 1; l >= 0; l--) CW_LEVEL( k_sizes, l );
	for (uint32_t l = 0; l < levels; l++) CW_LEVEL( k_addresses, l );
	#undef CW_LEVEL
	k_encode<<<(W + 127) / 128, 128, 0, s>>>( d_T, K, W ); LAUNCHED();
	return TBVH_OK;
}

// the CWBVH arrays of b and what refers to them go (a TLAS over them becomes stale)
void drop_cwbvh( tbvh_bvh b )
{
	if (b->d_cw_trav || b->d_cw_tris) b->generation = tbvh_next_generation(); // a TLAS may hold these addresses (api.cu tlas_check)
	b->d_cw_nodes.reset(), b->d_cw_tris.reset(), b->d_cw_trav.reset();
	delete b->cw_keep; // its arrays free themselves
	b->cw_keep = 0;
	b->info.layouts &= ~(1u << TBVH_LAYOUT_CWBVH), b->info.used_blocks = 0, b->info.cwbvh_tri_count = 0;
	b->cw_pending = 0, b->cw_rd_limit = -1.0f;
}

// bs[0 .. K): handles of one context holding BVH-layout trees.  On success each holds the CWBVH a conversion of its own tree gives;
// on failure none holds a CWBVH.
int bvh_to_cwbvh( const tbvh_bvh* bs, const uint32_t K, cudaStream_t s )
{
	std::vector<CwTree> T( K );
	uint32_t N = 0; // BVH2 nodes of the batch (the caller bounds the batch; a single tree's count is a uint32_t)
	for (uint32_t t = 0; t < K; t++)
	{
		const tbvh_bvh b = bs[t];
		drop_cwbvh( b );
		T[t] = CwTree{};
		T[t].nodes = b->d_nodes, T[t].prim_idx = b->d_prim_idx, T[t].verts = b->d_verts, T[t].nbase = N, T[t].used = b->info.used_nodes;
		N += cw_seg( T[t].used );
	}
	// scratch of one stage carved from one allocation: fewer cudaMalloc / cudaFree pairs per call
	size_t carve = 0;
	char* blob = 0;
	auto take = [&]( const size_t bytes ) { const size_t o = carve; carve += (bytes + 255) & ~(size_t)255; return o; };
	CwTree* d_T = 0;
	uint32_t* extra = 0, * base = 0, * tile = 0, * d_ext = 0, * lists = 0, * wtree = 0, * adopt = 0, * ifirst = 0, * leaf = 0, * tickets = 0, * counts = 0;
	uint32_t* ngroups = 0;
	uint2* groups = 0;
	unsigned long long* look = 0;
	float4* ext = 0;
	auto body = [&]() -> int
	{
		Scratch sc( s );
		// ---- SplitLeafs(3) over every tree, and each tree's first split-tree node
		{
			carve = 0;
			const size_t o_T = take( (size_t)K * sizeof( CwTree ) ), o_extra = take( ((size_t)N + 1) * 4 ), o_base = take( ((size_t)N + 1) * 4 );
			const size_t o_tile = take( ((size_t)N / 2048 + 2) * 4 ), o_ext = take( ((size_t)K + 1) * 4 );
			TRY( sc.alloc( blob, carve ) );
			d_T = (CwTree*)(blob + o_T), extra = (uint32_t*)(blob + o_extra), base = (uint32_t*)(blob + o_base), tile = (uint32_t*)(blob + o_tile);
			d_ext = (uint32_t*)(blob + o_ext);
		}
		CUDA_TRY( cudaMemcpyAsync( d_T, T.data(), (size_t)K * sizeof( CwTree ), cudaMemcpyHostToDevice, s ) );
		k_split_count<<<(N + 255) / 256, 256, 0, s>>>( d_T, K, N, extra, 3 ); LAUNCHED();
		{ const int r = exclusive_scan( extra, base, tile, N, s ); if (r != TBVH_OK) return r; }
		k_tree_bases<<<(K + 127) / 128, 128, 0, s>>>( d_T, K, base, d_ext ); LAUNCHED();
		std::vector<uint32_t> ext_base( (size_t)K + 1 );
		CUDA_TRY( cudaMemcpyAsync( ext_base.data(), d_ext, ((size_t)K + 1) * 4, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		const uint32_t total = ext_base[K];
		// the collapse's arrays (a wide node is an interior node of the split tree: fewer than total); leaf, tickets and look are zeroed
		// together
		const size_t look_words = (size_t)total / CW_LEVEL_T + CW_MAX_LEVELS + 1; // a block per CW_LEVEL_T nodes of each level
		{
			carve = 0;
			const size_t o_ext = take( (size_t)total * 32 ), o_lists = take( ((size_t)total + 1) * 4 ), o_wtree = take( ((size_t)total + 1) * 4 );
			const size_t o_adopt = take( ((size_t)total + 1) * 32 ), o_ifirst = take( ((size_t)total + 1) * 4 ), o_counts = take( CW_MAX_LEVELS * 4 );
			const size_t o_groups = K > 1 ? take( ((size_t)total + 1) * 8 ) : 0; // a run per tree and level: at most one per wide node
			const size_t o_leaf = take( (size_t)K * 4 ), o_tickets = take( (CW_MAX_LEVELS + 1) * 4 ), o_look = take( look_words * 8 );
			TRY( sc.alloc( blob, carve ) );
			ext = (float4*)(blob + o_ext), lists = (uint32_t*)(blob + o_lists), wtree = (uint32_t*)(blob + o_wtree), adopt = (uint32_t*)(blob + o_adopt);
			ifirst = (uint32_t*)(blob + o_ifirst), counts = (uint32_t*)(blob + o_counts), groups = K > 1 ? (uint2*)(blob + o_groups) : 0;
			leaf = (uint32_t*)(blob + o_leaf), tickets = (uint32_t*)(blob + o_tickets), look = (unsigned long long*)(blob + o_look);
			CUDA_TRY( cudaMemsetAsync( blob + o_leaf, 0, carve - o_leaf, s ) );
		}
		ngroups = tickets + CW_MAX_LEVELS;
		for (uint32_t t = 0; t < K; t++) T[t].ext = ext + (size_t)ext_base[t] * 2, T[t].shift = ext_base[t], T[t].scan = base + T[t].nbase;
		CUDA_TRY( cudaMemcpyAsync( d_T, T.data(), (size_t)K * sizeof( CwTree ), cudaMemcpyHostToDevice, s ) );
		TRY( cw_split_emit( d_T, K, N, s ) );
		// ---- collapse to 8-wide, level by level from the K roots
		std::vector<uint32_t> iota( K );
		for (uint32_t t = 0; t < K; t++) iota[t] = t;
		CUDA_TRY( cudaMemcpyAsync( lists, ext_base.data(), (size_t)K * 4, cudaMemcpyHostToDevice, s ) ); // level 0 = the roots
		CUDA_TRY( cudaMemcpyAsync( wtree, iota.data(), (size_t)K * 4, cudaMemcpyHostToDevice, s ) );
		std::vector<uint32_t> off; // level l occupies lists[off[l] .. off[l+1])
		off.push_back( 0 ), off.push_back( K );
		size_t look_used = 0;
		while (off[off.size() - 1] > off[off.size() - 2])
		{
			const uint32_t level = (uint32_t)off.size() - 2, lo = off[level], num = off[level + 1] - lo, grid = (num + CW_LEVEL_T - 1) / CW_LEVEL_T;
			k_collapse<<<grid, CW_LEVEL_T, 0, s>>>( ext, lists, wtree, lo, num, level == 0 ? K : 0, adopt, ifirst, leaf, look + look_used, tickets + level, counts + level,
				groups, ngroups ); LAUNCHED();
			look_used += grid;
			uint32_t next = 0;
			CUDA_TRY( cudaMemcpyAsync( &next, counts + level, 4, cudaMemcpyDeviceToHost, s ) );
			CUDA_TRY( cudaStreamSynchronize( s ) );
			off.push_back( lo + num + next );
			if (off.size() > CW_MAX_LEVELS) { tbvh_set_error( "CWBVH conversion: runaway depth" ); return TBVH_E_LIMIT; }
		}
		off.pop_back(); // the last level is empty
		const uint32_t levels = (uint32_t)off.size() - 1, W = off[levels];
		// ---- each tree's runs of wide nodes, one per level it reaches: its wide-node count and its own level offsets (a CwKeep's off).
		// Levels are grouped by tree in batch order, so sorted by first node the runs tile every level and a run ends where the next begins.
		std::vector<uint32_t> h_leaf( K );
		std::vector<uint2> groups_h;
		uint32_t G = 0;
		if (K > 1) CUDA_TRY( cudaMemcpyAsync( &G, ngroups, 4, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaMemcpyAsync( h_leaf.data(), leaf, (size_t)K * 4, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		std::vector<std::vector<uint32_t>> toff( K, std::vector<uint32_t>( 1, 0 ) );
		if (K > 1)
		{
			groups_h.resize( G );
			CUDA_TRY( cudaMemcpyAsync( groups_h.data(), groups, (size_t)G * 8, cudaMemcpyDeviceToHost, s ) );
			CUDA_TRY( cudaStreamSynchronize( s ) );
			std::sort( groups_h.begin(), groups_h.end(), []( const uint2& a, const uint2& b ) { return a.y < b.y; } );
			for (uint32_t g = 0; g < G; g++)
			{
				const uint32_t t = groups_h[g].x, end = g + 1 < G ? groups_h[g + 1].y : W;
				toff[t].push_back( toff[t].back() + (end - groups_h[g].y) );
			}
		}
		else toff[0] = off;
		// the same levels again as each tree's runs: the forest's wide nodes are the call's level order
		std::vector<const std::vector<uint32_t>*> toff_p( K );
		for (uint32_t t = 0; t < K; t++) toff_p[t] = &toff[t];
		const CwLevels lv = cw_levels( toff_p );
		// ---- outputs, per handle; the keep blocks of K > 1 trees that do not keep their collapse are scratch of the call
		size_t scratch_words = 0;
		for (uint32_t t = 0, wb = 0; t < K; t++)
		{
			const tbvh_bvh b = bs[t];
			const uint32_t wc = toff[t].back(), used = b->info.used_nodes;
			TRY( b->d_cw_nodes.alloc( (size_t)wc * 80 ) );
			TRY( b->d_cw_tris.alloc( (size_t)b->info.idx_count * 48 ) );
			T[t].cw_nodes = b->d_cw_nodes, T[t].cw_tris = b->d_cw_tris, T[t].wbase = wb, T[t].wide_count = wc, T[t].leaf_root = h_leaf[t] != 0;
			wb += wc;
			b->info.used_blocks = wc * 5, b->info.cwbvh_tri_count = b->info.idx_count;
			if (!b->refittable) { if (K > 1) scratch_words += (size_t)used + 1 + (size_t)wc * 10; continue; }
			// keep the collapse for tbvh_refit_layouts, sized to the wide tree
			CwKeep* k = new (std::nothrow) CwKeep();
			if (!k) { tbvh_set_error( "CWBVH conversion: out of host memory" ); return TBVH_E_ARG; }
			b->cw_keep = k;
			k->used = used, k->total = ext_base[t + 1] - ext_base[t], k->wide_count = wc, k->leaf_root = h_leaf[t] != 0, k->off = toff[t];
			TRY( k->base.alloc( ((size_t)used + 1 + (size_t)wc * 10) * 4 ) );
			k->list = k->base + used + 1, k->adopt = k->list + wc, k->ifirst = k->adopt + (size_t)wc * 8;
			T[t].keep = k->base;
		}
		// one allocation: the wide nodes (each tree's slice from its wbase), the runs, the scratch keep blocks
		carve = 0;
		const size_t o_wide = take( (size_t)W * sizeof( WideNode ) ), o_runs = take( lv.runs.size() * sizeof( CwRun ) ), o_keep = take( scratch_words * 4 );
		TRY( sc.alloc( blob, carve ) );
		const CwRun* d_runs = (const CwRun*)(blob + o_runs);
		uint32_t* spare = (uint32_t*)(blob + o_keep);
		for (uint32_t t = 0; t < K; t++)
		{
			CwTree& tr = T[t];
			tr.wide = (WideNode*)(blob + o_wide) + tr.wbase;
			// a single tree's forest is already tree-local: its table entry points into it, which spares a tree that keeps no collapse
			// (tbvh_convert of an SBVH) the k_keep pass and a copy of 10 words per wide node
			if (K == 1) { tr.list = lists, tr.adopt = adopt, tr.ifirst = ifirst; continue; }
			if (!tr.keep) tr.keep = spare, spare += (size_t)tr.used + 1 + (size_t)tr.wide_count * 10;
			tr.list = tr.keep + tr.used + 1, tr.adopt = tr.list + tr.wide_count, tr.ifirst = tr.adopt + (size_t)tr.wide_count * 8;
		}
		CUDA_TRY( cudaMemcpyAsync( d_T, T.data(), (size_t)K * sizeof( CwTree ), cudaMemcpyHostToDevice, s ) );
		CUDA_TRY( cudaMemcpyAsync( (void*)d_runs, lv.runs.data(), lv.runs.size() * sizeof( CwRun ), cudaMemcpyHostToDevice, s ) );
		if (K > 1 || T[0].keep) { k_keep<<<(uint32_t)(((size_t)W + N + 255) / 256), 256, 0, s>>>( d_T, K, d_runs, (uint32_t)lv.runs.size(), W, lists, adopt, ifirst, base, N ); LAUNCHED(); }
		TRY( cw_assign_encode( d_T, K, lv, d_runs, s ) );
		// the traversal nodes the kernels read and the pending bound of every wide tree (trace_cwbvh.cu); synchronises the stream
		return cw_make_trav( bs, K, s );
	};
	const int rc = body(); // the stream is drained and the scratch freed before a failure drops the handles' arrays
	for (uint32_t t = 0; t < K; t++)
	{
		if (rc != TBVH_OK) drop_cwbvh( bs[t] );
		else bs[t]->info.layouts |= 1u << TBVH_LAYOUT_CWBVH;
	}
	return rc;
}


void cw_keep_sizes( tbvh_bvh b, uint32_t* total, uint32_t* wide_count )
{
	const CwKeep* k = b->cw_keep;
	*total = k ? k->total : 0, *wide_count = k ? k->wide_count : 0;
}

// ---- Refits (tbvh_refit / tbvh_refit_layouts are K = 1 of tbvh_refit_batch).  BVH::Refit over the K trees' node space, the BVH2
// traversal records, then - keeping the layouts - the conversion chain over each KEPT collapse with the refitted boxes (SplitLeafs(3)
// boxes, leaf-root wrap, slot assignment, addresses, encode, traversal nodes) and BVH_GPU::ConvertFrom, in place.  The result of a
// tree is BVH8_CWBVH::ConvertFrom of an MBVH<8> with the collapse of its conversion and its refitted boxes, which
// tests/cwbvh_refit_oracle.c restates.  The kept collapses are tree-local, so every kernel maps a node through its tree's table
// entry; a batch level is each tree's run of the level, in batch order.  Tables and scratch come from the context's refit buffers:
// one upload, one read-back, one host synchronisation.
static int refit_space( tbvh_ctx c, const size_t dev, const size_t host )
{
	TRY( c->refit_dev.reserve( dev ) );
	TRY( c->refit_host.reserve( host ) );
	if (!c->refit_e0) CUDA_TRY( cudaEventCreate( &c->refit_e0 ) );
	if (!c->refit_e1) CUDA_TRY( cudaEventCreate( &c->refit_e1 ) );
	return TBVH_OK;
}

int refit_trees( const tbvh_bvh* bs, const uint32_t K, const bool keep_layouts, cudaStream_t s )
{
	const tbvh_ctx c = bs[0]->ctx;
	std::lock_guard<std::mutex> lock( c->refit_mutex );
	// what each tree takes part in; the caller bounds the sums (TBVH_REFIT_BATCH_MAX_NODES)
	std::vector<uint32_t> cw, gp;
	uint32_t N = 0, P = 0, NC = 0, NG = 0;
	for (uint32_t t = 0; t < K; t++)
	{
		const tbvh_bvh b = bs[t];
		if (!keep_layouts) drop_bvh_gpu( b ), drop_cwbvh( b ); // derived layouts describe the old boxes (the reference converts again too)
		else b->generation = tbvh_next_generation(); // the arrays stay, but a TLAS over this BLAS holds its old root box in its instances
		b->revision++;
		const uint32_t used = b->info.used_nodes;
		if (keep_layouts && b->cw_keep) cw.push_back( t ), NC += used;
		if (keep_layouts && (b->info.layouts & (1u << TBVH_LAYOUT_BVH_GPU))) gp.push_back( t ), NG += used;
		N += used, P += b->info.idx_count;
	}
	const uint32_t KC = (uint32_t)cw.size(), KG = (uint32_t)gp.size();
	auto body = [&]() -> int
	{
		// arrays a tree gets on its first refit: a kept collapse's scratch, and parents that the first refit fills
		for (uint32_t t = 0; t < K; t++) TRY( leaf_tris_alloc( bs[t] ) );
		std::vector<bool> fill( K, true );
		for (const uint32_t t : cw)
		{
			CwKeep* k = bs[t]->cw_keep;
			fill[t] = !k->parent;
			if (!k->ext) TRY( k->ext.alloc( (size_t)k->total * 32 ) );
			if (!k->wide) TRY( k->wide.alloc( (size_t)k->wide_count * sizeof( WideNode ) ) );
			if (!k->parent) TRY( k->parent.alloc( (size_t)k->used * 4 ) );
		}
		// the batch levels: each tree's run of every level it reaches
		std::vector<const std::vector<uint32_t>*> toff( KC );
		for (uint32_t i = 0; i < KC; i++) toff[i] = &bs[cw[i]]->cw_keep->off;
		const CwLevels lv = cw_levels( toff );
		const std::vector<CwRun>& runs = lv.runs;
		// device: tables | arrival counters | results (root boxes, exponent ranges) | parents | BVH_GPU workspace;  host: tables | results
		size_t carve = 0;
		auto take = [&]( const size_t bytes ) { const size_t o = carve; carve += (bytes + 255) & ~(size_t)255; return o; };
		const size_t o_rf = take( (size_t)K * sizeof( RfTree ) ), o_cr = take( (size_t)KC * sizeof( CwTree ) ), o_runs = take( runs.size() * sizeof( CwRun ) );
		const size_t o_ct = take( (size_t)KC * sizeof( CwTrav ) ), o_gt = take( (size_t)KG * sizeof( GpuTree ) ), tables = carve;
		const size_t o_arrive = take( (size_t)N * 4 ), res_words = (size_t)K * 8 + KC, o_res = take( res_words * 4 ), zeroed = carve - o_arrive;
		const size_t o_parent = take( (size_t)N * 4 ), o_gw = take( (size_t)NG * 16 );
		TRY( refit_space( c, carve, tables + res_words * 4 ) );
		char* const dev = c->refit_dev, * const host = (char*)c->refit_host.p;
		uint32_t* const res = (uint32_t*)(dev + o_res), * const h_res = (uint32_t*)(host + tables);
		RfTree* const rf = (RfTree*)(host + o_rf);
		CwTree* const cr = (CwTree*)(host + o_cr);
		CwTrav* const ct = (CwTrav*)(host + o_ct);
		GpuTree* const gt = (GpuTree*)(host + o_gt);
		bool any_fill = false;
		for (uint32_t t = 0, nb = 0, pb = 0; t < K; t++)
		{
			const tbvh_bvh b = bs[t];
			uint32_t* const parent = b->cw_keep ? b->cw_keep->parent : (uint32_t*)(dev + o_parent) + nb;
			rf[t] = RfTree{ b->d_nodes, b->d_prim_idx, b->d_verts, b->d_leaf_tris, parent, nb, b->info.used_nodes, pb, b->info.idx_count, fill[t] ? 1u : 0u };
			any_fill |= fill[t];
			nb += b->info.used_nodes, pb += b->info.idx_count;
		}
		for (uint32_t i = 0, nb = 0, wb = 0; i < KC; i++)
		{
			const tbvh_bvh b = bs[cw[i]];
			CwKeep* k = b->cw_keep;
			cr[i] = CwTree{ b->d_nodes, b->d_prim_idx, b->d_verts, b->d_cw_nodes, b->d_cw_tris, k->ext, k->base, k->list, k->adopt, k->ifirst, k->wide, 0, 0,
				nb, k->used, wb, k->wide_count, k->leaf_root ? 1u : 0u };
			ct[i] = CwTrav{ (const uint4*)b->d_cw_nodes.p, (uint4*)b->d_cw_trav.p, res + (size_t)K * 8 + i, wb, k->wide_count };
			nb += k->used, wb += k->wide_count;
		}
		for (uint32_t i = 0, nb = 0; i < KG; i++)
		{
			const tbvh_bvh b = bs[gp[i]];
			gt[i] = GpuTree{ b->d_nodes, b->d_nodes_gpu, nb, b->info.used_nodes };
			nb += b->info.used_nodes;
		}
		if (!runs.empty()) memcpy( host + o_runs, runs.data(), runs.size() * sizeof( CwRun ) );
		const RfTree* d_rf = (const RfTree*)(dev + o_rf);
		const CwTree* d_cr = (const CwTree*)(dev + o_cr);
		CUDA_TRY( cudaMemcpyAsync( dev, host, tables, cudaMemcpyHostToDevice, s ) );
		CUDA_TRY( cudaEventRecord( c->refit_e0, s ) );
		CUDA_TRY( cudaMemsetAsync( dev + o_arrive, 0, zeroed, s ) );
		TRY( refit_enqueue( d_rf, K, N, (uint32_t*)(dev + o_arrive), any_fill, s ) );
		TRY( leaf_tris_enqueue( d_rf, K, P, s ) );
		if (KC)
		{
			TRY( cw_split_emit( d_cr, KC, NC, s ) );
			bool any_leaf_root = false;
			for (uint32_t i = 0; i < KC; i++) any_leaf_root |= cr[i].leaf_root != 0;
			if (any_leaf_root) { k_wrap_leaf_roots<<<(KC + 127) / 128, 128, 0, s>>>( d_cr, KC ); LAUNCHED(); }
			TRY( cw_assign_encode( d_cr, KC, lv, (const CwRun*)(dev + o_runs), s ) );
			TRY( cw_expand( (const CwTrav*)(dev + o_ct), KC, lv.off.back(), 0, s ) );
		}
		if (KG) TRY( bvh_gpu_enqueue( (const GpuTree*)(dev + o_gt), KG, NG, (uint32_t*)(dev + o_gw), s ) );
		TRY( refit_roots( d_rf, K, res, s ) );
		CUDA_TRY( cudaEventRecord( c->refit_e1, s ) );
		CUDA_TRY( cudaMemcpyAsync( h_res, res, res_words * 4, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		float ms = 0;
		CUDA_TRY( cudaEventElapsedTime( &ms, c->refit_e0, c->refit_e1 ) );
		for (uint32_t t = 0; t < K; t++)
		{
			tbvh_bvh b = bs[t];
			b->info.build_ms = ms;
			memcpy( b->info.aabb_min, h_res + (size_t)t * 8, 12 ), memcpy( b->info.aabb_max, h_res + (size_t)t * 8 + 4, 12 );
		}
		// the exponents and origins moved: a stale limit could send rays with 2^e * rD past the float range down the integer path
		for (uint32_t i = 0; i < KC; i++) bs[cw[i]]->cw_rd_limit = cw_rd_limit_for( h_res[(size_t)K * 8 + i] );
		return TBVH_OK;
	};
	const int rc = body();
	if (rc != TBVH_OK)
	{
		cudaStreamSynchronize( s );
		for (uint32_t t = 0; t < K; t++) drop_bvh_gpu( bs[t] ), drop_cwbvh( bs[t] );
	}
	return rc;
}
