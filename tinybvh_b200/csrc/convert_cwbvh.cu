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
// (cwbvh_refit): the result is BVH8_CWBVH::ConvertFrom of an MBVH<8> with the collapse of the conversion and the boxes of the
// refitted tree, which tests/cwbvh_refit_oracle.c restates.
#include "common.cuh"
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
	uint32_t* base = 0;                           // used + 1: k_split_count scan, where each split leaf's chain goes
	uint32_t* list = 0;                           // wide_count: split-tree node of every wide node
	uint32_t* adopt = 0;                          // wide_count * 8: its children in ADOPTION order (k_assign breaks ties by it)
	uint32_t* ifirst = 0;                         // wide_count: wide node of its first interior child; the others follow
	// refit scratch: allocated by the first refit, kept until the CWBVH is dropped
	float4* ext = 0;                              // total * 2: the split tree with the refitted boxes
	WideNode* wide = 0;                           // wide_count
	uint32_t* parent = 0, * arrive = 0;           // used each: BVH::Refit's parents (topology only) and arrival counters
	uint32_t* misc = 0;                           // 16 words: root box (8) + exponent range (1), read back together
	cudaEvent_t e0 = 0, e1 = 0;
};

void cw_keep_free( tbvh_bvh b )
{
	CwKeep* k = b->cw_keep;
	if (!k) return;
	void* p[] = { k->base, k->list, k->adopt, k->ifirst, k->ext, k->wide, k->parent, k->arrive, k->misc };
	for (void* q : p) if (q) cudaFree( q );
	if (k->e0) cudaEventDestroy( k->e0 );
	if (k->e1) cudaEventDestroy( k->e1 );
	delete k;
	b->cw_keep = 0;
}

// BVH::SA (tiny_bvh.h:8477) in the oracle's pairing
__device__ __forceinline__ float node_sa( const float4 mn, const float4 mx )
{
	const float ex = __fsub_rn( mx.x, mn.x ), ey = __fsub_rn( mx.y, mn.y ), ez = __fsub_rn( mx.z, mn.z );
	return __fmaf_rn( ez, ex, __fmaf_rn( ey, ex, __fmul_rn( ez, ey ) ) );
}

// ---- SplitLeafs(3): a leaf with c > 3 primitives becomes a right-leaning chain of ceil(c/3) leaves that all keep the
// original bounds (:1996-2003).  New nodes are appended after the existing ones.
__global__ void k_split_count( const float4* __restrict__ nodes, uint32_t* __restrict__ extra, const uint32_t used, const uint32_t max_prims )
{
	const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= used) return;
	const uint32_t c = x == 1 ? 0 : __float_as_uint( nodes[(size_t)x * 2 + 1].w );
	extra[x] = c > max_prims ? 2 * ((c + max_prims - 1) / max_prims - 1) : 0;
}

__global__ void k_split_emit( const float4* __restrict__ nodes, const uint32_t* __restrict__ base, float4* __restrict__ ext, const uint32_t used, const uint32_t max_prims )
{
	const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= used) return;
	float4 a = nodes[(size_t)x * 2], b = nodes[(size_t)x * 2 + 1];
	const uint32_t c = x == 1 ? 0 : __float_as_uint( b.w ), first = __float_as_uint( a.w );
	if (c <= max_prims) { ext[(size_t)x * 2] = a, ext[(size_t)x * 2 + 1] = b; return; }
	const uint32_t k = (c + max_prims - 1) / max_prims; // leaves in the chain
	uint32_t cur = x, pair = used + base[x];
	for (uint32_t j = 0; j + 1 < k; j++, pair += 2)
	{
		// `cur` becomes interior over (leaf of max_prims, rest)
		ext[(size_t)cur * 2] = make_float4( a.x, a.y, a.z, __uint_as_float( pair ) );
		ext[(size_t)cur * 2 + 1] = make_float4( b.x, b.y, b.z, __uint_as_float( 0u ) );
		ext[(size_t)pair * 2] = make_float4( a.x, a.y, a.z, __uint_as_float( first + j * max_prims ) );
		ext[(size_t)pair * 2 + 1] = make_float4( b.x, b.y, b.z, __uint_as_float( max_prims ) );
		cur = pair + 1;
	}
	ext[(size_t)cur * 2] = make_float4( a.x, a.y, a.z, __uint_as_float( first + (k - 1) * max_prims ) );
	ext[(size_t)cur * 2 + 1] = make_float4( b.x, b.y, b.z, __uint_as_float( c - (k - 1) * max_prims ) );
}

// ---- MBVH<8>::ConvertFrom collapse for one level of wide nodes (:5010-5033): wide nodes lo .. lo+num-1 of `list`; their
// interior children are appended to `list` as the next level, each node's contiguously and in adoption order
__global__ void k_collapse( const float4* __restrict__ ext, uint32_t* __restrict__ list, const uint32_t lo, const uint32_t num, uint32_t* __restrict__ adopt,
	uint32_t* __restrict__ ifirst, uint32_t* __restrict__ next_count )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= num) return;
	const uint32_t w = lo + t, x = list[w];
	uint32_t c[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
	uint32_t n = 2;
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
	uint32_t ic = 0;
	for (uint32_t i = 0; i < 8; i++)
	{
		adopt[(size_t)w * 8 + i] = c[i];
		if (i < n && __float_as_uint( ext[(size_t)c[i] * 2 + 1].w ) == 0) ic++;
	}
	uint32_t at = lo + num + (ic ? atomicAdd( next_count, ic ) : 0u);
	ifirst[w] = at;
	for (uint32_t i = 0; i < n; i++) if (__float_as_uint( ext[(size_t)c[i] * 2 + 1].w ) == 0) list[at++] = c[i];
}

// ---- BVH8_CWBVH::ConvertFrom, greedy child -> slot assignment (:5910-5946) and per-node child statistics, one thread per wide node
__global__ void k_assign( const float4* __restrict__ ext, const uint32_t* __restrict__ list, const uint32_t* __restrict__ adopt, const uint32_t* __restrict__ ifirst,
	const uint32_t num, WideNode* __restrict__ wide )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= num) return;
	const uint32_t x = list[t];
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
	uint32_t wi = ifirst[t], lt = 0;
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
	if (t == 0) w.cbase = 1; // root: node 0 at address 0, its children from node 1, its triangles from record 0
	wide[t] = w;
}

// bottom-up: subtree node / triangle counts of wide nodes lo .. lo+num-1 (the next level's are final already)
__global__ void k_sizes( const uint32_t lo, const uint32_t num, WideNode* __restrict__ wide )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= num) return;
	const uint32_t x = lo + t;
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
__global__ void k_addresses( const uint32_t lo, const uint32_t num, WideNode* __restrict__ wide )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= num) return;
	const WideNode w = wide[lo + t];
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

__global__ void k_encode( const float4* __restrict__ ext, const uint32_t* __restrict__ list, const uint32_t num, const WideNode* __restrict__ wide,
	const uint32_t* __restrict__ prim_idx, const float4* __restrict__ verts, float4* __restrict__ out_nodes, float4* __restrict__ out_tris )
{
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= num) return;
	const uint32_t x = list[t];
	const WideNode w = wide[t];
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

__global__ void k_wrap_leaf_root( float4* ext, uint32_t* adopt )
{
	// MBVH<8>::ConvertFrom :5036-5044: a leaf root is copied to node 1 and the root becomes a one-child interior node
	ext[2] = ext[0], ext[3] = ext[1];
	ext[1].w = __uint_as_float( 0u );
	adopt[0] = 1;
	for (int i = 1; i < 8; i++) adopt[i] = 0;
}

// slot assignment, subtree sizes (bottom-up), addresses (top-down), encode: everything after the collapse that depends on boxes
static int cw_assign_encode( tbvh_bvh b, cudaStream_t s, const float4* ext, const uint32_t* list, const uint32_t* adopt, const uint32_t* ifirst,
	const std::vector<uint32_t>& off, WideNode* wide )
{
	const uint32_t levels = (uint32_t)off.size() - 1, wide_count = off[levels];
	k_assign<<<(wide_count + 127) / 128, 128, 0, s>>>( ext, list, adopt, ifirst, wide_count, wide ); LAUNCHED();
	for (int l = (int)levels - 1; l >= 0; l--)
	{
		const uint32_t num = off[l + 1] - off[l];
		k_sizes<<<(num + 127) / 128, 128, 0, s>>>( off[l], num, wide ); LAUNCHED();
	}
	for (uint32_t l = 0; l < levels; l++)
	{
		const uint32_t num = off[l + 1] - off[l];
		k_addresses<<<(num + 127) / 128, 128, 0, s>>>( off[l], num, wide ); LAUNCHED();
	}
	k_encode<<<(wide_count + 127) / 128, 128, 0, s>>>( ext, list, wide_count, wide, b->d_prim_idx, b->d_verts, b->d_cw_nodes, b->d_cw_tris ); LAUNCHED();
	return TBVH_OK;
}

int bvh_to_cwbvh( tbvh_bvh b, cudaStream_t s )
{
	const uint32_t used = b->info.used_nodes, idx_count = b->info.idx_count;
	std::vector<void*> scratch;
	#define CW_ALLOC( ptr, bytes ) do { CUDA_TRY( cudaMalloc( (void**)&(ptr), (bytes) ) ); scratch.push_back( (void*)(ptr) ); } while (0)
	if (b->d_cw_trav || b->d_cw_tris) b->generation = tbvh_next_generation(); // a TLAS may hold these addresses (api.cu tlas_check)
	if (b->d_cw_nodes) cudaFree( b->d_cw_nodes );
	if (b->d_cw_tris) cudaFree( b->d_cw_tris );
	if (b->d_cw_trav) cudaFree( b->d_cw_trav );
	b->d_cw_nodes = 0, b->d_cw_tris = 0, b->d_cw_trav = 0;
	cw_keep_free( b );
	uint32_t* extra = 0, * base = 0, * tile = 0, * lists = 0, * adopt = 0, * ifirst = 0, * d_count = 0;
	float4* ext = 0;
	WideNode* wide = 0;
	auto body = [&]() -> int
	{
		// ---- SplitLeafs(3)
		CW_ALLOC( extra, ((size_t)used + 1) * 4 ); CW_ALLOC( base, ((size_t)used + 1) * 4 ); CW_ALLOC( tile, ((size_t)used / 2048 + 2) * 4 );
		k_split_count<<<(used + 255) / 256, 256, 0, s>>>( b->d_nodes, extra, used, 3 ); LAUNCHED();
		{ const int r = exclusive_scan( extra, base, tile, used, s ); if (r != TBVH_OK) return r; }
		uint32_t n_extra = 0;
		CUDA_TRY( cudaMemcpyAsync( &n_extra, base + used, 4, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		const uint32_t total = used + n_extra;
		CW_ALLOC( ext, (size_t)total * 32 );
		k_split_emit<<<(used + 255) / 256, 256, 0, s>>>( b->d_nodes, base, ext, used, 3 ); LAUNCHED();
		// ---- collapse to 8-wide, level by level (a wide node is an interior node of the split tree: fewer than total)
		CW_ALLOC( lists, ((size_t)total + 1) * 4 );
		CW_ALLOC( adopt, ((size_t)total + 1) * 32 );
		CW_ALLOC( ifirst, ((size_t)total + 1) * 4 );
		CW_ALLOC( d_count, 4 );
		uint32_t rootw[8];
		CUDA_TRY( cudaMemcpyAsync( rootw, ext, 32, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		std::vector<uint32_t> off; // level l occupies lists[off[l] .. off[l+1])
		const uint32_t zero = 0;
		CUDA_TRY( cudaMemcpyAsync( lists, &zero, 4, cudaMemcpyHostToDevice, s ) ); // level 0 = { root }
		off.push_back( 0 ), off.push_back( 1 );
		const bool leaf_root = rootw[7] != 0;
		if (leaf_root) { k_wrap_leaf_root<<<1, 1, 0, s>>>( ext, adopt ); LAUNCHED(); }
		else
		{
			while (off[off.size() - 1] > off[off.size() - 2])
			{
				const uint32_t lo = off[off.size() - 2], num = off[off.size() - 1] - lo;
				CUDA_TRY( cudaMemsetAsync( d_count, 0, 4, s ) );
				k_collapse<<<(num + 127) / 128, 128, 0, s>>>( ext, lists, lo, num, adopt, ifirst, d_count ); LAUNCHED();
				uint32_t next = 0;
				CUDA_TRY( cudaMemcpyAsync( &next, d_count, 4, cudaMemcpyDeviceToHost, s ) );
				CUDA_TRY( cudaStreamSynchronize( s ) );
				off.push_back( lo + num + next );
				if (off.size() > 4096) { tbvh_set_error( "CWBVH conversion: runaway depth" ); return TBVH_E_LIMIT; }
			}
			off.pop_back(); // the last level is empty
		}
		const uint32_t levels = (uint32_t)off.size() - 1, wide_count = off[levels];
		CW_ALLOC( wide, (size_t)wide_count * sizeof( WideNode ) );
		CUDA_TRY( cudaMalloc( &b->d_cw_nodes, (size_t)wide_count * 80 ) );
		CUDA_TRY( cudaMalloc( &b->d_cw_tris, (size_t)idx_count * 48 ) );
		{ const int r = cw_assign_encode( b, s, ext, lists, adopt, ifirst, off, wide ); if (r != TBVH_OK) return r; }
		b->info.used_blocks = wide_count * 5, b->info.cwbvh_tri_count = idx_count;
		// the traversal nodes the kernels read and the pending bound of the wide tree (trace_cwbvh.cu)
		{ const int r = cw_make_trav( b, s ); if (r != TBVH_OK) return r; }
		if (b->refittable)
		{
			// keep the collapse for tbvh_refit_layouts, sized to the wide tree
			CwKeep* k = new (std::nothrow) CwKeep();
			if (!k) { tbvh_set_error( "CWBVH conversion: out of host memory" ); return TBVH_E_ARG; }
			b->cw_keep = k;
			k->used = used, k->total = total, k->wide_count = wide_count, k->leaf_root = leaf_root, k->off = off;
			CUDA_TRY( cudaMalloc( &k->base, ((size_t)used + 1) * 4 ) );
			CUDA_TRY( cudaMalloc( &k->list, (size_t)wide_count * 4 ) );
			CUDA_TRY( cudaMalloc( &k->adopt, (size_t)wide_count * 32 ) );
			CUDA_TRY( cudaMalloc( &k->ifirst, (size_t)wide_count * 4 ) );
			CUDA_TRY( cudaMemcpyAsync( k->base, base, ((size_t)used + 1) * 4, cudaMemcpyDeviceToDevice, s ) );
			CUDA_TRY( cudaMemcpyAsync( k->list, lists, (size_t)wide_count * 4, cudaMemcpyDeviceToDevice, s ) );
			CUDA_TRY( cudaMemcpyAsync( k->adopt, adopt, (size_t)wide_count * 32, cudaMemcpyDeviceToDevice, s ) );
			CUDA_TRY( cudaMemcpyAsync( k->ifirst, ifirst, (size_t)wide_count * 4, cudaMemcpyDeviceToDevice, s ) );
		}
		CUDA_TRY( cudaStreamSynchronize( s ) );
		return TBVH_OK;
	};
	const int rc = body();
	cudaStreamSynchronize( s );
	for (void* p : scratch) cudaFree( p );
	if (rc != TBVH_OK) cw_keep_free( b );
	#undef CW_ALLOC
	return rc;
}

// tbvh_refit_layouts on a handle that holds a CWBVH from tbvh_convert (b->cw_keep): d_verts already holds the new positions.
// BVH::Refit, the BVH2 traversal records, then the conversion chain over the KEPT collapse with the refitted boxes - SplitLeafs(3)
// boxes, leaf-root wrap, slot assignment, addresses, encode, traversal nodes - in place, with one synchronisation at the end.
int cwbvh_refit( tbvh_bvh b, cudaStream_t s )
{
	CwKeep* k = b->cw_keep;
	const bool first = !k->ext;
	if (first)
	{
		CUDA_TRY( cudaMalloc( &k->ext, (size_t)k->total * 32 ) );
		CUDA_TRY( cudaMalloc( &k->wide, (size_t)k->wide_count * sizeof( WideNode ) ) );
		CUDA_TRY( cudaMalloc( &k->parent, (size_t)k->used * 4 ) );
		CUDA_TRY( cudaMalloc( &k->arrive, (size_t)k->used * 4 ) );
		CUDA_TRY( cudaMalloc( &k->misc, 64 ) );
		CUDA_TRY( cudaEventCreate( &k->e0 ) );
		CUDA_TRY( cudaEventCreate( &k->e1 ) );
	}
	CUDA_TRY( cudaEventRecord( k->e0, s ) );
	{ const int r = refit_enqueue( b, s, k->parent, k->arrive, first ); if (r != TBVH_OK) return r; }
	{ const int r = make_leaf_tris( b, s ); if (r != TBVH_OK) return r; }
	k_split_emit<<<(k->used + 255) / 256, 256, 0, s>>>( b->d_nodes, k->base, k->ext, k->used, 3 ); LAUNCHED();
	if (k->leaf_root) { k_wrap_leaf_root<<<1, 1, 0, s>>>( k->ext, k->adopt ); LAUNCHED(); }
	{ const int r = cw_assign_encode( b, s, k->ext, k->list, k->adopt, k->ifirst, k->off, k->wide ); if (r != TBVH_OK) return r; }
	CUDA_TRY( cudaMemsetAsync( k->misc + 8, 0, 4, s ) );
	{ const int r = cw_expand_launch( b, s, k->misc + 8 ); if (r != TBVH_OK) return r; }
	CUDA_TRY( cudaEventRecord( k->e1, s ) );
	CUDA_TRY( cudaMemcpyAsync( k->misc, b->d_nodes, 32, cudaMemcpyDeviceToDevice, s ) );
	uint32_t h[9];
	CUDA_TRY( cudaMemcpyAsync( h, k->misc, 36, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	float ms = 0;
	CUDA_TRY( cudaEventElapsedTime( &ms, k->e0, k->e1 ) );
	b->info.build_ms = ms;
	memcpy( b->info.aabb_min, h, 12 ), memcpy( b->info.aabb_max, h + 4, 12 );
	// the exponents and origins moved: a stale limit could send rays with 2^e * rD past the float range down the integer path
	b->cw_rd_limit = cw_rd_limit_for( h[8] );
	return TBVH_OK;
}
