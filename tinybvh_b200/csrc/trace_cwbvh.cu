// tinybvh_b200/csrc/trace_cwbvh.cu - closest-hit / any-hit traversal of BVH8_CWBVH data on sm_90a.
//
// Results are those of the reference's own walk of the same data, BVH8_CWBVH::Intersect (tiny_bvh.h:7046-7154), bit for bit:
// children of a wide node are entered in the order the format defines (inner child in slot s owns bit 24 + (s ^ o) of the
// node's hit word, o = 7 - ray octant; highest bit first), a leaf child owns `count` consecutive bits from its triangle offset,
// a child is hit iff  max( tnear_x, tnear_y, tnear_z, 0 ) <= min( tfar_x, tfar_y, tfar_z, t )  with
// t_plane = fma( q, 2^e * rD, ( p - O ) * rD ),  triangles run through the oracle's Moeller-Trumbore (common.cuh mt_test).
// This file builds the traversal nodes (cw_make_trav) and holds the single-level kernel (k_trace_wide); the walk over them
// (node_hits, cw_trace) is include/tinybvh_b200_device/cw_walk.cuh and the per-ray body tbvh::cw_trace_ray, shared with the
// two-level kernel (trace_tlas.cu) and the device functions callers' kernels use.
//
// What is different from the reference kernels (traverse_cwbvh.cl) is everything the format does not dictate:
//
//  * The kernels do not read bvh8Data.  `cw_make_trav` expands every 80-byte node once into a 160-byte TRAVERSAL NODE made for
//    this GPU (walking the byte format spends much of each node visit turning bytes into floats and testing slots that hold no
//    child - the reference's 8-wide collapse fills 4.4 of 8 slots on Bistro, 36 % of the nodes have two children):
//        header   32 B   p.xyz | 2^ex 2^ey as float top halves | first inner child | first triangle (float4 units) | 2^ez, imask, pairs | children
//        pair j   32 B   the (2j)-th and (2j+1)-th NON-EMPTY child:  lo.x lo.y lo.z hi.x hi.y hi.z as half2 (child a, child b)
//                        - 0..255 is exact in fp16 - and one 32-bit hit word per child: a leaf child's triangle bits
//                        `unary(count) << offset`, an inner child's slot bit `1 << (24 + slot)`
//    Empty slots are gone: a node holds ceil(children/2) pair records (the rest of the four are zero and contribute no bit), and a
//    visited node is nearly always full (3.83 of 4 on Bistro camera rays), so the kernel runs all four pair steps without branching -
//    four pair steps instead of eight slot steps, and the eight loads leave together.
//  * A pair step evaluates the same plane of both children (cw_walk.cuh fma2), exactly rounded per component like the scalar fma.
//  * The quantised planes reach the registers as halves and are widened by one conversion each (no byte extraction, no
//    integer-to-float on the quarter-rate unit, no magic-number subtraction).
//  * Near / far planes are picked by the sign of rD once per pair on the packed words, inner-child bits are accumulated in slot order
//    and moved to octant order by one 3-stage bit butterfly per node - and when every ray of a warp points into the same direction
//    octant (camera and shadow rays), one warp-uniform switch before the walk picks the walk compiled for that octant, where both
//    are compile-time (cw_trace<OCT>, node_hits<OCT>).
//  * The slab test's max / min chains run on the bit patterns of the plane values as signed integers, two three-input integer
//    min / max instructions per child (cw_walk.cuh pair_hits<true>); warps with a ray for which that could differ from the float
//    test (cw_ray_fits) run the float test.
//  * The per-axis scales 2^e are stored as the top halves of their float patterns: one shift or mask each instead of a byte decode.
//
// Triangles are the reference's 48-byte records (e2, e1, v0 | primIdx) read straight from bvh8Tris.
#include "common.cuh"
#include "../../include/tinybvh_b200_device.cuh"
#include <vector>

// ---- bvh8Data -> traversal nodes ------------------------------------------------------------------------------------
// One thread per node.  Slot i of the source node: meta byte i (n1.z / n1.w), quantised bounds byte i of the six 8-byte rows at
// bytes 32..79 (lo.x, lo.y, lo.z, hi.x, hi.y, hi.z) - layout in SURVEY.md 8(a), written by BVH8_CWBVH::ConvertFrom (tiny_bvh.h:5948-6015).
// One wide tree of a pass is a CwTrav (common.cuh); a single tree is a one-entry table.
// Pair record j holds the (2j)-th and (2j+1)-th non-empty slots, taken lowest first off the mask of non-empty slots, and a slot's bytes
// are picked by shifting the 8-byte rows.  Every array here is indexed by unrolled loop counters only: a record array indexed by a
// slot's running position would live in local memory.
// range: max over a tree's nodes of 128 + the largest exponent byte, or 256 for a node with e = -128 or |p| > 2^126 (cw_ray_fits)
__global__ void k_cw_expand( const CwTrav* __restrict__ T, const uint32_t K, const uint32_t W, uint32_t* __restrict__ parent )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= W) return;
	const uint32_t tree = batch_entry<CwTrav, &CwTrav::wbase>( T, K, g );
	const CwTrav& tr = T[tree];
	const uint4* __restrict__ src = tr.src;
	uint4* __restrict__ dst = tr.dst;
	uint32_t* const res = tr.res;
	const uint32_t wbase = tr.wbase, x = g - wbase, count = tr.count;
	const uint4 n0 = src[(size_t)x * 5], n1 = src[(size_t)x * 5 + 1], n2 = src[(size_t)x * 5 + 2], n3 = src[(size_t)x * 5 + 3], n4 = src[(size_t)x * 5 + 4];
	{
		const int ex = (int8_t)(n0.w & 255u), ey = (int8_t)((n0.w >> 8) & 255u), ez = (int8_t)((n0.w >> 16) & 255u);
		const bool p_ok = fabsf( __uint_as_float( n0.x ) ) <= CW_ORIGIN_LIMIT && fabsf( __uint_as_float( n0.y ) ) <= CW_ORIGIN_LIMIT && fabsf( __uint_as_float( n0.z ) ) <= CW_ORIGIN_LIMIT;
		const bool bad = !p_ok || ex == -128 || ey == -128 || ez == -128;
		const uint32_t key = bad ? 256u : (uint32_t)(128 + max( ex, max( ey, ez ) ));
		// reduced over the lanes of the same tree only: one tree's exponents never reach another's limit
		const uint32_t same = __match_any_sync( __activemask(), tree );
		const uint32_t m = __reduce_max_sync( same, key );
		if ((threadIdx.x & 31) == __ffs( same ) - 1) atomicMax( res, m );
	}
	const uint64_t meta = ((uint64_t)n1.w << 32) | n1.z;
	const uint64_t row[6] = { ((uint64_t)n2.y << 32) | n2.x, ((uint64_t)n2.w << 32) | n2.z, ((uint64_t)n3.y << 32) | n3.x, ((uint64_t)n3.w << 32) | n3.z,
		((uint64_t)n4.y << 32) | n4.x, ((uint64_t)n4.w << 32) | n4.z };
	uint32_t full = 0, inner = 0; // non-empty slots, inner children
	#pragma unroll
	for (int i = 0; i < 8; i++)
	{
		const uint32_t m = (uint32_t)(meta >> (8 * i)) & 255u;
		if (m) full |= 1u << i; // an empty slot contributes no bit whatever its box test says
		if ((m & 0x18u) == 0x18u) inner++; // 0b001sssss with sssss = 24 + slot (tiny_bvh.h:5988); a triangle offset is < 24
	}
	const uint32_t kept = __popc( full );
	uint4* o = dst + (size_t)x * CW_NODE_F4;
	// 2^e per axis as the top half of its float bit pattern, ( e + 127 ) << 7 for the signed exponent byte e - including the
	// reference's own wrap for e = -128, ( -1 ) << 23 = 0xff800000 (tiny_bvh.h:7072-7074)
	const uint32_t sx = (uint32_t)(((int)(int8_t)(n0.w & 255u) + 127) * 128) & 0xffffu, sy = (uint32_t)(((int)(int8_t)((n0.w >> 8) & 255u) + 127) * 128) & 0xffffu;
	const uint32_t sz = (uint32_t)(((int)(int8_t)((n0.w >> 16) & 255u) + 127) * 128) & 0xffffu;
	o[0] = make_uint4( n0.x, n0.y, n0.z, sx | (sy << 16) );
	o[1] = make_uint4( n1.x, n1.y, sz | ((n0.w >> 24) << 16) | (((kept + 1) >> 1) << 24), kept );
	uint32_t rest = full;
	#pragma unroll
	for (int j = 0; j < 4; j++)
	{
		uint32_t word[8] = { 0, 0, 0, 0, 0, 0, 0, 0 }; // pair record j: six planes as half2 (child a, child b), two hit words
		#pragma unroll
		for (int side = 0; side < 2; side++)
		{
			if (rest == 0) break; // the records past ceil( kept / 2 ) stay zero
			const uint32_t sh = 8 * (__ffs( rest ) - 1); // the slot's byte in meta and in the rows
			rest &= rest - 1;
			const uint32_t m = (uint32_t)(meta >> sh) & 255u;
			const bool is_inner = (m & 0x18u) == 0x18u;
			#pragma unroll
			for (int r = 0; r < 6; r++)
			{
				const uint32_t q = (uint32_t)(row[r] >> sh) & 255u;
				const uint32_t h = CW_PLANES_BF16 ? __float_as_uint( (float)q ) >> 16 : (uint32_t)__half_as_ushort( __uint2half_rn( q ) );
				word[r] |= h << (16 * side);
			}
			word[6 + side] = is_inner ? 1u << (24u + (m & 7u)) : (m >> 5) << (m & 31u);
		}
		o[2 + 2 * j] = make_uint4( word[0], word[1], word[2], word[3] );
		o[3 + 2 * j] = make_uint4( word[4], word[5], word[6], word[7] );
	}
	// inner children sit at n1.x + 0 .. inner-1 (node units): note their parent, and whether it has siblings to leave pending, for
	// the pending pass
	if (parent) for (uint32_t c = 0; c < inner; c++) if (n1.x + c < count) parent[wbase + n1.x + c] = x | (inner >= 2 ? 0x80000000u : 0u);
}

// The walk pushes a node group only when the node it enters has inner siblings still to visit (cw_trace: rest > 0x00ffffff), so
// at a node it holds at most one group per ancestor with two or more inner children.  The largest such count over the nodes is
// what the pending stack must hold - on a chain (the 3-triangle leaves SplitLeafs makes of a long leaf) far less than the depth.
// It is found by pointer jumping: every node keeps an ancestor and the count of flagged nodes up to it, and each pass doubles
// the distance (anc' = anc(anc), cnt' = cnt + cnt(anc)), so ceil( log2( count ) ) + 1 passes reach the root from any node.  A node
// still short of the root then lies on a cycle (uploaded data): the tree is reported as such.  The trees of a batch jump together
// over one index space (W nodes); parent links never leave a tree.
#define CW_ROOT 0xffffffffu   // ancestor past the root
#define CW_CYCLE 0xffffffffu  // cw_pending of a tree with a cycle
__global__ void k_cw_jump_init( const CwTrav* __restrict__ T, const uint32_t K, const uint32_t* __restrict__ parent, const uint32_t W, uint32_t* __restrict__ anc, uint32_t* __restrict__ cnt )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= W) return;
	const uint32_t wb = T[batch_entry<CwTrav, &CwTrav::wbase>( T, K, g )].wbase, p = parent[g];
	// the root steps past itself - unless some node names it as a child, a cycle a walk would never leave: it then stays on itself;
	// a record no node points at (0xffffffff) gets ancestor W (out of range) and is not counted
	anc[g] = g == wb ? (p == 0xffffffffu ? CW_ROOT : g) : p == 0xffffffffu ? W : wb + (p & 0x7fffffffu), cnt[g] = (g == wb || p == 0xffffffffu) ? 0u : p >> 31;
}
__global__ void k_cw_jump( const uint32_t W, const uint32_t* __restrict__ anc, const uint32_t* __restrict__ cnt, uint32_t* __restrict__ anc2, uint32_t* __restrict__ cnt2 )
{
	const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= W) return;
	const uint32_t a = anc[x];
	if (a < W) anc2[x] = anc[a], cnt2[x] = min( cnt[x] + cnt[a], 0x40000000u );
	else anc2[x] = a, cnt2[x] = cnt[x];
}
__global__ void k_cw_pending( const CwTrav* __restrict__ T, const uint32_t K, const uint32_t W, const uint32_t* __restrict__ anc, const uint32_t* __restrict__ cnt )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= W) return;
	const uint32_t a = anc[g];
	uint32_t* pending = T[batch_entry<CwTrav, &CwTrav::wbase>( T, K, g )].res + 1;
	if (a == CW_ROOT) atomicMax( pending, cnt[g] );
	else if (a < W) atomicMax( pending, CW_CYCLE );
}

// k_cw_expand of the W nodes of the K trees of d_T into their allocated traversal nodes.  parent: where the pending pass finds every
// node's parent, or NULL (a refit: the topology and the pending bound stay)
int cw_expand( const CwTrav* d_T, const uint32_t K, const uint32_t W, uint32_t* parent, cudaStream_t s )
{
	k_cw_expand<<<(W + 127) / 128, 128, 0, s>>>( d_T, K, W, parent );
	LAUNCHED();
	return TBVH_OK;
}

// |rD| <= 2^( 127 - largest e ) keeps 2^e * rD finite (cw_ray_fits); 2^127 at most, and no ray fits a tree that has range 256
float cw_rd_limit_for( uint32_t range ) { return range < 256 ? ldexpf( 1.0f, 127 - max( 0, (int)range - 128 ) ) : -1.0f; }

int cw_make_trav( const tbvh_bvh* bs, const uint32_t K, cudaStream_t s )
{
	std::vector<CwTrav> T( K );
	uint32_t W = 0, most = 0; // nodes of the pass (the conversion's batch bound keeps it a uint32_t), nodes of the largest tree
	for (uint32_t t = 0; t < K; t++)
	{
		const tbvh_bvh b = bs[t];
		b->cw_pending = 0xffffffffu, b->cw_rd_limit = -1.0f;
		const uint32_t count = b->info.used_blocks / 5;
		if (count == 0) { tbvh_set_error( "cw_make_trav: no CWBVH nodes" ); return TBVH_E_STATE; }
		T[t] = CwTrav{ (const uint4*)b->d_cw_nodes.p, 0, 0, W, count };
		W += count, most = max( most, count );
	}
	for (uint32_t t = 0; t < K; t++)
	{
		TRY( bs[t]->d_cw_trav.alloc( (size_t)T[t].count * CW_NODE_F4 * 16 ) );
		T[t].dst = (uint4*)bs[t]->d_cw_trav.p;
	}
	std::vector<uint32_t> res( (size_t)K * 2 ); // range, pending bound per tree
	Scratch sc( s );
	// every node notes its parent, then the counts of ancestors that leave node groups pending are summed up to the root
	const size_t words = (((size_t)W * 5 + (size_t)K * 2) + 63) & ~(size_t)63; // the tree table follows, 256-byte aligned
	uint32_t* d_parent = 0;
	TRY( sc.alloc( d_parent, words * 4 + (size_t)K * sizeof( CwTrav ) ) );
	CwTrav* const d_T = (CwTrav*)(d_parent + words);
	uint32_t* const anc[2] = { d_parent + W, d_parent + 2 * (size_t)W }, * const cnt[2] = { d_parent + 3 * (size_t)W, d_parent + 4 * (size_t)W };
	uint32_t* const d_res = d_parent + 5 * (size_t)W;
	for (uint32_t t = 0; t < K; t++) T[t].res = d_res + 2 * (size_t)t;
	CUDA_TRY( cudaMemcpyAsync( d_T, T.data(), (size_t)K * sizeof( CwTrav ), cudaMemcpyHostToDevice, s ) );
	CUDA_TRY( cudaMemsetAsync( d_parent, 0xff, (size_t)W * 4, s ) );
	CUDA_TRY( cudaMemsetAsync( d_res, 0, (size_t)K * 8, s ) );
	TRY( cw_expand( d_T, K, W, d_parent, s ) );
	const uint32_t g = (W + 127) / 128;
	k_cw_jump_init<<<g, 128, 0, s>>>( d_T, K, d_parent, W, anc[0], cnt[0] ); LAUNCHED();
	int cur = 0;
	for (uint32_t reach = 1; reach < 2 * most; reach *= 2, cur ^= 1) { k_cw_jump<<<g, 128, 0, s>>>( W, anc[cur], cnt[cur], anc[cur ^ 1], cnt[cur ^ 1] ); LAUNCHED(); }
	k_cw_pending<<<g, 128, 0, s>>>( d_T, K, W, anc[cur], cnt[cur] ); LAUNCHED();
	CUDA_TRY( cudaMemcpyAsync( res.data(), d_res, (size_t)K * 8, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	for (uint32_t t = 0; t < K; t++) bs[t]->cw_pending = res[2 * (size_t)t + 1], bs[t]->cw_rd_limit = cw_rd_limit_for( res[2 * (size_t)t] );
	return TBVH_OK;
}

// ---- traversal ------------------------------------------------------------------------------------------------------

// OCTSW = 1: warps whose rays all point into one direction octant (camera and shadow rays: nearly all of them) walk with the
// instance compiled for that octant, picked once per warp before the walk; mixed warps use the per-lane form.  Warps in which
// every ray passes cw_ray_fits (rd_limit: cw_make_trav) run the integer-ordered slab test; any other warp runs the float test.
template <bool ANYHIT, bool STATS, int OCTSW>
__global__ void __launch_bounds__( 128 ) k_trace_wide( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	const char* rays, const uint32_t stride, char* hits, const uint32_t hit_stride, uint32_t* __restrict__ bits, const uint64_t n,
	unsigned long long* __restrict__ stats, const float rd_limit )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	bool occluded = false;
	const bool valid = i < n;
	float4 ro4 = make_float4( 0, 0, 0, 0 ), rd4 = ro4, rr4 = ro4, rh4 = ro4;
	if (valid) load_ray( rays, i, stride, ro4, rd4, rr4, rh4 );
	const float ox = ro4.x, oy = ro4.y, oz = ro4.z, dx = rd4.x, dy = rd4.y, dz = rd4.z;
	const float rdx = rr4.x, rdy = rr4.y, rdz = rr4.z;
	const uint32_t o = 7u - ((dx < 0 ? 4u : 0u) | (dy < 0 ? 2u : 0u) | (dz < 0 ? 1u : 0u)); // octinv of tiny_bvh.h:7053 (signs of D)
	const bool negx = rdx < 0, negy = rdy < 0, negz = rdz < 0;                                // plane swizzle uses rD (:7082)
	const uint32_t oct = (negx ? 4u : 0u) | (negy ? 2u : 0u) | (negz ? 1u : 0u);
	bool uni = false;
	if (OCTSW)
	{
		// the compiled-in octant serves both the plane choice (signs of rD) and the visiting order (signs of D): they must agree
		const uint32_t vm = __ballot_sync( 0xffffffffu, valid );
		const uint32_t oct0 = __shfl_sync( 0xffffffffu, oct, vm ? __ffs( vm ) - 1 : 0 );
		uni = __all_sync( 0xffffffffu, !valid || (oct == oct0 && o == 7u - oct) );
	}
	const bool iord = __all_sync( 0xffffffffu, !valid || tbvh::cw_ray_fits( ox, oy, oz, rdx, rdy, rdz, rd_limit ) );
	if (valid)
	{
		uint2 pending[CW_STACK];
		occluded = tbvh::cw_trace_ray<ANYHIT, STATS>( nodes, tris, ox, oy, oz, dx, dy, dz, rdx, rdy, rdz, rh4, (float4*)(hits + i * hit_stride), o, oct, negx,
			negy, negz, OCTSW && uni && iord, iord, pending, stats );
	}
	if (ANYHIT) store_occlusion_word( bits, i, n, occluded );
}

int cwbvh_trace_check( tbvh_bvh b, uint64_t n )
{
	if (!b->d_cw_trav || !b->d_cw_tris) { tbvh_set_error( "CWBVH layout not resident" ); return TBVH_E_STATE; }
	if (n == 0) return TBVH_OK;
	if (b->cw_pending == CW_CYCLE) { tbvh_set_error( "the wide tree's inner-child links form a cycle" ); return TBVH_E_ARG; }
	if (b->cw_pending > CW_STACK) { tbvh_set_error( "the wide tree can leave %u node groups pending, more than the %d a ray can hold (the reference's own limit)", b->cw_pending, CW_STACK ); return TBVH_E_LIMIT; }
	return TBVH_OK;
}

int cwbvh_trace_launch( tbvh_bvh b, const void* d_rays, uint32_t stride, void* d_hits, uint32_t hit_stride, uint32_t* d_bits,
	uint64_t n, bool anyhit, cudaStream_t s, unsigned long long* d_stats )
{
	TRY( cwbvh_trace_check( b, n ) );
	if (n == 0) return TBVH_OK;
	const uint32_t block = 128;
	const uint64_t grid = (n + block - 1) / block;
	if (grid > 0x7fffffffull) { tbvh_set_error( "ray batch too large for one launch" ); return TBVH_E_ARG; }
	const int sw = b->ctx->trace_variant == 0 ? 0 : 1; // trace_variant 0: the per-lane form only (A/B switch for measurements)
	#define LAUNCH( A, S, O ) k_trace_wide<A, S, O><<<(uint32_t)grid, block, 0, s>>>( b->d_cw_trav, b->d_cw_tris, (const char*)d_rays, stride, \
		(char*)d_hits, hit_stride, d_bits, n, d_stats, b->cw_rd_limit )
	if (anyhit) { if (d_stats) LAUNCH( true, true, 0 ); else if (sw) LAUNCH( true, false, 1 ); else LAUNCH( true, false, 0 ); }
	else { if (d_stats) LAUNCH( false, true, 0 ); else if (sw) LAUNCH( false, false, 1 ); else LAUNCH( false, false, 0 ); }
	#undef LAUNCH
	LAUNCHED();
	return TBVH_OK;
}
