// tinybvh_b200/csrc/mesh_distance.cu - distances between meshes (tbvh_mesh_distance / tbvh_mesh_distance_pairs): the nearest triangle of
// mesh B for every triangle of mesh A, and every pair within a distance, over B's BVH2 with the path bound of the proximity walk and the
// triangle-triangle distance tt_dist2.  DESIGN.md 4.13 states the rules; tests/meshdist_oracle.c restates them on the host in the same fp32
// operation order.
//
// Nearest: k_mesh_distance<NEAREST>, one launch.  Pairs: k_mesh_distance<COUNT>, k_mesh_distance<FILL> and the pipeline of
// tbvh_mesh_overlap_pairs (mesh_pairs_run).
#include "tri_pair.cuh"

namespace
{
enum { MD_NEAREST = 0, MD_COUNT = 1, MD_FILL = 2 };

struct MdRec { float d; uint32_t j; }; // the 8-byte result record of one triangle of A
} // namespace

// One thread per triangle i of A in 128-thread CTAs; B's BVH2 walked as cp_walk walks it, with the box-box bound of i's box against each
// node box as the path bound and the value of a reference (leaf, j) = max( tt_dist2, LBtri, P( leaf ) ) (DESIGN.md 4.13).  SELF: B is A,
// j != i and the two share no corner (values equal as the weld rule), and the pairs passes keep j > i.  NEAREST: best starts at r2 and
// falls to the smallest ( value, j ); results[i] = { sqrt( best ), j }, or { r_max, 0xffffffff } when nothing is found or i is not finite.
// COUNT / FILL: best stays r2 and every reference with value <= r2 is counted / written as (i << 32) | j from offsets[i] on, in the same
// order.  STACKN as k_closest_point.
template <int MODE, bool SELF, int STACKN>
__global__ void __launch_bounds__( 128 ) k_mesh_distance( const float4* __restrict__ nodes, const float4* __restrict__ tris, const float4* __restrict__ vb,
	const float4* __restrict__ va, const uint64_t n, const uint32_t root_ref, const uint32_t root_count, const float r_max, MdRec* __restrict__ results,
	uint64_t* __restrict__ counts, const uint64_t* __restrict__ offsets, uint64_t* __restrict__ keys )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	V3 t[3];
	#pragma unroll
	for (int c = 0; c < 3; c++) t[c] = mo_corner( va, i * 3 + c );
	const float r2 = __fmul_rn( r_max, r_max );
	float best = r2;
	uint32_t bj = tbvh::CP_NO_PRIM;
	uint64_t found = 0, o = MODE == MD_FILL ? offsets[i] : 0;
	if (md_finite3( t ))
	{
		const V3 mn{ fminf( fminf( t[0].x, t[1].x ), t[2].x ), fminf( fminf( t[0].y, t[1].y ), t[2].y ), fminf( fminf( t[0].z, t[1].z ), t[2].z ) };
		const V3 mx{ fmaxf( fmaxf( t[0].x, t[1].x ), t[2].x ), fmaxf( fmaxf( t[0].y, t[1].y ), t[2].y ), fmaxf( fmaxf( t[0].z, t[1].z ), t[2].z ) };
		tbvh::CpEntry stack[STACKN];
		int sp = 0;
		uint32_t ref = root_ref, cnt = root_count;
		float P = 0.0f;
		while (true)
		{
			if (cnt == 0)
			{
				const float4* q = nodes + (size_t)ref * 2;
				const float4 a0 = __ldg( q ), a1 = __ldg( q + 1 ), b0 = __ldg( q + 2 ), b1 = __ldg( q + 3 );
				const float Pa = fmaxf( md_node_bound( mn, mx, a0, a1 ), P ), Pb = fmaxf( md_node_bound( mn, mx, b0, b1 ), P );
				const bool ha = !(Pa > best), hb = !(Pb > best);
				const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w ), refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
				if (ha && hb)
				{
					const bool swp = Pb < Pa; // nearer child first, the left one on ties
					ref = swp ? refb : refa, cnt = swp ? cntb : cnta, P = swp ? Pb : Pa;
					stack[sp++] = swp ? tbvh::CpEntry{ refa, cnta, Pa } : tbvh::CpEntry{ refb, cntb, Pb };
					continue;
				}
				if (ha) { ref = refa, cnt = cnta, P = Pa; continue; }
				if (hb) { ref = refb, cnt = cntb, P = Pb; continue; }
			}
			else
			{
				for (uint32_t k = 0; k < cnt; k++)
				{
					const uint32_t j = __float_as_uint( __ldg( &tris[(size_t)(ref + k) * 3].w ) );
					if (SELF && (MODE == MD_NEAREST ? j == i : j <= i)) continue;
					const V3 u[3] = { mo_corner( vb, (size_t)j * 3 ), mo_corner( vb, (size_t)j * 3 + 1 ), mo_corner( vb, (size_t)j * 3 + 2 ) };
					// the box-box bound of the two triangles first: a reference it puts above best is skipped without the pair distance
					const float lb = fmaxf( md_box_bound( mn, mx, fminf( fminf( u[0].x, u[1].x ), u[2].x ), fminf( fminf( u[0].y, u[1].y ), u[2].y ),
						fminf( fminf( u[0].z, u[1].z ), u[2].z ), fmaxf( fmaxf( u[0].x, u[1].x ), u[2].x ), fmaxf( fmaxf( u[0].y, u[1].y ), u[2].y ),
						fmaxf( fmaxf( u[0].z, u[1].z ), u[2].z ) ), P );
					if (lb > best || !md_finite3( u )) continue;
					if (SELF)
					{
						bool shared = false;
						#pragma unroll
						for (int x = 0; x < 3; x++)
							#pragma unroll
							for (int y = 0; y < 3; y++) shared |= mo_eq( t[x], u[y] );
						if (shared) continue;
					}
					const float v = fmaxf( tt_dist2( t, u ), lb );
					if (MODE == MD_NEAREST) { if (v < best || (v == best && j < bj)) best = v, bj = j; }
					else if (v <= best)
					{
						if (MODE == MD_FILL) keys[o++] = (i << 32) | j;
						else found++;
					}
				}
			}
			// pop, pruning again against the current best
			bool popped = false;
			while (sp > 0)
			{
				const tbvh::CpEntry e = stack[--sp];
				if (!(e.P > best)) { ref = e.ref, cnt = e.cnt, P = e.P, popped = true; break; }
			}
			if (!popped) break;
		}
	}
	if (MODE == MD_COUNT) counts[i] = found;
	if (MODE == MD_NEAREST) results[i] = bj == tbvh::CP_NO_PRIM ? MdRec{ r_max, bj } : MdRec{ __fsqrt_rn( best ), bj };
}

static int md_launch( int mode, tbvh_bvh a, tbvh_bvh b, float r, MdRec* results, uint64_t* counts, const uint64_t* offsets, uint64_t* keys, cudaStream_t s )
{
	const uint64_t n = a->info.prim_count;
	const uint32_t grid = (uint32_t)((n + 127) / 128);
	const bool self = a == b, deep = b->info.max_depth + 1 > TBVH_STACK;
	#define MD_ARGS <<<grid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, b->d_verts, a->d_verts, n, b->root_ref, b->root_count, r, results, counts, offsets, keys )
	#define MD_MODE( M, D ) do { if (self) k_mesh_distance<M, true, D> MD_ARGS; else k_mesh_distance<M, false, D> MD_ARGS; } while (0)
	#define MD_DEPTH( D ) do { if (mode == MD_NEAREST) MD_MODE( MD_NEAREST, D ); else if (mode == MD_COUNT) MD_MODE( MD_COUNT, D ); else MD_MODE( MD_FILL, D ); } while (0)
	if (deep) MD_DEPTH( TBVH_STACK_DEEP ); else MD_DEPTH( TBVH_STACK );
	#undef MD_DEPTH
	#undef MD_MODE
	#undef MD_ARGS
	LAUNCHED();
	return TBVH_OK;
}

// the distance argument: r >= 0, +inf allowed (NaN and negative refused)
static int md_check_r( const char* fn, const float r )
{
	if (!(r >= 0.0f)) { tbvh_set_error( "%s: the distance must be >= 0 (+inf allowed), not %g", fn, (double)r ); return TBVH_E_ARG; }
	return TBVH_OK;
}

extern "C" {

int tbvh_mesh_distance( tbvh_bvh a, tbvh_bvh b, float r_max, void* results, int space, void* stream )
{
	TRY( md_check_r( __func__, r_max ) );
	TRY( mo_check( __func__, a, b, results, true, 0, false, space, 8 ) );
	CUDA_TRY( cudaSetDevice( a->ctx->device ) );
	const uint64_t n = a->info.prim_count;
	if (n == 0) return TBVH_OK;
	if (space == TBVH_DEVICE) return md_launch( MD_NEAREST, a, b, r_max, (MdRec*)results, 0, 0, 0, (cudaStream_t)stream );
	Scratch sc( a->ctx->stream );
	MdRec* d_out = 0;
	TRY( sc.alloc( d_out, n * 8 ) );
	TRY( md_launch( MD_NEAREST, a, b, r_max, d_out, 0, 0, 0, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( results, d_out, n * 8, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaStreamSynchronize( sc.s ) );
	return TBVH_OK;
}

int tbvh_mesh_distance_pairs( tbvh_bvh a, tbvh_bvh b, float r, uint32_t* pairs, uint64_t capacity, uint64_t* count, int space, void* stream )
{
	TRY( md_check_r( __func__, r ) );
	TRY( mo_check( __func__, a, b, pairs, capacity > 0, count, true, space, 8 ) );
	return mesh_pairs_run( __func__, a, pairs, capacity, count, space, stream,
		[&]( bool fill, uint64_t* counts, const uint64_t* offsets, uint64_t* keys, cudaStream_t s ) { return md_launch( fill ? MD_FILL : MD_COUNT, a, b, r, 0, counts, offsets, keys, s ); } );
}

} // extern "C"
