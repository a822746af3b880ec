// tinybvh_b200/csrc/mesh_toi.cu - times of impact between moving meshes (tbvh_mesh_toi / tbvh_mesh_toi_pairs): every vertex moves
// linearly from the handle's vertices (t = 0) to the call's end frame (t = 1), and for every triangle of mesh A the first time a triangle
// of mesh B comes within eta + xi, by conservative advancement on the pair distance tt_dist2 of 4.13, over B's BVH2 with swept boxes.
// DESIGN.md 4.15 states the rules; tests/toi_oracle.c restates them on the host in the same fp32 operation order.
//
// Every call: the end frames staged to float4 rows, k_swept_leaves and max_depth k_swept_pass launches (the swept boxes of B's slots),
// then nearest: k_mesh_toi<NEAREST>; pairs: k_mesh_toi<COUNT>, k_mesh_toi<FILL> and the pipeline of tbvh_mesh_overlap_pairs
// (mesh_pairs_run), and k_toi_times when the caller asks for the times.
#include "tri_pair.cuh"
#include <algorithm>

#define MT_MAX_ITERS (1u << 16) // the largest max_iters a call takes
// L is rounded up by 2^-16 of itself: its fp32 evaluation (the nine differences, the norm's fma chain and the square root) is within a
// few 2^-24 of the value on the rounded displacements
#define MT_L_UP 1.0000152587890625f

namespace
{
enum { MT_NEAREST = 0, MT_COUNT = 1, MT_FILL = 2 };

struct MtRec { float t, d; uint32_t j, iters; }; // the 16-byte result record of one triangle of A

// the position at t of a corner moving from x0 to x1: fma( t, x1, fma( -t, x0, x0 ) ), exactly x0 at 0 and x1 at 1
__device__ __forceinline__ V3 mt_at( const V3& x0, const V3& x1, const float t )
{
	return V3{ __fmaf_rn( t, x1.x, __fmaf_rn( -t, x0.x, x0.x ) ), __fmaf_rn( t, x1.y, __fmaf_rn( -t, x0.y, x0.y ) ), __fmaf_rn( t, x1.z, __fmaf_rn( -t, x0.z, x0.z ) ) };
}
__device__ __forceinline__ float mt_n2( const V3& w ) { return __fmaf_rn( w.z, w.z, __fmaf_rn( w.y, w.y, __fmul_rn( w.x, w.x ) ) ); }

// L( T, U ): the largest |dT_a - dU_b| over the nine corner pairs, d = x1 - x0, rounded up by MT_L_UP; symmetric bit for bit
__device__ __forceinline__ float mt_speed( const V3* t0, const V3* t1, const V3* u0, const V3* u1 )
{
	const V3 dT[3] = { v3sub( t1[0], t0[0] ), v3sub( t1[1], t0[1] ), v3sub( t1[2], t0[2] ) };
	const V3 dU[3] = { v3sub( u1[0], u0[0] ), v3sub( u1[1], u0[1] ), v3sub( u1[2], u0[2] ) };
	float m = 0.0f;
	#pragma unroll
	for (int a = 0; a < 3; a++)
		#pragma unroll
		for (int b = 0; b < 3; b++) m = fmaxf( m, mt_n2( v3sub( dT[a], dU[b] ) ) );
	return __fmul_rn( __fsqrt_rn( m ), MT_L_UP );
}

// Conservative advancement of one finite pair (DESIGN.md 4.15): true with the contact time t, the squared distance v at t and the
// iterations it (max_iters: unresolved), false for no contact within the step.  ABANDON: false as soon as the iterate ( t, j ) exceeds
// ( bt, bj ), which the iterates, only growing, never come back below.
template <bool ABANDON>
__device__ __forceinline__ bool mt_pair( const V3* t0, const V3* t1, const V3* u0, const V3* u1, const float eta, const float R2, const uint32_t max_iters,
	const uint32_t j, const float bt, const uint32_t bj, float& t, float& v, uint32_t& it )
{
	const float L = mt_speed( t0, t1, u0, u1 );
	t = 0.0f, it = 0;
	while (true)
	{
		if (ABANDON && (t > bt || (t == bt && j > bj))) return false;
		const V3 T[3] = { mt_at( t0[0], t1[0], t ), mt_at( t0[1], t1[1], t ), mt_at( t0[2], t1[2], t ) };
		const V3 U[3] = { mt_at( u0[0], u1[0], t ), mt_at( u0[1], u1[1], t ), mt_at( u0[2], u1[2], t ) };
		v = tt_dist2( T, U );
		if (v <= R2) return true;
		if (L == 0.0f) return false;
		const float tn = __fadd_rn( t, __fdiv_rn( __fsub_rn( __fsqrt_rn( v ), eta ), L ) );
		if (!(tn <= 1.0f)) return false;
		if (tn == t || it == max_iters) { it = max_iters; return true; }
		t = tn, it++;
	}
}

__device__ __forceinline__ void mt_grow( V3& mn, V3& mx, const V3& p )
{
	mn = V3{ fminf( mn.x, p.x ), fminf( mn.y, p.y ), fminf( mn.z, p.z ) }, mx = V3{ fmaxf( mx.x, p.x ), fmaxf( mx.y, p.y ), fmaxf( mx.z, p.z ) };
}
// the swept box of a triangle: the box of its six corners (min and max only)
__device__ __forceinline__ void mt_box( const V3* c0, const V3* c1, V3& mn, V3& mx )
{
	mn = c0[0], mx = c0[0];
	mt_grow( mn, mx, c0[1] ), mt_grow( mn, mx, c0[2] ), mt_grow( mn, mx, c1[0] ), mt_grow( mn, mx, c1[1] ), mt_grow( mn, mx, c1[2] );
}
__device__ __forceinline__ bool mt_finite( const V3* c0, const V3* c1 ) { return md_finite3( c0 ) && md_finite3( c1 ); }
} // namespace

// The swept boxes of B's slots, in an array laid out as trav() (two float4 per slot, the w words copied): a leaf slot gets the box of
// both frames' corners of every triangle it references, an interior slot the empty box (+inf, -inf).  Leaf ranges and triangles
// outside the arrays (slots no walk reaches) add nothing.
__global__ void k_swept_leaves( const float4* __restrict__ nodes, const float4* __restrict__ tris, const float4* __restrict__ v0, const float4* __restrict__ v1,
	const uint32_t S, const uint32_t refs, const uint32_t prims, float4* __restrict__ sb )
{
	const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= S) return;
	const float4 lo = nodes[(size_t)x * 2], hi = nodes[(size_t)x * 2 + 1];
	const uint32_t ref = __float_as_uint( lo.w ), cnt = __float_as_uint( hi.w );
	const float inf = __int_as_float( 0x7f800000 );
	V3 mn{ inf, inf, inf }, mx{ -inf, -inf, -inf };
	for (uint32_t k = ref; cnt && k < refs && k - ref < cnt; k++)
	{
		const uint32_t j = __float_as_uint( tris[(size_t)k * 3].w );
		if (j >= prims) continue;
		#pragma unroll
		for (int c = 0; c < 3; c++) mt_grow( mn, mx, mo_corner( v0, (size_t)j * 3 + c ) ), mt_grow( mn, mx, mo_corner( v1, (size_t)j * 3 + c ) );
	}
	sb[(size_t)x * 2] = make_float4( mn.x, mn.y, mn.z, lo.w ), sb[(size_t)x * 2 + 1] = make_float4( mx.x, mx.y, mx.z, hi.w );
}

// One pass of interior slots: the union of the two children's boxes.  The boxes only grow towards their fixed point and a pass reads
// each child's box as it is, so after max_depth passes every slot a walk reaches holds the box of its subtree, trees, DAGs and slots
// a walk reaches on several paths alike; min and max make the bits independent of the order.
__global__ void k_swept_pass( float4* sb, const uint32_t S )
{
	const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
	if (x >= S) return;
	const float4 lo = sb[(size_t)x * 2], hi = sb[(size_t)x * 2 + 1];
	const uint32_t c = __float_as_uint( lo.w );
	if (__float_as_uint( hi.w ) != 0 || c >= S - 1) return;
	const float4 al = sb[(size_t)c * 2], ah = sb[(size_t)c * 2 + 1], bl = sb[(size_t)c * 2 + 2], bh = sb[(size_t)c * 2 + 3];
	sb[(size_t)x * 2] = make_float4( fminf( al.x, bl.x ), fminf( al.y, bl.y ), fminf( al.z, bl.z ), lo.w );
	sb[(size_t)x * 2 + 1] = make_float4( fmaxf( ah.x, bh.x ), fmaxf( ah.y, bh.y ), fmaxf( ah.z, bh.z ), hi.w );
}

// One thread per triangle i of A in 128-thread CTAs; B's swept boxes walked with the box-box bound of 4.13 against i's swept box at
// R2 = ( eta + xi )^2 (the root untested), and every reached reference (leaf, j) whose swept box passes the same bound, both
// triangles finite (and, SELF, j != i sharing no corner in both frames) advanced by mt_pair.  NEAREST: results[i] = the smallest
// ( t, j ) with d = sqrt( v ) at t, or { +inf, +inf, 0xffffffff, 0 }; a pair is abandoned once it cannot beat the best so far.
// COUNT / FILL: every reached pair in contact within the step is counted / written as (i << 32) | j from offsets[i] on, pairs j > i
// when SELF.  STACKN as k_closest_point.
template <int MODE, bool SELF, int STACKN>
__global__ void __launch_bounds__( 128 ) k_mesh_toi( const float4* __restrict__ sb, const float4* __restrict__ tris, const float4* __restrict__ vb0,
	const float4* __restrict__ vb1, const float4* __restrict__ va0, const float4* __restrict__ va1, const uint64_t n, const uint32_t root_ref,
	const uint32_t root_count, const float eta, const float R2, const uint32_t max_iters, MtRec* __restrict__ results, uint64_t* __restrict__ counts,
	const uint64_t* __restrict__ offsets, uint64_t* __restrict__ keys )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	V3 t0[3], t1[3];
	#pragma unroll
	for (int c = 0; c < 3; c++) t0[c] = mo_corner( va0, i * 3 + c ), t1[c] = mo_corner( va1, i * 3 + c );
	const float inf = __int_as_float( 0x7f800000 );
	float bt = inf, bv = inf;
	uint32_t bj = tbvh::CP_NO_PRIM, bit = 0;
	uint64_t found = 0, o = MODE == MT_FILL ? offsets[i] : 0;
	if (mt_finite( t0, t1 ))
	{
		V3 mn, mx;
		mt_box( t0, t1, mn, mx );
		uint2 stack[STACKN];
		int sp = 0;
		uint32_t ref = root_ref, cnt = root_count;
		while (true)
		{
			if (cnt == 0)
			{
				const float4* q = sb + (size_t)ref * 2;
				const float4 a0 = __ldg( q ), a1 = __ldg( q + 1 ), b0 = __ldg( q + 2 ), b1 = __ldg( q + 3 );
				const bool ha = !(md_node_bound( mn, mx, a0, a1 ) > R2), hb = !(md_node_bound( mn, mx, b0, b1 ) > R2);
				const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w ), refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
				if (ha && hb) { stack[sp++] = make_uint2( refb, cntb ); ref = refa, cnt = cnta; continue; }
				if (ha) { ref = refa, cnt = cnta; continue; }
				if (hb) { ref = refb, cnt = cntb; continue; }
			}
			else
			{
				for (uint32_t k = 0; k < cnt; k++)
				{
					const uint32_t j = __float_as_uint( __ldg( &tris[(size_t)(ref + k) * 3].w ) );
					if (SELF && (MODE == MT_NEAREST ? j == i : j <= i)) continue;
					V3 u0[3], u1[3];
					#pragma unroll
					for (int c = 0; c < 3; c++) u0[c] = mo_corner( vb0, (size_t)j * 3 + c ), u1[c] = mo_corner( vb1, (size_t)j * 3 + c );
					V3 umn, umx;
					mt_box( u0, u1, umn, umx );
					if (md_box_bound( mn, mx, umn.x, umn.y, umn.z, umx.x, umx.y, umx.z ) > R2 || !mt_finite( u0, u1 )) continue;
					if (SELF)
					{
						bool shared = false;
						#pragma unroll
						for (int x = 0; x < 3; x++)
							#pragma unroll
							for (int y = 0; y < 3; y++) shared |= mo_eq( t0[x], u0[y] ) && mo_eq( t1[x], u1[y] );
						if (shared) continue;
					}
					float t, v;
					uint32_t it;
					if (MODE == MT_NEAREST)
					{
						if (mt_pair<true>( t0, t1, u0, u1, eta, R2, max_iters, j, bt, bj, t, v, it ) && (t < bt || (t == bt && j < bj))) bt = t, bv = v, bj = j, bit = it;
					}
					else if (mt_pair<false>( t0, t1, u0, u1, eta, R2, max_iters, j, 0.0f, 0, t, v, it ))
					{
						if (MODE == MT_FILL) keys[o++] = (i << 32) | j;
						else found++;
					}
				}
			}
			if (sp == 0) break;
			const uint2 e = stack[--sp];
			ref = e.x, cnt = e.y;
		}
	}
	if (MODE == MT_COUNT) counts[i] = found;
	if (MODE == MT_NEAREST)
	{
		const MtRec r = bj == tbvh::CP_NO_PRIM ? MtRec{ inf, inf, bj, 0 } : MtRec{ bt, __fsqrt_rn( bv ), bj, bit };
		reinterpret_cast<uint4*>( results )[i] = make_uint4( __float_as_uint( r.t ), __float_as_uint( r.d ), r.j, r.iters );
	}
}

// the contact time of each of the m pairs { i, j }, from the pair alone (mt_pair without abandoning)
__global__ void __launch_bounds__( 128 ) k_toi_times( const uint32_t* __restrict__ pairs, const uint64_t m, const float4* __restrict__ va0, const float4* __restrict__ va1,
	const float4* __restrict__ vb0, const float4* __restrict__ vb1, const float eta, const float R2, const uint32_t max_iters, float* __restrict__ times )
{
	const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= m) return;
	const uint32_t i = pairs[k * 2], j = pairs[k * 2 + 1];
	V3 t0[3], t1[3], u0[3], u1[3];
	#pragma unroll
	for (int c = 0; c < 3; c++)
	{
		t0[c] = mo_corner( va0, (size_t)i * 3 + c ), t1[c] = mo_corner( va1, (size_t)i * 3 + c );
		u0[c] = mo_corner( vb0, (size_t)j * 3 + c ), u1[c] = mo_corner( vb1, (size_t)j * 3 + c );
	}
	float t, v;
	uint32_t it;
	times[k] = mt_pair<false>( t0, t1, u0, u1, eta, R2, max_iters, j, 0.0f, 0, t, v, it ) ? t : __int_as_float( 0x7f800000 );
}

namespace
{
// device blocks of one call, allocated and freed in the order of stream s (stream-ordered allocation), so a device-space call stays
// asynchronous on the caller's stream
struct MtBufs
{
	cudaStream_t s;
	std::vector<void*> p;
	explicit MtBufs( cudaStream_t stream ) : s( stream ) {}
	MtBufs( const MtBufs& ) = delete;
	MtBufs& operator=( const MtBufs& ) = delete;
	~MtBufs() { for (void* q : p) cudaFreeAsync( q, s ); }
	template <class T> int alloc( T*& q, size_t bytes ) { void* x = 0; CUDA_TRY( cudaMallocAsync( &x, bytes, s ) ); p.push_back( x ); q = (T*)x; return TBVH_OK; }
};

// the end frames and B's swept boxes of one call, on bufs.s
struct MtFrames { const float4* a1; const float4* b1; float4* sb; };
} // namespace

static int mt_prepare( tbvh_bvh a, const void* a_end, uint32_t a_stride, tbvh_bvh b, const void* b_end, uint32_t b_stride, int space, MtBufs& bufs, MtFrames& f )
{
	const cudaStream_t s = bufs.s;
	float4* e = 0;
	TRY( bufs.alloc( e, (size_t)a->info.prim_count * 48 ) );
	TRY( copy_rows( e, a_end, a_stride, (size_t)a->info.prim_count * 3, space, s ) );
	f.a1 = e;
	if (b != a)
	{
		TRY( bufs.alloc( e, (size_t)b->info.prim_count * 48 ) );
		TRY( copy_rows( e, b_end, b_stride, (size_t)b->info.prim_count * 3, space, s ) );
	}
	f.b1 = e;
	const uint32_t S = trav_slots( b );
	TRY( bufs.alloc( f.sb, (size_t)S * 32 ) );
	const uint32_t g = (S + 255) / 256;
	k_swept_leaves<<<g, 256, 0, s>>>( b->trav(), b->d_leaf_tris, b->d_verts, f.b1, S, b->info.idx_count, b->info.prim_count, f.sb ); LAUNCHED();
	for (uint32_t k = 0; k < b->info.max_depth; k++) { k_swept_pass<<<g, 256, 0, s>>>( f.sb, S ); LAUNCHED(); }
	return TBVH_OK;
}

static int mt_launch( int mode, tbvh_bvh a, tbvh_bvh b, const MtFrames& f, float eta, float R2, uint32_t max_iters, MtRec* results, uint64_t* counts,
	const uint64_t* offsets, uint64_t* keys, cudaStream_t s )
{
	const uint64_t n = a->info.prim_count;
	const uint32_t grid = (uint32_t)((n + 127) / 128);
	const bool self = a == b, deep = b->info.max_depth + 1 > TBVH_STACK;
	#define MT_ARGS <<<grid, 128, 0, s>>>( f.sb, b->d_leaf_tris, b->d_verts, f.b1, a->d_verts, f.a1, n, b->root_ref, b->root_count, eta, R2, max_iters, results, counts, offsets, keys )
	#define MT_MODE( M, D ) do { if (self) k_mesh_toi<M, true, D> MT_ARGS; else k_mesh_toi<M, false, D> MT_ARGS; } while (0)
	#define MT_DEPTH( D ) do { if (mode == MT_NEAREST) MT_MODE( MT_NEAREST, D ); else if (mode == MT_COUNT) MT_MODE( MT_COUNT, D ); else MT_MODE( MT_FILL, D ); } while (0)
	if (deep) MT_DEPTH( TBVH_STACK_DEEP ); else MT_DEPTH( TBVH_STACK );
	#undef MT_DEPTH
	#undef MT_MODE
	#undef MT_ARGS
	LAUNCHED();
	return TBVH_OK;
}

// the refusals of both calls that precede mo_check's (TBVH_E_ARG)
static int mt_check( const char* fn, tbvh_bvh a, const void* a_end, uint32_t a_stride, tbvh_bvh b, const void* b_end, uint32_t b_stride, float eta, float xi, uint32_t max_iters )
{
	if (!(eta >= 0.0f && eta <= 3.402823466e38f)) { tbvh_set_error( "%s: eta must be finite and >= 0, not %g", fn, (double)eta ); return TBVH_E_ARG; }
	if (!(xi > 0.0f && xi <= 3.402823466e38f)) { tbvh_set_error( "%s: xi must be finite and > 0, not %g", fn, (double)xi ); return TBVH_E_ARG; }
	if (max_iters == 0 || max_iters > MT_MAX_ITERS) { tbvh_set_error( "%s: max_iters must be in [1, %u], not %u", fn, MT_MAX_ITERS, max_iters ); return TBVH_E_ARG; }
	if (!a_end || !b_end) { tbvh_set_error( "%s: NULL end frame", fn ); return TBVH_E_ARG; }
	if (a_stride < 12 || (a_stride & 3) || b_stride < 12 || (b_stride & 3)) { tbvh_set_error( "%s: an end-frame stride must be >= 12 and a multiple of 4", fn ); return TBVH_E_ARG; }
	if (a == b && (b_end != a_end || b_stride != a_stride)) { tbvh_set_error( "%s: a self query takes one end frame (b_end, b_stride equal to a_end, a_stride)", fn ); return TBVH_E_ARG; }
	return TBVH_OK;
}

static float mt_r2( float eta, float xi ) { const float e = eta + xi; return e * e; }

extern "C" {

int tbvh_mesh_toi( tbvh_bvh a, const void* a_end, uint32_t a_stride, tbvh_bvh b, const void* b_end, uint32_t b_stride, float eta, float xi, uint32_t max_iters,
	void* results, int space, void* stream )
{
	TRY( mt_check( __func__, a, a_end, a_stride, b, b_end, b_stride, eta, xi, max_iters ) );
	TRY( mo_check( __func__, a, b, results, true, 0, false, space, 16 ) );
	CUDA_TRY( cudaSetDevice( a->ctx->device ) );
	const uint64_t n = a->info.prim_count;
	if (n == 0) return TBVH_OK;
	const float R2 = mt_r2( eta, xi );
	if (space == TBVH_DEVICE)
	{
		MtBufs bufs( (cudaStream_t)stream );
		MtFrames f;
		TRY( mt_prepare( a, a_end, a_stride, b, b_end, b_stride, space, bufs, f ) );
		return mt_launch( MT_NEAREST, a, b, f, eta, R2, max_iters, (MtRec*)results, 0, 0, 0, bufs.s );
	}
	Scratch sc( a->ctx->stream );
	MtBufs bufs( sc.s ); // freed before sc drains the stream
	MtFrames f;
	MtRec* d_out = 0;
	TRY( bufs.alloc( d_out, n * 16 ) );
	TRY( mt_prepare( a, a_end, a_stride, b, b_end, b_stride, space, bufs, f ) );
	TRY( mt_launch( MT_NEAREST, a, b, f, eta, R2, max_iters, d_out, 0, 0, 0, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( results, d_out, n * 16, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaStreamSynchronize( sc.s ) );
	return TBVH_OK;
}

int tbvh_mesh_toi_pairs( tbvh_bvh a, const void* a_end, uint32_t a_stride, tbvh_bvh b, const void* b_end, uint32_t b_stride, float eta, float xi, uint32_t max_iters,
	uint32_t* pairs, float* times, uint64_t capacity, uint64_t* count, int space, void* stream )
{
	TRY( mt_check( __func__, a, a_end, a_stride, b, b_end, b_stride, eta, xi, max_iters ) );
	if (space == TBVH_DEVICE && ((uintptr_t)times & 3)) { tbvh_set_error( "%s: the device times must be 4-byte aligned", __func__ ); return TBVH_E_ARG; }
	TRY( mo_check( __func__, a, b, pairs, capacity > 0, count, true, space, 8 ) );
	const float R2 = mt_r2( eta, xi );
	Scratch sc( a->ctx->stream ); // drains the engine stream on return, after bufs has queued its frees
	MtBufs bufs( a->ctx->stream );
	MtFrames f = {};
	bool ready = false;
	TRY( mesh_pairs_run( __func__, a, pairs, capacity, count, space, stream,
		[&]( bool fill, uint64_t* counts, const uint64_t* offsets, uint64_t* keys, cudaStream_t s ) {
			if (!ready) { TRY( mt_prepare( a, a_end, a_stride, b, b_end, b_stride, space, bufs, f ) ); ready = true; }
			return mt_launch( fill ? MT_FILL : MT_COUNT, a, b, f, eta, R2, max_iters, 0, counts, offsets, keys, s ); } ) );
	const uint64_t m = std::min( *count, capacity );
	if (!times || m == 0) return TBVH_OK;
	// mesh_pairs_run has drained the engine stream: the pairs are in place
	const cudaStream_t s = sc.s;
	const uint32_t* d_pairs = pairs;
	float* d_times = times;
	if (space == TBVH_HOST)
	{
		uint32_t* p = 0;
		TRY( bufs.alloc( p, m * 8 ) );
		TRY( bufs.alloc( d_times, m * 4 ) );
		CUDA_TRY( cudaMemcpyAsync( p, pairs, m * 8, cudaMemcpyHostToDevice, s ) );
		d_pairs = p;
	}
	k_toi_times<<<(uint32_t)((m + 127) / 128), 128, 0, s>>>( d_pairs, m, a->d_verts, f.a1, b->d_verts, f.b1, eta, R2, max_iters, d_times );
	LAUNCHED();
	if (space == TBVH_HOST) CUDA_TRY( cudaMemcpyAsync( times, d_times, m * 4, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	return TBVH_OK;
}

} // extern "C"
