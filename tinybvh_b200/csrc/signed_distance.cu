// tinybvh_b200/csrc/signed_distance.cu - signed distances to closed meshes (tbvh_signed_distance_prepare / tbvh_signed_distance): the
// closest-point walk of include/tinybvh_b200_device/closest_walk.cuh, then the sign of ( p - c ) . N, N the angle-weighted pseudonormal
// (Baerentzen & Aanaes 2005) of the feature the closest point c lies on.  DESIGN.md 4.10 states the rules; tests/sdf_oracle.c restates
// them on the host in the same fp32 operation order.
//
// Prepare, on the engine stream, over the handle's d_verts (three float4 corners per primitive, prim order):
//   k_sd_faces      unit face normals into the table, corner angles into scratch
//   welding         three stable CUB radix sorts of the corner keys (z, then y, then x) give the corners in lexicographic position
//                   order, prim order inside each run of equal positions; k_sd_heads + exclusive_scan + k_sd_starts find the runs,
//                   k_sd_vertex_sums sums each run's theta * n in order (one thread per run) and names each welded vertex by its
//                   first corner
//   edges           k_sd_edge_keys: (min, max) of the welded vertices of every triangle edge; one stable 64-bit sort; the same run
//                   kernels sum each run's face normals in order
// The table holds SD_REC float4 per primitive: the face normal, the pseudonormals of vertices 0, 1, 2 and of edges AB, AC, BC, so a
// query's feature (tbvh::CpFeature) indexes its record directly.
#include "common.cuh"
#include "../../include/tinybvh_b200_device/closest_walk.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>

#define SD_REC 7 // float4 per primitive in the table

namespace
{
using tbvh::cp_dot;
using tbvh::cp_cross;

constexpr float SD_FLT_MAX = 3.402823466e38f;

// acos by Abramowitz & Stegun 4.4.46 (|error| <= 2e-8 on [0, 1]): sqrt( 1 - |x| ) times a degree-7 polynomial by Horner, pi - acos( -x )
// below 0.  A fixed formula, so that the host restatement gives the same bits (acosf differs between libm and the device).
__device__ __forceinline__ float sd_acos( const float x )
{
	const float a = x < 0.0f ? -x : x;
	float p = -0.0012624911f;
	p = __fmaf_rn( p, a, 0.0066700901f );
	p = __fmaf_rn( p, a, -0.0170881256f );
	p = __fmaf_rn( p, a, 0.0308918810f );
	p = __fmaf_rn( p, a, -0.0501743046f );
	p = __fmaf_rn( p, a, 0.0889789874f );
	p = __fmaf_rn( p, a, -0.2145988016f );
	p = __fmaf_rn( p, a, 1.5707963050f );
	const float r = __fmul_rn( __fsqrt_rn( __fsub_rn( 1.0f, a ) ), p );
	return x < 0.0f ? __fsub_rn( 3.14159265f, r ) : r;
}

// the angle between the corner edges a and b: 0 when either is zero-length (or not finite), else acos of the clamped cosine
__device__ __forceinline__ float sd_angle( const float ax, const float ay, const float az, const float bx, const float by, const float bz )
{
	const float la = cp_dot( ax, ay, az, ax, ay, az ), lb = cp_dot( bx, by, bz, bx, by, bz );
	if (!(la > 0.0f && la <= SD_FLT_MAX && lb > 0.0f && lb <= SD_FLT_MAX)) return 0.0f;
	float c = __fdiv_rn( cp_dot( ax, ay, az, bx, by, bz ), __fmul_rn( __fsqrt_rn( la ), __fsqrt_rn( lb ) ) );
	c = c > -1.0f ? c : -1.0f; // NaN gives -1
	c = c < 1.0f ? c : 1.0f;
	return sd_acos( c );
}

// the corner key of one coordinate: an order-preserving uint of the value with -0 read as +0; NaN gives the largest key (a NaN corner
// is a run of its own all the same: runs compare values, and NaN equals nothing)
__device__ __forceinline__ uint32_t sd_key( const float f )
{
	if (f != f) return 0xffffffffu;
	const uint32_t u = f == 0.0f ? 0u : __float_as_uint( f );
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float4 f4sub( const float4& a, const float4& b ) { return make_float4( __fsub_rn( a.x, b.x ), __fsub_rn( a.y, b.y ), __fsub_rn( a.z, b.z ), 0.0f ); }

// face normal n = e1 x e2 normalised (0 where |n|^2 is not finite and > 0) into the table; the three corner angles into theta
__global__ void k_sd_faces( const float4* __restrict__ verts, const uint32_t prims, float4* __restrict__ table, float* __restrict__ theta )
{
	const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= prims) return;
	const float4 v0 = __ldg( verts + (size_t)p * 3 ), v1 = __ldg( verts + (size_t)p * 3 + 1 ), v2 = __ldg( verts + (size_t)p * 3 + 2 );
	const float4 e1 = f4sub( v1, v0 ), e2 = f4sub( v2, v0 ), e3 = f4sub( v2, v1 ), f1 = f4sub( v0, v1 ), g0 = f4sub( v0, v2 ), g1 = f4sub( v1, v2 );
	// |n|^2 is of degree 4 in lengths: e1 and e2 are scaled by the power of two of their largest component first, which leaves n's
	// direction exact and keeps |n|^2 from over- or underflowing (from about 2^32 and below 2^-31 it would, and the normal would be 0)
	float inv;
	const float sc = tbvh::cp_pow2( fmaxf( fmaxf( fmaxf( fabsf( e1.x ), fabsf( e1.y ) ), fmaxf( fabsf( e1.z ), fabsf( e2.x ) ) ), fmaxf( fabsf( e2.y ), fabsf( e2.z ) ) ), inv );
	float nx, ny, nz;
	cp_cross( __fmul_rn( e1.x, sc ), __fmul_rn( e1.y, sc ), __fmul_rn( e1.z, sc ), __fmul_rn( e2.x, sc ), __fmul_rn( e2.y, sc ), __fmul_rn( e2.z, sc ), nx, ny, nz );
	const float nn = cp_dot( nx, ny, nz, nx, ny, nz );
	float4 n = make_float4( 0.0f, 0.0f, 0.0f, 0.0f );
	if (nn > 0.0f && nn <= SD_FLT_MAX)
	{
		const float l = __fsqrt_rn( nn );
		n = make_float4( __fdiv_rn( nx, l ), __fdiv_rn( ny, l ), __fdiv_rn( nz, l ), 0.0f );
	}
	table[(size_t)p * SD_REC] = n;
	theta[(size_t)p * 3] = sd_angle( e1.x, e1.y, e1.z, e2.x, e2.y, e2.z );
	theta[(size_t)p * 3 + 1] = sd_angle( e3.x, e3.y, e3.z, f1.x, f1.y, f1.z );
	theta[(size_t)p * 3 + 2] = sd_angle( g0.x, g0.y, g0.z, g1.x, g1.y, g1.z );
}

// keys[i] = the corner key of coordinate `axis` of corner order[i] (order NULL: corner i, and vals[i] = i)
__global__ void k_sd_corner_keys( const float4* __restrict__ verts, const uint32_t* __restrict__ order, const int axis, const uint32_t m,
	uint32_t* __restrict__ keys, uint32_t* __restrict__ vals )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= m) return;
	const uint32_t c = order ? order[i] : i;
	const float4 v = __ldg( verts + c );
	keys[i] = sd_key( axis == 0 ? v.x : axis == 1 ? v.y : v.z );
	if (!order) vals[i] = i;
}

// head[i] = sorted entry i starts a run: corners at unequal positions (welding, ekeys NULL) or unequal edge keys
__global__ void k_sd_heads( const float4* __restrict__ verts, const uint32_t* __restrict__ order, const uint64_t* __restrict__ ekeys, const uint32_t m,
	uint32_t* __restrict__ head )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= m) return;
	bool h = i == 0;
	if (!h && ekeys) h = ekeys[i] != ekeys[i - 1];
	else if (!h)
	{
		const float4 a = __ldg( verts + order[i] ), b = __ldg( verts + order[i - 1] );
		h = !(a.x == b.x && a.y == b.y && a.z == b.z);
	}
	head[i] = h ? 1u : 0u;
}

// start[r] = the first sorted entry of run r, start[runs] = m (run = the exclusive scan of the heads, run[m] = runs)
__global__ void k_sd_starts( const uint32_t* __restrict__ head, const uint32_t* __restrict__ run, const uint32_t m, uint32_t* __restrict__ start )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= m) return;
	if (head[i]) start[run[i]] = i;
	if (i == m - 1) start[run[m]] = m;
}

// one thread per welded vertex: the sum of theta * n over its corners in ascending corner order into slot 1 + corner of each corner's
// record; vid[c] = the vertex's first corner
__global__ void k_sd_vertex_sums( const uint32_t* __restrict__ order, const uint32_t* __restrict__ start, const uint32_t* __restrict__ runs,
	const float* __restrict__ theta, float4* __restrict__ table, uint32_t* __restrict__ vid )
{
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= *runs) return;
	const uint32_t a = start[r], b = start[r + 1];
	float sx = 0.0f, sy = 0.0f, sz = 0.0f;
	for (uint32_t i = a; i < b; i++)
	{
		const uint32_t c = order[i];
		const float t = theta[c];
		const float4 n = table[(size_t)(c / 3) * SD_REC];
		sx = __fmaf_rn( t, n.x, sx ), sy = __fmaf_rn( t, n.y, sy ), sz = __fmaf_rn( t, n.z, sz );
	}
	const uint32_t first = order[a];
	for (uint32_t i = a; i < b; i++)
	{
		const uint32_t c = order[i];
		table[(size_t)(c / 3) * SD_REC + 1 + c % 3] = make_float4( sx, sy, sz, 0.0f );
		vid[c] = first;
	}
}

// half-edge h = 3 prim + e (e: 0 = AB, 1 = AC, 2 = BC): the key (min, max) of its two welded vertices, and h
__global__ void k_sd_edge_keys( const uint32_t* __restrict__ vid, const uint32_t m, uint64_t* __restrict__ keys, uint32_t* __restrict__ vals )
{
	const uint32_t h = blockIdx.x * blockDim.x + threadIdx.x;
	if (h >= m) return;
	const uint32_t p = h / 3, e = h % 3;
	const uint32_t a = vid[p * 3 + (e == 2 ? 1 : 0)], b = vid[p * 3 + (e == 0 ? 1 : 2)];
	keys[h] = ((uint64_t)min( a, b ) << 32) | max( a, b );
	vals[h] = h;
}

// one thread per welded edge: the sum of the face normals of its half-edges in ascending order into slot 4 + e of each one's record
__global__ void k_sd_edge_sums( const uint32_t* __restrict__ order, const uint32_t* __restrict__ start, const uint32_t* __restrict__ runs,
	float4* __restrict__ table )
{
	const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= *runs) return;
	const uint32_t a = start[r], b = start[r + 1];
	float sx = 0.0f, sy = 0.0f, sz = 0.0f;
	for (uint32_t i = a; i < b; i++)
	{
		const float4 n = table[(size_t)(order[i] / 3) * SD_REC];
		sx = __fadd_rn( sx, n.x ), sy = __fadd_rn( sy, n.y ), sz = __fadd_rn( sz, n.z );
	}
	for (uint32_t i = a; i < b; i++)
	{
		const uint32_t h = order[i];
		table[(size_t)(h / 3) * SD_REC + 4 + h % 3] = make_float4( sx, sy, sz, 0.0f );
	}
}
} // namespace

// One query per thread in 128-thread CTAs, STACKN as k_closest_point: the closest-point walk, then the winner's triangle rebuilt from
// d_verts as leaf_tri_record builds it, its feature from cp_triangle_feature, and one gather of the feature's pseudonormal.
template <int STACKN>
__global__ void __launch_bounds__( 128 ) k_signed_distance( const float4* __restrict__ nodes, const float4* __restrict__ tris, const float4* __restrict__ verts,
	const float4* __restrict__ table, const float4* __restrict__ queries, float4* __restrict__ results, const uint64_t n, const uint32_t root_ref, const uint32_t root_count )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float4 q = __ldg( queries + i );
	const float4 miss = make_float4( q.w, 0.0f, 0.0f, __uint_as_float( tbvh::CP_NO_PRIM ) );
	if (!tbvh::cp_query_ok( q )) { results[i] = miss; return; }
	float best = __fmul_rn( q.w, q.w ), bu = 0.0f, bv = 0.0f;
	uint32_t bprim = tbvh::CP_NO_PRIM;
	tbvh::CpEntry stack[STACKN];
	tbvh::cp_walk<false>( nodes, tris, root_ref, root_count, q.x, q.y, q.z, best, bprim, bu, bv, stack );
	if (bprim == tbvh::CP_NO_PRIM) { results[i] = miss; return; }
	const float4 v0 = __ldg( verts + (size_t)bprim * 3 ), v1 = __ldg( verts + (size_t)bprim * 3 + 1 ), v2 = __ldg( verts + (size_t)bprim * 3 + 2 );
	const float4 e1 = f4sub( v1, v0 ), e2 = f4sub( v2, v0 );
	float u, v;
	uint32_t f;
	tbvh::cp_triangle_feature( q.x, q.y, q.z, v0, e1, e2, u, v, f ); // (u, v) = (bu, bv): the same function on the same record
	const float apx = __fsub_rn( q.x, v0.x ), apy = __fsub_rn( q.y, v0.y ), apz = __fsub_rn( q.z, v0.z );
	const float dx = __fsub_rn( apx, __fmaf_rn( bv, e2.x, __fmul_rn( bu, e1.x ) ) );
	const float dy = __fsub_rn( apy, __fmaf_rn( bv, e2.y, __fmul_rn( bu, e1.y ) ) );
	const float dz = __fsub_rn( apz, __fmaf_rn( bv, e2.z, __fmul_rn( bu, e1.z ) ) );
	const float4 N = __ldg( table + (size_t)bprim * SD_REC + f );
	const float s = cp_dot( dx, dy, dz, N.x, N.y, N.z ), d = __fsqrt_rn( best );
	results[i] = make_float4( s < 0.0f ? -d : d, bu, bv, __uint_as_float( bprim ) );
}

int sd_table_check( tbvh_bvh b )
{
	if (!b->d_sdf) { tbvh_set_error( "no signed-distance table: call tbvh_signed_distance_prepare first" ); return TBVH_E_STATE; }
	if (b->sdf_generation != b->generation || b->sdf_revision != b->revision)
	{
		tbvh_set_error( "the signed-distance table is stale: the tree or its vertices changed since tbvh_signed_distance_prepare" );
		return TBVH_E_STATE;
	}
	return TBVH_OK;
}

int sd_launch( tbvh_bvh b, const float4* d_queries, float4* d_results, uint64_t n, cudaStream_t s )
{
	const uint32_t grid = (uint32_t)((n + 127) / 128);
	if (b->info.max_depth + 1 > TBVH_STACK)
		k_signed_distance<TBVH_STACK_DEEP><<<grid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, b->d_verts, b->d_sdf, d_queries, d_results, n, b->root_ref, b->root_count );
	else k_signed_distance<TBVH_STACK><<<grid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, b->d_verts, b->d_sdf, d_queries, d_results, n, b->root_ref, b->root_count );
	LAUNCHED();
	return TBVH_OK;
}

// the runs of m sorted entries (corners at equal positions, or equal edge keys): head flags, their scan and each run's start
static int sd_runs( const float4* verts, const uint32_t* order, const uint64_t* ekeys, const uint32_t m, uint32_t* head, uint32_t* run, uint32_t* tile,
	uint32_t* start, cudaStream_t s )
{
	const uint32_t g = (m + 255) / 256;
	k_sd_heads<<<g, 256, 0, s>>>( verts, order, ekeys, m, head ); LAUNCHED();
	TRY( exclusive_scan( head, run, tile, m, s ) );
	k_sd_starts<<<g, 256, 0, s>>>( head, run, m, start ); LAUNCHED();
	return TBVH_OK;
}

// the table of b's triangles into `table` (allocated here), on s
static int sd_prepare( tbvh_bvh b, DevArray<float4>& table, cudaStream_t s )
{
	const uint32_t prims = b->info.prim_count, m = prims * 3, g = (m + 255) / 256;
	const float4* verts = b->d_verts;
	TRY( table.alloc( (size_t)prims * SD_REC * 16 ) );
	Scratch sc( s );
	float* theta = 0;
	uint32_t* key[2] = {}, * val[2] = {}, * head = 0, * run = 0, * start = 0, * tile = 0, * vid = 0;
	uint64_t* ekey[2] = {};
	TRY( sc.alloc( theta, (size_t)m * 4 ) );
	for (int k = 0; k < 2; k++) { TRY( sc.alloc( key[k], (size_t)m * 4 ) ); TRY( sc.alloc( val[k], (size_t)m * 4 ) ); TRY( sc.alloc( ekey[k], (size_t)m * 8 ) ); }
	TRY( sc.alloc( head, (size_t)m * 4 ) ); TRY( sc.alloc( run, ((size_t)m + 1) * 4 ) ); TRY( sc.alloc( start, ((size_t)m + 1) * 4 ) );
	TRY( sc.alloc( tile, ((size_t)m / 2048 + 2) * 4 ) ); TRY( sc.alloc( vid, (size_t)m * 4 ) );
	size_t tb = 0, tb2 = 0;
	CUDA_TRY( cub::DeviceRadixSort::SortPairs( (void*)0, tb, key[0], key[1], val[0], val[1], (int64_t)m, 0, 32, s ) );
	CUDA_TRY( cub::DeviceRadixSort::SortPairs( (void*)0, tb2, ekey[0], ekey[1], val[0], val[1], (int64_t)m, 0, 64, s ) );
	tb = std::max( tb, tb2 );
	void* temp = 0;
	TRY( sc.alloc( temp, tb ) );
	k_sd_faces<<<(prims + 255) / 256, 256, 0, s>>>( verts, prims, table, theta ); LAUNCHED();
	// welding: stable sorts by z, y, x leave the corners in lexicographic (x, y, z) order, ascending corner number inside a position
	const int axes[3] = { 2, 1, 0 };
	int cur = 0; // val[cur] holds the order so far
	for (int k = 0; k < 3; k++)
	{
		k_sd_corner_keys<<<g, 256, 0, s>>>( verts, k ? val[cur] : 0, axes[k], m, key[0], val[cur] ); LAUNCHED();
		TRY( sort_enqueue( s, [&]() { return cub::DeviceRadixSort::SortPairs( temp, tb, key[0], key[1], val[cur], val[cur ^ 1], (int64_t)m, 0, 32, s ); } ) );
		cur ^= 1;
	}
	TRY( sd_runs( verts, val[cur], 0, m, head, run, tile, start, s ) );
	k_sd_vertex_sums<<<g, 256, 0, s>>>( val[cur], start, run + m, theta, table, vid ); LAUNCHED();
	// edges: one stable sort of the (min, max) keys of the half-edges, ascending half-edge number inside an edge
	k_sd_edge_keys<<<g, 256, 0, s>>>( vid, m, ekey[0], val[0] ); LAUNCHED();
	TRY( sort_enqueue( s, [&]() { return cub::DeviceRadixSort::SortPairs( temp, tb, ekey[0], ekey[1], val[0], val[1], (int64_t)m, 0, 64, s ); } ) );
	TRY( sd_runs( verts, val[1], ekey[1], m, head, run, tile, start, s ) );
	k_sd_edge_sums<<<g, 256, 0, s>>>( val[1], start, run + m, table ); LAUNCHED();
	CUDA_TRY( cudaStreamSynchronize( s ) );
	return TBVH_OK;
}

extern "C" {

int tbvh_signed_distance_prepare( tbvh_bvh b )
{
	if (!b) { tbvh_set_error( "%s: NULL handle", __func__ ); return TBVH_E_ARG; }
	if (b->d_inst) { tbvh_set_error( "signed distances over a TLAS are not supported" ); return TBVH_E_UNSUPPORTED; }
	if (!b->trav() || !b->d_leaf_tris || !b->d_verts || b->info.prim_count == 0) { tbvh_set_error( "%s: no BVH-layout tree on this handle", __func__ ); return TBVH_E_STATE; }
	if (b->info.prim_count > (1u << 30)) { tbvh_set_error( "%s: %u triangles exceed the 2^30 that 32-bit corner numbers allow", __func__, b->info.prim_count ); return TBVH_E_LIMIT; }
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	b->d_sdf.reset();
	DevArray<float4> table;
	const int rc = sd_prepare( b, table, b->ctx->stream );
	if (rc != TBVH_OK) return rc;
	b->d_sdf = std::move( table );
	b->sdf_generation = b->generation, b->sdf_revision = b->revision;
	return TBVH_OK;
}

int tbvh_signed_distance( tbvh_bvh b, const void* queries, void* results, uint64_t n, int space, void* stream )
{
	return proximity_query( __func__, b, queries, results, n, space, stream, PROX_SIGNED );
}

} // extern "C"
