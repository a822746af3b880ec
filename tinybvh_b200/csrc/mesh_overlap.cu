// tinybvh_b200/csrc/mesh_overlap.cu - intersecting triangle pairs between two meshes and within one mesh (tbvh_mesh_overlap_pairs /
// tbvh_mesh_overlap_bits): one walk of B's BVH2 per triangle of A with the closed box test, and a pair test of orientation predicates
// only.  DESIGN.md 4.12 states the rules; tests/tritri_oracle.c restates them on the host in the same fp32 operation order.
//
// Pairs, on one stream: k_mesh_overlap<COUNT> (pairs per triangle of A), an exclusive scan, one host synchronisation for the raw total,
// k_mesh_overlap<FILL> ((i << 32) | j keys at the scanned offsets), a radix sort, DeviceSelect::Unique, and k_overlap_out, which writes
// the first min( unique, capacity ) pairs.  Bits: k_mesh_overlap<BITS>, one launch.
#include "tri_pair.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <algorithm>

namespace
{
enum { MO_COUNT = 0, MO_FILL = 1, MO_BITS = 2 };
} // namespace

// One thread per triangle i of A in 128-thread CTAs: the box of its corners against B's child-pair nodes (the root's box untested), and
// every reference of every reached leaf through the pair test; SELF: B is A and the pairs passes keep j > i, the bits pass j != i.
// COUNT: counts[i] = the pairs found (a reference reached on several paths counts once per path); FILL: their keys (i << 32) | j from
// offsets[i] on, in the same order; BITS: one bit per triangle (store_occlusion_word), the walk ends at the first pair.  STACKN as
// k_closest_point.
template <int MODE, bool SELF, int STACKN>
__global__ void __launch_bounds__( 128 ) k_mesh_overlap( const float4* __restrict__ nodes, const float4* __restrict__ tris, const float4* __restrict__ vb,
	const float4* __restrict__ va, const uint64_t n, const uint32_t root_ref, const uint32_t root_count, uint64_t* __restrict__ counts,
	const uint64_t* __restrict__ offsets, uint64_t* __restrict__ keys, uint32_t* __restrict__ bits )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	bool hit = false;
	if (i < n)
	{
		V3 t[3];
		#pragma unroll
		for (int c = 0; c < 3; c++) t[c] = mo_corner( va, i * 3 + c );
		const V3 mn{ fminf( fminf( t[0].x, t[1].x ), t[2].x ), fminf( fminf( t[0].y, t[1].y ), t[2].y ), fminf( fminf( t[0].z, t[1].z ), t[2].z ) };
		const V3 mx{ fmaxf( fmaxf( t[0].x, t[1].x ), t[2].x ), fmaxf( fmaxf( t[0].y, t[1].y ), t[2].y ), fmaxf( fmaxf( t[0].z, t[1].z ), t[2].z ) };
		uint2 stack[STACKN];
		int sp = 0;
		uint32_t ref = root_ref, cnt = root_count;
		uint64_t found = 0, o = MODE == MO_FILL ? offsets[i] : 0;
		while (true)
		{
			if (cnt == 0)
			{
				const float4* q = nodes + (size_t)ref * 2;
				const float4 a0 = __ldg( q ), a1 = __ldg( q + 1 ), b0 = __ldg( q + 2 ), b1 = __ldg( q + 3 );
				const bool ha = mo_box( mn, mx, a0, a1 ), hb = mo_box( mn, mx, b0, b1 );
				const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w ), refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
				if (ha && hb) { stack[sp++] = make_uint2( refb, cntb ); ref = refa, cnt = cnta; continue; }
				if (ha) { ref = refa, cnt = cnta; continue; }
				if (hb) { ref = refb, cnt = cntb; continue; }
			}
			else
			{
				for (uint32_t k = 0; k < cnt && !hit; k++)
				{
					const uint32_t j = __float_as_uint( __ldg( &tris[(size_t)(ref + k) * 3].w ) );
					if (SELF && (MODE == MO_BITS ? j == i : j <= i)) continue;
					const V3 u[3] = { mo_corner( vb, (size_t)j * 3 ), mo_corner( vb, (size_t)j * 3 + 1 ), mo_corner( vb, (size_t)j * 3 + 2 ) };
					if (!mo_test<SELF>( t, u )) continue;
					if (MODE == MO_BITS) hit = true;
					else if (MODE == MO_FILL) keys[o++] = (i << 32) | j;
					else found++;
				}
				if (hit) break;
			}
			if (sp == 0) break;
			const uint2 e = stack[--sp];
			ref = e.x, cnt = e.y;
		}
		if (MODE == MO_COUNT) counts[i] = found;
	}
	if (MODE == MO_BITS) store_occlusion_word( bits, i, n, hit );
}

// keys (i << 32) | j -> pairs [i, j] for the first min( *num, cap ) keys
__global__ void k_overlap_out( const uint64_t* __restrict__ keys, const int64_t* __restrict__ num, const uint64_t cap, uint32_t* __restrict__ pairs )
{
	const uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= cap || k >= (uint64_t)*num) return;
	const uint64_t x = keys[k];
	pairs[k * 2] = (uint32_t)(x >> 32), pairs[k * 2 + 1] = (uint32_t)x;
}

static int mo_launch( int mode, tbvh_bvh a, tbvh_bvh b, uint64_t* counts, const uint64_t* offsets, uint64_t* keys, uint32_t* bits, cudaStream_t s )
{
	const uint64_t n = a->info.prim_count;
	const uint32_t grid = (uint32_t)((n + 127) / 128);
	const bool self = a == b, deep = b->info.max_depth + 1 > TBVH_STACK;
	#define MO_ARGS <<<grid, 128, 0, s>>>( b->trav(), b->d_leaf_tris, b->d_verts, a->d_verts, n, b->root_ref, b->root_count, counts, offsets, keys, bits )
	#define MO_MODE( M, D ) do { if (self) k_mesh_overlap<M, true, D> MO_ARGS; else k_mesh_overlap<M, false, D> MO_ARGS; } while (0)
	#define MO_DEPTH( D ) do { if (mode == MO_COUNT) MO_MODE( MO_COUNT, D ); else if (mode == MO_FILL) MO_MODE( MO_FILL, D ); else MO_MODE( MO_BITS, D ); } while (0)
	if (deep) MO_DEPTH( TBVH_STACK_DEEP ); else MO_DEPTH( TBVH_STACK );
	#undef MO_DEPTH
	#undef MO_MODE
	#undef MO_ARGS
	LAUNCHED();
	return TBVH_OK;
}

int mo_check( const char* fn, tbvh_bvh a, tbvh_bvh b, const void* out, bool out_needed, uint64_t* count, bool need_count, int space, uintptr_t align )
{
	if (!a || !b || (out_needed && !out) || (need_count && !count)) { tbvh_set_error( "%s: NULL argument", fn ); return TBVH_E_ARG; }
	if (space != TBVH_HOST && space != TBVH_DEVICE) { tbvh_set_error( "%s: unknown space %d", fn, space ); return TBVH_E_ARG; }
	if (space == TBVH_DEVICE && ((uintptr_t)out & (align - 1))) { tbvh_set_error( "%s: the device output must be %u-byte aligned", fn, (unsigned)align ); return TBVH_E_ARG; }
	if (a->ctx != b->ctx) { tbvh_set_error( "%s: the two handles belong to different contexts", fn ); return TBVH_E_ARG; }
	if (a->d_inst || b->d_inst) { tbvh_set_error( "%s: queries on a TLAS are not supported", fn ); return TBVH_E_UNSUPPORTED; }
	for (tbvh_bvh h : { a, b })
		if (!h->trav() || !h->d_leaf_tris || !h->d_verts) { tbvh_set_error( "%s: no BVH-layout tree on a handle", fn ); return TBVH_E_STATE; }
	if (b->info.max_depth + 1 > TBVH_STACK_DEEP) { tbvh_set_error( "%s: BVH depth %u exceeds the %d-entry traversal stack", fn, b->info.max_depth, TBVH_STACK_DEEP ); return TBVH_E_LIMIT; }
	return TBVH_OK;
}

int mesh_pairs_run( const char* fn, tbvh_bvh a, uint32_t* pairs, uint64_t capacity, uint64_t* count, int space, void* stream, const PairsLaunch& launch )
{
	CUDA_TRY( cudaSetDevice( a->ctx->device ) );
	const uint64_t n = a->info.prim_count;
	if (n == 0) { *count = 0; return TBVH_OK; }
	// the pipeline runs on the engine stream (CUB's launches are counted by capture, which the legacy default stream does not allow),
	// behind everything queued on the caller's stream so far
	Scratch sc( a->ctx->stream );
	const cudaStream_t s = sc.s;
	if (space == TBVH_DEVICE)
	{
		TRY( sc.events() );
		CUDA_TRY( cudaEventRecord( sc.e0, (cudaStream_t)stream ) );
		CUDA_TRY( cudaStreamWaitEvent( s, sc.e0, 0 ) );
	}
	uint64_t* cnt = 0, * off = 0, * h = 0;
	TRY( sc.alloc( cnt, (n + 1) * 8 ) );
	TRY( sc.alloc( off, (n + 1) * 8 ) );
	TRY( sc.alloc_host( h, 16 ) );
	size_t tb = 0;
	CUDA_TRY( cub::DeviceScan::ExclusiveSum( (void*)0, tb, cnt, off, (int64_t)(n + 1), s ) );
	void* temp = 0;
	TRY( sc.alloc( temp, std::max( tb, (size_t)16 ) ) );
	CUDA_TRY( cudaMemsetAsync( cnt + n, 0, 8, s ) );
	TRY( launch( false, cnt, 0, 0, s ) );
	TRY( sort_enqueue( s, [&]() { return cub::DeviceScan::ExclusiveSum( temp, tb, cnt, off, (int64_t)(n + 1), s ); } ) );
	CUDA_TRY( cudaMemcpyAsync( h, off + n, 8, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	const uint64_t raw = h[0];
	if (raw > MO_MAX_KEYS)
	{
		*count = raw;
		tbvh_set_error( "%s: %llu raw pairs exceed the %llu a call sorts", fn, (unsigned long long)raw, MO_MAX_KEYS );
		return TBVH_E_LIMIT;
	}
	if (raw == 0) { *count = 0; return TBVH_OK; }
	uint64_t* keys[2] = {};
	int64_t* num = 0;
	uint32_t* out = pairs;
	const uint64_t m = std::min( raw, capacity );
	TRY( sc.alloc( keys[0], raw * 8 ) );
	TRY( sc.alloc( keys[1], raw * 8 ) );
	TRY( sc.alloc( num, 8 ) );
	if (space == TBVH_HOST && m) TRY( sc.alloc( out, m * 8 ) );
	// the sort needs the bits of i and all 32 of j
	int end_bit = 32;
	while (end_bit < 64 && (n - 1) >> (end_bit - 32)) end_bit++;
	size_t tb2 = 0, tb3 = 0;
	CUDA_TRY( cub::DeviceRadixSort::SortKeys( (void*)0, tb2, keys[0], keys[1], (int64_t)raw, 0, end_bit, s ) );
	CUDA_TRY( cub::DeviceSelect::Unique( (void*)0, tb3, keys[1], keys[0], num, (int64_t)raw, s ) );
	void* temp2 = 0;
	TRY( sc.alloc( temp2, std::max( tb2, tb3 ) ) );
	tb2 = tb3 = std::max( tb2, tb3 );
	TRY( launch( true, 0, off, keys[0], s ) );
	TRY( sort_enqueue( s, [&]() { return cub::DeviceRadixSort::SortKeys( temp2, tb2, keys[0], keys[1], (int64_t)raw, 0, end_bit, s ); } ) );
	TRY( sort_enqueue( s, [&]() { return cub::DeviceSelect::Unique( temp2, tb3, keys[1], keys[0], num, (int64_t)raw, s ); } ) );
	if (m)
	{
		k_overlap_out<<<(uint32_t)((m + 255) / 256), 256, 0, s>>>( keys[0], num, m, out );
		LAUNCHED();
	}
	CUDA_TRY( cudaMemcpyAsync( h + 1, num, 8, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	const uint64_t unique = h[1], w = std::min( unique, capacity );
	if (space == TBVH_HOST && w)
	{
		CUDA_TRY( cudaMemcpyAsync( pairs, out, w * 8, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
	}
	*count = unique;
	return TBVH_OK;
}

extern "C" {

int tbvh_mesh_overlap_pairs( tbvh_bvh a, tbvh_bvh b, uint32_t* pairs, uint64_t capacity, uint64_t* count, int space, void* stream )
{
	TRY( mo_check( __func__, a, b, pairs, capacity > 0, count, true, space, 8 ) );
	return mesh_pairs_run( __func__, a, pairs, capacity, count, space, stream,
		[&]( bool fill, uint64_t* counts, const uint64_t* offsets, uint64_t* keys, cudaStream_t s ) { return mo_launch( fill ? MO_FILL : MO_COUNT, a, b, counts, offsets, keys, 0, s ); } );
}

int tbvh_mesh_overlap_bits( tbvh_bvh a, tbvh_bvh b, uint32_t* bits, int space, void* stream )
{
	TRY( mo_check( __func__, a, b, bits, true, 0, false, space, 4 ) );
	CUDA_TRY( cudaSetDevice( a->ctx->device ) );
	const uint64_t n = a->info.prim_count;
	if (n == 0) return TBVH_OK;
	if (space == TBVH_DEVICE) return mo_launch( MO_BITS, a, b, 0, 0, 0, bits, (cudaStream_t)stream );
	const size_t bytes = ((n + 31) / 32) * 4;
	Scratch sc( a->ctx->stream );
	uint32_t* d_bits = 0;
	TRY( sc.alloc( d_bits, bytes ) );
	TRY( mo_launch( MO_BITS, a, b, 0, 0, 0, d_bits, sc.s ) );
	CUDA_TRY( cudaMemcpyAsync( bits, d_bits, bytes, cudaMemcpyDeviceToHost, sc.s ) );
	CUDA_TRY( cudaStreamSynchronize( sc.s ) );
	return TBVH_OK;
}

} // extern "C"
