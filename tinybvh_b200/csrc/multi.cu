// tinybvh_b200/csrc/multi.cu - one process, several GPUs: replicate a BVH, shard a ray batch by index (SURVEY.md 8(e)).
//
// A tbvh_group owns one engine context per device.  `tbvh_group_replicate` copies the traversal arrays of a built BVH to every
// device of the group (peer-to-peer over NVLink when the devices can reach each other - the one-process form of the "one broadcast
// of the built BVH"; multi-process jobs do the same exchange with NCCL, tinybvh_b200/multi.py).  `tbvh_group_intersect` /
// `_occluded` cut a HOST ray batch into contiguous, 32-ray-aligned index ranges, one per device (tbvh_shard_range), and run
// the host-buffer pipeline of each device from its own worker thread, bound to the CPUs of that device's NUMA node.  There is
// no traffic between devices during traversal and nothing to reduce: the ranges are disjoint, occlusion words never straddle two
// ranges.  `tbvh_group_host_alloc` places every range of a ray buffer on the NUMA node of the device that will read it.
#include "common.cuh"
#include <sched.h>
#include <sys/mman.h>
#include <string.h>
#include <thread>
#include <string>
#include <vector>
#include <new>

struct tbvh_group_t
{
	std::vector<tbvh_ctx> ctx;        // one per device
	std::vector<tbvh_bvh> replica;    // replica[g] lives on ctx[g]
	std::vector<char> owned;          // 0 where replica[g] IS the caller's source handle (its context belongs to the group)
	std::vector<std::pair<void*, size_t>> host_blocks; // tbvh_group_host_alloc results (mmap + cudaHostRegister)
};

static void release_replicas( tbvh_group g )
{
	for (size_t i = 0; i < g->replica.size(); i++) if (g->replica[i] && g->owned[i]) tbvh_bvh_destroy( g->replica[i] );
	g->replica.clear(), g->owned.clear();
}

// device-to-device copy of `bytes` from (src_dev) to a fresh allocation on (dst_dev)
static int peer_clone( void** dst, int dst_dev, const void* src, int src_dev, size_t bytes, cudaStream_t s )
{
	*dst = 0;
	if (!src || bytes == 0) return TBVH_OK;
	CUDA_TRY( cudaMalloc( dst, bytes ) );
	CUDA_TRY( cudaMemcpyPeerAsync( *dst, dst_dev, src, src_dev, bytes, s ) );
	return TBVH_OK;
}

// run fn( part ) on one worker thread per device, each bound to the CPUs of its device's NUMA node; first error wins
template <class F> static int per_device( tbvh_group g, F fn )
{
	const size_t parts = g->ctx.size();
	std::vector<int> rc( parts, TBVH_OK );
	std::vector<std::string> msg( parts );
	std::vector<std::thread> th;
	for (size_t p = 0; p < parts; p++) th.emplace_back( [&, p]()
	{
		tbvh_bind_thread_to_device( g->ctx[p]->device ); // best effort
		rc[p] = fn( (uint32_t)p );
		if (rc[p] != TBVH_OK) msg[p] = tbvh_last_error(); // the error text is thread-local
	} );
	for (auto& t : th) t.join();
	for (size_t p = 0; p < parts; p++) if (rc[p] != TBVH_OK) { tbvh_set_error( "device %d: %s", g->ctx[p]->device, msg[p].c_str() ); return rc[p]; }
	return TBVH_OK;
}

extern "C" {

void tbvh_shard_range( uint64_t n, uint32_t part, uint32_t parts, uint64_t* first, uint64_t* count )
{
	// contiguous index ranges with 32-ray-aligned boundaries: occlusion words never straddle two devices (tinybvh_b200/multi.py shard_range)
	const uint64_t units = (n + 31) / 32;
	const uint64_t lo = units * part / parts, hi = units * (part + 1) / parts;
	const uint64_t a = lo * 32 < n ? lo * 32 : n, e = hi * 32 < n ? hi * 32 : n;
	if (first) *first = a;
	if (count) *count = e - a;
}

int tbvh_group_create( const int* devices, int count, tbvh_group* out )
{
	ARG_CHECK( out, "out == NULL" );
	int have = 0;
	CUDA_TRY( cudaGetDeviceCount( &have ) );
	if (count <= 0) count = have, devices = 0; // all devices
	ARG_CHECK( count >= 1 && count <= 64, "device count out of range" );
	for (int i = 0; i < count; i++) ARG_CHECK( (devices ? devices[i] : i) >= 0 && (devices ? devices[i] : i) < have, "no such device" ); // a device may appear twice (two contexts on it)
	tbvh_group g = new (std::nothrow) tbvh_group_t();
	ARG_CHECK( g, "out of host memory" );
	for (int i = 0; i < count; i++)
	{
		const int dev = devices ? devices[i] : i;
		tbvh_ctx c = 0;
		const int rc = tbvh_ctx_create( dev, &c );
		if (rc != TBVH_OK) { for (tbvh_ctx x : g->ctx) tbvh_ctx_destroy( x ); delete g; return rc; }
		g->ctx.push_back( c );
	}
	// let every device reach every other one directly (NVLink / NVSwitch); not fatal when a pair cannot
	for (int i = 0; i < count; i++) for (int j = 0; j < count; j++) if (i != j)
	{
		int can = 0;
		cudaDeviceCanAccessPeer( &can, g->ctx[i]->device, g->ctx[j]->device );
		if (can) { cudaSetDevice( g->ctx[i]->device ); if (cudaDeviceEnablePeerAccess( g->ctx[j]->device, 0 ) != cudaSuccess) cudaGetLastError(); }
	}
	*out = g;
	return TBVH_OK;
}

int tbvh_group_destroy( tbvh_group g )
{
	if (!g) return TBVH_OK;
	release_replicas( g );
	for (auto& b : g->host_blocks) { cudaHostUnregister( b.first ); munmap( b.first, b.second ); }
	for (tbvh_ctx c : g->ctx) tbvh_ctx_destroy( c );
	delete g;
	return TBVH_OK;
}

int tbvh_group_size( tbvh_group g ) { return g ? (int)g->ctx.size() : 0; }
tbvh_ctx tbvh_group_ctx( tbvh_group g, int i ) { return g && i >= 0 && i < (int)g->ctx.size() ? g->ctx[i] : 0; }
tbvh_bvh tbvh_group_replica( tbvh_group g, int i ) { return g && i >= 0 && i < (int)g->replica.size() ? g->replica[i] : 0; }

// Copy the traversal state of `src` (any context) to every device of the group.  The BVH2 arrays (node pairs, leaf-ordered
// triangles, primIdx, vertices) and, when resident, the CWBVH arrays travel; derived layouts that only serve downloads do not.
int tbvh_group_replicate( tbvh_group g, tbvh_bvh src, double* ms_out )
{
	ARG_CHECK( g && src, "NULL argument" );
	if (src->d_inst) { tbvh_set_error( "tbvh_group_replicate: a TLAS points into its BLAS handles and cannot be replicated by itself" ); return TBVH_E_UNSUPPORTED; }
	if (!(src->info.layouts & (1u << TBVH_LAYOUT_BVH)) && !src->d_cw_trav) { tbvh_set_error( "tbvh_group_replicate: the source holds no tree" ); return TBVH_E_STATE; }
	release_replicas( g );
	const int sdev = src->ctx->device;
	CUDA_TRY( cudaSetDevice( sdev ) );
	CUDA_TRY( cudaStreamSynchronize( src->ctx->stream ) );
	cudaEvent_t e0 = 0, e1 = 0;
	CUDA_TRY( cudaEventCreate( &e0 ) );
	CUDA_TRY( cudaEventCreate( &e1 ) );
	CUDA_TRY( cudaEventRecord( e0, src->ctx->stream ) );
	int rc = TBVH_OK;
	for (size_t i = 0; i < g->ctx.size() && rc == TBVH_OK; i++)
	{
		tbvh_ctx c = g->ctx[i];
		if (c == src->ctx) { g->replica.push_back( src ), g->owned.push_back( 0 ); continue; }
		tbvh_bvh r = 0;
		rc = tbvh_bvh_create( c, &r );
		if (rc != TBVH_OK) break;
		g->replica.push_back( r ), g->owned.push_back( 1 );
		auto body = [&]() -> int
		{
			CUDA_TRY( cudaSetDevice( c->device ) );
			cudaStream_t s = c->stream;
			r->info = src->info, r->root_ref = src->root_ref, r->root_count = src->root_count, r->refittable = src->refittable, r->cw_pending = src->cw_pending, r->cw_rd_limit = src->cw_rd_limit;
			const size_t nodes_b = (size_t)(src->info.used_nodes < 2 ? 2 : src->info.used_nodes) * 32;
			TRY( peer_clone( (void**)&r->d_verts, c->device, src->d_verts, sdev, (size_t)src->info.prim_count * 48, s ) );
			TRY( peer_clone( (void**)&r->d_prim_idx, c->device, src->d_prim_idx, sdev, (size_t)src->info.idx_count * 4, s ) );
			if (src->d_nodes) TRY( peer_clone( (void**)&r->d_nodes, c->device, src->d_nodes, sdev, nodes_b, s ) );
			if (src->d_trav == src->d_nodes) r->d_trav = r->d_nodes;
			else if (src->d_trav) TRY( peer_clone( (void**)&r->d_trav, c->device, src->d_trav, sdev, (size_t)src->info.used_nodes_gpu * 64, s ) );
			if (src->d_leaf_tris) { TRY( peer_clone( (void**)&r->d_leaf_tris, c->device, src->d_leaf_tris, sdev, (size_t)src->leaf_tris_count * 48, s ) ); r->leaf_tris_count = src->leaf_tris_count; }
			if (src->d_nodes_gpu) TRY( peer_clone( (void**)&r->d_nodes_gpu, c->device, src->d_nodes_gpu, sdev, (size_t)src->info.used_nodes_gpu * 64, s ) );
			if (src->d_cw_nodes) TRY( peer_clone( (void**)&r->d_cw_nodes, c->device, src->d_cw_nodes, sdev, (size_t)src->info.used_blocks * 16, s ) );
			if (src->d_cw_tris) TRY( peer_clone( (void**)&r->d_cw_tris, c->device, src->d_cw_tris, sdev, (size_t)src->info.cwbvh_tri_count * 48, s ) );
			if (src->d_cw_trav) TRY( peer_clone( (void**)&r->d_cw_trav, c->device, src->d_cw_trav, sdev, (size_t)(src->info.used_blocks / 5) * 160, s ) );
			return TBVH_OK;
		};
		rc = body();
	}
	for (tbvh_ctx c : g->ctx) { cudaSetDevice( c->device ); cudaStreamSynchronize( c->stream ); }
	cudaSetDevice( sdev );
	cudaEventRecord( e1, src->ctx->stream );
	cudaEventSynchronize( e1 );
	float ms = 0;
	cudaEventElapsedTime( &ms, e0, e1 );
	if (ms_out) *ms_out = ms;
	cudaEventDestroy( e0 ), cudaEventDestroy( e1 );
	if (rc != TBVH_OK) release_replicas( g );
	return rc;
}

int tbvh_group_intersect( tbvh_group g, int layout, void* rays, uint32_t stride, uint64_t n )
{
	ARG_CHECK( g && rays && stride >= 64, "bad arguments" );
	if (g->replica.size() != g->ctx.size()) { tbvh_set_error( "tbvh_group_intersect: call tbvh_group_replicate first" ); return TBVH_E_STATE; }
	const uint32_t parts = (uint32_t)g->ctx.size();
	return per_device( g, [&]( uint32_t p ) -> int
	{
		uint64_t first, count;
		tbvh_shard_range( n, p, parts, &first, &count );
		if (count == 0) return TBVH_OK;
		return tbvh_intersect( g->replica[p], layout, (char*)rays + first * stride, stride, count );
	} );
}

int tbvh_group_occluded( tbvh_group g, int layout, const void* rays, uint32_t stride, uint64_t n, uint32_t* bits )
{
	ARG_CHECK( g && rays && bits && stride >= 64, "bad arguments" );
	if (g->replica.size() != g->ctx.size()) { tbvh_set_error( "tbvh_group_occluded: call tbvh_group_replicate first" ); return TBVH_E_STATE; }
	const uint32_t parts = (uint32_t)g->ctx.size();
	return per_device( g, [&]( uint32_t p ) -> int
	{
		uint64_t first, count;
		tbvh_shard_range( n, p, parts, &first, &count );
		if (count == 0) return TBVH_OK;
		return tbvh_occluded( g->replica[p], layout, (const char*)rays + first * stride, stride, count, bits + first / 32 );
	} );
}

// A page-locked buffer of n records of `stride` bytes whose index ranges (tbvh_shard_range) sit on the NUMA node of the device
// that will read them: anonymous memory, first touched by a thread bound to each device's node, then registered with CUDA.
int tbvh_group_host_alloc( tbvh_group g, uint32_t stride, uint64_t n, void** out )
{
	ARG_CHECK( g && out && stride > 0 && n > 0, "bad arguments" );
	const size_t bytes = ((size_t)stride * n + 4095) & ~(size_t)4095;
	void* p = mmap( 0, bytes, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0 );
	if (p == MAP_FAILED) { tbvh_set_error( "tbvh_group_host_alloc: mmap( %zu ) failed", bytes ); return TBVH_E_ARG; }
	const uint32_t parts = (uint32_t)g->ctx.size();
	per_device( g, [&]( uint32_t part ) -> int
	{
		uint64_t first, count;
		tbvh_shard_range( n, part, parts, &first, &count );
		// first touch, page by page, from this device's node (pages at a range boundary go to whoever touches them first)
		char* a = (char*)p + first * stride, * e = a + count * stride;
		if (part + 1 == parts) e = (char*)p + bytes;
		for (char* q = (char*)((uintptr_t)a & ~(uintptr_t)4095); q < e; q += 4096) *(volatile char*)q = 0;
		return TBVH_OK;
	} );
	const cudaError_t err = cudaHostRegister( p, bytes, cudaHostRegisterPortable );
	if (err != cudaSuccess) { munmap( p, bytes ); tbvh_set_error( "tbvh_group_host_alloc: cudaHostRegister -> %s", cudaGetErrorString( err ) ); return TBVH_E_CUDA; }
	g->host_blocks.push_back( { p, bytes } );
	*out = p;
	return TBVH_OK;
}

int tbvh_group_host_free( tbvh_group g, void* p )
{
	ARG_CHECK( g, "NULL group" );
	for (size_t i = 0; i < g->host_blocks.size(); i++) if (g->host_blocks[i].first == p)
	{
		cudaHostUnregister( p );
		munmap( p, g->host_blocks[i].second );
		g->host_blocks.erase( g->host_blocks.begin() + i );
		return TBVH_OK;
	}
	tbvh_set_error( "tbvh_group_host_free: not a block of this group" );
	return TBVH_E_ARG;
}

} // extern "C"
