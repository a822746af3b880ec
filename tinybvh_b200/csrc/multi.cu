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
#include <unordered_map>
#include <algorithm>
#include <string>
#include <vector>
#include <new>

// A scene replica: one distinct BLAS handle of the last replicated TLAS, and its copy on every device of the group.  The copies are
// internal to the group: they hold the arrays the two-level walk reads (ARR_BLAS_*) and the host state the BLAS table is made from.
struct SceneBlas
{
	tbvh_bvh src;                     // the source handle, and the generation and revision the copies were taken at
	uint32_t generation, revision, what;
	std::vector<size_t> bytes;        // the size of every copied array (handle_arrays order)
	std::vector<tbvh_bvh> rep;        // rep[g] lives on ctx[g]; 0 on the source's own context
};

// what one destination context keeps between calls: the copy kernel's table on the device and its host image
struct CopyScratch { DevArray<char> d; std::vector<char> h; };

struct tbvh_group_t
{
	std::vector<tbvh_ctx> ctx;        // one per device
	std::vector<tbvh_bvh> replica;    // replica[g] lives on ctx[g]
	std::vector<char> owned;          // 0 where replica[g] IS the caller's source handle (its context belongs to the group)
	bool scene = false;               // the replicas are TLASes over the BLAS copies below
	std::vector<SceneBlas> blas;
	std::vector<uint32_t> tlas_cap;   // scene: instances the arrays of replica TLAS g were allocated for
	std::vector<CopyScratch> scratch; // one per context
	std::vector<std::pair<void*, size_t>> host_blocks; // tbvh_group_host_alloc results (mmap + cudaHostRegister)
};

static void release_replicas( tbvh_group g )
{
	for (size_t i = 0; i < g->replica.size(); i++) if (g->replica[i] && g->owned[i]) tbvh_bvh_destroy( g->replica[i] );
	for (SceneBlas& e : g->blas) for (tbvh_bvh r : e.rep) tbvh_bvh_destroy( r );
	g->replica.clear(), g->owned.clear(), g->blas.clear(), g->tlas_cap.clear();
	g->scene = false;
}

// ---- what a replica carries -------------------------------------------------------------------------------------------------------
// The device arrays of handle `src` a replica takes, each as (handle h's owner of it, bytes).  With h = src the list names the source
// arrays; with h = the replica, the owners to allocate, in the same order (presence and sizes come from src alone).
//   ARR_TREE      a plain-BVH replica: everything a walk in any layout reads, plus vertices and primIdx
//   ARR_BLAS_BVH  what the two-level walk reads of a BLAS's BVH2 (its BlasRef trav / tris): trav() and the leaf triangles
//   ARR_BLAS_CW   ... of its CWBVH (cw_nodes / cw_tris): the traversal nodes and bvh8Tris
//   ARR_TLAS      a TLAS's own node array, primIdx and instance table (its BLAS table is made for the replica, not copied)
enum { ARR_TREE = 1, ARR_BLAS_BVH = 2, ARR_BLAS_CW = 4, ARR_TLAS = 8 };
struct HandleArray { DevMem* at; size_t bytes; };

template <class M> static void add_array( std::vector<HandleArray>& a, const tbvh_bvh src, tbvh_bvh h, M tbvh_bvh_t::* m, const size_t bytes )
{
	if ((src->*m).p && bytes) a.push_back( HandleArray{ &(h->*m), bytes } );
}

static std::vector<HandleArray> handle_arrays( const tbvh_bvh src, tbvh_bvh h, const uint32_t what )
{
	std::vector<HandleArray> a;
	const tbvh_info& I = src->info;
	const size_t nodes_b = (size_t)(I.used_nodes < 2 ? 2 : I.used_nodes) * 32, gpu_b = (size_t)I.used_nodes_gpu * 64;
	if (what & ARR_TREE)
	{
		add_array( a, src, h, &tbvh_bvh_t::d_verts, (size_t)I.prim_count * 48 );
		add_array( a, src, h, &tbvh_bvh_t::d_prim_idx, (size_t)I.idx_count * 4 );
		add_array( a, src, h, &tbvh_bvh_t::d_nodes, nodes_b );
		add_array( a, src, h, &tbvh_bvh_t::d_pairs, gpu_b );
		add_array( a, src, h, &tbvh_bvh_t::d_leaf_tris, (size_t)src->leaf_tris_count * 48 );
		add_array( a, src, h, &tbvh_bvh_t::d_nodes_gpu, gpu_b );
		add_array( a, src, h, &tbvh_bvh_t::d_cw_nodes, (size_t)I.used_blocks * 16 );
	}
	if (what & ARR_BLAS_BVH)
	{
		if (src->d_pairs.p) add_array( a, src, h, &tbvh_bvh_t::d_pairs, gpu_b );
		else add_array( a, src, h, &tbvh_bvh_t::d_nodes, nodes_b );
		add_array( a, src, h, &tbvh_bvh_t::d_leaf_tris, (size_t)src->leaf_tris_count * 48 );
	}
	if (what & (ARR_TREE | ARR_BLAS_CW))
	{
		add_array( a, src, h, &tbvh_bvh_t::d_cw_tris, (size_t)I.cwbvh_tri_count * 48 );
		add_array( a, src, h, &tbvh_bvh_t::d_cw_trav, (size_t)(I.used_blocks / 5) * 160 );
	}
	if (what & ARR_TLAS)
	{
		add_array( a, src, h, &tbvh_bvh_t::d_nodes, nodes_b );
		add_array( a, src, h, &tbvh_bvh_t::d_prim_idx, (size_t)I.idx_count * 4 );
		add_array( a, src, h, &tbvh_bvh_t::d_inst, (size_t)src->inst_count * sizeof( TlasInst ) );
	}
	return a;
}

// ---- the copy kernel: every segment of one destination in one launch ------------------------------------------------------------------
// Segment k covers 16-byte units [first, first + ceil( bytes / 16 )) of the launch.  Every array is the start of a cudaMalloc block, so
// both ends are 16-byte aligned; the last unit of a segment whose size is not a multiple of 16 (a primIdx) is copied a word at a time.
struct CopySeg { const char* src; char* dst; uint64_t bytes; uint32_t first, pad; };

__global__ void __launch_bounds__( 256 ) k_copy_segments( const CopySeg* __restrict__ T, const uint32_t K, const uint32_t units )
{
	for (uint32_t u = blockIdx.x * blockDim.x + threadIdx.x; u < units; u += gridDim.x * blockDim.x)
	{
		const uint32_t k = batch_entry<CopySeg, &CopySeg::first>( T, K, u );
		const char* src = T[k].src;
		char* dst = T[k].dst;
		const uint64_t o = (uint64_t)(u - T[k].first) * 16, bytes = T[k].bytes;
		if (o + 16 <= bytes) *(uint4*)(dst + o) = *(const uint4*)(src + o);
		else for (uint64_t b = o; b < bytes; b += 4) *(uint32_t*)(dst + b) = *(const uint32_t*)(src + b);
	}
}

// can a kernel on dst_dev read memory of src_dev?  (tbvh_group_create enables peer access between the group's devices; a source
// context outside the group may sit on another device)
static bool peer_readable( const int dst_dev, const int src_dev )
{
	if (dst_dev == src_dev) return true;
	int can = 0;
	if (cudaDeviceCanAccessPeer( &can, dst_dev, src_dev ) != cudaSuccess || !can) { cudaGetLastError(); return false; }
	if (cudaSetDevice( dst_dev ) != cudaSuccess) { cudaGetLastError(); return false; }
	const cudaError_t e = cudaDeviceEnablePeerAccess( src_dev, 0 );
	cudaGetLastError(); // cudaErrorPeerAccessAlreadyEnabled is the usual answer
	return e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled;
}

// Enqueue on context i's stream the copy of every segment (sources on src_dev, destinations on context i's device), then `tail_bytes`
// of host data to tail_dst on context i's device.  One table upload and one k_copy_segments launch; where context i's device cannot
// read src_dev, one cudaMemcpyPeerAsync per segment instead.  The host data must live until the stream has run the copies.
static int copy_to( tbvh_group g, const size_t i, const int src_dev, std::vector<CopySeg>& segs, const void* tail, const size_t tail_bytes, void* tail_dst )
{
	const tbvh_ctx c = g->ctx[i];
	const cudaStream_t s = c->stream;
	uint64_t units = 0;
	for (const CopySeg& q : segs) units += (q.bytes + 15) / 16;
	const bool kernel = peer_readable( c->device, src_dev ) && units + (tail_bytes + 15) / 16 < 0xffffffffull;
	CUDA_TRY( cudaSetDevice( c->device ) );
	if (!kernel)
	{
		for (const CopySeg& q : segs) CUDA_TRY( cudaMemcpyPeerAsync( q.dst, c->device, q.src, src_dev, q.bytes, s ) );
		if (tail_bytes) CUDA_TRY( cudaMemcpyAsync( tail_dst, tail, tail_bytes, cudaMemcpyHostToDevice, s ) );
		return TBVH_OK;
	}
	// the device image: the segment table, then the host data, which the table's last segment copies to tail_dst
	CopyScratch& X = g->scratch[i];
	const size_t K = segs.size() + (tail_bytes ? 1 : 0), tail_at = K * sizeof( CopySeg ), bytes = tail_at + tail_bytes;
	TRY( X.d.reserve( bytes ) );
	if (tail_bytes) segs.push_back( CopySeg{ (const char*)X.d + tail_at, (char*)tail_dst, tail_bytes, 0, 0 } );
	uint32_t first = 0;
	for (CopySeg& q : segs) q.first = first, first += (uint32_t)((q.bytes + 15) / 16);
	if (first == 0) return TBVH_OK;
	X.h.resize( bytes );
	memcpy( X.h.data(), segs.data(), tail_at );
	if (tail_bytes) memcpy( X.h.data() + tail_at, tail, tail_bytes );
	CUDA_TRY( cudaMemcpyAsync( X.d, X.h.data(), bytes, cudaMemcpyHostToDevice, s ) );
	const uint32_t grid = std::min<uint32_t>( (first + 255) / 256, (uint32_t)c->sm_count * 8 );
	k_copy_segments<<<grid, 256, 0, s>>>( (const CopySeg*)X.d.p, (uint32_t)K, first );
	LAUNCHED();
	return TBVH_OK;
}

// the segments that copy src's arrays (what) into h's
static void add_segments( std::vector<CopySeg>& segs, const tbvh_bvh src, tbvh_bvh h, const uint32_t what )
{
	const std::vector<HandleArray> from = handle_arrays( src, src, what ), to = handle_arrays( src, h, what );
	for (size_t j = 0; j < from.size(); j++) segs.push_back( CopySeg{ (const char*)from[j].at->p, (char*)to[j].at->p, from[j].bytes, 0, 0 } );
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
	g->scratch.resize( count );
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
	for (size_t i = 0; i < g->ctx.size(); i++) if (g->scratch[i].d) { cudaSetDevice( g->ctx[i]->device ); g->scratch[i].d.reset(); }
	for (auto& b : g->host_blocks) { cudaHostUnregister( b.first ); munmap( b.first, b.second ); }
	for (tbvh_ctx c : g->ctx) tbvh_ctx_destroy( c );
	delete g;
	return TBVH_OK;
}

int tbvh_group_size( tbvh_group g ) { return g ? (int)g->ctx.size() : 0; }
tbvh_ctx tbvh_group_ctx( tbvh_group g, int i ) { return g && i >= 0 && i < (int)g->ctx.size() ? g->ctx[i] : 0; }
tbvh_bvh tbvh_group_replica( tbvh_group g, int i ) { return g && i >= 0 && i < (int)g->replica.size() ? g->replica[i] : 0; }

// A plain BVH: the group's replicas are released and made again.  Every array of ARR_TREE travels; derived layouts that only serve
// downloads do not.
static int replicate_tree( tbvh_group g, tbvh_bvh src, bool& began )
{
	if (!(src->info.layouts & (1u << TBVH_LAYOUT_BVH)) && !src->d_cw_trav) { tbvh_set_error( "tbvh_group_replicate: the source holds no tree" ); return TBVH_E_STATE; }
	began = true;
	release_replicas( g );
	for (size_t i = 0; i < g->ctx.size(); i++)
	{
		tbvh_ctx c = g->ctx[i];
		if (c == src->ctx) { g->replica.push_back( src ), g->owned.push_back( 0 ); continue; }
		tbvh_bvh r = 0;
		TRY( tbvh_bvh_create( c, &r ) );
		g->replica.push_back( r ), g->owned.push_back( 1 );
		r->info = src->info, r->root_ref = src->root_ref, r->root_count = src->root_count, r->refittable = src->refittable, r->cw_pending = src->cw_pending, r->cw_rd_limit = src->cw_rd_limit;
		r->leaf_tris_count = src->d_leaf_tris ? src->leaf_tris_count : 0;
		for (const HandleArray& a : handle_arrays( src, r, ARR_TREE )) TRY( a.at->alloc( a.bytes ) );
		std::vector<CopySeg> segs;
		add_segments( segs, src, r, ARR_TREE );
		TRY( copy_to( g, i, src->ctx->device, segs, 0, 0, 0 ) );
	}
	return TBVH_OK;
}

// A TLAS: per device one replica TLAS over one replica of every distinct BLAS it links to (SceneBlas).  A later call refreshes them in
// place: unchanged BLASes are not copied, changed ones of unchanged sizes are copied into their arrays, the TLAS arrays are reused while
// they are large enough, and every byte bound for one device goes in one k_copy_segments launch.
static int replicate_scene( tbvh_group g, tbvh_bvh src, bool& began )
{
	// the refusals: the previous replicas stay as they are
	TRY( tlas_stale_check( src ) );
	const uint32_t walkable = src->tlas_blas_layouts & ((1u << TBVH_LAYOUT_BVH) | (1u << TBVH_LAYOUT_CWBVH));
	if (!src->d_nodes || !src->d_prim_idx || !src->d_inst || !walkable)
	{ tbvh_set_error( "tbvh_group_replicate: the TLAS can be walked in no layout (not every BLAS held a BVH or CWBVH tree it can walk)" ); return TBVH_E_STATE; }
	for (size_t i = 0; i < g->ctx.size(); i++) if (g->ctx[i]->inst_idx_bits != src->ctx->inst_idx_bits)
	{
		tbvh_set_error( "tbvh_group_replicate: device %zu of the group stores TLAS hits with inst_idx_bits %d, the source's context with %d", i,
			g->ctx[i]->inst_idx_bits, src->ctx->inst_idx_bits );
		return TBVH_E_STATE;
	}
	began = true;
	if (!g->scene) release_replicas( g );
	const size_t D = g->ctx.size();
	g->replica.resize( D, 0 ), g->owned.resize( D, 0 ), g->tlas_cap.resize( D, 0 );
	g->scene = true;
	// only the layouts the source can be walked in: a BLAS array no walk of the TLAS reads does not travel
	const uint32_t what = (walkable & (1u << TBVH_LAYOUT_BVH) ? ARR_BLAS_BVH : 0) | (walkable & (1u << TBVH_LAYOUT_CWBVH) ? ARR_BLAS_CW : 0);
	// the distinct BLAS handles in order of first appearance; BLAS k of the TLAS is entry slot[k].  Entries of handles the TLAS no
	// longer links to are released.
	const uint32_t nb = (uint32_t)src->links.size();
	std::unordered_map<tbvh_bvh, uint32_t> old_at, at;
	for (uint32_t j = 0; j < g->blas.size(); j++) old_at[g->blas[j].src] = j;
	std::vector<uint32_t> slot( nb );
	std::vector<SceneBlas> next;
	for (uint32_t k = 0; k < nb; k++)
	{
		const tbvh_bvh b = src->links[k].blas;
		auto f = at.find( b );
		if (f != at.end()) { slot[k] = f->second; continue; }
		slot[k] = at[b] = (uint32_t)next.size();
		auto o = old_at.find( b );
		if (o != old_at.end()) next.push_back( std::move( g->blas[o->second] ) ), g->blas[o->second].rep.clear();
		else next.push_back( SceneBlas{ b, 0, 0, 0, {}, std::vector<tbvh_bvh>( D, 0 ) } );
	}
	for (SceneBlas& e : g->blas) for (tbvh_bvh r : e.rep) tbvh_bvh_destroy( r );
	g->blas = std::move( next );
	// per entry: copy when the source moved on, reallocate when an array size changed
	std::vector<char> changed( g->blas.size() ), realloc( g->blas.size() );
	for (size_t j = 0; j < g->blas.size(); j++)
	{
		SceneBlas& e = g->blas[j];
		const tbvh_bvh b = e.src;
		std::vector<size_t> bytes;
		for (const HandleArray& a : handle_arrays( b, b, what )) bytes.push_back( a.bytes );
		changed[j] = e.generation != b->generation || e.revision != b->revision || e.what != what;
		realloc[j] = e.what != what || bytes != e.bytes;
		e.generation = b->generation, e.revision = b->revision, e.what = what, e.bytes = bytes;
	}
	std::vector<tbvh_bvh> hs( nb );
	for (size_t i = 0; i < D; i++)
	{
		const tbvh_ctx c = g->ctx[i];
		if (c == src->ctx)
		{
			// the source's own context: its replica is the source, and the group holds nothing there
			if (g->replica[i] && g->owned[i]) tbvh_bvh_destroy( g->replica[i] );
			for (SceneBlas& e : g->blas) if (e.rep[i]) tbvh_bvh_destroy( e.rep[i] ), e.rep[i] = 0;
			g->replica[i] = src, g->owned[i] = 0, g->tlas_cap[i] = 0;
			continue;
		}
		CUDA_TRY( cudaSetDevice( c->device ) );
		std::vector<CopySeg> segs;
		for (size_t j = 0; j < g->blas.size(); j++)
		{
			SceneBlas& e = g->blas[j];
			tbvh_bvh& r = e.rep[i];
			const bool fresh = r && !realloc[j];
			if (!fresh)
			{
				if (r) tbvh_bvh_destroy( r ), r = 0; // a new handle: a new generation for the replica TLAS's links
				TRY( tbvh_bvh_create( c, &r ) );
				for (const HandleArray& a : handle_arrays( e.src, r, what )) TRY( a.at->alloc( a.bytes ) );
			}
			if (!fresh || changed[j]) add_segments( segs, e.src, r, what );
			const tbvh_bvh b = e.src;
			r->info = b->info, r->root_ref = b->root_ref, r->root_count = b->root_count, r->cw_rd_limit = b->cw_rd_limit, r->cw_pending = b->cw_pending;
			r->leaf_tris_count = (what & ARR_BLAS_BVH) ? b->leaf_tris_count : 0, r->refittable = false;
		}
		// the replica TLAS: its arrays are kept while they hold the source's instances, its BLAS table is made over the replicas
		tbvh_bvh t = g->owned[i] ? g->replica[i] : 0;
		if (t && (g->tlas_cap[i] < src->inst_count || t->blas_count != src->blas_count)) tbvh_bvh_destroy( t ), t = 0;
		g->replica[i] = 0, g->owned[i] = 0;
		if (!t)
		{
			TRY( tbvh_bvh_create( c, &t ) );
			g->replica[i] = t, g->owned[i] = 1;
			const size_t cap = src->inst_count;
			TRY( t->d_nodes.alloc( (2 * cap + 2) * 32 ) ); // the builder's own allocation (build_sah.cu)
			TRY( t->d_prim_idx.alloc( cap * 4 ) );
			TRY( t->d_inst.alloc( cap * sizeof( TlasInst ) ) );
			TRY( t->d_blas.alloc( (size_t)src->blas_count * sizeof( BlasRef ) ) );
			g->tlas_cap[i] = src->inst_count;
		}
		g->replica[i] = t, g->owned[i] = 1;
		add_segments( segs, src, t, ARR_TLAS );
		t->info = src->info, t->root_ref = src->root_ref, t->root_count = src->root_count, t->refittable = false;
		t->inst_count = src->inst_count, t->blas_count = src->blas_count;
		for (uint32_t k = 0; k < nb; k++) hs[k] = g->blas[slot[k]].rep[i];
		TlasBlasTable B;
		TRY( tlas_blas_table( t, hs.data(), nb, B ) );
		// the walks refuse exactly what the source's refuse: its layouts and deep BLAS, not what the replicas' table finds
		t->tlas_blas_layouts = src->tlas_blas_layouts, t->tlas_deep_blas = src->tlas_deep_blas, t->tlas_deep_depth = src->tlas_deep_depth;
		t->links.clear();
		for (uint32_t k = 0; k < nb; k++) t->links.push_back( BlasLink{ hs[k], hs[k]->generation } );
		TRY( copy_to( g, i, src->ctx->device, segs, B.refs.data(), B.refs.size() * sizeof( BlasRef ), t->d_blas ) );
	}
	return TBVH_OK;
}

// Copy the traversal state of `src` (any context) to every device of the group (include/tinybvh_b200.h).
int tbvh_group_replicate( tbvh_group g, tbvh_bvh src, double* ms_out )
{
	ARG_CHECK( g && src, "NULL argument" );
	for (size_t i = 0; i < g->replica.size(); i++) ARG_CHECK( !(g->owned[i] && g->replica[i] == src), "the source is a replica of this group" );
	const int sdev = src->ctx->device;
	CUDA_TRY( cudaSetDevice( sdev ) );
	CUDA_TRY( cudaStreamSynchronize( src->ctx->stream ) );
	cudaEvent_t e0 = 0, e1 = 0;
	CUDA_TRY( cudaEventCreate( &e0 ) );
	CUDA_TRY( cudaEventCreate( &e1 ) );
	CUDA_TRY( cudaEventRecord( e0, src->ctx->stream ) );
	bool began = false; // past the refusals: a failure releases every replica
	const int rc = src->d_inst ? replicate_scene( g, src, began ) : replicate_tree( g, src, began );
	for (tbvh_ctx c : g->ctx) { cudaSetDevice( c->device ); cudaStreamSynchronize( c->stream ); }
	cudaSetDevice( sdev );
	cudaEventRecord( e1, src->ctx->stream );
	cudaEventSynchronize( e1 );
	float ms = 0;
	cudaEventElapsedTime( &ms, e0, e1 );
	if (ms_out) *ms_out = ms;
	cudaEventDestroy( e0 ), cudaEventDestroy( e1 );
	if (rc != TBVH_OK && began) release_replicas( g );
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
