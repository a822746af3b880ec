// tinybvh_b200/csrc/api.cu - C-ABI entry points (include/tinybvh_b200.h): contexts, handles, uploads, the host-buffer
// traversal pipeline.  Kernels live in trace_bvh2.cu / trace_cwbvh.cu / build_sah.cu / convert.cu.
#include "common.cuh"
#include "instance_update.cuh"
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <cmath>
#include <vector>
#include <thread>
#include <atomic>
#include <mutex>
#include <condition_variable>
#include <memory>
#include <functional>
#include <new>

static thread_local char g_err[512] = "";
unsigned long long g_tbvh_launches = 0;

void tbvh_set_error( const char* fmt, ... )
{
	va_list ap;
	va_start( ap, fmt );
	vsnprintf( g_err, sizeof( g_err ), fmt, ap );
	va_end( ap );
}

// ---- host topology: which NUMA node a device hangs off, and its CPUs (sysfs; no libnuma in the image) -----------------
#include <sched.h>
#include <unistd.h>
#include <sys/mman.h>
#include <sys/syscall.h>

static int read_int_file( const char* path, int fallback )
{
	FILE* f = fopen( path, "r" );
	if (!f) return fallback;
	int v = fallback;
	if (fscanf( f, "%d", &v ) != 1) v = fallback;
	fclose( f );
	return v;
}

static int device_numa_node( int device )
{
	char bus[32] = "";
	if (cudaDeviceGetPCIBusId( bus, sizeof( bus ), device ) != cudaSuccess) { cudaGetLastError(); return -1; }
	for (char* c = bus; *c; c++) if (*c >= 'A' && *c <= 'Z') *c += 'a' - 'A';
	char path[128];
	snprintf( path, sizeof( path ), "/sys/bus/pci/devices/%s/numa_node", bus );
	return read_int_file( path, -1 );
}

// CPUs of a NUMA node from /sys/devices/system/node/nodeN/cpulist ("0-31,64-95")
static bool node_cpus( int node, cpu_set_t* set )
{
	CPU_ZERO( set );
	if (node < 0) return false;
	char path[128], line[1024] = "";
	snprintf( path, sizeof( path ), "/sys/devices/system/node/node%d/cpulist", node );
	FILE* f = fopen( path, "r" );
	if (!f) return false;
	const bool ok = fgets( line, sizeof( line ), f ) != 0;
	fclose( f );
	if (!ok) return false;
	int any = 0;
	for (char* p = line; *p && *p != '\n';)
	{
		char* e;
		long lo = strtol( p, &e, 10 ), hi = lo;
		if (e == p) break;
		if (*e == '-') { p = e + 1; hi = strtol( p, &e, 10 ); }
		for (long c = lo; c <= hi && c < CPU_SETSIZE; c++) CPU_SET( (int)c, set ), any = 1;
		p = *e == ',' ? e + 1 : e;
	}
	return any != 0;
}

// run `fn` with the calling thread restricted to the CPUs of `node` (first-touch and driver allocations then land on that node),
// then restore the previous affinity.  Without topology information fn just runs.
template <class F> static auto on_node( int node, F fn ) -> decltype( fn() )
{
	cpu_set_t want, old;
	const bool have = node_cpus( node, &want ) && sched_getaffinity( 0, sizeof( old ), &old ) == 0 && sched_setaffinity( 0, sizeof( want ), &want ) == 0;
	auto r = fn();
	if (have) sched_setaffinity( 0, sizeof( old ), &old );
	return r;
}

// A few persistent host threads, bound to the CPUs of one NUMA node, that run fn( t, T ) in parallel and block the caller until
// every slice is done (d2h_mode 2: hits scattered into the caller's strided ray records).
struct HostPool
{
	HostPool( unsigned threads, int node ) : T( threads )
	{
		for (unsigned t = 0; t < T; t++) th.emplace_back( [this, t, node]()
		{
			cpu_set_t want;
			if (node_cpus( node, &want )) sched_setaffinity( 0, sizeof( want ), &want );
			uint64_t seen = 0;
			for (;;)
			{
				std::unique_lock<std::mutex> lk( m );
				cv_go.wait( lk, [&]() { return quit || gen != seen; } );
				if (quit) return;
				seen = gen;
				lk.unlock();
				job( t, T );
				lk.lock();
				if (++done == T) cv_done.notify_one();
			}
		} );
	}
	~HostPool() { { std::lock_guard<std::mutex> lk( m ); quit = true; } cv_go.notify_all(); for (auto& t : th) t.join(); }
	template <class F> void run( F fn )
	{
		{ std::lock_guard<std::mutex> lk( m ); job = fn, done = 0, gen++; }
		cv_go.notify_all();
		std::unique_lock<std::mutex> lk( m );
		cv_done.wait( lk, [&]() { return done == T; } );
	}
	unsigned T;
	std::vector<std::thread> th;
	std::mutex m;
	std::condition_variable cv_go, cv_done;
	std::function<void( unsigned, unsigned )> job;
	uint64_t gen = 0;
	unsigned done = 0;
	bool quit = false;
};

extern "C" {

const char* tbvh_last_error( void ) { return g_err; }
uint64_t tbvh_launch_count( void ) { return g_tbvh_launches; }

int tbvh_device_count( void )
{
	int n = 0;
	if (cudaGetDeviceCount( &n ) != cudaSuccess) { cudaGetLastError(); return 0; }
	return n;
}

int tbvh_device_numa_node( int device ) { return device_numa_node( device ); }

int tbvh_bind_thread_to_device( int device )
{
	cpu_set_t want;
	const int node = device_numa_node( device );
	if (!node_cpus( node, &want )) { tbvh_set_error( "tbvh_bind_thread_to_device: no NUMA information for device %d", device ); return TBVH_E_UNSUPPORTED; }
	if (sched_setaffinity( 0, sizeof( want ), &want ) != 0) { tbvh_set_error( "tbvh_bind_thread_to_device: sched_setaffinity failed" ); return TBVH_E_UNSUPPORTED; }
	return TBVH_OK;
}

int tbvh_ctx_destroy( tbvh_ctx c );

int tbvh_ctx_create( int device, tbvh_ctx* out )
{
	ARG_CHECK( out, "out == NULL" );
	int n = 0;
	CUDA_TRY( cudaGetDeviceCount( &n ) );
	if (device < 0 || device >= n) { tbvh_set_error( "tbvh_ctx_create: device %d of %d - no CUDA device, and there is no CPU fallback", device, n ); return TBVH_E_CUDA; }
	CUDA_TRY( cudaSetDevice( device ) );
	tbvh_ctx c = new (std::nothrow) tbvh_ctx_t();
	ARG_CHECK( c, "out of host memory" );
	c->device = device;
	c->numa_node = device_numa_node( device );
	auto body = [&]() -> int
	{
		cudaDeviceProp prop;
		CUDA_TRY( cudaGetDeviceProperties( &prop, device ) );
		c->sm_count = prop.multiProcessorCount;
		CUDA_TRY( cudaStreamCreateWithFlags( &c->stream, cudaStreamNonBlocking ) );
		CUDA_TRY( cudaStreamCreateWithFlags( &c->s_in, cudaStreamNonBlocking ) );
		CUDA_TRY( cudaStreamCreateWithFlags( &c->s_run, cudaStreamNonBlocking ) );
		CUDA_TRY( cudaStreamCreateWithFlags( &c->s_out, cudaStreamNonBlocking ) );
		for (int i = 0; i < 3; i++) CUDA_TRY( cudaStreamCreateWithFlags( &c->s_in_part[i], cudaStreamNonBlocking ) );
		CUDA_TRY( cudaEventCreateWithFlags( &c->ev_fork, cudaEventDisableTiming ) );
		for (int i = 0; i < TBVH_SLOTS; i++)
		{
			CUDA_TRY( cudaEventCreateWithFlags( &c->slot[i].in_done, cudaEventDisableTiming ) );
			CUDA_TRY( cudaEventCreateWithFlags( &c->slot[i].run_done, cudaEventDisableTiming ) );
			CUDA_TRY( cudaEventCreateWithFlags( &c->slot[i].out_done, cudaEventDisableTiming ) );
			for (int p = 0; p < 3; p++) CUDA_TRY( cudaEventCreateWithFlags( &c->ev_part[i][p], cudaEventDisableTiming ) );
		}
		TRY( c->d_counters.alloc( TBVH_COUNTERS * 8 ) );
		CUDA_TRY( cudaMemset( c->d_counters, 0, TBVH_COUNTERS * 8 ) );
		return TBVH_OK;
	};
	const int rc = body();
	if (rc != TBVH_OK) { tbvh_ctx_destroy( c ); return rc; }
	const char* hp = getenv( "TBVH_HOST_PATH" );
	c->host_path = hp && (!strcmp( hp, "zerocopy" ) || !strcmp( hp, "1" )) ? 1 : hp && !strcmp( hp, "2" ) ? 2 : 0;
	const char* tv = getenv( "TBVH_TRACE_VARIANT" );
	c->trace_variant = tv ? atoi( tv ) : 3; // octant switch: warp-uniform octant instances for coherent camera / shadow rays; mixed-octant warps pay a vote
	const char* bc = getenv( "TBVH_BUILD_CTAS" );
	if (bc) c->build_ctas = atoi( bc );
	const char* bm = getenv( "TBVH_BUILD_MODE" );
	if (bm) c->build_mode = atoi( bm ) ? 1 : 0;
	const char* st = getenv( "TBVH_SMALL_T" );
	c->small_t = st ? atoi( st ) : 128;
	const char* hs = getenv( "TBVH_HQ_SMALL" );
	if (hs) c->hq_small = atoi( hs );
	const char* hc = getenv( "TBVH_HQ_CLUSTER" );
	if (hc) c->hq_cluster = atoi( hc );
	const char* dm = getenv( "TBVH_D2H_MODE" );
	c->d2h_mode = dm ? atoi( dm ) : 1; // whole first cache lines back: one host-memory write per ray instead of a partial-line update
	if (c->d2h_mode < 0 || c->d2h_mode > 3) c->d2h_mode = 1;
	const char* sp = getenv( "TBVH_H2D_SPLIT" );
	c->h2d_split = sp ? atoi( sp ) : 1;
	if (c->h2d_split < 1) c->h2d_split = 1;
	if (c->h2d_split > 4) c->h2d_split = 4;
	const char* stn = getenv( "TBVH_SCATTER_THREADS" );
	if (stn && atoi( stn ) >= 1 && atoi( stn ) <= 64) c->scatter_threads = atoi( stn );
	const char* cr = getenv( "TBVH_CHUNK_RAYS" );
	if (cr && atol( cr ) >= 4096) c->chunk_rays = (size_t)atol( cr ) & ~(size_t)31;
	*out = c;
	return TBVH_OK;
}

static void free_slots( tbvh_ctx c )
{
	for (HostSlot& sl : c->slot) sl.d_rays.reset(), sl.d_hits.reset(), sl.d_bits.reset(), sl.h_hits.reset();
	c->slot_rays = 0, c->slot_rec = 0;
}

int tbvh_ctx_destroy( tbvh_ctx c )
{
	if (!c) return TBVH_OK;
	cudaSetDevice( c->device );
	cudaDeviceSynchronize();
	for (int i = 0; i < TBVH_SLOTS; i++)
	{
		if (c->slot[i].in_done) cudaEventDestroy( c->slot[i].in_done );
		if (c->slot[i].run_done) cudaEventDestroy( c->slot[i].run_done );
		if (c->slot[i].out_done) cudaEventDestroy( c->slot[i].out_done );
		for (int p = 0; p < 3; p++) if (c->ev_part[i][p]) cudaEventDestroy( c->ev_part[i][p] );
	}
	if (c->ev_fork) cudaEventDestroy( c->ev_fork );
	for (int i = 0; i < 3; i++) if (c->s_in_part[i]) cudaStreamDestroy( c->s_in_part[i] );
	if (c->s_in) cudaStreamDestroy( c->s_in );
	if (c->s_run) cudaStreamDestroy( c->s_run );
	if (c->s_out) cudaStreamDestroy( c->s_out );
	if (c->stream) cudaStreamDestroy( c->stream );
	if (c->refit_e0) cudaEventDestroy( c->refit_e0 );
	if (c->refit_e1) cudaEventDestroy( c->refit_e1 );
	delete c->pool;
	delete c; // its buffers (slots, counters, refit and gather staging) free themselves on the device set above
	return TBVH_OK;
}

int tbvh_set_option( tbvh_ctx c, const char* key, int value )
{
	ARG_CHECK( c && key, "NULL argument" );
	if (!strcmp( key, "trace_variant" )) c->trace_variant = value;
	else if (!strcmp( key, "small_t" )) c->small_t = value;
	else if (!strcmp( key, "small_mode" )) c->small_mode = value & 3;
	else if (!strcmp( key, "build_mode" )) c->build_mode = value ? 1 : 0;
	else if (!strcmp( key, "build_ctas" )) c->build_ctas = value < 0 ? 0 : value > 16 ? 16 : value;
	else if (!strcmp( key, "inst_idx_bits" )) c->inst_idx_bits = value;
	else if (!strcmp( key, "hq_small" )) c->hq_small = value;
	else if (!strcmp( key, "hq_cluster" )) c->hq_cluster = value;
	else if (!strcmp( key, "d2h_mode" )) c->d2h_mode = value >= 0 && value <= 3 ? value : 0;
	else if (!strcmp( key, "scatter_threads" ))
	{
		ARG_CHECK( value >= 1 && value <= 64, "scatter_threads must be 1..64" );
		std::lock_guard<std::mutex> lk( c->host_mutex );
		delete c->pool;
		c->pool = 0, c->scatter_threads = value;
	}
	else if (!strcmp( key, "h2d_split" )) c->h2d_split = value < 1 ? 1 : value > 4 ? 4 : value;
	else if (!strcmp( key, "host_path" ))
	{
		std::lock_guard<std::mutex> lk( c->host_mutex );
		c->host_path = value == 1 ? 1 : value == 2 ? 2 : 0;
	}
	else if (!strcmp( key, "chunk_rays" ))
	{
		ARG_CHECK( value >= 4096, "chunk_rays must be at least 4096" );
		std::lock_guard<std::mutex> lk( c->host_mutex );
		CUDA_TRY( cudaSetDevice( c->device ) );
		CUDA_TRY( cudaDeviceSynchronize() );
		free_slots( c );
		c->chunk_rays = (size_t)value & ~(size_t)31;
	}
	else { tbvh_set_error( "tbvh_set_option: unknown key '%s'", key ); return TBVH_E_ARG; }
	return TBVH_OK;
}

// Page-locked ray buffers.  The pages are allocated while the calling thread sits on the CPUs of the device's NUMA node, so the
// DMA engine reads local memory (a dual-socket host serves a remote GPU's reads over the inter-socket link otherwise).
// blocks handed out by the huge-page path (mmap + MADV_HUGEPAGE + cudaHostRegister): tbvh_host_free must munmap them
static std::mutex g_huge_mutex;
static std::vector<std::pair<void*, size_t>> g_huge;

static int host_alloc_on_node( int node, size_t bytes, void** out );
int tbvh_host_alloc_near( int device, size_t bytes, void** out ) { return host_alloc_on_node( device_numa_node( device ), bytes, out ); }
int tbvh_host_alloc_node( int node, size_t bytes, void** out ) { return host_alloc_on_node( node, bytes, out ); }
static int host_alloc_on_node( int node, size_t bytes, void** out )
{
	ARG_CHECK( out, "out == NULL" );
	static int huge = -1;
	if (huge < 0) { const char* e = getenv( "TBVH_HOST_HUGE" ); huge = e ? atoi( e ) : 1; } // default on: fewer page translations for DMA where an IOMMU translates addresses
	if (huge && bytes >= (8u << 20))
	{
		// anonymous memory advised into transparent huge pages, first touched on the device's node, then page-locked: 2 MiB pages
		// mean 512x fewer IOMMU / address-translation entries for the DMA engine than 4 KiB ones
		const size_t sz = (bytes + (2u << 20) - 1) & ~(size_t)((2u << 20) - 1);
		void* p = mmap( 0, sz, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0 );
		if (p != MAP_FAILED)
		{
			madvise( p, sz, MADV_HUGEPAGE );
			const cudaError_t e = on_node( node, [&]() { for (size_t o = 0; o < sz; o += 4096) ((volatile char*)p)[o] = 0; return cudaHostRegister( p, sz, cudaHostRegisterPortable ); } );
			if (e == cudaSuccess) { std::lock_guard<std::mutex> lk( g_huge_mutex ); g_huge.push_back( { p, sz } ); *out = p; return TBVH_OK; }
			cudaGetLastError();
			munmap( p, sz );
		}
	}
	const cudaError_t e = on_node( node, [&]() { return cudaHostAlloc( out, bytes, cudaHostAllocPortable ); } );
	if (e != cudaSuccess) { tbvh_set_error( "tbvh_host_alloc: cudaHostAlloc( %zu ) -> %s", bytes, cudaGetErrorString( e ) ); return TBVH_E_CUDA; }
	return TBVH_OK;
}
int tbvh_host_alloc( size_t bytes, void** out )
{
	int device = 0;
	if (cudaGetDevice( &device ) != cudaSuccess) { cudaGetLastError(); device = 0; }
	return tbvh_host_alloc_near( device, bytes, out );
}
int tbvh_host_free( void* p )
{
	if (!p) return TBVH_OK;
	{
		std::lock_guard<std::mutex> lk( g_huge_mutex );
		for (size_t i = 0; i < g_huge.size(); i++) if (g_huge[i].first == p)
		{
			cudaHostUnregister( p );
			munmap( p, g_huge[i].second );
			g_huge.erase( g_huge.begin() + i );
			return TBVH_OK;
		}
	}
	CUDA_TRY( cudaFreeHost( p ) );
	return TBVH_OK;
}
int tbvh_host_register( void* p, size_t bytes ) { CUDA_TRY( cudaHostRegister( p, bytes, cudaHostRegisterPortable ) ); return TBVH_OK; }
int tbvh_host_unregister( void* p ) { CUDA_TRY( cudaHostUnregister( p ) ); return TBVH_OK; }

static void live_add( tbvh_bvh b );
static void live_remove( tbvh_bvh b );

int tbvh_bvh_create( tbvh_ctx ctx, tbvh_bvh* out )
{
	ARG_CHECK( ctx && out, "NULL argument" );
	std::unique_ptr<tbvh_bvh_t> h( new (std::nothrow) tbvh_bvh_t() );
	ARG_CHECK( h, "out of host memory" );
	h->ctx = ctx;
	CUDA_TRY( cudaSetDevice( ctx->device ) );
	TRY( h->d_stats.alloc( 32 ) );
	CUDA_TRY( cudaMemset( h->d_stats, 0, 32 ) );
	tbvh_bvh b = h.release();
	b->generation = tbvh_next_generation();
	live_add( b );
	*out = b;
	return TBVH_OK;
}

static void free_layouts( tbvh_bvh b )
{
	drop_bvh_gpu( b );
	drop_cwbvh( b );
	DevMem* const arrays[] = { &b->d_verts, &b->d_vert_idx, &b->d_nodes, &b->d_prim_idx, &b->d_pairs, &b->d_leaf_tris, &b->d_aabbs, &b->d_inst, &b->d_blas, &b->d_inst_stage, &b->d_sdf, &b->d_wn, &b->d_wn_own };
	for (DevMem* a : arrays) a->reset();
	b->vert_count = 0, b->leaf_tris_count = 0;
	b->blas_table_bytes = 0, b->inst_count = 0, b->blas_count = 0, b->tlas_blas_layouts = 0;
	b->tlas_deep_blas = 0, b->tlas_deep_depth = 0;
	b->links.clear();
	b->generation = tbvh_next_generation(); // a TLAS built over the old arrays must notice (tlas_check)
	b->tree_stamp = tbvh_next_generation();
	memset( &b->info, 0, sizeof( b->info ) );
	b->refittable = true, b->stray_slots = false;
}

// what a handle holds once a builder or tbvh_optimize has written its tree into d_nodes / d_prim_idx
static void install_tree( tbvh_bvh b, const BuiltTree& r, const float ms )
{
	b->info.used_nodes = r.used_nodes, b->info.idx_count = r.idx_count, b->info.max_depth = r.max_depth;
	memcpy( b->info.aabb_min, r.root, 12 ), memcpy( b->info.aabb_max, r.root + 4, 12 );
	b->info.build_ms = ms, b->info.layouts = 1u << TBVH_LAYOUT_BVH;
	b->root_ref = r.root[3], b->root_count = r.root[7];
	b->d_pairs.reset(); // walked through its own nodes (trav)
	b->generation = tbvh_next_generation(); // new arrays: a TLAS built over the old ones must notice (tlas_check)
	b->tree_stamp = tbvh_next_generation(); // a new tree: the signed-distance and winding-number tables are stale
}

int tbvh_bvh_destroy( tbvh_bvh b )
{
	if (!b) return TBVH_OK;
	cudaSetDevice( b->ctx->device );
	live_remove( b );
	free_layouts( b );
	delete b; // d_stats frees itself on the device set above
	return TBVH_OK;
}

int tbvh_bvh_info( tbvh_bvh b, tbvh_info* out ) { ARG_CHECK( b && out, "NULL argument" ); *out = b->info; return TBVH_OK; }
int tbvh_set_stats( tbvh_bvh b, int enable ) { ARG_CHECK( b, "NULL handle" ); b->stats = enable; return TBVH_OK; }
int tbvh_get_stats( tbvh_bvh b, uint64_t* steps, uint64_t* tris )
{
	ARG_CHECK( b, "NULL handle" );
	unsigned long long h[2];
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	CUDA_TRY( cudaDeviceSynchronize() );
	CUDA_TRY( cudaMemcpy( h, b->d_stats, 16, cudaMemcpyDeviceToHost ) );
	if (steps) *steps = h[0];
	if (tris) *tris = h[1];
	return TBVH_OK;
}
int tbvh_get_stats_ex( tbvh_bvh b, uint64_t out[4] )
{
	ARG_CHECK( b && out, "NULL argument" );
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	CUDA_TRY( cudaDeviceSynchronize() );
	CUDA_TRY( cudaMemcpy( out, b->d_stats, 32, cudaMemcpyDeviceToHost ) );
	return TBVH_OK;
}

} // extern "C"

// ---- uploads ------------------------------------------------------------------------------------------------

// nv vertices `stride` bytes apart -> rows of a 16-byte-pitch array: the first min( stride, 16 ) bytes of each, so below stride 16
// the w lane of dst is left as it was
int copy_rows( float4* dst, const void* verts, uint32_t stride, size_t nv, int space, cudaStream_t s )
{
	const cudaMemcpyKind kind = space == TBVH_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
	if (stride == 16) CUDA_TRY( cudaMemcpyAsync( dst, verts, nv * 16, kind, s ) );
	else CUDA_TRY( cudaMemcpy2DAsync( dst, 16, verts, stride, stride < 16 ? stride : 16, nv, kind, s ) );
	return TBVH_OK;
}
// vertices -> engine-owned float4 array (xyz of each vertex, w copied when the stride holds it)
static int copy_verts( float4* dst, const void* verts, uint32_t stride, size_t nv, int space, cudaStream_t s )
{
	if (stride != 16) CUDA_TRY( cudaMemsetAsync( dst, 0, nv * 16, s ) );
	return copy_rows( dst, verts, stride, nv, space, s );
}
static int upload_verts( tbvh_bvh b, const void* verts, uint32_t stride, uint32_t prim_count, int space, cudaStream_t s )
{
	ARG_CHECK( verts && stride >= 12 && (stride & 3) == 0 && prim_count > 0, "bad vertex slice" );
	const size_t nv = (size_t)prim_count * 3;
	TRY( b->d_verts.alloc( nv * 16 ) );
	TRY( copy_verts( b->d_verts, verts, stride, nv, space, s ) );
	b->info.prim_count = prim_count;
	return TBVH_OK;
}

// indexed geometry (the `vertices, indices, primCount` overloads, tiny_bvh.h:889-900): the engine keeps its own copy of
// the vertices anyway, so the indices are resolved once, on the device, into the flat 3-vertices-per-triangle array the
// kernels read.  The tree is the one the reference builds with vertIdx set (same fragments, same primIdx numbering).
__global__ void k_gather_verts( const float4* __restrict__ src, const uint32_t* __restrict__ indices, float4* __restrict__ dst, const uint32_t n, const uint32_t vert_count, uint32_t* bad )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint32_t v = indices[i];
	if (v >= vert_count) { atomicAdd( bad, 1u ); dst[i] = make_float4( 0, 0, 0, 0 ); return; }
	dst[i] = src[v];
}
// An indexed refit (tbvh_refit_batch_indexed) reads the moved vertices through the indices kept from the build, as BVH::Refit reads
// them through vertIdx (tiny_bvh.h:3055): one thread per kept index of every indexed mesh of the call.  The indices were checked at
// build time and the vertex count is the build's, so there is no bounds check.  One mesh: its staged new vertices (16-byte pitch),
// its kept indices, the handle's d_verts, its first index in the call's index space, and full = the stride holds w (>= 16), when
// all four lanes are written; below stride 16 w of d_verts stays, as refit_copy leaves it (k_encode writes v.w differences).
struct IxMesh { const float4* src; const uint32_t* idx; float4* dst; uint32_t base, full; };
__global__ void k_refit_gather( const IxMesh* __restrict__ T, const uint32_t K, const uint32_t n )
{
	const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
	if (g >= n) return;
	const IxMesh& m = T[batch_entry<IxMesh, &IxMesh::base>( T, K, g )];
	const uint32_t i = g - m.base;
	const float4 v = m.src[m.idx[i]];
	if (m.full) m.dst[i] = v;
	else m.dst[i] = make_float4( v.x, v.y, v.z, m.dst[i].w );
}
// the gather into dst; indices past vert_count are counted into d_bad.  Synchronises the stream.  keep_idx: NULL, or where the
// device copy of the indices is handed to the caller instead of being freed here
static int gather_verts( float4* dst, const void* verts, uint32_t stride, uint32_t vert_count, const uint32_t* indices, uint32_t prim_count, int space, cudaStream_t s, uint32_t* d_bad,
	DevArray<uint32_t>* keep_idx )
{
	const size_t nv = (size_t)prim_count * 3;
	const cudaMemcpyKind kind = space == TBVH_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
	DevArray<uint32_t> d_idx; // declared before sc: freed after the stream is drained
	Scratch sc( s );
	float4* d_src = 0;
	TRY( sc.alloc( d_src, (size_t)vert_count * 16 ) );
	TRY( d_idx.alloc( nv * 4 ) );
	TRY( copy_verts( d_src, verts, stride, vert_count, space, s ) );
	CUDA_TRY( cudaMemcpyAsync( d_idx, indices, nv * 4, kind, s ) );
	k_gather_verts<<<(unsigned)((nv + 255) / 256), 256, 0, s>>>( d_src, d_idx, dst, (uint32_t)nv, vert_count, d_bad ); LAUNCHED();
	if (keep_idx) *keep_idx = std::move( d_idx );
	return TBVH_OK;
}

// depth of the deepest node (root = 0) of a tree of `words`-word nodes, by iterative DFS; children( n, c ) writes the two children of
// node n to c and says whether the walk descends into them
template <class Children> static uint32_t tree_depth( const uint32_t* nodes, const uint32_t words, Children children )
{
	std::vector<uint2> st;
	st.push_back( make_uint2( 0, 0 ) );
	uint32_t maxd = 0;
	while (!st.empty())
	{
		const uint2 e = st.back();
		st.pop_back();
		if (e.y > maxd) maxd = e.y;
		uint32_t c[2];
		if (children( nodes + (size_t)e.x * words, c )) { st.push_back( make_uint2( c[0], e.y + 1 ) ); st.push_back( make_uint2( c[1], e.y + 1 ) ); }
	}
	return maxd;
}

// true when the 32-byte node array is one tree over every slot but node 1: walked from the root, no child pointer leaves
// [0, used_nodes), node 1 is never reached, no slot is reached twice, and every other slot is reached
static bool slots_form_tree( const uint32_t* nodes, const uint32_t used_nodes )
{
	std::vector<uint8_t> seen( used_nodes, 0 );
	std::vector<uint32_t> st( 1, 0u );
	uint32_t reached = 0;
	while (!st.empty())
	{
		const uint32_t x = st.back();
		st.pop_back();
		if (x >= used_nodes || x == 1 || seen[x]) return false;
		seen[x] = 1, reached++;
		const uint32_t* n = nodes + (size_t)x * 8;
		if (n[7] == 0) st.push_back( n[3] + 1 ), st.push_back( n[3] );
	}
	return reached == used_nodes - (used_nodes > 1 ? 1 : 0);
}

// the shared part of tbvh_upload_bvh / tbvh_upload_bvh_gpu after the argument check: the handle emptied, the vertices, `used_nodes`
// nodes of `node_bytes` each into *d_nodes (room for at least min_nodes) and primIdx copied in.  *hn: the nodes as the host reads
// them (for device-space input, a copy in `host`)
static int upload_tree( tbvh_bvh b, DevArray<float4>& d_nodes, const void* nodes, uint32_t used_nodes, uint32_t node_bytes, uint32_t min_nodes,
	const uint32_t* prim_idx, uint32_t idx_count, const void* verts, uint32_t stride, uint32_t prim_count, int space, std::vector<uint32_t>& host, const uint32_t** hn )
{
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	cudaStream_t s = b->ctx->stream;
	free_layouts( b );
	TRY( upload_verts( b, verts, stride, prim_count, space, s ) );
	const cudaMemcpyKind kind = space == TBVH_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
	const size_t bytes = (size_t)used_nodes * node_bytes;
	TRY( d_nodes.alloc( (size_t)std::max( used_nodes, min_nodes ) * node_bytes ) );
	CUDA_TRY( cudaMemcpyAsync( d_nodes, nodes, bytes, kind, s ) );
	TRY( b->d_prim_idx.alloc( (size_t)idx_count * 4 ) );
	CUDA_TRY( cudaMemcpyAsync( b->d_prim_idx, prim_idx, (size_t)idx_count * 4, kind, s ) );
	*hn = (const uint32_t*)nodes;
	if (space == TBVH_DEVICE)
	{
		host.resize( bytes / 4 );
		CUDA_TRY( cudaMemcpyAsync( host.data(), nodes, bytes, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		*hn = host.data();
	}
	b->info.idx_count = idx_count;
	return TBVH_OK;
}

// the refusals of tbvh_refit / tbvh_refit_layouts / tbvh_refit_batch, in this order
static int refit_check( const char* fn, tbvh_bvh b, const void* verts, uint32_t stride, uint32_t prim_count, bool keep_layouts )
{
	if (!b || !verts) { tbvh_set_error( "%s: NULL argument", fn ); return TBVH_E_ARG; }
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	if (!(b->info.layouts & (1u << TBVH_LAYOUT_BVH)) || !b->d_nodes || b->d_pairs.p) { tbvh_set_error( "%s: no BVH-layout tree on this handle", fn ); return TBVH_E_STATE; }
	if (!b->refittable) { tbvh_set_error( b->d_inst ? "%s: a TLAS is rebuilt, not refitted (tiny_bvh.h:3060)" : "%s: refitting an SBVH (BVH::Refit, tiny_bvh.h:3057)", fn ); return TBVH_E_STATE; }
	if (keep_layouts && (b->info.layouts & (1u << TBVH_LAYOUT_CWBVH)) && !b->cw_keep)
	{ tbvh_set_error( "%s: the CWBVH on this handle was not converted from the resident tree (tbvh_convert)", fn ); return TBVH_E_STATE; }
	if (prim_count != b->info.prim_count || stride < 12 || (stride & 3) != 0) { tbvh_set_error( "%s: the vertex slice must describe the same triangles", fn ); return TBVH_E_ARG; }
	return TBVH_OK;
}

// the new vertices of a refit.  Unlike copy_verts the copy leaves w alone below stride 16 (k_encode writes v.w differences into bvh8Tris)
static int refit_copy( tbvh_bvh b, const void* verts, uint32_t stride, int space )
{
	return copy_rows( b->d_verts, verts, stride, (size_t)b->info.prim_count * 3, space, b->ctx->stream );
}

// the new vertices of the indexed meshes of a refit (meshes[k].vert_count > 0, n kept indices in all): each mesh's vert_count rows
// staged at a 16-byte pitch into the context's buffer, then one k_refit_gather for all of them.  The caller holds c->ix_mutex until
// the stream has run the gather.
static int refit_gather( tbvh_ctx c, const tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, uint64_t n )
{
	cudaStream_t s = c->stream;
	std::vector<IxMesh> T;
	size_t rows = 0;
	for (uint32_t k = 0, base = 0; k < count; k++) if (meshes[k].vert_count)
	{
		T.push_back( IxMesh{ 0, bvhs[k]->d_vert_idx, bvhs[k]->d_verts, base, meshes[k].stride >= 16 ? 1u : 0u } );
		rows += meshes[k].vert_count, base += meshes[k].prim_count * 3;
	}
	const size_t o_rows = (T.size() * sizeof( IxMesh ) + 255) & ~(size_t)255;
	TRY( c->ix_dev.reserve( o_rows + rows * 16 ) );
	float4* at = (float4*)(c->ix_dev + o_rows);
	for (uint32_t k = 0, i = 0; k < count; k++) if (meshes[k].vert_count)
	{
		T[i++].src = at;
		TRY( copy_rows( at, meshes[k].verts, meshes[k].stride, meshes[k].vert_count, space, s ) );
		at += meshes[k].vert_count;
	}
	CUDA_TRY( cudaMemcpyAsync( c->ix_dev, T.data(), T.size() * sizeof( IxMesh ), cudaMemcpyHostToDevice, s ) );
	k_refit_gather<<<(unsigned)((n + 255) / 256), 256, 0, s>>>( (const IxMesh*)c->ix_dev.p, (uint32_t)T.size(), (uint32_t)n ); LAUNCHED();
	return TBVH_OK;
}

// the handle list of a batch call: no NULL handle, one context, no handle twice
static int check_batch_handles( const char* fn, const tbvh_bvh* bvhs, uint32_t count )
{
	for (uint32_t k = 0; k < count; k++)
		if (!bvhs[k] || bvhs[k]->ctx != bvhs[0]->ctx) { tbvh_set_error( "%s: a handle is NULL or lives in another context", fn ); return TBVH_E_ARG; }
	std::vector<tbvh_bvh> sorted( bvhs, bvhs + count );
	std::sort( sorted.begin(), sorted.end() );
	if (std::adjacent_find( sorted.begin(), sorted.end() ) != sorted.end()) { tbvh_set_error( "%s: the same handle twice", fn ); return TBVH_E_ARG; }
	return TBVH_OK;
}

extern "C" {

int tbvh_upload_bvh( tbvh_bvh b, const void* nodes32, uint32_t used_nodes, const uint32_t* prim_idx, uint32_t idx_count,
	const void* verts, uint32_t stride, uint32_t prim_count, int space )
{
	ARG_CHECK( b && nodes32 && prim_idx && used_nodes >= 1 && idx_count >= 1, "bad tree arrays" );
	std::vector<uint32_t> host;
	const uint32_t* hn;
	TRY( upload_tree( b, b->d_nodes, nodes32, used_nodes, 32, 2, prim_idx, idx_count, verts, stride, prim_count, space, host, &hn ) );
	cudaStream_t s = b->ctx->stream;
	b->root_ref = hn[3], b->root_count = hn[7];
	b->info.used_nodes = used_nodes;
	b->info.max_depth = tree_depth( hn, 8, [&]( const uint32_t* n, uint32_t* c ) { c[0] = n[3], c[1] = n[3] + 1; return n[7] == 0 && n[3] + 1 < used_nodes; } );
	memcpy( b->info.aabb_min, hn, 12 ), memcpy( b->info.aabb_max, hn + 4, 12 );
	TRY( make_leaf_tris( b, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	b->info.layouts = 1u << TBVH_LAYOUT_BVH;
	b->stray_slots = !slots_form_tree( hn, used_nodes );
	return TBVH_OK;
}

int tbvh_upload_bvh_gpu( tbvh_bvh b, const void* nodes64, uint32_t used_nodes, const uint32_t* prim_idx, uint32_t idx_count,
	const void* verts, uint32_t stride, uint32_t prim_count, int space )
{
	ARG_CHECK( b && nodes64 && prim_idx && used_nodes >= 1 && idx_count >= 1, "bad tree arrays" );
	std::vector<uint32_t> host;
	const uint32_t* hn;
	TRY( upload_tree( b, b->d_nodes_gpu, nodes64, used_nodes, 64, 1, prim_idx, idx_count, verts, stride, prim_count, space, host, &hn ) );
	cudaStream_t s = b->ctx->stream;
	b->info.used_nodes_gpu = used_nodes;
	b->info.max_depth = tree_depth( hn, 16, [&]( const uint32_t* n, uint32_t* c ) { c[0] = n[3], c[1] = n[7]; return n[11] == 0 && n[3] < used_nodes && n[7] < used_nodes; } );
	// root as a child record: a leaf root keeps (firstTri, triCount); an interior root is pair 0 (pairs are indexed by 2*node)
	if (hn[11] > 0) b->root_ref = hn[15], b->root_count = hn[11]; else b->root_ref = 0, b->root_count = 0;
	TRY( bvh_gpu_to_bvh( b, used_nodes, s ) );
	TRY( make_leaf_tris( b, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	b->info.layouts = 1u << TBVH_LAYOUT_BVH_GPU;
	return TBVH_OK;
}

int tbvh_upload_cwbvh( tbvh_bvh b, const void* bvh8_data, uint32_t used_blocks, const void* bvh8_tris, uint32_t tri_count, int space )
{
	ARG_CHECK( b && bvh8_data && bvh8_tris && used_blocks >= 5 && tri_count >= 1, "bad CWBVH arrays" );
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	cudaStream_t s = b->ctx->stream;
	const cudaMemcpyKind kind = space == TBVH_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
	ARG_CHECK( used_blocks % 5 == 0, "usedBlocks must be a multiple of 5 (80-byte nodes)" );
	drop_cwbvh( b ); // the new arrays come without a kept collapse: tbvh_refit_layouts refuses them
	auto body = [&]() -> int
	{
		TRY( b->d_cw_nodes.alloc( (size_t)used_blocks * 16 ) );
		TRY( b->d_cw_tris.alloc( (size_t)tri_count * 48 ) );
		CUDA_TRY( cudaMemcpyAsync( b->d_cw_nodes, bvh8_data, (size_t)used_blocks * 16, kind, s ) );
		CUDA_TRY( cudaMemcpyAsync( b->d_cw_tris, bvh8_tris, (size_t)tri_count * 48, kind, s ) );
		b->info.used_blocks = used_blocks, b->info.cwbvh_tri_count = tri_count;
		return cw_make_trav( &b, 1, s ); // the traversal nodes the kernels read + the pending bound of the wide tree (synchronises the stream)
	};
	const int rc = body();
	if (rc != TBVH_OK) { cudaStreamSynchronize( s ); drop_cwbvh( b ); } // the copies may still be writing the arrays
	else b->info.layouts |= 1u << TBVH_LAYOUT_CWBVH;
	return rc;
}

// ---- BVH::SAHCost (tiny_bvh.h:1889-1897) over a downloaded node array: host recursion in the reference's own order
__attribute__( (optimize( "fp-contract=off" )) ) static float sah_rec( const float* nodes /* 8 words per node */, const uint32_t i, const float c_trav, const float c_int )
{
	const float* n = nodes + (size_t)i * 8;
	uint32_t leftFirst, triCount;
	memcpy( &leftFirst, n + 3, 4 ), memcpy( &triCount, n + 7, 4 );
	const float ex = n[4] - n[0], ey = n[5] - n[1], ez = n[6] - n[2];
	const float sa = fmaf( ez, ex, fmaf( ey, ex, ey * ez ) ); // BVHBase::SA :8477 in the reference build's pairing
	if (triCount > 0) return c_int * sa * triCount;
	return c_trav * sa + sah_rec( nodes, leftFirst, c_trav, c_int ) + sah_rec( nodes, leftFirst + 1, c_trav, c_int );
}
__attribute__( (optimize( "fp-contract=off" )) ) int tbvh_sah_cost_nodes( const void* nodes32, uint32_t used_nodes, float c_trav, float c_int, float* out )
{
	ARG_CHECK( nodes32 && used_nodes >= 1 && out, "bad arguments" );
	const float* n = (const float*)nodes32;
	const float cost = sah_rec( n, 0, c_trav, c_int );
	const float ex = n[4] - n[0], ey = n[5] - n[1], ez = n[6] - n[2];
	*out = cost / fmaf( ez, ex, fmaf( ey, ex, ey * ez ) ); // the root divides by its own area (:1896)
	return TBVH_OK;
}
int tbvh_sah_cost( tbvh_bvh b, float c_trav, float c_int, float* out )
{
	ARG_CHECK( b && out, "NULL argument" );
	if (!(b->info.layouts & (1u << TBVH_LAYOUT_BVH)) || !b->d_nodes) { tbvh_set_error( "tbvh_sah_cost: no BVH-layout tree on this handle" ); return TBVH_E_STATE; }
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	std::vector<float> nodes( (size_t)b->info.used_nodes * 8 );
	CUDA_TRY( cudaMemcpy( nodes.data(), b->d_nodes, nodes.size() * 4, cudaMemcpyDeviceToHost ) );
	return tbvh_sah_cost_nodes( nodes.data(), b->info.used_nodes, c_trav, c_int, out );
}

// ---- tbvh_optimize: the checks and the handle's bookkeeping around optimize.cu's rounds
int tbvh_optimize( tbvh_bvh b, uint32_t max_rounds, float c_trav, float c_int, uint32_t* rounds, float* sah )
{
	ARG_CHECK( b, "NULL handle" );
	ARG_CHECK( max_rounds > 0, "max_rounds must be at least 1" );
	ARG_CHECK( std::isfinite( c_trav ) && std::isfinite( c_int ) && c_trav > 0.0f && c_int > 0.0f, "c_trav and c_int must be finite and > 0" );
	if (b->d_inst) { tbvh_set_error( "tbvh_optimize: a TLAS is rebuilt per frame, not optimised" ); return TBVH_E_STATE; }
	if (!(b->info.layouts & (1u << TBVH_LAYOUT_BVH)) || !b->d_nodes) { tbvh_set_error( "tbvh_optimize: no BVH-layout tree on this handle" ); return TBVH_E_STATE; }
	if (b->stray_slots) { tbvh_set_error( "tbvh_optimize: the uploaded node array holds slots outside the tree (every slot but node 1 must belong to it)" ); return TBVH_E_STATE; }
	if (b->info.max_depth > 255) { tbvh_set_error( "tbvh_optimize: depth %u exceeds the search's 255 levels", b->info.max_depth ); return TBVH_E_LIMIT; }
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	uint32_t kept = 0, used = 0, depth = 0;
	float cost = 0.0f, ms = 0.0f;
	DevArray<float4> out;
	if (b->info.used_nodes >= 5 && b->root_count == 0) // a leaf root, or a root over two leaves, offers no move
	{
		const int rc = optimize_tree( b, max_rounds, c_trav, c_int, out, &used, &depth, &kept, &cost, &ms );
		if (rc != TBVH_OK) { cudaStreamSynchronize( b->ctx->stream ); free_layouts( b ); cudaGetLastError(); return rc; }
	}
	if (kept == 0)
	{
		if (rounds) *rounds = 0;
		return sah ? tbvh_sah_cost( b, c_trav, c_int, sah ) : TBVH_OK;
	}
	BuiltTree r = { {}, used, b->info.idx_count, depth };
	if (cudaMemcpy( r.root, out, 32, cudaMemcpyDeviceToHost ) != cudaSuccess)
	{
		tbvh_set_error( "tbvh_optimize: %s", cudaGetErrorString( cudaGetLastError() ) );
		free_layouts( b );
		return TBVH_E_CUDA;
	}
	drop_bvh_gpu( b );
	drop_cwbvh( b );
	b->d_nodes = std::move( out );
	install_tree( b, r, ms ); // d_leaf_tris depends on primIdx and the vertices alone: it stays
	if (rounds) *rounds = kept;
	if (sah) *sah = cost;
	return TBVH_OK;
}

// ---- BLASInstance::Update on the host: the arithmetic of instance_update.cuh, which the device kernel runs too (host code, so gcc's
// contraction is switched off for the function it is inlined into)
UPD_HOST_ATTR static void upd_instance_host( const float* T, float* iT, float* aabbMin, float* aabbMax, const float* bmin, const float* bmax )
{
	upd_instance( T, iT, aabbMin, aabbMax, bmin, bmax );
}
int tbvh_instance_update_box( void* instance, const float* bmin, const float* bmax )
{
	ARG_CHECK( instance && bmin && bmax, "NULL argument" );
	float T[16], iT[16], mn[3], mx[3];
	memcpy( T, instance, 64 );
	upd_instance_host( T, iT, mn, mx, bmin, bmax );
	memcpy( (char*)instance + 64, iT, 64 ), memcpy( (char*)instance + 128, mn, 12 ), memcpy( (char*)instance + 144, mx, 12 );
	return TBVH_OK;
}
int tbvh_instance_update( void* instance, tbvh_bvh blas )
{
	ARG_CHECK( instance && blas, "NULL argument" );
	if (!(blas->info.layouts & (1u << TBVH_LAYOUT_BVH))) { tbvh_set_error( "tbvh_instance_update: the BLAS holds no tree" ); return TBVH_E_STATE; }
	return tbvh_instance_update_box( instance, blas->info.aabb_min, blas->info.aabb_max );
}

extern "C++" int tlas_blas_table( const tbvh_bvh t, const tbvh_bvh* blasses, const uint32_t blas_count, TlasBlasTable& T )
{
	T.refs.assign( blas_count, BlasRef{} );
	T.layouts = (1u << TBVH_LAYOUT_BVH) | (1u << TBVH_LAYOUT_CWBVH), T.deep_blas = 0, T.deep_depth = 0;
	for (uint32_t k = 0; k < blas_count; k++)
	{
		const tbvh_bvh b = blasses[k];
		ARG_CHECK( b && b != t && b->ctx == t->ctx, "TLAS: a BLAS handle is NULL or lives in another context" );
		bool has_bvh = (b->info.layouts & (1u << TBVH_LAYOUT_BVH)) && b->trav() && b->d_leaf_tris;
		const bool has_cw = b->d_cw_trav && b->d_cw_tris;
		if (b->d_inst || (!has_bvh && !has_cw))
		{ tbvh_set_error( "TLAS: BLAS %u holds no triangle tree (IntersectTLAS walks LAYOUT_BVH BLASses, tiny_bvh.h:3341; traverse_tlas.cl CWBVH ones)", k ); return TBVH_E_STATE; }
		if (has_bvh && b->info.max_depth + 1 > TBVH_STACK)
		{
			// the two-level kernel walks a BVH2 BLAS with a TBVH_STACK-entry stack; the CWBVH walk does not use it, so a BLAS that
			// also holds its CWBVH stays usable through that layout, and a LAYOUT_BVH walk of the TLAS is refused (tlas_check)
			if (!has_cw) { tbvh_set_error( "TLAS: BLAS %u has depth %u, the two-level kernel walks a BLAS with a %d-entry stack", k, b->info.max_depth, TBVH_STACK ); return TBVH_E_LIMIT; }
			if (!T.deep_blas) T.deep_blas = k + 1, T.deep_depth = b->info.max_depth;
			has_bvh = false;
		}
		if (has_cw && b->cw_pending == 0xffffffffu) { tbvh_set_error( "TLAS: the wide tree of BLAS %u has a cycle in its inner-child links", k ); return TBVH_E_ARG; }
		if (has_cw && b->cw_pending > 128) { tbvh_set_error( "TLAS: the wide tree of BLAS %u can leave %u node groups pending (128 per ray, tiny_bvh.h:7048)", k, b->cw_pending ); return TBVH_E_LIMIT; }
		T.refs[k].trav = has_bvh ? b->trav() : 0, T.refs[k].tris = has_bvh ? b->d_leaf_tris.get() : 0, T.refs[k].root_ref = b->root_ref, T.refs[k].root_count = b->root_count, T.refs[k].pad1 = 0;
		T.refs[k].cw_nodes = has_cw ? b->d_cw_trav.get() : 0, T.refs[k].cw_tris = has_cw ? b->d_cw_tris.get() : 0, T.refs[k].cw_rd_limit = has_cw ? b->cw_rd_limit : -1.0f;
		T.layouts &= (has_bvh ? 1u << TBVH_LAYOUT_BVH : 0u) | (has_cw ? 1u << TBVH_LAYOUT_CWBVH : 0u);
	}
	return TBVH_OK;
}

// The refusals of both TLAS builds, before the handle is touched: the arguments, the BLAS list (update: every BLAS's root box must be
// known, tbvh_instance_update's refusal) and, for host records, every blasIdx.
static int tlas_refusals( tbvh_bvh t, const void* instances, uint32_t inst_stride, uint32_t inst_count, bool host, const tbvh_bvh* blasses, uint32_t blas_count,
	bool update, TlasBlasTable& B )
{
	ARG_CHECK( t && instances && blasses && inst_count > 0 && blas_count > 0 && inst_stride >= 160, "bad TLAS arguments" );
	CUDA_TRY( cudaSetDevice( t->ctx->device ) );
	TRY( tlas_blas_table( t, blasses, blas_count, B ) );
	if (update) for (uint32_t k = 0; k < blas_count; k++) if (!(blasses[k]->info.layouts & (1u << TBVH_LAYOUT_BVH)))
	{ tbvh_set_error( "TLAS: BLAS %u holds no BVH-layout tree, so its root box is not known (tbvh_instance_update)", k ); return TBVH_E_STATE; }
	if (host) for (uint32_t i = 0; i < inst_count; i++)
	{
		uint32_t blasIdx;
		memcpy( &blasIdx, (const char*)instances + (size_t)i * inst_stride + 140, 4 );
		ARG_CHECK( blasIdx < blas_count, "TLAS: an instance names a BLAS past blas_count" );
	}
	return TBVH_OK;
}

// the end of both TLAS builds: the reference builder over t->d_aabbs, and the BLAS generations the device table's addresses belong to.
// A tree too deep for the walk's stack is not installed.
static int tlas_finish( tbvh_bvh t, const uint32_t inst_count, const tbvh_bvh* blasses, const uint32_t blas_count, const TlasBlasTable& B, float c_trav, float c_int )
{
	t->info.prim_count = inst_count, t->inst_count = inst_count, t->blas_count = blas_count, t->tlas_blas_layouts = B.layouts;
	t->tlas_deep_blas = B.deep_blas, t->tlas_deep_depth = B.deep_depth;
	BuiltTree r;
	float ms = 0;
	TRY( build_sah_launch( &t, 1, c_trav, c_int, TBVH_BUILD_REFERENCE, &r, &ms ) ); // "Build(); // or BuildAVX, for large TLAS." :2258
	if (r.max_depth + 1 > TBVH_STACK) { tbvh_set_error( "TLAS depth %u exceeds the %d-entry stack of IntersectTLAS (tiny_bvh.h:3308)", r.max_depth, TBVH_STACK ); return TBVH_E_LIMIT; }
	install_tree( t, r, ms );
	t->refittable = false; // "do not refit a TLAS, use Build(..)" :3060
	for (uint32_t k = 0; k < blas_count; k++) t->links.push_back( BlasLink{ blasses[k], blasses[k]->generation } );
	return TBVH_OK;
}

// the failure rule of both TLAS builds past their refusals: the stream drained, the handle emptied, and the error this call's alone
static int tlas_failed( tbvh_bvh t, const int rc )
{
	cudaStreamSynchronize( t->ctx->stream );
	free_layouts( t );
	cudaGetLastError();
	return rc;
}

// BVH::Build( BLASInstance*, instCount, BVHBase**, blasCount ) tiny_bvh.h:2221 in its "blasses == 0" mode (:2245): the instances
// arrive Update()d - inverse transform and world-space box filled in - and the TLAS is the reference builder's tree over the boxes
int tbvh_build_tlas( tbvh_bvh t, const void* instances, uint32_t inst_stride, uint32_t inst_count, const tbvh_bvh* blasses, uint32_t blas_count, float c_trav, float c_int )
{
	TlasBlasTable B;
	TRY( tlas_refusals( t, instances, inst_stride, inst_count, true, blasses, blas_count, false, B ) );
	std::vector<float4> boxes( (size_t)inst_count * 2 );
	std::vector<TlasInst> inst( inst_count );
	for (uint32_t i = 0; i < inst_count; i++)
	{
		// BLASInstance :1443: transform @0, invTransform @64, aabbMin @128, blasIdx @140, aabbMax @144, mask @156
		const char* r = (const char*)instances + (size_t)i * inst_stride;
		memcpy( inst[i].inv, r + 64, 64 );
		memcpy( &inst[i].blasIdx, r + 140, 4 ), memcpy( &inst[i].mask, r + 156, 4 );
		inst[i].pad0 = inst[i].pad1 = 0;
		float mn[3], mx[3];
		memcpy( mn, r + 128, 12 ), memcpy( mx, r + 144, 12 );
		boxes[(size_t)i * 2] = make_float4( mn[0], mn[1], mn[2], 0 ), boxes[(size_t)i * 2 + 1] = make_float4( mx[0], mx[1], mx[2], 0 );
	}
	const std::vector<BlasRef>& refs = B.refs;
	free_layouts( t );
	cudaStream_t s = t->ctx->stream;
	auto body = [&]() -> int
	{
		TRY( t->d_aabbs.alloc( boxes.size() * 16 ) );
		TRY( t->d_inst.alloc( inst.size() * sizeof( TlasInst ) ) );
		TRY( t->d_blas.alloc( refs.size() * sizeof( BlasRef ) ) );
		CUDA_TRY( cudaMemcpyAsync( t->d_aabbs, boxes.data(), boxes.size() * 16, cudaMemcpyHostToDevice, s ) );
		CUDA_TRY( cudaMemcpyAsync( t->d_inst, inst.data(), inst.size() * sizeof( TlasInst ), cudaMemcpyHostToDevice, s ) );
		CUDA_TRY( cudaMemcpyAsync( t->d_blas, refs.data(), refs.size() * sizeof( BlasRef ), cudaMemcpyHostToDevice, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) ); // the host vectors go out of scope
		return tlas_finish( t, inst_count, blasses, blas_count, B, c_trav, c_int );
	};
	const int rc = body();
	return rc == TBVH_OK ? rc : tlas_failed( t, rc );
}

// BVH::Build( BLASInstance*, instCount, BVHBase**, blasCount ) tiny_bvh.h:2221 with the BLAS list given: every instance is Update()d
// (:2245-2250) by k_instance_update, which also writes the TlasInst entries and the builder's boxes, so no host loop walks the records.
int tbvh_build_tlas_update( tbvh_bvh t, void* instances, uint32_t inst_stride, uint32_t inst_count, int space, const tbvh_bvh* blasses, uint32_t blas_count,
	float c_trav, float c_int )
{
	ARG_CHECK( space == TBVH_HOST || space == TBVH_DEVICE, "unknown space" );
	if (space == TBVH_DEVICE) ARG_CHECK( ((uintptr_t)instances & 15) == 0 && (inst_stride & 15) == 0, "device records: the pointer and the stride must be multiples of 16" );
	else ARG_CHECK( (inst_stride & 3) == 0, "host records: the stride must be a multiple of 4" );
	TlasBlasTable B;
	TRY( tlas_refusals( t, instances, inst_stride, inst_count, space == TBVH_HOST, blasses, blas_count, true, B ) );
	// the device table: BlasRef[blas_count], then the root box of every BLAS (2 float4), then the flag word of the kernel
	const size_t box_at = (size_t)blas_count * sizeof( BlasRef ), flag_at = box_at + (size_t)blas_count * 32, table_bytes = flag_at + 16;
	std::vector<char> table( table_bytes, 0 );
	memcpy( table.data(), B.refs.data(), box_at );
	for (uint32_t k = 0; k < blas_count; k++)
		memcpy( table.data() + box_at + (size_t)k * 32, blasses[k]->info.aabb_min, 12 ), memcpy( table.data() + box_at + (size_t)k * 32 + 16, blasses[k]->info.aabb_max, 12 );
	// a frame of an animation rebuilds the TLAS it built last frame: same counts, so the instance boxes, the TlasInst and BLAS tables
	// and the staging of host records are kept; the tree itself is the builder's to allocate
	const bool reuse = t->d_inst && t->d_aabbs && t->d_blas && t->inst_count == inst_count && t->blas_count == blas_count && t->blas_table_bytes == table_bytes;
	DevArray<float4> aabbs;
	DevArray<TlasInst> inst;
	DevArray<char> blas, stage;
	if (reuse) aabbs = std::move( t->d_aabbs ), inst = std::move( t->d_inst ), blas = std::move( t->d_blas ), stage = std::move( t->d_inst_stage );
	free_layouts( t );
	t->d_aabbs = std::move( aabbs ), t->d_inst = std::move( inst ), t->d_blas = std::move( blas ), t->d_inst_stage = std::move( stage ), t->blas_table_bytes = table_bytes;
	cudaStream_t s = t->ctx->stream;
	auto body = [&]() -> int
	{
		Scratch sc( s );
		if (!reuse)
		{
			TRY( t->d_aabbs.alloc( (size_t)inst_count * 32 ) );
			TRY( t->d_inst.alloc( (size_t)inst_count * sizeof( TlasInst ) ) );
			TRY( t->d_blas.alloc( table_bytes ) );
		}
		if (space == TBVH_HOST && !t->d_inst_stage) TRY( t->d_inst_stage.alloc( (size_t)inst_count * 160 ) );
		TRY( sc.events() );
		CUDA_TRY( cudaMemcpyAsync( t->d_blas, table.data(), table_bytes, cudaMemcpyHostToDevice, s ) );
		// host records: bytes 0..159 in, one strided copy; bytes 64..159 (invTransform .. mask) back, one strided copy
		if (space == TBVH_HOST) CUDA_TRY( cudaMemcpy2DAsync( t->d_inst_stage, 160, instances, inst_stride, 160, inst_count, cudaMemcpyHostToDevice, s ) );
		CUDA_TRY( cudaEventRecord( sc.e0, s ) );
		TRY( instance_update_launch( space == TBVH_HOST ? (void*)t->d_inst_stage : instances, space == TBVH_HOST ? 160u : inst_stride, inst_count,
			(const float4*)(t->d_blas + box_at), blas_count, t->d_inst, t->d_aabbs, (uint32_t*)(t->d_blas + flag_at), s ) );
		CUDA_TRY( cudaEventRecord( sc.e1, s ) );
		if (space == TBVH_HOST) CUDA_TRY( cudaMemcpy2DAsync( (char*)instances + 64, inst_stride, t->d_inst_stage + 64, 160, 96, inst_count, cudaMemcpyDeviceToHost, s ) );
		uint32_t bad_blas = 0;
		CUDA_TRY( cudaMemcpyAsync( &bad_blas, t->d_blas + flag_at, 4, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) ); // the call's one synchronisation outside the builder: `table` and `bad_blas` are on this frame
		if (bad_blas) { tbvh_set_error( "tbvh_build_tlas_update: an instance names a BLAS past blas_count" ); return TBVH_E_ARG; }
		float update_ms = 0;
		CUDA_TRY( cudaEventElapsedTime( &update_ms, sc.e0, sc.e1 ) );
		TRY( tlas_finish( t, inst_count, blasses, blas_count, B, c_trav, c_int ) );
		t->info.build_ms += update_ms;
		return TBVH_OK;
	};
	const int rc = body();
	return rc == TBVH_OK ? rc : tlas_failed( t, rc );
}

// Many trees, one refit (include/tinybvh_b200.h): tbvh_refit_batch, and with `indexed` tbvh_refit_batch_indexed, whose meshes with a
// vert_count are the moved vertices of an indexed build; tbvh_refit and tbvh_refit_layouts are count = 1.  Refit validation is host-side
// only: every refusal comes before any handle or vertex array is touched, then the vertices are copied (indexed meshes: gathered) and
// the trees refitted together.
static int refit_batch( const char* fn, tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, int keep_layouts, bool indexed )
{
	if (!(bvhs && meshes && count > 0)) { tbvh_set_error( "%s: no meshes", fn ); return TBVH_E_ARG; }
	if (space != TBVH_HOST && space != TBVH_DEVICE) { tbvh_set_error( "%s: unknown space", fn ); return TBVH_E_ARG; }
	if (keep_layouts != 0 && keep_layouts != 1) { tbvh_set_error( "%s: keep_layouts is 0 or 1", fn ); return TBVH_E_ARG; }
	TRY( check_batch_handles( fn, bvhs, count ) );
	uint64_t nodes = 0, refs = 0, split = 0, wide = 0, ix = 0;
	for (uint32_t k = 0; k < count; k++)
	{
		const tbvh_mesh& m = meshes[k];
		if (!indexed && (m.indices || m.vert_count)) { tbvh_set_error( "%s: mesh %u: a refit takes a flat vertex slice (indices NULL, vert_count 0)", fn, k ); return TBVH_E_ARG; }
		if (m.indices) { tbvh_set_error( "%s: mesh %u: an indexed refit reads the indices kept from the build (indices NULL)", fn, k ); return TBVH_E_ARG; }
		TRY( refit_check( fn, bvhs[k], m.verts, m.stride, m.prim_count, keep_layouts != 0 ) );
		if (m.vert_count)
		{
			const tbvh_bvh b = bvhs[k];
			if (!b->d_vert_idx) { tbvh_set_error( "%s: mesh %u: the tree was not built from indexed geometry by a refittable builder, so it keeps no indices", fn, k ); return TBVH_E_STATE; }
			if (m.vert_count != b->vert_count) { tbvh_set_error( "%s: mesh %u: %u vertices, the tree was built from %u", fn, k, m.vert_count, b->vert_count ); return TBVH_E_ARG; }
			ix += (uint64_t)m.prim_count * 3;
		}
		uint32_t t = 0, w = 0;
		if (keep_layouts) cw_keep_sizes( bvhs[k], &t, &w );
		nodes += bvhs[k]->info.used_nodes, refs += bvhs[k]->info.idx_count, split += t, wide += w;
	}
	if (std::max( std::max( std::max( nodes, refs ), std::max( split, wide ) ), ix ) > TBVH_REFIT_BATCH_MAX_NODES)
	{
		tbvh_set_error( "%s: %llu BVH2 nodes, %llu primitive references, %llu split-tree and %llu wide nodes, %llu vertex indices in one batch (at most %u each)", fn,
			(unsigned long long)nodes, (unsigned long long)refs, (unsigned long long)split, (unsigned long long)wide, (unsigned long long)ix, (unsigned)TBVH_REFIT_BATCH_MAX_NODES );
		return TBVH_E_LIMIT;
	}
	const tbvh_ctx ctx = bvhs[0]->ctx;
	CUDA_TRY( cudaSetDevice( ctx->device ) );
	std::unique_lock<std::mutex> staging( ctx->ix_mutex, std::defer_lock );
	if (ix) staging.lock(); // released after refit_trees has synchronised the stream, so the gather has read the staged vertices
	auto copies = [&]() -> int
	{
		for (uint32_t k = 0; k < count; k++) if (!meshes[k].vert_count) TRY( refit_copy( bvhs[k], meshes[k].verts, meshes[k].stride, space ) );
		if (ix) TRY( refit_gather( ctx, bvhs, meshes, count, space, ix ) );
		return TBVH_OK;
	};
	const int rc = copies();
	if (rc != TBVH_OK) { cudaStreamSynchronize( ctx->stream ); for (uint32_t j = 0; j < count; j++) drop_bvh_gpu( bvhs[j] ), drop_cwbvh( bvhs[j] ); return rc; }
	return refit_trees( bvhs, count, keep_layouts != 0, ctx->stream );
}

// BVH::Refit (tiny_bvh.h:3055): same topology, new vertex positions; derived layouts are dropped (convert_cwbvh.cu refit_trees)
int tbvh_refit( tbvh_bvh b, const void* verts, uint32_t stride, uint32_t prim_count, int space )
{
	const tbvh_mesh m{ verts, stride, 0, 0, prim_count };
	return refit_batch( __func__, &b, &m, 1, space, 0, false );
}

// BVH::Refit, then every derived layout brought up to date in place (include/tinybvh_b200.h)
int tbvh_refit_layouts( tbvh_bvh b, const void* verts, uint32_t stride, uint32_t prim_count, int space )
{
	const tbvh_mesh m{ verts, stride, 0, 0, prim_count };
	return refit_batch( __func__, &b, &m, 1, space, 1, false );
}

int tbvh_refit_batch( tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, int keep_layouts )
{
	return refit_batch( __func__, bvhs, meshes, count, space, keep_layouts, false );
}

// Many trees, one refit, indexed meshes through their kept indices (include/tinybvh_b200.h)
int tbvh_refit_batch_indexed( tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, int keep_layouts )
{
	return refit_batch( __func__, bvhs, meshes, count, space, keep_layouts, true );
}

// The part of build_batch up to the build.  Every refusal comes before any handle is touched, the vertex staging included: each
// mesh's vertices go into a fresh array first, and only when every index has been found in range do the handles drop their old arrays
// and adopt the new ones.  The triangle counts are checked against the limits before any index or vertex is read.  hq: the SBVH
// builder's node space must fit too.  Only a call with indexed meshes waits for the device here: flat ones are copied and no more.
static int batch_stage( const char* fn, tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, bool hq )
{
	if (space != TBVH_HOST && space != TBVH_DEVICE) { tbvh_set_error( "%s: unknown space", fn ); return TBVH_E_ARG; }
	TRY( check_batch_handles( fn, bvhs, count ) );
	uint64_t total = 0;
	for (uint32_t k = 0; k < count; k++)
	{
		const tbvh_mesh& m = meshes[k];
		if (!(m.verts && m.stride >= 12 && (m.stride & 3) == 0 && m.prim_count > 0 && (!m.indices || m.vert_count > 0))) { tbvh_set_error( "%s: mesh %u: bad vertex slice", fn, k ); return TBVH_E_ARG; }
		total += m.prim_count;
	}
	if (total > TBVH_BATCH_MAX_PRIMS) { tbvh_set_error( "%s: %llu triangles in one batch (at most %u)", fn, (unsigned long long)total, (unsigned)TBVH_BATCH_MAX_PRIMS ); return TBVH_E_LIMIT; }
	if (hq && 3 * total + 2 > TBVH_BATCH_HQ_MAX_NODES)
	{ tbvh_set_error( "%s: %llu temporary SBVH nodes in one batch (at most %u)", fn, (unsigned long long)(3 * total + 2), (unsigned)TBVH_BATCH_HQ_MAX_NODES ); return TBVH_E_LIMIT; }
	bool indexed = false;
	for (uint32_t k = 0; k < count; k++)
	{
		const tbvh_mesh& m = meshes[k];
		indexed |= m.indices != 0;
		if (m.indices && space == TBVH_HOST)
			for (size_t i = 0; i < (size_t)m.prim_count * 3; i++)
				if (m.indices[i] >= m.vert_count) { tbvh_set_error( "%s: mesh %u: index %u points past the %u vertices", fn, k, m.indices[i], m.vert_count ); return TBVH_E_ARG; }
	}
	const tbvh_ctx ctx = bvhs[0]->ctx;
	CUDA_TRY( cudaSetDevice( ctx->device ) );
	cudaStream_t s = ctx->stream;
	std::vector<DevArray<float4>> staged( count );
	std::vector<DevArray<uint32_t>> staged_idx( count ); // indexed meshes of a refittable batch: the indices the handle keeps
	DevArray<uint32_t> d_bad;
	auto stage = [&]() -> int
	{
		if (indexed)
		{
			TRY( d_bad.alloc( 4 ) );
			CUDA_TRY( cudaMemsetAsync( d_bad, 0, 4, s ) );
		}
		for (uint32_t k = 0; k < count; k++)
		{
			const tbvh_mesh& m = meshes[k];
			TRY( staged[k].alloc( (size_t)m.prim_count * 3 * 16 ) );
			if (m.indices) TRY( gather_verts( staged[k], m.verts, m.stride, m.vert_count, m.indices, m.prim_count, space, s, d_bad, hq ? 0 : &staged_idx[k] ) );
			else TRY( copy_verts( staged[k], m.verts, m.stride, (size_t)m.prim_count * 3, space, s ) );
		}
		if (!indexed) return TBVH_OK;
		uint32_t bad = 0;
		CUDA_TRY( cudaMemcpyAsync( &bad, d_bad, 4, cudaMemcpyDeviceToHost, s ) );
		CUDA_TRY( cudaStreamSynchronize( s ) );
		if (bad) { tbvh_set_error( "%s: %u indices point past their mesh's vertices", fn, bad ); return TBVH_E_ARG; }
		return TBVH_OK;
	};
	const int rc = stage();
	if (rc != TBVH_OK) { cudaStreamSynchronize( s ); return rc; } // the staged arrays go once the copies into them are done
	for (uint32_t k = 0; k < count; k++)
	{
		const tbvh_bvh b = bvhs[k];
		free_layouts( b );
		b->info.prim_count = meshes[k].prim_count, b->vert_count = staged_idx[k] ? meshes[k].vert_count : 0;
		b->d_verts = std::move( staged[k] ), b->d_vert_idx = std::move( staged_idx[k] );
	}
	return TBVH_OK;
}

// Many meshes, one build (include/tinybvh_b200.h): tbvh_build_batch and tbvh_build_batch_hq; tbvh_build_flavour and tbvh_build_indexed
// are count = 1.  fn: the entry point the error texts name.  A failed build leaves each handle of the call empty.
static int build_batch( const char* fn, tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, float c_trav, float c_int, int flavour )
{
	if (!(bvhs && meshes && count > 0)) { tbvh_set_error( "%s: no meshes", fn ); return TBVH_E_ARG; }
	if (flavour != TBVH_BUILD_REFERENCE && flavour != TBVH_BUILD_AVX && flavour != TBVH_BUILD_HQ && flavour != TBVH_BUILD_PLOC) { tbvh_set_error( "%s: unknown builder flavour", fn ); return TBVH_E_ARG; }
	const bool hq = flavour == TBVH_BUILD_HQ;
	TRY( batch_stage( fn, bvhs, meshes, count, space, hq ) );
	std::vector<BuiltTree> built( count );
	float ms = 0;
	const int rc = hq ? build_hq_launch( bvhs, count, c_trav, c_int, built.data(), &ms )
		: flavour == TBVH_BUILD_PLOC ? build_ploc_launch( bvhs, count, c_trav, c_int, built.data(), &ms )
		: build_sah_launch( bvhs, count, c_trav, c_int, flavour, built.data(), &ms );
	for (uint32_t k = 0; k < count; k++)
	{
		if (rc != TBVH_OK) free_layouts( bvhs[k] );
		else install_tree( bvhs[k], built[k], ms ), bvhs[k]->refittable = !hq; // "can't refit an SBVH" (:3027)
	}
	return rc;
}

int tbvh_build_batch( tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, float c_trav, float c_int, int flavour )
{
	ARG_CHECK( bvhs && meshes && count > 0, "no meshes" );
	if (flavour == TBVH_BUILD_HQ) { tbvh_set_error( "tbvh_build_batch: SBVH (BuildHQ) batches are built by tbvh_build_batch_hq" ); return TBVH_E_UNSUPPORTED; }
	return build_batch( __func__, bvhs, meshes, count, space, c_trav, c_int, flavour );
}

int tbvh_build_batch_hq( tbvh_bvh* bvhs, const tbvh_mesh* meshes, uint32_t count, int space, float c_trav, float c_int )
{
	return build_batch( __func__, bvhs, meshes, count, space, c_trav, c_int, TBVH_BUILD_HQ );
}

int tbvh_build_flavour( tbvh_bvh b, const void* verts, uint32_t stride, uint32_t prim_count, int space, float c_trav, float c_int, int flavour )
{
	const tbvh_mesh m{ verts, stride, 0, 0, prim_count };
	return build_batch( __func__, &b, &m, 1, space, c_trav, c_int, flavour );
}

int tbvh_build_indexed( tbvh_bvh b, const void* verts, uint32_t stride, uint32_t vert_count, const uint32_t* indices, uint32_t prim_count, int space,
	float c_trav, float c_int, int flavour )
{
	ARG_CHECK( indices, "indices == NULL" ); // a mesh record without indices is a flat one
	const tbvh_mesh m{ verts, stride, vert_count, indices, prim_count };
	return build_batch( __func__, &b, &m, 1, space, c_trav, c_int, flavour );
}

int tbvh_build( tbvh_bvh b, const void* verts, uint32_t stride, uint32_t prim_count, int space, float c_trav, float c_int )
{
	return tbvh_build_flavour( b, verts, stride, prim_count, space, c_trav, c_int, TBVH_BUILD_REFERENCE );
}

// Many trees, one conversion (include/tinybvh_b200.h): tbvh_convert_batch; tbvh_convert( .., TBVH_LAYOUT_CWBVH ) is count = 1.  Every
// refusal comes before any handle is touched.
static int convert_batch( const char* fn, tbvh_bvh* bvhs, uint32_t count, int to_layout )
{
	if (!(bvhs && count > 0)) { tbvh_set_error( "%s: no handles", fn ); return TBVH_E_ARG; }
	TRY( check_batch_handles( fn, bvhs, count ) );
	uint64_t nodes = 0;
	for (uint32_t k = 0; k < count; k++)
	{
		const tbvh_bvh b = bvhs[k];
		if (!(b->info.layouts & (1u << TBVH_LAYOUT_BVH))) { tbvh_set_error( "%s: handle %u holds no BVH-layout tree", fn, k ); return TBVH_E_STATE; }
		if (b->d_inst) { tbvh_set_error( "%s: handle %u is a TLAS, which has no CWBVH layout", fn, k ); return TBVH_E_STATE; }
		// at least two nodes per tree (a leaf root is wrapped into node 1); SplitLeafs(3) adds at most 2 nodes per 3 primitives
		nodes += (uint64_t)std::max( b->info.used_nodes, 2u ) + 2 * (((uint64_t)b->info.idx_count + 2) / 3);
	}
	if (to_layout != TBVH_LAYOUT_CWBVH) { tbvh_set_error( "%s: target layout %d (only TBVH_LAYOUT_CWBVH converts in batches)", fn, to_layout ); return TBVH_E_UNSUPPORTED; }
	if (nodes > TBVH_CONVERT_BATCH_MAX_NODES) { tbvh_set_error( "%s: up to %llu split-tree nodes in one batch (at most %u)", fn, (unsigned long long)nodes, (unsigned)TBVH_CONVERT_BATCH_MAX_NODES ); return TBVH_E_LIMIT; }
	CUDA_TRY( cudaSetDevice( bvhs[0]->ctx->device ) );
	return bvh_to_cwbvh( bvhs, count, bvhs[0]->ctx->stream );
}

int tbvh_convert( tbvh_bvh b, int to_layout )
{
	ARG_CHECK( b, "NULL handle" );
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	if (!(b->info.layouts & (1u << TBVH_LAYOUT_BVH))) { tbvh_set_error( "tbvh_convert: source layout BVH not resident" ); return TBVH_E_STATE; }
	if (to_layout == TBVH_LAYOUT_BVH_GPU) return bvh_to_bvh_gpu( b, b->ctx->stream );
	if (to_layout == TBVH_LAYOUT_CWBVH) return convert_batch( __func__, &b, 1, to_layout );
	tbvh_set_error( "tbvh_convert: unsupported target layout %d", to_layout );
	return TBVH_E_UNSUPPORTED;
}

int tbvh_convert_batch( tbvh_bvh* bvhs, uint32_t count, int to_layout )
{
	return convert_batch( __func__, bvhs, count, to_layout );
}

static cudaMemcpyKind out_kind( int space ) { return space == TBVH_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost; }

int tbvh_download_bvh( tbvh_bvh b, void* nodes32, uint32_t* prim_idx, int space )
{
	ARG_CHECK( b, "NULL handle" );
	if (!(b->info.layouts & (1u << TBVH_LAYOUT_BVH))) { tbvh_set_error( "layout BVH not resident" ); return TBVH_E_STATE; }
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	if (nodes32) CUDA_TRY( cudaMemcpy( nodes32, b->d_nodes, (size_t)b->info.used_nodes * 32, out_kind( space ) ) );
	if (prim_idx) CUDA_TRY( cudaMemcpy( prim_idx, b->d_prim_idx, (size_t)b->info.idx_count * 4, out_kind( space ) ) );
	return TBVH_OK;
}

int tbvh_download_bvh_gpu( tbvh_bvh b, void* nodes64, int space )
{
	ARG_CHECK( b && nodes64, "NULL argument" );
	if (!(b->info.layouts & (1u << TBVH_LAYOUT_BVH_GPU)) || !b->d_nodes_gpu) { tbvh_set_error( "layout BVH_GPU not resident" ); return TBVH_E_STATE; }
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	CUDA_TRY( cudaMemcpy( nodes64, b->d_nodes_gpu, (size_t)b->info.used_nodes_gpu * 64, out_kind( space ) ) );
	return TBVH_OK;
}

int tbvh_download_cwbvh( tbvh_bvh b, void* bvh8_data, void* bvh8_tris, int space )
{
	ARG_CHECK( b, "NULL handle" );
	if (!(b->info.layouts & (1u << TBVH_LAYOUT_CWBVH))) { tbvh_set_error( "layout CWBVH not resident" ); return TBVH_E_STATE; }
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	if (bvh8_data) CUDA_TRY( cudaMemcpy( bvh8_data, b->d_cw_nodes, (size_t)b->info.used_blocks * 16, out_kind( space ) ) );
	if (bvh8_tris) CUDA_TRY( cudaMemcpy( bvh8_tris, b->d_cw_tris, (size_t)b->info.cwbvh_tri_count * 48, out_kind( space ) ) );
	return TBVH_OK;
}

// ---- traversal ------------------------------------------------------------------------------------------------

// live handles (a TLAS remembers its BLAS handles; a destroyed one must be noticed, not dereferenced)
static std::mutex g_live_mutex;
static std::vector<tbvh_bvh> g_live;
static void live_add( tbvh_bvh b ) { std::lock_guard<std::mutex> lk( g_live_mutex ); g_live.push_back( b ); }
static void live_remove( tbvh_bvh b ) { std::lock_guard<std::mutex> lk( g_live_mutex ); for (size_t i = 0; i < g_live.size(); i++) if (g_live[i] == b) { g_live[i] = g_live.back(); g_live.pop_back(); break; } }

// a TLAS points at the arrays of its BLASses: refuse to walk it once one of them was rebuilt, re-uploaded or destroyed
extern "C++" int tlas_check( tbvh_bvh t, int layout )
{
	// the layout argument of a traversal call on a TLAS names the layout the BLASses are walked in (trace_tlas.cu)
	const uint32_t want = layout == TBVH_LAYOUT_CWBVH ? 1u << TBVH_LAYOUT_CWBVH : 1u << TBVH_LAYOUT_BVH;
	if (layout != TBVH_LAYOUT_CWBVH && layout != TBVH_LAYOUT_BVH && layout != TBVH_LAYOUT_BVH_GPU) { tbvh_set_error( "unknown layout %d", layout ); return TBVH_E_ARG; }
	if (!(t->tlas_blas_layouts & want) && want == (1u << TBVH_LAYOUT_BVH) && t->tlas_deep_blas)
	{ tbvh_set_error( "TLAS: BLAS %u has depth %u, the two-level kernel walks a BVH-layout BLAS with a %d-entry stack (walk its CWBVH layout)", t->tlas_deep_blas - 1, t->tlas_deep_depth, TBVH_STACK ); return TBVH_E_LIMIT; }
	if (!(t->tlas_blas_layouts & want))
	{ tbvh_set_error( "TLAS: not every BLAS held its %s layout when the TLAS was built", layout == TBVH_LAYOUT_CWBVH ? "CWBVH" : "BVH" ); return TBVH_E_STATE; }
	return tlas_stale_check( t );
}

extern "C++" int tlas_stale_check( tbvh_bvh t )
{
	std::lock_guard<std::mutex> lk( g_live_mutex );
	for (const BlasLink& l : t->links)
	{
		bool alive = false;
		for (tbvh_bvh h : g_live) if (h == l.blas) { alive = true; break; }
		if (!alive || l.blas->generation != l.generation)
		{ tbvh_set_error( "TLAS is stale: a BLAS it was built over has been %s since (build the TLAS again, tiny_bvh.h:2221)", alive ? "rebuilt or re-uploaded" : "destroyed" ); return TBVH_E_STATE; }
	}
	return TBVH_OK;
}

static int trace_dispatch( tbvh_bvh b, int layout, const void* d_rays, uint32_t stride, void* d_hits, uint32_t hit_stride,
	uint32_t* d_bits, uint64_t n, bool anyhit, cudaStream_t s )
{
	unsigned long long* st = b->stats ? b->d_stats.get() : 0;
	if (layout == TBVH_LAYOUT_BVH || layout == TBVH_LAYOUT_BVH_GPU) return bvh2_trace_launch( b, d_rays, stride, d_hits, hit_stride, d_bits, n, anyhit, s, st );
	if (layout == TBVH_LAYOUT_CWBVH) return cwbvh_trace_launch( b, d_rays, stride, d_hits, hit_stride, d_bits, n, anyhit, s, st );
	tbvh_set_error( "unknown layout %d", layout );
	return TBVH_E_ARG;
}

int tbvh_intersect_device( tbvh_bvh b, int layout, void* d_rays, uint32_t stride, void* d_hits, uint64_t n, void* stream )
{
	ARG_CHECK( b && d_rays && stride >= 64 && (stride & 15) == 0, "bad ray buffer" );
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	if (b->stats) CUDA_TRY( cudaMemsetAsync( b->d_stats, 0, 32, (cudaStream_t)stream ) );
	if (b->d_inst)
	{
		// TLAS: hits carry the instance (hit.inst, byte 44) and are written into the ray records
		if (d_hits) { tbvh_set_error( "TLAS hits are written in place (t,u,v,prim at byte 48, inst at byte 44): pass d_hits = NULL" ); return TBVH_E_UNSUPPORTED; }
		TRY( tlas_check( b, layout ) );
		return tlas_trace_launch( b, layout, d_rays, stride, 0, n, false, (cudaStream_t)stream );
	}
	if (d_hits) return trace_dispatch( b, layout, d_rays, stride, d_hits, 16, 0, n, false, (cudaStream_t)stream );
	return trace_dispatch( b, layout, d_rays, stride, (char*)d_rays + 48, stride, 0, n, false, (cudaStream_t)stream );
}

int tbvh_occluded_device( tbvh_bvh b, int layout, const void* d_rays, uint32_t stride, uint32_t* d_bits, uint64_t n, void* stream )
{
	ARG_CHECK( b && d_rays && d_bits && stride >= 64 && (stride & 15) == 0, "bad ray buffer" );
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	if (b->stats) CUDA_TRY( cudaMemsetAsync( b->d_stats, 0, 32, (cudaStream_t)stream ) );
	if (b->d_inst) { TRY( tlas_check( b, layout ) ); return tlas_trace_launch( b, layout, d_rays, stride, d_bits, n, true, (cudaStream_t)stream ); }
	return trace_dispatch( b, layout, d_rays, stride, 0, 0, d_bits, n, true, (cudaStream_t)stream );
}

// what the batch launch of the same handle and layout passes its kernel, after the same refusals (host only)
int tbvh_device_view( tbvh_bvh b, int layout, tbvh_view* out )
{
	ARG_CHECK( b && out, "NULL argument" );
	*out = tbvh_view{};
	tbvh_view v{};
	if (b->d_inst)
	{
		TRY( tlas_check( b, layout ) );
		TRY( tlas_trace_check( b, layout ) );
		v.kind = layout == TBVH_LAYOUT_CWBVH ? TBVH_VIEW_TLAS_CWBVH : TBVH_VIEW_TLAS_BVH;
		v.nodes = b->d_nodes, v.prim_idx = b->d_prim_idx, v.inst = b->d_inst, v.blas = b->d_blas;
		v.root_ref = b->root_ref, v.root_count = b->root_count, v.inst_shift = tlas_inst_shift( b );
	}
	else if (layout == TBVH_LAYOUT_BVH || layout == TBVH_LAYOUT_BVH_GPU)
	{
		TRY( bvh2_trace_check( b, 1 ) );
		v.kind = TBVH_VIEW_BVH, v.nodes = b->trav(), v.tris = b->d_leaf_tris, v.root_ref = b->root_ref, v.root_count = b->root_count;
		v.stack = b->info.max_depth + 1 > TBVH_STACK ? TBVH_STACK_DEEP : TBVH_STACK;
	}
	else if (layout == TBVH_LAYOUT_CWBVH)
	{
		TRY( cwbvh_trace_check( b, 1 ) );
		v.kind = TBVH_VIEW_CWBVH, v.nodes = b->d_cw_trav, v.tris = b->d_cw_tris, v.cw_rd_limit = b->cw_rd_limit;
	}
	else { tbvh_set_error( "unknown layout %d", layout ); return TBVH_E_ARG; }
	*out = v;
	return TBVH_OK;
}

// plain device memory for callers of the *_device entry points that do not link the CUDA runtime themselves
int tbvh_device_alloc( tbvh_ctx c, size_t bytes, void** out )
{
	ARG_CHECK( c && out, "NULL argument" );
	CUDA_TRY( cudaSetDevice( c->device ) );
	CUDA_TRY( cudaMalloc( out, bytes ) );
	return TBVH_OK;
}
int tbvh_device_free( tbvh_ctx c, void* p )
{
	ARG_CHECK( c, "NULL context" );
	CUDA_TRY( cudaSetDevice( c->device ) );
	if (p) CUDA_TRY( cudaFree( p ) );
	return TBVH_OK;
}
int tbvh_device_sync( tbvh_ctx c )
{
	ARG_CHECK( c, "NULL context" );
	CUDA_TRY( cudaSetDevice( c->device ) );
	CUDA_TRY( cudaDeviceSynchronize() );
	return TBVH_OK;
}
int tbvh_copy_from_device( void* host, const void* d_src, size_t bytes )
{
	ARG_CHECK( host && d_src, "NULL argument" );
	CUDA_TRY( cudaMemcpy( host, d_src, bytes, cudaMemcpyDeviceToHost ) );
	return TBVH_OK;
}

// host records -> packed 64-byte device records (bytes 0..63 of each), asynchronous on `stream`: what a caller of the *_device
// entry points needs to get its batch into HBM (the speedtest's own upload, tiny_bvh_speedtest.cpp:1110-1115)
int tbvh_copy_rays_to_device( const void* rays, uint32_t stride, uint64_t n, void* d_rays, void* stream )
{
	ARG_CHECK( rays && d_rays && stride >= 64, "bad ray buffer" );
	if (n == 0) return TBVH_OK;
	CUDA_TRY( cudaMemcpy2DAsync( d_rays, 64, rays, stride, 64, n, cudaMemcpyHostToDevice, (cudaStream_t)stream ) );
	return TBVH_OK;
}

// ---- host-buffer path ---------------------------------------------------------------------------------------------
// tbvh_intersect / tbvh_intersect_packed / tbvh_occluded on HOST ray records.  Only bytes 0..63 of each record cross PCIe inbound
// and only the 16-byte hit (or one bit) outbound.  The batch is cut into chunks that flow through TBVH_SLOTS stage buffers:
//
//     s_in  : chunk k+1   host records --(2D copy of 64-byte rows, or a gather kernel through the pinned mapping)--> slot.d_rays
//     s_run : chunk k     traversal kernel: slot.d_rays -> slot.d_hits (packed 16-byte hits) / slot.d_bits
//     s_out : chunk k-1   slot.d_hits --(2D copy of 16-byte rows into Ray.hit, or one contiguous copy for the packed form)--> host
//
// Each direction owns a stream, so the inbound copy engine never waits for an outbound copy queued ahead of it; events hand a
// slot from stage to stage and back (out_done -> the next inbound copy into that slot).  One call at a time per context
// (host_mutex): concurrent callers on one handle are serialised, as SURVEY 8(b) asks.
__global__ void __launch_bounds__( 256 ) k_gather_rays( const float4* __restrict__ src, const uint32_t stride_f4, float4* __restrict__ dst, const uint64_t n )
{
	const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, r = t >> 2;
	if (r < n) dst[t] = src[r * stride_f4 + (t & 3)];
}

__global__ void __launch_bounds__( 256 ) k_scatter_hits( const float4* __restrict__ src, float4* __restrict__ dst, const uint32_t stride_f4, const uint64_t n )
{
	const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (r < n) dst[r * stride_f4 + 3] = src[r];
}

// device alias of a page-locked host pointer, or NULL when the memory is pageable
static void* mapped_alias( const void* host )
{
	cudaPointerAttributes a;
	if (cudaPointerGetAttributes( &a, host ) != cudaSuccess) { cudaGetLastError(); return 0; }
	if (a.type != cudaMemoryTypeHost || !a.devicePointer) return 0;
	return a.devicePointer;
}

static int ensure_slots( tbvh_ctx c )
{
	const size_t rec = c->host_path == 2 ? 128 : 64; // host_path 2 stages whole 128-byte records
	if (c->slot_rays == c->chunk_rays && c->slot_rec >= rec) return TBVH_OK;
	free_slots( c );
	for (HostSlot& sl : c->slot)
	{
		TRY( sl.d_rays.alloc( c->chunk_rays * rec ) );
		TRY( sl.d_hits.alloc( c->chunk_rays * 16 ) );
		TRY( sl.d_bits.alloc( c->chunk_rays / 8 + 4 ) );
	}
	c->slot_rays = c->chunk_rays, c->slot_rec = rec;
	return TBVH_OK;
}

// inbound stage of one chunk: on return s_in carries the copy and slot.in_done is recorded behind it
static int stage_in( tbvh_ctx c, const int k, const uint64_t chunk, const char* h, const char* h_dev, const uint32_t stride, const uint64_t cnt, uint32_t* staged_stride )
{
	HostSlot& sl = c->slot[k];
	*staged_stride = 64;
	if (chunk >= TBVH_SLOTS) CUDA_TRY( cudaStreamWaitEvent( c->s_in, sl.out_done, 0 ) ); // the slot's previous tenant has left the device
	if (c->host_path == 2 && stride == 128 && c->slot_rec >= 128)
	{
		// whole records, one contiguous copy: twice the bytes, but large read requests instead of the 2D copy's 64-byte rows
		CUDA_TRY( cudaMemcpyAsync( sl.d_rays, h, cnt * 128, cudaMemcpyHostToDevice, c->s_in ) );
		*staged_stride = 128;
	}
	else if (c->host_path == 1 && h_dev && (stride & 15) == 0)
	{
		const uint64_t threads = cnt * 4;
		k_gather_rays<<<(uint32_t)((threads + 255) / 256), 256, 0, c->s_in>>>( (const float4*)h_dev, stride / 16, (float4*)sl.d_rays.p, cnt );
		LAUNCHED();
	}
	else if (c->h2d_split > 1 && cnt >= 4096)
	{
		// rows of the chunk spread over several streams so more than one copy engine pulls them; s_in joins the parts
		const int parts = c->h2d_split;
		const uint64_t per = ((cnt + parts - 1) / parts + 31) & ~31ull;
		CUDA_TRY( cudaEventRecord( c->ev_fork, c->s_in ) );
		for (int p = 0; p < parts; p++)
		{
			const uint64_t a = per * p, e = a + per < cnt ? a + per : cnt;
			if (a >= e) break;
			cudaStream_t ps = p == 0 ? c->s_in : c->s_in_part[p - 1];
			if (p) CUDA_TRY( cudaStreamWaitEvent( ps, c->ev_fork, 0 ) );
			CUDA_TRY( cudaMemcpy2DAsync( (char*)sl.d_rays + a * 64, 64, h + a * stride, stride, 64, e - a, cudaMemcpyHostToDevice, ps ) );
			if (p) { CUDA_TRY( cudaEventRecord( c->ev_part[k][p - 1], ps ) ); CUDA_TRY( cudaStreamWaitEvent( c->s_in, c->ev_part[k][p - 1], 0 ) ); }
		}
	}
	else CUDA_TRY( cudaMemcpy2DAsync( sl.d_rays, 64, h, stride, 64, cnt, cudaMemcpyHostToDevice, c->s_in ) );
	CUDA_TRY( cudaEventRecord( sl.in_done, c->s_in ) );
	CUDA_TRY( cudaStreamWaitEvent( c->s_run, sl.in_done, 0 ) );
	return TBVH_OK;
}

static int drain( tbvh_ctx c )
{
	CUDA_TRY( cudaStreamSynchronize( c->s_out ) );
	CUDA_TRY( cudaStreamSynchronize( c->s_run ) );
	CUDA_TRY( cudaStreamSynchronize( c->s_in ) );
	return TBVH_OK;
}

// tbvh_intersect / tbvh_intersect_packed (closest hits: in place, or into packed_hits) and tbvh_occluded (bits: any hit).  They
// differ in the trace call and the outbound copy of each chunk only.
static int trace_host( const char* fn, tbvh_bvh b, int layout, void* rays, uint32_t stride, uint64_t n, void* packed_hits, uint32_t* bits )
{
	if (!(b && rays && stride >= 64)) { tbvh_set_error( "%s: bad ray buffer", fn ); return TBVH_E_ARG; }
	tbvh_ctx c = b->ctx;
	std::lock_guard<std::mutex> lk( c->host_mutex );
	CUDA_TRY( cudaSetDevice( c->device ) );
	TRY( ensure_slots( c ) );
	if (b->stats) CUDA_TRY( cudaMemset( b->d_stats, 0, 32 ) );
	const bool anyhit = bits != 0, tlas = b->d_inst != 0;
	if (tlas)
	{
		if (packed_hits) { tbvh_set_error( "tbvh_intersect_packed: TLAS hits carry the instance and are returned in the ray records" ); return TBVH_E_UNSUPPORTED; }
		TRY( tlas_check( b, layout ) );
	}
	char* dev_alias = (char*)mapped_alias( rays );
	const bool in_place = !anyhit && !packed_hits && !tlas; // closest hits written into the caller's records: d2h_mode picks how
	const bool scatter = in_place && c->d2h_mode == 3 && dev_alias && (stride & 15) == 0;
	// d2h_mode 1: the kernel writes the hit into the staged record and bytes 0..63 of every record - exactly its first cache line - travel
	// back, so the host receives FULL-line writes (no read-for-ownership of a partially written line); bytes 0..47 return unchanged
	const bool full_line = in_place && c->d2h_mode == 1 && stride >= 64;
	// d2h_mode 2: the hits leave the device packed (one contiguous copy per chunk) into page-locked staging, and a few host threads on
	// the device's NUMA node write them into the strided records while later chunks are in flight
	const bool host_scatter = in_place && c->d2h_mode == 2 && n >= 65536;
	if (host_scatter)
	{
		for (HostSlot& sl : c->slot) if (!sl.h_hits.p)
		{
			void* q = 0;
			const cudaError_t e = on_node( c->numa_node, [&]() { return cudaHostAlloc( &q, c->chunk_rays * 16, cudaHostAllocDefault ); } );
			if (e != cudaSuccess) { tbvh_set_error( "host staging: %s", cudaGetErrorString( e ) ); return TBVH_E_CUDA; }
			sl.h_hits.adopt( q, c->chunk_rays * 16 );
		}
		if (!c->pool) c->pool = new HostPool( (unsigned)c->scatter_threads, c->numa_node );
	}
	// hits of chunk `ch` (already on their way to slot staging) -> the caller's records
	auto scatter_chunk = [&]( const uint64_t ch ) -> int
	{
		HostSlot& sl = c->slot[ch % TBVH_SLOTS];
		CUDA_TRY( cudaEventSynchronize( sl.out_done ) );
		const uint64_t off = ch * c->chunk_rays, cnt = n - off < c->chunk_rays ? n - off : c->chunk_rays;
		char* dst = (char*)rays + off * stride + 48;
		const char* src = (const char*)sl.h_hits.p;
		c->pool->run( [=]( unsigned t, unsigned T )
		{
			const uint64_t per = (cnt + T - 1) / T, a = per * t, e = a + per < cnt ? a + per : cnt;
			for (uint64_t i = a; i < e; i++) memcpy( dst + i * stride, src + i * 16, 16 );
		} );
		return TBVH_OK;
	};
	uint64_t chunk = 0;
	int rc = TBVH_OK;
	for (uint64_t off = 0; off < n && rc == TBVH_OK; off += c->chunk_rays, chunk++)
	{
		const int k = (int)(chunk % TBVH_SLOTS);
		HostSlot& sl = c->slot[k];
		const uint64_t cnt = n - off < c->chunk_rays ? n - off : c->chunk_rays;
		char* h = (char*)rays + off * stride;
		char* hd = dev_alias ? dev_alias + off * stride : 0;
		uint32_t* d_bits = anyhit ? (uint32_t*)sl.d_bits : 0;
		auto body = [&]() -> int
		{
			if (host_scatter && chunk >= TBVH_SLOTS) TRY( scatter_chunk( chunk - TBVH_SLOTS ) ); // frees this slot's staging
			uint32_t ss = 64;
			TRY( stage_in( c, k, chunk, h, hd, stride, cnt, &ss ) );
			if (tlas) TRY( tlas_trace_launch( b, layout, sl.d_rays, ss, d_bits, cnt, anyhit, c->s_run ) );  // closest: hit + instance written into the staged records
			else if (full_line) TRY( trace_dispatch( b, layout, sl.d_rays, ss, (char*)sl.d_rays + 48, ss, 0, cnt, false, c->s_run ) );
			else TRY( trace_dispatch( b, layout, sl.d_rays, ss, anyhit ? 0 : sl.d_hits.get(), anyhit ? 0 : 16, d_bits, cnt, anyhit, c->s_run ) );
			CUDA_TRY( cudaEventRecord( sl.run_done, c->s_run ) );
			CUDA_TRY( cudaStreamWaitEvent( c->s_out, sl.run_done, 0 ) );
			if (anyhit) CUDA_TRY( cudaMemcpyAsync( bits + off / 32, sl.d_bits, ((cnt + 31) / 32) * 4, cudaMemcpyDeviceToHost, c->s_out ) ); // chunk_rays is a multiple of 32
			else if (tlas) CUDA_TRY( cudaMemcpy2DAsync( h + 44, stride, (char*)sl.d_rays + 44, ss, 20, cnt, cudaMemcpyDeviceToHost, c->s_out ) );
			else if (packed_hits) CUDA_TRY( cudaMemcpyAsync( (char*)packed_hits + off * 16, sl.d_hits, cnt * 16, cudaMemcpyDeviceToHost, c->s_out ) );
			else if (host_scatter) CUDA_TRY( cudaMemcpyAsync( sl.h_hits.p, sl.d_hits, cnt * 16, cudaMemcpyDeviceToHost, c->s_out ) );
			else if (full_line) CUDA_TRY( cudaMemcpy2DAsync( h, stride, sl.d_rays, ss, 64, cnt, cudaMemcpyDeviceToHost, c->s_out ) );
			else if (scatter)
			{
				k_scatter_hits<<<(uint32_t)((cnt + 255) / 256), 256, 0, c->s_out>>>( (const float4*)sl.d_hits, (float4*)hd, stride / 16, cnt );
				LAUNCHED();
			}
			else CUDA_TRY( cudaMemcpy2DAsync( h + 48, stride, sl.d_hits, 16, 16, cnt, cudaMemcpyDeviceToHost, c->s_out ) );
			CUDA_TRY( cudaEventRecord( sl.out_done, c->s_out ) );
			return TBVH_OK;
		};
		rc = body();
	}
	if (host_scatter && rc == TBVH_OK)
		for (uint64_t ch = chunk > TBVH_SLOTS ? chunk - TBVH_SLOTS : 0; ch < chunk && rc == TBVH_OK; ch++) rc = scatter_chunk( ch );
	const int rd = drain( c ); // also after an error: nothing of this call may still be in flight when the mutex is released
	return rc != TBVH_OK ? rc : rd;
}

int tbvh_intersect( tbvh_bvh b, int layout, void* rays, uint32_t stride, uint64_t n ) { return trace_host( __func__, b, layout, rays, stride, n, 0, 0 ); }

int tbvh_intersect_packed( tbvh_bvh b, int layout, const void* rays, uint32_t stride, uint64_t n, void* hits )
{
	ARG_CHECK( hits, "hits == NULL" );
	return trace_host( __func__, b, layout, (void*)rays, stride, n, hits, 0 );
}

int tbvh_occluded( tbvh_bvh b, int layout, const void* rays, uint32_t stride, uint64_t n, uint32_t* bits )
{
	ARG_CHECK( bits, "bad ray buffer" );
	return trace_host( __func__, b, layout, (void*)rays, stride, n, 0, bits );
}

} // extern "C"
