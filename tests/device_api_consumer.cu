// tests/device_api_consumer.cu - a caller's own kernels over include/tinybvh_b200_device.cuh, driven by tests/test_device_api_gpu.py
// through ctypes.  Built with nvcc -I include alone: the device functions need no library.
#include "tinybvh_b200_device.cuh"

// which device function a lane calls
enum Fn { FN_BVH = 0, FN_CWBVH = 1, FN_TLAS_BVH = 2, FN_TLAS_CWBVH = 3 };

__device__ __forceinline__ void intersect( const int fn, const tbvh_view& v, tbvh::Ray& r )
{
	if (fn == FN_BVH) tbvh::intersect_bvh( v, r );
	else if (fn == FN_CWBVH) tbvh::intersect_cwbvh( v, r );
	else if (fn == FN_TLAS_BVH) tbvh::intersect_tlas<TBVH_LAYOUT_BVH>( v, r );
	else tbvh::intersect_tlas<TBVH_LAYOUT_CWBVH>( v, r );
}

__device__ __forceinline__ bool isoccluded( const int fn, const tbvh_view& v, const tbvh::Ray& r )
{
	if (fn == FN_BVH) return tbvh::isoccluded_bvh( v, r );
	if (fn == FN_CWBVH) return tbvh::isoccluded_cwbvh( v, r );
	if (fn == FN_TLAS_BVH) return tbvh::isoccluded_tlas<TBVH_LAYOUT_BVH>( v, r );
	return tbvh::isoccluded_tlas<TBVH_LAYOUT_CWBVH>( v, r );
}

__device__ __forceinline__ tbvh::Ray load( const char* rays, const uint32_t i )
{
	const float4* p = (const float4*)(rays + (size_t)i * 64);
	return tbvh::Ray{ p[0], p[1], p[2], p[3] };
}

// One ray per thread.  sel == NULL: every ray is traced once by set 0.  Otherwise sel[i] = trips | set << 4: trips = 0 leaves the record
// alone, k > 0 traces it k times from a loop (each trip from the record as loaded, the last one kept); set picks (view, fn, rays, bits).
// Closest hit: the record is written back whole; any-hit: bit i of bits.
template <bool ANYHIT> __global__ void k_trace( const tbvh_view v0, const int fn0, char* rays0, uint32_t* bits0, const tbvh_view v1, const int fn1,
	char* rays1, uint32_t* bits1, const uint32_t* sel, const uint32_t n )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint32_t s = sel ? sel[i] : 1u, trips = s & 15u;
	if (trips == 0) return;
	const bool second = (s >> 4) & 1u;
	const tbvh_view& v = second ? v1 : v0;
	const int fn = second ? fn1 : fn0;
	char* rays = second ? rays1 : rays0;
	const tbvh::Ray r0 = load( rays, i );
	tbvh::Ray r = r0;
	bool occ = false;
	for (uint32_t k = 0; k < trips; k++)
	{
		if (ANYHIT) occ = isoccluded( fn, v, r0 );
		else { r = r0; intersect( fn, v, r ); }
	}
	if (ANYHIT) { if (occ) atomicOr( (second ? bits1 : bits0) + (i >> 5), 1u << (i & 31) ); }
	else
	{
		float4* p = (float4*)(rays + (size_t)i * 64);
		p[0] = r.O, p[1] = r.D, p[2] = r.rD, p[3] = r.hit;
	}
}

// A shadow ray from a closest hit, built in registers: from the hit point towards `light`, tmax = the distance to it minus eps; a ray
// that missed gets tmax 0 (never occluded).  The mask and everything else of the camera ray carry over.
__device__ __forceinline__ tbvh::Ray shadow_ray( const tbvh::Ray& c, const float3 light, const float eps )
{
	const bool hit = c.hit.x < BVH_FAR;
	const float t = hit ? c.hit.x : 0.0f;
	const float px = __fmaf_rn( c.D.x, t, c.O.x ), py = __fmaf_rn( c.D.y, t, c.O.y ), pz = __fmaf_rn( c.D.z, t, c.O.z );
	float dx = __fsub_rn( light.x, px ), dy = __fsub_rn( light.y, py ), dz = __fsub_rn( light.z, pz );
	const float len = __fsqrt_rn( __fmaf_rn( dz, dz, __fmaf_rn( dy, dy, __fmul_rn( dx, dx ) ) ) );
	const float rl = __fdiv_rn( 1.0f, len );
	dx = __fmul_rn( dx, rl ), dy = __fmul_rn( dy, rl ), dz = __fmul_rn( dz, rl );
	tbvh::Ray s;
	s.O = make_float4( __fmaf_rn( dx, eps, px ), __fmaf_rn( dy, eps, py ), __fmaf_rn( dz, eps, pz ), c.O.w );
	s.D = make_float4( dx, dy, dz, c.D.w );
	s.rD = make_float4( tbvh::safercp( dx ), tbvh::safercp( dy ), tbvh::safercp( dz ), 0.0f );
	s.hit = make_float4( hit ? __fsub_rn( len, __fmul_rn( 2.0f, eps ) ) : 0.0f, 0.0f, 0.0f, 0.0f );
	return s;
}

// camera ray -> closest hit -> shadow ray in registers -> any-hit, one kernel; writes the shadow records it built and the bits.
__global__ void k_camera_shadow( const tbvh_view v, const int fn_hit, const int fn_occ, const char* cam, char* shadow, uint32_t* bits, const uint32_t n,
	const float3 light, const float eps )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	tbvh::Ray r = load( cam, i );
	intersect( fn_hit, v, r );
	const tbvh::Ray s = shadow_ray( r, light, eps );
	float4* p = (float4*)(shadow + (size_t)i * 64);
	p[0] = s.O, p[1] = s.D, p[2] = s.rD, p[3] = s.hit;
	if (isoccluded( fn_occ, v, s )) atomicOr( bits + (i >> 5), 1u << (i & 31) );
}

// the shadow records of k_camera_shadow from camera records already traced (the two-launch form the measurement compares against)
__global__ void k_shadow_records( const char* cam, char* shadow, const uint32_t n, const float3 light, const float eps )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const tbvh::Ray s = shadow_ray( load( cam, i ), light, eps );
	float4* p = (float4*)(shadow + (size_t)i * 64);
	p[0] = s.O, p[1] = s.D, p[2] = s.rD, p[3] = s.hit;
}

extern "C"
{
int dc_trace( tbvh_view v0, int fn0, void* rays0, uint32_t* bits0, tbvh_view v1, int fn1, void* rays1, uint32_t* bits1, const uint32_t* sel,
	uint32_t n, int anyhit )
{
	if (n == 0) return 0;
	const uint32_t grid = (n + 127) / 128;
	if (anyhit) k_trace<true><<<grid, 128>>>( v0, fn0, (char*)rays0, bits0, v1, fn1, (char*)rays1, bits1, sel, n );
	else k_trace<false><<<grid, 128>>>( v0, fn0, (char*)rays0, bits0, v1, fn1, (char*)rays1, bits1, sel, n );
	return (int)cudaDeviceSynchronize();
}

int dc_camera_shadow( tbvh_view v, int fn_hit, int fn_occ, const void* cam, void* shadow, uint32_t* bits, uint32_t n, float lx, float ly, float lz, float eps )
{
	if (n == 0) return 0;
	k_camera_shadow<<<(n + 127) / 128, 128>>>( v, fn_hit, fn_occ, (const char*)cam, (char*)shadow, bits, n, make_float3( lx, ly, lz ), eps );
	return (int)cudaDeviceSynchronize();
}

// asynchronous on `stream` (tools/device_api_perf.py times them between device events)
int dc_camera_shadow_async( tbvh_view v, int fn_hit, int fn_occ, const void* cam, void* shadow, uint32_t* bits, uint32_t n, float lx, float ly, float lz, float eps,
	void* stream )
{
	if (n == 0) return 0;
	k_camera_shadow<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>( v, fn_hit, fn_occ, (const char*)cam, (char*)shadow, bits, n, make_float3( lx, ly, lz ), eps );
	return (int)cudaGetLastError();
}

int dc_shadow_records_async( const void* cam, void* shadow, uint32_t n, float lx, float ly, float lz, float eps, void* stream )
{
	if (n == 0) return 0;
	k_shadow_records<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>( (const char*)cam, (char*)shadow, n, make_float3( lx, ly, lz ), eps );
	return (int)cudaGetLastError();
}
}
