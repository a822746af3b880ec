// harness/device_api_b200.cu - tracing from one's own kernel (the role tiny_bvh_minimal_gpu.cpp plays in the reference, with the
// traversal called from inside the application's kernel as wavefront.cl does): random triangles -> BVH8_CWBVH::Build on the GPU ->
// DeviceView() -> a kernel of this file traces the host's camera rays with tbvh::intersect_cwbvh and shadow rays it makes with
// tbvh::isoccluded_cwbvh.  The hits are checked against the batch call on the same rays.
//   nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -Iinclude harness/device_api_b200.cu -Ltinybvh_b200 -ltinybvh_b200 \
//        -Xlinker -rpath,$PWD/tinybvh_b200 -o device_api_b200
#include "tinybvh_b200.hpp"
#include "tinybvh_b200_device.cuh"
#include <string.h>
#include <vector>

struct Vec4 { float x, y, z, w; };
static uint32_t seed = 0x12345678;
static float rnd() { seed ^= seed << 13, seed ^= seed >> 17, seed ^= seed << 5; return seed * 2.3283064365387e-10f; }

// one camera ray per thread from the 64-byte records the host wrote: the closest hit goes into the record, a ray back towards the
// camera from 1% short of the hit, made in registers, asks whether anything lies in between
__global__ void trace( const tbvh_view view, float4* rec, uint32_t* occluded, const int R )
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R) return;
	tbvh::Ray r = { rec[i * 4], rec[i * 4 + 1], rec[i * 4 + 2], rec[i * 4 + 3] };
	tbvh::intersect_cwbvh( view, r );
	rec[i * 4 + 3] = r.hit;
	if (r.hit.x < 1e30f)
	{
		const float t = r.hit.x * 0.99f;
		tbvh::Ray s;
		s.O = make_float4( r.O.x + r.D.x * t, r.O.y + r.D.y * t, r.O.z + r.D.z * t, r.O.w );
		s.D = make_float4( -r.D.x, -r.D.y, -r.D.z, 0 ), s.rD = make_float4( -r.rD.x, -r.rD.y, -r.rD.z, 0 );
		s.hit = make_float4( t, 0, 0, 0 );
		if (tbvh::isoccluded_cwbvh( view, s )) atomicAdd( occluded, 1u );
	}
}

int main()
{
	const int N = 8192, R = 1024;
	std::vector<Vec4> tris( N * 3 );
	for (int i = 0; i < N; i++)
	{
		const float x = rnd() * 4, y = rnd() * 4, z = rnd() * 4;
		for (int v = 0; v < 3; v++) tris[i * 3 + v] = { x + rnd() * 0.1f, y + rnd() * 0.1f, z + rnd() * 0.1f, 0 };
	}
	tinybvh_b200::BVH8_CWBVH bvh;
	bvh.Build( tris.data(), N );
	std::vector<tinybvh_b200::Ray> rays( R );
	for (int i = 0; i < R; i++)
	{
		const float O[3] = { 2, 2, -3 }, D[3] = { (i % 32) / 32.0f - 0.5f, (i / 32) / 32.0f - 0.5f, 1 };
		rays[i] = tinybvh_b200::Ray( O, D );
	}
	const tbvh_view view = bvh.DeviceView(); // take a new view whenever the tree changes
	float4* d_rec = 0;
	uint32_t* d_occ = 0;
	cudaMalloc( &d_rec, R * 64 ), cudaMalloc( &d_occ, 4 ), cudaMemset( d_occ, 0, 4 );
	cudaMemcpy2D( d_rec, 64, rays.data(), sizeof( tinybvh_b200::Ray ), 64, R, cudaMemcpyHostToDevice ); // bytes 0..63 of each record
	trace<<<(R + 127) / 128, 128>>>( view, d_rec, d_occ, R );
	std::vector<float4> out( R * 4 );
	uint32_t occ = 0;
	if (cudaMemcpy( out.data(), d_rec, R * 64, cudaMemcpyDeviceToHost ) != cudaSuccess || cudaMemcpy( &occ, d_occ, 4, cudaMemcpyDeviceToHost ) != cudaSuccess)
	{
		printf( "device_api_b200: kernel failed: %s\n", cudaGetErrorString( cudaGetLastError() ) );
		return 1;
	}
	cudaFree( d_rec ), cudaFree( d_occ );
	bvh.Intersect( rays.data(), R ); // the same rays through the batch call
	int hits = 0, mismatches = 0;
	for (int i = 0; i < R; i++)
	{
		const float4 h = out[i * 4 + 3];
		if (h.x < 1e30f) hits++;
		if (memcmp( &h, &rays[i].t, 16 ) != 0) mismatches++;
	}
	printf( "device_api_b200: %i tris, %i of %i rays hit from the caller's kernel, %i mismatches against the batch call, %u shadow rays occluded\n",
		N, hits, R, mismatches, occ );
	return hits > 0 && mismatches == 0 ? 0 : 1;
}
