// tests/closest_point_consumer.cu - a caller's own kernel over include/tinybvh_b200_device.cuh's proximity functions, built by
// tests/test_closest_point_gpu.py with nvcc -I include alone (no library link), as tests/device_api_consumer.cu is.
//
// cc_query: for every query i whose lane is selected (sel == NULL: all; else bit i & 31 of sel[i >> 5]: divergent lanes of one warp),
// out[i] = tbvh::closest_point_bvh( view, q[i] ) and bit i of bits = tbvh::sphere_overlaps_bvh( view, q[i] ).  Unselected queries are
// left as they were.
#include "tinybvh_b200_device.cuh"

__global__ void k_cc_query( const tbvh_view v, const float4* __restrict__ q, float4* out, uint32_t* bits, const uint32_t* sel, const uint32_t n )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	if (sel && !((sel[i >> 5] >> (i & 31)) & 1u)) return;
	const float4 qi = q[i];
	// closest point on even lanes first, then the overlap: different lanes of one warp run different functions at once
	if (i & 1)
	{
		if (tbvh::sphere_overlaps_bvh( v, qi )) atomicOr( bits + (i >> 5), 1u << (i & 31) );
		out[i] = tbvh::closest_point_bvh( v, qi );
	}
	else
	{
		out[i] = tbvh::closest_point_bvh( v, qi );
		if (tbvh::sphere_overlaps_bvh( v, qi )) atomicOr( bits + (i >> 5), 1u << (i & 31) );
	}
}

extern "C" int cc_query( const tbvh_view v, const void* q, void* out, uint32_t* bits, const uint32_t* sel, const uint32_t n )
{
	if (n == 0) return 0;
	k_cc_query<<<(n + 127) / 128, 128>>>( v, (const float4*)q, (float4*)out, bits, sel, n );
	if (cudaGetLastError() != cudaSuccess) return -1;
	return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}
