// tests/sphere_cast_consumer.cu - a caller's own kernel over include/tinybvh_b200_device.cuh's sphere casts, built by
// tests/test_sphere_cast_gpu.py with nvcc -I include alone (no library link), as tests/closest_point_consumer.cu is.
//
// sc_query: for every query i (two float4 rows) whose lane is selected (sel == NULL: all; else bit i & 31 of sel[i >> 5]: divergent lanes
// of one warp), out[i] = tbvh::sphere_cast_bvh( view, q0, q1 ) and bit i of bits = tbvh::sphere_cast_occluded_bvh( view, q0, q1 ).
// Unselected queries are left as they were.
#include "tinybvh_b200_device.cuh"

__global__ void k_sc_query( const tbvh_view v, const float4* __restrict__ q, float4* out, uint32_t* bits, const uint32_t* sel, const uint32_t n )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	if (sel && !((sel[i >> 5] >> (i & 31)) & 1u)) return;
	const float4 q0 = q[2 * i], q1 = q[2 * i + 1];
	// the cast on even lanes first, then the bit: different lanes of one warp run different functions at once
	if (i & 1)
	{
		if (tbvh::sphere_cast_occluded_bvh( v, q0, q1 )) atomicOr( bits + (i >> 5), 1u << (i & 31) );
		out[i] = tbvh::sphere_cast_bvh( v, q0, q1 );
	}
	else
	{
		out[i] = tbvh::sphere_cast_bvh( v, q0, q1 );
		if (tbvh::sphere_cast_occluded_bvh( v, q0, q1 )) atomicOr( bits + (i >> 5), 1u << (i & 31) );
	}
}

extern "C" int sc_query( const tbvh_view v, const void* q, void* out, uint32_t* bits, const uint32_t* sel, const uint32_t n )
{
	if (n == 0) return 0;
	k_sc_query<<<(n + 127) / 128, 128>>>( v, (const float4*)q, (float4*)out, bits, sel, n );
	if (cudaGetLastError() != cudaSuccess) return -1;
	return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}
