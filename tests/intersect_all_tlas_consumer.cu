// tests/intersect_all_tlas_consumer.cu - a caller's own kernel over include/tinybvh_b200_device.cuh's two-level multi-hit function, built by
// tests/test_intersect_all_tlas_gpu.py with nvcc -I include alone (no library link), as tests/intersect_all_consumer.cu is.
//
// iat_query: for every ray i whose lane is selected (sel == NULL: all; else bit i & 31 of sel[i >> 5]: divergent lanes of one warp), with
// k_i = ks[i] (a different k per lane), the k_i records of tbvh::intersect_all_tlas( view, ray i, k_i ) go to out + offs[i], its instances
// to insts + offs[i] and the count to counts[i].  reps > 1 calls it that many times in a loop (each call overwrites the same slots).
// Unselected rays are left as they were.
#include "tinybvh_b200_device.cuh"

__global__ void k_iat_query( const tbvh_view v, const float4* __restrict__ rays, const uint32_t* ks, const uint64_t* offs, float4* out, uint32_t* insts,
	uint32_t* counts, const uint32_t* sel, const uint32_t n, const uint32_t reps )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	if (sel && !((sel[i >> 5] >> (i & 31)) & 1u)) return;
	tbvh::Ray r;
	r.O = rays[i * 4], r.D = rays[i * 4 + 1], r.rD = rays[i * 4 + 2], r.hit = rays[i * 4 + 3];
	for (uint32_t it = 0; it < reps; it++) counts[i] = tbvh::intersect_all_tlas( v, r, ks[i], out + offs[i], insts + offs[i] );
}

extern "C" int iat_query( const tbvh_view v, const void* rays, const uint32_t* ks, const uint64_t* offs, void* out, uint32_t* insts, uint32_t* counts,
	const uint32_t* sel, const uint32_t n, const uint32_t reps )
{
	if (n == 0) return 0;
	k_iat_query<<<(n + 127) / 128, 128>>>( v, (const float4*)rays, ks, offs, (float4*)out, insts, counts, sel, n, reps );
	if (cudaGetLastError() != cudaSuccess) return -1;
	return cudaDeviceSynchronize() == cudaSuccess ? 0 : -1;
}
