// tinybvh_b200/csrc/instance_update.cu - BLASInstance::Update (tiny_bvh.h:8386) for a whole instance list on the device, for sm_90a.
//
// One thread per instance computes the inverse transform and the world box (instance_update.cuh: the host routine's own arithmetic)
// and the block writes, in one pass, the three things a TLAS build needs: the record's invTransform / aabbMin / aabbMax, the
// TlasInst entry the two-level kernel reads, and the two float4 box entries the builder reads.  A 192-byte record per thread would be
// a 6-way strided access, so records move through shared memory: the block's threads load and store consecutive 16-byte chunks.
#include "common.cuh"
#include "instance_update.cuh"

#define UPD_BLOCK 128
#define UPD_WORDS 25   // words of one instance in shared memory: 24 used; odd, so a thread walking its own instance meets no bank conflict

namespace
{
// BLASInstance :1443 in 16-byte chunks: transform 0..3, invTransform 4..7, (aabbMin, blasIdx) 8, (aabbMax, mask) 9
__global__ void __launch_bounds__( UPD_BLOCK ) k_instance_update( char* __restrict__ rec, const uint32_t stride, const uint32_t n,
	const float4* __restrict__ blas_box /* root box of BLAS k: [2 k] min, [2 k + 1] max */, const uint32_t blas_count,
	float4* __restrict__ tlas_inst /* TlasInst: 5 float4 per instance */, float4* __restrict__ aabbs, uint32_t* __restrict__ bad_blas )
{
	__shared__ float sm[UPD_BLOCK * UPD_WORDS];
	const uint32_t first = blockIdx.x * UPD_BLOCK, count = min( (uint32_t)UPD_BLOCK, n - first );
	// in: chunks 0..3 (transform), 8 and 9 (blasIdx and mask in their w lanes)
	for (uint32_t q = threadIdx.x; q < count * 6; q += UPD_BLOCK)
	{
		const uint32_t i = q / 6, c = q % 6;
		const float4 v = *(const float4*)(rec + (size_t)(first + i) * stride + (c < 4 ? c : c + 4) * 16);
		float* d = sm + i * UPD_WORDS + c * 4;
		d[0] = v.x, d[1] = v.y, d[2] = v.z, d[3] = v.w;
	}
	__syncthreads();
	if (threadIdx.x < count)
	{
		float* my = sm + threadIdx.x * UPD_WORDS;
		float T[16], iT[16], mn[3], mx[3];
		#pragma unroll
		for (int k = 0; k < 16; k++) T[k] = my[k];
		uint32_t blasIdx = __float_as_uint( my[19] );
		if (blasIdx >= blas_count) atomicOr( bad_blas, 1u ), blasIdx = 0; // reported by the call; never dereferenced
		const float4 b0 = __ldg( blas_box + 2 * blasIdx ), b1 = __ldg( blas_box + 2 * blasIdx + 1 );
		const float bmin[3] = { b0.x, b0.y, b0.z }, bmax[3] = { b1.x, b1.y, b1.z };
		upd_instance( T, iT, mn, mx, bmin, bmax );
		// out: chunks 4..9 of the record in words 0..23 (blasIdx and mask stay where they were loaded: words 19 and 23)
		#pragma unroll
		for (int k = 0; k < 16; k++) my[k] = iT[k];
		my[16] = mn[0], my[17] = mn[1], my[18] = mn[2], my[20] = mx[0], my[21] = mx[1], my[22] = mx[2];
	}
	__syncthreads();
	for (uint32_t q = threadIdx.x; q < count * 6; q += UPD_BLOCK)
	{
		const uint32_t i = q / 6, c = q % 6;
		const float* d = sm + i * UPD_WORDS + c * 4;
		*(float4*)(rec + (size_t)(first + i) * stride + (c + 4) * 16) = make_float4( d[0], d[1], d[2], d[3] );
	}
	for (uint32_t q = threadIdx.x; q < count * 5; q += UPD_BLOCK)
	{
		const uint32_t i = q / 5, c = q % 5;
		const float* d = sm + i * UPD_WORDS;
		tlas_inst[(size_t)first * 5 + q] = c < 4 ? make_float4( d[c * 4], d[c * 4 + 1], d[c * 4 + 2], d[c * 4 + 3] ) : make_float4( d[19], d[23], 0.0f, 0.0f );
	}
	for (uint32_t q = threadIdx.x; q < count * 2; q += UPD_BLOCK)
	{
		const float* d = sm + (q >> 1) * UPD_WORDS + 16 + (q & 1) * 4;
		aabbs[(size_t)first * 2 + q] = make_float4( d[0], d[1], d[2], 0.0f );
	}
}
} // namespace

int instance_update_launch( void* d_records, uint32_t stride, uint32_t n, const float4* d_blas_box, uint32_t blas_count, void* d_tlas_inst, float4* d_aabbs,
	uint32_t* d_bad_blas, cudaStream_t s )
{
	k_instance_update<<<(n + UPD_BLOCK - 1) / UPD_BLOCK, UPD_BLOCK, 0, s>>>( (char*)d_records, stride, n, d_blas_box, blas_count, (float4*)d_tlas_inst, d_aabbs, d_bad_blas );
	LAUNCHED();
	return TBVH_OK;
}
