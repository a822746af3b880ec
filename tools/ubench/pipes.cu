// micro-probe: issue rate of the instructions the CWBVH node step is made of, in warp-instructions / clock / SM.
// Every thread runs CHAINS independent dependency chains, STEPS unrolled steps per loop trip, so latency is hidden and the
// loop counter is < 1 % of the issued instructions.  Each block notes its SM and its first and last clock64() (SM clock); an
// SM's rate is the work of the blocks it ran over the span from the first start to the last end there.  Check the loop body with `cuobjdump -sass` after a
// compiler change: each kernel's loop must hold CHAINS x STEPS of the named opcode.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench/pipes tools/ubench/pipes.cu && tools/ubench/pipes
#include <cstdio>
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#define CHAINS 8
#define STEPS 16
#define BLOCK 256

enum { FMNMX, VIMNMX3, VIMNMX3_RELU, ISETP, FSETP, HADD2_F32, FFMA, KINDS };
static const char* NAME[KINDS] = { "FMNMX", "VIMNMX3", "VIMNMX3.RELU", "ISETP", "FSETP", "HADD2.F32", "FFMA" };

template <int KIND> __global__ void __launch_bounds__( BLOCK ) k_probe( const uint32_t* in, uint32_t* out, long long* span, const int iters )
{
	uint32_t a[CHAINS];
	const uint32_t b = in[1], c = in[2];
	#pragma unroll
	for (int k = 0; k < CHAINS; k++) a[k] = in[0] + k * 0x01010101u + threadIdx.x;
	uint32_t p[CHAINS];
	#pragma unroll
	for (int k = 0; k < CHAINS; k++) p[k] = a[k] & 1u;
	__syncthreads();
	const long long t0 = clock64();
	for (int i = 0; i < iters; i++)
	{
		#pragma unroll
		for (int s = 0; s < STEPS; s++)
		{
			#pragma unroll
			for (int k = 0; k < CHAINS; k++)
			{
				if (KIND == FMNMX) a[k] = __float_as_uint( fmaxf( -__uint_as_float( a[k] ), __uint_as_float( b ) ) ); // one FMNMX, negated operand
				if (KIND == VIMNMX3) a[k] = (s & 1) ? (uint32_t)__vimax3_s32( (int)a[k], (int)b, (int)c ) : (uint32_t)__vimin3_s32( (int)a[k], (int)b, (int)c );
				if (KIND == VIMNMX3_RELU) a[k] = (s & 1) ? (uint32_t)__vimax3_s32_relu( (int)a[k], (int)b, (int)c ) : (uint32_t)__vimin3_s32( (int)a[k], (int)b, (int)c );
				// predicate chains: setp with a boolean combine is one ISETP / FSETP (a[] holds the compared values, b / c the bounds)
				if (KIND == ISETP) asm volatile( "{ .reg .pred q; setp.ne.b32 q, %0, 0; setp.lt.xor.s32 q, %1, %2, q; selp.b32 %0, 1, 0, q; }" : "+r"( p[k] ) : "r"( a[k] ), "r"( s & 1 ? b : c ) );
				if (KIND == FSETP) asm volatile( "{ .reg .pred q; setp.ne.b32 q, %0, 0; setp.lt.xor.f32 q, %1, %2, q; selp.b32 %0, 1, 0, q; }" : "+r"( p[k] ) : "f"( __uint_as_float( a[k] ) ), "f"( __uint_as_float( s & 1 ? b : c ) ) );
				if (KIND == HADD2_F32) a[k] = __float_as_uint( __low2float( *(const __half2*)&a[k] ) );
				if (KIND == FFMA) a[k] = __float_as_uint( __fmaf_rn( __uint_as_float( a[k] ), __uint_as_float( b ), __uint_as_float( c ) ) );
			}
		}
	}
	const long long t1 = clock64();
	uint32_t r = 0;
	#pragma unroll
	for (int k = 0; k < CHAINS; k++) r ^= a[k] ^ p[k];
	out[blockIdx.x * BLOCK + threadIdx.x] = r;
	uint32_t sm;
	asm volatile( "mov.u32 %0, %%smid;" : "=r"( sm ) );
	if (threadIdx.x == 0) span[3 * blockIdx.x] = t0, span[3 * blockIdx.x + 1] = t1, span[3 * blockIdx.x + 2] = sm;
}

typedef void (*Kernel)( const uint32_t*, uint32_t*, long long*, int );
static const Kernel KERNEL[KINDS] = { k_probe<FMNMX>, k_probe<VIMNMX3>, k_probe<VIMNMX3_RELU>, k_probe<ISETP>, k_probe<FSETP>, k_probe<HADD2_F32>, k_probe<FFMA> };

int main()
{
	char line[256] = "nvidia-smi unavailable";
	if (FILE* f = popen( "nvidia-smi --id=0 --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv,noheader 2>/dev/null", "r" ))
	{
		if (!fgets( line, sizeof( line ), f )) line[0] = 0;
		pclose( f );
	}
	cudaDeviceProp prop;
	cudaGetDeviceProperties( &prop, 0 );
	printf( "device: %s, %d SMs; nvidia-smi (name, power limit, SM clock, max SM clock): %s", prop.name, prop.multiProcessorCount, line );
	const int blocks = prop.multiProcessorCount * (2048 / BLOCK), iters = 4096;
	uint32_t *d_in, *d_out;
	long long* d_cyc;
	const uint32_t h_in[3] = { 0x3f800000u, 0x3f000000u, 0xbf000000u }; // 1, 0.5, -0.5 as float bit patterns
	cudaMalloc( &d_in, sizeof( h_in ) );
	cudaMalloc( &d_out, (size_t)blocks * BLOCK * 4 );
	cudaMalloc( &d_cyc, (size_t)blocks * 24 );
	cudaMemcpy( d_in, h_in, sizeof( h_in ), cudaMemcpyHostToDevice );
	long long* h_cyc = new long long[3 * blocks];
	const int sms = prop.multiProcessorCount;
	long long* first = new long long[sms];
	long long* last = new long long[sms];
	int* nblk = new int[sms];
	cudaEvent_t e0, e1;
	cudaEventCreate( &e0 ), cudaEventCreate( &e1 );
	int bad = 0;
	for (int kind = 0; kind < KINDS; kind++)
	{
		KERNEL[kind]<<<blocks, BLOCK>>>( d_in, d_out, d_cyc, 16 ); // warm-up
		cudaEventRecord( e0 );
		KERNEL[kind]<<<blocks, BLOCK>>>( d_in, d_out, d_cyc, iters );
		cudaEventRecord( e1 );
		const cudaError_t err = cudaEventSynchronize( e1 );
		if (err != cudaSuccess) { printf( "%s: %s\n", NAME[kind], cudaGetErrorString( err ) ); bad = 1; break; }
		float ms = 0;
		cudaEventElapsedTime( &ms, e0, e1 );
		cudaMemcpy( h_cyc, d_cyc, (size_t)blocks * 24, cudaMemcpyDeviceToHost );
		for (int m = 0; m < sms; m++) first[m] = -1, last[m] = 0, nblk[m] = 0;
		for (int b = 0; b < blocks; b++)
		{
			const int m = (int)h_cyc[3 * b + 2];
			if (m < 0 || m >= sms) continue;
			if (first[m] < 0 || h_cyc[3 * b] < first[m]) first[m] = h_cyc[3 * b];
			if (h_cyc[3 * b + 1] > last[m]) last[m] = h_cyc[3 * b + 1];
			nblk[m]++;
		}
		double rate = 0, span = 0;
		int used = 0;
		for (int m = 0; m < sms; m++) if (nblk[m])
		{
			rate += (double)nblk[m] * (BLOCK / 32) * iters * STEPS * CHAINS / (double)(last[m] - first[m]);
			span += (double)(last[m] - first[m]), used++;
		}
		rate /= used, span /= used;
		printf( "%-13s %6.2f warp-inst/clk/SM  (%d SMs, %.0f cycles per SM, %.3f ms, implied SM clock %.0f MHz)\n", NAME[kind], rate, used, span, ms, span / (ms * 1e3) );
	}
	return bad;
}
