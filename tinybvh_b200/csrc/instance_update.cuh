// tinybvh_b200/csrc/instance_update.cuh - BLASInstance::Update (tiny_bvh.h:8386-8399) with InvertTransform (:8402-8428), stated once
// for the host (tbvh_instance_update, api.cu) and the device (k_instance_update, instance_update.cu).
//
// The frozen reference build vectorises the sixteen cofactor sums, and the lanes of different rows end up with different fused
// multiply-adds; the shapes below were identified by exhaustive search over every contraction gcc may legally form (3 x 2^4 per
// cofactor, 12 for the determinant, 6^4 for the corner transform) against BLASInstance::Update on 2,000 random matrices, and are
// pinned by the tests.  A cofactor is s0*(a0*b0)*c0 + ... + s5*(a5*b5)*c5 with p_k = round( a_k*b_k ):
//   rows 0,1 : t0 = round( p0*c0 ); acc = fma( +-p1, c1, t0 ); then fma( +-p_k, c_k, acc ) for k = 2..5
//   row 2    : acc = fma( p0, c0, +-round( p1*c1 ) ); k=2: acc +- round( p2*c2 ); k=3,4: fma; k=5: acc +- round( p5*c5 )
//   row 3    : acc = fma( p0, c0, +-round( p1*c1 ) ); k=2: fma; k=3,4: acc +- round(..); k=5: fma
//   det      = fma( T3, c12, fma( T2, c8, fma( T0, c0, round( T1*c4 ) ) ) ); every cell is then multiplied by 1/det
//   corner   : row = fma( Tz, z, fma( Tx, x, round( Ty*y ) ) ) + Tw, divided by w only when w != 1
// Every rounding is spelled out: _rn intrinsics on the device, so nvcc's contraction (-fmad) cannot change one; plain operators
// and fmaf on the host, where the caller switches the compiler's contraction off (UPD_HOST_ATTR on the function this is inlined into).
#pragma once
#include <math.h>

#ifdef __CUDA_ARCH__
#define UPD_MUL( a, b ) __fmul_rn( a, b )
#define UPD_ADD( a, b ) __fadd_rn( a, b )
#define UPD_SUB( a, b ) __fsub_rn( a, b )
#define UPD_FMA( a, b, c ) __fmaf_rn( a, b, c )
#define UPD_RCP( a ) __fdiv_rn( 1.0f, a )
#else
#define UPD_MUL( a, b ) ((a) * (b))
#define UPD_ADD( a, b ) ((a) + (b))
#define UPD_SUB( a, b ) ((a) - (b))
#define UPD_FMA( a, b, c ) fmaf( a, b, c )
#define UPD_RCP( a ) (1.0f / (a))
#endif
#define UPD_HOST_ATTR __attribute__( (optimize( "fp-contract=off" )) )

struct UpdTerm { signed char s; unsigned char a, b, c; };

__host__ __device__ __forceinline__ float upd_cofactor( const float* T, const UpdTerm* e, const int first_fused_left, const unsigned fused_mask )
{
	float p[6];
	#pragma unroll
	for (int k = 0; k < 6; k++) p[k] = UPD_MUL( T[e[k].a], T[e[k].b] );
	const float p0 = e[0].s < 0 ? -p[0] : p[0];
	float acc;
	if (first_fused_left) { const float t1 = UPD_MUL( p[1], T[e[1].c] ); acc = UPD_FMA( p0, T[e[0].c], e[1].s > 0 ? t1 : -t1 ); }
	else { const float t0 = UPD_MUL( p0, T[e[0].c] ); acc = UPD_FMA( e[1].s > 0 ? p[1] : -p[1], T[e[1].c], t0 ); }
	#pragma unroll
	for (int k = 2; k < 6; k++)
	{
		if (fused_mask & (1u << (k - 2))) acc = UPD_FMA( e[k].s > 0 ? p[k] : -p[k], T[e[k].c], acc );
		else { const float t = UPD_MUL( p[k], T[e[k].c] ); acc = e[k].s > 0 ? UPD_ADD( acc, t ) : UPD_SUB( acc, t ); }
	}
	return acc;
}

// T: transform (16, row-major) -> iT: invTransform (16); aabbMin / aabbMax (3 each): box of the eight transformed corners of
// [bmin, bmax], folded in corner order with the reference's tinybvh_min / tinybvh_max (a < b ? a : b: the later of two tied zeros
// gives the sign, a NaN corner replaces the bound)
__host__ __device__ __forceinline__ void upd_instance( const float* T, float* iT, float* aabbMin, float* aabbMax, const float* bmin, const float* bmax )
{
	// the six terms (sign, a, b, c) of each cofactor, in the reference's order
	const UpdTerm E[16][6] = {
	 {{+1,5,10,15},{-1,5,11,14},{-1,9,6,15},{+1,9,7,14},{+1,13,6,11},{-1,13,7,10}}, {{-1,1,10,15},{+1,1,11,14},{+1,9,2,15},{-1,9,3,14},{-1,13,2,11},{+1,13,3,10}},
	 {{+1,1,6,15},{-1,1,7,14},{-1,5,2,15},{+1,5,3,14},{+1,13,2,7},{-1,13,3,6}}, {{-1,1,6,11},{+1,1,7,10},{+1,5,2,11},{-1,5,3,10},{-1,9,2,7},{+1,9,3,6}},
	 {{-1,4,10,15},{+1,4,11,14},{+1,8,6,15},{-1,8,7,14},{-1,12,6,11},{+1,12,7,10}}, {{+1,0,10,15},{-1,0,11,14},{-1,8,2,15},{+1,8,3,14},{+1,12,2,11},{-1,12,3,10}},
	 {{-1,0,6,15},{+1,0,7,14},{+1,4,2,15},{-1,4,3,14},{-1,12,2,7},{+1,12,3,6}}, {{+1,0,6,11},{-1,0,7,10},{-1,4,2,11},{+1,4,3,10},{+1,8,2,7},{-1,8,3,6}},
	 {{+1,4,9,15},{-1,4,11,13},{-1,8,5,15},{+1,8,7,13},{+1,12,5,11},{-1,12,7,9}}, {{-1,0,9,15},{+1,0,11,13},{+1,8,1,15},{-1,8,3,13},{-1,12,1,11},{+1,12,3,9}},
	 {{+1,0,5,15},{-1,0,7,13},{-1,4,1,15},{+1,4,3,13},{+1,12,1,7},{-1,12,3,5}}, {{-1,0,5,11},{+1,0,7,9},{+1,4,1,11},{-1,4,3,9},{-1,8,1,7},{+1,8,3,5}},
	 {{-1,4,9,14},{+1,4,10,13},{+1,8,5,14},{-1,8,6,13},{-1,12,5,10},{+1,12,6,9}}, {{+1,0,9,14},{-1,0,10,13},{-1,8,1,14},{+1,8,2,13},{+1,12,1,10},{-1,12,2,9}},
	 {{-1,0,5,14},{+1,0,6,13},{+1,4,1,14},{-1,4,2,13},{-1,12,1,6},{+1,12,2,5}}, {{+1,0,5,10},{-1,0,6,9},{-1,4,1,10},{+1,4,2,9},{+1,8,1,6},{-1,8,2,5}} };
	float c[16];
	#pragma unroll
	for (int k = 0; k < 16; k++) c[k] = k < 8 ? upd_cofactor( T, E[k], 0, 15u ) : k < 12 ? upd_cofactor( T, E[k], 1, 6u ) : upd_cofactor( T, E[k], 1, 9u );
	const float t14 = UPD_MUL( T[1], c[4] );
	const float det = UPD_FMA( T[3], c[12], UPD_FMA( T[2], c[8], UPD_FMA( T[0], c[0], t14 ) ) );
	if (det == 0)
	{
		#pragma unroll
		for (int k = 0; k < 16; k++) iT[k] = c[k]; // "invert failed": the reference returns with the cofactors stored
	}
	else
	{
		const float invdet = UPD_RCP( det );
		#pragma unroll
		for (int k = 0; k < 16; k++) iT[k] = UPD_MUL( c[k], invdet );
	}
	#pragma unroll
	for (int k = 0; k < 3; k++) aabbMin[k] = 1e30f, aabbMax[k] = -1e30f;
	#pragma unroll
	for (int j = 0; j < 8; j++)
	{
		const float p[3] = { j & 1 ? bmax[0] : bmin[0], j & 2 ? bmax[1] : bmin[1], j & 4 ? bmax[2] : bmin[2] };
		float r[3];
		#pragma unroll
		for (int k = 0; k < 3; k++) { const float ty = UPD_MUL( T[k * 4 + 1], p[1] ); r[k] = UPD_ADD( UPD_FMA( T[k * 4 + 2], p[2], UPD_FMA( T[k * 4], p[0], ty ) ), T[k * 4 + 3] ); }
		const float wy = UPD_MUL( T[13], p[1] );
		const float w = UPD_ADD( UPD_FMA( T[14], p[2], UPD_FMA( T[12], p[0], wy ) ), T[15] );
		if (!(w == 1)) { const float rw = UPD_RCP( w ); r[0] = UPD_MUL( r[0], rw ), r[1] = UPD_MUL( r[1], rw ), r[2] = UPD_MUL( r[2], rw ); }
		#pragma unroll
		for (int k = 0; k < 3; k++) aabbMin[k] = aabbMin[k] < r[k] ? aabbMin[k] : r[k], aabbMax[k] = aabbMax[k] > r[k] ? aabbMax[k] : r[k];
	}
}
