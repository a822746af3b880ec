// include/tinybvh_b200_device/base.cuh - what every walk of include/tinybvh_b200_device.cuh shares: the constants, the oracle's
// Moeller-Trumbore test, the reference's min / max and safercp, the 64-byte ray record and the two-level tables.  The library's own
// kernels (tinybvh_b200/csrc) use the same definitions.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define BVH_FAR 1e30f          // the reference's own value (tiny_bvh.h); a different definition is an error
#define TBVH_STACK 64          // traversal stack entries per ray of the default BVH2 walks; deeper trees run the TBVH_STACK_DEEP instances
#define TBVH_STACK_DEEP 256    // the reference's own closest-hit stack (tiny_bvh.h:3249; any-hit uses 64, :3409)
#define TLAS_STACK 64          // the reference's IntersectTLAS stack (:3308)

namespace tbvh
{

// ---- device math in the oracle's exact operation order (oracle/tbvh_oracle.c header lists the pairing) ----
// Every fused pair is spelled __fmaf_rn, every unfused product / sum an _rn intrinsic, so nvcc's own
// contraction (-fmad) cannot change the rounding.

// MOLLER_TRUMBORE_TEST tiny_bvh.h:1644-1656 with e1,e2 precomputed (identical bits: v1-v0 is exact-rounded once).
// Returns true when the triangle is accepted for [0, tmax] ([0, tmax) with below_tmax); writes t,u,v.
__device__ __forceinline__ bool mt_test( const float ox, const float oy, const float oz, const float dx, const float dy, const float dz,
	const float4 v0, const float4 e1, const float4 e2, const float tmax, float& t, float& u, float& v, const bool below_tmax = false )
{
	const float hx = __fmaf_rn( dy, e2.z, -__fmul_rn( dz, e2.y ) );
	const float hy = __fmaf_rn( dz, e2.x, -__fmul_rn( dx, e2.z ) );
	const float hz = __fmaf_rn( dx, e2.y, -__fmul_rn( dy, e2.x ) );
	const float a = __fmaf_rn( e1.z, hz, __fmaf_rn( e1.x, hx, __fmul_rn( e1.y, hy ) ) );
	if (fabsf( a ) < 0.000001f) return false;
	const float f = __fdiv_rn( 1.0f, a );
	const float sx = __fsub_rn( ox, v0.x ), sy = __fsub_rn( oy, v0.y ), sz = __fsub_rn( oz, v0.z );
	u = __fmul_rn( f, __fmaf_rn( hz, sz, __fmaf_rn( hx, sx, __fmul_rn( hy, sy ) ) ) );
	const float qx = __fmaf_rn( -e1.y, sz, __fmul_rn( e1.z, sy ) );
	const float qy = __fmaf_rn( -e1.z, sx, __fmul_rn( e1.x, sz ) );
	const float qz = __fmaf_rn( -e1.x, sy, __fmul_rn( e1.y, sx ) );
	v = __fmul_rn( f, __fmaf_rn( dz, qz, __fmaf_rn( dy, qy, __fmul_rn( dx, qx ) ) ) );
	if (u < 0 || v < 0 || __fadd_rn( u, v ) > 1) return false;
	t = __fmul_rn( f, __fmaf_rn( e2.z, qz, __fmaf_rn( e2.x, qx, __fmul_rn( e2.y, qy ) ) ) );
	return !(t < 0 || (below_tmax ? t >= tmax : t > tmax));
}

// The reference folds bounds with tinybvh_min / tinybvh_max (tiny_bvh.h:445-446), a < b ? a : b and a > b ? a : b: on a tie the
// second operand wins, and a NaN in the second operand is returned.
__device__ __forceinline__ float ref_min( const float a, const float b ) { return a < b ? a : b; }
__device__ __forceinline__ float ref_max( const float a, const float b ) { return a > b ? a : b; }

// tinybvh_safercp (:442): the reciprocal of a transformed direction component
__device__ __forceinline__ float safercp( const float x ) { return (x > 1e-12f || x < -1e-12f) ? __fdiv_rn( 1.0f, x ) : (x >= 0 ? BVH_FAR : -BVH_FAR); }

// The 64-byte device ray record, in registers: O | mask, D | instIdx, rD | hit.inst (byte 44, a TLAS's instance), hit (t, u, v, prim)
struct Ray { float4 O, D, rD, hit; };

// ray record i of a traversal batch: O | mask, D, rD | inst, hit (t, u, v, prim) - four 16-byte loads
__device__ __forceinline__ void load_ray( const char* rays, const uint64_t i, const uint32_t stride, float4& ro4, float4& rd4, float4& rr4, float4& rh4 )
{
	const float4* rp = (const float4*)(rays + i * stride);
	ro4 = rp[0], rd4 = rp[1], rr4 = rp[2], rh4 = rp[3];
}

// the two-level tables: one TlasInst per instance (inverse transform, BLAS number, mask), one BlasRef per BLAS
struct TlasInst { float inv[16]; uint32_t blasIdx, mask, pad0, pad1; };                                  // 80 bytes
struct BlasRef { const float4* trav; const float4* tris; uint32_t root_ref, root_count; float cw_rd_limit; uint32_t pad1; const float4* cw_nodes; const float4* cw_tris; }; // 48 bytes: BVH-layout arrays, CWBVH traversal nodes + bvh8Tris (0 when absent) and their rD limit

} // namespace tbvh
