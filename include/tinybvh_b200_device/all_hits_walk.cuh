// include/tinybvh_b200_device/all_hits_walk.cuh - the multi-hit ray walk over the BVH2: the k nearest distinct triangles a ray crosses and
// their count.  Shared by the library's kernel (intersect_all.cu: k_intersect_all) and the device function of include/tinybvh_b200_device.cuh.
//
// Semantics are the engine's own (DESIGN.md 4.14), restated on the host by tests/allhits_oracle.c in the same fp32 operation order:
//  * per child box: bvh2_pair_step's slab arithmetic with the lane's own direction signs and the ray's own tmax (never lowered by a hit):
//    tmin_c = fmaxf( fmaxf( tx1, ty1 ), fmaxf( tz1, 0 ) ), tfar_c = fminf( fminf( tx2, ty2 ), fminf( tz2, tmax ) ); a child is reached when
//    its parent is and tfar_c >= tmin_c; the root's box is not tested.  Its path bound is P( child ) = fmaxf( P( parent ), tmin_c ), P( root )
//    = 0, so P never decreases down a path; a node an uploaded tree reaches on several paths is walked once per path;
//  * a reference (leaf, triangle) is accepted when mt_test accepts it on [0, tmax] with a t that is not NaN; its key is fmaxf( t, P( leaf ) );
//  * each distinct prim takes its least key over its accepted references, and the result is the k smallest ( key, prim ) pairs (keys
//    compared as floats, ties to the lower prim), plus the number of distinct prims saturated at k + 1.
// So the result does not depend on the visiting order, and a subtree with P > b, b the (k+1)-th key once k + 1 prims are held, is pruned
// exactly (not at P == b: a subtree at exactly b may still hold a lower prim).
#pragma once
#include "base.cuh"
#include "closest_walk.cuh"

#define TBVH_INTERSECT_ALL_MAX_K 64 // the largest k of tbvh_intersect_all / tbvh::intersect_all_bvh
#define TBVH_INTERSECT_ALL_REG_K 4  // k up to this holds its buffer in registers; larger k in local memory

namespace tbvh
{

// ( ka, pa ) before ( kb, pb ): keys as floats (-0 equals +0), ties to the lower prim
__device__ __forceinline__ bool ah_before( const float ka, const uint32_t pa, const float kb, const uint32_t pb ) { return ka < kb || (ka == kb && pa < pb); }

// The sorted buffer of the nearest distinct prims seen so far, at most c = k + 1 <= CAP entries, each prim once with its least key.
// REG: every loop runs over CAP with compile-time indices, so the arrays stay in registers; otherwise over the n entries held, in local memory.
// b, bp: the key and prim of entry c - 1 once the buffer holds c entries, else +inf (every key is <= +inf: nothing is pruned before the
// buffer is full).
template <int CAP, bool REG> struct AhBuffer
{
	float key[CAP], t[CAP], u[CAP], v[CAP];
	uint32_t prim[CAP];
	int n, c;
	float b;
	uint32_t bp;

	__device__ __forceinline__ void init( const int cap ) { n = 0, c = cap, b = __int_as_float( 0x7f800000 ), bp = CP_NO_PRIM; }

	// one accepted reference
	__device__ __forceinline__ void insert( const float kn, const uint32_t pn, const float tn, const float un, const float vn )
	{
		// j: the slot that is given up - the prim's own entry, else the end (or the last entry of a full buffer)
		int j = n;
		float kj = 0.0f;
		if (REG)
		{
			#pragma unroll
			for (int i = 0; i < CAP; i++) if (i < n && prim[i] == pn) j = i, kj = key[i];
		}
		else for (int i = 0; i < n; i++) if (prim[i] == pn) { j = i, kj = key[i]; break; }
		if (j < n) { if (!(kn < kj)) return; }                              // the prim is held with a key no larger
		else if (n == c) { if (!ah_before( kn, pn, b, bp )) return; j = c - 1; }
		else n++;
		// pos: the entries before j that come first (the buffer is sorted); entries pos .. j - 1 move up one slot, over slot j
		int pos = 0;
		if (REG)
		{
			#pragma unroll
			for (int i = 0; i < CAP; i++) if (i < j && ah_before( key[i], prim[i], kn, pn )) pos++;
			#pragma unroll
			for (int i = CAP - 1; i > 0; i--)
				if (i > pos && i <= j) key[i] = key[i - 1], t[i] = t[i - 1], u[i] = u[i - 1], v[i] = v[i - 1], prim[i] = prim[i - 1];
			#pragma unroll
			for (int i = 0; i < CAP; i++)
				if (i == pos) key[i] = kn, t[i] = tn, u[i] = un, v[i] = vn, prim[i] = pn;
			if (n == c)
			{
				#pragma unroll
				for (int i = 0; i < CAP; i++) if (i == c - 1) b = key[i], bp = prim[i];
			}
		}
		else
		{
			while (pos < j && ah_before( key[pos], prim[pos], kn, pn )) pos++;
			for (int i = j; i > pos; i--) key[i] = key[i - 1], t[i] = t[i - 1], u[i] = u[i - 1], v[i] = v[i - 1], prim[i] = prim[i - 1];
			key[pos] = kn, t[pos] = tn, u[pos] = un, v[pos] = vn, prim[pos] = pn;
			if (n == c) b = key[c - 1], bp = prim[c - 1];
		}
	}

	// the k = c - 1 records { t, u, v, prim }, slots past n { tmax, 0, 0, CP_NO_PRIM }; returns n, the count saturated at k + 1
	__device__ __forceinline__ uint32_t store( float4* out, const float tmax ) const
	{
		const int k = c - 1;
		const float4 empty = make_float4( tmax, 0.0f, 0.0f, __uint_as_float( CP_NO_PRIM ) );
		if (REG)
		{
			#pragma unroll
			for (int i = 0; i < CAP; i++) if (i < k) out[i] = i < n ? make_float4( t[i], u[i], v[i], __uint_as_float( prim[i] ) ) : empty;
		}
		else for (int i = 0; i < k; i++) out[i] = i < n ? make_float4( t[i], u[i], v[i], __uint_as_float( prim[i] ) ) : empty;
		return (uint32_t)n;
	}
};

// the k empty records of a ray that takes no walk (or of a view of another kind)
__device__ __forceinline__ void ah_store_empty( float4* out, const uint32_t k, const float tmax )
{
	for (uint32_t i = 0; i < k; i++) out[i] = make_float4( tmax, 0.0f, 0.0f, __uint_as_float( CP_NO_PRIM ) );
}

// One ray's multi-hit walk from (ref, cnt) = the root, with a caller-supplied stack deep enough for the tree (bvh2_walk's sizes); k in
// 1 .. CAP - 1.  Writes the k records to out and returns the count.  A ray whose tmax is NaN or negative takes no walk: count 0.
template <int CAP, bool REG> __device__ __forceinline__ uint32_t ah_walk( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	uint32_t ref, uint32_t cnt, const float4& O, const float4& D, const float4& rD, const float tmax, const uint32_t k, float4* out, CpEntry* stack )
{
	if (!(tmax >= 0.0f)) { ah_store_empty( out, k, tmax ); return 0; }
	AhBuffer<CAP, REG> buf;
	buf.init( (int)k + 1 );
	const float ox = O.x, oy = O.y, oz = O.z, dx = D.x, dy = D.y, dz = D.z, rdx = rD.x, rdy = rD.y, rdz = rD.z;
	const bool PX = dx >= 0, PY = dy >= 0, PZ = dz >= 0;
	// -(O*rD), rounded product, as bvh2_walk
	const float nrox = -__fmul_rn( ox, rdx ), nroy = -__fmul_rn( oy, rdy ), nroz = -__fmul_rn( oz, rdz );
	int sp = 0;
	float P = 0.0f;
	while (true)
	{
		if (cnt == 0)
		{
			const float4* p = nodes + (size_t)ref * 2;
			const float4 a0 = __ldg( p ), a1 = __ldg( p + 1 ), b0 = __ldg( p + 2 ), b1 = __ldg( p + 3 );
			// bvh2_pair_step's slab test with the lane's own signs (its OCT = -1 form), written beside it so that its callers keep their code
			const float tx1a = __fmaf_rn( PX ? a0.x : a1.x, rdx, nrox ), tx2a = __fmaf_rn( PX ? a1.x : a0.x, rdx, nrox );
			const float ty1a = __fmaf_rn( PY ? a0.y : a1.y, rdy, nroy ), ty2a = __fmaf_rn( PY ? a1.y : a0.y, rdy, nroy );
			const float tz1a = __fmaf_rn( PZ ? a0.z : a1.z, rdz, nroz ), tz2a = __fmaf_rn( PZ ? a1.z : a0.z, rdz, nroz );
			const float tx1b = __fmaf_rn( PX ? b0.x : b1.x, rdx, nrox ), tx2b = __fmaf_rn( PX ? b1.x : b0.x, rdx, nrox );
			const float ty1b = __fmaf_rn( PY ? b0.y : b1.y, rdy, nroy ), ty2b = __fmaf_rn( PY ? b1.y : b0.y, rdy, nroy );
			const float tz1b = __fmaf_rn( PZ ? b0.z : b1.z, rdz, nroz ), tz2b = __fmaf_rn( PZ ? b1.z : b0.z, rdz, nroz );
			const float tmina = fmaxf( fmaxf( tx1a, ty1a ), fmaxf( tz1a, 0.0f ) ), tminb = fmaxf( fmaxf( tx1b, ty1b ), fmaxf( tz1b, 0.0f ) );
			const float tfara = fminf( fminf( tx2a, ty2a ), fminf( tz2a, tmax ) ), tfarb = fminf( fminf( tx2b, ty2b ), fminf( tz2b, tmax ) );
			const float Pa = fmaxf( P, tmina ), Pb = fmaxf( P, tminb );
			const bool va = tfara >= tmina && !(Pa > buf.b), vb = tfarb >= tminb && !(Pb > buf.b);
			const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w ), refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
			if (va && vb)
			{
				const bool swp = Pb < Pa; // nearer child first, the left one on ties
				ref = swp ? refb : refa, cnt = swp ? cntb : cnta, P = swp ? Pb : Pa;
				stack[sp++] = swp ? CpEntry{ refa, cnta, Pa } : CpEntry{ refb, cntb, Pb };
				continue;
			}
			if (va) { ref = refa, cnt = cnta, P = Pa; continue; }
			if (vb) { ref = refb, cnt = cntb, P = Pb; continue; }
		}
		else
		{
			const float4* tp = tris + (size_t)ref * 3;
			for (uint32_t i = 0; i < cnt; i++, tp += 3)
			{
				const float4 v0 = __ldg( tp ), e1 = __ldg( tp + 1 ), e2 = __ldg( tp + 2 );
				float t, u, v;
				if (!mt_test( ox, oy, oz, dx, dy, dz, v0, e1, e2, tmax, t, u, v ) || t != t) continue;
				const float key = fmaxf( t, P );
				if (!(key > buf.b)) buf.insert( key, __float_as_uint( v0.w ), t, u, v );
			}
		}
		// pop, pruning again against the current bound
		while (true)
		{
			if (sp == 0) return buf.store( out, tmax );
			const CpEntry e = stack[--sp];
			if (!(e.P > buf.b)) { ref = e.ref, cnt = e.cnt, P = e.P; break; }
		}
	}
}

// the walk of one ray record for any k in 1 .. TBVH_INTERSECT_ALL_MAX_K: the register buffer up to TBVH_INTERSECT_ALL_REG_K, else local memory
template <int STACKN> __device__ __forceinline__ uint32_t ah_intersect_all( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	const uint32_t root_ref, const uint32_t root_count, const float4& O, const float4& D, const float4& rD, const float tmax, const uint32_t k, float4* out )
{
	CpEntry stack[STACKN];
	if (k <= TBVH_INTERSECT_ALL_REG_K) return ah_walk<TBVH_INTERSECT_ALL_REG_K + 1, true>( nodes, tris, root_ref, root_count, O, D, rD, tmax, k, out, stack );
	return ah_walk<TBVH_INTERSECT_ALL_MAX_K + 1, false>( nodes, tris, root_ref, root_count, O, D, rD, tmax, k, out, stack );
}

} // namespace tbvh
