// include/tinybvh_b200_device/all_hits_walk.cuh - the multi-hit ray walks over the BVH2 and over a TLAS: the k nearest distinct triangles
// (instance hits) a ray crosses and their count.  Shared by the library's kernels (intersect_all.cu: k_intersect_all, k_intersect_all_tlas)
// and the device functions of include/tinybvh_b200_device.cuh.
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
// Over a TLAS the same rules apply once to the TLAS and once more inside each instance: the BLAS root is reached with the path bound of the
// TLAS leaf and its box is not tested, the BLAS is walked with the ray transformed into its space (t is shared between the two, the
// direction is not re-normalised) and the same tmax, and a hit is an ( instance, prim ) pair, ties to the lower instance, then prim.
// tests/allhits_tlas_oracle.c restates the two-level rules.
#pragma once
#include "base.cuh"
#include "closest_walk.cuh"

#define TBVH_INTERSECT_ALL_MAX_K 64 // the largest k of tbvh_intersect_all( _tlas ) / tbvh::intersect_all_bvh / _tlas
#define TBVH_INTERSECT_ALL_REG_K 4  // k up to this holds its buffer in registers; larger k in local memory

namespace tbvh
{

// ( ka, pa ) before ( kb, pb ): keys as floats (-0 equals +0), ties to the lower prim
__device__ __forceinline__ bool ah_before( const float ka, const uint32_t pa, const float kb, const uint32_t pb ) { return ka < kb || (ka == kb && pa < pb); }
// ( ka, ia, pa ) before ( kb, ib, pb ): ties to the lower instance, then to the lower prim
__device__ __forceinline__ bool ah_before( const float ka, const uint32_t ia, const uint32_t pa, const float kb, const uint32_t ib, const uint32_t pb )
{
	return ka < kb || (ka == kb && (ia < ib || (ia == ib && pa < pb)));
}

// The instance column of AhBuffer: each entry's instance and bi, the instance of the bound; nothing without INST, so that the buffer of a
// single-level walk keeps its layout and code
template <int CAP, bool INST> struct AhInstColumn { uint32_t inst[CAP]; uint32_t bi; };
template <int CAP> struct AhInstColumn<CAP, false> {};

// The sorted buffer of the nearest distinct hits seen so far, at most c = k + 1 <= CAP entries, each hit once with its least key.  A hit is
// a prim, or with INST an ( instance, prim ) pair.
// REG: every loop runs over CAP with compile-time indices, so the arrays stay in registers; otherwise over the n entries held, in local memory.
// b, bp (bi): the key and prim (and instance) of entry c - 1 once the buffer holds c entries, else +inf (every key is <= +inf: nothing is
// pruned before the buffer is full).
template <int CAP, bool REG, bool INST = false> struct AhBuffer : AhInstColumn<CAP, INST>
{
	float key[CAP], t[CAP], u[CAP], v[CAP];
	uint32_t prim[CAP];
	int n, c;
	float b;
	uint32_t bp;

	__device__ __forceinline__ void init( const int cap )
	{
		n = 0, c = cap, b = __int_as_float( 0x7f800000 ), bp = CP_NO_PRIM;
		if constexpr (INST) this->bi = CP_NO_PRIM;
	}

	__device__ __forceinline__ uint32_t inst_of( const int i ) const { if constexpr (INST) return this->inst[i]; else return 0u; }
	__device__ __forceinline__ uint32_t bound_inst() const { if constexpr (INST) return this->bi; else return 0u; }
	__device__ __forceinline__ bool same( const int i, const uint32_t pn, const uint32_t in ) const { return prim[i] == pn && (!INST || inst_of( i ) == in); }
	__device__ __forceinline__ bool before( const float ka, const uint32_t ia, const uint32_t pa, const float kb, const uint32_t ib, const uint32_t pb ) const
	{
		return INST ? ah_before( ka, ia, pa, kb, ib, pb ) : ah_before( ka, pa, kb, pb );
	}
	__device__ __forceinline__ void move( const int i, const int from )
	{
		key[i] = key[from], t[i] = t[from], u[i] = u[from], v[i] = v[from], prim[i] = prim[from];
		if constexpr (INST) this->inst[i] = this->inst[from];
	}
	__device__ __forceinline__ void put( const int i, const float kn, const uint32_t pn, const float tn, const float un, const float vn, const uint32_t in )
	{
		key[i] = kn, t[i] = tn, u[i] = un, v[i] = vn, prim[i] = pn;
		if constexpr (INST) this->inst[i] = in;
	}
	__device__ __forceinline__ void take_bound( const int i ) { b = key[i], bp = prim[i]; if constexpr (INST) this->bi = this->inst[i]; }

	// one accepted reference of prim pn (of instance in, with INST)
	__device__ __forceinline__ void insert( const float kn, const uint32_t pn, const float tn, const float un, const float vn, const uint32_t in = 0 )
	{
		// j: the slot that is given up - the hit's own entry, else the end (or the last entry of a full buffer)
		int j = n;
		float kj = 0.0f;
		if (REG)
		{
			#pragma unroll
			for (int i = 0; i < CAP; i++) if (i < n && same( i, pn, in )) j = i, kj = key[i];
		}
		else for (int i = 0; i < n; i++) if (same( i, pn, in )) { j = i, kj = key[i]; break; }
		if (j < n) { if (!(kn < kj)) return; }                              // the hit is held with a key no larger
		else if (n == c) { if (!before( kn, in, pn, b, bound_inst(), bp )) return; j = c - 1; }
		else n++;
		// pos: the entries before j that come first (the buffer is sorted); entries pos .. j - 1 move up one slot, over slot j
		int pos = 0;
		if (REG)
		{
			#pragma unroll
			for (int i = 0; i < CAP; i++) if (i < j && before( key[i], inst_of( i ), prim[i], kn, in, pn )) pos++;
			#pragma unroll
			for (int i = CAP - 1; i > 0; i--)
				if (i > pos && i <= j) move( i, i - 1 );
			#pragma unroll
			for (int i = 0; i < CAP; i++)
				if (i == pos) put( i, kn, pn, tn, un, vn, in );
			if (n == c)
			{
				#pragma unroll
				for (int i = 0; i < CAP; i++) if (i == c - 1) take_bound( i );
			}
		}
		else
		{
			while (pos < j && before( key[pos], inst_of( pos ), prim[pos], kn, in, pn )) pos++;
			for (int i = j; i > pos; i--) move( i, i - 1 );
			put( pos, kn, pn, tn, un, vn, in );
			if (n == c) take_bound( c - 1 );
		}
	}

	// the k = c - 1 records { t, u, v, prim }, slots past n { tmax, 0, 0, CP_NO_PRIM }, and with INST the k instances to insts (past n
	// CP_NO_PRIM); returns n, the count saturated at k + 1
	__device__ __forceinline__ uint32_t store( float4* out, const float tmax, uint32_t* insts = nullptr ) const
	{
		const int k = c - 1;
		const float4 empty = make_float4( tmax, 0.0f, 0.0f, __uint_as_float( CP_NO_PRIM ) );
		if (REG)
		{
			#pragma unroll
			for (int i = 0; i < CAP; i++) if (i < k) out[i] = i < n ? make_float4( t[i], u[i], v[i], __uint_as_float( prim[i] ) ) : empty;
			if constexpr (INST)
			{
				#pragma unroll
				for (int i = 0; i < CAP; i++) if (i < k) insts[i] = i < n ? this->inst[i] : CP_NO_PRIM;
			}
		}
		else
		{
			for (int i = 0; i < k; i++) out[i] = i < n ? make_float4( t[i], u[i], v[i], __uint_as_float( prim[i] ) ) : empty;
			if constexpr (INST) for (int i = 0; i < k; i++) insts[i] = i < n ? this->inst[i] : CP_NO_PRIM;
		}
		return (uint32_t)n;
	}
};

// the k empty records of a ray that takes no walk (or of a view of another kind)
__device__ __forceinline__ void ah_store_empty( float4* out, const uint32_t k, const float tmax )
{
	for (uint32_t i = 0; i < k; i++) out[i] = make_float4( tmax, 0.0f, 0.0f, __uint_as_float( CP_NO_PRIM ) );
}
__device__ __forceinline__ void ah_store_empty( float4* out, uint32_t* insts, const uint32_t k, const float tmax )
{
	for (uint32_t i = 0; i < k; i++) out[i] = make_float4( tmax, 0.0f, 0.0f, __uint_as_float( CP_NO_PRIM ) ), insts[i] = CP_NO_PRIM;
}

// One ray's constants for the slab test: origin, direction, the stored rD, -(O*rD) (rounded product, as bvh2_walk) and the signs of D
struct AhRay
{
	float ox, oy, oz, dx, dy, dz, rdx, rdy, rdz, nrox, nroy, nroz;
	bool px, py, pz;
	__device__ __forceinline__ AhRay( const float ox_, const float oy_, const float oz_, const float dx_, const float dy_, const float dz_, const float rdx_,
		const float rdy_, const float rdz_ )
	{
		ox = ox_, oy = oy_, oz = oz_, dx = dx_, dy = dy_, dz = dz_, rdx = rdx_, rdy = rdy_, rdz = rdz_;
		nrox = -__fmul_rn( ox_, rdx_ ), nroy = -__fmul_rn( oy_, rdy_ ), nroz = -__fmul_rn( oz_, rdz_ );
		px = dx_ >= 0, py = dy_ >= 0, pz = dz_ >= 0;
	}
};

// The child pair of interior node (ref, 0) with path bound P: bvh2_pair_step's slab test with the lane's own signs (its OCT = -1 form),
// written beside it so that its callers keep their code, at the ray's own tmax.  A child is visited when reached and its bound is not above
// b.  Moves (ref, cnt, P) to the child to visit first (the nearer, the left one on ties) and pushes the other; false when neither is visited.
__device__ __forceinline__ bool ah_pair_step( const float4* __restrict__ nodes, const AhRay& r, const float tmax, const float b, uint32_t& ref,
	uint32_t& cnt, float& P, CpEntry* stack, int& sp )
{
	const float4* p = nodes + (size_t)ref * 2;
	const float4 a0 = __ldg( p ), a1 = __ldg( p + 1 ), b0 = __ldg( p + 2 ), b1 = __ldg( p + 3 );
	const float tx1a = __fmaf_rn( r.px ? a0.x : a1.x, r.rdx, r.nrox ), tx2a = __fmaf_rn( r.px ? a1.x : a0.x, r.rdx, r.nrox );
	const float ty1a = __fmaf_rn( r.py ? a0.y : a1.y, r.rdy, r.nroy ), ty2a = __fmaf_rn( r.py ? a1.y : a0.y, r.rdy, r.nroy );
	const float tz1a = __fmaf_rn( r.pz ? a0.z : a1.z, r.rdz, r.nroz ), tz2a = __fmaf_rn( r.pz ? a1.z : a0.z, r.rdz, r.nroz );
	const float tx1b = __fmaf_rn( r.px ? b0.x : b1.x, r.rdx, r.nrox ), tx2b = __fmaf_rn( r.px ? b1.x : b0.x, r.rdx, r.nrox );
	const float ty1b = __fmaf_rn( r.py ? b0.y : b1.y, r.rdy, r.nroy ), ty2b = __fmaf_rn( r.py ? b1.y : b0.y, r.rdy, r.nroy );
	const float tz1b = __fmaf_rn( r.pz ? b0.z : b1.z, r.rdz, r.nroz ), tz2b = __fmaf_rn( r.pz ? b1.z : b0.z, r.rdz, r.nroz );
	const float tmina = fmaxf( fmaxf( tx1a, ty1a ), fmaxf( tz1a, 0.0f ) ), tminb = fmaxf( fmaxf( tx1b, ty1b ), fmaxf( tz1b, 0.0f ) );
	const float tfara = fminf( fminf( tx2a, ty2a ), fminf( tz2a, tmax ) ), tfarb = fminf( fminf( tx2b, ty2b ), fminf( tz2b, tmax ) );
	const float Pa = fmaxf( P, tmina ), Pb = fmaxf( P, tminb );
	const bool va = tfara >= tmina && !(Pa > b), vb = tfarb >= tminb && !(Pb > b);
	const uint32_t refa = __float_as_uint( a0.w ), cnta = __float_as_uint( a1.w ), refb = __float_as_uint( b0.w ), cntb = __float_as_uint( b1.w );
	if (va && vb)
	{
		const bool swp = Pb < Pa; // nearer child first, the left one on ties
		ref = swp ? refb : refa, cnt = swp ? cntb : cnta, P = swp ? Pb : Pa;
		stack[sp++] = swp ? CpEntry{ refa, cnta, Pa } : CpEntry{ refb, cntb, Pb };
		return true;
	}
	if (va) { ref = refa, cnt = cnta, P = Pa; return true; }
	if (vb) { ref = refb, cnt = cntb, P = Pb; return true; }
	return false;
}

// The pop of a pruned walk: the next entry of the stack whose bound is not above b, false when none is left
__device__ __forceinline__ bool ah_pop( const CpEntry* stack, int& sp, const float b, uint32_t& ref, uint32_t& cnt, float& P )
{
	while (true)
	{
		if (sp == 0) return false;
		const CpEntry e = stack[--sp];
		if (!(e.P > b)) { ref = e.ref, cnt = e.cnt, P = e.P; return true; }
	}
}

// The multi-hit walk of one BVH2 subtree: from node (ref, cnt) reached with path bound P - its own box is not tested - into buf, with a
// caller-supplied stack deep enough for the tree (bvh2_walk's sizes); each accepted reference is a hit of instance `inst` (with INST).
template <int CAP, bool REG, bool INST> __device__ __forceinline__ void ah_subtree( AhBuffer<CAP, REG, INST>& buf, const float4* __restrict__ nodes,
	const float4* __restrict__ tris, uint32_t ref, uint32_t cnt, float P, const AhRay& r, const float tmax, const uint32_t inst, CpEntry* stack )
{
	int sp = 0;
	while (true)
	{
		if (cnt == 0)
		{
			if (ah_pair_step( nodes, r, tmax, buf.b, ref, cnt, P, stack, sp )) continue;
		}
		else
		{
			const float4* tp = tris + (size_t)ref * 3;
			for (uint32_t i = 0; i < cnt; i++, tp += 3)
			{
				const float4 v0 = __ldg( tp ), e1 = __ldg( tp + 1 ), e2 = __ldg( tp + 2 );
				float t, u, v;
				if (!mt_test( r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, v0, e1, e2, tmax, t, u, v ) || t != t) continue;
				const float key = fmaxf( t, P );
				if (!(key > buf.b)) buf.insert( key, __float_as_uint( v0.w ), t, u, v, inst );
			}
		}
		// pop, pruning again against the current bound
		if (!ah_pop( stack, sp, buf.b, ref, cnt, P )) return;
	}
}

// One ray's multi-hit walk from (ref, cnt) = the root, with a caller-supplied stack deep enough for the tree (bvh2_walk's sizes); k in
// 1 .. CAP - 1.  Writes the k records to out and returns the count.  A ray whose tmax is NaN or negative takes no walk: count 0.
template <int CAP, bool REG> __device__ __forceinline__ uint32_t ah_walk( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	uint32_t ref, uint32_t cnt, const float4& O, const float4& D, const float4& rD, const float tmax, const uint32_t k, float4* out, CpEntry* stack )
{
	if (!(tmax >= 0.0f)) { ah_store_empty( out, k, tmax ); return 0; }
	AhBuffer<CAP, REG> buf;
	buf.init( (int)k + 1 );
	ah_subtree( buf, nodes, tris, ref, cnt, 0.0f, AhRay( O.x, O.y, O.z, D.x, D.y, D.z, rD.x, rD.y, rD.z ), tmax, 0u, stack );
	return buf.store( out, tmax );
}

// One ray's multi-hit walk over a TLAS of BVH-layout BLASses (DESIGN.md 4.14, two levels): the TLAS from (root_ref, root_count) as a BVH2
// with the world ray's stored rD; per instance of a reached TLAS leaf: skip unless inst.mask & ray.mask; the ray in BLAS space as tlas_trace
// transforms it (inst_transform, rD' = safercp( D' )); the BLAS from its root, reached with the leaf's path bound, by ah_subtree with the
// same tmax.  A hit is an ( instance, prim ) pair.  stack: TLAS_STACK entries - a TLAS of depth below 64 leaves at most one entry per level
// pending, plus the rest of the current leaf; bstack: TBVH_STACK, the two-level walks' BLAS limit.  Writes the k records to out, the k
// instances to insts, and returns the count.
template <int CAP, bool REG> __device__ __forceinline__ uint32_t ah_walk_tlas( const float4* __restrict__ nodes, const uint32_t* __restrict__ prim_idx,
	const TlasInst* __restrict__ inst, const BlasRef* __restrict__ blas, uint32_t ref, uint32_t cnt, const float4& O, const float4& D, const float4& rD,
	const float tmax, const uint32_t k, float4* out, uint32_t* insts, CpEntry* stack, CpEntry* bstack )
{
	if (!(tmax >= 0.0f)) { ah_store_empty( out, insts, k, tmax ); return 0; }
	AhBuffer<CAP, REG, true> buf;
	buf.init( (int)k + 1 );
	const AhRay r( O.x, O.y, O.z, D.x, D.y, D.z, rD.x, rD.y, rD.z );
	const uint32_t rmask = __float_as_uint( O.w );
	int sp = 0;
	float P = 0.0f;
	while (true)
	{
		if (cnt == 0)
		{
			if (ah_pair_step( nodes, r, tmax, buf.b, ref, cnt, P, stack, sp )) continue;
		}
		else
		{
			// the leaf's first instance now, the rest of the leaf as a stack entry of the same bound: nothing of the TLAS walk but its stack
			// stays live across the BLAS walk
			if (cnt > 1) stack[sp++] = CpEntry{ ref + 1, cnt - 1, P };
			const uint32_t instIdx = __ldg( prim_idx + ref );
			const float4* ip = (const float4*)(inst + instIdx);
			const float4 meta = __ldg( ip + 4 );
			if (__float_as_uint( meta.y ) & rmask)
			{
				float tox, toy, toz, tdx, tdy, tdz;
				inst_transform( __ldg( ip ), __ldg( ip + 1 ), __ldg( ip + 2 ), __ldg( ip + 3 ), r.ox, r.oy, r.oz, r.dx, r.dy, r.dz, tox, toy, toz, tdx, tdy, tdz );
				const BlasRef B = blas[__float_as_uint( meta.x )];
				ah_subtree( buf, B.trav, B.tris, B.root_ref, B.root_count, P, AhRay( tox, toy, toz, tdx, tdy, tdz, safercp( tdx ), safercp( tdy ), safercp( tdz ) ),
					tmax, instIdx, bstack );
			}
		}
		if (!ah_pop( stack, sp, buf.b, ref, cnt, P )) return buf.store( out, tmax, insts );
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
