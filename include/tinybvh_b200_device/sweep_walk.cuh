// include/tinybvh_b200_device/sweep_walk.cuh - the sphere-cast walk over the BVH2: the first time a sphere moving along a line touches a
// triangle, its contact point, and whether any triangle is touched.  Shared by the library's kernel (sphere_cast.cu: k_sphere_cast) and the
// device functions of include/tinybvh_b200_device.cuh.
//
// Semantics are the engine's own (DESIGN.md 4.16), restated on the host by tests/sweep_oracle.c in the same fp32 operation order.  A query
// is { cx, cy, cz, r }, { dx, dy, dz, tmax }: the centre at t is c + t D, t in [0, tmax]; the sphere touches a triangle at t when the
// distance from c + t D to the closed triangle is <= r.
//  * per triangle (sc_triangle): contact at t = 0 with cp_triangle's (u, v) when cp_triangle( c )'s d2_raw <= r^2 (4.9's test); else the
//    least of the face, edge (AB, AC, BC) and vertex (A, B, C) times in [0, tmax], ties in that order;
//  * per node: the slab test of the line c + t D on [0, tmax] against the child box inflated by r (rounded outward); P( child ) =
//    fmaxf( P( parent ), tmin ), P( root ) = 0, the root box untested; a DAG leaf is walked once per path, so it takes its least P;
//  * a reference (leaf, triangle) in contact at t_tri has key fmaxf( t_tri, P( leaf ) ); the result is the smallest ( key, prim ),
//    whatever the visiting order, so a node with P > best is pruned exactly.
#pragma once
#include "closest_walk.cuh"

namespace tbvh
{

// |x| <= FLT_MAX: neither NaN nor infinite
__device__ __forceinline__ bool sc_finite( const float x ) { return fabsf( x ) <= 3.40282347e38f; }

// whether a query takes a walk: c and D finite, r finite and >= 0, tmax >= 0 (+inf allowed)
__device__ __forceinline__ bool sc_query_ok( const float4& q0, const float4& q1 )
{
	return sc_finite( q0.x ) && sc_finite( q0.y ) && sc_finite( q0.z ) && sc_finite( q0.w ) && q0.w >= 0.0f
		&& sc_finite( q1.x ) && sc_finite( q1.y ) && sc_finite( q1.z ) && q1.w >= 0.0f;
}

// The smaller root of a t^2 + 2 b t + c = 0 for a centre that starts outside (c > 0) and moves inward (b < 0), in the form without
// cancellation: c / (-b + sqrt( disc )), disc = b^2 - a c as the caller computes it without cancellation.  false when the centre starts
// inside, moves away or passes by (disc < 0).
__device__ __forceinline__ bool sc_root( const float b, const float c, const float disc, float& t )
{
	if (!(c > 0.0f) || !(b < 0.0f) || !(disc >= 0.0f)) return false;
	t = __fdiv_rn( c, __fadd_rn( -b, __fsqrt_rn( disc ) ) );
	return true;
}

// The cylinder of radius R around the edge A + s ev, s in [0, 1], met by the centre m0 + t D (m0 = the centre at 0 minus A): with
// dx = D x ev and mx = m0 x ev, |mx + t dx|^2 = R^2 |ev|^2 is  a = dx.dx, b = dx.mx, c = mx.mx - R^2 ev.ev, and by Lagrange's identity
// b^2 - a c = ev.ev ( a R^2 - g^2 ), g = D . mx (the distance between the two lines times |dx|): no difference of the large terms b^2 and
// a c, which would cost the bits of (distance to the edge / R)^2.  The root counts when the edge parameter ((m0 + t D) . ev) / ev.ev at it
// lies in [0, 1]; a zero-length edge has none.
__device__ __forceinline__ bool sc_edge( const float mx0, const float my0, const float mz0, const float evx, const float evy, const float evz,
	const float Dx, const float Dy, const float Dz, const float RR, float& t, float& s )
{
	const float ee = cp_dot( evx, evy, evz, evx, evy, evz );
	if (!(ee > 0.0f)) return false;
	float ax, ay, az, bx, by, bz;
	cp_cross( Dx, Dy, Dz, evx, evy, evz, ax, ay, az );
	cp_cross( mx0, my0, mz0, evx, evy, evz, bx, by, bz );
	const float a = cp_dot( ax, ay, az, ax, ay, az ), g = cp_dot( Dx, Dy, Dz, bx, by, bz );
	const float c = __fmaf_rn( -RR, ee, cp_dot( bx, by, bz, bx, by, bz ) );
	const float disc = __fmul_rn( __fmaf_rn( -g, g, __fmul_rn( a, RR ) ), ee );
	if (!sc_root( cp_dot( ax, ay, az, bx, by, bz ), c, disc, t )) return false;
	const float num = cp_dot( __fmaf_rn( t, Dx, mx0 ), __fmaf_rn( t, Dy, my0 ), __fmaf_rn( t, Dz, mz0 ), evx, evy, evz );
	if (!(num >= 0.0f && num <= ee)) return false;
	s = __fdiv_rn( num, ee );
	return true;
}

// the sphere around the vertex V met by the centre m0 + t D (m0 = the centre at 0 minus V): |m0 + t D|^2 = R^2, a = D.D, b = D.m0,
// c = m0.m0 - R^2 and b^2 - a c = a R^2 - |D x m0|^2 (Lagrange's identity, as for the edges)
__device__ __forceinline__ bool sc_vertex( const float mx0, const float my0, const float mz0, const float Dx, const float Dy, const float Dz,
	const float DD, const float R, const float RR, float& t )
{
	float hx, hy, hz;
	cp_cross( Dx, Dy, Dz, mx0, my0, mz0, hx, hy, hz );
	const float disc = __fsub_rn( __fmul_rn( DD, RR ), cp_dot( hx, hy, hz, hx, hy, hz ) );
	return sc_root( cp_dot( Dx, Dy, Dz, mx0, my0, mz0 ), __fmaf_rn( -R, R, cp_dot( mx0, my0, mz0, mx0, my0, mz0 ) ), disc, t );
}

// First contact of the sphere (c, r) moving along c + t D, t in [0, tmax], with the triangle of the leaf record (v0 | prim, e1, e2).
// Returns whether it touches; then t is the time and (u, v) the contact point v0 + u e1 + v e2.
//  * t = 0 when cp_triangle( c )'s d2_raw <= r^2, with its (u, v);
//  * else, on c - v0, e1, e2 and r scaled by the power of two of their largest component (cp_pow2) and D by its own, the least candidate
//    time tau, ties in the order face, AB, AC, BC, A, B, C, and t = tau 2^(e - f) (2^e, 2^f the two inverse factors), kept when <= tmax.
//    The face is taken at K, the corner opposite the longest edge (ties: A, then B), with a and b its two edges oriented so that
//    n = a x b = e1 x e2.  There the cross product is well conditioned: the angle at K is the largest, so a long thin triangle gets its
//    normal to full precision whichever corner is v0.  It counts while |n|^2 > 2^-22 |a| |b| L^2 (L the longest edge): n's components
//    each carry about 2^-24 |a| |b| of rounding, so its direction is off by about 2^-23 |a| |b| / |n| and the plane strays by that times
//    L across the triangle; below the bound this exceeds the width |n| / L, and the edges, which lie within the width of every point of
//    the triangle, answer at least as well (only flat caps, all of whose angles are near 0 or 180 degrees, fall below it).  The centre
//    starting farther than R from the plane and moving toward it: tau = (|h0| - R |n|) / -(s hd), h0 = (P - K) . n, hd = D . n, s the
//    sign of h0; it counts when the weights of the centre X at tau along a and b, alpha = (((X - K) x b) . n) / |n|^2 and
//    beta = ((a x (X - K)) . n) / |n|^2 (cp_triangle's cross-product form, unclamped), have alpha, beta >= 0 and alpha + beta <= 1; they
//    give (u, v) = (alpha, beta) at A, (1 - alpha - beta, alpha) at B, (beta, 1 - alpha - beta) at C.  The centre stands for the
//    touching point X - s R n / |n|: the two differ along n, which the two triple products do not see.
//  * Scaling the query and the mesh by 2^k, or D by 2^m and tmax by 2^-m, scales every intermediate by an exact power of two (or not at
//    all), so the result scales exactly wherever nothing over- or underflows.
__device__ __forceinline__ bool sc_triangle( const float4& q0, const float4& q1, const float4& v0, const float4& e1r, const float4& e2r,
	float& t, float& u, float& v )
{
	if (cp_triangle( q0.x, q0.y, q0.z, v0, e1r, e2r, u, v ) <= __fmul_rn( q0.w, q0.w )) { t = 0.0f; return true; }
	const float rx = __fsub_rn( q0.x, v0.x ), ry = __fsub_rn( q0.y, v0.y ), rz = __fsub_rn( q0.z, v0.z );
	const float m = fmaxf( fmaxf( fmaxf( fmaxf( fabsf( rx ), fabsf( ry ) ), fmaxf( fabsf( rz ), fabsf( e1r.x ) ) ), fmaxf( fmaxf( fabsf( e1r.y ), fabsf( e1r.z ) ),
		fmaxf( fabsf( e2r.x ), fabsf( e2r.y ) ) ) ), fmaxf( fabsf( e2r.z ), q0.w ) );
	float inv, invd;
	const float s = cp_pow2( m, inv ), sd = cp_pow2( fmaxf( fmaxf( fabsf( q1.x ), fabsf( q1.y ) ), fabsf( q1.z ) ), invd );
	const float Px = __fmul_rn( rx, s ), Py = __fmul_rn( ry, s ), Pz = __fmul_rn( rz, s ), R = __fmul_rn( q0.w, s ), RR = __fmul_rn( R, R );
	const float E1x = __fmul_rn( e1r.x, s ), E1y = __fmul_rn( e1r.y, s ), E1z = __fmul_rn( e1r.z, s );
	const float E2x = __fmul_rn( e2r.x, s ), E2y = __fmul_rn( e2r.y, s ), E2z = __fmul_rn( e2r.z, s );
	const float Dx = __fmul_rn( q1.x, sd ), Dy = __fmul_rn( q1.y, sd ), Dz = __fmul_rn( q1.z, sd );
	float best = 0.0f, bu = 0.0f, bv = 0.0f, tc, w;
	bool found = false;
	// face, at the corner K opposite the longest edge
	const float BCx = __fsub_rn( E2x, E1x ), BCy = __fsub_rn( E2y, E1y ), BCz = __fsub_rn( E2z, E1z );
	const float lab = cp_dot( E1x, E1y, E1z, E1x, E1y, E1z ), lac = cp_dot( E2x, E2y, E2z, E2x, E2y, E2z ), lbc = cp_dot( BCx, BCy, BCz, BCx, BCy, BCz );
	const int K = (lbc >= lab && lbc >= lac) ? 0 : lac >= lab ? 1 : 2;
	// K = A: a = e1, b = e2; K = B: a = BC, b = -e1; K = C: a = -e2, b = -BC
	const float ax = K == 0 ? E1x : K == 1 ? BCx : -E2x, ay = K == 0 ? E1y : K == 1 ? BCy : -E2y, az = K == 0 ? E1z : K == 1 ? BCz : -E2z;
	const float bx = K == 0 ? E2x : K == 1 ? -E1x : -BCx, by = K == 0 ? E2y : K == 1 ? -E1y : -BCy, bz = K == 0 ? E2z : K == 1 ? -E1z : -BCz;
	const float la = K == 0 ? lab : K == 1 ? lbc : lac, lb = K == 0 ? lac : K == 1 ? lab : lbc, LL = K == 0 ? lbc : K == 1 ? lac : lab;
	const float Kx = K == 0 ? Px : K == 1 ? __fsub_rn( Px, E1x ) : __fsub_rn( Px, E2x );
	const float Ky = K == 0 ? Py : K == 1 ? __fsub_rn( Py, E1y ) : __fsub_rn( Py, E2y );
	const float Kz = K == 0 ? Pz : K == 1 ? __fsub_rn( Pz, E1z ) : __fsub_rn( Pz, E2z );
	float nx, ny, nz;
	cp_cross( ax, ay, az, bx, by, bz, nx, ny, nz );
	const float nn = cp_dot( nx, ny, nz, nx, ny, nz );
	if (nn > __fmul_rn( __fmul_rn( __fsqrt_rn( __fmul_rn( la, lb ) ), LL ), 0x1p-22f ))
	{
		float h0 = cp_dot( Kx, Ky, Kz, nx, ny, nz ), hd = cp_dot( Dx, Dy, Dz, nx, ny, nz );
		if (h0 < 0.0f) h0 = -h0, hd = -hd;
		const float num = __fmaf_rn( -R, __fsqrt_rn( nn ), h0 );
		if (num > 0.0f && hd < 0.0f)
		{
			tc = __fdiv_rn( num, -hd );
			const float Xx = __fmaf_rn( tc, Dx, Kx ), Xy = __fmaf_rn( tc, Dy, Ky ), Xz = __fmaf_rn( tc, Dz, Kz );
			float fx, fy, fz, gx, gy, gz;
			cp_cross( Xx, Xy, Xz, bx, by, bz, fx, fy, fz );
			cp_cross( ax, ay, az, Xx, Xy, Xz, gx, gy, gz );
			const float in = __fdiv_rn( 1.0f, nn );
			const float al = __fmul_rn( cp_dot( fx, fy, fz, nx, ny, nz ), in ), be = __fmul_rn( cp_dot( gx, gy, gz, nx, ny, nz ), in );
			if (al >= 0.0f && be >= 0.0f && __fadd_rn( al, be ) <= 1.0f)
			{
				const float w0 = __fsub_rn( __fsub_rn( 1.0f, al ), be );
				best = tc, found = true;
				bu = K == 0 ? al : K == 1 ? w0 : be;
				bv = K == 0 ? be : K == 1 ? al : w0;
			}
		}
	}
	// edges AB, AC (from v0) and BC (from v1)
	if (sc_edge( Px, Py, Pz, E1x, E1y, E1z, Dx, Dy, Dz, RR, tc, w ) && (!found || tc < best)) best = tc, bu = w, bv = 0.0f, found = true;
	if (sc_edge( Px, Py, Pz, E2x, E2y, E2z, Dx, Dy, Dz, RR, tc, w ) && (!found || tc < best)) best = tc, bu = 0.0f, bv = w, found = true;
	const float Bx = __fsub_rn( Px, E1x ), By = __fsub_rn( Py, E1y ), Bz = __fsub_rn( Pz, E1z );
	if (sc_edge( Bx, By, Bz, BCx, BCy, BCz, Dx, Dy, Dz, RR, tc, w ) && (!found || tc < best))
		best = tc, bu = __fsub_rn( 1.0f, w ), bv = w, found = true;
	// vertices A, B, C
	const float DD = cp_dot( Dx, Dy, Dz, Dx, Dy, Dz );
	if (sc_vertex( Px, Py, Pz, Dx, Dy, Dz, DD, R, RR, tc ) && (!found || tc < best)) best = tc, bu = 0.0f, bv = 0.0f, found = true;
	if (sc_vertex( Bx, By, Bz, Dx, Dy, Dz, DD, R, RR, tc ) && (!found || tc < best)) best = tc, bu = 1.0f, bv = 0.0f, found = true;
	if (sc_vertex( __fsub_rn( Px, E2x ), __fsub_rn( Py, E2y ), __fsub_rn( Pz, E2z ), Dx, Dy, Dz, DD, R, RR, tc ) && (!found || tc < best))
		best = tc, bu = 0.0f, bv = 1.0f, found = true;
	if (!found) return false;
	t = __fmul_rn( __fmul_rn( best, inv ), sd );
	if (!(t <= q1.w)) return false;
	u = bu, v = bv;
	return true;
}

// The slab test of the line c + t D, t in [0, tmax], against the box [bmin - r, bmax + r] (rounded outward): tmin = the largest entry
// time and 0, tmax' = the smallest exit time and tmax; passes when tmin <= tmax'.  Per axis the times are (plane - c) / D, divided
// exactly rather than multiplied by a reciprocal; an axis with D = +-0 passes for all t when c lies in the inflated slab and for none
// otherwise.
__device__ __forceinline__ void sc_axis( const float lo, const float hi, const float c, const float d, float& tn, float& tf )
{
	if (d == 0.0f)
	{
		const bool in = lo <= c && c <= hi;
		tn = in ? -INFINITY : INFINITY, tf = in ? INFINITY : -INFINITY;
		return;
	}
	const float a = __fdiv_rn( __fsub_rn( lo, c ), d ), b = __fdiv_rn( __fsub_rn( hi, c ), d );
	tn = fminf( a, b ), tf = fmaxf( a, b );
}
__device__ __forceinline__ bool sc_box( const float4& bmin, const float4& bmax, const float4& q0, const float4& q1, float& tmin )
{
	float nx, fx, ny, fy, nz, fz;
	sc_axis( __fsub_rd( bmin.x, q0.w ), __fadd_ru( bmax.x, q0.w ), q0.x, q1.x, nx, fx );
	sc_axis( __fsub_rd( bmin.y, q0.w ), __fadd_ru( bmax.y, q0.w ), q0.y, q1.y, ny, fy );
	sc_axis( __fsub_rd( bmin.z, q0.w ), __fadd_ru( bmax.z, q0.w ), q0.z, q1.z, nz, fz );
	tmin = fmaxf( fmaxf( fmaxf( nx, ny ), nz ), 0.0f );
	return tmin <= fminf( fminf( fminf( fx, fy ), fz ), q1.w );
}

// One query's walk from (ref, cnt) = the root with a caller-supplied stack deep enough for the tree (bvh2_walk's sizes), on CpEntry
// records whose P is the path bound in t.  Closest (ANY = false): best / bt / bprim / bu / bv enter as (tmax, tmax, CP_NO_PRIM, 0, 0) and
// leave as the smallest ( key, prim ) with its t_tri.  ANY: returns true at the first reached reference in contact.
template <bool ANY> __device__ __forceinline__ bool sc_walk( const float4* __restrict__ nodes, const float4* __restrict__ tris, uint32_t ref, uint32_t cnt,
	const float4& q0, const float4& q1, float& best, float& bt, uint32_t& bprim, float& bu, float& bv, CpEntry* stack )
{
	int sp = 0;
	float P = 0.0f;
	while (true)
	{
		if (cnt == 0)
		{
			const float4* q = nodes + (size_t)ref * 2;
			const float4 a0 = __ldg( q ), a1 = __ldg( q + 1 ), b0 = __ldg( q + 2 ), b1 = __ldg( q + 3 );
			float ta, tb;
			const bool ha = sc_box( a0, a1, q0, q1, ta ), hb = sc_box( b0, b1, q0, q1, tb );
			const float Pa = fmaxf( P, ta ), Pb = fmaxf( P, tb );
			const bool va = ha && !(Pa > best), vb = hb && !(Pb > best); // strict: a subtree at exactly `best` may still hold a smaller prim
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
			for (uint32_t k = 0; k < cnt; k++, tp += 3)
			{
				const float4 v0 = __ldg( tp ), e1 = __ldg( tp + 1 ), e2 = __ldg( tp + 2 );
				float t, u, v;
				if (!sc_triangle( q0, q1, v0, e1, e2, t, u, v )) continue;
				if (ANY) return true;
				const float key = fmaxf( t, P );
				const uint32_t prim = __float_as_uint( v0.w );
				if (key < best || (key == best && prim < bprim)) best = key, bt = t, bprim = prim, bu = u, bv = v;
			}
		}
		// pop, pruning again against the current best
		while (true)
		{
			if (sp == 0) return false;
			const CpEntry e = stack[--sp];
			if (!(e.P > best)) { ref = e.ref, cnt = e.cnt, P = e.P; break; }
		}
	}
}

// the result record of one sphere cast: { t_tri, u, v, prim }, or { tmax, 0, 0, CP_NO_PRIM } when nothing is touched in [0, tmax]
template <int STACKN> __device__ __forceinline__ float4 sc_cast( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	const uint32_t root_ref, const uint32_t root_count, const float4& q0, const float4& q1 )
{
	if (!sc_query_ok( q0, q1 )) return make_float4( q1.w, 0.0f, 0.0f, __uint_as_float( CP_NO_PRIM ) );
	float best = q1.w, bt = q1.w, bu = 0.0f, bv = 0.0f;
	uint32_t bprim = CP_NO_PRIM;
	CpEntry stack[STACKN];
	sc_walk<false>( nodes, tris, root_ref, root_count, q0, q1, best, bt, bprim, bu, bv, stack );
	if (bprim == CP_NO_PRIM) return make_float4( q1.w, 0.0f, 0.0f, __uint_as_float( CP_NO_PRIM ) );
	return make_float4( bt, bu, bv, __uint_as_float( bprim ) );
}

// the blocked bit of one sphere cast: some reached reference is touched in [0, tmax]
template <int STACKN> __device__ __forceinline__ bool sc_blocked( const float4* __restrict__ nodes, const float4* __restrict__ tris,
	const uint32_t root_ref, const uint32_t root_count, const float4& q0, const float4& q1 )
{
	if (!sc_query_ok( q0, q1 )) return false;
	float best = q1.w, bt = q1.w, bu = 0.0f, bv = 0.0f;
	uint32_t bprim = CP_NO_PRIM;
	CpEntry stack[STACKN];
	return sc_walk<true>( nodes, tris, root_ref, root_count, q0, q1, best, bt, bprim, bu, bv, stack );
}

} // namespace tbvh
