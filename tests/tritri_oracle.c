/* tests/tritri_oracle.c - the oracle of tbvh_mesh_overlap_pairs / tbvh_mesh_overlap_bits.  TEST INFRASTRUCTURE ONLY.
 *
 * The engine's triangle-triangle overlap (tinybvh_b200/csrc/mesh_overlap.cu) follows its own definition, DESIGN.md §4.12; this file
 * restates it on the host in the same fp32 operation order (every fused pair written as fmaf, compiled with contraction off by
 * tests/tritri_oracle.py):
 *  - orc_tt_pairs:       the pair test (self = 0) or the self rules (self = 1) over arrays of triangle pairs;
 *  - orc_overlap_all:    every (A triangle, B triangle) pair, no tree;
 *  - orc_overlap_tree:   every (A triangle, B reference) pair the tree reaches: brute = 1 marks every slot whose whole path overlaps the
 *                        triangle's box, no pruning (the definition); brute = 0 is the pruned walk the kernel runs;
 *  - both tree forms give per-triangle counts and, on a second call with offsets, the raw keys (i << 32) | j in walk order, and the bits
 *    form (self: every j != i; the first pair ends the walk).
 * Trees are the reference's 32-byte node arrays (node 0 the root, node 1 unused, children paired at leftFirst); vertices are float4,
 * three per primitive.
 */
#include <math.h>
#include <float.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float mn[3]; uint32_t lf; float mx[3]; uint32_t cnt; } node32;

static float dot3( const float* a, const float* b ) { return fmaf( a[2], b[2], fmaf( a[1], b[1], a[0] * b[0] ) ); }
static void sub3( const float* a, const float* b, float* r ) { r[0] = a[0] - b[0], r[1] = a[1] - b[1], r[2] = a[2] - b[2]; }
static void cross3( const float* a, const float* b, float* r )
{
	r[0] = a[1] * b[2] - a[2] * b[1];
	r[1] = a[2] * b[0] - a[0] * b[2];
	r[2] = a[0] * b[1] - a[1] * b[0];
}
/* the side of x against the plane through o with normal n: ( x - o ) . n */
static float side( const float* x, const float* o, const float* n ) { float d[3]; sub3( x, o, d ); return dot3( d, n ); }
/* [b - a, c - a, d - a]: ( d - a ) . ( ( b - a ) x ( c - a ) ) */
static float orient3d( const float* a, const float* b, const float* c, const float* d )
{
	float u[3], v[3], n[3];
	sub3( b, a, u ), sub3( c, a, v ), cross3( u, v, n );
	return side( d, a, n );
}
/* ( b - a ) x ( c - a ) on the axes (i, j) */
static float orient2d( const float* a, const float* b, const float* c, const int i, const int j )
{
	return (b[i] - a[i]) * (c[j] - a[j]) - (b[j] - a[j]) * (c[i] - a[i]);
}
/* the projection that drops the axis of n's largest component: x when |nx| > |nz| and |nx| >= |ny|, else y when |ny| > |nz| and
 * |ny| >= |nx|, else z */
static void axes( const float* n, int* i, int* j )
{
	const float ax = fabsf( n[0] ), ay = fabsf( n[1] ), az = fabsf( n[2] );
	if (ax > az && ax >= ay) *i = 1, *j = 2;
	else if (ay > az && ay >= ax) *i = 2, *j = 0;
	else *i = 0, *j = 1;
}
static int same3( const float a, const float b, const float c ) { return (a > 0.0f && b > 0.0f && c > 0.0f) || (a < 0.0f && b < 0.0f && c < 0.0f); }
static int opp( const float s, const float x ) { return s > 0.0f ? x < 0.0f : s < 0.0f ? x > 0.0f : 0; }

/* the line through edge (a, b) of a triangle whose third corner is c separates the points y[0 .. k): all strictly on the far side */
static int sep2( const float* a, const float* b, const float* c, const float* const* y, const int k, const int i, const int j )
{
	const float s = orient2d( a, b, c, i, j );
	for (int t = 0; t < k; t++) if (!opp( s, orient2d( a, b, y[t], i, j ) )) return 0;
	return 1;
}

/* closed segment (a, b) against the closed triangle X, sa / sb the sides of a and b against X's plane, n X's normal */
static int seg_tri( const float* a, const float* b, const float sa, const float sb, const float* const* X, const float* n )
{
	if ((sa > 0.0f && sb > 0.0f) || (sa < 0.0f && sb < 0.0f)) return 0;
	if (sa == 0.0f && sb == 0.0f)
	{
		int i, j;
		axes( n, &i, &j );
		const float* ab[2] = { a, b };
		for (int e = 0; e < 3; e++) if (sep2( X[e], X[(e + 1) % 3], X[(e + 2) % 3], ab, 2, i, j )) return 0;
		return !same3( orient2d( a, b, X[0], i, j ), orient2d( a, b, X[1], i, j ), orient2d( a, b, X[2], i, j ) );
	}
	if (sa == 0.0f || sb == 0.0f)
	{
		/* one end on the plane: the segment meets it there only, so that point against X in the projection */
		int i, j;
		axes( n, &i, &j );
		const float* p[1] = { sa == 0.0f ? a : b };
		for (int e = 0; e < 3; e++) if (sep2( X[e], X[(e + 1) % 3], X[(e + 2) % 3], p, 1, i, j )) return 0;
		return 1;
	}
	const float o1 = orient3d( a, b, X[0], X[1] ), o2 = orient3d( a, b, X[1], X[2] ), o3 = orient3d( a, b, X[2], X[0] );
	return (o1 >= 0.0f && o2 >= 0.0f && o3 >= 0.0f) || (o1 <= 0.0f && o2 <= 0.0f && o3 <= 0.0f);
}

static uint32_t f2key( const float f ) { uint32_t u; memcpy( &u, &f, 4 ); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }

/* closest_walk.cuh cp_pow2 */
static float pow2( const float m )
{
	uint32_t f, c;
	memcpy( &f, &m, 4 );
	f >>= 23;
	if (!(m > 0.0f) || f == 255u) return 1.0f;
	c = f < 1u ? 1u : f > 253u ? 253u : f;
	const uint32_t sb = (254u - c) << 23;
	float s;
	memcpy( &s, &sb, 4 );
	return s;
}

/* tri_pair.cuh mo_pos: the corners read as x + 0 (-0 becomes +0, every other value keeps its bits) */
static void pos9( const float* x, float* r ) { for (int k = 0; k < 9; k++) r[k] = x[k] + 0.0f; }

/* tri_pair.cuh mo_test: a and b are three corners (9 floats) each; self = 1 applies the self rules */
int orc_tt( const float* a_in, const float* b_in, const int self )
{
	float a[9], b[9];
	pos9( a_in, a ), pos9( b_in, b );
	for (int k = 0; k < 9; k++) if (!(fabsf( a[k] ) <= FLT_MAX) || !(fabsf( b[k] ) <= FLT_MAX)) return 0;
	/* the closed boxes of the input corners */
	for (int k = 0; k < 3; k++)
		if (fmaxf( fmaxf( a[k], a[3 + k] ), a[6 + k] ) < fminf( fminf( b[k], b[3 + k] ), b[6 + k] ) ||
			fmaxf( fmaxf( b[k], b[3 + k] ), b[6 + k] ) < fminf( fminf( a[k], a[3 + k] ), a[6 + k] )) return 0;
	/* canonical order: the triangle whose nine ordered keys are lexicographically smaller is T */
	int swap = 0;
	for (int k = 0; k < 9; k++) { const uint32_t ka = f2key( a[k] ), kb = f2key( b[k] ); if (ka != kb) { swap = kb < ka; break; } }
	const float* rt = swap ? b : a, * ru = swap ? a : b;
	/* T's v0 subtracted from all six corners, then the power of two of their largest magnitude */
	float P[6][3], m = 0.0f;
	for (int c = 0; c < 6; c++) for (int k = 0; k < 3; k++) { P[c][k] = (c < 3 ? rt : ru)[(c % 3) * 3 + k] - rt[k]; m = fmaxf( m, fabsf( P[c][k] ) ); }
	const float s = pow2( m );
	for (int c = 0; c < 6; c++) for (int k = 0; k < 3; k++) P[c][k] = P[c][k] * s;
	const float* T[3] = { P[0], P[1], P[2] }, * U[3] = { P[3], P[4], P[5] };
	float e1[3], e2[3], nT[3], nU[3];
	sub3( T[1], T[0], e1 ), sub3( T[2], T[0], e2 ), cross3( e1, e2, nT );
	sub3( U[1], U[0], e1 ), sub3( U[2], U[0], e2 ), cross3( e1, e2, nU );
	if ((nT[0] == 0.0f && nT[1] == 0.0f && nT[2] == 0.0f) || (nU[0] == 0.0f && nU[1] == 0.0f && nU[2] == 0.0f)) return 0;
	float dU[3], dT[3];
	for (int c = 0; c < 3; c++) dU[c] = side( U[c], T[0], nT ), dT[c] = side( T[c], U[0], nU );
	if (self)
	{
		/* shared corners: equal positions as values (-0 equals +0, NaN equals nothing) */
		int shared = 0, ta = 0, ub = 0, tm = 0, um = 0;
		for (int x = 0; x < 3; x++)
			for (int y = 0; y < 3; y++)
				if (rt[x * 3] == ru[y * 3] && rt[x * 3 + 1] == ru[y * 3 + 1] && rt[x * 3 + 2] == ru[y * 3 + 2])
				{
					if (!(tm >> x & 1)) shared++, ta = x, ub = y;
					tm |= 1 << x, um |= 1 << y;
					break;
				}
		if (shared == 3) return 1;
		if (shared == 1)
			return seg_tri( T[(ta + 1) % 3], T[(ta + 2) % 3], dT[(ta + 1) % 3], dT[(ta + 2) % 3], U, nU ) ||
				seg_tri( U[(ub + 1) % 3], U[(ub + 2) % 3], dU[(ub + 1) % 3], dU[(ub + 2) % 3], T, nT );
		if (shared == 2)
		{
			for (int c = 0; c < 3; c++) if (dU[c] != 0.0f || dT[c] != 0.0f) return 0;
			/* the corners of T not shared and not: t3 the third of T, u3 the third of U; the shared edge (t1, t2) in T's order */
			const int t3 = (tm & 1) == 0 ? 0 : (tm & 2) == 0 ? 1 : 2, u3 = (um & 1) == 0 ? 0 : (um & 2) == 0 ? 1 : 2;
			int i, j;
			axes( nT, &i, &j );
			const float s1 = orient2d( T[(t3 + 1) % 3], T[(t3 + 2) % 3], T[t3], i, j ), s2 = orient2d( T[(t3 + 1) % 3], T[(t3 + 2) % 3], U[u3], i, j );
			return (s1 > 0.0f && s2 > 0.0f) || (s1 < 0.0f && s2 < 0.0f);
		}
	}
	if (same3( dU[0], dU[1], dU[2] ) || same3( dT[0], dT[1], dT[2] )) return 0;
	if (dU[0] == 0.0f && dU[1] == 0.0f && dU[2] == 0.0f)
	{
		/* coplanar: separated exactly when the line of some edge of either triangle has the other strictly on its far side */
		int i, j;
		axes( nT, &i, &j );
		for (int e = 0; e < 3; e++)
			if (sep2( T[e], T[(e + 1) % 3], T[(e + 2) % 3], U, 3, i, j ) || sep2( U[e], U[(e + 1) % 3], U[(e + 2) % 3], T, 3, i, j )) return 0;
		return 1;
	}
	/* two closed triangles not in one plane meet exactly when an edge of one meets the other */
	for (int e = 0; e < 3; e++)
	{
		if (seg_tri( T[e], T[(e + 1) % 3], dT[e], dT[(e + 1) % 3], U, nU )) return 1;
		if (seg_tri( U[e], U[(e + 1) % 3], dU[e], dU[(e + 1) % 3], T, nT )) return 1;
	}
	return 0;
}

/* orc_tt over n pairs: a, b are n x 9 floats */
void orc_tt_pairs( const float* a, const float* b, const uint64_t n, const int self, uint8_t* out )
{
	for (uint64_t k = 0; k < n; k++) out[k] = (uint8_t)orc_tt( a + k * 9, b + k * 9, self );
}

static void corners( const float* verts, const uint32_t p, float* t )
{
	for (int c = 0; c < 3; c++) for (int k = 0; k < 3; k++) t[c * 3 + k] = verts[((size_t)p * 3 + c) * 4 + k];
}

/* the closed box test in fp32 */
static int box_hit( const float* mn, const float* mx, const node32* n )
{
	return n->mn[0] <= mx[0] && mn[0] <= n->mx[0] && n->mn[1] <= mx[1] && mn[1] <= n->mx[1] && n->mn[2] <= mx[2] && mn[2] <= n->mx[2];
}

/* one pair found for triangle i: counts, keys (at *o) or the bit */
static int emit( const uint64_t i, const uint32_t j, uint32_t* counts, uint64_t* keys, uint64_t* o )
{
	if (keys) keys[(*o)++] = (i << 32) | j;
	else if (counts) counts[i]++;
	return 1;
}

/* every B triangle against A triangle i; self: j > i (bits: j != i) */
void orc_overlap_all( const float* va, const uint64_t na, const float* vb, const uint64_t nb, const int self, uint32_t* counts,
	const uint64_t* offsets, uint64_t* keys, uint32_t* bits )
{
	if (bits) memset( bits, 0, ((na + 31) / 32) * 4 );
	#pragma omp parallel for schedule( dynamic, 16 )
	for (int64_t i = 0; i < (int64_t)na; i++)
	{
		float t[9], u[9];
		corners( va, (uint32_t)i, t );
		uint64_t o = keys ? offsets[i] : 0;
		if (counts && !keys) counts[i] = 0;
		for (uint64_t j = 0; j < nb; j++)
		{
			if (self && (bits ? j == (uint64_t)i : j <= (uint64_t)i)) continue;
			corners( vb, (uint32_t)j, u );
			if (!orc_tt( t, u, self )) continue;
			if (bits) { _Pragma( "omp atomic" ) bits[i >> 5] |= 1u << (i & 31); break; }
			emit( i, (uint32_t)j, counts, keys, &o );
		}
	}
}

/* the references of leaf slot k against triangle i; returns 1 when the bits form is done */
static int leaf( const node32* nd, const uint32_t* prim_idx, const float* vb, const uint64_t i, const float* t, const int self, const int any,
	uint32_t* counts, uint64_t* keys, uint64_t* o )
{
	float u[9];
	for (uint32_t r = nd->lf; r < nd->lf + nd->cnt; r++)
	{
		const uint32_t j = prim_idx[r];
		if (self && (any ? j == i : j <= i)) continue;
		corners( vb, j, u );
		if (!orc_tt( t, u, self )) continue;
		if (any) return 1;
		emit( i, j, counts, keys, o );
	}
	return 0;
}

void orc_overlap_tree( const node32* nodes, const uint32_t used, const uint32_t* prim_idx, const float* vb, const float* va, const uint64_t na,
	const int self, const int brute, uint32_t* counts, const uint64_t* offsets, uint64_t* keys, uint32_t* bits )
{
	if (bits) memset( bits, 0, ((na + 31) / 32) * 4 );
	#pragma omp parallel
	{
		uint32_t* st = (uint32_t*)malloc( sizeof( uint32_t ) * (used + 2) );
		uint8_t* flag = brute ? (uint8_t*)malloc( used + 2 ) : 0;
		#pragma omp for schedule( dynamic, 16 )
		for (int64_t ii = 0; ii < (int64_t)na; ii++)
		{
			const uint64_t i = (uint64_t)ii;
			float t[9], mn[3], mx[3];
			corners( va, (uint32_t)i, t );
			for (int k = 0; k < 3; k++) mn[k] = fminf( fminf( t[k], t[3 + k] ), t[6 + k] ), mx[k] = fmaxf( fmaxf( t[k], t[3 + k] ), t[6 + k] );
			uint64_t o = keys ? offsets[i] : 0;
			if (counts && !keys) counts[i] = 0;
			int hit = 0;
			if (brute)
			{
				/* the definition: a slot is reached when every box on some path to it from the root, the root's excepted, overlaps.
				 * Mark the reached slots (each once, whatever the number of paths), then take every reference of every reached leaf
				 * in slot order: the same set of pairs as the walk, without its order or its repeats */
				memset( flag, 0, used + 2 );
				int sp = 0;
				st[sp++] = 0, flag[0] = 1;
				while (sp)
				{
					const node32* nd = nodes + st[--sp];
					if (nd->cnt) continue;
					for (uint32_t c = nd->lf; c < nd->lf + 2; c++) if (!flag[c] && box_hit( mn, mx, nodes + c )) flag[c] = 1, st[sp++] = c;
				}
				for (uint32_t k = 0; k < used && !hit; k++)
					if (flag[k] && nodes[k].cnt) hit = leaf( nodes + k, prim_idx, vb, i, t, self, bits != 0, counts, keys, &o );
			}
			else
			{
				int sp = 0;
				uint32_t x = 0;
				while (1)
				{
					const node32* nd = nodes + x;
					if (!nd->cnt)
					{
						const int a = box_hit( mn, mx, nodes + nd->lf ), b = box_hit( mn, mx, nodes + nd->lf + 1 );
						if (a && b) { st[sp++] = nd->lf + 1; x = nd->lf; continue; }
						if (a) { x = nd->lf; continue; }
						if (b) { x = nd->lf + 1; continue; }
					}
					else if ((hit = leaf( nd, prim_idx, vb, i, t, self, bits != 0, counts, keys, &o ))) break;
					if (!sp) break;
					x = st[--sp];
				}
			}
			if (bits && hit) { _Pragma( "omp atomic" ) bits[i >> 5] |= 1u << (i & 31); }
		}
		free( st );
		free( flag );
	}
}
