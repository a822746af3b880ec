/* tests/closest_oracle.c - the oracle of tbvh_closest_point / tbvh_sphere_overlap.  TEST INFRASTRUCTURE ONLY.
 *
 * The engine's proximity queries (include/tinybvh_b200_device/closest_walk.cuh) follow their own definition, DESIGN.md §4.9; this file
 * restates it on the host in the same fp32 operation order (every fused pair written as fmaf, compiled with contraction off by
 * tests/closest_oracle.py):
 *  - orc_cp_triangle: ClosestPtPointTriangle (Ericson, RTCD 5.1.5) on the leaf record (v0, e1, e2);
 *  - orc_cp_brute:    every reference (leaf, triangle) of a 32-byte-node tree with its path bound, no pruning - the definition itself;
 *  - orc_cp_walk:     the pruned walk of the same rules (nearer child first, strict pruning, pops pruned again), OpenMP over queries;
 *  - orc_cp_node_bounds: the path bound P of every reachable node for one point.
 * Trees are the reference's 32-byte node arrays (node 0 the root, node 1 unused, children paired at leftFirst); vertices are float4,
 * three per primitive, and the leaf records are built as the engine builds them (e1 = v1 - v0, e2 = v2 - v0 in fp32).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NO_PRIM 0xffffffffu

typedef struct { float mn[3]; uint32_t lf; float mx[3]; uint32_t cnt; } node32;

static float dot3( const float* a, const float* b ) { return fmaf( a[2], b[2], fmaf( a[1], b[1], a[0] * b[0] ) ); }
static float unit( const float x ) { const float y = x > 0.0f ? x : 0.0f; return y < 1.0f ? y : 1.0f; }
static float edge( const float num, const float den ) { return unit( num / den ); }
static float dist2( const float* ap, const float* e1, const float* e2, const float u, const float v )
{
	float d[3];
	for (int k = 0; k < 3; k++) d[k] = ap[k] - fmaf( v, e2[k], u * e1[k] );
	return fmaf( d[2], d[2], fmaf( d[1], d[1], d[0] * d[0] ) );
}

/* closest_walk.cuh cp_pow2: 2^-e bringing m >= 0 into [1, 2), e clamped to [-126, 126], *inv = 2^e; 1 when m is 0 or not finite */
static float pow2( const float m, float* inv )
{
	uint32_t f, c;
	memcpy( &f, &m, 4 );
	f >>= 23;
	if (!(m > 0.0f) || f == 255u) { *inv = 1.0f; return 1.0f; }
	c = f < 1u ? 1u : f > 253u ? 253u : f;
	const uint32_t ib = c << 23, sb = (254u - c) << 23;
	float s;
	memcpy( inv, &ib, 4 ), memcpy( &s, &sb, 4 );
	return s;
}

/* ap, e1, e2 scaled by the power of two of their largest component, d2_raw scaled back (closest_walk.cuh cp_triangle_feature) */
float orc_cp_triangle( const float* p, const float* v0, const float* e1r, const float* e2r, float* uo, float* vo )
{
	float ap[3], bp[3], cp[3], e1[3], e2[3], r[3], u, v, inv;
	for (int k = 0; k < 3; k++) r[k] = p[k] - v0[k];
	const float m = fmaxf( fmaxf( fmaxf( fmaxf( fabsf( r[0] ), fabsf( r[1] ) ), fmaxf( fabsf( r[2] ), fabsf( e1r[0] ) ) ),
		fmaxf( fmaxf( fabsf( e1r[1] ), fabsf( e1r[2] ) ), fmaxf( fabsf( e2r[0] ), fabsf( e2r[1] ) ) ) ), fabsf( e2r[2] ) );
	const float s = pow2( m, &inv );
	for (int k = 0; k < 3; k++) ap[k] = r[k] * s, e1[k] = e1r[k] * s, e2[k] = e2r[k] * s;
	const float d1 = dot3( e1, ap ), d2 = dot3( e2, ap );
	if (d1 <= 0.0f && d2 <= 0.0f) u = 0.0f, v = 0.0f; /* A */
	else
	{
		for (int k = 0; k < 3; k++) bp[k] = ap[k] - e1[k], cp[k] = ap[k] - e2[k];
		const float d3 = dot3( e1, bp ), d4 = dot3( e2, bp ), d5 = dot3( e1, cp ), d6 = dot3( e2, cp );
		const float vc = d1 * d4 - d3 * d2, vb = d5 * d2 - d1 * d6, va = d3 * d6 - d5 * d4;
		const float x = d4 - d3, y = d5 - d6;
		if (d3 >= 0.0f && d4 <= d3) u = 1.0f, v = 0.0f; /* B */
		else if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f) u = edge( d1, d1 - d3 ), v = 0.0f; /* AB */
		else if (d6 >= 0.0f && d5 <= d6) u = 0.0f, v = 1.0f; /* C */
		else if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) u = 0.0f, v = edge( d2, d2 - d6 ); /* AC */
		else if (va <= 0.0f && x >= 0.0f && y >= 0.0f) { const float w = edge( x, x + y ); u = 1.0f - w, v = w; } /* BC */
		else /* face: the clamped edge points AB, AC, BC and, when n = e1 x e2 is not 0, the face point; the nearest, ties to the face, AB, AC, BC */
		{
			float bc[3];
			for (int k = 0; k < 3; k++) bc[k] = e2[k] - e1[k];
			const float tab = edge( d1, dot3( e1, e1 ) ), tac = edge( d2, dot3( e2, e2 ) ), tbc = edge( dot3( bc, bp ), dot3( bc, bc ) );
			const float nx = e1[1] * e2[2] - e1[2] * e2[1], ny = e1[2] * e2[0] - e1[0] * e2[2], nz = e1[0] * e2[1] - e1[1] * e2[0];
			const float nn = fmaf( nz, nz, fmaf( ny, ny, nx * nx ) );
			const float dab = dist2( ap, e1, e2, tab, 0.0f );
			float dm = dab;
			u = tab, v = 0.0f;
			if (nn > 0.0f)
			{
				/* u = ((ap x e2) . n) / |n|^2, v = ((e1 x ap) . n) / |n|^2 */
				const float ax = ap[1] * e2[2] - ap[2] * e2[1], ay = ap[2] * e2[0] - ap[0] * e2[2], az = ap[0] * e2[1] - ap[1] * e2[0];
				const float bx = e1[1] * ap[2] - e1[2] * ap[1], by = e1[2] * ap[0] - e1[0] * ap[2], bz = e1[0] * ap[1] - e1[1] * ap[0];
				const float inv = 1.0f / nn;
				const float uf = unit( fmaf( az, nz, fmaf( ay, ny, ax * nx ) ) * inv );
				const float vmax = 1.0f - uf, w = unit( fmaf( bz, nz, fmaf( by, ny, bx * nx ) ) * inv );
				const float vf = w < vmax ? w : vmax, df = dist2( ap, e1, e2, uf, vf );
				if (df <= dab) u = uf, v = vf, dm = df;
			}
			const float dac = dist2( ap, e1, e2, 0.0f, tac );
			if (dac < dm) u = 0.0f, v = tac, dm = dac;
			const float ubc = 1.0f - tbc, dbc = dist2( ap, e1, e2, ubc, tbc );
			if (dbc < dm) u = ubc, v = tbc;
		}
	}
	*uo = u, *vo = v;
	return (dist2( ap, e1, e2, u, v ) * inv) * inv;
}

static float box_bound( const float* p, const node32* n )
{
	float g[3];
	for (int k = 0; k < 3; k++) g[k] = fmaxf( fmaxf( n->mn[k] - p[k], p[k] - n->mx[k] ), 0.0f );
	return fmaf( g[2], g[2], fmaf( g[1], g[1], g[0] * g[0] ) );
}

/* the engine's leaf record of reference r: v0 (w = primIdx), e1, e2 */
static void record( const float* verts, const uint32_t* prim_idx, const uint32_t r, float* v0, float* e1, float* e2, uint32_t* prim )
{
	const uint32_t pi = prim_idx[r];
	const float* a = verts + (size_t)pi * 12, * b = a + 4, * c = a + 8;
	for (int k = 0; k < 3; k++) v0[k] = a[k], e1[k] = b[k] - a[k], e2[k] = c[k] - a[k];
	*prim = pi;
}

static int query_ok( const float* q ) { return q[0] == q[0] && q[1] == q[1] && q[2] == q[2] && q[3] >= 0.0f; }

static void write_rec( float* out, const float d, const float u, const float v, const uint32_t prim )
{
	out[0] = d, out[1] = u, out[2] = v;
	memcpy( out + 3, &prim, 4 );
}

/* one reference against the running best: closest keeps the smallest (d2, prim); any reports d2 <= best */
static int consider( const float* p, const float* verts, const uint32_t* prim_idx, const uint32_t r, const float P, const int any,
	float* best, uint32_t* bprim, float* bu, float* bv )
{
	float v0[3], e1[3], e2[3], u, v;
	uint32_t prim;
	record( verts, prim_idx, r, v0, e1, e2, &prim );
	const float d2 = fmaxf( orc_cp_triangle( p, v0, e1, e2, &u, &v ), P );
	if (any) return d2 <= *best;
	if (d2 < *best || (d2 == *best && prim < *bprim)) *best = d2, *bprim = prim, *bu = u, *bv = v;
	return 0;
}

typedef struct { uint32_t node; float P; } pend;

/* path bound of every node reachable from the root for point p into P[used_nodes] (unreached slots: -1).  A node an uploaded tree
 * reaches on several paths (tbvh_upload_bvh accepts such a DAG) gets the least bound over them: the walk visits every path, and as
 * fmaxf is monotone, the least value of a reference over its paths is fmaxf( d2_raw, least P ). */
void orc_cp_node_bounds( const node32* nodes, const uint32_t used_nodes, const float* p, float* P )
{
	for (uint32_t i = 0; i < used_nodes; i++) P[i] = -1.0f;
	pend* st = (pend*)malloc( sizeof( pend ) * (used_nodes + 2) );
	int sp = 0;
	st[sp++] = (pend){ 0, 0.0f };
	while (sp)
	{
		const pend e = st[--sp];
		if (P[e.node] < 0.0f || e.P < P[e.node]) P[e.node] = e.P;
		const node32* n = nodes + e.node;
		if (n->cnt) continue;
		for (uint32_t c = n->lf; c < n->lf + 2; c++) st[sp++] = (pend){ c, fmaxf( box_bound( p, nodes + c ), e.P ) };
	}
	free( st );
}

/* the definition: every leaf with its path bound (the root, leaf or not, has P = 0), every reference of every leaf */
void orc_cp_brute( const node32* nodes, const uint32_t used_nodes, const uint32_t* prim_idx, const float* verts, const float* queries,
	const uint64_t n, float* results, uint32_t* bits )
{
	const int any = bits != 0;
	if (any) memset( bits, 0, ((n + 31) / 32) * 4 );
	#pragma omp parallel
	{
		float* P = (float*)malloc( sizeof( float ) * (used_nodes + 2) );
		#pragma omp for schedule( dynamic, 16 )
		for (int64_t i = 0; i < (int64_t)n; i++)
		{
			const float* q = queries + i * 4;
			float best = q[3] * q[3], bu = 0.0f, bv = 0.0f;
			uint32_t bprim = NO_PRIM;
			int hit = 0;
			if (query_ok( q ))
			{
				orc_cp_node_bounds( nodes, used_nodes, q, P );
				for (uint32_t k = 0; k < used_nodes && !hit; k++)
				{
					if (P[k] < 0.0f || !nodes[k].cnt) continue;
					for (uint32_t t = 0; t < nodes[k].cnt && !hit; t++)
						hit = consider( q, verts, prim_idx, nodes[k].lf + t, P[k], any, &best, &bprim, &bu, &bv );
				}
			}
			if (any) { if (hit) { _Pragma( "omp atomic" ) bits[i >> 5] |= 1u << (i & 31); } }
			else if (bprim == NO_PRIM) write_rec( results + i * 4, q[3], 0.0f, 0.0f, NO_PRIM );
			else write_rec( results + i * 4, sqrtf( best ), bu, bv, bprim );
		}
		free( P );
	}
}

/* the pruned walk the kernel runs, over the same rules */
void orc_cp_walk( const node32* nodes, const uint32_t used_nodes, const uint32_t* prim_idx, const float* verts, const float* queries,
	const uint64_t n, float* results, uint32_t* bits )
{
	const int any = bits != 0;
	if (any) memset( bits, 0, ((n + 31) / 32) * 4 );
	#pragma omp parallel
	{
		pend* st = (pend*)malloc( sizeof( pend ) * (used_nodes + 2) );
		#pragma omp for schedule( dynamic, 64 )
		for (int64_t i = 0; i < (int64_t)n; i++)
		{
			const float* q = queries + i * 4;
			float best = q[3] * q[3], bu = 0.0f, bv = 0.0f;
			uint32_t bprim = NO_PRIM;
			int hit = 0, sp = 0;
			uint32_t node = 0;
			float P = 0.0f;
			while (query_ok( q ))
			{
				const node32* nd = nodes + node;
				int next = 0;
				if (!nd->cnt)
				{
					const uint32_t a = nd->lf, b = nd->lf + 1;
					const float Pa = fmaxf( box_bound( q, nodes + a ), P ), Pb = fmaxf( box_bound( q, nodes + b ), P );
					const int va = !(Pa > best), vb = !(Pb > best);
					if (va && vb)
					{
						const int swp = Pb < Pa;
						node = swp ? b : a, P = swp ? Pb : Pa;
						st[sp++] = swp ? (pend){ a, Pa } : (pend){ b, Pb };
						next = 1;
					}
					else if (va) node = a, P = Pa, next = 1;
					else if (vb) node = b, P = Pb, next = 1;
				}
				else
				{
					for (uint32_t t = 0; t < nd->cnt && !hit; t++) hit = consider( q, verts, prim_idx, nd->lf + t, P, any, &best, &bprim, &bu, &bv );
					if (hit) break;
				}
				if (next) continue;
				while (sp && st[sp - 1].P > best) sp--;
				if (!sp) break;
				sp--, node = st[sp].node, P = st[sp].P;
			}
			if (any) { if (hit) { _Pragma( "omp atomic" ) bits[i >> 5] |= 1u << (i & 31); } }
			else if (bprim == NO_PRIM) write_rec( results + i * 4, q[3], 0.0f, 0.0f, NO_PRIM );
			else write_rec( results + i * 4, sqrtf( best ), bu, bv, bprim );
		}
		free( st );
	}
}

/* orc_cp_triangle over arrays: points (n x 4), records (n x 12: v0, e1, e2 as float4) -> out (n x 4: d2_raw, u, v, 0) */
void orc_cp_triangles( const float* points, const float* recs, const uint64_t n, float* out )
{
	for (uint64_t i = 0; i < n; i++)
	{
		const float* r = recs + i * 12;
		out[i * 4] = orc_cp_triangle( points + i * 4, r, r + 4, r + 8, out + i * 4 + 1, out + i * 4 + 2 );
		out[i * 4 + 3] = 0.0f;
	}
}
