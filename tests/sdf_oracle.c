/* tests/sdf_oracle.c - the oracle of tbvh_signed_distance_prepare / tbvh_signed_distance.  TEST INFRASTRUCTURE ONLY.
 *
 * Restates DESIGN.md §4.10 on the host in the engine's fp32 operation order (every fused pair written as fmaf, compiled with contraction
 * off by tests/sdf_oracle.py), over the closest-point oracle it includes:
 *  - orc_sd_triangle:  orc_cp_triangle with the feature of the closest point (face, vertex or edge) from the branch and clamp taken;
 *  - orc_sd_prepare:   the pseudonormal table - corners welded by position, unit face normals, vertex sums of theta * n in ascending
 *                      corner order, edge sums of n in ascending half-edge order - 7 float4 per triangle (face, v0, v1, v2, AB, AC, BC);
 *  - orc_sd_brute:     the signed record of every query: orc_cp_brute's record, signed by ( p - c ) . N of the winner's feature.
 */
#include "closest_oracle.c"

enum { F_FACE = 0, F_V0 = 1, F_V1 = 2, F_V2 = 3, F_AB = 4, F_AC = 5, F_BC = 6 };
#define SD_REC 7
#define SD_FLT_MAX 3.402823466e38f

static uint32_t efeat( const float t, const uint32_t a, const uint32_t b, const uint32_t e ) { return t == 0.0f ? a : t == 1.0f ? b : e; }

float orc_sd_triangle( const float* p, const float* v0, const float* e1r, const float* e2r, float* uo, float* vo, uint32_t* fo )
{
	float ap[3], bp[3], cp[3], e1[3], e2[3], r[3], u, v, inv;
	uint32_t f;
	for (int k = 0; k < 3; k++) r[k] = p[k] - v0[k];
	const float m = fmaxf( fmaxf( fmaxf( fmaxf( fabsf( r[0] ), fabsf( r[1] ) ), fmaxf( fabsf( r[2] ), fabsf( e1r[0] ) ) ),
		fmaxf( fmaxf( fabsf( e1r[1] ), fabsf( e1r[2] ) ), fmaxf( fabsf( e2r[0] ), fabsf( e2r[1] ) ) ) ), fabsf( e2r[2] ) );
	const float s = pow2( m, &inv );
	for (int k = 0; k < 3; k++) ap[k] = r[k] * s, e1[k] = e1r[k] * s, e2[k] = e2r[k] * s;
	const float d1 = dot3( e1, ap ), d2 = dot3( e2, ap );
	if (d1 <= 0.0f && d2 <= 0.0f) u = 0.0f, v = 0.0f, f = F_V0; /* A */
	else
	{
		for (int k = 0; k < 3; k++) bp[k] = ap[k] - e1[k], cp[k] = ap[k] - e2[k];
		const float d3 = dot3( e1, bp ), d4 = dot3( e2, bp ), d5 = dot3( e1, cp ), d6 = dot3( e2, cp );
		const float vc = d1 * d4 - d3 * d2, vb = d5 * d2 - d1 * d6, va = d3 * d6 - d5 * d4;
		const float x = d4 - d3, y = d5 - d6;
		if (d3 >= 0.0f && d4 <= d3) u = 1.0f, v = 0.0f, f = F_V1; /* B */
		else if (vc <= 0.0f && d1 >= 0.0f && d3 <= 0.0f) u = edge( d1, d1 - d3 ), v = 0.0f, f = efeat( u, F_V0, F_V1, F_AB ); /* AB */
		else if (d6 >= 0.0f && d5 <= d6) u = 0.0f, v = 1.0f, f = F_V2; /* C */
		else if (vb <= 0.0f && d2 >= 0.0f && d6 <= 0.0f) u = 0.0f, v = edge( d2, d2 - d6 ), f = efeat( v, F_V0, F_V2, F_AC ); /* AC */
		else if (va <= 0.0f && x >= 0.0f && y >= 0.0f) { const float w = edge( x, x + y ); u = 1.0f - w, v = w, f = efeat( w, F_V1, F_V2, F_BC ); } /* BC */
		else /* face: the clamped edge points AB, AC, BC and, when n = e1 x e2 is not 0, the face point; the nearest, ties to the face, AB, AC, BC */
		{
			float bc[3];
			for (int k = 0; k < 3; k++) bc[k] = e2[k] - e1[k];
			const float tab = edge( d1, dot3( e1, e1 ) ), tac = edge( d2, dot3( e2, e2 ) ), tbc = edge( dot3( bc, bp ), dot3( bc, bc ) );
			const float nx = e1[1] * e2[2] - e1[2] * e2[1], ny = e1[2] * e2[0] - e1[0] * e2[2], nz = e1[0] * e2[1] - e1[1] * e2[0];
			const float nn = fmaf( nz, nz, fmaf( ny, ny, nx * nx ) );
			const float dab = dist2( ap, e1, e2, tab, 0.0f );
			float dm = dab;
			u = tab, v = 0.0f, f = efeat( tab, F_V0, F_V1, F_AB );
			if (nn > 0.0f)
			{
				const float ax = ap[1] * e2[2] - ap[2] * e2[1], ay = ap[2] * e2[0] - ap[0] * e2[2], az = ap[0] * e2[1] - ap[1] * e2[0];
				const float bx = e1[1] * ap[2] - e1[2] * ap[1], by = e1[2] * ap[0] - e1[0] * ap[2], bz = e1[0] * ap[1] - e1[1] * ap[0];
				const float inv = 1.0f / nn;
				const float uf = unit( fmaf( az, nz, fmaf( ay, ny, ax * nx ) ) * inv );
				const float vmax = 1.0f - uf, w = unit( fmaf( bz, nz, fmaf( by, ny, bx * nx ) ) * inv );
				const float vf = w < vmax ? w : vmax, df = dist2( ap, e1, e2, uf, vf );
				if (df <= dab)
				{
					/* clamped onto an edge: uf == 0 -> AC, vf == 0 -> AB, vf limited by 1 - uf -> BC; two clamps: their vertex */
					const int cu = uf == 0.0f, cv = vf == 0.0f, cl = !(w < vmax);
					u = uf, v = vf, dm = df;
					f = cu ? (cv ? F_V0 : cl ? F_V2 : F_AC) : cv ? (cl ? F_V1 : F_AB) : cl ? F_BC : F_FACE;
				}
			}
			const float dac = dist2( ap, e1, e2, 0.0f, tac );
			if (dac < dm) u = 0.0f, v = tac, dm = dac, f = efeat( tac, F_V0, F_V2, F_AC );
			const float ubc = 1.0f - tbc, dbc = dist2( ap, e1, e2, ubc, tbc );
			if (dbc < dm) u = ubc, v = tbc, f = efeat( tbc, F_V1, F_V2, F_BC );
		}
	}
	*uo = u, *vo = v, *fo = f;
	return (dist2( ap, e1, e2, u, v ) * inv) * inv;
}

/* A&S 4.4.46 */
static float sd_acos( const float x )
{
	const float a = x < 0.0f ? -x : x;
	float p = -0.0012624911f;
	p = fmaf( p, a, 0.0066700901f );
	p = fmaf( p, a, -0.0170881256f );
	p = fmaf( p, a, 0.0308918810f );
	p = fmaf( p, a, -0.0501743046f );
	p = fmaf( p, a, 0.0889789874f );
	p = fmaf( p, a, -0.2145988016f );
	p = fmaf( p, a, 1.5707963050f );
	const float r = sqrtf( 1.0f - a ) * p;
	return x < 0.0f ? 3.14159265f - r : r;
}

static float sd_angle( const float* a, const float* b )
{
	const float la = dot3( a, a ), lb = dot3( b, b );
	if (!(la > 0.0f && la <= SD_FLT_MAX && lb > 0.0f && lb <= SD_FLT_MAX)) return 0.0f;
	float c = dot3( a, b ) / (sqrtf( la ) * sqrtf( lb ));
	c = c > -1.0f ? c : -1.0f;
	c = c < 1.0f ? c : 1.0f;
	return sd_acos( c );
}

static uint32_t sd_key( const float f )
{
	if (f != f) return 0xffffffffu;
	uint32_t u = 0;
	if (f != 0.0f) memcpy( &u, &f, 4 );
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

typedef struct { uint32_t k[3], c; } corner_t;
typedef struct { uint64_t k; uint32_t h; } half_t;
static int cmp_corner( const void* x, const void* y )
{
	const corner_t* a = (const corner_t*)x, * b = (const corner_t*)y;
	for (int i = 0; i < 3; i++) if (a->k[i] != b->k[i]) return a->k[i] < b->k[i] ? -1 : 1;
	return a->c < b->c ? -1 : a->c > b->c;
}
static int cmp_half( const void* x, const void* y )
{
	const half_t* a = (const half_t*)x, * b = (const half_t*)y;
	if (a->k != b->k) return a->k < b->k ? -1 : 1;
	return a->h < b->h ? -1 : a->h > b->h;
}

/* the table of `prims` triangles (verts: 3 float4 per triangle) into table (prims x 7 x float4) */
void orc_sd_prepare( const float* verts, const uint32_t prims, float* table )
{
	const uint32_t m = prims * 3;
	float* theta = (float*)malloc( sizeof( float ) * m );
	uint32_t* vid = (uint32_t*)malloc( sizeof( uint32_t ) * m );
	corner_t* cs = (corner_t*)malloc( sizeof( corner_t ) * m );
	half_t* hs = (half_t*)malloc( sizeof( half_t ) * m );
	memset( table, 0, sizeof( float ) * 4 * SD_REC * (size_t)prims );
	for (uint32_t p = 0; p < prims; p++)
	{
		const float* v[3] = { verts + (size_t)p * 12, verts + (size_t)p * 12 + 4, verts + (size_t)p * 12 + 8 };
		float e[3][3], g[3][3]; /* e[k]: corner k to corner k+1, g[k]: corner k to corner k+2 */
		for (int k = 0; k < 3; k++) for (int a = 0; a < 3; a++) e[k][a] = v[(k + 1) % 3][a] - v[k][a], g[k][a] = v[(k + 2) % 3][a] - v[k][a];
		/* e1 = v1 - v0 = e[0], e2 = v2 - v0 = g[0], scaled by the power of two of their largest component before the cross product */
		float a[3], b[3], inv;
		const float m = fmaxf( fmaxf( fmaxf( fabsf( e[0][0] ), fabsf( e[0][1] ) ), fmaxf( fabsf( e[0][2] ), fabsf( g[0][0] ) ) ), fmaxf( fabsf( g[0][1] ), fabsf( g[0][2] ) ) );
		const float sc = pow2( m, &inv );
		for (int k = 0; k < 3; k++) a[k] = e[0][k] * sc, b[k] = g[0][k] * sc;
		const float nx = a[1] * b[2] - a[2] * b[1], ny = a[2] * b[0] - a[0] * b[2], nz = a[0] * b[1] - a[1] * b[0];
		const float nn = fmaf( nz, nz, fmaf( ny, ny, nx * nx ) );
		float* n = table + (size_t)p * SD_REC * 4;
		if (nn > 0.0f && nn <= SD_FLT_MAX) { const float l = sqrtf( nn ); n[0] = nx / l, n[1] = ny / l, n[2] = nz / l; }
		/* corner 0: (v1 - v0, v2 - v0); corner 1: (v2 - v1, v0 - v1); corner 2: (v0 - v2, v1 - v2) */
		for (int k = 0; k < 3; k++) theta[p * 3 + k] = sd_angle( e[k], g[k] );
		for (int k = 0; k < 3; k++)
		{
			corner_t* c = cs + p * 3 + k;
			for (int a = 0; a < 3; a++) c->k[a] = sd_key( v[k][a] );
			c->c = p * 3 + k;
		}
	}
	qsort( cs, m, sizeof( corner_t ), cmp_corner );
	for (uint32_t a = 0, b; a < m; a = b)
	{
		const float* pa = verts + (size_t)cs[a].c * 4;
		for (b = a + 1; b < m; b++)
		{
			const float* pb = verts + (size_t)cs[b].c * 4;
			if (!(pa[0] == pb[0] && pa[1] == pb[1] && pa[2] == pb[2])) break;
		}
		float s[3] = { 0.0f, 0.0f, 0.0f };
		for (uint32_t i = a; i < b; i++)
		{
			const uint32_t c = cs[i].c;
			const float* n = table + (size_t)(c / 3) * SD_REC * 4;
			for (int k = 0; k < 3; k++) s[k] = fmaf( theta[c], n[k], s[k] );
		}
		for (uint32_t i = a; i < b; i++)
		{
			const uint32_t c = cs[i].c;
			memcpy( table + ((size_t)(c / 3) * SD_REC + 1 + c % 3) * 4, s, 12 );
			vid[c] = cs[a].c;
		}
	}
	for (uint32_t h = 0; h < m; h++)
	{
		const uint32_t p = h / 3, e = h % 3, a = vid[p * 3 + (e == 2 ? 1 : 0)], b = vid[p * 3 + (e == 0 ? 1 : 2)];
		hs[h].k = ((uint64_t)(a < b ? a : b) << 32) | (a < b ? b : a), hs[h].h = h;
	}
	qsort( hs, m, sizeof( half_t ), cmp_half );
	for (uint32_t a = 0, b; a < m; a = b)
	{
		for (b = a + 1; b < m && hs[b].k == hs[a].k; b++) {}
		float s[3] = { 0.0f, 0.0f, 0.0f };
		for (uint32_t i = a; i < b; i++)
		{
			const float* n = table + (size_t)(hs[i].h / 3) * SD_REC * 4;
			for (int k = 0; k < 3; k++) s[k] = s[k] + n[k];
		}
		for (uint32_t i = a; i < b; i++) memcpy( table + ((size_t)(hs[i].h / 3) * SD_REC + 4 + hs[i].h % 3) * 4, s, 12 );
	}
	free( theta ), free( vid ), free( cs ), free( hs );
}

/* the signed records of n queries: orc_cp_brute over the tree (walk: orc_cp_walk, which gives the same records), then the winner's
 * feature and the sign of ( p - c ) . N */
void orc_sd_brute( const node32* nodes, const uint32_t used_nodes, const uint32_t* prim_idx, const float* verts, const float* table,
	const float* queries, const uint64_t n, float* results, const int walk )
{
	if (walk) orc_cp_walk( nodes, used_nodes, prim_idx, verts, queries, n, results, 0 );
	else orc_cp_brute( nodes, used_nodes, prim_idx, verts, queries, n, results, 0 );
	for (uint64_t i = 0; i < n; i++)
	{
		float* r = results + i * 4;
		uint32_t prim;
		memcpy( &prim, r + 3, 4 );
		if (prim == NO_PRIM) continue;
		const float* q = queries + i * 4, * a = verts + (size_t)prim * 12, * b = a + 4, * c = a + 8;
		float e1[3], e2[3], ap[3], u, v;
		uint32_t f;
		for (int k = 0; k < 3; k++) e1[k] = b[k] - a[k], e2[k] = c[k] - a[k];
		orc_sd_triangle( q, a, e1, e2, &u, &v, &f );
		for (int k = 0; k < 3; k++) ap[k] = q[k] - a[k];
		float d[3];
		for (int k = 0; k < 3; k++) d[k] = ap[k] - fmaf( r[2], e2[k], r[1] * e1[k] );
		const float* N = table + ((size_t)prim * SD_REC + f) * 4;
		const float s = fmaf( d[2], N[2], fmaf( d[1], N[1], d[0] * N[0] ) );
		if (s < 0.0f) r[0] = -r[0];
	}
}

/* orc_sd_triangle over arrays: points (n x 4), records (n x 12: v0, e1, e2 as float4) -> out (n x 4: d2_raw, u, v, feature bits) */
void orc_sd_triangles( const float* points, const float* recs, const uint64_t n, float* out )
{
	for (uint64_t i = 0; i < n; i++)
	{
		const float* r = recs + i * 12;
		uint32_t f;
		out[i * 4] = orc_sd_triangle( points + i * 4, r, r + 4, r + 8, out + i * 4 + 1, out + i * 4 + 2, &f );
		memcpy( out + i * 4 + 3, &f, 4 );
	}
}
