/* tests/allhits_oracle.c - the oracle of tbvh_intersect_all.  TEST INFRASTRUCTURE ONLY.
 *
 * The engine's multi-hit ray query (include/tinybvh_b200_device/all_hits_walk.cuh) follows its own definition, DESIGN.md §4.14; this file
 * restates it on the host in the same fp32 operation order (every fused pair written as fmaf, compiled with contraction off by
 * tests/allhits_oracle.py):
 *  - orc_ah_brute: the definition itself - every reached node with its path bound (the least over its paths), every reference of every
 *                  reached leaf, each distinct prim at its least key, the k smallest ( key, prim ); also returns each record's key;
 *  - orc_ah_walk:  the pruned walk the kernel runs (nearer child first, or - reverse - the other one first), over the same rules.
 * Trees are the reference's 32-byte node arrays (node 0 the root, node 1 unused, children paired at leftFirst); vertices are float4, three
 * per primitive, and the leaf records are built as the engine builds them (e1 = v1 - v0, e2 = v2 - v0 in fp32).  Rays are 64-byte records
 * { O | mask, D | inst, rD | pad, t, u, v, prim } at `stride` bytes; t is the ray's tmax.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NO_PRIM 0xffffffffu

typedef struct { float mn[3]; uint32_t lf; float mx[3]; uint32_t cnt; } node32;
typedef struct { float O[3], D[3], rD[3], nro[3], tmax; int pos[3]; } ray_t;
typedef struct { float key, t, u, v; uint32_t prim; } ent;

static ray_t load( const char* rays, const uint32_t stride, const uint64_t i )
{
	const float* r = (const float*)(rays + i * stride);
	ray_t R;
	for (int a = 0; a < 3; a++)
	{
		R.O[a] = r[a], R.D[a] = r[4 + a], R.rD[a] = r[8 + a];
		R.nro[a] = -(R.O[a] * R.rD[a]);
		R.pos[a] = R.D[a] >= 0;
	}
	R.tmax = r[12];
	return R;
}

/* bvh2_pair_step's slab test of one child with the ray's tmax: 1 when reached, *tmin its entry distance */
static int slab( const ray_t* R, const node32* c, float* tmin )
{
	float t1[3], t2[3];
	for (int a = 0; a < 3; a++)
	{
		t1[a] = fmaf( R->pos[a] ? c->mn[a] : c->mx[a], R->rD[a], R->nro[a] );
		t2[a] = fmaf( R->pos[a] ? c->mx[a] : c->mn[a], R->rD[a], R->nro[a] );
	}
	*tmin = fmaxf( fmaxf( t1[0], t1[1] ), fmaxf( t1[2], 0.0f ) );
	const float tfar = fminf( fminf( t2[0], t2[1] ), fminf( t2[2], R->tmax ) );
	return tfar >= *tmin;
}

/* base.cuh mt_test on the engine's leaf record of reference r, accepted on [0, tmax] with a t that is not NaN */
static int tri_test( const ray_t* R, const float* verts, const uint32_t* prim_idx, const uint32_t r, float* to, float* uo, float* vo, uint32_t* prim )
{
	const uint32_t pi = prim_idx[r];
	const float* v0 = verts + (size_t)pi * 12, * v1 = v0 + 4, * v2 = v0 + 8;
	const float* O = R->O, * D = R->D;
	const float e1x = v1[0] - v0[0], e1y = v1[1] - v0[1], e1z = v1[2] - v0[2];
	const float e2x = v2[0] - v0[0], e2y = v2[1] - v0[1], e2z = v2[2] - v0[2];
	const float hx = fmaf( D[1], e2z, -(D[2] * e2y) );
	const float hy = fmaf( D[2], e2x, -(D[0] * e2z) );
	const float hz = fmaf( D[0], e2y, -(D[1] * e2x) );
	const float a = fmaf( e1z, hz, fmaf( e1x, hx, e1y * hy ) );
	if (fabsf( a ) < 0.000001f) return 0;
	const float f = 1 / a;
	const float sx = O[0] - v0[0], sy = O[1] - v0[1], sz = O[2] - v0[2];
	const float u = f * fmaf( hz, sz, fmaf( hx, sx, hy * sy ) );
	const float qx = fmaf( -e1y, sz, e1z * sy );
	const float qy = fmaf( -e1z, sx, e1x * sz );
	const float qz = fmaf( -e1x, sy, e1y * sx );
	const float v = f * fmaf( D[2], qz, fmaf( D[1], qy, D[0] * qx ) );
	if (u < 0 || v < 0 || u + v > 1) return 0;
	const float t = f * fmaf( e2z, qz, fmaf( e2x, qx, e2y * qy ) );
	if (t < 0 || t > R->tmax || t != t) return 0;
	*to = t, *uo = u, *vo = v, *prim = pi;
	return 1;
}

static int before( const ent* a, const ent* b ) { return a->key < b->key || (a->key == b->key && a->prim < b->prim); }
static int cmp_key( const void* x, const void* y ) { const ent* a = x, * b = y; return before( a, b ) ? -1 : before( b, a ) ? 1 : 0; }
static int cmp_prim( const void* x, const void* y )
{
	const ent* a = x, * b = y;
	if (a->prim != b->prim) return a->prim < b->prim ? -1 : 1;
	return a->key < b->key ? -1 : b->key < a->key ? 1 : 0;
}

static void write_row( float* hits, uint32_t* counts, float* keys, const uint64_t i, const uint32_t k, const float tmax, const ent* e, const uint32_t m, const uint32_t count )
{
	float* row = hits + i * k * 4;
	for (uint32_t s = 0; s < k; s++)
	{
		const uint32_t p = s < m ? e[s].prim : NO_PRIM;
		row[s * 4] = s < m ? e[s].t : tmax, row[s * 4 + 1] = s < m ? e[s].u : 0.0f, row[s * 4 + 2] = s < m ? e[s].v : 0.0f;
		memcpy( row + s * 4 + 3, &p, 4 );
		if (keys) keys[i * k + s] = s < m ? e[s].key : tmax;
	}
	counts[i] = count;
}

typedef struct { uint32_t node; float P; } pend;

/* path bound of every node the ray reaches into P[used_nodes] (unreached: -1): the root at 0, a child at fmaxf( P( parent ), tmin ) when
 * its slab test passes; a node reached on several paths takes the least */
static void node_bounds( const node32* nodes, const uint32_t used_nodes, const ray_t* R, float* P, pend* st )
{
	for (uint32_t i = 0; i < used_nodes; i++) P[i] = -1.0f;
	int sp = 0;
	st[sp++] = (pend){ 0, 0.0f };
	while (sp)
	{
		const pend e = st[--sp];
		if (P[e.node] < 0.0f || e.P < P[e.node]) P[e.node] = e.P;
		const node32* n = nodes + e.node;
		if (n->cnt) continue;
		for (uint32_t c = n->lf; c < n->lf + 2; c++)
		{
			float tmin;
			if (slab( R, nodes + c, &tmin )) st[sp++] = (pend){ c, fmaxf( e.P, tmin ) };
		}
	}
}

void orc_ah_brute( const node32* nodes, const uint32_t used_nodes, const uint32_t* prim_idx, const float* verts, const char* rays, const uint32_t stride,
	const uint64_t n, const uint32_t k, float* hits, uint32_t* counts, float* keys )
{
	#pragma omp parallel
	{
		float* P = (float*)malloc( sizeof( float ) * (used_nodes + 2) );
		pend* st = (pend*)malloc( sizeof( pend ) * (used_nodes + 2) );
		uint32_t cap = 1024;
		ent* e = (ent*)malloc( sizeof( ent ) * cap );
		#pragma omp for schedule( dynamic, 16 )
		for (int64_t i = 0; i < (int64_t)n; i++)
		{
			const ray_t R = load( rays, stride, i );
			uint32_t m = 0;
			if (R.tmax >= 0.0f)
			{
				node_bounds( nodes, used_nodes, &R, P, st );
				for (uint32_t nd = 0; nd < used_nodes; nd++)
				{
					if (P[nd] < 0.0f || !nodes[nd].cnt) continue;
					for (uint32_t r = nodes[nd].lf; r < nodes[nd].lf + nodes[nd].cnt; r++)
					{
						ent x;
						if (!tri_test( &R, verts, prim_idx, r, &x.t, &x.u, &x.v, &x.prim )) continue;
						x.key = fmaxf( x.t, P[nd] );
						if (m == cap) cap *= 2, e = (ent*)realloc( e, sizeof( ent ) * cap );
						e[m++] = x;
					}
				}
				/* each prim at its least key */
				qsort( e, m, sizeof( ent ), cmp_prim );
				uint32_t d = 0;
				for (uint32_t s = 0; s < m; s++) if (s == 0 || e[s].prim != e[s - 1].prim) e[d++] = e[s];
				m = d;
				qsort( e, m, sizeof( ent ), cmp_key );
			}
			write_row( hits, counts, keys, i, k, R.tmax, e, m < k ? m : k, m < k + 1 ? m : k + 1 );
		}
		free( P ), free( st ), free( e );
	}
}

/* the kernel's sorted buffer of at most c = k + 1 distinct prims */
static void insert( ent* buf, uint32_t* n, const uint32_t c, const ent* x )
{
	uint32_t j = *n;
	for (uint32_t i = 0; i < *n; i++) if (buf[i].prim == x->prim) { j = i; break; }
	if (j < *n) { if (!(x->key < buf[j].key)) return; }
	else if (*n == c) { if (!before( x, &buf[c - 1] )) return; j = c - 1; }
	else (*n)++;
	uint32_t pos = 0;
	while (pos < j && before( &buf[pos], x )) pos++;
	for (uint32_t i = j; i > pos; i--) buf[i] = buf[i - 1];
	buf[pos] = *x;
}

void orc_ah_walk( const node32* nodes, const uint32_t used_nodes, const uint32_t* prim_idx, const float* verts, const char* rays, const uint32_t stride,
	const uint64_t n, const uint32_t k, float* hits, uint32_t* counts, const int reverse )
{
	#pragma omp parallel
	{
		pend* st = (pend*)malloc( sizeof( pend ) * (used_nodes + 2) );
		ent* buf = (ent*)malloc( sizeof( ent ) * (k + 1) );
		#pragma omp for schedule( dynamic, 64 )
		for (int64_t i = 0; i < (int64_t)n; i++)
		{
			const ray_t R = load( rays, stride, i );
			uint32_t m = 0, node = 0;
			const uint32_t c = k + 1;
			int sp = 0;
			float P = 0.0f;
			while (R.tmax >= 0.0f)
			{
				const float b = m == c ? buf[c - 1].key : INFINITY;
				const node32* nd = nodes + node;
				int next = 0;
				if (!nd->cnt)
				{
					const uint32_t a = nd->lf, bb = nd->lf + 1;
					float ta, tb;
					const int ha = slab( &R, nodes + a, &ta ), hb = slab( &R, nodes + bb, &tb );
					const float Pa = fmaxf( P, ta ), Pb = fmaxf( P, tb );
					const int va = ha && !(Pa > b), vb = hb && !(Pb > b);
					if (va && vb)
					{
						const int swp = reverse ? !(Pb < Pa) : Pb < Pa;
						node = swp ? bb : a, P = swp ? Pb : Pa;
						st[sp++] = swp ? (pend){ a, Pa } : (pend){ bb, Pb };
						next = 1;
					}
					else if (va) node = a, P = Pa, next = 1;
					else if (vb) node = bb, P = Pb, next = 1;
				}
				else
				{
					for (uint32_t r = nd->lf; r < nd->lf + nd->cnt; r++)
					{
						ent x;
						if (!tri_test( &R, verts, prim_idx, r, &x.t, &x.u, &x.v, &x.prim )) continue;
						x.key = fmaxf( x.t, P );
						insert( buf, &m, c, &x );
					}
				}
				if (next) continue;
				const float b2 = m == c ? buf[c - 1].key : INFINITY;
				while (sp && st[sp - 1].P > b2) sp--;
				if (!sp) break;
				sp--, node = st[sp].node, P = st[sp].P;
			}
			write_row( hits, counts, 0, i, k, R.tmax, buf, m < k ? m : k, m );
		}
		free( st ), free( buf );
	}
}
