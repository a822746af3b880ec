/* tests/ploc_oracle.c - the oracle of TBVH_BUILD_PLOC.  TEST INFRASTRUCTURE ONLY.
 *
 * The reference has no bottom-up builder; tinybvh_b200/csrc/build_ploc.cu builds trees by parallel locally-ordered clustering
 * (Meister & Bittner 2018, "Parallel Locally-Ordered Clustering for Bounding Volume Hierarchy Construction"), and this file restates
 * its rules sequentially for one mesh: fragments, Morton order, clustering iterations, SAH leaf collapse, DFS numbering and the
 * boxes BVH::Refit computes.  The rules are DESIGN.md §4.8.  Every float operation that decides anything is written as the kernels
 * write it; compiled with contraction off (tests/ploc_oracle.py).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../oracle/tbvh_oracle.h"

#define PLOC_R 16        /* search radius (build_ploc.cu PLOC_R) */
#define PLOC_MAX_LEAF 4  /* most triangles of a collapsed leaf (build_ploc.cu PLOC_MAX_LEAF) */
#define PLOC_BITS 21     /* Morton bits per axis */
#define NONE 0xffffffffu

typedef struct { float mn[3], mx[3]; } box3;
typedef struct { box3 b; uint32_t lf, cnt; } rec; /* a node record: leaf (cnt 1, lf = sorted position) or interior (cnt 0, lf = child pair) */

static float fmn( const float a, const float b ) { return a < b ? a : b; } /* tinybvh_min */
static float fmx( const float a, const float b ) { return a > b ? a : b; } /* tinybvh_max */
static box3 fold( const box3 lo, const box3 hi )
{
	box3 r;
	for (int k = 0; k < 3; k++) r.mn[k] = fmn( lo.mn[k], hi.mn[k] ), r.mx[k] = fmx( lo.mx[k], hi.mx[k] );
	return r;
}
static float half_area( const box3 b ) /* oracle half_area */
{
	const float ex = b.mx[0] - b.mn[0], ey = b.mx[1] - b.mn[1], ez = b.mx[2] - b.mn[2];
	return fmaf( ez, ex, fmaf( ey, ex, ey * ez ) );
}
static uint32_t area_key( const float f ) /* ordered key, NaN above +inf */
{
	uint32_t u;
	memcpy( &u, &f, 4 );
	if (f != f) return 0xffffffffu;
	return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
static uint32_t quant( const float c, const float mn, const float ext )
{
	if (!(ext > 0.0f) || !(ext <= 3.40282347e38f)) return 0;
	const float f = ((c - mn) / ext) * 2097152.0f;
	if (!(f > 0.0f)) return 0;
	if (f >= 2097151.0f) return 2097151u;
	return (uint32_t)f;
}
static uint64_t spread21( const uint32_t v )
{
	uint64_t x = v & 0x1fffffu;
	x = (x | x << 32) & 0x1f00000000ffffull;
	x = (x | x << 16) & 0x1f0000ff0000ffull;
	x = (x | x << 8) & 0x100f00f00f00f00full;
	x = (x | x << 4) & 0x10c30c30c30c30c3ull;
	x = (x | x << 2) & 0x1249249249249249ull;
	return x;
}
typedef struct { uint64_t code; uint32_t idx; } mkey;
static int by_code( const void* a, const void* b )
{
	const mkey* x = (const mkey*)a, * y = (const mkey*)b;
	if (x->code != y->code) return x->code < y->code ? -1 : 1;
	return x->idx < y->idx ? -1 : x->idx > y->idx ? 1 : 0;
}

typedef struct
{
	rec* pool;          /* node slots: the root at 0, slot 1 unused, merge k's pair at 2 + 2k */
	uint32_t* parent, * cnt, * coll;
	float* cost;
	const uint32_t* order; /* sorted position -> triangle */
	float c_trav, c_int;
} ploc_tree;

static void set_parents( ploc_tree* T, const rec r, const uint32_t slot )
{
	if (r.cnt == 0) T->parent[r.lf] = T->parent[r.lf + 1] = slot;
}
/* step 4: triangles, cost and the collapse decision of every slot, children first */
static void collapse( ploc_tree* T, const uint32_t s )
{
	const rec* r = &T->pool[s];
	const float A = half_area( r->b );
	if (r->cnt == 1) { T->cnt[s] = 1, T->cost[s] = T->c_int * A * 1.0f, T->coll[s] = 0; return; }
	collapse( T, r->lf ), collapse( T, r->lf + 1 );
	const uint32_t N = T->cnt[r->lf] + T->cnt[r->lf + 1];
	const float leafc = T->c_int * A * (float)N, intc = T->c_trav * A + T->cost[r->lf] + T->cost[r->lf + 1];
	T->coll[s] = N <= PLOC_MAX_LEAF && leafc <= intc;
	T->cnt[s] = N, T->cost[s] = T->coll[s] ? leafc : intc;
}
static uint32_t emit_tris( const ploc_tree* T, const uint32_t s, uint32_t* primIdx, uint32_t at )
{
	const rec* r = &T->pool[s];
	if (r->cnt == 1) { primIdx[at] = T->order[r->lf]; return at + 1; }
	at = emit_tris( T, r->lf, primIdx, at );
	return emit_tris( T, r->lf + 1, primIdx, at );
}
/* step 5: DFS preorder, the k-th interior node's children at 2 + 2k, 3 + 2k; returns the next free slot */
static uint32_t write_dfs( const ploc_tree* T, const uint32_t s, orc_node* out, const uint32_t at, uint32_t nxt, uint32_t* primIdx, uint32_t* prim )
{
	const rec* r = &T->pool[s];
	orc_node* o = &out[at];
	o->minx = r->b.mn[0], o->miny = r->b.mn[1], o->minz = r->b.mn[2], o->maxx = r->b.mx[0], o->maxy = r->b.mx[1], o->maxz = r->b.mx[2];
	if (r->cnt == 1 || T->coll[s])
	{
		o->leftFirst = *prim, o->triCount = T->cnt[s];
		*prim = emit_tris( T, s, primIdx, *prim );
		return nxt;
	}
	const uint32_t c = nxt;
	o->leftFirst = c, o->triCount = 0;
	nxt = write_dfs( T, r->lf, out, c, nxt + 2, primIdx, prim );
	return write_dfs( T, r->lf + 1, out, c + 1, nxt, primIdx, prim );
}

/* The PLOC tree of one mesh: verts primCount*3 float4; nodes: room for 2*primCount+2; primIdx: room for primCount.  Returns usedNodes;
 * *iterations: clustering iterations; *sah: SAHCost of the result (orc_sah_cost). */
uint32_t orc_build_ploc( const float* verts, uint32_t primCount, float c_trav, float c_int, orc_node* nodes, uint32_t* primIdx, uint32_t* iterations, float* sah )
{
	const uint32_t n = primCount;
	/* step 1: fragments and the root box (bounds ordered as keys) */
	box3* frag = (box3*)malloc( (size_t)n * sizeof( box3 ) );
	box3 root;
	for (uint32_t i = 0; i < n; i++)
	{
		const float* v0 = verts + (size_t)i * 12, * v1 = v0 + 4, * v2 = v0 + 8;
		for (int a = 0; a < 3; a++) frag[i].mn[a] = fmn( v0[a], fmn( v1[a], v2[a] ) ), frag[i].mx[a] = fmx( v0[a], fmx( v1[a], v2[a] ) );
		if (i == 0) root = frag[0];
		else for (int a = 0; a < 3; a++)
		{
			if (area_key( frag[i].mn[a] ) < area_key( root.mn[a] )) root.mn[a] = frag[i].mn[a];
			if (area_key( frag[i].mx[a] ) > area_key( root.mx[a] )) root.mx[a] = frag[i].mx[a];
		}
	}
	/* step 2: Morton order */
	mkey* mk = (mkey*)malloc( (size_t)n * sizeof( mkey ) );
	float ext[3];
	for (int a = 0; a < 3; a++) ext[a] = root.mx[a] - root.mn[a];
	for (uint32_t i = 0; i < n; i++)
	{
		uint32_t q[3];
		for (int a = 0; a < 3; a++) q[a] = quant( (frag[i].mn[a] + frag[i].mx[a]) * 0.5f, root.mn[a], ext[a] );
		mk[i].code = spread21( q[0] ) << 2 | spread21( q[1] ) << 1 | spread21( q[2] ), mk[i].idx = i;
	}
	qsort( mk, n, sizeof( mkey ), by_code );
	uint32_t* order = (uint32_t*)malloc( (size_t)n * 4 );
	rec* cl = (rec*)malloc( (size_t)n * sizeof( rec ) ), * nx = (rec*)malloc( (size_t)n * sizeof( rec ) );
	for (uint32_t p = 0; p < n; p++) order[p] = mk[p].idx, cl[p].b = frag[mk[p].idx], cl[p].lf = p, cl[p].cnt = 1;
	/* step 3: clustering */
	ploc_tree T = { 0 };
	const size_t slots = 2 * (size_t)n;
	T.pool = (rec*)calloc( slots, sizeof( rec ) ), T.parent = (uint32_t*)malloc( slots * 4 ), T.cnt = (uint32_t*)calloc( slots, 4 ), T.coll = (uint32_t*)calloc( slots, 4 );
	T.cost = (float*)calloc( slots, 4 ), T.order = order, T.c_trav = c_trav, T.c_int = c_int;
	uint32_t* nn = (uint32_t*)malloc( (size_t)n * 4 );
	uint32_t m = n, iters = 0, pairs = 1;
	while (m > 1)
	{
		iters++;
		for (uint32_t i = 0; i < m; i++)
		{
			const uint32_t lo = i > PLOC_R ? i - PLOC_R : 0, hi = i + PLOC_R < m - 1 ? i + PLOC_R : m - 1;
			uint32_t best = NONE, bk = 0, bd = 0, bp = 0;
			for (uint32_t j = lo; j <= hi; j++) if (j != i)
			{
				const uint32_t k = area_key( half_area( j < i ? fold( cl[j].b, cl[i].b ) : fold( cl[i].b, cl[j].b ) ) );
				const uint32_t d = j < i ? i - j : j - i, par = j == (i ^ 1u) ? 0 : 1;
				if (best == NONE || k < bk || (k == bk && (d < bd || (d == bd && par < bp)))) best = j, bk = k, bd = d, bp = par;
			}
			nn[i] = best;
		}
		uint32_t w = 0;
		for (uint32_t i = 0; i < m; i++)
		{
			const uint32_t j = nn[i];
			if (nn[j] != i) { nx[w++] = cl[i]; continue; }
			if (j < i) continue;
			const uint32_t P = pairs++;
			T.pool[2 * P] = cl[i], T.pool[2 * P + 1] = cl[j];
			set_parents( &T, cl[i], 2 * P ), set_parents( &T, cl[j], 2 * P + 1 );
			nx[w].b = fold( cl[i].b, cl[j].b ), nx[w].lf = 2 * P, nx[w].cnt = 0, w++;
		}
		rec* tmp = cl; cl = nx, nx = tmp;
		m = w;
	}
	T.pool[0] = cl[0], T.parent[0] = NONE;
	set_parents( &T, cl[0], 0 );
	/* steps 4 and 5 */
	collapse( &T, 0 );
	memset( nodes, 0, 2 * sizeof( orc_node ) );
	uint32_t prim = 0;
	const uint32_t used = write_dfs( &T, 0, nodes, 0, 2, primIdx, &prim );
	orc_refit( nodes, used, primIdx, verts );
	if (iterations) *iterations = iters;
	if (sah) *sah = orc_sah_cost( nodes, 0, c_trav, c_int );
	free( frag ), free( mk ), free( order ), free( cl ), free( nx ), free( nn );
	free( T.pool ), free( T.parent ), free( T.cnt ), free( T.coll ), free( T.cost );
	return used;
}
