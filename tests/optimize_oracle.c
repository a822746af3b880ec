/* tests/optimize_oracle.c - the oracle of tbvh_optimize.  TEST INFRASTRUCTURE ONLY.
 *
 * The reference's optimiser (BVH::Optimize, tiny_bvh.h:3043, over BVH_Verbose::Optimize :4338) makes one reinsertion at a time, and
 * each one changes the tree the next one searches; no parallel optimiser can match it.  tbvh_optimize runs rounds of independent
 * reinsertions instead (Meister & Bittner 2018, "Parallel Reinsertion for Bounding Volume Hierarchy Optimization"), and this file
 * restates those rounds sequentially: every search on the round's tree, the winners taken in descending key order (what atomicMax
 * leaves), the same crossing rule, refold, acceptance, halving retry and numbering.  The rules are DESIGN.md §4.7.  Every float
 * operation that decides a move is written as the kernels write it; compiled with contraction off (tests/optimize_oracle.py).
 *
 * The tree lives in the reference's node layout throughout: a move copies four node records between the slots it owns, so a
 * node is named by its slot in the round's tree.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../oracle/tbvh_oracle.h"

#define OPT_NONE 0xffffffffu
#define OPT_VISITS 2048u /* stack pops per search: the fixed budget of tinybvh_b200/csrc/optimize.cu */

typedef struct { float mn[3], mx[3]; } box3;

static float sa( const box3 b ) /* BVHBase::SA :8477 in tbvh_sah_cost's pairing */
{
	const float ex = b.mx[0] - b.mn[0], ey = b.mx[1] - b.mn[1], ez = b.mx[2] - b.mn[2];
	return fmaf( ez, ex, fmaf( ey, ex, ey * ez ) );
}
static box3 fold( const box3 a, const box3 b ) /* tinybvh_min / tinybvh_max, a first */
{
	box3 r;
	for (int k = 0; k < 3; k++) r.mn[k] = a.mn[k] < b.mn[k] ? a.mn[k] : b.mn[k], r.mx[k] = a.mx[k] > b.mx[k] ? a.mx[k] : b.mx[k];
	return r;
}
static box3 nbox( const orc_node* n ) { box3 b = { { n->minx, n->miny, n->minz }, { n->maxx, n->maxy, n->maxz } }; return b; }
static void set_box( orc_node* n, const box3 b ) { n->minx = b.mn[0], n->miny = b.mn[1], n->minz = b.mn[2], n->maxx = b.mx[0], n->maxy = b.mx[1], n->maxz = b.mx[2]; }

typedef struct
{
	orc_node* nd;
	uint32_t n, L;
	uint32_t* parent, * depth, * height, * cand;
	float* area;
	uint64_t* key, * lock;
} opt_tree;

/* interior boxes refolded bottom-up (leaf boxes are never recomputed: an SBVH's are clipped), with every node's area and height */
static void refold( opt_tree* t, const uint32_t i )
{
	orc_node* x = &t->nd[i];
	if (x->triCount == 0)
	{
		const uint32_t l = x->leftFirst;
		t->parent[l] = t->parent[l + 1] = i;
		refold( t, l ), refold( t, l + 1 );
		set_box( x, fold( nbox( &t->nd[l] ), nbox( &t->nd[l + 1] ) ) );
		t->height[i] = 1 + (t->height[l] > t->height[l + 1] ? t->height[l] : t->height[l + 1]);
	}
	else t->height[i] = 0;
	t->area[i] = sa( nbox( x ) );
}
static void depths( opt_tree* t, const uint32_t i, const uint32_t d )
{
	t->depth[i] = d;
	if (t->nd[i].triCount == 0) depths( t, t->nd[i].leftFirst, d + 1 ), depths( t, t->nd[i].leftFirst + 1, d + 1 );
}
/* the round's tree refolded: its SAHCost (orc_sah_cost, the reference's BVH::SAHCost) and depth */
static float settle( opt_tree* t, const float c_trav, const float c_int, uint32_t* depth )
{
	t->parent[0] = OPT_NONE;
	refold( t, 0 );
	*depth = t->height[0];
	return orc_sah_cost( t->nd, 0, c_trav, c_int );
}

/* step 2: N's best target X, branch-and-bound from the root, left child first; OPT_NONE when none beats N's own place */
static uint32_t search( const opt_tree* t, const uint32_t N, uint32_t* st, float* sc )
{
	const uint32_t P = t->parent[N], S = t->nd[P].leftFirst == N ? N + 1 : N - 1;
	const box3 bN = nbox( &t->nd[N] );
	const float aN = t->area[N];
	const uint32_t hN = t->height[N];
	float best = t->area[P]; /* the induced cost of N's own place: A( S u N ), and no ancestor grows */
	uint32_t bestX = OPT_NONE, sp = 0, visits = 0;
	st[sp] = 0, sc[sp++] = 0.0f;
	while (sp > 0 && visits < OPT_VISITS)
	{
		visits++;
		const uint32_t x = st[--sp];
		const float ci = sc[sp];
		if (x == N) continue;
		if (!(ci + aN < best)) continue;
		const float aU = sa( fold( nbox( &t->nd[x] ), bN ) );
		if (x != P && x != S && t->depth[x] + 1 + hN <= t->L)
		{
			const float c = ci + aU;
			if (c < best) best = c, bestX = x;
		}
		if (t->nd[x].triCount == 0)
		{
			const float ci2 = ci + (aU - t->area[x]);
			const uint32_t l = t->nd[x].leftFirst;
			st[sp] = l + 1, sc[sp++] = ci2;
			st[sp] = l, sc[sp++] = ci2;
		}
	}
	return bestX;
}

/* step 3: the area the move N -> next to X saves on the round's tree.  Removal: S takes P's place, G and its ancestors
 * shrink (climb 1, up to the node below M, where M is the meeting point of X's path and G's path).  Insertion: P' = X u N in X's
 * place, its ancestors in the tree without N grow (climb 2).  Sum: climb 1's terms from G up, then P, then climb 2's from X's
 * parent up. */
static float area_saved( const opt_tree* t, const uint32_t N, const uint32_t X )
{
	const orc_node* nd = t->nd;
	const uint32_t* par = t->parent, * dep = t->depth;
	const uint32_t P = par[N], S = nd[P].leftFirst == N ? N + 1 : N - 1, G = par[P], PX = par[X];
	/* M: the deepest common ancestor of X's parent and G (X the root: above it, depth -1) */
	int dM = -1;
	if (G != OPT_NONE && PX != OPT_NONE)
	{
		uint32_t a = PX, b = G;
		while (dep[a] > dep[b]) a = par[a];
		while (dep[b] > dep[a]) b = par[b];
		while (a != b) a = par[a], b = par[b];
		dM = (int)dep[a];
	}
	float s = 0.0f;
	uint32_t J = OPT_NONE; /* the node of G's path just below M, and its box without N */
	box3 bJ = nbox( &nd[0] );
	if (G != OPT_NONE)
	{
		uint32_t q = G, came = P;
		box3 cb = nbox( &nd[S] );
		while (q != OPT_NONE && (int)dep[q] > dM)
		{
			const uint32_t l = nd[q].leftFirst;
			const box3 nb = fold( l == came ? cb : nbox( &nd[l] ), l + 1 == came ? cb : nbox( &nd[l + 1] ) );
			s = s + (t->area[q] - sa( nb ));
			if ((int)dep[q] == dM + 1) J = q, bJ = nb;
			came = q, cb = nb, q = par[q];
		}
	}
	box3 cb = fold( X == J ? bJ : nbox( &nd[X] ), nbox( &nd[N] ) );
	s = s + (t->area[P] - sa( cb ));
	uint32_t came = X;
	for (uint32_t q = PX; q != OPT_NONE; q = q == S ? G : par[q])
	{
		uint32_t l = nd[q].leftFirst, r = l + 1;
		if (l == P) l = S;
		if (r == P) r = S;
		const box3 lb = l == came ? cb : l == J ? bJ : nbox( &nd[l] ), rb = r == came ? cb : r == J ? bJ : nbox( &nd[r] );
		const box3 nb = fold( lb, rb );
		s = s + (t->area[q] - sa( nb ));
		came = q, cb = nb;
	}
	return s;
}

/* a winner's move on the node array: S's record into P's slot, P' (X, N) into X's slot, X and N into P's child pair */
static void apply( orc_node* nd, const uint32_t* par, const uint32_t N, const uint32_t X )
{
	const uint32_t P = par[N], c = nd[P].leftFirst, S = c == N ? N + 1 : N - 1;
	const orc_node rS = nd[S], rX = nd[X], rN = nd[N], rP = nd[P];
	nd[P] = rS;
	nd[X] = rP, nd[X].leftFirst = c, nd[X].triCount = 0;
	nd[c] = rX, nd[c + 1] = rN;
}

static int by_key_desc( const void* a, const void* b )
{
	const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
	return x < y ? 1 : x > y ? -1 : 0;
}

/* DFS preorder, the k-th interior node's children at 2 + 2k and 3 + 2k (BVH::ConvertFrom( BVH_Verbose )); returns the node count */
static uint32_t write_dfs( const orc_node* nd, const uint32_t i, orc_node* out, const uint32_t at, uint32_t nxt )
{
	out[at] = nd[i];
	if (nd[i].triCount > 0) return nxt;
	const uint32_t c = nxt;
	out[at].leftFirst = c;
	nxt = write_dfs( nd, nd[i].leftFirst, out, c, nxt + 2 );
	return write_dfs( nd, nd[i].leftFirst + 1, out, c + 1, nxt );
}

static uint32_t tree_depth( const orc_node* nd, const uint32_t i )
{
	if (nd[i].triCount > 0) return 0;
	const uint32_t l = tree_depth( nd, nd[i].leftFirst ), r = tree_depth( nd, nd[i].leftFirst + 1 );
	return 1 + (l > r ? l : r);
}

/* tbvh_optimize's rounds over nodes[0 .. usedNodes) (node 1 unused, every other node in the tree).  out_nodes: room for usedNodes;
 * round_sah: NULL or room for max_rounds values, the SAHCost after each accepted round.  Returns the output's node count. */
uint32_t orc_optimize( const orc_node* nodes, uint32_t usedNodes, const uint32_t* primIdx, uint32_t idxCount, float c_trav, float c_int,
	uint32_t max_rounds, orc_node* out_nodes, uint32_t* rounds, float* sah, float* round_sah )
{
	(void)primIdx, (void)idxCount; /* leaves keep their ranges: primIdx is not read */
	const uint32_t n = usedNodes;
	opt_tree T = { 0 };
	opt_tree* t = &T;
	t->n = n;
	t->nd = (orc_node*)malloc( (size_t)n * sizeof( orc_node ) );
	orc_node* saved = (orc_node*)malloc( (size_t)n * sizeof( orc_node ) );
	memcpy( t->nd, nodes, (size_t)n * sizeof( orc_node ) );
	t->parent = (uint32_t*)calloc( n, 4 ), t->depth = (uint32_t*)calloc( n, 4 ), t->height = (uint32_t*)calloc( n, 4 ), t->cand = (uint32_t*)calloc( n, 4 );
	t->area = (float*)calloc( n, 4 );
	t->key = (uint64_t*)calloc( n, 8 ), t->lock = (uint64_t*)calloc( n, 8 );
	uint64_t* win = (uint64_t*)calloc( n, 8 );
	uint32_t* won = (uint32_t*)calloc( n, 4 ), * st = (uint32_t*)malloc( 4 * 260 );
	float* sc = (float*)malloc( 4 * 260 );
	const uint32_t d0 = tree_depth( nodes, 0 );
	t->L = d0 > 63 ? d0 : 63;
	uint32_t accepted = 0;
	float cost = 0.0f;
	if (nodes[0].triCount == 0)
	{
		uint32_t depth;
		cost = settle( t, c_trav, c_int, &depth );
		while (accepted < max_rounds)
		{
			depths( t, 0, 0 );
			for (uint32_t N = 2; N < n; N++)
			{
				t->key[N] = 0, t->cand[N] = search( t, N, st, sc );
				if (t->cand[N] == OPT_NONE) continue;
				const float g = c_trav * area_saved( t, N, t->cand[N] );
				uint32_t gb;
				memcpy( &gb, &g, 4 );
				if (g > 0.0f && g <= 3.40282347e38f) t->key[N] = ((uint64_t)gb << 32) | N;
			}
			memset( t->lock, 0, (size_t)n * 8 ), memset( won, 0, (size_t)n * 4 );
			for (uint32_t N = 2; N < n; N++) if (t->key[N])
			{
				const uint32_t X = t->cand[N], P = t->parent[N], S = t->nd[P].leftFirst == N ? N + 1 : N - 1;
				const uint32_t v[6] = { N, P, S, t->parent[P], X, t->parent[X] };
				for (int k = 0; k < 6; k++) if (v[k] != OPT_NONE && t->lock[v[k]] < t->key[N]) t->lock[v[k]] = t->key[N];
			}
			for (uint32_t N = 2; N < n; N++) if (t->key[N])
			{
				const uint32_t X = t->cand[N], P = t->parent[N], S = t->nd[P].leftFirst == N ? N + 1 : N - 1;
				const uint32_t v[6] = { N, P, S, t->parent[P], X, t->parent[X] };
				int all = 1;
				for (int k = 0; k < 6; k++) if (v[k] != OPT_NONE && t->lock[v[k]] != t->key[N]) all = 0;
				won[N] = all;
			}
			uint32_t m = 0;
			for (uint32_t N = 2; N < n; N++) if (won[N])
			{
				int crossed = 0;
				for (uint32_t y = t->cand[N]; y != OPT_NONE; y = t->parent[y]) if (y != N && won[y]) crossed = 1;
				if (!crossed) win[m++] = t->key[N];
			}
			if (m == 0) break;
			qsort( win, m, 8, by_key_desc );
			memcpy( saved, t->nd, (size_t)n * sizeof( orc_node ) );
			const uint32_t* par = t->parent; /* the round's parents: settle() below overwrites them only after the moves */
			uint32_t* rpar = (uint32_t*)malloc( (size_t)n * 4 );
			memcpy( rpar, par, (size_t)n * 4 );
			int ok = 0;
			for (;;)
			{
				for (uint32_t k = 0; k < m; k++) { const uint32_t N = (uint32_t)(win[k] & 0xffffffffu); apply( t->nd, rpar, N, t->cand[N] ); }
				uint32_t d;
				const float c = settle( t, c_trav, c_int, &d );
				if (c < cost && d <= t->L) { cost = c, ok = 1; break; }
				memcpy( t->nd, saved, (size_t)n * sizeof( orc_node ) );
				if (m == 1) break;
				m /= 2;
			}
			free( rpar );
			if (!ok) break;
			if (round_sah) round_sah[accepted] = cost;
			accepted++;
		}
	}
	uint32_t used = n;
	if (accepted == 0) { memcpy( out_nodes, nodes, (size_t)n * sizeof( orc_node ) ); cost = orc_sah_cost( nodes, 0, c_trav, c_int ); }
	else used = write_dfs( t->nd, 0, out_nodes, 0, 2 ), memset( &out_nodes[1], 0, sizeof( orc_node ) );
	if (rounds) *rounds = accepted;
	if (sah) *sah = cost;
	free( t->nd ), free( saved ), free( t->parent ), free( t->depth ), free( t->height ), free( t->cand ), free( t->area ), free( t->key ), free( t->lock );
	free( win ), free( won ), free( st ), free( sc );
	return used;
}
