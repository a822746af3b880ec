/* tests/meshdist_oracle.c - the oracle of tbvh_mesh_distance / tbvh_mesh_distance_pairs.  TEST INFRASTRUCTURE ONLY.
 *
 * The engine's distances between meshes (tinybvh_b200/csrc/mesh_distance.cu) follow their own definition, DESIGN.md §4.13; this file
 * restates it on the host in the same fp32 operation order (every fused pair written as fmaf, compiled with contraction off by
 * tests/meshdist_oracle.py), over the restatements of the per-triangle point function (closest_oracle.c) and of the pair test
 * (tritri_oracle.c), which it includes:
 *  - orc_tt_dist2_pairs: the pair distance tt_dist2 over arrays of triangle pairs (NaN for a pair with a non-finite coordinate);
 *  - orc_md_tree:        every reference (leaf, j) of B's tree for every triangle i of A: brute = 1 takes every reachable leaf at the least
 *                        path bound over its paths, no pruning (the definition); brute = 0 is the pruned walk the kernel runs.  The nearest
 *                        form writes the 8-byte records { d, j }; the pairs form gives per-triangle counts and, on a second call with
 *                        offsets, the raw keys (i << 32) | j in walk order.
 * Trees are the reference's 32-byte node arrays (node 0 the root, node 1 unused, children paired at leftFirst); vertices are float4,
 * three per primitive.
 */
#include "closest_oracle.c"
/* the two restatements share helper names: the pair test's are renamed here */
#define node32 tt_node32
#define dot3 tt_dot3
#define pow2 tt_pow2
#include "tritri_oracle.c"
#undef node32
#undef dot3
#undef pow2

static int finite9( const float* a ) { for (int k = 0; k < 9; k++) if (!(fabsf( a[k] ) <= FLT_MAX)) return 0; return 1; }

/* the squared distance from p to the triangle (v0, v1, v2): orc_cp_triangle on (v0, v1 - v0, v2 - v0) */
static float md_point( const float* p, const float* v0, const float* v1, const float* v2 )
{
	float e1[3], e2[3], u, v;
	sub3( v1, v0, e1 ), sub3( v2, v0, e2 );
	return orc_cp_triangle( p, v0, e1, e2, &u, &v );
}

/* the edge-edge candidate of (p, p1) and (q, q1) at the unclamped solution by cross products; INFINITY when there is none */
static float md_edges( const float* p, const float* p1, const float* q, const float* q1 )
{
	float d1[3], d2[3], r[3], w[3], n[3], a[3], b[3], x[3];
	sub3( p1, p, d1 ), sub3( q1, q, d2 ), sub3( p, q, r ), sub3( q, p, w );
	cross3( d1, d2, n );
	const float nn = tt_dot3( n, n );
	if (!(nn > 0.0f)) return INFINITY;
	cross3( w, d2, a ), cross3( w, d1, b );
	const float s = tt_dot3( a, n ) / nn, t = tt_dot3( b, n ) / nn;
	if (!(s >= 0.0f && s <= 1.0f && t >= 0.0f && t <= 1.0f)) return INFINITY;
	for (int k = 0; k < 3; k++) x[k] = fmaf( s, d1[k], r[k] ) - t * d2[k];
	return tt_dot3( x, x );
}

/* the squared distance from p to the segment (q, q1): the clamped projection */
static float md_seg( const float* p, const float* q, const float* q1 )
{
	float d[3], r[3], w[3];
	sub3( q1, q, d ), sub3( p, q, r );
	const float t = edge( tt_dot3( r, d ), tt_dot3( d, d ) );
	for (int k = 0; k < 3; k++) w[k] = r[k] - t * d[k];
	return tt_dot3( w, w );
}

/* mesh_distance.cu tt_dist2: a and b are three corners (9 floats) each, read as x + 0; NaN when either has a non-finite coordinate */
float orc_tt_dist2( const float* a_in, const float* b_in )
{
	float a[9], b[9];
	pos9( a_in, a ), pos9( b_in, b );
	if (!finite9( a ) || !finite9( b )) return NAN;
	if (orc_tt( a, b, 0 )) return 0.0f;
	int swap = 0;
	for (int k = 0; k < 9; k++) { const uint32_t ka = f2key( a[k] ), kb = f2key( b[k] ); if (ka != kb) { swap = kb < ka; break; } }
	const float* rt = swap ? b : a, * ru = swap ? a : b;
	float P[6][3], m = 0.0f, inv;
	for (int c = 0; c < 6; c++) for (int k = 0; k < 3; k++) { P[c][k] = (c < 3 ? rt : ru)[(c % 3) * 3 + k] - rt[k]; m = fmaxf( m, fabsf( P[c][k] ) ); }
	const float s = pow2( m, &inv );
	for (int c = 0; c < 6; c++) for (int k = 0; k < 3; k++) P[c][k] = P[c][k] * s;
	const float* T[3] = { P[0], P[1], P[2] }, * U[3] = { P[3], P[4], P[5] };
	float d = md_point( U[0], T[0], T[1], T[2] );
	d = fminf( d, md_point( U[1], T[0], T[1], T[2] ) );
	d = fminf( d, md_point( U[2], T[0], T[1], T[2] ) );
	d = fminf( d, md_point( T[0], U[0], U[1], U[2] ) );
	d = fminf( d, md_point( T[1], U[0], U[1], U[2] ) );
	d = fminf( d, md_point( T[2], U[0], U[1], U[2] ) );
	for (int k = 0; k < 3; k++) for (int l = 0; l < 3; l++) d = fminf( d, md_edges( T[k], T[(k + 1) % 3], U[l], U[(l + 1) % 3] ) );
	for (int k = 0; k < 3; k++) for (int l = 0; l < 3; l++) d = fminf( fminf( d, md_seg( U[k], T[l], T[(l + 1) % 3] ) ), md_seg( T[k], U[l], U[(l + 1) % 3] ) );
	return (d * inv) * inv;
}

/* orc_tt_dist2 over n pairs: a, b are n x 9 floats */
void orc_tt_dist2_pairs( const float* a, const float* b, const uint64_t n, float* out )
{
	for (uint64_t k = 0; k < n; k++) out[k] = orc_tt_dist2( a + k * 9, b + k * 9 );
}

/* the box-box bound of [mn, mx] against [bmn, bmx] */
static float box2( const float* mn, const float* mx, const float* bmn, const float* bmx )
{
	float g[3];
	for (int k = 0; k < 3; k++) g[k] = fmaxf( fmaxf( bmn[k] - mx[k], mn[k] - bmx[k] ), 0.0f );
	return fmaf( g[2], g[2], fmaf( g[1], g[1], g[0] * g[0] ) );
}

static void tri_box( const float* t, float* mn, float* mx )
{
	for (int k = 0; k < 3; k++) mn[k] = fminf( fminf( t[k], t[3 + k] ), t[6 + k] ), mx[k] = fmaxf( fmaxf( t[k], t[3 + k] ), t[6 + k] );
}

typedef struct { float best; uint32_t bj; uint64_t found; uint64_t* keys; uint64_t o; } md_state;

/* one reference j, reached with path bound P, against triangle i; nearest lowers best, the pairs form counts / writes value <= best */
static void md_consider( const float* vb, const uint64_t i, const uint32_t j, const float* t, const float* mn, const float* mx, const float P,
	const int self, const int nearest, md_state* st )
{
	float u[9], umn[3], umx[3];
	if (self && (nearest ? j == i : j <= i)) return;
	corners( vb, j, u );
	tri_box( u, umn, umx );
	const float lb = fmaxf( box2( mn, mx, umn, umx ), P );
	if (lb > st->best || !finite9( u )) return;
	if (self)
		for (int x = 0; x < 3; x++)
			for (int y = 0; y < 3; y++)
				if (t[x * 3] == u[y * 3] && t[x * 3 + 1] == u[y * 3 + 1] && t[x * 3 + 2] == u[y * 3 + 2]) return;
	const float v = fmaxf( orc_tt_dist2( t, u ), lb );
	if (nearest) { if (v < st->best || (v == st->best && j < st->bj)) st->best = v, st->bj = j; }
	else if (v <= st->best) { if (st->keys) st->keys[st->o++] = (i << 32) | j; else st->found++; }
}

typedef struct { uint32_t node; float P; } md_pend;

/* results (na x 2 words { d, j }) for the nearest form, else counts (and keys at offsets) of the pairs form at r */
void orc_md_tree( const node32* nodes, const uint32_t used, const uint32_t* prim_idx, const float* vb, const float* va, const uint64_t na,
	const float r, const int self, const int brute, float* results, uint32_t* counts, const uint64_t* offsets, uint64_t* keys )
{
	const int nearest = results != 0;
	#pragma omp parallel
	{
		size_t cap = used + 2;
		md_pend* stk = (md_pend*)malloc( sizeof( md_pend ) * cap );
		float* PB = brute ? (float*)malloc( sizeof( float ) * (used + 2) ) : 0;
		#pragma omp for schedule( dynamic, 16 )
		for (int64_t ii = 0; ii < (int64_t)na; ii++)
		{
			const uint64_t i = (uint64_t)ii;
			float t[9], mn[3], mx[3];
			corners( va, (uint32_t)i, t );
			tri_box( t, mn, mx );
			md_state st = { r * r, NO_PRIM, 0, keys, keys ? offsets[i] : 0 };
			if (finite9( t ))
			{
				if (brute)
				{
					/* the least path bound of every reachable node (orc_cp_node_bounds with the box-box bound), every reference of every
					 * reachable leaf at its leaf's bound: the nearest record is the walk's, the pairs are the walk's set */
					for (uint32_t k = 0; k < used; k++) PB[k] = -1.0f;
					int sp = 0;
					stk[sp++] = (md_pend){ 0, 0.0f };
					while (sp)
					{
						const md_pend e = stk[--sp];
						if (PB[e.node] < 0.0f || e.P < PB[e.node]) PB[e.node] = e.P;
						else continue;
						const node32* nd = nodes + e.node;
						if (nd->cnt) continue;
						if (sp + 2 > cap) cap *= 2, stk = (md_pend*)realloc( stk, sizeof( md_pend ) * cap );
						for (uint32_t c = nd->lf; c < nd->lf + 2; c++) stk[sp++] = (md_pend){ c, fmaxf( box2( mn, mx, nodes[c].mn, nodes[c].mx ), e.P ) };
					}
					for (uint32_t k = 0; k < used; k++)
					{
						if (PB[k] < 0.0f || !nodes[k].cnt || PB[k] > st.best) continue;
						for (uint32_t x = 0; x < nodes[k].cnt; x++) md_consider( vb, i, prim_idx[nodes[k].lf + x], t, mn, mx, PB[k], self, nearest, &st );
					}
				}
				else
				{
					int sp = 0;
					uint32_t node = 0;
					float P = 0.0f;
					while (1)
					{
						const node32* nd = nodes + node;
						int next = 0;
						if (!nd->cnt)
						{
							const uint32_t a = nd->lf, b = nd->lf + 1;
							const float Pa = fmaxf( box2( mn, mx, nodes[a].mn, nodes[a].mx ), P ), Pb = fmaxf( box2( mn, mx, nodes[b].mn, nodes[b].mx ), P );
							const int ha = !(Pa > st.best), hb = !(Pb > st.best);
							if (ha && hb)
							{
								const int swp = Pb < Pa;
								node = swp ? b : a, P = swp ? Pb : Pa;
								stk[sp++] = swp ? (md_pend){ a, Pa } : (md_pend){ b, Pb };
								next = 1;
							}
							else if (ha) node = a, P = Pa, next = 1;
							else if (hb) node = b, P = Pb, next = 1;
						}
						else
							for (uint32_t x = 0; x < nd->cnt; x++) md_consider( vb, i, prim_idx[nd->lf + x], t, mn, mx, P, self, nearest, &st );
						if (next) continue;
						while (sp && stk[sp - 1].P > st.best) sp--;
						if (!sp) break;
						sp--, node = stk[sp].node, P = stk[sp].P;
					}
				}
			}
			if (nearest)
			{
				const float d = st.bj == NO_PRIM ? r : sqrtf( st.best );
				results[i * 2] = d;
				memcpy( results + i * 2 + 1, &st.bj, 4 );
			}
			else if (!keys) counts[i] = (uint32_t)st.found;
		}
		free( stk );
		free( PB );
	}
}
