/* tests/toi_oracle.c - the oracle of tbvh_mesh_toi / tbvh_mesh_toi_pairs.  TEST INFRASTRUCTURE ONLY.
 *
 * The engine's times of impact between moving meshes (tinybvh_b200/csrc/mesh_toi.cu) follow their own definition, DESIGN.md §4.15; this
 * file restates it on the host in the same fp32 operation order (every fused pair written as fmaf, compiled with contraction off by
 * tests/toi_oracle.py), over the restatement of the pair distance tt_dist2 (meshdist_oracle.c), which it includes:
 *  - orc_toi_pairs: conservative advancement of arrays of triangle pairs (both frames of both triangles);
 *  - orc_toi_tree:  every reference (leaf, j) of B's tree reached for every triangle i of A through the swept boxes, which are built here
 *                   from the tree's topology: brute = 1 takes every reached leaf and advances every pair to its end (the definition);
 *                   brute = 0 is the walk the kernel runs, which abandons a pair once it cannot beat the best record.  The nearest form
 *                   writes the 16-byte records { t, d, j, iters }; the pairs form gives per-triangle counts and, on a second call with
 *                   offsets, the raw keys (i << 32) | j.
 * Trees are the reference's 32-byte node arrays (node 0 the root, node 1 unused, children paired at leftFirst); vertices are float4,
 * three per primitive, start frame and end frame alike.
 */
#include "meshdist_oracle.c"

#define L_UP 1.0000152587890625f

/* the nine coordinates of three corners at t: fma( t, x1, fma( -t, x0, x0 ) ) */
static void at9( const float* x0, const float* x1, const float t, float* r ) { for (int k = 0; k < 9; k++) r[k] = fmaf( t, x1[k], fmaf( -t, x0[k], x0[k] ) ); }
static float n2( const float* w ) { return fmaf( w[2], w[2], fmaf( w[1], w[1], w[0] * w[0] ) ); }

/* L( T, U ): the largest |dT_a - dU_b| over the nine corner pairs, rounded up */
static float speed( const float* t0, const float* t1, const float* u0, const float* u1 )
{
	float dT[9], dU[9], m = 0.0f;
	for (int k = 0; k < 9; k++) dT[k] = t1[k] - t0[k], dU[k] = u1[k] - u0[k];
	for (int a = 0; a < 3; a++)
		for (int b = 0; b < 3; b++)
		{
			float w[3];
			sub3( dT + 3 * a, dU + 3 * b, w );
			m = fmaxf( m, n2( w ) );
		}
	return sqrtf( m ) * L_UP;
}

/* mesh_toi.cu mt_pair on a finite pair: 1 with the contact time, squared distance and iterations, 0 for no contact; abandon: 0 once
 * the iterate ( t, j ) exceeds ( bt, bj ) */
static int toi_pair( const float* t0, const float* t1, const float* u0, const float* u1, const float eta, const float R2, const uint32_t max_iters,
	const int abandon, const uint32_t j, const float bt, const uint32_t bj, float* to, float* vo, uint32_t* io )
{
	const float L = speed( t0, t1, u0, u1 );
	float t = 0.0f;
	uint32_t it = 0;
	for (;;)
	{
		if (abandon && (t > bt || (t == bt && j > bj))) return 0;
		float T[9], U[9];
		at9( t0, t1, t, T ), at9( u0, u1, t, U );
		const float v = orc_tt_dist2( T, U );
		*to = t, *vo = v, *io = it;
		if (v <= R2) return 1;
		if (L == 0.0f) return 0;
		const float tn = t + (sqrtf( v ) - eta) / L;
		if (!(tn <= 1.0f)) return 0;
		if (tn == t || it == max_iters) { *io = max_iters; return 1; }
		t = tn, it++;
	}
}

static float r2_of( const float eta, const float xi ) { const float e = eta + xi; return e * e; }

/* n pairs (each argument n x 9 floats): out[4 k ..] = { t, d, iters, contact } (iters and contact as floats), NaN t for a pair with a
 * non-finite corner */
void orc_toi_pairs( const float* t0, const float* t1, const float* u0, const float* u1, const uint64_t n, const float eta, const float xi,
	const uint32_t max_iters, float* out )
{
	const float R2 = r2_of( eta, xi );
	for (uint64_t k = 0; k < n; k++)
	{
		float* o = out + k * 4;
		if (!finite9( t0 + k * 9 ) || !finite9( t1 + k * 9 ) || !finite9( u0 + k * 9 ) || !finite9( u1 + k * 9 )) { o[0] = NAN, o[1] = NAN, o[2] = 0, o[3] = 0; continue; }
		float t, v;
		uint32_t it;
		const int c = toi_pair( t0 + k * 9, t1 + k * 9, u0 + k * 9, u1 + k * 9, eta, R2, max_iters, 0, 0, 0.0f, 0, &t, &v, &it );
		o[0] = c ? t : INFINITY, o[1] = c ? sqrtf( v ) : INFINITY, o[2] = (float)(c ? it : 0), o[3] = (float)c;
	}
}

static void grow( float* mn, float* mx, const float* p ) { for (int k = 0; k < 3; k++) mn[k] = fminf( mn[k], p[k] ), mx[k] = fmaxf( mx[k], p[k] ); }
static void swept( const float* c0, const float* c1, float* mn, float* mx )
{
	for (int k = 0; k < 3; k++) mn[k] = INFINITY, mx[k] = -INFINITY;
	for (int c = 0; c < 3; c++) grow( mn, mx, c0 + 3 * c ), grow( mn, mx, c1 + 3 * c );
}

/* the swept box of every node reachable from the root (6 floats each): the box of both frames of every triangle below */
static void swept_nodes( const node32* nodes, const uint32_t used, const uint32_t* prim_idx, const float* v0, const float* v1, float* SB )
{
	uint8_t* done = (uint8_t*)calloc( used, 1 );
	uint32_t* stk = (uint32_t*)malloc( sizeof( uint32_t ) * (size_t)(2 * used + 2) );
	int sp = 0;
	stk[sp++] = 0;
	while (sp)
	{
		const uint32_t x = stk[sp - 1];
		if (done[x]) { sp--; continue; }
		const node32* nd = nodes + x;
		float* b = SB + (size_t)x * 6;
		if (nd->cnt)
		{
			for (int k = 0; k < 3; k++) b[k] = INFINITY, b[3 + k] = -INFINITY;
			for (uint32_t r = 0; r < nd->cnt; r++)
			{
				float c0[9], c1[9];
				corners( v0, prim_idx[nd->lf + r], c0 ), corners( v1, prim_idx[nd->lf + r], c1 );
				for (int c = 0; c < 3; c++) grow( b, b + 3, c0 + 3 * c ), grow( b, b + 3, c1 + 3 * c );
			}
			done[x] = 1, sp--;
			continue;
		}
		const uint32_t a = nd->lf, c = nd->lf + 1;
		if (!done[a] || !done[c])
		{
			if (!done[a]) stk[sp++] = a;
			if (!done[c]) stk[sp++] = c;
			continue;
		}
		for (int k = 0; k < 3; k++) b[k] = fminf( SB[(size_t)a * 6 + k], SB[(size_t)c * 6 + k] ), b[3 + k] = fmaxf( SB[(size_t)a * 6 + 3 + k], SB[(size_t)c * 6 + 3 + k] );
		done[x] = 1, sp--;
	}
	free( done );
	free( stk );
}

typedef struct { float bt, bv; uint32_t bj, bit; uint64_t found; uint64_t* keys; uint64_t o; } toi_state;

static void toi_consider( const float* vb0, const float* vb1, const uint64_t i, const uint32_t j, const float* t0, const float* t1, const float* mn,
	const float* mx, const float eta, const float R2, const uint32_t max_iters, const int self, const int nearest, const int abandon, toi_state* st )
{
	float u0[9], u1[9], umn[3], umx[3];
	if (self && (nearest ? j == i : j <= i)) return;
	corners( vb0, j, u0 ), corners( vb1, j, u1 );
	swept( u0, u1, umn, umx );
	if (box2( mn, mx, umn, umx ) > R2 || !finite9( u0 ) || !finite9( u1 )) return;
	if (self)
		for (int x = 0; x < 3; x++)
			for (int y = 0; y < 3; y++)
				if (t0[x * 3] == u0[y * 3] && t0[x * 3 + 1] == u0[y * 3 + 1] && t0[x * 3 + 2] == u0[y * 3 + 2] &&
					t1[x * 3] == u1[y * 3] && t1[x * 3 + 1] == u1[y * 3 + 1] && t1[x * 3 + 2] == u1[y * 3 + 2]) return;
	float t, v;
	uint32_t it;
	if (!toi_pair( t0, t1, u0, u1, eta, R2, max_iters, abandon, j, st->bt, st->bj, &t, &v, &it )) return;
	if (nearest) { if (t < st->bt || (t == st->bt && j < st->bj)) st->bt = t, st->bv = v, st->bj = j, st->bit = it; }
	else if (st->keys) st->keys[st->o++] = (i << 32) | j;
	else st->found++;
}

/* results (na x 4 words { t, d, j, iters }) for the nearest form, else counts (and keys at offsets) of the pairs form */
void orc_toi_tree( const node32* nodes, const uint32_t used, const uint32_t* prim_idx, const float* vb0, const float* vb1, const float* va0,
	const float* va1, const uint64_t na, const float eta, const float xi, const uint32_t max_iters, const int self, const int brute, float* results,
	uint32_t* counts, const uint64_t* offsets, uint64_t* keys )
{
	const int nearest = results != 0;
	const float R2 = r2_of( eta, xi );
	float* SB = (float*)malloc( sizeof( float ) * 6 * (size_t)(used + 2) );
	swept_nodes( nodes, used, prim_idx, vb0, vb1, SB );
	#pragma omp parallel
	{
		uint32_t* stk = (uint32_t*)malloc( sizeof( uint32_t ) * (size_t)(2 * used + 2) );
		uint8_t* seen = brute ? (uint8_t*)malloc( used + 2 ) : 0;
		#pragma omp for schedule( dynamic, 16 )
		for (int64_t ii = 0; ii < (int64_t)na; ii++)
		{
			const uint64_t i = (uint64_t)ii;
			float t0[9], t1[9], mn[3], mx[3];
			corners( va0, (uint32_t)i, t0 ), corners( va1, (uint32_t)i, t1 );
			swept( t0, t1, mn, mx );
			toi_state st = { INFINITY, INFINITY, NO_PRIM, 0, 0, keys, keys ? offsets[i] : 0 };
			if (finite9( t0 ) && finite9( t1 ))
			{
				int sp = 0;
				if (brute)
				{
					/* the reached nodes: the root, and every child of a reached interior node whose swept box passes the bound (a node's
					 * bound does not depend on the path); then every reference of every reached leaf, each pair advanced to its end */
					memset( seen, 0, used + 2 );
					stk[sp++] = 0, seen[0] = 1;
					while (sp)
					{
						const node32* nd = nodes + stk[--sp];
						if (nd->cnt) continue;
						for (uint32_t c = nd->lf; c < nd->lf + 2; c++)
							if (!seen[c] && !(box2( mn, mx, SB + (size_t)c * 6, SB + (size_t)c * 6 + 3 ) > R2)) seen[c] = 1, stk[sp++] = c;
					}
					for (uint32_t k = 0; k < used; k++)
						if (seen[k] && nodes[k].cnt)
							for (uint32_t x = 0; x < nodes[k].cnt; x++)
								toi_consider( vb0, vb1, i, prim_idx[nodes[k].lf + x], t0, t1, mn, mx, eta, R2, max_iters, self, nearest, 0, &st );
				}
				else
				{
					uint32_t node = 0;
					for (;;)
					{
						const node32* nd = nodes + node;
						int next = 0;
						if (!nd->cnt)
						{
							const uint32_t a = nd->lf, b = nd->lf + 1;
							const int ha = !(box2( mn, mx, SB + (size_t)a * 6, SB + (size_t)a * 6 + 3 ) > R2), hb = !(box2( mn, mx, SB + (size_t)b * 6, SB + (size_t)b * 6 + 3 ) > R2);
							if (ha && hb) stk[sp++] = b, node = a, next = 1;
							else if (ha) node = a, next = 1;
							else if (hb) node = b, next = 1;
						}
						else
							for (uint32_t x = 0; x < nd->cnt; x++)
								toi_consider( vb0, vb1, i, prim_idx[nd->lf + x], t0, t1, mn, mx, eta, R2, max_iters, self, nearest, nearest, &st );
						if (next) continue;
						if (!sp) break;
						node = stk[--sp];
					}
				}
			}
			if (nearest)
			{
				float* o = results + i * 4;
				const uint32_t it = st.bj == NO_PRIM ? 0 : st.bit;
				o[0] = st.bt, o[1] = st.bj == NO_PRIM ? INFINITY : sqrtf( st.bv );
				memcpy( o + 2, &st.bj, 4 ), memcpy( o + 3, &it, 4 );
			}
			else if (!keys) counts[i] = (uint32_t)st.found;
		}
		free( stk );
		free( seen );
	}
	free( SB );
}
