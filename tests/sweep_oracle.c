/* tests/sweep_oracle.c - the oracle of tbvh_sphere_cast / tbvh_sphere_cast_occluded.  TEST INFRASTRUCTURE ONLY.
 *
 * The engine's sphere casts (include/tinybvh_b200_device/sweep_walk.cuh) follow their own definition, DESIGN.md §4.16; this file restates
 * it on the host in the same fp32 operation order (every fused pair written as fmaf, compiled with contraction off by tests/sweep_oracle.py),
 * over closest_oracle.c, whose cp_triangle, pow2, dot3 and tree conventions it includes rather than copies:
 *  - orc_sc_triangle: the first contact of a moving sphere with one leaf record (v0, e1, e2);
 *  - orc_sc_brute:    every reached reference (leaf, triangle) with its path bound, no pruning - the definition itself;
 *  - orc_sc_walk:     the pruned walk of the same rules (nearer child first, strict pruning, pops pruned again), OpenMP over queries;
 *  - orc_sc_node_bounds: the path bound P of every reached node for one query.
 * A query is 8 floats { cx, cy, cz, r, dx, dy, dz, tmax }; results are { t, u, v, prim } records or overlap-style bit words.
 */
#include "closest_oracle.c"

static void cross3( const float* a, const float* b, float* o )
{
	o[0] = a[1] * b[2] - a[2] * b[1], o[1] = a[2] * b[0] - a[0] * b[2], o[2] = a[0] * b[1] - a[1] * b[0];
}

static int finite_( const float x ) { return fabsf( x ) <= 3.40282347e38f; }

static int sc_query_ok( const float* q )
{
	return finite_( q[0] ) && finite_( q[1] ) && finite_( q[2] ) && finite_( q[3] ) && q[3] >= 0.0f
		&& finite_( q[4] ) && finite_( q[5] ) && finite_( q[6] ) && q[7] >= 0.0f;
}

/* sweep_walk.cuh sc_root: c / (-b + sqrt( disc )) for c > 0, b < 0, disc >= 0 */
static int sc_root( const float b, const float c, const float disc, float* t )
{
	if (!(c > 0.0f) || !(b < 0.0f) || !(disc >= 0.0f)) return 0;
	*t = c / (-b + sqrtf( disc ));
	return 1;
}

/* sc_edge: the cylinder around A + s ev met by m0 + t D (m0 = centre - A); b^2 - a c = ev.ev ( a R^2 - (D . mx)^2 ) */
static int sc_edge( const float* m0, const float* ev, const float* D, const float RR, float* t, float* s )
{
	float dx[3], mx[3], w[3];
	const float ee = dot3( ev, ev );
	if (!(ee > 0.0f)) return 0;
	cross3( D, ev, dx ), cross3( m0, ev, mx );
	const float a = dot3( dx, dx ), g = dot3( D, mx );
	const float c = fmaf( -RR, ee, dot3( mx, mx ) );
	const float disc = fmaf( -g, g, a * RR ) * ee;
	if (!sc_root( dot3( dx, mx ), c, disc, t )) return 0;
	for (int k = 0; k < 3; k++) w[k] = fmaf( *t, D[k], m0[k] );
	const float num = dot3( w, ev );
	if (!(num >= 0.0f && num <= ee)) return 0;
	*s = num / ee;
	return 1;
}

/* sc_vertex: b^2 - a c = a R^2 - |D x m0|^2 */
static int sc_vertex( const float* m0, const float* D, const float DD, const float R, const float RR, float* t )
{
	float h[3];
	cross3( D, m0, h );
	return sc_root( dot3( D, m0 ), fmaf( -R, R, dot3( m0, m0 ) ), DD * RR - dot3( h, h ), t );
}

/* sweep_walk.cuh sc_triangle: q = 8 floats, the leaf record (v0, e1, e2) -> contact, t, u, v */
int orc_sc_triangle( const float* q, const float* v0, const float* e1r, const float* e2r, float* to, float* uo, float* vo )
{
	float u, v, r[3], P[3], E1[3], E2[3], D[3], B[3], C[3], BC[3], n[3], inv, invd, tc, w;
	if (orc_cp_triangle( q, v0, e1r, e2r, &u, &v ) <= q[3] * q[3]) { *to = 0.0f, *uo = u, *vo = v; return 1; }
	for (int k = 0; k < 3; k++) r[k] = q[k] - v0[k];
	const float m = fmaxf( fmaxf( fmaxf( fmaxf( fabsf( r[0] ), fabsf( r[1] ) ), fmaxf( fabsf( r[2] ), fabsf( e1r[0] ) ) ),
		fmaxf( fmaxf( fabsf( e1r[1] ), fabsf( e1r[2] ) ), fmaxf( fabsf( e2r[0] ), fabsf( e2r[1] ) ) ) ), fmaxf( fabsf( e2r[2] ), q[3] ) );
	const float s = pow2( m, &inv ), sd = pow2( fmaxf( fmaxf( fabsf( q[4] ), fabsf( q[5] ) ), fabsf( q[6] ) ), &invd );
	for (int k = 0; k < 3; k++) P[k] = r[k] * s, E1[k] = e1r[k] * s, E2[k] = e2r[k] * s, D[k] = q[4 + k] * sd;
	const float R = q[3] * s, RR = R * R;
	float best = 0.0f, bu = 0.0f, bv = 0.0f;
	int found = 0;
	/* face, at the corner K opposite the longest edge (ties: A, then B), n = a x b = e1 x e2 */
	for (int k = 0; k < 3; k++) BC[k] = E2[k] - E1[k];
	const float lab = dot3( E1, E1 ), lac = dot3( E2, E2 ), lbc = dot3( BC, BC );
	const int K = (lbc >= lab && lbc >= lac) ? 0 : lac >= lab ? 1 : 2;
	float a[3], b[3], PK[3];
	for (int k = 0; k < 3; k++)
	{
		a[k] = K == 0 ? E1[k] : K == 1 ? BC[k] : -E2[k];
		b[k] = K == 0 ? E2[k] : K == 1 ? -E1[k] : -BC[k];
		PK[k] = K == 0 ? P[k] : K == 1 ? P[k] - E1[k] : P[k] - E2[k];
	}
	const float la = K == 0 ? lab : K == 1 ? lbc : lac, lb = K == 0 ? lac : K == 1 ? lab : lbc, LL = K == 0 ? lbc : K == 1 ? lac : lab;
	cross3( a, b, n );
	const float nn = dot3( n, n );
	if (nn > (sqrtf( la * lb ) * LL) * 0x1p-22f) /* the plane's rounding stays below the triangle's width */
	{
		float h0 = dot3( PK, n ), hd = dot3( D, n );
		if (h0 < 0.0f) h0 = -h0, hd = -hd;
		const float num = fmaf( -R, sqrtf( nn ), h0 );
		if (num > 0.0f && hd < 0.0f)
		{
			float X[3], f[3], g[3];
			tc = num / -hd;
			for (int k = 0; k < 3; k++) X[k] = fmaf( tc, D[k], PK[k] );
			cross3( X, b, f ), cross3( a, X, g );
			const float in = 1.0f / nn;
			const float al = dot3( f, n ) * in, be = dot3( g, n ) * in;
			if (al >= 0.0f && be >= 0.0f && al + be <= 1.0f)
			{
				const float w0 = (1.0f - al) - be;
				best = tc, found = 1;
				bu = K == 0 ? al : K == 1 ? w0 : be;
				bv = K == 0 ? be : K == 1 ? al : w0;
			}
		}
	}
	/* edges AB, AC, BC */
	if (sc_edge( P, E1, D, RR, &tc, &w ) && (!found || tc < best)) best = tc, bu = w, bv = 0.0f, found = 1;
	if (sc_edge( P, E2, D, RR, &tc, &w ) && (!found || tc < best)) best = tc, bu = 0.0f, bv = w, found = 1;
	for (int k = 0; k < 3; k++) B[k] = P[k] - E1[k], C[k] = P[k] - E2[k];
	if (sc_edge( B, BC, D, RR, &tc, &w ) && (!found || tc < best)) best = tc, bu = 1.0f - w, bv = w, found = 1;
	/* vertices A, B, C */
	const float DD = dot3( D, D );
	if (sc_vertex( P, D, DD, R, RR, &tc ) && (!found || tc < best)) best = tc, bu = 0.0f, bv = 0.0f, found = 1;
	if (sc_vertex( B, D, DD, R, RR, &tc ) && (!found || tc < best)) best = tc, bu = 1.0f, bv = 0.0f, found = 1;
	if (sc_vertex( C, D, DD, R, RR, &tc ) && (!found || tc < best)) best = tc, bu = 0.0f, bv = 1.0f, found = 1;
	if (!found) return 0;
	const float t = (best * inv) * sd;
	if (!(t <= q[7])) return 0;
	*to = t, *uo = bu, *vo = bv;
	return 1;
}

/* a - b rounded down / a + b rounded up (the device's __fsub_rd / __fadd_ru): the round-to-nearest result, moved one step when the exact
 * error (Knuth's two-sum, exact in round-to-nearest) says it rounded the other way.  A zero result's sign never reaches an output. */
static float two_sum_err( const float a, const float b, const float s )
{
	const float bb = s - a;
	return (a - (s - bb)) + (b - bb);
}
static float sub_rd( const float a, const float b )
{
	const float s = a - b;
	return two_sum_err( a, -b, s ) < 0.0f ? nextafterf( s, -INFINITY ) : s;
}
static float add_ru( const float a, const float b )
{
	const float s = a + b;
	return two_sum_err( a, b, s ) > 0.0f ? nextafterf( s, INFINITY ) : s;
}

/* sweep_walk.cuh sc_axis / sc_box */
static void sc_axis( const float lo, const float hi, const float c, const float d, float* tn, float* tf )
{
	if (d == 0.0f)
	{
		const int in = lo <= c && c <= hi;
		*tn = in ? -INFINITY : INFINITY, *tf = in ? INFINITY : -INFINITY;
		return;
	}
	const float a = (lo - c) / d, b = (hi - c) / d;
	*tn = fminf( a, b ), *tf = fmaxf( a, b );
}
static int sc_box( const node32* nd, const float* q, float* tmin )
{
	float tn[3], tf[3];
	for (int k = 0; k < 3; k++) sc_axis( sub_rd( nd->mn[k], q[3] ), add_ru( nd->mx[k], q[3] ), q[k], q[4 + k], tn + k, tf + k );
	*tmin = fmaxf( fmaxf( fmaxf( tn[0], tn[1] ), tn[2] ), 0.0f );
	return *tmin <= fminf( fminf( fminf( tf[0], tf[1] ), tf[2] ), q[7] );
}

/* one reference against the running best: closest keeps the smallest (key, prim); any reports a contact */
static int sc_consider( const float* q, const float* verts, const uint32_t* prim_idx, const uint32_t r, const float P, const int any,
	float* best, float* bt, uint32_t* bprim, float* bu, float* bv )
{
	float v0[3], e1[3], e2[3], t, u, v;
	uint32_t prim;
	record( verts, prim_idx, r, v0, e1, e2, &prim );
	if (!orc_sc_triangle( q, v0, e1, e2, &t, &u, &v )) return 0;
	if (any) return 1;
	const float key = fmaxf( t, P );
	if (key < *best || (key == *best && prim < *bprim)) *best = key, *bt = t, *bprim = prim, *bu = u, *bv = v;
	return 0;
}

/* path bound of every node the root reaches for query q into P[used_nodes] (unreached slots: -1); a node reached on several paths (a
 * DAG) takes the least */
void orc_sc_node_bounds( const node32* nodes, const uint32_t used_nodes, const float* q, float* P )
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
		for (uint32_t c = n->lf; c < n->lf + 2; c++)
		{
			float t;
			if (sc_box( nodes + c, q, &t )) st[sp++] = (pend){ c, fmaxf( e.P, t ) };
		}
	}
	free( st );
}

static void sc_store( const int any, const int hit, const uint64_t i, const float* q, const float bt, const float bu, const float bv,
	const uint32_t bprim, float* results, uint32_t* bits )
{
	if (any) { if (hit) { _Pragma( "omp atomic" ) bits[i >> 5] |= 1u << (i & 31); } }
	else if (bprim == NO_PRIM) write_rec( results + i * 4, q[7], 0.0f, 0.0f, NO_PRIM );
	else write_rec( results + i * 4, bt, bu, bv, bprim );
}

/* the definition: every reached leaf with its least path bound, every reference of every such leaf */
void orc_sc_brute( const node32* nodes, const uint32_t used_nodes, const uint32_t* prim_idx, const float* verts, const float* queries,
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
			const float* q = queries + i * 8;
			float best = q[7], bt = q[7], bu = 0.0f, bv = 0.0f;
			uint32_t bprim = NO_PRIM;
			int hit = 0;
			if (sc_query_ok( q ))
			{
				orc_sc_node_bounds( nodes, used_nodes, q, P );
				for (uint32_t k = 0; k < used_nodes && !hit; k++)
				{
					if (P[k] < 0.0f || !nodes[k].cnt) continue;
					for (uint32_t t = 0; t < nodes[k].cnt && !hit; t++)
						hit = sc_consider( q, verts, prim_idx, nodes[k].lf + t, P[k], any, &best, &bt, &bprim, &bu, &bv );
				}
			}
			sc_store( any, hit, i, q, bt, bu, bv, bprim, results, bits );
		}
		free( P );
	}
}

/* the pruned walk the kernel runs, over the same rules */
void orc_sc_walk( const node32* nodes, const uint32_t used_nodes, const uint32_t* prim_idx, const float* verts, const float* queries,
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
			const float* q = queries + i * 8;
			float best = q[7], bt = q[7], bu = 0.0f, bv = 0.0f;
			uint32_t bprim = NO_PRIM;
			int hit = 0, sp = 0;
			uint32_t node = 0;
			float P = 0.0f;
			while (sc_query_ok( q ))
			{
				const node32* nd = nodes + node;
				int next = 0;
				if (!nd->cnt)
				{
					const uint32_t a = nd->lf, b = nd->lf + 1;
					float ta, tb;
					const int ha = sc_box( nodes + a, q, &ta ), hb = sc_box( nodes + b, q, &tb );
					const float Pa = fmaxf( P, ta ), Pb = fmaxf( P, tb );
					const int va = ha && !(Pa > best), vb = hb && !(Pb > best);
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
					for (uint32_t t = 0; t < nd->cnt && !hit; t++) hit = sc_consider( q, verts, prim_idx, nd->lf + t, P, any, &best, &bt, &bprim, &bu, &bv );
					if (hit) break;
				}
				if (next) continue;
				while (sp && st[sp - 1].P > best) sp--;
				if (!sp) break;
				sp--, node = st[sp].node, P = st[sp].P;
			}
			sc_store( any, hit, i, q, bt, bu, bv, bprim, results, bits );
		}
		free( st );
	}
}

/* orc_sc_triangle over arrays: queries (n x 8), records (n x 12: v0, e1, e2 as float4) -> out (n x 4: t, u, v, contact 1 / 0) */
void orc_sc_triangles( const float* queries, const float* recs, const uint64_t n, float* out )
{
	for (uint64_t i = 0; i < n; i++)
	{
		const float* r = recs + i * 12;
		float t = 0.0f, u = 0.0f, v = 0.0f;
		const int hit = orc_sc_triangle( queries + i * 8, r, r + 4, r + 8, &t, &u, &v );
		out[i * 4] = t, out[i * 4 + 1] = u, out[i * 4 + 2] = v, out[i * 4 + 3] = hit ? 1.0f : 0.0f;
	}
}
