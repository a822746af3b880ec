/* tests/allhits_tlas_oracle.c - the oracle of tbvh_intersect_all_tlas.  TEST INFRASTRUCTURE ONLY.
 *
 * Multi-hit rays through a TLAS (include/tinybvh_b200_device/all_hits_walk.cuh ah_walk_tlas) follow the rules of tests/allhits_oracle.c,
 * DESIGN.md §4.14, applied once to the TLAS and once more inside each instance; this file restates them on the host in the same fp32
 * operation order (compiled with contraction off by tests/allhits_tlas_oracle.py), over that file's ray record, slab test, triangle test
 * and node bounds, which it includes:
 *  - orc_ah_tlas_brute: the definition itself - every reached TLAS node with its path bound; per instance of a reached TLAS leaf whose mask
 *                       shares a bit with the ray's, the ray in BLAS space (oracle/tbvh_oracle.c transform_ray) and every reached BLAS
 *                       node with its path bound, the BLAS root at the TLAS leaf's; every accepted reference as an ( instance, prim ) hit
 *                       at key fmaxf( t, P ); each hit at its least key, the k smallest ( key, instance, prim ); also each record's key;
 *  - orc_ah_tlas_walk:  the pruned walk of the same rules (nearer child first and a leaf's instances in primIdx order, or - reverse - the
 *                       other child first and the leaf's instances from the last).
 * Instances are the reference's 192-byte BLASInstance records, already updated (invTransform at byte 64, blasIdx at 140, mask at 156).
 */
#include "allhits_oracle.c"

typedef struct { float key, t, u, v; uint32_t prim, inst; } ihit;
typedef struct { const node32* nodes; uint32_t used_nodes; const uint32_t* prim_idx; const float* verts; } blas_t;

/* keys as floats, ties to the lower instance, then to the lower prim */
static int ibefore( const ihit* a, const ihit* b )
{
	return a->key < b->key || (a->key == b->key && (a->inst < b->inst || (a->inst == b->inst && a->prim < b->prim)));
}
static int icmp_key( const void* x, const void* y ) { const ihit* a = x, * b = y; return ibefore( a, b ) ? -1 : ibefore( b, a ) ? 1 : 0; }
static int icmp_pair( const void* x, const void* y )
{
	const ihit* a = x, * b = y;
	if (a->inst != b->inst) return a->inst < b->inst ? -1 : 1;
	if (a->prim != b->prim) return a->prim < b->prim ? -1 : 1;
	return a->key < b->key ? -1 : b->key < a->key ? 1 : 0;
}

/* row i: k records and k instances (NO_PRIM past m), the count, and with keys each record's key */
static void write_irow( float* hits, uint32_t* insts, uint32_t* counts, float* keys, const uint64_t i, const uint32_t k, const float tmax,
	const ihit* e, const uint32_t m, const uint32_t count )
{
	float* row = hits + i * k * 4;
	for (uint32_t s = 0; s < k; s++)
	{
		const uint32_t p = s < m ? e[s].prim : NO_PRIM;
		row[s * 4] = s < m ? e[s].t : tmax, row[s * 4 + 1] = s < m ? e[s].u : 0.0f, row[s * 4 + 2] = s < m ? e[s].v : 0.0f;
		memcpy( row + s * 4 + 3, &p, 4 );
		insts[i * k + s] = s < m ? e[s].inst : NO_PRIM;
		if (keys) keys[i * k + s] = s < m ? e[s].key : tmax;
	}
	counts[i] = count;
}

/* the kernel's sorted buffer of at most c = k + 1 distinct ( instance, prim ) hits */
static void iinsert( ihit* buf, uint32_t* n, const uint32_t c, const ihit* x )
{
	uint32_t j = *n;
	for (uint32_t i = 0; i < *n; i++) if (buf[i].prim == x->prim && buf[i].inst == x->inst) { j = i; break; }
	if (j < *n) { if (!(x->key < buf[j].key)) return; }
	else if (*n == c) { if (!ibefore( x, &buf[c - 1] )) return; j = c - 1; }
	else (*n)++;
	uint32_t pos = 0;
	while (pos < j && ibefore( &buf[pos], x )) pos++;
	for (uint32_t i = j; i > pos; i--) buf[i] = buf[i - 1];
	buf[pos] = *x;
}

static uint32_t rec_u32( const char* rec, const int off ) { uint32_t x; memcpy( &x, rec + off, 4 ); return x; }

static float safercp( const float x ) { return (x > 1e-12f || x < -1e-12f) ? 1.0f / x : (x >= 0 ? 1e30f : -1e30f); }

/* the ray in the space of instance record `rec`, restating oracle/tbvh_oracle.c transform_ray: tinybvh_transform_point / _vector in the
 * reference build's pairing, the point divided by w only when w != 1, rD' = safercp( D' ); tmax carries over */
static ray_t to_blas( const ray_t* R, const char* rec )
{
	float T[16];
	memcpy( T, rec + 64, 64 );
	const float* O = R->O, * D = R->D;
	ray_t B = *R;
	float r[3];
	for (int a = 0; a < 3; a++) r[a] = fmaf( T[a * 4 + 2], O[2], fmaf( T[a * 4], O[0], T[a * 4 + 1] * O[1] ) ) + T[a * 4 + 3];
	const float w = fmaf( O[2], T[14], fmaf( O[0], T[12], O[1] * T[13] ) ) + T[15];
	if (!(w == 1)) { const float rw = 1.0f / w; for (int a = 0; a < 3; a++) r[a] = r[a] * rw; }
	for (int a = 0; a < 3; a++)
	{
		B.O[a] = r[a];
		B.D[a] = fmaf( T[a * 4 + 2], D[2], fmaf( T[a * 4], D[0], T[a * 4 + 1] * D[1] ) );
		B.rD[a] = safercp( B.D[a] );
		B.nro[a] = -(B.O[a] * B.rD[a]);
		B.pos[a] = B.D[a] >= 0;
	}
	return B;
}

/* the ray record's mask (O.w) */
static uint32_t ray_mask( const char* rays, const uint32_t stride, const uint64_t i ) { return rec_u32( rays + i * stride, 12 ); }

static uint32_t max_used( const uint32_t tlas_used, const blas_t* blas, const uint32_t nblas )
{
	uint32_t u = tlas_used;
	for (uint32_t b = 0; b < nblas; b++) if (blas[b].used_nodes > u) u = blas[b].used_nodes;
	return u + 2;
}

void orc_ah_tlas_brute( const node32* tnodes, const uint32_t tlas_used, const uint32_t* tprim_idx, const char* inst, const blas_t* blas, const uint32_t nblas,
	const char* rays, const uint32_t stride, const uint64_t n, const uint32_t k, float* hits, uint32_t* insts, uint32_t* counts, float* keys )
{
	const uint32_t mu = max_used( tlas_used, blas, nblas );
	#pragma omp parallel
	{
		float* PT = (float*)malloc( sizeof( float ) * mu ), * PB = (float*)malloc( sizeof( float ) * mu );
		pend* st = (pend*)malloc( sizeof( pend ) * mu );
		uint32_t cap = 1024;
		ihit* e = (ihit*)malloc( sizeof( ihit ) * cap );
		#pragma omp for schedule( dynamic, 16 )
		for (int64_t i = 0; i < (int64_t)n; i++)
		{
			const ray_t R = load( rays, stride, i );
			const uint32_t rmask = ray_mask( rays, stride, i );
			uint32_t m = 0;
			if (R.tmax >= 0.0f)
			{
				node_bounds( tnodes, tlas_used, &R, PT, st );
				for (uint32_t tn = 0; tn < tlas_used; tn++)
				{
					if (PT[tn] < 0.0f || !tnodes[tn].cnt) continue;
					for (uint32_t j = tnodes[tn].lf; j < tnodes[tn].lf + tnodes[tn].cnt; j++)
					{
						const uint32_t ii = tprim_idx[j];
						const char* rec = inst + (size_t)ii * 192;
						if (!(rec_u32( rec, 156 ) & rmask)) continue;
						const blas_t* B = blas + rec_u32( rec, 140 );
						const ray_t RB = to_blas( &R, rec );
						/* node_bounds roots the BLAS at 0: with the root at P0 every bound is fmaxf( P0, .. ) of it, exactly (fmaxf neither
						 * rounds nor depends on the order, and the least over paths commutes with it) */
						node_bounds( B->nodes, B->used_nodes, &RB, PB, st );
						for (uint32_t nd = 0; nd < B->used_nodes; nd++)
						{
							if (PB[nd] < 0.0f || !B->nodes[nd].cnt) continue;
							const float P = fmaxf( PT[tn], PB[nd] );
							for (uint32_t r = B->nodes[nd].lf; r < B->nodes[nd].lf + B->nodes[nd].cnt; r++)
							{
								ihit x;
								if (!tri_test( &RB, B->verts, B->prim_idx, r, &x.t, &x.u, &x.v, &x.prim )) continue;
								x.key = fmaxf( x.t, P ), x.inst = ii;
								if (m == cap) cap *= 2, e = (ihit*)realloc( e, sizeof( ihit ) * cap );
								e[m++] = x;
							}
						}
					}
				}
				/* each ( instance, prim ) at its least key */
				qsort( e, m, sizeof( ihit ), icmp_pair );
				uint32_t d = 0;
				for (uint32_t s = 0; s < m; s++) if (s == 0 || e[s].prim != e[s - 1].prim || e[s].inst != e[s - 1].inst) e[d++] = e[s];
				m = d;
				qsort( e, m, sizeof( ihit ), icmp_key );
			}
			write_irow( hits, insts, counts, keys, i, k, R.tmax, e, m < k ? m : k, m < k + 1 ? m : k + 1 );
		}
		free( PT ), free( PB ), free( st ), free( e );
	}
}

/* the pruned walk of one BVH2 from its root, reached with path bound P0 and not tested, into the buffer (*m entries of at most c); each
 * accepted reference is a hit of instance `ii`; st: a stack of used_nodes + 2 entries */
static void walk_sub( ihit* buf, uint32_t* m, const uint32_t c, const node32* nodes, const uint32_t* prim_idx, const float* verts, const ray_t* R,
	const float P0, const uint32_t ii, const int reverse, pend* st )
{
	uint32_t node = 0;
	int sp = 0;
	float P = P0;
	while (1)
	{
		const float b = *m == c ? buf[c - 1].key : INFINITY;
		const node32* nd = nodes + node;
		int next = 0;
		if (!nd->cnt)
		{
			const uint32_t a = nd->lf, bb = nd->lf + 1;
			float ta, tb;
			const int ha = slab( R, nodes + a, &ta ), hb = slab( R, nodes + bb, &tb );
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
				ihit x;
				if (!tri_test( R, verts, prim_idx, r, &x.t, &x.u, &x.v, &x.prim )) continue;
				x.key = fmaxf( x.t, P ), x.inst = ii;
				iinsert( buf, m, c, &x );
			}
		}
		if (next) continue;
		const float b2 = *m == c ? buf[c - 1].key : INFINITY;
		while (sp && st[sp - 1].P > b2) sp--;
		if (!sp) break;
		sp--, node = st[sp].node, P = st[sp].P;
	}
}

void orc_ah_tlas_walk( const node32* tnodes, const uint32_t tlas_used, const uint32_t* tprim_idx, const char* inst, const blas_t* blas, const uint32_t nblas,
	const char* rays, const uint32_t stride, const uint64_t n, const uint32_t k, float* hits, uint32_t* insts, uint32_t* counts, const int reverse )
{
	const uint32_t mu = max_used( tlas_used, blas, nblas );
	#pragma omp parallel
	{
		pend* st = (pend*)malloc( sizeof( pend ) * mu ), * bst = (pend*)malloc( sizeof( pend ) * mu );
		ihit* buf = (ihit*)malloc( sizeof( ihit ) * (k + 1) );
		#pragma omp for schedule( dynamic, 64 )
		for (int64_t i = 0; i < (int64_t)n; i++)
		{
			const ray_t R = load( rays, stride, i );
			const uint32_t rmask = ray_mask( rays, stride, i );
			uint32_t m = 0, node = 0;
			const uint32_t c = k + 1;
			int sp = 0;
			float P = 0.0f;
			while (R.tmax >= 0.0f)
			{
				const float b = m == c ? buf[c - 1].key : INFINITY;
				const node32* nd = tnodes + node;
				int next = 0;
				if (!nd->cnt)
				{
					const uint32_t a = nd->lf, bb = nd->lf + 1;
					float ta, tb;
					const int ha = slab( &R, tnodes + a, &ta ), hb = slab( &R, tnodes + bb, &tb );
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
					/* the leaf's instances in primIdx order, or - reverse - from the last; an instance is pruned as a subtree is */
					for (uint32_t q = 0; q < nd->cnt; q++)
					{
						const uint32_t ii = tprim_idx[nd->lf + (reverse ? nd->cnt - 1 - q : q)];
						const char* rec = inst + (size_t)ii * 192;
						if (!(rec_u32( rec, 156 ) & rmask) || (m == c && P > buf[c - 1].key)) continue;
						const blas_t* B = blas + rec_u32( rec, 140 );
						const ray_t RB = to_blas( &R, rec );
						walk_sub( buf, &m, c, B->nodes, B->prim_idx, B->verts, &RB, P, ii, reverse, bst );
					}
				}
				if (next) continue;
				const float b2 = m == c ? buf[c - 1].key : INFINITY;
				while (sp && st[sp - 1].P > b2) sp--;
				if (!sp) break;
				sp--, node = st[sp].node, P = st[sp].P;
			}
			write_irow( hits, insts, counts, 0, i, k, R.tmax, buf, m < k ? m : k, m );
		}
		free( st ), free( bst ), free( buf );
	}
}
