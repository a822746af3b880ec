// tests/wn_oracle.c - tbvh_winding_number_prepare / tbvh_winding_number (tinybvh_b200/csrc/winding_number.cu, DESIGN.md 4.11) restated
// on the host over a Wald-layout node array (node 0 the root, node 1 unused): reachability level by level, ownership, the records,
// the fixed atan2, the walk order and the fp64 sum.  Compiled with -ffp-contract=off: every fused pair is an explicit fmaf, every
// other operation rounds on its own, so the results equal the device's bit for bit.
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <stdlib.h>

typedef struct { float mn[3]; uint32_t lf; float mx[3]; uint32_t cnt; } Node32;

#define WN_NONE 0xffffffffu
#define WN_NAN 0x7fffffffu
#define WN_DAG 1u
#define WN_RANGE 2u
static const float WN_PI = 3.14159274f, WN_HALF_PI = 1.57079637f, WN_TWO_PI = 6.28318548f, WN_FOUR_PI = 12.5663710f;

static float u2f( uint32_t u ) { float f; memcpy( &f, &u, 4 ); return f; }
static uint32_t f2u( float f ) { uint32_t u; memcpy( &u, &f, 4 ); return u; }
static float dot3( float ax, float ay, float az, float bx, float by, float bz ) { return fmaf( az, bz, fmaf( ay, by, ax * bx ) ); }
static void cross3( float ax, float ay, float az, float bx, float by, float bz, float* x, float* y, float* z )
{
	*x = ay * bz - az * by, *y = az * bx - ax * bz, *z = ax * by - ay * bx;
}
static float tmin( float a, float b ) { return a < b ? a : b; }
static float tmax( float a, float b ) { return a > b ? a : b; }

float orc_wn_atan2( float y, float x )
{
	if (!(x == x && y == y)) return u2f( WN_NAN );
	const float ax = fabsf( x ), ay = fabsf( y );
	const float mx = ax > ay ? ax : ay, mn = ax > ay ? ay : ax;
	const float t = !(mx > 0.0f) ? 0.0f : mn == mx ? 1.0f : mn / mx;
	const float u = t * t;
	float p = 0.0024567153f;
	p = fmaf( p, u, -0.014401324f );
	p = fmaf( p, u, 0.039781176f );
	p = fmaf( p, u, -0.072348543f );
	p = fmaf( p, u, 0.10498945f );
	p = fmaf( p, u, -0.14161229f );
	p = fmaf( p, u, 0.19985907f );
	p = fmaf( p, u, -0.33332598f );
	p = fmaf( p, u, 0.99999988f );
	float a = p * t;
	a = ay > ax ? WN_HALF_PI - a : a;
	a = x < 0.0f ? WN_PI - a : a;
	return y < 0.0f ? -a : a;
}

void orc_wn_atan2v( const float* y, const float* x, uint64_t n, float* out )
{
	for (uint64_t i = 0; i < n; i++) out[i] = orc_wn_atan2( y[i], x[i] );
}

// 2^-e bringing m >= 0 into [1, 2), e clamped to [-126, 126]; 1 when m is 0 or not finite (closest_walk.cuh cp_pow2)
static float pow2( float m )
{
	const uint32_t f = f2u( m ) >> 23;
	if (!(m > 0.0f) || f == 255u) return 1.0f;
	const uint32_t c = f < 1u ? 1u : f > 253u ? 253u : f;
	return u2f( (254u - c) << 23 );
}

// a, b, c scaled by the power of two of their largest component, as winding_number.cu wn_triangle
static float wn_triangle( float qx, float qy, float qz, const float* v0, const float* v1, const float* v2 )
{
	const float rax = v0[0] - qx, ray = v0[1] - qy, raz = v0[2] - qz;
	const float rbx = v1[0] - qx, rby = v1[1] - qy, rbz = v1[2] - qz;
	const float rcx = v2[0] - qx, rcy = v2[1] - qy, rcz = v2[2] - qz;
	const float s = pow2( fmaxf( fmaxf( fmaxf( fmaxf( fabsf( rax ), fabsf( ray ) ), fmaxf( fabsf( raz ), fabsf( rbx ) ) ),
		fmaxf( fmaxf( fabsf( rby ), fabsf( rbz ) ), fmaxf( fabsf( rcx ), fabsf( rcy ) ) ) ), fabsf( rcz ) ) );
	const float ax = rax * s, ay = ray * s, az = raz * s, bx = rbx * s, by = rby * s, bz = rbz * s, cx = rcx * s, cy = rcy * s, cz = rcz * s;
	float nx, ny, nz;
	cross3( bx, by, bz, cx, cy, cz, &nx, &ny, &nz );
	const float det = dot3( ax, ay, az, nx, ny, nz );
	const float la = sqrtf( dot3( ax, ay, az, ax, ay, az ) ), lb = sqrtf( dot3( bx, by, bz, bx, by, bz ) ), lc = sqrtf( dot3( cx, cy, cz, cx, cy, cz ) );
	float den = (la * lb) * lc;
	den = fmaf( dot3( ax, ay, az, bx, by, bz ), lc, den );
	den = fmaf( dot3( bx, by, bz, cx, cy, cz ), la, den );
	den = fmaf( dot3( cx, cy, cz, ax, ay, az ), lb, den );
	return orc_wn_atan2( det, den ) / WN_TWO_PI;
}

// 2^-h for 2^2h <= dd < 2^(2h+2) (h in [-63, 63]); 1 when dd is not finite
static float wn_scale( float dd )
{
	const uint32_t f = f2u( dd ) >> 23;
	if (f >= 255u) return 1.0f;
	const int h = ((int)(f < 1u ? 1u : f) - 127) >> 1;
	return u2f( (uint32_t)(127 - h) << 23 );
}

// r: 16 floats { p, r, N, M00, M01 .. M22 }; every term scaled by s^3, s = wn_scale( dd ), as winding_number.cu wn_far
static float wn_far( float dx, float dy, float dz, float dd, const float* r )
{
	const float* M = r + 7; // M[0] = M00 .. M[8] = M22
	const float s = wn_scale( dd ), s2 = s * s;
	const float ex = dx * s, ey = dy * s, ez = dz * s, ee = dd * s2;
	const float dN = dot3( ex, ey, ez, r[4] * s2, r[5] * s2, r[6] * s2 );
	const float tr = (((M[0] + M[4]) + M[8]) * s2) * s;
	const float m0 = dot3( M[0], M[1], M[2], ex, ey, ez ), m1 = dot3( M[3], M[4], M[5], ex, ey, ez ), m2 = dot3( M[6], M[7], M[8], ex, ey, ez );
	const float dMd = dot3( ex, ey, ez, (m0 * s2) * s, (m1 * s2) * s, (m2 * s2) * s );
	const float num = (dN + tr) - (3.0f * dMd) / ee;
	return num / ((WN_FOUR_PI * ee) * sqrtf( ee ));
}

typedef struct { const Node32* nodes; uint32_t S, root_ref, root_count, refs, prims; const uint32_t* prim_idx; } Tree;
static void node_of( const Tree* T, uint32_t i, uint32_t* ref, uint32_t* cnt )
{
	if (i == T->S) { *ref = T->root_ref, *cnt = T->root_count; return; }
	*ref = T->nodes[i].lf, *cnt = T->nodes[i].cnt;
}

// the table of a Wald-layout tree of `used` nodes: table (used + 1 records of 16 floats, the root's last), own (idx_count words);
// returns the flag word (WN_DAG / WN_RANGE); max_depth: the tree's depth (the number of reach steps)
uint32_t orc_wn_prepare( const Node32* nodes, uint32_t used, const uint32_t* prim_idx, uint32_t idx_count, const float* verts, uint32_t prims,
	uint32_t max_depth, float* table, uint32_t* own )
{
	const uint32_t S = used < 2 ? 2 : used;
	Tree T = { nodes, S, nodes[0].lf, nodes[0].cnt, idx_count, prims, prim_idx };
	uint32_t* level = malloc( ((size_t)S + 1) * 4 ), * hits = calloc( S, 4 ), * owner = malloc( (size_t)prims * 4 ), flag = 0;
	float* box = malloc( ((size_t)S + 1) * 6 * 4 );
	memset( level, 0xff, ((size_t)S + 1) * 4 );
	level[S] = 0;
	memset( owner, 0xff, (size_t)prims * 4 );
	memset( own, 0xff, (size_t)idx_count * 4 );
	memset( table, 0xff, ((size_t)S + 1) * 64 );
	// reachability: the order of marking within a step does not change which slots end marked, nor the flag
	for (uint32_t k = 1; k <= max_depth; k++)
		for (uint32_t i = 0; i <= S; i++)
		{
			if (level[i] != k - 1) continue;
			uint32_t ref, cnt;
			node_of( &T, i, &ref, &cnt );
			if (cnt) continue;
			if (ref >= S - 1) { flag |= WN_RANGE; continue; }
			for (uint32_t c = ref; c <= ref + 1; c++)
			{
				if (c == 1) continue;
				if (hits[c]++ != 0) flag |= WN_DAG;
				else level[c] = k;
			}
		}
	// ownership
	for (uint32_t i = 0; i <= S; i++)
	{
		if (level[i] == WN_NONE) continue;
		uint32_t ref, cnt;
		node_of( &T, i, &ref, &cnt );
		if (!cnt) continue;
		if ((uint64_t)ref + cnt > idx_count) { flag |= WN_RANGE; continue; }
		for (uint32_t k = ref; k < ref + cnt; k++)
		{
			const uint32_t prim = prim_idx[k];
			if (prim >= prims) flag |= WN_RANGE;
			else if (k < owner[prim]) owner[prim] = k;
		}
	}
	for (uint32_t i = 0; i <= S; i++)
	{
		if (level[i] == WN_NONE) continue;
		uint32_t ref, cnt;
		node_of( &T, i, &ref, &cnt );
		if (!cnt || (uint64_t)ref + cnt > idx_count) continue;
		for (uint32_t k = ref; k < ref + cnt; k++) own[k] = prim_idx[k] < prims && owner[prim_idx[k]] == k ? prim_idx[k] : WN_NONE;
	}
	// records, deepest level first
	for (uint32_t k = max_depth + 1; k-- > 0;)
		for (uint32_t i = 0; i <= S; i++)
		{
			if (level[i] != k) continue;
			uint32_t ref, cnt;
			node_of( &T, i, &ref, &cnt );
			float lo[3] = { INFINITY, INFINITY, INFINITY }, hi[3] = { -INFINITY, -INFINITY, -INFINITY }, p[3], N[3] = { 0, 0, 0 }, M[9];
			int any = 0;
			if (cnt)
			{
				if ((uint64_t)ref + cnt > idx_count) continue;
				for (uint32_t j = ref; j < ref + cnt; j++)
				{
					if (own[j] == WN_NONE) continue;
					any = 1;
					for (int c = 0; c < 3; c++)
					{
						const float* v = verts + ((size_t)own[j] * 3 + c) * 4;
						for (int a = 0; a < 3; a++) lo[a] = tmin( lo[a], v[a] ), hi[a] = tmax( hi[a], v[a] );
					}
				}
				if (!any) continue;
				for (int a = 0; a < 3; a++) p[a] = (lo[a] + hi[a]) * 0.5f;
				for (int j = 0; j < 9; j++) M[j] = 0.0f;
				for (uint32_t j = ref; j < ref + cnt; j++)
				{
					if (own[j] == WN_NONE) continue;
					const float* v0 = verts + (size_t)own[j] * 12, * v1 = v0 + 4, * v2 = v0 + 8;
					float n[3], d[3];
					cross3( v1[0] - v0[0], v1[1] - v0[1], v1[2] - v0[2], v2[0] - v0[0], v2[1] - v0[1], v2[2] - v0[2], n, n + 1, n + 2 );
					for (int a = 0; a < 3; a++) d[a] = ((v0[a] + v1[a]) + v2[a]) / 3.0f - p[a];
					for (int a = 0; a < 3; a++) n[a] = 0.5f * n[a], N[a] = N[a] + n[a];
					for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) M[a * 3 + b] = fmaf( d[a], n[b], M[a * 3 + b] );
				}
			}
			else
			{
				if (ref >= S - 1) continue;
				const uint32_t ch[2] = { ref, ref + 1 };
				int has[2];
				for (int c = 0; c < 2; c++)
				{
					has[c] = f2u( table[(size_t)ch[c] * 16 + 3] ) != WN_NONE;
					if (!has[c]) continue;
					any = 1;
					for (int a = 0; a < 3; a++) lo[a] = tmin( lo[a], box[(size_t)ch[c] * 6 + a] ), hi[a] = tmax( hi[a], box[(size_t)ch[c] * 6 + 3 + a] );
				}
				if (!any) continue;
				for (int a = 0; a < 3; a++) p[a] = (lo[a] + hi[a]) * 0.5f;
				int first = 1;
				for (int c = 0; c < 2; c++)
				{
					if (!has[c]) continue;
					const float* r = table + (size_t)ch[c] * 16;
					const float* cn = r + 4, * cm = r + 7;
					float d[3];
					for (int a = 0; a < 3; a++) d[a] = r[a] - p[a];
					for (int a = 0; a < 3; a++) N[a] = first ? cn[a] : N[a] + cn[a];
					for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) M[a * 3 + b] = fmaf( d[a], cn[b], first ? cm[a * 3 + b] : M[a * 3 + b] + cm[a * 3 + b] );
					first = 0;
				}
			}
			const float ex = hi[0] - lo[0], ey = hi[1] - lo[1], ez = hi[2] - lo[2];
			float r = 0.5f * sqrtf( dot3( ex, ey, ez, ex, ey, ez ) );
			r = r == r ? r : u2f( WN_NAN );
			float* o = table + (size_t)i * 16;
			o[0] = p[0], o[1] = p[1], o[2] = p[2], o[3] = r, o[4] = N[0], o[5] = N[1], o[6] = N[2];
			memcpy( o + 7, M, 36 );
			for (int a = 0; a < 3; a++) box[(size_t)i * 6 + a] = lo[a], box[(size_t)i * 6 + 3 + a] = hi[a];
		}
	free( level ), free( hits ), free( owner ), free( box );
	return flag;
}

// one slot of the walk (winding_number.cu wn_visit): the pair to descend into, or WN_NONE
static uint32_t visit( const Node32* nodes, uint32_t S, const uint32_t* own, const float* verts, const float* table, uint32_t slot,
	float qx, float qy, float qz, float beta, double* w )
{
	const float* rec = table + (size_t)slot * 16;
	if (f2u( rec[3] ) == WN_NONE) return WN_NONE;
	const float dx = rec[0] - qx, dy = rec[1] - qy, dz = rec[2] - qz;
	const float dd = dot3( dx, dy, dz, dx, dy, dz ), br = beta * rec[3];
	if (dd > br * br) { *w = *w + (double)wn_far( dx, dy, dz, dd, rec ); return WN_NONE; }
	const uint32_t ref = slot == S ? nodes[0].lf : nodes[slot].lf, cnt = slot == S ? nodes[0].cnt : nodes[slot].cnt;
	if (!cnt) return ref;
	for (uint32_t k = ref; k < ref + cnt; k++)
	{
		if (own[k] == WN_NONE) continue;
		const float* v0 = verts + (size_t)own[k] * 12;
		*w = *w + (double)wn_triangle( qx, qy, qz, v0, v0 + 4, v0 + 8 );
	}
	return WN_NONE;
}

// queries: n float4 { x, y, z, ignored }; out: n floats
void orc_wn_query( const Node32* nodes, uint32_t used, const uint32_t* own, const float* verts, const float* table, const float* queries,
	uint64_t n, float beta, float* out )
{
	const uint32_t S = used < 2 ? 2 : used;
	#pragma omp parallel for schedule(dynamic, 64)
	for (int64_t i = 0; i < (int64_t)n; i++)
	{
		const float qx = queries[i * 4], qy = queries[i * 4 + 1], qz = queries[i * 4 + 2];
		if (!(qx == qx && qy == qy && qz == qz)) { out[i] = u2f( WN_NAN ); continue; }
		double w = 0.0;
		uint32_t stack[256];
		int sp = 0;
		uint32_t pair = visit( nodes, S, own, verts, table, S, qx, qy, qz, beta, &w );
		for (;;)
		{
			if (pair != WN_NONE)
			{
				const uint32_t a = visit( nodes, S, own, verts, table, pair, qx, qy, qz, beta, &w );
				if (a != WN_NONE) { stack[sp++] = pair + 1; pair = a; continue; }
				pair = visit( nodes, S, own, verts, table, pair + 1, qx, qy, qz, beta, &w );
				continue;
			}
			if (sp == 0) break;
			pair = visit( nodes, S, own, verts, table, stack[--sp], qx, qy, qz, beta, &w );
		}
		const float r = (float)w;
		out[i] = r == r ? r : u2f( WN_NAN );
	}
}
