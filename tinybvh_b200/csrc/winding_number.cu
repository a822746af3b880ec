// tinybvh_b200/csrc/winding_number.cu - generalized winding numbers (tbvh_winding_number_prepare / tbvh_winding_number): the solid
// angles of the triangles a handle's BVH2 reaches, summed exactly near the query (Van Oosterom & Strackee) and by a second-order
// far-field expansion for subtrees far from it (Barill et al. 2018, "Fast Winding Numbers for Soups and Clouds").  DESIGN.md 4.11 states
// the rules; tests/wn_oracle.c restates them on the host in the same fp32 operation order and the same fp64 additions.
//
// Prepare, on the engine stream, over the S slots of trav() plus the root's record at index S:
//   k_wn_reach      one launch per level: the slots marked at the previous level mark their children; a slot targeted twice is a DAG
//   k_wn_owner      each triangle's owner: the smallest reached reference to it (atomicMin), bad leaf ranges or prims flagged
//   k_wn_own        per reference: its prim when it owns it, else 0xffffffff
//   k_wn_records    one launch per level, deepest first: leaves sum their owned triangles, interior records combine left then right
// One host synchronisation reads the flag word.  Records are 4 float4 { p, r }, { N, M00 }, { M01, M02, M10, M11 }, { M12, M20, M21, M22 }.
#include "common.cuh"
#include "../../include/tinybvh_b200_device/closest_walk.cuh"
#include <algorithm>

#define WN_REC 4 // float4 per record

namespace
{
using tbvh::cp_dot;
using tbvh::cp_cross;

constexpr uint32_t WN_NONE = 0xffffffffu;   // an unreached level, a reference that owns nothing, the bits of r in an empty record
constexpr uint32_t WN_NAN = 0x7fffffffu;    // the one NaN a record's r or a result holds
enum { WN_DAG = 1u, WN_RANGE = 2u };        // flag bits: a slot targeted twice; a child, leaf range or prim out of bounds
constexpr float WN_PI = 3.14159274f, WN_HALF_PI = 1.57079637f, WN_TWO_PI = 6.28318548f, WN_FOUR_PI = 12.5663710f;

// atan2 with one fixed formula on both sides (libm's atan2f and the device's differ): octant reduction to t = min / max in [0, 1],
// atan( t ) = t P( t^2 ) with a degree-8 P by Horner (coefficients fitted on the host, fp64 least squares on [0, 1]), then quadrant
// selects.  y < 0 decides the sign (atan2( -0, x < 0 ) = +pi), x < 0 the half plane (atan2( y, -0 ) = atan2( y, +0 )), 0 / 0 gives 0,
// inf / inf gives pi / 4; NaN gives NaN.
__device__ __forceinline__ float wn_atan2( const float y, const float x )
{
	if (!(x == x && y == y)) return __uint_as_float( WN_NAN );
	const float ax = fabsf( x ), ay = fabsf( y );
	const float mx = ax > ay ? ax : ay, mn = ax > ay ? ay : ax;
	const float t = !(mx > 0.0f) ? 0.0f : mn == mx ? 1.0f : __fdiv_rn( mn, mx );
	const float u = __fmul_rn( t, t );
	float p = 0.0024567153f;
	p = __fmaf_rn( p, u, -0.014401324f );
	p = __fmaf_rn( p, u, 0.039781176f );
	p = __fmaf_rn( p, u, -0.072348543f );
	p = __fmaf_rn( p, u, 0.10498945f );
	p = __fmaf_rn( p, u, -0.14161229f );
	p = __fmaf_rn( p, u, 0.19985907f );
	p = __fmaf_rn( p, u, -0.33332598f );
	p = __fmaf_rn( p, u, 0.99999988f );
	float a = __fmul_rn( p, t );
	a = ay > ax ? __fsub_rn( WN_HALF_PI, a ) : a;
	a = x < 0.0f ? __fsub_rn( WN_PI, a ) : a;
	return y < 0.0f ? -a : a;
}

// the solid angle of triangle (v0, v1, v2) seen from q over 4 pi: atan2( det, den ) / 2 pi (Van Oosterom & Strackee).  det and den are
// of degree 3 in lengths: a, b, c are first scaled by the power of two of their largest component (tbvh::cp_pow2), which leaves the
// angle's bits as they are wherever nothing over- or underflows and keeps det from underflowing near small triangles
__device__ __forceinline__ float wn_triangle( const float qx, const float qy, const float qz, const float4& v0, const float4& v1, const float4& v2 )
{
	const float rax = __fsub_rn( v0.x, qx ), ray = __fsub_rn( v0.y, qy ), raz = __fsub_rn( v0.z, qz );
	const float rbx = __fsub_rn( v1.x, qx ), rby = __fsub_rn( v1.y, qy ), rbz = __fsub_rn( v1.z, qz );
	const float rcx = __fsub_rn( v2.x, qx ), rcy = __fsub_rn( v2.y, qy ), rcz = __fsub_rn( v2.z, qz );
	float inv;
	const float s = tbvh::cp_pow2( fmaxf( fmaxf( fmaxf( fmaxf( fabsf( rax ), fabsf( ray ) ), fmaxf( fabsf( raz ), fabsf( rbx ) ) ),
		fmaxf( fmaxf( fabsf( rby ), fabsf( rbz ) ), fmaxf( fabsf( rcx ), fabsf( rcy ) ) ) ), fabsf( rcz ) ), inv );
	const float ax = __fmul_rn( rax, s ), ay = __fmul_rn( ray, s ), az = __fmul_rn( raz, s );
	const float bx = __fmul_rn( rbx, s ), by = __fmul_rn( rby, s ), bz = __fmul_rn( rbz, s );
	const float cx = __fmul_rn( rcx, s ), cy = __fmul_rn( rcy, s ), cz = __fmul_rn( rcz, s );
	float nx, ny, nz;
	cp_cross( bx, by, bz, cx, cy, cz, nx, ny, nz );
	const float det = cp_dot( ax, ay, az, nx, ny, nz );
	const float la = __fsqrt_rn( cp_dot( ax, ay, az, ax, ay, az ) ), lb = __fsqrt_rn( cp_dot( bx, by, bz, bx, by, bz ) ), lc = __fsqrt_rn( cp_dot( cx, cy, cz, cx, cy, cz ) );
	float den = __fmul_rn( __fmul_rn( la, lb ), lc );
	den = __fmaf_rn( cp_dot( ax, ay, az, bx, by, bz ), lc, den );
	den = __fmaf_rn( cp_dot( bx, by, bz, cx, cy, cz ), la, den );
	den = __fmaf_rn( cp_dot( cx, cy, cz, ax, ay, az ), lb, den );
	return __fdiv_rn( wn_atan2( det, den ), WN_TWO_PI );
}

// 2^-h for 2^2h <= dd < 2^(2h+2) (h in [-63, 63]), so that |d| 2^-h lies in [1, 2); 1 when dd is not finite
__device__ __forceinline__ float wn_scale( const float dd )
{
	const uint32_t f = __float_as_uint( dd ) >> 23;
	if (f >= 255u) return 1.0f;
	const int h = ((int)(f < 1u ? 1u : f) - 127) >> 1;
	return __uint_as_float( (uint32_t)(127 - h) << 23 );
}

// the far-field term of a record, d = p - q: ( d.N + tr M - 3 d^T M d / |d|^2 ) / ( 4 pi |d|^3 ).  Numerator and denominator are of
// degree 3 and d^T M d of degree 5 in lengths, so every term is evaluated scaled by s^3, s = wn_scale( dd ): d by s, N by s^2, tr M and
// M d by s^3 (M d s^4 before the last dot), |d|^2 by s^2.  The quotient is the unscaled one bit for bit wherever the unscaled terms
// neither over- nor underflow, and it stays finite where they would (a mesh more than about 2^25 units across, or less than 2^-26).
__device__ __forceinline__ float wn_far( const float dx, const float dy, const float dz, const float dd, const float4& r1, const float4& r2, const float4& r3 )
{
	const float s = wn_scale( dd ), s2 = __fmul_rn( s, s );
	const float ex = __fmul_rn( dx, s ), ey = __fmul_rn( dy, s ), ez = __fmul_rn( dz, s ), ee = __fmul_rn( dd, s2 );
	const float dN = cp_dot( ex, ey, ez, __fmul_rn( r1.x, s2 ), __fmul_rn( r1.y, s2 ), __fmul_rn( r1.z, s2 ) );
	const float tr = __fmul_rn( __fmul_rn( __fadd_rn( __fadd_rn( r1.w, r2.w ), r3.w ), s2 ), s );
	const float m0 = cp_dot( r1.w, r2.x, r2.y, ex, ey, ez ), m1 = cp_dot( r2.z, r2.w, r3.x, ex, ey, ez ), m2 = cp_dot( r3.y, r3.z, r3.w, ex, ey, ez );
	const float dMd = cp_dot( ex, ey, ez, __fmul_rn( __fmul_rn( m0, s2 ), s ), __fmul_rn( __fmul_rn( m1, s2 ), s ), __fmul_rn( __fmul_rn( m2, s2 ), s ) );
	const float num = __fsub_rn( __fadd_rn( dN, tr ), __fdiv_rn( __fmul_rn( 3.0f, dMd ), ee ) );
	return __fdiv_rn( num, __fmul_rn( __fmul_rn( WN_FOUR_PI, ee ), __fsqrt_rn( ee ) ) );
}

__device__ __forceinline__ float tmin( const float a, const float b ) { return a < b ? a : b; }
__device__ __forceinline__ float tmax( const float a, const float b ) { return a > b ? a : b; }

// the tree the prepare reads: slot i < S from trav(), slot S the root as a child record
struct WnTree
{
	const float4* nodes;
	const float4* tris;
	uint32_t S, root_ref, root_count, wald, refs, prims;
	__device__ __forceinline__ void node( const uint32_t i, uint32_t& ref, uint32_t& cnt ) const
	{
		if (i == S) { ref = root_ref, cnt = root_count; return; }
		ref = __float_as_uint( nodes[(size_t)i * 2].w ), cnt = __float_as_uint( nodes[(size_t)i * 2 + 1].w );
	}
};

// step k: every record marked at level k - 1 that is interior marks its two children at level k; a slot targeted by a second reached
// interior record sets WN_DAG.  Slot 1 of the Wald layout (LAYOUT_BVH's unused node) is never marked.
__global__ void k_wn_reach( const WnTree T, uint32_t* __restrict__ level, uint32_t* __restrict__ hits, uint32_t* __restrict__ flag, const uint32_t step )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > T.S || level[i] != step - 1) return;
	uint32_t ref, cnt;
	T.node( i, ref, cnt );
	if (cnt) return;
	if (ref >= T.S - 1) { atomicOr( flag, (uint32_t)WN_RANGE ); return; }
	for (uint32_t c = ref; c <= ref + 1; c++)
	{
		if (T.wald && c == 1) continue;
		if (atomicAdd( &hits[c], 1u ) != 0) atomicOr( flag, (uint32_t)WN_DAG );
		else level[c] = step;
	}
}

// owner[prim] = the smallest reached reference to prim
__global__ void k_wn_owner( const WnTree T, const uint32_t* __restrict__ level, uint32_t* __restrict__ owner, uint32_t* __restrict__ flag )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > T.S || level[i] == WN_NONE) return;
	uint32_t ref, cnt;
	T.node( i, ref, cnt );
	if (!cnt) return;
	if ((uint64_t)ref + cnt > T.refs) { atomicOr( flag, (uint32_t)WN_RANGE ); return; }
	for (uint32_t k = ref; k < ref + cnt; k++)
	{
		const uint32_t prim = __float_as_uint( T.tris[(size_t)k * 3].w );
		if (prim >= T.prims) atomicOr( flag, (uint32_t)WN_RANGE );
		else atomicMin( &owner[prim], k );
	}
}

__global__ void k_wn_own( const WnTree T, const uint32_t* __restrict__ level, const uint32_t* __restrict__ owner, uint32_t* __restrict__ own )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > T.S || level[i] == WN_NONE) return;
	uint32_t ref, cnt;
	T.node( i, ref, cnt );
	if (!cnt || (uint64_t)ref + cnt > T.refs) return;
	for (uint32_t k = ref; k < ref + cnt; k++)
	{
		const uint32_t prim = __float_as_uint( T.tris[(size_t)k * 3].w );
		own[k] = prim < T.prims && owner[prim] == k ? prim : WN_NONE;
	}
}

// the record of every slot at level `step` (children, one level deeper, are complete): a leaf sums its owned triangles in reference
// order, an interior record combines its non-empty children, left then right; a record that owns nothing stays empty
__global__ void k_wn_records( const WnTree T, const uint32_t* __restrict__ level, const uint32_t step, const uint32_t* __restrict__ own,
	const float4* __restrict__ verts, float4* __restrict__ wn, float4* __restrict__ box )
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > T.S || level[i] != step) return;
	uint32_t ref, cnt;
	T.node( i, ref, cnt );
	float lo[3] = { INFINITY, INFINITY, INFINITY }, hi[3] = { -INFINITY, -INFINITY, -INFINITY }, p[3], N[3] = { 0.0f, 0.0f, 0.0f }, M[9];
	bool any = false;
	if (cnt)
	{
		if ((uint64_t)ref + cnt > T.refs) return;
		for (uint32_t k = ref; k < ref + cnt; k++)
		{
			const uint32_t prim = own[k];
			if (prim == WN_NONE) continue;
			any = true;
			for (int c = 0; c < 3; c++)
			{
				const float4 v = verts[(size_t)prim * 3 + c];
				lo[0] = tmin( lo[0], v.x ), lo[1] = tmin( lo[1], v.y ), lo[2] = tmin( lo[2], v.z );
				hi[0] = tmax( hi[0], v.x ), hi[1] = tmax( hi[1], v.y ), hi[2] = tmax( hi[2], v.z );
			}
		}
		if (!any) return;
		for (int a = 0; a < 3; a++) p[a] = __fmul_rn( __fadd_rn( lo[a], hi[a] ), 0.5f );
		for (int j = 0; j < 9; j++) M[j] = 0.0f;
		for (uint32_t k = ref; k < ref + cnt; k++)
		{
			const uint32_t prim = own[k];
			if (prim == WN_NONE) continue;
			const float4 v0 = verts[(size_t)prim * 3], v1 = verts[(size_t)prim * 3 + 1], v2 = verts[(size_t)prim * 3 + 2];
			float n[3], d[3];
			cp_cross( __fsub_rn( v1.x, v0.x ), __fsub_rn( v1.y, v0.y ), __fsub_rn( v1.z, v0.z ), __fsub_rn( v2.x, v0.x ), __fsub_rn( v2.y, v0.y ), __fsub_rn( v2.z, v0.z ), n[0], n[1], n[2] );
			d[0] = __fsub_rn( __fdiv_rn( __fadd_rn( __fadd_rn( v0.x, v1.x ), v2.x ), 3.0f ), p[0] );
			d[1] = __fsub_rn( __fdiv_rn( __fadd_rn( __fadd_rn( v0.y, v1.y ), v2.y ), 3.0f ), p[1] );
			d[2] = __fsub_rn( __fdiv_rn( __fadd_rn( __fadd_rn( v0.z, v1.z ), v2.z ), 3.0f ), p[2] );
			for (int a = 0; a < 3; a++) n[a] = __fmul_rn( 0.5f, n[a] ), N[a] = __fadd_rn( N[a], n[a] );
			for (int a = 0; a < 3; a++) for (int j = 0; j < 3; j++) M[a * 3 + j] = __fmaf_rn( d[a], n[j], M[a * 3 + j] );
		}
	}
	else
	{
		// the children's boxes first (p is the centre of their union), then N and M shifted to p, left then right
		if (ref >= T.S - 1) return;
		const uint32_t ch[2] = { ref, ref + 1 };
		bool has[2];
		for (int c = 0; c < 2; c++)
		{
			has[c] = __float_as_uint( wn[(size_t)ch[c] * WN_REC].w ) != WN_NONE;
			if (!has[c]) continue;
			any = true;
			const float4 bl = box[(size_t)ch[c] * 2], bh = box[(size_t)ch[c] * 2 + 1];
			lo[0] = tmin( lo[0], bl.x ), lo[1] = tmin( lo[1], bl.y ), lo[2] = tmin( lo[2], bl.z );
			hi[0] = tmax( hi[0], bh.x ), hi[1] = tmax( hi[1], bh.y ), hi[2] = tmax( hi[2], bh.z );
		}
		if (!any) return;
		for (int a = 0; a < 3; a++) p[a] = __fmul_rn( __fadd_rn( lo[a], hi[a] ), 0.5f );
		bool first = true;
		for (int c = 0; c < 2; c++)
		{
			if (!has[c]) continue;
			const float4* r = wn + (size_t)ch[c] * WN_REC;
			const float4 r0 = r[0], r1 = r[1], r2 = r[2], r3 = r[3];
			const float cm[9] = { r1.w, r2.x, r2.y, r2.z, r2.w, r3.x, r3.y, r3.z, r3.w }, cn[3] = { r1.x, r1.y, r1.z };
			const float d[3] = { __fsub_rn( r0.x, p[0] ), __fsub_rn( r0.y, p[1] ), __fsub_rn( r0.z, p[2] ) };
			for (int a = 0; a < 3; a++) N[a] = first ? cn[a] : __fadd_rn( N[a], cn[a] );
			for (int a = 0; a < 3; a++) for (int j = 0; j < 3; j++)
				M[a * 3 + j] = __fmaf_rn( d[a], cn[j], first ? cm[a * 3 + j] : __fadd_rn( M[a * 3 + j], cm[a * 3 + j] ) );
			first = false;
		}
	}
	const float ex = __fsub_rn( hi[0], lo[0] ), ey = __fsub_rn( hi[1], lo[1] ), ez = __fsub_rn( hi[2], lo[2] );
	float r = __fmul_rn( 0.5f, __fsqrt_rn( cp_dot( ex, ey, ez, ex, ey, ez ) ) );
	r = r == r ? r : __uint_as_float( WN_NAN );
	float4* o = wn + (size_t)i * WN_REC;
	o[0] = make_float4( p[0], p[1], p[2], r ), o[1] = make_float4( N[0], N[1], N[2], M[0] );
	o[2] = make_float4( M[1], M[2], M[3], M[4] ), o[3] = make_float4( M[5], M[6], M[7], M[8] );
	box[(size_t)i * 2] = make_float4( lo[0], lo[1], lo[2], 0.0f ), box[(size_t)i * 2 + 1] = make_float4( hi[0], hi[1], hi[2], 0.0f );
}

// one slot of the walk: nothing when empty, its expansion when far, its owned triangles when a leaf; else the pair to descend into
__device__ __forceinline__ uint32_t wn_visit( const float4* __restrict__ nodes, const uint32_t* __restrict__ own, const float4* __restrict__ verts,
	const float4* __restrict__ wn, const uint32_t slot, const uint32_t root_slot, const uint32_t root_ref, const uint32_t root_count,
	const float qx, const float qy, const float qz, const float beta, double& w )
{
	const float4* rec = wn + (size_t)slot * WN_REC;
	const float4 r0 = __ldg( rec );
	if (__float_as_uint( r0.w ) == WN_NONE) return WN_NONE;
	const float dx = __fsub_rn( r0.x, qx ), dy = __fsub_rn( r0.y, qy ), dz = __fsub_rn( r0.z, qz );
	const float dd = cp_dot( dx, dy, dz, dx, dy, dz ), br = __fmul_rn( beta, r0.w );
	if (dd > __fmul_rn( br, br ))
	{
		w = __dadd_rn( w, (double)wn_far( dx, dy, dz, dd, __ldg( rec + 1 ), __ldg( rec + 2 ), __ldg( rec + 3 ) ) );
		return WN_NONE;
	}
	uint32_t ref = root_ref, cnt = root_count;
	if (slot != root_slot) ref = __float_as_uint( __ldg( nodes + (size_t)slot * 2 ).w ), cnt = __float_as_uint( __ldg( nodes + (size_t)slot * 2 + 1 ).w );
	if (!cnt) return ref;
	for (uint32_t k = ref; k < ref + cnt; k++)
	{
		const uint32_t prim = __ldg( own + k );
		if (prim == WN_NONE) continue;
		const float4 v0 = __ldg( verts + (size_t)prim * 3 ), v1 = __ldg( verts + (size_t)prim * 3 + 1 ), v2 = __ldg( verts + (size_t)prim * 3 + 2 );
		w = __dadd_rn( w, (double)wn_triangle( qx, qy, qz, v0, v1, v2 ) );
	}
	return WN_NONE;
}
} // namespace

// One query per thread in 128-thread CTAs; STACKN as k_closest_point.  The root record first, then at every pair the left child
// completely before the right: a left child that needs descending pushes the right one's slot.  Terms are fp32, the sum fp64.
template <int STACKN>
__global__ void __launch_bounds__( 128 ) k_winding_number( const float4* __restrict__ nodes, const uint32_t* __restrict__ own, const float4* __restrict__ verts,
	const float4* __restrict__ wn, const float4* __restrict__ queries, float* __restrict__ results, const uint64_t n, const float beta,
	const uint32_t root_ref, const uint32_t root_count, const uint32_t root_slot )
{
	const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float4 q = __ldg( queries + i );
	if (!(q.x == q.x && q.y == q.y && q.z == q.z)) { results[i] = __uint_as_float( WN_NAN ); return; }
	double w = 0.0;
	uint32_t stack[STACKN];
	int sp = 0;
	#define VISIT( s ) wn_visit( nodes, own, verts, wn, s, root_slot, root_ref, root_count, q.x, q.y, q.z, beta, w )
	uint32_t pair = VISIT( root_slot );
	while (true)
	{
		if (pair != WN_NONE)
		{
			const uint32_t a = VISIT( pair );
			if (a != WN_NONE) { stack[sp++] = pair + 1; pair = a; continue; }
			pair = VISIT( pair + 1 );
			continue;
		}
		if (sp == 0) break;
		pair = VISIT( stack[--sp] );
	}
	#undef VISIT
	const float r = __double2float_rn( w );
	results[i] = r == r ? r : __uint_as_float( WN_NAN );
}

// the slots of trav(): the pair array of a BVH_GPU upload, else the node array up to used_nodes
static uint32_t wn_slots( tbvh_bvh b )
{
	if (b->d_pairs.p) return (uint32_t)(b->d_pairs.bytes / 32);
	return (uint32_t)std::min<size_t>( std::max( b->info.used_nodes, 2u ), b->d_nodes.bytes / 32 );
}

int wn_table_check( tbvh_bvh b )
{
	if (!b->d_wn) { tbvh_set_error( "no winding-number table: call tbvh_winding_number_prepare first" ); return TBVH_E_STATE; }
	if (b->wn_tree_stamp != b->tree_stamp || b->wn_revision != b->revision)
	{
		tbvh_set_error( "the winding-number table is stale: the tree or its vertices changed since tbvh_winding_number_prepare" );
		return TBVH_E_STATE;
	}
	return TBVH_OK;
}

int wn_launch( tbvh_bvh b, const float4* d_queries, float* d_results, uint64_t n, float beta, cudaStream_t s )
{
	const uint32_t grid = (uint32_t)((n + 127) / 128), S = wn_slots( b );
	if (b->info.max_depth + 1 > TBVH_STACK)
		k_winding_number<TBVH_STACK_DEEP><<<grid, 128, 0, s>>>( b->trav(), b->d_wn_own, b->d_verts, b->d_wn, d_queries, d_results, n, beta, b->root_ref, b->root_count, S );
	else k_winding_number<TBVH_STACK><<<grid, 128, 0, s>>>( b->trav(), b->d_wn_own, b->d_verts, b->d_wn, d_queries, d_results, n, beta, b->root_ref, b->root_count, S );
	LAUNCHED();
	return TBVH_OK;
}

// the records and ownership of b's tree into table / own (allocated here), on s; *flag: WN_DAG / WN_RANGE
static int wn_prepare( tbvh_bvh b, DevArray<float4>& table, DevArray<uint32_t>& own, uint32_t* flag, cudaStream_t s )
{
	const uint32_t S = wn_slots( b ), refs = b->info.idx_count, prims = b->info.prim_count, depth = b->info.max_depth;
	const WnTree T = { b->trav(), b->d_leaf_tris, S, b->root_ref, b->root_count, b->d_pairs.p ? 0u : 1u, refs, prims };
	TRY( table.alloc( ((size_t)S + 1) * WN_REC * 16 ) );
	TRY( own.alloc( (size_t)std::max( refs, 1u ) * 4 ) );
	Scratch sc( s );
	uint32_t* level = 0, * hits = 0, * owner = 0, * d_flag = 0, * h_flag = 0;
	float4* box = 0;
	TRY( sc.alloc( level, ((size_t)S + 1) * 4 ) ); TRY( sc.alloc( hits, (size_t)S * 4 ) ); TRY( sc.alloc( owner, (size_t)prims * 4 ) );
	TRY( sc.alloc( box, ((size_t)S + 1) * 32 ) ); TRY( sc.alloc( d_flag, 4 ) ); TRY( sc.alloc_host( h_flag, 4 ) );
	CUDA_TRY( cudaMemsetAsync( level, 0xff, (size_t)S * 4, s ) );
	CUDA_TRY( cudaMemsetAsync( level + S, 0, 4, s ) );
	CUDA_TRY( cudaMemsetAsync( hits, 0, (size_t)S * 4, s ) );
	CUDA_TRY( cudaMemsetAsync( owner, 0xff, (size_t)prims * 4, s ) );
	CUDA_TRY( cudaMemsetAsync( own.get(), 0xff, (size_t)std::max( refs, 1u ) * 4, s ) );
	CUDA_TRY( cudaMemsetAsync( table.get(), 0xff, ((size_t)S + 1) * WN_REC * 16, s ) );
	CUDA_TRY( cudaMemsetAsync( d_flag, 0, 4, s ) );
	const uint32_t g = (S + 1 + 255) / 256;
	for (uint32_t k = 1; k <= depth; k++) { k_wn_reach<<<g, 256, 0, s>>>( T, level, hits, d_flag, k ); LAUNCHED(); }
	k_wn_owner<<<g, 256, 0, s>>>( T, level, owner, d_flag ); LAUNCHED();
	k_wn_own<<<g, 256, 0, s>>>( T, level, owner, own ); LAUNCHED();
	for (uint32_t k = depth + 1; k-- > 0;) { k_wn_records<<<g, 256, 0, s>>>( T, level, k, own, b->d_verts, table, box ); LAUNCHED(); }
	CUDA_TRY( cudaMemcpyAsync( h_flag, d_flag, 4, cudaMemcpyDeviceToHost, s ) );
	CUDA_TRY( cudaStreamSynchronize( s ) );
	*flag = *h_flag;
	return TBVH_OK;
}

extern "C" {

int tbvh_winding_number_prepare( tbvh_bvh b )
{
	if (!b) { tbvh_set_error( "%s: NULL handle", __func__ ); return TBVH_E_ARG; }
	if (b->d_inst) { tbvh_set_error( "winding numbers over a TLAS are not supported" ); return TBVH_E_UNSUPPORTED; }
	if (!b->trav() || !b->d_leaf_tris || !b->d_verts || b->info.prim_count == 0) { tbvh_set_error( "%s: no BVH-layout tree on this handle", __func__ ); return TBVH_E_STATE; }
	if (b->info.max_depth + 1 > TBVH_STACK_DEEP) { tbvh_set_error( "%s: BVH depth %u exceeds the %d-entry walk stack", __func__, b->info.max_depth, TBVH_STACK_DEEP ); return TBVH_E_LIMIT; }
	CUDA_TRY( cudaSetDevice( b->ctx->device ) );
	b->d_wn.reset(), b->d_wn_own.reset();
	DevArray<float4> table;
	DevArray<uint32_t> own;
	uint32_t flag = 0;
	const int rc = wn_prepare( b, table, own, &flag, b->ctx->stream );
	if (rc != TBVH_OK) return rc;
	if (flag & WN_DAG) { tbvh_set_error( "%s: the tree reaches a slot on two paths (a DAG): its triangles would count twice", __func__ ); return TBVH_E_STATE; }
	if (flag) { tbvh_set_error( "%s: a reached node names a child, leaf range or triangle outside the tree's arrays", __func__ ); return TBVH_E_STATE; }
	b->d_wn = std::move( table ), b->d_wn_own = std::move( own );
	b->wn_tree_stamp = b->tree_stamp, b->wn_revision = b->revision;
	return TBVH_OK;
}

int tbvh_winding_number( tbvh_bvh b, const void* queries, float* results, uint64_t n, float beta, int space, void* stream )
{
	return proximity_query( __func__, b, queries, results, n, space, stream, PROX_WINDING, beta );
}

} // extern "C"
