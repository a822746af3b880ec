// harness/mesh_distance_b200.cpp - distances between meshes through the C++ shim: NearestTriangles and DistancePairs over seeded soups of
// triangles with integer corners (B offset by a quarter unit, so no corner of A meets one of B), against a double-precision brute force
// over every pair: the least of the six vertex-triangle and nine clamped segment-segment distances, 0 where a separating-axis test finds
// no separation.  The nearest distances must agree within 1e-5 of the magnitude (and name a triangle at that distance), and the pairs
// within r must be the brute force's apart from pairs within 1e-5 of r.  Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <cmath>
#include <cstdio>
#include <algorithm>
#include <array>
#include <set>
#include <vector>

struct V4 { float x, y, z, w; };
struct Rec { float d; uint32_t j; };
typedef std::array<double, 3> D3;

static D3 sub( const D3& a, const D3& b ) { return { a[0] - b[0], a[1] - b[1], a[2] - b[2] }; }
static D3 add( const D3& a, const D3& b ) { return { a[0] + b[0], a[1] + b[1], a[2] + b[2] }; }
static D3 mul( const D3& a, double s ) { return { a[0] * s, a[1] * s, a[2] * s }; }
static D3 cross( const D3& a, const D3& b ) { return { a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0] }; }
static double dot( const D3& a, const D3& b ) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static D3 corner( const std::vector<V4>& v, size_t k ) { return { v[k].x, v[k].y, v[k].z }; }
static double clamp01( double x ) { return x < 0 ? 0 : x > 1 ? 1 : x; }

// closed non-degenerate triangles meet: no separating axis among the normals, the edge-edge cross products and the in-plane edge normals
static bool sat( const D3* T, const D3* U )
{
	D3 eT[3], eU[3];
	for (int k = 0; k < 3; k++) eT[k] = sub( T[(k + 1) % 3], T[k] ), eU[k] = sub( U[(k + 1) % 3], U[k] );
	const D3 nT = cross( eT[0], eT[1] ), nU = cross( eU[0], eU[1] );
	std::vector<D3> axes = { nT, nU };
	for (int a = 0; a < 3; a++)
	{
		for (int b = 0; b < 3; b++) axes.push_back( cross( eT[a], eU[b] ) );
		axes.push_back( cross( nT, eT[a] ) ), axes.push_back( cross( nU, eU[a] ) );
	}
	for (const D3& ax : axes)
	{
		if (ax[0] == 0 && ax[1] == 0 && ax[2] == 0) continue;
		double a0 = 1e300, a1 = -1e300, b0 = 1e300, b1 = -1e300;
		for (int k = 0; k < 3; k++)
		{
			const double p = dot( T[k], ax ), q = dot( U[k], ax );
			a0 = std::min( a0, p ), a1 = std::max( a1, p ), b0 = std::min( b0, q ), b1 = std::max( b1, q );
		}
		if (a1 < b0 || b1 < a0) return false;
	}
	return true;
}

// distance from p to the triangle (a, b, c): the plane point when inside, else the nearest of the three segments
static double seg_point( const D3& p, const D3& a, const D3& b )
{
	const D3 d = sub( b, a );
	const double dd = dot( d, d ), t = dd > 0 ? clamp01( dot( sub( p, a ), d ) / dd ) : 0;
	const D3 w = sub( p, add( a, mul( d, t ) ) );
	return std::sqrt( dot( w, w ) );
}
static double point_tri( const D3& p, const D3* T )
{
	double best = std::min( std::min( seg_point( p, T[0], T[1] ), seg_point( p, T[1], T[2] ) ), seg_point( p, T[2], T[0] ) );
	const D3 n = cross( sub( T[1], T[0] ), sub( T[2], T[0] ) );
	const double nn = dot( n, n );
	if (nn > 0)
	{
		const double t = dot( sub( p, T[0] ), n ) / nn;
		const D3 q = sub( p, mul( n, t ) );
		bool inside = true;
		for (int k = 0; k < 3; k++) inside &= dot( cross( sub( T[(k + 1) % 3], T[k] ), sub( q, T[k] ) ), n ) >= 0;
		if (inside) best = std::min( best, std::fabs( t ) * std::sqrt( nn ) );
	}
	return best;
}
// Ericson's ClosestPtSegmentSegment (RTCD 5.1.9)
static double seg_seg( const D3& p1, const D3& q1, const D3& p2, const D3& q2 )
{
	const D3 d1 = sub( q1, p1 ), d2 = sub( q2, p2 ), r = sub( p1, p2 );
	const double a = dot( d1, d1 ), e = dot( d2, d2 ), f = dot( d2, r );
	double s = 0, t = 0;
	if (a <= 0 && e <= 0) s = t = 0;
	else if (a <= 0) s = 0, t = clamp01( f / e );
	else
	{
		const double c = dot( d1, r );
		if (e <= 0) t = 0, s = clamp01( -c / a );
		else
		{
			const double b = dot( d1, d2 ), den = a * e - b * b;
			s = den != 0 ? clamp01( (b * f - c * e) / den ) : 0;
			t = (b * s + f) / e;
			if (t < 0) t = 0, s = clamp01( -c / a );
			else if (t > 1) t = 1, s = clamp01( (b - c) / a );
		}
	}
	const D3 w = sub( add( p1, mul( d1, s ) ), add( p2, mul( d2, t ) ) );
	return std::sqrt( dot( w, w ) );
}
static bool degenerate( const D3* T ) { const D3 n = cross( sub( T[1], T[0] ), sub( T[2], T[0] ) ); return n[0] == 0 && n[1] == 0 && n[2] == 0; }
static double tri_tri( const D3* T, const D3* U )
{
	if (!degenerate( T ) && !degenerate( U ) && sat( T, U )) return 0;
	double best = 1e300;
	for (int k = 0; k < 3; k++) best = std::min( best, std::min( point_tri( U[k], T ), point_tri( T[k], U ) ) );
	for (int k = 0; k < 3; k++) for (int l = 0; l < 3; l++) best = std::min( best, seg_seg( T[k], T[(k + 1) % 3], U[l], U[(l + 1) % 3] ) );
	return best;
}

static std::vector<V4> soup( uint32_t n, uint32_t seed, float offset )
{
	std::vector<V4> v;
	for (uint32_t i = 0; i < n; i++)
	{
		seed = seed * 1664525u + 1013904223u;
		const float c[3] = { (float)((seed >> 8) % 13) - 6, (float)((seed >> 12) % 13) - 6, (float)((seed >> 16) % 13) - 6 };
		for (int k = 0; k < 3; k++)
		{
			V4 p;
			float* q = &p.x;
			for (int a = 0; a < 3; a++) { seed = seed * 1664525u + 1013904223u; q[a] = c[a] + (float)((seed >> 10) % 5) - 2 + offset; }
			p.w = 0;
			v.push_back( p );
		}
	}
	return v;
}

int main()
{
	int fails = 0;
	const uint32_t na = 600, nb = 500;
	const float r = 0.3f;
	const std::vector<V4> A = soup( na, 11, 0.0f ), B = soup( nb, 23, 0.25f );
	tinybvh_b200::BVH a, b;
	a.Build( A.data(), na );
	b.BuildHQ( B.data(), nb );
	std::vector<Rec> rec( na );
	a.NearestTriangles( b, INFINITY, rec.data() );
	std::vector<std::array<uint32_t, 2>> got;
	a.DistancePairs( b, r, got );
	const std::set<std::array<uint32_t, 2>> have( got.begin(), got.end() );
	size_t want_pairs = 0;
	for (uint32_t i = 0; i < na; i++)
	{
		const D3 T[3] = { corner( A, 3 * i ), corner( A, 3 * i + 1 ), corner( A, 3 * i + 2 ) };
		double best = 1e300, at_rec = 1e300;
		for (uint32_t j = 0; j < nb; j++)
		{
			const D3 U[3] = { corner( B, 3 * j ), corner( B, 3 * j + 1 ), corner( B, 3 * j + 2 ) };
			const double d = tri_tri( T, U );
			best = std::min( best, d );
			if (j == rec[i].j) at_rec = d;
			const bool in = have.count( { i, j } ) != 0;
			if (d <= r) want_pairs++;
			if (in != (d <= r) && std::fabs( d - r ) > 1e-5 * 16) { if (fails < 20) printf( "DistancePairs: (%u, %u) at %g, r %g\n", i, j, d, (double)r ); fails++; }
		}
		if (rec[i].j >= nb || std::fabs( rec[i].d - best ) > 1e-5 * 16 || std::fabs( at_rec - best ) > 1e-5 * 16)
		{
			if (fails < 20) printf( "NearestTriangles: triangle %u: %g (triangle %u), the brute force %g\n", i, (double)rec[i].d, rec[i].j, best );
			fails++;
		}
	}
	for (size_t k = 1; k < got.size(); k++) if (!(got[k - 1] < got[k])) { printf( "DistancePairs: not sorted at %zu\n", k ); fails++; break; }
	// one mesh of both soups: its pairs across the soups (i < na, j >= na) are the two-mesh pairs, offset
	std::vector<V4> both = A;
	both.insert( both.end(), B.begin(), B.end() );
	tinybvh_b200::BVH m;
	m.Build( both.data(), na + nb );
	std::vector<std::array<uint32_t, 2>> self, cross_pairs;
	m.DistancePairs( m, r, self );
	for (const auto& p : self)
	{
		if (p[0] >= p[1]) { printf( "DistancePairs self: pair (%u, %u) not i < j\n", p[0], p[1] ); fails++; }
		if (p[0] < na && p[1] >= na) cross_pairs.push_back( { p[0], p[1] - na } );
	}
	if (cross_pairs != got) { printf( "DistancePairs self: %zu pairs across the soups, expected %zu\n", cross_pairs.size(), got.size() ); fails++; }
	printf( "%zu pairs within %g (brute force %zu), %zu self pairs\n", got.size(), (double)r, want_pairs, self.size() );
	printf( "%d failures\n", fails );
	return fails ? 1 : 0;
}
