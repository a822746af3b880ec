// harness/mesh_overlap_b200.cpp - intersecting triangle pairs through the C++ shim: OverlapPairs, SelfIntersections and OverlapBits over
// seeded soups of triangles with integer corners, against a brute force over every pair by separating axes in double precision (exact on
// such corners).  In the self query, the pairs between two soups whose corners never coincide (one is offset by half a unit) must be the
// pairs of the two-mesh query.  Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <cstdio>
#include <array>
#include <set>
#include <vector>

struct V4 { float x, y, z, w; };
typedef std::array<double, 3> D3;

static D3 sub( const D3& a, const D3& b ) { return { a[0] - b[0], a[1] - b[1], a[2] - b[2] }; }
static D3 cross( const D3& a, const D3& b ) { return { a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0] }; }
static double dot( const D3& a, const D3& b ) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
static D3 corner( const std::vector<V4>& v, size_t k ) { return { v[k].x, v[k].y, v[k].z }; }

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

static bool degenerate( const D3* T ) { const D3 n = cross( sub( T[1], T[0] ), sub( T[2], T[0] ) ); return n[0] == 0 && n[1] == 0 && n[2] == 0; }

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
	const std::vector<V4> A = soup( na, 11, 0.0f ), B = soup( nb, 23, 0.5f );
	tinybvh_b200::BVH a, b;
	a.Build( A.data(), na );
	b.BuildHQ( B.data(), nb );
	std::vector<std::array<uint32_t, 2>> got;
	a.OverlapPairs( b, got );
	std::vector<std::array<uint32_t, 2>> want;
	std::vector<uint32_t> member( na, 0 );
	for (uint32_t i = 0; i < na; i++)
	{
		const D3 T[3] = { corner( A, 3 * i ), corner( A, 3 * i + 1 ), corner( A, 3 * i + 2 ) };
		if (degenerate( T )) continue;
		for (uint32_t j = 0; j < nb; j++)
		{
			const D3 U[3] = { corner( B, 3 * j ), corner( B, 3 * j + 1 ), corner( B, 3 * j + 2 ) };
			if (!degenerate( U ) && sat( T, U )) want.push_back( { i, j } ), member[i] = 1;
		}
	}
	if (got != want) { printf( "OverlapPairs: %zu pairs, the brute force %zu\n", got.size(), want.size() ); fails++; }
	std::vector<uint32_t> bits( (na + 31) / 32 );
	a.OverlapBits( b, bits.data() );
	for (uint32_t i = 0; i < na; i++) if (((bits[i >> 5] >> (i & 31)) & 1) != member[i]) { if (fails < 20) printf( "OverlapBits: triangle %u\n", i ); fails++; }
	// one mesh of both soups: its pairs (i < na, j >= na) are the pairs above, offset
	std::vector<V4> both = A;
	both.insert( both.end(), B.begin(), B.end() );
	tinybvh_b200::BVH m;
	m.Build( both.data(), na + nb );
	std::vector<std::array<uint32_t, 2>> self;
	m.SelfIntersections( self );
	std::vector<std::array<uint32_t, 2>> cross_pairs;
	for (const auto& p : self)
	{
		if (p[0] >= p[1]) { printf( "SelfIntersections: pair (%u, %u) not i < j\n", p[0], p[1] ); fails++; }
		if (p[0] < na && p[1] >= na) cross_pairs.push_back( { p[0], p[1] - na } );
	}
	if (cross_pairs != want) { printf( "SelfIntersections: %zu pairs across the soups, expected %zu\n", cross_pairs.size(), want.size() ); fails++; }
	printf( "%zu pairs, %zu self pairs\n", want.size(), self.size() );
	printf( "%d failures\n", fails );
	return fails ? 1 : 0;
}
