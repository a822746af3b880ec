// harness/winding_number_b200.cpp - generalized winding numbers through the C++ shim: PrepareWindingNumber and WindingNumber over an
// icosphere of radius 1 (outward by the right-hand rule): 1 inside and 0 outside; about 0.5 at the centre of its open upper half; 2 inside
// the overlap of two spheres; a refit without a new PrepareWindingNumber must be refused.  Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <cmath>
#include <cstdio>
#include <array>
#include <map>
#include <vector>

struct V4 { float x, y, z, w; };

static std::vector<V4> icosphere( int sub, float cx )
{
	const double t = (1 + std::sqrt( 5.0 )) / 2;
	std::vector<std::array<double, 3>> V = { { -1, t, 0 }, { 1, t, 0 }, { -1, -t, 0 }, { 1, -t, 0 }, { 0, -1, t }, { 0, 1, t }, { 0, -1, -t }, { 0, 1, -t },
		{ t, 0, -1 }, { t, 0, 1 }, { -t, 0, -1 }, { -t, 0, 1 } };
	std::vector<std::array<int, 3>> F = { { 0, 11, 5 }, { 0, 5, 1 }, { 0, 1, 7 }, { 0, 7, 10 }, { 0, 10, 11 }, { 1, 5, 9 }, { 5, 11, 4 }, { 11, 10, 2 },
		{ 10, 7, 6 }, { 7, 1, 8 }, { 3, 9, 4 }, { 3, 4, 2 }, { 3, 2, 6 }, { 3, 6, 8 }, { 3, 8, 9 }, { 4, 9, 5 }, { 2, 4, 11 }, { 6, 2, 10 }, { 8, 6, 7 }, { 9, 8, 1 } };
	auto norm = []( std::array<double, 3> p ) { const double l = std::sqrt( p[0] * p[0] + p[1] * p[1] + p[2] * p[2] ); return std::array<double, 3>{ p[0] / l, p[1] / l, p[2] / l }; };
	for (auto& v : V) v = norm( v );
	for (int s = 0; s < sub; s++)
	{
		std::map<std::pair<int, int>, int> mid;
		auto m = [&]( int a, int b )
		{
			const std::pair<int, int> k( std::min( a, b ), std::max( a, b ) );
			auto it = mid.find( k );
			if (it != mid.end()) return it->second;
			V.push_back( norm( { V[a][0] + V[b][0], V[a][1] + V[b][1], V[a][2] + V[b][2] } ) );
			return mid[k] = (int)V.size() - 1;
		};
		std::vector<std::array<int, 3>> G;
		for (auto& f : F)
		{
			const int ab = m( f[0], f[1] ), bc = m( f[1], f[2] ), ca = m( f[2], f[0] );
			G.push_back( { f[0], ab, ca } ), G.push_back( { f[1], bc, ab } ), G.push_back( { f[2], ca, bc } ), G.push_back( { ab, bc, ca } );
		}
		F = G;
	}
	std::vector<V4> soup;
	for (auto& f : F) for (int k = 0; k < 3; k++) soup.push_back( V4{ (float)V[f[k]][0] + cx, (float)V[f[k]][1], (float)V[f[k]][2], 0 } );
	return soup;
}

static int check( const char* what, const float got, const float want, const float tol )
{
	if (std::fabs( got - want ) <= tol) return 0;
	printf( "%s: w = %.6g, expected %.6g +- %.3g\n", what, got, want, tol );
	return 1;
}

int main()
{
	int fails = 0;
	std::vector<V4> sphere = icosphere( 4, 0.0f );
	const uint32_t n = (uint32_t)sphere.size() / 3, nq = 4000;
	std::vector<V4> q( nq );
	uint32_t seed = 777;
	auto rnd = [&]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
	for (uint32_t i = 0; i < nq; i++) q[i] = V4{ rnd() * 4 - 2, rnd() * 4 - 2, rnd() * 4 - 2, 0 };
	tinybvh_b200::BVH bvh;
	bvh.Build( sphere.data(), n );
	bvh.PrepareWindingNumber();
	std::vector<float> w( nq );
	for (const float beta : { 2.0f, INFINITY })
	{
		bvh.WindingNumber( q.data(), nq, w.data(), beta );
		for (uint32_t i = 0; i < nq; i++)
		{
			const double r = std::sqrt( (double)q[i].x * q[i].x + (double)q[i].y * q[i].y + (double)q[i].z * q[i].z );
			// beta = 2 is within 0.073 of the exact value away from the surface (DESIGN.md 4.11)
			if (std::fabs( r - 1 ) > 0.1 && fails < 20) fails += check( r < 1 ? "inside the sphere" : "outside the sphere", w[i], r < 1 ? 1.0f : 0.0f, beta == 2.0f ? 0.11f : 1e-3f );
		}
	}
	// the open upper half: the triangles whose centroid lies above z = 0
	std::vector<V4> half;
	for (uint32_t t = 0; t < n; t++) if (sphere[3 * t].z + sphere[3 * t + 1].z + sphere[3 * t + 2].z > 0) for (int k = 0; k < 3; k++) half.push_back( sphere[3 * t + k] );
	tinybvh_b200::BVH hemi;
	hemi.Build( half.data(), (uint32_t)half.size() / 3 );
	hemi.PrepareWindingNumber();
	const V4 centre = { 0, 0, 0, 0 };
	float wc = 0;
	hemi.WindingNumber( &centre, 1, &wc, INFINITY );
	fails += check( "centre of the open hemisphere", wc, 0.5f, 0.05f );
	// two overlapping spheres: 2 in the lens both enclose
	std::vector<V4> two = sphere, other = icosphere( 4, 0.8f );
	two.insert( two.end(), other.begin(), other.end() );
	tinybvh_b200::BVH both;
	both.Build( two.data(), (uint32_t)two.size() / 3 );
	both.PrepareWindingNumber();
	const V4 lens[2] = { { 0.4f, 0, 0, 0 }, { 0.4f, 0.3f, -0.2f, 0 } };
	float wl[2];
	both.WindingNumber( lens, 2, wl, INFINITY );
	fails += check( "overlap of two spheres", wl[0], 2.0f, 0.05f ) + check( "overlap of two spheres", wl[1], 2.0f, 0.05f );
	if (tbvh_refit( bvh.handle(), sphere.data(), 16, n, TBVH_HOST ) != TBVH_OK) { printf( "refit failed\n" ); fails++; }
	if (tbvh_winding_number( bvh.handle(), q.data(), w.data(), nq, 2.0f, TBVH_HOST, 0 ) != TBVH_E_STATE) { printf( "a stale table was not refused\n" ); fails++; }
	printf( "%d failures\n", fails );
	return fails ? 1 : 0;
}
