// harness/signed_distance_b200.cpp - signed distances through the C++ shim: PrepareSignedDistance and SignedDistance over a closed mesh
// (an icosphere of radius 1 built by subdivision, outward by the right-hand rule).  Every record must equal ClosestPoint's but for the
// sign of the distance; points well inside the sphere must come out negative and points well outside positive; a refit without a new
// PrepareSignedDistance must be refused.  Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <array>
#include <map>
#include <vector>

struct V4 { float x, y, z, w; };
struct Rec { float d, u, v; uint32_t prim; };

static std::vector<V4> icosphere( int sub )
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
	for (auto& f : F) for (int k = 0; k < 3; k++) soup.push_back( V4{ (float)V[f[k]][0], (float)V[f[k]][1], (float)V[f[k]][2], 0 } );
	return soup;
}

int main()
{
	std::vector<V4> soup = icosphere( 4 );
	const uint32_t n = (uint32_t)soup.size() / 3, nq = 4000;
	std::vector<V4> q( nq );
	uint32_t seed = 777;
	auto rnd = [&]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
	for (uint32_t i = 0; i < nq; i++) q[i] = V4{ rnd() * 4 - 2, rnd() * 4 - 2, rnd() * 4 - 2, i % 5 == 0 ? 0.3f : INFINITY };
	int fails = 0;
	tinybvh_b200::BVH bvh;
	bvh.Build( soup.data(), n );
	bvh.PrepareSignedDistance();
	std::vector<Rec> cp( nq ), sd( nq );
	bvh.ClosestPoint( q.data(), nq, cp.data() );
	bvh.SignedDistance( q.data(), nq, sd.data() );
	for (uint32_t i = 0; i < nq; i++)
	{
		if (std::fabs( sd[i].d ) != cp[i].d || sd[i].u != cp[i].u || sd[i].v != cp[i].v || sd[i].prim != cp[i].prim)
		{
			if (fails < 5) printf( "query %u: signed record differs from the closest-point record\n", i );
			fails++;
			continue;
		}
		if (cp[i].prim == 0xffffffffu) { if (memcmp( &sd[i], &cp[i], 16 )) fails++; continue; }
		const double r = std::sqrt( (double)q[i].x * q[i].x + (double)q[i].y * q[i].y + (double)q[i].z * q[i].z );
		if (std::fabs( r - 1 ) > 0.01 && (sd[i].d < 0) != (r < 1))
		{
			if (fails < 5) printf( "query %u at radius %.4f: sd %.6g\n", i, r, sd[i].d );
			fails++;
		}
	}
	if (tbvh_refit( bvh.handle(), soup.data(), 16, n, TBVH_HOST ) != TBVH_OK) { printf( "refit failed\n" ); fails++; }
	if (tbvh_signed_distance( bvh.handle(), q.data(), sd.data(), nq, TBVH_HOST, 0 ) != TBVH_E_STATE) { printf( "a stale table was not refused\n" ); fails++; }
	printf( "%d failures\n", fails );
	return fails ? 1 : 0;
}
