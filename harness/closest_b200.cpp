// harness/closest_b200.cpp - proximity queries through the C++ shim: ClosestPoint and the batched and single-query IntersectSphere
// over a procedural scene.  Distances must match a double-precision brute force over every triangle; each overlap bit must say whether
// ClosestPoint with r_max = r finds a triangle; the single-query IntersectSphere must give the batch bit; and a BVH8_CWBVH built over
// the same scene (its BVH2 is BuildAVX's tree) must give the records of BVH::BuildAVX byte for byte.  Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

struct V4 { float x, y, z, w; };
struct V3 { float x, y, z; };
struct Rec { float d, u, v; uint32_t prim; };

// distance from p to triangle (a, b, c) in double precision: the plane point when inside, else the nearest edge point
static double tri_dist( const double* p, const V4& A, const V4& B, const V4& C )
{
	const double a[3] = { A.x, A.y, A.z }, b[3] = { B.x, B.y, B.z }, c[3] = { C.x, C.y, C.z };
	auto seg = [&]( const double* s, const double* t )
	{
		double d[3], dd = 0, w = 0;
		for (int k = 0; k < 3; k++) d[k] = t[k] - s[k], dd += d[k] * d[k], w += (p[k] - s[k]) * d[k];
		w = dd > 0 ? std::fmin( std::fmax( w / dd, 0.0 ), 1.0 ) : 0.0;
		double r = 0;
		for (int k = 0; k < 3; k++) { const double e = p[k] - (s[k] + w * d[k]); r += e * e; }
		return std::sqrt( r );
	};
	double best = std::fmin( std::fmin( seg( a, b ), seg( a, c ) ), seg( b, c ) );
	double e1[3], e2[3], n[3];
	for (int k = 0; k < 3; k++) e1[k] = b[k] - a[k], e2[k] = c[k] - a[k];
	n[0] = e1[1] * e2[2] - e1[2] * e2[1], n[1] = e1[2] * e2[0] - e1[0] * e2[2], n[2] = e1[0] * e2[1] - e1[1] * e2[0];
	const double nn = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
	if (nn > 0)
	{
		const double t = ((p[0] - a[0]) * n[0] + (p[1] - a[1]) * n[1] + (p[2] - a[2]) * n[2]) / nn;
		double q[3];
		for (int k = 0; k < 3; k++) q[k] = p[k] - t * n[k];
		bool inside = true;
		const double* v[3] = { a, b, c };
		for (int e = 0; e < 3; e++)
		{
			const double* s = v[e], * f = v[(e + 1) % 3];
			const double x[3] = { f[0] - s[0], f[1] - s[1], f[2] - s[2] }, y[3] = { q[0] - s[0], q[1] - s[1], q[2] - s[2] };
			const double cr[3] = { x[1] * y[2] - x[2] * y[1], x[2] * y[0] - x[0] * y[2], x[0] * y[1] - x[1] * y[0] };
			inside &= cr[0] * n[0] + cr[1] * n[1] + cr[2] * n[2] >= 0;
		}
		if (inside) best = std::fmin( best, std::fabs( t ) * std::sqrt( nn ) );
	}
	return best;
}

int main()
{
	const uint32_t n = 3000, nq = 2000;
	std::vector<V4> soup( n * 3 ), q( nq );
	uint32_t seed = 4242;
	auto rnd = [&]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
	for (uint32_t i = 0; i < n; i++)
	{
		const float cx = rnd() * 100, cy = rnd() * 20, cz = rnd() * 100;
		for (int k = 0; k < 3; k++) soup[i * 3 + k] = V4{ cx + rnd() * 3, cy + rnd() * 3, cz + rnd() * 3, 0 };
	}
	for (uint32_t i = 0; i < nq; i++) q[i] = V4{ rnd() * 120 - 10, rnd() * 40 - 10, rnd() * 120 - 10, i % 4 == 0 ? INFINITY : rnd() * 4 };
	int fails = 0;
	tinybvh_b200::BVH bvh;
	bvh.BuildAVX( soup.data(), n );
	std::vector<Rec> rec( nq ), rec8( nq );
	bvh.ClosestPoint( q.data(), nq, rec.data() );
	std::vector<uint32_t> bits( (nq + 31) / 32 );
	bvh.IntersectSphere( q.data(), nq, bits.data() );
	for (uint32_t i = 0; i < nq; i++)
	{
		const double p[3] = { q[i].x, q[i].y, q[i].z };
		double want = INFINITY;
		for (uint32_t t = 0; t < n; t++) want = std::fmin( want, tri_dist( p, soup[t * 3], soup[t * 3 + 1], soup[t * 3 + 2] ) );
		const bool found = rec[i].prim != 0xffffffffu;
		if (found && std::fabs( rec[i].d - want ) > 1e-4) { if (fails < 5) printf( "query %u: d %.7g, brute force %.7g\n", i, rec[i].d, want ); fails++; }
		if (!found && want < q[i].w - 1e-4) { if (fails < 5) printf( "query %u: missed a triangle at %.7g within %.7g\n", i, want, q[i].w ); fails++; }
		const bool bit = (bits[i >> 5] >> (i & 31)) & 1;
		if (bit != found) { if (fails < 5) printf( "query %u: overlap bit %d, closest point found %d\n", i, bit, found ); fails++; }
		if (i % 97 == 0 && bvh.IntersectSphere( V3{ q[i].x, q[i].y, q[i].z }, q[i].w ) != bit) { printf( "query %u: single-query IntersectSphere differs\n", i ); fails++; }
	}
	tinybvh_b200::BVH8_CWBVH cw;
	cw.Build( soup.data(), n );
	cw.ClosestPoint( q.data(), nq, rec8.data() );
	if (memcmp( rec.data(), rec8.data(), nq * sizeof( Rec ) )) { printf( "BVH8_CWBVH records differ from BVH::BuildAVX's\n" ); fails++; }
	printf( "%d failures\n", fails );
	return fails ? 1 : 0;
}
