// harness/intersect_all_b200.cpp - multi-hit rays through the C++ shim: IntersectAll over a procedural scene, held to a double-precision
// brute force over every triangle.  For each ray the records must be sorted, hold distinct prims, each crossed by the ray at the record's t
// (within 1e-4 of the scene's scale); the count must be the number of triangles the fp64 test finds, apart from crossings within 1e-5 of a
// triangle's edge or at t within 1e-4 of tmax, which fp32 may decide either way.  Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <vector>

struct V4 { float x, y, z, w; };
struct Ray64 { float O[3]; uint32_t mask; float D[3]; uint32_t inst; float rD[3]; uint32_t pad; float t, u, v; uint32_t prim; };
struct Rec { float t, u, v; uint32_t prim; };

// ray / triangle in double precision: 1 hit at *t, 0 a clear miss, -1 within 1e-5 of an edge (either answer is right in fp32)
static int tri_hit( const Ray64& r, const V4& A, const V4& B, const V4& C, double* t )
{
	const double o[3] = { r.O[0], r.O[1], r.O[2] }, d[3] = { r.D[0], r.D[1], r.D[2] };
	const double e1[3] = { (double)B.x - A.x, (double)B.y - A.y, (double)B.z - A.z }, e2[3] = { (double)C.x - A.x, (double)C.y - A.y, (double)C.z - A.z };
	const double h[3] = { d[1] * e2[2] - d[2] * e2[1], d[2] * e2[0] - d[0] * e2[2], d[0] * e2[1] - d[1] * e2[0] };
	const double a = e1[0] * h[0] + e1[1] * h[1] + e1[2] * h[2];
	if (std::fabs( a ) < 1e-9) return 0;
	const double s[3] = { o[0] - A.x, o[1] - A.y, o[2] - A.z };
	const double u = (s[0] * h[0] + s[1] * h[1] + s[2] * h[2]) / a;
	const double q[3] = { s[1] * e1[2] - s[2] * e1[1], s[2] * e1[0] - s[0] * e1[2], s[0] * e1[1] - s[1] * e1[0] };
	const double v = (d[0] * q[0] + d[1] * q[1] + d[2] * q[2]) / a;
	*t = (e2[0] * q[0] + e2[1] * q[1] + e2[2] * q[2]) / a;
	const double m = std::min( std::min( u, v ), 1 - u - v );
	if (std::fabs( m ) < 1e-5) return -1;
	return m > 0 ? 1 : 0;
}

int main()
{
	const uint32_t n = 3000, nr = 2000, K = 8;
	std::vector<V4> soup( n * 3 );
	uint32_t seed = 777;
	auto rnd = [&]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
	for (uint32_t i = 0; i < n; i++)
	{
		const float cx = rnd() * 100, cy = rnd() * 20, cz = rnd() * 100;
		for (int k = 0; k < 3; k++) soup[i * 3 + k] = V4{ cx + rnd() * 6, cy + rnd() * 6, cz + rnd() * 6, 0 };
	}
	std::vector<Ray64> rays( nr );
	for (uint32_t i = 0; i < nr; i++)
	{
		Ray64& r = rays[i];
		r = Ray64{};
		r.O[0] = rnd() * 100, r.O[1] = rnd() * 20, r.O[2] = i % 2 ? -10.0f : rnd() * 100;
		float d[3] = { rnd() - 0.5f, rnd() - 0.5f, i % 2 ? 1.0f : rnd() - 0.5f };
		const float l = std::sqrt( d[0] * d[0] + d[1] * d[1] + d[2] * d[2] );
		for (int k = 0; k < 3; k++) r.D[k] = d[k] / l, r.rD[k] = 1.0f / r.D[k];
		r.t = i % 3 == 0 ? 1e30f : rnd() * 80;
		r.mask = 0xffff;
	}
	tinybvh_b200::BVH bvh;
	bvh.Build( soup.data(), n );
	std::vector<Rec> rec( (size_t)nr * K );
	std::vector<uint32_t> counts( nr );
	bvh.IntersectAll( rays.data(), nr, K, rec.data(), counts.data() );
	int fails = 0;
	for (uint32_t i = 0; i < nr; i++)
	{
		const Ray64& r = rays[i];
		uint32_t sure = 0, maybe = 0;
		std::vector<double> ts( n, -1 );
		for (uint32_t t = 0; t < n; t++)
		{
			double th;
			const int h = tri_hit( r, soup[t * 3], soup[t * 3 + 1], soup[t * 3 + 2], &th );
			if (h == 0 || th < -1e-4 || th > r.t + 1e-4) continue;
			const bool edge = h < 0 || th < 1e-4 || th > r.t - 1e-4;
			if (edge) maybe++; else sure++;
			ts[t] = th;
		}
		const uint32_t c = counts[i], m = std::min( c, K );
		const bool count_ok = c == K + 1 ? sure + maybe >= K + 1 : (c >= sure && c <= sure + maybe);
		if (!count_ok) { if (fails < 5) printf( "ray %u: count %u, brute force %u sure + %u on an edge\n", i, c, sure, maybe ); fails++; }
		for (uint32_t s = 0; s < K; s++)
		{
			const Rec& x = rec[(size_t)i * K + s];
			if (s >= m) { if (x.prim != 0xffffffffu || x.t != r.t) { if (fails < 5) printf( "ray %u slot %u: not empty\n", i, s ); fails++; } continue; }
			if (x.prim >= n || ts[x.prim] < 0 || std::fabs( ts[x.prim] - x.t ) > 1e-4 * 100) { if (fails < 5) printf( "ray %u slot %u: prim %u at %g not crossed there\n", i, s, x.prim, x.t ); fails++; }
			if (s > 0 && (rec[(size_t)i * K + s - 1].t > x.t || rec[(size_t)i * K + s - 1].prim == x.prim)) { if (fails < 5) printf( "ray %u slot %u: out of order\n", i, s ); fails++; }
		}
	}
	printf( "%d failures\n", fails );
	return fails ? 1 : 0;
}
