// harness/intersect_all_tlas_b200.cpp - multi-hit rays through a TLAS with the C++ shim: IntersectAll over 200 instances of three BLASses
// (rotated, scaled and translated), held to a double-precision brute force over every instance's triangles in its BLAS's space.  For each
// ray the records must be sorted, hold distinct ( instance, prim ) pairs, each crossed by the ray at the record's t (within 1e-4 of the
// scene's scale); the count must be the number of pairs the fp64 test finds, apart from crossings within 1e-5 of a triangle's edge or at t
// within 1e-4 of tmax or 0, which fp32 may decide either way.  Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

struct V4 { float x, y, z, w; };
struct Ray64 { float O[3]; uint32_t mask; float D[3]; uint32_t inst; float rD[3]; uint32_t pad; float t, u, v; uint32_t prim; };
struct Rec { float t, u, v; uint32_t prim; };
struct Inst { float transform[16], invTransform[16], aabbMin[3]; uint32_t blasIdx; float aabbMax[3]; uint32_t mask, dummy[8]; }; // tinybvh::BLASInstance

// ray / triangle in double precision: 1 hit at *t, 0 a clear miss, -1 within 1e-5 of an edge (either answer is right in fp32)
static int tri_hit( const double o[3], const double d[3], const V4& A, const V4& B, const V4& C, double* t )
{
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
	const uint32_t M = 3, N = 200, nr = 1000, K = 8;
	uint32_t seed = 4242;
	auto rnd = [&]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
	std::vector<std::vector<V4>> soup( M );
	std::vector<tinybvh_b200::BVH*> blas( M );
	std::vector<tinybvh_b200::BVHBase*> base( M );
	for (uint32_t m = 0; m < M; m++)
	{
		const uint32_t n = 200 + 150 * m;
		for (uint32_t i = 0; i < n; i++)
		{
			const float cx = rnd() * 4 - 2, cy = rnd() * 4 - 2, cz = rnd() * 4 - 2;
			for (int k = 0; k < 3; k++) soup[m].push_back( V4{ cx + rnd() * 0.8f, cy + rnd() * 0.8f, cz + rnd() * 0.8f, 0 } );
		}
		blas[m] = new tinybvh_b200::BVH();
		blas[m]->Build( soup[m].data(), n );
		base[m] = blas[m];
	}
	std::vector<Inst> inst( N );
	memset( inst.data(), 0, sizeof( Inst ) * N );
	for (uint32_t i = 0; i < N; i++)
	{
		Inst& in = inst[i];
		const float a = rnd() * 6.28f, s = 0.5f + rnd();
		const float R[9] = { cosf( a ) * s, -sinf( a ) * s, 0, sinf( a ) * s, cosf( a ) * s, 0, 0, 0, s * (i % 2 ? -1.0f : 1.0f) }; // every other one mirrored
		for (int r = 0; r < 3; r++)
		{
			for (int c = 0; c < 3; c++) in.transform[r * 4 + c] = R[r * 3 + c];
			in.transform[r * 4 + 3] = (rnd() - 0.5f) * 30;
		}
		in.transform[15] = 1, in.blasIdx = i % M, in.mask = 0xffff;
	}
	tinybvh_b200::BVH tlas;
	tlas.Build( inst.data(), N, base.data(), M );
	std::vector<Ray64> rays( nr );
	for (uint32_t i = 0; i < nr; i++)
	{
		Ray64& r = rays[i];
		r = Ray64{};
		r.O[0] = (rnd() - 0.5f) * 36, r.O[1] = (rnd() - 0.5f) * 36, r.O[2] = i % 2 ? -30.0f : (rnd() - 0.5f) * 36;
		float d[3] = { rnd() - 0.5f, rnd() - 0.5f, i % 2 ? 1.0f : rnd() - 0.5f };
		const float l = std::sqrt( d[0] * d[0] + d[1] * d[1] + d[2] * d[2] );
		for (int k = 0; k < 3; k++) r.D[k] = d[k] / l, r.rD[k] = 1.0f / r.D[k];
		r.t = i % 3 == 0 ? 1e30f : rnd() * 60;
		r.mask = 0xffff;
	}
	std::vector<Rec> rec( (size_t)nr * K );
	std::vector<uint32_t> insts( (size_t)nr * K ), counts( nr );
	tlas.IntersectAll( rays.data(), nr, K, rec.data(), insts.data(), counts.data() );
	int fails = 0;
	std::vector<double> ts;
	for (uint32_t i = 0; i < nr; i++)
	{
		const Ray64& r = rays[i];
		uint32_t sure = 0, maybe = 0;
		std::vector<std::vector<double>> hit( N );
		for (uint32_t j = 0; j < N; j++)
		{
			const float* T = inst[j].invTransform; // the ray in BLAS space, in fp64; t is shared with world space
			double o[3], d[3];
			for (int k = 0; k < 3; k++)
			{
				o[k] = (double)T[k * 4] * r.O[0] + (double)T[k * 4 + 1] * r.O[1] + (double)T[k * 4 + 2] * r.O[2] + T[k * 4 + 3];
				d[k] = (double)T[k * 4] * r.D[0] + (double)T[k * 4 + 1] * r.D[1] + (double)T[k * 4 + 2] * r.D[2];
			}
			const std::vector<V4>& s = soup[inst[j].blasIdx];
			hit[j].assign( s.size() / 3, -1 );
			for (uint32_t t = 0; t < s.size() / 3; t++)
			{
				double th;
				const int h = tri_hit( o, d, s[t * 3], s[t * 3 + 1], s[t * 3 + 2], &th );
				if (h == 0 || th < -1e-4 || th > r.t + 1e-4) continue;
				const bool edge = h < 0 || th < 1e-4 || th > r.t - 1e-4;
				if (edge) maybe++; else sure++;
				hit[j][t] = th;
			}
		}
		const uint32_t c = counts[i], m = std::min( c, K );
		const bool count_ok = c == K + 1 ? sure + maybe >= K + 1 : (c >= sure && c <= sure + maybe);
		if (!count_ok) { if (fails < 5) printf( "ray %u: count %u, brute force %u sure + %u on an edge\n", i, c, sure, maybe ); fails++; }
		for (uint32_t s = 0; s < K; s++)
		{
			const Rec& x = rec[(size_t)i * K + s];
			const uint32_t in = insts[(size_t)i * K + s];
			if (s >= m) { if (x.prim != 0xffffffffu || in != 0xffffffffu || x.t != r.t) { if (fails < 5) printf( "ray %u slot %u: not empty\n", i, s ); fails++; } continue; }
			if (in >= N || x.prim >= hit[in].size() || hit[in][x.prim] < 0 || std::fabs( hit[in][x.prim] - x.t ) > 1e-4 * 60)
			{ if (fails < 5) printf( "ray %u slot %u: instance %u prim %u at %g not crossed there\n", i, s, in, x.prim, x.t ); fails++; }
			if (s > 0)
			{
				const Rec& p = rec[(size_t)i * K + s - 1];
				if (p.t > x.t || (p.prim == x.prim && insts[(size_t)i * K + s - 1] == in)) { if (fails < 5) printf( "ray %u slot %u: out of order\n", i, s ); fails++; }
			}
		}
	}
	printf( "%d failures\n", fails );
	for (uint32_t m = 0; m < M; m++) delete blas[m];
	return fails ? 1 : 0;
}
