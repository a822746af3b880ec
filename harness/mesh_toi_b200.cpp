// harness/mesh_toi_b200.cpp - times of impact between moving meshes through the C++ shim: TimeOfImpact and ImpactPairs on seeded small
// triangles falling onto a plate (two triangles at z = 0), against the double-precision first time of contact (h - eta) / v of each
// triangle whose lowest corner starts h above the plate and falls v within the step.  A resolved record must lie in
// [ (h - eta - xi) / v, (h - eta) / v ] within 1e-5, an unresolved one before (h - eta) / v; no contact only where (h - eta) / v > 1 - 1e-5;
// every pair ImpactPairs reports must come no earlier than its triangle's record, the pair the record names at exactly its time; and
// the self query over one mesh of both must give the same pairs across the two parts.  Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <cmath>
#include <cstdio>
#include <algorithm>
#include <array>
#include <vector>

struct V4 { float x, y, z, w; };
struct Rec { float t, d; uint32_t j, iters; };

int main()
{
	int fails = 0;
	const uint32_t na = 2000, iters = 64;
	const float eta = 0.02f, xi = 0.005f;
	std::vector<V4> A0, A1, B = { { -8, -8, 0, 0 }, { 8, -8, 0, 0 }, { 8, 8, 0, 0 }, { -8, -8, 0, 0 }, { 8, 8, 0, 0 }, { -8, 8, 0, 0 } };
	std::vector<double> h( na ), v( na );
	uint32_t seed = 7;
	auto rnd = [&]() { seed = seed * 1664525u + 1013904223u; return (float)(seed >> 8) / 16777216.0f; };
	for (uint32_t i = 0; i < na; i++)
	{
		const float x = rnd() * 14 - 7, y = rnd() * 14 - 7, hz = 0.05f + rnd() * 2, vz = 0.1f + rnd() * 3;
		h[i] = hz, v[i] = vz;
		const V4 c[3] = { { x, y, hz, 0 }, { x + 0.1f, y, hz + 0.05f, 0 }, { x, y + 0.1f, hz + 0.08f, 0 } };
		for (int k = 0; k < 3; k++) A0.push_back( c[k] ), A1.push_back( V4{ c[k].x, c[k].y, c[k].z - vz, 0 } );
		v[i] = (double)hz - (double)(hz - vz); // the fp32 displacement of the lowest corner
	}
	tinybvh_b200::BVH a, b;
	a.Build( A0.data(), na );
	b.BuildHQ( B.data(), 2 );
	std::vector<Rec> rec( na );
	a.TimeOfImpact( A1.data(), b, B.data(), eta, xi, iters, rec.data() );
	std::vector<std::array<uint32_t, 2>> pairs;
	std::vector<float> times;
	a.ImpactPairs( A1.data(), b, B.data(), eta, xi, iters, pairs, times );
	uint32_t hits = 0;
	for (uint32_t i = 0; i < na; i++)
	{
		const double hi = (h[i] - eta) / v[i], lo = (h[i] - eta - xi) / v[i];
		const Rec& r = rec[i];
		bool ok;
		if (r.j == 0xffffffffu) ok = hi > 1 - 1e-5;
		else if (r.iters == iters) ok = r.t <= hi + 1e-5 && r.j < 2;
		else ok = r.t >= lo - 1e-5 && r.t <= hi + 1e-5 && r.j < 2;
		if (r.j != 0xffffffffu) hits++;
		if (!ok) { if (fails < 20) printf( "TimeOfImpact: triangle %u: t %g (j %u, iters %u), fp64 bracket [%g, %g]\n", i, (double)r.t, r.j, r.iters, lo, hi ); fails++; }
	}
	// the record is the earliest of its triangle's pairs: every pair of i comes no earlier, and the one it names at exactly its time
	std::vector<float> first( na, INFINITY );
	for (size_t k = 0; k < pairs.size(); k++)
	{
		const uint32_t i = pairs[k][0];
		if (pairs[k][1] >= 2 || rec[i].j == 0xffffffffu || times[k] < rec[i].t || (pairs[k][1] == rec[i].j && times[k] != rec[i].t))
		{
			if (fails < 20) printf( "ImpactPairs: (%u, %u) at %g, record (%u, %g)\n", i, pairs[k][1], (double)times[k], rec[i].j, (double)rec[i].t );
			fails++;
		}
		first[i] = std::min( first[i], times[k] );
		if (k && !(pairs[k - 1] < pairs[k])) { printf( "ImpactPairs: not sorted at %zu\n", k ); fails++; }
	}
	for (uint32_t i = 0; i < na; i++)
		if ((rec[i].j == 0xffffffffu) != std::isinf( first[i] )) { if (fails < 20) printf( "ImpactPairs: triangle %u has pairs without a record or a record without pairs\n", i ); fails++; }
	// one mesh of both: its pairs across the two parts (i < na, j >= na) are the two-mesh pairs, offset
	std::vector<V4> S0 = A0, S1 = A1;
	S0.insert( S0.end(), B.begin(), B.end() ), S1.insert( S1.end(), B.begin(), B.end() );
	tinybvh_b200::BVH m;
	m.Build( S0.data(), na + 2 );
	std::vector<std::array<uint32_t, 2>> self, cross_pairs;
	std::vector<float> self_times;
	m.ImpactPairs( S1.data(), m, S1.data(), eta, xi, iters, self, self_times );
	for (const auto& p : self) if (p[0] < na && p[1] >= na) cross_pairs.push_back( { p[0], p[1] - na } );
	if (cross_pairs != pairs) { printf( "ImpactPairs self: %zu pairs across the parts, expected %zu\n", cross_pairs.size(), pairs.size() ); fails++; }
	printf( "%u of %u triangles reach the plate, %zu pairs, %zu self pairs\n", hits, na, pairs.size(), self.size() );
	if (hits < na / 4 || hits == na) { printf( "the scene should have triangles on both sides of the step\n" ); fails++; }
	printf( "%d failures\n", fails );
	return fails ? 1 : 0;
}
