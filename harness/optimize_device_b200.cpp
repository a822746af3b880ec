// harness/optimize_device_b200.cpp - OptimizeOnDevice through the C++ shim: a flat and an indexed BVH, a BVH_GPU and a BVH8_CWBVH over
// one procedural scene.  Every optimised tree must cost less than the built one, the indexed tree must equal the flat one (same
// triangles, same build), and the closest hits of every layout must keep their distances.  Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

struct V4 { float x, y, z, w; };
struct Ray128 { float O[3]; uint32_t mask; float D[3]; float pad0; float rD[3]; float pad1; float t, u, v; uint32_t prim; uint8_t rest[64]; };

int main()
{
	const uint32_t n = 20000;
	std::vector<V4> soup( n * 3 ), verts;
	std::vector<uint32_t> idx( n * 3 );
	uint32_t seed = 12345;
	auto rnd = [&]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
	for (uint32_t i = 0; i < n; i++)
	{
		const float cx = rnd() * 100, cy = rnd() * 20, cz = rnd() * 100;
		for (int k = 0; k < 3; k++)
		{
			soup[i * 3 + k] = V4{ cx + rnd(), cy + rnd(), cz + rnd(), 0 };
			idx[i * 3 + k] = (uint32_t)verts.size();
			verts.push_back( soup[i * 3 + k] );
		}
	}
	int fails = 0;
	tinybvh_b200::BVH flat, ix;
	flat.Build( soup.data(), n );
	ix.Build( verts.data(), idx.data(), n );
	float before = 0, after = 0;
	tbvh_sah_cost( flat.handle(), 1, 1, &before );
	std::vector<Ray128> rays( 4096 ), ref;
	for (auto& r : rays)
	{
		memset( &r, 0, sizeof( r ) );
		r.O[0] = 50, r.O[1] = 40, r.O[2] = 50, r.mask = 0xffff;
		r.D[0] = rnd() - 0.5f, r.D[1] = -1, r.D[2] = rnd() - 0.5f;
		for (int k = 0; k < 3; k++) r.rD[k] = 1.0f / r.D[k];
		r.t = 1e30f;
	}
	ref = rays;
	flat.Intersect( ref.data(), ref.size() );
	const uint32_t r1 = flat.OptimizeOnDevice( 4 ), r2 = ix.OptimizeOnDevice( 4 );
	tbvh_sah_cost( flat.handle(), 1, 1, &after );
	if (r1 == 0 || r1 != r2 || !(after < before)) { printf( "rounds %u / %u, SAH %f -> %f\n", r1, r2, before, after ); fails++; }
	std::vector<float> a( flat.usedNodes * 8 ), b( ix.usedNodes * 8 );
	std::vector<uint32_t> pa( flat.idxCount ), pb( ix.idxCount );
	tbvh_download_bvh( flat.handle(), a.data(), pa.data(), TBVH_HOST ), tbvh_download_bvh( ix.handle(), b.data(), pb.data(), TBVH_HOST );
	if (a.size() != b.size() || memcmp( a.data(), b.data(), a.size() * 4 )) { printf( "indexed tree differs from the flat one\n" ); fails++; }
	tinybvh_b200::BVH_GPU g;
	tinybvh_b200::BVH8_CWBVH cw;
	g.Build( soup.data(), n ), cw.Build( soup.data(), n );
	g.OptimizeOnDevice( 4 ), cw.OptimizeOnDevice( 4 );
	for (tinybvh_b200::BVHBase* o : { (tinybvh_b200::BVHBase*)&flat, (tinybvh_b200::BVHBase*)&g, (tinybvh_b200::BVHBase*)&cw })
	{
		std::vector<Ray128> got = rays;
		o->Intersect( got.data(), got.size() );
		for (size_t i = 0; i < got.size(); i++) if (memcmp( &got[i].t, &ref[i].t, 4 )) { printf( "layout %d: ray %zu t differs\n", o->Layout(), i ); fails++; break; }
	}
	printf( "%d failures\n", fails );
	return fails ? 1 : 0;
}
