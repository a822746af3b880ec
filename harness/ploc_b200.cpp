// harness/ploc_b200.cpp - BuildPLOC through the C++ shim: a flat and an indexed BVH, a BVH_GPU and a BVH8_CWBVH over one procedural
// scene, and a BuildBatch with TBVH_BUILD_PLOC.  The indexed tree and the batch tree must equal the flat one byte for byte, a Refit
// with the build's own vertices must change no byte, and the closest hits of every layout must equal those of the Build tree.
// Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <cstdio>
#include <cstring>
#include <vector>

struct V4 { float x, y, z, w; };
struct Ray128 { float O[3]; uint32_t mask; float D[3]; float pad0; float rD[3]; float pad1; float t, u, v; uint32_t prim; uint8_t rest[64]; };

static std::vector<float> nodes_of( tinybvh_b200::BVH& b, std::vector<uint32_t>& idx )
{
	std::vector<float> a( b.usedNodes * 8 );
	idx.resize( b.idxCount );
	tbvh_download_bvh( b.handle(), a.data(), idx.data(), TBVH_HOST );
	return a;
}

int main()
{
	const uint32_t n = 20000;
	std::vector<V4> soup( n * 3 ), verts;
	std::vector<uint32_t> idx( n * 3 );
	uint32_t seed = 777;
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
	tinybvh_b200::BVH flat, ix, batched, ref;
	flat.BuildPLOC( soup.data(), n );
	ix.BuildPLOC( verts.data(), idx.data(), n );
	tinybvh_b200::BVH* objs[1] = { &batched };
	const V4* vs[1] = { soup.data() };
	tinybvh_b200::BuildBatch( objs, vs, &n, 1, TBVH_BUILD_PLOC );
	ref.Build( soup.data(), n );
	std::vector<uint32_t> pa, pb, pc, pd;
	const std::vector<float> a = nodes_of( flat, pa ), b = nodes_of( ix, pb ), c = nodes_of( batched, pc );
	if (a.size() != b.size() || memcmp( a.data(), b.data(), a.size() * 4 ) || pa != pb) { printf( "indexed tree differs from the flat one\n" ); fails++; }
	if (a.size() != c.size() || memcmp( a.data(), c.data(), a.size() * 4 ) || pa != pc) { printf( "batch tree differs from the single one\n" ); fails++; }
	flat.Refit();
	const std::vector<float> d = nodes_of( flat, pd );
	if (memcmp( a.data(), d.data(), a.size() * 4 )) { printf( "Refit with the build's vertices changed the tree\n" ); fails++; }
	std::vector<Ray128> rays( 4096 ), want;
	for (auto& r : rays)
	{
		memset( &r, 0, sizeof( r ) );
		r.O[0] = 50, r.O[1] = 40, r.O[2] = 50, r.mask = 0xffff;
		r.D[0] = rnd() - 0.5f, r.D[1] = -1, r.D[2] = rnd() - 0.5f;
		for (int k = 0; k < 3; k++) r.rD[k] = 1.0f / r.D[k];
		r.t = 1e30f;
	}
	want = rays;
	ref.Intersect( want.data(), want.size() );
	tinybvh_b200::BVH_GPU g;
	tinybvh_b200::BVH8_CWBVH cw;
	g.BuildPLOC( soup.data(), n ), cw.BuildPLOC( soup.data(), n );
	for (tinybvh_b200::BVHBase* o : { (tinybvh_b200::BVHBase*)&flat, (tinybvh_b200::BVHBase*)&g, (tinybvh_b200::BVHBase*)&cw })
	{
		std::vector<Ray128> got = rays;
		o->Intersect( got.data(), got.size() );
		for (size_t i = 0; i < got.size(); i++) if (memcmp( &got[i].t, &want[i].t, 4 )) { printf( "layout %d: ray %zu t differs\n", o->Layout(), i ); fails++; break; }
	}
	printf( "%d failures\n", fails );
	return fails ? 1 : 0;
}
