// harness/refit_batch_b200.cpp - an animated scene's per-frame refit through the shim's RefitBatch: many meshes, each built into its
// own BVH (some from indexed geometry), the vertices moved, every tree refitted in one call, then checked against a separate Refit of a
// twin built from the same arrays.  No reference header.
//   g++ -O2 -std=c++17 -Iinclude harness/refit_batch_b200.cpp -Ltinybvh_b200 -ltinybvh_b200 -Wl,-rpath,$PWD/tinybvh_b200 -o refit_batch_b200
#include "tinybvh_b200.hpp"
#include <vector>

struct Vec4 { float x, y, z, w; };
static uint32_t seed = 0x13579bdf;
static float rnd() { seed ^= seed << 13, seed ^= seed >> 17, seed ^= seed << 5; return seed * 2.3283064365387e-10f; }

int main()
{
	const int M = 48;
	std::vector<std::vector<Vec4>> verts( M );
	std::vector<std::vector<uint32_t>> index( M );
	std::vector<uint32_t> counts( M );
	std::vector<tinybvh_b200::BVH*> batch( M ), single( M );
	for (int m = 0; m < M; m++)
	{
		counts[m] = 1 + (uint32_t)(rnd() * rnd() * 3000);
		const float ox = rnd() * 8, oy = rnd() * 8;
		const bool indexed = m % 3 == 1; // a vertex list plus 3 indices per triangle
		for (uint32_t i = 0; i < counts[m]; i++)
		{
			const float x = ox + rnd(), y = oy + rnd(), z = rnd() * 4;
			for (int v = 0; v < 3; v++) verts[m].push_back( { x + rnd() * 0.1f, y + rnd() * 0.1f, z + rnd() * 0.1f, 0 } );
			if (indexed) for (int v = 0; v < 3; v++) index[m].push_back( 3 * (counts[m] - 1 - i) + v );
		}
		batch[m] = new tinybvh_b200::BVH(), single[m] = new tinybvh_b200::BVH();
		if (indexed) batch[m]->Build( verts[m].data(), index[m].data(), counts[m] ), single[m]->Build( verts[m].data(), index[m].data(), counts[m] );
		else batch[m]->Build( verts[m].data(), counts[m] ), single[m]->Build( verts[m].data(), counts[m] );
	}
	int differ = 0;
	double ms = 0;
	for (int frame = 0; frame < 2; frame++)
	{
		// the animation moves every vertex in the caller's arrays; the objects re-read them through the pointers they kept
		for (int m = 0; m < M; m++) for (Vec4& v : verts[m]) v.x += (rnd() - 0.5f) * 0.2f, v.z += rnd() * 0.1f;
		tinybvh_b200::RefitBatch( batch.data(), M );
		ms = batch[0]->buildMs;
		for (int m = 0; m < M; m++)
		{
			single[m]->Refit();
			const tbvh_info a = batch[m]->Info(), b = single[m]->Info();
			std::vector<char> na( (size_t)a.used_nodes * 32 ), nb( (size_t)b.used_nodes * 32 );
			std::vector<uint32_t> ia( a.idx_count ), ib( b.idx_count );
			batch[m]->Download( na.data(), ia.data() ), single[m]->Download( nb.data(), ib.data() );
			bool same = na == nb && ia == ib && batch[m]->usedNodes == single[m]->usedNodes;
			for (int k = 0; k < 3; k++) same = same && batch[m]->aabbMin[k] == single[m]->aabbMin[k] && batch[m]->aabbMax[k] == single[m]->aabbMax[k];
			differ += !same;
		}
	}
	printf( "refit_batch_b200: %i meshes, 2 frames, last batch refit %.3f ms; %i trees differ from separate refits\n", M, ms, differ );
	for (int m = 0; m < M; m++) delete batch[m], delete single[m];
	return differ == 0 ? 0 : 1;
}
