// harness/batch_b200.cpp - many meshes through the shim's BuildBatch: one BVH per mesh (the first step of every instanced scene,
// one BLAS per mesh as tiny_scene.h builds them), built in one call, then checked against a separate Build of every mesh and
// walked with a batch of rays.  BVH8_CWBVH objects go through the overload that converts each tree afterwards.  A BuildHQ batch
// (TBVH_BUILD_HQ) is checked against a separate BuildHQ of every mesh.  No reference header.
//   g++ -O2 -std=c++17 -Iinclude harness/batch_b200.cpp -Ltinybvh_b200 -ltinybvh_b200 -Wl,-rpath,$PWD/tinybvh_b200 -o batch_b200
#include "tinybvh_b200.hpp"
#include <vector>

struct Vec4 { float x, y, z, w; };
static uint32_t seed = 0x2468ace1;
static float rnd() { seed ^= seed << 13, seed ^= seed >> 17, seed ^= seed << 5; return seed * 2.3283064365387e-10f; }

int main()
{
	const int M = 64, R = 1024;
	std::vector<std::vector<Vec4>> meshes( M );
	std::vector<const Vec4*> verts( M );
	std::vector<uint32_t> counts( M );
	uint32_t total = 0;
	for (int m = 0; m < M; m++)
	{
		counts[m] = 1 + (uint32_t)(rnd() * rnd() * 4000); // mostly small meshes, a few of some thousand triangles
		const float ox = rnd() * 8, oy = rnd() * 8;
		for (uint32_t i = 0; i < counts[m]; i++)
		{
			const float x = ox + rnd(), y = oy + rnd(), z = rnd() * 4;
			for (int v = 0; v < 3; v++) meshes[m].push_back( { x + rnd() * 0.1f, y + rnd() * 0.1f, z + rnd() * 0.1f, 0 } );
		}
		verts[m] = meshes[m].data(), total += counts[m];
	}
	std::vector<tinybvh_b200::BVH*> batch( M ), single( M );
	for (int m = 0; m < M; m++) batch[m] = new tinybvh_b200::BVH(), single[m] = new tinybvh_b200::BVH();
	tinybvh_b200::BuildBatch( batch.data(), verts.data(), counts.data(), M );
	int differ = 0;
	for (int m = 0; m < M; m++)
	{
		single[m]->Build( verts[m], counts[m] );
		const tbvh_info a = batch[m]->Info(), b = single[m]->Info();
		std::vector<char> na( (size_t)a.used_nodes * 32 ), nb( (size_t)b.used_nodes * 32 );
		std::vector<uint32_t> ia( a.idx_count ), ib( b.idx_count );
		batch[m]->Download( na.data(), ia.data() ), single[m]->Download( nb.data(), ib.data() );
		if (batch[m]->usedNodes != single[m]->usedNodes || batch[m]->triCount != counts[m] || a.max_depth != b.max_depth || na != nb || ia != ib) differ++;
	}
	// the wide layout: one batch, each object converted to its CWBVH
	std::vector<tinybvh_b200::BVH8_CWBVH*> wide( M );
	for (int m = 0; m < M; m++) wide[m] = new tinybvh_b200::BVH8_CWBVH();
	tinybvh_b200::BuildBatch( wide.data(), verts.data(), counts.data(), M );
	// rays down onto mesh 0 through both layouts of it
	tinybvh_b200::Ray* rays = (tinybvh_b200::Ray*)tinybvh_b200::malloc_pinned( 2 * R * sizeof( tinybvh_b200::Ray ) );
	for (int i = 0; i < 2 * R; i++)
	{
		const float O[3] = { batch[0]->aabbMin[0] + (batch[0]->aabbMax[0] - batch[0]->aabbMin[0]) * ((i % R) % 32) / 32.0f,
			batch[0]->aabbMin[1] + (batch[0]->aabbMax[1] - batch[0]->aabbMin[1]) * ((i % R) / 32) / 32.0f, 10 }, D[3] = { 0, 0, -1 };
		rays[i] = tinybvh_b200::Ray( O, D );
	}
	batch[0]->Intersect( rays, R );
	wide[0]->Intersect( rays + R, R );
	int hits = 0, mismatched = 0;
	// the CWBVH walk of the AVX flavour's tree and the BVH2 walk of the reference flavour's tree find the same nearest triangles
	for (int i = 0; i < R; i++) hits += rays[i].t < 1e30f, mismatched += (rays[i].t < 1e30f) != (rays[R + i].t < 1e30f) || rays[i].prim != rays[R + i].prim;
	printf( "batch_b200: %i meshes, %u tris, batch build %.3f ms; %i trees differ from separate builds; mesh 0: %i of %i rays hit, %i differ between layouts, %u CWBVH blocks\n",
		M, total, batch[0]->buildMs, differ, hits, R, mismatched, wide[0]->usedBlocks );
	// the SBVH builder: one BuildBatch with TBVH_BUILD_HQ against a separate BuildHQ of every mesh
	int differHQ = 0;
	std::vector<tinybvh_b200::BVH*> hq( M ), hqSingle( M );
	for (int m = 0; m < M; m++) hq[m] = new tinybvh_b200::BVH(), hqSingle[m] = new tinybvh_b200::BVH();
	tinybvh_b200::BuildBatch( hq.data(), verts.data(), counts.data(), M, TBVH_BUILD_HQ );
	for (int m = 0; m < M; m++)
	{
		hqSingle[m]->BuildHQ( verts[m], counts[m] );
		const tbvh_info a = hq[m]->Info(), b = hqSingle[m]->Info();
		std::vector<char> na( (size_t)a.used_nodes * 32 ), nb( (size_t)b.used_nodes * 32 );
		std::vector<uint32_t> ia( a.idx_count ), ib( b.idx_count );
		hq[m]->Download( na.data(), ia.data() ), hqSingle[m]->Download( nb.data(), ib.data() );
		if (hq[m]->usedNodes != hqSingle[m]->usedNodes || hq[m]->idxCount != hqSingle[m]->idxCount || a.max_depth != b.max_depth || na != nb || ia != ib) differHQ++;
	}
	printf( "batch_b200: BuildHQ batch %.3f ms; %i HQ trees differ from separate BuildHQ builds\n", hq[0]->buildMs, differHQ );
	tinybvh_b200::free_pinned( rays );
	for (int m = 0; m < M; m++) delete batch[m], delete single[m], delete wide[m], delete hq[m], delete hqSingle[m];
	return differ == 0 && differHQ == 0 && mismatched == 0 && hits > 0 ? 0 : 1;
}
