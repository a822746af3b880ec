// harness/refit_indexed_b200.cpp - an animated scene's indexed meshes refitted through the shim: each mesh is a welded grid (a vertex
// list plus 3 indices per triangle, as glTF meshes come), built into a BVH with Build( vertices, indices, primCount ), its vertices
// moved in place, and refitted by RefitBatch (together with flat meshes) or by its own Refit().  Every tree is checked against a twin
// built from the flat triangle soup vertices[indices] and refitted from the soup expanded each frame.  No reference header.
//   g++ -O2 -std=c++17 -Iinclude harness/refit_indexed_b200.cpp -Ltinybvh_b200 -ltinybvh_b200 -Wl,-rpath,$PWD/tinybvh_b200 -o refit_indexed_b200
#include "tinybvh_b200.hpp"
#include <vector>

struct Vec4 { float x, y, z, w; };
static uint32_t seed = 0x2468ace1;
static float rnd() { seed ^= seed << 13, seed ^= seed >> 17, seed ^= seed << 5; return seed * 2.3283064365387e-10f; }

// tree bytes, primIdx and root box of two objects
static bool same_tree( const tinybvh_b200::BVH& a, const tinybvh_b200::BVH& b )
{
	const tbvh_info ia = a.Info(), ib = b.Info();
	std::vector<char> na( (size_t)ia.used_nodes * 32 ), nb( (size_t)ib.used_nodes * 32 );
	std::vector<uint32_t> xa( ia.idx_count ), xb( ib.idx_count );
	a.Download( na.data(), xa.data() ), b.Download( nb.data(), xb.data() );
	bool same = na == nb && xa == xb && a.usedNodes == b.usedNodes;
	for (int k = 0; k < 3; k++) same = same && a.aabbMin[k] == b.aabbMin[k] && a.aabbMax[k] == b.aabbMax[k];
	return same;
}

int main()
{
	const int M = 24;
	std::vector<std::vector<Vec4>> verts( M ), soup( M );
	std::vector<std::vector<uint32_t>> index( M );
	std::vector<uint32_t> prims( M );
	// per mesh: `batched` refitted by RefitBatch, `single` by its own Refit(), `twin` built and refitted from the flat soup
	std::vector<tinybvh_b200::BVH*> batched( M ), single( M ), twin( M );
	for (int m = 0; m < M; m++)
	{
		const uint32_t nx = 1 + (uint32_t)(rnd() * 40), ny = 1 + (uint32_t)(rnd() * 40);
		const float ox = rnd() * 8, oy = rnd() * 8;
		for (uint32_t y = 0; y <= ny; y++) for (uint32_t x = 0; x <= nx; x++)
			verts[m].push_back( { ox + x * 0.1f, oy + y * 0.1f, rnd() * 0.05f, rnd() } );
		if (m % 4 == 3) for (int k = 0; k < 7; k++) verts[m].push_back( { rnd() * 100, rnd() * 100, rnd() * 100, 0 } ); // vertices no triangle uses
		for (uint32_t y = 0; y < ny; y++) for (uint32_t x = 0; x < nx; x++)
		{
			const uint32_t a = y * (nx + 1) + x, b = a + 1, c = a + nx + 1, d = c + 1;
			const uint32_t t[6] = { a, b, c, b, d, c };
			for (uint32_t v : t) index[m].push_back( v );
		}
		prims[m] = (uint32_t)index[m].size() / 3;
		for (uint32_t i = prims[m] - 1; i > 0; i--) // shuffled triangle order
		{
			const uint32_t j = (uint32_t)(rnd() * (i + 1)) % (i + 1);
			for (int k = 0; k < 3; k++) std::swap( index[m][3 * i + k], index[m][3 * j + k] );
		}
		soup[m].resize( index[m].size() );
		for (size_t i = 0; i < index[m].size(); i++) soup[m][i] = verts[m][index[m][i]];
		batched[m] = new tinybvh_b200::BVH(), single[m] = new tinybvh_b200::BVH(), twin[m] = new tinybvh_b200::BVH();
		if (m & 1)
		{
			batched[m]->BuildAVX( verts[m].data(), index[m].data(), prims[m] ), single[m]->BuildAVX( verts[m].data(), index[m].data(), prims[m] );
			twin[m]->BuildAVX( soup[m].data(), prims[m] );
		}
		else
		{
			batched[m]->Build( verts[m].data(), index[m].data(), prims[m] ), single[m]->Build( verts[m].data(), index[m].data(), prims[m] );
			twin[m]->Build( soup[m].data(), prims[m] );
		}
	}
	// flat meshes in the same RefitBatch call
	const int F = 6;
	std::vector<std::vector<Vec4>> flat( F );
	std::vector<tinybvh_b200::BVH*> flatObj( F ), flatTwin( F );
	for (int f = 0; f < F; f++)
	{
		const uint32_t n = 1 + (uint32_t)(rnd() * 500);
		for (uint32_t i = 0; i < 3 * n; i++) flat[f].push_back( { rnd() * 4, rnd() * 4, rnd() * 4, 0 } );
		flatObj[f] = new tinybvh_b200::BVH(), flatTwin[f] = new tinybvh_b200::BVH();
		flatObj[f]->Build( flat[f].data(), n ), flatTwin[f]->Build( flat[f].data(), n );
	}
	std::vector<tinybvh_b200::BVH*> all;
	for (int m = 0; m < M; m++) { all.push_back( batched[m] ); if (m < F) all.push_back( flatObj[m] ); }
	int differ = 0, trees = 0;
	for (int frame = 0; frame < 2; frame++)
	{
		// the animation moves the vertices in the caller's arrays; the objects re-read them through the pointers they kept
		for (int m = 0; m < M; m++)
		{
			for (Vec4& v : verts[m]) v.x += (rnd() - 0.5f) * 0.02f, v.z += rnd() * 0.05f, v.w = rnd();
			for (size_t i = 0; i < index[m].size(); i++) soup[m][i] = verts[m][index[m][i]];
		}
		for (int f = 0; f < F; f++) for (Vec4& v : flat[f]) v.y += (rnd() - 0.5f) * 0.1f;
		tinybvh_b200::RefitBatch( all.data(), (uint32_t)all.size() );
		for (int m = 0; m < M; m++)
		{
			single[m]->Refit(), twin[m]->Refit();
			differ += !same_tree( *batched[m], *twin[m] ), differ += !same_tree( *single[m], *twin[m] ), trees += 2;
		}
		for (int f = 0; f < F; f++) flatTwin[f]->Refit(), differ += !same_tree( *flatObj[f], *flatTwin[f] ), trees++;
	}
	printf( "refit_indexed_b200: %i indexed and %i flat meshes, 2 frames, %i comparisons; %i trees differ from their flat twins\n", M, F, trees, differ );
	for (int m = 0; m < M; m++) delete batched[m], delete single[m], delete twin[m];
	for (int f = 0; f < F; f++) delete flatObj[f], delete flatTwin[f];
	return differ == 0 ? 0 : 1;
}
