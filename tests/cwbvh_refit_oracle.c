/* tests/cwbvh_refit_oracle.c - the oracle of tbvh_refit_layouts' CWBVH.  TEST INFRASTRUCTURE ONLY.
 *
 * The reference has no CWBVH refit, so this is a COMPOSITION of the pinned pieces of oracle/tbvh_oracle_cwbvh.c, which it includes
 * as they are: SplitLeafs( 3 ) of the built and of the refitted tree, MBVH<8>::ConvertFrom of the built one, its boxes replaced by the
 * refitted split tree's (the leaf-root wrap copies the refitted root into node 1), then BVH8_CWBVH::ConvertFrom.  With refit == built it
 * is orc_cwbvh_from_bvh.  Compiled with the flags of that file (oracle/Makefile HQFLAGS: contraction off) by tests/cwbvh_refit_oracle.py.
 */
#include "../oracle/tbvh_oracle_cwbvh.c"

/* built / refit: the same topology (refit = orc_refit of built); verts: the refitted vertices.  data: triCount * 5 float4 blocks, tris:
 * idxCount * 3 float4.  Returns usedBlocks. */
uint32_t orc_cwbvh_refit_from_bvh( const orc_node* built, const orc_node* refit, uint32_t usedNodes, const uint32_t* primIdx, uint32_t idxCount,
	const float* verts, uint32_t triCount, float* data, float* tris )
{
	const size_t room = (size_t)usedNodes + 2 * (size_t)idxCount + 4;
	orc_node* b = (orc_node*)calloc( room, sizeof( orc_node ) ), * r = (orc_node*)calloc( room, sizeof( orc_node ) );
	memcpy( b, built, (size_t)usedNodes * sizeof( orc_node ) ), memcpy( r, refit, (size_t)usedNodes * sizeof( orc_node ) );
	const uint32_t used = split_leafs( b, usedNodes, 3 );
	split_leafs( r, usedNodes, 3 );
	mnode* m = (mnode*)calloc( room, sizeof( mnode ) );
	mbvh8_from_bvh( b, used, m );
	for (uint32_t i = 0; i < used; i++) if (i != 1)
		m[i].mn[0] = r[i].minx, m[i].mn[1] = r[i].miny, m[i].mn[2] = r[i].minz, m[i].mx[0] = r[i].maxx, m[i].mx[1] = r[i].maxy, m[i].mx[2] = r[i].maxz;
	if (b[0].triCount > 0) memcpy( m[1].mn, m[0].mn, 12 ), memcpy( m[1].mx, m[0].mx, 12 );
	const uint32_t blocks = cwbvh_encode( m, primIdx, verts, data, tris, triCount, idxCount );
	free( b ), free( r ), free( m );
	return blocks;
}
