/* oracle/tbvh_oracle_hq.c - plain-C restatement of the reference's SBVH builder, BVH::BuildHQ.
 *
 * TEST INFRASTRUCTURE ONLY (see tbvh_oracle.h).  Follows tiny_bvh.h: PrepareHQBuild :2648-2709, SplitCostSAH :2711-2716,
 * BuildHQTask :2731-3008 (single-threaded path), BuildHQ :3010-3040, Compact :3733-3770, ClipFrag :8614-8729,
 * SplitFrag :8731-8793.  hqbvhbins = 8, hqbvhoddeven = false, l_quads = false (the defaults of BVH).
 *
 * Floating point: like tbvh_oracle.c this file is compiled with -ffp-contract=off and spells every fused multiply-add the
 * frozen reference build (g++ -O3 -mavx2 -mfma, default -ffp-contract=fast) contains as an explicit fmaf(), read off the
 * disassembly of BVH::BuildHQTask / ClipFrag / SplitFrag in oracle/_ref/libtinybvh_ref.so:
 *   half area / SA       fmaf( ez, ex, fmaf( ey, ex, ey*ez ) )                      (:460, :8477)
 *   SplitCostSAH         fmaf( fmaf( lN, Aleft, Aright*rN ), c_int*rAparent, c_trav )  (:2711)
 *   object bin           trunc( fmaf( bmin+bmax, 0.5, -nmin ) * rpd )               (:2765, :2959)
 *   spatial bin plane    fmaf( j, planeDist, nodeMin )                              (:2838)
 *   clip interpolation   C = fmaf( f, v1-v0, v0 ) per component                     (:8640-8713, :8760-8787)
 * tests/test_oracle_pin.py pins clip_frag / split_frag against BVH::ClipFrag / SplitFrag on random fragments and the
 * whole build against BVH::BuildHQ byte for byte.
 */
#include "tbvh_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define BVH_FAR 1e30f
#define HQBINS 8

typedef struct { float bmin[3]; uint32_t primIdx; float bmax[3]; uint32_t clipped; } frag_t;
typedef struct { const float* verts; frag_t* fragment; uint32_t* primIdx; orc_node* nodes; uint32_t newNodePtr, nextFrag; float c_trav, c_int; } hq_t;

static inline float fmin_( float a, float b ) { return a < b ? a : b; }
static inline float fmax_( float a, float b ) { return a > b ? a : b; }
static inline float clampf_( float x, float a, float b ) { return x > a ? (x < b ? x : b) : a; }
static inline int clampi_( int x, int a, int b ) { return x > a ? (x < b ? x : b) : a; }
static inline float half_area3( const float* v ) { return v[0] < -BVH_FAR ? 0 : fmaf( v[2], v[0], fmaf( v[1], v[0], v[1] * v[2] ) ); } /* :460 */
static inline float sa_node( const orc_node* n ) /* BVHBase::SA :8477 */
{
	const float ex = n->maxx - n->minx, ey = n->maxy - n->miny, ez = n->maxz - n->minz;
	return fmaf( ez, ex, fmaf( ey, ex, ey * ez ) );
}
static inline float split_cost( const hq_t* h, float rAparent, float Aleft, int Nleft, float Aright, int Nright ) /* :2711 */
{
	return fmaf( fmaf( (float)Nleft, Aleft, Aright * (float)Nright ), h->c_int * rAparent, h->c_trav );
}
static inline void vget( const hq_t* h, uint32_t vi, float* o ) { const float* p = h->verts + (size_t)vi * 4; o[0] = p[0], o[1] = p[1], o[2] = p[2]; }

/* ClipFrag :8614-8729 */
static int clip_frag( const hq_t* h, const frag_t* orig, frag_t* nf, const float* bmin_in, const float* bmax_in, const float* minDim, uint32_t axis )
{
	float bmin[3], bmax[3], extent[3];
	for (int a = 0; a < 3; a++) bmin[a] = fmax_( bmin_in[a], orig->bmin[a] ), bmax[a] = fmin_( bmax_in[a], orig->bmax[a] ), extent[a] = bmax[a] - bmin[a];
	uint32_t Nin = 3, vidx = orig->primIdx * 3;
	if (orig->clipped)
	{
		float vin[16][3], vout[16][3];
		vget( h, vidx, vin[0] ), vget( h, vidx + 1, vin[1] ), vget( h, vidx + 2, vin[2] );
		for (uint32_t a = 0; a < 3; a++)
		{
			const float eps = minDim[a];
			if (extent[a] > eps)
			{
				uint32_t Nout = 0;
				const float l = bmin[a], r = bmax[a];
				for (uint32_t v = 0; v < Nin; v++)
				{
					const float* v0 = vin[v], * v1 = vin[(v + 1) % Nin];
					const int v0in = v0[a] >= l - eps, v1in = v1[a] >= l - eps;
					if (!(v0in || v1in)) continue; else if (v0in ^ v1in)
					{
						const float f = (l - v0[a]) / (v1[a] - v0[a]);
						float C[3] = { fmaf( f, v1[0] - v0[0], v0[0] ), fmaf( f, v1[1] - v0[1], v0[1] ), fmaf( f, v1[2] - v0[2], v0[2] ) };
						C[a] = l;
						memcpy( vout[Nout++], C, 12 );
					}
					if (v1in) memcpy( vout[Nout++], v1, 12 );
				}
				Nin = 0;
				for (uint32_t v = 0; v < Nout; v++)
				{
					const float* v0 = vout[v], * v1 = vout[(v + 1) % Nout];
					const int v0in = v0[a] <= r + eps, v1in = v1[a] <= r + eps;
					if (!(v0in || v1in)) continue; else if (v0in ^ v1in)
					{
						const float f = (r - v0[a]) / (v1[a] - v0[a]);
						float C[3] = { fmaf( f, v1[0] - v0[0], v0[0] ), fmaf( f, v1[1] - v0[1], v0[1] ), fmaf( f, v1[2] - v0[2], v0[2] ) };
						C[a] = r;
						memcpy( vin[Nin++], C, 12 );
					}
					if (v1in) memcpy( vin[Nin++], v1, 12 );
				}
			}
		}
		float mn[3] = { BVH_FAR, BVH_FAR, BVH_FAR }, mx[3] = { -BVH_FAR, -BVH_FAR, -BVH_FAR };
		for (uint32_t i = 0; i < Nin; i++) for (int k = 0; k < 3; k++) mn[k] = fmin_( mn[k], vin[i][k] ), mx[k] = fmax_( mx[k], vin[i][k] );
		nf->primIdx = orig->primIdx;
		for (int k = 0; k < 3; k++) nf->bmin[k] = fmax_( mn[k], bmin[k] ), nf->bmax[k] = fmin_( mx[k], bmax[k] );
		nf->clipped = 1;
		return Nin > 0;
	}
	else
	{
		int hasVerts = 0;
		float mn[3] = { BVH_FAR, BVH_FAR, BVH_FAR }, mx[3] = { -BVH_FAR, -BVH_FAR, -BVH_FAR }, vout[4][3], C[3];
		if (extent[axis] > minDim[axis])
		{
			const float l = bmin[axis], r = bmax[axis];
			uint32_t Nout = 0;
			{
				float v0[3], v1[3], v2[3];
				vget( h, vidx, v0 ), vget( h, vidx + 1, v1 ), vget( h, vidx + 2, v2 );
				const int v0in = v0[axis] >= l, v1in = v1[axis] >= l, v2in = v2[axis] >= l;
				if (v0in || v1in)
				{
					if (v0in ^ v1in)
					{
						const float f = clampf_( (l - v0[axis]) / (v1[axis] - v0[axis]), 0.0f, 1.0f );
						for (int k = 0; k < 3; k++) C[k] = fmaf( f, v1[k] - v0[k], v0[k] );
						C[axis] = l, memcpy( vout[Nout++], C, 12 );
					}
					if (v1in) memcpy( vout[Nout++], v1, 12 );
				}
				if (v1in || v2in)
				{
					if (v1in ^ v2in)
					{
						const float f = clampf_( (l - v1[axis]) / (v2[axis] - v1[axis]), 0.0f, 1.0f );
						for (int k = 0; k < 3; k++) C[k] = fmaf( f, v2[k] - v1[k], v1[k] );
						C[axis] = l, memcpy( vout[Nout++], C, 12 );
					}
					if (v2in) memcpy( vout[Nout++], v2, 12 );
				}
				if (v2in || v0in)
				{
					if (v2in ^ v0in)
					{
						const float f = clampf_( (l - v2[axis]) / (v0[axis] - v2[axis]), 0.0f, 1.0f );
						for (int k = 0; k < 3; k++) C[k] = fmaf( f, v0[k] - v2[k], v2[k] );
						C[axis] = l, memcpy( vout[Nout++], C, 12 );
					}
					if (v0in) memcpy( vout[Nout++], v0, 12 );
				}
			}
			for (uint32_t v = 0; v < Nout; v++)
			{
				const float* v0 = vout[v], * v1 = vout[(v + 1) % Nout];
				const int v0in = v0[axis] <= r, v1in = v1[axis] <= r;
				if (!(v0in || v1in)) continue; else if (v0in ^ v1in)
				{
					const float f = clampf_( (r - v0[axis]) / (v1[axis] - v0[axis]), 0.0f, 1.0f );
					for (int k = 0; k < 3; k++) C[k] = fmaf( f, v1[k] - v0[k], v0[k] );
					C[axis] = r, hasVerts = 1;
					for (int k = 0; k < 3; k++) mn[k] = fmin_( mn[k], C[k] ), mx[k] = fmax_( mx[k], C[k] );
				}
				if (v1in) { hasVerts = 1; for (int k = 0; k < 3; k++) mn[k] = fmin_( mn[k], v1[k] ), mx[k] = fmax_( mx[k], v1[k] ); }
			}
		}
		for (int k = 0; k < 3; k++) nf->bmin[k] = fmax_( mn[k], bmin[k] ), nf->bmax[k] = fmin_( mx[k], bmax[k] );
		nf->primIdx = orig->primIdx, nf->clipped = 1;
		return hasVerts;
	}
}

/* SplitFrag :8731-8793 */
static void split_frag( const hq_t* h, const frag_t* orig, frag_t* left, frag_t* right, const float* minDim, uint32_t splitAxis, float splitPos, int* leftOK, int* rightOK )
{
	float vin[16][3], vout[16][3], vleft[16][3], vright[16][3];
	uint32_t vidx = orig->primIdx * 3, Nin = 3, Nout = 0, Nleft = 0, Nright = 0;
	vget( h, vidx, vin[0] ), vget( h, vidx + 1, vin[1] ), vget( h, vidx + 2, vin[2] );
	const float extent[3] = { orig->bmax[0] - orig->bmin[0], orig->bmax[1] - orig->bmin[1], orig->bmax[2] - orig->bmin[2] };
	if (orig->clipped) for (int a = 0; a < 3; a++) if (extent[a] > minDim[a])
	{
		const float l = orig->bmin[a], r = orig->bmax[a];
		Nout = 0;
		for (uint32_t v = 0; v < Nin; v++)
		{
			const float* v0 = vin[v], * v1 = vin[(v + 1) % Nin];
			const int v0in = v0[a] >= l, v1in = v1[a] >= l;
			if (!(v0in || v1in)) continue; else if (v0in ^ v1in)
			{
				const float f = clampf_( (l - v0[a]) / (v1[a] - v0[a]), 0.0f, 1.0f );
				float C[3] = { fmaf( f, v1[0] - v0[0], v0[0] ), fmaf( f, v1[1] - v0[1], v0[1] ), fmaf( f, v1[2] - v0[2], v0[2] ) };
				C[a] = l, memcpy( vout[Nout++], C, 12 );
			}
			if (v1in) memcpy( vout[Nout++], v1, 12 );
		}
		Nin = 0;
		for (uint32_t v = 0; v < Nout; v++)
		{
			const float* v0 = vout[v], * v1 = vout[(v + 1) % Nout];
			const int v0in = v0[a] <= r, v1in = v1[a] <= r;
			if (!(v0in || v1in)) continue; else if (v0in ^ v1in)
			{
				const float f = clampf_( (r - v0[a]) / (v1[a] - v0[a]), 0.0f, 1.0f );
				float C[3] = { fmaf( f, v1[0] - v0[0], v0[0] ), fmaf( f, v1[1] - v0[1], v0[1] ), fmaf( f, v1[2] - v0[2], v0[2] ) };
				C[a] = r, memcpy( vin[Nin++], C, 12 );
			}
			if (v1in) memcpy( vin[Nin++], v1, 12 );
		}
	}
	for (uint32_t v = 0; v < Nin; v++)
	{
		const float* v0 = vin[v], * v1 = vin[(v + 1) % Nin];
		const int v0left = v0[splitAxis] < splitPos, v1left = v1[splitAxis] < splitPos;
		if (v0left && v1left) memcpy( vleft[Nleft++], v1, 12 ); else if (!v0left && !v1left) memcpy( vright[Nright++], v1, 12 ); else
		{
			const float f = clampf_( (splitPos - v0[splitAxis]) / (v1[splitAxis] - v0[splitAxis]), 0.0f, 1.0f );
			float C[3] = { fmaf( f, v1[0] - v0[0], v0[0] ), fmaf( f, v1[1] - v0[1], v0[1] ), fmaf( f, v1[2] - v0[2], v0[2] ) };
			C[splitAxis] = splitPos;
			if (v0left) { memcpy( vleft[Nleft++], C, 12 ), memcpy( vright[Nright++], C, 12 ), memcpy( vright[Nright++], v1, 12 ); }
			else { memcpy( vright[Nright++], C, 12 ), memcpy( vleft[Nleft++], C, 12 ), memcpy( vleft[Nleft++], v1, 12 ); }
		}
	}
	for (int k = 0; k < 3; k++) left->bmin[k] = right->bmin[k] = BVH_FAR, left->bmax[k] = right->bmax[k] = -BVH_FAR;
	for (uint32_t i = 0; i < Nleft; i++) for (int k = 0; k < 3; k++) left->bmin[k] = fmin_( left->bmin[k], vleft[i][k] ), left->bmax[k] = fmax_( left->bmax[k], vleft[i][k] );
	for (uint32_t i = 0; i < Nright; i++) for (int k = 0; k < 3; k++) right->bmin[k] = fmin_( right->bmin[k], vright[i][k] ), right->bmax[k] = fmax_( right->bmax[k], vright[i][k] );
	left->clipped = right->clipped = 1, left->primIdx = right->primIdx = orig->primIdx;
	*leftOK = Nleft > 0, *rightOK = Nright > 0;
}

typedef struct { uint32_t node, sliceStart, sliceEnd, depth; } task_t;
uint32_t orc_hq_failed_splits = 0; /* diagnostics: low 16 bits = 'spatial split failed' leaves (:2939), high bits = those that read stale idxTmp words */
uint32_t orc_hq_failed_max = 0;    /* diagnostics: fragment count of the largest node whose spatial split failed */

/* BuildHQTask :2731-3008, non-threaded */
static void build_hq_task( hq_t* h, uint32_t nodeIdx, uint32_t sliceStart, uint32_t sliceEnd, uint32_t* idxTmp )
{
	task_t* localTask = (task_t*)malloc( 4096 * sizeof( task_t ) );
	uint32_t localTasks = 0, depth = 0;
	float bestLMin[3] = { 0, 0, 0 }, bestLMax[3] = { 0, 0, 0 }, bestRMin[3] = { 0, 0, 0 }, bestRMax[3] = { 0, 0, 0 };
	orc_node* root = &h->nodes[0];
	frag_t* fragment = h->fragment;
	uint32_t* primIdx = h->primIdx;
	const float rootExt[3] = { root->maxx - root->minx, root->maxy - root->miny, root->maxz - root->minz };
	const float rootArea = half_area3( rootExt );
	const float minDim[3] = { rootExt[0] * 1e-7f, rootExt[1] * 1e-7f, rootExt[2] * 1e-7f };
	const uint32_t binCount = HQBINS;
	while (1)
	{
		while (1)
		{
			orc_node* node = &h->nodes[nodeIdx];
			const float nmin3[3] = { node->minx, node->miny, node->minz }, nmax3[3] = { node->maxx, node->maxy, node->maxz };
			float binMin[3][HQBINS][3], binMax[3][HQBINS][3];
			uint32_t count[3][HQBINS];
			for (int a = 0; a < 3; a++) for (uint32_t i = 0; i < binCount; i++) for (int k = 0; k < 3; k++) binMin[a][i][k] = BVH_FAR, binMax[a][i][k] = -BVH_FAR;
			memset( count, 0, sizeof( count ) );
			float rpd3[3];
			for (int a = 0; a < 3; a++) rpd3[a] = (float)binCount / (nmax3[a] - nmin3[a]);
			for (uint32_t i = 0; i < node->triCount; i++)
			{
				const frag_t* f = &fragment[primIdx[node->leftFirst + i]];
				for (int a = 0; a < 3; a++)
				{
					const int bi = clampi_( (int)(fmaf( f->bmin[a] + f->bmax[a], 0.5f, -nmin3[a] ) * rpd3[a]), 0, (int)binCount - 1 );
					for (int k = 0; k < 3; k++) binMin[a][bi][k] = fmin_( binMin[a][bi][k], f->bmin[k] ), binMax[a][bi][k] = fmax_( binMax[a][bi][k], f->bmax[k] );
					count[a][bi]++;
				}
			}
			const float noSplitCost = (float)node->triCount * h->c_int;
			float splitCost = noSplitCost;
			const float rSAV = 1.0f / sa_node( node );
			uint32_t bestAxis = 0, bestPos = 0;
			for (int a = 0; a < 3; a++) if ((nmax3[a] - nmin3[a]) > minDim[a])
			{
				float lBMin[HQBINS - 1][3], rBMin[HQBINS - 1][3], lBMax[HQBINS - 1][3], rBMax[HQBINS - 1][3];
				float l1[3] = { BVH_FAR, BVH_FAR, BVH_FAR }, l2[3] = { -BVH_FAR, -BVH_FAR, -BVH_FAR }, r1[3] = { BVH_FAR, BVH_FAR, BVH_FAR }, r2[3] = { -BVH_FAR, -BVH_FAR, -BVH_FAR };
				float AL[HQBINS - 1], AR[HQBINS - 1];
				int NL[HQBINS - 1], NR[HQBINS - 1];
				uint32_t lN = 0, rN = 0;
				for (uint32_t i = 0; i < binCount - 1; i++)
				{
					for (int k = 0; k < 3; k++)
					{
						lBMin[i][k] = l1[k] = fmin_( l1[k], binMin[a][i][k] ), rBMin[binCount - 2 - i][k] = r1[k] = fmin_( r1[k], binMin[a][binCount - 1 - i][k] );
						lBMax[i][k] = l2[k] = fmax_( l2[k], binMax[a][i][k] ), rBMax[binCount - 2 - i][k] = r2[k] = fmax_( r2[k], binMax[a][binCount - 1 - i][k] );
					}
					lN += count[a][i], rN += count[a][binCount - 1 - i];
					NL[i] = (int)lN, NR[binCount - 2 - i] = (int)rN;
					const float dl[3] = { l2[0] - l1[0], l2[1] - l1[1], l2[2] - l1[2] }, dr[3] = { r2[0] - r1[0], r2[1] - r1[1], r2[2] - r1[2] };
					AL[i] = lN == 0 ? BVH_FAR : half_area3( dl );
					AR[binCount - 2 - i] = rN == 0 ? BVH_FAR : half_area3( dr );
				}
				for (uint32_t i = 0; i < binCount - 1; i++)
				{
					const float C = split_cost( h, rSAV, AL[i], NL[i], AR[i], NR[i] );
					if (C >= splitCost) continue;
					splitCost = C, bestAxis = a, bestPos = i;
					for (int k = 0; k < 3; k++) bestLMin[k] = lBMin[i][k], bestRMin[k] = rBMin[i][k], bestLMax[k] = lBMax[i][k], bestRMax[k] = rBMax[i][k];
				}
			}
			/* consider a spatial split :2804-2872 */
			int spatial = 0, bestNL = 0, bestNR = 0;
			const int budget = (int)(sliceEnd - sliceStart);
			const float spatialUnion[3] = { bestLMax[0] - bestRMin[0], bestLMax[1] - bestRMin[1], bestLMax[2] - bestRMin[2] };
			const float spatialOverlap = half_area3( spatialUnion ) / rootArea;
			if (budget > (int)node->triCount && (spatialOverlap > 1e-4f || splitCost >= noSplitCost))
			{
				float minSplitCost = splitCost * 0.985f;
				for (int a = 0; a < 3; a++) if ((nmax3[a] - nmin3[a]) > minDim[a])
				{
					float sbinMin[HQBINS][3], sbinMax[HQBINS][3];
					int countIn[HQBINS], countOut[HQBINS];
					memset( countIn, 0, sizeof( countIn ) ), memset( countOut, 0, sizeof( countOut ) );
					for (uint32_t i = 0; i < binCount; i++) for (int k = 0; k < 3; k++) sbinMin[i][k] = BVH_FAR, sbinMax[i][k] = -BVH_FAR;
					const float planeDist = (nmax3[a] - nmin3[a]) / (binCount * 0.9999f);
					const float rPlaneDist = 1.0f / planeDist, nodeMin = nmin3[a];
					for (uint32_t i = 0; i < node->triCount; i++)
					{
						const uint32_t fi = primIdx[node->leftFirst + i];
						const int bin1 = clampi_( (int)((fragment[fi].bmin[a] - nodeMin) * rPlaneDist), 0, (int)binCount - 1 );
						const int bin2 = clampi_( (int)((fragment[fi].bmax[a] - nodeMin) * rPlaneDist), 0, (int)binCount - 1 );
						countIn[bin1]++, countOut[bin2]++;
						if (bin2 == bin1)
						{
							for (int k = 0; k < 3; k++) sbinMin[bin1][k] = fmin_( sbinMin[bin1][k], fragment[fi].bmin[k] ), sbinMax[bin1][k] = fmax_( sbinMax[bin1][k], fragment[fi].bmax[k] );
						}
						else for (int j = bin1; j <= bin2; j++)
						{
							float bmin[3] = { nmin3[0], nmin3[1], nmin3[2] }, bmax[3] = { nmax3[0], nmax3[1], nmax3[2] };
							bmin[a] = fmaf( (float)j, planeDist, nodeMin );
							bmax[a] = j == (int)(binCount - 2) ? nmax3[a] : (bmin[a] + planeDist);
							const frag_t orig = fragment[fi];
							frag_t tmpFrag;
							if (!clip_frag( h, &orig, &tmpFrag, bmin, bmax, minDim, (uint32_t)a )) continue;
							for (int k = 0; k < 3; k++) sbinMin[j][k] = fmin_( sbinMin[j][k], tmpFrag.bmin[k] ), sbinMax[j][k] = fmax_( sbinMax[j][k], tmpFrag.bmax[k] );
						}
					}
					float lBMin[HQBINS - 1][3], rBMin[HQBINS - 1][3], lBMax[HQBINS - 1][3], rBMax[HQBINS - 1][3];
					float l1[3] = { BVH_FAR, BVH_FAR, BVH_FAR }, l2[3] = { -BVH_FAR, -BVH_FAR, -BVH_FAR }, r1[3] = { BVH_FAR, BVH_FAR, BVH_FAR }, r2[3] = { -BVH_FAR, -BVH_FAR, -BVH_FAR };
					float AL[HQBINS], AR[HQBINS];
					int NL[HQBINS], NR[HQBINS];
					uint32_t lN = 0, rN = 0;
					for (uint32_t i = 0; i < binCount - 1; i++)
					{
						for (int k = 0; k < 3; k++)
						{
							lBMin[i][k] = l1[k] = fmin_( l1[k], sbinMin[i][k] ), rBMin[binCount - 2 - i][k] = r1[k] = fmin_( r1[k], sbinMin[binCount - 1 - i][k] );
							lBMax[i][k] = l2[k] = fmax_( l2[k], sbinMax[i][k] ), rBMax[binCount - 2 - i][k] = r2[k] = fmax_( r2[k], sbinMax[binCount - 1 - i][k] );
						}
						lN += (uint32_t)countIn[i], rN += (uint32_t)countOut[binCount - 1 - i];
						const float dl[3] = { l2[0] - l1[0], l2[1] - l1[1], l2[2] - l1[2] }, dr[3] = { r2[0] - r1[0], r2[1] - r1[1], r2[2] - r1[2] };
						AL[i] = lN == 0 ? BVH_FAR : half_area3( dl );
						AR[binCount - 2 - i] = rN == 0 ? BVH_FAR : half_area3( dr );
						NL[i] = (int)lN, NR[binCount - 2 - i] = (int)rN;
					}
					for (uint32_t i = 0; i < binCount - 1; i++)
					{
						const float Cspatial = split_cost( h, rSAV, AL[i], NL[i], AR[i], NR[i] );
						if (Cspatial < minSplitCost && NL[i] + NR[i] < budget && (int32_t)((uint32_t)NL[i] * (uint32_t)NR[i]) > 0) /* 32-bit wrap-around product, as the frozen reference build computes it (imul) */
						{
							spatial = 1, minSplitCost = splitCost = Cspatial, bestAxis = (uint32_t)a, bestPos = i;
							for (int k = 0; k < 3; k++) bestLMin[k] = lBMin[i][k], bestLMax[k] = lBMax[i][k], bestRMin[k] = rBMin[i][k], bestRMax[k] = rBMax[i][k];
							bestNL = NL[i], bestNR = NR[i];
							bestLMax[a] = bestRMin[a];
						}
					}
				}
			}
			if (splitCost >= noSplitCost)
			{
				for (uint32_t i = 0; i < node->triCount; i++) primIdx[node->leftFirst + i] = fragment[primIdx[node->leftFirst + i]].primIdx;
				break;
			}
			/* double-buffered partition :2882-2964 */
			uint32_t A = sliceStart, B = sliceEnd, src = node->leftFirst;
			if (spatial)
			{
				const float planeDist = (nmax3[bestAxis] - nmin3[bestAxis]) / (binCount * 0.9999f);
				const float rPlaneDist = 1.0f / planeDist, nodeMin = nmin3[bestAxis];
				for (uint32_t i = 0; i < node->triCount; i++)
				{
					const uint32_t fragIdx = primIdx[src++];
					const uint32_t bin1 = (uint32_t)fmax_( (fragment[fragIdx].bmin[bestAxis] - nodeMin) * rPlaneDist, 0.0f );
					const uint32_t bin2 = (uint32_t)fmax_( (fragment[fragIdx].bmax[bestAxis] - nodeMin) * rPlaneDist, 0.0f );
					if (bin2 <= bestPos) idxTmp[A++] = fragIdx; else if (bin1 > bestPos) idxTmp[--B] = fragIdx; else
					{
						/* unsplitting :2895-2926 */
						if (bestNR > 1)
						{
							float uLMin[3], uLMax[3], dl[3], dr[3];
							for (int k = 0; k < 3; k++) uLMin[k] = fmin_( bestLMin[k], fragment[fragIdx].bmin[k] ), uLMax[k] = fmax_( bestLMax[k], fragment[fragIdx].bmax[k] );
							for (int k = 0; k < 3; k++) dl[k] = uLMax[k] - uLMin[k], dr[k] = bestRMax[k] - bestRMin[k];
							const float AL = half_area3( dl ), AR = half_area3( dr );
							const float CunsplitLeft = split_cost( h, rSAV, AL, bestNL, AR, bestNR - 1 );
							if (CunsplitLeft <= splitCost)
							{
								bestNR--, splitCost = CunsplitLeft, idxTmp[A++] = fragIdx;
								for (int k = 0; k < 3; k++) bestLMin[k] = uLMin[k], bestLMax[k] = uLMax[k];
								continue;
							}
						}
						if (bestNL > 1)
						{
							float uRMin[3], uRMax[3], dl[3], dr[3];
							for (int k = 0; k < 3; k++) uRMin[k] = fmin_( bestRMin[k], fragment[fragIdx].bmin[k] ), uRMax[k] = fmax_( bestRMax[k], fragment[fragIdx].bmax[k] );
							for (int k = 0; k < 3; k++) dl[k] = bestLMax[k] - bestLMin[k], dr[k] = uRMax[k] - uRMin[k];
							const float AL = half_area3( dl ), AR = half_area3( dr );
							const float CunsplitRight = split_cost( h, rSAV, AL, bestNL - 1, AR, bestNR );
							if (CunsplitRight <= splitCost)
							{
								bestNL--, splitCost = CunsplitRight, idxTmp[--B] = fragIdx;
								for (int k = 0; k < 3; k++) bestRMin[k] = uRMin[k], bestRMax[k] = uRMax[k];
								continue;
							}
						}
						frag_t part1, part2;
						int leftOK = 0, rightOK = 0;
						const float splitPos = bestLMax[bestAxis];
						split_frag( h, &fragment[fragIdx], &part1, &part2, minDim, bestAxis, splitPos, &leftOK, &rightOK );
						if (leftOK && rightOK)
						{
							const uint32_t newFragIdx = h->nextFrag++;
							fragment[fragIdx] = part1, idxTmp[A++] = fragIdx, fragment[newFragIdx] = part2, idxTmp[--B] = newFragIdx;
						}
						else if (leftOK) idxTmp[A++] = fragIdx; else idxTmp[--B] = fragIdx;
					}
				}
				for (int k = 0; k < 3; k++) bestLMin[k] = bestRMin[k] = BVH_FAR, bestLMax[k] = bestRMax[k] = -BVH_FAR;
				for (uint32_t i = sliceStart; i < A; i++) for (int k = 0; k < 3; k++)
					bestLMin[k] = fmin_( bestLMin[k], fragment[idxTmp[i]].bmin[k] ), bestLMax[k] = fmax_( bestLMax[k], fragment[idxTmp[i]].bmax[k] );
				for (uint32_t i = B; i < sliceEnd; i++) for (int k = 0; k < 3; k++)
					bestRMin[k] = fmin_( bestRMin[k], fragment[idxTmp[i]].bmin[k] ), bestRMax[k] = fmax_( bestRMax[k], fragment[idxTmp[i]].bmax[k] );
			}
			else
			{
				const float rpd = rpd3[bestAxis], nmin = nmin3[bestAxis];
				for (uint32_t i = 0; i < node->triCount; i++)
				{
					const uint32_t fr = primIdx[src + i];
					int bi = (int)(fmaf( fragment[fr].bmin[bestAxis] + fragment[fr].bmax[bestAxis], 0.5f, -nmin ) * rpd);
					bi = clampi_( bi, 0, (int)binCount - 1 );
					if (bi <= (int)bestPos) idxTmp[A++] = fr; else idxTmp[--B] = fr;
				}
			}
			memcpy( primIdx + sliceStart, idxTmp + sliceStart, (size_t)(sliceEnd - sliceStart) * 4 );
			const uint32_t leftCount = A - sliceStart, rightCount = sliceEnd - B;
			if (leftCount == 0 || rightCount == 0)
			{
				orc_hq_failed_splits++;
				if (node->leftFirst != (leftCount ? sliceStart : B)) orc_hq_failed_splits += 1 << 16;
				if (node->triCount > orc_hq_failed_max) orc_hq_failed_max = node->triCount;
				for (uint32_t i = 0; i < node->triCount; i++) primIdx[node->leftFirst + i] = fragment[primIdx[node->leftFirst + i]].primIdx;
				node->minx = fmin_( bestLMin[0], bestRMin[0] ), node->miny = fmin_( bestLMin[1], bestRMin[1] ), node->minz = fmin_( bestLMin[2], bestRMin[2] );
				node->maxx = fmax_( bestLMax[0], bestRMax[0] ), node->maxy = fmax_( bestLMax[1], bestRMax[1] ), node->maxz = fmax_( bestLMax[2], bestRMax[2] );
				break;
			}
			const uint32_t lc = h->newNodePtr, rc = lc + 1;
			h->newNodePtr += 2;
			h->nodes[lc].minx = bestLMin[0], h->nodes[lc].miny = bestLMin[1], h->nodes[lc].minz = bestLMin[2];
			h->nodes[lc].maxx = bestLMax[0], h->nodes[lc].maxy = bestLMax[1], h->nodes[lc].maxz = bestLMax[2];
			h->nodes[lc].leftFirst = sliceStart, h->nodes[lc].triCount = leftCount;
			h->nodes[rc].minx = bestRMin[0], h->nodes[rc].miny = bestRMin[1], h->nodes[rc].minz = bestRMin[2];
			h->nodes[rc].maxx = bestRMax[0], h->nodes[rc].maxy = bestRMax[1], h->nodes[rc].maxz = bestRMax[2];
			h->nodes[rc].leftFirst = B, h->nodes[rc].triCount = rightCount;
			node->leftFirst = lc, node->triCount = 0;
			localTask[localTasks].node = rc, localTask[localTasks].depth = depth;
			localTask[localTasks].sliceStart = (A + B) >> 1, localTask[localTasks++].sliceEnd = sliceEnd;
			nodeIdx = lc, sliceEnd = (A + B) >> 1;
		}
		if (localTasks == 0) break;
		nodeIdx = localTask[--localTasks].node, depth = localTask[localTasks].depth;
		sliceStart = localTask[localTasks].sliceStart, sliceEnd = localTask[localTasks].sliceEnd;
	}
	free( localTask );
}

/* BVH::BuildHQ( verts ) :2641 + Compact :3733.  nodes: room for 3*primCount, primIdx: room for primCount + primCount/2.
 * Returns usedNodes; *idxCount receives primCount + primCount/2 (Compact does not shrink idxCount), *usedIdx the number of
 * index entries the leaves actually reference (the reference leaves the rest of its new array uninitialised). */
uint32_t orc_build_hq( const float* verts, uint32_t primCount, orc_node* nodes, uint32_t* primIdx, uint32_t* idxCount, uint32_t* usedIdx, float c_trav, float c_int )
{
	const uint32_t slack = primCount >> 1;
	hq_t h;
	h.verts = verts, h.c_trav = c_trav, h.c_int = c_int;
	h.fragment = (frag_t*)malloc( (size_t)(primCount + slack) * sizeof( frag_t ) );
	h.primIdx = (uint32_t*)calloc( (size_t)(primCount + slack), 4 );
	h.nodes = (orc_node*)calloc( (size_t)primCount * 3 + 2, sizeof( orc_node ) );
	uint32_t* idxTmp = (uint32_t*)calloc( (size_t)(primCount + slack), 4 );
	orc_node* root = &h.nodes[0];
	root->leftFirst = 0, root->triCount = primCount;
	float rmin[3] = { BVH_FAR, BVH_FAR, BVH_FAR }, rmax[3] = { -BVH_FAR, -BVH_FAR, -BVH_FAR };
	for (uint32_t i = 0; i < primCount; i++) /* PrepareHQBuild :2677-2686 */
	{
		const float* v0 = verts + (size_t)i * 12, * v1 = v0 + 4, * v2 = v0 + 8;
		for (int a = 0; a < 3; a++)
		{
			h.fragment[i].bmin[a] = fmin_( v0[a], fmin_( v1[a], v2[a] ) ), h.fragment[i].bmax[a] = fmax_( v0[a], fmax_( v1[a], v2[a] ) );
			rmin[a] = fmin_( rmin[a], h.fragment[i].bmin[a] ), rmax[a] = fmax_( rmax[a], h.fragment[i].bmax[a] );
		}
		h.fragment[i].primIdx = i, h.fragment[i].clipped = 0, h.primIdx[i] = i;
	}
	root->minx = rmin[0], root->miny = rmin[1], root->minz = rmin[2], root->maxx = rmax[0], root->maxy = rmax[1], root->maxz = rmax[2];
	h.newNodePtr = 2, h.nextFrag = primCount;
	build_hq_task( &h, 0, 0, primCount + slack, idxTmp );
	/* Compact :3733-3770 */
	uint32_t used = h.newNodePtr;
	if (h.nodes[0].triCount == 0)
	{
		orc_node* temp = nodes;
		uint32_t* idx = primIdx;
		memcpy( temp, h.nodes, 2 * sizeof( orc_node ) );
		uint32_t newNodePtr = 2, newIdxPtr = 0, nodeIdx = 0, stack[128], stackPtr = 0;
		while (1)
		{
			orc_node* node = &temp[nodeIdx];
			if (node->triCount > 0)
			{
				const uint32_t leafStart = newIdxPtr;
				for (uint32_t i = 0; i < node->triCount; i++) idx[newIdxPtr++] = h.primIdx[node->leftFirst + i];
				node->leftFirst = leafStart;
				if (!stackPtr) break;
				nodeIdx = stack[--stackPtr];
			}
			else
			{
				temp[newNodePtr] = h.nodes[node->leftFirst], temp[newNodePtr + 1] = h.nodes[node->leftFirst + 1];
				const uint32_t todo1 = newNodePtr, todo2 = newNodePtr + 1;
				node->leftFirst = newNodePtr, newNodePtr += 2;
				nodeIdx = todo1, stack[stackPtr++] = todo2;
			}
		}
		used = newNodePtr;
		*usedIdx = newIdxPtr;
		for (uint32_t i = newIdxPtr; i < primCount + slack; i++) idx[i] = 0;
	}
	else
	{
		memcpy( nodes, h.nodes, (size_t)used * sizeof( orc_node ) );
		memcpy( primIdx, h.primIdx, (size_t)(primCount + slack) * 4 );
		*usedIdx = primCount;
	}
	*idxCount = primCount + slack;
	free( h.fragment ), free( h.primIdx ), free( h.nodes ), free( idxTmp );
	return used;
}

/* test hooks: the two geometric helpers on their own (pinned against BVH::ClipFrag / BVH::SplitFrag) */
int orc_clip_frag( const float* verts, const void* orig, void* out, const float* bmin, const float* bmax, const float* minDim, uint32_t axis )
{
	hq_t h; memset( &h, 0, sizeof( h ) ); h.verts = verts;
	return clip_frag( &h, (const frag_t*)orig, (frag_t*)out, bmin, bmax, minDim, axis );
}
void orc_split_frag( const float* verts, const void* orig, void* left, void* right, const float* minDim, uint32_t axis, float pos, int* lok, int* rok )
{
	hq_t h; memset( &h, 0, sizeof( h ) ); h.verts = verts;
	split_frag( &h, (const frag_t*)orig, (frag_t*)left, (frag_t*)right, minDim, axis, pos, lok, rok );
}
