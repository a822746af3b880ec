// harness/tlas_frame_b200.cpp - the frame of an animated two-level scene through the shim: the vertices of every BLAS move, RefitBatch
// refits them in one call, every instance gets a new transform, and the TLAS is rebuilt by BuildUpdated (BLASInstance::Update on the
// device, one call) - checked against a twin TLAS that the existing Build (a host Update per instance, then the build) makes from the
// same records: instance records, TLAS nodes, primIdx and the hits of a ray batch must be identical.  No reference header.
//   g++ -O2 -std=c++17 -Iinclude harness/tlas_frame_b200.cpp -Ltinybvh_b200 -ltinybvh_b200 -Wl,-rpath,$PWD/tinybvh_b200 -o tlas_frame_b200
//   tlas_frame_b200 [--time] [instances] [blasses]     --time: one warm-up frame first, then the wall time of both paths per frame
//   (each call ends in a device synchronise; the order of the two paths alternates from frame to frame)
#include "tinybvh_b200.hpp"
#include <chrono>
#include <vector>

struct Vec4 { float x, y, z, w; };
struct Inst { float transform[16], invTransform[16], aabbMin[3]; uint32_t blasIdx; float aabbMax[3]; uint32_t mask, dummy[8]; }; // tinybvh::BLASInstance :1443
static uint32_t seed = 0x2468ace1;
static float rnd() { seed ^= seed << 13, seed ^= seed >> 17, seed ^= seed << 5; return seed * 2.3283064365387e-10f; }
static double now_ms() { return std::chrono::duration<double, std::milli>( std::chrono::steady_clock::now().time_since_epoch() ).count(); }

// rotation about y and z, a non-uniform scale and a translation, row-major as bvhmat4
static void new_transform( Inst& in, const float spread )
{
	const float a = rnd() * 6.28f, b = rnd() * 6.28f, ca = cosf( a ), sa = sinf( a ), cb = cosf( b ), sb = sinf( b );
	const float s[3] = { 0.5f + rnd(), 0.5f + rnd(), 0.5f + rnd() };
	const float R[9] = { ca * cb, -sb, sa * cb, ca * sb, cb, sa * sb, -sa, 0, ca };
	for (int r = 0; r < 3; r++)
	{
		for (int c = 0; c < 3; c++) in.transform[r * 4 + c] = R[r * 3 + c] * s[c];
		in.transform[r * 4 + 3] = (rnd() - 0.5f) * spread;
	}
	in.transform[12] = in.transform[13] = in.transform[14] = 0, in.transform[15] = 1;
}

int main( int argc, char** argv )
{
	bool timed = false;
	uint32_t N = 4000, M = 6, arg = 0;
	for (int i = 1; i < argc; i++)
	{
		if (!strcmp( argv[i], "--time" )) timed = true;
		else if (arg++ == 0) N = (uint32_t)atoi( argv[i] );
		else M = (uint32_t)atoi( argv[i] );
	}
	if (N == 0 || M == 0) { fprintf( stderr, "usage: tlas_frame_b200 [--time] [instances] [blasses]\n" ); return 2; }
	std::vector<std::vector<Vec4>> verts( M );
	std::vector<tinybvh_b200::BVH*> blas( M );
	std::vector<tinybvh_b200::BVHBase*> base( M );
	for (uint32_t m = 0; m < M; m++)
	{
		const uint32_t tris = 300 + (uint32_t)(rnd() * 2500);
		for (uint32_t i = 0; i < tris; i++)
		{
			const float x = rnd() * 2 - 1, y = rnd() * 2 - 1, z = rnd() * 2 - 1;
			for (int v = 0; v < 3; v++) verts[m].push_back( { x + rnd() * 0.2f, y + rnd() * 0.2f, z + rnd() * 0.2f, 0 } );
		}
		blas[m] = new tinybvh_b200::BVH();
		blas[m]->Build( verts[m].data(), tris );
		base[m] = blas[m];
	}
	const float spread = 4.0f * cbrtf( (float)N );
	std::vector<Inst> inst( N ), twin( N );
	memset( inst.data(), 0, sizeof( Inst ) * N );
	for (uint32_t i = 0; i < N; i++)
	{
		inst[i].blasIdx = (uint32_t)(rnd() * M) % M, inst[i].mask = i % 5 ? 0x3 : 0x2;
		for (int k = 0; k < 8; k++) inst[i].dummy[k] = 0xfeed0000u + i; // bytes no Update may touch
	}
	const uint32_t R = 16384;
	std::vector<tinybvh_b200::Ray> ra( R ), rb( R );
	tinybvh_b200::BVH tlas, ref;
	int differ = 0;
	for (int frame = timed ? -1 : 0; frame < 2; frame++)
	{
		for (uint32_t m = 0; m < M; m++) for (Vec4& v : verts[m]) v.x += (rnd() - 0.5f) * 0.1f, v.y += rnd() * 0.05f;
		tinybvh_b200::RefitBatch( blas.data(), M );
		for (uint32_t i = 0; i < N; i++) new_transform( inst[i], spread );
		twin = inst;
		double t_new = 0, t_old = 0;
		uint64_t l_new = 0, l_old = 0;
		for (int pass = 0; pass < 2; pass++)
		{
			const bool fresh = (pass == 0) == ((frame & 1) == 0); // which path goes first alternates
			const double t0 = now_ms();
			const uint64_t l0 = tbvh_launch_count();
			if (fresh) tlas.BuildUpdated( inst.data(), N, base.data(), M ), tlas.Sync(), t_new = now_ms() - t0, l_new = tbvh_launch_count() - l0;
			else ref.Build( twin.data(), N, base.data(), M ), ref.Sync(), t_old = now_ms() - t0, l_old = tbvh_launch_count() - l0;
		}
		bool same = memcmp( inst.data(), twin.data(), sizeof( Inst ) * N ) == 0;
		for (uint32_t i = 0; i < N && same; i++) for (int k = 0; k < 8; k++) same = same && inst[i].dummy[k] == 0xfeed0000u + i;
		const tbvh_info a = tlas.Info(), b = ref.Info();
		same = same && a.used_nodes == b.used_nodes && a.idx_count == b.idx_count && a.max_depth == b.max_depth && a.prim_count == b.prim_count && a.layouts == b.layouts;
		same = same && !memcmp( a.aabb_min, b.aabb_min, 12 ) && !memcmp( a.aabb_max, b.aabb_max, 12 );
		if (same)
		{
			std::vector<char> na( (size_t)a.used_nodes * 32 ), nb( (size_t)b.used_nodes * 32 );
			std::vector<uint32_t> ia( a.idx_count ), ib( b.idx_count );
			tlas.Download( na.data(), ia.data() ), ref.Download( nb.data(), ib.data() );
			same = na == nb && ia == ib;
		}
		for (uint32_t i = 0; i < R; i++)
		{
			const float O[3] = { (rnd() - 0.5f) * spread, (rnd() - 0.5f) * spread, -spread }, D[3] = { rnd() - 0.5f, rnd() - 0.5f, 1 };
			ra[i] = tinybvh_b200::Ray( O, D ), ra[i].mask = i & 1 ? 0x1 : 0x2, rb[i] = ra[i];
		}
		tlas.Intersect( ra.data(), R ), ref.Intersect( rb.data(), R );
		uint32_t hits = 0;
		for (uint32_t i = 0; i < R; i++) same = same && !memcmp( (char*)&ra[i] + 44, (char*)&rb[i] + 44, 20 ), hits += ra[i].t < 1e30f;
		if (frame >= 0) differ += !same;
		if (timed) printf( "tlas_frame_b200 frame %i: %u instances, %u blasses; Update loop + Build %.3f ms wall, %llu launches, build_ms %.3f; BuildUpdated %.3f ms wall, %llu launches, build_ms %.3f; %u of %u rays hit; %s\n",
			frame, N, M, t_old, (unsigned long long)l_old, b.build_ms, t_new, (unsigned long long)l_new, a.build_ms, hits, R, same ? "identical" : "DIFFERENT" );
	}
	printf( "tlas_frame_b200: %u instances over %u blasses, 2 frames; %i frames differ from Update + Build\n", N, M, differ );
	for (uint32_t m = 0; m < M; m++) delete blas[m];
	return differ == 0 ? 0 : 1;
}
