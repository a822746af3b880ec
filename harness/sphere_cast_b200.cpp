// harness/sphere_cast_b200.cpp - sphere casts through the C++ shim: SphereCast and SphereCastOccluded over a procedural scene.  Each
// first contact must lie between the double-precision first contacts at r + delta and r - delta over every triangle (the distance along
// the sweep is convex, so a ternary search and a bisection find them), a miss must have no contact at r - delta, the contact point must lie
// within r + delta of the centre at t, and each blocked bit must say whether SphereCast found a contact.  Prints "0 failures" on success.
#include "tinybvh_b200.hpp"
#include <cmath>
#include <cstdio>
#include <vector>

struct V4 { float x, y, z, w; };
struct Q8 { float cx, cy, cz, r, dx, dy, dz, tmax; };
struct Rec { float t, u, v; uint32_t prim; };

// distance from p to triangle (a, b, c) in double precision: the plane point when inside, else the nearest edge point
static double tri_dist( const double* p, const double* a, const double* b, const double* c )
{
	auto seg = [&]( const double* s, const double* t )
	{
		double d[3], dd = 0, w = 0;
		for (int k = 0; k < 3; k++) d[k] = t[k] - s[k], dd += d[k] * d[k], w += (p[k] - s[k]) * d[k];
		w = dd > 0 ? std::fmin( std::fmax( w / dd, 0.0 ), 1.0 ) : 0.0;
		double r = 0;
		for (int k = 0; k < 3; k++) { const double e = p[k] - (s[k] + w * d[k]); r += e * e; }
		return std::sqrt( r );
	};
	double best = std::fmin( std::fmin( seg( a, b ), seg( a, c ) ), seg( b, c ) );
	double e1[3], e2[3], n[3];
	for (int k = 0; k < 3; k++) e1[k] = b[k] - a[k], e2[k] = c[k] - a[k];
	n[0] = e1[1] * e2[2] - e1[2] * e2[1], n[1] = e1[2] * e2[0] - e1[0] * e2[2], n[2] = e1[0] * e2[1] - e1[1] * e2[0];
	const double nn = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
	if (nn > 0)
	{
		const double t = ((p[0] - a[0]) * n[0] + (p[1] - a[1]) * n[1] + (p[2] - a[2]) * n[2]) / nn;
		double q[3];
		for (int k = 0; k < 3; k++) q[k] = p[k] - t * n[k];
		bool inside = true;
		const double* v[3] = { a, b, c };
		for (int e = 0; e < 3; e++)
		{
			const double* s = v[e], * f = v[(e + 1) % 3];
			const double x[3] = { f[0] - s[0], f[1] - s[1], f[2] - s[2] }, y[3] = { q[0] - s[0], q[1] - s[1], q[2] - s[2] };
			const double cr[3] = { x[1] * y[2] - x[2] * y[1], x[2] * y[0] - x[0] * y[2], x[0] * y[1] - x[1] * y[0] };
			inside &= cr[0] * n[0] + cr[1] * n[1] + cr[2] * n[2] >= 0;
		}
		if (inside) best = std::fmin( best, std::fabs( t ) * std::sqrt( nn ) );
	}
	return best;
}

// the first t in [0, tmax] at which the centre comes within rho of the triangle, or -1
static double first_contact( const Q8& q, const double* a, const double* b, const double* c, const double rho )
{
	auto dist = [&]( const double t ) { const double p[3] = { q.cx + t * q.dx, q.cy + t * q.dy, q.cz + t * q.dz }; return tri_dist( p, a, b, c ); };
	if (dist( 0 ) <= rho) return 0;
	double lo = 0, hi = q.tmax;
	for (int i = 0; i < 100; i++) { const double x = lo + (hi - lo) / 3, y = hi - (hi - lo) / 3; if (dist( x ) <= dist( y )) hi = y; else lo = x; }
	double tm = (lo + hi) / 2;
	if (dist( q.tmax ) <= dist( tm )) tm = q.tmax;
	if (dist( tm ) > rho) return -1;
	lo = 0, hi = tm;
	for (int i = 0; i < 80; i++) { const double m = (lo + hi) / 2; if (dist( m ) <= rho) hi = m; else lo = m; }
	return hi;
}

int main()
{
	const uint32_t n = 1000, nq = 600;
	std::vector<V4> soup( n * 3 );
	std::vector<Q8> q( nq );
	uint32_t seed = 4242;
	auto rnd = [&]() { seed = seed * 1664525u + 1013904223u; return (seed >> 8) * (1.0f / 16777216.0f); };
	for (uint32_t i = 0; i < n; i++)
	{
		const float cx = rnd() * 100, cy = rnd() * 20, cz = rnd() * 100;
		for (int k = 0; k < 3; k++) soup[i * 3 + k] = V4{ cx + rnd() * 3, cy + rnd() * 3, cz + rnd() * 3, 0 };
	}
	for (uint32_t i = 0; i < nq; i++)
	{
		const float cx = rnd() * 120 - 10, cy = rnd() * 40 - 10, cz = rnd() * 120 - 10;
		const float tx = rnd() * 100, ty = rnd() * 20, tz = rnd() * 100;
		q[i] = Q8{ cx, cy, cz, i % 5 == 0 ? 0.0f : rnd() * 2, tx - cx, ty - cy, tz - cz, i % 3 == 0 ? 1.0f : 0.5f };
	}
	tinybvh_b200::BVH bvh;
	bvh.Build( soup.data(), n );
	std::vector<Rec> rec( nq );
	bvh.SphereCast( q.data(), nq, rec.data() );
	std::vector<uint32_t> bits( (nq + 31) / 32 );
	bvh.SphereCastOccluded( q.data(), nq, bits.data() );
	int fails = 0, hits = 0;
	const double delta = 2e-6 * 150; // of the scene's largest relative coordinate
	for (uint32_t i = 0; i < nq; i++)
	{
		double lo = INFINITY, hi = INFINITY;
		for (uint32_t t = 0; t < n; t++)
		{
			const double a[3] = { soup[t * 3].x, soup[t * 3].y, soup[t * 3].z }, b[3] = { soup[t * 3 + 1].x, soup[t * 3 + 1].y, soup[t * 3 + 1].z },
				c[3] = { soup[t * 3 + 2].x, soup[t * 3 + 2].y, soup[t * 3 + 2].z };
			const double l = first_contact( q[i], a, b, c, q[i].r + delta ), h = q[i].r >= delta ? first_contact( q[i], a, b, c, q[i].r - delta ) : -1;
			if (l >= 0) lo = std::fmin( lo, l );
			if (h >= 0) hi = std::fmin( hi, h );
		}
		const bool found = rec[i].prim != 0xffffffffu;
		hits += found;
		const double slack = 4 * std::ldexp( std::fabs( (double)rec[i].t ), -23 ) + 1e-12;
		if (found && !(rec[i].t >= lo - slack && rec[i].t <= std::fmin( hi, (double)q[i].tmax ) + slack))
		{ if (fails < 5) printf( "query %u: t %.9g outside [%.9g, %.9g]\n", i, rec[i].t, lo, hi ); fails++; }
		if (!found && hi < INFINITY) { if (fails < 5) printf( "query %u: missed a contact at %.9g\n", i, hi ); fails++; }
		if (found)
		{
			const V4* tri = soup.data() + rec[i].prim * 3;
			double d = 0;
			for (int k = 0; k < 3; k++)
			{
				const double c = (&q[i].cx)[k] + (double)rec[i].t * (&q[i].dx)[k];
				const double p = (&tri[0].x)[k] + rec[i].u * ((double)(&tri[1].x)[k] - (&tri[0].x)[k]) + rec[i].v * ((double)(&tri[2].x)[k] - (&tri[0].x)[k]);
				d += (c - p) * (c - p);
			}
			if (std::sqrt( d ) > q[i].r + delta) { if (fails < 5) printf( "query %u: contact point %.9g from the centre, r %.9g\n", i, std::sqrt( d ), q[i].r ); fails++; }
		}
		const bool bit = (bits[i >> 5] >> (i & 31)) & 1;
		if (bit != found) { if (fails < 5) printf( "query %u: blocked bit %d, SphereCast found %d\n", i, bit, found ); fails++; }
	}
	if (hits < (int)nq / 10 || hits == (int)nq) { printf( "%d of %u sweeps touch: the scene does not test both outcomes\n", hits, nq ); fails++; }
	printf( "%d failures\n", fails );
	return fails ? 1 : 0;
}
