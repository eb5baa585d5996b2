// nudge_b200 — scene queries against the current colliders: ray casts (nb_raycast, DESIGN.md section 8.14), overlap queries (nb_overlap,
// section 8.15) and shape casts (nb_shapecast, section 8.16; include/nudge_b200.h).  All three build with nb_collide's front end
// (launch_front_end, nb_api.cu) on the FrontEnd of the queries' own scratch (QueryScratch): world transforms and AABBs (k_collider_world),
// Morton codes and their sort, Morton-ordered leaves and the grid table (k_grid_build).  k_overlap walks it around its query; k_raycast and
// k_shapecast walk it along their path with one swept walk (swept_walk).  k_overlap's hit keys are sorted and written out by k_overlap_write.
// Included at the end of nb_api.cu.
#pragma once

// ---------------- the per-collider arithmetic the header states ----------------
// The slab test of a ray already in the box's frame (origin lo, direction ld, half extents hh): the entry t and the axis that set it (-1
// when none did) with its side s; slab_normal(axis, s) is the local normal.
NB_DEV bool sweep_slab(f3 lo, f3 ld, f3 hh, float max_t, float& t, int& axis, float& s) {
	const float los[3] = { lo.x, lo.y, lo.z }, lds[3] = { ld.x, ld.y, ld.z }, h[3] = { hh.x, hh.y, hh.z };
	float enter = 0.0f, exit = max_t;
	s = 0.0f; axis = -1;
	#pragma unroll
	for (int k = 0; k < 3; ++k) {
		if (lds[k] == 0.0f) {
			if (los[k] < -h[k] || los[k] > h[k]) return false;
		}
		else {
			const float t1 = (-h[k] - los[k]) / lds[k], t2 = (h[k] - los[k]) / lds[k];
			const bool lt = t1 < t2;
			const float near = lt ? t1 : t2, far = lt ? t2 : t1;
			if (near > enter) { enter = near; axis = k; s = lt ? -1.0f : 1.0f; }
			if (far < exit) exit = far;
			if (enter > exit) return false;
		}
	}
	t = enter;
	return true;
}
NB_DEV f3 slab_normal(int axis, float s) { return axis == 0 ? mk3(s, 0.0f, 0.0f) : axis == 1 ? mk3(0.0f, s, 0.0f) : mk3(0.0f, 0.0f, s); }
NB_DEV bool ray_sphere(f3 o, f3 d, float max_t, const xform& w, float r, float& t, f3& n) {
	const f3 c = mk3(w.p.x, w.p.y, w.p.z), m = sub3(o, c);
	const float a = dot3(d, d), b = dot3(m, d), cc = dot3(m, m) - r * r;
	if (cc <= 0.0f) { t = 0.0f; n = mk3(0.0f, 0.0f, 0.0f); return true; }
	const float disc = b * b - a * cc;
	if (disc < 0.0f) return false;
	t = (-b - sqrtf(disc)) / a;
	if (!(t >= 0.0f && t <= max_t)) return false;   // a NaN t (overflowed terms) is a miss too
	if (t == 0.0f) t = 0.0f;   // -0 -> +0: the hit key orders t by its bits
	const float inv = 1.0f / r;
	n = mul3(sub3(add3(o, mul3(t, d)), c), inv);
	return true;
}
NB_DEV bool is_zero3(f3 v) { return v.x == 0.0f && v.y == 0.0f && v.z == 0.0f; }
NB_DEV bool finite3(f3 v) { return isfinite(v.x) && isfinite(v.y) && isfinite(v.z); }
NB_DEV quat qconj(quat q) { q.v = mk3(-q.v.x, -q.v.y, -q.v.z); return q; }

// The colliders the queries test and the grid the front end built over them.
struct QueryScene {
	u32 K, nboxes;
	const nb_transform* world_xf; const float4* aabb_max; const u32* col_body; const u32* col_tag;
	const nb_box_collider* box_data; const nb_sphere_collider* sph_data; const uint8_t* sensor;
	const u32* order; const uint8_t* smallf; const u64* table_keys; const u64* table_vals; u32 table_mask; const u32* large_list;
};
// Whether a query of (mask, ignore_body, sensors) may test collider i: its category (k_collider_world's filter word) meets the mask, its
// body is not the ignored one, and it is no sensor unless the query asks for sensors.
NB_DEV bool query_may_test(const QueryScene& S, u32 i, u32 mask, u32 ignore, bool sensors) {
	const u32 category = asu(reinterpret_cast<const float*>(S.aabb_max)[4 * (size_t)i + 3]) & 0xffffu;
	return (category & mask) && __ldg(S.col_body + i) != ignore && !(S.sensor && !sensors && __ldg(S.sensor + i));
}
// Tests collider i and keeps the lane's best (t bits << 32 | i) and the normal that goes with it.
NB_DEV void ray_test(const QueryScene& S, u32 i, f3 o, f3 d, float max_t, u32 mask, u32 ignore, bool sensors, u64& best, f3& bn) {
	if (!query_may_test(S, i, mask, ignore, sensors)) return;
	const xform w = ld_xform(S.world_xf, i);
	float t;
	f3 n = mk3(0.0f, 0.0f, 0.0f);
	bool hit;
	if (i < S.nboxes) {
		const float4 sz = reinterpret_cast<const float4*>(S.box_data)[i];
		const quat q = mkq(w.q), qc = qconj(q);
		int axis; float s;
		hit = sweep_slab(qrot(qc, sub3(o, mk3(w.p.x, w.p.y, w.p.z))), qrot(qc, d), mk3(sz.x, sz.y, sz.z), max_t, t, axis, s);
		if (hit && axis >= 0) n = qrot(q, slab_normal(axis, s));
	}
	else hit = ray_sphere(o, d, max_t, w, S.sph_data[i - S.nboxes].radius, t, n);
	if (!hit) return;
	const u64 key = (u64)asu(t) << 32 | i;
	if (key < best) { best = key; bn = n; }
}
NB_DEV u64 warp_min_u64(u64 v) {
	#pragma unroll
	for (int s = 16; s; s >>= 1) { const u64 o = __shfl_xor_sync(0xffffffffu, v, s); v = o < v ? o : v; }
	return v;
}

// The last build's grid in quantised units: the Morton frame f (scale s = f.L[0]), msmax = the largest |offset| of the frame, the level
// j, the cell edge W = 2^j and ncell cells per axis.  ok: the scale is positive, finite and the same on every axis (otherwise a query tests
// every collider).
struct QueryGrid { MortonFrame f; float s, msmax, W; u32 j; int ncell; bool ok; };
NB_DEV QueryGrid query_grid(const u32* counts) {
	QueryGrid G;
	G.f = morton_frame(counts);
	G.s = G.f.L[0];
	G.msmax = fmaxf(fabsf(G.f.ms[0]), fmaxf(fabsf(G.f.ms[1]), fabsf(G.f.ms[2])));
	G.j = counts[CNT_GRID_LEVEL];
	G.W = (float)(1u << G.j);
	G.ncell = 1 << (16 - G.j);
	G.ok = G.s > 0.0f && isfinite(G.s) && G.f.L[1] == G.s && G.f.L[2] == G.s && G.f.L[3] == G.s;
	return G;
}

// The level-j cells that hold the min corner of every small collider touching the quantised box [lo, hi] widened by mu:
// [floor((lo - mu - W) / W), floor((hi + mu) / W)] per axis (a small collider fits a cell and is binned by its min corner), clamped to the
// grid's ncell cells per axis.  c0 / nc = the first cell and the count per axis; returns false when the range is empty.
NB_DEV bool cell_range(const QueryGrid& G, const float lo[3], const float hi[3], float mu, int c0[3], int nc[3]) {
	const float W = G.W;
	const int ncell = G.ncell;
	bool any = true;
	#pragma unroll
	for (int a = 0; a < 3; ++a) {
		const float l0 = lo[a] - mu - W, h0 = hi[a] + mu;
		const int l = (int)fminf(fmaxf(floorf(l0 / W), 0.0f), (float)ncell), h = (int)fmaxf(fminf(floorf(h0 / W), (float)(ncell - 1)), -1.0f);
		c0[a] = l; nc[a] = h - l + 1;
		if (h < l) any = false;
	}
	return any;
}
// The number of cells of a range cell_range found not empty.
NB_DEV float cell_count(const int nc[3]) { return (float)nc[0] * (float)nc[1] * (float)nc[2]; }

// Looks up the level-j cells c0 + [0, nc) per axis (nc >= 1) in the grid's hash table, flattens their ranges of Morton positions with a
// warp scan and deals the positions round-robin to the lanes, as k_grid_pairs deals its candidates: visit(i) runs once for every collider
// i binned in those cells, on one lane, skipping the large ones (the large list holds them) when skip_large.  Warp-uniform arguments; the
// whole warp calls it.
template<class F>
NB_DEV void grid_cells_visit(const QueryScene& S, const QueryGrid& G, const int c0[3], const int nc[3], u32 lane, bool skip_large, F visit) {
	const u32 j = G.j;
	const u32 ncells = (u32)(nc[0] * nc[1] * nc[2]);
	for (u32 cb = 0; cb < ncells; cb += 32) {
		const u32 ci = cb + lane;
		u32 qb = 0, len = 0;
		if (ci < ncells) {
			const u32 cx = (u32)c0[0] + ci % (u32)nc[0], cy = (u32)c0[1] + (ci / (u32)nc[0]) % (u32)nc[1], cz = (u32)c0[2] + ci / (u32)(nc[0] * nc[1]);
			const u64 prefix = morton48_of(cx << j, cy << j, cz << j) >> (3 * j);
			u32 slot = grid_hash(prefix, S.table_mask);
			u64 key;
			while ((key = S.table_keys[slot]) != prefix && key != NB_GRID_EMPTY) slot = (slot + 1) & S.table_mask;
			if (key != NB_GRID_EMPTY) { const u64 range = S.table_vals[slot]; qb = (u32)range; len = (u32)(range >> 32) - qb; }
		}
		const u32 incl = warp_incl_scan(len), off = incl - len, total = __shfl_sync(0xffffffffu, incl, 31);
		for (u32 t0 = 0; t0 < total; t0 += 32) {
			const u32 t = t0 + lane;
			u32 c = 0;   // the cell of candidate t: the last lane whose offset is <= t
			#pragma unroll
			for (int st = 16; st; st >>= 1) {
				const u32 probe = __shfl_sync(0xffffffffu, off, (c + st) & 31);
				if (c + st < 32 && probe <= t) c += st;
			}
			const u32 q = __shfl_sync(0xffffffffu, qb, c) + (t - __shfl_sync(0xffffffffu, off, c));
			if (t < total && (!skip_large || S.smallf[q])) visit(S.order[q]);
		}
	}
}

// Segments per ray or cast beyond which the swept walk gives up on the grid and tests every collider.
#define NB_RAY_MAX_SEGMENTS 262144u
// Cells per query, or per segment of a shape cast's walk, beyond which a walk gives up on the grid and tests every collider.
#define NB_OVERLAP_MAX_CELLS 4096u

// One warp's walk along the path o + t d, t in [0, max_t], of a ray or, with Cast, of a shape's centre (ext = its world extent: r for a
// sphere; for a box the extent k_collider_world builds from qmatrix(Q) and H); test(i) tests collider i and keeps the lane's
// best in `best`.  The large list first (every path tests it), then the grid: the path, clipped to the region that can hold the centre while
// the shape (or the ray's hit point) touches a small collider, is cut into segments of at most one cell along its dominant axis.  A small
// collider touched while the centre lies in a segment has its min-corner cell in [floor((lo - e - mu - W) / W), floor((hi + e + mu) / W)]
// per axis (cell_range): lo / hi = the segment's quantised extent, e = the shape's quantised extent (none for a ray), mu the margin
// (DESIGN.md sections 8.14, 8.16):
//   - 2 units plus 2^-16 of the magnitudes involved (twice the quantised origin and extent, the frame offset, 4 x 65,536), far above the
//     rounding of the quantisation, the transforms and the hit point;
//   - for a cast, k_overlap's 2^-6 (eumax + W), which covers the tests' rounding relative to the sizes and a rotation up to 2^-10 off unit
//     length;
//   - when `quad` (a cylinder, corner or sphere quadratic can run), its cancellation: disc = b*b - a*c rounds below 14 * 2^-24 |m|^2 |d|^2
//     (m = origin - centre), so the stated arithmetic can hit a sphere whose centre lies up to sqrt(28 * 2^-24) |m| < 2^-10.5 |m| beyond
//     its radius from the path; |m| <= t |d| + e + rc + that reach with rc below half a cell, so 2^-9 (t |du| + e + W) covers it.  mu_at(t)
//     is the margin at t; mu_clip bounds it over the whole grid (|m| of a centre in the grid is at most sqrt(3) (|ou| + 65536 + W + e)) and
//     only widens the clip.
// A ray's walk is the same code with the shape's terms left out (plus_e), so it pays for none of them.  Segments tile the clipped t range,
// so once the next segment starts beyond the warp's best t every closer hit has been tested.  A path tests every collider instead, counted
// in counts[fallback_slot], when its frame or margin is not finite, the margin at the far end exceeds two cells or the segments exceed
// NB_RAY_MAX_SEGMENTS; a cast also when !rot_ok (a BOX rotation more than 2^-10 from unit length) or one segment's cell range exceeds
// NB_OVERLAP_MAX_CELLS (a ray's cannot: the grid test bounds mu <= 2W and a segment spans at most about one cell per axis, so a ray's range
// is at most 8 cells per axis).  Repeated keys change nothing in the min.  A cast's cells skip the large colliders, which saves their costly
// second test; a ray tests them again, which costs less than loading every candidate's small flag (DESIGN.md section 8.16).
template<bool Cast, class F>
NB_DEV void swept_walk(const QueryScene& S, u32* counts, u32 fallback_slot, u32 lane, f3 o, f3 d, float max_t, f3 ext, bool quad,
		bool rot_ok, const u64& best, F test) {
	const u32 nlarge = counts[CNT_LARGE];
	for (u32 l = lane; l < nlarge; l += 32) test(S.order[S.large_list[l]]);
	const QueryGrid G = query_grid(counts);
	const float W = G.W, s = G.s;
	const float eu[3] = { ext.x * s, ext.y * s, ext.z * s };   // read only by a cast
	const float ou[3] = { o.x * s - G.f.ms[0], o.y * s - G.f.ms[1], o.z * s - G.f.ms[2] }, du[3] = { d.x * s, d.y * s, d.z * s };
	const float oumax = fmaxf(fabsf(ou[0]), fmaxf(fabsf(ou[1]), fabsf(ou[2]))), eumax = Cast ? fmaxf(eu[0], fmaxf(eu[1], eu[2])) : 0.0f;
	auto plus_e = [&](float x, float e) { return Cast ? x + e : x; };   // a term of the shape's, which a ray has not
	const float M = 2.0f * plus_e(oumax, eumax) + G.msmax + 262144.0f;
	const float mu0 = plus_e(2.0f + M * (1.0f / 65536.0f), (eumax + W) * (1.0f / 64.0f));
	const float dnorm = 1.01f * sqrtf(du[0] * du[0] + du[1] * du[1] + du[2] * du[2]);
	auto mu_at = [&](float t) { return mu0 + (quad ? (plus_e(t * dnorm, eumax) + W) * (1.0f / 512.0f) : 0.0f); };
	const float mu_clip = mu0 + (quad ? (plus_e(1.75f * plus_e(oumax + 65536.0f + W, eumax), eumax) + W) * (1.0f / 512.0f) : 0.0f);
	// the region holding the centre whenever the shape touches a small collider (quantised min corners lie in [0, 65536)), widened
	float tlo = 0.0f, thi = max_t, dmax = 0.0f;
	bool any = true;
	#pragma unroll
	for (int k = 0; k < 3; ++k) {
		const float lo = Cast ? -eu[k] - 2.0f * mu_clip : -2.0f * mu_clip, hi = plus_e(65536.0f + W, Cast ? eu[k] : 0.0f) + 2.0f * mu_clip;
		dmax = fmaxf(dmax, fabsf(du[k]));
		if (du[k] == 0.0f) { if (ou[k] < lo || ou[k] > hi) any = false; }
		else {
			const float t1 = (lo - ou[k]) / du[k], t2 = (hi - ou[k]) / du[k];
			tlo = fmaxf(tlo, fminf(t1, t2)); thi = fminf(thi, fmaxf(t1, t2));
		}
	}
	const float nsegf = ceilf((thi - tlo) * dmax / W);
	bool grid = G.ok && isfinite(mu_clip) && (!Cast || rot_ok)
		&& mu_at(fmaxf(thi, tlo)) <= 2.0f * W && dmax > 0.0f && isfinite(nsegf) && nsegf <= (float)NB_RAY_MAX_SEGMENTS;
	if (grid && any && tlo <= thi) {
		const u32 nseg = max(1u, (u32)nsegf);
		const float step = (thi - tlo) / (float)nseg;
		for (u32 k = 0; k < nseg; ++k) {
			const float ta = k == 0 ? tlo : tlo + (float)k * step, tb = k + 1 == nseg ? thi : tlo + (float)(k + 1) * step;
			const u64 wbest = warp_min_u64(best);
			if (wbest != ~(u64)0 && ta > asf((u32)(wbest >> 32))) break;   // every hit up to ta was tested
			float lo[3], hi[3];
			#pragma unroll
			for (int a = 0; a < 3; ++a) {
				const float ua = ou[a] + ta * du[a], ub = ou[a] + tb * du[a];
				lo[a] = Cast ? fminf(ua, ub) - eu[a] : fminf(ua, ub); hi[a] = plus_e(fmaxf(ua, ub), Cast ? eu[a] : 0.0f);
			}
			int c0[3], nc[3];
			if (!cell_range(G, lo, hi, mu_at(fmaxf(ta, tb)), c0, nc)) continue;
			if (Cast && cell_count(nc) > (float)NB_OVERLAP_MAX_CELLS) { grid = false; break; }   // every collider below
			grid_cells_visit(S, G, c0, nc, lane, Cast, test);
		}
	}
	if (!grid) {
		if (lane == 0) atomicAdd(&counts[fallback_slot], 1u);
		for (u32 i = lane; i < S.K; i += 32) test(i);
	}
}

// The warp's closest hit of the path from o along d (the least best over the lanes, the normal bn of the lane holding it) written to *out
// by that lane (lane 0 for a miss), with 4-byte stores since nb_ray_hit is only 4-byte aligned.  The whole warp calls it.
NB_DEV void write_closest_hit(const QueryScene& S, u64 best, f3 bn, f3 o, f3 d, u32 lane, nb_ray_hit* out) {
	const u64 wbest = warp_min_u64(best);
	const u32 winner = wbest == ~(u64)0 ? 0u : (u32)__ffs(__ballot_sync(0xffffffffu, best == wbest)) - 1;
	if (lane != winner) return;
	u32 w[12] = { 0, 0, 0, 0, 0, 0, 0, NB_RAY_NO_HIT, NB_RAY_NO_HIT, NB_RAY_NO_HIT, 0, 0 };   // a miss
	if (wbest != ~(u64)0) {
		const float t = asf((u32)(wbest >> 32));
		const u32 i = (u32)wbest;
		const f3 p = add3(o, mul3(t, d));
		w[0] = asu(p.x); w[1] = asu(p.y); w[2] = asu(p.z); w[3] = asu(t); w[4] = asu(bn.x); w[5] = asu(bn.y); w[6] = asu(bn.z);
		w[7] = i; w[8] = __ldg(S.col_body + i); w[9] = __ldg(S.col_tag + i);
	}
	u32* o32 = reinterpret_cast<u32*>(out);
	#pragma unroll
	for (int k = 0; k < 12; ++k) o32[k] = w[k];
}
// A ray's or cast's direction and max_t: finite, max_t >= 0 and the direction not zero.
NB_DEV bool sweep_valid(f3 d, float max_t) { return finite3(d) && isfinite(max_t) && max_t >= 0.0f && !is_zero3(d); }

// One warp per ray, swept_walk along it.  Without colliders (K = 0) every ray misses.  With boxes only, a ray falls back when its origin
// lies about 2^16 cells' widths outside the grid; with spheres, also when its clipped range ends more than about 1,000 cells' widths from the
// origin, which needs a grid of more than 1,000 cells per axis or an origin far outside.
__global__ void __launch_bounds__(NB_BLOCK) k_raycast(u32 n, const nb_ray* rays, nb_ray_hit* hits, u32 flags, QueryScene S, u32* counts) {
	const u32 lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
	const bool sensors = (flags & NB_RAY_SENSORS) != 0;
	for (u32 ri = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; ri < n; ri += nwarps) {   // ri is warp-uniform
		const nb_ray R = rays[ri];
		const f3 o = ld3(R.origin), d = ld3(R.direction);
		u64 best = ~(u64)0;
		f3 bn = mk3(0.0f, 0.0f, 0.0f);
		if (finite3(o) && sweep_valid(d, R.max_t) && S.K)
			swept_walk<false>(S, counts, CNT_RAY_FALLBACKS, lane, o, d, R.max_t, mk3(0.0f, 0.0f, 0.0f), S.K > S.nboxes, true, best,
				[&](u32 i) { ray_test(S, i, o, d, R.max_t, R.mask, R.ignore_body, sensors, best, bn); });
		write_closest_hit(S, best, bn, o, d, lane, hits + ri);
	}
}

// ---------------- overlap queries (nb_overlap): the per-collider arithmetic the header states ----------------
NB_DEV bool overlap_sphere_sphere(f3 c, float r, f3 p, float rc) { const f3 d = sub3(c, p); return dot3(d, d) <= (r + rc) * (r + rc); }
NB_DEV float box_gap(float l, float h) { return l < -h ? l + h : (l > h ? l - h : 0.0f); }
// The sphere (c, r) against the box (p, q, h): also a BOX query against a sphere collider, with the roles swapped.
NB_DEV bool overlap_sphere_box(f3 c, float r, f3 p, quat q, f3 h) {
	const f3 l = qrot(qconj(q), sub3(c, p));
	const f3 g = mk3(box_gap(l.x, h.x), box_gap(l.y, h.y), box_gap(l.z, h.z));
	return dot3(g, g) <= r * r;
}
NB_DEV float box_radius(f3 h, const f3 a[3], f3 L) { return (fabsf(h.x * dot3(a[0], L)) + fabsf(h.y * dot3(a[1], L))) + fabsf(h.z * dot3(a[2], L)); }
NB_DEV void box_axes(quat q, f3 a[3]) { a[0] = qrot(q, mk3(1.0f, 0.0f, 0.0f)); a[1] = qrot(q, mk3(0.0f, 1.0f, 0.0f)); a[2] = qrot(q, mk3(0.0f, 0.0f, 1.0f)); }
// The query box (c, axes u, H) against the box (p, q, h): the 15 axes in the header's order, the first that separates ends the test.
NB_DEV bool overlap_box_box(f3 c, const f3 u[3], f3 H, f3 p, quat q, f3 h) {
	f3 v[3]; box_axes(q, v);
	const f3 t = sub3(p, c);
	auto separates = [&](f3 L) { return fabsf(dot3(t, L)) > box_radius(H, u, L) + box_radius(h, v, L); };
	#pragma unroll
	for (int k = 0; k < 3; ++k) if (separates(u[k])) return false;
	#pragma unroll
	for (int k = 0; k < 3; ++k) if (separates(v[k])) return false;
	#pragma unroll
	for (int i = 0; i < 3; ++i) {
		#pragma unroll
		for (int k = 0; k < 3; ++k) if (separates(cross3(u[i], v[k]))) return false;
	}
	return true;
}

// A query as the walks hold it: the shape, and for a box its axes u_k = qrot(Q, e_k), computed once per query.
struct OverlapShape { bool box; f3 c; quat Q; f3 H; float r; f3 u[3]; };
// Loads query R into Q and returns whether it is valid; qq = dot(Q, Q) of a BOX rotation (1 for a sphere), ext = the world extent (a
// sphere's r; a box's as k_collider_world builds a box collider's from qmatrix(Q) and H).
NB_DEV bool load_shape(const nb_overlap_query& R, OverlapShape& Q, float& qq, f3& ext) {
	Q.box = R.shape == NB_OVERLAP_BOX;
	Q.c = ld3(R.center);
	bool valid = (R.shape == NB_OVERLAP_SPHERE || Q.box) && finite3(Q.c);
	qq = 1.0f;
	if (Q.box) {
		Q.Q = mkq(make_float4(R.rotation[0], R.rotation[1], R.rotation[2], R.rotation[3]));
		Q.H = ld3(R.half_extents);
		qq = dot3(Q.Q.v, Q.Q.v) + Q.Q.s * Q.Q.s;
		valid = valid && finite3(Q.Q.v) && isfinite(Q.Q.s) && qq != 0.0f && finite3(Q.H) && Q.H.x >= 0.0f && Q.H.y >= 0.0f && Q.H.z >= 0.0f;
		box_axes(Q.Q, Q.u);
		mat3 m = qmatrix(Q.Q);   // the extent as k_collider_world builds a box collider's
		m.c0 = mul3(m.c0, Q.H.x); m.c1 = mul3(m.c1, Q.H.y); m.c2 = mul3(m.c2, Q.H.z);
		ext = mk3(fabsf(m.c0.x) + fabsf(m.c1.x) + fabsf(m.c2.x), fabsf(m.c0.y) + fabsf(m.c1.y) + fabsf(m.c2.y), fabsf(m.c0.z) + fabsf(m.c1.z) + fabsf(m.c2.z));
	}
	else {
		Q.r = R.radius;
		valid = valid && isfinite(Q.r) && Q.r >= 0.0f;
		ext = mk3(Q.r, Q.r, Q.r);
	}
	return valid;
}

// Tests collider i against the query; a hit appends (query << kq | i) while the capacity lasts and counts in nhits.
NB_DEV void overlap_test(const QueryScene& S, u32 i, const OverlapShape& Q, u32 mask, u32 ignore, bool sensors, u64 qkey, u64* keys, u32 cap,
		u32* counts, u32& nhits) {
	if (!query_may_test(S, i, mask, ignore, sensors)) return;
	const xform w = ld_xform(S.world_xf, i);
	const f3 p = mk3(w.p.x, w.p.y, w.p.z);
	bool hit;
	if (i < S.nboxes) {
		const float4 sz = reinterpret_cast<const float4*>(S.box_data)[i];
		const f3 h = mk3(sz.x, sz.y, sz.z);
		hit = Q.box ? overlap_box_box(Q.c, Q.u, Q.H, p, mkq(w.q), h) : overlap_sphere_box(Q.c, Q.r, p, mkq(w.q), h);
	}
	else {
		const float rc = S.sph_data[i - S.nboxes].radius;
		hit = Q.box ? overlap_sphere_box(p, rc, Q.c, Q.Q, Q.H) : overlap_sphere_sphere(Q.c, Q.r, p, rc);
	}
	if (!hit) return;
	const u32 slot = warp_append_slot(&counts[CNT_OVERLAP_KEYS]);
	if (slot < cap) keys[slot] = qkey | i;
	++nhits;
}

// One warp per query.  Without colliders (K = 0) k_overlap is not launched.  A query on the grid tests the large list first, then the
// grid: the query's world AABB (its centre -/+ load_shape's extent) is taken into the Morton frame's quantised space, and cell_range gives
// the cells that can hold a touching small collider's min corner, lo / hi = the AABB's quantised extent.  mu is 2 units (the min corner's
// truncation and the cell-fit rule's +2) plus 2^-16 of the magnitudes involved (twice the quantised centre, the frame offset, 4 x 65,536),
// which bounds the rounding of the quantisation, the transforms and the tests' differences of positions, plus 2^-6 of (the query's quantised
// half extent + W), which bounds the tests' rounding relative to the query's and the collider's size and a query or collider rotation up to
// 2^-10 away from unit length (DESIGN.md section 8.15).  Those cells are looked up and dealt to the lanes by grid_cells_visit, which skips
// the large colliders (the large list tested them), so every collider is tested at most once.  A query that tests every collider instead
// (counted in CNT_OVERLAP_FALLBACKS): a cell range of more than NB_OVERLAP_MAX_CELLS cells, a frame or margin that is not finite, a BOX
// rotation with |dot(Q, Q) - 1| > 2^-10 (its extent need not bound what the stated test finds).
__global__ void __launch_bounds__(NB_BLOCK) k_overlap(u32 n, const nb_overlap_query* queries, u32 flags, QueryScene S, u32 kq, u64* keys, u32 cap,
		u32* counts) {
	const u32 lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
	const bool sensors = (flags & NB_OVERLAP_SENSORS) != 0;
	for (u32 qi = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; qi < n; qi += nwarps) {   // qi is warp-uniform
		const nb_overlap_query R = queries[qi];
		OverlapShape Q;
		float qq;
		f3 ext;
		if (!load_shape(R, Q, qq, ext)) continue;
		const u64 qkey = (u64)qi << kq;
		u32 nhits = 0;
		const QueryGrid G = query_grid(counts);
		const float W = G.W, s = G.s;
		const float cu[3] = { Q.c.x * s - G.f.ms[0], Q.c.y * s - G.f.ms[1], Q.c.z * s - G.f.ms[2] }, eu[3] = { ext.x * s, ext.y * s, ext.z * s };
		const float cumax = fmaxf(fabsf(cu[0]), fmaxf(fabsf(cu[1]), fabsf(cu[2]))), eumax = fmaxf(eu[0], fmaxf(eu[1], eu[2]));
		const float M = 2.0f * cumax + G.msmax + 262144.0f;
		const float mu = 2.0f + M * (1.0f / 65536.0f) + (eumax + W) * (1.0f / 64.0f);
		const float lo[3] = { cu[0] - eu[0], cu[1] - eu[1], cu[2] - eu[2] }, hi[3] = { cu[0] + eu[0], cu[1] + eu[1], cu[2] + eu[2] };
		int c0[3], nc[3];
		const bool cells = cell_range(G, lo, hi, mu, c0, nc);
		const bool grid = G.ok && isfinite(mu) && fabsf(qq - 1.0f) <= 1.0f / 1024.0f && (!cells || cell_count(nc) <= (float)NB_OVERLAP_MAX_CELLS);
		auto test = [&](u32 i) { overlap_test(S, i, Q, R.mask, R.ignore_body, sensors, qkey, keys, cap, counts, nhits); };
		if (!grid) {
			if (lane == 0) atomicAdd(&counts[CNT_OVERLAP_FALLBACKS], 1u);
			for (u32 i = lane; i < S.K; i += 32) test(i);
		}
		else {
			const u32 nlarge = counts[CNT_LARGE];
			for (u32 l = lane; l < nlarge; l += 32) test(S.order[S.large_list[l]]);
			if (cells) grid_cells_visit(S, G, c0, nc, lane, true, test);
		}
		#pragma unroll
		for (int o = 16; o; o >>= 1) nhits += __shfl_xor_sync(0xffffffffu, nhits, o);
		if (lane == 0 && nhits) atomicAdd(&counts[CNT_OVERLAP_TOTAL], nhits);
	}
}

// The output: offsets[q] = the first sorted key of query q or later (a binary search; offsets[n] = the total), then the hits, written with
// 4-byte stores since nb_overlap_hit and the offsets are only 4-byte aligned.  When the total exceeds the capacity only offsets[n] is
// written.  counts null: no collider or body, every query's range is empty.
__global__ void __launch_bounds__(NB_BLOCK) k_overlap_write(u32 n, const u64* keys, const u32* counts, u32 cap, u32 kq, const u32* col_body,
		const u32* col_tag, nb_overlap_hit* hits, u32* offsets) {
	const u32 total = counts ? counts[CNT_OVERLAP_TOTAL] : 0;
	const u64 tid = blockIdx.x * (u64)blockDim.x + threadIdx.x, stride = (u64)gridDim.x * blockDim.x;
	if (total > cap) { if (tid == 0) offsets[n] = total; return; }
	for (u64 q = tid; q <= n; q += stride) {
		const u64 first = q << kq;
		u32 lo = 0, hi = total;
		while (lo < hi) { const u32 mid = (lo + hi) >> 1; if (keys[mid] < first) lo = mid + 1; else hi = mid; }
		offsets[q] = lo;
	}
	const u64 cmask = ((u64)1 << kq) - 1;
	for (u64 i = tid; i < total; i += stride) {
		const u64 key = keys[i];
		const u32 c = (u32)(key & cmask);
		u32* out = reinterpret_cast<u32*>(hits + i);
		out[0] = (u32)(key >> kq); out[1] = c; out[2] = __ldg(col_body + c); out[3] = __ldg(col_tag + c);
	}
}

// ---------------- shape casts (nb_shapecast): the per-collider arithmetic the header states ----------------
// The quadratic of the edge cylinders and corner spheres: a, b, cc as stated, the entry t if it lies in [0, max_t] (-0 becomes +0).
NB_DEV bool sweep_root(float a, float b, float cc, float max_t, float& t) {
	const float disc = b * b - a * cc;
	if (disc < 0.0f) return false;
	t = (-b - sqrtf(disc)) / a;
	if (!(t >= 0.0f && t <= max_t)) return false;   // a NaN t misses too
	if (t == 0.0f) t = 0.0f;   // -0 -> +0: the hit key orders t by its bits
	return true;
}
// A sphere of radius r from lo along ld (the box's frame) against the box h centred at the origin: the 23 primitives of the rounded box in
// the header's order, the smallest t winning and the earlier primitive a tie.  nl = the local normal.
NB_DEV bool sweep_rounded_box(f3 lo, f3 ld, f3 h, float r, float max_t, float& t, f3& nl) {
	bool hit = false;
	float tk;
	#pragma unroll
	for (int k = 0; k < 3; ++k) {   // (a) the face boxes; with r == 0 they are one box
		if (k > 0 && r == 0.0f) break;
		const f3 hk = mk3(k == 0 ? h.x + r : h.x, k == 1 ? h.y + r : h.y, k == 2 ? h.z + r : h.z);
		int axis; float s;
		if (sweep_slab(lo, ld, hk, max_t, tk, axis, s) && (!hit || tk < t)) { hit = true; t = tk; nl = axis < 0 ? mk3(0.0f, 0.0f, 0.0f) : slab_normal(axis, s); }
	}
	if (r == 0.0f) return hit;
	const float los[3] = { lo.x, lo.y, lo.z }, lds[3] = { ld.x, ld.y, ld.z }, hs[3] = { h.x, h.y, h.z };
	const float inv = 1.0f / r;
	#pragma unroll
	for (int k = 0; k < 3; ++k) {   // (b) the edge cylinders along k
		const int i = k == 0 ? 1 : 0, j = k == 2 ? 1 : 2;
		const float a = lds[i] * lds[i] + lds[j] * lds[j];
		if (a == 0.0f) continue;
		#pragma unroll
		for (int e = 0; e < 4; ++e) {
			const float mi = los[i] - (e & 2 ? hs[i] : -hs[i]), mj = los[j] - (e & 1 ? hs[j] : -hs[j]);
			const float b = mi * lds[i] + mj * lds[j], cc = (mi * mi + mj * mj) - r * r;
			if (!sweep_root(a, b, cc, max_t, tk)) continue;
			const float z = los[k] + tk * lds[k];
			if (!(z >= -hs[k] && z <= hs[k]) || (hit && !(tk < t))) continue;
			float n3[3];
			n3[i] = (mi + tk * lds[i]) * inv; n3[j] = (mj + tk * lds[j]) * inv; n3[k] = 0.0f;
			hit = true; t = tk; nl = mk3(n3[0], n3[1], n3[2]);
		}
	}
	const float a = dot3(ld, ld);
	#pragma unroll
	for (int e = 0; e < 8; ++e) {   // (c) the corner spheres, x slowest
		const f3 c = mk3(e & 4 ? h.x : -h.x, e & 2 ? h.y : -h.y, e & 1 ? h.z : -h.z);
		const f3 m = sub3(lo, c);
		if (!sweep_root(a, dot3(m, ld), dot3(m, m) - r * r, max_t, tk) || (hit && !(tk < t))) continue;
		hit = true; t = tk; nl = mul3(sub3(add3(lo, mul3(tk, ld)), c), inv);
	}
	return hit;
}
// The query box (c, axes u, H) moving along d against the box (p, q, h): the swept separating axes in nb_overlap's order.
NB_DEV bool sweep_box_box(f3 c, const f3 u[3], f3 H, f3 d, float max_t, f3 p, quat q, f3 h, float& t, f3& n) {
	f3 v[3]; box_axes(q, v);
	const f3 t0 = sub3(p, c);
	float enter = 0.0f, exit = max_t, sb = 0.0f;
	f3 axis = mk3(0.0f, 0.0f, 0.0f);
	bool rec = false;
	auto bound = [&](f3 L) {   // false: the cast misses
		const float a = dot3(t0, L), b = dot3(d, L), R = box_radius(H, u, L) + box_radius(h, v, L);
		if (b == 0.0f) return !(fabsf(a) > R);
		const float t1 = (a - R) / b, t2 = (a + R) / b;
		const bool lt = t1 < t2;
		const float near = lt ? t1 : t2, far = lt ? t2 : t1;
		if (near > enter) { enter = near; axis = L; sb = b; rec = true; }
		if (far < exit) exit = far;
		return !(enter > exit);
	};
	#pragma unroll
	for (int k = 0; k < 3; ++k) if (!bound(u[k])) return false;
	#pragma unroll
	for (int k = 0; k < 3; ++k) if (!bound(v[k])) return false;
	#pragma unroll
	for (int i = 0; i < 3; ++i) {
		#pragma unroll
		for (int k = 0; k < 3; ++k) if (!bound(cross3(u[i], v[k]))) return false;
	}
	t = enter;
	if (!rec) n = mk3(0.0f, 0.0f, 0.0f);
	else {
		const float inv = 1.0f / sqrtf(dot3(axis, axis));
		n = mul3(sb > 0.0f ? mk3(-axis.x, -axis.y, -axis.z) : axis, inv);
	}
	return true;
}

// Tests collider i against the cast and keeps the lane's best (t bits << 32 | i) and the normal that goes with it.
NB_DEV void cast_test(const QueryScene& S, u32 i, const OverlapShape& Q, f3 d, float max_t, u32 mask, u32 ignore, bool sensors, u64& best, f3& bn) {
	if (!query_may_test(S, i, mask, ignore, sensors)) return;
	const xform w = ld_xform(S.world_xf, i);
	const f3 p = mk3(w.p.x, w.p.y, w.p.z);
	const quat q = mkq(w.q);
	float t = 0.0f;
	f3 n = mk3(0.0f, 0.0f, 0.0f), nl;
	bool hit;
	if (i < S.nboxes) {
		const float4 sz = reinterpret_cast<const float4*>(S.box_data)[i];
		const f3 h = mk3(sz.x, sz.y, sz.z);
		if (Q.box ? overlap_box_box(Q.c, Q.u, Q.H, p, q, h) : overlap_sphere_box(Q.c, Q.r, p, q, h)) hit = true;   // step 0
		else if (Q.box) hit = sweep_box_box(Q.c, Q.u, Q.H, d, max_t, p, q, h, t, n);
		else {
			const quat qc = qconj(q);
			hit = sweep_rounded_box(qrot(qc, sub3(Q.c, p)), qrot(qc, d), h, Q.r, max_t, t, nl);
			if (hit && !is_zero3(nl)) n = qrot(q, nl);
		}
	}
	else {
		const float rc = S.sph_data[i - S.nboxes].radius;
		if (Q.box ? overlap_sphere_box(p, rc, Q.c, Q.Q, Q.H) : overlap_sphere_sphere(Q.c, Q.r, p, rc)) hit = true;   // step 0
		else if (Q.box) {
			const quat qc = qconj(Q.Q);
			hit = sweep_rounded_box(qrot(qc, sub3(p, Q.c)), qrot(qc, mk3(-d.x, -d.y, -d.z)), Q.H, rc, max_t, t, nl);
			if (hit && !is_zero3(nl)) { const f3 m = qrot(Q.Q, nl); n = mk3(-m.x, -m.y, -m.z); }
		}
		else hit = ray_sphere(Q.c, d, max_t, w, Q.r + rc, t, n);
	}
	if (!hit) return;
	const u64 key = (u64)asu(t) << 32 | i;
	if (key < best) { best = key; bn = n; }
}

// One warp per cast, swept_walk along the centre's path with the shape's extent and k_overlap's size term; a quadratic runs against a
// sphere collider, and for a SPHERE cast of r > 0 against a box (its cylinders and corners).  Without colliders (K = 0) every cast misses.
// One block per SM: the inlined tests need 174 registers, and under the default bound ptxas caps them at 128 and spills.
__global__ void __launch_bounds__(NB_BLOCK, 1) k_shapecast(u32 n, const nb_shape_cast* casts, nb_ray_hit* hits, u32 flags, QueryScene S, u32* counts) {
	const u32 lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
	const bool sensors = (flags & NB_SHAPECAST_SENSORS) != 0;
	for (u32 ci = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; ci < n; ci += nwarps) {   // ci is warp-uniform
		const nb_shape_cast C = casts[ci];
		const nb_overlap_query& R = C.shape;
		OverlapShape Q;
		float qq;
		f3 ext;
		const f3 d = ld3(C.direction);
		const bool valid = load_shape(R, Q, qq, ext) && sweep_valid(d, C.max_t);
		u64 best = ~(u64)0;
		f3 bn = mk3(0.0f, 0.0f, 0.0f);
		if (valid && S.K)
			swept_walk<true>(S, counts, CNT_SHAPECAST_FALLBACKS, lane, Q.c, d, C.max_t, ext, S.K > S.nboxes || (!Q.box && Q.r > 0.0f),
				fabsf(qq - 1.0f) <= 1.0f / 1024.0f, best, [&](u32 i) { cast_test(S, i, Q, d, C.max_t, R.mask, R.ignore_body, sensors, best, bn); });
		write_closest_hit(S, best, bn, Q.c, d, lane, hits + ci);
	}
}

// ---------------- continuous collision (nb_upload_ccd_bodies, DESIGN.md section 8.18) ----------------
// Whether a cast whose sphere (c, r) touches collider i at t = 0 counts there: not when nb_overlap's test of the sphere holds (a start, which
// nb_collide's contact covers), and otherwise only when d points into the collider, dot(g, d') < 0 with g the step-0 test's gap (for a box
// in its frame, d' = d in that frame; for a sphere c - p, d' = d).  A sphere clamped onto a face can sit where the face slab counts its start
// as inside while step 0, rounded the other way, does not; moving away or along the face must still be free.
NB_DEV bool ccd_counts_at_zero(const QueryScene& S, u32 i, f3 c, float r, f3 d) {
	const xform w = ld_xform(S.world_xf, i);
	const f3 p = mk3(w.p.x, w.p.y, w.p.z);
	if (i < S.nboxes) {
		const float4 sz = reinterpret_cast<const float4*>(S.box_data)[i];
		const f3 h = mk3(sz.x, sz.y, sz.z);
		const quat q = mkq(w.q), qc = qconj(q);
		if (overlap_sphere_box(c, r, p, q, h)) return false;
		const f3 l = qrot(qc, sub3(c, p));
		return dot3(mk3(box_gap(l.x, h.x), box_gap(l.y, h.y), box_gap(l.z, h.z)), qrot(qc, d)) < 0.0f;
	}
	if (overlap_sphere_sphere(c, r, p, S.sph_data[i - S.nboxes].radius)) return false;
	return dot3(sub3(c, p), d) < 0.0f;
}

// Tests collider i against the swept sphere Q of body `body` along d (max_t = 1) and keeps the lane's best (t bits << 32 | i).  Only
// colliders the step could give the body a contact with count: Box2D's rule between the entry's filter word and the collider's
// (k_collider_world's, NB_FILTER_ALL without a table), not on a connected body under NB_FILTER_SKIP_CONNECTED (conn_n != 0), and
// cast_test's own body and sensor skips; the sphere arithmetic is cast_test's, with its t = 0 hits filtered by ccd_counts_at_zero.
NB_DEV void ccd_test(const QueryScene& S, u32 i, u32 body, u32 word, const u64* conn_keys, u32 conn_n, const OverlapShape& Q, f3 d, u64& best) {
	if (!filter_pass(word, asu(reinterpret_cast<const float*>(S.aabb_max)[4 * (size_t)i + 3]))) return;
	if (conn_n && connected(conn_keys, conn_n, body, __ldg(S.col_body + i))) return;
	u64 key = ~(u64)0;
	f3 n;
	cast_test(S, i, Q, d, 1.0f, ~0u, body, false, key, n);
	if (key >= best) return;
	if ((u32)(key >> 32) == 0u && !ccd_counts_at_zero(S, i, Q.c, Q.r, d)) return;
	best = key;
}

// One warp per set entry, on nb_advance's stream before k_advance<true>: the entry's body, when the step advances it (its island active in
// the last collide, not kinematic) and its translation d = v * dt is longer than the threshold and valid for a sweep, casts its sphere from
// its position along d against the step's front end (S: ctx->front as nb_collide left it) with swept_walk; fallbacks count in
// counts[CNT_CCD_FALLBACKS].  Lane 0 writes the body's translation factor ccd_t[body] (the hit's t, else 1) and hits[e] = (bits of t,
// collider or NB_RAY_NO_HIT).  One block per SM as for k_shapecast: the inlined walk and tests need 90 registers, and under the default bound
// ptxas caps them at 80 and spills.
__global__ void __launch_bounds__(NB_BLOCK, 1) k_ccd(u32 n, const nb_ccd_body* set, const nb_transform* xf, const nb_body_momentum* momentum,
		const u32* parent, const u32* active, const uint8_t* kind, float time_step, QueryScene S, const u64* conn_keys, u32 conn_n, u32* counts,
		float* ccd_t, uint2* hits) {
	const u32 lane = threadIdx.x & 31, nwarps = (gridDim.x * blockDim.x) >> 5;
	for (u32 e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < n; e += nwarps) {   // e is warp-uniform
		const uint4 E = reinterpret_cast<const uint4*>(set)[e];
		const u32 b = E.x, word = E.w;   // category | mask << 16, a collider filter word
		const float r = asf(E.y), thr = asf(E.z);
		const float4 l = reinterpret_cast<const float4*>(momentum + b)[0];
		const f3 d = mk3(l.x * time_step, l.y * time_step, l.z * time_step);
		u64 best = ~(u64)0;
		const bool advanced = active[parent[b]] && !(kind && (kind[b] & 1u));
		if (advanced && (d.x * d.x + d.y * d.y) + d.z * d.z > thr * thr && sweep_valid(d, 1.0f) && S.K) {
			const xform x = ld_xform(xf, b);
			OverlapShape Q;
			Q.box = false; Q.c = mk3(x.p.x, x.p.y, x.p.z); Q.r = r;
			swept_walk<true>(S, counts, CNT_CCD_FALLBACKS, lane, Q.c, d, 1.0f, mk3(r, r, r), S.K > S.nboxes || r > 0.0f, true, best,
				[&](u32 i) { ccd_test(S, i, b, word, conn_keys, conn_n, Q, d, best); });
		}
		const u64 wbest = warp_min_u64(best);
		if (lane == 0) {
			const bool hit = wbest != ~(u64)0;
			const u32 tb = hit ? (u32)(wbest >> 32) : asu(1.0f);
			ccd_t[b] = asf(tb);
			hits[e] = make_uint2(tb, hit ? (u32)wbest : NB_RAY_NO_HIT);
		}
	}
}

// The queries' scratch for the collider capacity, allocated once from the context's arena (synchronises then; never again).
static int ensure_query_scratch(nb_context* ctx) {
	QueryScratch& r = ctx->query;
	const u32 K = ctx->cfg.max_boxes + ctx->cfg.max_spheres;
	if (r.ready) return NB_OK;
	{ int e = alloc_front_end(ctx, r.front, K); if (e) return e; }
	for (int i = 0; i < 2; ++i) { ALLOC(r.sb.keys[i], K); ALLOC(r.sb.vals[i], K); }
	ALLOC(r.sb.hist, 256 * (size_t)ctx->sms); ALLOC(r.counts, CNT__COUNT);
	r.sb.bar = r.counts + CNT_BAR0;   // zeroed by alloc_zeroed: the sort's grid barrier starts from zero arrivals
	r.ready = true;   // only once every buffer exists: a failed allocation leaves the next call to try again
	return NB_OK;
}

// The refusals the three queries share, in the header's order: a sharded context, unknown flags, null buffers (`null_args`, naming
// `buffers`); then, for n > 0, the queries' scratch.
static int query_begin(nb_context* ctx, const char* call, u32 flags, u32 known_flags, bool null_args, const char* buffers, u32 n) {
	if (ctx->sharded) { ctx->error = std::string(call) + ": not supported on a context of nb_shard_create"; return NB_ERR_ARGUMENT; }
	if (flags & ~known_flags) { ctx->error = std::string(call) + ": unknown flags"; return NB_ERR_ARGUMENT; }
	if (null_args) { ctx->error = std::string(call) + ": null " + buffers; return NB_ERR_ARGUMENT; }
	return n ? ensure_query_scratch(ctx) : NB_OK;
}
// The front end on the queries' scratch without the kinematic and sensor tables (nothing without colliders or bodies: S.K = 0), and the
// scene the query kernels read.
static int query_scene(nb_context* ctx, const Launch& L, QueryScene& S) {
	const u32 K = ctx->B ? ctx->nboxes + ctx->nspheres : 0;
	const FrontEnd& f = ctx->query.front;
	if (int r = K ? launch_front_end(ctx, L, f, ctx->query.sb, ctx->query.counts, ctx->has_filter ? ctx->filter : nullptr, nullptr, nullptr) : NB_OK) return r;
	S = { K, ctx->nboxes, f.world_xf, f.aabb_max, f.col_body, f.col_tag, ctx->box_data, ctx->sph_data, ctx->has_sensor ? ctx->sensor : nullptr,
		  f.order, f.smallf, f.table_keys, f.table_vals, f.table_mask, f.large_list };
	return NB_OK;
}
// nb_raycast and nb_shapecast: n paths `in` (staged through `stage` from host pointers) into n hits, one warp each.
template<class In>
static int sweep_call(nb_context* ctx, const char* call, const char* buffers, const In* in, u32 n, nb_ray_hit* hits, u32 flags, u32 known_flags,
		DevBuf<In>& stage, void (*kernel)(u32, const In*, nb_ray_hit*, u32, QueryScene, u32*), int on_device, void* stream) {
	NB_RANGE(call);
	if (int r = query_begin(ctx, call, flags, known_flags, n && (!in || !hits), buffers, n)) return r;
	if (!n) return NB_OK;
	cudaStream_t st = (cudaStream_t)stream;
	QueryScratch& q = ctx->query;
	const In* din = in;
	nb_ray_hit* dhits = hits;
	if (!on_device) {
		GROW(stage, n, st); GROW(q.hits, n, st);
		CK(put_staged(ctx, stage.p, in, sizeof(In) * (size_t)n, st));
		din = stage.p; dhits = q.hits.p;
	}
	const Launch L = mk_launch(ctx, st);
	QueryScene S;
	if (int r = query_scene(ctx, L, S)) return r;
	launch_grid(L, kernel, GRID(std::min<u64>((u64)n * 32, 0xffffffffu)), n, din, dhits, flags, S, q.counts);
	CK(cudaGetLastError());
	if (!on_device) {
		CK(cudaMemcpyAsync(hits, dhits, sizeof(nb_ray_hit) * (size_t)n, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
	}
	return NB_OK;
}

extern "C" {

int nb_raycast(nb_context* ctx, const nb_ray* rays, uint32_t n, nb_ray_hit* hits, uint32_t flags, int on_device, void* stream) {
	return sweep_call(ctx, "nb_raycast", "rays or hits", rays, n, hits, flags, NB_RAY_SENSORS, ctx->query.rays, k_raycast, on_device, stream);
}

int nb_shapecast(nb_context* ctx, const nb_shape_cast* casts, uint32_t n, nb_ray_hit* hits, uint32_t flags, int on_device, void* stream) {
	return sweep_call(ctx, "nb_shapecast", "casts or hits", casts, n, hits, flags, NB_SHAPECAST_SENSORS, ctx->query.casts, k_shapecast, on_device, stream);
}

int nb_overlap(nb_context* ctx, const nb_overlap_query* queries, uint32_t n, nb_overlap_hit* hits, uint32_t capacity, uint32_t* offsets,
			   uint32_t flags, int on_device, void* stream) {
	NB_RANGE("nb_overlap");
	if (int r = query_begin(ctx, "nb_overlap", flags, NB_OVERLAP_SENSORS, n && (!queries || !offsets || (capacity && !hits)), "queries, offsets or hits", n))
		return r;
	if (!n) return NB_OK;
	cudaStream_t st = (cudaStream_t)stream;
	QueryScratch& q = ctx->query;
	for (int i = 0; i < 2; ++i) { GROW(q.okeys[i], std::max(capacity, 1u), st); q.osb.keys[i] = q.okeys[i].p; q.osb.vals[i] = nullptr; }
	q.osb.hist = q.sb.hist; q.osb.bar = q.sb.bar;   // the front end's sort has finished with them when the hit sort runs
	const nb_overlap_query* dq = queries;
	nb_overlap_hit* dh = hits;
	u32* doff = offsets;
	if (!on_device) {
		GROW(q.oq, n, st); GROW(q.oh, std::max(capacity, 1u), st); GROW(q.ooff, (size_t)n + 1, st);
		CK(put_staged(ctx, q.oq.p, queries, sizeof(nb_overlap_query) * (size_t)n, st));
		dq = q.oq.p; dh = q.oh.p; doff = q.ooff.p;
	}
	const Launch L = mk_launch(ctx, st);
	QueryScene S;
	if (int r = query_scene(ctx, L, S)) return r;
	const u32 grid_out = GRID(std::max<u64>((u64)n + 1, capacity));
	if (S.K) {
		u32* counts = q.counts;
		const u32 kq = bits_for(S.K);
		launch_grid(L, k_overlap, GRID(std::min<u64>((u64)n * 32, 0xffffffffu)), n, dq, flags, S, kq, q.osb.keys[0], capacity, counts);
		const int cur = nb_radix_sort(L, q.osb, counts + CNT_OVERLAP_KEYS, 0, (int)(kq + bits_for(n)), false, 0, 0, 0, nullptr, capacity);
		launch_grid(L, k_overlap_write, grid_out, n, (const u64*)q.osb.keys[cur], (const u32*)counts, capacity, kq, S.col_body, S.col_tag, dh, doff);
	}
	else launch_grid(L, k_overlap_write, grid_out, n, (const u64*)nullptr, (const u32*)nullptr, capacity, 1u, (const u32*)nullptr,
			(const u32*)nullptr, dh, doff);
	CK(cudaGetLastError());
	if (!on_device) {
		CK(cudaMemcpyAsync(offsets, doff, sizeof(u32) * ((size_t)n + 1), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		const u32 total = offsets[n];
		if (total > capacity) { ctx->error = "nb_overlap: " + std::to_string(total) + " hits exceed the capacity"; return NB_ERR_CAPACITY; }
		if (total) {
			CK(cudaMemcpyAsync(hits, dh, sizeof(nb_overlap_hit) * (size_t)total, cudaMemcpyDeviceToHost, st));
			CK(cudaStreamSynchronize(st));
		}
	}
	return NB_OK;
}

}  // extern "C"
