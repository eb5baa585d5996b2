// nudge_b200 — collide(): collider world transforms + AABBs, Morton order, grid broadphase,
// island detection, pair partition, box-box / box-sphere / sphere-sphere narrowphase with feature tags,
// active-body list and contact compaction.  Replaces nudge::collide (nudge.cpp:3000-4009) and the three
// narrowphase routines (nudge.cpp:1177-2604).
//
// Design: the reference's two-level "8 AABBs per coarse AABB, all coarse pairs" scheme
// (nudge.cpp:3204-3399) is O((K/8)^2); here the Morton-sorted colliders are binned into grid cells that are
// Morton prefixes, each collider looks only into its neighbouring cells, and pairs are appended with
// warp-aggregated atomics.  The pair SET is identical (all strictly overlapping AABBs); orientation and order
// come from the Morton rank and a radix sort exactly as nudge.cpp:3493-3498 defines them.  The narrowphase
// tests every pair, clips the box-box survivors, then moves the contacts to scanned offsets so that they land in the
// reference's order: box-box face contacts, box-box edge contacts, box-sphere, sphere-sphere.
#pragma once
#include "nb_prims.cuh"

enum {  // device counters (u32 each)
	CNT_PAIRS, CNT_LIVE0, CNT_LIVE1, CNT_LIVE2, CNT_LIVE3, CNT_SLEEP_COARSE, CNT_LIVE_TOTAL,
	CNT_FACE, CNT_EDGE, CNT_OTHER, CNT_STAGED, CNT_CONTACTS, CNT_SLEEP_FINE, CNT_SLEEPING, CNT_ACTIVE,
	CNT_CACHE, CNT_CULLED, CNT_FULL_BATCHES, CNT_BATCHES, CNT_LEVELS, CNT_ENTRIES, CNT_OVERFLOW, CNT_LVCH0, CNT_LVCH1, CNT_LVCH2,
	CNT_BMIN0, CNT_BMIN1, CNT_BMIN2, CNT_BMIN3, CNT_BMAX0, CNT_BMAX1, CNT_BMAX2, CNT_BMAX3,
	CNT_BAR0, CNT_BAR1, CNT_SCRATCH0, CNT_SCRATCH1, CNT_EXT_SUM, CNT_GRID_LEVEL, CNT_LARGE, CNT_SURV, CNT_TMP, CNT_CHAIN_CURSOR,
	CNT_EXT_HIST = 64 /* 18 bins */, CNT__COUNT = 96
};
enum { OVF_PAIRS = 1, OVF_CONTACTS = 2, OVF_SCHED = 4, OVF_LEVELS = 8 };

// ---------------- K1: collider world transform + AABB (nudge.cpp:3021-3079) ----------------
__global__ void __launch_bounds__(NB_BLOCK) k_collider_world(u32 nboxes, u32 nspheres, const nb_transform* body_xf,
		const nb_transform* box_xf, const nb_box_collider* box_data, const u32* box_tags,
		const nb_transform* sph_xf, const nb_sphere_collider* sph_data, const u32* sph_tags,
		nb_transform* world_xf, float4* aabb_min, float4* aabb_max, u32* col_tag, u32* col_body, u32* counts) {
	u32 K = nboxes + nspheres;
	float mn[3] = { INFINITY, INFINITY, INFINITY }, mx[3] = { -INFINITY, -INFINITY, -INFINITY };
	float ext_sum = 0.0f;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < K; i += gridDim.x * blockDim.x) {
		bool is_box = i < nboxes;
		xform l = is_box ? ld_xform(box_xf, i) : ld_xform(sph_xf, i - nboxes);
		u32 body = asu(l.p.w);
		xform b = ld_xform(body_xf, body);
		// Transform * Transform: nudge.cpp:1165-1175
		quat bq = mkq(b.q);
		f3 p = add3(qrot(bq, mk3(l.p.x, l.p.y, l.p.z)), mk3(b.p.x, b.p.y, b.p.z));
		quat q = qmul(bq, mkq(l.q));
		xform w; w.p = make_float4(p.x, p.y, p.z, asf(body)); w.q = make_float4(q.v.x, q.v.y, q.v.z, q.s);
		f3 ext;
		if (is_box) {
			mat3 m = qmatrix(q);
			float4 s = reinterpret_cast<const float4*>(box_data)[i];
			m.c0 = mul3(m.c0, s.x); m.c1 = mul3(m.c1, s.y); m.c2 = mul3(m.c2, s.z);
			ext = mk3(fabsf(m.c0.x) + fabsf(m.c1.x) + fabsf(m.c2.x), fabsf(m.c0.y) + fabsf(m.c1.y) + fabsf(m.c2.y), fabsf(m.c0.z) + fabsf(m.c1.z) + fabsf(m.c2.z));
		}
		else {
			float r = sph_data[i - nboxes].radius;
			ext = mk3(r, r, r);
		}
		float4 lo = make_float4(p.x - ext.x, p.y - ext.y, p.z - ext.z, 0.0f);
		float4 hi = make_float4(p.x + ext.x, p.y + ext.y, p.z + ext.z, 0.0f);
		st_xform(world_xf, i, w);
		aabb_min[i] = lo; aabb_max[i] = hi;
		col_tag[i] = is_box ? box_tags[i] : sph_tags[i - nboxes];
		col_body[i] = body;
		mn[0] = fminf(mn[0], lo.x); mn[1] = fminf(mn[1], lo.y); mn[2] = fminf(mn[2], lo.z);
		mx[0] = fmaxf(mx[0], lo.x); mx[1] = fmaxf(mx[1], lo.y); mx[2] = fmaxf(mx[2], lo.z);
		ext_sum += 2.0f * fmaxf(ext.x, fmaxf(ext.y, ext.z));
	}
	// mean AABB extent (only steers the grid cell size of the broadphase, never a result): warp sum, one float atomic per warp
	#pragma unroll
	for (int d = 16; d; d >>= 1) ext_sum += __shfl_xor_sync(0xffffffffu, ext_sum, d);
	if ((threadIdx.x & 31) == 0 && ext_sum > 0.0f) atomicAdd(reinterpret_cast<float*>(&counts[CNT_EXT_SUM]), ext_sum);
	// scene bounds over AABB *mins* (nudge.cpp:3087-3094): min/max are exact, so any reduction order gives the same bits
	#pragma unroll
	for (int k = 0; k < 3; ++k) {
		#pragma unroll
		for (int d = 16; d; d >>= 1) {
			mn[k] = fminf(mn[k], __shfl_xor_sync(0xffffffffu, mn[k], d));
			mx[k] = fmaxf(mx[k], __shfl_xor_sync(0xffffffffu, mx[k], d));
		}
	}
	if ((threadIdx.x & 31) == 0) {
		#pragma unroll
		for (int k = 0; k < 3; ++k) {
			atomicMin(&counts[CNT_BMIN0 + k], f2ord(mn[k]));
			atomicMax(&counts[CNT_BMAX0 + k], f2ord(mx[k]));
		}
	}
}

// ---------------- K2: Morton codes (nudge.cpp:3096-3163, 2606-2645) ----------------
NB_DEV void dilate3(u32 x, u32 offset, u32& lo32, u32& hi32) {
	u32 lo24 = x & 0xff, hi24 = (x >> 8) & 0xff;
	lo24 = (lo24 | (lo24 << 8)) & 0x0f00f00fu; hi24 = (hi24 | (hi24 << 8)) & 0x0f00f00fu;
	lo24 = (lo24 | (lo24 << 4)) & 0xc30c30c3u; hi24 = (hi24 | (hi24 << 4)) & 0xc30c30c3u;
	lo24 = (lo24 | (lo24 << 2)) & 0x49249249u; hi24 = (hi24 | (hi24 << 2)) & 0x49249249u;
	lo32 = (lo24 << offset) | (hi24 << (24 + offset));
	hi32 = hi24 >> (8 - offset);
}

struct MortonFrame { float L[4]; float ms[3]; };
NB_DEV MortonFrame morton_frame(const u32* counts) {
	MortonFrame f;
	float smin[4], smax[4], sc[4];
	#pragma unroll
	for (int k = 0; k < 3; ++k) { smin[k] = ord2f(counts[CNT_BMIN0 + k]); smax[k] = ord2f(counts[CNT_BMAX0 + k]); }
	smin[3] = 0.0f; smax[3] = 0.0f;
	#pragma unroll
	for (int k = 0; k < 4; ++k) sc[k] = 65535.0f * nb_rcp(smax[k] - smin[k]);
	float A[4] = { nb_min(sc[0], sc[2]), nb_min(sc[1], sc[2]), nb_min(sc[2], sc[0]), nb_min(sc[2], sc[1]) };
	f.L[0] = nb_min(A[0], A[1]); f.L[1] = nb_min(A[1], A[0]); f.L[2] = nb_min(A[2], A[3]); f.L[3] = nb_min(A[3], A[2]);
	f.ms[0] = smin[0] * f.L[0]; f.ms[1] = smin[1] * f.L[1]; f.ms[2] = smin[2] * f.L[2];
	return f;
}
// quantised min corner of collider i exactly as k_morton computes it (i = ORIGINAL collider index: the lane-dependent scale)
NB_DEV void morton_quantise(const MortonFrame& f, float4 p, u32 i, u32& x, u32& y, u32& z) {
	float s = f.L[i & 3];
	x = (u32)nb_toint(nb_msub(p.x, s, f.ms[0])); y = (u32)nb_toint(nb_msub(p.y, s, f.ms[1])); z = (u32)nb_toint(nb_msub(p.z, s, f.ms[2]));
}

// Also bins the colliders by the grid level they need (smallest l with quantised extent + 2 <= 2^l; 17 = never) for grid_setup.
NB_DEV u32 grid_level_needed(float4 lo, float4 hi, float scale) {
	float ext = fmaxf(hi.x - lo.x, fmaxf(hi.y - lo.y, hi.z - lo.z)) * scale + 2.0f;
	u32 l = 1;
	while (l <= 16 && !(ext <= (float)(1u << l))) ++l;  // NaN never fits
	return l;
}
__global__ void __launch_bounds__(NB_BLOCK) k_morton(u32 K, const float4* aabb_min, const float4* aabb_max, u32* counts, u64* keys, u32* vals, u64* keybits /* OR, AND of all codes: steers the sort's bucket digit */) {
	__shared__ u32 s_hist[18];
	u64 k_or = 0, k_and = ~(u64)0;
	if (threadIdx.x < 18) s_hist[threadIdx.x] = 0;
	__syncthreads();
	float smin[4], smax[4], sc[4];
	#pragma unroll
	for (int k = 0; k < 3; ++k) { smin[k] = ord2f(counts[CNT_BMIN0 + k]); smax[k] = ord2f(counts[CNT_BMAX0 + k]); }
	smin[3] = 0.0f; smax[3] = 0.0f;  // the unused0 lane of the AABB (nudge.cpp:879-884)
	#pragma unroll
	for (int k = 0; k < 4; ++k) sc[k] = 65535.0f * nb_rcp(smax[k] - smin[k]);
	float A[4] = { nb_min(sc[0], sc[2]), nb_min(sc[1], sc[2]), nb_min(sc[2], sc[0]), nb_min(sc[2], sc[1]) };  // nudge.cpp:3098
	float L[4] = { nb_min(A[0], A[1]), nb_min(A[1], A[0]), nb_min(A[2], A[3]), nb_min(A[3], A[2]) };          // nudge.cpp:3099
	float ms[3] = { smin[0] * L[0], smin[1] * L[1], smin[2] * L[2] };                                         // nudge.cpp:3100
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < K; i += gridDim.x * blockDim.x) {
		float4 p = aabb_min[i];
		float s = L[i & 3];  // SoA lane j is scaled by AoS lane j&3 (nudge.cpp:3143-3145); all four hold the same min
		u32 x = (u32)nb_toint(nb_msub(p.x, s, ms[0]));
		u32 y = (u32)nb_toint(nb_msub(p.y, s, ms[1]));
		u32 z = (u32)nb_toint(nb_msub(p.z, s, ms[2]));
		u32 lx, hx, ly, hy, lz, hz;
		dilate3(x, 2, lx, hx); dilate3(y, 1, ly, hy); dilate3(z, 0, lz, hz);
		const u64 code = (u64)(lx | ly | lz) | ((u64)(hx | hy | hz) << 32);
		keys[i] = code;
		vals[i] = i;
		k_or |= code; k_and &= code;
		atomicAdd(&s_hist[grid_level_needed(p, aabb_max[i], L[0])], 1u);
	}
	#pragma unroll
	for (int d = 16; d; d >>= 1) { k_or |= __shfl_xor_sync(0xffffffffu, k_or, d); k_and &= __shfl_xor_sync(0xffffffffu, k_and, d); }
	if ((threadIdx.x & 31) == 0) { atomicOr((unsigned long long*)&keybits[0], (unsigned long long)k_or); atomicAnd((unsigned long long*)&keybits[1], (unsigned long long)k_and); }
	__syncthreads();
	if (threadIdx.x < 18 && s_hist[threadIdx.x]) atomicAdd(&counts[CNT_EXT_HIST + threadIdx.x], s_hist[threadIdx.x]);
}

// Cell edge 2^j of the grid broadphase (K4 below): the finest level that leaves at most NB_GRID_MAX_LARGE colliders too big for a
// cell (those go through the brute-force kernel, K tests each), read off the histogram k_morton made.
#define NB_GRID_MAX_LARGE 64u
NB_DEV void grid_setup(u32* counts) {
	u32 j = 16, above = counts[CNT_EXT_HIST + 17];
	for (u32 l = 16; l >= 1; --l) {  // above = colliders needing a level > l
		if (above <= NB_GRID_MAX_LARGE) j = l;
		above += counts[CNT_EXT_HIST + l];
	}
	counts[CNT_GRID_LEVEL] = j; counts[CNT_LARGE] = 0;
}

// ---------------- K3: Morton-ordered leaves (+ the grid level, one thread) ----------------
__global__ void __launch_bounds__(NB_BLOCK) k_leaves(u32 K, const u32* sorted_vals, const u64* sorted_keys, const float4* aabb_min, const float4* aabb_max,
													 u32* order, u32* rank, float4* leaf_min, float4* leaf_max, u64* mkeys, u32* counts) {
	if (blockIdx.x == 0 && threadIdx.x == 0) grid_setup(counts);
	for (u32 pos = blockIdx.x * blockDim.x + threadIdx.x; pos < K; pos += gridDim.x * blockDim.x) {
		u32 i = sorted_vals[pos];
		order[pos] = i; rank[i] = pos; mkeys[pos] = sorted_keys[pos];
		leaf_min[pos] = aabb_min[i]; leaf_max[pos] = aabb_max[i];
	}
}

// ---------------- K4: grid broadphase on top of the Morton order ----------------
// The Morton-sorted colliders are already sorted by octree cell at every level: the colliders of the level-j cell with integer
// coordinates (cx,cy,cz) are the contiguous range of sorted positions whose 48-bit code has the prefix morton(cx,cy,cz) >> 3j.
// Level j is chosen per step so that a cell is at least twice the mean AABB extent.  A collider whose extent (in quantised
// units, +2 for rounding) fits one cell is "small": two overlapping small colliders have min-corner cells that differ by at
// most 1 per axis, so a small collider only has to look into the 27 cells around its own (found through a hash table
// cell -> sorted range).  The few "large" colliders (the ground; also anything whose quantised corner wrapped past 65535,
// nudge.cpp:2613-2616 masks it) are tested against everybody by brute force.  The union is exactly the set of strictly
// overlapping pairs, reported once, oriented by Morton position like nudge.cpp:3495.
#define NB_GRID_EMPTY (~(u64)0)
NB_DEV u64 morton48_of(u32 x, u32 y, u32 z) {
	u32 lx, hx, ly, hy, lz, hz;
	dilate3(x, 2, lx, hx); dilate3(y, 1, ly, hy); dilate3(z, 0, lz, hz);
	return (u64)(lx | ly | lz) | ((u64)(hx | hy | hz) << 32);
}
NB_DEV u32 grid_hash(u64 prefix, u32 mask) { return (u32)((prefix * 0x9E3779B97F4A7C15ull) >> 32) & mask; }


__global__ void __launch_bounds__(NB_BLOCK) k_grid_build(u32 K, const u32* order, float4* leaf_min, const float4* leaf_max, const u64* mkeys,
		uint8_t* smallf, u32* large_list, u64* table_keys, u64* table_vals, u32 table_mask, u32* counts) {
	const MortonFrame f = morton_frame(counts);
	const u32 j = counts[CNT_GRID_LEVEL];
	for (u32 p = blockIdx.x * blockDim.x + threadIdx.x; p < K; p += gridDim.x * blockDim.x) {
		float4 lo = leaf_min[p], hi = leaf_max[p];
		u32 qx, qy, qz; morton_quantise(f, lo, order[p], qx, qy, qz);
		bool small = grid_level_needed(lo, hi, f.L[0]) <= j && qx < 65536u && qy < 65536u && qz < 65536u;  // NaN extents are "large" too
		smallf[p] = small ? 1 : 0;
		lo.w = small ? -INFINITY : INFINITY; leaf_min[p] = lo;  // k_grid_pairs reads the class with the box: 0 > lo.w <=> small
		if (!small) large_list[atomicAdd(&counts[CNT_LARGE], 1u)] = p;
		const u64 prefix = mkeys[p] >> (3 * j);
		if (p == 0 || (mkeys[p - 1] >> (3 * j)) != prefix) {  // first collider of its cell: publish the cell's range
			u32 e = p + 1;
			while (e < K && (mkeys[e] >> (3 * j)) == prefix) ++e;
			u32 slot = grid_hash(prefix, table_mask);
			while (true) {
				u64 old = atomicCAS((unsigned long long*)&table_keys[slot], (unsigned long long)NB_GRID_EMPTY, (unsigned long long)prefix);
				if (old == NB_GRID_EMPTY) break;
				slot = (slot + 1) & table_mask;
			}
			table_vals[slot] = (u64)p | ((u64)e << 32);
		}
	}
}

NB_DEV bool boxes_overlap(float4 alo, float4 ahi, float4 blo, float4 bhi) {  // strict, nudge.cpp:3306-3310 / 3386-3390
	return bhi.x > alo.x && ahi.x > blo.x && bhi.y > alo.y && ahi.y > blo.y && bhi.z > alo.z && ahi.z > blo.z;
}
NB_DEV void emit_pair(u32 p, u32 q, const u32* order, u32 kbits, u64* pair_keys, u32 max_pairs, u32* counts) {  // p < q: Morton positions
	u32 slot = warp_append_slot(&counts[CNT_PAIRS]);
	if (slot < max_pairs) pair_keys[slot] = ((u64)order[p] << kbits) | (u64)order[q];  // hi = earlier, lo = later (nudge.cpp:3495)
	else atomicOr(&counts[CNT_OVERFLOW], OVF_PAIRS);
}

// One warp per small collider.  Lanes 0..26 each look up one neighbouring cell (cells whose Morton prefix is below the
// collider's own hold only earlier positions and are skipped); the candidate ranges are then flattened with a warp scan and
// dealt round-robin to all 32 lanes, so the walk takes ceil(candidates / 32) steps however unevenly the cells are filled.
// Hits go to a per-warp shared buffer (shared-memory atomic for the slot) that is flushed to the pair list with one global
// atomic per ~64 pairs: one global atomic per pair would serialise on the counter.
#define NB_GP_BUF 128
__global__ void __launch_bounds__(NB_BLOCK) k_grid_pairs(u32 K, const u32* order, const float4* leaf_min, const float4* leaf_max, const uint8_t* smallf, const u64* mkeys,
		const u64* table_keys, const u64* table_vals, u32 table_mask, u32 kbits, u64* pair_keys, u32 max_pairs, u32* counts) {
	__shared__ u64 buf[NB_WARPS][NB_GP_BUF];
	__shared__ u32 fill[NB_WARPS];
	const MortonFrame f = morton_frame(counts);
	const u32 j = counts[CNT_GRID_LEVEL];
	const int ncell = 1 << (16 - j);
	const u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
	const int dx = (int)(lane % 3) - 1, dy = (int)((lane / 3) % 3) - 1, dz = (int)(lane / 9) - 1;
	if (lane == 0) fill[wid] = 0;
	__syncwarp();
	auto flush = [&]() {  // warp-converged
		u32 cnt = min(fill[wid], (u32)NB_GP_BUF), base = 0;
		if (lane == 0) base = atomicAdd(&counts[CNT_PAIRS], cnt);
		base = __shfl_sync(0xffffffffu, base, 0);
		for (u32 i = lane; i < cnt; i += 32) {
			if (base + i < max_pairs) pair_keys[base + i] = buf[wid][i];
			else atomicOr(&counts[CNT_OVERFLOW], OVF_PAIRS);
		}
		__syncwarp();
		if (lane == 0) fill[wid] = 0;
		__syncwarp();
	};
	for (u32 p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < K; p += nwarps) {  // p is warp-uniform
		if (!smallf[p]) continue;
		const float4 lo = leaf_min[p], hi = leaf_max[p];
		u32 qb = 0, len = 0;
		if (lane < 27) {
			u32 qx, qy, qz; morton_quantise(f, lo, order[p], qx, qy, qz);
			// a cell on the + side only matters if this box reaches into it (max corner quantised like the min corner, +1 for rounding)
			u32 hx, hy, hz; morton_quantise(f, hi, order[p], hx, hy, hz);
			const int cx = (int)(qx >> j), cy = (int)(qy >> j), cz = (int)(qz >> j);
			const bool reach = (dx <= 0 || ((hx + 1) >> j) > (u32)cx) && (dy <= 0 || ((hy + 1) >> j) > (u32)cy) && (dz <= 0 || ((hz + 1) >> j) > (u32)cz);
			const int nx = cx + dx, ny = cy + dy, nz = cz + dz;
			if (reach && nx >= 0 && ny >= 0 && nz >= 0 && nx < ncell && ny < ncell && nz < ncell) {
				const u64 prefix = morton48_of((u32)nx << j, (u32)ny << j, (u32)nz << j) >> (3 * j);
				if (prefix >= (mkeys[p] >> (3 * j))) {
					u32 slot = grid_hash(prefix, table_mask);
					u64 k;
					while ((k = table_keys[slot]) != prefix && k != NB_GRID_EMPTY) slot = (slot + 1) & table_mask;
					if (k != NB_GRID_EMPTY) {
						const u64 range = table_vals[slot];
						qb = max((u32)range, p + 1);  // each pair once: from its earlier Morton position
						const u32 qe = (u32)(range >> 32);
						len = qe > qb ? qe - qb : 0;
					}
				}
			}
		}
		const u32 incl = warp_incl_scan(len), off = incl - len, total = __shfl_sync(0xffffffffu, incl, 31);
		const u64 hi_key = (u64)order[p] << kbits;  // hi = earlier, lo = later (nudge.cpp:3495)
		for (u32 t0 = 0; t0 < total; t0 += 32) {
			const u32 t = t0 + lane;
			// cell of candidate t: the last lane whose offset is <= t (offsets are non-decreasing)
			u32 c = 0;
			#pragma unroll
			for (int step = 16; step; step >>= 1) {
				u32 probe = __shfl_sync(0xffffffffu, off, (c + step) & 31);
				if (c + step < 32 && probe <= t) c += step;
			}
			const u32 q = __shfl_sync(0xffffffffu, qb, c) + (t - __shfl_sync(0xffffffffu, off, c));
			bool hit = false;
			if (t < total) {
				const float4 a = __ldg(leaf_min + q), bq = __ldg(leaf_max + q);  // two 128-bit loads; a.w carries the class
				hit = (bq.x > lo.x) & (hi.x > a.x) & (bq.y > lo.y) & (hi.y > a.y) & (bq.z > lo.z) & (hi.z > a.z) & (0.0f > a.w);  // strict, nudge.cpp:3306-3310
			}
			if (hit) {
				u32 slot = atomicAdd(&fill[wid], 1u);
				if (slot < NB_GP_BUF) buf[wid][slot] = hi_key | (u64)order[q];
				else {  // more than a buffer of hits from one step: straight to the list
					u32 g = atomicAdd(&counts[CNT_PAIRS], 1u);
					if (g < max_pairs) pair_keys[g] = hi_key | (u64)order[q];
					else atomicOr(&counts[CNT_OVERFLOW], OVF_PAIRS);
				}
			}
			__syncwarp();
			if (fill[wid] > NB_GP_BUF - 32) flush();
		}
	}
	if (fill[wid]) flush();
}

__global__ void __launch_bounds__(NB_BLOCK) k_large_pairs(u32 K, const u32* order, const float4* leaf_min, const float4* leaf_max, const uint8_t* smallf,
		const u32* large_list, u32 kbits, u64* pair_keys, u32 max_pairs, u32* counts) {
	const u32 nlarge = counts[CNT_LARGE];
	for (u32 l = 0; l < nlarge; ++l) {
		const u32 pl = large_list[l];
		const float4 lo = leaf_min[pl], hi = leaf_max[pl];
		for (u32 q = blockIdx.x * blockDim.x + threadIdx.x; q < K; q += gridDim.x * blockDim.x) {
			if (q == pl || (!smallf[q] && q < pl)) continue;  // a pair of two large colliders is reported from the earlier one
			if (boxes_overlap(lo, hi, leaf_min[q], leaf_max[q])) emit_pair(min(pl, q), max(pl, q), order, kbits, pair_keys, max_pairs, counts);
		}
	}
}

// ---------------- islands: lock-free union-find, smaller index becomes the root (nudge.cpp:3500-3703, 3788-3971) ----------------
// Invariant: parent[x] <= x, and only a current root is ever hooked (by CAS) under a smaller index.  Finds therefore
// terminate and stay inside x's set even when they read stale L1 lines, so they use ordinary cacheable loads: the root
// of the one giant pile component is read by every thread and would otherwise serialise in a single L2 slice.
NB_DEV u32 uf_find(u32* parent, u32 x) {  // with path halving: every write points a node at one of its ancestors
	while (true) {
		u32 p = parent[x];
		if (p == x) return x;
		u32 gp = parent[p];
		if (gp == p) return p;
		parent[x] = gp;
		x = gp;
	}
}
NB_DEV u32 uf_find_fresh(u32* parent, u32 x) {  // L2-coherent reads, for the final flatten
	while (true) { u32 p = __ldcg(parent + x); if (p == x) return x; x = p; }
}
NB_DEV void uf_unite(u32* parent, u32 a, u32 b) {
	if (!a || !b) return;  // body 0 is the static world and is ignored (nudge.cpp:3517-3519, 3583-3585)
	while (true) {
		a = uf_find(parent, a); b = uf_find(parent, b);
		if (a == b) return;
		if (a < b) { u32 t = a; a = b; b = t; }
		u32 old = atomicCAS(&parent[a], a, b);
		if (old == a) return;
		a = old;  // a was not a root any more: continue from its real parent
	}
}
// Islands and sleeping (nudge.cpp:3500-3703, 3788-3971): a set is active iff ANY member is awake (idle counter != 0xff), so a set
// can only be inactive if ALL its bodies are asleep.  Hence only edges between two asleep bodies need a union; an edge between an
// asleep and an awake body "taints" the asleep one (its whole asleep component is then active), and edges between awake bodies
// carry no information.  The resulting active/inactive decision per body is exactly the reference's, at almost no cost while the
// scene is moving.  active[] is indexed by the root of a body's asleep-component (an awake body is its own root).
NB_DEV void island_edge(u32* parent, u32* taint, const uint8_t* idle, u32 a, u32 b) {
	if (!a || !b || a == b) return;  // body 0 is the static world and is ignored (nudge.cpp:3517-3519, 3583-3585)
	const bool sa = idle[a] == 0xff, sb = idle[b] == 0xff;
	if (sa && sb) uf_unite(parent, a, b);
	else if (sa) taint[a] = 1;
	else if (sb) taint[b] = 1;
}
__global__ void __launch_bounds__(NB_BLOCK) k_uf_init(u32* parent, u32* active, u32* taint, u32 B) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) { parent[i] = i; active[i] = 0; taint[i] = 0; }
}
__global__ void __launch_bounds__(NB_BLOCK) k_uf_union_conn(u32* parent, u32* taint, const uint8_t* idle, const nb_body_pair* conn, u32 n) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) island_edge(parent, taint, idle, conn[i].a, conn[i].b);
}
__global__ void __launch_bounds__(NB_BLOCK) k_uf_union_pairs(u32* parent, u32* taint, const uint8_t* idle, const u64* pair_keys, u32 kbits, const u32* col_body, const u32* counts) {
	u32 n = counts[CNT_PAIRS];
	u64 mask = ((u64)1 << kbits) - 1;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		u64 k = pair_keys[i];
		island_edge(parent, taint, idle, col_body[(u32)(k & mask)], col_body[(u32)(k >> kbits)]);
	}
}
__global__ void __launch_bounds__(NB_BLOCK) k_uf_union_contacts(u32* parent, u32* taint, const uint8_t* idle, const uint2* bodies, const u32* counts) {
	u32 n = counts[CNT_STAGED];
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) { uint2 ab = bodies[i]; island_edge(parent, taint, idle, ab.x, ab.y); }
}
__global__ void __launch_bounds__(NB_BLOCK) k_uf_flatten_active(u32* parent, u32* active, const u32* taint, const uint8_t* idle, u32 B) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
		u32 r = uf_find_fresh(parent, i);
		parent[i] = r;  // roots never change here, so concurrent flattening is benign
		if (i >= 1 && (idle[i] != 0xff || taint[i])) active[r] = 1;  // nudge.cpp:3669-3672
	}
}

// ---------------- coarse island filter + partition by shape type (nudge.cpp:3674-3751) ----------------
__global__ void __launch_bounds__(NB_BLOCK) k_pair_flags(const u64* pair_keys, u32 kbits, u32 nboxes, const u32* col_body, const u32* parent, const u32* active,
														 u32* flags /*[5][stride]*/, u32 stride, const u32* counts) {
	u32 n = counts[CNT_PAIRS];
	u64 mask = ((u64)1 << kbits) - 1;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		u64 k = pair_keys[i];
		u32 lo = (u32)(k & mask), hi = (u32)(k >> kbits);
		u32 a = col_body[lo], b = col_body[hi];
		int cls = -1;
		if (a != b) {
			u32 set = a ? parent[a] : parent[b];  // sets[0] = 0 and both bodies share a set (nudge.cpp:3663, 3688)
			cls = active[set] ? (int)((lo >= nboxes ? 1u : 0u) | (hi >= nboxes ? 2u : 0u)) : 4;
		}
		#pragma unroll
		for (int c = 0; c < 5; ++c) flags[c*stride + i] = (c == cls) ? 1u : 0u;
	}
}

__global__ void __launch_bounds__(NB_BLOCK) k_partition(const u64* pair_keys, u32 kbits, const u32* flags, const u32* block_sums, u32 stride,
														const u32* col_tag, uint2* live, u64* sleeping_pairs, u32* counts) {  // NB_SCAN_GRID blocks
	u32 n = counts[CNT_PAIRS];
	u64 mask = ((u64)1 << kbits) - 1;
	u32 base[4] = { 0, counts[CNT_LIVE0], counts[CNT_LIVE0] + counts[CNT_LIVE1], counts[CNT_LIVE0] + counts[CNT_LIVE1] + counts[CNT_LIVE2] };
	if (blockIdx.x == 0 && threadIdx.x == 0) counts[CNT_LIVE_TOTAL] = base[3] + counts[CNT_LIVE3];
	scan_consume<5>(flags, stride, n, block_sums, [&](u32 i, const u32 (&v)[5], const u32 (&off)[5]) {
		u64 k = pair_keys[i];
		u32 lo = (u32)(k & mask), hi = (u32)(k >> kbits);
		#pragma unroll
		for (int c = 0; c < 4; ++c)
			if (v[c]) live[base[c] + off[c]] = (c == 2) ? make_uint2(hi, lo) : make_uint2(lo, hi);  // bucket 2 halves swapped (nudge.cpp:3746-3751)
		if (v[4]) {
			u64 ta = col_tag[lo], tb = col_tag[hi];
			sleeping_pairs[off[4]] = ta > tb ? ta | (tb << 32) : tb | (ta << 32);  // nudge.cpp:3697
		}
	});
}

// ---------------- narrowphase: box-box (nudge.cpp:1177-2487) ----------------
struct BoxIn { xform t; float3 s; u32 tag; };

NB_DEV void rel_rotation(float4 qa, float4 qb, float* m) {  // nudge.cpp:1228-1268 / 1465-1505
	f3 t = cross3(mk3(qb.x, qb.y, qb.z), mk3(qa.x, qa.y, qa.z));
	float rx = qa.x*qb.w - qb.x*qa.w - t.x;
	float ry = qa.y*qb.w - qb.y*qa.w - t.y;
	float rz = qa.z*qb.w - qb.z*qa.w - t.z;
	float rs = qa.x*qb.x + qa.y*qb.y + qa.z*qb.z + qa.w*qb.w;
	float kx = rx + rx, ky = ry + ry, kz = rz + rz;
	float xx = kx*rx, yy = ky*ry, zz = kz*rz, xy = kx*ry, xz = kx*rz, yz = ky*rz, sx = kx*rs, sy = ky*rs, sz = kz*rs;
	m[0] = 1.0f - yy - zz; m[1] = xy + sz; m[2] = xz - sy;
	m[3] = xy - sz; m[4] = 1.0f - xx - zz; m[5] = yz + sx;
	m[6] = xz + sy; m[7] = yz - sx; m[8] = 1.0f - xx - yy;
}

// Selects with run-time k: indexing a register array with a run-time value would move the array to local memory.
NB_DEV float sel3(float x, float y, float z, u32 k) { return k == 0 ? x : (k == 1 ? y : z); }
NB_DEV float sel3(float3 v, u32 k) { return sel3(v.x, v.y, v.z, k); }

// Pass 1: most separating face, nudge.cpp:1195-1410.  Returns false if separated; may swap a/b.
NB_DEV bool bb_faces(const BoxIn& A, const BoxIn& B, float& pen, u32& face, bool& swapped) {
	float m[9]; rel_rotation(A.t.q, B.t.q, m);
	float vx_x = nb_abs(m[0]), vx_y = nb_abs(m[1]), vx_z = nb_abs(m[2]);
	float vy_x = nb_abs(m[3]), vy_y = nb_abs(m[4]), vy_z = nb_abs(m[5]);
	float vz_x = nb_abs(m[6]), vz_y = nb_abs(m[7]), vz_z = nb_abs(m[8]);
	float3 sa = A.s, sb = B.s;
	float pax = sb.x + vx_x*sa.x + vy_x*sa.y + vz_x*sa.z;
	float pay = sb.y + vx_y*sa.x + vy_y*sa.y + vz_y*sa.z;
	float paz = sb.z + vx_z*sa.x + vy_z*sa.y + vz_z*sa.z;
	float pbx = sa.x + vx_x*sb.x + vx_y*sb.y + vx_z*sb.z;
	float pby = sa.y + vy_x*sb.x + vy_y*sb.y + vy_z*sb.z;
	float pbz = sa.z + vz_x*sb.x + vz_y*sb.y + vz_z*sb.z;
	f3 delta = mk3(A.t.p.x - B.t.p.x, A.t.p.y - B.t.p.y, A.t.p.z - B.t.p.z);
	f3 qa = mk3(A.t.q.x, A.t.q.y, A.t.q.z), qb = mk3(B.t.q.x, B.t.q.y, B.t.q.z);
	f3 t = cross3(qb, delta); t = add3(t, t);
	f3 u = cross3(qb, t);
	pax -= nb_abs(u.x + delta.x - B.t.q.w*t.x); pay -= nb_abs(u.y + delta.y - B.t.q.w*t.y); paz -= nb_abs(u.z + delta.z - B.t.q.w*t.z);
	t = cross3(delta, qa); t = add3(t, t);
	u = cross3(qa, t);
	pbx -= nb_abs(u.x - delta.x - A.t.q.w*t.x); pby -= nb_abs(u.y - delta.y - A.t.q.w*t.y); pbz -= nb_abs(u.z - delta.z - A.t.q.w*t.z);
	float payz = nb_min(pay, paz), pbyz = nb_min(pby, pbz);
	float pa = nb_min(pax, payz), pb = nb_min(pbx, pbyz);
	float p = nb_min(pa, pb);
	u32 aface = (payz == pa ? 1u : 0u) + (paz == pa ? 1u : 0u);
	u32 bface = (pbyz == pb ? 1u : 0u) + (pbz == pb ? 1u : 0u);
	swapped = pa == p;  // nudge.cpp:1381-1387
	face = swapped ? aface : bface;
	pen = p;
	return p > 0.0f;
}

struct ContactOut { float4* data; uint2* bodies; u64* tags; u32* features; };

NB_DEV void put_contact(const ContactOut& o, u32 at, float px, float py, float pz, float pen, float nx, float ny, float nz, u32 a, u32 b, u64 tag, u32 feature) {
	o.data[2*at + 0] = make_float4(px, py, pz, pen);
	o.data[2*at + 1] = make_float4(nx, ny, nz, 0.5f);  // friction is fixed: nudge.cpp:2105, 2456, 2515, 2598
	o.bodies[at] = make_uint2(a, b);
	o.tags[at] = tag; o.features[at] = feature;
}

// Pass 3: edge-edge closest points, nudge.cpp:2157-2479.
NB_DEV void bb_edge(const BoxIn& A, const BoxIn& B, float pen, u32 edge, const ContactOut& out, u32 at, const u32* s_rsqrt) {
	float ab[3][3], bb[3][3];
	#pragma unroll
	for (int w = 0; w < 2; ++w) {
		float4 q = w ? B.t.q : A.t.q;
		float kx = q.x + q.x, ky = q.y + q.y, kz = q.z + q.z;
		float xx = kx*q.x, yy = ky*q.y, zz = kz*q.z, xy = kx*q.y, xz = kx*q.z, yz = ky*q.z, sx = kx*q.w, sy = ky*q.w, sz = kz*q.w;
		float (*m)[3] = w ? bb : ab;
		m[0][0] = 1.0f - yy - zz; m[0][1] = xy + sz; m[0][2] = xz - sy;
		m[1][0] = xy - sz; m[1][1] = 1.0f - xx - zz; m[1][2] = yz + sx;
		m[2][0] = xz + sy; m[2][1] = yz - sx; m[2][2] = 1.0f - xx - yy;
	}
	u32 ua = (edge & 2) ? 2 : ((edge & 1) ? 1 : 0);                       // blendv on shifted bits, nudge.cpp:2257-2278
	u32 ub = (edge & (2u << 16)) ? 2 : ((edge & (1u << 16)) ? 1 : 0);
	f3 u = mk3(sel3(ab[0][0], ab[1][0], ab[2][0], ua), sel3(ab[0][1], ab[1][1], ab[2][1], ua), sel3(ab[0][2], ab[1][2], ab[2][2], ua));
	f3 v = mk3(sel3(bb[0][0], bb[1][0], bb[2][0], ub), sel3(bb[0][1], bb[1][1], bb[2][1], ub), sel3(bb[0][2], bb[1][2], bb[2][2], ub));
	f3 n = cross3(u, v);
	f3 delta = mk3(B.t.p.x - A.t.p.x, B.t.p.y - A.t.p.y, B.t.p.z - A.t.p.z);
	u32 flip = asu(n.x*delta.x + n.y*delta.y + n.z*delta.z) & NB_SIGN;
	n.x = nb_xor(n.x, flip); n.y = nb_xor(n.y, flip); n.z = nb_xor(n.z, flip);
	float sa[3] = { A.s.x, A.s.y, A.s.z }, sb[3] = { B.s.x, B.s.y, B.s.z };
	u32 asg[3], bsg[3];
	#pragma unroll
	for (int k = 0; k < 3; ++k) {
		asg[k] = asu(ab[k][0]*n.x + ab[k][1]*n.y + ab[k][2]*n.z) & NB_SIGN;
		bsg[k] = asu(bb[k][0]*n.x + bb[k][1]*n.y + bb[k][2]*n.z) & NB_SIGN;
	}
	u32 edge_x = (asg[0] >> 31) | ((bsg[0] ^ NB_SIGN) >> 15);
	u32 edge_y = (asg[1] >> 30) | ((bsg[1] ^ NB_SIGN) >> 14);
	u32 edge_z = (asg[2] >> 29) | ((bsg[2] ^ NB_SIGN) >> 13);
	u32 elo = edge & 0xffff, ehi = edge >> 16;  // per 16-bit lane (e + 1) + (e >> 1) == 1 << e for e in 0..2 (nudge.cpp:2381)
	u32 edge_w = (((elo + 1) + (elo >> 1)) & 0xffff) | ((((ehi + 1) + (ehi >> 1)) & 0xffff) << 16);
	u32 tag_hi = edge_x | edge_y | edge_z | edge_w;
	u32 tag_lo = tag_hi & ~edge_w;
	u32 tag = tag_lo | (tag_hi << 8);
	#pragma unroll
	for (int k = 0; k < 3; ++k) { sa[k] = nb_xor(sa[k], asg[k]); sb[k] = nb_xor(sb[k], bsg[k]); }
	#pragma unroll
	for (int k = 0; k < 3; ++k)
		#pragma unroll
		for (int j = 0; j < 3; ++j) { ab[k][j] *= sa[k]; bb[k][j] *= sb[k]; }
	float apos[3] = { A.t.p.x, A.t.p.y, A.t.p.z }, bpos[3] = { B.t.p.x, B.t.p.y, B.t.p.z };
	float ca[3], cb[3], o[3];
	#pragma unroll
	for (int j = 0; j < 3; ++j) {
		ca[j] = ab[0][j] + ab[1][j] + ab[2][j] + apos[j];
		cb[j] = bb[0][j] + bb[1][j] + bb[2][j] - bpos[j];  // negated on purpose (nudge.cpp:2428)
		o[j] = ca[j] + cb[j];
	}
	float ia = u.x*u.x + u.y*u.y + u.z*u.z;
	float ib = u.x*v.x + u.y*v.y + u.z*v.z;
	float ic = v.x*v.x + v.y*v.y + v.z*v.z;
	float id = o[0]*u.x + o[1]*u.y + o[2]*u.z;
	float ie = o[0]*v.x + o[1]*v.y + o[2]*v.z;
	float ir = 0.5f / (ia*ic - ib*ib);
	float s_a = (ib*ie - ic*id) * ir;
	float s_b = (ia*ie - ib*id) * ir;
	float px = (ca[0] - cb[0])*0.5f + u.x*s_a + v.x*s_b;
	float py = (ca[1] - cb[1])*0.5f + u.y*s_a + v.y*s_b;
	float pz = (ca[2] - cb[2])*0.5f + u.z*s_a + v.z*s_b;
	float fn = nb_rsqrt_t(n.x*n.x + n.y*n.y + n.z*n.z, s_rsqrt);  // nudge.cpp:842-847, 2453
	put_contact(out, at, px, py, pz, pen, n.x*fn, n.y*fn, n.z*fn, asu(A.t.p.w), asu(B.t.p.w), (u64)A.tag | ((u64)B.tag << 32), tag);
}

NB_DEV bool sphere_sphere(float ra, float rb, xform ta, xform tb, float* o /* p[3], pen, n[3] */) {  // nudge.cpp:2489-2521
	float r = ra + rb;
	f3 pa = mk3(ta.p.x, ta.p.y, ta.p.z);
	f3 dp = sub3(mk3(tb.p.x, tb.p.y, tb.p.z), pa);
	float l2 = dot3(dp, dp);
	if (l2 > r*r) return false;
	f3 n;
	float l = sqrtf(l2);
	if (l2 > 1e-4f) n = mul3(dp, 1.0f / l);
	else n = mk3(1.0f, 0.0f, 0.0f);
	f3 p = add3(pa, mul3(n, l - rb));
	o[0] = p.x; o[1] = p.y; o[2] = p.z; o[3] = r - l; o[4] = n.x; o[5] = n.y; o[6] = n.z;
	return true;
}

NB_DEV bool box_sphere(float3 size, float radius, xform ta, xform tb, float* o) {  // nudge.cpp:2523-2604
	quat a_to_world = mkq(ta.q);
	quat world_to_a = a_to_world; world_to_a.v.x = -world_to_a.v.x; world_to_a.v.y = -world_to_a.v.y; world_to_a.v.z = -world_to_a.v.z;
	f3 apos = mk3(ta.p.x, ta.p.y, ta.p.z);
	f3 offset_b = qrot(world_to_a, sub3(mk3(tb.p.x, tb.p.y, tb.p.z), apos));
	float dx = fabsf(offset_b.x), dy = fabsf(offset_b.y), dz = fabsf(offset_b.z);
	float w = size.x + radius, h = size.y + radius, d = size.z + radius;
	if (dx >= w || dy >= h || dz >= d) return false;
	f3 n; float penetration; float r = radius;
	u32 outside_x = dx > size.x, outside_y = dy > size.y, outside_z = dz > size.z;
	if (outside_x + outside_y + outside_z >= 2) {
		f3 corner = mk3(outside_x ? (offset_b.x > 0.0f ? size.x : -size.x) : offset_b.x,
						outside_y ? (offset_b.y > 0.0f ? size.y : -size.y) : offset_b.y,
						outside_z ? (offset_b.z > 0.0f ? size.z : -size.z) : offset_b.z);
		f3 dp = sub3(offset_b, corner);
		float l2 = dot3(dp, dp);
		if (l2 > r*r) return false;
		float l = sqrtf(l2);
		float m = 1.0f / l;
		n = mul3(dp, m);
		penetration = r - l;
	}
	else if (w - dx < h - dy && w - dx < d - dz) { n = mk3(offset_b.x > 0.0f ? 1.0f : -1.0f, 0.0f, 0.0f); penetration = w - dx; }
	else if (h - dy < d - dz) { n = mk3(0.0f, offset_b.y > 0.0f ? 1.0f : -1.0f, 0.0f); penetration = h - dy; }
	else { n = mk3(0.0f, 0.0f, offset_b.z > 0.0f ? 1.0f : -1.0f); penetration = d - dz; }
	f3 p = sub3(offset_b, mul3(n, r));
	p = add3(qrot(a_to_world, p), apos);
	n = qrot(a_to_world, n);
	o[0] = p.x; o[1] = p.y; o[2] = p.z; o[3] = penetration; o[4] = n.x; o[5] = n.y; o[6] = n.z;
	return true;
}

NB_DEV BoxIn load_box(const nb_transform* world_xf, const nb_box_collider* box_data, const u32* col_tag, u32 i) {
	BoxIn b;
	b.t = ld_xform(world_xf, i);
	float4 s = reinterpret_cast<const float4*>(box_data)[i];
	b.s = make_float3(s.x, s.y, s.z);
	b.tag = col_tag[i];
	return b;
}

// Box-box pair j of the live list; a owns the most separating face (nudge.cpp:1381-1387)
NB_DEV void load_pair(const uint2* live, const u32* np_info, const nb_transform* world_xf, const nb_box_collider* box_data, const u32* col_tag, u32 j,
					  BoxIn& A, BoxIn& B) {
	uint2 pr = live[j];
	bool swapped = np_info[j] & 4;
	A = load_box(world_xf, box_data, col_tag, swapped ? pr.y : pr.x); B = load_box(world_xf, box_data, col_tag, swapped ? pr.x : pr.y);
}

// The narrowphase runs in three passes so that the expensive face clipping only runs on the pairs that need it:
//   k_np_faces  every live pair, one thread per pair: box-box -> pass 1 (face SAT, cheap, rejects ~85 %); sphere pairs -> the whole (cheap) test
//   k_np_clip   surviving box-box pairs (compacted), four lanes per pair: pass 2 (+ pass 3 for edge contacts) -> contacts in a scratch buffer + counts
//   k_np_emit   moves the scratch contacts (and computes the sphere contacts) to the scanned offsets, in the reference's contact order
//               (box-box face contacts, box-box edge contacts, box-sphere, sphere-sphere: nudge.cpp:3753-3786)

__global__ void __launch_bounds__(NB_BLOCK) k_np_faces(const uint2* live, u32 nboxes, const nb_transform* world_xf, const nb_box_collider* box_data,
		const nb_sphere_collider* sph_data, const u32* col_tag, u32* cnt /*[4][stride]: face, edge, other, survivor*/, u32 stride, float* np_pen, u32* np_info, u32* counts) {
	u32 n = counts[CNT_LIVE_TOTAL];
	u32 n_bb = counts[CNT_LIVE0], n_bs_end = n_bb + counts[CNT_LIVE1] + counts[CNT_LIVE2];
	for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
		uint2 pr = live[j];  // x = low half, y = high half of the reference's pair word
		u32 surv = 0, other = 0;
		if (j < n_bb) {
			BoxIn A = load_box(world_xf, box_data, col_tag, pr.x), B = load_box(world_xf, box_data, col_tag, pr.y);  // a = low, b = high (nudge.cpp:1202-1203)
			float pen; u32 face; bool swapped;
			if (bb_faces(A, B, pen, face, swapped)) { surv = 1; np_pen[j] = pen; np_info[j] = face | (swapped ? 4u : 0u); }
		}
		else {
			float o[7];
			u32 a = pr.y, b = pr.x;  // a = high half, b = low half (nudge.cpp:3759-3760, 3775-3776)
			xform ta = ld_xform(world_xf, a), tb = ld_xform(world_xf, b);
			bool hit;
			if (j < n_bs_end) { float4 sz = reinterpret_cast<const float4*>(box_data)[a]; hit = box_sphere(make_float3(sz.x, sz.y, sz.z), sph_data[b - nboxes].radius, ta, tb, o); }
			else hit = sphere_sphere(sph_data[a - nboxes].radius, sph_data[b - nboxes].radius, ta, tb, o);
			other = hit ? 1u : 0u;
		}
		cnt[0*stride + j] = 0; cnt[1*stride + j] = 0; cnt[2*stride + j] = other; cnt[3*stride + j] = surv;
	}
	if (blockIdx.x == 0 && threadIdx.x == 0) counts[CNT_TMP] = 0;
}

__global__ void __launch_bounds__(NB_BLOCK) k_np_list(const u32* cnt, const u32* block_sums, u32 stride, u32* np_list, const u32* counts) {  // NB_SCAN_GRID blocks
	scan_consume<1>(cnt + 3 * (size_t)stride, 0, counts[CNT_LIVE0], block_sums, [&](u32 j, const u32 (&v)[1], const u32 (&off)[1]) { if (v[0]) np_list[off[0]] = j; });
}

// Passes 2 and 3 (nudge.cpp:1432-2479) for one pair, run by a group of four lanes; the whole warp calls this together.  The reference
// computes the face clipper's 16 candidate points as SIMD lanes (nudge.cpp:1810-1970): the corners of a's face (points 0-3) and of
// b's face (4-7), and the near (8-11) and far (12-15) intersections of b's edges with a's face.  Lane q of the group takes points q,
// 4 + q, 8 + q and 12 + q, which all follow from corner q and edge q.  A owns the most separating face.  The group's contacts go to
// consecutive slots reserved from `reserve` with one atomic per warp, in point order; `at` returns the first slot, n_face / n_edge
// the counts.  A group with !valid computes on whatever it was given and writes nothing.
NB_DEV void bb_clip(const BoxIn& A, const BoxIn& B, float face_penetration, u32 a_face, bool valid, const u32* s_rsqrt,
					u32* reserve, const ContactOut& out, u32 limit, u32& at, u32& n_face, u32& n_edge) {
	const u32 ALL = 0xffffffffu, lane = threadIdx.x & 31, q = lane & 3;
	float a_to_b[9]; rel_rotation(A.t.q, B.t.q, a_to_b);
	float3 sa = A.s, sb = B.s;
	f3 delta = mk3(A.t.p.x - B.t.p.x, A.t.p.y - B.t.p.y, A.t.p.z - B.t.p.z);
	f3 qa = mk3(A.t.q.x, A.t.q.y, A.t.q.z);
	f3 t = cross3(delta, qa); t = add3(t, t);
	f3 u = cross3(qa, t);
	float3 b_offset = make_float3(u.x - delta.x - A.t.q.w*t.x, u.y - delta.y - A.t.q.w*t.y, u.z - delta.z - A.t.q.w*t.z);

	// Edge axes (nudge.cpp:1578-1640): lane c = min(q, 2) takes column c of a_to_b (a's edge c) and row c (b's edge c), as the
	// reference's loop iteration i = c does.  Axis (i, j) is then p = epa[i*3 + j] + epb[j*3 + i] with epa from lane i, epb from lane j.
	const u32 c = min(q, 2u);
	float epa[3], epb[3];
	{
		float acx = sel3(a_to_b[0], a_to_b[1], a_to_b[2], c), acy = sel3(a_to_b[3], a_to_b[4], a_to_b[5], c), acz = sel3(a_to_b[6], a_to_b[7], a_to_b[8], c);
		float bcx = sel3(a_to_b[0], a_to_b[3], a_to_b[6], c), bcy = sel3(a_to_b[1], a_to_b[4], a_to_b[7], c), bcz = sel3(a_to_b[2], a_to_b[5], a_to_b[8], c);
		float ac2x = acx*acx, ac2y = acy*acy, ac2z = acz*acz;
		float bc2x = bcx*bcx, bc2y = bcy*bcy, bc2z = bcz*bcz;
		float aacx = nb_abs(acx), aacy = nb_abs(acy), aacz = nb_abs(acz);
		float abcx = nb_abs(bcx), abcy = nb_abs(bcy), abcz = nb_abs(bcz);
		float ra[3] = { ac2y + ac2z, ac2z + ac2x, ac2x + ac2y };
		float rb[3] = { bc2y + bc2z, bc2z + bc2x, bc2x + bc2y };
		#pragma unroll
		for (int k = 0; k < 3; ++k) {  // rsqrt | cmp_le -> NaN for degenerate axes (nudge.cpp:1611-1619)
			ra[k] = asf(asu(nb_rsqrt_t(ra[k], s_rsqrt)) | (ra[k] <= 1e-3f ? 0xffffffffu : 0u));
			rb[k] = asf(asu(nb_rsqrt_t(rb[k], s_rsqrt)) | (rb[k] <= 1e-3f ? 0xffffffffu : 0u));
		}
		float pa0 = aacy*sa.z + aacz*sa.y, pa1 = aacz*sa.x + aacx*sa.z, pa2 = aacx*sa.y + aacy*sa.x;
		float pb0 = abcy*sb.z + abcz*sb.y, pb1 = abcz*sb.x + abcx*sb.z, pb2 = abcx*sb.y + abcy*sb.x;
		float o0 = nb_abs(acy*b_offset.z - acz*b_offset.y);
		float o1 = nb_abs(acz*b_offset.x - acx*b_offset.z);
		float o2 = nb_abs(acx*b_offset.y - acy*b_offset.x);
		epa[0] = (pa0 - o0) * ra[0]; epa[1] = (pa1 - o1) * ra[1]; epa[2] = (pa2 - o2) * ra[2];
		epb[0] = pb0 * rb[0]; epb[1] = pb1 * rb[1]; epb[2] = pb2 * rb[2];
	}
	u32 a_edge = 0, b_edge = 0;
	float penetration = face_penetration;
	#pragma unroll
	for (int i = 0; i < 3; ++i)
		#pragma unroll
		for (int j = 0; j < 3; ++j) {  // the reference's fold in order (nudge.cpp:1647-1657): the first minimum wins, NaN never does
			float p = __shfl_sync(ALL, epa[j], i, 4) + __shfl_sync(ALL, epb[i], j, 4);
			bool mk = penetration > p;
			penetration = nb_min(penetration, p);
			if (mk) { a_edge = j; b_edge = i; }
		}
	bool is_edge = face_penetration > penetration + 1e-3f;  // nudge.cpp:1659-1661
	const u32 kind = (!valid || !(penetration > 0.0f)) ? 0 : (is_edge ? 2 : 1);  // 0 = separated, 1 = face contacts, 2 = edge contact

	// ---- face-face: nudge.cpp:1678-2112 ----
	u32 mask = 0, b_face, b_positive_face_bit, b_offset_neg;
	bool axis_near, axis_far;
	float d0, d1, d2, d3, px[4], py[4], pz[4], pen[4];
	{  // every group clips, whatever its kind, so that the warp stays converged at the shuffles; kind decides what is written
		float dirs0 = nb_abs(sel3(a_to_b[0], a_to_b[3], a_to_b[6], a_face));
		float dirs1 = nb_abs(sel3(a_to_b[1], a_to_b[4], a_to_b[7], a_face));
		float dirs2 = nb_abs(sel3(a_to_b[2], a_to_b[5], a_to_b[8], a_face));
		bool bit1 = dirs1 >= nb_max(dirs2, dirs0), bit2 = dirs2 >= nb_max(dirs1, dirs0);  // nudge.cpp:1721-1723
		float c0[3] = { a_to_b[0] * sb.x, a_to_b[3] * sb.x, a_to_b[6] * sb.x };
		float c1[3] = { a_to_b[1] * sb.y, a_to_b[4] * sb.y, a_to_b[7] * sb.y };
		float c2[3] = { a_to_b[2] * sb.z, a_to_b[5] * sb.z, a_to_b[8] * sb.z };
		b_face = bit2 ? 2 : (bit1 ? 1 : 0);
		float cc[3], dx[3], dy[3];
		#pragma unroll
		for (int k = 0; k < 3; ++k) {
			cc[k] = bit2 ? c2[k] : (bit1 ? c1[k] : c0[k]);
			dx[k] = bit2 ? c0[k] : (bit1 ? c2[k] : c1[k]);
			dy[k] = bit2 ? c1[k] : (bit1 ? c0[k] : c2[k]);
		}
		float b_offset_a = sel3(b_offset, a_face);
		b_positive_face_bit = ((asu(b_offset_a) ^ asu(sel3(cc[0], cc[1], cc[2], a_face))) >> 31) << a_face;
		b_offset_neg = (asu(b_offset_a) >> 31) << a_face;
		#pragma unroll
		for (int k = 0; k < 3; ++k) if (!b_positive_face_bit) cc[k] = nb_neg(cc[k]);
		cc[0] += b_offset.x; cc[1] += b_offset.y; cc[2] += b_offset.z;

		u32 X = (a_face + 1) % 3, Y = (a_face + 2) % 3, Z = a_face;
		float sx = sel3(sa, X), sy = sel3(sa, Y), cx = sel3(cc[0], cc[1], cc[2], X), cy = sel3(cc[0], cc[1], cc[2], Y);
		d0 = sel3(dx[0], dx[1], dx[2], X); d1 = sel3(dx[0], dx[1], dx[2], Y); d2 = sel3(dy[0], dy[1], dy[2], X); d3 = sel3(dy[0], dy[1], dy[2], Y);

		// corner q and edge q (nudge.cpp:1814-1890)
		const u32 npnp = (q & 1) ? 0u : NB_SIGN, pnpn = npnp ^ NB_SIGN, nnpp = q < 2 ? NB_SIGN : 0u;
		float k0 = cx*d3 - cy*d2, k1 = cx*d1 - cy*d0, k2 = d0*d3 - d1*d2;  // nudge.cpp:1814-1815
		float ox = k0, oy = k1, delta_max = nb_abs(k2);
		float sd0 = d0*sy, sd1 = d1*sx, sd2 = d2*sy, sd3 = d3*sx;           // nudge.cpp:1821
		float corner1x = cx + nb_xor(d0, npnp) + nb_xor(d2, nnpp);
		float corner1y = cy + nb_xor(d1, npnp) + nb_xor(d3, nnpp);
		float delta_x = ox + nb_xor(sd2, nnpp) + nb_xor(sd3, npnp);
		float delta_y = oy + nb_xor(sd0, nnpp) + nb_xor(sd1, npnp);
		bool mask0 = nb_max(nb_abs(delta_x), nb_abs(delta_y)) <= delta_max;
		bool mask1 = (nb_abs(corner1x) <= sx) && (nb_abs(corner1y) <= sy);
		float offset_x = q < 2 ? d0 : d2, offset_y = q < 2 ? d1 : d3;
		float pivot_x = cx + nb_xor(q < 2 ? d2 : d0, npnp);
		float pivot_y = cy + nb_xor(q < 2 ? d3 : d1, npnp);
		float pos_x = asf((asu(offset_x) & NB_SIGN) | asu(sx));  // copy sign: nudge.cpp:1858-1859
		float pos_y = asf((asu(offset_y) & NB_SIGN) | asu(sy));
		float rx = 1.0f / offset_x, ry = 1.0f / offset_y;          // nudge.cpp:1849
		float near_x = (pos_x + pivot_x) * rx, far_x = (pos_x - pivot_x) * rx;
		float near_y = (pos_y + pivot_y) * ry, far_y = (pos_y - pivot_y) * ry;
		float ea = nb_min(1.0f, near_x), eb = nb_min(1.0f, far_x);
		axis_near = ea > near_y; axis_far = eb > far_y;
		ea = nb_min(ea, near_y); eb = nb_min(eb, far_y);
		bool mm = (ea + eb) > 0.0f;
		bool mask_a = !(ea == 1.0f) && mm;  // _mm_cmpneq_ps is unordered: true on NaN (nudge.cpp:328-330, 1886)
		bool mask_b = !(eb == 1.0f) && mm;
		// an edge intersection is dropped when both vertices of its edge are inside (nudge.cpp:1834-1836)
		u32 corners = (mask0 ? 1u << q : 0u) | (mask1 ? 0x10u << q : 0u);  // bits 0-3: a's corners, 4-7: b's corners
		corners |= __shfl_xor_sync(ALL, corners, 1, 4);
		corners |= __shfl_xor_sync(ALL, corners, 2, 4);
		u32 need_a = (0xC35Au >> (4*q)) & 0xfu, need_b = (0xA5C3u >> (4*q)) & 0xfu;
		bool pre_a = (corners & need_a) == need_a, pre_b = ((corners >> 4) & need_b) == need_b;
		float x[4] = { nb_xor(sx, pnpn), corner1x, pivot_x - offset_x * ea, pivot_x + offset_x * eb };
		float y[4] = { nb_xor(sy, nnpp), corner1y, pivot_y - offset_y * ea, pivot_y + offset_y * eb };
		bool in[4] = { mask0, mask1, !pre_a && mask_a, !pre_b && mask_b };

		// z-plane through face b: nudge.cpp:1973-2019
		float dxt[3] = { d0, d1, sel3(dx[0], dx[1], dx[2], Z) }, dyt[3] = { d2, d3, sel3(dy[0], dy[1], dy[2], Z) }, ct[3] = { cx, cy, sel3(cc[0], cc[1], cc[2], Z) };
		float zn0 = dxt[1]*dyt[2] - dxt[2]*dyt[1];
		float zn1 = dxt[2]*dyt[0] - dxt[0]*dyt[2];
		float zn2 = dxt[0]*dyt[1] - dxt[1]*dyt[0];
		float dt = ct[0]*zn0 + ct[1]*zn1 + ct[2]*zn2;
		float inv = 1.0f / zn2;
		float plane0 = nb_neg(zn0) * inv, plane1 = nb_neg(zn1) * inv, plane2 = dt * inv;
		u32 z_sign = b_offset_neg ? NB_SIGN : 0;
		float penetration_offset = sel3(sa, Z);
		#pragma unroll
		for (int g = 0; g < 4; ++g) {
			float z = x[g]*plane0 + y[g]*plane1 + plane2;
			pen[g] = penetration_offset - nb_xor(z, z_sign);
			z += pen[g] * nb_xor(0.5f, z_sign);
			px[g] = x[g]; py[g] = y[g]; pz[g] = z;
			if (in[g] && pen[g] > 0.0f) mask |= 1u << (4*g + q);
		}
		mask |= __shfl_xor_sync(ALL, mask, 1, 4);
		mask |= __shfl_xor_sync(ALL, mask, 2, 4);
	}
	if (kind != 1) mask = 0;
	n_face = __popc(mask);
	n_edge = kind == 2 ? 1 : 0;

	// the warp's slots: an exclusive scan of the groups' counts and one atomic
	const u32 want = q == 0 ? n_face + n_edge : 0;
	const u32 incl = warp_incl_scan(want);
	u32 base = 0;
	if (lane == 31 && incl) base = atomicAdd(reserve, incl);
	base = __shfl_sync(ALL, base, 31);
	at = __shfl_sync(ALL, base + incl - want, lane & 28);

	if (kind == 1) {
		// labels: nudge.cpp:1902-1970
		u32 a_sign_face_bit = b_offset_neg ? (1u << a_face) : 0;
		u32 b_sign_face_bit = b_positive_face_bit ? 0 : (1u << b_face);
		u32 b_vertices = 0x00122436u >> (3 - b_face);
		u32 bv = q == 0 ? (b_vertices << 16) : (q == 1 ? (b_vertices << 8) : (q == 2 ? b_vertices : (b_vertices >> 8)));
		u32 winding = (asu(d0) >> 31) | ((asu(d1) >> 31) << 1) | ((asu(d2) >> 31) << 2) | ((asu(d3) >> 31) << 3);
		u64 a_edge_map = 0x1200362424003612llu >> (3 - a_face), b_edge_map = 0x2400361212003624llu >> (3 - b_face);
		u32 face_bits = a_sign_face_bit | (a_sign_face_bit << 8) | (b_sign_face_bit << 16) | (b_sign_face_bit << 24);
		u32 b_edge_q = ((u32)((b_edge_map >> (q << 4)) & 0x0707) << 16) | face_bits;
		u32 st[4];
		st[0] = (((0x12003624u >> (3 - a_face)) >> (8 * q)) & 0x7) | 0xffff0000u | a_sign_face_bit;
		st[1] = (bv & 0x70000) | 0x0000ffffu | (b_sign_face_bit << 16);
		#pragma unroll
		for (int g = 2; g < 4; ++g) {
			bool is_far = g == 3;
			u32 w = is_far ? (winding ^ 0xf) : winding;
			u32 yb = (is_far ? axis_far : axis_near) ? 1u : 0u;
			u32 e = yb*2 + ((w >> ((q < 2 ? 0 : 2) + yb)) & 1);
			st[g] = (u32)((a_edge_map >> (e << 4)) & 0x0707) | b_edge_q;
		}

		// a to world: nudge.cpp:2028-2056 (the diagonal is built as -((p + q) - 1))
		float w0[3], w1[3], w2[3];
		{
			float qx = A.t.q.x, qy = A.t.q.y, qz = A.t.q.z, qs = A.t.q.w;
			float kx = qx + qx, ky = qy + qy, kz = qz + qz, ks = nb_neg(qs + qs);
			w0[0] = nb_neg((ky*qy + kz*qz) - 1.0f); w0[1] = kx*qy + kz*qs; w0[2] = kx*qz + ks*qy;
			w1[0] = kx*qy + ks*qz; w1[1] = nb_neg((kz*qz + kx*qx) - 1.0f); w1[2] = ky*qz + kx*qs;
			w2[0] = kx*qz + ky*qs; w2[1] = ky*qz + ks*qx; w2[2] = nb_neg((kx*qx + ky*qy) - 1.0f);
		}
		float wn[3];
		#pragma unroll
		for (int k = 0; k < 3; ++k) wn[k] = a_face == 0 ? w0[k] : (a_face == 1 ? w1[k] : w2[k]);
		u32 a_body = asu(A.t.p.w), b_body = asu(B.t.p.w);
		u32 a_tag = A.tag, b_tag = B.tag;
		bool tag_swap = b_tag > a_tag;  // nudge.cpp:2074-2087
		u32 n_flip = (b_offset_neg ? NB_SIGN : 0u) ^ (tag_swap ? NB_SIGN : 0u);
		float nx = nb_xor(wn[0], n_flip), ny = nb_xor(wn[1], n_flip), nz = nb_xor(wn[2], n_flip);
		u64 high_tag = tag_swap ? (u64)b_tag | ((u64)a_tag << 32) : (u64)a_tag | ((u64)b_tag << 32);
		if (tag_swap) { u32 tt = a_body; a_body = b_body; b_body = tt; }
		u32 afi = (a_face ^ 1) ^ (a_face >> 1);  // nudge.cpp:2022
		u32 iX = (afi + 1) % 3, iY = (afi + 2) % 3, iZ = afi;
		#pragma unroll
		for (int g = 0; g < 4; ++g) {
			const u32 index = 4*g + q;
			if (!((mask >> index) & 1)) continue;
			u32 slot = at + __popc(mask & ((1u << index) - 1u));  // the contacts go in increasing point order, as the reference emits them
			float lx = sel3(px[g], py[g], pz[g], iX), ly = sel3(px[g], py[g], pz[g], iY), lz = sel3(px[g], py[g], pz[g], iZ);
			float wx = w0[0]*lx + w1[0]*ly + w2[0]*lz + A.t.p.x;
			float wy = w0[1]*lx + w1[1]*ly + w2[1]*lz + A.t.p.y;
			float wz = w0[2]*lx + w1[2]*ly + w2[2]*lz + A.t.p.z;
			u32 feature = tag_swap ? ((st[g] >> 16) | (st[g] << 16)) : st[g];  // nudge.cpp:2108
			if (slot < limit) put_contact(out, slot, wx, wy, wz, pen[g], nx, ny, nz, a_body, b_body, high_tag, feature);
		}
	}
	else if (kind == 2 && q == 0 && at < limit) {  // nudge.cpp:2116-2135: the box with the higher tag goes first
		bool keep = A.tag > B.tag;
		u32 feature = keep ? a_edge | (b_edge << 16) : b_edge | (a_edge << 16);
		BoxIn E0 = A, E1 = B;
		if (!keep) { E0 = B; E1 = A; }
		bb_edge(E0, E1, penetration, feature, out, at, s_rsqrt);
	}
}

// Clips the surviving box-box pairs ONCE: the contacts go to a scratch contact buffer in arrival order (np_start[j] = first slot),
// and k_np_emit moves them to their final, pair-ordered place after the scan.  Four lanes clip one pair (bb_clip); the loop runs
// over whole warps, eight pairs at a time.  The kernel is bound by latency at two blocks per SM; three fit in 80 registers without spills.
__global__ void __launch_bounds__(NB_BLOCK, 3) k_np_clip(const uint2* live, const u32* np_list, const float* np_pen, const u32* np_info, const nb_transform* world_xf,
		const nb_box_collider* box_data, const u32* col_tag, u32* cnt, u32 stride, ContactOut tmp, u32* np_start, u32 max_contacts, u32* counts) {
	// the rsqrtps table goes to shared memory: different indices per warp would serialise on the constant cache
	__shared__ u32 s_rsqrt[2048];
	for (u32 i = threadIdx.x; i < 2048; i += blockDim.x) s_rsqrt[i] = g_rsqrt_lut[i];
	__syncthreads();
	const u32 n = counts[CNT_SURV];
	const u32 warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps = (gridDim.x * blockDim.x) >> 5, g = (threadIdx.x & 31) >> 2;
	for (u32 k0 = warp * 8; k0 < n; k0 += warps * 8) {
		const u32 k = k0 + g;
		const bool valid = k < n;
		const u32 j = np_list[valid ? k : k0];
		BoxIn A, B; load_pair(live, np_info, world_xf, box_data, col_tag, j, A, B);
		u32 at, nface, nedge;
		bb_clip(A, B, np_pen[j], np_info[j] & 3, valid, s_rsqrt, &counts[CNT_TMP], tmp, max_contacts, at, nface, nedge);
		if (valid && (threadIdx.x & 3) == 0) {
			np_start[j] = at;
			cnt[0*stride + j] = nface;
			cnt[1*stride + j] = nedge;
		}
	}
}

NB_DEV void move_contact(const ContactOut& from, u32 src, const ContactOut& to, u32 dst) {
	to.data[2*dst + 0] = from.data[2*src + 0]; to.data[2*dst + 1] = from.data[2*src + 1];
	to.bodies[dst] = from.bodies[src]; to.tags[dst] = from.tags[src]; to.features[dst] = from.features[src];
}

__global__ void __launch_bounds__(NB_BLOCK) k_np_emit(const uint2* live, const u32* np_list, const u32* np_start, ContactOut tmp, u32 nboxes, const nb_transform* world_xf,
		const nb_box_collider* box_data, const nb_sphere_collider* sph_data, const u32* col_tag, const u32* cnt, const u32* offs, u32 stride,
		ContactOut out, u32 max_contacts, u32* counts) {
	const u32 n_surv = counts[CNT_SURV], n_bb = counts[CNT_LIVE0], n_all = counts[CNT_LIVE_TOTAL];
	const u32 n_bs_end = n_bb + counts[CNT_LIVE1] + counts[CNT_LIVE2];
	const u32 edge_base = counts[CNT_FACE], other_base = edge_base + counts[CNT_EDGE];
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		u32 staged = other_base + counts[CNT_OTHER];
		if (staged > max_contacts || counts[CNT_TMP] > max_contacts) { atomicOr(&counts[CNT_OVERFLOW], OVF_CONTACTS); staged = min(staged, max_contacts); }
		counts[CNT_STAGED] = staged;
	}
	const u32 total = n_surv + (n_all - n_bb);
	for (u32 t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
		if (t < n_surv) {
			u32 j = np_list[t];
			u32 nf = cnt[0*stride + j], ne = cnt[1*stride + j];
			if (!(nf | ne)) continue;
			u32 src = np_start[j], dst = nf ? offs[0*stride + j] : edge_base + offs[1*stride + j];
			for (u32 i = 0; i < nf + ne; ++i)
				if (src + i < max_contacts && dst + i < max_contacts) move_contact(tmp, src + i, out, dst + i);
		}
		else {
			u32 j = n_bb + (t - n_surv);
			if (!cnt[2*stride + j]) continue;
			uint2 pr = live[j];
			float o[7];
			u32 a = pr.y, b = pr.x;
			xform ta = ld_xform(world_xf, a), tb = ld_xform(world_xf, b);
			if (j < n_bs_end) { float4 sz = reinterpret_cast<const float4*>(box_data)[a]; box_sphere(make_float3(sz.x, sz.y, sz.z), sph_data[b - nboxes].radius, ta, tb, o); }
			else sphere_sphere(sph_data[a - nboxes].radius, sph_data[b - nboxes].radius, ta, tb, o);
			u32 at = other_base + offs[2*stride + j];
			if (at < max_contacts)
				put_contact(out, at, o[0], o[1], o[2], o[3], o[4], o[5], o[6], asu(ta.p.w), asu(tb.p.w), (u64)col_tag[a] | ((u64)col_tag[b] << 32), 0);  // nudge.cpp:3767, 3784
		}
	}
}

// ---------------- fine islands: active bodies + contact compaction (nudge.cpp:3965-4006) ----------------
__global__ void __launch_bounds__(NB_BLOCK) k_body_flags(const u32* parent, const u32* active, u32* flags, u32 B) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x)
		flags[i] = (i >= 1 && active[parent[i]]) ? 1u : 0u;
}
__global__ void __launch_bounds__(NB_BLOCK) k_active_scatter(const u32* flags, const u32* block_sums, u32* active_idx, u32 B) {  // NB_SCAN_GRID blocks
	scan_consume<1>(flags, 0, B, block_sums, [&](u32 i, const u32 (&v)[1], const u32 (&off)[1]) { if (v[0]) active_idx[off[0]] = i; });
}
__global__ void __launch_bounds__(NB_BLOCK) k_contact_flags(const uint2* bodies, const u64* tags, const u32* parent, const u32* active, u32* flags, u32 stride, const u32* counts) {
	u32 n = counts[CNT_STAGED];
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		uint2 ab = bodies[i];
		// The reference decides per span of equal pair tags from the span's first contact (nudge.cpp:3976-3999);
		// every contact of a span has the same bodies, so the per-contact decision is the same.
		u32 set = ab.x ? parent[ab.x] : parent[ab.y];
		bool keep = active[set] != 0;
		flags[i] = keep ? 1u : 0u;
		flags[stride + i] = (!keep && (i == 0 || tags[i - 1] != tags[i])) ? 1u : 0u;
	}
}
__global__ void __launch_bounds__(NB_BLOCK) k_contact_compact(ContactOut st, ContactOut fin, const u32* flags, const u32* block_sums, u32 stride, u64* sleeping_pairs, u32* counts) {  // NB_SCAN_GRID blocks
	u32 n = counts[CNT_STAGED];
	u32 sleep_base = counts[CNT_SLEEP_COARSE];
	if (blockIdx.x == 0 && threadIdx.x == 0) counts[CNT_SLEEPING] = sleep_base + counts[CNT_SLEEP_FINE];
	scan_consume<2>(flags, stride, n, block_sums, [&](u32 i, const u32 (&v)[2], const u32 (&off)[2]) {
		if (v[0]) {
			u32 d = off[0];
			fin.data[2*d] = st.data[2*i]; fin.data[2*d + 1] = st.data[2*i + 1];
			fin.bodies[d] = st.bodies[i]; fin.tags[d] = st.tags[i]; fin.features[d] = st.features[i];
		}
		if (v[1]) sleeping_pairs[sleep_base + off[1]] = st.tags[i];
	});
}
