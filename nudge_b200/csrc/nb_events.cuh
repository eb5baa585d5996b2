// nudge_b200 — contact begin / end events (nb_enable_contact_events, nb_download_contact_events; DESIGN.md §8.5).
//
// Runs inside nb_write_cached_impulses, before k_cache_merge overwrites the cache.  Three sorted lists are at hand: the old cache
// (cache_tags, keys ascending), the step's contacts in tag order (tags[sorted[i]]) and the kept entries of sleeping pairs (culled_tags,
// a subsequence of the old cache).  A pair is one key A | B << 32; its entries are consecutive in each list (a segment), so
//   k_event_flags    flags the segment heads of [old cache | contacts in tag order] that make an event: an old head whose key is
//                    neither among the contacts nor culled (END), a contact head whose key is not in the old cache (BEGIN);
//   k_scan_reduce<1> ranks the flags: ENDs first, then BEGINs, each in ascending key order, because that is the concatenation's order;
//   k_event_scatter  writes event `rank` at count + rank while that fits the buffer; a BEGIN walks its pair's contacts for the count,
//                    the deepest contact and the impulse sum.
// The event counters live in counts[] (CNT_EV_*) and survive k_reset_collide.  k_event_flags snapshots count and step into CNT_EV_BASE /
// CNT_EV_STAMP, so the scatter's blocks read stable values while its block 0 advances count, dropped and step.
// With sensor colliders (DESIGN.md section 8.7) the concatenation goes on with [old overlaps | current overlaps], both sorted by key (one
// entry per pair): an old key that is not current is a SENSOR_END, a current key that was not old a SENSOR_BEGIN.  So the same scan ranks
// contact ENDs, contact BEGINs, sensor ENDs, sensor BEGINs, each in ascending key order.  Without sensors both lists are null and empty.
#pragma once
#include "nb_solver.cuh"

static_assert(sizeof(nb_contact_event) == 80, "nb_contact_event is 5 x 16 bytes");
static_assert(sizeof(nb_sensor_overlap) == 16, "nb_sensor_overlap is one uint4 { tags lo, tags hi, body_a, body_b }");

NB_DEV bool sorted_has(const u64* keys, u32 n, u64 t) {
	u32 lo = 0, hi = n;
	while (lo < hi) { u32 mid = (lo + hi) >> 1; if (keys[mid] < t) lo = mid + 1; else hi = mid; }
	return lo < n && keys[lo] == t;
}
NB_DEV bool contacts_have(const u32* sorted, const u64* tags, u32 n, u64 t) {
	u32 lo = 0, hi = n;
	while (lo < hi) { u32 mid = (lo + hi) >> 1; if (tags[sorted[mid]] < t) lo = mid + 1; else hi = mid; }
	return lo < n && tags[sorted[lo]] == t;
}

NB_DEV u64 overlap_key(const uint4* list, u32 i) { const uint4 e = list[i]; return (u64)e.x | ((u64)e.y << 32); }
NB_DEV bool overlaps_have(const uint4* list, u32 n, u64 t) {
	u32 lo = 0, hi = n;
	while (lo < hi) { u32 mid = (lo + hi) >> 1; if (overlap_key(list, mid) < t) lo = mid + 1; else hi = mid; }
	return lo < n && overlap_key(list, lo) == t;
}

// s_old / s_cur: the overlaps as of the last call (CNT_SENSOR_OLD entries) and of the last collide (CNT_SENSOR_HITS), or null without sensors
__global__ void __launch_bounds__(NB_BLOCK) k_event_flags(const u64* cache_tags, const u32* sorted, const u64* tags, const u64* culled_tags,
		const uint4* s_old, const uint4* s_cur, u32* flags, u32* counts) {
	const u32 m = counts[CNT_CACHE], n = counts[CNT_CONTACTS], mc = counts[CNT_CULLED];
	const u32 so = s_old ? counts[CNT_SENSOR_OLD] : 0u, sc = s_cur ? counts[CNT_SENSOR_HITS] : 0u, mn = m + n;
	if (blockIdx.x == 0 && threadIdx.x == 0) { counts[CNT_EV_N] = mn + so + sc; counts[CNT_EV_BASE] = counts[CNT_EV_COUNT]; counts[CNT_EV_STAMP] = counts[CNT_EV_STEP]; }
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < mn + so + sc; i += gridDim.x * blockDim.x) {
		u32 f = 0;
		if (i < m) {
			const u64 t = cache_tags[i];
			if ((i == 0 || cache_tags[i - 1] != t) && !contacts_have(sorted, tags, n, t) && !sorted_has(culled_tags, mc, t)) f = 1;
		}
		else if (i < mn) {
			const u32 j = i - m;
			const u64 t = tags[sorted[j]];
			if ((j == 0 || tags[sorted[j - 1]] != t) && !sorted_has(cache_tags, m, t)) f = 1;
		}
		else if (i < mn + so) {
			const u32 j = i - mn;
			const u64 t = overlap_key(s_old, j);
			if ((j == 0 || overlap_key(s_old, j - 1) != t) && !overlaps_have(s_cur, sc, t)) f = 1;
		}
		else {
			const u32 j = i - mn - so;
			const u64 t = overlap_key(s_cur, j);
			if ((j == 0 || overlap_key(s_cur, j - 1) != t) && !overlaps_have(s_old, so, t)) f = 1;
		}
		flags[i] = f;
	}
}

// NB_SCAN_GRID blocks, after nb_scan_reduce<1> over the flags (total in CNT_EV_FLAGGED)
__global__ void __launch_bounds__(NB_BLOCK) k_event_scatter(const u32* flags, const u32* block_sums, const u64* cache_tags, const u32* sorted, const u64* tags,
		const float4* data, const uint2* bodies, const float4* impulses, const uint4* s_old, const uint4* s_cur, uint4* events /* 5 words per event */,
		u32 capacity, u32* counts) {
	const u32 m = counts[CNT_CACHE], n = counts[CNT_CONTACTS], base = counts[CNT_EV_BASE], step = counts[CNT_EV_STAMP];
	const u32 so = s_old ? counts[CNT_SENSOR_OLD] : 0u;
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		const u64 end = (u64)base + counts[CNT_EV_FLAGGED];
		const u64 kept = end < capacity ? end : capacity;
		counts[CNT_EV_COUNT] = (u32)kept;
		counts[CNT_EV_DROPPED] += (u32)(end - kept);
		counts[CNT_EV_STEP] = step + 1;
	}
	scan_consume<1>(flags, 0, counts[CNT_EV_N], block_sums, [&](u32 i, const u32 (&v)[1], const u32 (&off)[1]) {
		if (!v[0] || (u64)base + off[0] >= capacity) return;   // a full buffer: the event is counted in CNT_EV_DROPPED above
		uint4* e = events + 5 * (size_t)(base + off[0]);
		if (i < m) {
			const u64 t = cache_tags[i];
			e[0] = make_uint4((u32)t, (u32)(t >> 32), NB_CONTACT_END, step);
			e[1] = e[2] = e[3] = e[4] = make_uint4(0, 0, 0, 0);
			return;
		}
		if (i >= m + n) {   // a sensor event: tags, kind, step and the two bodies
			const bool end = i < m + n + so;
			const uint4 o = end ? s_old[i - m - n] : s_cur[i - m - n - so];
			e[0] = make_uint4(o.x, o.y, end ? NB_SENSOR_END : NB_SENSOR_BEGIN, step);
			e[1] = make_uint4(o.z, o.w, 0, 0);
			e[2] = e[3] = e[4] = make_uint4(0, 0, 0, 0);
			return;
		}
		const u32 j = i - m;
		const u32 c0 = sorted[j];
		const u64 t = tags[c0];
		u32 deepest = c0, count = 0;
		float depth = data[2 * c0].w, ix = 0.0f, iy = 0.0f, iz = 0.0f;
		for (u32 k = j; k < n; ++k) {
			const u32 c = sorted[k];
			if (tags[c] != t) break;
			const float p = data[2 * c].w;
			if (p > depth) { depth = p; deepest = c; }   // strictly deeper: ties keep the earlier contact, a NaN never wins
			const float4 im = impulses[c];
			ix = ix + im.x; iy = iy + im.y; iz = iz + im.z;   // tag order, one rounding per add (-fmad=false)
			++count;
		}
		const float4 p = data[2 * deepest], q = data[2 * deepest + 1];
		const uint2 ab = bodies[deepest];
		e[0] = make_uint4((u32)t, (u32)(t >> 32), NB_CONTACT_BEGIN, step);
		e[1] = make_uint4(ab.x, ab.y, count, asu(p.w));
		e[2] = make_uint4(asu(p.x), asu(p.y), asu(p.z), asu(q.x));
		e[3] = make_uint4(asu(q.y), asu(q.z), asu(ix), asu(iy));
		e[4] = make_uint4(asu(iz), 0, 0, 0);
	});
}

// The three launches of an enabled nb_write_cached_impulses.  `flags` holds the old cache, the contacts and both overlap lists.
static void launch_contact_events(const Launch& L, u32 grid, u32* flags, u32 stride, u32* block_sums, const u64* cache_tags, const u32* sorted, const ContactOut& fin,
								  const u64* culled_tags, const float4* impulses, const uint4* s_old, const uint4* s_cur, nb_contact_event* events, u32 capacity, u32* counts) {
	launch_grid(L, k_event_flags, grid, cache_tags, sorted, fin.tags, culled_tags, s_old, s_cur, flags, counts);
	nb_scan_reduce<1>(L, flags, stride, counts + CNT_EV_N, 0, block_sums, counts + CNT_EV_FLAGGED);
	launch_grid(L, k_event_scatter, NB_SCAN_GRID, flags, block_sums, cache_tags, sorted, fin.tags, fin.data, fin.bodies, impulses, s_old, s_cur,
		reinterpret_cast<uint4*>(events), capacity, counts);
}

// With sensors, at the end of every nb_write_cached_impulses (events on or off): the current overlaps become the old ones
__global__ void __launch_bounds__(NB_BLOCK) k_sensor_keep(const uint4* cur, uint4* old, u32* counts) {
	const u32 n = counts[CNT_SENSOR_HITS];
	if (blockIdx.x == 0 && threadIdx.x == 0) counts[CNT_SENSOR_OLD] = n;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) old[i] = cur[i];
}
