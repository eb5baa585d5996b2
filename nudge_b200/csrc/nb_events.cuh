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
#pragma once
#include "nb_solver.cuh"

static_assert(sizeof(nb_contact_event) == 80, "nb_contact_event is 5 x 16 bytes");

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

__global__ void __launch_bounds__(NB_BLOCK) k_event_flags(const u64* cache_tags, const u32* sorted, const u64* tags, const u64* culled_tags, u32* flags, u32* counts) {
	const u32 m = counts[CNT_CACHE], n = counts[CNT_CONTACTS], mc = counts[CNT_CULLED];
	if (blockIdx.x == 0 && threadIdx.x == 0) { counts[CNT_EV_N] = m + n; counts[CNT_EV_BASE] = counts[CNT_EV_COUNT]; counts[CNT_EV_STAMP] = counts[CNT_EV_STEP]; }
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < m + n; i += gridDim.x * blockDim.x) {
		u32 f = 0;
		if (i < m) {
			const u64 t = cache_tags[i];
			if ((i == 0 || cache_tags[i - 1] != t) && !contacts_have(sorted, tags, n, t) && !sorted_has(culled_tags, mc, t)) f = 1;
		}
		else {
			const u32 j = i - m;
			const u64 t = tags[sorted[j]];
			if ((j == 0 || tags[sorted[j - 1]] != t) && !sorted_has(cache_tags, m, t)) f = 1;
		}
		flags[i] = f;
	}
}

// NB_SCAN_GRID blocks, after nb_scan_reduce<1> over the flags (total in CNT_EV_FLAGGED)
__global__ void __launch_bounds__(NB_BLOCK) k_event_scatter(const u32* flags, const u32* block_sums, const u64* cache_tags, const u32* sorted, const u64* tags,
		const float4* data, const uint2* bodies, const float4* impulses, uint4* events /* 5 words per event */, u32 capacity, u32* counts) {
	const u32 m = counts[CNT_CACHE], n = counts[CNT_CONTACTS], base = counts[CNT_EV_BASE], step = counts[CNT_EV_STAMP];
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

// The three launches of an enabled nb_write_cached_impulses.
static void launch_contact_events(const Launch& L, u32 grid, u32* flags, u32 stride, u32* block_sums, const u64* cache_tags, const u32* sorted, const ContactOut& fin,
								  const u64* culled_tags, const float4* impulses, nb_contact_event* events, u32 capacity, u32* counts) {
	k_event_flags<<<grid, NB_BLOCK, 0, L.stream>>>(cache_tags, sorted, fin.tags, culled_tags, flags, counts);
	nb_scan_reduce<1>(L, flags, stride, counts + CNT_EV_N, 0, block_sums, counts + CNT_EV_FLAGGED);
	k_event_scatter<<<NB_SCAN_GRID, NB_BLOCK, 0, L.stream>>>(flags, block_sums, cache_tags, sorted, fin.tags, fin.data, fin.bodies, impulses,
		reinterpret_cast<uint4*>(events), capacity, counts);
	*L.counter += 2;
}
