// nudge_b200 — contact cache, constraint setup, the sequential-impulse sweeps and the integrator.
// Replaces nudge::read_cached_impulses / write_cached_impulses (nudge.cpp:4021-4158),
// setup_contact_constraints (4170-4638), apply_impulses (4640-4855), update_cached_impulses (4857-4884)
// and advance (4886-4926).
//
// Exact-order Gauss-Seidel on a GPU (SURVEY.md §0.4): the reference walks 8-lane batches in the order its
// sequential 16-bucket first-fit scheduler emits them (nudge.cpp:4206-4340), each batch reading the body
// velocities the previous one wrote.  We (1) replay that scheduler bit for bit with one warp per bucket to
// get every contact's batch index and lane, (2) chain the contacts of each body by batch index, and (3) run all
// sweeps as ONE co-resident dataflow kernel: every body carries a version counter, a contact waits until both
// of its bodies carry the token of its predecessor in the reference order, applies its impulse, and publishes
// its own token.  No grid barrier, sweeps pipeline into each other, and the result is bit-identical to the
// sequential walk because every body sees exactly the reference's sequence of updates.
// Rows are stored SoA (one float per contact per plane) so that a warp reads 128 contiguous bytes per plane;
// the slot of a contact is batch*8 + lane, i.e. the reference's own ContactConstraintV layout flattened.
#pragma once
#include "nb_collide.cuh"

#define NB_NONE 0xffffffffu

enum {  // constraint row planes, member order of ContactConstraintV (nudge.cpp:907-957)
	PA_Z, PA_X, PA_Y, PB_Z, PB_X, PB_Y, N_X, U_X, V_X, N_Y, U_Y, V_Y, N_Z, U_Z, V_Z, BIAS, FRICTION, NVTNI, FC_X, FC_Y, FC_Z,
	NA_X, NA_Y, NA_Z, NB_X, NB_Y, NB_Z, UA_X, UA_Y, UA_Z, VA_X, VA_Y, VA_Z, UB_X, UB_Y, UB_Z, VB_X, VB_Y, VB_Z, ROW_PLANES,
	MASS_A = ROW_PLANES, MASS_B, ROW_PLANES_TOTAL  // two extra planes: the bodies' inverse masses (the reference keeps them in BodyMomentum::unused0)
};

NB_DEV bool key_less(u64 ta, u32 fa, u64 tb, u32 fb) { return ta < tb || (ta == tb && fa < fb); }

// ---------------- contact cache read (nudge.cpp:4021-4108) ----------------
__global__ void __launch_bounds__(NB_BLOCK) k_tag_keys_feature(const u32* features, u64* keys, u32* vals, const u32* counts) {
	u32 n = counts[CNT_CONTACTS];
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) { keys[i] = features[i]; vals[i] = i; }
}
__global__ void __launch_bounds__(NB_BLOCK) k_tag_keys_pair(const u64* tags, const u32* vals, u64* keys, u32 tagbits, const u32* counts) {
	u32 n = counts[CNT_CONTACTS];
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		u64 t = tags[vals[i]];
		keys[i] = ((t >> 32) << tagbits) | (t & 0xffffffffu);  // major = B (bits 48-63 of the reference tag), then A
	}
}

// Contacts produced by nb_collide carry feature words whose four bytes are each 0..7 or 0xff (nudge.cpp:1902-1970, 2381-2390;
// sphere contacts: 0), so byte & 15 keeps their order and the whole tag fits one key: B | A | 16 feature bits.
__global__ void __launch_bounds__(NB_BLOCK) k_tag_keys_packed(const u64* tags, const u32* features, u64* keys, u32* vals, u32 tagbits, u32 spread, const u32* counts) {
	u32 n = counts[CNT_CONTACTS];
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		u64 t = tags[i]; u32 f = features[i];
		u32 f16 = (f & 0xf) | ((f >> 4) & 0xf0) | ((f >> 8) & 0xf00) | ((f >> 12) & 0xf000);
		u64 k = ((((t >> 32) << tagbits) | (t & 0xffffffffu)) << 16) | f16;
		// The major field B is the SMALLER collider tag of the pair, and the static world's colliders carry the smallest tags (the ground is
		// added first, example/main.cpp:398-409): every ground contact of a pile — 20 % of all contacts — had B = 0 and fell into one of the
		// sort's 256 top-digit buckets, sorted by a single block, which dominated the sort.  Order-preserving stretch: keys with B < 8 are
		// scaled up to fill the lower half of a key space one bit wider, the rest move to the upper half; the top digit then splits the
		// hot keys by A.  (spread = 0 when the key would not fit 64 bits: plain key.)
		if (spread) k = (t >> 32) < 8 ? k << (tagbits - 3) : k | ((u64)1 << (2 * tagbits + 16));
		keys[i] = k;
		vals[i] = i;
	}
}

// impulses[c] = cache entry with the same tag, else zero; the lower bound is the entry the reference's merge stops at
__global__ void __launch_bounds__(NB_BLOCK) k_cache_lookup(const u64* tags, const u32* features, const u64* cache_tags, const u32* cache_features,
														   const float4* cache_data, float4* impulses, const u32* counts) {
	u32 n = counts[CNT_CONTACTS], m = counts[CNT_CACHE];
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		u64 t = tags[i]; u32 f = features[i];
		u32 lo = 0, hi = m;
		while (lo < hi) { u32 mid = (lo + hi) >> 1; if (key_less(cache_tags[mid], cache_features[mid], t, f)) lo = mid + 1; else hi = mid; }
		float4 v = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		if (lo < m && cache_tags[lo] == t && cache_features[lo] == f) v = cache_data[lo];
		impulses[i] = v;
	}
}

// cache entries of sleeping pairs survive the frame ("culled", nudge.cpp:4064-4101)
__global__ void __launch_bounds__(NB_BLOCK) k_culled_flags(const u64* cache_tags, const u64* sleeping, u32* flags, const u32* counts) {
	u32 m = counts[CNT_CACHE], s = counts[CNT_SLEEPING];
	for (u32 e = blockIdx.x * blockDim.x + threadIdx.x; e < m; e += gridDim.x * blockDim.x) {
		u64 t = cache_tags[e];
		u32 lo = 0, hi = s;
		while (lo < hi) { u32 mid = (lo + hi) >> 1; if (sleeping[mid] < t) lo = mid + 1; else hi = mid; }
		flags[e] = (lo < s && sleeping[lo] == t) ? 1u : 0u;
	}
}
// NB_SCAN_GRID blocks, after nb_scan_reduce<1> over the flags
__global__ void __launch_bounds__(NB_BLOCK) k_culled_scatter(const u32* flags, const u32* block_sums, const u64* cache_tags, const u32* cache_features, const float4* cache_data,
															 u64* culled_tags, u32* culled_features, float4* culled_data, const u32* counts) {
	scan_consume<1>(flags, 0, counts[CNT_CACHE], block_sums, [&](u32 e, const u32 (&v)[1], const u32 (&d)[1]) {
		if (v[0]) { culled_tags[d[0]] = cache_tags[e]; culled_features[d[0]] = cache_features[e]; culled_data[d[0]] = cache_data[e]; }
	});
}

// ---------------- contact cache write: 2-way merge by rank (nudge.cpp:4110-4158) ----------------
__global__ void __launch_bounds__(NB_BLOCK) k_cache_merge(const u32* sorted, const u64* tags, const u32* features, const float4* impulses,
		const u64* culled_tags, const u32* culled_features, const float4* culled_data, u64* cache_tags, u32* cache_features, float4* cache_data, u32* counts) {
	u32 n = counts[CNT_CONTACTS], m = counts[CNT_CULLED];
	if (blockIdx.x == 0 && threadIdx.x == 0) counts[CNT_CACHE] = n + m;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n + m; i += gridDim.x * blockDim.x) {
		if (i < n) {  // contact i of the tag order goes after every culled entry with key <= its key (ties: culled first)
			u32 c = sorted[i]; u64 t = tags[c]; u32 f = features[c];
			u32 lo = 0, hi = m;
			while (lo < hi) { u32 mid = (lo + hi) >> 1; if (!key_less(t, f, culled_tags[mid], culled_features[mid])) lo = mid + 1; else hi = mid; }
			u32 d = i + lo;
			cache_tags[d] = t; cache_features[d] = f; cache_data[d] = impulses[c];
		}
		else {  // culled entry j goes after every contact with key < its key
			u32 j = i - n; u64 t = culled_tags[j]; u32 f = culled_features[j];
			u32 lo = 0, hi = n;
			while (lo < hi) { u32 mid = (lo + hi) >> 1; u32 c = sorted[mid]; if (key_less(tags[c], features[c], t, f)) lo = mid + 1; else hi = mid; }
			u32 d = j + lo;
			cache_tags[d] = t; cache_features[d] = f; cache_data[d] = culled_data[j];
		}
	}
}

// ---------------- per-body world inverse inertia (nudge.cpp:4182-4199) ----------------
__global__ void __launch_bounds__(NB_BLOCK) k_inertia(u32 B, const nb_transform* xf, const nb_body_properties* props, float4* inertia, nb_body_momentum* momentum) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
		float4 q = reinterpret_cast<const float4*>(xf + i)[1];
		float4 pr = reinterpret_cast<const float4*>(props)[i];
		mat3 m = qmatrix(mkq(q));
		float ix = pr.x, iy = pr.y, iz = pr.z;
		float xx = ix*m.c0.x*m.c0.x + iy*m.c1.x*m.c1.x + iz*m.c2.x*m.c2.x;
		float yy = ix*m.c0.y*m.c0.y + iy*m.c1.y*m.c1.y + iz*m.c2.y*m.c2.y;
		float zz = ix*m.c0.z*m.c0.z + iy*m.c1.z*m.c1.z + iz*m.c2.z*m.c2.z;
		float xy = ix*m.c0.x*m.c0.y + iy*m.c1.x*m.c1.y + iz*m.c2.x*m.c2.y;
		float xz = ix*m.c0.x*m.c0.z + iy*m.c1.x*m.c1.z + iz*m.c2.x*m.c2.z;
		float yz = ix*m.c0.y*m.c0.z + iy*m.c1.y*m.c1.z + iz*m.c2.y*m.c2.z;
		inertia[2*i] = make_float4(xx, yy, zz, 0.0f);
		inertia[2*i + 1] = make_float4(xy, xz, yz, 0.0f);
		momentum[i].unused0 = pr.w;  // nudge.cpp:4198
	}
}

// ---------------- scheduler replay: one warp per bucket (nudge.cpp:4206-4340) ----------------
// The reference's state per bucket is a list of partially filled 8-lane slots; a contact goes to the first slot
// holding neither of its bodies, a slot that receives its 8th contact is emitted and replaced by the last slot of
// the list.  Buckets only interact through the global emission order, which equals the order of the contact
// index at which each slot filled up, so 16 warps can replay them independently.
// State layout: a slot has 16 entries (8 "a" bodies, 8 "b" bodies, NB_NONE = empty).  List positions 0..7 live in
// registers, one ENTRY per lane: lane = 16*(position & 1) + entry, register index = position >> 1.  A contact is tested
// against two positions with one compare and one ballot, so the serial chain per contact is a handful of instructions.
// Positions 8.. use the same 16-entry layout in shared memory.  Invariant: every position >= vcount is all empty, so the
// reference's always-free sentinel (nudge.cpp:4225-4227, 4313) is simply "the first position that does not conflict".
#define NB_SCHED_REGSETS 4
#define NB_SCHED_REGPOS (2 * NB_SCHED_REGSETS)
#define NB_SCHED_SHARED 504
#define NB_SCHED_MAXV (NB_SCHED_REGPOS + NB_SCHED_SHARED - 1)   // positions held on chip; beyond that the list spills to global memory

// Parallel pre-pass for the replay: the body pair of every contact in tag order with the body-0 substitution of
// nudge.cpp:4238-4240 applied, and `back` = distance (in contacts of the same bucket, 1..7) to the nearest earlier contact of
// the bucket that shares a body, 0 if there is none within 7.  A run of 8 consecutive bucket contacts starting at a fresh
// slot is conflict free iff none of them has 0 < back <= its offset in the run.
__global__ void __launch_bounds__(NB_BLOCK) k_sched_prep(const u32* sorted, const uint2* bodies, uint2* cab, uint8_t* back, const u32* counts) {
	u32 n = counts[CNT_CONTACTS];
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		uint2 ab = bodies[sorted[i]];
		u32 ca = ab.x ? ab.x : ab.y, cb = ab.y ? ab.y : ab.x;
		cab[i] = make_uint2(ca, cb);
		u32 b = 0;
		#pragma unroll
		for (u32 k = 1; k <= 7; ++k) {
			if (!b && i >= 16 * k) {
				uint2 o = bodies[sorted[i - 16 * k]];
				u32 oa = o.x ? o.x : o.y, ob = o.y ? o.y : o.x;
				if (oa == ca || ob == ca || oa == cb || ob == cb) b = k;
			}
		}
		back[i] = (uint8_t)b;
	}
}

// slot_of[i] = uid << 3 | lane, where lane is the SIMD lane the contact lands in (= number of contacts already in its slot)
//
// ~99.9 % of all contacts go to list position 0 (measured), so the replay speculates: the next 8 - fill(position 0)
// contacts are tested against position 0 and against each other with ONE __match_any_sync; all contacts before the first
// conflict are accepted in parallel (they are exactly the ones the sequential first-fit would put there), and only the
// conflicting contact runs the general search.  A lone warp pays ~8 cycles per instruction, so instructions per contact
// are what matters here.
// A list longer than the on-chip positions (a body with thousands of contacts: all of them conflict with each other, each opens its
// own slot) SPILLS to global memory: positions >= NB_SCHED_REGPOS + NB_SCHED_SHARED live in spill_ent / spill_uid (per bucket,
// `spill_cap` positions, all entries NB_NONE between launches: the kernel clears what it used).  The reference has no limit here.
__global__ void __launch_bounds__(32) k_schedule(const uint2* cab, const uint8_t* back, u32* slot_of, u32* slot_done, u32* slot_left, u32 slots_per_bucket,
												 u32* complete_flag, u32* left_count /*[16]*/, u32* spill_ent, u32* spill_uid, u32 spill_cap, u32* counts) {
	__shared__ u32 S_ent[NB_SCHED_SHARED][16];
	__shared__ u32 S_uid[NB_SCHED_REGPOS + NB_SCHED_SHARED];
	const u32 bucket = blockIdx.x, lane = threadIdx.x, half = lane >> 4, ent = lane & 15, cidx = lane & 7;
	const u32 n = counts[CNT_CONTACTS];
	for (u32 k = lane; k < NB_SCHED_SHARED * 16; k += 32) (&S_ent[0][0])[k] = NB_NONE;
	__syncwarp();
	u32* const G_ent = spill_ent + (size_t)bucket * spill_cap * 16;
	u32* const G_uid = spill_uid + (size_t)bucket * spill_cap;
	u32 spill_high = 0;   // positions of the spill area this launch has touched (warp uniform)
	const u32 ONCHIP = NB_SCHED_REGPOS + NB_SCHED_SHARED;
	// entries / uid of a list position that is not in registers (pos >= NB_SCHED_REGPOS)
	auto ent_of = [&](u32 pos) -> u32* { return pos < ONCHIP ? &S_ent[pos - NB_SCHED_REGPOS][0] : G_ent + (size_t)(pos - ONCHIP) * 16; };
	auto uid_of = [&](u32 pos) -> u32* { return pos < ONCHIP ? &S_uid[pos] : G_uid + (pos - ONCHIP); };
	u32 vcount = 0, next_uid = 0;
	u32 f0 = 0, uid0 = 0;  // fill count and uid of list position 0 (warp uniform)
	u32 reg[NB_SCHED_REGSETS];
	#pragma unroll
	for (int k = 0; k < NB_SCHED_REGSETS; ++k) reg[k] = NB_NONE;
	u32* done = slot_done + (size_t)bucket * slots_per_bucket;
	u32* left = slot_left + (size_t)bucket * slots_per_bucket;

	// Removes the completed slot at list position j: the last slot of the list takes its place (nudge.cpp:4294-4306).
	auto remove_pos = [&](u32 j) {
		u32 last = vcount - 1;
		if (last == 0) {  // the list held only this slot
			if (lane < 16) reg[0] = NB_NONE;
			vcount = 0; f0 = 0;
			return;
		}
		u32 jh = j & 1;
		u32 v;  // entry `ent` of the last position, in every lane
		if (last < NB_SCHED_REGPOS) {
			u32 src = NB_NONE;
			#pragma unroll
			for (u32 k = 0; k < NB_SCHED_REGSETS; ++k) if (k == (last >> 1)) src = reg[k];
			v = __shfl_sync(0xffffffffu, src, 16 * (last & 1) + ent);
		}
		else v = ent_of(last)[ent];
		u32 last_uid = *uid_of(last);
		__syncwarp();
		if (j != last) {
			if (j < NB_SCHED_REGPOS) {
				#pragma unroll
				for (u32 k = 0; k < NB_SCHED_REGSETS; ++k) if (k == (j >> 1) && half == jh) reg[k] = v;
			}
			else if (lane < 16) ent_of(j)[lane] = v;
			if (lane == 0) *uid_of(j) = last_uid;
			if (j == 0) uid0 = last_uid;
		}
		if (last < NB_SCHED_REGPOS) {  // the vacated last position becomes empty again
			#pragma unroll
			for (u32 k = 0; k < NB_SCHED_REGSETS; ++k) if (k == (last >> 1) && half == (last & 1)) reg[k] = NB_NONE;
		}
		else if (lane < 16) ent_of(last)[lane] = NB_NONE;
		--vcount;
		if (j == 0) f0 = __popc(__ballot_sync(0xffffffffu, reg[0] != NB_NONE) & 0xffu);
		__syncwarp();
	};

	// General first-fit for one contact (nudge.cpp:4250-4314).  Returns false on capacity overflow.
	auto place_general = [&](u32 i, u32 ca, u32 cb) -> bool {
		u32 j = NB_NONE, f = 0;
		#pragma unroll
		for (u32 k = 0; k < NB_SCHED_REGSETS; ++k) {
			u32 hit = __ballot_sync(0xffffffffu, reg[k] == ca || reg[k] == cb);
			u32 occ = __ballot_sync(0xffffffffu, reg[k] != NB_NONE);
			if (j == NB_NONE) {
				if (!(hit & 0xffffu)) { j = 2 * k; f = __popc(occ & 0xffu); }
				else if (!(hit >> 16)) { j = 2 * k + 1; f = __popc((occ >> 16) & 0xffu); }
			}
		}
		if (j == NB_NONE) {  // all eight register positions conflict: continue in shared memory, two positions per round
			for (u32 pb = 0; ; pb += 2) {   // shared positions, then the spill area; the position right after the list is all empty: the search ends there at the latest
				u32 pos = pb + half;
				if (pb >= NB_SCHED_SHARED + spill_cap) return false;
				u32 v = pos < NB_SCHED_SHARED ? S_ent[pos][ent] : (pos < NB_SCHED_SHARED + spill_cap ? G_ent[(size_t)(pos - NB_SCHED_SHARED) * 16 + ent] : ca);
				u32 hit = __ballot_sync(0xffffffffu, v == ca || v == cb);
				u32 occ = __ballot_sync(0xffffffffu, v != NB_NONE);
				if (!(hit & 0xffffu)) { j = NB_SCHED_REGPOS + pb; f = __popc(occ & 0xffu); break; }
				if (!(hit >> 16)) { j = NB_SCHED_REGPOS + pb + 1; f = __popc((occ >> 16) & 0xffu); break; }
			}
		}
		if (j >= ONCHIP + spill_cap - 1) return false;   // keeps one always-empty position behind the list (the reference's sentinel, nudge.cpp:4225-4227)
		if (j >= ONCHIP) spill_high = max(spill_high, j - ONCHIP + 1);
		if (j < NB_SCHED_REGPOS) {
			u32 jh = j & 1;
			#pragma unroll
			for (u32 k = 0; k < NB_SCHED_REGSETS; ++k)
				if (k == (j >> 1)) {
					if (lane == 16 * jh + f) reg[k] = ca;
					if (lane == 16 * jh + 8 + f) reg[k] = cb;
				}
			if (j == 0) f0 = f + 1;
		}
		else {
			if (lane == 0) { u32* e = ent_of(j); e[f] = ca; e[8 + f] = cb; }
			__syncwarp();
		}
		u32 uid;
		if (j == vcount) {  // the sentinel was taken: a new slot (f is 0)
			uid = next_uid++;
			if (lane == 0) { *uid_of(j) = uid; done[uid] = NB_NONE; }
			if (j == 0) uid0 = uid;
			++vcount;
			__syncwarp();
		}
		else uid = j ? *uid_of(j) : uid0;
		if (lane == 0) slot_of[i] = (uid << 3) | f;
		if (f == 7) {
			if (lane == 0) { done[uid] = i; complete_flag[i] = 1; }
			remove_pos(j);
		}
		return true;
	};

	// software pipeline: the (ca, cb) of the next 32 contacts of this bucket are fetched while the current 32 are placed
	u32 nx_ca = 0, nx_cb = 0, nx_back = 0;
	{
		u32 i0 = bucket + 16 * lane;
		if (i0 < n) { uint2 ab = cab[i0]; nx_ca = ab.x; nx_cb = ab.y; nx_back = back[i0]; complete_flag[i0] = 0; }
	}
	for (u32 base = bucket; base < n; base += 16 * 32) {
		const u32 my_ca = nx_ca, my_cb = nx_cb, my_back = nx_back;
		{
			u32 i1 = base + 16 * 32 + 16 * lane;
			if (i1 < n) { uint2 ab = cab[i1]; nx_ca = ab.x; nx_cb = ab.y; nx_back = back[i1]; complete_flag[i1] = 0; }
		}
		const u32 steps = min(32u, (n - base + 15) / 16);
		u32 s = 0;
		while (s < steps) {
			// ---- fresh list: whole 8-contact runs with no internal conflict are complete slots; accept as many as are clean with one ballot ----
			if (vcount == 0 && steps - s >= 8) {
				const u32 off = (lane - s) & 7;                       // offset of this lane's contact in its run (runs start at s)
				const bool bad = lane >= s && lane < steps && my_back != 0 && my_back <= off;
				const u32 bal = __ballot_sync(0xffffffffu, bad);
				const u32 first_bad = bal ? (u32)(__ffs(bal) - 1) : steps;
				const u32 runs = (first_bad - s) >> 3;
				if (runs) {
					const u32 rel = lane - s;
					if (lane >= s && rel < 8 * runs) {
						const u32 uid = next_uid + (rel >> 3);
						const u32 i = base + 16 * lane;
						slot_of[i] = (uid << 3) | (rel & 7);
						if ((rel & 7) == 7) { done[uid] = i; complete_flag[i] = 1; }
					}
					next_uid += runs; s += 8 * runs;
					continue;
				}
			}
			// ---- speculative groups: the contacts that would fill list position 0 (lanes 0-15); when the list is empty the
			// upper half-warp speculates on the following eight as well ----
			const bool fresh = vcount == 0;  // implies f0 == 0
			u32 src = s + cidx - f0 + (half ? 8u : 0u);      // chunk index of the contact this lane would hold
			bool isnew = (half ? fresh : cidx >= f0) && src < steps;
			u32 va = __shfl_sync(0xffffffffu, my_ca, src & 31), vb = __shfl_sync(0xffffffffu, my_cb, src & 31);
			u32 cand = ent < 8 ? va : vb;
			u32 merged = isnew ? cand : ((!half && cidx < f0) ? reg[0] : 0xffffff00u + lane);  // unique dummies never match
			u32 peers = __match_any_sync(0xffffffffu, merged) & (half ? 0xffff0000u : 0x0000ffffu);
			u32 low = ((1u << cidx) - 1u) * 0x101u << (half ? 16 : 0);
			bool confl = isnew && (peers & low) != 0;  // equal to an entry of an EARLIER contact of its group (its own a/b partner is allowed)
			u32 cbal = __ballot_sync(0xffffffffu, confl);
			u32 vbal = __ballot_sync(0xffffffffu, isnew);
			u32 cm = (cbal | (cbal >> 8)) & 0xffu;
			if (fresh && cm == 0 && (vbal & 0xffu) == 0xffu) {
				// the first eight contacts are conflict free: a whole slot, emitted at once; same for the second eight if clean
				bool two = ((cbal >> 16) == 0) && (((vbal >> 16) & 0xffu) == 0xffu);
				u32 uid = next_uid + half;
				if ((!half || two) && ent < 8) slot_of[base + 16 * src] = (uid << 3) | cidx;
				if ((!half || two) && ent == 7) { u32 il = base + 16 * src; done[uid] = il; complete_flag[il] = 1; }
				next_uid += two ? 2 : 1;
				s += two ? 16 : 8;
				continue;
			}
			u32 avail = min(8u - f0, steps - s);
			u32 k = cm ? (u32)(__ffs(cm) - 1) : f0 + avail;   // first conflicting lane of position 0, or one past the last candidate
			if (k > f0) {
				if (vcount == 0) {  // position 0 was the sentinel: a new slot
					uid0 = next_uid++; vcount = 1;
					if (lane == 0) { S_uid[0] = uid0; done[uid0] = NB_NONE; }
				}
				bool take = !half && isnew && cidx < k;
				if (take) reg[0] = cand;
				if (take && ent < 8) slot_of[base + 16 * src] = (uid0 << 3) | cidx;
				s += k - f0; f0 = k;
				if (k == 8) {  // position 0 is complete
					u32 i_last = base + 16 * (s - 1);
					if (lane == 0) { done[uid0] = i_last; complete_flag[i_last] = 1; }
					__syncwarp();
					remove_pos(0);
					continue;  // re-evaluate against the slot that moved into position 0
				}
			}
			if (cm && s < steps) {  // the contact at s conflicts with position 0: general first-fit
				u32 ca = __shfl_sync(0xffffffffu, my_ca, s), cb = __shfl_sync(0xffffffffu, my_cb, s);
				if (!place_general(base + 16 * s, ca, cb)) {   // the list outgrew even the spill area: report, leave the spill area clean
					if (lane == 0) atomicOr(&counts[CNT_OVERFLOW], OVF_SCHED);
					__syncwarp();
					for (u32 k = lane; k < spill_high * 16; k += 32) G_ent[k] = NB_NONE;
					return;
				}
				++s;
			}
		}
	}
	// leftovers are flushed bucket-major in list order (nudge.cpp:4316-4338)
	__syncwarp();
	for (u32 jj = lane; jj < vcount; jj += 32) left[*uid_of(jj)] = jj;
	if (lane == 0) left_count[bucket] = vcount;
	__syncwarp();
	for (u32 k = lane; k < spill_high * 16; k += 32) G_ent[k] = NB_NONE;   // leave the spill area empty for the next launch
}

// batch index and slot (batch*8 + lane) of every contact + the length of every body's chain (chain_len: zero on entry)
__global__ void __launch_bounds__(NB_BLOCK) k_batch_index(const u32* sorted, const uint2* bodies, const u32* slot_of, const u32* slot_done, const u32* slot_left,
		u32 slots_per_bucket, const u32* complete_off, const u32* left_count, u32* batch_of, u32* slot_idx, u32* slot_contact, u32 max_slots,
		u32* chain_len, u32* counts) {
	u32 n = counts[CNT_CONTACTS];
	u32 nfull = counts[CNT_FULL_BATCHES];
	u32 left_base[17]; left_base[0] = 0;
	#pragma unroll
	for (int k = 0; k < 16; ++k) left_base[k + 1] = left_base[k] + left_count[k];
	// A schedule that overflowed (k_schedule's slot list, or more batches than the row planes hold) is partial: slot_of / slot_left /
	// complete_flag are stale beyond the point of failure.  Publish an EMPTY schedule instead (no batches, no chain entries): the
	// row builder, the solver (which would otherwise wait forever for tokens nobody writes) and update_cached_impulses then do
	// nothing, and the host sees OVF_SCHED in nb_download_counts / nb_download_contacts (NB_ERR_OVERFLOW).
	const bool sched_ovf = (counts[CNT_OVERFLOW] & OVF_SCHED) != 0 || 8 * (u64)(nfull + left_base[16]) > max_slots;
	if (blockIdx.x == 0 && threadIdx.x == 0) {
		u32 nb = nfull + left_base[16];
		if (sched_ovf) { atomicOr(&counts[CNT_OVERFLOW], OVF_SCHED); nb = 0; }
		counts[CNT_BATCHES] = nb; counts[CNT_ENTRIES] = sched_ovf ? 0 : 2 * n;
		counts[CNT_CHAIN_CURSOR] = 0;
	}
	if (sched_ovf) return;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		u32 bucket = i & 15, packed = slot_of[i], uid = packed >> 3, lane = packed & 7;
		u32 t = slot_done[(size_t)bucket * slots_per_bucket + uid];
		u32 batch = (t != NB_NONE) ? complete_off[t] : nfull + left_base[bucket] + slot_left[(size_t)bucket * slots_per_bucket + uid];
		batch_of[i] = batch;
		u32 slot = batch * 8 + lane;
		slot_idx[i] = slot;
		if (slot < max_slots) slot_contact[slot] = sorted[i];
		uint2 ab = bodies[sorted[i]];
		if (ab.x) atomicAdd(&chain_len[ab.x], 1u);   // a side on the static world (body 0) has no chain
		if (ab.y) atomicAdd(&chain_len[ab.y], 1u);
	}
}

// Per-body chains.  Entry e = 2*i + side is side `side` of the contact at tag position i; a body's chain is its entries in
// (batch, e) order, which is the order a stable sort of (body | batch) keys over e = 0, 1, ... would give.  The chains are built
// without that sort: k_batch_index counts the entries per body, k_chain_alloc hands every body a segment of that length (segments
// in any order), k_chain_scatter drops each entry into its body's segment (in any order), and k_chain_rank takes an entry's
// position in its chain as the number of entries of its segment with a smaller (batch, e).  Chains average about five entries;
// a hub body's segment is long, but it is read by all its entries at once and stays in L1.
//
// For each contact side: the slot whose token it must see on that body before it may run.  Per body the solver keeps a sequence
// token = number of contact applications the body has received in this launch.  The contact at position `seq` of a body's chain
// of length `len` therefore runs in sweep w when the token reads w*len + seq, and leaves w*len + seq + 1.  (expected - seen) is
// the number of applications still ahead of a waiting contact, which is what the solver's back-off sleeps on.  Body 0 (static
// world) is never waited for: its sides get (0, 0).
__global__ void __launch_bounds__(NB_BLOCK) k_chain_alloc(u32 nbodies, const u32* chain_len, u32* chain_next /* out: first free position of the segment */, u32* counts) {
	const u32 lane = threadIdx.x & 31;
	for (u32 base = blockIdx.x * blockDim.x; base < nbodies; base += gridDim.x * blockDim.x) {  // warp-uniform trip count
		const u32 b = base + threadIdx.x;
		const u32 len = b < nbodies ? chain_len[b] : 0;
		const u32 incl = warp_incl_scan(len);
		u32 at = 0;
		if (lane == 31 && incl) at = atomicAdd(&counts[CNT_CHAIN_CURSOR], incl);
		at = __shfl_sync(0xffffffffu, at, 31);
		if (len) chain_next[b] = at + incl - len;
	}
}
NB_DEV u64 chain_key(u32 batch, u32 e) { return ((u64)batch << 32) | e; }
__global__ void __launch_bounds__(NB_BLOCK) k_chain_scatter(const u32* sorted, const uint2* bodies, const u32* batch_of, u32* chain_next, u64* chain_keys, const u32* counts) {
	const u32 n = counts[CNT_ENTRIES] >> 1;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const uint2 ab = bodies[sorted[i]];
		const u32 batch = batch_of[i];
		if (ab.x) chain_keys[atomicAdd(&chain_next[ab.x], 1u)] = chain_key(batch, 2*i);
		if (ab.y) chain_keys[atomicAdd(&chain_next[ab.y], 1u)] = chain_key(batch, 2*i + 1);
	}
}
__global__ void __launch_bounds__(NB_BLOCK) k_chain_rank(const u32* sorted, const uint2* bodies, const u32* batch_of, const u32* slot_idx, const u32* chain_end, const u32* chain_len,
		const u64* chain_keys, uint2* wait /*[2][stride]: seq, len*/, u32 stride, const u32* counts) {
	const u32 n2 = counts[CNT_ENTRIES];
	for (u32 e = blockIdx.x * blockDim.x + threadIdx.x; e < n2; e += gridDim.x * blockDim.x) {
		const u32 i = e >> 1, side = e & 1;
		const uint2 ab = bodies[sorted[i]];
		const u32 body = side ? ab.y : ab.x;
		uint2 w = make_uint2(0, 0);
		if (body) {
			const u32 len = chain_len[body], end = chain_end[body];
			const u64 mine = chain_key(batch_of[i], e);
			u32 seq = 0;
			for (u32 j = end - len; j < end; ++j) seq += chain_keys[j] < mine ? 1u : 0u;
			w = make_uint2(seq, len);
		}
		const u32 slot = slot_idx[i];
		if (slot < stride) wait[side * stride + slot] = w;
	}
}

// ---------------- constraint rows (nudge.cpp:4350-4561), one thread per contact, SoA planes ----------------
struct Rows { float* plane; u32 stride; u32* a; u32* b; u32* contact; float* state; uint2* wait; };  // plane[k*stride + slot], wait[side*stride + slot] = (seq, len)

// SPLIT (throughput mode, nb_jacobi.cuh): body i is split into cnt[i] sub-bodies of mass m_i / cnt[i], one per contact (Tonge et al.,
// "Mass splitting for jitter-free parallel rigid body simulation", 2012), so every effective-mass term of body i is scaled by
// cnt[i]; the planes that APPLY an impulse to a body (NA.., UA.., MASS_A/B) stay unscaled because the sub-bodies are averaged back.
template<bool SPLIT>
__global__ void __launch_bounds__(NB_BLOCK) k_build_rows(const float4* contacts, const uint2* bodies,
		const nb_transform* xf, const float4* inertia, const nb_body_momentum* momentum, Rows R, const u32* counts, const u32* cnt) {
	__shared__ u32 s_rsqrt[2048];
	for (u32 i = threadIdx.x; i < 2048; i += blockDim.x) s_rsqrt[i] = g_rsqrt_lut[i];
	__syncthreads();
	u32 n = 8 * counts[CNT_BATCHES];
	for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
		u32 c = R.contact[j];
		if (c == NB_NONE) continue;  // unset lane of a leftover batch (the reference repeats lane 0 there, nudge.cpp:4321-4336)
		float4 cp = contacts[2*c], cn = contacts[2*c + 1];
		uint2 ab = bodies[c];
		u32 a = ab.x, b = ab.y;
		float position_x = cp.x, position_y = cp.y, position_z = cp.z, penetration = cp.w;
		float normal_x = cn.x, normal_y = cn.y, normal_z = cn.z, friction = cn.w;
		float a_mass_inverse = momentum[a].unused0, b_mass_inverse = momentum[b].unused0;
		float4 apos = reinterpret_cast<const float4*>(xf + a)[0], bpos = reinterpret_cast<const float4*>(xf + b)[0];
		f3 pa = mk3(position_x - apos.x, position_y - apos.y, position_z - apos.z);
		f3 pb = mk3(position_x - bpos.x, position_y - bpos.y, position_z - bpos.z);
		float4 Ad = inertia[2*a], Ao = inertia[2*a + 1], Bd = inertia[2*b], Bo = inertia[2*b + 1];  // (xx,yy,zz,-) (xy,xz,yz,-)
		f3 nrm = mk3(normal_x, normal_y, normal_z);
		f3 nat = cross3(pa, nrm);
		float na_x = Ad.x*nat.x + Ao.x*nat.y + Ao.y*nat.z;
		float na_y = Ao.x*nat.x + Ad.y*nat.y + Ao.z*nat.z;
		float na_z = Ao.y*nat.x + Ao.z*nat.y + Ad.z*nat.z;
		f3 nbt = cross3(pb, nrm);
		float nb_x = Bd.x*nbt.x + Bo.x*nbt.y + Bo.y*nbt.z;
		float nb_y = Bo.x*nbt.x + Bd.y*nbt.y + Bo.z*nbt.z;
		float nb_z = Bo.y*nbt.x + Bo.z*nbt.y + Bd.z*nbt.z;
		nat = cross3(mk3(na_x, na_y, na_z), pa);
		nbt = cross3(mk3(nb_x, nb_y, nb_z), pb);
		float rx = nat.x + nbt.x, ry = nat.y + nbt.y, rz = nat.z + nbt.z;
		float r_dot_n = rx*normal_x + ry*normal_y + rz*normal_z;
		float mass_inverse = a_mass_inverse + b_mass_inverse;
		float nvtni = mass_inverse + r_dot_n;
		float sa = 1.0f, sb = 1.0f;
		if (SPLIT) {
			sa = (float)max(cnt[a], 1u); sb = (float)max(cnt[b], 1u);
			float ka = a_mass_inverse + (nat.x*normal_x + nat.y*normal_y + nat.z*normal_z);
			float kb = b_mass_inverse + (nbt.x*normal_x + nbt.y*normal_y + nbt.z*normal_z);
			nvtni = sa*ka + sb*kb;
		}
		bool nonzero = nvtni < 0.0f || nvtni > 0.0f;  // _CMP_NEQ_OQ is ordered (nudge.cpp:636-638, 4439)
		nvtni = nonzero ? (-1.0f / nvtni) : 0.0f;
		float bias = -2.0f * nb_max(penetration - 1e-3f, 0.0f) * nvtni;  // nudge.cpp:4442 with the constants of 49-50
		float s = nb_abs(normal_x);
		float u_x = normal_z*s;
		float u_y = u_x - normal_z;
		float u_z = nb_madd(normal_x - normal_y, s, normal_y);
		u_x = nb_neg(u_x);
		{ float f = nb_rsqrt_t(u_x*u_x + u_y*u_y + u_z*u_z, s_rsqrt); u_x *= f; u_y *= f; u_z *= f; }
		f3 u = mk3(u_x, u_y, u_z);
		f3 v = cross3(u, nrm);
		f3 ua = cross3(pa, u), va = cross3(pa, v), ub = cross3(pb, u), vb = cross3(pb, v);
		float a_duu = Ad.x*ua.x*ua.x + Ad.y*ua.y*ua.y + Ad.z*ua.z*ua.z;
		float a_dvv = Ad.x*va.x*va.x + Ad.y*va.y*va.y + Ad.z*va.z*va.z;
		float a_duv = Ad.x*ua.x*va.x + Ad.y*ua.y*va.y + Ad.z*ua.z*va.z;
		float a_suu = Ao.x*ua.x*ua.y + Ao.y*ua.x*ua.z + Ao.z*ua.y*ua.z;
		float a_svv = Ao.x*va.x*va.y + Ao.y*va.x*va.z + Ao.z*va.y*va.z;
		float a_suv = Ao.x*(ua.x*va.y + ua.y*va.x) + Ao.y*(ua.x*va.z + ua.z*va.x) + Ao.z*(ua.y*va.z + ua.z*va.y);
		float b_duu = Bd.x*ub.x*ub.x + Bd.y*ub.y*ub.y + Bd.z*ub.z*ub.z;
		float b_dvv = Bd.x*vb.x*vb.x + Bd.y*vb.y*vb.y + Bd.z*vb.z*vb.z;
		float b_duv = Bd.x*ub.x*vb.x + Bd.y*ub.y*vb.y + Bd.z*ub.z*vb.z;
		float b_suu = Bo.x*ub.x*ub.y + Bo.y*ub.x*ub.z + Bo.z*ub.y*ub.z;
		float b_svv = Bo.x*vb.x*vb.y + Bo.y*vb.x*vb.z + Bo.z*vb.y*vb.z;
		float b_suv = Bo.x*(ub.x*vb.y + ub.y*vb.x) + Bo.y*(ub.x*vb.z + ub.z*vb.x) + Bo.z*(ub.y*vb.z + ub.z*vb.y);
		float friction_x = mass_inverse + a_duu + a_suu + a_suu + b_duu + b_suu + b_suu;
		float friction_y = mass_inverse + a_dvv + a_svv + a_svv + b_dvv + b_svv + b_svv;
		float friction_z = a_duv + a_duv + a_suv + a_suv + b_duv + b_duv + b_suv + b_suv;
		if (SPLIT) {
			friction_x = sa*(a_mass_inverse + a_duu + a_suu + a_suu) + sb*(b_mass_inverse + b_duu + b_suu + b_suu);
			friction_y = sa*(a_mass_inverse + a_dvv + a_svv + a_svv) + sb*(b_mass_inverse + b_dvv + b_svv + b_svv);
			friction_z = sa*(a_duv + a_duv + a_suv + a_suv) + sb*(b_duv + b_duv + b_suv + b_suv);
		}
		float ua_xt = Ad.x*ua.x + Ao.x*ua.y + Ao.y*ua.z, ua_yt = Ao.x*ua.x + Ad.y*ua.y + Ao.z*ua.z, ua_zt = Ao.y*ua.x + Ao.z*ua.y + Ad.z*ua.z;
		float va_xt = Ad.x*va.x + Ao.x*va.y + Ao.y*va.z, va_yt = Ao.x*va.x + Ad.y*va.y + Ao.z*va.z, va_zt = Ao.y*va.x + Ao.z*va.y + Ad.z*va.z;
		float ub_xt = Bd.x*ub.x + Bo.x*ub.y + Bo.y*ub.z, ub_yt = Bo.x*ub.x + Bd.y*ub.y + Bo.z*ub.z, ub_zt = Bo.y*ub.x + Bo.z*ub.y + Bd.z*ub.z;
		float vb_xt = Bd.x*vb.x + Bo.x*vb.y + Bo.y*vb.z, vb_yt = Bo.x*vb.x + Bd.y*vb.y + Bo.z*vb.z, vb_zt = Bo.y*vb.x + Bo.z*vb.y + Bd.z*vb.z;
		float* P = R.plane + j; const u32 S = R.stride;
		P[N_X*S] = normal_x; P[N_Y*S] = normal_y; P[N_Z*S] = normal_z;
		P[PA_X*S] = pa.x; P[PA_Y*S] = pa.y; P[PA_Z*S] = pa.z; P[PB_X*S] = pb.x; P[PB_Y*S] = pb.y; P[PB_Z*S] = pb.z;
		P[NVTNI*S] = nvtni; P[BIAS*S] = bias; P[FRICTION*S] = friction;
		P[U_X*S] = u.x; P[U_Y*S] = u.y; P[U_Z*S] = u.z; P[V_X*S] = v.x; P[V_Y*S] = v.y; P[V_Z*S] = v.z;
		P[FC_X*S] = friction_x; P[FC_Y*S] = friction_y; P[FC_Z*S] = friction_z;
		P[UA_X*S] = nb_neg(ua_xt); P[UA_Y*S] = nb_neg(ua_yt); P[UA_Z*S] = nb_neg(ua_zt);
		P[VA_X*S] = nb_neg(va_xt); P[VA_Y*S] = nb_neg(va_yt); P[VA_Z*S] = nb_neg(va_zt);
		P[NA_X*S] = nb_neg(na_x); P[NA_Y*S] = nb_neg(na_y); P[NA_Z*S] = nb_neg(na_z);
		P[UB_X*S] = ub_xt; P[UB_Y*S] = ub_yt; P[UB_Z*S] = ub_zt; P[VB_X*S] = vb_xt; P[VB_Y*S] = vb_yt; P[VB_Z*S] = vb_zt;
		P[NB_X*S] = nb_x; P[NB_Y*S] = nb_y; P[NB_Z*S] = nb_z;
		P[MASS_A*S] = a_mass_inverse; P[MASS_B*S] = b_mass_inverse;
		R.a[j] = a; R.b[j] = b;
	}
}

// ---------------- solver working set: momentum rows with an embedded token ----------------
// mw[2*body] = (velocity.xyz, token), mw[2*body+1] = (angular_velocity.xyz, token).  Each 16-byte half is read and written
// with single 128-bit relaxed GPU-scope accesses, so a half is always seen whole and carries the token of the contact
// that wrote it: the data validates itself, no fence and no separate flag are needed.
NB_DEV float4 ld128(const float4* p) {
	float4 v;
	asm volatile("{\n .reg .b128 q;\n ld.relaxed.gpu.global.b128 q, [%4];\n mov.b128 {%0,%1,%2,%3}, q;\n}" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
	return v;
}
NB_DEV void st128(float4* p, float4 v) {
	asm volatile("{\n .reg .b128 q;\n mov.b128 q, {%1,%2,%3,%4};\n st.relaxed.gpu.global.b128 [%0], q;\n}" :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__global__ void __launch_bounds__(NB_BLOCK) k_mw_in(u32 B, const nb_body_momentum* momentum, float4* mw) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
		const float4* p = reinterpret_cast<const float4*>(momentum + i);
		float4 l = p[0], w = p[1];
		l.w = 0.0f; w.w = 0.0f;  // token 0 = "nobody has written this body yet"
		mw[2*i] = l; mw[2*i + 1] = w;
	}
}
// mode 1 (sweeps): unused1 of touched bodies is zeroed like nudge.cpp:4823, 4849; unused0 keeps the inverse mass (4825-4827)
__global__ void __launch_bounds__(NB_BLOCK) k_mw_out(u32 B, nb_body_momentum* momentum, const float4* mw, int mode) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
		float4* p = reinterpret_cast<float4*>(momentum + i);
		float4 l = mw[2*i], w = mw[2*i + 1];
		float4 ol = p[0], ow = p[1];
		bool touched = asu(l.w) != 0;
		p[0] = make_float4(l.x, l.y, l.z, ol.w);
		p[1] = make_float4(w.x, w.y, w.z, (mode && touched) ? 0.0f : ow.w);
	}
}

// rcpps / rsqrtps of the solver arithmetic as a policy: LutMath reproduces the host CPU's instructions bit for bit (parity mode),
// FastMath uses the GPU's own reciprocal / rsqrt (throughput mode: more accurate, not bit-comparable with the reference).
struct LutMath {
	const u32* rcp_lut; const u32* rsqrt_lut;
	NB_DEV float rcp(float x) const { return nb_rcp_t(x, rcp_lut); }
	NB_DEV float rsqrt(float x) const { return nb_rsqrt_t(x, rsqrt_lut); }
};
struct FastMath {
	NB_DEV float rcp(float x) const { return __frcp_rn(x); }
	NB_DEV float rsqrt(float x) const { return rsqrtf(x); }   // rsqrt(0) = inf, rsqrt(<0) = NaN like rsqrtps
};

// One contact of the warm start (nudge.cpp:4563-4632); momentum rows passed in registers and updated in place.
// `state` points at the contact's slot in the three state planes (stride S floats apart).
// P[k*PS] = row plane k of this contact (global planes: P = R.plane + slot, PS = R.stride; a shared-memory tile: P = tile + lane, PS = tile width).
template<class M>
NB_DEV void warm_start_contact_p(const float* P, const u32 S, const float4 ci, float* state, const u32 SS, float4& al, float4& aw, float4& bl, float4& bw, const M m) {
	float a_mass_inverse = P[MASS_A*S], b_mass_inverse = P[MASS_B*S];
	float n_x = P[N_X*S], n_y = P[N_Y*S], n_z = P[N_Z*S];
	float u_x = P[U_X*S], u_y = P[U_Y*S], u_z = P[U_Z*S], v_x = P[V_X*S], v_y = P[V_Y*S], v_z = P[V_Z*S];
	float normal_impulse = nb_max(n_x*ci.x + n_y*ci.y + n_z*ci.z, 0.0f);
	float max_friction_impulse = normal_impulse * P[FRICTION*S];
	float fix = u_x*ci.x + u_y*ci.y + u_z*ci.z;
	float fiy = v_x*ci.x + v_y*ci.y + v_z*ci.z;
	float fcs = fix*fix + fiy*fiy;
	fcs = m.rsqrt(fcs);
	fcs = fcs * max_friction_impulse;
	fcs = nb_min(1.0f, fcs);  // first operand on NaN
	fix = fix * fcs; fiy = fiy * fcs;
	float lx = fix*u_x + fiy*v_x + n_x * normal_impulse;
	float ly = fix*u_y + fiy*v_y + n_y * normal_impulse;
	float lz = fix*u_z + fiy*v_z + n_z * normal_impulse;
	float aax = fix*P[UA_X*S] + fiy*P[VA_X*S] + normal_impulse*P[NA_X*S];
	float aay = fix*P[UA_Y*S] + fiy*P[VA_Y*S] + normal_impulse*P[NA_Y*S];
	float aaz = fix*P[UA_Z*S] + fiy*P[VA_Z*S] + normal_impulse*P[NA_Z*S];
	float bax = fix*P[UB_X*S] + fiy*P[VB_X*S] + normal_impulse*P[NB_X*S];
	float bay = fix*P[UB_Y*S] + fiy*P[VB_Y*S] + normal_impulse*P[NB_Y*S];
	float baz = fix*P[UB_Z*S] + fiy*P[VB_Z*S] + normal_impulse*P[NB_Z*S];
	al.x -= lx * a_mass_inverse; al.y -= ly * a_mass_inverse; al.z -= lz * a_mass_inverse;
	aw.x += aax; aw.y += aay; aw.z += aaz;
	bl.x += lx * b_mass_inverse; bl.y += ly * b_mass_inverse; bl.z += lz * b_mass_inverse;
	bw.x += bax; bw.y += bay; bw.z += baz;
	state[0] = normal_impulse; state[SS] = fix; state[2*SS] = fiy;
}
template<class M>
NB_DEV void warm_start_contact(const Rows& R, u32 j, const float4* impulses, float4& al, float4& aw, float4& bl, float4& bw, const M m) {
	warm_start_contact_p(R.plane + j, R.stride, impulses[R.contact[j]], R.state + j, R.stride, al, aw, bl, bw, m);
}

// One contact of one projected Gauss-Seidel sweep (nudge.cpp:4646-4853), same operation order, FMAs where the source has madd.
// The rows arrive in registers (rv[], st[]): they are fetched BEFORE the contact starts waiting for its bodies.
template<class M>
NB_DEV void solve_contact(const Rows& R, u32 j, const float (&rv)[ROW_PLANES_TOTAL], const float (&st)[3], float4& al, float4& aw, float4& bl, float4& bw, const M m) {
	const u32 S = R.stride;
	float a_velocity_x = al.x, a_velocity_y = al.y, a_velocity_z = al.z, a_mass_inverse = rv[MASS_A];
	float a_angular_velocity_x = aw.x, a_angular_velocity_y = aw.y, a_angular_velocity_z = aw.z;
	float b_velocity_x = bl.x, b_velocity_y = bl.y, b_velocity_z = bl.z, b_mass_inverse = rv[MASS_B];
	float b_angular_velocity_x = bw.x, b_angular_velocity_y = bw.y, b_angular_velocity_z = bw.z;
	float pa_z = rv[PA_Z], pa_x = rv[PA_X], pa_y = rv[PA_Y];
	float v_xa = nb_madd(a_angular_velocity_y, pa_z, a_velocity_x);
	float v_ya = nb_madd(a_angular_velocity_z, pa_x, a_velocity_y);
	float v_za = nb_madd(a_angular_velocity_x, pa_y, a_velocity_z);
	float pb_z = rv[PB_Z], pb_x = rv[PB_X], pb_y = rv[PB_Y];
	float v_xb = nb_madd(b_angular_velocity_y, pb_z, b_velocity_x);
	float v_yb = nb_madd(b_angular_velocity_z, pb_x, b_velocity_y);
	float v_zb = nb_madd(b_angular_velocity_x, pb_y, b_velocity_z);
	v_xa = nb_madd(b_angular_velocity_z, pb_y, v_xa);
	v_ya = nb_madd(b_angular_velocity_x, pb_z, v_ya);
	v_za = nb_madd(b_angular_velocity_y, pb_x, v_za);
	float n_x = rv[N_X], fu_x = rv[U_X], fv_x = rv[V_X];
	v_xb = nb_madd(a_angular_velocity_z, pa_y, v_xb);
	v_yb = nb_madd(a_angular_velocity_x, pa_z, v_yb);
	v_zb = nb_madd(a_angular_velocity_y, pa_x, v_zb);
	float n_y = rv[N_Y], fu_y = rv[U_Y], fv_y = rv[V_Y];
	float v_x = v_xb - v_xa, v_y = v_yb - v_ya, v_z = v_zb - v_za;
	float t_z = n_x * v_x, t_x = v_x * fu_x, t_y = v_x * fv_x;
	float n_z = rv[N_Z], fu_z = rv[U_Z], fv_z = rv[V_Z];
	float normal_bias = rv[BIAS];
	float old_normal_impulse = st[0];
	float normal_factor = rv[NVTNI];
	t_z = nb_madd(n_y, v_y, t_z); t_x = nb_madd(v_y, fu_y, t_x); t_y = nb_madd(v_y, fv_y, t_y);
	normal_bias = normal_bias + old_normal_impulse;
	t_z = nb_madd(n_z, v_z, t_z); t_x = nb_madd(v_z, fu_z, t_x); t_y = nb_madd(v_z, fv_z, t_y);
	float normal_impulse = nb_madd(normal_factor, t_z, normal_bias);
	float t_xx = t_x*t_x, t_yy = t_y*t_y, t_xy = t_x*t_y;
	float tl2 = t_xx + t_yy;
	normal_impulse = nb_max(normal_impulse, 0.0f);
	t_x *= tl2; t_y *= tl2;
	R.state[0*S + j] = normal_impulse;
	float max_friction_impulse = normal_impulse * rv[FRICTION];
	normal_impulse = normal_impulse - old_normal_impulse;
	float friction_factor = t_xx * rv[FC_X];
	float linear_impulse_x = n_x * normal_impulse;
	friction_factor = nb_madd(t_yy, rv[FC_Y], friction_factor);
	float linear_impulse_y = n_y * normal_impulse;
	friction_factor = nb_madd(t_xy, rv[FC_Z], friction_factor);
	float linear_impulse_z = n_z * normal_impulse;
	friction_factor = m.rcp(friction_factor);
	a_angular_velocity_x = nb_madd(rv[NA_X], normal_impulse, a_angular_velocity_x);
	a_angular_velocity_y = nb_madd(rv[NA_Y], normal_impulse, a_angular_velocity_y);
	a_angular_velocity_z = nb_madd(rv[NA_Z], normal_impulse, a_angular_velocity_z);
	float old_friction_impulse_x = st[1], old_friction_impulse_y = st[2];
	friction_factor = nb_min(1e+6f, friction_factor);  // first operand on NaN
	float friction_impulse_x = t_x*friction_factor, friction_impulse_y = t_y*friction_factor;
	friction_impulse_x = old_friction_impulse_x - friction_impulse_x;
	friction_impulse_y = old_friction_impulse_y - friction_impulse_y;
	float friction_clamp_scale = friction_impulse_x*friction_impulse_x + friction_impulse_y*friction_impulse_y;
	friction_clamp_scale = m.rsqrt(friction_clamp_scale);
	b_angular_velocity_x = nb_madd(rv[NB_X], normal_impulse, b_angular_velocity_x);
	b_angular_velocity_y = nb_madd(rv[NB_Y], normal_impulse, b_angular_velocity_y);
	b_angular_velocity_z = nb_madd(rv[NB_Z], normal_impulse, b_angular_velocity_z);
	friction_clamp_scale = friction_clamp_scale * max_friction_impulse;
	friction_clamp_scale = nb_min(1.0f, friction_clamp_scale);
	friction_impulse_x = friction_impulse_x * friction_clamp_scale;
	friction_impulse_y = friction_impulse_y * friction_clamp_scale;
	R.state[1*S + j] = friction_impulse_x; R.state[2*S + j] = friction_impulse_y;
	friction_impulse_x -= old_friction_impulse_x;
	friction_impulse_y -= old_friction_impulse_y;
	linear_impulse_x = nb_madd(fu_x, friction_impulse_x, linear_impulse_x);
	linear_impulse_y = nb_madd(fu_y, friction_impulse_x, linear_impulse_y);
	linear_impulse_z = nb_madd(fu_z, friction_impulse_x, linear_impulse_z);
	linear_impulse_x = nb_madd(fv_x, friction_impulse_y, linear_impulse_x);
	linear_impulse_y = nb_madd(fv_y, friction_impulse_y, linear_impulse_y);
	linear_impulse_z = nb_madd(fv_z, friction_impulse_y, linear_impulse_z);
	float a_mass_inverse_neg = nb_neg(a_mass_inverse);
	al.x = nb_madd(linear_impulse_x, a_mass_inverse_neg, a_velocity_x);
	al.y = nb_madd(linear_impulse_y, a_mass_inverse_neg, a_velocity_y);
	al.z = nb_madd(linear_impulse_z, a_mass_inverse_neg, a_velocity_z);
	a_angular_velocity_x = nb_madd(rv[UA_X], friction_impulse_x, a_angular_velocity_x);
	a_angular_velocity_y = nb_madd(rv[UA_Y], friction_impulse_x, a_angular_velocity_y);
	a_angular_velocity_z = nb_madd(rv[UA_Z], friction_impulse_x, a_angular_velocity_z);
	aw.x = nb_madd(rv[VA_X], friction_impulse_y, a_angular_velocity_x);
	aw.y = nb_madd(rv[VA_Y], friction_impulse_y, a_angular_velocity_y);
	aw.z = nb_madd(rv[VA_Z], friction_impulse_y, a_angular_velocity_z);
	bl.x = nb_madd(linear_impulse_x, b_mass_inverse, b_velocity_x);
	bl.y = nb_madd(linear_impulse_y, b_mass_inverse, b_velocity_y);
	bl.z = nb_madd(linear_impulse_z, b_mass_inverse, b_velocity_z);
	b_angular_velocity_x = nb_madd(rv[UB_X], friction_impulse_x, b_angular_velocity_x);
	b_angular_velocity_y = nb_madd(rv[UB_Y], friction_impulse_x, b_angular_velocity_y);
	b_angular_velocity_z = nb_madd(rv[UB_Z], friction_impulse_x, b_angular_velocity_z);
	bw.x = nb_madd(rv[VB_X], friction_impulse_y, b_angular_velocity_x);
	bw.y = nb_madd(rv[VB_Y], friction_impulse_y, b_angular_velocity_y);
	bw.z = nb_madd(rv[VB_Z], friction_impulse_y, b_angular_velocity_z);
}

// mode 0: warm start (one pass); mode 1: `sweeps` PGS sweeps; mode 2: the warm start followed by `sweeps` sweeps in the same
// launch (nb_step: nothing happens between setup and the first sweep, so the two pipelines can overlap).  Co-resident grid, no barrier.  Thread t owns slots t, t+T, ...
// (so the per-contact solver state stays private to one thread) and walks them sweep by sweep; within and across threads the
// items are visited in increasing (sweep, slot), which is a topological order of the dependency graph, so the lowest
// unfinished item is always runnable.  Inside a warp the lanes poll instead of blocking, so a lane may depend on another
// lane of its own warp.  mw must come from k_mw_in (all tokens 0).
//
// Waiting: the body's token says how many applications are still ahead of this contact (k_chain_rank).  While that number is
// >= 2 on either body only the linear halves are polled, and the warp sleeps hop_ns per missing application when all of its
// lanes are that far away; from 1 on, all four halves are fetched in one round trip so the hand-off costs a single L2 access.
#define NB_SOLVE_BACKOFF_NS 150u  // hop_ns of k_solve and k_solve_flow (__nanosleep may sleep up to twice as long)
__global__ void __launch_bounds__(NB_BLOCK, 2) k_solve(Rows R, const float4* impulses, float4* mw, int mode, u32 sweeps, u32 hop_ns, u32* counts) {
	__shared__ u32 s_rcp[2048];
	__shared__ u32 s_rsqrt[2048];
	for (u32 i = threadIdx.x; i < 2048; i += blockDim.x) { s_rcp[i] = g_rcp_lut[i]; s_rsqrt[i] = g_rsqrt_lut[i]; }
	__syncthreads();
	const u32 NS = 8 * counts[CNT_BATCHES];
	const u32 tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
	const u32 passes = mode == 0 ? 1 : (mode == 1 ? sweeps : sweeps + 1);
	const u32 S = R.stride;
	for (u32 w = 0; w < passes; ++w) {
		const bool sweep = mode == 1 || (mode == 2 && w > 0);  // this pass is a PGS sweep (else: the warm start)
		for (u32 s0 = 0; s0 < NS; s0 += nth) {  // uniform trip count for the whole grid
			u32 slot = s0 + tid;
			bool pending = false, near = false;
			u32 a = 0, b = 0, exp_a = 0, exp_b = 0;
			float rv[ROW_PLANES_TOTAL], st[3];
			if (slot < NS && R.contact[slot] != NB_NONE) {
				pending = true;
				a = R.a[slot]; b = R.b[slot];
				uint2 wa = R.wait[slot], wb = R.wait[S + slot];
				exp_a = w * wa.y + wa.x; exp_b = w * wb.y + wb.x;
				if (sweep) {
					const float* c = R.plane + slot;
					#pragma unroll
					for (int k = 0; k < ROW_PLANES_TOTAL; ++k) rv[k] = c[(size_t)k * S];
					st[0] = R.state[0*S + slot]; st[1] = R.state[1*S + slot]; st[2] = R.state[2*S + slot];
				}
			}
			while (__any_sync(0xffffffffu, pending)) {
				u32 want = 0xffffffffu;
				if (pending) {
					float4 al = ld128(mw + 2*a), bl = ld128(mw + 2*b), aw, bw;
					if (near) { aw = ld128(mw + 2*a + 1); bw = ld128(mw + 2*b + 1); }
					u32 ra = a ? exp_a - asu(al.w) : 0, rb = b ? exp_b - asu(bl.w) : 0;
					u32 r = max(ra, rb);
					if (r == 0 && near && (!a || asu(aw.w) == exp_a) && (!b || asu(bw.w) == exp_b)) {
						if (sweep) solve_contact(R, slot, rv, st, al, aw, bl, bw, LutMath{ s_rcp, s_rsqrt });
						else warm_start_contact(R, slot, impulses, al, aw, bl, bw, LutMath{ s_rcp, s_rsqrt });
						if (a) { float tk = asf(exp_a + 1); al.w = tk; aw.w = tk; st128(mw + 2*a, al); st128(mw + 2*a + 1, aw); }  // body 0 is static: never written (DESIGN.md §1)
						if (b) { float tk = asf(exp_b + 1); bl.w = tk; bw.w = tk; st128(mw + 2*b, bl); st128(mw + 2*b + 1, bw); }
						pending = false;
					}
					else {
						near = r <= 1;
						want = r >= 2 ? (r - 1) * hop_ns : 0;
					}
				}
				want = __reduce_min_sync(0xffffffffu, want);
				if (want != 0xffffffffu && want) __nanosleep(min(want, 20000u));
			}
		}
	}
}

// ---------------- update_cached_impulses (nudge.cpp:4857-4884) ----------------
__global__ void __launch_bounds__(NB_BLOCK) k_update_impulses(Rows R, float4* impulses, const u32* counts) {
	u32 n = 8 * counts[CNT_BATCHES];
	for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
		if (R.contact[j] == NB_NONE) continue;
		const float* c = R.plane + j; const u32 S = R.stride;
		float s0 = R.state[0*S + j], s1 = R.state[1*S + j], s2 = R.state[2*S + j];
		float4* dst = impulses + R.contact[j];
		float4 v = *dst;
		v.x = s0*c[N_X*S] + s1*c[U_X*S] + s2*c[V_X*S];
		v.y = s0*c[N_Y*S] + s1*c[U_Y*S] + s2*c[V_Y*S];
		v.z = s0*c[N_Z*S] + s1*c[U_Z*S] + s2*c[V_Z*S];
		*dst = v;
	}
}

// ---------------- user gravity/damping loop (example/main.cpp:291-305) and advance (nudge.cpp:4886-4926) ----------------
__global__ void __launch_bounds__(NB_BLOCK) k_gravity_damping(const u32* active_idx, nb_body_momentum* momentum, float time_step, float gravity, float damping_base, const u32* counts) {
	u32 n = counts[CNT_ACTIVE];
	float damping = 1.0f - time_step*damping_base;
	float dv = gravity * time_step;
	for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
		u32 i = active_idx[k];
		float4* p = reinterpret_cast<float4*>(momentum + i);
		float4 l = p[0], w = p[1];
		l.y -= dv;
		l.x *= damping; l.y *= damping; l.z *= damping;
		w.x *= damping; w.y *= damping; w.z *= damping;
		p[0] = l; p[1] = w;
	}
}

__global__ void __launch_bounds__(NB_BLOCK) k_advance(const u32* active_idx, nb_transform* xf, const nb_body_momentum* momentum, uint8_t* idle, float time_step, const u32* counts) {
	u32 n = counts[CNT_ACTIVE];
	float half_time_step = 0.5f * time_step;
	for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
		u32 i = active_idx[k];
		const float4* mp = reinterpret_cast<const float4*>(momentum + i);
		float4 l = mp[0], w = mp[1];
		f3 velocity = mk3(l.x, l.y, l.z), angular_velocity = mk3(w.x, w.y, w.z);
		if (dot3(velocity, velocity) < 1e-2f && dot3(angular_velocity, angular_velocity) < 1e-1f) {
			uint8_t c = idle[i];
			if (c < 0xff) idle[i] = c + 1;
		}
		else idle[i] = 0;
		xform t = ld_xform(xf, i);
		quat dr; dr.v = angular_velocity; dr.s = 0.0f;
		dr = qmul(dr, mkq(t.q));
		dr.v = mul3(dr.v, half_time_step); dr.s *= half_time_step;
		t.p.x += velocity.x * time_step; t.p.y += velocity.y * time_step; t.p.z += velocity.z * time_step;
		t.q.x += dr.v.x; t.q.y += dr.v.y; t.q.z += dr.v.z; t.q.w += dr.s;
		float f = 1.0f / sqrtf(t.q.w*t.q.w + t.q.x*t.q.x + t.q.y*t.q.y + t.q.z*t.q.z);  // nudge.cpp:1128-1133
		t.q.x *= f; t.q.y *= f; t.q.z *= f; t.q.w *= f;
		st_xform(xf, i, t);
	}
}
