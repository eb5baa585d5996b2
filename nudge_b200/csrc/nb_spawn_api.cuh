// nudge_b200 — spawning and despawning between steps (nb_add_bodies, nb_remove_bodies, nb_download_colliders, nb_download_connections;
// DESIGN.md section 8.10).
//
// A reference application spawns or despawns a body by editing its caller-owned arrays between two steps.  Here those arrays live in HBM,
// together with tables that hold body and collider indices (connections, filters, sensors, the kinematic set, user rows, the sensor overlap
// lists, the body force table), so the edit runs on the device and gives the bits that host edit followed by a re-upload gives (include/nudge_b200.h states it).
//
// Add is copies only: the new rows go to the ends of their arrays, and the filter / sensor entries of the existing spheres move up by the
// number of added boxes through a staging copy.
// Remove, nothing of it per step:
//   k_spawn_mark     a "removed" byte per body, scattered from the list (in the offs planes, which nb_collide overwrites anyway)
//   launch_wake      the wake, shared with nb_set_body_states (nb_body_state_api.cuh), where "removed" reads "moved":
//     k_spawn_flags  the colliders' (tag, body, removed) keys; the connection half of the wake set; for the removal also the keep flags of
//                    bodies, colliders (one counter for boxes, one for spheres, over boxes-then-spheres) and connections
//     nb_radix_sort  of those keys; k_spawn_wake then binary-searches both tags of every cache entry: the other side of a removed tag wakes
//   nb_scan_reduce + k_spawn_bodies / k_spawn_colliders / k_spawn_conns: the fused scan ranks each array once, and its consumer gathers the
//                    kept rows out of place into collide-stage scratch (the body gather also writes the old -> new map, and moves the
//                    body force rows into frc_spare)
//   k_spawn_rows     the kept user rows, by a host-computed permutation that re-levels them (nb_rows_api.cuh, level_rows)
//   k_spawn_overlaps the sensor overlap lists' bodies through the map
// then one synchronise for the new counts and largest tag, and device-to-device copies back.  No float atomics; the one atomic is a u32 max.
// Included at the end of nb_api.cu.
#pragma once

// Spawn counters, in words that k_reset_collide zeroes at every nb_collide (the broadphase's extent histogram): new body count, new box and
// sphere counts (one scan's two totals), new connection count, largest kept tag, key count of the wake sort.
enum { CNT_SPAWN_B = CNT_EXT_HIST, CNT_SPAWN_BOXES, CNT_SPAWN_SPHERES, CNT_SPAWN_CONN, CNT_SPAWN_MAXTAG, CNT_SPAWN_KEYS, CNT_SPAWN__N };

NB_DEV void spawn_wake(const uint8_t* kind, uint8_t* idle, u32 b) { if (b != 0 && !kin_is(kind, b)) idle[b] = 0; }

__global__ void __launch_bounds__(NB_BLOCK) k_spawn_mark(const u32* list, u32 n, uint8_t* removed) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) removed[list[i]] = 1;
}

// keys[k] = tag << kshift | body << 1 | removed.  A connection with exactly one removed side wakes the other.  With flags (the removal):
// flags[i] (body kept), flags[S + k] / flags[2S + k] (collider k kept and a box / a sphere), flags[3S + c] (connection kept).
__global__ void __launch_bounds__(NB_BLOCK) k_spawn_flags(u32 B, u32 nboxes, u32 K, u32 nconn, const uint8_t* removed, const nb_transform* box_xf,
		const u32* box_tags, const nb_transform* sph_xf, const u32* sph_tags, const nb_body_pair* conn, const uint8_t* kind, uint8_t* idle,
		u32* flags, u32 S, u64* keys, u32 kshift, u32* counts) {
	const u32 n = max(B, max(K, nconn));
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		if (i == 0) { counts[CNT_SPAWN_MAXTAG] = 1; counts[CNT_SPAWN_KEYS] = K; counts[CNT_SPAWN_BOXES] = 0; counts[CNT_SPAWN_SPHERES] = 0; counts[CNT_SPAWN_CONN] = 0; }
		if (flags && i < B) flags[i] = removed[i] ? 0u : 1u;
		if (i < K) {
			const bool box = i < nboxes;
			const u32 body = box ? box_xf[i].body : sph_xf[i - nboxes].body, tag = box ? box_tags[i] : sph_tags[i - nboxes];
			const u32 rem = removed[body];
			if (flags) { flags[S + i] = box && !rem; flags[2 * (size_t)S + i] = !box && !rem; }
			keys[i] = ((u64)tag << kshift) | ((u64)body << 1) | rem;
		}
		if (i < nconn) {
			const u32 a = conn[i].a, b = conn[i].b, ra = removed[a], rb = removed[b];
			if (flags) flags[3 * (size_t)S + i] = !(ra | rb);
			if (ra && !rb) spawn_wake(kind, idle, b);
			if (rb && !ra) spawn_wake(kind, idle, a);
		}
	}
}

// keys: sorted.  First key of tag `tag`'s run (or K).
NB_DEV u32 spawn_tag_run(const u64* keys, u32 K, u32 kshift, u32 tag) {
	u32 lo = 0, hi = K;
	while (lo < hi) { const u32 mid = (lo + hi) >> 1; if ((keys[mid] >> kshift) < tag) lo = mid + 1; else hi = mid; }
	return lo;
}
NB_DEV bool spawn_tag_removed(const u64* keys, u32 K, u32 kshift, u32 j, u32 tag) {
	for (; j < K && (u32)(keys[j] >> kshift) == tag; ++j) if (keys[j] & 1) return true;
	return false;
}
NB_DEV void spawn_wake_tag(const u64* keys, u32 K, u32 kshift, u32 j, u32 tag, const uint8_t* kind, uint8_t* idle) {
	const u64 bmask = ((u64)1 << (kshift - 1)) - 1;
	for (; j < K && (u32)(keys[j] >> kshift) == tag; ++j) if (!(keys[j] & 1)) spawn_wake(kind, idle, (u32)((keys[j] >> 1) & bmask));
}

// One thread per cache entry (key A | B << 32): a removed collider with tag B wakes every kept body with a collider of tag A, and vice versa.
__global__ void __launch_bounds__(NB_BLOCK) k_spawn_wake(const u64* cache_tags, const u64* keys, u32 K, u32 kshift, const uint8_t* kind, uint8_t* idle, const u32* counts) {
	const u32 n = counts[CNT_CACHE];
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const u64 t = cache_tags[i];
		const u32 ta = (u32)t, tb = (u32)(t >> 32);
		const u32 ja = spawn_tag_run(keys, K, kshift, ta), jb = spawn_tag_run(keys, K, kshift, tb);
		if (spawn_tag_removed(keys, K, kshift, jb, tb)) spawn_wake_tag(keys, K, kshift, ja, ta, kind, idle);
		if (spawn_tag_removed(keys, K, kshift, ja, ta)) spawn_wake_tag(keys, K, kshift, jb, tb, kind, idle);
	}
}

// Launched with NB_SCAN_GRID blocks after nb_scan_reduce<1> over the body flags.  map[i] = the new index of body i, or NB_REMOVED_BODY.
// With a body force table (frc non-null) its rows move too, their body field rewritten to the new index.
__global__ void __launch_bounds__(NB_BLOCK) k_spawn_bodies(u32 B, const u32* flags, const u32* block_sums, const nb_transform* xf, const nb_body_properties* props,
		const nb_body_momentum* mom, const uint8_t* idle, const uint8_t* kind, const nb_body_force* frc, nb_transform* xf_out, float4* props_out, float4* mom_out,
		uint8_t* idle_out, uint8_t* kind_out, nb_body_force* frc_out, u32* map) {
	scan_consume<1>(flags, 0, B, block_sums, [&](u32 i, const u32 (&v)[1], const u32 (&off)[1]) {
		if (!v[0]) { map[i] = NB_REMOVED_BODY; return; }
		const u32 d = off[0];
		st_xform(xf_out, d, ld_xform(xf, i));
		props_out[d] = reinterpret_cast<const float4*>(props)[i];
		const float4* m = reinterpret_cast<const float4*>(mom + i);
		mom_out[2 * d] = m[0]; mom_out[2 * d + 1] = m[1];
		idle_out[d] = idle[i];
		if (kind) kind_out[d] = kind[i];
		if (frc) {
			const float4* e = reinterpret_cast<const float4*>(frc + i);
			float4* o = reinterpret_cast<float4*>(frc_out + d);
			float4 a = e[0];
			a.x = asf(d);
			o[0] = a; o[1] = e[1]; o[2] = e[2];
		}
		map[i] = d;
	});
}

// Launched with NB_SCAN_GRID blocks after nb_scan_reduce<2> over the box / sphere flags of the colliders (boxes, then spheres).  Outputs by
// table index (boxes, then spheres): tags, transforms (body remapped), filter words, sensor bytes; box data by new box index and sphere radii
// by new sphere index.
__global__ void __launch_bounds__(NB_BLOCK) k_spawn_colliders(u32 nboxes, u32 K, const u32* flags, u32 S, const u32* block_sums, const u32* map,
		const u32* box_tags, const nb_box_collider* box_data, const nb_transform* box_xf, const u32* sph_tags, const nb_sphere_collider* sph_data,
		const nb_transform* sph_xf, const u32* filter, const uint8_t* sensor, u32* tag_out, float4* box_out, float* sph_out, nb_transform* xf_out,
		u32* filter_out, uint8_t* sensor_out, u32* counts) {
	const u32 kept_boxes = counts[CNT_SPAWN_BOXES];
	scan_consume<2>(flags, S, K, block_sums, [&](u32 i, const u32 (&v)[2], const u32 (&off)[2]) {
		if (!(v[0] | v[1])) return;
		const bool box = i < nboxes;
		const u32 j = box ? i : i - nboxes, d = box ? off[0] : kept_boxes + off[1];
		xform x = ld_xform(box ? box_xf : sph_xf, j);
		x.p.w = asf(map[asu(x.p.w)]);
		st_xform(xf_out, d, x);
		const u32 tag = box ? box_tags[j] : sph_tags[j];
		tag_out[d] = tag;
		atomicMax(&counts[CNT_SPAWN_MAXTAG], tag);
		if (box) box_out[off[0]] = reinterpret_cast<const float4*>(box_data)[j];
		else sph_out[off[1]] = sph_data[j].radius;
		if (filter) filter_out[d] = filter[i];
		if (sensor) sensor_out[d] = sensor[i];
	});
}

// Launched with NB_SCAN_GRID blocks after nb_scan_reduce<1> over the connection flags.
__global__ void __launch_bounds__(NB_BLOCK) k_spawn_conns(u32 nconn, const u32* flags, const u32* block_sums, const u32* map, const nb_body_pair* conn, uint2* out) {
	scan_consume<1>(flags, 0, nconn, block_sums, [&](u32 i, const u32 (&v)[1], const u32 (&off)[1]) {
		if (v[0]) out[off[0]] = make_uint2(map[conn[i].a], map[conn[i].b]);
	});
}

// out[p] = rows[perm[p]] with a and b remapped (the accumulated impulse and the rest of the row move with it).
__global__ void __launch_bounds__(NB_BLOCK) k_spawn_rows(const nb_constraint_row* rows, const u32* perm, u32 n, const u32* map, nb_constraint_row* out) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		nb_constraint_row r = rows[perm[i]];
		r.a = map[r.a]; r.b = map[r.b];
		out[i] = r;
	}
}

// The sensor overlap lists (tags, body_a, body_b as a uint4): bodies through the map; a side that is already NB_REMOVED_BODY stays so.
__global__ void __launch_bounds__(NB_BLOCK) k_spawn_overlaps(uint4* cur, uint4* old, u32 cap, const u32* map, const u32* counts) {
	const u32 ncur = min(counts[CNT_SENSOR_HITS], cap), nold = min(counts[CNT_SENSOR_OLD], cap);
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < ncur + nold; i += gridDim.x * blockDim.x) {
		uint4& e = i < ncur ? cur[i] : old[i - ncur];
		if (e.z != NB_REMOVED_BODY) e.z = map[e.z];
		if (e.w != NB_REMOVED_BODY) e.w = map[e.w];
	}
}

// The wake of rules (a) and (b) from one byte per body (`marked`, B of them): k_spawn_flags, then with colliders the sort of the (tag, body,
// marked) keys and k_spawn_wake over the contact cache.  keep_flags = the removal's keep-flag planes (ctx->flags), or null for a wake alone.
// 3 launches, 1 without colliders.  It uses collide-stage scratch (the step's sort buffers and the spawn counters), so it runs between steps.
static void launch_wake(nb_context* ctx, const Launch& L, const uint8_t* marked, u32* keep_flags) {
	const u32 B = ctx->B, nboxes = ctx->nboxes, K = ctx->nboxes + ctx->nspheres, nconn = ctx->nconn;
	const uint8_t* kind = kin_table(ctx);
	const u32 kshift = bits_for(B) + 1;
	launch_grid(L, k_spawn_flags, GRID(std::max(B, std::max(K, nconn))), B, nboxes, K, nconn, marked, ctx->box_xf, ctx->box_tags, ctx->sph_xf, ctx->sph_tags,
		ctx->conn, kind, ctx->idle, keep_flags, ctx->stride, ctx->sb.keys[0], kshift, ctx->counts);
	if (K) {
		const int cur = nb_radix_sort(L, ctx->sb, ctx->counts + CNT_SPAWN_KEYS, 0, (int)(ctx->tagbits + kshift), false, 0);
		launch_grid(L, k_spawn_wake, GRID(ctx->cfg.max_contacts), ctx->cache_tags, ctx->sb.keys[cur], K, kshift, kind, ctx->idle, ctx->counts);
	}
}

extern "C" {

int nb_remove_bodies(nb_context* ctx, const uint32_t* h, uint32_t n, void* stream) {
	NB_RANGE("nb_remove_bodies");
	ctx->report_ok = false;
	if (ctx->sharded) { ctx->error = "nb_remove_bodies: not supported on a context of nb_shard_create"; return NB_ERR_ARGUMENT; }
	if (!n) return NB_OK;
	if (!h) { ctx->error = "null body list"; return NB_ERR_ARGUMENT; }
	for (u32 i = 0; i < n; ++i) if (int r = check_body(ctx, "removed body", i, h[i], true)) return r;
	if (int r = bodies_distinct(ctx, "removed body", n, [&](u32 i) { return h[i]; })) return r;
	std::vector<u32> list(h, h + n);
	std::sort(list.begin(), list.end());   // for the binary searches of the remap
	const u32 S = ctx->stride, B = ctx->B, nboxes = ctx->nboxes, K = ctx->nboxes + ctx->nspheres, nconn = ctx->nconn;
	// the body map covers bodies below B: a row or connection naming a body beyond it (which their uploads allow) has no new index
	const RowLevels& us = ctx->urow_set;
	for (u32 i = 0; i < us.n; ++i)
		if (us.ab[i].a >= B || us.ab[i].b >= B) { ctx->error = "constraint row " + std::to_string(i) + " names a body at or beyond the body count (" + std::to_string(B) + ")"; return NB_ERR_ARGUMENT; }
	for (u32 i = 0; i < nconn; ++i)
		if (ctx->conn_host[i].a >= B || ctx->conn_host[i].b >= B) { ctx->error = "connection " + std::to_string(i) + " names a body at or beyond the body count (" + std::to_string(B) + ")"; return NB_ERR_ARGUMENT; }
	if (nconn > S) { ctx->error = "more connections than the context's scratch stride (" + std::to_string(S) + ")"; return NB_ERR_CAPACITY; }
	// host side of the edit: the new kinematic set and the kept user rows, re-levelled
	auto removed = [&](u32 b) { return std::binary_search(list.begin(), list.end(), b); };
	auto remap = [&](u32 b) { return b - (u32)(std::lower_bound(list.begin(), list.end(), b) - list.begin()); };
	std::vector<u32> kin;
	for (u32 b : ctx->kin_list) if (!removed(b)) kin.push_back(remap(b));
	std::vector<nb_ccd_body> ccd;   // the kept continuous-collision entries, renumbered (the remap keeps them ascending)
	for (nb_ccd_body e : ctx->ccd) if (!removed(e.body)) { e.body = remap(e.body); ccd.push_back(e); }
	std::vector<nb_body_pair> ab;
	std::vector<u32> src;   // old device position of each kept row, in upload order
	for (u32 i = 0; i < us.n; ++i) {
		const nb_body_pair p = us.ab[i];
		if (removed(p.a) || removed(p.b)) continue;
		ab.push_back({ remap(p.a), remap(p.b) }); src.push_back(us.order[i]);
	}
	RowLevels kept;   // fewer rows on the same bodies: no more levels than the set had
	if (int r = level_rows(ctx, std::move(ab), kept, "constraint rows")) return r;
	std::vector<nb_body_pair> conn;   // the host copy of the kept connections
	for (u32 i = 0; i < nconn; ++i) {
		const nb_body_pair p = ctx->conn_host[i];
		if (!removed(p.a) && !removed(p.b)) conn.push_back({ remap(p.a), remap(p.b) });
	}
	// the kept joints with their current impulses, remapped, their drives and springs renumbered, and the kept dynamic bodies that lose a joint
	cudaStream_t st = (cudaStream_t)stream;
	JointBundle jb;
	if (int r = get_joint_bundle(ctx, jb, st)) return r;
	std::vector<u32> joint_wake, joint_new(jb.joints.size(), ~0u);   // joint_new: old joint index -> new one (~0u: deleted)
	u32 kept_joints = 0;
	for (u32 i = 0; i < jb.joints.size(); ++i) {
		nb_joint j = jb.joints[i];
		if (removed(j.a) || removed(j.b)) {
			const u32 other = removed(j.a) ? j.b : j.a;
			if (other && !removed(other) && !std::binary_search(kin.begin(), kin.end(), remap(other))) joint_wake.push_back(remap(other));
			continue;
		}
		j.a = remap(j.a); j.b = remap(j.b);
		joint_new[i] = kept_joints;
		jb.joints[kept_joints++] = j;
	}
	jb.joints.resize(kept_joints);
	auto renumber = [&](auto& entries) {   // the entries of the kept joints, in joint order
		size_t k = 0;
		for (auto e : entries) if (joint_new[e.joint] != ~0u) { e.joint = joint_new[e.joint]; entries[k++] = e; }
		entries.resize(k);
	};
	renumber(jb.drives); renumber(jb.springs);
	const u32 nrows = kept.n;
	const bool rows_changed = nrows != us.n;   // a deleted row can change the levels, which nb_step's graph holds
	std::vector<u32> staging(list);   // the list, then the rows' gather permutation (new device position -> old one)
	staging.resize((size_t)n + nrows);
	for (u32 j = 0; j < nrows; ++j) staging[n + kept.order[j]] = src[j];

	JOIN_UPLOADS();   // the gathers read the momentum and property rows
	GROW(ctx->spawn_idx, std::max(staging.size(), joint_wake.size()), st);
	GROW(ctx->urows_spare, nrows, st);
	// pageable staging: the copy has consumed it when cudaMemcpyAsync returns
	CK(cudaMemcpyAsync(ctx->spawn_idx.p, staging.data(), sizeof(u32) * staging.size(), cudaMemcpyHostToDevice, st));
	Launch L = mk_launch(ctx, stream);
	uint8_t* rem = reinterpret_cast<uint8_t*>(ctx->offs);
	u32* flags = ctx->flags;
	u32* counts = ctx->counts;
	u32* map = ctx->parent;
	CK(cudaMemsetAsync(rem, 0, B, st));
	launch_grid(L, k_spawn_mark, GRID(n), ctx->spawn_idx.p, n, rem);
	launch_wake(ctx, L, rem, flags);
	// bodies: xf -> mw, properties -> inertia, idle -> taint, kind -> active (each rewritten by the step before it is read: k_mw_in, k_inertia,
	// k_uf_init); momentum -> jd, the throughput solver's accumulator, which must be all zeros between passes and is cleared after the copy back
	nb_scan_reduce<1>(L, flags, S, nullptr, B, ctx->block_sums, counts + CNT_SPAWN_B);
	launch_grid(L, k_spawn_bodies, NB_SCAN_GRID, B, flags, ctx->block_sums, ctx->xf, ctx->props, ctx->mom, ctx->idle, ctx->kind, ctx->has_frc ? ctx->frc : nullptr,
		reinterpret_cast<nb_transform*>(ctx->mw), ctx->inertia, ctx->jd, reinterpret_cast<uint8_t*>(ctx->taint), reinterpret_cast<uint8_t*>(ctx->active), ctx->frc_spare, map);
	// colliders, by table index: tags -> col_tag, transforms -> world_xf, filter -> order, sensor -> rank; box data -> aabb_min, radii -> col_body
	if (K) {
		nb_scan_reduce<2>(L, flags + S, S, nullptr, K, ctx->block_sums, counts + CNT_SPAWN_BOXES);
		launch_grid(L, k_spawn_colliders, NB_SCAN_GRID, nboxes, K, flags + S, S, ctx->block_sums, map, ctx->box_tags, ctx->box_data, ctx->box_xf,
			ctx->sph_tags, ctx->sph_data, ctx->sph_xf, ctx->has_filter ? ctx->filter : nullptr, ctx->has_sensor ? ctx->sensor : nullptr,
			ctx->front.col_tag, ctx->front.aabb_min, reinterpret_cast<float*>(ctx->front.col_body), ctx->front.world_xf, ctx->front.order, reinterpret_cast<uint8_t*>(ctx->front.rank), counts);
	}
	if (nconn) {
		nb_scan_reduce<1>(L, flags + 3 * (size_t)S, S, nullptr, nconn, ctx->block_sums, counts + CNT_SPAWN_CONN);
		launch_grid(L, k_spawn_conns, NB_SCAN_GRID, nconn, flags + 3 * (size_t)S, ctx->block_sums, map, ctx->conn, reinterpret_cast<uint2*>(ctx->conn_scratch));
	}
	if (nrows) launch_grid(L, k_spawn_rows, GRID(nrows), ctx->urows.p, ctx->spawn_idx.p + n, nrows, map, ctx->urows_spare.p);
	if (ctx->has_sensor) launch_grid(L, k_spawn_overlaps, GRID(2 * (size_t)ctx->sensor_cap), ctx->sensor_cur.p, ctx->sensor_old.p, ctx->sensor_cap, map, counts);
	CK(cudaGetLastError());
	u32 c[CNT_SPAWN__N - CNT_SPAWN_B];
	CK(cudaMemcpyAsync(c, counts + CNT_SPAWN_B, sizeof(c), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	const u32 B2 = c[0], nb2 = c[CNT_SPAWN_BOXES - CNT_SPAWN_B], ns2 = c[CNT_SPAWN_SPHERES - CNT_SPAWN_B], nc2 = c[CNT_SPAWN_CONN - CNT_SPAWN_B];
	const u32 maxtag = c[CNT_SPAWN_MAXTAG - CNT_SPAWN_B];
	// back into place
	auto d2d = [&](void* dst, const void* s, size_t bytes) { return bytes ? cudaMemcpyAsync(dst, s, bytes, cudaMemcpyDeviceToDevice, st) : cudaSuccess; };
	CK(d2d(ctx->xf, ctx->mw, sizeof(nb_transform) * (size_t)B2)); CK(d2d(ctx->props, ctx->inertia, sizeof(nb_body_properties) * (size_t)B2));
	CK(d2d(ctx->mom, ctx->jd, sizeof(nb_body_momentum) * (size_t)B2)); CK(d2d(ctx->idle, ctx->taint, B2));
	CK(cudaMemsetAsync(ctx->jd, 0, sizeof(nb_body_momentum) * (size_t)B2, st));
	if (ctx->kind) { CK(d2d(ctx->kind, ctx->active, B2)); CK(cudaMemsetAsync(ctx->kind + B2, 0, B - B2, st)); }   // bodies added later are dynamic
	if (ctx->has_frc) CK(d2d(ctx->frc, ctx->frc_spare, sizeof(nb_body_force) * (size_t)B2));
	CK(d2d(ctx->box_tags, ctx->front.col_tag, 4 * (size_t)nb2)); CK(d2d(ctx->sph_tags, ctx->front.col_tag + nb2, 4 * (size_t)ns2));
	CK(d2d(ctx->box_xf, ctx->front.world_xf, sizeof(nb_transform) * (size_t)nb2)); CK(d2d(ctx->sph_xf, ctx->front.world_xf + nb2, sizeof(nb_transform) * (size_t)ns2));
	CK(d2d(ctx->box_data, ctx->front.aabb_min, sizeof(nb_box_collider) * (size_t)nb2)); CK(d2d(ctx->sph_data, ctx->front.col_body, sizeof(nb_sphere_collider) * (size_t)ns2));
	if (ctx->has_filter) CK(d2d(ctx->filter, ctx->front.order, 4 * ((size_t)nb2 + ns2)));
	if (ctx->has_sensor) CK(d2d(ctx->sensor, ctx->front.rank, (size_t)nb2 + ns2));
	CK(d2d(ctx->conn, ctx->conn_scratch, sizeof(nb_body_pair) * (size_t)nc2));
	CK(d2d(ctx->urows.p, ctx->urows_spare.p, sizeof(nb_constraint_row) * (size_t)nrows));
	ctx->B = B2; ctx->nboxes = nb2; ctx->nspheres = ns2; ctx->nconn = nc2;
	ctx->conn_host.swap(conn);
	ctx->tagbits = bits_for((u64)maxtag + 1);
	ctx->kbits = bits_for(std::max(1u, nb2 + ns2));
	if (ctx->has_kin) {
		if (kin.empty()) drop_kinematic(ctx);
		else ctx->kin_list.swap(kin);
	}
	ctx->urow_set = std::move(kept);
	ctx->scene_edited = true;
	// nb_step's graph keys on B, the collider and connection counts, tagbits and kbits, so it re-records when they change; table contents
	// are read through unchanged pointers.  The row levels are host values inside the graph.
	if (rows_changed) ++ctx->graph_epoch;
	if (int r = wake_bodies(ctx, joint_wake, st)) return r;
	if (int r = put_joint_bundle(ctx, jb, st)) return r;
	if (int r = set_ccd(ctx, std::move(ccd), st)) return r;
	return build_conn_lookup(ctx, st);
}

int nb_add_bodies(nb_context* ctx, const nb_body_data* bodies, const nb_collider_data* colliders, const nb_spawn_tables* tables, void* stream) {
	NB_RANGE("nb_add_bodies");
	ctx->report_ok = false;
	if (ctx->sharded) { ctx->error = "nb_add_bodies: not supported on a context of nb_shard_create"; return NB_ERR_ARGUMENT; }
	const u32 n = bodies ? bodies->count : 0, nb = colliders ? colliders->boxes.count : 0, ns = colliders ? colliders->spheres.count : 0;
	if (n && (!bodies->transforms || !bodies->properties || !bodies->momentum || !bodies->idle_counters)) { ctx->error = "null body array"; return NB_ERR_ARGUMENT; }
	if (nb && (!colliders->boxes.tags || !colliders->boxes.data || !colliders->boxes.transforms)) { ctx->error = "null box array"; return NB_ERR_ARGUMENT; }
	if (ns && (!colliders->spheres.tags || !colliders->spheres.data || !colliders->spheres.transforms)) { ctx->error = "null sphere array"; return NB_ERR_ARGUMENT; }
	const nb_collision_filter* f = tables ? tables->filters : nullptr;
	const uint8_t* sf = tables ? tables->sensor_flags : nullptr;
	if (f && !ctx->has_filter) { ctx->error = "a collision filter table was given but the context has none"; return NB_ERR_ARGUMENT; }
	if (sf && !ctx->has_sensor) { ctx->error = "a sensor table was given but the context has none"; return NB_ERR_ARGUMENT; }
	if (nb + ns && ctx->has_filter && !f) { ctx->error = "the context has a collision filter table: give the added colliders' entries"; return NB_ERR_ARGUMENT; }
	if (nb + ns && ctx->has_sensor && !sf) { ctx->error = "the context has a sensor table: give the added colliders' flags"; return NB_ERR_ARGUMENT; }
	if ((u64)ctx->B + n > ctx->cfg.max_bodies) { ctx->error = "too many bodies"; return NB_ERR_CAPACITY; }
	if ((u64)ctx->nboxes + nb > ctx->cfg.max_boxes || (u64)ctx->nspheres + ns > ctx->cfg.max_spheres) { ctx->error = "too many colliders"; return NB_ERR_CAPACITY; }
	const u32 B0 = ctx->B, B2 = ctx->B + n;
	u32 maxtag = 1;
	for (u32 i = 0; i < nb + ns; ++i) {
		const nb_transform& x = i < nb ? colliders->boxes.transforms[i] : colliders->spheres.transforms[i - nb];
		if (x.body >= B2) { ctx->error = "added collider " + std::to_string(i) + " names body " + std::to_string(x.body) + ", at or beyond the new body count (" + std::to_string(B2) + ")"; return NB_ERR_ARGUMENT; }
		maxtag = std::max(maxtag, i < nb ? colliders->boxes.tags[i] : colliders->spheres.tags[i - nb]);
	}
	if (!n && !nb && !ns) return NB_OK;
	cudaStream_t st = (cudaStream_t)stream;
	JOIN_UPLOADS();   // ordered like nb_upload_momentum, after a pending nb_upload_bodies side copy
	// every host array through the staging copy: the caller's arrays may be reused when the call returns, pinned or not
	CK(put_staged(ctx, ctx->xf + B0, bodies ? bodies->transforms : nullptr, sizeof(nb_transform) * (size_t)n, st));
	CK(put_staged(ctx, ctx->props + B0, bodies ? bodies->properties : nullptr, sizeof(nb_body_properties) * (size_t)n, st));
	CK(put_staged(ctx, ctx->mom + B0, bodies ? bodies->momentum : nullptr, sizeof(nb_body_momentum) * (size_t)n, st));
	CK(put_staged(ctx, ctx->idle + B0, bodies ? bodies->idle_counters : nullptr, (size_t)n, st));
	if (ctx->kind && n) CK(cudaMemsetAsync(ctx->kind + B0, 0, n, st));   // new bodies are dynamic
	std::vector<nb_body_force> frc;   // with the default force entry
	if (ctx->has_frc && n) {
		for (u32 i = 0; i < n; ++i) frc.push_back(default_body_force(B0 + i));
		CK(put_staged(ctx, ctx->frc + B0, frc.data(), sizeof(nb_body_force) * (size_t)n, st));
	}
	const u32 ob = ctx->nboxes, os = ctx->nspheres;
	if (nb) {
		CK(put_staged(ctx, ctx->box_tags + ob, colliders->boxes.tags, 4 * (size_t)nb, st)); CK(put_staged(ctx, ctx->box_data + ob, colliders->boxes.data, sizeof(nb_box_collider) * (size_t)nb, st));
		CK(put_staged(ctx, ctx->box_xf + ob, colliders->boxes.transforms, sizeof(nb_transform) * (size_t)nb, st));
	}
	if (ns) {
		CK(put_staged(ctx, ctx->sph_tags + os, colliders->spheres.tags, 4 * (size_t)ns, st)); CK(put_staged(ctx, ctx->sph_data + os, colliders->spheres.data, sizeof(nb_sphere_collider) * (size_t)ns, st));
		CK(put_staged(ctx, ctx->sph_xf + os, colliders->spheres.transforms, sizeof(nb_transform) * (size_t)ns, st));
	}
	// per-collider tables [old boxes][new boxes][old spheres][new spheres]: the old sphere entries move up by nb through a staging copy in
	// collide-stage scratch (the two ranges may overlap)
	if (ctx->has_filter && nb + ns) {
		if (nb && os) {
			CK(cudaMemcpyAsync(ctx->front.order, ctx->filter + ob, 4 * (size_t)os, cudaMemcpyDeviceToDevice, st));
			CK(cudaMemcpyAsync(ctx->filter + ob + nb, ctx->front.order, 4 * (size_t)os, cudaMemcpyDeviceToDevice, st));
		}
		CK(put_staged(ctx, ctx->filter + ob, f, 4 * (size_t)nb, st));
		CK(put_staged(ctx, ctx->filter + ob + nb + os, f + nb, 4 * (size_t)ns, st));
	}
	if (ctx->has_sensor && nb + ns) {
		uint8_t* s = ctx->sensor;
		if (nb && os) {
			CK(cudaMemcpyAsync(ctx->front.rank, s + ob, os, cudaMemcpyDeviceToDevice, st));
			CK(cudaMemcpyAsync(s + ob + nb, ctx->front.rank, os, cudaMemcpyDeviceToDevice, st));
		}
		std::vector<uint8_t> flags01(nb + ns);
		for (u32 i = 0; i < nb + ns; ++i) flags01[i] = sf[i] ? 1 : 0;
		CK(put_staged(ctx, s + ob, flags01.data(), nb, st));
		CK(put_staged(ctx, s + ob + nb + os, flags01.data() + nb, ns, st));
	}
	ctx->B = B2; ctx->nboxes = ob + nb; ctx->nspheres = os + ns;
	ctx->tagbits = std::max(ctx->tagbits, bits_for((u64)maxtag + 1));   // bits_for is monotone: the same as over all tags
	ctx->kbits = bits_for(std::max(1u, ctx->nboxes + ctx->nspheres));
	ctx->scene_edited = true;   // the step's graph keys on the new counts
	CK(cudaGetLastError());
	return NB_OK;
}

int nb_download_colliders(nb_context* ctx, nb_collider_data* h, void* stream) {
	NB_RANGE("nb_download_colliders");
	if (!h) { ctx->error = "null collider struct"; return NB_ERR_ARGUMENT; }
	const u32 capb = h->boxes.count, caps = h->spheres.count;
	h->boxes.count = ctx->nboxes; h->spheres.count = ctx->nspheres;
	if (capb < ctx->nboxes || caps < ctx->nspheres) { ctx->error = "host collider arrays too small: " + std::to_string(ctx->nboxes) + " boxes, " + std::to_string(ctx->nspheres) + " spheres"; return NB_ERR_CAPACITY; }
	D2H(h->boxes.tags, ctx->box_tags, ctx->nboxes, u32); D2H(h->boxes.data, ctx->box_data, ctx->nboxes, nb_box_collider); D2H(h->boxes.transforms, ctx->box_xf, ctx->nboxes, nb_transform);
	D2H(h->spheres.tags, ctx->sph_tags, ctx->nspheres, u32); D2H(h->spheres.data, ctx->sph_data, ctx->nspheres, nb_sphere_collider); D2H(h->spheres.transforms, ctx->sph_xf, ctx->nspheres, nb_transform);
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	return NB_OK;
}

int nb_download_connections(nb_context* ctx, nb_body_connections* h, uint32_t capacity, void* stream) {
	NB_RANGE("nb_download_connections");
	if (!h) { ctx->error = "null connection struct"; return NB_ERR_ARGUMENT; }
	h->count = ctx->nconn;
	if (capacity < ctx->nconn) { ctx->error = "host connection array too small: " + std::to_string(ctx->nconn) + " connections"; return NB_ERR_CAPACITY; }
	D2H(h->data, ctx->conn, ctx->nconn, nb_body_pair);
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	return NB_OK;
}

}  // extern "C"
