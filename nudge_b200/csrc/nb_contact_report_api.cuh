// nudge_b200 — contact impulse reports (nb_get_body_contact_impulses, nb_get_contact_pair_impulses; DESIGN.md section 8.22).
//
// Both read what the last solved step left behind and nothing else: the contact set (fin, counts[CNT_CONTACTS]), its (tag, feature)
// order (sorted), the world impulses k_update_impulses wrote (impulses[c].xyz = J_c) and, for the lever arms, the row planes PA / PB of
// each contact's slot (rows.contact maps slot -> contact; 8 * counts[CNT_BATCHES] slots).  The step writes every one of them between
// nb_collide and nb_update_cached_impulses and nothing writes them after that until the next of those calls, so a report is legal while
// ctx->report_ok holds (set by nb_update_cached_impulses and by nb_step, cleared by every call that rewrites them or renumbers bodies).
// Nothing here runs per step and nothing changes nb_step's graph; the scratch is the calls' own.
//
// Per body, 3 launches: k_report_keys writes one key (body << (cb + 1)) | contact << 1 | side per contact side, at position 2c + side,
// with the side's slot as its value; nb_radix_sort orders them; k_body_report gives each requested row a warp, which finds the body's run
// of keys with two binary searches and sums the run in key order (ascending contact, side a before side b).
// Per pair, 5 launches: k_pair_heads flags the first contact of every run of equal tags in sorted order; nb_scan_reduce counts the runs;
// k_pair_sums (scan_consume) gives each run head a thread, which writes run r's row and its kept flag; nb_scan_reduce over the kept flags
// counts the kept rows into *count; k_pair_scatter (scan_consume) copies kept row r to out[rank] while rank < capacity.
// Included at the end of nb_api.cu.
#pragma once

static_assert(sizeof(nb_body_contact_impulse) == 32, "nb_body_contact_impulse is 32 bytes");
static_assert(sizeof(nb_contact_pair_impulse) == 48, "nb_contact_pair_impulse is 48 bytes");

// One key per contact side of the last solved step.  A body at or beyond the body count (possible only for nb_upload_contacts' rows) is
// keyed as B, which no valid row asks for.  Without slots (a schedule that overflowed publishes none) there are no keys.
__global__ void __launch_bounds__(NB_BLOCK) k_report_keys(const u32* slot_contact, const uint2* bodies, u32 B, u32 cb, u64* keys, u32* vals, u32* n_keys,
		const u32* counts) {
	const u32 slots = 8 * counts[CNT_BATCHES];
	if (blockIdx.x == 0 && threadIdx.x == 0) *n_keys = slots ? 2 * counts[CNT_CONTACTS] : 0u;
	for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < slots; j += gridDim.x * blockDim.x) {
		const u32 c = slot_contact[j];
		if (c == NB_NONE) continue;
		const uint2 ab = bodies[c];
		const u64 ka = min(ab.x, B), kb = min(ab.y, B);
		keys[2*c] = (ka << (cb + 1)) | ((u64)c << 1); vals[2*c] = j;
		keys[2*c + 1] = (kb << (cb + 1)) | ((u64)c << 1) | 1u; vals[2*c + 1] = j;
	}
}

// First position in keys[0, m) whose key is >= k.
NB_DEV u32 report_lower_bound(const u64* keys, u32 m, u64 k) {
	u32 lo = 0, hi = m;
	while (lo < hi) { const u32 mid = (lo + hi) >> 1; if (keys[mid] < k) lo = mid + 1; else hi = mid; }
	return lo;
}

// One warp per row.  Each lane loads one side of a chunk of 32 and forms J and cross(r, J) (independent per side); the sums then take
// the chunk's sides in order, every lane the same adds (shuffled from the side's lane), so the result is the sequential sum.
__global__ void __launch_bounds__(NB_BLOCK) k_body_report(const u32* bodies, u32 n, u32 B, u32 cb, const u64* keys, const u32* vals, const u32* n_keys,
		const float4* impulses, Rows R, nb_body_contact_impulse* out) {
	const u32 lane = threadIdx.x & 31, S = R.stride;
	const u32 m = *n_keys;
	for (u32 i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n; i += (gridDim.x * blockDim.x) >> 5) {
		const u32 b = bodies ? bodies[i] : i;
		float4* o = reinterpret_cast<float4*>(out + i);
		if (b >= B) {
			if (lane == 0) { o[0] = make_float4(0.0f, 0.0f, 0.0f, asf(NB_REMOVED_BODY)); o[1] = make_float4(0.0f, 0.0f, 0.0f, asf(0u)); }
			continue;
		}
		const u32 lo = report_lower_bound(keys, m, (u64)b << (cb + 1)), hi = report_lower_bound(keys, m, ((u64)b + 1) << (cb + 1));
		float ax = 0.0f, ay = 0.0f, az = 0.0f, tx = 0.0f, ty = 0.0f, tz = 0.0f;
		for (u32 base = lo; base < hi; base += 32) {
			const u32 k = base + lane;
			float jx = 0.0f, jy = 0.0f, jz = 0.0f, cx = 0.0f, cy = 0.0f, cz = 0.0f; u32 side = 0;
			if (k < hi) {
				const u64 key = keys[k];
				const u32 c = (u32)((key >> 1) & (((u64)1 << cb) - 1)), j = vals[k];
				side = (u32)key & 1u;
				const float* P = R.plane + j;
				const float rx = side ? P[PB_X*S] : P[PA_X*S], ry = side ? P[PB_Y*S] : P[PA_Y*S], rz = side ? P[PB_Z*S] : P[PA_Z*S];
				const float4 J = impulses[c];
				jx = J.x; jy = J.y; jz = J.z;
				cx = ry*jz - rz*jy; cy = rz*jx - rx*jz; cz = rx*jy - ry*jx;
			}
			const u32 cnt = min(32u, hi - base);
			for (u32 t = 0; t < cnt; ++t) {
				const float sx = __shfl_sync(0xffffffffu, jx, t), sy = __shfl_sync(0xffffffffu, jy, t), sz = __shfl_sync(0xffffffffu, jz, t);
				const float qx = __shfl_sync(0xffffffffu, cx, t), qy = __shfl_sync(0xffffffffu, cy, t), qz = __shfl_sync(0xffffffffu, cz, t);
				if (__shfl_sync(0xffffffffu, side, t)) { ax = ax + sx; ay = ay + sy; az = az + sz; tx = tx + qx; ty = ty + qy; tz = tz + qz; }
				else { ax = ax - sx; ay = ay - sy; az = az - sz; tx = tx - qx; ty = ty - qy; tz = tz - qz; }
			}
		}
		if (lane == 0) { o[0] = make_float4(ax, ay, az, asf(b)); o[1] = make_float4(tx, ty, tz, asf(hi - lo)); }
	}
}

// flags[j] = 1 for the first contact of a run of equal tags in sorted order
__global__ void __launch_bounds__(NB_BLOCK) k_pair_heads(const u32* sorted, const u64* tags, u32* flags, const u32* counts) {
	const u32 n = counts[CNT_CONTACTS];
	for (u32 j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x)
		flags[j] = (j == 0 || tags[sorted[j - 1]] != tags[sorted[j]]) ? 1u : 0u;
}

// NB_SCAN_GRID blocks, after nb_scan_reduce<1> over the head flags: run r's row (the contact event's walk of k_event_scatter, plus the
// normal impulse) and kept[r].
__global__ void __launch_bounds__(NB_BLOCK) k_pair_sums(const u32* heads, const u32* block_sums, const u32* sorted, const u64* tags, const float4* data,
		const uint2* bodies, const float4* impulses, float threshold, nb_contact_pair_impulse* rows, u32* kept, const u32* counts) {
	const u32 n = counts[CNT_CONTACTS];
	scan_consume<1>(heads, 0, n, block_sums, [&](u32 j, const u32 (&v)[1], const u32 (&off)[1]) {
		if (!v[0]) return;
		const u32 c0 = sorted[j];
		const u64 t = tags[c0];
		u32 deepest = c0, count = 0;
		float depth = data[2 * c0].w, ix = 0.0f, iy = 0.0f, iz = 0.0f, nsum = 0.0f;
		for (u32 k = j; k < n; ++k) {
			const u32 c = sorted[k];
			if (tags[c] != t) break;
			const float p = data[2 * c].w;
			if (p > depth) { depth = p; deepest = c; }   // strictly deeper: ties keep the earlier contact, a NaN never wins
			const float4 im = impulses[c], q = data[2 * c + 1];
			ix = ix + im.x; iy = iy + im.y; iz = iz + im.z;
			nsum = nsum + ((im.x*q.x + im.y*q.y) + im.z*q.z);
			++count;
		}
		const uint2 ab = bodies[deepest];
		uint4* o = reinterpret_cast<uint4*>(rows + off[0]);
		o[0] = make_uint4((u32)t, (u32)(t >> 32), ab.x, ab.y);
		o[1] = make_uint4(count, asu(nsum), asu(ix), asu(iy));
		o[2] = make_uint4(asu(iz), asu(data[2 * deepest].w), 0u, 0u);
		kept[off[0]] = (threshold == -INFINITY || nsum >= threshold) ? 1u : 0u;
	});
}

// NB_SCAN_GRID blocks, after nb_scan_reduce<1> over the kept flags of the n_runs runs
__global__ void __launch_bounds__(NB_BLOCK) k_pair_scatter(const u32* kept, const u32* block_sums, const u32* n_runs, const nb_contact_pair_impulse* rows,
		u32 capacity, nb_contact_pair_impulse* out) {
	scan_consume<1>(kept, 0, *n_runs, block_sums, [&](u32 r, const u32 (&v)[1], const u32 (&off)[1]) {
		if (!v[0] || off[0] >= capacity) return;
		const uint4* s = reinterpret_cast<const uint4*>(rows + r);
		uint4* o = reinterpret_cast<uint4*>(out + off[0]);
		o[0] = s[0]; o[1] = s[1]; o[2] = s[2];
	});
}

// The refusals both calls share: a context nb_shard_create was called on, and no solved step to report on.
static int report_legal(nb_context* ctx, const char* call) {
	if (ctx->sharded) { ctx->error = std::string(call) + ": not supported on a context of nb_shard_create"; return NB_ERR_ARGUMENT; }
	if (!ctx->report_ok) {
		ctx->error = std::string(call) + ": no solved step to report on (it is read after nb_update_cached_impulses or nb_step, and cleared by the calls "
			"that rewrite the contact set, the impulses or the solver rows, or renumber the bodies)";
		return NB_ERR_ARGUMENT;
	}
	return NB_OK;
}

extern "C" {

int nb_get_body_contact_impulses(nb_context* ctx, const uint32_t* bodies, uint32_t n, nb_body_contact_impulse* out, int on_device, void* stream) {
	NB_RANGE("nb_get_body_contact_impulses");
	if (int r = report_legal(ctx, "nb_get_body_contact_impulses")) return r;
	if (n && !out) { ctx->error = "null body contact impulse output"; return NB_ERR_ARGUMENT; }
	const u32 B = ctx->B, C = ctx->cfg.max_contacts, cb = bits_for(C), bb = bits_for((u64)B + 1);   // bb: room for the key of a body >= B
	if (bb + cb + 1 > 64) { ctx->error = "body contact impulses: the body and contact counts do not fit the sort key"; return NB_ERR_ARGUMENT; }
	if (!on_device) {
		if (!bodies && n > B) { ctx->error = "body contact impulses: " + std::to_string(n) + " rows of bodies 0 .. n-1, beyond the body count (" + std::to_string(B) + ")"; return NB_ERR_ARGUMENT; }
		if (bodies)
			for (u32 i = 0; i < n; ++i)
				if (bodies[i] >= B) { ctx->error = "body contact impulse " + std::to_string(i) + ": body " + std::to_string(bodies[i]) + " is at or beyond the body count (" + std::to_string(B) + ")"; return NB_ERR_ARGUMENT; }
	}
	if (!n) return NB_OK;
	cudaStream_t st = (cudaStream_t)stream;
	ALLOC(ctx->cr_n, 2); ALLOC(ctx->cr_sb.hist, 256 * (size_t)ctx->sms); ALLOC(ctx->cr_sb.bar, 2);
	for (int i = 0; i < 2; ++i) { ALLOC(ctx->cr_sb.keys[i], 2 * (size_t)C); ALLOC(ctx->cr_sb.vals[i], 2 * (size_t)C); }
	const u32* idx = bodies;
	nb_body_contact_impulse* dst = out;
	if (!on_device) {
		GROW(ctx->cr_rows, n, st);
		if (bodies) { GROW(ctx->cr_idx, n, st); CK(put_staged(ctx, ctx->cr_idx.p, bodies, sizeof(u32) * (size_t)n, st)); idx = ctx->cr_idx.p; }
		dst = ctx->cr_rows.p;
	}
	const Launch L = mk_launch(ctx, st);
	launch_grid(L, k_report_keys, GRID(ctx->cstride), ctx->rows.contact, ctx->fin.bodies, B, cb, ctx->cr_sb.keys[0], ctx->cr_sb.vals[0], ctx->cr_n, ctx->counts);
	const int cur = nb_radix_sort(L, ctx->cr_sb, ctx->cr_n, 0, (int)(bb + cb + 1), true, 0);
	launch_grid(L, k_body_report, GRID((size_t)n * 32), idx, n, B, cb, ctx->cr_sb.keys[cur], ctx->cr_sb.vals[cur], ctx->cr_n, ctx->impulses, ctx->rows, dst);
	CK(cudaGetLastError());
	if (!on_device) {
		CK(cudaMemcpyAsync(out, dst, sizeof(nb_body_contact_impulse) * (size_t)n, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
	}
	return NB_OK;
}

int nb_get_contact_pair_impulses(nb_context* ctx, float min_normal_impulse, nb_contact_pair_impulse* out, uint32_t capacity, uint32_t* count,
								 int on_device, void* stream) {
	NB_RANGE("nb_get_contact_pair_impulses");
	if (int r = report_legal(ctx, "nb_get_contact_pair_impulses")) return r;
	if (min_normal_impulse != min_normal_impulse) { ctx->error = "nb_get_contact_pair_impulses: the threshold is NaN"; return NB_ERR_ARGUMENT; }
	if (!count) { ctx->error = "null pair count"; return NB_ERR_ARGUMENT; }
	if (capacity && !out) { ctx->error = "null contact pair impulse output"; return NB_ERR_ARGUMENT; }
	cudaStream_t st = (cudaStream_t)stream;
	const u32 C = ctx->cfg.max_contacts;
	ALLOC(ctx->cp_n, 2); ALLOC(ctx->cp_heads, C); ALLOC(ctx->cp_kept, C); ALLOC(ctx->cp_rows, C); ALLOC(ctx->cp_block_sums, NB_SCAN_SUMS);
	const u32 cap = on_device ? capacity : std::min(capacity, C);   // more rows than contacts never exist
	nb_contact_pair_impulse* dst = out;
	u32* dcount = on_device ? count : ctx->cp_n + 1;
	if (!on_device) { GROW(ctx->cp_out, cap, st); dst = ctx->cp_out.p; }
	const Launch L = mk_launch(ctx, st);
	launch_grid(L, k_pair_heads, GRID(C), ctx->sorted, ctx->fin.tags, ctx->cp_heads, ctx->counts);
	nb_scan_reduce<1>(L, ctx->cp_heads, 0, ctx->counts + CNT_CONTACTS, 0, ctx->cp_block_sums, ctx->cp_n);
	launch_grid(L, k_pair_sums, NB_SCAN_GRID, ctx->cp_heads, ctx->cp_block_sums, ctx->sorted, ctx->fin.tags, ctx->fin.data, ctx->fin.bodies, ctx->impulses,
		min_normal_impulse, ctx->cp_rows, ctx->cp_kept, ctx->counts);
	nb_scan_reduce<1>(L, ctx->cp_kept, 0, ctx->cp_n, 0, ctx->cp_block_sums, dcount);
	launch_grid(L, k_pair_scatter, NB_SCAN_GRID, ctx->cp_kept, ctx->cp_block_sums, ctx->cp_n, ctx->cp_rows, cap, dst);
	CK(cudaGetLastError());
	if (on_device) return NB_OK;
	u32 kept = 0;
	CK(cudaMemcpyAsync(&kept, dcount, sizeof(u32), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	*count = kept;
	const u32 w = std::min(kept, cap);
	if (w) {
		CK(cudaMemcpyAsync(out, dst, sizeof(nb_contact_pair_impulse) * (size_t)w, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
	}
	if (kept > capacity) { ctx->error = "contact pair impulses: " + std::to_string(kept) + " rows are kept, the buffer holds " + std::to_string(capacity); return NB_ERR_CAPACITY; }
	return NB_OK;
}

}  // extern "C"
