// nudge_b200 — body states between calls (nb_get_body_states, nb_set_body_states; DESIGN.md section 8.19).
//
// A reference application reads or sets a body's pose and velocity by touching its host BodyData between two calls.  Here those rows live in
// HBM, so the gather and the edit run on the device, with the bits that host read or edit followed by nb_upload_bodies gives, and with
// device pointers they can sit inside the application's CUDA graph.  Nothing here runs per step and nothing changes nb_step's graph.
//
// Gather, 1 launch: k_get_body_states, one thread per row.
// Set, 3 launches, as nb_apply_body_impulses: k_state_keys makes one key (body << ib) | list position per entry, an entry that fails the
// checks getting body = B so that it sorts after every valid one; nb_radix_sort orders them; k_body_states gives the last key of each run of
// one body a thread, which writes the run's last entry (the later entry's fields win, and the fields are the call's), the idle byte of a
// dynamic body and, for a pose set, the body's "moved" byte.  The thread of the first skipped key writes the skip count.  A pose set then
// runs nb_remove_bodies' wake on the moved bytes (launch_wake, nb_spawn_api.cuh).
// Included at the end of nb_api.cu.
#pragma once

// The checks of one entry, the same on the host (which refuses the call) and on the device (which skips the entry): not body 0, below the
// body count, and every selected field finite (x - x is 0 exactly for a finite x).
__host__ __device__ __forceinline__ bool body_state_ok(const nb_body_state& s, u32 fields, u32 B) {
	if (s.body == 0 || s.body >= B) return false;
	bool ok = true;
	if (fields & NB_BODY_POSE) {
		for (int k = 0; k < 3; ++k) ok &= s.position[k] - s.position[k] == 0.0f;
		for (int k = 0; k < 4; ++k) ok &= s.rotation[k] - s.rotation[k] == 0.0f;
	}
	if (fields & NB_BODY_VELOCITY) {
		for (int k = 0; k < 3; ++k) ok &= s.velocity[k] - s.velocity[k] == 0.0f;
		for (int k = 0; k < 3; ++k) ok &= s.angular_velocity[k] - s.angular_velocity[k] == 0.0f;
	}
	return ok;
}

// Row i = body bodies[i] (or i): transform (position, index read, rotation), momentum row (velocity, idle counter, angular velocity, 0).
__global__ void __launch_bounds__(NB_BLOCK) k_get_body_states(const u32* bodies, u32 n, u32 B, const nb_transform* xf, const nb_body_momentum* mom,
		const uint8_t* idle, nb_body_state* out) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const u32 b = bodies ? bodies[i] : i;
		float4* o = reinterpret_cast<float4*>(out + i);
		if (b >= B) {
			const float4 z = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
			o[0] = make_float4(0.0f, 0.0f, 0.0f, asf(NB_REMOVED_BODY)); o[1] = z; o[2] = z; o[3] = z;
			continue;
		}
		const float4* x = reinterpret_cast<const float4*>(xf + b);
		const float4* m = reinterpret_cast<const float4*>(mom + b);
		float4 p = x[0], v = m[0], w = m[1];
		p.w = asf(b); v.w = asf((u32)idle[b]); w.w = asf(0u);
		o[0] = p; o[1] = x[1]; o[2] = v; o[3] = w;
	}
}

__global__ void __launch_bounds__(NB_BLOCK) k_state_keys(const nb_body_state* rows, u32 n, u32 fields, u32 B, u32 ib, u64* keys, u32* n_out, u32* skipped) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const u32 body = body_state_ok(rows[i], fields, B) ? rows[i].body : B;
		keys[i] = ((u64)body << ib) | i;
		if (i == 0) { *n_out = n; if (skipped) *skipped = 0; }   // the sort's key count; the skip count unless k_body_states finds skips
	}
}

// keys: sorted.  A row is (position, body), rotation, (velocity, idle_counter), (angular_velocity, reserved).
__global__ void __launch_bounds__(NB_BLOCK) k_body_states(const nb_body_state* rows, const u64* keys, u32 n, u32 ib, u32 B, u32 fields, const uint8_t* kind,
		nb_transform* xf, nb_body_momentum* momentum, uint8_t* idle, uint8_t* moved, u32* skipped) {
	const u64 mask = ((u64)1 << ib) - 1;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const u64 k = keys[i];
		const u32 body = (u32)(k >> ib);
		if (body >= B) {   // the skipped entries, at the end
			if (skipped && (i == 0 || (u32)(keys[i - 1] >> ib) != body)) *skipped = n - i;
			continue;
		}
		if (i + 1 < n && (u32)(keys[i + 1] >> ib) == body) continue;   // not the run's last entry
		const float4* e = reinterpret_cast<const float4*>(rows + (k & mask));
		if (fields & NB_BODY_POSE) {
			float4* x = reinterpret_cast<float4*>(xf + body);
			float4 p = x[0];
			const float4 a = e[0];
			p.x = a.x; p.y = a.y; p.z = a.z;   // p.w, the transform's body word, goes back as it was read
			x[0] = p; x[1] = e[1];
			moved[body] = 1;
		}
		if (fields & NB_BODY_VELOCITY) {
			float4* m = reinterpret_cast<float4*>(momentum + body);
			float4 v = m[0], w = m[1];
			const float4 c = e[2], d = e[3];
			v.x = c.x; v.y = c.y; v.z = c.z; w.x = d.x; w.y = d.y; w.z = d.z;   // unused0 / unused1 go back as they were read
			m[0] = v; m[1] = w;
		}
		if (!kin_is(kind, body)) idle[body] = 0;
	}
}

extern "C" {

int nb_get_body_states(nb_context* ctx, const uint32_t* bodies, uint32_t n, nb_body_state* out, int on_device, void* stream) {
	NB_RANGE("nb_get_body_states");
	if (!n) return NB_OK;
	if (!out) { ctx->error = "null body state output"; return NB_ERR_ARGUMENT; }
	cudaStream_t st = (cudaStream_t)stream;
	const u32 B = ctx->B;
	if (on_device) {
		JOIN_UPLOADS();
		launch_grid(mk_launch(ctx, st), k_get_body_states, GRID(n), bodies, n, B, ctx->xf, ctx->mom, ctx->idle, out);
		CK(cudaGetLastError());
		return NB_OK;
	}
	if (!bodies && n > B) { ctx->error = "body states: " + std::to_string(n) + " rows of bodies 0 .. n-1, beyond the body count (" + std::to_string(B) + ")"; return NB_ERR_ARGUMENT; }
	if (bodies)
		for (u32 i = 0; i < n; ++i)
			if (bodies[i] >= B) { ctx->error = "body state " + std::to_string(i) + ": body " + std::to_string(bodies[i]) + " is at or beyond the body count (" + std::to_string(B) + ")"; return NB_ERR_ARGUMENT; }
	JOIN_UPLOADS();
	GROW(ctx->bs_rows, n, st);
	if (bodies) { GROW(ctx->bs_idx, n, st); CK(put_staged(ctx, ctx->bs_idx.p, bodies, sizeof(u32) * (size_t)n, st)); }
	launch_grid(mk_launch(ctx, st), k_get_body_states, GRID(n), bodies ? ctx->bs_idx.p : nullptr, n, B, ctx->xf, ctx->mom, ctx->idle, ctx->bs_rows.p);
	CK(cudaGetLastError());
	CK(cudaMemcpyAsync(out, ctx->bs_rows.p, sizeof(nb_body_state) * (size_t)n, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	return NB_OK;
}

int nb_set_body_states(nb_context* ctx, const nb_body_state* states, uint32_t n, uint32_t fields, uint32_t* skipped, int on_device, void* stream) {
	NB_RANGE("nb_set_body_states");
	if (!fields || (fields & ~(u32)(NB_BODY_POSE | NB_BODY_VELOCITY))) { ctx->error = "body states: fields must be a nonzero combination of NB_BODY_POSE and NB_BODY_VELOCITY"; return NB_ERR_ARGUMENT; }
	if (ctx->sharded) { ctx->error = "nb_set_body_states: not supported on a context of nb_shard_create"; return NB_ERR_ARGUMENT; }
	if ((fields & NB_BODY_POSE) && ctx->in_step) { ctx->error = "nb_set_body_states: NB_BODY_POSE between nb_collide and the nb_advance that ends its step"; return NB_ERR_ARGUMENT; }
	if (n && !states) { ctx->error = "null body state list"; return NB_ERR_ARGUMENT; }
	if (fields & NB_BODY_POSE)   // the wake reads a byte per body at both ends of every connection, as nb_remove_bodies' does
		for (u32 i = 0; i < ctx->nconn; ++i)
			if (ctx->conn_host[i].a >= ctx->B || ctx->conn_host[i].b >= ctx->B) {
				ctx->error = "nb_set_body_states: connection " + std::to_string(i) + " names a body at or beyond the body count (" + std::to_string(ctx->B) + ")";
				return NB_ERR_ARGUMENT;
			}
	const u32 B = ctx->B, ib = bits_for(n), bb = bits_for((u64)B + 1);   // bb: room for the skip key B
	if (ib + bb > 64) { ctx->error = "body states: too many entries for the sort key"; return NB_ERR_ARGUMENT; }
	cudaStream_t st = (cudaStream_t)stream;
	if (!on_device) {
		for (u32 i = 0; i < n; ++i)
			if (!body_state_ok(states[i], fields, B)) {
				const u32 b = states[i].body;
				ctx->error = "body state " + std::to_string(i) + ": body " + std::to_string(b) + " " +
					(b == 0 ? "is the static world" : b >= B ? "is at or beyond the body count (" + std::to_string(B) + ")" : std::string("has a selected field that is not finite"));
				return NB_ERR_ARGUMENT;
			}
		if (skipped) *skipped = 0;
	}
	if (!n) {
		if (on_device && skipped) CK(cudaMemsetAsync(skipped, 0, sizeof(u32), st));
		return NB_OK;
	}
	JOIN_UPLOADS();   // ordered like nb_upload_momentum, after a pending nb_upload_bodies side copy
	ALLOC(ctx->bs_n, 1); ALLOC(ctx->bs_sb.hist, 256 * (size_t)ctx->sms); ALLOC(ctx->bs_sb.bar, 2);
	for (int i = 0; i < 2; ++i) { GROW(ctx->bs_keys[i], n, st); ctx->bs_sb.keys[i] = ctx->bs_keys[i].p; }
	const nb_body_state* rows = states;
	if (!on_device) {
		GROW(ctx->bs_rows, n, st);
		CK(put_staged(ctx, ctx->bs_rows.p, states, sizeof(nb_body_state) * (size_t)n, st));
		rows = ctx->bs_rows.p;
	}
	u32* dskip = on_device ? skipped : nullptr;
	uint8_t* moved = (fields & NB_BODY_POSE) ? reinterpret_cast<uint8_t*>(ctx->offs) : nullptr;   // the removal's byte per body
	if (moved) CK(cudaMemsetAsync(moved, 0, B, st));
	const Launch L = mk_launch(ctx, st);
	launch_grid(L, k_state_keys, GRID(n), rows, n, fields, B, ib, ctx->bs_sb.keys[0], ctx->bs_n, dskip);
	const int cur = nb_radix_sort(L, ctx->bs_sb, ctx->bs_n, 0, (int)(ib + bb), false, 0);
	launch_grid(L, k_body_states, GRID(n), rows, ctx->bs_sb.keys[cur], n, ib, B, fields, kin_table(ctx), ctx->xf, ctx->mom, ctx->idle, moved, dskip);
	if (moved) launch_wake(ctx, L, moved, nullptr);
	CK(cudaGetLastError());
	return NB_OK;
}

}  // extern "C"
