// nudge_b200 — body impulses between calls (nb_apply_body_impulses, nb_apply_radial_impulse; DESIGN.md section 8.9).
//
// A reference application pushes, spins or wakes a body by editing its host BodyData between two calls (momentum[i] += ...;
// idle_counters[i] = 0).  Here those rows live in HBM, so the edit runs on the device, with the float32 operations the header spells out,
// and gives the bits that host loop gives.  Nothing here runs per step and nothing changes nb_step's graph.
//
// List path, 3 launches: k_impulse_keys makes one key (body << ib) | list position per entry, nb_radix_sort orders them (the keys are
// unique, so stability does not matter), and k_body_impulses gives one thread to each run of equal bodies: it loads the body's
// rotation, properties and momentum once, applies the run's entries in list order in registers, and writes the momentum row and the idle
// byte once.  No float atomics, so the result does not depend on scheduling.  Radial path, 1 launch: k_radial_impulse, grid-stride over
// the bodies, reads each position and touches properties, momentum and the idle byte only for the bodies it hits.
// Included at the end of nb_api.cu.
#pragma once
#include <cmath>

__global__ void __launch_bounds__(NB_BLOCK) k_impulse_keys(const nb_body_impulse* rows, u32 n, u32 ib, u64* keys, u32* n_out) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		keys[i] = ((u64)rows[i].body << ib) | i;
		if (i == 0) *n_out = n;   // the sort's key count
	}
}

// keys: sorted; the thread of a run's first key applies the whole run.  A row is 48 bytes: (body, offset), (impulse, angular.x),
// (angular.y, angular.z, reserved).
__global__ void __launch_bounds__(NB_BLOCK) k_body_impulses(const nb_body_impulse* rows, const u64* keys, u32 n, u32 ib, const nb_transform* xf,
		const nb_body_properties* props, nb_body_momentum* momentum, uint8_t* idle) {
	const u64 mask = ((u64)1 << ib) - 1;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const u64 k = keys[i];
		const u32 body = (u32)(k >> ib);
		if (i > 0 && (u32)(keys[i - 1] >> ib) == body) continue;
		const float4 pr = reinterpret_cast<const float4*>(props)[body];
		float3 Wd, Wo;
		world_inverse_inertia(reinterpret_cast<const float4*>(xf + body)[1], pr, Wd, Wo);
		float4* row = reinterpret_cast<float4*>(momentum + body);
		float4 v = row[0], w = row[1];
		for (u32 j = i; j < n; ++j) {
			const u64 kj = keys[j];
			if ((u32)(kj >> ib) != body) break;
			const float4* e = reinterpret_cast<const float4*>(rows + (kj & mask));
			const float4 a = e[0], b = e[1], c = e[2];   // a.yzw offset, b.xyz impulse, (b.w, c.x, c.y) angular impulse
			v.x += pr.w * b.x; v.y += pr.w * b.y; v.z += pr.w * b.z;
			const float tx = (a.z*b.z - a.w*b.y) + b.w;
			const float ty = (a.w*b.x - a.y*b.z) + c.x;
			const float tz = (a.y*b.y - a.z*b.x) + c.y;
			w.x += (Wd.x*tx + Wo.x*ty) + Wo.y*tz;
			w.y += (Wo.x*tx + Wd.y*ty) + Wo.z*tz;
			w.z += (Wo.y*tx + Wo.z*ty) + Wd.z*tz;
		}
		row[0] = v; row[1] = w;   // the w lanes (unused0, unused1) go back as they were read
		idle[body] = 0;
	}
}

__global__ void __launch_bounds__(NB_BLOCK) k_radial_impulse(nb_radial_impulse e, u32 B, const uint8_t* kind, const nb_transform* xf,
		const nb_body_properties* props, nb_body_momentum* momentum, uint8_t* idle) {
	for (u32 i = 1 + blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
		const float4 p = reinterpret_cast<const float4*>(xf + i)[0];
		const float dx = p.x - e.center[0], dy = p.y - e.center[1], dz = p.z - e.center[2];
		const float dist = sqrtf((dx*dx + dy*dy) + dz*dz);
		if (!(dist < e.radius) || kin_is(kind, i)) continue;
		idle[i] = 0;
		if (dist > 0.0f) {
			const float k = (e.impulse * (1.0f - dist / e.radius)) / dist;
			const float m = props[i].mass_inverse;
			float4* row = reinterpret_cast<float4*>(momentum + i);
			float4 v = row[0];
			v.x += m * (dx * k); v.y += m * (dy * k); v.z += m * (dz * k);
			row[0] = v;
		}
	}
}

extern "C" {

int nb_apply_body_impulses(nb_context* ctx, const nb_body_impulse* h, uint32_t n, void* stream) {
	NB_RANGE("nb_apply_body_impulses");
	if (!n) return NB_OK;
	if (!h) { ctx->error = "null body impulse list"; return NB_ERR_ARGUMENT; }
	for (u32 i = 0; i < n; ++i) if (int r = check_body(ctx, "body impulse", i, h[i].body, false)) return r;   // a body may be listed again
	cudaStream_t st = (cudaStream_t)stream;
	JOIN_UPLOADS();   // ordered like nb_upload_momentum, after a pending nb_upload_bodies side copy
	ALLOC(ctx->imp_n, 1); ALLOC(ctx->imp_sb.hist, 256 * (size_t)ctx->sms); ALLOC(ctx->imp_sb.bar, 2);
	GROW(ctx->imp_rows, n, st);
	for (int i = 0; i < 2; ++i) { GROW(ctx->imp_keys[i], n, st); ctx->imp_sb.keys[i] = ctx->imp_keys[i].p; }
	CK(put_staged(ctx, ctx->imp_rows.p, h, sizeof(nb_body_impulse) * (size_t)n, st));
	const u32 ib = bits_for(n), bb = bits_for(ctx->B);
	const Launch L = mk_launch(ctx, st);
	launch_grid(L, k_impulse_keys, GRID(n), ctx->imp_rows.p, n, ib, ctx->imp_sb.keys[0], ctx->imp_n);
	const int cur = nb_radix_sort(L, ctx->imp_sb, ctx->imp_n, 0, (int)(ib + bb), false, 0);
	launch_grid(L, k_body_impulses, GRID(n), ctx->imp_rows.p, ctx->imp_sb.keys[cur], n, ib, ctx->xf, ctx->props, ctx->mom, ctx->idle);
	CK(cudaGetLastError());
	return NB_OK;
}

int nb_apply_radial_impulse(nb_context* ctx, const nb_radial_impulse* e, void* stream) {
	NB_RANGE("nb_apply_radial_impulse");
	if (!e) { ctx->error = "null radial impulse"; return NB_ERR_ARGUMENT; }
	if (!(e->radius > 0.0f) || !std::isfinite(e->radius)) { ctx->error = "radial impulse radius must be finite and above 0"; return NB_ERR_ARGUMENT; }
	JOIN_UPLOADS();
	if (ctx->B > 1) {
		launch_grid(mk_launch(ctx, stream), k_radial_impulse, GRID(ctx->B), *e, ctx->B, kin_table(ctx), ctx->xf, ctx->props, ctx->mom, ctx->idle);
	}
	CK(cudaGetLastError());
	return NB_OK;
}

}  // extern "C"
