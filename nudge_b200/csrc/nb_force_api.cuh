// nudge_b200 — per-body forces (nb_set_body_forces, nb_clear_body_forces, nb_download_body_forces; DESIGN.md section 8.11).
//
// The reference's application applies one gravity and one damping rate to every active body in its user loop (example/main.cpp:291-305,
// k_gravity_damping).  A game also needs a gravity scale, extra damping and constant forces and torques per body, inside the step.  They
// live in a device table of nb_body_force entries, one per body, that k_body_forces (nb_solver.cuh) reads in place of k_gravity_damping
// while the table exists.  The graph reads the table through an unchanged pointer, so editing entries keeps nb_step's graph; creating and
// removing the table re-records it (graph_epoch).
//
// Stored rows are canonical: body = the row index, reserved = 0.  Rows at and beyond the body count are never read: nb_add_bodies writes
// default rows for the bodies it appends, and nb_remove_bodies gathers the kept rows (k_spawn_bodies).  Included at the end of nb_api.cu.
#pragma once
#include <cmath>

static nb_body_force default_body_force(u32 body) {
	nb_body_force e;
	memset(&e, 0, sizeof(e));
	e.body = body; e.gravity_scale = 1.0f;
	return e;
}

// The entry checks of nb_set_body_forces that do not depend on the context (also applied to the rows of a loaded state file); null if the
// entry is valid, else what is wrong with it.
static const char* body_force_problem(const nb_body_force& e) {
	if (e.flags & ~(u32)NB_BODY_FORCE_LOCAL) return "unknown flag bits";
	const float f[] = { e.gravity_scale, e.linear_damping, e.angular_damping, e.force[0], e.force[1], e.force[2], e.torque[0], e.torque[1], e.torque[2] };
	for (float x : f) if (!std::isfinite(x)) return "a field that is not finite";
	if (e.linear_damping < 0.0f || e.angular_damping < 0.0f) return "a negative damping";
	return nullptr;
}

__global__ void __launch_bounds__(NB_BLOCK) k_body_force_defaults(nb_body_force* table, u32 B) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
		float4* e = reinterpret_cast<float4*>(table + i);
		e[0] = make_float4(asf(i), 0.0f, 1.0f, 0.0f); e[1] = make_float4(0.0f, 0.0f, 0.0f, 0.0f); e[2] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
	}
}

// Each listed entry into its body's row, and the body woken.
__global__ void __launch_bounds__(NB_BLOCK) k_body_force_scatter(const nb_body_force* rows, u32 n, nb_body_force* table, uint8_t* idle) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const float4* r = reinterpret_cast<const float4*>(rows + i);
		const float4 a = r[0], b = r[1], c = r[2];
		const u32 body = asu(a.x);
		float4* e = reinterpret_cast<float4*>(table + body);
		e[0] = a; e[1] = b; e[2] = c;
		idle[body] = 0;
	}
}

// Stored rows are canonical: the staged rows' reserved words are cleared before their copy.
static void clear_reserved(unsigned char* rows, size_t bytes) {
	for (size_t i = 0; i < bytes / sizeof(nb_body_force); ++i) reinterpret_cast<nb_body_force*>(rows)[i].reserved = 0;
}

// Creates the table (every body 0 .. B-1 with the default entry) unless it exists.
static int ensure_body_forces(nb_context* ctx, cudaStream_t st) {
	if (ctx->has_frc) return NB_OK;
	ALLOC(ctx->frc, ctx->cfg.max_bodies); ALLOC(ctx->frc_spare, ctx->cfg.max_bodies);   // the table and its gather buffer, on first use
	if (ctx->B) launch_grid(mk_launch(ctx, st), k_body_force_defaults, GRID(ctx->B), ctx->frc, ctx->B);
	CK(cudaGetLastError());
	ctx->has_frc = true;
	++ctx->graph_epoch;   // nb_step's graph re-records with k_body_forces
	return NB_OK;
}

extern "C" {

int nb_set_body_forces(nb_context* ctx, const nb_body_force* h, uint32_t n, void* stream) {
	NB_RANGE("nb_set_body_forces");
	if (n && !h) { ctx->error = "null body force list"; return NB_ERR_ARGUMENT; }
	for (u32 i = 0; i < n; ++i) {
		if (int r = check_body(ctx, "body force", i, h[i].body, false)) return r;
		if (const char* p = body_force_problem(h[i])) { ctx->error = "body force " + std::to_string(i) + ": " + p; return NB_ERR_ARGUMENT; }
	}
	if (int r = bodies_distinct(ctx, "body force", n, [&](u32 i) { return h[i].body; })) return r;
	cudaStream_t st = (cudaStream_t)stream;
	JOIN_UPLOADS();   // ordered like nb_upload_momentum, after a pending nb_upload_bodies side copy (the scatter writes idle counters)
	{ int r = ensure_body_forces(ctx, st); if (r) return r; }
	if (!n) return NB_OK;
	GROW(ctx->frc_rows, n, st);
	CK(put_staged(ctx, ctx->frc_rows.p, h, sizeof(nb_body_force) * (size_t)n, st, clear_reserved));
	launch_grid(mk_launch(ctx, st), k_body_force_scatter, GRID(n), ctx->frc_rows.p, n, ctx->frc, ctx->idle);
	CK(cudaGetLastError());
	return NB_OK;
}

int nb_clear_body_forces(nb_context* ctx, void* stream) {
	(void)stream;
	drop_body_forces(ctx);
	return NB_OK;
}

int nb_download_body_forces(nb_context* ctx, nb_body_force* h, uint32_t capacity, uint32_t* count, void* stream) {
	NB_RANGE("nb_download_body_forces");
	if (count) *count = ctx->B;
	if (capacity < ctx->B) { ctx->error = "host body force array too small: " + std::to_string(ctx->B) + " bodies"; return NB_ERR_CAPACITY; }
	if (ctx->B && !h) { ctx->error = "null body force array"; return NB_ERR_ARGUMENT; }
	if (ctx->has_frc) D2H(h, ctx->frc, ctx->B, nb_body_force);
	else for (u32 i = 0; i < ctx->B; ++i) h[i] = default_body_force(i);
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	return NB_OK;
}

}  // extern "C"
