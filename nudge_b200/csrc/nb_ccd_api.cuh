// nudge_b200 — continuous collision for fast bodies (nb_upload_ccd_bodies, nb_download_ccd_bodies; DESIGN.md section 8.18).
//
// The step is discrete: k_advance moves every awake body by v * dt without looking at what lies between its two poses.  A listed body casts
// a sphere along that translation inside nb_advance (k_ccd, nb_query_api.cuh) against the step's own front end, which nb_collide built and
// nothing after it rewrites, and k_advance<true> scales the translation by the first time of impact.  The set lives on the host (ascending by
// body) with a device copy of its rows; the per-body factor table ccd_t holds 1 outside the set, so k_advance<true> needs no lookup.  The
// graph reads the rows through an unchanged pointer, so new radii, thresholds or filters for the same bodies keep nb_step's graph; another
// body list re-records it (graph_epoch).  Included at the end of nb_api.cu.
#pragma once
#include <cmath>

// The factor of every body of capacity to 1 and the hits of the set's n entries to (1, no hit): the state of a set no advance has used.
__global__ void __launch_bounds__(NB_BLOCK) k_ccd_reset(float* ccd_t, u32 nbodies, uint2* hits, u32 n) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < max(nbodies, n); i += gridDim.x * blockDim.x) {
		if (i < nbodies) ccd_t[i] = 1.0f;
		if (i < n) hits[i] = make_uint2(asu(1.0f), NB_RAY_NO_HIT);
	}
}

// The entry checks of nb_upload_ccd_bodies that do not depend on the context (also applied to the rows of a loaded state file); null if the
// entry is valid, else what is wrong with it.
static const char* ccd_body_problem(const nb_ccd_body& e) {
	if (!std::isfinite(e.radius) || e.radius < 0.0f) return "a radius that is not finite or is below 0";
	if (std::isnan(e.motion_threshold) || e.motion_threshold < 0.0f) return "a NaN or negative motion threshold";
	return nullptr;
}

// Installs `set` (checked, ascending by body, possibly empty) in place of the context's.  The same body list keeps the graph and the factor
// table (k_ccd rewrites every entry's factor each advance); another list resets the table and re-records the graph.
static int set_ccd(nb_context* ctx, std::vector<nb_ccd_body> set, cudaStream_t st) {
	if (set.empty()) { drop_ccd(ctx); return NB_OK; }
	const u32 n = (u32)set.size();
	bool same = n == ctx->ccd.size();
	for (u32 i = 0; same && i < n; ++i) same = set[i].body == ctx->ccd[i].body;
	if (same && !memcmp(set.data(), ctx->ccd.data(), sizeof(nb_ccd_body) * (size_t)n)) return NB_OK;   // nothing changes
	ALLOC(ctx->ccd_t, ctx->cfg.max_bodies);   // the factor table, on first use
	GROW(ctx->ccd_rows, n, st); GROW(ctx->ccd_hits, n, st);
	CK(put_staged(ctx, ctx->ccd_rows.p, set.data(), sizeof(nb_ccd_body) * (size_t)n, st));
	if (!same) {
		launch_grid(mk_launch(ctx, st), k_ccd_reset, GRID(std::max(ctx->cfg.max_bodies, n)), ctx->ccd_t, ctx->cfg.max_bodies, ctx->ccd_hits.p, n);
		CK(cudaGetLastError());
		++ctx->graph_epoch;   // nb_step's graph re-records with k_ccd over the new rows
	}
	ctx->ccd.swap(set);
	return NB_OK;
}

// nb_advance's casts: k_ccd over the set against the step's front end (nb_collide's grid, world transforms and filter words).
static int launch_ccd(nb_context* ctx, const Launch& L, float time_step) {
	const FrontEnd& f = ctx->front;
	const QueryScene S = { ctx->B ? ctx->nboxes + ctx->nspheres : 0, ctx->nboxes, f.world_xf, f.aabb_max, f.col_body, f.col_tag, ctx->box_data, ctx->sph_data,
						   ctx->has_sensor ? ctx->sensor : nullptr, f.order, f.smallf, f.table_keys, f.table_vals, f.table_mask, f.large_list };
	const u32 n = (u32)ctx->ccd.size();
	launch_grid(L, k_ccd, GRID((u64)n * 32), n, (const nb_ccd_body*)ctx->ccd_rows.p, (const nb_transform*)ctx->xf, (const nb_body_momentum*)ctx->mom,
		(const u32*)ctx->parent, (const u32*)ctx->active, kin_table(ctx), time_step, S, (const u64*)ctx->conn_keys, ctx->conn_probe, ctx->counts,
		ctx->ccd_t, ctx->ccd_hits.p);
	CK(cudaGetLastError());
	return NB_OK;
}

extern "C" {

int nb_upload_ccd_bodies(nb_context* ctx, const nb_ccd_body* h, uint32_t n, void* stream) {
	NB_RANGE("nb_upload_ccd_bodies");
	if (ctx->sharded) { ctx->error = "nb_upload_ccd_bodies: not supported on a context of nb_shard_create"; return NB_ERR_ARGUMENT; }
	if (n && !h) { ctx->error = "null ccd body list"; return NB_ERR_ARGUMENT; }
	for (u32 i = 0; i < n; ++i) {
		if (int r = check_body(ctx, "ccd body", i, h[i].body, false)) return r;
		if (const char* p = ccd_body_problem(h[i])) { ctx->error = "ccd body " + std::to_string(i) + ": " + p; return NB_ERR_ARGUMENT; }
	}
	if (int r = bodies_distinct(ctx, "ccd body", n, [&](u32 i) { return h[i].body; })) return r;
	std::vector<nb_ccd_body> set(h, h + n);
	std::sort(set.begin(), set.end(), [](const nb_ccd_body& a, const nb_ccd_body& b) { return a.body < b.body; });
	return set_ccd(ctx, std::move(set), (cudaStream_t)stream);
}

int nb_download_ccd_bodies(nb_context* ctx, nb_ccd_body* h, uint32_t capacity, uint32_t* count, void* stream) {
	(void)stream;
	const u32 n = (u32)ctx->ccd.size();
	if (count) *count = n;
	if (capacity < n) { ctx->error = "host ccd body array too small: " + std::to_string(n) + " entries"; return NB_ERR_CAPACITY; }
	if (n && !h) { ctx->error = "null ccd body array"; return NB_ERR_ARGUMENT; }
	if (n) memcpy(h, ctx->ccd.data(), sizeof(nb_ccd_body) * (size_t)n);
	return NB_OK;
}

}  // extern "C"
