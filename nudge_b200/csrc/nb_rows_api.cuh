// nudge_b200 — user constraint rows on the device (SURVEY.md §8 f1).
//
// The reference has no joints; it marks the three places where an application adds its own (example/main.cpp:285 "Custom constraints
// should be added as body connections", :288 "Custom contacts can be added here", :316 "Custom constraint impulses should be applied
// here", i.e. after every apply_impulses sweep).  With the state resident in HBM the application cannot run that code on the host
// between two sweeps without a round trip per sweep, so the hook becomes data: an array of generic velocity-constraint ROWS
// (one scalar constraint each: Jacobian, bias, impulse bounds, accumulated impulse) that the library applies, in the caller's
// order, right after every contact sweep — sequential impulses exactly as a host loop at example/main.cpp:316 would do them:
//
//     eff    = 1 / (J M^-1 J^T + softness)              M^-1 from BodyProperties, rotated like nudge.cpp:4182-4199
//     delta  = -eff * (J v + bias + softness * impulse)
//     impulse' = clamp(impulse + delta, lo, hi);  v += M^-1 J^T (impulse' - impulse)
//
// Order: rows run in upload order wherever two rows share a body (the host assigns every row the level 1 + max(level of the
// previous row on either body); rows of one level touch disjoint bodies and run in parallel, levels run one after the other), so the
// result equals the sequential loop.  Islands: connect the bodies of a joint with nb_upload_connections (example/main.cpp:285).
// Included at the end of nb_api.cu.
#pragma once
#include <map>

// The two bodies of a row as the row update holds them: a kinematic side (kind non-null) is like body 0, infinite mass, its velocity read and
// never written.  k_user_rows loads and stores them around one row, k_joint_solve (nb_joint_api.cuh) around all rows of a joint.
struct RowBodies {
	bool da, db;   // dynamic sides
	float ma, mb; float4 Ad, Ao, Bd, Bo;   // inverse masses; world inverse inertia (xx,yy,zz,-) (xy,xz,yz,-)
	float4 al, aw, bl, bw;   // momentum rows
	float4* pa; float4* pb;
};
NB_DEV RowBodies row_bodies_load(u32 a, u32 b, nb_body_momentum* momentum, const nb_body_properties* props, const float4* inertia, const uint8_t* kind) {
	RowBodies s;
	s.da = solver_body(kind, a) != 0; s.db = solver_body(kind, b) != 0;
	s.ma = s.da ? props[a].mass_inverse : 0.0f; s.mb = s.db ? props[b].mass_inverse : 0.0f;
	s.Ad = inertia[2*a]; s.Ao = inertia[2*a + 1]; s.Bd = inertia[2*b]; s.Bo = inertia[2*b + 1];
	if (!s.da) { s.Ad = make_float4(0, 0, 0, 0); s.Ao = s.Ad; }
	if (!s.db) { s.Bd = make_float4(0, 0, 0, 0); s.Bo = s.Bd; }
	s.pa = reinterpret_cast<float4*>(momentum + a); s.pb = reinterpret_cast<float4*>(momentum + b);
	s.al = s.pa[0]; s.aw = s.pa[1]; s.bl = s.pb[0]; s.bw = s.pb[1];
	return s;
}
NB_DEV void row_bodies_store(const RowBodies& s) {
	if (s.da) { s.pa[0] = s.al; s.pa[1] = s.aw; }
	if (s.db) { s.pb[0] = s.bl; s.pb[1] = s.bw; }
}
// One row on the bodies in `s`: the warm start (the accumulated impulse applied as it is) or one sequential-impulse update.  Returns the
// row's accumulated impulse afterwards.
NB_DEV float row_apply(const nb_constraint_row& r, RowBodies& s, int warm) {
	const float4 Ad = s.Ad, Ao = s.Ao, Bd = s.Bd, Bo = s.Bo;
	const float ma = s.ma, mb = s.mb;
	float4& al = s.al; float4& aw = s.aw; float4& bl = s.bl; float4& bw = s.bw;
	// I^-1 J_ang
	const float iax = Ad.x*r.ang_a[0] + Ao.x*r.ang_a[1] + Ao.y*r.ang_a[2], iay = Ao.x*r.ang_a[0] + Ad.y*r.ang_a[1] + Ao.z*r.ang_a[2], iaz = Ao.y*r.ang_a[0] + Ao.z*r.ang_a[1] + Ad.z*r.ang_a[2];
	const float ibx = Bd.x*r.ang_b[0] + Bo.x*r.ang_b[1] + Bo.y*r.ang_b[2], iby = Bo.x*r.ang_b[0] + Bd.y*r.ang_b[1] + Bo.z*r.ang_b[2], ibz = Bo.y*r.ang_b[0] + Bo.z*r.ang_b[1] + Bd.z*r.ang_b[2];
	float delta, next = r.impulse;
	if (warm) delta = r.impulse;
	else {
		const float k = ma * (r.lin_a[0]*r.lin_a[0] + r.lin_a[1]*r.lin_a[1] + r.lin_a[2]*r.lin_a[2]) + (r.ang_a[0]*iax + r.ang_a[1]*iay + r.ang_a[2]*iaz)
					  + mb * (r.lin_b[0]*r.lin_b[0] + r.lin_b[1]*r.lin_b[1] + r.lin_b[2]*r.lin_b[2]) + (r.ang_b[0]*ibx + r.ang_b[1]*iby + r.ang_b[2]*ibz) + r.softness;
		const float jv = r.lin_a[0]*al.x + r.lin_a[1]*al.y + r.lin_a[2]*al.z + r.ang_a[0]*aw.x + r.ang_a[1]*aw.y + r.ang_a[2]*aw.z
					   + r.lin_b[0]*bl.x + r.lin_b[1]*bl.y + r.lin_b[2]*bl.z + r.ang_b[0]*bw.x + r.ang_b[1]*bw.y + r.ang_b[2]*bw.z;
		const float eff = k > 0.0f ? 1.0f / k : 0.0f;
		next = r.impulse - eff * (jv + r.bias + r.softness * r.impulse);
		next = fminf(fmaxf(next, r.lo), r.hi);
		delta = next - r.impulse;
	}
	if (s.da) { al.x += ma * r.lin_a[0] * delta; al.y += ma * r.lin_a[1] * delta; al.z += ma * r.lin_a[2] * delta; aw.x += iax * delta; aw.y += iay * delta; aw.z += iaz * delta; }
	if (s.db) { bl.x += mb * r.lin_b[0] * delta; bl.y += mb * r.lin_b[1] * delta; bl.z += mb * r.lin_b[2] * delta; bw.x += ibx * delta; bw.y += iby * delta; bw.z += ibz * delta; }
	return next;
}

__global__ void __launch_bounds__(NB_BLOCK) k_user_rows(nb_constraint_row* rows, u32 begin, u32 end, nb_body_momentum* momentum, const nb_body_properties* props, const float4* inertia,
		const uint8_t* kind, int warm) {
	for (u32 i = begin + blockIdx.x * blockDim.x + threadIdx.x; i < end; i += gridDim.x * blockDim.x) {
		const nb_constraint_row r = rows[i];
		RowBodies s = row_bodies_load(r.a, r.b, momentum, props, inertia, kind);
		const float next = row_apply(r, s, warm);
		if (!warm) rows[i].impulse = next;
		row_bodies_store(s);
	}
}

static int launch_user_rows(nb_context* ctx, int warm, cudaStream_t st) {
	const Launch L = mk_launch(ctx, st);
	const RowLevels& us = ctx->urow_set;
	for (u32 l = 0; l < us.levels; ++l) {
		const u32 b = us.level_off[l], e = us.level_off[l + 1];
		if (e > b) launch_grid(L, k_user_rows, GRID(e - b), ctx->urows.p, b, e, ctx->mom, ctx->props, ctx->inertia, kin_table(ctx), warm);
	}
	CK(cudaGetLastError());
	return NB_OK;
}

// Levels the entries (a, b) in upload order into `out`: an entry's level is 1 + the highest level of an earlier entry on either of its bodies
// (body 0 is shared freely).  More than 4096 levels are refused with "<what> form a dependency chain ...", and `out` is left as it was.
static int level_rows(nb_context* ctx, std::vector<nb_body_pair> ab, RowLevels& out, const char* what) {
	RowLevels s;
	s.n = (u32)ab.size();
	std::vector<u32> level(s.n);
	std::map<u32, u32> last;   // body -> level of the last entry that touched it
	for (u32 i = 0; i < s.n; ++i) {
		const u32 a = ab[i].a, b = ab[i].b;
		u32 l = 0;
		if (a) { auto it = last.find(a); if (it != last.end()) l = std::max(l, it->second + 1); }
		if (b) { auto it = last.find(b); if (it != last.end()) l = std::max(l, it->second + 1); }
		level[i] = l; if (a) last[a] = l; if (b) last[b] = l;
		s.levels = std::max(s.levels, l + 1);
	}
	if (s.levels > 4096) { ctx->error = std::string(what) + " form a dependency chain longer than 4096 levels: reorder them (e.g. red-black along a chain)"; return NB_ERR_CAPACITY; }
	s.level_off.assign(s.n ? s.levels + 1 : 0, 0);
	for (u32 i = 0; i < s.n; ++i) ++s.level_off[level[i] + 1];
	for (u32 l = 0; l < s.levels; ++l) s.level_off[l + 1] += s.level_off[l];
	std::vector<u32> cursor(s.level_off);
	s.order.resize(s.n);
	for (u32 i = 0; i < s.n; ++i) s.order[i] = cursor[level[i]]++;
	s.ab = std::move(ab);
	out = std::move(s);
	return NB_OK;
}

extern "C" {

// Replaces the set of user rows (host pointer; n = 0 removes them).  Rows stay in effect, with their accumulated impulses carried
// from step to step (warm start), until the next upload.  Synchronises the stream.
int nb_upload_constraint_rows(nb_context* ctx, const nb_constraint_row* rows, uint32_t n, void* stream) {
	cudaStream_t st = (cudaStream_t)stream;
	CK(cudaStreamSynchronize(st));
	if (n > ctx->urows.cap) GROW(ctx->urows, (size_t)n + n / 2 + 64, st);   // with headroom for a set that grows a little
	ctx->urow_set = RowLevels(); ++ctx->graph_epoch;   // a refused set leaves none
	if (!n) return NB_OK;
	std::vector<nb_body_pair> ab(n);
	for (u32 i = 0; i < n; ++i) {
		const u32 a = rows[i].a, b = rows[i].b;
		if (a >= ctx->cfg.max_bodies || b >= ctx->cfg.max_bodies) { ctx->error = "constraint row references a body beyond max_bodies"; return NB_ERR_ARGUMENT; }
		// k_user_rows gives each side its own read-modify-write of the momentum row, and the effective mass has no cross terms
		if (a && a == b) { ctx->error = "constraint row names the same body as a and b: put the whole Jacobian on a and set b = 0"; return NB_ERR_ARGUMENT; }
		ab[i].a = a; ab[i].b = b;
	}
	RowLevels set;
	if (int r = level_rows(ctx, std::move(ab), set, "constraint rows")) return r;
	std::vector<nb_constraint_row> sorted(n);
	for (u32 i = 0; i < n; ++i) sorted[set.order[i]] = rows[i];
	CK(cudaMemcpy(ctx->urows.p, sorted.data(), sizeof(nb_constraint_row) * n, cudaMemcpyHostToDevice));
	ctx->urow_set = std::move(set);
	return NB_OK;
}

// Copies the rows back in the caller's order (the accumulated impulses are the result).  Synchronises.
int nb_download_constraint_rows(nb_context* ctx, nb_constraint_row* rows, uint32_t n, void* stream) {
	if (n != ctx->urow_set.n) { ctx->error = "row count differs from the uploaded set"; return NB_ERR_ARGUMENT; }
	if (!n) return NB_OK;
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	std::vector<nb_constraint_row> sorted(n);
	CK(cudaMemcpy(sorted.data(), ctx->urows.p, sizeof(nb_constraint_row) * n, cudaMemcpyDeviceToHost));
	for (u32 i = 0; i < n; ++i) rows[i] = sorted[ctx->urow_set.order[i]];
	return NB_OK;
}

}  // extern "C"
