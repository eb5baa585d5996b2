// nudge_b200 — device-resident joints (nb_upload_joints, nb_download_joints; DESIGN.md section 8.13).
//
// A joint produces user constraint rows (nb_rows_api.cuh): k_joint_rows rebuilds them once per step from the bodies' transforms, by the
// arithmetic include/nudge_b200.h states, and k_joint_solve applies them with the row update of k_user_rows (row_apply), one thread per joint
// and one launch per joint level (level_rows over the joints' bodies).  The device table holds the joints by level, upload order within one;
// each entry's type word also carries the offset of the joint's first row (type | offset << 2).  The parameters live in the table, the
// accumulated impulses in the rows, which k_joint_rows rewrites around them.  Included at the end of nb_api.cu.
#pragma once

__host__ __device__ __forceinline__ u32 joint_row_count(u32 type) { return type == NB_JOINT_BALL ? 3u : type == NB_JOINT_HINGE ? 5u : type == NB_JOINT_FIXED ? 6u : 1u; }

NB_DEV f3 neg3(f3 a) { return mk3(-a.x, -a.y, -a.z); }
// Writes one row around its accumulated impulse.
NB_DEV void joint_row_put(nb_constraint_row* row, const nb_joint& j, f3 lin_a, f3 ang_a, f3 lin_b, f3 ang_b, float bias) {
	nb_constraint_row r;
	r.a = j.a; r.b = j.b;
	r.lin_a[0] = lin_a.x; r.lin_a[1] = lin_a.y; r.lin_a[2] = lin_a.z; r.ang_a[0] = ang_a.x; r.ang_a[1] = ang_a.y; r.ang_a[2] = ang_a.z;
	r.lin_b[0] = lin_b.x; r.lin_b[1] = lin_b.y; r.lin_b[2] = lin_b.z; r.ang_b[0] = ang_b.x; r.ang_b[1] = ang_b.y; r.ang_b[2] = ang_b.z;
	r.bias = bias; r.lo = -INFINITY; r.hi = INFINITY; r.impulse = row->impulse; r.softness = j.softness; r.reserved = 0.0f;
	*row = r;
}

// One thread per joint: the joint's rows from the two transforms (include/nudge_b200.h, Joints).
__global__ void __launch_bounds__(NB_BLOCK) k_joint_rows(const nb_joint* joints, u32 n, const nb_transform* xf, float dt, nb_constraint_row* rows) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const nb_joint j = joints[i];
		const u32 type = j.type & 3u;
		nb_constraint_row* row = rows + (j.type >> 2);
		const float k = j.beta / dt;
		const xform ta = ld_xform(xf, j.a);
		const quat qa = mkq(ta.q);
		const f3 zero = mk3(0.0f, 0.0f, 0.0f);
		quat qb = { zero, 1.0f };
		const f3 ra = qrot(qa, ld3(j.anchor_a)), wa = add3(mk3(ta.p.x, ta.p.y, ta.p.z), ra);
		f3 rb = zero, wb = ld3(j.anchor_b);
		if (j.b) {
			const xform tb = ld_xform(xf, j.b);
			qb = mkq(tb.q);
			rb = qrot(qb, ld3(j.anchor_b)); wb = add3(mk3(tb.p.x, tb.p.y, tb.p.z), rb);
		}
		const f3 err = sub3(wa, wb);
		if (type == NB_JOINT_DISTANCE) {
			const float dist = sqrtf(dot3(err, err));
			const f3 dir = dist > 0.0f ? mul3(err, 1.0f / dist) : mk3(0.0f, 1.0f, 0.0f);
			joint_row_put(row, j, dir, cross3(ra, dir), neg3(dir), neg3(cross3(rb, dir)), k * (dist - j.length));
			continue;
		}
		joint_row_put(row + 0, j, mk3(1.0f, 0.0f, 0.0f), mk3(0.0f, ra.z, -ra.y), mk3(-1.0f, 0.0f, 0.0f), mk3(0.0f, -rb.z, rb.y), k * err.x);
		joint_row_put(row + 1, j, mk3(0.0f, 1.0f, 0.0f), mk3(-ra.z, 0.0f, ra.x), mk3(0.0f, -1.0f, 0.0f), mk3(rb.z, 0.0f, -rb.x), k * err.y);
		joint_row_put(row + 2, j, mk3(0.0f, 0.0f, 1.0f), mk3(ra.y, -ra.x, 0.0f), mk3(0.0f, 0.0f, -1.0f), mk3(-rb.y, rb.x, 0.0f), k * err.z);
		if (type == NB_JOINT_HINGE) {
			const f3 u = qrot(qa, ld3(j.axis_a)), w = j.b ? qrot(qb, ld3(j.axis_b)) : ld3(j.axis_b), c = cross3(u, w);
			f3 t1 = fabsf(u.x) < 0.57735f ? mk3(0.0f, u.z, -u.y) : mk3(-u.z, 0.0f, u.x);
			t1 = mul3(t1, 1.0f / sqrtf(dot3(t1, t1)));
			const f3 t2 = cross3(u, t1);
			joint_row_put(row + 3, j, zero, t1, zero, neg3(t1), -(k * dot3(c, t1)));
			joint_row_put(row + 4, j, zero, t2, zero, neg3(t2), -(k * dot3(c, t2)));
		}
		else if (type == NB_JOINT_FIXED) {
			const quat rel = { ld3(j.rel_rotation), j.rel_rotation[3] };
			quat d = qmul(qa, rel);
			if (j.b) { const quat cb = { neg3(qb.v), qb.s }; d = qmul(d, cb); }
			if (d.s < 0.0f) d.v = neg3(d.v);
			joint_row_put(row + 3, j, zero, mk3(1.0f, 0.0f, 0.0f), zero, mk3(-1.0f, 0.0f, 0.0f), k * (2.0f * d.v.x));
			joint_row_put(row + 4, j, zero, mk3(0.0f, 1.0f, 0.0f), zero, mk3(0.0f, -1.0f, 0.0f), k * (2.0f * d.v.y));
			joint_row_put(row + 5, j, zero, mk3(0.0f, 0.0f, 1.0f), zero, mk3(0.0f, 0.0f, -1.0f), k * (2.0f * d.v.z));
		}
	}
}

// One thread per joint of the level [begin, end): the joint's rows one after the other, the two bodies' momentum kept in registers across them.
__global__ void __launch_bounds__(NB_BLOCK) k_joint_solve(const nb_joint* joints, u32 begin, u32 end, nb_constraint_row* rows, nb_body_momentum* momentum,
		const nb_body_properties* props, const float4* inertia, const uint8_t* kind, int warm) {
	for (u32 i = begin + blockIdx.x * blockDim.x + threadIdx.x; i < end; i += gridDim.x * blockDim.x) {
		const u32 packed = joints[i].type, first = packed >> 2, count = joint_row_count(packed & 3u);
		RowBodies s = row_bodies_load(joints[i].a, joints[i].b, momentum, props, inertia, kind);
		for (u32 r = first; r < first + count; ++r) {
			const float next = row_apply(rows[r], s, warm);
			if (!warm) rows[r].impulse = next;
		}
		row_bodies_store(s);
	}
}

// The step's joint launches: with `dt` the row build and the warm start (nb_setup_contact_constraints), without it one pass after a sweep.
static int launch_joints(nb_context* ctx, const float* dt, cudaStream_t st) {
	const Launch L = mk_launch(ctx, st);
	const JointSet& js = ctx->jset;
	if (dt) launch_grid(L, k_joint_rows, GRID(js.n), ctx->joints.p, js.n, ctx->xf, *dt, ctx->jrows.p);
	for (u32 l = 0; l < js.levels; ++l)
		launch_grid(L, k_joint_solve, GRID(js.level_off[l + 1] - js.level_off[l]), ctx->joints.p, js.level_off[l], js.level_off[l + 1], ctx->jrows.p, ctx->mom, ctx->props,
			ctx->inertia, kin_table(ctx), dt ? 1 : 0);
	CK(cudaGetLastError());
	return NB_OK;
}

static void drop_joints(nb_context* ctx) { if (ctx->jset.n) { ctx->jset = JointSet(); ++ctx->graph_epoch; } }

// What nb_upload_joints refuses in a joint of a context with B bodies (also applied to a loaded state file); null if the joint is valid.
static const char* joint_problem(const nb_joint& j, u32 B) {
	if (j.type > NB_JOINT_DISTANCE) return "unknown type";
	if (j.a == 0) return "a is the static world (put the world on b)";
	if (j.a == j.b) return "a and b are the same body";
	if (j.a >= B || j.b >= B) return "a body at or beyond the body count";
	const float* f = j.anchor_a;   // the struct is floats from here to its end
	for (size_t i = 0; i < (sizeof(nb_joint) - offsetof(nb_joint, anchor_a)) / sizeof(float); ++i) if (!std::isfinite(f[i])) return "a field that is not finite";
	return nullptr;
}
static int check_joints(nb_context* ctx, const nb_joint* h, u32 n, u32 B) {
	if (n && !h) { ctx->error = "null joint list"; return NB_ERR_ARGUMENT; }
	for (u32 i = 0; i < n; ++i)
		if (const char* p = joint_problem(h[i], B)) { ctx->error = "joint " + std::to_string(i) + ": " + p; return NB_ERR_ARGUMENT; }
	return NB_OK;
}

// Installs n checked joints in place of the set: levels, the table by level with the row offsets, and the rows holding the impulses.
static int set_joints(nb_context* ctx, const nb_joint* h, u32 n, cudaStream_t st) {
	if (!n) { drop_joints(ctx); return NB_OK; }
	JointSet js;
	std::vector<nb_body_pair> ab(n);
	for (u32 i = 0; i < n; ++i) { ab[i].a = h[i].a; ab[i].b = h[i].b; js.structure.insert(js.structure.end(), { h[i].type, h[i].a, h[i].b }); }
	if (int r = level_rows(ctx, std::move(ab), js, "joints")) return r;
	std::vector<nb_joint> table(n);
	for (u32 i = 0; i < n; ++i) table[js.order[i]] = h[i];
	for (nb_joint& j : table) { const u32 type = j.type; j.type = type | js.nrows << 2; js.nrows += joint_row_count(type); }
	std::vector<nb_constraint_row> rows(js.nrows);
	memset(rows.data(), 0, sizeof(nb_constraint_row) * rows.size());
	for (const nb_joint& j : table) for (u32 k = 0; k < joint_row_count(j.type & 3u); ++k) rows[(j.type >> 2) + k].impulse = j.impulse[k];
	const void* before[2] = { ctx->joints.p, ctx->jrows.p };
	GROW(ctx->joints, n, st); GROW(ctx->jrows, js.nrows, st);
	CK(put_staged(ctx, ctx->joints.p, table.data(), sizeof(nb_joint) * (size_t)n, st));
	CK(put_staged(ctx, ctx->jrows.p, rows.data(), sizeof(nb_constraint_row) * rows.size(), st));
	// the levels are host values in nb_step's graph, the buffers its kernel arguments
	if (js.structure != ctx->jset.structure || before[0] != ctx->joints.p || before[1] != ctx->jrows.p) ++ctx->graph_epoch;
	ctx->jset = std::move(js);
	return NB_OK;
}

// The joints in upload order with their rows' current impulses.  Synchronises.
static int get_joints(nb_context* ctx, std::vector<nb_joint>& out, cudaStream_t st) {
	const JointSet& js = ctx->jset;
	std::vector<nb_joint> table(js.n);
	std::vector<nb_constraint_row> rows(js.nrows);
	out.resize(js.n);
	if (!js.n) return NB_OK;
	CK(cudaMemcpyAsync(table.data(), ctx->joints.p, sizeof(nb_joint) * (size_t)js.n, cudaMemcpyDeviceToHost, st));
	CK(cudaMemcpyAsync(rows.data(), ctx->jrows.p, sizeof(nb_constraint_row) * rows.size(), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	for (u32 i = 0; i < js.n; ++i) {
		nb_joint j = table[js.order[i]];
		const u32 first = j.type >> 2;
		j.type &= 3u;
		for (u32 k = 0; k < 6; ++k) j.impulse[k] = k < joint_row_count(j.type) ? rows[first + k].impulse : 0.0f;
		out[i] = j;
	}
	return NB_OK;
}

__global__ void __launch_bounds__(NB_BLOCK) k_joint_wake(const u32* bodies, u32 n, uint8_t* idle) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) idle[bodies[i]] = 0;
}

extern "C" {

int nb_upload_joints(nb_context* ctx, const nb_joint* h, uint32_t n, void* stream) {
	NB_RANGE("nb_upload_joints");
	if (int r = check_joints(ctx, h, n, ctx->B)) return r;
	return set_joints(ctx, h, n, (cudaStream_t)stream);
}

int nb_download_joints(nb_context* ctx, nb_joint* h, uint32_t capacity, uint32_t* count, void* stream) {
	NB_RANGE("nb_download_joints");
	const u32 n = ctx->jset.n;
	if (count) *count = n;
	if (capacity < n) { ctx->error = "host joint array too small: " + std::to_string(n) + " joints"; return NB_ERR_CAPACITY; }
	if (n && !h) { ctx->error = "null joint array"; return NB_ERR_ARGUMENT; }
	std::vector<nb_joint> joints;
	if (int r = get_joints(ctx, joints, (cudaStream_t)stream)) return r;
	std::copy(joints.begin(), joints.end(), h);
	return NB_OK;
}

}  // extern "C"
