// nudge_b200 — device-resident joints (nb_upload_joints, nb_download_joints; DESIGN.md section 8.13).
//
// A joint produces user constraint rows (nb_rows_api.cuh): k_joint_rows rebuilds them once per step from the bodies' transforms, by the
// arithmetic include/nudge_b200.h states, and k_joint_solve applies them with the row update of k_user_rows (row_apply), one thread per joint
// and one launch per joint level (level_rows over the joints' bodies).  The device table holds the joints by level, upload order within one;
// each entry's type word also carries the offset of the joint's first row (type | offset << 2).  The parameters live in the table, the
// accumulated impulses in the rows, which k_joint_rows rewrites around them.
// Drives (nb_upload_joint_drives; DESIGN.md section 8.17) and springs (nb_upload_joint_springs; DESIGN.md section 8.21) are sparse tables
// keyed by joint (KeyedTable): an entry per joint in table order and the entries' rows in a buffer of their own, which both kernels take as
// arguments (null without a set), so that the joints' own rows are the same with and without them.  A drive's rows are motor, lower, upper;
// the break test and the broken flag live in k_joint_rows.  Sliders (FIXED + SLIDE) and ragdoll swing-cone and twist limits (BALL + CONE /
// TWIST; DESIGN.md section 8.20) are drives too: a slider rewrites its joint's point rows, a cone takes the motor's slot and a twist limit
// the limit's.  A spring row is Catto's soft step on one joint coordinate; k_joint_solve applies a joint's own rows, then its spring rows,
// then its drive rows.  Included at the end of nb_api.cu.
#pragma once

__host__ __device__ __forceinline__ u32 joint_row_count(u32 type) { return type == NB_JOINT_BALL ? 3u : type == NB_JOINT_HINGE ? 5u : type == NB_JOINT_FIXED ? 6u : 1u; }
__host__ __device__ __forceinline__ u32 drive_row_count(u32 flags) {
	return (flags & (NB_JOINT_MOTOR | NB_JOINT_CONE) ? 1u : 0u) + (flags & (NB_JOINT_LIMIT | NB_JOINT_TWIST) ? 2u : 0u);
}
__host__ __device__ __forceinline__ u32 spring_row_count(u32 type) { return type == NB_JOINT_BALL ? 3u : 1u; }

NB_DEV f3 neg3(f3 a) { return mk3(-a.x, -a.y, -a.z); }
// Writes one row around its accumulated impulse, with the joint's softness or, for a spring row, its own.
NB_DEV void row_put(nb_constraint_row* row, const nb_joint& j, f3 lin_a, f3 ang_a, f3 lin_b, f3 ang_b, float bias, float lo, float hi, float softness) {
	nb_constraint_row r;
	r.a = j.a; r.b = j.b;
	r.lin_a[0] = lin_a.x; r.lin_a[1] = lin_a.y; r.lin_a[2] = lin_a.z; r.ang_a[0] = ang_a.x; r.ang_a[1] = ang_a.y; r.ang_a[2] = ang_a.z;
	r.lin_b[0] = lin_b.x; r.lin_b[1] = lin_b.y; r.lin_b[2] = lin_b.z; r.ang_b[0] = ang_b.x; r.ang_b[1] = ang_b.y; r.ang_b[2] = ang_b.z;
	r.bias = bias; r.lo = lo; r.hi = hi; r.impulse = row->impulse; r.softness = softness; r.reserved = 0.0f;
	*row = r;
}
NB_DEV void joint_row_put(nb_constraint_row* row, const nb_joint& j, f3 lin_a, f3 ang_a, f3 lin_b, f3 ang_b, float bias, float lo = -INFINITY, float hi = INFINITY) {
	row_put(row, j, lin_a, ang_a, lin_b, ang_b, bias, lo, hi, j.softness);
}
// A spring row on the coordinate C with the Jacobian (lin_a, ang_a, lin_b, ang_b): the implicit spring-damper of stiffness k and damping c
// over one step is the row with softness 1 / (dt * (c + dt * k)) and bias (k * C - c * target_velocity) / (c + dt * k).
NB_DEV void spring_row_put(nb_constraint_row* row, const nb_joint& j, f3 lin_a, f3 ang_a, f3 lin_b, f3 ang_b, float C, const JointSpring& sp, float dt) {
	const float den = sp.damping + dt * sp.stiffness, lim = sp.max_force * dt;
	row_put(row, j, lin_a, ang_a, lin_b, ang_b, (sp.stiffness * C - sp.damping * sp.target_velocity) / den, -lim, lim, 1.0f / (dt * den));
}
// A broken joint's row: everything zero but a and b.
NB_DEV void joint_row_zero(nb_constraint_row* row, const nb_joint& j) {
	nb_constraint_row r;
	memset(&r, 0, sizeof(r));
	r.a = j.a; r.b = j.b;
	*row = r;
}
// A limit row's bias: speculative while the coordinate is inside (C > 0), Baumgarte once past the bound.
NB_DEV float limit_bias(float C, float dt, float k) { return C > 0.0f ? C / dt : k * C; }
// An angle limit's C from (s, c) = (sin x, cos x) of the half difference x = (theta - stop) / 2, x in [-pi, pi]: 2 sin x while c >= 0, then
// +-(4 - 2 |sin x|) with the sign of x.  Continuous and increasing in x, and (2/pi) * min(|2x|, pi) <= |C| <= |2x|: unlike 2 sin x it does not
// fold back toward 0 past a half turn, where a wide range's far stop would otherwise cap the speed away from the near one.
NB_DEV float angle_limit_measure(float s, float c) { const float t = 2.0f * s; return c >= 0.0f ? t : s >= 0.0f ? 4.0f - t : -4.0f - t; }
// The lower and upper angle limit rows of HINGE LIMIT and TWIST on the hinge Jacobian about u, from the angle's half-angle pair (sh, ch).
NB_DEV void angle_limit_rows(nb_constraint_row* drow, const nb_joint& j, const JointDrive& d, f3 u, float sh, float ch, float dt, float k) {
	const f3 zero = mk3(0.0f, 0.0f, 0.0f), nu = neg3(u);
	joint_row_put(drow + 0, j, zero, nu, zero, u, limit_bias(angle_limit_measure(sh * d.cl - ch * d.sl, ch * d.cl + sh * d.sl), dt, k), 0.0f, INFINITY);
	joint_row_put(drow + 1, j, zero, u, zero, nu, limit_bias(angle_limit_measure(d.su * ch - d.cu * sh, d.cu * ch + d.su * sh), dt, k), 0.0f, INFINITY);
}

// The break test of a BREAKABLE joint on the impulses the previous step left in its rows (own rows at `row`, appended ones at `drow`).
// A distance joint's and a slider's appended rows are linear, every other joint's angular.
NB_DEV bool joint_breaks(const nb_constraint_row* row, const nb_constraint_row* drow, u32 type, u32 flags, const JointDrive& d, float dt) {
	float P = 0.0f, A = 0.0f;
	const bool linear = type == NB_JOINT_DISTANCE || (flags & NB_JOINT_SLIDE);
	for (u32 r = 0; r < joint_row_count(type); ++r) { const float x = row[r].impulse; if (type == NB_JOINT_DISTANCE || r < 3) P = P + x * x; else A = A + x * x; }
	for (u32 r = 0; r < drive_row_count(flags); ++r) { const float x = drow[r].impulse; if (linear) P = P + x * x; else A = A + x * x; }
	const float f = d.break_force * dt, t = d.break_torque * dt;
	return P > f * f || A > t * t;
}

// The two unit vectors HINGE builds perpendicular to its axis u.
NB_DEV void hinge_basis(f3 u, f3& t1, f3& t2) {
	t1 = fabsf(u.x) < 0.57735f ? mk3(0.0f, u.z, -u.y) : mk3(-u.z, 0.0f, u.x);
	t1 = mul3(t1, 1.0f / sqrtf(dot3(t1, t1)));
	t2 = cross3(u, t1);
}
// qmul(q_a, rel_rotation), times conj(q_b) when b != 0: the rotation HINGE LIMIT, FIXED and the swing-twist limits measure.
NB_DEV quat joint_rel(quat qa, const nb_joint& j, quat qb) {
	const quat rel = { ld3(j.rel_rotation), j.rel_rotation[3] };
	quat d = qmul(qa, rel);
	if (j.b) { const quat cb = { neg3(qb.v), qb.s }; d = qmul(d, cb); }
	return d;
}

// FIXED + SLIDE: the joint's point rows across the slide axis u (rows 0, 1) and along it (row 2, which applies nothing), and the drive's
// rows on the slide coordinate s = dot(wb - wa, u).  sa = ra - err runs from a's position to b's anchor.
NB_DEV void slider_rows(nb_constraint_row* row, nb_constraint_row* drow, const nb_joint& j, const JointDrive& d, u32 flags, f3 u, f3 ra, f3 rb,
		f3 wa, f3 wb, float dt, float k, float* position) {
	const f3 err = sub3(wa, wb), sa = sub3(ra, err);
	f3 t1, t2;
	hinge_basis(u, t1, t2);
	joint_row_put(row + 0, j, t1, cross3(sa, t1), neg3(t1), neg3(cross3(rb, t1)), k * dot3(err, t1));
	joint_row_put(row + 1, j, t2, cross3(sa, t2), neg3(t2), neg3(cross3(rb, t2)), k * dot3(err, t2));
	const f3 cu = cross3(sa, u), cbu = cross3(rb, u);
	joint_row_put(row + 2, j, u, cu, neg3(u), neg3(cbu), k * dot3(err, u), 0.0f, 0.0f);
	const f3 nu = neg3(u), ncu = neg3(cu);   // J_s: lin_a = -u, ang_a = -cross(sa, u), lin_b = u, ang_b = cross(rb, u)
	const float s = dot3(sub3(wb, wa), u);
	if (flags & NB_JOINT_MOTOR) { const float lim = d.max_motor_torque * dt; joint_row_put(drow++, j, nu, ncu, u, cbu, -d.motor_speed, -lim, lim); }
	if (flags & NB_JOINT_LIMIT) {
		joint_row_put(drow + 0, j, nu, ncu, u, cbu, limit_bias(s - d.lower, dt, k), 0.0f, INFINITY);
		joint_row_put(drow + 1, j, u, cu, nu, neg3(cbu), limit_bias(d.upper - s, dt, k), 0.0f, INFINITY);
	}
	position[0] = s;
}

// BALL + CONE / TWIST: the swing-twist split of the relative rotation d about the twist axis u, the cone row (in the motor's slot) and the
// twist limit rows (HINGE LIMIT's rows on the twist's half-angle pair).
NB_DEV void swing_twist_rows(nb_constraint_row* drow, const nb_joint& j, const JointDrive& d, u32 flags, f3 u, quat q, float dt, float k, float* position) {
	const f3 zero = mk3(0.0f, 0.0f, 0.0f);
	if (q.s < 0.0f) { q.v = neg3(q.v); q.s = -q.s; }
	const float a_ = dot3(q.v, u), sh = -a_, ch = q.s;
	const f3 p = sub3(q.v, mul3(u, a_));
	const float ss = sqrtf(dot3(p, p)), cs = sqrtf(sh * sh + ch * ch);
	float st = 0.0f, ct = 1.0f;
	if (cs > 0.0f) { const float r = 1.0f / cs; st = sh * r; ct = ch * r; }
	if (flags & NB_JOINT_CONE) {   // (sc, cc) = (sin, cos) of cone / 2, in the motor's slots
		// the swing's direction of steepest change: the axis that turns u toward conj(q) u (p, the swing's own axis, is that axis turned
		// about u by half the twist)
		const quat cq = { neg3(q.v), q.s };
		const f3 g = cross3(qrot(cq, u), u);
		const float sg = sqrtf(dot3(g, g));
		const f3 n = sg > 0.0f ? mul3(g, 1.0f / sg) : zero;
		joint_row_put(drow++, j, zero, neg3(n), zero, n, limit_bias(2.0f * (d.motor_speed * cs - d.max_motor_torque * ss), dt, k), 0.0f, INFINITY);
	}
	if (flags & NB_JOINT_TWIST) { angle_limit_rows(drow, j, d, u, st, ct, dt, k); position[0] = st; position[1] = ct; }
	else { position[0] = ss; position[1] = cs; }
}

// One thread per joint: the joint's rows from the two transforms (include/nudge_b200.h, Joints), with a drive table its drive's rows at
// drows + row, and with a spring table its spring's rows at srows + row.
__global__ void __launch_bounds__(NB_BLOCK) k_joint_rows(const nb_joint* joints, u32 n, const nb_transform* xf, float dt, nb_constraint_row* rows, JointDrive* drives,
		nb_constraint_row* drows, JointSpring* springs, nb_constraint_row* srows) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const nb_joint j = joints[i];
		const u32 type = j.type & 3u;
		nb_constraint_row* row = rows + (j.type >> 2);
		const float k = j.beta / dt;
		u32 flags = 0;
		nb_constraint_row* drow = drows;
		JointDrive d;
		const JointSpring* sp = springs ? springs + i : nullptr;   // read where used: the entry is 16 words
		const bool sprung = sp && sp->present;
		nb_constraint_row* srow = sprung ? srows + sp->row : srows;
		if (drives) {
			d = drives[i];
			flags = d.flags; drow = drows + d.row;
			bool broken = d.broken != 0;
			if (!broken && (flags & NB_JOINT_BREAKABLE) && joint_breaks(row, drow, type, flags, d, dt)) { broken = true; drives[i].broken = 1u; }
			if (broken) {
				for (u32 r = 0; r < joint_row_count(type); ++r) joint_row_zero(row + r, j);
				for (u32 r = 0; r < drive_row_count(flags); ++r) joint_row_zero(drow + r, j);
				if (sprung) for (u32 r = 0; r < spring_row_count(type); ++r) joint_row_zero(srow + r, j);
				continue;
			}
		}
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
			const f3 ca = cross3(ra, dir), cb = neg3(cross3(rb, dir));
			// with a limit or a spring the own row stays in place with no force; the range rows and the spring row push
			if ((flags & NB_JOINT_LIMIT) || sprung) joint_row_put(row, j, dir, ca, neg3(dir), cb, k * (dist - j.length), 0.0f, 0.0f);
			else joint_row_put(row, j, dir, ca, neg3(dir), cb, k * (dist - j.length));
			if (flags & NB_JOINT_LIMIT) {
				joint_row_put(drow + 0, j, dir, ca, neg3(dir), cb, limit_bias(dist - d.lower, dt, k), 0.0f, INFINITY);
				joint_row_put(drow + 1, j, neg3(dir), neg3(ca), dir, neg3(cb), limit_bias(d.upper - dist, dt, k), 0.0f, INFINITY);
				drives[i].position[0] = dist;
			}
			if (sprung) { spring_row_put(srow, j, dir, ca, neg3(dir), cb, dist - sp->target[0], *sp, dt); springs[i].position[0] = dist; }
			continue;
		}
		if (flags & NB_JOINT_SLIDE) slider_rows(row, drow, j, d, flags, qrot(qa, ld3(j.axis_a)), ra, rb, wa, wb, dt, k, drives[i].position);
		else {
			joint_row_put(row + 0, j, mk3(1.0f, 0.0f, 0.0f), mk3(0.0f, ra.z, -ra.y), mk3(-1.0f, 0.0f, 0.0f), mk3(0.0f, -rb.z, rb.y), k * err.x);
			joint_row_put(row + 1, j, mk3(0.0f, 1.0f, 0.0f), mk3(-ra.z, 0.0f, ra.x), mk3(0.0f, -1.0f, 0.0f), mk3(rb.z, 0.0f, -rb.x), k * err.y);
			joint_row_put(row + 2, j, mk3(0.0f, 0.0f, 1.0f), mk3(ra.y, -ra.x, 0.0f), mk3(0.0f, 0.0f, -1.0f), mk3(-rb.y, rb.x, 0.0f), k * err.z);
		}
		if (type == NB_JOINT_HINGE) {
			const f3 u = qrot(qa, ld3(j.axis_a)), w = j.b ? qrot(qb, ld3(j.axis_b)) : ld3(j.axis_b), c = cross3(u, w);
			f3 t1, t2;
			hinge_basis(u, t1, t2);
			joint_row_put(row + 3, j, zero, t1, zero, neg3(t1), -(k * dot3(c, t1)));
			joint_row_put(row + 4, j, zero, t2, zero, neg3(t2), -(k * dot3(c, t2)));
			const f3 nu = neg3(u);   // the hinge Jacobian: ang_a = -u, ang_b = u
			if (flags & NB_JOINT_MOTOR) { const float lim = d.max_motor_torque * dt; joint_row_put(drow++, j, zero, nu, zero, u, -d.motor_speed, -lim, lim); }
			if ((flags & NB_JOINT_LIMIT) || sprung) {
				quat q = joint_rel(qa, j, qb);
				if (q.s < 0.0f) { q.v = neg3(q.v); q.s = -q.s; }
				const float sh = -dot3(q.v, u), ch = q.s;
				if (flags & NB_JOINT_LIMIT) { angle_limit_rows(drow, j, d, u, sh, ch, dt, k); drives[i].position[0] = sh; drives[i].position[1] = ch; }
				if (sprung) {   // x = (theta - target) / 2 from the target's pair (st, ct)
					const float st = sp->target[0], ct = sp->target[1];
					spring_row_put(srow, j, zero, nu, zero, u, angle_limit_measure(sh * ct - ch * st, ch * ct + sh * st), *sp, dt);
					springs[i].position[0] = sh; springs[i].position[1] = ch;
				}
			}
		}
		else if (type == NB_JOINT_FIXED) {
			quat d = joint_rel(qa, j, qb);
			if (d.s < 0.0f) d.v = neg3(d.v);
			joint_row_put(row + 3, j, zero, mk3(1.0f, 0.0f, 0.0f), zero, mk3(-1.0f, 0.0f, 0.0f), k * (2.0f * d.v.x));
			joint_row_put(row + 4, j, zero, mk3(0.0f, 1.0f, 0.0f), zero, mk3(0.0f, -1.0f, 0.0f), k * (2.0f * d.v.y));
			joint_row_put(row + 5, j, zero, mk3(0.0f, 0.0f, 1.0f), zero, mk3(0.0f, 0.0f, -1.0f), k * (2.0f * d.v.z));
		}
		else if (flags & (NB_JOINT_CONE | NB_JOINT_TWIST)) swing_twist_rows(drow, j, d, flags, qrot(qa, ld3(j.axis_a)), joint_rel(qa, j, qb), dt, k, drives[i].position);
		if (sprung && type == NB_JOINT_FIXED) {   // J_s and s as a slider has them
			const f3 u = qrot(qa, ld3(j.axis_a)), sa = sub3(ra, err);
			const float s = dot3(sub3(wb, wa), u);
			spring_row_put(srow, j, neg3(u), neg3(cross3(sa, u)), u, cross3(rb, u), s - sp->target[0], *sp, dt);
			springs[i].position[0] = s;
		}
		else if (sprung && type == NB_JOINT_BALL) {   // FIXED's angular rows on the target rotation
			const quat t = { mk3(sp->target[0], sp->target[1], sp->target[2]), sp->target[3] };
			quat q = qmul(qa, t);
			if (j.b) { const quat cb = { neg3(qb.v), qb.s }; q = qmul(q, cb); }
			if (q.s < 0.0f) { q.v = neg3(q.v); q.s = -q.s; }
			spring_row_put(srow + 0, j, zero, mk3(1.0f, 0.0f, 0.0f), zero, mk3(-1.0f, 0.0f, 0.0f), 2.0f * q.v.x, *sp, dt);
			spring_row_put(srow + 1, j, zero, mk3(0.0f, 1.0f, 0.0f), zero, mk3(0.0f, -1.0f, 0.0f), 2.0f * q.v.y, *sp, dt);
			spring_row_put(srow + 2, j, zero, mk3(0.0f, 0.0f, 1.0f), zero, mk3(0.0f, 0.0f, -1.0f), 2.0f * q.v.z, *sp, dt);
			springs[i].position[0] = sqrtf(dot3(q.v, q.v)); springs[i].position[1] = q.s;
		}
	}
}

// Applies rows [first, first + count) one after the other to the bodies in `s`, keeping each row's new impulse unless `warm`.
NB_DEV void joint_rows_apply(nb_constraint_row* rows, u32 first, u32 count, RowBodies& s, int warm) {
	for (u32 r = first; r < first + count; ++r) {
		const float next = row_apply(rows[r], s, warm);
		if (!warm) rows[r].impulse = next;
	}
}

// One thread per joint of the level [begin, end): the joint's rows one after the other, the two bodies' momentum kept in registers across them.
// With a spring table the spring's rows follow the joint's own, and with a drive table the drive's rows come last.
__global__ void __launch_bounds__(NB_BLOCK) k_joint_solve(const nb_joint* joints, u32 begin, u32 end, nb_constraint_row* rows, nb_body_momentum* momentum,
		const nb_body_properties* props, const float4* inertia, const uint8_t* kind, int warm, const JointDrive* drives, nb_constraint_row* drows,
		const JointSpring* springs, nb_constraint_row* srows) {
	for (u32 i = begin + blockIdx.x * blockDim.x + threadIdx.x; i < end; i += gridDim.x * blockDim.x) {
		const u32 packed = joints[i].type;
		RowBodies s = row_bodies_load(joints[i].a, joints[i].b, momentum, props, inertia, kind);
		joint_rows_apply(rows, packed >> 2, joint_row_count(packed & 3u), s, warm);
		if (springs && springs[i].present) joint_rows_apply(srows, springs[i].row, spring_row_count(packed & 3u), s, warm);
		if (drives) joint_rows_apply(drows, drives[i].row, drive_row_count(drives[i].flags), s, warm);
		row_bodies_store(s);
	}
}

// The step's joint launches: with `dt` the row build and the warm start (nb_setup_contact_constraints), without it one pass after a sweep.
static int launch_joints(nb_context* ctx, const float* dt, cudaStream_t st) {
	const Launch L = mk_launch(ctx, st);
	const JointSet& js = ctx->jset;
	JointDrive* drives = ctx->drives.set.n ? ctx->drives.table.p : nullptr;
	nb_constraint_row* drows = ctx->drives.set.n ? ctx->drives.rows.p : nullptr;
	JointSpring* springs = ctx->springs.set.n ? ctx->springs.table.p : nullptr;
	nb_constraint_row* srows = ctx->springs.set.n ? ctx->springs.rows.p : nullptr;
	if (dt) launch_grid(L, k_joint_rows, GRID(js.n), ctx->joints.p, js.n, ctx->xf, *dt, ctx->jrows.p, drives, drows, springs, srows);
	for (u32 l = 0; l < js.levels; ++l)
		launch_grid(L, k_joint_solve, GRID(js.level_off[l + 1] - js.level_off[l]), ctx->joints.p, js.level_off[l], js.level_off[l + 1], ctx->jrows.p, ctx->mom, ctx->props,
			ctx->inertia, kin_table(ctx), dt ? 1 : 0, (const JointDrive*)drives, drows, (const JointSpring*)springs, srows);
	CK(cudaGetLastError());
	return NB_OK;
}

template<class E> static void drop_keyed(nb_context* ctx, KeyedTable<E>& t) { if (t.set.n) { t.set = KeyedSet(); ++ctx->graph_epoch; } }
static void drop_joints(nb_context* ctx) { if (ctx->jset.n) { ctx->jset = JointSet(); ctx->drives.set = ctx->springs.set = KeyedSet(); ++ctx->graph_epoch; } }

// Whether a quaternion has unit length within the tolerance a HINGE LIMIT drive asks of its joint's rel_rotation.
static bool unit_quat(const float* q) {
	const double s = (double)q[0] * q[0] + (double)q[1] * q[1] + (double)q[2] * q[2] + (double)q[3] * q[3];
	return fabs(s - 1.0) <= 1e-3;
}
// Whether axis_a has unit length within the same tolerance, as a slider's or a swing-twist limit's axis must.
static bool unit_axis(const float* v) {
	const double s = (double)v[0] * v[0] + (double)v[1] * v[1] + (double)v[2] * v[2];
	return fabs(s - 1.0) <= 1e-3;
}

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
// The shape of n joints in upload order.
static JointShape joint_shape(const nb_joint* h, u32 n) {
	JointShape s;
	for (u32 i = 0; i < n; ++i) {
		s.structure.insert(s.structure.end(), { h[i].type, h[i].a, h[i].b });
		s.unit_rel.push_back(unit_quat(h[i].rel_rotation) ? 1 : 0); s.unit_axis.push_back(unit_axis(h[i].axis_a) ? 1 : 0);
	}
	return s;
}

// Installs n checked joints in place of the set: levels, the table by level with the row offsets, and the rows holding the impulses.
static int set_joints(nb_context* ctx, const nb_joint* h, u32 n, cudaStream_t st) {
	if (!n) { drop_joints(ctx); return NB_OK; }
	JointSet js;
	static_cast<JointShape&>(js) = joint_shape(h, n);
	std::vector<nb_body_pair> ab(n);
	for (u32 i = 0; i < n; ++i) { ab[i].a = h[i].a; ab[i].b = h[i].b; }
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
	// the levels are host values in nb_step's graph, the buffers its kernel arguments; the drives and springs follow the structure
	if (js.structure != ctx->jset.structure) { drop_keyed(ctx, ctx->drives); drop_keyed(ctx, ctx->springs); }
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

// What nb_upload_joint_drives refuses in a drive of a joint set of shape `js`; null if valid.
static const char* drive_problem(const nb_joint_drive& d, const JointShape& js) {
	if (d.joint >= js.structure.size() / 3) return "a joint index at or beyond the joint count";
	if (d.flags & ~(u32)(NB_JOINT_LIMIT | NB_JOINT_MOTOR | NB_JOINT_BREAKABLE | NB_JOINT_SLIDE | NB_JOINT_CONE | NB_JOINT_TWIST)) return "an unknown flag";
	const u32 type = js.structure[3 * (size_t)d.joint];
	const u32 fixed = d.flags & NB_JOINT_SLIDE ? NB_JOINT_SLIDE | NB_JOINT_LIMIT | NB_JOINT_MOTOR | NB_JOINT_BREAKABLE : NB_JOINT_SLIDE | NB_JOINT_BREAKABLE;
	const u32 takes = type == NB_JOINT_HINGE ? NB_JOINT_LIMIT | NB_JOINT_MOTOR | NB_JOINT_BREAKABLE : type == NB_JOINT_DISTANCE ? NB_JOINT_LIMIT | NB_JOINT_BREAKABLE
		: type == NB_JOINT_FIXED ? fixed : NB_JOINT_CONE | NB_JOINT_TWIST | NB_JOINT_BREAKABLE;
	if (d.flags & ~takes) return "a flag the joint's type does not take";
	const float fields[] = { d.lower, d.upper, d.motor_speed, d.max_motor_torque, d.impulse[0], d.impulse[1], d.impulse[2], d.position };
	for (float x : fields) if (!std::isfinite(x)) return "a field that is not finite";
	for (float x : { d.break_force, d.break_torque }) if (!std::isfinite(x) && x != INFINITY) return "a threshold that is neither finite nor +inf";
	if (d.max_motor_torque < 0.0f || d.break_force < 0.0f || d.break_torque < 0.0f) return "a negative torque or threshold";
	if (d.broken > 1) return "broken is not 0 or 1";
	const float pi = 3.14159265358979f;
	if (d.flags & NB_JOINT_LIMIT) {
		if (d.lower > d.upper) return "lower > upper";
		if (type == NB_JOINT_HINGE && (d.lower < -pi || d.upper > pi)) return "a hinge limit outside [-pi, pi]";
		if (type == NB_JOINT_DISTANCE && d.lower < 0.0f) return "a negative distance limit";
		if (type == NB_JOINT_HINGE && !js.unit_rel[d.joint]) return "a HINGE LIMIT whose joint's rel_rotation is not of unit length";
	}
	if (d.flags & NB_JOINT_TWIST) {
		if (d.lower > d.upper) return "lower > upper";
		if (d.lower < -pi || d.upper > pi) return "a twist limit outside [-pi, pi]";
	}
	// a cone keeps its half-angle pair in the motor's slots of the device table
	if ((d.flags & NB_JOINT_CONE) && !(d.cone > 0.0f && d.cone <= pi)) return "a cone outside (0, pi]";
	if ((d.flags & NB_JOINT_CONE) && (d.motor_speed != 0.0f || d.max_motor_torque != 0.0f)) return "a CONE drive with a motor speed or torque";
	if ((d.flags & (NB_JOINT_SLIDE | NB_JOINT_CONE | NB_JOINT_TWIST)) && !js.unit_axis[d.joint]) return "a SLIDE, CONE or TWIST drive whose joint's axis_a is not of unit length";
	if ((d.flags & (NB_JOINT_CONE | NB_JOINT_TWIST)) && !js.unit_rel[d.joint]) return "a CONE or TWIST drive whose joint's rel_rotation is not of unit length";
	return nullptr;
}

// Sparse tables keyed by joint (the drives, the springs) share their checks, their order and their installation.
// The checks: a null list with n > 0, each entry's own problem (`problem`, null if none), two entries on one joint; `what` names an entry.
template<class T, class Problem> static int check_keyed(nb_context* ctx, const T* h, u32 n, const char* what, Problem problem) {
	if (n && !h) { ctx->error = std::string("null ") + what + " list"; return NB_ERR_ARGUMENT; }
	for (u32 i = 0; i < n; ++i)
		if (const char* p = problem(h[i])) { ctx->error = std::string(what) + " " + std::to_string(i) + ": " + p; return NB_ERR_ARGUMENT; }
	std::vector<u32> joints(n);
	for (u32 i = 0; i < n; ++i) joints[i] = h[i].joint;
	std::sort(joints.begin(), joints.end());
	for (u32 i = 1; i < n; ++i)
		if (joints[i] == joints[i - 1]) { ctx->error = std::string("two ") + what + "s on joint " + std::to_string(joints[i]); return NB_ERR_ARGUMENT; }
	return NB_OK;
}
// The checked entries in joint order, and per table position of the joint set the entry on that joint (-1: none).
template<class T> static void keyed_order(const JointSet& js, const T* h, u32 n, std::vector<u32>& by_joint, std::vector<int>& at) {
	by_joint.resize(n);
	for (u32 i = 0; i < n; ++i) by_joint[i] = i;
	std::sort(by_joint.begin(), by_joint.end(), [&](u32 x, u32 y) { return h[x].joint < h[y].joint; });
	at.assign(js.n, -1);
	for (u32 i : by_joint) at[js.order[h[i].joint]] = (int)i;
}
// A row as an upload installs it: zeros but its accumulated impulse, which k_joint_rows builds the row around.
static nb_constraint_row impulse_row(float impulse) { nb_constraint_row r; memset(&r, 0, sizeof(r)); r.impulse = impulse; return r; }
// Installs `next`, with the row count of `rows`, in place of t's set: the device table (one entry per joint in table order) and its rows,
// staged.  Synchronises only when
// a buffer grows.  The table and the rows are arguments of the joint kernels, null without a set, and the structure decides which rows
// k_joint_solve applies: nb_step's graph is re-recorded when the structure changed or a buffer moved.
template<class E> static int put_keyed(nb_context* ctx, KeyedTable<E>& t, KeyedSet&& next, const std::vector<E>& table, const std::vector<nb_constraint_row>& rows,
		cudaStream_t st) {
	const void* before[2] = { t.table.p, t.rows.p };
	GROW(t.table, table.size(), st); GROW(t.rows, rows.size(), st);
	CK(put_staged(ctx, t.table.p, table.data(), sizeof(E) * table.size(), st));
	CK(put_staged(ctx, t.rows.p, rows.data(), sizeof(nb_constraint_row) * rows.size(), st));
	if (next.structure != t.set.structure || before[0] != t.table.p || before[1] != t.rows.p) ++ctx->graph_epoch;
	t.set = std::move(next);
	t.set.nrows = (u32)rows.size();
	return NB_OK;
}
// The host side of the download calls: the count, the capacity and null checks, then `get`.  Synchronises.
template<class T> static int download_keyed(nb_context* ctx, T* h, u32 capacity, u32* count, u32 n, const char* what,
		int (*get)(nb_context*, std::vector<T>&, cudaStream_t), cudaStream_t st) {
	if (count) *count = n;
	if (capacity < n) { ctx->error = std::string("host ") + what + " array too small: " + std::to_string(n) + " " + what + "s"; return NB_ERR_CAPACITY; }
	if (n && !h) { ctx->error = std::string("null ") + what + " array"; return NB_ERR_ARGUMENT; }
	std::vector<T> out;
	if (int r = get(ctx, out, st)) return r;
	std::copy(out.begin(), out.end(), h);
	return NB_OK;
}

static int check_drives(nb_context* ctx, const nb_joint_drive* h, u32 n, const JointShape& js) {
	return check_keyed(ctx, h, n, "drive", [&](const nb_joint_drive& d) { return drive_problem(d, js); });
}

// Installs n checked drives in place of the set: the table (one entry per joint in table order, with the limits' and the cone's half-angle
// pairs) and the drive rows holding the uploaded impulses, per driven joint in table order.
static int set_drives(nb_context* ctx, const nb_joint_drive* h, u32 n, cudaStream_t st) {
	if (!n) { drop_keyed(ctx, ctx->drives); return NB_OK; }
	const JointSet& js = ctx->jset;
	std::vector<u32> by_joint;
	std::vector<int> at;   // table position -> drive
	keyed_order(js, h, n, by_joint, at);
	KeyedSet ds;
	ds.n = n;
	for (u32 i : by_joint) ds.structure.insert(ds.structure.end(), { h[i].joint, h[i].flags });
	std::vector<JointDrive> table(js.n);
	memset(table.data(), 0, sizeof(JointDrive) * table.size());
	std::vector<nb_constraint_row> rows;
	for (u32 p = 0; p < js.n; ++p) {
		if (at[p] < 0) continue;
		const nb_joint_drive& d = h[at[p]];
		JointDrive& e = table[p];
		e.flags = d.flags; e.row = (u32)rows.size(); e.lower = d.lower; e.upper = d.upper;
		if (((d.flags & NB_JOINT_LIMIT) && js.structure[3 * (size_t)d.joint] == NB_JOINT_HINGE) || (d.flags & NB_JOINT_TWIST)) {
			e.sl = (float)sin(0.5 * d.lower); e.cl = (float)cos(0.5 * d.lower); e.su = (float)sin(0.5 * d.upper); e.cu = (float)cos(0.5 * d.upper);
		}
		e.motor_speed = d.motor_speed; e.max_motor_torque = d.max_motor_torque; e.break_force = d.break_force; e.break_torque = d.break_torque;
		e.broken = d.broken;
		if (d.flags & NB_JOINT_CONE) { e.motor_speed = (float)sin(0.5 * d.cone); e.max_motor_torque = (float)cos(0.5 * d.cone); e.cone = d.cone; }
		for (u32 k = 0; k < 3; ++k)
			if (d.flags & (k ? NB_JOINT_LIMIT | NB_JOINT_TWIST : NB_JOINT_MOTOR | NB_JOINT_CONE)) rows.push_back(impulse_row(d.impulse[k]));
	}
	return put_keyed(ctx, ctx->drives, std::move(ds), table, rows, st);
}

// The drives in joint-index order with their rows' current impulses, broken flags and positions.  Synchronises.
static int get_drives(nb_context* ctx, std::vector<nb_joint_drive>& out, cudaStream_t st) {
	const JointSet& js = ctx->jset;
	const KeyedSet& ds = ctx->drives.set;
	out.resize(ds.n);
	if (!ds.n) return NB_OK;
	std::vector<JointDrive> table(js.n);
	std::vector<nb_constraint_row> rows(ds.nrows);
	CK(cudaMemcpyAsync(table.data(), ctx->drives.table.p, sizeof(JointDrive) * table.size(), cudaMemcpyDeviceToHost, st));
	if (ds.nrows) CK(cudaMemcpyAsync(rows.data(), ctx->drives.rows.p, sizeof(nb_constraint_row) * rows.size(), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	for (u32 m = 0; m < ds.n; ++m) {
		const u32 joint = ds.structure[2 * (size_t)m];
		const JointDrive& e = table[js.order[joint]];
		nb_joint_drive& d = out[m];
		memset(&d, 0, sizeof(d));
		d.joint = joint; d.flags = e.flags; d.lower = e.lower; d.upper = e.upper; d.motor_speed = e.motor_speed; d.max_motor_torque = e.max_motor_torque;
		d.break_force = e.break_force; d.break_torque = e.break_torque; d.broken = e.broken;
		u32 r = e.row;
		for (u32 k = 0; k < 3; ++k) if (e.flags & (k ? NB_JOINT_LIMIT | NB_JOINT_TWIST : NB_JOINT_MOTOR | NB_JOINT_CONE)) d.impulse[k] = rows[r++].impulse;
		const u32 type = js.structure[3 * (size_t)joint];
		if (e.flags & (NB_JOINT_LIMIT | NB_JOINT_SLIDE | NB_JOINT_CONE | NB_JOINT_TWIST))
			d.position = type == NB_JOINT_HINGE || type == NB_JOINT_BALL ? (float)(2.0 * atan2((double)e.position[0], (double)e.position[1])) : e.position[0];
		if (e.flags & NB_JOINT_CONE) { d.motor_speed = 0.0f; d.max_motor_torque = 0.0f; d.cone = e.cone; }
	}
	return NB_OK;
}

// What nb_upload_joint_springs refuses in a spring of a joint set of shape `js`; null if valid.
static const char* spring_problem(const nb_joint_spring& s, const JointShape& js) {
	if (s.joint >= js.structure.size() / 3) return "a joint index at or beyond the joint count";
	if (s.reserved) return "reserved is not 0";
	const float fields[] = { s.target[0], s.target[1], s.target[2], s.target[3], s.target_velocity, s.stiffness, s.damping, s.impulse[0], s.impulse[1],
							 s.impulse[2], s.position };
	for (float x : fields) if (!std::isfinite(x)) return "a field that is not finite";
	if (!std::isfinite(s.max_force) && s.max_force != INFINITY) return "a max_force that is neither finite nor +inf";
	if (s.stiffness < 0.0f || s.damping < 0.0f || s.max_force < 0.0f) return "a negative stiffness, damping or max_force";
	if (s.stiffness == 0.0f && s.damping == 0.0f) return "stiffness and damping both 0";
	// bounds under which every row is finite for 1e-6 <= dt <= 1 (include/nudge_b200.h): dt * den >= 1e-24, so softness <= 1e24, and
	// |bias| <= |C| / dt + |target_velocity|
	const float gmin = 1e-12f, gmax = 1e12f;
	for (float x : { s.stiffness, s.damping }) if (x != 0.0f && (x < gmin || x > gmax)) return "a stiffness or damping outside {0} and [1e-12, 1e12]";
	if (fabsf(s.target_velocity) > gmax) return "a target velocity beyond 1e12";
	const u32 type = js.structure[3 * (size_t)s.joint];
	if ((type == NB_JOINT_FIXED || type == NB_JOINT_DISTANCE) && fabsf(s.target[0]) > gmax) return "a target beyond 1e12";
	if (type != NB_JOINT_BALL && (s.target[1] != 0.0f || s.target[2] != 0.0f || s.target[3] != 0.0f)) return "a nonzero target word the joint's type does not read";
	const float pi = 3.14159265358979f;
	if (type == NB_JOINT_HINGE && (s.target[0] < -pi || s.target[0] > pi)) return "a hinge target outside [-pi, pi]";
	if (type == NB_JOINT_HINGE && !js.unit_rel[s.joint]) return "a HINGE spring whose joint's rel_rotation is not of unit length";
	if (type == NB_JOINT_FIXED && !js.unit_axis[s.joint]) return "a FIXED spring whose joint's axis_a is not of unit length";
	if (type == NB_JOINT_DISTANCE && s.target[0] < 0.0f) return "a negative distance target";
	if (type == NB_JOINT_BALL && s.target_velocity != 0.0f) return "a BALL spring with a target velocity";
	if (type == NB_JOINT_BALL && !unit_quat(s.target)) return "a BALL target rotation not of unit length";
	return nullptr;
}
static int check_springs(nb_context* ctx, const nb_joint_spring* h, u32 n, const JointShape& js) {
	return check_keyed(ctx, h, n, "spring", [&](const nb_joint_spring& s) { return spring_problem(s, js); });
}

// Installs n checked springs in place of the set: the table (one entry per joint in table order, a hinge's target as its half-angle pair)
// and the spring rows holding the uploaded impulses, per sprung joint in table order.
static int set_springs(nb_context* ctx, const nb_joint_spring* h, u32 n, cudaStream_t st) {
	if (!n) { drop_keyed(ctx, ctx->springs); return NB_OK; }
	const JointSet& js = ctx->jset;
	std::vector<u32> by_joint;
	std::vector<int> at;   // table position -> spring
	keyed_order(js, h, n, by_joint, at);
	KeyedSet ss;
	ss.n = n;
	for (u32 i : by_joint) ss.structure.push_back(h[i].joint);
	std::vector<JointSpring> table(js.n);
	memset(table.data(), 0, sizeof(JointSpring) * table.size());
	std::vector<nb_constraint_row> rows;
	for (u32 p = 0; p < js.n; ++p) {
		if (at[p] < 0) continue;
		const nb_joint_spring& s = h[at[p]];
		const u32 type = js.structure[3 * (size_t)s.joint];
		JointSpring& e = table[p];
		e.present = 1; e.row = (u32)rows.size();
		for (u32 k = 0; k < 4; ++k) e.target[k] = s.target[k];
		if (type == NB_JOINT_HINGE) { e.target[0] = (float)sin(0.5 * s.target[0]); e.target[1] = (float)cos(0.5 * s.target[0]); e.angle = s.target[0]; }
		e.target_velocity = s.target_velocity; e.stiffness = s.stiffness; e.damping = s.damping; e.max_force = s.max_force;
		for (u32 k = 0; k < spring_row_count(type); ++k) rows.push_back(impulse_row(s.impulse[k]));
	}
	return put_keyed(ctx, ctx->springs, std::move(ss), table, rows, st);
}

// The springs in joint-index order with their rows' current impulses and positions.  Synchronises.
static int get_springs(nb_context* ctx, std::vector<nb_joint_spring>& out, cudaStream_t st) {
	const JointSet& js = ctx->jset;
	const KeyedSet& ss = ctx->springs.set;
	out.resize(ss.n);
	if (!ss.n) return NB_OK;
	std::vector<JointSpring> table(js.n);
	std::vector<nb_constraint_row> rows(ss.nrows);
	CK(cudaMemcpyAsync(table.data(), ctx->springs.table.p, sizeof(JointSpring) * table.size(), cudaMemcpyDeviceToHost, st));
	CK(cudaMemcpyAsync(rows.data(), ctx->springs.rows.p, sizeof(nb_constraint_row) * rows.size(), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	for (u32 m = 0; m < ss.n; ++m) {
		const u32 joint = ss.structure[m], type = js.structure[3 * (size_t)joint];
		const JointSpring& e = table[js.order[joint]];
		nb_joint_spring& s = out[m];
		memset(&s, 0, sizeof(s));
		s.joint = joint;
		for (u32 k = 0; k < 4; ++k) s.target[k] = e.target[k];
		if (type == NB_JOINT_HINGE) { s.target[0] = e.angle; s.target[1] = 0.0f; }
		s.target_velocity = e.target_velocity; s.stiffness = e.stiffness; s.damping = e.damping; s.max_force = e.max_force;
		for (u32 k = 0; k < spring_row_count(type); ++k) s.impulse[k] = rows[e.row + k].impulse;
		s.position = type == NB_JOINT_HINGE || type == NB_JOINT_BALL ? (float)(2.0 * atan2((double)e.position[0], (double)e.position[1])) : e.position[0];
	}
	return NB_OK;
}

__global__ void __launch_bounds__(NB_BLOCK) k_joint_wake(const u32* bodies, u32 n, uint8_t* idle) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) idle[bodies[i]] = 0;
}
// Sets the idle counter of each listed body to 0: the list staged into spawn_idx, then one launch of k_joint_wake (none for an empty list).
static int wake_bodies(nb_context* ctx, const std::vector<u32>& bodies, cudaStream_t st) {
	if (bodies.empty()) return NB_OK;
	GROW(ctx->spawn_idx, bodies.size(), st);
	CK(put_staged(ctx, ctx->spawn_idx.p, bodies.data(), sizeof(u32) * bodies.size(), st));
	launch_grid(mk_launch(ctx, st), k_joint_wake, GRID(bodies.size()), ctx->spawn_idx.p, (u32)bodies.size(), ctx->idle);
	CK(cudaGetLastError());
	return NB_OK;
}

// A whole joint set on the host in the public types, as a state file holds it and body removal renumbers it: the joints in upload order
// with their current impulses, and the drives and springs in joint order.
struct JointBundle { std::vector<nb_joint> joints; std::vector<nb_joint_drive> drives; std::vector<nb_joint_spring> springs; };
// The context's joint set.  Synchronises.
static int get_joint_bundle(nb_context* ctx, JointBundle& b, cudaStream_t st) {
	if (int r = get_joints(ctx, b.joints, st)) return r;
	if (int r = get_drives(ctx, b.drives, st)) return r;
	return get_springs(ctx, b.springs, st);
}
// The upload's checks for a context with B bodies: the joints, then the drives and springs against the bundle's own joints.
static int check_joint_bundle(nb_context* ctx, const JointBundle& b, u32 B) {
	const u32 n = (u32)b.joints.size();
	if (int r = check_joints(ctx, b.joints.data(), n, B)) return r;
	const JointShape shape = joint_shape(b.joints.data(), n);
	if (int r = check_drives(ctx, b.drives.data(), (u32)b.drives.size(), shape)) return r;
	return check_springs(ctx, b.springs.data(), (u32)b.springs.size(), shape);
}
// Installs a checked bundle in place of the context's joint set; an empty table removes the context's.
static int put_joint_bundle(nb_context* ctx, const JointBundle& b, cudaStream_t st) {
	if (int r = set_joints(ctx, b.joints.data(), (u32)b.joints.size(), st)) return r;
	if (int r = set_drives(ctx, b.drives.data(), (u32)b.drives.size(), st)) return r;
	return set_springs(ctx, b.springs.data(), (u32)b.springs.size(), st);
}

extern "C" {

int nb_upload_joints(nb_context* ctx, const nb_joint* h, uint32_t n, void* stream) {
	NB_RANGE("nb_upload_joints");
	if (int r = check_joints(ctx, h, n, ctx->B)) return r;
	return set_joints(ctx, h, n, (cudaStream_t)stream);
}

int nb_download_joints(nb_context* ctx, nb_joint* h, uint32_t capacity, uint32_t* count, void* stream) {
	NB_RANGE("nb_download_joints");
	return download_keyed(ctx, h, capacity, count, ctx->jset.n, "joint", get_joints, (cudaStream_t)stream);
}

int nb_upload_joint_drives(nb_context* ctx, const nb_joint_drive* h, uint32_t n, void* stream) {
	NB_RANGE("nb_upload_joint_drives");
	if (int r = check_drives(ctx, h, n, ctx->jset)) return r;
	return set_drives(ctx, h, n, (cudaStream_t)stream);
}

int nb_download_joint_drives(nb_context* ctx, nb_joint_drive* h, uint32_t capacity, uint32_t* count, void* stream) {
	NB_RANGE("nb_download_joint_drives");
	return download_keyed(ctx, h, capacity, count, ctx->drives.set.n, "drive", get_drives, (cudaStream_t)stream);
}

int nb_upload_joint_springs(nb_context* ctx, const nb_joint_spring* h, uint32_t n, void* stream) {
	NB_RANGE("nb_upload_joint_springs");
	const JointSet& js = ctx->jset;
	if (int r = check_springs(ctx, h, n, js)) return r;
	cudaStream_t st = (cudaStream_t)stream;
	if (int r = set_springs(ctx, h, n, st)) return r;
	// the sprung joints' dynamic bodies get idle counter 0, so that a new target reaches a body that has fallen asleep (as nb_remove_bodies
	// wakes a joint's kept side); not body 0, not a kinematic body
	std::vector<u32> wake;
	for (u32 i = 0; i < n; ++i)
		for (u32 k = 0; k < 2; ++k) {
			const u32 b = js.structure[3 * (size_t)h[i].joint + 1 + k];
			if (b && !std::binary_search(ctx->kin_list.begin(), ctx->kin_list.end(), b)) wake.push_back(b);
		}
	std::sort(wake.begin(), wake.end());
	wake.erase(std::unique(wake.begin(), wake.end()), wake.end());
	return wake_bodies(ctx, wake, st);
}

int nb_download_joint_springs(nb_context* ctx, nb_joint_spring* h, uint32_t capacity, uint32_t* count, void* stream) {
	NB_RANGE("nb_download_joint_springs");
	return download_keyed(ctx, h, capacity, count, ctx->springs.set.n, "spring", get_springs, (cudaStream_t)stream);
}

}  // extern "C"
