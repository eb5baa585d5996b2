// nudge_b200 — state serialisation (SURVEY.md §8 f3): the caller-owned PODs of nudge.h:73-129 (BodyData, ColliderData, BodyConnections,
// ContactCache; widened layout of include/nudge_b200.h) dumped from / loaded into the device-resident context as one flat file.
// Doubles as a checkpoint and makes a parity failure reproducible: tests dump the state they disagree on and tools/nb_replay steps it
// headless.  Included at the end of nb_api.cu.
//
// File layout (little endian): header { char magic[8] = "NBSTATE1"; u32 version; u32 bodies, boxes, spheres, connections, cache;
// u32 solver_mode; u32 reserved[8]; }, from version 8 a header extension { u32 ccd_bodies; u32 reserved[3]; }, and these sections in this
// order (state_sections, then the continuous-collision rows and the joint springs), each padded with zeros to 16 bytes:
//   section                                        element (B)  count            present when
//   transforms | properties | momentum | idle      32 16 32 1   bodies           always
//   box_tags | box_data | box_transforms           4 16 32      boxes            always
//   sphere_tags | sphere_data | sphere_transforms  4 4 32       spheres          always
//   connections                                    8            connections      always
//   cache_tags | cache_features | cache_data       8 4 16       cache            always
//   filter (category | mask << 16)                 4            boxes + spheres  reserved[1] != 0
//   sensor (0 or 1)                                1            boxes + spheres  reserved[2] != 0
//   kinematic (body indices, ascending)            4            reserved[4]      reserved[4] != 0
//   body forces (nb_body_force rows, body = row)   48           bodies           reserved[5] != 0
//   joints (nb_joint, upload order, current impulses) 112        reserved[6]      reserved[6] != 0
//   joint drives (nb_joint_drive, joint order)      56           reserved[7]      reserved[7] != 0
//   ccd bodies (nb_ccd_body, ascending by body)     16           ccd_bodies       version 8 or 9
//   joint springs (nb_joint_spring, joint order)    56           ext reserved[0]  version 9
// Each version defines more reserved words: version 2 reserved[0] = filter flags and reserved[1]; version 3 reserved[2] = 1 and
// reserved[3] = max_sensor_pairs; version 4 reserved[2] = 0 or 1 and reserved[4] >= 1; version 5 reserved[2] = 0 or 1, reserved[4] >= 0 and
// reserved[5] = 1; version 6 reserved[2] and reserved[5] = 0 or 1, reserved[4] >= 0 and reserved[6] >= 1; version 7 as 6 and reserved[7] >= 1;
// version 8 as 7 with reserved[6] >= 0, reserved[7] >= 0 (drives only with joints) and ccd_bodies >= 1.  All eight reserved words being
// taken, version 8 adds the extension.  Version 9 as 8 with ccd_bodies >= 0, reserved[6] >= 1 and the extension's reserved[0] >= 1 (the
// spring count; the extension's reserved words are ignored before version 9).  A context writes version 9 with joint springs, else 8 with a
// continuous-collision set, else 7 with joint drives, else 6 with joints, else 5 with a body force table, else 4 with a kinematic set, else 3 with sensors, else 2 with a
// filter table or flags, else 1.  Every version loads; words a version does not define are ignored, and a file without a table or flags
// removes the context's.  A kinematic body's velocities are its momentum row.
#pragma once

struct NbStateHeader { char magic[8]; u32 version, bodies, boxes, spheres, connections, cache, solver_mode, reserved[8]; };
struct NbStateExt { u32 ccd_bodies, reserved[3]; };   // version 8 on; version 9: reserved[0] = the spring count

// Reads and checks a state file's header and, from version 8, its extension (all zeros before), and zeroes the reserved words its version
// does not define, so that each section's presence is a plain word test.
static bool state_header_read(FILE* f, NbStateHeader& h, NbStateExt& x) {
	memset(&x, 0, sizeof(x));
	if (fread(&h, sizeof(h), 1, f) != 1 || memcmp(h.magic, "NBSTATE1", 8)) return false;
	if ((h.version == 8 || h.version == 9) && fread(&x, sizeof(x), 1, f) != 1) return false;
	if (h.version < 9) x.reserved[0] = 0;
	if (h.version < 2) h.reserved[0] = h.reserved[1] = 0;
	if (h.version < 3) h.reserved[2] = h.reserved[3] = 0;
	if (h.version < 4) h.reserved[4] = 0;
	if (h.version < 5) h.reserved[5] = 0;
	if (h.version < 6) h.reserved[6] = 0;
	if (h.version < 7) h.reserved[7] = 0;
	return h.version == 1 || h.version == 2 || (h.version == 3 && h.reserved[2] == 1) || (h.version == 4 && h.reserved[2] <= 1 && h.reserved[4] >= 1) ||
		   (h.version == 5 && h.reserved[2] <= 1 && h.reserved[5] == 1) || (h.version == 6 && h.reserved[2] <= 1 && h.reserved[5] <= 1 && h.reserved[6] >= 1) ||
		   (h.version == 7 && h.reserved[2] <= 1 && h.reserved[5] <= 1 && h.reserved[6] >= 1 && h.reserved[7] >= 1) ||
		   (h.version == 8 && h.reserved[2] <= 1 && h.reserved[5] <= 1 && (h.reserved[7] == 0 || h.reserved[6] >= 1) && x.ccd_bodies >= 1) ||
		   (h.version == 9 && h.reserved[2] <= 1 && h.reserved[5] <= 1 && h.reserved[6] >= 1 && x.reserved[0] >= 1);
}

// One section: `count` elements of `size` bytes in device memory at `dev` or, without it, in the host buffer `host`.  A load reads into
// `host` when it is given and then copies to `dev` when that is given.  word >= 0: a context holds the element count in counts[word] (a
// file holds it in the header; a snapshot copies it on the device, nb_snapshot_api.cuh).
struct StateSection { void* dev; std::vector<unsigned char>* host; size_t size, count; bool present; int word; };
struct StateHostCopies { std::vector<unsigned char> mom, box_tags, sph_tags, conn, sensor, kin, frc, joints, drives; };

// The sections of the file with header `h`, in file order.  A load keeps in `hc` the momentum rows (the kinematic velocities), the tags
// (tagbits), the connections (the context's host copy), the sensor flags (set_sensors), the kinematic indices, the body force rows, the joints
// and their drives (checked before they are copied to the device); a save writes the kinematic indices, the joints and the drives from hc.  Snapshots extend this list (snapshot_sections).
static std::vector<StateSection> state_sections(nb_context* ctx, const NbStateHeader& h, StateHostCopies& hc, bool load) {
	const size_t K = (size_t)h.boxes + h.spheres;
	return {
		{ ctx->xf, nullptr, sizeof(nb_transform), h.bodies, true, -1 }, { ctx->props, nullptr, sizeof(nb_body_properties), h.bodies, true, -1 },
		{ ctx->mom, &hc.mom, sizeof(nb_body_momentum), h.bodies, true, -1 }, { ctx->idle, nullptr, 1, h.bodies, true, -1 },
		{ ctx->box_tags, &hc.box_tags, 4, h.boxes, true, -1 }, { ctx->box_data, nullptr, sizeof(nb_box_collider), h.boxes, true, -1 },
		{ ctx->box_xf, nullptr, sizeof(nb_transform), h.boxes, true, -1 },
		{ ctx->sph_tags, &hc.sph_tags, 4, h.spheres, true, -1 }, { ctx->sph_data, nullptr, sizeof(nb_sphere_collider), h.spheres, true, -1 },
		{ ctx->sph_xf, nullptr, sizeof(nb_transform), h.spheres, true, -1 },
		{ ctx->conn, &hc.conn, sizeof(nb_body_pair), h.connections, true, -1 },
		{ ctx->cache_tags, nullptr, 8, h.cache, true, CNT_CACHE }, { ctx->cache_features, nullptr, 4, h.cache, true, CNT_CACHE },
		{ ctx->cache_data, nullptr, 16, h.cache, true, CNT_CACHE },
		{ ctx->filter, nullptr, 4, K, h.reserved[1] != 0, -1 },
		{ load ? nullptr : ctx->sensor, &hc.sensor, 1, K, h.reserved[2] != 0, -1 },
		{ nullptr, &hc.kin, 4, h.reserved[4], h.reserved[4] != 0, -1 },
		{ load ? nullptr : ctx->frc, &hc.frc, sizeof(nb_body_force), h.bodies, h.reserved[5] != 0, -1 },
		{ nullptr, &hc.joints, sizeof(nb_joint), h.reserved[6], h.reserved[6] != 0, -1 },
		{ nullptr, &hc.drives, sizeof(nb_joint_drive), h.reserved[7], h.reserved[7] != 0, -1 },
	};
}

// The header a save of the context writes, with `cache` cache entries.
static NbStateHeader state_header_of(const nb_context* ctx, u32 cache) {
	NbStateHeader h; memset(&h, 0, sizeof(h));
	memcpy(h.magic, "NBSTATE1", 8);
	const bool filtered = ctx->has_filter || ctx->filter_flags;
	h.version = ctx->sset.n ? 9 : !ctx->ccd.empty() ? 8 : ctx->dset.n ? 7 : ctx->jset.n ? 6 : ctx->has_frc ? 5 : ctx->has_kin ? 4 : ctx->has_sensor ? 3 : filtered ? 2 : 1;
	if (filtered) { h.reserved[0] = ctx->filter_flags; h.reserved[1] = ctx->has_filter ? 1 : 0; }
	if (ctx->has_sensor) { h.reserved[2] = 1; h.reserved[3] = ctx->sensor_cap; }
	if (ctx->has_kin) h.reserved[4] = (u32)ctx->kin_list.size();
	if (ctx->has_frc) h.reserved[5] = 1;
	h.reserved[6] = ctx->jset.n; h.reserved[7] = ctx->dset.n;
	h.bodies = ctx->B; h.boxes = ctx->nboxes; h.spheres = ctx->nspheres; h.connections = ctx->nconn; h.cache = cache; h.solver_mode = (u32)ctx->solver_mode;
	return h;
}

// The host side of a state that replaces the context's (nb_load_state, nb_snapshot_restore): the counts, the connections' host copy, the tag
// and key bits, the solver mode and the table set.  sensor_cap is max_sensor_pairs as the state gives it (0 in a file: the default).
struct StateShape {
	u32 B, nboxes, nspheres, nconn, tagbits, kbits, solver_mode, filter_flags, sensor_cap;
	bool has_filter, has_sensor, has_frc;
	std::vector<nb_body_pair> conn; std::vector<u32> kin;
};
static StateShape state_shape_of(const nb_context* ctx) {
	return { ctx->B, ctx->nboxes, ctx->nspheres, ctx->nconn, ctx->tagbits, ctx->kbits, (u32)ctx->solver_mode, ctx->filter_flags, ctx->has_sensor ? ctx->sensor_cap : 0,
			 ctx->has_filter, ctx->has_sensor, ctx->has_frc, ctx->conn_host, ctx->kin_list };
}
// A load's tables, from the file's host copies: the sensor flags (boxes + spheres of them while has_sensor), the kinematic rows (one per
// entry of StateShape::kin, with the loaded velocities) and the body force rows (B while has_frc).
struct StateFileTables { const uint8_t* sensor; const nb_kinematic_body* kin; const nb_body_force* frc; };

// Installs `s` in place of the context's shape.  A load (`file` non-null) rebuilds the tables on the device from the file's host copies and
// re-records nb_step's graph.  A restore finds the table contents already copied to the device and re-records only when the table set or the
// kinematic set changes (the graph's key holds the counts, the bits and the solver mode).
static int install_state(nb_context* ctx, StateShape& s, const StateFileTables* file, cudaStream_t st) {
	const bool same_tables = s.has_filter == ctx->has_filter && s.filter_flags == ctx->filter_flags && s.has_sensor == ctx->has_sensor &&
							 (!s.has_sensor || s.sensor_cap == ctx->sensor_cap) && s.kin == ctx->kin_list && s.has_frc == ctx->has_frc;
	ctx->B = s.B; ctx->nboxes = s.nboxes; ctx->nspheres = s.nspheres; ctx->nconn = s.nconn;
	ctx->conn_host.swap(s.conn);
	ctx->tagbits = s.tagbits; ctx->kbits = s.kbits;
	if (s.solver_mode == NB_SOLVER_PARITY || s.solver_mode == NB_SOLVER_THROUGHPUT) ctx->solver_mode = (int)s.solver_mode;
	ctx->has_filter = s.has_filter; ctx->filter_flags = s.filter_flags;
	if (!file) {
		if (!same_tables) ++ctx->graph_epoch;
		ctx->conn_probe = (ctx->filter_flags & NB_FILTER_SKIP_CONNECTED) ? ctx->nconn : 0;   // the key list itself was copied
		ctx->has_sensor = s.has_sensor; ctx->sensor_cap = s.has_sensor ? s.sensor_cap : 0;
		ctx->has_kin = !s.kin.empty(); ctx->kin_list.swap(s.kin);
		ctx->has_frc = s.has_frc;
		return NB_OK;
	}
	++ctx->graph_epoch;
	{ int r = build_conn_lookup(ctx, st); if (r) return r; }
	{ int r = set_sensors(ctx, file->sensor, s.has_sensor ? s.nboxes + s.nspheres : 0, s.sensor_cap, st); if (r) return r; }
	// the scatter rewrites the loaded momentum rows with their own values
	drop_kinematic(ctx);
	if (!s.kin.empty()) { int r = nb_upload_kinematic_bodies(ctx, file->kin, (u32)s.kin.size(), st); if (r) return r; }
	drop_body_forces(ctx);
	if (s.has_frc) {
		{ int r = ensure_body_forces(ctx, st); if (r) return r; }
		CK(cudaMemcpyAsync(ctx->frc, file->frc, sizeof(nb_body_force) * (size_t)s.B, cudaMemcpyHostToDevice, st));
	}
	return NB_OK;
}

static bool state_put(FILE* f, const StateSection& s, std::vector<unsigned char>& tmp, cudaStream_t st) {
	const size_t bytes = s.size * s.count, padded = (bytes + 15) & ~(size_t)15;
	if (s.dev) {
		tmp.assign(padded, 0);
		if (bytes && cudaMemcpyAsync(tmp.data(), s.dev, bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) return false;
		if (cudaStreamSynchronize(st) != cudaSuccess) return false;
	}
	else { tmp = *s.host; tmp.resize(padded, 0); }   // the host buffer holds exactly the section
	return padded == 0 || fwrite(tmp.data(), 1, padded, f) == padded;
}
static bool state_get(FILE* f, const StateSection& s, std::vector<unsigned char>& tmp, cudaStream_t st) {
	const size_t bytes = s.size * s.count, padded = (bytes + 15) & ~(size_t)15;
	std::vector<unsigned char>& buf = s.host ? *s.host : tmp;
	buf.resize(padded);
	if (padded && fread(buf.data(), 1, padded, f) != padded) return false;
	if (!s.dev) return true;
	if (bytes && cudaMemcpyAsync(s.dev, buf.data(), bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) return false;
	return cudaStreamSynchronize(st) == cudaSuccess;
}

extern "C" {

int nb_save_state(nb_context* ctx, const char* path, void* stream) {
	cudaStream_t st = (cudaStream_t)stream;
	{ int jr = join_uploads(ctx, st); if (jr) return jr; }
	u32 c[CNT__COUNT];
	int r = get_counts(ctx, c, stream); if (r) return r;
	FILE* f = fopen(path, "wb");
	if (!f) { ctx->error = std::string("cannot open ") + path; return NB_ERR_ARGUMENT; }
	const NbStateHeader h = state_header_of(ctx, c[CNT_CACHE]);
	StateHostCopies hc;
	const unsigned char* kin = reinterpret_cast<const unsigned char*>(ctx->kin_list.data());
	hc.kin.assign(kin, kin + 4 * ctx->kin_list.size());
	std::vector<nb_joint> joints;
	if ((r = get_joints(ctx, joints, st))) { fclose(f); return r; }
	hc.joints.assign(reinterpret_cast<const unsigned char*>(joints.data()), reinterpret_cast<const unsigned char*>(joints.data() + joints.size()));
	std::vector<nb_joint_drive> drives;
	if ((r = get_drives(ctx, drives, st))) { fclose(f); return r; }
	hc.drives.assign(reinterpret_cast<const unsigned char*>(drives.data()), reinterpret_cast<const unsigned char*>(drives.data() + drives.size()));
	std::vector<nb_joint_spring> springs;
	if ((r = get_springs(ctx, springs, st))) { fclose(f); return r; }
	std::vector<unsigned char> tmp;
	bool ok = fwrite(&h, sizeof(h), 1, f) == 1;
	const NbStateExt x = { (u32)ctx->ccd.size(), { (u32)springs.size(), 0, 0 } };
	if (h.version >= 8) ok = ok && fwrite(&x, sizeof(x), 1, f) == 1;
	for (const StateSection& s : state_sections(ctx, h, hc, false)) if (s.present) ok = ok && state_put(f, s, tmp, st);
	if (h.version >= 8) ok = ok && fwrite(ctx->ccd.data(), sizeof(nb_ccd_body), ctx->ccd.size(), f) == ctx->ccd.size();   // 16 bytes each: no padding
	if (h.version == 9) {   // 56 bytes each, the section padded to 16
		std::vector<unsigned char> b(reinterpret_cast<const unsigned char*>(springs.data()), reinterpret_cast<const unsigned char*>(springs.data() + springs.size()));
		b.resize((b.size() + 15) & ~(size_t)15, 0);
		ok = ok && fwrite(b.data(), 1, b.size(), f) == b.size();
	}
	ok = (fclose(f) == 0) && ok;
	if (!ok) { ctx->error = std::string("write failed: ") + path; return NB_ERR_CUDA; }
	return NB_OK;
}

// Sizes in a state file (to size an nb_config before nb_create): counts[0..4] = bodies, boxes, spheres, connections, cache entries.
int nb_state_info(const char* path, uint32_t counts[5]) {
	FILE* f = fopen(path, "rb");
	if (!f) return NB_ERR_ARGUMENT;
	NbStateHeader h;
	NbStateExt x;
	const bool ok = state_header_read(f, h, x);
	fclose(f);
	if (!ok) return NB_ERR_ARGUMENT;
	counts[0] = h.bodies; counts[1] = h.boxes; counts[2] = h.spheres; counts[3] = h.connections; counts[4] = h.cache;
	return NB_OK;
}

int nb_load_state(nb_context* ctx, const char* path, void* stream) {
	ctx->report_ok = false;
	cudaStream_t st = (cudaStream_t)stream;
	{ int jr = join_uploads(ctx, st); if (jr) return jr; }
	FILE* f = fopen(path, "rb");
	if (!f) { ctx->error = std::string("cannot open ") + path; return NB_ERR_ARGUMENT; }
	NbStateHeader h;
	NbStateExt x;
	if (!state_header_read(f, h, x)) { fclose(f); ctx->error = "not an nb state file"; return NB_ERR_ARGUMENT; }
	const nb_config& c = ctx->cfg;
	if (h.bodies > c.max_bodies || h.boxes > c.max_boxes || h.spheres > c.max_spheres || h.connections > c.max_connections || h.cache > c.max_contacts) {
		fclose(f); ctx->error = "state file exceeds the context's capacities"; return NB_ERR_CAPACITY;
	}
	StateHostCopies hc;
	std::vector<unsigned char> tmp;
	bool ok = true;
	for (const StateSection& s : state_sections(ctx, h, hc, true)) if (s.present) ok = ok && state_get(f, s, tmp, st);
	u32 maxtag = 1;
	if (ok) {
		for (u32 i = 0; i < h.boxes; ++i) maxtag = std::max(maxtag, reinterpret_cast<const u32*>(hc.box_tags.data())[i]);
		for (u32 i = 0; i < h.spheres; ++i) maxtag = std::max(maxtag, reinterpret_cast<const u32*>(hc.sph_tags.data())[i]);
	}
	// the kinematic set, with the velocities of the loaded momentum rows
	const u32* idx = reinterpret_cast<const u32*>(hc.kin.data());
	const nb_body_momentum* mom = reinterpret_cast<const nb_body_momentum*>(hc.mom.data());
	std::vector<nb_kinematic_body> kin(h.reserved[4]);
	for (size_t i = 0; ok && i < kin.size(); ++i) {
		ok = idx[i] != 0 && idx[i] < h.bodies && (i == 0 || idx[i] > idx[i - 1]);   // nonzero, in range, ascending
		if (!ok) break;
		memset(&kin[i], 0, sizeof(kin[i])); kin[i].body = idx[i];
		for (int c = 0; c < 3; ++c) { kin[i].velocity[c] = mom[idx[i]].velocity[c]; kin[i].angular_velocity[c] = mom[idx[i]].angular_velocity[c]; }
	}
	// the body force rows: each names its own row and passes nb_set_body_forces' entry checks
	const nb_body_force* frc = reinterpret_cast<const nb_body_force*>(hc.frc.data());
	for (u32 i = 0; ok && h.reserved[5] && i < h.bodies; ++i) ok = frc[i].body == i && !body_force_problem(frc[i]);
	const nb_joint* joints = reinterpret_cast<const nb_joint*>(hc.joints.data());
	ok = ok && check_joints(ctx, joints, h.reserved[6], h.bodies) == NB_OK;
	// the drives against the file's joints, through the upload's checks
	const nb_joint_drive* drives = reinterpret_cast<const nb_joint_drive*>(hc.drives.data());
	std::vector<u32> structure; std::vector<uint8_t> unit_rel, unit_ax;
	for (u32 i = 0; ok && i < h.reserved[6]; ++i) {
		structure.insert(structure.end(), { joints[i].type, joints[i].a, joints[i].b });
		unit_rel.push_back(unit_quat(joints[i].rel_rotation) ? 1 : 0); unit_ax.push_back(unit_axis(joints[i].axis_a) ? 1 : 0);
	}
	ok = ok && check_drives(ctx, drives, h.reserved[7], h.reserved[6], structure.data(), unit_rel.data(), unit_ax.data()) == NB_OK;
	// the continuous-collision set: the upload's entry checks, bodies nonzero, in range and ascending (a kinematic body may keep its entry)
	std::vector<nb_ccd_body> ccd(x.ccd_bodies);
	ok = ok && (ccd.empty() || fread(ccd.data(), sizeof(nb_ccd_body), ccd.size(), f) == ccd.size());
	for (size_t i = 0; ok && i < ccd.size(); ++i)
		ok = ccd[i].body != 0 && ccd[i].body < h.bodies && (i == 0 || ccd[i].body > ccd[i - 1].body) && !ccd_body_problem(ccd[i]);
	// the springs against the file's joints, through the upload's checks
	std::vector<nb_joint_spring> springs(x.reserved[0]);
	const size_t spring_bytes = sizeof(nb_joint_spring) * springs.size();
	std::vector<unsigned char> sb((spring_bytes + 15) & ~(size_t)15);
	ok = ok && (sb.empty() || fread(sb.data(), 1, sb.size(), f) == sb.size());
	if (ok && spring_bytes) memcpy(springs.data(), sb.data(), spring_bytes);
	ok = ok && check_springs(ctx, springs.data(), x.reserved[0], h.reserved[6], structure.data(), unit_rel.data(), unit_ax.data()) == NB_OK;
	fclose(f);
	if (!ok) { ctx->error = std::string("read failed: ") + path; return NB_ERR_CUDA; }
	ctx->scene_edited = false;   // the loaded scene replaces an edited one
	CK(cudaMemcpyAsync(ctx->counts + CNT_CACHE, &h.cache, 4, cudaMemcpyHostToDevice, st));
	CK(cudaStreamSynchronize(st));
	StateShape shape = { h.bodies, h.boxes, h.spheres, h.connections, bits_for((u64)maxtag + 1), bits_for(std::max(1u, h.boxes + h.spheres)), h.solver_mode,
						 h.reserved[0] & NB_FILTER_SKIP_CONNECTED, h.reserved[3], h.reserved[1] != 0, h.reserved[2] != 0, h.reserved[5] != 0, {}, {} };
	{ const nb_body_pair* p = reinterpret_cast<const nb_body_pair*>(hc.conn.data()); shape.conn.assign(p, p + h.connections); }
	shape.kin.assign(idx, idx + kin.size());
	const StateFileTables file = { hc.sensor.data(), kin.data(), frc };
	{ int r = install_state(ctx, shape, &file, st); if (r) return r; }
	drop_drives(ctx); drop_springs(ctx);   // a file without drives or springs removes them, also where its joints have the context's structure
	{ int r = set_joints(ctx, joints, h.reserved[6], st); if (r) return r; }
	{ int r = set_drives(ctx, drives, h.reserved[7], st); if (r) return r; }
	{ int r = set_springs(ctx, springs.data(), x.reserved[0], st); if (r) return r; }
	{ int r = set_ccd(ctx, std::move(ccd), st); if (r) return r; }   // a file of an older version removes the set
	CK(cudaStreamSynchronize(st));
	return NB_OK;
}

}  // extern "C"
