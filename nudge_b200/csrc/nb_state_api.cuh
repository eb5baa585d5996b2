// nudge_b200 — state serialisation (SURVEY.md §8 f3): the caller-owned PODs of nudge.h:73-129 (BodyData, ColliderData, BodyConnections,
// ContactCache; widened layout of include/nudge_b200.h) dumped from / loaded into the device-resident context as one flat file.
// Doubles as a checkpoint and makes a parity failure reproducible: tests dump the state they disagree on and tools/nb_replay steps it
// headless.  Included at the end of nb_api.cu.
//
// File layout (little endian): header { char magic[8] = "NBSTATE1"; u32 version; u32 bodies, boxes, spheres, connections, cache;
// u32 solver_mode; u32 reserved[8]; } followed by these sections in this order (state_sections), each padded with zeros to 16 bytes:
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
// Each version defines more reserved words: version 2 reserved[0] = filter flags and reserved[1]; version 3 reserved[2] = 1 and
// reserved[3] = max_sensor_pairs; version 4 reserved[2] = 0 or 1 and reserved[4] >= 1; version 5 reserved[2] = 0 or 1, reserved[4] >= 0 and
// reserved[5] = 1.  A context writes version 5 with a body force table, else 4 with a kinematic set, else 3 with sensors, else 2 with a
// filter table or flags, else 1.  Every version loads; words a version does not define are ignored, and a file without a table or flags
// removes the context's.  A kinematic body's velocities are its momentum row.
#pragma once

struct NbStateHeader { char magic[8]; u32 version, bodies, boxes, spheres, connections, cache, solver_mode, reserved[8]; };

// Reads and checks a state file's header, and zeroes the reserved words its version does not define, so that each section's presence is a
// plain word test.
static bool state_header_read(FILE* f, NbStateHeader& h) {
	if (fread(&h, sizeof(h), 1, f) != 1 || memcmp(h.magic, "NBSTATE1", 8)) return false;
	if (h.version < 2) h.reserved[0] = h.reserved[1] = 0;
	if (h.version < 3) h.reserved[2] = h.reserved[3] = 0;
	if (h.version < 4) h.reserved[4] = 0;
	if (h.version < 5) h.reserved[5] = 0;
	return h.version == 1 || h.version == 2 || (h.version == 3 && h.reserved[2] == 1) || (h.version == 4 && h.reserved[2] <= 1 && h.reserved[4] >= 1) ||
		   (h.version == 5 && h.reserved[2] <= 1 && h.reserved[5] == 1);
}

// One section: `count` elements of `size` bytes in device memory at `dev` or, without it, in the host buffer `host`.  A load reads into
// `host` when it is given and then copies to `dev` when that is given.
struct StateSection { void* dev; std::vector<unsigned char>* host; size_t size, count; bool present; };
struct StateHostCopies { std::vector<unsigned char> mom, box_tags, sph_tags, conn, sensor, kin, frc; };

// The sections of the file with header `h`, in file order.  A load keeps in `hc` the momentum rows (the kinematic velocities), the tags
// (tagbits), the connections (the context's host copy), the sensor flags (set_sensors), the kinematic indices and the body force rows (checked
// before they are copied to the device); a save writes the kinematic indices from hc.kin.
static std::vector<StateSection> state_sections(nb_context* ctx, const NbStateHeader& h, StateHostCopies& hc, bool load) {
	const size_t K = (size_t)h.boxes + h.spheres;
	return {
		{ ctx->xf, nullptr, sizeof(nb_transform), h.bodies, true }, { ctx->props, nullptr, sizeof(nb_body_properties), h.bodies, true },
		{ ctx->mom, &hc.mom, sizeof(nb_body_momentum), h.bodies, true }, { ctx->idle, nullptr, 1, h.bodies, true },
		{ ctx->box_tags, &hc.box_tags, 4, h.boxes, true }, { ctx->box_data, nullptr, sizeof(nb_box_collider), h.boxes, true },
		{ ctx->box_xf, nullptr, sizeof(nb_transform), h.boxes, true },
		{ ctx->sph_tags, &hc.sph_tags, 4, h.spheres, true }, { ctx->sph_data, nullptr, sizeof(nb_sphere_collider), h.spheres, true },
		{ ctx->sph_xf, nullptr, sizeof(nb_transform), h.spheres, true },
		{ ctx->conn, &hc.conn, sizeof(nb_body_pair), h.connections, true },
		{ ctx->cache_tags, nullptr, 8, h.cache, true }, { ctx->cache_features, nullptr, 4, h.cache, true }, { ctx->cache_data, nullptr, 16, h.cache, true },
		{ ctx->filter, nullptr, 4, K, h.reserved[1] != 0 },
		{ load ? nullptr : ctx->sensor, &hc.sensor, 1, K, h.reserved[2] != 0 },
		{ nullptr, &hc.kin, 4, h.reserved[4], h.reserved[4] != 0 },
		{ load ? nullptr : ctx->frc, &hc.frc, sizeof(nb_body_force), h.bodies, h.reserved[5] != 0 },
	};
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
	NbStateHeader h; memset(&h, 0, sizeof(h));
	memcpy(h.magic, "NBSTATE1", 8);
	const bool filtered = ctx->has_filter || ctx->filter_flags;
	h.version = ctx->has_frc ? 5 : ctx->has_kin ? 4 : ctx->has_sensor ? 3 : filtered ? 2 : 1;
	if (filtered) { h.reserved[0] = ctx->filter_flags; h.reserved[1] = ctx->has_filter ? 1 : 0; }
	if (ctx->has_sensor) { h.reserved[2] = 1; h.reserved[3] = ctx->sensor_cap; }
	if (ctx->has_kin) h.reserved[4] = (u32)ctx->kin_list.size();
	if (ctx->has_frc) h.reserved[5] = 1;
	h.bodies = ctx->B; h.boxes = ctx->nboxes; h.spheres = ctx->nspheres; h.connections = ctx->nconn; h.cache = c[CNT_CACHE]; h.solver_mode = (u32)ctx->solver_mode;
	StateHostCopies hc;
	const unsigned char* kin = reinterpret_cast<const unsigned char*>(ctx->kin_list.data());
	hc.kin.assign(kin, kin + 4 * ctx->kin_list.size());
	std::vector<unsigned char> tmp;
	bool ok = fwrite(&h, sizeof(h), 1, f) == 1;
	for (const StateSection& s : state_sections(ctx, h, hc, false)) if (s.present) ok = ok && state_put(f, s, tmp, st);
	ok = (fclose(f) == 0) && ok;
	if (!ok) { ctx->error = std::string("write failed: ") + path; return NB_ERR_CUDA; }
	return NB_OK;
}

// Sizes in a state file (to size an nb_config before nb_create): counts[0..4] = bodies, boxes, spheres, connections, cache entries.
int nb_state_info(const char* path, uint32_t counts[5]) {
	FILE* f = fopen(path, "rb");
	if (!f) return NB_ERR_ARGUMENT;
	NbStateHeader h;
	const bool ok = state_header_read(f, h);
	fclose(f);
	if (!ok) return NB_ERR_ARGUMENT;
	counts[0] = h.bodies; counts[1] = h.boxes; counts[2] = h.spheres; counts[3] = h.connections; counts[4] = h.cache;
	return NB_OK;
}

int nb_load_state(nb_context* ctx, const char* path, void* stream) {
	cudaStream_t st = (cudaStream_t)stream;
	{ int jr = join_uploads(ctx, st); if (jr) return jr; }
	FILE* f = fopen(path, "rb");
	if (!f) { ctx->error = std::string("cannot open ") + path; return NB_ERR_ARGUMENT; }
	NbStateHeader h;
	if (!state_header_read(f, h)) { fclose(f); ctx->error = "not an nb state file"; return NB_ERR_ARGUMENT; }
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
	fclose(f);
	if (!ok) { ctx->error = std::string("read failed: ") + path; return NB_ERR_CUDA; }
	ctx->B = h.bodies; ctx->nboxes = h.boxes; ctx->nspheres = h.spheres; ctx->nconn = h.connections;
	{ const nb_body_pair* p = reinterpret_cast<const nb_body_pair*>(hc.conn.data()); ctx->conn_host.assign(p, p + h.connections); }
	ctx->scene_edited = false;   // the loaded scene replaces an edited one
	ctx->tagbits = bits_for((u64)maxtag + 1);
	ctx->kbits = bits_for(std::max(1u, h.boxes + h.spheres));
	CK(cudaMemcpyAsync(ctx->counts + CNT_CACHE, &h.cache, 4, cudaMemcpyHostToDevice, st));
	CK(cudaStreamSynchronize(st));
	if (h.solver_mode == NB_SOLVER_PARITY || h.solver_mode == NB_SOLVER_THROUGHPUT) ctx->solver_mode = (int)h.solver_mode;
	ctx->has_filter = h.reserved[1] != 0; ctx->filter_flags = h.reserved[0] & NB_FILTER_SKIP_CONNECTED;
	++ctx->graph_epoch;
	{ int r = build_conn_lookup(ctx, st); if (r) return r; }
	{ int r = set_sensors(ctx, hc.sensor.data(), h.reserved[2] ? h.boxes + h.spheres : 0, h.reserved[3], st); if (r) return r; }
	// the scatter rewrites the loaded momentum rows with their own values
	drop_kinematic(ctx);
	if (!kin.empty()) { int r = nb_upload_kinematic_bodies(ctx, kin.data(), (u32)kin.size(), st); if (r) return r; }
	drop_body_forces(ctx);
	if (h.reserved[5]) {
		{ int r = ensure_body_forces(ctx, st); if (r) return r; }
		CK(cudaMemcpyAsync(ctx->frc, frc, sizeof(nb_body_force) * (size_t)h.bodies, cudaMemcpyHostToDevice, st));
	}
	CK(cudaStreamSynchronize(st));
	return NB_OK;
}

}  // extern "C"
