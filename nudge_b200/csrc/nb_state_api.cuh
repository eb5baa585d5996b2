// nudge_b200 — state serialisation (SURVEY.md §8 f3): the caller-owned PODs of nudge.h:73-129 (BodyData, ColliderData, BodyConnections,
// ContactCache; widened layout of include/nudge_b200.h) dumped from / loaded into the device-resident context as one flat file.
// Doubles as a checkpoint and makes a parity failure reproducible: tests dump the state they disagree on and tools/nb_replay steps it
// headless.  Included at the end of nb_api.cu.
//
// File layout (little endian): header { char magic[8] = "NBSTATE1"; u32 version = 1; u32 bodies, boxes, spheres, connections, cache;
// u32 solver_mode; u32 reserved[8]; } followed by the arrays in this order, each padded to 16 bytes:
//   transforms[bodies] (32 B) | properties[bodies] (16) | momentum[bodies] (32) | idle[bodies] (1)
//   box_tags[boxes] (4) | box_data[boxes] (16) | box_transforms[boxes] (32)
//   sphere_tags[spheres] (4) | sphere_data[spheres] (4) | sphere_transforms[spheres] (32)
//   connections[connections] (8) | cache_tags[cache] (8) | cache_features[cache] (4) | cache_data[cache] (16)
// Version 2 (a context with collision filters, nb_upload_collision_filters): the same header with reserved[0] = filter flags and
// reserved[1] = 1 if the table follows, and then filter[boxes + spheres] (4, category | mask << 16) after cache_data.  A context
// without a table or flags writes version 1; both versions load, and a version-1 load removes any table and flags.
// Version 3 (a context with sensor colliders, nb_upload_sensors): reserved[0..1] as in version 2, reserved[2] = 1 (the sensor table follows;
// a version-3 header without it is not a state file), reserved[3] = the context's max_sensor_pairs, and then sensor[boxes + spheres] (1 byte
// each, 0 or 1) after the filter table, if any.  A context without sensors writes version 1 or 2 as before; every version loads, and a
// version-1 or 2 load removes any sensor table.
// Version 4 (a context with kinematic bodies, nb_upload_kinematic_bodies): reserved[0..3] as in version 3 (reserved[2] = 0 without sensors),
// reserved[4] = the number of kinematic bodies (at least 1), and then their indices (u32, ascending) after the sensor table, if any.  The
// velocities are the momentum rows.  Versions 1-3 load and remove any kinematic set.
#pragma once

struct NbStateHeader { char magic[8]; u32 version, bodies, boxes, spheres, connections, cache, solver_mode, reserved[8]; };

static bool state_put(FILE* f, const void* dev, size_t bytes, std::vector<unsigned char>& tmp, cudaStream_t st) {
	const size_t padded = (bytes + 15) & ~(size_t)15;
	tmp.assign(padded, 0);
	if (bytes && cudaMemcpyAsync(tmp.data(), dev, bytes, cudaMemcpyDeviceToHost, st) != cudaSuccess) return false;
	if (cudaStreamSynchronize(st) != cudaSuccess) return false;
	return padded == 0 || fwrite(tmp.data(), 1, padded, f) == padded;
}
static bool state_version_ok(const NbStateHeader& h) {
	return h.version == 1 || h.version == 2 || (h.version == 3 && h.reserved[2] == 1) || (h.version == 4 && h.reserved[2] <= 1 && h.reserved[4] >= 1);
}
static bool state_get(FILE* f, void* dev, size_t bytes, std::vector<unsigned char>& tmp, cudaStream_t st) {
	const size_t padded = (bytes + 15) & ~(size_t)15;
	tmp.resize(padded);
	if (padded && fread(tmp.data(), 1, padded, f) != padded) return false;
	if (bytes && cudaMemcpyAsync(dev, tmp.data(), bytes, cudaMemcpyHostToDevice, st) != cudaSuccess) return false;
	return cudaStreamSynchronize(st) == cudaSuccess;
}

// Fills the velocities of `kin` (bodies set) from the device momentum rows.  Synchronises.
static int download_rows_into(nb_context* ctx, std::vector<nb_kinematic_body>& kin, cudaStream_t st) {
	std::vector<nb_body_momentum> m(ctx->B);
	CK(cudaMemcpyAsync(m.data(), ctx->mom, sizeof(nb_body_momentum) * (size_t)ctx->B, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	for (nb_kinematic_body& k : kin) {
		const nb_body_momentum& r = m[k.body];
		for (int c = 0; c < 3; ++c) { k.velocity[c] = r.velocity[c]; k.angular_velocity[c] = r.angular_velocity[c]; }
	}
	return NB_OK;
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
	h.version = ctx->has_kin ? 4 : ctx->has_sensor ? 3 : filtered ? 2 : 1;
	if (filtered) { h.reserved[0] = ctx->filter_flags; h.reserved[1] = ctx->has_filter ? 1 : 0; }
	if (ctx->has_sensor) { h.reserved[2] = 1; h.reserved[3] = ctx->sensor_cap; }
	if (ctx->has_kin) h.reserved[4] = (u32)ctx->kin_list.size();
	h.bodies = ctx->B; h.boxes = ctx->nboxes; h.spheres = ctx->nspheres; h.connections = ctx->nconn; h.cache = c[CNT_CACHE]; h.solver_mode = (u32)ctx->solver_mode;
	std::vector<unsigned char> tmp;
	bool ok = fwrite(&h, sizeof(h), 1, f) == 1;
	ok = ok && state_put(f, ctx->xf, sizeof(nb_transform) * (size_t)h.bodies, tmp, st) && state_put(f, ctx->props, sizeof(nb_body_properties) * (size_t)h.bodies, tmp, st)
		&& state_put(f, ctx->mom, sizeof(nb_body_momentum) * (size_t)h.bodies, tmp, st) && state_put(f, ctx->idle, h.bodies, tmp, st)
		&& state_put(f, ctx->box_tags, 4 * (size_t)h.boxes, tmp, st) && state_put(f, ctx->box_data, sizeof(nb_box_collider) * (size_t)h.boxes, tmp, st) && state_put(f, ctx->box_xf, sizeof(nb_transform) * (size_t)h.boxes, tmp, st)
		&& state_put(f, ctx->sph_tags, 4 * (size_t)h.spheres, tmp, st) && state_put(f, ctx->sph_data, sizeof(nb_sphere_collider) * (size_t)h.spheres, tmp, st) && state_put(f, ctx->sph_xf, sizeof(nb_transform) * (size_t)h.spheres, tmp, st)
		&& state_put(f, ctx->conn, sizeof(nb_body_pair) * (size_t)h.connections, tmp, st)
		&& state_put(f, ctx->cache_tags, 8 * (size_t)h.cache, tmp, st) && state_put(f, ctx->cache_features, 4 * (size_t)h.cache, tmp, st) && state_put(f, ctx->cache_data, 16 * (size_t)h.cache, tmp, st);
	if (h.reserved[1]) ok = ok && state_put(f, ctx->filter, 4 * ((size_t)h.boxes + h.spheres), tmp, st);
	if (h.reserved[2]) ok = ok && state_put(f, ctx->sensor, (size_t)h.boxes + h.spheres, tmp, st);
	if (h.reserved[4]) {
		const size_t bytes = 4 * ctx->kin_list.size(), padded = (bytes + 15) & ~(size_t)15;
		tmp.assign(padded, 0);
		memcpy(tmp.data(), ctx->kin_list.data(), bytes);
		ok = ok && fwrite(tmp.data(), 1, padded, f) == padded;
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
	bool ok = fread(&h, sizeof(h), 1, f) == 1 && !memcmp(h.magic, "NBSTATE1", 8) && state_version_ok(h);
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
	if (fread(&h, sizeof(h), 1, f) != 1 || memcmp(h.magic, "NBSTATE1", 8) || !state_version_ok(h)) { fclose(f); ctx->error = "not an nb state file"; return NB_ERR_ARGUMENT; }
	const nb_config& c = ctx->cfg;
	if (h.bodies > c.max_bodies || h.boxes > c.max_boxes || h.spheres > c.max_spheres || h.connections > c.max_connections || h.cache > c.max_contacts) {
		fclose(f); ctx->error = "state file exceeds the context's capacities"; return NB_ERR_CAPACITY;
	}
	std::vector<unsigned char> tmp;
	std::vector<u32> tags;
	bool ok = state_get(f, ctx->xf, sizeof(nb_transform) * (size_t)h.bodies, tmp, st) && state_get(f, ctx->props, sizeof(nb_body_properties) * (size_t)h.bodies, tmp, st)
		&& state_get(f, ctx->mom, sizeof(nb_body_momentum) * (size_t)h.bodies, tmp, st) && state_get(f, ctx->idle, h.bodies, tmp, st);
	u32 maxtag = 1;
	ok = ok && state_get(f, ctx->box_tags, 4 * (size_t)h.boxes, tmp, st);
	if (ok) for (u32 i = 0; i < h.boxes; ++i) maxtag = std::max(maxtag, reinterpret_cast<const u32*>(tmp.data())[i]);
	ok = ok && state_get(f, ctx->box_data, sizeof(nb_box_collider) * (size_t)h.boxes, tmp, st) && state_get(f, ctx->box_xf, sizeof(nb_transform) * (size_t)h.boxes, tmp, st)
		&& state_get(f, ctx->sph_tags, 4 * (size_t)h.spheres, tmp, st);
	if (ok) for (u32 i = 0; i < h.spheres; ++i) maxtag = std::max(maxtag, reinterpret_cast<const u32*>(tmp.data())[i]);
	ok = ok && state_get(f, ctx->sph_data, sizeof(nb_sphere_collider) * (size_t)h.spheres, tmp, st) && state_get(f, ctx->sph_xf, sizeof(nb_transform) * (size_t)h.spheres, tmp, st)
		&& state_get(f, ctx->conn, sizeof(nb_body_pair) * (size_t)h.connections, tmp, st)
		&& state_get(f, ctx->cache_tags, 8 * (size_t)h.cache, tmp, st) && state_get(f, ctx->cache_features, 4 * (size_t)h.cache, tmp, st) && state_get(f, ctx->cache_data, 16 * (size_t)h.cache, tmp, st);
	const bool table = h.version >= 2 && h.reserved[1];
	if (table) ok = ok && state_get(f, ctx->filter, 4 * ((size_t)h.boxes + h.spheres), tmp, st);
	std::vector<uint8_t> sensors;
	const bool has_sensors = h.version == 3 || (h.version == 4 && h.reserved[2]);
	if (ok && has_sensors) {
		const size_t k = (size_t)h.boxes + h.spheres, padded = (k + 15) & ~(size_t)15;
		sensors.resize(padded);
		ok = padded == 0 || fread(sensors.data(), 1, padded, f) == padded;
	}
	std::vector<nb_kinematic_body> kin;
	if (ok && h.version == 4) {
		const size_t n = h.reserved[4], padded = (4 * n + 15) & ~(size_t)15;
		std::vector<u32> idx(padded / 4);
		ok = fread(idx.data(), 1, padded, f) == padded;
		kin.resize(n);
		for (size_t i = 0; ok && i < n; ++i) {
			if (idx[i] == 0 || idx[i] >= h.bodies || (i && idx[i] <= idx[i - 1])) ok = false;   // nonzero, in range, ascending
			memset(&kin[i], 0, sizeof(kin[i])); kin[i].body = idx[i];
		}
	}
	fclose(f);
	if (!ok) { ctx->error = std::string("read failed: ") + path; return NB_ERR_CUDA; }
	ctx->B = h.bodies; ctx->nboxes = h.boxes; ctx->nspheres = h.spheres; ctx->nconn = h.connections;
	ctx->tagbits = bits_for((u64)maxtag + 1);
	ctx->kbits = bits_for(std::max(1u, h.boxes + h.spheres));
	CK(cudaMemcpyAsync(ctx->counts + CNT_CACHE, &h.cache, 4, cudaMemcpyHostToDevice, st));
	CK(cudaStreamSynchronize(st));
	if (h.solver_mode == NB_SOLVER_PARITY || h.solver_mode == NB_SOLVER_THROUGHPUT) ctx->solver_mode = (int)h.solver_mode;
	ctx->has_filter = table; ctx->filter_flags = h.version >= 2 ? (h.reserved[0] & NB_FILTER_SKIP_CONNECTED) : 0;
	++ctx->filter_version;
	{ int r = build_conn_lookup(ctx, st); if (r) return r; }
	{ int r = set_sensors(ctx, sensors.data(), has_sensors ? h.boxes + h.spheres : 0, has_sensors ? h.reserved[3] : 0, st); if (r) return r; }
	// the kinematic set: the velocities are already in the loaded momentum rows, so the scatter rewrites them with their own values
	drop_kinematic(ctx);
	if (!kin.empty()) {
		{ int r = download_rows_into(ctx, kin, st); if (r) return r; }
		{ int r = nb_upload_kinematic_bodies(ctx, kin.data(), (u32)kin.size(), st); if (r) return r; }
	}
	CK(cudaStreamSynchronize(st));
	return NB_OK;
}

}  // extern "C"
