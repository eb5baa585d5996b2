// nudge_b200 — device-resident snapshots (nb_snapshot_create, nb_snapshot_destroy, nb_snapshot_save, nb_snapshot_restore; DESIGN.md
// section 8.12).
//
// A snapshot is the context's between-steps state in HBM: the sections of a state file (state_sections, nb_state_api.cuh) plus what a file
// lacks, the user rows, the joint table, the joints' rows, the joint drive table, the joint spring table and rows, the continuous-collision set (host side), the kind bytes, the sensor overlap list, the count words the state owns and the NB_FILTER_SKIP_CONNECTED key list
// (snapshot_sections).  Save and restore are one launch of k_snapshot_copy in opposite directions; the host side (counts, bits, table set,
// the connections' host copy, the kinematic set, the rows' levelling) is kept in the snapshot and installed by install_state.
// Every section but the user rows, the joints and the overlap list has its room at the context's capacities in one arena, laid out once from the
// capacity header; those are sized at the save and grown by it.  Included at the end of nb_api.cu.
#pragma once

#define NB_SNAP_SECTIONS 64   // two per lane of k_snapshot_copy's first warp

// One section of k_snapshot_copy: `size` * n bytes from src to dst, n = min(*count_dev, count) when count_dev is given, else count.  src and
// dst are 16-byte aligned unless the section is shorter than 16 bytes.
struct SnapSection { const void* src; void* dst; const u32* count_dev; u32 size, count; };
struct SnapTable { SnapSection s[NB_SNAP_SECTIONS]; u32 n; };

// The counter words a snapshot owns, in its arena: the cache length, the contact-event step counter, the length of the sensor overlap list.
static const int kSnapWords[3] = { CNT_CACHE, CNT_EV_STEP, CNT_SENSOR_OLD };

// The table is a kernel parameter.  Each block sizes the sections (device counts included) into a prefix of 16-byte chunks, then walks
// the chunks of the concatenated live ranges grid-stride; a section's last chunk copies only its live bytes.
static_assert(NB_SNAP_SECTIONS == 64, "k_snapshot_copy's first warp sizes two sections per lane");
__device__ __forceinline__ u64 snap_section_bytes(const SnapTable& t, u32 i) {
	if (i >= t.n) return 0;
	const SnapSection& s = t.s[i];
	return (u64)s.size * (s.count_dev ? min(*s.count_dev, s.count) : s.count);
}
__global__ void __launch_bounds__(NB_BLOCK) k_snapshot_copy(const __grid_constant__ SnapTable t) {
	__shared__ u64 first[NB_SNAP_SECTIONS + 1];   // first chunk of each section; first[n] = the total
	__shared__ u64 bytes[NB_SNAP_SECTIONS];
	if (threadIdx.x < 32) {   // lane i: sections 2i and 2i + 1
		const u32 i = threadIdx.x;
		const u64 b0 = snap_section_bytes(t, 2 * i), b1 = snap_section_bytes(t, 2 * i + 1), c1 = (b1 + 15) >> 4;
		u64 c = ((b0 + 15) >> 4) + c1;
		for (int d = 1; d < 32; d <<= 1) { const u64 y = __shfl_up_sync(0xffffffffu, c, d); if (i >= (u32)d) c += y; }
		bytes[2 * i] = b0; bytes[2 * i + 1] = b1; first[2 * i + 1] = c - c1; first[2 * i + 2] = c;
		if (i == 0) first[0] = 0;
	}
	__syncthreads();
	const u64 total = first[t.n];
	u32 sec = 0;
	for (u64 c = (u64)blockIdx.x * blockDim.x + threadIdx.x; c < total; c += (u64)gridDim.x * blockDim.x) {
		while (c >= first[sec + 1]) ++sec;   // a thread's chunks ascend
		const u64 k = c - first[sec], b = bytes[sec];
		const SnapSection& s = t.s[sec];
		if (16 * (k + 1) <= b) reinterpret_cast<uint4*>(s.dst)[k] = reinterpret_cast<const uint4*>(s.src)[k];
		else for (u64 j = 16 * k; j < b; ++j) static_cast<uint8_t*>(s.dst)[j] = static_cast<const uint8_t*>(s.src)[j];
	}
}

struct nb_snapshot {
	nb_context* ctx;
	bool saved;
	DevBuf<unsigned char> arena; std::vector<size_t> off;   // the fixed sections, by position in snapshot_sections; words = the count words
	u32* words;
	DevBuf<nb_constraint_row> rows;                  // user rows in device order
	DevBuf<uint4> overlaps;                          // the sensor overlap list
	DevBuf<nb_joint> joints; DevBuf<nb_constraint_row> jrows;   // the joint table and the joints' rows (the drives' appended rows included)
	DevBuf<JointDrive> drives;                                  // the joint drive table
	DevBuf<JointSpring> springs; DevBuf<nb_constraint_row> srows;   // the joint spring table and the spring rows
	// the host side at the save
	NbStateHeader h; StateShape shape; RowLevels urow_set; JointSet jset; DriveSet dset; KeyedSet sset;
	std::vector<nb_ccd_body> ccd;                    // the continuous-collision set (its rows are host values; k_ccd rewrites the factors)
};

// A snapshot section: the context's buffer, the snapshot's copy, and the counter word (>= 0) that holds the element count on the device.
struct SnapPart { void* ctx_ptr; void* snap_ptr; size_t size, count; bool present; int word; };

// The sections of a snapshot with header `h`: the state file's (a file keeps the kinematic indices on the host, the snapshot keeps them in
// its host side and the kind bytes), then the snapshot's own.  The fixed sections come first, the rows and the overlap list last.  With `s`
// null the snapshot pointers are offsets into the arena, and there are no rows or joints.
static std::vector<SnapPart> snapshot_sections(nb_context* ctx, const nb_snapshot* s, const NbStateHeader& h, u32 conn_probe) {
	const JointSet none, &js = s ? s->jset : none;
	const KeyedSet knone, &ds = s ? s->dset : knone, &ss = s ? s->sset : knone;
	const u32 nrows = s ? s->urow_set.n : 0;
	StateHostCopies hc;
	std::vector<SnapPart> p;
	auto at = [&](size_t i) -> void* { return s ? s->arena.p + s->off[i] : nullptr; };
	for (const StateSection& x : state_sections(ctx, h, hc, false))
		p.push_back({ x.dev, at(p.size()), x.size, x.count, x.present && x.dev != nullptr, x.word });
	p.push_back({ ctx->kind, at(p.size()), 1, h.bodies, h.reserved[4] != 0, -1 });
	p.push_back({ ctx->conn_keys, at(p.size()), 8, conn_probe, conn_probe != 0, -1 });
	for (int j = 0; j < 3; ++j) p.push_back({ ctx->counts + kSnapWords[j], s ? s->words + j : nullptr, 4, 1, true, -1 });
	p.push_back({ ctx->urows.p, s ? s->rows.p : nullptr, sizeof(nb_constraint_row), nrows, nrows != 0, -1 });
	p.push_back({ ctx->joints.p, s ? s->joints.p : nullptr, sizeof(nb_joint), js.n, js.n != 0, -1 });
	p.push_back({ ctx->jrows.p, s ? s->jrows.p : nullptr, sizeof(nb_constraint_row), (size_t)js.nrows + ds.nrows, js.n != 0, -1 });
	p.push_back({ ctx->drives.p, s ? s->drives.p : nullptr, sizeof(JointDrive), js.n, ds.n != 0, -1 });
	p.push_back({ ctx->springs.p, s ? s->springs.p : nullptr, sizeof(JointSpring), js.n, ss.n != 0, -1 });
	p.push_back({ ctx->srows.p, s ? s->srows.p : nullptr, sizeof(nb_constraint_row), ss.nrows, ss.n != 0, -1 });
	p.push_back({ ctx->sensor_old.p, s ? s->overlaps.p : nullptr, sizeof(uint4), h.reserved[3], h.reserved[2] != 0, CNT_SENSOR_OLD });
	return p;
}
static const size_t kSnapFixed = 20 + 2;   // the state file's 20 sections, the kind bytes and the key list: the sections in the arena

// The table of one copy.  save: context -> snapshot; restore: snapshot -> context, with the overlap list also copied to the current list
// and its length to the current count (nb_download_sensor_overlaps returns what it returned at the save).  A device count is read on the
// side the copy comes from.
static int snapshot_table(nb_context* ctx, const nb_snapshot* s, bool save, SnapTable& t) {
	const u32 probe = (s->shape.filter_flags & NB_FILTER_SKIP_CONNECTED) ? s->shape.nconn : 0;
	std::vector<SnapPart> parts = snapshot_sections(ctx, s, s->h, probe);
	if (!save && s->shape.has_sensor) {
		parts.push_back({ ctx->sensor_cur.p, s->overlaps.p, sizeof(uint4), s->h.reserved[3], true, CNT_SENSOR_OLD });
		parts.push_back({ ctx->counts + CNT_SENSOR_HITS, s->words + 2, 4, 1, true, -1 });
	}
	t.n = 0;
	for (const SnapPart& x : parts) {
		if (!x.present || !x.count) continue;   // a device count is at most `count`
		if (t.n == NB_SNAP_SECTIONS) { ctx->error = "snapshot: too many sections"; return NB_ERR_ARGUMENT; }
		SnapSection& d = t.s[t.n++];
		const u32* count_dev = nullptr;
		if (x.word >= 0) {
			int j = 0; while (kSnapWords[j] != x.word) ++j;
			count_dev = save ? ctx->counts + x.word : s->words + j;
		}
		d.src = save ? x.ctx_ptr : x.snap_ptr; d.dst = save ? x.snap_ptr : x.ctx_ptr;
		d.count_dev = count_dev; d.size = (u32)x.size; d.count = (u32)x.count;
	}
	return NB_OK;
}

static int snapshot_launch(nb_context* ctx, const SnapTable& t, cudaStream_t st) {
	size_t chunks = 0;   // an upper bound: device counts at their limits
	for (u32 i = 0; i < t.n; ++i) chunks += ((size_t)t.s[i].size * t.s[i].count + 15) / 16;
	launch_grid(mk_launch(ctx, st), k_snapshot_copy, GRID(std::max<size_t>(chunks, 1)), t);
	CK(cudaGetLastError());
	return NB_OK;
}

static void free_snapshots(nb_context* ctx) {
	for (nb_snapshot* s : ctx->snapshots) delete s;
	ctx->snapshots.clear();
}

#define SNAPSHOT_OF_CTX(snap, what) do { \
	if (!(snap) || (snap)->ctx != ctx) { ctx->error = what ": the snapshot belongs to another context"; return NB_ERR_ARGUMENT; } \
	if (ctx->sharded) { ctx->error = what ": not supported on a context of nb_shard_create"; return NB_ERR_ARGUMENT; } } while (0)

extern "C" {

int nb_snapshot_create(nb_context* ctx, nb_snapshot** out) {
	if (!out) { ctx->error = "nb_snapshot_create: null output"; return NB_ERR_ARGUMENT; }
	*out = nullptr;
	if (ctx->sharded) { ctx->error = "nb_snapshot_create: not supported on a context of nb_shard_create"; return NB_ERR_ARGUMENT; }
	const nb_config& c = ctx->cfg;
	NbStateHeader cap; memset(&cap, 0, sizeof(cap));   // every device section present, at the capacities
	cap.bodies = c.max_bodies; cap.boxes = c.max_boxes; cap.spheres = c.max_spheres; cap.connections = c.max_connections; cap.cache = c.max_contacts;
	cap.reserved[1] = cap.reserved[2] = cap.reserved[5] = 1;   // the kinematic indices stay on the host: no room
	nb_snapshot* s = new nb_snapshot();
	s->ctx = ctx;
	size_t bytes = 0;
	const std::vector<SnapPart> parts = snapshot_sections(ctx, nullptr, cap, c.max_connections);
	for (size_t i = 0; i < kSnapFixed; ++i) { s->off.push_back(bytes); bytes += (parts[i].size * parts[i].count + 15) & ~(size_t)15; }
	if (int r = s->arena.alloc(ctx, bytes + 16)) { delete s; ctx->error = "nb_snapshot_create: " + ctx->error; return r; }
	s->words = reinterpret_cast<u32*>(s->arena.p + bytes);
	ctx->snapshots.push_back(s);
	*out = s;
	return NB_OK;
}

void nb_snapshot_destroy(nb_snapshot* s) {
	if (!s) return;
	nb_context* ctx = s->ctx;
	ctx->snapshots.erase(std::remove(ctx->snapshots.begin(), ctx->snapshots.end(), s), ctx->snapshots.end());
	delete s;   // cudaFree waits for the work that may still read it
}

int nb_snapshot_save(nb_context* ctx, nb_snapshot* s, void* stream) {
	NB_RANGE("nb_snapshot_save");
	SNAPSHOT_OF_CTX(s, "nb_snapshot_save");
	if (ctx->in_step && !ctx->scene_edited) { ctx->error = "nb_snapshot_save: between nb_collide and the nb_advance that ends its step"; return NB_ERR_ARGUMENT; }
	cudaStream_t st = (cudaStream_t)stream;
	JOIN_UPLOADS();   // the copy reads the momentum and property rows
	// grown: the only save that synchronises and allocates
	GROW(s->rows, ctx->urow_set.n, st); GROW(s->overlaps, ctx->has_sensor ? ctx->sensor_cap : 0, st);
	GROW(s->joints, ctx->jset.n, st); GROW(s->jrows, (size_t)ctx->jset.nrows + ctx->dset.nrows, st); GROW(s->drives, ctx->dset.n ? ctx->jset.n : 0, st);
	GROW(s->springs, ctx->sset.n ? ctx->jset.n : 0, st); GROW(s->srows, ctx->sset.nrows, st);
	s->h = state_header_of(ctx, ctx->cfg.max_contacts);   // the device count decides how many cache entries are copied
	s->shape = state_shape_of(ctx);
	s->urow_set = ctx->urow_set; s->jset = ctx->jset; s->dset = ctx->dset; s->sset = ctx->sset; s->ccd = ctx->ccd;
	SnapTable t;
	{ int r = snapshot_table(ctx, s, true, t); if (r) return r; }
	{ int r = snapshot_launch(ctx, t, st); if (r) return r; }
	s->saved = true;
	return NB_OK;
}

int nb_snapshot_restore(nb_context* ctx, const nb_snapshot* s, void* stream) {
	NB_RANGE("nb_snapshot_restore");
	ctx->report_ok = false;
	SNAPSHOT_OF_CTX(s, "nb_snapshot_restore");
	if (!s->saved) { ctx->error = "nb_snapshot_restore: the snapshot was never saved"; return NB_ERR_ARGUMENT; }
	cudaStream_t st = (cudaStream_t)stream;
	JOIN_UPLOADS();   // a pending side copy must not land on the restored rows
	// tables the context has never had, or has too small: created or grown here (the only restore that synchronises and allocates)
	if (s->shape.has_frc) { ALLOC(ctx->frc, ctx->cfg.max_bodies); ALLOC(ctx->frc_spare, ctx->cfg.max_bodies); }
	if (!s->shape.kin.empty()) ALLOC(ctx->kind, ctx->cfg.max_bodies);
	GROW(ctx->urows, s->urow_set.n, st);
	const void* joint_bufs[5] = { ctx->joints.p, ctx->jrows.p, ctx->drives.p, ctx->springs.p, ctx->srows.p };
	GROW(ctx->joints, s->jset.n, st); GROW(ctx->jrows, (size_t)s->jset.nrows + s->dset.nrows, st); GROW(ctx->drives, s->dset.n ? s->jset.n : 0, st);
	GROW(ctx->springs, s->sset.n ? s->jset.n : 0, st); GROW(ctx->srows, s->sset.nrows, st);
	if (s->shape.has_sensor) { int r = ensure_sensor_lists(ctx, s->shape.sensor_cap, st); if (r) return r; }
	SnapTable t;
	{ int r = snapshot_table(ctx, s, false, t); if (r) return r; }
	{ int r = snapshot_launch(ctx, t, st); if (r) return r; }
	StateShape shape = s->shape;
	{ int r = install_state(ctx, shape, nullptr, st); if (r) return r; }
	// the row and joint levels are host values in the graph, the joint buffers its kernel arguments
	if (s->urow_set.n != ctx->urow_set.n || s->urow_set.level_off != ctx->urow_set.level_off) ++ctx->graph_epoch;
	if (s->jset.structure != ctx->jset.structure || joint_bufs[0] != ctx->joints.p || joint_bufs[1] != ctx->jrows.p) ++ctx->graph_epoch;
	else if (s->dset.structure != ctx->dset.structure || joint_bufs[2] != ctx->drives.p) ++ctx->graph_epoch;
	else if (s->sset.structure != ctx->sset.structure || joint_bufs[3] != ctx->springs.p || joint_bufs[4] != ctx->srows.p) ++ctx->graph_epoch;
	ctx->urow_set = s->urow_set; ctx->jset = s->jset; ctx->dset = s->dset; ctx->sset = s->sset;
	{ int r = set_ccd(ctx, s->ccd, st); if (r) return r; }   // nothing when the context holds the same set
	ctx->scene_edited = true;   // the last collide's outputs belong to another state
	ctx->in_step = false;
	return NB_OK;
}

}  // extern "C"
