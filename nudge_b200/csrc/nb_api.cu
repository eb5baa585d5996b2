// nudge_b200 — host side of the C ABI (include/nudge_b200.h): context, HBM arena, kernel sequencing.
// The reference keeps all memory caller-owned and bump-allocates scratch from an Arena (nudge.cpp:990-1055);
// here the context plays both roles for device memory: the step's buffers are allocated at nb_create and reused every step, nothing is
// allocated or synchronised inside the step; a feature allocates its tables on its first call.  Every buffer is a DevBuf held by its
// owner (the context, a shard or a snapshot), which frees it and counts its bytes.
#include "nb_shard.cuh"
#include "nb_events.cuh"
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <algorithm>
#include <memory>
#include <math.h>
#include <nvtx3/nvToolsExt.h>

extern "C" void nb_host_sample_luts(u32* rcp_lut, u32* rsqrt_lut);   // nb_lut_host.cpp
extern "C" int nb_host_check_lut_model(const u32* rcp_lut, const u32* rsqrt_lut);

// A sub-step as a CUDA graph (nb_step, nb_shard_step; run_graphed): captured once per key and replayed while the key holds.  Every
// count the kernels need lives in device memory, so the graph only depends on the parameters and the scene shape held in the key.
struct StepKey { cudaStream_t stream; float ts, gravity, damping; u32 iterations, B, nboxes, nspheres, nconn, tagbits, kbits; int debug, solver_mode, transport; unsigned long long plan_version, graph_epoch; };
struct StepGraph { cudaGraphExec_t exec; StepKey key; unsigned long long launches; int enabled; };

// A device buffer of `cap` elements, freed with its owner, its bytes charged to `charged` (the context's device_bytes) while it holds
// them.  Move-only: the move swaps, so the buffer it replaces is freed and uncharged with the temporary.
template<class T> struct DevBuf {
	T* p = nullptr; size_t cap = 0; unsigned long long* charged = nullptr;
	DevBuf() = default; DevBuf(DevBuf&& o) noexcept { *this = std::move(o); }
	DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); std::swap(charged, o.charged); return *this; }
	~DevBuf() { if (p) { cudaFree(p); *charged -= cap * sizeof(T); } }
	int alloc(nb_context* ctx, size_t n);   // below nb_context
};

// Entries levelled by body (level_rows, nb_rows_api.cuh), the user rows or the joints: each one's (a, b) in upload order and device position
// (by level, upload order within one), and the levels' offsets (levels + 1, none without entries), host values in nb_step's graph.
struct RowLevels { u32 n = 0, levels = 0; std::vector<u32> level_off, order; std::vector<nb_body_pair> ab; };

// The shape of a joint set (joint_shape, nb_joint_api.cuh), what the drive and spring checks read: per joint in upload order its (type, a,
// b), and whether its rel_rotation / axis_a has unit length, as a drive or spring that reads them needs.
struct JointShape { std::vector<u32> structure; std::vector<uint8_t> unit_rel, unit_axis; };
// The host side of a joint set (nb_joint_api.cuh): its levels (the device table holds the joints by level), its shape, and the number of
// rows the joints generate.
struct JointSet : RowLevels, JointShape { u32 nrows = 0; };

// One joint's drive on the device (nb_joint_api.cuh; DESIGN.md section 8.17): one entry per joint in table order while a drive set exists,
// flags = 0 for a joint without a drive.  row = the first of its rows in the drive rows; (sl, cl) / (su, cu) = the hinge or twist limits'
// half-angle pairs; a CONE drive (section 8.20) keeps its half-angle pair (sc, cc) in motor_speed / max_motor_torque and the uploaded half-angle in
// cone (0 otherwise).  position = (sh, ch) of a hinge, (dist, 0) or (s, 0) of a slider, the twist's pair or the swing's (ss, cs), as of the
// last row build.  nb_debug_read("joint_drives") returns the table as it stands.
struct JointDrive {
	u32 flags, row; float lower, upper, sl, cl, su, cu;
	float motor_speed, max_motor_torque, break_force, break_torque, position[2]; u32 broken; float cone;
};
// The host side of a sparse table keyed by joint (the drives, the springs): the entry count, the entries' rows and per entry in joint order
// the structure nb_step's graph depends on: (joint, flags) of a drive, the joint of a spring.
struct KeyedSet { u32 n = 0, nrows = 0; std::vector<u32> structure; };
// A sparse table keyed by joint: the device table (one entry per joint in table order while set.n), its rows (each entry's row is an
// offset into them) and the host side.
template<class E> struct KeyedTable { DevBuf<E> table; DevBuf<nb_constraint_row> rows; KeyedSet set; };
// One joint's spring on the device (nb_upload_joint_springs, nb_joint_api.cuh; DESIGN.md section 8.21): one entry per joint in table order
// while a spring set exists, present = 0 for a joint without a spring.  row = its first spring row; target = the uploaded words, for a HINGE
// (st, ct) = (sin, cos) of target / 2 with the uploaded angle in `angle`; position = (sh, ch) of a hinge, (s, 0), (dist, 0), or (|d.xyz|,
// d.w) of a BALL, as of the last row build.  nb_debug_read("joint_springs") returns the table as it stands.
struct JointSpring {
	u32 present, row; float target[4];
	float target_velocity, stiffness, damping, max_force, position[2], angle; u32 reserved[3];
};
static_assert(sizeof(JointSpring) == 64, "JointSpring is 64 bytes");

// The buffers of nb_collide's front end (launch_front_end); leaf_* = the AABBs in Morton order, keybits = the OR and AND of the Morton codes.
// The context has one, the scene queries their own (nb_query_api.cuh), so that a query never touches what the step reads.
struct FrontEnd {
	nb_transform* world_xf; float4* aabb_min; float4* aabb_max; u32* col_tag; u32* col_body; u32* order; u32* rank;
	float4* leaf_min; float4* leaf_max; u64* mkeys; uint8_t* smallf; u32* large_list; u64* table_keys; u64* table_vals; u32 table_mask; u64* keybits;
};

// The scene queries' scratch (nb_query_api.cuh), shared by nb_raycast, nb_overlap and nb_shapecast: the front end, its sort buffers and
// counters, allocated on the first query for the collider capacity; rays / casts / hits = the staging of a ray or shape cast call with host
// pointers.  The overlap call's hit keys and their sort (osb points into okeys, with sb's histogram and grid barrier) hold the largest
// capacity a call asked for; oq / oh / ooff = the staging of an overlap call with host pointers.
struct QueryScratch {
	FrontEnd front; SortBuffers sb; u32* counts; DevBuf<nb_ray> rays; DevBuf<nb_shape_cast> casts; DevBuf<nb_ray_hit> hits; bool ready;
	DevBuf<u64> okeys[2]; SortBuffers osb; DevBuf<nb_overlap_query> oq; DevBuf<nb_overlap_hit> oh; DevBuf<u32> ooff;
};
// The slots of QueryScratch::counts the queries keep for themselves, in slots of nb_collide's counters the front end has no other use for.
// The fallbacks (queries that tested every collider instead of walking the grid, read by nb_debug_read) are summed over the context's
// calls, so none may be a slot launch_front_end writes or resets.  The overlap call's append cursor of its hit keys (nb_radix_sort lowers it
// to the capacity) and its total of hits (never lowered) start each call from k_reset_collide's zero.
enum {
	CNT_RAY_FALLBACKS = CNT_TMP, CNT_OVERLAP_FALLBACKS = CNT_SURV, CNT_SHAPECAST_FALLBACKS = CNT_SENSOR_TMP + 1,
	CNT_OVERLAP_KEYS = CNT_PAIRS, CNT_OVERLAP_TOTAL = CNT_SENSOR_PAIRS
};
// The step's counter slot of k_ccd's fallbacks (continuous collision, nb_ccd_api.cuh): summed over the context's advances, in a slot after
// the scheduler's fall-back flags that nothing else writes.
enum { CNT_CCD_FALLBACKS = CNT_SCHED_FB0 + 16 };
static_assert((int)CNT_CCD_FALLBACKS < (int)CNT_EXT_HIST, "the fallback slot lies between the scheduler's flags and the extent histogram");

struct nb_context {
	nb_config cfg;
	int sms;
	std::string error;
	unsigned long long launches;
	int lut_exact;
	// device_bytes: what the DevBufs charged to it hold, the context's, its shard's and its snapshots' (nb_debug_read); declared before
	// every buffer, which uncharges it when destroyed.  allocs: the context's buffers of alloc_zeroed.
	unsigned long long device_bytes; std::vector<DevBuf<unsigned char>> allocs;
	// the editing calls' shared host side: the staging copy of a caller's array (put_staged) and the duplicate check's byte per body, all
	// zeros between calls (bodies_distinct)
	std::vector<unsigned char> host_stage; std::vector<uint8_t> body_seen;
	u32 B, nboxes, nspheres, nconn;  // uploaded sizes
	u32 tagbits, kbits, bodybits;
	u32 stride;    // scratch stride
	u32 cstride;   // row plane stride
	u32 slots_per_bucket;
	int coop_blocks_solve;
	StepGraph graph; bool capturing;  // nb_step's graph; capturing: run_graphed is recording a step of this context
	unsigned long long graph_epoch;   // in the graphs' key: bumped by every change of which kernels a step launches or of their arguments
	u32* chain_start; u32* chain_len;  // per body: segment cursor (the segment's end once k_chain_scatter ran) / number of chain entries
	float4* warm;   // two rows per chain entry: the warm start's share of the entry's side (k_build_rows -> k_warm_start)
	bool contacts_internal;  // the current contact set came from nb_collide (not nb_upload_contacts)
	u32 upload_tagbits;      // bits of the largest A or B among the contacts nb_upload_contacts put in place (any uint32, not only collider tags)
	// throughput mode (nb_set_solver_mode): mass-splitting Jacobi, nb_jacobi.cuh
	int solver_mode; u32* jcnt; float4* jd; int jacobi_blocks1, jacobi_blocks2;
	// CUDA-event timing of the dominant solver kernel (nb_debug_timing): bench.py's roofline numerator is measured live
	int timing; cudaEvent_t tev[2][64]; int tev_n; bool tev_made;
	// user constraint rows (nb_upload_constraint_rows, nb_rows_api.cuh)
	float4* instances;   // nb_instance_matrices with a host destination (allocated on first use)
	// nb_upload_bodies sends what the collision stage does not read (momentum, properties) on a second stream, so that copy runs under
	// `collide`; the first consumer waits for ev_up_done (inside a captured step: an external event-wait node, re-armed by every upload)
	cudaStream_t copy_stream; cudaEvent_t ev_up_begin, ev_up_done; bool upload_pending, capture_joined; int copy_overlap;
	DevBuf<nb_constraint_row> urows; RowLevels urow_set;
	// contact events (nb_enable_contact_events, nb_events.cuh): ev_cap = 0 is off; the buffer is kept while it holds ev_cap events
	DevBuf<nb_contact_event> events; u32 ev_cap;
	// collision filters (nb_upload_collision_filters): one category | mask << 16 word per collider while has_filter; with
	// NB_FILTER_SKIP_CONNECTED and connections, conn_keys holds the sorted connection keys and conn_probe = their count (else 0)
	u32* filter; bool has_filter; u32 filter_flags; u64* conn_keys; u64* conn_scratch; u32* conn_sort_n; u32 conn_probe;
	// sensor colliders (nb_upload_sensors, DESIGN.md section 8.7): one 0/1 byte per collider while has_sensor; sensor_cap = candidate sensor
	// pairs per collide.  The candidate keys, the sort buffers (sensor_sb points into sensor_sort_keys / _vals) and the current / old overlap
	// lists are kept while they hold sensor_cap entries.
	uint8_t* sensor; bool has_sensor; u32 sensor_cap; DevBuf<u64> sensor_keys, sensor_sort_keys[2]; DevBuf<u32> sensor_sort_vals[2]; SortBuffers sensor_sb;
	DevBuf<uint4> sensor_cur, sensor_old;
	// kinematic bodies (nb_upload_kinematic_bodies, DESIGN.md section 8.8): kind[body] as in nb_collide.cuh (bit 0 kinematic, bit 1 moving),
	// allocated for max_bodies on the first upload of a set; kin_list = the set (host copy, ascending); kin_rows = the scatter's staging rows
	uint8_t* kind; bool has_kin; std::vector<u32> kin_list; DevBuf<nb_kinematic_body> kin_rows;
	// body impulses (nb_apply_body_impulses, DESIGN.md section 8.9): the call's own staging rows and sort keys (imp_sb points into imp_keys),
	// and its sort histogram, grid barrier and key count; none of it is shared with the step
	DevBuf<nb_body_impulse> imp_rows; DevBuf<u64> imp_keys[2]; SortBuffers imp_sb; u32* imp_n;
	// spawning (nb_add_bodies, nb_remove_bodies, DESIGN.md section 8.10): scene_edited refuses the stage calls that read the last collide's
	// outputs until the next collide; sharded = nb_shard_create was called on this context (edits are refused); spawn_idx / urows_spare =
	// the removal's index staging and row gather buffers; conn_host = the connections as uploaded or loaded, for the removal's index checks
	bool scene_edited, sharded; std::vector<nb_body_pair> conn_host; DevBuf<u32> spawn_idx; DevBuf<nb_constraint_row> urows_spare;
	// per-body forces (nb_set_body_forces, DESIGN.md section 8.11): frc = one entry per body while has_frc, allocated for max_bodies on the
	// first call, together with frc_spare (nb_remove_bodies gathers into it); frc_rows = the scatter's staging rows
	nb_body_force* frc; nb_body_force* frc_spare; bool has_frc; DevBuf<nb_body_force> frc_rows;
	// snapshots (nb_snapshot_save / nb_snapshot_restore, DESIGN.md section 8.12): in_step = between nb_collide and the nb_advance that ends its
	// step, where a save is refused; the context's snapshots, freed by nb_destroy; graph_records = captures of a step graph (nb_debug_read)
	bool in_step; std::vector<nb_snapshot*> snapshots; unsigned long long graph_records;
	// joints (nb_upload_joints, DESIGN.md section 8.13): the table by level, the rows k_joint_rows rebuilds every step around their accumulated
	// impulses, and the host side; step_dt = the time step of the nb_apply_gravity_damping since the last nb_collide (0: none yet)
	DevBuf<nb_joint> joints; DevBuf<nb_constraint_row> jrows; JointSet jset; float step_dt;
	// joint drives (nb_upload_joint_drives, DESIGN.md section 8.17) and joint springs (nb_upload_joint_springs, section 8.21)
	KeyedTable<JointDrive> drives; KeyedTable<JointSpring> springs;
	// continuous collision (nb_upload_ccd_bodies, DESIGN.md section 8.18, nb_ccd_api.cuh): ccd = the set (host copy, ascending by body) and
	// ccd_rows its device copy; ccd_t = the advance's translation factor per body (max_bodies of them, 1 outside the set), allocated on the
	// first upload; ccd_hits = (bits of t, collider) per entry of the last advance
	std::vector<nb_ccd_body> ccd; DevBuf<nb_ccd_body> ccd_rows; float* ccd_t; DevBuf<uint2> ccd_hits;
	// body states (nb_get_body_states, nb_set_body_states, DESIGN.md section 8.19, nb_body_state_api.cuh): a host-pointer call's staging (rows in
	// and out, the gather's indices), and the set's sort keys (bs_sb points into bs_keys) with its own histogram, grid barrier and key count
	DevBuf<nb_body_state> bs_rows; DevBuf<u32> bs_idx; DevBuf<u64> bs_keys[2]; SortBuffers bs_sb; u32* bs_n;
	// contact impulse reports (nb_get_body_contact_impulses, nb_get_contact_pair_impulses, DESIGN.md section 8.22, nb_contact_report_api.cuh):
	// report_ok = the contact set, its order, its impulses and its rows are those of a solved step (set by nb_update_cached_impulses and
	// nb_step, cleared by the calls that rewrite them or renumber bodies).  The per-body call's key count, sort buffers (2 keys per contact
	// of capacity, cr_sb's own histogram and grid barrier) and host-pointer staging; the pair call's run and kept counts, flags, per-run
	// rows, scan sums and host-pointer staging.
	bool report_ok; u32* cr_n; SortBuffers cr_sb; DevBuf<nb_body_contact_impulse> cr_rows; DevBuf<u32> cr_idx;
	u32* cp_n; u32* cp_heads; u32* cp_kept; nb_contact_pair_impulse* cp_rows; u32* cp_block_sums; DevBuf<nb_contact_pair_impulse> cp_out;
	// scene queries: ray casts (nb_raycast, DESIGN.md section 8.14), overlap queries (nb_overlap, section 8.15) and shape casts
	// (nb_shapecast, section 8.16)
	QueryScratch query;

	// scene
	nb_transform* xf; nb_body_properties* props; nb_body_momentum* mom; uint8_t* idle;
	u32* box_tags; nb_box_collider* box_data; nb_transform* box_xf;
	u32* sph_tags; nb_sphere_collider* sph_data; nb_transform* sph_xf;
	nb_body_pair* conn;
	u32* counts;
	// collide
	FrontEnd front;
	SortBuffers sb; u32 sort_cap;
	u64* pair_keys;  // alias into sb.keys[] after the pair sort
	u64* pair_keys_debug;  // copy kept for parity tests when debug is enabled (the sort buffers are reused later in the step)
	int debug;
	u32* flags; u32* offs; u32* block_sums;
	uint2* live; float* np_pen; u32* np_info; u32* np_list; u32* np_start;
	ContactOut staged, fin;
	u64* sleeping;
	u32* parent; u32* active; u32* active_idx; u32* taint;
	// cache
	u64* cache_tags; u32* cache_features; float4* cache_data;
	u64* culled_tags; u32* culled_features; float4* culled_data;
	u32* sorted; float4* impulses;
	// setup / solve
	float4* inertia;
	u32* sched_spill_ent; u32* sched_spill_uid; u32 sched_spill_cap;   // k_schedule's open-slot list beyond its on-chip positions
	u32* slot_of; u32* slot_done; u32* slot_left; u32* left_count; u32* batch_of; u32* slot_idx; float4* mw; uint2* cab; uint8_t* back;
	// the segmented scheduler replay (nb_solver.cuh above k_schedule): per speculative run its slots, "list empty after contact i"
	// and end state; per segment the run picked by the join
	u32* sched_slot_v; uint8_t* sched_empty; u32* sched_state; u32* sched_join_slot; uint2* sched_pick; uint2* sched_pick_res;
	Rows rows;
};

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { ctx->error = std::string(#call) + ": " + cudaGetErrorString(e_); return NB_ERR_CUDA; } } while (0)

// Frees the buffer, then allocates n elements charged to the context's device_bytes.  On failure the buffer is empty, and the error, which
// does not stick, is cleared, so that no later cudaGetLastError check reports it again.
template<class T> int DevBuf<T>::alloc(nb_context* ctx, size_t n) {
	*this = DevBuf();
	const cudaError_t e = cudaMalloc(&p, n * sizeof(T));
	if (e != cudaSuccess) { p = nullptr; cudaGetLastError(); ctx->error = std::string("cudaMalloc: ") + cudaGetErrorString(e); return NB_ERR_CUDA; }
	cap = n; charged = &ctx->device_bytes; *charged += n * sizeof(T);
	return NB_OK;
}

// The allocator of the buffers kept for their owner's lifetime: unless `p` exists already, n elements (at least one), zero-filled, held
// by `list`, the owner's (the context's allocs or a shard's).  A routine that allocates several can run again and allocate the rest.
template<class T>
static int alloc_zeroed(nb_context* ctx, std::vector<DevBuf<unsigned char>>& list, T*& p, size_t n) {
	if (p) return NB_OK;
	DevBuf<unsigned char> b;
	if (int r = b.alloc(ctx, (n ? n : 1) * sizeof(T))) return r;
	// Zeroed before the first use, which may come on a non-blocking stream that the legacy stream does not order against: a buffer
	// allocated on first use (the body-force table, the kinematic table, ...) would otherwise be cleared AFTER the kernels that fill it
	// when the legacy stream still holds other work (another context's step).
	cudaError_t e = cudaMemsetAsync(b.p, 0, b.cap, cudaStreamLegacy);
	if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);
	if (e != cudaSuccess) { ctx->error = std::string("cudaMemset: ") + cudaGetErrorString(e); return NB_ERR_CUDA; }
	p = reinterpret_cast<T*>(b.p);
	list.push_back(std::move(b));
	return NB_OK;
}
#define ALLOC_IN(list, p, n) do { int r_ = alloc_zeroed(ctx, list, p, (size_t)(n)); if (r_) return r_; } while (0)
#define ALLOC(p, n) ALLOC_IN(ctx->allocs, p, n)

// Makes `b` hold at least n elements.  A larger buffer replaces the old one once `st` has drained, since earlier work on it may still read
// the old one; the contents are neither kept nor cleared.  On failure the buffer is empty.
template<class T>
static int grow(nb_context* ctx, DevBuf<T>& b, size_t n, cudaStream_t st) {
	if (n <= b.cap) return NB_OK;
	CK(cudaStreamSynchronize(st));
	return b.alloc(ctx, n);
}
#define GROW(b, n, st) do { int r_ = grow(ctx, b, (size_t)(n), st); if (r_) return r_; } while (0)

// The host staging of the editing calls: enqueues the copy of `bytes` from the caller's `src` to `dst` on `st` through the context's pageable
// staging vector, which a pageable cudaMemcpyAsync has consumed when it returns, so the caller's array may be reused on return, pinned or not.
// `edit`, when given, rewrites the staged bytes first.
static cudaError_t put_staged(nb_context* ctx, void* dst, const void* src, size_t bytes, cudaStream_t st, void (*edit)(unsigned char*, size_t) = nullptr) {
	if (!bytes) return cudaSuccess;
	ctx->host_stage.assign((const unsigned char*)src, (const unsigned char*)src + bytes);
	if (edit) edit(ctx->host_stage.data(), bytes);
	return cudaMemcpyAsync(dst, ctx->host_stage.data(), bytes, cudaMemcpyHostToDevice, st);
}

static u32 bits_for(u64 n) { u32 b = 1; while (((u64)1 << b) < n) ++b; return b; }
static Launch mk_launch(nb_context* ctx, void* stream) { Launch L = { (cudaStream_t)stream, &ctx->launches, ctx->sms }; return L; }
#define GRID(n) nb_grid_for((unsigned)(n), ctx->sms)
// NVTX range per API call (SURVEY.md section 5): visible in Nsight timelines, a no-op costing tens of nanoseconds without a tool attached
struct NbRange { NbRange(const char* name) { nvtxRangePushA(name); } ~NbRange() { nvtxRangePop(); } };
#define NB_RANGE(name) NbRange nb_range_(name)
static int launch_user_rows(nb_context* ctx, int warm, cudaStream_t st);   // nb_rows_api.cuh
static int launch_joints(nb_context* ctx, const float* dt, cudaStream_t st);   // nb_joint_api.cuh
static void drop_joints(nb_context* ctx);
static void free_snapshots(nb_context* ctx);                               // nb_snapshot_api.cuh
static int set_ccd(nb_context* ctx, std::vector<nb_ccd_body> set, cudaStream_t st);   // nb_ccd_api.cuh
static int launch_ccd(nb_context* ctx, const Launch& L, float time_step);
static const char* ccd_body_problem(const nb_ccd_body& e);
// The stage calls that read the last nb_collide's outputs: refused after nb_add_bodies / nb_remove_bodies until the next collide
#define NOT_AFTER_EDIT() do { if (ctx->scene_edited) { ctx->error = "the scene was edited (nb_add_bodies / nb_remove_bodies) since the last nb_collide"; return NB_ERR_ARGUMENT; } } while (0)

__global__ void k_reset_collide(u32* counts, u32 K, u64* keybits) {
	if (threadIdx.x == 0) {
		keybits[0] = 0; keybits[1] = ~(u64)0;
		counts[CNT_SCRATCH1] = K;  // key count of the Morton sort
		counts[CNT_PAIRS] = 0; counts[CNT_OVERFLOW] = 0; counts[CNT_EXT_SUM] = 0;
		counts[CNT_SENSOR_PAIRS] = 0; counts[CNT_SENSOR_HITS] = 0; counts[CNT_SENSOR_TMP] = 0;
		for (int k = 0; k < 18; ++k) counts[CNT_EXT_HIST + k] = 0;
		for (int k = 0; k < 4; ++k) { counts[CNT_BMIN0 + k] = 0xffffffffu; counts[CNT_BMAX0 + k] = 0; }
	}
}

// The buffers of `f` for K colliders of capacity.
static int alloc_front_end(nb_context* ctx, FrontEnd& f, u32 K) {
	u32 tsz = 1024; while (tsz < 2 * K) tsz *= 2;
	f.table_mask = tsz - 1;
	ALLOC(f.keybits, 2); ALLOC(f.world_xf, K); ALLOC(f.aabb_min, K); ALLOC(f.aabb_max, K); ALLOC(f.col_tag, K); ALLOC(f.col_body, K);
	ALLOC(f.order, K); ALLOC(f.rank, K); ALLOC(f.leaf_min, K); ALLOC(f.leaf_max, K); ALLOC(f.mkeys, K); ALLOC(f.smallf, K);
	ALLOC(f.large_list, K); ALLOC(f.table_keys, tsz); ALLOC(f.table_vals, tsz);
	return NB_OK;
}

// nb_collide's front end on `f`, with its counters in `counts` and the Morton sort on `sb`: the counters' reset, then, with colliders and
// bodies, the world transforms and AABBs (with the filter, kinematic and sensor tables given; null: none), the Morton codes and their sort,
// the leaves in Morton order and the grid table.
static int launch_front_end(nb_context* ctx, const Launch& L, const FrontEnd& f, const SortBuffers& sb, u32* counts, const u32* filter,
							const uint8_t* kind, const uint8_t* sensor) {
	const u32 K = ctx->nboxes + ctx->nspheres;
	launch(L, k_reset_collide, 1, 32, 0, counts, K, f.keybits);
	if (K == 0 || ctx->B == 0) return NB_OK;
	launch_grid(L, k_collider_world, GRID(K), ctx->nboxes, ctx->nspheres, ctx->xf, ctx->box_xf, ctx->box_data, ctx->box_tags,
		ctx->sph_xf, ctx->sph_data, ctx->sph_tags, filter, kind, sensor, f.world_xf, f.aabb_min, f.aabb_max, f.col_tag, f.col_body, counts);
	launch_grid(L, k_morton, GRID(K), K, f.aabb_min, f.aabb_max, counts, sb.keys[0], sb.vals[0], f.keybits);
	// radix sort on the 48-bit code; ties keep index order like the stable sort of nudge.cpp:3165
	const int cur = nb_radix_sort(L, sb, counts + CNT_SCRATCH1, 0, 48, true, 0, 0, 0, f.keybits);
	launch_grid(L, k_leaves, GRID(K), K, sb.vals[cur], sb.keys[cur], f.aabb_min, f.aabb_max, f.order, f.rank, f.leaf_min, f.leaf_max, f.mkeys, counts);
	CK(cudaMemsetAsync(f.table_keys, 0xff, sizeof(u64) * ((size_t)f.table_mask + 1), L.stream));
	launch_grid(L, k_grid_build, GRID(K), K, f.order, f.leaf_min, f.leaf_max, f.mkeys, f.smallf, f.large_list, f.table_keys, f.table_vals, f.table_mask, counts);
	return NB_OK;
}

__global__ void __launch_bounds__(NB_BLOCK) k_copy_u64(const u64* src, u64* dst, const u32* n_ptr) {
	u32 n = *n_ptr;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = src[i];
}
__global__ void __launch_bounds__(NB_BLOCK) k_copy_u32(const u32* src, u32* dst, const u32* n_ptr) {
	u32 n = *n_ptr;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = src[i];
}
__global__ void __launch_bounds__(NB_BLOCK) k_debug_rcp(const float* x, float* y, u32 n, int rsq) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) y[i] = rsq ? nb_rsqrt(x[i]) : nb_rcp(x[i]);
}

// Ghost exchange for a scene sharded across GPUs (SURVEY.md §8e, K16): gather / scatter whole 32-byte BodyMomentum rows.
__global__ void __launch_bounds__(NB_BLOCK) k_pack_rows(const float4* rows, const u32* idx, u32 n, float4* out) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < 2 * n; i += gridDim.x * blockDim.x) out[i] = rows[2 * idx[i >> 1] + (i & 1)];
}
__global__ void __launch_bounds__(NB_BLOCK) k_unpack_rows(float4* rows, const u32* idx, const u32* src, u32 n, const float4* in) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < 2 * n; i += gridDim.x * blockDim.x) rows[2 * idx[i >> 1] + (i & 1)] = in[2 * src[i >> 1] + (i & 1)];
}

// Called by everything that touches momentum or properties on `st`: orders it after a pending nb_upload_bodies side copy.
static int join_uploads(nb_context* ctx, cudaStream_t st) {
	if (ctx->capturing) {   // in a captured step: one event-wait node that, at every replay, waits for the most recent upload's copy
		if (ctx->copy_stream && !ctx->capture_joined) { CK(cudaStreamWaitEvent(st, ctx->ev_up_done, cudaEventWaitExternal)); ctx->capture_joined = true; }
		return NB_OK;
	}
	if (ctx->upload_pending) { CK(cudaStreamWaitEvent(st, ctx->ev_up_done, 0)); ctx->upload_pending = false; }
	return NB_OK;
}
#define JOIN_UPLOADS() do { int r_ = join_uploads(ctx, (cudaStream_t)stream); if (r_) return r_; } while (0)

// The kinematic table as the kernels take it: null without a set, so that they load nothing extra.
static const uint8_t* kin_table(const nb_context* ctx) { return ctx->has_kin ? ctx->kind : nullptr; }
static void drop_kinematic(nb_context* ctx) { if (ctx->has_kin) { ctx->has_kin = false; ctx->kin_list.clear(); ++ctx->graph_epoch; } }
static void drop_body_forces(nb_context* ctx) { if (ctx->has_frc) { ctx->has_frc = false; ++ctx->graph_epoch; } }   // the step launches k_gravity_damping again
static void drop_ccd(nb_context* ctx) { if (!ctx->ccd.empty()) { ctx->ccd.clear(); ++ctx->graph_epoch; } }   // the step launches k_advance<false> again

// The checks of entry i of a body list (kinematic bodies, impulses, forces, removals): not body 0, the static world; below the body count;
// and, unless kinematic_ok, not kinematic.  A refused entry is NB_ERR_ARGUMENT with the message "<list> <i>: body <b> ...".
static int check_body(nb_context* ctx, const char* list, u32 i, u32 b, bool kinematic_ok) {
	std::string why;
	if (b == 0) why = "is the static world";
	else if (b >= ctx->B) why = "is at or beyond the body count (" + std::to_string(ctx->B) + ")";
	else if (!kinematic_ok && ctx->has_kin && std::binary_search(ctx->kin_list.begin(), ctx->kin_list.end(), b))
		why = "is kinematic (its velocity is set with nb_upload_kinematic_bodies)";
	else return NB_OK;
	ctx->error = std::string(list) + " " + std::to_string(i) + ": body " + std::to_string(b) + " " + why;
	return NB_ERR_ARGUMENT;
}
// The duplicate check of a body list whose entries (body(i), each checked by check_body) may name a body once: one mark per body in
// body_seen, which is all zeros between calls (O(n), where a sort of 65,536 entries costs ms).
template<class Body>
static int bodies_distinct(nb_context* ctx, const char* list, u32 n, Body body) {
	ctx->body_seen.resize(std::max<size_t>(ctx->body_seen.size(), ctx->B), 0);
	u32 twice = n;
	for (u32 i = 0; i < n && twice == n; ++i) if (ctx->body_seen[body(i)]++) twice = i;
	for (u32 i = 0; i < n; ++i) ctx->body_seen[body(i)] = 0;
	if (twice == n) return NB_OK;
	ctx->error = std::string(list) + " " + std::to_string(twice) + ": body " + std::to_string(body(twice)) + " is listed twice";
	return NB_ERR_ARGUMENT;
}

// The velocity scatter of nb_upload_kinematic_bodies: each listed body's velocity and angular velocity into its momentum row (the unused lanes
// are left alone), and its kind byte (the caller clears the table first when the set changes).
__global__ void __launch_bounds__(NB_BLOCK) k_kinematic_scatter(const nb_kinematic_body* rows, u32 n, nb_body_momentum* momentum, uint8_t* kind) {
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const nb_kinematic_body r = rows[i];
		nb_body_momentum& m = momentum[r.body];
		m.velocity[0] = r.velocity[0]; m.velocity[1] = r.velocity[1]; m.velocity[2] = r.velocity[2];
		m.angular_velocity[0] = r.angular_velocity[0]; m.angular_velocity[1] = r.angular_velocity[1]; m.angular_velocity[2] = r.angular_velocity[2];
		if (!kind[r.body]) kind[r.body] = 1;   // a new member; an old one keeps its moving bit until the next k_uf_init
	}
}

// Runs one sub-step `body()` through the graph slot `g`: on a capturable stream its launches are recorded once per key into a CUDA
// graph and replayed afterwards.  The grid-synchronising kernels (k_sort_coop's software grid barriers, k_solve's and
// k_solve_flow's spin waits) are captured as cooperative nodes, so the driver guarantees their co-residency at replay, also next to
// other work on the device.  NB_GRAPH=0, the legacy or per-thread default stream and debug mode use plain launches, and so does
// every later step once the driver refuses the capture.
template<class Body>
static int run_graphed(nb_context* ctx, StepGraph& g, cudaStream_t st, float time_step, uint32_t iterations, float gravity, float damping,
					   int transport, unsigned long long plan_version, Body body) {
	if (!g.enabled || st == nullptr || st == cudaStreamLegacy || st == cudaStreamPerThread || ctx->debug) return body();
	StepKey key;
	memset(&key, 0, sizeof(key));  // padding bytes included: the key is compared with memcmp
	key.stream = st; key.ts = time_step; key.gravity = gravity; key.damping = damping; key.iterations = iterations;
	key.B = ctx->B; key.nboxes = ctx->nboxes; key.nspheres = ctx->nspheres; key.nconn = ctx->nconn; key.tagbits = ctx->tagbits; key.kbits = ctx->kbits;
	key.debug = ctx->debug; key.solver_mode = ctx->solver_mode; key.transport = transport; key.plan_version = plan_version; key.graph_epoch = ctx->graph_epoch;
	if (!g.exec || memcmp(&key, &g.key, sizeof(key)) != 0) {
		if (g.exec) { cudaGraphExecDestroy(g.exec); g.exec = nullptr; }
		if (cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
			const unsigned long long before = ctx->launches;
			++ctx->graph_records;
			ctx->capturing = true;
			int r = body();
			ctx->capturing = false;
			cudaGraph_t graph = nullptr;
			cudaError_t e = cudaStreamEndCapture(st, &graph);
			if (r == NB_OK && e == cudaSuccess && graph) e = cudaGraphInstantiate(&g.exec, graph, 0);
			if (graph) cudaGraphDestroy(graph);
			g.launches = ctx->launches - before;
			ctx->launches = before;
			if (r != NB_OK || e != cudaSuccess) g.exec = nullptr;
		}
		if (!g.exec) {  // capture refused: stay on plain launches
			cudaGetLastError();
			g.enabled = 0;
			return body();
		}
		g.key = key;
	}
	CK(cudaGraphLaunch(g.exec, st));
	ctx->upload_pending = false;   // a pending side copy is ordered before the replay: by the graph's event-wait node or by the caller's host-side join
	ctx->launches += g.launches;
	ctx->contacts_internal = true;
	return NB_OK;
}

// One sub-step (example/main.cpp:274-328) of nb_step and nb_shard_step around their solve section `solve()`, which sets up the contact
// rows and sweeps them: nb_step's step_solve, or nb_shard_step's shard_solve with the ghost exchange.
template<class Solve>
static int step_body(nb_context* ctx, float time_step, float gravity, float damping, void* stream, Solve solve) {
	int r;
	if ((r = nb_collide(ctx, stream))) return r;
	if ((r = nb_apply_gravity_damping(ctx, time_step, gravity, damping, stream))) return r;
	if ((r = nb_read_cached_impulses(ctx, stream))) return r;
	if ((r = solve())) return r;
	if ((r = nb_update_cached_impulses(ctx, stream))) return r;
	if ((r = nb_write_cached_impulses(ctx, stream))) return r;
	return nb_advance(ctx, time_step, stream);
}

// The connected opt-out's lookup: the connection keys min(a,b) | max(a,b) << 32, radix sorted on the device, for the binary search of
// the broadphase (nb_collide.cuh, connected()).  Rebuilt when connections are uploaded or loaded and when the flag is set; never per step.
static int build_conn_lookup(nb_context* ctx, cudaStream_t st) {
	const u32 n = (ctx->filter_flags & NB_FILTER_SKIP_CONNECTED) ? ctx->nconn : 0;
	ctx->conn_probe = n;
	if (!n) return NB_OK;
	const Launch L = mk_launch(ctx, st);
	launch_grid(L, k_conn_keys, GRID(n), ctx->conn, n, ctx->conn_scratch);
	CK(cudaMemcpyAsync(ctx->conn_sort_n, &n, 4, cudaMemcpyHostToDevice, st));
	SortBuffers cs = { { ctx->conn_scratch, ctx->conn_keys }, { nullptr, nullptr }, ctx->sb.hist, ctx->sb.bar };
	nb_radix_sort(L, cs, ctx->conn_sort_n, 0, 64, false, 0);   // the result lands in keys[1] = conn_keys
	CK(cudaGetLastError());
	return NB_OK;
}

// Installs a sensor table of n flags (n = 0 removes it) with room for max_pairs candidate pairs (0: NB_SENSOR_PAIRS_PER_SENSOR per sensor
// collider, at least NB_SENSOR_PAIRS_MIN, at most the context's scratch stride), and empties the old overlap list, so that the next
// nb_write_cached_impulses begins every overlap.  Synchronises `st`.
#define NB_SENSOR_PAIRS_PER_SENSOR 256u
#define NB_SENSOR_PAIRS_MIN 1024u
// The candidate keys, sort buffers and overlap lists with room for `cap` entries (grown on `st` only when they are smaller).
static int ensure_sensor_lists(nb_context* ctx, u32 cap, cudaStream_t st) {
	GROW(ctx->sensor_keys, cap, st); GROW(ctx->sensor_cur, cap, st); GROW(ctx->sensor_old, cap, st);
	for (int i = 0; i < 2; ++i) { GROW(ctx->sensor_sort_keys[i], cap, st); GROW(ctx->sensor_sort_vals[i], cap, st); }
	ctx->sensor_sb = { { ctx->sensor_sort_keys[0].p, ctx->sensor_sort_keys[1].p }, { ctx->sensor_sort_vals[0].p, ctx->sensor_sort_vals[1].p }, ctx->sb.hist, ctx->sb.bar };
	return NB_OK;
}
static int set_sensors(nb_context* ctx, const uint8_t* host, u32 n, u32 max_pairs, cudaStream_t st) {
	CK(cudaStreamSynchronize(st));
	u32 cap = 0;
	if (n) {
		std::vector<uint8_t> f(n);
		u32 ns = 0;
		for (u32 i = 0; i < n; ++i) { f[i] = host[i] ? 1 : 0; ns += f[i]; }
		cap = max_pairs ? max_pairs : std::min<u64>(std::max<u64>(NB_SENSOR_PAIRS_MIN, (u64)NB_SENSOR_PAIRS_PER_SENSOR * ns), ctx->stride);
		if (cap > ctx->stride) {   // k_sensor_np's flags and the event flags live in the scratch planes
			ctx->error = "max_sensor_pairs exceeds the context's scratch capacity (" + std::to_string(ctx->stride) + ": the largest of max_pairs, max_contacts, bodies, colliders)";
			return NB_ERR_CAPACITY;
		}
		{ int r = ensure_sensor_lists(ctx, cap, st); if (r) return r; }
		CK(cudaMemcpyAsync(ctx->sensor, f.data(), n, cudaMemcpyHostToDevice, st));
	}
	CK(cudaMemsetAsync(ctx->counts + CNT_SENSOR_PAIRS, 0, 3 * sizeof(u32), st));   // candidates, current and old overlaps
	CK(cudaStreamSynchronize(st));
	ctx->has_sensor = n != 0; ctx->sensor_cap = cap;
	++ctx->graph_epoch;   // nb_step's graph re-records with or without the sensor launches
	return NB_OK;
}

// The sensor pairs' overlaps of one collide (nb_collide.cuh, below k_np_emit): test, compact, sort by key, gather.  5 launches.
static void launch_sensor_overlaps(nb_context* ctx, const Launch& L) {
	u32* counts = ctx->counts;
	const u32 cap = ctx->sensor_cap;
	const FrontEnd& f = ctx->front;
	launch_grid(L, k_sensor_np, GRID((size_t)cap * 4), ctx->sensor_keys.p, cap, ctx->kbits, ctx->nboxes, f.world_xf, ctx->box_data, ctx->sph_data,
		f.col_tag, f.col_body, ctx->flags, counts);
	nb_scan_reduce<1>(L, ctx->flags, ctx->stride, counts + CNT_SENSOR_PAIRS, 0, ctx->block_sums, counts + CNT_SENSOR_HITS);
	launch_grid(L, k_sensor_compact, NB_SCAN_GRID, ctx->flags, ctx->block_sums, ctx->sensor_keys.p, ctx->kbits, f.col_tag,
		ctx->sensor_sb.keys[0], ctx->sensor_sb.vals[0], counts);
	const int cur = nb_radix_sort(L, ctx->sensor_sb, counts + CNT_SENSOR_HITS, 0, (int)ctx->tagbits, true, 0, 32, (int)(32 + ctx->tagbits));
	launch_grid(L, k_sensor_gather, GRID(cap), ctx->sensor_sb.keys[cur], ctx->sensor_sb.vals[cur], ctx->sensor_keys.p, ctx->kbits, f.col_tag, f.col_body,
		ctx->sensor_cur.p, counts);
}

extern "C" {

int nb_pack_momentum(nb_context* ctx, const uint32_t* dev_indices, uint32_t n, void* dev_out, void* stream) {
	if (!n) return NB_OK;
	JOIN_UPLOADS();
	launch_grid(mk_launch(ctx, stream), k_pack_rows, GRID(2 * n), (const float4*)ctx->mom, dev_indices, n, (float4*)dev_out);
	CK(cudaGetLastError());
	return NB_OK;
}
int nb_unpack_momentum(nb_context* ctx, const uint32_t* dev_indices, const uint32_t* dev_sources, uint32_t n, const void* dev_in, void* stream) {
	if (!n) return NB_OK;
	JOIN_UPLOADS();
	launch_grid(mk_launch(ctx, stream), k_unpack_rows, GRID(2 * n), (float4*)ctx->mom, dev_indices, dev_sources, n, (const float4*)dev_in);
	CK(cudaGetLastError());
	return NB_OK;
}

int nb_create(const nb_config* config, nb_context** out) {
	if (!config || !out) return NB_ERR_ARGUMENT;
	nb_context* ctx = new nb_context();
	*out = ctx;
	ctx->cfg = *config;
	ctx->launches = 0;
	nb_config& c = ctx->cfg;
	if (!c.max_bodies) c.max_bodies = 1;
	u32 K = c.max_boxes + c.max_spheres;
	if (!c.max_pairs) c.max_pairs = 16 * (K ? K : 1);
	if (!c.max_contacts) c.max_contacts = 24 * c.max_bodies;
	int ndev = 0;
	CK(cudaGetDeviceCount(&ndev));
	if (ndev <= 0) { ctx->error = "no CUDA device: nudge_b200 has no CPU path"; return NB_ERR_CUDA; }
	CK(cudaSetDevice(c.device));
	cudaDeviceProp prop;
	CK(cudaGetDeviceProperties(&prop, c.device));
	ctx->sms = prop.multiProcessorCount;
	if (!prop.cooperativeLaunch) { ctx->error = "device lacks cooperative launch"; return NB_ERR_CUDA; }

	const u32 B = c.max_bodies, P = c.max_pairs, C = c.max_contacts;
	ctx->B = 0; ctx->nboxes = 0; ctx->nspheres = 0; ctx->nconn = 0;
	ctx->tagbits = 1; ctx->upload_tagbits = 1; ctx->kbits = bits_for(K ? K : 1); ctx->bodybits = bits_for(B);
	ctx->stride = ((std::max(std::max(P, C), std::max(B, K)) + 63) / 64) * 64;
	ctx->cstride = ((C + 8 * 16 * NB_SCHED_MAXV + 31) / 32) * 32;  // slots = batch*8 + lane; leftover batches of the 16 buckets may be partly empty (a hub body beyond that: OVF_SCHED from k_batch_index)
	ctx->slots_per_bucket = (C + 15) / 16 + 1;

	ALLOC(ctx->xf, B); ALLOC(ctx->props, B); ALLOC(ctx->mom, B); ALLOC(ctx->idle, B);
	ALLOC(ctx->box_tags, c.max_boxes); ALLOC(ctx->box_data, c.max_boxes); ALLOC(ctx->box_xf, c.max_boxes);
	ALLOC(ctx->sph_tags, c.max_spheres); ALLOC(ctx->sph_data, c.max_spheres); ALLOC(ctx->sph_xf, c.max_spheres);
	ALLOC(ctx->conn, c.max_connections);
	ALLOC(ctx->filter, K); ALLOC(ctx->sensor, K); ALLOC(ctx->conn_keys, c.max_connections); ALLOC(ctx->conn_scratch, c.max_connections); ALLOC(ctx->conn_sort_n, 1);
	ALLOC(ctx->counts, CNT__COUNT);
	{ int r = alloc_front_end(ctx, ctx->front, K); if (r) return r; }
	ctx->sort_cap = std::max(std::max(K, P), 2 * C);
	for (int i = 0; i < 2; ++i) { ALLOC(ctx->sb.keys[i], ctx->sort_cap); ALLOC(ctx->sb.vals[i], ctx->sort_cap); }
	ALLOC(ctx->sb.hist, 256 * (size_t)ctx->sms);
	ctx->sb.bar = ctx->counts + CNT_BAR0;
	{ const char* e = getenv("NB_GRAPH"); ctx->graph.enabled = e ? atoi(e) != 0 : 1; }
	CK(cudaFuncSetAttribute(k_sort_coop<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CoopSortSmem)));
	CK(cudaFuncSetAttribute(k_sort_coop<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CoopSortSmem)));
	ALLOC(ctx->flags, 5 * (size_t)ctx->stride); ALLOC(ctx->offs, 5 * (size_t)ctx->stride); ALLOC(ctx->block_sums, NB_SCAN_SUMS);
	ALLOC(ctx->live, P); ALLOC(ctx->np_pen, P); ALLOC(ctx->np_info, P); ALLOC(ctx->np_list, P); ALLOC(ctx->np_start, P);
	ALLOC(ctx->staged.data, 2 * (size_t)C); ALLOC(ctx->staged.bodies, C); ALLOC(ctx->staged.tags, C); ALLOC(ctx->staged.features, C);
	ALLOC(ctx->fin.data, 2 * (size_t)C); ALLOC(ctx->fin.bodies, C); ALLOC(ctx->fin.tags, C); ALLOC(ctx->fin.features, C);
	ALLOC(ctx->sleeping, (size_t)P + C);
	ALLOC(ctx->parent, B); ALLOC(ctx->active, B); ALLOC(ctx->active_idx, B); ALLOC(ctx->taint, B);
	ALLOC(ctx->cache_tags, C); ALLOC(ctx->cache_features, C); ALLOC(ctx->cache_data, C);
	ALLOC(ctx->culled_tags, C); ALLOC(ctx->culled_features, C); ALLOC(ctx->culled_data, C);
	ALLOC(ctx->sorted, C); ALLOC(ctx->impulses, C);
	ALLOC(ctx->inertia, 2 * (size_t)B);
	ALLOC(ctx->slot_of, C); ALLOC(ctx->slot_done, 16 * (size_t)ctx->slots_per_bucket); ALLOC(ctx->slot_left, 16 * (size_t)ctx->slots_per_bucket);
	ctx->sched_spill_cap = std::min<u32>(ctx->slots_per_bucket + 2, 16384u);
	ALLOC(ctx->sched_spill_ent, 16 * (size_t)ctx->sched_spill_cap * 16); ALLOC(ctx->sched_spill_uid, 16 * (size_t)ctx->sched_spill_cap);
	CK(cudaMemset(ctx->sched_spill_ent, 0xff, sizeof(u32) * 16 * (size_t)ctx->sched_spill_cap * 16));
	ALLOC(ctx->left_count, 16); ALLOC(ctx->batch_of, C); ALLOC(ctx->slot_idx, C); ALLOC(ctx->mw, 2 * (size_t)B); ALLOC(ctx->cab, C); ALLOC(ctx->back, C);
	ALLOC(ctx->sched_slot_v, 8 * (size_t)C); ALLOC(ctx->sched_empty, ((size_t)C + 3) & ~(size_t)3);   // 33 B per contact of capacity
	ALLOC(ctx->sched_state, 16 * NB_SCHED_SEGS * 8 * (size_t)NB_SCHED_STATE); ALLOC(ctx->sched_join_slot, 16 * NB_SCHED_SEGS * 8 * NB_SCHED_JOIN);
	ALLOC(ctx->sched_pick, 16 * NB_SCHED_SEGS * 8); ALLOC(ctx->sched_pick_res, 16 * NB_SCHED_SEGS);
	ALLOC(ctx->rows.plane, (size_t)ROW_PLANES_TOTAL * ctx->cstride); ALLOC(ctx->rows.state, 3 * (size_t)ctx->cstride);
	ALLOC(ctx->rows.a, ctx->cstride); ALLOC(ctx->rows.b, ctx->cstride); ALLOC(ctx->rows.contact, ctx->cstride); ALLOC(ctx->rows.wait, 2 * (size_t)ctx->cstride); ALLOC(ctx->chain_start, B); ALLOC(ctx->chain_len, B);
	ALLOC(ctx->warm, 4 * (size_t)C);
	ctx->rows.stride = ctx->cstride;
	ALLOC(ctx->jcnt, B); ALLOC(ctx->jd, 2 * (size_t)B);
	// upload of the rows `collide` does not read, on a copy stream of its own (NB_COPY_OVERLAP=0: everything on the caller's stream)
	{ const char* e = getenv("NB_COPY_OVERLAP"); ctx->copy_overlap = e ? atoi(e) != 0 : 1; }
	CK(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
	CK(cudaEventCreateWithFlags(&ctx->ev_up_begin, cudaEventDisableTiming)); CK(cudaEventCreateWithFlags(&ctx->ev_up_done, cudaEventDisableTiming));
	CK(cudaEventRecord(ctx->ev_up_done, ctx->copy_stream));   // a first, already complete record for the step graph's event-wait node
	ctx->solver_mode = NB_SOLVER_PARITY;
	CK(cudaFuncSetAttribute(k_jacobi_sweep<true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(JacobiSmem<1>)));
	CK(cudaFuncSetAttribute(k_jacobi_sweep<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(JacobiSmem<1>)));
	CK(cudaFuncSetAttribute(k_jacobi_sweep<true, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(JacobiSmem<2>)));
	CK(cudaFuncSetAttribute(k_jacobi_sweep<false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(JacobiSmem<2>)));
	{
		int per1 = 0, per2 = 0;
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per1, k_jacobi_sweep<false, 1>, NJ_TILE, sizeof(JacobiSmem<1>)));
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per2, k_jacobi_sweep<false, 2>, NJ_TILE, sizeof(JacobiSmem<2>)));
		if (per1 < 1 || per2 < 1) { ctx->error = "k_jacobi_sweep does not fit on an SM"; return NB_ERR_CUDA; }
		ctx->jacobi_blocks1 = ctx->sms * per1; ctx->jacobi_blocks2 = ctx->sms * per2;   // persistent: every CTA walks tiles blockIdx.x, + gridDim.x, ...
		if (const char* e = getenv("NB_SOLVER")) ctx->solver_mode = !strcmp(e, "throughput") ? NB_SOLVER_THROUGHPUT : NB_SOLVER_PARITY;
	}
	ctx->pair_keys = ctx->sb.keys[0];
	ctx->pair_keys_debug = nullptr; ctx->debug = 0;

	// rcpps / rsqrtps tables from this host's CPU (SURVEY.md §0.5)
	u32 rcp_lut[2048], rsqrt_lut[2048];
	nb_host_sample_luts(rcp_lut, rsqrt_lut);
	ctx->lut_exact = nb_host_check_lut_model(rcp_lut, rsqrt_lut);
	CK(cudaMemcpyToSymbol(c_rcp_lut, rcp_lut, sizeof(rcp_lut)));
	CK(cudaMemcpyToSymbol(c_rsqrt_lut, rsqrt_lut, sizeof(rsqrt_lut)));
	CK(cudaMemcpyToSymbol(g_rcp_lut, rcp_lut, sizeof(rcp_lut)));
	CK(cudaMemcpyToSymbol(g_rsqrt_lut, rsqrt_lut, sizeof(rsqrt_lut)));

	int per_sm = 0;
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_solve, NB_BLOCK, 0));
	{ int per_kin = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_kin, k_solve_kin, NB_BLOCK, 0)); per_sm = std::min(per_sm, per_kin); }
	if (per_sm < 1) { ctx->error = "k_solve does not fit on an SM"; return NB_ERR_CUDA; }
	ctx->coop_blocks_solve = ctx->sms * per_sm;  // all co-resident: the dataflow solver relies on it
	CK(cudaDeviceSynchronize());
	return NB_OK;
}

void nb_destroy(nb_context* ctx) {
	if (!ctx) return;
	cudaDeviceSynchronize();
	if (ctx->graph.exec) cudaGraphExecDestroy(ctx->graph.exec);
	if (ctx->tev_made) for (int i = 0; i < 64; ++i) { cudaEventDestroy(ctx->tev[0][i]); cudaEventDestroy(ctx->tev[1][i]); }
	if (ctx->copy_stream) { cudaStreamDestroy(ctx->copy_stream); cudaEventDestroy(ctx->ev_up_begin); cudaEventDestroy(ctx->ev_up_done); }
	free_snapshots(ctx);
	delete ctx;   // and with it its buffers
}

const char* nb_last_error(const nb_context* ctx) { return ctx ? ctx->error.c_str() : "null context"; }
uint64_t nb_launch_count(const nb_context* ctx) { return ctx->launches; }
int nb_lut_model_exact(const nb_context* ctx) { return ctx->lut_exact; }

#define H2D(dst, src, n, T) CK(cudaMemcpyAsync(dst, src, (size_t)(n) * sizeof(T), cudaMemcpyHostToDevice, (cudaStream_t)stream))
#define D2H(dst, src, n, T) CK(cudaMemcpyAsync(dst, src, (size_t)(n) * sizeof(T), cudaMemcpyDeviceToHost, (cudaStream_t)stream))

int nb_upload_bodies(nb_context* ctx, const nb_body_data* h, void* stream) {
	NB_RANGE("nb_upload_bodies");
	ctx->report_ok = false;
	if (h->count > ctx->cfg.max_bodies) { ctx->error = "too many bodies"; return NB_ERR_CAPACITY; }
	if (h->count != ctx->B) { drop_kinematic(ctx); drop_body_forces(ctx); drop_joints(ctx); drop_ccd(ctx); }   // the kinematic set, the force table, the joints and the CCD set belong to a body count
	ctx->B = h->count;
	cudaStream_t st = (cudaStream_t)stream;
	H2D(ctx->xf, h->transforms, h->count, nb_transform); H2D(ctx->idle, h->idle_counters, h->count, uint8_t);   // all the collision stage reads
	if (ctx->copy_overlap && ctx->copy_stream && st != nullptr && st != cudaStreamLegacy && st != cudaStreamPerThread) {
		CK(cudaEventRecord(ctx->ev_up_begin, st));                       // after everything already queued on the caller's stream (it may still use the old rows)
		CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_up_begin, 0));
		CK(cudaMemcpyAsync(ctx->mom, h->momentum, (size_t)h->count * sizeof(nb_body_momentum), cudaMemcpyHostToDevice, ctx->copy_stream));
		CK(cudaMemcpyAsync(ctx->props, h->properties, (size_t)h->count * sizeof(nb_body_properties), cudaMemcpyHostToDevice, ctx->copy_stream));
		CK(cudaEventRecord(ctx->ev_up_done, ctx->copy_stream));
		ctx->upload_pending = true;
	}
	else {
		H2D(ctx->props, h->properties, h->count, nb_body_properties); H2D(ctx->mom, h->momentum, h->count, nb_body_momentum);
	}
	return NB_OK;
}
#define ROWS_OK(count) do { if ((count) > ctx->cfg.max_bodies) { ctx->error = "row count exceeds max_bodies"; return NB_ERR_CAPACITY; } } while (0)
int nb_upload_momentum(nb_context* ctx, const nb_body_momentum* h, uint32_t count, void* stream) { ROWS_OK(count); JOIN_UPLOADS(); H2D(ctx->mom, h, count, nb_body_momentum); return NB_OK; }
int nb_upload_transforms(nb_context* ctx, const nb_transform* h, uint32_t count, void* stream) { ROWS_OK(count); H2D(ctx->xf, h, count, nb_transform); return NB_OK; }
int nb_download_momentum(nb_context* ctx, nb_body_momentum* h, uint32_t count, void* stream) { ROWS_OK(count); JOIN_UPLOADS(); D2H(h, ctx->mom, count, nb_body_momentum); return NB_OK; }
int nb_download_transforms(nb_context* ctx, nb_transform* h, uint32_t count, void* stream) { ROWS_OK(count); D2H(h, ctx->xf, count, nb_transform); return NB_OK; }

int nb_upload_colliders(nb_context* ctx, const nb_collider_data* h, void* stream) {
	ctx->report_ok = false;
	if (h->boxes.count > ctx->cfg.max_boxes || h->spheres.count > ctx->cfg.max_spheres) { ctx->error = "too many colliders"; return NB_ERR_CAPACITY; }
	if (ctx->has_filter && h->boxes.count + h->spheres.count != ctx->nboxes + ctx->nspheres) { ctx->has_filter = false; ++ctx->graph_epoch; }  // the table belongs to a collider count
	if (ctx->has_sensor && h->boxes.count + h->spheres.count != ctx->nboxes + ctx->nspheres) { ctx->has_sensor = false; ++ctx->graph_epoch; }  // so does the sensor table
	ctx->nboxes = h->boxes.count; ctx->nspheres = h->spheres.count;
	u32 maxtag = 1;
	for (u32 i = 0; i < h->boxes.count; ++i) maxtag = std::max(maxtag, h->boxes.tags[i]);
	for (u32 i = 0; i < h->spheres.count; ++i) maxtag = std::max(maxtag, h->spheres.tags[i]);
	ctx->tagbits = bits_for((u64)maxtag + 1);
	ctx->kbits = bits_for(std::max(1u, ctx->nboxes + ctx->nspheres));
	H2D(ctx->box_tags, h->boxes.tags, h->boxes.count, u32); H2D(ctx->box_data, h->boxes.data, h->boxes.count, nb_box_collider);
	H2D(ctx->box_xf, h->boxes.transforms, h->boxes.count, nb_transform);
	H2D(ctx->sph_tags, h->spheres.tags, h->spheres.count, u32); H2D(ctx->sph_data, h->spheres.data, h->spheres.count, nb_sphere_collider);
	H2D(ctx->sph_xf, h->spheres.transforms, h->spheres.count, nb_transform);
	return NB_OK;
}
int nb_upload_connections(nb_context* ctx, const nb_body_connections* h, void* stream) {
	if (h->count > ctx->cfg.max_connections) { ctx->error = "too many connections"; return NB_ERR_CAPACITY; }
	ctx->nconn = h->count;
	ctx->conn_host.assign(h->data, h->data + h->count);
	H2D(ctx->conn, h->data, h->count, nb_body_pair);
	return build_conn_lookup(ctx, (cudaStream_t)stream);
}

int nb_upload_collision_filters(nb_context* ctx, const nb_collision_filter* h, uint32_t n, uint32_t flags, void* stream) {
	const u32 K = ctx->nboxes + ctx->nspheres;
	if (n != 0 && n != K) { ctx->error = "collision filter count must be 0 or boxes + spheres (" + std::to_string(K) + ")"; return NB_ERR_ARGUMENT; }
	if (n && !h) { ctx->error = "null collision filter table"; return NB_ERR_ARGUMENT; }
	if (flags & ~(u32)NB_FILTER_SKIP_CONNECTED) { ctx->error = "unknown collision filter flags"; return NB_ERR_ARGUMENT; }
	cudaStream_t st = (cudaStream_t)stream;
	if (n) CK(cudaMemcpyAsync(ctx->filter, h, sizeof(nb_collision_filter) * (size_t)n, cudaMemcpyHostToDevice, st));   // category | mask << 16 as a u32
	ctx->has_filter = n != 0; ctx->filter_flags = flags;
	++ctx->graph_epoch;   // nb_step's graph re-records with the new kernel arguments
	int r = build_conn_lookup(ctx, st); if (r) return r;
	CK(cudaStreamSynchronize(st));
	return NB_OK;
}
int nb_upload_sensors(nb_context* ctx, const uint8_t* h, uint32_t n, uint32_t max_sensor_pairs, void* stream) {
	const u32 K = ctx->nboxes + ctx->nspheres;
	if (n != 0 && n != K) { ctx->error = "sensor table count must be 0 or boxes + spheres (" + std::to_string(K) + ")"; return NB_ERR_ARGUMENT; }
	if (n && !h) { ctx->error = "null sensor table"; return NB_ERR_ARGUMENT; }
	return set_sensors(ctx, h, n, max_sensor_pairs, (cudaStream_t)stream);
}
int nb_upload_kinematic_bodies(nb_context* ctx, const nb_kinematic_body* h, uint32_t n, void* stream) {
	NB_RANGE("nb_upload_kinematic_bodies");
	if (n && !h) { ctx->error = "null kinematic body table"; return NB_ERR_ARGUMENT; }
	for (u32 i = 0; i < n; ++i) if (int r = check_body(ctx, "kinematic body", i, h[i].body, true)) return r;
	if (int r = bodies_distinct(ctx, "kinematic body", n, [&](u32 i) { return h[i].body; })) return r;
	std::vector<u32> list(n);
	for (u32 i = 0; i < n; ++i) list[i] = h[i].body;
	std::sort(list.begin(), list.end());
	cudaStream_t st = (cudaStream_t)stream;
	JOIN_UPLOADS();   // ordered like nb_upload_momentum, after a pending nb_upload_bodies side copy
	if (!n) { drop_kinematic(ctx); return NB_OK; }
	ALLOC(ctx->kind, ctx->cfg.max_bodies);   // the kind table, on first use
	GROW(ctx->kin_rows, n, st);
	const bool same = ctx->has_kin && list == ctx->kin_list;
	if (!same) CK(cudaMemsetAsync(ctx->kind, 0, ctx->cfg.max_bodies, st));
	CK(put_staged(ctx, ctx->kin_rows.p, h, sizeof(nb_kinematic_body) * (size_t)n, st));
	launch_grid(mk_launch(ctx, st), k_kinematic_scatter, GRID(n), ctx->kin_rows.p, n, ctx->mom, ctx->kind);
	CK(cudaGetLastError());
	if (!same) { ctx->has_kin = true; ctx->kin_list.swap(list); ++ctx->graph_epoch; }   // nb_step's graph re-records with the table
	return NB_OK;
}
int nb_upload_cache(nb_context* ctx, const nb_contact_cache* h, void* stream) {
	if (h->count > ctx->cfg.max_contacts) { ctx->error = "cache too large"; return NB_ERR_CAPACITY; }
	H2D(ctx->cache_tags, h->tags, h->count, u64); H2D(ctx->cache_features, h->features, h->count, u32); H2D(ctx->cache_data, h->data, h->count, nb_cached_impulse);
	u32 n = h->count;
	CK(cudaMemcpyAsync(ctx->counts + CNT_CACHE, &n, 4, cudaMemcpyHostToDevice, (cudaStream_t)stream));
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	return NB_OK;
}
int nb_download_bodies(nb_context* ctx, nb_body_data* h, void* stream) {
	NB_RANGE("nb_download_bodies");
	u32 n = std::min(h->count, ctx->B);
	JOIN_UPLOADS();
	D2H(h->transforms, ctx->xf, n, nb_transform); D2H(h->momentum, ctx->mom, n, nb_body_momentum); D2H(h->idle_counters, ctx->idle, n, uint8_t);
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	return NB_OK;
}
static int get_counts(nb_context* ctx, u32* host, void* stream) {
	D2H(host, ctx->counts, CNT__COUNT, u32);
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	return NB_OK;
}
int nb_download_counts(nb_context* ctx, nb_counts* out, void* stream) {
	u32 h[CNT__COUNT];
	int r = get_counts(ctx, h, stream); if (r) return r;
	out->pairs = h[CNT_PAIRS]; out->live_pairs = h[CNT_LIVE_TOTAL]; out->contacts = h[CNT_CONTACTS]; out->sleeping = h[CNT_SLEEPING];
	out->active = h[CNT_ACTIVE]; out->cache = h[CNT_CACHE]; out->culled = h[CNT_CULLED]; out->batches = h[CNT_BATCHES]; out->levels = h[CNT_LEVELS];
	out->overflow = h[CNT_OVERFLOW];
	if (h[CNT_OVERFLOW]) {
		ctx->error = "capacity overflow during the last step (nb_counts.overflow: 1 pairs, 2 contacts, 4 batch scheduler, 32 sensor pairs)";
		if (h[CNT_OVERFLOW] & OVF_SENSORS) ctx->error += "; bit 32: more candidate sensor pairs than max_sensor_pairs (nb_upload_sensors), the step's overlaps and sensor events are undefined";
		return NB_ERR_OVERFLOW;
	}
	return NB_OK;
}
int nb_download_sensor_overlaps(nb_context* ctx, nb_sensor_overlap* host, uint32_t capacity, uint32_t* count, void* stream) {
	NB_RANGE("nb_download_sensor_overlaps");
	u32 c[CNT__COUNT];
	int r = get_counts(ctx, c, stream); if (r) return r;
	const u32 n = ctx->has_sensor ? c[CNT_SENSOR_HITS] : 0;
	if (count) *count = n;
	if (n > capacity) { ctx->error = "host overlap buffer too small: " + std::to_string(n) + " overlaps"; return NB_ERR_CAPACITY; }
	if (n && !host) { ctx->error = "null host overlap buffer"; return NB_ERR_ARGUMENT; }
	D2H(host, ctx->sensor_cur.p, n, nb_sensor_overlap);
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	return NB_OK;
}
int nb_download_contacts(nb_context* ctx, nb_contact_data* h, nb_active_bodies* ha, void* stream) {
	u32 c[CNT__COUNT];
	int r = get_counts(ctx, c, stream); if (r) return r;
	if (h) {
		u32 n = c[CNT_CONTACTS], s = c[CNT_SLEEPING];
		if (n > h->capacity) { ctx->error = "host contact buffer too small"; return NB_ERR_CAPACITY; }
		// sleeping pairs can number up to the broadphase pairs; the reference sizes that buffer like the contact arrays (nudge.h:73-82)
		if (h->sleeping_pairs && s > h->capacity) { ctx->error = "host sleeping-pair buffer too small (it is bounded by nb_contact_data.capacity)"; return NB_ERR_CAPACITY; }
		h->count = n; h->sleeping_count = s;
		D2H(h->data, ctx->fin.data, n, nb_contact); D2H(h->bodies, ctx->fin.bodies, n, nb_body_pair);
		D2H(h->tags, ctx->fin.tags, n, u64); D2H(h->features, ctx->fin.features, n, u32);
		if (h->sleeping_pairs) D2H(h->sleeping_pairs, ctx->sleeping, s, u64);
	}
	if (ha) {
		u32 n = c[CNT_ACTIVE];
		if (n > ha->capacity) { ctx->error = "host active-body buffer too small"; return NB_ERR_CAPACITY; }
		ha->count = n;
		D2H(ha->indices, ctx->active_idx, n, u32);
	}
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	return c[CNT_OVERFLOW] ? NB_ERR_OVERFLOW : NB_OK;
}
// Host -> HBM for the outputs of collide (the reference lets user code add or edit contacts between the calls, example/main.cpp:288).
int nb_upload_contacts(nb_context* ctx, const nb_contact_data* h, const nb_active_bodies* ha, void* stream) {
	ctx->scene_edited = false;
	ctx->report_ok = false;
	if (h) {
		if (h->count > ctx->cfg.max_contacts || h->sleeping_count > ctx->cfg.max_contacts) { ctx->error = "too many contacts"; return NB_ERR_CAPACITY; }
		ctx->contacts_internal = false;
		u32 maxtag = 1;
		for (u32 i = 0; i < h->count; ++i) maxtag = std::max({ maxtag, (u32)h->tags[i], (u32)(h->tags[i] >> 32) });
		ctx->upload_tagbits = bits_for((u64)maxtag + 1);
		H2D(ctx->fin.data, h->data, h->count, nb_contact); H2D(ctx->fin.bodies, h->bodies, h->count, nb_body_pair);
		H2D(ctx->fin.tags, h->tags, h->count, u64); H2D(ctx->fin.features, h->features, h->count, u32);
		if (h->sleeping_count) H2D(ctx->sleeping, h->sleeping_pairs, h->sleeping_count, u64);
		u32 n[2] = { h->count, h->sleeping_count };
		CK(cudaMemcpyAsync(ctx->counts + CNT_CONTACTS, &n[0], 4, cudaMemcpyHostToDevice, (cudaStream_t)stream));
		CK(cudaMemcpyAsync(ctx->counts + CNT_SLEEPING, &n[1], 4, cudaMemcpyHostToDevice, (cudaStream_t)stream));
	}
	if (ha) {
		if (ha->count > ctx->cfg.max_bodies) { ctx->error = "too many active bodies"; return NB_ERR_CAPACITY; }
		H2D(ctx->active_idx, ha->indices, ha->count, u32);
		u32 n = ha->count;
		CK(cudaMemcpyAsync(ctx->counts + CNT_ACTIVE, &n, 4, cudaMemcpyHostToDevice, (cudaStream_t)stream));
	}
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	return NB_OK;
}

int nb_download_cache(nb_context* ctx, nb_contact_cache* h, void* stream) {
	u32 c[CNT__COUNT];
	int r = get_counts(ctx, c, stream); if (r) return r;
	u32 n = c[CNT_CACHE];
	if (n > h->capacity) { ctx->error = "host cache buffer too small"; return NB_ERR_CAPACITY; }
	h->count = n;
	D2H(h->tags, ctx->cache_tags, n, u64); D2H(h->features, ctx->cache_features, n, u32); D2H(h->data, ctx->cache_data, n, nb_cached_impulse);
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	return NB_OK;
}

// ---------------- collide ----------------
int nb_collide(nb_context* ctx, void* stream) {
	NB_RANGE("nb_collide");
	ctx->scene_edited = false;
	ctx->report_ok = false;
	ctx->in_step = true;   // until the nb_advance that ends the step
	ctx->step_dt = 0.0f;
	Launch L = mk_launch(ctx, stream);
	const u32 K = ctx->nboxes + ctx->nspheres, B = ctx->B, nboxes = ctx->nboxes;
	u32* counts = ctx->counts;
	uint8_t* kind = ctx->has_kin ? ctx->kind : nullptr;
	if (kind) JOIN_UPLOADS();   // k_uf_init reads the kinematic bodies' momentum rows
	const uint8_t* sensor = ctx->has_sensor ? ctx->sensor : nullptr;   // null: the kernels never touch the sensor list
	const FrontEnd& f = ctx->front;
	int r = launch_front_end(ctx, L, f, ctx->sb, counts, ctx->has_filter ? ctx->filter : nullptr, kind, sensor);
	if (r || K == 0 || B == 0) return r;
	launch_grid(L, kind ? k_grid_pairs<true> : k_grid_pairs<false>, GRID((size_t)K * 32), K, f.order, f.leaf_min, f.leaf_max, f.smallf, f.mkeys, f.table_keys, f.table_vals, f.table_mask, ctx->kbits,
		f.col_body, ctx->conn_keys, ctx->conn_probe, sensor, ctx->sensor_keys.p, ctx->sensor_cap, ctx->sb.keys[0], ctx->cfg.max_pairs, counts);
	launch_grid(L, k_large_pairs, GRID(K), K, f.order, f.leaf_min, f.leaf_max, f.smallf, f.large_list, ctx->kbits,
		f.col_body, ctx->conn_keys, ctx->conn_probe, sensor, ctx->sensor_keys.p, ctx->sensor_cap, ctx->sb.keys[0], ctx->cfg.max_pairs, counts);
	// nudge.cpp:3498; the sort also clamps CNT_PAIRS to the capacity (the overflow bit is already set by emit_pair)
	int cur = nb_radix_sort(L, ctx->sb, counts + CNT_PAIRS, 0, (int)(2 * ctx->kbits), false, 0, 0, 0, nullptr, ctx->cfg.max_pairs);
	ctx->pair_keys = ctx->sb.keys[cur];
	if (ctx->debug) launch_grid(L, k_copy_u64, GRID(ctx->cfg.max_pairs), ctx->pair_keys, ctx->pair_keys_debug, counts + CNT_PAIRS);

	// coarse islands (nudge.cpp:3500-3703)
	const u32 P = ctx->cfg.max_pairs, S = ctx->stride;
	launch_grid(L, k_uf_init, GRID(B), ctx->parent, ctx->active, ctx->taint, kind, ctx->mom, B);
	if (ctx->nconn) launch_grid(L, k_uf_union_conn, GRID(ctx->nconn), ctx->parent, ctx->taint, ctx->idle, kind, ctx->conn, ctx->nconn);
	launch_grid(L, k_uf_union_pairs, GRID(P), ctx->parent, ctx->taint, ctx->idle, kind, ctx->pair_keys, ctx->kbits, f.col_body, counts);
	launch_grid(L, k_uf_flatten_active, GRID(B), ctx->parent, ctx->active, ctx->taint, ctx->idle, kind, B);
	launch_grid(L, k_pair_flags, GRID(P), ctx->pair_keys, ctx->kbits, nboxes, f.col_body, ctx->parent, ctx->active, kind, ctx->flags, S, counts);
	nb_scan_reduce<5>(L, ctx->flags, S, counts + CNT_PAIRS, 0, ctx->block_sums, counts + CNT_LIVE0);  // -> LIVE0..3, SLEEP_COARSE
	launch_grid(L, k_partition, NB_SCAN_GRID, ctx->pair_keys, ctx->kbits, ctx->flags, ctx->block_sums, S, f.col_tag, ctx->live, ctx->sleeping, counts);

	// narrowphase: count, scan, emit (nudge.cpp:3753-3786)
	launch_grid(L, k_np_faces, GRID(P), ctx->live, nboxes, f.world_xf, ctx->box_data, ctx->sph_data, f.col_tag, ctx->flags, S, ctx->np_pen, ctx->np_info, counts);
	nb_scan_reduce<1>(L, ctx->flags + 3 * (size_t)S, S, counts + CNT_LIVE0, 0, ctx->block_sums, counts + CNT_SURV);
	launch_grid(L, k_np_list, NB_SCAN_GRID, ctx->flags, ctx->block_sums, S, ctx->np_list, counts);
	launch_grid(L, k_np_clip, GRID(P), ctx->live, ctx->np_list, ctx->np_pen, ctx->np_info, f.world_xf, ctx->box_data, f.col_tag, ctx->flags, S,
		ctx->fin /* scratch: rewritten by k_contact_compact below */, ctx->np_start, ctx->cfg.max_contacts, counts);
	nb_scan<3>(L, ctx->flags, ctx->offs, S, counts + CNT_LIVE_TOTAL, 0, ctx->block_sums, counts + CNT_FACE);  // -> FACE, EDGE, OTHER
	launch_grid(L, k_np_emit, GRID(P), ctx->live, ctx->np_list, ctx->np_start, ctx->fin, nboxes, f.world_xf, ctx->box_data, ctx->sph_data, f.col_tag,
		ctx->flags, ctx->offs, S, ctx->staged, ctx->cfg.max_contacts, counts);

	// fine islands, active bodies, contact compaction (nudge.cpp:3788-4006)
	const u32 C = ctx->cfg.max_contacts;
	launch_grid(L, k_uf_init, GRID(B), ctx->parent, ctx->active, ctx->taint, kind, ctx->mom, B);
	if (ctx->nconn) launch_grid(L, k_uf_union_conn, GRID(ctx->nconn), ctx->parent, ctx->taint, ctx->idle, kind, ctx->conn, ctx->nconn);
	launch_grid(L, k_uf_union_contacts, GRID(C), ctx->parent, ctx->taint, ctx->idle, kind, ctx->staged.bodies, counts);
	launch_grid(L, k_uf_flatten_active, GRID(B), ctx->parent, ctx->active, ctx->taint, ctx->idle, kind, B);
	launch_grid(L, k_body_flags, GRID(B), ctx->parent, ctx->active, ctx->flags, B);
	nb_scan_reduce<1>(L, ctx->flags, S, nullptr, B, ctx->block_sums, counts + CNT_ACTIVE);
	launch_grid(L, k_active_scatter, NB_SCAN_GRID, ctx->flags, ctx->block_sums, ctx->active_idx, B);
	launch_grid(L, k_contact_flags, GRID(C), ctx->staged.bodies, ctx->staged.tags, ctx->parent, ctx->active, kind, ctx->flags, S, counts);
	nb_scan_reduce<2>(L, ctx->flags, S, counts + CNT_STAGED, 0, ctx->block_sums, counts + CNT_CONTACTS);  // -> CONTACTS, SLEEP_FINE
	launch_grid(L, k_contact_compact, NB_SCAN_GRID, ctx->staged, ctx->fin, ctx->flags, ctx->block_sums, S, ctx->sleeping, counts);

	// sort sleeping pairs (nudge.cpp:4008): key X | Y<<32, both below 2^tagbits
	launch_grid(L, k_copy_u64, GRID(C), ctx->sleeping, ctx->sb.keys[0], counts + CNT_SLEEPING);
	cur = nb_radix_sort(L, ctx->sb, counts + CNT_SLEEPING, 0, (int)ctx->tagbits, false, 0, 32, (int)(32 + ctx->tagbits));
	launch_grid(L, k_copy_u64, GRID(C), ctx->sb.keys[cur], ctx->sleeping, counts + CNT_SLEEPING);
	if (ctx->has_sensor) launch_sensor_overlaps(ctx, L);   // the scratch planes are free again here
	ctx->contacts_internal = true;
	CK(cudaGetLastError());
	return NB_OK;
}

int nb_apply_gravity_damping(nb_context* ctx, float time_step, float gravity, float damping, void* stream) {
	NB_RANGE("nb_apply_gravity_damping");
	JOIN_UPLOADS();   // first reader of the momentum rows in a step
	ctx->step_dt = time_step;
	const Launch L = mk_launch(ctx, stream);
	if (ctx->has_frc)   // the per-body force table (nb_force_api.cuh): the same stage, one launch
		launch_grid(L, k_body_forces, GRID(ctx->B), ctx->active_idx, kin_table(ctx), ctx->frc, ctx->xf, ctx->props, ctx->mom, ctx->idle,
			time_step, gravity, damping, ctx->counts);
	else
		launch_grid(L, k_gravity_damping, GRID(ctx->B), ctx->active_idx, kin_table(ctx), ctx->mom, time_step, gravity, damping, ctx->counts);
	CK(cudaGetLastError());
	return NB_OK;
}

// ---------------- contact cache ----------------
// The two halves of read_cached_impulses: (a) the tag ORDER of the contacts (one sort), (b) the cache LOOKUP of every contact's
// impulse plus the entries of sleeping pairs that survive the frame.
static int read_lookup(nb_context* ctx, void* stream) {
	const Launch L = mk_launch(ctx, stream);
	u32* counts = ctx->counts, *flags = ctx->flags;
	const u32 C = ctx->cfg.max_contacts, S = ctx->stride;
	launch_grid(L, k_cache_lookup, GRID(C), ctx->fin.tags, ctx->fin.features, ctx->cache_tags, ctx->cache_features, ctx->cache_data, ctx->impulses, counts);
	launch_grid(L, k_culled_flags, GRID(C), ctx->cache_tags, ctx->sleeping, flags, counts);
	nb_scan_reduce<1>(L, flags, S, counts + CNT_CACHE, 0, ctx->block_sums, counts + CNT_CULLED);
	launch_grid(L, k_culled_scatter, NB_SCAN_GRID, flags, ctx->block_sums, ctx->cache_tags, ctx->cache_features, ctx->cache_data,
		ctx->culled_tags, ctx->culled_features, ctx->culled_data, counts);
	CK(cudaGetLastError());
	return NB_OK;
}

static int read_sort(nb_context* ctx, void* stream) {
	const Launch L = mk_launch(ctx, stream);
	u32* counts = ctx->counts;
	const u32 C = ctx->cfg.max_contacts;
	// order contacts by tag: stable sort on the feature word, then on the pair word (nudge.cpp:4024-4044)
	int cur;
	if (ctx->contacts_internal && 2 * ctx->tagbits + 16 <= 64) {
		const u32 spread = (ctx->tagbits >= 3 && 2 * ctx->tagbits + 17 <= 64) ? 1u : 0u;
		launch_grid(L, k_tag_keys_packed, GRID(C), ctx->fin.tags, ctx->fin.features, ctx->sb.keys[0], ctx->sb.vals[0], ctx->tagbits, spread, counts);
		cur = nb_radix_sort(L, ctx->sb, counts + CNT_CONTACTS, 0, (int)(2 * ctx->tagbits + 16 + spread), true, 0);
	}
	else {  // contacts supplied through nb_upload_contacts (arbitrary feature words, tags beyond the colliders'), or tags wider than 24 bits
		const u32 pbits = ctx->contacts_internal ? ctx->tagbits : std::max(ctx->tagbits, ctx->upload_tagbits);
		launch_grid(L, k_tag_keys_feature, GRID(C), ctx->fin.features, ctx->sb.keys[0], ctx->sb.vals[0], counts);
		cur = nb_radix_sort(L, ctx->sb, counts + CNT_CONTACTS, 0, 32, true, 0);
		launch_grid(L, k_tag_keys_pair, GRID(C), ctx->fin.tags, ctx->sb.vals[cur], ctx->sb.keys[cur], pbits, counts);
		cur = nb_radix_sort(L, ctx->sb, counts + CNT_CONTACTS, 0, (int)(2 * pbits), true, cur);
	}
	launch_grid(L, k_copy_u32, GRID(C), ctx->sb.vals[cur], ctx->sorted, counts + CNT_CONTACTS);
	CK(cudaGetLastError());
	return NB_OK;
}

int nb_read_cached_impulses(nb_context* ctx, void* stream) {
	NB_RANGE("nb_read_cached_impulses");
	ctx->report_ok = false;
	NOT_AFTER_EDIT();
	int r = read_sort(ctx, stream); if (r) return r;
	return read_lookup(ctx, stream);
}

int nb_write_cached_impulses(nb_context* ctx, void* stream) {
	NB_RANGE("nb_write_cached_impulses");
	NOT_AFTER_EDIT();
	const u32 C = ctx->cfg.max_contacts;
	const uint4* s_old = ctx->has_sensor ? ctx->sensor_old.p : nullptr;
	const uint4* s_cur = ctx->has_sensor ? ctx->sensor_cur.p : nullptr;
	const Launch L = mk_launch(ctx, stream);
	if (ctx->ev_cap)   // the old cache is still intact here
		launch_contact_events(L, GRID(2 * (size_t)C), ctx->flags, ctx->stride, ctx->block_sums, ctx->cache_tags, ctx->sorted, ctx->fin,
							  ctx->culled_tags, ctx->impulses, s_old, s_cur, ctx->events.p, ctx->ev_cap, ctx->counts);
	if (ctx->has_sensor) launch_grid(L, k_sensor_keep, GRID(ctx->sensor_cap), ctx->sensor_cur.p, ctx->sensor_old.p, ctx->counts);
	launch_grid(L, k_cache_merge, GRID(C), ctx->sorted, ctx->fin.tags, ctx->fin.features, ctx->impulses,
		ctx->culled_tags, ctx->culled_features, ctx->culled_data, ctx->cache_tags, ctx->cache_features, ctx->cache_data, ctx->counts);
	CK(cudaGetLastError());
	return NB_OK;
}

// ---------------- contact events (nb_events.cuh) ----------------
int nb_enable_contact_events(nb_context* ctx, uint32_t capacity) {
	CK(cudaDeviceSynchronize());   // nothing in flight may still write the counters or the buffer
	ctx->ev_cap = 0;           // off until the buffer below exists (a failed allocation leaves events disabled)
	++ctx->graph_epoch;        // nb_step's graph re-records with or without the event launches
	GROW(ctx->events, capacity, cudaStreamLegacy);   // the device is idle: the stream it waits for does not matter
	CK(cudaMemset(ctx->counts + CNT_EV_COUNT, 0, 3 * sizeof(u32)));   // count, dropped, step
	CK(cudaDeviceSynchronize());
	ctx->ev_cap = capacity;
	return NB_OK;
}
int nb_download_contact_events(nb_context* ctx, nb_contact_event* host, uint32_t capacity, uint32_t* count, uint32_t* dropped, void* stream) {
	NB_RANGE("nb_download_contact_events");
	if (!ctx->ev_cap) { ctx->error = "contact events are not enabled (nb_enable_contact_events)"; return NB_ERR_ARGUMENT; }
	u32 c[CNT__COUNT];
	int r = get_counts(ctx, c, stream); if (r) return r;
	const u32 n = c[CNT_EV_COUNT], d = c[CNT_EV_DROPPED];
	if (count) *count = n;
	if (dropped) *dropped = d;
	if (n > capacity) { ctx->error = "host event buffer too small: " + std::to_string(n) + " events are stored"; return NB_ERR_CAPACITY; }
	if (n && !host) { ctx->error = "null host event buffer"; return NB_ERR_ARGUMENT; }
	D2H(host, ctx->events.p, n, nb_contact_event);
	CK(cudaMemsetAsync(ctx->counts + CNT_EV_COUNT, 0, 2 * sizeof(u32), (cudaStream_t)stream));   // count, dropped; in stream order
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	if (d) { ctx->error = std::to_string(d) + " contact events were dropped: the event buffer was full (raise the nb_enable_contact_events capacity or drain more often)"; return NB_ERR_OVERFLOW; }
	return NB_OK;
}

// ---------------- setup + solve ----------------
static void timing_begin(nb_context* ctx, cudaStream_t st) {
	if (!ctx->timing || ctx->capturing || ctx->tev_n >= 64) return;
	if (!ctx->tev_made) { for (int i = 0; i < 64; ++i) { cudaEventCreate(&ctx->tev[0][i]); cudaEventCreate(&ctx->tev[1][i]); } ctx->tev_made = true; }
	cudaEventRecord(ctx->tev[0][ctx->tev_n], st);
}
static void timing_end(nb_context* ctx, cudaStream_t st) {
	if (!ctx->timing || ctx->capturing || ctx->tev_n >= 64) return;
	cudaEventRecord(ctx->tev[1][ctx->tev_n++], st);
}

// Shared-memory stages of k_jacobi_sweep for the current body count: two tiles per CTA in flight once the body arrays (64 B per body:
// velocities + accumulators) take a large share of L2, else one stage and more CTAs.
static int jacobi_stages(const nb_context* ctx) { return ctx->B > 600000u ? 2 : 1; }

// throughput mode: the warm start and the sweeps as Jacobi passes (k_jacobi_sweep + k_jacobi_apply per pass), nb_jacobi.cuh
static int launch_solve_jacobi(nb_context* ctx, bool warm, u32 sweeps, cudaStream_t st) {
	const Launch L = mk_launch(ctx, st);
	Rows R = ctx->rows;
	const u32 B = ctx->B;
	launch_grid(L, k_mw_in, GRID(B), B, ctx->mom, ctx->mw);
	const int stages = jacobi_stages(ctx);
	if (warm) {
		if (stages == 1) launch(L, k_jacobi_sweep<true, 1>, ctx->jacobi_blocks1, NJ_TILE, sizeof(JacobiSmem<1>), R, ctx->impulses, ctx->mw, ctx->jd, ctx->counts);
		else launch(L, k_jacobi_sweep<true, 2>, ctx->jacobi_blocks2, NJ_TILE, sizeof(JacobiSmem<2>), R, ctx->impulses, ctx->mw, ctx->jd, ctx->counts);
		launch_grid(L, k_jacobi_apply, GRID(B), B, ctx->mw, ctx->jd, ctx->jcnt);
	}
	for (u32 w = 0; w < sweeps; ++w) {
		timing_begin(ctx, st);
		if (stages == 1) launch(L, k_jacobi_sweep<false, 1>, ctx->jacobi_blocks1, NJ_TILE, sizeof(JacobiSmem<1>), R, ctx->impulses, ctx->mw, ctx->jd, ctx->counts);
		else launch(L, k_jacobi_sweep<false, 2>, ctx->jacobi_blocks2, NJ_TILE, sizeof(JacobiSmem<2>), R, ctx->impulses, ctx->mw, ctx->jd, ctx->counts);
		timing_end(ctx, st);
		launch_grid(L, k_jacobi_apply, GRID(B), B, ctx->mw, ctx->jd, ctx->jcnt);
	}
	launch_grid(L, k_mw_out, GRID(B), B, ctx->mom, ctx->mw, sweeps > 0);
	return NB_OK;
}

// The solver on the bodies' working rows: loaded with the warm start applied (k_warm_start, from the shares k_build_rows left) or as
// they are (k_mw_in), then `sweeps` sweeps in one k_solve launch (none: the warm start alone), then stored back (k_mw_out).
static int launch_solve(nb_context* ctx, bool warm, u32 sweeps, cudaStream_t st) {
	if (ctx->solver_mode == NB_SOLVER_THROUGHPUT) return launch_solve_jacobi(ctx, warm, sweeps, st);
	const Launch L = mk_launch(ctx, st);
	const u32 B = ctx->B;
	if (warm) launch_grid(L, k_warm_start, GRID(B), B, ctx->mom, ctx->chain_start, ctx->chain_len, ctx->warm, ctx->mw);
	else launch_grid(L, k_mw_in, GRID(B), B, ctx->mom, ctx->mw);
	if (sweeps) {
		timing_begin(ctx, st);
		CK(launch_coop(L, ctx->has_kin ? k_solve_kin : k_solve, ctx->coop_blocks_solve, NB_BLOCK, 0, ctx->rows, ctx->mw, sweeps, NB_SOLVE_BACKOFF_NS, ctx->counts));
		timing_end(ctx, st);
	}
	launch_grid(L, k_mw_out, GRID(B), B, ctx->mom, ctx->mw, sweeps > 0);
	return NB_OK;
}

// The contact rows of the current contact set, everything of nb_setup_contact_constraints before the warm start.
static int build_contact_rows(nb_context* ctx, cudaStream_t st) {
	const Launch L = mk_launch(ctx, st);
	u32* counts = ctx->counts;
	const u32 C = ctx->cfg.max_contacts, S = ctx->stride, B = ctx->B;
	const uint8_t* kind = kin_table(ctx);
	launch_grid(L, k_inertia, GRID(B), B, ctx->xf, ctx->props, kind, ctx->inertia, ctx->mom);
	if (ctx->solver_mode == NB_SOLVER_THROUGHPUT) {
		// no batch schedule, no per-body chains: slots in tag order, per-body contact counts for the mass split, split rows
		CK(cudaMemsetAsync(ctx->rows.contact, 0xff, sizeof(u32) * ctx->cstride, st));
		CK(cudaMemsetAsync(ctx->jcnt, 0, sizeof(u32) * B, st));
		launch_grid(L, k_jacobi_prepare, GRID(C), ctx->sorted, ctx->fin.bodies, kind, ctx->jcnt, ctx->rows, ctx->cstride, counts);
		launch_grid(L, k_build_rows<true>, GRID(ctx->cstride), ctx->fin.data, ctx->fin.bodies, ctx->xf, ctx->inertia, ctx->mom, kind, ctx->rows, counts, ctx->jcnt,
			nullptr, nullptr, nullptr);
		return NB_OK;
	}
	launch_grid(L, k_sched_prep, GRID(C), ctx->sorted, ctx->fin.bodies, kind, ctx->cab, ctx->back, ctx->sched_empty, counts);
	// the scheduler replay in segments (nb_solver.cuh above k_schedule, DESIGN §2.7): speculative runs, the joins of every segment
	// from every run of the previous one, then per bucket the chain of picked runs (or the sequential replay if it broke), and the
	// merge of the picked joins and runs
	launch(L, k_sched_spec, dim3(16, NB_SCHED_SEGS, 8), 32, 0, ctx->cab, ctx->back, ctx->sched_slot_v, ctx->sched_empty, C, ctx->sched_state, counts);
	launch(L, k_sched_join, dim3(16, NB_SCHED_SEGS - 1, 8), 32, 0, ctx->cab, ctx->back, ctx->sched_join_slot, ctx->sched_empty, ctx->sched_state, ctx->sched_pick, counts);
	launch(L, k_schedule, 16, 32, 0, ctx->cab, ctx->back, ctx->slot_of, ctx->slot_done, ctx->slot_left, ctx->slots_per_bucket,
		ctx->flags, ctx->left_count, ctx->sched_spill_ent, ctx->sched_spill_uid, ctx->sched_spill_cap, ctx->sched_state, ctx->sched_pick, ctx->sched_pick_res, counts);
	launch_grid(L, k_sched_merge, GRID(C), ctx->slot_of, ctx->sched_slot_v, C, ctx->sched_join_slot, ctx->slot_done, ctx->slots_per_bucket, ctx->flags,
		ctx->sched_pick_res, counts);
	nb_scan<1>(L, ctx->flags, ctx->offs, S, counts + CNT_CONTACTS, 0, ctx->block_sums, counts + CNT_FULL_BATCHES);
	// per-body chains (nb_solver.cuh, above k_chain_alloc): count, segment, scatter, rank.  chain_len is zero for bodies without
	// entries, which nb_shard_step's dataflow solve relies on.  The entries go through sb.keys[0], free until the next collide.
	CK(cudaMemsetAsync(ctx->rows.contact, 0xff, sizeof(u32) * ctx->cstride, st));
	CK(cudaMemsetAsync(ctx->chain_len, 0, sizeof(u32) * B, st));
	launch_grid(L, k_batch_index, GRID(C), ctx->sorted, ctx->fin.bodies, ctx->slot_of, ctx->slot_done, ctx->slot_left, ctx->slots_per_bucket,
		ctx->offs, ctx->left_count, kind, ctx->batch_of, ctx->slot_idx, ctx->rows.contact, ctx->cstride, ctx->chain_len, counts);
	launch_grid(L, k_chain_alloc, GRID(B), B, ctx->chain_len, ctx->chain_start, counts);
	launch_grid(L, k_chain_scatter, GRID(C), ctx->sorted, ctx->fin.bodies, kind, ctx->batch_of, ctx->chain_start, ctx->sb.keys[0], counts);
	launch_grid(L, k_chain_rank, GRID(2 * C), ctx->sorted, ctx->fin.bodies, kind, ctx->batch_of, ctx->slot_idx, ctx->chain_start, ctx->chain_len, ctx->sb.keys[0], ctx->rows.wait, ctx->cstride, counts);
	launch_grid(L, k_build_rows<false>, GRID(ctx->cstride), ctx->fin.data, ctx->fin.bodies, ctx->xf, ctx->inertia, ctx->mom, kind, ctx->rows, counts, nullptr,
		ctx->impulses, ctx->chain_start, ctx->warm);
	return NB_OK;
}

int nb_setup_contact_constraints(nb_context* ctx, void* stream) {
	NB_RANGE("nb_setup_contact_constraints");
	ctx->report_ok = false;
	NOT_AFTER_EDIT();
	JOIN_UPLOADS();
	if (ctx->jset.n && !(ctx->step_dt > 0.0f)) { ctx->error = "joints need the step's time step: call nb_apply_gravity_damping after nb_collide"; return NB_ERR_ARGUMENT; }
	cudaStream_t st = (cudaStream_t)stream;
	int r = build_contact_rows(ctx, st); if (r) return r;
	// the warm start (nudge.cpp:4563-4632), then the user rows' accumulated impulses, then the joints' rows and theirs
	if ((r = launch_solve(ctx, true, 0, st))) return r;
	if (ctx->urow_set.n && (r = launch_user_rows(ctx, 1, st))) return r;
	if (ctx->jset.n && (r = launch_joints(ctx, &ctx->step_dt, st))) return r;
	CK(cudaGetLastError());
	return NB_OK;
}

int nb_apply_impulses(nb_context* ctx, uint32_t sweeps, void* stream) {
	NB_RANGE("nb_apply_impulses");
	ctx->report_ok = false;
	NOT_AFTER_EDIT();
	JOIN_UPLOADS();
	if (!sweeps) return NB_OK;
	cudaStream_t st = (cudaStream_t)stream;
	if (ctx->urow_set.n || ctx->jset.n) {   // user rows, then joints, run after EVERY sweep (example/main.cpp:314-317): one sweep per solver launch
		for (uint32_t w = 0; w < sweeps; ++w) {
			int r = launch_solve(ctx, false, 1, st); if (r) return r;
			if (ctx->urow_set.n && (r = launch_user_rows(ctx, 0, st))) return r;
			if (ctx->jset.n && (r = launch_joints(ctx, nullptr, st))) return r;
		}
		return NB_OK;
	}
	int r = launch_solve(ctx, false, sweeps, st); if (r) return r;
	CK(cudaGetLastError());
	return NB_OK;
}

int nb_update_cached_impulses(nb_context* ctx, void* stream) {
	NB_RANGE("nb_update_cached_impulses");
	NOT_AFTER_EDIT();
	launch_grid(mk_launch(ctx, stream), k_update_impulses, GRID(ctx->cstride), ctx->rows, ctx->impulses, ctx->counts);
	CK(cudaGetLastError());
	ctx->report_ok = true;   // the contact impulse reports read this step's contacts, impulses and rows
	return NB_OK;
}

int nb_advance(nb_context* ctx, float time_step, void* stream) {
	NB_RANGE("nb_advance");
	NOT_AFTER_EDIT();
	if (!ctx->ccd.empty() && !ctx->in_step) {   // the cast walks the last collide's grid, which must describe this step's poses
		ctx->error = "nb_advance: a continuous-collision set (nb_upload_ccd_bodies) needs an nb_collide since the last nb_advance";
		return NB_ERR_ARGUMENT;
	}
	JOIN_UPLOADS();
	const Launch L = mk_launch(ctx, stream);
	if (ctx->ccd.empty())
		launch_grid(L, k_advance<false>, GRID(ctx->B), ctx->active_idx, ctx->xf, ctx->mom, ctx->idle, time_step, ctx->counts, (const float*)nullptr);
	else {   // the casts (nb_ccd_api.cuh), then the advance with their factors
		if (int r = launch_ccd(ctx, L, time_step)) return r;
		launch_grid(L, k_advance<true>, GRID(ctx->B), ctx->active_idx, ctx->xf, ctx->mom, ctx->idle, time_step, ctx->counts, (const float*)ctx->ccd_t);
	}
	ctx->in_step = false;
	CK(cudaGetLastError());
	return NB_OK;
}

// nb_step's solve section: nb_setup_contact_constraints + nb_apply_impulses, or without user rows or joints between the sweeps, the row build and
// the warm start straight into the sweeps' working rows (the same arithmetic in the same order).
static int step_solve(nb_context* ctx, uint32_t iterations, void* stream) {
	if (iterations > 0 && !ctx->urow_set.n && !ctx->jset.n) {
		cudaStream_t st = (cudaStream_t)stream;
		int r = build_contact_rows(ctx, st); if (r) return r;
		if ((r = launch_solve(ctx, true, iterations, st))) return r;
		CK(cudaGetLastError());
		return NB_OK;
	}
	int r = nb_setup_contact_constraints(ctx, stream);
	return r ? r : nb_apply_impulses(ctx, iterations, stream);
}

// One sub-step (example/main.cpp:274-328), as a CUDA graph on a capturable stream (61 launches in parity mode, 3 more with contact events,
// 6 more with sensor colliders, 1 more with a continuous-collision set).
int nb_step(nb_context* ctx, float time_step, uint32_t iterations, float gravity, float damping, void* stream) {
	NB_RANGE("nb_step");
	ctx->capture_joined = false;   // a capture records the event-wait node for nb_upload_bodies' side copy
	ctx->scene_edited = false;     // the step begins with nb_collide (also when its graph is replayed)
	const int r = run_graphed(ctx, ctx->graph, (cudaStream_t)stream, time_step, iterations, gravity, damping, 0, 0,
							  [&] { return step_body(ctx, time_step, gravity, damping, stream, [&] { return step_solve(ctx, iterations, stream); }); });
	if (r == NB_OK) { ctx->in_step = false; ctx->report_ok = true; }   // the step ended with nb_advance (also when its graph was replayed)
	return r;
}

// ---------------- streams for hosts that do not link the CUDA runtime themselves ----------------
void* nb_stream_create(nb_context* ctx) {
	cudaStream_t s = nullptr;
	if (cudaSetDevice(ctx->cfg.device) != cudaSuccess || cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) { ctx->error = "cudaStreamCreate failed"; return nullptr; }
	return (void*)s;
}
void nb_stream_destroy(nb_context* ctx, void* stream) { (void)ctx; if (stream) { cudaStreamSynchronize((cudaStream_t)stream); cudaStreamDestroy((cudaStream_t)stream); } }
int nb_stream_synchronize(nb_context* ctx, void* stream) { CK(cudaStreamSynchronize((cudaStream_t)stream)); return NB_OK; }

// ---------------- solver mode and kernel timing ----------------
int nb_set_solver_mode(nb_context* ctx, int mode) {
	if (mode != NB_SOLVER_PARITY && mode != NB_SOLVER_THROUGHPUT) { ctx->error = "unknown solver mode"; return NB_ERR_ARGUMENT; }
	ctx->solver_mode = mode;
	return NB_OK;
}
int nb_get_solver_mode(const nb_context* ctx) { return ctx->solver_mode; }

// CUDA events around every launch of the dominant solver kernel (k_solve in parity mode, k_jacobi_sweep in throughput mode) while
// enabled; plain launches only (the stage calls, or nb_step with NB_GRAPH=0).  nb_debug_timing synchronises the stream and returns
// the number of timed launches and their summed duration, then clears the list.
int nb_debug_timing_enable(nb_context* ctx, int on) { ctx->timing = on; ctx->tev_n = 0; return NB_OK; }
int nb_debug_timing(nb_context* ctx, uint32_t* launches, float* total_ms, void* stream) {
	CK(cudaStreamSynchronize((cudaStream_t)stream));
	float sum = 0.0f;
	for (int i = 0; i < ctx->tev_n; ++i) { float ms = 0.0f; CK(cudaEventElapsedTime(&ms, ctx->tev[0][i], ctx->tev[1][i])); sum += ms; }
	if (launches) *launches = (uint32_t)ctx->tev_n;
	if (total_ms) *total_ms = sum;
	ctx->tev_n = 0;
	return NB_OK;
}

// ---------------- parity-test introspection ----------------
int nb_debug_read(nb_context* ctx, const char* name, void* dst, size_t max_bytes, size_t* bytes, void* stream) {
	u32 c[CNT__COUNT];
	int r = get_counts(ctx, c, stream); if (r) return r;
	const u32 K = ctx->nboxes + ctx->nspheres;
	struct Entry { const char* name; const void* ptr; size_t bytes; };
	const Entry table[] = {
		{ "counts", ctx->counts, sizeof(u32) * CNT__COUNT },
		{ "order", ctx->front.order, sizeof(u32) * K },
		{ "aabb_min", ctx->front.aabb_min, sizeof(float4) * K },
		{ "aabb_max", ctx->front.aabb_max, sizeof(float4) * K },
		{ "world_xf", ctx->front.world_xf, sizeof(nb_transform) * K },
		{ "pair_keys", ctx->pair_keys_debug, sizeof(u64) * (ctx->pair_keys_debug ? c[CNT_PAIRS] : 0) },
		{ "live", ctx->live, sizeof(uint2) * c[CNT_LIVE_TOTAL] },
		{ "sorted", ctx->sorted, sizeof(u32) * c[CNT_CONTACTS] },
		{ "impulses", ctx->impulses, sizeof(float4) * c[CNT_CONTACTS] },
		{ "culled_tags", ctx->culled_tags, sizeof(u64) * c[CNT_CULLED] },
		{ "culled_features", ctx->culled_features, sizeof(u32) * c[CNT_CULLED] },
		{ "culled_data", ctx->culled_data, sizeof(float4) * c[CNT_CULLED] },
		{ "cab", ctx->cab, sizeof(uint2) * c[CNT_CONTACTS] },
		{ "batch_of", ctx->batch_of, sizeof(u32) * c[CNT_CONTACTS] },
		{ "slot_idx", ctx->slot_idx, sizeof(u32) * c[CNT_CONTACTS] },
		{ "row_contact", ctx->rows.contact, sizeof(u32) * 8 * c[CNT_BATCHES] },
		{ "row_a", ctx->rows.a, sizeof(u32) * 8 * c[CNT_BATCHES] },
		{ "row_b", ctx->rows.b, sizeof(u32) * 8 * c[CNT_BATCHES] },
		{ "row_wait", ctx->rows.wait, sizeof(uint2) * 2 * (size_t)ctx->cstride },
		{ "row_planes", ctx->rows.plane, sizeof(float) * (size_t)ROW_PLANES * ctx->cstride },
		{ "row_states", ctx->rows.state, sizeof(float) * 3 * (size_t)ctx->cstride },
		{ "inertia", ctx->inertia, sizeof(float4) * 2 * ctx->B },
		{ "row_planes_all", ctx->rows.plane, sizeof(float) * (size_t)ROW_PLANES_TOTAL * ctx->cstride },
		{ "body_contacts", ctx->jcnt, sizeof(u32) * ctx->B },
		{ "kind", ctx->kind, ctx->has_kin ? (size_t)ctx->B : 0 },
		{ "joint_rows", ctx->jrows.p, sizeof(nb_constraint_row) * (size_t)ctx->jset.nrows },   // in table order: by joint level, upload order within one
		{ "joint_drives", ctx->drives.table.p, ctx->drives.set.n ? sizeof(JointDrive) * (size_t)ctx->jset.n : 0 },
		{ "joint_drive_rows", ctx->drives.rows.p, sizeof(nb_constraint_row) * (size_t)ctx->drives.set.nrows },   // per driven joint in table order
		{ "joint_springs", ctx->springs.table.p, ctx->springs.set.n ? sizeof(JointSpring) * (size_t)ctx->jset.n : 0 },
		{ "joint_spring_rows", ctx->springs.rows.p, sizeof(nb_constraint_row) * (size_t)ctx->springs.set.nrows },   // per sprung joint in table order
		{ "sensor_pairs", ctx->sensor_keys.p, sizeof(u64) * (ctx->has_sensor ? std::min(c[CNT_SENSOR_PAIRS], ctx->sensor_cap) : 0) },
		{ "ccd_hits", ctx->ccd_hits.p, sizeof(uint2) * ctx->ccd.size() },   // per entry of the last advance, in set order: (bits of t, collider)
	};
	if (!strcmp(name, "row_stride")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = ctx->cstride; if (bytes) *bytes = 4; return NB_OK; }
	if (!strcmp(name, "graph_active")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = ctx->graph.exec != nullptr; if (bytes) *bytes = 4; return NB_OK; }
	// how many times a step graph (nb_step, nb_shard_step) was captured since nb_create
	if (!strcmp(name, "graph_records")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = (u32)ctx->graph_records; if (bytes) *bytes = 4; return NB_OK; }
	// the device bytes the context and its snapshots hold now, as a uint64_t
	if (!strcmp(name, "device_bytes")) { if (max_bytes < 8) return NB_ERR_ARGUMENT; *(uint64_t*)dst = ctx->device_bytes; if (bytes) *bytes = 8; return NB_OK; }
	// the scene queries' own counters (0 before the first query): rays, overlap queries and shape casts that tested every collider instead
	// of walking the grid, summed over the context's calls, and the grid level of the last query's build
	const struct { const char* name; u32 slot; } query_counters[] = {
		{ "ray_fallbacks", CNT_RAY_FALLBACKS }, { "ray_grid_level", CNT_GRID_LEVEL }, { "overlap_fallbacks", CNT_OVERLAP_FALLBACKS },
		{ "shapecast_fallbacks", CNT_SHAPECAST_FALLBACKS },
	};
	for (const auto& e : query_counters)
		if (!strcmp(name, e.name)) {
			if (max_bytes < 4) return NB_ERR_ARGUMENT;
			u32 v = 0;
			if (ctx->query.ready) {
				CK(cudaMemcpyAsync(&v, ctx->query.counts + e.slot, 4, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
				CK(cudaStreamSynchronize((cudaStream_t)stream));
			}
			*(u32*)dst = v; if (bytes) *bytes = 4; return NB_OK;
		}
	// continuous collision: casts of the context's advances that tested every collider instead of walking the grid
	if (!strcmp(name, "ccd_fallbacks")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = c[CNT_CCD_FALLBACKS]; if (bytes) *bytes = 4; return NB_OK; }
	if (!strcmp(name, "sched_fallback")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = c[CNT_SCHED_FALLBACK]; if (bytes) *bytes = 4; return NB_OK; }
	// the last collide's broadphase: the grid level (cell edge 2^level quantised units) and how many colliders went to k_large_pairs
	if (!strcmp(name, "grid_level")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = c[CNT_GRID_LEVEL]; if (bytes) *bytes = 4; return NB_OK; }
	if (!strcmp(name, "grid_large")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = c[CNT_LARGE]; if (bytes) *bytes = 4; return NB_OK; }
	if (!strcmp(name, "kbits")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = ctx->kbits; if (bytes) *bytes = 4; return NB_OK; }
	if (!strcmp(name, "tagbits")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = ctx->tagbits; if (bytes) *bytes = 4; return NB_OK; }
	// the k_jacobi_sweep variant (shared-memory stages) and grid that throughput mode launches at the current body count
	if (!strcmp(name, "jacobi_stages")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = (u32)jacobi_stages(ctx); if (bytes) *bytes = 4; return NB_OK; }
	if (!strcmp(name, "jacobi_blocks")) { if (max_bytes < 4) return NB_ERR_ARGUMENT; *(u32*)dst = (u32)(jacobi_stages(ctx) == 2 ? ctx->jacobi_blocks2 : ctx->jacobi_blocks1); if (bytes) *bytes = 4; return NB_OK; }
	for (size_t i = 0; i < sizeof(table) / sizeof(table[0]); ++i)
		if (!strcmp(name, table[i].name)) {
			if (bytes) *bytes = table[i].bytes;
			if (!dst) return NB_OK;
			if (table[i].bytes > max_bytes) { ctx->error = "debug buffer too small"; return NB_ERR_CAPACITY; }
			CK(cudaMemcpyAsync(dst, table[i].ptr, table[i].bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
			CK(cudaStreamSynchronize((cudaStream_t)stream));
			return NB_OK;
		}
	ctx->error = std::string("unknown debug buffer ") + name;
	return NB_ERR_ARGUMENT;
}

// Keeps a copy of the sorted broadphase pair list for nb_debug_read("pair_keys") (one extra copy kernel per collide).
int nb_debug_enable(nb_context* ctx, int on) {
	if (on) ALLOC(ctx->pair_keys_debug, ctx->cfg.max_pairs);
	ctx->debug = on;
	return NB_OK;
}

// Runs the device radix sort / scan on host data (unit tests of the primitives).
int nb_debug_sort(nb_context* ctx, uint64_t* keys, uint32_t* vals, uint32_t n, int begin_bit, int end_bit) {
	if (n > ctx->sort_cap) { ctx->error = "too many keys"; return NB_ERR_CAPACITY; }
	Launch L = mk_launch(ctx, nullptr);
	CK(cudaMemcpy(ctx->sb.keys[0], keys, (size_t)n * 8, cudaMemcpyHostToDevice));
	if (vals) CK(cudaMemcpy(ctx->sb.vals[0], vals, (size_t)n * 4, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(ctx->counts + CNT_SCRATCH1, &n, 4, cudaMemcpyHostToDevice));
	int cur = nb_radix_sort(L, ctx->sb, ctx->counts + CNT_SCRATCH1, begin_bit, end_bit, vals != nullptr, 0);
	CK(cudaMemcpy(keys, ctx->sb.keys[cur], (size_t)n * 8, cudaMemcpyDeviceToHost));
	if (vals) CK(cudaMemcpy(vals, ctx->sb.vals[cur], (size_t)n * 4, cudaMemcpyDeviceToHost));
	return NB_OK;
}
int nb_debug_scan(nb_context* ctx, uint32_t* data, uint32_t n, uint32_t* total) {
	if (n > ctx->stride) { ctx->error = "too many values"; return NB_ERR_CAPACITY; }
	Launch L = mk_launch(ctx, nullptr);
	CK(cudaMemcpy(ctx->flags, data, (size_t)n * 4, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(ctx->counts + CNT_SCRATCH1, &n, 4, cudaMemcpyHostToDevice));
	nb_scan<1>(L, ctx->flags, ctx->offs, ctx->stride, ctx->counts + CNT_SCRATCH1, 0, ctx->block_sums, ctx->counts + CNT_SCRATCH0);
	CK(cudaMemcpy(data, ctx->offs, (size_t)n * 4, cudaMemcpyDeviceToHost));
	CK(cudaMemcpy(total, ctx->counts + CNT_SCRATCH0, 4, cudaMemcpyDeviceToHost));
	return NB_OK;
}

int nb_debug_rcp(nb_context* ctx, const float* x, float* y, uint32_t n, int rsq) {
	float* dx = (float*)ctx->sb.keys[0]; float* dy = (float*)ctx->sb.keys[1];
	if ((size_t)n * 4 > (size_t)ctx->sort_cap * 8) { ctx->error = "too many probes"; return NB_ERR_CAPACITY; }
	CK(cudaMemcpy(dx, x, (size_t)n * 4, cudaMemcpyHostToDevice));
	launch_grid(mk_launch(ctx, nullptr), k_debug_rcp, GRID(n), dx, dy, n, rsq);
	CK(cudaMemcpy(y, dy, (size_t)n * 4, cudaMemcpyDeviceToHost));
	return NB_OK;
}

}

#include "nb_force_api.cuh"   // before nb_state_api.cuh, whose version-5 section uses its entry checks
#include "nb_shard_api.cuh"
#include "nb_rows_api.cuh"
#include "nb_joint_api.cuh"
#include "nb_state_api.cuh"   // after nb_joint_api.cuh, whose joints its version-6 section holds
#include "nb_render_api.cuh"
#include "nb_impulse_api.cuh"
#include "nb_spawn_api.cuh"
#include "nb_snapshot_api.cuh"
#include "nb_query_api.cuh"
#include "nb_ccd_api.cuh"     // after nb_query_api.cuh, whose walk and sphere cast k_ccd runs
#include "nb_body_state_api.cuh"   // after nb_spawn_api.cuh, whose wake a pose set runs
#include "nb_contact_report_api.cuh"
