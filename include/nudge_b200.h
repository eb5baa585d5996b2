/* nudge_b200 — C ABI of the H100-native (sm_90a) rigid-body simulation step (drop-in for rasmusbarr/nudge's hot path).
 *
 * Every entry point replaces one reference interface (file:line into /root/reference):
 *
 *   nb_collide                      <- nudge::collide                    nudge.h:134, nudge.cpp:3000-4009
 *   nb_read_cached_impulses         <- nudge::read_cached_impulses       nudge.h:136, nudge.cpp:4021-4108
 *   nb_write_cached_impulses        <- nudge::write_cached_impulses      nudge.h:138, nudge.cpp:4110-4158
 *   nb_setup_contact_constraints    <- nudge::setup_contact_constraints  nudge.h:140, nudge.cpp:4170-4638
 *   nb_apply_impulses               <- nudge::apply_impulses             nudge.h:142, nudge.cpp:4640-4855
 *   nb_update_cached_impulses       <- nudge::update_cached_impulses     nudge.h:144, nudge.cpp:4857-4884
 *   nb_advance                      <- nudge::advance                    nudge.h:146, nudge.cpp:4886-4926
 *   nb_apply_gravity_damping        <- the user loop of example/main.cpp:291-305
 *   nb_step                         <- simulate(), example/main.cpp:274-328 (one sub-step)
 *   nb_upload_connections           <- BodyConnections of nudge::collide  nudge.h:108-111, example/main.cpp:285
 *   nb_upload_contacts              <- "custom contacts can be added here" example/main.cpp:288
 *   nb_upload_constraint_rows       <- "custom constraint impulses"        example/main.cpp:316
 *   nb_upload_joints                <- no reference counterpart: the rows an application would rebuild for example/main.cpp:316 every step
 *   nb_upload_joint_drives /
 *   nb_upload_joint_springs         <- no reference counterpart: limits, motors and PD springs an application would build as rows every step
 *   nb_instance_matrices            <- the draw loops of render()          example/main.cpp:224-268 (helpers :53-110)
 *   nb_download_contact_events      <- a host diff of ContactData / ContactCache between steps (collision callbacks)
 *   nb_upload_collision_filters     <- no reference counterpart (the reference collides every overlapping pair)
 *   nb_upload_sensors               <- no reference counterpart (the reference has no trigger volumes)
 *   nb_upload_kinematic_bodies      <- no reference counterpart (the reference's only non-dynamic body is the static world, body 0)
 *   nb_apply_body_impulses          <- no reference counterpart: the application's edit of BodyData between calls
 *   nb_apply_radial_impulse         <- no reference counterpart: the application's edit of BodyData between calls
 *   nb_add_bodies / nb_remove_bodies <- no reference counterpart: the application's edit of its caller-owned arrays between steps
 *   nb_save_state / nb_load_state   <- the caller-owned PODs               nudge.h:73-129
 *   nb_snapshot_*                   <- no reference counterpart: the application's copy of its caller-owned arrays, kept in HBM
 *   nb_raycast, nb_overlap,
 *   nb_shapecast                    <- no reference counterpart (the reference has no scene queries)
 *   nb_get_body_states /
 *   nb_set_body_states              <- no reference counterpart: the application's read and edit of BodyData between calls
 *   nb_get_body_contact_impulses /
 *   nb_get_contact_pair_impulses    <- no reference counterpart: the application's host sums over ContactData and ContactCache after a step
 *   nb_shard_*                      <- no reference counterpart (the reference is single threaded): SURVEY.md section 8e
 *
 * Data layout: the reference's caller-owned SoA structs (nudge.h:29-129) with every index-carrying field
 * widened to 32 bits (the reference caps at 8192 colliders / 65535 bodies, nudge.cpp:3010, nudge.h:68-71):
 *
 *   BodyPair{uint16 a,b}                             -> nb_body_pair{uint32 a,b}
 *   collider tag uint16                              -> uint32
 *   contact tag uint64 = feature | A<<32 | B<<48     -> tags[i] = A | (uint64)B<<32 ; features[i] = feature
 *   sleeping pair uint32 = X | Y<<16                 -> uint64 = X | (uint64)Y<<32
 *   ActiveBodies.indices uint16                      -> uint32
 *
 * The simulation state is DEVICE RESIDENT inside an nb_context (HBM); nb_upload_* / nb_download_* move the
 * caller's host arrays across.  All calls are asynchronous on the given CUDA stream unless stated; no call
 * falls back to the CPU — if the GPU or the CUDA extension is missing, nb_create fails.
 * The uint16 drop-in with the exact nudge.h signatures lives in nudge_b200/csrc/nudge_compat.cpp.
 *
 * Return value: 0 on success, otherwise a negative nb_status; nb_last_error() gives the text.
 */
#ifndef NUDGE_B200_H
#define NUDGE_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { float position[3]; uint32_t body; float rotation[4]; } nb_transform;          /* nudge.h:34-38 */
typedef struct { float inertia_inverse[3]; float mass_inverse; } nb_body_properties;            /* nudge.h:40-43 */
typedef struct { float velocity[3]; float unused0; float angular_velocity[3]; float unused1; } nb_body_momentum; /* nudge.h:45-50 */
typedef struct { float radius; } nb_sphere_collider;                                            /* nudge.h:52-54 */
typedef struct { float size[3]; float unused; } nb_box_collider;                                /* nudge.h:56-59 */
typedef struct { float position[3]; float penetration; float normal[3]; float friction; } nb_contact; /* nudge.h:61-66 */
typedef struct { uint32_t a, b; } nb_body_pair;                                                 /* nudge.h:68-71, widened */
typedef struct { float impulse[3]; float unused; } nb_cached_impulse;                           /* nudge.h:109-112 */

typedef struct {                                                                                /* nudge.h:73-82 */
	nb_contact* data; nb_body_pair* bodies; uint64_t* tags; uint32_t* features;
	uint32_t capacity, count;
	uint64_t* sleeping_pairs; uint32_t sleeping_count;
} nb_contact_data;

typedef struct { uint32_t* tags; nb_box_collider* data; nb_transform* transforms; uint32_t count; } nb_box_colliders;
typedef struct { uint32_t* tags; nb_sphere_collider* data; nb_transform* transforms; uint32_t count; } nb_sphere_colliders;
typedef struct { nb_box_colliders boxes; nb_sphere_colliders spheres; } nb_collider_data;        /* nudge.h:84-98 */
typedef struct { nb_transform* transforms; nb_body_properties* properties; nb_body_momentum* momentum; uint8_t* idle_counters; uint32_t count; } nb_body_data; /* nudge.h:100-106 */
typedef struct { nb_body_pair* data; uint32_t count; } nb_body_connections;                      /* nudge.h:108-111 */
typedef struct { uint64_t* tags; uint32_t* features; nb_cached_impulse* data; uint32_t capacity, count; } nb_contact_cache; /* nudge.h:114-119 */
typedef struct { uint32_t* indices; uint32_t capacity, count; } nb_active_bodies;                /* nudge.h:121-125 */

typedef struct nb_context nb_context;

typedef struct {
	uint32_t max_bodies, max_boxes, max_spheres, max_connections;
	uint32_t max_pairs;     /* broadphase pairs (about 7 per collider in a pile); 0 = 16 per collider */
	uint32_t max_contacts;  /* also the contact-cache capacity; 0 = 24 per body */
	int device;             /* CUDA device ordinal */
} nb_config;

enum nb_status { NB_OK = 0, NB_ERR_CUDA = -1, NB_ERR_CAPACITY = -2, NB_ERR_ARGUMENT = -3, NB_ERR_OVERFLOW = -4 };

/* Device counters of the last step (copied by nb_download_counts; synchronises the stream). */
typedef struct {
	uint32_t pairs, live_pairs, contacts, sleeping, active, cache, culled, batches, levels, overflow;
} nb_counts;

int nb_create(const nb_config* config, nb_context** out);
void nb_destroy(nb_context* ctx);
const char* nb_last_error(const nb_context* ctx);

/* Host <-> HBM.  Counts in the structs say how many rows to move; pointers are HOST pointers. */
/* nb_upload_bodies is asynchronous (keep the host arrays unchanged until the next synchronising call; pin them to get real overlap): on a created
 * stream the momentum and property rows travel on the library's own copy stream while `stream` goes on with the collision stage, and whatever
 * reads them first on `stream` is ordered after the copy by the library (NB_COPY_OVERLAP=0 disables it).  Use ONE stream per context. */
int nb_upload_bodies(nb_context*, const nb_body_data* host, void* stream);
int nb_upload_colliders(nb_context*, const nb_collider_data* host, void* stream);
int nb_upload_connections(nb_context*, const nb_body_connections* host, void* stream);
int nb_upload_cache(nb_context*, const nb_contact_cache* host, void* stream);
/* nb_upload_contacts replaces the contact set of the last nb_collide (custom contacts, e.g. against the static environment).  Their tags may be
 * any uint32 A and B, including tags no collider carries, and their feature words any uint32: nb_read_cached_impulses orders them by
 * (B, A, feature) over the full width of the largest uploaded tag. */
int nb_upload_contacts(nb_context*, const nb_contact_data* host /* may be null */, const nb_active_bodies* host_active /* may be null */, void* stream); /* synchronises */
int nb_download_bodies(nb_context*, nb_body_data* host, void* stream);
int nb_download_contacts(nb_context*, nb_contact_data* host, nb_active_bodies* host_active, void* stream); /* synchronises */
int nb_download_cache(nb_context*, nb_contact_cache* host, void* stream);                                  /* synchronises */
int nb_download_counts(nb_context*, nb_counts* out, void* stream);   /* synchronises; fills *out and returns NB_ERR_OVERFLOW when out->overflow != 0 */
int nb_upload_momentum(nb_context*, const nb_body_momentum* host, uint32_t count, void* stream);
int nb_upload_transforms(nb_context*, const nb_transform* host, uint32_t count, void* stream);
int nb_download_momentum(nb_context*, nb_body_momentum* host, uint32_t count, void* stream);
int nb_download_transforms(nb_context*, nb_transform* host, uint32_t count, void* stream);

/* Ghost exchange of a scene sharded across GPUs: gather momentum rows of `dev_indices` into a contiguous DEVICE buffer (n x 32 B), and
 * scatter rows `dev_sources[i]` of a DEVICE buffer into body `dev_indices[i]`.  The buffer in between travels through one ncclAllGather. */
int nb_pack_momentum(nb_context*, const uint32_t* dev_indices, uint32_t n, void* dev_out, void* stream);
int nb_unpack_momentum(nb_context*, const uint32_t* dev_indices, const uint32_t* dev_sources, uint32_t n, const void* dev_in, void* stream);

/* One scene sharded across GPUs (SURVEY.md section 8e): C++ host, one process or thread per GPU, one nb_context per rank holding the
 * rank's OWNED bodies plus GHOST copies of neighbouring bodies.  After the warm start and after every solver sweep the ghosts'
 * BodyMomentum rows are replaced by their owners' (nb_shard_exchange), either with ONE ncclAllGather (NB_SHARD_NCCL, what BASELINE.json
 * prescribes; NCCL is bound at run time with dlopen) or with this library's own push/pull kernels over CUDA-IPC peer memory
 * (NB_SHARD_PEER: neighbour-only traffic over NVLink, no collective).  Both give bit-identical ghost rows.
 *   rank 0: nb_shard_unique_id -> broadcast the 128 bytes -> every rank: nb_shard_create;  every rank: nb_shard_ipc_handle -> all-gather
 *   the 64-byte handles -> nb_shard_open_peer for every other rank;  after every (re)partition: nb_shard_plan;  then nb_shard_step per
 *   sub-step (or nb_shard_exchange between the stage calls).  nb_shard_partition is the (host, deterministic) partition rule.
 * The shard's device memory is its own: nb_shard_destroy frees it.  A failed nb_shard_create sets *out to null and leaves the context as it was. */
typedef struct nb_shard nb_shard;
enum nb_shard_transport { NB_SHARD_NCCL = 0, NB_SHARD_PEER = 1 };
int nb_shard_unique_id(void* nccl_id_out /* 128 bytes */);
int nb_shard_create(nb_context*, uint32_t rank, uint32_t world, const void* nccl_id /* null: peer transport only */, uint32_t ghost_capacity, uint32_t export_capacity, nb_shard** out);
void nb_shard_destroy(nb_shard*);
int nb_shard_ipc_handle(nb_shard*, void* handle_out /* 64 bytes */);
int nb_shard_open_peer(nb_shard*, uint32_t peer, const void* handle);
int nb_shard_plan(nb_shard*, const uint32_t* export_local, uint32_t n_export, const uint32_t* sub_off, const uint32_t* sub_rank, const uint32_t* sub_slot,
                  const uint32_t* ghost_local, const uint32_t* ghost_src, uint32_t n_ghost, uint32_t max_export, void* stream);
int nb_shard_exchange(nb_shard*, int transport, void* stream);
int nb_shard_step(nb_shard*, float time_step, uint32_t iterations, float gravity, float damping, int transport, void* stream);
int nb_shard_graph_active(const nb_shard*);
int nb_shard_debug_no_exchange(nb_shard*, int on);   /* diagnostic: nb_shard_step runs the rank's local problem without the ghost hand-over */
int nb_shard_partition(const float* pos_xyz, const float* radius, uint32_t n, uint32_t gx, uint32_t gz, float margin, uint32_t balance_iterations,
                       uint32_t* owner_out, uint32_t* ghost_off /* gx*gz + 1 */, uint32_t* ghost_ids, uint32_t ghost_capacity);
/* One rank's exchange plan (the arrays nb_shard_plan takes) from that partition; host code, two passes: with any output null only
 * sizes[] = { n_owned, n_export, n_ghost, n_subscriptions, max_export } is filled.  owned_ids = this rank's bodies (0-based, ascending):
 * local body 1 + k is owned_ids[k], local body 1 + n_owned + j is the j-th entry of the rank's ghost list. */
int nb_shard_build_plan(const uint32_t* owner, uint32_t n, const uint32_t* ghost_off, const uint32_t* ghost_ids, uint32_t world, uint32_t rank,
                        uint32_t sizes[5], uint32_t* owned_ids, uint32_t* export_local, uint32_t* sub_off /* n_export + 1 */, uint32_t* sub_rank, uint32_t* sub_slot,
                        uint32_t* ghost_local, uint32_t* ghost_src);
/* The colliders of one rank's local scene ([world body, owned..., ghosts...]) in the global collider order and the local index of their
 * bodies; host code, two passes (sizes = { kept boxes, kept spheres }). */
int nb_shard_local_scene(const uint32_t* owned_ids, uint32_t n_owned, const uint32_t* ghost_ids, uint32_t n_ghost, uint32_t n_bodies_global,
                         const uint32_t* box_body, uint32_t n_boxes, const uint32_t* sphere_body, uint32_t n_spheres, uint32_t sizes[2],
                         uint32_t* box_sel, uint32_t* box_local_body, uint32_t* sphere_sel, uint32_t* sphere_local_body);

/* The simulation step, device resident.  Same order of calls as example/main.cpp:274-328. */
int nb_collide(nb_context*, void* stream);
int nb_apply_gravity_damping(nb_context*, float time_step, float gravity, float damping, void* stream);
int nb_read_cached_impulses(nb_context*, void* stream);
int nb_setup_contact_constraints(nb_context*, void* stream);
int nb_apply_impulses(nb_context*, uint32_t sweeps, void* stream);  /* `sweeps` back-to-back calls of nudge::apply_impulses */
int nb_update_cached_impulses(nb_context*, void* stream);
int nb_write_cached_impulses(nb_context*, void* stream);
int nb_advance(nb_context*, float time_step, void* stream);
/* One sub-step = the eight calls above in order.  On a stream the caller created (not the legacy default stream) the launches
 * are recorded once into a CUDA graph and replayed; NB_GRAPH=0 in the environment keeps plain launches. */
int nb_step(nb_context*, float time_step, uint32_t iterations, float gravity, float damping, void* stream);

/* User constraint rows (SURVEY.md section 8 f1): the device-resident form of the hook at example/main.cpp:316 ("Custom constraint impulses
 * should be applied here", after every apply_impulses sweep).  One row = one scalar velocity constraint between bodies a and b
 * (0 = the static world):  J v + bias -> 0  with the accumulated impulse kept inside [lo, hi]; rows are applied by sequential impulses in
 * upload order after every contact sweep, their accumulated impulses warm-start the next step (nudge_b200/csrc/nb_rows_api.cuh).
 * a and b must differ unless both are 0: a row on one body puts its whole Jacobian on a with b = 0 (a == b != 0 is NB_ERR_ARGUMENT).
 * Connect the bodies of a joint with nb_upload_connections too, so that islands treat them as one (example/main.cpp:285), and set
 * NB_FILTER_SKIP_CONNECTED (nb_upload_collision_filters) so that the joined bodies do not also collide where they overlap. */
typedef struct {
	uint32_t a, b;
	float lin_a[3], ang_a[3];   /* Jacobian of body a: linear and angular part */
	float lin_b[3], ang_b[3];   /* Jacobian of body b */
	float bias;                 /* velocity target term (e.g. Baumgarte: beta / dt * position error) */
	float lo, hi;               /* bounds of the accumulated impulse: (-inf, inf) joint, [0, inf) unilateral, [-f, f] motor / friction */
	float impulse;              /* accumulated impulse: warm start on upload, result on download */
	float softness;             /* constraint force mixing added to the effective inverse mass; 0 = rigid */
	float reserved;
} nb_constraint_row;            /* 80 bytes */
int nb_upload_constraint_rows(nb_context*, const nb_constraint_row* host_rows, uint32_t n, void* stream);   /* replaces the set; n = 0 removes it; synchronises */
int nb_download_constraint_rows(nb_context*, nb_constraint_row* host_rows, uint32_t n, void* stream);       /* caller's order; synchronises */

/* Joints (ragdolls, doors, chains, welded parts; DESIGN.md section 8.13): constraints between two bodies that stay on the device.  A joint is a
 * producer of the user constraint rows above: once per step, inside nb_setup_contact_constraints (and so inside nb_step's graph), the library
 * rebuilds each joint's rows from the two bodies' current transforms, and it applies them exactly as it applies user rows.  Nothing crosses
 * PCIe and nothing synchronises between steps.
 * Rows per joint, in this order: BALL 3 (point x, y, z), HINGE 5 (point x, y, z, angular 1, 2), FIXED 6 (point x, y, z, angular x, y, z),
 * DISTANCE 1.  Every row has a, b and softness of its joint, lo = -inf, hi = +inf, reserved = 0, and keeps its accumulated impulse from the
 * previous step.  The arithmetic is float32, left to right as written, without fused multiply-adds, with
 *   cross(u, v) = (u.y*v.z - u.z*v.y, u.z*v.x - u.x*v.z, u.x*v.y - u.y*v.x),   dot(u, v) = (u.x*v.x + u.y*v.y) + u.z*v.z,
 *   qrot(q, r):  t = 2 * cross(q.xyz, r);  (r + q.w * t) + cross(q.xyz, t)                                      (nudge.cpp:1117-1120)
 *   qmul(l, r):  xyz = ((r.xyz * l.w) + (l.xyz * r.w)) + cross(l.xyz, r.xyz),  w = l.w*r.w - dot(l.xyz, r.xyz)  (nudge.cpp:1122-1126)
 * (p_a, q_a) and (p_b, q_b) the bodies' positions and rotations, and k = beta / dt, dt being the step's time step: nb_step has it, the stage
 * calls take it from the nb_apply_gravity_damping of the step (nb_setup_contact_constraints with joints and no nb_apply_gravity_damping since
 * the last nb_collide is NB_ERR_ARGUMENT).
 *   anchors:   ra = qrot(q_a, anchor_a);  wa = p_a + ra;  b != 0: rb = qrot(q_b, anchor_b), wb = p_b + rb;  b == 0: rb = (0, 0, 0), wb = anchor_b
 *   point rows (BALL, HINGE, FIXED):  err = wa - wb;  for the axis e = x, y, z:  lin_a = e,  lin_b = -e (the other components +0),
 *              ang_a = (0, ra.z, -ra.y) | (-ra.z, 0, ra.x) | (ra.y, -ra.x, 0),  ang_b = (0, -rb.z, rb.y) | (rb.z, 0, -rb.x) | (-rb.y, rb.x, 0),
 *              bias = k * err.e
 *   HINGE:     u = qrot(q_a, axis_a);  w = b != 0 ? qrot(q_b, axis_b) : axis_b;  c = cross(u, w)
 *              t1 = fabsf(u.x) < 0.57735f ? (0, u.z, -u.y) : (-u.z, 0, u.x);  t1 = t1 * (1 / sqrtf(dot(t1, t1)));  t2 = cross(u, t1)
 *              angular row i:  lin_a = lin_b = 0,  ang_a = t_i,  ang_b = -t_i,  bias = -(k * dot(c, t_i))
 *   FIXED:     g = qmul(q_a, rel_rotation);  d = b != 0 ? qmul(g, (-q_b.xyz, q_b.w)) : g;  if d.w < 0: d.xyz = -d.xyz
 *              angular row e = x, y, z:  lin_a = lin_b = 0,  ang_a = e,  ang_b = -e,  bias = k * (2 * d.e)
 *   DISTANCE:  v = wa - wb;  dist = sqrtf(dot(v, v));  n = dist > 0 ? v * (1 / dist) : (0, 1, 0)
 *              lin_a = n,  ang_a = cross(ra, n),  lin_b = -n,  ang_b = -cross(rb, n) (each component negated),  bias = k * (dist - length)
 * With the row update impulse' = impulse - eff * (J v + bias + softness * impulse) these signs make every error shrink.
 * Joints behave like their rows appended after the user rows: their accumulated impulses are applied in nb_setup_contact_constraints after the
 * contacts' warm start and the user rows', and their rows run after every contact sweep after the user rows, in both solver modes.  Joints run
 * in upload order wherever two joints share a body (one thread applies a joint's rows one after the other; joints of one dependency level
 * touch disjoint bodies and run in one launch), so the result is the sequential host loop over all generated rows in joint order.  A kinematic
 * side has infinite mass, as for rows.  Connect the joint's bodies with nb_upload_connections, and set NB_FILTER_SKIP_CONNECTED so that they do
 * not also collide; the library does not edit the connection list.
 * nb_upload_joints replaces the set (n = 0 removes it); impulse[0 .. rows-1] warm-start the joint's rows.  Every entry is checked on the host
 * before any device work, and an error changes nothing.  NB_ERR_ARGUMENT: a == 0, a == b, a or b at or beyond the body count, an unknown
 * type, a field that is not finite, a null pointer with n > 0.  NB_ERR_CAPACITY: the joints form a dependency chain of more than 4,096 levels
 * (order a long chain red-black).  Asynchronous on `stream`; the host array may be reused when the call returns.  nb_step re-records its graph
 * only when the structure (n, and each joint's type, a and b) changed: new parameters or impulses for the same structure keep it.
 * nb_download_joints returns the joints in upload order with impulse[] = the rows' current accumulated impulses (a joint that should fail
 * past a force takes a BREAKABLE drive instead, nb_joint_drive below, which breaks it on the device) and the unused impulse slots 0.
 * *count = the number of joints; NB_ERR_CAPACITY when capacity is smaller.  Synchronises.
 * nb_remove_bodies deletes the joints that name a removed body and remaps the others, keeping their order, parameters and accumulated
 * impulses; the kept body on the other side of a deleted joint gets idle counter 0 (not body 0, not a kinematic body).  nb_add_bodies leaves
 * the joints alone.  nb_upload_bodies keeps the set while the body count is unchanged and removes it when the count changes.
 * nb_snapshot_save / nb_snapshot_restore carry the set with its impulses.  nb_save_state writes it (state version 6), nb_load_state restores
 * it, and a file of an older version removes it.  Not supported by nb_shard_step (NB_ERR_ARGUMENT).
 * Cost per step with L joint levels and s sweeps: 1 + L * (s + 1) launches, and the contact sweeps run one per solver launch as with user
 * rows; without a set the step launches exactly what it launches without this feature. */
enum nb_joint_type { NB_JOINT_BALL = 0, NB_JOINT_HINGE = 1, NB_JOINT_FIXED = 2, NB_JOINT_DISTANCE = 3 };
typedef struct {
	uint32_t type, a, b;        /* a != 0; b = 0 is the static world; a != b */
	float anchor_a[3];          /* in a's body frame */
	float anchor_b[3];          /* in b's body frame; a world point when b = 0 */
	float axis_a[3], axis_b[3]; /* HINGE: the hinge axis in each body's frame (unit length; the world frame for b = 0).  axis_a is also the
	                               slide axis of FIXED with a SLIDE drive and the twist axis of BALL with a CONE or TWIST drive */
	float rel_rotation[4];      /* FIXED, HINGE with a LIMIT drive and BALL with a CONE or TWIST drive: conj(q_a) * q_b at rest (x, y, z, w;
	                               q_b = identity for b = 0) */
	float length;               /* DISTANCE: rest distance between the anchors */
	float beta;                 /* Baumgarte factor: bias = beta / dt * error */
	float softness;             /* copied into every row */
	float impulse[6];           /* accumulated impulses of the joint's rows: warm start on upload, result on download */
} nb_joint;                     /* 112 bytes */
int nb_upload_joints(nb_context*, const nb_joint* host, uint32_t n, void* stream);
int nb_download_joints(nb_context*, nb_joint* host, uint32_t capacity, uint32_t* count, void* stream);

/* Joint drives (doors, knees, flippers, wheels, fans, ropes, breakable bridges and welds; DESIGN.md section 8.17): hinge angle limits, hinge
 * motors, distance ranges and break thresholds, built and solved by the joints' own kernels inside the step.  Sliders (pistons, drawers,
 * rails, struts) and ragdoll shoulders, hips and necks (DESIGN.md section 8.20) are drives too: SLIDE frees a FIXED joint's translation along
 * axis_a, and CONE and TWIST limit a BALL joint's swing away from axis_a and its twist about it.  A drive set is a sparse table
 * keyed by joint: at most one drive per joint, naming it by its index in the current joint set's upload order.
 * Rows: a drive appends rows to its joint, solved right after the joint's own rows in this order: motor (MOTOR) or cone (CONE), lower limit
 * and upper limit (LIMIT or TWIST); so a drive has (MOTOR|CONE ? 1 : 0) + (LIMIT|TWIST ? 2 : 0) appended rows.  Every appended row has the joint's a, b and softness, reserved = 0, and keeps its accumulated impulse from step to step.  The
 * appended rows sit in a row buffer of their own: nb_debug_read("joint_rows") returns the joints' own rows, exactly as without drives, and
 * nb_debug_read("joint_drive_rows") the appended rows, per driven joint in the joint table's order (by joint level, upload order within
 * one).  Same arithmetic rules as above (float32, left to right, no fused
 * multiply-adds), with k = beta / dt and bias(C) = C > 0 ? C / dt : k * C (speculative: a limit row lets the coordinate reach its bound
 * within the step, and pulls it back at the joint's Baumgarte rate once past it):
 *   HINGE coordinate:  g = qmul(q_a, rel_rotation);  d = b != 0 ? qmul(g, (-q_b.xyz, q_b.w)) : g;  if d.w < 0: d = -d (all four);
 *              u = qrot(q_a, axis_a);  sh = -dot(d.xyz, u);  ch = d.w.  (sh, ch) = (sin, cos) of half of theta, b's rotation relative to a
 *              about u from the rest pose rel_rotation (b = 0: minus a's rotation); theta in (-pi, pi].  The hinge Jacobian: lin_a = lin_b = 0,
 *              ang_a = -u, ang_b = u.  The limits are converted once on the host at upload, each to its pair (sin(x/2), cos(x/2)), rounded from
 *              double to float32: (sl, cl) for lower, (su, cu) for upper.
 *   HINGE motor:       the hinge Jacobian, bias = -motor_speed, lo = -(max_motor_torque * dt), hi = max_motor_torque * dt.
 *   Angle measure:     for the pair (s, c) = (sin x, cos x) of a half difference x in [-pi, pi],  m(s, c) = c >= 0 ? 2*s : (s >= 0 ?
 *              4 - 2*s : -4 - 2*s):  continuous and increasing in x, with the sign of x, and (2/pi) * min(|2x|, pi) <= |m| <= |2x|.
 *   HINGE lower limit: C = m(sh*cl - ch*sl, ch*cl + sh*sl) (x = (theta - lower) / 2), the hinge Jacobian;  upper: C = m(su*ch - cu*sh,
 *              cu*ch + su*sh) (x = (upper - theta) / 2), ang_a = u, ang_b = -u, lin_a = lin_b = 0 (the hinge Jacobian with its angular
 *              parts negated);  both bias = bias(C), lo = 0, hi = +inf.
 *   DISTANCE limit:    the joint's own row is written with lo = hi = 0 (it stays in place and applies nothing);  lower: the own row's
 *              Jacobian with C = dist - lower;  upper: that Jacobian negated with C = upper - dist;  both bias = bias(C), lo = 0, hi = +inf.
 *   Slider:    FIXED + SLIDE.  u = qrot(q_a, axis_a) is the slide axis, t1, t2 built from u exactly as HINGE builds them, sa = ra - err
 *              (from a's position to b's anchor).  The joint's own rows 0 and 1 become, for t = t1, t2: lin_a = t, ang_a = cross(sa, t),
 *              lin_b = -t, ang_b = -cross(rb, t) (each component negated), bias = k * dot(err, t); row 2 is the same form on u with lo = hi = 0
 *              (it stays in place and applies nothing); rows 3 to 5 are FIXED's angular rows.  Each keeps its accumulated impulse.  The
 *              coordinate s = dot(wb - wa, u) has the Jacobian J_s: lin_a = -u, ang_a = -cross(sa, u), lin_b = u, ang_b = cross(rb, u).
 *   SLIDE motor:       J_s, bias = -motor_speed, lo = -(max_motor_torque * dt), hi = max_motor_torque * dt: for a slider motor_speed is
 *              a linear speed and max_motor_torque a force.
 *   SLIDE lower limit: J_s with C = s - lower;  upper: -J_s (every component negated) with C = upper - s;  both bias = bias(C), lo = 0,
 *              hi = +inf.
 *   Swing-twist:       BALL + CONE / TWIST.  d as the HINGE coordinate computes it (d.w >= 0), u = qrot(q_a, axis_a) the twist axis;
 *              a_ = dot(d.xyz, u), sh = -a_, ch = d.w;  the swing p = d.xyz - u * a_ (per component);  ss = sqrtf(dot(p, p)) and
 *              cs = sqrtf(sh*sh + ch*ch), the sine and cosine of half the swing angle;  the twist pair (sh', ch') = cs > 0 ? (sh * (1/cs),
 *              ch * (1/cs)) : (0, 1).
 *   TWIST limit:       the HINGE lower and upper limit rows, on the hinge Jacobian about u, with (sh', ch') in place of (sh, ch); lower and
 *              upper in [-pi, pi] converted to (sl, cl), (su, cu) as for a hinge.
 *   CONE:      (sc, cc) = (sin, cos) of cone/2, converted on the host in double and rounded to float32;  C = 2 * (sc*cs - cc*ss);
 *              g = cross(qrot((-d.xyz, d.w), u), u), sg = sqrtf(dot(g, g)), n = sg > 0 ? g * (1/sg) : (0, 0, 0) (the direction in which
 *              the swing changes fastest; a zero row has no effect);  ang_a = -n, ang_b = n, lin_a = lin_b = 0, bias = bias(C),
 *              lo = 0, hi = +inf.
 *   Breaking:  when k_joint_rows is about to rewrite a BREAKABLE joint's rows it takes the accumulated impulses the previous step left:
 *              P = the sum 0 + i*i in row order over the joint's linear rows (the point rows; DISTANCE's own and appended rows; a slider's
 *              appended rows), A = the same over its angular rows (HINGE's and FIXED's angular rows, the hinge's motor and limit rows, the cone
 *              and twist rows).  The joint breaks when
 *              P > (break_force*dt)*(break_force*dt) or A > (break_torque*dt)*(break_torque*dt); +inf never breaks.
 *   Broken:    a drive with broken = 1 has every row of its joint, appended rows included, written as a zero row: zero Jacobian, bias = 0,
 *              lo = hi = 0, impulse = 0, softness = 0, a and b kept, reserved = 0.  The rows stay in the set, so nothing structural changes
 *              and nb_step keeps its graph; broken stays 1 until an upload re-arms it.  Connections and idle counters are not touched (edit the
 *              connections to let the pieces collide).
 *   position:  each build of an unbroken LIMIT drive records the coordinate it used: (sh, ch) for a hinge, dist for a distance joint; each
 *              build of an unbroken SLIDE drive records s, and of a CONE or TWIST drive (sh', ch') with TWIST, (ss, cs) with CONE alone.
 * nb_upload_joint_drives replaces the drive set (n = 0 removes it); impulse[] warm-starts the appended rows, broken is installed as given (0
 * re-arms a broken joint), position is ignored and reads 0 until the next row build.  Every entry is checked on the host before any device
 * work, and an error changes nothing.  NB_ERR_ARGUMENT: a null pointer with n > 0; a joint index at or beyond the joint count, or two drives
 * on one joint; a flag the joint's type does not take (LIMIT: HINGE, DISTANCE, FIXED with SLIDE; MOTOR: HINGE, FIXED with SLIDE; SLIDE:
 * FIXED; CONE, TWIST: BALL; BREAKABLE: every type) or an unknown bit; lower > upper (LIMIT, TWIST), a hinge or twist limit outside [-pi, pi]
 * (pi rounded to float32, 3.14159274f), a negative distance limit; a CONE whose cone is outside (0, pi], or with a nonzero motor_speed or
 * max_motor_torque; a negative max_motor_torque, break_force or break_torque; a field that is not finite other than thresholds of +inf (cone
 * is read only with CONE); broken > 1; a HINGE LIMIT, CONE or TWIST whose joint's rel_rotation has |x*x + y*y + z*z + w*w - 1| > 1e-3 (in
 * double); a SLIDE, CONE or TWIST whose joint's axis_a has |x*x + y*y + z*z - 1| > 1e-3 (in double).  Asynchronous on `stream`, staged like nb_upload_joints (the host array
 * may be reused on return); it synchronises only when the drive table or its row buffer must grow.  nb_step re-records its graph only when the drive
 * structure (which joints, which flags) changed or a buffer moved: new speeds, torques, limits, thresholds, impulses or broken flags for the
 * same structure keep it, so a throttle may be uploaded every frame.
 * nb_download_joint_drives returns the drives in joint-index order with impulse[] = the appended rows' current accumulated impulses (0 where
 * a row is absent), broken, and position: 2*atan2(sh, ch) in double, rounded to float32, for a hinge, dist for a distance joint, s for a
 * slider, 2*atan2 of the recorded pair for a BALL (the twist angle with TWIST, the swing angle with CONE alone), 0 without LIMIT, SLIDE, CONE
 * or TWIST or before the first build.  A CONE drive returns motor_speed = max_motor_torque = 0 and its cone as uploaded; cone is 0 otherwise.  *count = the number of drives; NB_ERR_CAPACITY when capacity is smaller.  Synchronises.
 * The set follows its joints: nb_upload_joints keeps it (impulses and broken flags included) when the joint structure is unchanged and removes
 * it otherwise; nb_remove_bodies drops the drives of deleted joints and renumbers the rest; nb_add_bodies leaves it alone; nb_upload_bodies
 * removes it with the joints.  Snapshots carry it; nb_save_state writes it (state version 7) and nb_load_state installs it through the
 * upload's checks; a file of an older version removes it.  SLIDE, CONE and TWIST and the cone travel in the same rows (no new state version);
 * a build without them refuses such a file's drives as an unknown flag.  nb_debug_read("joint_drives") returns the device table: one 64-byte
 * entry per joint in table order, { flags, first appended row (an index into "joint_drive_rows"), lower, upper, sl, cl, su, cu, motor_speed, max_motor_torque, break_force,
 * break_torque, position[2] (sh, ch; dist, 0; s, 0; sh', ch' or ss, cs), broken, cone }, flags 0 and the rest 0 for a joint without a drive.
 * A SLIDE drive holds lower and upper raw, with sl .. cu 0; a TWIST drive holds their half-angle pairs as a hinge does; a CONE drive holds
 * (sc, cc) in motor_speed and max_motor_torque and its cone as uploaded in the last word (0 without CONE).
 * Cost: no launch; k_joint_rows and k_joint_solve take the drive table and its rows as two more arguments (null without a set), and
 * without a set the joints' rows, the launches and the graph are what they are without this feature. */
/* Bit 8 is unassigned (refused as an unknown flag). */
enum nb_joint_drive_flags { NB_JOINT_LIMIT = 1, NB_JOINT_MOTOR = 2, NB_JOINT_BREAKABLE = 4, NB_JOINT_SLIDE = 16, NB_JOINT_CONE = 32, NB_JOINT_TWIST = 64 };
typedef struct {
	uint32_t joint;             /* index of the joint in the current set's upload order */
	uint32_t flags;             /* LIMIT: HINGE, DISTANCE, FIXED with SLIDE.  MOTOR: HINGE, FIXED with SLIDE.  SLIDE: FIXED.  CONE, TWIST:
	                               BALL.  BREAKABLE: every type */
	float lower, upper;         /* LIMIT: HINGE angle in radians, -pi <= lower <= upper <= pi; DISTANCE length, 0 <= lower <= upper; slider
	                               coordinate s, lower <= upper.  TWIST: twist angle in radians, -pi <= lower <= upper <= pi */
	float motor_speed;          /* MOTOR: target of the hinge's relative angular velocity (rad/s) or of the slider's speed (units/s) */
	float max_motor_torque;     /* MOTOR: >= 0; the motor row's impulse stays in [-max_motor_torque*dt, +max_motor_torque*dt] (a force
	                               for a slider).  CONE: both motor fields must be 0 */
	float break_force, break_torque;   /* BREAKABLE: >= 0, +inf = never */
	float impulse[3];           /* accumulated impulses of the motor or cone, lower-limit and upper-limit rows (0 where absent) */
	float position;             /* download: the hinge angle, the distance, the slider coordinate, the twist angle or, with CONE alone,
	                               the swing angle at the last row build (0 without LIMIT, SLIDE, CONE or TWIST) */
	uint32_t broken;            /* 0 or 1; upload 0 to re-arm a broken joint */
	float cone;                 /* CONE: the swing cone's half-angle in radians, 0 < cone <= pi; ignored (and downloaded as 0) otherwise */
} nb_joint_drive;               /* 56 bytes */
int nb_upload_joint_drives(nb_context*, const nb_joint_drive* host, uint32_t n, void* stream);
int nb_download_joint_drives(nb_context*, nb_joint_drive* host, uint32_t capacity, uint32_t* count, void* stream);

/* Joint springs (PD actuators of robot arms and legs, vehicle suspension, bungee cords, powered ragdolls; DESIGN.md section 8.21): a joint
 * coordinate pulled toward a target by a spring-damper given in physical units, built and solved by the joints' own kernels inside the step,
 * so that an actuator needs no per-step host round trip.  The spring is Catto's soft step: the implicit (backward Euler) spring-damper
 * m*x'' = -stiffness*(x - target) - damping*(x' - target_velocity) over one step is one ordinary constraint row, and for a single row one
 * sweep of the row update gives exactly that step.  A spring set is a sparse table keyed by joint, like the drives: at most one spring per
 * joint, naming it by its index in the current joint set's upload order; a joint may have a drive and a spring.
 * Rows: HINGE, FIXED and DISTANCE springs have one spring row, BALL springs three.  k_joint_solve applies, per joint, its own rows, then its
 * spring rows, then its drive rows (so limits act last and hold against a spring); the warm start follows the same order.  The spring rows sit
 * in a row buffer of their own, like the drive rows: nb_debug_read("joint_rows") and ("joint_drive_rows") are what they are without
 * springs, and nb_debug_read("joint_spring_rows") returns the spring rows, per sprung joint in the joint table's order.  Same arithmetic rules as the joints' section (float32, left to right, no
 * fused multiply-adds), dt the step's time step:
 *   Spring row:  on a coordinate C with Jacobian J, of the joint's a and b:  den = damping + dt * stiffness;  softness = 1.0f / (dt * den);
 *              bias = (stiffness * C - damping * target_velocity) / den;  lo = -(max_force * dt), hi = max_force * dt;  reserved = 0.  The row
 *              keeps its accumulated impulse from step to step.
 *   HINGE:     J = the hinge Jacobian (lin_a = lin_b = 0, ang_a = -u, ang_b = u);  C = m(sh*ct - ch*st, ch*ct + sh*st) with (sh, ch) the HINGE
 *              coordinate and m the angle measure of the drives' section, and (st, ct) = (sin, cos) of target / 2, converted on the host in
 *              double and rounded to float32.  C is continuous and increasing in theta - target over [-2pi, 2pi] and exact to first order at
 *              the target; it never pushes across the +-pi seam, so a spring does not take the short way round through a limited hinge's gap
 *              (a target near +pi and an angle near -pi pull the long way, the way a LIMIT lets the hinge turn).  Needs a unit rel_rotation.
 *   FIXED:     J = J_s and C = s - target, with the slider's coordinate s = dot(wb - wa, u), u = qrot(q_a, axis_a), and sa = ra - err.  Meant
 *              for a FIXED joint with a SLIDE drive; without one the joint's point rows hold s and the spring only adds load, bounded by
 *              max_force (not refused, so that springs need not follow drive uploads).  Needs a unit axis_a.
 *   DISTANCE:  J = the joint's own row's Jacobian and C = dist - target.  A sprung distance joint's own row is written with lo = hi = 0 (it
 *              stays in place and applies nothing), as with LIMIT: the joint becomes a spring-damper, and with LIMIT a bungee with a range.
 *   BALL:      three rows.  d = qmul(q_a, target);  b != 0: d = qmul(d, (-q_b.xyz, q_b.w));  if d.w < 0: d = -d (all four).  Row e = x, y, z:
 *              lin_a = lin_b = 0, ang_a = e, ang_b = -e, C = 2 * d.e (FIXED's angular rows on the target rotation).  max_force bounds each
 *              row on its own (a box, not a ball).
 *   Breaking:  spring rows are not counted in the break test; a broken joint's spring rows are written as zero rows, like its drive rows.
 *   position:  each build of an unbroken spring records its coordinate: (sh, ch) for a HINGE, s for FIXED, dist for DISTANCE,
 *              (sqrtf(dot(d.xyz, d.xyz)), d.w) for a BALL.
 * nb_upload_joint_springs replaces the spring set (n = 0 removes it); impulse[] warm-starts the spring rows; position is ignored and reads 0
 * until the next row build.  Every entry is checked on the host before any device work, and an error changes nothing.  NB_ERR_ARGUMENT: a
 * null pointer with n > 0; a joint index at or beyond the joint count, or two springs on one joint; reserved != 0; a field that is not finite
 * other than max_force = +inf; a negative stiffness, damping or max_force; stiffness = damping = 0; a stiffness or damping that is neither 0
 * nor in [1e-12, 1e12]; |target_velocity| > 1e12; a FIXED or DISTANCE target beyond 1e12 in magnitude; a nonzero target word the joint's type
 * does not read; a HINGE target outside [-pi, pi] (pi rounded to float32) or whose joint's rel_rotation is not of unit length (as for HINGE
 * LIMIT); a negative DISTANCE target; a FIXED spring whose joint's axis_a is not of unit length; a BALL spring with a nonzero
 * target_velocity or a target with |x*x + y*y + z*z + w*w - 1| > 1e-3 (in double).  Within these bounds every spring row is finite for
 * time steps 1e-6 <= dt <= 1 (dt * den >= 1e-24, so softness <= 1e24, and |bias| <= |C| / dt + |target_velocity|) as long as the
 * coordinate is finite and within about 1e20 of its target.  The upload sets the idle counter of every dynamic body of a sprung joint to 0
 * (one launch; not body 0, not a kinematic body), so that a new target reaches a body that has fallen asleep; a joint drive upload wakes
 * nothing.  Asynchronous on `stream`, staged like nb_upload_joints; it synchronises only when the spring table, the row buffer or the wake's
 * index buffer must grow.  nb_step re-records its graph only when the spring structure (which
 * joints) changed or a buffer moved: new targets, gains, bounds or impulses for the same joints keep it, so targets may be uploaded every step.
 * nb_download_joint_springs returns the springs in joint-index order, the target as uploaded, impulse[] = the spring rows' current
 * accumulated impulses (0 where a row is absent), and position: 2*atan2(sh, ch) in double, rounded to float32, for a HINGE (its angle), s for
 * FIXED, dist for DISTANCE, 2*atan2 of the recorded pair for a BALL (the angle between the rotation and the target).  *count = the number of
 * springs; NB_ERR_CAPACITY when capacity is smaller.  Synchronises.
 * The set follows its joints as the drives do: nb_upload_joints keeps it when the joint structure is unchanged and removes it otherwise;
 * nb_remove_bodies drops the springs of deleted joints and renumbers the rest; nb_add_bodies leaves it alone; nb_upload_bodies removes it with
 * the joints.  Snapshots carry it; nb_save_state writes it (state version 9) and nb_load_state installs it through the upload's checks; a
 * file of an older version removes it.  nb_debug_read("joint_springs") returns the device table: one 64-byte entry per joint in table order,
 * { present, first spring row, target[4] (a HINGE: st, ct, 0, 0), target_velocity, stiffness, damping, max_force, position[2] (sh, ch; s, 0;
 * dist, 0; |d.xyz|, d.w), target angle (HINGE; else 0), reserved[3] = 0 }, all 0 for a joint without a spring.
 * Cost: no launch in the step; k_joint_rows and k_joint_solve take the spring table and its rows as two more arguments (null without a
 * set), and without a set the joints' and drives' rows, the launches and the graph are what they are without this feature. */
typedef struct {
	uint32_t joint;             /* index of the joint in the current set's upload order */
	uint32_t reserved;          /* must be 0 */
	float target[4];            /* HINGE: the target angle (rad) in [0], -pi <= target <= pi;  FIXED: the target slide coordinate s in [0];
	                               DISTANCE: the target length >= 0 in [0];  BALL: the target relative rotation conj(q_a) * q_b as (x, y, z, w),
	                               rel_rotation's convention.  Words a type does not read must be 0 */
	float target_velocity;      /* HINGE rad/s, FIXED and DISTANCE units/s; BALL: must be 0 */
	float stiffness;            /* 0 or in [1e-12, 1e12]: force per unit or torque per radian */
	float damping;              /* 0 or in [1e-12, 1e12]; stiffness + damping > 0 */
	float max_force;            /* >= 0 or +inf: every spring row's impulse stays in [-max_force*dt, max_force*dt] (a torque for HINGE and BALL) */
	float impulse[3];           /* the spring rows' accumulated impulses: warm start on upload, result on download (BALL 3 rows, else 1) */
	float position;             /* download: the coordinate at the last row build; ignored on upload */
} nb_joint_spring;              /* 56 bytes */
int nb_upload_joint_springs(nb_context*, const nb_joint_spring* host, uint32_t n, void* stream);
int nb_download_joint_springs(nb_context*, nb_joint_spring* host, uint32_t capacity, uint32_t* count, void* stream);

/* Contact events (collision callbacks; DESIGN.md section 8.5): which collider pairs started or stopped touching, computed on the device inside
 * nb_write_cached_impulses (so the stage calls, nb_step and its graph replay give the same stream).  A pair (key tags = A | (uint64)B << 32,
 * the pair word of nb_contact_data.tags) is touching after a step if the contact cache that step wrote holds an entry with that key (the
 * step's contacts plus the kept entries of sleeping pairs); after nb_upload_cache / nb_load_state the uploaded cache defines it.  With `old` =
 * the cache before the call, `cur` = the step's contacts and `culled` = the kept entries of sleeping pairs:
 *   NB_CONTACT_END:   key in old, not in cur, not in culled (a sleeping pair never ends; a pair ends when its island wakes and it is gone);
 *   NB_CONTACT_BEGIN: key in cur, not in old (a pair whose island wakes still touching does not begin again).
 * One call appends all its END events in ascending key order, then all its BEGIN events in ascending key order.  A BEGIN event carries the
 * pair's contact count, its deepest contact (the first of the pair's contacts in (tag, feature) order, replaced only by a later one with a
 * strictly greater penetration: position, normal, penetration, bodies) and the sum of the pair's final cached impulses in (tag, feature)
 * order (fp32, sequential; in NB_SOLVER_THROUGHPUT the impulses vary from run to run, everything else is deterministic).  An END event
 * carries tags, kind and step only, every other field is 0.  `step` counts the nb_write_cached_impulses calls since enabling (0 first).
 * Cost when enabled: 3 kernel launches per step; none when disabled (the default).  Not supported by nb_shard_step (NB_ERR_ARGUMENT): ghost
 * pairs would be reported by several ranks. */
typedef struct {
	uint64_t tags;                 /* A | (uint64)B << 32: the pair's collider tags (the cache key) */
	uint32_t kind, step;           /* NB_CONTACT_BEGIN = 1, NB_CONTACT_END = 2 (NB_SENSOR_BEGIN = 3, NB_SENSOR_END = 4: nb_upload_sensors); device sub-step counter */
	uint32_t body_a, body_b, contacts;
	float penetration, position[3], normal[3], impulse[3];
	uint32_t reserved[3];
} nb_contact_event;                /* 80 bytes */
enum nb_contact_event_kind { NB_CONTACT_BEGIN = 1, NB_CONTACT_END = 2, NB_SENSOR_BEGIN = 3, NB_SENSOR_END = 4 };
/* capacity = events the device buffer holds between two drains; 0 disables.  Every call resets count, dropped and step; the buffer is reused
 * unless the capacity grows.  Synchronises the device. */
int nb_enable_contact_events(nb_context*, uint32_t capacity);
/* Synchronises `stream`, copies the stored events to `host` and empties the device buffer.  *count / *dropped = events stored / events lost
 * because the buffer was full (the stored ones are always the first of the sequence).  NB_ERR_CAPACITY if `capacity` < *count (nothing is
 * drained; *count says how much room is needed); NB_ERR_OVERFLOW if events were dropped (the outputs are filled and the buffer is emptied);
 * NB_ERR_ARGUMENT if events are not enabled. */
int nb_download_contact_events(nb_context*, nb_contact_event* host, uint32_t capacity, uint32_t* count, uint32_t* dropped, void* stream);

/* Collision filters (DESIGN.md section 8.6): which collider pairs nb_collide reports.  One nb_collision_filter per collider, boxes first then
 * spheres (the collider index order of nb_upload_colliders).  Colliders i and j collide iff
 *   (category_i & mask_j) != 0 && (category_j & mask_i) != 0            (Box2D's rule; without a table every pair passes)
 * and, with NB_FILTER_SKIP_CONNECTED, their bodies are not joined by an entry of nb_upload_connections (either order, body 0 included;
 * connections still merge islands).  A rejected pair is not a broadphase pair: it is not counted in nb_counts.pairs, does not link or
 * wake islands, and never appears in the sleeping pairs, contacts, contact cache or events, except that a pair that was touching gets
 * the ordinary NB_CONTACT_END when it becomes rejected.  Contacts uploaded with nb_upload_contacts are taken as given.
 * n = boxes + spheres uploads a table, n = 0 removes it, any other n is NB_ERR_ARGUMENT; flags apply with or without a table.
 * nb_upload_colliders keeps the table while the total collider count is unchanged and removes it when the count changes (the flags
 * stay).  nb_save_state writes the table and flags (state version 2; version 1 without them), nb_load_state restores them.
 * In nb_shard_step every rank filters with the global filter of its colliders, ghosts included; shards carry no connections, so
 * NB_FILTER_SKIP_CONNECTED has no effect there.  Synchronises `stream`. */
typedef struct { uint16_t category, mask; } nb_collision_filter;   /* 4 bytes */
enum nb_filter_flags { NB_FILTER_SKIP_CONNECTED = 1 };
int nb_upload_collision_filters(nb_context*, const nb_collision_filter* host, uint32_t n, uint32_t flags, void* stream);

/* Sensor colliders (trigger volumes; DESIGN.md section 8.7): colliders that detect overlap and exert no force.  One byte per collider, boxes
 * first then spheres (the order of nb_upload_colliders): nonzero = sensor.  A pair of colliders is a SENSOR PAIR when exactly one of them is a
 * sensor (two sensors never interact), they are on different bodies, their AABBs overlap strictly and the pair passes the collision filter
 * and NB_FILTER_SKIP_CONNECTED as an ordinary pair would.  A sensor pair is not a broadphase pair: it is not counted in nb_counts.pairs,
 * does not link or wake islands, and never reaches the sleeping pairs, contacts, contact cache, solver or contact events.  It OVERLAPS when
 * the narrowphase would give it at least one contact (the same code and pair orientation as the contact pipeline), evaluated in every
 * nb_collide whether its bodies sleep or not.
 * Overlap list of the last nb_collide: one entry per overlapping pair, key tags = min(tag_i, tag_j) | (uint64)max(tag_i, tag_j) << 32 (the
 * collider tags, like the contact-event key), body_a = the body of the lower-tag collider, body_b = the other's (with equal tags, body_a is
 * the lower of the two body indices); ascending by tags.
 * Events (with nb_enable_contact_events): nb_write_cached_impulses compares the overlap list of the step's nb_collide (cur) with the one as of
 * its previous call (old) and appends, after the contact ENDs and BEGINs, NB_SENSOR_END for every key in old and not in cur, then NB_SENSOR_BEGIN
 * for every key in cur and not in old, each in ascending key order.  A sensor event carries tags, kind, step, body_a and body_b; every other
 * field is 0.  After nb_upload_sensors and nb_load_state old is empty, so the next step begins every overlap.
 * n = boxes + spheres uploads a table, n = 0 removes it, any other n is NB_ERR_ARGUMENT.  max_sensor_pairs = capacity for candidate sensor
 * pairs (AABB hits) per nb_collide; 0 = 256 per sensor collider, at least 1024, at most the context's scratch capacity (the largest of
 * max_pairs, max_contacts, bodies and colliders, which is also the upper limit: NB_ERR_CAPACITY above it).  More candidates set bit 32 of
 * nb_counts.overflow (nb_download_counts returns NB_ERR_OVERFLOW), and that step's overlaps and sensor events are undefined.
 * nb_upload_colliders keeps the table while the collider count is unchanged and removes it when the count changes.  nb_save_state writes it
 * (state version 3), nb_load_state restores it.  Not supported by nb_shard_step (NB_ERR_ARGUMENT): a ghost's overlaps would be reported by
 * several ranks.  Cost: 5 kernel launches per nb_collide and 1 per nb_write_cached_impulses with a table, none without.  Synchronises `stream`. */
typedef struct { uint64_t tags; uint32_t body_a, body_b; } nb_sensor_overlap;   /* 16 bytes */
int nb_upload_sensors(nb_context*, const uint8_t* host_flags, uint32_t n, uint32_t max_sensor_pairs, void* stream);
/* The overlaps of the last nb_collide, ascending by tags.  *count = their number; NB_ERR_CAPACITY if capacity < *count.  Synchronises `stream`. */
int nb_download_sensor_overlaps(nb_context*, nb_sensor_overlap* host, uint32_t capacity, uint32_t* count, void* stream);

/* Kinematic bodies (moving platforms, elevators, doors, turntables; DESIGN.md section 8.8): bodies that move at the velocity the application
 * gives them, push dynamic bodies and are never pushed back.  The call replaces the set of kinematic bodies with the n listed bodies and writes
 * each one's velocity and angular_velocity into its momentum row (the unused lanes are left alone); n = 0 removes the set, and every body is
 * dynamic again with its momentum row as it stands.  NB_ERR_ARGUMENT, changing nothing: body 0, a body at or beyond the uploaded body count,
 * or a body listed twice.  Asynchronous on `stream`, ordered like nb_upload_momentum; the host array may be reused when the call returns.
 * Calling it every step with the same set and new velocities is the intended way to drive platforms: one small copy and one scatter launch,
 * and nb_step's graph is kept.  A changed set re-records the graph.
 * A kinematic body has infinite mass and inertia wherever the step reads them (setup writes 0 into its momentum unused0), whatever its
 * properties row says.  Only the caller changes its velocity (this call, nb_upload_momentum, nb_upload_bodies): gravity, damping, the warm
 * start, the contact sweeps of both solver modes and the user constraint rows read it and never write it.  It is MOVING when any of its six
 * velocity components is nonzero (-0.0 counts as zero), as the momentum row stands at nb_collide.  A moving kinematic body is active (in the
 * active list, in body-index order) and nb_advance integrates it; one at rest is neither.  Islands: a kinematic body never joins a set; an
 * edge between a dynamic body and a moving kinematic body makes the dynamic body's set active; an edge to a kinematic body at rest is
 * ignored like an edge to body 0.  A pair of colliders on two non-dynamic bodies (kinematic or body 0), at least one of them kinematic, is not
 * a broadphase pair (not counted, no islands, contacts, cache or events), two colliders of one kinematic body included; sensor pairs keep
 * their rules.  The solver substitutes a kinematic side like body 0: no chain, never waited for, excluded from the throughput mass split.
 * nb_upload_bodies keeps the set while the body count is unchanged and removes it when the count changes.  nb_save_state writes it (state
 * version 4), nb_load_state restores it.  Not supported by nb_shard_step (NB_ERR_ARGUMENT).  No extra launch per step.
 * A body made kinematic keeps its nb_set_body_forces entry, which the force stage ignores while the body is kinematic. */
typedef struct { uint32_t body; float velocity[3]; float angular_velocity[3]; uint32_t reserved; } nb_kinematic_body;   /* 32 bytes */
int nb_upload_kinematic_bodies(nb_context*, const nb_kinematic_body* host, uint32_t n, void* stream);

/* Body impulses (hits, kicks, thrusters, explosions, waking; DESIGN.md section 8.9): edits of chosen bodies' momentum rows and idle counters on
 * the device between any two calls, the edit a reference application makes to its host BodyData.  The result is bit-identical to that host
 * loop written with the float32 operations below, left to right, without fused multiply-adds.
 * nb_apply_body_impulses applies the n entries one after the other, in list order wherever two entries name the same body.  For an entry with
 * body b, offset o, impulse J and angular impulse L, with m = b's mass_inverse and W = b's world inverse inertia (computed from b's current
 * rotation and properties row exactly as nb_setup_contact_constraints computes it, nudge.cpp:4182-4199):
 *   v.x += m * J.x                                    (likewise y, z)
 *   t.x  = (o.y*J.z - o.z*J.y) + L.x                  (cyclically for y, z: t = cross(o, J) + L)
 *   w.x += (W.xx*t.x + W.xy*t.y) + W.xz*t.z           (w.y += (W.xy*t.x + W.yy*t.y) + W.yz*t.z; w.z += (W.xz*t.x + W.yz*t.y) + W.zz*t.z)
 * Only the velocity and angular_velocity lanes are written (unused0 / unused1 are left alone), and every listed body gets idle counter 0, also
 * with a zero impulse: a zero impulse is the way to wake a body.  Its island (connected bodies included) is active from the next nb_collide.
 * NB_ERR_ARGUMENT, changing nothing (every entry is checked on the host before any device work): body 0, a body at or beyond the uploaded body
 * count, a kinematic body (drive those with nb_upload_kinematic_bodies), or n > 0 with a null pointer.  n = 0 is a no-op.
 * nb_apply_radial_impulse considers every body i in 1..count-1 that is not kinematic.  With d = p_i - center (p_i = the body's POSITION, its
 * centre of mass, not its colliders' surfaces) and dist = sqrtf((d.x*d.x + d.y*d.y) + d.z*d.z), the body is hit iff dist < radius.  A hit body
 * gets idle counter 0 and, if dist > 0, k = (impulse * (1.0f - dist / radius)) / dist, J = (d.x*k, d.y*k, d.z*k), v += m * J as above (no
 * angular part).  A negative impulse pulls inwards; impulse 0 only wakes.  NB_ERR_ARGUMENT: a null `e`, or a radius that is not finite or not
 * above 0.
 * Both calls are asynchronous on `stream` and ordered like nb_upload_momentum (after a pending nb_upload_bodies side copy); the host array may
 * be reused when the call returns.  They are legal between any two stage calls and keep nb_step's graph.  Launches per call: 3 for a list
 * (n > 0: keys, one radix sort by (body, list position), one thread per body run), 1 for the radial impulse; none per step.  Not tested on a
 * rank's context of nb_shard_step. */
typedef struct {
	uint32_t body;
	float offset[3];            /* world-frame vector from the body's position (its centre of mass) to where the impulse acts; 0 = the centre */
	float impulse[3];           /* linear impulse: velocity += mass_inverse * impulse */
	float angular_impulse[3];   /* extra angular impulse, world frame */
	uint32_t reserved[2];
} nb_body_impulse;              /* 48 bytes */
int nb_apply_body_impulses(nb_context*, const nb_body_impulse* host, uint32_t n, void* stream);
typedef struct { float center[3]; float radius; float impulse; uint32_t reserved[3]; } nb_radial_impulse;   /* 32 bytes */
int nb_apply_radial_impulse(nb_context*, const nb_radial_impulse* e, void* stream);

/* Per-body forces (balloons, zero-g debris, water drag, thrusters, wind, rockets; DESIGN.md section 8.11): a gravity scale, extra damping and a
 * constant force and torque per body, applied on the device inside the step's force stage (nb_apply_gravity_damping, also inside nb_step).
 * nb_set_body_forces writes the n listed bodies' entries into a per-body table; every other body keeps its entry.  The first call (n = 0
 * included) creates the table for max_bodies, every body with the default entry (flags 0, gravity_scale 1, everything else 0).  Every listed
 * body gets idle counter 0, so a body asleep on the ground wakes when its gravity scale changes.  NB_ERR_ARGUMENT, changing nothing (every
 * entry is checked on the host before any device work): body 0, a body at or beyond the body count, a kinematic body, a body listed twice, a
 * null list with n > 0, a field that is not finite, a negative damping, unknown flag bits.  Asynchronous on `stream`, ordered like
 * nb_upload_momentum; the host array may be reused when the call returns.  One copy and one scatter launch (plus one fill launch when it
 * creates the table); legal between any two calls; editing entries keeps nb_step's graph, creating or removing the table re-records it.
 * nb_clear_body_forces removes the table: the step then launches exactly what it launched before the table existed.
 * nb_download_body_forces fills B rows (B = the body count) with body = the row index; without a table these are default rows.
 * NB_ERR_CAPACITY when capacity < B (*count = B).  Synchronises `stream`.  The stored reserved word is 0.
 * The force stage with a table, float32, left to right, without fused multiply-adds.  For every body i of the active list that is not
 * kinematic, with e = i's entry, m = its mass_inverse, q = its rotation, W = its world inverse inertia (computed from q and its properties
 * row exactly as nb_setup_contact_constraints computes it), dt, g and d = the call's time step, gravity and damping:
 *   dv  = g * dt
 *   v.y = v.y - dv * e.gravity_scale
 *   if e.force has a nonzero component (-0.0 counts as zero):
 *       f = LOCAL ? qrot(q, e.force) : e.force        (qrot(q, r): t = 2 * cross(q.xyz, r); r + q.w * t + cross(q.xyz, t), nudge.cpp:1117-1120)
 *       k = m * dt;  v.x = v.x + f.x * k               (likewise y, z)
 *   if e.torque has a nonzero component:
 *       t = LOCAL ? qrot(q, e.torque) : e.torque
 *       w.x = w.x + ((W.xx*t.x + W.xy*t.y) + W.xz*t.z) * dt   (w.y: (W.xy*t.x + W.yy*t.y) + W.yz*t.z; w.z: (W.xz*t.x + W.yz*t.y) + W.zz*t.z)
 *   lin = 1 - dt * (d + e.linear_damping);  ang = 1 - dt * (d + e.angular_damping)
 *   v *= lin (x, y, z);  w *= ang (x, y, z)
 *   if force or torque has a nonzero component: idle[i] = 0
 * A default entry gives exactly the bits of the stage without a table (dv * 1 == dv, d + 0 damps like d, a zero force or torque is skipped).
 * Sleeping: only active bodies get the stage, as without a table.  A body carrying a nonzero force or torque gets idle counter 0 in every
 * step, so its island never sleeps while it is pushed; gravity scale and damping alone do not keep a body awake.
 * A kinematic body's entry is kept but ignored while it is kinematic.  nb_upload_bodies keeps the table while the body count is unchanged and
 * removes it when the count changes.  nb_add_bodies gives the new bodies the default entry; nb_remove_bodies moves the entries with their
 * bodies.  nb_save_state writes the table (state version 5), nb_load_state restores it.  Not supported by nb_shard_step (NB_ERR_ARGUMENT).
 * Cost per step: the stage's one launch reads the 48-byte entry of every active body; no extra launch. */
typedef struct {
	uint32_t body;
	uint32_t flags;             /* NB_BODY_FORCE_LOCAL: force and torque are in the body frame */
	float gravity_scale;        /* multiplies the step's gravity; default 1 */
	float linear_damping;       /* added to the step's damping rate for the velocity; default 0 */
	float angular_damping;      /* added to the step's damping rate for the angular velocity; default 0 */
	float force[3];             /* constant force through the centre of mass; default 0 */
	float torque[3];            /* constant torque; default 0 */
	uint32_t reserved;
} nb_body_force;                /* 48 bytes */
enum nb_body_force_flags { NB_BODY_FORCE_LOCAL = 1 };
int nb_set_body_forces(nb_context*, const nb_body_force* host, uint32_t n, void* stream);
int nb_clear_body_forces(nb_context*, void* stream);
int nb_download_body_forces(nb_context*, nb_body_force* host, uint32_t capacity, uint32_t* count, void* stream);

/* Spawning and despawning (projectiles, debris, pickups, destroyed crates; DESIGN.md section 8.10): bodies and colliders appended to or removed
 * from the device-resident scene between steps, with every table that holds body or collider indices kept.  Each call's result is bit-identical
 * to the host edit below applied to the arrays the context holds, followed by a re-upload of all of them (nb_upload_bodies, nb_upload_colliders,
 * nb_upload_connections, nb_upload_collision_filters with the same flags, nb_upload_sensors with the same max_sensor_pairs,
 * nb_upload_kinematic_bodies with the kinematic bodies' current velocities, nb_upload_constraint_rows with the rows' current impulses,
 * nb_set_body_forces with every non-default entry of the body force table), except that the sensor overlap lists are kept (remapped) where
 * nb_upload_sensors would empty them.
 *
 * nb_remove_bodies(list of n bodies), host edit:
 *   wake:        before anything moves, every kept body gets idle counter 0 when (a) a contact-cache entry's key pairs the tag of one of its
 *                colliders with the tag of a removed collider (tags are compared, so with duplicate tags every collider carrying one counts;
 *                the cache holds the kept entries of sleeping pairs, so a sleeping stack is found), or (b) a connection joins it to a removed
 *                body.  Body 0 and kinematic bodies are never woken.
 *   bodies:      the kept bodies keep their order: old index i becomes i - (number of removed indices below i).  Transform, properties, momentum
 *                row (unused lanes included) and idle counter move with their body.
 *   colliders:   every box and sphere whose transform.body is removed is removed; the kept ones keep their order and get the new index of their
 *                body in transform.body.  Tags are not changed.  The filter and sensor tables (boxes first, then spheres) drop the same entries.
 *   connections: an entry naming a removed body is dropped, the others keep their order with both sides remapped (body 0 stays 0).
 *   kinematic:   removed members leave the set, the others are remapped; an empty set is no set.
 *   forces:      the body force table's entries move with their bodies (a removed body's entry is dropped); the table stays.
 *   rows:        a user constraint row naming a removed body is deleted; the others keep their upload order, their accumulated impulse and the
 *                rest of the row, with a and b remapped (nb_download_constraint_rows then takes the new row count).
 *   joints:      a joint naming a removed body is deleted and the kept dynamic body on its other side gets idle counter 0; the others keep their
 *                upload order, parameters and accumulated impulses, with a and b remapped (as after nb_download_joints, the host edit and
 *                nb_upload_joints).  One more launch when a body is woken this way.
 *   overlaps:    the sensor overlap lists (the current one and the one nb_write_cached_impulses compares against) keep their keys; body_a and
 *                body_b are remapped, a removed side becomes NB_REMOVED_BODY.
 *   The contact cache is NOT edited: its keys are collider tags, so the kept entries stay valid.  A removed collider's entries drop out at the
 *   next nb_write_cached_impulses like any pair that stopped touching (with events: the ordinary NB_CONTACT_END, and NB_SENSOR_END with
 *   NB_REMOVED_BODY from the remapped overlap list).  A collider added with a removed collider's tag before that write continues its cache
 *   entries, as a re-upload with nb_upload_colliders would.
 *   NB_ERR_ARGUMENT, changing nothing (every check runs on the host before any device work): body 0, a body at or beyond the body count, a body
 *   listed twice, a null list with n > 0, a context that nb_shard_create was called on, a user constraint row or a connection that names a
 *   body at or beyond the body count (their uploads accept such indices; every collider's body must be below it too).  NB_ERR_CAPACITY: more connections than the context's
 *   scratch stride (the largest of max_pairs, max_contacts, max_bodies and the collider capacity).  n = 0 is a no-op without a launch.
 *   Synchronises `stream` once (the new collider counts and largest tag decide tagbits and kbits exactly as nb_upload_colliders does).
 *   Launches: 8 (mark, flags, one radix sort of (tag, body) keys, cache wake, body scan + gather, collider scan + gather), + 2 with connections
 *   (scan + gather), + 2 for the NB_FILTER_SKIP_CONNECTED lookup when connections remain, + 1 with user rows left, + 1 with a sensor table;
 *   the body force table adds none (the body gather moves its entries).
 *
 * nb_add_bodies, host edit: the bodies->count rows go to indices B .. B+n-1 and are dynamic; the boxes are appended after the existing boxes and
 *   the spheres after the existing spheres (a collider's transform.body may name any body below B + n, so n = 0 adds colliders to existing
 *   bodies).  While a filter or sensor table exists, `tables` gives the new colliders' entries (boxes first, then spheres), inserted at the
 *   same places: [old boxes][new boxes][old spheres][new spheres].  Connections, rows, the kinematic set and the overlap lists are unchanged.
 *   While a body force table exists the new bodies get the default entry (set theirs with nb_set_body_forces afterwards).
 *   NB_ERR_ARGUMENT, changing nothing: a null array with a nonzero count, a collider body at or beyond B + n, a table pointer that is null
 *   while that table exists and colliders are added, a table pointer given while that table does not exist, a shard context.
 *   NB_ERR_CAPACITY, changing nothing: max_bodies, max_boxes or max_spheres exceeded.  Asynchronous on `stream`, ordered like
 *   nb_upload_momentum; the host arrays may be reused when the call returns, and only the new rows cross PCIe.  Launches: none (copies only).
 *
 * Both calls are for the time between steps (after nb_advance or nb_step, before nb_collide).  After either, the stage calls that use the last
 * nb_collide's outputs (nb_read_cached_impulses, nb_setup_contact_constraints, nb_apply_impulses, nb_update_cached_impulses,
 * nb_write_cached_impulses, nb_advance) return NB_ERR_ARGUMENT until the next nb_collide, nb_step, nb_upload_contacts or nb_load_state.  nb_step re-records its
 * graph when the body, collider or connection counts, tagbits, kbits, the kinematic set or the user rows changed (removing n bodies and adding
 * n back in one gap keeps it); a step of the edited context launches what a freshly uploaded context of the same shape and tables launches.
 * Nothing runs per step.
 * nb_download_colliders fills the host struct (its counts are capacities on input, the stored counts on output; NB_ERR_CAPACITY when one is
 * too small); nb_download_connections fills `capacity` pairs at most (host->count = the stored count; NB_ERR_CAPACITY when it is larger).
 * Both synchronise. */
typedef struct { const nb_collision_filter* filters; const uint8_t* sensor_flags; } nb_spawn_tables;   /* entries of the ADDED colliders, boxes then spheres */
#define NB_REMOVED_BODY 0xffffffffu
int nb_add_bodies(nb_context*, const nb_body_data* bodies, const nb_collider_data* colliders, const nb_spawn_tables* tables /* may be null */, void* stream);
int nb_remove_bodies(nb_context*, const uint32_t* bodies, uint32_t n, void* stream);
int nb_download_colliders(nb_context*, nb_collider_data* host, void* stream);
int nb_download_connections(nb_context*, nb_body_connections* host, uint32_t capacity, void* stream);

/* CUDA streams for hosts that do not link the CUDA runtime (cgo / JNI / ctypes callers): a created stream is capturable, so nb_step
 * replays its CUDA graph there; a null stream means the legacy default stream and plain launches. */
void* nb_stream_create(nb_context*);
void nb_stream_destroy(nb_context*, void* stream);
int nb_stream_synchronize(nb_context*, void* stream);

/* State serialisation (SURVEY.md section 8 f3): the caller-owned PODs of nudge.h:73-129 (BodyData, ColliderData, BodyConnections,
 * ContactCache, widened layout) as one flat file, from / into the device-resident context.  Checkpoint, and what tools/nb_replay
 * steps headless; layout in nudge_b200/csrc/nb_state_api.cuh.  All three synchronise.  A context with a body force table writes version 5
 * (the table's B rows after the kinematic section); loading a file of versions 1-4 removes the context's table.  A context with joints
 * writes version 6 (the joints after the force table); loading a file of versions 1-5 removes the context's joints.  A context with joint
 * drives writes version 7 (reserved[7] = the drive count, the nb_joint_drive rows after the joints); loading a file of versions 1-6 removes
 * the context's drives.  A context with a continuous-collision set writes version 8 (a 16-byte header extension holding the entry count,
 * the nb_ccd_body rows last); loading a file of versions 1-7 removes the context's set.  Without a set a context writes what it wrote
 * before version 8 existed, byte for byte.  A context with joint springs writes version 9 (the extension as in version 8 with reserved[0] =
 * the spring count, the nb_joint_spring rows after the nb_ccd_body rows, padded to 16 bytes); loading a file of versions 1-8 removes the
 * context's springs, and without springs a context writes what it wrote before version 9 existed. */
int nb_save_state(nb_context*, const char* path, void* stream);
int nb_load_state(nb_context*, const char* path, void* stream);
int nb_state_info(const char* path, uint32_t counts[5] /* bodies, boxes, spheres, connections, cache entries */);

/* Device-resident snapshots (DESIGN.md section 8.12): the whole between-steps state in HBM, saved cheaply enough to do every step and restored
 * bit for bit, so that re-stepping with the same inputs repeats the run byte for byte (rollback netcode, resets, what-if planning).
 * A snapshot holds what the next nb_collide / nb_step and everything after it depend on: bodies (transforms, properties, momentum with its
 * unused lanes, idle counters); boxes and spheres (tags, data, transforms); connections; the contact cache (as many entries as the device count
 * says); the filter table, its flags and the NB_FILTER_SKIP_CONNECTED key list; the sensor table, max_sensor_pairs and the sensor overlap list
 * as of the last nb_write_cached_impulses; the kinematic set and its kind bytes; the body force table; the user constraint rows with their
 * accumulated impulses and their levelling; the joints with theirs and their drive table; the solver mode; the contact-event step counter; the body, collider and connection counts and the
 * tag and key bits.  It does not hold whether contact events are enabled, the undrained events, or the outputs of the last nb_collide.
 *
 * nb_snapshot_create allocates device memory for the context's capacities (DESIGN.md section 8.12 gives the bytes); nb_snapshot_destroy frees
 * it, and nb_destroy frees a context's remaining snapshots (their handles are then invalid).
 * nb_snapshot_save is legal between steps and after nb_add_bodies / nb_remove_bodies; between nb_collide and the nb_advance that ends its step
 * it is NB_ERR_ARGUMENT.  It is asynchronous on `stream`, ordered after a pending nb_upload_bodies copy, and is ONE kernel launch with no
 * synchronisation and no allocation, so it can be captured into the application's CUDA graph (the counts, bits and table set it records are
 * those at capture time).  The user rows and the sensor overlap list are sized at the save: a save that finds them grown beyond the snapshot's
 * room grows it, synchronises and allocates, and cannot be captured.
 * nb_snapshot_restore makes the context what it was at the save, bit for bit: tables that exist now and did not then are removed, missing
 * ones are created.  nb_download_sensor_overlaps then returns the overlap list of the save, and the stage calls that read the last collide's
 * outputs are refused until the next nb_collide or nb_step, as after nb_add_bodies.  With every table already allocated it is one kernel
 * launch and host bookkeeping, without synchronisation.  nb_step keeps its graph when the step's launches and their arguments are unchanged:
 * the same counts, tag and key bits, table set, kinematic set, user-row set, joint structure and drive structure; otherwise it re-records once.
 * NB_ERR_ARGUMENT, changing nothing: a snapshot of another context, restoring a snapshot that was never saved, a context that nb_shard_create
 * was called on. */
typedef struct nb_snapshot nb_snapshot;
int nb_snapshot_create(nb_context*, nb_snapshot** out);
void nb_snapshot_destroy(nb_snapshot*);
int nb_snapshot_save(nb_context*, nb_snapshot*, void* stream);
int nb_snapshot_restore(nb_context*, const nb_snapshot*, void* stream);

/* Renderer read-back (SURVEY.md section 8 f4; replaces the per-collider host loop of example/main.cpp:224-268 with its helpers at :53-110):
 * one column-major 4x4 model matrix (16 floats) per collider, boxes first, then spheres; rotation = body * collider, translation =
 * body.rotation applied to collider.position plus body.position, columns scaled by the box half extents / the sphere radius.
 * out_is_device != 0: `out` is a device pointer (a mapped GL / Vulkan buffer), the call is asynchronous on `stream`; otherwise `out`
 * is host memory and the call returns when it is filled.  *count = colliders; NB_ERR_CAPACITY if capacity (in matrices) is smaller. */
int nb_instance_matrices(nb_context*, float* out, uint32_t capacity, int out_is_device, uint32_t* count, void* stream);

/* Ray casts (picking, line of sight, bullets, wheel probes, lidar; DESIGN.md section 8.14): n rays against the colliders as the body
 * transforms stand when the call runs on `stream` (not as of the last nb_collide), answered on the device.  A collider's world transform
 * (p, q) is the one nb_collide computes: p = qrot(q_body, collider.position) + p_body, q = qmul(q_body, collider.rotation).  The point of a
 * ray at t is origin + t * direction; direction need not be unit length, and t and max_t are in units of its length.
 * Which colliders count: collider i is tested iff (category_i & ray.mask) != 0 (category_i from nb_upload_collision_filters, 0xffff without a
 * table), its body != ignore_body (NB_RAY_NO_HIT: ignore none), and it is not a sensor collider unless flags has NB_RAY_SENSORS.  Body 0 and
 * kinematic bodies are solid like any other.
 * Result: the CLOSEST hit, the smallest t in [0, max_t], ties to the smaller collider index (boxes first, then spheres: the index order of the
 * filter and sensor tables).  position = origin + t * direction (per component), collider, its body and tag, reserved 0.  An origin inside a
 * collider hits it at t = 0 with normal (0, 0, 0).  No hit: collider = body = tag = NB_RAY_NO_HIT and every other field 0.  A degenerate ray
 * (a field of origin, direction or max_t not finite, a zero direction, max_t < 0) hits nothing and does not fail the call.
 * The arithmetic is float32, left to right as written, without fused multiply-adds, IEEE division and sqrtf, with cross, dot and qrot as in
 * the joints' section above; o = origin, d = direction, (p, q) the collider's world transform, conj(q) = (-q.x, -q.y, -q.z, q.w):
 *   BOX (half extents h = size):  m = o - p;  lo = qrot(conj(q), m);  ld = qrot(conj(q), d);  enter = 0, exit = max_t, axis = none;
 *     for k = x, y, z in turn:  if ld.k == 0: miss when lo.k < -h.k or lo.k > h.k
 *       else:  t1 = (-h.k - lo.k) / ld.k;  t2 = (h.k - lo.k) / ld.k;  near = t1 < t2 ? t1 : t2;  far = t1 < t2 ? t2 : t1
 *              if near > enter: enter = near, axis = k, s = t1 < t2 ? -1 : +1;   if far < exit: exit = far;   miss when enter > exit
 *     t = enter;  normal = axis == none ? (0, 0, 0) : qrot(q, n_l), n_l = s in component `axis` and +0 in the other two (the lowest axis
 *     wins a tie, since enter only moves on a strictly greater near)
 *   SPHERE (radius r, centre p):  m = o - p;  a = dot(d, d);  b = dot(m, d);  c = dot(m, m) - r*r
 *     c <= 0: t = 0, normal (0, 0, 0);  otherwise disc = b*b - a*c, miss when disc < 0;  t = (-b - sqrtf(disc)) / a, miss unless
 *     0 <= t <= max_t (so a NaN t misses);  t == 0 becomes +0;  normal = (position - p) * (1 / r)
 * Which candidates the device tests is decided by a conservative grid walk (DESIGN.md section 8.14); whether and where a candidate is hit is
 * decided by the arithmetic above alone, so any traversal gives the same bytes.
 * on_device != 0: rays and hits are device pointers (4-byte alignment suffices, as for the host arrays); the call is asynchronous on `stream`, and after the first call on a context it makes no
 * synchronisation and no allocation, so it can be captured into the application's CUDA graph (a replay reads the transforms of its moment).
 * on_device == 0: host pointers; the rays are staged like the editing calls' arrays, and the call returns with `hits` filled.  Legal between
 * any two calls, stage calls included; it changes nothing that a step, a download or a snapshot can observe (its scratch is its own:
 * 181 to 213 bytes per collider of capacity, allocated on the first call).  NB_ERR_ARGUMENT, changing nothing: a null pointer with n > 0, unknown
 * flag bits, a context that nb_shard_create was called on.  Launches: 7 per call with n > 0 (reset, world transforms and AABBs, Morton codes,
 * one radix sort, leaves, grid table, the walk), 1 (the walk alone) when the scene has no collider or no body, none with n = 0. */
typedef struct { float origin[3]; float max_t; float direction[3]; uint32_t mask; uint32_t ignore_body; uint32_t reserved[3]; } nb_ray;        /* 48 bytes */
typedef struct { float position[3]; float t; float normal[3]; uint32_t collider; uint32_t body; uint32_t tag; uint32_t reserved[2]; } nb_ray_hit; /* 48 bytes */
enum nb_ray_flags { NB_RAY_SENSORS = 1 };   /* also test sensor colliders (default: they are skipped) */
#define NB_RAY_NO_HIT 0xffffffffu
int nb_raycast(nb_context*, const nb_ray* rays, uint32_t n, nb_ray_hit* hits, uint32_t flags, int on_device, void* stream);

/* Overlap queries (area damage, perception cones and boxes, selection boxes, spawn-point checks, proximity observations; DESIGN.md section
 * 8.15): which colliders touch each of n spheres or oriented boxes, against the colliders as the body transforms stand when the call runs on
 * `stream`, answered on the device.  A collider's world transform is nb_raycast's, and which colliders count is nb_raycast's rule: collider i
 * counts iff (category_i & query.mask) != 0, its body != ignore_body (NB_RAY_NO_HIT: ignore none), and it is not a sensor collider unless
 * flags has NB_OVERLAP_SENSORS.  Body 0 and kinematic bodies are solid like any other.
 * Result: the hits ordered by query, then by ascending collider index (boxes first, then spheres); offsets[q] .. offsets[q + 1] is query q's
 * range and offsets[n] the total.  A hit is (query, collider, its body, its tag).  The order is defined without reference to any traversal,
 * so any walk gives the same bytes.  Overflow: when the total exceeds `capacity` (in hits), only offsets[n] is defined and holds the total
 * needed; a host-pointer call then returns NB_ERR_CAPACITY, a device-pointer call writes it and returns NB_OK.
 * A degenerate query hits nothing and does not fail the call: an unknown shape, a field the shape reads that is not finite (SPHERE reads
 * center and radius; BOX center, rotation and half_extents; fields a shape does not read are not read), a negative radius or half extent, a
 * BOX rotation with dot(q, q) == 0.  The device decides this, since device-pointer queries cannot be checked on the host.
 * The tests are float32, left to right as written, without fused multiply-adds, with cross, dot and qrot as in the joints' section above;
 * (p, q) is the collider's world transform, h its half extents (box size), rc its radius, conj(q) = (-q.x, -q.y, -q.z, q.w), e_x, e_y, e_z
 * the unit axes.  A BOX query's rotation is used as given, not normalised.  Touching counts: every comparison is closed, unlike the
 * broadphase's strict AABB rule.
 *   SPHERE (c, r) vs SPHERE:  d = c - p;  overlap iff dot(d, d) <= (r + rc) * (r + rc)
 *   SPHERE (c, r) vs BOX:     l = qrot(conj(q), c - p);  per axis k: g_k = l_k < -h_k ? l_k + h_k : (l_k > h_k ? l_k - h_k : +0);
 *                             overlap iff dot(g, g) <= r * r
 *   BOX (c, Q, H) vs SPHERE:  the same with l = qrot(conj(Q), p - c), H for h and rc for r
 *   BOX (c, Q, H) vs BOX:     u_k = qrot(Q, e_k), v_k = qrot(q, e_k);  t = p - c;  the axes in this order: u_x, u_y, u_z, v_x, v_y, v_z, then
 *                             cross(u_i, v_j) for i = x, y, z and, inside, j = x, y, z;  for axis L:
 *                             ra = (fabsf(H.x * dot(u_x, L)) + fabsf(H.y * dot(u_y, L))) + fabsf(H.z * dot(u_z, L)), rb likewise with h and v;
 *                             separated when fabsf(dot(t, L)) > ra + rb;  overlap iff no axis separates
 * No epsilon guards parallel edges: a zero cross axis cannot separate (0 > 0 is false), and any nonzero axis is a valid separating test.
 * Which candidates the device tests is decided by a conservative grid walk (DESIGN.md section 8.15); whether a candidate overlaps is decided
 * by the tests above alone.
 * on_device != 0: queries, hits and offsets are device pointers (4-byte alignment suffices); the call is asynchronous on `stream`, and a call
 * whose capacity is at most the largest an earlier call on the context used makes no synchronisation and no allocation, so it can be
 * captured into the application's CUDA graph.  A call with a larger capacity grows the hit-key scratch (synchronises and allocates).
 * on_device == 0: host pointers; the queries are staged like the editing calls' arrays, and the call returns with offsets and hits filled.
 * Legal between any two calls, stage calls included; it changes nothing that a step, a download or a snapshot can observe.  Scratch: the
 * ray casts' (181 to 213 bytes per collider of capacity, allocated on the first query of either kind) plus 16 bytes per hit of capacity, and
 * for a host-pointer call 64 bytes per query, 4 per offset and 16 per hit of capacity.  NB_ERR_ARGUMENT, changing nothing: a null queries or
 * offsets pointer with n > 0, a null hits pointer with n > 0 and capacity > 0, unknown flag bits, a context that nb_shard_create was called
 * on.  Launches: 9 per call with n > 0 (reset, world transforms and AABBs, Morton codes, one radix sort, leaves, grid table, the walk, the
 * hit sort, the write), 1 (the write alone) when the scene has no collider or no body, none with n = 0 or a refused call; none per step. */
typedef struct {
	uint32_t shape;             /* NB_OVERLAP_SPHERE or NB_OVERLAP_BOX */
	float center[3];
	float rotation[4];          /* BOX: x, y, z, w, used as given (not normalised) */
	float half_extents[3];      /* BOX */
	float radius;               /* SPHERE; 0 = a point query */
	uint32_t mask;              /* collider i counts iff (category_i & mask) != 0, as for rays */
	uint32_t ignore_body;       /* NB_RAY_NO_HIT: ignore none */
	uint32_t reserved[2];
} nb_overlap_query;             /* 64 bytes */
typedef struct { uint32_t query, collider, body, tag; } nb_overlap_hit;   /* 16 bytes */
enum nb_overlap_shape { NB_OVERLAP_SPHERE = 0, NB_OVERLAP_BOX = 1 };
enum nb_overlap_flags { NB_OVERLAP_SENSORS = 1 };   /* also test sensor colliders (default: they are skipped) */
int nb_overlap(nb_context*, const nb_overlap_query* queries, uint32_t n, nb_overlap_hit* hits, uint32_t capacity, uint32_t* offsets /* n + 1 */,
               uint32_t flags, int on_device, void* stream);

/* Shape casts (character controllers, thick projectiles, wheel probes, placement, camera collision; DESIGN.md section 8.16): where each of
 * n spheres or oriented boxes first touches a collider when its centre moves from shape.center along direction, against the colliders as
 * the body transforms stand when the call runs on `stream`, answered on the device.  The centre at t is center + t * direction; direction
 * need not be unit length.  The shape translates only; it does not rotate during the sweep.  The shape, its mask and ignore_body follow
 * nb_overlap's struct and rules, and so does which colliders count (NB_SHAPECAST_SENSORS also tests sensor colliders).
 * Result: one nb_ray_hit per cast, the CLOSEST hit: the smallest t in [0, max_t], ties to the smaller collider index (boxes first, then
 * spheres).  position = center + t * direction (per component); normal = the collider's surface normal at the contact, pointing from the
 * collider towards the cast shape, of unit length up to rounding; collider, its body and tag as for rays; reserved 0.  No hit: collider =
 * body = tag = NB_RAY_NO_HIT and every other field 0.  A degenerate cast hits nothing and does not fail the call: a shape nb_overlap calls
 * degenerate, a field of direction or max_t that is not finite, a zero direction, max_t < 0.  The device decides this.
 * The arithmetic is float32, left to right as written, without fused multiply-adds, IEEE division and sqrtf, with cross, dot and qrot as in
 * the joints' section above and nb_overlap's notation; d = direction.  For each counted collider:
 *   0. START:  if nb_overlap's test of the shape at center and this collider holds, the hit is t = 0 with normal (0, 0, 0).  Otherwise:
 *   1. SPHERE (c, r) vs SPHERE:  nb_raycast's sphere test from origin c along d with radius rs = r + rc (its inside branch cannot be reached
 *      after step 0); normal = (c + t*d - p) * (1 / rs)
 *   2. SPHERE (c, r) vs BOX:  the ray lo + t*ld, lo = qrot(conj(q), c - p), ld = qrot(conj(q), d), against the box h rounded by r, which is
 *      the union of 23 primitives tested in this order; the smallest t wins, ties to the earlier primitive; n_l = the local normal:
 *      (a) three face boxes, k = x, y, z: nb_raycast's box test (the slab test) on lo, ld with h.k alone replaced by h.k + r; n_l = the slab
 *          test's local normal (s in component `axis`, +0 elsewhere; (0, 0, 0) when no axis was recorded)
 *      (b) twelve edge cylinders: axis k = x, y, z and, inside, the sign pairs (s_i, s_j) = (-,-), (-,+), (+,-), (+,+) of the other two axes
 *          i < j:  m_i = lo.i - s_i h.i;  m_j = lo.j - s_j h.j;  a = ld.i*ld.i + ld.j*ld.j;  b = m_i*ld.i + m_j*ld.j;
 *          cc = (m_i*m_i + m_j*m_j) - r*r;  miss when a == 0;  disc = b*b - a*cc, miss when disc < 0;  t = (-b - sqrtf(disc)) / a, miss
 *          unless 0 <= t <= max_t (a NaN t misses), t == 0 becomes +0;  miss unless -h.k <= lo.k + t*ld.k <= h.k;
 *          n_l = (m_i + t*ld.i) * (1 / r) in component i, (m_j + t*ld.j) * (1 / r) in j, +0 in k
 *      (c) eight corner spheres at e = (s_x h.x, s_y h.y, s_z h.z), signs in binary order with x slowest ((-,-,-), (-,-,+), (-,+,-), ...):
 *          m = lo - e;  a = dot(ld, ld);  b = dot(m, ld);  cc = dot(m, m) - r*r;  disc = b*b - a*cc, miss when disc < 0;
 *          t = (-b - sqrtf(disc)) / a, miss unless 0 <= t <= max_t, t == 0 becomes +0;  n_l = (lo + t*ld - e) * (1 / r)
 *      With r == 0 only (a) is tested (the three face boxes are then one box, so the cast is nb_raycast's ray).  normal = n_l == (0, 0, 0) ?
 *      (0, 0, 0) : qrot(q, n_l)
 *   3. BOX (c, Q, H) vs SPHERE:  test 2 with the roles swapped, the sphere collider moving along -d (negated per component) against the
 *      query box: lo = qrot(conj(Q), p - c), ld = qrot(conj(Q), -d), H for h, rc for r;  normal = n_l == (0, 0, 0) ? (0, 0, 0) : -qrot(Q, n_l)
 *   4. BOX (c, Q, H) vs BOX:  nb_overlap's 15 axes in its order with its ra and rb;  t0 = p - c;  enter = 0, exit = max_t, axis = none;  for
 *      each axis L:  a = dot(t0, L);  b = dot(d, L);  R = ra + rb;
 *        if b == 0: miss when fabsf(a) > R (otherwise the axis sets no bound)
 *        else: t1 = (a - R) / b;  t2 = (a + R) / b;  near = t1 < t2 ? t1 : t2;  far = t1 < t2 ? t2 : t1;
 *              if near > enter: enter = near, axis = L, sb = b;   if far < exit: exit = far;   miss when enter > exit
 *      t = enter;  normal = axis == none ? (0, 0, 0) : (sb > 0 ? -L : L) * (1 / sqrtf(dot(L, L)))
 *      A zero cross axis never bounds anything (b == 0 and fabsf(a) > R is false), as in nb_overlap's test.
 * The hit key is (bits of t) << 32 | collider, so the smallest t, then the smallest collider, wins.  Which candidates the device tests is
 * decided by a conservative grid walk (DESIGN.md section 8.16); whether and where a candidate is hit is decided by the arithmetic above alone.
 * on_device != 0: casts and hits are device pointers (4-byte alignment suffices); the call is asynchronous on `stream`, and after the first
 * scene query on the context it makes no synchronisation and no allocation, so it can be captured into the application's CUDA graph.
 * on_device == 0: host pointers; the casts are staged like the editing calls' arrays (80 bytes per cast), and the call returns with `hits`
 * filled.  Legal between any two calls, stage calls included; it changes nothing that a step, a download or a snapshot can observe.
 * Scratch: the ray casts'.  NB_ERR_ARGUMENT, changing nothing: a null pointer with n > 0, unknown flag bits, a context that nb_shard_create
 * was called on.  Launches: 7 per call with n > 0 (reset, world transforms and AABBs, Morton codes, one radix sort, leaves, grid table, the
 * walk), 1 (the walk alone) when the scene has no collider or no body, none with n = 0; none per step. */
typedef struct {
	nb_overlap_query shape;     /* the shape at t = 0, its mask and ignore_body: nb_overlap's struct and rules */
	float direction[3];         /* the shape's centre at t is center + t * direction; need not be unit length */
	float max_t;
} nb_shape_cast;                /* 80 bytes */
enum nb_shapecast_flags { NB_SHAPECAST_SENSORS = 1 };   /* also test sensor colliders (default: they are skipped) */
int nb_shapecast(nb_context*, const nb_shape_cast* casts, uint32_t n, nb_ray_hit* hits, uint32_t flags, int on_device, void* stream);

/* Continuous collision for fast bodies (bullets, dropped crates, debris; DESIGN.md section 8.18): CCD motion clamping, answered on the
 * device inside the step.  The step is otherwise discrete: a body that moves further in one step than what it should hit is thick passes
 * through it.  nb_upload_ccd_bodies replaces the set of listed bodies (n = 0 removes it; stored ascending by body);
 * nb_download_ccd_bodies returns it in that order (*count = its size; NB_ERR_CAPACITY when capacity is smaller, nothing written).
 * In every nb_advance (a stage call or inside nb_step, both solver modes) each listed body that the step advances (awake: its island is
 * active in the last nb_collide, and not kinematic) is handled as follows, with p = its position as nb_advance finds it and v = its
 * velocity after the solver:  d = (v.x*dt, v.y*dt, v.z*dt), the products the advance adds.  If (d.x*d.x + d.y*d.y) + d.z*d.z >
 * motion_threshold * motion_threshold and d is a valid direction for nb_shapecast with max_t = 1 (finite, not zero), a sphere of `radius`
 * is cast from p along d with max_t = 1, with nb_shapecast's sphere arithmetic above (steps 0, 1 and 2, float32, no fused multiply-adds),
 * against every collider at its pose of this step's nb_collide except:
 *   - the body's own colliders;  sensor colliders;
 *   - colliders failing Box2D's rule against (category, mask): (category & collider mask) != 0 and (collider category & mask) != 0, the
 *     collider's words from nb_upload_collision_filters (every bit set without a table);
 *   - with NB_FILTER_SKIP_CONNECTED, colliders of a body connected to this one;
 *   - colliders the sphere already touches at t = 0 (step 0 holds): unlike nb_shapecast they are not a t = 0 hit but are skipped, since
 *     nb_collide gives the body a contact with them anyway (a body resting on the ground keeps moving along it);
 *   - a hit at t = 0 on a collider step 0 does not hold for, unless d points into it: dot(g, d') < 0, with g the gap of nb_overlap's
 *     sphere test and d' = qrot(conj(q), d) for a box (g = (gap(l.x, h.x), gap(l.y, h.y), gap(l.z, h.z)), l = qrot(conj(q), c - p),
 *     gap(u, h) = u < -h ? u + h : (u > h ? u - h : 0)), g = c - p and d' = d for a sphere.  Where a clamp leaves the centre on a face, the
 *     face slab of step 2 can count the start as inside while step 0, rounded the other way, does not; without this rule every later cast
 *     from there would hit at t = 0, also one moving away from the face or along it.
 * The hit is the smallest (bits of t) << 32 | collider among the rest.  With a hit the translation is ((v.x*dt) * t, (v.y*dt) * t,
 * (v.z*dt) * t) in place of d (for t = 1 the same bits); the rotation, the velocity and the idle counter are integrated exactly as without
 * a set.  So a clamped body stops where its swept sphere first touches something; with radius below the body's inscribed radius its collider
 * then overlaps what it hit, and the next nb_collide gives an ordinary contact that the solver resolves.  Limitations: targets are taken at
 * their pose before the advance (a moving target is not swept), rotation is not swept, and the remaining time after the impact is dropped.
 * Refusals (NB_ERR_ARGUMENT, changing nothing; every entry checked on the host first): body 0, at or beyond the body count or kinematic; a
 * body listed twice; a radius that is not finite or below 0; a NaN or negative threshold; a null list with n > 0; a context that
 * nb_shard_create was called on.  nb_advance with a set refuses (NB_ERR_ARGUMENT, launching nothing) when no nb_collide ran since the last
 * nb_advance: the collide's grid must describe this step's poses.  A body made kinematic after the upload keeps its entry but is not
 * clamped while kinematic.  New radii, thresholds or filters for the same bodies keep nb_step's graph; another body list re-records it.
 * nb_upload_bodies keeps the set while the body count is unchanged and removes it otherwise; nb_add_bodies adds no entries;
 * nb_remove_bodies drops the removed bodies' entries and renumbers the rest.  Snapshots carry the set; nb_save_state writes it (state
 * version 8) and nb_load_state installs it, a file of an older version removes it.  Not supported by nb_shard_step (NB_ERR_ARGUMENT).
 * Launches: nb_step issues one more (the cast, k_ccd) with a set.  nb_debug_read("ccd_hits") returns, per entry of the last advance in set
 * order, two uint32 (bits of t, collider), (1.0f, NB_RAY_NO_HIT) when the body was not clamped; nb_debug_read("ccd_fallbacks") the casts
 * that tested every collider instead of walking the grid, summed over the context's advances. */
typedef struct {
	uint32_t body;
	float radius;              /* the swept sphere, centred on the body's position; should not exceed the body's inscribed radius */
	float motion_threshold;    /* cast only when the step's translation is longer than this; 0 = always, +inf = never */
	uint16_t category, mask;   /* the collision filter the cast applies (nb_collision_filter's meaning) */
} nb_ccd_body;                 /* 16 bytes */
int nb_upload_ccd_bodies(nb_context*, const nb_ccd_body* host, uint32_t n, void* stream);   /* replaces the set; n = 0 removes it */
int nb_download_ccd_bodies(nb_context*, nb_ccd_body* host, uint32_t capacity, uint32_t* count, void* stream);

/* Body states (observations, environment resets, respawns, teleports, netcode corrections; DESIGN.md section 8.19): the indexed gather and
 * scatter of chosen bodies' poses and velocities on the device, with one 64-byte row both ways, so that a gather, an edit in the
 * application's own device buffers and a set work on one array.
 * nb_get_body_states: row i holds body b = bodies[i] (bodies null: b = i): position and rotation from its transform, velocity and
 * angular_velocity from its momentum row, idle_counter = its idle counter, body = b, reserved = 0.  Body 0 is legal.  Legal between any two
 * calls; ordered after a pending nb_upload_bodies side copy.  One launch (none with n = 0).  A null out with n > 0 is NB_ERR_ARGUMENT.
 *   on_device == 0: host pointers; an index at or beyond the body count or a null bodies with n > B is NB_ERR_ARGUMENT, changing nothing;
 *   the call synchronises `stream` and returns with `out` filled.
 *   on_device != 0: bodies (may be null) and out are device pointers, out 16-byte aligned; asynchronous on `stream`.  An index at or beyond
 *   the body count gives body = NB_REMOVED_BODY and every other field 0.
 * nb_set_body_states: the result is bit-identical to this host edit of the arrays the context holds followed by nb_upload_bodies:
 *   for each entry, in list order (so where a body is listed twice the later entry's fields win):
 *     NB_BODY_POSE:      the body's transform gets position and rotation as given (no normalisation; its body word is left alone)
 *     NB_BODY_VELOCITY:  its momentum row gets velocity and angular_velocity as given (unused0 / unused1 are left alone); for a kinematic
 *                        body this is its kinematic velocity, exactly as nb_upload_kinematic_bodies writes it (the set is not changed)
 *     every listed dynamic body gets idle counter 0; a listed kinematic body keeps its idle counter
 *   wake, NB_BODY_POSE only: nb_remove_bodies' rules (a) and (b) with "removed" read as "moved": a body gets idle counter 0 when (a) a
 *     contact-cache entry's key pairs the tag of one of its colliders with the tag of a moved body's collider (tags are compared, so with
 *     duplicate tags this over-wakes exactly as removal does), or (b) a connection joins it to a moved body.  Body 0 and kinematic bodies are
 *     never woken.  With NB_BODY_VELOCITY alone no partner is woken, as with nb_apply_body_impulses: a woken body's island is found at the next
 *     nb_collide through its unchanged pairs.
 *   Not edited: the contact cache, the joints (their rows are rebuilt from the new transforms at the next step; their accumulated impulses
 *   are kept), the sensor overlap lists (recomputed at the next nb_collide; events follow as usual), the continuous-collision set and the body
 *   force table.  So a body moved to where it touches the same partner again warm-starts from the old cache entry, as the host edit would.
 *   Refusals (NB_ERR_ARGUMENT, changing nothing): fields == 0 or an unknown field bit; a context that nb_shard_create was called on;
 *   NB_BODY_POSE between nb_collide and the nb_advance that ends its step (the wake uses collide-stage scratch, and the advance's
 *   continuous collision assumes that the last nb_collide's grid describes the poses); NB_BODY_POSE while a connection names a body at
 *   or beyond the body count (nb_upload_connections accepts such indices; the wake, like nb_remove_bodies', needs them below it, and as
 *   for removal every collider's body must be below it too).  NB_BODY_VELOCITY alone is legal between any two calls.
 *   on_device == 0: host pointers; every entry is checked before any device work: body 0, a body at or beyond the body count, a selected
 *   field that is not finite, or a null pointer with n > 0 is NB_ERR_ARGUMENT.  *skipped (when not null) is set to 0.  The array may be
 *   reused when the call returns.
 *   on_device != 0: states (16-byte aligned) and skipped (may be null) are device pointers.  An entry failing the host path's checks is
 *   skipped on the device, and *skipped is written (not accumulated) with the number skipped.
 *   Asynchronous on `stream`, ordered like nb_upload_momentum.  Launches: 3 (keys, one radix sort by (body, list position), one thread per
 *   body run) for NB_BODY_VELOCITY alone; a pose set adds removal's wake: 3 more (flags and keys, one radix sort of (tag, body) keys, cache
 *   wake), 1 more without colliders; none with n = 0.
 * Neither call changes nb_step's graph, holds state, or adds anything to the step, a snapshot or a state file.  on_device != 0 can be captured
 * into the application's CUDA graph once an earlier call on the context had at least n entries (a call with more grows the scratch:
 * it synchronises and allocates, and a captured graph of the old size must be captured again).  A captured call holds the scene's shape
 * as of its capture: the body count, and for a set the collider and connection counts, the sort's digit count and, for a pose set's wake,
 * the tag bits; the refusals above are decided at capture.  Capture again after any edit of the scene's shape: nb_add_bodies,
 * nb_remove_bodies, nb_upload_bodies with another count, nb_upload_colliders, nb_upload_connections, nb_load_state. */
typedef struct {
	float position[3]; uint32_t body;              /* get: the index read; set: the body to edit */
	float rotation[4];                             /* x, y, z, w */
	float velocity[3]; uint32_t idle_counter;      /* get: the body's idle counter; set: ignored */
	float angular_velocity[3]; uint32_t reserved;  /* get: 0; set: ignored */
} nb_body_state;                                   /* 64 bytes */
enum nb_body_state_fields { NB_BODY_POSE = 1, NB_BODY_VELOCITY = 2 };
int nb_get_body_states(nb_context*, const uint32_t* bodies /* null: bodies 0 .. n-1 */, uint32_t n, nb_body_state* out, int on_device, void* stream);
int nb_set_body_states(nb_context*, const nb_body_state* states, uint32_t n, uint32_t fields, uint32_t* skipped /* may be null */, int on_device,
                       void* stream);

/* Contact impulse reports (net contact force per body for observations and rewards, impact strength per touching pair for sounds and damage,
 * the load on a pressure plate or a kinematic platform; DESIGN.md section 8.22): read on the device from the contact set of the last solved
 * step.  Nothing is computed per step: a step that nobody reports on costs nothing more, and neither call changes nb_step or its graph.
 * What both read: the contacts c of the last nb_collide or nb_upload_contacts (index order = nb_download_contacts' order), their (tag,
 * feature) order of nb_read_cached_impulses, and J_c, the world-frame impulse of contact c as nb_update_cached_impulses wrote it:
 * J_c = s0*n + s1*u + s2*v of k_update_impulses, the value the contact cache receives.  J_c is the step's total impulse (warm start plus
 * every sweep's delta); divide by the time step for a force.  Side a of a contact received -J_c, side b +J_c (the solver's convention).  In
 * throughput mode the impulses vary from run to run (see nb_set_solver_mode); the reports are a deterministic function of them.  After a
 * step whose schedule overflowed (NB_ERR_OVERFLOW with bit 4 from nb_download_counts) the per-body report has no contact sides and the
 * pair report reads impulses that were not solved.
 * When legal: from the end of nb_update_cached_impulses (also inside nb_step, and after its graph is replayed) until one of nb_collide,
 * nb_upload_contacts, nb_read_cached_impulses, nb_setup_contact_constraints, nb_apply_impulses (they rewrite the contacts, the impulses or the
 * solver rows), nb_add_bodies, nb_remove_bodies, nb_upload_bodies, nb_upload_colliders, nb_snapshot_restore or nb_load_state (they renumber or
 * replace bodies or state), each of which ends it also when it fails.  nb_write_cached_impulses, nb_advance, nb_apply_body_impulses,
 * nb_set_body_states, the scene queries and the gathers leave the report valid and unchanged.  Otherwise, on a fresh context, and on a
 * context nb_shard_create was called on, both calls are NB_ERR_ARGUMENT, changing nothing.  A device-pointer call decides this when it is
 * called or captured: capture it after nb_step in the same graph.
 * The arithmetic is float32, left to right as written, without fused multiply-adds, with cross and dot of the joints section above.
 *
 * nb_get_body_contact_impulses: row i holds b = bodies[i] (bodies null: b = i).  acc = tq = (+0, +0, +0), k = 0; for every contact c in
 * ascending index order, side a before side b, for each side of c whose body is b:
 *   r = position_c - p_b (per component), p_b the body's position as the step's solve used it (its position at the step's start: nothing
 *       moves a body between nb_collide and nb_advance), exactly the lever arm nb_setup_contact_constraints stored in the contact's row;
 *   side a: acc = acc - J_c, tq = tq - cross(r, J_c);  side b: acc = acc + J_c, tq = tq + cross(r, J_c);  k = k + 1.
 * impulse = acc, angular_impulse = tq (about p_b), contacts = k, body = b.  Body 0 and kinematic bodies report what acts on them (the load on
 * the ground or on a platform), though the solver never moves them.  A body whose island sleeps reports zeros and contacts = 0: a sleeping
 * island has no contacts in the step because it is not solved.  Joint and user-row impulses are not included; they are read with
 * nb_download_joints, nb_download_joint_drives, nb_download_joint_springs and nb_download_constraint_rows.  A null out with n > 0 is
 * NB_ERR_ARGUMENT.  Launches: 3 (one key per contact side, one radix sort by (body, contact, side), one warp per row that finds its body's
 * keys by binary search and sums them in that order); none with n = 0.
 *   on_device == 0: host pointers; an index at or beyond the body count or a null bodies with n > B is NB_ERR_ARGUMENT, changing nothing;
 *   the call synchronises `stream` and returns with `out` filled.
 *   on_device != 0: bodies (may be null) and out are device pointers, out 16-byte aligned; asynchronous on `stream`.  An index at or beyond
 *   the body count gives body = NB_REMOVED_BODY and every other field 0.
 *
 * nb_get_contact_pair_impulses: a pair is a run of contacts with equal tags in (tag, feature) order (with duplicate collider tags two
 * collider pairs may share a key and then form one row, as in the cache and the events).  Over the run, in that order from +0:
 * normal_impulse = the sum of dot(J_c, n_c), impulse = the sum of J_c, contacts = the run's length.  The deepest contact is the run's first,
 * replaced only by a later one with a strictly greater penetration (a tie keeps the earlier contact, a NaN never wins); body_a, body_b and
 * penetration are that contact's.  impulse, contacts, penetration and the bodies are those of an NB_CONTACT_BEGIN event for the same pair in
 * the same step, bit for bit.  A row is kept iff normal_impulse >= min_normal_impulse, or min_normal_impulse is -INFINITY (which keeps every
 * pair); kept rows come in ascending tags order.  *count = the number of kept rows, and the first min(capacity, *count) of them are written.
 * A NaN threshold or a null count is NB_ERR_ARGUMENT, and so is a null out with capacity > 0.  capacity = 0 asks for the count.
 * Launches: 5 (run-head flags, a scan that counts the runs, one thread per run head for its sums and its kept flag, a scan of the kept
 * flags into *count, the scatter).
 *   on_device == 0: host pointers; the call synchronises `stream`, and returns NB_ERR_CAPACITY after writing capacity rows when *count >
 *   capacity.
 *   on_device != 0: out (16-byte aligned) and count are device pointers; asynchronous on `stream`, NB_OK whatever the count.
 * Scratch: allocated for the context's contact capacity on a call's first use, which synchronises: 48 bytes per contact of capacity for the
 * per-body call (its sort keys and slots) and 56 for the pair call (its flags and per-run rows), plus for a host-pointer call 32 bytes per
 * row (and 4 per index) or 48 per row of min(capacity, contact capacity).  After that neither device-pointer call allocates or
 * synchronises, so both can be captured into the application's CUDA graph.  A captured per-body call holds the body count as of its
 * capture: capture again after nb_add_bodies, nb_remove_bodies or nb_upload_bodies with another count. */
typedef struct {
	float impulse[3]; uint32_t body;               /* net contact impulse on the body this step; the index read */
	float angular_impulse[3]; uint32_t contacts;   /* net contact angular impulse about the body's position; contact sides counted */
} nb_body_contact_impulse;                         /* 32 bytes */
typedef struct {
	uint64_t tags;                 /* the pair word A | (uint64)B << 32, the cache and event key */
	uint32_t body_a, body_b;       /* bodies of the pair's deepest contact (the event rule) */
	uint32_t contacts;
	float normal_impulse;          /* sum of dot(J_c, n_c) over the pair's contacts */
	float impulse[3];              /* sum of J_c (the impulse on body_b; body_a received its negation) */
	float penetration;             /* the deepest contact's penetration */
	uint32_t reserved[2];          /* 0 */
} nb_contact_pair_impulse;         /* 48 bytes */
int nb_get_body_contact_impulses(nb_context*, const uint32_t* bodies /* null: bodies 0 .. n-1 */, uint32_t n, nb_body_contact_impulse* out,
                                 int on_device, void* stream);
int nb_get_contact_pair_impulses(nb_context*, float min_normal_impulse, nb_contact_pair_impulse* out, uint32_t capacity, uint32_t* count,
                                 int on_device, void* stream);

/* Solver mode.  NB_SOLVER_PARITY (default): the reference's exact Gauss-Seidel order (nudge.cpp:4206-4340 schedule, 4640-4855 sweeps),
 * bit-identical impulses.  NB_SOLVER_THROUGHPUT: mass-splitting Jacobi over the same constraint rows (nudge_b200/csrc/nb_jacobi.cuh) -
 * order independent, HBM-streaming, converges to the same contact problem but its impulses after N sweeps differ from the reference's
 * (validated by invariants and against a CPU restatement within a tolerance, tests/test_gpu_throughput.py).  Takes effect from the
 * next nb_setup_contact_constraints / nb_step.  The NB_SOLVER=throughput environment variable selects it at nb_create. */
enum nb_solver_mode { NB_SOLVER_PARITY = 0, NB_SOLVER_THROUGHPUT = 1 };
int nb_set_solver_mode(nb_context*, int mode);
int nb_get_solver_mode(const nb_context*);

/* CUDA-event timing of the dominant solver kernel across plain (non-graph) launches; see nb_api.cu. */
int nb_debug_timing_enable(nb_context*, int on);
int nb_debug_timing(nb_context*, uint32_t* launches, float* total_ms, void* stream);

/* Kernel-launch counter (every kernel this library launches increments it) and named device buffers for parity tests. */
uint64_t nb_launch_count(const nb_context*);
int nb_debug_read(nb_context*, const char* name, void* dst, size_t max_bytes, size_t* bytes, void* stream); /* synchronises */

int nb_debug_enable(nb_context*, int on);  /* keep the sorted broadphase pair list readable as "pair_keys" */
int nb_debug_sort(nb_context*, uint64_t* keys, uint32_t* vals /* may be null */, uint32_t n, int begin_bit, int end_bit); /* host pointers, in place */
int nb_debug_scan(nb_context*, uint32_t* data, uint32_t n, uint32_t* total);                                             /* exclusive scan, in place */

/* rcpps / rsqrtps model (SURVEY.md §0.5): tables are sampled from the host CPU in nb_create. */
int nb_debug_rcp(nb_context*, const float* x, float* y, uint32_t n, int rsqrt);  /* runs the device LUT path; host pointers */
int nb_lut_model_exact(const nb_context*);  /* 1 if the host CPU's rcpps/rsqrtps match the truncated-mantissa model on 2^20 probes */

#ifdef __cplusplus
}
#endif
#endif
