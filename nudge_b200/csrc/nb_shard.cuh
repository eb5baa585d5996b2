// nudge_b200 — one scene sharded across GPUs: the C++ host of SURVEY.md §8(e), behind the C ABI (nb_shard_*, include/nudge_b200.h).
//
// One process (or thread) per GPU.  A rank simulates its OWNED bodies plus GHOST copies of neighbouring bodies with the complete
// single-GPU pipeline; after the warm start and after every solver sweep each ghost's BodyMomentum row (32 B) is replaced by its
// owner's.  Two transports for that exchange, bit-identical in effect:
//
//   NB_SHARD_NCCL  pack (gather export rows) -> ONE ncclAllGather over NVLink/NVSwitch -> unpack (scatter into ghost rows): what
//                  BASELINE.json's north_star prescribes.  NCCL is bound at run time (dlopen libnccl.so.2: the copy torch loaded,
//                  or the system one), so the library itself has no link-time dependency on it.
//   NB_SHARD_PEER  our own kernels over peer memory: k_shard_push stores each export row straight into every subscriber's inbox
//                  (CUDA-IPC mapped memory of the neighbouring GPU, st.global over NVLink) and raises a per-rank arrival flag with a
//                  system-scope release; k_shard_pull waits for the flags of all ranks and scatters its inbox into the ghost rows.
//                  Neighbour-only traffic (a row travels to its subscribers, not to everybody), no host involvement, two small
//                  launches per exchange, capturable in a CUDA graph with the rest of the step.
//
// Inbox protocol: two parities, selected by the exchange epoch.  Every rank signals every other rank every epoch (a flag store is
// 4 bytes), so a rank can run at most one epoch ahead of any peer: push #e+2 (same parity as #e) is issued after pull #e+1, which
// waited for every peer's push #e+1, which that peer issued after ITS pull #e — the rows of epoch e have been consumed everywhere
// before they are overwritten.  (This is the back-pressure the round-1 prototype lacked.)
#pragma once
#include "nb_jacobi.cuh"
#include <string>
#include <dlfcn.h>
#include <nccl.h>

#define NB_SHARD_FLAG_WORDS 64   // header of the inbox allocation: arrival epoch per source rank (world <= 64)
enum { OVF_EXCHANGE = 16 };      // counts[CNT_OVERFLOW] bit: a pull gave up waiting for a peer

struct ShardPlanDev {
	const u32* export_local;   // [n_export] local body index of every row this rank exports
	const u32* sub_off;        // [n_export + 1] CSR over the subscribers of each export row
	const uint2* sub_tgt;      // (rank, inbox slot on that rank)
	const u32* ghost_local;    // [n_ghost] local body index of inbox slot j
	const u32* ghost_src;      // [n_ghost] row in the all-gather buffer (owner * max_export + row in the owner's export list)
	u32 n_export, n_ghost;
};

NB_DEV void st_release_sys(u32* p, u32 v) { asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory"); }
NB_DEV u32 ld_acquire_sys(const u32* p) { u32 v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
NB_DEV float4 ld_volatile_f4(const float4* p) { float4 v; asm volatile("ld.volatile.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory"); return v; }

// The inbox push protocol of k_shard_push and k_mw_out_push.  peers[r] = base of rank r's inbox allocation (flags first, then
// [2][ghost_cap][2] float4); the push of epoch ep fills parity ep & 1.  push_row stores export row i into the inbox slot of every
// subscriber.  push_arrive, after a block's last push_row, lets the last block to finish raise this rank's flag on every peer and
// advance *epoch, so the pull that follows reads it.
NB_DEV void push_row(const ShardPlanDev& P, unsigned char* const* peers, u32 ghost_cap, u32 ep, u32 i, float4 l, float4 w) {
	for (u32 t = P.sub_off[i]; t < P.sub_off[i + 1]; ++t) {
		const uint2 tg = P.sub_tgt[t];
		float4* dst = reinterpret_cast<float4*>(peers[tg.x] + NB_SHARD_FLAG_WORDS * 4) + 2 * ((size_t)(ep & 1u) * ghost_cap + tg.y);
		dst[0] = l; dst[1] = w;
	}
}
NB_DEV void push_arrive(unsigned char* const* peers, u32 rank, u32 world, u32 ep, u32* epoch, u32* done) {
	__threadfence_system();
	__syncthreads();
	if (threadIdx.x == 0) {
		const u32 old = atomicAdd(done, 1u);
		if (old == gridDim.x - 1) {      // every block's rows are out (each fenced before it arrived here)
			__threadfence_system();
			for (u32 r = 0; r < world; ++r)
				if (r != rank) st_release_sys(reinterpret_cast<u32*>(peers[r]) + rank, ep);
			*done = 0;
			*epoch = ep;
		}
	}
}

// rows -> subscribers' inboxes
__global__ void __launch_bounds__(NB_BLOCK) k_shard_push(const float4* mom, ShardPlanDev P, unsigned char* const* peers, u32 ghost_cap, u32 rank, u32 world,
														 u32* epoch, u32* done) {
	const u32 ep = *epoch + 1;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n_export; i += gridDim.x * blockDim.x) {
		const u32 body = P.export_local[i];
		push_row(P, peers, ghost_cap, ep, i, mom[2 * body], mom[2 * body + 1]);
	}
	push_arrive(peers, rank, world, ep, epoch, done);
}

// waits until every peer has pushed this epoch, then scatters the inbox into the ghost rows
__global__ void __launch_bounds__(NB_BLOCK) k_shard_pull(float4* mom, ShardPlanDev P, unsigned char* inbox, u32 ghost_cap, u32 rank, u32 world, const u32* epoch, u32* counts, long long timeout_cycles) {
	const u32 ep = *epoch;
	__shared__ int ok;
	if (threadIdx.x == 0) {
		const u32* flags = reinterpret_cast<const u32*>(inbox);
		const long long t0 = clock64();
		int good = 1;
		for (u32 r = 0; r < world && good; ++r) {
			if (r == rank) continue;
			while ((int)(ld_acquire_sys(flags + r) - ep) < 0) {
				if (clock64() - t0 > timeout_cycles) { good = 0; atomicOr(&counts[CNT_OVERFLOW], OVF_EXCHANGE); break; }
				__nanosleep(200);
			}
		}
		ok = good;
	}
	__syncthreads();
	if (!ok) return;
	const float4* rows = reinterpret_cast<const float4*>(inbox + NB_SHARD_FLAG_WORDS * 4) + 2 * (size_t)(ep & 1u) * ghost_cap;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < 2 * P.n_ghost; i += gridDim.x * blockDim.x)
		mom[2 * P.ghost_local[i >> 1] + (i & 1)] = ld_volatile_f4(rows + i);
}

// k_mw_out (nb_solver.cuh) + k_shard_push: the end of the dataflow hand-over below.  A pushed row is the BodyMomentum row k_mw_out
// writes: (velocity, unused0 kept, angular velocity, unused1 = 0 if a contact touched the body in a sweep); computed from mw and the
// OLD row, so it does not matter whether the block that copies the body back has run yet.
__global__ void __launch_bounds__(NB_BLOCK) k_mw_out_push(u32 B, nb_body_momentum* momentum, const float4* mw, int mode, ShardPlanDev P, unsigned char* const* peers,
														  u32 ghost_cap, u32 rank, u32 world, u32* epoch, u32* done) {
	const u32 ep = *epoch + 1;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
		float4* p = reinterpret_cast<float4*>(momentum + i);
		float4 l = mw[2*i], w = mw[2*i + 1];
		float4 ol = p[0], ow = p[1];
		bool touched = asu(l.w) != 0;
		p[0] = make_float4(l.x, l.y, l.z, ol.w);
		p[1] = make_float4(w.x, w.y, w.z, (mode && touched) ? 0.0f : ow.w);
	}
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < P.n_export; i += gridDim.x * blockDim.x) {
		const u32 body = P.export_local[i];
		const float4* p = reinterpret_cast<const float4*>(momentum + body);
		float4 l = mw[2*body], w = mw[2*body + 1];
		const bool touched = asu(l.w) != 0;
		const float u0 = p[0].w, u1 = p[1].w;      // unused0 never changes here; unused1 only ever changes to what the rule below gives
		l.w = u0; w.w = (mode && touched) ? 0.0f : u1;
		push_row(P, peers, ghost_cap, ep, i, l, w);
	}
	push_arrive(peers, rank, world, ep, epoch, done);
}

// ---- the ghost hand-over carried by the solver's own dataflow: ALL passes of a sharded step in one launch per GPU ----
// Per-sweep exchanges cut the solver into nine launches (warm start + 8 sweeps) and lose what makes k_solve fast on one GPU:
// sweeps pipelining into each other.  Here the exchange rides on the dataflow itself: the thread that applies the LAST contact of
// an exported body in pass w also stores the body's row, tagged (epoch, w), into a pass-indexed inbox in every subscriber's memory
// (peer memory over NVLink); on the subscriber the FIRST contact of that ghost in pass w+1 waits for the tag exactly as it waits
// for a body token, and starts from the owner's values.  Interior contacts never wait for the network; only chains that cross a
// cell boundary pay the NVLink latency, once per pass.  Same block-Jacobi coupling and - because every body still sees the
// reference's sequence of read-modify-writes, with the ghost refreshed at the same points - bit-identical to the per-sweep
// exchange (bench.py's parity_check covers it).
//   inbox2: [2 epoch parities][passes_cap][ghost_cap] rows of 2 x float4, w lanes = tag = epoch * 64 + pass + 1 (each 16-byte half
//   validates itself, like the body tokens).  A row is written once per (epoch, pass) and read after; the step ends with a regular
//   push/pull of the final rows (k_mw_out_push / k_shard_pull), which is also the all-to-all handshake that keeps every rank within
//   one epoch of its peers, so two parities suffice.
struct ShardFlow {
	float4* inbox2;                   // this GPU's pass-indexed inbox
	float4* const* peer_inbox2;       // [world]
	const u32* export_row;            // [B] row in the export list, NB_NONE for bodies nobody subscribes to
	const u32* ghost_slot;            // [B] inbox slot of a ghost body, NB_NONE otherwise
	u32 ghost_cap, passes_cap;
};
NB_DEV size_t flow_row(const ShardFlow& X, u32 ep, u32 pass, u32 slot) { return 2 * ((((size_t)(ep & 1u) * X.passes_cap) + pass) * X.ghost_cap + slot); }
NB_DEV u32 flow_tag(u32 ep, u32 pass) { return ep * 64u + pass + 1u; }
NB_DEV float4 ld128_sys(const float4* p) {
	float4 v;
	asm volatile("{\n .reg .b128 q;\n ld.relaxed.sys.global.b128 q, [%4];\n mov.b128 {%0,%1,%2,%3}, q;\n}" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
	return v;
}
NB_DEV void st128_sys(float4* p, float4 v) {
	asm volatile("{\n .reg .b128 q;\n mov.b128 q, {%1,%2,%3,%4};\n st.relaxed.sys.global.b128 [%0], q;\n}" :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
NB_DEV void flow_publish(const ShardFlow& X, const ShardPlanDev& P, u32 row, u32 ep, u32 pass, float4 l, float4 w) {
	const float tag = asf(flow_tag(ep, pass));
	l.w = tag; w.w = tag;
	for (u32 t = P.sub_off[row]; t < P.sub_off[row + 1]; ++t) {
		const uint2 tg = P.sub_tgt[t];
		float4* dst = X.peer_inbox2[tg.x] + flow_row(X, ep, pass, tg.y);
		st128_sys(dst, l); st128_sys(dst + 1, w);
	}
}

// working copy like k_mw_in; an exported body WITHOUT contacts on this rank never gets a "last contact": its (unchanging) row is
// published for every pass up front.  chain_len is zero for bodies without chain entries (memset before k_batch_index counts them).
__global__ void __launch_bounds__(NB_BLOCK) k_mw_in_flow(u32 B, const nb_body_momentum* momentum, float4* mw, const u32* chain_len, ShardFlow X, ShardPlanDev P, const u32* epoch, u32 passes) {
	const u32 ep = *epoch + 1;
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
		const float4* p = reinterpret_cast<const float4*>(momentum + i);
		float4 l = p[0], w = p[1];
		l.w = 0.0f; w.w = 0.0f;
		mw[2*i] = l; mw[2*i + 1] = w;
		const u32 row = X.export_row[i];
		if (i && row != NB_NONE && chain_len[i] == 0)
			for (u32 q = 0; q < passes; ++q) flow_publish(X, P, row, ep, q, l, w);
	}
}

// k_solve(mode 2) with the hand-over woven in: pass 0 = warm start, passes 1..sweeps = PGS sweeps.
__global__ void __launch_bounds__(NB_BLOCK, 2) k_solve_flow(Rows R, const float4* impulses, float4* mw, u32 sweeps, u32 hop_ns, u32* counts, ShardFlow X, ShardPlanDev P, const u32* epoch, long long timeout_cycles) {
	__shared__ u32 s_rcp[2048];
	__shared__ u32 s_rsqrt[2048];
	for (u32 i = threadIdx.x; i < 2048; i += blockDim.x) { s_rcp[i] = g_rcp_lut[i]; s_rsqrt[i] = g_rsqrt_lut[i]; }
	__syncthreads();
	const u32 NS = 8 * counts[CNT_BATCHES];
	const u32 tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
	const u32 passes = sweeps + 1;
	const u32 S = R.stride;
	const u32 ep = *epoch + 1;
	for (u32 w = 0; w < passes; ++w) {
		const bool sweep = w > 0;
		const u32 tag_in = flow_tag(ep, w - 1);   // only used when sweep
		for (u32 s0 = 0; s0 < NS; s0 += nth) {  // uniform trip count for the whole grid
			u32 slot = s0 + tid;
			bool pending = false, near = false, ga = false, gb = false;
			u32 a = 0, b = 0, exp_a = 0, exp_b = 0, pub_a = NB_NONE, pub_b = NB_NONE;
			const float4* in_a = nullptr; const float4* in_b = nullptr;
			long long t_wait = 0;
			float rv[ROW_PLANES_TOTAL], st[3];
			if (slot < NS && R.contact[slot] != NB_NONE) {
				pending = true;
				a = R.a[slot]; b = R.b[slot];
				uint2 wa = R.wait[slot], wb = R.wait[S + slot];
				exp_a = w * wa.y + wa.x; exp_b = w * wb.y + wb.x;
				if (a && wa.x + 1 == wa.y) pub_a = X.export_row[a];     // the last contact of an exported body publishes its row for this pass
				if (b && wb.x + 1 == wb.y) pub_b = X.export_row[b];
				if (sweep) {
					// the first contact of a ghost in this pass starts from what its owner published at the end of the previous pass
					const u32 sa = (a && wa.x == 0) ? X.ghost_slot[a] : NB_NONE, sb = (b && wb.x == 0) ? X.ghost_slot[b] : NB_NONE;
					ga = sa != NB_NONE; gb = sb != NB_NONE;
					if (ga) in_a = X.inbox2 + flow_row(X, ep, w - 1, sa);
					if (gb) in_b = X.inbox2 + flow_row(X, ep, w - 1, sb);
					const float* c = R.plane + slot;
					#pragma unroll
					for (int k = 0; k < ROW_PLANES_TOTAL; ++k) rv[k] = c[(size_t)k * S];
					st[0] = R.state[0*S + slot]; st[1] = R.state[1*S + slot]; st[2] = R.state[2*S + slot];
				}
			}
			while (__any_sync(0xffffffffu, pending)) {
				u32 want = 0xffffffffu;
				if (pending) {
					float4 al, bl, aw, bw;
					al = ld128(mw + 2*a); bl = ld128(mw + 2*b);
					if (near) { aw = ld128(mw + 2*a + 1); bw = ld128(mw + 2*b + 1); }
					u32 ra = a ? exp_a - asu(al.w) : 0, rb = b ? exp_b - asu(bl.w) : 0;
					u32 r = max(ra, rb);
					bool ready = r == 0 && near && (!a || asu(aw.w) == exp_a) && (!b || asu(bw.w) == exp_b);
					if (ready && (ga || gb)) {
						// a peer that never publishes must not hang this GPU: after the timeout the lane goes on with its local values and
						// flags the step (nb_counts.overflow & 16); once the flag is up nobody waits for an inbox any more
						if (!t_wait) t_wait = clock64();
						const bool give_up = (clock64() - t_wait > timeout_cycles) || (*(volatile u32*)&counts[CNT_OVERFLOW] & OVF_EXCHANGE);
						if (ga) {
							float4 il = ld128_sys(in_a), iw = ld128_sys(in_a + 1);
							if (asu(il.w) == tag_in && asu(iw.w) == tag_in) { al.x = il.x; al.y = il.y; al.z = il.z; aw.x = iw.x; aw.y = iw.y; aw.z = iw.z; }
							else if (give_up) atomicOr(&counts[CNT_OVERFLOW], OVF_EXCHANGE);
							else ready = false;
						}
						if (ready && gb) {
							float4 il = ld128_sys(in_b), iw = ld128_sys(in_b + 1);
							if (asu(il.w) == tag_in && asu(iw.w) == tag_in) { bl.x = il.x; bl.y = il.y; bl.z = il.z; bw.x = iw.x; bw.y = iw.y; bw.z = iw.z; }
							else if (give_up) atomicOr(&counts[CNT_OVERFLOW], OVF_EXCHANGE);
							else ready = false;
						}
					}
					if (ready) {
						if (sweep) solve_contact(R, slot, rv, st, al, aw, bl, bw, LutMath{ s_rcp, s_rsqrt });
						else warm_start_contact(R, slot, impulses, al, aw, bl, bw, LutMath{ s_rcp, s_rsqrt });
						if (a) { float tk = asf(exp_a + 1); al.w = tk; aw.w = tk; st128(mw + 2*a, al); st128(mw + 2*a + 1, aw); }
						if (b) { float tk = asf(exp_b + 1); bl.w = tk; bw.w = tk; st128(mw + 2*b, bl); st128(mw + 2*b + 1, bw); }
						if (pub_a != NB_NONE) flow_publish(X, P, pub_a, ep, w, al, aw);  // this body is done for pass w: hand it to its subscribers
						if (pub_b != NB_NONE) flow_publish(X, P, pub_b, ep, w, bl, bw);
						pending = false;
					}
					else {
						near = r <= 1;
						want = r >= 2 ? (r - 1) * hop_ns : 0;
					}
				}
				want = __reduce_min_sync(0xffffffffu, want);
				if (want != 0xffffffffu && want) __nanosleep(min(want, 20000u));
			}
		}
	}
}

// ---- NCCL bound at run time ----
struct NcclApi {
	void* lib;
	ncclResult_t (*GetUniqueId)(ncclUniqueId*);
	ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
	ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
	ncclResult_t (*CommDestroy)(ncclComm_t);
	const char* (*GetErrorString)(ncclResult_t);
};
static NcclApi* nccl_api(std::string* err) {
	static NcclApi api; static int state = 0;   // 0 untried, 1 ok, -1 failed
	if (state == 0) {
		const char* names[] = { "libnccl.so.2", "libnccl.so" };
		for (const char* n : names) { api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (api.lib) break; }
		if (api.lib) {
			api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(api.lib, "ncclGetUniqueId");
			api.CommInitRank = (decltype(api.CommInitRank))dlsym(api.lib, "ncclCommInitRank");
			api.AllGather = (decltype(api.AllGather))dlsym(api.lib, "ncclAllGather");
			api.CommDestroy = (decltype(api.CommDestroy))dlsym(api.lib, "ncclCommDestroy");
			api.GetErrorString = (decltype(api.GetErrorString))dlsym(api.lib, "ncclGetErrorString");
		}
		state = (api.lib && api.GetUniqueId && api.CommInitRank && api.AllGather && api.CommDestroy && api.GetErrorString) ? 1 : -1;
	}
	if (state != 1) { if (err) *err = "NCCL (libnccl.so.2) could not be loaded"; return nullptr; }
	return &api;
}
