// nudge_b200 — throughput-mode solver: mass-splitting Jacobi over the same constraint rows as the exact-order solver.
//
// The reference's apply_impulses (nudge.cpp:4640-4855) is sequential Gauss-Seidel; replaying its order bit for bit (k_solve,
// nb_solver.cuh) is bounded by the dependency chain, not by memory.  This mode gives up the reference's ORDER (and therefore bit
// parity of the impulses — SURVEY.md §0.4, §7 "throughput mode") to become a pure stream over the rows:
//
//   per sweep   k_jacobi_sweep : every contact reads its two bodies' velocities as they were at the START of the sweep, runs the
//                                reference's per-contact arithmetic (solve_contact, same row planes, same clamps) and adds the
//                                velocity change it causes into a per-body accumulator;
//               k_jacobi_apply : velocity += accumulator, accumulator = 0.
//
// Plain Jacobi over-corrects a body that several contacts push at once; mass splitting (Tonge, Benevolenski, Voroshilov 2012) fixes
// that: body i is split into cnt[i] sub-bodies of mass m_i / cnt[i], one per contact, each contact solves against its own sub-body
// pair (effective-mass planes NVTNI / FC_* built with cnt-scaled inverse masses, k_build_rows<true>), and the sub-bodies are averaged
// back — which is exactly "add every contact's unscaled velocity change".  Unconditionally stable, order independent, one grid-wide
// dependency per sweep instead of ~70 per sweep.
//
// Data movement (north_star: "TMA bulk staging of contact batches ... warp shuffles for the per-batch impulse accumulation and
// Jacobi-style body-velocity updates"):
//   * slots are in TAG order (slot i = i-th contact of the contact-cache order), so a tile of 256 slots is 46 contiguous 1 KB
//     segments (41 row planes + 3 state planes + body indices a, b).  Warp 0 of the CTA issues them as 1-D bulk async copies
//     (cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes -> UBLKCP) into a shared-memory stage tracked by an mbarrier (the registers of the
//     CTA are the second stage of the ring); rows stream with an L2 evict-first policy so that the body arrays (velocities + accumulators, 64 B/body)
//     stay L2 resident while hundreds of MB of rows pass through.
//   * tag order sorts by (body B, body A, feature): lanes of a warp that share a body are neighbours, so the per-body velocity
//     changes are first summed across the warp with a segmented shuffle reduction and only the head lane of each run issues the
//     accumulate — one 128-bit vector reduction (red.global.add.v4.f32) per half row instead of three scalar atomics per lane.
//   * contacts against the static world (body 0, ~20 % of a pile) never touch memory for that side.
// Algorithmic bytes per sweep: 184 B per contact (160 row + 12 state read + 12 state written) + 64 B per active body.
#pragma once
#include "nb_solver.cuh"

#define NJ_TILE 256
#define NJ_PLANES (ROW_PLANES_TOTAL + 3 + 2)   // row planes, state planes, a, b
#define NJ_PLANE_A (ROW_PLANES_TOTAL + 3)
#define NJ_PLANE_B (ROW_PLANES_TOTAL + 4)

// STAGES shared-memory stages per CTA.  A thread moves its 46 values into registers as soon as a tile has landed, so the registers are
// one more stage of the ring and a shared stage can be refilled at once.  STAGES = 1: 47 KB per CTA, three CTAs (24 warps) per SM —
// meant for body arrays that are small next to L2;  STAGES = 2: 94 KB, two CTAs per SM but two tiles per CTA in flight — meant for
// scenes of a million bodies, whose gathers miss L2 (the choice is not yet re-measured on the H100).  nb_api.cu picks by body count.
template<int STAGES>
struct JacobiSmem {
	float tile[STAGES][NJ_PLANES][NJ_TILE];
	unsigned long long bar[STAGES];
};

NB_DEV u32 smem_addr(const void* p) { return (u32)__cvta_generic_to_shared(p); }
NB_DEV void mbar_init(unsigned long long* bar, u32 count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_addr(bar)), "r"(count) : "memory"); }
NB_DEV void mbar_expect_tx(unsigned long long* bar, u32 bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_addr(bar)), "r"(bytes) : "memory"); }
NB_DEV bool mbar_try_wait(unsigned long long* bar, u32 parity) {
	u32 ok;
	asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}" : "=r"(ok) : "r"(smem_addr(bar)), "r"(parity) : "memory");
	return ok != 0;
}
// 1-D bulk copy global -> shared through the TMA unit; completion is counted in bytes on the mbarrier
NB_DEV void bulk_g2s(void* dst, const void* src, u32 bytes, unsigned long long* bar, unsigned long long policy) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
		:: "r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)), "l"(policy) : "memory");
}
NB_DEV void red_add_v4(float4* p, float x, float y, float z) {
	asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" :: "l"(p), "f"(x), "f"(y), "f"(z), "f"(0.0f) : "memory");
}

// tag order: slot i = contact sorted[i]; per-body contact counts for the mass split (body 0 and kinematic bodies are never split)
__global__ void __launch_bounds__(NB_BLOCK) k_jacobi_prepare(const u32* sorted, const uint2* bodies, const uint8_t* kind, u32* cnt, Rows R, u32 max_slots, u32* counts) {
	u32 n = counts[CNT_CONTACTS];
	if (n > max_slots) n = max_slots;
	if (blockIdx.x == 0 && threadIdx.x == 0) { counts[CNT_BATCHES] = (n + 7) / 8; counts[CNT_FULL_BATCHES] = n / 8; counts[CNT_ENTRIES] = 0; }
	for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		u32 c = sorted[i];
		uint2 ab = solver_pair(kind, bodies[c]);
		R.contact[i] = c;
		if (ab.x) atomicAdd(&cnt[ab.x], 1u);
		if (ab.y) atomicAdd(&cnt[ab.y], 1u);
	}
}

// sums v[0..5] over RUNS of equal `key` among neighbouring lanes (a run = maximal stretch of adjacent lanes with the same key; the same
// key may come back later in the warp as a separate run); the first lane of each run ends up with the run's total.  `heads` has a bit
// for every lane that starts a run: lane i may take lane i+d's partial sum iff no run starts in (i, i+d].  The number of doubling
// steps follows the longest run of THIS warp (warp-uniform): runs are short (a body has a handful of contacts), so two or three
// steps instead of five, and none at all when every lane is its own run.
NB_DEV void seg_reduce6(u32 heads, float (&v)[6]) {
	const u32 lane = threadIdx.x & 31;
	const u32 later = lane < 31 ? heads >> (lane + 1) : 0u;   // bit k: a run starts at lane + 1 + k
	// length of the run this lane starts or sits in, measured to its end: distance to the next head (or to lane 32)
	const u32 to_end = later ? (u32)__ffs((int)later) : 32u - lane;
	const u32 longest = __reduce_max_sync(0xffffffffu, (heads >> lane) & 1u ? to_end : 0u);
	for (u32 d = 1; d < longest; d <<= 1) {
		const bool take = lane + d < 32 && (later & ((1u << d) - 1u)) == 0;
		#pragma unroll
		for (int i = 0; i < 6; ++i) { float t = __shfl_down_sync(0xffffffffu, v[i], d); if (take) v[i] += t; }
	}
}

// One Jacobi pass over all contacts.  WARM: the warm start (nudge.cpp:4563-4632) instead of a PGS sweep.
// V[2*body], V[2*body+1] = (velocity, -), (angular velocity, -) at the start of the pass (read only); D = accumulators.
template<bool WARM, int STAGES>
__global__ void __launch_bounds__(NJ_TILE, 4 - STAGES) k_jacobi_sweep(Rows R, const float4* impulses, const float4* __restrict__ V, float4* D, const u32* counts) {
	extern __shared__ __align__(128) unsigned char nj_smem_raw[];
	JacobiSmem<STAGES>& sm = *reinterpret_cast<JacobiSmem<STAGES>*>(nj_smem_raw);
	const u32 n = min(counts[CNT_CONTACTS], 8u * counts[CNT_BATCHES]);
	const u32 tiles = (n + NJ_TILE - 1) / NJ_TILE;
	const u32 S = R.stride;
	unsigned long long policy;
	asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
	if (threadIdx.x == 0) {
		for (int k = 0; k < STAGES; ++k) mbar_init(&sm.bar[k], 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();

	// warp 0 is the producer: one expect_tx for the whole tile, then 46 bulk copies of 1 KB spread over its lanes
	auto issue = [&](u32 tile, u32 stage) {
		if (threadIdx.x < 32) {
			if (threadIdx.x == 0) mbar_expect_tx(&sm.bar[stage], NJ_PLANES * NJ_TILE * 4);
			__syncwarp();
			const size_t t0 = (size_t)tile * NJ_TILE;
			for (u32 k = threadIdx.x; k < NJ_PLANES; k += 32) {
				const void* src;
				if (k < ROW_PLANES_TOTAL) src = R.plane + (size_t)k * S + t0;
				else if (k < ROW_PLANES_TOTAL + 3) src = R.state + (size_t)(k - ROW_PLANES_TOTAL) * S + t0;
				else src = (k == NJ_PLANE_A ? R.a : R.b) + t0;
				bulk_g2s(&sm.tile[stage][k][0], src, NJ_TILE * 4, &sm.bar[stage], policy);
			}
		}
	};

	// Ring of two: shared memory holds the tile in flight, registers hold the tile being solved.  Per tile: wait for the bulk copies,
	// read the body indices and start the velocity gathers (L2), copy the 44 row/state values into registers, ONE CTA barrier, refill
	// the shared stage with the next tile at once, then solve, store the impulse state and accumulate - all of which overlaps the
	// next tile's copies.
	u32 it = 0;
	u32 tile = blockIdx.x;
	#pragma unroll
	for (int k = 0; k < STAGES; ++k) if (tile + k * gridDim.x < tiles) issue(tile + k * gridDim.x, k);
	for (; tile < tiles; tile += gridDim.x, ++it) {
		const u32 stage = STAGES == 1 ? 0u : (it & 1u);
		while (!mbar_try_wait(&sm.bar[stage], (STAGES == 1 ? it : (it >> 1)) & 1u)) { }
		const u32 slot = tile * NJ_TILE + threadIdx.x;
		const bool valid = slot < n;
		const float* T = &sm.tile[stage][0][threadIdx.x];
		const u32 ra = valid ? asu(T[NJ_PLANE_A * NJ_TILE]) : 0u, rb = valid ? asu(T[NJ_PLANE_B * NJ_TILE]) : 0u;   // NB_READ_ONLY on a kinematic side
		const u32 a = NB_BODY_INDEX(ra), b = NB_BODY_INDEX(rb);
		float4 al = V[2*a], aw = V[2*a + 1], bl = V[2*b], bw = V[2*b + 1];      // body 0 for invalid lanes: zeros, harmless
		float4 ci = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
		if (WARM && valid) ci = impulses[R.contact[slot]];
		float rv[ROW_PLANES_TOTAL], st[3];
		#pragma unroll
		for (int k = 0; k < ROW_PLANES_TOTAL; ++k) rv[k] = T[k * NJ_TILE];
		#pragma unroll
		for (int k = 0; k < 3; ++k) st[k] = T[(ROW_PLANES_TOTAL + k) * NJ_TILE];
		__syncthreads();                                               // the stage is drained
		if (tile + STAGES * gridDim.x < tiles) issue(tile + STAGES * gridDim.x, stage);
		float da[6] = { 0, 0, 0, 0, 0, 0 }, db[6] = { 0, 0, 0, 0, 0, 0 };
		if (valid) {
			const float4 al0 = al, aw0 = aw, bl0 = bl, bw0 = bw;
			if (WARM) warm_start_contact_p(rv, 1, ci, R.state + slot, S, al, aw, bl, bw, FastMath());
			else solve_contact(R, slot, rv, st, al, aw, bl, bw, FastMath());
			da[0] = al.x - al0.x; da[1] = al.y - al0.y; da[2] = al.z - al0.z; da[3] = aw.x - aw0.x; da[4] = aw.y - aw0.y; da[5] = aw.z - aw0.z;
			db[0] = bl.x - bl0.x; db[1] = bl.y - bl0.y; db[2] = bl.z - bl0.z; db[3] = bw.x - bw0.x; db[4] = bw.y - bw0.y; db[5] = bw.z - bw0.z;
		}
		// per-body accumulation across the warp, then one vector reduction per half row from the head lane of each run
		const u32 lane = threadIdx.x & 31;
		const u32 pa = __shfl_up_sync(0xffffffffu, a, 1), pb = __shfl_up_sync(0xffffffffu, b, 1);
		const bool head_a = lane == 0 || pa != a, head_b = lane == 0 || pb != b;
		seg_reduce6(__ballot_sync(0xffffffffu, head_a), da);
		seg_reduce6(__ballot_sync(0xffffffffu, head_b), db);
		if ((int)ra > 0 && head_a) { red_add_v4(D + 2*a, da[0], da[1], da[2]); red_add_v4(D + 2*a + 1, da[3], da[4], da[5]); }   // neither body 0 nor kinematic
		if ((int)rb > 0 && head_b) { red_add_v4(D + 2*b, db[0], db[1], db[2]); red_add_v4(D + 2*b + 1, db[3], db[4], db[5]); }
	}
}

// velocity += accumulated change; accumulator = 0.  The w lane of the linear half marks a body some contact has touched
// (k_mw_out zeroes BodyMomentum::unused1 of those, nudge.cpp:4823, 4849).
__global__ void __launch_bounds__(NB_BLOCK) k_jacobi_apply(u32 B, float4* V, float4* D, const u32* cnt) {
	for (u32 i = 1 + blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
		if (!cnt[i]) continue;
		float4 dl = D[2*i], dw = D[2*i + 1];
		float4 l = V[2*i], w = V[2*i + 1];
		l.x += dl.x; l.y += dl.y; l.z += dl.z; l.w = asf(1u);
		w.x += dw.x; w.y += dw.y; w.z += dw.z;
		V[2*i] = l; V[2*i + 1] = w;
		D[2*i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f); D[2*i + 1] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
	}
}
