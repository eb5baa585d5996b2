// nudge_b200 — host side of nb_shard_* (include/nudge_b200.h): NCCL communicator, peer-memory inboxes, exchange plan, the sharded
// sub-step and its CUDA graph.  Included at the end of nb_api.cu (needs nb_context's internals).  Kernels: nb_shard.cuh.
#pragma once

struct nb_shard {
	nb_context* ctx;
	u32 rank, world;
	ncclComm_t comm; bool has_nccl;
	// peer-memory transport
	unsigned char* inbox; u32 ghost_cap; std::vector<unsigned char*> peers; unsigned char** peers_dev; std::vector<void*> opened; bool peers_ready;
	u32* epoch; u32* done;
	// plan (device copies)
	u32* d_export_local; u32* d_sub_off; uint2* d_sub_tgt; u32* d_ghost_local; u32* d_ghost_src;
	// dataflow hand-over inside ONE solver launch (k_solve_flow): pass-indexed inbox behind the per-sweep one in the same IPC allocation
	u32 passes_cap; size_t inbox2_offset; float4** peer_inbox2_dev; u32* d_export_row; u32* d_ghost_slot; int flow_blocks;
	u32 cap_export, cap_ghost, cap_sub;
	ShardPlanDev plan; u32 max_export; unsigned long long plan_version;
	// NCCL transport buffers
	float4* d_export; float4* d_gather;
	StepGraph graph;   // the sharded step as a CUDA graph
	long long pull_timeout_cycles;
	int no_exchange;   // nb_shard_debug_no_exchange: time the rank's local problem without the ghost hand-over (results are then not a simulation of the global scene)
};

#define SCK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { sh->ctx->error = std::string(#call) + ": " + cudaGetErrorString(e_); return NB_ERR_CUDA; } } while (0)

extern "C" {

int nb_shard_unique_id(void* id_out) {
	std::string err;
	NcclApi* api = nccl_api(&err);
	if (!api || !id_out) return NB_ERR_ARGUMENT;
	ncclUniqueId id;
	if (api->GetUniqueId(&id) != ncclSuccess) return NB_ERR_CUDA;
	memcpy(id_out, &id, sizeof(id));
	return NB_OK;
}

// ghost_capacity / export_capacity: upper bounds for the plans this shard will see (every rank must pass the same ghost_capacity).
// nccl_id: the 128 bytes rank 0 obtained from nb_shard_unique_id, or null to run without NCCL (peer transport only).
int nb_shard_create(nb_context* ctx, uint32_t rank, uint32_t world, const void* nccl_id, uint32_t ghost_capacity, uint32_t export_capacity, nb_shard** out) {
	if (!ctx || !out || !world || rank >= world || world > NB_SHARD_FLAG_WORDS || !ghost_capacity || !export_capacity) { if (ctx) ctx->error = "bad shard configuration"; return NB_ERR_ARGUMENT; }
	nb_shard* sh = new nb_shard();
	*out = sh;
	sh->ctx = ctx; sh->rank = rank; sh->world = world; sh->ghost_cap = ghost_capacity;
	sh->cap_export = export_capacity; sh->cap_ghost = ghost_capacity; sh->cap_sub = 4 * export_capacity + 64;
	CK(cudaSetDevice(ctx->cfg.device));
	sh->passes_cap = 24;
	sh->inbox2_offset = NB_SHARD_FLAG_WORDS * 4 + sizeof(float4) * 2 * 2 * (size_t)ghost_capacity;
	size_t inbox_bytes = sh->inbox2_offset + sizeof(float4) * 2 * 2 * (size_t)sh->passes_cap * ghost_capacity;
	ALLOC(sh->inbox, inbox_bytes);
	ALLOC(sh->peer_inbox2_dev, world); ALLOC(sh->d_export_row, ctx->cfg.max_bodies); ALLOC(sh->d_ghost_slot, ctx->cfg.max_bodies);
	{
		int per_sm = 0;
		CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_solve_flow, NB_BLOCK, 0));
		sh->flow_blocks = per_sm > 0 ? ctx->sms * per_sm : 0;
	}
	ALLOC(sh->peers_dev, world); ALLOC(sh->epoch, 1); ALLOC(sh->done, 1);
	ALLOC(sh->d_export_local, sh->cap_export); ALLOC(sh->d_sub_off, (size_t)sh->cap_export + 1); ALLOC(sh->d_sub_tgt, sh->cap_sub);
	ALLOC(sh->d_ghost_local, sh->cap_ghost); ALLOC(sh->d_ghost_src, sh->cap_ghost);
	ALLOC(sh->d_export, 2 * (size_t)export_capacity); ALLOC(sh->d_gather, 2 * (size_t)export_capacity * world);
	sh->peers.assign(world, nullptr); sh->peers[rank] = sh->inbox;
	sh->graph.enabled = ctx->graph.enabled;
	int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, ctx->cfg.device);
	sh->pull_timeout_cycles = (long long)(khz ? khz : 1500000) * 1000LL * 5;   // 5 s: a peer that never pushes is reported, not waited for forever
	if (nccl_id) {
		std::string err;
		NcclApi* api = nccl_api(&err);
		if (!api) { ctx->error = err; return NB_ERR_CUDA; }
		ncclUniqueId id; memcpy(&id, nccl_id, sizeof(id));
		ncclResult_t r = api->CommInitRank(&sh->comm, (int)world, id, (int)rank);
		if (r != ncclSuccess) { ctx->error = std::string("ncclCommInitRank: ") + api->GetErrorString(r); delete sh; *out = nullptr; return NB_ERR_CUDA; }
		sh->has_nccl = true;
	}
	return NB_OK;
}

void nb_shard_destroy(nb_shard* sh) {
	if (!sh) return;
	cudaDeviceSynchronize();
	if (sh->graph.exec) cudaGraphExecDestroy(sh->graph.exec);
	for (void* p : sh->opened) cudaIpcCloseMemHandle(p);
	if (sh->has_nccl) { NcclApi* api = nccl_api(nullptr); if (api) api->CommDestroy(sh->comm); }
	delete sh;   // device buffers belong to the nb_context's allocation list
}

// CUDA IPC handle (64 bytes) of this rank's inbox; the ranks swap them out of band and call nb_shard_open_peer for every other rank.
int nb_shard_ipc_handle(nb_shard* sh, void* handle_out) {
	cudaIpcMemHandle_t h;
	SCK(cudaIpcGetMemHandle(&h, sh->inbox));
	memcpy(handle_out, &h, sizeof(h));
	return NB_OK;
}
int nb_shard_open_peer(nb_shard* sh, uint32_t peer, const void* handle) {
	if (peer >= sh->world) { sh->ctx->error = "bad peer"; return NB_ERR_ARGUMENT; }
	if (peer != sh->rank && !sh->peers[peer]) {
		cudaIpcMemHandle_t h; memcpy(&h, handle, sizeof(h));
		void* p = nullptr;
		SCK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
		sh->opened.push_back(p);
		sh->peers[peer] = (unsigned char*)p;
	}
	bool all = true;
	for (u32 r = 0; r < sh->world; ++r) all = all && sh->peers[r];
	if (all) {
		SCK(cudaMemcpy(sh->peers_dev, sh->peers.data(), sizeof(unsigned char*) * sh->world, cudaMemcpyHostToDevice));
		std::vector<float4*> p2(sh->world);
		for (u32 r = 0; r < sh->world; ++r) p2[r] = reinterpret_cast<float4*>(sh->peers[r] + sh->inbox2_offset);
		SCK(cudaMemcpy(sh->peer_inbox2_dev, p2.data(), sizeof(float4*) * sh->world, cudaMemcpyHostToDevice));
		sh->peers_ready = true;
	}
	return NB_OK;
}

// The exchange plan of the current partition (host arrays; synchronises the stream).  export_local[n_export]: local body index of
// the rows this rank exports, in the order of its export list; sub_off[n_export+1] / sub_rank / sub_slot: the subscribers of each
// export row (rank, index in that rank's ghost list); ghost_local[n_ghost]: local body index of ghost j; ghost_src[n_ghost]: its
// row in the all-gather buffer = owner * max_export + position in the owner's export list; max_export: the largest export list of
// any rank (the all-gather is padded to it).
int nb_shard_plan(nb_shard* sh, const uint32_t* export_local, uint32_t n_export, const uint32_t* sub_off, const uint32_t* sub_rank, const uint32_t* sub_slot,
				  const uint32_t* ghost_local, const uint32_t* ghost_src, uint32_t n_ghost, uint32_t max_export, void* stream) {
	nb_context* ctx = sh->ctx;
	const u32 n_sub = n_export ? sub_off[n_export] : 0;
	if (n_export > sh->cap_export || n_ghost > sh->cap_ghost || n_sub > sh->cap_sub || max_export > sh->cap_export || n_export > max_export) { ctx->error = "exchange plan exceeds the shard's capacities"; return NB_ERR_CAPACITY; }
	std::vector<uint2> tg(n_sub);
	for (u32 i = 0; i < n_sub; ++i) {
		if (sub_rank[i] >= sh->world || sub_rank[i] == sh->rank || sub_slot[i] >= sh->ghost_cap) { ctx->error = "exchange plan: subscriber out of range"; return NB_ERR_ARGUMENT; }
		tg[i] = make_uint2(sub_rank[i], sub_slot[i]);
	}
	for (u32 i = 0; i < n_export; ++i) if (export_local[i] >= ctx->B) { ctx->error = "exchange plan: export row out of range"; return NB_ERR_ARGUMENT; }
	for (u32 i = 0; i < n_ghost; ++i) if (ghost_local[i] >= ctx->B || ghost_src[i] >= sh->world * max_export) { ctx->error = "exchange plan: ghost out of range"; return NB_ERR_ARGUMENT; }
	SCK(cudaStreamSynchronize((cudaStream_t)stream));
	if (n_export) SCK(cudaMemcpy(sh->d_export_local, export_local, sizeof(u32) * n_export, cudaMemcpyHostToDevice));
	u32 zero = 0;
	SCK(cudaMemcpy(sh->d_sub_off, n_export ? sub_off : &zero, sizeof(u32) * ((size_t)n_export + 1), cudaMemcpyHostToDevice));
	if (n_sub) SCK(cudaMemcpy(sh->d_sub_tgt, tg.data(), sizeof(uint2) * n_sub, cudaMemcpyHostToDevice));
	if (n_ghost) { SCK(cudaMemcpy(sh->d_ghost_local, ghost_local, sizeof(u32) * n_ghost, cudaMemcpyHostToDevice)); SCK(cudaMemcpy(sh->d_ghost_src, ghost_src, sizeof(u32) * n_ghost, cudaMemcpyHostToDevice)); }
	{
		std::vector<u32> erow(ctx->cfg.max_bodies, NB_NONE), gslot(ctx->cfg.max_bodies, NB_NONE);
		for (u32 i = 0; i < n_ghost; ++i) gslot[ghost_local[i]] = i;
		for (u32 i = 0; i < n_export; ++i) if (sub_off[i + 1] > sub_off[i]) erow[export_local[i]] = i;
		SCK(cudaMemcpy(sh->d_export_row, erow.data(), sizeof(u32) * erow.size(), cudaMemcpyHostToDevice));
		SCK(cudaMemcpy(sh->d_ghost_slot, gslot.data(), sizeof(u32) * gslot.size(), cudaMemcpyHostToDevice));
	}
	sh->plan.export_local = sh->d_export_local; sh->plan.sub_off = sh->d_sub_off; sh->plan.sub_tgt = sh->d_sub_tgt;
	sh->plan.ghost_local = sh->d_ghost_local; sh->plan.ghost_src = sh->d_ghost_src; sh->plan.n_export = n_export; sh->plan.n_ghost = n_ghost;
	sh->max_export = max_export;
	++sh->plan_version;
	return NB_OK;
}

// Ghost rows <- owners' rows.  Every rank must call it the same number of times with the same transport.
int nb_shard_exchange(nb_shard* sh, int transport, void* stream) {
	NB_RANGE("nb_shard_exchange");
	nb_context* ctx = sh->ctx;
	cudaStream_t st = (cudaStream_t)stream;
	if (sh->world == 1) return NB_OK;
	if (!ctx->capturing) { int jr = join_uploads(ctx, st); if (jr) return jr; }   // reads the momentum rows
	const ShardPlanDev P = sh->plan;
	if (transport == NB_SHARD_NCCL) {
		if (!sh->has_nccl) { ctx->error = "this shard was created without an NCCL id"; return NB_ERR_ARGUMENT; }
		NcclApi* api = nccl_api(nullptr);
		if (P.n_export) { k_pack_rows<<<GRID(2 * P.n_export), NB_BLOCK, 0, st>>>((const float4*)ctx->mom, P.export_local, P.n_export, sh->d_export); ++ctx->launches; }
		ncclResult_t r = api->AllGather(sh->d_export, sh->d_gather, (size_t)sh->max_export * 8, ncclFloat, sh->comm, st);
		if (r != ncclSuccess) { ctx->error = std::string("ncclAllGather: ") + api->GetErrorString(r); return NB_ERR_CUDA; }
		if (P.n_ghost) { k_unpack_rows<<<GRID(2 * P.n_ghost), NB_BLOCK, 0, st>>>((float4*)ctx->mom, P.ghost_local, P.ghost_src, P.n_ghost, sh->d_gather); ++ctx->launches; }
	}
	else if (transport == NB_SHARD_PEER) {
		if (!sh->peers_ready) { ctx->error = "peer inboxes not opened (nb_shard_open_peer for every rank)"; return NB_ERR_ARGUMENT; }
		const unsigned grid = std::max(1u, std::min(GRID(std::max(P.n_export, 1u)), 64u));
		k_shard_push<<<grid, NB_BLOCK, 0, st>>>((const float4*)ctx->mom, P, sh->peers_dev, sh->ghost_cap, sh->rank, sh->world, sh->epoch, sh->done);
		k_shard_pull<<<std::max(1u, std::min(GRID(2 * std::max(P.n_ghost, 1u)), 64u)), NB_BLOCK, 0, st>>>((float4*)ctx->mom, P, sh->inbox, sh->ghost_cap, sh->rank, sh->world, sh->epoch, ctx->counts, sh->pull_timeout_cycles);
		ctx->launches += 2;
	}
	else { ctx->error = "unknown transport"; return NB_ERR_ARGUMENT; }
	SCK(cudaGetLastError());
	return NB_OK;
}

// peer transport + exact-order solver: warm start and all sweeps in ONE solver launch, ghosts handed over by the dataflow
// (k_solve_flow); the step ends with one regular push/pull of the final rows, which is also the handshake between the ranks
static int shard_solve_flow(nb_shard* sh, uint32_t iterations, cudaStream_t st) {
	nb_context* ctx = sh->ctx;
	const u32 B = ctx->B;
	const ShardPlanDev P = sh->plan;
	ShardFlow X;
	X.inbox2 = reinterpret_cast<float4*>(sh->inbox + sh->inbox2_offset); X.peer_inbox2 = sh->peer_inbox2_dev;
	X.export_row = sh->d_export_row; X.ghost_slot = sh->d_ghost_slot; X.ghost_cap = sh->ghost_cap; X.passes_cap = sh->passes_cap;
	const u32 passes = iterations + 1;
	k_mw_in_flow<<<GRID(B), NB_BLOCK, 0, st>>>(B, ctx->mom, ctx->mw, ctx->chain_len, X, P, sh->epoch, passes); ++ctx->launches;
	Rows R = ctx->rows; const float4* impulses = ctx->impulses; float4* mw = ctx->mw; u32* counts = ctx->counts; u32 hop = NB_SOLVE_BACKOFF_NS; u32 sweeps = iterations;
	const u32* epoch = sh->epoch; long long timeout = sh->pull_timeout_cycles;
	void* args[] = { &R, &impulses, &mw, &sweeps, &hop, &counts, &X, (void*)&P, &epoch, &timeout };
	timing_begin(ctx, st);
	SCK(cudaLaunchCooperativeKernel((void*)k_solve_flow, dim3(sh->flow_blocks), dim3(NB_BLOCK), args, 0, st));
	timing_end(ctx, st);
	++ctx->launches;
	k_mw_out_push<<<GRID(B), NB_BLOCK, 0, st>>>(B, ctx->mom, ctx->mw, 1, P, sh->peers_dev, sh->ghost_cap, sh->rank, sh->world, sh->epoch, sh->done);
	k_shard_pull<<<std::max(1u, std::min(GRID(2 * std::max(P.n_ghost, 1u)), 64u)), NB_BLOCK, 0, st>>>((float4*)ctx->mom, P, sh->inbox, sh->ghost_cap, sh->rank, sh->world, sh->epoch, ctx->counts, sh->pull_timeout_cycles);
	ctx->launches += 2;
	SCK(cudaGetLastError());
	return NB_OK;
}

static int shard_step_body(nb_shard* sh, float time_step, uint32_t iterations, float gravity, float damping, int transport, void* stream) {
	nb_context* ctx = sh->ctx;
	int r;
	if ((r = nb_collide(ctx, stream))) return r;
	if ((r = nb_apply_gravity_damping(ctx, time_step, gravity, damping, stream))) return r;
	if ((r = nb_read_cached_impulses(ctx, stream))) return r;
	// the dataflow hand-over needs the peer inboxes, the exact-order solver without user rows between the sweeps, a solver grid and
	// room for every pass in the pass-indexed inbox; everything else exchanges between the solver launches
	if (sh->world > 1 && transport == NB_SHARD_PEER && sh->peers_ready && ctx->solver_mode == NB_SOLVER_PARITY && !ctx->urow_n &&
		sh->flow_blocks > 0 && iterations > 0 && iterations + 1 <= sh->passes_cap) {
		ctx->defer_warm_start = true;                          // setup without its warm-start launch: it runs inside k_solve_flow
		r = nb_setup_contact_constraints(ctx, stream);         // (chain_len reads 0 for bodies without contacts on this rank)
		ctx->defer_warm_start = false;
		if (r) return r;
		if ((r = shard_solve_flow(sh, iterations, (cudaStream_t)stream))) return r;
	}
	else {
		if ((r = nb_setup_contact_constraints(ctx, stream))) return r;        // includes the warm start
		if ((r = nb_shard_exchange(sh, transport, stream))) return r;
		for (uint32_t i = 0; i < iterations; ++i) {
			if ((r = nb_apply_impulses(ctx, 1, stream))) return r;
			if ((r = nb_shard_exchange(sh, transport, stream))) return r;
		}
	}
	if ((r = nb_update_cached_impulses(ctx, stream))) return r;
	if ((r = nb_write_cached_impulses(ctx, stream))) return r;
	return nb_advance(ctx, time_step, stream);
}

// One sub-step of the sharded scene (example/main.cpp:274-328 with the ghost exchange after the warm start and after every sweep).
// On a capturable stream the whole step — kernels, NCCL all-gathers or peer pushes/pulls — is recorded once per plan into a CUDA
// graph and replayed (run_graphed).
int nb_shard_step(nb_shard* sh, float time_step, uint32_t iterations, float gravity, float damping, int transport, void* stream) {
	NB_RANGE("nb_shard_step");
	nb_context* ctx = sh->ctx;
	if (sh->no_exchange) return nb_step(ctx, time_step, iterations, gravity, damping, stream);   // diagnostic: this rank's local problem alone
	{ int jr = join_uploads(ctx, (cudaStream_t)stream); if (jr) return jr; }   // a pending side copy of nb_upload_bodies: ordered here, on the host side (the sharded graph has no event-wait node)
	ctx->capture_joined = true;
	return run_graphed(ctx, sh->graph, (cudaStream_t)stream, time_step, iterations, gravity, damping, transport, sh->plan_version,
					   [&] { return shard_step_body(sh, time_step, iterations, gravity, damping, transport, stream); });
}

int nb_shard_graph_active(const nb_shard* sh) { return sh->graph.exec != nullptr; }
int nb_shard_debug_no_exchange(nb_shard* sh, int on) { sh->no_exchange = on; return NB_OK; }

// Partition of a scene for `gx * gz` ranks (rank = ix * gz + iz): equal-count columns along x, each cut into equal-count cells
// along z.  A body is OWNED by the cell its centre lies in; it is a GHOST of every other cell whose box, grown by
// radius[i] + max_radius + margin, contains its centre (two bodies can only touch if their centres are closer than the sum of their
// bounding radii).  pos: n x 3 floats (x, y, z), radius: n bounding radii.  owner_out[n]; ghost lists as CSR over ranks
// (ghost_off[world + 1], ghost_ids up to ghost_cap entries, ascending per rank).  balance_iterations > 0 re-cuts the cells that many
// times so that owned + ghost bodies, not owned bodies, are even across ranks.  Returns NB_ERR_CAPACITY if ghost_cap is too small
// (ghost_off[world] then holds the required size).  Pure host code, deterministic: every rank computes the same partition.
int nb_shard_partition(const float* pos, const float* radius, uint32_t n, uint32_t gx, uint32_t gz, float margin, uint32_t balance_iterations,
					   uint32_t* owner_out, uint32_t* ghost_off, uint32_t* ghost_ids, uint32_t ghost_cap) {
	if (!gx || !gz || !pos || !radius || !owner_out || !ghost_off) return NB_ERR_ARGUMENT;
	const u32 world = gx * gz;
	// x order (ties by body index) and, once for all the re-cuts, the z order with ties by x rank: walking it and dealing every body
	// to its column yields each column sorted by z exactly as a stable sort of the column's x-ordered slice would
	std::vector<std::pair<float, u32>> keyed(n);
	for (u32 i = 0; i < n; ++i) keyed[i] = std::make_pair(pos[3 * i], i);
	std::sort(keyed.begin(), keyed.end());
	std::vector<u32> idx(n), xrank(n), zorder(n);
	for (u32 k = 0; k < n; ++k) { idx[k] = keyed[k].second; xrank[keyed[k].second] = k; }
	for (u32 i = 0; i < n; ++i) keyed[i] = std::make_pair(pos[3 * i + 2], xrank[i]);
	std::sort(keyed.begin(), keyed.end());
	for (u32 k = 0; k < n; ++k) zorder[k] = idx[keyed[k].second];
	std::vector<std::pair<float, u32>>().swap(keyed);
	std::vector<u32> col_begin(gx + 1), col_fill(gx), cols(n);
	std::vector<float> xlo(gx), xhi(gx), zlo(world), zhi(world);
	float rmax = 0.0f;
	for (u32 i = 0; i < n; ++i) rmax = std::max(rmax, radius[i]);
	const float inf = INFINITY;
	// share of the bodies every column / every cell of a column OWNS: equal to start with; the balance iterations shrink the cells
	// that carry many ghosts (interior cells have more neighbours) until owned + ghosts is even - a rank's step time follows its
	// LOCAL body count, and every step ends with a handshake that waits for the slowest rank
	std::vector<double> colw(gx, 1.0 / gx), cellw(world, 1.0 / gz);
	std::vector<size_t> owned(world), ghosts(world);
	bool uniform = true;   // equal shares: exact integer cuts (k * m / parts), the rule the tests restate
	auto cut = [](size_t m, double lo) { double v = lo * (double)m + 0.5; size_t k = v <= 0.0 ? 0 : (size_t)v; return k > m ? m : k; };
	auto assign = [&]() {
		double cx0 = 0.0;
		for (u32 cx = 0; cx < gx; ++cx) {   // column cuts in the x order
			const double cx1 = cx + 1 == gx ? 1.0 : cx0 + colw[cx];
			const size_t b0 = uniform ? (size_t)n * cx / gx : cut(n, cx0), b1 = cx + 1 == gx ? n : (uniform ? (size_t)n * (cx + 1) / gx : cut(n, cx1));
			cx0 = cx1;
			xlo[cx] = (cx == 0 || b0 == 0 || b0 >= n) ? (cx == 0 ? -inf : xlo[cx - 1]) : 0.5f * (pos[3 * idx[b0 - 1]] + pos[3 * idx[b0]]);
			if (cx) xhi[cx - 1] = xlo[cx];
			col_begin[cx] = (u32)b0; col_begin[cx + 1] = (u32)std::max(b0, b1);
		}
		for (u32 cx = 0; cx < gx; ++cx) col_fill[cx] = col_begin[cx];
		for (u32 k = 0; k < n; ++k) {       // deal the z order to the columns
			const u32 i = zorder[k], xr = xrank[i];
			u32 cx = 0;
			while (cx + 1 < gx && xr >= col_begin[cx + 1]) ++cx;
			cols[col_fill[cx]++] = i;
		}
		for (u32 cx = 0; cx < gx; ++cx) {
			const u32* col = cols.data() + col_begin[cx];
			const size_t m = col_begin[cx + 1] - col_begin[cx];
			double cz0 = 0.0;
			for (u32 cz = 0; cz < gz; ++cz) {
				const u32 r = cx * gz + cz;
				const double cz1 = cz + 1 == gz ? 1.0 : cz0 + cellw[r];
				const size_t c0 = uniform ? m * cz / gz : cut(m, cz0), c1 = cz + 1 == gz ? m : (uniform ? m * (cz + 1) / gz : cut(m, cz1));
				cz0 = cz1;
				zlo[r] = (cz == 0 || c0 == 0 || c0 >= m) ? (cz == 0 ? -inf : zlo[r - 1]) : 0.5f * (pos[3 * col[c0 - 1] + 2] + pos[3 * col[c0] + 2]);
				if (cz) zhi[r - 1] = zlo[r];
				if (cz == gz - 1) zhi[r] = inf;
				owned[r] = c1 > c0 ? c1 - c0 : 0;
				for (size_t k = c0; k < c1; ++k) owner_out[col[k]] = r;
			}
		}
		xhi[gx - 1] = inf;
	};
	auto is_ghost = [&](u32 r, u32 i) {
		if (owner_out[i] == r) return false;
		const u32 cx = r / gz;
		const float h = radius[i] + rmax + margin, x = pos[3 * i], z = pos[3 * i + 2];
		return x >= xlo[cx] - h && x < xhi[cx] + h && z >= zlo[r] - h && z < zhi[r] + h;
	};
	assign();
	for (u32 it = 0; it < balance_iterations && world > 1; ++it) {
		std::fill(ghosts.begin(), ghosts.end(), (size_t)0);
		for (u32 i = 0; i < n; ++i) for (u32 r = 0; r < world; ++r) ghosts[r] += is_ghost(r, i);
		std::vector<double> coltot(gx, 0.0);
		for (u32 r = 0; r < world; ++r) coltot[r / gz] += (double)(owned[r] + ghosts[r]);
		double mean_col = 0.0; for (u32 c = 0; c < gx; ++c) mean_col += coltot[c] / gx;
		double sw = 0.0;
		for (u32 c = 0; c < gx; ++c) { colw[c] *= coltot[c] > 0 ? mean_col / coltot[c] : 1.0; sw += colw[c]; }
		for (u32 c = 0; c < gx; ++c) colw[c] /= sw;
		for (u32 c = 0; c < gx; ++c) {
			double mean_cell = coltot[c] / gz, s2 = 0.0;
			for (u32 z = 0; z < gz; ++z) { const u32 r = c * gz + z; const double t = (double)(owned[r] + ghosts[r]); cellw[r] *= t > 0 ? mean_cell / t : 1.0; s2 += cellw[r]; }
			for (u32 z = 0; z < gz; ++z) cellw[c * gz + z] /= s2;
		}
		uniform = false;
		assign();
	}
	std::fill(ghosts.begin(), ghosts.end(), (size_t)0);
	for (u32 i = 0; i < n; ++i) for (u32 r = 0; r < world; ++r) ghosts[r] += is_ghost(r, i);
	size_t total = 0;
	for (u32 r = 0; r < world; ++r) { ghost_off[r] = (u32)total; total += ghosts[r]; }
	ghost_off[world] = (u32)total;
	if (!ghost_ids || total > ghost_cap) return NB_ERR_CAPACITY;
	std::vector<u32> fill(ghost_off, ghost_off + world);
	for (u32 i = 0; i < n; ++i) for (u32 r = 0; r < world; ++r) if (is_ghost(r, i)) ghost_ids[fill[r]++] = i;   // ascending per rank
	return NB_OK;
}

// The exchange plan of one rank from a partition (nb_shard_partition's owner[] and ghost lists): the arrays nb_shard_plan takes.
// Local body order of a rank: [world body, owned bodies ascending, ghosts ascending].  A body is EXPORTED by its owner if it is a
// ghost anywhere; a rank's export row k is its k-th exported body (ascending), rows are padded to `max_export` per rank for the
// all-gather (ghost_src = owner * max_export + row), and for the peer transport every export row lists its subscribers
// (rank, inbox slot = position in that rank's ghost list), ordered by (row, rank).  Pure host code, every rank computes its own plan
// from the same partition.  Two-pass protocol: with any output pointer null only sizes[] is filled
// (sizes = { n_owned, n_export, n_ghost, n_subscriptions, max_export }); capacities are then exactly those sizes.
int nb_shard_build_plan(const uint32_t* owner, uint32_t n, const uint32_t* ghost_off, const uint32_t* ghost_ids, uint32_t world, uint32_t rank,
						uint32_t sizes[5], uint32_t* owned_ids, uint32_t* export_local, uint32_t* sub_off, uint32_t* sub_rank, uint32_t* sub_slot,
						uint32_t* ghost_local, uint32_t* ghost_src) {
	if (!owner || !ghost_off || !sizes || rank >= world || !world) return NB_ERR_ARGUMENT;
	if (ghost_off[world] && !ghost_ids) return NB_ERR_ARGUMENT;
	std::vector<uint8_t> exported(n, 0);
	for (u32 k = 0; k < ghost_off[world]; ++k) { if (ghost_ids[k] >= n) return NB_ERR_ARGUMENT; exported[ghost_ids[k]] = 1; }
	// position of every exported body in its owner's export list, export counts per rank, local index of this rank's owned bodies
	std::vector<u32> n_exp(world, 0), pos_in_export(n, 0), lid(n, 0);
	u32 n_owned = 0;
	for (u32 i = 0; i < n; ++i) {
		if (owner[i] >= world) return NB_ERR_ARGUMENT;
		if (exported[i]) pos_in_export[i] = n_exp[owner[i]]++;
		if (owner[i] == rank) lid[i] = 1 + n_owned++;
	}
	u32 max_export = 1;
	for (u32 r = 0; r < world; ++r) max_export = std::max(max_export, n_exp[r]);
	const u32 n_export = n_exp[rank], n_ghost = ghost_off[rank + 1] - ghost_off[rank];
	u32 n_sub = 0;
	for (u32 p = 0; p < world; ++p) if (p != rank) for (u32 k = ghost_off[p]; k < ghost_off[p + 1]; ++k) n_sub += owner[ghost_ids[k]] == rank;
	sizes[0] = n_owned; sizes[1] = n_export; sizes[2] = n_ghost; sizes[3] = n_sub; sizes[4] = max_export;
	if (!owned_ids || !export_local || !sub_off || !sub_rank || !sub_slot || !ghost_local || !ghost_src) return NB_OK;
	for (u32 i = 0, k = 0, e = 0; i < n; ++i) if (owner[i] == rank) { owned_ids[k++] = i; if (exported[i]) export_local[e++] = lid[i]; }
	for (u32 j = 0; j < n_ghost; ++j) {
		const u32 g = ghost_ids[ghost_off[rank] + j];
		if (owner[g] == rank) return NB_ERR_ARGUMENT;   // a rank's own body among its ghosts
		ghost_local[j] = 1 + n_owned + j;
		ghost_src[j] = owner[g] * max_export + pos_in_export[g];
	}
	// subscribers by export row: counting sort on the row; ranks ascend inside a row because p ascends in both passes
	for (u32 k = 0; k <= n_export; ++k) sub_off[k] = 0;
	for (u32 p = 0; p < world; ++p) if (p != rank) for (u32 k = ghost_off[p]; k < ghost_off[p + 1]; ++k) { const u32 g = ghost_ids[k]; if (owner[g] == rank) ++sub_off[pos_in_export[g] + 1]; }
	for (u32 k = 0; k < n_export; ++k) sub_off[k + 1] += sub_off[k];
	std::vector<u32> cursor(sub_off, sub_off + n_export);
	for (u32 p = 0; p < world; ++p) if (p != rank) for (u32 k = ghost_off[p]; k < ghost_off[p + 1]; ++k) {
		const u32 g = ghost_ids[k];
		if (owner[g] == rank) { const u32 at = cursor[pos_in_export[g]]++; sub_rank[at] = p; sub_slot[at] = k - ghost_off[p]; }
	}
	return NB_OK;
}


// Which colliders a rank's local scene holds and where their bodies sit locally.  Local body order: [world body (global 0), owned bodies,
// ghosts]; owned_ids / ghost_ids are 0-based like nb_shard_partition's (global body = id + 1).  A collider is kept if its body is one of
// those, in the global collider order (so contact tags order contacts the way the global scene would).  box_body / sphere_body = the
// global body of every collider (nb_transform.body).  Two passes like nb_shard_build_plan: with any output null only
// sizes = { kept boxes, kept spheres } is filled.  box_sel / sphere_sel = kept collider indices (ascending), *_local_body = their local body.
int nb_shard_local_scene(const uint32_t* owned_ids, uint32_t n_owned, const uint32_t* ghost_ids, uint32_t n_ghost, uint32_t n_bodies_global,
						 const uint32_t* box_body, uint32_t n_boxes, const uint32_t* sphere_body, uint32_t n_spheres, uint32_t sizes[2],
						 uint32_t* box_sel, uint32_t* box_local_body, uint32_t* sphere_sel, uint32_t* sphere_local_body) {
	if (!sizes || (n_owned && !owned_ids) || (n_ghost && !ghost_ids) || (n_boxes && !box_body) || (n_spheres && !sphere_body) || !n_bodies_global) return NB_ERR_ARGUMENT;
	std::vector<u32> lid(n_bodies_global, NB_NONE);
	lid[0] = 0;
	for (u32 k = 0; k < n_owned; ++k) { if (owned_ids[k] + 1 >= n_bodies_global) return NB_ERR_ARGUMENT; lid[owned_ids[k] + 1] = 1 + k; }
	for (u32 k = 0; k < n_ghost; ++k) { if (ghost_ids[k] + 1 >= n_bodies_global || lid[ghost_ids[k] + 1] != NB_NONE) return NB_ERR_ARGUMENT; lid[ghost_ids[k] + 1] = 1 + n_owned + k; }
	u32 kb = 0, ks = 0;
	const bool fill = box_sel && box_local_body && sphere_sel && sphere_local_body;
	for (u32 i = 0; i < n_boxes; ++i) {
		if (box_body[i] >= n_bodies_global) return NB_ERR_ARGUMENT;
		const u32 l = lid[box_body[i]];
		if (l != NB_NONE) { if (fill) { box_sel[kb] = i; box_local_body[kb] = l; } ++kb; }
	}
	for (u32 i = 0; i < n_spheres; ++i) {
		if (sphere_body[i] >= n_bodies_global) return NB_ERR_ARGUMENT;
		const u32 l = lid[sphere_body[i]];
		if (l != NB_NONE) { if (fill) { sphere_sel[ks] = i; sphere_local_body[ks] = l; } ++ks; }
	}
	sizes[0] = kb; sizes[1] = ks;
	return NB_OK;
}

}  // extern "C"
