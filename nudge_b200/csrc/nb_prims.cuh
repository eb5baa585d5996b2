// nudge_b200 — device-wide primitives: multi-counter exclusive scan, stable LSD radix sort, grid barrier.
//
// All element counts are read from device memory (the step never synchronises with the host), so every
// kernel runs on a fixed grid sized for the SM count and walks its share with a stride or a contiguous tile.
// These replace the reference's sequential radix sorts (nudge.cpp:2647-2836) and its many serial
// "count, then append" loops.
#pragma once
#include "nb_common.cuh"

#define NB_BLOCK 256
#define NB_WARPS (NB_BLOCK/32)

struct Launch { cudaStream_t stream; unsigned long long* counter; int sms; };

static inline unsigned nb_grid_for(unsigned n_cap, int sms, int per_sm = 8) {
	unsigned g = (n_cap + NB_BLOCK - 1) / NB_BLOCK;
	unsigned cap = (unsigned)(sms * per_sm);
	if (g > cap) g = cap;
	return g ? g : 1;
}

// ---------------- block-level exclusive scan (256 threads) ----------------
NB_DEV u32 warp_incl_scan(u32 v) {
	u32 lane = threadIdx.x & 31;
	#pragma unroll
	for (int d = 1; d < 32; d <<= 1) {
		u32 t = __shfl_up_sync(0xffffffffu, v, d);
		if (lane >= (u32)d) v += t;
	}
	return v;
}

// returns exclusive prefix of v within the block; *total = block sum.  smem: NB_WARPS+1 words.  Ends with a barrier.
NB_DEV u32 block_excl_scan(u32 v, u32* total, u32* smem) {
	u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	u32 incl = warp_incl_scan(v);
	if (lane == 31) smem[wid] = incl;
	__syncthreads();
	if (wid == 0) {
		u32 w = lane < NB_WARPS ? smem[lane] : 0;
		u32 wi = warp_incl_scan(w);
		if (lane < NB_WARPS) smem[lane] = wi - w;
		if (lane == NB_WARPS - 1) smem[NB_WARPS] = wi;
	}
	__syncthreads();
	u32 r = incl - v + smem[wid];
	*total = smem[NB_WARPS];
	__syncthreads();
	return r;
}

// ---------------- device-wide exclusive scan over N interleaved counters ----------------
// in/out: N arrays laid out as arr[c*stride + i]; count read from *n_ptr (or n_host if n_ptr is null).
// totals[c] receives the sum of counter c.  Two kernels: k_scan_reduce writes the tile sums and its last block to finish turns
// them into tile offsets (the spine); the downsweep then either writes `out` (k_scan_down) or happens inside the consumer that
// reads the offsets (scan_consume), when that consumer handles element i itself: one launch and one pass over `out` less.
#define NB_SCAN_GRID 592
#define NB_SCAN_ITEMS 4
#define NB_SCAN_DONE (16 * NB_SCAN_GRID)   // block_sums[NB_SCAN_DONE]: blocks of k_scan_reduce done (0 between launches)
#define NB_SCAN_SUMS (NB_SCAN_DONE + 1)    // words of block_sums: up to 16 counters

NB_DEV void scan_tile_range(u32 n, u32& begin, u32& end) {
	u32 chunk = NB_BLOCK * NB_SCAN_ITEMS;
	u32 tiles = (n + chunk - 1) / chunk;
	u32 per = (tiles + gridDim.x - 1) / gridDim.x;
	begin = min(n, blockIdx.x * per * chunk);
	end = min(n, begin + per * chunk);
}

template<int N>
__global__ void __launch_bounds__(NB_BLOCK) k_scan_reduce(const u32* in, u32 stride, const u32* n_ptr, u32 n_host, u32* block_sums, u32* totals) {
	__shared__ u32 sm[NB_WARPS + 1];
	__shared__ bool last;
	u32 n = n_ptr ? *n_ptr : n_host;
	u32 begin, end; scan_tile_range(n, begin, end);
	u32 acc[N];
	#pragma unroll
	for (int c = 0; c < N; ++c) acc[c] = 0;
	for (u32 i = begin + threadIdx.x; i < end; i += NB_BLOCK)
		#pragma unroll
		for (int c = 0; c < N; ++c) acc[c] += in[c*stride + i];
	#pragma unroll
	for (int c = 0; c < N; ++c) {
		u32 total; block_excl_scan(acc[c], &total, sm);
		if (threadIdx.x == 0) block_sums[c*NB_SCAN_GRID + blockIdx.x] = total;
	}
	// spine: the last block to finish turns the tile sums into exclusive tile offsets and writes the totals
	if (threadIdx.x == 0) { __threadfence(); last = atomicAdd(&block_sums[NB_SCAN_DONE], 1u) == gridDim.x - 1; }
	__syncthreads();
	if (!last) return;
	__threadfence();
	constexpr u32 PER = (NB_SCAN_GRID + NB_BLOCK - 1) / NB_BLOCK;
	const u32 t0 = threadIdx.x * PER;
	#pragma unroll
	for (int c = 0; c < N; ++c) {
		u32 v[PER], s = 0;
		#pragma unroll
		for (u32 k = 0; k < PER; ++k) { v[k] = t0 + k < NB_SCAN_GRID ? __ldcg(&block_sums[c*NB_SCAN_GRID + t0 + k]) : 0; s += v[k]; }
		u32 total; u32 ex = block_excl_scan(s, &total, sm);
		#pragma unroll
		for (u32 k = 0; k < PER; ++k) if (t0 + k < NB_SCAN_GRID) { block_sums[c*NB_SCAN_GRID + t0 + k] = ex; ex += v[k]; }
		if (threadIdx.x == 0 && totals) totals[c] = total;
	}
	if (threadIdx.x == 0) block_sums[NB_SCAN_DONE] = 0;
}

template<int N>
__global__ void __launch_bounds__(NB_BLOCK) k_scan_down(const u32* in, u32* out, u32 stride, const u32* n_ptr, u32 n_host, const u32* block_sums) {
	__shared__ u32 sm[NB_WARPS + 1];
	u32 n = n_ptr ? *n_ptr : n_host;
	u32 begin, end; scan_tile_range(n, begin, end);
	u32 run[N];
	#pragma unroll
	for (int c = 0; c < N; ++c) run[c] = block_sums[c*NB_SCAN_GRID + blockIdx.x];
	for (u32 base = begin; base < end; base += NB_BLOCK * NB_SCAN_ITEMS) {
		u32 i0 = base + threadIdx.x * NB_SCAN_ITEMS;
		#pragma unroll
		for (int c = 0; c < N; ++c) {
			u32 v[NB_SCAN_ITEMS]; u32 s = 0;
			#pragma unroll
			for (int k = 0; k < NB_SCAN_ITEMS; ++k) { v[k] = (i0 + k < end) ? in[c*stride + i0 + k] : 0; s += v[k]; }
			u32 total; u32 ex = block_excl_scan(s, &total, sm) + run[c];
			#pragma unroll
			for (int k = 0; k < NB_SCAN_ITEMS; ++k) { if (i0 + k < end) out[c*stride + i0 + k] = ex; ex += v[k]; }
			run[c] += total;
		}
	}
}

// block_excl_scan on 64-bit values
NB_DEV u64 block_excl_scan64(u64 v, u64* total, u64* smem) {
	u32 lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	u64 incl = v;
	#pragma unroll
	for (int d = 1; d < 32; d <<= 1) { u64 t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= (u32)d) incl += t; }
	if (lane == 31) smem[wid] = incl;
	__syncthreads();
	if (wid == 0) {
		u64 w = lane < NB_WARPS ? smem[lane] : 0, wi = w;
		#pragma unroll
		for (int d = 1; d < NB_WARPS; d <<= 1) { u64 t = __shfl_up_sync(0xffffffffu, wi, d); if (lane >= (u32)d) wi += t; }
		if (lane < NB_WARPS) smem[lane] = wi - w;
		if (lane == NB_WARPS - 1) smem[NB_WARPS] = wi;
	}
	__syncthreads();
	u64 r = incl - v + smem[wid];
	*total = smem[NB_WARPS];
	__syncthreads();
	return r;
}

// The downsweep inside a consumer kernel launched with NB_SCAN_GRID blocks after nb_scan_reduce: the block walks the tiles
// k_scan_reduce summed for it, 256 elements per round, and calls f(i, v, off) for every element i < n of them, with
// v[c] = in[c*stride + i] and off[c] = its exclusive prefix (what k_scan_down would have written to out[c*stride + i]).
// The N counters of a round are scanned together, packed into 64 / N bits each, so the values must be flags (0 or 1): a
// round's sum per counter is then at most 256.  Every thread of the block must call it.
template<int N, class F>
NB_DEV void scan_consume(const u32* in, u32 stride, u32 n, const u32* block_sums, F&& f) {
	static_assert(N >= 1 && (N == 1 || 64 / N > 9), "a round's sum of 0/1 flags needs 9 bits per counter");
	constexpr u32 W = 64 / N;
	constexpr u64 M = W == 64 ? ~(u64)0 : (((u64)1 << (W % 64)) - 1);
	__shared__ u64 sm[NB_WARPS + 1];
	u32 begin, end; scan_tile_range(n, begin, end);
	u32 run[N];
	#pragma unroll
	for (int c = 0; c < N; ++c) run[c] = block_sums[c*NB_SCAN_GRID + blockIdx.x];
	for (u32 base = begin; base < end; base += NB_BLOCK) {
		const u32 i = base + threadIdx.x;
		u32 v[N], off[N];
		u64 packed = 0;
		#pragma unroll
		for (int c = 0; c < N; ++c) { v[c] = i < end ? in[c*stride + i] : 0; packed |= (u64)v[c] << (c * W); }
		u64 total; const u64 ex = block_excl_scan64(packed, &total, sm);
		#pragma unroll
		for (int c = 0; c < N; ++c) { off[c] = run[c] + (u32)((ex >> (c * W)) & M); run[c] += (u32)((total >> (c * W)) & M); }
		if (i < end) f(i, v, off);
	}
}

// tile sums + spine only: the consumer, launched with NB_SCAN_GRID blocks, does the downsweep through scan_consume
template<int N>
static void nb_scan_reduce(const Launch& L, const u32* in, u32 stride, const u32* n_ptr, u32 n_host, u32* block_sums /*NB_SCAN_SUMS*/, u32* totals) {
	k_scan_reduce<N><<<NB_SCAN_GRID, NB_BLOCK, 0, L.stream>>>(in, stride, n_ptr, n_host, block_sums, totals);
	*L.counter += 1;
}
template<int N>
static void nb_scan(const Launch& L, const u32* in, u32* out, u32 stride, const u32* n_ptr, u32 n_host, u32* block_sums /*NB_SCAN_SUMS*/, u32* totals) {
	nb_scan_reduce<N>(L, in, stride, n_ptr, n_host, block_sums, totals);
	k_scan_down<N><<<NB_SCAN_GRID, NB_BLOCK, 0, L.stream>>>(in, out, stride, n_ptr, n_host, block_sums);
	*L.counter += 1;
}

// ---------------- grid-wide barrier for cooperative (co-resident) launches ----------------
NB_DEV u32 ld_acquire_u32(const u32* p) {
	u32 v;
	asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}

NB_DEV void grid_barrier(u32* bar /* [0]=arrivals, [1]=generation */, u32 nblocks) {
	__syncthreads();
	if (threadIdx.x == 0) {
		u32 gen = ld_acquire_u32(bar + 1);
		__threadfence();
		if (atomicAdd(bar, 1u) == nblocks - 1) {
			bar[0] = 0;
			__threadfence();
			atomicAdd(bar + 1, 1u);
		}
		else {
			while (ld_acquire_u32(bar + 1) == gen) { }
		}
		__threadfence();
	}
	__syncthreads();
}

// ---------------- single-launch radix sort (cooperative) ----------------
// One cooperative launch per sort: one block of 1024 threads per SM.  The digits are 8 bits wide, top-aligned (the host picks
// the shifts so that the last digit covers the highest populated bits).
//   n <= NB_CS_CAP      block 0 sorts everything in registers / shared memory (all digits, LSD), no grid barrier.
//   otherwise           MSD first: histogram of the TOP digit -> [block][digit] matrix | barrier | every block derives its
//                       scatter offsets from the matrix and scatters its keys into 256 buckets | barrier | each bucket
//                       is sorted on the remaining digits by one block and written back in place: in registers / shared
//                       memory when it has <= NB_CS_CAP keys, tile by tile through global memory when it is larger (a hot
//                       key).  Two grid barriers per SORT instead of two per digit.
//   a bucket > 8 caps   (very skewed keys, or large n): plain LSD over all digits, two grid barriers per digit.
// The result always lands in k1/v1.  Stable.  n == 0 costs one empty launch.
#define NB_CS_THREADS 1024
#define NB_CS_WARPS 32
#define NB_CS_ITEMS 4                       // keys per thread while scattering through global memory
#define NB_CS_TILE (NB_CS_THREADS * NB_CS_ITEMS)
#define NB_CS_LOCAL 8                       // keys per thread in the block-local sort
#define NB_CS_CAP (NB_CS_THREADS * NB_CS_LOCAL)
struct SortPasses { int n; int shift[12]; };
struct CoopSortSmem {
	u32 wc[NB_CS_WARPS][256];
	u32 h[256], tot[256], running[256], below[4][256], total[4][256], sm[8];
	u64 skeys[NB_CS_CAP];
	u32 svals[NB_CS_CAP];
};

// A digit is either 8 contiguous bits (np == 0) or up to 8 single bits gathered from the positions packed in `pos` (most
// significant first): the top digit of a sort whose producer recorded which key bits vary at all (OR and AND of the keys) is
// made of the 8 highest VARYING bits, which spreads e.g. Morton codes of a flat scene over all 256 buckets.
struct CsDigit { u32 shift; u32 np; u64 pos; };
NB_DEV u32 cs_digit(const CsDigit& D, u64 key) {
	if (!D.np) return (u32)(key >> D.shift) & 0xff;
	u32 d = 0; u64 pp = D.pos;
	for (u32 i = 0; i < D.np; ++i) { d = (d << 1) | ((u32)(key >> (pp & 63)) & 1u); pp >>= 8; }
	return d;
}
NB_DEV CsDigit cs_plain(int shift) { CsDigit D; D.shift = (u32)shift; D.np = 0; D.pos = 0; return D; }

// Ranks ITEMS keys per thread (item r of a thread sits at tile position wid*32*ITEMS + r*32 + lane, so position order = rank
// order).  Out: dg/rk per item, S.wc[w][d] = keys of digit d in warps before w, S.tot[d] = tile total.  Ends with a barrier.
template<int ITEMS>
NB_DEV void cs_rank(CoopSortSmem& S, const u64 (&key)[ITEMS], u32 nvalid, const CsDigit& D, u32 (&dg)[ITEMS], u32 (&rk)[ITEMS]) {
	const u32 tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, lt = (1u << lane) - 1u;
	const u32 nw = min((u32)NB_CS_WARPS, (nvalid + 32 * ITEMS - 1) / (32 * ITEMS));  // warps that hold keys
	for (u32 w = tid; w < nw * 256; w += NB_CS_THREADS) (&S.wc[0][0])[w] = 0;
	__syncthreads();
	if (wid < nw) {
		#pragma unroll
		for (int r = 0; r < ITEMS; ++r) {
			bool valid = wid * (32 * ITEMS) + r * 32 + lane < nvalid;
			u32 d = valid ? cs_digit(D, key[r]) : 0xffffffffu;
			u32 peers = __match_any_sync(0xffffffffu, d);
			u32 leader = __ffs(peers) - 1, old = 0;
			if (valid && lane == leader) { old = S.wc[wid][d]; S.wc[wid][d] = old + __popc(peers); }
			old = __shfl_sync(0xffffffffu, old, leader);
			dg[r] = d; rk[r] = old + __popc(peers & lt);
			__syncwarp();
		}
	}
	else {
		#pragma unroll
		for (int r = 0; r < ITEMS; ++r) { dg[r] = 0xffffffffu; rk[r] = 0; }
	}
	__syncthreads();
	if (tid < 256) {
		u32 sum = 0;
		for (u32 w = 0; w < nw; ++w) { u32 c = S.wc[w][tid]; S.wc[w][tid] = sum; sum += c; }
		S.tot[tid] = sum;
	}
	__syncthreads();
}

// S.running[d] = add[d] + exclusive prefix of src[d] over the 256 digits (threads 0..255 hold add).  Ends with a barrier.
NB_DEV void cs_scan_digits(CoopSortSmem& S, const u32* src, u32 add) {
	const u32 tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	u32 t = tid < 256 ? src[tid] : 0;
	u32 incl = warp_incl_scan(t);
	if (tid < 256 && lane == 31) S.sm[wid] = incl;
	__syncthreads();
	if (wid == 0) { u32 w = lane < 8 ? S.sm[lane] : 0; u32 wi = warp_incl_scan(w); if (lane < 8) S.sm[lane] = wi - w; }
	__syncthreads();
	if (tid < 256) S.running[tid] = incl - t + S.sm[wid] + add;
	__syncthreads();
}

// Sorts m <= NB_CS_CAP keys at src[0..m) on digits P.shift[0..npass) entirely inside the block; result to dst[0..m).
template<bool HAS_VALS, int LOCAL>
NB_DEV void cs_local_sort_n(CoopSortSmem& S, const u64* ksrc, const u32* vsrc, u64* kdst, u32* vdst, u32 m, const SortPasses& P, int npass) {
	const u32 tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	u64 key[LOCAL]; u32 val[LOCAL], dg[LOCAL], rk[LOCAL];
	#pragma unroll
	for (int r = 0; r < LOCAL; ++r) {
		u32 i = wid * (32 * LOCAL) + r * 32 + lane;
		key[r] = i < m ? __ldcg(ksrc + i) : 0;
		if (HAS_VALS) val[r] = i < m ? __ldcg(vsrc + i) : 0;
	}
	if (npass == 0) {  // nothing left to sort on: plain copy
		#pragma unroll
		for (int r = 0; r < LOCAL; ++r) {
			u32 i = wid * (32 * LOCAL) + r * 32 + lane;
			if (i < m) { kdst[i] = key[r]; if (HAS_VALS) vdst[i] = val[r]; }
		}
		return;
	}
	__syncthreads();  // every key of the bucket is in registers before anything is written back
	for (int p = 0; p < npass; ++p) {
		cs_rank<LOCAL>(S, key, m, cs_plain(P.shift[p]), dg, rk);
		cs_scan_digits(S, S.tot, 0);
		const bool last = p == npass - 1;
		#pragma unroll
		for (int r = 0; r < LOCAL; ++r)
			if (dg[r] != 0xffffffffu) {
				u32 pos = S.running[dg[r]] + S.wc[wid][dg[r]] + rk[r];
				if (last) { kdst[pos] = key[r]; if (HAS_VALS) vdst[pos] = val[r]; }
				else { S.skeys[pos] = key[r]; if (HAS_VALS) S.svals[pos] = val[r]; }
			}
		__syncthreads();
		if (!last) {
			#pragma unroll
			for (int r = 0; r < LOCAL; ++r) {
				u32 i = wid * (32 * LOCAL) + r * 32 + lane;
				if (i < m) { key[r] = S.skeys[i]; if (HAS_VALS) val[r] = S.svals[i]; }
			}
		}
	}
}

template<bool HAS_VALS>
NB_DEV void cs_local_sort(CoopSortSmem& S, const u64* ksrc, const u32* vsrc, u64* kdst, u32* vdst, u32 m, const SortPasses& P, int npass) {
	// fewer keys per thread for small buckets: the ranking cost grows with the keys a thread holds, not with m
	if (m <= NB_CS_THREADS) cs_local_sort_n<HAS_VALS, 1>(S, ksrc, vsrc, kdst, vdst, m, P, npass);
	else if (m <= 2 * NB_CS_THREADS) cs_local_sort_n<HAS_VALS, 2>(S, ksrc, vsrc, kdst, vdst, m, P, npass);
	else if (m <= 4 * NB_CS_THREADS) cs_local_sort_n<HAS_VALS, 4>(S, ksrc, vsrc, kdst, vdst, m, P, npass);
	else cs_local_sort_n<HAS_VALS, NB_CS_LOCAL>(S, ksrc, vsrc, kdst, vdst, m, P, npass);
}

// A bucket that does not fit the registers of one block (m > NB_CS_CAP: a hot key value such as the ground's tag) is still sorted
// by ONE block: plain LSD over the remaining digits, tile by tile through global memory, ping-ponging between the bucket's own
// region (ka/va, holds the input and receives the result) and the same region of the other buffer (kb/vb, free scratch).
template<bool HAS_VALS>
NB_DEV void cs_block_lsd(CoopSortSmem& S, u64* ka, u32* va, u64* kb, u32* vb, u32 m, const SortPasses& P, int npass) {
	const u32 tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	u64 key[NB_CS_ITEMS]; u32 val[NB_CS_ITEMS], dg[NB_CS_ITEMS], rk[NB_CS_ITEMS];
	u64* kin = ka; u64* kout = kb; u32* vin = va; u32* vout = vb;
	for (int p = 0; p < npass; ++p) {
		const u32 shift = (u32)P.shift[p];
		if (tid < 256) S.h[tid] = 0;
		__syncthreads();
		for (u32 i = tid; i < m; i += NB_CS_THREADS) atomicAdd(&S.h[(u32)(__ldcg(kin + i) >> shift) & 0xff], 1u);
		__syncthreads();
		cs_scan_digits(S, S.h, 0);
		for (u32 base = 0; base < m; base += NB_CS_TILE) {
			#pragma unroll
			for (int r = 0; r < NB_CS_ITEMS; ++r) {
				u32 i = base + wid * (32 * NB_CS_ITEMS) + r * 32 + lane;
				key[r] = i < m ? __ldcg(kin + i) : 0;
				if (HAS_VALS) val[r] = i < m ? __ldcg(vin + i) : 0;
			}
			cs_rank<NB_CS_ITEMS>(S, key, m - base, cs_plain((int)shift), dg, rk);
			#pragma unroll
			for (int r = 0; r < NB_CS_ITEMS; ++r)
				if (dg[r] != 0xffffffffu) {
					u32 pos = S.running[dg[r]] + S.wc[wid][dg[r]] + rk[r];
					kout[pos] = key[r];
					if (HAS_VALS) vout[pos] = val[r];
				}
			__syncthreads();
			if (tid < 256) S.running[tid] += S.tot[tid];
			__syncthreads();
		}
		{ u64* t = kin; kin = kout; kout = t; u32* tv = vin; vin = vout; vout = tv; }
	}
	if (kin != ka)
		for (u32 i = tid; i < m; i += NB_CS_THREADS) { ka[i] = __ldcg(kb + i); if (HAS_VALS) va[i] = __ldcg(vb + i); }
}

// A bucket of m > NB_CS_CAP keys (a hot key value such as the ground's tag; region ka/va in the result buffer, kb/vb = the same
// region of the other buffer, free scratch) is split once more by ONE block on the next digit `level` (counting sort ka -> kb,
// tile by tile); consecutive sub-buckets are then grouped into chunks of <= NB_CS_CAP keys, each sorted in registers on digits
// 0..level (kb -> ka).  A single sub-bucket that is still too large goes through cs_block_lsd.
template<bool HAS_VALS>
NB_DEV void cs_bucket_split(CoopSortSmem& S, u64* ka, u32* va, u64* kb, u32* vb, u32 m, const SortPasses& P, int level) {
	const u32 tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	if (level < 0) return;  // no digits left: the bucket is already in order
	{
		u64 key[NB_CS_ITEMS]; u32 val[NB_CS_ITEMS], dg[NB_CS_ITEMS], rk[NB_CS_ITEMS];
		const u32 shift = (u32)P.shift[level];
		if (tid < 256) S.h[tid] = 0;
		__syncthreads();
		for (u32 i = tid; i < m; i += NB_CS_THREADS) atomicAdd(&S.h[(u32)(__ldcg(ka + i) >> shift) & 0xff], 1u);
		__syncthreads();
		cs_scan_digits(S, S.h, 0);
		if (tid < 256) { S.total[0][tid] = S.h[tid]; S.total[1][tid] = S.running[tid]; }  // sub-bucket sizes and starts
		for (u32 base = 0; base < m; base += NB_CS_TILE) {
			#pragma unroll
			for (int r = 0; r < NB_CS_ITEMS; ++r) {
				u32 i = base + wid * (32 * NB_CS_ITEMS) + r * 32 + lane;
				key[r] = i < m ? __ldcg(ka + i) : 0;
				if (HAS_VALS) val[r] = i < m ? __ldcg(va + i) : 0;
			}
			cs_rank<NB_CS_ITEMS>(S, key, m - base, cs_plain((int)shift), dg, rk);
			#pragma unroll
			for (int r = 0; r < NB_CS_ITEMS; ++r)
				if (dg[r] != 0xffffffffu) {
					u32 pos = S.running[dg[r]] + S.wc[wid][dg[r]] + rk[r];
					kb[pos] = key[r];
					if (HAS_VALS) vb[pos] = val[r];
				}
			__syncthreads();
			if (tid < 256) S.running[tid] += S.tot[tid];
			__syncthreads();
		}
	}
	for (u32 d = 0; d < 256; ) {  // uniform across the block: everybody reads the same table
		u32 gs = S.total[1][d], gm = S.total[0][d], e = d + 1;
		if (gm <= NB_CS_CAP) while (e < 256 && gm + S.total[0][e] <= NB_CS_CAP) { gm += S.total[0][e]; ++e; }
		if (gm > NB_CS_CAP) {  // one value of this digit alone overflows the registers: LSD on the digits below, then move over
			cs_block_lsd<HAS_VALS>(S, kb + gs, vb + gs, ka + gs, va + gs, gm, P, level);
			__syncthreads();
			for (u32 i = tid; i < gm; i += NB_CS_THREADS) { ka[gs + i] = __ldcg(kb + gs + i); if (HAS_VALS) va[gs + i] = __ldcg(vb + gs + i); }
		}
		else if (gm) cs_local_sort<HAS_VALS>(S, kb + gs, vb + gs, ka + gs, va + gs, gm, P, level + 1);
		__syncthreads();
		d = e;
	}
}

template<bool HAS_VALS>
__global__ void __launch_bounds__(NB_CS_THREADS) k_sort_coop(u64* k0, u64* k1, u32* v0, u32* v1, u32* n_ptr, u32* hist /*[gridDim][256]*/, u32* bar, SortPasses P, const u64* keybits /* OR, AND of the keys, or null */, u32 n_max) {
	extern __shared__ __align__(16) unsigned char cs_smem_raw[];
	CoopSortSmem& S = *reinterpret_cast<CoopSortSmem*>(cs_smem_raw);
	const u32 n_in = *n_ptr, n = min(n_in, n_max);
	// a count that ran past the capacity is clamped in place (every block reads either value and sorts the same n keys)
	if (n_in > n_max && blockIdx.x == 0 && threadIdx.x == 0) *n_ptr = n_max;
	if (n == 0) return;
	if (n <= NB_CS_CAP) {
		if (blockIdx.x == 0) cs_local_sort<HAS_VALS>(S, k0, v0, k1, v1, n, P, P.n);
		return;
	}
	const u32 G = gridDim.x, b = blockIdx.x;
	const u32 tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const u32 tiles = (n + NB_CS_TILE - 1) / NB_CS_TILE, per = (tiles + G - 1) / G;
	const u32 begin = min(n, b * per * NB_CS_TILE), end = min(n, begin + per * NB_CS_TILE);
	u64 key[NB_CS_ITEMS]; u32 val[NB_CS_ITEMS], dg[NB_CS_ITEMS], rk[NB_CS_ITEMS];

	// one global counting-sort pass on digit `shift` from (kin, vin) to (kout, vout); leaves S.h = digit totals of the whole input
	auto global_pass = [&](const u64* kin, const u32* vin, u64* kout, u32* vout, const CsDigit& D) {
		if (tid < 256) S.h[tid] = 0;
		__syncthreads();
		for (u32 i = begin + tid; i < end; i += NB_CS_THREADS) atomicAdd(&S.h[cs_digit(D, __ldcg(kin + i))], 1u);
		__syncthreads();
		if (tid < 256) hist[b * 256 + tid] = S.h[tid];
		grid_barrier(bar, G);
		{
			u32 d = tid & 255, q = tid >> 8, bl = 0, tt = 0;
			for (u32 r0 = q; r0 < G; r0 += 32) {  // eight independent loads in flight per round trip
				u32 v[8];
				#pragma unroll
				for (int u = 0; u < 8; ++u) { u32 r = r0 + 4 * u; v[u] = r < G ? __ldcg(&hist[r * 256 + d]) : 0; }
				#pragma unroll
				for (int u = 0; u < 8; ++u) { tt += v[u]; if (r0 + 4 * u < b) bl += v[u]; }
			}
			S.below[q][d] = bl; S.total[q][d] = tt;
		}
		__syncthreads();
		u32 mine = 0;  // keys of digit tid in blocks before this one
		if (tid < 256) { S.h[tid] = S.total[0][tid] + S.total[1][tid] + S.total[2][tid] + S.total[3][tid]; mine = S.below[0][tid] + S.below[1][tid] + S.below[2][tid] + S.below[3][tid]; }
		__syncthreads();
	};
	auto global_scatter = [&](const u64* kin, const u32* vin, u64* kout, u32* vout, const CsDigit& D, u32 mine) {
		cs_scan_digits(S, S.h, mine);
		for (u32 base = begin; base < end; base += NB_CS_TILE) {
			#pragma unroll
			for (int r = 0; r < NB_CS_ITEMS; ++r) {
				u32 i = base + wid * (32 * NB_CS_ITEMS) + r * 32 + lane;
				key[r] = i < end ? __ldcg(kin + i) : 0;
				if (HAS_VALS) val[r] = i < end ? __ldcg(vin + i) : 0;
			}
			cs_rank<NB_CS_ITEMS>(S, key, end - base, D, dg, rk);
			#pragma unroll
			for (int r = 0; r < NB_CS_ITEMS; ++r)
				if (dg[r] != 0xffffffffu) {
					u32 pos = S.running[dg[r]] + S.wc[wid][dg[r]] + rk[r];
					kout[pos] = key[r];
					if (HAS_VALS) vout[pos] = val[r];
				}
			__syncthreads();
			if (tid < 256) S.running[tid] += S.tot[tid];
			__syncthreads();
		}
	};
	// `mine` has to survive between the two lambdas: recompute it from S.below (still intact)
	auto mine_of = [&]() { return tid < 256 ? S.below[0][tid] + S.below[1][tid] + S.below[2][tid] + S.below[3][tid] : 0u; };

	// ---- top digit first ----
	CsDigit top = cs_plain(P.shift[P.n - 1]);
	int nlocal = P.n - 1;  // digits left for the buckets
	if (keybits) {
		u64 varying = keybits[0] ^ keybits[1];
		top.np = 0; top.pos = 0;
		while (varying && top.np < 8) { u32 bit = 63 - __clzll((long long)varying); top.pos |= (u64)bit << (8 * top.np); ++top.np; varying &= ~((u64)1 << bit); }
		if (top.np) nlocal = P.n; else top = cs_plain(P.shift[P.n - 1]);  // (all keys equal: any digit will do)
	}
	global_pass(k0, v0, k1, v1, top);
	const int oversize = __syncthreads_or(tid < 256 && S.h[tid] > 8 * NB_CS_CAP);  // same answer in every block
	if (!oversize) {
		global_scatter(k0, v0, k1, v1, top, mine_of());
		__syncthreads();
		if (tid < 256) S.below[0][tid] = S.h[tid];  // bucket sizes; bucket starts = their exclusive scan
		__syncthreads();
		cs_scan_digits(S, S.below[0], 0);
		if (tid < 256) S.below[1][tid] = S.running[tid];
		grid_barrier(bar, G);
		// Bucket phase.  256 buckets on G = one block per SM (132 on an H100) means two rounds for most blocks and an idle tail for the
		// rest.  When the buckets are small the block instead takes every bucket that STARTS in
		// its slice [b n/G, (b+1) n/G) of the key range and sorts them together, once, on ALL digits (the top digit included: the group
		// spans several of its values) - one local sort of ~n/G keys per block, even across blocks, instead of two of n/256.
		const u32 slice = n / G + 1;
		const bool small = slice < NB_CS_CAP && !__syncthreads_or(tid < 256 && S.below[0][tid] > NB_CS_CAP - slice);
		if (small) {
			const u32 lo = (u32)((u64)b * n / G), hi = (u32)((u64)(b + 1) * n / G);
			const u32 d0 = (u32)__syncthreads_count(tid < 256 && S.below[1][tid] < lo);
			const u32 d1 = (u32)__syncthreads_count(tid < 256 && S.below[1][tid] < hi);
			const u32 s = d0 < 256 ? S.below[1][d0] : n, e = d1 < 256 ? S.below[1][d1] : n;
			if (e > s) cs_local_sort<HAS_VALS>(S, k1 + s, v1 + s, k1 + s, v1 + s, e - s, P, P.n);
			return;
		}
		for (u32 d = b; d < 256; d += G) {
			const u32 m = S.below[0][d], s = S.below[1][d];
			if (m > NB_CS_CAP) cs_bucket_split<HAS_VALS>(S, k1 + s, v1 + s, k0 + s, v0 + s, m, P, nlocal - 1);
			else if (m) cs_local_sort<HAS_VALS>(S, k1 + s, v1 + s, k1 + s, v1 + s, m, P, nlocal);
			__syncthreads();
		}
		return;
	}
	// ---- skewed keys: LSD over all digits ----
	grid_barrier(bar, G);  // every block is done with the top-digit matrix before it is reused
	u64* kin = k0; u64* kout = k1; u32* vin = v0; u32* vout = v1;
	for (int p = 0; p < P.n; ++p) {
		if (p || top.np || P.n > 1) global_pass(kin, vin, kout, vout, cs_plain(P.shift[p]));
		// (one plain digit: its histogram is already in place)
		global_scatter(kin, vin, kout, vout, cs_plain(P.shift[p]), mine_of());
		grid_barrier(bar, G);
		{ u64* t = kin; kin = kout; kout = t; u32* tv = vin; vin = vout; vout = tv; }
	}
	if (kin != k1)  // an even number of digits ended in k0/v0: the result belongs in k1/v1
		for (u32 i = blockIdx.x * NB_CS_THREADS + tid; i < n; i += G * NB_CS_THREADS) { k1[i] = __ldcg(k0 + i); if (HAS_VALS) v1[i] = __ldcg(v0 + i); }
}

struct SortBuffers { u64* keys[2]; u32* vals[2]; u32* hist /*[L.sms][256]*/; u32* bar; };

// Sorts bits [begin_bit, end_bit) of keys[cur] (+vals[cur]), then stably on [begin_bit2, end_bit2); returns which buffer (0/1)
// holds the result.  One k_sort_coop launch, one block per SM, cooperative: the driver guarantees that the blocks meeting at its
// grid barriers are co-resident, also next to other work on the device.  The first min(*n_ptr, n_max) keys are sorted, and *n_ptr
// is lowered to n_max if it was larger.
static int nb_radix_sort(const Launch& L, const SortBuffers& B, u32* n_ptr, int begin_bit, int end_bit, bool has_vals, int cur, int begin_bit2 = 0, int end_bit2 = 0, const u64* keybits = nullptr, u32 n_max = 0xffffffffu) {
	// 8-bit digits, top-aligned per bit range; the lowest digit of a range may overlap the next one (harmless for LSD order)
	SortPasses P; P.n = 0;
	auto add_range = [&](int lo, int hi) {
		int first = P.n;
		for (int shift = hi - 8; shift > lo; shift -= 8) P.shift[P.n++] = shift;
		if (hi > lo) P.shift[P.n++] = lo;
		for (int i = first, j = P.n - 1; i < j; ++i, --j) { int t = P.shift[i]; P.shift[i] = P.shift[j]; P.shift[j] = t; }  // ascending
	};
	add_range(begin_bit, end_bit);
	add_range(begin_bit2, end_bit2);
	u64* k0 = B.keys[cur]; u64* k1 = B.keys[cur ^ 1]; u32* v0 = B.vals[cur]; u32* v1 = B.vals[cur ^ 1]; u32* hist = B.hist; u32* bar = B.bar;
	void* args[] = { &k0, &k1, &v0, &v1, &n_ptr, &hist, &bar, &P, &keybits, &n_max };
	cudaLaunchCooperativeKernel(has_vals ? (void*)k_sort_coop<true> : (void*)k_sort_coop<false>, dim3(L.sms), dim3(NB_CS_THREADS), args, sizeof(CoopSortSmem), L.stream);
	*L.counter += 1;
	return cur ^ 1;
}

// ---------------- warp-aggregated append ----------------
NB_DEV u32 warp_append_slot(u32* counter) {
	u32 active = __activemask();
	u32 lane = threadIdx.x & 31;
	u32 leader = __ffs(active) - 1;
	u32 base = 0;
	if (lane == leader) base = atomicAdd(counter, (u32)__popc(active));
	base = __shfl_sync(active, base, leader);
	return base + __popc(active & ((1u << lane) - 1u));
}
