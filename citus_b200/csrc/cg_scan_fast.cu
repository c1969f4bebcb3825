/*
 * cg_scan_fast.cu -- the specialised form of the fused scan kernel for the shape that
 * dominates analytic shard tasks (BASELINE configs 1-3):
 *
 *     SELECT [key,] count(*), sum(c1) [, sum(c2), sum(c3)] FROM shard
 *     WHERE q0 BETWEEN lo0 AND hi0 [AND q1 BETWEEN lo1 AND hi1] [GROUP BY key]
 *
 * over 8-byte integer columns, for chunk groups without NULLs in the columns read
 * (chunk groups that have NULLs go through the general kernel in cg_scan.cu into the same
 * accumulators).  Same semantics and same reference citations as cg_scan.cu (K1 decode of
 * the NULL-free value stream = a dense int8 array, columnar_reader.c:1542-1572; K3 ExecQual;
 * K4 nodeAgg transition functions), but the plan shape is a template parameter, so the
 * per-row work is a handful of instructions: the kernel is bound by HBM loads and by the
 * L2 reduction requests, not by instruction issue.
 *
 *   NQ    range conjuncts, each on its own column (several btree conjuncts on one column
 *         are intersected into one [lo, hi] on the host)
 *   MODE  plain aggregate / direct-indexed table / hash table
 *   NS    sum(column) aggregates
 *   PACK  grouped modes: count(*) and sum number 0 share one 64-bit word
 *         (optimistic packing, see include/citus_gpu.h cg_partial_set_packing)
 * Column roles map to fixed register positions: quals first, then the key, then the sums.
 */
#include "cg_internal.h"

#define CGF_THREADS 256

/* streaming column data: read-only path, no L1 allocation, first to leave L2 -- each byte is
 * used once and must not push the group table out of the 50 MB L2 */
__device__ __forceinline__ void ldg16(const void *p, uint64_t &a, uint64_t &b, uint64_t policy)
{
	asm("ld.global.nc.L1::no_allocate.L2::cache_hint.v2.u64 {%0, %1}, [%2], %3;" : "=l"(a), "=l"(b) : "l"(p), "l"(policy));
}

/* one 64-bit word of a narrow image (DevPackCol): same streaming path and hint as ldg16 */
__device__ __forceinline__ uint64_t ldg8(const void *p, uint64_t policy)
{
	uint64_t a;
	asm("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(a) : "l"(p), "l"(policy));
	return a;
}

/* group-table update: fire-and-forget reduction at the L2 atomic unit */
__device__ __forceinline__ void red_add_u64(uint64_t *p, uint64_t v)
{
	asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ uint64_t policy_evict_first()
{
	uint64_t pol;
	asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
	return pol;
}

/* must match cg_home_slot() in cg_device.cuh */
__device__ __forceinline__ uint64_t home_slot(int64_t key, int hash_shift)
{
	return ((uint64_t) key * 0x9E3779B97F4A7C15ull) >> hash_shift;
}

__device__ __noinline__ void raise_flag(unsigned long long *stats, unsigned long long flag)
{
	atomicOr(stats + 2, flag);
}

/* slot of the group's entry, or ~0 after raising an error flag */
#define CGF_NOSLOT (~0ull)

__device__ __noinline__ uint64_t hash_slot_slow(const FPlan &P, int64_t key, uint64_t h)
{
	if (key == CG_HASH_EMPTY) return P.capacity + 1;
	const uint64_t mask = P.capacity - 1;
	for (uint32_t probes = 0; probes < 8192; probes++)
	{
		unsigned long long *kp = (unsigned long long *) (P.hkeys + h);
		long long cur = (long long) __ldcg(kp);
		if (cur == key) return h;
		if (cur == CG_HASH_EMPTY)
		{
			long long old = (long long) atomicCAS(kp, (unsigned long long) CG_HASH_EMPTY, (unsigned long long) key);
			if (old == CG_HASH_EMPTY || old == key) return h;
		}
		h = (h + 1) & mask;
	}
	raise_flag(P.stats, CG_ERRFLAG_TABLE_FULL);
	return CGF_NOSLOT;
}
template <int MODE>
__device__ __forceinline__ uint64_t fast_slot(const FPlan &P, int64_t key)
{
	if (MODE == CG_MODE_DENSE)
	{
		uint64_t slot = (uint64_t) key - (uint64_t) P.key_min;
		if (slot >= P.capacity)
		{
			raise_flag(P.stats, CG_ERRFLAG_KEY_RANGE);
			return CGF_NOSLOT;
		}
		return slot;
	}
	else
	{
		/* the home-slot probe is straight-line code (all lanes of the warp issue it together);
		 * only a miss enters the probing / claiming loop */
		uint64_t h = home_slot(key, P.hash_shift);
		long long cur = (long long) __ldcg((unsigned long long *) (P.hkeys + h));   /* keys only ever go EMPTY -> key */
		if (cur == key && key != CG_HASH_EMPTY) return h;
		return hash_slot_slow(P, key, h);
	}
}

/* word pointer of the group's entry, or NULL after raising an error flag */
template <int MODE>
__device__ __forceinline__ uint64_t *fast_entry(const FPlan &P, int64_t key)
{
	uint64_t slot = fast_slot<MODE>(P, key);
	return slot == CGF_NOSLOT ? nullptr : P.table + slot * (uint64_t) P.stride;
}

template <int NQ>
__device__ __forceinline__ bool fast_pass(const FPlan &P, const int64_t *v)
{
	bool pass = true;
#pragma unroll
	for (int q = 0; q < NQ; q++)
	{
		bool in = v[q] >= P.qlo[q] && v[q] <= P.qhi[q];
		pass = pass && (in != (bool) P.qneg[q]);
	}
	return pass;
}

/* wide (exact) update of one sum word / word pair */
__device__ __forceinline__ void wide_sum(const FPlan &P, uint64_t *e, int s, int64_t x)
{
	if (P.slimbs[s] == 1)
	{
		if (x > P.sbound[s] || x < -P.sbound[s]) raise_flag(P.stats, CG_ERRFLAG_SUM_BOUND);
		red_add_u64(e + P.sword[s], (uint64_t) x);
	}
	else
	{
		red_add_u64(e + P.sword[s], (uint64_t) (uint32_t) x);
		red_add_u64(e + P.sword[s] + 1, (uint64_t) (x >> 32));
	}
}

/*
 * Paired table update, hash tables with single-word sums.  The accumulator words of one
 * group are adjacent (one 32-byte sector, right behind the key the lookup just read); lanes
 * work in pairs: in round 0 both lanes of a pair update the row of the even lane (even lane:
 * word 0, odd lane: word 1, ...), in round 1 the row of the odd lane.  Must be called by all
 * 32 lanes.
 */
template <int NS>
__device__ __forceinline__ void paired_update(const FPlan &P, bool pass, uint64_t *e, const int64_t *sums)
{
	const unsigned lane = threadIdx.x & 31u;
	const bool odd = lane & 1u;
	__syncwarp();
	uint64_t pe = __shfl_xor_sync(0xffffffffu, (uint64_t) e, 1);
	bool ppass = __shfl_xor_sync(0xffffffffu, (int) pass, 1) != 0;
	int64_t ps[NS > 0 ? NS : 1];
#pragma unroll
	for (int s = 0; s < NS; s++) ps[s] = __shfl_xor_sync(0xffffffffu, sums[s], 1);
#pragma unroll
	for (int round = 0; round < 2; round++)
	{
		const bool mine = (odd == (round == 1));
		uint64_t *te = mine ? e : (uint64_t *) pe;
		const bool tpass = mine ? pass : ppass;
		if (tpass)
		{
#pragma unroll
			for (int j = 0; j < (NS + 2) / 2; j++)
			{
				const int w = 2 * j + (odd ? 1 : 0);     /* 0 = row count, 1.. = sums */
				if (w == 0) red_add_u64(te, 1ull);
				else if (w <= NS)
				{
					int64_t x = 0;
					int wordidx = 0;
#pragma unroll
					for (int s = 0; s < NS; s++)
						if (s == w - 1) { x = mine ? sums[s] : ps[s]; wordidx = P.sword[s]; }
					red_add_u64(te + wordidx, (uint64_t) x);
				}
			}
		}
	}
}

template <int NS>
struct FastAcc
{
	uint64_t rows;                      /* plain aggregate: rows passed; PACK: rows added to packed words */
	uint64_t lo[NS > 0 ? NS : 1];
	int64_t hi[NS > 0 ? NS : 1];
};

/* one row of a plain aggregate or of a direct-indexed / unpaired table */
template <int NQ, int MODE, int NS, bool PACK>
__device__ __forceinline__ void fast_row(const FPlan &P, const int64_t *v, FastAcc<NS> &acc, uint32_t &removed)
{
	constexpr int KEYPOS = NQ;
	constexpr int SUMPOS = NQ + (MODE != CG_MODE_GLOBAL ? 1 : 0);
	if (!fast_pass<NQ>(P, v))
	{
		removed++;
		return;
	}
	if (MODE == CG_MODE_GLOBAL)
	{
		acc.rows++;
#pragma unroll
		for (int s = 0; s < NS; s++)
		{
			int64_t x = v[SUMPOS + s];
			/* the limbs are exact whatever the bound; a violated bound is still the caller's error */
			if (P.slimbs[s] == 1 && (x > P.sbound[s] || x < -P.sbound[s])) raise_flag(P.stats, CG_ERRFLAG_SUM_BOUND);
			acc.lo[s] += (uint64_t) (uint32_t) x;
			acc.hi[s] += x >> 32;
		}
		return;
	}
	if (PACK)
	{
		/* one reduction for count(*) and sum 0: word += (x << C) + 1 (mod 2^64) */
		uint64_t slot = fast_slot<MODE>(P, v[KEYPOS]);
		if (slot == CGF_NOSLOT) return;
		int64_t x = v[SUMPOS];
		if (x > P.sbound[0] || x < -P.sbound[0]) raise_flag(P.stats, CG_ERRFLAG_SUM_BOUND);
		red_add_u64(P.packed + slot, ((uint64_t) x << P.pack_shift) + 1ull);
		acc.rows++;
		if (NS > 1)
		{
			uint64_t *e = P.table + slot * (uint64_t) P.stride;
#pragma unroll
			for (int s = 1; s < NS; s++) wide_sum(P, e, s, v[SUMPOS + s]);
		}
		return;
	}
	uint64_t *e = fast_entry<MODE>(P, v[KEYPOS]);
	if (e == nullptr) return;
	red_add_u64(e, 1ull);
#pragma unroll
	for (int s = 0; s < NS; s++) wide_sum(P, e, s, v[SUMPOS + s]);
}

__device__ __forceinline__ uint64_t warp_sum(uint64_t x)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
	return x;
}

/*
 * NARROW: the columns come from the shard's narrow images instead of the arena.  Rows [64 k, 64 k + 64) of a chunk column
 * are the `width` words [k * width, (k + 1) * width) of its bit stream, and a warp's 64 consecutive rows are one such
 * block (every warp starts at a multiple of 64 rows): lane i loads word i, and each lane takes the (at most two) words its
 * two rows' fields lie in from the lanes that loaded them.  Narrow plans have at most three columns (cg_host.cpp
 * set_narrow); their instances are held to 64 registers (four CTAs per SM, as the plain C2 instance), which they meet
 * without spilling.
 */
template <int NQ, int MODE, int NS, bool PACK, int U, bool NARROW>
__global__ void __launch_bounds__(CGF_THREADS, NARROW ? 4 : 0)
cg_scan_fast_kernel(const __grid_constant__ FPlan P)
{
	constexpr int NC = NQ + (MODE != CG_MODE_GLOBAL ? 1 : 0) + NS;
	constexpr int NCA = NC > 0 ? NC : 1;
	constexpr int KEYPOS = NQ;
	constexpr int SUMPOS = NQ + (MODE != CG_MODE_GLOBAL ? 1 : 0);
	/* the next scan launch of a chain may start as soon as every CTA of this one runs (cg_chain_scan, cg_host.cpp) */
	asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
	FastAcc<NS> acc;
	acc.rows = 0;
#pragma unroll
	for (int s = 0; s < NS; s++) { acc.lo[s] = 0; acc.hi[s] = 0; }
	uint32_t removed = 0;
	unsigned long long scanned = 0;
	const uint32_t tid = threadIdx.x;
	const uint32_t lane = tid & 31u;
	const uint64_t pol_stream = policy_evict_first();
	/* hash tables with single-word sums: lane-paired updates (decided per launch, uniform) */
	const bool paired = (MODE == CG_MODE_HASH) && !PACK && NS > 0 && (P.flags & CG_FAST_PAIRED);

	/* work unit = (chunk group, row range): small launches cut chunk groups into slices so that every SM has work */
	const uint32_t nunits = P.nselected * (uint32_t) P.slices;
	for (uint32_t unit = blockIdx.x; unit < nunits; unit += gridDim.x)
	{
		const uint32_t ci = P.slices == 1 ? unit : unit / (uint32_t) P.slices;
		const uint32_t sl = P.slices == 1 ? 0u : unit - ci * (uint32_t) P.slices;
		const DevChunkCol *cc = P.chunkcols + (uint64_t) P.selected[ci] * (uint64_t) P.nstaged;
		const uint32_t chunk_rows = __ldg(&cc[0].row_count);
		const uint32_t row0 = sl * P.slice_rows;
		const uint32_t rows = min(chunk_rows, row0 + P.slice_rows);       /* this unit covers rows [row0, rows) */
		const uint8_t *vp[NCA];
		/* narrow: the stream's first word (an index into P.narrow_base, which stays in the parameter bank), base, width */
		uint32_t nword[NCA], nwidth[NCA];
		int64_t nbase[NCA];
#pragma unroll
		for (int c = 0; c < NC; c++)
		{
			if (NARROW)
			{
				const DevPackCol *pc = P.packcols + (uint64_t) P.selected[ci] * (uint64_t) P.nstaged + P.slot[c];
				nword[c] = (uint32_t) (__ldg(&pc->off) / 8);
				nbase[c] = __ldg(&pc->base);
				nwidth[c] = __ldg(&pc->width);
			}
			else
				vp[c] = P.arena + __ldg(&cc[P.slot[c]].values_off);
		}
		scanned += (tid == 0 && sl == 0) ? chunk_rows : 0;
		if (NC == 0)
		{
			/* count(*) without any column: every row of the chunk group passes */
			if (tid == 0 && sl == 0) acc.rows += chunk_rows;
			continue;
		}
		for (uint32_t base = row0; base < rows; base += CGF_THREADS * 2 * U)
		{
			int64_t v0[U][NCA], v1[U][NCA];
			uint64_t raw[U][NCA];
#pragma unroll
			for (int u = 0; u < U; u++)
			{
				uint32_t r = base + (u * CGF_THREADS + tid) * 2;
				if (NARROW)
				{
					const uint32_t r0 = base + (u * CGF_THREADS + (tid & ~31u)) * 2;     /* the warp's first row */
#pragma unroll
					for (int c = 0; c < NC; c++)
					{
						raw[u][c] = 0;
						if (r0 < rows && lane < nwidth[c])
							raw[u][c] = ldg8((const uint64_t *) P.narrow_base + nword[c] + (r0 / 64u) * nwidth[c] + lane, pol_stream);
					}
				}
				else if (r < rows)
				{
#pragma unroll
					for (int c = 0; c < NC; c++)
					{
						uint64_t a, b;
						ldg16(vp[c] + (uint64_t) r * 8, a, b, pol_stream);
						v0[u][c] = (int64_t) a; v1[u][c] = (int64_t) b;
					}
				}
			}
#pragma unroll
			for (int u = 0; u < U; u++)
			{
				uint32_t r = base + (u * CGF_THREADS + tid) * 2;
				if (NARROW && base + (u * CGF_THREADS + (tid & ~31u)) * 2 < rows)
				{
					/* warp-uniform: the fields of rows r, r + 1 lie in bits [2 lane w, 2 lane w + 2 w) of the block, at most
					 * 64 bits (w <= 32) across words lo and lo + 1 (lo + 1 = 32 only when it is not needed) */
#pragma unroll
					for (int c = 0; c < NC; c++)
					{
						/* re-read per row block (a register move the compiler cannot hoist): the shift amounts derived from
						 * it are cheap to recompute, and hoisting them for every column would cost the registers of a
						 * fourth CTA per SM */
						uint32_t w;
						asm volatile("mov.b32 %0, %1;" : "=r"(w) : "r"(nwidth[c]));
						const uint32_t b0 = 2u * lane * w, lo = b0 >> 6, sh = b0 & 63u;
						const uint64_t a = __shfl_sync(0xffffffffu, raw[u][c], (int) lo);
						const uint64_t b = __shfl_sync(0xffffffffu, raw[u][c], (int) ((lo + 1) & 31u));
						const uint64_t x = (a >> sh) | ((b << 1) << (63u - sh));
						const uint64_t mask = (1ull << w) - 1ull;
						v0[u][c] = (int64_t) ((uint64_t) nbase[c] + (x & mask));
						v1[u][c] = (int64_t) ((uint64_t) nbase[c] + ((x >> w) & mask));
					}
				}
				if (MODE == CG_MODE_HASH && paired)
				{
					/* warp-converged: lanes past the end of the chunk group take part with pass = false */
#pragma unroll
					for (int half = 0; half < 2; half++)
					{
						const int64_t *v = half ? v1[u] : v0[u];
						const bool valid = r + half < rows;
						bool pass = valid && fast_pass<NQ>(P, v);
						removed += (valid && !pass) ? 1u : 0u;
						uint64_t *e = nullptr;
						if (pass)
						{
							e = fast_entry<MODE>(P, v[KEYPOS]);
							pass = e != nullptr;
#pragma unroll
							for (int s = 0; s < NS; s++)
								if (v[SUMPOS + s] > P.sbound[s] || v[SUMPOS + s] < -P.sbound[s])
									raise_flag(P.stats, CG_ERRFLAG_SUM_BOUND);
						}
						paired_update<NS>(P, pass, e, v + SUMPOS);
					}
				}
				else if (r < rows)
				{
					fast_row<NQ, MODE, NS, PACK>(P, v0[u], acc, removed);
					if (r + 1 < rows) fast_row<NQ, MODE, NS, PACK>(P, v1[u], acc, removed);
				}
			}
		}
	}

	unsigned long long rem = warp_sum(removed);
	unsigned long long scn = warp_sum(scanned);
	if ((tid & 31) == 0)
	{
		if (scn) atomicAdd(P.stats + 0, scn);
		if (rem) atomicAdd(P.stats + 1, rem);
	}
	if (PACK)
	{
		uint64_t added = warp_sum(acc.rows);
		if ((tid & 31) == 0 && added) atomicAdd(P.stats + CG_STAT_PACKED_ADDED, (unsigned long long) added);
	}
	if (MODE == CG_MODE_GLOBAL)
	{
		uint64_t rows_passed = warp_sum(acc.rows);
		if ((tid & 31) == 0 && rows_passed) red_add_u64(P.table, rows_passed);
#pragma unroll
		for (int s = 0; s < NS; s++)
		{
			uint64_t lo = warp_sum(acc.lo[s]);
			uint64_t hi = warp_sum((uint64_t) acc.hi[s]);
			if ((tid & 31) == 0 && (lo | hi))
			{
				if (P.slimbs[s] == 1) red_add_u64(P.table + P.sword[s], lo + (hi << 32));
				else
				{
					red_add_u64(P.table + P.sword[s], lo);
					red_add_u64(P.table + P.sword[s] + 1, hi);
				}
			}
		}
	}
}

/*
 * Drain of the packed words into the exact accumulators: word = (sum << C) + n (mod 2^64) with
 * n < 2^C, so n = word mod 2^C and sum = (word - n) >> C (arithmetic).  The drained counts are
 * added up; cg_host.cpp compares them with the rows the scan kernels added.
 */
__global__ void __launch_bounds__(256)
cg_drain_kernel(uint64_t *packed, uint64_t *table, uint64_t entries, int stride, int pack_word, int shift,
				unsigned long long *stats)
{
	const uint64_t mask = (1ull << shift) - 1ull;
	unsigned long long local = 0;
	for (uint64_t slot = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; slot < entries; slot += (uint64_t) gridDim.x * blockDim.x)
	{
		uint64_t w = packed[slot];
		if (w == 0) continue;
		uint64_t n = w & mask;
		int64_t sum = (int64_t) (w - n) >> shift;
		uint64_t *ent = table + slot * (uint64_t) stride;
		ent[0] += n;
		ent[pack_word] += (uint64_t) sum;
		packed[slot] = 0;
		local += n;
	}
	local = warp_sum(local);
	if ((threadIdx.x & 31) == 0 && local) atomicAdd(stats + CG_STAT_PACKED_DRAINED, local);
}

int cg_launch_drain(CgPartial *p, cudaStream_t stream)
{
	if (!p->d_packed || !p->packed_dirty) return CG_OK;
	int rc = cg_chain_end(cg_ctx(), stream);
	if (rc) return rc;
	unsigned blocks = (unsigned) ((p->entries + 255) / 256);
	if (blocks > (unsigned) cg_ctx()->sm_count * 8) blocks = (unsigned) cg_ctx()->sm_count * 8;
	cg_drain_kernel<<<blocks, 256, 0, stream>>>(p->d_packed, p->d_table, p->entries, p->stride, p->pack_word, p->pack_shift, p->d_stats);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	p->packed_dirty = false;
	p->read_packed_direct = false;
	p->wide_dirty = true;
	p->launches_since_drain = 0;
	p->rows_since_drain = 0;
	return CG_OK;
}

template <int NQ, int MODE, int NS, bool PACK, bool NARROW>
static int launch_fast_variant(CgContext *ctx, const FPlan &plan, cudaStream_t stream)
{
	constexpr int NC = NQ + (MODE != CG_MODE_GLOBAL ? 1 : 0) + NS;
	/* narrow plans never have more than three columns (set_narrow): no narrow instance for the wider shapes */
	if constexpr (NARROW && NC > 3)
		return launch_fast_variant<NQ, MODE, NS, PACK, false>(ctx, plan, stream);
	else
	{
	/* two row pairs per lane and iteration, as the plain instances, where they fit 64 registers without spilling (up to two
	 * columns): a lone launch of few, short work units then waits on as few dependent load rounds as the plain kernel.  A
	 * three-column plan (C2) takes one row pair: the registers of a second would cost the fourth CTA per SM */
	constexpr int U = NARROW ? (NC <= 2 ? 2 : 1) : (NC <= 3 ? 2 : 1);
	static int occ = 0;
	if (occ == 0)
	{
		CG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, cg_scan_fast_kernel<NQ, MODE, NS, PACK, U, NARROW>, CGF_THREADS, 0));
		if (occ < 1) occ = 1;
	}
	uint32_t grid = (uint32_t) (ctx->sm_count * occ);
	FPlan launch = plan;
	launch.slices = 1; launch.slice_rows = 1u << 30;
	if (plan.nselected < 2 * grid && plan.max_cg_rows > 0)
		cg_choose_slices(plan.nselected, grid, CGF_THREADS * 2 * U, plan.max_cg_rows, &launch.slices, &launch.slice_rows);
	const uint64_t units = (uint64_t) plan.nselected * (uint64_t) launch.slices;
	if (grid > units) grid = (uint32_t) units;
	if (grid == 0) return CG_OK;
	bool overlap;
	int rc = cg_chain_scan(ctx, stream, true, &overlap);
	if (rc) return rc;
	cudaLaunchAttribute attr;
	attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
	attr.val.programmaticStreamSerializationAllowed = 1;
	cudaLaunchConfig_t cfg = {};
	cfg.gridDim = dim3(grid);
	cfg.blockDim = dim3(CGF_THREADS);
	cfg.stream = stream;
	cfg.attrs = &attr;
	cfg.numAttrs = overlap ? 1 : 0;
	CG_CUDA(cudaLaunchKernelEx(&cfg, cg_scan_fast_kernel<NQ, MODE, NS, PACK, U, NARROW>, launch));
	g_cg_launches++;
	return CG_OK;
	}
}

template <int NQ, int MODE, bool NARROW>
static int launch_fast_ns(CgContext *ctx, const FPlan &plan, cudaStream_t stream)
{
	if (MODE != CG_MODE_GLOBAL && plan.packed)
	{
		constexpr int PM = MODE == CG_MODE_GLOBAL ? CG_MODE_DENSE : MODE;
		switch (plan.nsums)
		{
			case 1: return launch_fast_variant<NQ, PM, 1, true, NARROW>(ctx, plan, stream);
			case 2: return launch_fast_variant<NQ, PM, 2, true, NARROW>(ctx, plan, stream);
			default: return launch_fast_variant<NQ, PM, 3, true, NARROW>(ctx, plan, stream);
		}
	}
	switch (plan.nsums)
	{
		case 0: return launch_fast_variant<NQ, MODE, 0, false, NARROW>(ctx, plan, stream);
		case 1: return launch_fast_variant<NQ, MODE, 1, false, NARROW>(ctx, plan, stream);
		case 2: return launch_fast_variant<NQ, MODE, 2, false, NARROW>(ctx, plan, stream);
		default: return launch_fast_variant<NQ, MODE, 3, false, NARROW>(ctx, plan, stream);
	}
}

template <int NQ, bool NARROW>
static int launch_fast_mode(CgContext *ctx, const FPlan &plan, cudaStream_t stream)
{
	switch (plan.mode)
	{
		case CG_MODE_GLOBAL: return launch_fast_ns<NQ, CG_MODE_GLOBAL, NARROW>(ctx, plan, stream);
		case CG_MODE_DENSE: return launch_fast_ns<NQ, CG_MODE_DENSE, NARROW>(ctx, plan, stream);
		default: return launch_fast_ns<NQ, CG_MODE_HASH, NARROW>(ctx, plan, stream);
	}
}

int cg_launch_scan_fast(CgContext *ctx, const FPlan &plan, cudaStream_t stream)
{
	if (plan.narrow)
		switch (plan.nquals)
		{
			case 0: return launch_fast_mode<0, true>(ctx, plan, stream);
			case 1: return launch_fast_mode<1, true>(ctx, plan, stream);
			default: return launch_fast_mode<2, true>(ctx, plan, stream);
		}
	switch (plan.nquals)
	{
		case 0: return launch_fast_mode<0, false>(ctx, plan, stream);
		case 1: return launch_fast_mode<1, false>(ctx, plan, stream);
		default: return launch_fast_mode<2, false>(ctx, plan, stream);
	}
}
