/*
 * cg_scan.cu -- the fused columnar scan kernels (sm_90a).
 *
 * One launch does, for every selected chunk group of a staged shard, what the reference
 * does one row and one function call at a time (SURVEY.md 3.3):
 *   K1 decode      DeserializeBoolArray / DeserializeDatumArray
 *                  backend/columnar/columnar_reader.c:1506-1572   (exists bitmap, NULL-compacted
 *                  value stream -> row values; the prefix popcount lives in the rank directory)
 *   K3 filter      [PG] ExecQual under ExecScan, backend/columnar/columnar_customscan.c:1907-1913
 *   K4 aggregate   [PG] nodeAgg + transition functions for the worker half chosen by
 *                  planner/multi_logical_optimizer.c:3160-3484
 * reading every needed byte of HBM exactly once with 16-byte vector loads.  There is no
 * dense contraction on this path, so no tensor cores: the roofline is HBM bandwidth.
 *
 * Accumulators are 64-bit "words" combined by one commutative op each (CG_WORD_*), so
 * that per-thread registers (plain aggregate), global-memory group tables (GROUP BY)
 * and other GPUs' partials all merge with the same code.  An exact 128-bit integer SUM
 * is kept as two words: sum of the low 32 bits (unsigned) and sum of term >> 32
 * (signed); no carries are needed until the value is read (sum = hi * 2^32 + lo).
 */
#include <stdlib.h>

#include "cg_internal.h"

#define CG_THREADS 256

#include "cg_device.cuh"

/*
 * Find (or claim) the table entry of a group key.  Returns the word pointer of the
 * entry (word 0 = rows in group) or NULL after raising an error flag.
 *   dense: entry = key - key_min, NULL key -> entry `capacity`
 *   hash : open addressing, linear probing over a separate key array (8 B per slot, so the
 *          probed working set is a quarter of an array-of-structs table), 64-bit CAS to claim
 *          a slot; the NULL group and the key equal to the EMPTY sentinel live in two extra
 *          entries behind the addressable ones
 */
template <int MODE>
__device__ __forceinline__ uint64_t *find_entry(const KPlan &P, int64_t key, bool key_null)
{
	if (MODE == CG_MODE_DENSE)
	{
		uint64_t slot = dense_slot_of_packed(P, key, key_null);
		if (slot == ~0ull)
		{
			atomicOr(P.stats + 2, CG_ERRFLAG_KEY_RANGE);
			return nullptr;
		}
		return P.table + slot * (uint64_t) P.stride;
	}
	else
	{
		if (key_null) return P.table + P.capacity * (uint64_t) P.stride;
		if (key == CG_HASH_EMPTY) return P.table + (P.capacity + 1) * (uint64_t) P.stride;
		uint64_t mask = P.capacity - 1;
		uint64_t h = cg_home_slot(key, P.hash_shift);
		for (uint32_t probes = 0; probes < 8192; probes++)
		{
			unsigned long long *kp = (unsigned long long *) (P.hkeys + h);
			long long cur = (long long) __ldcg(kp);     /* L2: keys only ever go EMPTY -> key */
			if (cur == key) return P.table + h * (uint64_t) P.stride;
			if (cur == CG_HASH_EMPTY)
			{
				long long old = (long long) atomicCAS(kp, (unsigned long long) CG_HASH_EMPTY, (unsigned long long) key);
				if (old == CG_HASH_EMPTY || old == key) return P.table + h * (uint64_t) P.stride;
			}
			h = (h + 1) & mask;
		}
		atomicOr(P.stats + 2, CG_ERRFLAG_TABLE_FULL);
		return nullptr;
	}
}

/* per-thread accumulators of the plain-aggregate mode */
template <int NAC>
struct ThreadAcc
{
	uint64_t w[NAC][3];     /* [agg][word0, word0+1, NULL-input count] */
	uint64_t rows;
};

template <int NCC, int NAC, int MODE>
__device__ __forceinline__ void process_row(const KPlan &P, const int64_t (&v)[NCC], uint32_t nullmask,
											ThreadAcc<NAC> &acc, uint32_t &removed)
{
	/* K3: WHERE tree, three-valued: an atom on a NULL input is not TRUE */
	const bool pass = eval_where<NCC>(P, v, nullmask);
	if (!pass)
	{
		removed++;
		return;
	}

	uint64_t *entry = nullptr;
	if (MODE != CG_MODE_GLOBAL)
	{
		int64_t key;
		bool key_null;
		if (P.ngroup == 1)
		{
			int c = P.gcol[0];
			key_null = (nullmask >> c) & 1u;
			key = pick<NCC>(v, c);
		}
		else
		{
			int c0 = P.gcol[0], c1 = P.gcol[1];
			if (((nullmask >> c0) | (nullmask >> c1)) & 1u)
			{
				atomicOr(P.stats + 2, CG_ERRFLAG_NULL_MULTIKEY);
				return;
			}
			key_null = false;
			key = (int64_t) ((uint64_t) (uint32_t) pick<NCC>(v, c0) | ((uint64_t) (uint32_t) pick<NCC>(v, c1) << 32));
		}
		entry = find_entry<MODE>(P, key, key_null);
		if (entry == nullptr) return;
		atomicAdd((unsigned long long *) entry, 1ull);
	}
	else
		acc.rows++;

	/* K4: transition functions */
#pragma unroll
	for (int a = 0; a < NAC; a++)
	{
		if (a < P.naggs)
		{
			const KAgg &g = P.aggs[a];
			if (g.kind == CG_AGG_COUNT_STAR) continue;
			bool isnull = false;
			int64_t it = 1;
			double ft = 1.0;
#pragma unroll
			for (int f = 0; f < 3; f++)
			{
				if (f < g.nfactors)
				{
					int c = g.pcol[f];
					isnull = isnull || ((nullmask >> c) & 1u);
					if (g.is_float)
						ft *= __longlong_as_double(g.a[f]) + __longlong_as_double(g.b[f]) * __longlong_as_double(pick<NCC>(v, c));
				}
			}
			if (!g.is_float) it = int_term<NCC>(g, v, isnull, P.stats);
			if (isnull)
			{
				/* strict transition function: a NULL input is skipped, only counted */
				if (MODE == CG_MODE_GLOBAL) acc.w[a][2]++;
				else atomicAdd((unsigned long long *) entry + g.nullword, 1ull);
				continue;
			}
			if (g.kind == CG_AGG_COUNT) continue;   /* count(x) = rows - NULL inputs */
			uint64_t w0, w1 = 0;
			if (g.kind == CG_AGG_SUM)
			{
				if (g.is_float) w0 = (uint64_t) __double_as_longlong(ft);
				else if (g.nlimbs == 1)
				{
					if (it > g.bound || it < -g.bound) atomicOr(P.stats + 2, CG_ERRFLAG_SUM_BOUND);
					w0 = (uint64_t) it;
				}
				else { w0 = (uint64_t) (uint32_t) it; w1 = (uint64_t) (it >> 32); }
			}
			else /* MIN / MAX */
				w0 = g.is_float ? f8_ordered(__double_as_longlong(ft)) : (uint64_t) it;
			const bool two = (g.kind == CG_AGG_SUM && !g.is_float && g.nlimbs == 2);
			if (MODE == CG_MODE_GLOBAL)
			{
				acc.w[a][0] = word_combine(P.wordop[g.word0], acc.w[a][0], w0);
				if (two) acc.w[a][1] += w1;
			}
			else
			{
				word_apply_global(entry + g.word0, P.wordop[g.word0], w0);
				if (two) atomicAdd((unsigned long long *) entry + g.word0 + 1, (unsigned long long) w1);
			}
		}
	}
}

__device__ __forceinline__ uint64_t warp_reduce_word(uint64_t x, int op)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
	{
		uint64_t y = __shfl_xor_sync(0xffffffffu, x, o);
		x = word_combine(op, x, y);
	}
	return x;
}

/*
 * The fused kernel.  Persistent CTAs stride over the selected chunk groups; inside a
 * chunk group every thread takes two consecutive rows per step (one 16-byte load per
 * 8-byte column) and U steps are loaded before any is consumed.
 *   NCC  capacity of the per-thread column register file (plan columns <= NCC)
 *   NAC  capacity of the per-thread aggregate accumulators (plain aggregate mode)
 *   ALL8 every plan column is 8 bytes wide (skips the width switch)
 */
template <int NCC, int NAC, int MODE, bool ALL8, int U>
__global__ void __launch_bounds__(CG_THREADS, 4)
cg_scan_kernel(const __grid_constant__ KPlan P)
{
	ThreadAcc<NAC> acc;
	acc.rows = 0;
#pragma unroll
	for (int a = 0; a < NAC; a++)
	{
		acc.w[a][0] = (a < P.naggs && P.aggs[a].kind != CG_AGG_COUNT_STAR) ? word_identity(P.wordop[P.aggs[a].word0]) : 0;
		acc.w[a][1] = 0;
		acc.w[a][2] = 0;
	}
	uint32_t removed = 0;
	unsigned long long scanned = 0;
	const uint32_t tid = threadIdx.x;

	for (uint32_t ci = blockIdx.x; ci < P.nselected; ci += gridDim.x)
	{
		const DevChunkCol *cc = P.chunkcols + (uint64_t) P.selected[ci] * (uint64_t) P.nstaged;
		const uint8_t *vptr[NCC];
		const uint64_t *bptr[NCC];
		const uint32_t *rptr[NCC];
		uint32_t hasnull = 0;
		uint32_t rows = __ldg(&cc[0].row_count);
#pragma unroll
		for (int c = 0; c < NCC; c++)
		{
			if (c < P.ncols)
			{
				const DevChunkCol *d = cc + P.slot[c];
				vptr[c] = P.arena + __ldg(&d->values_off);
				bptr[c] = (const uint64_t *) (P.arena + __ldg(&d->exists_off));
				rptr[c] = (const uint32_t *) (P.arena + __ldg(&d->rank_off));
				if (__ldg(&d->value_count) != rows) hasnull |= 1u << c;
			}
		}
		scanned += (tid == 0) ? rows : 0;

		if (hasnull == 0)
		{
			for (uint32_t base = 0; base < rows; base += CG_THREADS * 2 * U)
			{
				int64_t v0[U][NCC], v1[U][NCC];
#pragma unroll
				for (int u = 0; u < U; u++)
				{
					uint32_t r = base + (u * CG_THREADS + tid) * 2;
					if (r < rows)
					{
#pragma unroll
						for (int c = 0; c < NCC; c++)
							if (c < P.ncols)
							{
								if (ALL8)
								{
									uint64_t a, b;
									ldg_stream16(vptr[c] + (uint64_t) r * 8, a, b);
									v0[u][c] = (int64_t) a; v1[u][c] = (int64_t) b;
								}
								else
									load_pair(vptr[c], r, P.len[c], P.isfloat[c], v0[u][c], v1[u][c]);
							}
					}
				}
#pragma unroll
				for (int u = 0; u < U; u++)
				{
					uint32_t r = base + (u * CG_THREADS + tid) * 2;
					if (r < rows)
					{
						process_row<NCC, NAC, MODE>(P, v0[u], 0u, acc, removed);
						if (r + 1 < rows) process_row<NCC, NAC, MODE>(P, v1[u], 0u, acc, removed);
					}
				}
			}
		}
		else
		{
			/* chunk group with NULLs: row -> value index through the rank directory
			 * (NULL rows occupy no bytes in the value stream, columnar_reader.c:1550-1555) */
			for (uint32_t r = tid * 2; r < rows; r += CG_THREADS * 2)
			{
				int64_t v0[NCC], v1[NCC];
				uint32_t n0 = 0, n1 = 0;
#pragma unroll
				for (int c = 0; c < NCC; c++)
					if (c < P.ncols)
					{
						int len = ALL8 ? 8 : P.len[c];
						bool isf = P.isfloat[c];
						if ((hasnull >> c) & 1u)
						{
							uint64_t w = ldg_stream8(bptr[c] + (r >> 6));
							uint32_t sh = r & 63u;
							uint32_t before = __ldg(rptr[c] + (r >> 6)) + __popcll(w & ((1ull << sh) - 1ull));
							uint32_t e0 = (uint32_t) (w >> sh) & 1u, e1 = (uint32_t) (w >> (sh + 1)) & 1u;
							v0[c] = e0 ? load_scalar(vptr[c] + (uint64_t) before * len, len, isf) : 0;
							v1[c] = (e1 && r + 1 < rows) ? load_scalar(vptr[c] + (uint64_t) (before + e0) * len, len, isf) : 0;
							n0 |= (e0 ^ 1u) << c;
							n1 |= (e1 ^ 1u) << c;
						}
						else
							load_pair(vptr[c], r, len, isf, v0[c], v1[c]);
					}
				process_row<NCC, NAC, MODE>(P, v0, n0, acc, removed);
				if (r + 1 < rows) process_row<NCC, NAC, MODE>(P, v1, n1, acc, removed);
			}
		}
	}

	/* counters and (plain aggregate) the block's accumulators: warp shuffle reduce, then one
	 * atomic per warp and word */
	unsigned long long rem = warp_reduce_word(removed, CG_WORD_ADD);
	unsigned long long scn = warp_reduce_word(scanned, CG_WORD_ADD);
	if ((tid & 31) == 0)
	{
		if (scn) atomicAdd(P.stats + 0, scn);
		if (rem) atomicAdd(P.stats + 1, rem);
	}
	if (MODE == CG_MODE_GLOBAL)
	{
		uint64_t rows_passed = warp_reduce_word(acc.rows, CG_WORD_ADD);
		if ((tid & 31) == 0 && rows_passed) atomicAdd((unsigned long long *) P.table, (unsigned long long) rows_passed);
#pragma unroll
		for (int a = 0; a < NAC; a++)
		{
			if (a < P.naggs && P.aggs[a].kind != CG_AGG_COUNT_STAR)
			{
				const KAgg &g = P.aggs[a];
				uint64_t nulls = warp_reduce_word(acc.w[a][2], CG_WORD_ADD);
				uint64_t x0 = warp_reduce_word(acc.w[a][0], P.wordop[g.word0]);
				uint64_t x1 = warp_reduce_word(acc.w[a][1], CG_WORD_ADD);
				if ((tid & 31) == 0)
				{
					if (nulls) atomicAdd((unsigned long long *) P.table + g.nullword, (unsigned long long) nulls);
					if (g.kind != CG_AGG_COUNT)
					{
						if (x0 != word_identity(P.wordop[g.word0])) word_apply_global(P.table + g.word0, P.wordop[g.word0], x0);
						if (g.kind == CG_AGG_SUM && !g.is_float && g.nlimbs == 2 && x1)
							atomicAdd((unsigned long long *) P.table + g.word0 + 1, (unsigned long long) x1);
					}
				}
			}
		}
	}
}

template <int NCC, int NAC, int MODE, bool ALL8, int U>
static int launch_variant(CgContext *ctx, const KPlan &plan, cudaStream_t stream)
{
	int occ = 0;
	CG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, cg_scan_kernel<NCC, NAC, MODE, ALL8, U>, CG_THREADS, 0));
	if (occ < 1) occ = 1;
	uint32_t grid = (uint32_t) (ctx->sm_count * occ);
	if (grid > plan.nselected) grid = plan.nselected;
	if (grid == 0) return CG_OK;
	cg_scan_kernel<NCC, NAC, MODE, ALL8, U><<<grid, CG_THREADS, 0, stream>>>(plan);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

template <int NCC, int NAC, int MODE>
static int launch_cols(CgContext *ctx, const KPlan &plan, bool all8, cudaStream_t stream)
{
	constexpr int U = (NCC <= 4) ? 2 : 1;
	if (all8) return launch_variant<NCC, NAC, MODE, true, U>(ctx, plan, stream);
	return launch_variant<NCC, NAC, MODE, false, U>(ctx, plan, stream);
}

template <int NCC>
static int launch_mode(CgContext *ctx, const KPlan &plan, bool all8, cudaStream_t stream)
{
	switch (plan.mode)
	{
		case CG_MODE_GLOBAL:
			if (plan.naggs <= 2) return launch_cols<NCC, 2, CG_MODE_GLOBAL>(ctx, plan, all8, stream);
			return launch_cols<NCC, CG_MAX_AGGS, CG_MODE_GLOBAL>(ctx, plan, all8, stream);
		case CG_MODE_DENSE:
			return launch_cols<NCC, CG_MAX_AGGS, CG_MODE_DENSE>(ctx, plan, all8, stream);
		default:
			return launch_cols<NCC, CG_MAX_AGGS, CG_MODE_HASH>(ctx, plan, all8, stream);
	}
}

int cg_launch_scan(CgContext *ctx, const KPlan &plan, bool any_nulls, bool all8, cudaStream_t stream)
{
	(void) any_nulls;
	if (plan.ncols <= 2) return launch_mode<2>(ctx, plan, all8, stream);
	if (plan.ncols <= 4) return launch_mode<4>(ctx, plan, all8, stream);
	return launch_mode<CG_KMAX_COLS>(ctx, plan, all8, stream);
}

/* ------------------------------------------------------------------------------ *
 *  Rank directory: for every (chunk group, staged column) that has NULLs,
 *  rank[b] = number of set exists bits before row 64*b.  One warp per item.
 *  (the prefix-popcount half of K1; DeserializeDatumArray's running offset)
 * ------------------------------------------------------------------------------ */
__global__ void __launch_bounds__(256)
cg_rank_kernel(const uint8_t *arena, const DevChunkCol *chunkcols, uint64_t first, uint64_t count)
{
	uint64_t item = first + (uint64_t) blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
	if (item >= first + count) return;
	const DevChunkCol d = chunkcols[item];
	if (d.value_count == d.row_count) return;
	const uint64_t *bm = (const uint64_t *) (arena + d.exists_off);
	uint32_t *rank = (uint32_t *) (arena + d.rank_off);
	uint32_t nblocks = (d.row_count + 63) / 64;
	uint32_t lane = threadIdx.x & 31;
	uint32_t running = 0;
	for (uint32_t b0 = 0; b0 < nblocks; b0 += 32)
	{
		uint32_t b = b0 + lane;
		uint32_t pc = (b < nblocks) ? (uint32_t) __popcll(bm[b]) : 0;
		uint32_t incl = pc;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1)
		{
			uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= (uint32_t) o) incl += y;
		}
		if (b < nblocks) rank[b] = running + incl - pc;
		running += __shfl_sync(0xffffffffu, incl, 31);
	}
}

int cg_launch_rank(CgContext *ctx, const uint8_t *arena, const DevChunkCol *chunkcols, uint64_t first,
				   uint64_t count, cudaStream_t stream)
{
	(void) ctx;
	if (count == 0) return CG_OK;
	uint64_t blocks = (count + 7) / 8;
	cg_rank_kernel<<<(unsigned) blocks, 256, 0, stream>>>(arena, chunkcols, first, count);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

/* ------------------------------------------------------------------------------ *
 *  Realign: the copy engine delivers whole 8 KB pages (24-byte header + 8168-byte payload,
 *  columnar_storage.c:21-31) with plain 1-D copies; chunk buffers sit in them at arbitrary
 *  byte offsets (exists bitmaps are ceil(rows/8) bytes long, so value streams are not even
 *  8-byte aligned in the logical byte stream) and run across page headers.  Every block moves
 *  one buffer to its 16-byte aligned arena slot -- the GPU half of ColumnarStorageRead's
 *  de-framing (columnar_storage.c:463-492, ReadFromBlock :669-689) -- with aligned 4-byte loads
 *  + byte permutes, and zero-fills the slot's padding.  Header, payload and page sizes are all
 *  multiples of 4, so an aligned word never straddles a header.
 * ------------------------------------------------------------------------------ */
__global__ void __launch_bounds__(128)
cg_realign_kernel(const uint8_t *raw, uint8_t *arena, const RealignItem *items)
{
	const RealignItem it = items[blockIdx.x];
	const uint32_t mis = (uint32_t) (it.src & 3u);
	const uint64_t w0 = it.src - mis;                                  /* first aligned word (raw offsets of page starts are multiples of 8192) */
	const uint32_t t0 = (uint32_t) (w0 % CG_BLCKSZ) - CG_PAGE_HEADER;    /* its payload coordinate in its page */
	const uint8_t *page0 = raw + (w0 - (w0 % CG_BLCKSZ));
	const uint32_t sel = 0x3210u + 0x1111u * mis;
	uint4 *dst = (uint4 *) (arena + it.dst);
	const uint32_t nvec = it.padded / 16;
	for (uint32_t i = threadIdx.x; i < nvec; i += blockDim.x)
	{
		uint32_t o[4] = {0, 0, 0, 0};
		if (16 * i < it.len)
		{
			uint32_t w[5];
			uint32_t t = t0 + 16 * i;
			uint32_t pg = t / CG_BYTES_PER_PAGE, within = t - pg * CG_BYTES_PER_PAGE;
			const uint8_t *p = page0 + (uint64_t) pg * CG_BLCKSZ + CG_PAGE_HEADER;
#pragma unroll
			for (int k = 0; k < 5; k++)
			{
				w[k] = __ldg((const uint32_t *) (p + within));
				within += 4;
				if (within == CG_BYTES_PER_PAGE) { within = 0; p += CG_BLCKSZ; }
			}
#pragma unroll
			for (int k = 0; k < 4; k++) o[k] = __byte_perm(w[k], w[k + 1], sel);
			if (16 * i + 16 > it.len)
			{
				/* the slot's tail: keep only the bytes that belong to the buffer */
#pragma unroll
				for (int k = 0; k < 4; k++)
				{
					int keep = (int) it.len - (int) (16 * i + 4 * k);
					if (keep <= 0) o[k] = 0;
					else if (keep < 4) o[k] &= (1u << (8 * keep)) - 1u;
				}
			}
		}
		dst[i] = make_uint4(o[0], o[1], o[2], o[3]);
	}
}

/*
 * The same de-framing as a Hopper bulk-copy pipeline.  The raw page span of a chunk buffer is fetched in 8 KB output tiles by
 * the copy unit itself -- cp.async.bulk global -> shared (1-D TMA, SASS UBLKCP), completion counted in bytes on an mbarrier
 * (SYNCS) -- three tiles in flight per CTA, issued by one thread; the other threads never touch global memory for loads: they
 * assemble aligned 16-byte vectors from shared memory (4-byte LDS + byte permutes, page headers skipped as above) and store
 * them.  Against the LDG version this removes five 4-byte global loads per 16 output bytes from the instruction stream.
 */
#define RT_TILE 8192u                       /* output bytes per tile */
#define RT_STAGE (RT_TILE + 128u)           /* raw bytes of a tile: + two page headers + alignment slack, multiple of 16 */
#define RT_STAGES 3
#define RT_THREADS 128

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes),
				 "r"(smem_u32(bar))
				 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
	uint32_t ok;
	do
	{
		asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
	} while (!ok);
}

/* raw offset of payload byte q of a buffer whose first byte sits at raw offset src0, payload coordinate w0 in its page */
__device__ __forceinline__ uint64_t raw_of(uint64_t src0, uint32_t w0, uint32_t q)
{
	return src0 + q + (uint64_t) CG_PAGE_HEADER * ((w0 + q) / CG_BYTES_PER_PAGE);
}

__global__ void __launch_bounds__(RT_THREADS)
cg_realign_tma_kernel(const uint8_t *raw, uint8_t *arena, const RealignItem *items)
{
	__shared__ __align__(128) uint8_t s_raw[RT_STAGES][RT_STAGE];
	__shared__ __align__(8) uint64_t s_bar[RT_STAGES];
	__shared__ uint32_t s_a0[RT_STAGES];                 /* raw offset (relative to the item's 16-byte floor) the stage starts at */
	const RealignItem it = items[blockIdx.x];
	uint4 *dst = (uint4 *) (arena + it.dst);
	const uint32_t nvec = it.padded / 16;
	const uint32_t nvec_data = (it.len + 15) / 16;
	/* the slot's padding behind the data */
	for (uint32_t i = nvec_data + threadIdx.x; i < nvec; i += RT_THREADS) dst[i] = make_uint4(0, 0, 0, 0);
	if (it.len == 0) return;
	const uint32_t mis = (uint32_t) (it.src & 3u);
	const uint32_t w0 = (uint32_t) (it.src % CG_BLCKSZ) - CG_PAGE_HEADER;      /* payload coordinate of the first byte in its page */
	const uint32_t sel = 0x3210u + 0x1111u * mis;
	const uint32_t ntiles = (it.len + RT_TILE - 1) / RT_TILE;
	if (threadIdx.x == 0)
	{
		for (int s = 0; s < RT_STAGES; s++) mbar_init(&s_bar[s], 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	__syncthreads();
	auto issue = [&](uint32_t t) {
		/* raw bytes of output tile t: from the aligned word holding its first byte to the one holding its last */
		const uint32_t q0 = t * RT_TILE, q1 = min(it.len, q0 + RT_TILE);
		const uint32_t nv = (q1 - q0 + 15) / 16;
		const uint64_t r0 = raw_of(it.src - mis, w0 - mis, q0);                 /* first aligned word of the tile */
		const uint64_t r1 = raw_of(it.src - mis, w0 - mis, q0 + 16 * nv) + 4;   /* end of the 5th word of the last vector */
		const uint64_t a0 = r0 & ~15ull;
		const uint32_t bytes = (uint32_t) (((r1 - a0) + 15ull) & ~15ull);
		const int s = (int) (t % RT_STAGES);
		s_a0[s] = (uint32_t) (r0 - a0);
		mbar_expect_tx(&s_bar[s], bytes);
		bulk_g2s(s_raw[s], raw + a0, bytes, &s_bar[s]);
	};
	if (threadIdx.x == 0)
		for (uint32_t t = 0; t < ntiles && t < RT_STAGES; t++) issue(t);
	for (uint32_t t = 0; t < ntiles; t++)
	{
		const int s = (int) (t % RT_STAGES);
		mbar_wait(&s_bar[s], (t / RT_STAGES) & 1u);
		const uint8_t *buf = s_raw[s];
		const uint32_t q0 = t * RT_TILE, q1 = min(it.len, q0 + RT_TILE);
		const uint32_t first = s_a0[s];                                         /* shared-memory offset of the tile's first aligned word */
		const uint32_t tw0 = (w0 - mis + q0) % CG_BYTES_PER_PAGE;               /* ... and its payload coordinate in its page */
		const uint32_t nv = (q1 - q0 + 15) / 16;
		for (uint32_t i = threadIdx.x; i < nv; i += RT_THREADS)
		{
			/* word k of this vector: payload coordinate tw0 + 16 i + 4 k, i.e. shared-memory offset first + 16 i + 4 k + 24 * (pages crossed) */
			uint32_t within = tw0 + 16 * i;
			uint32_t off = first + 16 * i;
			const uint32_t crossed = within / CG_BYTES_PER_PAGE;
			within -= crossed * CG_BYTES_PER_PAGE;
			off += crossed * CG_PAGE_HEADER;
			uint32_t w[5];
#pragma unroll
			for (int k = 0; k < 5; k++)
			{
				w[k] = *(const uint32_t *) (buf + off);
				within += 4; off += 4;
				if (within == CG_BYTES_PER_PAGE) { within = 0; off += CG_PAGE_HEADER; }
			}
			uint32_t o[4];
#pragma unroll
			for (int k = 0; k < 4; k++) o[k] = __byte_perm(w[k], w[k + 1], sel);
			const uint32_t ob = q0 + 16 * i;                                     /* output byte offset of the vector */
			if (ob + 16 > it.len)
			{
#pragma unroll
				for (int k = 0; k < 4; k++)
				{
					int keep = (int) it.len - (int) (ob + 4 * k);
					if (keep <= 0) o[k] = 0;
					else if (keep < 4) o[k] &= (1u << (8 * keep)) - 1u;
				}
			}
			dst[ob / 16] = make_uint4(o[0], o[1], o[2], o[3]);
		}
		__syncthreads();                                                        /* every thread is done with the stage */
		if (threadIdx.x == 0 && t + RT_STAGES < ntiles) issue(t + RT_STAGES);
	}
}

static int g_realign_tma = -1;
void cg_realign_set_tma(int on) { g_realign_tma = on ? 1 : 0; }

int cg_launch_realign(const uint8_t *raw, uint8_t *arena, const RealignItem *items, uint64_t nitems, cudaStream_t stream)
{
	if (nitems == 0) return CG_OK;
	if (g_realign_tma < 0) { const char *e = getenv("CG_REALIGN_TMA"); g_realign_tma = e ? (atoi(e) != 0) : 1; }
	if (g_realign_tma) cg_realign_tma_kernel<<<(unsigned) nitems, RT_THREADS, 0, stream>>>(raw, arena, items);
	else cg_realign_kernel<<<(unsigned) nitems, 128, 0, stream>>>(raw, arena, items);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

/* ------------------------------------------------------------------------------ *
 *  Group table: init, export (compaction), merge (K5 combine).
 * ------------------------------------------------------------------------------ */
struct TableView
{
	int64_t *hkeys;
	uint64_t *table;
	uint64_t capacity;
	uint64_t entries;
	int32_t stride;
	int32_t nwords;
	int32_t mode;
	int64_t key_min;
	int64_t key_min1;
	uint64_t range1;
	int32_t ngroup;
	uint8_t wordop[CG_KMAX_WORDS];
};

static TableView view_of(const CgPartial *p)
{
	TableView v;
	v.hkeys = p->d_hkeys; v.table = p->d_table; v.capacity = p->capacity; v.entries = p->entries; v.stride = p->stride;
	v.nwords = p->nwords; v.mode = p->mode; v.key_min = p->key_min;
	v.key_min1 = p->key_min1; v.range1 = p->range1; v.ngroup = p->desc.ngroup_cols;
	for (int i = 0; i < CG_KMAX_WORDS; i++) v.wordop[i] = p->wordop[i];
	return v;
}

__global__ void cg_table_init_kernel(const __grid_constant__ TableView T)
{
	uint64_t total = T.entries * (uint64_t) T.stride;
	for (uint64_t i = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t) gridDim.x * blockDim.x)
	{
		int w = (int) (i % (uint64_t) T.stride);
		T.table[i] = w < T.nwords ? word_identity(T.wordop[w]) : 0ull;
		if (T.mode == CG_MODE_HASH && w == 0) T.hkeys[i / (uint64_t) T.stride] = CG_HASH_EMPTY;
	}
}

int cg_launch_table_init(CgPartial *p, cudaStream_t stream)
{
	TableView v = view_of(p);
	uint64_t total = v.entries * (uint64_t) v.stride;
	/* a direct-indexed table whose wide words were never written since the last initialisation (packed words only) is
	 * still in its initial state: a reset only clears the packed words and the counters */
	if (!(p->table_initialised && !p->wide_dirty && p->mode != CG_MODE_HASH))
	{
		unsigned blocks = (unsigned) ((total + 255) / 256);
		if (blocks > (unsigned) cg_ctx()->sm_count * 16) blocks = (unsigned) cg_ctx()->sm_count * 16;
		if (blocks == 0) blocks = 1;
		cg_table_init_kernel<<<blocks, 256, 0, stream>>>(v);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
		p->table_initialised = true;
	}
	CG_CUDA(cudaMemsetAsync(p->d_stats, 0, 8 * sizeof(unsigned long long), stream));
	CG_CUDA(cudaMemsetAsync(p->d_table + total, 0, CG_COMM_TAIL * sizeof(uint64_t), stream));
	if (p->d_packed) CG_CUDA(cudaMemsetAsync(p->d_packed, 0, ((size_t) p->entries + CG_COMM_TAIL) * sizeof(uint64_t), stream));
	p->packed_dirty = false;
	p->wide_dirty = false;
	p->read_packed_direct = false;
	p->launches_since_drain = 0;
	p->rows_since_drain = 0;
	return CG_OK;
}

/* place of an occupied entry in the compacted output: ONE atomic per block and iteration (256 consecutive entries).  A
 * per-warp atomic is 31 k same-address atomics for a million groups -- tens of microseconds on one L2 line, more than
 * the kernel's memory traffic.  Every thread of the block calls this the same number of times. */
__device__ __forceinline__ unsigned long long export_position(bool occupied, unsigned long long *count)
{
	__shared__ unsigned int s_warp[32];
	__shared__ unsigned long long s_base;
	const unsigned lane = threadIdx.x & 31u, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31u) >> 5;
	const unsigned m = __ballot_sync(0xffffffffu, occupied);
	if (lane == 0) s_warp[warp] = __popc(m);
	__syncthreads();
	if (threadIdx.x == 0)
	{
		unsigned int total = 0;
		for (unsigned w = 0; w < nwarps; w++) total += s_warp[w];
		s_base = total ? atomicAdd(count, (unsigned long long) total) : 0ull;
	}
	__syncthreads();
	unsigned long long pos = s_base + __popc(m & ((1u << lane) - 1u));
	for (unsigned w = 0; w < warp; w++) pos += s_warp[w];
	__syncthreads();                      /* the next iteration overwrites the shared words */
	return pos;
}

__global__ void cg_export_kernel(const __grid_constant__ TableView T, uint64_t out_capacity, int64_t *keys,
								 uint8_t *nulls, uint64_t *words, unsigned long long *count)
{
	/* every lane of a warp runs the same number of iterations (the warp-wide ballot needs them all) */
	for (uint64_t base = (uint64_t) blockIdx.x * blockDim.x; base < T.entries; base += (uint64_t) gridDim.x * blockDim.x)
	{
		const uint64_t e = base + threadIdx.x;
		const bool valid = e < T.entries;
		const uint64_t *ent = T.table + (valid ? e : 0) * (uint64_t) T.stride;
		bool occupied = false;
		int64_t key = 0;
		bool key_null = false;
		if (!valid) { }
		else if (T.mode == CG_MODE_HASH)
		{
			if (e < T.capacity) { key = T.hkeys[e]; occupied = key != CG_HASH_EMPTY; }
			else { occupied = ent[0] > 0; key_null = (e == T.capacity); key = key_null ? 0 : CG_HASH_EMPTY; }
		}
		else if (T.mode == CG_MODE_DENSE)
		{
			occupied = ent[0] > 0;
			key_null = (e == T.capacity);
			if (key_null) key = 0;
			else if (T.ngroup == 2)
			{
				int64_t k0 = T.key_min + (int64_t) (e / T.range1), k1 = T.key_min1 + (int64_t) (e % T.range1);
				key = (int64_t) ((uint64_t) (uint32_t) k0 | ((uint64_t) (uint32_t) k1 << 32));
			}
			else key = T.key_min + (int64_t) e;
		}
		else
			occupied = true;    /* plain aggregate: exactly one result row, even over no input */
		const unsigned long long pos = export_position(occupied, count);
		if (!occupied || pos >= out_capacity) continue;
		if (keys) keys[pos] = key;
		if (nulls) nulls[pos] = key_null ? 1 : 0;
		if (words)
			for (int w = 0; w < T.nwords; w++) words[pos * (uint64_t) T.nwords + w] = ent[w];
	}
}

int cg_launch_export(CgPartial *p, uint64_t out_capacity, int64_t *d_keys, uint8_t *d_nulls, uint64_t *d_words,
					 unsigned long long *d_count, cudaStream_t stream)
{
	TableView v = view_of(p);
	CG_CUDA(cudaMemsetAsync(d_count, 0, 2 * sizeof(unsigned long long), stream));
	unsigned blocks = (unsigned) ((v.entries + 255) / 256);
	if (blocks > (unsigned) cg_ctx()->sm_count * 16) blocks = (unsigned) cg_ctx()->sm_count * 16;
	if (blocks == 0) blocks = 1;
	cg_export_kernel<<<blocks, 256, 0, stream>>>(v, out_capacity, d_keys, d_nulls, d_words, d_count);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

/*
 * Result rows straight from the packed words of a direct-indexed table whose wide accumulators were never written:
 * word = (sum << C) + n  ->  rows n, sum; every other accumulator word is its identity.  count[0] = groups, count[1] =
 * rows decoded (the overflow check: it must equal the rows the scan kernels added).
 */
__global__ void cg_export_packed_kernel(const __grid_constant__ TableView T, const uint64_t *packed, int shift, int pack_word,
										uint64_t out_capacity, int64_t *keys, uint8_t *nulls, uint64_t *words, unsigned long long *count)
{
	const uint64_t mask = (1ull << shift) - 1ull;
	unsigned long long decoded = 0;
	for (uint64_t base = (uint64_t) blockIdx.x * blockDim.x; base < T.entries; base += (uint64_t) gridDim.x * blockDim.x)
	{
		const uint64_t e = base + threadIdx.x;
		const uint64_t w = e < T.entries ? packed[e] : 0ull;
		const uint64_t n = w & mask;
		const int64_t sum = (int64_t) (w - n) >> shift;
		decoded += n;
		/* n == 0 with w != 0 is only reachable after an overflow, which the caller detects */
		const unsigned long long pos = export_position(n != 0, count);
		if (n == 0 || pos >= out_capacity) continue;
		if (keys) keys[pos] = e == T.capacity ? 0 : T.key_min + (int64_t) e;
		if (nulls) nulls[pos] = e == T.capacity ? 1 : 0;
		if (words)
			for (int x = 0; x < T.nwords; x++)
				words[pos * (uint64_t) T.nwords + x] = x == 0 ? n : x == pack_word ? (uint64_t) sum : word_identity(T.wordop[x]);
	}
	for (int o = 16; o > 0; o >>= 1) decoded += __shfl_xor_sync(0xffffffffu, decoded, o);
	__shared__ unsigned long long s_dec[32];
	if ((threadIdx.x & 31) == 0) s_dec[threadIdx.x >> 5] = decoded;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		unsigned long long t = 0;
		for (unsigned w = 0; w < (blockDim.x + 31u) >> 5; w++) t += s_dec[w];
		if (t) atomicAdd(count + 1, t);
	}
}

int cg_launch_export_packed(CgPartial *p, uint64_t out_capacity, int64_t *d_keys, uint8_t *d_nulls, uint64_t *d_words,
							unsigned long long *d_count, cudaStream_t stream)
{
	TableView v = view_of(p);
	CG_CUDA(cudaMemsetAsync(d_count, 0, 2 * sizeof(unsigned long long), stream));
	unsigned blocks = (unsigned) ((v.entries + 255) / 256);
	if (blocks > (unsigned) cg_ctx()->sm_count * 16) blocks = (unsigned) cg_ctx()->sm_count * 16;
	if (blocks == 0) blocks = 1;
	cg_export_packed_kernel<<<blocks, 256, 0, stream>>>(v, p->d_packed, p->pack_shift, p->pack_word, out_capacity, d_keys, d_nulls, d_words, d_count);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

/* K5: merge partial rows (from other shards / GPUs) into the table, word by word.
 * This is the coordinator's HashAggregate over sum(sum), sum(count), min(min), max(max)
 * (planner/multi_logical_optimizer.c:1807-1885, 2231-2275). */
__global__ void cg_merge_kernel(const __grid_constant__ KPlan P, const int64_t *keys, const uint8_t *nulls,
								const uint64_t *words, int64_t nrows)
{
	/* low words of two-limb sums: a row's low word may hold up to 64 bits of summed low halves; its carry
	 * (bits 32..63) moves to the high word, so the table's low word grows by < 2^32 per merged row */
	uint32_t lo_words = 0;
	for (int a = 0; a < P.naggs; a++)
		if (P.aggs[a].kind == CG_AGG_SUM && !P.aggs[a].is_float && P.aggs[a].nlimbs == 2) lo_words |= 1u << P.aggs[a].word0;
	for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (int64_t) gridDim.x * blockDim.x)
	{
		uint64_t *entry;
		if (P.mode == CG_MODE_GLOBAL) entry = P.table;
		else
		{
			bool kn = nulls ? nulls[i] != 0 : false;
			entry = (P.mode == CG_MODE_DENSE) ? find_entry<CG_MODE_DENSE>(P, keys[i], kn)
											  : find_entry<CG_MODE_HASH>(P, keys[i], kn);
			if (entry == nullptr) continue;
		}
		uint64_t carry = 0;
		for (int w = 0; w < P.nwords; w++)
		{
			uint64_t val = words[i * (int64_t) P.nwords + w];
			if ((lo_words >> w) & 1u) { carry = val >> 32; val &= 0xffffffffull; }
			else if (w > 0 && ((lo_words >> (w - 1)) & 1u)) val += carry;
			if (val != word_identity(P.wordop[w])) word_apply_global(entry + w, P.wordop[w], val);
		}
	}
}

int cg_launch_merge(CgPartial *p, const int64_t *d_keys, const uint8_t *d_nulls, const uint64_t *d_words,
					int64_t nrows, cudaStream_t stream)
{
	if (nrows <= 0) return CG_OK;
	KPlan plan;
	memset(&plan, 0, sizeof plan);
	plan.mode = p->mode; plan.nwords = p->nwords; plan.stride = p->stride; plan.table = p->d_table; plan.hkeys = p->d_hkeys;
	plan.capacity = p->capacity; plan.key_min = p->key_min; plan.stats = p->d_stats;
	plan.key_min1 = p->key_min1; plan.range1 = p->range1; plan.ngroup = p->desc.ngroup_cols;
	plan.hash_shift = 64;
	for (uint64_t c = p->capacity; c > 1; c >>= 1) plan.hash_shift--;
	for (int i = 0; i < CG_KMAX_WORDS; i++) plan.wordop[i] = p->wordop[i];
	plan.naggs = p->desc.naggs;
	for (int a = 0; a < p->desc.naggs; a++) plan.aggs[a] = p->aggs[a];
	unsigned blocks = (unsigned) ((nrows + 255) / 256);
	if (blocks > (unsigned) cg_ctx()->sm_count * 8) blocks = (unsigned) cg_ctx()->sm_count * 8;
	cg_merge_kernel<<<blocks, 256, 0, stream>>>(plan, d_keys, d_nulls, d_words, nrows);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	p->wide_dirty = true;
	return CG_OK;
}
