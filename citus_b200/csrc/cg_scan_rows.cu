/*
 * cg_scan_rows.cu -- the row-emitting scan of a staged shard (cg_scan_shard_rows, sm_90a):
 *
 *     SELECT atts FROM shard WHERE <tree>          in the shard's row order
 *
 * which is the filter query of a repartition join's map task (worker_partition_query_result runs it through
 * ColumnarScan into PartitionedResultDestReceiver, executor/partitioned_intermediate_results.c:115-298).  The rows come
 * out as device columns in the decoded form the routing, COPY, exchange and join calls take (CgJoinSide).
 *
 * The host cuts the chunk groups that survive skipping into tiles of CG_ROW_TILE rows, in shard order, and gives every
 * chunk group its run of bitmap words.  Two passes, with the block-offset scan of the repartition path between them:
 *   select  one CTA per tile reads the WHERE columns only and evaluates the tree (eval_where, the row path of the scan
 *           kernels); warp w of a step owns 64 consecutive rows, so its two ballots are one bitmap word.  The tile's
 *           count of passing rows goes to counts[t].
 *   offsets partition_scan_blocks with one partition: counts[t] becomes the first output row of tile t.
 *   write   one CTA per tile turns its bitmap words into ranks (a prefix over the tile's 32 words in shared memory, a
 *           popcount below the lane inside a word) and reads the projected columns of the passing rows only.
 * WHERE columns are read once, projected columns once, the bitmap one bit per row each way.
 */
#include "cg_internal.h"
#include "cg_device.cuh"

#define CGR_THREADS 256
#define CGR_WARPS (CGR_THREADS / 32)
#define CGR_TILE_WORDS (CG_ROW_TILE / 64)

/* the 32 bits of x on the even bits of a 64-bit word */
__device__ __forceinline__ uint64_t spread_even(uint32_t x)
{
	uint64_t v = x;
	v = (v | (v << 16)) & 0x0000ffff0000ffffull;
	v = (v | (v << 8)) & 0x00ff00ff00ff00ffull;
	v = (v | (v << 4)) & 0x0f0f0f0f0f0f0f0full;
	v = (v | (v << 2)) & 0x3333333333333333ull;
	v = (v | (v << 1)) & 0x5555555555555555ull;
	return v;
}

/* NCC: capacity of the per-thread column register file (WHERE plan columns <= NCC); the wider forms hold two rows of
 * NCC values per thread and run fewer CTAs per SM, so that none spills */
template <int NCC>
__global__ void __launch_bounds__(CGR_THREADS, NCC <= 2 ? 4 : NCC <= 4 ? 3 : 2)
cg_rows_select_kernel(const __grid_constant__ KPlan P, const RowTile *tiles, uint64_t *bitmap, unsigned long long *counts)
{
	__shared__ unsigned int s_cnt[CGR_WARPS];
	const RowTile t = tiles[blockIdx.x];
	const DevChunkCol *cc = P.chunkcols + (uint64_t) t.cg * (uint64_t) P.nstaged;
	const uint32_t cg_rows = __ldg(&cc[0].row_count);
	const uint32_t rows = min(cg_rows - t.row0, (uint32_t) CG_ROW_TILE);
	const uint8_t *vptr[NCC];
	const uint64_t *bptr[NCC];
	const uint32_t *rptr[NCC];
	uint32_t hasnull = 0;
#pragma unroll
	for (int c = 0; c < NCC; c++)
	{
		if (c < P.ncols)
		{
			const DevChunkCol *d = cc + P.slot[c];
			vptr[c] = P.arena + __ldg(&d->values_off);
			bptr[c] = (const uint64_t *) (P.arena + __ldg(&d->exists_off));
			rptr[c] = (const uint32_t *) (P.arena + __ldg(&d->rank_off));
			if (__ldg(&d->value_count) != cg_rows) hasnull |= 1u << c;
		}
	}
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	unsigned int cnt = 0;
	for (uint32_t w = warp; w * 64u < rows; w += CGR_WARPS)        /* warp-uniform */
	{
		const uint32_t rl = w * 64u + lane * 2u;                     /* row in the tile */
		const uint32_t r = t.row0 + rl;                              /* row in the chunk group */
		bool p0 = false, p1 = false;
		if (rl < rows)
		{
			int64_t v0[NCC], v1[NCC];
			uint32_t n0 = 0, n1 = 0;
#pragma unroll
			for (int c = 0; c < NCC; c++)
				if (c < P.ncols)
				{
					if ((hasnull >> c) & 1u)
						load_pair_nullable(vptr[c], bptr[c], rptr[c], r, cg_rows, P.len[c], P.isfloat[c], c, v0[c], v1[c], n0, n1);
					else
						load_pair(vptr[c], r, P.len[c], P.isfloat[c], v0[c], v1[c]);
				}
			p0 = eval_where<NCC>(P, v0, n0);
			p1 = rl + 1u < rows && eval_where<NCC>(P, v1, n1);
		}
		const uint32_t b0 = __ballot_sync(0xffffffffu, p0), b1 = __ballot_sync(0xffffffffu, p1);
		if (lane == 0) bitmap[t.word + w] = spread_even(b0) | (spread_even(b1) << 1);
		cnt += (unsigned int) (__popc(b0) + __popc(b1));
	}
	if (lane == 0) s_cnt[warp] = cnt;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		unsigned long long n = 0;
		for (int i = 0; i < CGR_WARPS; i++) n += s_cnt[i];
		counts[blockIdx.x] = n;
	}
}

__global__ void __launch_bounds__(CGR_THREADS, 4)
cg_rows_write_kernel(const __grid_constant__ KRowOut O, const RowTile *tiles, const uint64_t *bitmap, const unsigned long long *offsets)
{
	__shared__ uint32_t s_pre[CGR_TILE_WORDS];
	const RowTile t = tiles[blockIdx.x];
	const DevChunkCol *cc = O.chunkcols + (uint64_t) t.cg * (uint64_t) O.nstaged;
	const uint32_t cg_rows = __ldg(&cc[0].row_count);
	const uint32_t rows = min(cg_rows - t.row0, (uint32_t) CG_ROW_TILE);
	const uint32_t nw = (rows + 63u) / 64u;
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	if (warp == 0)
	{
		/* passing rows of the tile before each of its words */
		const uint32_t n = lane < nw ? (uint32_t) __popcll(bitmap[t.word + lane]) : 0u;
		uint32_t incl = n;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1)
		{
			const uint32_t y = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= (uint32_t) o) incl += y;
		}
		s_pre[lane] = incl - n;
	}
	__syncthreads();
	const unsigned long long base = offsets[blockIdx.x];
	for (uint32_t w = warp; w < nw; w += CGR_WARPS)
	{
		const uint64_t word = bitmap[t.word + w];
		const uint32_t sh = lane * 2u;
		const uint32_t e0 = (uint32_t) (word >> sh) & 1u, e1 = (uint32_t) (word >> (sh + 1u)) & 1u;
		if (!(e0 | e1)) continue;
		const unsigned long long pos = base + s_pre[w] + (unsigned long long) __popcll(word & ((1ull << sh) - 1ull));
		const uint32_t r = t.row0 + w * 64u + sh;
#pragma unroll 1
		for (int c = 0; c < O.ncols; c++)
		{
			const DevChunkCol *d = cc + O.slot[c];
			const uint8_t *vals = O.arena + __ldg(&d->values_off);
			int64_t v0, v1;
			uint32_t n0 = 0, n1 = 0;
			if (__ldg(&d->value_count) != cg_rows)
				load_pair_nullable(vals, (const uint64_t *) (O.arena + __ldg(&d->exists_off)), (const uint32_t *) (O.arena + __ldg(&d->rank_off)),
								   r, cg_rows, O.len[c], O.isfloat[c], 0, v0, v1, n0, n1);
			else
				load_pair(vals, r, O.len[c], O.isfloat[c], v0, v1);
			int64_t *col = O.cols[c];
			uint8_t *nul = O.nulls[c];
			if (e0)
			{
				col[pos] = v0;
				if (nul) nul[pos] = (uint8_t) n0;
			}
			if (e1)
			{
				col[pos + e0] = v1;
				if (nul) nul[pos + e0] = (uint8_t) n1;
			}
		}
	}
}

int cg_launch_rows_select(CgContext *ctx, const KPlan &plan, const RowTile *tiles, int64_t ntiles, uint64_t *bitmap,
						  unsigned long long *counts, cudaStream_t stream)
{
	(void) ctx;
	if (ntiles <= 0) return CG_OK;
	if (ntiles > 0x7fffffff) return cg_set_error(CG_EUNSUPPORTED, "%lld row tiles in one shard", (long long) ntiles);
	const unsigned grid = (unsigned) ntiles;
	if (plan.ncols <= 2) cg_rows_select_kernel<2><<<grid, CGR_THREADS, 0, stream>>>(plan, tiles, bitmap, counts);
	else if (plan.ncols <= 4) cg_rows_select_kernel<4><<<grid, CGR_THREADS, 0, stream>>>(plan, tiles, bitmap, counts);
	else cg_rows_select_kernel<CG_KMAX_COLS><<<grid, CGR_THREADS, 0, stream>>>(plan, tiles, bitmap, counts);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

int cg_launch_rows_write(CgContext *ctx, const KRowOut &out, const RowTile *tiles, int64_t ntiles, const uint64_t *bitmap,
						 const unsigned long long *offsets, cudaStream_t stream)
{
	(void) ctx;
	if (ntiles <= 0) return CG_OK;
	if (ntiles > 0x7fffffff) return cg_set_error(CG_EUNSUPPORTED, "%lld row tiles in one shard", (long long) ntiles);
	cg_rows_write_kernel<<<(unsigned) ntiles, CGR_THREADS, 0, stream>>>(out, tiles, bitmap, offsets);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}
