/*
 * cg_narrow.cu -- narrow images of staged 8-byte integer columns (DevPackCol, cg_internal.h).
 *
 * The arena keeps every value at its on-disk width, 8 bytes, whatever range the column spans.  The fast kernel is bound
 * by the bytes it streams from HBM and the group-table reductions it issues, which share the memory system, so fewer
 * column bytes leave more of it to the reductions.  cg_shard_stage therefore builds, once per shard and outside every
 * scan, a frame-of-reference bit-packed copy of each chunk column that fits 32 bits: an exact min / max reduction on the
 * GPU, the layout on the host (cg_narrow_plan), then one pass that packs the values.  The plain arena stays as it is:
 * every other kernel, and the chunk groups with NULLs, read it.
 */
#include "cg_internal.h"

#include <algorithm>
#include <vector>

/* device memory left free after the images: they are a speed-up and must not take what later allocations need */
#define CG_NARROW_HEADROOM (2ull << 30)

struct NarrowItem   /* one NULL-free (chunk group, candidate column) */
{
	uint64_t values_off;   /* arena: values */
	uint64_t out_off;      /* d_narrow: bit stream */
	int64_t base;
	uint32_t rows;
	uint32_t width;
};

/* exact minimum and maximum of each item's values (signed int64), one CTA per item */
__global__ void __launch_bounds__(256)
cg_narrow_minmax_kernel(const uint8_t *arena, const NarrowItem *items, uint64_t nitems, int64_t *mm)
{
	__shared__ int64_t smin[8], smax[8];
	for (uint64_t i = blockIdx.x; i < nitems; i += gridDim.x)
	{
		const NarrowItem it = items[i];
		const int64_t *v = (const int64_t *) (arena + it.values_off);
		int64_t lo = INT64_MAX, hi = INT64_MIN;
		for (uint32_t r = threadIdx.x; r < it.rows; r += blockDim.x)
		{
			int64_t x = v[r];
			lo = min(lo, x);
			hi = max(hi, x);
		}
#pragma unroll
		for (int o = 16; o > 0; o >>= 1)
		{
			lo = min(lo, (int64_t) __shfl_xor_sync(0xffffffffu, (long long) lo, o));
			hi = max(hi, (int64_t) __shfl_xor_sync(0xffffffffu, (long long) hi, o));
		}
		if ((threadIdx.x & 31) == 0) { smin[threadIdx.x >> 5] = lo; smax[threadIdx.x >> 5] = hi; }
		__syncthreads();
		if (threadIdx.x == 0)
		{
			for (int w = 1; w < (int) (blockDim.x >> 5); w++) { lo = min(lo, smin[w]); hi = max(hi, smax[w]); }
			mm[2 * i] = lo;
			mm[2 * i + 1] = hi;
		}
		__syncthreads();
	}
}

/* the bit streams: one thread per output word ORs in the fields of the rows that touch it */
__global__ void __launch_bounds__(256)
cg_narrow_pack_kernel(const uint8_t *arena, const NarrowItem *items, uint64_t nitems, uint8_t *out)
{
	for (uint64_t i = blockIdx.x; i < nitems; i += gridDim.x)
	{
		const NarrowItem it = items[i];
		const int64_t *v = (const int64_t *) (arena + it.values_off);
		uint64_t *dst = (uint64_t *) (out + it.out_off);
		const uint32_t w = it.width;
		const uint64_t nwords = cg_narrow_words(it.rows, w);
		for (uint64_t k = threadIdx.x; k < nwords; k += blockDim.x)
		{
			const uint64_t bit0 = k * 64;
			uint64_t r = bit0 / w;                               /* first row whose field reaches into word k */
			uint64_t rend = (bit0 + 63) / w + 1;                 /* past the last row that starts in word k */
			if (rend > it.rows) rend = it.rows;
			uint64_t word = 0;
			for (; r < rend; r++)
			{
				const uint64_t field = (uint64_t) v[r] - (uint64_t) it.base;     /* < 2^w */
				const int64_t pos = (int64_t) (r * w) - (int64_t) bit0;
				word |= pos >= 0 ? field << pos : field >> -pos;
			}
			dst[k] = word;
		}
	}
}

static uint32_t bits_of(uint64_t x)
{
	uint32_t b = 0;
	while (x) { b++; x >>= 1; }
	return b;
}

extern "C" int cg_narrow_plan(int64_t ncg, int32_t ncols, const uint8_t *candidate, const uint32_t *rows, const uint8_t *nullfree,
							  const int64_t *mins, const int64_t *maxs, uint8_t *col_narrow, uint8_t *widths, int64_t *bases,
							  uint64_t *offs, uint64_t *total_bytes)
{
	if (ncg < 0 || ncols < 0 || (ncols > 0 && (!candidate || !col_narrow)) ||
		(ncg > 0 && ncols > 0 && (!rows || !nullfree || !mins || !maxs || !widths || !bases || !offs)) || !total_bytes)
		return cg_set_error(CG_EINVAL, "cg_narrow_plan: bad arguments");
	for (int32_t c = 0; c < ncols; c++)
	{
		bool ok = candidate[c] != 0;
		for (int64_t g = 0; ok && g < ncg; g++)
		{
			const int64_t i = g * ncols + c;
			if (nullfree[i] && (uint64_t) maxs[i] - (uint64_t) mins[i] > (uint64_t) UINT32_MAX) ok = false;
		}
		col_narrow[c] = ok ? 1 : 0;
	}
	uint64_t off = 0;
	for (int64_t g = 0; g < ncg; g++)
		for (int32_t c = 0; c < ncols; c++)
		{
			const int64_t i = g * ncols + c;
			widths[i] = (uint8_t) CG_NARROW_NONE;
			bases[i] = 0;
			offs[i] = 0;
			if (!col_narrow[c] || !nullfree[i]) continue;
			const uint32_t w = bits_of((uint64_t) maxs[i] - (uint64_t) mins[i]);
			widths[i] = (uint8_t) w;
			bases[i] = mins[i];
			offs[i] = off;
			off += (cg_narrow_words(rows[g], w) * 8 + 15) & ~15ull;
		}
	*total_bytes = off;
	return CG_OK;
}

extern "C" uint64_t cg_shard_narrow_bytes(const CgShard *sh) { return sh ? sh->narrow_bytes : 0; }

extern "C" int32_t cg_shard_narrow_column(const CgShard *sh, int32_t att)
{
	if (!sh || att < 0 || att >= sh->natts || sh->slot_of_att[att] < 0 || sh->slot_narrow.empty()) return 0;
	return sh->slot_narrow[sh->slot_of_att[att]];
}

extern "C" int cg_shard_narrow_image(const CgShard *sh, int64_t cg, int32_t att, int64_t *base, uint32_t *width, void *host_buf,
									 uint64_t capacity, uint64_t *nbytes)
{
	if (!sh || !base || !width || !nbytes || cg < 0 || (uint64_t) cg >= sh->nchunkgroups || att < 0 || att >= sh->natts ||
		sh->slot_of_att[att] < 0)
		return cg_set_error(CG_EINVAL, "cg_shard_narrow_image: bad arguments");
	*base = 0;
	*width = CG_NARROW_NONE;
	*nbytes = 0;
	if (sh->h_packcols.empty()) return CG_OK;
	const DevPackCol &pc = sh->h_packcols[(uint64_t) cg * sh->staged.size() + sh->slot_of_att[att]];
	if (pc.width == CG_NARROW_NONE) return CG_OK;
	const uint64_t n = cg_narrow_words(sh->cg_rows[cg], pc.width) * 8;
	if (host_buf && capacity < n)
		return cg_set_error(CG_EINVAL, "cg_shard_narrow_image: the image takes %llu bytes", (unsigned long long) n);
	if (host_buf && n > 0)
	{
		/* the images are written once, at staging, and only read after it: no scan in flight can change them */
		CgContext *ctx = cg_ctx();
		if (!ctx) return CG_EINVAL;
		int rc = cg_chain_end(ctx, ctx->compute);
		if (rc) return rc;
		CG_CUDA(cudaMemcpyAsync(host_buf, sh->d_narrow + pc.off, n, cudaMemcpyDeviceToHost, ctx->compute));
		CG_CUDA(cudaStreamSynchronize(ctx->compute));
	}
	*base = pc.base;
	*width = pc.width;
	*nbytes = n;
	return CG_OK;
}

/* frees what a failed build allocated and clears the CUDA error it left, so that the shard stays exactly as staged */
static void narrow_abandon(CgShard *sh, NarrowItem *d_items, int64_t *d_mm)
{
	cudaStreamSynchronize(cg_ctx()->compute);
	cudaFree(d_items);
	cudaFree(d_mm);
	cudaFree(sh->d_narrow);
	cudaFree(sh->d_packcols);
	cudaGetLastError();
	sh->d_narrow = nullptr;
	sh->d_packcols = nullptr;
	sh->narrow_bytes = 0;
	sh->h_packcols.clear();
	sh->slot_narrow.clear();
}

void cg_shard_build_narrow(CgContext *ctx, CgShard *sh)
{
	const size_t ns = sh->staged.size();
	const uint64_t ncg = sh->nchunkgroups;
	if (ns == 0 || ncg == 0) return;
	std::vector<uint8_t> candidate(ns, 0);
	bool any = false;
	for (size_t j = 0; j < ns; j++)
	{
		const CgColumnDesc &cd = sh->columns[sh->staged[j]];
		candidate[j] = cd.attlen == 8 && cg_type_class(cd) == CG_TYPE_INT;
		any |= candidate[j] != 0;
	}
	if (!any) return;
	/* the NULL-free chunk columns of the candidates */
	std::vector<uint8_t> nullfree(ncg * ns, 0);
	std::vector<NarrowItem> items;
	std::vector<uint64_t> item_of(ncg * ns, ~0ull);
	for (uint64_t g = 0; g < ncg; g++)
		for (size_t j = 0; j < ns; j++)
		{
			const DevChunkCol &d = sh->h_chunkcols[g * ns + j];
			if (!candidate[j] || d.value_count != d.row_count || d.row_count == 0) continue;
			nullfree[g * ns + j] = 1;
			item_of[g * ns + j] = items.size();
			NarrowItem it = {};
			it.values_off = d.values_off;
			it.rows = d.row_count;
			items.push_back(it);
		}
	if (items.empty()) return;

	NarrowItem *d_items = nullptr;
	int64_t *d_mm = nullptr;
	const unsigned grid = (unsigned) std::min<uint64_t>(items.size(), (uint64_t) ctx->sm_count * 8);
	if (cg_chain_end(ctx, ctx->compute) != CG_OK ||
		cudaMalloc(&d_items, items.size() * sizeof(NarrowItem)) != cudaSuccess ||
		cudaMalloc(&d_mm, items.size() * 2 * sizeof(int64_t)) != cudaSuccess ||
		cudaMemcpyAsync(d_items, items.data(), items.size() * sizeof(NarrowItem), cudaMemcpyHostToDevice, ctx->compute) != cudaSuccess)
	{
		narrow_abandon(sh, d_items, d_mm);
		return;
	}
	cg_narrow_minmax_kernel<<<grid, 256, 0, ctx->compute>>>(sh->d_arena, d_items, items.size(), d_mm);
	g_cg_launches++;
	std::vector<int64_t> mm(items.size() * 2);
	if (cudaGetLastError() != cudaSuccess ||
		cudaMemcpyAsync(mm.data(), d_mm, mm.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, ctx->compute) != cudaSuccess ||
		cudaStreamSynchronize(ctx->compute) != cudaSuccess)
	{
		narrow_abandon(sh, d_items, d_mm);
		return;
	}

	std::vector<int64_t> mins(ncg * ns, 0), maxs(ncg * ns, 0), bases(ncg * ns);
	std::vector<uint8_t> widths(ncg * ns), col_narrow(ns);
	std::vector<uint64_t> offs(ncg * ns);
	for (uint64_t i = 0; i < ncg * ns; i++)
		if (item_of[i] != ~0ull) { mins[i] = mm[2 * item_of[i]]; maxs[i] = mm[2 * item_of[i] + 1]; }
	uint64_t total = 0;
	if (cg_narrow_plan((int64_t) ncg, (int32_t) ns, candidate.data(), sh->cg_rows.data(), nullfree.data(), mins.data(), maxs.data(),
					   col_narrow.data(), widths.data(), bases.data(), offs.data(), &total) != CG_OK ||
		std::find(col_narrow.begin(), col_narrow.end(), 1) == col_narrow.end())
	{
		narrow_abandon(sh, d_items, d_mm);
		return;
	}
	size_t free_b = 0, total_b = 0;
	const uint64_t want = std::max<uint64_t>(total, 16) + ncg * ns * sizeof(DevPackCol);
	/* the fast kernel addresses the streams by a 32-bit word index */
	if (total / 8 > UINT32_MAX ||
		cudaMemGetInfo(&free_b, &total_b) != cudaSuccess || (uint64_t) free_b < want + CG_NARROW_HEADROOM)
	{
		narrow_abandon(sh, d_items, d_mm);
		return;
	}
	/* the items of the columns with images, with their streams */
	std::vector<NarrowItem> pack;
	sh->h_packcols.assign(ncg * ns, DevPackCol{0, 0, CG_NARROW_NONE, 0});
	for (uint64_t i = 0; i < ncg * ns; i++)
	{
		if (widths[i] == (uint8_t) CG_NARROW_NONE) continue;
		DevPackCol &pc = sh->h_packcols[i];
		pc.off = offs[i]; pc.base = bases[i]; pc.width = widths[i];
		NarrowItem it = items[item_of[i]];
		it.out_off = offs[i]; it.base = bases[i]; it.width = widths[i];
		if (it.width > 0) pack.push_back(it);
	}
	sh->slot_narrow = col_narrow;
	if (cudaMalloc(&sh->d_narrow, std::max<uint64_t>(total, 16)) != cudaSuccess ||
		cudaMalloc(&sh->d_packcols, ncg * ns * sizeof(DevPackCol)) != cudaSuccess ||
		cudaMemcpyAsync(sh->d_packcols, sh->h_packcols.data(), ncg * ns * sizeof(DevPackCol), cudaMemcpyHostToDevice, ctx->compute) != cudaSuccess ||
		(!pack.empty() && cudaMemcpyAsync(d_items, pack.data(), pack.size() * sizeof(NarrowItem), cudaMemcpyHostToDevice, ctx->compute) != cudaSuccess))
	{
		narrow_abandon(sh, d_items, d_mm);
		return;
	}
	if (!pack.empty())
	{
		const unsigned pgrid = (unsigned) std::min<uint64_t>(pack.size(), (uint64_t) ctx->sm_count * 8);
		cg_narrow_pack_kernel<<<pgrid, 256, 0, ctx->compute>>>(sh->d_arena, d_items, pack.size(), sh->d_narrow);
		g_cg_launches++;
	}
	if (cudaGetLastError() != cudaSuccess || cudaStreamSynchronize(ctx->compute) != cudaSuccess)
	{
		narrow_abandon(sh, d_items, d_mm);
		return;
	}
	cudaFree(d_items);
	cudaFree(d_mm);
	sh->narrow_bytes = total + ncg * ns * sizeof(DevPackCol);
}
