/*
 * cg_values.cu -- SQL-level values in and out of the device-side aggregate state, for callers that hold rows
 * rather than shards:
 *   cg_partial_merge_values   the inverse of cg_partial_fetch: partial-aggregate ROWS (group key, per aggregate the
 *                             128-bit sum / count / min-max / float sum) are folded into a CgPartial.  This is what
 *                             the coordinator's TupleDestination does with the per-shard result rows it receives
 *                             (executor/adaptive_executor.c:3964-4189 -> tuple_destination.c:97) instead of storing
 *                             them for a CPU HashAggregate: the combine of planner/multi_logical_optimizer.c:
 *                             1807-1885, 2231-2275 runs in cg_merge_kernel.
 *   cg_agg_column             one aggregate over one host column in a single pass: the device half of the
 *                             worker_partial_agg / coord_combine_agg shims (utils/aggregate_utils.c:501-607,
 *                             820-1003 call the wrapped aggregate's sfunc / combinefunc once per row; the shims
 *                             batch the rows of name-matched built-ins and reduce the batch here).
 */
#include <vector>

#include "cg_device.cuh"

extern "C" int cg_partial_merge_values(CgPartial *p, int64_t nrows, const int64_t *keys, const uint8_t *key_nulls,
									   const int64_t *sum_hi, const uint64_t *sum_lo, const int64_t *count, const int64_t *minmax,
									   const double *fsum)
{
	CgContext *ctx = cg_ctx();
	if (!ctx || !p) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	for (int a = 0; a < p->desc.naggs; a++)
		if (p->aggs[a].kind == CG_AGG_VARIANCE)
			return cg_set_error(CG_EUNSUPPORTED, "aggregate %d: a variance state has no sum(x^2) among the host rows (merge its words with cg_partial_merge_rows)", a);
	if (nrows < 0) return cg_set_error(CG_EINVAL, "negative row count");
	if (nrows == 0) return CG_OK;
	const int na = p->desc.naggs, nw = p->nwords;
	if (p->mode != CG_MODE_GLOBAL && !keys) return cg_set_error(CG_EINVAL, "NULL keys");
	if (!count) return cg_set_error(CG_EINVAL, "NULL count array");
	std::vector<int64_t> hk((size_t) nrows);
	std::vector<uint8_t> hn((size_t) nrows);
	std::vector<uint64_t> hw((size_t) nrows * nw);
	for (int64_t i = 0; i < nrows; i++)
	{
		hk[i] = keys ? keys[i] : 0;
		hn[i] = key_nulls ? key_nulls[i] : 0;
		if (hn[i] && p->desc.composite_key)
			return cg_set_error(CG_EINVAL, "partial row %lld: NULL key flag on a composite partial (its codes encode NULLs)", (long long) i);
		uint64_t *w = &hw[(size_t) i * nw];
		for (int x = 0; x < nw; x++) w[x] = word_identity(p->wordop[x]);
		/* rows in the group: count(*) when the query has one, else the largest non-NULL input count (at least 1, so
		 * that a group whose aggregates all saw only NULLs still exists); NULL-input counters are rows - count */
		int64_t rows = 1;
		bool exact = false;
		for (int a = 0; a < na && !exact; a++)
		{
			/* a filtered count(*) is one more candidate, not the group's row count */
			if (p->aggs[a].kind == CG_AGG_COUNT_STAR && !p->aggs[a].filt) { rows = count[i * na + a]; exact = true; }
			else if (count[i * na + a] > rows) rows = count[i * na + a];
		}
		if (rows < 0) return cg_set_error(CG_EINVAL, "negative count in partial row %lld", (long long) i);
		w[0] = (uint64_t) rows;
		for (int a = 0; a < na; a++)
		{
			const KAgg &k = p->aggs[a];
			const int64_t c = count[i * na + a];
			if (k.kind == CG_AGG_COUNT_STAR && !k.filt) continue;
			if (c < 0 || c > rows) return cg_set_error(CG_EINVAL, "count of aggregate %d exceeds the group's rows in partial row %lld", a, (long long) i);
			w[k.nullword] = (uint64_t) (rows - c);
			if (k.kind == CG_AGG_COUNT_STAR || k.kind == CG_AGG_COUNT || c == 0) continue;
			if (k.kind == CG_AGG_SUM)
			{
				if (k.is_float)
				{
					if (!fsum) return cg_set_error(CG_EINVAL, "NULL fsum array");
					memcpy(&w[k.word0], &fsum[i * na + a], 8);
				}
				else
				{
					if (!sum_lo || !sum_hi) return cg_set_error(CG_EINVAL, "NULL sum arrays");
					__int128 s = ((__int128) sum_hi[i * na + a] << 64) | (__int128) (unsigned __int128) sum_lo[i * na + a];
					if (k.nlimbs == 1)
					{
						if (s > (__int128) INT64_MAX || s < (__int128) INT64_MIN)
							return cg_set_error(CG_EINVAL, "partial sum of aggregate %d does not fit the table's single-word accumulator", a);
						w[k.word0] = (uint64_t) (int64_t) s;
					}
					else
					{
						/* (low 32 bits unsigned, the rest signed): the same value as any other limb pair with this sum */
						w[k.word0] = (uint64_t) (uint32_t) (uint64_t) s;
						__int128 hi = s >> 32;
						if (hi > (__int128) INT64_MAX || hi < (__int128) INT64_MIN)
							return cg_set_error(CG_EINVAL, "partial sum of aggregate %d exceeds 96 bits", a);
						w[k.word0 + 1] = (uint64_t) (int64_t) hi;
					}
				}
			}
			else if (cg_kind_is_bool(k.kind))
			{
				if (!minmax) return cg_set_error(CG_EINVAL, "NULL minmax array");
				if (minmax[i * na + a] != 0 && minmax[i * na + a] != 1)
					return cg_set_error(CG_EINVAL, "bool_and / bool_or value %lld in partial row %lld", (long long) minmax[i * na + a], (long long) i);
				w[k.word0] = minmax[i * na + a] ? ~0ull : 0ull;
			}
			else
			{
				/* min / max, and bit_and / bit_or (sign-extended values) */
				if (!minmax) return cg_set_error(CG_EINVAL, "NULL minmax array");
				uint64_t u = (uint64_t) minmax[i * na + a];
				if (k.is_float) u = f8_ordered((int64_t) u);     /* order-preserving encoding of the words */
				w[k.word0] = u;
			}
		}
	}
	const size_t kb = ((size_t) nrows * 8 + 15) & ~(size_t) 15, nb = ((size_t) nrows + 15) & ~(size_t) 15, wb = (size_t) nrows * nw * 8;
	CgAsyncBuf buf;
	CG_CUDA(buf.alloc(kb + nb + wb, ctx->compute));
	uint8_t *d = buf.as<uint8_t>();
	CG_CUDA(cudaMemcpyAsync(d, hk.data(), (size_t) nrows * 8, cudaMemcpyHostToDevice, ctx->compute));
	CG_CUDA(cudaMemcpyAsync(d + kb, hn.data(), (size_t) nrows, cudaMemcpyHostToDevice, ctx->compute));
	CG_CUDA(cudaMemcpyAsync(d + kb + nb, hw.data(), wb, cudaMemcpyHostToDevice, ctx->compute));
	int rc = cg_launch_merge(p, (const int64_t *) d, d + kb, (const uint64_t *) (d + kb + nb), nrows, ctx->compute);
	if (rc) return rc;
	CG_CUDA(cudaStreamSynchronize(ctx->compute));          /* the host vectors go out of scope */
	return cg_partial_check(p);
}

/* ---------------------------------------------------------------------------------- */
struct ColAggOut
{
	unsigned long long count;      /* non-NULL inputs */
	unsigned long long lo;         /* sum of the low 32 bits */
	long long hi;                  /* sum of value >> 32 */
	long long imin, imax;
	unsigned long long fmin, fmax; /* order-preserving float encodings */
};

__global__ void __launch_bounds__(256)
cg_agg_column_kernel(const uint8_t *values, const uint8_t *isnull, long long n, int attlen, int is_float, ColAggOut *out)
{
	unsigned long long cnt = 0, lo = 0, fmin = ~0ull, fmax = 0;
	long long hi = 0, imin = INT64_MAX, imax = INT64_MIN;
	for (long long i = (long long) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long) gridDim.x * blockDim.x)
	{
		if (isnull && isnull[i]) continue;
		int64_t v = load_scalar(values + i * attlen, attlen, is_float != 0);
		cnt++;
		if (is_float)
		{
			uint64_t o = f8_ordered(v);
			fmin = o < fmin ? o : fmin; fmax = o > fmax ? o : fmax;
		}
		else
		{
			lo += (uint64_t) (uint32_t) v; hi += v >> 32;
			imin = v < imin ? v : imin; imax = v > imax ? v : imax;
		}
	}
	for (int o = 16; o > 0; o >>= 1)
	{
		cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
		lo += __shfl_xor_sync(0xffffffffu, lo, o);
		hi += __shfl_xor_sync(0xffffffffu, hi, o);
		long long a = __shfl_xor_sync(0xffffffffu, imin, o); imin = a < imin ? a : imin;
		a = __shfl_xor_sync(0xffffffffu, imax, o); imax = a > imax ? a : imax;
		unsigned long long b = __shfl_xor_sync(0xffffffffu, fmin, o); fmin = b < fmin ? b : fmin;
		b = __shfl_xor_sync(0xffffffffu, fmax, o); fmax = b > fmax ? b : fmax;
	}
	if ((threadIdx.x & 31) == 0 && cnt)
	{
		atomicAdd(&out->count, cnt);
		atomicAdd(&out->lo, lo);
		atomicAdd((unsigned long long *) &out->hi, (unsigned long long) hi);
		atomicMin(&out->imin, imin); atomicMax(&out->imax, imax);
		atomicMin(&out->fmin, fmin); atomicMax(&out->fmax, fmax);
	}
}

extern "C" int cg_agg_column(int32_t attlen, int32_t is_float, const void *values, const uint8_t *isnull, int64_t n,
							 int64_t *count, int64_t *sum_hi, uint64_t *sum_lo, int64_t *min_value, int64_t *max_value)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (n < 0 || (n > 0 && !values)) return cg_set_error(CG_EINVAL, "bad argument");
	if (attlen != 1 && attlen != 2 && attlen != 4 && attlen != 8) return cg_set_error(CG_EUNSUPPORTED, "attlen %d", attlen);
	if (is_float && attlen != 4 && attlen != 8) return cg_set_error(CG_EINVAL, "float with attlen %d", attlen);
	ColAggOut h;
	h.count = 0; h.lo = 0; h.hi = 0; h.imin = INT64_MAX; h.imax = INT64_MIN; h.fmin = ~0ull; h.fmax = 0;
	if (n > 0)
	{
		const size_t vb = ((size_t) n * attlen + 15 + 16) & ~(size_t) 15, zb = isnull ? (((size_t) n + 15) & ~(size_t) 15) : 0;
		CgAsyncBuf buf;
		CG_CUDA(buf.alloc(vb + zb + sizeof(ColAggOut), ctx->compute));
		uint8_t *d = buf.as<uint8_t>();
		ColAggOut *d_out = (ColAggOut *) (d + vb + zb);
		CG_CUDA(cudaMemcpyAsync(d, values, (size_t) n * attlen, cudaMemcpyHostToDevice, ctx->compute));
		if (isnull) CG_CUDA(cudaMemcpyAsync(d + vb, isnull, (size_t) n, cudaMemcpyHostToDevice, ctx->compute));
		CG_CUDA(cudaMemcpyAsync(d_out, &h, sizeof h, cudaMemcpyHostToDevice, ctx->compute));
		unsigned blocks = (unsigned) std::min<int64_t>((n + 255) / 256, (int64_t) ctx->sm_count * 8);
		cg_agg_column_kernel<<<blocks, 256, 0, ctx->compute>>>(d, isnull ? d + vb : nullptr, (long long) n, attlen, is_float, d_out);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
		CG_CUDA(cudaMemcpyAsync(&h, d_out, sizeof h, cudaMemcpyDeviceToHost, ctx->compute));
		CG_CUDA(cudaStreamSynchronize(ctx->compute));
	}
	if (count) *count = (int64_t) h.count;
	__int128 s = (__int128) (unsigned __int128) h.lo + ((__int128) h.hi << 32);
	if (sum_hi) *sum_hi = (int64_t) (s >> 64);
	if (sum_lo) *sum_lo = (uint64_t) s;
	if (is_float)
	{
		auto unorder = [](uint64_t u) { return (int64_t) (u == ~0ull ? 0x7ff8000000000000ull : (u >> 63) ? (u & 0x7fffffffffffffffull) : ~u); };
		if (min_value) *min_value = h.count ? unorder(h.fmin) : 0;
		if (max_value) *max_value = h.count ? unorder(h.fmax) : 0;
	}
	else
	{
		if (min_value) *min_value = h.count ? h.imin : 0;
		if (max_value) *max_value = h.count ? h.imax : 0;
	}
	return CG_OK;
}
