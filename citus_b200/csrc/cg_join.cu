/*
 * cg_join.cu -- the merge side of a dual-repartition join, for aggregate queries (K8).
 *
 * After worker_partition_query_result has routed both inputs by hash(join key), a MERGE task
 * reads the co-located partitions back with read_intermediate_results() and joins them with
 * PostgreSQL's executor (planner/multi_physical_planner.c:4304-4328 builds the function RTEs of
 * the merge query; executor/intermediate_results.c:789-1045 feeds them), one hash-table insert
 * per build row and one probe per probe row, then aggregates the joined rows.  With the
 * partitions already in HBM (the all-to-all delivered them), this file computes
 *
 *     SELECT count(*), sum(b.payload + p.payload) FROM build b JOIN probe p USING (key)
 *
 * -- the C4 check query of SURVEY.md 8(d) -- without materialising the joined rows: the build
 * side is aggregated per key while it is inserted (rows, sum of payload), and a probe row with
 * payload y that finds (c, s) contributes c joined rows and s + y * c to the sum, which is exactly
 * the sum over the c rows PostgreSQL's HashJoin would emit for it.  SQL semantics: a NULL key
 * joins nothing.  Sums are exact (128-bit).
 *
 * Open addressing over a separate key array (like the GROUP BY table in cg_scan.cu), load factor
 * <= 1/2, 64-bit CAS to claim a slot; values are one 32-byte sector per slot
 * [rows, sum of low 32 bits, sum of payload >> 32, unused].
 *
 * Two more forms follow: cg_join_rows emits the joined rows into device arrays, and cg_join_aggregate runs any scan
 * plan (WHERE tree, group key, aggregates) over the joined rows into a CgPartial, through the row path the
 * interpretive scan kernel uses (cg_device.cuh).  Both build one chained table over the build side.
 */
#include <vector>

#include "cg_internal.h"
#include "cg_device.cuh"

#define CGJ_THREADS 256
#define CGJ_EMPTY ((long long) 0x8000000000000000ull)

struct JoinTable
{
	long long *keys;              /* [cap + 1]; slot cap = the key equal to the EMPTY sentinel */
	unsigned long long *vals;     /* [cap + 1][4] */
	unsigned long long cap;       /* power of two */
	int shift;                    /* 64 - log2(cap) */
	unsigned long long *errors;
};

__global__ void cg_join_init_kernel(long long *keys, unsigned long long n)
{
	for (unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long) gridDim.x * blockDim.x)
		keys[i] = CGJ_EMPTY;
}

__device__ __forceinline__ unsigned long long join_home(long long key, int shift)
{
	return ((unsigned long long) key * 0x9E3779B97F4A7C15ull) >> shift;
}

/*
 * The slot of `key` in an open-addressing table of cap key slots (a power of two), for every key but the EMPTY sentinel,
 * whose slot is cap; ~0 when the key is absent (FIND) or the table is full (CLAIM).  CLAIM claims an empty slot with a
 * CAS and reads the keys through L2 (__ldcg: other threads are claiming slots); FIND stops at an empty slot and reads the
 * keys of a table an earlier kernel built through the read-only path (__ldg).
 */
enum JoinFind { CLAIM, FIND };

template <JoinFind MODE>
__device__ __forceinline__ unsigned long long join_find(long long *table, unsigned long long cap, int shift, long long key)
{
	unsigned long long h = join_home(key, shift), slot = ~0ull;
	for (unsigned long long probes = 0; probes <= cap; probes++)
	{
		long long cur = MODE == CLAIM ? (long long) __ldcg((unsigned long long *) table + h) : (long long) __ldg((const unsigned long long *) table + h);
		if (cur == key) { slot = h; break; }
		if (cur == CGJ_EMPTY)
		{
			if (MODE == FIND) break;
			long long old = (long long) atomicCAS((unsigned long long *) table + h, (unsigned long long) CGJ_EMPTY, (unsigned long long) key);
			if (old == CGJ_EMPTY || old == key) { slot = h; break; }
		}
		h = (h + 1) & (cap - 1);
	}
	return slot;
}

/* load factor <= 1/2: cap = the smallest power of two >= 2 * nbuild, at least 1024; shift = 64 - log2(cap) */
static void join_table_size(int64_t nbuild, unsigned long long *cap, int *shift)
{
	*cap = 1024;
	while (*cap < 2ull * (uint64_t) nbuild) *cap <<= 1;
	*shift = 64;
	for (unsigned long long c = *cap; c > 1; c >>= 1) (*shift)--;
}

__global__ void __launch_bounds__(CGJ_THREADS)
cg_join_build_kernel(JoinTable T, const long long *keys, const uint8_t *nulls, const long long *payload, long long n)
{
	for (long long r = (long long) blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long) gridDim.x * blockDim.x)
	{
		if (nulls && nulls[r]) continue;
		const long long key = keys[r];
		unsigned long long slot = T.cap;
		if (key != CGJ_EMPTY)
		{
			slot = join_find<CLAIM>(T.keys, T.cap, T.shift, key);
			if (slot == ~0ull) { atomicAdd(T.errors, 1ull); continue; }
		}
		const long long x = payload[r];
		unsigned long long *v = T.vals + slot * 4;
		atomicAdd(v + 0, 1ull);
		atomicAdd(v + 1, (unsigned long long) (unsigned int) x);
		atomicAdd(v + 2, (unsigned long long) (x >> 32));
	}
}

__device__ __forceinline__ unsigned long long join_wsum(unsigned long long x)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
	return x;
}

/* out[0] = joined rows; out[1..4] = the sum in 32-bit chunks (chunk 3 sign-extended), added without carries */
__global__ void __launch_bounds__(CGJ_THREADS)
cg_join_probe_kernel(JoinTable T, const long long *keys, const uint8_t *nulls, const long long *payload, long long n,
					 unsigned long long *out)
{
	unsigned long long matches = 0;
	unsigned __int128 sum = 0;
	for (long long r = (long long) blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long) gridDim.x * blockDim.x)
	{
		if (nulls && nulls[r]) continue;
		const long long key = keys[r];
		unsigned long long slot = T.cap;
		if (key != CGJ_EMPTY)
		{
			slot = join_find<FIND>(T.keys, T.cap, T.shift, key);
			if (slot == ~0ull) continue;
		}
		const ulonglong2 v01 = __ldg((const ulonglong2 *) (T.vals + slot * 4));
		const unsigned long long c = v01.x;
		if (c == 0) continue;
		const long long hi = (long long) __ldg(T.vals + slot * 4 + 2);
		matches += c;
		/* s + y * c with s = hi * 2^32 + lo, two's complement in 128 bits */
		__int128 s = ((__int128) hi << 32) + (__int128) (unsigned __int128) v01.y;
		s += (__int128) payload[r] * (__int128) (unsigned __int128) c;
		sum += (unsigned __int128) s;
	}
	unsigned long long c0 = (unsigned long long) (unsigned int) sum, c1 = (unsigned long long) (unsigned int) (sum >> 32),
					   c2 = (unsigned long long) (unsigned int) (sum >> 64),
					   c3 = (unsigned long long) (long long) (int) (unsigned int) (sum >> 96);
	matches = join_wsum(matches);
	c0 = join_wsum(c0); c1 = join_wsum(c1); c2 = join_wsum(c2); c3 = join_wsum(c3);
	if ((threadIdx.x & 31) == 0)
	{
		if (matches) atomicAdd(out + 0, matches);
		if (c0) atomicAdd(out + 1, c0);
		if (c1) atomicAdd(out + 2, c1);
		if (c2) atomicAdd(out + 3, c2);
		if (c3) atomicAdd(out + 4, c3);
	}
}

extern "C" int cg_join_count_sum(const int64_t *d_build_keys, const uint8_t *d_build_nulls, const int64_t *d_build_payload,
								 int64_t nbuild, const int64_t *d_probe_keys, const uint8_t *d_probe_nulls,
								 const int64_t *d_probe_payload, int64_t nprobe, int64_t *joined_rows, int64_t *sum_hi,
								 uint64_t *sum_lo)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (nbuild < 0 || nprobe < 0 || !joined_rows || !sum_hi || !sum_lo) return cg_set_error(CG_EINVAL, "bad argument");
	if ((nbuild > 0 && (!d_build_keys || !d_build_payload)) || (nprobe > 0 && (!d_probe_keys || !d_probe_payload)))
		return cg_set_error(CG_EINVAL, "NULL column");
	*joined_rows = 0; *sum_hi = 0; *sum_lo = 0;
	if (nbuild == 0 || nprobe == 0) return CG_OK;
	JoinTable T;
	join_table_size(nbuild, &T.cap, &T.shift);
	const size_t key_bytes = (T.cap + 1) * sizeof(long long), val_bytes = (T.cap + 1) * 4 * sizeof(unsigned long long);
	uint8_t *d_mem = nullptr;
	if (cudaMallocAsync((void **) &d_mem, key_bytes + 64 + val_bytes + 64, ctx->compute) != cudaSuccess)
	{
		cudaGetLastError();
		return cg_set_error(CG_ENOMEM, "cudaMallocAsync of %zu bytes for the join table failed", key_bytes + val_bytes);
	}
	T.keys = (long long *) d_mem;
	T.vals = (unsigned long long *) (d_mem + ((key_bytes + 63) & ~(size_t) 63));
	unsigned long long *d_out = (unsigned long long *) ((uint8_t *) T.vals + val_bytes);   /* 6 words: result + errors */
	T.errors = d_out + 5;
	CG_CUDA(cudaMemsetAsync(T.vals, 0, val_bytes + 64, ctx->compute));
	const unsigned blocks = (unsigned) (ctx->sm_count * 8);
	cg_join_init_kernel<<<blocks, CGJ_THREADS, 0, ctx->compute>>>(T.keys, T.cap + 1);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	cg_join_build_kernel<<<blocks, CGJ_THREADS, 0, ctx->compute>>>(T, (const long long *) d_build_keys, d_build_nulls,
																	  (const long long *) d_build_payload, (long long) nbuild);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	cg_join_probe_kernel<<<blocks, CGJ_THREADS, 0, ctx->compute>>>(T, (const long long *) d_probe_keys, d_probe_nulls,
																	  (const long long *) d_probe_payload, (long long) nprobe, d_out);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	unsigned long long h[6] = {0, 0, 0, 0, 0, 0};
	CG_CUDA(cudaMemcpyAsync(h, d_out, sizeof h, cudaMemcpyDeviceToHost, ctx->compute));
	CG_CUDA(cudaStreamSynchronize(ctx->compute));
	CG_CUDA(cudaFreeAsync(d_mem, ctx->compute));
	if (h[5]) return cg_set_error(CG_ETABLEFULL, "join table overflow (%llu rows)", h[5]);
	unsigned __int128 total = (unsigned __int128) h[1] + ((unsigned __int128) h[2] << 32) + ((unsigned __int128) h[3] << 64) +
							  ((unsigned __int128) h[4] << 96);
	*joined_rows = (int64_t) h[0];
	*sum_lo = (uint64_t) total;
	*sum_hi = (int64_t) (uint64_t) (total >> 64);
	return CG_OK;
}

/* ------------------------------------------------------------------------------ *
 *  The same join emitting its rows:
 *      SELECT b.key, b.payload, p.payload FROM build b JOIN probe p USING (key)
 *  for plans whose join output is not aggregated right away (the MERGE task of planner/multi_physical_planner.c:
 *  4304-4328 hands PostgreSQL's HashJoin output to whatever sits above it).  Build: every build row is linked into the
 *  chain of its key's slot (head[slot] <- row, next[row] <- old head: one atomic exchange per row) and the slot counts its
 *  rows.  Probe pass 1 looks the key up and records how many rows it joins; an exclusive prefix sum over the probe rows
 *  gives every probe row its place in the output; pass 2 walks the chain and writes the rows.  Row order is unspecified,
 *  as for any hash join.
 * ------------------------------------------------------------------------------ */
struct JoinRowsTable
{
	long long *keys;              /* [cap + 1] */
	unsigned int *count;          /* [cap + 1] build rows with this key */
	long long *head;              /* [cap + 1] first build row of the chain, -1 = none */
	long long *next;              /* [nbuild] */
	unsigned long long cap;
	int shift;
	unsigned long long *errors;
};

__global__ void cg_join_rows_init_kernel(JoinRowsTable T)
{
	for (unsigned long long i = (unsigned long long) blockIdx.x * blockDim.x + threadIdx.x; i <= T.cap; i += (unsigned long long) gridDim.x * blockDim.x)
	{
		T.keys[i] = CGJ_EMPTY; T.count[i] = 0; T.head[i] = -1;
	}
}

__global__ void __launch_bounds__(CGJ_THREADS)
cg_join_rows_build_kernel(JoinRowsTable T, const long long *keys, const uint8_t *nulls, long long n)
{
	for (long long r = (long long) blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long) gridDim.x * blockDim.x)
	{
		if (nulls && nulls[r]) continue;
		const long long key = keys[r];
		const unsigned long long slot = key == CGJ_EMPTY ? T.cap : join_find<CLAIM>(T.keys, T.cap, T.shift, key);
		if (slot == ~0ull) { atomicAdd(T.errors, 1ull); continue; }
		atomicAdd(T.count + slot, 1u);
		T.next[r] = (long long) atomicExch((unsigned long long *) T.head + slot, (unsigned long long) r);
	}
}

static size_t join_a64(size_t x) { return (x + 63) & ~(size_t) 63; }

/*
 * The chained table over the build keys, in one stream-ordered allocation (no host synchronisation): init and build
 * launches on `stream`.  The allocation holds the table, then `extra` bytes for the caller (*d_extra, 64-byte aligned),
 * then two zeroed words (*d_words): [0] is the caller's, [1] counts build rows that found no slot.  That count stays 0:
 * the table has at least 2 * nbuild slots and a claim probes every one of them.
 */
static int join_rows_table_build(CgContext *ctx, const int64_t *d_keys, const uint8_t *d_nulls, int64_t nbuild, size_t extra,
								 cudaStream_t stream, CgAsyncBuf *mem, JoinRowsTable *T, uint8_t **d_extra, unsigned long long **d_words)
{
	join_table_size(nbuild, &T->cap, &T->shift);
	const size_t kb = join_a64((T->cap + 1) * 8), cb = join_a64((T->cap + 1) * 4), hb = join_a64((T->cap + 1) * 8),
				 nb = join_a64((size_t) nbuild * 8);
	if (mem->alloc(kb + cb + hb + nb + extra + 64, stream) != cudaSuccess)
	{
		cudaGetLastError();
		return cg_set_error(CG_ENOMEM, "cudaMallocAsync of %zu bytes for the join failed", kb + cb + hb + nb + extra);
	}
	uint8_t *d = mem->as<uint8_t>();
	T->keys = (long long *) d; T->count = (unsigned int *) (d + kb); T->head = (long long *) (d + kb + cb); T->next = (long long *) (d + kb + cb + hb);
	*d_extra = d + kb + cb + hb + nb;
	*d_words = (unsigned long long *) (d + kb + cb + hb + nb + extra);
	T->errors = *d_words + 1;
	CG_CUDA(cudaMemsetAsync(*d_words, 0, 16, stream));
	const unsigned blocks = (unsigned) (ctx->sm_count * 8);
	cg_join_rows_init_kernel<<<blocks, CGJ_THREADS, 0, stream>>>(*T);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	cg_join_rows_build_kernel<<<blocks, CGJ_THREADS, 0, stream>>>(*T, (const long long *) d_keys, d_nulls, (long long) nbuild);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

/* matches[r] = rows probe row r joins; block sums for the scan (partition_scan_blocks with one partition) */
__global__ void __launch_bounds__(CGJ_THREADS)
cg_join_rows_count_kernel(JoinRowsTable T, const long long *keys, const uint8_t *nulls, long long n, unsigned int *matches,
						  unsigned long long *block_sums)
{
	__shared__ unsigned long long s_sum[CGJ_THREADS / 32];
	const long long r = (long long) blockIdx.x * blockDim.x + threadIdx.x;
	unsigned int m = 0;
	if (r < n && !(nulls && nulls[r]))
	{
		const long long key = keys[r];
		const unsigned long long slot = key == CGJ_EMPTY ? T.cap : join_find<FIND>(T.keys, T.cap, T.shift, key);
		if (slot != ~0ull) m = T.count[slot];
	}
	if (r < n) matches[r] = m;
	unsigned long long w = join_wsum((unsigned long long) m);
	if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = w;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		unsigned long long t = 0;
		for (int i = 0; i < CGJ_THREADS / 32; i++) t += s_sum[i];
		block_sums[blockIdx.x] = t;
	}
}

__global__ void __launch_bounds__(CGJ_THREADS)
cg_join_rows_emit_kernel(JoinRowsTable T, const long long *bpay, const long long *keys, const uint8_t *nulls, const long long *ppay, long long n,
						 const unsigned int *matches, const unsigned long long *block_offsets, unsigned long long capacity,
						 long long *out_key, long long *out_bpay, long long *out_ppay)
{
	__shared__ unsigned long long s_warp[CGJ_THREADS / 32];
	const long long r = (long long) blockIdx.x * blockDim.x + threadIdx.x;
	const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const unsigned int m = r < n ? matches[r] : 0u;
	/* place of this row's first output row: block offset + exclusive scan inside the block */
	unsigned long long incl = m;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1)
	{
		unsigned long long y = __shfl_up_sync(0xffffffffu, incl, o);
		if (lane >= (unsigned) o) incl += y;
	}
	if (lane == 31) s_warp[warp] = incl;
	__syncthreads();
	unsigned long long pos = block_offsets[blockIdx.x] + incl - m;
	for (unsigned w = 0; w < warp; w++) pos += s_warp[w];
	if (m == 0) return;
	const long long key = keys[r];
	const unsigned long long slot = key == CGJ_EMPTY ? T.cap : join_find<FIND>(T.keys, T.cap, T.shift, key);
	const long long y = ppay[r];
	for (long long b = T.head[slot]; b >= 0; b = T.next[b], pos++)
		if (pos < capacity)
		{
			out_key[pos] = key; out_bpay[pos] = bpay[b]; out_ppay[pos] = y;
		}
}

extern "C" int cg_join_rows(const int64_t *d_build_keys, const uint8_t *d_build_nulls, const int64_t *d_build_payload, int64_t nbuild,
							const int64_t *d_probe_keys, const uint8_t *d_probe_nulls, const int64_t *d_probe_payload, int64_t nprobe,
							int64_t capacity, int64_t *d_out_key, int64_t *d_out_build_payload, int64_t *d_out_probe_payload, int64_t *nrows)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (nbuild < 0 || nprobe < 0 || capacity < 0 || !nrows) return cg_set_error(CG_EINVAL, "bad argument");
	if ((nbuild > 0 && (!d_build_keys || !d_build_payload)) || (nprobe > 0 && (!d_probe_keys || !d_probe_payload)))
		return cg_set_error(CG_EINVAL, "NULL column");
	if (capacity > 0 && (!d_out_key || !d_out_build_payload || !d_out_probe_payload)) return cg_set_error(CG_EINVAL, "NULL output column");
	*nrows = 0;
	if (nbuild == 0 || nprobe == 0) return CG_OK;
	JoinRowsTable T;
	const long long nblocks = (nprobe + CGJ_THREADS - 1) / CGJ_THREADS;
	const size_t mb = join_a64((size_t) nprobe * 4), bb = join_a64((size_t) nblocks * 8);
	CgAsyncBuf mem;
	uint8_t *d_extra;
	unsigned long long *d_tot;     /* [0] total rows, [1] errors */
	if (int rc = join_rows_table_build(ctx, d_build_keys, d_build_nulls, nbuild, mb + bb, ctx->compute, &mem, &T, &d_extra, &d_tot)) return rc;
	unsigned int *d_matches = (unsigned int *) d_extra;
	unsigned long long *d_block = (unsigned long long *) (d_extra + mb);
	cg_join_rows_count_kernel<<<(unsigned) nblocks, CGJ_THREADS, 0, ctx->compute>>>(T, (const long long *) d_probe_keys, d_probe_nulls, (long long) nprobe,
																				  d_matches, d_block);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	CgAsyncBuf chunk_buf;
	if (int rc = partition_scan_blocks(ctx, d_block, d_tot, nblocks, 1, &chunk_buf)) return rc;
	unsigned long long h[2] = {0, 0};
	CG_CUDA(cudaMemcpyAsync(h, d_tot, sizeof h, cudaMemcpyDeviceToHost, ctx->compute));
	CG_CUDA(cudaStreamSynchronize(ctx->compute));
	if (h[1]) return cg_set_error(CG_ETABLEFULL, "join table overflow (%llu rows)", h[1]);
	*nrows = (int64_t) h[0];
	if ((int64_t) h[0] > capacity)
		return capacity == 0 ? CG_OK : cg_set_error(CG_EINVAL, "%llu joined rows exceed the caller's capacity %lld", h[0], (long long) capacity);
	if (h[0] == 0) return CG_OK;
	cg_join_rows_emit_kernel<<<(unsigned) nblocks, CGJ_THREADS, 0, ctx->compute>>>(T, (const long long *) d_build_payload, (const long long *) d_probe_keys,
																				 d_probe_nulls, (const long long *) d_probe_payload, (long long) nprobe,
																				 d_matches, d_block, (unsigned long long) capacity,
																				 (long long *) d_out_key, (long long *) d_out_build_payload,
																				 (long long *) d_out_probe_payload);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	CG_CUDA(cudaStreamSynchronize(ctx->compute));
	return CG_OK;
}

/* ------------------------------------------------------------------------------ *
 *  Any scan query over the joined rows (cg_join_aggregate):
 *      SELECT <group key, aggregates> FROM build b JOIN probe p USING (key) WHERE ... GROUP BY ...
 *  the Agg <- HashJoin of the MERGE task (planner/multi_physical_planner.c:598-687 gives it the worker half of the
 *  aggregates, the GROUP BY and the WHERE).  The build side goes into cg_join_rows' chained table; one thread per probe
 *  row loads the probe side's plan columns once (coalesced), finds the key's slot and walks the chain, and for every build
 *  row gathers the build side's plan columns and hands the joined row to the row path of the interpretive scan kernel
 *  (process_row, cg_device.cuh).  The joined rows are never materialised.
 * ------------------------------------------------------------------------------ */
/* where plan column c of the joined row comes from: column col[c] (null array nul[c], may be NULL) of the probe side
 * (probe bit c set) or of the build side */
struct JoinAggCols
{
	const long long *col[CG_KMAX_COLS];
	const uint8_t *nul[CG_KMAX_COLS];
	uint32_t probe;
};

template <int NCC, int NAC, int MODE, bool VAR, bool CASE = false>
__global__ void __launch_bounds__(CGJ_THREADS, 4)
cg_join_agg_kernel(const __grid_constant__ KPlan P, const JoinAggCols J, const JoinRowsTable T, const long long *keys, const uint8_t *key_nulls,
				   long long n)
{
	ThreadAcc<NAC, VAR> acc;
	thread_acc_init(P, acc);
	uint32_t removed = 0;
	unsigned long long joined = 0;
	for (long long r = (long long) blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (long long) gridDim.x * blockDim.x)
	{
		if (key_nulls && key_nulls[r]) continue;
		const long long key = keys[r];
		const unsigned long long slot = key == CGJ_EMPTY ? T.cap : join_find<FIND>(T.keys, T.cap, T.shift, key);
		if (slot == ~0ull) continue;
		long long b = (long long) __ldg((const unsigned long long *) T.head + slot);
		if (b < 0) continue;
		int64_t v[NCC];
		uint32_t pnull = 0;
#pragma unroll
		for (int c = 0; c < NCC; c++)
		{
			v[c] = 0;
			if (c < P.ncols && ((J.probe >> c) & 1u))
			{
				v[c] = J.col[c][r];
				if (J.nul[c] && J.nul[c][r]) pnull |= 1u << c;
			}
		}
		for (; b >= 0; b = (long long) __ldg((const unsigned long long *) T.next + b))
		{
			uint32_t nullmask = pnull;
#pragma unroll
			for (int c = 0; c < NCC; c++)
				if (c < P.ncols && !((J.probe >> c) & 1u))
				{
					v[c] = __ldg(J.col[c] + b);
					if (J.nul[c] && __ldg(J.nul[c] + b)) nullmask |= 1u << c;
				}
			joined++;
			process_row<NCC, NAC, MODE, VAR, CASE>(P, v, nullmask, acc, removed);
		}
	}
	flush_thread<NAC, MODE, VAR>(P, acc, removed, joined);
}

template <int MODE, bool VAR, bool CASE = false>
static int launch_join_agg(CgContext *ctx, const KPlan &plan, const JoinAggCols &J, const JoinRowsTable &T, const long long *keys,
						   const uint8_t *key_nulls, long long n, cudaStream_t stream)
{
	auto kernel = cg_join_agg_kernel<CG_KMAX_COLS, CG_MAX_AGGS, MODE, VAR, CASE>;
	int occ = 0;
	CG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, CGJ_THREADS, 0));
	if (occ < 1) occ = 1;
	long long grid = (long long) ctx->sm_count * occ, need = (n + CGJ_THREADS - 1) / CGJ_THREADS;
	if (grid > need) grid = need;
	bool overlap;
	int rc = cg_chain_scan(ctx, stream, false, &overlap);     /* an ordinary launch: ends a chain */
	if (rc) return rc;
	kernel<<<(unsigned) grid, CGJ_THREADS, 0, stream>>>(plan, J, T, keys, key_nulls, n);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

int cg_launch_join_aggregate(CgContext *ctx, const KPlan &plan, const CgJoinSide *const sides[2], cudaStream_t stream)
{
	const CgJoinSide &b = *sides[0], &p = *sides[1];
	JoinAggCols J;
	memset(&J, 0, sizeof J);
	for (int c = 0; c < plan.ncols; c++)
	{
		/* a plan column's slot is its joined-row attribute: build columns first, then probe columns */
		const bool probe = plan.slot[c] >= b.ncols;
		const CgJoinSide &s = probe ? p : b;
		const int i = probe ? plan.slot[c] - b.ncols : plan.slot[c];
		J.col[c] = (const long long *) s.d_cols[i];
		J.nul[c] = s.d_nulls ? s.d_nulls[i] : nullptr;
		if (probe) J.probe |= 1u << c;
	}
	int rc = cg_chain_end(ctx, stream);
	if (rc) return rc;
	JoinRowsTable T;
	CgAsyncBuf mem;
	uint8_t *d_extra;
	unsigned long long *d_words;
	rc = join_rows_table_build(ctx, b.d_cols[b.key], b.d_nulls ? b.d_nulls[b.key] : nullptr, b.nrows, 0, stream, &mem, &T, &d_extra, &d_words);
	if (rc) return rc;
	const long long *keys = (const long long *) p.d_cols[p.key];
	const uint8_t *key_nulls = p.d_nulls ? p.d_nulls[p.key] : nullptr;
	/* plans with a CASE argument: one instance per table kind, variance included */
	if (plan.ncase > 0)
		switch (plan.mode)
		{
			case CG_MODE_GLOBAL: return launch_join_agg<CG_MODE_GLOBAL, true, true>(ctx, plan, J, T, keys, key_nulls, p.nrows, stream);
			case CG_MODE_DENSE: return launch_join_agg<CG_MODE_DENSE, true, true>(ctx, plan, J, T, keys, key_nulls, p.nrows, stream);
			default: return launch_join_agg<CG_MODE_HASH, true, true>(ctx, plan, J, T, keys, key_nulls, p.nrows, stream);
		}
	const bool var = cg_plan_has_variance(plan.aggs, plan.naggs);
	switch (plan.mode)
	{
		case CG_MODE_GLOBAL:
			return var ? launch_join_agg<CG_MODE_GLOBAL, true>(ctx, plan, J, T, keys, key_nulls, p.nrows, stream)
					   : launch_join_agg<CG_MODE_GLOBAL, false>(ctx, plan, J, T, keys, key_nulls, p.nrows, stream);
		case CG_MODE_DENSE:
			return var ? launch_join_agg<CG_MODE_DENSE, true>(ctx, plan, J, T, keys, key_nulls, p.nrows, stream)
					   : launch_join_agg<CG_MODE_DENSE, false>(ctx, plan, J, T, keys, key_nulls, p.nrows, stream);
		default:
			return var ? launch_join_agg<CG_MODE_HASH, true>(ctx, plan, J, T, keys, key_nulls, p.nrows, stream)
					   : launch_join_agg<CG_MODE_HASH, false>(ctx, plan, J, T, keys, key_nulls, p.nrows, stream);
	}
}
