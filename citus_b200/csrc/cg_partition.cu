/*
 * cg_partition.cu -- K6: the map side of the hash repartition.
 *
 * Per row the reference does (executor/partitioned_intermediate_results.c:493-553
 * PartitionedResultDestReceiverReceive):
 *    NULL key              -> partition 0
 *    FindShardInterval     -> hashint4 / hashint8 of the key through fmgr
 *                             (utils/shardinterval_utils.c:260-282), then a binary search
 *                             of the int4 token ranges (SearchCachedShardInterval :373-414;
 *                             the synthetic intervals of planner/multi_physical_planner.c:
 *                             4667-4701 are passed as min/max arrays)
 *    receiveSlot           -> append the row to that partition's file
 * Here: one pass computes the partition index of every row and a histogram (per-block
 * counts in shared memory, one global atomic per block and partition), a second pass
 * scatters the payload columns into partition-contiguous order -- stable inside a
 * partition, like the reference's append order -- using per-block and per-warp offsets.
 *
 * [PG] hash_bytes_uint32 / hashint4 / hashint8: src/common/hashfn.c,
 * src/backend/access/hash/hashfunc.c (Jenkins lookup3 final mix); pinned by the
 * reference goldens through the oracle (tests/test_oracle_golden.py).
 */
#include <algorithm>
#include <initializer_list>
#include <vector>

#include "cg_internal.h"

#define CGP_THREADS 256
#define CGP_ROWS_PER_BLOCK 4096
#define CGP_MAX_P 1024
#define CGP_MAX_COLS 16

__device__ __forceinline__ uint32_t rot32(uint32_t x, int k) { return (x << k) | (x >> (32 - k)); }

__device__ __forceinline__ uint32_t hash_bytes_uint32(uint32_t k)
{
	uint32_t a, b, c;
	a = b = c = 0x9e3779b9u + 4u + 3923095u;
	a += k;
	c ^= b; c -= rot32(b, 14);
	a ^= c; a -= rot32(c, 11);
	b ^= a; b -= rot32(a, 25);
	c ^= b; c -= rot32(b, 16);
	a ^= c; a -= rot32(c, 4);
	b ^= a; b -= rot32(a, 14);
	c ^= b; c -= rot32(b, 24);
	return c;
}

__device__ __forceinline__ int32_t hashint8_dev(int64_t v)
{
	uint32_t lo = (uint32_t) v, hi = (uint32_t) ((uint64_t) v >> 32);
	lo ^= (v >= 0) ? hi : ~hi;
	return (int32_t) hash_bytes_uint32(lo);
}

/*
 * Routing and the stable scatter the repartition uses, built for instruction count (the scatter is issue-bound):
 *   routing   hashint4/8, then -- when the intervals are the uniform ones the planner generates
 *             (GenerateSyntheticShardIntervalArray, planner/multi_physical_planner.c:4667-4701) -- the reference's own
 *             shortcut CalculateUniformHashRangeIndex (utils/shardinterval_utils.c:424-452): (hash - INT32_MIN) / increment,
 *             a shift when P is a power of two; the interval search only for arbitrary bounds.  Done ONCE, in the histogram
 *             pass, which leaves a 2-byte partition number per row for the scatter pass.
 *   order     a block owns 4096 consecutive rows, each of its 8 warps a contiguous segment of 512.  Pass A: every warp
 *             histograms its segment into its own row of shared memory (match.any groups the lanes of a step by
 *             partition; the group's first lane adds the group size -- the row is warp-private, no atomics).  One
 *             barrier, then the per-(warp, partition) start offsets = block offset + counts of the warps before.  Pass B:
 *             every warp walks its segment again in input order; a row's destination is its partition's running offset +
 *             its rank among the lanes of the same partition in this step.  Output order inside a partition therefore
 *             equals input order, like the reference's append-to-file loop
 *             (executor/partitioned_intermediate_results.c:493-553).
 *   ranks     one match.any per row (pass A); its rank and group size travel to pass B in a register
 *   output    rows are placed in partition order in shared memory and leave as runs (a block's rows of one partition are
 *             contiguous in the output): coalesced stores; the partition of a local position is a 2-byte lookup
 * Traffic per row and table: keys 8 B + 2 B written (histogram pass), 2 B + every column read and written once.
 */
struct RouteParams
{
	const int64_t *keys;
	const uint8_t *nulls;
	int32_t key_len, by_hash;
	const int32_t *mins, *maxs;      /* device, [P] */
	uint32_t uniform_inc;            /* != 0: uniform hash intervals of this width */
	int32_t uniform_shift;           /* >= 0: the width is 2^shift */
};

struct StagedScatterParams
{
	const void *index;               /* uint16_t[n] (repartition) or int32_t[n] (public API) */
	int64_t n;
	int32_t P, ncols;
	const unsigned long long *block_offsets;   /* [nblocks][P] in output order */
	const unsigned long long *part_base;       /* [P] in output order */
	const int32_t *order;                      /* [P] output position of partition p, or NULL (already applied / identity) */
	const int64_t *cols[8];
	int64_t *out[8];
};

__device__ __forceinline__ int route_row(const RouteParams &R, const int32_t *s_min, const int32_t *s_max, int P, int64_t r, bool *unroutable)
{
	if (R.nulls && R.nulls[r]) return 0;
	const int64_t k = R.keys[r];
	if (R.by_hash && R.uniform_inc)
	{
		const uint32_t h = R.key_len == 4 ? hash_bytes_uint32((uint32_t) (int32_t) k) : (uint32_t) hashint8_dev(k);
		const uint32_t u = h ^ 0x80000000u;                                   /* hash - INT32_MIN */
		const uint32_t idx = R.uniform_shift >= 0 ? (u >> R.uniform_shift) : (u / R.uniform_inc);
		return (int) (idx < (uint32_t) P ? idx : (uint32_t) P - 1u);           /* the last interval is widened to INT32_MAX */
	}
	/* range partitioning compares the key itself: an int8 key outside the int4 interval bounds lies in no interval ("could
	 * not find shard"), it must not be truncated into one */
	const int64_t searched = R.by_hash ? (int64_t) (R.key_len == 4 ? (int32_t) hash_bytes_uint32((uint32_t) (int32_t) k) : hashint8_dev(k))
									   : (R.key_len == 4 ? (int64_t) (int32_t) k : k);
	/* SearchCachedShardInterval */
	int lower = 0, upper = P;
	while (lower < upper)
	{
		int middle = (lower + upper) / 2;
		if (searched < s_min[middle]) { upper = middle; continue; }
		if (searched <= s_max[middle]) return middle;
		lower = middle + 1;
	}
	*unroutable = true;
	return 0;
}

/* routing + histogram: index16[r] = output POSITION of the row's partition, block_counts[b][position], counts[p] (partition
 * order), errors */
__global__ void __launch_bounds__(CGP_THREADS)
cg_route_hist_kernel(const RouteParams R, int64_t n, int P, const int32_t *order, uint16_t *index16, unsigned long long *block_counts,
					 unsigned long long *counts, unsigned long long *errors)
{
	extern __shared__ unsigned int s_hist[];      /* [P] counts (by position), [P] mins, [P] maxs, [P] order */
	int32_t *s_min = (int32_t *) (s_hist + P), *s_max = s_min + P, *s_ord = s_max + P;
	for (int p = threadIdx.x; p < P; p += CGP_THREADS)
	{
		s_hist[p] = 0; s_ord[p] = order ? order[p] : p;
		if (!R.uniform_inc || !R.by_hash) { s_min[p] = R.mins[p]; s_max[p] = R.maxs[p]; }
	}
	__syncthreads();
	const int64_t base = (int64_t) blockIdx.x * CGP_ROWS_PER_BLOCK;
	unsigned int nbad = 0;
#pragma unroll 4
	for (int i = threadIdx.x; i < CGP_ROWS_PER_BLOCK; i += CGP_THREADS)
	{
		int64_t r = base + i;
		if (r >= n) break;
		bool bad = false;
		const int pos = s_ord[route_row(R, s_min, s_max, P, r, &bad)];
		index16[r] = (uint16_t) pos;
		atomicAdd(&s_hist[pos], 1u);
		nbad += bad ? 1u : 0u;
	}
	if (nbad) atomicAdd(errors, (unsigned long long) nbad);
	__syncthreads();
	for (int p = threadIdx.x; p < P; p += CGP_THREADS)
	{
		const unsigned int c = s_hist[s_ord[p]];
		block_counts[(uint64_t) blockIdx.x * P + s_ord[p]] = c;
		if (c) atomicAdd(counts + p, (unsigned long long) c);
	}
}

/* routing for caller arrays (cg_partition_index): index[r] = the row's partition, counts[p], errors */
__global__ void __launch_bounds__(CGP_THREADS)
cg_partition_index_kernel(const RouteParams R, int64_t n, int P, int32_t *index, unsigned long long *counts, unsigned long long *errors)
{
	extern __shared__ unsigned int s_count[];     /* [P] counts, [P] mins, [P] maxs */
	int32_t *s_min = (int32_t *) (s_count + P), *s_max = s_min + P;
	for (int p = threadIdx.x; p < P; p += CGP_THREADS)
	{
		s_count[p] = 0;
		if (!R.uniform_inc || !R.by_hash) { s_min[p] = R.mins[p]; s_max[p] = R.maxs[p]; }
	}
	__syncthreads();
	const int64_t base = (int64_t) blockIdx.x * CGP_ROWS_PER_BLOCK;
	unsigned int nbad = 0;
	for (int i = threadIdx.x; i < CGP_ROWS_PER_BLOCK; i += CGP_THREADS)
	{
		int64_t r = base + i;
		if (r >= n) break;
		bool bad = false;
		const int idx = route_row(R, s_min, s_max, P, r, &bad);
		index[r] = idx;
		atomicAdd(&s_count[idx], 1u);
		nbad += bad ? 1u : 0u;
	}
	if (nbad) atomicAdd(errors, (unsigned long long) nbad);
	__syncthreads();
	for (int p = threadIdx.x; p < P; p += CGP_THREADS)
	{
		const unsigned int c = s_count[p];
		if (c) atomicAdd(counts + p, (unsigned long long) c);
	}
}

template <typename IndexT, bool PEER>
__global__ void __launch_bounds__(CGP_THREADS, 4)     /* <= 64 registers: four CTAs per SM (the first build used 80 -> three) */
cg_scatter_staged_kernel(const __grid_constant__ StagedScatterParams A, const __grid_constant__ CgPeerScatter B)
{
	constexpr int WARPS = CGP_THREADS / 32;
	constexpr int SEG = CGP_ROWS_PER_BLOCK / WARPS;
	constexpr int STEPS = SEG / 32;
	extern __shared__ unsigned long long s_mem[];
	unsigned long long *s_stage = s_mem;                                        /* [4096] one column of the block, in partition order */
	unsigned long long *s_gbase = s_stage + CGP_ROWS_PER_BLOCK;                 /* [P] global position of the block's first row of p, minus its local start */
	unsigned int *s_cnt = (unsigned int *) (s_gbase + A.P);                     /* [WARPS][P] per-warp counts, then running local offsets */
	uint16_t *s_part = (uint16_t *) (s_cnt + WARPS * A.P);                      /* [4096] partition of every local position */
	unsigned long long *s_optr = (unsigned long long *) (s_part + CGP_ROWS_PER_BLOCK);   /* PEER: [P] address of output index 0 of p, this column */
	const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned int *mine = s_cnt + warp * A.P;
	for (int p = threadIdx.x; p < WARPS * A.P; p += CGP_THREADS) s_cnt[p] = 0;
	__syncthreads();
	const int64_t seg0 = (int64_t) blockIdx.x * CGP_ROWS_PER_BLOCK + (int64_t) warp * SEG;
	const IndexT *index = (const IndexT *) A.index;
	short idx[STEPS];
	unsigned short rk[STEPS];          /* rank among the lanes of the same partition in this step | group size << 5 */
	/* pass A: per-warp histogram; one match.any per row */
#pragma unroll
	for (int st = 0; st < STEPS; st++)
	{
		const int64_t r = seg0 + st * 32 + lane;
		int p = -1;
		if (r < A.n)
		{
			p = (int) index[r];
			if (A.order) p = A.order[p];
		}
		idx[st] = (short) p;
		const unsigned peers = __match_any_sync(0xffffffffu, p);
		const unsigned rank = __popc(peers & ((1u << lane) - 1u)), size = __popc(peers);
		rk[st] = (unsigned short) (rank | (size << 5));
		if (p >= 0 && rank == 0) mine[p] += size;
		__syncwarp();
	}
	__syncthreads();
	/* block totals per partition -> local starts (exclusive scan over P), global bases, per-warp running offsets */
	__shared__ unsigned int s_warp_tot[WARPS];
	__shared__ unsigned int s_block_rows;
	{
		const int per = (A.P + CGP_THREADS - 1) / CGP_THREADS;
		const int p0 = threadIdx.x * per, p1 = min(p0 + per, A.P);
		unsigned int local = 0;
		for (int p = p0; p < p1; p++)
			for (int w = 0; w < WARPS; w++) local += s_cnt[w * A.P + p];
		unsigned int incl = local;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1)
		{
			unsigned int y = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= (unsigned) o) incl += y;
		}
		if (lane == 31) s_warp_tot[warp] = incl;
		__syncthreads();
		unsigned int run = incl - local;
		for (unsigned w = 0; w < warp; w++) run += s_warp_tot[w];
		for (int p = p0; p < p1; p++)
		{
			s_gbase[p] = A.part_base[p] + A.block_offsets[(uint64_t) blockIdx.x * A.P + p] - run;
			for (int w = 0; w < WARPS; w++)
			{
				unsigned int c = s_cnt[w * A.P + p];
				s_cnt[w * A.P + p] = run;
				run += c;
			}
		}
		if (threadIdx.x == CGP_THREADS - 1) s_block_rows = run;
	}
	__syncthreads();
	const unsigned int block_rows = s_block_rows;
	/* pass B: local position of every row (input order inside a partition) */
	unsigned short lpos[STEPS];
#pragma unroll
	for (int st = 0; st < STEPS; st++)
	{
		const int p = idx[st];
		const unsigned rank = rk[st] & 31u;
		if (p >= 0)
		{
			lpos[st] = (unsigned short) (mine[p] + rank);
			s_part[lpos[st]] = (uint16_t) p;
		}
		__syncwarp();
		if (p >= 0 && rank == 0) mine[p] += rk[st] >> 5;
		__syncwarp();
	}
	/* column by column: into partition order in shared memory, out as coalesced runs */
	for (int c = 0; c < A.ncols; c++)
	{
		__syncthreads();
#pragma unroll
		for (int st = 0; st < STEPS; st++)
			if (idx[st] >= 0) s_stage[lpos[st]] = (unsigned long long) A.cols[c][seg0 + st * 32 + lane];
		if (PEER)
		{
			/* the rank that owns position p, and where this block's rows of p start in that rank's receive buffer */
			for (int p = threadIdx.x; p < A.P; p += CGP_THREADS)
			{
				int d = 0;
				while (d + 1 < B.nranks && p >= B.pos_begin[d + 1]) d++;
				s_optr[p] = (unsigned long long) B.base[d] +
							8ull * ((unsigned long long) ((long long) c * B.stride[d] + B.adj[d]) + s_gbase[p]);
			}
		}
		__syncthreads();
		if (PEER)
		{
			for (unsigned int j = threadIdx.x; j < block_rows; j += CGP_THREADS)
				((int64_t *) s_optr[s_part[j]])[j] = (int64_t) s_stage[j];          /* runs of one partition: coalesced stores over NVLink */
		}
		else
		{
			for (unsigned int j = threadIdx.x; j < block_rows; j += CGP_THREADS)
				A.out[c][s_gbase[s_part[j]] + j] = (int64_t) s_stage[j];
		}
	}
}

static size_t staged_scatter_smem(int P, bool peer = false)
{
	return sizeof(unsigned long long) * (CGP_ROWS_PER_BLOCK + (size_t) P) + sizeof(unsigned int) * ((CGP_THREADS / 32) * (size_t) P) +
		   sizeof(uint16_t) * CGP_ROWS_PER_BLOCK + (peer ? sizeof(unsigned long long) * (size_t) P : 0) + 16;
}

/* are [mins, maxs] the uniform hash intervals of width floor(2^32 / P), the last one widened to INT32_MAX? */
static void detect_uniform(const int32_t *mins, const int32_t *maxs, int P, RouteParams *R)
{
	R->uniform_inc = 0; R->uniform_shift = -1;
	const uint64_t inc = (1ull << 32) / (uint64_t) P;
	for (int i = 0; i < P; i++)
	{
		const int64_t lo = (int64_t) INT32_MIN + (int64_t) i * (int64_t) inc;
		const int64_t hi = i == P - 1 ? (int64_t) INT32_MAX : lo + (int64_t) inc - 1;
		if (mins[i] != lo || maxs[i] != hi) return;
	}
	R->uniform_inc = (uint32_t) inc;
	for (int sft = 0; sft < 32; sft++) if ((1ull << sft) == inc) R->uniform_shift = sft;
}

/*
 * A few kilobytes of host data for the kernels that follow on the compute stream: interval bounds, partition order, the
 * serializer's file layout.  They go through one pinned bounce buffer -- a pageable source would make the copy
 * synchronous -- into one device buffer.  The device buffer is reused in stream order, the bounce buffer once the
 * previous upload's copy has run.  d[i] receives the device address of host[i].
 */
struct HostArray
{
	const void *data;
	size_t bytes;
};
#define CGP_UPLOAD_BYTES ((3 * sizeof(unsigned long long) + 1) * CGP_MAX_P + 64)

static int upload_small(CgContext *ctx, std::initializer_list<HostArray> host, const void **d)
{
	static uint8_t *h_pin = nullptr, *d_buf = nullptr;
	static cudaEvent_t pin_free = nullptr;
	if (!h_pin) CG_CUDA(cudaHostAlloc((void **) &h_pin, CGP_UPLOAD_BYTES, cudaHostAllocDefault));
	if (!d_buf) CG_CUDA(cudaMalloc((void **) &d_buf, CGP_UPLOAD_BYTES));
	if (!pin_free) CG_CUDA(cudaEventCreateWithFlags(&pin_free, cudaEventDisableTiming));
	CG_CUDA(cudaEventSynchronize(pin_free));
	size_t off = 0;
	for (const HostArray &a : host)
	{
		if (off + a.bytes > CGP_UPLOAD_BYTES) return cg_set_error(CG_EINVAL, "%zu bytes of host arrays exceed the upload buffer", off + a.bytes);
		memcpy(h_pin + off, a.data, a.bytes);
		*d++ = d_buf + off;
		off += (a.bytes + 15) & ~(size_t) 15;
	}
	CG_CUDA(cudaMemcpyAsync(d_buf, h_pin, off, cudaMemcpyHostToDevice, ctx->compute));
	CG_CUDA(cudaEventRecord(pin_free, ctx->compute));
	return CG_OK;
}

extern "C" int cg_partition_index(const int64_t *d_keys, const uint8_t *d_nulls, int64_t n, int32_t key_len,
								  int32_t by_hash, const int32_t *mins, const int32_t *maxs, int32_t P,
								  int32_t *d_index, int64_t *d_counts)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (P <= 0) return cg_set_error(CG_EINVAL, "number of partitions cannot be 0");
	if (P > CGP_MAX_P) return cg_set_error(CG_EUNSUPPORTED, "more than %d partitions", CGP_MAX_P);
	if (key_len != 4 && key_len != 8) return cg_set_error(CG_EINVAL, "key_len must be 4 or 8");
	if (n < 0 || (n > 0 && !d_keys) || !d_index || !d_counts || !mins || !maxs) return cg_set_error(CG_EINVAL, "bad argument");
	CgAsyncBuf err_buf;
	CG_CUDA(err_buf.alloc(sizeof(unsigned long long), ctx->compute));
	unsigned long long *d_err = err_buf.as<unsigned long long>();
	RouteParams R = {d_keys, d_nulls, key_len, by_hash};
	const void *d[2];
	if (int rc = upload_small(ctx, {{mins, sizeof(int32_t) * P}, {maxs, sizeof(int32_t) * P}}, d)) return rc;
	R.mins = (const int32_t *) d[0]; R.maxs = (const int32_t *) d[1];
	detect_uniform(mins, maxs, P, &R);
	CG_CUDA(cudaMemsetAsync(d_err, 0, sizeof(unsigned long long), ctx->compute));
	CG_CUDA(cudaMemsetAsync(d_counts, 0, sizeof(int64_t) * P, ctx->compute));
	if (n > 0)
	{
		int64_t nblocks = (n + CGP_ROWS_PER_BLOCK - 1) / CGP_ROWS_PER_BLOCK;
		cg_partition_index_kernel<<<(unsigned) nblocks, CGP_THREADS, 3 * P * sizeof(int32_t), ctx->compute>>>(R, n, P, d_index,
																											  (unsigned long long *) d_counts, d_err);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
	}
	unsigned long long err = 0;
	CG_CUDA(cudaMemcpyAsync(&err, d_err, sizeof err, cudaMemcpyDeviceToHost, ctx->compute));
	CG_CUDA(cudaStreamSynchronize(ctx->compute));
	if (err) return cg_set_error(CG_EINVAL, "could not find shard for partition column value (%llu rows)", err);
	return CG_OK;
}

/*
 * Per-partition exclusive scan of block counts with all SMs (declared in cg_internal.h): block_counts[b][p] becomes the
 * start of block b inside partition p, totals[p] the partition's total.  The blocks are cut into chunks of CGP_SCAN_CHUNK;
 * pass 1 sums every (partition, chunk), pass 2 scans the chunk sums of a partition (one thread) and yields its total,
 * pass 3 rewrites every chunk as offsets.
 */
#define CGP_SCAN_CHUNK 2048
__global__ void __launch_bounds__(256)
cg_partition_scan_sum_kernel(const unsigned long long *block_counts, unsigned long long *chunk_sums, int64_t nblocks, int P, int nchunks)
{
	__shared__ unsigned long long s_w[8];
	const int p = blockIdx.x % P, c = blockIdx.x / P;
	const int64_t b0 = (int64_t) c * CGP_SCAN_CHUNK, b1 = b0 + CGP_SCAN_CHUNK < nblocks ? b0 + CGP_SCAN_CHUNK : nblocks;
	unsigned long long local = 0;
	for (int64_t b = b0 + threadIdx.x; b < b1; b += 256) local += block_counts[b * P + p];
	for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
	if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = local;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		unsigned long long t = 0;
		for (int i = 0; i < 8; i++) t += s_w[i];
		chunk_sums[(size_t) p * nchunks + c] = t;
	}
}

__global__ void cg_partition_scan_chunks_kernel(unsigned long long *chunk_sums, unsigned long long *totals, int P, int nchunks)
{
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= P) return;
	unsigned long long run = 0;
	for (int c = 0; c < nchunks; c++) { unsigned long long v = chunk_sums[(size_t) p * nchunks + c]; chunk_sums[(size_t) p * nchunks + c] = run; run += v; }
	totals[p] = run;
}

__global__ void __launch_bounds__(256)
cg_partition_scan_apply_kernel(unsigned long long *block_counts, const unsigned long long *chunk_sums, int64_t nblocks, int P, int nchunks)
{
	__shared__ unsigned long long s_w[8];
	const int p = blockIdx.x % P, c = blockIdx.x / P;
	const int64_t b0 = (int64_t) c * CGP_SCAN_CHUNK, b1 = b0 + CGP_SCAN_CHUNK < nblocks ? b0 + CGP_SCAN_CHUNK : nblocks;
	const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned long long run = chunk_sums[(size_t) p * nchunks + c];
	for (int64_t base = b0; base < b1; base += 256)
	{
		const int64_t b = base + threadIdx.x;
		const unsigned long long v = b < b1 ? block_counts[b * P + p] : 0ull;
		unsigned long long incl = v;
		for (int o = 1; o < 32; o <<= 1)
		{
			unsigned long long y = __shfl_up_sync(0xffffffffu, incl, o);
			if (lane >= (unsigned) o) incl += y;
		}
		if (lane == 31) s_w[warp] = incl;
		__syncthreads();
		unsigned long long before = run + incl - v;
		unsigned long long tile = 0;
		for (unsigned w = 0; w < 8; w++) { if (w < warp) before += s_w[w]; tile += s_w[w]; }
		if (b < b1) block_counts[b * P + p] = before;
		run += tile;
		__syncthreads();
	}
}

int partition_scan_blocks(CgContext *ctx, unsigned long long *d_block, unsigned long long *d_tot, int64_t nblocks, int P, CgAsyncBuf *scratch)
{
	const int nchunks = (int) ((nblocks + CGP_SCAN_CHUNK - 1) / CGP_SCAN_CHUNK);
	CG_CUDA(scratch->alloc(sizeof(unsigned long long) * (size_t) P * (size_t) std::max(nchunks, 1), ctx->compute));
	unsigned long long *d_chunks = scratch->as<unsigned long long>();
	cg_partition_scan_sum_kernel<<<(unsigned) (P * nchunks), 256, 0, ctx->compute>>>(d_block, d_chunks, nblocks, P, nchunks);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	cg_partition_scan_chunks_kernel<<<(P + 127) / 128, 128, 0, ctx->compute>>>(d_chunks, d_tot, P, nchunks);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	cg_partition_scan_apply_kernel<<<(unsigned) (P * nchunks), 256, 0, ctx->compute>>>(d_block, d_chunks, nblocks, P, nchunks);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

__global__ void cg_partition_base_kernel(const unsigned long long *totals, unsigned long long *base, int P)
{
	if (threadIdx.x == 0 && blockIdx.x == 0)
	{
		unsigned long long run = 0;
		for (int p = 0; p < P; p++) { base[p] = run; run += totals[p]; }
		base[P] = run;
	}
}

__global__ void cg_block_count_kernel(const int32_t *index, const int32_t *order, int64_t n, int P, unsigned long long *block_counts)
{
	extern __shared__ unsigned int s_count[];
	for (int p = threadIdx.x; p < P; p += CGP_THREADS) s_count[p] = 0;
	__syncthreads();
	int64_t base = (int64_t) blockIdx.x * CGP_ROWS_PER_BLOCK;
	for (int i = threadIdx.x; i < CGP_ROWS_PER_BLOCK; i += CGP_THREADS)
	{
		int64_t r = base + i;
		if (r >= n) break;
		int idx = index[r];
		if (order) idx = order[idx];
		atomicAdd(&s_count[idx], 1u);
	}
	__syncthreads();
	for (int p = threadIdx.x; p < P; p += CGP_THREADS) block_counts[(uint64_t) blockIdx.x * P + p] = s_count[p];
}

/* routing + scatter without an index array (the repartition exchange): d_counts[P] rows per partition and d_counts[P] =
 * rows whose hash lies in no interval are ready on the compute stream after the first kernel; the caller records an
 * event between the two phases through `after_counts` */
int cg_partition_route_scatter_async(const int64_t *d_keys, const uint8_t *d_nulls, int64_t n, int32_t key_len, int32_t by_hash,
									 const int32_t *mins, const int32_t *maxs, int32_t P, const int32_t *h_order,
									 const int64_t *const *d_cols, int32_t ncols, int64_t *const *d_out, int64_t *d_counts,
									 cudaEvent_t after_counts, const CgScatterHook *peer_hook)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (P <= 0 || P > CGP_MAX_P) return cg_set_error(CG_EINVAL, "bad partition count %d", P);
	if (key_len != 4 && key_len != 8) return cg_set_error(CG_EINVAL, "key_len must be 4 or 8");
	if (ncols < 1 || ncols > 8 || n < 0 || !d_counts || !mins || !maxs || !h_order) return cg_set_error(CG_EINVAL, "bad argument");
	const int64_t nblocks = (n + CGP_ROWS_PER_BLOCK - 1) / CGP_ROWS_PER_BLOCK;
	CgAsyncBuf block_buf, tot_buf, idx_buf, chunk_buf;
	CG_CUDA(block_buf.alloc(sizeof(unsigned long long) * (size_t) std::max<int64_t>(nblocks, 1) * P, ctx->compute));
	CG_CUDA(tot_buf.alloc(sizeof(unsigned long long) * (2 * P + 1), ctx->compute));
	CG_CUDA(idx_buf.alloc(sizeof(uint16_t) * (size_t) std::max<int64_t>(n, 1), ctx->compute));
	unsigned long long *d_block = block_buf.as<unsigned long long>(), *d_tot = tot_buf.as<unsigned long long>(), *d_base = d_tot + P;
	uint16_t *d_idx16 = idx_buf.as<uint16_t>();
	RouteParams R = {d_keys, d_nulls, key_len, by_hash};
	const void *d[3];
	const size_t pb = sizeof(int32_t) * P;
	if (int rc = upload_small(ctx, {{mins, pb}, {maxs, pb}, {h_order, pb}}, d)) return rc;
	R.mins = (const int32_t *) d[0]; R.maxs = (const int32_t *) d[1];
	const int32_t *d_order = (const int32_t *) d[2];
	detect_uniform(mins, maxs, P, &R);
	CG_CUDA(cudaMemsetAsync(d_tot, 0, sizeof(unsigned long long) * (2 * P + 1), ctx->compute));
	CG_CUDA(cudaMemsetAsync(d_counts, 0, sizeof(int64_t) * (P + 1), ctx->compute));
	if (n > 0)
	{
		cg_route_hist_kernel<<<(unsigned) nblocks, CGP_THREADS, 4 * P * sizeof(int32_t), ctx->compute>>>(R, n, P, d_order, d_idx16, d_block,
																										  (unsigned long long *) d_counts,
																										  (unsigned long long *) (d_counts + P));
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
	}
	if (after_counts) CG_CUDA(cudaEventRecord(after_counts, ctx->compute));
	if (n > 0)
	{
		int src_ = partition_scan_blocks(ctx, d_block, d_tot, nblocks, P, &chunk_buf);
		if (src_) return src_;
		cg_partition_base_kernel<<<1, 32, 0, ctx->compute>>>(d_tot, d_base, P);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
		StagedScatterParams S;
		memset(&S, 0, sizeof S);
		S.index = d_idx16; S.n = n; S.P = P; S.ncols = ncols; S.block_offsets = d_block; S.part_base = d_base; S.order = nullptr;
		for (int c = 0; c < ncols; c++) { S.cols[c] = d_cols[c]; S.out[c] = d_out ? d_out[c] : nullptr; }
		static bool smem_configured = false;
		if (!smem_configured)
		{
			CG_CUDA(cudaFuncSetAttribute(cg_scatter_staged_kernel<uint16_t, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) staged_scatter_smem(CGP_MAX_P)));
			CG_CUDA(cudaFuncSetAttribute(cg_scatter_staged_kernel<uint16_t, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) staged_scatter_smem(CGP_MAX_P, true)));
			smem_configured = true;
		}
		if (peer_hook)
		{
			CgPeerScatter B;
			memset(&B, 0, sizeof B);
			int hrc = peer_hook->fn(peer_hook->arg, &B);     /* the host learns every rank's counts here; the kernels above keep running */
			if (hrc) return hrc;
			cg_scatter_staged_kernel<uint16_t, true><<<(unsigned) nblocks, CGP_THREADS, staged_scatter_smem(P, true), ctx->compute>>>(S, B);
		}
		else
		{
			static const CgPeerScatter no_peer = {};
			cg_scatter_staged_kernel<uint16_t, false><<<(unsigned) nblocks, CGP_THREADS, staged_scatter_smem(P), ctx->compute>>>(S, no_peer);
		}
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
	}
	else if (peer_hook)
	{
		CgPeerScatter B;
		int hrc = peer_hook->fn(peer_hook->arg, &B);         /* no local rows: the counts are still exchanged (a collective) */
		if (hrc) return hrc;
	}
	return CG_OK;
}

extern "C" int cg_partition_scatter_ordered(const int32_t *d_index, int64_t n, int32_t P, const int32_t *h_order,
											const int64_t *const *d_cols, int32_t ncols, int64_t *const *d_out,
											int64_t *h_offsets)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (!h_offsets) return cg_set_error(CG_EINVAL, "NULL offsets");
	if (P <= 0 || P > CGP_MAX_P) return cg_set_error(CG_EINVAL, "bad partition count %d", P);
	if (ncols < 0 || ncols > 8) return cg_set_error(CG_EUNSUPPORTED, "at most 8 payload columns per call");
	if (n < 0) return cg_set_error(CG_EINVAL, "negative row count");
	if (h_order)
	{
		std::vector<uint8_t> seen(P, 0);
		for (int p = 0; p < P; p++)
		{
			if (h_order[p] < 0 || h_order[p] >= P || seen[h_order[p]]) return cg_set_error(CG_EINVAL, "order is not a permutation");
			seen[h_order[p]] = 1;
		}
	}
	int64_t nblocks = (n + CGP_ROWS_PER_BLOCK - 1) / CGP_ROWS_PER_BLOCK;
	CgAsyncBuf block_buf, tot_buf, chunk_buf;
	CG_CUDA(block_buf.alloc(sizeof(unsigned long long) * (size_t) std::max<int64_t>(nblocks, 1) * P, ctx->compute));
	CG_CUDA(tot_buf.alloc(sizeof(unsigned long long) * (2 * P + 1), ctx->compute));
	unsigned long long *d_block = block_buf.as<unsigned long long>(), *d_tot = tot_buf.as<unsigned long long>();
	unsigned long long *d_base = d_tot + P;
	CG_CUDA(cudaMemsetAsync(d_tot, 0, sizeof(unsigned long long) * (2 * P + 1), ctx->compute));
	const int32_t *d_order = nullptr;
	if (h_order)
	{
		const void *d;
		if (int rc = upload_small(ctx, {{h_order, sizeof(int32_t) * P}}, &d)) return rc;
		d_order = (const int32_t *) d;
	}
	if (n > 0)
	{
		cg_block_count_kernel<<<(unsigned) nblocks, CGP_THREADS, P * sizeof(unsigned int), ctx->compute>>>(d_index, d_order, n, P, d_block);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
		int src_ = partition_scan_blocks(ctx, d_block, d_tot, nblocks, P, &chunk_buf);
		if (src_) return src_;
		cg_partition_base_kernel<<<1, 32, 0, ctx->compute>>>(d_tot, d_base, P);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
		StagedScatterParams S;
		memset(&S, 0, sizeof S);
		S.index = d_index; S.n = n; S.P = P; S.ncols = ncols; S.block_offsets = d_block; S.part_base = d_base; S.order = d_order;
		for (int c = 0; c < ncols; c++) { S.cols[c] = d_cols[c]; S.out[c] = d_out[c]; }
		static bool smem_configured = false;
		if (!smem_configured)
		{
			CG_CUDA(cudaFuncSetAttribute(cg_scatter_staged_kernel<int32_t, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) staged_scatter_smem(CGP_MAX_P)));
			smem_configured = true;
		}
		static const CgPeerScatter no_peer = {};
		cg_scatter_staged_kernel<int32_t, false><<<(unsigned) nblocks, CGP_THREADS, staged_scatter_smem(P), ctx->compute>>>(S, no_peer);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
	}
	std::vector<unsigned long long> base(P + 1, 0);
	CG_CUDA(cudaMemcpyAsync(base.data(), d_base, sizeof(unsigned long long) * (P + 1), cudaMemcpyDeviceToHost, ctx->compute));
	CG_CUDA(cudaStreamSynchronize(ctx->compute));
	for (int p = 0; p <= P; p++) h_offsets[p] = (int64_t) base[p];
	return CG_OK;
}

extern "C" int cg_partition_scatter(const int32_t *d_index, int64_t n, int32_t P, const int64_t *const *d_cols,
									int32_t ncols, int64_t *const *d_out, int64_t *h_offsets)
{
	return cg_partition_scatter_ordered(d_index, n, P, nullptr, d_cols, ncols, d_out, h_offsets);
}

/* ------------------------------------------------------------------------------ *
 *  Return rows of worker_partition_query_result: (partition_index, rows_written,
 *  bytes_written), executor/partitioned_intermediate_results.c:270-291.  bytes_written is what
 *  the partition's file would hold in PostgreSQL's COPY format as TaskFileDestReceiver writes it
 *  (worker/worker_sql_task_protocol.c:91-251, commands/multi_copy.c AppendCopyRowData /
 *  AppendCopyBinaryHeaders / AppendCopyBinaryFooters):
 *    text   fields separated by '\t', row ended by '\n', NULL as "\N", integers in decimal
 *    binary 19-byte header ("PGCOPY\n\377\r\n\0" + int32 flags + int32 extension length) when the
 *           receiver starts, per row int16 field count + per field int32 length and the value
 *           bytes (NULL: length -1 and no bytes), int16 -1 trailer at shutdown
 *  With lazy start-up (generate_empty_results = false, :234) a partition that receives no row
 *  never starts its receiver: 0 bytes.  The rows themselves stay on the GPU (NCCL instead of
 *  files); only these counters are computed.
 * ------------------------------------------------------------------------------ */
__constant__ unsigned long long cg_pow10[20] = {1ull, 10ull, 100ull, 1000ull, 10000ull, 100000ull, 1000000ull, 10000000ull, 100000000ull,
												1000000000ull, 10000000000ull, 100000000000ull, 1000000000000ull, 10000000000000ull,
												100000000000000ull, 1000000000000000ull, 10000000000000000ull, 100000000000000000ull,
												1000000000000000000ull, 10000000000000000000ull};

__device__ __forceinline__ unsigned int decimal_text_len(int64_t v)
{
	/* strlen of pg_lltoa(v): digits + 1 for '-' */
	unsigned long long a = v < 0 ? 0ull - (unsigned long long) v : (unsigned long long) v;
	unsigned int bits = 64u - (unsigned int) __clzll((long long) (a | 1ull));
	unsigned int t = (bits * 1233u) >> 12;             /* floor(log10(2^bits)) or one less */
	unsigned int digits = t + (a >= cg_pow10[t] ? 1u : 0u);
	if (digits == 0) digits = 1;
	return digits + (v < 0 ? 1u : 0u);
}

/* the rows of both COPY entry points (cg_partition_copy_bytes, cg_partition_copy_serialize); row_len and the fields
 * after it are the serializer's */
struct CopyParams
{
	const int32_t *index;
	int64_t n;
	int32_t P, ncols, binary;
	const int64_t *cols[CGP_MAX_COLS];
	const uint8_t *nulls[CGP_MAX_COLS];
	int32_t len[CGP_MAX_COLS];
	uint32_t *row_len;                         /* [n] */
	unsigned long long *block_bytes;           /* [nblocks][P]: bytes of the block's rows per partition, then their start offsets */
	const unsigned long long *file_start;      /* [P]: offset of the first ROW byte of partition p in the output */
	uint8_t *out;
};

__device__ __forceinline__ unsigned int copy_row_len(const CopyParams &A, int64_t r)
{
	unsigned int b = A.binary ? 2u : 0u;
	for (int c = 0; c < A.ncols; c++)
	{
		bool isnull = A.nulls[c] && A.nulls[c][r];
		if (A.binary) b += 4u + (isnull ? 0u : (unsigned int) A.len[c]);
		else b += 1u + (isnull ? 2u : decimal_text_len(A.cols[c][r]));
	}
	return b;
}

/* the row description from either COPY entry point's arguments */
static CopyParams copy_params(const int32_t *d_index, int64_t n, int32_t P, const int64_t *const *d_cols, const uint8_t *const *d_nulls,
							  const int32_t *col_len, int32_t ncols, int32_t binary)
{
	CopyParams A;
	memset(&A, 0, sizeof A);
	A.index = d_index; A.n = n; A.P = P; A.ncols = ncols; A.binary = binary ? 1 : 0;
	for (int c = 0; c < ncols; c++) { A.cols[c] = d_cols[c]; A.nulls[c] = d_nulls ? d_nulls[c] : nullptr; A.len[c] = col_len[c]; }
	return A;
}

__global__ void __launch_bounds__(CGP_THREADS)
cg_partition_copy_bytes_kernel(const __grid_constant__ CopyParams A, unsigned long long *bytes, unsigned long long *rows)
{
	extern __shared__ unsigned int s_copy[];            /* [P] bytes, [P] rows of this block (< 2^32: 4096 rows) */
	unsigned int *s_bytes = s_copy, *s_rows = s_copy + A.P;
	for (int p = threadIdx.x; p < 2 * A.P; p += CGP_THREADS) s_copy[p] = 0;
	__syncthreads();
	int64_t base = (int64_t) blockIdx.x * CGP_ROWS_PER_BLOCK;
	for (int i = threadIdx.x; i < CGP_ROWS_PER_BLOCK; i += CGP_THREADS)
	{
		int64_t r = base + i;
		if (r >= A.n) break;
		int p = A.index[r];
		atomicAdd(&s_bytes[p], copy_row_len(A, r));
		atomicAdd(&s_rows[p], 1u);
	}
	__syncthreads();
	for (int p = threadIdx.x; p < A.P; p += CGP_THREADS)
	{
		if (s_rows[p])
		{
			atomicAdd(bytes + p, (unsigned long long) s_bytes[p]);
			atomicAdd(rows + p, (unsigned long long) s_rows[p]);
		}
	}
}

extern "C" int cg_partition_copy_bytes(const int32_t *d_index, int64_t n, int32_t P, const int64_t *const *d_cols,
									   const uint8_t *const *d_nulls, const int32_t *col_len, int32_t ncols, int32_t binary,
									   int32_t generate_empty_results, int64_t *rows_written, int64_t *bytes_written)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (P < 1 || P > CGP_MAX_P) return cg_set_error(CG_EINVAL, "partition count %d out of range", P);
	if (ncols < 1 || ncols > CGP_MAX_COLS) return cg_set_error(CG_EUNSUPPORTED, "1..%d columns", CGP_MAX_COLS);
	if (n < 0 || !d_cols || !col_len || !rows_written || !bytes_written) return cg_set_error(CG_EINVAL, "bad argument");
	CgAsyncBuf acc_buf;
	CG_CUDA(acc_buf.alloc(2 * (size_t) P * sizeof(unsigned long long), ctx->compute));
	unsigned long long *d_acc = acc_buf.as<unsigned long long>();
	CG_CUDA(cudaMemsetAsync(d_acc, 0, 2 * (size_t) P * sizeof(unsigned long long), ctx->compute));
	if (n > 0)
	{
		const CopyParams A = copy_params(d_index, n, P, d_cols, d_nulls, col_len, ncols, binary);
		int64_t nblocks = (n + CGP_ROWS_PER_BLOCK - 1) / CGP_ROWS_PER_BLOCK;
		cg_partition_copy_bytes_kernel<<<(unsigned) nblocks, CGP_THREADS, 2 * P * sizeof(unsigned int), ctx->compute>>>(A, d_acc, d_acc + P);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
	}
	std::vector<unsigned long long> h(2 * (size_t) P, 0);
	CG_CUDA(cudaMemcpyAsync(h.data(), d_acc, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->compute));
	CG_CUDA(cudaStreamSynchronize(ctx->compute));
	for (int p = 0; p < P; p++)
	{
		rows_written[p] = (int64_t) h[P + p];
		int64_t b = (int64_t) h[p];
		if (binary && (h[P + p] > 0 || generate_empty_results)) b += 19 + 2;   /* header at start-up, trailer at shutdown */
		bytes_written[p] = b;
	}
	return CG_OK;
}

/* ------------------------------------------------------------------------------ *
 *  R18: the partition files themselves.  TaskFileDestReceiver (worker/worker_sql_task_protocol.c:91-251) appends every
 *  row of a partition, in arrival order, to that partition's file in PostgreSQL's COPY format (commands/multi_copy.c
 *  AppendCopyRowData / AppendCopyBinaryHeaders / AppendCopyBinaryFooters):
 *    text    fields separated by '\t', row ended by '\n', NULL as "\N", integers in decimal (pg_lltoa)
 *    binary  "PGCOPY\n\377\r\n\0" + int32 flags 0 + int32 extension length 0, then per row int16 field count and per
 *            field int32 length (-1 = NULL) + the value in network byte order, then int16 -1
 *  Here every row's byte length is known before anything is written (copy_row_len), so a row's place in its file is a
 *  segmented prefix sum in input order -- per block and partition (shared memory), across blocks (partition_scan_blocks),
 *  inside a warp step (peers of the same partition to the left) -- and all rows are
 *  formatted in parallel straight into one device buffer that holds the P files back to back.
 * ------------------------------------------------------------------------------ */
__global__ void __launch_bounds__(CGP_THREADS)
cg_copy_len_kernel(const __grid_constant__ CopyParams A)
{
	extern __shared__ unsigned int s_bytes[];            /* [P] */
	for (int p = threadIdx.x; p < A.P; p += CGP_THREADS) s_bytes[p] = 0;
	__syncthreads();
	int64_t base = (int64_t) blockIdx.x * CGP_ROWS_PER_BLOCK;
	for (int i = threadIdx.x; i < CGP_ROWS_PER_BLOCK; i += CGP_THREADS)
	{
		int64_t r = base + i;
		if (r >= A.n) break;
		unsigned int b = copy_row_len(A, r);
		A.row_len[r] = b;
		atomicAdd(&s_bytes[A.index[r]], b);
	}
	__syncthreads();
	for (int p = threadIdx.x; p < A.P; p += CGP_THREADS) A.block_bytes[(uint64_t) blockIdx.x * A.P + p] = s_bytes[p];
}

__device__ __forceinline__ uint8_t *put_be(uint8_t *p, uint64_t v, int bytes)
{
	for (int i = bytes - 1; i >= 0; i--) *p++ = (uint8_t) (v >> (8 * i));
	return p;
}

__device__ __forceinline__ uint8_t *put_decimal(uint8_t *p, int64_t v)
{
	unsigned long long a = v < 0 ? 0ull - (unsigned long long) v : (unsigned long long) v;
	if (v < 0) *p++ = '-';
	unsigned int digits = decimal_text_len(v) - (v < 0 ? 1u : 0u);
	for (int i = (int) digits - 1; i >= 0; i--) { p[i] = (uint8_t) ('0' + a % 10ull); a /= 10ull; }
	return p + digits;
}

__global__ void __launch_bounds__(CGP_THREADS)
cg_copy_write_kernel(const __grid_constant__ CopyParams A)
{
	extern __shared__ unsigned long long s_run[];        /* [warps][P] running byte offsets */
	constexpr int WARPS = CGP_THREADS / 32;
	constexpr int SEG = CGP_ROWS_PER_BLOCK / WARPS;
	const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned long long *mine = s_run + warp * A.P;
	for (int p = lane; p < A.P; p += 32) mine[p] = 0;
	__syncwarp();
	const int64_t seg0 = (int64_t) blockIdx.x * CGP_ROWS_PER_BLOCK + (int64_t) warp * SEG;
	/* pass A: bytes of this warp's segment per partition (the row of shared memory is warp-private) */
	for (int step = 0; step < SEG; step += 32)
	{
		int64_t r = seg0 + step + lane;
		int idx = r < A.n ? A.index[r] : -1;
		unsigned int len = r < A.n ? A.row_len[r] : 0u;
		unsigned peers = __match_any_sync(0xffffffffu, idx);
		unsigned int total = 0;
		for (int src = 0; src < 32; src++)
		{
			unsigned int v = __shfl_sync(0xffffffffu, len, src);
			if ((peers >> src) & 1u) total += v;
		}
		if (idx >= 0 && lane == (unsigned) (__ffs(peers) - 1)) mine[idx] += total;
		__syncwarp();
	}
	__syncthreads();
	for (int p = threadIdx.x; p < A.P; p += CGP_THREADS)
	{
		unsigned long long run = A.file_start[p] + A.block_bytes[(uint64_t) blockIdx.x * A.P + p];
		for (int w = 0; w < WARPS; w++)
		{
			unsigned long long c = s_run[w * A.P + p];
			s_run[w * A.P + p] = run;
			run += c;
		}
	}
	__syncthreads();
	/* pass B: format every row at its place */
	for (int step = 0; step < SEG; step += 32)
	{
		int64_t r = seg0 + step + lane;
		int idx = r < A.n ? A.index[r] : -1;
		unsigned int len = r < A.n ? A.row_len[r] : 0u;
		unsigned peers = __match_any_sync(0xffffffffu, idx);
		unsigned int before = 0, total = 0;
		for (int src = 0; src < 32; src++)
		{
			unsigned int v = __shfl_sync(0xffffffffu, len, src);
			if ((peers >> src) & 1u) { total += v; if ((unsigned) src < lane) before += v; }
		}
		if (idx >= 0)
		{
			uint8_t *p = A.out + mine[idx] + before;
			if (A.binary)
			{
				p = put_be(p, (uint64_t) A.ncols, 2);
				for (int c = 0; c < A.ncols; c++)
				{
					if (A.nulls[c] && A.nulls[c][r]) p = put_be(p, 0xffffffffull, 4);
					else { p = put_be(p, (uint64_t) A.len[c], 4); p = put_be(p, (uint64_t) A.cols[c][r], A.len[c]); }
				}
			}
			else
				for (int c = 0; c < A.ncols; c++)
				{
					if (A.nulls[c] && A.nulls[c][r]) { *p++ = '\\'; *p++ = 'N'; }
					else p = put_decimal(p, A.cols[c][r]);
					*p++ = (c + 1 < A.ncols) ? '\t' : '\n';
				}
		}
		__syncwarp();
		if (idx >= 0 && lane == (unsigned) (__ffs(peers) - 1)) mine[idx] += total;
		__syncwarp();
	}
}

__global__ void cg_copy_frame_kernel(uint8_t *out, const unsigned long long *file_begin, const unsigned long long *file_end, const uint8_t *present, int P)
{
	int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= P || !present[p]) return;
	const uint8_t sig[19] = {'P', 'G', 'C', 'O', 'P', 'Y', '\n', 0xff, '\r', '\n', 0, 0, 0, 0, 0, 0, 0, 0, 0};
	for (int i = 0; i < 19; i++) out[file_begin[p] + i] = sig[i];
	out[file_end[p] - 2] = 0xff; out[file_end[p] - 1] = 0xff;
}

extern "C" int cg_partition_copy_serialize(const int32_t *d_index, int64_t n, int32_t P, const int64_t *const *d_cols,
										   const uint8_t *const *d_nulls, const int32_t *col_len, int32_t ncols, int32_t binary,
										   int32_t generate_empty_results, uint8_t *d_out, int64_t out_capacity,
										   int64_t *file_offsets /* [P + 1] */)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (P < 1 || P > CGP_MAX_P) return cg_set_error(CG_EINVAL, "partition count %d out of range", P);
	if (ncols < 1 || ncols > CGP_MAX_COLS) return cg_set_error(CG_EUNSUPPORTED, "1..%d columns", CGP_MAX_COLS);
	if (n < 0 || !d_cols || !col_len || !file_offsets) return cg_set_error(CG_EINVAL, "bad argument");
	for (int c = 0; c < ncols; c++)
		if (binary && col_len[c] != 2 && col_len[c] != 4 && col_len[c] != 8) return cg_set_error(CG_EUNSUPPORTED, "binary width %d", col_len[c]);
	const int64_t nblocks = (n + CGP_ROWS_PER_BLOCK - 1) / CGP_ROWS_PER_BLOCK;
	CgAsyncBuf len_buf, block_buf, tot_buf, chunk_buf;
	CG_CUDA(len_buf.alloc(sizeof(uint32_t) * (size_t) std::max<int64_t>(n, 1), ctx->compute));
	CG_CUDA(block_buf.alloc(sizeof(unsigned long long) * (size_t) std::max<int64_t>(nblocks, 1) * P, ctx->compute));
	CG_CUDA(tot_buf.alloc(sizeof(unsigned long long) * P, ctx->compute));
	unsigned long long *d_tot = tot_buf.as<unsigned long long>();
	CopyParams A = copy_params(d_index, n, P, d_cols, d_nulls, col_len, ncols, binary);
	A.row_len = len_buf.as<uint32_t>(); A.block_bytes = block_buf.as<unsigned long long>(); A.out = d_out;
	std::vector<unsigned long long> totals(P, 0);
	if (n > 0)
	{
		cg_copy_len_kernel<<<(unsigned) nblocks, CGP_THREADS, P * sizeof(unsigned int), ctx->compute>>>(A);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
		if (int rc = partition_scan_blocks(ctx, A.block_bytes, d_tot, nblocks, P, &chunk_buf)) return rc;
		CG_CUDA(cudaMemcpyAsync(totals.data(), d_tot, sizeof(unsigned long long) * P, cudaMemcpyDeviceToHost, ctx->compute));
		CG_CUDA(cudaStreamSynchronize(ctx->compute));
	}
	/* file layout: [header][rows][trailer] per partition, back to back; a partition without rows has no file content unless
	 * generate_empty_results (lazy start-up of the receivers, partitioned_intermediate_results.c:234) */
	std::vector<unsigned long long> begin(P), rows_at(P), end(P);
	std::vector<uint8_t> present(P);
	unsigned long long off = 0;
	for (int p = 0; p < P; p++)
	{
		present[p] = binary && (totals[p] > 0 || generate_empty_results);
		begin[p] = off;
		rows_at[p] = off + (present[p] ? 19 : 0);
		end[p] = rows_at[p] + totals[p] + (present[p] ? 2 : 0);
		off = end[p];
		file_offsets[p] = (int64_t) begin[p];
	}
	file_offsets[P] = (int64_t) off;
	if ((int64_t) off > out_capacity || (off > 0 && !d_out))
		return cg_set_error(CG_EINVAL, "the partition files need %llu bytes, the output buffer holds %lld", off, (long long) out_capacity);
	if (off == 0) return CG_OK;
	const size_t pb = sizeof(unsigned long long) * P;
	const void *d[4];
	if (int rc = upload_small(ctx, {{rows_at.data(), pb}, {begin.data(), pb}, {end.data(), pb}, {present.data(), (size_t) P}}, d)) return rc;
	A.file_start = (const unsigned long long *) d[0];
	const unsigned long long *d_begin = (const unsigned long long *) d[1], *d_end = (const unsigned long long *) d[2];
	const uint8_t *d_present = (const uint8_t *) d[3];
	if (n > 0)
	{
		static bool smem_configured = false;
		if (!smem_configured)
		{
			CG_CUDA(cudaFuncSetAttribute(cg_copy_write_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
										 (int) ((CGP_THREADS / 32) * CGP_MAX_P * sizeof(unsigned long long))));
			smem_configured = true;
		}
		cg_copy_write_kernel<<<(unsigned) nblocks, CGP_THREADS, (CGP_THREADS / 32) * P * sizeof(unsigned long long), ctx->compute>>>(A);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
	}
	if (binary)
	{
		cg_copy_frame_kernel<<<(P + 127) / 128, 128, 0, ctx->compute>>>(d_out, d_begin, d_end, d_present, P);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
	}
	CG_CUDA(cudaStreamSynchronize(ctx->compute));
	return CG_OK;
}
