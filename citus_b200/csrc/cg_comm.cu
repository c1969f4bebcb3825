/*
 * cg_comm.cu -- the exchange steps of the path, behind the C-ABI, over NCCL (NVLink 4 / NVSwitch).
 *
 * The reference moves partial results and repartitioned rows as libpq result rows and COPY files:
 *   executor/adaptive_executor.c:3964-4189 ReceiveResults  (one HeapTuple per partial row into the
 *       coordinator's tuplestore, then the combine query's HashAggregate,
 *       planner/multi_logical_optimizer.c:1807-1885, 2231-2275)
 *   executor/partitioned_intermediate_results.c:115-298 worker_partition_query_result  (P files per task)
 *   executor/intermediate_results.c:789-1045 fetch_intermediate_results / read_intermediate_results
 * Here one process drives one GPU (a PostgreSQL backend is one process), the per-GPU partial aggregates
 * and the partition-contiguous rows already sit in HBM, and the exchange is a collective on the library's
 * streams:
 *   cg_comm_combine               coord_combine of the commutative / associative built-ins: one ncclReduce of
 *                                 the accumulator array (the 8-byte packed words when nothing else was
 *                                 written) to the coordinator rank; row gather + merge kernel otherwise
 *   cg_comm_repartition_exchange  MAP_OUTPUT_FETCH: routing + scatter + one grouped ncclSend/ncclRecv of all
 *                                 columns, counts exchanged on the device side of a second stream
 * Peer window (one node, NVLink): every rank owns one cudaMalloc'ed window that all other ranks map with CUDA IPC.
 *   combine      the packed accumulator words are reduced by the ranks themselves: every rank stores slice s of its
 *                words into rank s's window, rank s sums the rows it received and stores the total into the
 *                coordinator rank's window (a reduce-scatter whose scatter target is one rank; stores only --
 *                a remote load is a round trip); two flag barriers in peer memory order it
 *   repartition  the scatter kernel stores every row straight into the receive buffer of the rank that owns the
 *                row's partition: routing, scatter and all-to-all are one pass, no send buffer, no second kernel
 * NCCL stays underneath for bootstrap (handles, counts, agreements) and as the path when IPC mapping is refused.
 * libnccl is resolved at first use (dlopen): a process that already carries a copy (torch bundles one) keeps
 * using that one; a CPU-only process never loads it.
 */
#include <dlfcn.h>
#include <nccl.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "cg_internal.h"

/* ---------------------------------------------------------------------------------- */
static struct NcclApi
{
	bool tried = false, ok = false;
	decltype(&ncclGetUniqueId) GetUniqueId;
	decltype(&ncclCommInitRank) CommInitRank;
	decltype(&ncclCommDestroy) CommDestroy;
	decltype(&ncclGetErrorString) GetErrorString;
	decltype(&ncclReduce) Reduce;
	decltype(&ncclAllReduce) AllReduce;
	decltype(&ncclAllGather) AllGather;
	decltype(&ncclSend) Send;
	decltype(&ncclRecv) Recv;
	decltype(&ncclGroupStart) GroupStart;
	decltype(&ncclGroupEnd) GroupEnd;
	decltype(&ncclGetVersion) GetVersion;
} g_nccl;

static bool load_nccl()
{
	if (g_nccl.tried) return g_nccl.ok;
	g_nccl.tried = true;
	void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);     /* the copy the process already has */
	if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
	if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
	if (!h) return false;
#define CG_NCCL_SYM(field, name) g_nccl.field = (decltype(g_nccl.field)) dlsym(h, name)
	CG_NCCL_SYM(GetUniqueId, "ncclGetUniqueId"); CG_NCCL_SYM(CommInitRank, "ncclCommInitRank"); CG_NCCL_SYM(CommDestroy, "ncclCommDestroy");
	CG_NCCL_SYM(GetErrorString, "ncclGetErrorString"); CG_NCCL_SYM(Reduce, "ncclReduce"); CG_NCCL_SYM(AllReduce, "ncclAllReduce");
	CG_NCCL_SYM(AllGather, "ncclAllGather"); CG_NCCL_SYM(Send, "ncclSend"); CG_NCCL_SYM(Recv, "ncclRecv");
	CG_NCCL_SYM(GroupStart, "ncclGroupStart"); CG_NCCL_SYM(GroupEnd, "ncclGroupEnd"); CG_NCCL_SYM(GetVersion, "ncclGetVersion");
#undef CG_NCCL_SYM
	g_nccl.ok = g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.CommDestroy && g_nccl.GetErrorString && g_nccl.Reduce &&
				g_nccl.AllReduce && g_nccl.AllGather && g_nccl.Send && g_nccl.Recv && g_nccl.GroupStart && g_nccl.GroupEnd;
	return g_nccl.ok;
}

#define CG_NCCL(call)                                                                                       \
	do {                                                                                                    \
		ncclResult_t r__ = (call);                                                                          \
		if (r__ != ncclSuccess)                                                                             \
			return cg_set_error(CG_ECOMM, "%s failed: %s (%s:%d)", #call, g_nccl.GetErrorString(r__), __FILE__, __LINE__); \
	} while (0)

#define CG_WIN_FLAG_BYTES 4096                       /* uint64 flags[8 kinds][CG_MAX_RANKS], kinds: 0 reduce-in, 1 reduce-out, 2 + slot exchange */
#define CG_WIN_WORDS ((size_t) 4 << 20)              /* 4 Mi packed words (32 MB) per direction */

struct PeerFlags
{
	unsigned long long *peer[CG_MAX_RANKS];          /* flag page of every rank (own included) */
	unsigned int *status;                            /* mapped host word: != 0 after a wait timed out */
	int me, nranks;
};

struct CgComm
{
	bool ready = false;
	int rank = 0, nranks = 1;
	/* peer window */
	bool win_ok = false;
	int use_peer = 1;                   /* cg_set_option("peer_window", 0) keeps everything on NCCL */
	uint8_t *win = nullptr;
	uint8_t *win_peer[CG_MAX_RANKS] = {};
	unsigned int *h_status = nullptr, *d_status = nullptr;
	unsigned long long epoch[8] = {};
	ncclComm_t comm = nullptr;
	cudaStream_t side = nullptr;        /* agreements and the repartition exchange: never behind the scans */
	int64_t *h_small = nullptr;         /* pinned */
	int64_t *d_small = nullptr;
	size_t small_words = 0;
	cudaEvent_t ev_scatter = nullptr, ev_index = nullptr;
	/* row gather of the combine */
	CgContext::DevBuf gather;
	/* repartition slots */
	struct Slot
	{
		CgContext::DevBuf send, recv, index;
		uint8_t *recv_peer[CG_MAX_RANKS] = {};   /* the receive buffers of all ranks, mapped here (peer window mode) */
		bool recv_shared = false;
		size_t recv_agreed = 0;                  /* bytes every rank's receive buffer has (the same everywhere) */
		cudaEvent_t done = nullptr, t0 = nullptr, t1 = nullptr;
		int64_t recv_rows = 0;
		int32_t ncols = 0;
		std::vector<int64_t> part_counts;   /* [nlocal][nranks] rows of each local partition by source rank */
		uint64_t sent_bytes = 0;
	};
	Slot slots[4];
};
static CgComm g_comm;

static int comm_ensure_small(size_t words)
{
	if (g_comm.small_words >= words) return CG_OK;
	if (g_comm.h_small) cudaFreeHost(g_comm.h_small);
	cudaFree(g_comm.d_small);
	g_comm.h_small = nullptr; g_comm.d_small = nullptr; g_comm.small_words = 0;
	size_t cap = std::max<size_t>(words, 4096);
	CG_CUDA(cudaHostAlloc((void **) &g_comm.h_small, cap * sizeof(int64_t), cudaHostAllocDefault));
	CG_CUDA(cudaMalloc((void **) &g_comm.d_small, cap * sizeof(int64_t)));
	g_comm.small_words = cap;
	return CG_OK;
}

static int devbuf_grow(CgContext::DevBuf *b, size_t bytes)
{
	if (b->cap >= bytes) return CG_OK;
	if (b->p) CG_CUDA(cudaFree(b->p));
	b->p = nullptr; b->cap = 0;
	size_t cap = bytes + bytes / 8 + 4096;
	if (cudaMalloc((void **) &b->p, cap) != cudaSuccess)
	{
		cudaGetLastError();
		return cg_set_error(CG_ENOMEM, "cudaMalloc of %zu bytes for an exchange buffer failed", cap);
	}
	b->cap = cap;
	return CG_OK;
}


static int comm_agree(int64_t *values, int n, ncclRedOp_t op);

/* ---------------------------------------------------------------------------------- *
 *  Peer window: CUDA IPC mappings of the other ranks' buffers, and barriers in them.
 * ---------------------------------------------------------------------------------- */
/* maps `mine` (the base of a cudaMalloc'ed allocation, or NULL when this rank has none) of every rank into this
 * process.  Collective.  *ok is the same on every rank: false leaves nothing mapped. */
static int comm_share(void *mine, uint8_t **peers, bool *ok)
{
	const int W = g_comm.nranks, me = g_comm.rank;
	*ok = false;
	for (int r = 0; r < CG_MAX_RANKS; r++) peers[r] = nullptr;
	cudaIpcMemHandle_t h;
	memset(&h, 0, sizeof h);
	int64_t good = 1;
	if (!mine || cudaIpcGetMemHandle(&h, mine) != cudaSuccess) { cudaGetLastError(); good = 0; }
	static_assert(sizeof(cudaIpcMemHandle_t) % sizeof(int64_t) == 0, "handle size");
	const size_t hw = sizeof(cudaIpcMemHandle_t) / sizeof(int64_t);
	int rc = comm_ensure_small(hw * (size_t) (W + 1));
	if (rc) return rc;
	memcpy(g_comm.h_small + hw * W, &h, sizeof h);
	CG_CUDA(cudaMemcpyAsync(g_comm.d_small + hw * W, g_comm.h_small + hw * W, sizeof h, cudaMemcpyHostToDevice, g_comm.side));
	CG_NCCL(g_nccl.AllGather(g_comm.d_small + hw * W, g_comm.d_small, hw, ncclInt64, g_comm.comm, g_comm.side));
	CG_CUDA(cudaMemcpyAsync(g_comm.h_small, g_comm.d_small, sizeof h * (size_t) W, cudaMemcpyDeviceToHost, g_comm.side));
	CG_CUDA(cudaStreamSynchronize(g_comm.side));
	std::vector<cudaIpcMemHandle_t> all(W);
	memcpy(all.data(), g_comm.h_small, sizeof h * (size_t) W);
	rc = comm_agree(&good, 1, ncclMin);
	if (rc) return rc;
	if (!good) return CG_OK;
	for (int r = 0; r < W; r++)
	{
		if (r == me) { peers[r] = (uint8_t *) mine; continue; }
		void *q = nullptr;
		if (cudaIpcOpenMemHandle(&q, all[r], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); good = 0; break; }
		peers[r] = (uint8_t *) q;
	}
	rc = comm_agree(&good, 1, ncclMin);
	if (rc) return rc;
	if (!good)
	{
		for (int r = 0; r < W; r++)
		{
			if (r != me && peers[r]) cudaIpcCloseMemHandle(peers[r]);
			peers[r] = nullptr;
		}
		cudaGetLastError();
		return CG_OK;
	}
	*ok = true;
	return CG_OK;
}

static void comm_unshare(uint8_t **peers)
{
	for (int r = 0; r < CG_MAX_RANKS; r++)
	{
		if (r != g_comm.rank && peers[r]) cudaIpcCloseMemHandle(peers[r]);
		peers[r] = nullptr;
	}
	cudaGetLastError();
}

__device__ __forceinline__ void st_release_sys(unsigned long long *p, unsigned long long v)
{
	asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long *p)
{
	unsigned long long v;
	asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
	return v;
}
__device__ __forceinline__ unsigned long long global_timer_ns()
{
	unsigned long long t;
	asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
	return t;
}

/* One warp.  Everything this rank's stream did before is visible to the ranks that see the flag; returns when every
 * rank has arrived at `epoch` of barrier `kind`.  Epochs only grow.  A wait that lasts 4 s gives up and raises the
 * status word: the host fails the next call instead of the GPU spinning for ever behind a rank that died. */
__global__ void cg_peer_barrier_kernel(const PeerFlags F, int kind, unsigned long long epoch)
{
	const int t = threadIdx.x;
	__threadfence_system();
	if (t < F.nranks)
	{
		st_release_sys(F.peer[t] + kind * CG_MAX_RANKS + F.me, epoch);
		const unsigned long long *flag = F.peer[F.me] + kind * CG_MAX_RANKS + t;
		const unsigned long long t0 = global_timer_ns();
		unsigned int polls = 0;
		while (ld_acquire_sys(flag) < epoch)
		{
			if ((++polls & 0x3ffu) == 0 && global_timer_ns() - t0 > 4000000000ull)      /* the timer is slow to read: rarely */
			{
				*(volatile unsigned int *) F.status = 1u + (unsigned) kind;
				break;
			}
		}
	}
	__threadfence_system();
}

__global__ void __launch_bounds__(256) cg_peer_copy_kernel(const unsigned long long *src, unsigned long long *dst, size_t words)
{
	const size_t stride = (size_t) gridDim.x * 256;
	for (size_t i = (size_t) blockIdx.x * 256 + threadIdx.x; i < words; i += stride) dst[i] = src[i];
}

/* All traffic between GPUs is stores (a remote store is posted; a remote load is a round trip):
 *   push     word i of this rank goes to the rank that owns slice i / chunk, into row `me` of that rank's input window
 *   reduce   the owner sums the nranks rows of its slice (local loads) and stores the total into the coordinator's
 *            output window */
struct PeerPush
{
	unsigned long long *in[CG_MAX_RANKS];            /* the input windows of all ranks: [nranks][chunk] words each */
	const unsigned long long *src;
	size_t words, chunk;                             /* this rank's words; slice length (even) */
	int me, nranks;
};

__global__ void __launch_bounds__(256) cg_peer_push_kernel(const __grid_constant__ PeerPush A)
{
	const size_t total = A.chunk * (size_t) A.nranks;
	const size_t stride = (size_t) gridDim.x * 512;
	for (size_t i = 2 * ((size_t) blockIdx.x * 256 + threadIdx.x); i < total; i += stride)
	{
		const unsigned long long a = i < A.words ? A.src[i] : 0ull, b = i + 1 < A.words ? A.src[i + 1] : 0ull;
		const size_t s = i / A.chunk;                /* chunk is even: both words have the same owner */
		unsigned long long *dst = A.in[s] + (size_t) A.me * A.chunk + (i - s * A.chunk);
		asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(a), "l"(b) : "memory");
	}
}

struct PeerReduce
{
	const unsigned long long *in;                    /* this rank's input window */
	unsigned long long *out;                         /* the coordinator's output window + this rank's slice begin */
	size_t chunk, len;                               /* row pitch; words of the slice that exist */
	int nranks;
};

__global__ void __launch_bounds__(256) cg_peer_reduce_kernel(const __grid_constant__ PeerReduce A)
{
	const size_t stride = (size_t) gridDim.x * 512;
	for (size_t j = 2 * ((size_t) blockIdx.x * 256 + threadIdx.x); j < A.len; j += stride)
	{
		unsigned long long a = 0, b = 0;
#pragma unroll 4
		for (int r = 0; r < A.nranks; r++)
		{
			unsigned long long x, y;             /* other GPUs wrote these words: not through L1 */
			asm volatile("ld.global.cg.v2.u64 {%0, %1}, [%2];" : "=l"(x), "=l"(y) : "l"(A.in + (size_t) r * A.chunk + j) : "memory");
			a += x; b += y;
		}
		asm volatile("st.global.v2.u64 [%0], {%1, %2};" ::"l"(A.out + j), "l"(a), "l"(b) : "memory");
	}
}

static PeerFlags comm_flags()
{
	PeerFlags F;
	memset(&F, 0, sizeof F);
	for (int r = 0; r < g_comm.nranks; r++) F.peer[r] = (unsigned long long *) g_comm.win_peer[r];
	F.status = g_comm.d_status; F.me = g_comm.rank; F.nranks = g_comm.nranks;
	return F;
}

static int comm_peer_barrier(int kind, cudaStream_t stream)
{
	const unsigned long long e = ++g_comm.epoch[kind];
	cg_peer_barrier_kernel<<<1, 32, 0, stream>>>(comm_flags(), kind, e);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}

static int comm_check_status()
{
	if (g_comm.h_status && *(volatile unsigned int *) g_comm.h_status)
		return cg_set_error(CG_ECOMM, "a wait on another rank in the peer window timed out (barrier kind %u)", *g_comm.h_status - 1u);
	return CG_OK;
}

static inline unsigned long long *win_in(int r) { return (unsigned long long *) (g_comm.win_peer[r] + CG_WIN_FLAG_BYTES); }
static inline unsigned long long *win_out(int r) { return win_in(r) + CG_WIN_WORDS; }

/* the window of this rank and its mappings everywhere: collective, at communicator start */
static int comm_window_setup()
{
	g_comm.win_ok = false;
	if (g_comm.nranks < 2 || g_comm.nranks > CG_MAX_RANKS) return CG_OK;
	const char *e = getenv("CG_PEER_WINDOW");
	int64_t want = (e && atoi(e) == 0) ? 0 : 1;
	int rc = comm_agree(&want, 1, ncclMin);
	if (rc) return rc;
	if (!want) return CG_OK;
	const size_t bytes = CG_WIN_FLAG_BYTES + 2 * CG_WIN_WORDS * sizeof(unsigned long long);
	if (cudaMalloc((void **) &g_comm.win, bytes) != cudaSuccess) { cudaGetLastError(); g_comm.win = nullptr; }
	if (g_comm.win)
	{
		CG_CUDA(cudaMemsetAsync(g_comm.win, 0, CG_WIN_FLAG_BYTES, g_comm.side));
		CG_CUDA(cudaStreamSynchronize(g_comm.side));
	}
	if (!g_comm.h_status)
	{
		CG_CUDA(cudaHostAlloc((void **) &g_comm.h_status, sizeof(unsigned int), cudaHostAllocMapped));
		*g_comm.h_status = 0;
		CG_CUDA(cudaHostGetDevicePointer((void **) &g_comm.d_status, g_comm.h_status, 0));
	}
	rc = comm_share(g_comm.win, g_comm.win_peer, &g_comm.win_ok);
	if (rc) return rc;
	if (!g_comm.win_ok && g_comm.win) { cudaFree(g_comm.win); g_comm.win = nullptr; }
	for (int k = 0; k < 8; k++) g_comm.epoch[k] = 0;
	return CG_OK;
}

/* 1 = peer window in use, 0 = NCCL only */
extern "C" int cg_comm_peer_window(void) { return g_comm.ready && g_comm.win_ok && g_comm.use_peer; }
void cg_comm_set_peer_window(int on) { g_comm.use_peer = on ? 1 : 0; }

extern "C" int cg_comm_unique_id(uint8_t *id)
{
	if (!id) return cg_set_error(CG_EINVAL, "NULL id");
	if (!load_nccl()) return cg_set_error(CG_ECOMM, "libnccl.so.2 is not available");
	static_assert(sizeof(ncclUniqueId) == CG_COMM_ID_BYTES, "ncclUniqueId size");
	ncclUniqueId u;
	CG_NCCL(g_nccl.GetUniqueId(&u));
	memcpy(id, &u, sizeof u);
	return CG_OK;
}

extern "C" int cg_comm_init(const uint8_t *id, int32_t rank, int32_t nranks)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (g_comm.ready) return cg_set_error(CG_EINVAL, "communicator already initialised (rank %d of %d)", g_comm.rank, g_comm.nranks);
	if (nranks < 1 || rank < 0 || rank >= nranks) return cg_set_error(CG_EINVAL, "rank %d of %d", rank, nranks);
	g_comm.rank = rank; g_comm.nranks = nranks;
	{
		/* highest priority: its few thread blocks are scheduled as soon as any scan block retires */
		int lo = 0, hi = 0;
		CG_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi));
		CG_CUDA(cudaStreamCreateWithPriority(&g_comm.side, cudaStreamNonBlocking, hi));
	}
	CG_CUDA(cudaEventCreateWithFlags(&g_comm.ev_scatter, cudaEventDisableTiming));
	CG_CUDA(cudaEventCreateWithFlags(&g_comm.ev_index, cudaEventDisableTiming));
	if (nranks > 1)
	{
		if (!id) return cg_set_error(CG_EINVAL, "NULL id");
		if (!load_nccl()) return cg_set_error(CG_ECOMM, "libnccl.so.2 is not available");
		ncclUniqueId u;
		memcpy(&u, id, sizeof u);
		CG_NCCL(g_nccl.CommInitRank(&g_comm.comm, nranks, u, rank));
		int rc = comm_window_setup();
		if (rc) return rc;
	}
	g_comm.ready = true;
	return CG_OK;
}

extern "C" int cg_comm_rank(int32_t *rank, int32_t *nranks)
{
	if (!g_comm.ready) return cg_set_error(CG_EINVAL, "cg_comm_init() has not been called");
	if (rank) *rank = g_comm.rank;
	if (nranks) *nranks = g_comm.nranks;
	return CG_OK;
}

extern "C" int cg_comm_destroy(void)
{
	if (!g_comm.ready) return CG_OK;
	cudaStreamSynchronize(g_comm.side);
	if (CgContext *ctx = cg_ctx()) cudaStreamSynchronize(ctx->compute);
	/* mappings of other ranks' memory go first; nobody frees what a peer may still have mapped */
	for (CgComm::Slot &s : g_comm.slots)
		if (s.recv_shared) { comm_unshare(s.recv_peer); s.recv_shared = false; }
	if (g_comm.win_ok) comm_unshare(g_comm.win_peer);
	if (g_comm.comm && g_comm.nranks > 1) { int64_t one = 1; comm_agree(&one, 1, ncclSum); }
	if (g_comm.win) cudaFree(g_comm.win);
	g_comm.win = nullptr; g_comm.win_ok = false;
	if (g_comm.h_status) cudaFreeHost(g_comm.h_status);
	g_comm.h_status = nullptr; g_comm.d_status = nullptr;
	if (g_comm.comm) g_nccl.CommDestroy(g_comm.comm);
	g_comm.comm = nullptr;
	for (CgComm::Slot &s : g_comm.slots)
	{
		cudaFree(s.send.p); cudaFree(s.recv.p); cudaFree(s.index.p);
		s.send = s.recv = s.index = CgContext::DevBuf();
		if (s.done) cudaEventDestroy(s.done);
		if (s.t0) cudaEventDestroy(s.t0);
		if (s.t1) cudaEventDestroy(s.t1);
		s.done = s.t0 = s.t1 = nullptr;
	}
	cudaFree(g_comm.gather.p); g_comm.gather = CgContext::DevBuf();
	if (g_comm.h_small) cudaFreeHost(g_comm.h_small);
	cudaFree(g_comm.d_small);
	g_comm.h_small = nullptr; g_comm.d_small = nullptr; g_comm.small_words = 0;
	cudaEventDestroy(g_comm.ev_scatter); cudaEventDestroy(g_comm.ev_index);
	cudaStreamDestroy(g_comm.side);
	g_comm.ready = false;
	return CG_OK;
}

/*
 * Small host-side agreement: values[i] <- op over ranks of values[i].  Runs on the side stream, so it never
 * queues behind scan kernels: the host of every rank learns the result while its GPU is still busy.
 */
static int comm_agree(int64_t *values, int n, ncclRedOp_t op)
{
	if (g_comm.nranks == 1) return CG_OK;
	int rc = comm_ensure_small((size_t) n);
	if (rc) return rc;
	memcpy(g_comm.h_small, values, sizeof(int64_t) * n);
	CG_CUDA(cudaMemcpyAsync(g_comm.d_small, g_comm.h_small, sizeof(int64_t) * n, cudaMemcpyHostToDevice, g_comm.side));
	CG_NCCL(g_nccl.AllReduce(g_comm.d_small, g_comm.d_small, (size_t) n, ncclInt64, op, g_comm.comm, g_comm.side));
	CG_CUDA(cudaMemcpyAsync(g_comm.h_small, g_comm.d_small, sizeof(int64_t) * n, cudaMemcpyDeviceToHost, g_comm.side));
	CG_CUDA(cudaStreamSynchronize(g_comm.side));
	memcpy(values, g_comm.h_small, sizeof(int64_t) * n);
	return CG_OK;
}

extern "C" int cg_comm_allreduce_i64(int64_t *values, int32_t n, int32_t op)
{
	if (!g_comm.ready) return cg_set_error(CG_EINVAL, "cg_comm_init() has not been called");
	if (!values || n < 0 || n > 4096) return cg_set_error(CG_EINVAL, "bad argument");
	ncclRedOp_t o = op == CG_COMM_SUM ? ncclSum : op == CG_COMM_MIN ? ncclMin : op == CG_COMM_MAX ? ncclMax : ncclNumOps;
	if (o == ncclNumOps) return cg_set_error(CG_EINVAL, "bad reduction op %d", op);
	return comm_agree(values, n, o);
}

/* all ranks' device work up to here is complete when the call returns on any rank */
extern "C" int cg_comm_barrier(void)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (!g_comm.ready) return cg_set_error(CG_EINVAL, "cg_comm_init() has not been called");
	CG_CUDA(cudaStreamSynchronize(ctx->compute));
	int64_t one = 1;
	int rc = comm_agree(&one, 1, ncclSum);
	if (rc) return rc;
	return CG_OK;
}

/* ---------------------------------------------------------------------------------- *
 *  Combine.
 * ---------------------------------------------------------------------------------- */
/* the words behind an accumulator array that travel with it: [0] rows pending in packed words,
 * [1 + b] number of ranks whose kernels raised error bit b */
__global__ void cg_comm_tail_write_kernel(uint64_t *tail, const unsigned long long *stats, int with_pending)
{
	if (threadIdx.x != 0 || blockIdx.x != 0) return;
	tail[0] = with_pending ? (uint64_t) (stats[CG_STAT_PACKED_ADDED] - stats[CG_STAT_PACKED_DRAINED]) : 0ull;
	const unsigned long long flags = stats[2];
	for (int b = 0; b < 8; b++) tail[1 + b] = (flags >> b) & 1ull;
	for (int b = 9; b < CG_COMM_TAIL; b++) tail[b] = 0;
}

__global__ void cg_comm_tail_absorb_kernel(uint64_t *tail, unsigned long long *stats, int with_pending)
{
	if (threadIdx.x != 0 || blockIdx.x != 0) return;
	if (with_pending) stats[CG_STAT_PACKED_ADDED] = stats[CG_STAT_PACKED_DRAINED] + tail[0];
	unsigned long long flags = 0;
	for (int b = 0; b < 8; b++) if (tail[1 + b]) flags |= 1ull << b;
	stats[2] |= flags;
	for (int b = 0; b < CG_COMM_TAIL; b++) tail[b] = 0;
}

extern "C" int cg_comm_combine(CgPartial *p, int32_t root, int32_t local_status)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (!g_comm.ready) return cg_set_error(CG_EINVAL, "cg_comm_init() has not been called");
	if (!p) return cg_set_error(CG_EINVAL, "NULL partial");
	if (root < 0 || root >= g_comm.nranks) return cg_set_error(CG_EINVAL, "root %d of %d ranks", root, g_comm.nranks);
	if (g_comm.nranks == 1) return local_status ? cg_set_error(local_status, "rank 0 failed before the combine") : CG_OK;

	bool additive = true;
	for (int w = 0; w < p->nwords; w++) if (p->wordop[w] != CG_WORD_ADD) additive = false;
	const bool dense = (p->mode == CG_MODE_DENSE || p->mode == CG_MODE_GLOBAL) && additive;

	if (!dense)
	{
		/* sparse keys or min/max words: compacted rows travel to the coordinator rank, which merges them
		 * (cg_merge_kernel).  The local partial is made current and checked first, so that what the ranks
		 * agree on includes every kernel-raised error. */
		int64_t nrows = 0;
		int st = local_status;
		if (st == 0) st = cg_partial_ngroups(p, &nrows);
		const size_t row_bytes = sizeof(int64_t) + sizeof(uint64_t) * (size_t) p->nwords + 8;   /* key + words + NULL flag (padded) */
		/* per rank: status, rows, and the key codec (composite codes of different bounds must not be merged) */
		int rc = comm_ensure_small((size_t) 3 * g_comm.nranks + 3);
		if (rc) return rc;
		g_comm.h_small[0] = st; g_comm.h_small[1] = nrows; g_comm.h_small[2] = (int64_t) cg_key_codec_id(&p->desc);
		CG_CUDA(cudaMemcpyAsync(g_comm.d_small, g_comm.h_small, 3 * sizeof(int64_t), cudaMemcpyHostToDevice, g_comm.side));
		CG_NCCL(g_nccl.AllGather(g_comm.d_small, g_comm.d_small + 3, 3, ncclInt64, g_comm.comm, g_comm.side));
		CG_CUDA(cudaMemcpyAsync(g_comm.h_small + 3, g_comm.d_small + 3, 3 * sizeof(int64_t) * g_comm.nranks, cudaMemcpyDeviceToHost, g_comm.side));
		CG_CUDA(cudaStreamSynchronize(g_comm.side));
		std::vector<int64_t> rows(g_comm.nranks);
		int failed = -1, failed_code = 0;
		bool same_codec = true;
		for (int r = 0; r < g_comm.nranks; r++)
		{
			rows[r] = g_comm.h_small[3 + 3 * r + 1];
			if (g_comm.h_small[3 + 3 * r] != 0 && failed < 0) { failed = r; failed_code = (int) g_comm.h_small[3 + 3 * r]; }
			if (g_comm.h_small[3 + 3 * r + 2] != g_comm.h_small[2]) same_codec = false;
		}
		if (failed >= 0)
		{
			if (failed == g_comm.rank) return failed_code;      /* own message is already set */
			return cg_set_error(failed_code, "rank %d failed before the combine (code %d)", failed, failed_code);
		}
		if (!same_codec) return cg_set_error(CG_EINVAL, "the partials of the ranks do not share one layout (group key codec)");
		/* layout of one rank's rows in the gather buffer: keys | words | nulls, each 16-byte aligned */
		auto seg = [&](int64_t n, size_t *off_words, size_t *off_nulls) {
			size_t k = ((size_t) n * sizeof(int64_t) + 15) & ~(size_t) 15;
			size_t w = ((size_t) n * p->nwords * sizeof(uint64_t) + 15) & ~(size_t) 15;
			size_t z = ((size_t) n + 15) & ~(size_t) 15;
			*off_words = k; *off_nulls = k + w;
			return k + w + z;
		};
		(void) row_bytes;
		if (g_comm.rank != root)
		{
			size_t ow, on;
			size_t bytes = seg(nrows, &ow, &on);
			rc = devbuf_grow(&g_comm.gather, std::max<size_t>(bytes, 64));
			if (rc) return rc;
			uint8_t *b = g_comm.gather.p;
			int64_t got = 0;
			rc = cg_partial_export_device(p, nrows, (int64_t *) b, b + on, (uint64_t *) (b + ow), &got);
			if (rc) return rc;
			if (nrows > 0)
			{
				CG_NCCL(g_nccl.Send(b, bytes, ncclUint8, root, g_comm.comm, ctx->compute));
			}
			return CG_OK;
		}
		size_t total = 0;
		std::vector<size_t> base(g_comm.nranks, 0);
		for (int r = 0; r < g_comm.nranks; r++)
		{
			if (r == root) continue;
			size_t ow, on;
			base[r] = total;
			total += seg(rows[r], &ow, &on);
		}
		rc = devbuf_grow(&g_comm.gather, std::max<size_t>(total, 64));
		if (rc) return rc;
		CG_NCCL(g_nccl.GroupStart());
		for (int r = 0; r < g_comm.nranks; r++)
		{
			if (r == root || rows[r] == 0) continue;
			size_t ow, on;
			size_t bytes = seg(rows[r], &ow, &on);
			ncclResult_t e = g_nccl.Recv(g_comm.gather.p + base[r], bytes, ncclUint8, r, g_comm.comm, ctx->compute);
			if (e != ncclSuccess) { g_nccl.GroupEnd(); return cg_set_error(CG_ECOMM, "ncclRecv failed: %s", g_nccl.GetErrorString(e)); }
		}
		CG_NCCL(g_nccl.GroupEnd());
		for (int r = 0; r < g_comm.nranks; r++)
		{
			if (r == root || rows[r] == 0) continue;
			size_t ow, on;
			seg(rows[r], &ow, &on);
			uint8_t *b = g_comm.gather.p + base[r];
			rc = cg_launch_merge(p, (const int64_t *) b, b + on, (const uint64_t *) (b + ow), rows[r], ctx->compute);
			if (rc) return rc;
		}
		return CG_OK;
	}

	/* identical direct-indexed layouts with additive words: agree (off the scan stream) on what to reduce */
	int rc = comm_check_status();
	if (rc) return rc;
	int64_t agree[5] = {local_status, p->wide_dirty ? 1 : 0, p->packed_dirty ? 1 : 0,
						(int64_t) (p->entries * 1000003ull + (uint64_t) p->stride * 31ull + (uint64_t) p->pack_shift + cg_key_codec_id(&p->desc)),
						(g_comm.win_ok && g_comm.use_peer) ? 0 : 1};
	int64_t lay_min = agree[3];
	rc = comm_agree(agree, 5, ncclMax);
	if (rc) return rc;
	if (agree[0] != 0)
	{
		if (local_status != 0) return local_status;
		return cg_set_error((int) agree[0], "another rank failed before the combine (code %d)", (int) agree[0]);
	}
	rc = comm_agree(&lay_min, 1, ncclMin);
	if (rc) return rc;
	if (lay_min != agree[3]) return cg_set_error(CG_EINVAL, "the partials of the ranks do not share one layout");
	const bool any_wide = agree[1] != 0, any_packed = agree[2] != 0, peer = agree[4] == 0;
	if (any_packed && !any_wide && p->d_packed)
	{
		/* every rank only wrote packed words: 8 bytes per group travel instead of the wide entry */
		uint64_t *tail = p->d_packed + p->entries;
		const size_t L = (size_t) p->entries + CG_COMM_TAIL;
		cg_comm_tail_write_kernel<<<1, 32, 0, ctx->compute>>>(tail, p->d_stats, 1);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
		const int W = g_comm.nranks, me = g_comm.rank;
		const size_t L2 = (L + 1) & ~(size_t) 1;
		const size_t chunk = (((L2 + W - 1) / W) + 1) & ~(size_t) 1;
		if (peer && chunk * W <= CG_WIN_WORDS)
		{
			/* the ranks reduce among themselves over NVLink: every rank pushes slice s of its words to rank s; barrier;
			 * rank s sums what it received into the coordinator's output window; barrier; the coordinator takes the total */
			PeerPush U;
			memset(&U, 0, sizeof U);
			for (int r = 0; r < W; r++) U.in[r] = win_in(r);
			U.src = (const unsigned long long *) p->d_packed; U.words = L; U.chunk = chunk; U.me = me; U.nranks = W;
			const unsigned push_grid = (unsigned) std::min<size_t>((chunk * W + 511) / 512, (size_t) ctx->sm_count * 8);
			cg_peer_push_kernel<<<push_grid, 256, 0, ctx->compute>>>(U);
			CG_CUDA(cudaGetLastError()); g_cg_launches++;
			rc = comm_peer_barrier(0, ctx->compute);
			if (rc) return rc;
			const size_t begin = std::min(L2, (size_t) me * chunk), end = std::min(L2, begin + chunk);
			if (end > begin)
			{
				PeerReduce A;
				memset(&A, 0, sizeof A);
				A.in = win_in(me); A.out = win_out(root) + begin; A.chunk = chunk; A.len = end - begin; A.nranks = W;
				const unsigned grid = (unsigned) std::min<size_t>((A.len + 511) / 512, (size_t) ctx->sm_count * 8);
				cg_peer_reduce_kernel<<<grid, 256, 0, ctx->compute>>>(A);
				CG_CUDA(cudaGetLastError()); g_cg_launches++;
			}
			rc = comm_peer_barrier(1, ctx->compute);
			if (rc) return rc;
			if (me == root)
			{
				const unsigned copy_grid = (unsigned) std::min<size_t>((L + 255) / 256, (size_t) ctx->sm_count * 8);
				cg_peer_copy_kernel<<<copy_grid, 256, 0, ctx->compute>>>(win_out(me), (unsigned long long *) p->d_packed, L);
				CG_CUDA(cudaGetLastError()); g_cg_launches++;
				cg_comm_tail_absorb_kernel<<<1, 32, 0, ctx->compute>>>(tail, p->d_stats, 1);
				CG_CUDA(cudaGetLastError()); g_cg_launches++;
				p->packed_dirty = true;
			}
			return CG_OK;
		}
		CG_NCCL(g_nccl.Reduce(p->d_packed, p->d_packed, (size_t) p->entries + CG_COMM_TAIL, ncclInt64, ncclSum, root, g_comm.comm, ctx->compute));
		if (g_comm.rank == root)
		{
			cg_comm_tail_absorb_kernel<<<1, 32, 0, ctx->compute>>>(tail, p->d_stats, 1);
			CG_CUDA(cudaGetLastError()); g_cg_launches++;
			p->packed_dirty = true;
		}
		return CG_OK;
	}
	rc = cg_launch_drain(p, ctx->compute);
	if (rc) return rc;
	uint64_t *tail = p->d_table + p->entries * (uint64_t) p->stride;
	cg_comm_tail_write_kernel<<<1, 32, 0, ctx->compute>>>(tail, p->d_stats, 0);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	CG_NCCL(g_nccl.Reduce(p->d_table, p->d_table, (size_t) (p->entries * (uint64_t) p->stride) + CG_COMM_TAIL, ncclInt64, ncclSum, root,
						  g_comm.comm, ctx->compute));
	if (g_comm.rank == root)
	{
		cg_comm_tail_absorb_kernel<<<1, 32, 0, ctx->compute>>>(tail, p->d_stats, 0);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
		p->wide_dirty = true;
	}
	return CG_OK;
}

/* ---------------------------------------------------------------------------------- *
 *  Repartition exchange.
 * ---------------------------------------------------------------------------------- */
/* partition p is owned by rank p mod nranks (the reference assigns merge tasks round-robin over the worker
 * nodes, planner/multi_physical_planner.c:4826-4950); positions in the send buffer are destination-major */
extern "C" int cg_comm_exchange_plan(int32_t P, int32_t nranks, int32_t rank, const int64_t *counts /* [nranks][P] */,
									 int32_t *position /* [P] */, int64_t *send_rows /* [nranks] */,
									 int64_t *recv_rows /* [nranks] */, int64_t *local_part_counts /* [nlocal][nranks] */,
									 int32_t *nlocal_out)
{
	if (P < 1 || nranks < 1 || rank < 0 || rank >= nranks || !position) return cg_set_error(CG_EINVAL, "bad exchange plan arguments");
	int pos = 0;
	for (int r = 0; r < nranks; r++)
		for (int p = r; p < P; p += nranks) position[p] = pos++;
	int nlocal = 0;
	for (int p = rank; p < P; p += nranks) nlocal++;
	if (nlocal_out) *nlocal_out = nlocal;
	if (!counts) return CG_OK;
	for (int r = 0; r < nranks; r++)
	{
		int64_t s = 0, v = 0;
		for (int p = r; p < P; p += nranks) s += counts[(size_t) rank * P + p];      /* what this rank routes to r */
		for (int p = rank; p < P; p += nranks) v += counts[(size_t) r * P + p];      /* what r routes to this rank */
		if (send_rows) send_rows[r] = s;
		if (recv_rows) recv_rows[r] = v;
	}
	if (local_part_counts)
	{
		int i = 0;
		for (int p = rank; p < P; p += nranks, i++)
			for (int r = 0; r < nranks; r++) local_part_counts[(size_t) i * nranks + r] = counts[(size_t) r * P + p];
	}
	return CG_OK;
}


/*
 * Where a rank's rows land when the scatter stores straight into the owners' receive buffers.  Pure host arithmetic
 * over the counts every rank holds after the count exchange (counts[r * P + p] = rows of partition p on rank r), so it
 * has a CPU test (tests/test_distributed_gloo.py).  The receive buffer of rank d holds, per column, the rows in
 * (source rank, local partition) order -- the layout the grouped ncclSend/ncclRecv path produces.  For this rank:
 *   pos_begin[d], pos_begin[d + 1]   the output positions (cg_comm_exchange_plan) that belong to rank d
 *   total[d]                         rows rank d receives = the column stride of its buffer
 *   adj[d]                           a row the local scatter would put at index i of the send order lands at adj[d] + i
 *                                    of rank d's column (rows of lower ranks come first, rows for lower ranks do not count)
 */
extern "C" int cg_comm_peer_plan(int32_t P, int32_t nranks, int32_t rank, const int64_t *counts, int32_t *pos_begin /* [nranks + 1] */,
								 int64_t *total /* [nranks] */, int64_t *adj /* [nranks] */)
{
	if (P < 1 || nranks < 1 || rank < 0 || rank >= nranks || !counts || !pos_begin || !total || !adj)
		return cg_set_error(CG_EINVAL, "bad peer plan arguments");
	std::vector<int64_t> M((size_t) nranks * nranks, 0);            /* M[r][d] rows rank r routes to rank d */
	for (int r = 0; r < nranks; r++)
		for (int p = 0; p < P; p++)
		{
			if (counts[(size_t) r * P + p] < 0) return cg_set_error(CG_EINVAL, "negative row count");
			M[(size_t) r * nranks + p % nranks] += counts[(size_t) r * P + p];
		}
	int64_t soff = 0;
	int pos = 0;
	for (int d = 0; d < nranks; d++)
	{
		int64_t roff = 0, t = 0;
		for (int r = 0; r < nranks; r++)
		{
			if (r < rank) roff += M[(size_t) r * nranks + d];
			t += M[(size_t) r * nranks + d];
		}
		total[d] = t;
		adj[d] = roff - soff;
		pos_begin[d] = pos;
		for (int p = d; p < P; p += nranks) pos++;
		soff += M[(size_t) rank * nranks + d];
	}
	pos_begin[nranks] = pos;
	return CG_OK;
}

/* ---- peer-window form of the exchange: the scatter stores into the owners' receive buffers ---- */
struct PeerExchange
{
	CgComm::Slot *S;
	int64_t *d_counts;
	int32_t P, ncols, nlocal;
	int64_t total_recv;
};

static int peer_exchange_hook(void *arg, CgPeerScatter *out)
{
	PeerExchange *X = (PeerExchange *) arg;
	CgComm::Slot &S = *X->S;
	CgContext *ctx = cg_ctx();
	const int W = g_comm.nranks, me = g_comm.rank, P = X->P;
	int rc = comm_ensure_small((size_t) (P + 1) * (W + 1) + 8);
	if (rc) return rc;
	CG_CUDA(cudaStreamWaitEvent(g_comm.side, g_comm.ev_index, 0));
	CG_NCCL(g_nccl.AllGather(X->d_counts, g_comm.d_small, (size_t) P + 1, ncclInt64, g_comm.comm, g_comm.side));
	CG_CUDA(cudaMemcpyAsync(g_comm.h_small, g_comm.d_small, sizeof(int64_t) * (P + 1) * W, cudaMemcpyDeviceToHost, g_comm.side));
	CG_CUDA(cudaStreamSynchronize(g_comm.side));
	/* every rank now holds every rank's counts: all of them take the same decisions below without talking again.
	 * Every rank has also passed its routing kernel, which its stream runs after whatever read this slot's previous
	 * contents: the receive buffers may be overwritten. */
	std::vector<int64_t> counts((size_t) W * P);
	int64_t unroutable = 0;
	for (int r = 0; r < W; r++)
	{
		memcpy(&counts[(size_t) r * P], g_comm.h_small + (size_t) r * (P + 1), sizeof(int64_t) * P);
		unroutable += g_comm.h_small[(size_t) r * (P + 1) + P];
	}
	if (unroutable)
		return cg_set_error(CG_EINVAL, "could not find shard for partition column value (%lld rows)", (long long) unroutable);
	std::vector<int64_t> total(W, 0), adj(W, 0);
	std::vector<int32_t> pos_begin(W + 1, 0);
	rc = cg_comm_peer_plan(P, W, me, counts.data(), pos_begin.data(), total.data(), adj.data());
	if (rc) return rc;
	int64_t need_rows = 0;
	for (int d = 0; d < W; d++) need_rows = std::max(need_rows, total[d]);
	const size_t need = (size_t) std::max<int64_t>(need_rows, 1) * sizeof(int64_t) * X->ncols;
	if (!S.recv_shared || need > S.recv_agreed)
	{
		/* one size for all ranks: grow together, map again.  Rare: the first exchange of a slot, or a larger table. */
		CG_CUDA(cudaStreamSynchronize(ctx->compute));
		if (S.recv_shared) { comm_unshare(S.recv_peer); S.recv_shared = false; }
		int64_t one = 1;
		rc = comm_agree(&one, 1, ncclSum);                       /* nobody frees while a peer still has the old buffer mapped */
		if (rc) return rc;
		if (S.recv.p) CG_CUDA(cudaFree(S.recv.p));
		S.recv = CgContext::DevBuf();
		const size_t cap = need + need / 8 + 4096;
		void *q = nullptr;
		if (cudaMalloc(&q, cap) != cudaSuccess) { cudaGetLastError(); q = nullptr; }
		bool ok = false;
		rc = comm_share(q, S.recv_peer, &ok);
		if (rc) return rc;
		if (!ok)
		{
			if (q) cudaFree(q);
			g_comm.win_ok = false;                                /* the next call takes the NCCL path */
			return cg_set_error(q ? CG_ECOMM : CG_ENOMEM, "a receive buffer of %zu bytes could not be %s on every rank", cap, q ? "mapped" : "allocated");
		}
		S.recv.p = (uint8_t *) q; S.recv.cap = cap;
		S.recv_shared = true; S.recv_agreed = cap;
	}
	std::vector<int64_t> send_rows(W), recv_rows(W);
	S.part_counts.assign((size_t) std::max(X->nlocal, 1) * W, 0);
	std::vector<int32_t> position(P);
	int nlocal = 0;
	cg_comm_exchange_plan(P, W, me, counts.data(), position.data(), send_rows.data(), recv_rows.data(), S.part_counts.data(), &nlocal);
	X->total_recv = total[me];
	S.recv_rows = total[me];
	S.ncols = X->ncols;
	S.sent_bytes = 0;
	memset(out, 0, sizeof *out);
	out->nranks = W;
	for (int d = 0; d < W; d++)
	{
		out->base[d] = (int64_t *) S.recv_peer[d];
		out->stride[d] = total[d];
		out->adj[d] = adj[d];
		out->pos_begin[d] = pos_begin[d];
		if (d != me) S.sent_bytes += (uint64_t) send_rows[d] * sizeof(int64_t) * X->ncols;
	}
	out->pos_begin[W] = pos_begin[W];
	CG_CUDA(cudaEventRecord(S.t0, ctx->compute));
	return CG_OK;
}

extern "C" int cg_comm_repartition_exchange(int32_t slot, const int64_t *const *d_cols, const uint8_t *d_key_nulls, int64_t n,
											int32_t ncols, int32_t key_len, int32_t P, const int32_t *mins, const int32_t *maxs,
											int64_t *recv_rows_out)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (!g_comm.ready) return cg_set_error(CG_EINVAL, "cg_comm_init() has not been called");
	if (slot < 0 || slot >= 4) return cg_set_error(CG_EINVAL, "slot %d", slot);
	if (ncols < 1 || ncols > 8 || !d_cols || n < 0) return cg_set_error(CG_EINVAL, "bad argument");
	CgComm::Slot &S = g_comm.slots[slot];
	const int W = g_comm.nranks, me = g_comm.rank;
	if (!S.done)
	{
		CG_CUDA(cudaEventCreateWithFlags(&S.done, cudaEventDisableTiming));
		CG_CUDA(cudaEventCreate(&S.t0));
		CG_CUDA(cudaEventCreate(&S.t1));
	}
	/* routing (hashint4/8 -> token ranges) + histogram, then the scatter into destination-major order, on the compute
	 * stream; the counts of every rank are exchanged on the side stream while the scatter runs */
	int rc = devbuf_grow(&S.index, (size_t) (P + 1) * sizeof(int64_t) + 64);
	if (rc) return rc;
	int64_t *d_counts = (int64_t *) S.index.p;
	std::vector<int32_t> position(P);
	int nlocal = 0;
	cg_comm_exchange_plan(P, W, me, nullptr, position.data(), nullptr, nullptr, nullptr, &nlocal);
	rc = comm_check_status();
	if (rc) return rc;
	if (W > 1 && g_comm.win_ok && g_comm.use_peer)
	{
		/* routing + histogram; counts of all ranks (side stream, while the offset scan runs); then ONE kernel that is
		 * both the scatter and the all-to-all: rows leave shared memory as runs into the owner's receive buffer */
		PeerExchange X;
		X.S = &S; X.d_counts = d_counts; X.P = P; X.ncols = ncols; X.nlocal = nlocal; X.total_recv = 0;
		CgScatterHook hook = {peer_exchange_hook, &X};
		rc = cg_partition_route_scatter_async(d_cols[0], d_key_nulls, n, key_len, 1, mins, maxs, P, position.data(), d_cols, ncols, nullptr,
											  d_counts, g_comm.ev_index, &hook);
		if (rc) return rc;
		rc = comm_peer_barrier(2 + slot, ctx->compute);          /* every rank's rows have landed everywhere */
		if (rc) return rc;
		CG_CUDA(cudaEventRecord(S.t1, ctx->compute));
		CG_CUDA(cudaEventRecord(S.done, ctx->compute));
		if (recv_rows_out) *recv_rows_out = X.total_recv;
		return CG_OK;
	}
	if (S.recv_shared)
	{
		/* the slot was used in peer-window mode before: its buffer goes back to being private */
		comm_unshare(S.recv_peer); S.recv_shared = false; S.recv_agreed = 0;
		int64_t one = 1;
		rc = comm_agree(&one, 1, ncclSum);
		if (rc) return rc;
	}
	/* one rank: the scatter's output IS the received table (no exchange); else it is the send buffer */
	rc = devbuf_grow(W == 1 ? &S.recv : &S.send, (size_t) std::max<int64_t>(n, 1) * sizeof(int64_t) * ncols);
	if (rc) return rc;
	std::vector<int64_t *> outs(ncols);
	for (int c = 0; c < ncols; c++) outs[c] = (int64_t *) (W == 1 ? S.recv.p : S.send.p) + (size_t) c * n;
	rc = cg_partition_route_scatter_async(d_cols[0], d_key_nulls, n, key_len, 1, mins, maxs, P, position.data(), d_cols, ncols, outs.data(),
										  d_counts, g_comm.ev_index);
	if (rc) return rc;
	CG_CUDA(cudaEventRecord(g_comm.ev_scatter, ctx->compute));
	/* (P counts + the "could not find shard" counter) of every rank */
	rc = comm_ensure_small((size_t) (P + 1) * (W + 1) + 8);
	if (rc) return rc;
	CG_CUDA(cudaStreamWaitEvent(g_comm.side, g_comm.ev_index, 0));
	if (W > 1)
		CG_NCCL(g_nccl.AllGather(d_counts, g_comm.d_small, (size_t) P + 1, ncclInt64, g_comm.comm, g_comm.side));
	else
		CG_CUDA(cudaMemcpyAsync(g_comm.d_small, d_counts, sizeof(int64_t) * (P + 1), cudaMemcpyDeviceToDevice, g_comm.side));
	CG_CUDA(cudaMemcpyAsync(g_comm.h_small, g_comm.d_small, sizeof(int64_t) * (P + 1) * W, cudaMemcpyDeviceToHost, g_comm.side));
	CG_CUDA(cudaStreamSynchronize(g_comm.side));               /* counts are on the host; the scatter keeps running */
	std::vector<int64_t> counts((size_t) W * P), send_rows(W), recv_rows(W);
	int64_t unroutable = 0;
	for (int r = 0; r < W; r++)
	{
		memcpy(&counts[(size_t) r * P], g_comm.h_small + (size_t) r * (P + 1), sizeof(int64_t) * P);
		unroutable += g_comm.h_small[(size_t) r * (P + 1) + P];
	}
	if (unroutable)         /* every rank sees the same counters: all fail together, nobody waits in the exchange */
		return cg_set_error(CG_EINVAL, "could not find shard for partition column value (%lld rows)", (long long) unroutable);
	S.part_counts.assign((size_t) std::max(nlocal, 1) * W, 0);
	cg_comm_exchange_plan(P, W, me, counts.data(), position.data(), send_rows.data(), recv_rows.data(), S.part_counts.data(), &nlocal);
	int64_t total_recv = 0;
	for (int r = 0; r < W; r++) total_recv += recv_rows[r];
	if (W > 1)
	{
		rc = devbuf_grow(&S.recv, (size_t) std::max<int64_t>(total_recv, 1) * sizeof(int64_t) * ncols);
		if (rc) return rc;
	}
	S.recv_rows = total_recv;
	S.ncols = ncols;
	S.sent_bytes = 0;
	CG_CUDA(cudaStreamWaitEvent(g_comm.side, g_comm.ev_scatter, 0));
	CG_CUDA(cudaEventRecord(S.t0, g_comm.side));
	if (W == 1)
	{
		/* nothing to move: total_recv == n and the scatter wrote the receive buffer */
	}
	else
	{
		/* one group for all columns and all peers: NCCL fuses it into one all-to-all over NVLink */
		CG_NCCL(g_nccl.GroupStart());
		int64_t soff = 0, roff = 0;
		for (int r = 0; r < W; r++)
		{
			for (int c = 0; c < ncols; c++)
			{
				ncclResult_t e = ncclSuccess;
				if (send_rows[r] > 0)
					e = g_nccl.Send(outs[c] + soff, (size_t) send_rows[r], ncclInt64, r, g_comm.comm, g_comm.side);
				if (e == ncclSuccess && recv_rows[r] > 0)
					e = g_nccl.Recv((int64_t *) S.recv.p + (size_t) c * total_recv + roff, (size_t) recv_rows[r], ncclInt64, r, g_comm.comm,
									g_comm.side);
				if (e != ncclSuccess) { g_nccl.GroupEnd(); return cg_set_error(CG_ECOMM, "ncclSend/Recv failed: %s", g_nccl.GetErrorString(e)); }
			}
			if (r != me) S.sent_bytes += (uint64_t) send_rows[r] * sizeof(int64_t) * ncols;
			soff += send_rows[r]; roff += recv_rows[r];
		}
		CG_NCCL(g_nccl.GroupEnd());
	}
	CG_CUDA(cudaEventRecord(S.t1, g_comm.side));
	CG_CUDA(cudaEventRecord(S.done, g_comm.side));
	if (recv_rows_out) *recv_rows_out = total_recv;
	return CG_OK;
}

/* the compute stream (the join that follows) waits for the slot's exchange on the device; the host does not block */
extern "C" int cg_comm_exchange_wait(int32_t slot)
{
	CgContext *ctx = cg_ctx();
	if (!ctx) return CG_EINVAL;
	if (int rc0 = cg_chain_end(ctx, ctx->compute)) return rc0;
	if (slot < 0 || slot >= 4 || !g_comm.slots[slot].done) return cg_set_error(CG_EINVAL, "no exchange in slot %d", slot);
	CG_CUDA(cudaStreamWaitEvent(ctx->compute, g_comm.slots[slot].done, 0));
	return CG_OK;
}

extern "C" int cg_comm_exchange_result(int32_t slot, int64_t **d_cols /* [ncols] */, int64_t *nrows, int64_t *part_counts,
									   int32_t *nlocal, uint64_t *sent_bytes, double *exchange_ms)
{
	if (slot < 0 || slot >= 4 || !g_comm.slots[slot].done) return cg_set_error(CG_EINVAL, "no exchange in slot %d", slot);
	CgComm::Slot &S = g_comm.slots[slot];
	if (d_cols) for (int c = 0; c < S.ncols; c++) d_cols[c] = (int64_t *) S.recv.p + (size_t) c * S.recv_rows;
	if (nrows) *nrows = S.recv_rows;
	if (nlocal) *nlocal = (int32_t) (S.part_counts.size() / (size_t) g_comm.nranks);
	if (part_counts) memcpy(part_counts, S.part_counts.data(), S.part_counts.size() * sizeof(int64_t));
	if (sent_bytes) *sent_bytes = S.sent_bytes;
	if (exchange_ms)
	{
		CG_CUDA(cudaEventSynchronize(S.t1));
		float ms = 0;
		CG_CUDA(cudaEventElapsedTime(&ms, S.t0, S.t1));
		*exchange_ms = ms;
	}
	return CG_OK;
}
