/*
 * oracle.c -- CPU restatement of the Citus hot path this repo accelerates.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under citus_b200/ may link, import or
 * execute this file; only tests/, __graft_entry__.smoke() and the
 * cpu_baseline / --impl reference legs of bench.py do.  It is the checker the
 * CUDA path is compared against, never the thing measured as "ours".
 *
 * Parity status: PINNED.  tests/test_oracle_golden.py checks this file against
 * the reference's own golden vectors (hashint4/hashint8/worker_hash values,
 * 4-way partition membership and the 1M-row partition row/byte counts, COPY
 * text/binary byte counts, columnar chunk-filtering row/chunk-group counts,
 * columnar_query aggregates, TPC-H Q1/Q6 over the 12 000-row lineitem fixture,
 * sum(l_suppkey)) -- see SURVEY.md section 4 / 8(c).  Compressed chunk BYTES
 * (lz4/zstd) are round-trip-only ("parity unpinned" for the encoded bytes, the
 * reference holds no golden compressed buffers); pglz's stream format is restated
 * with a stand-in matcher (see orc_pglz_compress).
 *
 * The arithmetic of this path mostly lives in PostgreSQL core (16-18), which is
 * not vendored in the Citus sources; the pieces restated from its published
 * algorithm are marked [PG] and anchored on the reference call sites.
 *
 * Every function cites the reference file:line it follows
 * (paths relative to the Citus sources' src/).
 */
#define _GNU_SOURCE
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <dlfcn.h>

typedef __int128 int128;

#define ORC_BLCKSZ 8192
#define ORC_PAGE_HEADER 24                     /* SizeOfPageHeaderData [PG] */
#define ORC_BYTES_PER_PAGE (ORC_BLCKSZ - ORC_PAGE_HEADER) /* include/columnar/columnar.h:57 */
#define ORC_FIRST_LOGICAL_OFFSET (2 * ORC_BYTES_PER_PAGE) /* include/columnar/columnar_storage.h:31-33 */
#define ORC_FIRST_ROW_NUMBER 1                 /* include/columnar/columnar_storage.h:21 */

/* include/columnar/columnar_compression.h:17-27 */
enum { ORC_COMP_NONE = 0, ORC_COMP_PGLZ = 1, ORC_COMP_LZ4 = 2, ORC_COMP_ZSTD = 3 };

/* column type classes (fixed-width by-value types only; by-reference types are
 * SURVEY.md 8(f) row 4, "next") */
enum { ORC_T_INT = 0, ORC_T_FLOAT = 1,
	   /* SURVEY.md 8(f) row 4, first slice: by-reference types whose VALUES are scaled integers / one character.
		* attlen is -1 (varlena), attalign 'i'; the low byte of atttype is the class, the rest the numeric scale:
		* a numeric(p, s) column holds value * 10^s as an int64 Datum in this file; char(1) holds the byte. */
	   ORC_T_NUMERIC = 2, ORC_T_BPCHAR1 = 3 };
#define ORC_TCLASS(t) ((t) & 0xff)
#define ORC_TSCALE(t) ((t) >> 8)

/* comparison operators of a pushed-down / row qual "col <op> const" */
enum { ORC_OP_LT = 0, ORC_OP_LE = 1, ORC_OP_EQ = 2, ORC_OP_GE = 3, ORC_OP_GT = 4, ORC_OP_NE = 5 };

/* aggregate kinds (worker half, multi_logical_optimizer.c:3160-3484) */
enum { ORC_AGG_COUNT_STAR = 0, ORC_AGG_COUNT = 1, ORC_AGG_SUM = 2, ORC_AGG_MIN = 3, ORC_AGG_MAX = 4 };

static char orc_errbuf[256];
const char *orc_last_error(void) { return orc_errbuf; }
#define ORC_FAIL(...) do { snprintf(orc_errbuf, sizeof orc_errbuf, __VA_ARGS__); return -1; } while (0)

/* ------------------------------------------------------------------------- *
 *  [PG] hash_bytes_uint32 / hashint4 / hashint8 (src/common/hashfn.c,
 *  src/backend/access/hash/hashfunc.c).  Reference call sites:
 *  executor/partitioned_intermediate_results.c:365-378 (typeEntry->hash_proc_finfo),
 *  utils/shardinterval_utils.c:266-269 (FunctionCall1Coll(hashFunction,...)).
 *  Goldens: test/regress/expected/partitioned_intermediate_results.out,
 *  distributed_planning.out:22-33, multi_utilities.out:269-272.
 * ------------------------------------------------------------------------- */
static inline uint32_t rot32(uint32_t x, int k) { return (x << k) | (x >> (32 - k)); }

uint32_t orc_hash_bytes_uint32(uint32_t k)
{
	uint32_t a, b, c;
	a = b = c = 0x9e3779b9u + (uint32_t) sizeof(uint32_t) + 3923095u;
	a += k;
	/* lookup3 final(a,b,c) */
	c ^= b; c -= rot32(b, 14);
	a ^= c; a -= rot32(c, 11);
	b ^= a; b -= rot32(a, 25);
	c ^= b; c -= rot32(b, 16);
	a ^= c; a -= rot32(c, 4);
	b ^= a; b -= rot32(a, 14);
	c ^= b; c -= rot32(b, 24);
	return c;
}

int32_t orc_hashint4(int32_t v) { return (int32_t) orc_hash_bytes_uint32((uint32_t) v); }

int32_t orc_hashint8(int64_t v)
{
	uint32_t lo = (uint32_t) (v & 0xffffffff);
	uint32_t hi = (uint32_t) ((uint64_t) v >> 32);
	lo ^= (v >= 0) ? hi : ~hi;
	return (int32_t) orc_hash_bytes_uint32(lo);
}

/* ------------------------------------------------------------------------- *
 *  Partition index arithmetic.
 * ------------------------------------------------------------------------- */

/* planner/multi_physical_planner.c:4667-4701 GenerateSyntheticShardIntervalArray;
 * HASH_TOKEN_COUNT include/distributed/metadata_utility.h:35 */
void orc_synthetic_intervals(int partitionCount, int32_t *mins, int32_t *maxs)
{
	uint64_t hashTokenIncrement = 4294967296ULL / (uint64_t) partitionCount;
	for (int i = 0; i < partitionCount; i++)
	{
		int32_t lo = (int32_t) ((int64_t) INT32_MIN + (int64_t) ((uint64_t) i * hashTokenIncrement));
		int32_t hi = (int32_t) ((int64_t) lo + (int64_t) (hashTokenIncrement - 1));
		if (i == partitionCount - 1)
			hi = INT32_MAX;
		mins[i] = lo;
		maxs[i] = hi;
	}
}

/* utils/shardinterval_utils.c:373-414 SearchCachedShardInterval (int4 btree cmp) */
int orc_search_interval(int32_t value, const int32_t *mins, const int32_t *maxs, int count)
{
	int lower = 0, upper = count;
	while (lower < upper)
	{
		int middle = (lower + upper) / 2;
		if (value < mins[middle]) { upper = middle; continue; }
		if (value <= maxs[middle]) return middle;
		lower = middle + 1;
	}
	return -1; /* INVALID_SHARD_INDEX */
}

/* utils/shardinterval_utils.c:424-452 CalculateUniformHashRangeIndex */
int orc_uniform_hash_range_index(int32_t hashedValue, int shardCount)
{
	int64_t normalized = (int64_t) hashedValue - (int64_t) INT32_MIN;
	int64_t hashRangeSize = 4294967296LL / shardCount;
	int shardIndex = (int) (normalized / hashRangeSize);
	if (shardIndex == shardCount)
		shardIndex = shardCount - 1;
	return shardIndex;
}

/*
 * executor/partitioned_intermediate_results.c:493-553
 * PartitionedResultDestReceiverReceive: NULL key -> partition 0; else
 * FindShardInterval (utils/shardinterval_utils.c:260-282) = hash then binary
 * search over the given min/max arrays (hasUniformHashDistribution is not set on
 * the synthetic cache entry, so the binary search is what runs).
 * keytype: 4 -> hashint4, 8 -> hashint8.  method 'h' hash / 'r' range.
 * out_index[n] gets the partition of every row, out_rows[P] the row counts.
 */
int orc_partition_rows(const int64_t *keys, const uint8_t *nulls, int64_t n, int keytype,
					   char method, const int32_t *mins, const int32_t *maxs, int P,
					   int32_t *out_index, int64_t *out_rows)
{
	memset(out_rows, 0, sizeof(int64_t) * (size_t) P);
	for (int64_t i = 0; i < n; i++)
	{
		int idx;
		if (nulls && nulls[i])
			idx = 0;
		else
		{
			int32_t searched;
			if (method == 'h')
				searched = (keytype == 4) ? orc_hashint4((int32_t) keys[i]) : orc_hashint8(keys[i]);
			else
				searched = (int32_t) keys[i];
			idx = orc_search_interval(searched, mins, maxs, P);
			if (idx < 0)
				ORC_FAIL("could not find shard for partition column value");
		}
		if (out_index) out_index[i] = idx;
		out_rows[idx]++;
	}
	return 0;
}

/* [PG] length of pg_ltoa / int8out text */
static int orc_int_text_len(int64_t v)
{
	char buf[32];
	return snprintf(buf, sizeof buf, "%lld", (long long) v);
}

/*
 * worker/worker_sql_task_protocol.c:167-251 + commands/multi_copy.c:1455-1530,
 * 1615-1645: bytes written to one partition file for rows of `ncols` integer
 * columns.  text: fields separated by '\t', NULL "\N", row ends '\n'.
 * binary: 11-byte signature + int32 flags + int32 extlen, per row int16 nfields
 * and per field int32 length (-1 NULL) + payload (attlen bytes), trailer int16.
 * Goldens: expected/partitioned_intermediate_results.out (21/14/5/9, 93/57/39/75,
 * 3586179..., 4500021).
 * cols[c][i] values, colnulls[c] may be NULL, collen[c] in {2,4,8}.
 */
int64_t orc_copy_file_bytes(const int64_t *const *cols, const uint8_t *const *colnulls,
							const int *collen, int ncols, const int32_t *row_partition,
							int partition, int64_t n, int binary)
{
	int64_t bytes = 0;
	int64_t rows = 0;
	for (int64_t i = 0; i < n; i++)
	{
		if (row_partition && row_partition[i] != partition) continue;
		rows++;
		if (binary)
		{
			bytes += 2;
			for (int c = 0; c < ncols; c++)
				bytes += 4 + ((colnulls && colnulls[c] && colnulls[c][i]) ? 0 : collen[c]);
		}
		else
		{
			for (int c = 0; c < ncols; c++)
			{
				if (colnulls && colnulls[c] && colnulls[c][i]) bytes += 2;
				else bytes += orc_int_text_len(cols[c][i]);
				bytes += 1; /* '\t' between fields, '\n' after the last */
			}
		}
	}
	if (binary)
		bytes += 11 + 4 + 4 + 2; /* header written at startup, footer at shutdown */
	(void) rows;
	return bytes;
}

/* ------------------------------------------------------------------------- *
 *  Columnar relation image: pages, stripes, skip nodes.
 * ------------------------------------------------------------------------- */

/* include/columnar/columnar.h:85-111 ColumnChunkSkipNode (+ catalog columnar.chunk,
 * sql/citus_columnar--11.1-1.sql:48-64) */
typedef struct OrcSkipNode
{
	int32_t has_minmax;
	int32_t compression_type;
	int64_t min_value;      /* raw Datum: sign-extended int or float8 bits */
	int64_t max_value;
	uint64_t row_count;
	uint64_t value_offset;  /* relative to stripe file_offset */
	uint64_t value_length;
	uint64_t exists_offset;
	uint64_t exists_length;
	uint64_t decompressed_size;
	int32_t compression_level;
	int32_t pad;
} OrcSkipNode;

/* include/columnar/columnar_metadata.h:21-42 StripeMetadata (+ columnar.stripe) */
typedef struct OrcStripe
{
	uint64_t id;
	uint64_t file_offset;
	uint64_t data_length;
	uint64_t row_count;
	uint64_t first_row_number;
	uint32_t column_count;
	uint32_t chunk_row_count;   /* chunk_group_row_limit in effect when written */
	uint32_t chunk_count;
	uint32_t skipnode_base;     /* index of skipnode[col 0][chunk 0] in the table's node array;
								 * node(col,chunk) = base + col*chunk_count + chunk */
} OrcStripe;

typedef struct OrcTable
{
	int natts;
	int *attlen;        /* 1,2,4,8 */
	char *attalign;     /* 'c','s','i','d' */
	int *atttype;       /* ORC_T_* */
	uint64_t stripe_row_limit;
	uint32_t chunk_row_limit;
	int compression;
	int compression_level;

	uint8_t *pages;     /* relation main fork: blocks of ORC_BLCKSZ */
	uint64_t nblocks;
	uint64_t cap_blocks;
	uint64_t reserved_offset; /* ColumnarMetapage.reservedOffset */
	uint64_t reserved_row;    /* reservedRowNumber */
	uint64_t reserved_stripe; /* reservedStripeId */

	OrcStripe *stripes; int nstripes, cap_stripes;
	OrcSkipNode *nodes; int nnodes, cap_nodes;

	/* write state (columnar_writer.c ColumnarWriteState) */
	uint64_t w_rows;            /* rows in the open stripe */
	uint8_t **w_exists;         /* [col] bool per row of the open chunk */
	uint8_t **w_chunk_values;   /* [col] serialized values of the open chunk */
	uint64_t *w_chunk_len;      /* [col] */
	uint64_t *w_chunk_cap;
	/* finished chunk buffers of the open stripe: [col][chunk] */
	uint8_t ***w_exists_buf; uint64_t **w_exists_len;
	uint8_t ***w_value_buf;  uint64_t **w_value_len;
	OrcSkipNode **w_nodes;   /* [col][chunk] */
	uint32_t w_max_chunks;
	uint32_t w_chunk_count;
	int borrowed;               /* pages / stripes / nodes belong to the caller */
} OrcTable;

/* --- liblz4 / libzstd through dlopen (headers are not installed here) --- */
typedef int (*lz4_bound_fn)(int);
typedef int (*lz4_comp_fn)(const char *, char *, int, int);
typedef int (*lz4_decomp_fn)(const char *, char *, int, int);
typedef size_t (*zstd_bound_fn)(size_t);
typedef size_t (*zstd_comp_fn)(void *, size_t, const void *, size_t, int);
typedef size_t (*zstd_decomp_fn)(void *, size_t, const void *, size_t);
typedef unsigned (*zstd_iserr_fn)(size_t);
static lz4_bound_fn p_lz4_bound; static lz4_comp_fn p_lz4_comp; static lz4_decomp_fn p_lz4_decomp;
static zstd_bound_fn p_zstd_bound; static zstd_comp_fn p_zstd_comp; static zstd_decomp_fn p_zstd_decomp;
static zstd_iserr_fn p_zstd_iserr;

static int orc_load_codecs(void)
{
	static int loaded = 0;
	if (loaded) return 0;
	void *l = dlopen("liblz4.so.1", RTLD_NOW);
	if (l)
	{
		p_lz4_bound = (lz4_bound_fn) dlsym(l, "LZ4_compressBound");
		p_lz4_comp = (lz4_comp_fn) dlsym(l, "LZ4_compress_default");
		p_lz4_decomp = (lz4_decomp_fn) dlsym(l, "LZ4_decompress_safe");
	}
	void *z = dlopen("libzstd.so.1", RTLD_NOW);
	if (z)
	{
		p_zstd_bound = (zstd_bound_fn) dlsym(z, "ZSTD_compressBound");
		p_zstd_comp = (zstd_comp_fn) dlsym(z, "ZSTD_compress");
		p_zstd_decomp = (zstd_decomp_fn) dlsym(z, "ZSTD_decompress");
		p_zstd_iserr = (zstd_iserr_fn) dlsym(z, "ZSTD_isError");
	}
	loaded = 1;
	return 0;
}

int orc_have_lz4(void) { orc_load_codecs(); return p_lz4_comp != NULL; }
int orc_have_zstd(void) { orc_load_codecs(); return p_zstd_comp != NULL; }

/* ------------------------------------------------------------------------------
 * pglz: [PG] src/common/pg_lzcompress.c (PostgreSQL is not part of the Citus sources;
 * the stream format is restated from its published description).  A stream is a
 * sequence of control bytes, each followed by up to 8 items, LSB first: bit clear =
 * one literal byte; bit set = a tag of 2 bytes [ (off >> 8) << 4 | (len - 3) ]
 * [ off & 0xff ], followed by one more byte (len - 18) when len - 3 == 15.
 * off in 1..4095, len in 3..273.
 *
 * orc_pglz_decompress restates pglz_decompress(source, slen, dest, rawsize,
 * check_complete = true) as the reference calls it (columnar_compression.c:245-250).
 * orc_pglz_compress is a plain greedy hash-chain matcher that emits the same format; it
 * is NOT PostgreSQL's matcher, so the compressed BYTES are "parity unpinned" (the
 * reference holds no golden pglz buffers); only decode(encode(x)) == x and the failure
 * rule of PGLZ_strategy_always (output must be smaller than (slen/100)*100) are kept.
 * ------------------------------------------------------------------------------ */
static int32_t orc_pglz_decompress(const uint8_t *source, int32_t slen, uint8_t *dest, int32_t rawsize)
{
	const uint8_t *sp = source, *srcend = source + slen;
	uint8_t *dp = dest, *destend = dest + rawsize;
	while (sp < srcend && dp < destend)
	{
		uint8_t ctrl = *sp++;
		for (int ctrlc = 0; ctrlc < 8 && sp < srcend && dp < destend; ctrlc++)
		{
			if (ctrl & 1)
			{
				int32_t len = (sp[0] & 0x0f) + 3;
				int32_t off = ((sp[0] & 0xf0) << 4) | sp[1];
				sp += 2;
				if (len == 18) len += *sp++;
				if (sp > srcend || off == 0 || off > (dp - dest)) return -1;
				if (len > destend - dp) len = (int32_t) (destend - dp);
				for (int32_t i = 0; i < len; i++) dp[i] = dp[i - off];   /* overlapping forward copy */
				dp += len;
			}
			else
				*dp++ = *sp++;
			ctrl >>= 1;
		}
	}
	if (dp != destend || sp != srcend) return -1;
	return (int32_t) (dp - dest);
}

static int32_t orc_pglz_compress(const uint8_t *src, int32_t slen, uint8_t *dst)
{
	enum { HSIZE = 8192, MAXOFF = 4095, MAXLEN = 273, CHAIN = 32 };
	if (slen <= 0) return -1;
	int32_t result_max = (slen / 100) * 100;
	int32_t *head = malloc(sizeof(int32_t) * HSIZE), *prev = malloc(sizeof(int32_t) * (size_t) slen);
	for (int i = 0; i < HSIZE; i++) head[i] = -1;
	uint8_t *bp = dst, *ctrlp = NULL;
	uint8_t ctrlb = 0, ctrl = 0;
	int32_t i = 0;
	int ok = 1;
#define ORC_PGLZ_HASH(p) ((((p)[0] << 6) ^ ((p)[1] << 3) ^ (p)[2]) & (HSIZE - 1))
	while (i < slen)
	{
		if (bp - dst >= result_max) { ok = 0; break; }
		if (ctrl == 0) { if (ctrlp) *ctrlp = ctrlb; ctrlp = bp++; ctrlb = 0; ctrl = 1; }
		int32_t best_len = 0, best_off = 0;
		if (i + 3 <= slen)
		{
			int h = ORC_PGLZ_HASH(src + i);
			int32_t cand = head[h];
			for (int depth = 0; cand >= 0 && i - cand <= MAXOFF && depth < CHAIN; depth++, cand = prev[cand])
			{
				int32_t l = 0, maxl = slen - i < MAXLEN ? slen - i : MAXLEN;
				while (l < maxl && src[cand + l] == src[i + l]) l++;
				if (l > best_len) { best_len = l; best_off = i - cand; }
			}
		}
		int32_t step = 1;
		if (best_len >= 3)
		{
			ctrlb |= ctrl;
			if (best_len > 17)
			{
				*bp++ = (uint8_t) (((best_off & 0xf00) >> 4) | 0x0f);
				*bp++ = (uint8_t) (best_off & 0xff);
				*bp++ = (uint8_t) (best_len - 18);
			}
			else
			{
				*bp++ = (uint8_t) (((best_off & 0xf00) >> 4) | (best_len - 3));
				*bp++ = (uint8_t) (best_off & 0xff);
			}
			step = best_len;
		}
		else
			*bp++ = src[i];
		ctrl = (uint8_t) (ctrl << 1);
		for (int32_t k = 0; k < step; k++, i++)
			if (i + 3 <= slen) { int h = ORC_PGLZ_HASH(src + i); prev[i] = head[h]; head[h] = i; }
	}
#undef ORC_PGLZ_HASH
	if (ctrlp) *ctrlp = ctrlb;
	free(head); free(prev);
	if (!ok || bp - dst >= result_max) return -1;
	return (int32_t) (bp - dst);
}

/* columnar/columnar_compression.c:62-157 CompressBuffer.  Returns compressed
 * length (>0) and sets *out, or 0 when "not compressed" (stored raw). */
static uint64_t orc_compress(const uint8_t *in, uint64_t len, int type, int level, uint8_t **out)
{
	orc_load_codecs();
	if (type == ORC_COMP_LZ4 && p_lz4_comp)
	{
		int bound = p_lz4_bound((int) len);
		uint8_t *buf = malloc((size_t) bound + 1);
		int n = p_lz4_comp((const char *) in, (char *) buf, (int) len, bound);
		if (n <= 0) { free(buf); return 0; }
		*out = buf;
		return (uint64_t) n;
	}
	if (type == ORC_COMP_PGLZ)
	{
		/* :120-150: PGLZ_MAX_OUTPUT(len) = len + 4, behind the 8-byte ColumnarCompressHeader
		 * {vl_len_ = SET_VARSIZE_COMPRESSED(total) (little endian: total << 2 | 0x02), rawsize} */
		uint8_t *buf = malloc((size_t) len + 4 + 8 + 16);
		int32_t n = orc_pglz_compress(in, (int32_t) len, buf + 8);
		if (n < 0) { free(buf); return 0; }
		uint32_t total = (uint32_t) n + 8, hdr = (total << 2) | 0x02u, raw = (uint32_t) len;
		memcpy(buf, &hdr, 4);
		memcpy(buf + 4, &raw, 4);
		*out = buf;
		return total;
	}
	if (type == ORC_COMP_ZSTD && p_zstd_comp)
	{
		size_t bound = p_zstd_bound(len);
		uint8_t *buf = malloc(bound + 1);
		size_t n = p_zstd_comp(buf, bound, in, len, level);
		if (p_zstd_iserr(n)) { free(buf); return 0; }
		*out = buf;
		return n;
	}
	return 0;
}

/* columnar/columnar_compression.c:165-270 DecompressBuffer */
static int orc_decompress(const uint8_t *in, uint64_t len, int type, uint64_t rawlen, uint8_t *out)
{
	orc_load_codecs();
	switch (type)
	{
		case ORC_COMP_NONE:
			memcpy(out, in, len);
			return 0;
		case ORC_COMP_LZ4:
		{
			if (!p_lz4_decomp) ORC_FAIL("liblz4 not available");
			int n = p_lz4_decomp((const char *) in, (char *) out, (int) len, (int) rawlen);
			if (n < 0 || (uint64_t) n != rawlen) ORC_FAIL("cannot decompress the buffer");
			return 0;
		}
		case ORC_COMP_ZSTD:
		{
			if (!p_zstd_decomp) ORC_FAIL("libzstd not available");
			size_t n = p_zstd_decomp(out, rawlen, in, len);
			if (p_zstd_iserr(n)) ORC_FAIL("zstd decompression failed");
			if (n != rawlen) ORC_FAIL("unexpected decompressed size");
			return 0;
		}
		case ORC_COMP_PGLZ:
		{
			/* :240-267 */
			uint32_t hdr, raw;
			if (len < 8) ORC_FAIL("cannot decompress the buffer");
			memcpy(&hdr, in, 4);
			memcpy(&raw, in + 4, 4);
			uint32_t varsize = (hdr >> 2) & 0x3FFFFFFFu;            /* VARSIZE of a 4-byte varlena header */
			if (varsize != len) ORC_FAIL("cannot decompress the buffer");
			if (raw != rawlen) ORC_FAIL("cannot decompress the buffer");
			if (orc_pglz_decompress(in + 8, (int32_t) (varsize - 8), out, (int32_t) raw) < 0)
				ORC_FAIL("cannot decompress the buffer");
			return 0;
		}
		default:
			ORC_FAIL("unexpected compression type: %d", type);
	}
}

/* ------------------------------------------------------------------------------
 * The MERGE task of a dual-repartition join (planner/multi_physical_planner.c:4304-4328:
 * both inputs come back through read_intermediate_results() and are joined by [PG]
 * nodeHashjoin, then aggregated by nodeAgg):
 *     SELECT count(*), sum(b.payload + p.payload) FROM build b JOIN probe p USING (key)
 * restated row-at-a-time: every probe row is matched against every build row with an
 * equal key (NULL keys never match), each joined row adds 1 and b.payload + p.payload
 * (int8 + int8 -> numeric sum: exact, kept in 128 bits).
 * ------------------------------------------------------------------------------ */
typedef struct { int64_t key; int64_t payload; } OrcJoinRow;
static int orc_join_row_cmp(const void *a, const void *b)
{
	int64_t x = ((const OrcJoinRow *) a)->key, y = ((const OrcJoinRow *) b)->key;
	return (x > y) - (x < y);
}

int orc_join_count_sum(const int64_t *bkeys, const uint8_t *bnulls, const int64_t *bpay, int64_t nb,
					   const int64_t *pkeys, const uint8_t *pnulls, const int64_t *ppay, int64_t np,
					   int64_t *joined, int64_t *sum_hi, uint64_t *sum_lo)
{
	OrcJoinRow *rows = malloc(sizeof(OrcJoinRow) * (size_t) (nb > 0 ? nb : 1));
	int64_t n = 0;
	for (int64_t i = 0; i < nb; i++)
		if (!(bnulls && bnulls[i])) { rows[n].key = bkeys[i]; rows[n].payload = bpay[i]; n++; }
	qsort(rows, (size_t) n, sizeof(OrcJoinRow), orc_join_row_cmp);
	__int128 sum = 0;
	int64_t count = 0;
	for (int64_t i = 0; i < np; i++)
	{
		if (pnulls && pnulls[i]) continue;
		int64_t lo = 0, hi = n;
		while (lo < hi) { int64_t mid = lo + (hi - lo) / 2; if (rows[mid].key < pkeys[i]) lo = mid + 1; else hi = mid; }
		for (int64_t j = lo; j < n && rows[j].key == pkeys[i]; j++)
		{
			count++;
			sum += (__int128) rows[j].payload + (__int128) ppay[i];
		}
	}
	free(rows);
	*joined = count;
	*sum_lo = (uint64_t) sum;
	*sum_hi = (int64_t) (sum >> 64);
	return 0;
}

/* the codecs alone, for known-answer tests of the stream formats */
int64_t orc_codec_compress(int type, int level, const uint8_t *in, uint64_t len, uint8_t *out, uint64_t cap)
{
	uint8_t *buf = NULL;
	uint64_t n = orc_compress(in, len, type, level, &buf);
	if (n == 0) return 0;
	if (n > cap) { free(buf); return -1; }
	memcpy(out, buf, n);
	free(buf);
	return (int64_t) n;
}

int orc_codec_decompress(int type, const uint8_t *in, uint64_t len, uint64_t rawlen, uint8_t *out)
{
	return orc_decompress(in, len, type, rawlen, out);
}

static int orc_align_of(char attalign)
{
	switch (attalign) { case 'c': return 1; case 's': return 2; case 'i': return 4; default: return 8; }
}


/* [PG] fetch_att for by-value types (tupmacs.h), sign-extending; float4 is promoted
 * to float8 bits so that every float Datum in this file is a float8 */
static inline int64_t orc_fetch_att(const uint8_t *p, int len, int atttype)
{
	int64_t v = 0;
	switch (len)
	{
		case 1: v = (int64_t) *(const int8_t *) p; break;
		case 2: { int16_t x; memcpy(&x, p, 2); v = x; break; }
		case 4: { int32_t x; memcpy(&x, p, 4); v = x; break; }
		default: memcpy(&v, p, 8); break;
	}
	if (atttype == ORC_T_FLOAT && len == 4)
	{
		float f; uint32_t u = (uint32_t) v; memcpy(&f, &u, 4);
		double d = f; memcpy(&v, &d, 8);
	}
	return v;
}


/* ------------------------------------------------------------------------- *
 *  [PG] varlena headers (varatt.h, little-endian): 1-byte header when bit 0 is set (total length = header >> 1,
 *  at most 127), else a 4-byte header (total length = header >> 2).  columnar_reader.c:1557-1565 advances by
 *  att_addlength_datum = VARSIZE_ANY and then aligns to the type's alignment ('i' = 4 for numeric, bpchar, text).
 *  [PG] numeric on-disk format (numeric.c): base-10000 digits d[0..n) with value = sum d[i] * 10000^(weight - i);
 *    short: uint16 header = 0x8000 | sign 0x2000 | dscale << 7 | weight sign 0x0040 | weight & 0x3F, when
 *           dscale <= 63 and -64 <= weight <= 63; long: uint16 sign (0x0000 / 0x4000, 0xC000 = NaN) | dscale, int16 weight.
 *    Leading and trailing zero digits are stripped; zero is no digits, weight 0, positive.
 *  PARITY: the reference repository holds no golden on-disk numeric bytes (the format is PostgreSQL's); what is
 *  pinned is decode(encode(x)) = x here and the TPC-H Q1/Q6 goldens computed through these columns.
 * ------------------------------------------------------------------------- */
static int orc_varlena_total(const uint8_t *p)
{
	if (p[0] & 1) return p[0] >> 1;
	uint32_t h; memcpy(&h, p, 4);
	return (int) (h >> 2);
}
static int orc_varlena_hdr(const uint8_t *p) { return (p[0] & 1) ? 1 : 4; }

static int orc_varlena_wrap(uint8_t *out, const uint8_t *payload, int n, int short_header)
{
	if (short_header && n + 1 <= 127) { out[0] = (uint8_t) (((n + 1) << 1) | 1); memcpy(out + 1, payload, (size_t) n); return n + 1; }
	uint32_t h = (uint32_t) (n + 4) << 2;
	memcpy(out, &h, 4); memcpy(out + 4, payload, (size_t) n);
	return n + 4;
}

/* scaled integer (value * 10^scale) -> numeric datum (with its varlena header); returns the datum's length */
static int orc_numeric_encode(int64_t scaled, int scale, int short_header, uint8_t *out)
{
	int neg = scaled < 0;
	unsigned __int128 a = neg ? (unsigned __int128) (-(int128) scaled) : (unsigned __int128) scaled;
	unsigned __int128 p10 = 1;
	for (int i = 0; i < scale; i++) p10 *= 10;
	unsigned __int128 ip = a / p10, fp = a % p10;
	int16_t digits[32]; int nd = 0;
	/* integer part, most significant base-10000 digit first */
	int16_t tmp[16]; int nt = 0;
	while (ip > 0) { tmp[nt++] = (int16_t) (ip % 10000); ip /= 10000; }
	int weight = nt - 1;
	for (int i = nt - 1; i >= 0; i--) digits[nd++] = tmp[i];
	/* fraction: `scale` decimal digits, right-padded with zeros to a multiple of 4 */
	int fgroups = (scale + 3) / 4;
	for (int i = scale; i < fgroups * 4; i++) fp *= 10;
	for (int g = fgroups - 1; g >= 0; g--) { tmp[g] = (int16_t) (fp % 10000); fp /= 10000; }
	for (int g = 0; g < fgroups; g++) digits[nd++] = tmp[g];
	/* strip leading / trailing zero digits (make_result / strip_var) */
	int first = 0;
	while (first < nd && digits[first] == 0) { first++; weight--; }
	while (nd > first && digits[nd - 1] == 0) nd--;
	int n = nd - first;
	if (n == 0) { weight = 0; neg = 0; }
	uint8_t body[80]; int len = 0;
	if (scale <= 0x3F && weight >= -64 && weight <= 63)
	{
		uint16_t h = (uint16_t) (0x8000 | (neg ? 0x2000 : 0) | (scale << 7) | (weight < 0 ? 0x0040 : 0) | (weight & 0x003F));
		memcpy(body, &h, 2); len = 2;
	}
	else
	{
		uint16_t sd = (uint16_t) ((neg ? 0x4000 : 0x0000) | (scale & 0x3FFF));
		int16_t w = (int16_t) weight;
		memcpy(body, &sd, 2); memcpy(body + 2, &w, 2); len = 4;
	}
	for (int i = 0; i < n; i++) { memcpy(body + len, &digits[first + i], 2); len += 2; }
	return orc_varlena_wrap(out, body, len, short_header);
}

/* numeric datum -> value * 10^scale; -1 if it is NaN / has more fractional digits than the scale / overflows int64 */
static int orc_numeric_decode(const uint8_t *datum, int scale, int64_t *out)
{
	int total = orc_varlena_total(datum), hdr = orc_varlena_hdr(datum);
	const uint8_t *p = datum + hdr;
	int n = total - hdr;
	if (n < 2) return -1;
	uint16_t h; memcpy(&h, p, 2);
	int neg, weight, nd;
	const uint8_t *dp;
	if ((h & 0xC000) == 0x8000)
	{
		neg = (h & 0x2000) != 0;
		weight = (h & 0x0040) ? (int) (h & 0x003F) - 64 : (int) (h & 0x003F);     /* sign-extended 7-bit weight */
		dp = p + 2; nd = (n - 2) / 2;
	}
	else
	{
		if ((h & 0xC000) == 0xC000) return -1;                                   /* NaN / infinity */
		neg = (h & 0xC000) == 0x4000;
		int16_t w; memcpy(&w, p + 2, 2); weight = w;
		dp = p + 4; nd = (n - 4) / 2;
	}
	int128 acc = 0;
	for (int i = 0; i < nd; i++) { int16_t d; memcpy(&d, dp + 2 * i, 2); acc = acc * 10000 + d; }
	/* acc * 10000^(weight - (nd - 1)) * 10^scale must be an integer */
	int e10 = 4 * (weight - (nd - 1)) + scale;
	if (nd == 0) { *out = 0; return 0; }
	while (e10 > 0) { acc *= 10; e10--; if (acc > (int128) INT64_MAX * 4) return -1; }
	while (e10 < 0) { if (acc % 10 != 0) return -1; acc /= 10; e10++; }
	if (acc > (int128) INT64_MAX) return -1;
	*out = neg ? -(int64_t) acc : (int64_t) acc;
	return 0;
}

/* stored form of a row value for a varlena class; returns the datum's length */
static int orc_varlena_encode(int atttype, int64_t v, int short_header, uint8_t *out)
{
	if (ORC_TCLASS(atttype) == ORC_T_NUMERIC) return orc_numeric_encode(v, ORC_TSCALE(atttype), short_header, out);
	uint8_t ch = (uint8_t) v;                        /* char(1): the blank-padded string of length 1 */
	return orc_varlena_wrap(out, &ch, 1, short_header);
}

static int orc_varlena_decode(int atttype, const uint8_t *datum, int64_t *out)
{
	if (ORC_TCLASS(atttype) == ORC_T_NUMERIC) return orc_numeric_decode(datum, ORC_TSCALE(atttype), out);
	if (orc_varlena_total(datum) - orc_varlena_hdr(datum) != 1) return -1;
	*out = (int64_t) (int8_t) datum[orc_varlena_hdr(datum)];
	return 0;
}

/* columnar_reader.c:1542-1572 DeserializeDatumArray, one datum: fetch_att (by-value) or the varlena at the current
 * offset (by-reference; its VALUE is decoded here because this file keeps every Datum as an int64), then
 * att_addlength_datum + att_align_nominal */
static int orc_read_datum(const OrcTable *t, int c, const uint8_t *buf, uint32_t *off, uint64_t limit, int64_t *v)
{
	int len = t->attlen[c], al = orc_align_of(t->attalign[c]);
	if (len < 0)
	{
		if ((uint64_t) *off + 1 > limit) return -1;
		len = orc_varlena_total(buf + *off);
		if (len < orc_varlena_hdr(buf + *off) || (uint64_t) *off + (uint64_t) len > limit) return -1;
		if (orc_varlena_decode(t->atttype[c], buf + *off, v)) return -2;
	}
	else
		*v = orc_fetch_att(buf + *off, len, t->atttype[c]);
	*off += (uint32_t) len;
	*off = (*off + (uint32_t) al - 1) & ~((uint32_t) al - 1);
	return 0;
}

static int orc_short_varlena_headers = 0;    /* 1: data as read back from heap tuples (packed 1-byte headers); 0: as produced by input functions */
void orc_set_short_varlena_headers(int on) { orc_short_varlena_headers = on; }

OrcTable *orc_table_create(int natts, const int *attlen, const int *atttype,
						   uint64_t stripe_row_limit, uint32_t chunk_row_limit,
						   int compression, int compression_level)
{
	OrcTable *t = calloc(1, sizeof *t);
	t->natts = natts;
	t->attlen = malloc(sizeof(int) * natts);
	t->atttype = malloc(sizeof(int) * natts);
	t->attalign = malloc(natts);
	for (int c = 0; c < natts; c++)
	{
		t->attlen[c] = attlen[c];
		t->atttype[c] = atttype[c];
		t->attalign[c] = attlen[c] < 0 ? 'i' : attlen[c] == 1 ? 'c' : attlen[c] == 2 ? 's' : attlen[c] == 4 ? 'i' : 'd';
	}
	t->stripe_row_limit = stripe_row_limit;  /* columnar.c:29 default 150000 */
	t->chunk_row_limit = chunk_row_limit;    /* columnar.c:30 default 10000 */
	t->compression = compression;
	t->compression_level = compression_level;
	/* block 0 = metapage, block 1 = empty (columnar_storage.c:21-31) */
	t->cap_blocks = 64;
	t->pages = calloc(t->cap_blocks, ORC_BLCKSZ);
	t->nblocks = 2;
	t->reserved_offset = ORC_FIRST_LOGICAL_OFFSET;
	t->reserved_row = ORC_FIRST_ROW_NUMBER;
	t->reserved_stripe = 1;
	t->w_max_chunks = (uint32_t) (stripe_row_limit / chunk_row_limit) + 1; /* columnar_writer.c:177 */
	t->w_exists = calloc(natts, sizeof(uint8_t *));
	t->w_chunk_values = calloc(natts, sizeof(uint8_t *));
	t->w_chunk_len = calloc(natts, sizeof(uint64_t));
	t->w_chunk_cap = calloc(natts, sizeof(uint64_t));
	t->w_exists_buf = calloc(natts, sizeof(uint8_t **));
	t->w_exists_len = calloc(natts, sizeof(uint64_t *));
	t->w_value_buf = calloc(natts, sizeof(uint8_t **));
	t->w_value_len = calloc(natts, sizeof(uint64_t *));
	t->w_nodes = calloc(natts, sizeof(OrcSkipNode *));
	for (int c = 0; c < natts; c++)
	{
		t->w_exists[c] = calloc(chunk_row_limit, 1);
		t->w_chunk_cap[c] = (uint64_t) chunk_row_limit * (attlen[c] < 0 ? 32 : 8);
		t->w_chunk_values[c] = malloc(t->w_chunk_cap[c]);
		t->w_exists_buf[c] = calloc(t->w_max_chunks, sizeof(uint8_t *));
		t->w_exists_len[c] = calloc(t->w_max_chunks, sizeof(uint64_t));
		t->w_value_buf[c] = calloc(t->w_max_chunks, sizeof(uint8_t *));
		t->w_value_len[c] = calloc(t->w_max_chunks, sizeof(uint64_t));
		t->w_nodes[c] = calloc(t->w_max_chunks, sizeof(OrcSkipNode));
	}
	return t;
}

void orc_table_free(OrcTable *t)
{
	if (!t) return;
	for (int c = 0; c < t->natts; c++)
	{
		free(t->w_exists[c]); free(t->w_chunk_values[c]);
		for (uint32_t k = 0; k < t->w_max_chunks; k++) { free(t->w_exists_buf[c][k]); free(t->w_value_buf[c][k]); }
		free(t->w_exists_buf[c]); free(t->w_exists_len[c]); free(t->w_value_buf[c]); free(t->w_value_len[c]);
		free(t->w_nodes[c]);
	}
	free(t->w_exists); free(t->w_chunk_values); free(t->w_chunk_len); free(t->w_chunk_cap);
	free(t->w_exists_buf); free(t->w_exists_len); free(t->w_value_buf); free(t->w_value_len); free(t->w_nodes);
	free(t->attlen); free(t->atttype); free(t->attalign);
	if (!t->borrowed) { free(t->pages); free(t->stripes); free(t->nodes); }
	free(t);
}

/* [PG] btree comparison of the column type (BTORDER_PROC), used for min/max */
static int orc_datum_cmp(int atttype, int64_t a, int64_t b)
{
	if (atttype == ORC_T_FLOAT)
	{
		double x, y;
		memcpy(&x, &a, 8); memcpy(&y, &b, 8);
		/* float8_cmp_internal: NaN sorts above everything */
		int xn = (x != x), yn = (y != y);
		if (xn || yn) return xn - yn;
		return (x > y) - (x < y);
	}
	return (a > b) - (a < b);
}

/* float8_cmp_internal on doubles (min/max transition and combine functions, float8smaller / float8larger) */
static int orc_float8_cmp(double x, double y)
{
	int64_t a, b;
	memcpy(&a, &x, 8); memcpy(&b, &y, 8);
	return orc_datum_cmp(ORC_T_FLOAT, a, b);
}

/* columnar_storage.c:117-126 LogicalToPhysical + ColumnarStorageWrite (WriteToBlock
 * keeps pd_lower at the end of the written payload, :698-744) */
static void orc_storage_write(OrcTable *t, uint64_t logical, const uint8_t *data, uint64_t amount)
{
	uint64_t written = 0;
	while (written < amount)
	{
		uint64_t L = logical + written;
		uint64_t blockno = L / ORC_BYTES_PER_PAGE;
		uint32_t offset = ORC_PAGE_HEADER + (uint32_t) (L % ORC_BYTES_PER_PAGE);
		uint64_t to_write = amount - written;
		if (to_write > ORC_BLCKSZ - offset) to_write = ORC_BLCKSZ - offset;
		if (blockno >= t->cap_blocks)
		{
			uint64_t ncap = t->cap_blocks * 2;
			while (ncap <= blockno) ncap *= 2;
			t->pages = realloc(t->pages, ncap * ORC_BLCKSZ);
			memset(t->pages + t->cap_blocks * ORC_BLCKSZ, 0, (ncap - t->cap_blocks) * ORC_BLCKSZ);
			t->cap_blocks = ncap;
		}
		if (blockno >= t->nblocks) t->nblocks = blockno + 1;
		uint8_t *page = t->pages + blockno * ORC_BLCKSZ;
		memcpy(page + offset, data + written, to_write);
		/* PageHeaderData.pd_lower lives at byte offset 12 (uint16) [PG bufpage.h] */
		uint16_t pd_lower = (uint16_t) (offset + to_write);
		uint16_t cur; memcpy(&cur, page + 12, 2);
		if (pd_lower > cur) memcpy(page + 12, &pd_lower, 2);
		written += to_write;
	}
}

/* columnar_storage.c:463-492 ColumnarStorageRead + :669-689 ReadFromBlock */
int orc_storage_read(const uint8_t *pages, uint64_t nblocks, uint64_t logical, uint8_t *out, uint64_t amount)
{
	if (amount == 0) return 0;
	if (logical < ORC_FIRST_LOGICAL_OFFSET)
		ORC_FAIL("attempted columnar read from invalid logical offset: %llu", (unsigned long long) logical);
	uint64_t done = 0;
	while (done < amount)
	{
		uint64_t L = logical + done;
		uint64_t blockno = L / ORC_BYTES_PER_PAGE;
		uint32_t offset = ORC_PAGE_HEADER + (uint32_t) (L % ORC_BYTES_PER_PAGE);
		uint64_t to_read = amount - done;
		if (to_read > ORC_BLCKSZ - offset) to_read = ORC_BLCKSZ - offset;
		if (blockno >= nblocks) ORC_FAIL("attempt to read columnar data past end of relation");
		const uint8_t *page = pages + blockno * ORC_BLCKSZ;
		uint16_t pd_lower; memcpy(&pd_lower, page + 12, 2);
		if (pd_lower < offset + to_read)
			ORC_FAIL("attempt to read columnar data of length %llu from offset %u of block %llu",
					 (unsigned long long) to_read, offset, (unsigned long long) blockno);
		memcpy(out + done, page + offset, to_read);
		done += to_read;
	}
	return 0;
}

/* columnar_writer.c:523-545 SerializeBoolArray */
static uint8_t *orc_serialize_bools(const uint8_t *bools, uint32_t n, uint64_t *len)
{
	uint32_t byteCount = (n + 7) / 8;
	uint8_t *buf = calloc(byteCount ? byteCount : 1, 1);
	for (uint32_t i = 0; i < n; i++)
		if (bools[i]) buf[i / 8] |= (uint8_t) (1 << (i % 8));
	*len = byteCount;
	return buf;
}

/* columnar_writer.c:592-654 SerializeChunkData for chunk `chunkIndex` of the open stripe */
static void orc_serialize_chunk(OrcTable *t, uint32_t chunkIndex, uint32_t rowCount)
{
	for (int c = 0; c < t->natts; c++)
	{
		t->w_exists_buf[c][chunkIndex] = orc_serialize_bools(t->w_exists[c], rowCount, &t->w_exists_len[c][chunkIndex]);
		OrcSkipNode *node = &t->w_nodes[c][chunkIndex];
		node->decompressed_size = t->w_chunk_len[c];
		uint8_t *comp = NULL;
		uint64_t clen = orc_compress(t->w_chunk_values[c], t->w_chunk_len[c], t->compression, t->compression_level, &comp);
		if (clen > 0)
		{
			t->w_value_buf[c][chunkIndex] = comp;
			t->w_value_len[c][chunkIndex] = clen;
			node->compression_type = t->compression;
		}
		else
		{
			uint8_t *raw = malloc(t->w_chunk_len[c] ? t->w_chunk_len[c] : 1);
			memcpy(raw, t->w_chunk_values[c], t->w_chunk_len[c]);
			t->w_value_buf[c][chunkIndex] = raw;
			t->w_value_len[c][chunkIndex] = t->w_chunk_len[c];
			node->compression_type = ORC_COMP_NONE;
		}
		node->compression_level = t->compression_level;
		t->w_chunk_len[c] = 0; /* resetStringInfo */
	}
}

/* columnar_writer.c:391-516 FlushStripe; stripe reservation columnar_storage.c:421-456
 * (ColumnarStorageReserveData) + :756-772 (AlignReservation) */
void orc_flush_stripe(OrcTable *t)
{
	if (t->w_rows == 0) return;
	uint32_t chunkRowCount = t->chunk_row_limit;
	uint32_t lastChunkIndex = (uint32_t) (t->w_rows / chunkRowCount);
	uint32_t lastChunkRowCount = (uint32_t) (t->w_rows % chunkRowCount);
	if (lastChunkRowCount > 0)
		orc_serialize_chunk(t, lastChunkIndex, lastChunkRowCount);
	uint32_t chunkCount = t->w_chunk_count;

	uint64_t stripeSize = 0;
	for (int c = 0; c < t->natts; c++)
	{
		for (uint32_t k = 0; k < chunkCount; k++)
		{
			t->w_nodes[c][k].exists_offset = stripeSize;
			t->w_nodes[c][k].exists_length = t->w_exists_len[c][k];
			stripeSize += t->w_exists_len[c][k];
		}
		for (uint32_t k = 0; k < chunkCount; k++)
		{
			t->w_nodes[c][k].value_offset = stripeSize;
			t->w_nodes[c][k].value_length = t->w_value_len[c][k];
			stripeSize += t->w_value_len[c][k];
		}
	}

	/* AlignReservation: stripes start at the beginning of a page */
	uint64_t aligned = t->reserved_offset;
	if (aligned % ORC_BYTES_PER_PAGE != 0)
		aligned = (aligned / ORC_BYTES_PER_PAGE + 1) * ORC_BYTES_PER_PAGE;
	uint64_t fileOffset = aligned;
	t->reserved_offset = aligned + stripeSize;

	if (t->nstripes == t->cap_stripes)
	{
		t->cap_stripes = t->cap_stripes ? t->cap_stripes * 2 : 16;
		t->stripes = realloc(t->stripes, sizeof(OrcStripe) * t->cap_stripes);
	}
	OrcStripe *s = &t->stripes[t->nstripes++];
	memset(s, 0, sizeof *s);
	s->id = t->reserved_stripe++;
	s->file_offset = fileOffset;
	s->data_length = stripeSize;
	s->row_count = t->w_rows;
	s->first_row_number = t->reserved_row;
	t->reserved_row += t->w_rows;
	s->column_count = (uint32_t) t->natts;
	s->chunk_row_count = chunkRowCount;
	s->chunk_count = chunkCount;
	s->skipnode_base = (uint32_t) t->nnodes;

	uint64_t need = (uint64_t) t->natts * chunkCount;
	if ((uint64_t) t->nnodes + need > (uint64_t) t->cap_nodes)
	{
		uint64_t ncap = t->cap_nodes ? (uint64_t) t->cap_nodes * 2 : 256;
		while (ncap < (uint64_t) t->nnodes + need) ncap *= 2;
		t->nodes = realloc(t->nodes, sizeof(OrcSkipNode) * ncap);
		t->cap_nodes = (int) ncap;
	}

	uint64_t cur = fileOffset;
	for (int c = 0; c < t->natts; c++)
	{
		for (uint32_t k = 0; k < chunkCount; k++)
		{
			orc_storage_write(t, cur, t->w_exists_buf[c][k], t->w_exists_len[c][k]);
			cur += t->w_exists_len[c][k];
		}
		for (uint32_t k = 0; k < chunkCount; k++)
		{
			orc_storage_write(t, cur, t->w_value_buf[c][k], t->w_value_len[c][k]);
			cur += t->w_value_len[c][k];
		}
		for (uint32_t k = 0; k < chunkCount; k++)
		{
			t->nodes[t->nnodes + c * (int) chunkCount + (int) k] = t->w_nodes[c][k];
			free(t->w_exists_buf[c][k]); t->w_exists_buf[c][k] = NULL;
			free(t->w_value_buf[c][k]); t->w_value_buf[c][k] = NULL;
			memset(&t->w_nodes[c][k], 0, sizeof(OrcSkipNode));
		}
	}
	t->nnodes += (int) need;
	t->w_rows = 0;
	t->w_chunk_count = 0;
}

/*
 * columnar_writer.c:150-260 ColumnarWriteRow, one row at a time like the reference:
 * per column set exists[], SerializeSingleDatum (:555-585, store_att_byval then pad
 * to attalign relative to the stream start), UpdateChunkSkipNodeMinMax (:663-718);
 * serialize the chunk when it fills, flush the stripe when it fills.
 */
void orc_write_row(OrcTable *t, const int64_t *values, const uint8_t *nulls)
{
	uint32_t chunkRowCount = t->chunk_row_limit;
	uint32_t chunkIndex = (uint32_t) (t->w_rows / chunkRowCount);
	uint32_t chunkRowIndex = (uint32_t) (t->w_rows % chunkRowCount);

	if (chunkRowIndex == 0)
		for (int c = 0; c < t->natts; c++) memset(t->w_exists[c], 0, chunkRowCount);

	for (int c = 0; c < t->natts; c++)
	{
		OrcSkipNode *node = &t->w_nodes[c][chunkIndex];
		if (nulls && nulls[c])
		{
			t->w_exists[c][chunkRowIndex] = 0;
		}
		else
		{
			uint8_t vbuf[96];
			int len = t->attlen[c];
			if (len < 0) len = orc_varlena_encode(t->atttype[c], values[c], orc_short_varlena_headers, vbuf);     /* VARSIZE_ANY(datum) */
			int aligned = (len + orc_align_of(t->attalign[c]) - 1) & ~(orc_align_of(t->attalign[c]) - 1);
			t->w_exists[c][chunkRowIndex] = 1;
			if (t->w_chunk_len[c] + (uint64_t) aligned > t->w_chunk_cap[c])
			{
				t->w_chunk_cap[c] *= 2;
				t->w_chunk_values[c] = realloc(t->w_chunk_values[c], t->w_chunk_cap[c]);
			}
			uint8_t *p = t->w_chunk_values[c] + t->w_chunk_len[c];
			memset(p, 0, (size_t) aligned);
			int64_t v = values[c];
			if (t->attlen[c] < 0)
				memcpy(p, vbuf, (size_t) len);
			else if (t->atttype[c] == ORC_T_FLOAT && len == 4)
			{
				double d; memcpy(&d, &v, 8);
				float f = (float) d; memcpy(p, &f, 4);
				d = f; memcpy(&v, &d, 8);
			}
			else
				memcpy(p, &v, (size_t) len); /* little-endian store_att_byval */
			t->w_chunk_len[c] += (uint64_t) aligned;

			if (!node->has_minmax)
			{
				node->has_minmax = 1; node->min_value = v; node->max_value = v;
			}
			else
			{
				if (orc_datum_cmp(t->atttype[c], v, node->min_value) < 0) node->min_value = v;
				if (orc_datum_cmp(t->atttype[c], v, node->max_value) > 0) node->max_value = v;
			}
		}
		node->row_count++;
	}
	t->w_chunk_count = chunkIndex + 1;
	if (chunkRowIndex == chunkRowCount - 1)
		orc_serialize_chunk(t, chunkIndex, chunkRowCount);
	t->w_rows++;
	if (t->w_rows >= t->stripe_row_limit)
		orc_flush_stripe(t);
}

/* Bulk insert: cols[c][i], colnulls[c] may be NULL.  Ends with a flush, like the end
 * of an INSERT / COPY statement (write_state_management.c flushes per statement). */
void orc_insert(OrcTable *t, const int64_t *const *cols, const uint8_t *const *colnulls, int64_t n)
{
	int64_t *vals = malloc(sizeof(int64_t) * (size_t) t->natts);
	uint8_t *nulls = malloc((size_t) t->natts);
	for (int64_t i = 0; i < n; i++)
	{
		for (int c = 0; c < t->natts; c++)
		{
			vals[c] = cols[c][i];
			nulls[c] = (colnulls && colnulls[c]) ? colnulls[c][i] : 0;
		}
		orc_write_row(t, vals, nulls);
	}
	orc_flush_stripe(t);
	free(vals); free(nulls);
}

/*
 * Synthetic rows for the benchmark's reference arm, written through the same row-at-a-time writer.  The
 * counter-based formula is the benchmark's own (include/citus_gpu.h cg_gen_relation), restated here so that
 * the reference arm builds its shards without loading the product library:
 *    value(row, col) = lo + splitmix64(seed ^ col << 56 ^ (first_row + row)) % (hi - lo)
 *    null(row, col)  = splitmix64(~seed ^ col << 56 ^ (first_row + row)) % 1000000 < null_ppm
 * kind 1 = the sequence lo + first_row + row.
 */
typedef struct OrcGenColumn { int32_t attlen; int32_t kind; int64_t lo; int64_t hi; uint32_t null_ppm; uint32_t reserved; } OrcGenColumn;

uint64_t orc_splitmix64(uint64_t x);

void orc_gen_insert(OrcTable *t, const OrcGenColumn *cols, int64_t nrows, uint64_t first_row, uint64_t seed)
{
	int64_t *vals = malloc(sizeof(int64_t) * (size_t) t->natts);
	uint8_t *nulls = malloc((size_t) t->natts);
	for (int64_t i = 0; i < nrows; i++)
	{
		uint64_t row = first_row + (uint64_t) i;
		for (int c = 0; c < t->natts; c++)
		{
			const OrcGenColumn *g = &cols[c];
			nulls[c] = g->null_ppm ? (orc_splitmix64(~seed ^ ((uint64_t) c << 56) ^ row) % 1000000ull < g->null_ppm) : 0;
			if (g->kind == 1) vals[c] = g->lo + (int64_t) row;
			else
			{
				uint64_t span = (uint64_t) (g->hi - g->lo);
				uint64_t h = orc_splitmix64(seed ^ ((uint64_t) c << 56) ^ row);
				vals[c] = g->lo + (int64_t) (span ? h % span : 0);
			}
		}
		orc_write_row(t, vals, nulls);
	}
	orc_flush_stripe(t);
	free(vals); free(nulls);
}

/* accessors for the ctypes wrapper / for handing the image to the product code */
const uint8_t *orc_table_pages(const OrcTable *t) { return t->pages; }
uint64_t orc_table_nblocks(const OrcTable *t) { return t->nblocks; }
int orc_table_nstripes(const OrcTable *t) { return t->nstripes; }
const OrcStripe *orc_table_stripes(const OrcTable *t) { return t->stripes; }
int orc_table_nnodes(const OrcTable *t) { return t->nnodes; }
const OrcSkipNode *orc_table_nodes(const OrcTable *t) { return t->nodes; }

/* ------------------------------------------------------------------------- *
 *  Scan: skip list -> chunk decode -> row qual -> aggregate.
 * ------------------------------------------------------------------------- */

typedef struct OrcQual { int32_t col; int32_t op; int64_t konst; } OrcQual; /* konst: int or float8 bits */

/* term = product over factors of (a + b * col); ncols==0 means the constant 1 (count(*)) */
typedef struct OrcAggSpec
{
	int32_t kind;        /* ORC_AGG_* */
	int32_t nfactors;    /* 0..3 */
	int32_t col[3];
	int32_t is_float;    /* SUM/MIN/MAX over float8: float8pl in scan order */
	int64_t a[3];
	int64_t b[3];
} OrcAggSpec;

typedef struct OrcAggState
{
	int128 isum;     /* [PG] int8_avg_accum / numeric_poly_sum: 128-bit accumulator */
	double fsum;     /* [PG] float8pl, sequential */
	int64_t count;   /* [PG] int8inc / int8inc_any; for SUM/MIN/MAX = number of non-NULL inputs */
	int64_t imin, imax;
	double fmin, fmax;
} OrcAggState;

typedef struct OrcGroup { int64_t key; int32_t key_null; int32_t used; } OrcGroup;

typedef struct OrcScanResult
{
	int64_t ngroups;
	int64_t *keys;           /* [ngroups] packed group key */
	uint8_t *key_nulls;
	int nagg;
	OrcAggState *states;     /* [ngroups][nagg] */
	int64_t rows_scanned;             /* rows handed to the qual (after chunk-group skipping) */
	int64_t rows_removed_by_filter;   /* EXPLAIN "Rows Removed by Filter" */
	int64_t chunk_groups_filtered;    /* "Columnar Chunk Groups Removed by Filter" */
	int64_t rows_passed;
	/* host hash table */
	OrcGroup *slots; int64_t *slot_index; int64_t cap;
	int64_t group_cap;
} OrcScanResult;

static int orc_qual_cmp_true(int atttype, int64_t v, int op, int64_t k)
{
	int c = orc_datum_cmp(atttype, v, k);
	switch (op)
	{
		case ORC_OP_LT: return c < 0;
		case ORC_OP_LE: return c <= 0;
		case ORC_OP_EQ: return c == 0;
		case ORC_OP_GE: return c >= 0;
		case ORC_OP_GT: return c > 0;
		default: return c != 0;
	}
}

/*
 * WHERE as a boolean tree over the atoms ([PG] BoolExpr AND / OR; NOT is folded into the operators):
 * postfix tokens, >= 0 = atom index, -1 = AND, -2 = OR, set per thread right before a scan; no tokens =
 * the atoms are an AND-list.
 *   row:   [PG] ExecQual (execExprInterp.c) -- the row passes iff the tree is TRUE; under three-valued logic
 *          without NOT that is: atom on a NULL input -> not TRUE, AND -> both TRUE, OR -> either TRUE
 *   chunk: [PG] predicate_refuted_by (predtest.c) against the base constraint of ONE column
 *          (columnar_reader.c:1132-1187 loops over whereClauseVars): the implicit AND-list and an AND clause
 *          are refuted when any arm is, an OR clause when every arm is; an atom on another column never is
 * Pinned by expected/columnar_chunk_filtering.out (pushdown_test: OR of equalities, OR of AND arms).
 */
static __thread int orc_nqexpr = 0;
static __thread int8_t orc_qexpr[32];
void orc_set_qual_expr(const int8_t *tokens, int n)
{
	orc_nqexpr = n < 0 ? 0 : (n > 32 ? 32 : n);
	for (int i = 0; i < orc_nqexpr; i++) orc_qexpr[i] = tokens[i];
}

/*
 * columnar_reader.c:1132-1187 SelectedChunkMask + :1234 BuildBaseConstraint +
 * :1358 UpdateConstraint; [PG] predicate_refuted_by (predtest.c) restated for the
 * clause shapes the GPU path accepts: "col <op> const" atoms with btree operators.
 * The base constraint (col >= min AND col <= max) is refuted by an atom on the same column
 * that contradicts either half:
 *    col <  k refutes col >= min  iff  min >= k
 *    col <= k refutes col >= min  iff  min >  k
 *    col =  k refutes either half iff  k < min or k > max
 *    col >= k refutes col <= max  iff  max <  k
 *    col >  k refutes col <= max  iff  max <= k
 *    col <> k refutes nothing (no btree refutation from a range to <>)
 * Pinned by expected/columnar_chunk_filtering.out.
 */
static int orc_atom_refuted(const OrcTable *t, const OrcSkipNode *node, int col, const OrcQual *q)
{
	if (q->col != col) return 0;
	int ty = t->atttype[col];
	int64_t k = q->konst;
	int cmin = orc_datum_cmp(ty, node->min_value, k);
	int cmax = orc_datum_cmp(ty, node->max_value, k);
	switch (q->op)
	{
		case ORC_OP_LT: return cmin >= 0;
		case ORC_OP_LE: return cmin > 0;
		case ORC_OP_EQ: return cmin > 0 || cmax < 0;
		case ORC_OP_GE: return cmax < 0;
		case ORC_OP_GT: return cmax <= 0;
		default: return 0;
	}
}

static int orc_chunk_refuted(const OrcTable *t, const OrcSkipNode *node, int col,
							 const OrcQual *quals, int nquals)
{
	if (!node->has_minmax) return 0;
	if (orc_nqexpr == 0)
	{
		for (int q = 0; q < nquals; q++)
			if (orc_atom_refuted(t, node, col, &quals[q])) return 1;
		return 0;
	}
	int st[32], sp = 0;
	for (int i = 0; i < orc_nqexpr; i++)
	{
		int tok = orc_qexpr[i];
		if (tok >= 0) st[sp++] = orc_atom_refuted(t, node, col, &quals[tok]);
		else { int b = st[--sp], a = st[--sp]; st[sp++] = tok == -1 ? (a || b) : (a && b); }
	}
	return st[0];
}

/* [PG] ExecQual: is the WHERE tree TRUE for row i? */
static int orc_row_passes(const OrcTable *t, const OrcQual *quals, int nquals, uint8_t **exists, int64_t **values, uint32_t i)
{
	int truth[32];
	for (int q = 0; q < nquals; q++)
	{
		int c = quals[q].col;
		truth[q] = exists[c][i] && orc_qual_cmp_true(t->atttype[c], values[c][i], quals[q].op, quals[q].konst);
	}
	if (orc_nqexpr == 0)
	{
		for (int q = 0; q < nquals; q++) if (!truth[q]) return 0;
		return 1;
	}
	int st[32], sp = 0;
	for (int k = 0; k < orc_nqexpr; k++)
	{
		int tok = orc_qexpr[k];
		if (tok >= 0) st[sp++] = truth[tok];
		else { int b = st[--sp], a = st[--sp]; st[sp++] = tok == -1 ? (a && b) : (a || b); }
	}
	return st[0];
}

static inline uint64_t orc_mix64(uint64_t x)
{
	x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33;
	return x;
}

static int64_t orc_group_lookup(OrcScanResult *r, int64_t key, int key_null)
{
	if ((r->ngroups + 1) * 2 > r->cap)
	{
		int64_t ncap = r->cap ? r->cap * 2 : 1024;
		OrcGroup *ns = calloc((size_t) ncap, sizeof(OrcGroup));
		int64_t *ni = malloc(sizeof(int64_t) * (size_t) ncap);
		for (int64_t i = 0; i < r->cap; i++)
			if (r->slots[i].used)
			{
				uint64_t h = orc_mix64((uint64_t) r->slots[i].key + (uint64_t) r->slots[i].key_null) & (uint64_t) (ncap - 1);
				while (ns[h].used) h = (h + 1) & (uint64_t) (ncap - 1);
				ns[h] = r->slots[i]; ni[h] = r->slot_index[i];
			}
		free(r->slots); free(r->slot_index);
		r->slots = ns; r->slot_index = ni; r->cap = ncap;
	}
	uint64_t h = orc_mix64((uint64_t) key + (uint64_t) key_null) & (uint64_t) (r->cap - 1);
	while (r->slots[h].used)
	{
		if (r->slots[h].key == key && r->slots[h].key_null == key_null) return r->slot_index[h];
		h = (h + 1) & (uint64_t) (r->cap - 1);
	}
	r->slots[h].used = 1; r->slots[h].key = key; r->slots[h].key_null = key_null;
	int64_t g = r->ngroups++;
	r->slot_index[h] = g;
	if (r->ngroups > r->group_cap)
	{
		r->group_cap = r->group_cap ? r->group_cap * 2 : 1024;
		r->keys = realloc(r->keys, sizeof(int64_t) * (size_t) r->group_cap);
		r->key_nulls = realloc(r->key_nulls, (size_t) r->group_cap);
		r->states = realloc(r->states, sizeof(OrcAggState) * (size_t) r->group_cap * (size_t) (r->nagg ? r->nagg : 1));
	}
	r->keys[g] = key; r->key_nulls[g] = (uint8_t) key_null;
	for (int a = 0; a < r->nagg; a++)
	{
		OrcAggState *s = &r->states[g * r->nagg + a];
		memset(s, 0, sizeof *s);
	}
	return g;
}

OrcScanResult *orc_result_create(int nagg)
{
	OrcScanResult *r = calloc(1, sizeof *r);
	r->nagg = nagg;
	return r;
}

void orc_result_free(OrcScanResult *r)
{
	if (!r) return;
	free(r->keys); free(r->key_nulls); free(r->states); free(r->slots); free(r->slot_index); free(r);
}

int64_t orc_result_ngroups(const OrcScanResult *r) { return r->ngroups; }
int64_t orc_result_counter(const OrcScanResult *r, int which)
{
	switch (which)
	{
		case 0: return r->rows_scanned;
		case 1: return r->rows_removed_by_filter;
		case 2: return r->chunk_groups_filtered;
		default: return r->rows_passed;
	}
}

/* all groups at once: keys[n], key_nulls[n], and per (group, aggregate) sum_hi / sum_lo / count [n * nagg] */
void orc_result_export(const OrcScanResult *r, int64_t *keys, uint8_t *key_nulls, int64_t *sum_hi, uint64_t *sum_lo, int64_t *count)
{
	for (int64_t g = 0; g < r->ngroups; g++)
	{
		keys[g] = r->keys[g]; key_nulls[g] = r->key_nulls[g];
		for (int a = 0; a < r->nagg; a++)
		{
			const OrcAggState *s = &r->states[g * r->nagg + a];
			sum_hi[g * r->nagg + a] = (int64_t) (s->isum >> 64);
			sum_lo[g * r->nagg + a] = (uint64_t) s->isum;
			count[g * r->nagg + a] = s->count;
		}
	}
}

/* copy out group g: key, null flag, and for aggregate a: sum (hi,lo), count, min, max, fsum */
void orc_result_group(const OrcScanResult *r, int64_t g, int64_t *key, int32_t *key_null)
{
	*key = r->keys[g]; *key_null = r->key_nulls[g];
}

void orc_result_agg(const OrcScanResult *r, int64_t g, int a, int64_t *sum_hi, uint64_t *sum_lo,
					int64_t *count, int64_t *imin, int64_t *imax, double *fsum, double *fmin, double *fmax)
{
	const OrcAggState *s = &r->states[g * r->nagg + a];
	*sum_hi = (int64_t) (s->isum >> 64); *sum_lo = (uint64_t) s->isum;
	*count = s->count; *imin = s->imin; *imax = s->imax; *fsum = s->fsum; *fmin = s->fmin; *fmax = s->fmax;
}

/*
 * One shard task: the subtree under ExecAgg in SURVEY.md 3.3.
 *   columnar_reader.c:1007-1060 LoadFilteredStripeBuffers (skip + load projected columns)
 *   columnar_reader.c:1583-1654 DeserializeChunkData (R5 DecompressBuffer,
 *       :1506-1534 DeserializeBoolArray, :1542-1572 DeserializeDatumArray)
 *   columnar_reader.c:868-901 ReadChunkGroupNextRow (row transposition)
 *   columnar_customscan.c:1907-1913 ExecScan -> [PG] ExecQual: three-valued logic, a
 *       NULL comparison drops the row; the qual is re-checked on every surviving row
 *   [PG] nodeAgg + transition functions: count(*) int8inc, count(x) skips NULL,
 *       sum(int) 128-bit accumulate, sum(float8) float8pl in scan order, min/max btree
 *       order; an aggregate over an expression with a NULL input sees NULL (strict ops).
 * group_cols: up to 2 columns; with 2 columns both must be <= 4 bytes wide and the
 * packed key is (uint32) k0 | (uint64)(uint32) k1 << 32.
 * Accumulates into `res` (so several shards / stripes can be merged like the
 * coordinator would, and per-shard results can be produced by fresh `res`).
 */
int orc_scan_aggregate(const OrcTable *t, const OrcQual *quals, int nquals,
					   int enable_qual_pushdown,
					   const int *group_cols, int ngroup_cols,
					   const OrcAggSpec *aggs, int nagg, OrcScanResult *res)
{
	if (res->nagg != nagg) ORC_FAIL("result has %d aggregates, scan has %d", res->nagg, nagg);
	if (ngroup_cols > 2) ORC_FAIL("at most 2 group columns");
	/* projection: columnar_customscan.c:1813-1851 ColumnarAttrNeeded */
	uint8_t *projected = calloc((size_t) t->natts, 1);
	for (int q = 0; q < nquals; q++) projected[quals[q].col] = 1;
	for (int g = 0; g < ngroup_cols; g++) projected[group_cols[g]] = 1;
	for (int a = 0; a < nagg; a++)
		for (int f = 0; f < aggs[a].nfactors; f++) projected[aggs[a].col[f]] = 1;

	uint32_t maxChunkRows = t->chunk_row_limit;
	uint8_t **exists = calloc((size_t) t->natts, sizeof(uint8_t *));
	int64_t **values = calloc((size_t) t->natts, sizeof(int64_t *));
	for (int c = 0; c < t->natts; c++)
		if (projected[c])
		{
			exists[c] = malloc(maxChunkRows);
			values[c] = malloc(sizeof(int64_t) * maxChunkRows);
		}
	/* a varlena numeric(15,2) datum is at most 4 + 2 + 2 * 5 bytes, padded to 16 */
	uint8_t *rawbuf = malloc((size_t) maxChunkRows * 32 * 2 + 1024 * 1024);
	uint64_t rawcap = (uint64_t) maxChunkRows * 32 * 2 + 1024 * 1024;
	uint8_t *valbuf = malloc((size_t) maxChunkRows * 32 + 16);
	uint8_t *bitbuf = malloc(maxChunkRows / 8 + 16);
	int rc = 0;

	for (int si = 0; si < t->nstripes && rc == 0; si++)
	{
		const OrcStripe *s = &t->stripes[si];
		for (uint32_t k = 0; k < s->chunk_count && rc == 0; k++)
		{
			/* SelectedChunkMask: loop over the columns that appear in the WHERE list */
			int selected = 1;
			if (enable_qual_pushdown)
				for (int c = 0; c < t->natts && selected; c++)
				{
					int has = 0;
					for (int q = 0; q < nquals; q++) if (quals[q].col == c) has = 1;
					if (!has) continue;
					const OrcSkipNode *node = &t->nodes[s->skipnode_base + (uint32_t) c * s->chunk_count + k];
					if (orc_chunk_refuted(t, node, c, quals, nquals)) selected = 0;
				}
			if (!selected) { res->chunk_groups_filtered++; continue; }

			uint32_t rowCount = (uint32_t) t->nodes[s->skipnode_base + k].row_count;
			for (int c = 0; c < t->natts && rc == 0; c++)
			{
				if (!projected[c]) continue;
				const OrcSkipNode *node = &t->nodes[s->skipnode_base + (uint32_t) c * s->chunk_count + k];
				if (node->exists_length > maxChunkRows / 8 + 16) { rc = -1; snprintf(orc_errbuf, sizeof orc_errbuf, "exists buffer too large"); break; }
				if (orc_storage_read(t->pages, t->nblocks, s->file_offset + node->exists_offset, bitbuf, node->exists_length)) { rc = -1; break; }
				if (node->value_length > rawcap) { rawcap = node->value_length * 2; rawbuf = realloc(rawbuf, rawcap); }
				if (orc_storage_read(t->pages, t->nblocks, s->file_offset + node->value_offset, rawbuf, node->value_length)) { rc = -1; break; }
				if (node->decompressed_size > (uint64_t) maxChunkRows * 32) { rc = -1; snprintf(orc_errbuf, sizeof orc_errbuf, "value buffer too large"); break; }
				if (orc_decompress(rawbuf, node->value_length, node->compression_type, node->decompressed_size, valbuf)) { rc = -1; break; }

				/* DeserializeBoolArray */
				if ((uint64_t) rowCount > node->exists_length * 8) { rc = -1; snprintf(orc_errbuf, sizeof orc_errbuf, "insufficient data for reading boolean array"); break; }
				for (uint32_t i = 0; i < rowCount; i++)
					exists[c][i] = (bitbuf[i / 8] & (1 << (i % 8))) != 0;
				/* DeserializeDatumArray: fetch_att, advance by attlen, align */
				uint32_t off = 0;
				for (uint32_t i = 0; i < rowCount; i++)
				{
					if (!exists[c][i]) continue;
					int e = orc_read_datum(t, c, valbuf, &off, node->decompressed_size, &values[c][i]);
					if (e == -2) { rc = -1; snprintf(orc_errbuf, sizeof orc_errbuf, "numeric value outside the column's scale / int64 range"); break; }
					if (e || off > node->decompressed_size) { rc = -1; snprintf(orc_errbuf, sizeof orc_errbuf, "insufficient data left in datum buffer"); break; }
				}
			}
			if (rc) break;

			for (uint32_t i = 0; i < rowCount && rc == 0; i++)
			{
				res->rows_scanned++;
				int pass = orc_row_passes(t, quals, nquals, exists, values, i);
				if (!pass) { res->rows_removed_by_filter++; continue; }
				res->rows_passed++;

				int64_t key = 0; int key_null = 0;
				if (ngroup_cols == 1)
				{
					int c = group_cols[0];
					if (!exists[c][i]) key_null = 1; else key = values[c][i];
				}
				else if (ngroup_cols == 2)
				{
					int c0 = group_cols[0], c1 = group_cols[1];
					if (!exists[c0][i] || !exists[c1][i]) { rc = -1; snprintf(orc_errbuf, sizeof orc_errbuf, "NULL in multi-column group key is not supported"); break; }
					key = (int64_t) ((uint64_t) (uint32_t) values[c0][i] | ((uint64_t) (uint32_t) values[c1][i] << 32));
				}
				int64_t g = orc_group_lookup(res, key, key_null);
				for (int a = 0; a < nagg; a++)
				{
					const OrcAggSpec *sp = &aggs[a];
					OrcAggState *st = &res->states[g * nagg + a];
					if (sp->kind == ORC_AGG_COUNT_STAR) { st->count++; continue; }
					int isnull = 0, overflow = 0;
					int128 iv = 1; double fv = 1.0;
					for (int f = 0; f < sp->nfactors; f++)
					{
						int c = sp->col[f];
						if (!exists[c][i]) { isnull = 1; break; }
						if (sp->is_float)
						{
							double d; memcpy(&d, &values[c][i], 8);
							double da, db; memcpy(&da, &sp->a[f], 8); memcpy(&db, &sp->b[f], 8);
							fv *= (da + db * d);
						}
						else
						{
							/* [PG] int8mul / int8pl: b*x, a + b*x and every partial product must fit int64 */
							int128 m = (int128) sp->b[f] * (int128) values[c][i];
							int128 t = (int128) sp->a[f] + m;
							if (m > INT64_MAX || m < INT64_MIN || t > INT64_MAX || t < INT64_MIN) overflow = 1;
							iv *= t;
							if (iv > INT64_MAX || iv < INT64_MIN) overflow = 1;
							if (overflow) iv = 0;
						}
					}
					if (isnull) continue;
					if (overflow && (sp->kind == ORC_AGG_SUM || sp->kind == ORC_AGG_MIN || sp->kind == ORC_AGG_MAX))
					{
						rc = -1;
						snprintf(orc_errbuf, sizeof orc_errbuf, "bigint out of range");
						break;
					}
					switch (sp->kind)
					{
						case ORC_AGG_COUNT: st->count++; break;
						case ORC_AGG_SUM:
							if (sp->is_float) st->fsum += fv; else st->isum += iv;
							st->count++;
							break;
						case ORC_AGG_MIN:
							if (sp->is_float) { if (st->count == 0 || orc_float8_cmp(fv, st->fmin) < 0) st->fmin = fv; }
							else { if (st->count == 0 || (int64_t) iv < st->imin) st->imin = (int64_t) iv; }
							st->count++;
							break;
						case ORC_AGG_MAX:
							if (sp->is_float) { if (st->count == 0 || orc_float8_cmp(fv, st->fmax) > 0) st->fmax = fv; }
							else { if (st->count == 0 || (int64_t) iv > st->imax) st->imax = (int64_t) iv; }
							st->count++;
							break;
					}
				}
			}
		}
	}

	for (int c = 0; c < t->natts; c++) { free(exists[c]); free(values[c]); }
	free(exists); free(values); free(projected); free(rawbuf); free(valbuf); free(bitbuf);
	return rc;
}

/*
 * Coordinator combine (R14): planner/multi_logical_optimizer.c:1807-1885 and
 * :2231-2275 -- sum(partial sums), sum(partial counts) (COALESCE(...,0) handled by the
 * caller), min/max of partial mins/maxs.  Merges `src` into `dst`, group by group.
 */
int orc_combine(OrcScanResult *dst, const OrcScanResult *src, const OrcAggSpec *aggs)
{
	if (dst->nagg != src->nagg) ORC_FAIL("aggregate count mismatch");
	for (int64_t g = 0; g < src->ngroups; g++)
	{
		int64_t d = orc_group_lookup(dst, src->keys[g], src->key_nulls[g]);
		for (int a = 0; a < src->nagg; a++)
		{
			const OrcAggState *s = &src->states[g * src->nagg + a];
			OrcAggState *o = &dst->states[d * dst->nagg + a];
			int had = o->count > 0;
			if (s->count == 0) continue;
			o->isum += s->isum;
			o->fsum += s->fsum;
			if (aggs[a].kind == ORC_AGG_MIN)
			{
				if (!had || s->imin < o->imin) o->imin = s->imin;
				if (!had || orc_float8_cmp(s->fmin, o->fmin) < 0) o->fmin = s->fmin;
			}
			if (aggs[a].kind == ORC_AGG_MAX)
			{
				if (!had || s->imax > o->imax) o->imax = s->imax;
				if (!had || orc_float8_cmp(s->fmax, o->fmax) > 0) o->fmax = s->fmax;
			}
			o->count += s->count;
		}
	}
	dst->rows_scanned += src->rows_scanned;
	dst->rows_removed_by_filter += src->rows_removed_by_filter;
	dst->chunk_groups_filtered += src->chunk_groups_filtered;
	dst->rows_passed += src->rows_passed;
	return 0;
}

/* Decode every row of the projected columns (used to cross-check the product-side
 * shard writer and the GPU decode kernel): out_values[c][row], out_nulls[c][row]. */
int orc_decode_all(const OrcTable *t, int64_t **out_values, uint8_t **out_nulls, int64_t *out_rows)
{
	int64_t row = 0;
	uint8_t *rawbuf = NULL; uint64_t rawcap = 0;
	uint8_t *valbuf = malloc((size_t) t->chunk_row_limit * 32 + 16);
	uint8_t *bitbuf = malloc(t->chunk_row_limit / 8 + 16);
	for (int si = 0; si < t->nstripes; si++)
	{
		const OrcStripe *s = &t->stripes[si];
		for (uint32_t k = 0; k < s->chunk_count; k++)
		{
			uint32_t rowCount = (uint32_t) t->nodes[s->skipnode_base + k].row_count;
			for (int c = 0; c < t->natts; c++)
			{
				const OrcSkipNode *node = &t->nodes[s->skipnode_base + (uint32_t) c * s->chunk_count + k];
				if (orc_storage_read(t->pages, t->nblocks, s->file_offset + node->exists_offset, bitbuf, node->exists_length)) return -1;
				if (node->value_length > rawcap) { rawcap = node->value_length * 2 + 64; rawbuf = realloc(rawbuf, rawcap); }
				if (orc_storage_read(t->pages, t->nblocks, s->file_offset + node->value_offset, rawbuf, node->value_length)) return -1;
				if (orc_decompress(rawbuf, node->value_length, node->compression_type, node->decompressed_size, valbuf)) return -1;
				uint32_t off = 0;
				for (uint32_t i = 0; i < rowCount; i++)
				{
					int ex = (bitbuf[i / 8] & (1 << (i % 8))) != 0;
					out_nulls[c][row + i] = !ex;
					out_values[c][row + i] = 0;
					if (!ex) continue;
					if (orc_read_datum(t, c, valbuf, &off, node->decompressed_size, &out_values[c][row + i])) return -1;
				}
			}
			row += rowCount;
		}
	}
	*out_rows = row;
	free(rawbuf); free(valbuf); free(bitbuf);
	return 0;
}

/* ------------------------------------------------------------------------- *
 *  Synthetic row generator shared with the product-side generator by
 *  SPECIFICATION only (counter-based, so both sides can produce row i of shard s
 *  independently): splitmix64(seed, shard, column, row).
 * ------------------------------------------------------------------------- */
uint64_t orc_splitmix64(uint64_t x)
{
	x += 0x9e3779b97f4a7c15ULL;
	x = (x ^ (x >> 30)) * 0xbf58476d1ce4e5b9ULL;
	x = (x ^ (x >> 27)) * 0x94d049bb133111ebULL;
	return x ^ (x >> 31);
}

/* ------------------------------------------------------------------------- *
 *  Attach to a relation image written by someone else (the product-side shard
 *  writer): the oracle's reader then decodes / scans it independently.
 *  OrcStripe / OrcSkipNode are field-for-field the reference's StripeMetadata /
 *  ColumnChunkSkipNode subset, the same layout include/citus_gpu.h uses.
 * ------------------------------------------------------------------------- */
OrcTable *orc_table_attach(const uint8_t *pages, uint64_t nblocks, const OrcStripe *stripes, int nstripes,
						   const OrcSkipNode *nodes, int nnodes, int natts, const int *attlen,
						   const int *atttype, uint32_t chunk_row_limit)
{
	OrcTable *t = orc_table_create(natts, attlen, atttype, 150000, chunk_row_limit, ORC_COMP_NONE, 3);
	free(t->pages);
	t->pages = malloc(nblocks * ORC_BLCKSZ);
	memcpy(t->pages, pages, nblocks * ORC_BLCKSZ);
	t->nblocks = nblocks; t->cap_blocks = nblocks;
	t->stripes = malloc(sizeof(OrcStripe) * (size_t) (nstripes ? nstripes : 1));
	memcpy(t->stripes, stripes, sizeof(OrcStripe) * (size_t) nstripes);
	t->nstripes = nstripes; t->cap_stripes = nstripes;
	t->nodes = malloc(sizeof(OrcSkipNode) * (size_t) (nnodes ? nnodes : 1));
	memcpy(t->nodes, nodes, sizeof(OrcSkipNode) * (size_t) nnodes);
	t->nnodes = nnodes; t->cap_nodes = nnodes;
	return t;
}

/* Same, without copying: the caller keeps the image alive (bench.py's cpu_baseline leg
 * attaches to the 2 GB shard images the product-side generator already holds).
 * nstripes may be smaller than the relation's stripe count: a bounded sample. */
OrcTable *orc_table_attach_view(const uint8_t *pages, uint64_t nblocks, const OrcStripe *stripes, int nstripes,
								const OrcSkipNode *nodes, int nnodes, int natts, const int *attlen,
								const int *atttype, uint32_t chunk_row_limit)
{
	OrcTable *t = orc_table_create(natts, attlen, atttype, 150000, chunk_row_limit, ORC_COMP_NONE, 3);
	free(t->pages);
	t->pages = (uint8_t *) pages;
	t->nblocks = nblocks; t->cap_blocks = nblocks;
	t->stripes = (OrcStripe *) stripes;
	t->nstripes = nstripes; t->cap_stripes = nstripes;
	t->nodes = (OrcSkipNode *) nodes;
	t->nnodes = nnodes; t->cap_nodes = nnodes;
	t->borrowed = 1;
	return t;
}
