/*
 * cg_decompress.cu -- value-stream decompression on the GPU (K7).
 *
 * Replaces DecompressBuffer, backend/columnar/columnar_compression.c:165-270, for the two
 * byte-oriented LZ77 codecs a columnar chunk can carry:
 *
 *   COMPRESSION_LZ4   :186-208  LZ4_decompress_safe(buffer, out, len, decompressedSize), and the
 *                               result must be exactly decompressedSize bytes.  liblz4 is not part
 *                               of the reference tree; the block format is the published one
 *                               (token = literal length << 4 | match length - 4, 255-continued
 *                               lengths, literals, 16-bit little-endian offset; the last sequence
 *                               has literals only).
 *   COMPRESSION_PG_LZ :240-267  8-byte ColumnarCompressHeader {vl_len_, rawsize} (:38-42), VARSIZE
 *                               must equal the buffer length, then PostgreSQL's
 *                               pglz_decompress(..., check_complete = true) (src/common/
 *                               pg_lzcompress.c: control byte = 8 items, LSB first; bit set = tag
 *                               [len-3 | off>>8 <<4][off & 0xff][+1 length byte when len == 18],
 *                               bit clear = one literal byte).
 *
 * The exists bitmap is never compressed (columnar_writer.c:606-653).  Zstandard streams have their
 * own kernel at the end of this file (cg_zstd.cuh holds the decoder).
 *
 * Eight lanes decode one chunk buffer, four streams per warp (a C2 relation has ~10^5 streams per
 * column, so the grid is wide; sequences of columnar value streams are a few bytes long, so
 * eight lanes fill a copy and a full warp per stream only wastes issue slots).
 * A stream is a chain of dependent steps -- token, lengths, literal copy, offset,
 * match copy -- so its rate is set by the latency of one step; both ends of the copy therefore
 * stay in shared memory: the compressed stream is pulled through a 256-byte ring per stream
 * (aligned 16-byte loads, one refill per 128 bytes consumed) and the decoded bytes go through a
 * 2 KB window per stream that is written to the arena in aligned 16-byte vectors (see struct Out).
 * A match of any length and any overlap is copied in parallel: byte i of the match is
 * out[pos - off + (i mod off)], which only reads bytes written before the match began.  Lanes
 * communicate through shared memory, ordered by __syncwarp(group mask).
 *
 * A malformed stream never writes outside the item's slot; it raises `flag` in *err and the
 * host reports CG_ECORRUPT ("cannot decompress the buffer") at its next synchronisation.
 */
#include <algorithm>
#include <stdlib.h>

#include "cg_internal.h"
#include "cg_lz4_lane.cuh"
#include "cg_zstd.cuh"

#define CGD_WARPS 4
#define CGD_GROUP 8u                    /* lanes per stream */
#define CGD_GROUPS (32u / CGD_GROUP)    /* streams per warp */
#define CGD_RING 256u
#define CGD_WIN 2048u
#define CGD_CHUNK 256u
#define CG_LZ4_LANES_DEFAULT 2      /* 2 = by launch size (see cg_lz4_lane_kernel); cg_set_option("lz4_lanes", 1 / 0) / CG_LZ4_LANES force one kernel */
#define CG_LZ4_LANES_MAX_WARPS_PER_SM 16

struct Stream
{
	const uint8_t *src;     /* 16-byte aligned */
	uint32_t len;           /* bytes in the stream */
	uint32_t loadable;      /* bytes that may be read (the slot, a multiple of 16) */
	uint32_t base;          /* ring holds [base, base + CGD_RING) */
	volatile uint8_t *ring;
	uint32_t glane, mask;   /* lane inside the group, the group's lanes */

	__device__ __forceinline__ void fill(uint32_t from)   /* 128 bytes at stream position `from` */
	{
		uint32_t p = from + 16u * glane;
		uint4 w = make_uint4(0, 0, 0, 0);
		if (p < loadable) w = *(const uint4 *) (src + p);
		*(uint4 *) ((uint8_t *) ring + (p & (CGD_RING - 1))) = w;
	}
	__device__ __forceinline__ void open()
	{
		base = 0;
		fill(0);
		fill(128);
		__syncwarp(mask);
	}
	/* after the call [ip, ip + 128) is in the ring */
	__device__ __forceinline__ void ensure(uint32_t ip)
	{
		while (ip >= base + 128u)
		{
			__syncwarp(mask);             /* every lane is done reading the half being replaced */
			fill(base + CGD_RING);
			base += 128u;
			__syncwarp(mask);
		}
	}
	__device__ __forceinline__ uint32_t at(uint32_t p) const { return ring[p & (CGD_RING - 1)]; }
};

/*
 * The output goes through a per-stream window in shared memory: the last CGD_WIN bytes of the
 * decoded stream live in a ring, matches whose source is still in the ring are shared-memory
 * copies (the common case: columnar value streams repeat at distances of a few values), and the
 * ring is written to the arena in aligned 16-byte vectors when it is full.  Only a match that
 * reaches further back than the ring reads the arena (after a flush).
 */
struct Out
{
	volatile uint8_t *ring;
	uint8_t *dst;           /* 16-byte aligned arena slot */
	uint32_t op;            /* bytes decoded so far */
	uint32_t flushed;       /* bytes already in dst (multiple of 16) */
	uint32_t glane, mask;

	/* ring -> dst for [flushed, upto & ~15) */
	__device__ __forceinline__ void flush(uint32_t upto)
	{
		upto &= ~15u;
		__syncwarp(mask);                 /* every lane has finished writing the ring */
		for (uint32_t pos = flushed + 16u * glane; pos < upto; pos += 16u * CGD_GROUP)
			*(uint4 *) (dst + pos) = *(const uint4 *) ((const uint8_t *) ring + (pos & (CGD_WIN - 1)));
		flushed = upto;
		__syncwarp(mask);                 /* the flushed part of the ring may be overwritten from here on */
	}
	/* before writing m more bytes (m <= CGD_CHUNK): nothing unflushed may be overwritten */
	__device__ __forceinline__ void make_room(uint32_t m)
	{
		if (op + m - flushed > CGD_WIN) flush(op);
	}
};

/* the n bytes at stream position ip (n may be large) */
__device__ __forceinline__ void put_literals(Stream &s, Out &o, uint32_t ip, uint32_t n)
{
	while (n)
	{
		s.ensure(ip);
		uint32_t m = min(min(n, s.base + CGD_RING - ip), CGD_CHUNK);
		o.make_room(m);
		for (uint32_t i = o.glane; i < m; i += CGD_GROUP) o.ring[(o.op + i) & (CGD_WIN - 1)] = (uint8_t) s.at(ip + i);
		ip += m; o.op += m; n -= m;
	}
}

/* n bytes starting `off` bytes back, LZ77 overlap semantics: byte i is out[op - off + (i mod off)] */
__device__ __forceinline__ void put_match(Out &o, uint32_t off, uint32_t n)
{
	/* i mod off for i = glane, glane + 8, ... kept incrementally (no division) */
	uint32_t k0 = o.glane, step = CGD_GROUP;
	if (off <= CGD_GROUP)
	{
		while (k0 >= off) k0 -= off;
		while (step >= off) step -= off;
	}
	while (n)
	{
		const uint32_t m = min(n, CGD_CHUNK);
		o.make_room(m);
		uint32_t k = k0;
		if (off + m <= CGD_WIN)
		{
			__syncwarp(o.mask);                          /* the bytes the match reads are in the ring */
			const uint32_t from = o.op - off;
			for (uint32_t i = o.glane; i < m; i += CGD_GROUP)
			{
				o.ring[(o.op + i) & (CGD_WIN - 1)] = o.ring[(from + k) & (CGD_WIN - 1)];
				k += step; if (k >= off) k -= off;
			}
		}
		else
		{
			/* far match: its source left the ring long ago and is in the arena once the ring is flushed
			 * (off > CGD_WIN - CGD_CHUNK, so the source ends before the unflushed tail) */
			o.flush(o.op);
			const uint8_t *from = o.dst + (o.op - off);
			for (uint32_t i = o.glane; i < m; i += CGD_GROUP)
			{
				o.ring[(o.op + i) & (CGD_WIN - 1)] = from[k];
				k += step; if (k >= off) k -= off;
			}
		}
		o.op += m; n -= m;
		__syncwarp(o.mask);               /* no lane runs ahead and overwrites ring bytes another lane still reads */
		/* a chunk that overlaps itself continues the same periodic pattern: (i + m) mod off */
	}
}

static __device__ bool lz4_block(Stream &s, Out &o, uint32_t rawlen)
{
	uint32_t ip = 0;
	const uint32_t clen = s.len;
	if (clen == 0) return false;
	for (;;)
	{
		s.ensure(ip);
		if (ip >= clen) return false;
		const uint32_t token = s.at(ip++);
		uint32_t lit = token >> 4;
		if (lit == 15)
		{
			uint32_t b;
			do
			{
				s.ensure(ip);
				if (ip >= clen) return false;
				b = s.at(ip++);
				lit += b;
				if (lit > rawlen) return false;
			} while (b == 255);
		}
		if (lit > clen - ip || lit > rawlen - o.op) return false;
		put_literals(s, o, ip, lit);
		ip += lit;
		if (ip == clen) break;                       /* the last sequence stops after its literals */
		s.ensure(ip);
		if (clen - ip < 2) return false;
		const uint32_t off = s.at(ip) | (s.at(ip + 1) << 8);
		ip += 2;
		uint32_t ml = token & 15;
		if (ml == 15)
		{
			uint32_t b;
			do
			{
				s.ensure(ip);
				if (ip >= clen) return false;
				b = s.at(ip++);
				ml += b;
				if (ml > rawlen) return false;
			} while (b == 255);
		}
		ml += 4;
		if (off == 0 || off > o.op || ml > rawlen - o.op) return false;
		put_match(o, off, ml);
	}
	return o.op == rawlen;
}

static __device__ bool pglz_stream(Stream &s, Out &o, uint32_t rawlen)
{
	/* ColumnarCompressHeader: int32 vl_len_ (4-byte varlena header, little endian: length << 2 | flags), int32 rawsize */
	if (s.len < 8) return false;
	uint32_t hdr = s.at(0) | (s.at(1) << 8) | (s.at(2) << 16) | (s.at(3) << 24);
	uint32_t raw = s.at(4) | (s.at(5) << 8) | (s.at(6) << 16) | (s.at(7) << 24);
	if (((hdr >> 2) & 0x3FFFFFFFu) != s.len) return false;     /* compressedDataSize + HDRSZ != buffer->len */
	if (raw != rawlen) return false;
	uint32_t sp = 8;
	const uint32_t srcend = s.len;
	while (sp < srcend && o.op < rawlen)
	{
		s.ensure(sp);
		uint32_t ctrl = s.at(sp++);
		for (int c = 0; c < 8 && sp < srcend && o.op < rawlen; c++, ctrl >>= 1)
		{
			s.ensure(sp);
			if (ctrl & 1)
			{
				uint32_t b0 = s.at(sp), b1 = s.at(sp + 1);
				uint32_t len = (b0 & 0x0f) + 3;
				uint32_t off = ((b0 & 0xf0) << 4) | b1;
				sp += 2;
				if (len == 18) len += s.at(sp++);
				if (sp > srcend || off == 0 || off > o.op) return false;
				len = min(len, rawlen - o.op);
				put_match(o, off, len);
			}
			else
			{
				o.make_room(1);
				if (o.glane == 0) o.ring[o.op & (CGD_WIN - 1)] = (uint8_t) s.at(sp);
				sp++; o.op++;
			}
		}
	}
	return o.op == rawlen && sp == srcend;           /* check_complete */
}

/* The four groups of a warp run the same code on different streams.  Their masks are run-time
 * values on purpose: giving each group its own copy of the code with a constant mask (one WARPSYNC
 * per barrier instead of a MATCH/VOTE sequence) made the groups diverge for good and was an order of
 * magnitude slower; with one copy the groups mostly stay converged. */
__global__ void __launch_bounds__(CGD_WARPS * 32)
cg_decompress_kernel(uint8_t *arena, const DecodeItem *items, uint32_t nitems, unsigned long long *err,
					 unsigned long long flag, int skip_lz4)
{
	__shared__ __align__(16) uint8_t rings[CGD_WARPS * CGD_GROUPS][CGD_RING];
	__shared__ __align__(16) uint8_t wins[CGD_WARPS * CGD_GROUPS][CGD_WIN];
	const uint32_t lane = threadIdx.x & 31u;
	const uint32_t group = threadIdx.x / CGD_GROUP;                 /* within the CTA */
	const uint32_t idx = blockIdx.x * (CGD_WARPS * CGD_GROUPS) + group;
	if (idx >= nitems) return;
	const DecodeItem it = items[idx];
	if (it.kind == CG_COMPRESSION_ZSTD) return;                     /* cg_zstd_kernel's */
	if (skip_lz4 && it.kind == CG_COMPRESSION_LZ4) return;          /* cg_lz4_lane_kernel's */
	Stream s;
	s.src = arena + it.src;
	s.len = it.comp_len;
	s.loadable = (it.comp_len + 15u) & ~15u;
	s.ring = rings[group];
	s.glane = lane % CGD_GROUP;
	s.mask = ((1u << CGD_GROUP) - 1u) << (lane - s.glane);
	s.open();
	Out o;
	o.ring = wins[group];
	o.dst = arena + it.dst;
	o.op = 0;
	o.flushed = 0;
	o.glane = s.glane;
	o.mask = s.mask;
	bool ok;
	if (it.kind == CG_COMPRESSION_LZ4) ok = lz4_block(s, o, it.raw_len);
	else if (it.kind == CG_COMPRESSION_PGLZ) ok = pglz_stream(s, o, it.raw_len);
	else ok = false;
	if (ok)
	{
		/* what is left in the ring, then the slot's zero padding (like every other arena slot) */
		o.flush(o.op);
		for (uint32_t i = o.flushed + o.glane; i < it.raw_len; i += CGD_GROUP) o.dst[i] = o.ring[i & (CGD_WIN - 1)];
	}
	for (uint32_t i = (ok ? it.raw_len : 0u) + o.glane; i < it.padded; i += CGD_GROUP) o.dst[i] = 0;
	if (!ok && o.glane == 0) atomicOr(err, flag);
}

/*
 * Zstandard (cg_zstd.cuh): entropy decoding (FSE state machines, Huffman bit streams) is a serial
 * dependency chain per stream, so the serial parts run on ONE lane as ordinary sequential code
 * -- the same source the CPU-side format tests run on the host -- and the parallelism comes from
 * the number of streams (a C2 shard has ~10^4) plus the warp-cooperative parts below.  One warp per CTA; its FSE tables (ZstdTables, ~7 KB)
 * live in shared memory, its Huffman table and literals buffer (132 KB) in a context-owned scratch area; persistent
 * CTAs stride over the decode list.  The other lanes only help with the slot's zero padding.
 */
#define CGD_ZSTD_SCRATCH (ZSTD_BLOCK_MAX + 64 + sizeof(HufEntry) * (1u << ZSTD_HUF_LOG_MAX))   /* literals + Huffman table */

/*
 * The warp-cooperative form of one frame.  What is serial stays on lane 0 and is the very code the
 * host tests exercise (headers, Huffman tree, FSE tables, zs_sequences_next: the entropy-coded
 * sequence stream is one dependency chain); what is not serial is spread over the warp:
 *   - raw / RLE blocks and literal sections: lane-parallel copies and fills
 *   - the four Huffman streams of a literals section: one lane each
 *   - sequence execution in batches of 32: lane 0 decodes 32 (literal length, match length, offset)
 *     triples into shared memory, a warp prefix sum gives every sequence its literal and output
 *     positions, the literal runs are copied one per lane, the matches in order with all lanes on
 *     each (byte i of a match is out[start - off + i mod off], as in the lz4 decoder).
 */
struct ZsShared
{
	ZsLitPlan L;
	ZsSeq S;
	uint32_t ll[32], ml[32], off[32];
	int status;
	uint32_t hdr_pos, has_fcs, fcs_lo, checksum;
};

static __device__ int64_t zstd_block_coop(ZstdTables &T, ZsShared &C, const uint8_t *src, uint32_t len, uint8_t *dst, uint32_t op,
										   uint32_t cap, uint8_t *lit, uint32_t lane)
{
	if (lane == 0) C.status = zs_literals_prepare(T, src, len, &C.L);
	__syncwarp();
	if (C.status < 0) return ZSTD_ERR;
	const uint32_t nlit = C.L.regen;
	if (C.L.kind == 0) { for (uint32_t i = lane; i < nlit; i += 32) lit[i] = C.L.raw[i]; }
	else if (C.L.kind == 1) { const uint8_t b = C.L.raw[0]; for (uint32_t i = lane; i < nlit; i += 32) lit[i] = b; }
	else if (lane < (uint32_t) C.L.nstreams)
	{
		if (zs_huf_stream(T, C.L.sptr[lane], C.L.slen[lane], lit + C.L.sout[lane], C.L.scount[lane]) < 0) C.status = ZSTD_ERR;
	}
	__syncwarp();
	if (C.status < 0) return ZSTD_ERR;
	if (lane == 0) C.status = zs_sequences_begin(T, src + C.L.consumed, len - C.L.consumed, &C.S);
	__syncwarp();
	if (C.status < 0) return ZSTD_ERR;
	const uint32_t nseq = C.S.nseq;
	uint32_t litpos = 0;
	for (uint32_t base = 0; base < nseq; base += 32)
	{
		const uint32_t nb = min(32u, nseq - base);
		if (lane == 0)
		{
			/* the iterator state lives in registers while the batch is decoded */
			ZsSeq S = C.S;
			int st = 0;
			for (uint32_t j = 0; j < nb && st == 0; j++)
			{
				uint32_t a, b, c;
				st = zs_sequences_next(T, &S, &a, &b, &c);
				C.ll[j] = a; C.ml[j] = b; C.off[j] = c;
			}
			C.S = S;
			C.status = st;
		}
		__syncwarp();
		if (C.status < 0) return ZSTD_ERR;
		const uint32_t l = lane < nb ? C.ll[lane] : 0u, m = lane < nb ? C.ml[lane] : 0u, o = lane < nb ? C.off[lane] : 1u;
		uint32_t pl = l, pt = l + m;                                 /* inclusive prefix sums over the batch */
#pragma unroll
		for (int d = 1; d < 32; d <<= 1)
		{
			const uint32_t a = __shfl_up_sync(0xffffffffu, pl, d), b = __shfl_up_sync(0xffffffffu, pt, d);
			if (lane >= (uint32_t) d) { pl += a; pt += b; }
		}
		const uint32_t tot_l = __shfl_sync(0xffffffffu, pl, 31), tot_t = __shfl_sync(0xffffffffu, pt, 31);
		if (tot_l > nlit - litpos || tot_t > cap - op) return ZSTD_ERR;
		const uint32_t my_lit = litpos + pl - l;                     /* where my literals come from */
		const uint32_t my_out = op + pt - (l + m);                   /* where they go; my match starts l bytes later */
		if (__any_sync(0xffffffffu, lane < nb && o > my_out + l)) return ZSTD_ERR;     /* offset beyond the output so far */
		for (uint32_t i = 0; i < l; i++) dst[my_out + i] = lit[my_lit + i];
		__syncwarp();
		for (uint32_t j = 0; j < nb; j++)
		{
			const uint32_t mj = __shfl_sync(0xffffffffu, m, j), oj = __shfl_sync(0xffffffffu, o, j);
			const uint32_t start = __shfl_sync(0xffffffffu, my_out + l, j);
			uint32_t k = lane, step = 32u;
			if (oj <= 32u)
			{
				while (k >= oj) k -= oj;
				while (step >= oj) step -= oj;
			}
			const uint8_t *from = dst + start - oj;
			for (uint32_t i = lane; i < mj; i += 32)
			{
				dst[start + i] = from[k];
				k += step; if (k >= oj) k -= oj;
			}
			__syncwarp();
		}
		litpos += tot_l; op += tot_t;
	}
	if (lane == 0) C.status = zs_sequences_end(&C.S);
	__syncwarp();
	if (C.status < 0) return ZSTD_ERR;
	const uint32_t rest = nlit - litpos;
	if (rest > cap - op) return ZSTD_ERR;
	for (uint32_t i = lane; i < rest; i += 32) dst[op + i] = lit[litpos + i];
	__syncwarp();
	return (int64_t) op + rest;
}

static __device__ int64_t zstd_frame_coop(ZstdTables &T, ZsShared &C, const uint8_t *src, uint32_t len, uint8_t *dst, uint32_t cap,
										   uint8_t *lit, uint32_t lane)
{
	if (lane == 0)
	{
		uint64_t fcs = 0;
		int checksum = 0;
		int hp = zs_frame_header(src, len, cap, &fcs, &checksum);
		C.status = hp < 0 ? ZSTD_ERR : 0;
		C.hdr_pos = (uint32_t) hp; C.has_fcs = fcs != ~0ull; C.fcs_lo = (uint32_t) fcs; C.checksum = (uint32_t) checksum;
		T.huf_log = 0; T.have_ll = T.have_of = T.have_ml = 0;
		T.rep[0] = 1; T.rep[1] = 4; T.rep[2] = 8;
	}
	__syncwarp();
	if (C.status < 0) return ZSTD_ERR;
	uint32_t pos = C.hdr_pos, op = 0;
	for (;;)
	{
		if (pos + 3 > len) return ZSTD_ERR;
		const uint32_t bh = src[pos] | ((uint32_t) src[pos + 1] << 8) | ((uint32_t) src[pos + 2] << 16);
		pos += 3;
		const uint32_t last = bh & 1u, type = (bh >> 1) & 3u, bsize = bh >> 3;
		if (type == 0)
		{
			if (bsize > ZSTD_BLOCK_MAX || pos + bsize > len || bsize > cap - op) return ZSTD_ERR;
			for (uint32_t i = lane; i < bsize; i += 32) dst[op + i] = src[pos + i];
			op += bsize; pos += bsize;
			__syncwarp();
		}
		else if (type == 1)
		{
			if (bsize > ZSTD_BLOCK_MAX || pos + 1 > len || bsize > cap - op) return ZSTD_ERR;
			const uint8_t b = src[pos];
			for (uint32_t i = lane; i < bsize; i += 32) dst[op + i] = b;
			op += bsize; pos += 1;
			__syncwarp();
		}
		else if (type == 2)
		{
			if (bsize > ZSTD_BLOCK_MAX || pos + bsize > len) return ZSTD_ERR;
			const int64_t nop = zstd_block_coop(T, C, src + pos, bsize, dst, op, cap, lit, lane);
			if (nop < 0 || nop - (int64_t) op > (int64_t) ZSTD_BLOCK_MAX) return ZSTD_ERR;
			op = (uint32_t) nop; pos += bsize;
		}
		else
			return ZSTD_ERR;
		if (last) break;
	}
	if (C.checksum) { if (pos + 4 > len) return ZSTD_ERR; pos += 4; }
	if (pos != len) return ZSTD_ERR;
	if (C.has_fcs && C.fcs_lo != op) return ZSTD_ERR;
	return (int64_t) op;
}

__global__ void __launch_bounds__(32)
cg_zstd_kernel(uint8_t *arena, const DecodeItem *items, uint32_t nitems, uint8_t *lit_scratch, unsigned long long *err,
			   unsigned long long flag, int coop)
{
	__shared__ ZstdTables T;
	__shared__ ZsShared C;
	__shared__ int s_ok;
	const uint32_t lane = threadIdx.x;
	uint8_t *lit = lit_scratch + (size_t) blockIdx.x * CGD_ZSTD_SCRATCH;
	if (lane == 0) T.huf = (HufEntry *) (lit + ZSTD_BLOCK_MAX + 64);
	__syncwarp();
	for (uint32_t idx = blockIdx.x; idx < nitems; idx += gridDim.x)
	{
		const DecodeItem it = items[idx];
		if (it.kind != CG_COMPRESSION_ZSTD) continue;
		uint8_t *dst = arena + it.dst;
		bool ok;
		if (coop)
		{
			/* "unexpected decompressed size" (columnar_compression.c:226-232) */
			ok = zstd_frame_coop(T, C, arena + it.src, it.comp_len, dst, it.raw_len, lit, lane) == (int64_t) it.raw_len;
			__syncwarp();
		}
		else
		{
			if (lane == 0) s_ok = zs_decode_frame(T, arena + it.src, it.comp_len, dst, it.raw_len, lit) == (int64_t) it.raw_len;
			__syncwarp();
			ok = s_ok != 0;
		}
		if (!ok && lane == 0) atomicOr(err, flag);
		for (uint32_t i = (ok ? it.raw_len : 0u) + lane; i < it.padded; i += 32) dst[i] = 0;
		__syncwarp();
	}
}

/*
 * LZ4, a lane per stream (cg_lz4_lane.cuh).  One warp per CTA; the first `active` lanes of the warp take a stream each,
 * and their windows (CGL_WIN bytes each, interleaved) are the CTA's dynamic shared memory.
 *
 * On launches of 1875 streams of 80 KB (one block of a shard), one stream per warp beats the eight lanes per stream of
 * cg_decompress_kernel; several streams per warp, every lane on its own, lose (lanes drift apart and a warp runs them one
 * after the other), and re-converging after every sequence does not help (the branches of a step still run one after
 * the other, each with its own load latencies).  On a whole shard in one launch (9375 streams, the DMA path) one stream
 * per warp is 63 warps per SM with 31 of 32 SIMD lanes idle, bound by instruction issue and slower than the eight-lane
 * kernel.  So: the lane kernel for launches of up to 16 warps per SM, the eight-lane kernel above that ("lz4_lanes" -1,
 * the default).
 */
#define CGL_CTA_WARPS 1u
__global__ void __launch_bounds__(CGL_CTA_WARPS * 32)
cg_lz4_lane_kernel(uint8_t *arena, const DecodeItem *items, uint32_t nitems, unsigned long long *err, unsigned long long flag,
				   uint32_t active, int lockstep)
{
	extern __shared__ __align__(16) uint8_t lane_win[];
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	const uint32_t idx = (blockIdx.x * CGL_CTA_WARPS + warp) * active + lane;
	DecodeItem it;
	memset(&it, 0, sizeof it);
	it.kind = 0xffffffffu;
	if (lane < active && idx < nitems) it = items[idx];
	const bool mine = it.kind == CG_COMPRESSION_LZ4;
	Lz4Lane L;
	L.src = arena + it.src; L.clen = it.comp_len;
	L.dst = arena + it.dst; L.rawlen = it.raw_len;
	L.wb = lane_win + (size_t) warp * CGL_WIN * active + 4u * (lane < active ? lane : 0u); L.wstride = 4u * active;
	int st = mine ? cgl_begin(L) : CGL_DONE;
	if (lockstep)
	{
		while (__any_sync(0xffffffffu, st == CGL_MORE))
		{
			if (st == CGL_MORE) st = cgl_step(L);
			__syncwarp();
		}
	}
	else
		while (st == CGL_MORE) st = cgl_step(L);
	if (!mine) return;
	if (!(st == CGL_DONE && cgl_finish(L, it.padded)))
	{
		for (uint32_t i = 0; i < it.padded; i++) L.dst[i] = 0;
		atomicOr(err, flag);
	}
}

static int g_lz4_lanes = -1;
static int g_lz4_lane_warps = 64;         /* > 0: as few streams per warp as fit into that many warps per SM, each lane on its own; 0: 32 streams per warp in step (probe) */
static int g_zstd_coop = -1;              /* 1: zstd_frame_coop (default), 0: zs_decode_frame on one lane; < 0: CG_ZSTD_COOP, else 1 */
void cg_decompress_set_lz4_lane_warps(int n) { g_lz4_lane_warps = n < 0 ? 0 : n > 64 ? 64 : n; }
void cg_decompress_set_lz4_lanes(int on) { g_lz4_lanes = on < 0 ? -1 : (on > 1 ? 2 : on); }      /* < 0: back to the default */
void cg_decompress_set_zstd_coop(int on) { g_zstd_coop = on < 0 ? -1 : (on ? 1 : 0); }         /* < 0: back to the default */

/* h_items: the host copy of the same items (which kernels are needed) */
int cg_launch_decompress(CgContext *ctx, uint8_t *arena, const DecodeItem *items, const DecodeItem *h_items, uint64_t nitems,
						 unsigned long long *err, unsigned long long flag, cudaStream_t stream)
{
	if (nitems == 0) return CG_OK;
	int rc = cg_chain_end(ctx, stream);
	if (rc) return rc;
	if (g_lz4_lanes < 0) { const char *e = getenv("CG_LZ4_LANES"); g_lz4_lanes = e ? atoi(e) : CG_LZ4_LANES_DEFAULT; if (g_lz4_lanes < 0 || g_lz4_lanes > 2) g_lz4_lanes = CG_LZ4_LANES_DEFAULT; }
	const int use_lanes = g_lz4_lanes == 2 ? (nitems <= (uint64_t) ctx->sm_count * CG_LZ4_LANES_MAX_WARPS_PER_SM ? 1 : 0) : g_lz4_lanes;
	bool any_lz = false, any_zstd = false, any_lz4 = false;
	for (uint64_t i = 0; i < nitems; i++)
	{
		if (h_items[i].kind == CG_COMPRESSION_ZSTD) any_zstd = true;
		else if (h_items[i].kind == CG_COMPRESSION_LZ4 && use_lanes) any_lz4 = true;
		else any_lz = true;
	}
	if (any_lz4)
	{
		uint32_t active = 32;
		int lockstep = 1;                         /* g_lz4_lane_warps == 0 (probe): 32 streams per warp, in step */
		if (g_lz4_lane_warps > 0)
		{
			/* as few streams per warp as fit into g_lz4_lane_warps warps per SM, every lane on its own */
			active = 1; lockstep = 0;
			while (active < 32 && (nitems + active - 1) / active > (uint64_t) ctx->sm_count * (uint64_t) g_lz4_lane_warps) active <<= 1;
		}
		const uint64_t per_cta = (uint64_t) CGL_CTA_WARPS * active;
		const unsigned blocks = (unsigned) ((nitems + per_cta - 1) / per_cta);
		const size_t smem = (size_t) CGL_WIN * active * CGL_CTA_WARPS;
		static bool configured = false;
		if (!configured)
		{
			CG_CUDA(cudaFuncSetAttribute(cg_lz4_lane_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) (CGL_WIN * 32u * CGL_CTA_WARPS)));
			configured = true;
		}
		cg_lz4_lane_kernel<<<blocks, CGL_CTA_WARPS * 32, smem, stream>>>(arena, items, (uint32_t) nitems, err, flag, active, lockstep);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
	}
	if (any_lz)
	{
		const unsigned per_block = CGD_WARPS * CGD_GROUPS;
		unsigned blocks = (unsigned) ((nitems + per_block - 1) / per_block);
		cg_decompress_kernel<<<blocks, CGD_WARPS * 32, 0, stream>>>(arena, items, (uint32_t) nitems, err, flag, use_lanes);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
	}
	if (any_zstd)
	{
		static int occ = 0;
		if (occ == 0)
		{
			CG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, cg_zstd_kernel, 32, 0));
			if (occ < 1) occ = 1;
		}
		const unsigned max_blocks = (unsigned) (ctx->sm_count * occ);
		const size_t need = (size_t) max_blocks * CGD_ZSTD_SCRATCH;
		if (ctx->zstd_scratch_bytes < need)
		{
			/* grown once; every launch uses block-indexed slices, launches on different streams would
			 * share them, so zstd decoding always runs on the stream it was first used with or after a sync */
			if (ctx->zstd_scratch) CG_CUDA(cudaFree(ctx->zstd_scratch));
			ctx->zstd_scratch = nullptr; ctx->zstd_scratch_bytes = 0;
			if (cudaMalloc((void **) &ctx->zstd_scratch, need) != cudaSuccess)
			{
				cudaGetLastError();
				return cg_set_error(CG_ENOMEM, "cudaMalloc of %zu bytes of zstd literal scratch failed", need);
			}
			ctx->zstd_scratch_bytes = need;
		}
		unsigned blocks = (unsigned) std::min<uint64_t>(nitems, max_blocks);
		if (g_zstd_coop < 0) { const char *e = getenv("CG_ZSTD_COOP"); g_zstd_coop = (e && atoi(e) == 0) ? 0 : 1; }
		cg_zstd_kernel<<<blocks, 32, 0, stream>>>(arena, items, (uint32_t) nitems, ctx->zstd_scratch, err, flag, g_zstd_coop);
		CG_CUDA(cudaGetLastError()); g_cg_launches++;
	}
	return CG_OK;
}
