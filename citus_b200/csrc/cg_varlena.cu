/*
 * cg_varlena.cu -- SURVEY.md 8(f) row 4, first slice: by-reference columns whose values are scaled integers
 * (numeric(p, s), e.g. TPC-H's decimal(15,2)) or one character (char(1) flags), so that the reference's own
 * lineitem DDL (test/regress/sql/multi_create_table.sql:12-28) scans without re-declaring the columns.
 *
 * In the value stream of such a column (columnar_writer.c:555-585 SerializeSingleDatum, columnar_reader.c:1557-1565
 * DeserializeDatumArray) every non-NULL row is a complete varlena -- [PG] 1-byte header when bit 0 is set (total
 * length = header >> 1) or 4-byte header (total length = header >> 2) -- padded to the type's alignment ('i' = 4)
 * relative to the start of the stream.  Where a datum starts therefore depends on all datums before it.  One warp
 * decodes one chunk: 8 KB tiles of the stream are staged in shared memory with coalesced 16-byte loads, lane 0 walks
 * the headers of the tile (shared-memory latency instead of global) and records where the datums start, then all
 * lanes decode datums in parallel into a dense fixed-width array (int64 value * 10^scale for numeric; for char(1) the
 * byte zero-extended to 16 bits, so that it compares unsigned like bpchar's memcmp) in the chunk's decoded slot.  The scan kernels then see an ordinary fixed-width column.
 * [PG] numeric on-disk format (numeric.c): base-10000 digits, value = sum d[i] * 10000^(weight - i); short header
 * 0x8000 | sign 0x2000 | dscale << 7 | weight (7 bits, two's complement), long header sign/dscale + int16 weight.
 */
#include "cg_internal.h"

#define CGV_TILE 8192
#define CGV_MAX_DATUMS (CGV_TILE / 4)
#define CGV_WARPS 3

__device__ __forceinline__ uint32_t vl_total(const uint8_t *p)
{
	return (p[0] & 1u) ? (uint32_t) (p[0] >> 1) : (*(const uint32_t *) p >> 2);
}

/* numeric datum -> value * 10^scale; false when NaN / +-Infinity / more fractional digits than the scale / outside
 * [-2^63, 2^63 - 1] */
__device__ bool numeric_to_scaled(const uint8_t *datum, uint32_t total, int scale, int64_t *out)
{
	const uint32_t hdr = (datum[0] & 1u) ? 1u : 4u;
	if (total < hdr + 2u) return false;
	const uint8_t *p = datum + hdr;
	const int n = (int) (total - hdr);
	const uint16_t h = (uint16_t) (p[0] | (p[1] << 8));
	bool neg;
	int weight, nd;
	const uint8_t *dp;
	if ((h & 0xC000u) == 0x8000u)
	{
		neg = (h & 0x2000u) != 0;
		weight = (h & 0x0040u) ? (int) (h & 0x003Fu) - 64 : (int) (h & 0x003Fu);
		dp = p + 2; nd = (n - 2) / 2;
	}
	else
	{
		if ((h & 0xC000u) == 0xC000u || n < 4) return false;
		neg = (h & 0xC000u) == 0x4000u;
		weight = (int) (int16_t) (p[2] | (p[3] << 8));
		dp = p + 4; nd = (n - 4) / 2;
	}
	if (nd == 0) { *out = 0; return true; }
	if (nd > 9) return false;                         /* more than 36 decimal digits cannot fit */
	unsigned __int128 acc = 0;
	for (int i = 0; i < nd; i++) acc = acc * 10000u + (uint32_t) (uint16_t) (dp[2 * i] | (dp[2 * i + 1] << 8));
	int e10 = 4 * (weight - (nd - 1)) + scale;
	if (e10 > 19) return false;
	while (e10 > 0) { acc *= 10u; e10--; if (acc > ((unsigned __int128) 1 << 100)) return false; }
	while (e10 < 0) { if (acc % 10u != 0) return false; acc /= 10u; e10++; }
	if (acc > (unsigned __int128) INT64_MAX + (neg ? 1u : 0u)) return false;
	*out = (int64_t) (neg ? 0u - (uint64_t) acc : (uint64_t) acc);
	return true;
}

__global__ void __launch_bounds__(CGV_WARPS * 32)
cg_varlena_decode_kernel(uint8_t *arena, const VarlenaItem *items, uint64_t nitems, unsigned long long *err, unsigned long long flag)
{
	__shared__ __align__(16) uint8_t s_tile[CGV_WARPS][CGV_TILE + 16];
	__shared__ uint16_t s_off[CGV_WARPS][CGV_MAX_DATUMS];
	const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const uint64_t item = (uint64_t) blockIdx.x * CGV_WARPS + warp;
	if (item >= nitems) return;
	const VarlenaItem it = items[item];
	const uint8_t *src = arena + it.src;                  /* 16-byte aligned slot */
	uint8_t *tile = s_tile[warp];
	uint16_t *offs = s_off[warp];
	uint32_t pos = 0;                                     /* stream offset of the next datum (multiple of 4) */
	uint32_t done = 0;                                    /* datums decoded so far */
	bool bad = false;
	while (done < it.count && !bad)
	{
		const uint32_t base = pos & ~15u;                 /* tile start, 16-byte aligned */
		const uint32_t avail = min((uint32_t) CGV_TILE, it.raw_len - base);
		for (uint32_t o = lane * 16; o < avail; o += 32 * 16)
			*(uint4 *) (tile + o) = *(const uint4 *) (src + base + o);        /* the slot is padded: reads past raw_len stay inside it */
		__syncwarp();
		uint32_t nd = 0;
		if (lane == 0)
		{
			uint32_t p = pos - base;
			while (done + nd < it.count && nd < CGV_MAX_DATUMS)
			{
				if (p + 4 > avail && !(p + 1 <= avail && (tile[p] & 1u))) break;       /* header not in the tile */
				const uint32_t total = vl_total(tile + p);
				if (total < 1u || total > 4096u) { nd = 0xffffffffu; break; }           /* malformed */
				if (p + total > avail) break;                                          /* the datum continues in the next tile */
				offs[nd++] = (uint16_t) p;
				p += (total + 3u) & ~3u;
			}
			if (nd != 0xffffffffu) pos = base + p;
		}
		nd = __shfl_sync(0xffffffffu, nd, 0);
		pos = __shfl_sync(0xffffffffu, pos, 0);
		if (nd == 0xffffffffu || nd == 0) { bad = true; break; }      /* malformed, or a datum larger than a tile */
		__syncwarp();
		for (uint32_t j = lane; j < nd; j += 32)
		{
			const uint8_t *d = tile + offs[j];
			const uint32_t total = vl_total(d);
			if (it.kind == CG_TYPE_NUMERIC)
			{
				int64_t v = 0;
				if (!numeric_to_scaled(d, total, (int) it.scale, &v)) bad = true;
				*(int64_t *) (arena + it.dst + (uint64_t) (done + j) * 8) = v;
			}
			else
			{
				const uint32_t hdr = (d[0] & 1u) ? 1u : 4u;
				if (total != hdr + 1u) bad = true;                      /* char(1): exactly one byte of payload */
				*(uint16_t *) (arena + it.dst + (uint64_t) (done + j) * 2) = d[hdr];   /* unsigned, like bpchar's memcmp */
			}
		}
		done += nd;
		bad = __any_sync(0xffffffffu, bad);
		__syncwarp();
	}
	if (bad && lane == 0) atomicOr(err, flag);
}

int cg_launch_varlena_decode(CgContext *ctx, uint8_t *arena, const VarlenaItem *items, uint64_t nitems, unsigned long long *err,
							 unsigned long long flag, cudaStream_t stream)
{
	if (nitems == 0) return CG_OK;
	int rc = cg_chain_end(ctx, stream);
	if (rc) return rc;
	const unsigned blocks = (unsigned) ((nitems + CGV_WARPS - 1) / CGV_WARPS);
	cg_varlena_decode_kernel<<<blocks, CGV_WARPS * 32, 0, stream>>>(arena, items, nitems, err, flag);
	CG_CUDA(cudaGetLastError()); g_cg_launches++;
	return CG_OK;
}
