/*
 * aocs.cu - the storage side of aocs_getnext on the device: one column's segment-file bytes in, one
 * decoded column of a relation out.
 *
 * Restates, for a whole column at once, what the reference does per row and per block:
 *   datumstreamread_block -> AppendOnlyStorageRead_GetBlockInfo / _Content
 *       (utils/datumstream/datumstream.c:1364; cdb/cdbappendonlystorageread.c:954,1136): walk the
 *       Append-Only storage blocks of the column file; header layout
 *       include/cdb/cdbappendonlystorage_int.h:64-147 (AOSmallContentHeader bit fields), length =
 *       8 + 2 x CRC-32C (if checksummed) + 8 (firstRowNum), cdb/cdbappendonlystorageformat.c:81-113;
 *       content rounded up to 8 bytes (include/cdb/cdbappendonlystorage.h:37-42)
 *   DatumStreamBlockRead_GetReadyOrig (utils/datumstream/datumstreamblock.c:153-354): 16-byte
 *       DatumStreamBlock_Orig header (include/utils/datumstreamblock.h:74-83), NULL bitmap of
 *       `nullsz` bytes when DSB_HAS_NULLBITMAP, datum area at the next MAXALIGN boundary
 *   DatumStreamBlockRead_AdvanceOrig / _Get (include/utils/datumstreamblock.h:1442-1540,1220-1440):
 *       NULL rows take no datum space; fixed width: next = cur + datumlen; varlena: next = cur +
 *       VARSIZE_ANY, then zero pad bytes are skipped up to the type's alignment
 *   numeric datums (include/utils/numeric.h:103-189: short / long header, base-10000 digits) become
 *       int64 scaled by the column's display scale, char(1) datums their byte - the same decoded form
 *       the rest of the path works on (DESIGN.md "data layout in HBM").
 *
 * The host walks the block headers (16 bytes read per block) into a directory; the file is copied to
 * the device as it lies; one warp decodes one block: NULL bitmap -> ballot / popcount gives every
 * row its physical datum index; fixed-width datums are then gathered in parallel; varlena datums are
 * located by lane 0 walking 32 lengths at a time, and decoded by all lanes.
 *
 *   Dense blocks (compresstype = rle_type, compresslevel 1: DatumStreamBlock_Dense + Rle_Extension,
 *       include/utils/datumstreamblock.h:86-170; GetReadyDense datumstreamblock.c:627-1010; AdvanceDense
 *       datumstreamblock.h:1725-1960): the NULL bitmap has one bit per NON-REPEATED position, the
 *       compress bitmap one bit per physical datum, a set bit = "repeats `count` more times", counts in
 *       the 1-4 byte codec of datumstreamblock.h:617-730.  A warp takes 32 positions at a time: lane 0
 *       decodes their repeat counts (and varlena offsets), a warp scan of the run lengths gives every
 *       position its first output row, short runs are written by their lane, long runs by the warp.
 *
 * Supported: uncompressed SmallContent / NonBulkDenseContent storage blocks holding Original or Dense
 * (RLE and / or delta range) datum stream blocks - everything `compresstype=rle_type,
 * compresslevel=1` writes.  Delta range encoding (int4 / int8 / date columns; AdvanceDenseDelta,
 * datumstreamblock.h:1625-1723: a set delta bit = "previous value +/- a 29-bit delta", codec :779-900)
 * is a running sum: per trip an affine-map scan across the warp.  Bulk-compressed (zlib / zstd) and
 * large-content blocks are refused with CBGPU_ERR_UNSUPPORTED, never guessed at.
 */
#include "common.cuh"
#include "inflate.cuh"
#include "like_match.cuh"
#include "zstd_dec.cuh"

#include <stdlib.h>
#include <string.h>

struct AocsDir
{
	long long	hoff;			/* storage block header offset in the file                            */
	int32_t		overall;		/* header + firstRowNum + stored content rounded up                   */
	int32_t		clen;			/* compressed length of the stored content, 0 = stored as is          */
	long long	zoff;			/* compressed content offset in the file (clen > 0)                   */
	long long	off;			/* content offset: in the file, or in the inflate area behind it      */
	long long	rowbase;		/* first output row of the block                                      */
	long long	first;			/* the block's firstRowNum (AO row number of its first row), -1 if absent */
	int32_t		rows;
	int32_t		dlen;
};

/* one distinct string of a dictionary: tag = 64-bit hash of its bytes (never 0), bytes at arena[off, off + len) */
struct DictSlot
{
	unsigned long long tag;
	uint32_t	off;
	uint32_t	len;
	int32_t		code;			/* assigned by cbgpu_dict_finalize                                    */
	int32_t		pad;
};

struct AocsParams
{
	const uint8_t *raw;
	const AocsDir *dir;
	int32_t		nblocks;
	int32_t		attlen;			/* 1 / 2 / 4 / 8, or -1 varlena                                       */
	int32_t		varkind;		/* CBGPU_AOCS_VAR_NUMERIC / _BPCHAR1                                  */
	int32_t		typalign;		/* 1 / 2 / 4 / 8                                                      */
	int32_t		dscale;			/* numeric: scale of the output integers                              */
	void	   *out;
	uint8_t    *outnull;		/* NULL when no block of the file has a NULL bitmap                   */
	int		   *status;
	/* dictionary columns (CBGPU_AOCS_VAR_DICT): the string set of a cbgpu_dict */
	struct DictSlot *dslots;
	uint8_t    *darena;
	unsigned long long *dcursor;	/* [0] arena bytes used, [1] entries                              */
	uint32_t	dmask;
	uint32_t	darena_cap;
	int32_t		dmode;			/* 1 collect distinct strings, 2 look codes up                        */
	int32_t		dtrim;			/* bpchar: trailing blanks do not count (bcTruelen, utils/adt/varchar.c) */
	int32_t		doutw;			/* 1 (CB_DICT8) or 4 (CB_DICT32)                                      */
	int32_t		dmax;			/* entries the table may hold                                         */
};

#define AOCS_WARPS 4

__device__ __forceinline__ uint32_t
aocs_le32(const uint8_t *p)
{
	return (uint32_t) p[0] | ((uint32_t) p[1] << 8) | ((uint32_t) p[2] << 16) | ((uint32_t) p[3] << 24);
}

/* numeric datum body -> integer scaled by 10^dscale; false when it does not fit or is not exact */
__device__ __forceinline__ bool
aocs_numeric(const uint8_t *body, int len, int dscale, int64_t *out)
{
	const uint32_t h = (uint32_t) body[0] | ((uint32_t) body[1] << 8);
	bool		neg;
	int			weight,
				off;

	if ((h & 0xC000u) == 0x8000u)
	{
		/* NUMERIC_SHORT: sign 0x2000, dscale 0x1F80 >> 7, weight sign 0x0040, weight 0x003F */
		neg = (h & 0x2000u) != 0;
		weight = (int) (h & 0x003Fu);
		if (h & 0x0040u)
			weight -= 64;
		off = 2;
	}
	else if ((h & 0xC000u) == 0xC000u)
		return false;			/* NaN / infinity have no integer form */
	else
	{
		neg = (h & 0xC000u) == 0x4000u;
		weight = (int) (int16_t) ((uint32_t) body[2] | ((uint32_t) body[3] << 8));
		off = 4;
	}
	const int	nd = (len - off) / 2;
	uint64_t	acc = 0;

	for (int i = 0; i < nd; i++)
	{
		const uint32_t d = (uint32_t) body[off + 2 * i] | ((uint32_t) body[off + 2 * i + 1] << 8);

		if (acc > (0x7fffffffffffffffull - d) / 10000ull)
			return false;
		acc = acc * 10000ull + d;
	}
	int			e10 = 4 * (weight - nd + 1) + dscale;

	if (nd == 0)
		acc = 0;
	else if (e10 >= 0)
	{
		for (; e10 > 0; e10--)
		{
			if (acc > 0x7fffffffffffffffull / 10ull)
				return false;
			acc *= 10ull;
		}
	}
	else
	{
		for (; e10 < 0; e10++)
		{
			if (acc % 10ull)
				return false;	/* more fractional digits than the column's scale */
			acc /= 10ull;
		}
	}
	*out = neg ? -(int64_t) acc : (int64_t) acc;
	return true;
}

/* ---------------------------------------------------------------------------------------------
 * CRC-32C (Castagnoli, reflected polynomial 0x82F63B78), as src/port/pg_crc32c_sb8.c computes it.
 * Append-only blocks store it WITHOUT the final inversion (cdbappendonlystorageformat.c:41-46,71-76):
 *   block checksum  (bytes 8..11)  = crc over bytes [16, overall block length)
 *   header checksum (bytes 12..15) = crc over bytes [0, 12)
 * (AppendOnlyStorageFormat_ComputeBlockChecksum / _ComputeHeaderChecksum :27-78, layout :125-190).
 * One warp per block: every lane runs the byte-wise table recurrence over its slice starting from 0,
 * then lane 0 stitches the slices: crc(A || B) = crc(A) * x^(8|B|) mod P  xor  crc0(B)  over GF(2).
 * --------------------------------------------------------------------------------------------- */
__device__ __forceinline__ uint32_t
crc32c_mulmod(uint32_t a, uint32_t b)
{
	/* a * b mod P in the reflected representation (bit 31 = x^0) */
	uint32_t	r = 0;

	for (int i = 0; i < 32; i++)
	{
		if (a & 0x80000000u)
			r ^= b;
		a <<= 1;
		b = (b >> 1) ^ ((b & 1u) ? 0x82F63B78u : 0u);
	}
	return r;
}

/* x^(8 n) mod P */
__device__ __forceinline__ uint32_t
crc32c_xpow8n(uint32_t n)
{
	uint32_t	result = 0x80000000u;	/* 1 */
	uint32_t	sq = 0x00800000u;		/* x^8 */

	while (n)
	{
		if (n & 1u)
			result = crc32c_mulmod(result, sq);
		sq = crc32c_mulmod(sq, sq);
		n >>= 1;
	}
	return result;
}

__global__ void __launch_bounds__(AOCS_WARPS * 32)
k_aocs_verify(const uint8_t *raw, const AocsDir *dir, int nblocks, int *status)
{
	__shared__ uint32_t tab[256];
	const int	lane = threadIdx.x & 31;
	const int	w = threadIdx.x >> 5;
	const int	nwarps = gridDim.x * AOCS_WARPS;

	for (int i = threadIdx.x; i < 256; i += blockDim.x)
	{
		uint32_t	c = (uint32_t) i;

		for (int k = 0; k < 8; k++)
			c = (c >> 1) ^ ((c & 1u) ? 0x82F63B78u : 0u);
		tab[i] = c;
	}
	__syncthreads();
	for (int b = blockIdx.x * AOCS_WARPS + w; b < nblocks; b += nwarps)
	{
		const uint8_t *h = raw + dir[b].hoff;
		const uint32_t len = (uint32_t) dir[b].overall - 16u;
		const uint8_t *d = h + 16;
		const uint32_t per = ((len + 31u) / 32u + 3u) & ~3u;	/* bytes per lane */
		const uint32_t lo = (uint32_t) lane * per < len ? (uint32_t) lane * per : len;
		const uint32_t hi = lo + per < len ? lo + per : len;
		uint32_t	c = 0;

		/* blocks are 8-byte aligned and padded to 8 bytes, slices are whole words */
		for (uint32_t i = lo; i < hi; i += 4)
		{
			c ^= *(const uint32_t *) (d + i);
			c = tab[c & 0xffu] ^ (c >> 8);
			c = tab[c & 0xffu] ^ (c >> 8);
			c = tab[c & 0xffu] ^ (c >> 8);
			c = tab[c & 0xffu] ^ (c >> 8);
		}
		/* stitch: start from the init value, advance it over each slice's length, add the slice's own crc */
		uint32_t	crc = 0xFFFFFFFFu;
		const uint32_t mfull = crc32c_xpow8n(per);

		for (int l = 0; l < 32; l++)
		{
			const uint32_t cl = __shfl_sync(0xffffffffu, c, l);
			const uint32_t nl = __shfl_sync(0xffffffffu, hi - lo, l);

			if (nl == 0)
				continue;
			crc = crc32c_mulmod(crc, nl == per ? mfull : crc32c_xpow8n(nl)) ^ cl;
		}
		if (lane == 0)
		{
			uint32_t	hc = 0xFFFFFFFFu;
			const uint32_t stored_block = aocs_le32(h + 8);
			const uint32_t stored_header = aocs_le32(h + 12);

			for (int i = 0; i < 12; i++)
				hc = tab[(hc ^ h[i]) & 0xffu] ^ (hc >> 8);
			if (hc != stored_header || crc != stored_block)
				atomicExch(status, CBGPU_ERR_CORRUPT);
		}
	}
}

/* ---------------------------------------------------------------------------------------------
 * Bulk-compressed blocks (compresstype=zlib; rle_type compresslevel 2-4): AppendOnlyStorageRead_Content's
 * gp_decompress step (cdbappendonlystorageread.c:1286-1310) on the device.  One warp per block: lane 0 runs the
 * serial Huffman decoder of inflate.cuh into a 32-entry queue, then the warp applies the queue: output positions by a
 * prefix sum over the entries' lengths; literals and matches whose source lies before the batch go in parallel (one
 * entry per lane), matches that read this batch's own output follow in order, each copied by the whole warp.
 * The result lands in the inflate area behind the file image (AocsDir.off), where k_aocs_decode reads it like a
 * block that was stored uncompressed.  Length mismatch (gp_compress.c:73-79) or a bad stream / Adler-32
 * (uncompress() -> Z_DATA_ERROR, pg_compression.c:342-365) raise CBGPU_ERR_CORRUPT.
 * --------------------------------------------------------------------------------------------- */
__device__ __forceinline__ bool
infl_apply_warp(uint8_t *out, uint32_t &outpos, uint32_t cap, const uint32_t *q, int n, int lane)
{
	const uint32_t e = lane < n ? q[lane] : 0u;
	const bool	lit = (e & INFL_LIT) != 0;
	const bool	match = lane < n && !lit;
	const uint32_t len = lane < n ? (lit ? 1u : (e & 511u)) : 0u;
	const uint32_t dist = (e >> 9) & 0xFFFFu;
	uint32_t	incl = len;
	bool		dep = false;

	for (int d = 1; d < 32; d <<= 1)
	{
		const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);

		if (lane >= d)
			incl += v;
	}
	const uint32_t total = __shfl_sync(0xffffffffu, incl, 31);
	const uint32_t start = outpos + incl - len;

	if (outpos + total > cap || __any_sync(0xffffffffu, match && dist > start))
		return false;
	if (lit)
		out[start] = (uint8_t) e;
	else if (match)
	{
		if (start - dist + len <= outpos)
		{
			const uint8_t *src = out + start - dist;

			for (uint32_t i = 0; i < len; i++)
				out[start + i] = src[i];
		}
		else
			dep = true;
	}
	__syncwarp();
	for (unsigned m = __ballot_sync(0xffffffffu, dep); m; m &= m - 1)
	{
		const int	k = __ffs(m) - 1;
		const uint32_t s = __shfl_sync(0xffffffffu, start, k);
		const uint32_t d = __shfl_sync(0xffffffffu, dist, k);
		const uint32_t l = __shfl_sync(0xffffffffu, len, k);

		for (uint32_t i = lane; i < l; i += 32)
			out[s + i] = out[s - d + (d >= l ? i : i % d)];
		__syncwarp();
	}
	outpos += total;
	return true;
}

__device__ __forceinline__ uint32_t
infl_adler32_warp(const uint8_t *d, uint32_t n, int lane)
{
	const uint32_t per = (n + 31u) / 32u;
	const uint32_t lo = (uint32_t) lane * per < n ? (uint32_t) lane * per : n;
	const uint32_t hi = lo + per < n ? lo + per : n;
	uint64_t	a = 0,
				b = 0;

	for (uint32_t i = lo; i < hi; i++)
	{
		a += d[i];
		b += a;
	}
	uint32_t	A = (uint32_t) (a % 65521u);
	uint32_t	B = (uint32_t) ((b + a * (uint64_t) (n - hi)) % 65521u);

	for (int o = 16; o; o >>= 1)
	{
		A += __shfl_xor_sync(0xffffffffu, A, o);
		B += __shfl_xor_sync(0xffffffffu, B, o);
	}
	A = (1u + A) % 65521u;
	B = (n % 65521u + B) % 65521u;
	return (B << 16) | A;
}

__global__ void __launch_bounds__(AOCS_WARPS * 32)
k_aocs_inflate(uint8_t *raw, const AocsDir *dir, int nblocks, int *status, int *anynull)
{
	__shared__ InflTables s_tab[AOCS_WARPS];
	__shared__ uint32_t s_q[AOCS_WARPS][INFL_QN];
	const int	lane = threadIdx.x & 31;
	const int	w = threadIdx.x >> 5;
	const int	nwarps = gridDim.x * AOCS_WARPS;

	if (*status == CBGPU_ERR_CORRUPT)
		return;
	for (int b = blockIdx.x * AOCS_WARPS + w; b < nblocks; b += nwarps)
	{
		const AocsDir D = dir[b];

		if (D.clen == 0)
			continue;
		const uint8_t *in = raw + D.zoff;
		uint8_t    *out = raw + D.off;
		const uint32_t cap = (uint32_t) D.dlen;
		const uint32_t inlen = (uint32_t) D.clen;
		uint32_t	outpos = 0;
		InflState	st;
		bool		ok = true;

		infl_init(st, in, inlen, 2);
		if (lane == 0)
			ok = infl_zlib_header_ok(in, inlen);
		ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
		while (ok)
		{
			int			n = 0,
						rc = INFL_ERROR;

			if (lane == 0)
				rc = infl_step<1>(st, infl_view(s_tab[w]), s_q[w], &n);
			__syncwarp();
			rc = __shfl_sync(0xffffffffu, rc, 0);
			n = __shfl_sync(0xffffffffu, n, 0);
			if (rc == INFL_ERROR || (n && !infl_apply_warp(out, outpos, cap, s_q[w], n, lane)))
			{
				ok = false;
				break;
			}
			if (rc == INFL_STORED)
			{
				const uint32_t src = __shfl_sync(0xffffffffu, st.stored_src, 0);
				const uint32_t len = __shfl_sync(0xffffffffu, st.stored_len, 0);

				if (outpos + len > cap)
				{
					ok = false;
					break;
				}
				for (uint32_t i = lane; i < len; i += 32)
					out[outpos + i] = in[src + i];
				outpos += len;
				__syncwarp();
			}
			if (rc == INFL_DONE)
				break;
		}
		if (ok)
		{
			const uint32_t c = __shfl_sync(0xffffffffu, infl_consumed(st), 0);

			if (outpos != cap || c + 4u > inlen)
				ok = false;
			else
			{
				const uint32_t want = ((uint32_t) in[c] << 24) | ((uint32_t) in[c + 1] << 16) | ((uint32_t) in[c + 2] << 8) | (uint32_t) in[c + 3];

				ok = infl_adler32_warp(out, cap, lane) == want;
			}
		}
		if (lane == 0)
		{
			if (!ok)
				atomicExch(status, CBGPU_ERR_CORRUPT);
			else if (cap > 2 && (out[2] & 1u))	/* DSB_HAS_NULLBITMAP of the inflated datum stream block */
				atomicOr(anynull, 1);
		}
	}
}

/* ---------------------------------------------------------------------------------------------
 * compresstype=zstd blocks: the same step for Zstandard frames (zstd_dec.cuh; the reference's zstd_decompress,
 * gpcontrib/zstd/zstd_compression.c:142-175).  One warp per storage block = one frame.  Lane 0 parses headers, builds
 * the FSE / Huffman tables in shared memory and decodes sequences 32 at a time; the four Huffman literal streams decode
 * on four lanes at once into the warp's scratch area; the warp then executes a batch of sequences: output and literal
 * positions by two prefix sums, literal runs and matches that reach behind the batch in parallel, the rest in order,
 * warp-wide.  Wrong sizes, malformed sections and (when the frame carries one) a wrong XXH64 checksum raise
 * CBGPU_ERR_CORRUPT, as the ZSTD_isError() / length checks of the reference do.
 * --------------------------------------------------------------------------------------------- */
#define ZSTD_SCRATCH (Z_BLOCK_MAX + 64u)

__device__ __forceinline__ void
warp_copy(uint8_t *dst, const uint8_t *src, uint32_t n, int lane)
{
	for (uint32_t i = lane; i < n; i += 32)
		dst[i] = src[i];
}

__device__ __forceinline__ bool
zstd_exec_warp(uint8_t *out, uint32_t &op, uint32_t cap, const uint8_t *lit, uint32_t &lp, uint32_t regen, const uint32_t *qll,
			   const uint32_t *qml, const uint32_t *qoff, int n, int lane)
{
	const uint32_t ll = lane < n ? qll[lane] : 0u;
	const uint32_t ml = lane < n ? qml[lane] : 0u;
	const uint32_t off = lane < n ? qoff[lane] : 1u;
	uint32_t	io = ll + ml,
				il = ll;

	for (int d = 1; d < 32; d <<= 1)
	{
		const uint32_t vo = __shfl_up_sync(0xffffffffu, io, d);
		const uint32_t vl = __shfl_up_sync(0xffffffffu, il, d);

		if (lane >= d)
		{
			io += vo;
			il += vl;
		}
	}
	const uint32_t total_out = __shfl_sync(0xffffffffu, io, 31);
	const uint32_t total_lit = __shfl_sync(0xffffffffu, il, 31);
	const uint32_t start = op + io - (ll + ml);
	const uint32_t lstart = lp + il - ll;
	const uint32_t mstart = start + ll;

	if (total_lit > regen - lp || total_out > cap - op || __any_sync(0xffffffffu, lane < n && (off == 0 || off > mstart)))
		return false;
	/* literal runs: short ones one per lane, long ones by the whole warp */
	if (ll <= 32)
		for (uint32_t i = 0; i < ll; i++)
			out[start + i] = lit[lstart + i];
	for (unsigned m = __ballot_sync(0xffffffffu, ll > 32); m; m &= m - 1)
	{
		const int	k = __ffs(m) - 1;

		warp_copy(out + __shfl_sync(0xffffffffu, start, k), lit + __shfl_sync(0xffffffffu, lstart, k), __shfl_sync(0xffffffffu, ll, k), lane);
	}
	/* matches whose source ends before the batch */
	bool		dep = false;

	if (lane < n && ml)
	{
		if (mstart - off + ml <= op && ml <= 64)
		{
			const uint8_t *src = out + mstart - off;

			for (uint32_t i = 0; i < ml; i++)
				out[mstart + i] = src[i];
		}
		else
			dep = true;
	}
	__syncwarp();
	for (unsigned m = __ballot_sync(0xffffffffu, dep); m; m &= m - 1)
	{
		const int	k = __ffs(m) - 1;
		const uint32_t s = __shfl_sync(0xffffffffu, mstart, k);
		const uint32_t d = __shfl_sync(0xffffffffu, off, k);
		const uint32_t l = __shfl_sync(0xffffffffu, ml, k);

		for (uint32_t i = lane; i < l; i += 32)
			out[s + i] = out[s - d + (d >= l ? i : i % d)];
		__syncwarp();
	}
	op += total_out;
	lp += total_lit;
	return true;
}

__global__ void __launch_bounds__(AOCS_WARPS * 32)
k_aocs_unzstd(uint8_t *raw, const AocsDir *dir, int nblocks, int *status, int *anynull, uint8_t *scratch)
{
	__shared__ ZTab s_tab[AOCS_WARPS];
	__shared__ uint32_t s_q[AOCS_WARPS][3][Z_SEQ_QN];
	__shared__ ZLitStreams s_st[AOCS_WARPS];
	const int	lane = threadIdx.x & 31;
	const int	w = threadIdx.x >> 5;
	const int	nwarps = gridDim.x * AOCS_WARPS;
	uint8_t    *litbuf = scratch + (size_t) (blockIdx.x * AOCS_WARPS + w) * ZSTD_SCRATCH;
	ZTab	   &T = s_tab[w];

	if (*status == CBGPU_ERR_CORRUPT)
		return;
	for (int b = blockIdx.x * AOCS_WARPS + w; b < nblocks; b += nwarps)
	{
		const AocsDir D = dir[b];

		if (D.clen == 0)
			continue;
		const uint8_t *z = raw + D.zoff;
		uint8_t    *out = raw + D.off;
		const uint32_t zl = (uint32_t) D.clen;
		const uint32_t cap = (uint32_t) D.dlen;
		uint32_t	op = 0,
					pos = 0;
		int			last = 0;
		bool		ok = true;
		ZFrame		F;
		ZSeqState	S;

		F.hdr = 0;
		F.content_size = 0;
		F.checksum = 0;
		S.rep[0] = 1;
		S.rep[1] = 4;
		S.rep[2] = 8;
		S.nseq = S.done = 0;
		if (lane == 0)
		{
			T.have_ll = T.have_of = T.have_ml = T.have_huf = 0;
			ok = z_frame_header(z, zl, F);
		}
		ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
		pos = __shfl_sync(0xffffffffu, F.hdr, 0);
		while (ok && !last)
		{
			int			type = 0;
			uint32_t	size = 0;

			if (lane == 0)
				ok = z_block_header(z, zl, pos, &last, &type, &size) && pos + 3 + (type == 1 ? 1u : size) <= zl;
			ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
			last = __shfl_sync(0xffffffffu, last, 0);
			type = __shfl_sync(0xffffffffu, type, 0);
			size = __shfl_sync(0xffffffffu, size, 0);
			if (!ok)
				break;
			pos += 3;
			if (type == 0 || type == 1)
			{
				if (size > cap - op)
				{
					ok = false;
					break;
				}
				if (type == 0)
					warp_copy(out + op, z + pos, size, lane);
				else
				{
					const uint8_t v = z[pos];

					for (uint32_t i = lane; i < size; i += 32)
						out[op + i] = v;
				}
				op += size;
				pos += type == 0 ? size : 1u;
				__syncwarp();
				continue;
			}
			/* compressed block */
			const uint8_t *blk = z + pos;
			const uint8_t *lit = litbuf;
			ZLit		L;
			uint32_t	after = 0,
						lp = 0;

			L.type = 0;
			L.regen = L.csize = L.hdr = 0;
			L.streams = 1;
			if (lane == 0)
				ok = z_lit_header(blk, size, L) && L.regen <= Z_BLOCK_MAX && L.hdr + (L.type == 0 ? L.regen : L.type == 1 ? 1u : L.csize) <= size;
			ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
			if (!ok)
				break;
			L.type = __shfl_sync(0xffffffffu, L.type, 0);
			L.regen = __shfl_sync(0xffffffffu, L.regen, 0);
			L.csize = __shfl_sync(0xffffffffu, L.csize, 0);
			L.hdr = __shfl_sync(0xffffffffu, L.hdr, 0);
			L.streams = __shfl_sync(0xffffffffu, L.streams, 0);
			if (L.type == 0)
			{
				lit = blk + L.hdr;
				after = L.hdr + L.regen;
			}
			else if (L.type == 1)
			{
				const uint8_t v = blk[L.hdr];

				for (uint32_t i = lane; i < L.regen; i += 32)
					litbuf[i] = v;
				after = L.hdr + 1;
			}
			else
			{
				uint32_t	tree = 0;

				if (lane == 0)
				{
					if (L.type == 2)
					{
						const int	used = z_huf_read_tree(blk + L.hdr, L.csize, T);

						ok = used >= 0;
						tree = ok ? (uint32_t) used : 0u;
					}
					else
						ok = T.have_huf != 0;
					ok = ok && z_lit_streams(L, blk + L.hdr + tree, L.csize - tree, s_st[w]);
				}
				__syncwarp();
				ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
				tree = __shfl_sync(0xffffffffu, tree, 0);
				if (!ok)
					break;
				/* the Huffman streams: one lane each */
				bool		sok = true;

				if (lane < L.streams)
					sok = z_huf_stream(T, blk + L.hdr + tree + s_st[w].off[lane], s_st[w].len[lane], litbuf + s_st[w].outoff[lane],
									   s_st[w].count[lane]);
				ok = !__any_sync(0xffffffffu, !sok);
				if (!ok)
					break;
				after = L.hdr + L.csize;
			}
			__syncwarp();
			if (lane == 0)
				ok = z_seq_begin(blk + after, size - after, T, S);
			ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
			if (!ok)
				break;
			const uint32_t nseq = __shfl_sync(0xffffffffu, S.nseq, 0);

			for (uint32_t done = 0; done < nseq && ok; done += Z_SEQ_QN)
			{
				const int	n = (int) (nseq - done < Z_SEQ_QN ? nseq - done : Z_SEQ_QN);

				if (lane == 0)
					for (int k = 0; k < n && ok; k++)
						ok = z_seq_next(T, S, &s_q[w][0][k], &s_q[w][1][k], &s_q[w][2][k]);
				__syncwarp();
				ok = __shfl_sync(0xffffffffu, ok ? 1 : 0, 0) != 0;
				if (ok)
					ok = zstd_exec_warp(out, op, cap, lit, lp, L.regen, s_q[w][0], s_q[w][1], s_q[w][2], n, lane);
				__syncwarp();
			}
			if (ok && nseq)
				ok = __shfl_sync(0xffffffffu, S.bs.pos == 0 ? 1 : 0, 0) != 0;
			if (ok && L.regen - lp > cap - op)
				ok = false;
			if (!ok)
				break;
			warp_copy(out + op, lit + lp, L.regen - lp, lane);
			op += L.regen - lp;
			pos += size;
			__syncwarp();
		}
		if (ok && lane == 0)
		{
			if (op != cap || (F.content_size != ~0ull && F.content_size != op))
				ok = false;
			else if (F.checksum)
				ok = pos + 4 <= zl &&
					(uint32_t) z_xxh64(out, op) == ((uint32_t) z[pos] | ((uint32_t) z[pos + 1] << 8) | ((uint32_t) z[pos + 2] << 16) | ((uint32_t) z[pos + 3] << 24));
		}
		if (lane == 0)
		{
			if (!ok)
				atomicExch(status, CBGPU_ERR_CORRUPT);
			else if (cap > 2 && (out[2] & 1u))
				atomicOr(anynull, 1);
		}
		__syncwarp();
	}
}

/* value of the datum at d (fixed width: the value; numeric: scaled integer; char(1): the byte) */
/* ---------------------------------------------------------------------------------------------
 * Dictionary columns: bpchar(n) / varchar / text values become codes into a per-column dictionary (DESIGN.md, data
 * layout: CB_DICT8 / CB_DICT32 with a per-code hashbpchar).  Two passes over the column's files, both through the same
 * block decode: COLLECT inserts every physical datum's bytes into an open-addressing set keyed by a 64-bit hash (claim
 * by compare-and-swap on the tag; the winner copies the bytes into the arena; nobody waits on anybody, so lanes of one
 * warp hitting the same string cannot stall each other); cbgpu_dict_finalize orders the distinct strings on the host and
 * assigns codes; LOOKUP finds the tag again and now also compares the bytes, so two different strings with one 64-bit
 * hash are reported (CBGPU_ERR_UNSUPPORTED) instead of sharing a code.
 * --------------------------------------------------------------------------------------------- */
__host__ __device__ __forceinline__ unsigned long long
dict_hash64(const uint8_t *p, int n)
{
	unsigned long long h = 0xcbf29ce484222325ull;	/* FNV-1a, then a finaliser */

	for (int i = 0; i < n; i++)
		h = (h ^ p[i]) * 0x100000001b3ull;
	h ^= h >> 32;
	h *= 0xd6e8feb86659fd93ull;
	h ^= h >> 32;
	return h ? h : 1ull;
}

__device__ __forceinline__ int64_t
aocs_dict_value(const AocsParams &P, const uint8_t *body, int len)
{
	if (P.dtrim)
		while (len > 0 && body[len - 1] == ' ')
			len--;
	const unsigned long long tag = dict_hash64(body, len);
	uint32_t	i = (uint32_t) tag & P.dmask;

	for (uint32_t probes = 0; probes <= P.dmask; probes++, i = (i + 1) & P.dmask)
	{
		DictSlot   *sl = P.dslots + i;
		unsigned long long t = sl->tag;

		if (t == 0 && P.dmode == 1)
		{
			t = atomicCAS(&sl->tag, 0ull, tag);
			if (t == 0)
			{
				/* ours: room in the arena, then the bytes */
				const unsigned long long off = atomicAdd(P.dcursor, (unsigned long long) ((len + 3) & ~3));

				if (atomicAdd(P.dcursor + 1, 1ull) >= (unsigned long long) P.dmax || off + (unsigned long long) len > P.darena_cap)
				{
					atomicExch(P.status, CBGPU_ERR_NOMEM);
					sl->len = 0;
					sl->off = 0;
					return 0;
				}
				for (int k = 0; k < len; k++)
					P.darena[off + k] = body[k];
				sl->off = (uint32_t) off;
				sl->len = (uint32_t) len;
				return 0;
			}
		}
		if (t == tag)
		{
			if (P.dmode == 1)
				return 0;
			/* lookup: the dictionary is final, compare the bytes */
			bool		same = sl->len == (uint32_t) len;

			for (int k = 0; same && k < len; k++)
				same = P.darena[sl->off + k] == body[k];
			if (!same)
			{
				atomicExch(P.status, CBGPU_ERR_UNSUPPORTED);	/* two strings, one 64-bit hash */
				return 0;
			}
			return sl->code;
		}
		if (t == 0)
			break;
	}
	/* lookup of a string the collect pass never saw, or a full table */
	atomicExch(P.status, P.dmode == 1 ? CBGPU_ERR_NOMEM : CBGPU_ERR_INVALID);
	return 0;
}

__device__ __forceinline__ int64_t
aocs_value(const AocsParams &P, const uint8_t *d)
{
	int64_t		v = 0;

	if (P.attlen > 0)
	{
		switch (P.attlen)
		{
			case 1: v = (int64_t) *d; break;
			case 2: v = (int64_t) *(const int16_t *) d; break;
			case 4: v = (int64_t) *(const int32_t *) d; break;
			default: v = *(const long long *) d; break;
		}
		return v;
	}
	const uint32_t b0 = d[0];
	const int	hdr = (b0 & 1u) ? 1 : 4;
	const int	size = (b0 & 1u) ? (int) (b0 >> 1) : (int) ((aocs_le32(d) >> 2) & 0x3FFFFFFFu);

	if (P.varkind == CBGPU_AOCS_VAR_NUMERIC)
	{
		if (size - hdr < 2 || !aocs_numeric(d + hdr, size - hdr, P.dscale, &v))
			atomicExch(P.status, CBGPU_ERR_OVERFLOW);
	}
	else if (P.varkind == CBGPU_AOCS_VAR_DICT)
	{
		if (hdr == 4 && (b0 & 3u) != 0)
			atomicExch(P.status, CBGPU_ERR_UNSUPPORTED);	/* compressed or external varlena: not stored in AOCS blocks */
		else
			v = aocs_dict_value(P, d + hdr, size - hdr);
	}
	else
		v = size - hdr > 0 ? (int64_t) d[hdr] : (int64_t) ' ';
	return v;
}

__device__ __forceinline__ void
aocs_store(const AocsParams &P, int64_t orow, int64_t v, bool isnull)
{
	if (!P.out)
		return;					/* collecting a dictionary: nothing is stored */
	switch (P.attlen > 0 ? P.attlen : (P.varkind == CBGPU_AOCS_VAR_NUMERIC ? 8 : P.varkind == CBGPU_AOCS_VAR_DICT ? P.doutw : 1))
	{
		case 1: ((uint8_t *) P.out)[orow] = (uint8_t) v; break;
		case 2: ((int16_t *) P.out)[orow] = (int16_t) v; break;
		case 4: ((int32_t *) P.out)[orow] = (int32_t) v; break;
		default: ((int64_t *) P.out)[orow] = v; break;
	}
	if (P.outnull)
		P.outnull[orow] = isnull ? 1 : 0;
}

/* one Dense (optionally RLE) datum stream block, by one warp */
__device__ __forceinline__ void
aocs_decode_dense(const AocsParams &P, const AocsDir &D, const uint8_t *blk, uint32_t *s_off, uint32_t *s_rep, int32_t *s_del)
{
	const int	lane = threadIdx.x & 31;
	const uint32_t flags = (uint32_t) blk[2] | ((uint32_t) blk[3] << 8);
	const int32_t logical = (int32_t) aocs_le32(blk + 4);
	const int32_t physical = (int32_t) aocs_le32(blk + 8);
	const uint32_t psize = aocs_le32(blk + 12);
	const bool	rle = (flags & 2u) != 0;
	const bool	delta = (flags & 4u) != 0;
	uint32_t	p = 16;
	uint32_t	nn_count = 0,
				c_count = 0,
				rc_size = 0,
				d_count = 0,
				d_size = 0;
	const uint8_t *bitmap = NULL,
			   *cbitmap = NULL,
			   *rc = NULL,
			   *dbitmap = NULL,
			   *dl = NULL;

	if (logical != D.rows || (flags & ~7u) || (delta && P.attlen != 4 && P.attlen != 8))
	{
		if (lane == 0)
			atomicExch(P.status, CBGPU_ERR_INVALID);
		return;
	}
	if (rle)
	{
		nn_count = aocs_le32(blk + p);
		c_count = aocs_le32(blk + p + 4);
		rc_size = aocs_le32(blk + p + 12);
		p += 16;
	}
	if (delta)
	{
		/* DatumStreamBlock_Delta_Extension (datumstreamblock.h:172-195) */
		d_count = aocs_le32(blk + p);
		d_size = aocs_le32(blk + p + 8);
		p += 12;
	}
	if (flags & 1u)
	{
		const uint32_t nb = rle ? nn_count : (uint32_t) logical;

		bitmap = blk + p;
		p += (nb + 7u) >> 3;
	}
	if (rle)
	{
		cbitmap = blk + p;
		p += (c_count + 7u) >> 3;
		rc = blk + p;
		p += rc_size;
	}
	if (delta)
	{
		dbitmap = blk + p;
		p += (d_count + 7u) >> 3;
		dl = blk + p;
		p += d_size;
	}
	p = (p + 7u) & ~7u;
	if ((int64_t) p + psize > D.dlen + 8)
	{
		if (lane == 0)
			atomicExch(P.status, CBGPU_ERR_INVALID);
		return;
	}
	const uint8_t *data = blk + p;
	/* positions = the items the NULL bitmap counts: NULLs and non-repeated datums */
	/* without a NULL bitmap every position is a value: compress / delta bitmaps count them when present */
	const uint32_t npos = bitmap ? (rle ? nn_count : (uint32_t) logical) : (rle ? c_count : (delta ? d_count : (uint32_t) physical));
	uint32_t	dbase = 0,		/* non-NULL positions before this trip */
				pbase = 0,		/* physical datums before this trip */
				cur = 0,		/* byte offset of the next varlena datum */
				rcp = 0,		/* byte offset of the next repeat count */
				dlp = 0;		/* byte offset of the next delta */
	int64_t		rowbase = 0;	/* logical rows before this trip */
	unsigned long long running = 0;	/* the value deltas apply to (AdvanceDenseDelta's delta_datum_p) */

	for (uint32_t p0 = 0; p0 < npos; p0 += 32)
	{
		const uint32_t pos = p0 + lane;
		const bool	inr = pos < npos;
		const bool	isnull = inr && bitmap && ((bitmap[pos >> 3] >> (pos & 7)) & 1);
		const unsigned nn = __ballot_sync(0xffffffffu, inr && !isnull);
		const int	k = __popc(nn & ((1u << lane) - 1));
		const int	cnt = __popc(nn);
		const uint32_t di = dbase + (uint32_t) k;
		const bool	cb = inr && !isnull && rle && ((cbitmap[di >> 3] >> (di & 7)) & 1);
		const unsigned cm = __ballot_sync(0xffffffffu, cb);
		const bool	isdelta = inr && !isnull && delta && ((dbitmap[di >> 3] >> (di & 7)) & 1);
		const unsigned dm = __ballot_sync(0xffffffffu, isdelta);
		const unsigned pm = nn & ~dm;		/* positions holding a physical datum */

		if (lane == 0)
		{
			/* repeat counts of this trip's compressed datums (DatumStreamInt32Compress_Decode) ... */
			uint32_t	r = rcp;
			const int	nc = __popc(cm);

			for (int i = 0; i < nc; i++)
			{
				const uint32_t b0 = rc[r];
				const int	len = (int) (b0 >> 6) + 1;
				uint32_t	v = b0 & 0x3Fu;

				for (int j = 1; j < len; j++)
					v = (v << 8) | rc[r + j];
				s_rep[i] = v;
				r += (uint32_t) len;
			}
			rcp = r;
			/* ... its deltas (DatumStreamInt32CompressReserved3_Decode: 2 length bits, "positive" bit, 29 bits) ... */
			{
				uint32_t	q = dlp;
				const int	nd = __popc(dm);

				for (int i = 0; i < nd; i++)
				{
					const uint32_t b0 = dl[q];
					const int	len = (int) (b0 >> 6) + 1;
					uint32_t	v = b0 & 0x1Fu;

					for (int j = 1; j < len; j++)
						v = (v << 8) | dl[q + j];
					s_del[i] = (b0 & 0x20u) ? (int32_t) v : -(int32_t) v;
					q += (uint32_t) len;
				}
				dlp = q;
			}
			/* ... and, for varlena columns, where its datums start */
			if (P.attlen < 0)
			{
				uint32_t	c = cur;

				for (int i = 0; i < cnt; i++)
				{
					s_off[i] = c;
					const uint32_t b0 = data[c];
					const uint32_t size = (b0 & 1u) ? (b0 >> 1) : ((aocs_le32(data + c) >> 2) & 0x3FFFFFFFu);

					if (size == 0 || c + size > psize)
					{
						atomicExch(P.status, CBGPU_ERR_INVALID);
						c = psize;
						break;
					}
					c += size;
					if (c < psize && data[c] == 0)
						c = (c + (uint32_t) P.typalign - 1u) & ~((uint32_t) P.typalign - 1u);
				}
				cur = c;
			}
		}
		rcp = __shfl_sync(0xffffffffu, rcp, 0);
		dlp = __shfl_sync(0xffffffffu, dlp, 0);
		cur = __shfl_sync(0xffffffffu, cur, 0);
		__syncwarp();
		/* run length of every position, its first output row by a warp scan */
		const uint32_t len = !inr ? 0u : (isnull ? 1u : 1u + (cb ? s_rep[__popc(cm & ((1u << lane) - 1))] : 0u));
		uint32_t	x = len;

#pragma unroll
		for (int d = 1; d < 32; d <<= 1)
		{
			const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);

			if (lane >= d)
				x += y;
		}
		const uint32_t total = __shfl_sync(0xffffffffu, x, 31);
		const int64_t first = rowbase + (int64_t) (x - len);
		int64_t		v = 0;

		if (inr && !isnull && !isdelta)
		{
			const uint32_t ph = pbase + (uint32_t) __popc(pm & ((1u << lane) - 1));

			v = aocs_value(P, P.attlen > 0 ? data + (size_t) ph * P.attlen : data + s_off[k]);
		}
		if (delta)
		{
			/* value = previous value + delta: an affine map per position (physical datum: x -> v; delta:
			 * x -> x + d; NULL / idle lane: x -> x), composed across the warp by a scan, applied to the
			 * value the previous trip ended on.  4-byte types wrap like the reference's uint32 arithmetic. */
			unsigned long long a = (inr && !isnull && !isdelta) ? 0ull : 1ull;
			unsigned long long b = (inr && !isnull) ? (isdelta ? (unsigned long long) (long long) s_del[__popc(dm & ((1u << lane) - 1))]
													   : (unsigned long long) v) : 0ull;

#pragma unroll
			for (int d = 1; d < 32; d <<= 1)
			{
				const unsigned long long a1 = __shfl_up_sync(0xffffffffu, a, d);
				const unsigned long long b1 = __shfl_up_sync(0xffffffffu, b, d);

				if (lane >= d)
				{
					b = a * b1 + b;
					a = a * a1;
				}
			}
			const unsigned long long val = a * running + b;

			running = __shfl_sync(0xffffffffu, val, 31);
			if (inr && !isnull)
				v = P.attlen == 4 ? (int64_t) (int32_t) (uint32_t) val : (int64_t) val;
		}
		if (__any_sync(0xffffffffu, first + (int64_t) len > D.rows))
		{
			if (lane == 0)
				atomicExch(P.status, CBGPU_ERR_INVALID);	/* repeat counts run past the block's row count */
			return;
		}
		/* short runs by their own lane, long runs by the whole warp */
		if (len > 0 && len <= 8)
			for (uint32_t i = 0; i < len; i++)
				aocs_store(P, D.rowbase + first + i, v, isnull);
		unsigned	longm = __ballot_sync(0xffffffffu, len > 8);

		while (longm)
		{
			const int	src = __ffs(longm) - 1;
			const int64_t f = __shfl_sync(0xffffffffu, first, src);
			const uint32_t l = __shfl_sync(0xffffffffu, len, src);
			const int64_t vv = __shfl_sync(0xffffffffu, v, src);

			longm &= longm - 1;
			for (uint32_t i = lane; i < l; i += 32)
				aocs_store(P, D.rowbase + f + i, vv, false);
		}
		dbase += (uint32_t) cnt;
		pbase += (uint32_t) __popc(pm);
		rowbase += total;
		__syncwarp();
	}
	if (rowbase != D.rows && lane == 0)
		atomicExch(P.status, CBGPU_ERR_INVALID);
}

__global__ void __launch_bounds__(AOCS_WARPS * 32)
k_aocs_decode(AocsParams P)
{
	__shared__ uint32_t s_off[AOCS_WARPS][32];
	__shared__ uint32_t s_rep[AOCS_WARPS][32];
	__shared__ int32_t s_del[AOCS_WARPS][32];
	const int	lane = threadIdx.x & 31;
	const int	w = threadIdx.x >> 5;
	const int	nwarps = gridDim.x * AOCS_WARPS;

	if (*P.status == CBGPU_ERR_CORRUPT)
		return;					/* k_aocs_verify (same stream, just before) rejected a block: decode nothing */
	for (int b = blockIdx.x * AOCS_WARPS + w; b < P.nblocks; b += nwarps)
	{
		const AocsDir D = P.dir[b];
		const uint8_t *blk = P.raw + D.off;
		/* DatumStreamBlock_Orig */
		const int	version = (int) (int16_t) ((uint32_t) blk[0] | ((uint32_t) blk[1] << 8));
		const uint32_t flags = (uint32_t) blk[2] | ((uint32_t) blk[3] << 8);
		const int	ndatum = (int) (int16_t) ((uint32_t) blk[4] | ((uint32_t) blk[5] << 8));
		const uint32_t nullsz = aocs_le32(blk + 8);
		const uint32_t sz = aocs_le32(blk + 12);
		const uint8_t *bitmap = (flags & 1u) ? blk + 16 : NULL;
		uint32_t	p0 = 16 + ((flags & 1u) ? nullsz : 0u);

		p0 = (p0 + 7u) & ~7u;
		if (version == 1 || version == 2)
		{
			aocs_decode_dense(P, D, blk, s_off[w], s_rep[w], s_del[w]);
			continue;
		}
		if (version != 0 || ndatum != D.rows || (flags & ~1u) != 0 || (int64_t) p0 + sz > D.dlen + 8)
		{
			if (lane == 0)
				atomicExch(P.status, CBGPU_ERR_INVALID);
			continue;
		}
		const uint8_t *data = blk + p0;
		uint32_t	phys = 0,		/* physical datums before this trip (fixed width) */
					cur = 0;		/* byte offset of the next datum (varlena) */

		for (int r0 = 0; r0 < D.rows; r0 += 32)
		{
			const int	r = r0 + lane;
			const bool	inr = r < D.rows;
			const bool	isnull = inr && bitmap && ((bitmap[r >> 3] >> (r & 7)) & 1);
			const unsigned nn = __ballot_sync(0xffffffffu, inr && !isnull);
			const int	k = __popc(nn & ((1u << lane) - 1));
			const int	cnt = __popc(nn);
			const int64_t orow = D.rowbase + r;

			if (P.attlen < 0)
			{
				/* lane 0 finds where this trip's datums start: VARSIZE_ANY + zero-pad skipping */
				if (lane == 0)
				{
					uint32_t	c = cur;

					for (int i = 0; i < cnt; i++)
					{
						s_off[w][i] = c;
						const uint32_t b0 = data[c];
						const uint32_t size = (b0 & 1u) ? (b0 >> 1) : ((aocs_le32(data + c) >> 2) & 0x3FFFFFFFu);

						if (size == 0 || c + size > sz)
						{
							atomicExch(P.status, CBGPU_ERR_INVALID);
							c = sz;
							break;
						}
						c += size;
						if (c < sz && data[c] == 0)
							c = (c + (uint32_t) P.typalign - 1u) & ~((uint32_t) P.typalign - 1u);
					}
					cur = c;
				}
				cur = __shfl_sync(0xffffffffu, cur, 0);
				__syncwarp();
			}
			if (inr)
			{
				int64_t		v = 0;

				if (!isnull)
				{
					if (P.attlen > 0)
					{
						const uint8_t *d = data + (size_t) (phys + k) * P.attlen;

						switch (P.attlen)
						{
							case 1: v = (int64_t) *d; break;
							case 2: v = (int64_t) *(const int16_t *) d; break;
							case 4: v = (int64_t) *(const int32_t *) d; break;
							default: v = *(const long long *) d; break;
						}
					}
					else
						v = aocs_value(P, data + s_off[w][k]);
				}
				aocs_store(P, orow, v, isnull);
			}
			phys += (uint32_t) cnt;
			__syncwarp();
		}
	}
}

/* what the header walk over a column file found */
struct AocsWalk
{
	AocsDir    *dir;
	int64_t		ndir;
	int64_t		rows;
	int64_t		ztotal;			/* bytes of the inflate area behind the file image                    */
	int64_t		ncompressed;
	bool		anynull;		/* some uncompressed block has a NULL bitmap                          */
};

/* AppendOnlyStorageRead_GetBlockInfo for every block of the file.  compress_kind < 0: contents are not looked at
 * (visibility map application needs the row numbers only). */
static int
aocs_walk(cbgpu_ctx *ctx, const uint8_t *raw, int64_t nbytes, int32_t checksum, int32_t compress_kind, int64_t row_offset, AocsWalk *W)
{
	AocsDir    *dir = NULL;
	int64_t		ndir = 0,
				capdir = 0,
				pos = 0,
				rows = 0,
				ztotal = 0,
				ncompressed = 0;
	bool		anynull = false;

	memset(W, 0, sizeof(*W));
	while (pos < nbytes)
	{
		uint32_t	w0, w1;
		int			kind, has_first, nrow, dlen, clen, hlen;

		if (pos + 8 > nbytes)
		{
			free(dir);
			return cb_fail(ctx, CBGPU_ERR_INVALID, "AOCS column file ends inside a block header%s (offset %lld)", "", pos);
		}
		memcpy(&w0, raw + pos, 4);
		memcpy(&w1, raw + pos + 4, 4);
		kind = (int) ((w0 & 0x70000000u) >> 28);
		has_first = (int) ((w0 & 0x08000000u) >> 27);
		int			ext = 0;
		int64_t		stored;

		if (kind == 3)
		{
			/* AoHeaderKind_NonBulkDenseContent (cdbappendonlystorage_int.h:259-325): 30-bit row count */
			nrow = (int) (w1 & 0x3FFFFFFFu);
			dlen = (int) (w0 & 0x001FFFFFu);
			clen = 0;
		}
		else
		{
			/* SmallContent (:64-147) and BulkDenseContent (:350-466) share the length fields */
			nrow = (int) ((w0 & 0x00FFFC00u) >> 10);
			dlen = (int) (((w0 & 0x000003FFu) << 11) | ((w1 & 0xFFE00000u) >> 21));
			clen = (int) (w1 & 0x001FFFFFu);
		}
		if ((w0 >> 31) != 0 || (kind != 1 /* AoHeaderKind_SmallContent */ && kind != 3 && kind != 4 /* BulkDenseContent */))
		{
			free(dir);
			return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED,
						   "AOCS block at offset %s%lld is not a SmallContent / NonBulkDenseContent / BulkDenseContent block (large-content blocks are not decoded on the device)",
						   "", pos);
		}
		if (kind == 4)
		{
			/* the extension header with the 30-bit row count follows the checksums (cdbappendonlystorageformat.c:1547-1640) */
			ext = 8;
			if (pos + 8 + (checksum ? 8 : 0) + 8 > nbytes)
			{
				free(dir);
				return cb_fail(ctx, CBGPU_ERR_INVALID, "AOCS column file ends inside a block header%s (offset %lld)", "", pos);
			}
			memcpy(&w1, raw + pos + 8 + (checksum ? 8 : 0) + 4, 4);
			nrow = (int) (w1 & 0x3FFFFFFFu);
		}
		hlen = 8 + (checksum ? 8 : 0) + ext + (has_first ? 8 : 0);
		stored = clen ? clen : dlen;
		if (pos + hlen + stored > nbytes || dlen < 16 || (clen && compress_kind >= 0 && compress_kind != CBGPU_AOCS_COMPRESS_ZLIB && compress_kind != CBGPU_AOCS_COMPRESS_ZSTD))
		{
			free(dir);
			if (clen && pos + hlen + stored <= nbytes && dlen >= 16)
				return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED,
							   "AOCS block at offset %s%lld is bulk-compressed: pass the column's compresstype (zlib or zstd; quicklz is not decoded on the device)", "", pos);
			return cb_fail(ctx, CBGPU_ERR_INVALID, "AOCS block at offset %s%lld runs past the end of the file", "", pos);
		}
		if (ndir == capdir)
		{
			capdir = capdir ? capdir * 2 : 1024;
			dir = (AocsDir *) realloc(dir, sizeof(AocsDir) * (size_t) capdir);
			if (!dir)
				return CBGPU_ERR_NOMEM;
		}
		dir[ndir].hoff = pos;
		dir[ndir].overall = (int32_t) (hlen + (stored + 7) / 8 * 8);
		dir[ndir].clen = clen;
		dir[ndir].zoff = pos + hlen;
		if (clen)
		{
			/* inflated behind the file image */
			dir[ndir].off = (nbytes + 15) / 16 * 16 + ztotal;
			ztotal += ((int64_t) dlen + 15) / 16 * 16;
			ncompressed++;
		}
		else
		{
			dir[ndir].off = pos + hlen;
			if (compress_kind >= 0 && (raw[pos + hlen + 2] & 1))	/* DSB_HAS_NULLBITMAP */
				anynull = true;
		}
		dir[ndir].first = -1;
		if (has_first)
			memcpy(&dir[ndir].first, raw + pos + hlen - 8, 8);
		dir[ndir].rowbase = row_offset + rows;
		dir[ndir].rows = nrow;
		dir[ndir].dlen = dlen;
		ndir++;
		rows += nrow;
		pos += hlen + (stored + 7) / 8 * 8;
	}
	W->dir = dir;
	W->ndir = ndir;
	W->rows = rows;
	W->ztotal = ztotal;
	W->ncompressed = ncompressed;
	W->anynull = anynull;
	return CBGPU_OK;
}

extern "C" int
cbgpu_aocs_decode_column(cbgpu_ctx *ctx, const void *file_bytes, int64_t nbytes, int32_t checksum, int32_t attlen, int32_t varkind,
						 int32_t typalign, cbgpu_rel *rel, int32_t col, int64_t row_offset, int64_t *nrows_out)
{
	return cbgpu_aocs_decode_column_ex(ctx, file_bytes, nbytes, checksum, CBGPU_AOCS_COMPRESS_NONE, attlen, varkind, typalign, rel, col,
									   row_offset, nrows_out);
}

/* a dictionary: the device string set, and after finalize its entries on the host in code order */
struct cbgpu_dict
{
	cbgpu_ctx  *ctx;
	DictSlot   *d_slots;
	uint8_t    *d_arena;
	unsigned long long *d_cursor;
	uint32_t   *d_hashes;		/* per code, after finalize                                           */
	uint2	   *d_offlen;		/* per code, after finalize: (offset, length) of its bytes in d_arena */
	uint32_t	nslots;
	uint32_t	arena_cap;
	int32_t		max_entries;
	int32_t		bpchar;
	int32_t		finalized;
	int32_t		n;
	char	   *texts;			/* host copy of the arena                                             */
	uint32_t   *off, *len;		/* per code                                                           */
	int32_t    *sorted;			/* codes in memcmp order == identity; kept for lookups: slot index per code */
};

static int	aocs_decode_impl(cbgpu_ctx *ctx, const void *file_bytes, int64_t nbytes, int32_t checksum, int32_t compress_kind, int32_t attlen,
							 int32_t varkind, int32_t typalign, cbgpu_rel *rel, int32_t col, int64_t row_offset, int64_t *nrows_out,
							 const cbgpu_dict *dict, int dmode);

extern "C" int
cbgpu_aocs_decode_column_ex(cbgpu_ctx *ctx, const void *file_bytes, int64_t nbytes, int32_t checksum, int32_t compress_kind,
							int32_t attlen, int32_t varkind, int32_t typalign, cbgpu_rel *rel, int32_t col, int64_t row_offset,
							int64_t *nrows_out)
{
	if (varkind == CBGPU_AOCS_VAR_DICT)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "dictionary columns are decoded by cbgpu_aocs_decode_dict_column%s (%lld)", "", varkind);
	return aocs_decode_impl(ctx, file_bytes, nbytes, checksum, compress_kind, attlen, varkind, typalign, rel, col, row_offset, nrows_out,
							NULL, 0);
}

static int
aocs_decode_impl(cbgpu_ctx *ctx, const void *file_bytes, int64_t nbytes, int32_t checksum, int32_t compress_kind, int32_t attlen,
				 int32_t varkind, int32_t typalign, cbgpu_rel *rel, int32_t col, int64_t row_offset, int64_t *nrows_out,
				 const cbgpu_dict *dict, int dmode)
{
	const uint8_t *raw = (const uint8_t *) file_bytes;
	CbCallMem	mem(ctx);
	AocsDir    *dir = NULL;
	AocsWalk	W;
	int64_t		ndir = 0,
				rows = 0,
				ztotal = 0,
				ncompressed = 0;
	bool		anynull = false;
	int		   *d_flag = NULL;
	uint8_t    *d_scratch = NULL;
	AocsParams	P;
	uint8_t    *d_raw = NULL;
	AocsDir    *d_dir = NULL;
	int			outw;
	int			nblk;

	*nrows_out = 0;
	if (dmode != 1)
	{
		if (col < 0 || col >= rel->ncols)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_aocs_decode_column: bad column%s %lld", "", col);
		outw = cb_type_w(rel->types[col]);
		if (attlen > 0 ? (attlen != outw || (attlen != 1 && attlen != 2 && attlen != 4 && attlen != 8))
			: !((varkind == CBGPU_AOCS_VAR_NUMERIC && rel->types[col] == CB_NUMERIC) || (varkind == CBGPU_AOCS_VAR_BPCHAR1 && outw == 1) ||
				(varkind == CBGPU_AOCS_VAR_DICT && (rel->types[col] == CB_DICT8 || rel->types[col] == CB_DICT32))))
			return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "AOCS column of length %s%lld does not decode into this relation column", "", attlen);
	}
	else
		outw = 0;
	if (typalign != 1 && typalign != 2 && typalign != 4 && typalign != 8)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "type alignment %s%lld", "", typalign);
	{
		const int	rc = aocs_walk(ctx, raw, nbytes, checksum, compress_kind < 0 ? 0 : compress_kind, row_offset, &W);

		if (rc)
			return rc;
		dir = mem.keep(W.dir);
		ndir = W.ndir;
		rows = W.rows;
		ztotal = W.ztotal;
		ncompressed = W.ncompressed;
		anynull = W.anynull;
	}
	if (dmode != 1 && (row_offset < 0 || row_offset + rows > rel->capacity))
		return cb_fail(ctx, CBGPU_ERR_INVALID, "AOCS column file holds %s%lld rows: more than the relation has room for", "", rows);
	if (ndir == 0)
		return CBGPU_OK;
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	CB_CUDA(ctx, mem.alloc(&d_raw, (size_t) ((nbytes + 15) / 16 * 16 + ztotal + 16)));
	CB_CUDA(ctx, mem.alloc(&d_dir, sizeof(AocsDir) * (size_t) ndir));
	CB_CUDA(ctx, mem.copy_in(d_raw, raw, (size_t) nbytes));
	CB_CUDA(ctx, mem.copy_in(d_dir, dir, sizeof(AocsDir) * (size_t) ndir));
	if (ctx->trace_on)
		cb_trace_mark(ctx, "aocs:h2d");
	nblk = (int) ((ndir + AOCS_WARPS - 1) / AOCS_WARPS);
	if (nblk > ctx->sm_count * 16)
		nblk = ctx->sm_count * 16;
	if (checksum)
	{
		/* AppendOnlyStorageRead verifies header and block checksums before handing a block on */
		k_aocs_verify<<<nblk, AOCS_WARPS * 32, 0, ctx->stream>>>(d_raw, d_dir, (int) ndir, ctx->d_status);
		CB_LAUNCHED(ctx, "k_aocs_verify");
	}
	if (ncompressed)
	{
		int			flag = 0;

		CB_CUDA(ctx, mem.alloc(&d_flag, sizeof(int)));
		CB_CUDA(ctx, cudaMemsetAsync(d_flag, 0, sizeof(int), ctx->stream));
		if (compress_kind == CBGPU_AOCS_COMPRESS_ZSTD)
		{
			/* a literal scratch area per warp bounds the grid */
			const int	zblk = nblk < ctx->sm_count * 4 ? nblk : ctx->sm_count * 4;

			CB_CUDA(ctx, mem.alloc(&d_scratch, (size_t) zblk * AOCS_WARPS * ZSTD_SCRATCH));
			k_aocs_unzstd<<<zblk, AOCS_WARPS * 32, 0, ctx->stream>>>(d_raw, d_dir, (int) ndir, ctx->d_status, d_flag, d_scratch);
			CB_LAUNCHED(ctx, "k_aocs_unzstd");
			CB_CUDA(ctx, mem.free(d_scratch));
		}
		else
		{
			k_aocs_inflate<<<nblk, AOCS_WARPS * 32, 0, ctx->stream>>>(d_raw, d_dir, (int) ndir, ctx->d_status, d_flag);
			CB_LAUNCHED(ctx, "k_aocs_inflate");
		}
		if (dmode != 1 && !anynull && !rel->nulls[col])
		{
			/* whether an inflated block carries a NULL bitmap is only known now */
			CB_CUDA(ctx, cudaMemcpyAsync(&flag, d_flag, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
			CB_CUDA(ctx, mem.sync());
			anynull = flag != 0;
		}
		CB_CUDA(ctx, mem.free(d_flag));
	}
	if (dmode != 1 && anynull && !rel->nulls[col])
	{
		int			rc = cbgpu_rel_add_nullmap(rel, col);

		if (rc)
			return rc;
	}
	memset(&P, 0, sizeof(P));
	P.raw = d_raw;
	P.dir = d_dir;
	P.nblocks = (int32_t) ndir;
	P.attlen = attlen;
	P.varkind = varkind;
	P.typalign = typalign;
	if (dmode != 1)
	{
		P.dscale = rel->dscales[col];
		P.out = rel->data[col];
		P.outnull = rel->nulls[col];
	}
	P.status = ctx->d_status;
	if (dict)
	{
		P.dslots = dict->d_slots;
		P.darena = dict->d_arena;
		P.dcursor = dict->d_cursor;
		P.dmask = dict->nslots - 1;
		P.darena_cap = dict->arena_cap;
		P.dmode = dmode;
		P.dtrim = dict->bpchar;
		P.doutw = outw;
		P.dmax = dict->max_entries;
	}
	k_aocs_decode<<<nblk, AOCS_WARPS * 32, 0, ctx->stream>>>(P);
	CB_LAUNCHED(ctx, "k_aocs_decode");
	CB_CUDA(ctx, mem.sync());	/* the caller's file buffer and `dir` are free again */
	CB_CUDA(ctx, mem.free(d_raw));
	CB_CUDA(ctx, mem.free(d_dir));
	*nrows_out = rows;
	return cbgpu_check_status(ctx);
}

/* ---- dictionaries ---- */
extern "C" int
cbgpu_dict_create(cbgpu_ctx *ctx, int32_t max_entries, int64_t arena_bytes, int32_t bpchar, cbgpu_dict **out)
{
	uint32_t	nslots = 64;

	*out = NULL;
	if (max_entries < 1 || max_entries > (1 << 26) || arena_bytes < 16 || arena_bytes > 0xFFFFFFF0ll)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_dict_create: %s%lld entries", "", max_entries);
	while (nslots < (uint32_t) max_entries * 2u)
		nslots <<= 1;
	CbOwned<cbgpu_dict> d((cbgpu_dict *) calloc(1, sizeof(cbgpu_dict)), cbgpu_dict_free);

	if (!d)
		return CBGPU_ERR_NOMEM;
	d->ctx = ctx;
	d->nslots = nslots;
	d->arena_cap = (uint32_t) arena_bytes;
	d->max_entries = max_entries;
	d->bpchar = bpchar != 0;
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	CB_CUDA(ctx, cudaMallocAsync(&d->d_slots, sizeof(DictSlot) * (size_t) nslots, ctx->stream));
	CB_CUDA(ctx, cudaMemsetAsync(d->d_slots, 0, sizeof(DictSlot) * (size_t) nslots, ctx->stream));
	CB_CUDA(ctx, cudaMallocAsync(&d->d_arena, (size_t) arena_bytes + 16, ctx->stream));
	CB_CUDA(ctx, cudaMallocAsync(&d->d_cursor, 2 * sizeof(unsigned long long), ctx->stream));
	CB_CUDA(ctx, cudaMemsetAsync(d->d_cursor, 0, 2 * sizeof(unsigned long long), ctx->stream));
	*out = d.release();
	return CBGPU_OK;
}

extern "C" void
cbgpu_dict_free(cbgpu_dict *d)
{
	if (!d)
		return;
	cudaSetDevice(d->ctx->device);
	if (d->d_slots)
		cudaFreeAsync(d->d_slots, d->ctx->stream);
	if (d->d_arena)
		cudaFreeAsync(d->d_arena, d->ctx->stream);
	if (d->d_cursor)
		cudaFreeAsync(d->d_cursor, d->ctx->stream);
	if (d->d_hashes)
		cudaFreeAsync(d->d_hashes, d->ctx->stream);
	if (d->d_offlen)
		cudaFreeAsync(d->d_offlen, d->ctx->stream);
	free(d->texts);
	free(d->off);
	free(d->len);
	free(d->sorted);
	free(d);
}

extern "C" int
cbgpu_aocs_dict_collect(cbgpu_ctx *ctx, const void *file_bytes, int64_t nbytes, int32_t checksum, int32_t compresstype, int32_t typalign,
						cbgpu_dict *dict)
{
	int64_t		n = 0;

	if (!dict || dict->finalized)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_aocs_dict_collect: the dictionary is %s (%lld)", dict ? "already finalized" : "missing", 0);
	return aocs_decode_impl(ctx, file_bytes, nbytes, checksum, compresstype, -1, CBGPU_AOCS_VAR_DICT, typalign, NULL, 0, 0, &n, dict, 1);
}

extern "C" int
cbgpu_aocs_decode_dict_column(cbgpu_ctx *ctx, const void *file_bytes, int64_t nbytes, int32_t checksum, int32_t compresstype,
							  int32_t typalign, const cbgpu_dict *dict, cbgpu_rel *rel, int32_t col, int64_t row_offset, int64_t *nrows)
{
	int			rc;

	*nrows = 0;
	if (!dict || !dict->finalized)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_aocs_decode_dict_column: the dictionary is %s (%lld)", dict ? "not finalized" : "missing", 0);
	if (col >= 0 && col < rel->ncols && rel->types[col] == CB_DICT8 && dict->n > 256)
		return cb_fail(ctx, CBGPU_ERR_OVERFLOW, "%s%lld distinct values do not fit a CB_DICT8 column", "", dict->n);
	rc = aocs_decode_impl(ctx, file_bytes, nbytes, checksum, compresstype, -1, CBGPU_AOCS_VAR_DICT, typalign, rel, col, row_offset, nrows, dict, 2);
	if (rc)
		return rc;
	/* the column hashes as the reference's hashbpchar / hashtext would hash the strings: its own copy of the per-code
	 * hashes, so the relation outlives the dictionary */
	if (dict->n > 0)
	{
		if (rel->dict_hash[col] && rel->dict_n[col] > 0)
		{
			cudaFreeAsync(rel->dict_hash[col], ctx->stream);
			rel->dict_hash[col] = NULL;
		}
		CB_CUDA(ctx, cudaMallocAsync(&rel->dict_hash[col], (size_t) dict->n * sizeof(uint32_t), ctx->stream));
		CB_CUDA(ctx, cudaMemcpyAsync(rel->dict_hash[col], dict->d_hashes, (size_t) dict->n * sizeof(uint32_t), cudaMemcpyDeviceToDevice,
									 ctx->stream));
		rel->dict_n[col] = dict->n;
	}
	/* the declared n of a character(n) column is the loader's to give (cbgpu_rel_set_dict); until it does, -1 = unknown, and a
	 * LIKE over the column is refused rather than matched without its padding */
	if (rel->dict[col] != dict)
		rel->dict_bpchar_len[col] = dict->bpchar ? -1 : 0;
	rel->dict[col] = dict;
	return CBGPU_OK;
}

static const DictSlot *g_dict_sort_slots;
static const char *g_dict_sort_texts;

static int
dict_slot_cmp(const void *a, const void *b)
{
	const DictSlot *x = g_dict_sort_slots + *(const int32_t *) a;
	const DictSlot *y = g_dict_sort_slots + *(const int32_t *) b;
	const uint32_t m = x->len < y->len ? x->len : y->len;
	const int	c = memcmp(g_dict_sort_texts + x->off, g_dict_sort_texts + y->off, m);

	if (c)
		return c;
	return x->len < y->len ? -1 : x->len > y->len;
}

/* The last step of building a dictionary whose entries are in code order on the host (texts, off[], len[], and the slot
 * table with the codes assigned): the per-code hashes, the slot table and the per-code (offset, length) pairs k_dict_like
 * reads go to the device. */
static int
dict_publish(cbgpu_dict *d, CbCallMem *mem, const DictSlot *slots, int32_t n)
{
	cbgpu_ctx  *ctx = d->ctx;
	uint32_t   *hashes = mem->keep((uint32_t *) malloc(sizeof(uint32_t) * (size_t) (n ? n : 1)));
	uint2	   *offlen = mem->keep((uint2 *) malloc(sizeof(uint2) * (size_t) (n ? n : 1)));

	if (!hashes || !offlen)
		return CBGPU_ERR_NOMEM;
	for (int32_t c = 0; c < n; c++)
	{
		/* hashbpchar over the blank-trimmed bytes == hashtext over the same bytes: both hash_any (utils/adt/varchar.c:981-1010) */
		hashes[c] = pg_hash_bytes_host((const unsigned char *) d->texts + d->off[c], (int) d->len[c]);
		offlen[c] = make_uint2(d->off[c], d->len[c]);
	}
	CB_CUDA(ctx, mem->copy_in(d->d_slots, slots, sizeof(DictSlot) * (size_t) d->nslots));
	CB_CUDA(ctx, cudaMallocAsync(&d->d_hashes, sizeof(uint32_t) * (size_t) (n ? n : 1), ctx->stream));
	CB_CUDA(ctx, mem->copy_in(d->d_hashes, hashes, sizeof(uint32_t) * (size_t) n));
	CB_CUDA(ctx, cudaMallocAsync(&d->d_offlen, sizeof(uint2) * (size_t) (n ? n : 1), ctx->stream));
	CB_CUDA(ctx, mem->copy_in(d->d_offlen, offlen, sizeof(uint2) * (size_t) n));
	CB_CUDA(ctx, mem->sync());
	d->n = n;
	d->finalized = 1;
	return CBGPU_OK;
}

extern "C" int
cbgpu_dict_finalize(cbgpu_dict *d, int32_t *nentries)
{
	cbgpu_ctx  *ctx = d->ctx;
	CbCallMem	mem(ctx);
	DictSlot   *slots;
	unsigned long long cur[2];
	int32_t		n = 0;
	int			rc;

	if (nentries)
		*nentries = 0;
	if (d->finalized)
	{
		if (nentries)
			*nentries = d->n;
		return CBGPU_OK;
	}
	rc = cbgpu_check_status(ctx);
	if (rc)
		return rc;
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	CB_CUDA(ctx, cudaMemcpyAsync(cur, d->d_cursor, sizeof(cur), cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	slots = mem.keep((DictSlot *) malloc(sizeof(DictSlot) * (size_t) d->nslots));
	d->texts = (char *) malloc((size_t) cur[0] + 16);
	d->sorted = (int32_t *) malloc(sizeof(int32_t) * (size_t) (cur[1] ? cur[1] : 1));
	d->off = (uint32_t *) malloc(sizeof(uint32_t) * (size_t) (cur[1] ? cur[1] : 1));
	d->len = (uint32_t *) malloc(sizeof(uint32_t) * (size_t) (cur[1] ? cur[1] : 1));
	if (!slots || !d->texts || !d->sorted || !d->off || !d->len)
		return CBGPU_ERR_NOMEM;
	CB_CUDA(ctx, cudaMemcpyAsync(slots, d->d_slots, sizeof(DictSlot) * (size_t) d->nslots, cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaMemcpyAsync(d->texts, d->d_arena, (size_t) cur[0], cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	for (uint32_t i = 0; i < d->nslots; i++)
		if (slots[i].tag)
			d->sorted[n++] = (int32_t) i;
	if ((unsigned long long) n != cur[1])
		return cb_fail(ctx, CBGPU_ERR_INVALID, "dictionary set holds %s%lld entries, its counter says otherwise", "", n);
	g_dict_sort_slots = slots;
	g_dict_sort_texts = d->texts;
	qsort(d->sorted, (size_t) n, sizeof(int32_t), dict_slot_cmp);
	for (int32_t c = 0; c < n; c++)
	{
		DictSlot   *sl = slots + d->sorted[c];

		sl->code = c;
		d->off[c] = sl->off;
		d->len[c] = sl->len;
	}
	rc = dict_publish(d, &mem, slots, n);
	if (rc == CBGPU_OK && nentries)
		*nentries = n;
	return rc;
}

extern "C" int
cbgpu_dict_entry(const cbgpu_dict *d, int32_t code, const char **text, int32_t *len)
{
	if (!d || !d->finalized || code < 0 || code >= d->n)
		return CBGPU_ERR_INVALID;
	*text = d->texts + d->off[code];
	*len = (int32_t) d->len[code];
	return CBGPU_OK;
}

extern "C" int32_t
cbgpu_dict_lookup(const cbgpu_dict *d, const char *text, int32_t len)
{
	int32_t		lo = 0,
				hi;

	if (!d || !d->finalized || len < 0)
		return -1;
	if (d->bpchar)
		while (len > 0 && text[len - 1] == ' ')
			len--;
	hi = d->n - 1;
	while (lo <= hi)
	{
		const int32_t mid = (lo + hi) / 2;
		const uint32_t m = d->len[mid] < (uint32_t) len ? d->len[mid] : (uint32_t) len;
		int			c = memcmp(d->texts + d->off[mid], text, m);

		if (c == 0)
			c = d->len[mid] < (uint32_t) len ? -1 : d->len[mid] > (uint32_t) len;
		if (c == 0)
			return mid;
		if (c < 0)
			lo = mid + 1;
		else
			hi = mid - 1;
	}
	return -1;
}

extern "C" int32_t
cbgpu_dict_nentries(const cbgpu_dict *d)
{
	return d && d->finalized ? d->n : 0;
}

extern "C" int32_t
cbgpu_dict_is_bpchar(const cbgpu_dict *d)
{
	return d && d->bpchar;
}

static int
dict_text_cmp(const char *a, int32_t la, const char *b, int32_t lb)
{
	const int	c = memcmp(a, b, (size_t) (la < lb ? la : lb));

	return c ? c : la < lb ? -1 : la > lb;
}

extern "C" int
cbgpu_dict_from_texts(cbgpu_ctx *ctx, int32_t n, const char *const *texts, const int32_t *lens, int32_t bpchar, cbgpu_dict **out)
{
	int64_t		arena = 0;
	cbgpu_dict *raw = NULL;
	unsigned long long cur[2];
	int			rc;

	*out = NULL;
	if (n < 0 || (n > 0 && (!texts || !lens)))
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_dict_from_texts: %s%lld strings", "", n);
	for (int32_t c = 0; c < n; c++)
	{
		if (lens[c] < 0 || (lens[c] > 0 && !texts[c]))
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_dict_from_texts: string %s%lld is malformed", "", c);
		if (bpchar && lens[c] > 0 && texts[c][lens[c] - 1] == ' ')
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_dict_from_texts: string %s%lld of a bpchar dictionary has trailing blanks", "", c);
		if (c > 0 && dict_text_cmp(texts[c - 1], lens[c - 1], texts[c], lens[c]) >= 0)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_dict_from_texts: string %s%lld is not above the one before it in byte order", "", c);
		arena += (lens[c] + 3) & ~3;
		if (arena > 0xFFFFFFF0ll)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_dict_from_texts: %s%lld strings exceed the arena's 32-bit offsets", "", n);
	}
	rc = cbgpu_dict_create(ctx, n > 0 ? n : 1, arena < 16 ? 16 : arena, bpchar, &raw);
	if (rc)
		return rc;
	CbOwned<cbgpu_dict> d(raw, cbgpu_dict_free);
	CbCallMem	mem(ctx);
	DictSlot   *slots = mem.keep((DictSlot *) calloc(d->nslots, sizeof(DictSlot)));
	uint32_t	pos = 0;

	d->texts = (char *) malloc((size_t) arena + 16);
	d->sorted = (int32_t *) malloc(sizeof(int32_t) * (size_t) (n ? n : 1));
	d->off = (uint32_t *) malloc(sizeof(uint32_t) * (size_t) (n ? n : 1));
	d->len = (uint32_t *) malloc(sizeof(uint32_t) * (size_t) (n ? n : 1));
	if (!slots || !d->texts || !d->sorted || !d->off || !d->len)
		return CBGPU_ERR_NOMEM;
	/* the slot table the collect pass would have built: the same tags and probe sequence, so that
	 * cbgpu_aocs_decode_dict_column finds these strings as it finds collected ones */
	for (int32_t c = 0; c < n; c++)
	{
		const unsigned long long tag = dict_hash64((const uint8_t *) texts[c], lens[c]);
		uint32_t	i = (uint32_t) tag & (d->nslots - 1);

		while (slots[i].tag)
			i = (i + 1) & (d->nslots - 1);
		slots[i] = {tag, pos, (uint32_t) lens[c], c, 0};
		if (lens[c] > 0)
			memcpy(d->texts + pos, texts[c], (size_t) lens[c]);
		d->sorted[c] = (int32_t) i;
		d->off[c] = pos;
		d->len[c] = (uint32_t) lens[c];
		pos += (uint32_t) ((lens[c] + 3) & ~3);
	}
	cur[0] = pos;
	cur[1] = (unsigned long long) n;
	CB_CUDA(ctx, mem.copy_in(d->d_arena, d->texts, pos));
	CB_CUDA(ctx, mem.copy_in(d->d_cursor, cur, sizeof(cur)));
	rc = dict_publish(d.get(), &mem, slots, n);
	if (rc)
		return rc;
	*out = d.release();
	return CBGPU_OK;
}

/* ---- LIKE over a dictionary: one match per distinct string, a bitmap over the codes ---- */
#define LIKE_MAX_PATTERN 2048
#define LIKE_THREADS 256

struct DictLikeParams
{
	const uint8_t *arena;
	const uint2 *offlen;
	uint32_t   *bits;			/* ceil(n / 32) words, bit c of word c / 32 = code c matches          */
	int32_t		n;
	int32_t		bpchar_len;		/* character(n): n, the entries are matched blank-padded to n characters; 0 otherwise */
	int32_t		plen;
	uint8_t		pat[LIKE_MAX_PATTERN];
};

/* One thread per entry; every lane of a warp steps through the loop together, so the warp's 32 results are one ballot and
 * one word store.  The pattern is read by every thread at its own position: it is staged in shared memory. */
__global__ void __launch_bounds__(LIKE_THREADS)
k_dict_like(const __grid_constant__ DictLikeParams P)
{
	__shared__ uint8_t pat[LIKE_MAX_PATTERN];

	for (int i = threadIdx.x; i < P.plen; i += blockDim.x)
		pat[i] = P.pat[i];
	__syncthreads();
	for (int64_t base = (int64_t) blockIdx.x * blockDim.x; base < P.n; base += (int64_t) gridDim.x * blockDim.x)
	{
		const int64_t c = base + threadIdx.x;
		bool		m = false;

		if (c < P.n)
		{
			const uint2 ol = P.offlen[c];
			const uint8_t *t = P.arena + ol.x;
			int			pad = P.bpchar_len > 0 ? P.bpchar_len - like_utf8_chars(t, (int) ol.y) : 0;

			m = like_match(t, (int) ol.y, pad > 0 ? pad : 0, pat, P.plen);
		}
		const uint32_t w = __ballot_sync(0xffffffffu, m);

		if ((threadIdx.x & 31) == 0 && c < P.n)
			P.bits[c >> 5] = w;
	}
}

extern "C" int
cbgpu_dict_match_like(cbgpu_ctx *ctx, const cbgpu_dict *dict, const char *pattern, int32_t len, int32_t bpchar_len, uint32_t *bits_dev)
{
	DictLikeParams *P;
	int64_t		blocks;

	if (!dict || !dict->finalized || len < 0 || (len > 0 && !pattern) || (dict->n > 0 && !bits_dev))
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_dict_match_like: bad argument%s (%lld)", "", len);
	/* a bpchar dictionary holds its strings blank-trimmed: matching them needs the column's n, and only it has one */
	if (dict->bpchar ? bpchar_len < 1 : bpchar_len != 0)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_dict_match_like: %sbpchar_len %lld does not fit the dictionary (character(n) needs n >= 1, "
					   "varchar / text 0)", "", bpchar_len);
	if (like_pattern_check((const uint8_t *) pattern, len))
		return cb_fail(ctx, CBGPU_ERR_INVALID, "LIKE pattern must not end with escape character%s", "", 0);
	if (len > LIKE_MAX_PATTERN)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "LIKE pattern of %s%lld bytes is longer than the GPU path takes", "", len);
	if (dict->n == 0)
		return CBGPU_OK;
	P = (DictLikeParams *) cb_scratch(ctx, 0, sizeof(DictLikeParams));
	if (!P)
		return CBGPU_ERR_NOMEM;
	P->arena = dict->d_arena;
	P->offlen = dict->d_offlen;
	P->bits = bits_dev;
	P->n = dict->n;
	P->bpchar_len = bpchar_len;
	P->plen = len;
	if (len > 0)
		memcpy(P->pat, pattern, (size_t) len);
	blocks = ((int64_t) dict->n + LIKE_THREADS - 1) / LIKE_THREADS;
	if (blocks > (int64_t) ctx->sm_count * 16)
		blocks = (int64_t) ctx->sm_count * 16;
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	k_dict_like<<<(int) blocks, LIKE_THREADS, 0, ctx->stream>>>(*P);
	CB_LAUNCHED(ctx, "k_dict_like");
	return CBGPU_OK;
}

/* ---------------------------------------------------------------------------------------------
 * Visibility map: pg_aovisimap entries -> the relation's one-bit-per-row visibility bitmap.
 * AppendOnlyVisimap_IsVisible (access/appendonly/appendonly_visimap.c:198) looks a row up by its AO row number: the
 * entry for (rownum / 32768) * 32768 (AppendOnlyVisimapEntry_GetFirstRowNum, appendonly_visimap_entry.c:427-437) holds a
 * bitmap of HIDDEN rows, bit (rownum - first_row_no) (:451-493), stored through Bitmap_Compress
 * (utils/misc/bitmap_compression.c:31-190: MSB-first bit stream (utils/misc/bitstream.c:52-70,160-178), 1 bit type, 3
 * unused, 12 bits block count; per 32-bit block a 2-bit flag: 00 zero, 01 ones, 11 raw 32 bits, 10 repeat the last
 * block 8-bit-count + 1 times).  A row's number is its block's firstRowNum + its position in the block.
 *   k_visimap_expand  one thread per entry: the compressed stream -> 1024 words (a 32768-row range)
 *   k_visimap_apply   one thread per byte of the relation's bitmap (8 rows): block by binary search over the row
 *                     bases, entry by binary search over the sorted first row numbers, bit test, write 1 = visible
 * --------------------------------------------------------------------------------------------- */
#define VISIMAP_RANGE 32768
#define VISIMAP_WORDS (VISIMAP_RANGE / 32)

struct VisiEntryDev
{
	long long	first;			/* first_row_no                                                       */
	long long	off;			/* payload offset in the uploaded buffer, -1 = NULL visimap (all visible) */
	int32_t		len;
	int32_t		pad;
};

__global__ void
k_visimap_expand(const uint8_t *data, const VisiEntryDev *ent, int nent, uint32_t *words, int *status)
{
	const int	e = blockIdx.x * blockDim.x + threadIdx.x;

	if (e >= nent)
		return;
	uint32_t   *out = words + (size_t) e * VISIMAP_WORDS;
	const VisiEntryDev E = ent[e];
	uint32_t	n = 0;

	if (E.off >= 0)
	{
		const uint8_t *p = data + E.off;
		const uint32_t nbits = ((uint32_t) E.len - 4u) * 8u;
		uint32_t	pos = 0;
		bool		bad = false;
		/* n bits, most significant first; past the end: error (Bitstream_CheckForError) */
		auto		get = [&](int k) -> uint32_t {
			uint32_t	v = 0;

			if (pos + (uint32_t) k > nbits)
			{
				bad = true;
				return 0u;
			}
			for (int i = 0; i < k; i++, pos++)
				v = (v << 1) | ((p[4 + (pos >> 3)] >> (7 - (pos & 7))) & 1u);
			return v;
		};

		if (E.len < 6 || p[0] != 1 || p[1] || p[2] || p[3])
			bad = true;			/* AppendOnlyVisimapData.version */
		else
		{
			const uint32_t type = get(1);

			get(3);
			n = get(12);
			if (n > VISIMAP_WORDS)
				bad = true;
			else if (type == 0)
			{
				if (2u + 4u * n > (uint32_t) E.len - 4u)
					bad = true;
				else
					for (uint32_t i = 0; i < n; i++)
						out[i] = aocs_le32(p + 4 + 2 + 4 * i);
			}
			else
			{
				uint32_t	last = 0,
							repeat = 0;

				for (uint32_t i = 0; i < n && !bad; i++)
				{
					if (repeat)
						repeat--;
					else
					{
						const uint32_t flag = get(2);

						if (flag == 0)
							last = 0;
						else if (flag == 1)
							last = 0xFFFFFFFFu;
						else if (flag == 3)
							last = get(32);
						else if (i == 0)
							bad = true;
						else
							repeat = get(8);
					}
					out[i] = last;
				}
				if (repeat)
					bad = true;
			}
		}
		if (bad)
		{
			atomicExch(status, CBGPU_ERR_CORRUPT);
			n = 0;
		}
	}
	for (uint32_t i = n; i < VISIMAP_WORDS; i++)
		out[i] = 0;
}

__global__ void
k_visimap_apply(const AocsDir *dir, int ndir, const VisiEntryDev *ent, int nent, const uint32_t *words, uint8_t *vis, long long row_lo,
				long long row_hi, unsigned long long *nhidden)
{
	const long long byte0 = row_lo >> 3;
	const long long B = byte0 + (long long) blockIdx.x * blockDim.x + threadIdx.x;

	if (B * 8 >= row_hi)
		return;
	uint32_t	bits = vis[B];
	int			blk = -1;
	int			hidden = 0;

	for (int j = 0; j < 8; j++)
	{
		const long long g = B * 8 + j;	/* row of the relation */

		if (g < row_lo || g >= row_hi)
			continue;
		if (blk < 0 || g >= dir[blk].rowbase + dir[blk].rows)
		{
			int			lo = 0,
						hi = ndir - 1;

			while (lo < hi)
			{
				const int	mid = (lo + hi + 1) >> 1;

				if (dir[mid].rowbase <= g)
					lo = mid;
				else
					hi = mid - 1;
			}
			blk = lo;
		}
		const long long rn = dir[blk].first + (g - dir[blk].rowbase);
		const long long want = rn / VISIMAP_RANGE * VISIMAP_RANGE;
		int			lo = 0,
					hi = nent - 1;
		bool		hide = false;

		while (lo < hi)
		{
			const int	mid = (lo + hi) >> 1;

			if (ent[mid].first < want)
				lo = mid + 1;
			else
				hi = mid;
		}
		if (nent > 0 && ent[lo].first == want)
		{
			const uint32_t o = (uint32_t) (rn - want);

			hide = (words[(size_t) lo * VISIMAP_WORDS + (o >> 5)] >> (o & 31)) & 1u;
		}
		if (hide)
		{
			bits &= ~(1u << j);
			hidden++;
		}
		else
			bits |= 1u << j;
	}
	vis[B] = (uint8_t) bits;
	if (hidden)
		atomicAdd(nhidden, (unsigned long long) hidden);
}

static int
visi_entry_cmp(const void *a, const void *b)
{
	const long long x = ((const VisiEntryDev *) a)->first, y = ((const VisiEntryDev *) b)->first;

	return x < y ? -1 : x > y;
}

extern "C" int
cbgpu_aocs_apply_visimap(cbgpu_ctx *ctx, const void *file_bytes, int64_t nbytes, int32_t checksum, const cbgpu_visimap_entry *entries,
						 int32_t nentries, cbgpu_rel *rel, int64_t row_offset, int64_t *nhidden_out)
{
	CbCallMem	mem(ctx);
	AocsWalk	W;
	VisiEntryDev *ent = NULL;
	uint8_t    *blob = NULL;
	int64_t		blobsz = 0;
	uint8_t    *d_blob = NULL;
	VisiEntryDev *d_ent = NULL;
	AocsDir    *d_dir = NULL;
	uint32_t   *d_words = NULL;
	unsigned long long *d_cnt = NULL;
	unsigned long long cnt = 0;
	int			rc;

	if (nhidden_out)
		*nhidden_out = 0;
	if (nentries < 0 || (nentries > 0 && !entries))
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_aocs_apply_visimap: bad entry list%s (%lld)", "", nentries);
	rc = aocs_walk(ctx, (const uint8_t *) file_bytes, nbytes, checksum, -1, row_offset, &W);
	if (rc)
		return rc;
	mem.keep(W.dir);
	if (row_offset < 0 || row_offset + W.rows > rel->capacity)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "AOCS column file holds %s%lld rows: more than the relation has room for", "", W.rows);
	for (int64_t i = 0; i < W.ndir; i++)
		if (W.dir[i].first < 0)
			return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "AOCS block %s%lld carries no first row number: rows cannot be matched to visimap entries", "", i);
	if (W.ndir == 0)
		return CBGPU_OK;
	ent = mem.keep((VisiEntryDev *) malloc(sizeof(VisiEntryDev) * (size_t) (nentries ? nentries : 1)));
	for (int i = 0; i < nentries; i++)
		blobsz += entries[i].data ? ((int64_t) entries[i].len + 7) / 8 * 8 : 0;
	blob = mem.keep((uint8_t *) calloc((size_t) blobsz + 8, 1));
	if (!ent || !blob)
		return CBGPU_ERR_NOMEM;
	blobsz = 0;
	for (int i = 0; i < nentries; i++)
	{
		if (entries[i].first_row_num < 0 || entries[i].first_row_num % VISIMAP_RANGE != 0 || (entries[i].data && entries[i].len < 6))
			return cb_fail(ctx, CBGPU_ERR_INVALID, "visimap entry %s%lld: first row number is not a multiple of 32768, or the data is too short", "", i);
		ent[i].first = entries[i].first_row_num;
		ent[i].len = entries[i].data ? entries[i].len : 0;
		ent[i].pad = 0;
		ent[i].off = -1;
		if (entries[i].data)
		{
			ent[i].off = blobsz;
			memcpy(blob + blobsz, entries[i].data, (size_t) entries[i].len);
			blobsz += ((int64_t) entries[i].len + 7) / 8 * 8;
		}
	}
	qsort(ent, (size_t) nentries, sizeof(VisiEntryDev), visi_entry_cmp);
	for (int i = 1; i < nentries; i++)
		if (ent[i].first == ent[i - 1].first)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "two visimap entries for first row number %s%lld", "", (long long) ent[i].first);
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	if (!rel->visimap)
	{
		const size_t bytes = (size_t) ((rel->capacity + 7) / 8);

		CB_CUDA(ctx, cudaMallocAsync(&rel->visimap, ((bytes + 255) & ~(size_t) 255) + 256, ctx->stream));
		CB_CUDA(ctx, cudaMemsetAsync(rel->visimap, 0xFF, ((bytes + 255) & ~(size_t) 255) + 256, ctx->stream));
	}
	CB_CUDA(ctx, mem.alloc(&d_dir, sizeof(AocsDir) * (size_t) W.ndir));
	CB_CUDA(ctx, mem.copy_in(d_dir, W.dir, sizeof(AocsDir) * (size_t) W.ndir));
	CB_CUDA(ctx, mem.alloc(&d_cnt, sizeof(unsigned long long)));
	CB_CUDA(ctx, cudaMemsetAsync(d_cnt, 0, sizeof(unsigned long long), ctx->stream));
	if (nentries)
	{
		CB_CUDA(ctx, mem.alloc(&d_ent, sizeof(VisiEntryDev) * (size_t) nentries));
		CB_CUDA(ctx, mem.copy_in(d_ent, ent, sizeof(VisiEntryDev) * (size_t) nentries));
		CB_CUDA(ctx, mem.alloc(&d_blob, (size_t) blobsz + 8));
		CB_CUDA(ctx, mem.copy_in(d_blob, blob, (size_t) blobsz + 8));
		CB_CUDA(ctx, mem.alloc(&d_words, sizeof(uint32_t) * VISIMAP_WORDS * (size_t) nentries));
		k_visimap_expand<<<(nentries + 127) / 128, 128, 0, ctx->stream>>>(d_blob, d_ent, nentries, d_words, ctx->d_status);
		CB_LAUNCHED(ctx, "k_visimap_expand");
	}
	{
		const long long lo = row_offset,
					hi = row_offset + W.rows;
		const long long nbytes_out = ((hi + 7) >> 3) - (lo >> 3);

		k_visimap_apply<<<(unsigned) ((nbytes_out + 255) / 256), 256, 0, ctx->stream>>>(d_dir, (int) W.ndir, d_ent, nentries, d_words,
																						 rel->visimap, lo, hi, d_cnt);
		CB_LAUNCHED(ctx, "k_visimap_apply");
	}
	CB_CUDA(ctx, cudaMemcpyAsync(&cnt, d_cnt, sizeof(cnt), cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, mem.sync());
	CB_CUDA(ctx, mem.free(d_dir));
	CB_CUDA(ctx, mem.free(d_cnt));
	if (nentries)
	{
		CB_CUDA(ctx, mem.free(d_ent));
		CB_CUDA(ctx, mem.free(d_blob));
		CB_CUDA(ctx, mem.free(d_words));
	}
	if (nhidden_out)
		*nhidden_out = (int64_t) cnt;
	return cbgpu_check_status(ctx);
}
