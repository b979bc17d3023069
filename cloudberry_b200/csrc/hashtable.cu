/*
 * hashtable.cu - hash join build (K2) and the stand-alone pair-emitting probe (K3).
 *
 * Build restates MultiExecPrivateHash -> ExecHashGetHashValue -> ExecHashTableInsert
 * (backend/executor/nodeHash.c:167, 2089, 1877): per inner row hash = rotl1-xor of the per-key
 * hash functions (no finaliser), rows with a NULL key are not inserted (strict operators, :2161).
 * The reference chains MinimalTuples off nbuckets = pow2(ntuples / 5) bucket heads; the device
 * table is open addressing with linear probing over slots = hash32 << 32 | inner row id, at load
 * factor <= 0.5, and late-materialises: the inner payload stays in its column arrays and is
 * gathered by row id only for surviving rows.  The slot position uses the same 32-bit hash value
 * the reference computes (bucketno = hashvalue & (nbuckets - 1), nodeHash.c:2233).  The slot
 * format and the N:1 walk live in common.cuh (ht_slot_entry .. ht_find), for every probing kernel.
 *
 * Probe restates ExecScanHashBucket (nodeHash.c:2255-2308): compare the stored hash value first,
 * then the key equality (hashqualclauses).
 */
#include "common.cuh"
#include "pipeline.cuh"
#include "xmatch.h"

#include <stdlib.h>

struct BuildParams
{
	HtDev		ht;
	int64_t		nrows;
	int		   *flags;			/* [0] duplicate key seen, [1] rows inserted, [2] a key outside the key-in-slot domain */
};

__device__ __forceinline__ bool
ht_row_hash(const HtDev &ht, uint32_t row, uint32_t *hash, int64_t *key0)
{
	uint32_t	h = 0;

	for (int k = 0; k < ht.nkeys; k++)
	{
		if (ht.keynulls[k] && ht.keynulls[k][row])
			return false;
		int64_t		v = cb_load_widen(ht.keydata[k], ht.keytype[k], row);

		if (k == 0)
			*key0 = v;
		h = jh_key_fold(h, ht.keytype[k], v, ht.keydict[k]);
	}
	*hash = h;
	return true;
}

__device__ __forceinline__ bool
ht_keys_equal_rows(const HtDev &ht, uint32_t ra, uint32_t rb)
{
	for (int k = 0; k < ht.nkeys; k++)
		if (cb_load_widen(ht.keydata[k], ht.keytype[k], ra) != cb_load_widen(ht.keydata[k], ht.keytype[k], rb))
			return false;
	return true;
}

__global__ void
k_ht_clear(unsigned long long *slots, size_t n)
{
	size_t		i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	size_t		stride = (size_t) gridDim.x * blockDim.x;

	for (; i < n; i += stride)
		slots[i] = HT_EMPTY;
}

__global__ void __launch_bounds__(256)
k_ht_build(BuildParams p)
{
	const int64_t stride = (int64_t) gridDim.x * blockDim.x;
	int			inserted = 0;
	bool		dup = false;
	bool		outside = false;

	for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < p.nrows; i += stride)
	{
		uint32_t	h = 0, w;
		int64_t		key0 = 0;
		bool		v = ht_row_hash(p.ht, (uint32_t) i, &h, &key0);

		if (v && !ht_in_batch(p.ht.nbatch, p.ht.batch_shift, p.ht.batch_id, h))
			v = false;			/* another batch's row */
		if (v && p.ht.keyslot && !ht_key_in_domain(p.ht.keyslot, key0))
		{
			outside = true;		/* the host builds the table again with hash values in the slots */
			v = false;
		}
		const uint32_t tag = ht_probe_tag(p.ht.keyslot, h, key0);
		const unsigned long long e = ht_slot_entry(tag, (uint32_t) i);
		uint32_t	pos = h & p.ht.mask;
		const uint32_t bits = ht_bloom_bits(h, &w, p.ht.bloom_mask);

		if (p.ht.bloom)
		{
			const uint32_t word = v ? p.ht.bloom[w] : 0xFFFFFFFFu;

			if ((word & bits) != bits)
				atomicOr(p.ht.bloom + w, bits);
		}
		if (!v)
			continue;
		unsigned long long cur = p.ht.slots[pos];

		for (;;)
		{
			unsigned long long c = cur;

			if (ht_slot_empty(c))
			{
				c = atomicCAS(p.ht.slots + pos, HT_EMPTY, e);
				if (ht_slot_empty(c))
					break;
			}
			/* occupied: the same key -> a duplicate on the build side (key-in-slot tables see it in the tag; the others
			 * compare hash values first, then the keys by row id) */
			if (!dup && ht_tag_match(c, tag) && (p.ht.keyslot || ht_keys_equal_rows(p.ht, ht_slot_row(c), (uint32_t) i)))
				dup = true;
			pos = (pos + 1) & p.ht.mask;
			cur = p.ht.slots[pos];
		}
		inserted++;
	}
	if (dup)
		atomicExch(p.flags, 1);
	if (outside)
		atomicExch(p.flags + 2, 1);
	/* one atomic per warp for the inserted count */
	for (int o = 16; o; o >>= 1)
		inserted += __shfl_xor_sync(0xffffffffu, inserted, o);
	if ((threadIdx.x & 31) == 0 && inserted)
		atomicAdd(p.flags + 1, inserted);
}

/* one fill of the table: every build row (nbatch <= 1) or the rows of batch `batch` */
static int
ht_fill(cbgpu_hashtable *ht, int batch)
{
	cbgpu_ctx  *ctx = ht->ctx;
	cbgpu_rel  *inner = ht->inner;
	BuildParams p;
	int			h_flags[3];

	ht->d.batch_id = batch;
	if (ht->d.bloom)
		CB_CUDA(ctx, cudaMemsetAsync(ht->d.bloom, 0, ((size_t) ht->d.bloom_mask + 1) * sizeof(uint32_t), ctx->stream));
	for (;;)
	{
		int			blocks = (int) ((ht->nslots + 255) / 256);

		CB_CUDA(ctx, cudaMemsetAsync(ht->d_flags, 0, 3 * sizeof(int), ctx->stream));
		if (blocks > ctx->sm_count * 8)
			blocks = ctx->sm_count * 8;
		k_ht_clear<<<blocks, 256, 0, ctx->stream>>>(ht->d.slots, (size_t) ht->nslots);
		CB_LAUNCHED(ctx, "k_ht_clear");
		p.ht = ht->d;
		p.nrows = inner->nrows;
		p.flags = ht->d_flags;
		if (inner->nrows > 0)
		{
			blocks = (int) ((inner->nrows + 255) / 256);
			if (blocks > ctx->sm_count * 8)
				blocks = ctx->sm_count * 8;
			k_ht_build<<<blocks, 256, 0, ctx->stream>>>(p);
			CB_LAUNCHED(ctx, "k_ht_build");
		}
		CB_CUDA(ctx, cudaMemcpyAsync(h_flags, ht->d_flags, sizeof(h_flags), cudaMemcpyDeviceToHost, ctx->stream));
		CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		if (h_flags[2] && ht->d.keyslot)
		{
			/* an int8 key beyond 32 bits: the general layout (hash value in the slot, key verified by row id) */
			ht->d.keyslot = 0;
			if (ht->d.bloom)
				CB_CUDA(ctx, cudaMemsetAsync(ht->d.bloom, 0, ((size_t) ht->d.bloom_mask + 1) * sizeof(uint32_t), ctx->stream));
			continue;
		}
		break;
	}
	if (h_flags[0])
		ht->has_dups = 1;
	ht->ninserted = h_flags[1];
	return CBGPU_OK;
}

/* rows per batch of a build side (the batch number of every row's key hash), to size the resident table for the fullest */
__global__ void
k_ht_batch_histogram(HtDev ht, int64_t nrows, unsigned long long *hist)
{
	for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < nrows; i += (int64_t) gridDim.x * blockDim.x)
	{
		uint32_t	h;
		int64_t		key0;

		if (ht_row_hash(ht, (uint32_t) i, &h, &key0))
			atomicAdd(hist + (h >> ht.batch_shift), 1ull);
	}
}

static int
ht_create(cbgpu_ctx *ctx, cbgpu_rel *inner, const int32_t *keycols, int32_t nkeys, int32_t nbatch, cbgpu_hashtable **out)
{
	cbgpu_hashtable *ht;
	CbCallMem	mem(ctx);
	int64_t		nslots = 64;
	int64_t		resident_rows = inner->nrows;

	*out = NULL;
	if (nkeys < 1 || nkeys > CBP_MAX_KEYS)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "hash join with %s%lld key columns is beyond the GPU path's limit (4)", "", nkeys);
	if (nbatch < 1 || nbatch > 4096 || (nbatch & (nbatch - 1)) != 0)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "hash join with %s%lld batches (a power of two up to 4096 is expected)", "", nbatch);
	/* published at once: whatever fails from here on, cbgpu_ht_build frees it */
	*out = ht = (cbgpu_hashtable *) calloc(1, sizeof(cbgpu_hashtable));
	if (!ht)
		return CBGPU_ERR_NOMEM;
	ht->ctx = ctx;
	ht->inner = inner;
	ht->total_rows = inner->nrows;
	ht->d.nkeys = nkeys;
	ht->d.nbatch = nbatch;
	ht->d.batch_shift = 32;
	for (int b = nbatch; b > 1; b >>= 1)
		ht->d.batch_shift--;
	for (int k = 0; k < nkeys; k++)
	{
		int			c = keycols[k];

		if (c < 0 || c >= inner->ncols)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_ht_build: bad key column%s %lld", "", c);
		if (inner->types[c] == CB_NUMERIC)
			return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "numeric hash join keys (hash_numeric) are not on the GPU path%s", "", 0);
		if ((inner->types[c] == CB_DICT8 || inner->types[c] == CB_DICT32) && !inner->dict_hash[c])
			return cb_fail(ctx, CBGPU_ERR_INVALID, "dictionary column %s%lld used as a join key without dict hashes", "", c);
		ht->d.keydata[k] = inner->data[c];
		ht->d.keynulls[k] = inner->nulls[c];
		ht->d.keydict[k] = inner->dict_hash[c];
		ht->d.keytype[k] = inner->types[c];
	}
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	if (nbatch > 1 && inner->nrows > 0)
	{
		/* the fullest batch sizes the table (hash skew: duplicate keys all land in one batch) */
		unsigned long long *d_hist,
				   *h_hist = mem.keep((unsigned long long *) calloc((size_t) nbatch, sizeof(unsigned long long)));
		int			blocks = (int) ((inner->nrows + 255) / 256);

		if (!h_hist)
			return CBGPU_ERR_NOMEM;
		if (blocks > ctx->sm_count * 8)
			blocks = ctx->sm_count * 8;
		CB_CUDA(ctx, mem.alloc(&d_hist, sizeof(unsigned long long) * (size_t) nbatch));
		CB_CUDA(ctx, cudaMemsetAsync(d_hist, 0, sizeof(unsigned long long) * (size_t) nbatch, ctx->stream));
		k_ht_batch_histogram<<<blocks, 256, 0, ctx->stream>>>(ht->d, inner->nrows, d_hist);
		CB_LAUNCHED(ctx, "k_ht_batch_histogram");
		CB_CUDA(ctx, cudaMemcpyAsync(h_hist, d_hist, sizeof(unsigned long long) * (size_t) nbatch, cudaMemcpyDeviceToHost, ctx->stream));
		CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		CB_CUDA(ctx, mem.free(d_hist));
		resident_rows = 0;
		for (int b = 0; b < nbatch; b++)
			if ((int64_t) h_hist[b] > resident_rows)
				resident_rows = (int64_t) h_hist[b];
	}
	while (nslots < resident_rows * 2)
		nslots <<= 1;
	if (nslots > (1ll << 32))
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "hash join build side too large for 32-bit slots%s (%lld rows)", "", inner->nrows);
	ht->nslots = nslots;
	ht->d.mask = (uint32_t) (nslots - 1);
	CB_CUDA(ctx, cudaMallocAsync(&ht->d.slots, (size_t) nslots * sizeof(unsigned long long), ctx->stream));
	CB_CUDA(ctx, cudaMallocAsync(&ht->d_flags, 3 * sizeof(int), ctx->stream));
	/* one integer key: try the key-in-slot layout (int8 keys: as long as every build value lies in [0, 2^32)) */
	if (nkeys == 1)
		switch (ht->d.keytype[0])
		{
			case CB_INT8:
				ht->d.keyslot = 2;
				break;
			case CB_INT4: case CB_DATE: case CB_DICT8: case CB_DICT32: case CB_BPCHAR1: case CB_BOOL:
				ht->d.keyslot = 1;
				break;
			default:
				break;
		}
	{
		/* ~16 filter bits per build row, at least one cache line */
		int64_t		words = 32;
		const int	div = ctx->opt_bloom_div;	/* rows per 32-bit filter word (CBGPU_BLOOM_DIV, tuning aid), default 2 */

		while (words < resident_rows / div)
			words <<= 1;
		CB_CUDA(ctx, cudaMallocAsync(&ht->d.bloom, (size_t) words * sizeof(uint32_t), ctx->stream));
		ht->d.bloom_mask = (uint32_t) (words - 1);
		ht->built_bytes = nslots * 8 + words * 4;
	}
	return CBGPU_OK;
}

/* what a single-batch table over `rows` build rows takes on the device (slots at load factor <= 0.5 + the filter):
 * the caller's figure for choosing nbatch against its memory budget (ExecChooseHashTableSize, nodeHash.c:856-1100) */
extern "C" int64_t
cbgpu_ht_bytes_for(int64_t rows)
{
	int64_t		nslots = 64,
				words = 32;

	while (nslots < rows * 2)
		nslots <<= 1;
	while (words < rows / 2)
		words <<= 1;
	return nslots * 8 + words * 4;
}

extern "C" int
cbgpu_ht_build(cbgpu_ctx *ctx, cbgpu_rel *inner, const int32_t *keycols, int32_t nkeys, int32_t nbatch, cbgpu_hashtable **out)
{
	int			rc = ht_create(ctx, inner, keycols, nkeys, nbatch, out);

	/* every batch is built once now: duplicates on the build side decide the join's shape (N:1 or N:M) before the
	 * first probe, and the key-in-slot layout must hold for all batches alike */
	for (int b = 0; b < nbatch && rc == CBGPU_OK; b++)
		rc = ht_fill(*out, b);
	if (rc == CBGPU_OK && (*out)->d.keyslot == 0 && nbatch > 1)
		rc = ht_fill(*out, nbatch - 1);	/* a late fallback to hash-in-slot: the resident batch must use the final layout */
	if (rc != CBGPU_OK && *out)
	{
		cbgpu_ht_free(*out);
		*out = NULL;
	}
	return rc;
}

extern "C" int
cbgpu_ht_nbatch(const cbgpu_hashtable *ht)
{
	return ht->d.nbatch > 1 ? ht->d.nbatch : 1;
}

extern "C" int
cbgpu_ht_load_batch(cbgpu_hashtable *ht, int32_t batch)
{
	if (batch < 0 || batch >= cbgpu_ht_nbatch(ht))
		return cb_fail(ht->ctx, CBGPU_ERR_INVALID, "hash join batch %s%lld out of range", "", batch);
	if (ht->d.nbatch > 1 && ht->d.batch_id == batch)
		return CBGPU_OK;
	return ht_fill(ht, batch);
}

extern "C" void
cbgpu_ht_free(cbgpu_hashtable *ht)
{
	if (!ht)
		return;
	cudaSetDevice(ht->ctx->device);
	if (ht->d.slots)
		cudaFreeAsync(ht->d.slots, ht->ctx->stream);
	if (ht->d.bloom)
		cudaFreeAsync(ht->d.bloom, ht->ctx->stream);
	if (ht->d_flags)
		cudaFreeAsync(ht->d_flags, ht->ctx->stream);
	free(ht);
}

extern "C" int64_t
cbgpu_ht_nrows(const cbgpu_hashtable *ht)
{
	return ht->d.nbatch > 1 ? ht->total_rows : ht->ninserted;
}

extern "C" int
cbgpu_ht_has_duplicates(const cbgpu_hashtable *ht)
{
	return ht->has_dups;
}

extern "C" const uint32_t *
cbgpu_ht_key_dict_hash(const cbgpu_hashtable *ht, int32_t k)
{
	return (k >= 0 && k < ht->d.nkeys) ? ht->d.keydict[k] : NULL;
}

/* ---------------------------------------------------------------------------------------------
 * K3 stand-alone: (outer_idx, inner_idx) pairs for every match (INNER join), two passes:
 * count matches per outer row -> exclusive scan -> write pairs.  Output order is outer-row major,
 * so the pair list is deterministic.
 * --------------------------------------------------------------------------------------------- */
/* the join filter of a filtered pair probe; ops == NULL: none */
struct JoinFilterDev
{
	const CbpColumn *cols;		/* device copies of the program                                       */
	const CbpOp *ops;
	int32_t		nops;
	int32_t		jointype;		/* CB_JOIN_LEFT, SEMI or ANTI                                         */
	uint32_t   *decision;		/* SEMI / ANTI: [rows of the pass] the first passing build row, or 0xFFFFFFFF */
	int		   *status;			/* the context's status word: CBGPU_ERR_OVERFLOW                      */
};

struct ProbeParams
{
	HtDev		ht;
	const void *okey[CBP_MAX_KEYS];
	const uint8_t *onulls[CBP_MAX_KEYS];
	const uint32_t *odict[CBP_MAX_KEYS];
	int32_t		otype[CBP_MAX_KEYS];
	const uint32_t *sel;
	int64_t		n;
	int32_t		left;			/* LEFT join: an outer row without a partner yields one pair (row, 0xFFFFFFFF)  */
	uint8_t    *matched;		/* RIGHT / FULL join: [inner rows] set to 1 for every build row that found a partner
								 * (HeapTupleHeaderSetMatch, nodeHashjoin.c:560); NULL otherwise */
	int64_t		ninner;
	unsigned long long *counts;	/* [n + 1] match counts, then their exclusive scan                    */
	uint32_t   *out_outer;
	uint32_t   *out_inner;
	JoinFilterDev f;
};

/* an outer row's key hash (ht_row_hash over the probe side's columns) and its batch: the bits ht_in_batch tests, and batch 0
 * for a NULL key, which never matches (the N:1 probe and the reference put such rows there too).  The batch partition and the
 * pair probe both decide a row's batch here, so that a row is probed, or NULL-extended, in exactly one pass. */
__device__ __forceinline__ int32_t
ht_probe_row_batch(const ProbeParams &p, uint32_t row, int64_t *key, uint32_t *hash, bool *keynull)
{
	uint32_t	h = 0;
	bool		isnull = false;

	for (int k = 0; k < p.ht.nkeys; k++)
	{
		if (p.onulls[k] && p.onulls[k][row])
			isnull = true;
		key[k] = cb_load_widen(p.okey[k], p.otype[k], row);
		h = jh_key_fold(h, p.otype[k], key[k], p.odict[k]);
	}
	*hash = h;
	*keynull = isnull;
	return (p.ht.nbatch <= 1 || isnull) ? 0 : (int32_t) (h >> p.ht.batch_shift);
}

/* an outer row's key, hash and batch (*mine: the resident batch is the row's own), and whether it needs the table at all: its
 * key is not NULL, the Bloom filter may hold it, it lies in the key-in-slot domain and its batch is resident */
__device__ __forceinline__ bool
ht_probe_admits(const ProbeParams &p, uint32_t row, int64_t *key, uint32_t *h, bool *mine)
{
	bool		isnull;

	*mine = ht_probe_row_batch(p, row, key, h, &isnull) == p.ht.batch_id || p.ht.nbatch <= 1;
	if (!isnull && p.ht.bloom)
	{
		uint32_t	w;
		uint32_t	bits = ht_bloom_bits(*h, &w, p.ht.bloom_mask);

		if ((__ldg(p.ht.bloom + w) & bits) != bits)
			isnull = true;		/* certainly absent */
	}
	if (!isnull && p.ht.keyslot && !ht_key_in_domain(p.ht.keyslot, key[0]))
		isnull = true;			/* outside the build side's key domain: no partner */
	if (!isnull && !*mine)
		isnull = true;			/* multi-batch join: this row belongs to another pass */
	return !isnull;
}

template <bool WRITE>
__global__ void __launch_bounds__(256)
k_ht_probe_pairs(ProbeParams p)
{
	int64_t		i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
	int64_t		stride = (int64_t) gridDim.x * blockDim.x;

	for (; i < p.n; i += stride)
	{
		uint32_t	row = p.sel ? p.sel[i] : (uint32_t) i;
		uint32_t	h;
		int64_t		key[CBP_MAX_KEYS];
		bool		mine;
		unsigned long long cnt = 0;
		unsigned long long base = WRITE ? p.counts[i] : 0;

		if (ht_probe_admits(p, row, key, &h, &mine))
		{
			const uint32_t tag = ht_probe_tag(p.ht.keyslot, h, key[0]);
			uint32_t	pos = h & p.ht.mask;

			for (;;)
			{
				unsigned long long e = p.ht.slots[pos];

				if (ht_slot_empty(e))
					break;
				if (ht_slot_match(p.ht, e, tag, key, p.ht.nkeys))
				{
					if (WRITE)
					{
						p.out_outer[base + cnt] = row;
						p.out_inner[base + cnt] = ht_slot_row(e);
					}
					else if (p.matched)
						p.matched[ht_slot_row(e)] = 1;
					cnt++;
				}
				pos = (pos + 1) & p.ht.mask;
			}
		}
		if (p.left && cnt == 0 && mine)
		{
			/* no partner (or a NULL key, which never has one): the outer row survives with a NULL inner side */
			if (WRITE)
			{
				p.out_outer[base] = row;
				p.out_inner[base] = 0xFFFFFFFFu;
			}
			cnt = 1;
		}
		if (!WRITE)
			p.counts[i] = cnt;
	}
}

/* the join filter over one key-equal candidate (outer row orow, build row irow): true only for a non-NULL true result */
__device__ __forceinline__ bool
join_filter_passes(const JoinFilterDev &f, uint32_t orow, uint32_t irow)
{
	int64_t		st[CBP_STACK];
	uint64_t	snull = 0;
	int			sp = 0;

	for (int pc = 0; pc < f.nops; pc++)
	{
		const CbpOp op = f.ops[pc];

		if (op.code == CBP_LOAD)
		{
			const CbpColumn &c = f.cols[op.a];
			const uint32_t r = c.src ? irow : orow;
			const bool	isnull = c.nulls && c.nulls[r];

			st[sp] = isnull ? 0 : cb_load_widen(c.data, c.type, r);
			snull = isnull ? (snull | (1ull << sp)) : (snull & ~(1ull << sp));
			sp++;
		}
		else
			cbp_scalar_op(op, st, snull, sp, true, f.status);
	}
	return !(snull & 1) && st[0] != 0;
}

/* The pair probe of a LEFT / SEMI / ANTI join with a join filter: ExecScanHashBucket's walk (nodeHash.c:2255) with the joinqual
 * tested on every key-equal candidate (nodeHashjoin.c:583-713).  SEMI / ANTI stop at the first passing candidate (single_match
 * :626, :610) and walk once: the count pass keeps each row's decision, the write pass only emits it.  LEFT emits every passing
 * pair, so its write pass walks again. */
template <bool WRITE>
__global__ void __launch_bounds__(256)
k_ht_probe_filtered(ProbeParams p)
{
	int64_t		i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
	int64_t		stride = (int64_t) gridDim.x * blockDim.x;
	const bool	left = p.f.jointype == CB_JOIN_LEFT;

	for (; i < p.n; i += stride)
	{
		const uint32_t row = p.sel ? p.sel[i] : (uint32_t) i;

		if (WRITE && !left)
		{
			const unsigned long long at = p.counts[i];

			if (p.counts[i + 1] != at)
			{
				p.out_outer[at] = row;
				p.out_inner[at] = p.f.decision[i];
			}
			continue;
		}
		uint32_t	h;
		int64_t		key[CBP_MAX_KEYS];
		bool		mine;
		unsigned long long cnt = 0;
		const unsigned long long base = WRITE ? p.counts[i] : 0;
		uint32_t	first = 0xFFFFFFFFu;

		if (ht_probe_admits(p, row, key, &h, &mine))
		{
			const uint32_t tag = ht_probe_tag(p.ht.keyslot, h, key[0]);
			uint32_t	pos = h & p.ht.mask;

			for (;;)
			{
				unsigned long long e = p.ht.slots[pos];

				if (ht_slot_empty(e))
					break;
				if (ht_slot_match(p.ht, e, tag, key, p.ht.nkeys) && join_filter_passes(p.f, row, ht_slot_row(e)))
				{
					if (!left)
					{
						first = ht_slot_row(e);
						break;
					}
					if (WRITE)
					{
						p.out_outer[base + cnt] = row;
						p.out_inner[base + cnt] = ht_slot_row(e);
					}
					cnt++;
				}
				pos = (pos + 1) & p.ht.mask;
			}
		}
		if (!left)
		{
			/* SEMI: the row with its first passing partner; ANTI: the row when none passed (a NULL key included) */
			p.f.decision[i] = first;
			p.counts[i] = p.f.jointype == CB_JOIN_SEMI ? first != 0xFFFFFFFFu : (first == 0xFFFFFFFFu && mine);
			continue;
		}
		if (cnt == 0 && mine)
		{
			/* no passing partner: the outer row survives once with a NULL inner side */
			if (WRITE)
			{
				p.out_outer[base] = row;
				p.out_inner[base] = 0xFFFFFFFFu;
			}
			cnt = 1;
		}
		if (!WRITE)
			p.counts[i] = cnt;
	}
}

/* single-CTA chained exclusive scan (the pair-emitting probe is the general N:M fallback, not a
 * hot kernel; correctness and determinism matter here, not speed) */
__global__ void
k_exclusive_scan_u64(unsigned long long *a, int64_t n)
{
	__shared__ unsigned long long carry;
	__shared__ unsigned long long warp_tot[32];

	if (threadIdx.x == 0)
		carry = 0;
	__syncthreads();
	for (int64_t base = 0; base < n; base += blockDim.x)
	{
		int64_t		i = base + threadIdx.x;
		unsigned long long v = i < n ? a[i] : 0;
		unsigned long long x = v;
		int			lane = threadIdx.x & 31,
					w = threadIdx.x >> 5;

		for (int o = 1; o < 32; o <<= 1)
		{
			unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);

			if (lane >= o)
				x += y;
		}
		if (lane == 31)
			warp_tot[w] = x;
		__syncthreads();
		if (w == 0)
		{
			unsigned long long t = lane < (int) (blockDim.x >> 5) ? warp_tot[lane] : 0;

			for (int o = 1; o < 32; o <<= 1)
			{
				unsigned long long y = __shfl_up_sync(0xffffffffu, t, o);

				if (lane >= o)
					t += y;
			}
			warp_tot[lane] = t;
		}
		__syncthreads();
		unsigned long long prev = (w ? warp_tot[w - 1] : 0) + carry;

		if (i < n)
			a[i] = prev + x - v;
		__syncthreads();
		if (threadIdx.x == blockDim.x - 1)
			carry = prev + x;
		__syncthreads();
	}
	if (threadIdx.x == 0)
		a[n] = carry;
}

/* RIGHT / FULL join: the build rows no probe row matched, each as a pair (0xFFFFFFFF, row) behind the matches
 * (ExecScanHashTableForUnmatched, nodeHash.c:2360; HJ_FILL_INNER_TUPLES, nodeHashjoin.c:676-706).  Rows whose key is NULL
 * were never inserted and never match: they are emitted too (the reference keeps them in the table for this, keep_nulls
 * nodeHash.c:209). */
__global__ void
k_ht_unmatched_count(ProbeParams p)
{
	int64_t		i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
	int64_t		stride = (int64_t) gridDim.x * blockDim.x;

	for (; i < p.ninner; i += stride)
		p.counts[p.n + i] = p.matched[i] ? 0 : 1;
}

__global__ void
k_ht_unmatched_write(ProbeParams p)
{
	int64_t		i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
	int64_t		stride = (int64_t) gridDim.x * blockDim.x;

	for (; i < p.ninner; i += stride)
		if (!p.matched[i])
		{
			unsigned long long at = p.counts[p.n + i];

			p.out_outer[at] = 0xFFFFFFFFu;
			p.out_inner[at] = (uint32_t) i;
		}
}

/* ---------------------------------------------------------------------------------------------
 * The probe side of a multi-batch pair join, partitioned by batch once (the reference writes each outer tuple to its batch's
 * file instead: ExecHashJoinSaveTuple, nodeHashjoin.c): a stable counting sort of the outer row ids into nbatch runs.  Each
 * CTA owns a contiguous chunk of rows.  k_ht_partition_count reads the key columns, keeps every row's batch and counts its
 * chunk's rows per batch; an exclusive scan over the [batch][CTA] counts gives each (batch, CTA) its first position; then
 * k_ht_partition_write places the rows tile by tile, the warps of a tile in order, so each run lists its rows in relation
 * order and the pair list's probe-row order is the same on every run.
 * --------------------------------------------------------------------------------------------- */
#define HT_PART_THREADS 256

__global__ void __launch_bounds__(HT_PART_THREADS)
k_ht_partition_count(ProbeParams p, int64_t chunk, uint16_t *rowbatch, unsigned long long *hist)
{
	extern __shared__ uint32_t cnt[];	/* [nbatch] */
	const int64_t lo = (int64_t) blockIdx.x * chunk;
	const int64_t hi = lo + chunk < p.n ? lo + chunk : p.n;

	for (int b = threadIdx.x; b < p.ht.nbatch; b += blockDim.x)
		cnt[b] = 0;
	__syncthreads();
	for (int64_t i0 = lo; i0 < hi; i0 += blockDim.x)
	{
		const int64_t i = i0 + threadIdx.x;
		int32_t		b = -1;

		if (i < hi)
		{
			int64_t		key[CBP_MAX_KEYS];
			uint32_t	h;
			bool		isnull;

			b = ht_probe_row_batch(p, (uint32_t) i, key, &h, &isnull);
			rowbatch[i] = (uint16_t) b;
		}
		/* one shared-memory atomic per batch and warp: with a skewed key every row lands in the same counter */
		const unsigned peers = __match_any_sync(0xffffffffu, b);

		if (b >= 0 && (int) (threadIdx.x & 31) == __ffs(peers) - 1)
			atomicAdd(cnt + b, (uint32_t) __popc(peers));
	}
	__syncthreads();
	for (int b = threadIdx.x; b < p.ht.nbatch; b += blockDim.x)
		hist[(int64_t) b * gridDim.x + blockIdx.x] = cnt[b];
}

__global__ void __launch_bounds__(HT_PART_THREADS)
k_ht_partition_write(int64_t n, int32_t nbatch, int64_t chunk, const uint16_t *rowbatch, const unsigned long long *start,
					 unsigned long long *offsets, uint32_t *rows)
{
	extern __shared__ uint32_t cur[];	/* [nbatch] where the chunk's next row of each batch goes (row ids are 32 bits) */
	const int64_t lo = (int64_t) blockIdx.x * chunk;
	const int64_t hi = lo + chunk < n ? lo + chunk : n;
	const int	lane = threadIdx.x & 31,
				warp = threadIdx.x >> 5;

	for (int b = threadIdx.x; b < nbatch; b += blockDim.x)
		cur[b] = (uint32_t) start[(int64_t) b * gridDim.x + blockIdx.x];
	if (blockIdx.x == 0)
		for (int b = threadIdx.x; b <= nbatch; b += blockDim.x)
			offsets[b] = start[(int64_t) b * gridDim.x];	/* b == nbatch: the scan's total, n */
	__syncthreads();
	for (int64_t i0 = lo; i0 < hi; i0 += blockDim.x)
	{
		const int64_t i = i0 + threadIdx.x;
		const int32_t b = i < hi ? (int32_t) rowbatch[i] : -1;
		const unsigned peers = __match_any_sync(0xffffffffu, b);
		const uint32_t rank = __popc(peers & ((1u << lane) - 1));

		/* warp w's rows follow those of warps 0 .. w-1 of the same tile */
		for (int w = 0; w < (int) (blockDim.x >> 5); w++)
		{
			if (warp == w)
			{
				const uint32_t at = b >= 0 ? cur[b] : 0;

				__syncwarp();
				if (b >= 0)
				{
					rows[at + rank] = (uint32_t) i;
					if (rank == 0)
						cur[b] = at + (uint32_t) __popc(peers);
				}
			}
			__syncthreads();
		}
	}
}

/* the device and host buffers of a pair probe: allocated through `mem`, freed whatever the outcome */
struct PairProbe
{
	CbCallMem	mem;
	uint16_t   *rowbatch = NULL;	/* [n] each outer row's batch                                          */
	unsigned long long *hist = NULL;	/* [nbatch][partition CTAs] row counts, then their exclusive scan      */
	unsigned long long *d_offsets = NULL;	/* [nbatch + 1] where each batch's run starts in rows           */
	unsigned long long *h_offsets = NULL;
	uint32_t   *rows = NULL;		/* [n] outer row ids grouped by batch                                   */
	unsigned long long *counts = NULL;	/* match counts of one run (the last also of the build rows), then their scan */
	uint8_t    *matched = NULL;	/* RIGHT / FULL: [inner rows], kept across all passes                   */
	uint32_t   *decision = NULL;	/* SEMI / ANTI with a join filter: each row's decision in the current pass */
	CbpColumn  *fcols = NULL;	/* the join filter's columns and ops on the device                      */
	CbpOp	   *fops = NULL;
	uint32_t   *grow[2] = {};	/* the output's next, larger arrays while they are being filled (cudaMalloc: not in mem) */
	int64_t		cap = 0;		/* pairs the output arrays hold                                         */

	explicit	PairProbe(cbgpu_ctx *ctx) : mem(ctx) {}
};

/* the probe side's key columns of a pair probe */
static int
probe_params(cbgpu_ctx *ctx, const cbgpu_hashtable *ht, cbgpu_rel *outer, const int32_t *keycols, int32_t nkeys, ProbeParams *p)
{
	if (nkeys != ht->d.nkeys)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_ht_probe_pairs: key count mismatch%s %lld", "", nkeys);
	memset(p, 0, sizeof(*p));
	p->ht = ht->d;
	for (int k = 0; k < nkeys; k++)
	{
		int			c = keycols[k];

		if (c < 0 || c >= outer->ncols)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_ht_probe_pairs: bad key column%s %lld", "", c);
		p->okey[k] = outer->data[c];
		p->onulls[k] = outer->nulls[c];
		p->odict[k] = outer->dict_hash[c];
		p->otype[k] = outer->types[c];
	}
	return CBGPU_OK;
}

/* a join filter checked op by op (the stack depth it reaches, what it leaves), then copied to the device */
static int
join_filter_to_dev(cbgpu_ctx *ctx, const cbgpu_join_filter *jf, int32_t jointype, PairProbe *b, JoinFilterDev *f)
{
	XProg	   *x = (XProg *) cb_scratch(ctx, 2, sizeof(XProg));	/* the pipeline's slot: the two calls never overlap */
	const XAllow allow = {"join filter", XM_SCALAR_OPS, NULL, 0, CBGPU_ERR_INVALID};

	if (!x)
		return CBGPU_ERR_NOMEM;
	if (jf->ncols < 0 || jf->ncols > CBP_MAX_COLS || (jf->ncols > 0 && !jf->cols))
		return cb_fail(ctx, CBGPU_ERR_INVALID, "join filter with %s%lld columns (0 .. 40 expected)", "", jf->ncols);
	if (jf->nops < 1 || jf->nops > CBP_MAX_OPS || !jf->ops)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "join filter with %s%lld ops (1 .. 128 expected)", "", jf->nops);
	for (int k = 0; k < jf->ncols; k++)
	{
		const CbpColumn *c = &jf->cols[k];

		if (c->src != 0 && c->src != 1)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "join filter column %s%lld: src is neither 0 (probe side) nor 1 (build side)", "", k);
		if (c->type < CB_INT4 || c->type > CB_BOOL || !c->data)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "join filter column %s%lld: no data, or a type the filter cannot load", "", k);
	}
	int			rc = xm_walk(ctx, allow, jf->ncols, jf->ops, jf->nops, x);

	if (rc != CBGPU_OK)
		return rc;
	if (x->depth != 1)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "join filter leaves %s%lld values (one expected)", "", x->depth);
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	if (jf->ncols > 0)
	{
		CB_CUDA(ctx, b->mem.alloc(&b->fcols, sizeof(CbpColumn) * (size_t) jf->ncols));
		CB_CUDA(ctx, cudaMemcpyAsync(b->fcols, jf->cols, sizeof(CbpColumn) * (size_t) jf->ncols, cudaMemcpyHostToDevice, ctx->stream));
	}
	CB_CUDA(ctx, b->mem.alloc(&b->fops, sizeof(CbpOp) * (size_t) jf->nops));
	CB_CUDA(ctx, cudaMemcpyAsync(b->fops, jf->ops, sizeof(CbpOp) * (size_t) jf->nops, cudaMemcpyHostToDevice, ctx->stream));
	f->cols = b->fcols;
	f->ops = b->fops;
	f->nops = jf->nops;
	f->jointype = jointype;
	f->status = ctx->d_status;
	return CBGPU_OK;
}

/* one count (write = false) or write pass over p.n probe rows: the filtered kernel when the probe has a join filter */
static int
probe_pass(cbgpu_ctx *ctx, const ProbeParams &p, int blocks, bool write)
{
	if (p.f.ops && write)
	{
		k_ht_probe_filtered<true><<<blocks, 256, 0, ctx->stream>>>(p);
		CB_LAUNCHED(ctx, "k_ht_probe_filtered<write>");
	}
	else if (p.f.ops)
	{
		k_ht_probe_filtered<false><<<blocks, 256, 0, ctx->stream>>>(p);
		CB_LAUNCHED(ctx, "k_ht_probe_filtered<count>");
	}
	else if (write)
	{
		k_ht_probe_pairs<true><<<blocks, 256, 0, ctx->stream>>>(p);
		CB_LAUNCHED(ctx, "k_ht_probe_pairs<write>");
	}
	else
	{
		k_ht_probe_pairs<false><<<blocks, 256, 0, ctx->stream>>>(p);
		CB_LAUNCHED(ctx, "k_ht_probe_pairs<count>");
	}
	return CBGPU_OK;
}

/* room for `need` pairs in out, keeping the out->npairs written so far (capacity doubles: the copies stay linear) */
static int
pairs_reserve(cbgpu_ctx *ctx, PairProbe *b, cbgpu_pairs *out, int64_t need)
{
	const int64_t cap = b->cap * 2 > need ? b->cap * 2 : need;

	if (need <= b->cap)
		return CBGPU_OK;
	CB_CUDA(ctx, cudaMalloc(&b->grow[0], (size_t) cap * sizeof(uint32_t)));
	CB_CUDA(ctx, cudaMalloc(&b->grow[1], (size_t) cap * sizeof(uint32_t)));
	if (out->npairs)
	{
		CB_CUDA(ctx, cudaMemcpyAsync(b->grow[0], out->outer_idx, (size_t) out->npairs * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
		CB_CUDA(ctx, cudaMemcpyAsync(b->grow[1], out->inner_idx, (size_t) out->npairs * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
		CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	}
	if (out->outer_idx)
		cudaFree(out->outer_idx);
	if (out->inner_idx)
		cudaFree(out->inner_idx);
	out->outer_idx = b->grow[0];
	out->inner_idx = b->grow[1];
	b->grow[0] = b->grow[1] = NULL;
	b->cap = cap;
	return CBGPU_OK;
}

/* the pairs whose counts p.counts[0 .. nc) holds, appended to out: scan, one read-back, room, then `write` */
static int
pairs_append(cbgpu_ctx *ctx, PairProbe *b, ProbeParams *p, int64_t nc, cbgpu_pairs *out, bool *any)
{
	unsigned long long t = 0;

	k_exclusive_scan_u64<<<1, 1024, 0, ctx->stream>>>(p->counts, nc);
	CB_LAUNCHED(ctx, "k_exclusive_scan_u64");
	CB_CUDA(ctx, cudaMemcpyAsync(&t, p->counts + nc, sizeof(t), cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if ((unsigned long long) out->npairs + t > 0xFFFFFFF0ull)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "join result of %s%lld pairs exceeds the GPU path's 32-bit row ids", "",
					   (long long) (out->npairs + t));
	*any = t > 0;
	if (t == 0)
		return CBGPU_OK;
	int			rc = pairs_reserve(ctx, b, out, out->npairs + (int64_t) t);

	if (rc != CBGPU_OK)
		return rc;
	p->out_outer = out->outer_idx + out->npairs;
	p->out_inner = out->inner_idx + out->npairs;
	out->npairs += (int64_t) t;
	return CBGPU_OK;
}

/* HJ_NEED_NEW_BATCH (nodeHashjoin.c:709-738): each batch resident in turn, probed by its own run of outer rows.  A one-batch
 * table is one run of every outer row in relation order over the table as built: nothing is partitioned or reloaded.  The
 * last run also counts the build rows left unmatched (every count pass has marked its matches by then), so one scan and one
 * read-back serve both. */
static int
ht_probe_batches(cbgpu_ctx *ctx, cbgpu_hashtable *ht, ProbeParams p, int fill_inner, int (*interrupted)(void *arg), void *arg,
				 PairProbe *b, cbgpu_pairs *out, int64_t *passes)
{
	const int32_t nbatch = ht->d.nbatch;
	const int64_t n = p.n;
	const int64_t ninner = fill_inner ? ht->inner->nrows : 0;
	int64_t		maxrun = 0;
	int			iblocks = (int) ((ninner + 255) / 256);
	bool		any;
	int			rc;

	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	b->h_offsets = b->mem.keep((unsigned long long *) calloc((size_t) nbatch + 1, sizeof(unsigned long long)));
	if (!b->h_offsets)
		return cb_fail(ctx, CBGPU_ERR_NOMEM, "host memory for %s%lld batch offsets", "", nbatch);
	if (nbatch == 1)
		b->h_offsets[1] = (unsigned long long) n;
	else if (n > 0)
	{
		/* at most 2^18 [batch][CTA] counts: the scan over them runs on one CTA */
		int64_t		grid = (int64_t) ctx->sm_count * 2,
					chunk;
		const size_t shmem = (size_t) nbatch * sizeof(uint32_t);

		if (grid > (1 << 18) / nbatch)
			grid = (1 << 18) / nbatch;
		if (grid > (n + HT_PART_THREADS - 1) / HT_PART_THREADS)
			grid = (n + HT_PART_THREADS - 1) / HT_PART_THREADS;
		chunk = (n + grid - 1) / grid;
		CB_CUDA(ctx, b->mem.alloc(&b->rowbatch, (size_t) n * sizeof(uint16_t)));
		CB_CUDA(ctx, b->mem.alloc(&b->hist, ((size_t) nbatch * grid + 1) * sizeof(unsigned long long)));
		CB_CUDA(ctx, b->mem.alloc(&b->d_offsets, ((size_t) nbatch + 1) * sizeof(unsigned long long)));
		CB_CUDA(ctx, b->mem.alloc(&b->rows, (size_t) n * sizeof(uint32_t)));
		k_ht_partition_count<<<(int) grid, HT_PART_THREADS, shmem, ctx->stream>>>(p, chunk, b->rowbatch, b->hist);
		CB_LAUNCHED(ctx, "k_ht_partition_count");
		k_exclusive_scan_u64<<<1, 1024, 0, ctx->stream>>>(b->hist, nbatch * grid);
		CB_LAUNCHED(ctx, "k_exclusive_scan_u64");
		k_ht_partition_write<<<(int) grid, HT_PART_THREADS, shmem, ctx->stream>>>(n, nbatch, chunk, b->rowbatch, b->hist, b->d_offsets,
																				   b->rows);
		CB_LAUNCHED(ctx, "k_ht_partition_write");
		CB_CUDA(ctx, cudaMemcpyAsync(b->h_offsets, b->d_offsets, ((size_t) nbatch + 1) * sizeof(unsigned long long),
									 cudaMemcpyDeviceToHost, ctx->stream));
		CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	}
	for (int32_t k = 0; k < nbatch; k++)
		if ((int64_t) (b->h_offsets[k + 1] - b->h_offsets[k]) > maxrun)
			maxrun = (int64_t) (b->h_offsets[k + 1] - b->h_offsets[k]);
	CB_CUDA(ctx, b->mem.alloc(&b->counts, (size_t) (maxrun + ninner + 1) * sizeof(unsigned long long)));
	p.counts = b->counts;
	if (p.f.ops && p.f.jointype != CB_JOIN_LEFT && maxrun)
	{
		CB_CUDA(ctx, b->mem.alloc(&b->decision, (size_t) maxrun * sizeof(uint32_t)));
		p.f.decision = b->decision;
	}
	if (ninner)
	{
		CB_CUDA(ctx, b->mem.alloc(&b->matched, (size_t) ninner));
		CB_CUDA(ctx, cudaMemsetAsync(b->matched, 0, (size_t) ninner, ctx->stream));
		p.matched = b->matched;
	}
	if (iblocks > ctx->sm_count * 8)
		iblocks = ctx->sm_count * 8;
	for (int32_t batch = 0; batch < nbatch; batch++)
	{
		const int64_t m = (int64_t) (b->h_offsets[batch + 1] - b->h_offsets[batch]);
		const int64_t nu = batch == nbatch - 1 ? ninner : 0;	/* build rows whose pairs follow this run's */
		int			blocks = (int) ((m + 255) / 256);

		if (nbatch > 1)
		{
			if (interrupted && interrupted(arg))
				return cb_fail(ctx, CBGPU_ERR_INTERRUPTED, "canceling statement due to user request%s", "");
			if ((rc = cbgpu_ht_load_batch(ht, batch)) != CBGPU_OK)
				return rc;
			(*passes)++;
			p.ht = ht->d;
			p.sel = b->rows + b->h_offsets[batch];
		}
		if (m + nu == 0)
			continue;
		if (blocks > ctx->sm_count * 8)
			blocks = ctx->sm_count * 8;
		p.n = m;
		p.ninner = nu;
		if (m && (rc = probe_pass(ctx, p, blocks, false)) != CBGPU_OK)
			return rc;
		if (nu)
		{
			k_ht_unmatched_count<<<iblocks, 256, 0, ctx->stream>>>(p);
			CB_LAUNCHED(ctx, "k_ht_unmatched_count");
		}
		if ((rc = pairs_append(ctx, b, &p, m + nu, out, &any)) != CBGPU_OK)
			return rc;
		if (any && m && (rc = probe_pass(ctx, p, blocks, true)) != CBGPU_OK)
			return rc;
		if (any && nu)
		{
			k_ht_unmatched_write<<<iblocks, 256, 0, ctx->stream>>>(p);
			CB_LAUNCHED(ctx, "k_ht_unmatched_write");
		}
	}
	return CBGPU_OK;
}

extern "C" int
cbgpu_ht_probe_pairs(cbgpu_ctx *ctx, cbgpu_hashtable *ht, cbgpu_rel *outer, const int32_t *keycols, int32_t nkeys, int32_t jointype,
					 const cbgpu_join_filter *filter, int (*interrupted)(void *arg), void *arg, cbgpu_pairs *out, int64_t *passes)
{
	const bool	taken = filter ? jointype == CB_JOIN_LEFT || jointype == CB_JOIN_SEMI || jointype == CB_JOIN_ANTI
		: jointype == CB_JOIN_INNER || jointype == CB_JOIN_LEFT || jointype == CB_JOIN_RIGHT || jointype == CB_JOIN_FULL;
	PairProbe	b(ctx);
	ProbeParams p;
	int64_t		npasses = 0;
	int			rc;

	memset(out, 0, sizeof(*out));
	if (!taken)
		rc = cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_ht_probe_pairs: join type %s%lld (INNER, LEFT, RIGHT or FULL without a join "
					 "filter, LEFT, SEMI or ANTI with one)", "", jointype);
	else
		rc = probe_params(ctx, ht, outer, keycols, nkeys, &p);
	if (rc == CBGPU_OK && filter)
		rc = join_filter_to_dev(ctx, filter, jointype, &b, &p.f);
	if (rc == CBGPU_OK)
	{
		p.n = outer->nrows;
		p.left = jointype == CB_JOIN_LEFT || jointype == CB_JOIN_FULL;
		rc = ht_probe_batches(ctx, ht, p, jointype == CB_JOIN_RIGHT || jointype == CB_JOIN_FULL, interrupted, arg, &b, out, &npasses);
	}
	if (rc == CBGPU_OK && filter)
		rc = cb_check_status(ctx, "join filter");	/* integer overflow inside the filter */
	if (passes)
		*passes = npasses;
	for (int k = 0; k < 2; k++)
		if (b.grow[k])
			cudaFree(b.grow[k]);
	if (rc != CBGPU_OK)
		cbgpu_pairs_free(out);
	return rc;
}

extern "C" void
cbgpu_pairs_free(cbgpu_pairs *p)
{
	if (!p)
		return;
	if (p->outer_idx)
		cudaFree(p->outer_idx);
	if (p->inner_idx)
		cudaFree(p->inner_idx);
	p->outer_idx = p->inner_idx = NULL;
	p->npairs = 0;
}
