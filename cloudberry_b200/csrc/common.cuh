/*
 * common.cuh - shared internals of libcbgpu.so: context / relation structs, error plumbing, the
 * reference's hash functions as device code, and the 128-bit accumulate primitives.
 *
 * Hashing must be bit-exact with the reference (parity gate): each device function cites the
 * reference function it restates (paths under /root/reference/src).
 */
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/cbgpu.h"

#include <stdlib.h>
#include <string.h>

#include <memory>

#define CB_MAX_COLS_REL 64

struct cbgpu_ctx
{
	int			device;
	cudaStream_t stream;
	char		err[512];
	int			sm_count;
	int64_t		launches;
	cudaEvent_t ev_t0, ev_t1, ev_k0, ev_k1;
	double		last_kernel_ms;
	const char *last_kernel_name;
	bool		kernel_timed;
	/* log of the pipeline kernels since cbgpu_kernel_log_reset(): own event pair per entry */
#define CB_KLOG 32
	cudaEvent_t klog_ev[CB_KLOG][2];
	const char *klog_name[CB_KLOG];
	int			klog_n;
	bool		klog_ready;
	/* launch trace (cbgpu_trace_begin): one event after every kernel launch */
#define CB_TRACE 1024
	bool		trace_on;
	int			trace_n;
	cudaEvent_t *trace_ev;		/* CB_TRACE + 1 events, created on first use                         */
	const char *trace_name[CB_TRACE];
	void	   *flush_buf;
	size_t		flush_bytes;
	int		   *d_status;		/* device status word: nonzero = CBGPU error code raised by a kernel */
	int		   *h_status;		/* pinned mirror                                                      */
	int64_t		status_seen_at;	/* ctx->launches when h_status was last fetched (-1: never): every
								 * synchronising read-back fetches the status word too, so the check
								 * after it costs no second round trip                                 */
	/* environment knobs (DESIGN.md 9), read ONCE when the context is created - not per launch */
	bool		opt_debug, opt_pf_spec;
	int			opt_bloom_div;
	/* host-side scratch of the launch path (decompiled programs, kernel parameter blocks: too large for the
	 * stack), owned by the context so that two contexts on two threads never share any: slot -> malloc'ed block */
#define CB_SCRATCH_SLOTS 6
	void	   *scratch[CB_SCRATCH_SLOTS];
	size_t		scratch_bytes[CB_SCRATCH_SLOTS];
	/* scan-level runtime filter decisions, remembered per (build relation, rows, key column): the sample that
	 * decides "worth building" costs a host round trip, the answer does not change while the table does not */
#define CB_EARLY_CACHE 16
	struct
	{
		const void *keydata;
		int64_t		nrows;
		const void *red0;
		int			worth;
	}			early_cache[CB_EARLY_CACHE];
	int			early_cache_n;
	/* pinned (mapped) host buffer small aggregate tables are snapshotted into by the kernel that finishes them: group count,
	 * flags and the groups themselves arrive with ONE synchronisation (struct AggSnap, below) */
	/* pipelines whose prefilter pass cut too little (k_prefilter, probe_chain.cu): not tried again */
	uint64_t	pf_cache[32];
	int			pf_cache_n;
	int			opt_pf_keep_div;	/* the prefilter's result is used when survivors * this <= rows (CBGPU_PREFILTER_KEEP_DIV, 12) */
	int64_t		opt_pf_min_rows;	/* scans below this many rows stay in the fused kernel (CBGPU_PREFILTER_MIN_ROWS)        */
	struct AggSnap *agg_snap;
	void	   *small_dev;		/* device scratch of the small-group scan kernel, grown on demand              */
	size_t		small_dev_bytes;
};

/* zero-filled scratch block `slot` of at least `bytes` (grown on demand, freed with the context) */
static inline void *
cb_scratch(cbgpu_ctx *ctx, int slot, size_t bytes)
{
	if (ctx->scratch_bytes[slot] < bytes)
	{
		free(ctx->scratch[slot]);
		ctx->scratch[slot] = malloc(bytes);
		ctx->scratch_bytes[slot] = ctx->scratch[slot] ? bytes : 0;
	}
	if (ctx->scratch[slot])
		memset(ctx->scratch[slot], 0, bytes);
	return ctx->scratch[slot];
}

struct cbgpu_rel
{
	cbgpu_ctx  *ctx;
	int64_t		nrows;
	int64_t		capacity;
	int32_t		ncols;
	int32_t		types[CB_MAX_COLS_REL];
	int32_t		dscales[CB_MAX_COLS_REL];
	void	   *data[CB_MAX_COLS_REL];
	uint8_t	   *nulls[CB_MAX_COLS_REL];
	uint32_t   *dict_hash[CB_MAX_COLS_REL];
	int32_t		dict_n[CB_MAX_COLS_REL];
	uint8_t	   *visimap;
	bool		owns[CB_MAX_COLS_REL];
	void	   *slab;			/* small relations: the one allocation all columns live in (owns[] = false) */
	const cbgpu_dict *dict[CB_MAX_COLS_REL];	/* borrowed (cbgpu_rel_set_dict), NULL: none       */
	int32_t		dict_bpchar_len[CB_MAX_COLS_REL];
};

/* agg table, device view (struct of arrays; open addressing, linear probing) */
struct AggDev
{
	uint32_t	mask;			/* capacity - 1                                                       */
	int32_t		nkeys;
	int32_t		naccs;
	/* partitioned aggregation (the reference's spill-and-reload of over-budget hash aggregation, nodeAgg.c:2149
	 * hash_agg_check_limits, :3215 agg_refill_hash_table, done by re-scanning instead of spilling): a pass aggregates only the
	 * rows whose group hash has part_id in its top bits; npart <= 1: off */
	int32_t		npart;
	int32_t		part_shift;
	int32_t		part_id;
	int32_t    *state;			/* [cap] 0 empty, 1 being written, 2 ready                            */
	uint32_t   *hash;			/* [cap]                                                              */
	int64_t    *keys;			/* [cap][nkeys]                                                       */
	uint32_t   *keynull;		/* [cap] bit k = key k is NULL                                        */
	int64_t    *n;				/* [cap][naccs]                                                       */
	unsigned long long *sum;	/* [cap][naccs][2] lo, hi (float8 state: bits in lo)                  */
	int32_t    *ngroups;
	int32_t    *full;			/* set when an insert found no free slot                              */
};

/* what a finishing kernel leaves in pinned host memory for tables of at most AGG_SNAP_MAXCAP slots and AGG_SNAP_MAXG
 * groups: everything agg_retrieve_hash_table (nodeAgg.c:2952) would walk the table for */
#define AGG_SNAP_MAXG 64
#define AGG_SNAP_MAXCAP 4096
struct AggSnap
{
	int32_t		ngroups;		/* -1: not taken (retry / audit flags say why)                        */
	int32_t		full;
	int32_t		anynull;
	int32_t		retry;
	int32_t		audit;
	int32_t		pad[3];
	uint32_t	keynull[AGG_SNAP_MAXG];
	int64_t		keys[AGG_SNAP_MAXG][CBP_MAX_GROUP_KEYS];
	int64_t		n[AGG_SNAP_MAXG][CBP_MAX_AGGS];
	int64_t		lo[AGG_SNAP_MAXG][CBP_MAX_AGGS];
	int64_t		hi[AGG_SNAP_MAXG][CBP_MAX_AGGS];
};

struct cbgpu_aggtable
{
	cbgpu_ctx  *ctx;
	AggDev		d;
	void	   *base;			/* the one device allocation all of d's arrays live in                */
	int64_t		capacity;
	int32_t		kinds[CBP_MAX_AGGS];
	/* group count / "some group key is NULL", valid until the table is written again */
	bool		counted;
	int64_t		ngroups;
	int32_t		anynull;
	/* the groups themselves, when a snapshot brought them along (cb_agg_adopt_snapshot) */
	bool		snap_valid;
	AggSnap    *snap;			/* host copy, allocated on first use                                  */
};

#ifdef __CUDACC__
/* one CTA walks a small table and writes the snapshot (call with all threads of the block, after the block's own
 * updates of the table are ordered by __syncthreads) */
__device__ __forceinline__ void
agg_snapshot_block(const AggDev &t, AggSnap *out)
{
	__shared__ int s_n,
				s_an;
	const size_t cap = (size_t) t.mask + 1;

	if (threadIdx.x == 0)
	{
		s_n = 0;
		s_an = 0;
	}
	__syncthreads();
	for (size_t i = threadIdx.x; i < cap; i += blockDim.x)
	{
		if (((volatile int32_t *) t.state)[i] != 2)
			continue;
		const int	g = atomicAdd(&s_n, 1);

		if (t.keynull[i])
			s_an = 1;
		if (g >= AGG_SNAP_MAXG)
			continue;
		out->keynull[g] = t.keynull[i];
		for (int k = 0; k < t.nkeys; k++)
			out->keys[g][k] = t.keys[i * t.nkeys + k];
		for (int a = 0; a < t.naccs; a++)
		{
			out->n[g][a] = ((volatile int64_t *) t.n)[i * t.naccs + a];
			out->lo[g][a] = (int64_t) ((volatile unsigned long long *) t.sum)[(i * t.naccs + a) * 2];
			out->hi[g][a] = (int64_t) ((volatile unsigned long long *) t.sum)[(i * t.naccs + a) * 2 + 1];
		}
	}
	__syncthreads();
	if (threadIdx.x == 0)
	{
		out->full = *(volatile int32_t *) t.full;
		out->anynull = s_an;
		out->ngroups = s_n;
	}
	__threadfence_system();
}
#endif
void		cb_agg_adopt_snapshot(cbgpu_aggtable *t, const AggSnap *snap);


#define CB_HD __host__ __device__ __forceinline__

/* join hash table, device view.  The slot format is owned by the ht_slot_* / ht_probe_tag / ht_tag_match helpers below and
 * ht_slot_match / ht_find further down: every build and probe goes through them. */
#define HT_EMPTY 0xFFFFFFFFFFFFFFFFull
struct HtDev
{
	unsigned long long *slots;
	uint32_t	mask;
	/* blocked Bloom filter over the build keys' hash values: 2 bits in one 32-bit word, ~16 bits per
	 * key, small enough to stay L2-resident.  A probe that fails it skips the table (DRAM) access:
	 * the reference's runtime filter (PassByBloomFilter, executor/nodeSeqscan.c:413; built from the
	 * build side in executor/nodeHash.c:4321-4432, lib/bloomfilter.c) applied at the probe. */
	uint32_t   *bloom;
	uint32_t	bloom_mask;
	int32_t		nkeys;
	const void *keydata[CBP_MAX_KEYS];	/* inner key columns, for match verification                  */
	const uint8_t *keynulls[CBP_MAX_KEYS];
	const uint32_t *keydict[CBP_MAX_KEYS];
	int32_t		keytype[CBP_MAX_KEYS];
	/* key-in-slot tables: one integer key whose every build value fits 32 bits is stored IN the slot's upper
	 * word instead of the hash value (slot = key32 << 32 | rowid32), so a probe settles a match on the slot
	 * alone - no second random access to the build side's key column.  1: the int32 domain (int4 / date /
	 * dictionary codes, and int8 keys between INT32_MIN and INT32_MAX are not used: see 2), 2: the uint32 domain
	 * (int8 keys in [0, 2^32): TPC-H order keys up to SF 1000).  0: hash in the slot, key verified by row id. */
	int32_t		keyslot;
	/* multi-batch hybrid hash join (nodeHash.c:980-990 nbatch, :2223-2242 ExecHashGetBucketAndBatch: the batch number
	 * comes from hash bits the bucket number does not use): the table holds ONE batch of the build side at a time - the
	 * rows whose (hash >> batch_shift) == batch_id - and a probe row of another batch is not this pass's business
	 * (it is neither matched nor, for outer / anti joins, emitted unmatched: its own pass does that).  nbatch <= 1: off. */
	int32_t		nbatch;
	int32_t		batch_shift;
	int32_t		batch_id;
};

CB_HD bool
ht_in_batch(int32_t nbatch, int32_t batch_shift, int32_t batch_id, uint32_t hash)
{
	return nbatch <= 1 || (int32_t) (hash >> batch_shift) == batch_id;
}

/* is an outer key value inside a key-in-slot table's domain?  Outside it nothing can match. */
CB_HD bool
ht_key_in_domain(int32_t keyslot, int64_t key)
{
	return keyslot == 1 ? key == (int64_t) (int32_t) key : (uint64_t) key <= 0xFFFFFFFFull;
}

/* A slot is tag32 << 32 | row32, HT_EMPTY = ~0, probed linearly from hash & mask.  The tag is the key itself in a key-in-slot
 * table (keyslot 1 or 2: a tag match is a key match, given ht_key_in_domain), and the key hash otherwise (a tag match is
 * confirmed by the build row's key columns).  The build side tags its rows with the same function a probe compares with. */
CB_HD uint32_t
ht_probe_tag(int32_t keyslot, uint32_t hash, int64_t key0)
{
	return keyslot ? (uint32_t) key0 : hash;
}

CB_HD unsigned long long
ht_slot_entry(uint32_t tag, uint32_t row)
{
	return ((unsigned long long) tag << 32) | row;
}

CB_HD bool
ht_slot_empty(unsigned long long e)
{
	return e == HT_EMPTY;
}

CB_HD uint32_t
ht_slot_row(unsigned long long e)
{
	return (uint32_t) e;
}

CB_HD bool
ht_tag_match(unsigned long long e, uint32_t tag)
{
	return (uint32_t) (e >> 32) == tag;
}

struct cbgpu_hashtable
{
	cbgpu_ctx  *ctx;
	HtDev		d;
	cbgpu_rel  *inner;
	int64_t		nslots;
	int64_t		ninserted;
	int		   *d_flags;		/* [0] duplicates seen, [1] inserted count                            */
	int			has_dups;
	int64_t		total_rows;		/* multi-batch: rows of all batches                                   */
	int64_t		built_bytes;	/* slots + filter of what is resident                                 */
};

/* ---------------------------------------------------------------------------------------------
 * error plumbing
 * --------------------------------------------------------------------------------------------- */
static inline int
cb_fail(cbgpu_ctx *ctx, int code, const char *fmt, const char *a = "", long long b = 0)
{
	if (ctx)
		snprintf(ctx->err, sizeof(ctx->err), fmt, a, b);
	return code;
}

#define CB_CUDA(ctx, call) \
	do { \
		cudaError_t e__ = (call); \
		if (e__ != cudaSuccess) \
		{ \
			if (ctx) \
				snprintf((ctx)->err, sizeof((ctx)->err), "%s:%d: %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
			(void) cudaGetLastError();	/* not sticky: do not let the next launch check trip over it */ \
			/* the device is full: a limit of this path (inputs must fit HBM), reported as such so that a caller can leave the \
			 * sub-tree to the CPU executor (cb_exec.c, cb_cluster_init_plan) instead of treating it as a broken device */ \
			return e__ == cudaErrorMemoryAllocation ? CBGPU_ERR_NOMEM : CBGPU_ERR_CUDA; \
		} \
	} while (0)

/* kernel launch bookkeeping (every kernel of ours goes through this) */
void		cb_trace_mark(cbgpu_ctx *ctx, const char *name);
#define CB_LAUNCHED(ctx, name) \
	do { \
		(ctx)->launches++; \
		if ((ctx)->trace_on) \
			cb_trace_mark(ctx, name); \
		cudaError_t e__ = cudaGetLastError(); \
		if (e__ != cudaSuccess) \
		{ \
			snprintf((ctx)->err, sizeof((ctx)->err), "launch %s: %s", name, cudaGetErrorString(e__)); \
			return CBGPU_ERR_CUDA; \
		} \
	} while (0)

/* a constructor's object until it is handed out: CB_CUDA and CB_LAUNCHED return from the middle of a function, and on
 * any early return the object goes through its own free function (which skips members never allocated) */
template <typename T> using CbOwned = std::unique_ptr<T, void (*)(T *)>;

/* the buffers one call allocates for its own duration: device buffers (stream-ordered on ctx->stream) and malloc'ed host
 * buffers, freed when the call returns by whichever exit.  copy_in queues a copy from host memory; until sync() has
 * waited for it, the destructor drains the stream first, so that the caller may free that memory once the call returns
 * and the call's own host buffers are not freed under the copy.  A free that fails here is ignored: the call's error
 * stands. */
struct CbCallMem
{
	cbgpu_ctx  *ctx;
	void	   *dev[16] = {};
	void	   *host[4] = {};
	int			ndev = 0,
				nhost = 0;
	bool		in_flight = false;

	explicit	CbCallMem(cbgpu_ctx *c) : ctx(c) {}
	CbCallMem(const CbCallMem &) = delete;
	CbCallMem &operator=(const CbCallMem &) = delete;

	~CbCallMem()
	{
		if (in_flight)
			(void) cudaStreamSynchronize(ctx->stream);
		for (int i = 0; i < ndev; i++)
			if (dev[i] && cudaFreeAsync(dev[i], ctx->stream) != cudaSuccess)
				(void) cudaGetLastError();
		for (int i = 0; i < nhost; i++)
			::free(host[i]);
	}

	template <typename T> cudaError_t
	alloc(T **p, size_t bytes)
	{
		if (ndev == (int) (sizeof(dev) / sizeof(dev[0])))
			return cudaErrorInvalidValue;
		cudaError_t e = cudaMallocAsync((void **) p, bytes, ctx->stream);

		if (e == cudaSuccess)
			dev[ndev++] = *p;
		return e;
	}

	/* a buffer freed before the call ends: where it frees today, so that peak memory stays as it is */
	cudaError_t
	free(void *p)
	{
		return cudaFreeAsync(detach(p), ctx->stream);
	}

	/* a buffer handed to the caller: no longer freed here */
	template <typename T> T *
	detach(T *p)
	{
		for (int i = 0; i < ndev; i++)
			if (dev[i] == p)
				dev[i] = NULL;
		return p;
	}

	/* a malloc'ed host buffer (NULL when malloc failed), freed when the call returns */
	template <typename T> T *
	keep(T *p)
	{
		if (nhost == (int) (sizeof(host) / sizeof(host[0])))
		{
			::free(p);
			return NULL;
		}
		return (T *) (host[nhost++] = p);
	}

	cudaError_t
	copy_in(void *dst, const void *src, size_t bytes)
	{
		in_flight = true;
		return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream);
	}

	cudaError_t
	sync(void)
	{
		cudaError_t e = cudaStreamSynchronize(ctx->stream);

		if (e == cudaSuccess)
			in_flight = false;
		return e;
	}
};

int			cb_check_status(cbgpu_ctx *ctx, const char *what);	/* sync + read device status word */
/* enqueue the status word's copy next to another device-to-host copy; call cb_status_fetched after the sync */
#define CB_STATUS_RIDE(ctx) cudaMemcpyAsync((ctx)->h_status, (ctx)->d_status, sizeof(int), cudaMemcpyDeviceToHost, (ctx)->stream)
#define CB_STATUS_FETCHED(ctx) ((ctx)->status_seen_at = (ctx)->launches)

static inline int
cb_type_w(int t)
{
	return cb_type_width((CbTypeId) t);
}

/* ---------------------------------------------------------------------------------------------
 * the reference's hash functions, device + host
 * --------------------------------------------------------------------------------------------- */

CB_HD uint32_t
pg_rot(uint32_t x, int k)
{
	return (x << k) | (x >> (32 - k));
}

/* final() of common/hashfn.c:133-142 */
#define PG_FINAL(a, b, c) \
	do { \
		c ^= b; c -= pg_rot(b, 14); \
		a ^= c; a -= pg_rot(c, 11); \
		b ^= a; b -= pg_rot(a, 25); \
		c ^= b; c -= pg_rot(b, 16); \
		a ^= c; a -= pg_rot(c, 4); \
		b ^= a; b -= pg_rot(a, 14); \
		c ^= b; c -= pg_rot(b, 24); \
	} while (0)

/* mix() of common/hashfn.c:99-107 */
#define PG_MIX(a, b, c) \
	do { \
		a -= c; a ^= pg_rot(c, 4); c += b; \
		b -= a; b ^= pg_rot(a, 6); a += c; \
		c -= b; c ^= pg_rot(b, 8); b += a; \
		a -= c; a ^= pg_rot(c, 16); c += b; \
		b -= a; b ^= pg_rot(a, 19); a += c; \
		c -= b; c ^= pg_rot(b, 4); b += a; \
	} while (0)

/* hash_bytes_uint32 (common/hashfn.c:627-640) = hashint4 (access/hash/hashfunc.c:72); dates hash
 * as int4 (catalog/pg_amproc.dat:310) */
CB_HD uint32_t
pg_hash_uint32(uint32_t k)
{
	uint32_t	a, b, c;

	a = b = c = 0x9e3779b9u + (uint32_t) sizeof(uint32_t) + 3923095u;
	a += k;
	PG_FINAL(a, b, c);
	return c;
}

/* hashint8 (access/hash/hashfunc.c:84-102) */
CB_HD uint32_t
pg_hashint8(int64_t val)
{
	uint32_t	lohalf = (uint32_t) val;
	uint32_t	hihalf = (uint32_t) ((uint64_t) val >> 32);

	lohalf ^= (val >= 0) ? hihalf : ~hihalf;
	return pg_hash_uint32(lohalf);
}

/* hash_bytes (common/hashfn.c:146-360) over exactly 8 bytes given as two little-endian words */
CB_HD uint32_t
pg_hash_bytes8(uint32_t w0, uint32_t w1)
{
	uint32_t	a, b, c;

	a = b = c = 0x9e3779b9u + 8u + 3923095u;
	b += w1;
	a += w0;
	PG_FINAL(a, b, c);
	return c;
}

/* hash_bytes over 0 or 1 byte: hashbpchar of a character(1) value (utils/adt/varchar.c:981-1004,
 * bcTruelen strips a trailing blank so ' ' hashes zero bytes) */
CB_HD uint32_t
pg_hash_bpchar1(uint8_t ch)
{
	uint32_t	a, b, c;
	uint32_t	len = (ch == (uint8_t) ' ') ? 0u : 1u;

	a = b = c = 0x9e3779b9u + len + 3923095u;
	if (len)
		a += ch;
	PG_FINAL(a, b, c);
	return c;
}

/* hashfloat8 (access/hash/hashfunc.c:194-216) */
CB_HD uint32_t
pg_hashfloat8(uint64_t bits)
{
	if ((bits << 1) == 0)
		return 0;				/* +0 and -0 */
	if (((bits >> 52) & 0x7ff) == 0x7ff && (bits & 0xfffffffffffffull) != 0)
		bits = 0x7ff8000000000000ull;	/* get_float8_nan() */
	return pg_hash_bytes8((uint32_t) bits, (uint32_t) (bits >> 32));
}

/* general hash_bytes for the host side (dictionary strings) */
static inline uint32_t
pg_hash_bytes_host(const unsigned char *k, int keylen)
{
	uint32_t	a, b, c;
	int			len = keylen;

	a = b = c = 0x9e3779b9u + (uint32_t) len + 3923095u;
	while (len >= 12)
	{
		a += (k[0] + ((uint32_t) k[1] << 8) + ((uint32_t) k[2] << 16) + ((uint32_t) k[3] << 24));
		b += (k[4] + ((uint32_t) k[5] << 8) + ((uint32_t) k[6] << 16) + ((uint32_t) k[7] << 24));
		c += (k[8] + ((uint32_t) k[9] << 8) + ((uint32_t) k[10] << 16) + ((uint32_t) k[11] << 24));
		PG_MIX(a, b, c);
		k += 12;
		len -= 12;
	}
	switch (len)
	{
		case 11: c += ((uint32_t) k[10] << 24);
		case 10: c += ((uint32_t) k[9] << 16);
		case 9:  c += ((uint32_t) k[8] << 8);
		case 8:  b += ((uint32_t) k[7] << 24);
		case 7:  b += ((uint32_t) k[6] << 16);
		case 6:  b += ((uint32_t) k[5] << 8);
		case 5:  b += k[4];
		case 4:  a += ((uint32_t) k[3] << 24);
		case 3:  a += ((uint32_t) k[2] << 16);
		case 2:  a += ((uint32_t) k[1] << 8);
		case 1:  a += k[0];
	}
	PG_FINAL(a, b, c);
	return c;
}

/* murmurhash32 (include/common/hashfn.h:93-103): finaliser of TupleHashTableHash_internal
 * (executor/execGrouping.c:495) */
CB_HD uint32_t
pg_murmurhash32(uint32_t h)
{
	h ^= h >> 16;
	h *= 0x85ebca6bu;
	h ^= h >> 13;
	h *= 0xc2b2ae35u;
	h ^= h >> 16;
	return h;
}

/* per-key combine: rotate left 1 then XOR (NULL contributes nothing): executor/nodeHash.c:2134,
 * executor/execGrouping.c:474, cdb/cdbhash.c:196 */
CB_HD uint32_t
pg_hash_combine(uint32_t acc, uint32_t h, bool isnull)
{
	acc = (acc << 1) | (acc >> 31);
	return isnull ? acc : (acc ^ h);
}

/* jump_consistent_hash (cdb/cdbhash.c:530-541).  The double-precision divide and the
 * int64 * double product must round as on the host: plain IEEE ops, no fma contraction. */
CB_HD int32_t
pg_jump_consistent_hash(uint64_t key, int32_t num_segments)
{
	int64_t		b = -1;
	int64_t		j = 0;

	while (j < num_segments)
	{
		b = j;
		key = key * 2862933555777941757ULL + 1;
#ifdef __CUDA_ARCH__
		double		q = __ddiv_rn((double) (1LL << 31), (double) ((key >> 33) + 1));

		j = (int64_t) __dmul_rn((double) (b + 1), q);
#else
		double		q = (double) (1LL << 31) / (double) ((key >> 33) + 1);

		j = (int64_t) ((double) (b + 1) * q);
#endif
	}
	return (int32_t) b;
}

/* hash function of one key datum by type (pg_amproc: hashint4, hashint8, hashfloat8, hashbpchar,
 * hashchar for bool) on the 64-bit widened value; a dictionary code's hash is its entry of the per-code table */
CB_HD uint32_t
pg_hash_datum(int type, int64_t v, const uint32_t *dict)
{
	switch (type)
	{
		case CB_INT4: case CB_DATE:
			return pg_hash_uint32((uint32_t) (int32_t) v);
		case CB_INT8:
			return pg_hashint8(v);
		case CB_FLOAT8:
			return pg_hashfloat8((uint64_t) v);
		case CB_BPCHAR1:
			return pg_hash_bpchar1((uint8_t) v);
		case CB_DICT8: case CB_DICT32:
#ifdef __CUDA_ARCH__
			return dict ? __ldg(dict + v) : 0u;
#else
			return dict ? dict[v] : 0u;
#endif
		case CB_BOOL:
			return pg_hash_uint32((uint32_t) (int32_t) (int8_t) v);
		default:
			return 0u;
	}
}

/* The hash compositions whose values are observable, written once for every sink (DESIGN §2).  Key k has type types[k],
 * per-code hash table dicts[k] and value keys[k]; bit k of knull marks it NULL.  pg_hash_keys is the rotate-xor over the
 * keys that the group hash and cdbhash share (a NULL contributes nothing). */
CB_HD uint32_t
pg_hash_keys(int nkeys, const int32_t *types, const uint32_t *const *dicts, const int64_t *keys, uint32_t knull)
{
	uint32_t	h = 0;

	for (int k = 0; k < nkeys; k++)
	{
		const bool	isn = (knull >> k) & 1;

		h = pg_hash_combine(h, isn ? 0u : pg_hash_datum(types[k], keys[k], dicts[k]), isn);
	}
	return h;
}

/* float8eq groups -0 with +0 and all NaNs together (hashfloat8 gives them one hash value, hashfunc.c:194-216); the
 * aggregate table compares key bits, so a group key is made canonical first */
CB_HD int64_t
agg_group_key(int type, int64_t v)
{
	if (type == CB_FLOAT8 && ((uint64_t) v << 1) == 0)
		return 0;
	if (type == CB_FLOAT8 && ((v >> 52) & 0x7ff) == 0x7ff && (v & 0xfffffffffffffll) != 0)
		return 0x7FF8000000000000ll;
	return v;
}

/* TupleHashTableHash_internal (executor/execGrouping.c:437-495): hash_iv 0, rotate-xor per key, then murmurhash32 */
CB_HD uint32_t
agg_group_hash(int nkeys, const int32_t *types, const uint32_t *const *dicts, const int64_t *keys, uint32_t knull)
{
	return pg_murmurhash32(pg_hash_keys(nkeys, types, dicts, keys, knull));
}

/* the Motion's destination of a row: cdbhashinit / cdbhash / cdbhashreduce (cdb/cdbhash.c:171,189,253) */
CB_HD int32_t
cdb_route(int nkeys, const int32_t *types, const uint32_t *const *dicts, const int64_t *keys, uint32_t knull, int32_t nsegs)
{
	return pg_jump_consistent_hash(pg_hash_keys(nkeys, types, dicts, keys, knull), nsegs);
}

/* int8pl / int8mi / int8mul (utils/adt/int8.c) raise "bigint out of range"; the kernels refuse such a row, and scaled
 * numerics share the check (a product that leaves 64 bits is refused, never wrapped).  Each returns the wrapped result
 * and sets *ovf when the exact one does not fit. */
CB_HD int64_t
i64_add_ovf(int64_t x, int64_t y, bool *ovf)
{
	const int64_t r = (int64_t) ((uint64_t) x + (uint64_t) y);

	*ovf = ((x ^ r) & (y ^ r)) < 0;
	return r;
}

CB_HD int64_t
i64_sub_ovf(int64_t x, int64_t y, bool *ovf)
{
	const int64_t r = (int64_t) ((uint64_t) x - (uint64_t) y);

	*ovf = ((x ^ y) & (x ^ r)) < 0;
	return r;
}

CB_HD int64_t
i64_mul_ovf(int64_t x, int64_t y, bool *ovf)
{
	const int64_t r = (int64_t) ((uint64_t) x * (uint64_t) y);

#ifdef __CUDA_ARCH__
	*ovf = __mul64hi(x, y) != (r >> 63);
#else
	*ovf = (int64_t) (((__int128) x * y) >> 64) != (r >> 63);
#endif
	return r;
}

/* ---------------------------------------------------------------------------------------------
 * hash of a join key for the device's OWN structures: join hash tables, their Bloom filters, the scan-level
 * runtime filters.  Which slot a key lands in is not observable from outside (the reference's bucket number,
 * nodeHash.c:2233, is not either), so these do not pay for the reference's lookup3 mix (hash_bytes_uint32,
 * common/hashfn.c:627: ~22 dependent integer operations, a quarter of the join pipeline's instructions when
 * measured): a two-multiply finaliser instead.  Everything observable keeps the reference's functions bit
 * for bit - Motion placement (cdbhash, pg_hash_datum above) and the group hash (TupleHashTableHash).
 * int8 keys fold their halves the way hashint8 does, so an int4 key and an int8 key of equal value still meet
 * (cross-type joins).
 * --------------------------------------------------------------------------------------------- */
CB_HD uint32_t
jh_mix32(uint32_t x)
{
	x ^= x >> 16;
	x *= 0x7feb352du;
	x ^= x >> 15;
	x *= 0x846ca68bu;
	x ^= x >> 16;
	return x;
}

CB_HD uint32_t
jh_int8(int64_t val)
{
	uint32_t	lohalf = (uint32_t) val;
	const uint32_t hihalf = (uint32_t) ((uint64_t) val >> 32);

	lohalf ^= (val >= 0) ? hihalf : ~hihalf;
	return jh_mix32(lohalf);
}

#ifdef __CUDACC__
__device__ __forceinline__ uint32_t
jh_hash_datum(int type, int64_t v, const uint32_t *dict)
{
	switch (type)
	{
		case CB_INT4: case CB_DATE:
			return jh_mix32((uint32_t) (int32_t) v);
		case CB_INT8:
			return jh_int8(v);
		default:
			return pg_hash_datum(type, v, dict);	/* dictionary codes: the per-code table; bpchar(1), bool */
	}
}
#endif

/* Bloom word index and bit pattern of a 32-bit key hash: two multiplicative remixes, the word from
 * the top bits of one, the two bit positions from the top bits of the other */
CB_HD uint32_t
ht_bloom_bits(uint32_t h, uint32_t *word, uint32_t bloom_mask)
{
	const uint32_t m1 = h * 0x9e3779b1u;
	const uint32_t m2 = h * 0x85ebca6bu;

	*word = (m1 >> 4) & bloom_mask;
	return (1u << (m2 >> 27)) | (1u << ((m2 >> 22) & 31));
}

#ifdef __CUDACC__
/* L2 eviction-priority policies for per-load cache hints: columns streamed once should not push
 * out the structures every row consults (Bloom filters, inter-stage queues) */
__device__ __forceinline__ uint64_t
l2_policy_evict_first(void)
{
	uint64_t	p;

	asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
	return p;
}

__device__ __forceinline__ uint64_t
l2_policy_evict_last(void)
{
	uint64_t	p;

	asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
	return p;
}

__device__ __forceinline__ uint32_t
ldg_hint_u32(const uint32_t *a, uint64_t pol)
{
	uint32_t	v;

	asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(a), "l"(pol));
	return v;
}

__device__ __forceinline__ int32_t
ldg_stream_s32(const int32_t *a, uint64_t pol)
{
	int32_t		v;

	asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(a), "l"(pol));
	return v;
}

__device__ __forceinline__ int64_t
ldg_stream_s64(const long long *a, uint64_t pol)
{
	long long	v;

	asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.s64 %0, [%1], %2;" : "=l"(v) : "l"(a), "l"(pol));
	return v;
}

__device__ __forceinline__ int4
ldg_stream_v4(const int4 *a, uint64_t pol)
{
	int4		v;

	asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.s32 {%0, %1, %2, %3}, [%4], %5;"
				 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(a), "l"(pol));
	return v;
}

__device__ __forceinline__ unsigned long long
ldg_stream_u64(const unsigned long long *a, uint64_t pol)
{
	unsigned long long v;

	asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(a), "l"(pol));
	return v;
}
#endif

#ifdef __CUDACC__
/* ---- TMA bulk-copy pipeline primitives (sm_90+ PTX; SASS: UBLKCP / SYNCS) ---- */
__device__ __forceinline__ uint32_t
smem_u32(const void *p)
{
	return (uint32_t) __cvta_generic_to_shared(p);
}

__device__ __forceinline__ void
mbar_init(uint64_t *bar, unsigned count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count));
}

__device__ __forceinline__ void
mbar_expect_tx(uint64_t *bar, unsigned bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void
mbar_arrive(uint64_t *bar)
{
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ void
mbar_wait(uint64_t *bar, unsigned parity)
{
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"WAIT_%=:\n"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
		"@p bra DONE_%=;\n"
		"bra WAIT_%=;\n"
		"DONE_%=:\n"
		"}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}

/* one contiguous global -> shared bulk copy, completion counted in bytes on `bar` */
__device__ __forceinline__ void
tma_load_1d(void *dst, const void *src, unsigned bytes, uint64_t *bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
				 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

#endif

/* widen a column element to 64 bits (float8: raw bits) */
__device__ __forceinline__ int64_t
cb_load_widen(const void *data, int type, uint32_t row)
{
	switch (type)
	{
		case CB_INT4: case CB_DATE: case CB_DICT32:
			return (int64_t) __ldg((const int32_t *) data + row);
		case CB_INT8: case CB_NUMERIC: case CB_FLOAT8:
			return __ldg((const long long *) data + row);
		default:
			return (int64_t) __ldg((const uint8_t *) data + row);
	}
}

#ifdef __CUDACC__
/* the join-table hash of a row's keys is h = 0 folded with each key in turn: h = jh_key_fold(h, type, value, dict).  Build and
 * probe sides must agree on it bit for bit (the int4 / int8 fast forms of probe_chain.cu are this fold over one key). */
__device__ __forceinline__ uint32_t
jh_key_fold(uint32_t h, int type, int64_t v, const uint32_t *dict)
{
	return pg_hash_combine(h, jh_hash_datum(type, v, dict), false);
}

/* does slot entry e hold a build row whose key equals the probe's?  Tag first, then (unless the table is key-in-slot) the
 * build row's key columns by row id */
__device__ __forceinline__ bool
ht_slot_match(const HtDev &ht, unsigned long long e, uint32_t tag, const int64_t *key, int nkeys)
{
	if (!ht_tag_match(e, tag))
		return false;
	for (int k = 0; k < nkeys && !ht.keyslot; k++)
		if (cb_load_widen(ht.keydata[k], ht.keytype[k], ht_slot_row(e)) != key[k])
			return false;
	return true;
}

/* slot `pos` of a table: LDG, through the read-only cache (the table in global memory); else a plain load through a generic
 * pointer, global or shared memory (a CTA's copy of a small table) */
template <bool LDG>
__device__ __forceinline__ unsigned long long
ht_slot_load(const unsigned long long *slots, uint32_t pos)
{
	return LDG ? __ldg(slots + pos) : slots[pos];
}

/* ExecScanHashBucket (nodeHash.c:2255) for an N:1 join: the walk from slot `pos`, whose entry `e` the caller loaded already
 * (so that a caller can issue several rows' first loads together), to the first build row whose key equals the probe's.
 * False when there is none, or when a key-in-slot table cannot hold the key at all. */
template <bool LDG>
__device__ __forceinline__ bool
ht_find(const HtDev &ht, const unsigned long long *slots, uint32_t pos, unsigned long long e, uint32_t hash, const int64_t *key,
		int nkeys, uint32_t *row)
{
	const uint32_t tag = ht_probe_tag(ht.keyslot, hash, key[0]);

	if (ht.keyslot && !ht_key_in_domain(ht.keyslot, key[0]))
		return false;
	while (!ht_slot_empty(e))
	{
		if (ht_slot_match(ht, e, tag, key, nkeys))
		{
			*row = ht_slot_row(e);
			return true;
		}
		pos = (pos + 1) & ht.mask;
		e = ht_slot_load<LDG>(slots, pos);
	}
	return false;
}
#endif

/* ---------------------------------------------------------------------------------------------
 * exact 128-bit accumulate built from 64-bit atomics.  Additions commute, so the final (hi, lo)
 * pair is exact once all adds have landed: lo wraps, each wrap carries into hi.
 * (The reference keeps int8 sums in an Int128AggState, utils/adt/numeric.c:5340.)
 * --------------------------------------------------------------------------------------------- */
__device__ __forceinline__ void
atomic_add128(unsigned long long *acc, unsigned long long lo, unsigned long long hi)
{
	if (lo)
	{
		unsigned long long old = atomicAdd(acc, lo);

		if (old + lo < old)
			hi += 1;
	}
	if (hi)
		atomicAdd(acc + 1, hi);
}

__device__ __forceinline__ void
atomic_add128_signed(unsigned long long *acc, long long v)
{
	atomic_add128(acc, (unsigned long long) v, v < 0 ? ~0ull : 0ull);
}

/* group lookup / insert in an agg table.  Returns the slot, or -1 when the table is full.
 *
 * A slot is claimed with one CAS (0 -> 1), filled, then published (state 2).  A lane that meets a
 * slot in state 1 re-reads it on the NEXT trip of the same loop instead of spinning in a loop of
 * its own: the claiming lane may sit in the same warp (adjacent rows of one group), and it can only
 * finish its store if the divergent paths reconverge at the bottom of every trip. */
__device__ __forceinline__ int
agg_find_or_insert(const AggDev &t, uint32_t hash, const int64_t *keys, uint32_t nullmask)
{
	uint32_t	pos = hash & t.mask;
	uint32_t	probes = 0;
	int			result = -2;

	while (result == -2)
	{
		int			s = *((volatile int *) (t.state + pos));

		if (s == 0)
		{
			s = atomicCAS(t.state + pos, 0, 1);
			if (s == 0)
			{
				/* initialize_hash_entry (executor/nodeAgg.c:2220): copy the grouping keys */
				for (int k = 0; k < t.nkeys; k++)
					t.keys[(size_t) pos * t.nkeys + k] = keys[k];
				t.keynull[pos] = nullmask;
				t.hash[pos] = hash;
				__threadfence();
				*((volatile int *) (t.state + pos)) = 2;
				result = (int) pos;
			}
		}
		if (result == -2 && s == 2)
		{
			bool		same = false;

			__threadfence();
			if (*((volatile uint32_t *) (t.hash + pos)) == hash && *((volatile uint32_t *) (t.keynull + pos)) == nullmask)
			{
				/* TupleHashTableMatch (executor/execGrouping.c:548): NULLs group together */
				same = true;
				for (int k = 0; k < t.nkeys; k++)
					if (!((nullmask >> k) & 1) && *((volatile long long *) (t.keys + (size_t) pos * t.nkeys + k)) != keys[k])
						same = false;
			}
			if (same)
				result = (int) pos;
			else if (++probes > t.mask)
			{
				atomicExch(t.full, 1);
				result = -1;
			}
			else
				pos = (pos + 1) & t.mask;
		}
		/* s == 1: the owner is filling the slot; look again */
	}
	return result;
}
