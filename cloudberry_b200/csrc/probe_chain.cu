/*
 * probe_chain.cu - K3 fused: scan -> range quals -> up to four N:1 hash-join probes -> sink, compiled
 * (not interpreted), one persistent kernel whose stages run on full batches.
 *
 * Restates the outer side of ExecHashJoinImpl (backend/executor/nodeHashjoin.c:203-738):
 * HJ_NEED_NEW_OUTER fetches the next outer tuple (here: the next row of the driving scan that
 * passes its quals, ExecScan execScan.c:162), ExecHashGetHashValue hashes the join keys
 * (nodeHash.c:2089), ExecScanHashBucket finds the match (nodeHash.c:2255), and the joined tuple
 * feeds the next join's outer side - for the whole chain of joins at once, then the sink:
 * hash aggregation (agg_fill_hash_table, nodeAgg.c:2726) or materialisation for a parent Hash /
 * Motion.  Shapes covered: TPC-H Q3 / Q5 / Q10-style star and chain joins on integer keys.
 *
 * Design.  The pipeline is a chain of stages joined by queues of row-id tuples:
 *
 *     F      quals (+ visimap) over a tile of driving rows           -> queue 0 (shared memory)
 *     B_j    Bloom filter of build side j (L2-resident)              -> queue 2j+1 (+ key hash)
 *     H_j    hash table j (HBM), stored hash, key verification       -> queue 2j+2 (+ inner row id)
 *     sink   aggregate / materialise
 *
 * A persistent CTA (4 per SM) schedules them itself: the deepest stage with a full batch
 * (PC_BATCH entries, PC_U per thread) runs; otherwise the next tile is scanned; at the end the
 * queues drain front to back.  So every stage always runs with full warps over rows that are still
 * alive, a probe behind a selective qual, filter or join costs only its survivors (late
 * materialisation: key and payload columns are gathered by row id in the stage that needs them),
 * and inside a stage each thread issues the loads of its PC_U rows back to back before using any -
 * the memory-level parallelism a row-at-a-time loop over dependent (column -> filter word -> slot ->
 * key) loads lacks.  Queue 0 carries most rows and lives in shared memory; the deeper queues see
 * few rows and live in a per-CTA slice of global memory that stays in L2.
 */
#include "pipeline.cuh"
#include "xmatch.h"

#include <stdio.h>
#include <stdlib.h>

#define PC_THREADS 256
#define PC_TILE 2048			/* driving rows per run of stage F                                    */
#define PC_BATCH 1024			/* queue entries per run of any other stage                           */
#define PC_OCC 4				/* resident CTAs per SM the register budget is set for                */
#define PC_U (PC_BATCH / PC_THREADS)
#define PC_Q0CAP (PC_BATCH + PC_TILE)
#define PC_QCAP (2 * PC_BATCH)	/* a consumer runs at PC_BATCH, a producer adds at most PC_BATCH      */
#define PC_MAXP 4
#define PC_MAXOUT 8
#define PC_NQ (2 * PC_MAXP + 1)

struct PcCol
{
	const void *data;
	const uint32_t *dict;
	int32_t		type;
	int32_t		src;			/* 0 = driving relation, 1 + j = inner side of probe j                */
};

struct PcFilter
{
	const void *col;			/* int32 / date column, or a 1-byte one (dictionary code, char(1), bool) */
	int32_t		width;			/* 4 or 1                                                             */
	int32_t		lo;
	uint32_t	span;
};

struct PcProbe
{
	HtDev		ht;
	int32_t		nkeys;
	int32_t		jointype;
	int32_t		kind;			/* 0: one int32 key, hashint4; 1: one int64 key, hashint8; 2: general */
	PcCol		key[2];
	int32_t		keytype[2];		/* hash function by the OUTER key's type (cross-type int4/int8 joins) */
	/* how the table is reached.  0: Bloom filter stage B_j, then the table in HBM (stage H_j).  1: ONE stage straight into
	 * the table - the prefilter pass applied its Bloom filter already.  2: the same, with the table's slots staged into the
	 * CTA's shared memory by a TMA bulk copy (cp.async.bulk + mbarrier) when the kernel starts - dimension tables of a few
	 * thousand rows (nation, region, date): such a probe never leaves the SM.  (nodeHash.c builds ONE table kind;
	 * SURVEY.md 8 row a6 asks for this split.) */
	int32_t		mode;
	int32_t		smem_off;		/* mode 2: first slot inside the dynamic shared memory, in slots       */
};

#define PC_MAXEARLY 2
struct PcEarly
{
	const void *col;			/* driving-relation column (4 or 8 bytes wide)                         */
	int32_t		width;
	int32_t		hashtype;		/* CbTypeId whose hash function keys the filter                       */
	const uint32_t *bloom;
	uint32_t	mask;
};

struct PcParams
{
	int64_t		nrows;
	/* the driving rows are sel[0 .. nrows) instead of 0 .. nrows: what k_prefilter left of a big scan (quals, visimap and
	 * scan-level filters are then done: nfilters = nearly = 0, visimap = NULL) */
	const uint32_t *sel;
	const uint8_t *visimap;
	int32_t		nfilters;
	int32_t		np;
	PcFilter	filt[2];
	PcProbe		probe[PC_MAXP];
	/* scan-level runtime filters (the reference's PassByBloomFilter in the SeqScan, executor/nodeSeqscan.c:413,
	 * built by CreateRuntimeFilter executor/nodeHashjoin.c:2217 per hash-clause column that traces down to the
	 * scan): a Bloom filter over ONE key column of a later probe's build side, checked in stage F */
	int32_t		nearly;
	PcEarly		early[PC_MAXEARLY];
	uint32_t   *qmem;			/* global queues: [CTA][q_cta_words]                                  */
	int64_t		q_cta_words;
	int32_t		q_off[PC_NQ];	/* queue k >= 1: word offset inside the CTA's slice                   */
	int32_t		q_cap[PC_NQ];	/* ... and its capacity in entries                                    */
	/* stage F also runs probe 0's key hash and Bloom test (its key is a column of the driving relation, read
	 * 16 bytes at a time like the qual columns) and feeds queue 1 directly: the rows the quals pass never
	 * go through queue 0 and a separate gather of their keys */
	int32_t		fuse0;
	uint32_t	smem_table_bytes;	/* shared-memory tables of the mode 2 probes, all together             */
	/* sink */
	int32_t		sink_kind;		/* CBP_SINK_AGG or CBP_SINK_MATERIALIZE                               */
	AggDev		agg;
	int32_t		nkeys;
	PcCol		key[CBP_MAX_KEYS];
	int32_t		naccs;
	int32_t		acc_term[CBP_MAX_AGGS];	/* -1 = count, else index of the value term               */
	int32_t		nterms;
	int32_t		term_kind[2];	/* 0 = column a, 1 = a * (k - b), 2 = a - b, 3 = a + b                */
	PcCol		term_a[2], term_b[2];
	long long	term_k[2];
	int32_t		nout;
	PcCol		out[PC_MAXOUT];
	void	   *outcol[PC_MAXOUT];
	int32_t		outtype[PC_MAXOUT];
	unsigned long long *out_count;
	int64_t		out_capacity;
	/* PARTITION: cdbhash over the first nhash output columns picks the destination segment */
	int32_t		nhash;
	int32_t		hashtype[CBP_MAX_KEYS];
	const uint32_t *hashdict[CBP_MAX_KEYS];
	int32_t		nsegs;
	int64_t		seg_capacity;
	void *const *part_cols;		/* direct Motion: destination d's column c at part_cols[d * nout + c]  */
	unsigned long long *const *part_counts;
	int32_t    *part_flags;		/* a full destination ORs CBGPU_DX_OVERFLOW in here (NULL: status word) */
	int64_t		seg_base[64];
	int64_t		seg_cap[64];
	int		   *status;
};

/* shared scratch of the PARTITION sink: destination and rank within it for every entry of a run */
struct PcPart
{
	unsigned	count[64];
	unsigned long long base[64];
	uint8_t		seg[PC_BATCH];
	uint16_t	rank[PC_BATCH];
};

/* a queue as a stage sees it: word w of entry e at q[w * cap + e]; words 0 .. = row ids by source */
struct PcQ
{
	const uint32_t *q;
	uint32_t	cap;
	uint32_t	iota_base;		/* q == NULL: entry e is driving row iota_base + e (no quals) ...     */
	const uint32_t *sel;		/* ... or, after a prefilter pass, sel[iota_base + e]                 */
};

__device__ __forceinline__ uint32_t
pc_row(const PcQ &Q, int src, uint32_t e)
{
	return Q.q ? Q.q[(size_t) src * Q.cap + e] : (Q.sel ? Q.sel[Q.iota_base + e] : Q.iota_base + e);
}

__device__ __forceinline__ int64_t
pc_load(const PcCol &c, const PcQ &Q, uint32_t e)
{
	return cb_load_widen(c.data, c.type, pc_row(Q, c.src, e));
}

/* reserve one output position per surviving lane: one shared-memory atomic per warp; every lane of
 * the warp calls (full-mask ballot: the warp is converged afterwards) */
__device__ __forceinline__ uint32_t
pc_reserve(unsigned *cnt, bool alive)
{
	const unsigned m = __ballot_sync(0xffffffffu, alive);
	const int	lane = threadIdx.x & 31;
	unsigned	base = 0;

	if (m == 0)
		return 0;
	if (lane == (__ffs(m) - 1))
		base = atomicAdd(cnt, (unsigned) __popc(m));
	base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
	return base + __popc(m & ((1u << lane) - 1));
}

template <int KIND>
__device__ __forceinline__ uint32_t
pc_key_hash(const PcProbe &pr, int64_t k0, int64_t k1)
{
	if (KIND == 0)
		return pg_hash_combine(0u, jh_mix32((uint32_t) (int32_t) k0), false);
	if (KIND == 1)
		return pg_hash_combine(0u, jh_int8(k0), false);
	uint32_t	h = pg_hash_combine(0u, jh_hash_datum(pr.keytype[0], k0, pr.key[0].dict), false);

	if (pr.nkeys > 1)
		h = pg_hash_combine(h, jh_hash_datum(pr.keytype[1], k1, pr.key[1].dict), false);
	return h;
}

template <int KIND>
__device__ __forceinline__ int64_t
pc_load_key0(const PcProbe &pr, uint32_t row, uint64_t pol_stream)
{
	/* a key column of the driving relation is read once, front to back: first in line for eviction */
	if (KIND == 0)
		return pr.key[0].src == 0 ? (int64_t) ldg_stream_s32((const int32_t *) pr.key[0].data + row, pol_stream)
			: (int64_t) __ldg((const int32_t *) pr.key[0].data + row);
	if (KIND == 1)
		return pr.key[0].src == 0 ? ldg_stream_s64((const long long *) pr.key[0].data + row, pol_stream)
			: __ldg((const long long *) pr.key[0].data + row);
	return cb_load_widen(pr.key[0].data, pr.key[0].type, row);
}

/* stage B_j: hash the join keys (ExecHashGetHashValue, nodeHash.c:2089) and test the build side's
 * Bloom filter.  in: entries [base, base + n) of Q (j + 1 row ids); out: the same row ids + hash. */
template <int KIND>
__device__ __noinline__ void
pc_stage_bloom(const PcProbe &pr, int j, PcQ Q, unsigned base, unsigned n, uint32_t *out, unsigned ocap, unsigned *ocnt)
{
	/* an anti join keeps the rows WITHOUT a match: the filter cannot drop anything */
	const bool	use_bloom = pr.ht.bloom != NULL && pr.jointype != CB_JOIN_ANTI;
	const uint64_t pol_stream = l2_policy_evict_first();
	const uint64_t pol_keep = l2_policy_evict_last();
	const int	lane = threadIdx.x & 31;
	uint32_t	e[PC_U], h[PC_U], w[PC_U], bits[PC_U], word[PC_U], bal[PC_U];
	int64_t		k0[PC_U], k1[PC_U];
	bool		v[PC_U];

#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		const unsigned i = u * PC_THREADS + threadIdx.x;
		uint32_t	r0;

		v[u] = i < n;
		e[u] = base + (v[u] ? i : 0u);
		r0 = pc_row(Q, pr.key[0].src, e[u]);
		k0[u] = pc_load_key0<KIND>(pr, r0, pol_stream);
		k1[u] = (KIND == 2 && pr.nkeys > 1) ? pc_load(pr.key[1], Q, e[u]) : 0;
	}
#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		h[u] = pc_key_hash<KIND>(pr, k0[u], k1[u]);
		bits[u] = ht_bloom_bits(h[u], &w[u], pr.ht.bloom_mask);
	}
	if (use_bloom)
	{
		/* the filter is consulted by every row: last in line for eviction from L2 */
#pragma unroll
		for (int u = 0; u < PC_U; u++)
			word[u] = ldg_hint_u32(pr.ht.bloom + w[u], pol_keep);
	}
	/* one reservation per warp for all PC_U rows of every lane; entries stay in row order */
	unsigned	tot = 0,
				wb = 0;

#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		const bool	pass = v[u] && (!use_bloom || (word[u] & bits[u]) == bits[u]);

		bal[u] = __ballot_sync(0xffffffffu, pass);
		tot += __popc(bal[u]);
	}
	if (tot == 0)
		return;
	if (lane == 0)
		wb = atomicAdd(ocnt, tot);
	wb = __shfl_sync(0xffffffffu, wb, 0);
#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		if ((bal[u] >> lane) & 1)
		{
			const uint32_t pos = wb + __popc(bal[u] & ((1u << lane) - 1));

			for (int s = 0; s <= j; s++)
				out[(size_t) s * ocap + pos] = pc_row(Q, s, e[u]);
			out[(size_t) (j + 1) * ocap + pos] = h[u];
		}
		wb += __popc(bal[u]);
	}
}

/* stage H_j: ExecScanHashBucket (nodeHash.c:2255) for the rows that passed the filter: linear
 * probing from hash & mask, stored hash compared first, then the key itself.
 * in: j + 1 row ids + hash; out: j + 2 row ids. */
template <int KIND>
__device__ __noinline__ void
pc_stage_ht(const PcProbe &pr, int j, PcQ Q, unsigned base, unsigned n, uint32_t *out, unsigned ocap, unsigned *ocnt)
{
	const uint64_t pol_stream = l2_policy_evict_first();
	const int	lane = threadIdx.x & 31;
	uint32_t	e[PC_U], h[PC_U], pos[PC_U], irow[PC_U], bal[PC_U];
	unsigned long long slot[PC_U];
	bool		v[PC_U];

#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		const unsigned i = u * PC_THREADS + threadIdx.x;

		v[u] = i < n;
		e[u] = base + (v[u] ? i : 0u);
		h[u] = Q.q[(size_t) (j + 1) * Q.cap + e[u]];
		pos[u] = h[u] & pr.ht.mask;
	}
#pragma unroll
	for (int u = 0; u < PC_U; u++)
		slot[u] = v[u] ? __ldg(pr.ht.slots + pos[u]) : HT_EMPTY;
	unsigned	tot = 0,
				wb = 0;

#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		bool		found = false;

		irow[u] = 0;
		if (slot[u] != HT_EMPTY)
		{
			const int64_t k0 = pc_load_key0<KIND>(pr, pc_row(Q, pr.key[0].src, e[u]), pol_stream);
			const int64_t k1 = (KIND == 2 && pr.nkeys > 1) ? pc_load(pr.key[1], Q, e[u]) : 0;
			unsigned long long x = slot[u];
			uint32_t	p = pos[u];

			if (pr.ht.keyslot)
			{
				/* key-in-slot table: the slot settles it, no access to the build side's key column */
				const uint32_t tag = (uint32_t) k0;

				if (ht_key_in_domain(pr.ht.keyslot, k0))
					while (x != HT_EMPTY)
					{
						if ((uint32_t) (x >> 32) == tag)
						{
							found = true;
							irow[u] = (uint32_t) x;
							break;
						}
						p = (p + 1) & pr.ht.mask;
						x = __ldg(pr.ht.slots + p);
					}
			}
			else
				while (x != HT_EMPTY)
				{
					if ((uint32_t) (x >> 32) == h[u])
					{
						const uint32_t r = (uint32_t) x;

						if (cb_load_widen(pr.ht.keydata[0], pr.ht.keytype[0], r) == k0 &&
							(KIND != 2 || pr.nkeys < 2 || cb_load_widen(pr.ht.keydata[1], pr.ht.keytype[1], r) == k1))
						{
							found = true;
							irow[u] = r;
							break;
						}
					}
					p = (p + 1) & pr.ht.mask;
					x = __ldg(pr.ht.slots + p);
				}
		}
		/* full-mask ballot: the warp reconverges here */
		bal[u] = __ballot_sync(0xffffffffu, v[u] && (pr.jointype == CB_JOIN_ANTI ? !found : found));
		tot += __popc(bal[u]);
	}
	if (tot == 0)
		return;
	if (lane == 0)
		wb = atomicAdd(ocnt, tot);
	wb = __shfl_sync(0xffffffffu, wb, 0);
#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		if ((bal[u] >> lane) & 1)
		{
			const uint32_t opos = wb + __popc(bal[u] & ((1u << lane) - 1));

			for (int s = 0; s <= j; s++)
				out[(size_t) s * ocap + opos] = pc_row(Q, s, e[u]);
			out[(size_t) (j + 1) * ocap + opos] = irow[u];
		}
		wb += __popc(bal[u]);
	}
}

/* stage D_j (PcProbe.mode 1 / 2): key hash and table probe in one stage, for tables that stay in L2 (`slots` = the
 * table in global memory) or were staged into shared memory (`slots` = the CTA's copy).
 * in: j + 1 row ids; out: j + 2 row ids, into queue 2j + 2 (queue 2j + 1 stays empty). */
template <int KIND>
__device__ __noinline__ void
pc_stage_direct(const PcProbe &pr, int j, PcQ Q, unsigned base, unsigned n, uint32_t *out, unsigned ocap, unsigned *ocnt, const unsigned long long *slots)
{
	const uint64_t pol_stream = l2_policy_evict_first();
	const int	lane = threadIdx.x & 31;
	uint32_t	e[PC_U], h[PC_U], pos[PC_U], irow[PC_U], bal[PC_U];
	int64_t		k0[PC_U], k1[PC_U];
	unsigned long long slot[PC_U];
	bool		v[PC_U];

#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		const unsigned i = u * PC_THREADS + threadIdx.x;

		v[u] = i < n;
		e[u] = base + (v[u] ? i : 0u);
		k0[u] = pc_load_key0<KIND>(pr, pc_row(Q, pr.key[0].src, e[u]), pol_stream);
		k1[u] = (KIND == 2 && pr.nkeys > 1) ? pc_load(pr.key[1], Q, e[u]) : 0;
	}
#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		h[u] = pc_key_hash<KIND>(pr, k0[u], k1[u]);
		pos[u] = h[u] & pr.ht.mask;
	}
#pragma unroll
	for (int u = 0; u < PC_U; u++)
		slot[u] = v[u] ? slots[pos[u]] : HT_EMPTY;
	unsigned	tot = 0,
				wb = 0;

#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		bool		found = false;
		unsigned long long x = slot[u];
		uint32_t	p = pos[u];

		irow[u] = 0;
		if (pr.ht.keyslot)
		{
			const uint32_t tag = (uint32_t) k0[u];

			if (ht_key_in_domain(pr.ht.keyslot, k0[u]))
				while (x != HT_EMPTY)
				{
					if ((uint32_t) (x >> 32) == tag)
					{
						found = true;
						irow[u] = (uint32_t) x;
						break;
					}
					p = (p + 1) & pr.ht.mask;
					x = slots[p];
				}
		}
		else
			while (x != HT_EMPTY)
			{
				if ((uint32_t) (x >> 32) == h[u])
				{
					const uint32_t r = (uint32_t) x;

					if (cb_load_widen(pr.ht.keydata[0], pr.ht.keytype[0], r) == k0[u] &&
						(KIND != 2 || pr.nkeys < 2 || cb_load_widen(pr.ht.keydata[1], pr.ht.keytype[1], r) == k1[u]))
					{
						found = true;
						irow[u] = r;
						break;
					}
				}
				p = (p + 1) & pr.ht.mask;
				x = slots[p];
			}
		/* full-mask ballot: the warp reconverges here */
		bal[u] = __ballot_sync(0xffffffffu, v[u] && (pr.jointype == CB_JOIN_ANTI ? !found : found));
		tot += __popc(bal[u]);
	}
	if (tot == 0)
		return;
	if (lane == 0)
		wb = atomicAdd(ocnt, tot);
	wb = __shfl_sync(0xffffffffu, wb, 0);
#pragma unroll
	for (int u = 0; u < PC_U; u++)
	{
		if ((bal[u] >> lane) & 1)
		{
			const uint32_t opos = wb + __popc(bal[u] & ((1u << lane) - 1));

			for (int s = 0; s <= j; s++)
				out[(size_t) s * ocap + opos] = pc_row(Q, s, e[u]);
			out[(size_t) (j + 1) * ocap + opos] = irow[u];
		}
		wb += __popc(bal[u]);
	}
}

/* sink over entries [base, base + n) of the last queue (np + 1 row ids) */
__device__ __noinline__ void
pc_stage_sink(const PcParams &P, PcQ Q, unsigned base, unsigned n, unsigned long long *s_obase, PcPart *part)
{
	if (P.sink_kind == CBP_SINK_AGG)
	{
		for (unsigned b = 0; b < n; b += PC_THREADS)
		{
			const unsigned i = b + threadIdx.x;

			if (i < n)
			{
				const uint32_t e = base + i;
				int64_t		kv[CBP_MAX_KEYS];
				uint32_t	h = 0;

				/* TupleHashTableHash_internal (executor/execGrouping.c:437-495) */
				for (int k = 0; k < P.nkeys; k++)
				{
					kv[k] = pc_load(P.key[k], Q, e);
					h = pg_hash_combine(h, pg_hash_datum(P.key[k].type, kv[k], P.key[k].dict), false);
				}
				h = pg_murmurhash32(h);
				int64_t		tv[2] = {0, 0};

				for (int t = 0; t < P.nterms; t++)
				{
					int64_t		a = pc_load(P.term_a[t], Q, e);

					if (P.term_kind[t] == 1)
					{
						int64_t		bb = pc_load(P.term_b[t], Q, e);
						int64_t		k = P.term_k[t];
						int64_t		d = (int64_t) ((uint64_t) k - (uint64_t) bb);
						int64_t		r = (int64_t) ((uint64_t) a * (uint64_t) d);

						/* numeric_mul / numeric_sub are exact; a product that leaves 64 bits is refused */
						if ((((k ^ bb) & (k ^ d)) < 0) || (__mul64hi(a, d) != (r >> 63)))
							atomicExch(P.status, CBGPU_ERR_OVERFLOW);
						tv[t] = r;
					}
					else if (P.term_kind[t] >= 2)
					{
						const int64_t bb = pc_load(P.term_b[t], Q, e);
						const int64_t r = P.term_kind[t] == 2 ? (int64_t) ((uint64_t) a - (uint64_t) bb) : (int64_t) ((uint64_t) a + (uint64_t) bb);

						/* int8mi / int8pl raise "bigint out of range" (utils/adt/int8.c:448,427): refused */
						if (P.term_kind[t] == 2 ? (((a ^ bb) & (a ^ r)) < 0) : ((~(a ^ bb) & (a ^ r)) < 0))
							atomicExch(P.status, CBGPU_ERR_OVERFLOW);
						tv[t] = r;
					}
					else
						tv[t] = a;
				}
				int			slot = agg_find_or_insert(P.agg, h, kv, 0);

				if (slot >= 0)
					for (int a = 0; a < P.naccs; a++)
					{
						atomicAdd((unsigned long long *) (P.agg.n + (size_t) slot * P.agg.naccs + a), 1ull);
						if (P.acc_term[a] >= 0)
							atomic_add128_signed(P.agg.sum + ((size_t) slot * P.agg.naccs + a) * 2, tv[P.acc_term[a]]);
					}
			}
			__syncwarp();		/* lanes that waited on a group being created rejoin before the next trip */
		}
	}
	else if (P.sink_kind == CBP_SINK_PARTITION)
	{
		/* execMotionSender / evalHashKey (nodeMotion.c:203,1088): destination = cdbhashreduce of the hash
		 * keys (cdb/cdbhash.c:189,253).  Rows are counted per destination in shared memory, the run
		 * takes one slice per destination from the send buffer, then every row is stored. */
		if (threadIdx.x < 64)
			part->count[threadIdx.x] = 0;
		__syncthreads();
		for (unsigned i = threadIdx.x; i < n; i += PC_THREADS)
		{
			uint32_t	h = 0;

			for (int k = 0; k < P.nhash; k++)
				h = pg_hash_combine(h, pg_hash_datum(P.hashtype[k], pc_load(P.out[k], Q, base + i), P.hashdict[k]), false);
			const int	seg = pg_jump_consistent_hash(h, P.nsegs);

			part->seg[i] = (uint8_t) seg;
			part->rank[i] = (uint16_t) atomicAdd(&part->count[seg], 1u);
		}
		__syncthreads();
		if (threadIdx.x < P.nsegs && part->count[threadIdx.x])
		{
			unsigned long long b = atomicAdd(P.out_count + threadIdx.x, (unsigned long long) part->count[threadIdx.x]);

			/* direct Motion: the slice is reserved in the DESTINATION segment's buffer, over NVLink */
			if (P.part_cols)
				b = atomicAdd_system(P.part_counts[threadIdx.x], (unsigned long long) part->count[threadIdx.x]);
			part->base[threadIdx.x] = b;
			if ((int64_t) (b + part->count[threadIdx.x]) > P.seg_cap[threadIdx.x])
			{
				/* a full Motion destination is not an error: the host redoes the pass with exact sizes */
				if (P.part_flags)
					atomicOr(P.part_flags, CBGPU_DX_OVERFLOW);
				else
					atomicExch(P.status, CBGPU_ERR_NOMEM);
			}
		}
		__syncthreads();
		for (unsigned i = threadIdx.x; i < n; i += PC_THREADS)
		{
			const int	seg = part->seg[i];
			const unsigned long long pos = part->base[seg] + part->rank[i];

			if ((int64_t) pos < P.seg_cap[seg])
			{
				const uint64_t dst = P.part_cols ? pos : (uint64_t) P.seg_base[seg] + pos;

				for (int c = 0; c < P.nout; c++)
					sink_store(P.part_cols ? P.part_cols[seg * P.nout + c] : P.outcol[c], P.outtype[c], dst, pc_load(P.out[c], Q, base + i));
			}
		}
	}
	else
	{
		/* one reservation of n output rows per run, then coalesced stores */
		if (threadIdx.x == 0)
			*s_obase = atomicAdd(P.out_count, (unsigned long long) n);
		__syncthreads();
		const unsigned long long ob = *s_obase;

		if ((int64_t) (ob + n) > P.out_capacity)
		{
			if (threadIdx.x == 0)
				atomicExch(P.status, CBGPU_ERR_NOMEM);
		}
		else
			for (unsigned i = threadIdx.x; i < n; i += PC_THREADS)
				for (int c = 0; c < P.nout; c++)
					sink_store(P.outcol[c], P.outtype[c], ob + i, pc_load(P.out[c], Q, base + i));
	}
}

__device__ __forceinline__ int32_t
pc_filter_value(const PcFilter &f, int64_t row)
{
	return f.width == 4 ? __ldg((const int32_t *) f.col + row) : (int32_t) __ldg((const uint8_t *) f.col + row);
}

/* eight consecutive 1-byte values as eight ints */
__device__ __forceinline__ void
pc_unpack8(unsigned long long v, int4 *a, int4 *b)
{
	const unsigned lo = (unsigned) v,
				hi = (unsigned) (v >> 32);

	*a = make_int4((int) (lo & 0xff), (int) ((lo >> 8) & 0xff), (int) ((lo >> 16) & 0xff), (int) (lo >> 24));
	*b = make_int4((int) (hi & 0xff), (int) ((hi >> 8) & 0xff), (int) ((hi >> 16) & 0xff), (int) (hi >> 24));
}

/* bit u set when row u of the eight (a.x .. b.w) lies in [lo, lo + span] */
__device__ __forceinline__ unsigned
pc_range8(int4 a, int4 b, int32_t lo, uint32_t span)
{
	return ((unsigned) ((unsigned) (a.x - lo) <= span) << 0) | ((unsigned) ((unsigned) (a.y - lo) <= span) << 1) |
		((unsigned) ((unsigned) (a.z - lo) <= span) << 2) | ((unsigned) ((unsigned) (a.w - lo) <= span) << 3) |
		((unsigned) ((unsigned) (b.x - lo) <= span) << 4) | ((unsigned) ((unsigned) (b.y - lo) <= span) << 5) |
		((unsigned) ((unsigned) (b.z - lo) <= span) << 6) | ((unsigned) ((unsigned) (b.w - lo) <= span) << 7);
}

/* the key values of a thread's 8 consecutive driving rows: int8 keys fill four 16-byte words, int4 keys two */
struct PcKeys8
{
	int4		q[4];
};

/* WIDE: 8-byte keys.  Unconditional 16-byte loads (a warp reads 2 KB / 1 KB contiguous): for warps whose rows are mostly alive */
template <bool WIDE>
__device__ __forceinline__ PcKeys8
pc_keys8_vec(const void *col, int64_t row0, uint64_t pol)
{
	PcKeys8		k;

	if (WIDE)
	{
		const int4 *p = (const int4 *) ((const long long *) col + row0);

#pragma unroll
		for (int i = 0; i < 4; i++)
			k.q[i] = ldg_stream_v4(p + i, pol);
	}
	else
	{
		const int4 *p = (const int4 *) ((const int32_t *) col + row0);

		k.q[0] = ldg_stream_v4(p, pol);
		k.q[1] = ldg_stream_v4(p + 1, pol);
		k.q[2] = k.q[3] = make_int4(0, 0, 0, 0);
	}
	return k;
}

/* one load per alive row: for warps with few survivors, and for a relation's last, partial tile */
template <bool WIDE>
__device__ __forceinline__ PcKeys8
pc_keys8_pred(const void *col, int64_t row0, unsigned am, uint64_t pol)
{
	PcKeys8		k;
	int			v[8];

	if (WIDE)
	{
		long long	t[8];

#pragma unroll
		for (int u = 0; u < 8; u++)
			t[u] = ((am >> u) & 1) ? ldg_stream_s64((const long long *) col + row0 + u, pol) : 0;
#pragma unroll
		for (int i = 0; i < 4; i++)
			k.q[i] = make_int4((int) (unsigned) t[2 * i], (int) (unsigned) ((unsigned long long) t[2 * i] >> 32), (int) (unsigned) t[2 * i + 1],
							   (int) (unsigned) ((unsigned long long) t[2 * i + 1] >> 32));
	}
	else
	{
#pragma unroll
		for (int u = 0; u < 8; u++)
			v[u] = ((am >> u) & 1) ? ldg_stream_s32((const int32_t *) col + row0 + u, pol) : 0;
		k.q[0] = make_int4(v[0], v[1], v[2], v[3]);
		k.q[1] = make_int4(v[4], v[5], v[6], v[7]);
		k.q[2] = k.q[3] = make_int4(0, 0, 0, 0);
	}
	return k;
}

template <bool WIDE>
__device__ __forceinline__ int64_t
pc_keys8_get(const PcKeys8 &k, int u)
{
	if (WIDE)
	{
		const int4	t = k.q[u >> 1];
		const unsigned lo = (u & 1) ? (unsigned) t.z : (unsigned) t.x;
		const unsigned hi = (u & 1) ? (unsigned) t.w : (unsigned) t.y;

		return (int64_t) (((unsigned long long) hi << 32) | lo);
	}
	const int4	t = k.q[u >> 2];

	return (int64_t) ((u & 3) == 0 ? t.x : (u & 3) == 1 ? t.y : (u & 3) == 2 ? t.z : t.w);
}

/* is this warp's tile dense enough for unconditional 16-byte key loads?  (warp-uniform: the lanes must not split over
 * the two load paths, a warp would run both) */
__device__ __forceinline__ bool
pc_warp_dense(bool full, unsigned am, unsigned at_least = 64u)
{
	return __all_sync(0xffffffffu, full) && __reduce_add_sync(0xffffffffu, (unsigned) __popc(am)) >= at_least;
}

/* stage F's tail when probe 0 is fused into it (P.fuse0): hash of the 8 keys, Bloom words of the alive ones in flight
 * together, survivors to queue 1 as (row id, hash) in row order - one warp scan, one shared-memory atomic.
 * WIDE: int8 key, else int4 / date. */
template <bool WIDE>
__device__ __forceinline__ void
pc_stage_f_probe0(const PcProbe &pr, int64_t row0, const PcKeys8 &keys, unsigned am, uint32_t *out, unsigned cap, unsigned *ocnt)
{
	const bool	use_bloom = pr.ht.bloom != NULL && pr.jointype != CB_JOIN_ANTI;
	const uint64_t pol_keep = l2_policy_evict_last();
	const int	lane = threadIdx.x & 31;
	uint32_t	h[8];

#pragma unroll
	for (int u = 0; u < 8; u++)
		h[u] = WIDE ? jh_int8(pc_keys8_get<true>(keys, u)) : jh_mix32((uint32_t) (int32_t) pc_keys8_get<false>(keys, u));
	if (use_bloom)
	{
		uint32_t	bits[8], word[8];

#pragma unroll
		for (int u = 0; u < 8; u++)
		{
			uint32_t	w;

			bits[u] = ht_bloom_bits(h[u], &w, pr.ht.bloom_mask);
			word[u] = ((am >> u) & 1) ? ldg_hint_u32(pr.ht.bloom + w, pol_keep) : 0u;
		}
#pragma unroll
		for (int u = 0; u < 8; u++)
			if ((word[u] & bits[u]) != bits[u])
				am &= ~(1u << u);
	}
	const unsigned c = __popc(am);
	unsigned	x = c;

#pragma unroll
	for (int d = 1; d < 32; d <<= 1)
	{
		const unsigned y = __shfl_up_sync(0xffffffffu, x, d);

		if (lane >= d)
			x += y;
	}
	const unsigned total = __shfl_sync(0xffffffffu, x, 31);
	unsigned	wb = 0;

	if (lane == 31 && total)
		wb = atomicAdd(ocnt, total);
	wb = __shfl_sync(0xffffffffu, wb, 31);
	unsigned	pos = wb + x - c;

#pragma unroll
	for (int u = 0; u < 8; u++)
		if ((am >> u) & 1)
		{
			out[pos] = (uint32_t) (row0 + u);
			out[(size_t) cap + pos] = h[u];
			pos++;
		}
}

/* a scan-level runtime filter over the thread's 8 rows: returns the alive mask with the rows that miss it cleared */
template <bool WIDE>
__device__ __forceinline__ unsigned
pc_early_filter8(const PcEarly &E, int64_t row0, bool full, unsigned am, uint64_t pol)
{
	const PcKeys8 keys = pc_warp_dense(full, am) ? pc_keys8_vec<WIDE>(E.col, row0, pol) : pc_keys8_pred<WIDE>(E.col, row0, am, pol);
	uint32_t	bits[8], word[8];

#pragma unroll
	for (int u = 0; u < 8; u++)
	{
		const int64_t kv = pc_keys8_get<WIDE>(keys, u);
		uint32_t	w;

		bits[u] = ht_bloom_bits(pg_hash_combine(0u, WIDE ? jh_int8(kv) : jh_mix32((uint32_t) (int32_t) kv), false), &w, E.mask);
		word[u] = ((am >> u) & 1) ? __ldg(E.bloom + w) : 0u;
	}
#pragma unroll
	for (int u = 0; u < 8; u++)
		if ((word[u] & bits[u]) != bits[u])
			am &= ~(1u << u);
	return am;
}

/* the same test over keys that are in registers already */
template <bool WIDE>
__device__ __forceinline__ unsigned
pc_bloom8_keys(const PcEarly &E, const PcKeys8 &keys, unsigned am)
{
	uint32_t	bits[8], word[8];

#pragma unroll
	for (int u = 0; u < 8; u++)
	{
		const int64_t kv = pc_keys8_get<WIDE>(keys, u);
		uint32_t	w;

		bits[u] = ht_bloom_bits(pg_hash_combine(0u, WIDE ? jh_int8(kv) : jh_mix32((uint32_t) (int32_t) kv), false), &w, E.mask);
		word[u] = ((am >> u) & 1) ? __ldg(E.bloom + w) : 0u;
	}
#pragma unroll
	for (int u = 0; u < 8; u++)
		if ((word[u] & bits[u]) != bits[u])
			am &= ~(1u << u);
	return am;
}

/* ---------------------------------------------------------------------------------------------
 * k_prefilter: the selective head of a join pipeline over a big scan, as a kernel of its own.
 *
 * k_probe_chain keeps a whole pipeline in one kernel, which costs it registers (64 per thread: half occupancy) - fine for
 * the stages that see few rows, wasteful for the one that sees them all.  When a scan of tens of millions of rows is cut
 * down hard before the first hash-table access - range quals, visimap, scan-level runtime filters, and the Bloom filter of
 * every INNER / SEMI probe whose single integer key is a column of the scan itself (the reference pushes exactly these
 * filters into its SeqScan: PassByBloomFilter, nodeSeqscan.c:413) - this lean kernel does the cutting at full occupancy and
 * leaves the surviving row ids, in row order per tile, for k_probe_chain to start from (PcParams.sel).
 * --------------------------------------------------------------------------------------------- */
#define PF_MAXBLOOM 6
struct PfParams
{
	int64_t		nrows;
	const uint8_t *visimap;
	int32_t		nfilters;
	PcFilter	filt[2];
	int32_t		nbloom;
	PcEarly		bloom[PF_MAXBLOOM];
	uint32_t   *out;
	unsigned long long *out_count;
};

template <bool SPEC>
__global__ void __launch_bounds__(PC_THREADS, SPEC ? 4 : 8)
k_prefilter(const __grid_constant__ PfParams P)
{
	__shared__ uint32_t buf[PC_TILE];
	__shared__ unsigned s_cnt;
	__shared__ unsigned long long s_gbase;
	const int64_t ntiles = (P.nrows + PC_TILE - 1) / PC_TILE;
	const unsigned o0 = threadIdx.x * 8;
	const int	lane = threadIdx.x & 31;
	const uint64_t pol_stream = l2_policy_evict_first();

	for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x)
	{
		const int64_t base = tile * PC_TILE;
		const unsigned nvalid = (unsigned) (P.nrows - base < PC_TILE ? P.nrows - base : PC_TILE);
		const bool	full = o0 + 8 <= nvalid;
		unsigned	am = 0;

		PcKeys8		keys0;
		bool		have0 = false;

		if (threadIdx.x == 0)
			s_cnt = 0;
		/* SPEC: the first filter's keys are requested together with the qual columns - one HBM latency per tile instead of
		 * two, for 8 - 16 more registers per thread (4 resident CTAs instead of 8) */
		if (SPEC && P.nbloom > 0 && __all_sync(0xffffffffu, full))
		{
			keys0 = P.bloom[0].width == 8 ? pc_keys8_vec<true>(P.bloom[0].col, base + o0, pol_stream)
				: pc_keys8_vec<false>(P.bloom[0].col, base + o0, pol_stream);
			have0 = true;
		}
		if (full)
		{
			int4		a0 = make_int4(0, 0, 0, 0), b0 = a0, a1 = a0, b1 = a0;
			unsigned	vm = 0xff;

			if (P.nfilters > 0)
			{
				if (P.filt[0].width == 4)
				{
					a0 = ldg_stream_v4((const int4 *) ((const int32_t *) P.filt[0].col + base + o0), pol_stream);
					b0 = ldg_stream_v4((const int4 *) ((const int32_t *) P.filt[0].col + base + o0) + 1, pol_stream);
				}
				else
					pc_unpack8(ldg_stream_u64((const unsigned long long *) ((const uint8_t *) P.filt[0].col + base + o0), pol_stream), &a0, &b0);
			}
			if (P.nfilters > 1)
			{
				if (P.filt[1].width == 4)
				{
					a1 = ldg_stream_v4((const int4 *) ((const int32_t *) P.filt[1].col + base + o0), pol_stream);
					b1 = ldg_stream_v4((const int4 *) ((const int32_t *) P.filt[1].col + base + o0) + 1, pol_stream);
				}
				else
					pc_unpack8(ldg_stream_u64((const unsigned long long *) ((const uint8_t *) P.filt[1].col + base + o0), pol_stream), &a1, &b1);
			}
			if (P.visimap)
				vm = __ldg(P.visimap + ((base + o0) >> 3));
			am = vm;
			if (P.nfilters > 0)
				am &= pc_range8(a0, b0, P.filt[0].lo, P.filt[0].span);
			if (P.nfilters > 1)
				am &= pc_range8(a1, b1, P.filt[1].lo, P.filt[1].span);
		}
		else
			for (int u = 0; u < 8; u++)
			{
				const int64_t r = base + o0 + u;
				bool		alive = o0 + u < nvalid;

				if (alive && P.visimap)
					alive = (__ldg(P.visimap + (r >> 3)) >> (r & 7)) & 1;
				if (alive && P.nfilters > 0)
					alive = (unsigned) (pc_filter_value(P.filt[0], r) - P.filt[0].lo) <= P.filt[0].span;
				if (alive && P.nfilters > 1)
					alive = (unsigned) (pc_filter_value(P.filt[1], r) - P.filt[1].lo) <= P.filt[1].span;
				am |= (unsigned) alive << u;
			}
		for (int f = 0; f < P.nbloom && __any_sync(0xffffffffu, am != 0); f++)
		{
			if (SPEC && f == 0 && have0)
				am = P.bloom[0].width == 8 ? pc_bloom8_keys<true>(P.bloom[0], keys0, am) : pc_bloom8_keys<false>(P.bloom[0], keys0, am);
			else
				am = P.bloom[f].width == 8 ? pc_early_filter8<true>(P.bloom[f], base + o0, full, am, pol_stream)
					: pc_early_filter8<false>(P.bloom[f], base + o0, full, am, pol_stream);
		}
		__syncthreads();				/* s_cnt = 0 is in */
		{
			/* the tile's survivors, in row order within each warp: one scan + one shared atomic per warp */
			const unsigned c = __popc(am);
			unsigned	x = c;

#pragma unroll
			for (int d = 1; d < 32; d <<= 1)
			{
				const unsigned y = __shfl_up_sync(0xffffffffu, x, d);

				if (lane >= d)
					x += y;
			}
			const unsigned total = __shfl_sync(0xffffffffu, x, 31);
			unsigned	wb = 0;

			if (lane == 31 && total)
				wb = atomicAdd(&s_cnt, total);
			wb = __shfl_sync(0xffffffffu, wb, 31);
			unsigned	pos = wb + x - c;

#pragma unroll
			for (int u = 0; u < 8; u++)
				if ((am >> u) & 1)
					buf[pos++] = (uint32_t) (base + o0 + u);
		}
		__syncthreads();
		if (threadIdx.x == 0 && s_cnt)
			s_gbase = atomicAdd(P.out_count, (unsigned long long) s_cnt);
		__syncthreads();
		for (unsigned i = threadIdx.x; i < s_cnt; i += PC_THREADS)
			P.out[s_gbase + i] = buf[i];
		__syncthreads();				/* buf and s_cnt are free for the next tile */
	}
}

__global__ void __launch_bounds__(PC_THREADS, PC_OCC)
k_probe_chain(const __grid_constant__ PcParams P)
{
	__shared__ uint32_t q0[PC_Q0CAP];
	__shared__ PcProbe sprobe[PC_MAXP];	/* the stages read their probe through a pointer: keep it near */
	__shared__ unsigned cnt[PC_NQ];		/* entries waiting in queue k                                 */
	__shared__ int s_stage;
	__shared__ unsigned s_n, s_base;
	__shared__ long long s_tile;
	__shared__ unsigned long long s_obase;
	__shared__ PcPart part;
	__shared__ uint64_t s_tbar;			/* completion of the shared-memory tables' bulk copies                */
	extern __shared__ __align__(16) unsigned long long s_tables[];
	const int	np = P.np;
	const int	last = 2 * np + 1;		/* the sink's stage number; stage s reads queue s - 1         */
	const bool	iota = P.nfilters == 0 && P.visimap == NULL && P.nearly == 0;	/* always so with P.sel */
	const int64_t tile_rows = iota ? PC_BATCH : PC_TILE;
	const int64_t ntiles = (P.nrows + tile_rows - 1) / tile_rows;
	uint32_t   *const qg = P.qmem + (size_t) blockIdx.x * (size_t) P.q_cta_words;
	int64_t		next_tile = blockIdx.x;	/* thread 0's */

	if (threadIdx.x < PC_NQ)
		cnt[threadIdx.x] = 0;
	for (int i = threadIdx.x; i < (int) (np * sizeof(PcProbe) / sizeof(uint32_t)); i += PC_THREADS)
		((uint32_t *) sprobe)[i] = ((const uint32_t *) P.probe)[i];
	if (P.smem_table_bytes)
	{
		/* the small dimension tables: one TMA bulk copy each, global -> this CTA's shared memory; everybody waits on the
		 * transaction barrier once */
		if (threadIdx.x == 0)
		{
			mbar_init(&s_tbar, 1);
			asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		}
		__syncthreads();
		if (threadIdx.x == 0)
		{
			mbar_expect_tx(&s_tbar, P.smem_table_bytes);
			for (int j = 0; j < np; j++)
				if (P.probe[j].mode == 2)
					tma_load_1d(s_tables + P.probe[j].smem_off, P.probe[j].ht.slots, (P.probe[j].ht.mask + 1u) * 8u, &s_tbar);
		}
		mbar_wait(&s_tbar, 0);
	}
	for (;;)
	{
		__syncthreads();				/* the previous run's pushes are in */
		if (threadIdx.x == 0)
		{
			int			s = -1;
			bool		from_tile = false;

			/* the deepest stage with a full batch; else scan on; else drain front to back */
			for (int k = last; k >= 1; k--)
				if (cnt[k - 1] >= PC_BATCH)
				{
					s = k;
					break;
				}
			if (s < 0)
			{
				if (next_tile < ntiles)
				{
					s = iota ? 1 : 0;
					from_tile = true;
					s_tile = next_tile;
					next_tile += gridDim.x;
				}
				else
					for (int k = 1; k <= last; k++)
						if (cnt[k - 1] > 0)
						{
							s = k;
							break;
						}
			}
			if (s >= 1 && !from_tile)
			{
				const unsigned c = cnt[s - 1];
				const unsigned n = c < PC_BATCH ? c : PC_BATCH;

				s_n = n;
				s_base = c - n;			/* the newest n entries */
				cnt[s - 1] = c - n;
			}
			s_stage = from_tile ? -2 - s : s;	/* -2: F, -3: B_0 straight from the tile */
		}
		__syncthreads();
		const int	code = s_stage;

		if (code == -1)
			break;
		if (code == -2)
		{
			/* stage F: ExecQual on a tile of driving rows.  A thread owns 8 consecutive rows: its qual
			 * columns arrive as two 16-byte loads each, issued before any is used; the survivors of
			 * a warp's 256 rows go to queue 0 in row order with one warp scan and one atomic. */
			const int64_t base = s_tile * PC_TILE;
			const unsigned nvalid = (unsigned) (P.nrows - base < PC_TILE ? P.nrows - base : PC_TILE);
			const unsigned o0 = threadIdx.x * 8;
			const int	lane = threadIdx.x & 31;
			const uint64_t pol_stream = l2_policy_evict_first();
			const bool	full = o0 + 8 <= nvalid;
			const bool	wide0 = sprobe[0].kind == 1;
			unsigned	am = 0;

			if (full)
			{
				int4		a0 = make_int4(0, 0, 0, 0), b0 = a0, a1 = a0, b1 = a0;
				unsigned	vm = 0xff;

				/* 8 rows of a 4-byte column are two 16-byte loads, of a 1-byte column one 8-byte load */
				if (P.nfilters > 0)
				{
					if (P.filt[0].width == 4)
					{
						a0 = ldg_stream_v4((const int4 *) ((const int32_t *) P.filt[0].col + base + o0), pol_stream);
						b0 = ldg_stream_v4((const int4 *) ((const int32_t *) P.filt[0].col + base + o0) + 1, pol_stream);
					}
					else
						pc_unpack8(ldg_stream_u64((const unsigned long long *) ((const uint8_t *) P.filt[0].col + base + o0), pol_stream), &a0, &b0);
				}
				if (P.nfilters > 1)
				{
					if (P.filt[1].width == 4)
					{
						a1 = ldg_stream_v4((const int4 *) ((const int32_t *) P.filt[1].col + base + o0), pol_stream);
						b1 = ldg_stream_v4((const int4 *) ((const int32_t *) P.filt[1].col + base + o0) + 1, pol_stream);
					}
					else
						pc_unpack8(ldg_stream_u64((const unsigned long long *) ((const uint8_t *) P.filt[1].col + base + o0), pol_stream), &a1, &b1);
				}
				if (P.visimap)
					vm = __ldg(P.visimap + ((base + o0) >> 3));
				am = vm;
				if (P.nfilters > 0)
					am &= pc_range8(a0, b0, P.filt[0].lo, P.filt[0].span);
				if (P.nfilters > 1)
					am &= pc_range8(a1, b1, P.filt[1].lo, P.filt[1].span);
			}
			else
				for (int u = 0; u < 8; u++)
				{
					const int64_t r = base + o0 + u;
					bool		alive = o0 + u < nvalid;

					if (alive && P.visimap)
						alive = (__ldg(P.visimap + (r >> 3)) >> (r & 7)) & 1;
					if (alive && P.nfilters > 0)
						alive = (unsigned) (pc_filter_value(P.filt[0], r) - P.filt[0].lo) <= P.filt[0].span;
					if (alive && P.nfilters > 1)
						alive = (unsigned) (pc_filter_value(P.filt[1], r) - P.filt[1].lo) <= P.filt[1].span;
					am |= (unsigned) alive << u;
				}
			/* scan-level runtime filters: the key columns of the rows still alive, 8 filter words in flight */
			for (int f = 0; f < P.nearly && __any_sync(0xffffffffu, am != 0); f++)
				am = P.early[f].width == 8 ? pc_early_filter8<true>(P.early[f], base + o0, full, am, pol_stream)
					: pc_early_filter8<false>(P.early[f], base + o0, full, am, pol_stream);
			/* every lane votes (full-mask).  Only a warp whose rows mostly survived runs probe 0 here: its 8 hashes and
			 * filter words per thread are work for live rows.  A sparse warp hands its few survivors to queue 0, where
			 * stage B_0 will see them packed into full batches. */
			if (P.fuse0 && pc_warp_dense(full, am, 96u))
			{
				if (wide0)
					pc_stage_f_probe0<true>(sprobe[0], base + o0, pc_keys8_vec<true>(sprobe[0].key[0].data, base + o0, pol_stream), am,
											qg + P.q_off[1], (unsigned) P.q_cap[1], &cnt[1]);
				else
					pc_stage_f_probe0<false>(sprobe[0], base + o0, pc_keys8_vec<false>(sprobe[0].key[0].data, base + o0, pol_stream), am,
											 qg + P.q_off[1], (unsigned) P.q_cap[1], &cnt[1]);
				continue;
			}
			const unsigned c = __popc(am);
			unsigned	x = c;

#pragma unroll
			for (int d = 1; d < 32; d <<= 1)
			{
				const unsigned y = __shfl_up_sync(0xffffffffu, x, d);

				if (lane >= d)
					x += y;
			}
			const unsigned total = __shfl_sync(0xffffffffu, x, 31);
			unsigned	wb = 0;

			if (lane == 31 && total)
				wb = atomicAdd(&cnt[0], total);
			wb = __shfl_sync(0xffffffffu, wb, 31);
			unsigned	pos = wb + x - c;

#pragma unroll
			for (int u = 0; u < 8; u++)
				if ((am >> u) & 1)
					q0[pos++] = (uint32_t) (base + o0 + u);
			continue;
		}
		int			s = code;
		PcQ			Q;
		unsigned	n = s_n,
					base = s_base;

		if (code == -3)
		{
			const int64_t tb = s_tile * PC_BATCH;

			s = 1;
			Q.q = NULL;
			Q.cap = 0;
			Q.iota_base = (uint32_t) tb;
			Q.sel = P.sel;
			n = (unsigned) (P.nrows - tb < PC_BATCH ? P.nrows - tb : PC_BATCH);
			base = 0;
		}
		else if (s == 1)
		{
			Q.q = q0;
			Q.cap = PC_Q0CAP;
			Q.iota_base = 0;
			Q.sel = NULL;
		}
		else
		{
			Q.q = qg + P.q_off[s - 1];
			Q.cap = (uint32_t) P.q_cap[s - 1];
			Q.iota_base = 0;
			Q.sel = NULL;
		}
		if (s == last)
			pc_stage_sink(P, Q, base, n, &s_obase, &part);
		else
		{
			const int	j = (s - 1) >> 1;
			const PcProbe &pr = sprobe[j];
			uint32_t   *out = qg + P.q_off[s];

			if ((s & 1) && pr.mode != 0)
			{
				/* one stage for this probe: straight into queue 2j + 2 */
				const unsigned long long *slots = pr.mode == 2 ? s_tables + pr.smem_off : pr.ht.slots;
				uint32_t   *out2 = qg + P.q_off[s + 1];

				if (pr.kind == 0)
					pc_stage_direct<0>(pr, j, Q, base, n, out2, (unsigned) P.q_cap[s + 1], &cnt[s + 1], slots);
				else if (pr.kind == 1)
					pc_stage_direct<1>(pr, j, Q, base, n, out2, (unsigned) P.q_cap[s + 1], &cnt[s + 1], slots);
				else
					pc_stage_direct<2>(pr, j, Q, base, n, out2, (unsigned) P.q_cap[s + 1], &cnt[s + 1], slots);
			}
			else if (s & 1)
			{
				if (pr.kind == 0)
					pc_stage_bloom<0>(pr, j, Q, base, n, out, (unsigned) P.q_cap[s], &cnt[s]);
				else if (pr.kind == 1)
					pc_stage_bloom<1>(pr, j, Q, base, n, out, (unsigned) P.q_cap[s], &cnt[s]);
				else
					pc_stage_bloom<2>(pr, j, Q, base, n, out, (unsigned) P.q_cap[s], &cnt[s]);
			}
			else
			{
				if (pr.kind == 0)
					pc_stage_ht<0>(pr, j, Q, base, n, out, (unsigned) P.q_cap[s], &cnt[s]);
				else if (pr.kind == 1)
					pc_stage_ht<1>(pr, j, Q, base, n, out, (unsigned) P.q_cap[s], &cnt[s]);
				else
					pc_stage_ht<2>(pr, j, Q, base, n, out, (unsigned) P.q_cap[s], &cnt[s]);
			}
		}
	}
}

/* ---------------------------------------------------------------------------------------------
 * matcher
 * --------------------------------------------------------------------------------------------- */
static bool
pc_col(const CbPipeline *p, int c, PcCol *out, int base)
{
	if (p->cols[c].nulls != NULL || p->cols[c].type == CB_FLOAT8 || p->cols[c].type == CB_NUMERIC128)
		return false;
	out->data = p->cols[c].data;
	out->dict = p->cols[c].dict_hash;
	out->type = p->cols[c].type;
	out->src = p->cols[c].src == 0 ? 0 : p->cols[c].src - base + 1;
	return true;
}

/* Bloom filter over key column `kc` of probe k's build side, restricted to the build rows that can still find a
 * partner in every later INNER probe whose keys all come from that same build side (`red`): a row of the driving scan
 * whose key misses it can never reach the sink - probe k would drop it, or a later probe would */
struct PcEarlyBuild
{
	int64_t		nrows;			/* rows of probe k's inner relation                                   */
	HtDev		self;			/* probe k's table: key columns / NULL maps of the build side         */
	int32_t		kc;
	int32_t		hashtype;
	int32_t		nred;
	HtDev		red[PC_MAXP];
	int32_t		red_nkeys[PC_MAXP];
	PcCol		red_key[PC_MAXP][2];	/* columns of the build relation (indexed by its row)             */
	int32_t		red_keytype[PC_MAXP][2];
	uint32_t   *bloom;			/* NULL: only count the rows that would go in                         */
	uint32_t	mask;
	unsigned long long *passed;
};

__global__ void
k_pc_early_build(PcEarlyBuild B)
{
	for (int64_t r = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; r < B.nrows; r += (int64_t) gridDim.x * blockDim.x)
	{
		bool		ok = true;

		for (int k = 0; k < B.self.nkeys; k++)
			if (B.self.keynulls[k] && B.self.keynulls[k][r])
				ok = false;		/* never inserted into probe k's table (nodeHash.c:2161) */
		for (int m = 0; m < B.nred && ok; m++)
		{
			const HtDev &T = B.red[m];
			int64_t		kv[2] = {0, 0};
			uint32_t	h = 0;
			bool		found = false;

			for (int i = 0; i < B.red_nkeys[m]; i++)
			{
				kv[i] = cb_load_widen(B.red_key[m][i].data, B.red_key[m][i].type, (uint32_t) r);
				h = pg_hash_combine(h, jh_hash_datum(B.red_keytype[m][i], kv[i], B.red_key[m][i].dict), false);
			}
			uint32_t	pos = h & T.mask;

			for (; !(T.keyslot && !ht_key_in_domain(T.keyslot, kv[0]));)
			{
				const unsigned long long e = T.slots[pos];

				if (e == HT_EMPTY)
					break;
				if ((uint32_t) (e >> 32) == (T.keyslot ? (uint32_t) kv[0] : h))
				{
					const uint32_t ir = (uint32_t) e;

					if (T.keyslot || (cb_load_widen(T.keydata[0], T.keytype[0], ir) == kv[0] &&
									  (B.red_nkeys[m] < 2 || cb_load_widen(T.keydata[1], T.keytype[1], ir) == kv[1])))
					{
						found = true;
						break;
					}
				}
				pos = (pos + 1) & T.mask;
			}
			ok = found;
		}
		if (ok && !B.bloom)
			atomicAdd(B.passed, 1ull);
		if (ok && B.bloom)
		{
			uint32_t	w;
			const int64_t kv = cb_load_widen(B.self.keydata[B.kc], B.self.keytype[B.kc], (uint32_t) r);
			const uint32_t bits = ht_bloom_bits(pg_hash_combine(0u, jh_hash_datum(B.hashtype, kv, NULL), false), &w, B.mask);

			atomicOr(B.bloom + w, bits);
		}
	}
}

#define PC_REJECT(n) \
	do { \
		if (ctx->opt_debug) \
			fprintf(stderr, "k_probe_chain: pipeline not matched (reason %d, line %d)\n", n, __LINE__); \
		return CBGPU_OK; \
	} while (0)

int
cb_try_probe_chain(cbgpu_ctx *ctx, const CbPipeline *p, const PipeDev *d, bool *handled)
{
	XProg	   *xp = (XProg *) cb_scratch(ctx, 2, sizeof(XProg));
	PcParams   *Pp = (PcParams *) cb_scratch(ctx, 3, sizeof(PcParams));
	if (!xp || !Pp)
		return CBGPU_ERR_NOMEM;
	XProg	   &x = *xp;
	PcParams   &P = *Pp;
	const CbpSink *s = &p->sink;
	int			np = 0;
	int			base = 1;
	int			term_node[2] = {-1, -1};

	*handled = false;
	if (p->nprobes < 0 || p->nprobes > PC_MAXP || p->drv_nsrc != 0)
		PC_REJECT(1);		/* no probes at all is fine: quals -> sink (a filtered scan feeding a Hash or a Motion) */
	if (s->kind != CBP_SINK_AGG && s->kind != CBP_SINK_MATERIALIZE && s->kind != CBP_SINK_PARTITION)
		PC_REJECT(2);
	if (s->kind == CBP_SINK_PARTITION && s->nsegs > 64)
		PC_REJECT(2);
	if (!xm_decompile(p, &x))
		PC_REJECT(3);
	memset(&P, 0, sizeof(P));
	/* sections: quals (before the first probe only), then the probes in program order */
	for (int i = 0; i < x.nsections; i++)
	{
		XSection   *sec = &x.sections[i];

		if (sec->kind == 0)
		{
			int			code, col;
			int64_t		v, lo = INT32_MIN, hi = INT32_MAX;

			if (np > 0)
				PC_REJECT(4);	/* a qual behind a join: generic kernel */
			if (!xm_is_cmp_const(&x, sec->node, &code, &col, &v) || p->cols[col].src != 0 || p->cols[col].nulls ||
				(cb_type_w(p->cols[col].type) != 4 && cb_type_w(p->cols[col].type) != 1))
				PC_REJECT(5);
			if (cb_type_w(p->cols[col].type) == 1)
			{
				/* 1-byte columns hold unsigned values (cb_load_widen): clamp the range to them */
				lo = 0;
				hi = 255;
			}
			switch (code)
			{
				case CBP_EQ: lo = hi = v; break;
				case CBP_LT: hi = v - 1; break;
				case CBP_LE: hi = v; break;
				case CBP_GT: lo = v + 1; break;
				case CBP_GE: lo = v; break;
				default: PC_REJECT(6);
			}
			if (lo > INT32_MAX || hi < INT32_MIN || lo > hi)
				PC_REJECT(7);
			if (hi > INT32_MAX)
				hi = INT32_MAX;
			if (lo < INT32_MIN)
				lo = INT32_MIN;
			if (((uintptr_t) p->cols[col].data & 15) != 0)
				PC_REJECT(100);		/* stage F reads the qual columns 16 bytes at a time */
			{
				int			f = P.nfilters;

				/* a second qual on the same column narrows the first one's range (date BETWEEN) */
				for (int g = 0; g < P.nfilters; g++)
					if (P.filt[g].col == p->cols[col].data)
					{
						const int64_t olo = P.filt[g].lo,
									ohi = olo + (int64_t) P.filt[g].span;

						lo = lo > olo ? lo : olo;
						hi = hi < ohi ? hi : ohi;
						f = g;
					}
				if (lo > hi)
					PC_REJECT(7);
				if (f == P.nfilters && P.nfilters >= 2)
					PC_REJECT(4);
				P.filt[f].col = p->cols[col].data;
				P.filt[f].width = cb_type_w(p->cols[col].type);
				P.filt[f].lo = (int32_t) lo;
				P.filt[f].span = (uint32_t) (hi - lo);
				if (f == P.nfilters)
					P.nfilters++;
			}
		}
		else
		{
			const CbpProbe *pp = &p->probes[sec->probe];
			PcProbe    *q = &P.probe[np];

			if (sec->probe != np || pp->nkeys > 2)
				PC_REJECT(8);
			if (pp->jointype != CB_JOIN_INNER && pp->jointype != CB_JOIN_SEMI && pp->jointype != CB_JOIN_ANTI)
				PC_REJECT(9);
			if ((pp->jointype != CB_JOIN_INNER) && np != p->nprobes - 1)
				PC_REJECT(10);	/* semi / anti only as the last probe (its inner side has no columns) */
			q->ht = d->probes[np].ht;
			q->nkeys = pp->nkeys;
			q->jointype = pp->jointype;
			if (!q->ht.bloom)
				PC_REJECT(11);
			for (int k = 0; k < pp->nkeys; k++)
			{
				int			col;

				if (!xm_is_load(&x, sec->keys[k], &col) || !pc_col(p, col, &q->key[k], base))
					PC_REJECT(12);
				if (q->key[k].src > np)
					PC_REJECT(13);
				q->keytype[k] = pp->keytype[k];
				q->key[k].type = p->cols[col].type;
				if (q->ht.keynulls[k])
					PC_REJECT(14);
			}
			if (pp->nkeys == 1 && (q->key[0].type == CB_INT4 || q->key[0].type == CB_DATE) &&
				(q->keytype[0] == CB_INT4 || q->keytype[0] == CB_DATE))
				q->kind = 0;
			else if (pp->nkeys == 1 && q->key[0].type == CB_INT8 && q->keytype[0] == CB_INT8)
				q->kind = 1;
			else
				q->kind = 2;
			np++;
		}
	}
	if (np != p->nprobes)
		PC_REJECT(15);
	P.np = np;
	P.nrows = p->nrows;
	P.visimap = p->visimap;
	P.status = ctx->d_status;
	P.sink_kind = s->kind;
	if (s->kind == CBP_SINK_AGG)
	{
		if (x.depth < s->nkeys)
			PC_REJECT(16);
		P.agg = d->sink.agg;
		P.nkeys = s->nkeys;
		for (int k = 0; k < s->nkeys; k++)
		{
			int			col;

			if (!xm_is_load(&x, x.stack[k], &col) || !pc_col(p, col, &P.key[k], base))
				PC_REJECT(17);
			P.key[k].type = s->keytype[k];
			P.key[k].dict = s->key_dict_hash[k];
		}
		P.naccs = s->naccs;
		for (int a = 0; a < s->naccs; a++)
		{
			int			node, col, b, c;
			int64_t		k;
			int			t = -1;

			if (s->accs[a].kind == CBP_ACC_COUNT && s->accs[a].arg < 0)
			{
				P.acc_term[a] = -1;
				continue;
			}
			if (s->accs[a].kind != CBP_ACC_SUM_INT)
				PC_REJECT(18);
			node = x.stack[s->nkeys + s->accs[a].arg];
			for (int u = 0; u < P.nterms; u++)
				if (term_node[u] == node)
					t = u;
			if (t >= 0)
			{
				P.acc_term[a] = t;	/* aggregates over the same expression share the value */
				continue;
			}
			if (P.nterms >= 2)
				PC_REJECT(19);
			t = P.nterms;
			term_node[t] = node;
			if (xm_is_rev(&x, node, &b, &k, &c))
			{
				P.term_kind[t] = 1;
				P.term_k[t] = k;
				if (!pc_col(p, b, &P.term_a[t], base) || !pc_col(p, c, &P.term_b[t], base))
					PC_REJECT(20);
			}
			else if ((x.nodes[node].code == CBP_SUB || x.nodes[node].code == CBP_ADD) && xm_is_load(&x, x.nodes[node].l, &b) &&
					 xm_is_load(&x, x.nodes[node].r, &c))
			{
				P.term_kind[t] = x.nodes[node].code == CBP_SUB ? 2 : 3;
				if (!pc_col(p, b, &P.term_a[t], base) || !pc_col(p, c, &P.term_b[t], base))
					PC_REJECT(30);
			}
			else if (xm_is_load(&x, node, &col))
			{
				P.term_kind[t] = 0;
				if (!pc_col(p, col, &P.term_a[t], base))
					PC_REJECT(21);
			}
			else
				PC_REJECT(22);
			P.nterms++;
			P.acc_term[a] = t;
		}
	}
	else
	{
		if (s->nout > PC_MAXOUT || x.depth != s->nout)
			PC_REJECT(23);
		P.nout = s->nout;
		for (int c = 0; c < s->nout; c++)
		{
			int			col;

			if (!xm_is_load(&x, x.stack[c], &col) || !pc_col(p, col, &P.out[c], base) || d->sink.outnull[c])
				PC_REJECT(24);
			P.outcol[c] = d->sink.outcol[c];
			P.outtype[c] = d->sink.outtype[c];
		}
		P.out_count = d->sink.out_count;
		P.out_capacity = d->sink.out_capacity;
		if (s->kind == CBP_SINK_PARTITION)
		{
			P.nhash = d->sink.nhash;
			P.nsegs = d->sink.nsegs;
			P.seg_capacity = d->sink.seg_capacity;
			P.part_cols = d->sink.part_cols;
			P.part_counts = d->sink.part_counts;
			P.part_flags = d->sink.part_flags;
			for (int g = 0; g < P.nsegs && g < 64; g++)
			{
				P.seg_base[g] = d->sink.seg_base[g];
				P.seg_cap[g] = d->sink.seg_cap[g];
			}
			for (int k = 0; k < P.nhash; k++)
			{
				P.hashtype[k] = d->sink.hashtype[k];
				P.hashdict[k] = d->sink.hashdict[k];
			}
		}
	}

	/* scan-level runtime filters.  The reference pushes a Bloom filter per integer hash-clause column down to the
	 * SeqScan the column comes from (CreateRuntimeFilter / FindTargetNodes, nodeHashjoin.c:2217,2407).  Probe k's own
	 * filter is consulted in stage B_k anyway; what stage F can add is a filter that knows MORE than probe k's build
	 * side: the build rows that also survive the later probes keyed only by that build side's columns (a dimension
	 * joined to its sub-dimension further up the plan).  Rows of the scan that miss it are dropped before the first
	 * hash-table access instead of after several. */
	void	   *early_mem[PC_MAXEARLY] = {NULL, NULL};

	for (int k = 0; k < np && P.nearly < PC_MAXEARLY; k++)
	{
		PcEarlyBuild *Bp = (PcEarlyBuild *) cb_scratch(ctx, 4, sizeof(PcEarlyBuild));
		if (!Bp)
			return CBGPU_ERR_NOMEM;
		PcEarlyBuild &B = *Bp;
		PcProbe    *q = &P.probe[k];
		const cbgpu_rel *inner = p->probes[k].ht->inner;
		int			kc = -1;
		int64_t		words = 32;

		memset(&B, 0, sizeof(B));
		if (q->jointype != CB_JOIN_INNER || !inner || inner->nrows < 1)
			continue;
		for (int m = k + 1; m < np; m++)
		{
			bool		all = P.probe[m].jointype == CB_JOIN_INNER;

			for (int i = 0; i < P.probe[m].nkeys; i++)
				if (P.probe[m].key[i].src != k + 1)
					all = false;
			if (!all)
				continue;
			B.red[B.nred] = P.probe[m].ht;
			B.red_nkeys[B.nred] = P.probe[m].nkeys;
			for (int i = 0; i < P.probe[m].nkeys; i++)
			{
				B.red_key[B.nred][i] = P.probe[m].key[i];
				B.red_keytype[B.nred][i] = P.probe[m].keytype[i];
			}
			B.nred++;
		}
		if (B.nred == 0)
			continue;
		for (int i = 0; i < q->nkeys && kc < 0; i++)
			if (q->key[i].src == 0 && (q->key[i].type == CB_INT4 || q->key[i].type == CB_DATE || q->key[i].type == CB_INT8))
				kc = i;
		if (kc < 0)
			continue;
		{
			/* worth it only if the later probes thin the build side out: try the first 64 K build rows - once per
			 * (build side, shape of the reducing tables): the sample costs a host round trip, and its answer stands
			 * while the tables do (the decision is about speed, never about results) */
			unsigned long long *d_passed,
						h_passed = 0;
			const int64_t sample = inner->nrows < 65536 ? inner->nrows : 65536;
			const void *sig = (const void *) (uintptr_t) ((uintptr_t) B.red[0].mask * 31u + (uintptr_t) B.nred * 7u + (uintptr_t) B.red[0].keytype[0]);
			int			known = -1;

			for (int i = 0; i < ctx->early_cache_n; i++)
				if (ctx->early_cache[i].keydata == q->ht.keydata[kc] && ctx->early_cache[i].nrows == inner->nrows && ctx->early_cache[i].red0 == sig)
					known = ctx->early_cache[i].worth;
			if (known < 0)
			{
				CB_CUDA(ctx, cudaMallocAsync(&d_passed, sizeof(*d_passed), ctx->stream));
				CB_CUDA(ctx, cudaMemsetAsync(d_passed, 0, sizeof(*d_passed), ctx->stream));
				B.nrows = sample;
				B.self = q->ht;
				B.kc = kc;
				B.hashtype = q->keytype[kc];
				B.bloom = NULL;
				B.passed = d_passed;
				k_pc_early_build<<<(int) ((sample + 255) / 256), 256, 0, ctx->stream>>>(B);
				CB_LAUNCHED(ctx, "k_pc_early_build");
				CB_CUDA(ctx, cudaMemcpyAsync(&h_passed, d_passed, sizeof(h_passed), cudaMemcpyDeviceToHost, ctx->stream));
				CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
				CB_CUDA(ctx, cudaFreeAsync(d_passed, ctx->stream));
				known = (int64_t) h_passed * 2 <= sample;
				{
					const int	slot = ctx->early_cache_n < CB_EARLY_CACHE ? ctx->early_cache_n++ : (int) (inner->nrows % CB_EARLY_CACHE);

					ctx->early_cache[slot].keydata = q->ht.keydata[kc];
					ctx->early_cache[slot].nrows = inner->nrows;
					ctx->early_cache[slot].red0 = sig;
					ctx->early_cache[slot].worth = known;
				}
			}
			if (!known)
				continue;
		}
		while (words < inner->nrows / 2)
			words <<= 1;
		CB_CUDA(ctx, cudaMallocAsync(&early_mem[P.nearly], (size_t) words * sizeof(uint32_t), ctx->stream));
		CB_CUDA(ctx, cudaMemsetAsync(early_mem[P.nearly], 0, (size_t) words * sizeof(uint32_t), ctx->stream));
		B.nrows = inner->nrows;
		B.self = q->ht;
		B.kc = kc;
		B.hashtype = q->keytype[kc];
		B.bloom = (uint32_t *) early_mem[P.nearly];
		B.mask = (uint32_t) (words - 1);
		{
			int			eb = (int) ((inner->nrows + 255) / 256);

			if (eb > ctx->sm_count * 8)
				eb = ctx->sm_count * 8;
			k_pc_early_build<<<eb, 256, 0, ctx->stream>>>(B);
			CB_LAUNCHED(ctx, "k_pc_early_build");
		}
		P.early[P.nearly].col = q->key[kc].data;
		P.early[P.nearly].width = cb_type_w(q->key[kc].type);
		P.early[P.nearly].hashtype = q->keytype[kc];
		P.early[P.nearly].bloom = B.bloom;
		P.early[P.nearly].mask = B.mask;
		P.nearly++;
	}
	/* ---- a selective head over a big scan runs as its own lean kernel (k_prefilter); the chain starts from its survivors ---- */
	uint32_t   *pf_sel = NULL;
	unsigned long long *pf_count = NULL;
	bool		pf_bloom_done[PC_MAXP] = {false, false, false, false};	/* probe j's Bloom filter was applied by the prefilter pass */
	bool		pf_cand[PC_MAXP] = {false, false, false, false};

	if (P.nrows >= ctx->opt_pf_min_rows && np >= 1)	/* below ~16 M rows the fused kernel's fixed costs win */
	{
		PfParams   *Fp = (PfParams *) cb_scratch(ctx, 6, sizeof(PfParams));

		if (!Fp)
			return CBGPU_ERR_NOMEM;
		PfParams   &F = *Fp;
		const uint64_t sig = (uint64_t) (uintptr_t) (P.nfilters ? P.filt[0].col : NULL) ^ ((uint64_t) (uintptr_t) P.probe[0].key[0].data << 1) ^
			((uint64_t) P.nrows << 20) ^ (uint64_t) P.nfilters ^ ((uint64_t) np << 4) ^ ((uint64_t) P.nearly << 8);
		bool		known_unselective = false;

		memset(&F, 0, sizeof(F));
		F.nrows = P.nrows;
		F.visimap = P.visimap;
		F.nfilters = P.nfilters;
		F.filt[0] = P.filt[0];
		F.filt[1] = P.filt[1];
		for (int f = 0; f < P.nearly; f++)
			F.bloom[F.nbloom++] = P.early[f];
		for (int j = 0; j < np && F.nbloom < PF_MAXBLOOM; j++)
		{
			const PcProbe &q = P.probe[j];

			if ((q.jointype != CB_JOIN_INNER && q.jointype != CB_JOIN_SEMI) || q.nkeys != 1 || (q.kind != 0 && q.kind != 1) ||
				q.key[0].src != 0 || !q.ht.bloom || ((uintptr_t) q.key[0].data & 15) != 0)
				continue;
			F.bloom[F.nbloom].col = q.key[0].data;
			F.bloom[F.nbloom].width = q.kind == 1 ? 8 : 4;
			F.bloom[F.nbloom].hashtype = q.keytype[0];
			F.bloom[F.nbloom].bloom = q.ht.bloom;
			F.bloom[F.nbloom].mask = q.ht.bloom_mask;
			F.nbloom++;
			pf_cand[j] = true;
		}
		for (int i = 0; i < ctx->pf_cache_n; i++)
			if (ctx->pf_cache[i] == sig)
				known_unselective = true;
		if (F.nbloom + F.nfilters > 0 && !known_unselective)
		{
			unsigned long long nsel = 0;
			const int64_t ft = (P.nrows + PC_TILE - 1) / PC_TILE;

			CB_CUDA(ctx, cudaMallocAsync(&pf_sel, (size_t) P.nrows * sizeof(uint32_t), ctx->stream));
			CB_CUDA(ctx, cudaMallocAsync(&pf_count, sizeof(unsigned long long), ctx->stream));
			CB_CUDA(ctx, cudaMemsetAsync(pf_count, 0, sizeof(unsigned long long), ctx->stream));
			F.out = pf_sel;
			F.out_count = pf_count;
			const int	pkl = cb_klog_begin(ctx, "k_prefilter");

			/* 32 registers per thread: all 64 warps of an SM resident - this pass lives on occupancy.  CBGPU_PF_SPEC trades
			 * that for the first filter's keys requested together with the qual columns (64 registers, 4 CTAs per SM). */
			if (ctx->opt_pf_spec)
				k_prefilter<true><<<ctx->sm_count * 4 < ft ? ctx->sm_count * 4 : (int) ft, PC_THREADS, 0, ctx->stream>>>(F);
			else
				k_prefilter<false><<<ctx->sm_count * 8 < ft ? ctx->sm_count * 8 : (int) ft, PC_THREADS, 0, ctx->stream>>>(F);
			CB_LAUNCHED(ctx, "k_prefilter");
			cb_klog_end(ctx, pkl);
			CB_CUDA(ctx, cudaMemcpyAsync(&nsel, pf_count, sizeof(nsel), cudaMemcpyDeviceToHost, ctx->stream));
			CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
			if (ctx->opt_debug)
				fprintf(stderr, "k_prefilter: %lld of %lld rows survive %d qual(s) + %d filter(s)\n", (long long) nsel, (long long) P.nrows, F.nfilters, F.nbloom);
			/* worth it only when few rows survive: the chain over the survivors is latency-bound and, run on its own, no
			 * longer hides behind the scan as it does inside the fused kernel (opt_pf_keep_div: at most a twelfth of the
			 * rows by default) */
			if (nsel * (unsigned long long) ctx->opt_pf_keep_div <= (unsigned long long) P.nrows)
			{
				P.sel = pf_sel;
				P.nrows = (int64_t) nsel;
				P.nfilters = 0;
				P.visimap = NULL;
				P.nearly = 0;
				for (int j = 0; j < np; j++)
					pf_bloom_done[j] = pf_cand[j];
			}
			else
			{
				/* it cut too little to pay for a second pass over its survivors: the fused kernel does the whole job, and the
				 * next run of this pipeline does not ask again */
				if (ctx->pf_cache_n < (int) (sizeof(ctx->pf_cache) / sizeof(ctx->pf_cache[0])))
					ctx->pf_cache[ctx->pf_cache_n++] = sig;
			}
		}
	}
	/* persistent grid: 4 CTAs per SM; queue k >= 1 holds (k + 3) / 2 words per entry */
	const bool	iota = P.nfilters == 0 && P.visimap == NULL && P.nearly == 0;
	const int64_t ntiles = (P.nrows + (iota ? PC_BATCH : PC_TILE) - 1) / (iota ? PC_BATCH : PC_TILE);
	int			blocks = ctx->sm_count * PC_OCC;
	int64_t		words = 0;

	if (blocks > ntiles)
		blocks = (int) ntiles;
	if (blocks < 1)
		blocks = 1;				/* nothing survived the prefilter: one CTA finds no tile and leaves */
	/* how each table is reached (PcProbe.mode): a few thousand slots -> staged into shared memory by TMA (32 KB per CTA for
	 * all of them together: four CTAs per SM stay resident); everything else Bloom filter first, then the table, unless the
	 * prefilter pass applied that filter already */
	{
		uint32_t	smem_slots = 0;

		for (int j = 0; j < np; j++)
		{
			const uint64_t bytes = ((uint64_t) P.probe[j].ht.mask + 1) * 8;

			P.probe[j].mode = 0;
			if (bytes <= 32768 && (smem_slots * 8 + bytes) <= 32768 && ((uintptr_t) P.probe[j].ht.slots & 15) == 0)
			{
				P.probe[j].mode = 2;
				P.probe[j].smem_off = (int32_t) smem_slots;
				smem_slots += (uint32_t) (bytes / 8);
			}
			else if (pf_bloom_done[j])
				P.probe[j].mode = 1;	/* the rows that reach it passed its Bloom filter in the prefilter pass: straight to the table */
		}
		P.smem_table_bytes = smem_slots * 8;
	}
	/* probe 0 rides in stage F when its one integer key is a column of the driving relation that can be read 16 bytes at
	 * a time, and stage F exists at all (without quals / visimap / scan-level filters the tiles start at B_0 already) */
	P.fuse0 = !iota && np >= 1 && P.probe[0].mode == 0 && P.probe[0].nkeys == 1 && (P.probe[0].kind == 0 || P.probe[0].kind == 1) &&
		P.probe[0].key[0].src == 0 && ((uintptr_t) P.probe[0].key[0].data & 15) == 0;
	for (int k = 1; k <= 2 * np; k++)
	{
		P.q_off[k] = (int32_t) words;
		P.q_cap[k] = (k == 1 && P.fuse0) ? PC_Q0CAP : PC_QCAP;
		words += (int64_t) P.q_cap[k] * ((k + 3) / 2);
	}
	P.q_cta_words = words;
	CB_CUDA(ctx, cudaMallocAsync(&P.qmem, (size_t) blocks * (size_t) (words ? words : 1) * sizeof(uint32_t), ctx->stream));
	if (ctx->opt_debug)
		fprintf(stderr, "k_probe_chain: modes %d %d %d %d (0 filter + HBM table, 1 table only, 2 table in shared memory: %u bytes) fuse0 %d\n",
				P.probe[0].mode, P.probe[1].mode, P.probe[2].mode, P.probe[3].mode, P.smem_table_bytes, P.fuse0);
	if (ctx->opt_debug)
		fprintf(stderr, "k_probe_chain: np %d nrows %lld tiles %lld blocks %d queue words/CTA %lld filters %d sink %d kinds %d %d %d %d\n", np,
				(long long) P.nrows, (long long) ntiles, blocks, (long long) words, P.nfilters, P.sink_kind, P.probe[0].kind,
				P.probe[1].kind, P.probe[2].kind, P.probe[3].kind);
	if (ctx->opt_debug && P.nearly)
		fprintf(stderr, "k_probe_chain: %d scan-level runtime filter(s)\n", P.nearly);
	CB_CUDA(ctx, cudaEventRecord(ctx->ev_k0, ctx->stream));
	int			kl = cb_klog_begin(ctx, "k_probe_chain");

	{
		static bool attr_done = false;	/* idempotent: a race between two contexts sets the same value twice */

		if (!attr_done)
		{
			CB_CUDA(ctx, cudaFuncSetAttribute(k_probe_chain, cudaFuncAttributeMaxDynamicSharedMemorySize, 32768));
			attr_done = true;
		}
	}
	k_probe_chain<<<blocks, PC_THREADS, P.smem_table_bytes, ctx->stream>>>(P);
	ctx->last_kernel_name = "k_probe_chain";
	if (kl >= 0)
		ctx->klog_name[kl] = ctx->last_kernel_name;
	CB_LAUNCHED(ctx, "k_probe_chain");
	cb_klog_end(ctx, kl);
	CB_CUDA(ctx, cudaEventRecord(ctx->ev_k1, ctx->stream));
	CB_CUDA(ctx, cudaFreeAsync(P.qmem, ctx->stream));
	if (pf_sel)
		CB_CUDA(ctx, cudaFreeAsync(pf_sel, ctx->stream));
	if (pf_count)
		CB_CUDA(ctx, cudaFreeAsync(pf_count, ctx->stream));
	for (int f = 0; f < PC_MAXEARLY; f++)
		if (early_mem[f])
			CB_CUDA(ctx, cudaFreeAsync(early_mem[f], ctx->stream));
	ctx->kernel_timed = true;
	*handled = true;
	return CBGPU_OK;
}
