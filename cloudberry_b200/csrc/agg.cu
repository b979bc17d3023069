/*
 * agg.cu - aggregate hash tables (allocation, read-back, conversion to a relation) and device top-N.
 *
 * The table stands in for the reference's TupleHashTable of AggStatePerGroupData
 * (backend/executor/execGrouping.c:317, backend/executor/nodeAgg.c:2220-2319).  Per group it holds
 * the grouping keys and, per accumulator, (N, 128-bit exact sum) - the same content as the
 * reference's Int128AggState / NumericAggState{N, sumX} (backend/utils/adt/numeric.c:5340, 4602)
 * or float8 {N, Sx} - so partial states can be redistributed and combined (two-stage aggregation,
 * nodes/nodes.h:977-1000 AggSplit) and finalised exactly on the host.
 */
#include "common.cuh"

#include <stdlib.h>

static int64_t
next_pow2(int64_t v)
{
	int64_t		p = 1;

	while (p < v)
		p <<= 1;
	return p;
}

struct AggKinds
{
	int32_t		k[CBP_MAX_AGGS];
};

__global__ void
k_agg_init(AggDev t, const AggKinds kk)
{
	const int32_t *kinds = kk.k;
	size_t		cap = (size_t) t.mask + 1;
	size_t		i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	size_t		stride = (size_t) gridDim.x * blockDim.x;

	for (; i < cap; i += stride)
	{
		t.state[i] = 0;
		for (int a = 0; a < t.naccs; a++)
		{
			unsigned long long lo = 0;

			if (kinds[a] == CBP_ACC_MIN || kinds[a] == CBP_ACC_MERGE_MIN)
				lo = 0x7fffffffffffffffull;
			else if (kinds[a] == CBP_ACC_MAX || kinds[a] == CBP_ACC_MERGE_MAX)
				lo = 0x8000000000000000ull;
			t.n[i * t.naccs + a] = 0;
			t.sum[(i * t.naccs + a) * 2] = lo;
			t.sum[(i * t.naccs + a) * 2 + 1] = 0;
		}
	}
	if (blockIdx.x == 0 && threadIdx.x == 0)
	{
		*t.ngroups = 0;
		*t.full = 0;
	}
}

extern "C" int
cbgpu_agg_reset(cbgpu_aggtable *t)
{
	cbgpu_ctx  *ctx = t->ctx;
	AggKinds	kk;

	t->counted = false;
	t->snap_valid = false;
	memcpy(kk.k, t->kinds, sizeof(kk.k));
	int			blocks = (int) ((t->capacity + 255) / 256);

	if (blocks > ctx->sm_count * 8)
		blocks = ctx->sm_count * 8;
	k_agg_init<<<blocks, 256, 0, ctx->stream>>>(t->d, kk);
	CB_LAUNCHED(ctx, "k_agg_init");
	return CBGPU_OK;
}

extern "C" int
cbgpu_agg_create(cbgpu_ctx *ctx, int32_t nkeys, int32_t naccs, const int32_t *acc_kinds, int64_t capacity_groups,
				 cbgpu_aggtable **out)
{
	int64_t		cap;
	int			rc;

	*out = NULL;
	if (nkeys < 0 || nkeys > CBP_MAX_GROUP_KEYS)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "GROUP BY with %s%lld columns is beyond the GPU path's limit (8)", "", nkeys);
	if (naccs < 0 || naccs > CBP_MAX_AGGS)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "aggregate with %s%lld accumulators is beyond the GPU path's limit (16)", "", naccs);
	CbOwned<cbgpu_aggtable> t((cbgpu_aggtable *) calloc(1, sizeof(cbgpu_aggtable)), cbgpu_agg_free);

	if (!t)
		return CBGPU_ERR_NOMEM;
	t->ctx = ctx;
	cap = next_pow2((capacity_groups < 16 ? 16 : capacity_groups) * 2);
	if (cap > (1ll << 31))
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "aggregate table of %s%lld slots exceeds the GPU path's limit", "", cap);
	t->capacity = cap;
	t->d.mask = (uint32_t) (cap - 1);
	t->d.nkeys = nkeys;
	t->d.naccs = naccs;
	for (int a = 0; a < naccs; a++)
		t->kinds[a] = acc_kinds ? acc_kinds[a] : CBP_ACC_SUM_INT;
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	{
		/* one allocation for all the arrays (a table is created per query: seven pool calls were a measurable part of a
		 * Q1 step) */
		size_t		off[8];
		size_t		sz[7] = {(size_t) cap * sizeof(int32_t), (size_t) cap * sizeof(uint32_t), (size_t) cap * sizeof(int64_t) * (nkeys ? nkeys : 1),
							 (size_t) cap * sizeof(uint32_t), (size_t) cap * sizeof(int64_t) * (naccs ? naccs : 1),
							 (size_t) cap * 2 * sizeof(unsigned long long) * (naccs ? naccs : 1), sizeof(int32_t) * 4};
		char	   *base;

		off[0] = 0;
		for (int i = 0; i < 7; i++)
			off[i + 1] = off[i] + ((sz[i] + 255) & ~(size_t) 255);
		CB_CUDA(ctx, cudaMallocAsync(&base, off[7], ctx->stream));
		t->base = base;
		t->d.state = (int32_t *) (base + off[0]);
		t->d.hash = (uint32_t *) (base + off[1]);
		t->d.keys = (int64_t *) (base + off[2]);
		t->d.keynull = (uint32_t *) (base + off[3]);
		t->d.n = (int64_t *) (base + off[4]);
		t->d.sum = (unsigned long long *) (base + off[5]);
		t->d.ngroups = (int32_t *) (base + off[6]);
	}
	t->d.full = t->d.ngroups + 1;
	if ((rc = cbgpu_agg_reset(t.get())) == CBGPU_OK)
		*out = t.release();
	return rc;
}

/* device bytes one slot of an aggregate table takes (two slots per group are provisioned: load factor <= 0.5) */
extern "C" int64_t
cbgpu_agg_slot_bytes(int32_t nkeys, int32_t naccs)
{
	return 4 + 4 + 4 + 8 * (int64_t) (nkeys ? nkeys : 1) + (8 + 16) * (int64_t) (naccs ? naccs : 1);
}

extern "C" int
cbgpu_agg_set_partition(cbgpu_aggtable *t, int32_t npart, int32_t part)
{
	if (npart < 1 || npart > 65536 || (npart & (npart - 1)) != 0 || part < 0 || part >= npart)
		return cb_fail(t->ctx, CBGPU_ERR_INVALID, "aggregate partition %s%lld out of range", "", part);
	t->d.npart = npart;
	t->d.part_id = part;
	t->d.part_shift = 32;
	for (int b = npart; b > 1; b >>= 1)
		t->d.part_shift--;
	return CBGPU_OK;
}

extern "C" void
cbgpu_agg_free(cbgpu_aggtable *t)
{
	if (!t)
		return;
	cudaSetDevice(t->ctx->device);
	if (t->base)
		cudaFreeAsync(t->base, t->ctx->stream);
	free(t->snap);
	free(t);
}

/* number of published groups (TupleHashTable's `members`), and whether any group key is NULL */
__global__ void
k_agg_count(AggDev t, int *anynull)
{
	size_t		cap = (size_t) t.mask + 1;
	size_t		i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	size_t		stride = (size_t) gridDim.x * blockDim.x;
	int			c = 0;
	int			an = 0;

	for (; i < cap; i += stride)
		if (t.state[i] == 2)
		{
			c++;
			an |= t.keynull[i] != 0;
		}
	for (int o = 16; o > 0; o >>= 1)
	{
		c += __shfl_xor_sync(0xffffffffu, c, o);
		an |= __shfl_xor_sync(0xffffffffu, an, o);
	}
	if ((threadIdx.x & 31) == 0)
	{
		if (c)
			atomicAdd(t.ngroups, c);
		if (an)
			*anynull = 1;
	}
}

/* small tables: count, flags and the groups themselves in one kernel and one round trip */
__global__ void __launch_bounds__(256)
k_agg_snapshot(AggDev t, AggSnap *out)
{
	if (threadIdx.x == 0)
		out->retry = out->audit = 0;
	agg_snapshot_block(t, out);
}

/* the snapshot the stream has just been synchronised on describes table t */
void
cb_agg_adopt_snapshot(cbgpu_aggtable *t, const AggSnap *snap)
{
	t->snap_valid = false;
	if (snap->ngroups < 0)
		return;
	t->ngroups = snap->ngroups;
	t->anynull = snap->anynull;
	t->counted = !snap->full;
	if (snap->full || snap->ngroups > AGG_SNAP_MAXG)
		return;
	if (!t->snap)
		t->snap = (AggSnap *) malloc(sizeof(AggSnap));
	if (!t->snap)
		return;
	memcpy(t->snap, snap, sizeof(AggSnap));
	t->snap_valid = true;
}

extern "C" int
cbgpu_agg_ngroups(cbgpu_aggtable *t, int64_t *ngroups)
{
	cbgpu_ctx  *ctx = t->ctx;
	int32_t		h[3];

	if (!t->counted && t->capacity <= AGG_SNAP_MAXCAP && ctx->agg_snap)
	{
		ctx->agg_snap->ngroups = -1;
		k_agg_snapshot<<<1, 256, 0, ctx->stream>>>(t->d, ctx->agg_snap);
		CB_LAUNCHED(ctx, "k_agg_snapshot");
		CB_CUDA(ctx, CB_STATUS_RIDE(ctx));
		CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		CB_STATUS_FETCHED(ctx);
		if (ctx->agg_snap->full)
			return cb_fail(ctx, CBGPU_ERR_NOMEM, "aggregate hash table overflow (%s capacity %lld slots)", "", t->capacity);
		cb_agg_adopt_snapshot(t, ctx->agg_snap);
	}
	if (!t->counted)
	{
		/* groups are counted here, once per fill, rather than with one same-address atomic per new
		 * group; d.ngroups = {count, table-full flag, any-NULL-key flag} */
		CB_CUDA(ctx, cudaMemsetAsync(t->d.ngroups, 0, sizeof(int32_t), ctx->stream));
		CB_CUDA(ctx, cudaMemsetAsync(t->d.ngroups + 2, 0, sizeof(int32_t), ctx->stream));
		{
			int			blocks = (int) ((t->capacity + 1023) / 1024);

			if (blocks > ctx->sm_count * 8)
				blocks = ctx->sm_count * 8;
			k_agg_count<<<blocks, 256, 0, ctx->stream>>>(t->d, t->d.ngroups + 2);
			CB_LAUNCHED(ctx, "k_agg_count");
		}
		CB_CUDA(ctx, cudaMemcpyAsync(h, t->d.ngroups, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
		CB_CUDA(ctx, CB_STATUS_RIDE(ctx));
		CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		CB_STATUS_FETCHED(ctx);
		if (h[1])
			return cb_fail(ctx, CBGPU_ERR_NOMEM, "aggregate hash table overflow (%s capacity %lld slots)", "", t->capacity);
		t->ngroups = h[0];
		t->anynull = h[2];
		t->counted = true;
	}
	*ngroups = t->ngroups;
	return CBGPU_OK;
}

/* the table is about to be written (a pipeline's AGG sink, a reset): forget the cached count */
void
cb_agg_touch(cbgpu_aggtable *t)
{
	t->counted = false;
	t->snap_valid = false;
}

/* compaction: slots in `ready` state -> dense rows (agg_retrieve_hash_table's table walk,
 * backend/executor/nodeAgg.c:3014) */
struct AggOut
{
	int64_t    *keys;
	uint32_t   *keynull;
	int64_t    *n;
	int64_t    *lo;
	int64_t    *hi;
	int32_t    *counter;
	int64_t		maxgroups;
};

__global__ void
k_agg_compact(AggDev t, AggOut o)
{
	size_t		cap = (size_t) t.mask + 1;
	size_t		i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	size_t		stride = (size_t) gridDim.x * blockDim.x;

	for (; i < cap; i += stride)
	{
		if (t.state[i] != 2)
			continue;
		int			g = atomicAdd(o.counter, 1);

		if (g >= o.maxgroups)
			continue;
		for (int k = 0; k < t.nkeys; k++)
			o.keys[(size_t) g * t.nkeys + k] = t.keys[i * t.nkeys + k];
		o.keynull[g] = t.keynull[i];
		for (int a = 0; a < t.naccs; a++)
		{
			o.n[(size_t) g * t.naccs + a] = t.n[i * t.naccs + a];
			o.lo[(size_t) g * t.naccs + a] = (int64_t) t.sum[(i * t.naccs + a) * 2];
			o.hi[(size_t) g * t.naccs + a] = (int64_t) t.sum[(i * t.naccs + a) * 2 + 1];
		}
	}
}

extern "C" int
cbgpu_agg_read(cbgpu_aggtable *t, int64_t maxgroups, int64_t *keys, uint32_t *keynull, int64_t *n, int64_t *sum_lo,
			   int64_t *sum_hi, int64_t *ngroups)
{
	cbgpu_ctx  *ctx = t->ctx;
	CbCallMem	mem(ctx);
	int64_t		ng;
	int			rc = cbgpu_agg_ngroups(t, &ng);
	AggOut		o;
	int			nk = t->d.nkeys ? t->d.nkeys : 1;
	int			na = t->d.naccs ? t->d.naccs : 1;

	if (rc)
		return rc;
	*ngroups = ng;
	if (ng > maxgroups)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_agg_read: %s%lld groups exceed the caller's buffer", "", ng);
	if (ng == 0)
		return CBGPU_OK;
	if (t->snap_valid && t->snap->ngroups == ng)
	{
		/* the groups came with the count */
		for (int64_t g = 0; g < ng; g++)
		{
			keynull[g] = t->snap->keynull[g];
			for (int k = 0; k < t->d.nkeys; k++)
				keys[g * t->d.nkeys + k] = t->snap->keys[g][k];
			for (int a = 0; a < t->d.naccs; a++)
			{
				n[g * t->d.naccs + a] = t->snap->n[g][a];
				sum_lo[g * t->d.naccs + a] = t->snap->lo[g][a];
				sum_hi[g * t->d.naccs + a] = t->snap->hi[g][a];
			}
		}
		return CBGPU_OK;
	}
	o.maxgroups = ng;
	CB_CUDA(ctx, mem.alloc(&o.keys, sizeof(int64_t) * ng * nk));
	CB_CUDA(ctx, mem.alloc(&o.keynull, sizeof(uint32_t) * ng));
	CB_CUDA(ctx, mem.alloc(&o.n, sizeof(int64_t) * ng * na));
	CB_CUDA(ctx, mem.alloc(&o.lo, sizeof(int64_t) * ng * na));
	CB_CUDA(ctx, mem.alloc(&o.hi, sizeof(int64_t) * ng * na));
	CB_CUDA(ctx, mem.alloc(&o.counter, sizeof(int32_t)));
	CB_CUDA(ctx, cudaMemsetAsync(o.counter, 0, sizeof(int32_t), ctx->stream));
	int			blocks = (int) ((t->capacity + 255) / 256);

	if (blocks > ctx->sm_count * 8)
		blocks = ctx->sm_count * 8;
	k_agg_compact<<<blocks, 256, 0, ctx->stream>>>(t->d, o);
	CB_LAUNCHED(ctx, "k_agg_compact");
	if (t->d.nkeys)
		CB_CUDA(ctx, cudaMemcpyAsync(keys, o.keys, sizeof(int64_t) * ng * t->d.nkeys, cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaMemcpyAsync(keynull, o.keynull, sizeof(uint32_t) * ng, cudaMemcpyDeviceToHost, ctx->stream));
	if (t->d.naccs)
	{
		CB_CUDA(ctx, cudaMemcpyAsync(n, o.n, sizeof(int64_t) * ng * t->d.naccs, cudaMemcpyDeviceToHost, ctx->stream));
		CB_CUDA(ctx, cudaMemcpyAsync(sum_lo, o.lo, sizeof(int64_t) * ng * t->d.naccs, cudaMemcpyDeviceToHost, ctx->stream));
		CB_CUDA(ctx, cudaMemcpyAsync(sum_hi, o.hi, sizeof(int64_t) * ng * t->d.naccs, cudaMemcpyDeviceToHost, ctx->stream));
	}
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return CBGPU_OK;
}

/* groups -> relation: key columns (typed), then per accumulator N, sum.lo, sum.hi (int8 each) */
struct AggRelOut
{
	void	   *key[CBP_MAX_GROUP_KEYS];
	uint8_t    *keynulls[CBP_MAX_GROUP_KEYS];
	int32_t		keytype[CBP_MAX_GROUP_KEYS];
	int64_t    *acc[CBP_MAX_AGGS * 3];
	int32_t    *counter;
};

__global__ void
k_agg_to_rel(AggDev t, AggRelOut o)
{
	size_t		cap = (size_t) t.mask + 1;
	size_t		i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	size_t		stride = (size_t) gridDim.x * blockDim.x;

	for (; i < cap; i += stride)
	{
		if (t.state[i] != 2)
			continue;
		int			g = atomicAdd(o.counter, 1);
		uint32_t	nm = t.keynull[i];

		for (int k = 0; k < t.nkeys; k++)
		{
			int64_t		v = t.keys[i * t.nkeys + k];

			switch (o.keytype[k])
			{
				case CB_INT4: case CB_DATE: case CB_DICT32:
					((int32_t *) o.key[k])[g] = (int32_t) v;
					break;
				case CB_INT8: case CB_NUMERIC: case CB_FLOAT8:
					((int64_t *) o.key[k])[g] = v;
					break;
				default:
					((uint8_t *) o.key[k])[g] = (uint8_t) v;
			}
			if (o.keynulls[k])
				o.keynulls[k][g] = (nm >> k) & 1;
		}
		for (int a = 0; a < t.naccs; a++)
		{
			o.acc[a * 3][g] = t.n[i * t.naccs + a];
			o.acc[a * 3 + 1][g] = (int64_t) t.sum[(i * t.naccs + a) * 2];
			o.acc[a * 3 + 2][g] = (int64_t) t.sum[(i * t.naccs + a) * 2 + 1];
		}
	}
}

__global__ void
k_agg_anynull(AggDev t, int *flag)
{
	size_t		cap = (size_t) t.mask + 1;
	size_t		i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	size_t		stride = (size_t) gridDim.x * blockDim.x;

	for (; i < cap; i += stride)
		if (t.state[i] == 2 && t.keynull[i])
			*flag = 1;
}

extern "C" int
cbgpu_agg_to_rel(cbgpu_aggtable *t, const int32_t *keytypes, cbgpu_rel **out)
{
	cbgpu_ctx  *ctx = t->ctx;
	CbCallMem	mem(ctx);
	int64_t		ng;
	int			rc = cbgpu_agg_ngroups(t, &ng);
	int32_t		types[CBP_MAX_GROUP_KEYS + CBP_MAX_AGGS * 3];
	int			ncols = t->d.nkeys + t->d.naccs * 3;
	cbgpu_rel  *created;
	AggRelOut	o;
	int			h_flag = 0;

	*out = NULL;
	if (rc)
		return rc;
	for (int k = 0; k < t->d.nkeys; k++)
		types[k] = keytypes[k];
	for (int a = 0; a < t->d.naccs * 3; a++)
		types[t->d.nkeys + a] = CB_INT8;
	rc = cbgpu_rel_create(ctx, ng, ncols, types, NULL, &created);
	if (rc)
		return rc;
	CbOwned<cbgpu_rel> rel(created, cbgpu_rel_free);

	memset(&o, 0, sizeof(o));
	int			blocks = (int) ((t->capacity + 255) / 256);

	if (blocks > ctx->sm_count * 8)
		blocks = ctx->sm_count * 8;
	/* NULL group keys need null byte-maps on the key columns (flag gathered with the group count) */
	h_flag = t->anynull;
	for (int k = 0; k < t->d.nkeys; k++)
	{
		o.key[k] = rel->data[k];
		o.keytype[k] = keytypes[k];
		if (h_flag && ng > 0)
		{
			CB_CUDA(ctx, cudaMallocAsync(&rel->nulls[k], (size_t) ng, ctx->stream));
			o.keynulls[k] = rel->nulls[k];
		}
	}
	for (int a = 0; a < t->d.naccs * 3; a++)
		o.acc[a] = (int64_t *) rel->data[t->d.nkeys + a];
	CB_CUDA(ctx, mem.alloc(&o.counter, sizeof(int32_t)));
	CB_CUDA(ctx, cudaMemsetAsync(o.counter, 0, sizeof(int32_t), ctx->stream));
	if (ng > 0)
	{
		k_agg_to_rel<<<blocks, 256, 0, ctx->stream>>>(t->d, o);
		CB_LAUNCHED(ctx, "k_agg_to_rel");
	}
	*out = rel.release();
	return CBGPU_OK;
}

/* ---------------------------------------------------------------------------------------------
 * top-N: ORDER BY keys LIMIT n over a relation (bounded sort above the Agg)
 * --------------------------------------------------------------------------------------------- */
#define TOPN_MAXK 64
#define TOPN_MAXKEYS 4

struct TopnParams
{
	const void *key[TOPN_MAXKEYS];
	int32_t		keytype[TOPN_MAXKEYS];
	int32_t		desc[TOPN_MAXKEYS];
	int32_t		uns[TOPN_MAXKEYS];
	int32_t		nkeys;
	int32_t		k;
	const uint32_t *in_idx;		/* NULL = identity over nrows                                         */
	int64_t		nin;
	uint32_t   *out_idx;		/* [nthreads * k], padded with 0xFFFFFFFF                             */
};

/* true when row a sorts strictly before row b */
__device__ __forceinline__ bool
topn_before(const TopnParams &p, const int64_t *ka, uint32_t ra, const int64_t *kb, uint32_t rb)
{
	for (int i = 0; i < p.nkeys; i++)
	{
		int64_t		x = ka[i],
					y = kb[i];

		if (x == y)
			continue;
		bool		lt = p.uns[i] ? ((uint64_t) x < (uint64_t) y) : (x < y);

		return p.desc[i] ? !lt : lt;
	}
	return ra < rb;
}

__global__ void
k_topn(TopnParams p)
{
	uint32_t	best_row[TOPN_MAXK];
	int64_t		best_key[TOPN_MAXK][TOPN_MAXKEYS];
	int			nbest = 0;
	int64_t		tid = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
	int64_t		stride = (int64_t) gridDim.x * blockDim.x;

	for (int64_t i = tid; i < p.nin; i += stride)
	{
		uint32_t	row = p.in_idx ? p.in_idx[i] : (uint32_t) i;
		int64_t		key[TOPN_MAXKEYS];

		if (row == 0xFFFFFFFFu)
			continue;
		for (int k = 0; k < p.nkeys; k++)
			key[k] = cb_load_widen(p.key[k], p.keytype[k], row);
		if (nbest == p.k && !topn_before(p, key, row, best_key[nbest - 1], best_row[nbest - 1]))
			continue;
		/* insertion into the sorted local list */
		int			pos = nbest < p.k ? nbest : p.k - 1;

		while (pos > 0 && topn_before(p, key, row, best_key[pos - 1], best_row[pos - 1]))
		{
			best_row[pos] = best_row[pos - 1];
			for (int k = 0; k < p.nkeys; k++)
				best_key[pos][k] = best_key[pos - 1][k];
			pos--;
		}
		best_row[pos] = row;
		for (int k = 0; k < p.nkeys; k++)
			best_key[pos][k] = key[k];
		if (nbest < p.k)
			nbest++;
	}
	for (int j = 0; j < p.k; j++)
		p.out_idx[tid * p.k + j] = j < nbest ? best_row[j] : 0xFFFFFFFFu;
}

/* --- threshold selection: the usual case (n >> k) costs two streaming passes over ONE key column ---
 * A: per-CTA minimum of the leading non-constant sort key, mapped so that smaller = sorts first;
 * K: the k-th smallest CTA minimum T bounds the answer (k rows - those minima - are <= T);
 * B: rows with key <= T become candidates (a few dozen when the key is not heavily tied);
 * C: one CTA ranks the candidates with the full comparator. */
#define TOPN_BLOCKS 1024
#define TOPN_CAND 4096

__device__ __forceinline__ unsigned long long
topn_ukey(const TopnParams &p, int i, uint32_t row)
{
	unsigned long long u = (unsigned long long) cb_load_widen(p.key[i], p.keytype[i], row);

	if (!p.uns[i])
		u ^= 0x8000000000000000ull;
	return p.desc[i] ? ~u : u;
}

__global__ void __launch_bounds__(256)
k_topn_min(TopnParams p, int keyi, unsigned long long *bmin, unsigned long long *bmax)
{
	__shared__ unsigned long long smin[8], smax[8];
	unsigned long long lo = ~0ull,
				hi = 0;

	for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < p.nin; i += (int64_t) gridDim.x * blockDim.x)
	{
		const unsigned long long u = topn_ukey(p, keyi, (uint32_t) i);

		lo = u < lo ? u : lo;
		hi = u > hi ? u : hi;
	}
	for (int o = 16; o > 0; o >>= 1)
	{
		const unsigned long long a = __shfl_xor_sync(0xffffffffu, lo, o);
		const unsigned long long b = __shfl_xor_sync(0xffffffffu, hi, o);

		lo = a < lo ? a : lo;
		hi = b > hi ? b : hi;
	}
	if ((threadIdx.x & 31) == 0)
	{
		smin[threadIdx.x >> 5] = lo;
		smax[threadIdx.x >> 5] = hi;
	}
	__syncthreads();
	if (threadIdx.x == 0)
	{
		for (int w = 1; w < (int) (blockDim.x >> 5); w++)
		{
			lo = smin[w] < lo ? smin[w] : lo;
			hi = smax[w] > hi ? smax[w] : hi;
		}
		bmin[blockIdx.x] = lo;
		bmax[blockIdx.x] = hi;
	}
}

/* out[0] = k-th smallest block minimum (or the maximum when there are fewer than k blocks),
 * out[1] = global minimum, out[2] = global maximum */
__global__ void __launch_bounds__(TOPN_BLOCKS)
k_topn_kth(const unsigned long long *bmin, const unsigned long long *bmax, int nblocks, int k, unsigned long long *out)
{
	__shared__ unsigned long long v[TOPN_BLOCKS];
	__shared__ unsigned long long gmax;
	const int	t = threadIdx.x;

	v[t] = t < nblocks ? bmin[t] : ~0ull;
	if (t == 0)
	{
		unsigned long long m = 0;

		for (int i = 0; i < nblocks; i++)
			m = bmax[i] > m ? bmax[i] : m;
		gmax = m;
	}
	__syncthreads();
	for (int size = 2; size <= TOPN_BLOCKS; size <<= 1)
		for (int stride = size >> 1; stride > 0; stride >>= 1)
		{
			const int	partner = t ^ stride;

			if (partner > t)
			{
				const bool	up = (t & size) == 0;
				const unsigned long long a = v[t],
							b = v[partner];

				if ((a > b) == up)
				{
					v[t] = b;
					v[partner] = a;
				}
			}
			__syncthreads();
		}
	if (t == 0)
	{
		out[0] = nblocks >= k ? v[k - 1] : gmax;
		out[1] = v[0];
		out[2] = gmax;
	}
}

__global__ void __launch_bounds__(256)
k_topn_filter(TopnParams p, int keyi, const unsigned long long *thr, uint32_t *cand, int *ncand)
{
	const unsigned long long T = thr[0];

	for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < p.nin; i += (int64_t) gridDim.x * blockDim.x)
		if (topn_ukey(p, keyi, (uint32_t) i) <= T)
		{
			const int	pos = atomicAdd(ncand, 1);

			if (pos < TOPN_CAND)
				cand[pos] = (uint32_t) i;
		}
}

/* rank every candidate among the candidates with the full comparator; ranks < k are the answer */
__global__ void __launch_bounds__(1024)
k_topn_final(TopnParams p, const uint32_t *cand, const int *ncand, int64_t nall, uint32_t *out)
{
	const int	m = cand ? (*ncand < TOPN_CAND ? *ncand : TOPN_CAND) : (int) nall;

	for (int j = threadIdx.x; j < p.k; j += blockDim.x)
		out[j] = 0xFFFFFFFFu;
	__syncthreads();
	for (int i = threadIdx.x; i < m; i += blockDim.x)
	{
		const uint32_t ri = cand ? cand[i] : (uint32_t) i;
		int64_t		ki[TOPN_MAXKEYS];
		int			rank = 0;

		for (int k = 0; k < p.nkeys; k++)
			ki[k] = cb_load_widen(p.key[k], p.keytype[k], ri);
		for (int j = 0; j < m && rank < p.k; j++)
		{
			const uint32_t rj = cand ? cand[j] : (uint32_t) j;
			int64_t		kj[TOPN_MAXKEYS];

			if (j == i)
				continue;
			for (int k = 0; k < p.nkeys; k++)
				kj[k] = cb_load_widen(p.key[k], p.keytype[k], rj);
			rank += topn_before(p, kj, rj, ki, ri);
		}
		if (rank < p.k)
			out[rank] = ri;
	}
}

/* ---------------------------------------------------------------------------------------------
 * merge receive: a Gather Motion whose senders' streams are sorted (Motion.sendSorted; execMotionSortedReceiver,
 * nodeMotion.c:433, merges them with a binary heap under CdbMergeComparator :1010).  The gathered relation holds the
 * streams one after another, so it is a sequence of sorted runs: a row's place in the merged order is its place in its
 * own run plus, for every other run, the number of rows there that go before it (binary search; equal keys: the earlier
 * run first) - every row finds its place independently, no heap, no passes.
 * --------------------------------------------------------------------------------------------- */
#define MERGE_MAXRUNS 64

struct MergeParams
{
	const void *key[TOPN_MAXKEYS];
	const uint8_t *nulls[TOPN_MAXKEYS];
	int32_t		keytype[TOPN_MAXKEYS];
	int32_t		desc[TOPN_MAXKEYS];
	int32_t		uns[TOPN_MAXKEYS];
	int32_t		nkeys;
	int32_t		nruns;
	int64_t		n;
	int64_t		start[MERGE_MAXRUNS + 1];
	int32_t    *nfound;			/* run starts found (k_merge_find_runs)                               */
	unsigned long long *found;
	uint32_t   *order;
};

/* < 0: row a sorts before row b; 0: equal keys.  NULLS LAST ascending, NULLS FIRST descending (the defaults) */
__device__ __forceinline__ int
merge_cmp(const MergeParams &p, int64_t a, int64_t b)
{
	for (int i = 0; i < p.nkeys; i++)
	{
		const bool	an = p.nulls[i] && p.nulls[i][a];
		const bool	bn = p.nulls[i] && p.nulls[i][b];
		int			c;

		if (an || bn)
			c = (an && bn) ? 0 : (an ? 1 : -1);
		else
		{
			const int64_t x = cb_load_widen(p.key[i], p.keytype[i], (uint32_t) a);
			const int64_t y = cb_load_widen(p.key[i], p.keytype[i], (uint32_t) b);

			if (x == y)
				c = 0;
			else if (p.uns[i])
				c = (uint64_t) x < (uint64_t) y ? -1 : 1;
			else
				c = x < y ? -1 : 1;
		}
		if (p.desc[i])
			c = -c;
		if (c)
			return c;
	}
	return 0;
}

/* a run starts wherever a row sorts before its predecessor */
__global__ void
k_merge_find_runs(MergeParams p)
{
	int64_t		i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x + 1;
	const int64_t stride = (int64_t) gridDim.x * blockDim.x;

	for (; i < p.n; i += stride)
		if (merge_cmp(p, i, i - 1) < 0)
		{
			const int	at = atomicAdd(p.nfound, 1);

			if (at < MERGE_MAXRUNS)
				p.found[at] = (unsigned long long) i;
		}
}

__global__ void
k_merge_place(MergeParams p)
{
	int64_t		i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
	const int64_t stride = (int64_t) gridDim.x * blockDim.x;

	for (; i < p.n; i += stride)
	{
		int			r = 0;
		int64_t		pos;

		while (r + 1 < p.nruns && p.start[r + 1] <= i)
			r++;
		pos = i - p.start[r];
		for (int q = 0; q < p.nruns; q++)
		{
			int64_t		lo = p.start[q],
						hi = p.start[q + 1];

			if (q == r)
				continue;
			/* rows of run q that go before row i: those that sort before it, and - in an earlier run - its equals too */
			while (lo < hi)
			{
				const int64_t mid = lo + (hi - lo) / 2;
				const int	c = merge_cmp(p, mid, i);

				if (c < 0 || (c == 0 && q < r))
					lo = mid + 1;
				else
					hi = mid;
			}
			pos += lo - p.start[q];
		}
		p.order[pos] = (uint32_t) i;
	}
}

extern "C" int
cbgpu_merge_sorted_runs(cbgpu_ctx *ctx, cbgpu_rel *rel, const int32_t *keycols, const int32_t *descending, const int32_t *unsigned_cmp,
						int32_t nkeys, int32_t max_runs, uint32_t **order_dev, int32_t *nruns_out)
{
	CbCallMem	mem(ctx);
	MergeParams p;
	int32_t		nfound = 0;
	unsigned long long found[MERGE_MAXRUNS];
	int			blocks;

	*order_dev = NULL;
	if (nruns_out)
		*nruns_out = rel->nrows > 0;
	if (nkeys < 1 || nkeys > TOPN_MAXKEYS || max_runs < 1 || max_runs > MERGE_MAXRUNS)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "merge receive supports 1..4 sort keys and up to 64 senders (%s got %lld keys)", "", nkeys);
	memset(&p, 0, sizeof(p));
	for (int i = 0; i < nkeys; i++)
	{
		if (keycols[i] < 0 || keycols[i] >= rel->ncols)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_merge_sorted_runs: bad key column%s %lld", "", keycols[i]);
		p.key[i] = rel->data[keycols[i]];
		p.nulls[i] = rel->nulls[keycols[i]];
		p.keytype[i] = rel->types[keycols[i]];
		p.desc[i] = descending[i];
		p.uns[i] = unsigned_cmp ? unsigned_cmp[i] : 0;
		if (p.keytype[i] == CB_FLOAT8)
			return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "merge receive over a float8 key%s", "", 0);
	}
	p.nkeys = nkeys;
	p.n = rel->nrows;
	if (rel->nrows < 2)
		return CBGPU_OK;
	blocks = (int) ((rel->nrows + 255) / 256);
	if (blocks > ctx->sm_count * 8)
		blocks = ctx->sm_count * 8;
	CB_CUDA(ctx, mem.alloc(&p.nfound, sizeof(int32_t) + MERGE_MAXRUNS * sizeof(unsigned long long) + 8));
	p.found = (unsigned long long *) ((char *) p.nfound + 8);
	CB_CUDA(ctx, cudaMemsetAsync(p.nfound, 0, sizeof(int32_t), ctx->stream));
	k_merge_find_runs<<<blocks, 256, 0, ctx->stream>>>(p);
	CB_LAUNCHED(ctx, "k_merge_find_runs");
	CB_CUDA(ctx, cudaMemcpyAsync(&nfound, p.nfound, sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaMemcpyAsync(found, p.found, sizeof(found), cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	CB_CUDA(ctx, mem.free(p.nfound));
	if (nfound + 1 > max_runs)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "merge receive: %s%lld sorted runs arrived from fewer senders - a sender's stream is not in the Motion's sort order",
					   "", (long long) nfound + 1);
	if (nruns_out)
		*nruns_out = nfound + 1;
	if (nfound == 0)
		return CBGPU_OK;		/* one run: arrival order is the order */
	/* run starts in ascending order (found in atomic order) */
	for (int a = 1; a < nfound; a++)
		for (int b = a; b > 0 && found[b] < found[b - 1]; b--)
		{
			unsigned long long t = found[b];

			found[b] = found[b - 1];
			found[b - 1] = t;
		}
	p.nruns = nfound + 1;
	p.start[0] = 0;
	for (int a = 0; a < nfound; a++)
		p.start[a + 1] = (int64_t) found[a];
	p.start[p.nruns] = rel->nrows;
	CB_CUDA(ctx, mem.alloc(&p.order, (size_t) rel->nrows * sizeof(uint32_t)));
	k_merge_place<<<blocks, 256, 0, ctx->stream>>>(p);
	CB_LAUNCHED(ctx, "k_merge_place");
	*order_dev = mem.detach(p.order);
	return CBGPU_OK;
}

extern "C" int
cbgpu_topn(cbgpu_ctx *ctx, cbgpu_rel *rel, const int32_t *keycols, const int32_t *descending, const int32_t *unsigned_cmp,
		   int32_t nkeys, int64_t limit, uint32_t *host_idx, int64_t *nout)
{
	CbCallMem	mem(ctx);
	TopnParams	p;
	uint32_t   *cand1 = NULL,
			   *cand2 = NULL;
	int64_t		n1;
	bool		done = false;

	if (nkeys < 1 || nkeys > TOPN_MAXKEYS || limit < 1 || limit > TOPN_MAXK)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "device top-N supports 1..4 sort keys and LIMIT <= 64 (%s got %lld)", "", limit);
	memset(&p, 0, sizeof(p));
	for (int i = 0; i < nkeys; i++)
	{
		if (keycols[i] < 0 || keycols[i] >= rel->ncols)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_topn: bad key column%s %lld", "", keycols[i]);
		if (rel->nulls[keycols[i]])
			return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "device top-N over a nullable sort key (%s column %lld)", "", keycols[i]);
		p.key[i] = rel->data[keycols[i]];
		p.keytype[i] = rel->types[keycols[i]];
		p.desc[i] = descending[i];
		p.uns[i] = unsigned_cmp ? unsigned_cmp[i] : 0;
		if (p.keytype[i] == CB_FLOAT8)
			return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "device top-N over a float8 key%s", "", 0);
	}
	p.nkeys = nkeys;
	p.k = (int32_t) limit;
	*nout = 0;
	if (rel->nrows == 0)
		return CBGPU_OK;
	{
		/* threshold selection first (see above); the tournament below only when it cannot decide */
		unsigned long long *scratch = NULL;		/* [TOPN_BLOCKS] minima, [TOPN_BLOCKS] maxima, [3] threshold / min / max */
		uint32_t   *cand = NULL;
		int		   *ncand = NULL;
		unsigned long long h3[3];
		int			hn = 0;

		p.in_idx = NULL;
		p.nin = rel->nrows;
		CB_CUDA(ctx, mem.alloc(&cand1, (TOPN_MAXK + 1) * sizeof(uint32_t)));
		if (rel->nrows <= TOPN_CAND)
		{
			k_topn_final<<<1, 1024, 0, ctx->stream>>>(p, NULL, NULL, rel->nrows, cand1);
			CB_LAUNCHED(ctx, "k_topn_final");
			done = true;
		}
		else
		{
			/* every block of k_topn_min must see a row: an empty block's minimum is ~0, and when fewer than k blocks hold
			 * rows the k-th smallest minimum admits every row.  At most one block per 64 rows, each of 256 threads halved
			 * down to 64 until the grid's last block starts inside the rows: > TOPN_CAND rows give > TOPN_MAXK blocks,
			 * all with rows */
			int			nblocks = (int) ((rel->nrows + 63) / 64);
			int			tpb = 256;

			if (nblocks > TOPN_BLOCKS)
				nblocks = TOPN_BLOCKS;
			while (tpb > 64 && (int64_t) (nblocks - 1) * tpb >= rel->nrows)
				tpb >>= 1;
			CB_CUDA(ctx, mem.alloc(&scratch, (2 * TOPN_BLOCKS + 3) * sizeof(unsigned long long)));
			CB_CUDA(ctx, mem.alloc(&cand, TOPN_CAND * sizeof(uint32_t)));
			CB_CUDA(ctx, mem.alloc(&ncand, sizeof(int)));
			for (int keyi = 0; keyi < nkeys && !done; keyi++)
			{
				k_topn_min<<<nblocks, tpb, 0, ctx->stream>>>(p, keyi, scratch, scratch + TOPN_BLOCKS);
				CB_LAUNCHED(ctx, "k_topn_min");
				k_topn_kth<<<1, TOPN_BLOCKS, 0, ctx->stream>>>(scratch, scratch + TOPN_BLOCKS, nblocks, p.k, scratch + 2 * TOPN_BLOCKS);
				CB_LAUNCHED(ctx, "k_topn_kth");
				CB_CUDA(ctx, cudaMemcpyAsync(h3, scratch + 2 * TOPN_BLOCKS, sizeof(h3), cudaMemcpyDeviceToHost, ctx->stream));
				CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
				if (h3[1] == h3[2])
					continue;	/* a constant key (e.g. the high half of small 128-bit sums) decides nothing */
				CB_CUDA(ctx, cudaMemsetAsync(ncand, 0, sizeof(int), ctx->stream));
				k_topn_filter<<<nblocks, 256, 0, ctx->stream>>>(p, keyi, scratch + 2 * TOPN_BLOCKS, cand, ncand);
				CB_LAUNCHED(ctx, "k_topn_filter");
				CB_CUDA(ctx, cudaMemcpyAsync(&hn, ncand, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
				CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
				if (hn <= TOPN_CAND)
				{
					k_topn_final<<<1, 1024, 0, ctx->stream>>>(p, cand, ncand, 0, cand1);
					CB_LAUNCHED(ctx, "k_topn_final");
					done = true;
				}
				break;			/* heavily tied key: the tournament sorts it out */
			}
			CB_CUDA(ctx, mem.free(scratch));
			CB_CUDA(ctx, mem.free(cand));
			CB_CUDA(ctx, mem.free(ncand));
		}
	}
	/* tournament: every pass gives each thread up to per_thread candidates and keeps its best k, until one
	 * thread holds the answer.  per_thread >= 4k, so a pass leaves at most half its input (k per thread,
	 * padded); a pass that does not shrink its input is an error, never an endless loop */
	if (!done)
	{
		const int	threads = 128;
		const int64_t per_thread = limit * 4 > 64 ? limit * 4 : 64;
		const uint32_t *in = NULL;
		int64_t		nin = rel->nrows;
		int			which = 0;
		int64_t		cap = ((rel->nrows + per_thread - 1) / per_thread + threads) * limit;

		CB_CUDA(ctx, mem.free(cand1));
		CB_CUDA(ctx, mem.alloc(&cand1, cap * sizeof(uint32_t)));
		CB_CUDA(ctx, mem.alloc(&cand2, cap * sizeof(uint32_t)));
		for (;;)
		{
			int64_t		nthreads = (nin + per_thread - 1) / per_thread;
			int			blocks = (int) ((nthreads + threads - 1) / threads);
			int			tpb = nthreads < threads ? (int) nthreads : threads;
			uint32_t   *outbuf = which ? cand2 : cand1;

			if (nthreads <= 1)
			{
				blocks = 1;
				tpb = 1;
			}
			p.in_idx = in;
			p.nin = nin;
			p.out_idx = outbuf;
			k_topn<<<blocks, tpb, 0, ctx->stream>>>(p);
			CB_LAUNCHED(ctx, "k_topn");
			n1 = (int64_t) blocks * tpb * limit;
			if (blocks == 1 && tpb == 1)
			{
				if (outbuf != cand1)
					CB_CUDA(ctx, cudaMemcpyAsync(cand1, outbuf, limit * sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
				break;
			}
			if (n1 >= nin)
				return cb_fail(ctx, CBGPU_ERR_INVALID, "device top-N: a tournament pass did not shrink its input%s (%lld candidates)", "", nin);
			in = outbuf;
			nin = n1;
			which ^= 1;
		}
	}
	CB_CUDA(ctx, cudaMemcpyAsync(host_idx, cand1, limit * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	int64_t		n = 0;

	while (n < limit && host_idx[n] != 0xFFFFFFFFu)
		n++;
	*nout = n;
	return CBGPU_OK;
}

/* ---------------------------------------------------------------------------------------------
 * top-N for any LIMIT (cbgpu_topn_select).  Every key maps to a 64-bit image whose unsigned order is the sort order
 * (topn_ukey, plus float8's order), preceded by a one-bit NULL digit: NULLS LAST ascending, FIRST descending, as rows_cmp and
 * the merge receive order them.  One pass reduces each key's smallest and largest image and whether a NULL occurs; the host
 * reads that back once and keeps the 8-bit digits that can vary.  An MSD radix select over those digits then takes the first
 * min(limit, rows) rows - each pass counts the digit over the rows still tied, one CTA picks the digit where the remaining
 * rank falls, and the tied rows are compacted stably - with no host synchronisation between passes: a pass after the one that
 * decided exits at once.  What is still tied when the digits run out gives its lowest rows.  A stable LSD radix sort over the
 * same digits orders the chosen rows.  Both start from row order, so equal keys keep it: the lower row index wins, as in
 * topn_before.  Count and scatter are a stable counting sort modelled on k_ht_partition_count / _write.
 * --------------------------------------------------------------------------------------------- */
#define TSEL_THREADS 256
#define TSEL_MAXDIGITS (TOPN_MAXKEYS * 9)
#define TSEL_NULLDIGIT 64			/* the shift that names a key's NULL digit */

struct TselKey
{
	const void *data;
	const uint8_t *nullmap;			/* NULL map (1 = NULL), or NULL                                       */
	const long long *ncol;			/* int8 column whose 0 means NULL, or NULL                            */
	int32_t		type;
	int32_t		desc;
	int32_t		uns;
	int32_t		f8;
};

struct TselKeys
{
	TselKey		k[TOPN_MAXKEYS];
	int32_t		nkeys;
};

/* the selection's progress, on the device: pass p reads ntied[p] rows and leaves ntied[p + 1] */
struct TselState
{
	unsigned long long need;		/* rows the tied set still owes the answer                            */
	unsigned long long nsel;		/* rows chosen so far                                                 */
	unsigned long long m;			/* min(limit, rows)                                                   */
	unsigned long long ntied[TSEL_MAXDIGITS + 1];
	int32_t		decided;			/* the pass that completed the selection, -1 while none has           */
	int32_t		bucket[TSEL_MAXDIGITS];	/* each pass's chosen digit                                    */
	int32_t		take[TSEL_MAXDIGITS];	/* 1: every row with that digit is chosen                      */
};

__device__ __forceinline__ unsigned long long
tsel_image(const TselKey &k, uint32_t row, bool *isnull)
{
	unsigned long long u = (unsigned long long) cb_load_widen(k.data, k.type, row);

	*isnull = (k.nullmap && __ldg(k.nullmap + row)) || (k.ncol && __ldg(k.ncol + row) == 0);
	if (k.f8)
	{
		/* float8_cmp_internal: -0 = +0, every NaN equal and above +Infinity; then sign-magnitude to unsigned order */
		if ((u << 1) == 0)
			u = 0;
		else if ((u & 0x7FF0000000000000ull) == 0x7FF0000000000000ull && (u & 0x000FFFFFFFFFFFFFull))
			u = 0x7FF8000000000000ull;
		u = (u >> 63) ? ~u : (u | 0x8000000000000000ull);
	}
	else if (!k.uns)
		u ^= 0x8000000000000000ull;
	return k.desc ? ~u : u;
}

/* digit `shift` of a row's key: the NULL digit, or 8 bits of the image (0 for a NULL, which its NULL digit already placed) */
__device__ __forceinline__ int
tsel_digit(const TselKey &k, int shift, uint32_t row)
{
	bool		isnull;
	const unsigned long long u = tsel_image(k, row, &isnull);

	if (shift == TSEL_NULLDIGIT)
		return isnull != (k.desc != 0);
	return isnull ? 0 : (int) ((u >> shift) & 255u);
}

/* red[0..3] smallest image, red[4..7] largest (non-NULL rows), red[8..11] nonzero when the key has a NULL */
__global__ void __launch_bounds__(TSEL_THREADS)
k_tsel_image(TselKeys p, int64_t n, unsigned long long *red)
{
	unsigned long long mn[TOPN_MAXKEYS],
				mx[TOPN_MAXKEYS];
	unsigned	nulls = 0;

#pragma unroll
	for (int i = 0; i < TOPN_MAXKEYS; i++)
	{
		mn[i] = ~0ull;
		mx[i] = 0;
	}
	for (int64_t r = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t) gridDim.x * blockDim.x)
#pragma unroll
		for (int i = 0; i < TOPN_MAXKEYS; i++)
			if (i < p.nkeys)
			{
				bool		isnull;
				const unsigned long long u = tsel_image(p.k[i], (uint32_t) r, &isnull);

				if (isnull)
					nulls |= 1u << i;
				else
				{
					mn[i] = u < mn[i] ? u : mn[i];
					mx[i] = u > mx[i] ? u : mx[i];
				}
			}
	nulls = __reduce_or_sync(0xffffffffu, nulls);
#pragma unroll
	for (int i = 0; i < TOPN_MAXKEYS; i++)
		if (i < p.nkeys)
		{
			for (int o = 16; o > 0; o >>= 1)
			{
				const unsigned long long a = __shfl_xor_sync(0xffffffffu, mn[i], o);
				const unsigned long long b = __shfl_xor_sync(0xffffffffu, mx[i], o);

				mn[i] = a < mn[i] ? a : mn[i];
				mx[i] = b > mx[i] ? b : mx[i];
			}
			if ((threadIdx.x & 31) == 0)
			{
				atomicMin(red + i, mn[i]);
				atomicMax(red + TOPN_MAXKEYS + i, mx[i]);
				if ((nulls >> i) & 1)
					atomicOr(red + 2 * TOPN_MAXKEYS + i, 1ull);
			}
		}
}

/* the rows a count / scatter CTA owns: a contiguous chunk of the *nrows input positions */
__device__ __forceinline__ void
tsel_chunk(const unsigned long long *nrows, int64_t *lo, int64_t *hi)
{
	const int64_t n = (int64_t) *nrows;
	const int64_t chunk = (n + gridDim.x - 1) / gridDim.x;

	*lo = (int64_t) blockIdx.x * chunk < n ? (int64_t) blockIdx.x * chunk : n;
	*hi = *lo + chunk < n ? *lo + chunk : n;
}

/* cnt[CTA][digit]: how many of the CTA's rows have each digit; in = NULL reads rows 0 .. n-1.  st: a selection pass */
__global__ void __launch_bounds__(TSEL_THREADS)
k_tsel_count(TselKey k, int shift, const uint32_t *in, const unsigned long long *nrows, const TselState *st, uint32_t *cnt)
{
	__shared__ uint32_t h[256];
	int64_t		lo,
				hi;

	if (st && st->decided >= 0)
		return;
	h[threadIdx.x] = 0;
	__syncthreads();
	tsel_chunk(nrows, &lo, &hi);
	for (int64_t i0 = lo; i0 < hi; i0 += blockDim.x)
	{
		const int64_t i = i0 + threadIdx.x;
		const int	d = i < hi ? tsel_digit(k, shift, in ? in[i] : (uint32_t) i) : -1;
		/* one shared-memory atomic per digit and warp: a tied key puts every row on the same counter */
		const unsigned peers = __match_any_sync(0xffffffffu, d);

		if (d >= 0 && (int) (threadIdx.x & 31) == __ffs(peers) - 1)
			atomicAdd(h + d, (uint32_t) __popc(peers));
	}
	__syncthreads();
	cnt[(int64_t) blockIdx.x * 256 + threadIdx.x] = h[threadIdx.x];
}

/* one CTA, one thread per digit value: where each (CTA, digit) run of rows goes (off).  Sorting: after every row of a smaller
 * digit.  Selecting (st): the digit b where the remaining rank falls; rows of smaller digits are chosen (after those chosen
 * before), rows of digit b are the next tied set - or chosen too when the rank ends with them, which decides the selection */
__global__ void __launch_bounds__(256)
k_tsel_plan(const uint32_t *cnt, int grid, TselState *st, int pass, uint32_t *off)
{
	__shared__ unsigned long long cum[257];	/* cum[d]: rows with a smaller digit */
	__shared__ int chosen;
	const int	d = threadIdx.x;
	unsigned long long tot = 0,
				base;

	if (st && st->decided >= 0)
		return;
	for (int c = 0; c < grid; c++)
		tot += cnt[(int64_t) c * 256 + d];
	cum[d + 1] = tot;
	if (d == 0)
		cum[0] = 0;
	__syncthreads();
	for (int s = 1; s < 256; s <<= 1)
	{
		const unsigned long long add = d + 1 > s ? cum[d + 1 - s] : 0;

		__syncthreads();
		cum[d + 1] += add;
		__syncthreads();
	}
	base = cum[d];
	if (st)
	{
		const unsigned long long need = st->need;

		if (cum[d] < need && need <= cum[d + 1])
			chosen = d;
		__syncthreads();
		const int	b = chosen;
		const bool	take = cum[b + 1] == need;

		base = (d < b || (d == b && take)) ? st->nsel + cum[d] : 0;
		__syncthreads();	/* every thread has read st */
		if (d == 0)
		{
			st->bucket[pass] = b;
			st->take[pass] = take;
			st->nsel += take ? cum[b + 1] : cum[b];
			st->need = take ? 0 : need - cum[b];
			st->ntied[pass + 1] = take ? 0 : cum[b + 1] - cum[b];
			if (take)
				st->decided = pass;
		}
	}
	for (int c = 0; c < grid; c++)
	{
		off[(int64_t) c * 256 + d] = (uint32_t) base;
		base += cnt[(int64_t) c * 256 + d];
	}
}

/* each row to off[CTA][digit] plus its rank among the CTA's earlier rows of that digit: the rows of a tile by warp, the rows
 * of a warp by lane.  Sorting: every row to out.  Selecting (st): digits below the chosen one to out, the chosen one to
 * out_eq (or out when it completes the selection), larger digits nowhere */
__global__ void __launch_bounds__(TSEL_THREADS)
k_tsel_scatter(TselKey k, int shift, const uint32_t *in, const unsigned long long *nrows, const TselState *st, int pass,
			   const uint32_t *off, uint32_t *out, uint32_t *out_eq)
{
	__shared__ uint32_t cur[256];
	__shared__ uint32_t wpos[TSEL_THREADS / 32][256];	/* rows per (warp, digit) of a tile, then where each warp's run starts */
	const int	lane = threadIdx.x & 31,
				warp = threadIdx.x >> 5;
	int			b = 256,
				take = 1;
	int64_t		lo,
				hi;

	if (st && st->decided >= 0 && st->decided < pass)
		return;
	if (st)
	{
		b = st->bucket[pass];
		take = st->take[pass];
	}
	cur[threadIdx.x] = off[(int64_t) blockIdx.x * 256 + threadIdx.x];
	tsel_chunk(nrows, &lo, &hi);
	for (int64_t i0 = lo; i0 < hi; i0 += blockDim.x)
	{
		const int64_t i = i0 + threadIdx.x;
		const uint32_t row = i < hi ? (in ? in[i] : (uint32_t) i) : 0;
		const int	d = i < hi ? tsel_digit(k, shift, row) : -1;
		const unsigned peers = __match_any_sync(0xffffffffu, d);

		for (int w = 0; w < TSEL_THREADS / 32; w++)
			wpos[w][threadIdx.x] = 0;
		__syncthreads();
		if (d >= 0 && lane == __ffs(peers) - 1)
			wpos[warp][d] = (uint32_t) __popc(peers);
		__syncthreads();
		{
			uint32_t	run = cur[threadIdx.x];

			for (int w = 0; w < TSEL_THREADS / 32; w++)
			{
				const uint32_t c = wpos[w][threadIdx.x];

				wpos[w][threadIdx.x] = run;
				run += c;
			}
			cur[threadIdx.x] = run;
		}
		__syncthreads();
		if (d >= 0 && d <= b)
		{
			const uint32_t at = wpos[warp][d] + (uint32_t) __popc(peers & ((1u << lane) - 1));

			if (d < b || take)
				out[at] = row;
			else
				out_eq[at] = row;
		}
		__syncthreads();
	}
}

/* a selection no digit decided: the tied set's first rows (row order) complete it; tied = NULL: rows 0 .. */
__global__ void
k_tsel_finish(const uint32_t *tied, const TselState *st, uint32_t *sel)
{
	if (st->decided >= 0)
		return;
	const int64_t need = (int64_t) st->need;
	const int64_t at = (int64_t) st->nsel;

	for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < need; i += (int64_t) gridDim.x * blockDim.x)
		sel[at + i] = tied ? tied[i] : (uint32_t) i;
}

extern "C" int
cbgpu_topn_select(cbgpu_ctx *ctx, cbgpu_rel *rel, const cbgpu_sort_key *keys, int32_t nkeys, int64_t limit, uint32_t *host_idx,
				  int64_t *nout)
{
	TselState	hst;				/* before mem: its copy to the device may still be queued when mem drains the stream */
	unsigned long long red[3 * TOPN_MAXKEYS];
	CbCallMem	mem(ctx);
	TselKeys	p;
	int			dshift[TSEL_MAXDIGITS],
				dkey[TSEL_MAXDIGITS],
				nd = 0;
	unsigned long long *dred = NULL;
	TselState  *st = NULL;
	uint32_t   *cnt = NULL,
			   *sel[2] = {NULL, NULL},
			   *tied[2] = {NULL, NULL};

	*nout = 0;
	if (nkeys < 1 || nkeys > TOPN_MAXKEYS)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "device top-N supports 1..4 sort keys (%s%lld keys)", "", nkeys);
	if (limit < 1)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "device top-N needs LIMIT >= 1 (%sgot %lld)", "", limit);
	memset(&p, 0, sizeof(p));
	for (int i = 0; i < nkeys; i++)
	{
		const cbgpu_sort_key *k = &keys[i];
		int			w;

		if (k->col < 0 || k->col >= rel->ncols)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_topn_select: bad key column%s %lld", "", k->col);
		w = cb_type_w(rel->types[k->col]);
		if (w != 1 && w != 4 && w != 8)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_topn_select: key column%s %lld is not 1, 4 or 8 bytes wide", "", k->col);
		if (k->float8 && w != 8)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_topn_select: float8 order over a column narrower than 8 bytes%s (column %lld)", "",
						   k->col);
		p.k[i].data = rel->data[k->col];
		p.k[i].type = rel->types[k->col];
		p.k[i].desc = k->descending != 0;
		p.k[i].uns = k->unsigned_cmp != 0;
		p.k[i].f8 = k->float8 != 0;
		if (k->nulls == CBGPU_SORT_NULLS_MAP)
			p.k[i].nullmap = rel->nulls[k->col];
		else if (k->nulls == CBGPU_SORT_NULLS_COUNT)
		{
			if (k->null_col < 0 || k->null_col >= rel->ncols || rel->types[k->null_col] != CB_INT8)
				return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_topn_select: NULL-source column%s %lld is not an int8 column", "",
							   k->null_col);
			p.k[i].ncol = (const long long *) rel->data[k->null_col];
		}
		else if (k->nulls != CBGPU_SORT_NULLS_NONE)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_topn_select: unknown NULL source%s %lld", "", k->nulls);
	}
	p.nkeys = nkeys;
	if (rel->nrows == 0)
		return CBGPU_OK;

	const int64_t n = rel->nrows;
	const int64_t m = limit < n ? limit : n;
	const int	sms = ctx->sm_count > 0 ? ctx->sm_count : 1;

	/* the image pass and its read-back: which digits can vary */
	CB_CUDA(ctx, mem.alloc(&dred, sizeof(red)));
	CB_CUDA(ctx, cudaMemsetAsync(dred, 0xFF, TOPN_MAXKEYS * sizeof(unsigned long long), ctx->stream));
	CB_CUDA(ctx, cudaMemsetAsync(dred + TOPN_MAXKEYS, 0, 2 * TOPN_MAXKEYS * sizeof(unsigned long long), ctx->stream));
	{
		const int64_t want = (n + TSEL_THREADS - 1) / TSEL_THREADS;
		const int	blocks = (int) (want < (int64_t) sms * 8 ? want : (int64_t) sms * 8);

		k_tsel_image<<<blocks, TSEL_THREADS, 0, ctx->stream>>>(p, n, dred);
		CB_LAUNCHED(ctx, "k_tsel_image");
	}
	CB_CUDA(ctx, cudaMemcpyAsync(red, dred, sizeof(red), cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	CB_CUDA(ctx, mem.free(dred));
	for (int i = 0; i < nkeys; i++)
	{
		const unsigned long long mn = red[i],
					mx = red[TOPN_MAXKEYS + i];
		const bool	values = mn <= mx;

		if (values && red[2 * TOPN_MAXKEYS + i])
		{
			dkey[nd] = i;
			dshift[nd++] = TSEL_NULLDIGIT;
		}
		if (values && mn != mx)
			for (int b = (63 - __builtin_clzll(mn ^ mx)) / 8; b >= 0; b--)
			{
				dkey[nd] = i;
				dshift[nd++] = 8 * b;
			}
	}

	/* counts and offsets of one pass: grid CTAs x 256 digits each */
	const int64_t rows_max = m < n ? n : m;
	int64_t		want = (rows_max + TSEL_THREADS - 1) / TSEL_THREADS;
	const int	grid_sel = (int) (want < (int64_t) sms * 4 ? want : (int64_t) sms * 4);
	const int	npass = m < n ? nd : 0;		/* a LIMIT that takes every row selects nothing */

	want = (m + TSEL_THREADS - 1) / TSEL_THREADS;
	const int	grid_sort = (int) (want < (int64_t) sms * 4 ? want : (int64_t) sms * 4);

	memset(&hst, 0, sizeof(hst));
	hst.need = (unsigned long long) m;
	hst.m = (unsigned long long) m;
	hst.ntied[0] = (unsigned long long) n;
	hst.decided = -1;
	CB_CUDA(ctx, mem.alloc(&st, sizeof(TselState)));
	CB_CUDA(ctx, mem.copy_in(st, &hst, sizeof(hst)));
	CB_CUDA(ctx, mem.alloc(&sel[0], (size_t) m * sizeof(uint32_t)));
	if (nd > 0)
		CB_CUDA(ctx, mem.alloc(&cnt, (size_t) 2 * 256 * (grid_sel > grid_sort ? grid_sel : grid_sort) * sizeof(uint32_t)));
	for (int t = 0; t < (npass < 2 ? npass : 2); t++)
		CB_CUDA(ctx, mem.alloc(&tied[t], (size_t) n * sizeof(uint32_t)));

	/* MSD radix select, most significant digit first */
	uint32_t   *const off = cnt ? cnt + (size_t) 256 * (grid_sel > grid_sort ? grid_sel : grid_sort) : NULL;

	for (int d = 0; d < npass; d++)
	{
		const TselKey k = p.k[dkey[d]];
		const uint32_t *in = d == 0 ? NULL : tied[(d - 1) & 1];

		k_tsel_count<<<grid_sel, TSEL_THREADS, 0, ctx->stream>>>(k, dshift[d], in, st->ntied + d, st, cnt);
		CB_LAUNCHED(ctx, "k_tsel_count");
		k_tsel_plan<<<1, 256, 0, ctx->stream>>>(cnt, grid_sel, st, d, off);
		CB_LAUNCHED(ctx, "k_tsel_plan");
		k_tsel_scatter<<<grid_sel, TSEL_THREADS, 0, ctx->stream>>>(k, dshift[d], in, st->ntied + d, st, d, off, sel[0], tied[d & 1]);
		CB_LAUNCHED(ctx, "k_tsel_scatter");
	}
	{
		const int64_t want_f = (m + TSEL_THREADS - 1) / TSEL_THREADS;
		const int	blocks = (int) (want_f < (int64_t) sms * 4 ? want_f : (int64_t) sms * 4);

		k_tsel_finish<<<blocks, TSEL_THREADS, 0, ctx->stream>>>(npass == 0 ? NULL : tied[(npass - 1) & 1], st, sel[0]);
		CB_LAUNCHED(ctx, "k_tsel_finish");
	}
	for (int t = 0; t < 2; t++)
		if (tied[t])
			CB_CUDA(ctx, mem.free(tied[t]));

	/* stable LSD radix sort of the chosen rows, least significant digit first */
	int			cur = 0;

	if (nd > 0)
		CB_CUDA(ctx, mem.alloc(&sel[1], (size_t) m * sizeof(uint32_t)));
	for (int d = nd - 1; d >= 0; d--)
	{
		const TselKey k = p.k[dkey[d]];

		k_tsel_count<<<grid_sort, TSEL_THREADS, 0, ctx->stream>>>(k, dshift[d], sel[cur], &st->m, NULL, cnt);
		CB_LAUNCHED(ctx, "k_tsel_count");
		k_tsel_plan<<<1, 256, 0, ctx->stream>>>(cnt, grid_sort, NULL, 0, off);
		CB_LAUNCHED(ctx, "k_tsel_plan");
		k_tsel_scatter<<<grid_sort, TSEL_THREADS, 0, ctx->stream>>>(k, dshift[d], sel[cur], &st->m, NULL, 0, off, sel[cur ^ 1], NULL);
		CB_LAUNCHED(ctx, "k_tsel_scatter");
		cur ^= 1;
	}
	CB_CUDA(ctx, cudaMemcpyAsync(host_idx, sel[cur], (size_t) m * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, mem.sync());
	*nout = m;
	return CBGPU_OK;
}
