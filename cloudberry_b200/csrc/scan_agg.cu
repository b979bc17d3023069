/*
 * scan_agg.cu - K1+K4 fused: columnar scan -> qual -> low-cardinality hash aggregate in one pass
 * (the TPC-H Q1 class: few groups keyed by one or two char(1)/dictionary columns, SUM/AVG/COUNT
 * over int64-scaled numerics and products of the form b*(k-c) and b*(k-c)*(k2+d)).
 *
 * What it fuses, in the reference: aocs_getnext over the projected columns (backend/access/aocs/
 * aocsam.c:1418,1138), the pushed-down scan qual (aocsam.c:1269, execScan.c:162), the numeric
 * arithmetic of the aggregate arguments (numeric_mul / numeric_sub, backend/utils/adt/numeric.c:
 * 2645,2567 - here exact scaled-integer products), LookupTupleHashEntry (backend/executor/
 * execGrouping.c:317) and the transition functions (numeric_avg_accum, int8inc: nodeAgg.c:856).
 *
 * Shape: one persistent CTA per SM.  A producer warp streams the projected columns into a
 * shared-memory ring with TMA bulk copies (cp.async.bulk + mbarrier; SASS UBLKCP / SYNCS), several
 * tiles ahead of the consumers, so the HBM pipe stays full whatever the consumers do.  Consumer
 * warps read rows from shared memory, evaluate the qual and the arithmetic, and accumulate per
 * group in registers (G <= 4 or 8 slots; slot keys live in a per-CTA shared table, cached in
 * registers).  Per-CTA totals are reduced with shuffles and committed once per CTA and group into
 * the global aggregate table with exact 128-bit adds.
 * HBM-bound by design: algorithmic bytes/row = sum of the projected column widths (Q1: 38 B/row).
 *
 * Exactness: per-row products and per-thread partial sums are 64-bit.  The kernel ORs the raw
 * input magnitudes per column and audits, from those bit counts, that no product or partial sum
 * could have left 63 bits (and, in the NARROW variant, that the 32-bit multiply-accumulate form was
 * valid).  A failed audit commits nothing; the host re-runs the next wider variant and finally the
 * generic kernel, whose every operation is overflow-checked.  Group totals are 128-bit.
 */
#include "pipeline.cuh"
#include "xmatch.h"

#define SA_NSUM 6				/* sA sB sC sD sREV sCHG */

struct SmallAggParams
{
	int64_t		nrows;
	const long long *colA;		/* optional plain column                                              */
	const long long *colB;		/* b of b*(k-c)                                                       */
	const long long *colC;
	const long long *colD;		/* optional: d of (k2+d), or a second plain column                    */
	long long	k,
				k2;
	const int32_t *fcol;		/* optional filter column (int4/date)                                 */
	int32_t		flo;			/* the qual folded to a closed range: flo <= value <= flo + fspan     */
	uint32_t	fspan;
	const uint8_t *key0;		/* optional group key columns (char(1) / dictionary code)             */
	const uint8_t *key1;
	const uint8_t *visimap;
	/* commit: agg accumulator a takes sum index accsum[a] (0..5) or -1 for a pure count */
	AggDev		agg;
	int32_t		nkeys;
	int32_t		keytype[2];
	const uint32_t *keydict[2];
	int32_t		naccs;
	int32_t		accsum[CBP_MAX_AGGS];
	int32_t		want_chg;		/* the b*(k-c)*(k2+d) sum is requested                                */
	int		   *status;
	int		   *retry;			/* set when a CTA saw more than G distinct groups                     */
	int		   *audit;			/* set when this variant's arithmetic could have overflowed           */
	AggSnap    *snap;			/* pinned host: k_small_commit reports the flags and, for small tables, the groups  */
	int			snap_groups;	/* 1: the table is small enough to be snapshotted                     */
	/* per-CTA partial results, committed by k_small_commit once no CTA raised retry / audit */
	unsigned long long *scratch;	/* [grid][G][SA_NSUM + 1][2]                                      */
	unsigned   *skeys;			/* [grid][G]                                                          */
};

template <int G>
struct SaAcc
{
	unsigned	cnt[G];
	long long	s[G][SA_NSUM];
};

/*
 * acc += hit * v with hit in {0, 1}.
 * Wide form: IMAD.WIDE.U32 (hit * v.lo + acc, a 64-bit add with carry) + IMAD (hit * v.hi + acc.hi):
 * two fma-pipe instructions per accumulator and row, no compare / select per accumulator; two's
 * complement makes it exact for negative v.  Narrow form (v known to fit 32 unsigned bits, audited
 * after the fact): the IMAD.WIDE.U32 alone.
 */
template <bool NARROW>
__device__ __forceinline__ void
sa_madd(long long &acc, unsigned hit, long long v)
{
	if (NARROW)
		asm("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc) : "r"(hit), "r"((unsigned) v));
	else
		asm("{\n\t"
			".reg .b32 vlo, vhi, tlo, thi;\n\t"
			".reg .b64 t;\n\t"
			"mov.b64 {vlo, vhi}, %2;\n\t"
			"mad.wide.u32 t, %1, vlo, %0;\n\t"
			"mov.b64 {tlo, thi}, t;\n\t"
			"mad.lo.u32 thi, %1, vhi, thi;\n\t"
			"mov.b64 %0, {tlo, thi};\n\t"
			"}"
			: "+l"(acc) : "r"(hit), "l"(v));
}

/* slow path, once per new group per thread: claim a slot in the CTA's shared key table */
template <int G>
__device__ __noinline__ void
sa_insert_key(unsigned *gkeys, unsigned key, int *retry)
{
	bool		placed = false;

	for (int g = 0; g < G && !placed; g++)
	{
		unsigned	cur = ((volatile unsigned *) gkeys)[g];

		if (cur == 0)
			cur = atomicCAS(gkeys + g, 0u, key);
		if (cur == 0 || cur == key)
			placed = true;
	}
	if (!placed)
		atomicExch(retry, 1);	/* more distinct groups than register slots */
}

/* TMA bulk-copy pipeline primitives (mbar_*, tma_load_1d): common.cuh */
#define SA_TILE 896				/* rows per pipeline stage                                            */
#define SA_STAGES 5
/* consumer threads (one extra warp produces): 448 + 32 threads leave 128 registers per thread for
 * the 4-group kernel; the 8-group kernel needs twice the accumulators and runs half the threads */
#define SA_NCONS(G) ((G) <= 4 ? 448 : 224)

struct __align__(128) SaStage
{
	long long	a[SA_TILE];
	long long	b[SA_TILE];
	long long	c[SA_TILE];
	long long	d[SA_TILE];
	int32_t		f[SA_TILE];
	uint8_t		k0[SA_TILE];
	uint8_t		k1[SA_TILE];
};

/* per-thread consumer state */
template <int G>
struct SaState
{
	SaAcc<G>	acc;
	unsigned	gk[G];			/* cached copy of the CTA's group key table                           */
	unsigned long long magAB,	/* OR of the raw a / b, c and d values seen (sign bits included)      */
				magC, magD;
	unsigned	rows_seen;
};

/*
 * one row.  MASK: which of the six sums are wanted (bit s = sum s; the host sets bit 0 / bits 3,5
 * only when column a / d exists).  SHAPE: which optional inputs exist, fixed at compile time so
 * the row loop carries no per-row presence tests: 1 = qual column + two key columns (the Q1 shape),
 * 2 = qual column, no keys (Q6 shape), 0 = decided at run time.  CHECK: bounds / visimap tests
 * (last tile, relations with a visibility map).
 */
template <int G, int MASK, bool NARROW, int SHAPE, bool CHECK>
__device__ __forceinline__ void
sa_row(const SmallAggParams &P, SaState<G> &S, unsigned *gkeys, const SaStage *st, int r, int rows, int64_t r0)
{
	const bool	hasF = SHAPE ? true : P.fcol != NULL;
	const bool	hasK0 = SHAPE == 1 ? true : (SHAPE == 2 ? false : P.key0 != NULL);
	const bool	hasK1 = SHAPE == 1 ? true : (SHAPE == 2 ? false : P.key1 != NULL);
	bool		pass = true;
	long long	a = (MASK & 1) ? st->a[r] : 0;
	long long	b = st->b[r];
	long long	c = st->c[r];
	long long	d = (MASK & 0x28) ? st->d[r] : 0;
	int32_t		f = hasF ? st->f[r] : P.flo;
	unsigned	k0 = hasK0 ? st->k0[r] : 0;
	unsigned	k1 = hasK1 ? st->k1[r] : 0;

	if (CHECK)
	{
		pass = r < rows;
		if (!pass)
			a = b = c = d = 0;	/* stale shared memory must not reach the audit masks */
		if (P.visimap && pass)
		{
			/* AppendOnlyVisimap_IsVisible (access/appendonly/appendonly_visimap.c:198) */
			const int64_t gr = r0 + r;

			pass = (__ldg(P.visimap + (gr >> 3)) >> (gr & 7)) & 1;
		}
	}
	/* the qual as a closed range (EQ/LT/LE/GT/GE folded by the host): one unsigned compare */
	pass = pass && ((unsigned) (f - P.flo) <= P.fspan);
	long long	kc = P.k - c;
	long long	rev = b * kc;
	long long	chg = (MASK & 0x20) ? rev * (P.k2 + d) : 0;
	/* the key carries a valid bit (0 = empty slot); a row that fails the qual gets a key no slot holds */
	unsigned	key = pass ? (0x10000u | k0 | (k1 << 8)) : 0xFFFFFFFFu;
	unsigned	hit[G];
	unsigned	known = 0;

#pragma unroll
	for (int g = 0; g < G; g++)
	{
		hit[g] = key == S.gk[g] ? 1u : 0u;
		known |= hit[g];
	}
	if (pass && !known)
	{
		sa_insert_key<G>(gkeys, key, P.retry);
#pragma unroll
		for (int g = 0; g < G; g++)
		{
			S.gk[g] = ((volatile unsigned *) gkeys)[g];
			hit[g] = key == S.gk[g] ? 1u : 0u;
		}
	}
	/* audit masks take every in-range row (also rows the qual rejects: only more conservative) */
	S.magAB |= (unsigned long long) (a | b);
	S.magC |= (unsigned long long) c;
	S.magD |= (unsigned long long) d;
	S.rows_seen += pass ? 1u : 0u;
#pragma unroll
	for (int g = 0; g < G; g++)
	{
		S.acc.cnt[g] += hit[g];
		if (MASK & 0x01)
			sa_madd<NARROW>(S.acc.s[g][0], hit[g], a);
		if (MASK & 0x02)
			sa_madd<NARROW>(S.acc.s[g][1], hit[g], b);
		if (MASK & 0x04)
			sa_madd<NARROW>(S.acc.s[g][2], hit[g], c);
		if (MASK & 0x08)
			sa_madd<NARROW>(S.acc.s[g][3], hit[g], d);
		if (MASK & 0x10)
			sa_madd<NARROW>(S.acc.s[g][4], hit[g], rev);
		if (MASK & 0x20)
			sa_madd<false>(S.acc.s[g][5], hit[g], chg);
	}
}

/*
 * One persistent CTA per SM.  Warp 0 is the producer: for each tile it arms the stage's "full"
 * mbarrier with the byte count and issues one TMA bulk copy per projected column
 * (cp.async.bulk global -> shared), up to SA_STAGES tiles ahead, so ~170 KB of loads are in flight
 * per SM regardless of what the consumers are doing.  The consumer warps wait on "full", read
 * their rows from shared memory (row-per-thread, conflict free), evaluate the qual and the
 * arithmetic, accumulate per group in registers, and release the stage through "empty".
 */
template <int G, int MASK, bool NARROW, int SHAPE>
__global__ void __launch_bounds__(SA_NCONS(G) + 32, 1)
k_scan_agg_small(const __grid_constant__ SmallAggParams P)
{
	extern __shared__ __align__(128) unsigned char smem_raw[];
	SaStage    *stages = (SaStage *) smem_raw;
	__shared__ uint64_t full_bar[SA_STAGES];
	__shared__ uint64_t empty_bar[SA_STAGES];
	__shared__ unsigned gkeys[G];
	__shared__ unsigned long long red[G][SA_NSUM + 1][2];	/* 128-bit CTA totals                     */
	constexpr int NCONS = SA_NCONS(G);
	SaState<G>	S;
	const int	warp = threadIdx.x >> 5;
	const int	lane = threadIdx.x & 31;
	const int64_t ntiles = (P.nrows + SA_TILE - 1) / SA_TILE;

	if (threadIdx.x == 0)
	{
		for (int s = 0; s < SA_STAGES; s++)
		{
			mbar_init(&full_bar[s], 1);
			mbar_init(&empty_bar[s], NCONS / 32);
		}
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	if (threadIdx.x < G)
		gkeys[threadIdx.x] = 0;
	for (int i = threadIdx.x; i < G * (SA_NSUM + 1) * 2; i += blockDim.x)
		(&red[0][0][0])[i] = 0;
	S.magAB = S.magC = S.magD = 0;
	S.rows_seen = 0;
#pragma unroll
	for (int g = 0; g < G; g++)
	{
		S.acc.cnt[g] = 0;
		S.gk[g] = 0;
#pragma unroll
		for (int s = 0; s < SA_NSUM; s++)
			S.acc.s[g][s] = 0;
	}
	__syncthreads();

	if (warp == 0)
	{
		/* ---- producer ---- */
		if (lane == 0)
		{
			int			it = 0;

			for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x, it++)
			{
				const int	s = it % SA_STAGES;
				const unsigned ph = (it / SA_STAGES) & 1;
				const int64_t r0 = t * SA_TILE;
				const int64_t rows = P.nrows - r0 < SA_TILE ? P.nrows - r0 : SA_TILE;
				/* bulk copies move multiples of 16 bytes; relations are allocated padded, so the
				 * few bytes past the last row are readable and simply ignored */
				const unsigned b8 = (unsigned) (rows * 8 + 15) & ~15u;
				const unsigned b4 = (unsigned) (rows * 4 + 15) & ~15u;
				const unsigned b1 = (unsigned) (rows + 15) & ~15u;
				const bool	wantA = (MASK & 1) != 0;
				const bool	wantD = (MASK & 0x28) != 0;
				unsigned	total = 2 * b8 + (wantA ? b8 : 0) + (wantD ? b8 : 0) + (P.fcol ? b4 : 0) +
					(P.key0 ? b1 : 0) + (P.key1 ? b1 : 0);
				SaStage    *st = &stages[s];

				mbar_wait(&empty_bar[s], ph ^ 1);
				mbar_expect_tx(&full_bar[s], total);
				tma_load_1d(st->b, P.colB + r0, b8, &full_bar[s]);
				tma_load_1d(st->c, P.colC + r0, b8, &full_bar[s]);
				if (wantA)
					tma_load_1d(st->a, P.colA + r0, b8, &full_bar[s]);
				if (wantD)
					tma_load_1d(st->d, P.colD + r0, b8, &full_bar[s]);
				if (P.fcol)
					tma_load_1d(st->f, P.fcol + r0, b4, &full_bar[s]);
				if (P.key0)
					tma_load_1d(st->k0, P.key0 + r0, b1, &full_bar[s]);
				if (P.key1)
					tma_load_1d(st->k1, P.key1 + r0, b1, &full_bar[s]);
			}
		}
	}
	else
	{
		/* ---- consumers ---- */
		const int	ct = threadIdx.x - 32;
		int			it = 0;

		for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x, it++)
		{
			const int	s = it % SA_STAGES;
			const unsigned ph = (it / SA_STAGES) & 1;
			const int64_t r0 = t * SA_TILE;
			const int	rows = (int) (P.nrows - r0 < SA_TILE ? P.nrows - r0 : SA_TILE);
			const SaStage *st = &stages[s];

			mbar_wait(&full_bar[s], ph);
			if (rows == SA_TILE && !P.visimap)
			{
#pragma unroll
				for (int j = 0; j < SA_TILE / NCONS; j++)
					sa_row<G, MASK, NARROW, SHAPE, false>(P, S, gkeys, st, ct + j * NCONS, rows, r0);
			}
			else
			{
#pragma unroll
				for (int j = 0; j < SA_TILE / NCONS; j++)
					sa_row<G, MASK, NARROW, SHAPE, true>(P, S, gkeys, st, ct + j * NCONS, rows, r0);
			}
			/* this warp is done with the stage: one arrival per consumer warp frees it */
			__syncwarp();
			if (lane == 0)
				mbar_arrive(&empty_bar[s]);
		}
	}

	/* overflow audit.  The masks OR every raw input of their column (a negative value sets bit 63 and
	 * fails the audit).  |k - c| < 2^(max(bits c, bits k) + 1), likewise k2 + d; a product has at most
	 * the sum of its factors' bit counts, a thread's partial sum at most bits(value) + bits(rows
	 * accumulated); all must stay below 63 bits.  NARROW additionally needs every single-IMAD
	 * operand (a, b, c, d, b*(k-c)) in [0, 2^32): below 2^32 by the bit counts, and b*(k-c) not
	 * negative, which holds when every c seen is at most k (c < 2^bc, so 2^bc - 1 <= k proves it). */
	{
		int			bab = 64 - __clzll(S.magAB),
					bc = 64 - __clzll(S.magC),
					bd = 64 - __clzll(S.magD);
		unsigned long long ak = (unsigned long long) (P.k < 0 ? -P.k : P.k),
					ak2 = (unsigned long long) (P.k2 < 0 ? -P.k2 : P.k2);
		int			bk = 64 - __clzll(ak),
					bk2 = 64 - __clzll(ak2);
		int			brev = bab + (bc > bk ? bc : bk) + 1;
		int			bchg = (MASK & 0x20) ? brev + (bd > bk2 ? bd : bk2) + 1 : 0;
		int			brows = 32 - __clz(S.rows_seen);
		int			worst = brev > bchg ? brev : bchg;

		if (bc > worst)
			worst = bc;
		if (bd > worst)
			worst = bd;
		if (worst + brows >= 63)
			atomicExch(P.audit, 1);
		if (NARROW && (bab > 32 || bc > 32 || bd > 32 || ((MASK & 0x10) && brev > 32)))
			atomicExch(P.audit, 1);
		if (NARROW && (MASK & 0x10) && (P.k < 0 || bc > 62 || (long long) ((1ull << bc) - 1) > P.k))
			atomicExch(P.audit, 1);
		/* negative inputs: the unsigned narrow form and the bit-count bounds do not hold */
		if ((long long) (S.magAB | S.magC | S.magD) < 0)
			atomicExch(P.audit, 1);
	}

	/* CTA reduction: warp shuffle, then one 128-bit shared add per warp, group and sum */
#pragma unroll
	for (int g = 0; g < G; g++)
	{
#pragma unroll
		for (int s = 0; s <= SA_NSUM; s++)
		{
			long long	v = s < SA_NSUM ? S.acc.s[g][s < SA_NSUM ? s : 0] : (long long) S.acc.cnt[g];

			if (s < SA_NSUM && !((MASK >> s) & 1))
				continue;
			/* per-thread partials fit 63 bits (audited above); 32 of them need up to 68 bits, so
			 * reduce (lo, hi) pairs */
			unsigned long long lo = (unsigned long long) v;
			long long	hi = v < 0 ? -1 : 0;

#pragma unroll
			for (int o = 16; o; o >>= 1)
			{
				unsigned long long lo2 = __shfl_xor_sync(0xffffffffu, lo, o);
				long long	hi2 = __shfl_xor_sync(0xffffffffu, hi, o);
				unsigned long long nl = lo + lo2;

				hi = hi + hi2 + (nl < lo ? 1 : 0);
				lo = nl;
			}
			if (lane == 0 && (lo | (unsigned long long) hi))
			{
				unsigned long long old = atomicAdd(&red[g][s][0], lo);

				atomicAdd(&red[g][s][1], (unsigned long long) hi + (old + lo < old ? 1ull : 0ull));
			}
		}
	}
	__syncthreads();

	/* park the CTA's totals; k_small_commit folds them into the aggregate table */
	for (int i = threadIdx.x; i < G * (SA_NSUM + 1) * 2; i += blockDim.x)
		P.scratch[(size_t) blockIdx.x * G * (SA_NSUM + 1) * 2 + i] = (&red[0][0][0])[i];
	if (threadIdx.x < G)
		P.skeys[(size_t) blockIdx.x * G + threadIdx.x] = gkeys[threadIdx.x];
}

/* commit each (CTA, group) partial once: find-or-insert by the reference's group hash
 * (TupleHashTableHash_internal, executor/execGrouping.c:437-495), then exact 128-bit adds */
__global__ void
k_small_commit(const __grid_constant__ SmallAggParams P, int G, int nblocks)
{
	/* ONE CTA (the host launches <<<1, 256>>>): commit, then report - flags, and for a small table its groups - straight
	 * into pinned host memory, so the step's fate and its result arrive with one synchronisation */
	if (*P.retry || *P.audit)
	{
		if (threadIdx.x == 0)
		{
			P.snap->retry = *P.retry;
			P.snap->audit = *P.audit;
			P.snap->ngroups = -1;
			__threadfence_system();
		}
		return;
	}
	if (threadIdx.x == 0)
		P.snap->retry = P.snap->audit = 0;
	for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < nblocks * G; e += gridDim.x * blockDim.x)
	{
		unsigned	key = P.skeys[e];
		const unsigned long long *r = P.scratch + (size_t) e * (SA_NSUM + 1) * 2;
		unsigned long long cnt = r[SA_NSUM * 2];

		if (key == 0 || cnt == 0)
			continue;
		int64_t		kv[2] = {(int64_t) (key & 0xff), (int64_t) ((key >> 8) & 0xff)};
		int			slot = agg_find_or_insert(P.agg, agg_group_hash(P.nkeys, P.keytype, P.keydict, kv, 0), kv, 0);

		if (slot < 0)
			continue;
		for (int a = 0; a < P.naccs; a++)
		{
			int			s = P.accsum[a];

			atomicAdd((unsigned long long *) (P.agg.n + (size_t) slot * P.agg.naccs + a), cnt);
			if (s >= 0)
				atomic_add128(P.agg.sum + ((size_t) slot * P.agg.naccs + a) * 2, r[s * 2], r[s * 2 + 1]);
		}
	}
	__syncthreads();
	if (P.snap_groups)
		agg_snapshot_block(P.agg, P.snap);
	else
	{
		if (threadIdx.x == 0)
			P.snap->ngroups = -1;
		__threadfence_system();
	}
}

/* ---------------------------------------------------------------------------------------------
 * matcher: does the descriptor have the small-group scan->agg shape?
 * --------------------------------------------------------------------------------------------- */
static bool
col_plain(const CbPipeline *p, int c, int width)
{
	return p->cols[c].src == 0 && p->cols[c].nulls == NULL && cb_type_w(p->cols[c].type) == width &&
		p->cols[c].type != CB_FLOAT8;
}

static int
try_small_agg(cbgpu_ctx *ctx, const CbPipeline *p, const PipeDev *d, const XProg *xp, bool *handled)
{
	const XProg &x = *xp;
	SmallAggParams P;
	int			colB = -1,
				colC = -1,
				colD = -1,
				colA = -1;
	int64_t		k = 0,
				k2 = 0;
	bool		have_rev = false,
				have_chg = false;
	const CbpSink *s = &p->sink;

	*handled = false;
	if (s->kind != CBP_SINK_AGG || p->nprobes != 0 || p->drv_nsrc != 0 || s->nkeys > 2)
		return CBGPU_OK;
	if (x.f8ord || x.inset || x.depth < s->nkeys)
		return CBGPU_OK;
	memset(&P, 0, sizeof(P));
	P.fspan = 0xFFFFFFFFu;		/* no qual: every value is inside the range */
	/* quals: at most one CMP(int32 column, const) */
	if (x.nsections > 1)
		return CBGPU_OK;
	if (x.nsections == 1)
	{
		int			code,
					col;
		int64_t		v,
					lo,
					hi;

		if (x.sections[0].kind != 0 || !xm_is_cmp_const(&x, x.sections[0].node, &code, &col, &v) ||
			!col_plain(p, col, 4) || v < INT32_MIN || v > INT32_MAX || !xm_qual_range(code, v, INT32_MIN, INT32_MAX, &lo, &hi))
			return CBGPU_OK;
		P.fcol = (const int32_t *) p->cols[col].data;
		P.flo = (int32_t) lo;
		P.fspan = (uint32_t) (hi - lo);
	}
	/* keys: one-byte columns */
	for (int i = 0; i < s->nkeys; i++)
	{
		int			col;

		if (!xm_is_load(&x, x.stack[i], &col) || !col_plain(p, col, 1))
			return CBGPU_OK;
		if (i == 0)
			P.key0 = (const uint8_t *) p->cols[col].data;
		else
			P.key1 = (const uint8_t *) p->cols[col].data;
		P.keytype[i] = s->keytype[i];
		P.keydict[i] = s->key_dict_hash[i];
	}
	/* first pass over the accumulators: find the product terms, they fix b, c, d */
	for (int a = 0; a < s->naccs; a++)
	{
		int			b,
					c,
					dd;
		int64_t		kk,
					kk2;

		if (s->accs[a].kind == CBP_ACC_COUNT && s->accs[a].arg < 0)
			continue;
		if (s->accs[a].kind != CBP_ACC_SUM_INT)
			return CBGPU_OK;
		int			node = x.stack[s->nkeys + s->accs[a].arg];

		if (xm_is_chg(&x, node, &b, &kk, &c, &kk2, &dd))
		{
			if ((have_rev || have_chg) && (b != colB || c != colC || kk != k))
				return CBGPU_OK;
			if (have_chg && (dd != colD || kk2 != k2))
				return CBGPU_OK;
			colB = b; colC = c; colD = dd; k = kk; k2 = kk2;
			have_chg = true;
		}
		else if (xm_is_rev(&x, node, &b, &kk, &c))
		{
			if ((have_rev || have_chg) && (b != colB || c != colC || kk != k))
				return CBGPU_OK;
			colB = b; colC = c; k = kk;
			have_rev = true;
		}
	}
	if (!have_rev && !have_chg)
		return CBGPU_OK;		/* plain-column-only aggregates go to the generic kernel for now */
	/* second pass: map every accumulator onto one of the six sums */
	P.naccs = s->naccs;
	for (int a = 0; a < s->naccs; a++)
	{
		int			b,
					c,
					dd,
					col;
		int64_t		kk,
					kk2;

		if (s->accs[a].kind == CBP_ACC_COUNT)
		{
			P.accsum[a] = -1;
			continue;
		}
		int			node = x.stack[s->nkeys + s->accs[a].arg];

		if (xm_is_chg(&x, node, &b, &kk, &c, &kk2, &dd))
			P.accsum[a] = 5;
		else if (xm_is_rev(&x, node, &b, &kk, &c))
			P.accsum[a] = 4;
		else if (xm_is_load(&x, node, &col))
		{
			if (col == colB)
				P.accsum[a] = 1;
			else if (col == colC)
				P.accsum[a] = 2;
			else if (col == colD)
				P.accsum[a] = 3;
			else if (colA < 0 || col == colA)
			{
				colA = col;
				P.accsum[a] = 0;
			}
			else if (colD < 0)
			{
				colD = col;		/* a second free column rides in d's slot (k2 stays 0: unused) */
				P.accsum[a] = 3;
			}
			else
				return CBGPU_OK;
		}
		else
			return CBGPU_OK;
	}
	if (!col_plain(p, colB, 8) || !col_plain(p, colC, 8) || (colA >= 0 && !col_plain(p, colA, 8)) ||
		(colD >= 0 && !col_plain(p, colD, 8)))
		return CBGPU_OK;
	P.nrows = p->nrows;
	P.colA = colA >= 0 ? (const long long *) p->cols[colA].data : NULL;
	P.colB = (const long long *) p->cols[colB].data;
	P.colC = (const long long *) p->cols[colC].data;
	P.colD = colD >= 0 ? (const long long *) p->cols[colD].data : NULL;
	P.k = k;
	P.k2 = k2;
	P.visimap = p->visimap;
	P.agg = d->sink.agg;
	P.nkeys = s->nkeys;
	P.status = ctx->d_status;

	P.want_chg = have_chg;

	/* which of the six sums does the plan need? */
	int			need = 0;

	for (int a = 0; a < s->naccs; a++)
		if (P.accsum[a] >= 0)
			need |= 1 << P.accsum[a];
	if (have_chg)
		need |= 0x20;

	/* instantiated sum masks, cheapest first: b*(k-c) alone (Q3/Q5/Q10-style revenue), the Q1 set
	 * (a, b, c, rev, chg), everything.  A mask that reads column a / d needs that column. */
	static const int masks[3] = {0x10, 0x37, 0x3f};
	int			mask = -1;

	for (int i = 0; i < 3 && mask < 0; i++)
		if ((need & ~masks[i]) == 0 && (!(masks[i] & 0x01) || P.colA) && (!(masks[i] & 0x28) || P.colD))
			mask = masks[i];
	if (mask < 0)
		return CBGPU_OK;		/* e.g. a and d both absent but a plain sum wanted elsewhere: generic kernel */
	const int	shape = (P.fcol && P.key0 && P.key1) ? 1 : ((P.fcol && !P.key0 && !P.key1) ? 2 : 0);

	int		   *d_flags;
	int64_t		ntiles = (p->nrows + SA_TILE - 1) / SA_TILE;
	int			blocks = ctx->sm_count;
	const size_t smem = sizeof(SaStage) * SA_STAGES;
	int			G = 4;
	bool		narrow = true;

	if (blocks > ntiles)
		blocks = (int) ntiles;
	{
		/* per-context device scratch, kept between queries: [flags 256 B][per-CTA partial sums][per-CTA keys] */
		const size_t sbytes = (size_t) blocks * 8 * (SA_NSUM + 1) * 2 * sizeof(unsigned long long);
		const size_t kbytes = (size_t) blocks * 8 * sizeof(unsigned);
		const size_t need = 256 + sbytes + ((kbytes + 255) & ~(size_t) 255);

		if (ctx->small_dev_bytes < need)
		{
			if (ctx->small_dev)
			{
				CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
				CB_CUDA(ctx, cudaFree(ctx->small_dev));
				ctx->small_dev = NULL;
				ctx->small_dev_bytes = 0;
			}
			CB_CUDA(ctx, cudaMalloc(&ctx->small_dev, need));
			ctx->small_dev_bytes = need;
		}
		d_flags = (int *) ctx->small_dev;
		P.scratch = (unsigned long long *) ((char *) ctx->small_dev + 256);
		P.skeys = (unsigned *) ((char *) ctx->small_dev + 256 + sbytes);
	}
	P.retry = d_flags;
	P.audit = d_flags + 1;
	P.snap = ctx->agg_snap;
	P.snap_groups = s->agg->capacity <= AGG_SNAP_MAXCAP;
	/* ladder: (4 groups, narrow) -> wider arithmetic on a failed audit, 8 groups when a CTA saw more
	 * than 4 keys -> the generic kernel.  A failed attempt commits nothing. */
	for (;;)
	{
		CB_CUDA(ctx, cudaMemsetAsync(d_flags, 0, 2 * sizeof(int), ctx->stream));
		CB_CUDA(ctx, cudaEventRecord(ctx->ev_k0, ctx->stream));
		int			kl = cb_klog_begin(ctx, "k_scan_agg_small");
#define SA_LAUNCH(GG, MM, NN, SS) \
		do { \
			static bool attr_done = false; \
			if (!attr_done) \
			{ \
				CB_CUDA(ctx, cudaFuncSetAttribute(k_scan_agg_small<GG, MM, NN, SS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem)); \
				attr_done = true; \
			} \
			k_scan_agg_small<GG, MM, NN, SS><<<blocks, SA_NCONS(GG) + 32, smem, ctx->stream>>>(P); \
			ctx->last_kernel_name = "k_scan_agg_small<" #GG "," #MM "," #NN "," #SS ">"; \
			if (kl >= 0) \
				ctx->klog_name[kl] = ctx->last_kernel_name; \
		} while (0)
#define SA_PICK_SHAPE(MM, NN) \
		do { \
			if (shape == 1) SA_LAUNCH(4, MM, NN, 1); \
			else if (shape == 2) SA_LAUNCH(4, MM, NN, 2); \
			else SA_LAUNCH(4, MM, NN, 0); \
		} while (0)
#define SA_PICK(NN) \
		do { \
			if (mask == 0x10) SA_PICK_SHAPE(0x10, NN); \
			else if (mask == 0x37) SA_PICK_SHAPE(0x37, NN); \
			else SA_PICK_SHAPE(0x3f, NN); \
		} while (0)
		if (G == 8)
		{
			/* rare: 5..8 groups per CTA.  One instantiation: all sums, wide arithmetic. */
			if (!P.colA || !P.colD)
				break;
			SA_LAUNCH(8, 0x3f, false, 0);
		}
		else if (narrow)
			SA_PICK(true);
		else
			SA_PICK(false);
		CB_LAUNCHED(ctx, "k_scan_agg_small");
		cb_klog_end(ctx, kl);
		CB_CUDA(ctx, cudaEventRecord(ctx->ev_k1, ctx->stream));
		ctx->kernel_timed = true;
		ctx->agg_snap->ngroups = -1;
		ctx->agg_snap->retry = ctx->agg_snap->audit = 0;
		k_small_commit<<<1, 256, 0, ctx->stream>>>(P, G, blocks);
		CB_LAUNCHED(ctx, "k_small_commit");
		CB_CUDA(ctx, CB_STATUS_RIDE(ctx));
		CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		CB_STATUS_FETCHED(ctx);
		const int	h_flags[2] = {ctx->agg_snap->retry, ctx->agg_snap->audit};

		if (h_flags[1])
		{
			if (!narrow || G == 8)
				break;			/* too wide even for 64-bit partials: generic kernel */
			narrow = false;
			continue;
		}
		if (h_flags[0])
		{
			if (G == 8)
				break;			/* more than 8 groups in one CTA: generic kernel */
			G = 8;
			continue;
		}
		*handled = true;
		/* the commit kernel brought the (small) table's groups along: count and read-back are answered from here */
		cb_agg_adopt_snapshot((cbgpu_aggtable *) s->agg, ctx->agg_snap);
		break;
	}
	return CBGPU_OK;
}

int
cb_try_specialised(cbgpu_ctx *ctx, const CbPipeline *p, const PipeDev *d, const XProg *x, bool *handled)
{
	int			rc = try_small_agg(ctx, p, d, x, handled);

	if (rc != CBGPU_OK || *handled)
		return rc;
	return cb_try_probe_chain(ctx, p, d, x, handled);
}
