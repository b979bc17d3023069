/*
 * pipeline.cuh - device-side form of a pipeline descriptor and the sink primitives shared by the
 * generic and the pattern-specialised pipeline kernels.
 */
#pragma once
#include "common.cuh"

#define CBP_MAX_STAGES 12

/* internal fused opcodes produced by the host-side peephole pass (never part of the C ABI) */
#define XOP_FILTER_COL 100		/* a = col | cmp << 16, imm = constant                               */
#define XOP_PROBE_COLS 101		/* a = probe, imm = key column indexes, 8 bits each                  */
#define XOP_MULCSUB 102			/* a = colA | colB << 16, imm = k: push colA * (k - colB)            */

struct DProbe
{
	HtDev		ht;
	int32_t		jointype;
	int32_t		nkeys;
	int32_t		keytype[CBP_MAX_KEYS];
	const uint32_t *keydict[CBP_MAX_KEYS];
	int32_t		null_key_drops;
};

/* Where the rows of a MATERIALIZE or PARTITION sink go, filled once by cb_pipeline_to_dev.  Destination d takes rows at
 * positions [0, seg_cap[d]): in a direct Motion at those positions of the destination's own window (part_*), otherwise at
 * seg_base[d] + position of the output columns.  MATERIALIZE is destination 0 with seg_base 0 and the output's capacity. */
struct SinkOut
{
	int32_t		nout;
	void	   *outcol[CBP_MAX_OUT];
	uint8_t    *outnull[CBP_MAX_OUT];
	int32_t		outtype[CBP_MAX_OUT];
	unsigned long long *out_count;	/* per destination: every row routed there, stored or not            */
	/* PARTITION: cdb_route over the first nhash output columns picks the destination */
	int32_t		nhash;
	int32_t		hashtype[CBP_MAX_KEYS];
	const uint32_t *hashdict[CBP_MAX_KEYS];
	int32_t		nsegs;
	void *const *part_cols;		/* direct Motion: destination d's column c at part_cols[d * nout + c]  */
	unsigned long long *const *part_counts;	/* ... and its row counter (peer memory)               */
	uint8_t *const *part_nulls;	/* ... and its NULL bytes, for the columns in part_nullmask           */
	unsigned long long part_nullmask;
	int32_t    *part_flags;		/* a full destination ORs CBGPU_DX_OVERFLOW in here (NULL: status word) */
	int64_t		seg_base[64];
	int64_t		seg_cap[64];
};

struct DSink
{
	int32_t		kind;
	AggDev		agg;
	int32_t		nkeys;
	int32_t		keytype[CBP_MAX_GROUP_KEYS];	/* the key's hash function: a numeric key's is int8's            */
	const uint32_t *keydict[CBP_MAX_GROUP_KEYS];
	int32_t		naccs;
	CbpAcc		accs[CBP_MAX_AGGS];
	SinkOut		out;
};

struct PipeDev
{
	int64_t		nrows;
	const uint8_t *visimap;
	int32_t		drv_nsrc;
	const uint32_t *drv_idx[CBP_MAX_SRC];
	int32_t		ncols;
	CbpColumn	cols[CBP_MAX_COLS];
	int32_t		nops;
	CbpOp		ops[CBP_MAX_OPS];
	int32_t		nprobes;
	int32_t		src_base;		/* probe j's inner rows are source src_base + j                      */
	int32_t		nsrc;			/* sources in use                                                    */
	int32_t		nstages;		/* program stages (cut after every FILTER / PROBE)                   */
	int32_t		stage_pc[CBP_MAX_STAGES + 2];
	int32_t		q_off[CBP_MAX_STAGES];	/* per-warp queue b: word offset and words per entry               */
	int32_t		q_ew[CBP_MAX_STAGES];
	int32_t		q_words;		/* words of queue space per warp                                     */
	DProbe		probes[CBP_MAX_SRC - 1];
	DSink		sink;
	int		   *status;
	CbpSet		sets[CBP_MAX_SETS];	/* code sets of INSET                                             */
};

/* one accumulator update of advance_aggregates (backend/executor/nodeAgg.c:856).  `args` are the
 * stack values after the keys; argnull their NULL bits. */
__device__ __forceinline__ void
sink_acc_update(const AggDev &t, int slot, int a, const CbpAcc &acc, const int64_t *args, uint64_t argnull)
{
	int64_t    *np = t.n + (size_t) slot * t.naccs + a;
	unsigned long long *sp = t.sum + ((size_t) slot * t.naccs + a) * 2;

	switch (acc.kind)
	{
		case CBP_ACC_COUNT:		/* int8inc / int8inc_any (utils/adt/int8.c:805) */
			if (acc.arg < 0 || !((argnull >> acc.arg) & 1))
				atomicAdd((unsigned long long *) np, 1ull);
			break;
		case CBP_ACC_SUM_INT:	/* int4_sum / int8_avg_accum / numeric_avg_accum: N += 1, sumX += v */
			if (!((argnull >> acc.arg) & 1))
			{
				atomicAdd((unsigned long long *) np, 1ull);
				atomic_add128_signed(sp, args[acc.arg]);
			}
			break;
		case CBP_ACC_SUM_FLOAT:	/* float8pl / float8_accum Sx (tree order here: tolerance, not bit-exact) */
			if (!((argnull >> acc.arg) & 1))
			{
				atomicAdd((unsigned long long *) np, 1ull);
				atomicAdd((double *) sp, __longlong_as_double(args[acc.arg]));
			}
			break;
		case CBP_ACC_MIN:
			if (!((argnull >> acc.arg) & 1))
			{
				atomicAdd((unsigned long long *) np, 1ull);
				atomicMin((long long *) sp, (long long) args[acc.arg]);
			}
			break;
		case CBP_ACC_MAX:
			if (!((argnull >> acc.arg) & 1))
			{
				atomicAdd((unsigned long long *) np, 1ull);
				atomicMax((long long *) sp, (long long) args[acc.arg]);
			}
			break;
		case CBP_ACC_MERGE_COUNT:	/* int8pl over partial counts */
			if (!((argnull >> acc.arg) & 1))
				atomicAdd((unsigned long long *) np, (unsigned long long) args[acc.arg]);
			break;
		case CBP_ACC_MERGE_INT:	/* int8_avg_combine / numeric_avg_combine (numeric.c:5726, 4946) */
			if (!((argnull >> acc.arg) & 1))
			{
				atomicAdd((unsigned long long *) np, (unsigned long long) args[acc.arg]);
				atomic_add128(sp, (unsigned long long) args[acc.arg + 1], (unsigned long long) args[acc.arg + 2]);
			}
			break;
		case CBP_ACC_MERGE_MIN:
		case CBP_ACC_MERGE_MAX:
			if (!((argnull >> acc.arg) & 1) && args[acc.arg] > 0)
			{
				atomicAdd((unsigned long long *) np, (unsigned long long) args[acc.arg]);
				if (acc.kind == CBP_ACC_MERGE_MIN)
					atomicMin((long long *) sp, (long long) args[acc.arg + 1]);
				else
					atomicMax((long long *) sp, (long long) args[acc.arg + 1]);
			}
			break;
		case CBP_ACC_MERGE_FLOAT:	/* float8_combine (float.c:2886): N and Sx add */
			if (!((argnull >> acc.arg) & 1))
			{
				atomicAdd((unsigned long long *) np, (unsigned long long) args[acc.arg]);
				atomicAdd((double *) sp, __longlong_as_double(args[acc.arg + 1]));
			}
			break;
	}
}

__device__ __forceinline__ int
fcmp_pg(double x, double y)
{
	/* float8_cmp_internal (include/utils/float.h): NaN equals NaN and sorts above everything */
	if (x != x)
		return (y != y) ? 0 : 1;
	if (y != y)
		return -1;
	return x < y ? -1 : (x > y ? 1 : 0);
}

/* One scalar op of a postfix program over the value stack st[0 .. sp) with NULL bits snull: CONST, DUP, POP, integer and float8
 * arithmetic, I2F, F8ORD, the compares and three-valued AND / OR / NOT.  The pipeline kernel and the join-filter probe both
 * run their programs through it; each reads columns (LOAD) and consumes results (FILTER) itself.  Integer overflow of a live
 * row (`alive`, operands not NULL) stores CBGPU_ERR_OVERFLOW in *status (i64_add_ovf and its siblings). */
__device__ __forceinline__ void
cbp_scalar_op(const CbpOp &op, int64_t *st, uint64_t &snull, int &sp, bool alive, int *status)
{
	const int	code = op.code;
	const int	a = op.a;

	switch (code)
	{
		case CBP_CONST:
			st[sp] = op.imm;
			snull &= ~(1ull << sp);
			sp++;
			break;
		case CBP_DUP:
			st[sp] = st[a];
			snull = ((snull >> a) & 1) ? (snull | (1ull << sp)) : (snull & ~(1ull << sp));
			sp++;
			break;
		case CBP_POP:
			sp--;
			break;
		case CBP_ADD: case CBP_SUB: case CBP_MUL:
			{
				int64_t		y = st[sp - 1],
							x = st[sp - 2];
				bool		n = ((snull >> (sp - 1)) | (snull >> (sp - 2))) & 1;
				bool		ovf;
				const int64_t r = code == CBP_ADD ? i64_add_ovf(x, y, &ovf) : code == CBP_SUB ? i64_sub_ovf(x, y, &ovf) : i64_mul_ovf(x, y, &ovf);

				if (alive && !n && ovf)
					atomicExch(status, CBGPU_ERR_OVERFLOW);
				sp--;
				st[sp - 1] = r;
				snull = n ? (snull | (1ull << (sp - 1))) : (snull & ~(1ull << (sp - 1)));
				break;
			}
		case CBP_FADD: case CBP_FSUB: case CBP_FMUL:
			{
				double		y = __longlong_as_double(st[sp - 1]),
							x = __longlong_as_double(st[sp - 2]);
				bool		n = ((snull >> (sp - 1)) | (snull >> (sp - 2))) & 1;
				double		r = code == CBP_FADD ? __dadd_rn(x, y) : code == CBP_FSUB ? __dsub_rn(x, y) : __dmul_rn(x, y);

				sp--;
				st[sp - 1] = __double_as_longlong(r);
				snull = n ? (snull | (1ull << (sp - 1))) : (snull & ~(1ull << (sp - 1)));
				break;
			}
		case CBP_F8ORD:
			{
				long long	b = st[sp - 1];

				if (__longlong_as_double(b) != __longlong_as_double(b))
					b = 0x7FF8000000000000ll;	/* every NaN is the same value, above +Infinity */
				st[sp - 1] = b >= 0 ? b : (b ^ 0x7FFFFFFFFFFFFFFFll);
				break;
			}
		case CBP_I2F:
			{
				double		scale = 1.0;

				for (int k = 0; k < a; k++)
					scale *= 10.0;
				st[sp - 1] = __double_as_longlong(__ddiv_rn((double) st[sp - 1], scale));
				break;
			}
		case CBP_EQ: case CBP_NE: case CBP_LT: case CBP_LE: case CBP_GT: case CBP_GE:
		case CBP_FEQ: case CBP_FNE: case CBP_FLT: case CBP_FLE: case CBP_FGT: case CBP_FGE:
			{
				int64_t		y = st[sp - 1],
							x = st[sp - 2];
				bool		n = ((snull >> (sp - 1)) | (snull >> (sp - 2))) & 1;
				int			c;
				bool		r;

				if (code >= CBP_FEQ)
					c = fcmp_pg(__longlong_as_double(x), __longlong_as_double(y));
				else
					c = x < y ? -1 : (x > y ? 1 : 0);
				switch (code)
				{
					case CBP_EQ: case CBP_FEQ: r = c == 0; break;
					case CBP_NE: case CBP_FNE: r = c != 0; break;
					case CBP_LT: case CBP_FLT: r = c < 0; break;
					case CBP_LE: case CBP_FLE: r = c <= 0; break;
					case CBP_GT: case CBP_FGT: r = c > 0; break;
					default: r = c >= 0; break;
				}
				sp--;
				st[sp - 1] = r;
				snull = n ? (snull | (1ull << (sp - 1))) : (snull & ~(1ull << (sp - 1)));
				break;
			}
		case CBP_AND: case CBP_OR:
			{
				/* three-valued logic of ExecEvalBoolAnd/OrStep (execExprInterp.c) */
				bool		yn = (snull >> (sp - 1)) & 1,
							xn = (snull >> (sp - 2)) & 1;
				bool		y = st[sp - 1] != 0,
							x = st[sp - 2] != 0;
				bool		r,
							n;

				if (code == CBP_AND)
				{
					bool		anyfalse = (!xn && !x) || (!yn && !y);

					r = !anyfalse;
					n = !anyfalse && (xn || yn);
				}
				else
				{
					bool		anytrue = (!xn && x) || (!yn && y);

					r = anytrue;
					n = !anytrue && (xn || yn);
				}
				sp--;
				st[sp - 1] = r;
				snull = n ? (snull | (1ull << (sp - 1))) : (snull & ~(1ull << (sp - 1)));
				break;
			}
		case CBP_NOT:
			st[sp - 1] = !st[sp - 1];
			break;
	}
}

__device__ __forceinline__ void
sink_store(void *col, int type, uint64_t pos, int64_t v)
{
	switch (type)
	{
		case CB_INT4: case CB_DATE: case CB_DICT32:
			((int32_t *) col)[pos] = (int32_t) v;
			break;
		case CB_INT8: case CB_NUMERIC: case CB_FLOAT8:
			((int64_t *) col)[pos] = v;
			break;
		default:
			((uint8_t *) col)[pos] = (uint8_t) v;
	}
}

/* One lane reserves n rows for destination d and gets the position of the first.  out_count[d] counts every row routed to d,
 * stored or not: a staged Motion's retry sizes its exact buffers from these counts.  A direct Motion takes its slice of the
 * destination's window from that segment's own counter; the local count stays as a statistic.  Rows from seg_cap[d] on are
 * not stored (sink_put_row): a full Motion destination is not an error, the host redoes the pass with exact sizes. */
__device__ __forceinline__ unsigned long long
sink_reserve(const SinkOut &o, int d, unsigned n, int *status)
{
	unsigned long long pos = atomicAdd(o.out_count + d, (unsigned long long) n);

	if (o.part_cols)
		pos = atomicAdd_system(o.part_counts[d], (unsigned long long) n);
	if ((int64_t) (pos + n) > o.seg_cap[d])
	{
		if (o.part_flags)
			atomicOr(o.part_flags, CBGPU_DX_OVERFLOW);
		else
			atomicExch(status, CBGPU_ERR_NOMEM);
	}
	return pos;
}

/* Store the row reserved at `pos` for destination d: column c's value is val(c), and bit c of nullbits its NULL flag, which
 * goes to the column's NULL bytes; a NULL for a column that has none is refused. */
template <class Val>
__device__ __forceinline__ void
sink_put_row(const SinkOut &o, int d, unsigned long long pos, Val val, uint64_t nullbits, int *status)
{
	const bool	direct = o.part_cols != NULL;
	const uint64_t dst = direct ? pos : (uint64_t) o.seg_base[d] + pos;

	if ((int64_t) pos >= o.seg_cap[d])
		return;
	for (int c = 0; c < o.nout; c++)
	{
		uint8_t    *nulls = !direct ? o.outnull[c] : ((o.part_nullmask >> c) & 1) ? o.part_nulls[d * o.nout + c] : NULL;

		sink_store(direct ? o.part_cols[d * o.nout + c] : o.outcol[c], o.outtype[c], dst, val(c));
		if (nulls)
			nulls[dst] = (nullbits >> c) & 1;
		else if ((nullbits >> c) & 1)
			atomicExch(status, CBGPU_ERR_INVALID);
	}
}

struct XProg;					/* xmatch.h: the program's expression trees */

void		cb_agg_touch(cbgpu_aggtable *t);
int			cb_klog_begin(cbgpu_ctx *ctx, const char *name);
void		cb_klog_end(cbgpu_ctx *ctx, int i);
int			cb_pipeline_to_dev(cbgpu_ctx *ctx, const CbPipeline *p, PipeDev *d, XProg *x);
int			cb_try_probe_chain(cbgpu_ctx *ctx, const CbPipeline *p, const PipeDev *d, const XProg *x, bool *handled);
int			cb_try_specialised(cbgpu_ctx *ctx, const CbPipeline *p, const PipeDev *d, const XProg *x, bool *handled);
