/*
 * pipeline_program.c - pipeline descriptors built in C and handed to cbgpu_pipeline_run, for
 * tests/test_host_pipeline_program_fake_runtime.py.  Each malformed postfix program must be refused with its code before any
 * launch; each valid one must reach the kernel its shape calls for.  Runs over the no-op runtime of tests/fake_runtime.py
 * (LD_PRELOADed: no kernel computes anything, only the host side is under test).  Prints one line per case:
 *   <name> <return code> <kernels launched> <kernel name, or the error message>
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "cbgpu.h"

#define NROWS 1000

/* the driving relation's columns, lineitem-like */
enum { SHIPDATE, RF, LS, QTY, PRICE, DISC, TAX, ORDERKEY, NCOLS };

static const int32_t col_type[NCOLS] = {CB_DATE, CB_BPCHAR1, CB_BPCHAR1, CB_NUMERIC, CB_NUMERIC, CB_NUMERIC, CB_NUMERIC, CB_INT8};

static cbgpu_ctx *ctx;
static cbgpu_rel *li,
		   *orders,
		   *out;
static cbgpu_hashtable *ht;
static cbgpu_aggtable *agg_q1,
		   *agg_q3;
static void *out_count;
static CbPipeline P;

static void
check(int rc, const char *what)
{
	if (rc != CBGPU_OK)
	{
		fprintf(stderr, "%s: %d %s\n", what, rc, cbgpu_last_error(ctx));
		exit(1);
	}
}

static void
op(int code, int a, int64_t imm)
{
	CbpOp		o = {code, a, imm};

	P.ops[P.nops++] = o;
}

/* a descriptor over the driving relation: every column loadable, `nprobes` (0 or 1) probes of the orders table */
static void
begin(int nprobes)
{
	memset(&P, 0, sizeof(P));
	P.nrows = NROWS;
	P.ncols = NCOLS;
	for (int c = 0; c < NCOLS; c++)
	{
		P.cols[c].data = cbgpu_rel_col_devptr(li, c);
		P.cols[c].type = col_type[c];
	}
	P.nprobes = nprobes;
	if (nprobes)
	{
		P.probes[0].ht = ht;
		P.probes[0].jointype = CB_JOIN_INNER;
		P.probes[0].nkeys = 1;
		P.probes[0].keytype[0] = CB_INT8;
	}
}

/* one row of the stack's single value per surviving row */
static void
sink_materialize(void)
{
	P.sink.kind = CBP_SINK_MATERIALIZE;
	P.sink.nout = 1;
	P.sink.out = out;
	P.sink.out_count = (int64_t *) out_count;
}

/* LOAD col; CONST v; cmp; FILTER */
static void
qual(int col, int cmp, int64_t v)
{
	op(CBP_LOAD, col, 0);
	op(CBP_CONST, 0, v);
	op(cmp, 0, 0);
	op(CBP_FILTER, 0, 0);
}

/* price * (100 - disc) */
static void
revenue(void)
{
	op(CBP_LOAD, PRICE, 0);
	op(CBP_CONST, 0, 100);
	op(CBP_LOAD, DISC, 0);
	op(CBP_SUB, 0, 0);
	op(CBP_MUL, 0, 0);
}

/* TPC-H Q1: one qual on a date, group by two char(1) columns, sums of two columns, of a revenue and of a charge, count(*);
 * `f8ord`: a float8 order key computed and dropped on the way */
static void
q1(int cmp, int64_t v, int f8ord)
{
	begin(0);
	qual(SHIPDATE, cmp, v);
	op(CBP_LOAD, RF, 0);
	op(CBP_LOAD, LS, 0);
	if (f8ord)
	{
		op(CBP_LOAD, PRICE, 0);
		op(CBP_F8ORD, 0, 0);
		op(CBP_POP, 0, 0);
	}
	op(CBP_LOAD, QTY, 0);
	op(CBP_LOAD, PRICE, 0);
	revenue();
	revenue();
	op(CBP_CONST, 0, 100);
	op(CBP_LOAD, TAX, 0);
	op(CBP_ADD, 0, 0);
	op(CBP_MUL, 0, 0);
	op(CBP_END, 0, 0);
	P.sink.kind = CBP_SINK_AGG;
	P.sink.agg = agg_q1;
	P.sink.nkeys = 2;
	P.sink.keytype[0] = P.sink.keytype[1] = CB_BPCHAR1;
	P.sink.naccs = 5;
	for (int a = 0; a < 4; a++)
	{
		P.sink.accs[a].kind = CBP_ACC_SUM_INT;
		P.sink.accs[a].arg = a;
	}
	P.sink.accs[4].kind = CBP_ACC_COUNT;
	P.sink.accs[4].arg = -1;
}

/* TPC-H Q3's lineitem pipeline: quals, a probe of the orders table, sum of revenue grouped by the order key.  nquals quals
 * (col, cmp, v) before the probe; `behind`: the last one after it instead */
static void
q3(int nquals, const int64_t (*quals)[3], int behind, int f8ord)
{
	begin(1);
	for (int i = 0; i < nquals - (behind ? 1 : 0); i++)
		qual((int) quals[i][0], (int) quals[i][1], quals[i][2]);
	op(CBP_LOAD, ORDERKEY, 0);
	op(CBP_PROBE, 0, 0);
	if (behind)
		qual((int) quals[nquals - 1][0], (int) quals[nquals - 1][1], quals[nquals - 1][2]);
	op(CBP_LOAD, ORDERKEY, 0);
	if (f8ord)
	{
		op(CBP_LOAD, PRICE, 0);
		op(CBP_F8ORD, 0, 0);
		op(CBP_POP, 0, 0);
	}
	revenue();
	op(CBP_END, 0, 0);
	P.sink.kind = CBP_SINK_AGG;
	P.sink.agg = agg_q3;
	P.sink.nkeys = 1;
	P.sink.keytype[0] = CB_INT8;
	P.sink.naccs = 1;
	P.sink.accs[0].kind = CBP_ACC_SUM_INT;
	P.sink.accs[0].arg = 0;
}

static void
run(const char *name)
{
	const int64_t before = cbgpu_kernel_launches(ctx);
	const int	rc = cbgpu_pipeline_run(ctx, &P);

	printf("%s %d %lld %s\n", name, rc, (long long) (cbgpu_kernel_launches(ctx) - before),
		   rc ? cbgpu_last_error(ctx) : cbgpu_last_kernel_name(ctx));
}

/* LOAD QTY, then `code` (a, 0), then END: one op that breaks an otherwise valid program */
static void
bad_after_load(const char *name, int code, int a)
{
	begin(1);
	op(CBP_LOAD, QTY, 0);
	op(code, a, 0);
	op(CBP_END, 0, 0);
	sink_materialize();
	run(name);
}

/* `code` (a, 0) on an empty stack, then LOAD QTY; END */
static void
bad_first(const char *name, int code, int a)
{
	begin(1);
	op(code, a, 0);
	op(CBP_LOAD, QTY, 0);
	op(CBP_END, 0, 0);
	sink_materialize();
	run(name);
}

/* n CONSTs, then n - 1 ANDs, then END: the stack is n values deep at its deepest and one value is left */
static void
deep(const char *name, int n)
{
	begin(0);
	for (int i = 0; i < n; i++)
		op(CBP_CONST, 0, 1);
	for (int i = 1; i < n; i++)
		op(CBP_AND, 0, 0);
	op(CBP_END, 0, 0);
	sink_materialize();
	run(name);
}

int
main(void)
{
	const int32_t key = 0,
				out_type = CB_INT8,
				q1_kinds[5] = {CBP_ACC_SUM_INT, CBP_ACC_SUM_INT, CBP_ACC_SUM_INT, CBP_ACC_SUM_INT, CBP_ACC_COUNT},
				q3_kind = CBP_ACC_SUM_INT;

	check(cbgpu_ctx_create(0, &ctx), "cbgpu_ctx_create");
	check(cbgpu_rel_create(ctx, NROWS, NCOLS, col_type, NULL, &li), "lineitem");
	check(cbgpu_rel_create(ctx, 100, 1, &col_type[ORDERKEY], NULL, &orders), "orders");
	check(cbgpu_ht_build(ctx, orders, &key, 1, 1, &ht), "cbgpu_ht_build");
	check(cbgpu_rel_create(ctx, NROWS, 1, &out_type, NULL, &out), "output relation");
	check(cbgpu_dev_alloc(ctx, sizeof(int64_t), &out_count), "output counter");
	check(cbgpu_agg_create(ctx, 2, 5, q1_kinds, 64, &agg_q1), "Q1 aggregate");
	check(cbgpu_agg_create(ctx, 1, 1, &q3_kind, 1024, &agg_q3), "Q3 aggregate");

	/* refusals */
	bad_after_load("load_missing_column", CBP_LOAD, NCOLS);
	bad_after_load("load_negative_column", CBP_LOAD, -1);
	bad_after_load("dup_out_of_range", CBP_DUP, 1);
	bad_after_load("dup_negative", CBP_DUP, -1);
	bad_after_load("underflow_binary", CBP_ADD, 0);
	bad_after_load("underflow_compare", CBP_FLT, 0);
	bad_first("underflow_unary", CBP_NOT, 0);
	bad_first("underflow_f8ord", CBP_F8ORD, 0);
	bad_first("underflow_filter", CBP_FILTER, 0);
	bad_first("underflow_pop", CBP_POP, 0);
	bad_after_load("probe_bad_index", CBP_PROBE, 1);
	bad_after_load("probe_negative_index", CBP_PROBE, -1);
	bad_first("probe_too_few_keys", CBP_PROBE, 0);
	bad_after_load("end_before_last", CBP_END, 0);
	bad_after_load("unknown_opcode", CBP_F8ORD + 1, 0);
	bad_after_load("internal_opcode", 100, 0);	/* the host's own fused ops are not part of the ABI */
	bad_after_load("negative_opcode", -1, 0);
	begin(0);
	op(CBP_LOAD, QTY, 0);
	sink_materialize();
	run("no_end");
	deep("depth_49", 49);
	deep("depth_48", 48);

	/* routes */
	{
		const int64_t date_gt[1][3] = {{SHIPDATE, CBP_GT, 9000}},
					date_ne[1][3] = {{SHIPDATE, CBP_NE, 9000}},
					date_empty[1][3] = {{SHIPDATE, CBP_LT, -2147483648ll}},
					date_between[2][3] = {{SHIPDATE, CBP_GE, 8000}, {SHIPDATE, CBP_LE, 9000}},
					date_between_empty[2][3] = {{SHIPDATE, CBP_GE, 9000}, {SHIPDATE, CBP_LE, 8000}},
					byte_lt[1][3] = {{RF, CBP_LT, 1000}},
					byte_empty[1][3] = {{RF, CBP_LT, 0}};

		q1(CBP_LE, 10471, 0);
		run("q1");
		q1(CBP_LE, 10471, 1);
		run("q1_f8ord");
		q1(CBP_NE, 10471, 0);
		run("q1_ne");
		q1(CBP_LT, -2147483648ll, 0);
		run("q1_empty");
		q1(CBP_GT, 2147483647ll, 0);
		run("q1_empty_top");
		q1(CBP_LE, 1ll << 40, 0);
		run("q1_wide_const");
		q3(1, date_gt, 0, 0);
		run("q3");
		q3(1, date_gt, 0, 1);
		run("q3_f8ord");
		q3(2, date_between, 1, 0);
		run("q3_qual_behind_probe");
		q3(1, date_ne, 0, 0);
		run("q3_ne");
		q3(1, date_empty, 0, 0);
		run("q3_empty");
		q3(2, date_between, 0, 0);
		run("q3_between");
		q3(2, date_between_empty, 0, 0);
		run("q3_between_empty");
		q3(1, byte_lt, 0, 0);
		run("q3_byte_qual");
		q3(1, byte_empty, 0, 0);
		run("q3_byte_empty");
	}

	cbgpu_agg_free(agg_q3);
	cbgpu_agg_free(agg_q1);
	cbgpu_dev_free(ctx, out_count);
	cbgpu_rel_free(out);
	cbgpu_ht_free(ht);
	cbgpu_rel_free(orders);
	cbgpu_rel_free(li);
	cbgpu_ctx_destroy(ctx);
	return 0;
}
