/*
 * inset_program.c - pipeline descriptors holding CBP_INSET, handed to cbgpu_pipeline_run over the no-op runtime of
 * tests/fake_runtime.py, for tests/test_host_string_predicates_fake_runtime.py.  Shapes the fused kernels take (TPC-H Q1 for the
 * small scan-aggregate kernel, Q3 for the probe chain) with an INSET computed and dropped on the way must run on the generic
 * kernel, which is the only one that reads code sets; an INSET naming a set the descriptor does not declare, and a malformed
 * set, are refused before any launch; a join filter takes no INSET.  Prints one line per case:
 *   <name> <return code> <kernels launched> <kernel name, or the error message>
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "cbgpu.h"

#define NROWS 1000

enum { SHIPDATE, RF, LS, QTY, PRICE, DISC, CODE, ORDERKEY, NCOLS };

static const int32_t col_type[NCOLS] = {CB_DATE, CB_BPCHAR1, CB_BPCHAR1, CB_NUMERIC, CB_NUMERIC, CB_NUMERIC, CB_DICT32, CB_INT8};

static cbgpu_ctx *ctx;
static cbgpu_rel *li,
		   *orders;
static cbgpu_hashtable *ht;
static cbgpu_aggtable *agg_q1,
		   *agg_q3;
static void *bits;
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

static void
begin(int nprobes, int nsets)
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
	P.nsets = nsets;
	for (int i = 0; i < nsets; i++)
	{
		P.sets[i].bits = bits;
		P.sets[i].nbits = 64;
	}
}

/* LOAD CODE; INSET set; POP: a code-set test computed and dropped */
static void
inset(int set)
{
	op(CBP_LOAD, CODE, 0);
	op(CBP_INSET, set, 0);
	op(CBP_POP, 0, 0);
}

static void
revenue(void)
{
	op(CBP_LOAD, PRICE, 0);
	op(CBP_CONST, 0, 100);
	op(CBP_LOAD, DISC, 0);
	op(CBP_SUB, 0, 0);
	op(CBP_MUL, 0, 0);
}

/* Q1's shape: a date qual, two char(1) keys, sums, count(*) */
static void
q1(int with_inset)
{
	begin(0, 1);
	op(CBP_LOAD, SHIPDATE, 0);
	op(CBP_CONST, 0, 10000);
	op(CBP_LE, 0, 0);
	op(CBP_FILTER, 0, 0);
	op(CBP_LOAD, RF, 0);
	op(CBP_LOAD, LS, 0);
	if (with_inset)
		inset(0);
	op(CBP_LOAD, QTY, 0);
	op(CBP_LOAD, PRICE, 0);
	revenue();
	revenue();
	op(CBP_CONST, 0, 100);
	op(CBP_LOAD, DISC, 0);
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

/* Q3's lineitem pipeline: a date qual, a probe of orders, sum of revenue by order key */
static void
q3(int with_inset)
{
	begin(1, 1);
	op(CBP_LOAD, SHIPDATE, 0);
	op(CBP_CONST, 0, 10000);
	op(CBP_GT, 0, 0);
	op(CBP_FILTER, 0, 0);
	op(CBP_LOAD, ORDERKEY, 0);
	op(CBP_PROBE, 0, 0);
	op(CBP_LOAD, ORDERKEY, 0);
	if (with_inset)
		inset(0);
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

int
main(void)
{
	const int32_t key = 0,
				q1_kinds[5] = {CBP_ACC_SUM_INT, CBP_ACC_SUM_INT, CBP_ACC_SUM_INT, CBP_ACC_SUM_INT, CBP_ACC_COUNT},
				q3_kind = CBP_ACC_SUM_INT;

	check(cbgpu_ctx_create(0, &ctx), "cbgpu_ctx_create");
	check(cbgpu_rel_create(ctx, NROWS, NCOLS, col_type, NULL, &li), "lineitem");
	check(cbgpu_rel_create(ctx, 100, 1, &col_type[ORDERKEY], NULL, &orders), "orders");
	check(cbgpu_ht_build(ctx, orders, &key, 1, 1, &ht), "cbgpu_ht_build");
	check(cbgpu_agg_create(ctx, 2, 5, q1_kinds, 64, &agg_q1), "Q1 aggregate");
	check(cbgpu_agg_create(ctx, 1, 1, &q3_kind, 1024, &agg_q3), "Q3 aggregate");
	check(cbgpu_dev_alloc(ctx, 8, &bits), "code set");

	/* routes: without INSET the fused kernels take these shapes, with it the generic kernel does */
	q1(0);
	run("q1");
	q1(1);
	run("q1_inset");
	q3(0);
	run("q3");
	q3(1);
	run("q3_inset");
	P.force_generic = 1;
	run("q3_inset_forced");

	/* refusals */
	q1(1);
	P.nsets = 0;
	run("inset_no_sets");		/* the INSET is op 7 */
	q1(1);
	P.ops[7].a = 1;
	run("inset_undeclared_set");
	q1(1);
	P.ops[7].a = -1;
	run("inset_negative_set");
	q1(1);
	P.nsets = CBP_MAX_SETS + 1;
	run("too_many_sets");
	q1(1);
	P.sets[0].bits = NULL;
	run("set_without_bits");
	q1(1);
	P.sets[0].nbits = -1;
	run("set_negative_size");
	{
		/* a join filter: LOAD 0; INSET 0 - no code sets there */
		CbpColumn	fc = {cbgpu_rel_col_devptr(orders, 0), NULL, NULL, CB_INT8, 0};
		CbpOp		fops[2] = {{CBP_LOAD, 0, 0}, {CBP_INSET, 0, 0}};
		cbgpu_join_filter jf = {1, &fc, 2, fops};
		cbgpu_pairs pairs;
		const int64_t before = cbgpu_kernel_launches(ctx);
		const int	rc = cbgpu_ht_probe_pairs(ctx, ht, orders, &key, 1, CB_JOIN_SEMI, &jf, NULL, NULL, &pairs, NULL);

		printf("join_filter_inset %d %lld %s\n", rc, (long long) (cbgpu_kernel_launches(ctx) - before), cbgpu_last_error(ctx));
	}
	return 0;
}
