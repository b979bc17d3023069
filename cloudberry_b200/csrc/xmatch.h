/*
 * xmatch.h - the host's one reading of a postfix program (a pipeline's or a join filter's): what each op does to the value
 * stack, the walk that checks a program and rebuilds its expression trees, and the helpers the pattern matchers use to
 * route a descriptor to a hand-fused kernel (the role the reference's ExecReadyInterpretedExpr / EEOP fast-path selection
 * plays for common expression shapes, backend/executor/execExprInterp.c:260-330).
 */
#pragma once
#include "pipeline.cuh"

struct XNode
{
	int			code;			/* CbpOpCode */
	int			a;
	int64_t		imm;
	int			l, r;
};

struct XSection
{
	int			kind;			/* 0 = FILTER (root node in `node`), 1 = PROBE (`probe`, keys in `keys`) */
	int			node;
	int			probe;
	int			keys[CBP_MAX_KEYS];
};

struct XProg
{
	XNode		nodes[CBP_MAX_OPS];	/* an op makes at most one node */
	int			n;
	XSection	sections[CBP_MAX_OPS];
	int			nsections;
	int			stack[CBP_STACK];	/* node ids left on the stack at END: keys then args / outputs    */
	int			depth;
	bool		f8ord;			/* the program holds an F8ORD: float arithmetic stays with the generic kernel */
	bool		inset;			/* the program holds an INSET: only the generic kernel reads code sets */
};

/* the values an op pops and pushes, internal fused ops (pipeline.cuh) included; PROBE pops its probe's keys */
struct XEffect
{
	int			pops,
				pushes;
};

static inline XEffect
xm_effect(const CbpOp &op, const CbpProbe *probes)
{
	switch (op.code)
	{
		case CBP_LOAD: case CBP_CONST: case CBP_DUP: case CBP_STATE: case XOP_MULCSUB:
			return {0, 1};
		case CBP_NOT: case CBP_I2F: case CBP_F8ORD: case CBP_INSET:
			return {1, 1};
		case CBP_FILTER: case CBP_POP:
			return {1, 0};
		case CBP_PROBE:
			return {probes[op.a].nkeys, 0};
		case CBP_END: case XOP_FILTER_COL: case XOP_PROBE_COLS:
			return {0, 0};
		default:				/* binary operators */
			return {2, 1};
	}
}

/* opcodes as bits of XAllow.ops */
#define XM_OP(c) (1u << (c))
#define XM_PIPELINE_OPS (XM_OP(CBP_INSET + 1) - 1)	/* every CbpOpCode up to INSET (STATE is HAVING's alone) */
/* join filters: no FILTER / PROBE / END, and no INSET (they take no code sets) */
#define XM_SCALAR_OPS (XM_PIPELINE_OPS & ~(XM_OP(CBP_FILTER) | XM_OP(CBP_PROBE) | XM_OP(CBP_END) | XM_OP(CBP_INSET)))
/* HAVING (cbgpu_having_select): leaves, compares and the boolean operators */
#define XM_HAVING_OPS (XM_OP(CBP_LOAD) | XM_OP(CBP_CONST) | XM_OP(CBP_STATE) | ((XM_OP(CBP_FGE + 1) - 1) & ~(XM_OP(CBP_EQ) - 1)) | \
					   XM_OP(CBP_AND) | XM_OP(CBP_OR) | XM_OP(CBP_NOT))

/* what a caller lets a program hold, and how it reports a refusal */
struct XAllow
{
	const char *what;			/* "pipeline" / "join filter": the subject of the messages           */
	uint32_t	ops;			/* XM_OP(code) set: the opcodes allowed (END only as the last op)     */
	const CbpProbe *probes;		/* PROBE a takes probes[a], a < nprobes                               */
	int			nprobes;
	int			too_deep;		/* the code of a stack deeper than CBP_STACK                          */
	int			nsets;			/* INSET a takes code set a, a < nsets                                */
};

/* Checks a program of 1 .. CBP_MAX_OPS ops over `ncols` columns op by op and builds its expression trees in *x: FILTER and
 * PROBE close a section, what is left on the stack at the end is x->stack[0 .. x->depth).  CBGPU_ERR_INVALID for a bad LOAD
 * column or DUP index, a bad PROBE, a stack underflow, an END before the last op and an opcode the caller does not allow;
 * allow.too_deep for a stack deeper than CBP_STACK.  The caller checks the final state. */
static inline int
xm_walk(cbgpu_ctx *ctx, const XAllow &allow, int ncols, const CbpOp *ops, int nops, XProg *x)
{
	x->n = 0;
	x->nsections = 0;
	x->depth = 0;
	x->f8ord = false;
	x->inset = false;
	for (int i = 0; i < nops; i++)
	{
		const CbpOp *op = &ops[i];

		if (op->code < 0 || op->code >= 32 || !(allow.ops & XM_OP(op->code)))
			return cb_fail(ctx, CBGPU_ERR_INVALID, "%s op %lld: opcode not supported", allow.what, i);
		if (op->code == CBP_LOAD && (op->a < 0 || op->a >= ncols))
			return cb_fail(ctx, CBGPU_ERR_INVALID, "%s op %lld: LOAD of a missing column", allow.what, i);
		if (op->code == CBP_DUP && (op->a < 0 || op->a >= x->depth))
			return cb_fail(ctx, CBGPU_ERR_INVALID, "%s op %lld: DUP out of range", allow.what, i);
		if (op->code == CBP_PROBE && (op->a < 0 || op->a >= allow.nprobes || allow.probes[op->a].nkeys < 0 ||
									  allow.probes[op->a].nkeys > CBP_MAX_KEYS))
			return cb_fail(ctx, CBGPU_ERR_INVALID, "%s op %lld: bad PROBE", allow.what, i);
		if (op->code == CBP_INSET && (op->a < 0 || op->a >= allow.nsets))
			return cb_fail(ctx, CBGPU_ERR_INVALID, "%s op %lld: INSET of a code set the descriptor does not declare", allow.what, i);
		if (op->code == CBP_END && i != nops - 1)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "%s op %lld: END before the last op", allow.what, i);
		const XEffect e = xm_effect(*op, allow.probes);
		const int	base = x->depth - e.pops;	/* where the op's values start on the stack */

		if (base < 0)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "%s op %lld: stack underflow", allow.what, i);
		if (base + e.pushes > CBP_STACK)
			return cb_fail(ctx, allow.too_deep, "%s op %lld: stack deeper than CBP_STACK", allow.what, i);
		switch (op->code)
		{
			case CBP_DUP:
				x->stack[base] = x->stack[op->a];
				break;
			case CBP_FILTER:
				x->sections[x->nsections++] = {0, x->stack[base], -1, {}};
				break;
			case CBP_PROBE:
				{
					XSection   *s = &x->sections[x->nsections++];

					*s = {1, -1, op->a, {}};
					for (int k = 0; k < e.pops; k++)
						s->keys[k] = x->stack[base + k];
					break;
				}
			case CBP_POP:
			case CBP_END:
				break;
			default:			/* LOAD, CONST and the operators: one node over the values they pop */
				x->nodes[x->n] = {op->code, op->a, op->imm, e.pops > 0 ? x->stack[base] : -1, e.pops > 1 ? x->stack[base + 1] : -1};
				x->stack[base] = x->n++;
				x->f8ord |= op->code == CBP_F8ORD;
				x->inset |= op->code == CBP_INSET;
				break;
		}
		x->depth = base + e.pushes;
	}
	return CBGPU_OK;
}

static inline bool
xm_is_load(const XProg *x, int node, int *col)
{
	if (node < 0 || x->nodes[node].code != CBP_LOAD)
		return false;
	*col = x->nodes[node].a;
	return true;
}

static inline bool
xm_is_const(const XProg *x, int node, int64_t *v)
{
	if (node < 0 || x->nodes[node].code != CBP_CONST)
		return false;
	*v = x->nodes[node].imm;
	return true;
}

/* MUL(LOAD b, SUB(CONST k, LOAD c))  -  e.g. l_extendedprice * (1 - l_discount) */
static inline bool
xm_is_rev(const XProg *x, int node, int *b, int64_t *k, int *c)
{
	if (node < 0 || x->nodes[node].code != CBP_MUL)
		return false;
	int			s = x->nodes[node].r;

	if (!xm_is_load(x, x->nodes[node].l, b) || s < 0 || x->nodes[s].code != CBP_SUB)
		return false;
	return xm_is_const(x, x->nodes[s].l, k) && xm_is_load(x, x->nodes[s].r, c);
}

/* MUL(rev, ADD(CONST k2, LOAD d))  -  e.g. ... * (1 + l_tax) */
static inline bool
xm_is_chg(const XProg *x, int node, int *b, int64_t *k, int *c, int64_t *k2, int *d)
{
	if (node < 0 || x->nodes[node].code != CBP_MUL)
		return false;
	int			s = x->nodes[node].r;

	if (!xm_is_rev(x, x->nodes[node].l, b, k, c) || s < 0 || x->nodes[s].code != CBP_ADD)
		return false;
	return xm_is_const(x, x->nodes[s].l, k2) && xm_is_load(x, x->nodes[s].r, d);
}

/* CMP(LOAD col, CONST v) */
static inline bool
xm_is_cmp_const(const XProg *x, int node, int *code, int *col, int64_t *v)
{
	if (node < 0)
		return false;
	int			c = x->nodes[node].code;

	if (c < CBP_EQ || c > CBP_GE)
		return false;
	*code = c;
	return xm_is_load(x, x->nodes[node].l, col) && xm_is_const(x, x->nodes[node].r, v);
}

/* The rows `col CMP v` keeps, as a closed range [*lo, *hi] inside int32, over a column whose values lie in [dlo, dhi]
 * (inside int32): EQ keeps [v, v], the other compares bound one end of the domain.  False for NE (not a range) and for an
 * empty range. */
static inline bool
xm_qual_range(int code, int64_t v, int64_t dlo, int64_t dhi, int64_t *lo, int64_t *hi)
{
	int64_t		l = dlo,
				h = dhi;

	switch (code)
	{
		case CBP_EQ: l = h = v; break;
		case CBP_LT: if (v == INT64_MIN) return false; h = v - 1; break;
		case CBP_LE: h = v; break;
		case CBP_GT: if (v == INT64_MAX) return false; l = v + 1; break;
		case CBP_GE: l = v; break;
		default: return false;
	}
	if (l > h || l > INT32_MAX || h < INT32_MIN)
		return false;
	*lo = l < INT32_MIN ? INT32_MIN : l;
	*hi = h > INT32_MAX ? INT32_MAX : h;
	return true;
}

/* A HAVING program (cbgpu_having_select) over a groups relation whose columns have types[0 .. ncols): xm_walk with the HAVING
 * opcodes, then operand kinds.  LOAD, CONST and STATE are exact or float8 values, a compare takes two exact operands (EQ..GE)
 * or two float8 ones (FEQ..FGE) and makes a boolean, AND / OR / NOT take booleans, and the program leaves nquals (>= 1)
 * booleans.  So every compare's operands are the two leaf ops before it (having_eval.cuh relies on that).  CBGPU_ERR_INVALID
 * for a malformed program; CBGPU_ERR_UNSUPPORTED for more than CBH_MAX_DEPTH booleans on the stack at once. */
static inline int
xm_check_having(cbgpu_ctx *ctx, const int32_t *types, int ncols, const CbpOp *ops, int nops, int nquals, XProg *x)
{
	enum { K_EXACT = 1, K_F8, K_BOOL };
	const XAllow allow = {"HAVING", XM_HAVING_OPS, NULL, 0, CBGPU_ERR_UNSUPPORTED, 0};
	int			kind[CBP_MAX_OPS];
	int			nbool = 0;

	if (nops < 1 || nops > CBP_MAX_OPS || nquals < 1)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "HAVING program of %s%lld ops", "", nops);
	int			rc = xm_walk(ctx, allow, ncols, ops, nops, x);

	if (rc)
		return rc;
	for (int i = 0; i < x->n; i++)
	{
		const XNode *nd = &x->nodes[i];
		const int64_t scale = nd->code == CBP_STATE ? nd->imm >> 8 : nd->code == CBP_LOAD ? nd->imm : nd->a & 0xFFFF;

		switch (nd->code)
		{
			case CBP_LOAD:
				if (types[nd->a] == CB_FLOAT8)
					kind[i] = K_F8;
				else if (types[nd->a] == CB_INT4 || types[nd->a] == CB_INT8 || types[nd->a] == CB_DATE ||
						 types[nd->a] == CB_NUMERIC || types[nd->a] == CB_BPCHAR1)
					kind[i] = K_EXACT;
				else
					return cb_fail(ctx, CBGPU_ERR_INVALID, "HAVING op %s%lld: LOAD of a column that is not a number", "", i);
				break;
			case CBP_CONST:
				if (nd->a & ~(0xFFFF | CBH_CONST_F8 | CBH_CONST_NULL))
					return cb_fail(ctx, CBGPU_ERR_INVALID, "HAVING op %s%lld: bad CONST flags", "", i);
				kind[i] = (nd->a & CBH_CONST_F8) ? K_F8 : K_EXACT;
				break;
			case CBP_STATE:
				{
					const int	k = (int) (nd->imm & 0xFF);

					if (nd->a < 0 || nd->a + 2 >= ncols || types[nd->a] != CB_INT8 || types[nd->a + 1] != CB_INT8 ||
						types[nd->a + 2] != CB_INT8)
						return cb_fail(ctx, CBGPU_ERR_INVALID, "HAVING op %s%lld: STATE of columns that are not (N, lo, hi)", "", i);
					if (k < CBH_COUNT || k > CBH_FMAX || nd->imm < 0)
						return cb_fail(ctx, CBGPU_ERR_INVALID, "HAVING op %s%lld: unknown aggregate kind", "", i);
					kind[i] = k >= CBH_FSUM ? K_F8 : K_EXACT;
					break;
				}
			case CBP_AND: case CBP_OR: case CBP_NOT:
				if (kind[nd->l] != K_BOOL || (nd->code != CBP_NOT && kind[nd->r] != K_BOOL))
					return cb_fail(ctx, CBGPU_ERR_INVALID, "HAVING op %s%lld: AND / OR / NOT of a value that is not a boolean", "", i);
				kind[i] = K_BOOL;
				break;
			default:			/* the compares */
				{
					const int	want = nd->code >= CBP_FEQ ? K_F8 : K_EXACT;

					if (kind[nd->l] != want || kind[nd->r] != want)
						return cb_fail(ctx, CBGPU_ERR_INVALID, "HAVING op %s%lld: a compare takes two exact or two float8 operands", "", i);
					kind[i] = K_BOOL;
					break;
				}
		}
		if (kind[i] != K_BOOL && (scale < 0 || scale > CBH_MAX_SCALE))
			return cb_fail(ctx, CBGPU_ERR_INVALID, "HAVING op %s%lld: scale out of range", "", i);
	}
	if (x->depth != nquals)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "HAVING program leaves %s%lld values, not one per qual", "", x->depth);
	for (int q = 0; q < x->depth; q++)
		if (kind[x->stack[q]] != K_BOOL)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "HAVING program leaves a value that is not a boolean%s (qual %lld)", "", q);
	for (int i = 0; i < nops; i++)
	{
		nbool += ops[i].code >= CBP_EQ && ops[i].code <= CBP_FGE ? 1 : ops[i].code == CBP_AND || ops[i].code == CBP_OR ? -1 : 0;
		if (nbool > CBH_MAX_DEPTH)
			return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "HAVING program holds more than %s%lld booleans at once", "", CBH_MAX_DEPTH);
	}
	return CBGPU_OK;
}
