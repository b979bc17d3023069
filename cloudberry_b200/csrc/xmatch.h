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
		case CBP_LOAD: case CBP_CONST: case CBP_DUP: case XOP_MULCSUB:
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
#define XM_PIPELINE_OPS (XM_OP(CBP_INSET + 1) - 1)	/* every CbpOpCode (INSET is the last) */
/* join filters: no FILTER / PROBE / END, and no INSET (they take no code sets) */
#define XM_SCALAR_OPS (XM_PIPELINE_OPS & ~(XM_OP(CBP_FILTER) | XM_OP(CBP_PROBE) | XM_OP(CBP_END) | XM_OP(CBP_INSET)))

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
