/*
 * having_eval.cuh - the value arithmetic of HAVING (Agg.plan.qual, ExecQual over the finalised aggregates, nodeAgg.c:2460 /
 * 3100) over a groups relation in cbgpu_agg_to_rel's layout, for one group.
 *
 * Host and device code: k_having_eval runs it once per group, and the CPU tests compile it for the host.
 *
 * An exact value is the rational num / (den * 10^scale) with a 128-bit num, so that `sum(x) > 100.00` or `avg(x) <= y` decide
 * as numeric arithmetic does: a compare cross-multiplies, and a cross-product that needs more than 128 bits is reported
 * instead of compared.  A float8 value compares as float8_cmp_internal (utils/float.h) orders it.
 *
 * The program is one cbgpu_having_select has checked (xm_check_having, xmatch.h): every operand of a compare is a leaf (LOAD,
 * CONST, STATE), so a compare's operands are the two ops before it, and the stack only ever holds booleans - at most
 * CBH_MAX_DEPTH of them, kept as bit masks.  No value stack of rationals exists to spill.
 */
#pragma once
#include <stdint.h>
#include "../../include/cbgpu.h"

#if defined(__CUDACC__)
#define HV_HD __host__ __device__ __forceinline__
#else
#define HV_HD static inline
#endif

/* the columns of a groups relation: values at their stored width (1, 4 or 8 bytes), NULL bytes or NULL */
#define HV_MAX_COLS 64
typedef struct HvCols
{
	const void *data[HV_MAX_COLS];
	const uint8_t *nulls[HV_MAX_COLS];
	int32_t		width[HV_MAX_COLS];
} HvCols;

typedef struct HvVal
{
	__int128	num;			/* exact: the numerator; float8: the bits                             */
	int64_t		den;			/* exact: > 0                                                         */
	int32_t		scale;
	int32_t		isnull;
} HvVal;

HV_HD int64_t
hv_col(const HvCols *c, int col, int64_t g)
{
	switch (c->width[col])
	{
		case 1: return ((const uint8_t *) c->data[col])[g];
		case 4: return ((const int32_t *) c->data[col])[g];
		default: return ((const int64_t *) c->data[col])[g];
	}
}

/* *v *= m (m > 0) when the product fits in a signed 128-bit integer; 0 when it does not */
HV_HD int
hv_mul_u64(__int128 *v, uint64_t m)
{
	const int	neg = *v < 0;
	unsigned __int128 mag = neg ? (unsigned __int128) 0 - (unsigned __int128) *v : (unsigned __int128) *v;
	const unsigned __int128 lo = (unsigned __int128) (uint64_t) mag * m;
	const unsigned __int128 hi = (unsigned __int128) (uint64_t) (mag >> 64) * m;
	const unsigned __int128 limit = ((unsigned __int128) 1 << 127) - (neg ? 0 : 1);
	unsigned __int128 r;

	if (hi >> 64)
		return 0;
	r = lo + (hi << 64);
	if (r < lo || r > limit)
		return 0;
	*v = neg ? (__int128) ((unsigned __int128) 0 - r) : (__int128) r;
	return 1;
}

/* *v *= 10^k, or 0 when that leaves 128 bits */
HV_HD int
hv_scale_up(__int128 *v, int k)
{
	while (k > 0)
	{
		const int	step = k < 18 ? k : 18;
		uint64_t	p = 1;

		for (int i = 0; i < step; i++)
			p *= 10;
		if (*v != 0 && !hv_mul_u64(v, p))
			return 0;
		k -= step;
	}
	return 1;
}

/* float8 bits from a CBP_F8ORD image: the map is its own inverse on non-NaN values, and the one NaN image is a NaN */
HV_HD int64_t
hv_f8ord_inverse(int64_t b)
{
	return b >= 0 ? b : (int64_t) ((uint64_t) b ^ 0x7FFFFFFFFFFFFFFFull);
}

HV_HD double
hv_f8(int64_t bits)
{
	union
	{
		int64_t		i;
		double		d;
	}			u;

	u.i = bits;
	return u.d;
}

HV_HD int64_t
hv_f8_bits(double d)
{
	union
	{
		int64_t		i;
		double		d;
	}			u;

	u.d = d;
	return u.i;
}

/* one leaf op's value for group g: a grouping column (LOAD), a constant (CONST) or an aggregate (STATE) */
HV_HD HvVal
hv_leaf(const CbpOp *op, const HvCols *c, int64_t g)
{
	HvVal		r;

	r.num = 0;
	r.den = 1;
	r.scale = 0;
	r.isnull = 0;
	if (op->code == CBP_LOAD)
	{
		r.isnull = c->nulls[op->a] ? c->nulls[op->a][g] != 0 : 0;
		r.num = hv_col(c, op->a, g);
		r.scale = (int32_t) op->imm;
	}
	else if (op->code == CBP_CONST)
	{
		r.isnull = (op->a & CBH_CONST_NULL) != 0;
		r.num = op->imm;
		r.scale = op->a & 0xFFFF;
	}
	else
	{
		const int64_t n = hv_col(c, op->a, g);
		const int64_t lo = hv_col(c, op->a + 1, g);
		const int	kind = (int) (op->imm & 0xFF);

		r.scale = (int32_t) (op->imm >> 8);
		r.isnull = kind != CBH_COUNT && n == 0;
		switch (kind)
		{
			case CBH_COUNT:
				r.num = n;
				break;
			case CBH_SUM:
			case CBH_AVG:
				r.num = (__int128) (((unsigned __int128) (uint64_t) hv_col(c, op->a + 2, g) << 64) | (uint64_t) lo);
				if (kind == CBH_AVG && n > 0)
					r.den = n;
				break;
			case CBH_MIN:
			case CBH_MAX:
			case CBH_FSUM:
				r.num = lo;
				break;
			case CBH_FAVG:
				r.num = n > 0 ? hv_f8_bits(hv_f8(lo) / (double) n) : 0;
				break;
			default:			/* CBH_FMIN / CBH_FMAX */
				r.num = hv_f8ord_inverse(lo);
				break;
		}
	}
	return r;
}

/* a ? b as -1 / 0 / 1, or HV_OVERFLOW when a cross-product needs more than 128 bits */
#define HV_OVERFLOW 2
HV_HD int
hv_cmp_exact(const HvVal *a, const HvVal *b)
{
	__int128	L = a->num,
				R = b->num;

	if (!hv_mul_u64(&L, (uint64_t) b->den) || !hv_mul_u64(&R, (uint64_t) a->den) ||
		!hv_scale_up(&L, b->scale > a->scale ? b->scale - a->scale : 0) ||
		!hv_scale_up(&R, a->scale > b->scale ? a->scale - b->scale : 0))
		return HV_OVERFLOW;
	return L < R ? -1 : L > R ? 1 : 0;
}

/* float8_cmp_internal: NaN equals NaN and sorts above everything, -0 equals +0 */
HV_HD int
hv_cmp_f8(int64_t xb, int64_t yb)
{
	const double x = hv_f8(xb),
				y = hv_f8(yb);

	if (x != x)
		return y != y ? 0 : 1;
	if (y != y)
		return -1;
	return x < y ? -1 : x > y ? 1 : 0;
}

/* Runs the checked program ops[0 .. nops) for group g: bit q (q < 32) of the result is whether boolean q it leaves is true (not
 * NULL, not false); HV_OVERFLOWED is set when a compare of two non-NULL exact values needs more than 128 bits. */
#define HV_OVERFLOWED (1ull << 32)
HV_HD uint64_t
hv_program(const CbpOp *ops, int nops, const HvCols *c, int64_t g)
{
	uint32_t	val = 0,
				nul = 0;
	uint64_t	ovf = 0;
	int			sp = 0;

	for (int i = 0; i < nops; i++)
	{
		const int	code = ops[i].code;

		if (code >= CBP_EQ && code <= CBP_FGE)
		{
			const HvVal x = hv_leaf(&ops[i - 2], c, g),
						y = hv_leaf(&ops[i - 1], c, g);
			int			cmp = 0,
						r;
			const int	isnull = x.isnull || y.isnull;

			if (!isnull)
				cmp = code >= CBP_FEQ ? hv_cmp_f8((int64_t) x.num, (int64_t) y.num) : hv_cmp_exact(&x, &y);
			if (cmp == HV_OVERFLOW)
			{
				ovf = HV_OVERFLOWED;
				cmp = 0;
			}
			switch (code >= CBP_FEQ ? code - (CBP_FEQ - CBP_EQ) : code)
			{
				case CBP_EQ: r = cmp == 0; break;
				case CBP_NE: r = cmp != 0; break;
				case CBP_LT: r = cmp < 0; break;
				case CBP_LE: r = cmp <= 0; break;
				case CBP_GT: r = cmp > 0; break;
				default: r = cmp >= 0; break;
			}
			val = (val & ~(1u << sp)) | ((uint32_t) (r && !isnull) << sp);
			nul = (nul & ~(1u << sp)) | ((uint32_t) isnull << sp);
			sp++;
		}
		else if (code == CBP_AND || code == CBP_OR)
		{
			/* three-valued logic of ExecEvalBoolAndStep / OrStep (execExprInterp.c) */
			const int	xv = (val >> (sp - 2)) & 1,
						xn = (nul >> (sp - 2)) & 1,
						yv = (val >> (sp - 1)) & 1,
						yn = (nul >> (sp - 1)) & 1;
			int			r,
						n;

			if (code == CBP_AND)
			{
				const int	anyfalse = (!xn && !xv) || (!yn && !yv);

				r = !anyfalse;
				n = !anyfalse && (xn || yn);
			}
			else
			{
				const int	anytrue = (!xn && xv) || (!yn && yv);

				r = anytrue;
				n = !anytrue && (xn || yn);
			}
			sp--;
			val = (val & ~(1u << (sp - 1))) | ((uint32_t) (r && !n) << (sp - 1));
			nul = (nul & ~(1u << (sp - 1))) | ((uint32_t) n << (sp - 1));
		}
		else if (code == CBP_NOT)
		{
			const uint32_t bit = 1u << (sp - 1);

			if (!(nul & bit))
				val ^= bit;
		}
	}
	return (val & ~nul & (sp >= 32 ? 0xFFFFFFFFu : (1u << sp) - 1)) | ovf;
}
