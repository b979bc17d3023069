/*
 * cb_plan.h - plan-tree and expression structs the GPU executor consumes.
 *
 * These mirror, field for field where the hot path reads them, the reference's planner output
 * so that a backend shim can translate a PlannedStmt sub-tree 1:1 (reference structs cited):
 *
 *   Plan        src/include/nodes/plannodes.h:263-337   (plan_node_id, targetlist, qual, lefttree, righttree)
 *   SeqScan     src/include/nodes/plannodes.h (Scan.scanrelid)
 *   Hash        src/include/nodes/plannodes.h:1551-1567 (hashkeys)
 *   HashJoin    src/include/nodes/plannodes.h:1193-1208 (Join.jointype, hashclauses/hashkeys, hashqualclauses)
 *   Agg         src/include/nodes/plannodes.h:1342-1363 (aggstrategy, aggsplit, numCols, grpColIdx, numGroups, streaming)
 *   Motion      src/include/nodes/plannodes.h:1651-1676 (motionType, hashExprs, numHashSegments)
 *   Var/Const/OpExpr/BoolExpr/Aggref/TargetEntry   src/include/nodes/primnodes.h
 *
 * PostgreSQL `List *` members become (count, array) pairs; Oids of operators / functions become
 * the small enums below (the shim resolves pg_operator / pg_proc Oids to them).
 *
 * Plain C, no CUDA or torch types: this header is shared by the product (cloudberry_b200/csrc),
 * by the CPU oracle (oracle/, test infrastructure only) and by the ctypes mirror used in tests.
 */
#ifndef CB_PLAN_H
#define CB_PLAN_H

#include <stdbool.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- column / datum types (device encodings: DESIGN.md "data layout in HBM") ---- */
typedef enum CbTypeId
{
	CB_INT4 = 1,		/* integer                         int32                                  */
	CB_INT8 = 2,		/* bigint                          int64                                  */
	CB_DATE = 3,		/* date (DateADT, utils/date.h:23) int32 days since 2000-01-01            */
	CB_NUMERIC = 4,		/* numeric(p,s)                    int64 scaled by 10^dscale              */
	CB_BPCHAR1 = 5,		/* character(1)                    uint8 (the byte)                       */
	CB_DICT8 = 6,		/* bpchar/varchar, dictionary code uint8  (hash = per-code hashbpchar)    */
	CB_DICT32 = 7,		/* same, int32 code                                                       */
	CB_FLOAT8 = 8,		/* double precision                IEEE binary64                          */
	CB_BOOL = 9,		/* expression results only                                                */
	CB_NUMERIC128 = 10,	/* aggregate outputs: int128 scaled by 10^dscale (little endian lo,hi)    */
	CB_TEXT = 11		/* a string literal (CbExpr.conststr): LIKE patterns, IN list elements    */
} CbTypeId;

static inline int
cb_type_width(CbTypeId t)
{
	switch (t)
	{
		case CB_INT4: case CB_DATE: case CB_DICT32: return 4;
		case CB_INT8: case CB_NUMERIC: case CB_FLOAT8: return 8;
		case CB_BPCHAR1: case CB_DICT8: case CB_BOOL: return 1;
		case CB_NUMERIC128: return 16;
		case CB_TEXT: return 0;		/* constants only, never a column */
	}
	return 0;
}

/* ---- node tags ---- */
typedef enum CbNodeTag
{
	T_CbInvalid = 0,
	/* plan nodes */
	T_CbSeqScan = 100, T_CbHash, T_CbHashJoin, T_CbAgg, T_CbMotion, T_CbLimitSort,
	/* expression nodes */
	T_CbVar = 200, T_CbConst, T_CbOpExpr, T_CbBoolExpr, T_CbAggref,
	T_CbScalarArrayOpExpr		/* primnodes.h ScalarArrayOpExpr: args[0] op ANY (useOr) / ALL (!useOr) of args[1 ..] */
} CbNodeTag;

/* special varnos (primnodes.h: INNER_VAR 65000, OUTER_VAR 65001) */
#define CB_INNER_VAR 65000
#define CB_OUTER_VAR 65001

typedef enum CbOp
{
	CB_OP_ADD = 1, CB_OP_SUB, CB_OP_MUL,				/* int4/int8/numeric/float8 arithmetic     */
	CB_OP_EQ = 10, CB_OP_NE, CB_OP_LT, CB_OP_LE, CB_OP_GT, CB_OP_GE,	/* comparisons -> bool            */
	CB_OP_LIKE = 20, CB_OP_NOTLIKE		/* ~~ / !~~ (textlike, bpcharlike): args (Var, CB_TEXT Const) */
} CbOp;

typedef enum CbBoolOp { CB_AND_EXPR = 0, CB_OR_EXPR, CB_NOT_EXPR } CbBoolOp;	/* primnodes.h BoolExprType */

/* aggregate functions on the path (SURVEY.md 8a row a9; include/catalog/pg_aggregate.dat) */
typedef enum CbAggFn
{
	CB_AGG_COUNT_STAR = 1,	/* int8inc                       */
	CB_AGG_COUNT,			/* int8inc_any                   */
	CB_AGG_SUM,				/* int4_sum / int8_avg_accum / numeric_avg_accum / float8pl */
	CB_AGG_AVG,				/* int8_avg_accum / numeric_avg_accum / float8_accum        */
	CB_AGG_MIN,				/* int4smaller ...               */
	CB_AGG_MAX				/* int4larger ...                */
} CbAggFn;

typedef struct CbExpr
{
	CbNodeTag	tag;
	CbTypeId	restype;	/* result type                                                            */
	int32_t		dscale;		/* numeric display scale of the result (numeric.c: add/sub max, mul sum)  */
	/* T_CbVar */
	int32_t		varno;		/* CB_OUTER_VAR / CB_INNER_VAR, or scanrelid for a scan-level Var         */
	int32_t		varattno;	/* 1-based attribute number                                               */
	/* T_CbConst */
	int64_t		constval;	/* ints/date/numeric(scaled)/dict code; float8 bits for CB_FLOAT8         */
	bool		constisnull;
	/* T_CbOpExpr / T_CbBoolExpr / T_CbAggref */
	int32_t		op;			/* CbOp | CbBoolOp | CbAggFn                                              */
	int32_t		nargs;
	struct CbExpr **args;
	/* T_CbConst of type CB_TEXT: the string's bytes (no terminator needed) */
	const char *conststr;
	int32_t		constlen;
	/* T_CbScalarArrayOpExpr: true = ANY (x IN (...) is `=` with useOr), false = ALL (x NOT IN (...) is `<>` without) */
	bool		useOr;
} CbExpr;

typedef struct CbTargetEntry
{
	CbExpr	   *expr;
	int32_t		resno;		/* 1-based position in the node's output                                  */
	const char *resname;
} CbTargetEntry;

/* ---- plan nodes ---- */
typedef struct CbPlan
{
	CbNodeTag	type;
	int32_t		plan_node_id;
	double		plan_rows;		/* planner's row estimate                                             */
	int32_t		ntargets;
	CbTargetEntry *targetlist;
	int32_t		nquals;			/* implicitly-ANDed                                                   */
	CbExpr	  **qual;
	struct CbPlan *lefttree;	/* outer                                                              */
	struct CbPlan *righttree;	/* inner                                                              */
} CbPlan;

typedef struct CbSeqScan
{
	CbPlan		plan;
	int32_t		scanrelid;		/* 1-based index into CbEState.es_range_table                         */
} CbSeqScan;

typedef struct CbHash
{
	CbPlan		plan;
	int32_t		nhashkeys;
	CbExpr	  **hashkeys;		/* over OUTER_VAR (the Hash node's child)                             */
} CbHash;

/* nodes/nodes.h JoinType */
typedef enum CbJoinType
{
	CB_JOIN_INNER = 0, CB_JOIN_LEFT, CB_JOIN_FULL, CB_JOIN_RIGHT, CB_JOIN_SEMI, CB_JOIN_ANTI,
	CB_JOIN_LASJ_NOTIN			/* left anti semi join with NOT IN semantics (nodes/nodes.h:897; nodeHashjoin.c:371-390, 578-590) */
} CbJoinType;

typedef struct CbHashJoin
{
	CbPlan		plan;			/* lefttree = outer (probe) side, righttree = the CbHash node         */
	CbJoinType	jointype;
	int32_t		nhashkeys;
	CbExpr	  **hashkeys;		/* outer-side key expressions (over OUTER_VAR), pairwise with the
								 * inner CbHash.hashkeys; equality is the hash clause                 */
	int32_t		njoinquals;		/* extra non-hash join quals (Vars may be OUTER_VAR and INNER_VAR)    */
	CbExpr	  **joinqual;
} CbHashJoin;

/* nodes/nodes.h AggStrategy / AggSplit */
typedef enum CbAggStrategy { CB_AGG_PLAIN = 0, CB_AGG_SORTED, CB_AGG_HASHED, CB_AGG_MIXED } CbAggStrategy;
typedef enum CbAggSplit
{
	CB_AGGSPLIT_SIMPLE = 0,			/* one-stage                                                      */
	CB_AGGSPLIT_INITIAL_SERIAL,		/* partial: emit transition states                                */
	CB_AGGSPLIT_FINAL_DESERIAL		/* final: combine transition states                               */
} CbAggSplit;

typedef struct CbAgg
{
	CbPlan		plan;			/* targetlist: group Vars (OUTER_VAR) and T_CbAggref entries          */
	CbAggStrategy aggstrategy;
	CbAggSplit	aggsplit;
	int32_t		numCols;
	int32_t	   *grpColIdx;		/* 1-based attnos in the child's output                               */
	int64_t		numGroups;		/* planner estimate                                                   */
	bool		streaming;
} CbAgg;

/* plannodes.h:1636 MotionType */
typedef enum CbMotionType
{
	CB_MOTIONTYPE_GATHER = 0, CB_MOTIONTYPE_GATHER_SINGLE, CB_MOTIONTYPE_HASH, CB_MOTIONTYPE_BROADCAST
} CbMotionType;

typedef struct CbSortKey { int32_t attno; bool descending; } CbSortKey;
typedef struct CbMotion
{
	CbPlan		plan;
	CbMotionType motionType;
	int32_t		motionID;
	int32_t		nhashExprs;
	CbExpr	  **hashExprs;		/* over OUTER_VAR                                                     */
	int32_t		numHashSegments;
	/* sendSorted (plannodes.h Motion.sendSorted / numSortCols / sortColIdx): every sender's stream is ordered by these
	 * keys and the receiver merges the streams (execMotionSortedReceiver, nodeMotion.c:433; CdbMergeComparator :1010).
	 * Gather motions only; 0 keys = arrival order */
	int32_t		nsortkeys;
	CbSortKey  *sortkeys;
} CbMotion;

/*
 * Sort + Limit above the aggregate (nodeSort.c / nodeLimit.c) are out of scope as general
 * operators, but Q3 needs a device top-N so ~1.2M groups are not drained through slots
 * (SURVEY.md 8a row a8).  CbLimitSort = Limit(Sort(child)) with a bounded heap, as
 * tuplesort's bounded mode would run it.
 */
typedef struct CbLimitSort
{
	CbPlan		plan;
	int32_t		nkeys;
	CbSortKey  *keys;
	int64_t		limit;
} CbLimitSort;

#ifdef __cplusplus
}
#endif
#endif							/* CB_PLAN_H */
