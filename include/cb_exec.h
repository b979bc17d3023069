/*
 * cb_exec.h - the host executor: the reference's PlanState / ExecProcNode operator API for the
 * scan -> hash join -> hash aggregate (+ Motion) path, in plain C over the CUDA C ABI (cbgpu.h).
 *
 * Names, argument meaning and life cycle follow the reference (paths under /root/reference/src):
 *
 *   cb_ExecInitNode      ExecInitNode            backend/executor/execProcnode.c:190
 *   cb_ExecProcNode      ExecProcNode            include/executor/executor.h (-> ps->ExecProcNode,
 *                                                typedef ExecProcNodeMtd include/nodes/execnodes.h:1056)
 *   cb_MultiExecProcNode MultiExecProcNode       backend/executor/execProcnode.c:718 (Hash build)
 *   cb_ExecEndNode       ExecEndNode             backend/executor/execProcnode.c:791
 *   cb_ExecReScan        ExecReScan              backend/executor/execAmi.c
 *   cb_ExecSquelchNode   ExecSquelchNode         backend/executor/execAmi.c:763
 *   CbPlanState          PlanState               include/nodes/execnodes.h:1065-1164
 *   CbTupleTableSlot     TupleTableSlot (virtual) include/executor/tuptable.h:115-132
 *   CbEState             EState                  include/nodes/execnodes.h
 *   CbInterconnect       MotionIPCLayer          include/cdb/ml_ipc.h:36-210
 *
 * Contract kept: ExecProcNode returns one tuple per call in the node's result slot and NULL (or an
 * empty slot) at end of data; a parent pulls its children through the same entry point.  Inside,
 * operators exchange device column batches and whole sub-trees (scan + joins + aggregate) are
 * fused into one kernel, so only post-aggregation rows are ever materialised one by one.
 *
 * Errors: the reference ereport(ERROR)s, i.e. siglongjmp (utils/elog.h:185).  Here every entry
 * point records (code, message) in the EState and returns NULL / a negative code; a backend shim
 * calls ereport after cb_ExecEndNode has released device memory.  If es_error_hook is set it is
 * called with the same (code, message) at the point of failure.
 */
#ifndef CB_EXEC_H
#define CB_EXEC_H

#include "cbgpu.h"

#ifdef __cplusplus
extern "C" {
#endif

struct CbPlanState;
struct CbEState;
struct CbInterconnect;

/* a numeric result Datum (by reference, like the reference's Numeric varlena) */
typedef struct CbNumericDatum
{
	int64_t		lo, hi;			/* unscaled 128-bit value (two's complement) when it fits           */
	int32_t		dscale;
	char		text[84];		/* exact decimal text, as numeric_out() prints it                   */
} CbNumericDatum;

typedef struct CbTupleTableSlot
{
	bool		tts_empty;		/* TTS_FLAG_EMPTY                                                    */
	int32_t		tts_nvalid;
	int32_t	   *tts_types;		/* CbTypeId per attribute                                            */
	int64_t    *tts_values;		/* Datum: by value (ints, date, codes, float8 bits) or a pointer
								 * to a CbNumericDatum for CB_NUMERIC / CB_NUMERIC128                */
	bool	   *tts_isnull;
	/* partial aggregate states (AGGSPLIT_INITIAL_SERIAL outputs): N and the 128-bit sum per column */
	int64_t    *tts_state_n;
	int64_t    *tts_state_lo;
	int64_t    *tts_state_hi;
} CbTupleTableSlot;

typedef CbTupleTableSlot *(*CbExecProcNodeMtd) (struct CbPlanState *pstate);

typedef struct CbInstrumentation
{
	double		ntuples;		/* tuples emitted through ExecProcNode                               */
	double		nloops;
	int64_t		kernels;		/* device kernels launched on behalf of this node                    */
	double		device_ms;		/* CUDA-event time of this node's pipelines                          */
	int64_t		rows_in;		/* rows of the driving relation(s) this node's pipelines scanned     */
	int64_t		motion_repartitions;	/* Motion sender: passes redone with exact sizes after a destination
								 * outgrew its share (data skew)                                     */
	int64_t		hashjoin_nbatch;	/* Hash: batches the build side was split into (1: it fitted)        */
	int64_t		agg_npartitions;	/* Agg: passes a partitioned aggregation took (1: the table fitted)  */
	double		having_ms;		/* Agg: time of the device HAVING step (host clock around cbgpu_having_select's
								 * launches and its one read-back of the selected count)             */
} CbInstrumentation;

typedef struct CbPlanState
{
	CbNodeTag	type;
	CbPlan	   *plan;
	struct CbEState *state;
	CbExecProcNodeMtd ExecProcNode;
	CbInstrumentation instrument;
	struct CbPlanState *lefttree;
	struct CbPlanState *righttree;
	CbTupleTableSlot *ps_ResultTupleSlot;
	bool		squelched;
	void	   *priv;			/* node-private state                                                */
} CbPlanState;

typedef void (*CbErrorHook) (struct CbEState *estate, int code, const char *message);

typedef struct CbEState
{
	cbgpu_ctx  *es_ctx;
	int32_t		es_nrels;
	cbgpu_rel **es_range_table;	/* scanrelid - 1 -> relation                                         */
	int32_t		es_segindex;	/* GpIdentity.segindex                                               */
	int32_t		es_numsegments;
	struct CbInterconnect *es_interconnect;	/* NULL when es_numsegments == 1                         */
	int32_t		es_errcode;
	char		es_errmsg[512];
	CbErrorHook es_error_hook;
	int32_t		es_force_generic;	/* tests: never use the pattern-specialised kernels              */
	int64_t		es_processed;
	void	   *es_cluster;		/* in-process multi-segment runs: the owning CbCluster               */
	/* CHECK_FOR_INTERRUPTS / QueryFinishPending for the batch executor (miscadmin.h:161; execProcnode.c:642; the
	 * reference polls them per tuple in nodeAgg.c:2342, nodeHashjoin.c:260): called between pipelines, i.e. before every
	 * kernel that walks a relation.  Non-zero = stop: the query ends with CBGPU_ERR_INTERRUPTED (peers are told through the
	 * interconnect's abandon()).  The callback must NOT longjmp (ereport): CUDA / NCCL frames are live; the shim raises the
	 * error after cb_ExecEndNode has released device memory.  NULL: never interrupted. */
	int			(*es_interrupt_pending) (struct CbEState *estate);
	void	   *es_interrupt_arg;
	/* operator memory budget in KB (PlanStateOperatorMemKB, execnodes.h:1166; nodeHash.c:980-990 turns it into nbatch):
	 * a hash join build side or an aggregate table larger than this is processed in several passes (multi-batch hybrid
	 * hash join, partitioned aggregation).  0 = whatever the device holds. */
	int64_t		es_operator_mem_kb;
	int64_t		es_hashjoin_batches_run;	/* passes of multi-batch hash joins so far (statistics)           */
	int64_t		es_agg_partitions_run;		/* passes of partitioned aggregations so far                      */
} CbEState;

CbEState   *cb_CreateExecutorState(cbgpu_ctx *ctx, cbgpu_rel **range_table, int32_t nrels);
void		cb_FreeExecutorState(CbEState *estate);
const char *cb_estate_error(CbEState *estate);

CbPlanState *cb_ExecInitNode(CbPlan *node, CbEState *estate, int eflags);
CbTupleTableSlot *cb_ExecProcNode(CbPlanState *node);
/* Hash nodes only: runs the build (MultiExecHash, nodeHash.c:130); returns the hash table */
cbgpu_hashtable *cb_MultiExecProcNode(CbPlanState *node);
/* batch-oriented twin of cb_ExecProcNode: the node's whole output as one device-resident column
 * batch (one column per scalar output, N / sum-lo / sum-hi per transition state); the relation
 * becomes the caller's.  Scan, HashJoin and Motion sub-trees; Agg / LimitSort finalise on the host
 * and return CBGPU_ERR_UNSUPPORTED. */
int			cb_ExecProcNodeBatch(CbPlanState *node, cbgpu_rel **out);
void		cb_ExecEndNode(CbPlanState *node);
void		cb_ExecReScan(CbPlanState *node);
void		cb_ExecSquelchNode(CbPlanState *node);

/* slot accessors (slot_getattr, executor/tuptable.h) */
#define CbTupIsNull(slot) ((slot) == NULL || (slot)->tts_empty)
int			cb_slot_natts(const CbTupleTableSlot *slot);
int			cb_slot_isnull(const CbTupleTableSlot *slot, int attno);
int64_t		cb_slot_int64(const CbTupleTableSlot *slot, int attno);
double		cb_slot_float8(const CbTupleTableSlot *slot, int attno);
/* value as text the way the reference prints it (numeric_out, int8out, float8out %.17g) */
int			cb_slot_text(const CbTupleTableSlot *slot, int attno, char *buf, int buflen);

/* numeric finalisation helpers (numeric_sum / numeric_avg, utils/adt/numeric.c:6091,6056 with
 * select_div_scale :9194): exact text from (sum, dscale[, N]) */
void		cb_numeric_sum_text(int64_t lo, int64_t hi, int32_t dscale, char *out, int32_t outlen);
void		cb_numeric_avg_text(int64_t lo, int64_t hi, int32_t dscale, int64_t n, char *out, int32_t outlen);
/* A partial aggregate state (N, exact 128-bit sum scaled by 10^dscale) as the bytea the reference's serialisation function
 * makes of it, for a Finalize stage that runs on a CPU process behind a Motion - and back (AGGSPLIT_INITIAL_SERIAL /
 * FINAL_DESERIAL, nodes/nodes.h:977-1000): numeric_avg_serialize / _deserialize (utils/adt/numeric.c:5025-5156) for sum / avg
 * over numeric, int8_avg_serialize / _deserialize (numeric.c:5793-5870) for sum / avg over int8.  Serialise: the bytes written,
 * or -1 when `cap` is too small.  Deserialise: 0, -1 malformed, -2 NaN / infinity inputs, -3 not representable as a 128-bit sum
 * at its display scale. */
int			cb_numeric_avg_serialize(int64_t n, int64_t sum_lo, int64_t sum_hi, int32_t dscale, uint8_t *out, int32_t cap);
int			cb_int8_avg_serialize(int64_t n, int64_t sum_lo, int64_t sum_hi, uint8_t *out, int32_t cap);
int			cb_numeric_avg_deserialize(const uint8_t *in, int32_t len, int32_t with_tail, int64_t *n, int64_t *sum_lo, int64_t *sum_hi,
									   int32_t *dscale);

/* ------------------------------------------------------------------------------------------
 * interconnect: what the reference reaches through MotionIPCLayer (include/cdb/ml_ipc.h:36)
 * ------------------------------------------------------------------------------------------ */
typedef struct CbInterconnect
{
	const char *name;
	int32_t		nsegs;
	int32_t		segindex;
	/* Redistribute (staged): `send` holds this segment's rows grouped by destination (destination d's rows
	 * start at row offsets[d], counts[d] of them).  Returns the rows addressed to this segment. */
	int			(*redistribute) (struct CbInterconnect *ic, struct CbEState *estate, int32_t motion_id,
								 cbgpu_rel *send, const int64_t *counts, const int64_t *offsets, cbgpu_rel **recv);
	/* Gather: every segment's rows to segment `root`; other segments get an empty relation */
	int			(*gather) (struct CbInterconnect *ic, struct CbEState *estate, int32_t motion_id, int32_t root,
						   cbgpu_rel *send, int64_t nrows, cbgpu_rel **recv);
	/* Broadcast: every segment receives every segment's rows */
	int			(*broadcast) (struct CbInterconnect *ic, struct CbEState *estate, int32_t motion_id,
							  cbgpu_rel *send, int64_t nrows, cbgpu_rel **recv);
	void		(*teardown) (struct CbInterconnect *ic);
	void	   *priv;
	/* optional (NULL when the interconnect has no peer memory): Redistribute fused into the sender
	 * slice's kernel (cbgpu_motion_direct_begin / _end, include/cbgpu.h).  begin is local and returns the
	 * PARTITION sink's destination tables; a non-zero return means "use redistribute() for this Motion" and
	 * is the same on every segment.  end signals, waits for every sender, takes delivery; *outcome ==
	 * CBGPU_DX_RETRY: nothing was delivered (a destination overflowed somewhere), every segment redoes the
	 * Motion through redistribute(). */
	int			(*direct_begin) (struct CbInterconnect *ic, struct CbEState *estate, int32_t motion_id, int32_t ncols,
								 const int32_t *types, const int32_t *dscales, cbgpu_direct_dest *dest);
	int			(*direct_end) (struct CbInterconnect *ic, struct CbEState *estate, int32_t motion_id, int32_t local_flags,
							   uint64_t local_nullmask, const int64_t *dev_sent_counts, int64_t *sent_counts, cbgpu_rel **recv,
							   int32_t *outcome);
	/* this segment failed before (after_direct = 0) or after (1: the direct attempt ended in CBGPU_DX_RETRY)
	 * the Motion's first exchange and will not take part: tell the peers, which then fail with
	 * CBGPU_ERR_PEER instead of waiting (the reference's senders notice a dead peer through the
	 * interconnect's own error path, ic_udpifc.c; TeardownInterconnect hasErrors, ml_ipc.h:106).  Optional. */
	void		(*abandon) (struct CbInterconnect *ic, struct CbEState *estate, int32_t motion_id, int32_t after_direct);
} CbInterconnect;

/* interconnect over NCCL (cbgpu_motion_*): one process per GPU-segment.  SetupInterconnect
 * (executor/execMain.c:531) equivalent: attach the result to CbEState.es_interconnect and set
 * es_segindex / es_numsegments. */
CbInterconnect *cb_interconnect_nccl_create(cbgpu_motion *motion);
void		cb_interconnect_destroy(CbInterconnect *ic);

/*
 * In-process cluster: N segment executors over one context (the reference tests "multi-node" the
 * same way: gpdemo runs every segment on one host, gpAux/gpdemo/demo_cluster.sh).  Each segment has
 * its own range table; Motion nodes exchange device batches through the local interconnect.
 */
typedef struct CbCluster CbCluster;
CbCluster  *cb_cluster_create(cbgpu_ctx *ctx, int32_t nsegs);
/* range table of one segment (pointers are borrowed) */
int			cb_cluster_set_range_table(CbCluster *c, int32_t seg, cbgpu_rel **range_table, int32_t nrels);
CbEState   *cb_cluster_estate(CbCluster *c, int32_t seg);
/* ExecInitNode on every segment; returns the root PlanState of segment 0's copy */
int			cb_cluster_init_plan(CbCluster *c, CbPlan *plan);
/* pull the next tuple of the whole query: the top slice of each segment in turn (a slice that
 * receives from a Gather Motion runs on segment 0 only) */
CbTupleTableSlot *cb_cluster_next(CbCluster *c);
int32_t		cb_cluster_current_segment(CbCluster *c);
/* root PlanState of one segment's copy of the plan, from cb_cluster_init_plan to cb_cluster_end (its instrumentation) */
CbPlanState *cb_cluster_root(CbCluster *c, int32_t seg);
void		cb_cluster_end(CbCluster *c);
void		cb_cluster_destroy(CbCluster *c);
const char *cb_cluster_error(CbCluster *c);

/* ------------------------------------------------------------------------------------------
 * AOCS segment files from disk (the storage side of aocs_beginscan / open_next_scan_seg, access/aocs/aocsam.c)
 * ------------------------------------------------------------------------------------------ */
/* <basepath>[.<(filenum - 1) * 128 + segno>]: FormatAOSegmentFileName (access/appendonly/aomd.c:84-117); basepath =
 * relpathbackend() of the relation, filenum = pg_attribute_encoding.filenum of the column (1-based), segno 0..127.
 * 0, or -1 when the arguments are out of range or `out` is too small. */
int			cb_aocs_segfile_path(const char *basepath, int segno, int filenum, char *out, size_t outsz);

typedef struct CbAocsColumnSpec
{
	int32_t		relcol;			/* column of the device relation to fill                               */
	int32_t		filenum;		/* pg_attribute_encoding.filenum                                       */
	int32_t		attlen;			/* pg_attribute.attlen: 1/2/4/8, or -1 with varkind                    */
	int32_t		varkind;		/* CBGPU_AOCS_VAR_*                                                    */
	int32_t		typalign;		/* bytes                                                               */
	int32_t		compresstype;	/* CBGPU_AOCS_COMPRESS_*                                               */
	int64_t		eof;			/* pg_aocsseg.vpinfo eof of the column for this segno; < 0 = whole file */
	cbgpu_dict *dict;			/* varkind CBGPU_AOCS_VAR_DICT: the column's (finalized) dictionary    */
} CbAocsColumnSpec;
/* first pass for a string column: the distinct values of this segment file join spec->dict (cbgpu_aocs_dict_collect) */
int			cb_aocs_dict_collect_segfile(cbgpu_ctx *ctx, const char *basepath, int segno, int checksum, const CbAocsColumnSpec *spec,
										 char *err, size_t errsz);
/* Reads every listed column's segment file of `segno` up to its EOF and decodes it on the device into rows
 * [row_offset, +nrows) of `rel` (cbgpu_aocs_decode_column_ex: block CRC-32C when checksum != 0, zlib / zstd
 * decompression, datum stream decode), checks that the columns agree on the row count, then applies the segment
 * file's pg_aovisimap rows (cbgpu_aocs_apply_visimap; none and no earlier bitmap = nothing to do).  err (optional)
 * receives a message naming the file. */
int			cb_aocs_load_segfile(cbgpu_ctx *ctx, const char *basepath, int segno, int checksum, int ncols,
								 const CbAocsColumnSpec *cols, cbgpu_rel *rel, int64_t row_offset,
								 const cbgpu_visimap_entry *entries, int nentries, int64_t *nrows, int64_t *nhidden,
								 char *err, size_t errsz);

/* ------------------------------------------------------------------------------------------
 * Rows in the reference's Motion wire format (cdb/motion/tupser.c: SerializeTuple :349, CvtChunksToTup :515;
 * include/cdb/tupchunk.h), for interconnect traffic between GPU segments and un-replaced CPU operators
 * ------------------------------------------------------------------------------------------ */
#define CB_TUPSER_MAX_ATTS 1600	/* MaxTupleAttributeNumber */
#define CB_TUPSER_MAX_TEXT 8192	/* longest character(n) padding done here                              */
typedef struct CbTupAttr
{
	int32_t		type;			/* CbTypeId of the column                                              */
	int32_t		dscale;			/* CB_NUMERIC: scale of the int64 values                               */
	int32_t		bpchar_len;		/* dictionary column declared character(n): n, else 0 (varchar / text) */
	int32_t		ntexts;			/* dictionary columns: the texts of codes 0 .. ntexts-1, in byte order  */
	const char *const *texts;	/* (what cbgpu_dict_entry returns for each code; character(n) texts     */
	const int32_t *text_lens;	/* without their trailing blanks)                                      */
	struct CbAggStateDatum *state;	/* CB_TUPSER_STATE_*: where cb_tupser_next puts the row's state        */
} CbTupAttr;
/* A partial aggregate state as a tuple attribute: on the wire it is the bytea the aggregate's serialisation function makes
 * (cb_numeric_avg_serialize / cb_int8_avg_serialize above; AGGSPLIT_INITIAL_SERIAL target lists are typed bytea), in the
 * executor it is (N, exact 128-bit sum).  cb_tupser_row takes values[i] = a pointer to the CbAggStateDatum to send;
 * cb_tupser_next fills attrs[i].state and returns that pointer in values[i].  dscale = the sum's display scale. */
typedef struct CbAggStateDatum
{
	int64_t		n,
				lo,
				hi;
} CbAggStateDatum;
#define CB_TUPSER_STATE_NUMERIC 101	/* sum / avg over numeric: numeric_avg_serialize form                  */
#define CB_TUPSER_STATE_INT8 102	/* sum / avg over int8: int8_avg_serialize form                        */
/* One row (values as the executor holds them: by-value datums, scaled numerics, dictionary codes) -> its tuple chunks:
 * TC_WHOLE, or TC_PARTIAL_START / _MID / _END when [int32 length][MinimalTuple body] exceeds max_chunk
 * (Gp_max_tuple_chunk_size) minus the 4-byte chunk header.  Returns the bytes written, < 0 on error (-2: out too small). */
int64_t		cb_tupser_row(const CbTupAttr *attrs, int natts, const int64_t *values, const uint8_t *isnull, int max_chunk,
						  unsigned char *out, int64_t outcap);
/* the TC_END_OF_STREAM chunk a sender finishes with */
int			cb_tupser_end_of_stream(unsigned char *out, int64_t outcap);
#define CB_TUPSER_END 0			/* TC_END_OF_STREAM                                                    */
#define CB_TUPSER_NEED_MORE (-1)	/* the buffer ends inside a tuple: call again with more bytes          */
#define CB_TUPSER_BAD (-2)		/* chunk sequence or tuple layout the reference would reject           */
/* The next row of a chunk stream: 1 and *consumed bytes used, or one of the codes above.  Strings are mapped to the
 * attribute's dictionary codes (a string it does not hold: CB_TUPSER_BAD). */
int64_t		cb_tupser_next(const CbTupAttr *attrs, int natts, const unsigned char *in, int64_t inlen, int64_t *consumed,
						   int64_t *values, uint8_t *isnull);

#ifdef __cplusplus
}
#endif
#endif							/* CB_EXEC_H */
