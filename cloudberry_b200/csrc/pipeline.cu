/*
 * pipeline.cu - cbgpu_pipeline_run: descriptor validation, dispatch, and the generic pipeline kernel.
 *
 * A pipeline is the GPU form of one slice-internal chain of the reference's pull executor between
 * two pipeline breakers: the driving scan (aocs_getnext, backend/access/aocs/aocsam.c:1418), its
 * quals (ExecScan -> ExecQual, backend/executor/execScan.c:162), zero or more hash-join probes
 * (ExecHashJoinImpl HJ_NEED_NEW_OUTER / HJ_SCAN_BUCKET, backend/executor/nodeHashjoin.c:476,575)
 * and one sink: hash aggregation (agg_fill_hash_table, backend/executor/nodeAgg.c:2726),
 * materialisation for a Hash build side (MultiExecPrivateHash, nodeHash.c:167) or the sending half
 * of a Redistribute Motion (execMotionSender + evalHashKey, backend/executor/nodeMotion.c:203,1088).
 *
 * The generic kernel interprets the descriptor's postfix program one row per thread, warp
 * synchronously (all lanes step the same program counter; dead rows are masked), with late
 * materialisation: a column is read only when an expression needs it, and only for rows still
 * alive.  Pattern-specialised kernels (scan_agg.cu, ...) take over when the descriptor matches a
 * shape they fuse by hand; results are identical (tests run both).
 */
#include "pipeline.cuh"
#include "xmatch.h"

#include <stdlib.h>

/* ---------------------------------------------------------------------------------------------
 * host: descriptor -> device form, and the program's expression trees in *xp
 * --------------------------------------------------------------------------------------------- */
int
cb_pipeline_to_dev(cbgpu_ctx *ctx, const CbPipeline *p, PipeDev *d, XProg *xp)
{
	memset(d, 0, sizeof(*d));
	if (p->nrows < 0 || p->nrows > 0xFFFFFFF0ll)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "pipeline over %s%lld rows exceeds 32-bit row ids", "", p->nrows);
	if (p->ncols < 0 || p->ncols > CBP_MAX_COLS || p->nops < 1 || p->nops > CBP_MAX_OPS ||
		p->nprobes < 0 || p->nprobes > CBP_MAX_SRC - 1 || p->drv_nsrc < 0 || p->drv_nsrc > CBP_MAX_SRC)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "pipeline descriptor exceeds the GPU path's limits%s (%lld ops)", "", p->nops);
	d->nrows = p->nrows;
	d->visimap = p->visimap;
	d->drv_nsrc = p->drv_nsrc;
	for (int s = 0; s < CBP_MAX_SRC; s++)
		d->drv_idx[s] = s < p->drv_nsrc ? p->drv_idx[s] : NULL;
	d->ncols = p->ncols;
	for (int c = 0; c < p->ncols; c++)
	{
		d->cols[c] = p->cols[c];
		if (p->cols[c].src < 0 || p->cols[c].src >= CBP_MAX_SRC || cb_type_w(p->cols[c].type) == 0)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline column %s%lld malformed", "", c);
	}
	d->nops = p->nops;
	memcpy(d->ops, p->ops, sizeof(CbpOp) * (size_t) p->nops);
	if (p->nsets < 0 || p->nsets > CBP_MAX_SETS)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline declares %s%lld code sets", "", p->nsets);
	for (int i = 0; i < p->nsets; i++)
	{
		if (p->sets[i].nbits < 0 || (p->sets[i].nbits > 0 && !p->sets[i].bits))
			return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline code set %s%lld malformed", "", i);
		d->sets[i] = p->sets[i];
	}
	{
		const XAllow allow = {"pipeline", XM_PIPELINE_OPS, p->probes, p->nprobes, CBGPU_ERR_UNSUPPORTED, p->nsets};
		const int	rc = xm_walk(ctx, allow, p->ncols, p->ops, p->nops, xp);

		if (rc != CBGPU_OK)
			return rc;
	}
	if (p->ops[p->nops - 1].code != CBP_END)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline program does not end with END%s", "", 0);
	d->nprobes = p->nprobes;
	d->src_base = p->drv_nsrc > 1 ? p->drv_nsrc : 1;
	if (d->src_base + p->nprobes > CBP_MAX_SRC)
		return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "pipeline joins more than %s%lld sources", "", CBP_MAX_SRC);
	for (int j = 0; j < p->nprobes; j++)
	{
		const CbpProbe *pp = &p->probes[j];

		if (!pp->ht || pp->nkeys != pp->ht->d.nkeys)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline probe %s%lld: hash table / key count mismatch", "", j);
		if (pp->jointype != CB_JOIN_INNER && pp->jointype != CB_JOIN_LEFT && pp->jointype != CB_JOIN_SEMI && pp->jointype != CB_JOIN_ANTI)
			return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "join type %s%lld is not implemented on the GPU path", "", pp->jointype);
		if (pp->ht->has_dups && (pp->jointype == CB_JOIN_INNER || pp->jointype == CB_JOIN_LEFT))
			return cb_fail(ctx, CBGPU_ERR_INVALID, "fused probe %s%lld needs unique build keys; use cbgpu_ht_probe_pairs", "", j);
		d->probes[j].ht = pp->ht->d;
		d->probes[j].jointype = pp->jointype;
		d->probes[j].null_key_drops = pp->null_key_drops;
		d->probes[j].nkeys = pp->nkeys;
		for (int k = 0; k < pp->nkeys; k++)
		{
			d->probes[j].keytype[k] = pp->keytype[k];
			d->probes[j].keydict[k] = pp->key_dict_hash[k];
		}
	}
	const CbpSink *s = &p->sink;
	DSink	   *ds = &d->sink;
	SinkOut    *o = &ds->out;

	ds->kind = s->kind;
	switch (s->kind)
	{
		case CBP_SINK_AGG:
			if (s->nkeys < 0 || s->nkeys > CBP_MAX_GROUP_KEYS)
				return cb_fail(ctx, CBGPU_ERR_UNSUPPORTED, "GROUP BY with %s%lld columns is beyond the GPU path's limit (8)", "", s->nkeys);
			if (!s->agg || s->nkeys != s->agg->d.nkeys || s->naccs != s->agg->d.naccs)
				return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline sink: agg table shape mismatch%s", "", 0);
			ds->agg = s->agg->d;
			cb_agg_touch(s->agg);
			ds->nkeys = s->nkeys;
			ds->naccs = s->naccs;
			for (int k = 0; k < s->nkeys; k++)
			{
				/* the group hash only places a group in this table (a Motion routes by cdb_route, which refuses numeric keys):
				 * a numeric key column has one scale, so its scaled int64 identifies the value and hashes as an int8 */
				ds->keytype[k] = s->keytype[k] == CB_NUMERIC ? CB_INT8 : s->keytype[k];
				ds->keydict[k] = s->key_dict_hash[k];
			}
			{
				int			nargs = xp->depth - s->nkeys;

				for (int a = 0; a < s->naccs; a++)
				{
					int			need = s->accs[a].kind == CBP_ACC_MERGE_INT ? 3 : (s->accs[a].kind == CBP_ACC_MERGE_FLOAT || s->accs[a].kind == CBP_ACC_MERGE_MIN || s->accs[a].kind == CBP_ACC_MERGE_MAX) ? 2 : 1;

					ds->accs[a] = s->accs[a];
					if (s->accs[a].arg >= 0 && s->accs[a].arg + need > nargs)
						return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline sink: accumulator %s%lld argument beyond the stack", "", a);
					if (s->accs[a].arg < 0 && s->accs[a].kind != CBP_ACC_COUNT)
						return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline sink: accumulator %s%lld needs an argument", "", a);
				}
				if (nargs < 0)
					return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline sink: fewer stack values than keys%s", "", 0);
			}
			break;
		case CBP_SINK_MATERIALIZE:
		case CBP_SINK_PARTITION:
			if (!s->out || s->nout != xp->depth || s->nout > CBP_MAX_OUT || s->nout > s->out->ncols || !s->out_count)
				return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline sink: output shape mismatch%s (%lld values)", "", xp->depth);
			o->nout = s->nout;
			for (int c = 0; c < s->nout; c++)
			{
				o->outcol[c] = s->out->data[c];
				o->outnull[c] = s->out->nulls[c];
				o->outtype[c] = s->out->types[c];
			}
			o->out_count = (unsigned long long *) s->out_count;
			o->seg_cap[0] = s->out->capacity;
			if (s->kind == CBP_SINK_PARTITION)
			{
				if (s->nsegs < 1 || s->nsegs > 64 || s->nhash < 1 || s->nhash > CBP_MAX_KEYS || s->nhash > s->nout ||
					(!s->part_cols && !s->seg_base && s->seg_capacity * s->nsegs > s->out->capacity) || (s->part_cols && !s->part_counts) ||
					(s->part_cols && s->part_nullmask && !s->part_nulls) || (!s->seg_base != !s->seg_cap))
					return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline sink: bad partition description%s", "", 0);
				o->part_cols = s->part_cols;
				o->part_counts = s->part_counts;
				o->part_nulls = s->part_nulls;
				o->part_nullmask = s->part_cols ? s->part_nullmask : 0;
				o->part_flags = s->part_flags;
				o->nhash = s->nhash;
				o->nsegs = s->nsegs;
				for (int g = 0; g < s->nsegs; g++)
				{
					o->seg_base[g] = s->seg_base ? s->seg_base[g] : (int64_t) g * s->seg_capacity;
					o->seg_cap[g] = s->part_cols ? s->seg_capacity : s->seg_cap ? s->seg_cap[g] : s->seg_capacity;
					if (!s->part_cols && (o->seg_base[g] < 0 || o->seg_cap[g] < 0 || o->seg_base[g] + o->seg_cap[g] > s->out->capacity))
						return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline sink: destination %s%lld's range lies outside the send buffer", "", g);
				}
				for (int k = 0; k < s->nhash; k++)
				{
					o->hashtype[k] = s->hashtype[k];
					o->hashdict[k] = s->hash_dict_hash[k];
				}
			}
			break;
		default:
			return cb_fail(ctx, CBGPU_ERR_INVALID, "pipeline sink kind %s%lld unknown", "", s->kind);
	}
	/* peephole: the three shapes nearly every plan on this path contains run as single fused ops
	 * (no stack traffic): `col CMP const` quals, probes keyed by plain columns, a * (k - b) */
	{
		CbpOp	   *x = (CbpOp *) cb_scratch(ctx, 0, sizeof(CbpOp) * CBP_MAX_OPS);
		int			n = 0;
		int			i = 0;

		while (i < p->nops)
		{
			const CbpOp *o = &d->ops[i];

			if (i + 3 < p->nops && o[0].code == CBP_LOAD && o[1].code == CBP_CONST && o[2].code >= CBP_EQ && o[2].code <= CBP_GE &&
				o[3].code == CBP_FILTER && d->cols[o[0].a].type != CB_FLOAT8 && o[0].a < 0x10000)
			{
				x[n].code = XOP_FILTER_COL;
				x[n].a = o[0].a | (o[2].code << 16);
				x[n].imm = o[1].imm;
				n++;
				i += 4;
				continue;
			}
			if (i + 4 < p->nops && o[0].code == CBP_LOAD && o[1].code == CBP_CONST && o[2].code == CBP_LOAD && o[3].code == CBP_SUB &&
				o[4].code == CBP_MUL && o[0].a < 0x8000 && o[2].a < 0x8000)
			{
				x[n].code = XOP_MULCSUB;
				x[n].a = o[0].a | (o[2].a << 16);
				x[n].imm = o[1].imm;
				n++;
				i += 5;
				continue;
			}
			if (o[0].code == CBP_LOAD)
			{
				/* LOAD x nkeys then PROBE */
				int			k = 0;

				while (i + k < p->nops && d->ops[i + k].code == CBP_LOAD && k < CBP_MAX_KEYS && d->ops[i + k].a < 256)
					k++;
				if (i + k < p->nops && d->ops[i + k].code == CBP_PROBE && p->probes[d->ops[i + k].a].nkeys <= k)
				{
					int			nk = p->probes[d->ops[i + k].a].nkeys;
					int			skip = k - nk;	/* leading LOADs that are not keys stay as they are */
					uint64_t	cols = 0;

					for (int j = 0; j < skip; j++)
						x[n++] = d->ops[i + j];
					for (int j = 0; j < nk; j++)
						cols |= (uint64_t) d->ops[i + skip + j].a << (8 * j);
					x[n].code = XOP_PROBE_COLS;
					x[n].a = d->ops[i + k].a;
					x[n].imm = (int64_t) cols;
					n++;
					i += k + 1;
					continue;
				}
			}
			x[n++] = *o;
			i++;
		}
		memcpy(d->ops, x, sizeof(CbpOp) * (size_t) n);
		d->nops = n;
	}
	/* stage boundaries: after every PROBE (rows die there and the stack is empty) */
	{
		int			ns = 0,
					dep = 0;

		d->stage_pc[ns++] = 0;
		for (int i = 0; i < d->nops; i++)
		{
			const int	c = d->ops[i].code;
			const XEffect e = xm_effect(d->ops[i], p->probes);

			dep += e.pushes - e.pops;
			if ((c == CBP_PROBE || c == XOP_PROBE_COLS) && dep == 0 && ns < CBP_MAX_STAGES && i + 1 < d->nops)
				d->stage_pc[ns++] = i + 1;
		}
		d->nsrc = d->src_base + p->nprobes;
		/* queue shapes; keep the per-CTA queue area within 24 KB so 8 CTAs (64 warps) stay resident:
		 * the deepest cuts see the fewest rows and are dropped first */
		for (;;)
		{
			int			words = 0,
						probes = 0,
						pc = 0;

			for (int b = 0; b + 1 < ns; b++)
			{
				for (; pc < d->stage_pc[b + 1]; pc++)
					if (d->ops[pc].code == CBP_PROBE || d->ops[pc].code == XOP_PROBE_COLS)
						probes++;
				d->q_off[b] = words;
				d->q_ew[b] = d->src_base + probes + 1;
				words += 64 * d->q_ew[b];
			}
			d->q_words = words;
			if (words * 4 * 8 <= 24 * 1024 || ns <= 1)
				break;
			ns--;
		}
		d->nstages = ns;
		d->stage_pc[ns] = d->nops;
	}
	d->status = ctx->d_status;
	return CBGPU_OK;
}

/* ---------------------------------------------------------------------------------------------
 * generic kernel
 * --------------------------------------------------------------------------------------------- */
/* fetch column `ci` for this lane's row: value widened to 64 bits, NULL flag */
__device__ __forceinline__ int64_t
gen_load_col(const PipeDev &P, int ci, const uint32_t *ridx, uint32_t rnull, bool alive, bool *isnull)
{
	const CbpColumn &c = P.cols[ci];
	bool		n = (rnull >> c.src) & 1;
	int64_t		v = 0;

	if (alive && !n)
	{
		uint32_t	r = ridx[c.src];

		if (c.nulls && c.nulls[r])
			n = true;
		else
			v = cb_load_widen(c.data, c.type, r);
	}
	*isnull = n;
	return v;
}

#define GEN_THREADS 256
#define GEN_QCAP 64				/* entries per inter-stage queue (a stage runs as soon as 32 are waiting) */

/*
 * Staged execution.  The program is cut into stages at the points where rows can die and the
 * expression stack is empty (after every FILTER / PROBE).  Each warp owns one small queue per stage
 * boundary in shared memory, holding the source row ids of the rows that survived so far.  The warp
 * always runs the deepest stage that has a full warp's worth (32) of rows waiting, else feeds
 * stage 0 with the next 32 driving rows, and drains partial queues at the end.  So the ops behind a
 * selective qual or join probe execute with (nearly) full warps instead of once per original warp:
 * the device-side form of the row-at-a-time late materialisation of aocs_getnext_withqual
 * (backend/access/aocs/aocsam.c:1269,1359) and of probing only tuples that passed the scan qual.
 */
__global__ void __launch_bounds__(GEN_THREADS)
k_pipeline_generic(const __grid_constant__ PipeDev P)
{
	extern __shared__ uint32_t gen_smem[];
	const int	lane = threadIdx.x & 31;
	const int	warp_in_cta = threadIdx.x >> 5;
	const int	nq = P.nstages - 1;			/* queues per warp */
	/* queue b's entries hold the row ids of the sources known after stage b, plus the NULL-extension
	 * mask: q_ew[b] words each, at word offset q_off[b] of the warp's area */
	uint32_t   *myq = gen_smem + (size_t) warp_in_cta * P.q_words;
	int			qcnt[CBP_MAX_STAGES];		/* warp-uniform */
	const int64_t nchunks = (P.nrows + 31) / 32;
	int64_t		chunk = (int64_t) blockIdx.x * (GEN_THREADS / 32) + warp_in_cta;
	const int64_t chunk_stride = (int64_t) gridDim.x * (GEN_THREADS / 32);

#pragma unroll
	for (int s = 0; s < CBP_MAX_STAGES; s++)
		qcnt[s] = 0;

	for (;;)
	{
		/* ---- choose a stage ---- */
		int			stage = -1;
		int			navail = 0;

		for (int s = nq; s >= 1; s--)
			if (qcnt[s - 1] >= 32)
			{
				stage = s;
				navail = 32;
				break;
			}
		if (stage < 0)
		{
			if (chunk < nchunks)
				stage = 0;
			else
			{
				for (int s = 1; s <= nq; s++)
					if (qcnt[s - 1] > 0)
					{
						stage = s;
						navail = qcnt[s - 1];
						break;
					}
				if (stage < 0)
					break;
			}
		}

		/* ---- fetch this lane's row ---- */
		bool		alive;
		uint32_t	ridx[CBP_MAX_SRC];
		uint32_t	rnull = 0;		/* bit s: source s is NULL-extended (left join miss)              */
		int64_t		st[CBP_STACK];
		uint64_t	snull = 0;
		int			sp = 0;

#pragma unroll
		for (int s = 0; s < CBP_MAX_SRC; s++)
			ridx[s] = 0;
		if (stage == 0)
		{
			const int64_t base = chunk * 32 + lane;

			chunk += chunk_stride;
			alive = base < P.nrows;
			if (alive)
			{
				if (P.drv_nsrc == 0)
					ridx[0] = (uint32_t) base;
				else
					for (int s = 0; s < P.drv_nsrc; s++)
					{
						ridx[s] = P.drv_idx[s] ? P.drv_idx[s][base] : (uint32_t) base;
						/* a LEFT join's unmatched outer row arrives as a pair with no inner row, a RIGHT / FULL join's
						 * unmatched build row as a pair with no outer row: that source is NULL (ExecHashJoinImpl
						 * HJ_FILL_OUTER_TUPLE / HJ_FILL_INNER_TUPLES, nodeHashjoin.c:640-706) */
						if (P.drv_idx[s] && ridx[s] == 0xFFFFFFFFu)
						{
							rnull |= 1u << s;
							ridx[s] = 0;
						}
					}
				/* AppendOnlyVisimap_IsVisible (backend/access/appendonly/appendonly_visimap.c:198) */
				if (P.visimap && !(rnull & 1) && !((P.visimap[ridx[0] >> 3] >> (ridx[0] & 7)) & 1))
					alive = false;
			}
		}
		else
		{
			/* pop the newest `navail` entries of the queue feeding this stage */
			uint32_t   *q = myq + P.q_off[stage - 1];
			const int	ew = P.q_ew[stage - 1];
			const int	first = qcnt[stage - 1] - navail;

			alive = lane < navail;
			if (alive)
			{
				const uint32_t *e = q + (size_t) (first + lane) * ew;

				for (int s = 0; s < ew - 1; s++)
					ridx[s] = e[s];
				rnull = e[ew - 1];
			}
			qcnt[stage - 1] = first;
			__syncwarp();
		}

		/* ---- run the stage's ops ---- */
		const int	pc_end = P.stage_pc[stage + 1];

		for (int pc = P.stage_pc[stage]; pc < pc_end; pc++)
		{
			if (!__any_sync(0xffffffffu, alive))
				break;
			const int	code = P.ops[pc].code;
			const int	a = P.ops[pc].a;

			if (code == CBP_END)
				break;
			if (code == XOP_FILTER_COL)
			{
				/* fused LOAD col; CONST v; CMP; FILTER */
				bool		isn;
				int64_t		x = gen_load_col(P, a & 0xffff, ridx, rnull, alive, &isn);
				int64_t		y = P.ops[pc].imm;
				bool		r;

				switch (a >> 16)
				{
					case CBP_EQ: r = x == y; break;
					case CBP_NE: r = x != y; break;
					case CBP_LT: r = x < y; break;
					case CBP_LE: r = x <= y; break;
					case CBP_GT: r = x > y; break;
					default: r = x >= y; break;
				}
				if (isn || !r)
					alive = false;
				continue;
			}
			if (code == XOP_MULCSUB)
			{
				/* fused LOAD a; CONST k; LOAD b; SUB; MUL  ->  a * (k - b), overflow refused */
				bool		an,
							bn;
				int64_t		x = gen_load_col(P, a & 0xffff, ridx, rnull, alive, &an);
				int64_t		b = gen_load_col(P, a >> 16, ridx, rnull, alive, &bn);
				bool		ovf_sub,
							ovf_mul;
				const int64_t r = i64_mul_ovf(x, i64_sub_ovf(P.ops[pc].imm, b, &ovf_sub), &ovf_mul);

				if (alive && !an && !bn && (ovf_sub || ovf_mul))
					atomicExch(P.status, CBGPU_ERR_OVERFLOW);
				st[sp] = r;
				snull = (an || bn) ? (snull | (1ull << sp)) : (snull & ~(1ull << sp));
				sp++;
				continue;
			}
			if (code == CBP_PROBE || code == XOP_PROBE_COLS)
			{
				const DProbe &pr = P.probes[a];
				uint32_t	h = 0;
				bool		knull = false;
				int64_t		key[CBP_MAX_KEYS];
				bool		found = false;
				uint32_t	irow = 0;

				if (code == CBP_PROBE)
				{
					sp -= pr.nkeys;
					for (int k = 0; k < pr.nkeys; k++)
					{
						key[k] = st[sp + k];
						if ((snull >> (sp + k)) & 1)
							knull = true;
					}
					snull &= (1ull << sp) - 1;
				}
				else
				{
					/* fused LOAD key columns; PROBE: the column indexes ride in imm, 8 bits each */
					const uint64_t kc = (uint64_t) P.ops[pc].imm;

					for (int k = 0; k < pr.nkeys; k++)
					{
						bool		isn;

						key[k] = gen_load_col(P, (int) ((kc >> (8 * k)) & 0xff), ridx, rnull, alive, &isn);
						if (isn)
							knull = true;
					}
				}
				for (int k = 0; k < pr.nkeys; k++)
					h = jh_key_fold(h, pr.keytype[k], key[k], pr.keydict[k]);
				if (knull && pr.null_key_drops)
					alive = false;		/* NOT IN over a non-empty set: NULL <> everything is unknown, the row goes */
				bool		maybe = alive && !knull;

				if (maybe && pr.ht.bloom)
				{
					/* runtime Bloom filter first: it is L2-resident, the table is not */
					uint32_t	w;
					uint32_t	bits = ht_bloom_bits(h, &w, pr.ht.bloom_mask);

					maybe = (__ldg(pr.ht.bloom + w) & bits) == bits;
				}
				if (alive && pr.ht.nbatch > 1 &&
					(knull ? pr.ht.batch_id != 0 : !ht_in_batch(pr.ht.nbatch, pr.ht.batch_shift, pr.ht.batch_id, h)))
				{
					/* multi-batch join: this row's batch is not resident - its own pass joins (or, for outer / anti joins,
					 * emits) it; in this pass it does not exist.  A NULL key hashes to 0 in the reference (ExecHashGetHashValue
					 * keep_nulls, nodeHash.c:2171-2190), i.e. belongs to batch 0 */
					alive = false;
					maybe = false;
				}
				if (maybe && pr.ht.keyslot && !ht_key_in_domain(pr.ht.keyslot, key[0]))
					maybe = false;		/* outside the build side's key domain: no partner */
				if (maybe)
				{
					/* ht_find's walk written out (through ht_find or ht_slot_match, ptxas gives this kernel more stack and spills) */
					uint32_t	pos = h & pr.ht.mask;
					unsigned long long e = pr.ht.slots[pos];
					const uint32_t tag = ht_probe_tag(pr.ht.keyslot, h, key[0]);

					while (!ht_slot_empty(e))
					{
						if (ht_tag_match(e, tag))
						{
							bool		eq = true;

							irow = ht_slot_row(e);
							for (int k = 0; k < pr.nkeys && !pr.ht.keyslot; k++)
								if (cb_load_widen(pr.ht.keydata[k], pr.ht.keytype[k], irow) != key[k])
									eq = false;
							if (eq)
							{
								found = true;
								break;
							}
						}
						pos = (pos + 1) & pr.ht.mask;
						e = pr.ht.slots[pos];
					}
				}
				/* join-type handling of the probe states (nodeHashjoin.c:583-713) */
				switch (pr.jointype)
				{
					case CB_JOIN_INNER:
					case CB_JOIN_SEMI:
						if (!found)
							alive = false;
						break;
					case CB_JOIN_ANTI:
						if (found)
							alive = false;
						break;
					case CB_JOIN_LEFT:
						if (!found)
							rnull |= 1u << (P.src_base + a);
						break;
				}
				ridx[P.src_base + a] = irow;
				continue;
			}
			switch (code)
			{
				case CBP_LOAD:
					{
						const CbpColumn &c = P.cols[a];
						bool		isnull = (rnull >> c.src) & 1;
						int64_t		v = 0;

						if (alive && !isnull)
						{
							uint32_t	r = ridx[c.src];

							if (c.nulls && c.nulls[r])
								isnull = true;
							else
								v = cb_load_widen(c.data, c.type, r);
						}
						st[sp] = v;
						snull = isnull ? (snull | (1ull << sp)) : (snull & ~(1ull << sp));
						sp++;
						break;
					}
				case CBP_FILTER:
					sp--;
					/* ExecQual: NULL counts as false */
					if (((snull >> sp) & 1) || !st[sp])
						alive = false;
					snull &= ~(1ull << sp);
					break;
				case CBP_INSET:
					{
						/* a NULL code stays NULL (its bit keeps the stack slot's NULL flag) */
						const CbpSet &set = P.sets[a];
						const int64_t v = st[sp - 1];

						st[sp - 1] = alive && v >= 0 && v < set.nbits && ((set.bits[v >> 5] >> (v & 31)) & 1);
						break;
					}
				default:
					cbp_scalar_op(P.ops[pc], st, snull, sp, alive, P.status);
					break;
			}
		}

		if (stage < nq)
		{
			/* survivors wait in the next queue (there is room: it held < 32 entries) */
			uint32_t   *q = myq + P.q_off[stage];
			const int	ew = P.q_ew[stage];
			const uint32_t m = __ballot_sync(0xffffffffu, alive);

			if (alive)
			{
				uint32_t   *e = q + (size_t) (qcnt[stage] + __popc(m & ((1u << lane) - 1))) * ew;

				for (int s = 0; s < ew - 1; s++)
					e[s] = ridx[s];
				e[ew - 1] = rnull;
			}
			qcnt[stage] += __popc(m);
			__syncwarp();
			continue;
		}
		/* ---- sink ---- */
		const DSink &S = P.sink;

		if (S.kind == CBP_SINK_AGG)
		{
			if (alive)
			{
				const uint32_t knull = (uint32_t) (snull & ((1ull << S.nkeys) - 1));

				for (int k = 0; k < S.nkeys; k++)
					st[k] = ((knull >> k) & 1) ? 0 : agg_group_key(S.keytype[k], st[k]);
				const uint32_t h = agg_group_hash(S.nkeys, S.keytype, S.keydict, st, knull);

				/* partitioned aggregation: this pass owns the groups whose hash carries its number */
				int			slot = (S.agg.npart > 1 && (int32_t) (h >> S.agg.part_shift) != S.agg.part_id) ? -1 : agg_find_or_insert(S.agg, h, st, knull);

				if (slot >= 0)
					for (int a = 0; a < S.naccs; a++)
						sink_acc_update(S.agg, slot, a, S.accs[a], st + S.nkeys, snull >> S.nkeys);
			}
		}
		else
		{
			/* one output position per surviving row; positions handed out per warp and per
			 * destination so the counters see one atomic per (warp, destination) */
			const SinkOut &O = S.out;
			const int	seg = S.kind == CBP_SINK_PARTITION && alive ? cdb_route(O.nhash, O.hashtype, O.hashdict, st, (uint32_t) snull, O.nsegs) : 0;
			const uint32_t amask = __ballot_sync(0xffffffffu, alive);

			if (alive)
			{
				const uint32_t peers = __match_any_sync(amask, seg);
				const int	leader = __ffs(peers) - 1;
				unsigned long long pos = 0;

				if (lane == leader)
					pos = sink_reserve(O, seg, __popc(peers), P.status);
				pos = __shfl_sync(peers, pos, leader) + __popc(peers & ((1u << lane) - 1));
				sink_put_row(O, seg, pos, [&](int c) { return st[c]; }, snull, P.status);
			}
		}
	}
}

extern "C" int
cbgpu_pipeline_run(cbgpu_ctx *ctx, const CbPipeline *p)
{
	PipeDev    *dp = (PipeDev *) cb_scratch(ctx, 1, sizeof(PipeDev));	/* large: off the stack, per context (re-entrant) */
	XProg	   *xp = (XProg *) cb_scratch(ctx, 2, sizeof(XProg));
	if (!dp || !xp)
		return CBGPU_ERR_NOMEM;
	PipeDev    &d = *dp;
	int			rc = cb_pipeline_to_dev(ctx, p, &d, xp);
	bool		handled = false;

	if (rc)
		return rc;
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	{
		/* an earlier asynchronous failure must not be blamed on (or hidden by) this launch */
		cudaError_t stale = cudaGetLastError();

		if (stale != cudaSuccess)
			return cb_fail(ctx, CBGPU_ERR_CUDA, "CUDA error pending before the pipeline launch: %s", cudaGetErrorString(stale));
	}
	ctx->kernel_timed = false;
	if (p->nrows == 0)
		return CBGPU_OK;
	bool		multibatch = false;

	for (int j = 0; j < p->nprobes; j++)
		if (p->probes[j].ht && p->probes[j].ht->d.nbatch > 1)
			multibatch = true;	/* the compiled kernels know nothing of batches: the interpreter runs the passes */
	if (p->sink.kind == CBP_SINK_AGG && p->sink.agg && p->sink.agg->d.npart > 1)
		multibatch = true;		/* ... nor of aggregate partitions */
	if (!p->force_generic && !multibatch)
	{
		rc = cb_try_specialised(ctx, p, &d, xp, &handled);
		if (rc)
			return rc;
	}
	if (!handled)
	{
		int64_t		warps = (p->nrows + 31) / 32;
		int64_t		blocks = (warps + 7) / 8;
		size_t		smem = (size_t) (GEN_THREADS / 32) * (size_t) d.q_words * sizeof(uint32_t);
		static bool attr_done = false;

		if (blocks > (int64_t) ctx->sm_count * 8)
			blocks = (int64_t) ctx->sm_count * 8;
		if (!attr_done)
		{
			CB_CUDA(ctx, cudaFuncSetAttribute(k_pipeline_generic, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024));
			attr_done = true;
		}
		CB_CUDA(ctx, cudaEventRecord(ctx->ev_k0, ctx->stream));
		int			kl = cb_klog_begin(ctx, "k_pipeline_generic");

		k_pipeline_generic<<<(int) blocks, GEN_THREADS, smem, ctx->stream>>>(d);
		CB_LAUNCHED(ctx, "k_pipeline_generic");
		cb_klog_end(ctx, kl);
		CB_CUDA(ctx, cudaEventRecord(ctx->ev_k1, ctx->stream));
		ctx->kernel_timed = true;
		ctx->last_kernel_name = "k_pipeline_generic";
	}
	return CBGPU_OK;
}
