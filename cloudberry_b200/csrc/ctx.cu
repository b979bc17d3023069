/*
 * ctx.cu - context, HBM-resident relations, timing helpers.
 *
 * A relation here is the decoded, projected form of an AOCS table: what aocs_beginscan
 * (backend/access/aocs/aocsam.c:549) + the datum-stream block cursor (include/utils/
 * datumstreamblock.h:1220-1614) hand the executor one Datum at a time, laid out instead as one
 * contiguous fixed-width array per projected column (DESIGN.md "data layout in HBM").
 */
#include "common.cuh"

#include <nvtx3/nvToolsExt.h>

#include <stdlib.h>

extern "C" int
cbgpu_device_count(void)
{
	int			n = 0;

	if (cudaGetDeviceCount(&n) != cudaSuccess)
		return 0;
	return n;
}

/* why this thread's last cbgpu_ctx_create failed: cbgpu_last_error(NULL) */
static thread_local char create_err[sizeof(((cbgpu_ctx *) 0)->err)];

static void
ctx_create_failed(cbgpu_ctx *ctx)
{
	memcpy(create_err, ctx->err, sizeof(create_err));
	cbgpu_ctx_destroy(ctx);
}

extern "C" int
cbgpu_ctx_create(int device, cbgpu_ctx **out)
{
	CbOwned<cbgpu_ctx> owned((cbgpu_ctx *) calloc(1, sizeof(cbgpu_ctx)), ctx_create_failed);
	cbgpu_ctx  *ctx = owned.get();
	cudaDeviceProp prop;

	*out = NULL;
	if (!ctx)
	{
		snprintf(create_err, sizeof(create_err), "cbgpu_ctx_create: out of host memory");
		return CBGPU_ERR_NOMEM;
	}
	ctx->device = device;
	CB_CUDA(ctx, cudaSetDevice(device));
	CB_CUDA(ctx, cudaGetDeviceProperties(&prop, device));
	ctx->sm_count = prop.multiProcessorCount;
	CB_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
	{
		/* every device allocation of the library is stream-ordered (cudaMallocAsync); keep freed
		 * blocks cached in the pool so per-query hash tables / result buffers cost no driver call */
		cudaMemPool_t pool;
		unsigned long long keep = ~0ull;

		CB_CUDA(ctx, cudaDeviceGetDefaultMemPool(&pool, device));
		CB_CUDA(ctx, cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
	}
	CB_CUDA(ctx, cudaEventCreate(&ctx->ev_t0));
	CB_CUDA(ctx, cudaEventCreate(&ctx->ev_t1));
	CB_CUDA(ctx, cudaEventCreate(&ctx->ev_k0));
	CB_CUDA(ctx, cudaEventCreate(&ctx->ev_k1));
	CB_CUDA(ctx, cudaMalloc(&ctx->d_status, sizeof(int)));
	CB_CUDA(ctx, cudaMemsetAsync(ctx->d_status, 0, sizeof(int), ctx->stream));
	CB_CUDA(ctx, cudaMallocHost(&ctx->h_status, sizeof(int)));
	*ctx->h_status = 0;
	CB_CUDA(ctx, cudaMallocHost(&ctx->agg_snap, sizeof(AggSnap)));
	memset(ctx->agg_snap, 0, sizeof(AggSnap));
	ctx->opt_debug = getenv("CBGPU_DEBUG") != NULL;
	ctx->opt_pf_spec = getenv("CBGPU_PF_SPEC") != NULL;
	ctx->opt_pf_keep_div = getenv("CBGPU_PREFILTER_KEEP_DIV") && atoi(getenv("CBGPU_PREFILTER_KEEP_DIV")) > 0 ? atoi(getenv("CBGPU_PREFILTER_KEEP_DIV")) : 12;
	ctx->opt_pf_min_rows = getenv("CBGPU_PREFILTER_MIN_ROWS") ? atoll(getenv("CBGPU_PREFILTER_MIN_ROWS")) : ((int64_t) 16 << 20);
	ctx->opt_bloom_div = getenv("CBGPU_BLOOM_DIV") && atoi(getenv("CBGPU_BLOOM_DIV")) > 0 ? atoi(getenv("CBGPU_BLOOM_DIV")) : 2;
	/* L2 is 50 MB on H100: flush buffer comfortably larger */
	ctx->flush_bytes = (size_t) 512 << 20;
	ctx->flush_buf = NULL;
	*out = owned.release();
	return CBGPU_OK;
}

extern "C" void
cbgpu_ctx_destroy(cbgpu_ctx *ctx)
{
	if (!ctx)
		return;
	cudaEvent_t ev[] = {ctx->ev_t0, ctx->ev_t1, ctx->ev_k0, ctx->ev_k1};

	cudaSetDevice(ctx->device);
	if (ctx->stream)
		cudaStreamSynchronize(ctx->stream);
	if (ctx->flush_buf)
		cudaFree(ctx->flush_buf);
	if (ctx->d_status)
		cudaFree(ctx->d_status);
	if (ctx->h_status)
		cudaFreeHost(ctx->h_status);
	if (ctx->agg_snap)
		cudaFreeHost(ctx->agg_snap);
	if (ctx->small_dev)
		cudaFree(ctx->small_dev);
	for (int i = 0; i < CB_SCRATCH_SLOTS; i++)
		free(ctx->scratch[i]);
	for (int i = 0; i < 4; i++)
		if (ev[i])
			cudaEventDestroy(ev[i]);
	if (ctx->stream)
		cudaStreamDestroy(ctx->stream);
	free(ctx);
}

extern "C" const char *
cbgpu_last_error(cbgpu_ctx *ctx)
{
	return ctx ? ctx->err : create_err[0] ? create_err : "no context";
}

extern "C" void
cbgpu_range_push(const char *name)
{
	nvtxRangePushA(name);
}

extern "C" void
cbgpu_range_pop(void)
{
	nvtxRangePop();
}

extern "C" int
cbgpu_sync(cbgpu_ctx *ctx)
{
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return CBGPU_OK;
}

int
cb_check_status(cbgpu_ctx *ctx, const char *what)
{
	if (ctx->status_seen_at != ctx->launches)
	{
		/* no read-back has fetched the word since the last launch: do it now */
		CB_CUDA(ctx, CB_STATUS_RIDE(ctx));
		CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		CB_STATUS_FETCHED(ctx);
	}
	if (*ctx->h_status != 0)
	{
		int			code = *ctx->h_status;

		CB_CUDA(ctx, cudaMemsetAsync(ctx->d_status, 0, sizeof(int), ctx->stream));
		*ctx->h_status = 0;
		snprintf(ctx->err, sizeof(ctx->err), "%s: %s", what,
				 code == CBGPU_ERR_OVERFLOW ? "value out of range (integer/numeric overflow)" :
				 code == CBGPU_ERR_NOMEM ? "device table or output buffer full" :
				 code == CBGPU_ERR_CORRUPT ? "stored block fails its checksum" :
				 code == CBGPU_ERR_PEER ? "a peer segment did not signal within the interconnect's time limit" : "device-side error");
		if (code > 0 || code < CBGPU_ERR_INTERRUPTED)
		{
			/* kernels only ever store one of the library's codes: anything else means the word itself was damaged */
			snprintf(ctx->err, sizeof(ctx->err), "%s: device status word holds %d, not an error code of this library", what, code);
			return CBGPU_ERR_CUDA;
		}
		return code;
	}
	return CBGPU_OK;
}

extern "C" int
cbgpu_check_status(cbgpu_ctx *ctx)
{
	return cb_check_status(ctx, "GPU pipeline");
}

extern "C" int
cbgpu_sm_count(cbgpu_ctx *ctx)
{
	return ctx->sm_count;
}

extern "C" int64_t
cbgpu_kernel_launches(cbgpu_ctx *ctx)
{
	return ctx->launches;
}

extern "C" int
cbgpu_timer_start(cbgpu_ctx *ctx)
{
	CB_CUDA(ctx, cudaEventRecord(ctx->ev_t0, ctx->stream));
	return CBGPU_OK;
}

extern "C" int
cbgpu_timer_stop_ms(cbgpu_ctx *ctx, double *ms)
{
	float		f = 0;

	CB_CUDA(ctx, cudaEventRecord(ctx->ev_t1, ctx->stream));
	CB_CUDA(ctx, cudaEventSynchronize(ctx->ev_t1));
	CB_CUDA(ctx, cudaEventElapsedTime(&f, ctx->ev_t0, ctx->ev_t1));
	*ms = f;
	return CBGPU_OK;
}

extern "C" double
cbgpu_last_kernel_ms(cbgpu_ctx *ctx)
{
	float		f = 0;

	if (!ctx->kernel_timed)
		return -1.0;
	if (cudaEventSynchronize(ctx->ev_k1) != cudaSuccess)
		return -1.0;
	if (cudaEventElapsedTime(&f, ctx->ev_k0, ctx->ev_k1) != cudaSuccess)
		return -1.0;
	return f;
}

/* pipeline-kernel log: every pipeline launch brackets itself with its own event pair */
int
cb_klog_begin(cbgpu_ctx *ctx, const char *name)
{
	int			i = ctx->klog_n;

	if (i >= CB_KLOG)
		return -1;
	if (!ctx->klog_ready)
	{
		for (int k = 0; k < CB_KLOG; k++)
		{
			cudaEventCreate(&ctx->klog_ev[k][0]);
			cudaEventCreate(&ctx->klog_ev[k][1]);
		}
		ctx->klog_ready = true;
	}
	ctx->klog_name[i] = name;
	cudaEventRecord(ctx->klog_ev[i][0], ctx->stream);
	ctx->klog_n = i + 1;
	return i;
}

void
cb_klog_end(cbgpu_ctx *ctx, int i)
{
	if (i >= 0)
		cudaEventRecord(ctx->klog_ev[i][1], ctx->stream);
}

/* launch trace: an event after every launch; entry i's time = event i -> event i + 1, i.e. the
 * kernel plus whatever idle gap preceded it on the stream */
void
cb_trace_mark(cbgpu_ctx *ctx, const char *name)
{
	if (ctx->trace_n >= CB_TRACE)
		return;
	ctx->trace_name[ctx->trace_n] = name;
	cudaEventRecord(ctx->trace_ev[ctx->trace_n + 1], ctx->stream);
	ctx->trace_n++;
}

extern "C" int
cbgpu_trace_begin(cbgpu_ctx *ctx)
{
	if (!ctx->trace_ev)
	{
		ctx->trace_ev = (cudaEvent_t *) calloc(CB_TRACE + 1, sizeof(cudaEvent_t));
		if (!ctx->trace_ev)
			return CBGPU_ERR_NOMEM;
		for (int i = 0; i <= CB_TRACE; i++)
			CB_CUDA(ctx, cudaEventCreate(&ctx->trace_ev[i]));
	}
	ctx->trace_n = 0;
	ctx->trace_on = true;
	CB_CUDA(ctx, cudaEventRecord(ctx->trace_ev[0], ctx->stream));
	return CBGPU_OK;
}

extern "C" int
cbgpu_trace_end(cbgpu_ctx *ctx)
{
	ctx->trace_on = false;
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return ctx->trace_n;
}

extern "C" int
cbgpu_trace_get(cbgpu_ctx *ctx, int i, char *name, int namelen, double *ms)
{
	float		f = 0;

	if (i < 0 || i >= ctx->trace_n)
		return CBGPU_ERR_INVALID;
	CB_CUDA(ctx, cudaEventElapsedTime(&f, ctx->trace_ev[i], ctx->trace_ev[i + 1]));
	*ms = f;
	if (name && namelen > 0)
		snprintf(name, (size_t) namelen, "%s", ctx->trace_name[i]);
	return CBGPU_OK;
}

extern "C" void
cbgpu_kernel_log_reset(cbgpu_ctx *ctx)
{
	ctx->klog_n = 0;
}

extern "C" int
cbgpu_kernel_log_longest(cbgpu_ctx *ctx, char *name, int namelen, double *ms)
{
	float		best = -1.f;
	int			bi = -1;

	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	for (int i = 0; i < ctx->klog_n; i++)
	{
		float		f = 0;

		if (cudaEventElapsedTime(&f, ctx->klog_ev[i][0], ctx->klog_ev[i][1]) == cudaSuccess && f > best)
		{
			best = f;
			bi = i;
		}
	}
	*ms = best;
	if (name && namelen > 0)
		snprintf(name, (size_t) namelen, "%s", bi >= 0 ? ctx->klog_name[bi] : "");
	return CBGPU_OK;
}

extern "C" const char *
cbgpu_last_kernel_name(cbgpu_ctx *ctx)
{
	return ctx->last_kernel_name ? ctx->last_kernel_name : "";
}

__global__ void
k_flush_fill(uint4 *p, size_t n, uint32_t v)
{
	size_t		i = (size_t) blockIdx.x * blockDim.x + threadIdx.x;
	size_t		stride = (size_t) gridDim.x * blockDim.x;

	for (; i < n; i += stride)
		p[i] = make_uint4(v, v, v, v);
}

extern "C" int
cbgpu_flush_l2(cbgpu_ctx *ctx)
{
	static uint32_t gen = 0;

	if (!ctx->flush_buf)
		CB_CUDA(ctx, cudaMalloc(&ctx->flush_buf, ctx->flush_bytes));
	k_flush_fill<<<ctx->sm_count * 4, 512, 0, ctx->stream>>>((uint4 *) ctx->flush_buf, ctx->flush_bytes / 16, ++gen);
	CB_LAUNCHED(ctx, "k_flush_fill");
	return CBGPU_OK;
}

extern "C" void *
cbgpu_host_alloc(size_t bytes)
{
	void	   *p = NULL;

	if (cudaMallocHost(&p, bytes ? bytes : 1) != cudaSuccess)
		return NULL;
	return p;
}

extern "C" void
cbgpu_host_free(void *p)
{
	if (p)
		cudaFreeHost(p);
}

extern "C" uint32_t
cbgpu_hashbpchar(const char *s, int32_t len)
{
	/* bcTruelen (utils/adt/varchar.c:704): ignore trailing blanks */
	while (len > 0 && s[len - 1] == ' ')
		len--;
	return pg_hash_bytes_host((const unsigned char *) s, len);
}

/* ---------------------------------------------------------------------------------------------
 * relations
 * --------------------------------------------------------------------------------------------- */
extern "C" int
cbgpu_rel_create(cbgpu_ctx *ctx, int64_t nrows, int32_t ncols, const int32_t *types, const int32_t *dscales,
				 cbgpu_rel **out)
{
	*out = NULL;
	if (ncols < 0 || ncols > CB_MAX_COLS_REL || nrows < 0 || nrows > 0xFFFFFFF0ll)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_create: bad shape (%s nrows=%lld)", "", nrows);
	CbOwned<cbgpu_rel> r((cbgpu_rel *) calloc(1, sizeof(cbgpu_rel)), cbgpu_rel_free);

	if (!r)
		return CBGPU_ERR_NOMEM;
	r->ctx = ctx;
	r->nrows = nrows;
	r->capacity = nrows;
	r->ncols = ncols;
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	size_t		total = 0;
	size_t		colbytes[CB_MAX_COLS_REL];

	for (int i = 0; i < ncols; i++)
	{
		size_t		bytes = (size_t) (nrows ? nrows : 1) * cb_type_w(types[i]);

		if (cb_type_w(types[i]) == 0)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_create: bad column type%s %lld", "", types[i]);
		r->types[i] = types[i];
		r->dscales[i] = dscales ? dscales[i] : 0;
		/* pad so 16-byte vector loads and TMA bulk copies may read a whole final vector */
		colbytes[i] = (bytes + 255) & ~(size_t) 255;
		total += colbytes[i];
	}
	if (ncols > 1 && total <= ((size_t) 64 << 20))
	{
		/* intermediate results (group relations, Motion buffers of a few rows) are created per query with dozens of
		 * columns: one pool call instead of one per column */
		char	   *base;

		CB_CUDA(ctx, cudaMallocAsync(&base, total, ctx->stream));
		r->slab = base;
		for (int i = 0; i < ncols; i++)
		{
			r->data[i] = base;
			r->owns[i] = false;
			base += colbytes[i];
		}
	}
	else
		for (int i = 0; i < ncols; i++)
		{
			CB_CUDA(ctx, cudaMallocAsync(&r->data[i], colbytes[i], ctx->stream));
			r->owns[i] = true;
		}
	*out = r.release();
	return CBGPU_OK;
}

extern "C" void
cbgpu_rel_free(cbgpu_rel *rel)
{
	if (!rel)
		return;
	/* stream-ordered frees: memory returns to the context's pool once the work queued before this
	 * point has drained; no host synchronisation */
	cudaSetDevice(rel->ctx->device);
	for (int i = 0; i < rel->ncols; i++)
	{
		if (rel->owns[i] && rel->data[i])
			cudaFreeAsync(rel->data[i], rel->ctx->stream);
		if (rel->nulls[i])
			cudaFreeAsync(rel->nulls[i], rel->ctx->stream);
		if (rel->dict_hash[i] && rel->dict_n[i] >= 0)
			cudaFreeAsync(rel->dict_hash[i], rel->ctx->stream);
	}
	if (rel->visimap)
		cudaFreeAsync(rel->visimap, rel->ctx->stream);
	if (rel->slab)
		cudaFreeAsync(rel->slab, rel->ctx->stream);
	free(rel);
}

extern "C" int64_t
cbgpu_rel_nrows(const cbgpu_rel *rel)
{
	return rel->nrows;
}

extern "C" int32_t
cbgpu_rel_ncols(const cbgpu_rel *rel)
{
	return rel->ncols;
}

extern "C" int32_t
cbgpu_rel_col_type(const cbgpu_rel *rel, int32_t col)
{
	return (col >= 0 && col < rel->ncols) ? rel->types[col] : 0;
}

extern "C" int32_t
cbgpu_rel_col_dscale(const cbgpu_rel *rel, int32_t col)
{
	return (col >= 0 && col < rel->ncols) ? rel->dscales[col] : 0;
}

extern "C" int
cbgpu_rel_load_column(cbgpu_rel *rel, int32_t col, const void *host, const uint8_t *nulls)
{
	cbgpu_ctx  *ctx = rel->ctx;

	if (col < 0 || col >= rel->ncols)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_load_column: bad column%s %lld", "", col);
	if (rel->nrows == 0)
		return CBGPU_OK;
	CB_CUDA(ctx, cudaMemcpyAsync(rel->data[col], host, (size_t) rel->nrows * cb_type_w(rel->types[col]),
								 cudaMemcpyHostToDevice, ctx->stream));
	if (nulls)
	{
		if (!rel->nulls[col])
			CB_CUDA(ctx, cudaMallocAsync(&rel->nulls[col], (size_t) rel->capacity, ctx->stream));
		CB_CUDA(ctx, cudaMemcpyAsync(rel->nulls[col], nulls, (size_t) rel->nrows, cudaMemcpyHostToDevice, ctx->stream));
	}
	else if (rel->nulls[col])
	{
		cudaFreeAsync(rel->nulls[col], ctx->stream);
		rel->nulls[col] = NULL;
	}
	return CBGPU_OK;
}

/* host columns shipped in a narrower integer width than the column's own (PCIe is the bottleneck of a load: a
 * numeric(15,2) whose values fit 16 bits travels as int16) and sign-extended on the device */
template <typename NARROW, typename WIDE>
__global__ void
k_widen(const NARROW *__restrict__ src, WIDE *__restrict__ dst, int64_t n)
{
	int64_t		i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
	const int64_t stride = (int64_t) gridDim.x * blockDim.x;

	for (; i < n; i += stride)
		dst[i] = (WIDE) src[i];
}

extern "C" int
cbgpu_rel_load_column_narrow(cbgpu_rel *rel, int32_t col, const void *host, int32_t host_width)
{
	cbgpu_ctx  *ctx = rel->ctx;
	CbCallMem	mem(ctx);
	void	   *stage;
	int			w;
	int			blocks;

	if (col < 0 || col >= rel->ncols)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_load_column_narrow: bad column%s %lld", "", col);
	w = cb_type_w(rel->types[col]);
	if (host_width == w)
		return cbgpu_rel_load_column(rel, col, host, NULL);
	if (rel->types[col] == CB_FLOAT8 || (w != 8 && w != 4) || (host_width != 1 && host_width != 2 && host_width != 4) || host_width > w)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_load_column_narrow: a %s%lld-byte host column cannot be widened into this column", "", host_width);
	if (rel->nrows == 0)
		return CBGPU_OK;
	CB_CUDA(ctx, mem.alloc(&stage, (size_t) rel->nrows * host_width));
	CB_CUDA(ctx, cudaMemcpyAsync(stage, host, (size_t) rel->nrows * host_width, cudaMemcpyHostToDevice, ctx->stream));
	blocks = ctx->sm_count * 8;
	if (w == 8)
	{
		if (host_width == 1)
			k_widen<int8_t, int64_t><<<blocks, 256, 0, ctx->stream>>>((const int8_t *) stage, (int64_t *) rel->data[col], rel->nrows);
		else if (host_width == 2)
			k_widen<int16_t, int64_t><<<blocks, 256, 0, ctx->stream>>>((const int16_t *) stage, (int64_t *) rel->data[col], rel->nrows);
		else
			k_widen<int32_t, int64_t><<<blocks, 256, 0, ctx->stream>>>((const int32_t *) stage, (int64_t *) rel->data[col], rel->nrows);
	}
	else
	{
		if (host_width == 1)
			k_widen<int8_t, int32_t><<<blocks, 256, 0, ctx->stream>>>((const int8_t *) stage, (int32_t *) rel->data[col], rel->nrows);
		else
			k_widen<int16_t, int32_t><<<blocks, 256, 0, ctx->stream>>>((const int16_t *) stage, (int32_t *) rel->data[col], rel->nrows);
	}
	CB_LAUNCHED(ctx, "k_widen");
	return CBGPU_OK;
}

extern "C" int
cbgpu_rel_read_column(cbgpu_rel *rel, int32_t col, int64_t lo, int64_t hi, void *host, uint8_t *nulls)
{
	cbgpu_ctx  *ctx = rel->ctx;
	int			w;

	if (col < 0 || col >= rel->ncols || lo < 0 || hi > rel->nrows || lo > hi)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_read_column: bad range%s %lld", "", lo);
	w = cb_type_w(rel->types[col]);
	if (hi > lo)
	{
		CB_CUDA(ctx, cudaMemcpyAsync(host, (char *) rel->data[col] + (size_t) lo * w, (size_t) (hi - lo) * w,
									 cudaMemcpyDeviceToHost, ctx->stream));
		if (nulls)
		{
			if (rel->nulls[col])
				CB_CUDA(ctx, cudaMemcpyAsync(nulls, rel->nulls[col] + lo, (size_t) (hi - lo), cudaMemcpyDeviceToHost, ctx->stream));
			else
				memset(nulls, 0, (size_t) (hi - lo));
		}
	}
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return CBGPU_OK;
}

/* a few rows of every column in ONE round trip: result sets above an aggregate or a top-N are a handful of
 * rows, and one synchronising copy per row and column is what their delivery would otherwise cost */
struct ReadRows
{
	const void *data[CB_MAX_COLS_REL];
	const uint8_t *nulls[CB_MAX_COLS_REL];
	int32_t		types[CB_MAX_COLS_REL];
	int32_t		ncols;
	const uint32_t *idx;
	int64_t		n;
	long long  *out;
	uint8_t    *outnull;
};

__global__ void
k_read_rows(ReadRows p)
{
	const int64_t total = p.n * p.ncols;

	for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t) gridDim.x * blockDim.x)
	{
		const int64_t r = i / p.ncols;
		const int	c = (int) (i % p.ncols);
		const uint32_t row = p.idx ? p.idx[r] : (uint32_t) r;

		p.out[i] = cb_load_widen(p.data[c], p.types[c], row);
		p.outnull[i] = p.nulls[c] ? p.nulls[c][row] : (uint8_t) 0;
	}
}

extern "C" int
cbgpu_rel_read_rows(cbgpu_rel *rel, const uint32_t *host_idx, int64_t n, int64_t *out, uint8_t *outnull)
{
	cbgpu_ctx  *ctx = rel->ctx;
	CbCallMem	mem(ctx);
	ReadRows	p;
	uint32_t   *d_idx = NULL;
	char	   *d_buf = NULL;
	const int64_t total = n * rel->ncols;

	if (n < 0 || (!host_idx && n > rel->nrows) || rel->ncols > CB_MAX_COLS_REL)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_read_rows: bad row count%s %lld", "", n);
	if (total == 0)
		return CBGPU_OK;
	for (int64_t r = 0; host_idx && r < n; r++)
		if ((int64_t) host_idx[r] >= rel->nrows)
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_read_rows: row %s%lld out of range", "", (long long) host_idx[r]);
	memset(&p, 0, sizeof(p));
	for (int c = 0; c < rel->ncols; c++)
	{
		p.data[c] = rel->data[c];
		p.nulls[c] = rel->nulls[c];
		p.types[c] = rel->types[c];
	}
	p.ncols = rel->ncols;
	p.n = n;
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	CB_CUDA(ctx, mem.alloc(&d_buf, (size_t) total * 9));
	p.out = (long long *) d_buf;
	p.outnull = (uint8_t *) (d_buf + (size_t) total * 8);
	if (host_idx)
	{
		CB_CUDA(ctx, mem.alloc(&d_idx, (size_t) n * sizeof(uint32_t)));
		CB_CUDA(ctx, mem.copy_in(d_idx, host_idx, (size_t) n * sizeof(uint32_t)));
		p.idx = d_idx;
	}
	{
		int			blocks = (int) ((total + 255) / 256);

		if (blocks > ctx->sm_count * 8)
			blocks = ctx->sm_count * 8;
		k_read_rows<<<blocks, 256, 0, ctx->stream>>>(p);
		CB_LAUNCHED(ctx, "k_read_rows");
	}
	CB_CUDA(ctx, cudaMemcpyAsync(out, p.out, (size_t) total * 8, cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaMemcpyAsync(outnull, p.outnull, (size_t) total, cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, CB_STATUS_RIDE(ctx));
	CB_CUDA(ctx, mem.sync());
	CB_STATUS_FETCHED(ctx);
	return CBGPU_OK;
}

extern "C" int
cbgpu_rel_set_visimap(cbgpu_rel *rel, const uint8_t *bits)
{
	cbgpu_ctx  *ctx = rel->ctx;
	size_t		bytes = (size_t) ((rel->nrows + 7) / 8);

	if (!bits)
	{
		if (rel->visimap)
		{
			cudaFreeAsync(rel->visimap, ctx->stream);
			rel->visimap = NULL;
		}
		return CBGPU_OK;
	}
	if (!rel->visimap)
		CB_CUDA(ctx, cudaMallocAsync(&rel->visimap, ((bytes + 255) & ~(size_t) 255) + 256, ctx->stream));
	CB_CUDA(ctx, cudaMemcpyAsync(rel->visimap, bits, bytes, cudaMemcpyHostToDevice, ctx->stream));
	return CBGPU_OK;
}

extern "C" int
cbgpu_rel_read_visimap(cbgpu_rel *rel, uint8_t *bits)
{
	cbgpu_ctx  *ctx = rel->ctx;
	const size_t bytes = (size_t) ((rel->nrows + 7) / 8);

	if (!rel->visimap)
	{
		memset(bits, 0xFF, bytes);
		return CBGPU_OK;
	}
	CB_CUDA(ctx, cudaMemcpyAsync(bits, rel->visimap, bytes, cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return CBGPU_OK;
}

extern "C" int
cbgpu_rel_set_dict_hash(cbgpu_rel *rel, int32_t col, const uint32_t *hashes, int32_t n)
{
	cbgpu_ctx  *ctx = rel->ctx;

	if (col < 0 || col >= rel->ncols || n <= 0)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_set_dict_hash: bad argument%s %lld", "", col);
	if (rel->dict_hash[col])
	{
		cudaFreeAsync(rel->dict_hash[col], ctx->stream);
		rel->dict_hash[col] = NULL;
	}
	CB_CUDA(ctx, cudaMallocAsync(&rel->dict_hash[col], (size_t) n * sizeof(uint32_t), ctx->stream));
	CB_CUDA(ctx, cudaMemcpyAsync(rel->dict_hash[col], hashes, (size_t) n * sizeof(uint32_t), cudaMemcpyHostToDevice, ctx->stream));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	rel->dict_n[col] = n;
	return CBGPU_OK;
}

extern "C" int
cbgpu_rel_set_nrows(cbgpu_rel *rel, int64_t nrows)
{
	if (nrows < 0 || nrows > rel->capacity)
		return cb_fail(rel->ctx, CBGPU_ERR_INVALID, "cbgpu_rel_set_nrows: beyond capacity%s %lld", "", nrows);
	rel->nrows = nrows;
	return CBGPU_OK;
}

extern "C" void *
cbgpu_rel_col_devptr(cbgpu_rel *rel, int32_t col)
{
	return (col >= 0 && col < rel->ncols) ? rel->data[col] : NULL;
}

extern "C" size_t
cbgpu_rel_nbytes(const cbgpu_rel *rel)
{
	size_t		b = 0;

	for (int i = 0; i < rel->ncols; i++)
		b += (size_t) rel->nrows * cb_type_w(rel->types[i]);
	return b;
}

extern "C" int
cbgpu_read_u32(cbgpu_ctx *ctx, const uint32_t *dev, int64_t n, uint32_t *host)
{
	if (n > 0)
		CB_CUDA(ctx, cudaMemcpyAsync(host, dev, (size_t) n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return CBGPU_OK;
}

extern "C" int
cbgpu_dev_alloc(cbgpu_ctx *ctx, size_t bytes, void **dev)
{
	CB_CUDA(ctx, cudaSetDevice(ctx->device));
	CB_CUDA(ctx, cudaMallocAsync(dev, bytes ? bytes : 8, ctx->stream));
	CB_CUDA(ctx, cudaMemsetAsync(*dev, 0, bytes ? bytes : 8, ctx->stream));
	return CBGPU_OK;
}

extern "C" int
cbgpu_dev_read(cbgpu_ctx *ctx, const void *dev, size_t bytes, void *host)
{
	CB_CUDA(ctx, cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, ctx->stream));
	CB_CUDA(ctx, CB_STATUS_RIDE(ctx));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	CB_STATUS_FETCHED(ctx);
	return CBGPU_OK;
}

extern "C" int
cbgpu_dev_write(cbgpu_ctx *ctx, void *dev, size_t bytes, const void *host)
{
	CB_CUDA(ctx, cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, ctx->stream));
	CB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return CBGPU_OK;
}

extern "C" void
cbgpu_dev_free(cbgpu_ctx *ctx, void *dev)
{
	if (!dev)
		return;
	cudaSetDevice(ctx->device);
	cudaFreeAsync(dev, ctx->stream);
}

extern "C" int
cbgpu_rel_add_nullmap(cbgpu_rel *rel, int32_t col)
{
	cbgpu_ctx  *ctx = rel->ctx;

	if (col < 0 || col >= rel->ncols)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_add_nullmap: bad column%s %lld", "", col);
	if (rel->nulls[col])
		return CBGPU_OK;
	CB_CUDA(ctx, cudaMallocAsync(&rel->nulls[col], (size_t) (rel->capacity ? rel->capacity : 1), ctx->stream));
	CB_CUDA(ctx, cudaMemsetAsync(rel->nulls[col], 0, (size_t) (rel->capacity ? rel->capacity : 1), ctx->stream));
	return CBGPU_OK;
}

extern "C" int
cbgpu_rel_copy_rows(cbgpu_rel *dst, int64_t dst_lo, cbgpu_rel *src, int64_t src_lo, int64_t n)
{
	cbgpu_ctx  *ctx = dst->ctx;

	if (dst->ncols != src->ncols || dst_lo < 0 || src_lo < 0 || dst_lo + n > dst->capacity || src_lo + n > src->capacity)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_copy_rows: shape / range mismatch%s (%lld rows)", "", n);
	if (n == 0)
		return CBGPU_OK;
	for (int c = 0; c < dst->ncols; c++)
	{
		int			w = cb_type_w(dst->types[c]);

		if (dst->types[c] != src->types[c])
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_copy_rows: column %s%lld type mismatch", "", c);
		CB_CUDA(ctx, cudaMemcpyAsync((char *) dst->data[c] + (size_t) dst_lo * w, (char *) src->data[c] + (size_t) src_lo * w,
									 (size_t) n * w, cudaMemcpyDeviceToDevice, ctx->stream));
		if (src->nulls[c])
		{
			int			rc = cbgpu_rel_add_nullmap(dst, c);

			if (rc)
				return rc;
			CB_CUDA(ctx, cudaMemcpyAsync(dst->nulls[c] + dst_lo, src->nulls[c] + src_lo, (size_t) n, cudaMemcpyDeviceToDevice, ctx->stream));
		}
	}
	return CBGPU_OK;
}

/* dst rows [0, n) = src rows idx[0..n) (device index list), every column and NULL map: an ordered gather (the merged
 * order of a sorted Motion, a selection) */
struct TakeRows
{
	const void *src[CB_MAX_COLS_REL];
	void	   *dst[CB_MAX_COLS_REL];
	const uint8_t *snull[CB_MAX_COLS_REL];
	uint8_t    *dnull[CB_MAX_COLS_REL];
	int32_t		width[CB_MAX_COLS_REL];
	int32_t		ncols;
	int64_t		n;
	const uint32_t *idx;
};

__global__ void
k_take_rows(TakeRows p)
{
	int64_t		i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
	const int64_t stride = (int64_t) gridDim.x * blockDim.x;

	for (; i < p.n; i += stride)
	{
		const uint32_t r = p.idx[i];

		for (int c = 0; c < p.ncols; c++)
		{
			switch (p.width[c])
			{
				case 1: ((uint8_t *) p.dst[c])[i] = ((const uint8_t *) p.src[c])[r]; break;
				case 4: ((uint32_t *) p.dst[c])[i] = ((const uint32_t *) p.src[c])[r]; break;
				case 16: ((uint4 *) p.dst[c])[i] = ((const uint4 *) p.src[c])[r]; break;
				default: ((unsigned long long *) p.dst[c])[i] = ((const unsigned long long *) p.src[c])[r]; break;
			}
			if (p.dnull[c])
				p.dnull[c][i] = p.snull[c][r];
		}
	}
}

extern "C" int
cbgpu_rel_take_rows(cbgpu_rel *dst, cbgpu_rel *src, const uint32_t *dev_idx, int64_t n)
{
	cbgpu_ctx  *ctx = dst->ctx;
	TakeRows	p;

	if (dst->ncols != src->ncols || n < 0 || n > dst->capacity || dst->ncols > CB_MAX_COLS_REL)
		return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_take_rows: shape / range mismatch%s (%lld rows)", "", n);
	if (n == 0)
		return CBGPU_OK;
	memset(&p, 0, sizeof(p));
	for (int c = 0; c < dst->ncols; c++)
	{
		if (dst->types[c] != src->types[c])
			return cb_fail(ctx, CBGPU_ERR_INVALID, "cbgpu_rel_take_rows: column %s%lld type mismatch", "", c);
		if (src->nulls[c])
		{
			int			rc = cbgpu_rel_add_nullmap(dst, c);

			if (rc)
				return rc;
		}
		p.src[c] = src->data[c];
		p.dst[c] = dst->data[c];
		p.snull[c] = src->nulls[c];
		p.dnull[c] = src->nulls[c] ? dst->nulls[c] : NULL;
		p.width[c] = cb_type_w(dst->types[c]);
	}
	p.ncols = dst->ncols;
	p.n = n;
	p.idx = dev_idx;
	{
		int			blocks = (int) ((n + 255) / 256);

		if (blocks > ctx->sm_count * 8)
			blocks = ctx->sm_count * 8;
		k_take_rows<<<blocks, 256, 0, ctx->stream>>>(p);
		CB_LAUNCHED(ctx, "k_take_rows");
	}
	if (dst->nrows < n)
		dst->nrows = n;
	return CBGPU_OK;
}

extern "C" int
cbgpu_rel_has_nulls(const cbgpu_rel *rel, int32_t col)
{
	return (col >= 0 && col < rel->ncols && rel->nulls[col]) ? 1 : 0;
}

extern "C" const uint32_t *
cbgpu_rel_dict_hash_dev(const cbgpu_rel *rel, int32_t col)
{
	return (col >= 0 && col < rel->ncols) ? rel->dict_hash[col] : NULL;
}

extern "C" const uint8_t *
cbgpu_rel_nulls_dev(const cbgpu_rel *rel, int32_t col)
{
	return (col >= 0 && col < rel->ncols) ? rel->nulls[col] : NULL;
}

extern "C" const uint8_t *
cbgpu_rel_visimap_dev(const cbgpu_rel *rel)
{
	return rel->visimap;
}

extern "C" int
cbgpu_rel_share_dict_hash(cbgpu_rel *dst, int32_t dcol, const cbgpu_rel *src, int32_t scol)
{
	if (dcol < 0 || dcol >= dst->ncols || scol < 0 || scol >= src->ncols)
		return cb_fail(dst->ctx, CBGPU_ERR_INVALID, "cbgpu_rel_share_dict_hash: bad column%s %lld", "", dcol);
	dst->dict_hash[dcol] = src->dict_hash[scol];
	/* negative count: borrowed, not freed with dst (the source may itself be a borrower) */
	dst->dict_n[dcol] = src->dict_n[scol] > 0 ? -src->dict_n[scol] : (src->dict_n[scol] < 0 ? src->dict_n[scol] : -1);
	dst->dict[dcol] = src->dict[scol];
	dst->dict_bpchar_len[dcol] = src->dict_bpchar_len[scol];
	return CBGPU_OK;
}

extern "C" int
cbgpu_rel_set_dict(cbgpu_rel *rel, int32_t col, const cbgpu_dict *dict, int32_t bpchar_len)
{
	if (col < 0 || col >= rel->ncols || (rel->types[col] != CB_DICT8 && rel->types[col] != CB_DICT32) || !dict)
		return cb_fail(rel->ctx, CBGPU_ERR_INVALID, "cbgpu_rel_set_dict: bad argument%s %lld", "", col);
	if (cbgpu_dict_is_bpchar(dict) ? bpchar_len < 1 : bpchar_len != 0)
		return cb_fail(rel->ctx, CBGPU_ERR_INVALID, "cbgpu_rel_set_dict: %sbpchar_len %lld does not fit the dictionary (character(n) "
					   "needs n >= 1, varchar / text 0)", "", bpchar_len);
	rel->dict[col] = dict;
	rel->dict_bpchar_len[col] = bpchar_len;
	return CBGPU_OK;
}

extern "C" const cbgpu_dict *
cbgpu_rel_dict(const cbgpu_rel *rel, int32_t col, int32_t *bpchar_len)
{
	if (col < 0 || col >= rel->ncols)
		return NULL;
	if (bpchar_len)
		*bpchar_len = rel->dict_bpchar_len[col];
	return rel->dict[col];
}
