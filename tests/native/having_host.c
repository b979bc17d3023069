/*
 * having_host.c - cloudberry_b200/csrc/having_eval.cuh (the evaluator k_having_eval runs) compiled for the host, for
 * tests/test_having_host.py.  Reads cases from stdin: int32 count, then per case int32 ncols, int32 nops; per column int32
 * width, uint8 null, int64 value (one group); per op int32 code, int32 a, int64 imm.  Writes hv_program's uint64 result per
 * case to stdout.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../cloudberry_b200/csrc/having_eval.cuh"

static int
read_exact(void *buf, size_t n)
{
	return fread(buf, 1, n, stdin) == n;
}

int
main(void)
{
	int32_t		count;

	if (!read_exact(&count, 4))
		return 2;
	for (int32_t i = 0; i < count; i++)
	{
		int32_t		hdr[2];
		HvCols		cols;
		CbpOp	   *ops;
		uint64_t	r;

		if (!read_exact(hdr, sizeof(hdr)) || hdr[0] < 0 || hdr[0] > HV_MAX_COLS || hdr[1] < 1)
			return 2;
		memset(&cols, 0, sizeof(cols));
		for (int c = 0; c < hdr[0]; c++)
		{
			int32_t		w;
			uint8_t		null;
			int64_t		v;

			if (!read_exact(&w, 4) || !read_exact(&null, 1) || !read_exact(&v, 8) || (w != 1 && w != 4 && w != 8))
				return 2;
			/* exact-size buffers, so that a read past either end is seen by AddressSanitizer */
			void	   *d = malloc((size_t) w);
			uint8_t    *n = malloc(1);

			if (!d || !n)
				return 2;
			if (w == 1)
				*(uint8_t *) d = (uint8_t) v;
			else if (w == 4)
				*(int32_t *) d = (int32_t) v;
			else
				*(int64_t *) d = v;
			*n = null;
			cols.data[c] = d;
			cols.nulls[c] = n;
			cols.width[c] = w;
		}
		ops = malloc(sizeof(CbpOp) * (size_t) hdr[1]);
		if (!ops)
			return 2;
		for (int k = 0; k < hdr[1]; k++)
			if (!read_exact(&ops[k].code, 4) || !read_exact(&ops[k].a, 4) || !read_exact(&ops[k].imm, 8))
				return 2;
		r = hv_program(ops, hdr[1], &cols, 0);
		fwrite(&r, sizeof(r), 1, stdout);
		for (int c = 0; c < hdr[0]; c++)
		{
			free((void *) cols.data[c]);
			free((void *) cols.nulls[c]);
		}
		free(ops);
	}
	return 0;
}
