/*
 * like_host.c - cloudberry_b200/csrc/like_match.cuh (the matcher k_dict_like runs) compiled for the host, for
 * tests/test_like_host.py.  Reads cases from stdin: int32 count, then per case int32 text length, int32 bpchar_len (0:
 * varchar / text), int32 pattern length, the text bytes, the pattern bytes.  Writes one byte per case to stdout: '1' match,
 * '0' no match, 'E' a malformed pattern.
 */
#include <stdio.h>
#include <stdlib.h>

#include "../../cloudberry_b200/csrc/like_match.cuh"

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
		int32_t		hdr[3];
		uint8_t    *t,
				   *p;
		int			pad;
		char		r;

		if (!read_exact(hdr, sizeof(hdr)) || hdr[0] < 0 || hdr[2] < 0)
			return 2;
		/* exact-size buffers, so that a read past either end is seen by AddressSanitizer */
		t = malloc(hdr[0] ? (size_t) hdr[0] : 1);
		p = malloc(hdr[2] ? (size_t) hdr[2] : 1);
		if (!t || !p || !read_exact(t, (size_t) hdr[0]) || !read_exact(p, (size_t) hdr[2]))
			return 2;
		pad = hdr[1] > 0 ? hdr[1] - like_utf8_chars(t, hdr[0]) : 0;
		if (pad < 0)
			pad = 0;
		if (like_pattern_check(p, hdr[2]))
			r = 'E';
		else
			r = like_match(t, hdr[0], pad, p, hdr[2]) ? '1' : '0';
		fputc(r, stdout);
		free(t);
		free(p);
	}
	return 0;
}
