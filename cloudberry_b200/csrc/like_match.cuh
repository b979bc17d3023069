/*
 * like_match.cuh - SQL LIKE over one string, as the reference's MatchText (backend/utils/adt/like_match.c) decides it for a
 * UTF-8 server encoding: `%` matches any sequence of characters (the empty one included), `_` exactly one character (1 to 4
 * bytes, the length taken from the lead byte as pg_utf_mblen does), `\` makes the next pattern byte literal, every other
 * byte matches itself.  Case-sensitive, byte-wise.
 *
 * Host and device code: k_dict_like runs it once per dictionary entry, and the CPU tests compile it for the host.
 *
 * The text is `t[0 .. tlen)` followed by `pad` blanks: a character(n) value is stored without its trailing blanks, while
 * bpcharlike matches the blank-padded value (textlike over the bpchar datum).
 *
 * MatchText recurses at every `%`; here the match is iterative, with the classic single-star backtrack: only the last `%`
 * seen is ever resumed, one character further along the text.  That finds a match whenever one exists because every
 * stretch of pattern between two `%` matches a fixed number of characters.
 */
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define LIKE_HD __host__ __device__ __forceinline__
#else
#define LIKE_HD static inline
#endif

/* 0: the pattern is well formed; -1: it ends in an escape with nothing to escape ("LIKE pattern must not end with escape
 * character", like_match.c) */
LIKE_HD int
like_pattern_check(const uint8_t *p, int plen)
{
	for (int i = 0; i < plen; i++)
		if (p[i] == '\\' && ++i >= plen)
			return -1;
	return 0;
}

/* characters of a UTF-8 string: its bytes less its continuation bytes */
LIKE_HD int
like_utf8_chars(const uint8_t *t, int tlen)
{
	int			n = 0;

	for (int i = 0; i < tlen; i++)
		n += (t[i] & 0xC0) != 0x80;
	return n;
}

/* byte i of the padded text */
LIKE_HD uint8_t
like_byte(const uint8_t *t, int tlen, int i)
{
	return i < tlen ? t[i] : (uint8_t) ' ';
}

/* bytes of the character starting at byte i (pg_utf_mblen), never past the end n */
LIKE_HD int
like_char_len(const uint8_t *t, int tlen, int n, int i)
{
	const uint8_t c = like_byte(t, tlen, i);
	const int	l = (c & 0x80) == 0 ? 1 : (c & 0xE0) == 0xC0 ? 2 : (c & 0xF0) == 0xE0 ? 3 : (c & 0xF8) == 0xF0 ? 4 : 1;

	return l < n - i ? l : n - i;
}

/* 1 when t (plus pad blanks) matches the pattern, else 0; the pattern must pass like_pattern_check */
LIKE_HD int
like_match(const uint8_t *t, int tlen, int pad, const uint8_t *p, int plen)
{
	const int	n = tlen + pad;
	int			ti = 0,
				pi = 0,
				star_p = -1,	/* pattern position behind the last `%`, and the text position it resumes from */
				star_t = 0;

	while (ti < n)
	{
		if (pi < plen)
		{
			const uint8_t c = p[pi];

			if (c == '%')
			{
				star_p = ++pi;
				star_t = ti;
				continue;
			}
			if (c == '_')
			{
				ti += like_char_len(t, tlen, n, ti);
				pi++;
				continue;
			}
			if (c == '\\' ? (pi + 1 < plen && p[pi + 1] == like_byte(t, tlen, ti)) : c == like_byte(t, tlen, ti))
			{
				pi += c == '\\' ? 2 : 1;
				ti++;
				continue;
			}
		}
		/* mismatch, or pattern used up with text left: the last `%` takes one more character */
		if (star_p < 0)
			return 0;
		star_t += like_char_len(t, tlen, n, star_t);
		ti = star_t;
		pi = star_p;
	}
	while (pi < plen && p[pi] == '%')
		pi++;
	return pi == plen;
}
