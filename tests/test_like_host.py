"""SQL LIKE as the kernels decide it (cloudberry_b200/csrc/like_match.cuh, compiled for the host) against an independent
reference: the pattern translated to a regular expression and matched with re.fullmatch on the decoded text, character(n)
values padded with blanks to n characters first (bpcharlike = textlike over the padded value).  Not gpu: k_dict_like runs the
same source, and tests/test_gpu_string_predicates.py holds its bitmaps against the same reference."""
import os
import random
import re
import shutil
import struct
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "native", "like_host.c")

# ASCII, the pattern metacharacters as data, 2-, 3- and 4-byte UTF-8 characters
ALPHABET = ["a", "b", "c", "A", " ", "%", "_", "\\", "é", "€", "𝄞"]


def like_ref(text, bpchar_len, pattern):
    """True / False, or None for a pattern that ends in a lone escape (an error in the reference)"""
    s = text + " " * max(0, bpchar_len - len(text)) if bpchar_len else text
    out, i = [], 0
    while i < len(pattern):
        c = pattern[i]
        if c == "\\":
            if i + 1 >= len(pattern):
                return None
            out.append(re.escape(pattern[i + 1]))
            i += 2
            continue
        out.append(".*" if c == "%" else "." if c == "_" else re.escape(c))
        i += 1
    return re.fullmatch("".join(out), s, re.DOTALL) is not None


def _rand_text(rng, n):
    return "".join(rng.choice(ALPHABET) for _ in range(n))


def _pattern_from(rng, text):
    """a pattern likely to match (or nearly match) `text`: characters replaced by `_`, runs by `%`, literals escaped"""
    out = []
    i = 0
    while i < len(text):
        r = rng.random()
        if r < 0.15:
            out.append("_")
        elif r < 0.25:
            out.append("%")
            i += rng.randrange(0, 3)
            continue
        elif r < 0.3:
            out.append(rng.choice(ALPHABET))
        elif text[i] in "%_\\" or r < 0.35:
            out.append("\\" + text[i])
        else:
            out.append(text[i])
        i += 1
    if rng.random() < 0.2:
        out.append(rng.choice(["%", "%%", " ", "  ", "_", "\\\\", "\\a"]))
    return "".join(out)


def make_cases(rng, n):
    """(text, bpchar_len, pattern): varchar and char(n) values (stored without trailing blanks), the empty string, random
    and derived patterns, patterns longer than the text, escapes of metacharacters and of ordinary characters"""
    fixed = [("", 0, "%"), ("", 0, ""), ("", 0, "_"), ("", 3, "___"), ("", 3, "__"), ("ab", 4, "ab"), ("ab", 4, "ab%"),
             ("ab", 4, "ab  "), ("ab", 0, "ab  "), ("a%b", 0, "a\\%b"), ("axb", 0, "a\\%b"), ("a_b", 0, "a\\_b"),
             ("a\\b", 0, "a\\\\b"), ("ab", 0, "\\a\\b"), ("ab", 0, "ab\\"), ("€x", 0, "_x"), ("𝄞", 0, "_"), ("𝄞", 0, "__"),
             ("aaa", 0, "%a%a%a%"), ("aa", 0, "%a%a%a%"), ("abc", 0, "%%%"), ("abc", 0, "a%%c"), ("PROMO BRUSHED", 0, "PROMO%"),
             ("forest green", 0, "%green%"), ("é", 2, "é_"), ("é", 2, "é")]
    cases = list(fixed)
    while len(cases) < n:
        text = _rand_text(rng, rng.randrange(0, 12))
        bp = 0
        if rng.random() < 0.35:
            text = text.rstrip(" ")
            bp = len(text) + rng.randrange(0, 4)
        if rng.random() < 0.5:
            pat = _pattern_from(rng, text)
        else:
            pat = "".join(rng.choice(ALPHABET + ["%", "_", "\\%", "\\_", "\\\\", "%", "\\a"]) for _ in range(rng.randrange(0, 14)))
        cases.append((text, bp, pat))
    return cases


def run_host(exe, cases):
    buf = [struct.pack("<i", len(cases))]
    for text, bp, pat in cases:
        t, p = text.encode(), pat.encode()
        buf.append(struct.pack("<iii", len(t), bp, len(p)) + t + p)
    out = subprocess.run([exe], input=b"".join(buf), stdout=subprocess.PIPE, stderr=subprocess.PIPE, check=True)
    assert len(out.stdout) == len(cases), out.stderr.decode()[-2000:]
    return [{"1": True, "0": False, "E": None}[chr(c)] for c in out.stdout]


def _build(tmp, name, extra):
    cc = shutil.which("gcc") or shutil.which("cc")
    if not cc:
        pytest.skip("no C compiler")
    exe = str(tmp / name)
    subprocess.check_call([cc, "-std=c11", "-O1", "-g", "-Wall", "-Werror"] + extra + ["-o", exe, SRC])
    return exe


def _check(exe, seed, n):
    rng = random.Random(seed)
    cases = make_cases(rng, n)
    got = run_host(exe, cases)
    bad = [(c, g, like_ref(*c)) for c, g in zip(cases, got) if g != like_ref(*c)]
    assert not bad, bad[:10]
    return got


def test_like_matches_reference(tmp_path):
    got = _check(_build(tmp_path, "like_host", []), 20261016, 120000)
    # the corpus exercises every outcome
    assert got.count(True) > 5000 and got.count(False) > 5000 and got.count(None) > 100


def test_like_under_sanitizers(tmp_path):
    try:
        exe = _build(tmp_path, "like_host_san", ["-fsanitize=address,undefined", "-fno-sanitize-recover=all"])
    except subprocess.CalledProcessError:
        pytest.skip("the C compiler has no AddressSanitizer / UBSan runtime")
    _check(exe, 20261016, 120000)
