"""Host restatement of nats_rouge_f (include/nats_b200.h) in integers: the ROUGE-1, ROUGE-2 and ROUGE-L F of token-id
sequences, each exactly np.float32(2 h) / np.float32(m + c).  The kernel must match it bit for bit; it is itself checked
against nats_b200.evaluate (ROUGE.pl's restatement) in tests/test_scst_host.py."""
from collections import Counter

import numpy as np

UNK = 1


def words(seq, length=None, cap=None):
    """a row's words: its first min(length, cap) entries (length clamped to [0, cap]) up to the first 0 (excluded)"""
    seq = [int(t) for t in seq]
    cap = len(seq) if cap is None else cap
    L = len(seq) if length is None else min(max(int(length), 0), cap)
    out = []
    for t in seq[:L]:
        if t == 0:
            break
        out.append(t)
    return out


def _grams(w, n):
    return [tuple(w[i:i + n]) for i in range(len(w) - n + 1)]


def ngram_hits(a, b, n):
    """ROUGE.pl's clipped hits sum_g min(c_ref(g), c_cand(g)); an n-gram holding UNK matches nothing"""
    ca = Counter(g for g in _grams(a, n) if UNK not in g)
    cb = Counter(g for g in _grams(b, n) if UNK not in g)
    return sum(min(c, cb[g]) for g, c in ca.items() if g in cb)


def lcs(a, b):
    prev = [0] * (len(b) + 1)
    for x in a:
        cur = [0] * (len(b) + 1)
        for j, y in enumerate(b, 1):
            cur[j] = prev[j - 1] + 1 if (x == y and x != UNK) else max(prev[j], cur[j - 1])
        prev = cur
    return prev[-1]


def fval(h, m, c):
    return np.float32(0.) if h == 0 else np.float32(2 * h) / np.float32(m + c)


def rouge_words(cand, ref):
    """(R1, R2, RL) F of two word lists (EOS already cut) as float32"""
    m, c = len(ref), len(cand)
    return np.array([fval(ngram_hits(ref, cand, 1), m, c),
                     fval(ngram_hits(ref, cand, 2), max(0, m - 1), max(0, c - 1)),
                     fval(lcs(ref, cand), m, c)], dtype=np.float32)


def rouge_rows(cands, refs, rows_per_ref=1, cand_len=None, ref_len=None, cand_cap=None, ref_cap=None):
    """[3, n] over rows: row r against refs[r // rows_per_ref]; lengths default to the rows' own"""
    n = len(cands)
    out = np.zeros((3, n), dtype=np.float32)
    for r in range(n):
        q = r // rows_per_ref
        a = words(refs[q], None if ref_len is None else ref_len[q], ref_cap)
        b = words(cands[r], None if cand_len is None else cand_len[r], cand_cap)
        out[:, r] = rouge_words(b, a)
    return out
