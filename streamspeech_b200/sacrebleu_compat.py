"""sacrebleu 2.2.0's `corpus_bleu` restated: what asr_bleu/compute_asr_bleu.py scores with `sacrebleu.corpus_bleu(hyps, [refs])`.

Defaults only, as the script uses them: the 13a tokenizer, n-grams up to 4, `exp` smoothing, no lowercasing, one reference stream.
sacrebleu is third-party code that is neither in the reference tree nor installed here, so this restatement is pinned to known-answer
tests (tests/test_asr_bleu.py), not to sacrebleu itself (DESIGN.md §11).  fairseq's token-id BLEU of the offline generator is a
different scorer (generate.BleuScorer).
"""
from __future__ import annotations

import math
import re
from collections import Counter
from typing import List, Sequence

MAX_NGRAM_ORDER = 4

# tokenizer_13a.py / tokenizer_re.py: the mteval-v13a.pl rules
_RE_13A = [
    (re.compile(r"([\{-\~\[-\` -\&\(-\+\:-\@\/])"), r" \1 "),  # punctuation and symbols
    (re.compile(r"([^0-9])([\.,])"), r"\1 \2 "),                # period and comma unless preceded by a digit
    (re.compile(r"([\.,])([^0-9])"), r" \1 \2"),                # ... unless followed by a digit
    (re.compile(r"([0-9])(-)"), r"\1 \2 "),                     # dash after a digit
]


def tokenize_13a(line: str) -> str:
    line = line.replace("<skipped>", "").replace("-\n", "").replace("\n", " ")
    if "&" in line:
        line = line.replace("&quot;", '"').replace("&amp;", "&").replace("&lt;", "<").replace("&gt;", ">")
    line = f" {line} "
    for rx, repl in _RE_13A:
        line = rx.sub(repl, line)
    return " ".join(line.split())


def ngram_counts(words: Sequence[str], max_order: int = MAX_NGRAM_ORDER) -> Counter:
    c = Counter()
    for n in range(1, max_order + 1):
        for i in range(len(words) - n + 1):
            c[tuple(words[i:i + n])] += 1
    return c


def _log(x: float) -> float:
    return -9999999999 if x == 0 else math.log(x)


class BLEUScore:
    """sacrebleu.metrics.bleu.BLEUScore: `str()` and `format(width)` give the line compute_asr_bleu.py prints and writes"""

    name = "BLEU"

    def __init__(self, score: float, counts: List[int], totals: List[int], precisions: List[float], bp: float, sys_len: int, ref_len: int):
        self.score, self.counts, self.totals, self.precisions = score, counts, totals, precisions
        self.bp, self.sys_len, self.ref_len = bp, sys_len, ref_len
        self.ratio = sys_len / ref_len if ref_len else 0
        self.prec_str = "/".join(f"{p:.1f}" for p in precisions)
        self._verbose = f"{self.prec_str} (BP = {self.bp:.3f} ratio = {self.ratio:.3f} hyp_len = {self.sys_len:d} ref_len = {self.ref_len:d})"

    def format(self, width: int = 2, score_only: bool = False) -> str:
        if score_only:
            return f"{self.score:.{width}f}"
        return f"{self.name} = {self.score:.{width}f} {self._verbose}"

    def __repr__(self) -> str:
        return self.format()

    __str__ = __repr__


def compute_bleu(correct: List[int], total: List[int], sys_len: int, ref_len: int) -> BLEUScore:
    """BLEU.compute_bleu with smooth_method='exp', effective order off"""
    bp = (math.exp(1 - ref_len / sys_len) if sys_len > 0 else 0.0) if sys_len < ref_len else 1.0
    precisions = [0.0] * MAX_NGRAM_ORDER
    if not any(correct):
        return BLEUScore(0.0, correct, total, precisions, bp, sys_len, ref_len)
    smooth_mteval = 1.0
    for n in range(1, MAX_NGRAM_ORDER + 1):
        if total[n - 1] == 0:
            break
        if correct[n - 1] == 0:
            smooth_mteval *= 2
            precisions[n - 1] = 100.0 / (smooth_mteval * total[n - 1])
        else:
            precisions[n - 1] = 100.0 * correct[n - 1] / total[n - 1]
    score = bp * math.exp(sum(_log(p) for p in precisions) / MAX_NGRAM_ORDER)
    return BLEUScore(score, correct, total, precisions, bp, sys_len, ref_len)


def corpus_bleu(hypotheses: Sequence[str], references: Sequence[Sequence[str]]) -> BLEUScore:
    """sacrebleu.corpus_bleu(hypotheses, references) with its defaults; references = list of reference streams"""
    if len(references) != 1:
        raise ValueError("one reference stream is supported (compute_asr_bleu.py passes [refs])")
    refs = references[0]
    if len(refs) != len(hypotheses):
        raise ValueError(f"{len(hypotheses)} hypotheses but {len(refs)} references")
    correct, total = [0] * MAX_NGRAM_ORDER, [0] * MAX_NGRAM_ORDER
    sys_len = ref_len = 0
    for hyp, ref in zip(hypotheses, refs):
        hw = tokenize_13a(hyp.rstrip()).split()
        rw = tokenize_13a(ref.rstrip()).split()
        sys_len += len(hw)
        ref_len += len(rw)
        hc, rc = ngram_counts(hw), ngram_counts(rw)
        for ng, c in hc.items():
            n = len(ng) - 1
            total[n] += c
            if ng in rc:
                correct[n] += min(c, rc[ng])
    return compute_bleu(correct, total, sys_len, ref_len)
