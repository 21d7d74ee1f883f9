"""Scoring - host-side mirror of speech/utils/score.py:7-18 (reference), SURVEY.md section 8f
rank 4.  The reference depends on the `editdistance` C extension; the Levenshtein distance here
is the library's host function `sb_edit_distance` (csrc/api.cu)."""
import ctypes

from .. import _lib


def edit_distance(a, b):
    """Levenshtein distance of two sequences of hashable tokens (`editdistance.eval(a, b)`)."""
    lib = _lib.load()
    ids = {}
    ia = [ids.setdefault(t, len(ids)) for t in a]
    ib = [ids.setdefault(t, len(ids)) for t in b]
    ca = (ctypes.c_int * max(len(ia), 1))(*ia)
    cb = (ctypes.c_int * max(len(ib), 1))(*ib)
    d = lib.sb_edit_distance(ca, len(ia), cb, len(ib))
    if d < 0:
        raise _lib.SpeechB200Error("sb_edit_distance: invalid arguments")
    return int(d)


def compute_cer(results):
    """results: list of (ground truth, prediction) sequence pairs -> total edit distance divided
    by the total label length (score.py:7-18)."""
    dist = sum(edit_distance(label, pred) for label, pred in results)
    total = sum(len(label) for label, _ in results)
    return dist / total


def compute_wer(results, delimiter):
    """results: list of (ground truth, prediction) label sequence pairs -> word error rate: the
    total word edit distance divided by the total number of reference words.  A word is a maximal
    run of labels other than `delimiter` (the space class of a character model)."""
    def words(seq):
        out, cur = [], []
        for v in seq:
            if v == delimiter:
                if cur:
                    out.append(tuple(cur))
                cur = []
            else:
                cur.append(v)
        if cur:
            out.append(tuple(cur))
        return out

    pairs = [(words(label), words(pred)) for label, pred in results]
    dist = sum(edit_distance(label, pred) for label, pred in pairs)
    total = sum(len(label) for label, _ in pairs)
    return dist / total
