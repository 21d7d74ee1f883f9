"""Developer tool: CTC prefix beam search with a word n-gram LM, B = 64 utterances of T' = 247
frames of a character model, S = 29 (26 letters, the apostrophe, the space and the blank).

    python tools/ctc_wordlm_decode_bench.py [--reps N] [--out F]

Synthetic, seeded data: a vocabulary of 5k or 20k made-up words, a Markov chain over them (each word
has a few likely successors) writes the LMs' training text and each utterance's transcript; the
posteriors are CTC-shaped (each character on one or two frames between blanks, the space between
words) with Gaussian noise on the logits, so some characters are ambiguous.  The word LMs are
WordLM.train 3- and 4-grams on that text; the character LM is a NGramLM.train 5-gram on the same
text spelled out.

Prints the card name and power limit, then JSON lines:
  - "load": the CPU time of WordLM.from_arpa plus device_tables for a synthetic 20k-word 3-gram
    ARPA file of about 1.5 M n-grams (random values);
  - per (vocabulary, order, beam): ms per call of the search alone (log-probabilities on the
    device; median of --reps after one warm-up) with no LM, the character 5-gram and the word LM,
    on the route sb_ctc_prefix_beam takes (full scan at S = 29) and on the forced shortlist route,
    with the fraction of frames the shortlist's bound check rescanned in full;
  - "infer": CTC.infer of the benchmark's encoder (biGRU 2 x 1024, exact lengths off) with the
    search at beam 32, no LM / word LM.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, ".")

from speech_b200 import _lib  # noqa: E402
from speech_b200.lm import NGramLM, WordLM  # noqa: E402

B, T = 64, 247
SYMBOLS = [chr(ord("a") + i) for i in range(26)] + ["'", " "]
S, DELIM, BLANK = 29, 27, 28
ALPHA, BETA, GAMMA = 0.8, 1.0, -4.0


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def vocabulary(rng, n):
    words = set()
    while len(words) < n:
        words.add("".join(rng.choice(SYMBOLS[:26], rng.randint(2, 9))))
    return sorted(words)


def texts(rng, words, n, fan=4):
    nxt = rng.randint(0, len(words), (len(words), fan))
    out = []
    for _ in range(n):
        w = int(rng.randint(len(words)))
        seq = [w]
        for _ in range(rng.randint(3, 15)):
            w = int(nxt[w, rng.randint(fan)]) if rng.rand() < 0.9 else int(rng.randint(len(words)))
            seq.append(w)
        out.append(" ".join(words[i] for i in seq))
    return out


def posteriors(rng, sentences):
    x = rng.randn(B, T, S).astype(np.float32) * 1.5
    for b in range(B):
        labels = [SYMBOLS.index(c) for c in sentences[b]]
        t = 0
        for c in labels:
            if t + 4 >= T:
                break
            for _ in range(rng.randint(1, 3)):
                x[b, t, c] += 5.0 + rng.randn()
                t += 1
            x[b, t, BLANK] += 4.0
            t += 1
        x[b, t:, BLANK] += 5.0
    return torch.log_softmax(torch.from_numpy(x), 2).cuda().contiguous()


def search(lib, logp, K, lm=None, forced=False):
    lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
    nbytes = _lib.workspace_size(lib.sb_ctc_prefix_beam_workspace_size, B, T, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    lab = torch.empty(B, T, dtype=torch.int32, device="cuda")
    n = torch.empty(B, dtype=torch.int32, device="cuda")
    sc = torch.empty(B, dtype=torch.float64, device="cuda")
    outs = (lab.data_ptr(), n.data_ptr(), sc.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr())
    args = (logp.data_ptr(), lens.data_ptr(), B, T, S, K, BLANK)

    def call():
        if lm is None:
            fn = lib.sb_ctc_prefix_beam_shortlist if forced else lib.sb_ctc_prefix_beam
            st = fn(*args, *outs)
        elif isinstance(lm, WordLM):
            fn = lib.sb_ctc_prefix_beam_wordlm_shortlist if forced else lib.sb_ctc_prefix_beam_wordlm
            st = fn(*args, ctypes.byref(lm.device_tables(logp.device)[0]), ALPHA, BETA, GAMMA,
                    *outs)
        else:
            fn = lib.sb_ctc_prefix_beam_lm_shortlist if forced else lib.sb_ctc_prefix_beam_lm
            st = fn(*args, ctypes.byref(lm.device_tables(logp.device)[0]), 0.5, 1.0, *outs)
        _lib.check(st, "decode")
        torch.cuda.synchronize()

    return call


def timed(call, reps):
    call()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts) * 1e3


def rescanned(lib, call):
    got = ctypes.c_ulonglong(0)
    _lib.check(lib.sb_debug_ctc_lm_rescans(ctypes.byref(got)), "rescans")     # reset
    call()
    _lib.check(lib.sb_debug_ctc_lm_rescans(ctypes.byref(got)), "rescans")
    return got.value / (B * T)


def synthetic_arpa(path, rng, W=20000, n2=500000, n3=1000000):
    words = vocabulary(rng, W)
    with open(path, "w") as fh:
        fh.write("\\data\\\nngram 1=%d\nngram 2=%d\nngram 3=%d\n\n\\1-grams:\n" % (W + 3, n2, n3))
        fh.write("-99\t<s>\t-0.3\n-1.5\t</s>\n-3.0\t<unk>\t-0.2\n")
        for w, p, b in zip(words, -rng.rand(W) * 4 - 1, -rng.rand(W)):
            fh.write("%.4f\t%s\t%.4f\n" % (p, w, b))
        fh.write("\n\\2-grams:\n")
        big = np.unique(rng.randint(0, W, (n2 * 2, 2)), axis=0)[:n2]
        for (a, c), p, b in zip(big, -rng.rand(n2) * 3, -rng.rand(n2)):
            fh.write("%.4f\t%s %s\t%.4f\n" % (p, words[a], words[c], b))
        fh.write("\n\\3-grams:\n")
        tri = big[rng.randint(0, n2, n3)]
        tri = np.unique(np.concatenate([tri, rng.randint(0, W, (n3, 1))], 1), axis=0)
        tri = tri[:n3]
        for (a, c, d), p in zip(tri, -rng.rand(len(tri)) * 2):
            fh.write("%.4f\t%s %s %s\n" % (p, words[a], words[c], words[d]))
        fh.write("\n\\end\\\n")
    return len(tri)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    lib = _lib.load()
    print("card:", card(), flush=True)
    lines = []

    def emit(rec):
        print(json.dumps(rec), flush=True)
        lines.append(rec)

    rng = np.random.RandomState(0)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "w3.arpa")
        n3 = synthetic_arpa(path, rng)
        # the trigram count is what unique() left, so rewrite the header's count
        text = open(path).read().replace("ngram 3=1000000", "ngram 3=%d" % n3, 1)
        open(path, "w").write(text)
        t0 = time.perf_counter()
        wlm = WordLM.from_arpa(path, SYMBOLS)
        t1 = time.perf_counter()
        wlm.device_tables("cuda")
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        emit({"load": "20k-word 3-gram", "ngrams": 20003 + 500000 + n3,
              "from_arpa_s": round(t1 - t0, 2), "device_tables_s": round(t2 - t1, 2)})

    char_lm = None
    for W in (5000, 20000):
        rng = np.random.RandomState(W)
        words = vocabulary(rng, W)
        train = texts(rng, words, 4 * W)
        sentences = texts(rng, words, B)
        logp = posteriors(rng, sentences)
        if char_lm is None:
            t0 = time.perf_counter()
            char_lm = NGramLM.train([[SYMBOLS.index(c) for c in t] for t in train[:20000]], 5, S,
                                    BLANK)
            emit({"char_lm": "5-gram", "train_s": round(time.perf_counter() - t0, 2)})
        for order in (3, 4):
            t0 = time.perf_counter()
            lm = WordLM.train(train, order, SYMBOLS, oov_penalty=GAMMA)
            lm.device_tables("cuda")
            build_s = time.perf_counter() - t0
            for K in (1, 8, 32):
                rec = {"words": W, "order": order, "beam": K, "lm_build_s": round(build_s, 1),
                       "lm_ngrams": int(len(lm.host_tables()["logp"]))}
                for name, m in (("none", None), ("char5", char_lm), ("word", lm)):
                    rec["ms_full_" + name] = round(timed(search(lib, logp, K, m), args.reps), 3)
                    forced = search(lib, logp, K, m, forced=True)
                    rec["ms_shortlist_" + name] = round(timed(forced, args.reps), 3)
                    if m is not None:
                        rec["rescan_" + name] = round(rescanned(lib, forced), 4)
                emit(rec)

    from speech_b200.models import CTC
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": [[32, 5, 8, 2], [32, 5, 8, 2]],
                                       "rnn": {"dim": 1024, "bidirectional": True, "layers": 2}}}
    model = CTC(161, S - 1, cfg).cuda()
    model.set_eval()
    frames = 4 * T + 12                    # T' = 247 after the two stride-2 convs
    inputs = [np.random.RandomState(b).randn(frames, 161).astype(np.float32) for b in range(B)]
    batch = (inputs, [[0]] * B)
    for name, kw in (("none", {}), ("word", {"lm": lm, "lm_weight": ALPHA,
                                             "insertion_bonus": BETA})):
        ms = timed(lambda: model.infer(batch, beam_size=32, **kw), args.reps)
        emit({"infer": name, "beam": 32, "B": B, "ms": round(ms, 2)})
    if args.out:
        with open(args.out, "w") as fh:
            json.dump({"card": card(), "results": lines}, fh, indent=1)


if __name__ == "__main__":
    main()
