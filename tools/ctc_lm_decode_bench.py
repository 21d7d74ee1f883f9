"""Developer tool: CTC prefix beam search with and without n-gram LM fusion, B = 64 utterances of
T' = 247 frames (the benchmark's decode shape).

    python tools/ctc_lm_decode_bench.py [--sizes 29 1000 5000] [--reps N] [--out F]

Synthetic, seeded data: a Markov chain over the S - 1 non-blank classes (each class has a few
likely successors) writes the LM's training text and each utterance's label sequence; the
posteriors are CTC-shaped (labels spread over frames with blanks between them) with Gaussian noise
on the logits, so the acoustic evidence is ambiguous on some frames.  The LM is NGramLM.train on
that text: a 5-gram at S = 29, a 3-gram at S = 1000 and 5000.

Prints the card name and power limit, then one JSON line per case (S, beam) with:
  - utt/s and ms per call of the search alone (log-probabilities already on the device), LM off
    and on (lm_weight 0.5, insertion_bonus 1.0), median of --reps after one warm-up, host clock
    between synchronisations;
  - the route sb_ctc_prefix_beam_lm takes (full scan or shortlist);
  - the forced shortlist route with the LM: ms per call and the fraction of frames its bound check
    could not prove and rescanned in full (sb_debug_ctc_lm_rescans).
"""
import argparse
import ctypes
import json
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")

from speech_b200 import _lib  # noqa: E402
from speech_b200.lm import NGramLM  # noqa: E402

B, T = 64, 247
ALPHA, BETA = 0.5, 1.0


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def chain(rng, V, fan=4):
    nxt = rng.randint(0, V, (V, fan))
    return lambda c: int(nxt[c, rng.randint(fan)]) if rng.rand() < 0.9 else int(rng.randint(V))


def sentence(rng, step, V, n):
    c = int(rng.randint(V))
    out = [c]
    for _ in range(n - 1):
        c = step(c)
        out.append(c)
    return out


def posteriors(rng, step, S):
    blank = S - 1
    logits = rng.randn(B, T, S).astype(np.float32) * 1.5
    for b in range(B):
        labels = sentence(rng, step, S - 1, rng.randint(40, 90))
        pos = np.sort(rng.choice(T, len(labels), replace=False))
        logits[b, :, blank] += 4.0
        for t, c in zip(pos, labels):
            logits[b, t, c] += 5.0 + rng.randn()
    return torch.log_softmax(torch.from_numpy(logits), 2).cuda().contiguous()


def run(lib, logp, K, lm=None, forced=False):
    S = logp.shape[2]
    lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
    nbytes = _lib.workspace_size(lib.sb_ctc_prefix_beam_workspace_size, B, T, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    lab = torch.empty(B, T, dtype=torch.int32, device="cuda")
    n = torch.empty(B, dtype=torch.int32, device="cuda")
    sc = torch.empty(B, dtype=torch.float64, device="cuda")
    outs = (lab.data_ptr(), n.data_ptr(), sc.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr())

    def call():
        if lm is None:
            st = lib.sb_ctc_prefix_beam(logp.data_ptr(), lens.data_ptr(), B, T, S, K, S - 1, *outs)
        else:
            fn = lib.sb_ctc_prefix_beam_lm_shortlist if forced else lib.sb_ctc_prefix_beam_lm
            st = fn(logp.data_ptr(), lens.data_ptr(), B, T, S, K, S - 1,
                    ctypes.byref(lm.device_tables(logp.device)[0]), ALPHA, BETA, *outs)
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[29, 1000, 5000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    lib = _lib.load()
    print("card:", card(), flush=True)
    lines = []
    for S, order, beams, n_text in ((29, 5, (1, 8, 32), 4000), (1000, 3, (8,), 10000),
                                    (5000, 3, (8,), 20000)):
        if S not in args.sizes:
            continue
        rng = np.random.RandomState(S)
        step = chain(rng, S - 1)
        text = [sentence(rng, step, S - 1, rng.randint(10, 60)) for _ in range(n_text)]
        t0 = time.perf_counter()
        lm = NGramLM.train(text, order, S, S - 1)
        logp = posteriors(rng, step, S)
        lm.device_tables(logp.device)
        build_s = time.perf_counter() - t0
        print("S = %d: %d-gram built and uploaded in %.1f s" % (S, order, build_s), flush=True)
        for K in beams:
            off = timed(run(lib, logp, K), args.reps)
            print("  beam %d: LM off %.3f ms" % (K, off), flush=True)
            on = timed(run(lib, logp, K, lm), args.reps)
            print("  beam %d: LM on %.3f ms" % (K, on), flush=True)
            full_fits = (K * S + K) * 13 + 16 <= 200 * 1024
            forced = run(lib, logp, K, lm, forced=True)
            got = ctypes.c_ulonglong(0)
            _lib.check(lib.sb_debug_ctc_lm_rescans(ctypes.byref(got)), "rescans")   # reset
            forced()
            _lib.check(lib.sb_debug_ctc_lm_rescans(ctypes.byref(got)), "rescans")
            rescans = got.value / (B * T)
            ms_forced = timed(forced, args.reps)
            lib.sb_debug_ctc_lm_rescans(ctypes.byref(got))
            rec = {"S": S, "beam": K, "lm_order": order,
                   "lm_ngrams": int(len(lm.host_tables()["logp"])),
                   "lm_build_s": round(build_s, 2),
                   "route": "full" if full_fits else "shortlist",
                   "ms_lm_off": round(off, 3), "ms_lm_on": round(on, 3),
                   "utt_s_lm_off": round(B / off * 1e3, 1), "utt_s_lm_on": round(B / on * 1e3, 1),
                   "lm_cost": round(on / off, 3),
                   "ms_lm_shortlist_forced": round(ms_forced, 3),
                   "shortlist_rescan_fraction": round(rescans, 4)}
            print(json.dumps(rec), flush=True)
            lines.append(rec)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump({"card": card(), "results": lines}, fh, indent=1)


if __name__ == "__main__":
    main()
