"""Developer tool: Seq2Seq.recognize with and without shallow fusion of an n-gram LM.

    python tools/s2s_lm_recognize_bench.py [--cases 32:5:1 ..] [--reps N] [--max-len N] [--out F]

The model and shapes of tools/s2s_recognize_bench.py: the WSJ-shaped attention model (conv + 3x
biGRU-512, log_t, embedding 512, untrained), B = 16 utterances of T = 800 input frames,
max_len = 100.  A case V:order:beam trains an `order`-gram (interpolated Kneser-Ney) on 2000
synthetic sentences over the V - 2 symbols (a Zipf-like unigram so that contexts repeat) and
fuses it with lm_weight 0.5, insertion_bonus 1.0.  Prints the card name and power limit, then one
JSON line per case with:
  - utt/s of recognize (encoder included) without and with the LM, from the host clock between
    synchronisations, median of --reps after one warm-up;
  - the same for the search alone (beam_search_batch on precomputed encoder states), and its ms
    per step the batch ran, which compares the two when the LM changes where the searches stop;
  - the route of the selection (split or one CTA per utterance) and the steps the batch ran.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from s2s_recognize_bench import card, model_and_inputs, timed  # noqa: E402


def synthetic_lm(V, order, n=2000, seed=0):
    from speech_b200.lm import NGramLM
    rng = np.random.RandomState(seed)
    w = 1.0 / np.arange(1, V - 1) ** 1.1
    w /= w.sum()
    sentences = [[V - 1] + rng.choice(V - 2, rng.randint(5, 60), p=w).tolist() + [V - 2]
                 for _ in range(n)]
    return NGramLM.train(sentences, order, V, V - 1, end=V - 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", default=["32:5:1", "32:5:4", "32:5:8",
                                                   "5000:3:1", "5000:3:4", "5000:3:8"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--max-len", type=int, default=100)
    ap.add_argument("--lm-weight", type=float, default=0.5)
    ap.add_argument("--insertion-bonus", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from speech_b200.functions import s2s
    print("card:", card(), flush=True)
    lines = []
    lms = {}
    for case in args.cases:
        V, order, K = (int(v) for v in case.split(":"))
        B, L, a, bonus = args.batch, args.max_len, args.lm_weight, args.insertion_bonus
        if (V, order) not in lms:
            lms[(V, order)] = synthetic_lm(V, order)
        lm = lms[(V, order)]
        m, inputs = model_and_inputs(V, B, args.frames)
        start, end = V - 1, V - 2
        with torch.no_grad():
            x_enc = m.encode(m.stage_inputs(inputs))
        fusion = {"lm": lm, "lm_weight": a, "insertion_bonus": bonus}

        def search(with_lm):
            with torch.no_grad():
                return s2s.beam_search_batch(m, x_enc, start, end, K, L, None,
                                             *((lm, a, bonus) if with_lm else ()))

        t_rec = timed(lambda: m.recognize(inputs, beam_size=K, max_len=L), args.reps)
        t_rec_lm = timed(lambda: m.recognize(inputs, beam_size=K, max_len=L, **fusion), args.reps)
        t_s = timed(lambda: search(False), args.reps)
        t_s_lm = timed(lambda: search(True), args.reps)
        steps = max(r[2] for r in search(False))
        steps_lm = max(r[2] for r in search(True))
        rec = {"V": V, "order": order, "beam": K, "B": B, "T_frames": int(x_enc.shape[1]),
               "max_len": L, "lm_weight": a, "insertion_bonus": bonus,
               "split_select": not s2s.beam_select_fits(K, V - 1),
               "recognize_utt_per_s": round(B / t_rec, 2),
               "recognize_lm_utt_per_s": round(B / t_rec_lm, 2),
               "search_ms": round(1e3 * t_s, 2), "search_lm_ms": round(1e3 * t_s_lm, 2),
               "batch_steps": steps, "batch_steps_lm": steps_lm,
               "search_ms_per_step": round(1e3 * t_s / steps, 3),
               "search_lm_ms_per_step": round(1e3 * t_s_lm / steps_lm, 3)}
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del m, x_enc
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump({"card": card(), "cases": lines}, fh, indent=1)


if __name__ == "__main__":
    main()
