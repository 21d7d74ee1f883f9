"""Developer tool: Seq2Seq.recognize with a word n-gram LM, against no LM and a character n-gram.

    python tools/s2s_wordlm_recognize_bench.py [--beams 1 4 10] [--reps N] [--out F]

The WSJ-shaped attention model of tools/s2s_recognize_bench.py (conv + 3x biGRU-512, log_t,
embedding 512, untrained) with a CTC head, at V = 32: 29 one-character symbols, the space, END and
START; B = 16 utterances of T = 800 input frames, max_len = 100.  Synthetic word text: words of
2-8 letters drawn with a Zipf-like unigram so that contexts repeat, every lexicon word at least
once.  LMs, all trained by interpolated Kneser-Ney on that text: a 5k-word 3-gram and a 20k-word
4-gram (WordLM, lm_weight 0.8, insertion_bonus 1 per word, oov_penalty -4), and a character
5-gram over 3000 sentences of the 5k text (NGramLM, lm_weight 0.8, insertion_bonus 1 per
character).  Prints the card name and power limit, then one JSON line per (beam, LM, ctc_weight
in {0, 0.3}) with:
  - ms per call of the search alone (beam_search_batch on precomputed encoder states and CTC
    log-probabilities), and of recognize (encoder included), median of --reps after a warm-up,
    from the host clock between synchronisations;
  - the steps the batch's search ran, and the search's ms per step, which compares LMs that
    change where the searches stop.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from s2s_recognize_bench import card, timed  # noqa: E402

LETTERS = "abcdefghijklmnopqrstuvwxyz'.-"
SYMBOLS = list(LETTERS) + [" ", "</s>", "<s>"]
V = len(SYMBOLS)                                   # 32: END = 30, START = 31, the space 29


def synthetic_text(n_words, n_sentences, seed):
    rng = np.random.RandomState(seed)
    letters = list(LETTERS[:26])
    vocab = set()
    while len(vocab) < n_words:
        vocab.add("".join(rng.choice(letters, rng.randint(2, 9))))
    vocab = sorted(vocab)
    rng.shuffle(vocab)
    w = 1.0 / np.arange(1, n_words + 1) ** 1.1
    w /= w.sum()
    texts = [" ".join(rng.choice(vocab, rng.randint(5, 20), p=w)) for _ in range(n_sentences)]
    texts += [" ".join(vocab[i:i + 10]) for i in range(0, n_words, 10)]
    return texts


def model(B, frames):
    import bench
    from speech_b200.models import Seq2Seq
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": bench.WSJ_CONV,
                                       "rnn": {"dim": 512, "bidirectional": True, "layers": 3}},
           "decoder": {"embedding_dim": 512, "layers": 1, "log_t": True, "ctc_weight": 0.3}}
    m = Seq2Seq(bench.F_IN, V, cfg).cuda()
    m.set_eval()
    rng = np.random.RandomState(0)
    inputs = [rng.randn(frames, bench.F_IN).astype(np.float32) for _ in range(B)]
    return m, inputs


def lms():
    from speech_b200.lm import NGramLM, WordLM
    t5k = synthetic_text(5000, 4000, 1)
    t20k = synthetic_text(20000, 6000, 2)
    kw = dict(blank=V - 1, end=V - 2, oov_penalty=-4.0)
    cls = {c: i for i, c in enumerate(SYMBOLS[:V - 2])}
    chars = [[V - 1] + [cls[c] for c in t] + [V - 2] for t in t5k[:3000]]
    return {"char5": NGramLM.train(chars, 5, V, V - 1, end=V - 2),
            "word3_5k": WordLM.train(t5k, 3, SYMBOLS, **kw),
            "word4_20k": WordLM.train(t20k, 4, SYMBOLS, **kw)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--beams", nargs="+", type=int, default=[1, 4, 10])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--max-len", type=int, default=100)
    ap.add_argument("--lm-weight", type=float, default=0.8)
    ap.add_argument("--insertion-bonus", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from speech_b200.functions import s2s
    print("card:", card(), flush=True)
    models = lms()
    m, inputs = model(args.batch, args.frames)
    B, L, a, bonus, lam = args.batch, args.max_len, args.lm_weight, args.insertion_bonus, 0.3
    with torch.no_grad():
        x = m._encode(m.stage_inputs(inputs), None)
        y = torch.log_softmax(m.ctc_fc(x).float(), dim=-1).contiguous()
    lines = []
    for K in args.beams:
        M = min(V - 1, 3 * K // 2)
        for name in ["none"] + list(models):
            lm = models.get(name)
            fusion = {} if lm is None else {"lm": lm, "lm_weight": a, "insertion_bonus": bonus}
            for w in (0.0, lam):
                ctc = (y, w, M) if w > 0 else None

                def search():
                    with torch.no_grad():
                        return s2s.beam_search_batch(m, x, V - 1, V - 2, K, L, None,
                                                     ctc=ctc, **fusion)

                def rec():
                    return m.recognize(inputs, beam_size=K, max_len=L, ctc_weight=w, **fusion)
                t_s = timed(search, args.reps)
                t_r = timed(rec, args.reps)
                steps = max(r[2] for r in search())
                line = {"beam": K, "lm": name, "ctc_weight": w, "B": B,
                        "T_frames": int(x.shape[1]), "max_len": L,
                        "search_ms": round(1e3 * t_s, 2), "recognize_ms": round(1e3 * t_r, 2),
                        "batch_steps": steps, "search_ms_per_step": round(1e3 * t_s / steps, 3)}
                if lm is not None:
                    line.update(lm_weight=a, insertion_bonus=bonus, order=lm.order)
                    if name != "char5":
                        line.update(words=lm.num_words, oov_penalty=lm.oov_penalty)
                print(json.dumps(line), flush=True)
                lines.append(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump({"card": card(), "cases": lines}, fh, indent=1)


if __name__ == "__main__":
    main()
