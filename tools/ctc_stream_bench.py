"""Developer tool: cost of streaming recognition (CTC.stream) against offline CTC.infer.

    python tools/ctc_stream_bench.py [--streams 1,16,64] [--chunks 4,8,16,32] [--out F]

Model: bench.py's CTC encoder made unidirectional (conv [[32,5,8,2],[32,5,8,2]], 5 x GRU-1024),
V+1 = 29, and V+1 = 5000 for the shortlist route of the search (beam 8 there).  Each stream
receives 10 s of audio (1000 feature frames, 247 encoder frames) in chunks of 4 / 8 / 16 / 32
encoder frames (16 to 128 feature frames, 160 to 1280 ms), at beam 1 and 8, without an LM and with
a 3-gram (lm_weight 0.5, insertion_bonus 1.0).
Prints the card name and power limit, then one JSON line per case:
  enc_ms / search_ms   median device ms per push of the encoder (conv, projections, recurrence,
                       output projection, softmax) and of the search step, CUDA events around each
                       part, after one warm-up utterance;
  rtf                  summed device time of every push over the audio's duration;
  offline_ms           device ms of one CTC.infer over the same B utterances (median of 3).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import bench  # noqa: E402
from rnnt_recognize_bench import card  # noqa: E402

CFG = {"dropout": 0.0, "encoder": {"conv": [[32, 5, 8, 2], [32, 5, 8, 2]],
                                   "rnn": {"dim": 1024, "bidirectional": False, "layers": 5}}}
SECONDS = bench.T_IN / 100.0      # 10 ms per feature frame


def events():
    return [torch.cuda.Event(enable_timing=True) for _ in range(3)]


def run_stream(st, feats, chunk):
    """stream every utterance through st in chunks of `chunk` encoder frames; -> per-push
    (encoder ms, search ms)"""
    step = chunk * st.stride
    enc, srch = [], []
    for p in range(0, bench.T_IN, step):
        xs, counts = st._conv_inputs([f[p:p + step] for f in feats])
        T = max(counts)
        if T == 0:
            st._advance(xs, counts)
            continue
        e = events()
        e[0].record()
        with torch.no_grad():
            emit, Te, X = st._encode(xs, counts, T)
            logp = st._logp(X, Te) if Te else None
        e[1].record()
        if Te:
            st.search.push(logp, emit)
        e[2].record()
        e[2].synchronize()
        st._advance(xs, counts)
        enc.append(e[0].elapsed_time(e[1]))
        srch.append(e[1].elapsed_time(e[2]))
    return enc, srch


def offline_ms(m, batch, kw, reps=3):
    m.infer(batch, **kw)
    times = []
    for _ in range(reps):
        e = events()
        e[0].record()
        m.infer(batch, **kw)
        e[1].record()
        e[1].synchronize()
        times.append(e[0].elapsed_time(e[1]))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,16,64")
    ap.add_argument("--chunks", default="4,8,16,32")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from speech_b200.lm import NGramLM
    from speech_b200.models import CTC
    print("card:", card(), flush=True)
    out = open(a.out, "w") if a.out else None
    for V1 in (29, 5000):
        torch.manual_seed(0)
        m = CTC(bench.F_IN, V1 - 1, CFG).cuda()
        m.set_eval()
        rng = np.random.RandomState(1)
        lm = NGramLM.train([rng.randint(0, V1 - 1, rng.randint(5, 40)).tolist()
                            for _ in range(2000)], 3, num_classes=V1, blank=V1 - 1)
        for B in [int(s) for s in a.streams.split(",")]:
            inputs = [torch.from_numpy(x).cuda() for x in bench.synth_batch(B)[0][:B]]
            batch = ([x.cpu().numpy() for x in inputs], [[0]] * B)
            for K in ((1, 8) if V1 == 29 else (8,)):
                for with_lm in (False, True):
                    kw = {"beam_size": K}
                    if with_lm:
                        kw.update(lm=lm, lm_weight=0.5, insertion_bonus=1.0)
                    off = offline_ms(m, batch, kw)
                    for chunk in [int(c) for c in a.chunks.split(",")]:
                        st = m.stream(B, max_frames=300, **kw)
                        run_stream(st, inputs, chunk)                 # warm-up utterance
                        for b in range(B):
                            st.reset(b)
                        enc, srch = run_stream(st, inputs, chunk)
                        row = {"V1": V1, "B": B, "beam": K, "lm": "3-gram" if with_lm else None,
                               "chunk_frames": chunk, "chunk_ms": chunk * st.stride * 10,
                               "pushes": len(enc), "enc_ms": float(np.median(enc)),
                               "search_ms": float(np.median(srch)),
                               "rtf": (sum(enc) + sum(srch)) / 1e3 / SECONDS,
                               "offline_ms": off}
                        line = json.dumps(row)
                        print(line, flush=True)
                        if out:
                            out.write(line + "\n")
                            out.flush()
    if out:
        out.close()


if __name__ == "__main__":
    main()
