"""Developer tool: cost of streaming Transducer recognition (Transducer.stream) against offline
Transducer.recognize.

    python tools/rnnt_stream_bench.py [--chunks 16,128] [--cases all] [--out F]

Model: bench.py's RNN-T made unidirectional (conv [[32,5,8,2],[32,5,8,2]], 3 x GRU-1024 encoder,
GRU-1024 prediction network, embedding 256), S = 4 symbols per frame.  Each stream receives 10 s
of audio (1000 feature frames, 247 encoder frames) in chunks of 16 / 128 feature frames (160 /
1280 ms).  Cases: V+1 = 29 at B = 1, beam 1; V+1 = 29 at B = 64, beam 4, without an LM and with a
3-gram (lm_weight 0.5, insertion_bonus 1.0); V+1 = 1024 at B = 64, beam 4 (slab joint, full
route); V+1 = 5001 at B = 64, beam 8 (the stream's 64-entry shortlist route).
Prints the card name and power limit, then one JSON line per case and chunk:
  enc_ms / search_ms   median device ms per push of the encoder (conv, projections, recurrence,
                       fc1) and of the search (joint rows, rounds, prediction steps), CUDA events
                       around each part, after a warm-up of 2 s of audio;
  push_total_ms        summed device ms of every push of the 10 s;
  rtf                  push_total_ms over the audio's duration;
  launches_per_push    C-ABI launches per push (the package's own kernels and GEMMs);
  offline_ms           device ms of one Transducer.recognize over the same B utterances.
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

SECONDS = bench.T_IN / 100.0      # 10 ms per feature frame
S = 4
CASES = [  # V+1, B, beam, LM order
    (29, 1, 1, 0), (29, 64, 4, 0), (29, 64, 4, 3), (1024, 64, 4, 0), (5001, 64, 8, 0)]


def events():
    return [torch.cuda.Event(enable_timing=True) for _ in range(3)]


def model(V1):
    from speech_b200.models import Transducer
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "exact_lengths": True,
           "encoder": {"conv": bench.WSJ_CONV,
                       "rnn": {"dim": 1024, "bidirectional": False, "layers": 3}},
           "decoder": {"embedding_dim": 256, "layers": 1}}
    m = Transducer(bench.F_IN, V1 - 1, cfg).cuda()
    m.set_eval()
    return m


def run_stream(st, feats, chunk, frames):
    """stream feats[:, :frames] through st in chunks of `chunk` feature frames; -> per-push
    (encoder ms, search ms), launches"""
    from speech_b200 import _lib
    enc, srch = [], []
    n0 = _lib.launch_count
    for p in range(0, frames, chunk):
        xs, counts = st._conv_inputs([f[p:min(p + chunk, frames)] for f in feats])
        T = max(counts)
        if T == 0:
            st._advance(xs, counts)
            continue
        e = events()
        e[0].record()
        with torch.no_grad():
            emit, Te, X = st._encode(xs, counts, T)
            if Te:
                st._fc1(X, Te)
        e[1].record()
        if Te:
            st.search.push(emit)
        e[2].record()
        e[2].synchronize()
        st._advance(xs, counts)
        enc.append(e[0].elapsed_time(e[1]))
        srch.append(e[1].elapsed_time(e[2]))
    return enc, srch, _lib.launch_count - n0


def offline_ms(m, inputs, kw):
    e = events()
    e[0].record()
    labels = m.recognize(inputs, **kw)
    e[1].record()
    e[1].synchronize()
    return e[0].elapsed_time(e[1]), labels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", default="16,128")
    ap.add_argument("--cases", default="all", help="comma-separated case indices, or all")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from speech_b200.lm import NGramLM
    print("card:", card(), flush=True)
    out = open(a.out, "w") if a.out else None
    cases = CASES if a.cases == "all" else [CASES[int(i)] for i in a.cases.split(",")]
    for V1, B, K, order in cases:
        m = model(V1)
        rng = np.random.RandomState(1)
        inputs = bench.synth_batch(B)[0][:B]
        feats = [torch.from_numpy(x).cuda() for x in inputs]
        kw = {"beam_size": K, "max_symbols_per_frame": S}
        if order:
            kw.update(lm=NGramLM.train([rng.randint(0, V1 - 1, rng.randint(5, 40)).tolist()
                                        for _ in range(2000)], order, num_classes=V1,
                                       blank=V1 - 1),
                      lm_weight=0.5, insertion_bonus=1.0)
        m.recognize([x[:200] for x in inputs], **kw)                  # warm-up
        off, want = offline_ms(m, inputs, kw)
        for chunk in [int(c) for c in a.chunks.split(",")]:
            st = m.stream(B, max_frames=300, **kw)
            run_stream(st, feats, chunk, 200)                         # warm-up: 2 s
            for b in range(B):
                st.reset(b)
            enc, srch, launches = run_stream(st, feats, chunk, bench.T_IN)
            same = st.partial() == [tuple(w) for w in want]
            total = sum(enc) + sum(srch)
            row = {"V1": V1, "B": B, "beam": K, "S": S, "lm": "%d-gram" % order if order else None,
                   "route": "full" if st.search.kp is None else "shortlist kp=%d" % st.search.kp,
                   "chunk_ms": chunk * 10, "pushes": len(enc),
                   "enc_ms": float(np.median(enc)), "search_ms": float(np.median(srch)),
                   "push_total_ms": total, "rtf": total / 1e3 / SECONDS,
                   "launches_per_push": launches / max(1, len(enc)), "offline_ms": off,
                   "equals_offline": same}
            line = json.dumps(row)
            print(line, flush=True)
            if out:
                out.write(line + "\n")
                out.flush()
        del m
        torch.cuda.empty_cache()
    if out:
        out.close()


if __name__ == "__main__":
    main()
