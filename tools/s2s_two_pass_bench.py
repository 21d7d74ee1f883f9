"""Developer tool: two-pass decoding of the attention model (Seq2Seq.recognize_two_pass and
Seq2Seq.stream), against the one-pass joint search recognize(beam_size=K, ctc_weight=0.3).

    python tools/s2s_two_pass_bench.py [--beams 4 10] [--reps N] [--out F]

The WSJ-shaped hybrid model of tools/s2s_wordlm_recognize_bench.py made unidirectional (conv +
3x GRU-512, log_t, embedding 512, CTC head, untrained) with a lookahead of tau = 4 frames, at
V = 32; B = 16 utterances of --frames input frames (default 1000, 10 s at a 10 ms hop).  Prints
the card name and power limit, then one JSON line per beam with device ms (CUDA events, median
of --reps after a warm-up) of:
  - first_ms: the first pass over precomputed CTC log-probabilities (reset, one step over all
    frames, N-best read); score_ms: the teacher-forced scoring and the selection over precomputed
    encoder states; two_pass_ms: both, from the same inputs; joint_ms: the one-pass joint search
    (beam_search_batch with the CTC head, max_len 100) on the same inputs;
  - stream_push_ms_<c>: median device ms per push of B streams fed chunks of c ms of features
    (encoder, CTC head, search step, arena append), and rescored_ms: rescored() after finish.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from s2s_recognize_bench import card  # noqa: E402

V = 32


def model(B, frames):
    import bench
    from speech_b200.models import Seq2Seq
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "exact_lengths": True,
           "encoder": {"conv": bench.WSJ_CONV, "lookahead": 4,
                       "rnn": {"dim": 512, "bidirectional": False, "layers": 3}},
           "decoder": {"embedding_dim": 512, "layers": 1, "log_t": True, "ctc_weight": 0.3}}
    m = Seq2Seq(bench.F_IN, V, cfg).cuda()
    m.set_eval()
    rng = np.random.RandomState(0)
    inputs = [rng.randn(frames, bench.F_IN).astype(np.float32) for _ in range(B)]
    return m, inputs


def device_ms(fn, reps):
    """median device ms of fn() over reps calls after one warm-up (CUDA events)"""
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def stream_pushes(m, inputs, K, chunk):
    """device ms of every push of one pass through the utterances in chunks of `chunk` input
    frames, and of rescored() after finish"""
    st = m.stream(len(inputs), beam_size=K, max_frames=1000, ctc_weight=0.3)
    ts = []
    for p in range(0, max(len(x) for x in inputs), chunk):
        chunks = [x[p:p + chunk] for x in inputs]
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        st.push(chunks)
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    st.finish()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    st.rescored()
    b.record()
    torch.cuda.synchronize()
    return ts, a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--beams", nargs="+", type=int, default=[4, 10])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--chunks-ms", nargs="+", type=int, default=[160, 1280])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from speech_b200.functions import s2s
    print("card:", card(), flush=True)
    m, inputs = model(args.batch, args.frames)
    B = args.batch
    lens = m.input_lens(inputs)
    with torch.no_grad():
        x = m._encode(m.stage_inputs(inputs), lens)
        y = torch.log_softmax(m.ctc_fc(x).float(), dim=-1).contiguous()
    lines = []
    for K in args.beams:
        def first():
            with torch.no_grad():
                return s2s.ctc_first_pass(y, lens, K)
        nbest = first()

        def second():
            with torch.no_grad():
                return s2s.rescore(m, x, nbest, lens, K, 0.3, False)

        def both():
            with torch.no_grad():
                return s2s.recognize_two_pass(m, x, y, lens, K, 0.3, False)

        def joint():
            with torch.no_grad():
                return s2s.beam_search_batch(m, x, V - 1, V - 2, K, 100, lens,
                                             ctc=(y, 0.3, min(V - 1, 3 * K // 2)))
        line = {"beam": K, "B": B, "T_frames": int(x.shape[1]), "ctc_weight": 0.3,
                "first_ms": round(device_ms(first, args.reps), 2),
                "score_ms": round(device_ms(second, args.reps), 2),
                "two_pass_ms": round(device_ms(both, args.reps), 2),
                "joint_ms": round(device_ms(joint, args.reps), 2),
                "hyp_len_max": int(nbest[1].max())}
        for c in args.chunks_ms:
            stream_pushes(m, inputs, K, c // 10)                      # warm-up
            pushes, resc = stream_pushes(m, inputs, K, c // 10)
            line["stream_push_ms_%d" % c] = round(float(np.median(pushes)), 3)
            line["stream_pushes_%d" % c] = len(pushes)
            line["rescored_ms_%d" % c] = round(resc, 2)
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump({"card": card(), "cases": lines}, fh, indent=1)


if __name__ == "__main__":
    main()
