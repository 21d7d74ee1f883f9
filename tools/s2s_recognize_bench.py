"""Developer tool: Seq2Seq.recognize (beam search of a whole minibatch) against a Python loop of
Seq2Seq.beam_search over the same utterances.

    python tools/s2s_recognize_bench.py [--cases 32:1 32:4 ...] [--reps N] [--max-len N] [--out F]

The WSJ-shaped attention model of bench.py's other_config_measurements (conv + 3x biGRU-512,
log_t, embedding 512) with V tokens, B = 16 utterances of T = 800 input frames, max_len = 100.
Prints the card name and power limit, then one JSON line per case (V, beam) with:
  - utt/s of recognize (one call for the 16 utterances) and of the loop (16 beam_search calls,
    each encoding its own utterance), both from the host clock between synchronisations, median
    of --reps after one warm-up;
  - the same for the search alone on precomputed encoder states: beam_search_batch on (B, T', H)
    against 16 calls on (1, T', H) slices (the encoder's share of the above is the difference);
  - routes: whether the attention kernel projects (fc_fused) and whether the selection is split;
  - steps each utterance's own search ran, the steps the batch ran (its last utterance's), and
    the share of row-steps spent on utterances that had already stopped: their K rows stay in the
    cell and attention kernels until the whole batch stops.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def model_and_inputs(V, B, frames):
    import bench
    from speech_b200.models import Seq2Seq
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": bench.WSJ_CONV,
                                       "rnn": {"dim": 512, "bidirectional": True, "layers": 3}},
           "decoder": {"embedding_dim": 512, "layers": 1, "log_t": True}}
    m = Seq2Seq(bench.F_IN, V, cfg).cuda()
    m.set_eval()
    rng = np.random.RandomState(0)
    inputs = [rng.randn(frames, bench.F_IN).astype(np.float32) for _ in range(B)]
    return m, inputs


def timed(fn, reps):
    fn()                                           # warm-up
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", default=["32:1", "32:4", "32:8",
                                                   "5000:1", "5000:4", "5000:8"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--max-len", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from speech_b200.functions import s2s
    print("card:", card(), flush=True)
    lines = []
    for case in args.cases:
        V, K = (int(v) for v in case.split(":"))
        B, L = args.batch, args.max_len
        m, inputs = model_and_inputs(V, B, args.frames)
        start, end = V - 1, V - 2
        singles = [([x], [[start, end]]) for x in inputs]
        with torch.no_grad():
            x_enc = m.encode(m.stage_inputs(inputs))

        def batched():
            m.recognize(inputs, beam_size=K, max_len=L)

        def loop():
            for one in singles:
                m.beam_search(one, beam_size=K, max_len=L)

        def search_batched():
            with torch.no_grad():
                s2s.beam_search_batch(m, x_enc, start, end, K, L)

        def search_loop():
            with torch.no_grad():
                for b in range(B):
                    s2s.beam_search_batch(m, x_enc[b:b + 1], start, end, K, L)

        t_rec, t_loop = timed(batched, args.reps), timed(loop, args.reps)
        t_sb, t_sl = timed(search_batched, args.reps), timed(search_loop, args.reps)
        with torch.no_grad():
            res = s2s.beam_search_batch(m, x_enc, start, end, K, L)
        steps = [r[2] for r in res]
        run = max(steps)
        idle = sum(run - s for s in steps) / float(run * B)
        rec = {"V": V, "beam": K, "B": B, "T_frames": int(x_enc.shape[1]), "max_len": L,
               "fc_fused": s2s.fc_fused(x_enc.shape[2], V - 1),
               "split_select": not s2s.beam_select_fits(K, V - 1),
               "recognize_utt_per_s": round(B / t_rec, 2),
               "loop_utt_per_s": round(B / t_loop, 2),
               "speedup": round(t_loop / t_rec, 2),
               "search_batched_utt_per_s": round(B / t_sb, 2),
               "search_loop_utt_per_s": round(B / t_sl, 2),
               "search_speedup": round(t_sl / t_sb, 2),
               "utt_steps": steps, "batch_steps": run,
               "stopped_row_step_share": round(idle, 4)}
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
