"""Developer tool: joint CTC/attention decoding and training of the attention model.

    python tools/s2s_ctc_recognize_bench.py [--vocab 33 1001] [--beam 10] [--reps N] [--out F]
                                            [--profile DIR]

The WSJ-shaped attention model of tools/s2s_recognize_bench.py (conv + 3x biGRU-512, log_t,
embedding 512) with a CTC head, B = 16 utterances of T = 800 input frames (T' = 197),
max_len = 100.  Prints the card name and power limit, then one JSON line per vocabulary with:
  - recognize time at ctc_weight = 0 and at 0.3 for the default pre-beam M = min(V-1, 3K/2) and,
    where V - 1 <= 128, for M = V - 1 (median of --reps after one warm-up, host clock between
    synchronisations);
  - one loss + backward with and without the head (same weights otherwise);
  - the steps the batch's search ran at ctc_weight = 0 and 0.3 (the default M);
  - with --profile, a separate torch.profiler run of recognize at ctc_weight = 0.3 and the default
    M: the CUDA time of the candidate, selection and extension kernels, and of every kernel.
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


def model(V, w, B, frames):
    import bench
    from speech_b200.models import Seq2Seq
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": bench.WSJ_CONV,
                                       "rnn": {"dim": 512, "bidirectional": True, "layers": 3}},
           "decoder": {"embedding_dim": 512, "layers": 1, "log_t": True, "ctc_weight": w}}
    m = Seq2Seq(bench.F_IN, V, cfg).cuda()
    rng = np.random.RandomState(0)
    inputs = [rng.randn(frames, bench.F_IN).astype(np.float32) for _ in range(B)]
    labels = [[V - 1] + rng.randint(0, V - 2, 60).tolist() + [V - 2] for _ in range(B)]
    return m, inputs, labels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vocab", nargs="+", type=int, default=[33, 1001])
    ap.add_argument("--beam", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--frames", type=int, default=800)
    ap.add_argument("--max-len", type=int, default=100)
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default=None)
    args = ap.parse_args()
    print("card:", card(), flush=True)
    K = args.beam
    lines = []
    for V in args.vocab:
        m, inputs, labels = model(V, 0.3, args.batch, args.frames)
        m.set_eval()
        rec = dict(V=V, K=K, B=args.batch, frames=args.frames, max_len=args.max_len)

        def run(w, M=None):
            return lambda: m.recognize(inputs, beam_size=K, max_len=args.max_len, ctc_weight=w,
                                       ctc_prebeam=M)
        rec["recognize_s_w0"] = timed(run(0.0), args.reps)
        rec["M_default"] = min(V - 1, 3 * K // 2)
        rec["recognize_s_w03_Mdefault"] = timed(run(0.3), args.reps)
        if V - 1 <= 128:
            rec["recognize_s_w03_MC"] = timed(run(0.3, V - 1), args.reps)
        # steps the batch's search ran (its last utterance's), which the weight changes too
        from speech_b200.functions import s2s
        with torch.no_grad():
            x = m._encode(m.stage_inputs(inputs), None)
            y = torch.log_softmax(m.ctc_fc(x).float(), dim=-1).contiguous()
            for key, ctc in (("steps_w0", None), ("steps_w03", (y, 0.3, rec["M_default"]))):
                res = s2s.beam_search_batch(m, x, V - 1, V - 2, K, args.max_len, ctc=ctc)
                rec[key] = max(r[2] for r in res)
        m.set_train()
        m.scheduled_sampling = False

        def step(w):
            def f():
                m.ctc_weight = w
                m.zero_grad(set_to_none=True)
                m.loss((inputs, labels)).backward()
            return f
        rec["loss_bwd_s_head"] = timed(step(0.3), args.reps)
        rec["loss_bwd_s_nohead"] = timed(step(0.0), args.reps)   # the head's module stays idle
        m.ctc_weight = 0.3
        m.set_eval()
        if args.profile:
            from torch.profiler import ProfilerActivity, profile
            run(0.3)()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run(0.3)()
                torch.cuda.synchronize()
            tot = 0.0
            parts = {"candidate": 0.0, "select": 0.0, "extend": 0.0}
            for ev in prof.key_averages():
                t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
                if ev.key.startswith("void") or "kernel" in ev.key:
                    tot += t
                    for name, kern in (("candidate", "s2s_ctc_cand"), ("select", "s2s_ctc_select"),
                                       ("extend", "s2s_ctc_extend")):
                        if kern in ev.key:
                            parts[name] += t
            for name, t in parts.items():
                rec["profile_%s_us" % name] = t
            rec["profile_all_kernels_us"] = tot
            os.makedirs(args.profile, exist_ok=True)
            prof.export_chrome_trace(os.path.join(args.profile, "s2s_ctc_V%d.json" % V))
        line = json.dumps(rec)
        print(line, flush=True)
        lines.append(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write("card: %s\n" % card() + "\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
