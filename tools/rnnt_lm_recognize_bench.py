"""Developer tool: Transducer.recognize with and without shallow fusion of an n-gram LM.

    python tools/rnnt_lm_recognize_bench.py [--cases 29:1 29:4 ...] [--orders 3 5] [--reps N]
                                            [--frames N] [--out F]

The model and batch of tools/rnnt_recognize_bench.py (bench.py's RNN-T: 3x biGRU-1024 encoder,
GRU-1024 prediction network, B = 32, T' = 247) with V+1 output classes, max_symbols_per_frame = 4.
Each order's LM is NGramLM.train (interpolated Kneser-Ney) on 2000 seeded synthetic label
sequences over the V labels (a Zipf-like unigram so that contexts repeat), fused with
lm_weight 0.5 and insertion_bonus 1.0.  LM-less and LM calls alternate in one process.
Prints the card name and power limit, then one JSON line per case (V+1, beam) with, for the
LM-less call and for each order:
  - ms per recognize call, device-timed (CUDA events around the call; median of --reps);
  - launches per frame (C-ABI launches of one call over T');
  - the device-time split from torch.profiler in a run of its own: the prediction step, the GEMMs,
    the joint's row kernels, the LM-fused rows (sb_rnnt_search_lm_rows) and the other search
    kernels;
  - rerun: utterances the shortlist route searched again from 64-entry lists.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from rnnt_recognize_bench import card, model_and_batch  # noqa: E402


def synthetic_lm(V1, order, n=2000, seed=0):
    from speech_b200.lm import NGramLM
    rng = np.random.RandomState(seed)
    w = 1.0 / np.arange(1, V1) ** 1.1
    w /= w.sum()
    seqs = [rng.choice(V1 - 1, rng.randint(5, 60), p=w).tolist() for _ in range(n)]
    return NGramLM.train(seqs, order, V1, V1 - 1)


def split(names_times):
    out = {"pred_step": 0.0, "gemm": 0.0, "joint_rows": 0.0, "lm_rows": 0.0, "search": 0.0,
           "other": 0.0}
    for name, us in names_times.items():
        n = name.lower()
        part = ("pred_step" if "pred_step" in n else "lm_rows" if "lm_rows" in n else
                "gemm" if "gemm" in n else
                "joint_rows" if "joint" in n or "shortlist_rows" in n else
                "search" if "search" in n else "other")
        out[part] += us
    return {k: round(v / 1000.0, 3) for k, v in out.items()}


class RerunCount:
    """counts the utterances search_batch sends to the 64-entry rerun (wraps _search_once)"""

    def __init__(self):
        from speech_b200 import transducer_decoders as td
        self.td, self.inner, self.n = td, td._search_once, 0
        td._search_once = self

    def __call__(self, provider, tl, T, K, S, max_len, L, blank, kp, fusion=None):
        out = self.inner(provider, tl, T, K, S, max_len, L, blank, kp, fusion)
        if kp is not None and kp != self.td.SHORTLIST_RERUN:
            self.n += sum(1 for f in out[2] if f)
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", default=["29:1", "29:4", "29:8", "1024:4", "4096:4"])
    ap.add_argument("--orders", nargs="+", type=int, default=[3, 5])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=0)
    ap.add_argument("--lm-weight", type=float, default=0.5)
    ap.add_argument("--insertion-bonus", type=float, default=1.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from speech_b200 import _lib
    from speech_b200.models.transducer_model import PredictionRows
    from torch.profiler import ProfilerActivity, profile
    print("card:", card(), flush=True)
    reruns = RerunCount()
    lines = []
    for case in args.cases:
        V1, beam = (int(v) for v in case.split(":"))
        m, batch = model_and_batch(V1, args.frames)
        inputs = batch[0]
        T = PredictionRows(m, inputs[:1]).T
        variants = [("none", {})] + [
            ("%d-gram" % o, {"lm": synthetic_lm(V1, o), "lm_weight": args.lm_weight,
                             "insertion_bonus": args.insertion_bonus}) for o in args.orders]
        for _, kw in variants:                                        # warm-up
            m.recognize(inputs, beam_size=beam, **kw)
        torch.cuda.synchronize()
        times = {name: [] for name, _ in variants}
        launches, rerun = {}, {}
        for _ in range(args.reps):                                    # alternated
            for name, kw in variants:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                n0, r0 = _lib.launch_count, reruns.n
                torch.cuda.synchronize()
                e0.record()
                m.recognize(inputs, beam_size=beam, **kw)
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1))
                launches[name] = _lib.launch_count - n0
                rerun[name] = reruns.n - r0
        rec = {"V1": V1, "beam": beam, "B": len(inputs), "T_frames": T,
               "lm_weight": args.lm_weight, "insertion_bonus": args.insertion_bonus}
        for name, kw in variants:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                m.recognize(inputs, beam_size=beam, **kw)
                torch.cuda.synchronize()
            kern = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" and e.device_time_total:
                    kern[e.key] = kern.get(e.key, 0.0) + e.device_time_total
            ms = sorted(times[name])[len(times[name]) // 2]
            rec[name] = {"ms": round(ms, 2), "launches_per_frame": round(launches[name] / T, 1),
                         "split_ms": split(kern), "rerun_utterances": rerun[name]}
        base = rec["none"]["ms"]
        for name, _ in variants[1:]:
            rec[name]["x_lm_less"] = round(rec[name]["ms"] / base, 3)
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del m
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump({"card": card(), "cases": lines}, fh, indent=1)


if __name__ == "__main__":
    main()
