"""Developer tool: Transducer.recognize (label-free beam search) on the benchmark's RNN-T model.

    python tools/rnnt_recognize_bench.py [--cases 29:1 29:4 ...] [--reps N] [--frames N] [--out F]

bench.py's rnnt_workload (3x biGRU-1024 encoder, GRU-1024 prediction network, embedding 256, B = 32,
T = 1000 input frames, T' = 247) with V+1 output classes, max_symbols_per_frame = 4.  Prints the
card name and power limit, then one JSON line per case (V+1, beam) with:
  - ms per recognize call, device-timed (CUDA events around the call; median of --reps calls after
    one warm-up), and host_ms, the host clock around the same calls: a call ends in the copy of
    its results, so host_ms exceeds the device time only where enqueueing is the slower of the two;
  - launches per frame (C-ABI launches of one call over T');
  - the device-time split between the prediction step (sb_rnnt_pred_step), the GEMMs (fc1 of the
    new states; on the large-vocabulary route also the joint's logits), the joint's row kernels and
    the search kernels, from torch.profiler in a run of its own, and every kernel
    name that profile lists on the recognize path (no cuBLAS / cuDNN kernel is expected);
  - infer_ms: Transducer.infer (teacher-forced lattice) on the same batch, beam and vocabulary, as
    a yardstick.
--frames N cuts the inputs to N input frames (a quick run).
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


def model_and_batch(V1, frames):
    import bench
    from speech_b200.models import Transducer
    m, batch = bench.rnnt_workload(32, 0)
    if V1 != bench.VOCAB + 1:
        torch.manual_seed(0)
        cfg = {"dropout": 0.0, "encoder": {"conv": bench.WSJ_CONV,
                                           "rnn": {"dim": 1024, "bidirectional": True, "layers": 3}},
               "decoder": {"embedding_dim": 256, "layers": 1}}
        m = Transducer(bench.F_IN, V1 - 1, cfg).cuda()
        rng = np.random.RandomState(3)
        batch = (batch[0], tuple(rng.randint(0, V1 - 1, size=len(l)).tolist() for l in batch[1]))
    if frames:
        batch = (tuple(x[:frames] for x in batch[0]), batch[1])
    m.set_eval()
    return m, batch


def split(names_times):
    """device ms per part: the prediction GRU step, the GEMMs (fc1 of the new states and, on the
    large-vocabulary route, the joint's logits), the joint's row kernels, the search kernels"""
    out = {"pred_step": 0.0, "gemm": 0.0, "joint_rows": 0.0, "search": 0.0, "other": 0.0}
    for name, us in names_times.items():
        n = name.lower()
        part = ("pred_step" if "pred_step" in n else "gemm" if "gemm" in n else
                "joint_rows" if "joint" in n or "shortlist_rows" in n else
                "search" if "search" in n else "other")
        out[part] += us
    return {k: round(v / 1000.0, 3) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="+", default=["29:1", "29:4", "29:8", "1024:4", "4096:4"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from speech_b200 import _lib
    print("card:", card(), flush=True)
    lines = []
    for case in args.cases:
        V1, beam = (int(v) for v in case.split(":"))
        m, batch = model_and_batch(V1, args.frames)
        inputs = batch[0]
        m.recognize(inputs, beam_size=beam)                   # warm-up
        torch.cuda.synchronize()
        dev_ms, host_ms, launches = [], [], []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n0 = _lib.launch_count
            torch.cuda.synchronize()
            e0.record()
            h0 = time.perf_counter()
            m.recognize(inputs, beam_size=beam)
            e1.record()
            torch.cuda.synchronize()
            host_ms.append((time.perf_counter() - h0) * 1e3)
            dev_ms.append(e0.elapsed_time(e1))
            launches.append(_lib.launch_count - n0)
        from speech_b200.models.transducer_model import PredictionRows
        T = PredictionRows(m, inputs[:1]).T
        m.infer(batch, beam_size=beam)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.infer(batch, beam_size=beam)
        torch.cuda.synchronize()
        infer_ms = (time.perf_counter() - t0) * 1e3
        # device-time split, in a run of its own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            m.recognize(inputs, beam_size=beam)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():                  # device-side events: the kernels
            if e.device_type.name == "CUDA" and e.device_time_total:
                kern[e.key] = kern.get(e.key, 0.0) + e.device_time_total
        vendor = [k for k in kern if any(s in k.lower() for s in ("cublas", "cudnn", "gemv",
                                                                  "sgemm", "cutlass"))]
        rec = {"V1": V1, "beam": beam, "B": len(inputs), "T_frames": T,
               "ms": round(sorted(dev_ms)[len(dev_ms) // 2], 2),
               "host_ms": round(sorted(host_ms)[len(host_ms) // 2], 2),
               "launches_per_frame": round(launches[0] / max(T, 1), 1),
               "split_ms": split(kern), "vendor_kernels": vendor,
               "kernels": sorted(kern, key=lambda k: -kern[k])[:12],
               "infer_ms": round(infer_ms, 2)}
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
