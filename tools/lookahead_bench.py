"""Developer tool: cost of the lookahead convolution (csrc/lookahead.cu) on the GPU.

    python tools/lookahead_bench.py [--reps N] [--steps N] [--out F]

Prints the card name and power limit, then one JSON line per case:
  kernel   sb_lookahead_fwd (fp32 r) and sb_lookahead_bwd (dh + dW, the reduction included) at
           B = 64, T' = 247, H = 1024, tau in {2, 5, 10, 20}: device us per call (CUDA events over
           --reps calls), and the bytes the algorithm must move (fwd: read h, write r; bwd: read
           dr and h, write dh) over that time as a share of the H100 SXM data-sheet 3.35 TB/s
  train    one training step (loss + backward) of bench.py's CTC encoder made unidirectional
           (conv [[32,5,8,2],[32,5,8,2]], 5 x GRU-1024, B = 64, 1000 input frames), tau 0 and 5:
           median device ms over --steps steps
  stream   CTC.stream at 16 streams, beam 8, 160 ms chunks (16 feature frames) of 10 s utterances,
           tau 0 and 5: median device ms per push, and the finish() call
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

HBM = 3.35e12


def cfg(tau):
    enc = {"conv": [[32, 5, 8, 2], [32, 5, 8, 2]],
           "rnn": {"dim": 1024, "bidirectional": False, "layers": 5}}
    if tau:
        enc["lookahead"] = tau
    return {"dropout": 0.0, "encoder": enc}


def timed(fn, reps):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernels(reps, emit):
    from speech_b200 import ops
    B, T, H = 64, 247, 1024
    g = torch.Generator(device="cuda").manual_seed(0)
    h = torch.randn(T * B, H, device="cuda", generator=g)
    dr = torch.randn(T * B, H, device="cuda", generator=g)
    r = torch.empty_like(h)
    for tau in (2, 5, 10, 20):
        w = torch.randn(tau + 1, H, device="cuda", generator=g)
        fwd = timed(lambda: ops.lookahead_fwd(h, w, None, r, None, T, B, H, tau), reps)
        bwd = timed(lambda: ops.lookahead_bwd(dr, h, w, None, T, B, H, tau), reps)
        n = T * B * H
        emit({"case": "kernel", "tau": tau, "fwd_us": round(fwd * 1e3, 2),
              "bwd_us": round(bwd * 1e3, 2),
              "fwd_hbm_share": round(8 * n / (fwd * 1e-3) / HBM, 3),
              "bwd_hbm_share": round(12 * n / (bwd * 1e-3) / HBM, 3)})


def train(steps, emit):
    from speech_b200.models import CTC
    inputs, labels = bench.synth_batch(bench.GLOBAL_B)
    for tau in (0, 5):
        torch.manual_seed(0)
        m = CTC(bench.F_IN, bench.VOCAB, cfg(tau)).cuda()
        batch = (inputs, labels)
        times = []
        for i in range(steps + 2):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            m.loss(batch).backward()
            e1.record()
            torch.cuda.synchronize()
            m.zero_grad(set_to_none=True)
            if i >= 2:
                times.append(e0.elapsed_time(e1))
        emit({"case": "train", "tau": tau, "B": bench.GLOBAL_B,
              "step_ms": round(float(np.median(times)), 3)})


def stream(emit):
    from speech_b200.models import CTC
    B, chunk = 16, 16
    rng = np.random.RandomState(0)
    feats = [rng.randn(bench.T_IN, bench.F_IN).astype(np.float32) for _ in range(B)]
    for tau in (0, 5):
        torch.manual_seed(0)
        m = CTC(bench.F_IN, bench.VOCAB, cfg(tau)).cuda()
        m.set_eval()
        st = m.stream(B, beam_size=8, max_frames=300)
        for warm in (True, False):
            for b in range(B):
                st.reset(b)
            times = []
            for p in range(0, bench.T_IN, chunk):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                st.push([f[p:p + chunk] for f in feats])
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            st.finish()
            e1.record()
            torch.cuda.synchronize()
        emit({"case": "stream", "tau": tau, "streams": B, "chunk_ms": chunk * 10,
              "push_ms": round(float(np.median(times)), 3),
              "finish_ms": round(e0.elapsed_time(e1), 3), "frames": st.frames[0]})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lookahead_bench needs a CUDA device")
    from speech_b200 import _lib
    _lib.load()
    lines = ["card: " + card()]
    print(lines[0], flush=True)

    def emit(d):
        s = json.dumps(d)
        print(s, flush=True)
        lines.append(s)
    kernels(a.reps, emit)
    train(a.steps, emit)
    stream(emit)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
