"""Cost of the exact-lengths mode: ms per training step (zero_grad -> loss -> backward -> clip +
SGD, device events) of the north-star CTC step (B=64) and of the RNN-T configuration (B=32) in
three cases:
  default   the reference's padded semantics
  equal     exact_lengths on, every utterance T=1000 frames (the alignment is skipped)
  mixed     exact_lengths on, input lengths drawn from 600..1000 (one utterance at 1000, so the
            padded shape is that of the other two cases)
plus, from a separate profiled step of the mixed case, the device time of the time_align kernels.

    python tools/exact_lengths_bench.py [--steps N] [--warmup W] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def batch(nutt, lens, vocab, label_range, seed):
    rng = np.random.RandomState(seed)
    inputs = [rng.randn(n, 80).astype(np.float32) for n in lens]
    labels = [rng.randint(0, vocab, size=rng.randint(*label_range)).tolist() for _ in range(nutt)]
    return tuple(inputs), tuple(labels)


def time_steps(m, b, steps, warm):
    from speech_b200 import ops
    from speech_b200.optim import FlatSGD
    m.set_train()
    opt = FlatSGD(m, lr=1e-4, momentum=0.0, max_grad_norm=200.0)

    def step():
        opt.zero_grad()
        loss = m.loss(b)
        loss.backward()
        opt.step()
        return loss
    for _ in range(warm):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    ops.profile_begin()
    step()
    prof = ops.profile_end()
    align = prof.get("time_align", (0, 0.0, 0.0))
    return {"ms_per_step": round(ms, 3), "loss": float(loss.item()),
            "time_align_launches": align[0], "time_align_ms": round(align[1], 3)}


def workload(name, exact):
    from speech_b200.models import CTC, Transducer
    import bench
    torch.manual_seed(0)
    if name == "ctc_northstar_B64":
        cfg = dict(bench.MODEL_CFG, exact_lengths=exact)
        return CTC(bench.F_IN, bench.VOCAB, cfg).cuda(), 64, (40, 121)
    cfg = {"dropout": 0.0, "exact_lengths": exact,
           "encoder": {"conv": bench.WSJ_CONV,
                       "rnn": {"dim": 1024, "bidirectional": True, "layers": 3}},
           "decoder": {"embedding_dim": 256, "layers": 1}}
    return Transducer(bench.F_IN, bench.VOCAB, cfg).cuda(), 32, (40, 100)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("exact_lengths_bench: needs a CUDA device")
    res = {"card": card()}
    for name in ("ctc_northstar_B64", "rnnt_B32"):
        rows = {}
        for case in ("default", "equal", "mixed"):
            m, nutt, lab = workload(name, case != "default")
            if case == "mixed":
                lens = [1000] + np.random.RandomState(7).randint(600, 1001, nutt - 1).tolist()
            else:
                lens = [1000] * nutt
            rows[case] = time_steps(m, batch(nutt, lens, 28, lab, 1), args.steps, args.warmup)
            del m
            torch.cuda.empty_cache()
        d = rows["default"]["ms_per_step"]
        for case in ("equal", "mixed"):
            rows[case]["vs_default"] = round(rows[case]["ms_per_step"] / d - 1.0, 4)
        res[name] = rows
    txt = json.dumps(res, indent=1)
    print(txt)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(txt + "\n")


if __name__ == "__main__":
    main()
