"""Developer tool: the RNN-T joint + lattice loss at the benchmark's RNN-T shape over a range of
vocabularies (V+1 = 64 runs the resident-weight kernel of csrc/joint.cu, larger ones the slab path
of csrc/joint_vocab.cu), against a materialised PyTorch joint of the same shape.

    python tools/joint_vocab_bench.py [--out FILE.json] [--vocab 64 128 256 1024 4096]

Shape: B = 32, T' = 247 frames (1000 input frames after the conv stack), U+1 = 100 (labels of
40-100), H = 1024.  Per vocabulary it prints the device time of loss (forward) and backward (CUDA
events over warmed repeats), their split between GEMMs and the row / slab kernels, the achieved
TFLOP/s of the four GEMM passes (forward, recompute, dW2, dz; 2 * nodes * H * V1 FLOPs each) over
the 989 TFLOP/s dense-BF16 data-sheet figure of the H100 SXM, the host enqueue time of one step,
the peak memory, and a sweep of the slab size Tc.  The card's name and power limit are read in the
same run.  Needs a CUDA device."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from speech_b200 import ops                                       # noqa: E402
from speech_b200.functions import transducer                      # noqa: E402

B, T, U1, H = 32, 247, 100, 1024
PEAK_TFLOPS = 989.0


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(), "nvidia_smi": q.stdout.strip()}


def inputs(V1, seed=0):
    rng = np.random.RandomState(seed)
    dev = "cuda"
    fx = torch.from_numpy(rng.randn(B, T, H).astype(np.float32) * 0.5).to(dev).requires_grad_(True)
    fy = torch.from_numpy(rng.randn(B, U1, H).astype(np.float32) * 0.5).to(dev).requires_grad_(True)
    w2 = torch.from_numpy((rng.randn(V1, H) / np.sqrt(H)).astype(np.float32)).to(dev)
    w2.requires_grad_(True)
    b2 = torch.zeros(V1, device=dev, requires_grad=True)
    ylen = rng.randint(40, U1, size=B).astype(np.int32)
    ylen[0] = U1 - 1
    ymat = rng.randint(0, V1 - 1, size=(B, U1 - 1))
    flat = np.concatenate([ymat[b, :ylen[b]] for b in range(B)]).astype(np.int32)
    xlen = np.full(B, T, np.int32)
    return (fx, fy, w2, b2, torch.from_numpy(ymat), torch.from_numpy(flat), torch.from_numpy(xlen),
            torch.from_numpy(ylen))


def step(args):
    loss = transducer.JointTransducerLoss()(*args)
    loss.backward()
    return loss


def time_ours(args, reps):
    """-> forward ms, backward ms (device events), host enqueue ms of one step, peak MB"""
    for _ in range(2):
        step(args)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    fwd = bwd = enq = 0.0
    for _ in range(reps):
        torch.cuda.synchronize()
        h0 = time.perf_counter()
        ev[0].record()
        loss = transducer.JointTransducerLoss()(*args)
        ev[1].record()
        loss.backward()
        ev[2].record()
        enq += time.perf_counter() - h0
        torch.cuda.synchronize()
        fwd += ev[0].elapsed_time(ev[1])
        bwd += ev[1].elapsed_time(ev[2])
    for a in args[:4]:
        a.grad = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    step(args)
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2**20
    return fwd / reps, bwd / reps, enq / reps * 1e3, peak


def kernel_split(args, V1):
    """Per-launch CUDA events (a run of its own): device ms per kernel class, GEMM passes apart."""
    ops._prof_detail = True
    ops.profile_begin()
    loss = transducer.JointTransducerLoss()(*args)
    fwd = ops.profile_end()
    ops.profile_begin()
    loss.backward()
    bwd = ops.profile_end()
    ops._prof_detail = False
    nodes = B * T * U1
    res = {"gemm_ms": 0.0, "rows_ms": 0.0, "slab_ms": 0.0, "resident_joint_ms": 0.0,
           "lattice_loss_ms": 0.0, "gemm_passes": {}}
    for phase, prof in (("forward", fwd), ("backward", bwd)):
        for name, (n, ms, fl) in prof.items():
            if name.startswith("gemm"):
                res["gemm_ms"] += ms
                if " acc" in name:
                    key = "dW2"
                elif " bT" in name:
                    key = "dz"
                else:
                    key = "forward" if phase == "forward" else "recompute"
                p = res["gemm_passes"].setdefault(key, {"ms": 0.0, "launches": 0})
                p["ms"] += ms
                p["launches"] += n
            elif name == "rnnt_joint_rows":
                res["rows_ms"] += ms
            elif name == "rnnt_joint_slab":
                res["slab_ms"] += ms
            elif name == "rnnt_joint":
                res["resident_joint_ms"] += ms
            else:
                res["lattice_loss_ms"] += ms
    flops = 2.0 * nodes * H * V1
    for p in res["gemm_passes"].values():
        p["tflops"] = flops / p["ms"] / 1e9
        p["share_of_989"] = p["tflops"] / PEAK_TFLOPS
    return res


def torch_yardstick(args, V1, reps=3):
    """Materialised joint in PyTorch (bf16 relu(fx + fy), matmul, fp32 log_softmax, gather of the
    blank / label columns, sum) forward + backward: device ms and peak MB."""
    fx, fy, w2, b2, ymat = args[:5]
    lab = torch.cat([ymat, torch.zeros(B, 1, dtype=ymat.dtype)], 1).cuda()
    idx = torch.stack([torch.full_like(lab, V1 - 1), lab], -1)[:, None].expand(B, T, U1, 2)

    def run():
        z = torch.relu(fx.bfloat16()[:, :, None] + fy.bfloat16()[:, None])
        lp = torch.log_softmax((z @ w2.bfloat16().t() + b2.bfloat16()).float(), -1)
        lp.gather(3, idx).sum().backward()
    try:
        run()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            run()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        for a in args[:4]:
            a.grad = None
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        run()
        torch.cuda.synchronize()
        peak = (torch.cuda.max_memory_allocated() - base) / 2**20
        return {"fwd_bwd_ms": ms, "peak_MB": peak}
    except torch.cuda.OutOfMemoryError as e:
        return {"error": "out of memory: %s" % str(e).splitlines()[0]}
    finally:
        for a in args[:4]:
            a.grad = None
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vocab", type=int, nargs="+", default=[64, 128, 256, 1024, 4096])
    ap.add_argument("--sweep", type=int, nargs="+", default=[1024, 4096],
                    help="vocabularies at which Tc in {1, 2, 4, 8} is swept")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("joint_vocab_bench: needs a CUDA device")
    out = {"card": card(), "shape": {"B": B, "T": T, "U1": U1, "H": H}, "vocab": {}}
    print(json.dumps(out["card"]), flush=True)
    default_frames = transducer.joint_vocab_slab_frames
    for V1 in a.vocab:
        args = inputs(V1)
        fwd, bwd, enq, peak = time_ours(args, a.reps)
        r = {"path": "resident" if V1 <= transducer.JOINT_RESIDENT_MAX_CLASSES else "slab",
             "Tc": min(default_frames(B, U1, V1), T), "fwd_ms": fwd, "bwd_ms": bwd,
             "device_ms": fwd + bwd, "host_enqueue_ms": enq, "peak_MB": peak}
        r["split"] = kernel_split(args, V1)
        if V1 in a.sweep and r["path"] == "slab":
            r["tc_sweep"] = {}
            for tc in (1, 2, 4, 8):
                transducer.joint_vocab_slab_frames = lambda *_, tc=tc: tc
                f, b, e, p = time_ours(args, a.reps)
                r["tc_sweep"][tc] = {"fwd_ms": f, "bwd_ms": b, "device_ms": f + b,
                                     "host_enqueue_ms": e, "peak_MB": p}
                transducer.joint_vocab_slab_frames = default_frames
        r["torch_yardstick"] = torch_yardstick(args, V1)
        out["vocab"][V1] = r
        print("V1=%d %s" % (V1, json.dumps(r)), flush=True)
        del args
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
