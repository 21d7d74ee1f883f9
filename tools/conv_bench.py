"""Second conv layer of the benchmark's front-end (B = 64, T = 1000: P1 is 64 x 498 x 37 x 32 f32,
kernel 5 x 8, stride 2, 32 -> 32 channels) per pass, im2col + GEMM against the direct-convolution
kernels: device time (CUDA events), the algorithmic HBM bytes of the pass, achieved GB/s and its
share of the H100 SXM data-sheet 3.35 TB/s.

    python tools/conv_bench.py [--reps N] [--B B] [--T T]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from speech_b200 import _lib, ops  # noqa: E402

HBM_PEAK = 3.35e12      # bytes/s, NVIDIA H100 SXM data sheet (not a measured peak)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return out.stdout.strip().splitlines()[0]
    except Exception as e:   # the GPU name from torch is still worth printing
        return "%s (nvidia-smi: %r)" % (torch.cuda.get_device_name(), e)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--B", type=int, default=64)
    ap.add_argument("--T", type=int, default=1000)
    args = ap.parse_args()
    lib = _lib.load()
    sp = _lib.stream_ptr()
    torch.manual_seed(0)
    B, Ci, Co, kh, kw, s = args.B, 32, 32, 5, 8, 2
    Ti, Fi = (args.T - 5) // 2 + 1, 37
    To, Fo = (Ti - kh) // s + 1, (Fi - kw) // s + 1
    K = kh * kw * Ci
    M, Mp = B * To * Fo, B * Ti * Fi
    dev = "cuda"
    P = torch.randn(Mp, Ci, device=dev)
    Wp = (torch.randn(Co, K, device=dev) * 0.05).bfloat16()
    bias = torch.randn(Co, device=dev)
    dC = (torch.randn(M, Co, device=dev) * 0.1).bfloat16()
    A = torch.empty(M, K, dtype=torch.bfloat16, device=dev)
    C = torch.empty(M, Co, device=dev)
    dCp = torch.empty(Mp, Ci, dtype=torch.bfloat16, device=dev)
    db = torch.zeros(Ci, device=dev)
    dWT = torch.zeros(K, Co, device=dev)

    def check(rc, name):
        _lib.check(rc, name)

    def im2col():
        check(lib.sb_conv_im2col(P.data_ptr(), None, 1.0, A.data_ptr(), B, Ti, Fi, Ci, kh, kw, s,
                                 K, 1, sp), "im2col")

    def fwd_old():
        im2col()
        ops.gemm_bf16_tn(A, Wp, out=C, bias=bias)

    def fwd_new():
        check(lib.sb_conv_fwd_direct(P.data_ptr(), None, 1.0, Wp.data_ptr(), K, bias.data_ptr(),
                                     C.data_ptr(), B, Ti, Fi, Ci, Co, kh, kw, s, sp), "fwd_direct")

    def dgrad_old():
        dA = ops.gemm_bf16_tn(dC, Wp, b_mn=True)
        check(lib.sb_conv_col2im_relu(dA.data_ptr(), dA.stride(0), P.data_ptr(), None, 1.0,
                                      dCp.data_ptr(), db.data_ptr(), B, Ti, Fi, Ci, kh, kw, s, sp),
              "col2im")

    def dgrad_new():
        check(lib.sb_conv_dgrad_direct(dC.data_ptr(), Wp.data_ptr(), K, P.data_ptr(), None, 1.0,
                                       dCp.data_ptr(), db.data_ptr(), B, Ti, Fi, Ci, Co, kh, kw, s,
                                       sp), "dgrad_direct")

    def wgrad_old():    # the patch matrix A is already there, saved by the forward
        ops.gemm_bf16_tn(A, dC, out=dWT, accumulate=True, a_mn=True, b_mn=True)

    def wgrad_new():
        check(lib.sb_conv_wgrad_direct(P.data_ptr(), None, 1.0, dC.data_ptr(), dWT.data_ptr(), B,
                                       Ti, Fi, Ci, Co, kh, kw, s, sp), "wgrad_direct")

    # least HBM traffic of each pass: its inputs read once, its outputs written once
    fbytes = {"forward": Mp * Ci * 4 + M * Co * 4 + Co * K * 2,
              "dgrad": M * Co * 2 + Mp * Ci * 4 + Mp * Ci * 2 + Co * K * 2,
              "wgrad": Mp * Ci * 4 + M * Co * 2 + K * Co * 4}
    res = {"card": card(), "shape": {"B": B, "Ti": Ti, "Fi": Fi, "Ci": Ci, "Co": Co, "kh": kh,
                                     "kw": kw, "stride": s, "M": M}, "passes": {}}
    im2col()
    for name, old, new in (("forward", fwd_old, fwd_new), ("dgrad", dgrad_old, dgrad_new),
                           ("wgrad", wgrad_old, wgrad_new)):
        r = {"bytes": fbytes[name]}
        for tag, fn in (("im2col_gemm", old), ("direct", new)):
            ms = timed(fn, args.reps)
            r[tag] = {"ms": ms, "GB_s": fbytes[name] / (ms * 1e-3) / 1e9,
                      "frac_of_3.35TB_s": fbytes[name] / (ms * 1e-3) / HBM_PEAK}
        res["passes"][name] = r
    print(json.dumps(res, indent=1))
    for name, r in res["passes"].items():
        print("%-8s %7.1f MB  im2col+GEMM %.3f ms  direct %.3f ms (%.0f GB/s, %.0f %% of 3.35 TB/s)"
              % (name, r["bytes"] / 1e6, r["im2col_gemm"]["ms"], r["direct"]["ms"],
                 r["direct"]["GB_s"], 100 * r["direct"]["frac_of_3.35TB_s"]))


if __name__ == "__main__":
    main()
