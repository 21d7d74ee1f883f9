"""Developer tool: us per time step of the GRU forward recurrence kernel alone (sb_gru_fwd), by
default both directions of H = 1024 at T = 247, alternating three developer-flag settings: 32 (the
K-split forward kernels disabled: gru_fwd_kernel), 0 (the default selection: gru_fwd_ks_kernel<2>
at H = 1024 on a 132-SM H100) and 1024 (gru_fwd_ks_kernel<2> forced wherever it applies).
    python tools/gru_fwd_ks2_bench.py [--H 1024] [--ndir 2] [Bp ...]        (default: 32 64)"""
import argparse
import ctypes
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from speech_b200 import _lib, ops  # noqa: E402

lib = _lib.load()
T, REPS, ROUNDS = 247, 20, 7
FLAGS = (32, 0, 1024)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return "%s | %s | %d SMs" % (torch.cuda.get_device_name(0), q,
                                 torch.cuda.get_device_properties(0).multi_processor_count)


def timed(fn, flags):
    lib.sb_debug_gru_flags(flags)
    try:
        fn()                                        # warm-up (module load, attributes)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(REPS):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / REPS / T * 1e3, lib.sb_debug_gru_fwd_kernel().decode()
    finally:
        lib.sb_debug_gru_flags(0)


def main(bps, H, ndir):
    print("device:", card())
    print("H = %d, %d direction(s), T = %d" % (H, ndir, T))
    torch.manual_seed(0)
    sp = _lib.stream_ptr()
    for Bp in bps:
        M, D, K3 = T * Bp, ndir * H, 3 * H
        gi = torch.randn(M, ndir * K3, device="cuda")
        whh = (torch.randn(ndir, K3, H, device="cuda") / H ** 0.5).to(torch.bfloat16)
        bhh = torch.randn(ndir, K3, device="cuda") * 0.1
        y = torch.empty(M, D, device="cuda")
        xn = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
        gates = torch.empty(M, ndir, 4, H, device="cuda")
        nf = ctypes.c_size_t(0)
        _lib.check(lib.sb_gru_fwd_workspace_size(Bp, H, ndir, ctypes.byref(nf)), "ws")
        wf = ops._workspace(nf.value, "cuda")

        def fwd():
            _lib.check(lib.sb_gru_fwd(gi.data_ptr(), whh.data_ptr(), bhh.data_ptr(), y.data_ptr(),
                                      xn.data_ptr(), gates.data_ptr(), wf.data_ptr(), nf.value,
                                      T, Bp, H, ndir, sp), "sb_gru_fwd")

        res = {}
        for _ in range(ROUNDS):
            for f in FLAGS:
                res.setdefault(f, []).append(timed(fwd, f))
        med = {}
        for f in FLAGS:
            us = sorted(u for u, _ in res[f])
            med[f] = us[len(us) // 2]
            print("Bp %3d fwd flags %3d (%-5s): us/step median %.2f  (min %.2f max %.2f, %d runs)"
                  % (Bp, f, res[f][-1][1], med[f], us[0], us[-1], len(us)))
        print("Bp %3d fwd: default - flag 32 = %+.2f us/step" % (Bp, med[0] - med[32]))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--H", type=int, default=1024)
    ap.add_argument("--ndir", type=int, default=2, choices=[1, 2])
    ap.add_argument("bp", type=int, nargs="*")
    a = ap.parse_args()
    main(a.bp or [32, 64], a.H, a.ndir)
