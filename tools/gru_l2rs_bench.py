"""Developer tool: us per time step of the GRU recurrence kernels alone (sb_gru_fwd, sb_gru_bwd),
both directions of H = 1024 at T = 247, under developer flags (sb_debug_gru_flags), alternated.
    python tools/gru_l2rs_bench.py [Bp ...]        (default: 32 64)
Backward flags compared: 0 (default selection), 256 (L2 reduce-scatter mode forced), 512 (that
mode disabled); the forward runs at the default selection for scale."""
import ctypes
import sys

import torch

sys.path.insert(0, ".")
from speech_b200 import _lib, ops  # noqa: E402

lib = _lib.load()
T, H, ndir, REPS, ROUNDS = 247, 1024, 2, 20, 3
FLAGS = (0, 256, 512)


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
        return e0.elapsed_time(e1) / REPS / T * 1e3, lib.sb_debug_gru_cluster(0)
    finally:
        lib.sb_debug_gru_flags(0)


def main(bps):
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
        dy = torch.randn(M, D, device="cuda") * 0.1
        dgi = torch.empty(M, ndir * K3, dtype=torch.bfloat16, device="cuda")
        dghn = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
        dbih = torch.zeros(ndir * K3, device="cuda")
        dbhh = torch.zeros(ndir * K3, device="cuda")
        nf, nb = ctypes.c_size_t(0), ctypes.c_size_t(0)
        _lib.check(lib.sb_gru_fwd_workspace_size(Bp, H, ndir, ctypes.byref(nf)), "ws")
        _lib.check(lib.sb_gru_bwd_workspace_size(Bp, H, ndir, ctypes.byref(nb)), "ws")
        wf, wb = ops._workspace(nf.value, "cuda"), ops._workspace(nb.value, "cuda")

        def fwd():
            _lib.check(lib.sb_gru_fwd(gi.data_ptr(), whh.data_ptr(), bhh.data_ptr(), y.data_ptr(),
                                      xn.data_ptr(), gates.data_ptr(), wf.data_ptr(), nf.value,
                                      T, Bp, H, ndir, sp), "sb_gru_fwd")

        def bwd():
            _lib.check(lib.sb_gru_bwd(dy.data_ptr(), y.data_ptr(), gates.data_ptr(),
                                      whh.data_ptr(), dgi.data_ptr(), dghn.data_ptr(),
                                      dbih.data_ptr(), dbhh.data_ptr(), wb.data_ptr(), nb.value,
                                      T, Bp, H, ndir, sp), "sb_gru_bwd")

        fwd()
        res = {}
        for _ in range(ROUNDS):
            for name, fn in (("fwd", fwd), ("bwd", bwd)):
                for f in (FLAGS if name == "bwd" else (0,)):
                    us, cs = timed(fn, f)
                    res.setdefault((name, f), []).append((us, cs))
        for (name, f), v in sorted(res.items()):
            us = sorted(u for u, _ in v)
            print("Bp %3d %s flags %3d: us/step median %.2f  (min %.2f max %.2f)  cluster %d"
                  % (Bp, name, f, us[len(us) // 2], us[0], us[-1], v[-1][1]))


if __name__ == "__main__":
    main([int(a) for a in sys.argv[1:]] or [32, 64])
