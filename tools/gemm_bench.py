"""Developer tool: time sb_gemm_bf16_tn at the GEMM shapes of one north-star training step
(B = 64, T' = 247, M = 247 * 64 = 15808 tokens, 5 x biGRU-1024, conv2 of the front-end), with
the call sites' operand layouts (MN-major views, bias, accumulate, the library's K split), under:
    c2      the default selection (gemm_bf16_tn_c2_kernel for N > 128, TMA-store epilogue)
    regs    sb_debug_gemm_flags(2): the same kernel, output stored straight from the registers
    legacy  sb_debug_gemm_flags(1): gemm_bf16_tn_kernel at 128 x 128 for every N > 64
    cublas  torch.matmul on the same bf16 operands (bf16 output), as a yardstick
    nostore sb_debug_gemm_flags(4), with --nostore: the c2 kernel with no output at all (timing
            only: the mainloop alone)
    python tools/gemm_bench.py [--reps 20] [--rounds 3] [--nostore] [--only SUBSTRING]"""
import argparse
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from speech_b200 import _lib, ops  # noqa: E402

lib = _lib.load()
M, BP = 15808, 64
H, D, K3 = 1024, 2048, 3072


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return "%s | %s | %d SMs" % (torch.cuda.get_device_name(0), q,
                                 torch.cuda.get_device_properties(0).multi_processor_count)


def shapes():
    """-> [(name, launches per step, ours(), cublas(), flops)]"""
    g = torch.Generator(device="cuda").manual_seed(0)

    def rnd(*s):
        return (torch.randn(*s, device="cuda", generator=g) * 0.5).to(torch.bfloat16)

    X = rnd(M, D)                      # layer input (layers 1-4), token-major
    X0 = rnd(M, 480)                   # layer-0 input (conv features, 32 x 15)
    W = rnd(2 * K3, D)                 # [w_ih fwd | w_ih rev]
    W0 = rnd(2 * K3, 480)
    bias = torch.randn(2 * K3, device="cuda")
    dgi = rnd(M, 2 * K3)
    dghn = rnd(M, D)
    hb = rnd(M, D)
    gi = torch.empty(M, 2 * K3, device="cuda")
    dx = torch.empty(M, D, device="cuda")
    dx0 = torch.empty(M, 480, device="cuda")
    dwih = torch.zeros(2 * K3, D, device="cuda")
    dwih0 = torch.zeros(2 * K3, 480, device="cuda")
    dwhh = torch.zeros(K3, H, device="cuda")
    Ms = M - BP
    out = []

    def add(name, n, ours, cub, flops):
        out.append((name, n, ours, cub, flops))

    add("gi 15808x6144x2048 bias", 4,
        lambda: ops.gemm_bf16_tn(X, W, out=gi, bias=bias),
        lambda: torch.matmul(X, W.t()), 2.0 * M * 2 * K3 * D)
    add("gi 15808x6144x480 bias (layer 0)", 1,
        lambda: ops.gemm_bf16_tn(X0, W0, out=gi, bias=bias),
        lambda: torch.matmul(X0, W0.t()), 2.0 * M * 2 * K3 * 480)
    add("dX 15808x2048x6144 bT", 4,
        lambda: ops.gemm_bf16_tn(dgi, W, out=dx, b_mn=True),
        lambda: torch.matmul(dgi, W), 2.0 * M * D * 2 * K3)
    add("dX 15808x480x6144 bT (layer 0)", 1,
        lambda: ops.gemm_bf16_tn(dgi, W0, out=dx0, b_mn=True),
        lambda: torch.matmul(dgi, W0), 2.0 * M * 480 * 2 * K3)
    add("dW_ih 3072x2048x15808 aT bT acc (per direction)", 8,
        lambda: ops.gemm_bf16_tn(dgi[:, :K3], X, out=dwih[:K3], accumulate=True,
                                 a_mn=True, b_mn=True),
        lambda: torch.matmul(dgi[:, :K3].t(), X), 2.0 * K3 * D * M)
    add("dW_ih 6144x2048x15808 aT bT acc (both directions)", 4,
        lambda: ops.gemm_bf16_tn(dgi, X, out=dwih, accumulate=True, a_mn=True, b_mn=True),
        lambda: torch.matmul(dgi.t(), X), 2.0 * 2 * K3 * D * M)
    add("dW_ih 3072x480x15808 aT bT acc (layer 0, per direction)", 2,
        lambda: ops.gemm_bf16_tn(dgi[:, :K3], X0, out=dwih0[:K3], accumulate=True,
                                 a_mn=True, b_mn=True),
        lambda: torch.matmul(dgi[:, :K3].t(), X0), 2.0 * K3 * 480 * M)
    add("dW_hh 2048x1024x15744 aT bT acc (r,z rows)", 10,
        lambda: ops.gemm_bf16_tn(dgi[BP:, :2 * H], hb[:Ms, :H], out=dwhh[:2 * H],
                                 accumulate=True, a_mn=True, b_mn=True),
        lambda: torch.matmul(dgi[BP:, :2 * H].t(), hb[:Ms, :H]), 2.0 * 2 * H * H * Ms)
    add("dW_hh 1024x1024x15744 aT bT acc (n rows)", 10,
        lambda: ops.gemm_bf16_tn(dghn[BP:, :H], hb[:Ms, :H], out=dwhh[2 * H:],
                                 accumulate=True, a_mn=True, b_mn=True),
        lambda: torch.matmul(dghn[BP:, :H].t(), hb[:Ms, :H]), 2.0 * H * H * Ms)
    dl = rnd(M, 32)                    # fc output gradient (vocabulary padded to 32)
    wT = rnd(D, 32)
    dy = torch.empty(M, D, device="cuda")
    add("fc dY 15808x2048x32", 1,
        lambda: ops.gemm_bf16_tn(dl, wT, out=dy),
        lambda: torch.matmul(dl, wT.t()), 2.0 * M * D * 32)
    MC = BP * 247 * 15                 # conv2 patch rows: B x T' x F'
    dC = rnd(MC, 32)
    Wp = rnd(32, 1280)                 # [Co][Kp] = [K][N]
    dA = torch.empty(MC, 1280, device="cuda")
    add("conv2 dA 237120x1280x32 bT", 1,
        lambda: ops.gemm_bf16_tn(dC, Wp, out=dA, b_mn=True),
        lambda: torch.matmul(dC, Wp), 2.0 * MC * 1280 * 32)
    return out


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


def run_ours(fn, flags, reps):
    lib.sb_debug_gemm_flags(flags)
    try:
        ms = timed(fn, reps)
        return ms, (lib.sb_debug_gemm_kernel().decode(), lib.sb_debug_gemm_epilogue().decode())
    finally:
        lib.sb_debug_gemm_flags(0)


def main(reps, rounds, nostore, only):
    print("device:", card())
    print("ms per launch (median of %d rounds of %d launches); TFLOP/s = 2MNK / time" % (rounds, reps))
    flags = {"c2": 0, "regs": 2, "legacy": 1}
    if nostore:
        flags["nostore"] = 4
    cols = list(flags) + ["cublas"]
    step = {k: 0.0 for k in cols}
    for name, n, ours, cub, flops in shapes():
        if only and not any(o in name for o in only):
            continue
        res = {k: [] for k in cols}
        kern = {}
        for _ in range(rounds):
            for k, f in flags.items():
                ms, kern[k] = run_ours(ours, f, reps)
                res[k].append(ms)
            res["cublas"].append(timed(cub, reps))
        med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
        print("%-52s x%-2d " % (name, n) + " | ".join(
            "%s %7.3f ms %5.0f TF/s%s" % (k, med[k], flops / med[k] / 1e9,
                                          " (%s %s)" % kern[k] if k in kern else "")
            for k in cols) + " | c2/regs %.3f" % (med["c2"] / med["regs"]))
        if "both directions" in name:
            continue              # an alternative to the per-direction launches, not extra work
        for k in cols:
            step[k] += n * med[k]
    print("per-step GEMM time of these shapes (per-direction dW_ih): " +
          ", ".join("%s %.2f ms" % (k, step[k]) for k in cols))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--nostore", action="store_true",
                    help="add a column with the c2 kernel's output stores skipped (flag 4)")
    ap.add_argument("--only", action="append", default=[],
                    help="time only the shapes whose name contains this (repeatable)")
    a = ap.parse_args()
    main(a.reps, a.rounds, a.nostore, a.only)
