"""Developer tool: the wide GRU recurrence kernels, measured with CUDA events after warm-up.
    python tools/gru_wide_bench.py [--widths 1024,1152,...] [--rows 32,64,128] [--T 250]
1. us per step of sb_gru_fwd and sb_gru_bwd alone for bidirectional layers (forward and backward
   alternated, REPS launches each), with the plan (sb_debug_gru_plan) and the achieved ingress per
   SM: the gathered h_{t-1} / dgh_t plus the streamed W_hh bytes of one CTA per step, over the
   step time.
2. one bidirectional layer, forward + backward, through ops.gru_stack against cuDNN nn.GRU in
   bf16 and fp32 on the same card, alternated (B = 64 unless --rows says otherwise).
3. utt/s of a training step (zero_grad, loss, backward, FlatSGD step) of the north-star CTC
   configuration of bench.py with rnn.dim set to --ctc-dim (0 skips), B = 64, T = 1000.
--ring-sweep K1,K2,..: part 1 once per gather-ring size (sb_debug_gru_wide_ring, KB), the sizes
alternated within each width and row count.
Prints the card name and power limit first."""
import argparse
import ctypes
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from speech_b200 import _lib, ops  # noqa: E402

lib = _lib.load()
REPS, ROUNDS = 5, 3


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:   # noqa: BLE001
        q = torch.cuda.get_device_name(0)
    return q


def events(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def plan(backward):
    out = (ctypes.c_int * 3)()
    lib.sb_debug_gru_plan(backward, out)
    return tuple(out)


def kernels(H, Bp, T, ring_kb=0):
    if ring_kb:
        lib.sb_debug_gru_wide_ring(ring_kb)
    ndir = 2
    Hp = ops.gru_padded_width(Bp, H, ndir)
    M, D, K3 = T * Bp, ndir * Hp, 3 * Hp
    g = torch.Generator(device="cuda").manual_seed(H + Bp)
    gi = torch.randn(M, ndir * K3, device="cuda", generator=g)
    whh = (torch.randn(ndir, K3, Hp, device="cuda", generator=g) / Hp ** 0.5).to(torch.bfloat16)
    bhh = torch.randn(ndir, K3, device="cuda", generator=g) * 0.1
    y = torch.empty(M, D, device="cuda")
    xn = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
    gates = torch.empty(M, ndir, 4, Hp, device="cuda")
    dy = torch.randn(M, D, device="cuda", generator=g) * 0.1
    dgi = torch.empty(M, ndir * K3, dtype=torch.bfloat16, device="cuda")
    dghn = torch.empty(M, D, dtype=torch.bfloat16, device="cuda")
    dbih = torch.zeros(ndir * K3, device="cuda")
    dbhh = torch.zeros(ndir * K3, device="cuda")
    nf, nb = ctypes.c_size_t(0), ctypes.c_size_t(0)
    _lib.check(lib.sb_gru_fwd_workspace_size(Bp, Hp, ndir, ctypes.byref(nf)), "ws")
    _lib.check(lib.sb_gru_bwd_workspace_size(Bp, Hp, ndir, ctypes.byref(nb)), "ws")
    wf, wb = ops._workspace(nf.value, "cuda"), ops._workspace(nb.value, "cuda")
    sp = _lib.stream_ptr()

    def fwd():
        _lib.check(lib.sb_gru_fwd(gi.data_ptr(), whh.data_ptr(), bhh.data_ptr(), y.data_ptr(),
                                  xn.data_ptr(), gates.data_ptr(), wf.data_ptr(), nf.value,
                                  T, Bp, Hp, ndir, sp), "sb_gru_fwd")

    def bwd():
        _lib.check(lib.sb_gru_bwd(dy.data_ptr(), y.data_ptr(), gates.data_ptr(), whh.data_ptr(),
                                  dgi.data_ptr(), dghn.data_ptr(), dbih.data_ptr(),
                                  dbhh.data_ptr(), wb.data_ptr(), nb.value, T, Bp, Hp, ndir, sp),
                   "sb_gru_bwd")

    fwd(); bwd(); torch.cuda.synchronize()
    names = (lib.sb_debug_gru_fwd_kernel().decode(), lib.sb_debug_gru_bwd_kernel().decode())
    plans = (plan(0), plan(1))
    tf, tb = [], []
    for _ in range(ROUNDS):
        tf.append(events(fwd, REPS) / (T - 1) * 1e3)
        tb.append(events(bwd, REPS) / (T - 1) * 1e3)
    res = {"H": H, "Hp": Hp, "Bp": Bp, "T": T, "ring_KB": lib.sb_debug_gru_wide_ring(0)}
    for key, t, name, (U, R, S), nw, kdim in (("fwd", tf, names[0], plans[0], 3, Hp),
                                              ("bwd", tb, names[1], plans[1], 1, 3 * Hp)):
        us = min(t)
        row = {"kernel": name, "us_per_step": round(us, 2), "spread": round(max(t) - us, 2)}
        if U:
            ingress = Bp * kdim * 2 + S * nw * U * 128     # bytes per CTA per step
            row.update({"U": U, "resident_chunks": R, "streamed_chunks": S,
                        "ingress_KB": round(ingress / 1024, 1),
                        "B_per_ns_per_SM": round(ingress / (us * 1e3), 1)})
        res[key] = row
    return res


def layer(H, B, T):
    """forward + backward of one bidirectional layer (In = H): ops.gru_stack vs cuDNN"""
    torch.manual_seed(H)
    rnn = torch.nn.GRU(H, H, 1, batch_first=True, bidirectional=True).cuda()
    x = torch.randn(B, T, H, device="cuda", requires_grad=True)
    rnn_bf = torch.nn.GRU(H, H, 1, batch_first=True, bidirectional=True).cuda().to(torch.bfloat16)
    xb = x.detach().to(torch.bfloat16).requires_grad_(True)

    def ours():
        ops.gru_stack(x, rnn).sum().backward()

    def cudnn32():
        rnn(x)[0].sum().backward()

    def cudnn16():
        rnn_bf(xb)[0].sum().backward()

    fns = {"ours": ours, "cudnn_fp32": cudnn32, "cudnn_bf16": cudnn16}
    for f in fns.values():
        f()
    torch.cuda.synchronize()
    ts = {k: [] for k in fns}
    for _ in range(ROUNDS):
        for k, f in fns.items():
            ts[k].append(events(f, REPS))
    return {"H": H, "B": B, "T": T, **{k + "_ms": round(min(v), 3) for k, v in ts.items()}}


def ctc_step(dim, steps=10, warmup=3):
    import numpy as np
    import bench
    from speech_b200.models import CTC
    from speech_b200.optim import FlatSGD
    cfg = {"dropout": 0.0, "encoder": dict(bench.MODEL_CFG["encoder"])}
    cfg["encoder"]["rnn"] = dict(cfg["encoder"]["rnn"], dim=dim)
    torch.manual_seed(0)
    model = CTC(bench.F_IN, bench.VOCAB, cfg).cuda()
    opt = FlatSGD(model, lr=1e-3, momentum=0.0, max_grad_norm=200.0)
    rng = np.random.RandomState(0)
    B = bench.GLOBAL_B
    batch = ([rng.randn(bench.T_IN, bench.F_IN).astype(np.float32) for _ in range(B)],
             [rng.randint(0, bench.VOCAB, 100).tolist() for _ in range(B)])

    def step():
        opt.zero_grad()
        model.loss(batch).backward()
        opt.step()

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    ms = events(step, steps)
    return {"rnn_dim": dim, "B": B, "T": bench.T_IN, "ms_per_step": round(ms, 2),
            "utt_per_s": round(B / ms * 1e3, 1), "fwd_kernel": lib.sb_debug_gru_fwd_kernel().decode(),
            "bwd_kernel": lib.sb_debug_gru_bwd_kernel().decode()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", default="1024,1152,1280,1536,2048")
    ap.add_argument("--rows", default="32,64,128")
    ap.add_argument("--layer-widths", default="1024,1280,1536,2048")
    ap.add_argument("--layer-rows", default="64")
    ap.add_argument("--T", type=int, default=250)
    ap.add_argument("--ring-sweep", default="")
    ap.add_argument("--ctc-dim", type=int, default=1280)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    rings = [int(v) for v in a.ring_sweep.split(",") if v] or [0]
    default_ring = lib.sb_debug_gru_wide_ring(0)
    for H in [int(v) for v in a.widths.split(",") if v]:
        for Bp in [int(v) for v in a.rows.split(",") if v]:
            for kb in rings:
                print("kernels", kernels(H, Bp, a.T, kb), flush=True)
            lib.sb_debug_gru_wide_ring(default_ring)
    for H in [int(v) for v in a.layer_widths.split(",") if v]:
        for B in [int(v) for v in a.layer_rows.split(",") if v]:
            print("layer", layer(H, B, a.T), flush=True)
    if a.ctc_dim:
        print("ctc_step", ctc_step(a.ctc_dim), flush=True)


if __name__ == "__main__":
    main()
