"""Developer tool: the CTC model over vocabulary sizes.

    python tools/ctc_vocab_bench.py [--vocab 29 256 ...] [--steps N] [--out F]

Prints the card name and power limit, then one JSON line per V (= symbols + blank):
  - loss: device ms of sb_ctc_fwd_bwd (costs and gradients) at B = 64, T' = 247, labels of 10..40
    and of 40..120 symbols; where the fused kernel holds the shape, also the fused and the compact
    entry (sb_ctc_fwd_bwd_compact) side by side;
  - step: ms per training step of the north-star CTC model (bench.py's MODEL_CFG, B = 64, T = 1000
    input frames) and its peak memory;
  - decode: ms per CTC.infer call on that batch at beam 1, 8 and 10; where the full scan fits, also
    device ms of the full-scan and the shortlist entries side by side on the same log-probabilities.
"""
import argparse
import ctypes
import json
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:   # noqa: BLE001
        q = torch.cuda.get_device_name(0)
    return q


def _dev_ms(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def loss_times(V, lmin, lmax, rng):
    from speech_b200 import _lib
    lib = _lib.load()
    B, T = 64, 247
    acts = torch.randn(B, T, V, device="cuda")
    llen = rng.randint(lmin, lmax + 1, B).astype(np.int32)
    flat = rng.randint(0, V - 1, int(llen.sum())).astype(np.int32)
    offs = np.concatenate([[0], np.cumsum(llen)[:-1]]).astype(np.int32)
    d = torch.from_numpy(np.concatenate([flat, offs, llen, np.full(B, T, np.int32)])).cuda()
    n = len(flat)
    ptrs = [d.data_ptr(), d[n:].data_ptr(), d[n + B:].data_ptr(), d[n + 2 * B:].data_ptr()]
    grads = torch.empty_like(acts)
    costs = torch.empty(B, device="cuda")
    out = {}
    for name, size_fn, fn in (("default", lib.sb_ctc_workspace_size, lib.sb_ctc_fwd_bwd),
                              ("compact", lib.sb_ctc_compact_workspace_size,
                               lib.sb_ctc_fwd_bwd_compact)):
        nb = ctypes.c_size_t(0)
        size_fn(B, T, V, int(llen.max()), ctypes.byref(nb))
        ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")

        def run():
            _lib.check(fn(acts.data_ptr(), grads.data_ptr(), *ptrs, B, T, V, V - 1,
                          int(llen.max()), costs.data_ptr(), ws.data_ptr(), nb.value,
                          _lib.stream_ptr()), name)
        out[name] = round(_dev_ms(run), 3)
        del ws
    return out


def step_and_decode(V, steps, rng):
    import bench
    from speech_b200.models import CTC
    from speech_b200.optim import FlatSGD
    torch.manual_seed(0)
    m = CTC(bench.F_IN, V - 1, bench.MODEL_CFG).cuda()
    opt = FlatSGD(m, lr=1e-4)
    B = bench.GLOBAL_B
    inputs = [rng.randn(bench.T_IN, bench.F_IN).astype(np.float32) for _ in range(B)]
    labels = [rng.randint(0, V - 1, rng.randint(40, 121)).tolist() for _ in range(B)]
    batch = m.collate(inputs, labels)

    def step():
        opt.zero_grad()
        m.loss((inputs, labels)).backward()
        opt.step()
    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    torch.cuda.synchronize()
    res = {"step_ms": round((time.perf_counter() - t0) / steps * 1e3, 2),
           "peak_gb": round(torch.cuda.max_memory_allocated() / 2**30, 2)}
    dec = {}
    for K in (1, 8, 10):
        m.infer((inputs, labels), beam_size=K)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.infer((inputs, labels), beam_size=K)
        torch.cuda.synchronize()
        dec["infer_b%d_ms" % K] = round((time.perf_counter() - t0) * 1e3, 2)
    with torch.no_grad():
        logp = torch.log(m.forward_impl(batch[0], softmax=True)).contiguous()
    res.update(dec)
    res["decode_entries"] = decode_entries(logp, V)
    del m, opt
    return res


def decode_entries(logp, S):
    from speech_b200 import _lib
    lib = _lib.load()
    B, T, _ = logp.shape
    lens = torch.full((B,), T, dtype=torch.int32, device="cuda")
    out = {}
    for K in (1, 8, 10):
        if K * (S + 1) * 13 + 16 > 200 * 1024:
            continue                       # the full scan does not fit: shortlist only (infer above)
        nb = ctypes.c_size_t(0)
        lib.sb_ctc_prefix_beam_workspace_size(B, T, K, ctypes.byref(nb))
        ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
        lab = torch.empty(B, T, dtype=torch.int32, device="cuda")
        ln = torch.empty(B, dtype=torch.int32, device="cuda")
        sc = torch.empty(B, dtype=torch.float64, device="cuda")
        for name, fn in (("full", lib.sb_ctc_prefix_beam), ("shortlist",
                                                             lib.sb_ctc_prefix_beam_shortlist)):
            def run():
                _lib.check(fn(logp.data_ptr(), lens.data_ptr(), B, T, S, K, S - 1, lab.data_ptr(),
                              ln.data_ptr(), sc.data_ptr(), ws.data_ptr(), nb.value,
                              _lib.stream_ptr()), name)
            out["b%d_%s_ms" % (K, name)] = round(_dev_ms(run, reps=2), 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vocab", type=int, nargs="+",
                    default=[29, 256, 1024, 4096, 8192, 16384, 32768])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    print("card:", card(), flush=True)
    rng = np.random.RandomState(0)
    rows = []
    for V in args.vocab:
        row = {"V": V}
        row["loss_l10_40_ms"] = loss_times(V, 10, 40, rng)
        row["loss_l40_120_ms"] = loss_times(V, 40, 120, rng)
        row.update(step_and_decode(V, args.steps, rng))
        torch.cuda.empty_cache()
        print(json.dumps(row), flush=True)
        rows.append(row)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump({"card": card(), "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
