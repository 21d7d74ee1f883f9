"""Developer tool: Transducer.infer over vocabulary sizes.

    python tools/rnnt_decode_vocab_bench.py [--vocab 29 1024 ...] [--beams 1 4 8] [--reps N] [--out F]

The benchmark's RNN-T model (bench.py's rnnt_workload: 3x biGRU-1024 encoder, GRU-1024 prediction
network, B = 32, T = 1000 input frames, 40..100 labels) with V+1 output classes.  Prints the card
name and power limit, then one JSON line per V+1 with, per beam:
  - the route Transducer.infer takes ("full": the (B, T', U+1, V+1) lattice and
    sb_rnnt_decode_static; "shortlist": the slab joint with sb_rnnt_shortlist_rows and
    sb_rnnt_decode_static_shortlist): ms per infer call (median, min, max of --reps calls) and the
    largest peak memory growth of those calls in GB;
  - where the full route runs, the same for the shortlist route forced on the same batch, the two
    routes' calls alternated (full, shortlist, full, ...), and whether both return the same
    predictions;
  - enc_ms: the encoder and the joint inputs alone (the part both routes share).
Times are host clocks around calls that end in a device synchronise (every infer copies its labels
to the host), after one warm-up call per route.
"""
import argparse
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


def _call(fn):
    """(result, ms, peak memory growth GB) of one call"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    return out, ms, (torch.cuda.max_memory_allocated() - base) / 2**30


def _timed(fns, reps):
    """one warm-up call of each fn, then reps rounds calling them in turn ->
    per fn (last result, {"ms": median, "ms_min", "ms_max", "peak_gb"}), or (None, "oom")"""
    try:
        for fn in fns:
            fn()
        samples = [[] for _ in fns]
        for _ in range(reps):
            for j, fn in enumerate(fns):
                samples[j].append(_call(fn))
    except torch.cuda.OutOfMemoryError:
        torch.cuda.empty_cache()
        return [(None, "oom") for _ in fns]
    res = []
    for smp in samples:
        ms = sorted(s[1] for s in smp)
        res.append((smp[-1][0], {"ms": round(float(np.median(ms)), 2), "ms_min": round(ms[0], 2),
                                 "ms_max": round(ms[-1], 2),
                                 "peak_gb": round(max(s[2] for s in smp), 3)}))
    return res


def run(V1, beams, reps):
    import bench
    from speech_b200.models import Transducer
    from speech_b200.transducer_decoders import decode_static_fits
    torch.manual_seed(0)
    cfg = {"dropout": 0.0, "encoder": {"conv": bench.WSJ_CONV,
                                       "rnn": {"dim": 1024, "bidirectional": True, "layers": 3}},
           "decoder": {"embedding_dim": 256, "layers": 1}}
    m = Transducer(bench.F_IN, V1 - 1, cfg).cuda()
    m.set_eval()
    rng = np.random.RandomState(3)
    inputs = [rng.randn(bench.T_IN, bench.F_IN).astype(np.float32) for _ in range(32)]
    labels = [rng.randint(0, V1 - 1, size=rng.randint(40, 100)).tolist() for _ in range(32)]
    batch = (inputs, labels)

    def enc():
        x, _, _, _ = m.collate(*batch)
        y = m.label_collate(labels).cuda()
        with torch.no_grad():
            fx, fy = m.joint_inputs(m.encode(x), y)
        return fx.sum().item()
    row = {"V1": V1, "enc_ms": _timed([enc], reps)[0][1]}
    for K in beams:
        fits = decode_static_fits(K, V1)
        fns = [lambda: m.infer(batch, beam_size=K)]
        if fits:
            fns.append(lambda: m._infer_shortlists(batch, K))
        res = _timed(fns, reps)
        r = {"route": "full" if fits else "shortlist", "infer": res[0][1]}
        if fits:
            r["shortlist_forced"] = res[1][1]
            r["same_preds"] = None if res[0][0] is None else res[0][0] == res[1][0]
        row["beam%d" % K] = r
    del m
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--vocab", type=int, nargs="+", default=[29, 1024, 4096, 16384, 32768])
    ap.add_argument("--beams", type=int, nargs="+", default=[1, 4, 8])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    print("card:", card(), flush=True)
    rows = []
    print("reps per point:", args.reps, flush=True)
    for V1 in args.vocab:
        row = run(V1, args.beams, args.reps)
        print(json.dumps(row), flush=True)
        rows.append(row)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump({"card": card(), "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
