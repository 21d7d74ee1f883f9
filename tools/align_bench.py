"""Developer tool: cost of the Viterbi (forced) alignments.

    python tools/align_bench.py [--reps N] [--out F]

Prints the card name and power limit, then one JSON line per case:
  - CTC.align on bench.py's CTC model (5-layer biGRU-1024, B = 64, T = 1000 input frames so
    T' = 247, labels 40..120) at V+1 = 29 and 5000;
  - Transducer.align on bench.py's RNN-T model (3-layer biGRU-1024, B = 32, T = 1000, labels
    40..99) at V+1 = 29 (resident joint) and 1024 (slab joint).
Each line has the device ms of one align call (CUDA events around the call: encoder, projection
or joint, Viterbi and the copies back), and, on the same logits or lattice, the device ms of the
Viterbi C entry point alone (sb_ctc_viterbi, which includes the compact row reduction, or
sb_rnnt_viterbi) beside that of the loss with costs only (sb_ctc_fwd_bwd / sb_rnnt_fwd_bwd_compact
with a NULL gradient).  Every number is the median of --reps calls after a warm-up call.
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
from rnnt_recognize_bench import card, model_and_batch  # noqa: E402
from speech_b200 import _lib  # noqa: E402
from speech_b200.functions import transducer as rnnt_fn  # noqa: E402


def device_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times))


def call(rc, what):
    _lib.check(rc, what)


def ctc_case(V1, reps):
    from speech_b200.models import CTC
    torch.manual_seed(0)
    m = CTC(bench.F_IN, V1 - 1, bench.MODEL_CFG).cuda()
    m.set_eval()
    inputs, labels = bench.synth_batch(64)
    if V1 != bench.VOCAB + 1:
        rng = np.random.RandomState(3)
        labels = [rng.randint(0, V1 - 1, size=len(l)).tolist() for l in labels]
    batch = (tuple(inputs), tuple(labels))
    align_ms = device_ms(lambda: m.align(batch), reps)
    x, y, x_lens, y_lens = m.collate(*batch)
    with torch.no_grad():
        acts = m(batch).float().contiguous()
    lib = _lib.load()
    B, T, V = acts.shape
    dev = acts.device
    (lab, off, llen, alen), max_l = _lib.pack_labels(y, y_lens, x_lens, B, dev, num_classes=V)
    nv = _lib.workspace_size(lib.sb_ctc_viterbi_workspace_size, B, T, V, max_l)
    nl = _lib.workspace_size(lib.sb_ctc_workspace_size, B, T, V, max_l)
    wv = torch.empty(nv, dtype=torch.uint8, device=dev)
    wl = torch.empty(nl, dtype=torch.uint8, device=dev)
    path = torch.empty(B, T, dtype=torch.int32, device=dev)
    scores = torch.empty(B, dtype=torch.float64, device=dev)
    costs = torch.empty(B, dtype=torch.float32, device=dev)
    sp = _lib.stream_ptr()
    vit = device_ms(lambda: call(lib.sb_ctc_viterbi(
        acts.data_ptr(), lab.data_ptr(), off.data_ptr(), llen.data_ptr(), alen.data_ptr(), B, T, V,
        V - 1, max_l, path.data_ptr(), scores.data_ptr(), wv.data_ptr(), nv, sp), "viterbi"), reps)
    loss = device_ms(lambda: call(lib.sb_ctc_fwd_bwd(
        acts.data_ptr(), None, lab.data_ptr(), off.data_ptr(), llen.data_ptr(), alen.data_ptr(), B,
        T, V, V - 1, max_l, costs.data_ptr(), wl.data_ptr(), nl, sp), "loss"), reps)
    return {"case": "CTC.align", "V1": V1, "B": B, "T_in": bench.T_IN, "T_enc": T,
            "align_ms": round(align_ms, 3), "viterbi_kernel_ms": round(vit, 4),
            "loss_costs_only_ms": round(loss, 4)}


def rnnt_case(V1, reps):
    m, batch = model_and_batch(V1, None)
    align_ms = device_ms(lambda: m.align(batch), reps)
    x, y, x_lens, y_lens = m.collate(*batch)
    y_mat = m.label_collate(batch[1]).cuda()
    with torch.no_grad():
        fx, fy = m.joint_inputs(m._encode(x.cuda(), None), y_mat)
        ops = rnnt_fn._joint_operands(fx, fy, m.fc2.fc, y_mat)
        lat, _ = rnnt_fn.compact_lattice(*ops, m.blank)
    lib = _lib.load()
    B, T, U1 = fx.shape[0], fx.shape[1], fy.shape[1]
    dev = fx.device
    (lab, off, ylen, xlen), _ = _lib.pack_labels(y, y_lens, x_lens, B, dev, lattice_rows=U1)
    nv = _lib.workspace_size(lib.sb_rnnt_viterbi_workspace_size, B, T, U1)
    nl = _lib.workspace_size(lib.sb_rnnt_workspace_size, B, T, U1)
    wv = torch.empty(nv, dtype=torch.uint8, device=dev)
    wl = torch.empty(nl, dtype=torch.uint8, device=dev)
    frames = torch.empty(B, U1 - 1, dtype=torch.int32, device=dev)
    scores = torch.empty(B, dtype=torch.float64, device=dev)
    costs = torch.empty(B, dtype=torch.float32, device=dev)
    sp = _lib.stream_ptr()
    vit = device_ms(lambda: call(lib.sb_rnnt_viterbi(
        lat.data_ptr(), lab.data_ptr(), off.data_ptr(), ylen.data_ptr(), xlen.data_ptr(), B, T, U1,
        frames.data_ptr(), scores.data_ptr(), wv.data_ptr(), nv, sp), "viterbi"), reps)
    loss = device_ms(lambda: call(lib.sb_rnnt_fwd_bwd_compact(
        lat.data_ptr(), None, lab.data_ptr(), off.data_ptr(), ylen.data_ptr(), xlen.data_ptr(), B,
        T, U1, m.blank, costs.data_ptr(), wl.data_ptr(), nl, sp), "loss"), reps)
    return {"case": "Transducer.align", "V1": V1, "B": B, "T_in": bench.T_IN, "T_enc": T,
            "U1": U1, "align_ms": round(align_ms, 3), "viterbi_kernel_ms": round(vit, 4),
            "loss_costs_only_ms": round(loss, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from speech_b200.csrc import build
    build.build()
    print("card:", card(), flush=True)
    lines = []
    for V1 in (29, 5000):
        lines.append(ctc_case(V1, args.reps))
        print(json.dumps(lines[-1]), flush=True)
    for V1 in (29, 1024):
        lines.append(rnnt_case(V1, args.reps))
        print(json.dumps(lines[-1]), flush=True)
    if args.out:
        with open(args.out, "w") as fh:
            json.dump({"card": card(), "cases": lines}, fh, indent=1)


if __name__ == "__main__":
    main()
