"""Developer tool: the attention model (Seq2Seq) over vocabulary sizes.

    python tools/s2s_vocab_bench.py [--classes 31 1000 ...] [--forced 1000 3000] [--steps N]

WSJ-shaped model: conv [[32,5,8,2]]x2, 3x biGRU-512, log_t, 80 features, B = 16, T = 800, labels of
60-100 tokens.  Per C (classes = vocab_size - 1): ms per training step, greedy us per decode step
(B = 16), beam-8 us per decode step (one utterance), and the per-launch device times of the output
projection (s2s_fc_rows), its log-softmax (s2s_fc_logp), the fused attention step (s2s_attn_fwd,
which carries the projection where C <= 7 H), the projection backward (s2s_dout or the GEMM) and
the beam selection.  --forced: classes to run again with the many-CTA projection forced inside the
fused range (C <= 3584 at H = 512).  Decode loops enqueue max_len steps; steps after the stop rule
are no-ops and still count in the per-step time.  Prints the card name and power limit first."""
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


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def measure(C, steps, dec_len, forced):
    from speech_b200 import ops
    from speech_b200.functions import s2s
    from speech_b200.models import Seq2Seq
    saved = s2s.fc_fused
    if forced:
        s2s.fc_fused = lambda H, C: False
    try:
        torch.manual_seed(0)
        rng = np.random.RandomState(2)
        cfg = {"dropout": 0.0, "encoder": {"conv": [[32, 5, 8, 2], [32, 5, 8, 2]],
                                           "rnn": {"dim": 512, "bidirectional": True, "layers": 3}},
               "decoder": {"embedding_dim": 512, "layers": 1, "log_t": True}}
        V = C + 1
        m = Seq2Seq(80, V, cfg).cuda()
        lab = lambda: [V - 1] + rng.randint(0, V - 2, size=rng.randint(60, 100)).tolist() + [V - 2]
        batch = (tuple(rng.randn(800, 80).astype(np.float32) for _ in range(16)),
                 tuple(lab() for _ in range(16)))
        opt = torch.optim.SGD(m.parameters(), lr=1e-4)

        def train():
            opt.zero_grad()
            m.loss(batch).backward()
            opt.step()

        res = {"C": C, "route": "many-CTA" if not s2s.fc_fused(512, C) else "fused",
               "forced": forced}
        res["train_ms"] = 1e3 * _time(train, steps)
        ops.profile_begin()
        train()
        prof_train = ops.profile_end()
        m.set_eval()
        one = ((batch[0][0],), (batch[1][0],))
        res["greedy_us_per_step"] = 1e6 * _time(lambda: m.infer(batch, max_len=dec_len), 2) / dec_len
        res["beam8_us_per_step"] = 1e6 * _time(
            lambda: m.beam_search(one, beam_size=8, max_len=dec_len), 2) / dec_len
        ops.profile_begin()
        m.infer(batch, max_len=dec_len)
        prof_greedy = ops.profile_end()
        ops.profile_begin()
        m.beam_search(one, beam_size=8, max_len=dec_len)
        prof_beam = ops.profile_end()
        kt = {}
        for tag, prof in (("train", prof_train), ("greedy", prof_greedy), ("beam8", prof_beam)):
            for name, (n, ms, _) in prof.items():
                if name.startswith("s2s_fc") or name.startswith("s2s_beam_select") or \
                        name in ("s2s_attn_fwd", "s2s_dout"):
                    kt["%s/%s" % (tag, name)] = {"launches": n, "us_per_launch": 1e3 * ms / n}
            if tag == "train":
                g = [v for k, v in prof.items() if k.startswith("gemm")]
                kt["train/gemm_all"] = {"launches": sum(v[0] for v in g),
                                        "ms_total": sum(v[1] for v in g)}
        res["kernels"] = kt
        del m, opt
        torch.cuda.empty_cache()
        return res
    finally:
        s2s.fc_fused = saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--classes", type=int, nargs="*", default=[31, 1000, 3000, 8000, 16000, 32000])
    ap.add_argument("--forced", type=int, nargs="*", default=[1000, 3000])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--dec-len", type=int, default=50)
    a = ap.parse_args()
    print("card:", card(), flush=True)
    for C in a.classes:
        print(json.dumps(measure(C, a.steps, a.dec_len, False)), flush=True)
        if C in a.forced:
            print(json.dumps(measure(C, a.steps, a.dec_len, True)), flush=True)


if __name__ == "__main__":
    main()
