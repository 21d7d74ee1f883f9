"""Developer tool: run every kernel once at small sizes (for compute-sanitizer).
    compute-sanitizer --tool memcheck python tools/sanitize.py"""
import sys
import numpy as np, torch
sys.path.insert(0, ".")
from speech_b200.models import CTC, Seq2Seq, Transducer
from speech_b200.optim import FlatSGD
torch.manual_seed(0); np.random.seed(0)
cfg = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                                   "rnn": {"dim": 256, "bidirectional": True, "layers": 2}},
       "decoder": {"embedding_dim": 256, "layers": 1}}
inputs = [np.random.randn(90 + 3 * i, 80).astype(np.float32) for i in range(5)]
labels = [np.random.randint(0, 28, 7 + i).tolist() for i in range(5)]
m = CTC(80, 28, cfg).cuda()
opt = FlatSGD(m, lr=1e-3)
for _ in range(2):
    opt.zero_grad(); loss = m.loss((inputs, labels)); loss.backward(); opt.step()
print("ctc step ok", loss.item())
print("infer", [len(p) for p in m.infer((inputs, labels), beam_size=4)])
from speech_b200.lm import NGramLM
lm = NGramLM.train(labels, 4, 29, 28)
print("infer with LM", [len(p) for p in m.infer((inputs, labels), beam_size=4, lm=lm,
                                                  lm_weight=0.5, insertion_bonus=1.0)])
s = Seq2Seq(80, 30, cfg).cuda()
lab2 = [[29] + l + [28] for l in labels]
l2 = s.loss((inputs, lab2)); l2.backward()
print("seq2seq ok", l2.item(), [len(h) for h in s.infer((inputs, lab2), max_len=12)],
      s.beam_search(([inputs[0]], [lab2[0]]), beam_size=3, max_len=8))
print("seq2seq recognize", [len(h) for h in s.recognize(inputs, beam_size=3, max_len=8)])
lm2 = NGramLM.train(lab2, 3, 30, 29, end=28)
print("seq2seq recognize with LM", [len(h) for h in s.recognize(
    inputs, beam_size=3, max_len=8, lm=lm2, lm_weight=0.5, insertion_bonus=1.0)])
from speech_b200.functions import s2s as s2s_fn
fits = s2s_fn.beam_select_fits
s2s_fn.beam_select_fits = lambda K, C: False     # the split selection with the LM
print("seq2seq recognize with LM, split select", [len(h) for h in s.recognize(
    inputs, beam_size=3, max_len=8, lm=lm2, lm_weight=0.5, insertion_bonus=1.0)])
s2s_fn.beam_select_fits = fits
sc_dec = {"embedding_dim": 256, "layers": 1, "ctc_weight": 0.3}
sc = Seq2Seq(80, 30, dict(cfg, decoder=sc_dec)).cuda()
lc = sc.loss((inputs, lab2)); lc.backward()
print("seq2seq joint CTC loss", lc.item(), "recognize", [len(h) for h in sc.recognize(
    inputs, beam_size=3, max_len=8, ctc_weight=0.3)], "with LM", [len(h) for h in sc.recognize(
    inputs, beam_size=3, max_len=8, lm=lm2, lm_weight=0.5, insertion_bonus=1.0, ctc_weight=0.5,
    ctc_prebeam=29)])
from speech_b200.lm import WordLM
wsyms = list("abcdefghijklmnopqrstuvwxyz") + [" ", "'", "</s>", "<s>"]
wlm = WordLM.train(["the cat sat", "a cat", "the mat sat"], 3, wsyms, blank=29, end=28,
                   oov_penalty=-2.0)
wargs = dict(beam_size=3, max_len=8, lm=wlm, lm_weight=0.5, insertion_bonus=1.0)
print("seq2seq recognize with a word LM", [len(h) for h in s.recognize(inputs, **wargs)])
s2s_fn.beam_select_fits = lambda K, C: False     # the split selection with the word LM
print("seq2seq recognize with a word LM, split select",
      [len(h) for h in s.recognize(inputs, **wargs)])
s2s_fn.beam_select_fits = fits
print("seq2seq joint CTC with a word LM",
      [len(h) for h in sc.recognize(inputs, ctc_weight=0.3, **wargs)])
scu = Seq2Seq(80, 30, dict(cfg, encoder=dict(cfg["encoder"], lookahead=2, rnn=dict(
    cfg["encoder"]["rnn"], bidirectional=False)), decoder=sc_dec)).cuda()
print("seq2seq two-pass", [len(h) for h in scu.recognize_two_pass(inputs, beam_size=4)])
sst = scu.stream(2, beam_size=4, max_frames=100)
for k in range(0, 60, 20):
    sst.push([inputs[0][k:k + 20], inputs[1][k:k + 20]])
sst.finish()
print("seq2seq two-pass stream", sst.partial(), [len(h) for h in sst.rescored()])
t = Transducer(80, 28, cfg).cuda()
l3 = t.loss((inputs, labels)); l3.backward()
print("transducer ok", l3.item())
t2 = Transducer(80, 300, cfg).cuda()       # V+1 = 301: the large-vocabulary joint path
labels2 = [np.random.randint(0, 300, 7 + i).tolist() for i in range(5)]
l4 = t2.loss((inputs, labels2)); l4.backward()
print("transducer V+1=301 ok", l4.item(), [len(p) for p in t2.infer((inputs, labels2))])
cfg_x = dict(cfg, exact_lengths=True)          # per-utterance lengths through every layer
for cls in (CTC, Transducer):
    mx = cls(80, 28, cfg_x).cuda()
    lx = mx.loss((inputs, labels)); lx.backward()
    print("exact lengths", cls.__name__, lx.item(), [len(p) for p in mx.infer((inputs, labels))])
sx = Seq2Seq(80, 30, cfg_x).cuda()
l5 = sx.loss((inputs, lab2)); l5.backward()
print("exact lengths Seq2Seq", l5.item(), [len(h) for h in sx.infer((inputs, lab2), max_len=12)])
# zero-padded shapes: GRU width 1000 (run at 1008), conv channels 4 and 12 (run at 8 and 16),
# and a Transducer of width 100 (GRUs at 112, joint at 104)
cfg_p = {"dropout": 0.0, "encoder": {"conv": [[4, 5, 8, 2], [12, 5, 8, 2]],
                                     "rnn": {"dim": 1000, "bidirectional": True, "layers": 1}},
         "decoder": {"embedding_dim": 32, "layers": 1}}
mp = CTC(80, 28, cfg_p).cuda()
opt_p = FlatSGD(mp, lr=1e-3)
opt_p.zero_grad(); l6 = mp.loss((inputs, labels)); l6.backward(); opt_p.step()
print("padded CTC dim 1000 ok", l6.item())
cfg_p["encoder"]["rnn"]["dim"] = 100
tp = Transducer(80, 28, cfg_p).cuda()
l7 = tp.loss((inputs, labels)); l7.backward()
print("padded Transducer dim 100 ok", l7.item(), [len(p) for p in tp.infer((inputs, labels))])
# the L2 reduce-scatter mode of the K-split backward recurrence kernel, forced
from speech_b200 import _lib
_lib.load().sb_debug_gru_flags(256)
mr = CTC(80, 28, cfg).cuda()
l8 = mr.loss((inputs, labels)); l8.backward()
torch.cuda.synchronize()
_lib.load().sb_debug_gru_flags(0)
print("L2 reduce-scatter GRU ok", l8.item())
# the K-split forward recurrence kernel over 2-CTA clusters, forced
_lib.load().sb_debug_gru_flags(1024)
mk = CTC(80, 28, cfg).cuda()
l9 = mk.loss((inputs, labels)); l9.backward()
torch.cuda.synchronize()
fwd_kernel = _lib.load().sb_debug_gru_fwd_kernel().decode()
_lib.load().sb_debug_gru_flags(0)
assert fwd_kernel == "ks2", fwd_kernel
print("2-CTA K-split GRU forward ok", l9.item())
# the wide recurrence kernels with every W_hh chunk streamed (flag 2048) at a small width
_lib.load().sb_debug_gru_flags(2048)
mw = CTC(80, 28, cfg).cuda()
l10 = mw.loss((inputs, labels)); l10.backward()
torch.cuda.synchronize()
kernels = (_lib.load().sb_debug_gru_fwd_kernel().decode(),
           _lib.load().sb_debug_gru_bwd_kernel().decode())
_lib.load().sb_debug_gru_flags(0)
assert kernels == ("wide", "wide"), kernels
print("streamed wide GRU ok", l10.item())
# the 128 x 256 GEMM over 2-CTA clusters: odd M-tile count (unpaired last tile), ragged N and K,
# MN-major operands, accumulating with and without the library's K split; under both epilogues
# (flag 2: stores straight from the registers instead of through shared memory and TMA)
from speech_b200 import ops
A = torch.randn(304, 200, device="cuda").bfloat16()
Bm = torch.randn(200, 304, device="cuda").bfloat16()[:, :303]       # N = 303, row pitch 304
Ak = torch.randn(5000, 304, device="cuda").bfloat16()
Bk = torch.randn(5000, 304, device="cuda").bfloat16()[:, :303]
for gemm_flags, want in ((0, ("tma", "tma_reduce", "regs")), (2, ("regs", "regs", "regs"))):
    _lib.load().sb_debug_gemm_flags(gemm_flags)
    got = []
    out = torch.zeros(304, 304, device="cuda")[:, :303]              # ragged N, padded row pitch
    ops.gemm_bf16_tn(A, Bm.t().contiguous(), out=out, bias=torch.randn(303, device="cuda"))
    got.append(_lib.load().sb_debug_gemm_epilogue().decode())
    acc = torch.zeros(304, 304, device="cuda")[:, :303]
    ops.gemm_bf16_tn(A.t().contiguous(), Bm, out=acc, accumulate=True, a_mn=True, b_mn=True)
    got.append(_lib.load().sb_debug_gemm_epilogue().decode())
    ops.gemm_bf16_tn(Ak, Bk, out=acc, accumulate=True, a_mn=True, b_mn=True)    # split K
    got.append(_lib.load().sb_debug_gemm_epilogue().decode())
    torch.cuda.synchronize()
    _lib.load().sb_debug_gemm_flags(0)
    gemm_kernel = _lib.load().sb_debug_gemm_kernel().decode()
    assert gemm_kernel == "c2_128x256", gemm_kernel
    assert tuple(got) == want, (gemm_flags, got)
print("2-CTA GEMM ok")
# the attention model at a large vocabulary (C = 9000 > 7 H): the many-CTA projection over
# several class tiles and row blocks, its log-softmax, the GEMM backward of the projection, and the
# split beam selection (beam 8 x 9000 candidates: several tiles)
cfg_v = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                     "rnn": {"dim": 64, "bidirectional": True, "layers": 1}},
         "decoder": {"embedding_dim": 64, "layers": 1, "sample_prob": 0.5}}
sv = Seq2Seq(80, 9001, cfg_v).cuda()
lab3 = [[9000] + np.random.randint(0, 8999, 7 + i).tolist() + [8999] for i in range(5)]
l11 = sv.loss((inputs, lab3)); l11.backward()              # scheduled sampling: per-step projection
sv.scheduled_sampling = False
l12 = sv.loss((inputs, lab3)); l12.backward()              # one projection over all rows
sv.set_eval()
print("seq2seq C=9000 ok", l11.item(), l12.item(),
      [len(h) for h in sv.infer((inputs, lab3), max_len=6)],
      sv.beam_search(([inputs[0]], [lab3[0]]), beam_size=8, max_len=5))
torch.cuda.synchronize()
# the CTC model at a subword-sized vocabulary (V = 20001): the compact loss path (column map, row
# compaction, fused lattice at the compact width, gradient expansion) and the shortlist beam search
cv = CTC(80, 20000, cfg).cuda()
labels4 = [np.random.randint(0, 20000, 7 + i).tolist() for i in range(5)]
l13 = cv.loss((inputs, labels4)); l13.backward()
print("ctc V=20001 ok", l13.item(), [len(p) for p in cv.infer((inputs, labels4), beam_size=8)])
lp = torch.log_softmax(torch.randn(2, 30, 29, device="cuda"), 2).contiguous()
lens = torch.tensor([30, 21], dtype=torch.int32, device="cuda")
import ctypes
lib = _lib.load()
nb = ctypes.c_size_t(0)
lib.sb_ctc_prefix_beam_workspace_size(2, 30, 4, ctypes.byref(nb))
ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
o_lab = torch.empty(2, 30, dtype=torch.int32, device="cuda")
o_len = torch.empty(2, dtype=torch.int32, device="cuda")
o_sc = torch.empty(2, dtype=torch.float64, device="cuda")
_lib.check(lib.sb_ctc_prefix_beam_shortlist(lp.data_ptr(), lens.data_ptr(), 2, 30, 29, 4, 28,
                                            o_lab.data_ptr(), o_len.data_ptr(), o_sc.data_ptr(),
                                            ws.data_ptr(), nb.value, _lib.stream_ptr()),
           "sb_ctc_prefix_beam_shortlist")
# the LM-fused shortlist kernel, forced, with a weight strong enough that its bound check fails
# on some frames (so the rescan runs too)
_lib.check(lib.sb_ctc_prefix_beam_lm_shortlist(lp.data_ptr(), lens.data_ptr(), 2, 30, 29, 4, 28,
                                               ctypes.byref(lm.device_tables(lp.device)[0]), 2.0,
                                               1.0, o_lab.data_ptr(), o_len.data_ptr(),
                                               o_sc.data_ptr(), ws.data_ptr(), nb.value,
                                               _lib.stream_ptr()),
           "sb_ctc_prefix_beam_lm_shortlist")
_resc = ctypes.c_ulonglong(0)
_lib.check(lib.sb_debug_ctc_lm_rescans(ctypes.byref(_resc)), "sb_debug_ctc_lm_rescans")
print("LM shortlist route ok", o_len.tolist(), "frames rescanned:", _resc.value)
acts = torch.randn(2, 30, 29, device="cuda")
nc = ctypes.c_size_t(0)
lib.sb_ctc_compact_workspace_size(2, 30, 29, 3, ctypes.byref(nc))
wc = torch.empty(nc.value, dtype=torch.uint8, device="cuda")
# [labels | offsets | label_lens | act_lens]
dl = torch.tensor([1, 2, 2, 3, 4, 5, 0, 3, 3, 3, 30, 21], dtype=torch.int32, device="cuda")
g = torch.empty_like(acts)
c = torch.empty(2, device="cuda")
_lib.check(lib.sb_ctc_fwd_bwd_compact(acts.data_ptr(), g.data_ptr(), dl.data_ptr(),
                                      dl[6:].data_ptr(), dl[8:].data_ptr(), dl[10:].data_ptr(), 2,
                                      30, 29, 28, 3, c.data_ptr(), wc.data_ptr(), nc.value,
                                      _lib.stream_ptr()), "sb_ctc_fwd_bwd_compact")
torch.cuda.synchronize()
print("ctc compact / shortlist entries ok", c.tolist(), o_len.tolist())
# the Transducer at a subword-sized vocabulary (V+1 = 20001): infer's shortlist route (slab joint
# with the shortlist producer, then the shortlist beam search), the producer on a given lattice and
# the search's flag rerun at 64-entry lists
tv = Transducer(80, 20000, cfg).cuda()
l14 = tv.loss((inputs, labels4)); l14.backward()
print("transducer V+1=20001 ok", l14.item(), [len(p) for p in tv.infer((inputs, labels4), beam_size=4)])
from speech_b200.transducer_decoders import decode_static
sys.path.insert(0, "tests")
from test_rnnt_shortlist_host import tie_lattice          # the lattice the tests flag
tie, blank = tie_lattice()
print("rnnt shortlist rerun ok", decode_static(tie, 2, blank))
torch.cuda.synchronize()
# label-free search (csrc/rnnt_search.cu): prediction step, rounds, frame ends, final backtrack;
# full candidate lists at V+1 = 29, shortlists at V+1 = 301 (beam 32) and 20001
for tm, V1, beam in ((t, 29, 4), (t2, 301, 32), (tv, 20001, 4)):
    tm.set_eval()
    print("recognize V+1=%d beam %d" % (V1, beam),
          [len(p) for p in tm.recognize(inputs[:3], beam_size=beam, max_symbols_per_frame=2)])
# with an n-gram LM: the fused rows and the f64 rounds, full rows at V+1 = 29, shortlists at
# V+1 = 301 (forced, as the split selection above) and 20001
from speech_b200 import transducer_decoders as tdec
lm_t = NGramLM.train(labels, 3, 29, 28)
print("recognize with LM V+1=29", [len(p) for p in t.recognize(
    inputs[:3], beam_size=4, max_symbols_per_frame=2, lm=lm_t, lm_weight=0.5,
    insertion_bonus=1.0)])
fits_t = tdec.decode_static_fits
tdec.decode_static_fits = lambda K, V: False     # the shortlist route with the LM
lm_t2 = NGramLM.train(labels2, 3, 301, 300)
print("recognize with LM V+1=301, shortlists", [len(p) for p in t2.recognize(
    inputs[:3], beam_size=4, max_symbols_per_frame=2, lm=lm_t2, lm_weight=0.5,
    insertion_bonus=1.0)])
tdec.decode_static_fits = fits_t
lm_tv = NGramLM.train(labels4, 3, 20001, 20000)
print("recognize with LM V+1=20001", [len(p) for p in tv.recognize(
    inputs[:3], beam_size=4, max_symbols_per_frame=2, lm=lm_tv, lm_weight=0.5,
    insertion_bonus=1.0)])
torch.cuda.synchronize()
# Viterbi alignments: CTC at V = 29 and at V = 20001 (the compact rows), with an infeasible
# utterance; the Transducer on the resident joint (V+1 = 29) and the slab joint (V+1 = 301)
print("ctc align", m.align((inputs, labels[:4] + [[3] * 60])))
print("ctc align V=20001", cv.align((inputs, labels4)))
for tm in (t, t2):
    tm.set_eval()
    print("transducer align", tm.align((inputs, labels if tm is t else labels2)))
torch.cuda.synchronize()
# long transcripts: the Viterbi kernels with 2, 4 and 8 states (CTC) and 2 and 4 columns (Transducer)
# per thread
from speech_b200.functions import ctc as ctc_fn, transducer as rnnt_fn
for L in (200, 400, 900):
    T = L + L // 2 + 10
    lab = torch.from_numpy(np.random.randint(0, 28, L).astype(np.int32))
    path, sc = ctc_fn.ctc_viterbi(torch.randn(2, T, 29, device="cuda"), torch.cat([lab, lab]),
                                  torch.tensor([T, T - 5]), torch.tensor([L, L]))
    print("ctc viterbi L=%d" % L, sc.tolist())
fc2 = torch.nn.Linear(64, 29).cuda()
for U in (300, 700):
    ym = torch.from_numpy(np.random.randint(0, 28, (2, U)))
    fr, sc = rnnt_fn.rnnt_viterbi(torch.randn(2, 40, 64, device="cuda"),
                                  torch.randn(2, U + 1, 64, device="cuda"), fc2, ym,
                                  ym.reshape(-1).int(), torch.tensor([40, 30]),
                                  torch.tensor([U, U]), 28)
    print("rnnt viterbi U=%d" % U, sc.tolist())
torch.cuda.synchronize()
# Transducer streaming with an LM: the resumed search (reset, rounds over local frames, the
# parity copy) on the full route (V+1 = 29) and the 64-entry shortlist route (V+1 = 20001)
cfg_s = {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                                     "rnn": {"dim": 64, "bidirectional": False, "layers": 2}},
         "decoder": {"embedding_dim": 16, "layers": 1}}
for V, lm_s in ((28, lm_t), (20000, lm_tv)):
    ts = Transducer(80, V, cfg_s).cuda()
    ts.set_eval()
    st = ts.stream(3, beam_size=4, max_symbols_per_frame=2, max_frames=64, lm=lm_s,
                   lm_weight=0.5, insertion_bonus=1.0)
    for p, k in ((0, 17), (17, 5), (22, 40)):
        st.push([x[p:p + k] for x in inputs[:3]])
    st.reset(1)
    st.push([inputs[0][:0], inputs[3][:30], inputs[2][:0]])
    print("transducer stream V+1=%d" % (V + 1), st.frames, st.partial(return_scores=True))
torch.cuda.synchronize()
# the direct-convolution kernels of the conv layers past the first (forward, data and weight
# gradient): the benchmark's stack, a stride-3 layer and a stack with dropout
from speech_b200 import ops
for specs, B, T, F, p in (([[32, 5, 8, 2], [32, 5, 8, 2]], 2, 60, 80, 0.0),
                          ([[16, 3, 4, 1], [8, 2, 3, 3]], 2, 33, 21, 0.0),
                          ([[16, 5, 8, 2], [24, 3, 4, 1]], 2, 40, 40, 0.3)):
    layers, in_c = [], 1
    for out_c, kh, kw, st in specs:
        layers += [torch.nn.Conv2d(in_c, out_c, (kh, kw), stride=(st, st)), torch.nn.ReLU(),
                   torch.nn.Dropout(p)]
        in_c = out_c
    conv = torch.nn.Sequential(*layers).cuda()
    ops.profile_begin()
    y = ops.conv_stack(torch.randn(B, T, F, device="cuda"), conv, True)
    y.sum().backward()
    print("direct conv", specs, "dropout", p, sorted(n for n in ops.profile_end() if "direct" in n))
torch.cuda.synchronize()
# word-LM fusion: sb_ctc_prefix_beam_wordlm on the full scan (infer) and the forced shortlist
# route, and a CTC stream stepped with the word LM (stream step and best)
from speech_b200.lm import WordLM
wsyms = [chr(ord("a") + i) for i in range(26)] + ["'", " "]
wlm = WordLM.train(["abc de f", "de abc", "f f abc", "b'c de"], 3, wsyms, oov_penalty=-2.0)
print("infer with word LM", [len(p) for p in m.infer((inputs, labels), beam_size=4, lm=wlm,
                                                       lm_weight=0.5, insertion_bonus=1.0)])
_lib.check(lib.sb_ctc_prefix_beam_wordlm_shortlist(
    lp.data_ptr(), lens.data_ptr(), 2, 30, 29, 4, 28, ctypes.byref(wlm.device_tables(lp.device)[0]),
    0.5, 1.0, -2.0, o_lab.data_ptr(), o_len.data_ptr(), o_sc.data_ptr(), ws.data_ptr(), nb.value,
    _lib.stream_ptr()), "sb_ctc_prefix_beam_wordlm_shortlist")
print("word LM shortlist route ok", o_len.tolist())
cs = CTC(80, 28, {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2], [8, 5, 8, 2]],
                                              "rnn": {"dim": 64, "bidirectional": False,
                                                      "layers": 2}}}).cuda()
cs.set_eval()
st = cs.stream(3, beam_size=4, max_frames=64, lm=wlm, lm_weight=0.5, insertion_bonus=1.0)
for p, k in ((0, 17), (17, 5), (22, 40)):
    st.push([x[p:p + k] for x in inputs[:3]])
print("ctc stream with word LM", st.frames, st.partial(return_scores=True))
torch.cuda.synchronize()
