"""Joint CTC/attention training and decoding of the attention model on the GPU
(Seq2Seq(ctc_weight) / recognize(ctc_weight, ctc_prebeam) -> functions/s2s.py: beam_search_batch
-> csrc/s2s_ctc.cu):

- the search equals the float64 reference loop of tests/s2s_ctc_ref.py over decode_step (tokens
  exact, scores to 1e-9 relative) over beams, pre-beams, weights, with and without a 3-gram LM,
  on the fused and the many-CTA projection;
- each utterance of a batch gets its B = 1 search bit for bit, also in the exact-lengths mode, and
  a model with a head at ctc_weight = 0 gives the plain search bit for bit;
- the CTC scores decide where the attention does not, and overrule an early END;
- the joint loss and its gradients equal their two parts';
- the scoring and extension kernels alone, on hand-built beams (the root, a repeated label, END,
  T_b < T', too few frames), equal the float64 prefix scorer, -inf exactly where it is.
"""
import ctypes

import numpy as np
import pytest
import torch

from s2s_ctc_ref import beam_search_ctc

pytestmark = pytest.mark.gpu


def _cfg(H=32, layers=2, w=0.3):
    return {"dropout": 0.0, "encoder": {"conv": [[8, 5, 8, 2]],
                                        "rnn": {"dim": H, "bidirectional": True, "layers": layers}},
            "decoder": {"embedding_dim": H, "layers": 1, "ctc_weight": w}}


def _model(V, seed, exact=False, sharpen=2.0, H=32, layers=2):
    from speech_b200.models import Seq2Seq
    torch.manual_seed(seed)
    np.random.seed(seed)
    cfg = _cfg(H, layers)
    if exact:
        cfg = dict(cfg, exact_lengths=True)
    m = Seq2Seq(40, V, cfg).cuda()
    m.set_eval()
    with torch.no_grad():
        m.fc.fc.weight.mul_(sharpen)
        m.embedding.weight.mul_(3.0)
        m.ctc_fc.fc.weight.mul_(4.0)
    return m


def _inputs(T, n=3, step=9, seed=0):
    rng = np.random.RandomState(seed)
    return [rng.randn(T - step * i, 40).astype(np.float32) for i in range(n)]


def _encode(m, inputs):
    lens = m.input_lens(inputs)
    with torch.no_grad():
        x = m._encode(m.stage_inputs(inputs), lens)
        y = torch.log_softmax(m.ctc_fc(x).float(), dim=-1).contiguous()
    return x, y, lens


def _check_against_reference(m, inputs, K, M, w, max_len, lm=None, ref_lm=None, a=0.0, bonus=0.0):
    V = m.embedding.num_embeddings
    x, y, _ = _encode(m, inputs)
    labels, scores = m.recognize(inputs, beam_size=K, max_len=max_len, return_scores=True, lm=lm,
                                 lm_weight=a, insertion_bonus=bonus, ctc_weight=w, ctc_prebeam=M)
    Mr = min(V - 1, 3 * K // 2) if M is None else M
    yh = y.cpu().numpy()
    for b in range(len(inputs)):
        ref, ref_score = beam_search_ctc(m, x[b:b + 1], yh[b], yh.shape[1], V - 1, V - 2, K,
                                         max_len, w, Mr, ref_lm, a, bonus)
        assert labels[b] == list(ref), (K, M, w, b, labels[b], ref)
        assert abs(scores[b] - ref_score) <= 1e-9 * max(1.0, abs(ref_score)), (K, M, w, b)


@pytest.mark.parametrize("w", [0.3, 0.7])
@pytest.mark.parametrize("M", [1, None, 10])
@pytest.mark.parametrize("K", [1, 4, 10])
def test_search_equals_the_reference_loop(cuda_lib, K, M, w):
    V = 11
    m = _model(V, 30)
    _check_against_reference(m, _inputs(80, seed=1), K, M, w, 12)


@pytest.mark.parametrize("K,M", [(1, None), (4, None), (4, 10)])
def test_search_with_a_3gram_lm_equals_the_reference_loop(cuda_lib, tmp_path, K, M):
    from speech_b200.lm import NGramLM
    from s2s_lm_ref import EndArpaLM
    V = 11
    m = _model(V, 31)
    rng = np.random.RandomState(8)
    sents = [[V - 1] + rng.randint(0, V - 2, rng.randint(0, 10)).tolist() + [V - 2]
             for _ in range(60)]
    lm = NGramLM.train(sents, 3, V, V - 1, end=V - 2)
    syms = {c: ("w%d" % c if c < V - 2 else ("</s>", "<s>")[c - V + 2]) for c in range(V)}
    p = str(tmp_path / "lm.arpa")
    lm.to_arpa(p, syms)
    ref_lm = EndArpaLM(p, [syms[c] for c in range(V)], V - 1, V - 2)
    _check_against_reference(m, _inputs(80, seed=2), K, M, 0.4, 12, lm, ref_lm, 0.6, 0.3)


def test_many_cta_projection_equals_the_reference_loop(cuda_lib):
    from speech_b200.functions import s2s
    V = 5001
    m = _model(V, 32, sharpen=1.0, H=64, layers=1)
    assert not s2s.fc_fused(64, V - 1)
    _check_against_reference(m, _inputs(60, n=2, step=7, seed=3), 4, None, 0.3, 5)


def _single(m, x, y, b, K, max_len, w, M, frames=None):
    from speech_b200.functions import s2s
    V = m.embedding.num_embeddings
    n = x.shape[1] if frames is None else frames
    with torch.no_grad():
        (toks, score, _), = s2s.beam_search_batch(m, x[b:b + 1, :n], V - 1, V - 2, K, max_len,
                                                  ctc=(y[b:b + 1, :n].contiguous(), w, M))
    return list(toks), score


@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("K", [1, 4, 10])
def test_batch_equals_single_utterance_search(cuda_lib, K, exact):
    V = 11
    m = _model(V, 33, exact=exact)
    inputs = _inputs(100, n=4, step=15, seed=4)
    x, y, lens = _encode(m, inputs)
    if exact:
        assert len(set(lens)) == len(lens)
    labels, scores = m.recognize(inputs, beam_size=K, max_len=15, return_scores=True,
                                 ctc_weight=0.5)
    M = min(V - 1, 3 * K // 2)
    for b in range(len(inputs)):
        assert (labels[b], scores[b]) == _single(m, x, y, b, K, 15, 0.5, M,
                                                 lens[b] if exact else None), (K, b)


@pytest.mark.parametrize("K", [1, 4])
def test_a_head_at_weight_zero_gives_the_plain_search(cuda_lib, K):
    V = 11
    m = _model(V, 34)
    inputs = _inputs(90, seed=5)
    plain = m.recognize(inputs, beam_size=K, max_len=15, return_scores=True)
    assert m.recognize(inputs, beam_size=K, max_len=15, return_scores=True,
                       ctc_weight=0.0) == plain
    del m.ctc_fc
    m.ctc_weight = 0.0
    assert m.recognize(inputs, beam_size=K, max_len=15, return_scores=True) == plain


def _spelled(B, T, C, seq, peak=8.0):
    """CTC log-probs (B, T, C) whose best path spells seq: each label on two frames, blanks between"""
    x = torch.zeros(B, T, C)
    x[:, :, C - 1] = peak
    t = 1
    for s in seq:
        x[:, t:t + 2, C - 1] = 0.0
        x[:, t:t + 2, s] = peak
        t += 4
    return torch.log_softmax(x, -1).cuda().contiguous()


@pytest.mark.parametrize("K", [1, 4])
def test_uniform_attention_spells_the_ctc_sequence(cuda_lib, K):
    from speech_b200.functions import s2s
    V = 12
    m = _model(V, 35)
    with torch.no_grad():
        m.fc.fc.weight.zero_()
        m.fc.fc.bias.zero_()
    x, _, _ = _encode(m, _inputs(140, n=2, step=9, seed=6))
    seq = [3, 7, 1, 1, 8, 0]
    y = _spelled(x.shape[0], x.shape[1], V - 1, seq)
    res = s2s.beam_search_batch(m, x, V - 1, V - 2, K, 20, ctc=(y, 0.5, V - 1))
    assert [list(r[0]) for r in res] == [[V - 1] + seq + [V - 2]] * x.shape[0]


def test_ctc_overrules_an_early_end(cuda_lib):
    from speech_b200.functions import s2s
    V = 12
    m = _model(V, 36)
    with torch.no_grad():
        m.fc.fc.weight.zero_()
        m.fc.fc.bias.zero_()
        m.fc.fc.bias[V - 2] = 3.0                       # END first everywhere
    x, _, _ = _encode(m, _inputs(140, n=2, step=9, seed=7))
    seq = [5, 2, 9]
    y = _spelled(x.shape[0], x.shape[1], V - 1, seq)
    plain = s2s.beam_search_batch(m, x, V - 1, V - 2, 4, 20)
    assert [list(r[0]) for r in plain] == [[V - 1, V - 2]] * x.shape[0]
    res = s2s.beam_search_batch(m, x, V - 1, V - 2, 4, 20, ctc=(y, 0.5, V - 1))
    assert [list(r[0]) for r in res] == [[V - 1] + seq + [V - 2]] * x.shape[0]


def _batch(V, n, seed, T=90):
    rng = np.random.RandomState(seed)
    inputs = [rng.randn(T - 7 * i, 40).astype(np.float32) for i in range(n)]
    labels = [[V - 1] + rng.randint(0, V - 2, rng.randint(1, 6)).tolist() + [V - 2]
              for _ in range(n)]
    return inputs, labels


@pytest.mark.parametrize("exact", [False, True])
def test_joint_loss_and_gradients_are_the_sum_of_their_parts(cuda_lib, exact):
    from speech_b200.models import Seq2Seq
    V, w = 11, 0.4
    torch.manual_seed(40)
    cfg = _cfg(w=w)
    if exact:
        cfg = dict(cfg, exact_lengths=True)
    m = Seq2Seq(40, V, cfg).cuda()
    m.set_train()
    m.scheduled_sampling = False
    inputs, labels = _batch(V, 4, 41)
    B = len(inputs)
    loss = m.loss((inputs, labels))
    loss.backward()
    g_joint = {k: p.grad.detach().clone() for k, p in m.named_parameters()}
    # the attention part: a head-less copy with the same weights
    cfg0 = dict(cfg, decoder=dict(cfg["decoder"], ctc_weight=0))
    m0 = Seq2Seq(40, V, cfg0).cuda()
    m0.load_state_dict({k: v for k, v in m.state_dict().items() if not k.startswith("ctc_fc")})
    m0.set_train()
    m0.scheduled_sampling = False
    ce = m0.loss((inputs, labels))
    ce.backward()
    # the CTC part over the head's logits, in float64 on the CPU
    lens = m.input_lens(inputs)
    m.zero_grad()
    x = m._encode(m.stage_inputs(inputs), lens)
    logits = m.ctc_fc(x)
    lg = logits.detach().cpu().double().requires_grad_(True)
    frames = lens if lens is not None else [logits.shape[1]] * B
    tg = torch.tensor([t for s in labels for t in s[1:-1]])
    ctc = torch.nn.functional.ctc_loss(lg.log_softmax(-1).transpose(0, 1), tg,
                                       torch.tensor(frames), torch.tensor([len(s) - 2 for s in labels]),
                                       blank=V - 2, reduction="sum", zero_infinity=False)
    want = (1 - w) * float(ce) + w * float(ctc) / B
    assert abs(float(loss) - want) <= 1e-4 * abs(want), (float(loss), want)
    ctc.backward()
    logits.backward((lg.grad * (w / B)).float().cuda())
    for k, p in m0.named_parameters():
        ref = (1 - w) * p.grad
        if m.get_parameter(k).grad is not None:
            ref = ref + m.get_parameter(k).grad
        # the weight gradients run on bf16 GEMM operands: the joint pass rounds the summed (or
        # (1 - w)-scaled) gradients, the parts round theirs separately
        tol = 1e-2 * float(ref.abs().max()) + 1e-6
        assert float((g_joint[k] - ref).abs().max()) <= tol, k
    for k in ("ctc_fc.fc.weight", "ctc_fc.fc.bias"):
        ref = m.get_parameter(k).grad
        tol = 1e-2 * float(ref.abs().max()) + 1e-6
        assert float((g_joint[k] - ref).abs().max()) <= tol, k


# ---------------------------------------------------------------------------------------------
# the scoring and extension kernels alone, on hand-built beams
# ---------------------------------------------------------------------------------------------
class _BeamState(ctypes.Structure):
    """the layout of csrc/s2s_beam.cuh's BeamState (its size is checked against the library's)"""
    _fields_ = [("done", ctypes.c_int), ("out_len", ctypes.c_int),
                ("score", ctypes.c_double * 32), ("node", ctypes.c_int * 32),
                ("token", ctypes.c_int * 32), ("nlive", ctypes.c_int), ("ncomplete", ctypes.c_int),
                ("best_c_score", ctypes.c_double), ("best_c_node", ctypes.c_int),
                ("have_complete", ctypes.c_int), ("nodes_used", ctypes.c_int),
                ("final_score", ctypes.c_double)]


def _logsm(rng, *shape):
    x = torch.from_numpy(rng.randn(*shape) * 2.0).float()
    return torch.log_softmax(x, -1).contiguous()


def _close(got, ref, what):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    assert np.array_equal(np.isneginf(got), np.isneginf(ref)), (what, got, ref)
    f = np.isfinite(ref)
    assert np.all(np.abs(got[f] - ref[f]) <= 1e-10 * np.maximum(1.0, np.abs(ref[f]))), \
        (what, got, ref)


# rows of each utterance: the root, a label, a repeat of the last label, and a hypothesis as long
# as utterance 1's frames (its label extensions have too few frames: psi = -inf)
HYPS = [(), (2,), (4, 4), (0, 1, 0, 1, 0, 1)]


@pytest.mark.parametrize("M", [7, 3])
@pytest.mark.parametrize("w", [0.3, 0.7])
def test_scoring_and_extension_kernels_equal_the_reference(cuda_lib, M, w):
    from s2s_ctc_ref import prefix_scores, vectors_of
    from speech_b200 import _lib
    lib = _lib.load()
    assert ctypes.sizeof(_BeamState) == _lib.workspace_size(lib.sb_s2s_beam_state_size)
    V, K, B, T = 8, 4, 2, 14
    C, start, end = V - 1, V - 1, V - 2
    lens = [T, 6]                                     # utterance 1: T_b < T'
    rng = np.random.RandomState(int(10 * w) + M)
    y = _logsm(rng, B, T, C)
    logp = _logsm(rng, B * K, C)
    R, node_cap, c_cap, max_len = B * K, 64, 64, 50
    states = (_BeamState * B)()
    nodes = np.zeros((B, node_cap, 2), np.int32)
    A = rng.randn(R) * 3.0
    gam = np.full((2, R, 2, T), -np.inf)
    yh = y.numpy()
    for b in range(B):
        st = states[b]
        nodes[b, 0] = (-1, start)
        used = 1
        for r, h in enumerate(HYPS):
            q = 0
            for tok in h:
                nodes[b, used] = (q, tok)
                q, used = used, used + 1
            st.node[r], st.token[r], st.score[r] = q, (h[-1] if h else start), A[b * K + r]
            gn, gb = vectors_of(yh[b], lens[b], h)
            gam[0, b * K + r, 0, :lens[b]] = gn
            gam[0, b * K + r, 1, :lens[b]] = gb
        st.nlive, st.nodes_used = len(HYPS), used
    dev = torch.device("cuda")
    d_state = torch.frombuffer(bytearray(bytes(states)), dtype=torch.uint8).to(dev)
    d_nodes = torch.from_numpy(nodes).to(dev)
    d_y, d_logp = y.to(dev), logp.to(dev)
    d_lens = torch.tensor(lens, dtype=torch.int32, device=dev)
    nbytes = _lib.workspace_size(lib.sb_s2s_ctc_state_size, K, M, T, B)
    buf = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    dbl = buf[:8 * (R + 4 * R * T + 3 * R * M)].view(torch.float64)
    dbl[:R] = torch.from_numpy(A).to(dev)
    dbl[R:R + 4 * R * T] = torch.from_numpy(gam.reshape(-1)).to(dev)
    stop = torch.zeros(2, dtype=torch.int32, device=dev)
    shape = (K, C, M, T, start, end, w)
    cargs = (d_y.data_ptr(), d_lens.data_ptr(), buf.data_ptr(), nbytes)
    sp = _lib.stream_ptr()
    _lib.check(lib.sb_s2s_ctc_candidates(d_logp.data_ptr(), *cargs[:2], d_state.data_ptr(),
                                         d_nodes.data_ptr(), node_cap, *cargs[2:], *shape, 0,
                                         stop.data_ptr(), B, None, 0.0, 0.0, sp), "candidates")
    torch.cuda.synchronize()
    o = R + 4 * R * T
    val = dbl[o:o + R * M].cpu().numpy().reshape(R, M)
    anew = dbl[o + R * M:o + 2 * R * M].cpu().numpy().reshape(R, M)
    psic = dbl[o + 2 * R * M:o + 3 * R * M].cpu().numpy().reshape(R, M)
    cls = buf[8 * (o + 3 * R * M):].view(torch.int32)[:R * M].cpu().numpy().reshape(R, M)
    lp = logp.numpy().astype(np.float64)
    saw_neginf = False
    for b in range(B):
        for r, h in enumerate(HYPS):
            row = b * K + r
            P = [(1.0 - w) * float(v) for v in lp[row]]
            top = sorted(sorted(range(C), key=lambda c: P[c], reverse=True)[:M])
            gn, gb = vectors_of(yh[b], lens[b], h)
            psi = prefix_scores(yh[b], gn, gb, h[-1] if h else None, top, end)
            assert cls[row].tolist() == top, (b, r)
            assert anew[row].tolist() == [A[row] + P[c] for c in top], (b, r)
            _close(psic[row], psi, ("psi", b, r))
            _close(val[row], [(A[row] + P[c]) + w * p for c, p in zip(top, psi)], ("value", b, r))
            saw_neginf |= bool(np.isneginf(psic[row]).any())
    assert saw_neginf
    # the selection's new rows: their A and vectors, against the hypotheses the arena holds
    c_scores = torch.zeros(B, c_cap, dtype=torch.float64, device=dev)
    parent = torch.zeros(R, dtype=torch.int32, device=dev)
    tok = torch.zeros(R, dtype=torch.int32, device=dev)
    out = torch.zeros(B, max_len + 2, dtype=torch.int32, device=dev)
    _lib.check(lib.sb_s2s_ctc_select_batch(*cargs, d_state.data_ptr(), c_scores.data_ptr(),
                                           d_nodes.data_ptr(), parent.data_ptr(), tok.data_ptr(),
                                           out.data_ptr(), *shape, 0, max_len, node_cap, c_cap,
                                           stop.data_ptr(), B, sp), "select")
    torch.cuda.synchronize()
    after = _BeamState * B
    sts = after.from_buffer_copy(bytes(d_state.cpu().numpy().tobytes()))
    nd = d_nodes.cpu().numpy()
    g1 = dbl[R:R + 4 * R * T].cpu().numpy().reshape(2, R, 2, T)[1]
    a1 = dbl[:R].cpu().numpy()
    for b in range(B):
        st = sts[b]
        assert st.done == 0 and st.nlive > 0
        for k in range(st.nlive):
            h, q = [], st.node[k]
            while nd[b, q, 0] >= 0:
                h.append(int(nd[b, q, 1]))
                q = nd[b, q, 0]
            h = tuple(reversed(h))
            gn, gb = vectors_of(yh[b], lens[b], h)
            _close(g1[b * K + k, 0, :lens[b]], gn, ("gn", b, k))
            _close(g1[b * K + k, 1, :lens[b]], gb, ("gb", b, k))
            r = int(parent[b * K + k])
            j = cls[b * K + r].tolist().index(h[-1])
            assert a1[b * K + k] == anew[b * K + r, j] and st.score[k] == val[b * K + r, j]


@pytest.mark.parametrize("K", [1, 4])
def test_exact_lengths_search_equals_the_reference_loop(cuda_lib, K):
    V = 11
    m = _model(V, 37, exact=True)
    inputs = _inputs(100, n=3, step=15, seed=9)
    x, y, lens = _encode(m, inputs)
    assert len(set(lens)) == len(lens) and max(lens) == x.shape[1]
    labels, scores = m.recognize(inputs, beam_size=K, max_len=12, return_scores=True,
                                 ctc_weight=0.5)
    yh = y.cpu().numpy()
    for b in range(len(inputs)):
        ref, ref_score = beam_search_ctc(m, x[b:b + 1], yh[b], lens[b], V - 1, V - 2, K, 12, 0.5,
                                         min(V - 1, 3 * K // 2), lens=[lens[b]])
        assert labels[b] == list(ref), (K, b, labels[b], ref)
        assert abs(scores[b] - ref_score) <= 1e-9 * max(1.0, abs(ref_score)), (K, b)
