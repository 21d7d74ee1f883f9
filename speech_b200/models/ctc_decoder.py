"""CTC prefix beam search - drop-in for speech/models/ctc_decoder.py:38-113 (reference).

`decode(probs, beam_size=10, blank=0)` keeps the reference's signature and return value
((label tuple, negative log-likelihood)); the search itself runs in the sm_90a kernel
sb_ctc_prefix_beam (csrc/decode.cu), one CTA per utterance.  `decode_batch` is the batched
entry CTC.infer uses (the reference loops over utterances in Python, ctc_model.py:59-60).

Both take an optional n-gram LM for shallow fusion, and the returned score is then the fused one:
  * speech_b200.lm.NGramLM, over the model's classes: an extension by symbol s scores
    p_s + (lm_weight * lm(s | prefix) + insertion_bonus) in place of p_s (sb_ctc_prefix_beam_lm);
  * speech_b200.lm.WordLM, over words (Hannun et al. 2014): the delimiter that ends a word scores
    p_s + ((lm_weight * lm(word | words) + insertion_bonus) + OOV penalty), so insertion_bonus is
    per word; a word leaving the lexicon is charged the LM's oov_penalty once, and the end of the
    utterance adds the trailing word and </s> (sb_ctc_prefix_beam_wordlm, include/speech_b200.h).
Without an LM the calls are the LM-less search.

`StreamSearch` owns the state of the resumable search (sb_ctc_stream_*) that CTC.stream,
Seq2Seq.stream and the attention model's two-pass first pass advance frame by frame.
"""
import math

import numpy as np
import torch

from .. import _lib, ops
from ..lm import NGramLM, WordLM, fusion_args, fusion_kind

# entry points by LM kind, and the stream's with their ops._launch profile names
_OFFLINE = {None: "sb_ctc_prefix_beam", NGramLM: "sb_ctc_prefix_beam_lm",
            WordLM: "sb_ctc_prefix_beam_wordlm"}
_STREAM_STEP = {None: ("ctc_stream_step", "sb_ctc_stream_step"),
                NGramLM: ("ctc_stream_step_lm", "sb_ctc_stream_step_lm"),
                WordLM: ("ctc_stream_step_wordlm", "sb_ctc_stream_step_wordlm")}
# only a word LM changes the ranking at the end (the partial word and </s>)
_STREAM_BEST = {None: ("ctc_stream_best", "sb_ctc_stream_best"),
                NGramLM: ("ctc_stream_best", "sb_ctc_stream_best"),
                WordLM: ("ctc_stream_best_wordlm", "sb_ctc_stream_best_wordlm")}


def check_lm(lm, lm_weight, insertion_bonus, num_classes, blank, search="CTC"):
    """ValueError unless the fusion arguments are usable with a model of num_classes classes whose
    blank is `blank`; `search` names the search in the refusal of an LM with an end class"""
    if lm is None:
        if lm_weight != 0.0 or insertion_bonus != 0.0:
            raise ValueError("lm_weight / insertion_bonus need an lm")
        return
    if isinstance(lm, WordLM) and search != "CTC":
        raise ValueError("a word LM fuses into the CTC search only; the %s search takes an NGramLM"
                         % search)
    if lm.end is not None:
        raise ValueError("the LM reads class %d as </s>; the %s search has no end class"
                         % (lm.end, search))
    if lm.num_classes != num_classes:
        raise ValueError("the LM covers %d classes, the model has %d"
                         % (lm.num_classes, num_classes))
    if lm.blank != blank:
        raise ValueError("the LM's blank is class %d, the search's is %d" % (lm.blank, blank))
    if not (math.isfinite(lm_weight) and lm_weight >= 0.0):
        raise ValueError("lm_weight must be finite and >= 0, got %r" % (lm_weight,))
    if not math.isfinite(insertion_bonus):
        raise ValueError("insertion_bonus must be finite, got %r" % (insertion_bonus,))


def _run(logp, lens, beam_size, blank, lm=None, lm_weight=0.0, insertion_bonus=0.0):
    lib = _lib.load()
    B, T, S = logp.shape
    dev = logp.device
    kind = fusion_kind(lm)
    if kind is NGramLM:
        nbytes = _lib.workspace_size(lib.sb_ctc_prefix_beam_lm_workspace_size, B, T, beam_size,
                                     lm.order)
    else:
        nbytes = _lib.workspace_size(lib.sb_ctc_prefix_beam_workspace_size, B, T, beam_size)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out_labels = torch.empty(B, T, dtype=torch.int32, device=dev)
    out_lens = torch.empty(B, dtype=torch.int32, device=dev)
    out_scores = torch.empty(B, dtype=torch.float64, device=dev)
    outs = (out_labels.data_ptr(), out_lens.data_ptr(), out_scores.data_ptr(), ws.data_ptr(),
            nbytes, _lib.stream_ptr())
    name = _OFFLINE[kind]
    with torch.cuda.device(dev):
        fusion = fusion_args(lm, lm_weight, insertion_bonus, dev)
        _lib.check(getattr(lib, name)(logp.data_ptr(), lens.data_ptr(), B, T, S, int(beam_size),
                                      int(blank), *fusion, *outs), name)
    labels = out_labels.cpu().numpy()
    n = out_lens.cpu().numpy()
    scores = out_scores.cpu().numpy()
    return [(tuple(int(v) for v in labels[b, :n[b]]), float(scores[b])) for b in range(B)]


def decode_batch(probs, beam_size=10, blank=0, lens=None, with_scores=False, lm=None,
                 lm_weight=0.0, insertion_bonus=0.0):
    """probs (B, T, S) post-softmax CUDA tensor -> list of label tuples (one per utterance).
    lm: an NGramLM over the S classes, fused with lm_weight >= 0 and insertion_bonus; the scores
    (with_scores) are then acoustic + lm_weight * LM + insertion_bonus * length.  Or a WordLM
    spelled in the S classes: insertion_bonus is then per word, and the scores are acoustic +
    lm_weight * word LM (</s> included) + insertion_bonus * words + oov_penalty * OOV words."""
    _lib.require_cuda(probs, "probs")
    check_lm(lm, lm_weight, insertion_bonus, probs.shape[-1], blank)
    logp = torch.log(probs.detach().float()).contiguous()
    B, T, S = logp.shape
    if lens is None:
        lens = torch.full((B,), T, dtype=torch.int32, device=probs.device)
    else:
        lens = torch.as_tensor(lens, dtype=torch.int32).to(probs.device)
    res = _run(logp, lens, beam_size, blank, lm, lm_weight, insertion_bonus)
    return res if with_scores else [r[0] for r in res]


def decode(probs, beam_size=10, blank=0, lm=None, lm_weight=0.0, insertion_bonus=0.0):
    """Reference signature: probs (T, S) array of post-softmax probabilities (host).

    Returns (label tuple, negative log-likelihood).  The log is taken on the host in the input
    dtype exactly as the reference does (np.log, ctc_decoder.py:52); the beam search runs on
    cuda:current.  lm, lm_weight, insertion_bonus: as decode_batch (the score is then the fused
    one).
    """
    if not torch.cuda.is_available():
        raise _lib.SpeechB200Error("speech_b200: decode() needs a CUDA device (no CPU path)")
    probs = np.asarray(probs)
    check_lm(lm, lm_weight, insertion_bonus, probs.shape[-1], blank)
    with np.errstate(divide="ignore"):
        logp = np.log(probs)
    lp = torch.from_numpy(np.ascontiguousarray(logp, dtype=np.float32))[None].cuda()
    lens = torch.full((1,), lp.shape[1], dtype=torch.int32, device=lp.device)
    return _run(lp, lens, beam_size, blank, lm, lm_weight, insertion_bonus)[0]


class StreamSearch:
    """The resumable prefix beam search of B streams (sb_ctc_stream_*): each stream's beam stays
    on the device between pushes, for up to max_frames frames per stream between resets.  lm,
    lm_weight, insertion_bonus: as decode_batch (the caller checks them); a WordLM's oov_penalty
    is read at each launch."""

    def __init__(self, B, max_frames, beam_size, blank, device, lm=None, lm_weight=0.0,
                 insertion_bonus=0.0):
        lib = _lib.load()
        self.B, self.Tm, self.K, self.blank, self.dev = (int(B), int(max_frames), int(beam_size),
                                                         int(blank), device)
        self.lm, self.lm_weight, self.insertion_bonus = lm, lm_weight, insertion_bonus
        self.kind = fusion_kind(lm)
        nbytes = _lib.workspace_size(lib.sb_ctc_stream_state_size, self.B, self.Tm, self.K,
                                     0 if lm is None else lm.order)
        self.state = torch.empty(nbytes, dtype=torch.uint8, device=device)
        self.reset(0, self.B)

    def _fusion(self):
        return fusion_args(self.lm, self.lm_weight, self.insertion_bonus, self.dev)

    def reset(self, first, count):
        """streams first .. first + count - 1 back to the empty prefix at frame 0"""
        lib = _lib.load()
        with torch.cuda.device(self.dev):
            ops._launch("ctc_stream_reset", 0.0, lambda: lib.sb_ctc_stream_reset(
                self.state.data_ptr(), self.B, self.Tm, self.K, first, count, _lib.stream_ptr()))

    def push(self, logp, counts):
        """advance stream b by counts[b] frames of logp (B, T, S), contiguous float32
        log-probabilities"""
        lib = _lib.load()
        B, T, S = logp.shape
        n = torch.tensor(list(counts), dtype=torch.int32).to(self.dev)
        ws_bytes = _lib.workspace_size(lib.sb_ctc_stream_workspace_size, B, T, self.K)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.dev)
        name, symbol = _STREAM_STEP[self.kind]
        with torch.cuda.device(self.dev):
            fusion = self._fusion()
            ops._launch(name, 0.0, lambda: getattr(lib, symbol)(
                logp.data_ptr(), n.data_ptr(), B, T, S, self.K, self.blank, *fusion, self.Tm,
                self.state.data_ptr(), ws.data_ptr(), ws_bytes, _lib.stream_ptr()))

    def best(self, return_scores=False):
        """Best label tuple of each stream so far (one device-to-host copy); with return_scores,
        (labels, score) pairs, the score as decode_batch(with_scores=True) reports it.  With a
        WordLM the stored beams are ranked by the end-of-utterance rule, as if each stream ended
        here (its partial word completed, then </s>)."""
        lib = _lib.load()
        B, Tm = self.B, self.Tm
        off = B * Tm + 2 * B + (B * Tm) % 2          # float64 scores 8-byte aligned
        buf = torch.empty(off + 2 * B, dtype=torch.int32, device=self.dev)
        labels, lens, ovf = buf[:B * Tm], buf[B * Tm:B * Tm + B], buf[B * Tm + B:B * Tm + 2 * B]
        scores = buf[off:].view(torch.float64)
        name, symbol = _STREAM_BEST[self.kind]
        with torch.cuda.device(self.dev):
            fusion = self._fusion() if self.kind is WordLM else ()
            ops._launch(name, 0.0, lambda: getattr(lib, symbol)(
                self.state.data_ptr(), B, Tm, self.K, *fusion, labels.data_ptr(), lens.data_ptr(),
                scores.data_ptr(), ovf.data_ptr(), _lib.stream_ptr()))
        host = buf.cpu()
        lab = host[:B * Tm].view(B, Tm).numpy()
        n = host[B * Tm:B * Tm + B].numpy()
        sc = host[off:].view(torch.float64).numpy()
        res = [tuple(int(v) for v in lab[b, :n[b]]) for b in range(B)]
        return [(r, float(s)) for r, s in zip(res, sc)] if return_scores else res

    def nbest(self):
        """Every stored beam entry of every stream (sb_ctc_stream_nbest), on the device: labels
        (B, K, max_frames) int32, lens (B, K) int32 (-1: empty slot), c (B, K) float64
        log-probabilities lse(p_b, p_nb) (-inf: empty slot), in the search's stored order"""
        lib = _lib.load()
        B, Tm, K, dev = self.B, self.Tm, self.K, self.dev
        labels = torch.empty(B, K, Tm, dtype=torch.int32, device=dev)
        lens = torch.empty(B, K, dtype=torch.int32, device=dev)
        c = torch.empty(B, K, dtype=torch.float64, device=dev)
        count = torch.empty(B, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            ops._launch("ctc_stream_nbest", 0.0, lambda: lib.sb_ctc_stream_nbest(
                self.state.data_ptr(), B, Tm, K, labels.data_ptr(), lens.data_ptr(),
                c.data_ptr(), count.data_ptr(), _lib.stream_ptr()))
        return labels, lens, c
