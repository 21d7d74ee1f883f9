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
"""
import math

import numpy as np
import torch

from .. import _lib
from ..lm import WordLM


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
    if lm is None or isinstance(lm, WordLM):
        nbytes = _lib.workspace_size(lib.sb_ctc_prefix_beam_workspace_size, B, T, beam_size)
    else:
        nbytes = _lib.workspace_size(lib.sb_ctc_prefix_beam_lm_workspace_size, B, T, beam_size,
                                     lm.order)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out_labels = torch.empty(B, T, dtype=torch.int32, device=dev)
    out_lens = torch.empty(B, dtype=torch.int32, device=dev)
    out_scores = torch.empty(B, dtype=torch.float64, device=dev)
    outs = (out_labels.data_ptr(), out_lens.data_ptr(), out_scores.data_ptr(), ws.data_ptr(),
            nbytes, _lib.stream_ptr())
    with torch.cuda.device(dev):
        if lm is None:
            _lib.check(lib.sb_ctc_prefix_beam(logp.data_ptr(), lens.data_ptr(), B, T, S,
                                              int(beam_size), int(blank), *outs),
                       "sb_ctc_prefix_beam")
        elif isinstance(lm, WordLM):
            tables, _ = lm.device_tables(dev)
            _lib.check(lib.sb_ctc_prefix_beam_wordlm(logp.data_ptr(), lens.data_ptr(), B, T, S,
                                                     int(beam_size), int(blank), tables,
                                                     float(lm_weight), float(insertion_bonus),
                                                     lm.oov_penalty, *outs),
                       "sb_ctc_prefix_beam_wordlm")
        else:
            tables, _ = lm.device_tables(dev)
            _lib.check(lib.sb_ctc_prefix_beam_lm(logp.data_ptr(), lens.data_ptr(), B, T, S,
                                                 int(beam_size), int(blank), tables,
                                                 float(lm_weight), float(insertion_bonus), *outs),
                       "sb_ctc_prefix_beam_lm")
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
