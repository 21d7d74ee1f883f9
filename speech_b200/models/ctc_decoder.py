"""CTC prefix beam search - drop-in for speech/models/ctc_decoder.py:38-113 (reference).

`decode(probs, beam_size=10, blank=0)` keeps the reference's signature and return value
((label tuple, negative log-likelihood)); the search itself runs in the sm_90a kernel
sb_ctc_prefix_beam (csrc/decode.cu), one CTA per utterance.  `decode_batch` is the batched
entry CTC.infer uses (the reference loops over utterances in Python, ctc_model.py:59-60).
"""
import numpy as np
import torch

from .. import _lib


def _run(logp, lens, beam_size, blank):
    lib = _lib.load()
    B, T, S = logp.shape
    dev = logp.device
    nbytes = _lib.workspace_size(lib.sb_ctc_prefix_beam_workspace_size, B, T, beam_size)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    out_labels = torch.empty(B, T, dtype=torch.int32, device=dev)
    out_lens = torch.empty(B, dtype=torch.int32, device=dev)
    out_scores = torch.empty(B, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _lib.check(lib.sb_ctc_prefix_beam(logp.data_ptr(), lens.data_ptr(), B, T, S,
                                          int(beam_size), int(blank), out_labels.data_ptr(),
                                          out_lens.data_ptr(), out_scores.data_ptr(),
                                          ws.data_ptr(), nbytes, _lib.stream_ptr()),
                   "sb_ctc_prefix_beam")
    labels = out_labels.cpu().numpy()
    n = out_lens.cpu().numpy()
    scores = out_scores.cpu().numpy()
    return [(tuple(int(v) for v in labels[b, :n[b]]), float(scores[b])) for b in range(B)]


def decode_batch(probs, beam_size=10, blank=0, lens=None, with_scores=False):
    """probs (B, T, S) post-softmax CUDA tensor -> list of label tuples (one per utterance)."""
    _lib.require_cuda(probs, "probs")
    logp = torch.log(probs.detach().float()).contiguous()
    B, T, S = logp.shape
    if lens is None:
        lens = torch.full((B,), T, dtype=torch.int32, device=probs.device)
    else:
        lens = torch.as_tensor(lens, dtype=torch.int32).to(probs.device)
    res = _run(logp, lens, beam_size, blank)
    return res if with_scores else [r[0] for r in res]


def decode(probs, beam_size=10, blank=0):
    """Reference signature: probs (T, S) array of post-softmax probabilities (host).

    Returns (label tuple, negative log-likelihood).  The log is taken on the host in the input
    dtype exactly as the reference does (np.log, ctc_decoder.py:52); the beam search runs on
    cuda:current.
    """
    if not torch.cuda.is_available():
        raise _lib.SpeechB200Error("speech_b200: decode() needs a CUDA device (no CPU path)")
    with np.errstate(divide="ignore"):
        logp = np.log(np.asarray(probs))
    lp = torch.from_numpy(np.ascontiguousarray(logp, dtype=np.float32))[None].cuda()
    lens = torch.full((1,), lp.shape[1], dtype=torch.int32, device=lp.device)
    return _run(lp, lens, beam_size, blank)[0]
