"""CTC model - host-side mirror of speech/models/ctc_model.py:13-70 (reference)."""
import numpy as np
import torch

from . import model
from .ctc_decoder import check_lm, decode, decode_batch
from ..functions import ctc


class CTC(model.Model):

    def __init__(self, freq_dim, output_dim, config):
        super().__init__(freq_dim, config)
        self.blank = output_dim                      # blank is the LAST class (ctc_model.py:18)
        self.fc = model.LinearND(self.encoder_dim, output_dim + 1)
        self._add_lookahead()

    def _collated(self, batch):
        """reference-style (inputs, labels) pair, or a loader.StagedBatch prepared ahead of time"""
        from ..loader import StagedBatch
        if isinstance(batch, StagedBatch):
            return batch.tensors()
        return self.collate(*batch)

    def _forward_impl(self, x, lens, softmax=False):
        # without lengths, the call the default mode has always made
        if lens is None:
            return self.forward_impl(x, softmax=softmax) if softmax else self.forward_impl(x)
        return self.forward_impl(x, softmax=softmax, lens=lens)

    def forward(self, batch):
        x, y, x_lens, y_lens = self._collated(batch)
        with self._grad_ctx():
            return self._forward_impl(x, self.exact_lens(x_lens))

    def forward_impl(self, x, softmax=False, lens=None):
        if self.is_cuda:
            x = x.cuda(non_blocking=True)
        x = self.encode_logits(x) if lens is None else self.encode_logits(x, lens)
        if softmax:
            return torch.nn.functional.softmax(x, dim=2)
        return x

    def encode_logits(self, x, lens=None):
        """encode + fc with the halves-sum and the projection fused into one contraction on the
        bf16 top-layer output (same math as model.py:75-77 followed by ctc_model.py:29).
        lens (optional): valid frames per utterance (exact-lengths mode, Model.encode)."""
        from .. import _lib, ops
        _lib.require_cuda(x, "forward_impl() input")
        if getattr(self, "parity_mode", False) and not torch.is_grad_enabled():
            if lens is not None:
                raise NotImplementedError("parity_mode does not support exact_lengths")
            if self.lookahead is not None:
                raise NotImplementedError("parity_mode does not support a lookahead layer")
            # reference-precision forward (split-bf16 GEMMs, fp32 recurrence): a measuring stick
            # for the bf16 operand path, see ops.encode_logits_parity
            return ops.encode_logits_parity(x, self.conv, self.rnn, self.fc.fc)
        x = ops.conv_stack(x, self.conv, self.training)
        p = self.rnn.dropout if self.training else 0.0
        return ops.gru_stack_logits(x, self.rnn, self.fc.fc, dropout=p, lens=lens,
                                    lookahead=self.lookahead)

    def loss(self, batch):
        x, y, x_lens, y_lens = self._collated(batch)
        with self._grad_ctx():
            out = self._forward_impl(x, self.exact_lens(x_lens))
            return self.ctc_loss(out, y, x_lens, y_lens)

    def ctc_loss(self, out, y, x_lens, y_lens):
        """warp-ctc call of the reference (ctc_model.py:38-39): raw logits, blank = last class."""
        return ctc.CTCLoss()(out, y, x_lens, y_lens)

    def collate(self, inputs, labels):
        return self.lattice_batch(inputs, labels)

    def infer(self, batch, beam_size=1, lm=None, lm_weight=0.0, insertion_bonus=0.0):
        """Best label sequence of each utterance.  lm: an n-gram LM over this model's classes
        (speech_b200.lm.NGramLM) fused into the beam search with lm_weight and insertion_bonus,
        or a word n-gram LM spelled in them (speech_b200.lm.WordLM), whose lm_weight scales the
        word LM and whose insertion_bonus is per word (ctc_decoder)."""
        check_lm(lm, lm_weight, insertion_bonus, self.blank + 1, self.blank)
        x, y, x_lens, y_lens = self._collated(batch)
        lens = self.exact_lens(x_lens)
        with torch.no_grad():
            probs = self._forward_impl(x, lens, softmax=True)
        return decode_batch(probs, beam_size=beam_size, blank=self.blank, lens=lens, lm=lm,
                            lm_weight=lm_weight, insertion_bonus=insertion_bonus)

    def align(self, batch, return_scores=False):
        """Viterbi (forced) alignment of each transcript to its audio: the single best path through
        the lattice `loss` sums over (functions.ctc.ctc_viterbi).  batch: what `loss` takes; the
        timestamps of a hypothesis come from `align((inputs, hypotheses))`.  Frames searched: the
        padded T', or each utterance's own conv_out_size(T_b) in the exact-lengths mode.
        Returns, per utterance, a list of (first_frame, last_frame) encoder-frame pairs, one per
        label, or None where no alignment exists (too few frames for the labels and their adjacent
        repeats); with return_scores also the paths' float64 log-probabilities (-inf for None).
        Encoder frame t starts at input frame t * prod(conv strides) (10 ms per input frame with
        the reference featuriser)."""
        x, y, x_lens, y_lens = self._collated(batch)
        with torch.no_grad():
            out = self._forward_impl(x, self.exact_lens(x_lens))
        path, scores = ctc.ctc_viterbi(out, y, x_lens, y_lens, blank=self.blank)
        path, scores = path.cpu().numpy(), scores.cpu().numpy()
        spans = []
        for b, n in enumerate(y_lens.tolist()):
            if scores[b] == -np.inf:
                spans.append(None)
                continue
            # a path visits labels 0..n-1 in order, each on at least one frame
            t = np.flatnonzero(path[b] >= 0)
            j, k = path[b][t], np.arange(n)
            first = t[np.searchsorted(j, k, "left")]
            last = t[np.searchsorted(j, k, "right") - 1]
            spans.append(list(zip(first.tolist(), last.tolist())))
        return (spans, scores) if return_scores else spans

    def stream(self, num_streams, beam_size=1, max_frames=3000, lm=None, lm_weight=0.0,
               insertion_bonus=0.0):
        """Streaming recognition of num_streams (<= 128) utterances at once with a unidirectional
        encoder: a speech_b200.streaming.CTCStream, whose push(chunks) feeds feature frames as
        they arrive and partial() returns each stream's best labels so far; the final partial()
        equals infer's search over the whole utterances (see that module).  max_frames caps the
        encoder frames per stream between resets; lm, lm_weight, insertion_bonus: as infer."""
        from ..streaming import CTCStream
        return CTCStream(self, num_streams, beam_size, max_frames, lm, lm_weight, insertion_bonus)

    @staticmethod
    def max_decode(pred, blank):
        """Greedy collapse: merge repeats, then drop blanks (reference ctc_model.py:62-70)."""
        seq = []
        prev = None
        for p in pred:
            if p != blank and p != prev:
                seq.append(p)
            prev = p
        return seq
