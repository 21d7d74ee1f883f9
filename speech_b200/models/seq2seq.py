"""Attention sequence-to-sequence model - host-side mirror of speech/models/seq2seq.py:14-248
(Seq2Seq) and :331-360 (NNAttention, the only attention module the reference instantiates).

The encoder runs on the sm_90a kernels (ops.conv_stack / ops.gru_stack).  The per-token decoder
(embedding + GRUCell + NNAttention + fc, seq2seq.py:92-108,114-137) keeps the reference's module
structure and state_dict names (the nn modules are parameter containers); its arithmetic is two
kernels per token, forward and backward (functions/s2s.py -> csrc/s2s.cu), and both the greedy
loop and the beam search run device-resident: one device->host copy per decode.
Reference quirks kept on purpose: end-padding is part of the loss (:58-63), `hx` starts at zero,
scheduled sampling draws from Python's `random` (:94), `beam_search` handles one utterance (:197)
and needs the py3 fix list(filter(...)) (:211) - applied here.
"""
import math
import random

import numpy as np
import torch
import torch.nn as nn

from . import model
from ..lm import WordLM


class Seq2Seq(model.Model):

    # Hybrid CTC/attention (config["decoder"]["ctc_weight"], default 0): a CTC head `ctc_fc` on
    # the encoder, trained jointly and used by recognize(ctc_weight=...).  A class attribute, so
    # that pickles written before the key existed read it as 0 (no head).
    ctc_weight = 0.0

    def __init__(self, freq_dim, vocab_size, config):
        super().__init__(freq_dim, config)
        dec = config["decoder"]
        rnn_dim = self.encoder_dim
        self.embedding = nn.Embedding(vocab_size, dec["embedding_dim"])
        self.dec_rnn = nn.GRUCell(input_size=dec["embedding_dim"], hidden_size=rnn_dim)
        self.attend = NNAttention(rnn_dim, log_t=dec.get("log_t", False))
        self.sample_prob = dec.get("sample_prob", 0)
        self.scheduled_sampling = (self.sample_prob != 0)
        # the start-of-sequence token is never predicted: vocab_size - 1 classes (:32-34)
        self.fc = model.LinearND(rnn_dim, vocab_size - 1)
        w = dec.get("ctc_weight", 0)
        if isinstance(w, bool) or not isinstance(w, (int, float)) or not 0.0 <= w < 1.0:
            raise ValueError("decoder ctc_weight must be a number in [0, 1), got %r" % (w,))
        if w > 0:
            # created after every reference module, so that they keep their initial values under
            # a seed; classes 0..V-3 are the labels, V-2 the blank (END and START never occur)
            self.ctc_weight = float(w)
            self.ctc_fc = model.LinearND(rnn_dim, vocab_size - 1)
        self._add_lookahead()

    def set_eval(self):
        self.eval()
        self.volatile = True
        self.scheduled_sampling = False

    def set_train(self):
        self.train()
        self.volatile = False
        self.scheduled_sampling = (self.sample_prob != 0)

    def _to_dev(self, x, y):
        if self.is_cuda:
            x = x.cuda(non_blocking=True)
            y = y.cuda(non_blocking=True)
        return x, y

    def input_lens(self, inputs):
        """Exact-lengths mode: encoder frames conv_out_size(T_b) of every utterance, which the
        encoder and the attention then keep to; None in the default (padded) mode."""
        if not self.exact_lengths:
            return None
        return [max(0, self.conv_out_size(i.shape[0], 0)) for i in inputs]

    def loss(self, batch):
        if self.ctc_weight > 0:
            return self._joint_loss(batch)
        lens = self.input_lens(batch[0])
        x, y = self.collate(*batch)
        x, y = self._to_dev(x, y)
        with self._grad_ctx():
            out, _ = self.forward_impl(x, y) if lens is None else self.forward_impl(x, y, lens)
            bsz, _, out_dim = out.shape
            ce = nn.functional.cross_entropy(out.reshape(-1, out_dim), y[:, 1:].reshape(-1),
                                             reduction="sum")
            # (1,)-shaped so that train.py:33 `loss.data[0]` works on current torch
            return (ce / bsz).reshape(1)

    def _ctc_targets(self, labels):
        """flat int32 CTC targets (each transcript without its START and END) and their lengths;
        ValueError unless every transcript is [START, labels in 0..V-3, END]"""
        V = self.embedding.num_embeddings
        flat, lengths = [], []
        for seq in labels:
            seq = [int(t) for t in seq]
            if len(seq) < 2 or seq[0] != V - 1 or seq[-1] != V - 2 or \
                    any(not 0 <= t < V - 2 for t in seq[1:-1]):
                raise ValueError("with a CTC head every transcript must be [START (%d), labels in "
                                 "0..%d, END (%d)], got %r" % (V - 1, V - 3, V - 2, seq))
            flat += seq[1:-1]
            lengths.append(len(seq) - 2)
        return torch.tensor(flat, dtype=torch.int32), torch.tensor(lengths, dtype=torch.int32)

    def _joint_loss(self, batch):
        """((1 - w) CE_sum + w CTC_sum) / B, w = ctc_weight: the encoder states feed both the
        attention decoder and the CTC head (functions.ctc.CTCLoss, a sum, blank V-2), over the
        padded T' frames or each utterance's own conv_out_size(T_b) in the exact-lengths mode"""
        from ..functions import ctc
        targets, target_lens = self._ctc_targets(batch[1])
        lens = self.input_lens(batch[0])
        x, y = self.collate(*batch)
        x, y = self._to_dev(x, y)
        with self._grad_ctx():
            enc = self._encode(x, lens)
            out, _ = self.decode(enc, y) if lens is None else self.decode(enc, y, lens)
            bsz, _, out_dim = out.shape
            ce = nn.functional.cross_entropy(out.reshape(-1, out_dim), y[:, 1:].reshape(-1),
                                             reduction="sum")
            logits = self.ctc_fc(enc)
            frames = lens if lens is not None else [logits.shape[1]] * bsz
            ctc_sum = ctc.CTCLoss()(logits, targets, torch.tensor(frames, dtype=torch.int32),
                                    target_lens)
            w = self.ctc_weight
            return (((1.0 - w) * ce + w * ctc_sum.reshape(())) / bsz).reshape(1)

    def forward_impl(self, x, y, lens=None):
        x = self._encode(x, lens)
        return self.decode(x, y) if lens is None else self.decode(x, y, lens)

    def forward(self, batch):
        lens = self.input_lens(batch[0])
        x, y = self.collate(*batch)
        x, y = self._to_dev(x, y)
        with self._grad_ctx():
            return (self.forward_impl(x, y) if lens is None else self.forward_impl(x, y, lens))[0]

    def decode(self, x, y, lens=None):
        """Teacher-forced decode (:78-112).  x (B, T', H); y (B, U) -> logits (B, U-1, V-1),
        alignments (B, U-1, T').  The scheduled-sampling coin flips are drawn here from Python's
        `random` in the reference's order (:93-94: one draw per step after the first, only while
        sampling is on); the steps themselves run on the device.  lens (optional): frames each
        utterance attends over."""
        from ..functions import s2s
        steps = y.shape[1] - 1
        flags = [False] * max(steps, 1)
        if self.scheduled_sampling:
            for t in range(1, steps):
                flags[t] = random.random() < self.sample_prob
        return s2s.decode(self, x, y, flags, lens)

    def decode_step(self, x, y, state=None, softmax=False, lens=None):
        """One decoder step (:114-137).  y (B, 1) -> (logits (B, V-1), (hx, ax, sx))."""
        from ..functions import s2s
        return s2s.decode_step(self, x, y, state, softmax, lens)

    def predict(self, batch):
        probs = self(batch)
        return [seq.tolist() for seq in torch.max(probs, dim=2)[1].cpu().numpy()]

    def infer_decode(self, x, y, end_tok, max_len):
        """(:145-160) kept for API parity: per-step logits and the arg-max tokens."""
        probs, argmaxs, state = [], [y], None
        for _ in range(max_len):
            out, state = self.decode_step(x, y, state=state)
            probs.append(out)
            y = torch.max(out, dim=1)[1].unsqueeze(dim=1)
            argmaxs.append(y)
            if bool((y == end_tok).all()):
                break
        return torch.cat(probs), torch.cat(argmaxs, dim=1)

    def infer(self, batch, max_len=200):
        """Greedy decode (:162-178): the start token, then arg-max until every row emitted end in
        the same step; device-resident (functions/s2s.py: greedy)."""
        from ..functions import s2s
        lens = self.input_lens(batch[0])
        x, y = self.collate(*batch)
        end_tok = int(y[0, -1])
        x, y = self._to_dev(x, y)
        with torch.no_grad():
            x = self._encode(x, lens)
            return s2s.greedy(self, x, y[:, 0], end_tok, max_len, lens)

    def beam_search(self, batch, beam_size=10, max_len=200):
        """Beam search for ONE utterance (:180-227).  Hypothesis scores are sums of log-softmax
        (float64); pruning is the reference's stable descending sort, i.e. ties keep (beam index,
        then vocabulary index) order; device-resident (functions/s2s.py: beam_search)."""
        from ..functions import s2s
        x, y = self.collate(*batch)
        start_tok, end_tok = int(y[0, 0]), int(y[0, -1])
        x, y = self._to_dev(x, y)
        with torch.no_grad():
            x = self.encode(x)
            return [s2s.beam_search(self, x, start_tok, end_tok, beam_size, max_len)]

    def recognize(self, inputs, beam_size=10, max_len=200, start_tok=None, end_tok=None,
                  return_scores=False, lm=None, lm_weight=0.0, insertion_bonus=0.0,
                  ctc_weight=0.0, ctc_prebeam=None):
        """Beam search of every utterance of a batch at once, from the audio alone.  inputs: the
        (T_i, F) arrays of batch[0].  Each utterance gets `beam_search`'s search on its own (float64
        scores, stable-descending tie order, the same completion and stop rules), bit for bit, and
        one stopping never changes another's search.  start_tok / end_tok default to the
        Preprocessor's convention: START = vocab_size - 1, END = vocab_size - 2.  Frames attended:
        the padded T' for every utterance, or its own conv_out_size(T_b) in the exact-lengths mode.
        Returns B token lists (START first; END last where a hypothesis completed, else the best
        live one), and their float64 scores with return_scores.  Device-resident
        (functions/s2s.py: beam_search_batch).

        Shallow fusion: lm, a speech_b200.lm.NGramLM over the vocabulary with blank = start_tok and
        end = end_tok (NGramLM.from_arpa(path, preproc.int_to_char, blank=V - 1, end=V - 2)).
        Candidate c of a hypothesis h then scores logp(c) + (lm_weight * lm(c | h) +
        insertion_bonus), where lm(end_tok | h) is lm(</s> | h) and the end token earns no bonus;
        the context of h starts at <s>, its start token.  The returned scores are the fused ones.
        With lm=None (the default) this is the LM-less search.
        lm may also be a speech_b200.lm.WordLM with the same layout (WordLM.from_arpa(path,
        preproc.int_to_char, blank=V - 1, end=V - 2), the space its delimiter): a word is then
        scored when the delimiter that ends it is chosen, lm_weight * lm(w | words) +
        insertion_bonus (per word), and END adds the trailing word and lm(</s> | words); a class
        that takes the partial word out of the lexicon adds lm.oov_penalty (include/speech_b200.h,
        sb_s2s_beam_select_wordlm_batch).  The score of a completed hypothesis is acoustic +
        lm_weight * (word LM with </s>) + insertion_bonus * words + oov_penalty * OOV words.

        Joint CTC/attention decoding (Watanabe et al. 2017, Algorithm 2): ctc_weight = w in
        (0, 1) needs the CTC head (config["decoder"]["ctc_weight"] > 0) and the default START /
        END.  Each live hypothesis h extends only by the ctc_prebeam classes c (default
        min(V-1, 3 * beam_size // 2), at most 128) with the largest P = (1 - w) logp(c) (+ the LM
        part above), and scores A_h + P + w * psi(h + c), psi the CTC prefix log-probability of
        h + c over the head's log-softmax (the full CTC probability of h for END), A the attention
        and LM part.  The returned scores are then A + w * psi.  With ctc_weight = 0 (the default)
        this is the search above, untouched."""
        from ..functions import s2s
        V = self.embedding.num_embeddings
        start_tok = V - 1 if start_tok is None else int(start_tok)
        end_tok = V - 2 if end_tok is None else int(end_tok)
        if not 1 <= int(beam_size) <= s2s.BEAM_MAX_WIDTH:
            raise ValueError("beam_size must lie in [1, %d], got %r"
                             % (s2s.BEAM_MAX_WIDTH, beam_size))
        if int(max_len) < 1:
            raise ValueError("max_len must be >= 1, got %r" % (max_len,))
        if not 0 <= start_tok < V:
            raise ValueError("start_tok %d is not a token of the vocabulary (%d)" % (start_tok, V))
        if not 0 <= end_tok < V - 1:
            raise ValueError("end_tok %d is not a class the model predicts (%d)" % (end_tok, V - 1))
        if len(inputs) == 0:
            raise ValueError("recognize needs at least one utterance")
        self._check_lm(lm, lm_weight, insertion_bonus, V, start_tok, end_tok)
        M = self._check_ctc(ctc_weight, ctc_prebeam, int(beam_size), V, start_tok, end_tok)
        lens = self.input_lens(inputs)
        x = self.stage_inputs(inputs)
        with torch.no_grad():
            x = self._encode(x, lens)
            ctc = None
            if ctc_weight > 0:
                y = torch.log_softmax(self.ctc_fc(x).float(), dim=-1).contiguous()
                ctc = (y, float(ctc_weight), M)
            res = s2s.beam_search_batch(self, x, start_tok, end_tok, int(beam_size), int(max_len),
                                        lens, lm, lm_weight, insertion_bonus, ctc)
        labels = [list(r[0]) for r in res]
        return (labels, [r[1] for r in res]) if return_scores else labels

    def recognize_two_pass(self, inputs, beam_size=10, ctc_weight=0.5, return_scores=False):
        """Two-pass decoding (attention rescoring, Zhang et al. 2020, arXiv:2012.05481) of every
        utterance of a batch: the CTC head's prefix beam search (beam_size, no LM) gives each
        utterance an N-best of n_b <= beam_size entries y_i with log-probabilities c_i; the
        attention decoder then scores each one teacher-forced, a_i = sum of the float32
        log-softmax values of y_i's labels and END after START, summed in float64 in order.  The
        result is the entry with the largest r_i = (1 - w) a_i + w c_i (float64, w = ctc_weight
        in [0, 1]; ties to the lower beam index) as [START] + y + [END], and r with
        return_scores.  w = 1 gives the first pass's best, w = 0 the N-best entry the attention
        prefers.  Needs the CTC head (config["decoder"]["ctc_weight"] > 0).  Frames: the padded
        T' for every utterance, or its own conv_out_size(T_b) in the exact-lengths mode."""
        from ..functions import s2s
        self._check_two_pass(beam_size, ctc_weight)
        if len(inputs) == 0:
            raise ValueError("recognize_two_pass needs at least one utterance")
        lens = self.input_lens(inputs)
        x = self.stage_inputs(inputs)
        with torch.no_grad():
            x = self._encode(x, lens)
            y = torch.log_softmax(self.ctc_fc(x).float(), dim=-1).contiguous()
            return s2s.recognize_two_pass(self, x, y, lens, int(beam_size), float(ctc_weight),
                                          return_scores)

    def stream(self, num_streams, beam_size=10, max_frames=3000, ctc_weight=0.5):
        """Two-pass recognition as the audio arrives (speech_b200.streaming.Seq2SeqStream): the CTC
        head's prefix beam search advances with every push (partial()), and rescored() runs the
        attention over each stream's N-best as recognize_two_pass does.  Needs a unidirectional
        encoder and the CTC head."""
        from ..streaming import Seq2SeqStream
        return Seq2SeqStream(self, num_streams, beam_size, max_frames, ctc_weight)

    def _check_two_pass(self, beam_size, ctc_weight):
        """ValueError unless two-pass decoding can run with these arguments"""
        from ..functions import s2s
        if self.ctc_weight <= 0:
            raise ValueError("two-pass decoding needs a CTC head (config decoder ctc_weight > 0)")
        if isinstance(beam_size, bool) or int(beam_size) != beam_size or \
                not 1 <= int(beam_size) <= s2s.BEAM_MAX_WIDTH:
            raise ValueError("beam_size must lie in [1, %d], got %r"
                             % (s2s.BEAM_MAX_WIDTH, beam_size))
        if isinstance(ctc_weight, bool) or not isinstance(ctc_weight, (int, float)) or \
                not 0.0 <= ctc_weight <= 1.0:
            raise ValueError("ctc_weight must be a number in [0, 1], got %r" % (ctc_weight,))

    def _check_ctc(self, ctc_weight, ctc_prebeam, beam_size, V, start_tok, end_tok):
        """ValueError unless the joint-decoding arguments of recognize are usable; -> the
        pre-beam width M"""
        C = V - 1
        if isinstance(ctc_weight, bool) or not isinstance(ctc_weight, (int, float)) or \
                not 0.0 <= ctc_weight < 1.0:
            raise ValueError("ctc_weight must be a number in [0, 1), got %r" % (ctc_weight,))
        M = min(C, (3 * beam_size) // 2) if ctc_prebeam is None else ctc_prebeam
        if isinstance(M, bool) or int(M) != M or not 1 <= M <= min(C, 128):
            raise ValueError("ctc_prebeam must lie in [1, %d], got %r" % (min(C, 128), M))
        if ctc_weight > 0:
            if self.ctc_weight <= 0:
                raise ValueError("ctc_weight > 0 needs a CTC head (config decoder ctc_weight > 0)")
            if start_tok != V - 1 or end_tok != V - 2:
                raise ValueError("joint CTC decoding needs START = %d and END = %d, got %d / %d"
                                 % (V - 1, V - 2, start_tok, end_tok))
        return int(M)

    @staticmethod
    def _check_lm(lm, lm_weight, insertion_bonus, V, start_tok, end_tok):
        """ValueError unless the fusion arguments of recognize are usable"""
        if lm is None:
            if lm_weight != 0.0 or insertion_bonus != 0.0:
                raise ValueError("lm_weight / insertion_bonus need an lm")
            return
        if not (math.isfinite(lm_weight) and lm_weight >= 0.0):
            raise ValueError("lm_weight must be finite and >= 0, got %r" % (lm_weight,))
        if not math.isfinite(insertion_bonus):
            raise ValueError("insertion_bonus must be finite, got %r" % (insertion_bonus,))
        if lm.num_classes != V:
            raise ValueError("the LM covers %d classes, the vocabulary has %d" % (lm.num_classes, V))
        if lm.blank != start_tok:
            raise ValueError("the LM's blank is class %d, the start token is %d"
                             % (lm.blank, start_tok))
        if lm.end != end_tok:
            raise ValueError("the LM's end class is %r, the end token is %d" % (lm.end, end_tok))
        if isinstance(lm, WordLM) and lm.delimiter in (start_tok, end_tok):
            raise ValueError("the word LM's delimiter %d is the start or the end token"
                             % lm.delimiter)
        if start_tok < V - 1:
            raise ValueError("with an LM the start token must be the class the model never "
                             "predicts (%d), got %d" % (V - 1, start_tok))

    def collate(self, inputs, labels):
        return self.stage_inputs(inputs), torch.from_numpy(end_pad_concat(labels))


end_pad_concat = model.end_pad_labels      # the reference's module-level name (seq2seq.py:239)


class NNAttention(nn.Module):
    """Additive attention with a location feature (seq2seq.py:331-360): score_t =
    w . relu(eh_t + dhx + conv1d(prev alignment)_t) + b, optional log(T) sharpening, softmax over
    time, context = sum_t a_t eh_t."""

    def __init__(self, n_channels, kernel_size=15, log_t=False):
        super().__init__()
        assert kernel_size % 2 == 1, "Kernel size should be odd for 'same' conv."
        self.conv = nn.Conv1d(1, n_channels, kernel_size, padding=(kernel_size - 1) // 2)
        self.nn = nn.Sequential(nn.ReLU(), model.LinearND(n_channels, 1))
        self.log_t = log_t

    def forward(self, eh, dhx, ax=None, lens=None):
        """(sx (B,1,H), ax (B,T)) of one attention step on the fused kernel (csrc/s2s.cu).  The
        module is a parameter container for the decoder: training differentiates the whole
        decode through functions/s2s.py, so this stand-alone call carries no autograd."""
        from ..functions import s2s
        if torch.is_grad_enabled() and (eh.requires_grad or dhx.requires_grad):
            raise RuntimeError("NNAttention.forward is inference-only; gradients flow through "
                               "Seq2Seq.decode (speech_b200.functions.s2s)")
        return s2s.attn_step(self, eh, dhx, ax, lens)
