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
import random

import numpy as np
import torch
import torch.nn as nn

from . import model


class Seq2Seq(model.Model):

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

    def loss(self, batch):
        x, y = self.collate(*batch)
        x, y = self._to_dev(x, y)
        with self._grad_ctx():
            out, _ = self.forward_impl(x, y)
            bsz, _, out_dim = out.shape
            ce = nn.functional.cross_entropy(out.reshape(-1, out_dim), y[:, 1:].reshape(-1),
                                             reduction="sum")
            # (1,)-shaped so that train.py:33 `loss.data[0]` works on current torch
            return (ce / bsz).reshape(1)

    def forward_impl(self, x, y):
        x = self.encode(x)
        return self.decode(x, y)

    def forward(self, batch):
        x, y = self.collate(*batch)
        x, y = self._to_dev(x, y)
        with self._grad_ctx():
            return self.forward_impl(x, y)[0]

    def decode(self, x, y):
        """Teacher-forced decode (:78-112).  x (B, T', H); y (B, U) -> logits (B, U-1, V-1),
        alignments (B, U-1, T').  The scheduled-sampling coin flips are drawn here from Python's
        `random` in the reference's order (:93-94: one draw per step after the first, only while
        sampling is on); the steps themselves run on the device."""
        from ..functions import s2s
        steps = y.shape[1] - 1
        flags = [False] * max(steps, 1)
        if self.scheduled_sampling:
            for t in range(1, steps):
                flags[t] = random.random() < self.sample_prob
        return s2s.decode(self, x, y, flags)

    def decode_step(self, x, y, state=None, softmax=False):
        """One decoder step (:114-137).  y (B, 1) -> (logits (B, V-1), (hx, ax, sx))."""
        from ..functions import s2s
        return s2s.decode_step(self, x, y, state, softmax)

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
        x, y = self.collate(*batch)
        end_tok = int(y[0, -1])
        x, y = self._to_dev(x, y)
        with torch.no_grad():
            x = self.encode(x)
            return s2s.greedy(self, x, y[:, 0], end_tok, max_len)

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

    def forward(self, eh, dhx, ax=None):
        """(sx (B,1,H), ax (B,T)) of one attention step on the fused kernel (csrc/s2s.cu).  The
        module is a parameter container for the decoder: training differentiates the whole
        decode through functions/s2s.py, so this stand-alone call carries no autograd."""
        from .. import ops
        if torch.is_grad_enabled() and (eh.requires_grad or dhx.requires_grad):
            raise RuntimeError("NNAttention.forward is inference-only; gradients flow through "
                               "Seq2Seq.decode (speech_b200.functions.s2s)")
        return ops.attn_step(eh, dhx, ax, self.conv, self.nn[1].fc, self.log_t)
