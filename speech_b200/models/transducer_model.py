"""RNN-Transducer model - host-side mirror of speech/models/transducer_model.py:14-116.

Encoder and prediction network run on the sm_90a GRU kernels (ops.gru_stack); the joint network
(fc1 shared by both streams, transducer_model.py:71-73), the log-softmax and the loss run fused
(csrc/joint.cu + csrc/rnnt.cu): training never materialises the (B,T',U+1,H) hidden tensor nor the
(B,T',U+1,V+1) log-probabilities, only a compact {blank, label} lattice; `forward` / `infer` still
return the reference's full log-probability tensor, written by the same fused kernel.
The fused kernel keeps fc2's weight in shared memory, which holds up to V+1 = 64 classes; larger
vocabularies run the same computation a slab of frames at a time (GEMM logits + row kernels of
csrc/joint_vocab.cu), so only one slab's logits ever exist.  Where the full lattice is too large
for the beam search, `infer` decodes from per-node shortlists that the slab path writes instead.
"""
import torch
import torch.nn as nn

from . import model
from .. import ops
from ..functions import transducer as transducer_fn
from ..transducer_decoders import decode_static_batch, decode_static_fits, decode_static_shortlist


class Transducer(model.Model):

    def __init__(self, freq_dim, vocab_size, config):
        super().__init__(freq_dim, config)
        dec = config["decoder"]
        rnn_dim = self.encoder_dim
        self.embedding = nn.Embedding(vocab_size, dec["embedding_dim"])
        self.dec_rnn = nn.GRU(input_size=dec["embedding_dim"], hidden_size=rnn_dim,
                              num_layers=dec["layers"], batch_first=True,
                              dropout=config["dropout"])
        self.blank = vocab_size                       # blank is the LAST class (:28)
        self.fc1 = model.LinearND(rnn_dim, rnn_dim)
        self.fc2 = model.LinearND(rnn_dim, vocab_size + 1)

    def forward(self, batch):
        x, y, x_lens, y_lens = self.collate(*batch)
        y_mat = self.label_collate(batch[1])
        with self._grad_ctx():
            lens = self.exact_lens(x_lens)
            return self.forward_impl(x, y_mat) if lens is None else \
                self.forward_impl(x, y_mat, lens=lens)

    def forward_impl(self, x, y, lens=None):
        if self.is_cuda:
            x = x.cuda(non_blocking=True)
            y = y.cuda(non_blocking=True)
        return self.decode(self._encode(x, lens), y)

    def loss(self, batch):
        x, y, x_lens, y_lens = self.collate(*batch)
        y_mat = self.label_collate(batch[1])
        with self._grad_ctx():
            if self.is_cuda:
                x = x.cuda(non_blocking=True)
                y_mat = y_mat.cuda(non_blocking=True)
            # in the exact-lengths mode x_lens are the utterances' own frames: the loss gives
            # frames >= x_lens[b] exactly zero gradient (sb_rnnt_fwd_bwd_compact), and so does
            # the encoder
            fx, fy = self.joint_inputs(self._encode(x, self.exact_lens(x_lens)), y_mat)
            fc2 = self.fc2.fc
            H = fc2.in_features
            return transducer_fn.JointTransducerLoss(blank=self.blank)(
                fx, fy, ops.pad_blocks(fc2.weight, 1, 1, H, fx.shape[2]), fc2.bias, y_mat, y,
                x_lens, y_lens)

    def joint_inputs(self, x, y):
        """fc1 of both streams (the SAME fc1, :73): x (B,T',H) encoder states -> fx (B,T',Hj);
        labels y (B,U) -> embedding, zero start vector, prediction GRU -> fy (B,U+1,Hj).
        Hj is H rounded up to the joint kernels' multiple of 8: fc1 gets zero output units, which
        stay 0 through relu(fx + fy), and fc2 zero input columns for them (exact)."""
        emb = self.embedding(y)
        start = torch.zeros((emb.shape[0], 1, emb.shape[2]), device=emb.device, dtype=emb.dtype)
        pred_in = torch.cat([start, emb], dim=1)           # zero vector stands for "no label yet"
        p = self.dec_rnn.dropout if self.training else 0.0
        pred = ops.gru_stack(pred_in, self.dec_rnn, dropout=p)
        fc1 = self.fc1.fc
        H = fc1.out_features
        Hj = (H + 7) // 8 * 8
        if Hj == H:
            return self.fc1(x), self.fc1(pred)
        w1, b1 = ops.pad_blocks(fc1.weight, 0, 1, H, Hj), ops.pad_blocks(fc1.bias, 0, 1, H, Hj)
        return ops.linear(x, w1, b1), ops.linear(pred, w1, b1)

    def decode(self, x, y):
        """x (B, T', H) encoder states, y (B, U) labels -> (B, T', U+1, V+1) log-probs (:54-77),
        written by the fused joint kernel (no autograd through this tensor: `loss` trains through
        the compact lattice instead)."""
        fx, fy = self.joint_inputs(x, y)
        return transducer_fn.joint_log_probs(fx, fy, self.fc2.fc, y, self.blank)

    def collate(self, inputs, labels):
        return self.lattice_batch(inputs, labels)

    def infer(self, batch, beam_size=4):
        """Beam search on the TEACHER-FORCED lattice, as the reference does (:92-101), including
        its use of the un-subsampled input length as the time bound (clamped by slicing); in the
        exact-lengths mode the bound is each utterance's own conv_out_size(T_b) frames.
        Where the full-lattice search does not fit (beam_size * (V+1) * 8 bytes over 200 KB) the
        joint writes per-node shortlists instead of the (B, T', U+1, V+1) tensor, and the search
        runs on those, with the same predictions."""
        if not decode_static_fits(beam_size, self.fc2.fc.out_features):
            return self._infer_shortlists(batch, beam_size)
        with torch.no_grad():
            out = self(batch)                                  # (B, T', U+1, V+1) on the device
        # the reference slices lp[:T, :U] per utterance with the UN-subsampled T (clamped by
        # numpy slicing to T') and U = labels + 1; the search itself runs batched on the GPU
        tlens, ulens = self._search_lens(batch, out.shape[1])
        preds, _ = decode_static_batch(out, tlens, ulens, beam_size, self.blank)
        return preds

    def _search_lens(self, batch, frames):
        if self.exact_lengths:
            tlens = [max(0, self.conv_out_size(i.shape[0], 0)) for i in batch[0]]
        else:
            tlens = [min(i.shape[0], frames) for i in batch[0]]
        return tlens, [len(l) + 1 for l in batch[1]]

    def _infer_shortlists(self, batch, beam_size):
        # the joint inputs exactly as `forward` computes them
        with torch.no_grad():
            x, y, x_lens, y_lens = self.collate(*batch)
            y_mat = self.label_collate(batch[1])
            with self._grad_ctx():
                lens = self.exact_lens(x_lens)
                if self.is_cuda:
                    x = x.cuda(non_blocking=True)
                    y_mat = y_mat.cuda(non_blocking=True)
                fx, fy = self.joint_inputs(self._encode(x, lens), y_mat)
        T, U1 = fx.shape[1], fy.shape[1]
        tlens, ulens = self._search_lens(batch, T)
        tlens = [min(t, T) for t in tlens]
        ulens = [min(u, U1) for u in ulens]
        V1 = self.fc2.fc.out_features

        # a rerun of flagged utterances (rows) recomputes the slab joint of the whole batch and
        # keeps their rows: the joint's GEMM may sum a row differently in a smaller batch, and the
        # rerun's lists must hold the same values as the first pass (and as `forward`) bit for bit
        def produce(kp, rows):
            with torch.no_grad():
                sl = transducer_fn.joint_shortlists(fx, fy, self.fc2.fc, y_mat, self.blank, kp)
            return sl if rows is None else tuple(a[rows].contiguous() for a in sl)
        preds, _ = decode_static_shortlist(produce, tlens, ulens, V1, beam_size, self.blank)
        return preds

    def label_collate(self, labels):
        return torch.from_numpy(model.end_pad_labels(labels))
