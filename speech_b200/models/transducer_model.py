"""RNN-Transducer model - host-side mirror of speech/models/transducer_model.py:14-116.

Encoder and prediction network run on the sm_90a GRU kernels (ops.gru_stack); the joint network
(fc1 shared by both streams, transducer_model.py:71-73), the log-softmax and the loss run fused
(csrc/joint.cu + csrc/rnnt.cu): training never materialises the (B,T',U+1,H) hidden tensor nor the
(B,T',U+1,V+1) log-probabilities, only a compact {blank, label} lattice; `forward` / `infer` still
return the reference's full log-probability tensor, written by the same fused kernel.
"""
import torch
import torch.nn as nn

from . import model
from .. import ops
from ..functions import transducer as transducer_fn
from ..transducer_decoders import decode_static_batch


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
            return self.forward_impl(x, y_mat)

    def forward_impl(self, x, y):
        if self.is_cuda:
            x = x.cuda(non_blocking=True)
            y = y.cuda(non_blocking=True)
        return self.decode(self.encode(x), y)

    def loss(self, batch):
        x, y, x_lens, y_lens = self.collate(*batch)
        y_mat = self.label_collate(batch[1])
        with self._grad_ctx():
            if self.is_cuda:
                x = x.cuda(non_blocking=True)
                y_mat = y_mat.cuda(non_blocking=True)
            fx, fy = self.joint_inputs(self.encode(x), y_mat)
            fc2 = self.fc2.fc
            return transducer_fn.JointTransducerLoss(blank=self.blank)(
                fx, fy, fc2.weight, fc2.bias, y_mat, y, x_lens, y_lens)

    def joint_inputs(self, x, y):
        """fc1 of both streams (the SAME fc1, :73): x (B,T',H) encoder states -> fx (B,T',H);
        labels y (B,U) -> embedding, zero start vector, prediction GRU -> fy (B,U+1,H)."""
        emb = self.embedding(y)
        start = torch.zeros((emb.shape[0], 1, emb.shape[2]), device=emb.device, dtype=emb.dtype)
        pred_in = torch.cat([start, emb], dim=1)           # zero vector stands for "no label yet"
        p = self.dec_rnn.dropout if self.training else 0.0
        pred = ops.gru_stack(pred_in, self.dec_rnn, dropout=p)
        return self.fc1(x), self.fc1(pred)

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
        its use of the un-subsampled input length as the time bound (clamped by slicing)."""
        with torch.no_grad():
            out = self(batch)                                  # (B, T', U+1, V+1) on the device
        # the reference slices lp[:T, :U] per utterance with the UN-subsampled T (clamped by
        # numpy slicing to T') and U = labels + 1; the search itself runs batched on the GPU
        tlens = [min(i.shape[0], out.shape[1]) for i in batch[0]]
        ulens = [len(l) + 1 for l in batch[1]]
        preds, _ = decode_static_batch(out, tlens, ulens, beam_size, self.blank)
        return preds

    def label_collate(self, labels):
        return torch.from_numpy(model.end_pad_labels(labels))
