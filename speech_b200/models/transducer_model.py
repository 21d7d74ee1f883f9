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
import numpy as np
import torch
import torch.nn as nn

from . import model
from .. import ops
from ..functions import transducer as transducer_fn
from .. import _lib
from .ctc_decoder import check_lm
from ..transducer_decoders import (decode_static_batch, decode_static_fits, decode_static_shortlist,
                                   search_batch)


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
        self._add_lookahead()

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

    def recognize(self, inputs, beam_size=4, max_symbols_per_frame=4, max_len=None,
                  return_scores=False, lm=None, lm_weight=0.0, insertion_bonus=0.0):
        """Beam search from the audio alone: `infer`'s search with the row of each hypothesis
        computed by the prediction network reading the hypothesis's own labels (dropout off),
        instead of the reference transcript.  inputs: the (T_i, F) arrays of batch[0].  A frame
        emits at most max_symbols_per_frame labels; a hypothesis with max_len labels (default: no
        cap beyond frames * max_symbols_per_frame) is not extended.  Frames searched: the padded T'
        for every utterance, or its own conv_out_size(T_b) in the exact-lengths mode.
        lm (optional): a speech_b200.lm.NGramLM over the model's V+1 classes (labels 0..V-1, the
        blank V, no end class), fused into every label extension as lp + (lm_weight * lm(k | h) +
        insertion_bonus), h the hypothesis's last order-1 labels after <s>; blank emissions keep
        their log-probability.  Bad fusion arguments raise ValueError before any launch.
        Returns the label lists (and their float64 scores with return_scores: log-probabilities,
        or with an LM the fused scores)."""
        check_lm(lm, lm_weight, insertion_bonus, self.fc2.fc.out_features, self.blank,
                 search="Transducer")
        rows = PredictionRows(self, inputs)
        labels, scores = search_batch(rows, rows.tlens, beam_size, self.blank,
                                      max_symbols_per_frame, max_len, lm, lm_weight,
                                      insertion_bonus)
        return (labels, scores) if return_scores else labels

    def stream(self, num_streams, beam_size=4, max_symbols_per_frame=4, max_frames=3000,
               max_len=None, lm=None, lm_weight=0.0, insertion_bonus=0.0):
        """Streaming recognition of num_streams utterances with a unidirectional encoder:
        `recognize`'s search resumed chunk by chunk (speech_b200.streaming.TransducerStream)."""
        from ..streaming import TransducerStream
        return TransducerStream(self, num_streams, beam_size, max_symbols_per_frame, max_frames,
                                max_len, lm, lm_weight, insertion_bonus)

    def align(self, batch, return_scores=False):
        """Viterbi (forced) alignment of each transcript to its audio: the single best path through
        the compact lattice `loss` sums over (functions.transducer.rnnt_viterbi).
        batch: what `loss` takes; the timestamps of a hypothesis come from
        `align((inputs, model.recognize(inputs)))`.  Frames searched: the padded T', or each
        utterance's own conv_out_size(T_b) in the exact-lengths mode.  Returns, per utterance, the
        encoder frame at which each label is emitted, or None where no alignment exists (no
        frames); with return_scores also the paths' float64 log-probabilities (-inf for None).
        Encoder frame t starts at input frame t * prod(conv strides) (10 ms per input frame with
        the reference featuriser)."""
        inputs, labels = batch
        x, y, x_lens, y_lens = self.collate(inputs, labels)
        # any filler past a row's own labels: fy at u <= U_b reads labels < u only
        y_mat = self.label_collate([list(seq) or [0] for seq in labels])
        with torch.no_grad():
            if self.is_cuda:
                x = x.cuda(non_blocking=True)
                y_mat = y_mat.cuda(non_blocking=True)
            fx, fy = self.joint_inputs(self._encode(x, self.exact_lens(x_lens)), y_mat)
            frames, scores = transducer_fn.rnnt_viterbi(fx, fy, self.fc2.fc, y_mat, y, x_lens,
                                                        y_lens, self.blank)
        frames, scores = frames.cpu().numpy(), scores.cpu().numpy()
        out = [None if scores[b] == -np.inf else frames[b, :n].tolist()
               for b, n in enumerate(y_lens.tolist())]
        return (out, scores) if return_scores else out

    def label_collate(self, labels):
        return torch.from_numpy(model.end_pad_labels(labels))


def fc1_operands(model):
    """joint_inputs' fc1 weight and bias padded to Hj outputs: (w1 (Hj, H) f32, b1 (Hj) f32)"""
    fc1 = model.fc1.fc
    H = fc1.out_features
    Hj = (H + 7) // 8 * 8
    w1 = ops.pad_blocks(fc1.weight.detach(), 0, 1, H, Hj)
    b1 = ops.pad_blocks(fc1.bias.detach(), 0, 1, H, Hj).float().contiguous()
    return w1, b1


class PredictionNet:
    """The prediction and joint networks of a Transducer as a row provider of B utterances
    (transducer_decoders.search_batch / StreamSearch): per level one sb_rnnt_pred_step per
    prediction-network layer and fc1 of the new states (the wgmma GEMM, bf16 operands: the
    arithmetic of ops.linear with joint_inputs' padded weights) into an arena of per-slot states,
    and the joint rows at frame t with `forward`'s kernels (fused at T = 1, U1 = K where fc2 is
    resident, else one slab of the large-vocabulary joint).  The encoder's fc1 rows are the
    caller's: fxT, time-major, frame t a (>= B, Hj) float32 block whose first B rows are read."""

    def __init__(self, model, B, device, w1=None, b1=None):
        if w1 is None:
            w1, b1 = fc1_operands(model)
        H = model.fc1.fc.out_features
        Hj = (H + 7) // 8 * 8
        self.model = model
        self.B = B
        self.device = device
        self.fxT = None
        self.H, self.Hj, self.Hp = H, Hj, (H + 7) // 8 * 8
        self.w1 = torch.nn.functional.pad(w1.to(torch.bfloat16), (0, self.Hp - H)).contiguous()
        self.b1 = b1
        fc2 = model.fc2.fc
        self.V1 = fc2.out_features
        self.w2 = ops.pad_blocks(fc2.weight.detach().to(torch.bfloat16), 1, 1, H, Hj).contiguous()
        self.b2 = fc2.bias.detach().float().contiguous()
        self.slabs = transducer_fn.joint_uses_slabs(Hj, self.V1)
        rnn = model.dec_rnn
        self.layers = rnn.num_layers
        self.emb = model.embedding.weight.detach().float().contiguous()
        self.gru = [tuple(getattr(rnn, "%s_l%d" % (n, l)).detach().float().contiguous()
                          for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))
                    for l in range(self.layers)]

    def begin(self, slots):
        B, K, S, dev = self.B, slots.K, slots.S, self.device
        R = B * K
        self.K = K
        self.hid = torch.zeros(S + 2, self.layers, R, self.H, dtype=torch.float32, device=dev)
        self.fy = torch.zeros(S + 2, R, self.Hj, dtype=torch.float32, device=dev)
        self.ybf = torch.zeros(R, self.Hp, dtype=torch.bfloat16, device=dev)
        self.ym = torch.zeros(R + 1, dtype=torch.int32, device=dev)
        self.lat = torch.empty(R, 2, dtype=torch.float32, device=dev)
        if self.slabs:
            self.ld = (self.V1 + 7) // 8 * 8
            self.z = torch.empty(R, self.Hj, dtype=torch.bfloat16, device=dev)
            self.logits = torch.empty(R, self.ld, dtype=torch.float32, device=dev)
            self.lse = torch.empty(R, dtype=torch.float32, device=dev)
        self._step(None, 0, None, None)                  # the empty hypothesis, into block 0

    def _step(self, src, dst, par, sym):
        """states of block dst's rows: GRU layers from block src's states at slots par, inputs
        emb[sym] (None: the zero start vector / zero state), then fc1"""
        lib = _lib.load()
        R, H = self.B * self.K, self.H
        sp = _lib.stream_ptr()
        E = self.emb.shape[1]
        for l, (w_ih, w_hh, b_ih, b_hh) in enumerate(self.gru):
            x = None if l == 0 else self.hid[dst, l - 1]
            h_prev = None if src is None else self.hid[src, l]
            y = self.ybf if l == self.layers - 1 else None
            ops._launch("rnnt_pred_step", 6.0 * R * H * (H + (E if l == 0 else H)),
                        lambda: lib.sb_rnnt_pred_step(
                            self.emb.data_ptr() if l == 0 else None,
                            _lib.ptr(sym) if l == 0 else None, _lib.ptr(x), _lib.ptr(h_prev),
                            _lib.ptr(par), w_ih.data_ptr(), w_hh.data_ptr(), b_ih.data_ptr(),
                            b_hh.data_ptr(), self.hid[dst, l].data_ptr(), _lib.ptr(y), self.Hp,
                            R, self.K, E if l == 0 else H, H, sp))
        ops.gemm_bf16_tn(self.ybf, self.w1, out=self.fy[dst], bias=self.b1)

    def extend(self, src, dst, slots):
        self._step(src, dst, slots.par, slots.sym)

    def rows(self, t, block, slots):
        lib = _lib.load()
        B, K, Hj, V1 = self.B, self.K, self.Hj, self.V1
        blank = self.model.blank
        fx, fy = self.fxT[t], self.fy[block]
        sp = _lib.stream_ptr()
        if not self.slabs:
            ops._launch("rnnt_joint", 2.0 * B * K * Hj * V1,
                        lambda: lib.sb_rnnt_joint_fwd(fx.data_ptr(), fy.data_ptr(),
                                                      self.w2.data_ptr(), self.b2.data_ptr(),
                                                      self.ym.data_ptr(), self.lat.data_ptr(),
                                                      slots.lp.data_ptr(), B, 1, K, Hj, V1,
                                                      blank, sp))
            return
        ops._launch("rnnt_joint_slab", 0.0,
                    lambda: lib.sb_rnnt_joint_build_slab(fx.data_ptr(), fy.data_ptr(),
                                                         self.z.data_ptr(), B, 1, K, Hj, 0, 1, sp))
        ops.gemm_bf16_tn(self.z, self.w2, out=self.logits, bias=self.b2)
        ops._launch("rnnt_joint_rows", 0.0,
                    lambda: lib.sb_rnnt_joint_vocab_fwd_rows(
                        self.logits.data_ptr(), self.ld, self.ym.data_ptr(), self.lat.data_ptr(),
                        self.lse.data_ptr(), _lib.ptr(slots.lp), B, 1, K, V1, blank, 0, 1, sp))
        if slots.sl is not None:
            val, idx, meta = slots.sl
            ops._launch("rnnt_shortlist_rows", 0.0,
                        lambda: lib.sb_rnnt_shortlist_rows(
                            self.logits.data_ptr(), self.ld, self.lse.data_ptr(), B, 1, K, V1,
                            blank, slots.kp, 0, 1, 1, val.data_ptr(), idx.data_ptr(),
                            meta.data_ptr(), sp))

    def arenas(self):
        return self.hid, self.layers, self.H, self.fy, self.Hj


class PredictionRows(PredictionNet):
    """Row provider of transducer_decoders.search_batch for a Transducer on a batch of inputs: the
    encoder's fc1 outputs once (time-major, frame t = a contiguous (B, Hj) block), then the rows of
    PredictionNet."""

    def __init__(self, model, inputs):
        with torch.no_grad():
            x = model.stage_inputs(inputs)
            if model.exact_lengths:
                tl = [max(0, model.conv_out_size(i.shape[0], 0)) for i in inputs]
                enc = model._encode(x, torch.tensor(tl, dtype=torch.int32))
            else:
                enc = model._encode(x, None)
            w1, b1 = fc1_operands(model)
            H = model.fc1.fc.out_features
            fx = model.fc1(enc) if w1.shape[0] == H else ops.linear(enc, w1, b1)
            super().__init__(model, fx.shape[0], fx.device, w1, b1)
        self.T = fx.shape[1]
        self.tlens = tl if model.exact_lengths else [self.T] * self.B
        self.fxT = fx.detach().float().transpose(0, 1).contiguous()        # (T', B, Hj)
