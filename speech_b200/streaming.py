"""Streaming recognition with a unidirectional encoder: hypotheses while the audio arrives.

    st = model.stream(num_streams, beam_size=8, lm=lm, lm_weight=0.5)   # CTC or Transducer
    st.push([feats_0, feats_1, ...])      # (n_b, F) new feature frames per stream, n_b may be 0
    hyps = st.partial()                   # best label list of each stream so far

Every stage carries what the next chunk needs and nothing more (EncoderStream, shared by both):
  * conv front-end: a stream keeps its input frames from next_b * prod(strides) onward, next_b its
    next encoder frame, and runs the stack over that carry plus the chunk.  The stack is a valid
    (unpadded) convolution, so its complete output frames are exactly the whole utterance's.
  * GRU layers: the input projection, then the recurrence from each stream's carried state
    (sb_gru_fwd_h0); the new state is the fp32 y and bf16 xn at the stream's last new frame.
CTCStream then runs the fused projection, softmax and log as CTC.infer computes them, and one step
of the resumable prefix beam search (models.ctc_decoder.StreamSearch), whose beams stay on the
device.
With B streams, the final partial(return_scores=True) equals decode_batch(with_scores=True) on the
logits of CTC.infer over the same B utterances in the exact-lengths mode, bit for bit: each stage
computes the same values as the offline pass.  The recurrence kernel is selected by the number of
batch rows, so against an offline batch of another size the results agree only to the GRU's
rounding tolerance.

With a lookahead layer (config["encoder"]["lookahead"] = tau) a stream holds back, per stream, the
top layer's fp32 states of its last <= tau frames (`pending`): a push runs sb_lookahead_fwd over
[pending | new frames] with len_b = pending_b + n_b and searches the first
max(0, pending_b + n_b - tau) of them, whose windows lie wholly below len_b and so carry the bits of
the offline pass.  finish() runs the lookahead over the pending frames alone (len_b = pending_b),
so the trailing frames see zeros as in the offline exact-lengths pass, and searches them; a
finished stream takes no more frames until it is reset.  `frames` counts the frames searched.

TransducerStream runs fc1 on the top layer's bf16 xn of the new frames (the wgmma GEMM with the
padded weights of transducer_model.PredictionNet, as the offline ops.linear does on the same
values), then Transducer.recognize's label-free search resumed over them
(transducer_decoders.StreamSearch): the search state, trie and prediction-state arenas stay on the
device.  Between pushes every stream's beam states are in block 0 of the arenas: a push of n_b
frames leaves stream b's beam in block 0 or S + 1 by the parity of n_b (the beam block flips once
per frame for the whole batch), and one masked copy per arena moves the odd ones back.  After
every push, partial(return_scores=True) equals Transducer.recognize(inputs_so_far, ...,
return_scores=True) in the exact-lengths mode bit for bit, given two preconditions: the same B
(as above), and an offline fc1 on the GEMM, which holds where B * T' >= 128 or H is not a multiple
of 8 (below 128 rows LinearND runs fp32 nn.Linear; the GEMM picks its tile by N only and never
splits K without accumulating, so a row's output does not depend on the number of rows).
Where the search's candidates do not fit the full route (decode_static_fits), the stream reads
64-entry lists from the first frame; partial raises for a stream whose lists flagged a selection,
as recognize would after its rerun, until that stream is reset.
"""
import numpy as np
import torch

from . import _lib, features, ops
from .models.ctc_decoder import StreamSearch, check_lm

MAX_STREAMS = ops.GRU_MAX_BATCH   # one recurrence launch per layer and push


def lookahead_counts(pending, counts, tau, ends=()):
    """With a lookahead of tau frames: the frames each stream searches, and the frames it holds
    back, after counts[b] new encoder frames join its pending[b] ones.  A frame is searched once
    its tau future frames are there, or when its stream ends (streams in `ends`)."""
    tot = [p + n for p, n in zip(pending, counts)]
    emit = [n if b in ends else max(0, n - tau) for b, n in enumerate(tot)]
    return emit, [n - e for n, e in zip(tot, emit)]


class EncoderStream:
    """The encoder half of a stream (see the module docstring): conv carry, per-layer GRU operands
    and states, frames and push_audio.  Subclasses check their arguments, then call
    _init_encoder.  keep_f32: _decode also finds the fp32 top-layer states of the frames it
    searches (post-lookahead) in self.y32, laid out as its bf16 operand."""

    keep_f32 = False

    @staticmethod
    def _check(model, num_streams, beam_size, max_frames):
        B = int(num_streams)
        if not 1 <= B <= MAX_STREAMS:
            raise ValueError("num_streams must lie in [1, %d], got %d" % (MAX_STREAMS, B))
        if model.rnn.bidirectional:
            raise ValueError("a bidirectional encoder cannot stream: it needs the whole utterance")
        if getattr(model, "parity_mode", False):
            raise ValueError("parity_mode has no streaming path")
        if not 1 <= int(beam_size) <= 32:
            raise ValueError("beam_size must lie in [1, 32], got %r" % (beam_size,))
        if int(max_frames) < 1:
            raise ValueError("max_frames must be >= 1, got %r" % (max_frames,))
        return B

    def _init_encoder(self, model, B, max_frames, what):
        if not model.is_cuda:
            raise _lib.SpeechB200Error("%s needs the model on a CUDA device" % what)
        lib = _lib.load()
        self.model = model
        self.B, self.Bp = B, ops._round_up(B, 8)
        self.max_frames = int(max_frames)
        self.dev = dev = next(model.parameters()).device
        self.stride = int(np.prod([c.stride[0] for c in model.conv.children()
                                   if isinstance(c, torch.nn.Conv2d)]))
        rnn = model.rnn
        self.H = H = rnn.hidden_size
        self.Hp = Hp = ops.gru_padded_width(self.Bp, H, 1)
        _, weights = ops._gru_weights(rnn)
        self.layers = []
        with torch.no_grad():
            Kl = ops._round_up(rnn.input_size, 8)
            for l in range(rnn.num_layers):
                self.layers.append(ops.gru_layer_operands(weights[l * 4:(l + 1) * 4], l, Kl, 1, H,
                                                          Hp, dev))
                Kl = Hp
        self.ws_bytes = _lib.workspace_size(lib.sb_gru_fwd_workspace_size, self.Bp, Hp, 1)
        self.ws = ops._workspace(self.ws_bytes, dev)
        self.h = [torch.zeros(self.Bp, Hp, dtype=torch.float32, device=dev) for _ in self.layers]
        self.hb = [torch.zeros(self.Bp, Hp, dtype=torch.bfloat16, device=dev) for _ in self.layers]
        self.carry = [None] * B                  # input frames from next_b * stride on
        self.pcm = [np.zeros(0, np.int16) for _ in range(B)]    # push_audio's carried samples
        self.next = [0] * B                      # encoder frames produced per stream
        self.done = [False] * B                  # finished streams (until reset)
        la = model.lookahead
        self.tau = 0 if la is None else la.kernel_size[0] - 1
        self.npend = [0] * B                     # top-layer frames held back for the lookahead
        self.y32 = None              # with keep_f32: fp32 top-layer states of the frames searched
        if self.tau:
            with torch.no_grad():
                self.taps = ops.lookahead_taps(la.weight, H, Hp)
            self.pend = torch.zeros(B * self.tau, Hp, dtype=torch.float32, device=dev)

    @property
    def frames(self):
        """encoder frames searched per stream; frame t starts at input frame t * prod(strides)"""
        return [n - p for n, p in zip(self.next, self.npend)]

    @property
    def pending(self):
        """encoder frames per stream held back until the lookahead's future frames arrive"""
        return list(self.npend)

    def _reset_encoder(self, b):
        b = int(b)
        if not 0 <= b < self.B:
            raise ValueError("stream %d out of range [0, %d)" % (b, self.B))
        self.carry[b] = None
        self.pcm[b] = np.zeros(0, np.int16)
        self.next[b] = 0
        self.done[b] = False
        self.npend[b] = 0
        for h, hb in zip(self.h, self.hb):
            h[b].zero_()
            hb[b].zero_()
        return b

    # ---- conv front-end ----
    def _conv_inputs(self, chunks):
        """the carry + chunk of each stream and the encoder frames it completes (host only)"""
        if len(chunks) != self.B:
            raise ValueError("push takes one chunk per stream (%d), got %d" % (self.B, len(chunks)))
        xs, counts = [], []
        for b, c in enumerate(chunks):
            c = torch.as_tensor(c)
            if c.dim() != 2:
                raise ValueError("chunk %d must be (frames, features), got shape %s"
                                 % (b, tuple(c.shape)))
            c = c.to(self.dev, torch.float32)
            x = c if self.carry[b] is None else torch.cat([self.carry[b], c], 0)
            xs.append(x)
            counts.append(max(0, self.model.conv_out_size(x.shape[0], 0)))
        F = xs[0].shape[1]
        if any(x.shape[1] != F for x in xs):
            raise ValueError("every chunk must have the same number of features")
        for b, n in enumerate(counts):
            if self.next[b] + n > self.max_frames:
                raise ValueError("stream %d would pass max_frames = %d (%d + %d encoder frames)"
                                 % (b, self.max_frames, self.next[b], n))
        return xs, counts

    def _advance(self, xs, counts):
        """drop the input frames no later encoder frame reads: frame next_b starts at input frame
        next_b * stride of the stream, and so every strided layer stays aligned"""
        for b, n in enumerate(counts):
            self.carry[b] = xs[b][n * self.stride:]
            self.next[b] += n

    def _encoder(self, xs, counts, T):
        """(T * Bp, Hp) bf16 xn and f32 y of the top GRU layer at the new encoder frames (frame t
        of stream b at row t * Bp + b; rows past counts[b] unused)"""
        lib = _lib.load()
        B, Bp, Hp, dev = self.B, self.Bp, self.Hp, self.dev
        L = max(x.shape[0] for x in xs)
        x = torch.zeros(B, L, xs[0].shape[1], dtype=torch.float32, device=dev)
        for b, xb in enumerate(xs):
            x[b, :xb.shape[0]] = xb
        feats = ops.conv_stack(x, self.model.conv, False)[:, :T]       # (B, T, In)
        In = feats.shape[2]
        X = torch.zeros(T, Bp, ops._round_up(In, 8), dtype=torch.bfloat16, device=dev)
        X[:, :B, :In] = feats.transpose(0, 1)
        X = X.view(T * Bp, -1)
        last = torch.tensor(counts + [0] * (Bp - B), dtype=torch.int64).to(dev) * Bp + \
            torch.arange(Bp, device=dev)                                # frame counts[b] of y
        sp = _lib.stream_ptr()
        for l, (wih, whh, bih, bhh) in enumerate(self.layers):
            gi = ops.gemm_bf16_tn(X, wih, bias=bih)
            y = torch.empty((T + 1) * Bp, Hp, dtype=torch.float32, device=dev)
            xn = torch.empty((T + 1) * Bp, Hp, dtype=torch.bfloat16, device=dev)
            h, hb = self.h[l], self.hb[l]
            ops._launch("gru_fwd", 2.0 * T * Bp * 3 * Hp * Hp,
                        lambda: lib.sb_gru_fwd_h0(gi.data_ptr(), whh.data_ptr(), bhh.data_ptr(),
                                                  h.data_ptr(), hb.data_ptr(), y.data_ptr(),
                                                  xn.data_ptr(), None, self.ws.data_ptr(),
                                                  self.ws_bytes, T, Bp, Hp, 1, sp))
            h.copy_(y[last])
            hb.copy_(xn[last])
            X = xn[Bp:]
        return X, y[Bp:]

    def _lookahead(self, Y, counts, T, ends):
        """The lookahead over [pending | counts[b] new frames of Y] of every stream, len_b their
        sum: -> (frames to search per stream, Te, (Te * Bp, Hp) bf16 operand of the projection).
        A stream of `ends` searches all its frames, any other the frames whose window is complete;
        the rest become its new pending frames."""
        B, Bp, Hp, tau, dev = self.B, self.Bp, self.Hp, self.tau, self.dev
        tot = [p + n for p, n in zip(self.npend, counts)]
        Tl = max(tot)
        emit, keep = lookahead_counts(self.npend, counts, tau, ends)
        # one gather from [pending rows | Y rows | a zero row]
        zero = B * tau + T * Bp
        idx = np.full((Tl, Bp), zero, np.int64)
        for b in range(B):
            p = self.npend[b]
            idx[:p, b] = b * tau + np.arange(p)
            idx[p:tot[b], b] = B * tau + np.arange(counts[b]) * Bp + b
        parts = [self.pend] + ([Y[:T * Bp]] if T else []) + [self.pend.new_zeros(1, Hp)]
        src = torch.cat(parts)
        h = src[torch.from_numpy(idx.reshape(-1)).to(dev)]
        lens = torch.tensor(tot + [0] * (Bp - B), dtype=torch.int32).to(dev)
        rb = torch.empty(Tl * Bp, Hp, dtype=torch.bfloat16, device=dev)
        r = torch.empty(Tl * Bp, Hp, dtype=torch.float32, device=dev) if self.keep_f32 else None
        ops.lookahead_fwd(h, self.taps, lens, r, rb, Tl, Bp, Hp, tau)
        pidx = np.full((B, tau), Tl * Bp, np.int64)
        for b in range(B):
            pidx[b, :keep[b]] = (emit[b] + np.arange(keep[b])) * Bp + b
        self.npend = keep
        self.pend = torch.cat([h, h.new_zeros(1, Hp)])[torch.from_numpy(pidx.reshape(-1)).to(dev)]
        Te = max(emit)
        self.y32 = None if r is None else r[:Te * Bp]
        return emit, Te, rb[:Te * Bp]

    def push(self, chunks):
        """Feed one (n_b, F) chunk of feature frames to every stream (n_b may be 0; a finished
        stream takes none): runs the encoder over the encoder frames the chunks complete and
        advances each stream's search over the frames it can search.  -> encoder frames completed
        per stream."""
        xs, counts = self._conv_inputs(chunks)
        for b, c in enumerate(chunks):
            if self.done[b] and len(c) > 0:
                raise ValueError("stream %d is finished: reset(%d) before pushing to it" % (b, b))
        T = max(counts)
        if T > 0:
            with torch.no_grad():
                emit, Te, X = self._encode(xs, counts, T)
                if Te > 0:
                    self._decode(X, emit, Te)
        self._advance(xs, counts)
        return counts

    def _encode(self, xs, counts, T):
        """The encoder over counts[b] new encoder frames per stream (T = max(counts) > 0), and the
        lookahead if the model has one: -> (frames to search per stream, Te = their maximum,
        (Te * Bp, Hp) bf16 operand of the output projection, frame t of stream b at row
        t * Bp + b)"""
        X, Y = self._encoder(xs, counts, T)
        if not self.tau:
            self.y32 = Y if self.keep_f32 else None
            return counts, T, X
        return self._lookahead(Y, counts, T, ())

    def finish(self, streams=None):
        """End the listed streams (all when None): search their pending frames, the lookahead
        seeing zeros past each utterance's end, and refuse further frames until reset(b).
        Finishing a finished stream does nothing."""
        bs = range(self.B) if streams is None else [int(b) for b in streams]
        for b in bs:
            if not 0 <= b < self.B:
                raise ValueError("stream %d out of range [0, %d)" % (b, self.B))
        ends = {b for b in bs if not self.done[b]}
        if self.tau and any(self.npend[b] for b in ends):
            with torch.no_grad():
                emit, Te, X = self._lookahead(None, [0] * self.B, 0, ends)
                self._decode(X, emit, Te)
        for b in ends:
            self.done[b] = True

    def push_audio(self, pcm, sample_rate=16000, mean=None, std=None, window_size=20, step_size=10,
                   eps=1e-10):
        """Feed int16 PCM samples per stream: featurised by features.log_specgram_batch (same
        arguments) over the samples carried from the last call plus the new ones, so that every
        feature frame is the one the whole-utterance featuriser computes; then push."""
        if len(pcm) != self.B:
            raise ValueError("push_audio takes one array per stream (%d), got %d"
                             % (self.B, len(pcm)))
        nperseg = int(window_size * sample_rate / 1e3)
        step = nperseg - int(step_size * sample_rate / 1e3)
        audio = []
        for b, a in enumerate(pcm):
            a = np.asarray(a)
            if a.dtype != np.int16 or a.ndim != 1:
                raise ValueError("push_audio expects 1-D int16 arrays")
            if self.done[b] and a.size > 0:
                raise ValueError("stream %d is finished: reset(%d) before pushing to it" % (b, b))
            audio.append(np.concatenate([self.pcm[b], a]))
        nf = [features.frame_count(len(a), nperseg, step) for a in audio]
        if max(nf) > 0:
            feats, _ = features.log_specgram_batch(audio, sample_rate, mean=mean, std=std,
                                                   window_size=window_size, step_size=step_size,
                                                   eps=eps, device=self.dev)
            chunks = [feats[b, :nf[b]] for b in range(self.B)]
        else:
            chunks = [torch.zeros(0, nperseg // 2 + 1, device=self.dev) for _ in range(self.B)]
        counts = self.push(chunks)
        for b, a in enumerate(audio):
            self.pcm[b] = a[nf[b] * step:]
        return counts


class CTCStream(EncoderStream):
    """B streams of one unidirectional CTC model (see the module docstring).  Built by
    CTC.stream; the model's weights are read once, when the stream is built."""

    def __init__(self, model, num_streams, beam_size=1, max_frames=3000, lm=None, lm_weight=0.0,
                 insertion_bonus=0.0):
        B = self._check(model, num_streams, beam_size, max_frames)
        check_lm(lm, lm_weight, insertion_bonus, model.blank + 1, model.blank)
        self._init_encoder(model, B, max_frames, "CTC.stream")
        with torch.no_grad():
            self.fc_w = ops.fc_operand(model.fc.fc.weight, 1, self.H, self.Hp)
            self.fc_b = model.fc.fc.bias.detach().float().contiguous()
        self.search = StreamSearch(B, self.max_frames, beam_size, model.blank, self.dev, lm,
                                   lm_weight, insertion_bonus)

    def reset(self, b):
        """start slot b afresh: conv carry, GRU states, pending frames and search"""
        self.search.reset(self._reset_encoder(b), 1)

    def _decode(self, X, counts, T):
        self.search.push(self._logp(X, T), counts)

    def _logp(self, X, T):
        """(B, T, S) log-probabilities of the (T * Bp, Hp) bf16 top-layer operand X (rows past
        each stream's frames unused)"""
        B, Bp = self.B, self.Bp
        out = ops.gemm_bf16_tn(X, self.fc_w, bias=self.fc_b, remap=(Bp, T, B))
        out = out.view(B, T, -1)
        # CTC.infer: softmax over the classes, then decode_batch's float32 log
        probs = torch.nn.functional.softmax(out, dim=2)
        return torch.log(probs.float()).contiguous()

    def partial(self, return_scores=False):
        """Best label list of each stream so far (one device-to-host copy); with return_scores,
        (labels, score) pairs, the score as decode_batch(with_scores=True) reports it.  With a
        WordLM the stored beams are ranked by the end-of-utterance rule, as if each stream ended
        here (its partial word completed, then </s>)."""
        return self.search.best(return_scores)


class TransducerStream(EncoderStream):
    """B streams of one Transducer with a unidirectional encoder (see the module docstring).
    Built by Transducer.stream; the model's weights are read once, when the stream is built.
    beam_size, max_symbols_per_frame, max_len and the LM arguments are Transducer.recognize's;
    max_frames caps the encoder frames per stream between resets (it sizes the search's trie)."""

    def __init__(self, model, num_streams, beam_size=4, max_symbols_per_frame=4, max_frames=3000,
                 max_len=None, lm=None, lm_weight=0.0, insertion_bonus=0.0):
        from .models.transducer_model import PredictionNet
        from .transducer_decoders import StreamSearch, check_stream_args
        B = self._check(model, num_streams, beam_size, max_frames)
        check_stream_args(beam_size, max_symbols_per_frame, max_frames, max_len,
                          model.fc2.fc.out_features, model.blank, lm, lm_weight, insertion_bonus)
        self._init_encoder(model, B, max_frames, "Transducer.stream")
        with torch.no_grad():
            self.pred = PredictionNet(model, B, self.dev)
        self.Kr = ops._round_up(self.H, 8)     # the contraction of the offline ops.linear
        self.search = StreamSearch(self.pred, beam_size, max_symbols_per_frame, max_frames,
                                   model.blank, max_len, lm, lm_weight, insertion_bonus)

    def reset(self, b):
        """start slot b afresh: conv carry, GRU states, pending frames, search and its prediction
        states"""
        self.search.reset(self._reset_encoder(b))

    def _decode(self, X, counts, T):
        self._fc1(X, T)
        self.search.push(counts)

    def _fc1(self, X, T):
        """fc1 of the (T * Bp, Hp) bf16 top-layer operand X into the prediction network's fxT:
        (T, Bp, Hj), frame t of stream b at [t, b].  X's columns H .. Kr - 1 are zero (padded GRU
        units and lookahead taps stay 0), as the offline ops.linear's zero padding of bf16(y)."""
        fx = ops.gemm_bf16_tn(X[:, :self.Kr], self.pred.w1, bias=self.pred.b1)
        self.pred.fxT = fx.view(T, self.Bp, -1)

    def partial(self, return_scores=False):
        """Best label list of each stream so far (one device-to-host copy); with return_scores,
        (labels, score) pairs, the float64 score as Transducer.recognize(return_scores=True)
        reports it.  Raises SpeechB200Error naming the streams whose shortlists flagged a
        selection (the large-vocabulary route only)."""
        labels, scores = self.search.best()
        res = [tuple(int(v) for v in lab) for lab in labels]
        return list(zip(res, scores)) if return_scores else res


class Seq2SeqStream(EncoderStream):
    """B streams of two-pass recognition with one hybrid CTC/attention Seq2Seq (unidirectional
    encoder, CTC head).  Built by Seq2Seq.stream; the model's weights are read once, when the
    stream is built.

    First pass, per push: the CTC head (ctc_fc with bias) on the top layer's new bf16 states, on
    the wgmma GEMM with the padded weights of the offline ops.linear, a float32 log_softmax, and one
    step of the resumable prefix beam search (StreamSearch, blank V - 2, no LM).  The fp32
    top-layer states of the frames searched (post-lookahead: the values Seq2Seq._encode returns)
    are appended to a per-stream arena of B * max_frames * H * 4 bytes.
    partial() is the first pass's best so far; rescored() reads every stream's N-best
    (StreamSearch.nbest) and runs the attention rescoring of Seq2Seq.recognize_two_pass over the
    frames searched so far.  After finish(), rescored(return_scores=True) equals
    recognize_two_pass(inputs, return_scores=True) bit for bit in the exact-lengths mode with the
    same B, where the offline ctc_fc runs on the GEMM (B * T' >= 128 or H not a multiple of 8, as
    for TransducerStream)."""

    keep_f32 = True

    def __init__(self, model, num_streams, beam_size=10, max_frames=3000, ctc_weight=0.5):
        B = self._check(model, num_streams, beam_size, max_frames)
        model._check_two_pass(beam_size, ctc_weight)
        self._init_encoder(model, B, max_frames, "Seq2Seq.stream")
        self.K, self.ctc_weight = int(beam_size), float(ctc_weight)
        self.Kr = ops._round_up(self.H, 8)     # the contraction of the offline ops.linear
        with torch.no_grad():
            fc = model.ctc_fc.fc
            self.fc_w = torch.nn.functional.pad(fc.weight.detach().to(torch.bfloat16),
                                                (0, self.Kr - self.H)).contiguous()
            self.fc_b = fc.bias.detach().float().contiguous()
        self.arena = torch.zeros(B, self.max_frames, self.H, dtype=torch.float32, device=self.dev)
        self.searched = [0] * B
        self.search = StreamSearch(B, self.max_frames, self.K,
                                   model.embedding.num_embeddings - 2, self.dev)

    def reset(self, b):
        """start slot b afresh: conv carry, GRU states, pending frames, search and arena"""
        b = self._reset_encoder(b)
        self.searched[b] = 0
        self.arena[b].zero_()
        self.search.reset(b, 1)

    def _decode(self, X, counts, T):
        B, Bp, H = self.B, self.Bp, self.H
        logits = ops.gemm_bf16_tn(X[:, :self.Kr], self.fc_w, bias=self.fc_b)
        y = logits.view(T, Bp, -1)[:, :B].transpose(0, 1).contiguous()
        y = torch.log_softmax(y.float(), dim=-1).contiguous()
        self.search.push(y, counts)
        src, dst = [], []
        for b, n in enumerate(counts):
            src += [t * Bp + b for t in range(n)]
            dst += [b * self.max_frames + self.searched[b] + t for t in range(n)]
            self.searched[b] += n
        if src:
            rows = self.y32[torch.tensor(src, device=self.dev), :H]
            self.arena.view(-1, H).index_copy_(0, torch.tensor(dst, device=self.dev), rows)

    def partial(self, return_scores=False):
        """Best label list of each stream so far, the first pass alone (one device-to-host copy);
        with return_scores, (labels, score) pairs, the score -c_0 as CTCStream.partial reports it."""
        return self.search.best(return_scores)

    def rescored(self, return_scores=False):
        """The second pass over every stream's frames searched so far: each stream's N-best
        rescored by the attention as Seq2Seq.recognize_two_pass does; -> its output.  Raises
        ValueError while a stream has searched no frame (the attention needs one)."""
        from .functions import s2s
        empty = [b for b, f in enumerate(self.searched) if f == 0]
        if empty:
            raise ValueError("streams %s have searched no frame yet" % empty)
        T = max(self.searched)
        with torch.no_grad(), torch.cuda.device(self.dev):
            return s2s.rescore(self.model, self.arena[:, :T], self.search.nbest(),
                               list(self.searched), self.K, self.ctc_weight, return_scores)
