"""Encoder base class - host-side mirror of speech/models/model.py:10-113 (reference).

Same constructor, attributes, state_dict key names (`conv.{0,2,..}.{weight,bias}`,
`rnn.weight_ih_l{k}[_reverse]` ...) and picklability as the reference `Model`; the nn.Conv2d /
nn.GRU modules are kept as PARAMETER CONTAINERS (identical construction order => identical
initialisation under the same torch seed) while the arithmetic of `encode` runs in the
hand-written sm_90a kernels (speech_b200/ops.py -> csrc/).  There is no CPU path: calling
`encode` on a CPU tensor raises.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from .. import _lib, ops


class Model(nn.Module):

    # Exact-lengths mode (config key "exact_lengths"; off by default, as in the reference): every
    # utterance is encoded, scored and decoded over its own frames, len_b = conv_out_size(T_b, 0),
    # so its results do not depend on the other utterances of its minibatch.  A class attribute,
    # so that pickles written before the key existed read it as False.
    exact_lengths = False

    # Lookahead convolution (config["encoder"]["lookahead"] = tau; absent or 0 by default): Deep
    # Speech 2's row convolution r[t, d] = sum_{j=0..tau} W[d, j] h[t + j, d] over the top layer
    # of a unidirectional encoder, so every frame sees tau frames of future context.  Read through
    # a property of the class, so that pickles written before the key existed read it as None; a
    # plain class attribute would shadow the registered submodule.
    @property
    def lookahead(self):
        return self._modules.get("lookahead")

    @lookahead.setter
    def lookahead(self, value):
        # nn.Module.__setattr__ registers a module value itself; only None, on a model that has
        # no layer, reaches here
        if value is not None:
            raise TypeError("lookahead must be an nn.Conv1d or None, got %r" % (value,))
        self._modules["lookahead"] = None

    def __init__(self, input_dim, config):
        super().__init__()
        self.input_dim = input_dim
        enc = config["encoder"]
        layers = []
        in_c = 1
        out_c = 1
        for out_c, h, w, s in enc["conv"]:
            layers.append(nn.Conv2d(in_c, out_c, (h, w), stride=(s, s), padding=0))
            layers.append(nn.ReLU())
            if config["dropout"] != 0:
                layers.append(nn.Dropout(p=config["dropout"]))
            in_c = out_c
        self.conv = nn.Sequential(*layers)
        conv_out = out_c * self.conv_out_size(input_dim, 1)
        assert conv_out > 0, "Convolutional output frequency dimension is negative."

        rnn_cfg = enc["rnn"]
        self.rnn = nn.GRU(input_size=conv_out, hidden_size=rnn_cfg["dim"],
                          num_layers=rnn_cfg["layers"], batch_first=True,
                          dropout=config["dropout"], bidirectional=rnn_cfg["bidirectional"])
        self._encoder_dim = rnn_cfg["dim"]
        self.volatile = False
        self.exact_lengths = bool(config.get("exact_lengths", False))
        tau = enc.get("lookahead", 0)
        if isinstance(tau, bool) or not isinstance(tau, int) or not 0 <= tau <= 32:
            raise ValueError("encoder lookahead must be an int in [0, 32], got %r" % (tau,))
        if tau > 0 and rnn_cfg["bidirectional"]:
            raise ValueError("encoder lookahead needs a unidirectional encoder: a bidirectional "
                             "one already sees the whole utterance")
        self._lookahead_tau = tau

    def _add_lookahead(self):
        """Each family calls this after creating all its other modules, so that with the same
        seed a model with a lookahead initialises every other parameter as one without."""
        tau = self._lookahead_tau
        if tau > 0:
            H = self.encoder_dim
            self.lookahead = nn.Conv1d(H, H, tau + 1, groups=H, bias=False)

    # reference: model.py:44-52 (valid convolution, ceil((n - k + 1) / s) per layer)
    def conv_out_size(self, n, dim):
        for c in self.conv.children():
            if isinstance(c, nn.Conv2d):
                k, s = c.kernel_size[dim], c.stride[dim]
                n = int(math.ceil((n - k + 1) / s))
        return n

    def forward(self, batch):
        raise NotImplementedError

    def loss(self, batch):
        raise NotImplementedError

    def infer(self, batch):
        raise NotImplementedError

    def encode(self, x, lens=None):
        """x (B, T, F) float32 on the CUDA device -> (B, T', encoder_dim)   (model.py:60-79).
        lens (optional): valid output frames per utterance (x_lens of the exact-lengths mode);
        states at frames < lens[b] are then those of the utterance alone, later frames are zero."""
        _lib.require_cuda(x, "encode() input")
        x = ops.conv_stack(x, self.conv, self.training)          # (B, T', C*F') c-major features
        p = self.rnn.dropout if self.training else 0.0
        x = ops.gru_stack(x, self.rnn, dropout=p, lens=lens,     # (B, T', ndir*H)
                          lookahead=self.lookahead)
        if self.rnn.bidirectional:
            half = x.shape[-1] // 2
            x = x[:, :, :half] + x[:, :, half:]
        return x

    def set_eval(self):
        self.eval()
        self.volatile = True

    def set_train(self):
        self.train()
        self.volatile = False

    @property
    def is_cuda(self):
        return next(self.parameters()).is_cuda

    @property
    def encoder_dim(self):
        return self._encoder_dim

    # ---- batch assembly shared by the three model families ------------------------------------
    def stage_inputs(self, inputs):
        """list of (T_i, F) arrays -> zero padded (B, max T, F) float32 tensor, already on the
        model's device when that is a GPU (pinned staging + asynchronous copy)."""
        if self.is_cuda:
            return zero_pad_concat_device(inputs, next(self.parameters()).device)
        return torch.from_numpy(zero_pad_concat(inputs))

    def lattice_batch(self, inputs, labels):
        """[x, flat int32 labels, x_lens, y_lens] as the CTC and transducer losses take them
        (ctc_model.py:42-53, transducer_model.py:79-90): every utterance is scored over the
        padded T' - or, in the exact-lengths mode, over its own conv_out_size(T_b) frames; labels
        and lengths stay on the host."""
        if self.exact_lengths:
            # the valid conv makes these frames exact: output frame t reads input frames
            # <= t*s + k - 1 <= T_b - 1 in every layer
            x_lens = torch.tensor([max(0, self.conv_out_size(i.shape[0], 0)) for i in inputs],
                                  dtype=torch.int32)
        else:
            frames = self.conv_out_size(max(i.shape[0] for i in inputs), 0)
            x_lens = torch.full((len(inputs),), frames, dtype=torch.int32)
        y_lens = torch.tensor([len(seq) for seq in labels], dtype=torch.int32)
        flat = torch.tensor([int(tok) for seq in labels for tok in seq], dtype=torch.int32)
        return [self.stage_inputs(inputs), flat, x_lens, y_lens]

    def _encode(self, x, lens):
        # without lengths, call encode exactly as the default mode always has (callers may
        # substitute a one-argument encode, e.g. to feed precomputed encoder states)
        return self.encode(x) if lens is None else self.encode(x, lens)

    def exact_lens(self, x_lens):
        """x_lens for the encoder in the exact-lengths mode, else None (the reference's padding)."""
        return x_lens if self.exact_lengths else None

    def _grad_ctx(self):
        # the reference marks eval batches `volatile`; on modern torch that is no_grad
        return torch.no_grad() if self.volatile else torch.enable_grad()


class LinearND(nn.Module):
    """nn.Linear over the last dimension of an N-D input (reference model.py:115-133)."""

    def __init__(self, *args):
        super().__init__()
        self.fc = nn.Linear(*args)

    def forward(self, x):
        # time-batched projections run on the package's wgmma GEMM (forward and backward);
        # per-token rows of the attention decoder (a handful of rows) stay in fp32
        _lib.require_cuda(x, "LinearND input")
        if x.numel() // x.shape[-1] >= 128 and self.fc.out_features >= 8:
            return ops.linear(x, self.fc.weight, self.fc.bias)
        lead = x.shape[:-1]
        out = self.fc(x.reshape(-1, x.shape[-1]))
        return out.view(*lead, out.shape[-1])


def zero_pad_concat(inputs):
    """list of (T_i, F) arrays -> (B, max T, F) float32, zero padded (reference model.py:135-141)."""
    max_t = max(inp.shape[0] for inp in inputs)
    out = np.zeros((len(inputs), max_t, inputs[0].shape[1]), dtype=np.float32)
    for e, inp in enumerate(inputs):
        out[e, :inp.shape[0], :] = inp
    return out


def end_pad_labels(labels):
    """(B, max U) int64 matrix of label sequences, short rows filled with the LAST token of the
    FIRST sequence - the end token (seq2seq.py:239-248, transducer_model.py:103-116)."""
    filler = labels[0][-1]
    width = max(len(seq) for seq in labels)
    mat = np.full((len(labels), width), fill_value=filler, dtype=np.int64)
    for row, seq in enumerate(labels):
        mat[row, :len(seq)] = seq
    return mat


_pinned = {}
_pool = None
_staging_lock = __import__("threading").Lock()   # the training thread and a loader.BatchPrefetcher
                                                 # worker may both assemble batches


def _staging(shape):
    buf = _pinned.get(shape)
    if buf is None:
        buf = [torch.zeros(shape, dtype=torch.float32).pin_memory(), None]   # tensor, last H2D event
        _pinned.clear()
        _pinned[shape] = buf
    return buf


def zero_pad_concat_pinned(inputs):
    """zero_pad_concat into a reused PINNED staging tensor (host tensor; H2D is the caller's)."""
    max_t = max(inp.shape[0] for inp in inputs)
    shape = (len(inputs), max_t, inputs[0].shape[1])
    buf = _staging(shape)
    if buf[1] is not None:
        buf[1].synchronize()
        buf[1] = None
    arr = buf[0].numpy()
    for e, inp in enumerate(inputs):
        n = inp.shape[0]
        arr[e, :n, :] = inp
        if n < max_t:
            arr[e, n:, :] = 0.0
    return buf[0]


def zero_pad_concat_device(inputs, device, chunk=8, threads=4):
    """Batch assembly straight to the GPU (SURVEY.md section 8f rank 1): utterances are written
    into a reused pinned staging buffer by a few host threads, chunk by chunk, and every finished
    chunk is copied to the device asynchronously while the next ones are still being filled, so
    the host memcpy and the PCIe transfer overlap.  Returns the (B, max T, F) float32 CUDA tensor
    zero-padded like the reference's zero_pad_concat (model.py:135-141)."""
    with _staging_lock:
        return _zero_pad_concat_device_locked(inputs, device, chunk, threads)


def _zero_pad_concat_device_locked(inputs, device, chunk, threads):
    global _pool
    from concurrent.futures import ThreadPoolExecutor
    max_t = max(inp.shape[0] for inp in inputs)
    B, F = len(inputs), inputs[0].shape[1]
    shape = (B, max_t, F)
    buf = _staging(shape)
    if buf[1] is not None:
        buf[1].synchronize()           # the previous batch's H2D must be done before we overwrite
    arr = buf[0].numpy()
    out = torch.empty(shape, dtype=torch.float32, device=device)

    def fill(lo, hi):
        for e in range(lo, hi):
            n = inputs[e].shape[0]
            arr[e, :n, :] = inputs[e]
            if n < max_t:
                arr[e, n:, :] = 0.0
        return lo, hi

    if _pool is None:
        _pool = ThreadPoolExecutor(max_workers=threads)
    futs = [_pool.submit(fill, lo, min(B, lo + chunk)) for lo in range(0, B, chunk)]
    for f in futs:                      # in order: chunk k goes out while k+1.. are being filled
        lo, hi = f.result()
        out[lo:hi].copy_(buf[0][lo:hi], non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    buf[1] = ev
    return out
