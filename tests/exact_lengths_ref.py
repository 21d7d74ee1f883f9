"""Length-aware CPU restatement of the encoder and the CTC loss (test infrastructure, never
imported by speech_b200/): what the exact-lengths mode must compute.

  packed_encode     oracle.model_ref.RefEncoder with its nn.GRU run over pack_padded_sequence of
                    each utterance's own len_b = time_out(T_b) frames (same weights); frames
                    >= len_b are zero, as pad_packed_sequence leaves them
  packed_ctc_costs  per-utterance CTC over frames < len_b (log_softmax + F.ctc_loss)
  masked_decode_ref Seq2Seq teacher-forced decode with NNAttention masked to each utterance's frames
The per-utterance RNN-T restatement is oracle/rnnt_ref.py, which already takes x_lens.
"""
import torch
import torch.nn.functional as F
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence


def packed_encode(enc, x, in_lens):
    """enc: oracle.model_ref.RefEncoder; x (B, T, F) zero padded; in_lens: input frames T_b.
    -> (B, T', dim) encoder states, (B,) int64 len_b."""
    y = enc.conv(x.unsqueeze(1))                          # valid conv: frames < len_b are exact
    b, c, t, f = y.shape
    y = y.transpose(1, 2).reshape(b, t, c * f)
    lens = torch.tensor([max(0, enc.time_out(int(n))) for n in in_lens], dtype=torch.int64)
    packed = pack_padded_sequence(y, lens, batch_first=True, enforce_sorted=False)
    out, _ = enc.rnn(packed)
    out, _ = pad_packed_sequence(out, batch_first=True, total_length=t)
    if enc.rnn.bidirectional:
        out = out[..., :enc.dim] + out[..., enc.dim:]
    return out, lens


def packed_ctc_costs(logits, lens, labels_flat, label_lens, blank):
    """logits (B, T', V+1), lens (B,) valid frames -> (B,) costs over each utterance's frames."""
    lp = F.log_softmax(logits, 2).transpose(0, 1)
    return F.ctc_loss(lp, labels_flat.long(), torch.as_tensor(lens).long(),
                      torch.as_tensor(label_lens).long(), blank=blank, reduction="none",
                      zero_infinity=False)


def masked_decode_ref(m, x, y, lens):
    """Teacher-forced Seq2Seq decode (seq2seq.py:78-112) with the NNAttention of :344-360 masked to
    each utterance's frames, in float64 on the CPU with the model's parameters: scores at
    t >= lens[b] are -inf (a_t = 0), log_t scales by log(lens[b]), the location conv reads the
    (zero) alignment past lens[b].  x (B, T, H) encoder states, y (B, U) tokens.
    -> logits (B, U-1, C), alignments (B, U-1, T), the float64 leaf x, {name: float64 parameter}."""
    import math
    import torch.nn as nn
    H = x.shape[2]
    emb = m.embedding.weight.detach().double().cpu().requires_grad_(True)
    cell = nn.GRUCell(emb.shape[1], H).double()
    cell.load_state_dict({k: v.detach().double().cpu() for k, v in m.dec_rnn.state_dict().items()})
    conv = nn.Conv1d(1, H, m.attend.conv.kernel_size[0], padding=m.attend.conv.padding[0]).double()
    conv.load_state_dict({k: v.detach().double().cpu() for k, v in m.attend.conv.state_dict().items()})
    lin = nn.Linear(H, 1).double()
    lin.load_state_dict({k: v.detach().double().cpu()
                         for k, v in m.attend.nn[1].fc.state_dict().items()})
    fc = nn.Linear(H, m.fc.fc.out_features).double()
    fc.load_state_dict({k: v.detach().double().cpu() for k, v in m.fc.fc.state_dict().items()})
    x = x.detach().double().cpu().requires_grad_(True)
    y = y.cpu()
    B, T = x.shape[0], x.shape[1]
    lens_t = torch.as_tensor(lens, dtype=torch.int64)
    valid = torch.arange(T)[None, :] < lens_t[:, None]
    scale = torch.tensor([math.log(int(n)) if m.attend.log_t else 1.0 for n in lens],
                         dtype=torch.float64)[:, None]
    hx = torch.zeros(B, H, dtype=torch.float64)
    ax = sx = None
    out, aligns = [], []
    for t in range(y.shape[1] - 1):
        ix = emb[y[:, t]]
        if sx is not None:
            ix = ix + sx
        hx = cell(ix, hx)
        pax = x + hx.unsqueeze(1)
        if ax is not None:
            pax = pax + conv(ax.unsqueeze(1)).transpose(1, 2)
        pax = lin(torch.relu(pax)).squeeze(2) * scale
        pax = pax.masked_fill(~valid, -float("inf"))
        ax = torch.softmax(pax, dim=1)
        sx = torch.sum(x * ax.unsqueeze(2), dim=1)
        aligns.append(ax)
        out.append(fc(hx + sx))
    params = {"embedding.weight": emb, "dec_rnn.weight_ih": cell.weight_ih,
              "dec_rnn.weight_hh": cell.weight_hh, "dec_rnn.bias_ih": cell.bias_ih,
              "dec_rnn.bias_hh": cell.bias_hh, "attend.conv.weight": conv.weight,
              "attend.conv.bias": conv.bias, "attend.nn.1.fc.weight": lin.weight,
              "attend.nn.1.fc.bias": lin.bias, "fc.fc.weight": fc.weight, "fc.fc.bias": fc.bias}
    return torch.stack(out, 1), torch.stack(aligns, 1), x, params
