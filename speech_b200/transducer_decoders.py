"""Drop-in for `transducer.decoders` of awni/transducer (imported at
speech/models/transducer_model.py:10, used at :100 as `td.decode_static(lp, beam_size, blank)[0]`).

The beam search runs on the GPU (csrc/tdecode.cu, one CTA per utterance; hypotheses in a canonical
trie, float64 scores); `decode_static` keeps the reference's per-utterance call signature and
returns (labels, log_probability) so that `[0]` is the label list, `decode_static_batch` searches
a whole minibatch of lattices with one launch and one device->host copy (what
`Transducer.infer` uses).  The dependency is un-vendored (Makefile:10-12), so the algorithm is the
standard transducer beam search on a static lattice; its CPU restatement and how it is pinned are
in oracle/decode_static_ref.py (test infrastructure - not imported here).  There is no CPU path.

The search keeps every candidate in shared memory where beam_size * V * 8 bytes fit in 200 KB
(`decode_static_fits`).  Larger vocabularies search per-node shortlists instead (the kp = beam_size
best non-blank classes, csrc/tdecode.cu), with the same results bit for bit: the kernel flags any
selection the lists cannot prove, and flagged utterances are searched again from lists of
SHORTLIST_RERUN entries.
"""
import torch

from . import _lib, ops
from .lm import fusion_args

SHORTLIST_RERUN = 64      # list length of the second search of flagged utterances (the maximum)


def decode_static_fits(beam_size, V):
    """True where sb_rnnt_decode_static holds the beam_size * V candidates in shared memory
    (beam_size * V * 8 + 16 <= 200 KB, beam_size <= 32); elsewhere the shortlist search runs."""
    return bool(_lib.load().sb_rnnt_decode_static_fits(int(beam_size), int(V)))


def alloc_shortlists(B, T, U1, kp, device):
    """Empty batch-first shortlists: values (B,T,U1,kp) f32, classes (B,T,U1,kp) int32 and
    {blank lp, next lp} (B,T,U1,2) f32, as sb_rnnt_shortlist_rows writes them."""
    return (torch.empty(B, T, U1, kp, dtype=torch.float32, device=device),
            torch.empty(B, T, U1, kp, dtype=torch.int32, device=device),
            torch.empty(B, T, U1, 2, dtype=torch.float32, device=device))


def shortlists_of_lp(lp, kp, blank):
    """Shortlists of a given (B, T, U1, V) float32 CUDA log-probability tensor."""
    lib = _lib.load()
    B, T, U1, V = lp.shape
    val, idx, meta = alloc_shortlists(B, T, U1, kp, lp.device)
    with torch.cuda.device(lp.device):
        sp = _lib.stream_ptr()
        ops._launch("rnnt_shortlist_rows", 0.0,
                    lambda: lib.sb_rnnt_shortlist_rows(lp.data_ptr(), V, None, B, T, U1, V,
                                                       int(blank), int(kp), 0, T, 0,
                                                       val.data_ptr(), idx.data_ptr(),
                                                       meta.data_ptr(), sp))
    return val, idx, meta


def _shortlist_search(sl, tl, ul, V, beam_size, blank):
    """One sb_rnnt_decode_static_shortlist launch over the shortlists sl of len(tl) utterances ->
    (label lists, log-probabilities, flag counts) on the host."""
    lib = _lib.load()
    val, idx, meta = sl
    B, T, U1, kp = val.shape
    dev = val.device
    lens = torch.tensor(list(tl) + list(ul), dtype=torch.int32).pin_memory().to(dev,
                                                                                non_blocking=True)
    nbytes = _lib.workspace_size(lib.sb_rnnt_decode_static_workspace_size, B, T, U1,
                                 int(beam_size))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    labels = torch.empty(B, U1, dtype=torch.int32, device=dev)
    counts = torch.empty(2, B, dtype=torch.int32, device=dev)      # lengths, flags
    scores = torch.empty(B, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        sp = _lib.stream_ptr()
        ops._launch("rnnt_decode_static", 0.0,
                    lambda: lib.sb_rnnt_decode_static_shortlist(
                        val.data_ptr(), idx.data_ptr(), meta.data_ptr(), kp, lens[:B].data_ptr(),
                        lens[B:].data_ptr(), B, T, U1, V, int(beam_size), int(blank),
                        labels.data_ptr(), counts[0].data_ptr(), scores.data_ptr(),
                        counts[1].data_ptr(), ws.data_ptr(), nbytes, sp))
    lab = labels.cpu()
    n, flags = counts.cpu().tolist()
    return [lab[b, :n[b]].tolist() for b in range(B)], scores.cpu().tolist(), flags


def decode_static_shortlist(produce, tlens, ulens, V, beam_size, blank):
    """Beam search over shortlists: produce(kp, rows) returns the shortlists (alloc_shortlists'
    layout) of the utterances `rows` (None: all of them) at kp entries per node.  Searches from
    kp = beam_size lists, then searches again every utterance the kernel flagged from
    SHORTLIST_RERUN-entry lists; an utterance flagged there too raises rather than return an
    unproven hypothesis.  tlens / ulens are already clamped to the lattice.
    Returns (list of label lists, list of log-probabilities)."""
    labels, scores, flags = _shortlist_search(produce(int(beam_size), None), tlens, ulens, V,
                                              beam_size, blank)
    rerun = [b for b, f in enumerate(flags) if f]
    if rerun:
        sl = produce(SHORTLIST_RERUN, rerun)
        lab2, sc2, fl2 = _shortlist_search(sl, [tlens[b] for b in rerun],
                                           [ulens[b] for b in rerun], V, beam_size, blank)
        if any(fl2):
            raise _lib.SpeechB200Error(
                "speech_b200: the shortlist beam search cannot order tied candidates of "
                "utterance(s) %s even from %d-entry lists" %
                ([b for b, f in zip(rerun, fl2) if f], SHORTLIST_RERUN))
        for j, b in enumerate(rerun):
            labels[b], scores[b] = lab2[j], sc2[j]
    return labels, scores


def decode_static_batch(lp, tlens, ulens, beam_size, blank):
    """lp (B, T, U1, V) float32 CUDA log-probabilities; tlens / ulens: frames and lattice rows
    (labels + 1) of every utterance.  Returns (list of label lists, list of log-probabilities)."""
    _lib.require_cuda(lp, "lp")
    lib = _lib.load()
    lp = lp.detach().float().contiguous()
    B, T, U1, V = lp.shape
    dev = lp.device
    tl = [min(int(t), T) for t in tlens]
    ul = [min(int(u), U1) for u in ulens]
    if not decode_static_fits(beam_size, V):
        def produce(kp, rows):
            return shortlists_of_lp(lp if rows is None else lp[rows].contiguous(), kp, blank)
        return decode_static_shortlist(produce, tl, ul, V, beam_size, blank)
    lens = torch.tensor(tl + ul, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
    nbytes = _lib.workspace_size(lib.sb_rnnt_decode_static_workspace_size, B, T, U1,
                                 int(beam_size))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    labels = torch.empty(B, U1, dtype=torch.int32, device=dev)
    olens = torch.empty(B, dtype=torch.int32, device=dev)
    scores = torch.empty(B, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        sp = _lib.stream_ptr()
        ops._launch("rnnt_decode_static", 0.0,
                    lambda: lib.sb_rnnt_decode_static(lp.data_ptr(), lens[:B].data_ptr(),
                                                      lens[B:].data_ptr(), B, T, U1, V,
                                                      int(beam_size), int(blank),
                                                      labels.data_ptr(), olens.data_ptr(),
                                                      scores.data_ptr(), ws.data_ptr(),
                                                      nbytes, sp))
    lab = labels.cpu()
    n = olens.cpu().tolist()
    sc = scores.cpu().tolist()
    return [lab[b, :n[b]].tolist() for b in range(B)], sc


def decode_static(lp, beam_size, blank=0):
    """One utterance: lp (T, U, V) log-probabilities (numpy array or tensor; copied to the GPU if
    it is not there already) -> (labels, log_probability)."""
    lp = torch.as_tensor(lp)
    if not lp.is_cuda:
        lp = lp.cuda()
    T, U, V = lp.shape
    labels, scores = decode_static_batch(lp.unsqueeze(0), [T], [U], beam_size, blank)
    return labels[0], scores[0]


# ------------------------------------------------------------------------------------------------
# Label-free search (csrc/rnnt_search.cu): decode_static's search with the row of hypothesis h at
# frame t computed from h itself.  A row provider supplies the rows; Transducer.recognize passes the
# prediction and joint networks (models/transducer_model.PredictionRows), tests pass a static
# lattice.  Its CPU restatement is oracle/rnnt_search_ref.py.  With an n-gram LM (shallow fusion)
# each level's acoustic rows become fused float64 rows or shortlists on the device
# (sb_rnnt_search_lm_rows) before the round reads them.
# ------------------------------------------------------------------------------------------------
class SearchSlots:
    """Device tensors of one search that a row provider reads: B, K, S, T, kp (None: full rows);
    par / sym / slot_lens (B, K) int32 (csrc/rnnt_search.cu), lp (B, K, V1) f32 or sl (the
    shortlists, alloc_shortlists(B, 1, K, kp)) that rows() fills: whichever is not None.
    With an LM (fused=True) rows() always fills the acoustic rows lp and sl is None; the search
    writes the fused float64 values itself, into flp (B, K, V1) f64 on the full route or fsl =
    (values (B, K, kp) f64, classes (B, K, kp) int32, {blank lp, next value} (B, K, 2) f64)."""

    def __init__(self, B, K, S, T, V1, kp, dev, fused=False):
        self.B, self.K, self.S, self.T, self.kp = B, K, S, T, kp
        self.par, self.sym, self.slot_lens = torch.zeros(3, B, K, dtype=torch.int32, device=dev)
        full = kp is None or fused
        self.lp = torch.empty(B, K, V1, dtype=torch.float32, device=dev) if full else None
        self.sl = None if full else alloc_shortlists(B, 1, K, kp, dev)
        self.flp = self.fsl = None
        if fused and kp is None:
            self.flp = torch.empty(B, K, V1, dtype=torch.float64, device=dev)
        elif fused:
            self.fsl = (torch.empty(B, K, kp, dtype=torch.float64, device=dev),
                        torch.empty(B, K, kp, dtype=torch.int32, device=dev),
                        torch.empty(B, K, 2, dtype=torch.float64, device=dev))


def _search_frame(lib, provider, slots, tl_dev, t, cur, max_len, blank, ws, nbytes, sp,
                  lm_args=()):
    """the launches of frame t: per level the provider's rows, the round (with an LM first the
    fused rows, lm_args = lm.fusion_args(...)) and the new frontier's states, then frame_end into
    block S + 1 - cur.  slots.T sizes the workspace, t < slots.T."""
    B, K, S, T, kp, V1 = slots.B, slots.K, slots.S, slots.T, slots.kp, provider.V1
    sl = slots.sl
    for level in range(S + 1):
        block = cur if level == 0 else level
        provider.rows(t, block, slots)
        if not lm_args:
            ops._launch("rnnt_search", 0.0, lambda: lib.sb_rnnt_search_round(
                _lib.ptr(slots.lp), *(_lib.ptr(a) for a in (sl or (None,) * 3)), kp or 0,
                tl_dev.data_ptr(), t, level, max_len, slots.par.data_ptr(),
                slots.sym.data_ptr(), slots.slot_lens.data_ptr(), B, T, S, V1, K, blank,
                ws.data_ptr(), nbytes, sp))
        else:
            fsl = tuple(_lib.ptr(a) for a in (slots.fsl or (None,) * 3))
            ops._launch("rnnt_search_lm_rows", 0.0, lambda: lib.sb_rnnt_search_lm_rows(
                slots.lp.data_ptr(), _lib.ptr(slots.flp), *fsl, kp or 0,
                tl_dev.data_ptr(), t, level, B, T, S, V1, K, blank, *lm_args, ws.data_ptr(),
                nbytes, sp))
            ops._launch("rnnt_search", 0.0, lambda: lib.sb_rnnt_search_round_lm(
                _lib.ptr(slots.flp), *fsl, kp or 0, tl_dev.data_ptr(), t, level,
                max_len, slots.par.data_ptr(), slots.sym.data_ptr(),
                slots.slot_lens.data_ptr(), B, T, S, V1, K, blank, ws.data_ptr(), nbytes,
                sp))
        if level < S:
            provider.extend(block, level + 1, slots)
    hid, layers, H, fy, Hj = provider.arenas()
    ops._launch("rnnt_search", 0.0, lambda: lib.sb_rnnt_search_frame_end(
        tl_dev.data_ptr(), t, slots.slot_lens.data_ptr(), _lib.ptr(hid), layers, H,
        _lib.ptr(fy), Hj, cur, S + 1 - cur, B, T, S, K, ws.data_ptr(), nbytes, sp))


def _search_once(provider, tl, T, K, S, max_len, L, blank, kp, fusion=None):
    """one search at list length kp (None: full rows); fusion: None or (NGramLM, lm_weight,
    insertion_bonus) -> (label lists, scores, flag counts)"""
    lib = _lib.load()
    B, V1, dev = provider.B, provider.V1, provider.device
    slots = SearchSlots(B, K, S, T, V1, kp, dev, fused=fusion is not None)
    lm_args = () if fusion is None else fusion_args(*fusion, dev)
    nbytes = _lib.workspace_size(lib.sb_rnnt_search_workspace_size, B, T, S, K)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    tl_dev = torch.tensor(tl, dtype=torch.int32).pin_memory().to(dev, non_blocking=True)
    # results: labels (B, L) | lengths (B) | flags (B) | scores (B) f64, one device->host copy
    n_int = B * (L + 2)
    n_int += n_int % 2
    out = torch.zeros(n_int + 2 * B, dtype=torch.int32, device=dev)
    labels, lens, flags = out[:B * L], out[B * L:B * L + B], out[B * L + B:B * L + 2 * B]
    scores = out[n_int:].view(torch.float64)
    with torch.cuda.device(dev):
        sp = _lib.stream_ptr()
        provider.begin(slots)
        ops._launch("rnnt_search", 0.0, lambda: lib.sb_rnnt_search_init(
            slots.slot_lens.data_ptr(), B, T, S, K, ws.data_ptr(), nbytes, sp))
        cur = 0
        for t in range(T):
            _search_frame(lib, provider, slots, tl_dev, t, cur, max_len, blank, ws, nbytes, sp,
                          lm_args)
            cur = S + 1 - cur
        ops._launch("rnnt_search", 0.0, lambda: lib.sb_rnnt_search_final(
            labels.data_ptr(), L, lens.data_ptr(), scores.data_ptr(), flags.data_ptr(), B, T, S,
            K, ws.data_ptr(), nbytes, sp))
    host = out.cpu()
    lab = host[:B * L].view(B, L)
    n = host[B * L:B * L + B].tolist()
    fl = host[B * L + B:B * L + 2 * B].tolist()
    sc = host[n_int:].view(torch.float64).tolist()
    return [lab[b, :n[b]].tolist() for b in range(B)], sc, fl


def search_batch(provider, tlens, beam_size, blank, max_symbols_per_frame, max_len=None, lm=None,
                 lm_weight=0.0, insertion_bonus=0.0):
    """Label-free beam search of a batch.  provider: B, T (frames available), V1, device, and
    begin(slots) (states of the empty hypothesis in block 0), rows(t, block, slots) (rows of the K
    frontier slots of `block` at frame t into slots.lp and / or slots.sl, whichever is not None;
    with an LM only slots.lp is given), extend(src, dst, slots) (states
    of the new frontier, slots.par / slots.sym, in block dst from block src), arenas() -> (hid,
    layers, H, fy, Hj) (None, 0, 0, None, 0 without states).  tlens: frames searched per utterance
    (clamped to T).  A frame emits at most max_symbols_per_frame labels; a hypothesis with max_len
    labels (default: frames * max_symbols_per_frame) is not extended.  Rows through shortlists
    where the full candidate list does not fit (decode_static_fits), with decode_static_shortlist's
    rerun of flagged utterances from SHORTLIST_RERUN-entry lists (the whole batch, so that every row
    is computed as in the first pass).
    lm (optional): a speech_b200.lm.NGramLM over the V1 classes with the search's blank and no end
    class, fused into every label extension as lp_k + (lm_weight * lm(k | h) + insertion_bonus);
    blank emissions keep lp_blank.  The fused values are the scores everywhere, the returned ones
    included; lm_weight = insertion_bonus = 0 gives the LM-less search's results bit for bit.
    Bad fusion arguments raise ValueError before any launch.
    Returns (list of label lists, list of float64 scores)."""
    from .models.ctc_decoder import check_lm
    B, T, V1 = provider.B, provider.T, provider.V1
    K, S = int(beam_size), int(max_symbols_per_frame)
    if K <= 0 or S <= 0:
        raise ValueError("beam_size and max_symbols_per_frame must be positive")
    check_lm(lm, lm_weight, insertion_bonus, V1, blank, search="Transducer")
    fusion = None if lm is None else (lm, lm_weight, insertion_bonus)
    tl = [max(0, min(int(t), T)) for t in tlens]
    if len(tl) != B:
        raise ValueError("tlens must have one entry per utterance")
    if T == 0:
        return [[] for _ in range(B)], [0.0] * B
    cap = T * S if max_len is None else min(int(max_len), T * S)
    L = max(1, cap)
    if decode_static_fits(K, V1):
        labels, scores, _ = _search_once(provider, tl, T, K, S, cap, L, blank, None, fusion)
        return labels, scores
    labels, scores, flags = _search_once(provider, tl, T, K, S, cap, L, blank, K, fusion)
    rerun = [b for b, f in enumerate(flags) if f]
    if rerun:
        lab2, sc2, fl2 = _search_once(provider, tl, T, K, S, cap, L, blank, SHORTLIST_RERUN,
                                      fusion)
        bad = [b for b in rerun if fl2[b]]
        if bad:
            raise _lib.SpeechB200Error(
                "speech_b200: the shortlist beam search cannot order tied candidates of "
                "utterance(s) %s even from %d-entry lists" % (bad, SHORTLIST_RERUN))
        for b in rerun:
            labels[b], scores[b] = lab2[b], sc2[b]
    return labels, scores


# ------------------------------------------------------------------------------------------------
# Streaming (streaming.TransducerStream): search_batch's loop resumed push by push.  The workspace
# is sized for T = max_frames and every launch passes that T; a push of counts[b] new frames per
# stream runs frames t = 0 .. max(counts) - 1 of the push with tlens = counts, so stream b takes
# its own frames and the kernels skip it after them.  The beam's prediction states sit in block
# `cur` of the arenas, which flips once per frame for the whole batch: after the push, a stream
# with an odd count has its beam in block S + 1, and settle_beams copies it to block 0, so that
# between pushes every stream's beam is in block 0.
# ------------------------------------------------------------------------------------------------
def check_stream_args(beam_size, max_symbols_per_frame, max_frames, max_len, V1, blank, lm,
                      lm_weight, insertion_bonus):
    """the stream search's ValueErrors, raised before any launch"""
    from .models.ctc_decoder import check_lm
    if not 1 <= int(beam_size) <= 32:
        raise ValueError("beam_size must lie in [1, 32], got %r" % (beam_size,))
    if int(max_symbols_per_frame) < 1:
        raise ValueError("max_symbols_per_frame must be >= 1, got %r" % (max_symbols_per_frame,))
    if int(max_frames) < 1:
        raise ValueError("max_frames must be >= 1, got %r" % (max_frames,))
    if max_len is not None and int(max_len) < 1:
        raise ValueError("max_len must be >= 1 or None, got %r" % (max_len,))
    check_lm(lm, lm_weight, insertion_bonus, V1, blank, search="Transducer")


def settle_beams(arenas, counts, K):
    """Block S + 1 rows -> block 0 rows of every stream with an odd count, one masked copy per
    arena.  arenas: tensors (S + 2, ..., B * K, width) or None; counts: (B,) frames of the push."""
    odd = (counts.to(torch.int64) % 2 == 1).repeat_interleave(K).view(-1, 1)
    for a in arenas:
        if a is not None:
            a[0].copy_(torch.where(odd.to(a.device), a[-1], a[0]))


class StreamSearch:
    """The label-free search of provider.B streams, resumed across pushes (see above).
    provider: as search_batch's (B, V1, device, begin, rows, extend, arenas; T is not read), with
    rows(t, block, slots) reading frame t of the current push.  Candidates go through the full rows
    where they fit (decode_static_fits) and otherwise through SHORTLIST_RERUN-entry lists from the
    first frame: a stream cannot rerun, and where those lists flag a selection the offline search
    would rerun and flag it too (csrc/tsearch.cuh), so best() raises for it instead.  max_len None:
    no cap beyond max_frames * max_symbols_per_frame, which never binds."""

    def __init__(self, provider, beam_size, max_symbols_per_frame, max_frames, blank, max_len=None,
                 lm=None, lm_weight=0.0, insertion_bonus=0.0):
        B, V1, dev = provider.B, provider.V1, provider.device
        check_stream_args(beam_size, max_symbols_per_frame, max_frames, max_len, V1, blank, lm,
                          lm_weight, insertion_bonus)
        lib = _lib.load()
        self.provider, self.B, self.blank, self.dev = provider, B, int(blank), dev
        self.K, self.S, self.Tm = K, S, Tm = (int(beam_size), int(max_symbols_per_frame),
                                              int(max_frames))
        self.max_len = Tm * S if max_len is None else min(int(max_len), Tm * S)
        self.kp = None if decode_static_fits(K, V1) else SHORTLIST_RERUN
        self.slots = SearchSlots(B, K, S, Tm, V1, self.kp, dev, fused=lm is not None)
        self.lm_args = fusion_args(lm, lm_weight, insertion_bonus, dev)
        self.nbytes = _lib.workspace_size(lib.sb_rnnt_search_workspace_size, B, Tm, S, K)
        self.ws = torch.empty(self.nbytes, dtype=torch.uint8, device=dev)
        self.frames = [0] * B
        with torch.cuda.device(dev):
            provider.begin(self.slots)
            self._reset(0, B)
        # the empty hypothesis's prediction state (the same in every row of block 0), for reset
        hid, _, _, fy, _ = provider.arenas()
        self.empty = [None if a is None else a[0].narrow(-2, 0, 1).clone() for a in (hid, fy)]

    def _reset(self, first, count):
        lib, s = _lib.load(), self.slots
        ops._launch("rnnt_search", 0.0, lambda: lib.sb_rnnt_search_reset(
            s.slot_lens.data_ptr(), self.B, self.Tm, self.S, self.K, first, count,
            self.ws.data_ptr(), self.nbytes, _lib.stream_ptr()))

    def reset(self, b):
        """stream b back to the empty hypothesis at frame 0; the others are untouched"""
        hid, _, _, fy, _ = self.provider.arenas()
        with torch.cuda.device(self.dev):
            self._reset(b, 1)
            for a, e in zip((hid, fy), self.empty):
                if a is not None:
                    a[0].narrow(-2, b * self.K, self.K).copy_(e.expand_as(
                        a[0].narrow(-2, 0, self.K)))
        self.frames[b] = 0

    def push(self, counts):
        """search counts[b] more frames of stream b (the provider's frames 0 .. counts[b] - 1)"""
        counts = [int(n) for n in counts]
        if len(counts) != self.B:
            raise ValueError("push takes one frame count per stream (%d), got %d"
                             % (self.B, len(counts)))
        if any(n < 0 or f + n > self.Tm for f, n in zip(self.frames, counts)):
            raise ValueError("a push would take a stream past max_frames = %d" % self.Tm)
        P = max(counts)
        if P == 0:
            return
        lib, S = _lib.load(), self.S
        tl_dev = torch.tensor(counts, dtype=torch.int32).pin_memory().to(self.dev,
                                                                          non_blocking=True)
        with torch.cuda.device(self.dev):
            sp = _lib.stream_ptr()
            cur = 0
            for t in range(P):
                _search_frame(lib, self.provider, self.slots, tl_dev, t, cur, self.max_len,
                              self.blank, self.ws, self.nbytes, sp, self.lm_args)
                cur = S + 1 - cur
            if any(n % 2 for n in counts):
                hid, _, _, fy, _ = self.provider.arenas()
                settle_beams((hid, fy), tl_dev, self.K)
        self.frames = [f + n for f, n in zip(self.frames, counts)]

    def best(self):
        """(label lists, float64 scores) of every stream's best hypothesis so far, one
        device->host copy; raises where the shortlists flagged a selection of a stream"""
        lib, B = _lib.load(), self.B
        L = max(1, min(self.max_len, max(self.frames) * self.S))
        n_int = B * (L + 2)
        n_int += n_int % 2
        out = torch.zeros(n_int + 2 * B, dtype=torch.int32, device=self.dev)
        labels, lens, flags = out[:B * L], out[B * L:B * L + B], out[B * L + B:B * L + 2 * B]
        scores = out[n_int:].view(torch.float64)
        with torch.cuda.device(self.dev):
            ops._launch("rnnt_search", 0.0, lambda: lib.sb_rnnt_search_final(
                labels.data_ptr(), L, lens.data_ptr(), scores.data_ptr(), flags.data_ptr(), B,
                self.Tm, self.S, self.K, self.ws.data_ptr(), self.nbytes, _lib.stream_ptr()))
        host = out.cpu()
        fl = host[B * L + B:B * L + 2 * B].tolist()
        bad = [b for b, f in enumerate(fl) if f]
        if bad:
            raise _lib.SpeechB200Error(
                "speech_b200: the shortlist beam search cannot order tied candidates of "
                "stream(s) %s even from %d-entry lists (reset them to go on)"
                % (bad, SHORTLIST_RERUN))
        lab = host[:B * L].view(B, L)
        n = host[B * L:B * L + B].tolist()
        sc = host[n_int:].view(torch.float64).tolist()
        return [lab[b, :n[b]].tolist() for b in range(B)], sc
