"""Backoff n-gram language models for shallow fusion: NGramLM over the model's own classes, for
the CTC prefix beam search, the attention model's beam search and the Transducer's label-free beam
search; WordLM over words spelled in a character model's classes, for the CTC prefix beam search
and the attention model's beam search (see WordLM).  Both read and write ARPA files and train
interpolated Kneser-Ney models through the same module functions.

The LM is over the acoustic model's own output classes (characters or subword units); the blank is
never an LM token.  Orders 1..10, with a sentence start <s>, an end </s> and optionally <unk>.
For the attention model, whose vocabulary has an end class and a start class, the end class is
the LM's </s> and the start class takes the blank's place (it is never predicted):
Values are held as the ARPA file's log10 numbers and converted once to natural log
(`v10 * math.log(10)`) for lookup, so `from_arpa(to_arpa(lm))` reproduces every float64 value.

    lm = NGramLM.from_arpa("chars.arpa", preproc.int_to_char)    # blank = last class
    lm = NGramLM.train(transcripts, order=5, num_classes=V + 1, blank=V)
    model.infer(batch, beam_size=8, lm=lm, lm_weight=0.8, insertion_bonus=1.5)

    lm = NGramLM.from_arpa("chars.arpa", preproc.int_to_char, blank=V - 1, end=V - 2)
    lm = NGramLM.train([preproc.encode(t) for t in texts], order=5, num_classes=V, blank=V - 1,
                       end=V - 2)
    s2s_model.recognize(inputs, beam_size=8, lm=lm, lm_weight=0.5, insertion_bonus=0.5)

The Transducer's classes are laid out as CTC's (labels 0..V-1, the blank V last, no end class), so
the same LM shape serves its label-free beam search:

    lm = NGramLM.from_arpa("chars.arpa", preproc.int_to_char)    # blank = last class
    lm = NGramLM.train(transcripts, order=5, num_classes=V + 1, blank=V)
    transducer.recognize(inputs, beam_size=8, lm=lm, lm_weight=0.5, insertion_bonus=1.0)

lm(s | h) follows ARPA backoff: h is the prefix's last order-1 symbols, preceded by <s> where the
prefix is shorter; when the n-gram (h, s) is stored its log-probability is used, otherwise the
backoff weight of h (0 when h is not stored) is added and the oldest context token dropped.
A class the LM does not know reads as <unk>.

Device tables (csrc/ngram.cuh, SbNgramLm in include/speech_b200.h): one open-addressed map with
two kinds of key, (context node, older token) -> context node and (context node, token) ->
n-gram, over a trie of contexts read most recent token first.  They are built once and cached
per device.
"""
import math
from collections import Counter, defaultdict
from collections.abc import Mapping

import numpy as np

LN10 = math.log(10.0)
MAX_ORDER = 10
BOS, EOS, UNK = "<s>", "</s>", "<unk>"
_HASH_MUL = 0x9E3779B97F4A7C15
_MASK64 = (1 << 64) - 1


def _finite(v, what):
    if not math.isfinite(v):
        raise ValueError("n-gram LM: non-finite value %r in %s" % (v, what))
    return v


def _check_order(order):
    if not isinstance(order, (int, np.integer)) or not 1 <= order <= MAX_ORDER:
        raise ValueError("n-gram LM: order must be in 1..%d, got %r" % (MAX_ORDER, order))
    return int(order)


def _class_names(symbols, blank, num_classes, end=None):
    """{class: symbol} of the classes but the blank and the end, validated"""
    names = {}
    seen = {BOS: None, EOS: None, UNK: None}
    for c in range(num_classes):
        if c == blank or c == end:
            continue
        s = symbols[c] if symbols is not None else str(c)
        if not isinstance(s, str) or s == "" or any(ch.isspace() for ch in s):
            raise ValueError("n-gram LM: symbol %r of class %d is empty or has whitespace" % (s, c))
        if s in seen:
            raise ValueError("n-gram LM: symbol %r of class %d is a duplicate or reserved" % (s, c))
        seen[s] = c
        names[c] = s
    return names


def _as_list(symbols):
    """symbols as a list indexed by class: a sequence, or a mapping class -> symbol (such as the
    reference Preprocessor.int_to_char) with keys 0 .. len - 1"""
    if isinstance(symbols, Mapping):
        try:
            return [symbols[c] for c in range(len(symbols))]
        except KeyError:
            raise ValueError("n-gram LM: a symbol mapping needs the keys 0 .. %d"
                             % (len(symbols) - 1)) from None
    return list(symbols)


def _layout(symbols, blank):
    """(num_classes, blank) of a symbol list: classes 0.. len(symbols) - 1, and the blank either
    one of them (its entry is ignored) or, by default, the class after the last (CTC's convention)"""
    symbols = _as_list(symbols)
    if blank is None:
        blank = len(symbols)
    if not 0 <= blank <= len(symbols):
        raise ValueError("n-gram LM: blank %r outside 0..%d" % (blank, len(symbols)))
    return (len(symbols) + 1 if blank == len(symbols) else len(symbols)), int(blank), symbols


def _check_end(end, blank, num_classes):
    """the end class (None: the LM has none), validated"""
    if end is None:
        return None
    if not isinstance(end, (int, np.integer)) or not 0 <= end < num_classes:
        raise ValueError("n-gram LM: end %r outside 0..%d" % (end, num_classes - 1))
    if end == blank:
        raise ValueError("n-gram LM: the end class %d is the blank" % end)
    return int(end)


# ------------------------------------------------------------------------------------------------
# ARPA files, Kneser-Ney training and the device tables, shared by NGramLM and WordLM.  An LM is
# held as ngrams[n] = {token tuple: (log10 prob, log10 backoff or None)}, n = 1..order.
# ------------------------------------------------------------------------------------------------
def _read_arpa(path, vocabulary):
    """(order, ngrams, dropped) of an ARPA file.  vocabulary(unigram words) -> {word: token} is
    called once the 1-gram section is read; n-grams with a word it does not map are dropped and
    counted."""
    with open(path, "r", encoding="utf-8") as fh:
        lines = [ln.strip() for ln in fh]
    lines = [ln for ln in lines if ln]
    try:
        i = lines.index("\\data\\")
    except ValueError:
        raise ValueError("n-gram LM: %s has no \\data\\ section" % path) from None
    i += 1
    counts = {}
    while i < len(lines) and lines[i].startswith("ngram "):
        key, _, val = lines[i][6:].partition("=")
        try:
            counts[int(key)] = int(val)
        except ValueError:
            raise ValueError("n-gram LM: bad count line %r" % lines[i]) from None
        i += 1
    if not counts:
        raise ValueError("n-gram LM: %s declares no n-gram counts" % path)
    order = max(counts)
    _check_order(order)
    if sorted(counts) != list(range(1, order + 1)) or any(v < 0 for v in counts.values()):
        raise ValueError("n-gram LM: counts must be given for orders 1..%d" % order)
    ngrams = {n: {} for n in range(1, order + 1)}
    dropped = 0
    word_tok = None
    for n in range(1, order + 1):
        header = "\\%d-grams:" % n
        if i >= len(lines) or lines[i] != header:
            raise ValueError("n-gram LM: missing section %s" % header)
        i += 1
        section = []
        for _ in range(counts[n]):
            if i >= len(lines) or lines[i].startswith("\\"):
                raise ValueError("n-gram LM: section %s has fewer than %d entries"
                                 % (header, counts[n]))
            f = lines[i].split()
            i += 1
            if len(f) not in (n + 1, n + 2):
                raise ValueError("n-gram LM: malformed %d-gram line %r" % (n, " ".join(f)))
            try:
                p = float(f[0])
                b = float(f[n + 1]) if len(f) == n + 2 else None
            except ValueError:
                raise ValueError("n-gram LM: malformed number in %r" % " ".join(f)) from None
            _finite(p, "a %d-gram probability" % n)
            if b is not None:
                _finite(b, "a %d-gram backoff" % n)
            section.append((f[1:n + 1], p, b))
        if word_tok is None:
            word_tok = vocabulary([words[0] for words, _, _ in section])
        for words, p, b in section:
            if any(w not in word_tok for w in words):
                dropped += 1
                continue
            g = tuple(word_tok[w] for w in words)
            if g in ngrams[n]:
                raise ValueError("n-gram LM: duplicate %d-gram %r" % (n, " ".join(words)))
            ngrams[n][g] = (p, b)
    if i >= len(lines) or lines[i] != "\\end\\":
        raise ValueError("n-gram LM: %s: expected \\end\\ after the %d-grams (wrong counts?)"
                         % (path, order))
    return order, ngrams, dropped


def _write_arpa(path, order, ngrams, names):
    """ARPA file of ngrams, names[token] the word of each token; values written with repr, which
    reads back to the same float64"""
    out = ["", "\\data\\"]
    out += ["ngram %d=%d" % (n, len(ngrams[n])) for n in range(1, order + 1)]
    for n in range(1, order + 1):
        out += ["", "\\%d-grams:" % n]
        for g, (p, b) in sorted(ngrams[n].items()):
            line = "%r\t%s" % (p, " ".join(names[t] for t in g))
            out.append(line if b is None else "%s\t%r" % (line, b))
    out += ["", "\\end\\", ""]
    with open(path, "w", encoding="utf-8") as fh:
        fh.write("\n".join(out))


def _kneser_ney(sequences, order, vocab, bos, eos):
    """Interpolated Kneser-Ney in backoff form over token sequences (each read as <s> w1 .. wn
    </s>); vocab: the tokens the unigram level spreads its uniform share over (</s> included)."""
    raw = {n: Counter() for n in range(1, order + 1)}
    for seq in sequences:
        w = [bos] + list(seq) + [eos]
        for n in range(1, order + 1):
            for j in range(len(w) - n + 1):
                raw[n][tuple(w[j:j + n])] += 1
    raw[1].pop((bos,), None)                            # <s> is never predicted
    # KN counts: raw at the top order and for n-grams that begin with <s>, else the number of
    # distinct tokens seen before the n-gram
    kn = {order: raw[order]}
    for n in range(order - 1, 0, -1):
        left = Counter(g[1:] for g in raw[n + 1])
        kn[n] = {g: (c if g[0] == bos else left[g]) for g, c in raw[n].items()}
    disc, denom, types = {}, {}, {}
    for n in range(1, order + 1):
        n1 = sum(1 for c in kn[n].values() if c == 1)
        n2 = sum(1 for c in kn[n].values() if c == 2)
        d = n1 / (n1 + 2 * n2) if n1 + 2 * n2 else 0.0
        disc[n] = d if 0.0 < d < 1.0 else 0.5
        den, typ = defaultdict(int), defaultdict(int)
        for g, c in kn[n].items():
            den[g[:-1]] += c
            typ[g[:-1]] += 1
        denom[n], types[n] = den, typ

    def gamma(n, h):
        return disc[n] * types[n][h] / denom[n][h]

    memo = {}

    def prob(h, w):
        """P_n(w | h), n = len(h) + 1"""
        key = (h, w)
        if key in memo:
            return memo[key]
        n = len(h) + 1
        lower = prob(h[1:], w) if n > 1 else 1.0 / len(vocab)
        den = denom[n].get(h, 0)
        if den == 0:
            v = lower
        else:
            c = kn[n].get(h + (w,), 0)
            v = max(c - disc[n], 0.0) / den + gamma(n, h) * lower
        memo[key] = v
        return v

    ngrams = {n: {} for n in range(1, order + 1)}
    for w in vocab:
        ngrams[1][(w,)] = (math.log10(prob((), w)), None)
    ngrams[1][(bos,)] = (-99.0, None)
    for n in range(2, order + 1):
        for g in kn[n]:
            ngrams[n][g] = (math.log10(prob(g[:-1], g[-1])), None)
    for n in range(1, order):
        for h in denom[n + 1]:
            p, _ = ngrams[n][h]
            ngrams[n][h] = (p, math.log10(gamma(n + 1, h)))
    return ngrams


def _pack_map(entries):
    """(keys, vals, cap) of the open-addressed map of include/speech_b200.h over (key, value)
    pairs, inserted in order with linear probing"""
    cap = 64
    while cap < 2 * len(entries):
        cap <<= 1
    keys = [0] * cap
    vals = [-1] * cap
    mask = cap - 1
    for k, v in entries:
        h = ((k * _HASH_MUL) & _MASK64) >> 32 & mask
        while keys[h] != 0:
            h = (h + 1) & mask
        keys[h] = k
        vals[h] = v
    return np.array(keys, np.uint64), np.array(vals, np.int32), cap


def _map_key(node, tok, kind):
    return (node << 32) | ((tok + 1) << 1) | kind


def _backoff_tables(order, ngrams, bos, eos, with_eos):
    """The n-gram tables of SbNgramLm but tok: keys, vals, logp, bow, cap, order, bos, lm_upper,
    lm_abs.  with_eos: the n-grams that predict </s> are stored (a search scores it)."""
    ctx = {(): 0}
    entries = []                       # (key, value)
    bow = [0.0]

    def ctx_node(h):
        """node of context h (oldest .. newest), created with backoff 0 when missing"""
        if h in ctx:
            return ctx[h]
        parent = ctx_node(h[1:])
        nid = len(bow)
        ctx[h] = nid
        bow.append(0.0)
        entries.append((_map_key(parent, h[0], 0), nid))
        return nid

    def usable(g):
        # contexts: <s> only as the oldest token, never </s>
        return all(t != eos for t in g) and all(t != bos for t in g[1:])

    logp = []
    upper_p, abs_p = -math.inf, 0.0
    upper_b = [0.0] * (order + 1)
    abs_b = [0.0] * (order + 1)
    for n in range(1, order + 1):
        for g, (p10, b10) in sorted(ngrams[n].items()):
            p = p10 * LN10
            if b10 is not None and n < order:
                b = b10 * LN10
                upper_b[n] = max(upper_b[n], b)
                abs_b[n] = max(abs_b[n], abs(b))
                if usable(g):
                    bow[ctx_node(g)] = b
            if g[-1] == bos or (g[-1] == eos and not with_eos) or not usable(g[:-1]):
                continue                # never looked up
            upper_p, abs_p = max(upper_p, p), max(abs_p, abs(p))
            entries.append((_map_key(ctx_node(g[:-1]), g[-1], 1), len(logp)))
            logp.append(p)
    keys, vals, cap = _pack_map(entries)
    return {
        "keys": keys, "vals": vals, "logp": np.array(logp or [0.0], np.float64),
        "bow": np.array(bow, np.float64), "cap": cap, "order": order, "bos": bos,
        "lm_upper": upper_p + sum(upper_b), "lm_abs": abs_p + sum(abs_b),
    }


def _device(device):
    import torch
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    return device


def _to_device(h, names, device):
    import torch
    return {k: torch.from_numpy(h[k].view(np.int64) if h[k].dtype == np.uint64 else h[k])
            .to(device) for k in names}


class NGramLM:
    """Backoff n-gram LM over class ids.  Tokens: class c -> c, <s> -> C, </s> -> C + 1,
    <unk> -> C + 2 (C = num_classes); the end class, where there is one, -> </s>.  Build with
    from_arpa or train."""

    def __init__(self, order, num_classes, blank, ngrams, end=None):
        # ngrams[n]: {token tuple: (log10 prob, log10 backoff or None)}, n = 1..order
        self._order = order
        self._num_classes = num_classes
        self._blank = blank
        self._end = _check_end(end, blank, num_classes)
        self._ngrams = ngrams
        self._bos, self._eos, self._unk = num_classes, num_classes + 1, num_classes + 2
        uni = ngrams[1]
        tok = np.full(num_classes, -1, np.int32)
        for c in range(num_classes):
            if c == blank:
                continue
            if c == self._end:
                if (self._eos,) not in uni:
                    raise ValueError("n-gram LM: the end class %d needs a %s unigram" % (c, EOS))
                tok[c] = self._eos
            elif (c,) in uni:
                tok[c] = c
            elif (self._unk,) in uni:
                tok[c] = self._unk
            else:
                raise ValueError("n-gram LM: class %d is not in the LM and it has no %s" % (c, UNK))
        self._tok = tok
        self._host = None
        self._dev = {}

    @property
    def order(self):
        return self._order

    @property
    def num_classes(self):
        return self._num_classes

    @property
    def blank(self):
        return self._blank

    @property
    def end(self):
        """the class read as </s> (the attention model's END), or None"""
        return self._end

    # ------------------------------------------------------------------------------------------
    # ARPA
    # ------------------------------------------------------------------------------------------
    @classmethod
    def from_arpa(cls, path, symbols, blank=None, end=None):
        """Read an ARPA file.  symbols[c] is the token string of class c (e.g. the reference
        Preprocessor.int_to_char in id order); blank defaults to the class after the last symbol.
        end (optional): the class that is the LM's </s>; its symbol, like the blank's, is ignored.
        n-grams over words that are neither a class symbol nor <s>, </s>, <unk> are dropped."""
        num_classes, blank, symbols = _layout(symbols, blank)
        end = _check_end(end, blank, num_classes)
        names = _class_names(symbols, blank, num_classes, end)
        word_tok = {s: c for c, s in names.items()}
        word_tok.update({BOS: num_classes, EOS: num_classes + 1, UNK: num_classes + 2})
        order, ngrams, _ = _read_arpa(path, lambda unigram_words: word_tok)
        return cls(order, num_classes, blank, ngrams, end)

    def to_arpa(self, path, symbols=None):
        """Write an ARPA file; str(c) names class c unless symbols are given (same layout as
        from_arpa).  Values are written with repr, which reads back to the same float64."""
        if symbols is not None:
            symbols = _as_list(symbols)
        if symbols is not None and len(symbols) < self._num_classes - (
                self._blank == self._num_classes - 1):
            raise ValueError("n-gram LM: symbols do not cover the LM's classes")
        names = _class_names(symbols, self._blank, self._num_classes, self._end)
        names.update({self._bos: BOS, self._eos: EOS, self._unk: UNK})
        _write_arpa(path, self._order, self._ngrams, names)

    # ------------------------------------------------------------------------------------------
    # training: interpolated Kneser-Ney in backoff form
    # ------------------------------------------------------------------------------------------
    @classmethod
    def train(cls, sequences, order, num_classes, blank, end=None):
        """Interpolated Kneser-Ney over label-id sequences (each read as <s> w1 .. wn </s>).
        With an end class, one leading blank and one trailing end are stripped from each sequence
        where present (so Preprocessor.encode outputs, START .. END, go straight in); a blank or
        an end anywhere else is an error.

        One discount per order, D = n1 / (n1 + 2 n2) (0.5 where that is undefined or outside
        (0, 1)); lower orders use continuation counts, except n-grams that begin with <s>, which
        keep raw counts; the unigram level is interpolated with the uniform distribution over the
        classes (but the blank and the end) and </s>.  Each seen n-gram stores its full interpolated probability and each
        context its interpolation mass, which makes the backoff form the interpolated model."""
        order = _check_order(order)
        C = int(num_classes)
        if C < 2 or not 0 <= blank < C:
            raise ValueError("n-gram LM: need num_classes >= 2 and 0 <= blank < num_classes")
        end = _check_end(end, blank, C)
        bos, eos = C, C + 1
        seqs = []
        for seq in sequences:
            seq = [int(v) for v in seq]
            if end is not None:
                seq = seq[1:] if seq and seq[0] == blank else seq
                seq = seq[:-1] if seq and seq[-1] == end else seq
            if any(v < 0 or v >= C or v == blank or v == end for v in seq):
                raise ValueError("n-gram LM: a training label is out of range, the blank or "
                                 "the end")
            seqs.append(seq)
        vocab = [c for c in range(C) if c != blank and c != end] + [eos]
        ngrams = _kneser_ney(seqs, order, vocab, bos, eos)
        return cls(order, C, blank, ngrams, end)

    # ------------------------------------------------------------------------------------------
    # device tables
    # ------------------------------------------------------------------------------------------
    def host_tables(self):
        """The tables of SbNgramLm as numpy arrays (built once): keys (uint64), vals (int32),
        logp and bow (float64, natural log), tok (int32), and the scalars cap, order, bos,
        lm_upper, lm_abs.  See include/speech_b200.h for the map's keys and hash.  With an end
        class the n-grams that predict </s> are stored too (the attention search scores it)."""
        if self._host is not None:
            return self._host
        self._host = _backoff_tables(self._order, self._ngrams, self._bos, self._eos,
                                     self._end is not None)
        self._host["tok"] = self._tok.copy()
        return self._host

    def device_tables(self, device):
        """(SbNgramLm ctypes struct, tensors it points into) on `device`, built once per device"""
        from . import _lib
        device = _device(device)
        if device not in self._dev:
            h = self.host_tables()
            t = _to_device(h, ("keys", "vals", "logp", "bow", "tok"), device)
            st = _lib.SbNgramLm(t["keys"].data_ptr(), t["vals"].data_ptr(), t["logp"].data_ptr(),
                                t["bow"].data_ptr(), t["tok"].data_ptr(), h["cap"], h["order"],
                                self._num_classes, h["bos"], self._blank, h["lm_upper"],
                                h["lm_abs"])
            self._dev[device] = (st, t)
        return self._dev[device]

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_dev"] = {}
        return d

    def __setstate__(self, d):
        d.setdefault("_end", None)          # pickled before LMs had an end class
        self.__dict__.update(d)


class WordLM:
    """Backoff word n-gram LM for the CTC prefix beam search or the attention beam search of a
    character model (Hannun et al. 2014, arXiv:1408.2873): a word is scored when the delimiter
    class (the space) that ends it is emitted, and a lexicon of the LM's words, spelled in the
    model's classes, tracks the partial word.  Word tokens: the spellable words 0..W-1 in sorted
    order, <s> W, </s> W + 1, <unk> W + 2.
    Build with from_arpa or train; the search semantics are in include/speech_b200.h (SbWordLm).

        wlm = WordLM.from_arpa("3-gram.arpa", preproc.int_to_char)     # delimiter " ", blank last
        model.infer(batch, beam_size=32, lm=wlm, lm_weight=0.8, insertion_bonus=1.0)

    The attention model's layout has START as the blank and an end class END, scored with the
    trailing word and </s> where a hypothesis ends (include/speech_b200.h, the s2s word-LM entry
    points); the CTC search refuses an LM with an end class:

        wlm = WordLM.from_arpa("3-gram.arpa", preproc.int_to_char, blank=V - 1, end=V - 2)
        s2s_model.recognize(inputs, beam_size=10, lm=wlm, lm_weight=0.8, insertion_bonus=1.0)

    A class whose symbol is one character spells that character; the delimiter's and the blank's
    symbols spell nothing.  oov_penalty (<= 0, settable) is added once per word that leaves the
    lexicon: 0 scores such words as <unk>, -inf keeps the search to the lexicon.  An LM without an
    <unk> unigram needs oov_penalty = -inf."""

    def __init__(self, order, words, ngrams, symbols, num_classes, blank, delimiter, oov_penalty,
                 dropped=0, end=None):
        self._order = order
        self._words = list(words)
        self._ngrams = ngrams
        self._num_classes, self._blank, self._delim = num_classes, blank, delimiter
        self._end = _check_end(end, blank, num_classes)
        if self._end is not None and self._end == delimiter:
            raise ValueError("word LM: the end class %d is the delimiter" % end)
        self._symbols = list(symbols)
        W = len(self._words)
        self._bos, self._eos, self._unk = W, W + 1, W + 2
        if (self._eos,) not in ngrams[1]:
            raise ValueError("word LM: the LM has no %s unigram" % EOS)
        self._dropped = int(dropped)
        chars = _spelling(self._symbols, blank, delimiter, self._end)
        self._spell = [tuple(chars[ch] for ch in w) for w in self._words]
        self._oov = None
        self.oov_penalty = oov_penalty
        self._host = None
        self._dev = {}

    @property
    def order(self):
        return self._order

    @property
    def num_classes(self):
        return self._num_classes

    @property
    def blank(self):
        return self._blank

    @property
    def end(self):
        """the class that ends a hypothesis (the attention model's END), scored with </s> and the
        trailing word, or None (the CTC search, which has no end class)"""
        return self._end

    @property
    def delimiter(self):
        """the class that ends a word"""
        return self._delim

    @property
    def num_words(self):
        return len(self._words)

    @property
    def words(self):
        """the lexicon, word token w at index w"""
        return list(self._words)

    @property
    def dropped(self):
        """n-grams from_arpa left out because a word in them cannot be spelled"""
        return self._dropped

    @property
    def has_unk(self):
        return (self._unk,) in self._ngrams[1]

    @property
    def oov_penalty(self):
        return self._oov

    @oov_penalty.setter
    def oov_penalty(self, v):
        v = float(v)
        if math.isnan(v) or v > 0.0:
            raise ValueError("word LM: oov_penalty must be <= 0, got %r" % (v,))
        if v != -math.inf and not self.has_unk:
            raise ValueError("word LM: the LM has no %s unigram, so out-of-vocabulary words "
                             "need oov_penalty = -inf, got %r" % (UNK, v))
        self._oov = v

    def spell(self, word):
        """the classes of a word, or None where a character has no class"""
        chars = _spelling(self._symbols, self._blank, self._delim, self._end)
        if word == "" or any(ch not in chars for ch in word):
            return None
        return tuple(chars[ch] for ch in word)

    # ------------------------------------------------------------------------------------------
    # ARPA and training
    # ------------------------------------------------------------------------------------------
    @classmethod
    def from_arpa(cls, path, symbols, delimiter=" ", blank=None, oov_penalty=0.0, end=None):
        """Read an ARPA word LM.  symbols[c] is the string of class c (e.g. the reference
        Preprocessor.int_to_char), blank defaults to the class after the last symbol, delimiter is
        the symbol of the word boundary.  The lexicon is every unigram word spelled character by
        character through the classes; n-grams with a word that cannot be spelled are dropped
        (counted in `dropped`).  ValueError if no word can be spelled (such as an upper-case LM
        against lower-case symbols).  end (optional): the class that ends a hypothesis, for the
        attention model (blank=V - 1, end=V - 2); it spells nothing."""
        num_classes, blank, symbols = _layout(symbols, blank)
        end = _check_end(end, blank, num_classes)
        delim = _delimiter_class(symbols, blank, delimiter, end)
        chars = _spelling(symbols, blank, delim, end)
        vocab = []

        def vocabulary(unigram_words):
            reserved = (BOS, EOS, UNK)
            ws = sorted({w for w in unigram_words if w not in reserved and
                         all(ch in chars for ch in w)})
            if not ws:
                raise ValueError("word LM: no word of %s can be spelled with the classes %r "
                                 "(a case mismatch?)" % (path, sorted(chars)))
            vocab.extend(ws)
            tok = {w: t for t, w in enumerate(ws)}
            tok.update({BOS: len(ws), EOS: len(ws) + 1, UNK: len(ws) + 2})
            return tok

        order, ngrams, dropped = _read_arpa(path, vocabulary)
        return cls(order, vocab, ngrams, symbols, num_classes, blank, delim, oov_penalty, dropped,
                   end)

    def to_arpa(self, path):
        """Write an ARPA file that from_arpa reads back to the same LM"""
        names = self._words + [BOS, EOS, UNK]
        _write_arpa(path, self._order, self._ngrams, names)

    @classmethod
    def train(cls, texts, order, symbols, delimiter=" ", blank=None, oov_penalty=0.0, end=None):
        """Interpolated Kneser-Ney (as NGramLM.train) over the whitespace-split words of each text,
        read as <s> w1 .. wn </s>.  The lexicon is the texts' spellable words; a word that cannot
        be spelled is read as <unk>, and the unigram level spreads its uniform share over the
        words, </s> and <unk>, so <unk> always has a unigram.  end: as in from_arpa."""
        order = _check_order(order)
        num_classes, blank, symbols = _layout(symbols, blank)
        end = _check_end(end, blank, num_classes)
        delim = _delimiter_class(symbols, blank, delimiter, end)
        chars = _spelling(symbols, blank, delim, end)
        texts = [t.split() for t in texts]
        words = sorted({w for t in texts for w in t if all(ch in chars for ch in w)})
        if not words:
            raise ValueError("word LM: no training word can be spelled with the classes %r"
                             % sorted(chars))
        W = len(words)
        tok = {w: t for t, w in enumerate(words)}
        seqs = [[tok.get(w, W + 2) for w in t] for t in texts]
        ngrams = _kneser_ney(seqs, order, list(range(W)) + [W + 1, W + 2], W, W + 1)
        return cls(order, words, ngrams, symbols, num_classes, blank, delim, oov_penalty, end=end)

    # ------------------------------------------------------------------------------------------
    # device tables
    # ------------------------------------------------------------------------------------------
    def host_tables(self):
        """The tables of SbWordLm as numpy arrays (built once): the word n-gram's keys, vals,
        logp, bow and tok (the identity over the W + 3 tokens) with its scalars, as
        NGramLM.host_tables; the lexicon map lex_keys (uint64) / lex_vals (int32) of
        (node, class) -> child node and lex_word (int32, the word token of each node, -1 where
        none ends there), node 0 the empty word; lex_cap, and the counts."""
        if self._host is not None:
            return self._host
        W = len(self._words)
        h = _backoff_tables(self._order, self._ngrams, self._bos, self._eos, True)
        h["tok"] = np.arange(W + 3, dtype=np.int32)
        child = {}
        lex_word = [-1]
        entries = []
        for w, spelling in enumerate(self._spell):
            node = 0
            for c in spelling:
                nxt = child.get((node, c))
                if nxt is None:
                    nxt = child[(node, c)] = len(lex_word)
                    lex_word.append(-1)
                    entries.append((_map_key(node, c, 0), nxt))
                node = nxt
            lex_word[node] = w
        h["lex_keys"], h["lex_vals"], h["lex_cap"] = _pack_map(entries)
        h["lex_word"] = np.array(lex_word, np.int32)
        self._host = h
        return h

    def device_tables(self, device):
        """(SbWordLm ctypes struct, tensors it points into) on `device`, built once per device"""
        from . import _lib
        device = _device(device)
        if device not in self._dev:
            h = self.host_tables()
            t = _to_device(h, ("keys", "vals", "logp", "bow", "tok", "lex_keys", "lex_vals",
                               "lex_word"), device)
            ng = _lib.SbNgramLm(t["keys"].data_ptr(), t["vals"].data_ptr(), t["logp"].data_ptr(),
                                t["bow"].data_ptr(), t["tok"].data_ptr(), h["cap"], h["order"],
                                len(self._words) + 3, h["bos"], -1, h["lm_upper"], h["lm_abs"])
            st = _lib.SbWordLm(ng, t["lex_keys"].data_ptr(), t["lex_vals"].data_ptr(),
                               t["lex_word"].data_ptr(), h["lex_cap"], len(self._words),
                               int(self.has_unk), self._num_classes, self._blank, self._delim)
            self._dev[device] = (st, t)
        return self._dev[device]

    def __getstate__(self):
        d = dict(self.__dict__)
        d["_dev"] = {}
        return d

    def __setstate__(self, d):
        d.setdefault("_end", None)          # pickled before word LMs had an end class
        self.__dict__.update(d)


def fusion_kind(lm):
    """None, NGramLM or WordLM: the key of each search's table of entry points"""
    return None if lm is None else WordLM if isinstance(lm, WordLM) else NGramLM


def fusion_args(lm, lm_weight, insertion_bonus, device):
    """The C arguments of shallow fusion with `lm` on `device`, as every fused entry point takes
    them: () without an LM, (SbNgramLm, lm_weight, insertion_bonus) for an NGramLM and
    (SbWordLm, lm_weight, insertion_bonus, oov_penalty) for a WordLM.  The tables are built once
    per device; oov_penalty is read at each call, since it is settable."""
    if lm is None:
        return ()
    tables, _ = lm.device_tables(device)
    args = (tables, float(lm_weight), float(insertion_bonus))
    return args + (float(lm.oov_penalty),) if isinstance(lm, WordLM) else args


def _delimiter_class(symbols, blank, delimiter, end=None):
    """the one class but the blank and the end whose symbol is `delimiter`"""
    cs = [c for c, s in enumerate(symbols) if c != blank and c != end and s == delimiter]
    if len(cs) != 1:
        raise ValueError("word LM: %d classes have the delimiter symbol %r (need exactly one)"
                         % (len(cs), delimiter))
    return cs[0]


def _spelling(symbols, blank, delim, end=None):
    """{character: class} of the one-character symbols but the blank's, the delimiter's and the
    end class's"""
    chars = {}
    for c, s in enumerate(symbols):
        if c == blank or c == delim or c == end:
            continue
        if not isinstance(s, str) or s == "":
            raise ValueError("word LM: symbol %r of class %d is not a string" % (s, c))
        if len(s) == 1:
            if s in chars or s.isspace():
                raise ValueError("word LM: symbol %r of class %d is a duplicate or whitespace"
                                 % (s, c))
            chars[s] = c
    return chars
