"""ARPA n-gram language model for beam search (row N6): the parse, the vocabulary trie and the device tables.

The parse and the trie are numpy (they run, and are tested, without a GPU); the device tables are built by
`ds2_lm_build` lazily, once per device, at the first decode.  Rules L0-L2 of csrc/beam_decode.cu define what is
accepted and what the tables mean; everything refused raises `Ds2Error` with "language-model scoring" in the message.

The parse is vectorised over the file's bytes: token boundaries and line numbers come from numpy over the byte array,
the tokens from one `bytes.split()`, word ids from one `map` over a dict, so loading a LibriSpeech-pruned-3-gram-sized
file costs seconds rather than a Python statement per n-gram."""
import gc
import gzip
import os
import re
from dataclasses import dataclass, field
from typing import Dict, List

import numpy as np

from ._lib import Ds2Error

MAX_ORDER = 5
MAX_WORDS = 1 << 24
SPECIAL = (b"<s>", b"</s>", b"<unk>")


def _refuse(msg):
    raise Ds2Error(f"BeamCTCDecoder: language-model scoring: {msg}")


@dataclass
class ArpaModel:
    """order N; words[i] = the i-th unigram (bytes); per order n (index n-1): ids (count, n) int32 oldest first,
    logp / backoff (count,) float32 log10 values (an unwritten backoff is 0)"""
    order: int
    words: List[bytes]
    ids: List[np.ndarray]
    logp: List[np.ndarray]
    backoff: List[np.ndarray]
    index: Dict[bytes, int] = field(repr=False, default_factory=dict)


def _read_bytes(path):
    if not path or not os.path.isfile(path):
        _refuse(f"{path!r} not found")
    with open(path, "rb") as f:
        raw = f.read()
    if raw[:2] == b"\x1f\x8b":
        try:
            raw = gzip.decompress(raw)
        except (OSError, EOFError) as e:
            _refuse(f"{path!r}: corrupt gzip stream ({e})")
    if not raw.lstrip().startswith(b"\\data\\"):
        _refuse(f"{path!r} is not an ARPA file (it does not start with \\data\\; KenLM binary models are not "
                "supported, build one from the ARPA text)")
    return raw


def _section_fields(sec: bytes):
    """tokens of a section and the number of tokens on each non-empty line, from the bytes"""
    b = np.frombuffer(sec, np.uint8)
    sep = (b == 32) | (b == 9) | (b == 10) | (b == 13) | (b == 11) | (b == 12)
    start = np.flatnonzero(~sep & np.concatenate([[True], sep[:-1]]))
    line = np.searchsorted(np.flatnonzero(b == 10), start)
    per_line = np.bincount(line)
    return sec.split(), per_line[per_line > 0]


def _has_duplicate_rows(g: np.ndarray) -> bool:
    """exact: rows whose 64-bit mix collides are compared in full"""
    h = np.zeros(len(g), np.uint64)
    with np.errstate(over="ignore"):
        for k in range(g.shape[1]):
            h = (h ^ g[:, k].astype(np.uint64)) * np.uint64(0x9E3779B97F4A7C15)
            h ^= h >> np.uint64(29)
    o = np.argsort(h, kind="stable")
    same = np.flatnonzero(h[o][1:] == h[o][:-1])
    if len(same) == 0:
        return False
    cand = np.unique(np.concatenate([o[same], o[same + 1]]))
    rows = g[cand]
    return len(np.unique(rows, axis=0)) != len(rows)


def _floats(tok) -> np.ndarray:
    """decimal strings (bytes) -> fp32, through the correctly rounded fp64 value"""
    return np.asarray(tok.tolist(), dtype="S").astype(np.float64).astype(np.float32)


def read_arpa(path) -> ArpaModel:
    """parse an ARPA file (rule L0); the millions of short-lived token objects are made with the cyclic garbage
    collector paused, which otherwise rescans them many times over"""
    enabled = gc.isenabled()
    gc.disable()
    try:
        return _read_arpa(path)
    finally:
        if enabled:
            gc.enable()


def _read_arpa(path) -> ArpaModel:
    raw = _read_bytes(path)
    heads, n, at = [], 1, 0
    while True:                                  # section markers "\\n-grams:" at line starts, in order
        k = raw.find(b"\\%d-grams:" % n, at)
        if k < 0:
            break
        heads.append((k, raw.find(b"\n", k) + 1 or len(raw)))
        at, n = heads[-1][1], n + 1
    end = raw.rfind(b"\\end\\")
    end = None if end < 0 or (heads and end < heads[-1][1]) else end
    if not heads or end is None:
        _refuse(f"{path!r}: no n-gram sections or no \\end\\ marker")
    header = raw[:heads[0][0]]
    counts = {int(n): int(c) for n, c in re.findall(rb"^[ \t]*ngram[ \t]+(\d+)[ \t]*=[ \t]*(\d+)", header, re.M)}
    N = max(counts) if counts else 0
    if N < 1 or sorted(counts) != list(range(1, N + 1)):
        _refuse(f"{path!r}: bad \\data\\ header {counts}")
    if N > MAX_ORDER:
        _refuse(f"{path!r}: order {N} > {MAX_ORDER}")
    if counts[1] >= MAX_WORDS:
        _refuse(f"{path!r}: {counts[1]} words, at most {MAX_WORDS - 1} are supported")
    if len(heads) != N or b"\\%d-grams:" % (N + 1) in raw[heads[-1][1]:]:
        _refuse(f"{path!r}: {len(heads)} n-gram sections, the \\data\\ header's order is {N}")
    bounds = [h[1] for h in heads]
    stops = [h[0] for h in heads[1:]] + [end]
    words, index = None, None
    ids, logp, backoff = [], [], []
    for n in range(1, N + 1):
        tok, nf = _section_fields(raw[bounds[n - 1]:stops[n - 1]])
        if len(nf) != counts[n]:
            _refuse(f"{path!r}: {len(nf)} {n}-grams, the \\data\\ header says {counts[n]}")
        if np.any((nf != n + 1) & (nf != n + 2)):
            _refuse(f"{path!r}: a {n}-gram line without {n + 1} or {n + 2} fields")
        at = np.concatenate([[0], np.cumsum(nf)[:-1]]).astype(np.int64)
        tok = np.array(tok, dtype=object)
        try:
            lp = _floats(tok[at])
            bo = np.zeros(len(nf), np.float32)
            has = nf == n + 2
            bo[has] = _floats(tok[at[has] + n + 1])
        except ValueError as e:
            _refuse(f"{path!r}: a {n}-gram value is not a number ({e})")
        if n == 1:
            words = list(tok[at + 1])
            index = dict(zip(words, range(len(words))))
            if len(index) != len(words):
                _refuse(f"{path!r}: duplicate 1-grams")
            g = np.arange(len(words), dtype=np.int32)[:, None]
        else:
            w = tok[(at[:, None] + 1 + np.arange(n)[None, :]).reshape(-1)].tolist()
            try:
                g = np.array(list(map(index.__getitem__, w)), dtype=np.int32).reshape(-1, n)
            except KeyError as e:
                _refuse(f"{path!r}: the {n}-gram word {e} is not a 1-gram")
            if _has_duplicate_rows(g):
                _refuse(f"{path!r}: duplicate {n}-grams")
        ids.append(np.ascontiguousarray(g))
        logp.append(lp)
        backoff.append(bo)
    if b"<s>" not in index:
        _refuse(f"{path!r}: no <s> unigram")
    return ArpaModel(order=N, words=words, ids=ids, logp=logp, backoff=backoff, index=index)


@dataclass
class VocabTrie:
    """rule L1's V as a trie over label indices: node 0 is the root (the empty partial word); per node a 64-bit
    child mask over labels, the index of its first child (children contiguous, in label order) and the word id of
    its prefix (-1 if the prefix is not a word of V).  Nodes are numbered level by level."""
    mask: np.ndarray      # (NT,) uint64
    first: np.ndarray     # (NT,) int32
    word: np.ndarray      # (NT,) int32
    n_words: int          # |V|

    def child(self, node, c):
        """the child of `node` by label c, or -1"""
        m = int(self.mask[node])
        if not (m >> c) & 1:
            return -1
        return int(self.first[node]) + bin(m & ((1 << c) - 1)).count("1")


def build_trie(model: ArpaModel, labels, blank_index: int) -> VocabTrie:
    labels = list(labels)
    if ' ' not in labels:
        _refuse("the labels have no ' ' (space), so words cannot be delimited")
    space = labels.index(' ')
    if space == blank_index:
        _refuse("the space is the blank label")
    if len(labels) > 64:
        _refuse(f"{len(labels)} labels, at most 64 are supported")
    lab_of = {ch: i for i, ch in enumerate(labels) if i not in (blank_index, space)}
    text = []
    for w in model.words:
        try:
            text.append(w.decode("utf-8"))
        except UnicodeDecodeError:
            text.append(None)
    plain = [t for t, w in zip(text, model.words) if w not in SPECIAL]
    if plain and all(t is not None and len(t) == 1 for t in plain):
        _refuse("the model is character-based (every word is one character); only word-level models are supported")
    vid, seqs = [], []
    for i, (t, w) in enumerate(zip(text, model.words)):
        if t is None or w in SPECIAL or not t:
            continue
        s = [lab_of.get(ch, -1) for ch in t]
        if min(s) >= 0:
            vid.append(i)
            seqs.append(s)
    if not vid:
        _refuse("no word of the model can be spelled with the labels (a lowercase model with uppercase labels?)")
    nV = len(vid)
    L = np.array([len(s) for s in seqs], np.int64)
    D = int(L.max())
    lab = np.full((nV, D), -1, np.int64)
    for k, s in enumerate(seqs):
        lab[k, :len(s)] = s
    vid = np.array(vid, np.int64)
    parents_of_level, labs_of_level = [np.array([-1])], [np.array([-1])]
    node = np.zeros(nV, np.int64)          # node of each word's prefix at the current depth
    word_at = {}
    n_nodes = 1
    for d in range(1, D + 1):
        sel = np.nonzero(L >= d)[0]
        code = node[sel] * 64 + lab[sel, d - 1]
        uniq, inv = np.unique(code, return_inverse=True)
        ids = n_nodes + np.arange(len(uniq))
        parents_of_level.append(uniq // 64)
        labs_of_level.append(uniq % 64)
        node[sel] = ids[inv.reshape(-1)]
        done = sel[L[sel] == d]
        word_at.update(zip(node[done].tolist(), vid[done].tolist()))
        n_nodes += len(uniq)
    parent = np.concatenate(parents_of_level)
    clab = np.concatenate(labs_of_level)
    mask = np.zeros(n_nodes, np.uint64)
    first = np.zeros(n_nodes, np.int32)
    has_parent = np.arange(n_nodes) > 0
    np.bitwise_or.at(mask, parent[has_parent], np.left_shift(np.uint64(1), clab[has_parent].astype(np.uint64)))
    p, at = np.unique(parent[has_parent], return_index=True)
    first[p] = (at + 1).astype(np.int32)
    word = np.full(n_nodes, -1, np.int32)
    if word_at:
        k = np.fromiter(word_at.keys(), np.int64, len(word_at))
        word[k] = np.fromiter(word_at.values(), np.int64, len(word_at))
    return VocabTrie(mask=mask, first=first, word=word, n_words=nV)


class LanguageModel:
    """the parsed model, its trie over `labels`, and the device tables per device (built at first use)"""

    def __init__(self, path, labels, blank_index):
        self.path = path
        self.model = read_arpa(path)
        self.trie = build_trie(self.model, labels, blank_index)
        self.order = self.model.order
        self.space = list(labels).index(' ')
        self._tables = {}

    def device_tables(self, device):
        """the ds2_lm_build buffer on `device` (a CUDA torch.device), built on the current stream at the first call"""
        import ctypes as C
        import torch
        from ._lib import check, current_stream, get_lib, ptr
        key = torch.device(device).index
        if key in self._tables:
            return self._tables[key]
        lib = get_lib()
        m, tr = self.model, self.trie
        counts = (C.c_int64 * m.order)(*[len(x) for x in m.logp])
        nbytes = lib.ds2_lm_bytes(m.order, counts, len(tr.mask))
        if nbytes == 0:
            raise Ds2Error(f"BeamCTCDecoder: language-model scoring: ds2_lm_bytes refused the model {self.path!r}")
        dev = torch.device(device)
        up = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in m.ids + m.logp + m.backoff]
        n = m.order
        arr = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts])
        tmask = torch.from_numpy(tr.mask.view(np.int64)).to(dev)
        tfirst = torch.from_numpy(tr.first).to(dev)
        tword = torch.from_numpy(tr.word).to(dev)
        buf = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            check(lib.ds2_lm_build(n, counts, arr(up[:n]), arr(up[n:2 * n]), arr(up[2 * n:]), len(m.words),
                                   m.index[b"<s>"], len(tr.mask), ptr(tmask), ptr(tfirst), ptr(tword), ptr(buf),
                                   nbytes, current_stream()), "ds2_lm_build")
        self._tables[key] = buf
        return buf

    @property
    def table_bytes(self):
        import ctypes as C
        from ._lib import get_lib
        counts = (C.c_int64 * self.order)(*[len(x) for x in self.model.logp])
        return int(get_lib().ds2_lm_bytes(self.order, counts, len(self.trie.mask)))
