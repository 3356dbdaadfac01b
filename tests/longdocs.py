"""TEST INFRASTRUCTURE: a collection of long documents, long arrays and positions past 65535, in the reference's own posting
encoding (src/index.cpp:1330-1393), for tests/test_long_documents.py.

Documents are token-id sequences over one vocabulary; list id == token id in every field. A Zipf vocabulary and heavy-tailed
lengths (1 to about 5,000 tokens) make frequent tokens repeat inside a document and give them dense lists. A few documents
of 65,540 to 140,000 tokens carry MARKER tokens at chosen positions around the uint16 wrap of Match's offsets
(src/posting_list.cpp:906: position p becomes offset (uint16_t) p - 1, so 65,536 becomes MAX_DISPLACEMENT and 65,537
becomes 0). Positions skip indices now and then, as the tokenizer does."""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np

from typesense_b200 import structs as S

VOCAB = 3000
N_MARKERS = 12                    # token ids VOCAB .. VOCAB + 11: placed by hand, rare everywhere
MARK = VOCAB
UNQUERIED = VOCAB + N_MARKERS     # token ids from here on are never queried (the filler of the scorer-switch test)
N_TOKENS = UNQUERIED + 64

# (marker, 1-based position) in the 140,000-token document LONG_WRAP
WRAP_PLACEMENTS = [(0, 65535), (1, 65536), (2, 65537), (3, 131073), (4, 131074), (9, 3), (9, 65540), (10, 131075)] + \
                  [(5, 65531), (6, 65534), (7, 65538), (8, 65542), (11, 65546)]     # windows straddling the wrap


def zipf_tokens(rng, n: int, s: float = 1.1) -> np.ndarray:
    w = 1.0 / np.arange(1, VOCAB + 1) ** s
    return rng.choice(VOCAB, size=n, p=w / w.sum()).astype(np.int64)


def positions_with_gaps(rng, n: int, gap_p: float = 0.03) -> np.ndarray:
    """1-based token_index + 1 of n tokens; an index is skipped with probability gap_p"""
    return np.cumsum(1 + (rng.random(n) < gap_p).astype(np.int64) * rng.integers(1, 4, n))


class Doc:
    __slots__ = ("tok", "pos")

    def __init__(self, tok, pos=None):
        self.tok = np.asarray(tok, np.int64)
        self.pos = np.arange(1, len(self.tok) + 1, dtype=np.int64) if pos is None else np.asarray(pos, np.int64)


def plain_field(docs: Sequence[Doc], n_lists: int = N_TOKENS) -> S.FlatField:
    """src/index.cpp:1330-1348: per (token, doc) the 1-based positions, then 0 when the token is the document's last."""
    tok, doc, key, val = [], [], [], []
    for d, D in enumerate(docs):
        if len(D.tok) == 0:
            continue
        tok += [D.tok, D.tok[-1:]]
        doc += [np.full(len(D.tok) + 1, d, np.int64)]
        key += [D.pos, np.asarray([1 << 20])]                  # the trailing 0 sorts after every position
        val += [D.pos, np.zeros(1, np.int64)]
    return _flatten(np.concatenate(tok), np.concatenate(doc), np.concatenate(key), np.concatenate(val), n_lists, False)


def array_field(docs: Sequence[Sequence[Doc]], n_lists: int = N_TOKENS) -> S.FlatField:
    """src/index.cpp:1351-1393: per element and token the element's 1-based positions, the last one repeated, the element
    index, and 0 when the token is the element's last."""
    tok, doc, key, val = [], [], [], []
    for d, elems in enumerate(docs):
        for ai, E in enumerate(elems):
            if len(E.tok) == 0:
                continue
            u, last_i = np.unique(E.tok[::-1], return_index=True)
            last_pos = E.pos[::-1][last_i]                        # each token's last position in the element
            base = (np.int64(ai) << 21)
            tok += [E.tok, u, u, E.tok[-1:]]
            key += [base | E.pos, np.full(len(u), base | ((1 << 21) - 3)), np.full(len(u), base | ((1 << 21) - 2)),
                    np.asarray([base | ((1 << 21) - 1)])]
            val += [E.pos, last_pos, np.full(len(u), ai), np.zeros(1, np.int64)]
            doc += [np.full(len(E.tok) + 2 * len(u) + 1, d, np.int64)]
    return _flatten(np.concatenate(tok), np.concatenate(doc), np.concatenate(key), np.concatenate(val), n_lists, True)


def _flatten(tok, doc, key, val, n_lists, is_array) -> S.FlatField:
    order = np.lexsort((key, doc, tok))
    tok, doc, val = tok[order], doc[order], val[order]
    new = np.ones(len(tok), bool)
    new[1:] = (tok[1:] != tok[:-1]) | (doc[1:] != doc[:-1])
    starts = np.flatnonzero(new)
    ids = doc[starts].astype(np.uint32)
    list_off = np.zeros(n_lists + 1, np.uint64)
    list_off[1:] = np.cumsum(np.bincount(tok[starts], minlength=n_lists))
    pos_off = np.append(starts, len(tok)).astype(np.uint64)
    return S.FlatField(list_off, ids, pos_off, val.astype(np.uint32), is_array)


def split_elements(rng, D: Doc, max_elems: int = 300) -> List[Doc]:
    """one document's tokens cut into 1..max_elems array elements, positions restarting at 1 in each"""
    n = len(D.tok)
    k = int(min(n, rng.integers(1, max_elems + 1)))
    cuts = np.sort(rng.choice(np.arange(1, n), k - 1, replace=False)) if k > 1 else np.zeros(0, np.int64)
    return [Doc(t) for t in np.split(D.tok, cuts)]


class LongCollection:
    """n_regular heavy-tailed documents, then the long documents:
      LONG_WRAP   140,000 tokens, markers at WRAP_PLACEMENTS
      LONG_LAST    65,540 tokens, its last token (marker 9) past 65535; marker 2 at 65,537
      LONG_GAPS   ~100,000 tokens with frequent gaps, marker 1 at 65,536 and marker 0 at 65,535
    Fields (same documents in each class):
      0 plain, every position < 65536 (the regular documents only): Pos16
      1 plain, the regular documents and the long ones: PlainOk, not Pos16
      2 array: the regular documents cut into 1..300 elements, plus ARRAY_WIDE with 70,000 one-token elements"""

    def __init__(self, n_regular: int = 1500, seed: int = 1):
        rng = np.random.default_rng(seed)
        self.rng = rng
        lens = np.minimum(5000, (10 * (1 + rng.pareto(1.1, n_regular))).astype(np.int64))
        lens[rng.random(n_regular) < 0.06] = 0
        lens = np.where(lens == 0, rng.integers(1, 4, n_regular), lens)           # some 1-3 token documents
        docs = [Doc(zipf_tokens(rng, int(n)), positions_with_gaps(rng, int(n), 0.02)) for n in lens]
        # short documents that exercise the verbatim test: a token at position 1 with and without the trailing 0
        for i, t in enumerate((0, 1, 2, 3, 5, 8)):
            docs[3 * i] = Doc([t, 40 + i, t, 60 + i])
            docs[3 * i + 1] = Doc([t])
            docs[3 * i + 2] = Doc([t, t])
        # markers in a few regular documents at small positions, so marker queries rank several documents
        for m in range(N_MARKERS):
            for d in rng.choice(n_regular, 3, replace=False):
                D = docs[int(d)]
                if len(D.tok) > 2:
                    D.tok[int(rng.integers(0, len(D.tok)))] = MARK + m
        self.n_regular = n_regular
        self.LONG_WRAP, self.LONG_LAST, self.LONG_GAPS = n_regular, n_regular + 1, n_regular + 2
        self.ARRAY_WIDE = n_regular + 3
        wrap = Doc(zipf_tokens(rng, 140000))
        for m, p in WRAP_PLACEMENTS:
            wrap.tok[p - 1] = MARK + m
        last = Doc(zipf_tokens(rng, 65540))
        last.tok[-1] = MARK + 9
        last.tok[65536] = MARK + 2
        gaps = Doc(zipf_tokens(rng, 60000), positions_with_gaps(rng, 60000, 0.4))
        gaps.tok[np.searchsorted(gaps.pos, 65536)] = MARK + 1
        gaps.pos[np.searchsorted(gaps.pos, 65536)] = 65536
        i0 = np.searchsorted(gaps.pos, 65535)
        if gaps.pos[i0] == 65535:
            gaps.tok[i0] = MARK + 0
        self.docs = docs + [wrap, last, gaps]
        self.n_docs = n_regular + 4
        self.elems = [split_elements(rng, D) for D in docs] + [[], [], []]
        wide = [Doc([int(t)]) for t in zipf_tokens(rng, 70000)]
        for i in (0, 65535, 65536, 65537, 69999):
            wide[i] = Doc([MARK + 9, int(rng.integers(0, 20))])
        self.elems.append(wide)
        self.flats = [plain_field(docs), plain_field(self.docs), array_field(self.elems)]
        self.pts = np.where(rng.random(self.n_docs) < 0.1, np.int64(np.iinfo(np.int64).min),
                            rng.integers(0, 5, self.n_docs)).astype(np.int64)

    def span(self, rng, n_tok: int, long_doc_p: float = 0.35):
        """n_tok contiguous tokens of one document (a long one with probability long_doc_p, often near the wrap)"""
        if rng.random() < long_doc_p:
            D = self.docs[self.n_regular + int(rng.integers(0, 3))]
            centre = int(rng.choice([65530, 65536, 131070, len(D.tok) - n_tok, int(rng.integers(0, len(D.tok)))]))
            s = int(np.clip(centre - int(rng.integers(0, n_tok + 1)), 0, max(0, len(D.tok) - n_tok)))
        else:
            D = self.docs[int(rng.integers(0, self.n_regular))]
            s = int(rng.integers(0, max(1, len(D.tok) - n_tok + 1)))
        return [int(t) for t in D.tok[s:s + n_tok]]
