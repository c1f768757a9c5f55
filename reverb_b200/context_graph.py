"""Context biasing graph for CTC prefix beam search (host side), compiled to flat arrays.

Behaviour = `asr/wenet/utils/context_graph.py` of the reference (ContextGraph :104-265, tokenize :24-58): an
Aho-Corasick automaton over the token sequences of the biasing phrases.  Every node carries the bonus accumulated from
the root (`depth * context_score`), a fail link and the summed bonus of the phrases that END at it or at a node on its
output chain; the search feeds it one token at a time (`forward_one_step`) and closes a hypothesis with `finalize`.
The reference's observable quirks are kept: when a token does not extend the current node, the fail walk stops at the
root WITHOUT retrying the root's own children unless the loop lands there (:217-225, same in the construction :168-176);
a phrase that ends on an already existing node does not mark it as a phrase end (:150-161).

Representation: states are plain integers (0 = root) indexing parallel lists — `children[s]` (token -> state),
`fail[s]`, `bonus[s]`, `emit[s]` — instead of linked node objects; `ASRModel.decode(context_graph=...)` and
`reverb_b200.search.ctc_prefix_beam_search_biased` only use `root`, `forward_one_step` and `finalize`, so the
reference's own `ContextGraph` object can be passed as well.  The GPU search takes either form through `device_tables`,
which compiles the automaton to the flat tables the device holds (csrc/context.cu).
"""
from __future__ import annotations

import os
import re
from typing import Dict, Iterable, List, Optional, Sequence, Tuple

import numpy as np

_CJK = re.compile(r"([一-鿿])")


def tokenize(context_list_path, symbol_table: Dict[str, int], bpe_model: Optional[str] = None) -> List[List[int]]:
    """One biasing phrase per line -> token ids.  `context_list_path` is a file path or the lines themselves (any
    iterable of strings).  With a sentencepiece model: upper-cased text, CJK characters on their own, everything else
    through `encode_as_pieces` (text/tokenize_utils.py:19-60); without: one symbol per character, space written as the
    word-boundary mark.  Symbols missing from the table become <unk> if the table has it and are dropped otherwise."""
    encode = None
    if bpe_model is not None:
        import sentencepiece as spm
        sp = spm.SentencePieceProcessor()
        sp.load(bpe_model)

        def encode(text: str) -> List[str]:
            pieces: List[str] = []
            for part in _CJK.split(text.upper()):
                if part.strip():
                    pieces.extend([part] if _CJK.fullmatch(part) else sp.encode_as_pieces(part))
            return pieces
    unk = symbol_table.get("<unk>")

    def phrase(line: str) -> List[int]:
        text = line.strip()
        symbols = encode(text) if encode else [("▁" if ch == " " else ch) for ch in text]
        ids = [symbol_table.get(sym, unk) for sym in symbols]
        return [i for i in ids if i is not None]
    if isinstance(context_list_path, (str, os.PathLike)):
        with open(context_list_path, "r") as f:
            return [phrase(line) for line in f]
    return [phrase(line) for line in context_list_path]


class ContextGraph:
    root = 0

    def __init__(self, context_list_path: Optional[str] = None, symbol_table: Optional[Dict[str, int]] = None,
                 bpe_model: Optional[str] = None, context_score: float = 6.0,
                 token_lists: Optional[Iterable[Sequence[int]]] = None):
        """Positional arguments as in the reference (`context_list_path, symbol_table, bpe_model, context_score`);
        `token_lists` builds the graph from token ids directly."""
        self.context_score = context_score
        self.context_list = ([list(t) for t in token_lists] if token_lists is not None
                             else tokenize(context_list_path, symbol_table or {}, bpe_model))
        self.children: List[Dict[int, int]] = [{}]
        self.token: List[int] = [-1]
        self.bonus: List[float] = [0.0]       # accumulated bonus root -> node ("node_score")
        self.emit: List[float] = [0.0]        # bonus of the phrases recognised on arrival ("output_score")
        self.ends: List[bool] = [False]
        self.fail: List[int] = [0]
        self._insert_phrases()
        self._link()

    @property
    def num_nodes(self) -> int:
        return len(self.token) - 1

    def _insert_phrases(self) -> None:
        for phrase in self.context_list:
            s = 0
            for pos, tok in enumerate(phrase):
                nxt = self.children[s].get(tok)
                if nxt is None:
                    nxt = len(self.token)
                    last = pos == len(phrase) - 1
                    depth_bonus = self.bonus[s] + self.context_score
                    self.children[s][tok] = nxt
                    self.children.append({})
                    self.token.append(tok)
                    self.bonus.append(depth_bonus)
                    self.emit.append(depth_bonus if last else 0)
                    self.ends.append(last)
                    self.fail.append(0)
                s = nxt

    def _fallback(self, start: int, tok: int) -> int:
        """Walk fail links from `start` until a node with a `tok` child is found or the root is reached; take that child
        if there is one.  (The root's children are only consulted when the walk ends on the root.)"""
        s = start
        while tok not in self.children[s]:
            s = self.fail[s]
            if s == 0:
                break
        return self.children[s].get(tok, s)

    def _link(self) -> None:
        order = list(self.children[0].values())          # breadth first; depth-1 nodes fail to the root
        head = 0
        while head < len(order):
            parent = order[head]
            head += 1
            for tok, node in self.children[parent].items():
                f = self.fail[parent]
                self.fail[node] = self.children[f][tok] if tok in self.children[f] else self._fallback(self.fail[f], tok)
                # nearest phrase end on the fail chain contributes its (already complete) output bonus
                out = self.fail[node]
                while not self.ends[out]:
                    out = self.fail[out]
                    if out == 0:
                        out = -1
                        break
                if out >= 0:
                    self.emit[node] += self.emit[out]
                order.append(node)

    # -- queries ------------------------------------------------------------------------------------------------------
    def forward_one_step(self, state: int, token: int) -> Tuple[float, int]:
        nxt = self.children[state].get(token)
        if nxt is not None:
            gained = self.context_score
        else:
            nxt = self._fallback(self.fail[state], token)
            gained = self.bonus[nxt] - self.bonus[state]
        return gained + self.emit[nxt], nxt

    def finalize(self, state: int) -> Tuple[float, int]:
        """Take back the bonus of a match that did not complete; the next state is the root."""
        return -self.bonus[state], 0


# -- device tables ----------------------------------------------------------------------------------------------------
def _linked_states(root) -> list:
    """The states of a linked-node graph (the reference's `ContextState`: `.next`, `.fail`, `.node_score`,
    `.output_score`, `.token_score`) indexed by their `id` when the ids number the states 0..n-1 with the root at 0,
    else in breadth-first order from the root."""
    order, seen, head = [root], {id(root)}, 0
    while head < len(order):
        for child in order[head].next.values():
            if id(child) not in seen:
                seen.add(id(child))
                order.append(child)
        head += 1
    ids = [getattr(s, "id", None) for s in order]
    if all(isinstance(i, int) for i in ids) and sorted(ids) == list(range(len(order))) and ids[0] == 0:
        states = [None] * len(order)
        for s in order:
            states[s.id] = s
        return states
    return order


def device_tables(graph) -> Dict[str, np.ndarray]:
    """Compile a context graph — this module's `ContextGraph` or the reference's linked `ContextState` graph — to the
    flat tables the GPU search reads (include/rvb_b200.h rvb_context_graph_create): state 0 = root; `off` (n + 1) /
    `tok` / `dst` the children in CSR by state, sorted by token; `fail` (n); `bonus` (node_score), `emit`
    (output_score) and `token_score` as float64, the host values as they are."""
    if isinstance(graph.root, (int, np.integer)):
        n = len(graph.children)
        children = [sorted(c.items()) for c in graph.children]
        fail = list(graph.fail)
        bonus, emit = list(graph.bonus), list(graph.emit)
        # forward_one_step scores a matched child with the graph's context_score (the reference: node.token_score)
        token_score = [0.0] + [float(graph.context_score)] * (n - 1)
    else:
        states = _linked_states(graph.root)
        index = {id(s): i for i, s in enumerate(states)}
        n = len(states)
        children = [sorted((tok, index[id(c)]) for tok, c in s.next.items()) for s in states]
        fail = [index[id(s.fail)] if s.fail is not None else 0 for s in states]
        bonus = [s.node_score for s in states]
        emit = [s.output_score for s in states]
        token_score = [s.token_score for s in states]
    off = np.zeros(n + 1, dtype=np.int64)
    off[1:] = np.cumsum([len(c) for c in children])
    tok = np.fromiter((t for c in children for t, _ in c), dtype=np.int64, count=int(off[-1]))
    dst = np.fromiter((d for c in children for _, d in c), dtype=np.int64, count=int(off[-1]))
    return {"off": off, "tok": tok, "dst": dst, "fail": np.asarray(fail, dtype=np.int64),
            "bonus": np.asarray(bonus, dtype=np.float64), "emit": np.asarray(emit, dtype=np.float64),
            "token_score": np.asarray(token_score, dtype=np.float64)}


def check_device_tables(t: Dict[str, np.ndarray], vocab: int, blank_id: int) -> None:
    """ValueError unless `t` (device_tables) is a graph the GPU search can walk: at most 2^31 - 1 states, a trie
    reachable from the root, tokens in [0, vocab) and not the blank, fail links to strictly shallower states (every fail
    walk ends at the root), finite scores.  The native upload repeats these checks."""
    n = int(t["fail"].shape[0])
    if not 1 <= n <= np.iinfo(np.int32).max:
        raise ValueError(f"context graph: {n} states do not fit int32 indices")
    off, tok, dst, fail = t["off"], t["tok"], t["dst"], t["fail"]
    if off.shape[0] != n + 1 or off[0] != 0 or off[-1] != n - 1 or tok.shape[0] != n - 1 or dst.shape[0] != n - 1 \
            or np.any(np.diff(off) < 0):
        raise ValueError("context graph: the child tables are not a trie over the states")
    for name in ("bonus", "emit", "token_score"):
        if t[name].shape[0] != n or not np.all(np.isfinite(t[name])):
            raise ValueError(f"context graph: {name} must hold one finite value per state")
    bad = (tok < 0) | (tok >= vocab) | (tok == blank_id)
    if np.any(bad):
        raise ValueError(f"context graph: token {int(tok[np.argmax(bad)])} is not a non-blank id of the "
                         f"{vocab}-entry vocabulary (blank {blank_id})")
    depth = np.full(n, -1, dtype=np.int64)
    depth[0] = 0
    order, head = [0], 0
    while head < len(order):
        s = order[head]
        head += 1
        lo, hi = int(off[s]), int(off[s + 1])
        if np.any(np.diff(tok[lo:hi]) <= 0):
            raise ValueError(f"context graph: children of state {s} are not sorted by token")
        for c in dst[lo:hi].tolist():
            if not 0 < c < n or depth[c] >= 0:
                raise ValueError(f"context graph: state {c} is out of range or has two parents")
            depth[c] = depth[s] + 1
            order.append(c)
    if len(order) != n:
        raise ValueError(f"context graph: {n - len(order)} states are unreachable from the root")
    if fail[0] != 0 or np.any((fail < 0) | (fail >= n)) or np.any(depth[fail[1:]] >= depth[1:]):
        raise ValueError("context graph: a fail link does not lead toward the root")
