"""Context biasing, host side of the GPU search: the flat device tables of a context graph (either graph form), their
checks, tokenizing phrases from a list, and the CLI flags.  No GPU needed."""
import ctypes

import numpy as np
import pytest

from reverb_b200 import synth
from reverb_b200.context_graph import ContextGraph, check_device_tables, device_tables, tokenize

PHRASES = [[1, 2, 3], [2, 3], [3], [1, 2], [2, 3, 4, 5], [5], [4, 5, 1], [6, 7], [7, 6, 7, 6], [9] * 5, [9, 9, 8]]


class _State:
    """A linked-node state with the attributes of the reference's ContextState."""

    def __init__(self, id, token, token_score, node_score, output_score, is_end):
        self.id, self.token, self.token_score = id, token, token_score
        self.node_score, self.output_score, self.is_end = node_score, output_score, is_end
        self.next, self.fail = {}, None


class _LinkedGraph:
    def __init__(self, g: ContextGraph, ids=True):
        states = [_State(i if ids else None, g.token[i], 0.0 if i == 0 else g.context_score, g.bonus[i], g.emit[i],
                         g.ends[i]) for i in range(len(g.token))]
        for i, s in enumerate(states):
            s.next = {tok: states[c] for tok, c in g.children[i].items()}
            s.fail = states[g.fail[i]]
        self.root = states[0]


def _step(t, s, u):
    """forward_one_step over the device tables, as csrc/ctc.cu ctx_step walks them."""
    def child(s):
        lo, hi = int(t["off"][s]), int(t["off"][s + 1])
        hit = np.nonzero(t["tok"][lo:hi] == u)[0]
        return int(t["dst"][lo + hit[0]]) if hit.size else -1
    n = child(s)
    if n >= 0:
        gained = t["token_score"][n]
    else:
        f = int(t["fail"][s])
        while (n := child(f)) < 0:
            f = int(t["fail"][f])
            if f == 0:
                n = child(0)
                break
        n = n if n >= 0 else f
        gained = t["bonus"][n] - t["bonus"][s]
    return gained + t["emit"][n], n


@pytest.mark.parametrize("phrases", [PHRASES, synth.context_phrases(300, 40, seed=2)], ids=["nested", "random"])
def test_tables_walk_like_the_host_automaton(phrases):
    g = ContextGraph(token_lists=phrases, context_score=2.5)
    t = device_tables(g)
    check_device_tables(t, 50, 0)
    rng = np.random.default_rng(0)
    for _ in range(20):
        s = 0
        for u in rng.integers(1, 12 if phrases is PHRASES else 40, size=40).tolist():
            want = g.forward_one_step(s, u)
            got = _step(t, s, u)
            assert got == want
            s = got[1]
        assert -t["bonus"][s] == g.finalize(s)[0]


def test_linked_node_graph_gives_identical_tables():
    g = ContextGraph(token_lists=PHRASES + synth.context_phrases(200, 30, seed=4), context_score=3.0)
    want = device_tables(g)
    got = device_tables(_LinkedGraph(g))
    assert sorted(got) == sorted(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and np.array_equal(got[k], want[k]), k
    # without ids the states are numbered breadth first: another numbering of the same automaton
    bfs = device_tables(_LinkedGraph(g, ids=False))
    check_device_tables(bfs, 40, 0)
    s_bfs = s_host = 0
    for u in np.random.default_rng(1).integers(1, 30, size=300).tolist():
        a, s_bfs = _step(bfs, s_bfs, u)
        b, s_host = g.forward_one_step(s_host, u)
        assert a == b


def test_tokenize_from_lines_equals_tokenize_from_file(tmp_path):
    table = {"<blank>": 0, "<unk>": 1, "a": 2, "b": 3, "▁": 4, "中": 5}
    lines = ["ab a", "zb", "  b中 ", ""]
    p = tmp_path / "ctx.txt"
    p.write_text("\n".join(lines) + "\n")
    assert tokenize(lines, table) == tokenize(str(p), table) == tokenize(p, table)
    assert tokenize(iter(lines), table) == tokenize(str(p), table)


def _bad(t, **changes):
    t = {k: v.copy() for k, v in t.items()}
    for k, (i, v) in changes.items():
        t[k][i] = v
    return t


def test_malformed_graphs_raise_value_error_before_any_launch():
    from reverb_b200.engine import DeviceContextGraph
    g = ContextGraph(token_lists=PHRASES, context_score=3.0)
    t = device_tables(g)
    with pytest.raises(ValueError, match="token 12"):
        DeviceContextGraph(ContextGraph(token_lists=[[3, 12]]), 12, 0)     # token >= V
    with pytest.raises(ValueError, match="token 0"):
        DeviceContextGraph(ContextGraph(token_lists=[[3, 0, 4]]), 12, 0)   # the blank
    with pytest.raises(ValueError, match="token 7"):
        DeviceContextGraph(ContextGraph(token_lists=[[7]]), 12, 7)         # another blank id
    with pytest.raises(ValueError, match="fail link"):
        check_device_tables(_bad(t, fail=(5, 5)), 12, 0)                   # a fail link that never reaches the root
    with pytest.raises(ValueError, match="sorted"):
        check_device_tables(_bad(t, tok=(0, 3)), 12, 0)
    with pytest.raises(ValueError, match="two parents|unreachable"):
        check_device_tables(_bad(t, dst=(1, int(t["dst"][0]))), 12, 0)
    with pytest.raises(ValueError, match="finite"):
        check_device_tables(_bad(t, bonus=(2, np.nan)), 12, 0)


def test_native_upload_repeats_the_checks():
    """rvb_context_graph_create refuses a bad table before it allocates anything (so also without a GPU)."""
    from reverb_b200 import _lib
    lib = _lib.load()
    t = device_tables(ContextGraph(token_lists=[[3, 4], [5]], context_score=3.0))
    a = {k: np.ascontiguousarray(v, dtype=np.float64 if v.dtype == np.float64 else np.int32) for k, v in t.items()}
    a["tok"][0] = 99

    def p(x):
        return x.ctypes.data_as(ctypes.c_void_p)
    h = lib.rvb_context_graph_create(len(a["fail"]), p(a["off"]), p(a["tok"]), p(a["dst"]), p(a["fail"]),
                                     p(a["bonus"]), p(a["emit"]), p(a["token_score"]), 12, 0)
    assert not h and "token 99" in _lib.last_error()


def test_cli_context_flags():
    from reverb_b200.recognize_wav import get_args
    a = get_args(["--audio_file", "a.wav", "--result_dir", "o"])
    assert a.context_list_path is None and a.context_graph_score == 6.0
    a = get_args(["--audio_file", "a.wav", "--result_dir", "o", "--context_list_path", "c.txt",
                  "--context_graph_score", "2.5"])
    assert a.context_list_path == "c.txt" and a.context_graph_score == 2.5
