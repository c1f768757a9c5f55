"""ORACLE (test infrastructure): CPU restatement of the reference's CTC forced alignment, written from its update
rules — `insert_blank` (asr/wenet/utils/ctc_utils.py:95-102) and `force_align` (:105-161) — plus the per-token
reduction and the float64 forward log-likelihood the engine adds on the same trellis.

Rules restated (fp32 throughout, like the reference's `log_alpha`):
  states z = [b, y0, b, y1, ..., b, y_{U-1}, b], S = 2U + 1                                       (:95-102)
  alpha[0][0] = logp[0][z0], alpha[0][1] = logp[0][z1], everything else -inf                      (:119-126)
  alpha[t][s] = max(cands) + logp[t][z_s], cands = [alpha[t-1][s], alpha[t-1][s-1]] and, only when z_s is not
      blank, s >= 2 and z_s != z_{s-2}, alpha[t-1][s-2]; the back-pointer is the FIRST maximum       (:128-144)
  end state = S-1 unless alpha[T-1][S-2] is strictly greater; then follow the back-pointers          (:146-155)
Not restated: at s = 0 the reference's second candidate is alpha[t-1][s-1] = alpha[t-1][-1], which Python reads as the
LAST state (:133), so its trellis lets a path run through the labels and start over.  Such a path is not an alignment
of y; here state 0 has the single predecessor it should.  make_golden_align.py checks that the two agree on every
pinned case.
The reference keeps the states in int16 and fails with IndexError on an empty label; neither is reproduced: states
are int32 and U == 0 is a ValueError.
"""
import numpy as np

NEG_INF = np.float32(-np.inf)


def feasible(labels, n_frames: int) -> bool:
    """An alignment exists iff U >= 1 and T >= U + #(adjacent equal labels)."""
    U = len(labels)
    return U >= 1 and n_frames >= U + sum(1 for a, b in zip(labels[:-1], labels[1:]) if a == b)


def states_of(labels, blank_id: int = 0) -> np.ndarray:
    z = np.full(2 * len(labels) + 1, blank_id, dtype=np.int64)
    z[1::2] = np.asarray(labels, dtype=np.int64)
    return z


def viterbi(logp: np.ndarray, labels, blank_id: int = 0):
    """logp (T, V) float32 -> (state per frame int32 (T,), Viterbi score float32)."""
    if len(labels) == 0:
        raise ValueError("empty label sequence")
    logp = np.asarray(logp, dtype=np.float32)
    T = logp.shape[0]
    z = states_of(labels, blank_id)
    S = len(z)
    skip = np.zeros(S, dtype=bool)
    skip[2:] = (z[2:] != blank_id) & (z[2:] != z[:-2])
    alpha = np.full(S, NEG_INF, dtype=np.float32)
    alpha[0], alpha[1] = logp[0, z[0]], logp[0, z[1]]
    back = np.zeros((T, S), dtype=np.int8)
    for t in range(1, T):
        c0 = alpha
        c1 = np.concatenate(([NEG_INF], alpha[:-1]))
        c2 = np.where(skip, np.concatenate(([NEG_INF, NEG_INF], alpha[:-2])), NEG_INF)
        best, step = c0.copy(), np.zeros(S, dtype=np.int8)
        m = c1 > best
        best[m], step[m] = c1[m], 1
        m = skip & (c2 > best)
        best[m], step[m] = c2[m], 2
        alpha = (best + logp[t, z]).astype(np.float32)
        back[t] = step
    s = S - 2 if alpha[S - 2] > alpha[S - 1] else S - 1
    score = alpha[s]
    states = np.zeros(T, dtype=np.int32)
    for t in range(T - 1, -1, -1):
        states[t] = s
        s -= int(back[t, s])
    return states, np.float32(score)


def force_align(logp: np.ndarray, labels, blank_id: int = 0) -> np.ndarray:
    """The reference's return value: the token id (blank or label) of every frame."""
    states, _ = viterbi(logp, labels, blank_id)
    return states_of(labels, blank_id)[states].astype(np.int32)


def token_spans(logp: np.ndarray, states: np.ndarray, labels):
    """Per label: first frame, last frame, peak frame (largest logp[t][y_u] of the span, first on ties), that log-prob."""
    U = len(labels)
    first, last, peak = (np.zeros(U, dtype=np.int32) for _ in range(3))
    peak_logp = np.zeros(U, dtype=np.float32)
    for u in range(U):
        ts = np.nonzero(states == 2 * u + 1)[0]
        assert len(ts) and ts[-1] - ts[0] + 1 == len(ts), "every label owns one contiguous span"
        vals = np.asarray(logp, dtype=np.float32)[ts, labels[u]]
        k = int(np.argmax(vals))
        first[u], last[u], peak[u], peak_logp[u] = ts[0], ts[-1], ts[k], vals[k]
    return first, last, peak, peak_logp


def forward_loglik(logp: np.ndarray, labels, blank_id: int = 0) -> float:
    """log p(y | x): the forward algorithm over the same states in float64."""
    lp = np.asarray(logp, dtype=np.float64)
    z = states_of(labels, blank_id)
    S = len(z)
    skip = np.zeros(S, dtype=bool)
    skip[2:] = (z[2:] != blank_id) & (z[2:] != z[:-2])
    alpha = np.full(S, -np.inf)
    alpha[0], alpha[1] = lp[0, z[0]], lp[0, z[1]]
    for t in range(1, lp.shape[0]):
        c1 = np.concatenate(([-np.inf], alpha[:-1]))
        c2 = np.where(skip, np.concatenate(([-np.inf, -np.inf], alpha[:-2])), -np.inf)
        alpha = np.logaddexp(np.logaddexp(alpha, c1), c2) + lp[t, z]
    return float(np.logaddexp(alpha[S - 1], alpha[S - 2]))


def align(logp: np.ndarray, labels, blank_id: int = 0) -> dict:
    states, score = viterbi(logp, labels, blank_id)
    first, last, peak, peak_logp = token_spans(logp, states, labels)
    return {"frames": states_of(labels, blank_id)[states].astype(np.int32), "first": first, "last": last, "peak": peak,
            "peak_logp": peak_logp, "score": score}
