"""ORACLE (test infrastructure, never shipped, never the thing measured).

NumPy restatement of the action-sampling contract of tb_sample_actions_f32 (include/torchbeast_b200.h):
Philox4x32-10 keyed by the seed with counter (step + t, stream id), a 24-bit uniform u, and the first action whose
cumulative softmax mass exceeds u.  The softmax here is float64, so it is the exact distribution the kernel's fp32
arithmetic approximates; `margin` says how far each row's u*S lies from the nearest cumulative boundary, relative to
S, which is where fp32 and float64 rounding may legitimately pick different neighbours.
"""
import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_LO = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)


def philox4x32_10(counter, key):
    """Philox4x32-10 (Salmon et al., SC 2011).  counter: 4 uint32 arrays (or scalars) c0..c3; key: 2 uint32 k0, k1.
    Returns the 4 output words as uint32 arrays broadcast to a common shape."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint32) for c in counter)
    k0, k1 = (np.asarray(k, dtype=np.uint32) for k in key)
    c0, c1, c2, c3, k0, k1 = np.broadcast_arrays(c0, c1, c2, c3, k0, k1)
    k0, k1 = k0.copy(), k1.copy()
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = _M0 * c0.astype(np.uint64)
            p1 = _M1 * c2.astype(np.uint64)
            hi0, lo0 = (p0 >> _S32).astype(np.uint32), (p0 & _LO).astype(np.uint32)
            hi1, lo1 = (p1 >> _S32).astype(np.uint32), (p1 & _LO).astype(np.uint32)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0 = k0 + _W0
            k1 = k1 + _W1
    return c0, c1, c2, c3


def uniforms(T, B, seed, step, stream_ids=None):
    """u [T, B] float64: the 24-bit uniform of row (t, b) under the contract."""
    sid = np.arange(B, dtype=np.uint64) if stream_ids is None else np.asarray(stream_ids, dtype=np.int64).view(np.uint64)
    with np.errstate(over="ignore"):
        ctr = np.uint64(step) + np.arange(T, dtype=np.uint64)
    ctr, sid = np.broadcast_arrays(ctr[:, None], sid[None, :])
    seed = np.uint64(seed)
    x, _, _, _ = philox4x32_10((ctr & _LO, ctr >> _S32, sid & _LO, sid >> _S32), (seed & _LO, seed >> _S32))
    return (x >> np.uint32(8)).astype(np.float64) * 2.0 ** -24


def sample_actions(logits, seed, step, stream_ids=None):
    """logits [T, B, A] -> (actions int64 [T, B], margin float64 [T, B]).

    Rows with a NaN, with every logit -inf, or with a +inf logit get action -1 and margin +inf (the answer does not
    depend on rounding)."""
    x = np.asarray(logits, dtype=np.float64)
    T, B, A = x.shape
    u = uniforms(T, B, seed, step, stream_ids)
    with np.errstate(invalid="ignore"):
        m = np.max(np.where(np.isnan(x), -np.inf, x), axis=-1)
    bad = np.isnan(x).any(axis=-1) | ~np.isfinite(m)
    m = np.where(bad, 0.0, m)
    with np.errstate(invalid="ignore", over="ignore"):
        e = np.where(bad[..., None], 0.0, np.exp(x - m[..., None]))
    c = np.cumsum(e, axis=-1)               # running sums in index order; S is the last one
    S = c[..., -1]
    target = u * S
    above = c > target[..., None]
    first = np.argmax(above, axis=-1)
    last_pos = A - 1 - np.argmax((e > 0)[..., ::-1], axis=-1)
    actions = np.where(above.any(axis=-1), first, last_pos).astype(np.int64)
    with np.errstate(invalid="ignore", divide="ignore"):
        margin = np.min(np.abs(c - target[..., None]), axis=-1) / S
    actions[bad] = -1
    margin[bad] = np.inf
    return actions, margin


def margin_threshold(A):
    """Rows whose margin is below this may differ between the fp32 kernel and this float64 restatement: A fp32 additions
    and A precise expf calls (2 ulp each) plus the rounding of u*S, with a factor of 8 to spare."""
    return 8.0 * (A + 2) * 2.0 ** -24


def chi2(actions, probs):
    """Pearson's chi-squared statistic of the action counts against the probabilities `probs` [A]."""
    probs = np.asarray(probs, dtype=np.float64)
    counts = np.bincount(np.asarray(actions).reshape(-1), minlength=probs.size).astype(np.float64)
    expected = counts.sum() * probs
    return float(np.sum((counts - expected) ** 2 / expected))


def softmax(logits):
    x = np.asarray(logits, dtype=np.float64)
    e = np.exp(x - x.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)
