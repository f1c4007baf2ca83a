"""NumPy restatement of prioritised replay (include/torchbeast_b200.h): the draw of tb_replay_sample_prioritized, in the
header's summation order, and the priority update of tb_replay_update_priorities.  The survivor rule is the uniform
buffer's (tests/replay_oracle.py); the Philox is the action-sampling oracle's."""
import numpy as np

from oracle.sampling_np import philox4x32_10
from tests.replay_oracle import survivors

_LO = np.uint64(0xFFFFFFFF)
CHUNKS, WARP = 1024, 32


def survivor_slots(head, size, capacity, Bf):
    """int64 [n]: slot of survivor k, newest first."""
    return (head - 1 - np.arange(survivors(size, capacity, Bf))) % capacity


def cdf(q):
    """C [n] in the header's summation order: 1024 contiguous chunks summed in k order, their totals combined in order
    within each warp of 32 chunks, the warp totals in order; C_k = B_g + (P_i + r_k)."""
    n = len(q)
    L = -(-n // CHUNKS)
    pad = np.zeros(CHUNKS * L)
    pad[:n] = q                                       # adding the zeros of empty positions is exact
    r = np.cumsum(pad.reshape(CHUNKS, L), axis=1)     # np.cumsum adds in order
    tot = r[:, -1].reshape(CHUNKS // WARP, WARP)
    P = np.concatenate([np.zeros((CHUNKS // WARP, 1)), np.cumsum(tot, axis=1)[:, :-1]], axis=1)
    G = np.cumsum(tot, axis=1)[:, -1]
    base = np.concatenate([[0.0], np.cumsum(G)[:-1]])
    C = base[:, None, None] + (P[:, :, None] + r.reshape(CHUNKS // WARP, WARP, L))
    return C.reshape(-1)[:n]


def uniforms(R, seed, step, stream_id):
    """float64 [R]: u_j = ((w1 << 32 | w0) >> 11) * 2^-53 of replayed column j."""
    seed, step = np.uint64(seed % 2 ** 64), np.uint64(step % 2 ** 64)
    j = np.arange(R, dtype=np.uint32)
    w0, w1, _, _ = philox4x32_10((step & _LO, step >> np.uint64(32), j, np.uint32(stream_id)),
                                 (seed & _LO, seed >> np.uint64(32)))
    bits = ((w1.astype(np.uint64) << np.uint64(32)) | w0.astype(np.uint64)) >> np.uint64(11)
    return bits.astype(np.float64) * 2.0 ** -53


def prioritized(priorities, R, head, size, capacity, Bf, seed, step, stream_id, alpha, beta, eps):
    """(slots int64 [R], weights float32 [R], margin float64 [R]) of one prioritised draw; margin_j = the distance of
    u_j * S from the nearest CDF boundary, over S (a draw whose margin is below the error of q may differ on a device
    whose pow rounds differently)."""
    surv = survivor_slots(head, size, capacity, Bf)
    q = (priorities[surv].astype(np.float64) + eps) ** alpha
    C = cdf(q)
    S = C[-1]
    target = uniforms(R, seed, step, stream_id) * S
    k = np.searchsorted(C, target, side="right")      # the smallest k with C_k > target (C is non-decreasing)
    k = np.minimum(k, len(q) - 1)
    w = ((q.min() / q[k]) ** beta).astype(np.float32)
    margin = np.abs(target[:, None] - C[None, :]).min(axis=1) / S
    return surv[k], w, margin


def priority_update(vs, values, batch_slots, eta, priorities):
    """The priorities after tb_replay_update_priorities: a new float32 array."""
    out = priorities.copy()
    T, B = vs.shape
    e = np.abs(vs.astype(np.float64) - values.astype(np.float64))
    with np.errstate(invalid="ignore", over="ignore"):
        s = np.zeros(B)
        for t in range(T):                             # in t order
            s = s + e[t]
        p = (eta * e.max(axis=0) + (1.0 - eta) * (s / T)).astype(np.float32)
    p = np.where(np.isfinite(p), p, np.float32(0))
    for c in range(B):                                 # later columns overwrite earlier ones: the largest j wins
        out[batch_slots[c]] = p[c]
    return out
