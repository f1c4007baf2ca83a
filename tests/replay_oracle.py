"""NumPy restatement of the replay slot rule of tb_replay_mix (include/torchbeast_b200.h), on top of the Philox of the
action-sampling oracle, plus the warm-up accounting of torchbeast_b200.replay.ReplayBuffer."""
import numpy as np

from oracle.sampling_np import philox4x32_10

_LO = np.uint64(0xFFFFFFFF)


def survivors(size, capacity, Bf):
    """n: the newest stored columns a call with Bf fresh columns leaves in place."""
    return min(size, capacity - Bf)


def slots(R, head, size, capacity, Bf, seed, step, stream_id):
    """int64 [R]: the slot of each replayed column of one call, read against the state (head, size, seed, step)."""
    n = survivors(size, capacity, Bf)
    seed, step = np.uint64(seed % 2 ** 64), np.uint64(step % 2 ** 64)
    j = np.arange(R, dtype=np.uint32)
    x, _, _, _ = philox4x32_10((step & _LO, step >> np.uint64(32), j, np.uint32(stream_id)),
                               (seed & _LO, seed >> np.uint64(32)))
    k = (x.astype(np.uint64) * np.uint64(n)) >> np.uint64(32)
    return (head - 1 - k.astype(np.int64)) % capacity


def overwritten(head, capacity, Bf):
    """The slots a call with Bf fresh columns writes."""
    return (head + np.arange(Bf)) % capacity


def advance(head, size, step, capacity, Bf):
    """(head, size, step) after one call."""
    return (head + Bf) % capacity, min(size + Bf, capacity), step + 1


def mixing(size, capacity, Bf, min_size):
    """Whether a call draws replayed columns (else it inserts only: the warm-up)."""
    return survivors(size, capacity, Bf) >= min_size
