"""Experience replay for the learner: a device-resident ring of earlier batch columns (tb_replay_mix, csrc/replay.cu).

Attach a buffer to the learner model and every learn() call mixes `replay_columns` replayed columns into its batch:

    model.replay = ReplayBuffer(capacity=4096, replay_columns=16, seed=1234)

A call with Bf fresh columns trains on Bf + R columns: the fresh ones first, then R columns drawn uniformly, with
replacement, from the min(size, capacity - Bf) newest stored columns; then the fresh columns are stored.  Until that
many columns reach `min_size` (default R) a call stores its fresh columns and trains on them alone, exactly as without a
buffer.  The draws depend only on (seed, step, stream id, head, size), so a run is reproducible, eager or graphed
(include/torchbeast_b200.h states the rule).  The stored leaves are those of GraphedLearner.KEYS present in the batch
and the initial agent state; other batch leaves are not stored and not passed on.
"""
import ctypes

import torch

from torchbeast_b200 import _lib


class _Leaf(ctypes.Structure):
    """tb_replay_leaf (include/torchbeast_b200.h)."""
    _fields_ = [("fresh", ctypes.c_void_p), ("out", ctypes.c_void_p), ("ring", ctypes.c_void_p),
                ("outer", ctypes.c_int64), ("row_bytes", ctypes.c_int64)]


def _i64(u):
    """The int64 with the bits of the uint64 u."""
    u %= 2 ** 64
    return u - 2 ** 64 if u >= 2 ** 63 else u


def _dp_rank():
    import torch.distributed as dist
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


class ReplayBuffer:
    """A device ring of `capacity` batch columns mixed into each learner batch.

    `seed` and `step` are plain public ints, like ActionSampler's: a checkpoint stores them, and a restored buffer
    continues the same draws once it has refilled (ring contents are not checkpointed, so a resumed run warms up again).
    `stream_id` (default: the data-parallel rank) separates the draws of buffers that share a seed.  `head` and `size`
    mirror the device state on the host; inserts are deterministic, so the mirror is exact without a device read.
    The ring is allocated on the first call, from that batch's leaf shapes and dtypes; a later batch whose columns
    differ raises.  Calls must be serialised by the caller (learner.learn holds its lock around them)."""

    def __init__(self, capacity, replay_columns, seed=0, min_size=None, stream_id=None, device=None):
        self.capacity = int(capacity)
        self.replay_columns = int(replay_columns)
        if self.replay_columns < 1:
            raise _lib.TorchBeastB200Error("replay_columns must be at least 1, got %d" % self.replay_columns)
        if self.replay_columns > 4096:  # TB_REPLAY_MAX_R
            raise _lib.TorchBeastB200Error("replay_columns must be at most 4096, got %d" % self.replay_columns)
        if self.capacity < 2:
            raise _lib.TorchBeastB200Error("capacity must be at least 2, got %d" % self.capacity)
        self.min_size = self.replay_columns if min_size is None else int(min_size)
        if not 1 <= self.min_size < self.capacity:
            raise _lib.TorchBeastB200Error("min_size must be in [1, capacity - Bf], got %d for capacity %d"
                                           % (self.min_size, self.capacity))
        self.seed = int(seed)
        self.step = 0
        self.stream_id = stream_id
        self.device = None if device is None else torch.device(device)
        self.head = 0
        self.size = 0
        self.spec = None          # (Bf, ((name, outer, row shape, dtype), ...)) of the first batch
        self.rings = None         # one [capacity, outer, *row] tensor per leaf
        self.state = None         # int64 [4] device: head, size, seed, step
        self.last_slots = None    # int64 [R] device: the slots of the last mixing call's replayed columns
        self._published = None    # (seed, step) the device holds once the enqueued calls have run

    # ---- column spec ------------------------------------------------------------------------------------------------
    @staticmethod
    def _leaves(batch, state):
        from torchbeast_b200.learner import GraphedLearner
        named = [(k, batch[k]) for k in GraphedLearner.KEYS if k in batch]
        return named + [("agent_state%d" % i, s) for i, s in enumerate(state)]

    def _spec_of(self, batch, state):
        leaves = self._leaves(batch, state)
        Bf = batch["frame"].shape[1] if batch["frame"].dim() >= 2 else 0
        for k, t in leaves:
            if t.dim() < 2 or t.shape[1] != Bf:
                raise _lib.TorchBeastB200Error("replay: every leaf must be [outer, B, ...] with B = %d, got %s %r"
                                               % (Bf, k, tuple(t.shape)))
        return Bf, tuple((k, t.shape[0], tuple(t.shape[2:]), t.dtype) for k, t in leaves)

    def prepare(self, batch, state=()):
        """Check `batch` / `state` against the buffer's column spec (allocating the ring on the first call) and enqueue
        the copy of `seed` / `step` to the device if they were changed on the host.  Returns Bf.  Not capturable."""
        spec = self._spec_of(batch, state)
        Bf = spec[0]
        if self.spec is None:
            if Bf < 1 or self.capacity <= Bf:
                raise _lib.TorchBeastB200Error("replay: capacity (%d) must exceed the fresh batch width (%d)"
                                               % (self.capacity, Bf))
            if self.min_size > self.capacity - Bf:
                raise _lib.TorchBeastB200Error("replay: min_size must be in [1, capacity - Bf] = [1, %d], got %d"
                                               % (self.capacity - Bf, self.min_size))
            dev = self.device or batch["frame"].device
            _lib.require_cuda(torch.empty(0, device=dev))
            if self.stream_id is None:
                self.stream_id = _dp_rank()
            if not 0 <= int(self.stream_id) < 2 ** 32:
                raise _lib.TorchBeastB200Error("replay: stream_id must be in [0, 2^32), got %d" % self.stream_id)
            # zeros, not empty: the never-written slots then compare equal between runs
            self.rings = [torch.zeros((self.capacity, outer) + row, dtype=dt, device=dev) for _, outer, row, dt in spec[1]]
            self.state = torch.zeros(4, dtype=torch.int64, device=dev)
            self.device, self.spec = dev, spec
        elif spec != self.spec:
            raise _lib.TorchBeastB200Error("replay: the batch columns changed from %r to %r" % (self.spec, spec))
        for _, t in self._leaves(batch, state):
            if t.device != self.device:
                raise _lib.TorchBeastB200Error("replay: batch leaves must be on %s, got %s" % (self.device, t.device))
        want = (self.seed % 2 ** 64, self.step % 2 ** 64)
        if self._published != want:
            # a fresh pinned buffer, as learner.publish_hparams: not handed out again until the copy is done
            host = torch.tensor([_i64(want[0]), _i64(want[1])], dtype=torch.int64).pin_memory()
            self.state[2:].copy_(host, non_blocking=True)
            self._published = want
        return Bf

    def mixing(self, Bf):
        """Whether a call with Bf fresh columns draws replayed columns: n = min(size, capacity - Bf) >= min_size."""
        return min(self.size, self.capacity - Bf) >= self.min_size

    # ---- device calls -----------------------------------------------------------------------------------------------
    def launch(self, batch, state, mixing):
        """Enqueue tb_replay_mix + tb_replay_advance on the current stream (capturable; the host mirror is not touched).
        mixing: returns the mixed (batch, state) of width Bf + R, else inserts only and returns the inputs."""
        Bf, leaves_spec = self.spec
        R = self.replay_columns if mixing else 0
        fresh = [t.contiguous() for _, t in self._leaves(batch, state)]
        outs = [torch.empty((t.shape[0], Bf + R) + tuple(t.shape[2:]), dtype=t.dtype, device=t.device) if mixing else None
                for t in fresh]
        slots = torch.empty(R, dtype=torch.int64, device=self.device) if mixing else None
        table = (_Leaf * len(fresh))(*[
            _Leaf(f.data_ptr(), 0 if o is None else o.data_ptr(), r.data_ptr(), f.shape[0],
                  f[0, 0].numel() * f.element_size())
            for f, o, r in zip(fresh, outs, self.rings)])
        p = _lib.ptr
        _lib.check(_lib.lib().tb_replay_mix(table, len(fresh), Bf, R, self.capacity, p(self.state[2:]),
                                            p(self.state[:2]), int(self.stream_id), p(slots), _lib.stream_ptr()),
                   "tb_replay_mix")
        _lib.check(_lib.lib().tb_replay_advance(p(self.state[:2]), p(self.state[2:]), Bf, self.capacity,
                                                _lib.stream_ptr()),
                   "tb_replay_advance")
        if not mixing:
            return batch, state
        self.last_slots = slots
        names = [k for k, _, _, _ in leaves_spec]
        n_state = len(state)
        mixed = dict(zip(names[:len(names) - n_state], outs[:len(outs) - n_state]))
        return mixed, tuple(outs[len(outs) - n_state:])

    def advance_host(self, Bf):
        """The host mirror of tb_replay_advance."""
        self.head = (self.head + Bf) % self.capacity
        self.size = min(self.size + Bf, self.capacity)
        self.step += 1
        self._published = (self.seed % 2 ** 64, self.step % 2 ** 64)

    def mix(self, batch, state=()):
        """One eager call: returns (batch, state, fresh_columns).  While mixing, batch / state are the mixed [.., Bf+R, ..]
        leaves and fresh_columns = Bf; during warm-up they are the inputs unchanged and fresh_columns is None."""
        Bf = self.prepare(batch, state)
        mixing = self.mixing(Bf)
        batch, state = self.launch(batch, state, mixing)
        self.advance_host(Bf)
        return batch, tuple(state), (Bf if mixing else None)

    # ---- GraphedLearner's throw-away runs ---------------------------------------------------------------------------
    def save(self, calls):
        """Device copies of the state and of every slot the next `calls` calls overwrite (enqueued on the current
        stream); restore() puts them back.  Cheaper than copying the ring, and exact: a call writes only its Bf slots."""
        Bf = self.spec[0]
        idx = (self.head + torch.arange(min(calls * Bf, self.capacity), device=self.device)) % self.capacity
        return self.state.clone(), idx, [r.index_select(0, idx) for r in self.rings]

    def restore(self, saved):
        state, idx, rows = saved
        self.state.copy_(state)
        for r, v in zip(self.rings, rows):
            r.index_copy_(0, idx, v)

    def __repr__(self):
        return "ReplayBuffer(capacity=%d, replay_columns=%d, seed=%d, step=%d, size=%d)" % (
            self.capacity, self.replay_columns, self.seed, self.step, self.size)
