"""Learner-queue ingest: pinned host ring -> device slots (SURVEY.md 8(f) N1).

Replaces the reference's `BatchingQueue.dequeue_many` + `torch::cat(dim=1)` + pageable `t.to(device)`
(/root/reference/src/cc/actorpool.cc:49-55,147-186,444-447; torchbeast/polybeast_learner.py:307): instead of
concatenating B per-actor rollouts into a fresh pageable tensor and copying that synchronously, every actor
writes its `[T+1, ...]` rollout straight into column b of a PINNED `[T+1, B, ...]` slot (`column(slot, b)`),
and a full slot goes to the GPU as ONE asynchronous copy on a dedicated stream (all leaves of a slot are carved
from one pinned allocation at the offsets of one device allocation), double-buffered so the copy of rollout
i+1 overlaps the learner step on rollout i.  The same layout the reference delivers (SURVEY 8(b) B2): leaves are
`[T+1, B, ...]`, time-major, contiguous; row 0 of a rollout is the last row of that actor's previous rollout.

    stager = RolloutStager(spec_for(T, B, A, use_last_action=True), device)
    i = stager.acquire_host()            # a free pinned slot (blocks only if all `depth` slots are in flight)
    stager.column(i, b)["frame"][...] = ...   # per-actor writes, any thread
    stager.submit(i)                     # async H2D on the copy stream
    dev, j = stager.get()                # oldest submitted slot, ready-event waited on the CURRENT stream
    ... learn on dev ...
    stager.release(j)                    # after the consumer's last kernel was enqueued
`put(batch)` is the drop-in path for a caller that already holds a [T+1, B, ...] host batch (the reference's nest):
copies it into a pinned slot (no-op for leaves that already ARE that slot's tensors) and submits it.
"""
import collections
import threading

import torch

from torchbeast_b200 import _lib, action_space

LEAF_ORDER = ("frame", "reward", "done", "episode_return", "episode_step", "policy_logits", "baseline", "action", "last_action")


FRAME_FORMATS = ("stacked", "unstacked")


def spec_for(T, B, num_actions, use_last_action=True, frame_shape=(4, 84, 84), extra=(), frame_format="stacked",
             frame_dtype=torch.uint8):
    """Leaf name -> (shape, dtype) of one [T+1, B, ...] rollout batch (monobeast.py:299-316 buffers / the B2 nest).
    frame_format="unstacked": the frame leaf is [T+4, B, H, W], one newest frame per step after step 0's first three
    channels; the learner rebuilds the stacks on the GPU (include/torchbeast_b200.h, "unstacked rollouts").
    num_actions a tuple (A_1, ..., A_D): a factored action space (torchbeast_b200.action_space), whose policy_logits
    are [T+1, B, sum A_k] and whose action and last_action are [T+1, B, D].  num_actions a Gaussian(D): a continuous
    space, whose policy_logits are the (mu, log sigma) rows [T+1, B, 2D] and whose action and last_action are float32
    [T+1, B, D].  frame_dtype: the frame leaf's dtype, e.g. torch.float32 with frame_shape=(O,) for an MLPNet's
    observation vectors."""
    dims = action_space.dims_of(num_actions)
    D = action_space.continuous_dim_of(num_actions)
    act = (T + 1, B) if dims is None else (T + 1, B, len(dims))
    act_dtype = torch.int64
    if D is not None:
        act, act_dtype = (T + 1, B, D), torch.float32
    num_actions = action_space.width(num_actions)
    if frame_format not in FRAME_FORMATS:
        raise ValueError("frame_format must be one of %s, got %r" % (FRAME_FORMATS, frame_format))
    T1 = T + 1
    frame = (T1, B) + tuple(frame_shape) if frame_format == "stacked" else (T1 + 3, B) + tuple(frame_shape[1:])
    spec = collections.OrderedDict(
        frame=(frame, frame_dtype),
        reward=((T1, B), torch.float32),
        done=((T1, B), torch.bool),
        episode_return=((T1, B), torch.float32),
        episode_step=((T1, B), torch.int32),
        policy_logits=((T1, B, num_actions), torch.float32),
        baseline=((T1, B), torch.float32),
        action=(act, act_dtype),
    )
    if use_last_action:
        spec["last_action"] = (act, act_dtype)
    for name, shape, dtype in extra:
        spec[name] = (tuple(shape), dtype)
    return spec


def spec_like(batch):
    return collections.OrderedDict((k, (tuple(v.shape), v.dtype)) for k, v in batch.items())


def _carve(spec):
    """Byte offsets of every leaf inside one slot allocation (256-byte aligned) and the slot size."""
    offs, off = {}, 0
    for name, (shape, dtype) in spec.items():
        n = 1
        for d in shape:
            n *= d
        nbytes = n * torch.empty((), dtype=dtype).element_size()
        offs[name] = (off, nbytes)
        off += (nbytes + 255) & ~255
    return offs, off


class RolloutStager:
    def __init__(self, spec, device, depth=2):
        if depth < 1:
            raise ValueError("depth must be >= 1")
        self.spec = collections.OrderedDict(spec)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.TorchBeastB200Error("RolloutStager stages onto a CUDA device")
        self.depth = depth
        self._offs, self.slot_bytes = _carve(self.spec)
        self._host_raw = [torch.empty(self.slot_bytes, dtype=torch.uint8).pin_memory() for _ in range(depth)]
        self._dev_raw = [torch.empty(self.slot_bytes, dtype=torch.uint8, device=self.device) for _ in range(depth)]
        self.host = [self._views(r) for r in self._host_raw]
        self.dev = [self._views(r) for r in self._dev_raw]
        self.h2d_bytes = sum(n for _, n in self._offs.values())
        self._stream = torch.cuda.Stream(device=self.device)
        self._ready = [torch.cuda.Event() for _ in range(depth)]     # H2D of slot i finished (recorded on the copy stream)
        self._freed = [torch.cuda.Event() for _ in range(depth)]     # consumer of device slot i is done (compute stream)
        self._copied = [torch.cuda.Event() for _ in range(depth)]    # host slot i may be rewritten
        self._lock = threading.Condition()
        self._free_host = collections.deque(range(depth))
        self._submitted = collections.deque()
        self._in_use = set()
        for e in self._freed:
            e.record()

    def _views(self, raw):
        out = collections.OrderedDict()
        for name, (shape, dtype) in self.spec.items():
            off, nbytes = self._offs[name]
            out[name] = raw[off:off + nbytes].view(dtype).view(shape)
        return out

    # ---- producer side -------------------------------------------------------------------------
    def acquire_host(self, timeout=None):
        """Index of a pinned slot nobody is writing, copying or training on."""
        with self._lock:
            if not self._lock.wait_for(lambda: len(self._free_host) > 0, timeout=timeout):
                raise TimeoutError("RolloutStager: no free slot (consumer stalled?)")
            i = self._free_host.popleft()
        self._copied[i].synchronize()  # its previous H2D has drained: the host memory may be overwritten
        return i

    def column(self, i, b):
        """Views `[T+1, ...]` of batch column b of host slot i: what ONE actor fills (actorpool.cc:493-506 per rollout).
        With an unstacked spec the frame view is `[T+4, H, W]`: rows 0..3 = the four channels of the stack at the rollout's
        first step, row 3+t = the newest frame of step t (include/torchbeast_b200.h, "unstacked rollouts")."""
        return collections.OrderedDict((k, v[:, b]) for k, v in self.host[i].items())

    def prepare_rollout(self, rollout, what="prepare_rollout"):
        """Pre-built argument block for write_prepared() when the same host arrays are handed over repeatedly (a fixed pool
        of synthetic rollouts): keeps the per-rollout Python work to one C call per distinct leaf row count (one call; two
        with an unstacked frame leaf, whose T+4 rows differ from the other leaves' T+1)."""
        import ctypes
        names = [k for k in self.spec if k in rollout]
        for k in names:
            t = rollout[k]
            if t.is_cuda or not t.is_contiguous() or t.dtype != self.spec[k][1] or \
                    t.numel() * t.element_size() != self._offs[k][1] // self.spec[k][0][1]:
                raise _lib.TorchBeastB200Error("%s: leaf %r must be a contiguous CPU [%d, ...] tensor of the slot's dtype"
                                               % (what, k, self.spec[k][0][0]))
        groups = collections.OrderedDict()  # leaf row count -> leaf names
        for k in names:
            groups.setdefault(self.spec[k][0][0], []).append(k)
        calls = []
        for rows_t, ks in groups.items():
            n, B = len(ks), self.spec[ks[0]][0][1]
            offs = (ctypes.c_int64 * n)(*[self._offs[k][0] for k in ks])
            rows = (ctypes.c_int64 * n)(*[self._offs[k][1] // (rows_t * B) for k in ks])
            srcs = (ctypes.c_void_p * n)(*[rollout[k].data_ptr() for k in ks])
            calls.append((ctypes.cast(offs, ctypes.c_void_p), ctypes.cast(rows, ctypes.c_void_p), n, rows_t, B,
                          ctypes.cast(srcs, ctypes.c_void_p), (offs, rows, srcs)))
        return calls, rollout  # keep the arrays and tensors alive

    def write_prepared(self, i, b, prep):
        import ctypes
        base = ctypes.c_void_p(self._host_raw[i].data_ptr())
        for offs, rows, n, T, B, srcs, _keep in prep[0]:
            rc = _lib.lib().tb_host_write_rollout_column(base, offs, rows, n, T, B, int(b), srcs)
            if rc:
                _lib.check(rc, "tb_host_write_rollout_column")

    def write_column(self, i, b, rollout):
        """Native per-actor hand-over: copy `rollout` (dict leaf -> contiguous [T+1, ...] CPU tensor; [T+4, ...] for an
        unstacked frame leaf) into column b of pinned slot i with native calls (tb_host_write_rollout_column) that run
        without the GIL - N actor threads then copy in parallel instead of serialising on the interpreter."""
        self.write_prepared(i, b, self.prepare_rollout(rollout, "write_column"))

    def submit(self, i):
        """Slot i is complete: one async H2D copy of the whole slot on the copy stream."""
        with torch.cuda.stream(self._stream):
            self._stream.wait_event(self._freed[i])          # the previous consumer of device slot i is done with it
            self._dev_raw[i].copy_(self._host_raw[i], non_blocking=True)
            self._ready[i].record(self._stream)
            self._copied[i].record(self._stream)
        with self._lock:
            self._submitted.append(i)
            self._lock.notify_all()

    def put(self, batch, timeout=None):
        """Stage a host batch (dict of [T+1, B, ...] CPU tensors, pinned or pageable): memcpy into a pinned slot unless the
        leaves already are that slot's own tensors, then submit.  Returns the slot index."""
        for i in range(self.depth):  # filled in place by the caller?
            h = self.host[i]
            if all(k in batch and batch[k].data_ptr() == h[k].data_ptr() for k in h if k in batch) and \
                    any(k in batch for k in h):
                with self._lock:
                    if i in self._free_host:
                        self._free_host.remove(i)
                self.submit(i)
                return i
        i = self.acquire_host(timeout)
        h = self.host[i]
        for k, dst in h.items():
            if k in batch:
                dst.copy_(batch[k])
        self.submit(i)
        return i

    # ---- consumer side -------------------------------------------------------------------------
    def get(self, timeout=None):
        """(device batch dict, slot index) of the oldest submitted slot; the CURRENT stream waits for its copy."""
        with self._lock:
            if not self._lock.wait_for(lambda: len(self._submitted) > 0, timeout=timeout):
                raise TimeoutError("RolloutStager: nothing submitted")
            i = self._submitted.popleft()
            self._in_use.add(i)
        torch.cuda.current_stream(self.device).wait_event(self._ready[i])
        return self.dev[i], i

    def release(self, i):
        """The consumer has enqueued its last use of device slot i on the current stream."""
        self._freed[i].record(torch.cuda.current_stream(self.device))
        with self._lock:
            self._in_use.discard(i)
            self._free_host.append(i)
            self._lock.notify_all()

    def stage(self, batch):
        """put + get in one call (single-threaded callers: correct, but nothing to overlap with)."""
        self.put(batch)
        return self.get()
