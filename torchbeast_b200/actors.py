"""Synthetic actor pool + learner queue: BASELINE.json configs[2] ("polybeast_learner 48 synthetic actors").

Stands in for the reference's ActorPool loops + BatchingQueue (/root/reference/src/cc/actorpool.cc:342-470 actor loop,
:147-186 dequeue_many, :493-506 the rollout nest) WITHOUT environments, gRPC or inference: `num_actors` host threads each
produce `[T+1, ...]` rollouts of synthetic 84x84x4 uint8 frames and write them straight into one batch column of a
PINNED `[T+1, B, ...]` slot of a RolloutStager (N1: no per-rollout tensors, no torch.cat, no pageable copy); a slot
whose B columns are complete is handed to the learner threads through `LearnerQueue` as the reference's nest
`((env_outputs, actor_outputs), initial_agent_state)` (SURVEY 8(b) B2) whose leaves ARE the slot's tensors, so
polybeast_learner.learn() submits it with one async H2D copy.  Row 0 of every rollout repeats the last row of that
actor's previous rollout (actorpool.cc:443).  Out of scope: real environments / inference (SURVEY section 2).

Frames and `done` come from synthetic environment streams that follow the reference's actor side: done = 1 on the first
frame of every episode (core/environment.py), and FrameStack(4) fills all four slots with that frame.  frame_format=
"unstacked" hands over the same steps as one newest frame per step (staging.spec_for(..., frame_format="unstacked")), so
one seed gives the same stacks in both formats."""
import collections
import queue
import threading

import numpy as np
import torch


class LearnerQueue:
    """Iterator protocol of the reference's BatchingQueue as polybeast_learner.learn uses it (pl:306, 380)."""

    def __init__(self, maxsize=0):
        self._q = queue.Queue(maxsize)
        self._closed = False

    def put(self, item):
        self._q.put(item)

    def close(self):
        self._closed = True
        self._q.put(None)

    def size(self):
        return self._q.qsize()

    def __iter__(self):
        return self

    def __next__(self):
        item = self._q.get()
        if item is None:
            self._q.put(None)  # wake the other learner threads too
            raise StopIteration
        return item


def _frame_stream(rs, steps, done_prob=0.01, hw=(84, 84)):
    """One column's environment stream as a cycle: (stacks u8 [steps, 4, *hw], done bool [steps]).  Step 0 starts an
    episode (initial()); the last step starts one on step 0's frame again, so its stack equals step 0's and the stream
    can be handed over round and round with row 0 of each rollout repeating the previous rollout's last row."""
    obs = rs.randint(0, 256, size=(steps,) + tuple(hw), dtype=np.uint8)
    done = rs.rand(steps) < done_prob
    done[0] = done[-1] = True
    obs[-1] = obs[0]
    stacks = np.empty((steps, 4) + tuple(hw), dtype=np.uint8)
    slots = collections.deque(maxlen=4)
    for s in range(steps):
        if done[s]:
            slots.extend([obs[s]] * 4)  # FrameStack.reset
        else:
            slots.append(obs[s])        # FrameStack.step
        stacks[s] = np.stack(slots)
    return torch.from_numpy(stacks), torch.from_numpy(done)


class SyntheticActors:
    POOL = 4  # rollouts each actor hands over in turn

    def __init__(self, stager, num_actors, T, B, num_actions, learner_queue, state_shape=None, seed=0, frame_pool=8,
                 frame_format="stacked"):
        if frame_format not in ("stacked", "unstacked"):
            raise ValueError("frame_format must be 'stacked' or 'unstacked', got %r" % (frame_format,))
        self.frame_format = frame_format
        self.stager, self.n, self.T, self.B, self.A = stager, num_actors, T, B, num_actions
        self.queue = learner_queue
        self.state_shape = state_shape  # (layers, H) or None
        self._lock = threading.Lock()        # column counters / statistics
        self._claim_lock = threading.Lock()  # column hand-out (may block waiting for a free slot: never held with _lock)
        self._slot = None
        self._next_col = 0
        self._remaining = {}
        self._stop = False
        self._threads = []
        self.rollouts = 0
        rs = np.random.RandomState(seed)
        # `frame_pool` environment streams, each cut into POOL chained rollouts; actor k hands over those of stream
        # k % frame_pool.  The host work per rollout is the copy into the pinned column, as it is for a real actor handing
        # over frames it received from its environment.
        T1 = T + 1
        self._rollout_frames, self._rollout_done = [], []
        for _ in range(frame_pool):
            stacks, done = _frame_stream(rs, self.POOL * T + 1)
            rolls = [stacks[j * T:j * T + T1] for j in range(self.POOL)]
            if frame_format == "unstacked":
                rolls = [torch.cat([r[0, :3], r[:, 3]]) for r in rolls]
            self._rollout_frames.append(rolls)
            self._rollout_done.append([done[j * T:j * T + T1] for j in range(self.POOL)])
        self._seed = seed

    def _claim(self):
        """(slot index, column) for the next rollout; blocks while every slot is in flight."""
        with self._claim_lock:
            if self._slot is None:
                i = self.stager.acquire_host(timeout=0.5)
                with self._lock:
                    self._remaining[i] = self.B
                self._slot = i
                self._next_col = 0
            i, b = self._slot, self._next_col
            self._next_col += 1
            if self._next_col == self.B:
                self._slot = None
            return i, b

    def _done(self, i):
        with self._lock:
            self._remaining[i] -= 1
            full = self._remaining[i] == 0
            if full:
                del self._remaining[i]
        if full:
            h = self.stager.host[i]
            env = (h["frame"], h["reward"], h["done"], h["episode_step"], h["episode_return"])
            agent = (h["action"], h["policy_logits"], h["baseline"])
            state = ()
            if self.state_shape is not None:
                layers, H = self.state_shape
                state = tuple(torch.zeros(layers, self.B, H) for _ in range(2))
            self.queue.put(((env, agent), state))

    def _make_pool(self, k):
        """A few pre-generated rollouts per actor (what its environment steps would have produced): the per-rollout host work
        that remains is the hand-over into the pinned column, as for a real actor."""
        rs = np.random.RandomState(self._seed * 1000 + k)
        T1, A, pool = self.T + 1, self.A, self.POOL
        stream = k % len(self._rollout_frames)
        out = []
        for j in range(pool):
            out.append(dict(
                frame=self._rollout_frames[stream][j],
                reward=torch.from_numpy(rs.randn(T1).astype(np.float32)),
                done=self._rollout_done[stream][j],
                episode_return=torch.from_numpy(rs.randn(T1).astype(np.float32)),
                episode_step=torch.from_numpy(rs.randint(0, 1000, size=T1).astype(np.int32)),
                policy_logits=torch.from_numpy(rs.randn(T1, A).astype(np.float32)),
                baseline=torch.from_numpy(rs.randn(T1).astype(np.float32)),
                action=torch.from_numpy(rs.randint(0, A, size=T1).astype(np.int64))))
        # row 0 of a rollout = last row of this actor's previous rollout (actorpool.cc:443): the pool is handed over cyclically,
        # so that overlap is baked in once (the shared frame / done streams are cycles that already have it)
        for j in range(pool):
            prev = out[(j - 1) % pool]
            for key, v in out[j].items():
                if key not in ("frame", "done"):
                    v[0].copy_(prev[key][-1])
        return [self.stager.prepare_rollout(r) for r in out]

    def _actor(self, k):
        pool = self._make_pool(k)
        n = 0
        while not self._stop:
            try:
                i, b = self._claim()
            except TimeoutError:
                continue
            self.stager.write_prepared(i, b, pool[n % len(pool)])   # ONE native, GIL-free call copies all leaves into the column
            n += 1
            with self._lock:
                self.rollouts += 1
            self._done(i)

    def start(self):
        for k in range(self.n):
            t = threading.Thread(target=self._actor, args=(k,), daemon=True)
            t.start()
            self._threads.append(t)

    def stop(self):
        self._stop = True
        self.queue.close()
