"""NumPy restatement of unstacked rollouts (include/torchbeast_b200.h, "unstacked rollouts").

`restack` is the format contract written out as indexing.  `simulate` plays the reference's actor side -
core/environment.py (done = 1 on the first frame of every episode, including initial()) in front of
atari_wrappers.FrameStack(k=4) (reset fills all four slots with that frame) - and `rollout` cuts the same steps out of
its output once as stacked frames and once as the unstacked rows an actor writes, so tests can check the first
against `restack` of the second.
"""
import collections

import numpy as np


def restack(frames, done):
    """frames u8 [T1+3, B, ...], done [T1, B] (any non-zero value starts an episode) -> stacks [T1, B, 4, ...]:
    stack[t, b, c] = frames[3 + max(t - 3 + c, last_done(t, b)), b], last_done = largest s <= t with done[s, b], else -3."""
    done = np.asarray(done) != 0
    T1, B = done.shape
    assert frames.shape[:2] == (T1 + 3, B), (frames.shape, done.shape)
    out = np.empty((T1, B, 4) + frames.shape[2:], dtype=frames.dtype)
    last = np.full(B, -3)
    cols = np.arange(B)
    for t in range(T1):
        last = np.where(done[t], t, last)
        for c in range(4):
            out[t, :, c] = frames[3 + np.maximum(t - 3 + c, last), cols]
    return out


def simulate(steps, B, seed=0, done_prob=0.05, hw=(84, 84), done=None):
    """Environment + FrameStack(4) for `steps` steps of B independent columns.  `done` [steps, B] (optional) fixes
    which steps start an episode; step 0 always does (initial()).  Returns (stacks u8 [steps, B, 4, *hw],
    done bool [steps, B])."""
    rs = np.random.RandomState(seed)
    if done is None:
        done = rs.rand(steps, B) < done_prob
    done = np.array(done, dtype=bool).reshape(steps, B)
    done[0] = True
    obs = rs.randint(0, 256, size=(steps, B) + tuple(hw)).astype(np.uint8)
    stacks = np.empty((steps, B, 4) + tuple(hw), dtype=np.uint8)
    for b in range(B):
        slots = collections.deque(maxlen=4)
        for s in range(steps):
            if done[s, b]:
                slots.extend([obs[s, b]] * 4)   # FrameStack.reset on the episode's first frame
            else:
                slots.append(obs[s, b])         # FrameStack.step
            stacks[s, b] = np.stack(slots)
    return stacks, done


def unstack(stacks):
    """What an actor writes for a rollout of stacks [T1, B, 4, ...]: its step-0 stack's first three channels, then the
    newest frame of every step -> [T1+3, B, ...]."""
    return np.concatenate([np.swapaxes(stacks[0, :, :3], 0, 1), stacks[:, :, 3]], axis=0)


def rollout(stacks, done, start, T1):
    """Steps [start, start + T1) of a simulated stream in both formats: (stacked [T1, B, 4, ...], unstacked
    [T1+3, B, ...], done [T1, B]).  Consecutive rollouts share a row (start = previous start + T1 - 1), as the
    learner queue delivers them."""
    st = stacks[start:start + T1]
    return st, unstack(st), done[start:start + T1]
