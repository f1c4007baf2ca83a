"""CPU: the replay slot rule (tests/replay_oracle.py) never draws a slot its own call overwrites and draws uniformly over
the survivors; the buffer's host mirror and warm-up follow the rule; bad arguments are rejected on the host."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

from tests import replay_oracle as RO


@pytest.mark.parametrize("capacity,Bf,R", [(6, 5, 8), (37, 5, 16), (40, 8, 8), (23, 7, 32), (1000, 32, 16)])
def test_slots_never_overwritten_and_always_valid(capacity, Bf, R):
    head = size = step = 0
    for call in range(3 * capacity // Bf + 5):   # through several wrap-arounds
        n = RO.survivors(size, capacity, Bf)
        if n >= 1:
            s = RO.slots(R, head, size, capacity, Bf, seed=11, step=step, stream_id=call % 3)
            assert s.dtype == np.int64 and s.shape == (R,)
            assert not set(s.tolist()) & set(RO.overwritten(head, capacity, Bf).tolist())
            newest = {(head - 1 - k) % capacity for k in range(n)}       # the n newest stored columns
            assert set(s.tolist()) <= newest
        head, size, step = RO.advance(head, size, step, capacity, Bf)
    assert size == capacity


def test_one_survivor():
    # capacity = Bf + 1: once full, every draw is the newest column
    capacity, Bf = 9, 8
    s = RO.slots(64, head=3, size=capacity, capacity=capacity, Bf=Bf, seed=5, step=17, stream_id=0)
    assert (s == 2).all()


def test_uniform_over_survivors_chi_square():
    capacity, Bf, R = 37, 5, 64
    n = capacity - Bf
    counts = np.zeros(n)
    head = 4
    for step in range(320):                         # 20480 draws
        s = RO.slots(R, head, capacity, capacity, Bf, seed=1234, step=step, stream_id=0)
        counts += np.bincount((head - 1 - s) % capacity, minlength=n)
    expected = counts.sum() / n
    chi2 = float(np.sum((counts - expected) ** 2 / expected))
    assert chi2 < stats.chi2.ppf(0.999, n - 1), chi2


def test_stream_ids_and_steps_draw_differently():
    a = RO.slots(32, 10, 100, 100, 8, seed=1, step=0, stream_id=0)
    assert not np.array_equal(a, RO.slots(32, 10, 100, 100, 8, seed=1, step=0, stream_id=1))
    assert not np.array_equal(a, RO.slots(32, 10, 100, 100, 8, seed=1, step=1, stream_id=0))
    assert not np.array_equal(a, RO.slots(32, 10, 100, 100, 8, seed=2, step=0, stream_id=0))
    assert np.array_equal(a, RO.slots(32, 10, 100, 100, 8, seed=1, step=0, stream_id=0))


@pytest.mark.parametrize("capacity,Bf,R,min_size", [(10, 4, 2, None), (10, 4, 3, 6), (13, 5, 8, 1), (6, 5, 4, 1)])
def test_host_mirror_and_warm_up_follow_the_rule(capacity, Bf, R, min_size):
    from torchbeast_b200.replay import ReplayBuffer
    buf = ReplayBuffer(capacity, R, seed=3, min_size=min_size)
    m = R if min_size is None else min_size
    head = size = step = 0
    phases = []
    for _ in range(12):
        assert buf.mixing(Bf) == RO.mixing(size, capacity, Bf, m) == (min(size, capacity - Bf) >= m)
        phases.append(buf.mixing(Bf))
        buf.advance_host(Bf)
        head, size, step = RO.advance(head, size, step, capacity, Bf)
        assert (buf.head, buf.size, buf.step) == (head, size, step)
    # warm-up, then mixing for good
    assert phases[0] is False and phases[-1] is True
    assert phases == sorted(phases)


def test_constructor_validation():
    from torchbeast_b200._lib import TorchBeastB200Error
    from torchbeast_b200.replay import ReplayBuffer
    with pytest.raises(TorchBeastB200Error, match="replay_columns"):
        ReplayBuffer(100, 0)
    with pytest.raises(TorchBeastB200Error, match="replay_columns"):
        ReplayBuffer(100, -3)
    with pytest.raises(TorchBeastB200Error, match="min_size"):
        ReplayBuffer(100, 8, min_size=0)
    with pytest.raises(TorchBeastB200Error, match="min_size"):
        ReplayBuffer(100, 8, min_size=100)
    with pytest.raises(TorchBeastB200Error, match="capacity"):
        ReplayBuffer(1, 1)


def _batch(T, B, A=6):
    return dict(frame=torch.zeros(T + 1, B, 4, 84, 84, dtype=torch.uint8), reward=torch.zeros(T + 1, B),
                done=torch.zeros(T + 1, B, dtype=torch.bool), policy_logits=torch.zeros(T + 1, B, A),
                action=torch.zeros(T + 1, B, dtype=torch.int64), episode_return=torch.zeros(T + 1, B))


def test_first_call_validation():
    from torchbeast_b200._lib import TorchBeastB200Error
    from torchbeast_b200.replay import ReplayBuffer
    with pytest.raises(TorchBeastB200Error, match="capacity"):
        ReplayBuffer(8, 2).prepare(_batch(2, 8))               # capacity must exceed Bf
    with pytest.raises(TorchBeastB200Error, match="min_size"):
        ReplayBuffer(10, 2, min_size=7).prepare(_batch(2, 4))  # min_size > capacity - Bf
    bad = _batch(2, 4)
    bad["reward"] = torch.zeros(3, 5)
    with pytest.raises(TorchBeastB200Error, match="every leaf"):
        ReplayBuffer(10, 2).prepare(bad)
    with pytest.raises(TorchBeastB200Error, match="CUDA tensors only"):
        ReplayBuffer(10, 2).prepare(_batch(2, 4))               # there is no host replay path


def test_entry_points_validate_on_the_host():
    from torchbeast_b200 import _lib
    from torchbeast_b200.replay import _Leaf
    h = _lib.lib()
    dev = ctypes.c_void_p(256)   # never dereferenced: every check below fails before a launch
    leaves = (_Leaf * 2)(_Leaf(256, 512, 1024, 3, 16), _Leaf(256, None, 1024, 3, 4))

    def mix(lv=leaves, n=2, Bf=4, R=2, cap=10, ss=dev, hs=dev, sid=0):
        rc = h.tb_replay_mix(lv, n, Bf, R, cap, ss, hs, sid, None, None)
        assert rc != 0
        return h.tb_last_error().decode()

    assert "null pointer" in mix(lv=None)
    assert "null pointer" in mix(ss=None)
    assert "null pointer" in mix(hs=None)
    assert "num_leaves" in mix(n=0)
    assert "num_leaves" in mix(n=17)
    assert "R must be" in mix(R=-1)
    assert "R must be" in mix(R=4097)
    assert "Bf must be" in mix(Bf=0)
    assert "capacity" in mix(cap=4)
    assert "stream_id" in mix(sid=-1)
    assert "stream_id" in mix(sid=2 ** 32)
    assert "null pointer in leaf 1" in mix(lv=(_Leaf * 2)(_Leaf(256, 512, 1024, 3, 16), _Leaf(256, None, None, 3, 4)))
    assert "null pointer in leaf 0" in mix(lv=(_Leaf * 1)(_Leaf(None, 512, 1024, 3, 16)), n=1)
    assert "outer >= 1" in mix(lv=(_Leaf * 1)(_Leaf(256, 512, 1024, 0, 16)), n=1)
    assert "row_bytes >= 1" in mix(lv=(_Leaf * 1)(_Leaf(256, 512, 1024, 3, 0)), n=1)
    assert h.tb_replay_advance(None, dev, 4, 10, None) != 0 and b"null pointer" in h.tb_last_error()
    assert h.tb_replay_advance(dev, None, 4, 10, None) != 0 and b"null pointer" in h.tb_last_error()
    assert h.tb_replay_advance(dev, dev, 0, 10, None) != 0 and b"Bf must be" in h.tb_last_error()
    assert h.tb_replay_advance(dev, dev, 4, 4, None) != 0 and b"capacity" in h.tb_last_error()
