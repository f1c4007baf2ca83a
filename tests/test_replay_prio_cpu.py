"""CPU: the prioritised replay rule of tests/replay_prio_oracle.py (draws proportional to q = (p + eps)^alpha over the
survivors, importance weights, the priority update) and the host-side validation of the prioritised entry points."""
import ctypes

import numpy as np
import pytest
from scipy import stats

from tests import replay_oracle as RO
from tests import replay_prio_oracle as PO


def _priorities(capacity, seed):
    return np.random.RandomState(seed).gamma(0.7, size=capacity).astype(np.float32)


@pytest.mark.parametrize("capacity,Bf,R", [(6, 5, 8), (37, 5, 16), (40, 8, 8), (1000, 32, 16), (3000, 16, 64)])
def test_draws_are_survivors_and_never_overwritten(capacity, Bf, R):
    pr = _priorities(capacity, capacity)
    head = size = step = 0
    for call in range(3 * capacity // Bf + 5):
        if RO.survivors(size, capacity, Bf) >= 1:
            s, w, _ = PO.prioritized(pr, R, head, size, capacity, Bf, seed=11, step=step, stream_id=call % 3,
                                     alpha=0.6, beta=0.4, eps=1e-6)
            assert s.dtype == np.int64 and s.shape == (R,)
            assert not set(s.tolist()) & set(RO.overwritten(head, capacity, Bf).tolist())
            assert set(s.tolist()) <= set(PO.survivor_slots(head, size, capacity, Bf).tolist())
        head, size, step = RO.advance(head, size, step, capacity, Bf)


def test_cdf_is_non_decreasing_and_sums_to_the_total():
    for n in (1, 31, 1024, 1025, 5000, 65536 - 16):
        q = np.random.RandomState(n).gamma(0.3, size=n) ** 0.6
        C = PO.cdf(q)
        assert np.all(np.diff(C) >= 0)
        assert abs(C[-1] - q.sum()) <= 1e-12 * q.sum()


def _counts(capacity, Bf, R, alpha, calls, pr):
    n = capacity - Bf
    counts = np.zeros(n)
    head = 4
    for step in range(calls):
        s, _, _ = PO.prioritized(pr, R, head, capacity, capacity, Bf, seed=1234, step=step, stream_id=0,
                                 alpha=alpha, beta=0.5, eps=1e-6)
        counts += np.bincount((head - 1 - s) % capacity, minlength=n)
    return counts


@pytest.mark.parametrize("alpha", [0.6, 1.0])
def test_draws_follow_q_over_S_chi_square(alpha):
    capacity, Bf, R = 37, 5, 64
    pr = _priorities(capacity, 7)
    pr[np.arange(0, capacity, 5)] += 3.0     # a few heavy slots
    counts = _counts(capacity, Bf, R, alpha, 320, pr)
    q = (pr[PO.survivor_slots(4, capacity, capacity, Bf)].astype(np.float64) + 1e-6) ** alpha
    expected = counts.sum() * q / q.sum()
    chi2 = float(np.sum((counts - expected) ** 2 / expected))
    assert chi2 < stats.chi2.ppf(0.999, len(q) - 1), chi2
    # and far from uniform
    uniform = counts.sum() / len(q)
    assert float(np.sum((counts - uniform) ** 2 / uniform)) > 10 * stats.chi2.ppf(0.999, len(q) - 1)


def test_alpha_zero_is_uniform_chi_square():
    capacity, Bf, R = 37, 5, 64
    counts = _counts(capacity, Bf, R, 0.0, 320, _priorities(capacity, 3))
    expected = counts.sum() / (capacity - Bf)
    chi2 = float(np.sum((counts - expected) ** 2 / expected))
    assert chi2 < stats.chi2.ppf(0.999, capacity - Bf - 1), chi2


@pytest.mark.parametrize("beta", [0.0, 0.4, 1.0])
def test_weights_are_normalised_importance_weights(beta):
    capacity, Bf, R, alpha, eps = 300, 8, 128, 0.7, 1e-6
    pr = _priorities(capacity, 5)
    s, w, _ = PO.prioritized(pr, R, 17, capacity, capacity, Bf, seed=9, step=3, stream_id=1, alpha=alpha, beta=beta,
                             eps=eps)
    q_all = (pr[PO.survivor_slots(17, capacity, capacity, Bf)].astype(np.float64) + eps) ** alpha
    q = (pr[s].astype(np.float64) + eps) ** alpha
    want = (q_all.min() / q) ** beta
    np.testing.assert_allclose(w, want, rtol=1e-7)
    assert np.all(w > 0) and np.all(w <= 1)
    # (n P)^-beta over its largest value: the same numbers
    P = q / q_all.sum()
    n = len(q_all)
    np.testing.assert_allclose(w, (n * P) ** -beta / (n * q_all.min() / q_all.sum()) ** -beta, rtol=1e-6)
    if beta == 0.0:
        assert np.all(w == 1)


def test_priority_update_rule():
    T, Bf, R, capacity, eta = 5, 3, 4, 12, 0.9
    rs = np.random.RandomState(0)
    vs, values = rs.randn(T, Bf + R).astype(np.float32), rs.randn(T, Bf + R).astype(np.float32)
    values[2, 1] = np.nan                                   # fresh column 1: non-finite, stored as 0
    slots = np.array([0, 1, 2, 7, 9, 7, 7], dtype=np.int64)  # slot 7 drawn three times: column 6 wins
    before = np.full(capacity, 5.0, dtype=np.float32)
    after = PO.priority_update(vs, values, slots, eta, before)
    e = np.abs(vs.astype(np.float64) - values.astype(np.float64))
    p = eta * e.max(axis=0) + (1 - eta) * e.mean(axis=0)
    for c in (0, 2, 4, 6):
        assert after[slots[c]] == pytest.approx(p[c], rel=1e-6)
    assert after[1] == 0.0
    untouched = sorted(set(range(capacity)) - set(slots.tolist()))
    assert np.all(after[untouched] == 5.0)
    assert after[7] == np.float32(p[6]) and after[7] != np.float32(p[3])


def test_constructor_validation():
    from torchbeast_b200._lib import TorchBeastB200Error
    from torchbeast_b200.replay import ReplayBuffer
    for kw, msg in ((dict(priority_exponent=-0.1), "priority_exponent"),
                    (dict(priority_exponent=float("inf")), "priority_exponent"),
                    (dict(priority_exponent=0.6, importance_exponent=-0.01), "importance_exponent"),
                    (dict(priority_exponent=0.6, importance_exponent=1.5), "importance_exponent"),
                    (dict(priority_exponent=0.6, priority_eta=1.01), "priority_eta"),
                    (dict(priority_exponent=0.6, priority_eta=-1), "priority_eta"),
                    (dict(priority_exponent=0.6, priority_eps=0.0), "priority_eps"),
                    (dict(priority_exponent=0.6, priority_eps=float("nan")), "priority_eps")):
        with pytest.raises(TorchBeastB200Error, match=msg):
            ReplayBuffer(100, 8, **kw)
    b = ReplayBuffer(100, 8, priority_exponent=0.0, importance_exponent=1.0, priority_eta=0.0)
    assert b.prioritized and (b.priority_exponent, b.importance_exponent, b.priority_eta) == (0.0, 1.0, 0.0)
    assert not ReplayBuffer(100, 8).prioritized
    assert ReplayBuffer(100, 8, importance_exponent=7).importance_exponent == 7   # unused without priority_exponent


def test_replay_and_loss_entry_points_validate_on_the_host():
    from torchbeast_b200 import _lib
    from torchbeast_b200.replay import _Leaf
    h = _lib.lib()
    dev = ctypes.c_void_p(256)   # never dereferenced: every check below fails before a launch

    def sample(pr=dev, prio=dev, hs=dev, ss=dev, Bf=4, R=2, cap=10, sid=0, bs=dev, w=dev):
        assert h.tb_replay_sample_prioritized(pr, prio, hs, ss, Bf, R, cap, sid, bs, w, None) != 0
        return h.tb_last_error().decode()

    for k in ("pr", "prio", "hs", "ss", "bs", "w"):
        assert "null pointer" in sample(**{k: None})
    assert "R must be" in sample(R=-1)
    assert "R must be" in sample(R=4097)
    assert "Bf must be" in sample(Bf=0)
    assert "capacity" in sample(cap=4)
    assert "stream_id" in sample(sid=2 ** 32)

    def update(vs=dev, va=dev, T=4, B=6, bs=dev, prio=dev, pr=dev):
        assert h.tb_replay_update_priorities(vs, va, T, B, bs, prio, pr, None) != 0
        return h.tb_last_error().decode()

    for k in ("vs", "va", "bs", "prio", "pr"):
        assert "null pointer" in update(**{k: None})
    assert "at least 1" in update(T=0)
    assert "at least 1" in update(B=0)

    leaves = (_Leaf * 1)(_Leaf(256, 512, 1024, 3, 16))

    def mix(lv=leaves, n=1, Bf=4, R=2, cap=10, slots=dev, hs=dev):
        assert h.tb_replay_mix_slots(lv, n, Bf, R, cap, slots, hs, None) != 0
        return h.tb_last_error().decode()

    assert "null pointer" in mix(lv=None)
    assert "null pointer" in mix(slots=None)
    assert "null pointer" in mix(hs=None)
    assert "num_leaves" in mix(n=0)
    assert "R must be" in mix(R=4097)
    assert "capacity" in mix(cap=4)
    assert "null pointer in leaf 0" in mix(lv=(_Leaf * 1)(_Leaf(None, 512, 1024, 3, 16)))

    # PopArt (a task) with importance weights has no kernel
    args = ([dev] * 8 + [4, 4, 6, 0.99, 0.5, 0.01, 1, 1.0, 1.0, None, dev, dev, dev, dev, 3, dev] + [None] * 3
            + [dev] * 8 + [1, dev, None])
    assert h.tb_impala_loss_f32(*args) != 0 and b"column_weights" in h.tb_last_error()
