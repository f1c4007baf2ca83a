"""CPU: the NumPy restatement of the action-sampling contract (oracle/sampling_np.py) against Philox known-answer vectors
and the contract's own properties, and the host-side argument validation of tb_sample_actions_f32."""
import numpy as np
import pytest
import torch

from oracle import sampling_np as S

CHI2_LOGITS = np.array([0, 0.5, -1, 2, 1, -0.25], dtype=np.float32)
CHI2_999_DF5 = 20.515  # 0.999 quantile of chi-squared with 5 degrees of freedom


@pytest.mark.parametrize("counter,key,expected", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(counter, key, expected):
    """Random123's known-answer vectors for Philox4x32-10."""
    assert tuple(int(w) for w in S.philox4x32_10(counter, key)) == expected


def test_uniform_is_word0_of_the_counter_and_key():
    seed, step, sid = 0x0123456789ABCDEF, (1 << 32) + 5, -3
    u = S.uniforms(2, 1, seed, step, np.array([sid]))
    for t in range(2):
        c = step + t
        s = sid % 2 ** 64
        x = S.philox4x32_10((c & 0xffffffff, c >> 32, s & 0xffffffff, s >> 32), (seed & 0xffffffff, seed >> 32))[0]
        assert u[t, 0] == (int(x) >> 8) * 2.0 ** -24
    assert np.all((u >= 0) & (u < 1))


def test_neg_inf_never_chosen_and_single_finite_logit_always_chosen():
    B, A = 4096, 7
    rs = np.random.RandomState(0)
    x = rs.randn(1, B, A).astype(np.float32)
    x[:, :, [1, 4]] = -np.inf
    a, _ = S.sample_actions(x, seed=5, step=0)
    assert not np.isin(a, [1, 4]).any() and (a >= 0).all()
    assert set(np.unique(a)) == {0, 2, 3, 5, 6}
    one = np.full((1, B, A), -np.inf, dtype=np.float32)
    one[:, :, 3] = -50.0
    a, _ = S.sample_actions(one, seed=5, step=0)
    assert (a == 3).all()


def test_nan_and_all_neg_inf_rows_give_minus_one():
    x = np.zeros((1, 4, 3), dtype=np.float32)
    x[0, 0, 1] = np.nan
    x[0, 1, :] = -np.inf
    x[0, 2, 2] = np.inf
    a, margin = S.sample_actions(x, seed=0, step=0)
    assert a[0].tolist()[:3] == [-1, -1, -1] and a[0, 3] >= 0
    assert np.isinf(margin[0, :3]).all()


def test_one_call_equals_consecutive_single_step_calls():
    rs = np.random.RandomState(1)
    T, B, A = 5, 64, 6
    x = (3 * rs.randn(T, B, A)).astype(np.float32)
    ids = rs.randint(-2 ** 62, 2 ** 62, size=B)
    full, _ = S.sample_actions(x, seed=77, step=2 ** 32 - 2, stream_ids=ids)  # the step crosses a 32-bit word
    rows = [S.sample_actions(x[t:t + 1], seed=77, step=2 ** 32 - 2 + t, stream_ids=ids)[0] for t in range(T)]
    np.testing.assert_array_equal(full, np.concatenate(rows))


def test_chi_squared_over_two_to_the_twenty_streams():
    N = 1 << 20
    a, margin = S.sample_actions(np.broadcast_to(CHI2_LOGITS, (1, N, 6)), seed=0, step=0)
    chi2 = S.chi2(a, S.softmax(CHI2_LOGITS))
    assert chi2 < CHI2_999_DF5
    assert abs(chi2 - 2.0) < 0.5  # the statistic this seed gives
    assert (margin < S.margin_threshold(6)).mean() < 1e-3


def test_host_side_validation():
    from torchbeast_b200 import _lib
    h = _lib.lib()
    assert h.tb_sample_actions_f32(None, 2, 4, 6, 0, 0, None, None, None) != 0
    assert b"null pointer" in h.tb_last_error()
    for T, B in ((-1, 4), (4, -1)):
        assert h.tb_sample_actions_f32(None, T, B, 6, 0, 0, None, None, None) != 0
        assert b"negative size" in h.tb_last_error()
    assert h.tb_sample_actions_f32(None, 2, 4, 0, 0, 0, None, None, None) != 0
    assert b"A must be at least 1" in h.tb_last_error()
    assert h.tb_sample_actions_f32(None, 2 ** 40, 2 ** 40, 6, 0, 0, None, None, None) != 0
    assert b"overflow" in h.tb_last_error()
    # empty problems are a no-op success; seed and step take the full uint64 range
    assert h.tb_sample_actions_f32(None, 0, 4, 6, 2 ** 64 - 1, 2 ** 64 - 1, None, None, None) == 0
    assert h.tb_sample_actions_f32(None, 3, 0, 6, 0, 0, None, None, None) == 0


def test_sampler_refuses_cpu_logits_and_nets_default_to_no_sampler():
    from torchbeast_b200 import _lib, nets
    from torchbeast_b200.sampling import ActionSampler
    s = ActionSampler(seed=3, step=7)
    with pytest.raises(_lib.TorchBeastB200Error, match="CUDA tensors only"):
        s.sample(torch.zeros(1, 2, 6))
    assert (s.seed, s.step) == (3, 7)
    assert nets.FlatParamModule.action_sampler is None
