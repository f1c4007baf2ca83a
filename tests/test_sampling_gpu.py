"""GPU: seeded action sampling (tb_sample_actions_f32 through torchbeast_b200.sampling.ActionSampler) against the NumPy
restatement of its contract (oracle/sampling_np.py), its reproducibility properties, edge rows, and the training-mode
forwards of AtariNet / ResNet and polybeast's inference loop with a sampler attached."""
import types
import unittest.mock as mock

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT
from oracle import sampling_np as S

pytestmark = pytest.mark.gpu

CHI2_LOGITS = np.array([0, 0.5, -1, 2, 1, -0.25], dtype=np.float32)


def _sampler(seed, step=0):
    from torchbeast_b200.sampling import ActionSampler
    return ActionSampler(seed, step)


def _check_against_oracle(x, got, seed, step, stream_ids=None):
    """Every row whose oracle margin is at least the threshold has exactly the oracle's action; returns the fraction of
    rows below the threshold."""
    want, margin = S.sample_actions(x, seed, step, stream_ids)
    sure = margin >= S.margin_threshold(x.shape[-1])
    bad = np.argwhere(sure & (got != want))
    assert bad.size == 0, (bad[:5], got[tuple(bad[:5].T)], want[tuple(bad[:5].T)])
    return 1.0 - sure.mean()


@pytest.mark.parametrize("A", [2, 6, 7, 18, 100])
def test_matches_oracle(A):
    T, B = 4, 16384
    rs = np.random.RandomState(A)
    x = (3 * rs.randn(T, B, A)).astype(np.float32)
    x[rs.rand(T, B, A) < 0.1] = -np.inf  # at A = 2 this also makes about 1 % of the rows all -inf
    s = _sampler(seed=0xDEADBEEF12345, step=1000)
    got = s.sample(torch.from_numpy(x).cuda())
    assert got.dtype == torch.int64 and tuple(got.shape) == (T, B) and s.step == 1004
    below = _check_against_oracle(x, got.cpu().numpy(), 0xDEADBEEF12345, 1000)
    assert below < 0.01


def test_chi_squared_matches_oracle():
    N = 1 << 20
    x = np.ascontiguousarray(np.broadcast_to(CHI2_LOGITS, (1, N, 6)))
    got = _sampler(0).sample(torch.from_numpy(x).cuda()).cpu().numpy()
    want, margin = S.sample_actions(x, 0, 0)
    _check_against_oracle(x, got, 0, 0)
    p = S.softmax(CHI2_LOGITS)
    assert abs(S.chi2(got, p) - S.chi2(want, p)) < 1e-2
    assert S.chi2(got, p) < 20.515  # 0.999 quantile, 5 degrees of freedom


def test_reproducible():
    T, B, A = 3, 4096, 6
    g = torch.Generator().manual_seed(0)
    x = (2 * torch.randn(T, B, A, generator=g)).cuda()
    ids = torch.randint(-2 ** 40, 2 ** 40, (B,), generator=g).cuda()
    first = _sampler(11, 50).sample(x, ids)
    assert torch.equal(first, _sampler(11, 50).sample(x, ids))  # a repeated call is bitwise the same
    s = _sampler(11, 50)
    rows = torch.cat([s.sample(x[t:t + 1], ids) for t in range(T)])
    assert torch.equal(first, rows) and s.step == 53  # one [T, B] call == T calls of [1, B]
    perm = torch.randperm(B, generator=g).cuda()
    assert torch.equal(_sampler(11, 50).sample(x[:, perm].contiguous(), ids[perm]), first[:, perm])
    # the default stream ids are the column indices
    assert torch.equal(_sampler(11, 50).sample(x), _sampler(11, 50).sample(x, torch.arange(B)))
    assert not torch.equal(_sampler(11, 50).sample(x), first)


def test_different_seed_changes_one_minus_sum_p_squared():
    N = 1 << 18
    x = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(CHI2_LOGITS, (1, N, 6)))).cuda()
    a, b = _sampler(1).sample(x), _sampler(2).sample(x)
    p = S.softmax(CHI2_LOGITS)
    changed = float((a != b).double().mean())
    assert abs(changed - (1.0 - float((p ** 2).sum()))) < 0.01


def test_edge_rows():
    A = 5
    rows = np.array([
        [-np.inf, -np.inf, 3.0, -np.inf, -np.inf],     # single finite logit
        [0.0, np.nan, 1.0, 2.0, 3.0],                  # NaN
        [-np.inf] * A,                                 # all -inf
        [1e30, -1e30, 0.0, 1e30, -1e30],               # spanning +-1e30: only the two maxima have mass
        [0.0, 1.0, np.inf, 2.0, 3.0],                  # +inf: no distribution
        [-1e30, -1e30, -1e30, -1e30, -1e30],           # all equal, far from zero
    ], dtype=np.float32)
    B = 2048
    x = np.ascontiguousarray(np.broadcast_to(rows[:, None, :], (rows.shape[0], B, A)))
    got = _sampler(9).sample(torch.from_numpy(x).cuda()).cpu().numpy()
    torch.cuda.synchronize()  # nothing faulted
    assert (got[0] == 2).all()
    assert (got[1] == -1).all() and (got[2] == -1).all() and (got[4] == -1).all()
    assert set(np.unique(got[3])) == {0, 3}
    assert set(np.unique(got[5])) == set(range(A))
    _check_against_oracle(x, got, 9, 0)


def _net(kind, use_lstm, A, seed):
    from torchbeast_b200 import monobeast, polybeast_learner
    if kind == "atari":
        model = monobeast.AtariNet((4, 84, 84), A, use_lstm)
        params = LT.random_params(LT.atarinet_param_shapes(A, use_lstm), seed=seed)
    else:
        model = polybeast_learner.Net(A, use_lstm)
        params = LT.random_params(LT.resnet_param_shapes(A, use_lstm), seed=seed)
    model.load_state_dict(params)
    return model


@pytest.mark.parametrize("use_lstm", [False, True])
@pytest.mark.parametrize("kind", ["atari", "resnet"])
def test_training_forward_samples_with_the_attached_sampler(kind, use_lstm):
    A, T, B = 6, 2, 8
    model = _net(kind, use_lstm, A, seed=5)
    model.train()
    model.action_sampler = _sampler(seed=21, step=100)
    cb = {k: v.cuda() for k, v in LT.synthetic_batch(T - 1, B, A, seed=6).items()}
    state = model.initial_state(B)
    with torch.no_grad():
        out, _ = model(cb, state)
    if kind == "atari":
        action, logits = out["action"], out["policy_logits"]
    else:
        action, logits = out[0], out[1]
    assert tuple(action.shape) == (T, B) and action.dtype == torch.int64
    assert model.action_sampler.step == 100 + T
    _check_against_oracle(logits.cpu().numpy(), action.cpu().numpy(), 21, 100)
    # caller-supplied stream ids (e.g. actor indices) name each column's stream
    ids = torch.arange(B, dtype=torch.int64) * 7 + 3
    model.action_sampler.step = 100
    with torch.no_grad():
        out, _ = model(dict(cb, stream_ids=ids), state)
    action = out["action"] if kind == "atari" else out[0]
    _check_against_oracle(logits.cpu().numpy(), action.cpu().numpy(), 21, 100, ids.numpy())


@pytest.mark.parametrize("kind", ["atari", "resnet"])
def test_two_inference_calls_advance_the_step_by_two(kind):
    from torchbeast_b200 import polybeast_learner
    A, B = 6, 48
    model = _net(kind, True, A, seed=7)
    model.train()
    model.action_sampler = _sampler(seed=3)
    batch = LT.synthetic_batch(1, B, A, seed=8)
    mbs, state = [], model.initial_state(B)
    for t in range(2):
        env = tuple(batch[k][t:t + 1] for k in ("frame", "reward", "done", "episode_step", "episode_return", "last_action"))
        mb = mock.MagicMock()
        mb.get_inputs = mock.Mock(return_value=(env, tuple(s.cpu() for s in state)))
        mbs.append(mb)
    batcher = mock.MagicMock()
    batcher.__iter__.return_value = iter(mbs)
    polybeast_learner.inference(types.SimpleNamespace(actor_device="cuda:0"), batcher, model)
    assert model.action_sampler.step == 2
    for t, mb in enumerate(mbs):
        (outputs,), _ = mb.set_outputs.call_args
        (action, logits, _), _ = outputs
        _check_against_oracle(logits.numpy(), action.numpy(), 3, t)
