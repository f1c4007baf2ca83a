"""CPU: MLPNet (vector observations).  Constructor limits and their messages, the state_dict spec against
tests/mlpnet_oracle.py and the parameter count against tb_mlpnet_param_count, the header's constants, the staging spec's
frame_dtype, the statistics merge against a two-pass mean and variance, and learn() raising before anything is staged
for a frame leaf the net does not take."""
import ctypes
import os
import re
import types

import numpy as np
import pytest
import torch

from tests import mlpnet_oracle as MO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _net(*args, **kw):
    from torchbeast_b200 import nets
    return nets.MLPNet(*args, device="cpu", **kw)


@pytest.mark.parametrize("kw,match", [
    (dict(observation_size=0), r"observation_size must be an int O in \[1, 4096\]"),
    (dict(observation_size=4097), r"observation_size must be an int O in \[1, 4096\]"),
    (dict(observation_size=(3, 4)), r"observation_size must be an int O"),
    (dict(observation_size=2.5), r"observation_size must be an int O"),
    (dict(hidden=()), r"hidden must be 1 to 4 widths, each a multiple of 8 in \[8, 512\]"),
    (dict(hidden=(8,) * 5), r"hidden must be 1 to 4 widths"),
    (dict(hidden=(12,)), r"hidden must be 1 to 4 widths"),
    (dict(hidden=(520,)), r"hidden must be 1 to 4 widths"),
    (dict(hidden=(0,)), r"hidden must be 1 to 4 widths"),
    (dict(num_actions=32), r"the policy head takes at most 31 outputs"),
    (dict(num_actions=(20, 12)), r"the policy head takes at most 31 outputs"),
    (dict(num_tasks=65), r"num_tasks must be in \[1, 64\]"),
    (dict(precision="fp16"), r"precision must be one of"),
])
def test_constructor_limits(kw, match):
    from torchbeast_b200 import _lib
    args = dict(observation_size=17, num_actions=6, hidden=(64, 64))
    args.update(kw)
    with pytest.raises(_lib.TorchBeastB200Error, match=match):
        _net(args.pop("observation_size"), args.pop("num_actions"), **args)


def test_gaussian_width_limit():
    from torchbeast_b200 import _lib
    from torchbeast_b200.action_space import Gaussian
    with pytest.raises(_lib.TorchBeastB200Error, match="Gaussian"):
        _net(17, Gaussian(16))
    _net(17, Gaussian(15), hidden=(512,), use_lstm=True)  # 512 + 15 + 1 = 528 <= 700


CASES = [
    dict(O=17, hidden=(256, 256), A=6, lstm=False),
    dict(O=3, hidden=(8,), A=1, lstm=True),
    dict(O=376, hidden=(64, 32, 16, 8), A=5, lstm=True, tasks=3),
    dict(O=4096, hidden=(512,), A=(3, 4, 2), lstm=True),
    dict(O=67, hidden=(128, 64, 32), A="gaussian", lstm=False, tasks=2),
    dict(O=1, hidden=(16, 24), A="gaussian", lstm=True, norm=True),
]


def _space(A):
    from torchbeast_b200.action_space import Gaussian
    return Gaussian(6) if A == "gaussian" else A


@pytest.mark.parametrize("case", range(len(CASES)))
def test_spec_keys_and_param_count(case):
    from torchbeast_b200 import _lib, nets
    c = CASES[case]
    model = _net(c["O"], _space(c["A"]), hidden=c["hidden"], use_lstm=c["lstm"], num_tasks=c.get("tasks"),
                 normalize_observations=c.get("norm", False))
    D = 6 if c["A"] == "gaussian" else None
    A = 12 if D else (sum(c["A"]) if isinstance(c["A"], tuple) else c["A"])
    want = MO.spec(c["O"], c["hidden"], A, c["lstm"], c.get("tasks", 1), continuous_dim=D)
    assert nets.mlpnet_param_spec(c["O"], c["hidden"], A, c["lstm"], c.get("tasks", 1), D) == want
    sd = model.state_dict()
    names = [n for n, _ in want]
    extra = (["popart.mu", "popart.nu"] if c.get("tasks") else []) + (list(nets.ObsNorm.KEYS) if c.get("norm") else [])
    assert list(sd) == names + extra
    for n, shape in want:
        assert tuple(sd[n].shape) == shape and sd[n].dtype == torch.float32, n
    total = sum(int(np.prod(s)) for _, s in want)
    assert model.flat_params.numel() == total
    assert _lib.lib().tb_mlpnet_param_count(*model._c_args()) == total
    assert model.observation_shape == (c["O"],)
    assert model.core_size == c["hidden"][-1] + 1 + (D if D else A)


def test_obs_norm_buffers():
    from torchbeast_b200 import nets
    model = _net(17, 6, normalize_observations=True)
    sd = model.state_dict()
    for k, v in zip(nets.ObsNorm.KEYS, (0.0, 1.0, 0.0)):
        assert sd[k].dtype == torch.float64 and tuple(sd[k].shape) == (17,) and torch.all(sd[k] == v), k
    model.float()  # the statistics stay float64
    assert model.obs_norm.mean.dtype == torch.float64
    # state_dict round trip, and copy_params_from, carry the statistics
    other = _net(17, 6, normalize_observations=True)
    model.obs_norm.mean.fill_(2.5); model.obs_norm.var.fill_(3.0); model.obs_norm.count.fill_(7.0)
    other.load_state_dict(model.state_dict())
    assert torch.equal(other.obs_norm.var, model.obs_norm.var) and torch.equal(other.flat_params, model.flat_params)
    third = _net(17, 6, normalize_observations=True)
    third.load_state_dict({k: v.clone() for k, v in model.state_dict().items()})
    assert torch.equal(third.obs_norm.count, model.obs_norm.count)
    fourth = _net(17, 6, normalize_observations=True)
    fourth.copy_params_from(model)
    assert torch.equal(fourth.obs_norm.mean, model.obs_norm.mean)
    assert _net(17, 6).obs_norm is None


def test_header_constants_and_config_layout():
    from torchbeast_b200 import nets
    text = open(os.path.join(ROOT, "include", "torchbeast_b200.h")).read()
    consts = dict(re.findall(r"#define (TB_MLP_MAX_\w+|TB_OBS_NORM_\w+) (\S+)", text))
    assert int(consts["TB_MLP_MAX_OBS"]) == nets.MLP_MAX_OBS
    assert int(consts["TB_MLP_MAX_LAYERS"]) == nets.MLP_MAX_LAYERS == len(nets.MLPConfig().hidden)
    assert int(consts["TB_MLP_MAX_WIDTH"]) == nets.MLP_MAX_WIDTH
    assert float(consts["TB_OBS_NORM_EPS"]) == nets.ObsNorm.EPS == MO.EPS
    assert float(consts["TB_OBS_NORM_CLIP"].rstrip("f")) == nets.ObsNorm.CLIP == MO.CLIP
    body = re.search(r"typedef struct tb_mlp_config \{(.*?)\} tb_mlp_config;", text, re.S).group(1)
    fields = re.findall(r"int (\w+)(?:\[\w+\])?;", body)
    assert fields == [f for f, _ in nets.MLPConfig._fields_]
    assert ctypes.sizeof(nets.MLPConfig) == 4 * (len(fields) - 1 + nets.MLP_MAX_LAYERS)


def test_c_entry_rejects_what_the_constructor_rejects():
    from torchbeast_b200 import _lib, nets
    lib = _lib.lib()

    def count(O=17, hidden=(64,), A=6, lstm=0, V=1, D=0):
        cfg = nets.MLPConfig()
        cfg.obs_dim, cfg.num_layers = O, len(hidden)
        for i, h in enumerate(hidden[:nets.MLP_MAX_LAYERS]):
            cfg.hidden[i] = h
        cfg.num_actions, cfg.num_values, cfg.use_lstm = A, V, lstm
        return lib.tb_mlpnet_param_count(ctypes.byref(cfg), None, D)

    assert count() > 0
    for bad in (dict(O=0), dict(O=4097), dict(hidden=(12,)), dict(hidden=(520,)), dict(hidden=()),
                dict(hidden=(8,) * 5), dict(A=32), dict(V=65), dict(A=7, D=3)):
        assert count(**bad) == -1, bad
    # Gaussian(6): the core takes 6 last-action columns, not 12, so the policy and baseline rows are 6 shorter
    assert count(A=12) - count(A=12, D=6) == (12 + 1) * 6
    assert lib.tb_mlpnet_workspace_bytes(None, None, 0, 5, 3, 2) == 0


def test_spec_for_frame_dtype():
    from torchbeast_b200 import staging
    default = staging.spec_for(4, 2, 6)
    assert default["frame"] == ((5, 2, 4, 84, 84), torch.uint8)
    assert staging.spec_for(4, 2, 6, frame_dtype=torch.uint8) == default
    vec = staging.spec_for(4, 2, 6, frame_shape=(17,), frame_dtype=torch.float32)
    assert vec["frame"] == ((5, 2, 17), torch.float32)
    assert {k: v for k, v in vec.items() if k != "frame"} == {k: v for k, v in default.items() if k != "frame"}


@pytest.mark.parametrize("chunks", [1, 3, 7])
def test_statistics_merge_equals_two_pass_moments(chunks):
    rs = np.random.RandomState(chunks)
    O = 9
    scale = np.array([1e-3, 1.0, 10.0, 1e3, 1.0, 5.0, 1.0, 1.0, 1.0])
    x = rs.randn(40 * chunks, O) * scale + np.array([0, 5, -3, 1e4, 0, 0, 0, 2, 0])
    x[rs.rand(*x.shape) < 0.05] = np.nan
    x[3, 4] = np.inf
    x[5, 4] = -np.inf
    x[:, 6] = np.nan  # a feature with no finite entry keeps (0, 0, 1)
    count, mean, var = np.zeros(O), np.zeros(O), np.ones(O)
    for part in np.array_split(x, chunks):
        count, mean, var = MO.merge(count, mean, var, part)
    n, m, v = MO.two_pass(x)
    np.testing.assert_array_equal(count, n)
    np.testing.assert_allclose(mean, m, rtol=1e-12, atol=1e-12 * np.abs(m).max())
    np.testing.assert_allclose(var, v, rtol=1e-10)
    assert (count[6], mean[6], var[6]) == (0.0, 0.0, 1.0)


def _flags():
    return types.SimpleNamespace(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.01,
                                 grad_norm_clipping=40.0)


def _batch(T, B, O, frame=None):
    return dict(frame=torch.zeros(T + 1, B, O) if frame is None else frame, reward=torch.zeros(T + 1, B),
                done=torch.zeros(T + 1, B, dtype=torch.bool), episode_return=torch.zeros(T + 1, B),
                episode_step=torch.zeros(T + 1, B, dtype=torch.int32), policy_logits=torch.zeros(T + 1, B, 6),
                baseline=torch.zeros(T + 1, B), action=torch.zeros(T + 1, B, dtype=torch.int64),
                last_action=torch.zeros(T + 1, B, dtype=torch.int64))


@pytest.mark.parametrize("case", ["history", "unstacked", "uint8", "wrong_O", "image"])
def test_learn_raises_before_staging(case):
    from torchbeast_b200 import _lib, learner
    T, B, O = 4, 2, 17
    model = _net(O, 6, hidden=(32,))
    frame = {"unstacked": torch.zeros(T + 4, B, 84, 84, dtype=torch.uint8),
             "uint8": torch.zeros(T + 1, B, O, dtype=torch.uint8), "wrong_O": torch.zeros(T + 1, B, O + 1),
             "image": torch.zeros(T + 1, B, 4, 84, 84, dtype=torch.uint8)}.get(case)
    if case == "history":
        model.frame_history = object()
    stager_before = getattr(model, "_tb_stager", None)
    with pytest.raises(_lib.TorchBeastB200Error, match="frame_history" if case == "history" else "float32 \\[T,B,17\\]"):
        learner.learn(_flags(), model, None, _batch(T, B, O, frame), (), None, None)
    assert getattr(model, "_tb_stager", None) is stager_before is None
