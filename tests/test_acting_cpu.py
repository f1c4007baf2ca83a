"""CPU: the graphed acting forward's bucket rule, host validation of tb_sample_actions_dev_f32, what GraphedActor refuses,
and the inference flag's default."""
import ctypes
import types

import pytest


def test_bucket_is_the_next_power_of_two():
    from torchbeast_b200 import _lib
    from torchbeast_b200.acting import bucket_size
    assert [bucket_size(b) for b in (1, 2, 3, 4, 5, 31, 32, 33, 48, 64, 65, 500, 512)] == \
        [1, 2, 4, 4, 8, 32, 32, 64, 64, 64, 128, 512, 512]
    # the network's kernel choices switch at B = 32: padding never crosses it
    assert all((bucket_size(b) <= 32) == (b <= 32) for b in range(1, 1025))
    with pytest.raises(_lib.TorchBeastB200Error):
        bucket_size(0)


def test_device_step_sampler_host_validation():
    from torchbeast_b200 import _lib
    h = _lib.lib()
    pair = (ctypes.c_uint64 * 2)()  # any non-null address: validation fails before anything is launched
    for T, B in ((2, 4), (0, 4), (3, 0)):
        assert h.tb_sample_actions_dev_f32(None, T, B, 6, None, None, None, None) != 0
        assert b"null seed_step" in h.tb_last_error()
    assert h.tb_sample_actions_dev_f32(None, 2, 4, 6, pair, None, None, None) != 0
    assert b"null pointer" in h.tb_last_error()
    for T, B in ((-1, 4), (4, -1)):
        assert h.tb_sample_actions_dev_f32(None, T, B, 6, pair, None, None, None) != 0
        assert b"negative size" in h.tb_last_error()
    assert h.tb_sample_actions_dev_f32(None, 2, 4, 0, pair, None, None, None) != 0
    assert b"A must be at least 1" in h.tb_last_error()
    assert h.tb_sample_actions_dev_f32(None, 2 ** 40, 2 ** 40, 6, pair, None, None, None) != 0
    assert b"overflow" in h.tb_last_error()
    # empty problems are a no-op success
    assert h.tb_sample_actions_dev_f32(None, 0, 4, 6, pair, None, None, None) == 0
    assert h.tb_sample_actions_dev_f32(None, 3, 0, 6, pair, None, None, None) == 0


def test_graphed_actor_refuses_a_cpu_model():
    from torchbeast_b200 import _lib, monobeast
    from torchbeast_b200.acting import GraphedActor
    model = monobeast.AtariNet((4, 84, 84), 6, False, device="cpu")
    with pytest.raises(_lib.TorchBeastB200Error, match="CUDA"):
        GraphedActor(model)


def test_graphed_actor_refuses_training_mode_without_a_sampler():
    """GraphedActor.__call__ asks acting.replay_sampler for the sampler before it touches the device."""
    from torchbeast_b200 import _lib, monobeast
    from torchbeast_b200.acting import replay_sampler
    from torchbeast_b200.sampling import ActionSampler
    model = monobeast.AtariNet((4, 84, 84), 6, False, device="cpu")
    model.train()
    with pytest.raises(_lib.TorchBeastB200Error, match="action_sampler"):
        replay_sampler(model)
    s = model.action_sampler = ActionSampler(seed=1)
    assert replay_sampler(model) is s
    model.eval()  # greedy: no sampler is used, none is needed
    assert replay_sampler(model) is None
    model.action_sampler = None
    assert replay_sampler(model) is None


def test_inference_graph_defaults_to_off(monkeypatch):
    from torchbeast_b200 import polybeast_learner
    monkeypatch.delenv("TB_INFERENCE_GRAPH", raising=False)
    assert polybeast_learner.inference_graph_enabled(types.SimpleNamespace()) is False
    assert polybeast_learner.inference_graph_enabled(types.SimpleNamespace(inference_graph=None)) is False
    assert polybeast_learner.inference_graph_enabled(types.SimpleNamespace(inference_graph=True)) is True
    monkeypatch.setenv("TB_INFERENCE_GRAPH", "1")
    assert polybeast_learner.inference_graph_enabled(types.SimpleNamespace()) is True
    assert polybeast_learner.inference_graph_enabled(types.SimpleNamespace(inference_graph=False)) is False
