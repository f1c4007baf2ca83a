"""GPU: the inference path of polybeast's own model, the IMPALA ResNet (reference polybeast_learner.py:269-285): T = 1,
B in {1, 48, 512} actors through polybeast_learner.inference with a mock DynamicBatcher batch; outputs on the CPU with the
reference's shapes, logits / baseline / carried LSTM state equal to the torch oracle's forward.  At B > 32 the H=256 LSTM
runs on the fp32 cooperative kernels rather than the single-cluster one."""
import types
import unittest.mock as mock

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("use_lstm", [False, True])
@pytest.mark.parametrize("B", [1, 48, 512])
def test_resnet_inference_matches_oracle(B, use_lstm):
    from torchbeast_b200 import polybeast_learner
    A = 6
    batch = LT.synthetic_batch(0, B, A, seed=51, with_last_action=False)  # T + 1 = 1 row
    params = LT.random_params(LT.resnet_param_shapes(A, use_lstm), seed=52)
    model = polybeast_learner.Net(A, use_lstm)
    model.load_state_dict(params)
    model.eval()
    state = ()
    if use_lstm:
        rs = np.random.RandomState(53)
        state = tuple(torch.from_numpy(rs.randn(1, B, 256).astype(np.float32) * 0.1) for _ in range(2))
    env = (batch["frame"], batch["reward"], batch["done"], batch["episode_step"], batch["episode_return"])
    mb = mock.MagicMock()
    mb.get_inputs = mock.Mock(return_value=(env, state))
    mb.set_outputs = mock.Mock()
    batcher = mock.MagicMock()
    batcher.__iter__.return_value = iter([mb])
    polybeast_learner.inference(types.SimpleNamespace(actor_device="cuda:0", use_lstm=use_lstm), batcher, model)
    mb.set_outputs.assert_called_once()
    (outputs,), kw = mb.set_outputs.call_args
    assert kw == {}
    (action, logits, baseline), core_state = outputs
    assert tuple(action.shape) == (1, B) and tuple(logits.shape) == (1, B, A) and tuple(baseline.shape) == (1, B)
    for t in (action, logits, baseline) + tuple(core_state):
        assert t.device == torch.device("cpu")
    assert len(core_state) == (2 if use_lstm else 0)
    ol, ob, ostate = LT.resnet_forward(params, batch["frame"], batch["reward"], batch["done"], state)
    np.testing.assert_allclose(logits.numpy(), ol.numpy(), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(baseline.numpy(), ob.numpy(), rtol=1e-4, atol=1e-4)
    assert torch.equal(action, logits.argmax(-1))  # eval mode: greedy (polybeast_learner.py:258-260)
    for a, b in zip(core_state, ostate):
        assert tuple(a.shape) == (1, B, 256)
        np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("B", [1, 48])
def test_resnet_state_carry_over_two_inference_calls(B):
    """Two T=1 calls carrying the state == one T=2 forward (what an actor sees across DynamicBatcher calls)."""
    from torchbeast_b200 import polybeast_learner
    A = 6
    batch = LT.synthetic_batch(1, B, A, seed=61, with_last_action=False)
    params = LT.random_params(LT.resnet_param_shapes(A, True), seed=62)
    model = polybeast_learner.Net(A, True)
    model.load_state_dict(params)
    model.eval()
    cb = {k: v.cuda() for k, v in batch.items()}
    with torch.no_grad():
        (_, full, _), _ = model(cb, model.initial_state(B))
        st = model.initial_state(B)
        rows = []
        for t in range(2):
            (_, logits, _), st = model({k: v[t:t + 1] for k, v in cb.items()}, st)
            rows.append(logits)
    np.testing.assert_allclose(torch.cat(rows).cpu().numpy(), full.cpu().numpy(), rtol=1e-5, atol=1e-5)
