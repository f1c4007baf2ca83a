"""CPU: stacks of more than two layers - torch.nn.LSTM's parameter set, and the workspace of the segment chain."""
import ctypes

import pytest
import torch


@pytest.mark.parametrize("layers", [3, 4, 7])
def test_deep_lstm_has_torch_parameters(layers):
    from torchbeast_b200 import lstm as tl
    m = tl.LSTM(40, 24, layers, device="cpu")
    ref = torch.nn.LSTM(40, 24, num_layers=layers)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == \
           [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    m.load_state_dict(ref.state_dict(), strict=True)


def test_deep_lstm_rejects_zero_layers():
    from torchbeast_b200 import _lib
    from torchbeast_b200 import lstm as tl
    with pytest.raises(_lib.TorchBeastB200Error, match="num_layers"):
        tl.LSTM(8, 16, 0, device="cpu")


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_workspace_grows_with_depth(precision):
    from torchbeast_b200 import _lib
    lib = _lib.lib()
    sizes = [lib.tb_lstm_workspace_bytes(81, 32, 600, 519, L, precision) for L in range(1, 9)]
    assert all(n > 0 for n in sizes)
    assert all(b > a for a, b in zip(sizes, sizes[1:]))


def test_plan_still_takes_one_or_two_layers():
    from torchbeast_b200 import _lib
    fwd, bwd = ctypes.c_int(), ctypes.c_int()
    assert _lib.lib().tb_lstm_plan(8, 257, 256, 3, 2, ctypes.byref(fwd), ctypes.byref(bwd)) != 0
