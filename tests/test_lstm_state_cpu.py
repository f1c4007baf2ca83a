"""CPU: the autograd forward of the standalone LSTM validates its arguments host-side and has no CPU fallback."""
import pytest
import torch


def test_lstm_forward_rejects_cpu_tensors_and_bad_shapes():
    from torchbeast_b200 import _lib
    from torchbeast_b200 import lstm as tl
    m = tl.LSTM(8, 16, 2, device="cpu")
    x = torch.zeros(3, 2, 8)
    with pytest.raises(_lib.TorchBeastB200Error, match="CUDA tensors only"):
        m(x)
    with pytest.raises(_lib.TorchBeastB200Error, match="CUDA tensors only"):
        m(x, (torch.zeros(2, 2, 16), torch.zeros(2, 2, 16)), torch.ones(3, 2))
    with pytest.raises(_lib.TorchBeastB200Error, match="input must be"):
        m(torch.zeros(3, 2, 7))
    with pytest.raises(_lib.TorchBeastB200Error, match="hx must be"):
        m(x, (torch.zeros(1, 2, 16), torch.zeros(1, 2, 16)))
    with pytest.raises(_lib.TorchBeastB200Error, match="notdone must be"):
        m(x, None, torch.ones(3, 3))
