"""CPU: the largest hidden size.  Every precision falls back to the fp32 step kernels above the other recurrence kinds'
limits, and the backward one holds whole rows of H in shared memory, so H <= TB_LSTM_MAX_HIDDEN = 700.  Every tb_lstm_*
entry checks that before it touches the device; a larger H used to pass the plan and the forward and fail only in the
backward."""
import ctypes
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_H = 700


def _lib():
    from torchbeast_b200 import _lib
    return _lib.lib()


def _plan(H, layers=1, precision=0, In=None):
    fwd, bwd = ctypes.c_int(), ctypes.c_int()
    return _lib().tb_lstm_plan(4, In or H, H, layers, precision, ctypes.byref(fwd), ctypes.byref(bwd))


def test_bound_is_stated_alike_in_header_and_module():
    from torchbeast_b200 import lstm
    with open(ROOT + "/include/torchbeast_b200.h") as f:
        assert "#define TB_LSTM_MAX_HIDDEN %d\n" % MAX_H in f.read()
    assert lstm.MAX_HIDDEN == MAX_H


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_largest_hidden_size_is_accepted(precision):
    assert _plan(MAX_H, precision=precision) == 0
    assert _plan(MAX_H, layers=2, precision=precision, In=3) == 0
    assert _lib().tb_lstm_workspace_bytes(7, 4, 3, MAX_H, 2, precision) > 0


@pytest.mark.parametrize("H", [MAX_H + 1, 768, 1024, 1061])
@pytest.mark.parametrize("precision", [0, 1, 2])
def test_larger_hidden_size_is_rejected_everywhere(H, precision):
    lib = _lib()
    msg = "hidden size %d above %d" % (H, MAX_H)
    assert _plan(H, precision=precision) != 0
    assert msg in lib.tb_last_error().decode()
    fwd, bwd = (ctypes.c_int * 3)(), (ctypes.c_int * 3)()
    assert lib.tb_lstm_plan_layers(4, 3, H, 3, precision, ctypes.cast(fwd, ctypes.c_void_p), ctypes.cast(bwd, ctypes.c_void_p)) != 0
    assert lib.tb_lstm_workspace_bytes(7, 4, 3, H, 1, precision) == 0
    assert msg in lib.tb_last_error().decode()
    # the size check comes before any pointer is read or any kernel is launched
    assert lib.tb_lstm_forward(None, None, None, None, None, 7, 4, 3, H, 1, precision, None, None, None, None, None) != 0
    assert msg in lib.tb_last_error().decode()
    assert lib.tb_lstm_backward(None, None, None, None, None, 7, 4, 3, H, 1, precision, None, None, None) != 0
    assert msg in lib.tb_last_error().decode()
    assert lib.tb_lstm_backward_state(None, None, None, None, None, 7, 4, 3, H, 1, precision, None, None, None, None, None,
                                      None, None) != 0
    assert msg in lib.tb_last_error().decode()


def test_module_raises_above_the_bound():
    from torchbeast_b200 import _lib
    from torchbeast_b200 import lstm as tl
    m = tl.LSTM(3, MAX_H + 1, device="cpu")
    with pytest.raises(_lib.TorchBeastB200Error, match="hidden size %d above %d" % (MAX_H + 1, MAX_H)):
        m.plan(4)
