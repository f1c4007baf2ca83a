"""CPU: what acting on newest frames (torchbeast_b200.acting.FrameHistory attached as model.frame_history) refuses on the
host, before anything reaches the device, and the host-side checks of tb_frame_history_fill_u8."""
import ctypes

import pytest
import torch


def _model(S=5, history_device="cpu"):
    from torchbeast_b200 import monobeast
    from torchbeast_b200.acting import FrameHistory
    model = monobeast.AtariNet((4, 84, 84), 6, True, device="cpu")
    model.frame_history = FrameHistory(S, device=history_device)
    return model


def _inputs(B, frame=None, **kw):
    inputs = dict(frame=torch.zeros(1, B, 84, 84, dtype=torch.uint8) if frame is None else frame,
                  reward=torch.zeros(1, B), done=torch.ones(1, B, dtype=torch.bool),
                  last_action=torch.zeros(1, B, dtype=torch.int64))
    inputs.update(kw)
    return inputs


def test_num_streams_must_be_positive():
    from torchbeast_b200 import _lib
    from torchbeast_b200.acting import FrameHistory
    for S in (0, -3):
        with pytest.raises(_lib.TorchBeastB200Error, match="num_streams"):
            FrameHistory(S, device="cpu")
    h = FrameHistory(4, device="cpu")
    assert h.num_streams == 4 and tuple(h.buffer.shape) == (4, 3, 84, 84) and h.buffer.dtype == torch.uint8
    assert not h.buffer.any()


def test_reset_zeroes_the_given_streams_or_all_in_place():
    from torchbeast_b200.acting import FrameHistory
    h = FrameHistory(4, device="cpu")
    address = h.buffer.data_ptr()
    h.buffer.fill_(7)
    h.reset(torch.tensor([1, 3]))
    assert not h.buffer[[1, 3]].any() and bool((h.buffer[[0, 2]] == 7).all())
    h.reset([0])
    assert not h.buffer[0].any() and bool((h.buffer[2] == 7).all())
    h.reset()
    assert not h.buffer.any() and h.buffer.data_ptr() == address


@pytest.mark.parametrize("frame", [torch.zeros(1, 2, 80, 80, dtype=torch.uint8), torch.zeros(1, 2, 84, 84),
                                   torch.zeros(1, 3, 84, 84, dtype=torch.uint8)])
def test_wrong_frame_shape_with_a_history(frame):
    from torchbeast_b200 import _lib
    model = _model()
    with pytest.raises(_lib.TorchBeastB200Error, match="newest frames"):
        model(_inputs(2, frame=frame), model.initial_state(2))


@pytest.mark.parametrize("ids", [[0, 0], [0, 5], [-1, 1], [4, 4]])
def test_duplicate_or_out_of_range_host_ids(ids):
    from torchbeast_b200 import _lib
    model = _model(S=5)
    with pytest.raises(_lib.TorchBeastB200Error, match="distinct and in"):
        model(_inputs(2, stream_ids=torch.tensor(ids)), model.initial_state(2))


def test_ids_must_be_an_integer_vector_of_the_batch():
    from torchbeast_b200 import _lib
    model = _model()
    for ids in (torch.tensor([0, 1, 2]), torch.tensor([0.0, 1.0]), torch.tensor([[0, 1]])):
        with pytest.raises(_lib.TorchBeastB200Error, match="stream_ids"):
            model(_inputs(2, stream_ids=ids), model.initial_state(2))


def test_default_ids_need_a_stream_per_column():
    from torchbeast_b200 import _lib
    model = _model(S=2)
    with pytest.raises(_lib.TorchBeastB200Error, match="at least 3 streams"):
        model(_inputs(3), model.initial_state(3))


def test_valid_host_ids_reach_the_device_check():
    """Everything on the host passes; the CPU model then stops where every forward does."""
    from torchbeast_b200 import _lib
    model = _model(S=5)
    with pytest.raises(_lib.TorchBeastB200Error, match="CUDA"):
        model(_inputs(2, stream_ids=torch.tensor([4, 0])), model.initial_state(2))


def test_history_on_another_device_than_the_model():
    from torchbeast_b200 import _lib
    model = _model(history_device="meta")
    with pytest.raises(_lib.TorchBeastB200Error, match="frame_history is on meta"):
        model(_inputs(2), model.initial_state(2))


def test_fill_checks_every_tensor_before_the_kernel():
    from torchbeast_b200 import _lib
    from torchbeast_b200.acting import FrameHistory
    h = FrameHistory(4, device="cpu")
    frames = torch.zeros(5, 3, 84, 84, dtype=torch.uint8)
    done = torch.zeros(2, 3, dtype=torch.uint8)
    ids = torch.arange(3)
    bad = [
        (torch.zeros(5, 3, 84, 84), done, ids, "frames"),
        (torch.zeros(3, 3, 84, 84, dtype=torch.uint8), torch.zeros(0, 3, dtype=torch.uint8), ids, "frames"),
        (torch.zeros(5, 3, 84, 80, dtype=torch.uint8), done, ids, "frames"),
        (torch.zeros(3, 5, 84, 84, dtype=torch.uint8).transpose(0, 1), done, ids, "frames"),
        (frames, torch.zeros(1, 3, dtype=torch.uint8), ids, "done"),
        (frames, torch.zeros(2, 3, dtype=torch.int32), ids, "done"),
        (frames, torch.zeros(3, 2, dtype=torch.uint8).t(), ids, "done"),
        (frames, done, ids.to(torch.int32), "stream_ids"),
        (frames, done, torch.arange(4), "stream_ids"),
        (frames, done, torch.arange(6)[::2], "stream_ids"),
        (frames, done.to("meta"), ids, "device"),
    ]
    for f, d, i, what in bad:
        with pytest.raises(_lib.TorchBeastB200Error, match=what):
            h.fill(f, d, i)
    # well-formed tensors pass every check and stop at the CPU buffer, before any launch
    with pytest.raises(_lib.TorchBeastB200Error, match="CUDA"):
        h.fill(frames, done.bool(), ids)


def test_fill_abi_host_validation():
    from torchbeast_b200 import _lib
    h = _lib.lib()
    assert "tb_frame_history_fill_u8" in _lib.declared_symbols()
    buf = ctypes.create_string_buffer(64)
    base = ctypes.addressof(buf)
    aligned = ctypes.c_void_p((base + 15) & ~15)
    # nothing is launched: every call fails its host-side checks
    for T, B, HW, S in ((0, 1, 7056, 1), (1, 0, 7056, 1), (1, 1, 7056, 0), (1, 1, 7050, 1), (1, 1, 0, 1)):
        assert h.tb_frame_history_fill_u8(aligned, aligned, aligned, T, B, HW, aligned, S, None) != 0
        assert b"bad sizes" in h.tb_last_error()
    for nulls in range(4):
        args = [aligned] * 4
        args[nulls] = None
        assert h.tb_frame_history_fill_u8(args[0], args[1], args[2], 1, 1, 7056, args[3], 1, None) != 0
        assert b"null pointer" in h.tb_last_error()
    misaligned = ctypes.c_void_p(aligned.value + 1)
    assert h.tb_frame_history_fill_u8(misaligned, aligned, aligned, 1, 1, 7056, aligned, 1, None) != 0
    assert b"16-byte aligned" in h.tb_last_error()
    assert h.tb_frame_history_fill_u8(aligned, aligned, aligned, 1, 1, 7056, misaligned, 1, None) != 0
    assert b"16-byte aligned" in h.tb_last_error()
