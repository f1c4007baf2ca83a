"""CPU: unstacked rollouts - the restack formula against the environment + FrameStack simulator, the staging layout of
an unstacked frame leaf, the host-side writers, Python-side validation and the new C-ABI entries (host calls only)."""
import ctypes
import types

import numpy as np
import pytest
import torch

from oracle import frames_np as F


def _check(done_pattern, T1, starts, B=None):
    done = np.asarray(done_pattern, dtype=bool)
    stacks, done = F.simulate(done.shape[0], done.shape[1], seed=len(starts), hw=(3, 4), done=done)
    for start in starts:
        st, un, d = F.rollout(stacks, done, start, T1)
        assert un.shape == (T1 + 3,) + st.shape[1:2] + (3, 4)
        assert np.array_equal(F.restack(un, d), st), start
        # uint8 done with values other than 1 are episode starts too
        assert np.array_equal(F.restack(un, d.astype(np.uint8) * 7), st), start


def test_restack_matches_simulator_on_edge_cases():
    S, B = 30, 6
    d = np.zeros((S, B), dtype=bool)       # column 0: one episode (no done after step 0)
    d[5, 1] = True                          # column 1: a done at t = 0 of the rollout starting at 5
    d[[8, 9, 10], 2] = True                 # column 2: consecutive dones (one-step episodes)
    d[13, 3] = True                         # column 3: a done in the last row of the rollout [5, 14)
    d[[6, 8, 11, 12], 4] = True             # column 4: episodes shorter than 4 steps
    d[1::3, 5] = True                       # column 5: a 3-step episode cycle
    # rollouts of T1 = 9 chained like the learner queue's (row 0 = previous rollout's last row), plus T1 = 1
    _check(d, 9, [0, 8, 16])
    _check(d, 9, [5, 13])
    _check(d, 1, [0, 3, 13, 29])


def test_restack_random_streams():
    stacks, done = F.simulate(60, 5, seed=3, done_prob=0.3, hw=(2, 2))
    for start, T1 in ((0, 21), (20, 21), (40, 21), (7, 4), (59, 1)):
        st, un, d = F.rollout(stacks, done, start, T1)
        assert np.array_equal(F.restack(un, d), st)


def test_no_done_rows_are_the_newest_frames():
    stacks, done = F.simulate(12, 2, seed=0, hw=(1, 2), done=np.zeros((12, 2), dtype=bool))
    st, un, d = F.rollout(stacks, done, 4, 6)
    assert not d.any()
    for t in range(6):
        for c in range(4):
            assert np.array_equal(st[t, :, c], un[t + c])


def test_spec_for_unstacked_shapes_and_bytes():
    from torchbeast_b200 import staging
    spec = staging.spec_for(80, 32, 6, frame_format="unstacked")
    assert spec["frame"] == ((84, 32, 84, 84), torch.uint8)
    stacked = staging.spec_for(80, 32, 6)
    assert all(spec[k] == stacked[k] for k in stacked if k != "frame")
    offs, _ = staging._carve(spec)
    assert offs["frame"][1] == 18_966_528
    h2d = sum(n for _, n in offs.values())
    h2d_stacked = sum(n for _, n in staging._carve(stacked)[0].values())
    assert h2d_stacked - h2d == 81 * 32 * 4 * 7056 - 18_966_528
    with pytest.raises(ValueError, match="frame_format"):
        staging.spec_for(4, 2, 6, frame_format="planar")


def _host_stager(spec):
    """A RolloutStager's host half (slot carving, column views, native writers) without its device buffers."""
    from torchbeast_b200 import staging
    st = staging.RolloutStager.__new__(staging.RolloutStager)
    st.spec = spec
    st._offs, st.slot_bytes = staging._carve(spec)
    st._host_raw = [torch.zeros(st.slot_bytes, dtype=torch.uint8)]
    st.host = [st._views(st._host_raw[0])]
    return st


@pytest.mark.parametrize("frame_format", ["stacked", "unstacked"])
def test_native_writers_place_unstacked_leaves(frame_format):
    from torchbeast_b200 import _lib, staging
    T, B, A = 3, 4, 6
    st = _host_stager(staging.spec_for(T, B, A, use_last_action=False, frame_format=frame_format))
    rs = np.random.RandomState(0)
    rolls = {}
    for b, how in ((2, "prepared"), (0, "column")):
        roll = {k: torch.from_numpy((rs.rand(*((shape[0],) + shape[2:])) * 100).astype(np.float64)).to(dtype)
                for k, (shape, dtype) in st.spec.items()}
        if how == "prepared":
            st.write_prepared(0, b, st.prepare_rollout(roll))
        else:
            st.write_column(0, b, roll)
        rolls[b] = roll
    for k in st.spec:
        for b, roll in rolls.items():
            assert torch.equal(st.column(0, b)[k], roll[k]), (k, b)
        assert float(st.host[0][k][:, 1].double().abs().sum()) == 0, k
    assert tuple(st.column(0, 2)["frame"].shape) == ((T + 4, 84, 84) if frame_format == "unstacked" else (T + 1, 4, 84, 84))
    bad = dict(rolls[0], frame=torch.zeros((T + 1, 4, 84, 84) if frame_format == "unstacked" else (T + 4, 84, 84),
                                           dtype=torch.uint8))
    with pytest.raises(_lib.TorchBeastB200Error, match="frame"):
        st.write_column(0, 1, bad)


def test_frame_validation():
    from torchbeast_b200 import _lib, nets
    r = torch.zeros(5, 2)
    assert nets.frame_is_unstacked(torch.zeros(8, 2, 84, 84, dtype=torch.uint8), r)
    assert not nets.frame_is_unstacked(torch.zeros(5, 2, 4, 84, 84, dtype=torch.uint8), r)
    for bad in (torch.zeros(5, 2, 84, 84, dtype=torch.uint8),      # T1 rows instead of T1 + 3
                torch.zeros(8, 3, 84, 84, dtype=torch.uint8),      # wrong B
                torch.zeros(8, 2, 84, 83, dtype=torch.uint8),      # wrong frame size
                torch.zeros(8, 2, 84, 84, dtype=torch.float32),    # wrong dtype
                torch.zeros(8, 2, 7056, dtype=torch.uint8),        # wrong rank
                torch.zeros(5, 2, 3, 84, 84, dtype=torch.uint8)):  # stacked with 3 channels
        with pytest.raises(_lib.TorchBeastB200Error, match="frame"):
            nets.frame_is_unstacked(bad, r)
    assert nets._done_bytes(torch.ones(5, 2, dtype=torch.bool), 5, 2).dtype == torch.uint8
    for bad in (None, torch.ones(5, 2, dtype=torch.float32), torch.ones(4, 2, dtype=torch.bool)):
        with pytest.raises(_lib.TorchBeastB200Error, match="done"):
            nets._done_bytes(bad, 5, 2)


def test_acting_paths_reject_unstacked_frames():
    from torchbeast_b200 import _lib, nets, polybeast_learner
    model = nets.AtariNet((4, 84, 84), 6, False, device="cpu")

    class Batch:
        def get_inputs(self):
            return (torch.zeros(4, 1, 84, 84, dtype=torch.uint8), torch.zeros(1, 1), torch.zeros(1, 1, dtype=torch.bool)), ()

        def set_outputs(self, outputs):
            raise AssertionError("an unstacked frame reached the forward")

    with pytest.raises(_lib.TorchBeastB200Error, match="stacked frames"):
        polybeast_learner.inference(types.SimpleNamespace(actor_device="cpu"), [Batch()], model)


def test_unstacked_frames_host_side_checks():
    from torchbeast_b200 import _lib
    h = _lib.lib()
    for name in ("tb_restack_frames_u8", "tb_unstacked_scratch_bytes", "tb_atarinet_forward", "tb_resnet_forward",
                 "tb_resnet_backward"):
        assert name in _lib.declared_symbols() and hasattr(ctypes.CDLL(_lib.LIB_PATH), name)
    stacked = 81 * 32 * 4 * 7056
    # the restack is fused into AtariNet bf16 / bf16x3 and ResNet bf16x3; the other backends get a stacked scratch
    assert [h.tb_unstacked_scratch_bytes(0, 81, 32, p) for p in (0, 1, 2)] == [stacked, 0, 0]
    assert [h.tb_unstacked_scratch_bytes(1, 81, 32, p) for p in (0, 1, 2)] == [stacked, stacked, 0]
    assert h.tb_unstacked_scratch_bytes(2, 81, 32, 0) == ctypes.c_size_t(-1).value
    assert h.tb_unstacked_scratch_bytes(0, 81, 32, 3) == ctypes.c_size_t(-1).value
    assert h.tb_restack_frames_u8(None, None, 4, 2, 7056, None, None) != 0 and b"null pointer" in h.tb_last_error()
    assert h.tb_restack_frames_u8(None, None, 4, 2, 7055, None, None) != 0 and b"bad sizes" in h.tb_last_error()
    P = ctypes.c_void_p(256)  # never dereferenced: every call below fails its host-side checks before a launch
    args = [None, P] + [None] * 6 + [4, 2, 6, 1, 0, 0] + [None] * 7
    assert h.tb_atarinet_forward(*args) != 0 and b"null pointer" in h.tb_last_error()
    default = [4, 84, 84, 16, 32, 32]
    args = [None, P] + [None] * 5 + default + [4, 2, 6, 1, 0, 0] + [None] * 7
    assert h.tb_resnet_forward(*args) != 0 and b"null pointer" in h.tb_last_error()
    args = [None] * 5 + default + [4, 2, 6, 1, 0, 0] + [None] * 3
    assert h.tb_resnet_backward(*args) != 0 and b"null pointer" in h.tb_last_error()
    # unstacked frames (done != NULL) rebuild (4, 84, 84) stacks for the default widths only
    for geometry in ([3, 64, 64, 16, 32, 32], [4, 84, 84, 32, 64, 64], [4, 84, 84, 16, 32, 64]):
        for precision in (0, 1, 2):
            args = [P] * 7 + geometry + [4, 2, 6, 1, 0, precision] + [P] * 7
            assert h.tb_resnet_forward(*args) != 0
            assert h.tb_last_error().decode().startswith("resnet_forward: unstacked frames (done != NULL) need the "
                                                         "(4, 84, 84) observation and the default widths (16, 32, 32)")
    # the backward re-reads the frame the first conv read, except at precision 2: a NULL frame then gets as far as the
    # geometry check (an unsupported shape stops it there)
    for precision in (0, 1, 2):
        args = [None] + [P] * 4 + [4, 16, 16, 16, 32, 32] + [4, 2, 6, 1, 0, precision] + [P] * 3
        assert h.tb_resnet_backward(*args) != 0
        want = b"resnet_backward: observation 16 x 16" if precision == 2 else b"resnet_backward: null pointer"
        assert h.tb_last_error().startswith(want), (precision, h.tb_last_error())
    # phase 3 is the whole backward, 1 and 2 its two halves; nothing else
    for phase in (0, 4, -1):
        args = [P] * 4 + [4, 2, 6, 1, 0, 0, P, P, phase, P]
        assert h.tb_atarinet_backward(*args) != 0 and b"atarinet_backward: phase must be" in h.tb_last_error()


def test_shard_rollout_keeps_the_unstacked_format():
    """Each rank's shard of an unstacked rollout restacks to that rank's shard of the stacked twin."""
    from torchbeast_b200 import learner
    stacks, done = F.simulate(12, 8, seed=5, done_prob=0.3, hw=(3, 4))
    st, un, d = F.rollout(stacks, done, 4, 6)
    state = (torch.randn(2, 8, 5), torch.randn(2, 8, 5))
    for rank in range(4):
        s_un, state_un = learner.shard_rollout(
            dict(frame=torch.from_numpy(np.ascontiguousarray(un)), done=torch.from_numpy(d.copy())), state, rank, 4)
        s_st, state_st = learner.shard_rollout(dict(frame=torch.from_numpy(np.ascontiguousarray(st))), state, rank, 4)
        assert tuple(s_un["frame"].shape) == (9, 2, 3, 4) and s_un["frame"].is_contiguous()
        assert np.array_equal(F.restack(s_un["frame"].numpy(), s_un["done"].numpy()), s_st["frame"].numpy())
        assert all(torch.equal(a, b) for a, b in zip(state_un, state_st))
