"""IMPALA ResNet on other observation shapes, without a GPU: the Python parameter spec against the C ABI's layout, the
default layout and workspace sizes pinned to the values they had before the ABI took an observation shape, and the
supported range enforced when the model is constructed."""
import pytest
import torch

from torchbeast_b200 import _lib
from torchbeast_b200.nets import ResNet, resnet_fc_in, resnet_obs_range, resnet_param_spec

DEFAULT_WIDTHS = (16, 32, 32)
SHAPES = [(4, 84, 84), (3, 64, 64), (3, 72, 96), (12, 64, 64), (1, 84, 84), (3, 37, 53), (16, 17, 126), (5, 126, 33),
          (2, 17, 33)]


def _numel(shape):
    n = 1
    for d in shape:
        n *= d
    return n


def _pooled(s):
    for _ in range(3):
        s = -(-s // 2)   # MaxPool2d(3, 2, 1): ceil
    return s


@pytest.mark.parametrize("obs", SHAPES)
@pytest.mark.parametrize("use_lstm", [False, True])
@pytest.mark.parametrize("num_values", [1, 4])
def test_spec_agrees_with_resnet_param_count(obs, use_lstm, num_values):
    spec = dict(resnet_param_spec(7, use_lstm, num_values=num_values, observation_shape=obs))
    C, H, W = obs
    assert spec["feat_convs.0.0.weight"] == (16, C, 3, 3)
    assert spec["fc.weight"] == (256, 32 * _pooled(H) * _pooled(W)) and resnet_fc_in(obs) == 32 * _pooled(H) * _pooled(W)
    total = sum(_numel(s) for s in spec.values())
    assert _lib.lib().tb_resnet_param_count(C, H, W, *DEFAULT_WIDTHS, 7, num_values, int(use_lstm)) == total
    for precision in range(3):
        assert _lib.lib().tb_resnet_supported(C, H, W, *DEFAULT_WIDTHS, precision) == 1
        assert _lib.lib().tb_resnet_workspace_bytes(C, H, W, *DEFAULT_WIDTHS, 5, 3, 7, int(use_lstm), precision) > 0


# the (4, 84, 84) parameter count (A, use_lstm, V) and workspace bytes (T1, B, use_lstm; precision 0 / 1 / 2, A = 6) as
# the library reported them before it took an observation shape (the (4, 84, 84) constants): the default layout and
# workspace must not move
PARAM_COUNTS = {(6, 0, 1): 1091038, (6, 0, 4): 1091812, (6, 1, 1): 1618391, (6, 1, 4): 1619162,
                (18, 0, 1): 1094134, (18, 0, 4): 1094908, (18, 1, 1): 1621475, (18, 1, 4): 1622246}
WORKSPACE_BYTES = {
    (1, 1, 0): (44085248, 39484160, 49403392), (1, 1, 1): (46398208, 42347520, 53013760),
    (5, 3, 0): (115836416, 77276160, 127442944), (5, 3, 1): (118385152, 80442368, 132078592),
    (81, 8, 0): (3360040704, 1786116352, 3655878912), (81, 8, 1): (3372379392, 1801719296, 3688049920),
    (81, 32, 0): (13323289344, 7034123008, 14492030208), (81, 32, 1): (13365783040, 7088050688, 14570695680),
    (81, 64, 0): (26607620864, 14031465216, 28940231936), (81, 64, 1): (26690321408, 14136493056, 29080890880),
}


def test_default_geometry_layout_and_workspace_unchanged():
    lib = _lib.lib()
    for (A, lstm, V), count in PARAM_COUNTS.items():
        assert lib.tb_resnet_param_count(4, 84, 84, *DEFAULT_WIDTHS, A, V, lstm) == count
        assert sum(_numel(s) for _, s in resnet_param_spec(A, bool(lstm), num_values=V)) == count
    for (T1, B, lstm), sizes in WORKSPACE_BYTES.items():
        for precision, nbytes in enumerate(sizes):
            assert lib.tb_resnet_workspace_bytes(4, 84, 84, *DEFAULT_WIDTHS, T1, B, 6, lstm, precision) == nbytes
    d = dict(resnet_param_spec(6, True))
    assert d["feat_convs.0.0.weight"] == (16, 4, 3, 3) and d["fc.weight"] == (256, 3872)


def test_model_layout_at_new_shape():
    model = ResNet(5, True, device=torch.device("cpu"), observation_shape=(3, 72, 96))
    assert model.observation_shape == (3, 72, 96)
    shapes = {n: tuple(p.shape) for n, p in model.named_parameters()}
    assert shapes["feat_convs.0.0.weight"] == (16, 3, 3, 3)
    assert shapes["fc.weight"] == (256, 32 * 9 * 12)
    assert ResNet(5, device=torch.device("cpu")).observation_shape == (4, 84, 84)


def test_range_is_the_libraries_and_exactly_what_resnet_supported_accepts():
    """The documented range, read from the C library, is the set tb_resnet_supported accepts on every backend, and
    its lower bounds are the smallest sides whose last section is 3 high and 5 wide (the smallest image of the
    shifted-window kernels; the narrowest row their weight gradient takes)."""
    rng = resnet_obs_range()
    assert rng == {"C": (1, 16), "H": (17, 126), "W": (33, 126)}
    assert _pooled(rng["H"][0]) == 3 and _pooled(rng["H"][0] - 1) == 2
    assert _pooled(rng["W"][0]) == 5 and _pooled(rng["W"][0] - 1) == 4
    lib = _lib.lib()
    for precision in range(3):
        for H in range(1, 131):
            for W in range(1, 131):
                want = rng["H"][0] <= H <= rng["H"][1] and rng["W"][0] <= W <= rng["W"][1]
                assert lib.tb_resnet_supported(3, H, W, *DEFAULT_WIDTHS, precision) == int(want), (H, W, precision)
        for C in range(0, 18):
            assert lib.tb_resnet_supported(C, 64, 64, *DEFAULT_WIDTHS, precision) == int(rng["C"][0] <= C <= rng["C"][1])


# (3, 32, 17) .. (3, 32, 32): last section 3 or 4 wide, narrower than the weight-gradient kernel's last pixel step allows
BAD = [(0, 84, 84), (17, 84, 84), (3, 16, 64), (3, 64, 16), (3, 32, 17), (3, 64, 32), (3, 64, 127), (3, 127, 64), (3, 8, 8),
       (3, 64), (3, 64, 64, 1)]


@pytest.mark.parametrize("obs", BAD)
def test_out_of_range_shape_raises_and_every_entry_refuses_it(obs):
    rng = resnet_obs_range()
    with pytest.raises(_lib.TorchBeastB200Error, match=r"observation_shape must be \(C, H, W\) with C in \[%d, %d\], H in "
                                                      r"\[%d, %d\] and W in \[%d, %d\]" % (rng["C"] + rng["H"] + rng["W"])):
        ResNet(6, device=torch.device("cpu"), observation_shape=obs)
    if len(obs) == 3:
        lib = _lib.lib()
        for precision in range(3):
            assert lib.tb_resnet_supported(*obs, *DEFAULT_WIDTHS, precision) == 0
            assert lib.tb_last_error().decode().startswith("resnet_supported: observation")
        assert lib.tb_resnet_param_count(*obs, *DEFAULT_WIDTHS, 6, 1, 0) == -1
        assert lib.tb_resnet_workspace_bytes(*obs, *DEFAULT_WIDTHS, 2, 2, 6, 0, 2) == 0


def test_range_edges_are_supported():
    rng = resnet_obs_range()
    (h0, h1), (w0, w1) = rng["H"], rng["W"]
    for obs in ((1, h0, w0), (16, h1, w1), (16, h0, w1), (1, h1, w0)):
        ResNet(6, device=torch.device("cpu"), observation_shape=obs)


def test_frame_checks_name_the_model_shape():
    from torchbeast_b200.nets import frame_is_unstacked
    reward = torch.zeros(2, 3)
    assert frame_is_unstacked(torch.zeros(2, 3, 3, 64, 64, dtype=torch.uint8), reward, (3, 64, 64)) is False
    with pytest.raises(_lib.TorchBeastB200Error, match=r"frame must be uint8 \[T,B,3,64,64\], got"):
        frame_is_unstacked(torch.zeros(2, 3, 4, 84, 84, dtype=torch.uint8), reward, (3, 64, 64))
    with pytest.raises(_lib.TorchBeastB200Error, match=r"unstacked rollouts and newest frames rebuild \(4, 84, 84\) stacks"):
        frame_is_unstacked(torch.zeros(5, 3, 84, 84, dtype=torch.uint8), reward, (3, 64, 64))
    with pytest.raises(_lib.TorchBeastB200Error, match=r"frame must be uint8 \[T,B,4,84,84\], got"):
        frame_is_unstacked(torch.zeros(2, 3, 3, 64, 64, dtype=torch.uint8), reward)


def test_frame_history_rejected_on_new_shape():
    from torchbeast_b200.acting import FrameHistory
    model = ResNet(6, device=torch.device("cpu"), observation_shape=(3, 64, 64))
    model.frame_history = FrameHistory(2, device=torch.device("cpu"))
    inputs = dict(frame=torch.zeros(1, 2, 64, 64, dtype=torch.uint8), reward=torch.zeros(1, 2),
                  done=torch.zeros(1, 2, dtype=torch.bool))
    with pytest.raises(_lib.TorchBeastB200Error, match=r"a frame_history rebuilds \(4, 84, 84\) stacks"):
        model._forward_frame(inputs)
