"""IMPALA ResNet section widths without a GPU: the Python parameter spec against the C ABI, the fc width, the supported
set the library reports, construction errors, and the oracle's default shapes."""
import itertools
import math

import pytest

from oracle import learner_torch as LT
from torchbeast_b200 import _lib, nets

A = 6
ALL = list(itertools.product((16, 32, 64), repeat=3))
SHAPES = [(4, 84, 84), (3, 64, 64), (3, 72, 96), (2, 17, 33), (16, 126, 126)]


def lib():
    return _lib.lib()


def test_library_states_the_widths():
    assert nets.resnet_widths() == (16, 32, 64)


@pytest.mark.parametrize("obs", SHAPES)
@pytest.mark.parametrize("channels", [(16, 32, 32), (32, 64, 64), (64, 64, 64), (16, 64, 32), (64, 16, 32)])
def test_spec_matches_resnet_param_count_at_every_width(obs, channels):
    for use_lstm, num_values in ((False, 1), (True, 1), (True, 4)):
        spec = nets.resnet_param_spec(A, use_lstm, num_values, observation_shape=obs, channels=channels)
        d = dict(spec)
        assert d["feat_convs.0.0.weight"] == (channels[0], obs[0], 3, 3)
        assert d["feat_convs.1.0.weight"] == (channels[1], channels[0], 3, 3)
        assert d["feat_convs.2.0.weight"] == (channels[2], channels[1], 3, 3)
        for i in range(3):
            assert d["resnet1.%d.1.weight" % i] == d["resnet2.%d.3.weight" % i] == (channels[i], channels[i], 3, 3)
        assert d["fc.weight"] == (256, nets.resnet_fc_in(obs, channels))
        total = sum(math.prod(s) for _, s in spec)
        assert lib().tb_resnet_param_count(*obs, *channels, A, num_values, int(use_lstm)) == total


def test_fc_in():
    assert nets.resnet_fc_in() == 3872
    assert nets.resnet_fc_in((4, 84, 84), (32, 64, 64)) == 64 * 11 * 11
    assert nets.resnet_fc_in((3, 64, 64), (32, 64, 64)) == 64 * 8 * 8
    assert nets.resnet_fc_in((3, 72, 96), (16, 32, 16)) == 16 * 9 * 12
    assert nets.resnet_fc_in((2, 17, 33), (64, 64, 64)) == 64 * 3 * 5


@pytest.mark.parametrize("obs", SHAPES + [(1, 17, 126), (5, 126, 33)])
def test_every_width_tuple_is_supported_at_every_shape_and_backend(obs):
    """The library's supported set: each section 16, 32 or 64, in all 27 combinations, at every shape of the range."""
    L = lib()
    for ch in ALL:
        for precision in (0, 1, 2):
            assert L.tb_resnet_supported(*obs, *ch, precision) == 1, (ch, precision, L.tb_last_error())
            assert L.tb_resnet_workspace_bytes(*obs, *ch, 5, 3, A, 1, precision) > 0


@pytest.mark.parametrize("bad", [8, 48, 128, 0, -16, 24])
def test_other_widths_are_refused_by_every_entry(bad):
    L = lib()
    for pos in range(3):
        ch = [16, 32, 32]
        ch[pos] = bad
        for precision in (0, 1, 2):
            assert L.tb_resnet_supported(4, 84, 84, *ch, precision) == 0
            assert L.tb_last_error().decode().startswith("resnet_supported: section %d has %d channels" % (pos, bad))
        assert L.tb_resnet_param_count(4, 84, 84, *ch, A, 1, 1) == -1
        assert L.tb_resnet_workspace_bytes(4, 84, 84, *ch, 5, 3, A, 1, 2) == 0


def test_construction_errors_quote_the_supported_set():
    from torchbeast_b200 import polybeast_learner
    for bad in ((16, 32), (16, 32, 48), (16, 32, 32, 32), "abc", (8, 16, 32)):
        with pytest.raises(_lib.TorchBeastB200Error, match=r"ResNet channels must be three section widths, each one of "
                                                            r"\(16, 32, 64\), got"):
            polybeast_learner.Net(A, False, device="cpu", channels=bad)
    m = nets.ResNet(A, True, device="cpu", observation_shape=(3, 64, 64), channels=[32, 64, 64])
    assert m.channels == (32, 64, 64)
    assert m.fc.weight.shape == (256, 64 * 8 * 8)
    assert nets.ResNet(A, True, device="cpu").channels == (16, 32, 32)


def test_oracle_shapes_at_the_default_are_the_spec():
    for use_lstm in (False, True):
        assert LT.resnet_param_shapes(A, use_lstm) == dict(nets.resnet_param_spec(A, use_lstm))
        assert LT.resnet_param_shapes(A, use_lstm) == dict(nets.resnet_param_spec(A, use_lstm, channels=(16, 32, 32)))
