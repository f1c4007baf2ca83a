"""CPU: the device hyper-parameter block of the graphed learner - its packing against the compiled tb_hparams layout,
the values the packer takes from flags and from each fused optimizer, the errors it shares with the host entry points,
and which values choose a new graph (no kernel runs)."""
import ctypes
import types

import numpy as np
import pytest
import torch

from torchbeast_b200 import _lib, optim
from torchbeast_b200.learner import HPARAMS, GraphedLearner, pack_hparams
from torchbeast_b200.nets import AtariNet

FIELDS = ("discounting", "baseline_cost", "entropy_cost", "clip_rho", "clip_pg_rho", "clip_rewards", "max_norm",
          "alpha", "eps", "momentum", "weight_decay", "beta1", "beta2")  # tb_hparams_layout's order


def _flags(**kw):
    f = dict(discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, reward_clipping="abs_one",
             grad_norm_clipping=40.0)
    f.update(kw)
    return types.SimpleNamespace(**f)


def _net():
    return AtariNet((4, 84, 84), 6, True, device="cpu")


def _batch(done_dtype=torch.bool):
    return {"done": torch.zeros(3, 2, dtype=done_dtype)}


def test_layout_matches_the_library():
    out = (ctypes.c_int64 * (1 + len(FIELDS)))()
    _lib.check(_lib.lib().tb_hparams_layout(ctypes.cast(out, ctypes.c_void_p)), "tb_hparams_layout")
    assert out[0] == HPARAMS.itemsize == 64
    assert list(out[1:]) == [HPARAMS.fields[name][1] for name in FIELDS]
    assert sorted(HPARAMS.names) == sorted(FIELDS)
    for name in FIELDS:
        want = {"clip_rewards": np.int32, "beta1": np.float64, "beta2": np.float64}.get(name, np.float32)
        assert HPARAMS.fields[name][0] == np.dtype(want), name


def test_pack_reference_rmsprop():
    opt = optim.RMSprop(_net(), lr=0.00048, momentum=0, eps=0.01, alpha=0.99)
    rec = pack_hparams(_flags(), opt)
    assert rec.dtype == HPARAMS and rec.shape == ()
    assert rec["discounting"] == np.float32(0.99) and rec["baseline_cost"] == np.float32(0.5)
    assert rec["entropy_cost"] == np.float32(0.0006) and rec["clip_rewards"] == 1
    assert rec["clip_rho"] == 1.0 and rec["clip_pg_rho"] == 1.0  # learn()'s V-trace clips
    assert rec["max_norm"] == np.float32(40.0)
    assert rec["alpha"] == np.float32(0.99) and rec["eps"] == np.float32(0.01)
    assert rec["momentum"] == 0 and rec["weight_decay"] == 0
    assert rec["beta1"] == 0 and rec["beta2"] == 0


def test_pack_centered_momentum_weight_decay_rmsprop():
    opt = optim.RMSprop(_net(), lr=4.8e-4, alpha=0.95, eps=1e-4, weight_decay=1e-4, momentum=0.9, centered=True)
    rec = pack_hparams(_flags(reward_clipping="none", grad_norm_clipping=None, discounting=0.97), opt)
    assert rec["clip_rewards"] == 0
    assert rec["max_norm"] < 0
    assert rec["discounting"] == np.float32(0.97)
    assert rec["alpha"] == np.float32(0.95) and rec["eps"] == np.float32(1e-4)
    assert rec["momentum"] == np.float32(0.9) and rec["weight_decay"] == np.float32(1e-4)
    # what the host entry point would get: the value rounded to float32 by the C argument conversion
    assert rec["weight_decay"] == ctypes.c_float(1e-4).value


@pytest.mark.parametrize("cls", [optim.Adam, optim.AdamW])
def test_pack_adam(cls):
    betas = (0.8123456789012345, 0.9991234567890123)
    opt = cls(_net(), lr=3e-4, betas=betas, eps=1e-6, weight_decay=0.02)
    rec = pack_hparams(_flags(), opt)
    assert rec["beta1"].dtype == np.float64 and rec["beta1"] == betas[0] and rec["beta2"] == betas[1]  # round trip
    assert rec["eps"] == np.float32(1e-6) and rec["weight_decay"] == np.float32(0.02)
    assert rec["alpha"] == 0 and rec["momentum"] == 0
    raw = np.frombuffer(rec.tobytes(), dtype=np.uint8)
    assert raw.size == 64
    assert np.frombuffer(raw[HPARAMS.fields["beta2"][1]:][:8].tobytes(), dtype="<f8")[0] == betas[1]


def test_pack_follows_changes():
    opt = optim.RMSprop(_net(), lr=4.8e-4, eps=0.01, momentum=0.5)
    flags = _flags()
    flags.entropy_cost, flags.baseline_cost = 0.01, 0.25
    opt.param_groups[0]["eps"] = 1e-3
    opt.param_groups[0]["momentum"] = 0.7
    rec = pack_hparams(flags, opt)
    assert rec["entropy_cost"] == np.float32(0.01) and rec["baseline_cost"] == np.float32(0.25)
    assert rec["eps"] == np.float32(1e-3) and rec["momentum"] == np.float32(0.7)


def test_unknown_reward_clipping_raises_like_the_loss():
    # impala_loss_fwd_bwd raises this ValueError for the same value (it checks CUDA tensors first, so not run here)
    with pytest.raises(ValueError, match=r"^reward_clipping must be 'abs_one' or 'none'$"):
        pack_hparams(_flags(reward_clipping="soft_asymmetric"), optim.RMSprop(_net()))


def _host_error(fn, *args):
    """The message _lib.check raises for a call the library rejects host side, before anything is launched."""
    with pytest.raises(_lib.TorchBeastB200Error) as err:
        _lib.check(fn(*args), fn.__name__)
    return str(err.value)


# non-null stand-ins: the calls below fail their host-side checks before any launch or device access
_P = ctypes.c_void_p(256)


@pytest.mark.parametrize("centered,weight_decay", [(False, 0), (False, 1e-4), (True, 0)])
def test_momentum_without_buffer_matches_the_null_hp_entry_point_error(centered, weight_decay):
    opt = optim.RMSprop(_net(), lr=4.8e-4, centered=centered, weight_decay=weight_decay)
    assert opt.momentum_buffer is None
    opt.param_groups[0]["momentum"] = 0.9
    lib = _lib.lib()
    if not centered and weight_decay == 0:
        want = _host_error(lib.tb_clip_rmsprop_step_f32, _P, _P, _P, None, 8, _P, 40.0, None, 1e-3, 0.99, 0.01, 0.9,
                           None, None, None)
    else:
        want = _host_error(lib.tb_clip_rmsprop_ex_step_f32, _P, _P, _P, _P if centered else None, None, 8, _P, 40.0,
                           None, 1e-3, 0.99, 0.01, weight_decay, 0.9, None, None, None)
    assert "momentum needs a buffer" in want
    with pytest.raises(_lib.TorchBeastB200Error) as err:
        pack_hparams(_flags(), opt)
    assert str(err.value) == want


@pytest.mark.parametrize("betas", [(1.0, 0.999), (0.9, 1.0), (-0.1, 0.999), (0.9, -1e-9)])
def test_betas_outside_range_match_the_null_hp_entry_point_error(betas):
    opt = optim.Adam(_net(), lr=3e-4)
    opt.param_groups[0]["betas"] = betas
    want = _host_error(_lib.lib().tb_clip_adam_step_f32, None, None, None, None, 0, _P, 40.0, None, 3e-4,
                       float(betas[0]), float(betas[1]), 1e-8, 0.0, 0, _P, None, None, None)
    assert "betas must be in [0, 1)" in want
    with pytest.raises(_lib.TorchBeastB200Error) as err:
        pack_hparams(_flags(), opt)
    assert str(err.value) == want


def test_structure_changes_with_structural_values_only():
    batch = _batch()
    opt = optim.RMSprop(_net(), lr=4.8e-4, eps=0.01, momentum=0.5)
    key = GraphedLearner.structure_of(opt, batch)
    g = opt.param_groups[0]
    # non-structural: every value the block carries, and the lr
    for k, v in (("lr", 1e-3), ("alpha", 0.9), ("eps", 1e-5), ("momentum", 0.7)):
        g[k] = v
        assert GraphedLearner.structure_of(opt, batch) == key, k
    # structural: momentum zero vs non-zero, weight_decay zero vs non-zero, done dtype
    g["momentum"] = 0.0
    off = GraphedLearner.structure_of(opt, batch)
    assert off != key
    g["momentum"] = 1e-50  # rounds to 0.0f, as the host entry point's argument: no momentum buffer, like 0
    assert GraphedLearner.structure_of(opt, batch) == off
    g["momentum"] = 0.7
    assert GraphedLearner.structure_of(opt, batch) == key
    g["weight_decay"] = 1e-4
    wd_key = GraphedLearner.structure_of(opt, batch)
    assert wd_key != key
    g["weight_decay"] = 2e-4
    assert GraphedLearner.structure_of(opt, batch) == wd_key
    g["weight_decay"] = 0
    assert GraphedLearner.structure_of(opt, _batch(torch.uint8)) != key
    # centered
    centered = optim.RMSprop(_net(), lr=4.8e-4, eps=0.01, momentum=0.5, centered=True)
    assert GraphedLearner.structure_of(centered, batch) != key


def test_adam_structure():
    batch = _batch()
    adam, adamw = optim.Adam(_net(), weight_decay=0.01), optim.AdamW(_net(), weight_decay=0.01)
    key = GraphedLearner.structure_of(adam, batch)
    assert GraphedLearner.structure_of(adamw, batch) != key
    g = adam.param_groups[0]
    for k, v in (("lr", 1e-2), ("betas", (0.5, 0.9)), ("eps", 1e-3), ("weight_decay", 0.0), ("weight_decay", 0.1)):
        g[k] = v
        assert GraphedLearner.structure_of(adam, batch) == key, k
    assert GraphedLearner.structure_of(adam, _batch(torch.uint8)) != key
    # an RMSprop is another launch sequence altogether
    assert GraphedLearner.structure_of(optim.RMSprop(_net()), batch) != key
