"""CPU: constructor validation and state_dict round trips of the fused Adam / AdamW / RMSprop (no kernel runs)."""
import pytest
import torch

from torchbeast_b200 import _lib, optim
from torchbeast_b200.nets import AtariNet


def _net():
    return AtariNet((4, 84, 84), 6, True, device="cpu")


def _ref_params(model):
    """Reference-shaped parameters in the flat buffer's order (what a torch optimizer's checkpoint holds)."""
    return [torch.nn.Parameter(torch.zeros(s)) for _, s in model._spec]


def _assert_views(opt, keys):
    for p, off, n, shape in opt.model._views:
        for key in keys:
            assert opt.state[p][key].data_ptr() == getattr(opt, key).data_ptr() + 4 * off, key
            assert tuple(opt.state[p][key].shape) == tuple(shape)


@pytest.mark.parametrize("cls", [optim.Adam, optim.AdamW])
def test_adam_constructor_validation(cls):
    m = _net()
    with pytest.raises(_lib.TorchBeastB200Error, match="amsgrad"):
        cls(m, amsgrad=True)
    with pytest.raises(_lib.TorchBeastB200Error, match="maximize"):
        cls(m, maximize=True)
    with pytest.raises(ValueError):
        cls(m, betas=(0.9, 1.0))
    with pytest.raises(_lib.TorchBeastB200Error, match="FlatParamModule"):
        cls([torch.nn.Parameter(torch.zeros(3))])
    o = cls(m, lr=3e-4, foreach=True, capturable=True, differentiable=False, fused=True)
    with pytest.raises(_lib.TorchBeastB200Error, match="param group"):
        o.add_param_group({"params": [torch.nn.Parameter(torch.zeros(3))]})
    # the param group has exactly torch's keys, with torch's defaults for the implementation switches
    ref = (torch.optim.Adam if cls is optim.Adam else torch.optim.AdamW)(_ref_params(m), lr=3e-4)
    want = {k: v for k, v in ref.param_groups[0].items() if k != "params"}
    got = {k: v for k, v in o.param_groups[0].items() if k != "params"}
    assert got == want
    assert got["decoupled_weight_decay"] == (cls is optim.AdamW)
    assert float(o.state[m.fc.bias]["step"]) == 0


def test_rmsprop_accepts_centered_and_weight_decay():
    m = _net()
    o = optim.RMSprop(m, lr=0.00048, alpha=0.99, eps=0.01, weight_decay=1e-4, momentum=0.9, centered=True)
    assert o.grad_avg is not None and o.grad_avg.shape == m.flat_params.shape
    _assert_views(o, ("square_avg", "momentum_buffer", "grad_avg"))
    assert optim.RMSprop(_net()).grad_avg is None
    with pytest.raises(_lib.TorchBeastB200Error, match="param group"):
        o.add_param_group({"params": [torch.nn.Parameter(torch.zeros(3))]})
    # a non-centered state_dict cannot feed a centered optimizer (it has no grad_avg), nor the other way round
    with pytest.raises(_lib.TorchBeastB200Error, match="centered"):
        o.load_state_dict(optim.RMSprop(_net(), momentum=0.9).state_dict())


@pytest.mark.parametrize("cls", [optim.Adam, optim.AdamW])
def test_adam_state_dict_round_trip(tmp_path, cls):
    m = _net()
    o = cls(m, lr=2e-4, betas=(0.8, 0.99), weight_decay=0.01)
    o.exp_avg.copy_(torch.randn_like(o.exp_avg))
    o.exp_avg_sq.copy_(torch.rand_like(o.exp_avg_sq))
    o.step_device.fill_(7)
    sd = o.state_dict()
    steps = [s["step"] for s in sd["state"].values()]
    assert all(float(s) == 7.0 and s.dtype == torch.float32 for s in steps)
    assert len({id(s) for s in steps}) == len(steps)  # torch increments each parameter's step tensor on its own
    f = tmp_path / "ck.tar"
    torch.save({"optimizer_state_dict": sd}, f)
    o2 = cls(_net(), lr=0.1)
    o2.load_state_dict(torch.load(f, weights_only=True)["optimizer_state_dict"])
    assert torch.equal(o2.exp_avg, o.exp_avg) and torch.equal(o2.exp_avg_sq, o.exp_avg_sq)
    assert int(o2.step_device) == 7 and o2.param_groups[0]["lr"] == 2e-4 and o2.param_groups[0]["betas"] == (0.8, 0.99)
    assert float(o2._lr_dev) == pytest.approx(2e-4)
    _assert_views(o2, ("exp_avg", "exp_avg_sq"))
    for p, _, _, _ in o2.model._views:  # the live per-parameter step follows the device counter
        assert o2.state[p]["step"].data_ptr() == o2.step_device.data_ptr()
    o2.step_device.fill_(9)
    assert all(int(o2.state[p]["step"]) == 9 for p, _, _, _ in o2.model._views)


@pytest.mark.parametrize("name", ["Adam", "AdamW"])
def test_torch_adam_state_dict_feeds_the_flat_buffers(name):
    m = _net()
    ref_params = _ref_params(m)
    ro = getattr(torch.optim, name)(ref_params, lr=5e-4, weight_decay=0.02)
    for _ in range(3):
        for i, p in enumerate(ref_params):
            p.grad = torch.full_like(p, float(i + 1)) * torch.randn_like(p)
        ro.step()
    o = getattr(optim, name)(m, lr=1.0)
    o.load_state_dict(ro.state_dict())
    for i, (p, off, n, shape) in enumerate(m._views):
        assert torch.equal(o.exp_avg[off:off + n], ro.state[ref_params[i]]["exp_avg"].reshape(-1)), i
        assert torch.equal(o.exp_avg_sq[off:off + n], ro.state[ref_params[i]]["exp_avg_sq"].reshape(-1)), i
    assert int(o.step_device) == 3 and o.param_groups[0]["lr"] == 5e-4
    assert o.param_groups[0]["decoupled_weight_decay"] == (name == "AdamW")
    _assert_views(o, ("exp_avg", "exp_avg_sq"))


def test_ours_feeds_torch_adam():
    m = _net()
    o = optim.Adam(m, lr=5e-4, weight_decay=0.01)
    o.exp_avg.copy_(torch.randn_like(o.exp_avg))
    o.exp_avg_sq.copy_(torch.rand_like(o.exp_avg_sq))
    o.step_device.fill_(4)
    ref_params = _ref_params(m)
    ro = torch.optim.Adam(ref_params, lr=1.0)
    ro.load_state_dict(o.state_dict())
    assert ro.param_groups[0]["lr"] == 5e-4 and ro.param_groups[0]["weight_decay"] == 0.01
    for i, (p, off, n, shape) in enumerate(m._views):
        st = ro.state[ref_params[i]]
        assert float(st["step"]) == 4.0
        assert torch.equal(st["exp_avg"].reshape(-1), o.exp_avg[off:off + n]), i
        assert torch.equal(st["exp_avg_sq"].reshape(-1), o.exp_avg_sq[off:off + n]), i
    # and torch can step from it: every parameter's count advances once
    for p in ref_params:
        p.grad = torch.ones_like(p)
    ro.step()
    assert all(float(ro.state[p]["step"]) == 5.0 for p in ref_params)


def test_torch_centered_rmsprop_state_dict_feeds_the_flat_buffers(tmp_path):
    m = _net()
    ref_params = _ref_params(m)
    ro = torch.optim.RMSprop(ref_params, lr=0.00048, alpha=0.99, eps=0.01, momentum=0.5, centered=True,
                             weight_decay=1e-4)
    for _ in range(2):
        for i, p in enumerate(ref_params):
            p.grad = torch.randn_like(p) * (i + 1)
        ro.step()
    o = optim.RMSprop(m, lr=0.1, alpha=0.99, eps=0.01, momentum=0.5, centered=True, weight_decay=1e-4)
    o.load_state_dict(ro.state_dict())
    for i, (p, off, n, shape) in enumerate(m._views):
        for key in ("square_avg", "momentum_buffer", "grad_avg"):
            assert torch.equal(getattr(o, key)[off:off + n], ro.state[ref_params[i]][key].reshape(-1)), (i, key)
    assert o._steps == 2 and o.param_groups[0]["lr"] == 0.00048
    _assert_views(o, ("square_avg", "momentum_buffer", "grad_avg"))
    # and our own state_dict round-trips through torch.save / weights_only load, grad_avg included
    f = tmp_path / "ck.tar"
    torch.save(o.state_dict(), f)
    o2 = optim.RMSprop(_net(), lr=0.1, momentum=0.5, centered=True)
    o2.load_state_dict(torch.load(f, weights_only=True))
    assert torch.equal(o2.grad_avg, o.grad_avg) and torch.equal(o2.square_avg, o.square_avg)
    assert o2._steps == 2 and o2.param_groups[0]["weight_decay"] == 1e-4
    _assert_views(o2, ("square_avg", "momentum_buffer", "grad_avg"))
