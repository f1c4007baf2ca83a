"""CPU: the float64 factored-action-space oracle against torch autograd of the same formulas (per-segment log-softmax,
summed log-probabilities, entropy and KL); its Philox rule against the flat sampler's; the tb_action_space layout, the
bindings and the host-side checks of the factored entry points; the net, staging and learner checks that need no
GPU."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from oracle import sampling_np as SO
from tests import factored_oracle as FO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(T, B, dims, seed):
    rs = np.random.RandomState(seed)
    A = sum(dims)
    acts = np.stack([rs.randint(0, a, size=(T, B)) for a in dims], -1).astype(np.int64)
    return dict(bl=2 * rs.randn(T, B, A), tl=2 * rs.randn(T, B, A), actions=acts, rewards=2 * rs.randn(T, B),
                done=rs.rand(T, B) < 0.2, values=rs.randn(T, B), bootstrap=rs.randn(B), weights=rs.rand(B))


def _torch_loss(d, dims, beta=None, weighted=False, ent_cost=0.0006, bl_cost=0.5):
    """The factored loss block by torch autograd: per-segment log_softmax, log pi(a) summed over components."""
    tl = torch.tensor(d["tl"], dtype=torch.float64, requires_grad=True)
    segs_t = [torch.log_softmax(s, -1) for s in tl.split(dims, -1)]
    segs_b = [torch.log_softmax(s, -1) for s in torch.from_numpy(d["bl"]).split(dims, -1)]
    a = torch.from_numpy(d["actions"])
    tlp = sum(s.gather(-1, a[..., k:k + 1])[..., 0] for k, s in enumerate(segs_t))
    blp = sum(s.gather(-1, a[..., k:k + 1])[..., 0] for k, s in enumerate(segs_b))
    kl = sum((s.exp() * (s - sb)).sum(-1) for s, sb in zip(segs_t, segs_b))
    ent_row = sum((s.exp() * s).sum(-1) for s in segs_t)
    w = torch.from_numpy(d["weights"]) if weighted else torch.ones(tl.shape[1], dtype=torch.float64)
    with torch.no_grad():
        rho = torch.exp(tlp - blp)
        if beta is not None:
            rho = torch.where(kl <= beta, rho, torch.zeros(()))
        r = torch.from_numpy(d["rewards"]).clamp(-1, 1)
        g = (~torch.from_numpy(d["done"])).double() * 0.99
        v, bs = torch.from_numpy(d["values"]), torch.from_numpy(d["bootstrap"])
        v_next = torch.cat([v[1:], bs[None]])
        deltas = rho.clamp(max=1.0) * (r + g * v_next - v)
        acc, vs = torch.zeros_like(bs), torch.zeros_like(v)
        for t in range(v.shape[0] - 1, -1, -1):
            acc = deltas[t] + g[t] * rho[t].clamp(max=1.0) * acc
            vs[t] = acc + v[t]
        pg_adv = rho.clamp(max=1.0) * (r + g * torch.cat([vs[1:], bs[None]]) - v)
    pg = (-tlp * pg_adv * w).sum()
    ent = ent_cost * (ent_row * w).sum()
    base = bl_cost * (0.5 * (vs - v) ** 2 * w).sum()
    total = pg + base + ent
    total.backward()
    return dict(kl=kl.detach().numpy(), log_rhos=(tlp - blp).detach().numpy(), vs=vs.numpy(), pg_adv=pg_adv.numpy(),
                losses=np.array([pg.item(), base.item(), ent.item(), total.item()]), grad_logits=tl.grad.numpy())


@pytest.mark.parametrize("T,B,dims,seed,beta,weighted", [
    (5, 4, (3, 3, 2), 0, None, False), (6, 3, (3, 3, 2), 1, 0.8, True), (4, 5, (2, 1, 5, 1, 4, 3, 1), 2, None, True),
    (7, 2, (6,), 3, 0.3, False), (3, 3, tuple(range(1, 17)), 4, None, False)])
def test_oracle_loss_matches_autograd(T, B, dims, seed, beta, weighted):
    d = _inputs(T, B, dims, seed)
    want = _torch_loss(d, dims, beta, weighted)
    o = FO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], d["values"], d["bootstrap"], dims,
                       weights=d["weights"] if weighted else None, trust_beta=beta)
    for k in ("kl", "log_rhos", "vs", "pg_adv", "losses", "grad_logits"):
        np.testing.assert_allclose(o[k], want[k], rtol=1e-10, atol=1e-12, err_msg=k)


def test_oracle_popart_matches_autograd_in_normalised_space():
    T, B, dims, K = 5, 3, (3, 3, 2), 2
    d = _inputs(T, B, dims, 7)
    rs = np.random.RandomState(8)
    n = rs.randn(T + 1, B, K)
    task = rs.randint(0, K, size=(T + 1, B))
    mu, nu = np.array([0.3, -0.2]), np.array([1.5, 0.9])
    o = FO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], n, None, dims, popart=(task, mu, nu))
    sig = np.sqrt(nu - mu * mu)
    nt = torch.tensor(n, requires_grad=True)
    nk = nt.gather(-1, torch.from_numpy(task)[..., None])[..., 0]
    v = torch.from_numpy(sig[task]) * nk + torch.from_numpy(mu[task])
    vs = torch.from_numpy(o["vs"])
    dd = (vs - torch.from_numpy(mu[task[:T]])) / torch.from_numpy(sig[task[:T]]) - nk[:T]
    (0.5 * 0.5 * (dd ** 2).sum()).backward()
    np.testing.assert_allclose(o["grad_values"], nt.grad.numpy(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(o["losses"][1], 0.5 * 0.5 * (dd.detach() ** 2).sum().item(), rtol=1e-12)
    # the V-trace runs on the unnormalised values: the flat oracle of the same values gives the same vs
    flat = FO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], v.detach().numpy()[:T],
                          v.detach().numpy()[T], dims)
    np.testing.assert_allclose(o["vs"], flat["vs"], rtol=1e-12, atol=1e-12)


def test_oracle_properties_of_size_one_components():
    """A size-1 component adds exactly 0; a space of size-1 components around one segment is that segment's flat loss."""
    T, B = 4, 3
    d = _inputs(T, B, (5,), 9)
    big = FO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], d["values"], d["bootstrap"], (5,))
    pad = lambda x: np.concatenate([np.random.RandomState(1).randn(T, B, 1), x, np.random.RandomState(2).randn(T, B, 2)], -1)
    acts = np.concatenate([np.zeros((T, B, 1), np.int64), d["actions"], np.zeros((T, B, 2), np.int64)], -1)
    o = FO.impala_loss(pad(d["bl"]), pad(d["tl"]), acts, d["rewards"], d["done"], d["values"], d["bootstrap"],
                       (1, 5, 1, 1))
    for k in ("vs", "log_rhos", "losses", "kl"):
        np.testing.assert_allclose(o[k], big[k], rtol=1e-13, atol=1e-15, err_msg=k)
    np.testing.assert_allclose(o["grad_logits"][..., 1:6], big["grad_logits"], rtol=1e-13, atol=1e-15)
    assert np.all(o["grad_logits"][..., [0, 6, 7]] == 0)


def test_oracle_out_of_range_component_is_nan():
    d = _inputs(3, 2, (3, 2), 10)
    acts = d["actions"].copy()
    acts[1, 0, 1] = 2
    o = FO.impala_loss(d["bl"], d["tl"], acts, d["rewards"], d["done"], d["values"], d["bootstrap"], (3, 2))
    assert np.isnan(o["target_alp"][1, 0]) and np.isnan(o["losses"][3])
    assert np.isfinite(np.delete(o["target_alp"].ravel(), 2)).all()


def test_sampler_oracle_one_component_is_the_flat_rule():
    x = 3 * np.random.RandomState(11).randn(4, 5, 6)
    want, _ = SO.sample_actions(x, 2 ** 40 + 7, 13)
    got, _ = FO.sample_actions(x, (6,), 2 ** 40 + 7, 13)
    assert np.array_equal(got[..., 0], want)
    # components 4..7 use the words of the block keyed hi32(seed) + 1
    w = FO.factored_words(2, 3, 5, 0, 9)
    assert np.array_equal((w[..., 0] >> 8) * 2.0 ** -24, SO.uniforms(2, 3, 5, 0))
    blk = SO.philox4x32_10((np.arange(2)[:, None] + np.zeros((1, 3), np.int64), 0, np.arange(3)[None, :], 0), (5, 1))
    for k in range(4, 8):
        assert np.array_equal(w[..., k], blk[k % 4])


def test_header_layout_and_bindings():
    from torchbeast_b200 import _lib, action_space
    with open(os.path.join(ROOT, "include", "torchbeast_b200.h")) as f:
        text = f.read()
    assert "#define TB_MAX_ACTION_COMPONENTS 16" in text
    for name in ("tb_impala_loss_factored_f32", "tb_sample_actions_factored_f32", "tb_atarinet_forward_factored",
                 "tb_action_space_layout"):
        assert name in _lib.declared_symbols() and hasattr(ctypes.CDLL(_lib.LIB_PATH), name)
    out = (ctypes.c_int64 * 3)()
    assert _lib.lib().tb_action_space_layout(ctypes.cast(out, ctypes.c_void_p)) == 0
    C = action_space.CActionSpace
    assert list(out) == [ctypes.sizeof(C), C.num_components.offset, C.dims.offset] == [68, 0, 4]


P = ctypes.c_void_p(256)  # never dereferenced: every case below fails a host-side check before any launch


def _space(dims, D=None):
    from torchbeast_b200 import action_space
    s = action_space.CActionSpace()
    s.num_components = len(dims) if D is None else D
    for k, a in enumerate(dims[:16]):
        s.dims[k] = a
    return ctypes.byref(s)


def _loss(space, A=8, over=None):
    from torchbeast_b200 import _lib
    a = [P] * 8 + [4, 2, A, 0.99, 0.5, 0.01, 1, 1.0, 1.0] + [None] * 5 + [0] + [None] * 3 + [P] * 7 + [P, P, 1, space,
                                                                                                   P, None]
    for i, v in (over or {}).items():
        a[i] = v
    rc = _lib.lib().tb_impala_loss_factored_f32(*a)
    return rc, _lib.lib().tb_last_error().decode()


def _sample(space, A=8):
    from torchbeast_b200 import _lib
    rc = _lib.lib().tb_sample_actions_factored_f32(P, 2, 3, A, 1, 0, None, None, space, P, None)
    return rc, _lib.lib().tb_last_error().decode()


def _forward(space, A=8):
    from torchbeast_b200 import _lib
    rc = _lib.lib().tb_atarinet_forward_factored(P, None, P, None, P, None, None, P, 2, 3, A, 1, 0, 0, P, None, P, P,
                                                 None, None, space, None)
    return rc, _lib.lib().tb_last_error().decode()


@pytest.mark.parametrize("call", [_loss, _sample, _forward])
@pytest.mark.parametrize("space,A,msg", [
    (None, 8, "null action space"),
    ((3, 3, 2, 0), 8, "component 3 has 0 actions"),
    ((3, -1, 2), 8, "component 1 has -1 actions"),
    ((3, 3, 2), 9, "add up to 8, not A = 9"),
    ((3, 3, 3), 8, "add up to more than A = 8"),
    ((), 8, "num_components 0 outside [1, 16]"),
    ((1,) * 17, 17, "num_components 17 outside [1, 16]"),
])
def test_host_side_checks(call, space, A, msg):
    arg = None if space is None else _space(space)
    rc, err = call(arg, A=A)
    assert rc != 0 and msg in err, err


def test_loss_null_pointers_are_rejected():
    rc, err = _loss(_space((3, 3, 2)), over={2: None})
    assert rc != 0 and "null input pointer" in err, err


def test_dims_of_and_width():
    from torchbeast_b200 import action_space
    from torchbeast_b200._lib import TorchBeastB200Error
    assert action_space.dims_of(6) is None and action_space.width(6) == 6
    assert action_space.dims_of((3, 3, 2)) == (3, 3, 2) and action_space.width([3, 3, 2]) == 8
    for bad in ((), (3, 0), (2.0, 3), (True, 2), (1,) * 17):
        with pytest.raises(TorchBeastB200Error):
            action_space.dims_of(bad)


def test_staging_spec_takes_the_tuple():
    from torchbeast_b200 import staging
    spec = staging.spec_for(80, 32, (3, 3, 2))
    assert spec["policy_logits"] == ((81, 32, 8), torch.float32)
    assert spec["action"] == ((81, 32, 3), torch.int64) and spec["last_action"] == ((81, 32, 3), torch.int64)
    assert staging.spec_for(80, 32, 6) == staging.spec_for(80, 32, 6)
    assert staging.spec_for(80, 32, 6)["action"] == ((81, 32), torch.int64)


class _Net:
    def __init__(self, dims, A):
        self.action_dims, self.num_actions = dims, A


@pytest.mark.parametrize("flags,batch,teacher,msg", [
    (dict(upgo_cost=0.5), {}, None, "UPGO (flags.upgo_cost)"),
    (dict(kickstart_cost=0.1), {}, None, "kickstarting (flags.kickstart_cost)"),
    (dict(), {"legal_actions": torch.ones(1)}, None, "legal-action masks"),
    (dict(), {}, _Net(None, 8), "the teacher's action space 8 differs from the learner's (3, 3, 2)"),
    (dict(), {}, _Net((3, 5), 8), "differs"),
])
def test_factored_learner_raises_for_what_is_not_built(flags, batch, teacher, msg):
    from torchbeast_b200 import action_space
    from torchbeast_b200._lib import TorchBeastB200Error
    t = None if teacher is None else types.SimpleNamespace(net=teacher)
    with pytest.raises(TorchBeastB200Error) as e:
        action_space.check_learner(_Net((3, 3, 2), 8), types.SimpleNamespace(**flags), batch, t)
    assert msg in str(e.value)
    action_space.check_learner(_Net(None, 8), types.SimpleNamespace(**flags), batch, None)  # flat: no check


def test_nets_take_the_tuple_on_the_host():
    from torchbeast_b200 import nets
    from torchbeast_b200._lib import TorchBeastB200Error
    net = nets.AtariNet((4, 84, 84), (3, 3, 2), use_lstm=False, device="cpu")
    assert net.action_dims == (3, 3, 2) and net.num_actions == 8 and net.core_size == 521
    assert net.policy.weight.shape == (8, 521)
    assert nets.AtariNet((4, 84, 84), 6, device="cpu").action_dims is None
    with pytest.raises(TorchBeastB200Error, match="512 \\+ sum\\(num_actions\\) \\+ 1 <= 700"):
        nets.AtariNet((4, 84, 84), (100, 100), use_lstm=True, device="cpu")
    res = nets.ResNet((5, 4), device="cpu")
    assert res.action_dims == (5, 4) and res.num_actions == 9 and res.policy.weight.shape == (9, 257)
