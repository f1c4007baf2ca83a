"""CPU: the float64 Gaussian-policy oracle against torch autograd of torch.distributions.Normal (log-prob, entropy, KL
and the mu / log-sigma gradients of the whole loss); its Philox / Box-Muller rule; the header constants, the bindings
and the host-side checks of the continuous entry points; the staging spec, the nets' construction and the learner's
"not built" checks, none of which needs a GPU."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from oracle import sampling_np as SO
from tests import gaussian_oracle as GO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(T, B, D, seed):
    rs = np.random.RandomState(seed)
    bl = np.concatenate([rs.randn(T, B, D), rs.uniform(-1.0, 0.5, (T, B, D))], -1)
    tl = bl + 0.3 * rs.randn(T, B, 2 * D)
    mu, l = GO.split(bl)
    acts = mu + np.exp(l) * rs.randn(T, B, D)
    return dict(bl=bl, tl=tl, actions=acts, rewards=2 * rs.randn(T, B), done=rs.rand(T, B) < 0.2,
                values=rs.randn(T, B), bootstrap=rs.randn(B), weights=rs.rand(B))


def _normal(rows):
    D = rows.shape[-1] // 2
    return torch.distributions.Normal(rows[..., :D], rows[..., D:].exp())


def _torch_loss(d, beta=None, weighted=False, ent_cost=0.0006, bl_cost=0.5):
    """The Gaussian loss block by torch autograd of torch.distributions.Normal in float64."""
    tl = torch.tensor(d["tl"], dtype=torch.float64, requires_grad=True)
    pi, mu_b = _normal(tl), _normal(torch.from_numpy(d["bl"]))
    a = torch.from_numpy(d["actions"])
    tlp, blp = pi.log_prob(a).sum(-1), mu_b.log_prob(a).sum(-1)
    kl = torch.distributions.kl_divergence(pi, mu_b).sum(-1)
    ent_row = -pi.entropy().sum(-1)
    w = torch.from_numpy(d["weights"]) if weighted else torch.ones(tl.shape[1], dtype=torch.float64)
    with torch.no_grad():
        rho = torch.exp(tlp - blp)
        if beta is not None:
            rho = torch.where(kl <= beta, rho, torch.zeros(()))
        r = torch.from_numpy(d["rewards"]).clamp(-1, 1)
        g = (~torch.from_numpy(d["done"])).double() * 0.99
        v, bs = torch.from_numpy(d["values"]), torch.from_numpy(d["bootstrap"])
        deltas = rho.clamp(max=1.0) * (r + g * torch.cat([v[1:], bs[None]]) - v)
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
    return dict(kl=kl.detach().numpy(), target_alp=tlp.detach().numpy(), behavior_alp=blp.detach().numpy(),
                log_rhos=(tlp - blp).detach().numpy(), vs=vs.numpy(), pg_adv=pg_adv.numpy(),
                losses=np.array([pg.item(), base.item(), ent.item(), total.item()]), grad_logits=tl.grad.numpy(),
                ent=ent_row.detach().numpy())


@pytest.mark.parametrize("T,B,D,seed,beta,weighted", [
    (5, 4, 1, 0, None, False), (6, 3, 6, 1, "median", True), (4, 5, 21, 2, None, True),
    (7, 2, 3, 3, "median", False), (3, 3, 64, 4, None, False)])
def test_oracle_loss_matches_autograd(T, B, D, seed, beta, weighted):
    d = _inputs(T, B, D, seed)
    if beta == "median":  # some rows exceed beta, some do not
        beta = float(np.median(GO.kl(d["tl"], d["bl"])))
    want = _torch_loss(d, beta, weighted)
    o = GO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], d["values"], d["bootstrap"],
                       weights=d["weights"] if weighted else None, trust_beta=beta)
    # c is the fp32 constant, 2.3e-8 from 0.5 log 2 pi: log pi(a) and ent move by D times that, the rest not at all
    tol = dict(rtol=1e-10, atol=3e-8 * D * T * B)
    for k in ("kl", "log_rhos", "vs", "pg_adv", "grad_logits"):
        np.testing.assert_allclose(o[k], want[k], rtol=1e-10, atol=1e-12, err_msg=k)
    for k in ("target_alp", "behavior_alp", "losses"):
        np.testing.assert_allclose(o[k], want[k], err_msg=k, **tol)
    np.testing.assert_allclose(GO.entropy_term(d["tl"], d["actions"]), want["ent"], rtol=1e-10, atol=3e-8 * D)
    if beta is not None:
        assert 0 < o["trusted"] < T * B  # some rows exceed beta, some do not


def test_oracle_popart_matches_autograd_in_normalised_space():
    T, B, D, K = 5, 3, 4, 2
    d = _inputs(T, B, D, 7)
    rs = np.random.RandomState(8)
    n = rs.randn(T + 1, B, K)
    task = rs.randint(0, K, size=(T + 1, B))
    mu, nu = np.array([0.3, -0.2]), np.array([1.5, 0.9])
    o = GO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], n, None, popart=(task, mu, nu))
    sig = np.sqrt(nu - mu * mu)
    nt = torch.tensor(n, requires_grad=True)
    nk = nt.gather(-1, torch.from_numpy(task)[..., None])[..., 0]
    v = torch.from_numpy(sig[task]) * nk + torch.from_numpy(mu[task])
    vs = torch.from_numpy(o["vs"])
    dd = (vs - torch.from_numpy(mu[task[:T]])) / torch.from_numpy(sig[task[:T]]) - nk[:T]
    (0.5 * 0.5 * (dd ** 2).sum()).backward()
    np.testing.assert_allclose(o["grad_values"], nt.grad.numpy(), rtol=1e-12, atol=1e-14)
    # the V-trace runs on the unnormalised values; the policy gradient's advantage is divided by sigma_k
    flat = GO.impala_loss(d["bl"], d["tl"], d["actions"], d["rewards"], d["done"], v.detach().numpy()[:T],
                          v.detach().numpy()[T])
    np.testing.assert_allclose(o["vs"], flat["vs"], rtol=1e-12, atol=1e-12)
    want = GO.row_grad(d["tl"], d["actions"], flat["pg_adv"] / sig[task[:T]], 0.0006)
    np.testing.assert_allclose(o["grad_logits"], want, rtol=1e-12, atol=1e-14)


def test_oracle_non_finite_entries_poison_their_row():
    d = _inputs(3, 2, 3, 10)
    tl, acts = d["tl"].copy(), d["actions"].copy()
    tl[1, 0, 4] = np.inf
    acts[2, 1, 0] = np.nan
    o = GO.impala_loss(d["bl"], tl, acts, d["rewards"], d["done"], d["values"], d["bootstrap"])
    assert np.isnan(o["target_alp"][1, 0]) and np.isnan(o["target_alp"][2, 1]) and np.isnan(o["kl"][1, 0])
    assert np.isnan(o["grad_logits"][1, 0]).all() and np.isnan(o["grad_logits"][2, 1]).all()
    assert np.isnan(o["losses"][3])  # the V-trace carries the NaN back to the earlier rows, as in the flat loss
    alp = o["target_alp"].copy()
    alp[1, 0] = alp[2, 1] = 0
    assert np.isfinite(alp).all()
    assert np.isfinite(o["kl"][2, 1])  # the KL does not read the action


def test_sampler_oracle_words_and_transform():
    T, B, D, seed, step = 2, 3, 5, 2 ** 40 + 7, 13
    x0, x1 = GO.gaussian_words(T, B, seed, step, D)
    ctr = step + np.arange(T)[:, None] + np.zeros((1, B), np.int64)
    for k in range(D):
        blk = SO.philox4x32_10((ctr, 0, np.arange(B)[None, :], 0), (seed & 0xFFFFFFFF, (seed >> 32) + k // 2))
        assert np.array_equal(x0[..., k], blk[2 * (k % 2)]) and np.array_equal(x1[..., k], blk[2 * (k % 2) + 1])
    # component 0's x0 is the flat sampler's word
    assert np.array_equal((x0[..., 0] >> 8) * 2.0 ** -24, SO.uniforms(T, B, seed, step))
    rows = np.concatenate([np.random.RandomState(0).randn(T, B, D), np.full((T, B, D), -0.5)], -1)
    a, z = GO.sample(rows, seed, step)
    u1, u2 = GO.uniforms(T, B, seed, step, D)
    assert (u1 > 0).all() and (u1 <= 1).all() and (u2 >= 0).all() and (u2 < 1).all()
    np.testing.assert_allclose(a, rows[..., :D] + np.exp(-0.5) * z, rtol=0, atol=1e-15)
    rows[1, 2, 0] = np.nan
    rows[0, 1, D + 3] = -np.inf
    a, _ = GO.sample(rows, seed, step)
    assert np.isnan(a[1, 2, 0]) and np.isnan(a[0, 1, 3]) and np.isfinite(np.delete(a.ravel(), [5 * 5, 3 + 5])).all()


def test_header_constants_and_bindings():
    from torchbeast_b200 import _lib, action_space
    with open(os.path.join(ROOT, "include", "torchbeast_b200.h")) as f:
        text = f.read()
    assert "#define TB_MAX_CONTINUOUS_DIM 64" in text and action_space.MAX_CONTINUOUS_DIM == 64
    line = [ln for ln in text.splitlines() if ln.startswith("#define TB_GAUSSIAN_HALF_LOG_2PI")][0]
    c = np.float32(float(line.split()[2].rstrip("f")))
    assert c == np.float32(0.5 * np.log(2 * np.pi)) and float(c) == GO.HALF_LOG_2PI
    for name in ("tb_impala_loss_gaussian_f32", "tb_sample_gaussian_f32", "tb_atarinet_forward_continuous",
                 "tb_atarinet_backward_continuous", "tb_atarinet_param_count_continuous",
                 "tb_atarinet_workspace_bytes_continuous"):
        assert name in _lib.declared_symbols() and hasattr(ctypes.CDLL(_lib.LIB_PATH), name)


P = ctypes.c_void_p(256)  # never dereferenced: every case below fails a host-side check before any launch


def _err():
    from torchbeast_b200 import _lib
    return _lib.lib().tb_last_error().decode()


def _loss(A, over=None):
    from torchbeast_b200 import _lib
    a = [P] * 8 + [4, 2, A, 0.99, 0.5, 0.01, 1, 1.0, 1.0] + [None] * 5 + [0] + [None] * 3 + [P] * 7 + [P, P, 1, P, None]
    for i, v in (over or {}).items():
        a[i] = v
    return _lib.lib().tb_impala_loss_gaussian_f32(*a), _err()


def _sample(A, over=None):
    from torchbeast_b200 import _lib
    a = [P, 2, 3, A, 1, 0, None, None, P, None]
    for i, v in (over or {}).items():
        a[i] = v
    return _lib.lib().tb_sample_gaussian_f32(*a), _err()


def _forward(A, over=None):
    from torchbeast_b200 import _lib
    a = [P, None, P, None, P, None, None, P, 2, 3, A, 1, 0, 0, P, None, P, P, None, None, None]
    for i, v in (over or {}).items():
        a[i] = v
    return _lib.lib().tb_atarinet_forward_continuous(*a), _err()


def _backward(A, over=None):
    from torchbeast_b200 import _lib
    a = [P, P, None, P, 2, 3, A, 1, 0, 0, P, P, 3, None]
    for i, v in (over or {}).items():
        a[i] = v
    return _lib.lib().tb_atarinet_backward_continuous(*a), _err()


@pytest.mark.parametrize("call", [_loss, _sample, _forward, _backward])
@pytest.mark.parametrize("A", [0, 1, 7, 130, -2])
def test_host_side_rejects_bad_widths(call, A):
    rc, err = call(A)
    assert rc != 0 and "must be 2D with 1 <= D <= 64" in err, err


def test_layout_queries_reject_bad_widths():
    from torchbeast_b200 import _lib
    assert _lib.lib().tb_atarinet_param_count_continuous(7, 1, 0) == -1
    assert _lib.lib().tb_atarinet_workspace_bytes_continuous(2, 3, 130, 0, 2) == 0


@pytest.mark.parametrize("call,index,msg", [
    (_loss, 2, "null actions"), (_loss, 0, "null input pointer"), (_sample, 0, "null pointer"),
    (_sample, 8, "null pointer"), (_forward, 4, "null last_action"), (_forward, 0, "null pointer"),
    (_backward, 0, "null pointer")])
def test_null_pointers_are_rejected(call, index, msg):
    rc, err = call(12, over={index: None})
    assert rc != 0 and msg in err, err


def test_gaussian_space_values():
    from torchbeast_b200 import action_space
    from torchbeast_b200._lib import TorchBeastB200Error
    g = action_space.Gaussian(6)
    assert action_space.width(g) == 12 and action_space.continuous_dim_of(g) == 6 and action_space.dims_of(g) is None
    assert action_space.continuous_dim_of(6) is None and action_space.continuous_dim_of((3, 2)) is None
    assert action_space.width(6) == 6 and action_space.width((3, 2)) == 5
    assert g == action_space.Gaussian(6) and hash(g) == hash(action_space.Gaussian(6))
    for bad in (0, 65, -1, 2.0, True, "6"):
        with pytest.raises(TorchBeastB200Error):
            action_space.Gaussian(bad)


def test_staging_spec_takes_the_space():
    from torchbeast_b200 import staging
    from torchbeast_b200.action_space import Gaussian
    spec = staging.spec_for(80, 32, Gaussian(6))
    assert spec["policy_logits"] == ((81, 32, 12), torch.float32)
    assert spec["action"] == ((81, 32, 6), torch.float32) and spec["last_action"] == ((81, 32, 6), torch.float32)
    assert staging.spec_for(80, 32, 6)["action"] == ((81, 32), torch.int64)


@pytest.mark.parametrize("D,use_lstm", [(1, False), (6, True), (15, True)])
def test_nets_build_with_a_gaussian_space(D, use_lstm):
    from torchbeast_b200 import nets
    from torchbeast_b200.action_space import Gaussian
    net = nets.AtariNet((4, 84, 84), Gaussian(D), use_lstm=use_lstm, device="cpu")
    core = 512 + D + 1
    assert net.continuous_dim == D and net.num_actions == 2 * D and net.action_dims is None
    assert net.core_size == core
    sd = net.state_dict()
    assert sd["policy.weight"].shape == (2 * D, core) and sd["policy.bias"].shape == (2 * D,)
    assert sd["baseline.weight"].shape == (1, core)
    if use_lstm:
        assert sd["core.weight_ih_l0"].shape == (4 * core, core) and net.core.input_size == core
    res = nets.ResNet(Gaussian(D), use_lstm=use_lstm, device="cpu")
    assert res.continuous_dim == D and res.num_actions == 2 * D
    assert res.state_dict()["policy.weight"].shape == (2 * D, 256 if use_lstm else 257)
    assert nets.AtariNet((4, 84, 84), 6, device="cpu").continuous_dim is None


def test_nets_reject_heads_wider_than_they_take():
    from torchbeast_b200 import nets
    from torchbeast_b200._lib import TorchBeastB200Error
    from torchbeast_b200.action_space import Gaussian
    for make in (lambda: nets.AtariNet((4, 84, 84), Gaussian(16), device="cpu"),
                 lambda: nets.ResNet(Gaussian(16), device="cpu")):
        with pytest.raises(TorchBeastB200Error, match="D <= 15"):
            make()


class _Net:
    def __init__(self, D, A, dims=None):
        self.continuous_dim, self.num_actions, self.action_dims = D, A, dims


@pytest.mark.parametrize("flags,batch,teacher,msg", [
    (dict(upgo_cost=0.5), {}, None, "UPGO (flags.upgo_cost)"),
    (dict(kickstart_cost=0.1), {}, None, "kickstarting (flags.kickstart_cost)"),
    (dict(), {"legal_actions": torch.ones(1)}, None, "legal-action masks"),
    (dict(), {"action": torch.zeros(3, 2, 6, dtype=torch.int64)}, None, "torch.int64 actions"),
    (dict(), {"last_action": torch.zeros(3, 2, dtype=torch.int64)}, None, "torch.int64 actions"),
    (dict(), {}, _Net(None, 12), "the teacher's action space 12 differs from the learner's Gaussian(dim=6)"),
    (dict(), {}, _Net(5, 10), "differs"),
])
def test_continuous_learner_raises_for_what_is_not_built(flags, batch, teacher, msg):
    from torchbeast_b200 import action_space
    from torchbeast_b200._lib import TorchBeastB200Error
    t = None if teacher is None else types.SimpleNamespace(net=teacher)
    with pytest.raises(TorchBeastB200Error) as e:
        action_space.check_learner(_Net(6, 12), types.SimpleNamespace(**flags), batch, t)
    assert msg in str(e.value)
    ok = {"action": torch.zeros(3, 2, 6), "last_action": torch.zeros(3, 2, 6)}
    action_space.check_learner(_Net(6, 12), types.SimpleNamespace(), ok, None)
    action_space.check_learner(_Net(None, 12), types.SimpleNamespace(**flags), batch, None)  # flat: no check
