"""CPU: the PopArt restatement (tests/popart_oracle.py) reduces to the reference learn step with one task, identity
statistics and beta = 0; the statistics update and the output-preserving rescale; the nets' PopArt state; the C ABI."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import learner_torch as LT
from tests import popart_oracle as PO
from tests.common import golden
from tests.test_oracle_golden import LEARN_CASES


def _golden_case(fname, net):
    g = golden(fname)
    T, B, A, seed, use_lstm = [int(x) for x in g["meta"]]
    batch = LT.synthetic_batch(T, B, A, seed=seed, with_last_action=(net == "atari"))
    shapes = LT.atarinet_param_shapes(A, bool(use_lstm)) if net == "atari" else LT.resnet_param_shapes(A, bool(use_lstm))
    p = LT.random_params(shapes, seed=seed + 100)
    state = ()
    if use_lstm:
        L, H = (2, 512 + A + 1) if net == "atari" else (1, 256)
        rs = np.random.RandomState(seed + 7)
        state = tuple(torch.from_numpy(rs.randn(L, B, H).astype(np.float32) * 0.1) for _ in range(2))
    hyper = type("H", (LT.Hyper,), dict(grad_norm_clipping=float(g["clip"])))
    return g, p, batch, state, hyper, A


@pytest.mark.parametrize("fname,net", LEARN_CASES)
def test_identity_popart_step_matches_reference(fname, net):
    g, p, batch, state, hyper, A = _golden_case(fname, net)
    o = PO.learner_step(p, batch, state, hyper=hyper, net=net, num_actions=A, beta=0.0)
    for k in ("total_loss", "pg_loss", "baseline_loss", "entropy_loss"):
        np.testing.assert_allclose(float(o[k]), float(g[k]), rtol=2e-5, atol=2e-5, err_msg=k)
    coef = min(1.0, float(g["clip"]) / (float(o["grad_norm"]) + 1e-6))
    np.testing.assert_allclose(float(o["grad_norm"]) * coef, float(g["clipped_grad_norm"]), rtol=1e-4)
    for n, gr in o["grads"].items():
        head = (gr * coef).flatten()[:16].numpy()
        scale = max(float(g["grad_stats/" + n][2]), 1e-6)
        np.testing.assert_allclose(head, g["grad_head/" + n], rtol=2e-3, atol=2e-4 * scale, err_msg=n)
        np.testing.assert_allclose(o["params"][n].flatten()[:16].numpy(), g["param_head/" + n], rtol=1e-4, atol=1e-5,
                                   err_msg=n)
    assert float(o["mu"][0]) == 0.0 and float(o["nu"][0]) == 1.0
    # and it is exactly the plain oracle step, not just close to it
    ref = LT.learner_step(p, batch, state, hyper=hyper, net=net, num_actions=A)
    assert torch.equal(o["total_loss"], ref["total_loss"])
    for n in ref["params"]:
        assert torch.equal(o["params"][n], ref["params"][n]), n


def _random_stats(rs, K):
    mu = torch.from_numpy(rs.randn(K) * 10.0)
    sig = torch.from_numpy(10.0 ** rs.uniform(-2, 3, size=K))
    return mu, sig * sig + mu * mu


def test_update_preserves_unnormalised_outputs():
    rs = np.random.RandomState(0)
    K, F, N = 5, 37, 64
    mu, nu = _random_stats(rs, K)
    W = torch.from_numpy(rs.randn(K, F))
    b = torch.from_numpy(rs.randn(K))
    x = torch.from_numpy(rs.randn(N, F))
    sums = torch.from_numpy(np.stack([rs.randint(1, 50, K).astype(np.float64), rs.randn(K) * 100, rs.rand(K) * 1e4]))
    sums[2] = torch.maximum(sums[2], sums[1] ** 2 / sums[0])  # a realisable second moment
    mu2, nu2, W2, b2 = PO.popart_update(sums, 0.3, mu, nu, W, b)
    before = PO.sigma(mu, nu) * (x @ W.t() + b) + mu
    after = PO.sigma(mu2, nu2) * (x @ W2.t() + b2) + mu2
    np.testing.assert_allclose(after.numpy(), before.numpy(), rtol=1e-12, atol=1e-12 * float(before.abs().max()))


def test_statistics_update_matches_numpy():
    rs = np.random.RandomState(1)
    T, B, K, beta = 9, 6, 4, 0.25
    vs = rs.randn(T, B) * 5.0
    task = rs.randint(0, K, size=(T, B))
    task[task == 2] = 1            # task 2 is absent from the batch
    task[:, 0] = -1                # out-of-range ids count nowhere
    task[3, 1] = K
    mu, nu = _random_stats(rs, K)
    sums = PO.task_sums(torch.from_numpy(vs), torch.from_numpy(task), K)
    mu2, nu2, W2, b2 = PO.popart_update(sums, beta, mu, nu, torch.ones(K, 3, dtype=torch.float64),
                                        torch.zeros(K, dtype=torch.float64))
    for k in range(K):
        x = vs[task == k]
        if k == 2:
            assert x.size == 0
            assert float(mu2[k]) == float(mu[k]) and float(nu2[k]) == float(nu[k])
            assert torch.equal(W2[k], torch.ones(3, dtype=torch.float64)) and float(b2[k]) == 0.0
            continue
        np.testing.assert_allclose(float(mu2[k]), (1 - beta) * float(mu[k]) + beta * x.mean(), rtol=1e-12)
        np.testing.assert_allclose(float(nu2[k]), (1 - beta) * float(nu[k]) + beta * (x * x).mean(), rtol=1e-12)
    assert float(sums[0].sum()) == float(((task >= 0) & (task < K)).sum())


def test_out_of_range_rows_add_nothing():
    rs = np.random.RandomState(2)
    T, B, A, K = 6, 3, 5, 2
    v = LT.synthetic_batch(T, B, A, seed=4)
    n = torch.from_numpy(rs.randn(T + 1, B, K)).requires_grad_(True)
    tl = torch.from_numpy(rs.randn(T, B, A)).requires_grad_(True)
    task = torch.from_numpy(rs.randint(0, K, size=(T + 1, B)))
    task[:, 1] = -1
    mu, nu = _random_stats(rs, K)
    o = PO.popart_losses(v["policy_logits"][1:], tl, v["action"][1:], v["reward"][1:], v["done"][1:], n, task, mu, nu)
    gt, gn = torch.autograd.grad(o["total_loss"], [tl, n])
    assert torch.count_nonzero(gt[:, 1]) == 0 and torch.count_nonzero(gn[:, 1]) == 0
    keep = [0, 2]
    o2 = PO.popart_losses(v["policy_logits"][1:, keep], tl[:, keep], v["action"][1:, keep], v["reward"][1:, keep],
                          v["done"][1:, keep], n[:, keep], task[:, keep], mu, nu)
    for k in ("pg_loss", "baseline_loss", "entropy_loss"):
        np.testing.assert_allclose(float(o[k]), float(o2[k]), rtol=1e-12)


@pytest.mark.parametrize("net", ["atari", "resnet"])
def test_nets_popart_state(net):
    from torchbeast_b200 import _lib, nets
    make = (lambda **kw: nets.AtariNet((4, 84, 84), 6, True, device="cpu", **kw)) if net == "atari" else \
        (lambda **kw: nets.ResNet(6, True, device="cpu", **kw))
    plain, m = make(), make(num_tasks=1)
    sd = m.state_dict()
    assert list(sd) == list(plain.state_dict()) + ["popart.mu", "popart.nu"]
    assert sd["popart.mu"].dtype == torch.float64 and tuple(sd["popart.mu"].shape) == (1,)
    assert torch.equal(sd["popart.nu"], torch.ones(1, dtype=torch.float64))
    assert tuple(sd["baseline.weight"].shape) == tuple(plain.state_dict()["baseline.weight"].shape)
    assert m.flat_params.numel() == plain.flat_params.numel()
    sd = {k: v.clone() for k, v in sd.items()}
    sd["popart.mu"].fill_(3.0)
    sd["popart.nu"].fill_(25.0)
    m2 = make(num_tasks=1)
    m2.load_state_dict(sd)
    assert float(m2.popart.mu) == 3.0 and float(m2.popart.sigma()) == 4.0
    np.testing.assert_allclose(m2.popart.unnormalize(torch.ones(2, 3, 1)).numpy(), np.full((2, 3), 7.0))
    assert getattr(plain, "popart", None) is None
    m4 = make(num_tasks=4)
    sd4 = m4.state_dict()
    F = plain.state_dict()["baseline.weight"].shape[1]
    assert tuple(sd4["baseline.weight"].shape) == (4, F) and tuple(sd4["baseline.bias"].shape) == (4,)
    assert tuple(sd4["popart.mu"].shape) == (4,)
    assert m4.flat_params.numel() == plain.flat_params.numel() + 3 * (F + 1)
    assert [k for k in sd4 if k != "baseline.weight"] == [k for k in sd if k != "baseline.weight"]
    b = torch.tensor([[[1.0, 2.0, 3.0, 4.0]]])
    m4.popart.mu.copy_(torch.tensor([0.0, 10.0, 20.0, 30.0], dtype=torch.float64))
    m4.popart.nu.copy_(m4.popart.mu ** 2 + 1.0)  # sigma = 1
    np.testing.assert_allclose(m4.popart.unnormalize(b, torch.tensor([[2]])).numpy(), [[23.0]])
    for bad in (0, 65):
        with pytest.raises(_lib.TorchBeastB200Error, match="num_tasks must be in"):
            make(num_tasks=bad)


def test_popart_num_values_abi_and_host_side_checks():
    from tests.test_abi_cpu import header_symbols
    from torchbeast_b200 import _lib
    for s in ("tb_impala_loss_f32", "tb_popart_update", "tb_atarinet_param_count", "tb_atarinet_forward",
              "tb_atarinet_backward", "tb_resnet_param_count", "tb_resnet_forward", "tb_resnet_backward"):
        assert s in header_symbols() and s in _lib.declared_symbols()
    h = _lib.lib()
    assert h.tb_popart_update(None, None, None, None, 65, None, None, 8, None) != 0
    assert b"bad sizes" in h.tb_last_error()
    P = ctypes.c_void_p(256)  # never dereferenced: every call below fails its host-side checks before a launch

    def popart_error(T=4, K=3, mu=P, nu=P, task_sums=P, zero_tail=1):
        args = ([None] * 6 + [P, None] + [T, 2, 6, 0.99, 0.5, 0.0006, 1, 1.0, 1.0, None, None, P, mu, nu, K, task_sums]
                + [None] * 11 + [zero_tail, None, None])
        assert h.tb_impala_loss_f32(*args) != 0
        return h.tb_last_error()

    assert b"num_tasks" in popart_error(K=0)
    assert b"num_tasks" in popart_error(K=65)
    for k in ("mu", "nu", "task_sums"):
        assert b"null PopArt pointer" in popart_error(**{k: None})
    assert b"bad sizes" in popart_error(T=0)
    assert b"zero_tail" in popart_error(zero_tail=0)
    # num_values = 1 is the plain layout (the parameter counts of the reference's nets), each further value adds one
    # head row
    assert h.tb_atarinet_param_count(6, 1, 1) == sum(int(np.prod(s)) for s in LT.atarinet_param_shapes(6, True).values())
    assert h.tb_resnet_param_count(4, 84, 84, 16, 32, 32, 6, 1, 1) == sum(int(np.prod(s)) for s in
                                                                        LT.resnet_param_shapes(6, True).values())
    assert h.tb_atarinet_param_count(6, 57, 1) - h.tb_atarinet_param_count(6, 1, 1) == 56 * (512 + 6 + 1 + 1)
    assert h.tb_resnet_param_count(4, 84, 84, 16, 32, 32, 6, 57, 1) - h.tb_resnet_param_count(4, 84, 84, 16, 32, 32, 6, 1, 1) \
        == 56 * (256 + 1)
