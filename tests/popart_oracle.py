"""PopArt restated in plain torch (float32 / float64): the normalised IMPALA loss, the per-task statistics, the
output-preserving head update and one whole learn() step with them (include/torchbeast_b200.h, "PopArt value
normalisation").  Test infrastructure only; with one task, identity statistics and beta = 0 it reduces to
oracle/learner_torch.learner_step, which tests/test_popart_cpu.py pins against the golden fixtures."""
import torch
import torch.nn.functional as F

from oracle import learner_torch as LT


def sigma(mu, nu):
    return (nu - mu * mu).clamp_min(0).sqrt().clamp(1e-4, 1e6)


def popart_losses(blogits, tlogits, actions, rewards, done, n, task, mu, nu, hyper=LT.Hyper):
    """Steps 1-4 on shifted inputs (blogits / actions / rewards / done = batch[1:], tlogits = learner logits[:-1]) with
    the normalised head n [T+1, B, K] and task [T+1, B].  Differentiable in tlogits and n.  Returns
    dict(pg_loss, baseline_loss, entropy_loss, total_loss, vs, pg_advantages, task_sums [3, K])."""
    dtype = n.dtype
    K = n.shape[-1]
    valid = (task >= 0) & (task < K)
    tk = task.clamp(0, K - 1)
    mu, nu = mu.to(dtype), nu.to(dtype)
    sig, m = sigma(mu, nu)[tk], mu[tk]
    nk = n.gather(-1, tk.unsqueeze(-1)).squeeze(-1)
    v = torch.where(valid, sig * nk + m, torch.zeros_like(nk))
    rewards = rewards.to(dtype)
    if hyper.reward_clipping == "abs_one":
        rewards = rewards.clamp(-1, 1)
    discounts = LT._notdone(done, dtype) * hyper.discounting
    vs, pg_adv, _, _, _ = LT.vtrace_from_logits_torch(blogits.to(dtype), tlogits.detach(), actions, discounts, rewards,
                                                      v[:-1].detach(), v[-1].detach())
    w = valid[:-1].to(dtype)
    lsm = torch.log_softmax(tlogits, -1)
    nll = -lsm.gather(-1, actions.unsqueeze(-1)).squeeze(-1)
    pg = torch.sum(w * nll * (pg_adv / sig[:-1]))
    bl = hyper.baseline_cost * 0.5 * torch.sum(w * ((vs - m[:-1]) / sig[:-1] - nk[:-1]) ** 2)
    en = hyper.entropy_cost * torch.sum(w * torch.sum(lsm.exp() * lsm, -1))
    return dict(pg_loss=pg, baseline_loss=bl, entropy_loss=en, total_loss=pg + bl + en, vs=vs, pg_advantages=pg_adv,
                task_sums=task_sums(vs, task[:-1], K))


def task_sums(vs, task, K):
    """[3, K]: count, sum vs, sum vs^2 of each task (ids outside [0, K) count nowhere), in float64."""
    vs, out = vs.double().flatten(), torch.zeros(3, K, dtype=torch.float64)
    task = task.flatten()
    for k in range(K):
        x = vs[task == k]
        out[0, k], out[1, k], out[2, k] = x.numel(), x.sum(), (x * x).sum()
    return out


def popart_update(sums, beta, mu, nu, weight, bias):
    """Steps 6-7 in float64: returns (mu', nu', weight', bias') for weight [K, F], bias [K]."""
    mu, nu, weight, bias = mu.double(), nu.double(), weight.double(), bias.double()
    count = sums[0]
    has = count > 0
    c = count.clamp_min(1)
    mu2 = torch.where(has, (1 - beta) * mu + beta * sums[1] / c, mu)
    nu2 = torch.where(has, (1 - beta) * nu + beta * sums[2] / c, nu)
    s, s2 = sigma(mu, nu), sigma(mu2, nu2)
    weight2 = torch.where(has[:, None], weight * (s / s2)[:, None], weight)
    bias2 = torch.where(has, (s * bias + mu - mu2) / s2, bias)
    return mu2, nu2, weight2, bias2


def learner_step(p, batch, core_state=(), hyper=LT.Hyper, net="atari", num_actions=6, mu=None, nu=None, beta=0.0,
                 task=None):
    """oracle/learner_torch.learner_step with PopArt: `p` has the reference's parameter shapes except baseline.weight
    [K, F] / baseline.bias [K]; task [T+1, B] (default zeros).  Returns that function's dict (baseline [T+1, B, K]) plus
    mu / nu after the update; params are after the optimizer step AND the head rescale."""
    params = {k: v.detach().clone().requires_grad_(True) for k, v in p.items()}
    dtype = params["fc.weight"].dtype
    K = params["baseline.weight"].shape[0]
    outs = []
    for k in range(K):  # the reference forwards have one value output: value k is the forward with head row k
        pk = dict(params, **{"baseline.weight": params["baseline.weight"][k:k + 1],
                             "baseline.bias": params["baseline.bias"][k:k + 1]})
        if net == "atari":
            outs.append(LT.atarinet_forward(pk, batch["frame"], batch["reward"], batch["done"], batch["last_action"],
                                            core_state, num_actions))
        else:
            outs.append(LT.resnet_forward(pk, batch["frame"], batch["reward"], batch["done"], core_state, num_actions))
    logits = outs[0][0]
    baseline = torch.stack([o[1] for o in outs], -1)
    mu = torch.zeros(K, dtype=torch.float64) if mu is None else mu
    nu = torch.ones(K, dtype=torch.float64) if nu is None else nu
    task = torch.zeros(baseline.shape[:2], dtype=torch.int64) if task is None else task
    o = popart_losses(batch["policy_logits"][1:], logits[:-1], batch["action"][1:], batch["reward"][1:],
                      batch["done"][1:], baseline, task, mu, nu, hyper)
    names = list(params)
    grads = torch.autograd.grad(o["total_loss"], [params[n] for n in names], allow_unused=True)
    grads = {n: (g if g is not None else torch.zeros_like(params[n])) for n, g in zip(names, grads)}
    gnorm = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).to(dtype)
    coef = torch.clamp(hyper.grad_norm_clipping / (gnorm + 1e-6), max=1.0)
    new_p = {}
    for n in names:
        g = grads[n] * coef
        sq = (1 - hyper.alpha) * g * g
        new_p[n] = p[n].detach() - hyper.learning_rate * g / (sq.sqrt() + hyper.epsilon)
    mu2, nu2, w2, b2 = popart_update(o["task_sums"], beta, mu, nu, new_p["baseline.weight"], new_p["baseline.bias"])
    new_p["baseline.weight"], new_p["baseline.bias"] = w2.to(dtype), b2.to(dtype)
    return dict(pg_loss=o["pg_loss"].detach(), baseline_loss=o["baseline_loss"].detach(),
                entropy_loss=o["entropy_loss"].detach(), total_loss=o["total_loss"].detach(),
                policy_logits=logits.detach(), baseline=baseline.detach(), vs=o["vs"], pg_advantages=o["pg_advantages"],
                grads=grads, grad_norm=gnorm, params=new_p, mu=mu2, nu=nu2)
