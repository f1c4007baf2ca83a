"""UPGO of tb_upgo_loss_f32 (include/torchbeast_b200.h) restated in float64: the trace switch, the return by its
literal recursion, the advantage, and the loss with its gradient by autograd.  `return_general` is an independent
closed form of the same return, a generalized lambda-return, to check the recursion against."""
import numpy as np
import torch


def trace_switch(rewards, discounts, values, bootstrap):
    """lambda [T, B]: lambda_t = (r_t + g_t V_{t+1} >= V_t) for t >= 1; row 0 is not used (set to 0)."""
    r, g, v = (np.asarray(x, np.float64) for x in (rewards, discounts, values))
    v_next = np.concatenate([v[1:], np.asarray(bootstrap, np.float64)[None]], 0)
    lam = (r + g * v_next >= v).astype(np.float64)
    lam[0] = 0.0
    return lam


def returns(rewards, discounts, values, bootstrap):
    """G [T, B] by the recursion: G_{T-1} = r + g V_T, G_t = r_t + g_t (lam_{t+1} G_{t+1} + (1 - lam_{t+1}) V_{t+1})."""
    r, g, v, bs = (np.asarray(x, np.float64) for x in (rewards, discounts, values, bootstrap))
    lam = trace_switch(r, g, v, bs)
    T = r.shape[0]
    G = np.empty_like(r)
    G[T - 1] = r[T - 1] + g[T - 1] * bs
    for t in range(T - 2, -1, -1):
        G[t] = r[t] + g[t] * (lam[t + 1] * G[t + 1] + (1 - lam[t + 1]) * v[t + 1])
    return G


def return_general(rewards, discounts, values, bootstrap):
    """G_t = sum_{k >= t} (prod_{j=t}^{k-1} g_j lam_{j+1}) (r_k + g_k (1 - lam_{k+1}) V_{k+1}), with lam_T = 0 and
    V_T the bootstrap: the lambda-return with a per-step lambda, summed term by term instead of recursively."""
    r, g, v, bs = (np.asarray(x, np.float64) for x in (rewards, discounts, values, bootstrap))
    T = r.shape[0]
    lam = np.concatenate([trace_switch(r, g, v, bs), np.zeros((1,) + r.shape[1:])], 0)   # lam[T] = 0
    v_ext = np.concatenate([v, bs[None]], 0)
    G = np.zeros_like(r)
    for t in range(T):
        coef = np.ones(r.shape[1:])
        for k in range(t, T):
            G[t] += coef * (r[k] + g[k] * (1 - lam[k + 1]) * v_ext[k + 1])
            coef = coef * g[k] * lam[k + 1]
    return G


def loss(target_logits, actions, rewards, discounts, values, bootstrap, log_rhos, upgo_cost, clip_pg_rho=1.0,
         mask=None, weights=None, sigma=None, valid=None):
    """The UPGO advantage, loss and gradient in float64.  `rewards` are clipped and `discounts` built by the caller, as
    the kernel builds them; `values` / `bootstrap` are unnormalised.  mask [T, B]: the trust mask (None: all trusted).
    weights [B]: column weights.  sigma [T, B]: PopArt sigma of each row's task (None: 1); valid [T, B]: rows whose task
    is in range (None: all).  Returns dict(G, adv, loss, grad_logits [T, B, A])."""
    f = lambda x: np.asarray(x, np.float64)  # noqa: E731
    v = f(values)
    G = returns(rewards, discounts, v, bootstrap)
    rho = np.exp(f(log_rhos))
    if mask is not None:
        rho = np.where(mask, rho, 0.0)
    rho_bar = rho if clip_pg_rho is None else np.minimum(rho, clip_pg_rho)
    adv = rho_bar * (G - v)
    if sigma is not None:
        adv = adv / f(sigma)
    if valid is not None:
        adv = np.where(valid, adv, 0.0)
    B = v.shape[1]
    w = torch.ones(B, dtype=torch.float64) if weights is None else torch.from_numpy(f(weights))
    tl = torch.tensor(f(target_logits), requires_grad=True)
    lpa = torch.log_softmax(tl, -1).gather(-1, torch.from_numpy(np.asarray(actions, np.int64))[..., None])[..., 0]
    total = upgo_cost * (-lpa * torch.from_numpy(adv) * w).sum()
    total.backward()
    return dict(G=G, adv=adv, loss=total.item(), grad_logits=tl.grad.numpy())
