"""Learning over legal actions restated in float64 NumPy, with no sentinel: each row's illegal entries are dropped and
the softmax, the entropy, the V-trace rho, the trust region's KL, UPGO and the kickstarting KL are taken over the legal
entries only.  A row with no legal entry keeps all of them (it is left unmasked).  Dropped entries get probability 0
and gradient 0; their log-probability slot holds 0 and is only ever multiplied by that probability 0."""
import numpy as np

from tests import upgo_oracle as UO


def keep(legal):
    """The entries each row keeps: legal, or every entry of a row with none."""
    legal = np.asarray(legal).astype(bool)
    return legal | ~legal.any(-1, keepdims=True)


def log_softmax(x, legal):
    """(lp, p): the log-softmax and the softmax of every row over its kept entries, computed on those entries alone."""
    x = np.asarray(x, np.float64)
    k = keep(legal)
    lp, p = np.zeros_like(x), np.zeros_like(x)
    for idx in np.ndindex(x.shape[:-1]):
        j = np.flatnonzero(k[idx])
        z = x[idx][j]
        m = z.max()
        lz = (z - m) - np.log(np.exp(z - m).sum())
        lp[idx + (j,)] = lz
        p[idx + (j,)] = np.exp(lz)
    return lp, p


def loss(behavior_logits, target_logits, actions, rewards, discounts, values, bootstrap, legal, beta=None, mask=None,
         baseline_cost=0.5, entropy_cost=0.0006, clip_rho=1.0, clip_pg_rho=1.0, weights=None):
    """The loss block (V-trace, pg / baseline / entropy losses and their gradients, the trust region's KL and mask) of
    every [T, B] row over its legal set legal [T, B, A].  `discounts` as given; the mask is kl <= beta, or `mask`
    (the kernel's own, so rows within rounding of beta cannot flip); `weights` [B]: column weights.  Returns a dict."""
    f = lambda x: np.asarray(x, np.float64)  # noqa: E731
    r, g, v, bs = f(rewards), f(discounts), f(values), f(bootstrap)
    actions = np.asarray(actions, np.int64)
    T, B, A = np.shape(target_logits)
    lt, pi = log_softmax(target_logits, legal)
    lb, _ = log_softmax(behavior_logits, legal)
    kl = (pi * (lt - lb)).sum(-1)
    if mask is None:
        mask = np.ones((T, B), bool) if beta is None else kl <= beta
    tlp = np.take_along_axis(lt, actions[..., None], -1)[..., 0]
    blp = np.take_along_axis(lb, actions[..., None], -1)[..., 0]
    log_rhos = tlp - blp
    rho = np.where(mask, np.exp(log_rhos), 0.0)
    rho_bar = rho if clip_rho is None else np.minimum(rho, clip_rho)
    cs = np.minimum(rho, 1.0)
    rho_pg = rho if clip_pg_rho is None else np.minimum(rho, clip_pg_rho)
    v_next = np.concatenate([v[1:], bs[None]], 0)
    deltas = rho_bar * (r + g * v_next - v)
    acc = np.zeros(B)
    vs = np.zeros((T, B))
    for t in range(T - 1, -1, -1):
        acc = deltas[t] + g[t] * cs[t] * acc
        vs[t] = acc
    vs = vs + v
    vs_next = np.concatenate([vs[1:], bs[None]], 0)
    pg_adv = rho_pg * (r + g * vs_next - v)
    w = np.ones(B) if weights is None else f(weights)
    ent_row = (pi * lt).sum(-1)
    pg = (-tlp * pg_adv * w).sum()
    base = baseline_cost * (0.5 * (vs - v) ** 2 * w).sum()
    ent = entropy_cost * (ent_row * w).sum()
    onehot = np.eye(A)[actions]
    grad_logits = (pg_adv[..., None] * (pi - onehot) + entropy_cost * pi * (lt - ent_row[..., None])) * w[None, :, None]
    return dict(kl=kl, mask=mask, log_rhos=log_rhos, vs=vs, pg_adv=pg_adv, losses=np.array([pg, base, ent, pg + base + ent]),
                grad_logits=grad_logits, kl_sum=kl.sum(), trusted=int(mask.sum()))


def upgo(target_logits, actions, rewards, discounts, values, bootstrap, log_rhos, legal, cost, clip_pg_rho=1.0,
         mask=None, weights=None):
    """UPGO (tests/upgo_oracle.py's return) with log pi(a) and pi over the legal set: dict(adv, loss, grad_logits)."""
    v = np.asarray(values, np.float64)
    G = UO.returns(rewards, discounts, v, bootstrap)
    rho = np.exp(np.asarray(log_rhos, np.float64))
    if mask is not None:
        rho = np.where(mask, rho, 0.0)
    rho_bar = rho if clip_pg_rho is None else np.minimum(rho, clip_pg_rho)
    adv = rho_bar * (G - v)
    lt, pi = log_softmax(target_logits, legal)
    actions = np.asarray(actions, np.int64)
    lpa = np.take_along_axis(lt, actions[..., None], -1)[..., 0]
    w = np.ones(v.shape[1]) if weights is None else np.asarray(weights, np.float64)
    onehot = np.eye(lt.shape[-1])[actions]
    return dict(adv=adv, loss=cost * (-lpa * adv * w).sum(),
                grad_logits=cost * (adv * w)[..., None] * (pi - onehot))


def kickstart(teacher_logits, target_logits, legal, cost, weights=None):
    """KL(p_teacher || p_learner) of every row over the legal set: dict(kl, kl_sum, loss, grad_logits)."""
    lt, pt = log_softmax(teacher_logits, legal)
    ls, ps = log_softmax(target_logits, legal)
    kl = (pt * (lt - ls)).sum(-1)
    w = np.ones(kl.shape[1]) if weights is None else np.asarray(weights, np.float64)
    return dict(kl=kl, kl_sum=kl.sum(), loss=cost * (w[None, :] * kl).sum(),
                grad_logits=cost * w[None, :, None] * (ps - pt))


def mask_logits(x, legal, actions=None, fill=np.float32(np.finfo(np.float32).min)):
    """tb_mask_logits_f32 restated in NumPy (float32, bit for bit): out = legal ? x : fill on a row with a legal entry,
    the row as it is otherwise, NaN on a row whose in-range action is illegal."""
    x = np.asarray(x, np.float32)
    legal = np.asarray(legal).astype(bool)
    any_legal = legal.any(-1, keepdims=True)
    out = np.where(legal | ~any_legal, x, np.float32(fill)).astype(np.float32)
    if actions is not None:
        A = x.shape[-1]
        a = np.asarray(actions, np.int64)
        inr = (a >= 0) & (a < A)
        picked = np.take_along_axis(legal, np.clip(a, 0, A - 1)[..., None], -1)[..., 0]
        bad = inr & ~picked & any_legal[..., 0]
        out[bad] = np.nan
    return out
