"""The trust region of tb_impala_loss_f32 (include/torchbeast_b200.h) restated in float64 NumPy: the KL of every
row, the mask, V-trace with rho_t * m_t in place of rho_t, the three losses and their closed-form gradients."""
import numpy as np


def log_softmax(x):
    m = x.max(-1, keepdims=True)
    return (x - m) - np.log(np.exp(x - m).sum(-1, keepdims=True))


def policy_kl(behavior_logits, target_logits):
    """KL(pi || mu) of every row: pi = softmax(target), mu = softmax(behaviour)."""
    lt = log_softmax(np.asarray(target_logits, np.float64))
    lb = log_softmax(np.asarray(behavior_logits, np.float64))
    return (np.exp(lt) * (lt - lb)).sum(-1)


def loss(behavior_logits, target_logits, actions, rewards, discounts, values, bootstrap, beta=None, mask=None,
         baseline_cost=0.5, entropy_cost=0.0006, clip_rho=1.0, clip_pg_rho=1.0, weights=None):
    """Everything the trust-region loss computes, in float64.  `discounts` are used as given (apply the reward clip and
    the done -> discount rule before).  The mask is kl <= beta, or `mask` when given (a test passes the kernel's own,
    so that rows within rounding of beta cannot flip); beta None and no mask trusts every row.  `weights` [B]: the
    column weights of the weighted loss.  Returns a dict."""
    f = lambda x: np.asarray(x, np.float64)  # noqa: E731
    bl, tl = f(behavior_logits), f(target_logits)
    r, g, v, bs = f(rewards), f(discounts), f(values), f(bootstrap)
    T, B, A = tl.shape
    kl = policy_kl(bl, tl)
    if mask is None:
        mask = np.ones((T, B), bool) if beta is None else kl <= beta
    lt, lb = log_softmax(tl), log_softmax(bl)
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
    vs_minus_v = np.zeros((T, B))
    for t in range(T - 1, -1, -1):
        acc = deltas[t] + g[t] * cs[t] * acc
        vs_minus_v[t] = acc
    vs = vs_minus_v + v
    vs_next = np.concatenate([vs[1:], bs[None]], 0)
    pg_adv = rho_pg * (r + g * vs_next - v)
    w = np.ones(B) if weights is None else f(weights)
    pi = np.exp(lt)
    ent_row = (pi * lt).sum(-1)
    pg = (-tlp * pg_adv * w).sum()
    base = baseline_cost * (0.5 * (vs - v) ** 2 * w).sum()
    ent = entropy_cost * (ent_row * w).sum()
    onehot = np.eye(A)[actions]
    grad_logits = (pg_adv[..., None] * (pi - onehot) + entropy_cost * pi * (lt - ent_row[..., None])) * w[None, :, None]
    grad_values = -baseline_cost * (vs - v) * w[None, :]
    return dict(kl=kl, mask=mask, log_rhos=log_rhos, behavior_alp=blp, target_alp=tlp, vs=vs, pg_adv=pg_adv,
                losses=np.array([pg, base, ent, pg + base + ent]), grad_logits=grad_logits, grad_values=grad_values,
                trusted=int(mask.sum()), kl_sum=kl.sum())
