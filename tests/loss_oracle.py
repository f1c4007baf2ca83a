"""The V-trace scan, action_log_probs, the plain fused IMPALA loss and the three stand-alone losses of csrc/vtrace.cu
restated in float64 NumPy, in the kernels' operation order.

Besides the values, every function returns per-element magnitudes for an error bound on the kernel: a running-error
analysis, to first order.  The inputs are exact; every float operation rounds its result by at most u |result|
(u = 2^-24 for float32, 2^-53 for float64), and the CUDA library's exp and log are within EXP_ULP and LOG_ULP ulps, an
ulp being at most 2 u |result|.  A quantity q then differs from the exact value by at most u mag(q), with mag built by
  a + b:  mag(a) + mag(b) + |a + b|          a * b:  |a| mag(b) + |b| mag(a) + |a b|
  exp(y): exp(y) (mag(y) + 2 EXP_ULP)        log(s): mag(s) / s + 2 LOG_ULP |log s|
  min(a, c), max(a, c) with c exact: mag(a) (both are 1-Lipschitz)
and a fused multiply-add is charged as the two operations it replaces.  A kernel and this restatement each lie within
u mag of the exact value, so they differ by at most BOUND_C u mag with BOUND_C = 2: for a float64 kernel both halves
count, for a float32 kernel the restatement's own error is 2^-29 of the bound and the second half is slack for the
second-order terms the analysis drops (below n u = 1e-4 of the bound at the longest unroll tested).  Nothing in the
constant is fitted to measured errors.

The scan: within a chunk the recurrence acc_t = delta_t + (g_t c_t) acc_{t+1} rounds each step's product and sum, and
the affine map that carries a chunk (bb = delta + dc bb, a = dc a) rounds three values per step; where chunks meet,
the carry-in is composed from the later chunks' maps, at most twice per edge per level (warps in a CTA, CTAs of a
cluster, the cluster's per-CTA maps): six more roundings.  Every rounding is of a value no larger than the same
recurrence run on absolute values, |delta_t| + (g_t c_t) |.|_{t+1}, so every step is charged SCAN_ROUNDINGS = 9 times
that.  The loss sums are fp64 in the kernels: n terms add at most n u64 sum|term|, and their float32 rounding once."""
import numpy as np

U32, U64 = 2.0 ** -24, 2.0 ** -53
BOUND_C = 2.0
EXP_ULP, LOG_ULP = 2, 1     # expf / exp: 2 / 1 ulp, logf / log: 1 ulp (CUDA C Programming Guide, Mathematical Functions)
SCAN_ROUNDINGS = 9
MASKED_LOGIT = float(np.finfo(np.float32).min)   # TB_MASKED_LOGIT

MISTAKES = ("cbar_clip_rho", "pg_clip_rho", "pg_bootstrap_values", "entropy_uncentred", "baseline_half", "fp32_sums")


def bound(mag, u):
    return BOUND_C * u * np.asarray(mag, np.float64)


def _f(x):
    return np.asarray(x, np.float64)


def _has_clip(c):
    """None, NaN and negative thresholds mean no clipping (the kernels test c >= 0)"""
    return c is not None and c >= 0


def _exp_mag(e, mag_y):
    return e * mag_y + 2 * EXP_ULP * e


def log_softmax_rows(x):
    """The max, log-sum-exp and log-probabilities of every row of x [..., A], as RowOps / alp_dyn form them: m = the
    running max, s = exp(x_0 - m) + exp(x_1 - m) + ... summed from j = 0, logs = log(s), lp_j = (x_j - m) - logs."""
    x = _f(x)
    m = x.max(-1, keepdims=True)
    y = x - m
    with np.errstate(over="ignore", invalid="ignore"):
        e = np.exp(y)
    mag_e = np.where(e > 0, _exp_mag(e, np.abs(y)), 0.0)
    part = np.cumsum(e, -1)
    s = part[..., -1:]
    mag_s = mag_e.sum(-1, keepdims=True) + part[..., 1:].sum(-1, keepdims=True)
    logs = np.log(s)
    mag_logs = mag_s / s + 2 * LOG_ULP * np.abs(logs)
    lp = y - logs
    return dict(m=m, y=y, logs=logs, mag_logs=mag_logs, lp=lp, mag_lp=np.abs(y) + mag_logs + np.abs(lp))


def action_log_probs(logits, actions):
    """(log pi(a) [...], mag [...]) for logits [..., A] and actions [...]"""
    r = log_softmax_rows(logits)
    a = np.asarray(actions, np.int64)[..., None]
    return np.take_along_axis(r["lp"], a, -1)[..., 0], np.take_along_axis(r["mag_lp"], a, -1)[..., 0]


def scan(log_rhos, discounts, rewards, values, bootstrap, clip_rho=1.0, clip_pg_rho=1.0, mag_log_rhos=None,
         mistake=None):
    """vs, pg_adv [T, B] of from_importance_weights and their magnitudes.  mag_log_rhos: the magnitude of log_rhos when
    they are computed (the fused loss), else they are exact inputs.  `mistake` (see MISTAKES) changes one operation."""
    lr, g, r, v, bs = map(_f, (log_rhos, discounts, rewards, values, bootstrap))
    T, B = v.shape
    rho = np.exp(lr)
    mag_rho = _exp_mag(rho, 0.0 if mag_log_rhos is None else _f(mag_log_rhos))
    c = np.minimum(rho, clip_rho if (mistake == "cbar_clip_rho" and _has_clip(clip_rho)) else 1.0)
    rb = np.minimum(rho, clip_rho) if _has_clip(clip_rho) else rho
    pg_clip = clip_rho if mistake == "pg_clip_rho" else clip_pg_rho
    rp = np.minimum(rho, pg_clip) if _has_clip(pg_clip) else rho
    vs, mag_vs = np.empty((T, B)), np.empty((T, B))
    acc, mag_acc, aabs = np.zeros(B), np.zeros(B), np.zeros(B)
    for t in range(T - 1, -1, -1):
        vn = v[t + 1] if t + 1 < T else bs
        gv = g[t] * vn
        td = (r[t] + gv) - v[t]
        mag_td = np.abs(gv) + np.abs(r[t] + gv) + np.abs(td)
        delta = rb[t] * td
        mag_delta = rb[t] * mag_td + np.abs(td) * mag_rho[t] + np.abs(delta)
        dc = g[t] * c[t]
        mag_dc = g[t] * mag_rho[t] + dc
        aabs_next = aabs
        acc = delta + dc * acc
        aabs = np.abs(delta) + dc * aabs_next
        mag_acc = mag_delta + dc * mag_acc + aabs_next * mag_dc + SCAN_ROUNDINGS * aabs
        vs[t] = acc + v[t]
        mag_vs[t] = mag_acc + np.abs(vs[t])
    vs_next = np.concatenate([vs[1:], bs[None]], 0)
    mag_vsn = np.concatenate([mag_vs[1:], np.zeros((1, B))], 0)
    if mistake == "pg_bootstrap_values":
        vs_next = np.concatenate([v[1:], bs[None]], 0)
    gv = g * vs_next
    inner = (r + gv) - v
    mag_inner = g * mag_vsn + np.abs(gv) + np.abs(r + gv) + np.abs(inner)
    pg = rp * inner
    mag_pg = rp * mag_inner + np.abs(inner) * mag_rho + np.abs(pg)
    return dict(vs=vs, pg_adv=pg, mag_vs=mag_vs, mag_pg=mag_pg)


def _sum(terms, mag_terms, u, fp32=False):
    """sum over every term in row order, in fp64 as the kernels' grid sums (any order: the bound holds for all), or,
    with fp32, sequentially in float32; and the magnitude of the fp64 sum's result"""
    terms = np.ravel(terms)
    if fp32:
        s = float(np.cumsum(terms.astype(np.float32), dtype=np.float32)[-1]) if terms.size else 0.0
    else:
        s = float(terms.sum())
    return s, float(np.sum(mag_terms)) + terms.size * (U64 / u) * float(np.abs(terms).sum())


def _entropy_rows(ls):
    """sum_j p_j lp_j of every row and its magnitude, with p_j = exp(lp_j) and the row summed from j = 0"""
    pr = np.exp(ls["lp"])
    mag_pr = _exp_mag(pr, ls["mag_lp"])
    term = pr * ls["lp"]
    ent = term.sum(-1)
    mag_term = pr * ls["mag_lp"] + np.abs(ls["lp"]) * mag_pr + np.abs(term)
    mag_ent = mag_term.sum(-1) + np.cumsum(np.abs(term), -1)[..., 1:].sum(-1)
    return pr, mag_pr, ent, mag_ent


def impala_loss(behavior_logits, target_logits, actions, rewards, values, bootstrap, done=None, discounts=None,
                discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, clip_rewards=True, clip_rho=1.0,
                clip_pg_rho=1.0, mistake=None):
    """Every output of tb_impala_loss_f32 without its feature groups, with magnitudes (mag_<name>).  The scalars are
    taken as the float32 values the kernel holds; the discount of a step is discounts[t, b] when given, else 0 where
    done and discounting elsewhere.  Returns a dict: vs, pg_adv, log_rhos, behavior_alp, target_alp [T, B],
    losses [4], grad_logits [T, B, A], grad_values [T, B]."""
    f32 = lambda x: float(np.float32(x))  # noqa: E731
    bc, ec = f32(baseline_cost), f32(entropy_cost)
    r = _f(rewards)
    if clip_rewards:
        r = np.clip(r, -1.0, 1.0)
    g = _f(discounts) if discounts is not None else np.where(np.asarray(done, bool), 0.0, f32(discounting))
    v = _f(values)
    a = np.asarray(actions, np.int64)
    tls, bls = log_softmax_rows(target_logits), log_softmax_rows(behavior_logits)
    pick = lambda x: np.take_along_axis(x, a[..., None], -1)[..., 0]  # noqa: E731
    tlp, mag_tlp, blp, mag_blp = pick(tls["lp"]), pick(tls["mag_lp"]), pick(bls["lp"]), pick(bls["mag_lp"])
    lr = tlp - blp
    mag_lr = mag_tlp + mag_blp + np.abs(lr)
    sc = scan(lr, g, r, v, bootstrap, f32(clip_rho) if clip_rho is not None else None,
              f32(clip_pg_rho) if clip_pg_rho is not None else None, mag_lr, mistake)
    vs, adv, mag_vs, mag_adv = sc["vs"], sc["pg_adv"], sc["mag_vs"], sc["mag_pg"]
    d = vs - v
    mag_d = mag_vs + np.abs(d)
    pr, mag_pr, ent, mag_ent = _entropy_rows(tls)
    onehot = np.eye(tls["lp"].shape[-1])[a]
    q = pr - onehot
    t1 = adv[..., None] * q
    mag_t1 = np.abs(adv)[..., None] * (mag_pr + np.abs(q)) + np.abs(q) * mag_adv[..., None] + np.abs(t1)
    lp, mag_lp = tls["lp"], tls["mag_lp"]
    h = lp if mistake == "entropy_uncentred" else lp - ent[..., None]
    mag_h = mag_lp + mag_ent[..., None] + np.abs(h)
    ep = ec * pr
    t2 = ep * h
    mag_t2 = ep * mag_h + np.abs(h) * (ec * mag_pr + ep) + np.abs(t2)
    gl = t1 + t2
    mag_gl = mag_t1 + mag_t2 + np.abs(gl)
    gv = -(0.5 * bc if mistake == "baseline_half" else bc) * d
    mag_gv = bc * mag_d + np.abs(gv)
    # the losses: -tlp * adv, d * d and ent_row in float, summed in fp64 (the mistake: in float32)
    fp32 = mistake == "fp32_sums"
    pg_terms = -tlp * adv
    s_pg, m_pg = _sum(pg_terms, np.abs(tlp) * mag_adv + np.abs(adv) * mag_tlp + np.abs(pg_terms), U32, fp32)
    s_bl, m_bl = _sum(0.5 * d * d, np.abs(d) * mag_d + 0.5 * d * d, U32, fp32)
    s_en, m_en = _sum(ent, mag_ent, U32, fp32)
    L = np.array([s_pg, bc * s_bl, ec * s_en, 0.0])
    L[3] = L[0] + L[1] + L[2]
    mag_L = np.array([m_pg, bc * m_bl, ec * m_en, 0.0])
    mag_L[3] = mag_L[:3].sum()
    mag_L += np.abs(L)
    return dict(vs=vs, pg_adv=adv, log_rhos=lr, behavior_alp=blp, target_alp=tlp, losses=L, grad_logits=gl,
                grad_values=gv, mag_vs=mag_vs, mag_pg_adv=mag_adv, mag_log_rhos=mag_lr, mag_behavior_alp=mag_blp,
                mag_target_alp=mag_tlp, mag_losses=mag_L, mag_grad_logits=mag_gl, mag_grad_values=mag_gv)


# ---- the three stand-alone losses (tb_baseline_loss_*, tb_entropy_loss_*, tb_pg_loss_*) -----------------------------
def baseline_loss(adv, u=U32):
    """out = sum 0.5 a^2 (fp64 sum of float products: exact for float32 input), grad = a"""
    a = _f(adv)
    terms = 0.5 * a * a
    s, m = _sum(terms, (u == U64) * terms, u)
    return dict(out=s, mag_out=m + abs(s), grad=a, mag_grad=np.zeros_like(a))


def entropy_loss(logits, u=U32):
    """out = sum over rows of sum_j p_j lp_j, grad_j = p_j (lp_j - ent_row)"""
    ls = log_softmax_rows(logits)
    pr, mag_pr, ent, mag_ent = _entropy_rows(ls)
    s, m = _sum(ent, mag_ent, u)
    h = ls["lp"] - ent[..., None]
    mag_h = ls["mag_lp"] + mag_ent[..., None] + np.abs(h)
    grad = pr * h
    return dict(out=s, mag_out=m + abs(s), grad=grad, mag_grad=pr * mag_h + np.abs(h) * mag_pr + np.abs(grad))


def pg_loss(logits, actions, adv, u=U32):
    """out = sum -log pi(a) adv, grad_j = adv (p_j - onehot(a)_j)"""
    ls = log_softmax_rows(logits)
    a = np.asarray(actions, np.int64)
    ad = _f(adv)
    lpa = np.take_along_axis(ls["lp"], a[..., None], -1)[..., 0]
    mag_lpa = np.take_along_axis(ls["mag_lp"], a[..., None], -1)[..., 0]
    terms = -lpa * ad
    s, m = _sum(terms, np.abs(ad) * mag_lpa + np.abs(terms), u)
    pr = np.exp(ls["lp"])
    mag_pr = _exp_mag(pr, ls["mag_lp"])
    q = pr - np.eye(ls["lp"].shape[-1])[a]
    grad = ad[..., None] * q
    return dict(out=s, mag_out=m + abs(s), grad=grad,
                mag_grad=np.abs(ad)[..., None] * (mag_pr + np.abs(q)) + np.abs(grad))
