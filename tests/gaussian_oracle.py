"""Float64 NumPy restatement of the continuous (diagonal-Gaussian) action-space contract (include/torchbeast_b200.h,
"continuous (diagonal-Gaussian) action spaces"): the fused loss of tb_impala_loss_gaussian_f32 (V-trace on
log rho = log pi(a) - log mu(a), the three losses, the mu / log-sigma gradients, the trust region, column weights and
PopArt) and the Philox / Box-Muller rule of tb_sample_gaussian_f32.  The V-trace part is loss_oracle.scan's recurrence
with the trust region's rho = 0 rows.  Test infrastructure only."""
import numpy as np

from oracle import sampling_np as SO

HALF_LOG_2PI = float(np.float32(0.5 * np.log(2.0 * np.pi)))  # TB_GAUSSIAN_HALF_LOG_2PI, the fp32 constant c


def split(rows):
    """(mu, log sigma) of rows [..., 2D], float64."""
    x = np.asarray(rows, np.float64)
    D = x.shape[-1] // 2
    return x[..., :D], x[..., D:]


def _poison(value, *arrays):
    """value with NaN wherever a row of any of `arrays` [..., n] holds a non-finite entry."""
    bad = np.zeros(np.shape(value), bool)
    for a in arrays:
        bad |= ~np.isfinite(a).all(-1)
    return np.where(bad, np.nan, value)


def log_prob(rows, actions):
    """log pi(a) = sum_k (-0.5 z_k^2 - l_k - c), z_k = (a_k - mu_k) exp(-l_k); [...]."""
    mu, l = split(rows)
    a = np.asarray(actions, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        z = (a - mu) * np.exp(-l)
        lp = np.sum(-0.5 * z * z - l - HALF_LOG_2PI, -1)
    return _poison(lp, mu, l, a)


def entropy_term(rows, actions):
    """ent = sum_k -(l_k + 0.5 + c) (= -H, the sign the flat loss uses for sum p log p); NaN on a non-finite row."""
    mu, l = split(rows)
    with np.errstate(invalid="ignore"):
        ent = np.sum(-(l + 0.5 + HALF_LOG_2PI), -1)
    return _poison(ent, mu, l, np.asarray(actions, np.float64))


def kl(trows, brows):
    """KL(pi || mu_b) = sum_k ((lb_k - l_k) + 0.5 (exp(2 (l_k - lb_k)) + ((mu_k - mub_k) exp(-lb_k))^2) - 0.5)."""
    mu, l = split(trows)
    mub, lb = split(brows)
    with np.errstate(invalid="ignore", over="ignore"):
        dm = (mu - mub) * np.exp(-lb)
        out = np.sum((lb - l) + 0.5 * (np.exp(2.0 * (l - lb)) + dm * dm) - 0.5, -1)
    return _poison(out, mu, l, mub, lb)


def row_grad(rows, actions, adv, entropy_cost):
    """The gradient row [..., 2D]: mu_k gets -adv z_k exp(-l_k), l_k gets adv (1 - z_k^2) - entropy_cost."""
    mu, l = split(rows)
    a = np.asarray(actions, np.float64)
    adv = np.asarray(adv, np.float64)[..., None]
    with np.errstate(invalid="ignore", over="ignore"):
        s = np.exp(-l)
        z = (a - mu) * s
        g = np.concatenate([-adv * z * s, adv * (1.0 - z * z) - entropy_cost], -1)
    bad = ~(np.isfinite(mu).all(-1) & np.isfinite(l).all(-1) & np.isfinite(a).all(-1))
    g[bad] = np.nan
    return g


def impala_loss(blogits, tlogits, actions, rewards, done, values, bootstrap, discounting=0.99, baseline_cost=0.5,
                entropy_cost=0.0006, clip_rewards=True, clip_rho=1.0, clip_pg_rho=1.0, weights=None, trust_beta=None,
                popart=None):
    """The Gaussian loss block on shifted inputs [T, B, ...]: rows [T, B, 2D], actions [T, B, D], done bool [T, B].
    popart: (task [T+1, B], mu [K], nu [K]) with values [T+1, B, K] the normalised head (bootstrap unused).  Returns a
    dict of float64 arrays named like the kernel's outputs."""
    f = np.float64
    bl, tl = np.asarray(blogits, f), np.asarray(tlogits, f)
    T, B, A = tl.shape
    r = np.asarray(rewards, f)
    if clip_rewards:
        r = np.clip(r, -1, 1)
    g = (~np.asarray(done, bool)).astype(f) * discounting
    w = np.ones(B) if weights is None else np.asarray(weights, f)
    if popart is not None:
        task, pmu, pnu = popart
        n = np.asarray(values, f)
        sig = np.clip(np.sqrt(np.maximum(pnu - pmu * pmu, 0)), 1e-4, 1e6)
        ok = (task >= 0) & (task < n.shape[-1])
        tk = np.clip(task, 0, n.shape[-1] - 1)
        nk = np.take_along_axis(n, tk[..., None], -1)[..., 0]
        v_all = np.where(ok, sig[tk] * nk + pmu[tk], 0.0)
        v, v_boot = v_all[:T], v_all[T]
    else:
        v, v_boot = np.asarray(values, f), np.asarray(bootstrap, f)
    tlp, blp = log_prob(tl, actions), log_prob(bl, actions)
    log_rhos = tlp - blp
    kl_rows = kl(tl, bl)
    rho = np.exp(log_rhos)
    if trust_beta is not None:
        rho = np.where(kl_rows <= trust_beta, rho, 0.0)
    rb = np.minimum(rho, clip_rho) if clip_rho is not None else rho
    cs = np.minimum(rho, 1.0)
    rp = np.minimum(rho, clip_pg_rho) if clip_pg_rho is not None else rho
    v_next = np.concatenate([v[1:], v_boot[None]], 0)
    delta = rb * (r + g * v_next - v)
    acc = np.zeros(B)
    vs = np.empty((T, B))
    for t in range(T - 1, -1, -1):
        acc = delta[t] + g[t] * cs[t] * acc
        vs[t] = acc + v[t]
    vs_next = np.concatenate([vs[1:], v_boot[None]], 0)
    adv = rp * (r + g * vs_next - v)
    ent = entropy_term(tl, actions)
    if popart is not None:
        tkT, okT = tk[:T], ok[:T]
        adv_l = adv * np.where(okT, 1.0 / sig[tkT], 0.0)
        d = np.where(okT, (vs - pmu[tkT]) / sig[tkT] - nk[:T], 0.0)
        row_on = okT.astype(f)
    else:
        adv_l, d, row_on = adv, vs - v, np.ones((T, B))
    pg = np.sum(-tlp * adv_l * w * row_on)
    bl_loss = baseline_cost * np.sum(0.5 * d * d * w * row_on)
    en = entropy_cost * np.sum(ent * w * row_on)
    grad = row_grad(tl, actions, adv_l, entropy_cost) * (w[None, :, None] * row_on[..., None])
    if popart is not None:
        K = n.shape[-1]
        gv = np.zeros((T + 1, B, K))
        tt, bb = np.nonzero(okT)
        gv[tt, bb, tkT[tt, bb]] = -baseline_cost * d[tt, bb]
    else:
        gv = -baseline_cost * d * w
    out = dict(vs=vs, pg_adv=adv, log_rhos=log_rhos, target_alp=tlp, behavior_alp=blp, kl=kl_rows,
               losses=np.array([pg, bl_loss, en, pg + bl_loss + en]), grad_logits=grad, grad_values=gv,
               trusted=None if trust_beta is None else float(np.sum(kl_rows <= trust_beta)))
    if popart is not None:
        K = n.shape[-1]
        sums = np.zeros((3, K))
        for k in range(K):
            sel = tk[:T][ok[:T]] == k
            vals = vs[ok[:T]][sel]
            sums[:, k] = (vals.size, vals.sum(), (vals * vals).sum())
        out["task_sums"] = sums
    return out


def gaussian_words(T, B, seed, step, D, stream_ids=None):
    """(x0, x1) uint32 [T, B, D] each: component k's word pair (2 (k % 2), 2 (k % 2) + 1) of the Philox block keyed
    (lo32(seed), hi32(seed) + k // 2) under the flat sampler's counter (step + t, stream id)."""
    sid = np.arange(B, dtype=np.uint64) if stream_ids is None else np.asarray(stream_ids, dtype=np.int64).view(np.uint64)
    lo = np.uint64(0xFFFFFFFF)
    with np.errstate(over="ignore"):
        ctr = np.uint64(step) + np.arange(T, dtype=np.uint64)
    ctr, sid = np.broadcast_arrays(ctr[:, None], sid[None, :])
    seed = np.uint64(seed)
    x0 = np.empty((T, B, D), dtype=np.uint32)
    x1 = np.empty((T, B, D), dtype=np.uint32)
    for k in range(D):
        with np.errstate(over="ignore"):
            k1 = (np.uint32(seed >> np.uint64(32)) + np.uint32(k // 2)).astype(np.uint32)
        words = SO.philox4x32_10((ctr & lo, ctr >> np.uint64(32), sid & lo, sid >> np.uint64(32)),
                                 (np.uint32(seed & lo), k1))
        x0[..., k], x1[..., k] = words[2 * (k % 2)], words[2 * (k % 2) + 1]
    return x0, x1


def uniforms(T, B, seed, step, D, stream_ids=None):
    """(u1 in (0, 1], u2 in [0, 1)) float64 [T, B, D], exact: 24-bit values times 2^-24."""
    x0, x1 = gaussian_words(T, B, seed, step, D, stream_ids)
    u1 = ((x0 >> np.uint32(8)).astype(np.float64) + 1.0) * 2.0 ** -24
    u2 = (x1 >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
    return u1, u2


def sample(rows, seed, step, stream_ids=None):
    """rows [T, B, 2D] -> actions float64 [T, B, D]: a_k = mu_k + exp(l_k) sqrt(-2 log u1) cos(2 pi u2); NaN where
    mu_k or l_k is non-finite.  Also returns z [T, B, D]."""
    mu, l = split(rows)
    T, B, D = mu.shape
    u1, u2 = uniforms(T, B, seed, step, D, stream_ids)
    z = np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)
    with np.errstate(invalid="ignore", over="ignore"):
        a = mu + np.exp(l) * z
    a[~(np.isfinite(mu) & np.isfinite(l))] = np.nan
    return a, z


def sample_tolerance(rows, z):
    """A bound on |fp32 sample - float64 rule| per component: sqrtf, logf and cospif are within 1-2 ulp (CUDA C
    Programming Guide, Mathematical Functions); the fp32 z then carries a relative error of a few 2^-24 plus the
    absolute one of cospif near its zeros, and expf(l) * z + mu two more roundings.  8 ulp of every term, plus the
    cospif absolute error scaled by sigma sqrt(-2 log u1) <= sigma * 5.8, is generous and still 10^4 below one
    standard deviation."""
    mu, l = split(rows)
    sig = np.exp(l)
    u = 2.0 ** -24
    return 8 * u * (np.abs(mu) + sig * np.abs(z) + np.abs(mu + sig * z)) + 8 * u * sig * 5.8
