"""Float64 NumPy restatement of the factored (multi-discrete) action-space contract (include/torchbeast_b200.h,
"multi-discrete (factored) action spaces"): the fused loss of tb_impala_loss_factored_f32 (V-trace on the summed
log rho, the three losses, the per-segment gradients, the trust region and PopArt) and the Philox rule of
tb_sample_actions_factored_f32.  Test infrastructure only."""
import numpy as np

from oracle import sampling_np as SO


def offsets(dims):
    return np.concatenate([[0], np.cumsum(dims)]).astype(np.int64)


def log_softmax_segments(x, dims):
    """Per-segment log-softmax of x [..., sum dims], float64."""
    x = np.asarray(x, dtype=np.float64)
    off = offsets(dims)
    out = np.empty_like(x)
    for k in range(len(dims)):
        s = x[..., off[k]:off[k + 1]]
        m = s.max(axis=-1, keepdims=True)
        out[..., off[k]:off[k + 1]] = (s - m) - np.log(np.exp(s - m).sum(axis=-1, keepdims=True))
    return out


def action_log_probs(x, actions, dims):
    """log pi(a) = sum_k log pi_k(a_k) [...]; an a_k outside [0, A_k) gives NaN."""
    lp = log_softmax_segments(x, dims)
    off = offsets(dims)
    out = np.zeros(lp.shape[:-1])
    for k, a in enumerate(dims):
        ak = actions[..., k]
        ok = (ak >= 0) & (ak < a)
        picked = np.take_along_axis(lp[..., off[k]:off[k + 1]], np.clip(ak, 0, a - 1)[..., None], -1)[..., 0]
        out = out + np.where(ok, picked, np.nan)
    return out


def segment_sums(v, dims):
    """[..., sum dims] -> [..., D]: the sum over each segment."""
    off = offsets(dims)
    return np.stack([v[..., off[k]:off[k + 1]].sum(-1) for k in range(len(dims))], -1)


def impala_loss(blogits, tlogits, actions, rewards, done, values, bootstrap, dims, discounting=0.99,
                baseline_cost=0.5, entropy_cost=0.0006, clip_rewards=True, clip_rho=1.0, clip_pg_rho=1.0,
                weights=None, trust_beta=None, popart=None):
    """The factored loss block on shifted inputs [T, B, ...]; actions [T, B, D]; done bool [T, B].
    popart: (task [T+1, B], mu [K], nu [K]) with values [T+1, B, K] the normalised head (bootstrap unused).
    Returns a dict of float64 arrays named like the kernel's outputs."""
    f = np.float64
    bl, tl = np.asarray(blogits, f), np.asarray(tlogits, f)
    T, B, A = tl.shape
    r = np.asarray(rewards, f)
    if clip_rewards:
        r = np.clip(r, -1, 1)
    g = (~np.asarray(done, bool)).astype(f) * discounting
    w = np.ones(B) if weights is None else np.asarray(weights, f)
    if popart is not None:
        task, mu, nu = popart
        n = np.asarray(values, f)
        sig = np.clip(np.sqrt(np.maximum(nu - mu * mu, 0)), 1e-4, 1e6)
        ok = (task >= 0) & (task < n.shape[-1])
        tk = np.clip(task, 0, n.shape[-1] - 1)
        nk = np.take_along_axis(n, tk[..., None], -1)[..., 0]
        v_all = np.where(ok, sig[tk] * nk + mu[tk], 0.0)
        v, v_boot = v_all[:T], v_all[T]
    else:
        v, v_boot = np.asarray(values, f), np.asarray(bootstrap, f)
    tlp, blp = action_log_probs(tl, actions, dims), action_log_probs(bl, actions, dims)
    log_rhos = tlp - blp
    lpt, lpb = log_softmax_segments(tl, dims), log_softmax_segments(bl, dims)
    pt = np.exp(lpt)
    kl = segment_sums(pt * (lpt - lpb), dims).sum(-1)
    rho = np.exp(log_rhos)
    if trust_beta is not None:
        rho = np.where(kl <= trust_beta, rho, 0.0)
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
    ent_k = segment_sums(pt * lpt, dims)  # [T, B, D]
    ent = ent_k.sum(-1)
    if popart is not None:
        tkT, okT = tk[:T], ok[:T]
        pg_scale = np.where(okT, 1.0 / sig[tkT], 0.0)
        adv_l = adv * pg_scale
        nkT = nk[:T]
        d = np.where(okT, (vs - mu[tkT]) / sig[tkT] - nkT, 0.0)
        row_on = okT.astype(f)
    else:
        adv_l, d, row_on = adv, vs - v, np.ones((T, B))
    pg = np.sum(-tlp * adv_l * w * row_on)
    bl_loss = baseline_cost * np.sum(0.5 * d * d * w * row_on)
    en = entropy_cost * np.sum(ent * w * row_on)
    onehot = np.zeros((T, B, A))
    off = offsets(dims)
    for k in range(len(dims)):
        ak = actions[..., k]
        ok_a = (ak >= 0) & (ak < dims[k])
        tt, bb = np.nonzero(ok_a)
        onehot[tt, bb, off[k] + ak[tt, bb]] = 1.0
    ent_cols = np.repeat(ent_k, dims, axis=-1)
    grad = adv_l[..., None] * (pt - onehot) + entropy_cost * pt * (lpt - ent_cols)
    grad = grad * (w[None, :, None] * row_on[..., None])
    if popart is not None:
        K = n.shape[-1]
        gv = np.zeros((T + 1, B, K))
        tt, bb = np.nonzero(okT)
        gv[tt, bb, tkT[tt, bb]] = -baseline_cost * d[tt, bb]
    else:
        gv = -baseline_cost * d * w
    out = dict(vs=vs, pg_adv=adv, log_rhos=log_rhos, target_alp=tlp, behavior_alp=blp, kl=kl,
               losses=np.array([pg, bl_loss, en, pg + bl_loss + en]), grad_logits=grad, grad_values=gv,
               trusted=None if trust_beta is None else float(np.sum(kl <= trust_beta)))
    if popart is not None:
        K = n.shape[-1]
        sums = np.zeros((3, K))
        for k in range(K):
            sel = tk[:T][ok[:T]] == k
            vals = vs[ok[:T]][sel]
            sums[:, k] = (vals.size, vals.sum(), (vals * vals).sum())
        out["task_sums"] = sums
    return out


def factored_words(T, B, seed, step, D, stream_ids=None):
    """x [T, B, D] uint32: component k's Philox word, word k % 4 of the block keyed (lo32(seed), hi32(seed) + k // 4)
    under the flat sampler's counter."""
    sid = np.arange(B, dtype=np.uint64) if stream_ids is None else np.asarray(stream_ids, dtype=np.int64).view(np.uint64)
    lo = np.uint64(0xFFFFFFFF)
    with np.errstate(over="ignore"):
        ctr = np.uint64(step) + np.arange(T, dtype=np.uint64)
    ctr, sid = np.broadcast_arrays(ctr[:, None], sid[None, :])
    seed = np.uint64(seed)
    out = np.empty((T, B, D), dtype=np.uint32)
    for k in range(D):
        with np.errstate(over="ignore"):
            k1 = (np.uint32(seed >> np.uint64(32)) + np.uint32(k // 4)).astype(np.uint32)
        words = SO.philox4x32_10((ctr & lo, ctr >> np.uint64(32), sid & lo, sid >> np.uint64(32)),
                                 (np.uint32(seed & lo), k1))
        out[..., k] = words[k % 4]
    return out


def sample_actions(logits, dims, seed, step, stream_ids=None):
    """logits [T, B, sum dims] -> (actions int64 [T, B, D], margin float64 [T, B, D]), each segment by the flat
    contract's steps 2-5 (oracle.sampling_np) with its own uniform."""
    x = np.asarray(logits, dtype=np.float64)
    T, B, _ = x.shape
    u = (factored_words(T, B, seed, step, len(dims), stream_ids) >> np.uint32(8)).astype(np.float64) * 2.0 ** -24
    off = offsets(dims)
    acts = np.empty((T, B, len(dims)), dtype=np.int64)
    margin = np.empty((T, B, len(dims)))
    for k in range(len(dims)):
        a, m = _sample_with_u(x[..., off[k]:off[k + 1]], u[..., k])
        acts[..., k], margin[..., k] = a, m
    return acts, margin


def _sample_with_u(x, u):
    """oracle.sampling_np.sample_actions with the uniforms given."""
    A = x.shape[-1]
    with np.errstate(invalid="ignore"):
        m = np.max(np.where(np.isnan(x), -np.inf, x), axis=-1)
    bad = np.isnan(x).any(axis=-1) | ~np.isfinite(m)
    m = np.where(bad, 0.0, m)
    with np.errstate(invalid="ignore", over="ignore"):
        e = np.where(bad[..., None], 0.0, np.exp(x - m[..., None]))
    c = np.cumsum(e, axis=-1)
    S = c[..., -1]
    target = u * S
    above = c > target[..., None]
    first = np.argmax(above, axis=-1)
    last_pos = A - 1 - np.argmax((e > 0)[..., ::-1], axis=-1)
    actions = np.where(above.any(axis=-1), first, last_pos).astype(np.int64)
    with np.errstate(invalid="ignore", divide="ignore"):
        margin = np.min(np.abs(c - target[..., None]), axis=-1) / S
    actions[bad] = -1
    margin[bad] = np.inf
    return actions, margin
