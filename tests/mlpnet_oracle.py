"""Float64 references for MLPNet (include/torchbeast_b200.h, "MLPNet"): the state_dict spec, the net as a torch module
of its own, the fp32 staging rule, and the running observation statistics in NumPy."""
import numpy as np
import torch

CLIP, EPS = 10.0, 1e-8


def spec(obs_dim, hidden, num_actions, use_lstm, num_values=1, continuous_dim=None):
    """[(name, shape)] in state_dict order, restated from the header: torso, then AtariNet's core / policy / baseline."""
    out, fan_in = [], obs_dim
    for i, h in enumerate(hidden):
        out += [("torso.%d.weight" % i, (h, fan_in)), ("torso.%d.bias" % i, (h,))]
        fan_in = h
    core = hidden[-1] + 1 + (num_actions if continuous_dim is None else continuous_dim)
    if use_lstm:
        for l in range(2):
            out += [("core.weight_ih_l%d" % l, (4 * core, core)), ("core.weight_hh_l%d" % l, (4 * core, core)),
                    ("core.bias_ih_l%d" % l, (4 * core,)), ("core.bias_hh_l%d" % l, (4 * core,))]
    out += [("policy.weight", (num_actions, core)), ("policy.bias", (num_actions,)),
            ("baseline.weight", (num_values, core)), ("baseline.bias", (num_values,))]
    return out


def normalize(x, mean, var):
    """The float64 normalisation: clamp((x - mean) / sqrt(var + 1e-8), -10, 10)."""
    return ((x - mean) / torch.sqrt(var + EPS)).clamp(-CLIP, CLIP)


def stage_f32(x, mean=None, var=None):
    """The staging kernel's fp32 rule, bit for bit: mean_f = float(mean), inv_std_f = float(1 / sqrt(var + 1e-8))
    formed in float64, y = (x - mean_f) * inv_std_f in two fp32 roundings, clamped to [-10, 10] (NaN stays NaN)."""
    x = x.to(torch.float32)
    if mean is None:
        return x
    mean_f = mean.to(torch.float64).to(torch.float32)
    inv_f = (1.0 / torch.sqrt(var.to(torch.float64) + EPS)).to(torch.float32)
    return ((x - mean_f) * inv_f).clamp(-CLIP, CLIP)


def _lstm(x, notdone, state, p, core):
    """2-layer LSTM over [T, B, F] with state *= notdone_t before each step (torch.nn.LSTM gate order i, f, g, o)."""
    h, c = [s.clone() for s in state[0]], [s.clone() for s in state[1]]
    ys = []
    for t in range(x.shape[0]):
        inp = x[t]
        for l in range(2):
            h[l], c[l] = h[l] * notdone[t][:, None], c[l] * notdone[t][:, None]
            g = inp @ p["core.weight_ih_l%d" % l].T + p["core.bias_ih_l%d" % l] + h[l] @ p["core.weight_hh_l%d" % l].T \
                + p["core.bias_hh_l%d" % l]
            i, f, gg, o = g.split(core, -1)
            c[l] = torch.sigmoid(f) * c[l] + torch.sigmoid(i) * torch.tanh(gg)
            h[l] = torch.sigmoid(o) * torch.tanh(c[l])
            inp = h[l]
        ys.append(inp)
    return torch.stack(ys), (torch.stack(h), torch.stack(c))


def forward(params, frame, reward, last_action, done=None, state=None, hidden=(256,), num_actions=6, space=None,
            mean=None, var=None):
    """logits [T, B, A], baseline [T, B, V], (hN, cN) of the net on float64 `params` (a dict of tensors, e.g. with
    requires_grad).  space: None (one-hot), a tuple of component sizes (K-hot) or ("gaussian", D) (raw values)."""
    f64 = torch.float64
    x = frame.to(f64)
    if mean is not None:
        x = normalize(x, mean.to(f64), var.to(f64))
    for i in range(len(hidden)):
        x = torch.relu(x @ params["torso.%d.weight" % i].T + params["torso.%d.bias" % i])
    T, B = x.shape[:2]
    r = reward.to(f64).clamp(-1, 1)[..., None]
    if space is None:
        enc = torch.nn.functional.one_hot(last_action.long(), num_actions).to(f64)
    elif space[0] == "gaussian":
        enc = last_action.to(f64)
    else:
        enc = torch.cat([torch.nn.functional.one_hot(last_action[..., k].long(), a).to(f64)
                         for k, a in enumerate(space)], -1)
    core = torch.cat([x, r, enc], -1)
    new_state = ()
    if "core.weight_ih_l0" in params:
        notdone = (~done).to(f64)
        core, new_state = _lstm(core, notdone, state, params, core.shape[-1])
    logits = core @ params["policy.weight"].T + params["policy.bias"]
    baseline = core @ params["baseline.weight"].T + params["baseline.bias"]
    return logits, baseline, new_state


def merge(count, mean, var, x):
    """The header's statistics merge of rows x [N, O] (float64; non-finite entries skipped per feature) into (count,
    mean, var), restated in NumPy.  Returns the new (count, mean, var)."""
    x = np.asarray(x, np.float64)
    fin = np.isfinite(x)
    xs = np.where(fin, x, 0.0)
    nb, s, s2 = fin.sum(0).astype(np.float64), xs.sum(0), (xs * xs).sum(0)
    count, mean, var = (np.array(a, np.float64, copy=True) for a in (count, mean, var))
    on = nb > 0
    mb = np.where(on, s / np.where(on, nb, 1), 0.0)
    vb = np.maximum(np.where(on, s2 / np.where(on, nb, 1), 0.0) - mb * mb, 0.0)
    tot = count + nb
    d = mb - mean
    safe = np.where(on, tot, 1)
    new_mean = mean + d * nb / safe
    new_var = (var * count + vb * nb + d * d * count * nb / safe) / safe
    return np.where(on, tot, count), np.where(on, new_mean, mean), np.where(on, new_var, var)


def two_pass(x):
    """(count, mean, population variance) of each feature over rows x [N, O], non-finite entries skipped."""
    x = np.asarray(x, np.float64)
    out = [], [], []
    for j in range(x.shape[1]):
        col = x[:, j][np.isfinite(x[:, j])]
        out[0].append(float(len(col)))
        m = col.mean() if len(col) else 0.0
        out[1].append(m)
        out[2].append(((col - m) ** 2).mean() if len(col) else 1.0)
    return tuple(np.array(a) for a in out)
