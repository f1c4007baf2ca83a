"""The fused optimizer step of csrc/optim.cu restated in float64 NumPy: clip_grad_norm_'s coefficient, then one
torch.optim.RMSprop / Adam / AdamW step in the op order of torch's single-tensor implementations.

Besides the new values, each step returns per-element magnitudes for an error bound on a float32 kernel that starts
from the same float32 state: a running-error analysis, to first order.  Every input is exact except the clipped
gradient g*coef (rounded once), and every float32 operation rounds its result by at most u|result|, u = 2^-24.  A
quantity q then differs from the restatement by at most c u mag(q), with mag built by these rules:
  a + b:   mag(a) + mag(b) + |a + b|     a * b:   |a| mag(b) + |b| mag(a) + |a b|
  a / b:   mag(a) / |b| + |a| mag(b) / b^2 + |a / b|
  sqrt(x): mag(x) / sqrt(x) + sqrt(x)    (|sqrt(x + d) - sqrt(x)| <= |d| / sqrt(x) for any x + d >= 0)
lumped per buffer: a state buffer x = d x_prev + term gets mag = |d x_prev| + mag(term), where mag(term) replaces the
clipped gradient g' by G = |g coef| + |wd p| (g' = g coef + wd p can cancel, its error cannot).  The "update"
magnitude bounds lr times the update, so that the parameter is within 4 u |p| + c u mag["update"]: the 4 u |p| is the
float32 parameter's own roundings (at most three when AdamW's p *= 1 - lr wd comes first)."""
import numpy as np


def _f64(x):
    return None if x is None else np.asarray(x, np.float64)


def _lerp(start, end, weight):
    """torch.lerp: start + w (end - start) for |w| < 0.5, else end - (end - start) (1 - w)"""
    if abs(weight) < 0.5:
        return start + weight * (end - start)
    return end - (end - start) * (1.0 - weight)


def _sqrt_mag(x, mag):
    return np.where(mag > 0, mag / np.sqrt(x), 0.0) + np.sqrt(x)


def clip_coef(norm32, max_norm):
    """float32 min(max_norm / (norm + 1e-6), 1) as torch's clip_grad_norm_ forms it: NaN when the norm is NaN (torch
    clamps with torch.clamp, which propagates NaN), 0 when it is infinite.  max_norm < 0: 1, no clipping."""
    if max_norm < 0:
        return np.float32(1.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        c = np.float32(max_norm) / (np.float32(norm32) + np.float32(1e-6))
    return np.float32(1.0) if c > 1 else c  # NaN > 1 is false: a NaN coefficient stays NaN


# non-finite gradients are inputs too: they propagate as in torch, without warnings
@np.errstate(invalid="ignore", divide="ignore", over="ignore")
def rmsprop_step(p, g, sq, ga, buf, coef, lr, alpha, eps, wd, momentum):
    """One clip + torch.optim.RMSprop step.  ga (grad_avg) None: not centered; buf (momentum_buffer) None: no momentum.
    Returns (new, mag): new has p, g (the clipped gradient) and the state buffers; mag the state buffers' magnitudes and
    "update"."""
    p, g, sq, ga, buf = map(_f64, (p, g, sq, ga, buf))
    gc = g * float(coef)
    gi = gc + wd * p if wd != 0 else gc
    G = np.abs(gc) + np.abs(wd * p)
    sq_new = sq * alpha + (1.0 - alpha) * gi * gi
    mag = {"square_avg": np.abs(alpha * sq) + (1.0 - alpha) * G * G}
    new = {"g": gc, "square_avg": sq_new}
    if ga is not None:
        ga_new = _lerp(ga, gi, 1.0 - alpha)
        x = sq_new - ga_new * ga_new
        mag["grad_avg"] = np.abs(alpha * ga) + (1.0 - alpha) * G
        mag_x = mag["square_avg"] + 2.0 * np.abs(ga_new) * mag["grad_avg"] + ga_new * ga_new
        new["grad_avg"] = ga_new
    else:
        x, mag_x = sq_new, mag["square_avg"]
    avg = np.sqrt(x) + eps
    mag_avg = _sqrt_mag(x, mag_x) + avg
    step = gi / avg
    mag_step = G / avg + np.abs(gi) * mag_avg / (avg * avg)
    if buf is not None:
        buf_new = buf * momentum + step
        mag["momentum_buffer"] = np.abs(momentum * buf) + mag_step
        new["momentum_buffer"] = buf_new
        new["p"] = p + (-lr) * buf_new
        mag["update"] = abs(lr) * mag["momentum_buffer"]
    else:
        new["p"] = p + ((-lr) * gi) / avg  # addcdiv: (value * t1) / t2
        mag["update"] = abs(lr) * mag_step
    return new, mag


@np.errstate(invalid="ignore", divide="ignore", over="ignore")
def adam_step(p, g, m, v, coef, lr, beta1, beta2, eps, wd, decoupled, t):
    """One clip + torch.optim.Adam (decoupled False: L2 weight decay) / AdamW (decoupled True) step, non-amsgrad; t is
    the step being taken (1 for the first).  Returns (new, mag) as rmsprop_step does, with exp_avg and exp_avg_sq."""
    p, g, m, v = map(_f64, (p, g, m, v))
    gc = g * float(coef)
    gi, G, p_in = gc, np.abs(gc), p
    if wd != 0:
        if decoupled:
            p = p * (1.0 - lr * wd)
        else:
            gi = gc + wd * p
            G = G + np.abs(wd * p)
    m_new = _lerp(m, gi, 1.0 - beta1)
    v_new = v * beta2 + (1.0 - beta2) * gi * gi
    bc1 = 1.0 - np.float64(beta1) ** t  # NumPy: t = 0 gives an infinite step, not an exception
    bc2 = 1.0 - np.float64(beta2) ** t
    step_size = lr / bc1
    bc2_sqrt = bc2 ** 0.5
    denom = np.sqrt(v_new) / bc2_sqrt + eps
    mag = {"exp_avg": np.abs(beta1 * m) + (1.0 - beta1) * G, "exp_avg_sq": np.abs(beta2 * v) + (1.0 - beta2) * G * G}
    mag_denom = _sqrt_mag(v_new, mag["exp_avg_sq"]) / bc2_sqrt + denom
    mag_step = mag["exp_avg"] / denom + np.abs(m_new) * mag_denom / (denom * denom)
    mag["update"] = abs(step_size) * mag_step + (abs(lr * wd) * np.abs(p_in) if decoupled else 0.0)
    new = {"g": gc, "exp_avg": m_new, "exp_avg_sq": v_new, "p": p + ((-step_size) * m_new) / denom}
    return new, mag
