"""The kickstarting term of tb_kickstart_loss_f32 (include/torchbeast_b200.h) restated in float64 NumPy: the row
log-softmaxes, KL(p_T || p_S) per row with 0 * log 0 = 0, the weighted loss and its closed-form gradient
cost * w_b * (p_S - p_T) with respect to the learner's logits."""
import numpy as np


def log_softmax(x):
    x = np.asarray(x, np.float64)
    m = x.max(-1, keepdims=True)
    return (x - m) - np.log(np.exp(x - m).sum(-1, keepdims=True))


def row_kl(teacher_logits, target_logits):
    """KL_t [T, B] = sum_a p_T(a) (log p_T(a) - log p_S(a)); a term with p_T(a) == 0 (a -inf teacher logit) is 0."""
    lt, ls = log_softmax(teacher_logits), log_softmax(target_logits)
    pt = np.exp(lt)
    with np.errstate(invalid="ignore"):
        terms = np.where(pt == 0.0, 0.0, pt * (lt - ls))
    return terms.sum(-1)


def loss(teacher_logits, target_logits, cost, weights=None):
    """dict(kl [T, B], kl_sum, loss = cost * sum_{t,b} w_b KL_t, grad_logits [T, B, A] = cost * w_b * (p_S - p_T))."""
    kl = row_kl(teacher_logits, target_logits)
    B = kl.shape[1]
    w = np.ones(B) if weights is None else np.asarray(weights, np.float64)
    pt, ps = np.exp(log_softmax(teacher_logits)), np.exp(log_softmax(target_logits))
    grad = cost * w[None, :, None] * (ps - pt)
    return dict(kl=kl, kl_sum=kl.sum(), loss=cost * (w[None, :] * kl).sum(), grad_logits=grad)
