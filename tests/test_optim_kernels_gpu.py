"""GPU: the optimizer kernels of csrc/optim.cu in isolation - tb_grad_sumsq_f32 and the three clip + step entry points -
against the float64 restatement in tests/optim_oracle.py and, for non-finite gradients, against torch's clip_grad_norm_
and optimizers in float64.

The step kernels run each configuration for five chained steps, with the state carried through; before every step the
restatement takes the kernel's float32 state, so each step is checked on its own:
- exact: the clipped gradient written back is float32(g * coef) bit for bit, and grad_norm_out is sqrtf(sumsq);
- bounded: a state buffer within C u mag and the parameter within 4 u |p| + C u mag["update"], u = 2^-24, with the
  magnitudes of the restatement (see its docstring).  C = 8 covers the roundings along the longest chain, the momentum
  buffer's: the clipped gradient, the weight-decay term, the square average, its root plus eps, the division and the
  buffer's own update.  Each check also shows that the bound rejects the restatement with one plausible mistake: the
  unclipped gradient, a momentum buffer that is not decayed, or Adam's bias corrections taken at step t - 1;
- the paths: the 128-bit loops, their n % 4 scalar tails, the scalar fallback when any buffer is not 16-byte aligned
  (each moved 1 to 3 floats in turn), and clip_rmsprop_kernel's momentum loop; clipping off, inactive and active; lr
  from the device scalar and from the argument; Adam's device step counter from 0, 1, 9 and 10^6.
Every buffer lies inside a larger allocation between sentinel words that must come back untouched, and the first step
of each configuration runs twice from the same state and must give the same bits."""
import numpy as np
import pytest
import torch

from tests import optim_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C = 8
PAD = 8                   # sentinel floats before a buffer's 16-byte boundary and after its end
SENTINEL = 0x7FC0BEEF     # a NaN with a payload no kernel writes
GRID_CAP = 132 * 4 * 256 * 4  # tb_grad_sumsq_f32's last size before its grid cap (kNumSMs * 4 CTAs of 256 float4)
LEARNER_N = 6_005_848     # the AtariNet + LSTM flat buffer at A = 6


def lib():
    from torchbeast_b200 import _lib
    return _lib.lib()


def P(t):
    from torchbeast_b200 import _lib
    return _lib.ptr(t)


def stream():
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    rc = getattr(lib(), name)(*args)
    assert rc == 0, "%s: %s" % (name, lib().tb_last_error().decode())


def sync():
    torch.cuda.synchronize()


def same_bits(a, b):
    """float32 arrays equal bit for bit, any NaN matching any NaN"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int32), b[~nb].view(np.int32))


class Slab:
    """n float32 values `off` floats past a 16-byte boundary, between sentinel words, in one allocation"""

    def __init__(self, values, off=0):
        values = np.asarray(values, np.float32)
        self.lo, self.n = PAD + off, values.size
        words = torch.full((self.lo + self.n + PAD,), SENTINEL, dtype=torch.int32, device="cuda")
        self.base = words.view(torch.float32)
        self.t = self.base[self.lo:self.lo + self.n]
        self.t.copy_(torch.from_numpy(values))
        assert (self.t.data_ptr() % 16 == 0) == (off % 4 == 0)

    def get(self):
        return self.t.cpu().numpy()

    def set(self, values):
        self.t.copy_(torch.from_numpy(np.asarray(values, np.float32)))

    def sentinels_intact(self):
        b = self.base.view(torch.int32)
        return bool((b[:self.lo] == SENTINEL).all()) and bool((b[self.lo + self.n:] == SENTINEL).all())


def scalar(value, dtype=torch.float32):
    return torch.tensor([value], dtype=dtype, device="cuda")


# ---------------------------------------------------------------------------------------------------------------------
# tb_grad_sumsq_f32
# ---------------------------------------------------------------------------------------------------------------------
SUMSQ_SIZES = [0, 1, 3, 4, 5, 1023, GRID_CAP - 1, GRID_CAP + 5, LEARNER_N, LEARNER_N + 3]


def workspace():
    """a fresh workspace: ticket counter 0, the per-CTA partials NaN (every CTA must write its own before the fold)"""
    ws = torch.zeros(lib().tb_workspace_bytes(), dtype=torch.uint8, device="cuda")
    ws[64:].view(torch.float64).fill_(float("nan"))
    return ws


def sumsq(g, ws):
    """tb_grad_sumsq_f32 of a Slab, twice: the same bits both times, and the ticket counter back at 0 after each"""
    outs = []
    for _ in range(2):
        out = Slab(np.full(1, np.nan, np.float32))
        call("tb_grad_sumsq_f32", P(g.t), g.n, P(out.t), P(ws), stream())
        sync()
        assert int(ws[:4].view(torch.int32)[0]) == 0, "the ticket counter was not reset"
        assert out.sentinels_intact() and g.sentinels_intact()
        outs.append(out.get())
    assert same_bits(outs[0], outs[1]), "a second call gave other bits"
    return outs[0][0]


@pytest.mark.parametrize("n", SUMSQ_SIZES)
def test_grad_sumsq_exact(n):
    """integers in [-64, 64]: each float4's fp32 partial stays below 2^24 and the fp64 total is exact, so the result is
    float32(exact sum) whatever the grid and the fold order"""
    gen = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randint(-64, 65, (n,), device="cuda", generator=gen)
    g = Slab(np.zeros(n, np.float32))
    g.t.copy_(x)
    got = sumsq(g, workspace())
    assert same_bits(got, np.float32(float((x.long() ** 2).sum()))), (got, int((x.long() ** 2).sum()))


@pytest.mark.parametrize("n", SUMSQ_SIZES)
def test_grad_sumsq_bounded(n):
    """randn: each float4's partial takes four fp32 roundings (one square, three fmas: at most 4 u of the partial), the
    fp64 sums add nothing visible and the result rounds once to fp32, so |out - S| <= 5 u S for the fp64 sum S of the
    squares; the bound must see the largest square dropped"""
    gen = torch.Generator(device="cuda").manual_seed(100 + n)
    g = Slab(np.zeros(n, np.float32))
    g.t.normal_(generator=gen)
    got = float(sumsq(g, workspace()))
    sq = g.t.double() ** 2
    S = float(sq.sum())
    tol = 5.0 * U * S * (1 + 1e-9) + 1e-300
    assert abs(got - S) <= tol, (got, S, abs(got - S) / tol)
    if n:
        assert float(sq.max()) > tol, "the bound cannot see a dropped element"


def test_grad_sumsq_shared_workspace_across_sizes():
    """one workspace reused across grids of every size: the counter a multi-CTA call leaves behind must not disturb the
    next (the learner's optimizer shares one workspace per stream)"""
    ws = workspace()
    for n in (LEARNER_N, 5, GRID_CAP + 5, 1, GRID_CAP - 1):
        gen = torch.Generator(device="cuda").manual_seed(7 * n)
        x = torch.randint(-64, 65, (n,), device="cuda", generator=gen)
        g = Slab(np.zeros(n, np.float32))
        g.t.copy_(x)
        assert same_bits(sumsq(g, ws), np.float32(float((x.long() ** 2).sum()))), n


def test_grad_sumsq_rejects_misaligned_before_any_launch():
    g = Slab(np.ones(100, np.float32), off=1)
    out = Slab(np.full(1, np.nan, np.float32))
    before = lib().tb_launch_count()
    rc = lib().tb_grad_sumsq_f32(P(g.t), g.n, P(out.t), P(workspace()), stream())
    assert rc != 0
    assert "tb_grad_sumsq_f32: gradient buffer must be 16-byte aligned" in lib().tb_last_error().decode()
    assert lib().tb_launch_count() == before
    sync()
    assert np.isnan(out.get()).all() and out.sentinels_intact()


# ---------------------------------------------------------------------------------------------------------------------
# the clip + step kernels
# ---------------------------------------------------------------------------------------------------------------------
LR = 1e-2
MAX_NORM = 40.0
# per chained step: the clip (off: max_norm < 0; below: the norm under the threshold, coef exactly 1; above) and where
# lr comes from
SCHEDULE = [("above", True), ("below", False), ("off", True), ("above", False), ("above", True)]
NORMS = {"above": 60.0, "below": 20.0, "off": 60.0}


def f32(x):
    return float(np.float32(x))


def state_keys(kind, o):
    if kind == "adam":
        return ["exp_avg", "exp_avg_sq"]
    return ["square_avg"] + (["grad_avg"] if o.get("centered") else []) + (["momentum_buffer"] if o["momentum"] else [])


def initial_state(kind, o, n, rs, step0):
    """a state as after some training at gradients of rms s = 60 / sqrt(n); Adam from step 0 starts from zeros"""
    s = NORMS["above"] / np.sqrt(max(n, 1))
    st = {"p": rs.randn(n) * 5 * LR}
    if kind == "adam":
        live = step0 > 0
        st["exp_avg"], st["exp_avg_sq"] = rs.randn(n) * 0.3 * s * live, rs.rand(n) * s * s * live
    else:
        st["square_avg"] = (0.5 + rs.rand(n)) * s * s
        if o.get("centered"):
            st["grad_avg"] = rs.randn(n) * 0.1 * s
        if o["momentum"]:
            st["momentum_buffer"] = rs.randn(n) * 0.3
    return {k: v.astype(np.float32) for k, v in st.items()}


def launch(kind, o, b, n, sumsq_t, max_norm, lr_dev, step_dev, norm_out):
    """one entry-point call on the Slabs b; lr_dev None: lr from the argument, else from the device scalar, with a
    wrong argument beside it"""
    lr = -7.0 if lr_dev is not None else LR
    t = lambda key: P(b[key].t) if key in b else None  # noqa: E731
    if kind == "rmsprop":
        call("tb_clip_rmsprop_step_f32", t("p"), t("g"), t("square_avg"), t("momentum_buffer"), n, P(sumsq_t), max_norm,
             P(lr_dev), lr, o["alpha"], o["eps"], o["momentum"], None, P(norm_out), stream())
    elif kind == "rmsprop_ex":
        call("tb_clip_rmsprop_ex_step_f32", t("p"), t("g"), t("square_avg"), t("grad_avg"), t("momentum_buffer"), n,
             P(sumsq_t), max_norm, P(lr_dev), lr, o["alpha"], o["eps"], o["wd"], o["momentum"], None, P(norm_out),
             stream())
    else:
        call("tb_clip_adam_step_f32", t("p"), t("g"), t("exp_avg"), t("exp_avg_sq"), n, P(sumsq_t), max_norm, P(lr_dev),
             lr, o["beta1"], o["beta2"], o["eps"], o["wd"], int(o["decoupled"]), P(step_dev), None, P(norm_out),
             stream())


def oracle(kind, o, s, coef, t, momentum=None):
    """the restatement from the float32 state s, with the float32 values the kernel takes (Adam's betas are double)"""
    if kind == "adam":
        return O.adam_step(s["p"], s["g"], s["exp_avg"], s["exp_avg_sq"], coef, f32(LR), o["beta1"], o["beta2"],
                           f32(o["eps"]), f32(o["wd"]), o["decoupled"], t)
    return O.rmsprop_step(s["p"], s["g"], s["square_avg"], s.get("grad_avg"), s.get("momentum_buffer"), coef, f32(LR),
                          f32(o["alpha"]), f32(o["eps"]), f32(o.get("wd", 0.0)),
                          f32(o["momentum"] if momentum is None else momentum))


def worst(got, want, mag, p0, keys):
    """max over the buffers of |got - want| / bound; a non-finite difference counts as infinitely far"""
    r = 0.0
    for key in keys + ["p"]:
        if key == "p":
            tol = 4 * U * np.maximum(np.abs(p0), np.abs(want["p"])) + C * U * mag["update"]
        else:
            tol = C * U * mag[key]
        err = np.abs(np.asarray(got[key], np.float64) - want[key])
        ratio = np.where(np.isfinite(err), err / (tol + 1e-300), np.inf)
        r = max(r, float(ratio.max(initial=0.0)))
    return r


def mistakes(kind, o, s, coef, t):
    """the restatement with one plausible mistake each, where the mistake changes the step"""
    out = {}
    if coef < 1:
        out["unclipped gradient"] = oracle(kind, o, s, 1.0, t)[0]
    if o.get("momentum") and np.any(s["momentum_buffer"] != 0):
        out["momentum buffer not decayed"] = oracle(kind, o, s, coef, t, momentum=1.0)[0]
    if kind == "adam" and t < 100 and (o["beta1"] > 0 or o["beta2"] > 0):
        out["bias corrections at t - 1"] = oracle(kind, o, s, coef, t - 1)[0]
    return out


def chain(kind, o, n, offs=None, step0=0, seed=0):
    """the SCHEDULE's chained calls of one configuration; offs: {buffer: floats off its 16-byte boundary}"""
    offs = offs or {}
    keys = state_keys(kind, o)
    rs = np.random.RandomState(seed)
    init = initial_state(kind, o, n, rs, step0)
    b = {k: Slab(v, offs.get(k, 0)) for k, v in init.items()}
    b["g"] = Slab(np.zeros(n, np.float32), offs.get("g", 0))
    step_dev = scalar(step0, torch.int64) if kind == "adam" else None
    lr_t = Slab(np.full(1, LR, np.float32))
    rejected = set()
    for k, (clip, lr_from_device) in enumerate(SCHEDULE):
        g = rs.randn(n)
        g = (g * (NORMS[clip] / np.linalg.norm(g))).astype(np.float32)
        b["g"].set(g)
        S = np.float32((g.astype(np.float64) ** 2).sum())
        norm32 = np.sqrt(S)
        max_norm = -1.0 if clip == "off" else MAX_NORM
        coef = O.clip_coef(norm32, max_norm)
        assert (coef == 1) == (clip != "above")
        s = {key: slab.get() for key, slab in b.items()}
        t = step0 + k + 1
        for repeat in range(2 if k == 0 else 1):
            if repeat:
                first = {key: slab.get() for key, slab in b.items()}
                for key, slab in b.items():
                    slab.set(s[key])
                if step_dev is not None:
                    step_dev.fill_(step0)
            norm_out = Slab(np.full(1, np.nan, np.float32))
            sumsq_t = Slab(np.full(1, S, np.float32))
            launch(kind, o, b, n, sumsq_t.t, max_norm, lr_t.t if lr_from_device else None, step_dev, norm_out.t)
            sync()
            assert same_bits(norm_out.get(), [norm32]), (norm_out.get(), norm32)
            assert norm_out.sentinels_intact() and sumsq_t.sentinels_intact() and lr_t.sentinels_intact()
            if step_dev is not None:
                assert int(step_dev[0]) == step0 + k + 1, "the step counter must advance by exactly 1"
        got = {key: slab.get() for key, slab in b.items()}
        if k == 0:
            assert all(same_bits(got[key], first[key]) for key in b), "a second call gave other bits"
        assert all(slab.sentinels_intact() for slab in b.values()), "a write outside a buffer"
        want, mag = oracle(kind, o, s, coef, t)
        assert same_bits(got["g"], np.float32(want["g"])), "the clipped gradient written back"
        if clip != "above":
            assert same_bits(got["g"], g), "coef 1 must leave the gradient bit-identical"
        r = worst(got, want, mag, s["p"], keys)
        assert r <= 1.0, "step %d (%s): %.3g of the bound" % (k, clip, r)
        for what, wrong in mistakes(kind, o, s, coef, t).items():
            assert worst(wrong, want, mag, s["p"], keys) > 1.0, "the bound cannot see: %s (step %d)" % (what, k)
            rejected.add(what)
    assert rejected, "no mistake applied"
    return rejected


def paths(buffers, n=4096):
    """(id, n, offs): the 128-bit loop, its three tail lengths, each buffer misaligned in turn, and a size that takes
    several grid-stride passes of both loops"""
    out = [("vec", n, {})] + [("tail%d" % r, n + r, {}) for r in (1, 2, 3)]
    out += [("mis_%s%d" % (key, 1 + i % 3), n + 1, {key: 1 + i % 3}) for i, key in enumerate(buffers)]
    return out + [("large", (1 << 21) + 3, {})]


RMS = [(m, pid, n, offs) for m in (0.0, 0.9)
       for pid, n, offs in paths(["p", "g", "square_avg"] + (["momentum_buffer"] if m else []))]


@pytest.mark.parametrize("momentum,path,n,offs", RMS, ids=["mom%g-%s" % (c[0], c[1]) for c in RMS])
def test_clip_rmsprop(momentum, path, n, offs):
    """tb_clip_rmsprop_step_f32, the reference's RMSprop; with momentum it runs the scalar loop over every element"""
    o = dict(alpha=0.99, eps=1e-4, momentum=momentum)
    rejected = chain("rmsprop", o, n, offs, seed=n + len(path))
    assert "unclipped gradient" in rejected and (not momentum or "momentum buffer not decayed" in rejected)


EX_OPTS = [(c, m, wd) for c in (False, True) for m in (0.0, 0.9) for wd in (0.0, 0.05)]
EX = [(c, m, wd, pid, n, offs) for c, m, wd in EX_OPTS
      for pid, n, offs in paths(["p", "g", "square_avg"] + (["grad_avg"] if c else []) +
                                (["momentum_buffer"] if m else []))
      if pid in ("vec", "tail3") or pid.startswith("mis_") or (pid == "large" and c and m and wd)]


@pytest.mark.parametrize("centered,momentum,wd,path,n,offs", EX,
                         ids=["c%d_mom%g_wd%g-%s" % (c[0], c[1], c[2], c[3]) for c in EX])
def test_clip_rmsprop_ex(centered, momentum, wd, path, n, offs):
    o = dict(alpha=0.99, eps=1e-4, momentum=momentum, wd=wd, centered=centered)
    chain("rmsprop_ex", o, n, offs, seed=n + 3 * centered + 5 * (momentum > 0))


ADAM_OPTS = [(d, wd, b1, b2) for d in (False, True) for wd in (0.0, 0.05)
             for b1, b2 in ((0.9, 0.999), (0.0, 0.999), (0.9, 0.0))]


@pytest.mark.parametrize("decoupled,wd,beta1,beta2", ADAM_OPTS,
                         ids=["%s_wd%g_b%g,%g" % ("adamw" if c[0] else "adam", c[1], c[2], c[3]) for c in ADAM_OPTS])
def test_clip_adam_options(decoupled, wd, beta1, beta2):
    """Adam / AdamW, L2 or decoupled decay, beta1 = 0 and beta2 = 0 as edges; from step 9, where the bias corrections
    still move the step"""
    o = dict(beta1=beta1, beta2=beta2, eps=1e-6, wd=wd, decoupled=decoupled)
    chain("adam", o, 4099, step0=9, seed=int(10 * wd) + 2 * decoupled)


@pytest.mark.parametrize("step0", [0, 1, 9, 10 ** 6])
def test_clip_adam_step_counter(step0):
    """t = step_device + 1 in the bias corrections, and the counter advances by exactly one per call; at 10^6 the
    corrections are 1 and only the clip can be told apart"""
    o = dict(beta1=0.9, beta2=0.999, eps=1e-6, wd=0.0, decoupled=False)
    rejected = chain("adam", o, 4097, step0=step0, seed=step0 % 1000)
    assert ("bias corrections at t - 1" in rejected) == (step0 < 100)


ADAM_PATHS = paths(["p", "g", "exp_avg", "exp_avg_sq"])


@pytest.mark.parametrize("path,n,offs", ADAM_PATHS, ids=[c[0] for c in ADAM_PATHS])
def test_clip_adam_paths(path, n, offs):
    o = dict(beta1=0.9, beta2=0.999, eps=1e-6, wd=0.05, decoupled=True)
    chain("adam", o, n, offs, step0=1, seed=n)


ZERO = [("rmsprop", dict(alpha=0.99, eps=1e-4, momentum=0.9)),
        ("rmsprop_ex", dict(alpha=0.99, eps=1e-4, momentum=0.9, wd=0.05, centered=True))] + \
       [("adam", dict(beta1=0.9, beta2=0.999, eps=1e-6, wd=0.05, decoupled=True, step0=s)) for s in (0, 1, 9, 10 ** 6)]


@pytest.mark.parametrize("kind,o", ZERO, ids=["rmsprop", "rmsprop_ex"] + ["adam_step%d" % c[1]["step0"] for c in ZERO[2:]])
def test_empty_buffer(kind, o):
    """n = 0: the RMSprop steps return before any launch; Adam still counts the step and reports the norm.  Nothing
    else is written."""
    step0 = o.get("step0", 0)
    b = {k: Slab(np.zeros(0, np.float32)) for k in ["p", "g"] + state_keys(kind, o)}
    step_dev = scalar(step0, torch.int64) if kind == "adam" else None
    norm_out = Slab(np.full(1, np.nan, np.float32))
    sumsq_t = Slab(np.full(1, 2500.0, np.float32))
    launch(kind, o, b, 0, sumsq_t.t, MAX_NORM, None, step_dev, norm_out.t)
    sync()
    assert all(slab.sentinels_intact() for slab in b.values()) and sumsq_t.sentinels_intact()
    if kind == "adam":
        assert int(step_dev[0]) == step0 + 1
        assert same_bits(norm_out.get(), [50.0])
    else:
        assert norm_out.sentinels_intact() and np.isnan(norm_out.get()).all()


# ---------------------------------------------------------------------------------------------------------------------
# non-finite gradients, against torch
# ---------------------------------------------------------------------------------------------------------------------
NF_OPTS = {
    "rmsprop": ("rmsprop", dict(alpha=0.99, eps=1e-4, momentum=0.0)),
    "rmsprop_momentum": ("rmsprop", dict(alpha=0.99, eps=1e-4, momentum=0.9)),
    "rmsprop_ex": ("rmsprop_ex", dict(alpha=0.99, eps=1e-4, momentum=0.9, wd=0.05, centered=True)),
    "adam": ("adam", dict(beta1=0.9, beta2=0.999, eps=1e-6, wd=0.05, decoupled=False)),
    "adamw": ("adam", dict(beta1=0.9, beta2=0.999, eps=1e-6, wd=0.05, decoupled=True)),
}
NF = [(name, bad, path) for name in NF_OPTS for bad in ("nan", "inf", "-inf") for path in ("vector", "scalar")]


def torch_step(kind, o, s, g, step0):
    """clip_grad_norm_(MAX_NORM) + the torch optimizer, float64 on the CPU, from the float32 state s"""
    p = torch.nn.Parameter(torch.from_numpy(s["p"].astype(np.float64)))
    if kind == "adam":
        cls = torch.optim.AdamW if o["decoupled"] else torch.optim.Adam
        opt = cls([p], lr=f32(LR), betas=(o["beta1"], o["beta2"]), eps=f32(o["eps"]), weight_decay=f32(o["wd"]),
                  foreach=False)
    else:
        opt = torch.optim.RMSprop([p], lr=f32(LR), alpha=f32(o["alpha"]), eps=f32(o["eps"]),
                                  weight_decay=f32(o.get("wd", 0.0)), momentum=f32(o["momentum"]),
                                  centered=o.get("centered", False), foreach=False)
    opt.state[p].update({k: torch.from_numpy(s[k].astype(np.float64)) for k in state_keys(kind, o)},
                        step=torch.tensor(float(step0)))
    p.grad = torch.from_numpy(g.astype(np.float64))
    torch.nn.utils.clip_grad_norm_([p], MAX_NORM)
    opt.step()
    out = {k: opt.state[p][k].numpy() for k in state_keys(kind, o)}
    out.update(p=p.detach().numpy(), g=p.grad.numpy())
    return out


@pytest.mark.parametrize("name,bad,path", NF, ids=["%s-%s-%s" % c for c in NF])
def test_nonfinite_gradient_matches_torch(name, bad, path):
    """one NaN or +-inf gradient element at n = 4097.  torch's clip_grad_norm_ makes the norm NaN / inf and its clamp
    keeps a NaN coefficient, so one NaN poisons the whole step, while inf gives coefficient 0 and NaN (inf * 0) at its
    own element only.  The kernels must put NaN exactly where torch does and meet the bound elsewhere.  The scalar path:
    the parameter buffer misaligned."""
    kind, o = NF_OPTS[name]
    n, step0 = 4097, 3
    rs = np.random.RandomState(17)
    init = initial_state(kind, o, n, rs, step0)
    g = (rs.randn(n) * (NORMS["above"] / np.sqrt(n))).astype(np.float32)
    g[1234] = np.float32(bad)
    b = {k: Slab(v, 2 if (k == "p" and path == "scalar") else 0) for k, v in init.items()}
    b["g"] = Slab(g)
    # the norm as the learner forms it: tb_grad_sumsq_f32 of the same gradient
    sumsq_t = Slab(np.full(1, -1.0, np.float32))
    call("tb_grad_sumsq_f32", P(b["g"].t), n, P(sumsq_t.t), P(workspace()), stream())
    step_dev = scalar(step0, torch.int64) if kind == "adam" else None
    norm_out = Slab(np.full(1, -1.0, np.float32))
    s = {key: slab.get() for key, slab in b.items()}
    launch(kind, o, b, n, sumsq_t.t, MAX_NORM, None, step_dev, norm_out.t)
    sync()
    norm = norm_out.get()[0]
    assert np.isnan(norm) if bad == "nan" else norm == np.inf
    got = {key: slab.get() for key, slab in b.items()}
    ref = torch_step(kind, o, s, g, step0)
    for key in ["g", "p"] + state_keys(kind, o):
        assert np.array_equal(np.isnan(got[key]), np.isnan(ref[key])), \
            "%s: NaN at %d elements, torch at %d" % (key, np.isnan(got[key]).sum(), np.isnan(ref[key]).sum())
    coef = O.clip_coef(norm, MAX_NORM)
    _, mag = oracle(kind, o, s, coef, step0 + 1)
    finite = ~np.isnan(ref["p"])
    if finite.any():
        for key in ["p"] + state_keys(kind, o):
            assert np.array_equal(np.isfinite(got[key]), np.isfinite(ref[key])), key
        sel = {k: v[finite] for k, v in got.items()}
        r = worst(sel, {k: v[finite] for k, v in ref.items()}, {k: v[finite] for k, v in mag.items()}, s["p"][finite],
                  state_keys(kind, o))
        assert r <= 1.0, "%.3g of the bound" % r
        unclipped = oracle(kind, o, s, 1.0, step0 + 1)[0]
        assert worst({k: v[finite] for k, v in unclipped.items()}, {k: v[finite] for k, v in ref.items()},
                     {k: v[finite] for k, v in mag.items()}, s["p"][finite], state_keys(kind, o)) > 1.0, \
            "the bound cannot see the unclipped gradient"
    assert all(slab.sentinels_intact() for slab in b.values())
