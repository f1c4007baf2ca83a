"""GPU: the kernels of csrc/vtrace.cu in isolation, through the C entry points - the V-trace scan, action_log_probs,
the fused IMPALA loss with every feature group, UPGO, kickstarting and the three stand-alone losses.

- Layouts: the launch rules (pick_warps, pick_grid, kWideWarps, pick_cluster) are restated below from the device's SM
  count, every case is named by the layout it takes (wide; split-T with W warps, trailing warps empty or not; the
  cluster scan with C CTAs), and a profiler trace checks once that each launch runs the kernel instantiation the rules
  and TB_DISPATCH_A choose.
- Values: the scan, action_log_probs, the plain fused loss and the stand-alone losses against the float64 restatement
  of tests/loss_oracle.py, every element within its error bound (BOUND_C u mag; u of the kernel's type), and each bound
  shown to reject the restatement with a plausible mistake by at least ten times.  The other launch sites (weights,
  trust region, PopArt, UPGO, kickstarting) at every row width against their own oracles at those oracles' tolerances.
- Contract clauses: bit-identities (a NaN, negative or +inf clip is no clip, discounts in place of done, forward only,
  zero_tail, run to run), the early return of empty sizes, and memory hygiene: every output between guard bytes that
  must come back untouched and prefilled with 0xFF bytes (NaN) so that an element left unwritten shows, and a private
  workspace whose per-CTA partials are NaN giving the bits of a clean one, with its ticket counter back at 0."""
import math
import re

import numpy as np
import pytest
import torch

from tests import kickstart_oracle as KO
from tests import loss_oracle as LO
from tests import trust_region_oracle as TO
from tests import upgo_oracle as UO

pytestmark = pytest.mark.gpu

INSTANTIATED = [2, 3, 4, 5, 6, 7, 8, 9, 10, 12, 14, 16, 18]   # TB_DISPATCH_A's cases; any other A runs kA = 0
LOSS_AS = INSTANTIATED + [1, 11, 13, 17, 19, 256]
ALP_AS = INSTANTIATED + [1, 11, 19, 300]
GUARD = 64                    # guard bytes before and after every buffer
MAX_PARTIAL_CTAS = 4096       # kMaxPartialCtas
LAYOUTS = {"wide": (4, 40), "split": (37, 5)}   # the loss's two layouts at the A sweep's shapes
COSTS = dict(baseline_cost=0.5, entropy_cost=0.01)


# ---- launch rules (csrc/vtrace.cu), restated ------------------------------------------------------------------------
def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pick_warps(T, tiles):
    w = sm_count() * 16 // max(tiles, 1)
    return max(1, min(w, min((T + 3) // 4, 16)))


def pick_cluster(T, tiles, W):
    if W < 16 or tiles * 16 > sm_count() * 2:
        return 0
    c = 8
    while c > 1 and (T < 16 * c * 4 or -(-T // (16 * c)) > 8):
        c >>= 1
    if c > 1 and -(-T // (16 * c)) > 8:
        return 0
    return c if c > 1 else 0


def layout(T, B, scan=False):
    """'wide', 'split_W<W>' (with '_empty' when trailing warps get no time steps) or 'cluster_C<C>'"""
    tiles = -(-B // 32)
    W = pick_warps(T, tiles)
    if W == 1:
        return "wide"
    if scan and pick_cluster(T, tiles, W):
        return "cluster_C%d" % pick_cluster(T, tiles, W)
    chunk = -(-T // W)
    return "split_W%d" % W + ("_empty" if (W - 1) * chunk >= T else "")


def loss_grid(T, B):
    tiles = -(-B // 32)
    if pick_warps(T, tiles) == 1:
        return min(-(-tiles // 8), MAX_PARTIAL_CTAS)   # kWideWarps = 8 column tiles per CTA
    return max(1, min(sm_count() * 8, MAX_PARTIAL_CTAS, tiles))


# the scan's cases on a 132-SM H100, by the layout they take: T around 4/5, 127/128, 255/256, 511/512, 1024/1025 and B
# around 512/513 (16 / 17 column tiles, where the cluster rule stops)
SCAN_CASES = {
    "wide_T4": (4, 100), "wide_B34000": (6, 34000),
    "split_W2_T5": (5, 40), "split_W2_B30000": (12, 30000),
    "split_W8_empty": (33, 8000), "split_W16_empty": (65, 40), "split_W16_T127": (127, 64),
    "cluster_C2_T128": (128, 64), "cluster_C2_T255": (255, 64), "cluster_C4_T256": (256, 64),
    "cluster_C4_T511": (511, 64), "cluster_C8_T512": (512, 64), "cluster_C8_T1024": (1024, 64),
    "split_W16_T1025": (1025, 64), "cluster_C8_B512": (600, 512), "split_W16_B513": (600, 513),
}


def _expected_layout(name):
    return re.sub(r"_(T|B)\d+$", "", name)


def on_h100_sxm():
    return sm_count() == 132


# ---- C calls and guarded buffers --------------------------------------------------------------------------------------
def lib():
    from torchbeast_b200 import _lib
    return _lib.lib()


_ARGS = []   # the tensors of the call being assembled: a temporary must outlive the pointer taken from it


def P(x):
    """the device pointer of a Buf (never NULL, also when empty) or a tensor"""
    import ctypes
    if isinstance(x, Buf):
        return ctypes.c_void_p(x.raw.data_ptr() + GUARD)
    _ARGS.append(x)
    return ctypes.c_void_p(x.data_ptr())


def stream():
    return torch.cuda.current_stream().cuda_stream


def call(name, *args):
    rc = getattr(lib(), name)(*args)
    _ARGS.clear()   # freed blocks are reused in stream order, after the launch
    assert rc == 0, "%s: %s" % (name, lib().tb_last_error().decode())


class Buf:
    """n elements of dtype between GUARD guard bytes, prefilled with 0xFF bytes (NaN) or with `values`"""

    def __init__(self, n, dtype=torch.float32, values=None):
        nb = n * torch.empty(0, dtype=dtype).element_size()
        self.nb = nb
        self.raw = torch.randint(0, 256, (GUARD + nb + GUARD,), dtype=torch.uint8, device="cuda")
        self.raw[GUARD:GUARD + nb] = 255
        self.t = self.raw[GUARD:GUARD + nb].view(dtype)
        if values is not None:
            self.t.copy_(torch.from_numpy(np.ascontiguousarray(values)).reshape(-1))
        self.init = self.raw.clone()

    def get(self):
        return self.t.cpu().numpy()

    def guards_intact(self):
        g = GUARD + self.nb
        return torch.equal(self.raw[:GUARD], self.init[:GUARD]) and torch.equal(self.raw[g:], self.init[g:])


def dev(x, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    return t if dtype is None else t.to(dtype)


def workspace(stale=True):
    """ticket counter 0; with `stale` the per-CTA partials are NaN (every CTA must write its own before the fold)"""
    ws = torch.zeros(lib().tb_workspace_bytes(), dtype=torch.uint8, device="cuda")
    if stale:
        ws[64:].view(torch.float64).fill_(float("nan"))
    return ws


def counter(ws):
    return int(ws[:4].view(torch.int32)[0])


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    iv = np.int64 if a.dtype == np.float64 else np.int32
    return np.array_equal(a.view(iv), b.view(iv)) if a.dtype.kind == "f" else np.array_equal(a, b)


def within(got, want, mag, u, what):
    err = np.abs(np.asarray(got, np.float64) - want)
    tol = LO.bound(mag, u)
    bad = ~(err <= tol)
    assert not bad.any(), "%s: %d elements outside the bound, worst %.3g of it" % (
        what, int(bad.sum()), float(np.nanmax(np.where(np.isfinite(err), err / (tol + 1e-300), np.inf))))


def ratio(got, want, mag, u):
    err = np.abs(np.asarray(got, np.float64) - want)
    return float((err / (LO.bound(mag, u) + 1e-300)).max(initial=0.0))


# ---- inputs -------------------------------------------------------------------------------------------------------------
def _q(rs, shape, lim=2.0):
    """multiples of 1/16: UPGO's trace switch r + g V' >= V is then exact in float32 and float64 alike"""
    return (np.round(rs.uniform(-lim, lim, size=shape) * 16) / 16).astype(np.float32)


def loss_inputs(T, B, A, seed, masked=True, quantised=False):
    """Logits with TB_MASKED_LOGIT entries at the same places in both policies, never at the taken action; rewards
    beyond [-1, 1] for the reward clip; done in about one step of ten."""
    rs = np.random.RandomState(seed)
    tl = (1.5 * rs.randn(T, B, A)).astype(np.float32)
    bl = (tl + 0.7 * rs.randn(T, B, A)).astype(np.float32)
    a = rs.randint(0, A, size=(T, B))
    if masked and A > 1:
        m = (rs.rand(T, B, A) < 0.2) & (np.arange(A) != a[..., None])
        tl[m] = bl[m] = LO.MASKED_LOGIT
    x = dict(bl=bl, tl=tl, a=a, done=rs.rand(T, B) < 0.1)
    if quantised:
        x.update(r=_q(rs, (T, B)), v=_q(rs, (T, B)), bs=_q(rs, (B,)))
    else:
        x.update(r=(2 * rs.randn(T, B)).astype(np.float32), v=rs.randn(T, B).astype(np.float32),
                 bs=rs.randn(B).astype(np.float32))
    return x


class Loss:
    """One tb_impala_loss_f32 call; every output a guarded Buf.  features: weights [B], beta (trust region), popart
    (identity statistics, K = 1: the plain loss on a PopArt head)."""

    def __init__(self, x, gamma=0.99, clip_rho=1.0, clip_pg=1.0, clip_rewards=1, grads=True, zero_tail=1,
                 discounts=False, weights=None, beta=None, popart=False, ws=None, costs=COSTS):
        T, B, A = x["tl"].shape
        self.T, self.B, self.A, self.x = T, B, A, x
        self.ws = workspace() if ws is None else ws
        N, R = T * B, (T + zero_tail) * B
        self.out = {k: Buf(N) for k in ("vs", "pg_adv", "log_rhos", "behavior_alp", "target_alp")}
        self.out["losses"] = Buf(4)
        if grads:
            self.out["grad_logits"], self.out["grad_values"] = Buf(R * A), Buf(R)
        if beta is not None:
            self.out["kl"], self.out["trust_out"] = Buf(N), Buf(2)
            self.beta = dev(np.array([beta], np.float32))
        if popart:
            self.out["task_sums"] = Buf(3, torch.float64)
        o = lambda k: P(self.out[k]) if k in self.out else None  # noqa: E731
        self.inp = dict(bl=dev(x["bl"]), tl=dev(x["tl"]), a=dev(x["a"].astype(np.int64)), r=dev(x["r"]),
                        done=dev(x["done"].astype(np.uint8)), v=dev(x["v"]), bs=dev(x["bs"]))
        i = self.inp
        if discounts:
            i["disc"] = dev(np.where(x["done"], 0.0, np.float32(gamma)).astype(np.float32))
        values, task, mu, nu = i["v"], None, None, None
        if popart:
            values = dev(np.concatenate([x["v"], x["bs"][None]], 0)[..., None])
            task, mu, nu = dev(np.zeros((T + 1, B), np.int64)), dev(np.zeros(1)), dev(np.ones(1))
        self.values = values
        cw = None if weights is None else dev(np.asarray(weights, np.float32))
        self.cw = cw
        c = lambda v: -1.0 if v is None else float(v)  # noqa: E731
        call("tb_impala_loss_f32", P(i["bl"]), P(i["tl"]), P(i["a"]), P(i["r"]),
             None if discounts else P(i["done"]), P(i["disc"]) if discounts else None, P(values), P(i["bs"]),
             T, B, A, gamma, costs["baseline_cost"], costs["entropy_cost"], clip_rewards, c(clip_rho), c(clip_pg),
             None, P(cw) if cw is not None else None, P(task) if popart else None, P(mu) if popart else None,
             P(nu) if popart else None, 1 if popart else 0, o("task_sums"),
             P(self.beta) if beta is not None else None, o("kl"), o("trust_out"), o("vs"), o("pg_adv"), o("log_rhos"),
             o("behavior_alp"), o("target_alp"), o("losses"), o("grad_logits"), o("grad_values"), zero_tail,
             P(self.ws), stream())
        self.task, self.mu, self.nu, self.gamma, self.clip_pg, self.clip_rewards = task, mu, nu, gamma, clip_pg, clip_rewards

    def host(self):
        torch.cuda.synchronize()
        assert counter(self.ws) == 0, "the ticket counter was not reset"
        for k, b in self.out.items():
            assert b.guards_intact(), "a write outside %s" % k
        T, B, A = self.T, self.B, self.A
        h = {k: b.get() for k, b in self.out.items()}
        for k in ("vs", "pg_adv", "log_rhos", "behavior_alp", "target_alp", "kl"):
            if k in h:
                h[k] = h[k].reshape(T, B)
        if "grad_logits" in h and B > 0:
            h["grad_logits"] = h["grad_logits"].reshape(-1, B, A)
            h["grad_values"] = h["grad_values"].reshape(-1, B)
        return h


def oracle(x, **kw):
    return LO.impala_loss(x["bl"], x["tl"], x["a"], x["r"], x["v"], x["bs"], done=x["done"], **kw)


def check_loss(h, o, T, what=""):
    """every output of the plain loss within its bound, nothing left unwritten"""
    for k in ("vs", "pg_adv", "log_rhos", "behavior_alp", "target_alp", "losses"):
        assert np.all(np.isfinite(h[k])), "%s%s: unwritten or not finite" % (what, k)
        within(h[k], o[k], o["mag_" + k], LO.U32, what + k)
    if "grad_logits" in h:
        within(h["grad_logits"][:T], o["grad_logits"], o["mag_grad_logits"], LO.U32, what + "grad_logits")
        within(h["grad_values"][:T], o["grad_values"], o["mag_grad_values"], LO.U32, what + "grad_values")


def alp_call(logits, actions, dtype=torch.float32):
    N, A = logits.shape
    out = Buf(N, dtype)
    call("tb_action_log_probs_f32" if dtype == torch.float32 else "tb_action_log_probs_f64",
         P(dev(logits, dtype)), P(dev(actions.astype(np.int64))), N, A, P(out), stream())
    torch.cuda.synchronize()
    assert out.guards_intact()
    return out.get()


# ---- layouts and kernel names ---------------------------------------------------------------------------------------
def test_cases_take_the_layouts_they_are_named_for():
    if not on_h100_sxm():
        pytest.skip("the case table is laid out for 132 SMs; this device has %d" % sm_count())
    for name, (T, B) in SCAN_CASES.items():
        assert layout(T, B, scan=True) == _expected_layout(name), (name, layout(T, B, scan=True))
    assert layout(*LAYOUTS["wide"]) == "wide" and layout(*LAYOUTS["split"]).startswith("split_W")


def _kernel_sites(A):
    """(label, launch function, expected kernel names) of every TB_DISPATCH_A launch site at row width A"""
    kA = A if A in INSTANTIATED else 0
    x = loss_inputs(5, 3, A, A, masked=False, quantised=True)
    w = np.linspace(0.5, 1.5, 3)
    sites = []
    for pop, wt, tr in ((False, False, False), (False, True, False), (False, False, True), (False, True, True),
                        (True, False, False), (True, False, True)):
        flags = "%s, %s, %s, false" % tuple("true" if f else "false" for f in (pop, wt, tr))
        names = ["impala_loss_kernel<%d, %s>" % (kA, flags)] + (["popart_task_sums_kernel"] if pop else [])
        kw = dict(weights=w if wt else None, beta=0.3 if tr else None, popart=pop)
        sites.append(("loss" + str((pop, wt, tr)), lambda kw=kw: Loss(x, **kw), names))
        uflags = "%s, %s, %s" % tuple("true" if f else "false" for f in (pop, wt, tr))
        sites.append(("upgo" + str((pop, wt, tr)), lambda kw=kw: upgo(Loss(x, **kw), 0.5, launch_only=True),
                      names + ["upgo_loss_kernel<%d, %s>" % (kA, uflags)]))
    for wt in (False, True):
        sites.append(("kickstart", lambda wt=wt: kickstart(x["tl"], x["bl"], 0.5, w if wt else None, launch_only=True),
                      ["kickstart_loss_kernel<%d, %s>" % (kA, "true" if wt else "false")]))
    for dt, tn in ((torch.float32, "float"), (torch.float64, "double")):
        sites.append(("alp", lambda dt=dt: alp_call(x["tl"].reshape(-1, A), x["a"].reshape(-1), dt),
                      ["action_log_probs_kernel<%s, %d>" % (tn, kA)]))
    return sites


KNOWN = ("impala_loss_kernel", "popart_task_sums_kernel", "upgo_loss_kernel", "kickstart_loss_kernel",
         "action_log_probs_kernel", "vtrace_scan_kernel", "vtrace_scan_cluster_kernel")


def _short(name):
    """'void tb::impala_loss_kernel<7, false, false, false, false>(tb::LossArgs)' -> 'impala_loss_kernel<7, ...>'"""
    m = re.search(r"tb::(\w+)(<[^()]*>)?\(", name)
    if not m or m.group(1) not in KNOWN:
        return None
    return m.group(1) + re.sub(r"\s+", " ", m.group(2) or "").replace("(bool)0", "false").replace("(bool)1", "true")


def test_every_launch_runs_the_expected_kernel():
    """One profiled pass over every TB_DISPATCH_A site at every instantiated A and at 11 (kA = 0), and the scan at
    every layout case in float32 and float64: the kernels that ran, in order, are the ones the rules choose."""
    from torch.profiler import ProfilerActivity, profile
    plan = []
    for A in INSTANTIATED + [11]:
        plan += _kernel_sites(A)
    for name, (T, B) in SCAN_CASES.items():
        lay = layout(T, B, scan=True)
        for dt, tn in ((torch.float32, "float"), (torch.float64, "double")):
            kern = "vtrace_scan_cluster_kernel" if lay.startswith("cluster") else "vtrace_scan_kernel"
            plan.append((name, lambda T=T, B=B, dt=dt: scan_call(scan_inputs(T, B, 1), dt, (1.0, 1.0),
                                                                 launch_only=True), ["%s<%s, 8>" % (kern, tn)]))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _, fn, _ in plan:
            fn()
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    if not kernels:
        pytest.skip("the profiler recorded no CUDA kernel activity on this machine")
    got = [s for s in (_short(e.name) for e in sorted(kernels, key=lambda e: e.time_range.start)) if s]
    want = [n for _, _, names in plan for n in names]
    assert len(got) == len(want), (len(got), len(want))
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, "launch %d: ran %s, expected %s" % (i, g, w)


# ---- the scan ---------------------------------------------------------------------------------------------------------
def scan_inputs(T, B, seed):
    rs = np.random.RandomState(seed)
    return dict(lr=(0.8 * rs.randn(T, B)).astype(np.float32),
                g=(np.float32(0.99) * (rs.rand(T, B) > 0.05)).astype(np.float32),
                r=rs.randn(T, B).astype(np.float32), v=rs.randn(T, B).astype(np.float32),
                bs=rs.randn(B).astype(np.float32))


def scan_call(s, dtype, clips, launch_only=False):
    T, B = s["v"].shape
    vs, pg = Buf(T * B, dtype), Buf(T * B, dtype)
    c = [-1.0 if x is None else x for x in clips]
    call("tb_vtrace_from_importance_weights_f32" if dtype == torch.float32 else "tb_vtrace_from_importance_weights_f64",
         *[P(dev(s[k], dtype)) for k in ("lr", "g", "r", "v", "bs")], T, B, c[0], c[1], P(vs), P(pg), stream())
    if launch_only:
        return None
    torch.cuda.synchronize()
    assert vs.guards_intact() and pg.guards_intact()
    return vs.get().reshape(T, B), pg.get().reshape(T, B)


SCAN_CLIPS = [(1.0, 1.0), (None, None), (0.5, 3.75)]


@pytest.mark.parametrize("clips", SCAN_CLIPS, ids=["clip%s,%s" % c for c in SCAN_CLIPS])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", sorted(SCAN_CASES))
def test_scan_within_bound(case, dtype, clips):
    T, B = SCAN_CASES[case]
    s = scan_inputs(T, B, T * 7 + B)
    vs, pg = scan_call(s, dtype, clips)
    assert np.all(np.isfinite(vs)) and np.all(np.isfinite(pg)), "an element was left unwritten"
    o = LO.scan(s["lr"], s["g"], s["r"], s["v"], s["bs"], *clips)
    u = LO.U32 if dtype == torch.float32 else LO.U64
    within(vs, o["vs"], o["mag_vs"], u, "vs")
    within(pg, o["pg_adv"], o["mag_pg"], u, "pg_adv")
    if clips == (0.5, 3.75):   # c-bar clipped at clip_rho instead of 1: ten times outside the bound at least
        wrong = LO.scan(s["lr"], s["g"], s["r"], s["v"], s["bs"], *clips, mistake="cbar_clip_rho")
        assert ratio(wrong["vs"], o["vs"], o["mag_vs"], u) >= 10


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("case", ["wide_T4", "split_W16_empty", "cluster_C2_T128", "cluster_C8_T512"])
def test_scan_bit_identities(case, dtype):
    """a NaN, negative or +inf threshold is no clip; two runs give the same bits"""
    T, B = SCAN_CASES[case]
    s = scan_inputs(T, B, 3)
    ref = scan_call(s, dtype, (None, None))
    for c in (math.nan, -1.0, -5.0, math.inf):
        got = scan_call(s, dtype, (c, c))
        assert same_bits(got[0], ref[0]) and same_bits(got[1], ref[1]), c
    again = scan_call(s, dtype, (None, None))
    assert same_bits(again[0], ref[0]) and same_bits(again[1], ref[1])


def test_scan_empty_sizes_write_nothing():
    for T, B in ((0, 5), (5, 0), (0, 0)):
        vs, pg = Buf(8), Buf(8)
        z = dev(np.zeros(8, np.float32))
        call("tb_vtrace_from_importance_weights_f32", P(z), P(z), P(z), P(z), P(z), T, B, 1.0, 1.0, P(vs), P(pg),
             stream())
        torch.cuda.synchronize()
        assert vs.guards_intact() and pg.guards_intact() and np.isnan(vs.get()).all() and np.isnan(pg.get()).all()


# ---- action_log_probs --------------------------------------------------------------------------------------------------
def alp_rows(N, A, seed):
    """randn rows, every fifth shifted by +1e4 and every seventh by -1e4, every ninth all equal"""
    rs = np.random.RandomState(seed)
    x = (3 * rs.randn(N, A)).astype(np.float32)
    x[::5] += np.float32(1e4)
    x[3::7] -= np.float32(1e4)
    x[1::9] = np.float32(0.375)
    return x, rs.randint(0, A, size=N)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("A", ALP_AS)
def test_action_log_probs_within_bound(A, dtype):
    x, a = alp_rows(1000, A, A)
    got = alp_call(x, a, dtype)
    want, mag = LO.action_log_probs(x, a)
    within(got, want, mag, LO.U32 if dtype == torch.float32 else LO.U64, "alp")
    if A == 1:
        assert not got.any()


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("A", [1, 6, 19])
def test_action_log_probs_across_the_grid_cap(A, dtype):
    """one row past 8 * SMs CTAs of 256 rows: the grid-stride loop takes a second pass"""
    N = sm_count() * 8 * 256 + 1
    x, a = alp_rows(N, A, 5)
    got = alp_call(x, a, dtype)
    want, mag = LO.action_log_probs(x, a)
    within(got, want, mag, LO.U32 if dtype == torch.float32 else LO.U64, "alp")


# ---- the plain fused loss -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lay", sorted(LAYOUTS))
@pytest.mark.parametrize("A", LOSS_AS)
def test_fused_loss_within_bound(A, lay):
    T, B = LAYOUTS[lay]
    x = loss_inputs(T, B, A, 31 * A + T)
    L = Loss(x, clip_rho=2.0, clip_pg=0.5)
    h = L.host()
    o = oracle(x, clip_rho=2.0, clip_pg_rho=0.5, **COSTS)
    check_loss(h, o, T)
    assert not h["grad_logits"][T].any() and not h["grad_values"][T].any()
    # target_alp / behavior_alp are alp_row's bits, as tb_action_log_probs_f32 forms them on the same rows
    for k, lg in (("target_alp", "tl"), ("behavior_alp", "bl")):
        alone = alp_call(x[lg].reshape(-1, A), x["a"].reshape(-1))
        diff = np.abs(h[k].reshape(-1).view(np.int32).astype(np.int64) - alone.view(np.int32).astype(np.int64))
        assert not diff.any(), "%s differs from tb_action_log_probs_f32 by up to %d ulp" % (k, diff.max())


LOSS_LAYOUT_CASES = ["wide_T4", "wide_B34000", "split_W2_T5", "split_W8_empty", "split_W16_empty", "split_W16_T1025",
                     "split_W16_B513", "cluster_C8_B512"]


@pytest.mark.parametrize("case", LOSS_LAYOUT_CASES)
def test_fused_loss_layout_cases(case):
    """the scan's layout shapes through the loss (which has no cluster path: the cluster shapes split T over 16 warps)"""
    T, B = SCAN_CASES[case]
    x = loss_inputs(T, B, 6, T + B)
    h = Loss(x).host()
    check_loss(h, oracle(x, **COSTS), T)


MISTAKE_SHAPES = {"wide": (4, 19200), "split": (80, 960)}   # T * B = 76800 rows in both


@pytest.mark.parametrize("lay", sorted(MISTAKE_SHAPES))
def test_bounds_reject_plausible_mistakes(lay):
    """The kernel within the bound, and each mistake at least ten times outside it on some output: c-bar clipped at
    clip_rho, the pg advantage clipped with clip_rho, bootstrapped from V_{t+1}, the entropy gradient without -H and the
    baseline gradient off by 1/2.  clip_rho = 2 and clip_pg_rho = 0.5 differ."""
    T, B = MISTAKE_SHAPES[lay]
    assert layout(T, B).startswith(lay)
    x = loss_inputs(T, B, 6, 5, masked=False)
    kw = dict(clip_rho=2.0, clip_pg_rho=0.5, **COSTS)
    h = Loss(x, clip_rho=2.0, clip_pg=0.5).host()
    o = oracle(x, **kw)
    check_loss(h, o, T)
    keys = ("vs", "pg_adv", "grad_logits", "grad_values", "losses")
    for mistake in LO.MISTAKES[:-1]:
        wrong = oracle(x, mistake=mistake, **kw)
        r = max(ratio(wrong[k], o[k], o["mag_" + k], LO.U32) for k in keys)
        assert r >= 10, "%s is only %.3g times the bound" % (mistake, r)


def test_bound_rejects_float32_loss_sums():
    """The loss sums accumulated in float32 (row by row) instead of fp64, at 10^6 rows: the baseline loss, whose terms
    all have one sign, lands at least ten times outside its bound.  In the wide layout: over a long split unroll the
    magnitude of vs, and with it the baseline loss's bound, grows with the trace, and at 10^6 rows the float32 sum is
    only a few times outside it."""
    T, B = 4, 256000
    assert layout(T, B) == "wide"
    x = loss_inputs(T, B, 6, 5, masked=False)
    kw = dict(clip_rho=2.0, clip_pg_rho=0.5, **COSTS)
    h = Loss(x, clip_rho=2.0, clip_pg=0.5, grads=False).host()
    o = oracle(x, **kw)
    within(h["losses"], o["losses"], o["mag_losses"], LO.U32, "losses")
    wrong = oracle(x, mistake="fp32_sums", **kw)
    r = ratio(wrong["losses"], o["losses"], o["mag_losses"], LO.U32)
    assert r >= 10, "float32 loss sums are only %.3g times the bound" % r


# ---- bit identities and the contract's edges --------------------------------------------------------------------------
def _same(a, b, keys=None):
    for k, v in a.items():
        if keys is None or k in keys:
            assert same_bits(v, b[k]), k


@pytest.mark.parametrize("A", [6, 11])
@pytest.mark.parametrize("lay", sorted(LAYOUTS))
def test_fused_loss_bit_identities(lay, A):
    T, B = LAYOUTS[lay]
    x = loss_inputs(T, B, A, 77)
    ref = Loss(x, clip_rho=None, clip_pg=None).host()
    for c in (math.nan, -1.0, math.inf):     # NaN and negative mean None; +inf clips nothing
        _same(ref, Loss(x, clip_rho=c, clip_pg=c).host())
    base = Loss(x).host()
    _same(base, Loss(x).host())                                      # run to run
    _same(base, Loss(x, discounts=True).host())                      # discounts = where(done, 0, gamma)
    fwd = Loss(x, grads=False).host()                                # forward only
    _same(base, fwd, ("vs", "pg_adv", "log_rhos", "behavior_alp", "target_alp", "losses"))
    zt0 = Loss(x, zero_tail=0).host()                                # T rows of gradient, guards right after them
    assert zt0["grad_logits"].shape[0] == T
    _same({k: base[k][:T] for k in ("grad_logits", "grad_values")}, zt0)
    assert not base["grad_logits"][T].any() and not base["grad_values"][T].any()


def test_fused_loss_without_reward_clip():
    T, B = LAYOUTS["split"]
    x = loss_inputs(T, B, 6, 8)
    check_loss(Loss(x, clip_rewards=0).host(), oracle(x, clip_rewards=False, **COSTS), T)


@pytest.mark.parametrize("zero_tail", [0, 1])
@pytest.mark.parametrize("T,B", [(0, 5), (4, 0), (0, 0)])
def test_fused_loss_empty_sizes(T, B, zero_tail):
    """the early return: losses and trust_out zeroed, with zero_tail the B gradient rows zeroed, nothing else written"""
    A = 6
    x = loss_inputs(max(T, 1), max(B, 1), A, 1)
    x = {k: (v[:T, :B] if v.ndim >= 2 else v[:B]) for k, v in x.items()}
    L = Loss(x, beta=0.5, zero_tail=zero_tail)
    h = L.host()
    assert same_bits(h["losses"], np.zeros(4, np.float32)) and same_bits(h["trust_out"], np.zeros(2, np.float32))
    rows = B * zero_tail
    assert h["grad_logits"].size == rows * A and not h["grad_logits"].any() and not h["grad_values"].any()


# ---- every other launch site at every row width -------------------------------------------------------------------------
def upgo(L, cost, launch_only=False):
    """tb_upgo_loss_f32 after the loss call L, with L's features; returns host (upgo_adv, upgo_out)"""
    T, B, A = L.T, L.B, L.A
    adv, out = Buf(T * B), Buf(1)
    i = L.inp
    pop = L.task is not None
    call("tb_upgo_loss_f32", P(i["tl"]), P(i["a"]), P(i["r"]), P(i["done"]), None, P(L.values), P(i["bs"]), T, B, A,
         L.gamma, L.clip_rewards, -1.0 if L.clip_pg is None else L.clip_pg, None, P(L.cw) if L.cw is not None else None,
         P(L.task) if pop else None, P(L.mu) if pop else None, P(L.nu) if pop else None, 1 if pop else 0,
         P(L.out["log_rhos"]), P(L.beta) if "kl" in L.out else None, P(L.out["kl"]) if "kl" in L.out else None,
         P(dev(np.array([cost], np.float32))), P(adv), P(out), P(L.out["losses"]),
         P(L.out["grad_logits"]) if "grad_logits" in L.out else None, P(L.ws), stream())
    if launch_only:
        return None
    torch.cuda.synchronize()
    assert adv.guards_intact() and out.guards_intact() and counter(L.ws) == 0
    return adv.get().reshape(T, B), out.get()[0]


def kickstart(teacher, target, cost, weights=None, launch_only=False, ws=None, grad_rows=1):
    T, B, A = target.shape
    rs = np.random.RandomState(T + B)
    gl0, l0 = rs.randn((T + grad_rows) * B * A).astype(np.float32), rs.randn(4).astype(np.float32)
    gl, losses, out = Buf(gl0.size, values=gl0), Buf(4, values=l0), Buf(2)
    ws = workspace() if ws is None else ws
    call("tb_kickstart_loss_f32", P(dev(teacher)), P(dev(target)), T, B, A,
         P(dev(np.asarray(weights, np.float32))) if weights is not None else None,
         P(dev(np.array([cost], np.float32))), P(out), P(losses), P(gl), P(ws), stream())
    if launch_only:
        return None
    torch.cuda.synchronize()
    assert gl.guards_intact() and losses.guards_intact() and out.guards_intact() and counter(ws) == 0
    return dict(gl0=gl0.reshape(-1, B, A), gl=gl.get().reshape(-1, B, A), l0=l0, losses=losses.get(), out=out.get())


SITES = ["weighted", "trust", "weighted_trust", "popart", "popart_trust", "upgo", "upgo_weighted", "upgo_trust",
         "upgo_weighted_trust", "upgo_popart", "upgo_popart_trust", "kickstart", "kickstart_weighted"]


def _check_trust_oracle(h, o, T):
    """test_trust_region_gpu.py's tolerances"""
    for k in ("log_rhos", "behavior_alp", "target_alp"):
        np.testing.assert_allclose(h[k], o[k], rtol=1e-5, atol=1e-5, err_msg=k)
    np.testing.assert_allclose(h["vs"], o["vs"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(h["pg_adv"], o["pg_adv"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(h["losses"], o["losses"], rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(h["grad_logits"][:T], o["grad_logits"], rtol=1e-4, atol=1e-5)
    assert not h["grad_logits"][T].any()
    gv = h["grad_values"].reshape(T + 1, -1)
    np.testing.assert_allclose(gv[:T], o["grad_values"], rtol=1e-4, atol=1e-5)
    assert not gv[T].any()


@pytest.mark.parametrize("lay", sorted(LAYOUTS))
@pytest.mark.parametrize("A", LOSS_AS)
@pytest.mark.parametrize("site", SITES)
def test_launch_site_against_its_oracle(site, A, lay):
    T, B = LAYOUTS[lay]
    seed = 3 * A + T + len(site)
    if site.startswith("kickstart"):
        rs = np.random.RandomState(seed)
        teacher, target = (2 * rs.randn(T, B, A)).astype(np.float32), (2 * rs.randn(T, B, A)).astype(np.float32)
        w = rs.rand(B).astype(np.float32) if site.endswith("weighted") else None
        out = kickstart(teacher, target, 0.7, w)
        o = KO.loss(teacher, target, 0.7, weights=w)
        kl_scale, N = np.abs(o["kl"]).sum(), o["kl"].size
        assert abs(float(out["out"][1]) - o["kl_sum"]) <= 2e-5 * kl_scale + 2e-6 * N
        assert abs(float(out["out"][0]) - o["loss"]) <= 0.7 * (2e-5 * kl_scale + 2e-6 * N)
        added = out["gl"][:T].astype(np.float64) - out["gl0"][:T]
        np.testing.assert_allclose(added, o["grad_logits"], rtol=1e-4, atol=4e-6)
        assert same_bits(out["gl"][T:], out["gl0"][T:])
        assert same_bits(out["losses"][3], np.float32(np.float64(out["l0"][3]) + np.float64(out["out"][0])))
        assert same_bits(out["losses"][:3], out["l0"][:3])
        return
    gamma = 0.75
    x = loss_inputs(T, B, A, seed, masked=False, quantised=True)
    w = None
    if "weighted" in site:
        w = np.random.RandomState(seed).rand(B).astype(np.float32)
        w[1] = 0.0
    beta = None
    if "trust" in site:
        beta = float(np.float32(np.median(TO.policy_kl(x["bl"], x["tl"]))))
    L = Loss(x, gamma=gamma, weights=w, beta=beta, popart="popart" in site, costs=COSTS)
    h = L.host()
    r, g = np.clip(x["r"], -1, 1), np.where(x["done"], 0.0, gamma)
    mask = None
    if beta is not None:
        kl64 = TO.policy_kl(x["bl"], x["tl"])
        assert np.all(np.abs(h["kl"] - kl64) <= 1e-5 + 1e-4 * kl64)
        mask = h["kl"] <= np.float32(beta)
    o = TO.loss(x["bl"], x["tl"], x["a"], r, g, x["v"], x["bs"], mask=mask, weights=w, **COSTS)
    if beta is not None:
        assert h["trust_out"][0] == o["trusted"]
        np.testing.assert_allclose(h["trust_out"][1], o["kl_sum"], rtol=1e-4)
    _check_trust_oracle(h, o, T)
    if not site.startswith("upgo"):
        return
    cost = 1.3
    adv, up = upgo(L, cost)
    after = L.host()
    uo = UO.loss(x["tl"], x["a"], r, g, x["v"], x["bs"], h["log_rhos"], cost, mask=mask, weights=w)
    np.testing.assert_allclose(adv, uo["adv"], rtol=1e-4, atol=1e-4)
    lt = TO.log_softmax(np.asarray(x["tl"], np.float64))
    lpa = np.take_along_axis(lt, x["a"][..., None], -1)[..., 0]
    scale = cost * np.abs((1.0 if w is None else w[None, :]) * lpa * uo["adv"]).sum()
    assert abs(float(up) - uo["loss"]) <= 1e-5 * scale + 1e-6
    np.testing.assert_allclose(after["grad_logits"][:T] - h["grad_logits"][:T], uo["grad_logits"], rtol=1e-4,
                               atol=1e-5)
    assert same_bits(after["grad_logits"][T], h["grad_logits"][T])
    assert same_bits(after["losses"][:3], h["losses"][:3])
    assert same_bits(after["losses"][3], np.float32(np.float64(h["losses"][3]) + np.float64(up)))


# ---- workspace hygiene of every reducing kernel --------------------------------------------------------------------------
def _standalone(kind, dtype, N, A, grad, ws, seed=0):
    """one stand-alone loss call; returns host (out, grad or None, inputs)"""
    rs = np.random.RandomState(seed)
    npdt = np.float32 if dtype == torch.float32 else np.float64
    sfx = "_f32" if dtype == torch.float32 else "_f64"
    out = Buf(1, dtype)
    g = Buf(N if kind == "baseline" else N * A, dtype) if grad else None
    if kind == "baseline":
        adv = rs.randn(N).astype(npdt)
        call("tb_baseline_loss" + sfx, P(dev(adv)), N, P(out), P(g) if grad else None, P(ws), stream())
        inputs = dict(adv=adv)
    else:
        x, a = alp_rows(N, A, seed)
        x = x.astype(npdt)
        adv = rs.randn(N).astype(npdt)
        if kind == "entropy":
            call("tb_entropy_loss" + sfx, P(dev(x)), N, A, P(out), P(g) if grad else None, P(ws), stream())
        else:
            call("tb_pg_loss" + sfx, P(dev(x)), P(dev(a.astype(np.int64))), P(dev(adv)), N, A, P(out),
                 P(g) if grad else None, P(ws), stream())
        inputs = dict(x=x, a=a, adv=adv)
    torch.cuda.synchronize()
    assert out.guards_intact() and (g is None or g.guards_intact())
    assert counter(ws) == 0, "the ticket counter was not reset"
    return out.get()[0], (g.get() if grad else None), inputs


def _reducers():
    """(id, run(ws) -> dict of host outputs): every reducing kernel on a single-CTA and a multi-CTA grid"""
    out = []
    for name, (T, B) in (("1cta_split", (37, 5)), ("1cta_wide", (4, 200)), ("ncta_split", (37, 300)),
                         ("ncta_wide", (4, 3000))):
        x = loss_inputs(T, B, 6, T + B, quantised=True)
        out.append(("loss_" + name, T, B, lambda ws, x=x: Loss(x, ws=ws).host()))
        out.append(("loss_trust_" + name, T, B, lambda ws, x=x: Loss(x, beta=0.3, ws=ws).host()))

        def up(ws, x=x):
            L = Loss(x, ws=ws)
            adv, u = upgo(L, 0.9)
            return dict(L.host(), upgo_adv=adv, upgo_out=np.float32(u))
        out.append(("upgo_" + name, T, B, up))
    for name, (T, B) in (("1cta", (4, 50)), ("ncta", (37, 3000))):
        rs = np.random.RandomState(T)
        te, ta = rs.randn(T, B, 6).astype(np.float32), rs.randn(T, B, 6).astype(np.float32)
        out.append(("kickstart_" + name, T, B, lambda ws, te=te, ta=ta: kickstart(te, ta, 0.5, ws=ws)))
    for kind in ("baseline", "entropy", "pg"):
        for name, N in (("1cta", 200), ("ncta", 300000)):
            out.append(("%s_%s" % (kind, name), N, 1, lambda ws, kind=kind, N=N: dict(
                zip(("out", "grad"), _standalone(kind, torch.float32, N, 6, True, ws)[:2]))))
    return out


REDUCERS = _reducers()


@pytest.mark.parametrize("idx", range(len(REDUCERS)), ids=[r[0] for r in REDUCERS])
def test_stale_workspace_gives_the_bits_of_a_clean_one(idx):
    rid, T, B, run = REDUCERS[idx]
    if rid.startswith(("loss", "upgo")):
        grid = loss_grid(T, B)
        assert (grid == 1) == ("1cta" in rid), (rid, grid)
    clean = run(workspace(stale=False))
    stale_ws = workspace(stale=True)
    stale = run(stale_ws)
    again = run(stale_ws)                    # reused: the counter the previous call left must be 0
    for k, v in clean.items():
        assert same_bits(v, stale[k]) and same_bits(v, again[k]), (rid, k)


# ---- the stand-alone losses ---------------------------------------------------------------------------------------------
def _standalone_cases():
    ns = [0, 1, 255, 256, 257, "cap+1", 10 ** 6]   # cap + 1: one row past reduce_grid's 4 * SMs CTAs of 256
    cases = [("baseline", n, 1) for n in ns]
    for kind in ("entropy", "pg"):
        for n in ns:
            for A in (1, 2, 6, 18, 19, 300):
                if (n == "cap+1" and A == 300) or (n == 10 ** 6 and A not in (1, 6)):
                    continue
                cases.append((kind, n, A))
    return cases


STANDALONE = _standalone_cases()


@pytest.mark.parametrize("grad", [True, False], ids=["grad", "nograd"])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("kind,N,A", STANDALONE, ids=["%s-N%s-A%d" % c for c in STANDALONE])
def test_standalone_loss_within_bound(kind, N, A, dtype, grad):
    if N == "cap+1":
        N = 4 * sm_count() * 256 + 1
    u = LO.U32 if dtype == torch.float32 else LO.U64
    out, g, inp = _standalone(kind, dtype, N, A, grad, workspace(), seed=N % 1000 + A)
    if N == 0:
        assert out == 0 and same_bits(np.asarray(out), np.zeros((), out.dtype)), "N = 0 must write 0"
        return
    if kind == "baseline":
        o = LO.baseline_loss(inp["adv"], u)
    elif kind == "entropy":
        o = LO.entropy_loss(inp["x"], u)
    else:
        o = LO.pg_loss(inp["x"], inp["a"], inp["adv"], u)
    within(out, o["out"], o["mag_out"], u, "out")
    if kind == "entropy" and A == 1:
        assert out == 0 and (g is None or not g.any())
    if grad:
        if kind == "baseline":
            assert same_bits(g, inp["adv"]), "the baseline gradient is the advantage itself"
        else:
            within(g.reshape(N, A), o["grad"], o["mag_grad"], u, "grad")
