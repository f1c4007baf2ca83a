"""GPU: unstacked rollouts give bit-identical results to their restacked twins - the restack kernel against the NumPy
oracle, every network backend's learner forward / backward, monobeast.learn from host buffers (eager and graphed) and
the SyntheticActors -> polybeast_learner.learn pipeline; plus the launch count of each backend."""
import gc
import threading
import types

import numpy as np
import pytest
import torch

from oracle import frames_np as F
from oracle import learner_torch as LT

pytestmark = pytest.mark.gpu

@pytest.fixture(autouse=True)
def _collect_graphs():
    """Models and the GraphedLearners stored on them reference each other, so a test's CUDA graphs outlive it as cyclic
    garbage.  Collect them here: a collection that happens to run inside a later test's stream capture would destroy
    graphs (and free their memory pools) from the capturing thread, which invalidates that capture."""
    yield
    gc.collect()
    torch.cuda.synchronize()


FLAGS = dict(reward_clipping="abs_one", discounting=0.99, baseline_cost=0.5, entropy_cost=0.0006, grad_norm_clipping=40.0)


def _twin(T, B, seed, done_prob=0.2):
    """(unstacked frames, restacked frames, done) of one simulated rollout of T+1 steps that starts mid-stream."""
    stacks, done = F.simulate(T + 8, B, seed=seed, done_prob=done_prob)
    st, un, d = F.rollout(stacks, done, 7, T + 1)
    return torch.from_numpy(np.ascontiguousarray(un)), torch.from_numpy(np.ascontiguousarray(st)), torch.from_numpy(d.copy())


@pytest.mark.parametrize("T1,B", [(1, 3), (5, 33), (81, 32), (3, 1)])
def test_restack_kernel_matches_oracle(T1, B):
    from torchbeast_b200 import _lib
    un, st, d = _twin(T1 - 1, B, seed=T1 * 100 + B)
    assert np.array_equal(F.restack(un.numpy(), d.numpy()), st.numpy())
    frames = un.cuda()
    for done in (d.cuda().view(torch.uint8), d.to(torch.uint8).cuda() * 3):
        out = torch.empty(T1, B, 4, 84, 84, dtype=torch.uint8, device="cuda")
        _lib.check(_lib.lib().tb_restack_frames_u8(_lib.ptr(frames), _lib.ptr(done), T1, B, 84 * 84, _lib.ptr(out),
                                                   _lib.stream_ptr()), "tb_restack_frames_u8")
        assert torch.equal(out.cpu(), st)


def _model(net, use_lstm, precision, A=6):
    from torchbeast_b200 import nets
    if net == "atari":
        m = nets.AtariNet((4, 84, 84), A, use_lstm, precision=precision)
        m.load_state_dict(LT.random_params(LT.atarinet_param_shapes(A, use_lstm), seed=11))
    else:
        m = nets.ResNet(A, use_lstm, precision=precision)
        m.reset_parameters_like_torch(seed=11)
    return m


def _run(model, batch, state, g_logits, g_base):
    from torchbeast_b200 import _lib
    n0 = _lib.lib().tb_launch_count()
    out = model.learner_forward(batch, state)
    fg = model.learner_backward(g_logits, g_base).clone()
    torch.cuda.synchronize()
    return out, fg, _lib.lib().tb_launch_count() - n0


CASES = [(net, lstm, prec, 4, 2) for net in ("atari", "resnet") for lstm in (False, True) for prec in ("fp32", "bf16", "bf16x3")]
CASES += [(net, lstm, "bf16x3", 80, 32) for net in ("atari", "resnet") for lstm in (False, True)]


@pytest.mark.parametrize("net,use_lstm,precision,T,B", CASES)
def test_learner_forward_backward_bit_identical(net, use_lstm, precision, T, B):
    A = 6
    un, st, done = _twin(T, B, seed=T + B + use_lstm)
    batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=5).items()}
    batch["done"] = done.cuda()
    model = _model(net, use_lstm, precision)
    state = model.initial_state(B)
    state = tuple(0.1 * torch.randn_like(s) for s in state)
    g = torch.Generator(device="cuda").manual_seed(1)
    g_logits = torch.randn(T + 1, B, A, device="cuda", generator=g)
    g_base = torch.randn(T + 1, B, device="cuda", generator=g)
    _run(model, dict(batch, frame=un.cuda()), state, g_logits, g_base)  # first calls: allocations, one-time set-up
    ref, ref_g, n_stacked = _run(model, dict(batch, frame=st.cuda()), state, g_logits, g_base)
    got, got_g, n_unstacked = _run(model, dict(batch, frame=un.cuda()), state, g_logits, g_base)
    assert torch.equal(got.policy_logits, ref.policy_logits) and torch.equal(got.baseline, ref.baseline)
    assert all(torch.equal(a, b) for a, b in zip(got.core_state, ref.core_state))
    assert torch.equal(got_g, ref_g)
    fused = precision == "bf16x3" or (net == "atari" and precision == "bf16")
    # the restack is fused into the frame-image pass, or it is the one extra launch into the stacked scratch
    assert n_unstacked == n_stacked + (0 if fused else 1), (n_unstacked, n_stacked)
    assert (model._scratch_buf is None) == fused


@pytest.mark.parametrize("net", ["atari", "resnet"])
def test_autograd_forward_accepts_unstacked(net):
    A, T, B = 6, 4, 2
    un, st, done = _twin(T, B, seed=9)
    batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=6).items()}
    batch["done"] = done.cuda()
    grads = []
    for frame in (st, un):
        model = _model(net, True, "bf16x3")
        model.eval()
        out, _ = model(dict(batch, frame=frame.cuda()), tuple(model.initial_state(B)))
        logits, baseline = (out["policy_logits"], out["baseline"]) if net == "atari" else out[1:]
        (logits.square().sum() + baseline.sum()).backward()
        grads.append(torch.cat([p.grad.reshape(-1) for p in model.parameters()]))
    assert torch.equal(grads[0], grads[1])


@pytest.mark.parametrize("graph", [False, True])
def test_monobeast_learn_from_host_buffers(graph):
    from torchbeast_b200 import monobeast, optim
    T, B, A = 6, 4, 6
    un, st, done = _twin(T, B, seed=21, done_prob=0.3)
    host = LT.synthetic_batch(T, B, A, seed=7)
    host["done"] = done
    params = LT.random_params(LT.atarinet_param_shapes(A, True), seed=4)
    flags = types.SimpleNamespace(unroll_length=T, batch_size=B, cuda_graph=graph, **FLAGS)
    results = []
    for frame in (st, un):
        model = monobeast.AtariNet((4, 84, 84), A, True)
        actor = monobeast.AtariNet((4, 84, 84), A, True)
        model.load_state_dict(params)
        opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
        state = tuple(torch.zeros(2, B, 512 + A + 1) for _ in range(2))
        stats = [monobeast.learn(flags, actor, model, dict(host, frame=frame.pin_memory()), state, opt, None)
                 for _ in range(2)]
        torch.cuda.synchronize()
        results.append((stats, model.flat_params.clone(), opt.square_avg.clone()))
    (s0, p0, q0), (s1, p1, q1) = results
    keys = ("total_loss", "pg_loss", "baseline_loss", "entropy_loss", "episode_returns")
    assert [[s[k] for k in keys] for s in s0] == [[s[k] for k in keys] for s in s1]
    assert torch.equal(p0, p1) and torch.equal(q0, q1)


class _Take:
    """The first n batches of a LearnerQueue (so both pipelines take exactly the same steps)."""

    def __init__(self, q, n):
        self.q, self.n = q, n

    def size(self):
        return self.q.size()

    def __iter__(self):
        for _ in range(self.n):
            yield next(self.q)


def test_polybeast_pipeline_matches_stacked():
    from torchbeast_b200 import actors, monobeast, optim, polybeast_learner, staging
    T, B, A, steps = 5, 4, 6, 3
    dev = torch.device("cuda", 0)
    params = LT.random_params(LT.atarinet_param_shapes(A, True), seed=8)
    results = []
    for fmt in ("stacked", "unstacked"):
        model = monobeast.AtariNet((4, 84, 84), A, True)
        actor = monobeast.AtariNet((4, 84, 84), A, True)
        model.load_state_dict(params)
        opt = optim.RMSprop(model, lr=0.00048, momentum=0, eps=0.01, alpha=0.99)
        stager = staging.RolloutStager(staging.spec_for(T, B, A, use_last_action=False, frame_format=fmt), dev, depth=3)
        model._tb_stager = stager
        q = actors.LearnerQueue()
        # one actor thread fills the columns in a fixed order: the batches do not depend on thread timing
        pool = actors.SyntheticActors(stager, 1, T, B, A, q, state_shape=(2, 512 + A + 1), seed=3, frame_format=fmt)
        flags = types.SimpleNamespace(unroll_length=T, batch_size=B, **FLAGS)
        log = []

        class Log:
            def log(self, s):
                log.append(dict(s))
        pool.start()
        th = threading.Thread(target=polybeast_learner.learn,
                              args=(flags, _Take(q, steps), model, actor, opt, None, {}, Log(), threading.Lock()))
        th.start()
        th.join(timeout=120)
        pool.stop()
        assert not th.is_alive() and len(log) == steps
        torch.cuda.synchronize()
        results.append(([(s["total_loss"], s["pg_loss"], s["episode_returns"]) for s in log], model.flat_params.clone()))
    assert results[0][0] == results[1][0]
    assert torch.equal(results[0][1], results[1][1])


def _unstacked_batch(T, B, A, seed):
    un, _, done = _twin(T, B, seed=seed)
    batch = {k: v.cuda() for k, v in LT.synthetic_batch(T, B, A, seed=seed).items()}
    batch["done"], batch["frame"] = done.cuda(), un.cuda()
    return batch


@pytest.mark.parametrize("net,precision", [("atari", "fp32"), ("resnet", "bf16")])
def test_learner_graphs_keep_their_stacked_scratch(net, precision):
    """Backends that restack into a scratch: learn() with cuda_graph over two alternating unstacked batch shapes, with an
    eager forward of a third shape in between (each new shape replaces the model's scratch), equals eager learn_step step
    for step - every graph replays into the scratch it was captured with."""
    from torchbeast_b200 import learner, optim
    A = 6
    runs = []
    for graph in (False, True):
        model = _model(net, False, precision)
        actor = _model(net, False, precision)
        opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
        flags = types.SimpleNamespace(cuda_graph=graph, **FLAGS)
        third = _unstacked_batch(2, 5, A, seed=82)
        out = []
        for step in range(6):
            T, B = ((4, 2), (6, 3))[step % 2]
            batch = _unstacked_batch(T, B, A, seed=90 + step)
            if graph:
                s = learner.learn(flags, model, actor, batch, (), opt, None)
            else:
                s = learner.learn_step(flags, model, actor, batch, (), opt, None)
            model.learner_forward(third, ())
            out.append((s["total_loss"], s["pg_loss"], model.flat_params.clone()))
        if graph:
            scratch = [g.scratch for g in model._tb_graphs.values()]
            assert len(scratch) == 2 and all(t is not None for t in scratch)
            assert sorted(t.numel() for t in scratch) == [5 * 2 * 4 * 7056, 7 * 3 * 4 * 7056]
            assert all(t.data_ptr() != model._scratch_buf.data_ptr() for t in scratch)
        runs.append(out)
    for (le, pe, we), (lg, pg, wg) in zip(*runs):
        assert le == lg and pe == pg and torch.equal(we, wg)


def test_graphed_actor_rejects_unstacked_frames():
    from torchbeast_b200 import _lib
    from torchbeast_b200.acting import GraphedActor
    model = _model("atari", True, "bf16x3")  # training mode without a sampler: the frame is refused first, by shape
    inputs = dict(frame=torch.zeros(4, 3, 84, 84, dtype=torch.uint8, device="cuda"), reward=torch.zeros(1, 3, device="cuda"),
                  done=torch.zeros(1, 3, dtype=torch.bool, device="cuda"),
                  last_action=torch.zeros(1, 3, dtype=torch.int64, device="cuda"))
    with pytest.raises(_lib.TorchBeastB200Error, match="stacked frames"):
        GraphedActor(model)(inputs, model.initial_state(3))
