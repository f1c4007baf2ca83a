"""Network modules whose forward/backward are the hand-written sm_90a kernels.

`AtariNet` keeps the reference's constructor, `initial_state`, `forward` contract and
state_dict keys/shapes (/root/reference/torchbeast/monobeast.py:545-635, BASELINE.md section 5) so
reference checkpoints load, but its parameters are views into ONE flat device buffer (and its
gradients into one flat gradient buffer): that is what the C-ABI kernels, the fused
clip+RMSprop step and the single NCCL all-reduce operate on.
"""
import collections
import ctypes
import weakref

import torch
from torch import nn

from torchbeast_b200 import _lib, action_space
from torchbeast_b200.legal_actions import mask_policy

LearnerOutputs = collections.namedtuple("LearnerOutputs", "policy_logits baseline core_state")


class _ParamGroup(nn.Module):
    """Namespace module so parameters get the reference's dotted names (conv1.weight, ...)."""


class PopArt(nn.Module):
    """PopArt value statistics of a net built with `num_tasks` = K (van Hasselt et al. 2016, Hessel et al. 2019):
    buffers `mu` and `nu` (float64 [K], first and second moment of each task's V-trace targets; state_dict keys
    popart.mu and popart.nu) start at 0 and 1.  The net's value head then has K normalised outputs, baseline [T, B, K]:
    the value of task k is sigma_k * baseline[..., k] + mu_k with sigma_k = clamp(sqrt(nu_k - mu_k^2), 1e-4, 1e6).
    learn() updates them."""

    MAX_TASKS = 64

    def __init__(self, num_tasks, device):
        super().__init__()
        num_tasks = int(num_tasks)
        if not 1 <= num_tasks <= self.MAX_TASKS:
            raise _lib.TorchBeastB200Error("num_tasks must be in [1, %d], got %d" % (self.MAX_TASKS, num_tasks))
        self.num_tasks = num_tasks
        self.register_buffer("mu", torch.zeros(num_tasks, dtype=torch.float64, device=device))
        self.register_buffer("nu", torch.ones(num_tasks, dtype=torch.float64, device=device))

    def _apply(self, fn, recurse=True):
        # the statistics stay float64 through .float() and the like
        super()._apply(fn, recurse)
        for key, buf in list(self._buffers.items()):
            self._buffers[key] = buf.to(torch.float64)
        return self

    def sigma(self):
        return (self.nu - self.mu * self.mu).clamp_min(0).sqrt().clamp(1e-4, 1e6)

    def unnormalize(self, baseline, task=None):
        """The unnormalised value [T, B] (float32) of each row's own task from a normalised `baseline` [T, B, K]; `task`
        int64 [T, B] (default: task 0; ids must be in [0, K))."""
        if task is None:
            task = torch.zeros(baseline.shape[:-1], dtype=torch.int64, device=baseline.device)
        task = task.to(device=self.mu.device, dtype=torch.int64)
        n = baseline.to(torch.float64).gather(-1, task.unsqueeze(-1).to(baseline.device)).squeeze(-1)
        return (self.sigma()[task] * n + self.mu[task]).to(torch.float32)


def atarinet_param_spec(num_actions, use_lstm, in_channels=4, num_values=1, continuous_dim=None):
    """continuous_dim D (a Gaussian(D) space, num_actions = 2D): the core takes D last-action columns, 512 + D + 1."""
    core = 512 + (num_actions if continuous_dim is None else continuous_dim) + 1
    spec = [
        ("conv1.weight", (32, in_channels, 8, 8)), ("conv1.bias", (32,)),
        ("conv2.weight", (64, 32, 4, 4)), ("conv2.bias", (64,)),
        ("conv3.weight", (64, 64, 3, 3)), ("conv3.bias", (64,)),
        ("fc.weight", (512, 3136)), ("fc.bias", (512,)),
    ]
    if use_lstm:
        for layer in range(2):
            spec += [
                ("core.weight_ih_l%d" % layer, (4 * core, core)), ("core.weight_hh_l%d" % layer, (4 * core, core)),
                ("core.bias_ih_l%d" % layer, (4 * core,)), ("core.bias_hh_l%d" % layer, (4 * core,)),
            ]
    spec += [
        ("policy.weight", (num_actions, core)), ("policy.bias", (num_actions,)),
        ("baseline.weight", (num_values, core)), ("baseline.bias", (num_values,)),
    ]
    return spec


ATARI_SHAPE = (4, 84, 84)
LSTM_MAX_HIDDEN = 700  # TB_LSTM_MAX_HIDDEN
HEADS_MAX_OUTPUTS = 31  # the fused policy / baseline heads take A < 32
RESNET_CHANNELS = (16, 32, 32)   # the IMPALA paper's section widths


def resnet_obs_range():
    """{"C": (min, max), "H": (min, max), "W": (min, max)}: the observations u8 [C, H, W] the ResNet takes on every
    backend, as the C library states them (include/torchbeast_b200.h, tb_resnet_obs_range)."""
    r = (ctypes.c_int * 6)()
    _lib.check(_lib.lib().tb_resnet_obs_range(ctypes.cast(r, ctypes.c_void_p)), "tb_resnet_obs_range")
    return {"C": (r[0], r[1]), "H": (r[2], r[3]), "W": (r[4], r[5])}


def resnet_widths():
    """The channel counts each ResNet section takes (16, 32, 64), as the C library states them (tb_resnet_widths)."""
    r = (ctypes.c_int * 3)()
    _lib.check(_lib.lib().tb_resnet_widths(ctypes.cast(r, ctypes.c_void_p)), "tb_resnet_widths")
    return tuple(r)


def frame_is_unstacked(frame, reward, observation_shape=ATARI_SHAPE, channels=RESNET_CHANNELS):
    """False for a stacked frame u8 [T1, B, C, H, W] with [C, H, W] = observation_shape; True for an unstacked rollout
    u8 [T1+3, B, 84, 84] with T1 = reward.shape[0] (include/torchbeast_b200.h, "unstacked rollouts"), which only a
    (4, 84, 84) net with the default section widths takes.  Anything else raises."""
    obs = tuple(observation_shape)
    stacked = "[T,B,%d,%d,%d]" % obs
    if frame.dtype != torch.uint8 or frame.dim() not in (4, 5):
        raise _lib.TorchBeastB200Error("frame must be uint8 %s%s, got %s %r"
                                       % (stacked, " or unstacked [T+3,B,84,84]" if obs == ATARI_SHAPE else "",
                                          frame.dtype, tuple(frame.shape)))
    if frame.dim() == 5:
        if tuple(frame.shape[2:]) != obs:
            raise _lib.TorchBeastB200Error("frame must be uint8 %s, got %s %r" % (stacked, frame.dtype, tuple(frame.shape)))
        return False
    if obs != ATARI_SHAPE:
        raise _lib.TorchBeastB200Error(
            "unstacked rollouts and newest frames rebuild (4, 84, 84) stacks; this net takes stacked frames uint8 %s, "
            "got %r" % (stacked, tuple(frame.shape)))
    if tuple(channels) != RESNET_CHANNELS:
        raise _lib.TorchBeastB200Error(
            "unstacked rollouts and newest frames run on the default widths %r; this net has channels=%r and takes "
            "stacked frames uint8 %s, got %r" % (RESNET_CHANNELS, tuple(channels), stacked, tuple(frame.shape)))
    T1, B = reward.shape[:2]
    if tuple(frame.shape) != (T1 + 3, B, 84, 84):
        raise _lib.TorchBeastB200Error(
            "an unstacked frame must be uint8 [T1+3, B, 84, 84] with [T1, B] = reward's shape %r, got %r"
            % ((T1, B), tuple(frame.shape)))
    return True


def _done_bytes(done, T1, B):
    """The restack's view of `done`: [T1, B] bool or uint8 as contiguous bytes (non-zero = an episode starts)."""
    if done is None or done.dtype not in (torch.bool, torch.uint8) or tuple(done.shape) != (T1, B):
        raise _lib.TorchBeastB200Error("done must be bool or uint8 [%d, %d] with an unstacked frame, got %s"
                                       % (T1, B, None if done is None else "%s %r" % (done.dtype, tuple(done.shape))))
    return done.contiguous().view(torch.uint8)


def _scratch(module, net, T1, B):
    """Caller-owned stacked scratch for the backends that read stacked frames; None where the restack is fused."""
    nbytes = _lib.lib().tb_unstacked_scratch_bytes(net, T1, B, module.PRECISIONS[module.precision])
    if nbytes == 0:
        return None
    key = (T1, B, module._flat.device, module.precision)
    if module._scratch_key != key:
        module._scratch_buf = torch.empty(nbytes, dtype=torch.uint8, device=module._flat.device)
        module._scratch_key = key
    return module._scratch_buf


def _numel(shape):
    n = 1
    for d in shape:
        n *= d
    return n


class FlatParamModule(nn.Module):
    """nn.Module whose Parameters alias one flat fp32 buffer (`flat_params`) in spec order."""

    # flat buffer address -> module: lets load_state_dict() recognise a sibling's state_dict (whose tensors alias that
    # sibling's flat buffer) and take the one-copy path without hanging anything on the dict itself
    _flat_owners = weakref.WeakValueDictionary()

    # torchbeast_b200.sampling.ActionSampler used by training-mode forwards instead of torch.multinomial; None keeps the
    # reference's sampling.  Not part of the state_dict: checkpoint its `seed` and `step` alongside.
    action_sampler = None
    # torchbeast_b200.acting.FrameHistory: with one attached, forward() also takes each stream's newest frame u8
    # [T, B, 84, 84] and rebuilds the four-frame stacks on the device from that stream's history.  None: forward takes
    # the stacked and unstacked frames only.  Not part of the state_dict.
    frame_history = None

    def _baseline_shape(self, T1, B):
        """[T1, B], or [T1, B, K] for a net with K PopArt tasks."""
        return (T1, B) if getattr(self, "popart", None) is None else (T1, B, self.num_values)

    def value_head(self):
        """(baseline.weight [K, F], baseline.bias [K]): the value head's views of the flat parameter buffer."""
        return self.baseline.weight.data, self.baseline.bias.data

    def _forward_frame(self, inputs):
        """inputs["frame"], or, with a frame_history attached and newest frames [T, B, 84, 84] (T = reward's), the
        unstacked rollout [T+3, B, 84, 84] the history builds from them (acting.FrameHistory.stack)."""
        frame, reward = inputs["frame"], inputs["reward"]
        obs = tuple(getattr(self, "observation_shape", ATARI_SHAPE))
        if self.frame_history is not None and obs != ATARI_SHAPE:
            raise _lib.TorchBeastB200Error("a frame_history rebuilds (4, 84, 84) stacks; this net takes stacked frames "
                                           "uint8 [T,B,%d,%d,%d]: detach the history (model.frame_history = None)" % obs)
        channels = tuple(getattr(self, "channels", RESNET_CHANNELS))
        if self.frame_history is not None and channels != RESNET_CHANNELS:
            raise _lib.TorchBeastB200Error("a frame_history feeds the default widths %r; this net has channels=%r and "
                                           "takes stacked frames: detach the history (model.frame_history = None)"
                                           % (RESNET_CHANNELS, channels))
        if self.frame_history is None or frame.dim() != 4 or frame.shape[0] != reward.shape[0]:
            return frame
        if frame.shape[1] != reward.shape[1]:
            raise _lib.TorchBeastB200Error("newest frames [T, B, 84, 84] must match reward's [T, B] = %r, got frame %r"
                                           % (tuple(reward.shape[:2]), tuple(frame.shape)))
        return self.frame_history.stack(frame, inputs.get("done"), inputs.get("stream_ids"), self._flat.device)

    # component sizes (A_1, ..., A_D) of a factored action space (torchbeast_b200.action_space), or None: one categorical
    # over num_actions choices.  num_actions is the policy-logit width either way.
    action_dims = None
    # D of a continuous (Gaussian(D)) action space, whose policy rows are (mu, log sigma) of width num_actions = 2D
    continuous_dim = None

    def _set_action_space(self, num_actions):
        """num_actions: an int, a tuple of component sizes (a factored space) or a Gaussian(D) (a continuous one); sets
        num_actions to the logit width."""
        self.action_dims = action_space.dims_of(num_actions)
        self.continuous_dim = action_space.continuous_dim_of(num_actions)
        self.num_actions = action_space.width(num_actions)
        if self.continuous_dim is not None and self.num_actions > HEADS_MAX_OUTPUTS:
            raise _lib.TorchBeastB200Error("the policy head takes at most %d outputs: Gaussian(D) needs D <= %d, got %r"
                                           % (HEADS_MAX_OUTPUTS, HEADS_MAX_OUTPUTS // 2, num_actions))

    def _sample(self, logits, inputs):
        """Training-mode action [T, B] (factored: [T, B, D]) of the reference-compatible forwards
        (monobeast.py:618-619).  With a sampler, an optional inputs["stream_ids"] (int64 [B], e.g. actor indices) names
        each column's random stream."""
        T, B, A = logits.shape
        if self.action_sampler is not None:
            if self.action_dims is not None:
                return self.action_sampler.sample(logits, inputs.get("stream_ids"), action_dims=self.action_dims)
            if self.continuous_dim is not None:
                return self.action_sampler.sample(logits, inputs.get("stream_ids"), continuous_dim=self.continuous_dim)
            return self.action_sampler.sample(logits, inputs.get("stream_ids"))
        if self.action_dims is not None:
            return action_space.multinomial(logits, self.action_dims)
        if self.continuous_dim is not None:
            return action_space.gaussian_normal(logits, self.continuous_dim)
        return torch.multinomial(torch.softmax(logits.detach().view(T * B, A), dim=1), num_samples=1).view(T, B)

    def _greedy(self, logits):
        """Eval-mode action: argmax over the row, or per segment of a factored space; the mean of a Gaussian one."""
        T, B = logits.shape[:2]
        if self.action_dims is not None:
            return action_space.greedy(logits, self.action_dims)
        if self.continuous_dim is not None:
            return action_space.gaussian_mean(logits, self.continuous_dim)
        return torch.argmax(logits.detach().view(T * B, self.num_actions), dim=1)  # don't sample when testing

    def _build_flat(self, spec, device):
        self._spec = list(spec)
        total = sum(_numel(s) for _, s in self._spec)
        self._flat = torch.zeros(total, dtype=torch.float32, device=device)
        self._flat_grad = None
        self._views = []
        off = 0
        for name, shape in self._spec:
            *groups, leaf = name.split(".")
            mod = self
            for gname in groups:  # nested namespaces: "feat_convs.0.0.weight" -> feat_convs -> "0" -> "0"
                if gname not in mod._modules:
                    mod.add_module(gname, _ParamGroup())
                mod = mod._modules[gname]
            n = _numel(shape)
            p = nn.Parameter(self._flat[off:off + n].view(shape))
            mod.register_parameter(leaf, p)
            self._views.append((p, off, n, shape))
            off += n
        self._total = total
        FlatParamModule._flat_owners[self._flat.data_ptr()] = self

    # keep the aliasing across .to()/.cuda()/.float(): move the flat buffer, re-point the views
    def _apply(self, fn, recurse=True):
        new_flat = fn(self._flat)
        if new_flat.dtype != torch.float32:
            raise _lib.TorchBeastB200Error("torchbeast_b200 networks are float32 only")
        self._flat = new_flat.contiguous()
        FlatParamModule._flat_owners[self._flat.data_ptr()] = self
        self._flat_grad = None
        for p, off, n, shape in self._views:
            p.data = self._flat[off:off + n].view(shape)
            p.grad = None
        for key, buf in list(self._buffers.items()):
            if buf is not None:
                self._buffers[key] = fn(buf)
        if getattr(self, "popart", None) is not None:
            self.popart._apply(fn)
        return self

    @property
    def flat_params(self):
        return self._flat

    @property
    def flat_grad(self):
        """Flat gradient buffer; every Parameter's .grad is (re)pointed at its slice."""
        if self._flat_grad is None or self._flat_grad.device != self._flat.device:
            self._flat_grad = torch.zeros_like(self._flat)
        return self._flat_grad

    def attach_grads(self):
        """Point every Parameter's .grad at its slice of the flat gradient buffer.  A gradient that lives elsewhere
        (autograd wrote it: model(...) -> loss.backward()) is COPIED into its slice first, so the fused optimizer
        steps on it instead of silently discarding it."""
        fg = self.flat_grad
        for p, off, n, shape in self._views:
            if p.grad is None:
                p.grad = fg[off:off + n].view(shape)
            elif p.grad.data_ptr() != fg.data_ptr() + 4 * off:
                fg[off:off + n].copy_(p.grad.detach().reshape(-1))
                p.grad = fg[off:off + n].view(shape)
        return fg

    def copy_params_from(self, other):
        """actor_model.load_state_dict(model.state_dict()) as ONE device copy (monobeast.py:295), plus the PopArt
        statistics when both nets have them."""
        self._flat.copy_(other._flat, non_blocking=True)
        if getattr(self, "popart", None) is not None and getattr(other, "popart", None) is not None:
            self.popart.mu.copy_(other.popart.mu, non_blocking=True)
            self.popart.nu.copy_(other.popart.nu, non_blocking=True)

    def _aliased_sibling(self, state_dict):
        """The FlatParamModule whose live flat buffer EVERY tensor of `state_dict` aliases at this module's own
        offsets (i.e. `sibling.state_dict()` as returned, unedited), or None."""
        names = [n for n, _ in self._spec]
        if len(state_dict) != len(names):
            return None
        first = state_dict.get(names[0])
        if not isinstance(first, torch.Tensor):
            return None
        src = FlatParamModule._flat_owners.get(first.data_ptr())
        if src is None or src is self or src._total != self._total or list(src._spec) != list(self._spec):
            return None
        base = src._flat.data_ptr()
        for (name, shape), (_, off, n, _s) in zip(self._spec, self._views):
            t = state_dict.get(name)
            if not isinstance(t, torch.Tensor) or t.data_ptr() != base + 4 * off or tuple(t.shape) != tuple(shape) \
                    or t.dtype != torch.float32 or not t.is_contiguous():
                return None
        return src

    def load_state_dict(self, state_dict, strict=True, assign=False):
        """Reference checkpoints / state_dicts load key by key; `actor.load_state_dict(model.state_dict())`
        (monobeast.py:295) is recognised by aliasing and becomes ONE device copy.  The dict itself carries nothing
        but tensors, so torch.save / torch.load(weights_only=True) / copy.deepcopy behave as for any nn.Module."""
        stats = ("popart.mu", "popart.nu")
        has_stats = getattr(self, "popart", None) is not None and all(k in state_dict for k in stats)
        params = {k: v for k, v in state_dict.items() if k not in stats} if has_stats else state_dict
        src = self._aliased_sibling(params)
        if src is not None:
            self.copy_params_from(src)
            if has_stats:  # from any net with the same number of tasks (its statistics may be host tensors)
                self.popart.mu.copy_(state_dict["popart.mu"])
                self.popart.nu.copy_(state_dict["popart.nu"])
            return torch.nn.modules.module._IncompatibleKeys([], [])
        return super().load_state_dict(state_dict, strict=strict)

    def reset_parameters_like_torch(self, seed=None):
        """Same init distributions as the reference modules (nn.Conv2d / nn.Linear / nn.LSTM
        defaults: U(-1/sqrt(fan_in), 1/sqrt(fan_in)); LSTM: U(-1/sqrt(H), 1/sqrt(H)))."""
        gen = torch.Generator(device="cpu")
        if seed is not None:
            gen.manual_seed(seed)
        else:
            gen.manual_seed(int(torch.randint(0, 2 ** 31 - 1, (1,)).item()))
        hidden = None
        for name, shape in self._spec:
            if name.startswith("core.weight_hh"):
                hidden = shape[1]
        with torch.no_grad():
            for (name, shape), (p, off, n, _) in zip(self._spec, self._views):
                if name.startswith("core."):
                    bound = 1.0 / (hidden ** 0.5)
                else:
                    wshape = dict(self._spec)[name.rsplit(".", 1)[0] + ".weight"]
                    bound = 1.0 / (_numel(wshape[1:]) ** 0.5)
                vals = (torch.rand(n, generator=gen, dtype=torch.float32) * 2 - 1) * bound
                self._flat[off:off + n].copy_(vals)


class _AtariNetFunction(torch.autograd.Function):
    """Autograd bridge for users who call model(...) and loss.backward() themselves.
    learn() does not go through autograd (it calls learner_forward/learner_backward)."""

    @staticmethod
    def forward(ctx, module, frame, done, reward, notdone, last_action, h0, c0, *params):
        logits, baseline, hN, cN = module._launch_forward(frame, reward, notdone, last_action, h0, c0, done)
        ctx.module = module
        ctx.notdone = notdone
        ctx.shape = baseline.shape
        ctx.mark_non_differentiable(hN, cN)
        return logits, baseline, hN, cN

    @staticmethod
    def backward(ctx, g_logits, g_baseline, _ghn, _gcn):
        module = ctx.module
        T1, B = ctx.shape[:2]
        if g_logits is None:
            g_logits = torch.zeros(T1, B, module.num_actions, device=module._flat.device)
        if g_baseline is None:
            g_baseline = torch.zeros(module._baseline_shape(T1, B), device=module._flat.device)
        grads = torch.empty_like(module._flat)
        module._launch_backward(g_logits.contiguous(), g_baseline.contiguous(), ctx.notdone, grads)
        outs = tuple(grads[off:off + n].view(shape) for _, off, n, shape in module._views)
        return (None,) * 8 + outs


class AtariNet(FlatParamModule):
    """CUDA AtariNet (reference monobeast.py:545-635).  conv 8/4 -> 4/2 -> 3/1 -> fc 512 ->
    cat[reward, one-hot last action] -> optional 2-layer LSTM(519) -> policy / baseline heads."""

    # "bf16x3" (default): every dense product on wgmma tensor cores with SPLIT bf16 operands - x = hi + lo, two bf16
    #     planes, accumulated as hi.hi + hi.lo + lo.hi in fp32 (3 MMAs, ~2^-17 relative per product): holds the
    #     reference's fp32 results to the 1e-4 parity contract (tests/test_learner_baseline_gpu.py);
    # "bf16": single-plane bf16 operands (1 MMA, 2^-9): fastest, mixed-precision tolerances only;
    # "fp32": exact fp32 FFMA (SIMT) GEMMs - the slow parity anchor.
    PRECISIONS = {"fp32": 0, "bf16": 1, "bf16x3": 2}
    DEFAULT_PRECISION = "bf16x3"
    needs_last_action = True  # forward consumes inputs["last_action"] (monobeast.py:593-597); polybeast's Net does not

    def __init__(self, observation_shape, num_actions, use_lstm=False, device=None, precision=None, num_tasks=None):
        super().__init__()
        if tuple(observation_shape) != (4, 84, 84):
            raise _lib.TorchBeastB200Error(
                "torchbeast_b200.AtariNet is specialised for (4, 84, 84) uint8 frames, got %r" % (tuple(observation_shape),))
        self.observation_shape = tuple(observation_shape)
        self._set_action_space(num_actions)
        num_actions = self.num_actions
        self.use_lstm = use_lstm
        D = self.continuous_dim
        self.core_size = 512 + (num_actions if D is None else D) + 1
        if self.action_dims is not None and use_lstm and self.core_size > LSTM_MAX_HIDDEN:
            raise _lib.TorchBeastB200Error(
                "AtariNet with an LSTM needs 512 + sum(num_actions) + 1 <= %d, got %d for num_actions=%r"
                % (LSTM_MAX_HIDDEN, self.core_size, self.action_dims))
        if D is not None and use_lstm and self.core_size > LSTM_MAX_HIDDEN:
            raise _lib.TorchBeastB200Error("AtariNet with an LSTM needs 512 + D + 1 <= %d, got %d for Gaussian(%d)"
                                           % (LSTM_MAX_HIDDEN, self.core_size, D))
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        popart = None if num_tasks is None else PopArt(num_tasks, device)
        self.num_values = 1 if popart is None else popart.num_tasks
        self._build_flat(atarinet_param_spec(num_actions, use_lstm, num_values=self.num_values, continuous_dim=D),
                         device)
        self.reset_parameters_like_torch()
        if popart is not None:
            self.popart = popart  # registered after the parameters: its keys come last in the state_dict
        if use_lstm:
            self.core.num_layers = 2
            self.core.hidden_size = self.core_size
            self.core.input_size = self.core_size
        import os
        self.precision = precision or os.environ.get("TB_PRECISION", self.DEFAULT_PRECISION)
        if self.precision not in self.PRECISIONS:
            raise _lib.TorchBeastB200Error("precision must be one of %s" % sorted(self.PRECISIONS))
        self._ws = None
        self._ws_key = None
        self._scratch_buf = self._scratch_key = None
        if D is None:
            count = _lib.lib().tb_atarinet_param_count(num_actions, self.num_values, int(use_lstm))
        else:
            count = _lib.lib().tb_atarinet_param_count_continuous(num_actions, self.num_values, int(use_lstm))
        assert count == self._total, "parameter layout disagrees with the C-ABI (%d vs %d)" % (count, self._total)

    def initial_state(self, batch_size):
        if not self.use_lstm:
            return tuple()
        return tuple(torch.zeros(2, batch_size, self.core_size, device=self._flat.device) for _ in range(2))

    # ---- raw launches ---------------------------------------------------------------------
    def _workspace(self, T1, B):
        key = (T1, B, self._flat.device, self.precision)
        if self._ws_key != key:
            ws_bytes = _lib.lib().tb_atarinet_workspace_bytes if self.continuous_dim is None \
                else _lib.lib().tb_atarinet_workspace_bytes_continuous
            nbytes = ws_bytes(T1, B, self.num_actions, int(self.use_lstm), self.PRECISIONS[self.precision])
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self._flat.device)
            self._ws_key = key
        return self._ws

    def _launch_forward(self, frame, reward, notdone, last_action, h0, c0, done=None):
        """`done` is read only with an unstacked frame (frame_is_unstacked), to rebuild the stacks."""
        _lib.require_cuda(frame, reward, last_action, self._flat)
        unstacked = frame_is_unstacked(frame, reward)
        T1, B = reward.shape[:2] if unstacked else frame.shape[:2]
        if unstacked:
            _lib.require_cuda(done)
            done = _done_bytes(done, T1, B)
        dev = self._flat.device
        frame = frame.contiguous()
        reward = reward.to(torch.float32).contiguous()
        D = self.continuous_dim
        if D is not None:
            if last_action.dtype != torch.float32 or tuple(last_action.shape) != (T1, B, D):
                raise _lib.TorchBeastB200Error("last_action must be float32 [T, B, D] = %r for Gaussian(%d), got %s %r"
                                               % ((T1, B, D), D, last_action.dtype, tuple(last_action.shape)))
            last_action = last_action.contiguous()
        else:
            last_action = last_action.to(torch.int64).contiguous()
        logits = torch.empty(T1, B, self.num_actions, dtype=torch.float32, device=dev)
        baseline = torch.empty(self._baseline_shape(T1, B), dtype=torch.float32, device=dev)
        if self.use_lstm:
            hN = torch.empty(2, B, self.core_size, dtype=torch.float32, device=dev)
            cN = torch.empty_like(hN)
            h0 = h0.to(torch.float32).contiguous(); c0 = c0.to(torch.float32).contiguous()
        else:
            hN = cN = torch.empty(0, device=dev)
            h0 = c0 = notdone = None
        ws = self._workspace(T1, B)
        p = _lib.ptr
        args = (p(frame), p(done) if unstacked else None, p(reward), p(notdone), p(last_action), p(h0), p(c0),
                p(self._flat), T1, B, self.num_actions, self.num_values, int(self.use_lstm),
                self.PRECISIONS[self.precision], p(ws), p(_scratch(self, 0, T1, B)) if unstacked else None, p(logits),
                p(baseline), p(hN) if self.use_lstm else None, p(cN) if self.use_lstm else None)
        if D is not None:
            _lib.check(_lib.lib().tb_atarinet_forward_continuous(*args, _lib.stream_ptr()),
                       "tb_atarinet_forward_continuous")
        elif self.action_dims is None:
            _lib.check(_lib.lib().tb_atarinet_forward(*args, _lib.stream_ptr()), "tb_atarinet_forward")
        else:
            D = len(self.action_dims)
            if tuple(last_action.shape) != (T1, B, D):
                raise _lib.TorchBeastB200Error("last_action must be int64 [T, B, D] = %r for num_actions=%r, got %r"
                                               % ((T1, B, D), self.action_dims, tuple(last_action.shape)))
            _lib.check(_lib.lib().tb_atarinet_forward_factored(*args, ctypes.byref(action_space.c_space(self.action_dims)),
                                                               _lib.stream_ptr()),
                       "tb_atarinet_forward_factored")
        return logits, baseline, hN, cN

    def _launch_backward(self, g_logits, g_baseline, notdone, grads_out, phase=3):
        """phase 3: the whole backward; 1 then 2: heads + LSTM, then the conv/fc trunk."""
        T1, B = g_baseline.shape[:2]
        ws = self._workspace(T1, B)
        p = _lib.ptr
        name = "tb_atarinet_backward" if self.continuous_dim is None else "tb_atarinet_backward_continuous"
        _lib.check(
            getattr(_lib.lib(), name)(
                p(g_logits), p(g_baseline), p(notdone) if self.use_lstm else None, p(self._flat), T1, B,
                self.num_actions, self.num_values, int(self.use_lstm), self.PRECISIONS[self.precision], p(ws),
                p(grads_out), int(phase), _lib.stream_ptr()),
            name)

    def grad_split(self):
        """Flat-gradient offset where the LSTM + heads slice starts (final after backward phase 1 for precision
        fp32 / bf16x3): what a data-parallel learner all-reduces first, overlapped with the trunk backward."""
        return int(_lib.lib().tb_atarinet_grad_split(self.num_actions, int(self.use_lstm)))

    @staticmethod
    def _notdone(done):
        # `(~done).float()`: logical for bool, bitwise for uint8 - exactly the reference's expression
        return (~done).float().contiguous()

    # ---- learner fast path (no autograd graph) ----------------------------------------------
    @torch.no_grad()
    def learner_forward(self, inputs, core_state=()):
        notdone = self._notdone(inputs["done"]) if self.use_lstm else None
        h0, c0 = core_state if self.use_lstm else (None, None)
        logits, baseline, hN, cN = self._launch_forward(
            inputs["frame"], inputs["reward"], notdone, inputs["last_action"], h0, c0, inputs.get("done"))
        self._saved_notdone = notdone
        return LearnerOutputs(mask_policy(logits, inputs), baseline, (hN, cN) if self.use_lstm else tuple())

    @torch.no_grad()
    def learner_backward(self, grad_logits, grad_baseline, between=None, aux_stream=None):
        """Writes d loss / d params into flat_grad (and points every .grad at its slice).  `between(flat_grad, split)`:
        called after the heads + LSTM phase, before the conv/fc trunk phase is launched; flat_grad[split:] is then final
        in stream order on `aux_stream` once that stream has waited for the current one (data-parallel learners enqueue
        that slice's all-reduce on it there)."""
        fg = self.attach_grads()
        if between is None:
            self._launch_backward(grad_logits, grad_baseline, self._saved_notdone, fg)
            return fg
        # The tensor-core backends fork the LSTM weight-gradient GEMMs onto a side stream: make it the caller's (aux_stream)
        # so that what `between` enqueues there is ordered behind them and overlaps the trunk backward of phase 2.
        import ctypes
        lib = _lib.lib()
        if aux_stream is not None:
            lib.tb_set_aux_stream(ctypes.c_void_p(aux_stream.cuda_stream))
        try:
            self._launch_backward(grad_logits, grad_baseline, self._saved_notdone, fg, phase=1)
            between(fg, self.grad_split())
            self._launch_backward(grad_logits, grad_baseline, self._saved_notdone, fg, phase=2)
        finally:
            if aux_stream is not None:
                lib.tb_set_aux_stream(None)
        return fg

    # ---- reference-compatible forward ---------------------------------------------------------
    def forward(self, inputs, core_state=()):
        frame, done = self._forward_frame(inputs), inputs.get("done")
        notdone = self._notdone(done) if self.use_lstm else None
        h0, c0 = core_state if self.use_lstm else (None, None)
        params = [v[0] for v in self._views]
        if torch.is_grad_enabled() and any(q.requires_grad for q in params):
            logits, baseline, hN, cN = _AtariNetFunction.apply(
                self, frame, done, inputs["reward"], notdone, inputs["last_action"], h0, c0, *params)
        else:
            logits, baseline, hN, cN = self._launch_forward(frame, inputs["reward"], notdone, inputs["last_action"], h0, c0,
                                                            done)
        logits = mask_policy(logits, inputs)  # with inputs["legal_actions"]: the sampler and argmax pick legal actions
        T, B = baseline.shape[:2]
        action = self._sample(logits, inputs) if self.training else self._greedy(logits)
        out = dict(policy_logits=logits, baseline=baseline, action=action.view((T, B) + action.shape[2:]))
        return out, ((hN, cN) if self.use_lstm else tuple())




def resnet_fc_in(observation_shape=ATARI_SHAPE, channels=RESNET_CHANNELS):
    """Input features of the ResNet's fc layer: channels[2] x H_3 x W_3, each of the three max-pools (3, 2, 1) taking a
    side s to ceil(s / 2) (84 -> 42 -> 21 -> 11: 32 x 121 = 3872)."""
    _, h, w = observation_shape
    for _ in range(3):
        h, w = (h + 1) // 2, (w + 1) // 2
    return channels[2] * h * w


def resnet_param_spec(num_actions, use_lstm, num_values=1, observation_shape=ATARI_SHAPE, channels=RESNET_CHANNELS):
    """State_dict order/shapes of the reference's polybeast_learner.Net (pl:134-204, BASELINE.md section 5) for
    observations u8 [C, H, W] and section widths `channels`: feat_convs.i.0.weight (channels[i], C or channels[i-1],
    3, 3), the residual convs (channels[i], channels[i], 3, 3) and fc.weight (256, resnet_fc_in(...))."""
    spec = []
    cin = observation_shape[0]
    for i, ch in enumerate(channels):
        spec += [("feat_convs.%d.0.weight" % i, (ch, cin, 3, 3)), ("feat_convs.%d.0.bias" % i, (ch,))]
        cin = ch
    for blk in ("resnet1", "resnet2"):
        for i, ch in enumerate(channels):
            for j in (1, 3):
                spec += [("%s.%d.%d.weight" % (blk, i, j), (ch, ch, 3, 3)), ("%s.%d.%d.bias" % (blk, i, j), (ch,))]
    spec += [("fc.weight", (256, resnet_fc_in(observation_shape, channels))), ("fc.bias", (256,))]
    head_in = 257
    if use_lstm:
        spec += [("core.weight_ih_l0", (1024, 257)), ("core.weight_hh_l0", (1024, 256)),
                 ("core.bias_ih_l0", (1024,)), ("core.bias_hh_l0", (1024,))]
        head_in = 256
    spec += [("policy.weight", (num_actions, head_in)), ("policy.bias", (num_actions,)),
             ("baseline.weight", (num_values, head_in)), ("baseline.bias", (num_values,))]
    return spec


class _ResNetFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, frame, done, reward, notdone, h0, c0, *params):
        logits, baseline, hN, cN, saved = module._launch_forward(frame, reward, notdone, h0, c0, done)
        ctx.module, ctx.notdone, ctx.saved, ctx.shape = module, notdone, saved, baseline.shape
        ctx.mark_non_differentiable(hN, cN)
        return logits, baseline, hN, cN

    @staticmethod
    def backward(ctx, g_logits, g_baseline, _ghn, _gcn):
        module = ctx.module
        T1, B = ctx.shape[:2]
        dev = module._flat.device
        if g_logits is None:
            g_logits = torch.zeros(T1, B, module.num_actions, device=dev)
        if g_baseline is None:
            g_baseline = torch.zeros(module._baseline_shape(T1, B), device=dev)
        grads = torch.empty_like(module._flat)
        module._launch_backward(ctx.saved, g_logits.contiguous(), g_baseline.contiguous(), ctx.notdone, grads)
        return (None,) * 7 + tuple(grads[off:off + n].view(shape) for _, off, n, shape in module._views)


class ResNet(FlatParamModule):
    """CUDA IMPALA ResNet (reference polybeast_learner.py:134-266 `Net`): three sections of
    conv3x3 + maxpool3/2 + two residual blocks, fc 3872->256, cat[reward], optional LSTM(257->256), heads.
    forward(inputs, core_state) returns ((action, policy_logits, baseline), core_state) like the reference.

    observation_shape (keyword-only, default the Atari stack (4, 84, 84)): the u8 [C, H, W] of each frame, e.g.
    (3, 64, 64) for Procgen or (3, 72, 96) for DMLab; C from 1 to 16, H from 17 and W from 33 to 126
    (resnet_obs_range()), on every precision.  The fc then reads 32 x ceil(H/8) x ceil(W/8) features (resnet_fc_in).  Unstacked rollouts and a
    frame_history are (4, 84, 84) only.

    channels (keyword-only, default (16, 32, 32)): the widths of the three sections, each 16, 32 or 64
    (resnet_widths()), in any combination and at every supported observation shape, e.g. (32, 64, 64) for "IMPALA x2"
    (Cobbe et al., 2020).  Unstacked rollouts and a frame_history take the default widths only."""

    PRECISIONS = {"fp32": 0, "bf16": 1, "bf16x3": 2}

    def __init__(self, num_actions, use_lstm=False, device=None, precision=None, num_tasks=None, *,
                 observation_shape=ATARI_SHAPE, channels=RESNET_CHANNELS):
        super().__init__()
        import os
        self._set_action_space(num_actions)
        num_actions = self.num_actions
        self.use_lstm = use_lstm
        obs = tuple(int(d) for d in observation_shape)
        if len(obs) != 3 or not _lib.lib().tb_resnet_supported(*obs, *RESNET_CHANNELS, self.PRECISIONS["bf16x3"]):
            rng = resnet_obs_range()
            raise _lib.TorchBeastB200Error(
                "ResNet observation_shape must be (C, H, W) with C in [%d, %d], H in [%d, %d] and W in [%d, %d], got %r"
                % (sum((rng[k] for k in ("C", "H", "W")), ()) + (tuple(observation_shape),)))
        self.observation_shape = obs
        try:
            ch = tuple(int(c) for c in channels)
        except (TypeError, ValueError):
            ch = ()
        if len(ch) != 3 or not _lib.lib().tb_resnet_supported(*obs, *ch, self.PRECISIONS["bf16x3"]):
            raise _lib.TorchBeastB200Error(
                "ResNet channels must be three section widths, each one of %r, got %r" % (resnet_widths(), channels))
        self.channels = ch
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        popart = None if num_tasks is None else PopArt(num_tasks, device)
        self.num_values = 1 if popart is None else popart.num_tasks
        self._build_flat(resnet_param_spec(num_actions, use_lstm, num_values=self.num_values, observation_shape=obs,
                                           channels=ch), device)
        self._fix_module_names()
        self.reset_parameters_like_torch()
        if popart is not None:
            self.popart = popart  # registered after the parameters: its keys come last in the state_dict
        if use_lstm:
            self.core.num_layers, self.core.hidden_size, self.core.input_size = 1, 256, 257
        # patch-matrix GEMMs: "bf16x3" (default: split-bf16 tensor-core products over fp32 activations, parity-green),
        # "fp32" (SIMT) or "bf16" (single-plane operands and activations, not parity-grade)
        self.precision = precision or os.environ.get("TB_RESNET_PRECISION", "bf16x3")
        if self.precision not in self.PRECISIONS:
            raise _lib.TorchBeastB200Error("ResNet precision must be 'fp32', 'bf16' or 'bf16x3'")
        self._ws = None
        self._ws_key = None
        self._scratch_buf = self._scratch_key = None
        count = _lib.lib().tb_resnet_param_count(*obs, *ch, num_actions, self.num_values, int(use_lstm))
        assert count == self._total, "parameter layout disagrees with the C-ABI (%d vs %d)" % (count, self._total)

    def _fix_module_names(self):
        pass  # names with more than one dot are handled by _build_flat (see FlatParamModule._register)

    def initial_state(self, batch_size=1):
        if not self.use_lstm:
            return tuple()
        return tuple(torch.zeros(1, batch_size, 256, device=self._flat.device) for _ in range(2))

    def _workspace(self, T1, B):
        key = (T1, B, self._flat.device, self.precision)
        if self._ws_key != key:
            nbytes = _lib.lib().tb_resnet_workspace_bytes(*self.observation_shape, *self.channels, T1, B,
                                                          self.num_actions, int(self.use_lstm),
                                                          self.PRECISIONS[self.precision])
            if nbytes == 0:
                raise _lib.TorchBeastB200Error("tb_resnet_workspace_bytes: %s" % _lib.lib().tb_last_error().decode())
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self._flat.device)
            self._ws_key = key
        return self._ws

    def _launch_forward(self, frame, reward, notdone, h0, c0, done=None):
        """Returns (logits, baseline, hN, cN, saved): `saved` is the frame _launch_backward re-reads - the stacked frame,
        or with an unstacked one the stacked scratch it was rebuilt into (None where the backend needs none).  `done` is
        read only with an unstacked frame, to rebuild the stacks."""
        _lib.require_cuda(frame, reward, self._flat)
        unstacked = frame_is_unstacked(frame, reward, self.observation_shape, self.channels)
        T1, B = reward.shape[:2] if unstacked else frame.shape[:2]
        if unstacked:
            _lib.require_cuda(done)
            done = _done_bytes(done, T1, B)
        dev = self._flat.device
        frame = frame.contiguous()
        reward = reward.to(torch.float32).contiguous()
        logits = torch.empty(T1, B, self.num_actions, dtype=torch.float32, device=dev)
        baseline = torch.empty(self._baseline_shape(T1, B), dtype=torch.float32, device=dev)
        if self.use_lstm:
            hN = torch.empty(1, B, 256, dtype=torch.float32, device=dev)
            cN = torch.empty_like(hN)
            h0 = h0.to(torch.float32).contiguous(); c0 = c0.to(torch.float32).contiguous()
        else:
            hN = cN = torch.empty(0, device=dev)
            h0 = c0 = notdone = None
        p = _lib.ptr
        scratch = _scratch(self, 1, T1, B) if unstacked else None
        _lib.check(
            _lib.lib().tb_resnet_forward(
                p(frame), p(done) if unstacked else None, p(reward), p(notdone), p(h0), p(c0), p(self._flat),
                *self.observation_shape, *self.channels, T1, B, self.num_actions, self.num_values, int(self.use_lstm),
                self.PRECISIONS[self.precision], p(self._workspace(T1, B)), p(scratch), p(logits), p(baseline),
                p(hN) if self.use_lstm else None, p(cN) if self.use_lstm else None, _lib.stream_ptr()),
            "tb_resnet_forward")
        return logits, baseline, hN, cN, scratch if unstacked else frame

    def _launch_backward(self, frame, g_logits, g_baseline, notdone, grads_out):
        """`frame`: the `saved` of the forward."""
        T1, B = g_baseline.shape[:2]
        p = _lib.ptr
        _lib.check(
            _lib.lib().tb_resnet_backward(
                p(frame), p(g_logits), p(g_baseline), p(notdone) if self.use_lstm else None, p(self._flat),
                *self.observation_shape, *self.channels, T1, B, self.num_actions, self.num_values, int(self.use_lstm),
                self.PRECISIONS[self.precision], p(self._workspace(T1, B)), p(grads_out), _lib.stream_ptr()),
            "tb_resnet_backward")

    @torch.no_grad()
    def learner_forward(self, inputs, core_state=()):
        notdone = (~inputs["done"]).float().contiguous() if self.use_lstm else None
        h0, c0 = core_state if self.use_lstm else (None, None)
        logits, baseline, hN, cN, saved = self._launch_forward(inputs["frame"], inputs["reward"], notdone, h0, c0,
                                                               inputs.get("done"))
        self._saved = (saved, notdone)
        return LearnerOutputs(mask_policy(logits, inputs), baseline, (hN, cN) if self.use_lstm else tuple())

    @torch.no_grad()
    def learner_backward(self, grad_logits, grad_baseline):
        fg = self.attach_grads()
        frame, notdone = self._saved
        self._launch_backward(frame, grad_logits, grad_baseline, notdone, fg)
        return fg

    def forward(self, inputs, core_state=()):
        frame, done = self._forward_frame(inputs), inputs.get("done")
        notdone = (~done).float().contiguous() if self.use_lstm else None
        h0, c0 = core_state if self.use_lstm else (None, None)
        params = [v[0] for v in self._views]
        if torch.is_grad_enabled() and any(q.requires_grad for q in params):
            logits, baseline, hN, cN = _ResNetFunction.apply(self, frame, done, inputs["reward"], notdone, h0, c0, *params)
        else:
            logits, baseline, hN, cN, _ = self._launch_forward(frame, inputs["reward"], notdone, h0, c0, done)
        logits = mask_policy(logits, inputs)  # with inputs["legal_actions"]: the sampler and argmax pick legal actions
        T, B = baseline.shape[:2]
        action = self._sample(logits, inputs) if self.training else self._greedy(logits)
        return (action.view((T, B) + action.shape[2:]), logits, baseline), ((hN, cN) if self.use_lstm else tuple())


Net = AtariNet
