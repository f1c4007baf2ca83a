"""Network modules whose forward/backward are the hand-written sm_90a kernels.

`AtariNet` keeps the reference's constructor, `initial_state`, `forward` contract and
state_dict keys/shapes (/root/reference/torchbeast/monobeast.py:545-635, BASELINE.md section 5) so
reference checkpoints load, but its parameters are views into ONE flat device buffer (and its
gradients into one flat gradient buffer): that is what the C-ABI kernels, the fused
clip+RMSprop step and the single NCCL all-reduce operate on.
"""
import collections
import weakref

import torch
from torch import nn

from torchbeast_b200 import _lib

LearnerOutputs = collections.namedtuple("LearnerOutputs", "policy_logits baseline core_state")


class _ParamGroup(nn.Module):
    """Namespace module so parameters get the reference's dotted names (conv1.weight, ...)."""


def atarinet_param_spec(num_actions, use_lstm, in_channels=4):
    core = 512 + num_actions + 1
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
        ("baseline.weight", (1, core)), ("baseline.bias", (1,)),
    ]
    return spec


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

    def _sample(self, logits, inputs):
        """Training-mode action [T, B] of the reference-compatible forwards (monobeast.py:618-619).  With a sampler,
        an optional inputs["stream_ids"] (int64 [B], e.g. actor indices) names each column's random stream."""
        T, B, A = logits.shape
        if self.action_sampler is not None:
            return self.action_sampler.sample(logits, inputs.get("stream_ids"))
        return torch.multinomial(torch.softmax(logits.detach().view(T * B, A), dim=1), num_samples=1).view(T, B)

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
        """actor_model.load_state_dict(model.state_dict()) as ONE device copy (monobeast.py:295)."""
        self._flat.copy_(other._flat, non_blocking=True)

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
        src = self._aliased_sibling(state_dict)
        if src is not None:
            self.copy_params_from(src)
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
    def forward(ctx, module, frame, reward, notdone, last_action, h0, c0, *params):
        logits, baseline, hN, cN = module._launch_forward(frame, reward, notdone, last_action, h0, c0)
        ctx.module = module
        ctx.notdone = notdone
        ctx.shape = frame.shape[:2]
        ctx.mark_non_differentiable(hN, cN)
        return logits, baseline, hN, cN

    @staticmethod
    def backward(ctx, g_logits, g_baseline, _ghn, _gcn):
        module = ctx.module
        T1, B = ctx.shape
        if g_logits is None:
            g_logits = torch.zeros(T1, B, module.num_actions, device=module._flat.device)
        if g_baseline is None:
            g_baseline = torch.zeros(T1, B, device=module._flat.device)
        grads = torch.empty_like(module._flat)
        module._launch_backward(g_logits.contiguous(), g_baseline.contiguous(), ctx.notdone, grads)
        outs = tuple(grads[off:off + n].view(shape) for _, off, n, shape in module._views)
        return (None,) * 7 + outs


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

    def __init__(self, observation_shape, num_actions, use_lstm=False, device=None, precision=None):
        super().__init__()
        if tuple(observation_shape) != (4, 84, 84):
            raise _lib.TorchBeastB200Error(
                "torchbeast_b200.AtariNet is specialised for (4, 84, 84) uint8 frames, got %r" % (tuple(observation_shape),))
        self.observation_shape = tuple(observation_shape)
        self.num_actions = num_actions
        self.use_lstm = use_lstm
        self.core_size = 512 + num_actions + 1
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        self._build_flat(atarinet_param_spec(num_actions, use_lstm), device)
        self.reset_parameters_like_torch()
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
        count = _lib.lib().tb_atarinet_param_count(num_actions, int(use_lstm))
        assert count == self._total, "parameter layout disagrees with the C-ABI (%d vs %d)" % (count, self._total)

    def initial_state(self, batch_size):
        if not self.use_lstm:
            return tuple()
        return tuple(torch.zeros(2, batch_size, self.core_size, device=self._flat.device) for _ in range(2))

    # ---- raw launches ---------------------------------------------------------------------
    def _workspace(self, T1, B):
        key = (T1, B, self._flat.device, self.precision)
        if self._ws_key != key:
            nbytes = _lib.lib().tb_atarinet_workspace_bytes(T1, B, self.num_actions, int(self.use_lstm),
                                                            self.PRECISIONS[self.precision])
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self._flat.device)
            self._ws_key = key
        return self._ws

    def _launch_forward(self, frame, reward, notdone, last_action, h0, c0):
        _lib.require_cuda(frame, reward, last_action, self._flat)
        T1, B = frame.shape[:2]
        if frame.dtype != torch.uint8 or tuple(frame.shape[2:]) != self.observation_shape:
            raise _lib.TorchBeastB200Error("frame must be uint8 [T,B,4,84,84], got %s %r" % (frame.dtype, tuple(frame.shape)))
        dev = self._flat.device
        frame = frame.contiguous()
        reward = reward.to(torch.float32).contiguous()
        last_action = last_action.to(torch.int64).contiguous()
        logits = torch.empty(T1, B, self.num_actions, dtype=torch.float32, device=dev)
        baseline = torch.empty(T1, B, dtype=torch.float32, device=dev)
        if self.use_lstm:
            hN = torch.empty(2, B, self.core_size, dtype=torch.float32, device=dev)
            cN = torch.empty_like(hN)
            h0 = h0.to(torch.float32).contiguous(); c0 = c0.to(torch.float32).contiguous()
        else:
            hN = cN = torch.empty(0, device=dev)
            h0 = c0 = notdone = None
        ws = self._workspace(T1, B)
        p = _lib.ptr
        _lib.check(
            _lib.lib().tb_atarinet_forward(
                p(frame), p(reward), p(notdone), p(last_action), p(h0), p(c0), p(self._flat), T1, B,
                self.num_actions, int(self.use_lstm), self.PRECISIONS[self.precision], p(ws), p(logits), p(baseline),
                p(hN) if self.use_lstm else None, p(cN) if self.use_lstm else None, _lib.stream_ptr()),
            "tb_atarinet_forward")
        return logits, baseline, hN, cN

    def _launch_backward(self, g_logits, g_baseline, notdone, grads_out, phase=None):
        T1, B = g_baseline.shape
        ws = self._workspace(T1, B)
        p = _lib.ptr
        if phase is None:
            _lib.check(
                _lib.lib().tb_atarinet_backward(
                    p(g_logits), p(g_baseline), p(notdone) if self.use_lstm else None, p(self._flat), T1, B,
                    self.num_actions, int(self.use_lstm), self.PRECISIONS[self.precision], p(ws), p(grads_out),
                    _lib.stream_ptr()),
                "tb_atarinet_backward")
        else:
            _lib.check(
                _lib.lib().tb_atarinet_backward_phase(
                    p(g_logits), p(g_baseline), p(notdone) if self.use_lstm else None, p(self._flat), T1, B,
                    self.num_actions, int(self.use_lstm), self.PRECISIONS[self.precision], p(ws), p(grads_out), int(phase),
                    _lib.stream_ptr()),
                "tb_atarinet_backward_phase")

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
            inputs["frame"], inputs["reward"], notdone, inputs["last_action"], h0, c0)
        self._saved_notdone = notdone
        return LearnerOutputs(logits, baseline, (hN, cN) if self.use_lstm else tuple())

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
        frame = inputs["frame"]
        T, B = frame.shape[:2]
        notdone = self._notdone(inputs["done"]) if self.use_lstm else None
        h0, c0 = core_state if self.use_lstm else (None, None)
        params = [v[0] for v in self._views]
        if torch.is_grad_enabled() and any(q.requires_grad for q in params):
            logits, baseline, hN, cN = _AtariNetFunction.apply(
                self, frame, inputs["reward"], notdone, inputs["last_action"], h0, c0, *params)
        else:
            logits, baseline, hN, cN = self._launch_forward(frame, inputs["reward"], notdone, inputs["last_action"], h0, c0)
        if self.training:
            action = self._sample(logits, inputs)
        else:
            action = torch.argmax(logits.detach().view(T * B, self.num_actions), dim=1)  # don't sample when testing
        out = dict(policy_logits=logits, baseline=baseline, action=action.view(T, B))
        return out, ((hN, cN) if self.use_lstm else tuple())




def resnet_param_spec(num_actions, use_lstm):
    """State_dict order/shapes of the reference's polybeast_learner.Net (pl:134-204, BASELINE.md section 5)."""
    spec = []
    cin = 4
    for i, ch in enumerate([16, 32, 32]):
        spec += [("feat_convs.%d.0.weight" % i, (ch, cin, 3, 3)), ("feat_convs.%d.0.bias" % i, (ch,))]
        cin = ch
    for blk in ("resnet1", "resnet2"):
        for i, ch in enumerate([16, 32, 32]):
            for j in (1, 3):
                spec += [("%s.%d.%d.weight" % (blk, i, j), (ch, ch, 3, 3)), ("%s.%d.%d.bias" % (blk, i, j), (ch,))]
    spec += [("fc.weight", (256, 3872)), ("fc.bias", (256,))]
    head_in = 257
    if use_lstm:
        spec += [("core.weight_ih_l0", (1024, 257)), ("core.weight_hh_l0", (1024, 256)),
                 ("core.bias_ih_l0", (1024,)), ("core.bias_hh_l0", (1024,))]
        head_in = 256
    spec += [("policy.weight", (num_actions, head_in)), ("policy.bias", (num_actions,)),
             ("baseline.weight", (1, head_in)), ("baseline.bias", (1,))]
    return spec


class _ResNetFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, module, frame, reward, notdone, h0, c0, *params):
        logits, baseline, hN, cN = module._launch_forward(frame, reward, notdone, h0, c0)
        ctx.module, ctx.notdone, ctx.frame = module, notdone, frame
        ctx.mark_non_differentiable(hN, cN)
        return logits, baseline, hN, cN

    @staticmethod
    def backward(ctx, g_logits, g_baseline, _ghn, _gcn):
        module = ctx.module
        T1, B = ctx.frame.shape[:2]
        dev = module._flat.device
        if g_logits is None:
            g_logits = torch.zeros(T1, B, module.num_actions, device=dev)
        if g_baseline is None:
            g_baseline = torch.zeros(T1, B, device=dev)
        grads = torch.empty_like(module._flat)
        module._launch_backward(ctx.frame, g_logits.contiguous(), g_baseline.contiguous(), ctx.notdone, grads)
        return (None,) * 6 + tuple(grads[off:off + n].view(shape) for _, off, n, shape in module._views)


class ResNet(FlatParamModule):
    """CUDA IMPALA ResNet (reference polybeast_learner.py:134-266 `Net`): three sections of
    conv3x3 + maxpool3/2 + two residual blocks, fc 3872->256, cat[reward], optional LSTM(257->256), heads.
    forward(inputs, core_state) returns ((action, policy_logits, baseline), core_state) like the reference."""

    PRECISIONS = {"fp32": 0, "bf16": 1, "bf16x3": 2}

    def __init__(self, num_actions, use_lstm=False, device=None, precision=None):
        super().__init__()
        import os
        self.num_actions = num_actions
        self.use_lstm = use_lstm
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")
        self._build_flat(resnet_param_spec(num_actions, use_lstm), device)
        self._fix_module_names()
        self.reset_parameters_like_torch()
        if use_lstm:
            self.core.num_layers, self.core.hidden_size, self.core.input_size = 1, 256, 257
        # patch-matrix GEMMs: "bf16x3" (default: split-bf16 tensor-core products over fp32 activations, parity-green),
        # "fp32" (SIMT) or "bf16" (single-plane operands and activations, not parity-grade)
        self.precision = precision or os.environ.get("TB_RESNET_PRECISION", "bf16x3")
        if self.precision not in self.PRECISIONS:
            raise _lib.TorchBeastB200Error("ResNet precision must be 'fp32', 'bf16' or 'bf16x3'")
        self._ws = None
        self._ws_key = None
        count = _lib.lib().tb_resnet_param_count(num_actions, int(use_lstm))
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
            nbytes = _lib.lib().tb_resnet_workspace_bytes(T1, B, self.num_actions, int(self.use_lstm),
                                                          self.PRECISIONS[self.precision])
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self._flat.device)
            self._ws_key = key
        return self._ws

    def _launch_forward(self, frame, reward, notdone, h0, c0):
        _lib.require_cuda(frame, reward, self._flat)
        T1, B = frame.shape[:2]
        if frame.dtype != torch.uint8 or tuple(frame.shape[2:]) != (4, 84, 84):
            raise _lib.TorchBeastB200Error("frame must be uint8 [T,B,4,84,84], got %s %r" % (frame.dtype, tuple(frame.shape)))
        dev = self._flat.device
        frame = frame.contiguous()
        reward = reward.to(torch.float32).contiguous()
        logits = torch.empty(T1, B, self.num_actions, dtype=torch.float32, device=dev)
        baseline = torch.empty(T1, B, dtype=torch.float32, device=dev)
        if self.use_lstm:
            hN = torch.empty(1, B, 256, dtype=torch.float32, device=dev)
            cN = torch.empty_like(hN)
            h0 = h0.to(torch.float32).contiguous(); c0 = c0.to(torch.float32).contiguous()
        else:
            hN = cN = torch.empty(0, device=dev)
            h0 = c0 = notdone = None
        p = _lib.ptr
        _lib.check(
            _lib.lib().tb_resnet_forward(
                p(frame), p(reward), p(notdone), p(h0), p(c0), p(self._flat), T1, B, self.num_actions, int(self.use_lstm),
                self.PRECISIONS[self.precision], p(self._workspace(T1, B)), p(logits), p(baseline),
                p(hN) if self.use_lstm else None, p(cN) if self.use_lstm else None, _lib.stream_ptr()),
            "tb_resnet_forward")
        return logits, baseline, hN, cN

    def _launch_backward(self, frame, g_logits, g_baseline, notdone, grads_out):
        T1, B = g_baseline.shape
        p = _lib.ptr
        _lib.check(
            _lib.lib().tb_resnet_backward(
                p(frame.contiguous()), p(g_logits), p(g_baseline), p(notdone) if self.use_lstm else None, p(self._flat),
                T1, B, self.num_actions, int(self.use_lstm), self.PRECISIONS[self.precision], p(self._workspace(T1, B)),
                p(grads_out), _lib.stream_ptr()),
            "tb_resnet_backward")

    @torch.no_grad()
    def learner_forward(self, inputs, core_state=()):
        notdone = (~inputs["done"]).float().contiguous() if self.use_lstm else None
        h0, c0 = core_state if self.use_lstm else (None, None)
        logits, baseline, hN, cN = self._launch_forward(inputs["frame"], inputs["reward"], notdone, h0, c0)
        self._saved = (inputs["frame"], notdone)
        return LearnerOutputs(logits, baseline, (hN, cN) if self.use_lstm else tuple())

    @torch.no_grad()
    def learner_backward(self, grad_logits, grad_baseline):
        fg = self.attach_grads()
        frame, notdone = self._saved
        self._launch_backward(frame, grad_logits, grad_baseline, notdone, fg)
        return fg

    def forward(self, inputs, core_state=()):
        frame = inputs["frame"]
        T, B = frame.shape[:2]
        notdone = (~inputs["done"]).float().contiguous() if self.use_lstm else None
        h0, c0 = core_state if self.use_lstm else (None, None)
        params = [v[0] for v in self._views]
        if torch.is_grad_enabled() and any(q.requires_grad for q in params):
            logits, baseline, hN, cN = _ResNetFunction.apply(self, frame, inputs["reward"], notdone, h0, c0, *params)
        else:
            logits, baseline, hN, cN = self._launch_forward(frame, inputs["reward"], notdone, h0, c0)
        if self.training:
            action = self._sample(logits, inputs)
        else:
            action = torch.argmax(logits.detach().view(T * B, self.num_actions), dim=1)  # don't sample when testing
        return (action.view(T, B), logits, baseline), ((hN, cN) if self.use_lstm else tuple())


Net = AtariNet
