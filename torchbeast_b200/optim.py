"""Flat-buffer optimizers with fused global-norm clipping: RMSprop, Adam and AdamW.

Drop-ins for `torch.optim.RMSprop(model.parameters(), lr, momentum, eps, alpha)` as the
reference builds it (/root/reference/torchbeast/monobeast.py:388-394,
polybeast_learner.py:472-478), and for `torch.optim.Adam` / `AdamW`, over a FlatParamModule:
same constructor arguments, `param_groups[0]["lr"]` is honoured so
`torch.optim.lr_scheduler.LambdaLR` works unchanged, `state_dict()` carries the per-parameter
state entries torch's optimizers write, and `load_state_dict()` accepts torch's.
"""
import numpy as np
import torch

from torchbeast_b200 import _lib


class FusedOptimizer(torch.optim.Optimizer):
    """Base of the flat-buffer optimizers; what learner.optimizer_step and GraphedLearner rely on:

    * `step(max_grad_norm=None)`: clip_grad_norm_ + the update on the model's flat buffers, launches only, no host sync;
    * `flat_state()`: the device tensors a step updates besides the parameters (state buffers, device step counter);
      `snapshot()` / `restore(snapshot)` copy them (and any host-side counter) out and back;
    * `lr_from_device` / `sync_lr_to_device()`: read the learning rate from a device scalar, so a captured CUDA graph
      sees scheduler updates;
    * `step(..., hparams_dev=block)`: read max_norm and the other values of param_groups[0] from a device tb_hparams
      block (learner.HPARAMS) instead, so a captured graph follows changes to them; `hparams()` gives those values,
      checked as the host entry point checks them, and `structure()` the values that choose a kernel or a buffer.

    Subclasses name their flat buffers in `_buffers()` (per-parameter state key -> buffer or None), set the
    per-parameter "step" entry in `_set_step_entry` and launch their update in `_update`.
    """

    def __init__(self, model, defaults):
        if not hasattr(model, "flat_params"):
            raise _lib.TorchBeastB200Error(
                "torchbeast_b200.optim.%s needs a FlatParamModule (e.g. AtariNet)" % type(self).__name__)
        self.model = model
        super().__init__(list(model.parameters()), defaults)
        flat = model.flat_params
        self._sumsq = torch.zeros(1, dtype=torch.float32, device=flat.device)
        self.grad_norm = torch.zeros(1, dtype=torch.float32, device=flat.device)
        # learning rate as a device scalar: lets a captured CUDA graph see scheduler updates
        self._lr_dev = torch.full((1,), float(defaults["lr"]), dtype=torch.float32, device=flat.device)
        self.lr_from_device = False

    def add_param_group(self, param_group):
        if self.param_groups:
            raise _lib.TorchBeastB200Error(
                "torchbeast_b200.optim.%s steps one flat buffer: a second param group is not supported" %
                type(self).__name__)
        super().add_param_group(param_group)

    def _buffers(self):
        raise NotImplementedError

    def _set_step_entry(self, st):
        raise NotImplementedError

    def _set_loaded_step(self, steps):
        raise NotImplementedError

    def _update(self, flat, grad, max_norm, lr_device, stream, hparams_dev=None):
        raise NotImplementedError

    def hparams(self):
        raise NotImplementedError

    def structure(self):
        raise NotImplementedError

    def _validate_group(self, group):
        pass

    def flat_state(self):
        return [b for b in self._buffers().values() if b is not None]

    def snapshot(self):
        return [t.clone() for t in self.flat_state()]

    def restore(self, snapshot):
        for dst, src in zip(self.flat_state(), snapshot):
            dst.copy_(src)

    def _point_state_at_flat(self):
        """Per-parameter views of the flat buffers so state_dict() looks like the torch optimizer's."""
        bufs = self._buffers()
        for p, off, n, shape in self.model._views:
            st = self.state[p]
            self._set_step_entry(st)
            for key, buf in bufs.items():
                if buf is not None:
                    st[key] = buf[off:off + n].view(shape)

    def load_state_dict(self, state_dict):
        """Resume like the reference does (`optimizer.load_state_dict(checkpoint["optimizer_state_dict"])`,
        polybeast_learner.py:535-548): torch replaces the per-parameter state tensors with copies, so the loaded
        values are copied INTO the flat buffers the fused kernel reads and the per-parameter entries are re-pointed
        at them.  Accepts state_dicts of the matching torch.optim optimizer (same per-parameter keys) and of this
        class."""
        for group in state_dict["param_groups"]:
            self._validate_group(group)
        self._loading = True  # torch calls __setstate__ with the loaded copies: keep them until they are in the flat buffers
        try:
            super().load_state_dict(state_dict)
        finally:
            self._loading = False
        steps = 0
        bufs = self._buffers()
        with torch.no_grad():
            for p, off, n, shape in self.model._views:
                st = self.state.get(p, {})
                for key, buf in bufs.items():
                    if buf is not None and st.get(key) is not None:
                        buf[off:off + n].copy_(st[key].reshape(-1))
                if "step" in st:
                    steps = max(steps, int(float(st["step"])))
        self._set_loaded_step(steps)
        self._point_state_at_flat()
        self._lr_dev.fill_(float(self.param_groups[0]["lr"]))

    def __setstate__(self, state):
        super().__setstate__(state)
        if hasattr(self, "model") and not getattr(self, "_loading", False):
            self._point_state_at_flat()

    @torch.no_grad()
    def step(self, closure=None, max_grad_norm=None, hparams_dev=None):
        """clip_grad_norm_(max_grad_norm) (skipped when None) + the update on the flat buffers.  With `hparams_dev` (a
        device tb_hparams block) the kernel reads max_norm and the optimizer's values from it when it runs; the
        structural values (`structure()`) still come from param_groups[0]."""
        if closure is not None:
            raise _lib.TorchBeastB200Error("closure is not supported")
        flat, grad = self.model.flat_params, self.model.attach_grads()
        p, st = _lib.ptr, _lib.stream_ptr()
        _lib.check(_lib.lib().tb_grad_sumsq_f32(p(grad), grad.numel(), p(self._sumsq), p(_lib.workspace()), st),
                   "tb_grad_sumsq_f32")
        self._update(flat, grad, -1.0 if max_grad_norm is None else float(max_grad_norm),
                     p(self._lr_dev) if self.lr_from_device else None, st, hparams_dev)
        return None

    def sync_lr_to_device(self):
        """Publish param_groups[0]['lr'] to the device scalar a captured graph reads (async fill)."""
        self._lr_dev.fill_(float(self.param_groups[0]["lr"]))


class RMSprop(FusedOptimizer):
    """torch.optim.RMSprop on the flat buffers.  The reference's configuration (centered=False, weight_decay=0) runs
    tb_clip_rmsprop_step_f32; centered and weight_decay run tb_clip_rmsprop_ex_step_f32, with a flat grad_avg buffer
    when centered."""

    def __init__(self, model, lr=0.01, alpha=0.99, eps=1e-8, weight_decay=0, momentum=0, centered=False):
        defaults = dict(lr=lr, alpha=alpha, eps=eps, momentum=momentum, weight_decay=weight_decay,
                        centered=bool(centered))
        super().__init__(model, defaults)
        flat = model.flat_params
        self.square_avg = torch.zeros_like(flat)
        self.momentum_buffer = torch.zeros_like(flat) if momentum != 0 else None
        self.grad_avg = torch.zeros_like(flat) if centered else None
        self._steps = 0
        self._point_state_at_flat()

    def _buffers(self):
        return {"square_avg": self.square_avg, "momentum_buffer": self.momentum_buffer, "grad_avg": self.grad_avg}

    def _validate_group(self, group):
        if bool(group.get("centered", False)) != (self.grad_avg is not None):
            raise _lib.TorchBeastB200Error("torchbeast_b200.optim.RMSprop: the state_dict's `centered` differs from "
                                           "this optimizer's; construct it with centered=%s" % group.get("centered"))

    def _set_step_entry(self, st):
        st["step"] = torch.tensor(float(self._steps))

    def _set_loaded_step(self, steps):
        self._steps = steps

    def snapshot(self):
        return super().snapshot(), self._steps

    def restore(self, snapshot):
        super().restore(snapshot[0])
        self._steps = snapshot[1]

    def _entry(self):
        """The host entry point of the current configuration: the default kernel, or the one with the options."""
        if self.grad_avg is None and self.param_groups[0]["weight_decay"] == 0:
            return "tb_clip_rmsprop_step_f32"
        return "tb_clip_rmsprop_ex_step_f32"

    def _momentum_on(self):
        # the host entry points compare the float argument: a momentum that rounds to 0.0f passes no buffer
        return bool(np.float32(self.param_groups[0]["momentum"]) != 0)

    def hparams(self):
        group = self.param_groups[0]
        if self._momentum_on() and self.momentum_buffer is None:
            raise _lib.TorchBeastB200Error("%s failed (1): %s: momentum needs a buffer" % (self._entry(), self._entry()))
        return dict(alpha=group["alpha"], eps=group["eps"], momentum=group["momentum"],
                    weight_decay=group["weight_decay"])

    def structure(self):
        return ("rmsprop", self.grad_avg is not None, self.param_groups[0]["weight_decay"] != 0, self._momentum_on())

    def _update(self, flat, grad, max_norm, lr_device, stream, hparams_dev=None):
        group = self.param_groups[0]
        lib, p = _lib.lib(), _lib.ptr
        if hparams_dev is not None:
            mom = self.momentum_buffer if self._momentum_on() else None
            if self._entry() == "tb_clip_rmsprop_step_f32":
                _lib.check(
                    lib.tb_clip_rmsprop_step_hp_f32(
                        p(flat), p(grad), p(self.square_avg), p(mom), flat.numel(), p(self._sumsq), p(hparams_dev),
                        lr_device, float(group["lr"]), p(self.grad_norm), stream),
                    "tb_clip_rmsprop_step_hp_f32")
            else:
                _lib.check(
                    lib.tb_clip_rmsprop_ex_step_hp_f32(
                        p(flat), p(grad), p(self.square_avg), p(self.grad_avg), p(mom), flat.numel(), p(self._sumsq),
                        p(hparams_dev), lr_device, float(group["lr"]), p(self.grad_norm), stream),
                    "tb_clip_rmsprop_ex_step_hp_f32")
        elif self.grad_avg is None and group["weight_decay"] == 0:
            _lib.check(
                lib.tb_clip_rmsprop_step_f32(
                    p(flat), p(grad), p(self.square_avg), p(self.momentum_buffer), flat.numel(), p(self._sumsq),
                    max_norm, lr_device, float(group["lr"]), float(group["alpha"]), float(group["eps"]),
                    float(group["momentum"]), p(self.grad_norm), stream),
                "tb_clip_rmsprop_step_f32")
        else:
            _lib.check(
                lib.tb_clip_rmsprop_ex_step_f32(
                    p(flat), p(grad), p(self.square_avg), p(self.grad_avg), p(self.momentum_buffer), flat.numel(),
                    p(self._sumsq), max_norm, lr_device, float(group["lr"]), float(group["alpha"]),
                    float(group["eps"]), float(group["weight_decay"]), float(group["momentum"]), p(self.grad_norm),
                    stream),
                "tb_clip_rmsprop_ex_step_f32")
        self._steps += 1

    def state_dict(self):
        for st in self.state.values():  # torch.optim.RMSprop keeps a per-parameter step count in its state_dict
            st["step"] = torch.tensor(float(self._steps))
        return super().state_dict()


class Adam(FusedOptimizer):
    """torch.optim.Adam (non-amsgrad) on the flat buffers: one tb_clip_adam_step_f32 call per step.

    The step count lives on the device (`step_device`, int64, completed steps), so the bias corrections of a captured
    CUDA graph advance on every replay.  Every per-parameter state["step"] is a view of it; state_dict() writes host
    float copies, as torch does.  foreach / capturable / differentiable / fused choose among torch's implementations
    and are accepted and ignored: the param group records torch's defaults for them, so a torch optimizer that loads
    this state_dict runs its own default implementation."""

    def __init__(self, model, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *, foreach=None,
                 maximize=False, capturable=False, differentiable=False, fused=None, decoupled_weight_decay=False):
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                        maximize=maximize, foreach=None, capturable=False, differentiable=False, fused=None,
                        decoupled_weight_decay=bool(decoupled_weight_decay))
        self._validate_group(defaults)
        super().__init__(model, defaults)
        flat = model.flat_params
        self.exp_avg = torch.zeros_like(flat)
        self.exp_avg_sq = torch.zeros_like(flat)
        self.step_device = torch.zeros(1, dtype=torch.int64, device=flat.device)
        self._point_state_at_flat()

    def _validate_group(self, group):
        name = type(self).__name__
        if group.get("amsgrad", False):
            raise _lib.TorchBeastB200Error("torchbeast_b200.optim.%s: amsgrad is not supported" % name)
        if group.get("maximize", False):
            raise _lib.TorchBeastB200Error("torchbeast_b200.optim.%s: maximize is not supported" % name)
        b1, b2 = group["betas"]
        if not 0.0 <= float(group["lr"]):
            raise ValueError("Invalid learning rate: %s" % group["lr"])
        if not 0.0 <= float(group["eps"]):
            raise ValueError("Invalid epsilon value: %s" % group["eps"])
        if not (0.0 <= float(b1) < 1.0 and 0.0 <= float(b2) < 1.0):
            raise ValueError("Invalid beta parameters: %s" % (group["betas"],))
        if not 0.0 <= float(group["weight_decay"]):
            raise ValueError("Invalid weight_decay value: %s" % group["weight_decay"])

    def _buffers(self):
        return {"exp_avg": self.exp_avg, "exp_avg_sq": self.exp_avg_sq}

    def flat_state(self):
        return super().flat_state() + [self.step_device]

    def _set_step_entry(self, st):
        st["step"] = self.step_device[0]

    def _set_loaded_step(self, steps):
        self.step_device.fill_(steps)

    def hparams(self):
        group = self.param_groups[0]
        beta1, beta2 = (float(b) for b in group["betas"])
        if not (0.0 <= beta1 < 1.0 and 0.0 <= beta2 < 1.0):
            raise _lib.TorchBeastB200Error(
                "tb_clip_adam_step_f32 failed (1): tb_clip_adam_step_f32: betas must be in [0, 1)")
        return dict(beta1=beta1, beta2=beta2, eps=group["eps"], weight_decay=group["weight_decay"])

    def structure(self):
        return ("adam", bool(self.param_groups[0]["decoupled_weight_decay"]))

    def _update(self, flat, grad, max_norm, lr_device, stream, hparams_dev=None):
        group = self.param_groups[0]
        beta1, beta2 = group["betas"]
        p = _lib.ptr
        if hparams_dev is not None:
            _lib.check(
                _lib.lib().tb_clip_adam_step_hp_f32(
                    p(flat), p(grad), p(self.exp_avg), p(self.exp_avg_sq), flat.numel(), p(self._sumsq),
                    p(hparams_dev), lr_device, float(group["lr"]), int(bool(group["decoupled_weight_decay"])),
                    p(self.step_device), p(self.grad_norm), stream),
                "tb_clip_adam_step_hp_f32")
            return
        _lib.check(
            _lib.lib().tb_clip_adam_step_f32(
                p(flat), p(grad), p(self.exp_avg), p(self.exp_avg_sq), flat.numel(), p(self._sumsq), max_norm,
                lr_device, float(group["lr"]), float(beta1), float(beta2), float(group["eps"]),
                float(group["weight_decay"]), int(bool(group["decoupled_weight_decay"])), p(self.step_device),
                p(self.grad_norm), stream),
            "tb_clip_adam_step_f32")

    def state_dict(self):
        sd = super().state_dict()
        # one host read of the device counter; a distinct tensor per parameter, as torch's optimizers increment each
        steps = float(self.step_device[0])
        sd["state"] = {k: dict(v, step=torch.tensor(steps)) for k, v in sd["state"].items()}
        return sd


class AdamW(Adam):
    """torch.optim.AdamW (decoupled weight decay) on the flat buffers."""

    def __init__(self, model, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, amsgrad=False, *,
                 maximize=False, foreach=None, capturable=False, differentiable=False, fused=None):
        super().__init__(model, lr, betas, eps, weight_decay, amsgrad, foreach=foreach, maximize=maximize,
                         capturable=capturable, differentiable=differentiable, fused=fused,
                         decoupled_weight_decay=True)
