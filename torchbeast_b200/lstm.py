"""Stacked LSTM over an unroll with per-step done-reset, on its own (C ABI tb_lstm_{forward,backward}).

The recurrence the reference spells as a Python loop of seq_len-1 `nn.LSTM` calls (monobeast.py:603-611,
polybeast_learner.py:241-249), with layers / batch / unroll / input size as free parameters and any hidden size up to
MAX_HIDDEN - BASELINE.json configs[4] stresses it at T=600, B=128, H=512.  Above MAX_HIDDEN (TB_LSTM_MAX_HIDDEN in
include/torchbeast_b200.h) the backward's step kernel cannot hold a row of H in shared memory, so every call, the plan
included, raises.  `LSTM` keeps torch.nn.LSTM's parameter names and shapes, so
`lstm.load_state_dict(torch_lstm.state_dict())` works, and `lstm(input, (h0, c0))` is an autograd forward with
torch.nn.LSTM's sequence-first shapes plus an optional done-reset mask."""
import ctypes

import torch
from torch import nn
from torch.autograd.function import once_differentiable

from torchbeast_b200 import _lib

PRECISIONS = {"fp32": 0, "bf16": 1, "bf16x3": 2}
# recurrence kinds, numbered as TB_LSTM_* in include/torchbeast_b200.h
KINDS = ("step", "persistent", "persistent_mma", "cluster", "wave_bf16", "wave_split")
MAX_HIDDEN = 700  # TB_LSTM_MAX_HIDDEN


class _LSTMFunction(torch.autograd.Function):
    """One unroll through tb_lstm_forward, backpropagated by tb_lstm_backward_state.  Each call allocates its own workspace
    and keeps it, with its inputs and parameters, in ctx: forwards may be backpropagated in any order, and a chain of
    unrolls whose states feed each other (truncated BPTT) backpropagates through all of them."""

    @staticmethod
    def forward(ctx, module, x, notdone, h0, c0, *params):
        T1, B = x.shape[:2]
        H, L, prec = module.hidden_size, module.num_layers, PRECISIONS[module.precision]
        x, notdone = x.float().contiguous(), notdone.float().contiguous()
        h0, c0 = h0.float().contiguous(), c0.float().contiguous()
        params = [q.float().contiguous() for q in params]
        ws = torch.empty(_lib.lib().tb_lstm_workspace_bytes(T1, B, module.input_size, H, L, prec), dtype=torch.uint8,
                         device=x.device)
        y = torch.empty(T1, B, H, device=x.device)
        hN, cN = torch.empty(L, B, H, device=x.device), torch.empty(L, B, H, device=x.device)
        p, arr = _lib.ptr, lambda ts: ctypes.cast(LSTM._ptr_array(ts), ctypes.c_void_p)
        _lib.check(_lib.lib().tb_lstm_forward(p(x), p(notdone), p(h0), p(c0), arr(params), T1, B, module.input_size, H, L,
                                              prec, p(ws), p(y), p(hN), p(cN), _lib.stream_ptr()), "tb_lstm_forward")
        ctx.save_for_backward(x, notdone, ws, *params)
        ctx.dims = (T1, B, module.input_size, H, L, prec)
        ctx.set_materialize_grads(False)
        return y, hN, cN

    @staticmethod
    @once_differentiable
    def backward(ctx, dy, dhN, dcN):
        x, notdone, ws, *params = ctx.saved_tensors
        T1, B, In, H, L, prec = ctx.dims
        dy = torch.zeros(T1, B, H, device=x.device) if dy is None else dy.float().contiguous()
        dhN = None if dhN is None else dhN.float().contiguous()
        dcN = None if dcN is None else dcN.float().contiguous()
        dx = torch.empty_like(x)
        grads = [torch.empty_like(q) for q in params]
        dh0 = torch.empty(L, B, H, device=x.device) if ctx.needs_input_grad[3] else None
        dc0 = torch.empty(L, B, H, device=x.device) if ctx.needs_input_grad[4] else None
        p, arr = _lib.ptr, lambda ts: ctypes.cast(LSTM._ptr_array(ts), ctypes.c_void_p)
        _lib.check(_lib.lib().tb_lstm_backward_state(p(dy), p(x), p(notdone), arr(params), arr(grads), T1, B, In, H, L, prec,
                                                     p(ws), p(dx), p(dhN), p(dcN), p(dh0), p(dc0), _lib.stream_ptr()),
                   "tb_lstm_backward_state")
        return (None, dx, None, dh0, dc0, *grads)


class LSTM(nn.Module):
    def __init__(self, input_size, hidden_size, num_layers=1, device=None, precision="fp32"):
        super().__init__()
        if num_layers < 1:
            raise _lib.TorchBeastB200Error("torchbeast_b200.lstm.LSTM: num_layers must be >= 1, got %r" % (num_layers,))
        self.input_size, self.hidden_size, self.num_layers = input_size, hidden_size, num_layers
        self.precision = precision
        dev = device or (torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else "cpu")
        bound = 1.0 / hidden_size ** 0.5
        for l in range(num_layers):
            in_l = input_size if l == 0 else hidden_size
            for name, shape in (("weight_ih", (4 * hidden_size, in_l)), ("weight_hh", (4 * hidden_size, hidden_size)),
                                ("bias_ih", (4 * hidden_size,)), ("bias_hh", (4 * hidden_size,))):
                self.register_parameter("%s_l%d" % (name, l), nn.Parameter((torch.rand(shape, device=dev) * 2 - 1) * bound))
        self._ws = None

    def _plist(self):
        return [getattr(self, "%s_l%d" % (n, l)) for l in range(self.num_layers) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]

    def _workspace(self, T1, B):
        n = _lib.lib().tb_lstm_workspace_bytes(T1, B, self.input_size, self.hidden_size, self.num_layers, PRECISIONS[self.precision])
        if self._ws is None or self._ws.numel() < n or self._ws.device != self.weight_ih_l0.device:
            self._ws = torch.empty(n, dtype=torch.uint8, device=self.weight_ih_l0.device)
        return self._ws

    def plan(self, B):
        """(forward kind, backward kind): the recurrence implementations a batch of B runs on the current device (1 or 2
        layers; plan_layers takes any depth)."""
        fwd, bwd = ctypes.c_int(), ctypes.c_int()
        _lib.check(_lib.lib().tb_lstm_plan(B, self.input_size, self.hidden_size, self.num_layers, PRECISIONS[self.precision],
                                           ctypes.byref(fwd), ctypes.byref(bwd)), "tb_lstm_plan")
        return KINDS[fwd.value], KINDS[bwd.value]

    def plan_layers(self, B):
        """[(forward kind, backward kind)] per layer.  The stack runs as segments of two layers (the top one alone when
        num_layers is odd), each planned on its own; both layers of a wavefront segment report its kind."""
        L = self.num_layers
        fwd, bwd = (ctypes.c_int * L)(), (ctypes.c_int * L)()
        _lib.check(_lib.lib().tb_lstm_plan_layers(B, self.input_size, self.hidden_size, L, PRECISIONS[self.precision],
                                                  ctypes.cast(fwd, ctypes.c_void_p), ctypes.cast(bwd, ctypes.c_void_p)),
                   "tb_lstm_plan_layers")
        return [(KINDS[f], KINDS[b]) for f, b in zip(fwd, bwd)]

    @staticmethod
    def _ptr_array(tensors):
        arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
        return arr

    def forward(self, input, hx=None, notdone=None):
        """input [T, B, In], hx = (h0, c0) each [layers, B, H] (None: zeros), notdone [T, B] (None: no reset) ->
        output [T, B, H], (h_n, c_n) each [layers, B, H].  Step t first multiplies the state by notdone[t]; without
        notdone this is torch.nn.LSTM.  Differentiable with respect to input, h0, c0 and every parameter (once)."""
        if input.dim() != 3 or input.shape[2] != self.input_size:
            raise _lib.TorchBeastB200Error("LSTM: input must be [T, B, %d], got %s" % (self.input_size, tuple(input.shape)))
        T, B = input.shape[:2]
        state_shape = (self.num_layers, B, self.hidden_size)
        if hx is not None and (len(hx) != 2 or any(tuple(s.shape) != state_shape for s in hx)):
            raise _lib.TorchBeastB200Error("LSTM: hx must be (h0, c0), each %s" % (state_shape,))
        if notdone is not None and tuple(notdone.shape) != (T, B):
            raise _lib.TorchBeastB200Error("LSTM: notdone must be [%d, %d], got %s" % (T, B, tuple(notdone.shape)))
        _lib.require_cuda(input, notdone, *(hx or ()))
        if hx is None:
            hx = (torch.zeros(state_shape, device=input.device), torch.zeros(state_shape, device=input.device))
        if notdone is None:
            notdone = torch.ones(T, B, device=input.device)
        y, hN, cN = _LSTMFunction.apply(self, input, notdone, hx[0], hx[1], *self._plist())
        return y, (hN, cN)

    @torch.no_grad()
    def forward_unroll(self, x, notdone, state):
        """x [T1, B, In], notdone [T1, B] float (1 - done), state (h0, c0) each [layers, B, H] -> y [T1, B, H], (hN, cN)."""
        _lib.require_cuda(x, notdone, *state)
        T1, B = x.shape[:2]
        H, L = self.hidden_size, self.num_layers
        x = x.float().contiguous(); notdone = notdone.float().contiguous()
        h0, c0 = state[0].float().contiguous(), state[1].float().contiguous()
        y = torch.empty(T1, B, H, device=x.device)
        hN, cN = torch.empty(L, B, H, device=x.device), torch.empty(L, B, H, device=x.device)
        params = [p.detach().contiguous() for p in self._plist()]
        self._saved = (x, notdone, params)
        p = _lib.ptr
        _lib.check(_lib.lib().tb_lstm_forward(p(x), p(notdone), p(h0), p(c0), ctypes.cast(self._ptr_array(params), ctypes.c_void_p),
                                              T1, B, self.input_size, H, L, PRECISIONS[self.precision], p(self._workspace(T1, B)),
                                              p(y), p(hN), p(cN), _lib.stream_ptr()), "tb_lstm_forward")
        return y, (hN, cN)

    @torch.no_grad()
    def backward_unroll(self, dy):
        """dy [T1, B, H] -> dx [T1, B, In]; parameter gradients are written into .grad of every parameter."""
        x, notdone, params = self._saved
        T1, B = x.shape[:2]
        dy = dy.float().contiguous()
        dx = torch.empty_like(x)
        grads = [torch.empty_like(q) for q in params]
        p = _lib.ptr
        _lib.check(_lib.lib().tb_lstm_backward(p(dy), p(x), p(notdone), ctypes.cast(self._ptr_array(params), ctypes.c_void_p),
                                               ctypes.cast(self._ptr_array(grads), ctypes.c_void_p), T1, B, self.input_size,
                                               self.hidden_size, self.num_layers, PRECISIONS[self.precision],
                                               p(self._workspace(T1, B)), p(dx), _lib.stream_ptr()), "tb_lstm_backward")
        for q, g in zip(self._plist(), grads):
            q.grad = g
        return dx
