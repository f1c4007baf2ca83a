"""Stacked LSTM over an unroll with per-step done-reset, on its own (C ABI tb_lstm_{forward,backward}).

The recurrence the reference spells as a Python loop of seq_len-1 `nn.LSTM` calls (monobeast.py:603-611,
polybeast_learner.py:241-249), with hidden size / layers / batch / unroll as free parameters - BASELINE.json configs[4]
stresses it at T=600, B=128, H=512.  `LSTM` keeps torch.nn.LSTM's parameter names and shapes, so
`lstm.load_state_dict(torch_lstm.state_dict())` works."""
import ctypes

import torch
from torch import nn

from torchbeast_b200 import _lib

PRECISIONS = {"fp32": 0, "bf16": 1, "bf16x3": 2}
# recurrence kinds, numbered as TB_LSTM_* in include/torchbeast_b200.h
KINDS = ("step", "persistent", "persistent_mma", "cluster", "wave_bf16", "wave_split")


class LSTM(nn.Module):
    def __init__(self, input_size, hidden_size, num_layers=1, device=None, precision="fp32"):
        super().__init__()
        if num_layers not in (1, 2):
            raise _lib.TorchBeastB200Error("torchbeast_b200.lstm.LSTM supports 1 or 2 layers")
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
        """(forward kind, backward kind): the recurrence implementations a batch of B runs on the current device."""
        fwd, bwd = ctypes.c_int(), ctypes.c_int()
        _lib.check(_lib.lib().tb_lstm_plan(B, self.input_size, self.hidden_size, self.num_layers, PRECISIONS[self.precision],
                                           ctypes.byref(fwd), ctypes.byref(bwd)), "tb_lstm_plan")
        return KINDS[fwd.value], KINDS[bwd.value]

    @staticmethod
    def _ptr_array(tensors):
        arr = (ctypes.c_void_p * len(tensors))(*[t.data_ptr() for t in tensors])
        return arr

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
