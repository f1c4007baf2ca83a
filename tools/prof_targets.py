"""Small driver for ncu captures: one bf16 LSTM learn step at the bench size, then the V-trace scan
and the fused loss kernel on a wide batch (HBM-bound regime)."""
import os, sys, types
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import synthetic_host_batch, flags_ns
from torchbeast_b200 import _lib, learner, monobeast, optim

T, B, A = 80, 32, 6
model = monobeast.AtariNet((4, 84, 84), A, True)
actor = monobeast.AtariNet((4, 84, 84), A, True)
opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
batch = {k: v.cuda() for k, v in synthetic_host_batch(T, B, A, 1, False).items()}
state = model.initial_state(B)
for _ in range(2):
    learner.learn_step(flags_ns(T, B), model, actor, batch, state, opt, None, stats_sync=False)
torch.cuda.synchronize()
lib, p, st = _lib.lib(), _lib.ptr, _lib.stream_ptr()
g = torch.Generator(device="cuda").manual_seed(0)
t, b = 80, 1 << 20
lr = 0.5 * torch.randn(t, b, device="cuda", generator=g); dc = torch.full((t, b), 0.99, device="cuda")
rw = torch.randn(t, b, device="cuda", generator=g).clamp(-1, 1); va = torch.randn(t, b, device="cuda", generator=g)
bs = torch.randn(b, device="cuda", generator=g); vs = torch.empty_like(va); pg = torch.empty_like(va)
for _ in range(2):
    lib.tb_vtrace_from_importance_weights_f32(p(lr), p(dc), p(rw), p(va), p(bs), t, b, 1.0, 1.0, p(vs), p(pg), st)
b2 = 1 << 18
bl = torch.randn(t, b2, A, device="cuda", generator=g); tl = torch.randn(t, b2, A, device="cuda", generator=g)
ac = torch.randint(0, A, (t, b2), device="cuda", generator=g); dn = (torch.rand(t, b2, device="cuda", generator=g) < 0.01).view(torch.uint8)
outs = [torch.empty(t, b2, device="cuda") for _ in range(5)]
losses = torch.empty(4, device="cuda"); gl = torch.empty(t + 1, b2, A, device="cuda"); gv = torch.empty(t + 1, b2, device="cuda")
for _ in range(2):
    lib.tb_impala_loss_f32(p(bl), p(tl), p(ac), p(rw[:, :b2].contiguous()), p(dn), None, p(va[:, :b2].contiguous()), p(bs[:b2].contiguous()),
                           t, b2, A, 0.99, 0.5, 0.0006, 1, 1.0, 1.0, *[None] * 5, 0, *[None] * 4, *[p(o) for o in outs], p(losses),
                           p(gl), p(gv), 1, p(_lib.workspace()), st)
torch.cuda.synchronize()
print("done", float(losses[3]))
