"""Two eager learn steps of the IMPALA ResNet (+LSTM) at T=80, B=8 (one GPU's shard of BASELINE configs[3]) - the target of
ncu captures (ncu -k regex:sw_conv ... python tools/resnet_step.py)."""
import sys
import torch
sys.path.insert(0, ".")
from bench import synthetic_host_batch, flags_ns
from torchbeast_b200 import learner, optim, polybeast_learner
T, B, A = 80, 8, 6
model = polybeast_learner.Net(A, True); actor = polybeast_learner.Net(A, True)
opt = optim.RMSprop(model, lr=0.00048, eps=0.01, alpha=0.99)
batch = {k: v.cuda() for k, v in synthetic_host_batch(T, B, A, 1, False).items()}
state = model.initial_state(B)
for _ in range(2):
    stats = learner.learn_step(flags_ns(T, B), model, actor, batch, state, opt, None, stats_sync=True)
torch.cuda.synchronize()
print("ok", stats["total_loss"])
