"""GPU: tb_sample_actions_dev_f32, the sampler entry that reads (seed, step) from device memory, against the by-value
entry tb_sample_actions_f32, launched directly and captured in a CUDA graph whose step is updated between replays."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SEED = 2 ** 64 - 0x1234567  # the top bit set: the seed is taken as its two's-complement bits
STEP = 2 ** 32 - 2          # with T = 3 the counter crosses a 32-bit word


def _logits(T, B, A, seed):
    rs = np.random.RandomState(seed)
    x = (3 * rs.randn(T, B, A)).astype(np.float32)
    x[rs.rand(T, B, A) < 0.1] = -np.inf
    return torch.from_numpy(x).cuda()


def _pair(seed, step):
    from torchbeast_b200.acting import _as_int64
    return torch.tensor([_as_int64(seed), _as_int64(step)], dtype=torch.int64).cuda()


@pytest.mark.parametrize("with_ids", [False, True])
@pytest.mark.parametrize("T", [1, 3])
@pytest.mark.parametrize("A", [2, 6, 7, 18, 100])
def test_device_entry_equals_by_value_entry(A, T, with_ids):
    from torchbeast_b200.acting import _DeviceStepSampler
    from torchbeast_b200.sampling import ActionSampler
    B = 4099
    x = _logits(T, B, A, seed=A * 10 + T)
    ids = torch.randint(-2 ** 62, 2 ** 62, (B,), generator=torch.Generator().manual_seed(A)).cuda() if with_ids else None
    want = ActionSampler(SEED, STEP).sample(x, ids)
    got = _DeviceStepSampler(_pair(SEED, STEP)).sample(x, ids)
    assert got.dtype == torch.int64 and tuple(got.shape) == (T, B)
    assert torch.equal(got, want)


@pytest.mark.parametrize("with_ids", [False, True])
def test_captured_launch_samples_at_the_published_step(with_ids):
    from torchbeast_b200.acting import _as_int64, _DeviceStepSampler
    from torchbeast_b200.sampling import ActionSampler
    T, B, A = 3, 512, 18
    x = _logits(T, B, A, seed=5)
    ids = torch.arange(B, dtype=torch.int64).cuda() * 1009 - 7 if with_ids else None
    seed_step = torch.zeros(2, dtype=torch.int64, device="cuda")
    s = _DeviceStepSampler(seed_step)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        s.sample(x, ids)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        actions = s.sample(x, ids)
    seen = []
    for seed, step in ((SEED, 0), (SEED, STEP), (SEED, STEP + 1), (3, 2 ** 64 - 1), (3, 17)):
        seed_step.copy_(torch.tensor([_as_int64(seed), _as_int64(step)]))
        g.replay()
        want = ActionSampler(seed, step).sample(x, ids)
        assert torch.equal(actions, want), (seed, step)
        seen.append(actions.clone())
    assert not torch.equal(seen[0], seen[1])  # the replay really follows the step
