"""GPU: the bf16x3 two-layer wavefront kernels, which run as 2-CTA clusters where each CTA of a pair loads one 16-row half
of every exchanged tile and multicasts it to both.  Same check as test_lstm_abi_gpu.test_lstm_abi_vs_torch, at shapes
that sit on the edges of that pairing."""
import pytest

from tests.test_lstm_abi_gpu import test_lstm_abi_vs_torch as _abi_vs_torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("T1,B,In,H,layers,precision", [
    (81, 32, 519, 519, 2, "bf16x3"),   # bench.py's shape: 130 forward CTAs, 2 x 66 backward CTAs (one padding CTA per role)
    (2, 17, 519, 519, 2, "bf16x3"),    # rank 1's row half holds one real row, the rest zero-filled
    (1, 16, 519, 519, 2, "bf16x3"),    # rank 1's row half entirely zero-filled; T1 = 1 like the acting forward
    (5, 32, 500, 500, 2, "bf16x3"),    # 125 forward CTAs: one padding CTA completes the last pair
])
def test_lstm_cluster_pairing_vs_torch(T1, B, In, H, layers, precision):
    _abi_vs_torch(T1, B, In, H, layers, precision)
