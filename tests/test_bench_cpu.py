"""Host-side pieces of bench.py that can be checked without a GPU: the clock sampler's parsing / time-window filter,
--dump-outputs (identical files on identical inputs, sampling, size limit) and argument checks."""
import datetime
import importlib.util
import os
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bench():
    argv = sys.argv
    sys.argv = ["bench.py"]
    try:
        spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        sys.argv = argv
    return mod


class _Proc:
    def terminate(self):
        pass


class _Thread:
    def join(self, timeout=None):
        pass


def _row(now, dt, mhz, power_cap="Not Active"):
    ts = datetime.datetime.fromtimestamp(now + dt).strftime("%Y/%m/%d %H:%M:%S.%f")[:-3]
    return [ts, str(mhz), "1965", "500.0", "Not Active", "Not Active", "Not Active", power_cap]


def test_clock_sampler_filters_to_the_timed_region():
    b = _bench()
    now = time.time()
    s = b.ClockSampler(0)
    s.proc, s.thread = _Proc(), _Thread()
    s.rows = [_row(now, -1.0, 1000), _row(now, 0.01, 1965), _row(now, 0.05, 1960, "Active"), _row(now, 0.3, 900)]
    out = s.stop(now, now + 0.1)
    assert out["samples"] == 2 and out["in_timed_region"] and out["sm_mhz"] == 1962.5
    assert out["reasons"] == ["sw_power_cap"] and out["sm_max_mhz"] == 1965.0


def test_clock_sampler_survives_garbage():
    b = _bench()
    now = time.time()
    s = b.ClockSampler(0)
    s.proc, s.thread = _Proc(), _Thread()
    s.rows = [["garbage"], ["x", "y"]]
    assert s.stop(now, now + 0.1) is None
    s.proc = _Proc()
    s.rows = [["not a timestamp", "1950", "1965", "1", "Not Active", "Not Active", "Not Active", "Not Active"]]
    out = s.stop(now, now + 0.1)
    assert out["samples"] == 1 and out["in_timed_region"] is False


def _dump_case(b):
    import collections

    import torch

    g = torch.Generator().manual_seed(0)
    VT = collections.namedtuple("VT", "vs grad_logits note")
    out = dict(losses=torch.randn(4, generator=g),
               vtrace=VT(torch.randn(80, 32, generator=g), torch.randn(81, 32, 6, generator=g), "not an array"))
    model = types.SimpleNamespace(flat_params=torch.randn(b.DUMP_SAMPLE + 1000, generator=g))
    return out, model


def test_dump_outputs_writes_the_same_files_twice(tmp_path):
    import numpy as np

    b = _bench()
    out, model = _dump_case(b)
    for d in ("a", "b"):
        b.dump_outputs(str(tmp_path / d), out, model)
    names = sorted(os.listdir(tmp_path / "a"))
    assert names == sorted(os.listdir(tmp_path / "b"))
    assert names == ["grad_logits.npy", "losses.npy", "params.npy", "params_sample_index.npy", "vs.npy"]
    for n in names:
        x, y = np.load(tmp_path / "a" / n), np.load(tmp_path / "b" / n)
        assert x.dtype in (np.float32, np.float64) and np.array_equal(x, y), n
    # small arrays whole, the large one as a sample of its own elements at the stored indices
    np.testing.assert_array_equal(np.load(tmp_path / "a" / "vs.npy"), out["vtrace"].vs.numpy().reshape(-1))
    idx = np.load(tmp_path / "a" / "params_sample_index.npy").astype(np.int64)
    assert idx.size == b.DUMP_SAMPLE and np.all(np.diff(idx) > 0)
    np.testing.assert_array_equal(np.load(tmp_path / "a" / "params.npy"), model.flat_params.numpy()[idx])


def test_dump_outputs_refuses_more_than_the_limit(tmp_path):
    b = _bench()
    out, model = _dump_case(b)
    b.DUMP_LIMIT = 1024
    try:
        b.dump_outputs(str(tmp_path / "d"), out, model)
    except SystemExit as e:
        assert "more than" in str(e)
    else:
        raise AssertionError("no error above the limit")
    assert not (tmp_path / "d").exists()


def test_steps_must_be_positive():
    import subprocess

    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "0"], capture_output=True, text=True)
    assert r.returncode != 0 and "--steps must be at least 1" in r.stderr
