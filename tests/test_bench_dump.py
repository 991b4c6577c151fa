"""CPU: bench.dump_outputs keeps the files it writes within the limit (headers included), samples the same elements on
every call and writes small outputs whole."""
import os

import numpy as np

import bench


def _dir_bytes(d):
    return sum(os.path.getsize(os.path.join(d, f)) for f in os.listdir(d))


def test_dump_outputs_stays_within_limit_and_is_repeatable(tmp_path):
    rng = np.random.default_rng(0)
    outs = [rng.random((300, 1000)).astype(np.float32), rng.integers(0, 65535, (7, 64, 64)).astype(np.uint16), rng.random(500000)]
    limit = 1_000_000                                  # every share is 333 KB: the first and third output are over it
    a, b = str(tmp_path / "a"), str(tmp_path / "b")
    bench.dump_outputs(a, ("x", "depth"), outs, limit_bytes=limit)
    bench.dump_outputs(b, ("x", "depth"), outs, limit_bytes=limit)
    assert sorted(os.listdir(a)) == ["depth.npy", "out2.npy", "x.npy"]
    assert _dir_bytes(a) <= limit
    for f in os.listdir(a):
        x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        assert x.dtype == np.float32 and np.array_equal(x, y)
    assert np.array_equal(np.load(os.path.join(a, "depth.npy")), outs[1].astype(np.float32))      # under its share: whole
    x = np.load(os.path.join(a, "x.npy"))
    assert x.ndim == 1 and x.size < outs[0].size and np.isin(x, outs[0]).all()
    assert x.size * 4 > 0.95 * (limit / 3)             # the sample uses its share


def test_dump_outputs_default_limit_is_64_mb():
    assert bench.DUMP_LIMIT_BYTES == 64 * 10 ** 6
    # three outputs over their share, the largest case the workloads have: payload + reserved headers fit
    share = (bench.DUMP_LIMIT_BYTES // 3 - bench.NPY_HEADER_BYTES) // 4
    assert 3 * (share * 4 + bench.NPY_HEADER_BYTES) <= bench.DUMP_LIMIT_BYTES
