"""The GPU index-training kernels against the exact Lloyd reference (tests/train_oracle.py), bit for bit.

lgpu_kmeans_train (csrc/kmeans.cu, assign_nearest in api.cu) and lgpu_pq_train produce the centroids and codebooks every
float index built with the accelerator is searched with.  The search oracle consumes whatever they produce, so a wrong
centre never shows up as a search mismatch; only these comparisons catch it.  Every case is rehearsed on the CPU by
tests/test_train_host.py, which checks that it reaches the branch it is named for.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from lancedb_b200 import _native
from tests import train_oracle as T

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(got, want, what):
    bad = np.argwhere(_bits(got) != _bits(want))
    assert bad.size == 0, (f"{what}: {len(bad)} values differ, first at {tuple(bad[0])}: "
                           f"{got[tuple(bad[0])]!r} != {want[tuple(bad[0])]!r}")


@pytest.mark.parametrize("name", list(T.KMEANS_CASES))
def test_kmeans_train_matches_exact_lloyd(name):
    x, init, iters = T.kmeans_case(name)
    got = _native.kmeans_train(x, init, iters)
    _same(got, T.lloyd(x, init, iters), name)
    if name == "empty":
        _same(got[5], init[5], "a centre no row reaches")
    if name == "tie":                                   # centre 41 = centre 7: every row of theirs goes to 7
        one = _native.kmeans_train(x, init, 1)
        _same(one, T.lloyd(x, init, 1), "tie, one iteration")
        _same(one[41], init[41], "the higher of two identical centres")
    if name == "iters0":                                # iters = 0 runs one iteration
        _same(got, _native.kmeans_train(x, init, 1), "iters 0 vs 1")


def test_kmeans_inertia_is_the_sum_of_nearest_distances():
    x, init, iters = T.kmeans_case("k300")
    c, got = _native.kmeans_train(x, init, iters, want_inertia=True)
    _same(c, T.lloyd(x, init, iters), "k300 with inertia")
    want = T.inertia(x, c)                              # f64 sums in another order: not bitwise
    assert abs(got - want) <= 1e-9 * want, (got, want)


_CHILD = """
import sys
import numpy as np
from lancedb_b200 import _native
from tests import train_oracle as T
out = {}
for name in sys.argv[2:]:
    x, init, iters = T.kmeans_case(name)
    out[name] = _native.kmeans_train(x, init, iters)
np.savez(sys.argv[1], **out)
"""


def test_kmeans_without_tensor_cores_gives_the_same_bits(tmp_path):
    """LGPU_NO_TENSOR_CORE=1 (read once per process) sends the assignment through the exact kernels: same centres"""
    names = ["k300", "k2048"]
    path = tmp_path / "notc.npz"
    env = dict(os.environ, PYTHONPATH=ROOT, LGPU_NO_TENSOR_CORE="1")
    r = subprocess.run([sys.executable, "-c", _CHILD, str(path), *names], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    z = np.load(path)
    for name in names:
        x, init, iters = T.kmeans_case(name)
        _same(z[name], _native.kmeans_train(x, init, iters), f"{name}: exact vs tensor-core assignment")


def test_kmeans_refusals():
    rng = np.random.default_rng(91)
    x = rng.standard_normal((300, 4097)).astype(np.float32)
    with pytest.raises(ValueError, match="dim <= 4096"):
        _native.kmeans_train(x, x[:8], 1)
    x = rng.standard_normal((300, 16)).astype(np.float32)
    with pytest.raises(ValueError):
        _native.kmeans_train(x, x[:0], 1)                                       # k = 0
    with pytest.raises(ValueError):
        _native.kmeans_train(x[:0], x[:8], 1)                                   # n = 0
    c = x[:8].copy()
    with pytest.raises(ValueError):                                            # null rows
        _native.check(_native.load().lgpu_kmeans_train(None, 300, 16, c.ctypes.data, 8, 1, 0, None))
    with pytest.raises(ValueError):                                            # null centres
        _native.check(_native.load().lgpu_kmeans_train(x.ctypes.data, 300, 16, None, 8, 1, 0, None))


@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf])
def test_training_refuses_non_finite_rows(value):
    """A NaN or infinite row would be summed into a centre or codeword and poison it; the C ABI names the row"""
    rng = np.random.default_rng(92)
    x = T.dyadic(rng, (500, 32))
    init = x[:16].copy()
    cb = np.ascontiguousarray(x[:256].reshape(256, 4, 8).transpose(1, 0, 2))
    x[137, 30] = value
    with pytest.raises(ValueError, match=r"training row 137 "):
        _native.kmeans_train(x, init, 2)
    with pytest.raises(ValueError, match=r"training row 137 "):
        _native.pq_train(x, cb, 2)


@pytest.mark.parametrize("name", list(T.PQ_CASES))
def test_pq_train_matches_exact_lloyd(name):
    x, cb, iters, _ = T.pq_case(name)
    got = _native.pq_train(x, cb, iters)
    _same(got, T.pq_lloyd(x, cb, iters), name)
    if name == "tie":
        _same(got[:, 200], cb[:, 200], "the higher of two identical codewords")


def test_pq_train_on_gaussian_data_is_within_one_ulp():
    """Codeword sums are f64 atomics in whatever order they run: on data that is not dyadic the f64 sum may differ in its
    last bits from the ascending-order one, and the rounded mean by one f32 ulp.  That is why the other cases use
    dyadic data, whose sums are exact in any order."""
    rng = np.random.default_rng(93)
    x = rng.standard_normal((3000, 32)).astype(np.float32)
    cb = np.ascontiguousarray(x[rng.choice(3000, 256, replace=False)].reshape(256, 4, 8).transpose(1, 0, 2))
    got, want = _native.pq_train(x, cb, 1), T.pq_lloyd(x, cb, 1)
    assert np.array_equal(np.sign(got), np.sign(want))
    ulps = np.abs(_bits(got).astype(np.int64) - _bits(want).astype(np.int64))
    assert ulps.max() <= 1, ulps.max()


def test_pq_train_refuses_an_unsupported_sub_vector_length():
    rng = np.random.default_rng(94)
    x = rng.standard_normal((300, 30)).astype(np.float32)
    with pytest.raises(ValueError, match="sub-vector length"):
        _native.pq_train(x, np.zeros((2, 256, 15), np.float32), 1)
