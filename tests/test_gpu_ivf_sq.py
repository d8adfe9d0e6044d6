"""IVF_SQ on the GPU, what only this kind has: the integer tensor-core scan kernel against NumPy integers, and the
rejections.  The search cases IVF_SQ shares with IVF_RQ and 4-bit IVF_PQ are in test_gpu_ivf_kinds.py."""
import ctypes as C

import numpy as np
import pytest

from lancedb_b200 import _native
from tests.sq_oracle import random_sq_index

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.mark.parametrize("B,N,dim", [(1, 1, 1), (7, 300, 7), (8, 257, 31), (9, 5000, 32), (130, 1000, 33),
                                     (33, 2000, 768), (5, 4099, 1000), (130, 5000, 64)])
def test_debug_sq_distances_equal_numpy_integers(B, N, dim):
    rng = np.random.default_rng(B * 1000 + dim)
    q = rng.integers(0, 256, (B, dim), dtype=np.uint8)
    x = rng.integers(0, 256, (N, dim), dtype=np.uint8)
    x[: min(N, 3)] = 255                                 # extreme rows
    got = _native.debug_sq_distances(q, x)
    qi, xi = q.astype(np.int64), x.astype(np.int64)
    want = (xi * xi).sum(1)[None, :] + (qi * qi).sum(1)[:, None] - 2 * (qi @ xi.T)
    assert np.array_equal(got.astype(np.int64), want)


def test_debug_sq_distances_above_2_31_wrap_exactly():
    # 65536 x 255^2 = 4261478400 > 2^31: the s32 accumulator wraps, the u32 result must not
    dim = 65536
    q = np.zeros((3, dim), np.uint8)
    q[1] = 255
    q[2, ::2] = 255
    x = np.full((5, dim), 255, np.uint8)
    x[1] = 0
    got = _native.debug_sq_distances(q, x).astype(np.int64)
    qi, xi = q.astype(np.int64), x.astype(np.int64)
    want = (xi * xi).sum(1)[None, :] + (qi * qi).sum(1)[:, None] - 2 * (qi @ xi.T)
    assert np.array_equal(got, want) and want.max() == 65536 * 65025


def test_ivf_sq_rejections():
    rng = np.random.default_rng(28)
    ix = random_sq_index(rng, n=500, dim=16, nlist=4)
    gpu = _native.GpuIvfSq(ix)
    with pytest.raises(ValueError, match="IVF_PQ"):
        gpu.debug_filter_bounds(ix.vectors[:2], 2, 10)
    with pytest.raises(ValueError, match="IVF_PQ"):
        gpu.debug_partition_distances(ix.vectors[0], 0, 10)
    gpu.close()
    # the C ABI itself rejects dot and dimensions above 65536
    lib = _native.load()
    c = np.zeros((1, 16), f32); off = np.zeros(2, np.uint64)
    for metric, dim in ((2, 16), (0, 65537)):
        desc = _native.SqDesc(_native.ABI_VERSION, dim, 1, metric, 0, 0, 0, 0.0, 1.0, c.ctypes.data, off.ctypes.data,
                              None, None, None)
        h = C.c_void_p()
        with pytest.raises(ValueError):
            _native.check(lib.lgpu_ivf_sq_open(C.byref(desc), C.byref(h)))
