"""IVF_RQ on the GPU, what only this kind has: the binary tensor-core scan kernel against NumPy integers and the
oracle's estimates, and the rejections.  The search cases IVF_RQ shares with IVF_SQ and 4-bit IVF_PQ are in
test_gpu_ivf_kinds.py."""
import ctypes as C

import numpy as np
import pytest

from lancedb_b200 import _native
from tests import rq_oracle
from tests.rq_oracle import random_rq_index, rq_estimates_np, rq_slot_np

pytestmark = pytest.mark.gpu
f32 = np.float32


@pytest.mark.parametrize("B,N,dim,metric", [(1, 1, 1, "l2"), (7, 300, 7, "cosine"), (8, 257, 255, "l2"),
                                            (9, 33, 256, "l2"), (13, 1000, 257, "cosine"), (33, 2000, 768, "l2"),
                                            (5, 4099, 1000, "cosine"), (3, 700, 4096, "l2")])
def test_debug_rq_distances_equal_numpy_and_oracle(B, N, dim, metric):
    rng = np.random.default_rng(B * 1000 + dim)
    q = rng.standard_normal((B, dim)).astype(f32)
    if B > 2:
        q[1] = 0.25                                       # delta = 0: every u is 0
        q[2, 0] = 1e30                                    # one huge component: the other u collapse to 0
    codes = rng.integers(0, 256, (N, (dim + 7) // 8), dtype=np.uint8)   # stray padding bits are cleared at open
    codes[: min(N, 2)] = 255
    add = (rng.random(N) * 10).astype(f32)
    scale = (-rng.random(N) * 3).astype(f32)
    est, ip = _native.debug_rq_distances(q, codes, add, scale, metric)
    zero = np.zeros(dim, f32)
    for b in range(B):
        u, lo, delta, qq, S = rq_slot_np(q[b], zero)
        want_ip = rq_estimates_np(codes, add, scale, u, lo, delta, qq, S, dim, ip_only=True)
        assert np.array_equal(ip[b].astype(np.int64), want_ip), b
        want = rq_estimates_np(codes, add, scale, u, lo, delta, qq, S, dim, metric)
        assert np.array_equal(est[b].view(np.uint32), want.view(np.uint32)), b
        if b < 2:                                         # the C oracle's own arithmetic on the first rows
            cu, clo, cdelta, cqq, cS = rq_oracle.rq_slot(q[b], zero)
            c = rq_oracle.rq_estimates(codes[:64], add[:64], scale[:64], cu, clo, cdelta, cqq, cS, dim, metric)
            assert np.array_equal(est[b, :64].view(np.uint32), c.view(np.uint32)), b


def test_debug_rq_distances_non_finite_slot_has_no_rows():
    dim, N = 40, 50
    rng = np.random.default_rng(3)
    q = rng.standard_normal((3, dim)).astype(f32)
    q[0, 4] = np.nan
    q[1, 5] = np.inf
    codes = rng.integers(0, 256, (N, 5), dtype=np.uint8)
    est, _ = _native.debug_rq_distances(q, codes, np.ones(N, f32), -np.ones(N, f32))
    assert np.isnan(est[:2]).all() and np.isfinite(est[2]).all()


def test_ivf_rq_rejections():
    rng = np.random.default_rng(38)
    ix = random_rq_index(rng, n=500, dim=16, nlist=4)
    gpu = _native.GpuIvfRq(ix)
    with pytest.raises(ValueError, match="IVF_PQ"):
        gpu.debug_filter_bounds(ix.vectors[:2], 2, 10)
    with pytest.raises(ValueError, match="IVF_PQ"):
        gpu.debug_partition_distances(ix.vectors[0], 0, 10)
    gpu.close()
    # the C ABI itself rejects dot, num_bits != 1, dimensions above 4096 and a missing rotation
    lib = _native.load()
    c = np.zeros((1, 16), f32); off = np.zeros(2, np.uint64); P = np.eye(16, dtype=f32)
    for metric, dim, bits, rot in ((2, 16, 1, P), (0, 16, 8, P), (0, 4097, 1, P), (0, 16, 1, None)):
        desc = _native.RqDesc(_native.ABI_VERSION, dim, 1, metric, 0, bits, 0, c.ctypes.data,
                              None if rot is None else rot.ctypes.data, off.ctypes.data, None, None, None, None, None)
        h = C.c_void_p()
        with pytest.raises(ValueError):
            _native.check(lib.lgpu_ivf_rq_open(C.byref(desc), C.byref(h)))
