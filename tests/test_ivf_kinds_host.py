"""Every IVF kind through Table.create_index and AsyncTable.create_index with the native handles stubbed: the index
is trained with the arguments given, listed under its index_type, and opened by its own handle class."""
import asyncio
from dataclasses import replace

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import _native, aio

HANDLES = ("GpuIvfPq", "GpuIvfSq", "GpuIvfHnswSq", "GpuIvfRq", "GpuIvfBinary")

# index_type, Table.create_index arguments, the aio config with the same parameters (IVF_SQ has none), the handle
# class that opens the index, and what the trained data must hold; every index has 3 partitions
CASES = [
    ("IVF_PQ", dict(metric="dot", num_sub_vectors=4, num_bits=4),
     aio.IvfPq(distance_type="dot", num_sub_vectors=4, num_bits=4), "GpuIvfPq", dict(metric="dot", m=4, num_bits=4)),
    ("IVF_SQ", dict(metric="cosine"), None, "GpuIvfSq", dict(metric="cosine")),
    ("IVF_HNSW_SQ", dict(metric="cosine", m=3, ef_construction=8),
     aio.HnswSq(distance_type="cosine", m=3, ef_construction=8), "GpuIvfHnswSq", dict(metric="cosine", m=3)),
    ("IVF_RQ", dict(metric="cosine", num_bits=1), aio.IvfRq(distance_type="cosine"), "GpuIvfRq",
     dict(metric="cosine", num_bits=1)),
    ("IVF_FLAT", dict(metric="hamming"), aio.IvfFlat(distance_type="hamming"), "GpuIvfBinary", dict(metric="hamming")),
]
ASYNC = [c for c in CASES if c[2] is not None]


@pytest.fixture
def opened(monkeypatch):
    """Replaces every IVF handle class with a stub that records (its class name, the data it was opened with)."""
    log = []
    for name in HANDLES:
        def init(self, data, device=0, _name=name):
            log.append((_name, data))
        monkeypatch.setattr(_native, name, type(name, (), {"__init__": init, "close": lambda self: None}))
    return log


def _table(kind):
    rng = np.random.default_rng(3)
    db = lancedb.connect("memory://")
    if kind != "IVF_FLAT":
        return db.create_table("t", {"vector": rng.standard_normal((300, 16)).astype(np.float32)})
    x = rng.integers(0, 256, (300, 4), dtype=np.uint8)
    schema = pa.schema([pa.field("vector", pa.list_(pa.uint8(), 4))])
    return db.create_table("t", pa.table({"vector": pa.FixedSizeListArray.from_arrays(pa.array(x.reshape(-1)), 4)},
                                         schema=schema))


def _check(t, opened, kind, handle, want):
    assert [name for name, _ in opened] == [handle]
    data = opened[0][1]
    assert data.index_type == kind and data.nlist == 3 and data.nrows == 300
    assert {a: getattr(data, a) for a in want} == want
    assert t.list_indices() == [{"name": "vector_idx", "index_type": kind, "columns": ["vector"]}]
    assert t.index_stats("vector_idx")["index_type"] == kind


@pytest.mark.parametrize("kind,args,config,handle,want", CASES, ids=[c[0] for c in CASES])
def test_table_create_index_trains_lists_and_opens_each_kind(opened, kind, args, config, handle, want):
    t = _table(kind)
    t.create_index(index_type=kind, num_partitions=3, max_iterations=2, **args)
    _check(t, opened, kind, handle, want)


@pytest.mark.parametrize("kind,args,config,handle,want", ASYNC, ids=[c[0] for c in ASYNC])
def test_async_create_index_trains_lists_and_opens_each_kind(opened, kind, args, config, handle, want):
    t = _table(kind)
    asyncio.run(aio.AsyncTable(t).create_index("vector", config=replace(config, num_partitions=3, max_iterations=2),
                                               accelerator=None))
    _check(t, opened, kind, handle, want)
