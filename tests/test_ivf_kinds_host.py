"""Every IVF kind through Table.create_index and AsyncTable.create_index with the native handles stubbed: the index
is trained with the arguments given, keeps its vectors, is listed and described under its index_type, is opened by its
own handle class, and is refused by save_lance_index unless it is an 8-bit IVF_PQ index."""
import asyncio
from dataclasses import replace

import numpy as np
import pyarrow as pa
import pytest

import lancedb_b200 as lancedb
from lancedb_b200 import aio
from lancedb_b200.index import IVF_KINDS
from tests.util import record_opens

# index_type, Table.create_index arguments, the aio config with the same parameters (IVF_SQ has none), the handle
# class that opens the index, what the trained data must hold, and what save_lance_index's refusal names; every index
# has 3 partitions
CASES = [
    ("IVF_PQ", dict(metric="dot", num_sub_vectors=4, num_bits=4),
     aio.IvfPq(distance_type="dot", num_sub_vectors=4, num_bits=4), "GpuIvfPq", dict(metric="dot", m=4, num_bits=4),
     "8-bit"),
    ("IVF_SQ", dict(metric="cosine"), None, "GpuIvfSq", dict(metric="cosine"), "IVF_PQ"),
    ("IVF_HNSW_SQ", dict(metric="cosine", m=3, ef_construction=8),
     aio.HnswSq(distance_type="cosine", m=3, ef_construction=8), "GpuIvfHnswSq", dict(metric="cosine", m=3), "IVF_PQ"),
    ("IVF_RQ", dict(metric="cosine", num_bits=1), aio.IvfRq(distance_type="cosine"), "GpuIvfRq",
     dict(metric="cosine", num_bits=1), "IVF_PQ"),
    ("IVF_FLAT", dict(metric="hamming"), aio.IvfFlat(distance_type="hamming"), "GpuIvfBinary", dict(metric="hamming"),
     "IVF_PQ"),
]
ASYNC = [c for c in CASES if c[2] is not None]


@pytest.fixture
def opened(monkeypatch):
    return record_opens(monkeypatch)


def _table(kind):
    rng = np.random.default_rng(3)
    db = lancedb.connect("memory://")
    if kind != "IVF_FLAT":
        return db.create_table("t", {"vector": rng.standard_normal((300, 16)).astype(np.float32)})
    x = rng.integers(0, 256, (300, 4), dtype=np.uint8)
    schema = pa.schema([pa.field("vector", pa.list_(pa.uint8(), 4))])
    return db.create_table("t", pa.table({"vector": pa.FixedSizeListArray.from_arrays(pa.array(x.reshape(-1)), 4)},
                                         schema=schema))


def _check(t, opened, kind, handle, want, refusal):
    assert [name for name, _ in opened] == [handle]
    data = opened[0][1]
    assert isinstance(data, IVF_KINDS[kind].data) and data.index_type == kind and data.nlist == 3 and data.nrows == 300
    assert {a: getattr(data, a) for a in want} == want and data.vectors is not None
    assert t.list_indices() == [{"name": "vector_idx", "index_type": kind, "columns": ["vector"]}]
    st = t.index_stats("vector_idx")
    assert st["index_type"] == kind and st["distance_type"] == want["metric"] and st["num_indexed_rows"] == 300
    with pytest.raises(NotImplementedError, match=refusal):
        t.save_lance_index("/nonexistent")


@pytest.mark.parametrize("kind,args,config,handle,want,refusal", CASES, ids=[c[0] for c in CASES])
def test_table_create_index_trains_lists_and_opens_each_kind(opened, kind, args, config, handle, want, refusal):
    t = _table(kind)
    t.create_index(index_type=kind, num_partitions=3, max_iterations=2, **args)
    _check(t, opened, kind, handle, want, refusal)


@pytest.mark.parametrize("kind,args,config,handle,want,refusal", ASYNC, ids=[c[0] for c in ASYNC])
def test_async_create_index_trains_lists_and_opens_each_kind(opened, kind, args, config, handle, want, refusal):
    t = _table(kind)
    asyncio.run(aio.AsyncTable(t).create_index("vector", config=replace(config, num_partitions=3, max_iterations=2),
                                               accelerator=None))
    _check(t, opened, kind, handle, want, refusal)
